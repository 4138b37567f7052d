"""What B200.GPUS_PER_STEP buys: four virtual GPUs per iteration packed v to a step, k = 4 / v steps per iteration.

bench.py's workload per virtual GPU (config 2: R50-I3D-NL + FBO-NL-2L, 2 clips of 32 x 224^2, R = 4 boxes, L = 300 bank
rows), NUM_GPUS = 4, in ROUNDS alternating rounds of three sessions:
  v=1 k=4  ITER_SIZE 4: four 2-clip micro-steps per iteration (the boundary one also runs the SGD graph)
  v=2 k=2  GPUS_PER_STEP 2, ITER_SIZE 2: two 4-clip steps per iteration
  v=4 k=1  GPUS_PER_STEP 4: one 8-clip step per iteration
Each session: WARMUP untimed iterations (at least the two eager runs and the capture), then ITERS iterations, every
RunNet a graph replay between CUDA events; peak device memory of the session.  Then the tensor-core GEMM tiles of one
eager step per network stage at v = 1 and v = 4 (the tiling vlfb_gemm_plan reports for every vlfb_gemm launch, on 132
SMs), which show how far the packed step's GEMMs fill the H100.

    python scripts/bench_gpus_per_step.py [--rounds 3] [--iters 10] [--warmup 2] [--out FILE.json]

Prints the card name and power limit first: the numbers belong to them."""
import argparse
import gc
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'video-long-term-feature-banks_b200', 'lib')):
    sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

YAML = 'ava_r50_lfb_nl.yaml'


def _session(v, k, warmup, iters):
    import harness as H
    from oracle import model as OM
    from vlfb import workspace
    workspace.ResetWorkspace()
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    ov = ['NUM_GPUS', v * k, 'TRAIN.BATCH_SIZE', 2 * v * k, 'TEST.BATCH_SIZE', 2 * v * k, 'B200.ITER_SIZE', k,
          'B200.GPUS_PER_STEP', v]
    H.setup_cfg(YAML, ov)
    ocfg = H.oracle_cfg(YAML, ov)
    model, sfx = H.build('train', True)
    H.feed_params(OM.make_params(ocfg, seed=2))
    H.feed_inputs(OM.make_inputs(ocfg, n_clips=2 * v, rois_per_clip=2, seed=100), sfx)
    workspace.FeedBlob('gpu_0/lr', np.array(1e-4, dtype=np.float32))
    name = model.net.Proto().name
    net = workspace.current().nets[name]
    for _ in range(max(warmup * k, 3)):              # two eager runs and the capture stay out of the timed window
        workspace.RunNet(name)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(iters * k + 1)]
    ev[0].record()
    for i in range(iters * k):
        workspace.RunNet(name)
        ev[i + 1].record()
    loss = float(workspace.FetchBlob('gpu_0/loss'))
    torch.cuda.synchronize()
    ms = [ev[i].elapsed_time(ev[i + 1]) for i in range(iters * k)]
    boundary = [m for i, m in enumerate(ms) if i % k == k - 1]
    inner = [m for i, m in enumerate(ms) if i % k != k - 1]
    res = dict(iter_ms=sum(ms) / iters, boundary_ms=float(np.mean(boundary)),
               micro_ms=float(np.mean(inner)) if inner else None, graphs=len(net._graphs),
               peak_mib=torch.cuda.max_memory_allocated() / 2.0 ** 20, loss_finite=bool(np.isfinite(loss)))
    workspace.ResetWorkspace()
    return res


def _tile_counts(v):
    """stage -> [GEMM launches, output tiles, launches with fewer tiles than 132 SMs] of one eager step at v x 2 clips."""
    import ctypes as C
    import harness as H
    from bench import stage_of
    from oracle import model as OM
    from vlfb import kernels as K, libvlfb as L, workspace
    workspace.ResetWorkspace()
    ov = ['NUM_GPUS', v, 'TRAIN.BATCH_SIZE', 2 * v, 'TEST.BATCH_SIZE', 2 * v, 'B200.GPUS_PER_STEP', v]
    H.setup_cfg(YAML, ov)
    ocfg = H.oracle_cfg(YAML, ov)
    model, sfx = H.build('train', True)
    H.feed_params(OM.make_params(ocfg, seed=2))
    H.feed_inputs(OM.make_inputs(ocfg, n_clips=2 * v, rois_per_clip=2, seed=100), sfx)
    workspace.FeedBlob('gpu_0/lr', np.array(1e-4, dtype=np.float32))
    counts = {}
    run_gemm = K._run_gemm

    def counted(p, *a, **kw):
        plan = L.GemmPlan()
        if L.load().vlfb_gemm_plan(C.byref(p), 132, C.byref(plan)) == 0:
            c = counts.setdefault(stage_of(K.LABEL), [0, 0, 0])
            c[0] += 1
            c[1] += plan.tiles
            c[2] += plan.tiles < 132
        return run_gemm(p, *a, **kw)

    workspace.current().force_eager = True
    K._run_gemm = counted
    try:
        workspace.RunNet(model.net.Proto().name)
        torch.cuda.synchronize()
    finally:
        K._run_gemm = run_gemm
        workspace.ResetWorkspace()
    return counts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default='')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_gpus_per_step: no GPU')
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip()
    print(card, flush=True)
    shapes = ((1, 4), (2, 2), (4, 1))
    runs = dict((vk, []) for vk in shapes)
    for rnd in range(a.rounds):
        for v, k in shapes:
            res = _session(v, k, a.warmup, a.iters)
            runs[(v, k)].append(res)
            print('round %d v=%d k=%d  %8.2f ms/iteration  graphs %d  peak %.0f MiB  loss finite %s' % (
                rnd, v, k, res['iter_ms'], res['graphs'], res['peak_mib'], res['loss_finite']), flush=True)
    summary = {'card': card}
    for (v, k), rs in runs.items():
        summary['v=%d k=%d' % (v, k)] = dict(iter_ms=float(np.median([r['iter_ms'] for r in rs])),
                                             peak_mib=max(r['peak_mib'] for r in rs), rounds=rs)
    base = summary['v=1 k=4']['iter_ms']
    print('median ms/iteration (4 virtual GPUs): ' + '; '.join(
        '%s %.2f (%.3fx of v=1)' % (key, summary[key]['iter_ms'], summary[key]['iter_ms'] / base)
        for key in ('v=1 k=4', 'v=2 k=2', 'v=4 k=1')) + '; peak MiB ' + ', '.join(
        '%.0f' % summary[key]['peak_mib'] for key in ('v=1 k=4', 'v=2 k=2', 'v=4 k=1')), flush=True)
    tiles = dict((v, _tile_counts(v)) for v in (1, 4))
    summary['gemm_tiles'] = dict(('v=%d' % v, t) for v, t in tiles.items())
    print('GEMM tiles per step by stage (launches, tiles, launches under 132 tiles): ' + '; '.join(
        '%s v=1 %d/%d/%d v=4 %d/%d/%d' % ((st,) + tuple(tiles[1].get(st, [0] * 3)) + tuple(tiles[4].get(st, [0] * 3)))
        for st in sorted(set(tiles[1]) | set(tiles[4]))), flush=True)
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(summary, f, indent=1)


if __name__ == '__main__':
    main()
