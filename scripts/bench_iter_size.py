"""What B200.ITER_SIZE costs: gradient accumulation over k micro-steps against one update per step.

bench.py's training step (config 2: R50-I3D-NL + FBO-NL-2L, 2 clips of 32 x 224^2 per micro-step, R = 4 boxes, L = 300
bank rows), in ROUNDS alternating rounds of two sessions:
  k=1  ITER_SIZE 1, NUM_GPUS 1: every RunNet is a whole step (forward + backward + SGD)
  k=4  ITER_SIZE 4, NUM_GPUS 4: four micro-steps per iteration; three replay forward + backward only, the fourth (the
       boundary) also runs the SGD graph
Each session: WARMUP untimed iterations (at least the two eager runs and the capture), then ITERS iterations, every
RunNet between CUDA events (the replays are device-bound); peak device memory of the session.

    python scripts/bench_iter_size.py [--rounds 3] [--iters 10] [--warmup 2] [--out FILE.json]

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


def _session(k, warmup, iters):
    import harness as H
    from oracle import model as OM
    from vlfb import workspace
    workspace.ResetWorkspace()
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    ov = ['NUM_GPUS', k, 'TRAIN.BATCH_SIZE', 2 * k, 'TEST.BATCH_SIZE', 2 * k, 'B200.ITER_SIZE', k]
    H.setup_cfg(YAML, ov)
    ocfg = H.oracle_cfg(YAML, ov)
    model, sfx = H.build('train', True)
    H.feed_params(OM.make_params(ocfg, seed=2))
    H.feed_inputs(OM.make_inputs(ocfg, n_clips=2, rois_per_clip=2, seed=100), sfx)
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default='')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_iter_size: no GPU')
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip()
    print(card, flush=True)
    runs = {1: [], 4: []}
    for rnd in range(a.rounds):
        for k in (1, 4):
            res = _session(k, a.warmup, a.iters)
            runs[k].append(res)
            print('round %d k=%d  %8.2f ms/iteration  boundary %7.2f ms  non-boundary %s ms  graphs %d  peak %.0f MiB  '
                  'loss finite %s' % (rnd, k, res['iter_ms'], res['boundary_ms'],
                                      '-' if res['micro_ms'] is None else '%7.2f' % res['micro_ms'], res['graphs'],
                                      res['peak_mib'], res['loss_finite']), flush=True)
    summary = {'card': card}
    for k, rs in runs.items():
        summary['k=%d' % k] = dict(
            iter_ms=float(np.median([r['iter_ms'] for r in rs])), boundary_ms=float(np.median([r['boundary_ms'] for r in rs])),
            micro_ms=None if k == 1 else float(np.median([r['micro_ms'] for r in rs])),
            peak_mib=max(r['peak_mib'] for r in rs), rounds=rs)
    s1, s4 = summary['k=1'], summary['k=4']
    print('median: k=1 %.2f ms/step; k=4 %.2f ms/iteration (non-boundary micro-step %.2f ms, boundary %.2f ms) = %.3f x '
          '4 steps; SGD pass ~ %.2f ms; peak %.0f vs %.0f MiB' % (
              s1['iter_ms'], s4['iter_ms'], s4['micro_ms'], s4['boundary_ms'], s4['iter_ms'] / (4 * s1['iter_ms']),
              s4['boundary_ms'] - s4['micro_ms'], s1['peak_mib'], s4['peak_mib']))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(summary, f, indent=1)


if __name__ == '__main__':
    main()
