"""Cost of B200.COMPUTE 'tf32x3': bench.py's training step (ava_r50_lfb_nl.yaml, 2 clips of 32 x 224^2, R = 4 RoIs,
L = 300 bank rows, the yaml's dropout, graph replay) in 'tf32' and 'tf32x3' mode, in one process, alternating: ROUNDS
rounds of WARMUP warm-up and STEPS timed steps per mode (CUDA events around the replays).  Also records each mode's
peak device memory and its last step's loss and `pred`, and the card's name, power limit and maximum SM clock.

    python scripts/bench_compute_mode.py OUT_DIR [--rounds 3] [--warmup 3] [--steps 10]

Writes OUT_DIR/compute_mode.json and OUT_DIR/pred_<mode>.npy, and prints a summary.  Needs a GPU."""
import argparse
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
MODES = ('tf32', 'tf32x3')
OV = ['NUM_GPUS', 1, 'TRAIN.BATCH_SIZE', 2]


def _session(mode):
    """A fresh workspace holding bench.py's net in `mode`, fed with its weights and inputs.  (One workspace cannot
    hold both: the two modes store the same input blobs differently.)"""
    import harness as H
    from core.config import config as cfg
    from oracle import model as OM
    from vlfb import workspace
    workspace.ResetWorkspace()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    ov = OV + ['B200.COMPUTE', mode]
    H.setup_cfg(YAML, ov)
    cfg.RNG_SEED = 2
    model, sfx = H.build('train', True)
    ocfg = H.oracle_cfg(YAML, ov)
    H.feed_params(OM.make_params(ocfg, seed=2))
    workspace.FeedBlob('gpu_0/lr', np.array(1e-4, dtype=np.float32))
    for k, v in OM.make_inputs(ocfg, n_clips=2, rois_per_clip=2, seed=100).items():
        workspace.FeedBlob('gpu_0/%s%s' % (k, sfx), v)
    return workspace, model.net.Proto().name


def _round(mode, warmup, steps):
    ws, name = _session(mode)
    for _ in range(warmup):                 # eager, eager (grad-finish fusion), capture + replay
        ws.RunNet(name)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        ws.RunNet(name)
    e1.record()
    torch.cuda.synchronize()
    return dict(ms=e0.elapsed_time(e1) / steps, peak_bytes=int(torch.cuda.max_memory_allocated()),
                loss=float(ws.FetchBlob('gpu_0/loss')), pred=ws.FetchBlob('gpu_0/pred').copy())


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('out_dir')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--steps', type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_compute_mode.py needs a CUDA device')
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(card)
    res = dict((m, []) for m in MODES)
    for r in range(a.rounds):
        for m in MODES:
            res[m].append(_round(m, a.warmup, a.steps))
            print('round %d %-6s %.2f ms/step' % (r, m, res[m][-1]['ms']), flush=True)
    os.makedirs(a.out_dir, exist_ok=True)
    out = dict(card=card, workload='%s: 2 clips 32x224^2, R=4, L=300, fwd+bwd+SGD, graph replay' % YAML,
               rounds=a.rounds, warmup=a.warmup, steps=a.steps, modes={})
    for m in MODES:
        ms = [x['ms'] for x in res[m]]
        out['modes'][m] = dict(step_ms=ms, median_ms=float(np.median(ms)),
                               peak_mib=max(x['peak_bytes'] for x in res[m]) / 2.0 ** 20, loss=res[m][-1]['loss'])
        np.save(os.path.join(a.out_dir, 'pred_%s.npy' % m), res[m][-1]['pred'])
        print('%-6s step ms %s (median %.2f), peak %.0f MiB, last loss %.6f' % (
            m, ' '.join('%.2f' % v for v in ms), out['modes'][m]['median_ms'], out['modes'][m]['peak_mib'],
            out['modes'][m]['loss']))
    out['ratio'] = out['modes']['tf32x3']['median_ms'] / out['modes']['tf32']['median_ms']
    p0, p1 = res['tf32'][-1]['pred'], res['tf32x3'][-1]['pred']
    out['pred_rel_diff'] = float(np.abs(p1 - p0).max() / max(np.abs(p1).max(), 1e-30))
    print('tf32x3 / tf32 step time: %.2fx; last pred differs by %.2e (max-norm)' % (out['ratio'], out['pred_rel_diff']))
    with open(os.path.join(a.out_dir, 'compute_mode.json'), 'w') as f:
        json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
