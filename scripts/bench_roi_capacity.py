"""What B200.ROI_CAPACITY buys on a varying-box workload, and what its padding costs.

bench.py's training step (config 2: R50-I3D-NL + FBO-NL-2L, 2 clips of 32 x 224^2, L = 300 bank rows) fed a new batch
every step, in ROUNDS alternating rounds of five sessions:
  seq/C=0   r drawn uniformly from 2..24 per step (seeded), today's behaviour: the RoI count is part of the graph key
  seq/C=24  the same r sequence with a 24-row capacity: one captured graph
  r4/C=0    r = 4 every step (bench.py's workload)
  r4/C=4    the same with a capacity that is never padded
  r4/C=24   the same at a 24-row capacity: 20 padded rows per step
Each session: WARMUP untimed steps, then STEPS steps timed on the host clock up to a device synchronise (eager steps are
host-bound, so device events alone would understate them); graph captures and eager runs counted in the timed window;
peak device memory of the session.  AVA batches vary R every step, so a real run of the C = 0 net mostly runs eagerly or
recaptures; the sequence sessions measure that.

    python scripts/bench_roi_capacity.py [--rounds 3] [--steps 40] [--warmup 5] [--out FILE.json]

Prints the card name and power limit first: the numbers belong to them."""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'video-long-term-feature-banks_b200', 'lib')):
    sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

YAML = 'ava_r50_lfb_nl.yaml'
OV = ['NUM_GPUS', 1, 'TRAIN.BATCH_SIZE', 2]          # bench.py's configuration
MAX_R = 24
PER_ROI = ('proposals', 'labels', 'lfb')


def _session(cap, rows, warmup, steps):
    import harness as H
    from oracle import model as OM
    from vlfb import workspace
    workspace.ResetWorkspace()
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    H.setup_cfg(YAML, OV + ['B200.ROI_CAPACITY', cap])
    ocfg = H.oracle_cfg(YAML, OV)
    model, sfx = H.build('train', True)
    H.feed_params(OM.make_params(ocfg, seed=2))
    workspace.FeedBlob('gpu_0/lr', np.array(1e-4, dtype=np.float32))
    name = model.net.Proto().name
    net = workspace.current().nets[name]
    inputs = OM.make_inputs(ocfg, n_clips=2, rois_per_clip=MAX_R // 2, seed=100)
    host = dict((k, v.contiguous().pin_memory()) for k, v in inputs.items())
    count = {'capture': 0, 'replay': 0}
    capture, replay = net._capture, net._replay

    def counted_capture():
        count['capture'] += 1
        return capture()

    def counted_replay(entry):
        count['replay'] += 1
        return replay(entry)
    net._capture, net._replay = counted_capture, counted_replay

    def step(r):
        for k, v in host.items():
            workspace.FeedBlob('gpu_0/%s%s' % (k, sfx), v[:r] if k in PER_ROI else v)
        workspace.RunNet(name)

    for r in rows[:warmup]:
        step(r)
    torch.cuda.synchronize()
    count['capture'] = count['replay'] = 0
    t0 = time.perf_counter()
    for r in rows[warmup:warmup + steps]:
        step(r)
    loss = float(workspace.FetchBlob('gpu_0/loss'))
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    res = dict(ms=ms, captures=count['capture'], eager=steps - count['replay'], graphs=len(net._graphs),
               peak_gib=torch.cuda.max_memory_allocated() / 2.0 ** 30, loss_finite=bool(np.isfinite(loss)))
    net._capture, net._replay = capture, replay
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=40)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--out', default='')
    a = ap.parse_args()
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip()
    print(card, flush=True)
    n = a.warmup + a.steps
    seq = [int(v) for v in np.random.RandomState(0).randint(2, MAX_R + 1, size=n)]
    sessions = [('seq/C=0', 0, seq), ('seq/C=24', 24, seq), ('r4/C=0', 0, [4] * n), ('r4/C=4', 4, [4] * n),
                ('r4/C=24', 24, [4] * n)]
    runs = dict((s[0], []) for s in sessions)
    for rnd in range(a.rounds):
        for label, cap, rows in sessions:
            res = _session(cap, rows, a.warmup, a.steps)
            runs[label].append(res)
            print('round %d %-9s %7.2f ms/step  captures %2d  eager %2d  graphs %d  peak %.2f GiB  loss finite %s' % (
                rnd, label, res['ms'], res['captures'], res['eager'], res['graphs'], res['peak_gib'], res['loss_finite']),
                flush=True)
    summary = {}
    for label in runs:
        ms = [r['ms'] for r in runs[label]]
        summary[label] = dict(median_ms=float(np.median(ms)), ms=ms, captures=[r['captures'] for r in runs[label]],
                              eager=[r['eager'] for r in runs[label]],
                              peak_gib=max(r['peak_gib'] for r in runs[label]))
        print('%-9s median %.2f ms/step (%s)' % (label, summary[label]['median_ms'], ' '.join('%.2f' % v for v in ms)))
    print('varying r: C=24 vs C=0 speed-up %.2fx' % (summary['seq/C=0']['median_ms'] / summary['seq/C=24']['median_ms']))
    print('r = 4: C=4 vs C=0 %+.1f %%, C=24 vs C=0 %+.1f %%' % (
        100.0 * (summary['r4/C=4']['median_ms'] / summary['r4/C=0']['median_ms'] - 1.0),
        100.0 * (summary['r4/C=24']['median_ms'] / summary['r4/C=0']['median_ms'] - 1.0)))
    out = dict(card=card, sequence=seq, warmup=a.warmup, steps=a.steps, sessions=summary)
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
