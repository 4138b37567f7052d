"""Cost of B200.DETERMINISTIC: the benchmarked training step (bench.py's network, 2 clips of 32 x 224^2) in default and
deterministic mode, alternating, ROUNDS rounds of STEPS timed steps each (CUDA events around graph replays), plus the
GEMM time per kind from one profiled step of each mode and the launches whose schedule differs between them.

    python scripts/bench_deterministic.py [--rounds 3] [--steps 10]

Prints the card name and power limit first: the numbers belong to them."""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'video-long-term-feature-banks_b200', 'lib')):
    sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

FULL = ['NUM_GPUS', 1, 'TRAIN.BATCH_SIZE', 2, 'TRAIN.DROPOUT_RATE', 0.0, 'FBO_NL.INPUT_DROPOUT_ON', False,
        'FBO_NL.LFB_DROPOUT_ON', False]


def _session(det):
    import harness as H
    from oracle import model as OM
    from vlfb import workspace
    workspace.ResetWorkspace()
    ov = FULL + ['B200.DETERMINISTIC', det]
    H.setup_cfg('ava_r50_lfb_nl.yaml', ov)
    ocfg = H.oracle_cfg('ava_r50_lfb_nl.yaml', ov)
    params = OM.make_params(ocfg, seed=2)
    inputs = OM.make_inputs(ocfg, n_clips=2, rois_per_clip=2, crop=224, frames=32)
    model, sfx = H.build('train', True)
    H.feed_params(params)
    H.feed_inputs(inputs, sfx)
    model.UpdateWorkspaceLr(10)
    name = model.net.Proto().name
    for _ in range(3):                      # eager, eager (grad-finish fusion), capture
        workspace.RunNet(name)
    torch.cuda.synchronize()
    return workspace, name


def _time(det, steps):
    ws, name = _session(det)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        ws.RunNet(name)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def _gemm_kinds(det):
    """ms per GEMM kind in one eager step, and the GEMM launch records (VLFB_DEBUG child process)."""
    from vlfb import kernels as K
    ws, name = _session(det)
    K._PROFILE = []
    ws.current().force_eager = True
    ws.RunNet(name)
    ws.current().force_eager = False
    prof, K._PROFILE = K._PROFILE, None
    torch.cuda.synchronize()
    by = {}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for label, fn, *_ in prof:
        fn()
        e0.record()
        for _ in range(3):
            fn()
        e1.record()
        torch.cuda.synchronize()
        kind = label.split()[0]
        by[kind] = by.get(kind, 0.0) + e0.elapsed_time(e1) / 3
    return by


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--records', action='store_true', help='(child) print the VLFB_DEBUG records of one eager step')
    a = ap.parse_args()
    if a.records:
        from vlfb import workspace
        for det in (False, True):
            print('MODE', int(det), file=sys.stderr, flush=True)     # in the stream the library's records go to
            ws, name = _session(det)
            ws.current().force_eager = True
            ws.RunNet(name)
            torch.cuda.synchronize()
            ws.current().force_eager = False
        return
    print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip())
    t = {False: [], True: []}
    for r in range(a.rounds):
        for det in (False, True):
            t[det].append(_time(det, a.steps))
    for det in (False, True):
        print('%-13s step ms: %s  (median %.2f)' % ('deterministic' if det else 'default',
                                                   ' '.join('%.2f' % v for v in t[det]), float(np.median(t[det]))))
    print('cost of the deterministic mode: %+.1f %%' % (100.0 * (np.median(t[True]) / np.median(t[False]) - 1.0)))
    for det in (False, True):
        by = _gemm_kinds(det)
        print('%-13s GEMM ms per kind: %s' % ('deterministic' if det else 'default',
                                              ' '.join('%s=%.2f' % kv for kv in sorted(by.items()))))
    env = dict(os.environ, VLFB_DEBUG='1')
    r = subprocess.run([sys.executable, os.path.abspath(__file__), '--records'], env=env, capture_output=True, text=True)
    import gemm_paths as GP
    recs, mode = {0: [], 1: []}, 0
    for line in r.stderr.splitlines():
        if line.startswith('MODE'):
            mode = int(line.split()[1])
        rec = GP.parse_record(line)
        if rec:
            recs[mode].append(rec)
    keys = ('split', 'sk', 'fix', 'bn', 'wide', 'units')
    changed = 0
    for r0, r1 in zip(recs[0], recs[1]):
        if any(r0.get(k) != r1.get(k) for k in keys):
            changed += 1
            print('  M=%d N=%d K=%d z=%d: %s -> %s' % (r0['M'], r0['N'], r0['K'], r0['z'],
                                                     ' '.join('%s=%s' % (k, r0.get(k)) for k in keys),
                                                     ' '.join('%s=%s' % (k, r1.get(k)) for k in keys)))
    print('launches whose schedule changed: %d of %d' % (changed, len(recs[0])))
    if not recs[0] or r.returncode != 0:
        raise SystemExit('the launch-record pass failed (exit %d): %s' % (r.returncode, r.stderr[-2000:]))


if __name__ == '__main__':
    main()
