"""Device time of split-TF32 GEMMs (precision = VLFB_PREC_X3) against TF32 ones at the production convolution shapes of
bench.py's network (2 clips): forward, dgrad and wgrad of each layer, TF32 and X3 alternating over 3 rounds.  Each entry
is the mean of REPS back-to-back launches between CUDA events after 3 warm-up launches.  Prints the card name and its
power limit, read in the same run, then one line per shape and a JSON summary line.

    python scripts/bench_gemm_x3.py
"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'video-long-term-feature-banks_b200', 'lib'))
sys.path.insert(0, os.path.join(ROOT, 'scripts'))
from bench_gemm_shapes import CONVS  # noqa: E402
from vlfb import kernels as K  # noqa: E402
from vlfb import libvlfb as L  # noqa: E402

REPS = int(os.environ.get('REPS', '10'))
ROUNDS = 3


def timed(fn):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(REPS):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / REPS * 1e3      # us


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as ex:
        out = 'nvidia-smi unavailable (%s)' % ex
    return out or torch.cuda.get_device_name()


def main():
    assert torch.cuda.is_available(), 'this benchmark needs a GPU'
    print('card:', card(), flush=True)
    rows = []
    for name, ci, co, ker, pads, dil, (n, t, h, w) in CONVS:
        g = K.conv_geom((n, t, h, w, ci), co, ker, (1, 1, 1), pads, dil)
        x = torch.randn((n, t, h, w, ci), device='cuda')
        wt5 = torch.randn((co,) + tuple(ker) + (ci,), device='cuda') * 0.05
        y = torch.empty(K.out_shape(g), device='cuda')
        dy = torch.randn(K.out_shape(g), device='cuda')
        wt = torch.empty((ci,) + tuple(ker) + (co,), device='cuda')
        K.weight_transpose(wt5, wt, precision=L.PREC_X3)
        dx = torch.empty_like(x)
        dw = torch.zeros_like(wt5)
        ops = {'fwd': lambda pr: K.conv_fwd(x, wt5, y, g, precision=pr),
               'dgrad': lambda pr: K.conv_dgrad(dy, wt, dx, g, precision=pr),
               'wgrad': lambda pr: K.conv_wgrad(dy, x, dw, g, precision=pr)}
        for op, fn in ops.items():
            t = {L.PREC_TF32: [], L.PREC_X3: []}
            for _ in range(ROUNDS):
                for pr in (L.PREC_TF32, L.PREC_X3):
                    t[pr].append(timed(lambda: fn(pr)))
            tf, x3 = sorted(t[L.PREC_TF32])[1], sorted(t[L.PREC_X3])[1]
            rows.append(dict(shape=name, op=op, tf32_us=round(tf, 1), x3_us=round(x3, 1), ratio=round(x3 / tf, 2)))
            print('%-26s %-5s tf32 %8.1f us  x3 %8.1f us  x%.2f' % (name, op, tf, x3, x3 / tf), flush=True)
    tot = dict((k, round(sum(r[k] for r in rows), 1)) for k in ('tf32_us', 'x3_us'))
    by_op = dict((op, round(sum(r['x3_us'] for r in rows if r['op'] == op) /
                            sum(r['tf32_us'] for r in rows if r['op'] == op), 2)) for op in ('fwd', 'dgrad', 'wgrad'))
    print(json.dumps(dict(card=card(), reps=REPS, rounds=ROUNDS, total=tot, ratio=round(tot['x3_us'] / tot['tf32_us'], 2),
                          ratio_by_op=by_op)))


if __name__ == '__main__':
    main()
