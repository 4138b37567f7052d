"""Device time of every weight-gradient launch of the benchmarked network (R50-I3D-NL, 2 clips of 32 x 224^2;
tests/wgrad_cases.py), for one or more builds of the library, in alternating rounds:

    python scripts/bench_wgrad.py --lib base=/path/libvlfb_base.so --lib new=/path/libvlfb.so [--rounds 2] [--iters 50]

Each round runs every library in its own process (the library is chosen with VLFB_LIB when it is loaded).  A launch is
timed with CUDA events around `iters` back-to-back launches after a warm-up; a library's time is its median over rounds.
Per launch the table gives ms, TFLOP/s of useful FLOPs, the launch's path record (tile width, stream-K, split, stages)
and the least time the hardware could take, max(FLOP / 495 TFLOP/s dense TF32, bytes / 3.35 TB/s), as a share of the
measured time.  Those are the H100 SXM data-sheet rates; the card's name and power limit are printed with the table."""
import argparse
import json
import os
import statistics
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (os.path.join(ROOT, 'video-long-term-feature-banks_b200', 'lib'), os.path.join(ROOT, 'tests')):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import wgrad_cases as WC  # noqa: E402

PEAK_TF32 = 495e12
PEAK_BW = 3.35e12


def child(iters, warmup):
    import torch
    import gemm_paths as GP
    from vlfb import kernels as K
    K.set_gemm_backend('tcgen05')
    dev = torch.device('cuda')
    gen = torch.Generator(device=dev).manual_seed(7)
    out = []
    for label, shape, co, ker, st, pd, dil, _ in WC.PRODUCTION:
        g = K.conv_geom(shape, co, ker, st, pd, dil)
        x = torch.randn(shape, device=dev, generator=gen)
        if shape[4] == 4:
            x[..., 3] = 0
        dy = torch.randn(K.out_shape(g), device=dev, generator=gen)
        dw = torch.zeros((co, ker[0], ker[1], 8 if shape[4] == 4 else ker[2], shape[4]), device=dev)
        fn = lambda: K.conv_wgrad(dy, x, dw, g)   # noqa: E731
        _, text = GP.capture_fd2(lambda: (fn(), torch.cuda.synchronize()))
        recs = [r for r in (GP.parse_record(l) for l in text.splitlines()) if r is not None]
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(dict(label=label, ms=e0.elapsed_time(e1) / iters, rec=recs[0] if recs else None))
        del x, dy, dw
    print('BENCH_WGRAD ' + json.dumps(out), flush=True)


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return q[0] if q else 'unknown'
    except (OSError, subprocess.TimeoutExpired):
        return 'unknown'


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--lib', action='append', default=[], metavar='NAME=PATH', help='library build (repeatable)')
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--json', default='', help='also write the results here')
    ap.add_argument('--child', action='store_true', help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args.iters, args.warmup)
    if args.iters < 50:
        raise SystemExit('--iters must be >= 50')
    libs = [tuple(s.split('=', 1)) for s in args.lib] or [('default', '')]
    print('card (name, power limit, max SM clock): %s' % card(), flush=True)
    runs = dict((n, []) for n, _ in libs)
    for r in range(args.rounds):
        for name, path in libs:
            env = dict(os.environ)
            env.pop('VLFB_LIB', None)
            if path:
                env['VLFB_LIB'] = os.path.abspath(path)
            env['VLFB_DEBUG'] = '1'
            cmd = [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [
                os.path.abspath(__file__), '--child', '--iters', str(args.iters), '--warmup', str(args.warmup)]
            p = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True)
            line = [l for l in p.stdout.splitlines() if l.startswith('BENCH_WGRAD ')]
            if p.returncode != 0 or not line:
                raise SystemExit('%s round %d failed (exit %d):\n%s' % (name, r, p.returncode, p.stderr[-3000:]))
            runs[name].append(json.loads(line[0][len('BENCH_WGRAD '):]))
    res = {}
    for name, _ in libs:
        rows = []
        for i, (label, shape, co, ker, st, pd, dil, count) in enumerate(WC.PRODUCTION):
            ms = statistics.median(run[i]['ms'] for run in runs[name])
            fl, by = WC.useful_flops(shape, co, ker, st, pd, dil), WC.min_bytes(shape, co, ker, st, pd, dil)
            lb = max(fl / PEAK_TF32, by / PEAK_BW) * 1e3
            rec = runs[name][0][i]['rec'] or {}
            rows.append(dict(label=label, count=count, ms=ms, spread=max(run[i]['ms'] for run in runs[name]) -
                             min(run[i]['ms'] for run in runs[name]), tflops=fl / ms * 1e-9, bound_ms=lb,
                             co_le_64=co <= 64,
                             rec=dict((k, rec.get(k)) for k in ('bn', 'wide', 'sk', 'split', 'stages', 'tiles'))))
        res[name] = rows
    names = [n for n, _ in libs]
    print('%-34s %3s ' % ('launch', 'n') + ' '.join('%24s' % ('%s ms  TF/s  %%bound' % n) for n in names) +
          '  path (%s)' % names[-1])
    for i in range(len(WC.PRODUCTION)):
        r0 = res[names[-1]][i]
        cols = ' '.join('%10.3f %6.1f %5.1f%%' % (res[n][i]['ms'], res[n][i]['tflops'], 100 * res[n][i]['bound_ms'] / res[n][i]['ms'])
                        for n in names)
        print('%-34s %3d %s  bn=%s wide=%s sk=%s split=%s stages=%s tiles=%s' % (
            r0['label'], r0['count'], cols, *[r0['rec'][k] for k in ('bn', 'wide', 'sk', 'split', 'stages', 'tiles')]))
    for grp, sel in (('Co <= 64', True), ('Co > 64', False)):
        tot = ' '.join('%s %.3f ms' % (n, sum(r['ms'] * r['count'] for r in res[n] if r['co_le_64'] == sel)) for n in names)
        print('per step, %s: %s' % (grp, tot))
    print('per step, all wgrad: ' + ' '.join('%s %.3f ms' % (n, sum(r['ms'] * r['count'] for r in res[n])) for n in names))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(dict(card=card(), results=res), f, indent=1)


if __name__ == '__main__':
    main()
