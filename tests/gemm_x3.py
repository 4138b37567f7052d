"""Split-TF32 GEMM (vlfb_gemm_params_t.precision = VLFB_PREC_X3) against fp64: the path table of tests/gemm_paths.py and
seeded draws of tests/gemm_fuzz.py, run in split mode on operands that are NOT rounded to TF32.

    VLFB_DEBUG=1 python tests/gemm_x3.py --config NAME [--seed S --count N] --out FILE

In this process every vlfb_gemm call carries precision = VLFB_PREC_X3 (set at the C ABI boundary, so the wrappers and
the raw cases alike), the dgrad weight operand is transposed without rounding, the case operands are plain fp32 draws
and the elementwise bound of gemm_paths.finish is tau_x3(K) instead of tau(K):

  a = a_hi + a_lo and b = b_hi + b_lo with x_hi = x truncated to TF32, so |x_lo| < 2^-10 |x|.  The kernel sums
  a_hi b_hi + a_hi trunc(b_lo) + trunc(a_lo) b_hi, whose distance from a b is at most
  |a_lo b_lo| + |a_hi (b_lo - trunc(b_lo))| + |(a_lo - trunc(a_lo)) b_hi| < 3 * 2^-20 |a b|
  (truncating a lo part to TF32 loses < 2^-10 of it).  The fp32 accumulation adds three MMAs per k8 step, so its term is
  that of tau(K) with 3 ceil(K / 8) additions.  The product term is 2^-10 / (3 * 2^-20), about 2^8, below the
  2 * 2^-11 of TF32 products of unrounded operands.

Besides the elementwise bound, every call must take the path the case declares (tile widths may only be narrower: a
split launch keeps >= 3 pipeline stages next to its lo images; on a narrower tile every path field must be that of the
case's TF32 launch forced to the same width) and its record must say prec=1.  Each path-table record also lists the
kernel builds the split launch and the case's TF32 launch ran, so that the suite can check that the table reaches the
split form of every build it reaches with TF32 products.  Cases with K <= KMAX must also meet twice gemm_paths'
global relative error (4e-5 without output rounding, scaled like gemm_paths for draws), which TF32 products of
unrounded operands (~2^-11) miss by an order of magnitude.
"""
import argparse
import functools
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (os.path.join(ROOT, 'video-long-term-feature-banks_b200', 'lib'), HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import gemm_fuzz as GF  # noqa: E402
import gemm_paths as GP  # noqa: E402

SPLIT_PRODUCT = 3 * 2.0 ** -20


def tau_x3(K):
    return SPLIT_PRODUCT + GP.TAU_SAFETY * (3 * -(-K // 8) + 8) * 2.0 ** -23


SPLIT = [True]            # False while tf32_records runs a case's TF32 twin


def split_mode(K):
    """Switch this process to split mode (see the module docstring)."""
    import torch
    from vlfb import libvlfb as L
    lib = L.load()
    gemm = lib.vlfb_gemm

    def gemm_x3(pp, stream):
        pp._obj.precision = L.PREC_X3 if SPLIT[0] else L.PREC_TF32
        return gemm(pp, stream)

    lib.vlfb_gemm = gemm_x3
    K.weight_transpose = functools.partial(K.weight_transpose, precision=L.PREC_X3)
    GP.rnd = lambda shape, gen, scale=1.0: torch.randn(shape, generator=gen) * scale
    GP.tau = tau_x3


# path fields a split launch shares with the TF32 launch at the same tile width (stages, lag, tiles, units and the split
# factor follow from the lo images' shared memory and the cost model; prec differs by definition)
PATH_FIELDS = ('kinds', 'mask', 'bn', 'tma', 'patch', 'par', 'cp', 'sk', 'fix', 'lean', 'bits2', 'wide', 'det')


def tf32_records(K, c, dev, tile_n=None):
    """Launch records of the case run with TF32 products (its TF32 twin), optionally at tile width `tile_n`.  Only the
    records are used: the operands are not TF32-exact, so the values are not checked."""
    c = dict(c)
    if tile_n:
        c['opts'] = dict(c.get('opts', {}), tile_n=tile_n)
    P = GP.prepare(c, dev)
    SPLIT[0] = False
    try:
        _, text = GP.capture_fd2(lambda: GP.run_case(K, P, dev))
    finally:
        SPLIT[0] = True
    return [r for r in (GP.parse_record(l) for l in text.splitlines()) if r is not None]


def build_of(r):
    """(A kind, B kind, MASK, CP, FIX) of the kernel build a launch record ran."""
    return [r['kinds'][0], r['kinds'][1], r['mask'], r['cp'], r['fix']]


def path_errors(K, c, dev, rec, declared):
    """Errors of a split launch record against the path the case declares for TF32 products.  A split launch may run a
    narrower tile than declared (its lo images must leave >= 3 stages); then it must take every path field of the TF32
    launch of the case at that narrower width."""
    bad = []
    for r in rec['paths']:
        if r.get('prec') != 1:
            bad.append('record prec=%r' % r.get('prec'))
    if declared is None or len(rec['paths']) != 1:
        return bad
    r = rec['paths'][0]
    want = dict(declared)
    want.pop('split', None)           # the split factor is chosen with the width by the cost model
    bn = want.get('bn')
    if bn is not None and r['bn'] > bn:
        bad.append('bn=%d wider than the declared %d' % (r['bn'], bn))
    elif bn is not None and r['bn'] < bn:
        twin = tf32_records(K, c, dev, tile_n=r['bn'])
        if len(twin) != 1:
            return bad + ['TF32 twin at bn=%d: %d launch records' % (r['bn'], len(twin))]
        want = dict((k, twin[0][k]) for k in PATH_FIELDS)
        rec['twin'] = dict((k, list(v) if isinstance(v, tuple) else v) for k, v in want.items())
    bad += GP.matches(dict((k, tuple(v) if isinstance(v, list) else v) for k, v in r.items()), want)
    return bad


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--config', required=True, choices=sorted(GP.CONFIGS))
    ap.add_argument('--seed', type=int, default=None, help='fuzz draws of this seed instead of the path table')
    ap.add_argument('--count', type=int, default=0)
    ap.add_argument('--out', required=True)
    args = ap.parse_args(argv)
    for k, v in GP.CONFIGS[args.config].items():
        if os.environ.get(k) != v:
            raise SystemExit('configuration %s needs %s=%s in the environment' % (args.config, k, v))
    if os.environ.get('VLFB_DEBUG') != '1':
        raise SystemExit('the path records need VLFB_DEBUG=1')
    import torch
    from vlfb import kernels as K
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device('cuda')
    K.set_gemm_backend('tcgen05')
    split_mode(K)
    if args.seed is None:
        # the path table without the production-size weight gradients (their K runs to 10^6: the table's cases cover
        # every path of those launches at sizes the fp64 reference handles quickly)
        jobs = [(c['name'], c, c['runs'][args.config]) for c in GP.CASES
                if args.config in c['runs'] and not c.get('long_k')]
    else:
        jobs = [('draw %d' % i, GF.draw(args.seed, i, args.config), None) for i in range(args.count)]
    with open(args.out, 'w') as f:
        for name, c, declared in jobs:
            print('[gemm_x3] config=%s %s' % (args.config, name), flush=True)
            try:
                if declared is None and c.get('family') == 'gconv':
                    r = GF.run_draw(K, c, args.config, dev)
                    rec = dict(case=name, paths=[], errors=r['errors'], engine='gconv', worst_ratio=r['worst_ratio'])
                else:
                    rec = GP.check_case(K, c, args.config, dev, declared=False)
                    rec['case'] = name
                    # the global check at twice the table's tolerance: three accumulations per k8 step and the product
                    # term, still an order of magnitude below TF32 products of unrounded operands
                    tol = 2 * (6e-4 if c.get('epi', {}).get('tf32') else 2e-5)
                    if declared is None:
                        tol *= max(1.0, (GP.describe(c)['K'] / 2048.0) ** 0.5)
                    rec['errors'] = [e for e in rec['errors'] if not e.startswith('global rel_err')]
                    if GP.describe(c)['K'] <= GP.KMAX and not rec['rel_err'] < tol:
                        rec['errors'].append('global rel_err %.3g >= %g' % (rec['rel_err'], tol))
                    if rec['engine'] != 'simt':
                        rec['errors'] += path_errors(K, c, dev, rec, declared)
                        rec['x3_builds'] = [build_of(r) for r in rec['paths']]
                        if declared is not None:
                            rec['tf32_builds'] = [build_of(r) for r in tf32_records(K, c, dev)]
                rec['ok'] = not rec['errors']
            except Exception as ex:                   # a failing call is a result of the case, not of the run
                rec = dict(case=name, ok=False, paths=[], errors=['%s: %s' % (type(ex).__name__, ex)])
            rec['config'] = args.config
            f.write(json.dumps(rec) + '\n')
            f.flush()
            torch.cuda.empty_cache()
    print('[gemm_x3] config=%s done' % args.config, flush=True)


if __name__ == '__main__':
    main()
