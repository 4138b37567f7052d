"""vlfb_gemm on seeded random draws from its legal parameter space (tests/gemm_fuzz.py), on every engine, against fp64.

Each (configuration, seed) runs tests/gemm_fuzz.py once in its own process with VLFB_DEBUG=1.  Every draw must match
its fp64 reference elementwise, leave its guard band and stream-K counters untouched, run on the engine the ABI
predicts and, when deterministic, give the same bits twice.  A coverage floor keeps the generator at the edges: each
named cell must be reached by at least FLOOR passing draws."""
import pytest

import gemm_fuzz as GF
import gemm_paths as GP
from util import run_worker

pytestmark = pytest.mark.gpu

TIMEOUT = 900            # seconds per worker; a worker that times out fails its tests and is not started again
RUNS = GF.RUNS
FLOOR = 3


def _run(cfg, seed, count):
    return run_worker('gemm_fuzz.py', ['--config', cfg, '--seed', str(seed), '--count', str(count)],
                      env=GP.CONFIGS[cfg], timeout=TIMEOUT)


@pytest.mark.parametrize('cfg,seed,count', RUNS)
def test_every_draw_matches_fp64(cfg, seed, count):
    proc, recs = _run(cfg, seed, count)
    assert proc.returncode == 0, 'worker exit %d\n%s\n%s' % (proc.returncode, proc.stdout[-3000:], proc.stderr[-3000:])
    assert [r['index'] for r in recs] == list(range(count))
    bad = ['seed %d index %d (%s): %s\n    %s' % (seed, r['index'], r['family'], '; '.join(r['errors']), r['reproducer'])
           for r in recs if not r['ok']]
    assert not bad, 'configuration %s:\n  ' % cfg + '\n  '.join(bad)


def _zero_tap_class(g):
    """Whether a strided dgrad has a parity class without taps (its tiles run the epilogue only)."""
    for ph in range(g['st'][1]):
        for pw in range(g['st'][2]):
            if (ph + g['pd'][1]) % g['st'][1] >= g['ker'][1] or (pw + g['pd'][2]) % g['st'][2] >= g['ker'][2]:
                return True
    return False


def coverage_cells():
    """name -> predicate(record, path record or None, draw)."""
    cells = {}
    builds = [(2, 0, 0), (5, 0, 0), (3, 0, 0), (1, 4, 0), (1, 6, 0), (0, 0, 0), (0, 1, 0), (1, 0, 0), (1, 1, 0),
              (3, 0, 1), (0, 0, 1)]
    mn = (GP.OP_DENSE_MN, GP.OP_CONV_MN, GP.OP_STEM_MN)
    for ak, bk, mask in builds:
        for cp in ((1,) if ak in mn or bk in mn else (0, 1)):
            def build(r, p, c, ak=ak, bk=bk, mask=mask, cp=cp):
                return p is not None and tuple(p['kinds']) == (ak, bk) and p['mask'] == mask and p['cp'] == cp
            cells['build %d,%d mask=%d cp=%d' % (ak, bk, mask, cp)] = build
            cells['build %d,%d mask=%d cp=%d static' % (ak, bk, mask, cp)] = \
                lambda r, p, c, b=build: b(r, p, c) and p['sk'] == 0 and p['split'] == 1
            if not mask and ak != 3 and ak != 2 and ak != 5:     # atomic calls: the dense and wgrad builds
                cells['build %d,%d mask=%d cp=%d split-K' % (ak, bk, mask, cp)] = \
                    lambda r, p, c, b=build: b(r, p, c) and p['sk'] == 0 and p['split'] > 1
                cells['build %d,%d mask=%d cp=%d stream-K atomic' % (ak, bk, mask, cp)] = \
                    lambda r, p, c, b=build: b(r, p, c) and p['sk'] == 1 and p['fix'] == 0
            if cp == 0 or (ak in mn and bk in mn and not mask):   # fix-ups: TMA builds, MN x MN deterministic
                cells['build %d,%d mask=%d cp=%d stream-K fix-up' % (ak, bk, mask, cp)] = \
                    lambda r, p, c, b=build: b(r, p, c) and p['sk'] == 1 and p['fix'] == 1
    wide = lambda p: p is not None and p.get('wide') == 1                                        # noqa: E731
    cells.update({
        'wide tiles x ACCUM': lambda r, p, c: wide(p) and c.get('epi', {}).get('accum'),
        'wide tiles x deterministic fix-up': lambda r, p, c: wide(p) and p['fix'] == 1 and p['det'] == 1,
        'wide tiles x split-K': lambda r, p, c: wide(p) and p['split'] > 1,
        'wide tiles x stream-K': lambda r, p, c: wide(p) and p['sk'] == 1,
        'wide tiles x batch > 1': lambda r, p, c: wide(p) and c.get('Z', 1) > 1,
        # (the in-kernel sign bits exist in the lean epilogue only: the general one always writes them in a second pass)
        'lean epilogue x in-kernel sign bits': lambda r, p, c: p is not None and c['epi'].get('bits') and p['lean'] == 1 and p['bits2'] == 0,
        'lean epilogue x second-pass sign bits': lambda r, p, c: p is not None and c['epi'].get('bits') and p['lean'] == 1 and p['bits2'] == 1,
        'general epilogue x second-pass sign bits': lambda r, p, c: p is not None and c['epi'].get('bits') and p['lean'] == 0 and p['bits2'] == 1,
        'parity classes x ACCUM': lambda r, p, c: p is not None and p['par'] > 0 and c['epi'].get('accum'),
        'parity classes x ACCUM with a zero-tap class': lambda r, p, c: p is not None and p['par'] > 0 and c['epi'].get('accum') and _zero_tap_class(c['geom']),
        'im2col fallback forced by geometry': lambda r, p, c: p is not None and r['config'] in ('default', 'nopar', 'nopatch') and c['op'] in ('conv_fwd', 'conv_dgrad') and tuple(p['kinds'])[0] in (2, 3) and p['par'] == 0 and (c['op'] == 'conv_fwd' or tuple(c['geom']['st']) == (1, 1, 1)) and not GF.im2col_encodable(c) and p['tma'][0] == 0,
        'SIMT engine by !tc_ok': lambda r, p, c: r['engine'] == 'simt' and c.get('engine') != 'simt',
        'SIMT engine by request': lambda r, p, c: r['engine'] == 'simt' and c.get('engine') == 'simt',
    })
    for d in ('fwd', 'dgrad', 'wgrad'):
        g = lambda c, d=d: c['family'] == 'gconv' and c['dir'] == d                               # noqa: E731
        cells['grouped %s x stride > 1' % d] = lambda r, p, c, g=g: g(c) and max(c['s']) > 1
        cells['grouped %s x dilation > 1' % d] = lambda r, p, c, g=g: g(c) and max(c['d']) > 1
        cells['grouped %s x deterministic' % d] = lambda r, p, c, g=g: g(c) and c['epi'].get('det')
    return cells


def test_coverage_floor():
    """Each cell is reached by at least FLOOR passing draws (over every configuration and seed)."""
    counts = dict((k, 0) for k in coverage_cells())
    cells = coverage_cells()
    for cfg, seed, count in RUNS:
        _, recs = _run(cfg, seed, count)
        for r in recs:
            if not r['ok']:
                continue
            p = r['paths'][0] if r['engine'] == 'tc' and len(r['paths']) == 1 else None
            for name, pred in cells.items():
                if pred(r, p, r['draw']):
                    counts[name] += 1
    low = ['%s: %d' % (k, v) for k, v in sorted(counts.items()) if v < FLOOR]
    assert not low, 'cells below the floor of %d passing draws:\n  ' % FLOOR + '\n  '.join(low)
