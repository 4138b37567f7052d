"""The split-TF32 GEMM (vlfb_gemm_params_t.precision = VLFB_PREC_X3) against fp64 at the bound of its error analysis.

tests/gemm_x3.py runs, in its own process per configuration of the library's switches, every case of the GEMM path table
(tests/gemm_paths.py) and, in the default configuration, a seeded set of draws of tests/gemm_fuzz.py, all with
unrounded fp32 operands and precision = VLFB_PREC_X3 on every call.  Each must match fp64 within tau_x3, take the path
its case declares (no wider tile) and report prec=1."""
import pytest

import gemm_paths as GP
from util import run_worker

pytestmark = pytest.mark.gpu

FUZZ_SEED, FUZZ_COUNT = 7, 48


def _check(args, env):
    proc, recs = run_worker('gemm_x3.py', args, env=env, timeout=1800)
    assert proc.returncode == 0, 'worker exit %d\n%s\n%s' % (proc.returncode, proc.stdout[-3000:], proc.stderr[-3000:])
    return recs


@pytest.mark.parametrize('cfg', sorted(GP.CONFIGS))
def test_split_gemm_paths_match_fp64(cfg):
    recs = _check(['--config', cfg], GP.CONFIGS[cfg])
    want = [c['name'] for c in GP.CASES if cfg in c['runs'] and not c.get('long_k')]
    assert [r['case'] for r in recs] == want
    bad = ['%s: %s' % (r['case'], '; '.join(r['errors'])) for r in recs if not r['ok']]
    assert not bad, 'configuration %s:\n  ' % cfg + '\n  '.join(bad)


def test_split_table_reaches_every_build_the_tf32_table_reaches():
    """Over all configurations, every (A kind, B kind, MASK, CP, FIX) kernel build the path table runs with TF32 products
    also runs in split form (gemm_tc3_kernel)."""
    x3, tf32 = set(), set()
    for cfg in sorted(GP.CONFIGS):
        for r in _check(['--config', cfg], GP.CONFIGS[cfg]):
            x3.update(tuple(b) for b in r.get('x3_builds', []))
            tf32.update(tuple(b) for b in r.get('tf32_builds', []))
    assert tf32, 'no tensor-core launch record from the TF32 twins'
    missing = sorted(tf32 - x3)
    assert not missing, 'builds reached with TF32 products only (kinds a, b, mask, cp, fix): %s' % missing


def test_split_gemm_fuzz_matches_fp64():
    recs = _check(['--config', 'default', '--seed', str(FUZZ_SEED), '--count', str(FUZZ_COUNT)], {})
    assert len(recs) == FUZZ_COUNT
    bad = ['%s: %s' % (r['case'], '; '.join(r['errors'])) for r in recs if not r['ok']]
    assert not bad, '\n'.join(bad)
