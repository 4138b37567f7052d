"""How the cp.async producers of the tensor-core GEMM publish a K chunk, checked on the compiler output (no GPU needed).

With both operands MN-major (every weight gradient; the consumers read those stage tiles through their generic-proxy
rewrite only), a producer thread ends a chunk with `cp.async.mbarrier.arrive.noinc`: the stage barrier's arrival fires
when the thread's copies land, so the producers run ahead of the MMAs by the whole ring.  In SASS that is
`ARRIVES.LDGSTSBAR`.  Every other build publishes after `cp.async.wait_group` and a proxy fence (its wgmma reads the
stage tiles through the async proxy) and must not contain it.  The compile and SASS parsing are the ones of
test_gemm_pipeline_cpu.py.
"""
import os
import subprocess
import tempfile

import pytest

import __graft_entry__ as G
import test_gemm_pipeline_cpu as PIPE


@pytest.fixture(scope='module')
def compiled():
    nvcc, cuobjdump = PIPE._tool('nvcc'), PIPE._tool('cuobjdump')
    if nvcc is None or cuobjdump is None:
        pytest.skip('nvcc / cuobjdump not found')
    with tempfile.TemporaryDirectory() as tmp:
        obj = os.path.join(tmp, 'gemm_tc.o')
        r = subprocess.run([nvcc] + G.NVCC_FLAGS + ['-Xptxas', '-v', '-c', PIPE.SRC, '-o', obj],
                           capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0, r.stderr[-4000:]
        sass = subprocess.run([cuobjdump, '-sass', obj], capture_output=True, text=True, check=True, timeout=600).stdout
    return PIPE.parse(r.stdout + r.stderr, sass)


def test_mn_major_cp_async_chunks_are_published_by_copy_completion(compiled):
    bad, async_builds = [], 0
    for key, body in sorted(compiled['funcs'].items()):
        ak, bk, _, cp, _ = key
        want = cp == 1 and ak in PIPE.MN_KINDS and bk in PIPE.MN_KINDS
        has = any('ARRIVES.LDGSTSBAR' in ins for _, ins in body)          # (possibly predicated: @P0 ARRIVES...)
        async_builds += want
        if has != want:
            bad.append('%s: %s' % (PIPE._fmt(key), 'no ARRIVES.LDGSTSBAR' if want else 'unexpected ARRIVES.LDGSTSBAR'))
    assert async_builds, 'no cp.async build with two MN-major operands'
    assert not bad, '\n'.join(bad)
