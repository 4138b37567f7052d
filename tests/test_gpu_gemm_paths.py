"""The loader / tile-width / schedule matrix of the tensor-core GEMM (csrc/gemm_tc.cu) against fp64.

Every configuration of the library's switches runs tests/gemm_paths.py in its own process (the switches are read once per
process).  Each case must match its fp64 reference elementwise, leave its guard band untouched and take the path it
declares; together the configurations must cover every instantiation, loader, tile width, schedule and special form of
the kernel, each named in the failure message when it is missing."""
import pytest

import gemm_paths as GP
from util import run_worker

pytestmark = pytest.mark.gpu

# seconds per configuration; the default one also runs the production weight gradients
TIMEOUT = dict(default=4500)


def _run(cfg):
    return run_worker('gemm_paths.py', ['--config', cfg], env=GP.CONFIGS[cfg], timeout=TIMEOUT.get(cfg, 900))


@pytest.mark.parametrize('cfg', sorted(GP.CONFIGS))
def test_gemm_paths_match_fp64_and_declared_path(cfg):
    proc, recs = _run(cfg)
    want = [c['name'] for c in GP.CASES if cfg in c['runs']]
    assert proc.returncode == 0, 'worker exit %d\n%s\n%s' % (proc.returncode, proc.stdout[-3000:], proc.stderr[-3000:])
    assert [r['case'] for r in recs] == want
    bad = ['%s: %s' % (r['case'], '; '.join(r['errors'])) for r in recs if not r['ok']]
    assert not bad, 'configuration %s:\n  ' % cfg + '\n  '.join(bad)


MN_KINDS = (GP.OP_DENSE_MN, GP.OP_CONV_MN, GP.OP_STEM_MN)


def _strided(case_name):
    g = GP.case_by_name(case_name).get('geom')
    return g is not None and tuple(g['st']) != (1, 1, 1)


def test_gemm_path_coverage():
    """The union over all configurations reaches every path of the kernel (checked on passing cases only)."""
    seen = []
    for cfg in sorted(GP.CONFIGS):
        _, recs = _run(cfg)
        for r in recs:
            if r['ok'] and len(r['paths']) == 1:
                p = dict(r['paths'][0])
                p['kinds'], p['tma_a'], p['tma_b'] = tuple(p['kinds']), p['tma'][0], p['tma'][1]
                seen.append((r['case'], r['flags'], p))
    assert seen, 'no passing case'

    def any_(pred):
        return any(pred(n, f, p) for n, f, p in seen)

    need = {}
    # (A kind, B kind, mask): TMA-only (cp=0) builds exist for K-major pairs only
    builds = [(2, 0, 0), (5, 0, 0), (3, 0, 0), (1, 4, 0), (1, 6, 0), (0, 0, 0), (0, 1, 0), (1, 0, 0), (1, 1, 0),
              (3, 0, 1), (0, 0, 1)]
    for ak, bk, mask in builds:
        for cp in ((1,) if ak in MN_KINDS or bk in MN_KINDS else (0, 1)):
            need['instantiation kinds=%d,%d mask=%d cp=%d' % (ak, bk, mask, cp)] = \
                (lambda ak=ak, bk=bk, mask=mask, cp=cp:
                 any_(lambda n, f, p: p['kinds'] == (ak, bk) and p['mask'] == mask and p['cp'] == cp))
    for v in range(4):
        need['loader tma_a=%d' % v] = lambda v=v: any_(lambda n, f, p: p['tma_a'] == v)
    for v in range(2):
        need['loader tma_b=%d' % v] = lambda v=v: any_(lambda n, f, p: p['tma_b'] == v)
    for bn in (32, 64, 96, 128):
        for cp in (0, 1):
            need['tile width %d cp=%d' % (bn, cp)] = lambda bn=bn, cp=cp: any_(lambda n, f, p: p['bn'] == bn and p['cp'] == cp)
        need['N tail against width %d' % bn] = lambda bn=bn: any_(lambda n, f, p: p['bn'] == bn and p['N'] % bn != 0)
    need.update({
        'schedule static': lambda: any_(lambda n, f, p: p['sk'] == 0 and p['split'] == 1),
        'schedule split-K atomic (split > 1)': lambda: any_(lambda n, f, p: p['sk'] == 0 and p['split'] > 1),
        'schedule stream-K fix-up, lean epilogue': lambda: any_(lambda n, f, p: p['sk'] == 1 and p['fix'] == 1 and p['lean'] == 1),
        'schedule stream-K fix-up, general epilogue': lambda: any_(lambda n, f, p: p['sk'] == 1 and p['fix'] == 1 and p['lean'] == 0),
        'schedule stream-K fix-up with ACCUM': lambda: any_(lambda n, f, p: p['sk'] == 1 and p['fix'] == 1 and f['accum']),
        'schedule stream-K atomic cp=0': lambda: any_(lambda n, f, p: p['sk'] == 1 and p['fix'] == 0 and f['atomic'] and p['cp'] == 0),
        'schedule stream-K atomic cp=1': lambda: any_(lambda n, f, p: p['sk'] == 1 and p['fix'] == 0 and f['atomic'] and p['cp'] == 1),
        'conv1 fwd patch tiles (tma_a=3)': lambda: any_(lambda n, f, p: p['kinds'] == (5, 0) and p['tma_a'] == 3 and p['patch'] == 1),
        'conv1 fwd TMA rows without patches': lambda: any_(lambda n, f, p: p['kinds'] == (5, 0) and p['tma_a'] == 3 and p['patch'] == 0),
        'strided dgrad as parity classes': lambda: any_(lambda n, f, p: p['kinds'] == (3, 0) and p['par'] > 0),
        'strided dgrad by the gather loader': lambda: any_(lambda n, f, p: p['kinds'] == (3, 0) and p['par'] == 0 and p['tma_a'] == 0 and _strided(n)),
        'sign bits in-kernel': lambda: any_(lambda n, f, p: f['relu'] and p['bits2'] == 0 and 'bits' in GP.case_by_name(n).get('epi', {})),
        'sign bits in a second pass': lambda: any_(lambda n, f, p: p['bits2'] == 1),
        'M tail of 1 row': lambda: any_(lambda n, f, p: p['M'] % 128 == 1),
        'M tail of 64 rows': lambda: any_(lambda n, f, p: p['M'] % 128 == 64),
        'M tail of 127 rows': lambda: any_(lambda n, f, p: p['M'] % 128 == 127),
        'N % 4 != 0 with ldd % 4 != 0: the 4 x 157 x 2048 FC': lambda: any_(lambda n, f, p: (p['M'], p['N'], p['K']) == (4, 157, 2048)),
        'K % 32 != 0': lambda: any_(lambda n, f, p: p['K'] % 32 != 0),
        'K < 32': lambda: any_(lambda n, f, p: p['K'] < 32),
        'K == 32 (one chunk)': lambda: any_(lambda n, f, p: p['K'] == 32),
        'batch > 1': lambda: any_(lambda n, f, p: p['z'] > 1 and p['kinds'][1] in (0, 1) and p['kinds'][0] in (0, 1)),
        'taps > 1': lambda: any_(lambda n, f, p: p['z'] > 1 and p['kinds'][1] in (4, 6)),
        'wide tiles N <= bn': lambda: any_(lambda n, f, p: p.get('wide') == 1 and p['N'] <= p['bn']),
        'wide tiles bn < N < 2 bn': lambda: any_(lambda n, f, p: p.get('wide') == 1 and p['bn'] < p['N'] < 2 * p['bn']),
        'wide tiles N = 2 bn q + 16': lambda: any_(lambda n, f, p: p.get('wide') == 1 and p['N'] >= 2 * p['bn'] and
                                                   p['N'] % (2 * p['bn']) == 16),
    })
    for bn in (32, 64, 128):
        need['wide tiles bn=%d' % bn] = lambda bn=bn: any_(lambda n, f, p: p.get('wide') == 1 and p['bn'] == bn)
    # every B operand of a weight gradient under both multi-CTA schedules, on 128-row and on 64 x 2bn wide tiles
    # (conv1 has Co = 64: its STEM_MN launches are always wide)
    scheds = {'stream-K': lambda p: p['sk'] == 1, 'split-K > 1': lambda p: p['sk'] == 0 and p['split'] > 1}
    for bk, wides in ((GP.OP_CONV_MN, (0, 1)), (GP.OP_DENSE_MN, (0, 1)), (GP.OP_STEM_MN, (1,))):
        for sname, sched in scheds.items():
            for wide in wides:
                need['wgrad B kind %d %s on %s tiles' % (bk, sname, 'wide' if wide else 'narrow')] = \
                    (lambda bk=bk, sched=sched, wide=wide:
                     any_(lambda n, f, p: p['kinds'][0] == GP.OP_DENSE_MN and p['kinds'][1] == bk and sched(p) and
                          p.get('wide', 0) == wide))
    missing = [name for name, pred in need.items() if not pred()]
    assert not missing, 'not covered by any passing case: ' + '; '.join(missing)


def test_mn_major_operands_are_staged_by_cp_async():
    """Every launch record, in every configuration: an MN-major operand has no TMA loader and runs in a cp.async build."""
    bad = []
    for cfg in sorted(GP.CONFIGS):
        _, recs = _run(cfg)
        for r in recs:
            for p in r['paths']:
                ak, bk = p['kinds']
                if (ak in MN_KINDS and p['tma'][0] != 0) or (bk in MN_KINDS and p['tma'][1] != 0) or \
                        ((ak in MN_KINDS or bk in MN_KINDS) and p['cp'] != 1):
                    bad.append('%s / %s: kinds=%d,%d tma=%d,%d cp=%d' % (cfg, r['case'], ak, bk, p['tma'][0], p['tma'][1], p['cp']))
    assert not bad, '\n'.join(bad)
