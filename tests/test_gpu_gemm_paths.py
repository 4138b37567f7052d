"""The loader / tile-width / schedule matrix of the tensor-core GEMM (csrc/gemm_tc.cu) against fp64.

Every configuration of the library's switches runs tests/gemm_paths.py in its own process (the switches are read once per
process).  Each case must match its fp64 reference elementwise, leave its guard band untouched and take the path it
declares; together the configurations must cover every instantiation, loader, tile width, schedule and special form of
the kernel, each named in the failure message when it is missing."""
import json
import os
import subprocess
import sys

import pytest

import gemm_paths as GP

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
TIMEOUT = 900            # seconds per configuration; the child is killed when it expires
_RESULTS = {}


def _launch(cfg, tmp_dir):
    """Runs the worker of one configuration ONCE; the outcome (records, or the timeout) is kept for every later test."""
    out = os.path.join(tmp_dir, 'gemm_paths_%s.jsonl' % cfg)
    env = dict((k, v) for k, v in os.environ.items() if k not in GP.SWITCHES)
    env.update(GP.CONFIGS[cfg])
    env['VLFB_DEBUG'] = '1'
    cmd = [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [
        os.path.join(HERE, 'gemm_paths.py'), '--config', cfg, '--out', out]
    try:
        proc = subprocess.run(cmd, env=env, cwd=os.path.dirname(HERE), capture_output=True, text=True, timeout=TIMEOUT)
    except subprocess.TimeoutExpired as ex:
        so = ex.stdout.decode() if isinstance(ex.stdout, bytes) else (ex.stdout or '')
        last = [l for l in so.splitlines() if l.startswith('[gemm_paths]')]
        return dict(timeout=last[-1] if last else '(none)')
    recs = []
    if os.path.exists(out):
        with open(out) as f:
            recs = [json.loads(l) for l in f if l.strip()]
    return dict(proc=proc, recs=recs)


def _run(cfg, tmp_dir):
    """(process, records) of a configuration; fails -- without starting it again -- if its worker timed out."""
    if cfg not in _RESULTS:
        _RESULTS[cfg] = _launch(cfg, tmp_dir)
    r = _RESULTS[cfg]
    if 'timeout' in r:
        pytest.fail('configuration %s timed out after %d s; last progress line: %s' % (cfg, TIMEOUT, r['timeout']))
    return r['proc'], r['recs']


@pytest.fixture(scope='module')
def tmp_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp('gemm_paths'))


@pytest.mark.parametrize('cfg', sorted(GP.CONFIGS))
def test_gemm_paths_match_fp64_and_declared_path(cfg, tmp_dir):
    proc, recs = _run(cfg, tmp_dir)
    want = [c['name'] for c in GP.CASES if cfg in c['runs']]
    assert proc.returncode == 0, 'worker exit %d\n%s\n%s' % (proc.returncode, proc.stdout[-3000:], proc.stderr[-3000:])
    assert [r['case'] for r in recs] == want
    bad = ['%s: %s' % (r['case'], '; '.join(r['errors'])) for r in recs if not r['ok']]
    assert not bad, 'configuration %s:\n  ' % cfg + '\n  '.join(bad)


MN_KINDS = (GP.OP_DENSE_MN, GP.OP_CONV_MN, GP.OP_STEM_MN)


def _strided(case_name):
    g = GP.case_by_name(case_name).get('geom')
    return g is not None and tuple(g['st']) != (1, 1, 1)


def test_gemm_path_coverage(tmp_dir):
    """The union over all configurations reaches every path of the kernel (checked on passing cases only)."""
    seen = []
    for cfg in sorted(GP.CONFIGS):
        _, recs = _run(cfg, tmp_dir)
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
    })
    missing = [name for name, pred in need.items() if not pred()]
    assert not missing, 'not covered by any passing case: ' + '; '.join(missing)


def test_mn_major_operands_are_staged_by_cp_async(tmp_dir):
    """Every launch record, in every configuration: an MN-major operand has no TMA loader and runs in a cp.async build."""
    bad = []
    for cfg in sorted(GP.CONFIGS):
        _, recs = _run(cfg, tmp_dir)
        for r in recs:
            for p in r['paths']:
                ak, bk = p['kinds']
                if (ak in MN_KINDS and p['tma'][0] != 0) or (bk in MN_KINDS and p['tma'][1] != 0) or \
                        ((ak in MN_KINDS or bk in MN_KINDS) and p['cp'] != 1):
                    bad.append('%s / %s: kinds=%d,%d tma=%d,%d cp=%d' % (cfg, r['case'], ak, bk, p['tma'][0], p['tma'][1], p['cp']))
    assert not bad, '\n'.join(bad)
