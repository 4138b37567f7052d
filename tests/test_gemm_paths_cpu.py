"""CPU checks of the GEMM path harness (tests/gemm_paths.py): the record parser, the legality of every case under the
C ABI's rules, and that the elementwise comparison rejects the errors a wrong path would make."""
import ctypes

import pytest
import torch

import gemm_paths as GP

SAMPLE = ('vlfb gemm_tc: kinds=3,0 mask=1 M=3600 N=64 K=1152 z=1 bn=64 sk=0 split=1 tiles=32 units=32 stages=6 lag=2 '
          'tma=2,1 cap=132 patch=0 par=4 cp=0 fix=0 lean=1 bits2=0')


def test_parse_record():
    r = GP.parse_record(SAMPLE + '\n')
    assert r['kinds'] == (3, 0) and r['tma'] == (2, 1) and r['mask'] == 1
    assert (r['M'], r['N'], r['K'], r['z'], r['bn'], r['par'], r['cp'], r['fix'], r['lean'], r['bits2'], r['lag']) == \
        (3600, 64, 1152, 1, 64, 4, 0, 0, 1, 0, 2)
    assert GP.parse_record('some other line') is None
    assert GP.matches(r, dict(kinds=(3, 0), par='>0', bn=64)) == []
    assert GP.matches(r, dict(par=0, cp=1)) == ['par=4 (declared 0)', 'cp=0 (declared 1)']


def test_record_keys_are_printed_by_the_library():
    """The keys the harness reads are the ones gemm_tc.cu launch() prints."""
    import os
    src = open(os.path.join(GP.ROOT, 'video-long-term-feature-banks_b200', 'csrc', 'gemm_tc.cu')).read()
    fmt = src[src.index('"vlfb gemm_tc: '):]
    fmt = fmt[:fmt.index(';')]
    keys = set(k for k in GP.parse_record(SAMPLE))
    for k in keys:
        assert (' %s=' % k) in fmt.replace('"', ' ').replace('gemm_tc:', ''), k


def test_case_table_is_well_formed():
    names = [c['name'] for c in GP.CASES]
    assert len(names) == len(set(names))
    for c in GP.CASES:
        assert c['runs'] and set(c['runs']) <= set(GP.CONFIGS), c['name']
        assert 'default' in c['runs'] or len(c['runs']) >= 1
    assert all(any(cfg in c['runs'] for c in GP.CASES) for cfg in GP.CONFIGS)


@pytest.mark.parametrize('name', [c['name'] for c in GP.CASES])
def test_case_is_a_legal_tensor_core_call(name):
    c = GP.case_by_name(name)
    assert GP.abi_errors(c) == []
    # (a SIMT fallback would have no path record to check against the declared path; only a case that asks for the
    # SIMT engine runs there)
    assert GP.engine(c) == c.get('engine', 'tc')
    assert GP.describe(c)['K'] <= GP.KMAX or c.get('long_k')
    assert c.get('opts', {}).get('tile_n', 0) in (0, 32, 64, 96, 128)
    # ... and the host-only plan query accepts its extents
    from vlfb import libvlfb as L
    lib = L.load()
    d = GP.describe(c)
    p = L.GemmParams()
    p.M, p.N, p.K, p.batch, p.taps, p.split_k = d['M'], d['N'], d['K'], d['batch'], d['taps'], d['flags']['split_k']
    p.flags = L.EPI_ATOMIC if d['flags']['atomic'] else 0
    p.tile_n = c.get('opts', {}).get('tile_n', 0)
    out = L.GemmPlan()
    assert lib.vlfb_gemm_plan(ctypes.byref(p), 132, ctypes.byref(out)) == 0
    if p.tile_n:
        assert out.tile_n == p.tile_n


_PREP = {}


def _prep(name):
    if name not in _PREP:
        _PREP[name] = GP.prepare(GP.case_by_name(name), torch.device('cpu'))
    return _PREP[name]


def _dense_names():
    return [c['name'] for c in GP.CASES if c['op'] in ('matmul', 'raw')]


def _cpu_cases():
    """The cases whose fp64 reference is quick on the CPU: all but the long-K weight gradients."""
    return [c for c in GP.CASES if not c.get('long_k')]


def test_exact_result_rounded_to_fp32_passes_every_case():
    for c in _cpu_cases():
        P = _prep(c['name'])
        r = GP.compare(P.ref.float(), P.ref, P.bound)
        assert r['ok'] and r['rel_err'] < 2e-5, (c['name'], r)


def _without_k_chunk(P, chunk):
    """The case's fp64 result with the 32 k of K chunk `chunk` left out (what a loader that skipped it would give)."""
    c = P.case
    if c['op'] in ('matmul', 'raw'):
        A = P.A.clone()
        A[:, :, 32 * chunk:32 * chunk + 32] = 0
        acc = torch.bmm(A.double(), P.B.double().transpose(1, 2))
    else:
        assert c['op'] == 'conv_wgrad'                      # k = output position (n, to, ho, wo)
        dy = P.dy.clone()
        Co = dy.shape[1]
        pos = dy.permute(0, 2, 3, 4, 1).reshape(-1, Co)
        pos[32 * chunk:32 * chunk + 32] = 0
        dy = pos.reshape(dy.shape[0], *dy.shape[2:], Co).permute(0, 4, 1, 2, 3)
        acc, _ = GP.conv_refs(c, P.x, P.w, dy, torch.device('cpu'))
    bad, _ = GP.finish(acc, P.mag, P.epi, P.K)
    return bad


@pytest.mark.parametrize('which', ['largest K of the table', 'largest K of the dense cases'])
def test_missing_k_chunk_of_the_largest_k_case_is_rejected(which):
    names = [c['name'] for c in _cpu_cases()] if which.endswith('table') else _dense_names()
    name = max(names, key=lambda n: GP.describe(GP.case_by_name(n))['K'])
    P = _prep(name)
    assert P.K >= 2048, name
    for chunk in (0, P.K // 32 // 2, (P.K - 1) // 32):
        assert not GP.compare(_without_k_chunk(P, chunk).float(), P.ref, P.bound)['ok'], (name, chunk)


def test_missing_tail_row_and_column_are_rejected():
    P = _prep('raw_kk_t32_tails')
    Z, M, N = P.ref.shape
    assert M % 128 == 1 and N % 32 != 0
    row = P.ref.clone()
    row[:, M - 1, :] = 0
    assert not GP.compare(row.float(), P.ref, P.bound)['ok']
    col = P.ref.clone()
    col[:, :, N - 1] = 0
    assert not GP.compare(col.float(), P.ref, P.bound)['ok']
    nan = P.ref.clone()
    nan[1, M - 1, N - 1] = float('nan')                   # an element never written keeps its NaN fill
    assert not GP.compare(nan.float(), P.ref, P.bound)['ok']


def test_bias_one_tf32_ulp_off_is_rejected():
    P = _prep('raw_k16_big_bias')
    cb = P.epi['cb']
    off = P.ref.clone()
    off[:, :, 0] += GP.ulp_tf32(cb[0:1])
    assert not GP.compare(off.float(), P.ref, P.bound)['ok']


def test_single_guard_write_is_detected():
    P = _prep('raw_mnk_t64_k32')
    buf = torch.full((P.layout['size'],), float('nan'))
    buf[P.index.reshape(-1)] = P.ref.reshape(-1).float()
    assert GP.guard_touched(buf, P.index) == 0
    Z, M, N = P.ref.shape
    gap = int(P.index[0, 0, N - 1]) + 1                    # the ldd gap right after a row
    assert gap not in set(P.index.reshape(-1).tolist())
    buf[gap] = 0.0
    assert GP.guard_touched(buf, P.index) == 1
    buf[gap] = float('nan')
    buf[int(P.index[Z - 1, M - 1, N - 1]) + P.layout['ldd']] = -float('nan')   # past row M: another NaN is not the fill
    assert GP.guard_touched(buf, P.index) == 1
