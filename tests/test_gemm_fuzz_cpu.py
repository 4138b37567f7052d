"""CPU checks of the vlfb_gemm sweep generator (tests/gemm_fuzz.py): reproducible, legal, capped draws, and a
comparison that rejects the faults a wrong kernel would make at the drawn shapes."""
import ctypes
import json
import os
import subprocess
import sys

import pytest
import torch

import gemm_fuzz as GF
import gemm_paths as GP

HERE = os.path.dirname(os.path.abspath(__file__))
ALL = [(cfg, seed, i) for cfg, seed, count in GF.RUNS for i in range(count)]


def _draws():
    return [(cfg, seed, i, GF.draw(seed, i, cfg)) for cfg, seed, i in ALL]


def test_same_seed_gives_the_same_draws_to_the_byte():
    a = [json.dumps(c, sort_keys=True) for *_, c in _draws()]
    assert a == [json.dumps(c, sort_keys=True) for *_, c in _draws()]
    # ... and in another interpreter, whatever its hash seed
    code = ('import json, gemm_fuzz as GF\n'
            'print(json.dumps([GF.draw(s, i, c) for c, s, i in %r], sort_keys=True))' % (ALL[::97],))
    out = subprocess.check_output([sys.executable, '-c', code], cwd=HERE,
                                  env=dict(os.environ, PYTHONHASHSEED='12345')).decode()
    assert json.loads(out) == [json.loads(a[k]) for k in range(0, len(ALL), 97)]
    assert json.dumps(GF.draw(1, 0), sort_keys=True) != json.dumps(GF.draw(2, 0), sort_keys=True)


def test_every_draw_is_legal_and_planned():
    from vlfb import libvlfb as L
    lib = L.load()
    ws = int(lib.vlfb_gemm_workspace_bytes())
    for cfg, seed, i, c in _draws():
        assert c['family'] in GF.CONFIG_FAMILIES[cfg]
        if c['family'] == 'gconv':
            assert GF.gconv_errors(c) == [], (cfg, seed, i)
            continue
        assert GP.abi_errors(c) == [], (cfg, seed, i, GP.abi_errors(c))
        if GP.engine(c) != 'tc':
            continue
        d = GP.describe(c)
        p = L.GemmParams()
        p.M, p.N, p.K, p.batch, p.taps, p.split_k = d['M'], d['N'], d['K'], d['batch'], d['taps'], GP.effective_split_k(c)
        p.flags = L.EPI_ATOMIC if d['flags']['atomic'] else 0
        p.tile_n, p.stream_k = c['opts']['tile_n'], c['opts']['stream_k']
        p.deterministic = int(c.get('deterministic', 0))
        if c.get('workspace', True):
            p.workspace, p.workspace_bytes = 4096, ws       # host-only query: never dereferenced
        out = L.GemmPlan()
        assert lib.vlfb_gemm_plan(ctypes.byref(p), 132, ctypes.byref(out)) == 0, (cfg, seed, i)
        assert out.split_k >= 1 and out.tiles >= 1 and 32 <= out.tile_n <= 128, (cfg, seed, i)
        if p.deterministic and d['flags']['atomic']:
            assert out.split_k == 1, (cfg, seed, i)


def test_every_draw_stays_within_the_caps():
    for cfg, seed, i, c in _draws():
        assert GF.cap_errors(c) == [], (cfg, seed, i)
        macs, nbytes = GF._ints(c)
        assert macs <= GF.MAX_MACS and nbytes <= GF.MAX_BYTES
        if c['family'] != 'gconv':
            assert GP.describe(c)['K'] <= GF.KMAX


def test_draws_reach_the_edges():
    """The mixtures put sizes where the kernels' tiling changes: the generator has not drifted to the middle."""
    dense = [c for *_, c in _draws() if c['family'] == 'dense']
    Ms, Ks = [c['M'] for c in dense], [c['K'] for c in dense]
    assert sum(m <= 64 for m in Ms) >= 20 and sum(m % 128 in (1, 127) for m in Ms) >= 10
    assert sum(k < 32 for k in Ks) >= 10 and Ks.count(32) >= 5 and sum(k >= 512 for k in Ks) >= 20
    assert sum(k % 32 in (1, 2, 3) for k in Ks) >= 10
    assert sum(bool(c['opts']['tile_n'] > 128) for c in dense) >= 10
    for f in ('a_pad', 'a_off', 'b_shared', 'd_off', 'ldd', 'engine'):
        assert sum(f in c for c in dense) >= 5, f
    assert sum(c.get('split_k') == 0 and not c['epi'].get('atomic') for c in dense) >= 10
    assert sum(c['epi'].get('alpha', 1) < 0 for c in dense) >= 5


# ----------------------------------------------------------------------------------------------- planted faults
def _sample():
    """Small dense draws of the committed seeds (the fp64 references run on the CPU here), with N > 32 so that a wide
    tile's second warpgroup has columns."""
    out = []
    for cfg, seed, i, c in _draws():
        if c['family'] == 'dense' and c['N'] > 32 and c['Z'] * c['M'] * c['N'] * c['K'] <= 1 << 22:
            c = json.loads(json.dumps(c))
            c['epi'].update(bias=True, row_scale=True)          # the faults below need both
            c['epi'].pop('mask_float', None), c['epi'].pop('mask_bits', None)
            out.append(c)
        if len(out) == 6:
            break
    assert len(out) == 6
    return out


SAMPLE = _sample()


def _rejected(P, bad):
    return not GP.compare(bad.float(), P.ref, P.bound)['ok']


@pytest.mark.parametrize('k', range(len(SAMPLE)))
def test_planted_faults_are_rejected_at_drawn_shapes(k):
    c = SAMPLE[k]
    P = GP.prepare(c, torch.device('cpu'))
    assert GP.compare(P.ref.float(), P.ref, P.bound)['ok']
    # the last (partial) K chunk dropped
    A = P.A.clone()
    A[:, :, 32 * ((c['K'] - 1) // 32):] = 0
    bad, _ = GP.finish(torch.bmm(A.double(), P.B.double().transpose(1, 2)), P.mag, P.epi, P.K)
    assert _rejected(P, bad), 'missing last K chunk'
    # the bias added by every split of a 2-way split-K, not by the first one only
    extra = (P.epi['cb'].view(1, 1, -1) * P.epi['rs'].view(1, -1, 1))
    assert _rejected(P, P.ref + extra), 'bias added per split'
    # the row scale skipped on the second warpgroup's columns of a 64 x 2BN wide tile (BN = 32)
    epi = dict(P.epi)
    epi['rs'] = torch.ones_like(P.epi['rs'])
    noscale, _ = GP.finish(P.acc, P.mag, epi, P.K)
    cols = (torch.arange(c['N']) % 64) >= 32
    bad = torch.where(cols.view(1, 1, -1), noscale, P.ref)
    assert _rejected(P, bad), 'row scale skipped on warpgroup 1'
    # one guard element written
    buf = torch.full((P.layout['size'],), float('nan'))
    buf[P.index.reshape(-1)] = P.ref.reshape(-1).float()
    assert GP.guard_touched(buf, P.index) == 0
    inside = set(P.index.reshape(-1).tolist())
    for pos in (P.layout['d0'] - 1, int(P.index.max()) + 1,
                next((j for j in range(int(P.index.min()), int(P.index.max())) if j not in inside), None)):
        if pos is None:
            continue
        b = buf.clone()
        b[pos] = 0.0
        assert GP.guard_touched(b, P.index) == 1, pos
