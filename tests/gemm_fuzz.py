"""Seeded random sweep of vlfb_gemm over its legal parameter space, on every engine, against fp64.

Each draw is one case dict in the format the path table (gemm_paths.py) or the grouped table (gconv_cases.py) already
runs, and is checked by the same reference, bound, guard band, sign-bit and stream-K counter code; only the declared
path is missing (a draw has none).  `draw(seed, i, config)` depends on nothing else, so a failing draw is rerun from
its seed and index alone:

    VLFB_DEBUG=1 python tests/gemm_fuzz.py --config default --seed S --count N --index I --out FILE

Sizes are drawn from mixtures placed at the edges of the kernels' tiling (M at 1-64 for wide tiles, 65-127, and
128 j + {-1, 0, 1}; N around 16, 32, 2 BN and the tile widths; K below 32, at 32, at 32 j + {1, 2, 3} and >= 512), and
every draw stays within KMAX, MAX_MACS and MAX_BYTES so that the fp64 references stay fast and the GPU never sees a
large allocation.  tests/test_gpu_gemm_fuzz.py runs fixed seeds; tests/test_gemm_fuzz_cpu.py checks the generator.
"""
import argparse
import json
import os
import random
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (os.path.join(ROOT, 'video-long-term-feature-banks_b200', 'lib'), ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import gemm_paths as GP  # noqa: E402
import gconv_cases as GC  # noqa: E402

FAMILIES = ('dense', 'conv_fwd', 'conv_dgrad', 'conv_wgrad', 'stem_fwd', 'stem_wgrad', 'gconv')
# the families whose calls a configuration's switches can change (the grouped kernels read none of them)
CONFIG_FAMILIES = {
    'default': FAMILIES,
    'tma0': ('dense', 'conv_fwd', 'conv_dgrad', 'stem_fwd'),
    'im2col0': ('conv_fwd', 'conv_dgrad', 'stem_fwd'),
    'nopar': ('conv_dgrad',),
    'nopatch': ('stem_fwd',),
}
# the committed sweep: (configuration, seed, draws); each runs once
RUNS = [('default', 1, 800), ('default', 2, 800), ('default', 3, 800),
        ('tma0', 11, 150), ('im2col0', 12, 150), ('nopar', 13, 150), ('nopatch', 14, 150)]
KMAX = GP.KMAX
MAX_MACS = 2 ** 31
MAX_BYTES = 256 << 20
TILE_N = (0, 0, 32, 64, 96, 128, 160, 192, 224, 256)


# ----------------------------------------------------------------------------------------------- size mixtures
def _m(r):
    x = r.random()
    if x < 0.35:
        return r.randint(1, 64)
    if x < 0.5:
        return r.randint(65, 127)
    return 128 * r.randint(1, 8) + r.choice((-1, 0, 1))


def _n(r):
    return max(1, r.choice((16, 32, 64, 96, 128, 192, 256)) + r.choice((-4, -1, 0, 0, 0, 1, 4)))


def _k(r):
    x = r.random()
    if x < 0.15:
        return r.randint(1, 31)
    if x < 0.25:
        return 32
    if x < 0.7:
        return 32 * r.randint(1, 12) + r.choice((0, 1, 2, 3, 4))
    return r.randint(512, 4096)


def _opts(r):
    return dict(tile_n=r.choice(TILE_N), stream_k=r.choice((-1, 0, 1, 1)))


# ----------------------------------------------------------------------------------------------- families
def _dense(r):
    Z = r.choice((1, 1, 1, 2, 3))
    c = dict(op='raw', Z=Z, M=_m(r), N=_n(r), K=_k(r), a_mn=r.random() < 0.35, b_mn=r.random() < 0.35,
             gn=r.choice((0, 0, 3, 4, 8)), gm=r.choice((0, 1, 2)), opts=_opts(r))
    mode = r.choice(('store', 'accum', 'atomic', 'atomic'))
    x = r.random()
    if x < 0.45:                                   # enough tiles and K chunks for split-K and stream-K schedules
        c.update(Z=1, M=128 * r.randint(3, 8) + r.choice((-1, 0, 1)), N=r.choice((128, 192, 256)),
                 K=4 * r.randint(256, 1024), a_mn=r.random() < 0.5, b_mn=r.random() < 0.5)
        c['opts']['stream_k'] = r.choice((0, 0, 1, 1))
        if r.random() < 0.3:                       # one row tile: no 128-row TMA box, the cp.async build
            c.update(M=r.randint(65, 127), N=256, K=4 * r.randint(512, 1024))
        if c['a_mn'] and r.random() < 0.8:         # (an MN-major A with M % 4 != 0 runs on the SIMT engine)
            c['M'] += -c['M'] % 4
        mode = r.choice(('store', 'atomic', 'atomic', 'atomic'))
    elif x < 0.6:                                  # wide tiles: both operands MN-major, M <= 64
        c.update(a_mn=True, b_mn=True, M=r.randint(1, 64))
        if r.random() < 0.7:
            c['M'] = 4 * r.randint(1, 16)
        c['Z'] = Z = r.choice((1, 2, 3))
        mode = r.choice(('store', 'accum', 'atomic'))
    for w in 'ab':
        if r.random() < 0.25 and w + '_pad' not in c:
            c[w + '_pad'] = r.choice((1, 3, 4, 8))
        if r.random() < 0.1:
            c[w + '_off'] = r.choice((1, 2, 4, 7))
        if Z > 1 and r.random() < 0.4:
            if r.random() < 0.5:
                c[w + '_shared'] = True
            else:
                c[w + '_gap'] = r.choice((4, 5, 64))
    if r.random() < 0.2:
        c['d_off'] = r.choice((1, 2, 3, 4, 13))
    if r.random() < 0.2:
        c['ldd'] = c['N'] + r.choice((0, 1, 5, 16))
    if Z > 1 and r.random() < 0.3:
        c['d_gap'] = r.choice((0, 3, 40))
    e = {}
    if r.random() < 0.3:
        e['alpha'] = r.choice((0.5, -1.0, -0.25, 2.0))
    for f, pr in (('scale', 0.3), ('bias', 0.4), ('row_scale', 0.3), ('residual', 0.25), ('relu', 0.3), ('tf32', 0.2)):
        if r.random() < pr:
            e[f] = True
    c['split_k'] = r.choice((1, 1, 0))
    c['deterministic'] = int(r.random() < (0.5 if x < 0.45 else 0.25))
    if r.random() < 0.15:
        e['mask_float' if r.random() < 0.5 else 'mask_bits'] = True
    if mode == 'accum':
        e['accum'] = True
    elif mode == 'atomic':
        e['atomic'] = True
        c['split_k'] = r.choice((0, 0, 2, 3, 5) if x < 0.45 else (0, 0, 1, 2, 3, 5))
        if c['split_k'] != 1:                      # a split sums partial values: a linear epilogue, never deterministic
            for f in ('residual', 'relu', 'tf32', 'mask_float', 'mask_bits'):
                e.pop(f, None)
            if x < 0.45 and c['a_mn'] and c['b_mn'] and r.random() < 0.5:
                c.update(split_k=0, deterministic=1)     # the cp.async fix-up of MN x MN deterministic launches
            c['deterministic'] = int(c['split_k'] == 0 and c['deterministic'])
    if r.random() < 0.12:                          # sign bits out: one dense batch, N % 32 == 0, a ReLU
        e.update(bits=True, relu=True)
        e.pop('atomic', None)
        for f in ('ldd', 'a_pad', 'b_pad', 'a_off', 'b_off', 'd_off'):   # aligned: the lean epilogue, unless d_off
            c.pop(f, None)
        c.update(Z=1, N=32 * r.randint(1, 8), gn=0, split_k=r.choice((0, 1)), a_mn=False, b_mn=False)
        if r.random() < 0.6:
            e['mask_bits'] = True
        if r.random() < 0.3:
            c['d_off'] = r.choice((1, 2, 3))
    c['epi'] = e
    c['workspace'] = r.random() > 0.15
    if r.random() < 0.15:
        c['engine'] = 'simt'
    if e.get('mask_float') or e.get('mask_bits'):
        if c.get('engine') != 'simt':          # masks on the tensor cores: DENSE_K x DENSE_K
            c['a_mn'] = c['b_mn'] = False
    return c


def _pads(r, ker, dil):
    return tuple(r.choice((0, d * (k // 2), d * (k // 2), d * (k // 2) + r.randint(1, 3), r.randint(0, k * d)))
                 for k, d in zip(ker, dil))


def _conv(r, op):
    """conv fwd / dgrad / wgrad through the kernels.py wrappers (C != 4)."""
    x = r.random()
    if x < 0.2:                                   # pointwise: DENSE_K / DENSE_MN operands
        ker, st, dil, pd = (1, 1, 1), (1, 1, 1), (1, 1, 1), (0, 0, 0)
    elif op == 'conv_dgrad' and x < 0.5:          # parity-class friendly: stride 2 in H / W, even extents
        k = r.choice((1, 3))
        ker, st, dil = (r.choice((1, 3)), k, k), (1, 2, 2), (1, 1, 1)
        pd = (ker[0] // 2, k // 2, k // 2)
    elif op == 'conv_dgrad' and x < 0.75:         # unit stride: im2col over dY
        ker, st, dil = (r.choice((1, 3)), 3, 3), (1, 1, 1), (1, r.choice((1, 2)), r.choice((1, 2)))
        pd = _pads(r, ker, dil)
    elif op != 'conv_dgrad' and x < 0.4:          # im2col corners out of TMA's range: a long dilated kernel
        k = r.choice((5, 7, 8 if op == 'conv_wgrad' else 7))
        ker, st, dil = (1, k, r.choice((3, 5, 7))), (1, r.choice((1, 2)), r.choice((1, 2, 3))), (1, 1, 3)
        pd = (0, r.randint(0, 3), r.choice((0, 1, 17)))
    else:
        ker = (r.choice((1, 1, 3, 5)), r.choice((1, 3, 5, 7, 8)), r.choice((1, 3, 5, 7, 8)))
        st = tuple(r.choice((1, 1, 2, 3)) for _ in range(3))
        dil = tuple(r.choice((1, 1, 2, 3)) for _ in range(3))
        pd = _pads(r, ker, dil)
    pointwise = ker == (1, 1, 1) and st == (1, 1, 1) and pd == (0, 0, 0)
    n, T = r.choice((1, 1, 2)), r.randint(1, 5)
    H, W = r.randint(3, 22), r.randint(3, 22)
    if st[1] == 2 and op == 'conv_dgrad':
        H, W = H + H % 2, W + W % 2
    c4 = lambda: 4 * r.randint(2, 40)             # (C = 4 would be the stem)  # noqa: E731
    if op == 'conv_fwd':
        C = (r.choice((c4(), 32 * r.randint(1, 4), 7)) if pointwise else 32 * r.randint(1, 4))
        Co = r.choice((c4(), 32 * r.randint(1, 5), r.randint(1, 160)))
    elif op == 'conv_dgrad':
        Co = (r.choice((c4(), 32 * r.randint(1, 4), 9)) if pointwise else 32 * r.randint(1, 4))
        C = r.choice((16 * r.randint(1, 8), 16 * r.randint(1, 8), c4(), r.randint(1, 160)))
    else:
        C = c4() if not pointwise else r.choice((c4(), 6))
        Co = r.choice((c4(), c4(), r.randint(1, 160)))
    C = 8 if C == 4 else C
    c = dict(op=op, geom=GP.G(n, T, H, W, C, Co, ker, st, pd, dil), opts=_opts(r))
    e = {}
    if op == 'conv_fwd':
        for f, pr in (('scale', 0.4), ('bias', 0.5), ('residual', 0.3), ('relu', 0.4), ('tf32', 0.3)):
            if r.random() < pr:
                e[f] = True
        if Co % 32 == 0 and r.random() < 0.3:
            e.update(bits=True, relu=True)
    elif op == 'conv_dgrad':
        parity = st == (1, 2, 2) and dil == (1, 1, 1)
        for f, pr in (('accum', 0.6 if parity else 0.4), ('residual', 0.1 if parity else 0.3), ('tf32', 0.3)):
            if r.random() < pr:
                e[f] = True
        if r.random() < 0.3:
            e['mask_bits' if (n * T * H * W * C) % 32 == 0 and r.random() < 0.6 else 'mask_float'] = True
    else:
        if r.random() < 0.5:
            e['row_scale'] = True
        c['deterministic'] = int(r.random() < 0.4)
    c['epi'] = e
    if r.random() < 0.08:
        c['engine'] = 'simt'
    return c


def _stem(r, op):
    """conv1 (C = 4: 3 channels + a zero pad) on a dense or a W-padded (pitched) clip."""
    kT, kH, kW = r.choice((1, 3, 5)), r.randint(1, 7), r.randint(1, 7)
    st = (r.choice((1, 1, 2)), r.choice((1, 2, 2, 3)), r.choice((1, 2, 2, 3)))
    pd = (r.randint(0, kT // 2 + 1), r.randint(0, kH // 2 + 1), r.randint(0, kW // 2 + 1))
    if r.random() < 0.3:                          # conv1 itself, with even Ho and Wo % 16 == 0 for the patch tiles
        kT, kH, kW, st, pd = 5, 7, 7, (1, 2, 2), (2, 3, 3)
        H, W = 16 * r.randint(1, 3), 32 * r.randint(1, 2)
    else:
        H, W = r.randint(4, 40), r.randint(4, 40)
    c = dict(op=op, geom=GP.G(r.choice((1, 1, 2)), r.randint(1, 6), H, W, 4, r.choice((32, 64, 64, 96)), (kT, kH, kW),
                              st, pd), pitched=r.random() < 0.6, opts=_opts(r))
    e = {}
    if op == 'conv_fwd':
        for f, pr in (('scale', 0.4), ('bias', 0.5), ('relu', 0.5), ('tf32', 0.2)):
            if r.random() < pr:
                e[f] = True
        if r.random() < 0.3:
            e.update(bits=True, relu=True)
    else:
        if r.random() < 0.5:
            e['row_scale'] = True
        c['deterministic'] = int(r.random() < 0.4)
    c['epi'] = e
    return c


def _gconv(r):
    d = r.choice(('fwd', 'dgrad', 'wgrad'))
    cig, cog, G = 4 * r.randint(1, 16), 4 * r.randint(1, 16), r.choice((1, 2, 4, 8)) * 2
    ker = (r.choice((1, 3)), r.choice((1, 3, 5)), r.choice((3, 5)))
    st = tuple(r.choice((1, 1, 2, 3)) for _ in range(3))
    dil = tuple(r.choice((1, 1, 2, 3)) for _ in range(3))
    pd = _pads(r, ker, dil)
    shape = (r.choice((1, 2)), r.randint(1, 5), r.randint(3, 16), r.randint(3, 16), cig * G)
    e = {}
    if d == 'wgrad':
        for f, pr in (('row_scale', 0.4), ('col_scale', 0.3), ('accum', 0.5)):
            if r.random() < pr:
                e[f] = 1
    else:
        for f, pr in (('scale', 0.3), ('bias', 0.4), ('residual', 0.3), ('accum', 0.3), ('relu', 0.3), ('tf32', 0.3),
                      ('row_scale', 0.2)):
            if r.random() < pr:
                e[f] = 1
        if r.random() < 0.25:
            e['mask'] = r.choice(('float', 'bits'))
        if r.random() < 0.25:
            e.update(bits=1, relu=1)
    if r.random() < 0.3:
        e['alpha'] = r.choice((0.5, -0.75, 2.0))
    if r.random() < 0.4:
        e['det'] = 1
    return GC.make_case('', d, shape, cog * G, G, k=ker, s=st, p=pd, d=dil, family='gconv', seed=r.randint(0, 9999),
                        **e)


# ----------------------------------------------------------------------------------------------- legality and caps
def gconv_errors(c):
    """The rules validate_gconv (csrc/api.cu) and the grouped table apply to a grouped case: [] when legal."""
    err = []
    G = c['groups']
    cig, cog = c['C'] // G, c['Co'] // G
    if c['C'] % G or c['Co'] % G or not (cig % 4 == 0 and cog % 4 == 0 and 4 <= cig <= 64 and 4 <= cog <= 64):
        err.append('grouped widths')
    out = [(x + 2 * p - d * (k - 1) - 1) // s + 1 for x, p, d, k, s in
           zip((c['T'], c['H'], c['W']), c['p'], c['d'], c['k'], c['s'])]
    if min(out) < 1:
        err.append('empty output')
    e = c['epi']
    ncols = c['Co'] if c['dir'] == 'fwd' else c['C']
    if e.get('bits') and not (e.get('relu') and ncols % 32 == 0):
        err.append('relu_bits_out needs RELU and N % 32 == 0')
    rows = c['N'] * (out[0] * out[1] * out[2] if c['dir'] == 'fwd' else c['T'] * c['H'] * c['W'])
    if (e.get('mask') == 'bits' or e.get('bits')) and (rows * ncols) % 32:
        err.append('packed bits need a multiple of 32 elements')
    return err


def _ints(c):
    """(MACs, bytes of the buffers) of a draw."""
    if c['family'] == 'gconv':
        kt, kh, kw = c['k']
        out = [(x + 2 * p - d * (k - 1) - 1) // s + 1 for x, p, d, k, s in
               zip((c['T'], c['H'], c['W']), c['p'], c['d'], c['k'], c['s'])]
        pos = c['N'] * max(out[0], 0) * max(out[1], 0) * max(out[2], 0)
        macs = pos * c['Co'] * kt * kh * kw * (c['C'] // c['groups'])
        elems = c['N'] * c['T'] * c['H'] * c['W'] * c['C'] + pos * c['Co'] + c['Co'] * kt * kh * kw * c['C']
        return macs, 16 * elems
    d = GP.describe(c)
    taps = d['taps'] * d['batch']
    macs = d['M'] * d['N'] * d['K'] * taps
    if c['op'] == 'raw':
        elems = sum((ld * (c['K'] if c[w + '_mn'] else (c['M'] if w == 'a' else c['N'])) + bs) * c['Z'] + off
                    for w in 'ab' for ld, bs, off in [GP.operand_layout(c, w)])
        elems += (c.get('ldd', c['N'] + c.get('gn', 0))) * (c['M'] + c.get('gm', 0) + 8) * c['Z'] * 4
    else:
        g = c['geom']
        To, Ho, Wo = GP.out_dims(g)
        elems = (g['N'] * g['T'] * g['H'] * max(g['W'], (Wo - 1) * g['st'][2] + 8) * g['C'] +
                 g['N'] * To * Ho * Wo * g['Co'] + 4 * d['M'] * d['N'] * taps)
    return macs, 16 * elems                       # fp32 buffers, fp64 references and their magnitudes


def cap_errors(c):
    err = []
    macs, nbytes = _ints(c)
    if c['family'] != 'gconv' and GP.describe(c)['K'] > KMAX:
        err.append('K > KMAX')
    if macs > MAX_MACS:
        err.append('MACs')
    if nbytes > MAX_BYTES:
        err.append('bytes')
    return err


def legal(c):
    if c['family'] == 'gconv':
        return not gconv_errors(c) and not cap_errors(c)
    return not GP.abi_errors(c) and not cap_errors(c)


def draw(seed, i, config='default'):
    """Draw i of `seed`: one legal case within the caps, from the families `config` affects.  Reproducible: it
    depends on (seed, i, config) only."""
    r = random.Random('gemm_fuzz:%d:%d:%s' % (seed, i, config))
    fams = [f for f in CONFIG_FAMILIES[config] for _ in range(4 if f == 'dense' else 1)]   # dense: the most fields
    fam = r.choice(fams)
    for attempt in range(1000):
        if fam == 'dense':
            c = _dense(r)
        elif fam in ('conv_fwd', 'conv_dgrad', 'conv_wgrad'):
            c = _conv(r, fam)
        elif fam == 'stem_fwd':
            c = _stem(r, 'conv_fwd')
        elif fam == 'stem_wgrad':
            c = _stem(r, 'conv_wgrad')
        else:
            c = _gconv(r)
        c['family'] = fam
        c['name'] = 'fuzz_%d_%d' % (seed, i)
        c['seed'] = seed * 100003 + i
        if legal(c):
            return c
    raise AssertionError('no legal draw for seed %d index %d' % (seed, i))


def im2col_encodable(c):
    """Whether the TMA im2col tensor map of a fwd or unit-stride dgrad draw can be encoded (box corners in [-16, 15],
    gemm_tc.cu make_tmap_im2col); False forces the cp.async gather loader by geometry."""
    g = c['geom']
    for k, p, d in zip(g['ker'], g['pd'], g['dil']):
        lo, hi = (-p, p - (k - 1) * d) if c['op'] == 'conv_fwd' else (p - (k - 1) * d, -p)
        if not (-16 <= lo <= 15 and -16 <= hi <= 15):
            return False
    return True


def reproducer(config, seed, count, index):
    env = ' '.join('%s=%s' % kv for kv in sorted(GP.CONFIGS[config].items()))
    return ('%s VLFB_DEBUG=1 python tests/gemm_fuzz.py --config %s --seed %d --count %d --index %d --out /tmp/draw.jsonl'
            % (env, config, seed, count, index)).strip()


# ----------------------------------------------------------------------------------------------- running (GPU)
def run_draw(K, c, config, dev):
    """One draw's JSON record: the draw, its path records, the engine, the worst |err| / bound and the errors."""
    import torch
    if c['family'] == 'gconv':
        det = bool(c['epi'].get('det'))
        st = GC.run_case(c, dev.type, keep_out=det)
        errors = [] if st['ok'] else ['values %s, guard %s, bits %s, record %s (worst %.3g x bound)' % (
            'ok' if st['finite'] and st['ratio'] <= 1 else 'WRONG', st['guard_ok'], st['bits_ok'], st['record_ok'],
            st['ratio'])]
        if det:
            st2 = GC.run_case(c, dev.type, keep_out=True)
            if not torch.equal(st['out'], st2['out']):
                errors.append('deterministic call: a second run gave other bits')
        torch.cuda.empty_cache()
        return dict(engine='gconv', paths=[st['record']] if st['record'] else [], worst_ratio=st['ratio'],
                    errors=errors, ok=not errors)
    r = GP.check_case(K, c, config, dev, declared=False)
    return dict(engine=r['engine'], paths=r['paths'], worst_ratio=r['worst_ratio'], errors=r['errors'], ok=r['ok'])


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--config', required=True, choices=sorted(CONFIG_FAMILIES))
    ap.add_argument('--seed', type=int, required=True)
    ap.add_argument('--count', type=int, required=True)
    ap.add_argument('--index', type=int, default=None, help='rerun this one draw')
    ap.add_argument('--out', required=True)
    args = ap.parse_args(argv)
    for k, v in GP.CONFIGS[args.config].items():
        if os.environ.get(k) != v:
            raise SystemExit('configuration %s needs %s=%s in the environment' % (args.config, k, v))
    if os.environ.get('VLFB_DEBUG') != '1':
        raise SystemExit('the path records need VLFB_DEBUG=1')
    import torch
    from vlfb import kernels as K
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device('cuda')
    K.set_gemm_backend('tcgen05')
    idx = [args.index] if args.index is not None else range(args.count)
    with open(args.out, 'w') as f:
        for i in idx:
            c = draw(args.seed, i, args.config)
            print('[gemm_fuzz] config=%s seed=%d index=%d family=%s' % (args.config, args.seed, i, c['family']),
                  flush=True)
            t0 = time.time()
            try:
                rec = run_draw(K, c, args.config, dev)
            except Exception as ex:                   # a failing call is a result of the draw, not of the run
                rec = dict(engine=None, paths=[], worst_ratio=None, errors=['%s: %s' % (type(ex).__name__, ex)],
                           ok=False)
            rec.update(config=args.config, seed=args.seed, index=i, family=c['family'], draw=c,
                       seconds=round(time.time() - t0, 3),
                       reproducer=reproducer(args.config, args.seed, args.count, i))
            f.write(json.dumps(rec, sort_keys=True) + '\n')
            f.flush()
    print('[gemm_fuzz] config=%s seed=%d done' % (args.config, args.seed), flush=True)


if __name__ == '__main__':
    main()
