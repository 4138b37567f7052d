"""Grouped convolution (vlfb_gemm with groups > 1, csrc/gconv.cu): a table of seeded, self-describing cases, each ONE
vlfb_gemm call through the vlfb.kernels wrappers, checked elementwise against an fp64 reference
(torch.nn.functional.conv3d(groups=) and its autograd).

Every output sits in a NaN-filled buffer with guard bands on both sides.  A case passes when
  * every element satisfies |got - ref| <= tau(K) * |alpha s r| * sum|a||b| + 4u (|alpha s r acc| + |bias| + |res| +
    |d_prev|) (+ one TF32 ulp of |ref| when the output is rounded), where K is the number of terms of the sum: taps*Cig
    (fwd), taps*Cog (dgrad), output positions (wgrad; the position split adds at most one term per split, already
    inside K) and tau(K) = (K + 8) * 2^-24;
  * both guard bands are still bit-exact NaN;
  * the sign bits (relu_bits_out) equal the packed signs of the stored output;
  * the library's VLFB_DEBUG record of the launch says path=gconv with the case's direction and widths.

Run as a script (tests/test_gpu_gconv.py does, in a subprocess with VLFB_DEBUG=1) it writes one JSON line per case.
On the CPU the same comparison runs on an emulated kernel, with planted bugs (test_gconv_cpu.py).
"""
import argparse
import ctypes
import json
import os
import re
import sys

import torch
import torch.nn.functional as F

from util import capture_fd2, compare, guard_touched, nan_buffer, pack_sign_bits, parse_record, tf32_round

U32 = 2.0 ** -24
TF32_ULP = 2.0 ** -10
GUARD = 64                     # floats of NaN on each side of every output

# ------------------------------------------------------------------------------------------------ cases
CASES = []


def make_case(name, dir, shape, co, groups, k=(1, 3, 3), s=(1, 1, 1), p=None, d=(1, 1, 1), family=None, seed=0, **epi):
    """One case dict.  epi: the epilogue fields (scale, bias, ...) and det = 1 for a deterministic call."""
    n, t, h, w, c = shape
    if p is None:
        p = tuple(dd * (kk // 2) for kk, dd in zip(k, d))
    return dict(name=name, dir=dir, N=n, T=t, H=h, W=w, C=c, Co=co, groups=groups, k=tuple(k), s=tuple(s),
                p=tuple(p), d=tuple(d), family=family or dir, seed=seed, epi=epi)


def _case(*a, **kw):
    CASES.append(make_case(*a, **kw))


# widths: Cig = Cog of 4, 8, 16, 32, 64 in every direction, plus Cig != Cog
for dir_ in ('fwd', 'dgrad', 'wgrad'):
    for cg in (4, 8, 16, 32, 64):
        _case('%s_cg%d' % (dir_, cg), dir_, (1, 2, 9, 7, cg * 4), cg * 4, 4, seed=cg)
    _case('%s_cig8_cog16' % dir_, dir_, (2, 3, 6, 5, 64), 128, 8, k=(3, 3, 3), seed=3)
    _case('%s_cig16_cog4' % dir_, dir_, (1, 3, 7, 6, 128), 32, 8, k=(3, 3, 3), s=(1, 2, 2), seed=4)
    # stride / dilation / kernel, ragged H and W, N > 1
    _case('%s_s2' % dir_, dir_, (2, 2, 11, 13, 64), 64, 8, s=(1, 2, 2), seed=5)
    _case('%s_s2_t' % dir_, dir_, (1, 5, 9, 10, 32), 32, 4, k=(3, 3, 3), s=(2, 2, 2), seed=6)
    _case('%s_d2' % dir_, dir_, (2, 2, 10, 9, 64), 64, 16, d=(1, 2, 2), seed=7)
    _case('%s_d2_s2' % dir_, dir_, (1, 3, 13, 11, 64), 64, 16, k=(3, 3, 3), s=(1, 2, 2), d=(2, 2, 2), seed=8)
    _case('%s_nopad' % dir_, dir_, (3, 1, 7, 9, 32), 32, 8, p=(0, 0, 0), seed=9)
    _case('%s_ragged_co' % dir_, dir_, (1, 2, 5, 5, 96), 96, 4, seed=10)       # Co not a multiple of the 64-ch CTA

# epilogues of fwd (conv + affine (+ residual) + ReLU, sign bits, ACCUM, TF32)
_case('fwd_affine_relu_bits', 'fwd', (2, 2, 8, 8, 128), 128, 32, seed=20, scale=1, bias=1, relu=1, tf32=1, bits=1)
_case('fwd_residual_relu', 'fwd', (1, 2, 7, 9, 64), 64, 8, seed=21, scale=1, bias=1, residual=1, relu=1)
_case('fwd_accum_alpha', 'fwd', (1, 2, 7, 9, 64), 64, 8, seed=22, accum=1, alpha=0.75, row_scale=1)
_case('fwd_mask_tf32', 'fwd', (1, 2, 6, 6, 64), 64, 16, seed=23, mask='float', tf32=1)
_case('fwd_maskbits', 'fwd', (1, 2, 8, 8, 64), 64, 16, seed=24, mask='bits')
# dgrad grad-finish: + earlier contributions (residual or ACCUM), ReLU backward (float or bit mask), TF32
_case('dgrad_finish_residual_bits', 'dgrad', (2, 2, 8, 8, 128), 128, 32, s=(1, 2, 2), seed=30, residual=1,
      mask='bits', tf32=1)
_case('dgrad_finish_accum_mask', 'dgrad', (1, 2, 9, 7, 64), 64, 8, seed=31, accum=1, mask='float', tf32=1)
_case('dgrad_scale_relu_bits', 'dgrad', (1, 2, 8, 8, 64), 64, 8, seed=32, scale=1, bias=1, relu=1, bits=1, alpha=0.5)
# wgrad: row_scale (the affine scale), col_scale (a column mask), alpha; dw accumulates into nonzero values
_case('wgrad_row_scale', 'wgrad', (2, 2, 9, 7, 64), 64, 8, seed=40, row_scale=1, accum=1)
_case('wgrad_col_scale_alpha', 'wgrad', (1, 3, 8, 8, 32), 32, 4, k=(3, 3, 3), seed=41, col_scale=1, alpha=0.5)
# above any grid cap: fwd / dgrad tile counts and wgrad splits beyond 132 * 16 CTAs
for dir_ in ('fwd', 'dgrad', 'wgrad'):
    _case('%s_grid' % dir_, dir_, (4, 8, 40, 40, 64), 64, 16, seed=50, family='grid_' + dir_)

# production rows of ResNeXt-50 branch2b at 2 clips of 32 x 224^2 (32x4d and 32x8d)
PRODUCTION = [('res2', (2, 32, 56, 56), 1, 1), ('res3_0', (2, 16, 56, 56), 2, 1), ('res3', (2, 16, 28, 28), 1, 1),
              ('res4_0', (2, 16, 28, 28), 2, 1), ('res4', (2, 16, 14, 14), 1, 1), ('res5', (2, 16, 14, 14), 1, 2)]
STAGE_WIDTH = {'res2': 1, 'res3': 2, 'res4': 4, 'res5': 8}
for width in (4, 8):
    for stage, (n, t, h, w), stride, dil in PRODUCTION:
        c = 32 * width * STAGE_WIDTH[stage.split('_')[0]]
        for dir_ in ('fwd', 'dgrad', 'wgrad'):
            epi = dict(scale=1, bias=1, relu=1, tf32=1, bits=1) if dir_ == 'fwd' else (
                dict(mask='bits', tf32=1) if dir_ == 'dgrad' else dict(row_scale=1))
            _case('prod_32x%dd_%s_%s' % (width, stage, dir_), dir_, (n, t, h, w, c), c, 32, s=(1, stride, stride),
                  d=(1, dil, dil), family='prod_' + dir_, seed=60, **epi)


# ------------------------------------------------------------------------------------------------ geometry
def geom_of(case):
    from vlfb.kernels import conv_geom
    return conv_geom((case['N'], case['T'], case['H'], case['W'], case['C']), case['Co'], case['k'], case['s'],
                     case['p'], case['d'])


def positions(case):
    g = geom_of(case)
    return g.N * g.To * g.Ho * g.Wo


def terms(case):
    """Number of products in one output element's sum."""
    taps = case['k'][0] * case['k'][1] * case['k'][2]
    if case['dir'] == 'fwd':
        return taps * case['C'] // case['groups']
    if case['dir'] == 'dgrad':
        return taps * case['Co'] // case['groups']
    return positions(case)


def grid_ctas(case):
    """CTAs of the launch, as csrc/gconv.cu sizes it (wgrad: the position split is capped at about 4 x 132 CTAs of
    256 threads; `wgrad_split_capped` tells whether the cap binds)."""
    g = geom_of(case)
    if case['dir'] == 'wgrad':
        cig = g.C // case['groups']
        pairs = g.kT * g.kH * g.kW * cig // 4
        units = (g.Co // 4) * -(-pairs // 4)
        block = units if units >= 256 else -(-units // 32) * 32
        block = min(block, 256)
        gy = -(-units // block)
        k = positions(case)
        splits = max(1, min((132 * 4 * 256) // (gy * block), -(-k // 32)))
        per = -(-k // splits)
        return -(-k // per) * gy
    m = g.N * g.To * g.Ho * g.Wo if case['dir'] == 'fwd' else g.N * g.T * g.H * g.W
    cd = g.Co if case['dir'] == 'fwd' else g.C
    return -(-m // 64) * -(-cd // 64)


GRID_CAP = 132 * 16


def wgrad_split_capped(case):
    g = geom_of(case)
    pairs = g.kT * g.kH * g.kW * (g.C // case['groups']) // 4
    units = (g.Co // 4) * -(-pairs // 4)
    block = min(256, units if units >= 256 else -(-units // 32) * 32)
    gy = -(-units // block)
    return (132 * 4 * 256) // (gy * block) < -(-positions(case) // 32)


def check_table():
    names = [c['name'] for c in CASES]
    assert len(names) == len(set(names)), 'duplicate case names'
    widths = {}
    for c in CASES:
        g = geom_of(c)
        G = c['groups']
        assert c['C'] % G == 0 and c['Co'] % G == 0
        cig, cog = c['C'] // G, c['Co'] // G
        assert cig % 4 == 0 and cog % 4 == 0 and 4 <= cig <= 64 and 4 <= cog <= 64, c['name']
        assert g.To > 0 and g.Ho > 0 and g.Wo > 0, c['name']
        if c['epi'].get('bits'):
            assert c['epi'].get('relu') and (c['Co'] if c['dir'] == 'fwd' else c['C']) % 32 == 0, c['name']
        widths.setdefault(c['dir'], set()).update([(cig, cog)])
    for d in ('fwd', 'dgrad', 'wgrad'):
        ws = widths[d]
        assert all((cg, cg) in ws for cg in (4, 8, 16, 32, 64)), d
        assert any(a != b for a, b in ws), d
        cs = [c for c in CASES if c['dir'] == d]
        assert any(c['s'][1] == 2 for c in cs) and any(c['d'][1] == 2 for c in cs), d
        assert any(c['k'] == (3, 3, 3) for c in cs) and any(c['k'] == (1, 3, 3) for c in cs), d
        assert any(c['N'] > 1 for c in cs) and any(c['H'] != c['W'] and c['H'] % 8 for c in cs), d
        above = (lambda c: wgrad_split_capped(c)) if d == 'wgrad' else (lambda c: grid_ctas(c) > GRID_CAP)
        assert any(above(c) for c in cs), 'no %s case above the grid cap' % d
    fields = set()
    for c in CASES:
        fields.update(k if k != 'mask' else 'mask_' + c['epi']['mask'] for k in c['epi'])
    for f in ('scale', 'bias', 'residual', 'relu', 'mask_float', 'mask_bits', 'accum', 'tf32', 'bits', 'row_scale',
              'col_scale', 'alpha'):
        assert f in fields, 'no case uses the epilogue field %s' % f
    prod = set(c['name'] for c in CASES if c['name'].startswith('prod_'))
    assert len(prod) == 2 * len(PRODUCTION) * 3


# ------------------------------------------------------------------------------------------------ reference
def _nc(x):
    return x.permute(0, 4, 1, 2, 3)


def _cl(x):
    return x.permute(0, 2, 3, 4, 1).contiguous()


def make_tensors(case, device):
    """fp32 TF32-rounded operands (channels-last) and epilogue tensors, seeded."""
    g = geom_of(case)
    G = case['groups']
    gen = torch.Generator(device='cpu').manual_seed(1000 + case['seed'])

    def rnd(*shape, scale=1.0):
        return (torch.randn(shape, generator=gen) * scale).to(device)

    kt, kh, kw = case['k']
    t = {}
    t['x'] = tf32_round(rnd(g.N, g.T, g.H, g.W, g.C))
    t['w'] = tf32_round(rnd(g.Co, kt, kh, kw, g.C // G, scale=0.2))
    t['dy'] = tf32_round(rnd(g.N, g.To, g.Ho, g.Wo, g.Co))
    e = case['epi']
    d = case['dir']
    ncols = g.Co if d == 'fwd' else (g.C if d == 'dgrad' else kh * kw * (g.C // G))
    out_shape = (g.N, g.To, g.Ho, g.Wo, g.Co) if d == 'fwd' else (
        (g.N, g.T, g.H, g.W, g.C) if d == 'dgrad' else (g.Co, kt, kh, kw, g.C // G))
    t['out_shape'] = out_shape
    if e.get('scale'):
        t['scale'] = rnd(g.Co).abs() + 0.5
    if e.get('bias'):
        t['bias'] = rnd(ncols, scale=0.3)
    if e.get('row_scale'):
        t['row_scale'] = rnd(g.Co if d == 'wgrad' else out_shape[0] * out_shape[1] * out_shape[2] * out_shape[3]).abs() + 0.5
    if e.get('col_scale'):
        t['col_scale'] = (rnd(ncols) > -0.5).to(torch.float32)          # a column mask, as conv_wgrad's col_mask
    if e.get('residual'):
        t['residual'] = rnd(*out_shape)
    if e.get('accum'):
        t['prev'] = rnd(*out_shape)
    if e.get('mask'):
        t['mask'] = rnd(*out_shape)
    return t


def reference(case, t):
    """fp64 result and the per-element bound."""
    g = geom_of(case)
    G = case['groups']
    e = case['epi']
    d = case['dir']
    conv = dict(stride=case['s'], padding=case['p'], dilation=case['d'], groups=G)
    x64, w64, dy64 = _nc(t['x']).double(), t['w'].permute(0, 4, 1, 2, 3).double(), _nc(t['dy']).double()
    if d == 'fwd':
        acc = _cl(F.conv3d(x64, w64, **conv))
        mag = _cl(F.conv3d(x64.abs(), w64.abs(), **conv))
    elif d == 'dgrad':
        def dgrad(dy_, w_):
            xs = torch.zeros((g.N, g.C, g.T, g.H, g.W), dtype=torch.float64, device=dy_.device, requires_grad=True)
            F.conv3d(xs, w_, **conv).backward(dy_)
            return _cl(xs.grad)
        wsc = w64
        if e.get('scale'):           # the dgrad B operand arrives with the affine scale folded (weight_transpose)
            wsc = w64 * t['scale'].double().view(-1, 1, 1, 1, 1)
            wsc = tf32_round(wsc.float()).double()
        acc = dgrad(dy64, wsc)
        mag = dgrad(dy64.abs(), wsc.abs())
    else:
        def wgrad(x_, dy_):
            ws = torch.zeros_like(w64, requires_grad=True)
            F.conv3d(x_, ws, **conv).backward(dy_)
            return ws.grad.permute(0, 2, 3, 4, 1).contiguous()
        acc = wgrad(x64, dy64)
        mag = wgrad(x64.abs(), dy64.abs())
    alpha = float(e.get('alpha', 1.0))
    fac = torch.full_like(acc, alpha)
    bias_term = torch.zeros_like(acc)
    rs = 1.0
    if d == 'wgrad':
        if e.get('row_scale'):
            fac = fac * t['row_scale'].double().view(-1, 1, 1, 1, 1)
        if e.get('col_scale'):
            kt = case['k'][0]
            cs = t['col_scale'].double().view(1, case['k'][1], case['k'][2], -1)
            fac = fac * cs.unsqueeze(1).expand(1, kt, *cs.shape[1:])
    else:
        if e.get('scale') and d == 'fwd':
            fac = fac * t['scale'].double()
        if e.get('row_scale'):
            rs = t['row_scale'].double().view(*acc.shape[:4], 1)
            fac = fac * rs
        if e.get('bias'):
            bias_term = t['bias'].double().expand_as(acc) * rs
    v = acc * fac + bias_term           # (acc * alpha * s + bias) * row_scale, the epilogue's order
    extra = v.abs() + bias_term.abs()
    if e.get('residual'):
        v = v + t['residual'].double()
        extra = extra + t['residual'].double().abs()
    if e.get('accum'):
        v = v + t['prev'].double()
        extra = extra + t['prev'].double().abs()
    if e.get('relu'):
        v = v.clamp(min=0)
    if e.get('mask') and d != 'wgrad':
        v = torch.where(t['mask'].double() > 0, v, torch.zeros_like(v))
    bound = (terms(case) + 8) * U32 * (fac.abs() * mag) + 4 * U32 * extra
    if e.get('tf32'):
        bound = bound * (1 + TF32_ULP) + TF32_ULP * v.abs()
    return v, bound


def reference_of_call(dir, g, groups, x=None, w=None, dy=None, wt=None, scale=None, bias=None, residual=None,
                      relu=False, tf32=False, prev=None, mask=None, row_scale=None, col_scale=None):
    """`reference` of one grouped vlfb.kernels call from its arguments: dir 'fwd' (conv_fwd: x, w, scale, bias,
    residual, relu, tf32), 'dgrad' (conv_dgrad: dy, wt [C][taps][Cog] with any scale already folded in, prev = dx when
    it accumulates, residual, mask = the ReLU mask as floats, tf32) or 'wgrad' (conv_wgrad: dy, x, prev = dw, row_scale,
    col_scale = the col_mask).  Tensors channels-last as the wrapper takes them.  Returns (fp64 result in the output's
    shape, bound)."""
    case = dict(dir=dir, N=g.N, T=g.T, H=g.H, W=g.W, C=g.C, Co=g.Co, groups=int(groups), k=(g.kT, g.kH, g.kW),
                s=(g.sT, g.sH, g.sW), p=(g.pT, g.pH, g.pW), d=(g.dT, g.dH, g.dW), epi={})
    G, cig, cog, taps = int(groups), g.C // int(groups), g.Co // int(groups), g.kT * g.kH * g.kW
    dev = next(v for v in (x, dy, w, wt) if v is not None).device
    z = lambda *s: torch.zeros(s, dtype=torch.float64, device=dev)
    if wt is not None:               # w[gi Cog + o][tap][i] = wt[gi Cig + i][tap][o]
        w = wt.reshape(G, cig, taps, cog).permute(0, 3, 2, 1).reshape(g.Co, g.kT, g.kH, g.kW, cig)
    t = dict(x=x if x is not None else z(g.N, g.T, g.H, g.W, g.C),
             w=w if w is not None else z(g.Co, g.kT, g.kH, g.kW, cig),
             dy=dy if dy is not None else z(g.N, g.To, g.Ho, g.Wo, g.Co))
    for k, v in (('scale', scale), ('bias', bias), ('residual', residual), ('prev', prev), ('mask', mask),
                 ('row_scale', row_scale), ('col_scale', col_scale)):
        if v is not None:
            t[k] = v
            case['epi']['accum' if k == 'prev' else k] = 1
    if relu:
        case['epi']['relu'] = 1
    if tf32:
        case['epi']['tf32'] = 1
    return reference(case, t)


# ------------------------------------------------------------------------------------------------ running
def prepare(case, t, out, bits):
    """The vlfb_gemm parameter block of the case (dgrad: the grouped wt is built here) and the tensors it reads."""
    from vlfb import kernels as K
    g = geom_of(case)
    e = case['epi']
    G = case['groups']
    d = case['dir']
    mask = t.get('mask') if e.get('mask') == 'float' else None
    mbits = pack_sign_bits(t['mask']) if e.get('mask') == 'bits' else None
    if d == 'fwd':
        p = _params_fwd(K, case, t, out, g, G, mask, mbits, bits)
    elif d == 'dgrad':
        p = _params_dgrad(K, case, t, out, g, G, mask, mbits, bits)
    else:
        p = _params_wgrad(K, case, t, out, g, G)
    p.alpha = float(e.get('alpha', 1.0))
    p.deterministic = int(e.get('det', 0))
    return p, (mask, mbits)


def fire(p):
    """ONE vlfb_gemm call."""
    from vlfb import kernels as K
    from vlfb import libvlfb as L
    K._check(L.load().vlfb_gemm(ctypes.byref(p), K._stream()), 'vlfb_gemm')


def launch(case, t, out, bits):
    p, keep = prepare(case, t, out, bits)
    fire(p)
    return keep                 # kept alive until the launch completes


def _epi(K, p, t, e, mask, mbits, bits, col_scale):
    from vlfb import libvlfb as L
    if e.get('scale') and col_scale:
        p.col_scale = t['scale'].data_ptr()
    if e.get('bias'):
        p.col_bias = t['bias'].data_ptr()
    if e.get('row_scale'):
        p.row_scale = t['row_scale'].data_ptr()
    if e.get('residual'):
        p.residual = t['residual'].data_ptr()
    if e.get('relu'):
        p.flags |= L.EPI_RELU
    if e.get('accum'):
        p.flags |= L.EPI_ACCUM
    if e.get('tf32'):
        p.flags |= L.EPI_TF32
    if mask is not None:
        p.relu_mask = mask.data_ptr()
    if mbits is not None:
        p.relu_mask_bits = mbits.data_ptr()
    if bits is not None:
        p.relu_bits_out = bits.data_ptr()


def _params_fwd(K, case, t, out, g, G, mask, mbits, bits):
    from vlfb import libvlfb as L
    cig = g.C // G
    Kd = g.kT * g.kH * g.kW * cig
    p = K._base_params(g.N * g.To * g.Ho * g.Wo, g.Co, Kd, out, g.Co)
    p.a = K._operand(t['x'], L.OP_CONV_K)
    p.b = K._operand(t['w'], L.OP_DENSE_K, ld=Kd)
    p.g = g
    p.groups = G
    _epi(K, p, t, case['epi'], mask, mbits, bits, col_scale=True)
    return p


def _params_dgrad(K, case, t, out, g, G, mask, mbits, bits):
    from vlfb import libvlfb as L
    cog = g.Co // G
    taps = g.kT * g.kH * g.kW
    wt = torch.empty((g.C, taps, cog), dtype=torch.float32, device=out.device)
    K.weight_transpose(t['w'], wt, t.get('scale'), groups=G)       # scale folded: the affine of the fwd conv
    t['wt'] = wt
    Kd = taps * cog
    p = K._base_params(g.N * g.T * g.H * g.W, g.C, Kd, out, g.C)
    p.a = K._operand(t['dy'], L.OP_DGRAD_K)
    p.b = K._operand(wt, L.OP_DENSE_K, ld=Kd)
    p.g = g
    p.groups = G
    _epi(K, p, t, case['epi'], mask, mbits, bits, col_scale=False)     # dgrad: the scale is folded into wt
    return p


def _params_wgrad(K, case, t, out, g, G):
    from vlfb import libvlfb as L
    cig = g.C // G
    n = g.kH * g.kW * cig
    p = K._base_params(g.Co, n, g.N * g.To * g.Ho * g.Wo, out, g.kT * n)
    p.a = K._operand(t['dy'], L.OP_DENSE_MN, ld=g.Co)
    p.b = K._operand(t['x'], L.OP_CONV_MN)
    p.g = g
    p.taps = g.kT
    p.d_tap_stride = n
    p.split_k = 0
    p.groups = G
    p.flags |= L.EPI_ATOMIC
    e = case['epi']
    if e.get('row_scale'):
        p.row_scale = t['row_scale'].data_ptr()
    if e.get('col_scale'):
        p.col_scale = t['col_scale'].data_ptr()
    return p


def verdict(buf, got, bits, ref, bound):
    """(ok, stats dict) of one launch's output `got` (inside the guarded `buf`) and its sign bits."""
    cmp = compare(got, ref, bound)
    guard_ok = guard_touched(buf, torch.arange(GUARD, GUARD + got.numel(), device=buf.device)) == 0
    bits_ok = bits is None or torch.equal(bits.cpu(), pack_sign_bits(got.reshape(-1).cpu()))
    return cmp['ok'] and guard_ok and bits_ok, dict(ratio=cmp['worst_ratio'], guard_ok=guard_ok, bits_ok=bits_ok,
                                                    finite=cmp['nonfinite'] == 0)


def _setup(case, device):
    """The case's tensors, fp64 reference and bound, and its output: GUARD elements of NaN on each side of it in
    `buf`, starting from the case's prev (or zero for a wgrad, which accumulates)."""
    t = make_tensors(case, device)
    ref, bound = reference(case, t)
    n = 1
    for s in t['out_shape']:
        n *= s
    buf = nan_buffer(n + 2 * GUARD, device)
    out = buf[GUARD:GUARD + n].view(t['out_shape'])
    if 'prev' in t:
        out.copy_(t['prev'])
    elif case['dir'] == 'wgrad':
        out.zero_()
    bits = torch.zeros(n // 32, dtype=torch.int32, device=device) if case['epi'].get('bits') else None
    return t, ref, bound, buf, out, bits


def run_case(case, device='cuda', keep_out=False):
    """Runs the case once; returns its stats (with keep_out, also 'out': the guarded output buffer and the sign bits as
    int32 bits, for a bitwise comparison of two runs)."""
    t, ref, bound, buf, out, bits = _setup(case, device)

    def go():
        keep = launch(case, t, out, bits)
        torch.cuda.synchronize()
        return keep
    _, text = capture_fd2(go)
    ok, st = verdict(buf, out, bits, ref, bound)
    rec = next((r for r in (parse_record(l, 'gconv') for l in text.splitlines()) if r is not None), None)
    G = case['groups']
    want = dict(path='gconv', dir=case['dir'], groups=str(G), cig=str(case['C'] // G), cog=str(case['Co'] // G))
    st['record'] = rec
    st['record_ok'] = rec is not None and all(rec.get(k) == v for k, v in want.items())
    st['ok'] = ok and st['record_ok']
    if keep_out:
        st['out'] = torch.cat([buf.view(torch.int32)] + ([bits] if bits is not None else [])).cpu()
    return st


# ------------------------------------------------------------------------------------------------ CPU emulation
def emulate(case, t, buf, out, bits, plant=None):
    """What a correct kernel stores (fp32 torch ops), optionally with a planted bug."""
    e = case['epi']
    G = case['groups']
    conv = dict(stride=case['s'], padding=case['p'], dilation=case['d'], groups=G)
    x, w, dy = _nc(t['x']), t['w'].permute(0, 4, 1, 2, 3), _nc(t['dy'])
    if plant == 'missing_tap':
        w = w.clone()
        w[:, :, -1, -1, -1] = 0
    if plant == 'neighbour_group':
        cig = case['C'] // G
        x = torch.roll(x, cig, dims=1)
    if plant == 'wrong_dilation':
        conv['padding'] = tuple(p - (d - 1) * (k // 2) for p, d, k in zip(case['p'], case['d'], case['k']))
        conv['dilation'] = (1, 1, 1)
    d = case['dir']
    if d == 'fwd':
        v = _cl(F.conv3d(x, w, **conv)) * float(e.get('alpha', 1.0))
        if e.get('scale'):
            v = v * t['scale']
        if e.get('bias'):
            v = v + t['bias']
    elif d == 'dgrad':
        ws = w if not e.get('scale') else tf32_round(w * t['scale'].view(-1, 1, 1, 1, 1))
        xs = torch.zeros_like(x, requires_grad=True)
        F.conv3d(xs, ws, **conv).backward(dy)
        v = _cl(xs.grad) * float(e.get('alpha', 1.0))
        if plant == 'dgrad_parity':
            v = torch.roll(v, 1, dims=3)
        if e.get('bias'):
            v = v + t['bias']
    else:
        ws = torch.zeros_like(w, requires_grad=True)
        F.conv3d(x, ws, **conv).backward(dy)
        v = ws.grad.permute(0, 2, 3, 4, 1) * float(e.get('alpha', 1.0))
        if e.get('row_scale'):
            v = v * t['row_scale'].view(-1, 1, 1, 1, 1)
    if d != 'wgrad' and e.get('row_scale'):
        v = v * t['row_scale'].view(*v.shape[:4], 1)
    if e.get('residual'):
        v = v + t['residual']
    if e.get('accum') or d == 'wgrad':
        v = v + out
    if e.get('relu'):
        v = v.clamp(min=0)
    if e.get('mask') and d != 'wgrad':
        v = torch.where(t['mask'] > 0, v, torch.zeros_like(v))
    if e.get('tf32'):
        v = tf32_round(v.contiguous())
    if plant == 'missing_border_row':
        v = v.clone()
        v[:, :, -1] = 0
    out.copy_(v)
    if plant == 'guard_write':
        buf[GUARD + out.numel()] = 0.0
    if bits is not None:
        bits.copy_(pack_sign_bits(out.reshape(-1)))


def run_case_cpu(case, plant=None):
    t, ref, bound, buf, out, bits = _setup(case, 'cpu')
    emulate(case, t, buf, out, bits, plant)
    return verdict(buf, out, bits, ref, bound)


def _by_name(name):
    return next(c for c in CASES if c['name'] == name)


# planted bug -> (a small case that exercises it, plant name)
PLANTS = {
    'missing_tap': (_by_name('fwd_cg8'), 'missing_tap'),
    'neighbour_group': (_by_name('fwd_cig8_cog16'), 'neighbour_group'),
    'wrong_dilation': (_by_name('fwd_d2'), 'wrong_dilation'),
    'dgrad_parity': (_by_name('dgrad_s2'), 'dgrad_parity'),
    'missing_border_row': (_by_name('fwd_s2'), 'missing_border_row'),
    'guard_write': (_by_name('dgrad_cg4'), 'guard_write'),
}


# ------------------------------------------------------------------------------------------------ ABI rules
def _base():
    from vlfb import libvlfb as L
    from vlfb.kernels import conv_geom
    p = L.GemmParams()
    p.g = conv_geom((1, 1, 8, 8, 128), 128, (1, 3, 3), (1, 1, 1), (0, 1, 1))
    p.a.ptr, p.a.kind = 256, L.OP_CONV_K
    p.b.ptr, p.b.kind, p.b.ld = 512, L.OP_DENSE_K, 36
    p.d, p.ldd = 1024, 128
    p.M, p.N, p.K, p.batch, p.taps, p.split_k, p.alpha, p.groups = 64, 128, 36, 1, 1, 1, 1.0, 32
    return p


def _rule(code, needle, **kw):
    def make():
        from vlfb import libvlfb as L
        p = _base()
        for k, v in kw.items():
            if k == 'a_kind':
                p.a.kind = getattr(L, v)
            elif k == 'a_ptr':
                p.a.ptr = v
            elif k == 'a_ld':
                p.a.ld = v
            elif k == 'b_kind':
                p.b.kind = getattr(L, v)
            elif k == 'b_ld':
                p.b.ld = v
            elif k.startswith('g_'):
                setattr(p.g, k[2:], v)
            else:
                setattr(p, k, v)
        return p, code, needle
    return make


BADARG, UNSUPPORTED = -1, -2
ABI_RULES = {
    'negative_groups': _rule(BADARG, 'groups >= 0', groups=-1),
    'c_not_divisible': _rule(BADARG, 'must divide', groups=3),
    'cig_below_4': _rule(UNSUPPORTED, 'multiples of 4 in [4, 64]', groups=64),
    'cig_above_64': _rule(UNSUPPORTED, 'multiples of 4 in [4, 64]', groups=2, g_C=256, g_Co=256),
    'cig_not_multiple_of_4': _rule(UNSUPPORTED, 'multiples of 4 in [4, 64]', groups=16, g_C=96, K=54),
    'dense_k_a': _rule(UNSUPPORTED, 'DENSE_K A operand', a_kind='OP_DENSE_K'),
    'stem': _rule(UNSUPPORTED, 'STEM_*', a_kind='OP_STEM_K'),
    'batch': _rule(UNSUPPORTED, 'batch == 1', batch=2),
    'split_k': _rule(UNSUPPORTED, 'split_k <= 1', split_k=2, flags=4),
    'fwd_atomic': _rule(UNSUPPORTED, 'no VLFB_EPI_ATOMIC', flags=4),
    'fwd_wrong_k': _rule(BADARG, 'K = taps*Cig', K=128 * 9, b_ld=128 * 9),
    'dgrad_wrong_k': _rule(BADARG, 'K = taps*Cog', a_kind='OP_DGRAD_K', K=128 * 9, b_ld=128 * 9),
    'wgrad_needs_atomic': _rule(BADARG, 'VLFB_EPI_ATOMIC', a_kind='OP_DENSE_MN', a_ld=128, b_kind='OP_CONV_MN',
                                M=128, N=36, K=64, flags=0),
    'wgrad_epilogue': _rule(BADARG, 'alpha, col_scale and row_scale only', a_kind='OP_DENSE_MN', a_ld=128,
                            b_kind='OP_CONV_MN', M=128, N=36, K=64, flags=4 | 1),
    'misaligned': _rule(BADARG, '16-byte aligned', a_ptr=260),
    'bits_need_relu': _rule(BADARG, 'relu_bits_out', relu_bits_out=2048),
    'too_large': _rule(BADARG, '2^31', g_N=1 << 18, M=64 << 18),
}


# ------------------------------------------------------------------------------------------------ script
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--only', default='')
    args = ap.parse_args()
    if os.environ.get('VLFB_DEBUG') != '1':
        raise SystemExit('the path records need VLFB_DEBUG=1')
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    with open(args.out, 'w') as f:
        for c in CASES:
            if args.only and not re.search(args.only, c['name']):
                continue
            print('[gconv_cases] %s' % c['name'], flush=True)
            st = run_case(c)
            st.update(name=c['name'], family=c['family'])
            f.write(json.dumps(st) + '\n')
            f.flush()
            torch.cuda.empty_cache()


if __name__ == '__main__':
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    for p_ in (os.path.join(root, 'video-long-term-feature-banks_b200', 'lib'), root, here):
        if p_ not in sys.path:
            sys.path.insert(0, p_)
    main()
