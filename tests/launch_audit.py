"""Launch audit: every kernel call of a real step, checked against fp64 from the call's own tensors.

`Audit` stands in for the kernel module the executor calls through (vlfb.executor.K).  Each outermost call of an
audited wrapper
  1. binds its arguments (inspect.signature of the wrapped function) and clones every tensor argument, outputs
     included (accumulate flags, atomics and aliasing read them), and snapshots the storage around every output;
  2. runs the real call (and synchronizes on CUDA);
  3. computes the wrapper's reference in fp64 from the clones and checks every written element against the family's
     bound (streaming_cases.py / gemm_paths.py derive them), bit for bit where the operation is exact;
  4. checks that nothing else in the outputs' storage changed (row gaps, neighbouring Concat slices, a margin
     before and after the view), bit for bit;
  5. checks that every float tensor the call reads is finite;
  6. for GEMMs on a TF32 engine: checks that both operands are TF32-exact (low 13 mantissa bits zero).  The value
     reference reads the operands as the tensor core does (truncated), so a rounding lapse is reported once, as an
     exactness failure.  On the SIMT engine and the CPU stand-in the operands are used as they are.
Each call is compared with its own inputs, so TF32 differences never build up across the network and the tolerance
stays at kernel level.  A wrapper without a reference is a failure, not a skip.

The module also runs audited nets on the GPU in a subprocess (the GEMM path records of VLFB_DEBUG are read once per
process):  python tests/launch_audit.py --net NAME --out FILE
"""
import argparse
import inspect
import json
import os
import sys
import time
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (os.path.join(ROOT, 'video-long-term-feature-banks_b200', 'lib'), ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import gconv_cases as GC  # noqa: E402
import gemm_paths as GP  # noqa: E402
import streaming_cases as SC  # noqa: E402
from streaming_cases import U, C_SUM, sum_bound  # noqa: E402
from util import capture_fd2, compare, pack_sign_bits, parse_record, tf32_round  # noqa: E402

GEMM_WRAPPERS = ('conv_fwd', 'conv_dgrad', 'conv_wgrad', 'conv_wgrad_det', 'matmul', 'matmul_det')
DET_WRAPPERS = ('colsum_det', 'spatial_bn_fwd_det', 'spatial_bn_bwd_det', 'roi_align_bwd_det')
AUDITED = GEMM_WRAPPERS + SC.STREAMING_WRAPPERS + DET_WRAPPERS

# The two operands of each GEMM wrapper (the A and B the tensor core reads).
GEMM_OPERANDS = {'conv_fwd': ('x', 'w'), 'conv_dgrad': ('dy', 'wt'), 'conv_wgrad': ('dy', 'x'),
                 'conv_wgrad_det': ('dy', 'x'), 'matmul': ('a', 'b'), 'matmul_det': ('a', 'b')}

# GEMM operands allowed to be not TF32-exact: (wrapper, operand) -> reason.  Empty: every operand of the audited nets is
# rounded by its producer.
EXACTNESS_EXCEPTIONS = {}

# Float inputs allowed to hold non-finite values: (wrapper, argument) -> reason.
NONFINITE_EXCEPTIONS = {}

MARGIN = 64                    # elements checked before and after every output's span


class NoReference(Exception):
    pass


# ----------------------------------------------------------------------------------------------- small helpers
def _bits(t):
    return t.contiguous().view({4: torch.int32, 8: torch.int64, 2: torch.int16, 1: torch.uint8}[t.element_size()])


def tf32_trunc(t):
    """The operand as the tensor core reads it: the low 13 mantissa bits dropped."""
    i = t.float().contiguous().view(torch.int32)
    return (i & ~0x1FFF).view(torch.float32).to(t.dtype).view(t.shape)


def not_tf32_exact(t):
    """Number of elements of t that a TF32 operand cannot hold exactly."""
    f = t.float()
    bad = (f.contiguous().view(torch.int32) & 0x1FFF) != 0
    if t.dtype != torch.float32:
        bad = bad | (f.to(t.dtype) != t)
    return int(bad.sum())


def _d(t):
    return None if t is None else t.double()


def _geom(g):
    return dict((f, int(getattr(g, f))) for f in SC.GEOM_FIELDS)


def _offsets(v):
    """Storage element offsets of every element of the view v (same shape as v)."""
    off = torch.full((), v.storage_offset(), dtype=torch.int64, device=v.device)
    for d, (s, st) in enumerate(zip(v.shape, v.stride())):
        shape = [1] * v.dim()
        shape[d] = s
        off = off + (torch.arange(s, device=v.device, dtype=torch.int64) * st).view(shape)
    return off.expand(v.shape)


def _storage(t):
    n = t.untyped_storage().nbytes() // t.element_size()
    return torch.empty(0, dtype=t.dtype, device=t.device).set_(t.untyped_storage(), 0, (n,), (1,))


def _tensors(v, path):
    """(path, tensor) of every tensor inside an argument (dicts and lists of the FBO stack / transpose jobs)."""
    if torch.is_tensor(v):
        yield path, v
    elif isinstance(v, dict):
        for k in v:
            yield from _tensors(v[k], '%s.%s' % (path, k))
    elif isinstance(v, (list, tuple)):
        for i, x in enumerate(v):
            yield from _tensors(x, '%s[%d]' % (path, i))


def _clone(v):
    if torch.is_tensor(v):
        return v.clone()
    if isinstance(v, dict):
        return dict((k, _clone(x)) for k, x in v.items())
    if isinstance(v, list):
        return [_clone(x) for x in v]
    if isinstance(v, tuple):
        return tuple(_clone(x) for x in v)
    return v


def layout(a):
    """Strides, storage offsets and 16-byte alignment of the tensor arguments of a call."""
    out = {}
    for name, v in a.items():
        for path, t in _tensors(v, name):
            out[path] = dict(stride=list(t.stride()), offset=int(t.storage_offset()),
                             align16=int((t.data_ptr() % 16) // t.element_size()) if t.numel() else 0)
    return out


# ----------------------------------------------------------------------------------------------- outputs of each wrapper
# wrapper -> (written arguments that the call also reads, written arguments it only writes).  Paths name tensors inside
# dicts / lists ('layers[*].theta').  Everything else is an input.
_OUT = {
    'conv_fwd': ((), ('y', 'relu_bits')), 'conv_dgrad': (('dx',), ()), 'conv_wgrad': (('dw',), ()),
    'conv_wgrad_det': (('dw',), ()), 'matmul': (('d',), ()), 'matmul_det': (('d',), ()),
    'weight_transpose': ((), ('wt',)), 'weight_transpose_multi': ((), ('jobs[*][1]',)),
    'affine_fwd': ((), ('y',)), 'affine_bwd': ((), ('dx',)),
    'spatial_bn_fwd': (('rm', 'rv'), ('sm', 'siv', 'y')), 'spatial_bn_fwd_det': (('rm', 'rv'), ('sm', 'siv', 'y')),
    'spatial_bn_infer': ((), ('y',)), 'spatial_bn_bwd': (('ds', 'db'), ('dx',)),
    'spatial_bn_bwd_det': (('ds', 'db'), ('dx',)),
    'maxpool_fwd': ((), ('y', 'argmax')), 'maxpool_bwd': (('dx',), ()), 'maxpool_bwd_gather': ((), ('dx',)),
    'avgpool_fwd': ((), ('y',)), 'avgpool_bwd': (('dx',), ()),
    'roi_align_fwd': ((), ('out',)), 'roi_align_bwd': (('dfeat',), ()), 'roi_align_bwd_det': (('dfeat',), ()),
    'softmax_fwd': ((), ('p',)), 'softmax_bwd': ((), ('dx',)), 'layernorm_fwd': ((), ('y', 'mean', 'std')),
    'layernorm_bwd': ((), ('dx',)), 'relu_fwd': ((), ('y',)), 'relu_bwd': ((), ('dx',)), 'axpby': ((), ('out',)),
    'fill': ((), ('x',)), 'round_tf32': ((), ('y',)), 'add_tf32': ((), ('out',)), 'relu_tf32': ((), ('y',)),
    'add_relu_bwd_tf32': ((), ('out',)), 'relu_bits': ((), ('bits',)), 'relu_bwd_tf32': ((), ('dx',)),
    'colsum': (('out',), ()), 'colsum_det': (('out',), ()), 'sigmoid_fwd': ((), ('y',)), 'dropout': ((), ('y',)),
    'copy2d': (('dst',), ()), 'nc_to_cl': ((), ('dst',)), 'cl_to_nc': ((), ('dst',)),
    'sigmoid_ce_fwd': ((), ('loss',)), 'sigmoid_ce_bwd': ((), ('dlogits',)),
    'softmax_ce_fwd': ((), ('prob', 'loss')), 'softmax_ce_bwd': ((), ('dlogits',)),
    'sgd_nesterov': (('p', 'g', 'm'), ('p_tf32',)),
    'fbo_nl_fwd': ((), tuple('layers[*].' + k for k in ('theta', 'prob', 's', 't', 'xhat', 'ln_mean', 'ln_std', 'out',
                                                        'a_out'))),
    'fbo_nl_bwd': (tuple('layers[*].g' + k for k in SC.FBO_W), ('da0', 'dbp')),
    'fbo_bank_scan': ((), ('out', 'prob')), 'cast_bf16': ((), ('y',)), 'lfb_gather': ((), ('out',)),
    'roi_align_table': ((), ()),
}


def _match(path, pattern):
    import re
    return re.fullmatch(re.escape(pattern).replace(r'\[\*\]', r'\[\d+\]'), path) is not None


# outputs read only when the call's accumulate flag is set
_ACCUM_OUT = {'matmul': 'd', 'matmul_det': 'd', 'conv_dgrad': 'dx', 'copy2d': 'dst', 'colsum': 'out', 'colsum_det': 'out',
              'avgpool_bwd': 'dx'}


def _role(fn, path, a=None):
    reads, writes = _OUT[fn]
    if _ACCUM_OUT.get(fn) == path and a is not None and not a.get('accumulate'):
        return 'out'
    if any(_match(path, p) for p in writes):
        return 'out'
    if any(_match(path, p) for p in reads):
        return 'inout'
    return 'in'


# ----------------------------------------------------------------------------------------------- references
# REF[fn](c) -> [(output name, the output view after the call, fp64 reference, bound or None for bit-exact)].
# c: .b = the arguments before the call (clones), .a = the arguments themselves (after the call), .ret = the return
# value, .engine, .dev.
REF = {}


def ref(*names):
    def reg(f):
        for n in names:
            REF[n] = f
        return f
    return reg


def _gemm_operand(c, t):
    return tf32_trunc(t) if c.engine == 'tcgen05' else t


def _gemm_bound(c, mag, K):
    """mag scaled so that finish()'s tau(K) bound also covers a sequential fp32 chain of K terms (the SIMT engine)."""
    if c.engine == 'tcgen05':
        return mag
    return mag * max(1.0, C_SUM * (K + 2) * U / GP.tau(K))


def _case_geom(g):
    return dict(N=g.N, T=g.T, H=g.H, W=g.W, C=g.C, Co=g.Co, ker=(g.kT, g.kH, g.kW), st=(g.sT, g.sH, g.sW),
                pd=(g.pT, g.pH, g.pW), dil=(g.dT, g.dH, g.dW))


def _ncthw(x):
    return x.permute(0, 4, 1, 2, 3)


def _conv_acc(op, g, x=None, w=None, dy=None):
    """(acc, mag) of the convolution GEMM in its output layout (gemm_paths.conv_refs): x / dy channels-last, w
    [Co, kT, kH, kW, C] (stem [Co, kT, kH, 8, 4])."""
    c = dict(op=op, geom=_case_geom(g))
    To, Ho, Wo = g.To, g.Ho, g.Wo
    dev = (x if x is not None else dy).device
    z = lambda *s: torch.zeros(s, dtype=torch.float64, device=dev)
    xn = _ncthw(x) if x is not None else z(g.N, g.C, g.T, g.H, g.W)
    wn = w.permute(0, 4, 1, 2, 3) if w is not None else z(g.Co, g.C, g.kT, g.kH, 8 if g.C == 4 else g.kW)
    dyn = _ncthw(dy) if dy is not None else z(g.N, g.Co, To, Ho, Wo)
    return GP.conv_refs(c, xn, wn, dyn, dev)


@ref('conv_fwd')
def _conv_fwd(c):
    b, a = c.b, c.a
    g = b['g']
    x, w = _d(_gemm_operand(c, b['x'])), _d(_gemm_operand(c, b['w']))
    if int(b.get('groups') or 1) > 1:
        r, bound = GC.reference_of_call('fwd', g, b['groups'], x=x, w=w, scale=_d(b['scale']), bias=_d(b['bias']),
                                        residual=_d(b['residual']), relu=bool(b['relu']), tf32=bool(b['tf32_out']))
        return _with_bits(c, [('y', a['y'], r, bound)])
    acc, mag = _conv_acc('conv_fwd', g, x=x, w=w)
    Kd = g.kT * g.kH * (32 if g.C == 4 else g.kW * g.C)
    Z, M, N = acc.shape
    epi = dict(relu=bool(b['relu']), tf32=bool(b['tf32_out']), cs=_d(b['scale']), cb=_d(b['bias']))
    if b['residual'] is not None:
        epi['res'] = _d(b['residual']).reshape(Z, M, N)
    r, bound = GP.finish(acc, _gemm_bound(c, mag, Kd), epi, Kd)
    y = a['y']
    return _with_bits(c, [('y', y, r.view(y.shape), bound.reshape(y.shape))])


def _with_bits(c, out):
    if c.b['relu_bits'] is not None:
        bits = c.a['relu_bits']
        out.append(('relu_bits', bits, pack_sign_bits(c.a['y'].reshape(-1)).view(bits.shape), None))
    return out


def _unpack_bits(bits, n):
    v = bits.reshape(-1).to(torch.int64) & 0xFFFFFFFF
    return (((v.view(-1, 1) >> torch.arange(32, device=bits.device)) & 1) > 0).reshape(-1)[:n]


@ref('conv_dgrad')
def _conv_dgrad(c):
    b, a = c.b, c.a
    g = b['g']
    if int(b.get('groups') or 1) > 1:
        mask = None
        if b['relu_mask'] is not None:
            mask = _d(b['relu_mask'])
        if b['relu_mask_bits'] is not None:
            mask = _unpack_bits(b['relu_mask_bits'], a['dx'].numel()).double().view(a['dx'].shape)
        r, bound = GC.reference_of_call('dgrad', g, b['groups'], dy=_d(_gemm_operand(c, b['dy'])),
                                        wt=_d(_gemm_operand(c, b['wt'])), residual=_d(b['residual']),
                                        prev=_d(b['dx']) if b['accumulate'] else None, mask=mask,
                                        tf32=bool(b['tf32_out']))
        return [('dx', a['dx'], r, bound)]
    taps = g.kT * g.kH * g.kW
    wt = _d(_gemm_operand(c, b['wt']))
    w = wt.reshape(g.C, taps, g.Co).permute(2, 1, 0).reshape(g.Co, g.kT, g.kH, g.kW, g.C)
    dy = _d(_gemm_operand(c, b['dy']))
    acc, mag = _conv_acc('conv_dgrad', g, w=w, dy=dy)
    Kd = taps * g.Co
    Z, M, N = acc.shape
    epi = dict(tf32=bool(b['tf32_out']))
    if b['accumulate']:
        epi['prev'] = _d(b['dx']).reshape(Z, M, N)
    if b['residual'] is not None:
        epi['res'] = _d(b['residual']).reshape(Z, M, N)
    if b['relu_mask'] is not None:
        epi['keep'] = (b['relu_mask'] > 0).reshape(Z, M, N)
    if b['relu_mask_bits'] is not None:
        epi['keep'] = _unpack_bits(b['relu_mask_bits'], Z * M * N).view(Z, M, N)
    r, bound = GP.finish(acc, _gemm_bound(c, mag, Kd), epi, Kd)
    dx = a['dx']
    return [('dx', dx, r.view(dx.shape), bound.reshape(dx.shape))]


@ref('conv_wgrad', 'conv_wgrad_det')
def _conv_wgrad(c):
    b, a = c.b, c.a
    g = b['g']
    dy, x = _d(_gemm_operand(c, b['dy'])), _d(_gemm_operand(c, b['x']))
    if int(b.get('groups') or 1) > 1:
        r, bound = GC.reference_of_call('wgrad', g, b['groups'], x=x, dy=dy, prev=_d(b['dw']),
                                        row_scale=_d(b['row_scale']), col_scale=_d(b['col_mask']))
        return [('dw', a['dw'], r, bound)]
    acc, mag = _conv_acc('conv_wgrad', g, x=x, dy=dy)          # [kT, Co, n]
    Kd = g.N * g.To * g.Ho * g.Wo
    Z, M, N = acc.shape
    dw = a['dw']
    epi = dict(prev=_d(b['dw']).reshape(M, Z, N).permute(1, 0, 2), rs=_d(b['row_scale']))
    if b['col_mask'] is not None:
        cm = _d(b['col_mask']).reshape(-1)
        epi['cs'] = cm.repeat(N // cm.numel()) if cm.numel() != N else cm
    r, bound = GP.finish(acc, _gemm_bound(c, mag, Kd), epi, Kd)
    back = lambda t: t.permute(1, 0, 2).reshape(dw.shape)
    return [('dw', dw, back(r), back(bound))]


@ref('matmul', 'matmul_det')
def _matmul(c):
    b, a = c.b, c.a
    A, B = _d(_gemm_operand(c, b['a'])), _d(_gemm_operand(c, b['b']))
    acc, mag = torch.bmm(A, B), torch.bmm(A.abs(), B.abs())
    Kd = A.shape[2]
    epi = dict(alpha=float(b['alpha']), cb=_d(b['bias']), tf32=bool(c.ret))
    if b['accumulate']:
        epi['prev'] = _d(b['d'])
    r, bound = GP.finish(acc, _gemm_bound(c, mag, Kd), epi, Kd)
    return [('d', a['d'], r, bound)]


@ref('weight_transpose')
def _weight_transpose(c):
    from vlfb.kernels import grouped_wt_slices
    b, a = c.b, c.a
    slabs = grouped_wt_slices(b['w'], a['wt'], b['scale'], max(int(b.get('groups', 1) or 1), 1))
    return [('wt%d' % i, wt, _wt_ref(w, s).view(wt.shape), None) for i, (w, wt, s) in enumerate(slabs)]


def _wt_ref(w, s):
    co, ci = w.shape[0], w.shape[-1]
    w3 = w.reshape(co, -1, ci)
    if s is not None:
        w3 = w3 * s.view(-1, 1, 1)             # one rounding in the tensors' dtype, as the kernel's product
    return tf32_round(w3.permute(2, 1, 0).contiguous())


@ref('weight_transpose_multi')
def _weight_transpose_multi(c):
    return [('jobs[%d]' % i, wt, _wt_ref(w, s).view(wt.shape), None)
            for i, ((w, _, s), (_, wt, _)) in enumerate(zip(c.b['jobs'], c.a['jobs']))]


@ref('axpby')
def _axpby(c):
    b = c.b
    x = _d(b['x'])
    y = _d(b['y']) if b['y'] is not None and float(b['b']) != 0.0 else torch.zeros_like(x)
    r, bound = SC.axpby_ref(x, float(b['a']), y, float(b['b']) if b['y'] is not None else 0.0)
    return [('out', c.a['out'], r.view(c.a['out'].shape), bound.view(c.a['out'].shape))]


@ref('fill')
def _fill(c):
    x = c.a['x']
    return [('x', x, torch.full_like(x, float(c.b['v'])), None)]


@ref('round_tf32')
def _round_tf32(c):
    return [('y', c.a['y'], tf32_round(c.b['x']).view(c.a['y'].shape), None)]


@ref('add_tf32')
def _add_tf32(c):
    return [('out', c.a['out'], tf32_round(c.b['x'] + c.b['y']).view(c.a['out'].shape), None)]


@ref('relu_tf32')
def _relu_tf32(c):
    return [('y', c.a['y'], tf32_round(c.b['x'].clamp(min=0)).view(c.a['y'].shape), None)]


@ref('relu_fwd')
def _relu_fwd(c):
    return [('y', c.a['y'], c.b['x'].clamp(min=0).view(c.a['y'].shape), None)]


def _where_pos(y, v):
    return torch.where(y.reshape(v.shape) > 0, v, torch.zeros((), dtype=v.dtype, device=v.device))


@ref('relu_bwd')
def _relu_bwd(c):
    return [('dx', c.a['dx'], _where_pos(c.b['y'], c.b['dy']).view(c.a['dx'].shape), None)]


@ref('relu_bwd_tf32')
def _relu_bwd_tf32(c):
    return [('dx', c.a['dx'], _where_pos(c.b['y'], tf32_round(c.b['dy'])).view(c.a['dx'].shape), None)]


@ref('add_relu_bwd_tf32')
def _add_relu_bwd_tf32(c):
    s = tf32_round(c.b['a'] + c.b['b'])
    if c.b['y'] is not None:
        s = _where_pos(c.b['y'], s)
    return [('out', c.a['out'], s.view(c.a['out'].shape), None)]


@ref('relu_bits')
def _relu_bits(c):
    return [('bits', c.a['bits'], pack_sign_bits(c.b['x'].reshape(-1)).view(c.a['bits'].shape), None)]


@ref('sigmoid_fwd')
def _sigmoid_fwd(c):
    r, bound = SC.sigmoid_ref(_d(c.b['x']))
    return [('y', c.a['y'], r.view(c.a['y'].shape), bound.view(c.a['y'].shape))]


@ref('affine_fwd', 'affine_bwd')
def _affine(c):
    b = c.b
    if c.fn == 'affine_fwd':
        r, bound = SC.affine_ref(_d(b['x']), _d(b['s']), _d(b['b']))
        return [('y', c.a['y'], r, bound)]
    r, bound = SC.affine_ref(_d(b['dy']), _d(b['s']), torch.zeros_like(_d(b['s'])))
    return [('dx', c.a['dx'], r, bound)]


@ref('colsum', 'colsum_det')
def _colsum(c):
    b = c.b
    rows, cols, ld = int(b['rows']), int(b['cols']), int(b['ld'])
    xs = _d(b['x']).reshape(-1)[:rows * ld].view(rows, ld)[:, :cols]
    prev = _d(b['out']).reshape(-1)[:cols] if b['accumulate'] else None
    # colsum_terms counts the default kernel's chains; the fixed-order kernel is held to any order of the rows
    n = SC.colsum_terms(rows, cols)[0]
    r, bound = SC.colsum_ref(xs, prev, max(n, rows + 8) if c.fn == 'colsum_det' else n)
    return [('out', c.a['out'].reshape(-1)[:cols], r, bound)]


@ref('copy2d')
def _copy2d(c):
    b, a = c.b, c.a
    rows, cols, lds, ldd = int(b['rows']), int(b['cols']), int(b['lds']), int(b['ldd'])
    src = torch.as_strided(b['src'], (rows, cols), (lds, 1), b['src'].storage_offset() + int(b['src_off']))
    dst = torch.as_strided(a['dst'], (rows, cols), (ldd, 1), a['dst'].storage_offset() + int(b['dst_off']))
    if not b['accumulate']:
        return [('dst', dst, src.clone(), None)]
    prev = torch.as_strided(b['dst'], (rows, cols), (ldd, 1), b['dst'].storage_offset() + int(b['dst_off']))
    return [('dst', dst, _d(prev) + _d(src), sum_bound(1, _d(prev).abs() + _d(src).abs(), k=0))]


@ref('dropout')
def _dropout(c):
    b = c.b
    x = b['x']
    ratio = float(b['ratio'])
    step = int(b['step'].view(-1)[0]) if b['step'] is not None else 0
    if c.engine == 'fake':
        raise NoReference('dropout of the CPU stand-in (its mask is not the Philox stream of vlfb_dropout_fwd)')
    keep = torch.from_numpy(SC.dropout_keep(x.numel(), ratio, int(b['seed']), int(b['offset']), step)).to(x.device)
    inv = float(np.float32(1.0) / (np.float32(1.0) - np.float32(ratio)))
    r = torch.where(keep.view(x.shape), x * inv, torch.zeros((), dtype=x.dtype, device=x.device))
    return [('y', c.a['y'], r.view(c.a['y'].shape), None)]


@ref('nc_to_cl')
def _nc_to_cl(c):
    b, a = c.b, c.a
    n, C_, inner = int(b['n']), int(b['c']), int(b['inner'])
    cpad = int(b['cpad'] or C_)
    v = torch.zeros((n, inner, cpad), dtype=b['src'].dtype, device=b['src'].device)
    v[:, :, :C_] = b['src'].reshape(n, C_, inner).permute(0, 2, 1)
    if b['tf32_out']:
        v = tf32_round(v)
    dst = a['dst']
    pitch = int(b.get('pitch', 0) or 0)
    if pitch:
        W, left = int(b['width']), int(b['left'])
        rows = n * inner // W
        view = torch.as_strided(dst, (rows, W, cpad), (pitch * cpad, cpad, 1), dst.storage_offset() + left * cpad)
        return [('dst', view, v.view(rows, W, cpad), None)]
    return [('dst', dst, v.view(dst.shape), None)]


@ref('cl_to_nc')
def _cl_to_nc(c):
    b = c.b
    n, C_, inner = int(b['n']), int(b['c']), int(b['inner'])
    cpad = int(b['cpad'] or C_)
    r = b['src'].reshape(n, inner, cpad)[:, :, :C_].permute(0, 2, 1)
    return [('dst', c.a['dst'], r.reshape(c.a['dst'].shape), None)]


@ref('softmax_fwd')
def _softmax_fwd(c):
    b = c.b
    r, bound = SC.softmax_fwd_ref(_d(b['x']), float(b['scale']), bool(b['tf32_out']))
    return [('p', c.a['p'], r.view(c.a['p'].shape), bound.view(c.a['p'].shape))]


@ref('softmax_bwd')
def _softmax_bwd(c):
    b = c.b
    r, bound = SC.softmax_bwd_refb(_d(b['p']), _d(b['dp']), float(b['scale']), bool(b['tf32_out']))
    return [('dx', c.a['dx'], r.view(c.a['dx'].shape), bound.view(c.a['dx'].shape))]


@ref('layernorm_fwd')
def _layernorm_fwd(c):
    b = c.b
    cols = int(b['cols'])
    r, bound, mu, dmu, sd, dsd = SC.layernorm_fwd_ref(_d(b['x']).reshape(-1, cols), float(b['eps']))
    out = [('y', c.a['y'], r.view(c.a['y'].shape), bound.view(c.a['y'].shape))]
    if b['mean'] is not None:
        out.append(('mean', c.a['mean'], mu.view(-1), dmu.view(-1)))
    if b['std'] is not None:
        out.append(('std', c.a['std'], sd.view(-1), dsd.view(-1)))
    return out


@ref('layernorm_bwd')
def _layernorm_bwd(c):
    b = c.b
    cols = int(b['cols'])
    r, bound = SC.layernorm_bwd_refb(_d(b['dy']).reshape(-1, cols), _d(b['y']).reshape(-1, cols),
                                     _d(b['std']).reshape(-1, 1))
    return [('dx', c.a['dx'], r.view(c.a['dx'].shape), bound.view(c.a['dx'].shape))]


@ref('maxpool_fwd')
def _maxpool_fwd(c):
    b, a = c.b, c.a
    g = _geom(b['g'])
    y, arg = SC.maxpool_ref(_d(b['x']), g)
    out = [('y', a['y'], y.to(a['y'].dtype).view(a['y'].shape), None)]
    if b['argmax'] is not None:
        # carve-out: among equal maxima any index of the window holding the maximum is the kernel's choice
        got = a['argmax'].long()
        C_ = g['C']
        xv = b['x'].reshape(-1, C_)
        vals = xv.gather(0, got.reshape(-1, C_).clamp(0, xv.shape[0] - 1)).view(got.shape)
        tie = (vals == y.to(vals.dtype)) & (got >= 0) & (got < xv.shape[0])
        out.append(('argmax', a['argmax'], torch.where(tie, a['argmax'], arg.to(a['argmax'].dtype)), None))
    return out


@ref('maxpool_bwd', 'maxpool_bwd_gather')
def _maxpool_bwd(c):
    b, a = c.b, c.a
    g = _geom(b['g'])
    if c.fn == 'maxpool_bwd':
        r, bound = SC.maxpool_bwd_refb(g, b['argmax'], b['dy'], prev=_d(b['dx']).view(a['dx'].shape))
    else:
        keep = (b['y'] > 0) if b['y'] is not None else None
        r, bound = SC.maxpool_bwd_refb(g, b['argmax'], b['dy'], keep, tf32_out=bool(b['tf32_out']))
    return [('dx', a['dx'], r.view(a['dx'].shape), bound.view(a['dx'].shape))]


@ref('avgpool_fwd', 'avgpool_bwd')
def _avgpool(c):
    b, a = c.b, c.a
    g = _geom(b['g'])
    if (g['pT'], g['pH'], g['pW']) != (0, 0, 0):
        raise NoReference('padded average pooling')
    if c.fn == 'avgpool_fwd':
        r, bound = SC.avgpool_fwd_ref(_d(b['x']), g)
        return [('y', a['y'], r.reshape(a['y'].shape), bound.reshape(a['y'].shape))]
    prev = _d(b['dx']).view(a['dx'].shape) if b['accumulate'] else None
    r, bound = SC.avgpool_bwd_refb(_d(b['dy']), g, prev)
    return [('dx', a['dx'], r.view(a['dx'].shape), bound.view(a['dx'].shape))]


def _live_count(b, R):
    lr = b.get('live_rows')
    return R if lr is None else min(int(lr.view(-1)[0]), R)


@ref('roi_align_fwd', 'roi_align_bwd', 'roi_align_bwd_det')
def _roi_align(c):
    b, a = c.b, c.a
    scale, sr = float(b['spatial_scale']), int(b['sampling_ratio'])
    if c.fn == 'roi_align_fwd':
        N, H, W, C_ = b['feat'].shape
        R, PH, PW, _ = b['out'].shape
    else:
        N, H, W, C_ = b['dfeat'].shape
        R, PH, PW, _ = b['dout'].shape
    live = _live_count(b, R)
    M, nmax = SC.roi_matrix(b['rois'][:live].float(), N, H, W, PH, PW, scale, sr)
    M = M.to(b['rois'].device)
    if c.fn == 'roi_align_fwd':
        f2 = _d(b['feat']).reshape(N * H * W, C_)
        r = torch.zeros((R * PH * PW, C_), dtype=torch.float64, device=f2.device)
        bound = torch.zeros_like(r)
        r[:live * PH * PW], bound[:live * PH * PW] = SC.roi_align_fwd_ref(M, nmax, f2)
        if c.engine == 'fake':
            # the CPU stand-in samples like the fp64 oracle (torchvision), not with the kernel's fp32 sample table
            import torchvision
            tv = torchvision.ops.roi_align(_d(b['feat']).permute(0, 3, 1, 2), _d(b['rois'][:live]), (PH, PW), scale,
                                           sr, False)
            r[:live * PH * PW] = tv.permute(0, 2, 3, 1).reshape(-1, C_)
        return [('out', a['out'], r.view(a['out'].shape), bound.view(a['out'].shape))]
    d2 = _d(b['dout']).reshape(R * PH * PW, C_)[:live * PH * PW]
    r, bound = SC.roi_align_bwd_ref(M, d2, _d(b['dfeat']).reshape(N * H * W, C_))
    return [('dfeat', a['dfeat'], r.view(a['dfeat'].shape), bound.view(a['dfeat'].shape))]


@ref('sigmoid_ce_fwd', 'sigmoid_ce_bwd')
def _sigmoid_ce(c):
    b, a = c.b, c.a
    x, t, scale = _d(b['logits']), b['targets'], float(b['scale'])
    if c.fn == 'sigmoid_ce_fwd':
        r, bound = SC.sigmoid_ce_fwd_ref(x, t, scale)
        return [('loss', a['loss'].reshape(-1)[:1], r, bound)]
    dl = float(b['dloss'].view(-1)[0]) if b['dloss'] is not None else 1.0
    r, bound = SC.sigmoid_ce_bwd_ref(x, t, scale, dl)
    return [('dlogits', a['dlogits'], r, bound)]


@ref('softmax_ce_fwd', 'softmax_ce_bwd')
def _softmax_ce(c):
    b, a = c.b, c.a
    scale, labd = float(b['scale']), b['labels'].long()
    if c.fn == 'softmax_ce_bwd':
        r, bound = SC.softmax_ce_bwd_ref(_d(b['prob']), labd, scale)
        return [('dlogits', a['dlogits'], r, bound)]
    r = SC.softmax_ce_fwd_ref(_d(b['logits']), labd, scale)
    return [('prob', a['prob'], *r['prob']), ('loss', a['loss'].reshape(-1)[:1], *r['loss'])]


@ref('sgd_nesterov')
def _sgd(c):
    b, a = c.b, c.a
    mu, wd = float(np.float32(b['momentum'])), float(np.float32(b['wd']))
    r = SC.sgd_ref(_d(b['p']), _d(b['g']), _d(b['m']), float(b['lr'].view(-1)[0]), mu, wd, bool(b['nesterov']))
    out = [(k, a[k], *r[k]) for k in ('p', 'g', 'm')]
    if b['p_tf32'] is not None:
        # exactly the TF32 rounding of the stored p
        out.append(('p_tf32', a['p_tf32'], tf32_round(a['p']), None))
    return out


@ref('spatial_bn_fwd', 'spatial_bn_fwd_det', 'spatial_bn_infer')
def _bn_fwd(c):
    b, a = c.b, c.a
    C_ = b['x'].shape[-1]
    xd = _d(b['x']).reshape(-1, C_)
    eps = float(np.float32(b['eps']))
    if c.fn == 'spatial_bn_infer':
        r, bound = SC.bn_infer_ref(xd, _d(b['s']), _d(b['b']), _d(b['rm']), _d(b['rv']), eps)
        return [('y', a['y'], r.view(a['y'].shape), bound.view(a['y'].shape))]
    # bn_chain counts the default kernel's fp32 chains; the fixed-order kernel is held to any order of the rows
    n = SC.bn_chain(xd.shape[0], C_) if c.fn == 'spatial_bn_fwd' else xd.shape[0]
    run = (_d(b['rm']), _d(b['rv']), float(np.float32(b['momentum']))) if b['rm'] is not None else ()
    r = SC.bn_fwd_ref(xd, _d(b['s']), _d(b['b']), n, eps, *run)
    y, yb = r['y']
    return [('y', a['y'], y.view(a['y'].shape), yb.view(a['y'].shape))] + [(k, a[k], *r[k]) for k in r if k != 'y']


@ref('spatial_bn_bwd', 'spatial_bn_bwd_det')
def _bn_bwd(c):
    b, a = c.b, c.a
    C_ = b['x'].shape[-1]
    xd, dyd = _d(b['x']).reshape(-1, C_), _d(b['dy']).reshape(-1, C_)
    n = SC.bn_chain(xd.shape[0], C_) if c.fn == 'spatial_bn_bwd' else xd.shape[0]
    r = SC.bn_bwd_refb(dyd, xd, _d(b['s']), _d(b['sm']), _d(b['siv']), n, _d(b['ds']), _d(b['db']))
    dx, dxb = r['dx']
    return [('dx', a['dx'], dx.view(a['dx'].shape), dxb.view(a['dx'].shape))] + \
        [(k, a[k], *r[k]) for k in ('ds', 'db') if k in r]


@ref('fbo_bank_scan')
def _bank_scan(c):
    b, a = c.b, c.a
    R, L, D = b['bank'].shape
    bf16 = b['bank'].dtype == torch.bfloat16
    live = _live_count(b, R)
    S = SC.scan_splits(live, L, D, bf16) if c.engine != 'fake' else 1
    r = SC.bank_scan_ref(_d(b['bank']), _d(b['q']), float(b['scale']), S, bf16, bool(b['tf32_out']))
    out = []
    for k in ('out', 'prob'):
        if b[k] is None:
            continue
        ref_, bound = (t.clone() for t in r[k])
        ref_[live:], bound[live:] = 0, 0                # padded rows: exact zeros
        out.append((k, a[k], ref_, bound))
    return out


@ref('cast_bf16')
def _cast_bf16(c):
    y = c.a['y']
    return [('y', y, c.b['x'].float().reshape(y.shape).to(torch.bfloat16), None)]


@ref('lfb_gather')
def _lfb_gather(c):
    b, a = c.b, c.a
    D = a['out'].shape[-1]
    rows = b['bank'].reshape(-1, D)
    i = b['idx'].reshape(-1).long()
    ok = (i >= 0) & (i < rows.shape[0])
    r = torch.where(ok.view(-1, 1), rows[i.clamp(0, rows.shape[0] - 1)], torch.zeros((), dtype=rows.dtype,
                                                                                     device=rows.device))
    if b['tf32_out']:
        r = tf32_round(r)
    return [('out', a['out'], r.view(a['out'].shape), None)]


def _fbo_weights(layers):
    return [dict((k, _d(ld[k]).requires_grad_(True)) for k in SC.FBO_W if ld.get(k) is not None) for ld in layers]


def _fbo_keeps(c, cfgd, layers, R, dA):
    ratio = float(cfgd.get('drop_ratio', 0.0) or 0.0)
    if ratio <= 0:
        return [None] * len(layers), 1.0
    if c.engine == 'fake':
        raise NoReference('FBO dropout of the CPU stand-in (not the Philox stream of csrc/fbo.cu)')
    st = int(cfgd['step'].view(-1)[0]) if cfgd.get('step') is not None else 0
    keeps = [torch.from_numpy(SC.dropout_keep(R * dA, ratio, int(cfgd.get('seed', 0)),
                                              int(ld.get('drop_offset', 0)) + (st << 32), 0)).view(R, dA).double()
             .to(layers[0]['w_theta'].device) for ld in layers]
    return keeps, float(np.float32(1.0) / (np.float32(1.0) - np.float32(ratio)))


def _fbo_forward(c, cfgd, layers, a0, bp):
    R, dA = a0.shape
    keeps, inv = _fbo_keeps(c, cfgd, layers, R, dA)
    Ws = _fbo_weights(layers)
    for W in Ws:
        for k in SC.FBO_W:
            if k not in W:
                W[k] = torch.zeros(layers[0]['w_theta'].shape[0] if k != 'b_out' else dA, dtype=torch.float64,
                                   device=a0.device)
    a64, b64 = _d(a0).requires_grad_(True), _d(bp).requires_grad_(True)
    A, outs = SC.fbo_ref(a64, b64, Ws, float(cfgd['scale']), bool(cfgd['pre_act_ln']), keeps, inv,
                         eps=float(cfgd.get('ln_eps', 1e-5)))
    return A, outs, Ws, a64, b64


def _fbo_bnd(cfgd, r, nl):
    return SC.fbo_bound(r, SC.fbo_tau(cfgd['L'], cfgd['dA'], cfgd['d'], cfgd['dB'], nl))


@ref('fbo_nl_fwd')
def _fbo_nl_fwd(c):
    b, a = c.b, c.a
    cfgd = b['cfgd']
    R = cfgd['R']
    live = _live_count(cfgd, R)
    _, outs, _, _, b64 = _fbo_forward(c, cfgd, b['layers'], b['a0'], b['bp'])
    res = []
    nl = len(b['layers'])
    for i, (ld, o) in enumerate(zip(a['layers'], outs)):
        t = o['t'].detach()
        extra = dict(s=torch.einsum('rl,rld->rd', o['prob'].detach(), b64.detach()), ln_mean=t.mean(1),
                     ln_std=(t.var(1, unbiased=False) + float(cfgd.get('ln_eps', 1e-5))).sqrt())
        for k in ('theta', 'prob', 's', 't', 'xhat', 'ln_mean', 'ln_std', 'out', 'a_out'):
            if ld.get(k) is None or (k in ('ln_mean', 'ln_std') and not cfgd['pre_act_ln']):
                continue
            r = (o[k] if k in o else extra[k]).detach()
            bound = _fbo_bnd(cfgd, r, nl)
            if live < R:
                r, bound = r.clone(), bound.clone()
                r[live:], bound[live:] = 0, 0
            res.append(('L%d.%s' % (i, k), ld[k], r.view(ld[k].shape), bound.view(ld[k].shape)))
    return res


@ref('fbo_nl_bwd')
def _fbo_nl_bwd(c):
    b, a = c.b, c.a
    cfgd = b['cfgd']
    R = cfgd['R']
    live = _live_count(cfgd, R)
    A, outs, Ws, a64, b64 = _fbo_forward(c, cfgd, b['layers'], b['a0'], b['bp'])
    dl = _d(b['da_last']).clone()
    dl[live:] = 0
    (A * dl).sum().backward()
    nl = len(b['layers'])
    res = []
    for i, (ldb, lda) in enumerate(zip(b['layers'], a['layers'])):
        for k in SC.FBO_W:
            if lda.get('g' + k) is None or ldb.get(k) is None:
                continue
            grad = Ws[i][k].grad.detach()
            bound = _fbo_bnd(cfgd, grad, nl)
            if k == 'b_phi':
                bound = SC.fbo_b_phi_bound(outs[i]['theta'], outs[i]['aff'].grad,
                                           SC.fbo_tau(cfgd['L'], cfgd['dA'], cfgd['d'], cfgd['dB'], nl))
            prev = _d(ldb['g' + k])
            res.append(('L%d.g%s' % (i, k), lda['g' + k], grad + prev, bound + 2 * U * prev.abs()))
    da0, dbp = a64.grad.detach(), b64.grad.detach()
    res.append(('da0', a['da0'], da0, _fbo_bnd(cfgd, da0, nl)))
    res.append(('dbp', a['dbp'], dbp, _fbo_bnd(cfgd, dbp, nl)))
    return res


@ref('roi_align_table')
def _roi_table(c):
    raise NoReference('roi_align_table (the executor does not call it)')


# ----------------------------------------------------------------------------------------------- the interposer
def _wrapper_signature(name):
    from vlfb import kernels
    return inspect.signature(getattr(kernels, name))


class Audit:
    """Wraps a kernel module; install() routes vlfb.executor through it.  records: one dict per audited call."""

    def __init__(self, kernels, engine, net='', sink=None):
        self.K = kernels
        self.engine = engine                      # 'tcgen05', 'simt' or 'fake' (the CPU stand-in)
        self.net = net
        self.run = 0
        self.records = []
        self.sink = sink
        self.depth = 0
        self.calls = {}
        self.proxy = types.ModuleType('audited_kernels')
        for name in dir(kernels):
            if not name.startswith('__'):
                setattr(self.proxy, name, getattr(kernels, name))
        for name in AUDITED:
            f = getattr(kernels, name, None)
            if f is not None:
                setattr(self.proxy, name, self._wrap(name, f))

    # -- installation
    def install(self):
        from vlfb import executor
        self._saved = executor.K
        executor.K = self.proxy
        return self

    def uninstall(self):
        from vlfb import executor
        executor.K = self._saved

    # -- one call
    def _wrap(self, name, f):
        sig = inspect.signature(f)

        def call(*args, **kwargs):
            if self.depth > 0:
                return f(*args, **kwargs)
            self.depth += 1
            try:
                return self._audited(name, f, sig, args, kwargs)
            finally:
                self.depth -= 1
        call.__name__ = name
        return call

    def _audited(self, name, f, sig, args, kwargs):
        bound = sig.bind(*args, **kwargs)
        bound.apply_defaults()
        a = dict(bound.arguments)
        for p in sig.parameters.values():          # a stand-in's **kwargs: flattened, the wrapper's defaults filled in
            if p.kind == p.VAR_KEYWORD:
                a.update(a.pop(p.name, {}))
        for k, p in _wrapper_signature(name).parameters.items():
            if k not in a and p.default is not p.empty:
                a[k] = p.default
        rec = dict(net=self.net, run=self.run, label=getattr(self.proxy, 'LABEL', ''), wrapper=name,
                   signature=SC.signature(name, f, args, kwargs)['args'], layout=layout(a), errors=[], outputs={})
        self.calls[name] = self.calls.get(name, 0) + 1
        before = dict((k, _clone(v)) for k, v in a.items())
        snaps = self._snapshots(name, a)
        text = ''
        if name in GEMM_WRAPPERS and os.environ.get('VLFB_DEBUG') and not self.engine.startswith('fake'):
            ret, text = capture_fd2(lambda: self._run(f, args, kwargs))
            rec['paths'] = [dict((k, list(v) if isinstance(v, tuple) else v) for k, v in r.items())
                            for r in (parse_record(l) for l in text.splitlines()) if r is not None]
            rec['paths'] += [dict(r, path='gconv') for r in (parse_record(l, 'gconv') for l in text.splitlines())
                             if r is not None]
        else:
            ret = self._run(f, args, kwargs)
        try:
            self._check(name, rec, before, a, ret, snaps)
        except NoReference as e:
            rec['errors'].append('no reference: %s' % e)
        rec['worst'] = max([o['worst'] for o in rec['outputs'].values()] or [0.0])
        rec['ok'] = not rec['errors']
        self.records.append(rec)
        if self.sink is not None:
            self.sink.write(json.dumps(rec) + '\n')
        return ret

    def _run(self, f, args, kwargs):
        ret = f(*args, **kwargs)
        if not self.engine.startswith('fake'):
            torch.cuda.synchronize()
        return ret

    def _snapshots(self, name, a):
        """(path, storage, lo, hi, bits before) of every written argument: its span plus MARGIN elements each side."""
        snaps = []
        for k, v in a.items():
            for path, t in _tensors(v, k):
                if _role(name, path, a) == 'in' or t.numel() == 0:
                    continue
                st = _storage(t)
                span = t.storage_offset() + sum((s - 1) * abs(d) for s, d in zip(t.shape, t.stride()))
                lo, hi = max(0, t.storage_offset() - MARGIN), min(st.numel(), span + 1 + MARGIN)
                if name == 'copy2d':                   # the written rows start dst_off past the view
                    hi = min(st.numel(), hi + int(a['dst_off']) + int(a['rows']) * int(a['ldd']))
                snaps.append((path, st, lo, hi, _bits(st[lo:hi]).clone()))
        return snaps

    def _check(self, name, rec, b, a, ret, snaps):
        if name not in REF:
            raise NoReference(name)
        # 5. finite inputs
        for k, v in b.items():
            for path, t in _tensors(v, k):
                if _role(name, path, b) == 'out' or not t.dtype.is_floating_point or t.numel() == 0:
                    continue
                if (name, path) in NONFINITE_EXCEPTIONS:
                    continue
                n = int((~torch.isfinite(t)).sum())
                if n:
                    rec['errors'].append('%s: input %s has %d non-finite elements' % (self._where(rec), path, n))
        # 6. TF32-exact GEMM operands
        if name in GEMM_OPERANDS and self.engine in ('tcgen05', 'fake_tf32'):
            for op in GEMM_OPERANDS[name]:
                if (name, op) in EXACTNESS_EXCEPTIONS:
                    continue
                n = not_tf32_exact(b[op])
                if n:
                    rec['errors'].append('%s: operand %s not TF32-exact in %d of %d elements' % (
                        self._where(rec), op, n, b[op].numel()))
        # 3. values
        c = types.SimpleNamespace(fn=name, b=b, a=a, ret=ret, engine='fake' if self.engine.startswith('fake') else
                                  self.engine)
        results = REF[name](c)
        written = {}
        for oname, got, r, bnd in results:
            if bnd is None and got.dtype.is_floating_point:          # -0.0 and +0.0 are the same value
                r = r.reshape(got.shape)
                r = torch.where((got == 0) & (r == 0), got.to(r.dtype), r)
            cmp = compare(got, r, bnd)
            rec['outputs'][oname] = dict(worst=cmp['worst_ratio'], exact=bnd is None)
            if not cmp['ok']:
                at = int(np.ravel_multi_index(cmp['worst_at'], r.shape)) if cmp['worst_at'] else -1
                g, rr = got.reshape(-1)[at] if at >= 0 else None, r.reshape(-1)[at] if at >= 0 else None
                rec['errors'].append('%s: %s: %d elements outside the bound (%d not finite), worst %.3g x bound at flat '
                                     '%d (got %r, ref %r)' % (self._where(rec), oname, cmp['nbad'], cmp['nonfinite'],
                                                             cmp['worst_ratio'], at, None if g is None else float(g),
                                                             None if rr is None else float(rr)))
            key = (got.untyped_storage().data_ptr(), got.dtype)
            written.setdefault(key, []).append(_offsets(got).reshape(-1))
        # 4. nothing else in the outputs' storage changed
        for path, st, lo, hi, old in snaps:
            new = _bits(st[lo:hi])
            changed = new != old
            for off in written.get((st.untyped_storage().data_ptr(), st.dtype), []):
                sel = off[(off >= lo) & (off < hi)] - lo
                changed[sel] = False
            n = int(changed.sum())
            if n:
                first = int(changed.nonzero()[0]) + lo
                rec['errors'].append('%s: %d elements of %s\'s storage outside the written set changed (first at '
                                     'storage offset %d)' % (self._where(rec), n, path, first))

    def _where(self, rec):
        return '%s run %d step %r %s' % (self.net, rec['run'], rec['label'], rec['wrapper'])

    # -- summaries
    def failures(self):
        return [r for r in self.records if not r['ok']]

    def summary(self):
        """wrapper -> (calls audited, worst |err| / bound)."""
        out = {}
        for r in self.records:
            n, w = out.get(r['wrapper'], (0, 0.0))
            out[r['wrapper']] = (n + 1, max(w, r['worst']))
        return out


def report(audit):
    lines = ['%-24s %6s  %s' % ('wrapper', 'calls', 'worst |err|/bound')]
    for k, (n, w) in sorted(audit.summary().items()):
        lines.append('%-24s %6d  %.3g' % (k, n, w))
    return '\n'.join(lines)


# ----------------------------------------------------------------------------------------------- audited nets
TINY = ['NUM_GPUS', 1, 'TRAIN.BATCH_SIZE', 2, 'TRAIN.CROP_SIZE', 64, 'TRAIN.VIDEO_LENGTH', 8,
        'TEST.BATCH_SIZE', 2, 'TEST.CROP_SIZE', 64, 'TEST.VIDEO_LENGTH', 8, 'LFB.WINDOW_SIZE', 4,
        'TRAIN.DROPOUT_RATE', 0.0, 'FBO_NL.INPUT_DROPOUT_ON', False, 'FBO_NL.LFB_DROPOUT_ON', False]
RESNEXT = ['RESNETS.NUM_GROUPS', 32, 'RESNETS.WIDTH_PER_GROUP', 4, 'MODEL.USE_AFFINE', False, 'NONLOCAL.USE_AFFINE', False,
           'NONLOCAL.USE_BN', True, 'MODEL.DILATIONS_AFTER_CONV5', False]
DROPOUT = TINY[:-6] + ['TRAIN.DROPOUT_RATE', 0.3, 'FBO_NL.INPUT_DROPOUT_ON', True, 'FBO_NL.LFB_DROPOUT_ON', True]

# The wrappers every audited train step of the tiny AVA FBO-NL net must reach.
AVA_TRAIN_WRAPPERS = {'conv_fwd', 'conv_dgrad', 'conv_wgrad', 'matmul', 'axpby', 'fill', 'round_tf32', 'copy2d',
                      'maxpool_fwd', 'roi_align_fwd', 'roi_align_bwd', 'softmax_fwd', 'softmax_bwd', 'sigmoid_ce_fwd',
                      'sigmoid_ce_bwd', 'fbo_nl_fwd', 'fbo_nl_bwd', 'sgd_nesterov', 'weight_transpose_multi'}

# name -> (yaml, overrides, split, runs, wrappers the net must reach, extra settings)
NETS = {
    'ava_train': ('ava_r50_lfb_nl.yaml', TINY, 'train', 2, AVA_TRAIN_WRAPPERS, {}),
    'ava_train_simt': ('ava_r50_lfb_nl.yaml', TINY, 'train', 2, AVA_TRAIN_WRAPPERS, {'backend': 'simt'}),
    'ava_train_dropout': ('ava_r50_lfb_nl.yaml', DROPOUT, 'train', 2, AVA_TRAIN_WRAPPERS | {'dropout'}, {}),
    'charades_train': ('charades_r50_lfb_nl.yaml', TINY + ['MODEL.NUM_CLASSES', 157], 'train', 2,
                       {'conv_fwd', 'conv_dgrad', 'conv_wgrad', 'matmul', 'sigmoid_ce_fwd', 'sigmoid_ce_bwd',
                        'sgd_nesterov'}, {}),
    'charades_softmax_train': ('charades_r50_lfb_nl.yaml', TINY + ['MODEL.NUM_CLASSES', 157, 'MODEL.MULTI_LABEL', False],
                               'train', 2, {'conv_fwd', 'conv_dgrad', 'conv_wgrad', 'matmul', 'softmax_ce_fwd',
                                            'softmax_ce_bwd', 'sgd_nesterov'}, {}),
    'ava_val_fold_f32': ('ava_r50_lfb_nl.yaml', TINY + ['B200.LFB_DTYPE', 'f32'], 'val', 1,
                         {'conv_fwd', 'fbo_bank_scan', 'roi_align_fwd'}, {}),
    'ava_val_fold_bf16': ('ava_r50_lfb_nl.yaml', TINY + ['B200.LFB_DTYPE', 'bf16'], 'val', 1,
                          {'conv_fwd', 'fbo_bank_scan', 'roi_align_fwd', 'cast_bf16'}, {}),
    'ava_lfb_infer_only': ('ava_r50_lfb_nl.yaml', TINY, 'lfb_infer_only', 1, {'conv_fwd', 'roi_align_fwd'}, {}),
    'ava_train_det': ('ava_r50_lfb_nl.yaml', TINY + ['B200.DETERMINISTIC', True], 'train', 2,
                      {'conv_fwd', 'conv_dgrad', 'conv_wgrad_det', 'matmul_det', 'roi_align_bwd_det', 'sgd_nesterov'},
                      {}),
    'ava_train_capacity': ('ava_r50_lfb_nl.yaml', TINY + ['B200.ROI_CAPACITY', 8], 'train', 2,
                           AVA_TRAIN_WRAPPERS, {}),
    # ResNeXt 32x4d with trainable SpatialBN: grouped convolutions (csrc/gconv.cu) and the BN kernels
    'resnext_bn_train': ('ava_r50_lfb_nl.yaml', TINY + RESNEXT, 'train', 2,
                         {'conv_fwd', 'conv_dgrad', 'conv_wgrad', 'spatial_bn_fwd', 'spatial_bn_bwd', 'sgd_nesterov'},
                         {'grouped': True}),
    'resnext_bn_train_det': ('ava_r50_lfb_nl.yaml', TINY + RESNEXT + ['B200.DETERMINISTIC', True], 'train', 2,
                             {'conv_fwd', 'conv_dgrad', 'conv_wgrad_det', 'spatial_bn_fwd_det', 'spatial_bn_bwd_det',
                              'colsum_det', 'sgd_nesterov'}, {'grouped': True}),
    # the benchmarked step (BASELINE config 2): 2 clips of 32 x 224^2, R = 4 RoIs, L = 300 bank rows, the yaml's dropout.
    # One unaudited warm-up run, then one audited run of every call (about half a minute on an H100).
    'config2_train': ('ava_r50_lfb_nl.yaml', ['NUM_GPUS', 1, 'TRAIN.BATCH_SIZE', 2, 'TEST.BATCH_SIZE', 2], 'train', 1,
                      AVA_TRAIN_WRAPPERS, {'crop': 224, 'frames': 32, 'warmup': 1}),
}


def run_net(audit, name, runs=None, rois_per_clip=2, seed=2):
    """Builds net `name` of NETS, feeds the oracle's parameters and inputs, and runs its audited steps eagerly (the
    optimizer update included); `runs` overrides the net's count.  Run 2 of a train net takes the paths that need a
    first run: the grad-finish fusion, sole() rounding and the lazy gradient sums.  A net with a warm-up runs it
    unaudited first."""
    import contextlib
    import harness as H
    import resnext_oracle as RO
    from vlfb import workspace
    from core.config import config as cfg
    yaml_name, overrides, split, n_runs, must, extra = NETS[name]
    runs = n_runs if runs is None else runs
    H.setup_cfg(yaml_name, overrides)
    cfg.B200.CUDA_GRAPH = False
    ocfg = H.oracle_cfg(yaml_name, overrides)
    infer_only = split == 'lfb_infer_only'
    sp = 'val' if infer_only else split
    with (RO.grouped() if extra.get('grouped') else contextlib.nullcontext()) as OMg:
        if OMg is None:
            from oracle import model as OMg
        params = OMg.make_params(ocfg, seed=seed, split=sp, lfb_infer_only=infer_only) if split != 'train' else \
            OMg.make_params(ocfg, seed=seed)
        inputs = OMg.make_inputs(ocfg, n_clips=2, rois_per_clip=rois_per_clip, crop=extra.get('crop', 64),
                                 frames=extra.get('frames', 8))
    model, sfx = H.build(sp, split == 'train', lfb_infer_only=infer_only)
    audit.net = name
    audit.install()
    audit.proxy.LABEL = 'feed'            # run 0: the parameters and inputs fed before the first step
    try:
        H.feed_params(dict((k, v) for k, v in params.items() if split == 'train' or workspace.HasBlob(k)))
        H.feed_inputs(inputs, sfx)
        if split == 'train':
            model.UpdateWorkspaceLr(10)
        for _ in range(extra.get('warmup', 0)):
            audit.uninstall()
            workspace.RunNet(model.net.Proto().name)
            audit.install()
        for r in range(runs):
            print('[launch_audit] net=%s run=%d' % (name, r + 1), flush=True)
            audit.run = r + 1
            workspace.RunNet(model.net.Proto().name)
    finally:
        audit.uninstall()
    missing = sorted(set(must) - set(audit.calls))
    return missing


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--net', required=True, choices=sorted(NETS))
    ap.add_argument('--out', required=True)
    args = ap.parse_args(argv)
    from vlfb import kernels, workspace
    backend = NETS[args.net][5].get('backend', 'tcgen05')
    kernels.set_gemm_backend(backend)
    workspace.ResetWorkspace()
    t0 = time.time()
    with open(args.out, 'w') as sink:
        audit = Audit(kernels, backend, sink=sink)
        missing = run_net(audit, args.net)
        sink.write(json.dumps(dict(summary=dict((k, list(v)) for k, v in audit.summary().items()), missing=missing,
                                   seconds=time.time() - t0)) + '\n')
    kernels.set_gemm_backend('tcgen05')
    print(report(audit))
    return 0


if __name__ == '__main__':
    sys.exit(main())
