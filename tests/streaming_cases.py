"""Case table of the streaming kernels (csrc/ops.cu, csrc/bn.cu, csrc/fbo.cu): the non-GEMM entry points of vlfb.h.

Each case is ONE seeded call of a vlfb.kernels wrapper, described by the wrapper's launch signature (`signature`: the
shapes, geometry and flags of its arguments) plus content options.  `prepare` builds its inputs, places every output
inside a NaN-filled buffer with a guard band (a lead-in, a tail, and the row / pixel / channel gaps of strided and
padded layouts) and computes an fp64 reference with an elementwise bound; `check_case` runs the call and checks
  - every in-range element: finite and |got - ref| <= bound, or bit-exact where the operation is exact;
  - the global max|got - ref| / max|ref| of the older suite;
  - every guard element: still the NaN fill, bit for bit (outputs a call reads first -- accumulate flags, the
    scatter backwards -- start from finite seeded contents that the reference adds to);
  - determinism between two runs where the ABI promises it (no atomics).
tests/test_gpu_streaming.py runs the table; tests/test_streaming_cpu.py checks the table, the references and the bounds
without a GPU.

Tolerances.  u = 2^-24 (fp32 unit roundoff).  A sum or dot product of n terms computed in fp32 in any order is within
(n - 1) u sum|terms| of the exact value (each partial sum is rounded once, and every partial sum is bounded by
sum|terms|); the bound used is C_SUM (n + k) u sum|terms| with C_SUM = 2 and k the few extra roundings of the family
(a scale, a division, a store), stated where the bound is built.  sum|terms| is computed in fp64 from the operands.
__expf(a) = ex2.approx(a log2(e)): the argument rounding gives a relative error of |a| u and ex2.approx itself
2^-22.5, hence the C_EXP 2^-22 + C_ARG |a| u terms of every exp-based bound.  Derivations per family are at its builder.
"""
import inspect
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (os.path.join(ROOT, 'video-long-term-feature-banks_b200', 'lib'), HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from util import BITS, compare, guard_touched, nan_buffer, pack_sign_bits, tf32_round, ulp_tf32  # noqa: E402,F401

# ----------------------------------------------------------------------------------------------- launch signatures
# The wrappers of vlfb.kernels that launch a streaming kernel (the GEMM wrappers conv_fwd / conv_dgrad / conv_wgrad /
# matmul are tests/gemm_paths.py's).
STREAMING_WRAPPERS = (
    'affine_fwd', 'affine_bwd', 'spatial_bn_fwd', 'spatial_bn_infer', 'spatial_bn_bwd', 'maxpool_fwd', 'maxpool_bwd',
    'maxpool_bwd_gather', 'avgpool_fwd', 'avgpool_bwd', 'roi_align_fwd', 'roi_align_bwd', 'roi_align_table',
    'softmax_fwd', 'softmax_bwd', 'layernorm_fwd', 'layernorm_bwd', 'relu_fwd', 'relu_bwd', 'axpby', 'fill',
    'round_tf32', 'add_tf32', 'relu_tf32', 'add_relu_bwd_tf32', 'relu_bits', 'relu_bwd_tf32', 'colsum', 'sigmoid_fwd',
    'dropout', 'copy2d', 'nc_to_cl', 'cl_to_nc', 'weight_transpose', 'weight_transpose_multi', 'sigmoid_ce_fwd',
    'sigmoid_ce_bwd', 'softmax_ce_fwd', 'softmax_ce_bwd', 'sgd_nesterov', 'fbo_nl_fwd', 'fbo_nl_bwd', 'fbo_bank_scan',
    'cast_bf16', 'lfb_gather')

# Arguments that are not part of a signature: generator seeds / counter offsets and the host-side cache of
# weight_transpose_multi.  Other float arguments (scales, eps, learning rates) are values, not geometry, and are dropped
# too; drop_ratio only counts as "dropout on or off".
_DROP = object()
_SKIP_NAMES = ('seed', 'offset', 'drop_offset', 'cache')
GEOM_FIELDS = ('N', 'T', 'H', 'W', 'C', 'To', 'Ho', 'Wo', 'Co', 'kT', 'kH', 'kW', 'sT', 'sH', 'sW', 'pT', 'pH', 'pW',
               'dT', 'dH', 'dW')


def _sig_value(name, v):
    if name in _SKIP_NAMES:
        return _DROP
    if name == 'drop_ratio':
        return bool(v and float(v) > 0)
    if v is None:
        return None
    if torch.is_tensor(v):
        return dict(shape=list(v.shape), dtype=str(v.dtype).replace('torch.', ''))
    if isinstance(v, bool):
        return v
    if isinstance(v, (int, np.integer)):
        return int(v)
    if isinstance(v, float):
        return _DROP
    if all(hasattr(v, f) for f in GEOM_FIELDS):
        return dict((f, int(getattr(v, f))) for f in GEOM_FIELDS)
    if isinstance(v, dict):
        out = {}
        for k in sorted(v):
            s = _sig_value(k, v[k])
            if s is not _DROP:
                out[k] = s
        return out
    if isinstance(v, (list, tuple)):
        return [_sig_value('', x) for x in v]
    raise TypeError('no signature for argument %s of type %s' % (name, type(v).__name__))


def signature(fn, func, args, kwargs):
    """{'fn': wrapper name, 'args': {parameter: shape / geometry / flag}} of one call of a vlfb.kernels wrapper."""
    b = inspect.signature(func).bind(*args, **kwargs)
    b.apply_defaults()
    out = {}
    for k, v in b.arguments.items():
        s = _sig_value(k, v)
        if s is not _DROP:
            out[k] = s
    return dict(fn=fn, args=out)


# ----------------------------------------------------------------------------------------------- constants / helpers
U = 2.0 ** -24
C_SUM = 2.0
C_EXP = 2.0
C_ARG = 2.0
GUARD = 64                     # lead-in guard elements (keeps an unshifted output 16-byte aligned)
TAIL = 64
# stream_grid (common.cuh) caps a grid at 132 * 16 blocks: above CAP_ITEMS work items of 256-thread blocks (one item per
# thread) the grid-stride loops run more than once; the 4-per-thread kernels need 4 x that.
CAP_ITEMS = 132 * 16 * 256


def T(*shape, dtype='float32'):
    return dict(shape=[int(s) for s in shape], dtype=dtype)


def geom(N, T_, H, W, C, ker, st, pd):
    To = (T_ + 2 * pd[0] - ker[0]) // st[0] + 1
    Ho = (H + 2 * pd[1] - ker[1]) // st[1] + 1
    Wo = (W + 2 * pd[2] - ker[2]) // st[2] + 1
    return dict(N=N, T=T_, H=H, W=W, C=C, To=To, Ho=Ho, Wo=Wo, Co=C, kT=ker[0], kH=ker[1], kW=ker[2], sT=st[0],
                sH=st[1], sW=st[2], pT=pd[0], pH=pd[1], pW=pd[2], dT=1, dH=1, dW=1)


def bf16_rne(t):
    """fp32 -> bf16 bits (round to nearest even) as int32, the rule of vlfb_cast_f32_to_bf16."""
    i = t.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    return ((i + 0x7FFF + ((i >> 16) & 1)) >> 16).to(torch.int32)


# ----------------------------------------------------------------------------------------------- Philox4x32-10 (numpy)
PHILOX_M = (0xD2511F53, 0xCD9E8D57)
PHILOX_W = (0x9E3779B9, 0xBB67AE85)


def philox4x32_10(ctr, key):
    """Random123 Philox4x32-10 of 64-bit counters `ctr` (words 2, 3 = 0) under the 64-bit key `key`: uint32 [n, 4]."""
    ctr = np.asarray(ctr, dtype=np.uint64).reshape(-1)
    m32 = np.uint64(0xFFFFFFFF)
    c0, c1 = ctr & m32, ctr >> np.uint64(32)
    c2 = np.zeros_like(c0)
    c3 = np.zeros_like(c0)
    k0, k1 = np.uint64(int(key) & 0xFFFFFFFF), np.uint64((int(key) >> 32) & 0xFFFFFFFF)
    for _ in range(10):
        p0 = c0 * np.uint64(PHILOX_M[0])            # < 2^64: exact in uint64
        p1 = c2 * np.uint64(PHILOX_M[1])
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & m32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & m32
        k0 = (k0 + np.uint64(PHILOX_W[0])) & m32
        k1 = (k1 + np.uint64(PHILOX_W[1])) & m32
    return np.stack([c0, c1, c2, c3], 1).astype(np.uint32)


def dropout_keep(n, ratio, seed, offset, step=0):
    """The keep mask of vlfb_dropout_fwd: element j uses word j & 3 of block offset + (j >> 2) + (step << 32) under key
    `seed`; u = (word >> 8) 2^-24 and the element is kept iff u >= ratio (fp32 comparison)."""
    nb = (n + 3) // 4
    ctr = (np.uint64(offset) + np.arange(nb, dtype=np.uint64) + (np.uint64(step) << np.uint64(32)))
    r = philox4x32_10(ctr, seed).reshape(-1)[:n]
    u = (r >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    return u >= np.float32(ratio)


# ----------------------------------------------------------------------------------------------- placement
class Prepared:
    """Inputs, output placements, the call and the fp64 references of one case."""

    def __init__(self, case, dev):
        self.case, self.dev = case, dev
        self.outs = []             # dict(name, buf, index, ref, bound (None = bit-exact), tol)
        self.call = None           # call(K): the one wrapper call
        self.det = False
        self.keep = []


# The global check of the older suite, max|got - ref| / max|ref| < tol, kept beside the elementwise bound: TOL unless a
# case states its own (the TF32-rounded outputs: one TF32 ulp, 6e-4).
TOL = 1e-4


def place(P, name, shape, ref, bound=None, dtype=torch.float32, off=0, prev=None, tol=None):
    """A contiguous output of `shape` at GUARD + off of a NaN buffer; `prev` = its finite starting contents."""
    n = int(np.prod(shape)) if len(shape) else 1
    buf = nan_buffer(GUARD + n + off + TAIL, P.dev, dtype)
    index = torch.arange(n, device=P.dev).view(shape) + GUARD + off
    if prev is not None:
        buf[index.reshape(-1)] = prev.reshape(-1).to(dtype)
    P.outs.append(dict(name=name, buf=buf, index=index, ref=ref, bound=bound, tol=TOL if tol is None else tol))
    return buf[GUARD + off:GUARD + off + n].view(shape)


def add_out(P, name, buf, index, ref, bound=None, tol=None):
    P.outs.append(dict(name=name, buf=buf, index=index, ref=ref, bound=bound, tol=TOL if tol is None else tol))


def inp(P, t, off=0):
    """The fp32 / int tensor t on the device, `off` elements past a 16-byte boundary (off > 0: the scalar paths)."""
    t = t.contiguous()
    b = torch.zeros(t.numel() + off + 4, dtype=t.dtype, device=P.dev)     # never a NULL pointer, even when empty
    b[off:off + t.numel()] = t.reshape(-1).to(P.dev)
    d = b[off:off + t.numel()].view(t.shape)
    P.keep.append(d)
    return d


def randn(shape, gen, scale=1.0):
    return torch.randn(tuple(shape), generator=gen) * scale


def content(shape, gen, kind):
    """fp32 test content: 'randn'; 'int' (small integers: ties in every window); 'ties' (TF32 rounding ties: low 13 bits
    0x1000, both signs, incl. mantissas whose rounding carries into the next binade) mixed with random values."""
    shape = tuple(shape)
    if kind == 'int':
        return torch.randint(-4, 5, shape, generator=gen).float()
    x = torch.randn(shape, generator=gen)
    if kind == 'ties':
        n = x.numel()
        i = x.view(-1).view(torch.int32).clone()
        sel = torch.arange(n) % 3 != 2
        i[sel] = (i[sel] & ~0x1FFF) | 0x1000
        car = torch.arange(n) % 7 == 0               # mantissa 1.1111111111 1 -> carry into the next binade
        i[car] = (i[car] & ~0x7FFFFF) | 0x7FF000
        x = i.view(torch.float32).view(shape)
    return x


def sum_bound(n, mag, k=2):
    return C_SUM * (n + k) * U * mag


def exact_f64(t):
    return t.double()


# ----------------------------------------------------------------------------------------------- references
# Each family's fp64 reference and elementwise bound as a function of the call's inputs (fp64 tensors on any device):
# the builders below call them on seeded inputs, tests/launch_audit.py on the tensors of a real step.  The derivation of
# every bound is at the family's builder.
def axpby_ref(x, a, y, b):
    ref = a * x + b * y
    return ref, sum_bound(0, (a * x).abs() + (b * y).abs())


def sigmoid_ref(x):
    ref = torch.sigmoid(x)
    return ref, ref * (1 - ref) * (C_EXP * 2.0 ** -22 + C_ARG * x.abs() * U) + 3 * U * ref


def softmax_fwd_ref(x, scale, tf32_out):
    cols = x.shape[-1]
    sx = scale * x
    z = sx - sx.max(-1, keepdim=True).values
    ref = torch.softmax(z, -1)
    e = C_ARG * (z.abs() + sx.abs()) * U
    zbar = (ref * e).sum(-1, keepdim=True)
    bound = ref * (C_SUM * (cols + 4) * U + C_EXP * 2.0 ** -22 + e + zbar)
    if tf32_out:
        bound = bound + ulp_tf32(ref)
    return ref, bound


def softmax_bwd_refb(p, dp, scale, tf32_out):
    cols = p.shape[-1]
    ref = softmax_bwd_ref(p, dp, scale)
    bound = sum_bound(cols, scale * p * (dp.abs() + (p * dp).abs().sum(-1, keepdim=True)), k=4)
    if tf32_out:
        bound = bound + ulp_tf32(ref)
    return ref, bound


def layernorm_fwd_ref(x, eps):
    """x [rows, cols] -> (y, y bound, mean, mean bound, std, std bound), the statistics as [rows, 1]."""
    cols = x.shape[1]
    mu = x.mean(1, keepdim=True)
    dv = x - mu
    var = (dv * dv).mean(1, keepdim=True)
    sd = (var + eps).sqrt()
    ref = dv / sd
    n = -(-cols // 32) + 5
    dmu = sum_bound(n, x.abs().mean(1, keepdim=True)) + U * mu.abs()
    dvar = sum_bound(n, var) + 2 * dmu * dv.abs().mean(1, keepdim=True) + dmu ** 2
    dsd = sd * (0.5 * dvar / (var + eps) + 2 * U)
    bound = (dmu + U * dv.abs()) / sd + ref.abs() * (dsd / sd + 2 * U)
    return ref, bound, mu, dmu, sd, dsd


def layernorm_bwd_refb(dy, y, sd):
    cols = dy.shape[1]
    ref = layernorm_bwd_ref(dy, y, sd)
    mag = (dy.abs() + dy.abs().mean(1, keepdim=True) + y.abs() * (dy * y).abs().mean(1, keepdim=True)) / sd
    return ref, sum_bound(cols, mag, k=6)


def colsum_ref(xs, prev, n):
    """xs [rows, cols] fp64, prev [cols] or None (accumulate), n = terms of one fp32 chain."""
    ref, mag = xs.sum(0), xs.abs().sum(0)
    if prev is not None:
        ref, mag = ref + prev, mag + prev.abs()
    return ref, sum_bound(n, mag)


def maxpool_bwd_refb(g, arg, dy, keep=None, prev=None, tf32_out=False):
    """scatter form: prev = the finite contents dx starts from; gather form: keep = y > 0 (or None)."""
    nk = g['kT'] * g['kH'] * g['kW']
    ref, mag = _scatter_windows(g, arg, dy, keep)
    if prev is not None:
        ref, mag = ref + prev, mag + prev.abs()
    bound = sum_bound(nk, mag)
    if tf32_out:
        bound = bound + ulp_tf32(ref)
    return ref, bound


def avgpool_fwd_ref(x, g):
    import torch.nn.functional as F
    nk = g['kT'] * g['kH'] * g['kW']
    pool = lambda t: F.avg_pool3d(_nc(t, g), (g['kT'], g['kH'], g['kW']), (g['sT'], g['sH'], g['sW'])).permute(0, 2, 3, 4, 1)
    return pool(x), sum_bound(nk, pool(x.abs()), k=3)


def avgpool_bwd_refb(dy, g, prev=None):
    nk = g['kT'] * g['kH'] * g['kW']
    ref, mag = avgpool_bwd_ref(dy, g), avgpool_bwd_ref(dy.abs(), g)
    if prev is not None:
        ref, mag = ref + prev, mag + prev.abs()
    return ref, sum_bound(nk, mag, k=3)


def affine_ref(x, s, b):
    ref = x * s + b
    return ref, sum_bound(0, (x * s).abs() + b.abs())


def roi_align_fwd_ref(M, nmax, feat2):
    """M, nmax = roi_matrix(...); feat2 [N H W, C] fp64 -> [R PH PW, C]."""
    return M @ feat2, sum_bound(nmax, M.abs() @ feat2.abs())


def roi_align_bwd_ref(M, dout2, prev):
    """dout2 [R PH PW, C], prev [N H W, C] (the finite contents the atomics add to)."""
    ref = M.t() @ dout2 + prev
    mag = M.abs().t() @ dout2.abs() + prev.abs()
    terms = int((M != 0).sum(0).max()) + 1 if M.numel() else 1
    return ref, sum_bound(terms, mag)


def sigmoid_ce_fwd_ref(x, t, scale):
    valid = t != -1
    cnt = max(float(valid.sum()), 1e-5)
    l = torch.nn.functional.binary_cross_entropy_with_logits(x, t.clamp(min=0).double(), reduction='none')
    l = torch.where(valid, l, torch.zeros_like(l))
    ref = (scale * l.sum() / cnt).view(1)
    mag = (l.abs() + torch.where(valid, x.abs() + 2, torch.zeros_like(x)) * 2.0 ** -21).sum()
    return ref, (sum_bound(x.numel(), mag, k=3) * abs(scale) / cnt).view(1)


def sigmoid_ce_bwd_ref(x, t, scale, dl):
    valid = t != -1
    cnt = max(float(valid.sum()), 1e-5)
    k = scale * dl / cnt
    sg = torch.sigmoid(x)
    ref = torch.where(valid, k * (sg - t.double()), torch.zeros_like(x))
    bound = abs(k) * (sg * (1 - sg) * (C_EXP * 2.0 ** -22 + C_ARG * x.abs() * U) + 4 * U * (sg + t.double().abs()))
    return ref, bound


def sgd_ref(pd, gd, md, lr, mu, wd, nesterov):
    """{'p', 'g', 'm'}: (value after the step, bound)."""
    g2 = gd + wd * pd
    eg = 2 * U * (gd.abs() + wd * pd.abs())
    m2 = mu * md + lr * g2
    em = 2 * U * (mu * md.abs() + lr * g2.abs()) + lr * eg
    if nesterov:
        st = (1 + mu) * m2 - mu * md
        es = 3 * U * ((1 + mu) * m2.abs() + mu * md.abs()) + (1 + mu) * em
    else:
        st, es = m2, em
    p2 = pd - st
    ep = 2 * U * (pd.abs() + st.abs()) + es
    return dict(p=(p2, ep), g=(st, es), m=(m2, em))


def fbo_tau(L, dA, d, dB, nl):
    return C_SUM * (dA + d + dB + L + 8) * U * nl


def fbo_bound(ref, tau):
    """The FBO stack's mixed bound: tau times the element's magnitude plus its row's mean magnitude."""
    r = ref.detach()
    m = r.abs().reshape(r.shape[0], -1).mean(1).view((-1,) + (1,) * (r.dim() - 1)) if r.dim() > 1 else r.abs().mean()
    return tau * (r.abs() + m)


def fbo_b_phi_bound(theta, aff_grad, tau):
    """Bound of the phi bias gradient, theta_o sum_j dscore_j: exactly 0, up to the cancellation of the sum."""
    return tau * theta.detach().abs().t() @ (aff_grad.abs().sum(1))


def bn_infer_ref(x, s, b, rm, rv, eps):
    fs = s / (rv + eps).sqrt()
    ref = (x - rm) * fs + b
    return ref, 6 * U * ((x - rm).abs() * fs.abs() + b.abs())


def bn_fwd_ref(x, s, b, n, eps, rm=None, rv=None, mom=None):
    """x [rows, C]; n = terms of one fp32 chain.  {'y', 'sm', 'siv' (, 'rm', 'rv')}: (ref, bound)."""
    rows = x.shape[0]
    x0 = x[0]
    dev_ = x - x0
    d = dev_.mean(0)
    mean = x0 + d
    E2 = (dev_ * dev_).mean(0)
    var = (x - mean).pow(2).mean(0)
    dd = sum_bound(n, dev_.abs().mean(0))
    dmean = dd + U * mean.abs()
    dvar = sum_bound(n, E2, k=3) + 2 * d.abs() * dd + dd ** 2
    inv = 1.0 / (var + eps).sqrt()
    dinv = inv * 0.5 * dvar / (var + eps)
    fs = s * inv
    dfs = s.abs() * dinv + U * fs.abs()
    ref = (x - mean) * fs + b
    bound = fs.abs() * (dmean + U * (x - mean).abs()) + (x - mean).abs() * dfs + 2 * U * ((x - mean).abs() * fs.abs() + b.abs())
    out = dict(y=(ref, bound), sm=(mean, dmean), siv=(inv, dinv + U * inv))
    if rm is not None:
        unb = var * rows / (rows - 1) if rows > 1 else var
        dunb = dvar * rows / (rows - 1) if rows > 1 else dvar
        rm_ref, rv_ref = rm * mom + mean * (1 - mom), rv * mom + unb * (1 - mom)
        out['rm'] = (rm_ref, (1 - mom) * dd + 2 * U * (rm_ref.abs() + rm.abs()))
        out['rv'] = (rv_ref, (1 - mom) * dunb + 2 * U * (rv_ref.abs() + rv.abs()))
    return out


def bn_bwd_refb(dy, x, s, sm, siv, n, ds_prev=None, db_prev=None):
    """{'dx' (, 'ds', 'db')}: (ref, bound); ds_prev / db_prev = the accumulated gradients' contents (None: not
    computed)."""
    m = x.shape[0]
    s1, s2 = dy.sum(0), (dy * (x - sm)).sum(0)
    ds1 = sum_bound(n, dy.abs().sum(0))
    ds2 = sum_bound(n, (dy * (x - sm)).abs().sum(0), k=3)
    A, B = s * siv, -s * siv ** 3 * s2 / m
    Cc = -A * s1 / m - B * sm
    dA = U * A.abs()
    dB = s.abs() * siv ** 3 / m * ds2 + U * B.abs()
    dC = A.abs() * ds1 / m + dA * s1.abs() / m + sm.abs() * dB + U * ((A * s1 / m).abs() + (B * sm).abs()) * 2
    ref = bn_bwd_ref(dy, x, s, sm, siv)
    bound = dy.abs() * dA + x.abs() * dB + dC + 3 * U * ((A * dy).abs() + (B * x).abs() + Cc.abs())
    out = dict(dx=(ref, bound))
    if ds_prev is not None:
        out['ds'] = (ds_prev + s2 * siv, siv * ds2 + 2 * U * (ds_prev.abs() + (s2 * siv).abs()))
    if db_prev is not None:
        out['db'] = (db_prev + s1, ds1 + 2 * U * (db_prev.abs() + s1.abs()))
    return out


def softmax_ce_bwd_ref(pd, labd, scale):
    rows = pd.shape[0]
    onehot = torch.zeros_like(pd).scatter_(1, labd.view(-1, 1), 1.0)
    return (pd - onehot) * scale / rows, 3 * U * (pd + onehot) * abs(scale) / rows


def softmax_ce_fwd_ref(xd, labd, scale):
    """{'prob', 'loss'}: (ref, bound)."""
    rows, cols = xd.shape
    n = -(-cols // 256) + 10
    mx = xd.max(1, keepdim=True).values
    z = xd - mx
    ref = torch.softmax(xd, 1)
    e = C_ARG * (z.abs() + xd.abs()) * U
    rs = C_SUM * (n + 4) * U + C_EXP * 2.0 ** -22 + (ref * e).sum(1, keepdim=True)
    logs = torch.logsumexp(z, 1)
    lr = logs - z.gather(1, labd.view(-1, 1)).view(-1)
    dl = 2.0 ** -21 + 4 * U * logs.abs() + rs.view(-1) + 2 * U * (xd.gather(1, labd.view(-1, 1)).view(-1).abs() + mx.view(-1).abs())
    loss_ref = (scale * lr.sum() / rows).view(1)
    lb = abs(scale) / rows * (dl.sum() + sum_bound(rows, lr.abs().sum(), k=3))
    return dict(prob=(ref, ref * (rs + e)), loss=(loss_ref, lb.view(1)))


def bank_scan_ref(bd, qd, scale, S, bf16, tf32_out):
    """bd [R, L, D], qd [R, D] fp64, S = the split of a RoI's rows over CTAs.  {'out', 'prob'}: (ref, bound)."""
    R, L, D = bd.shape
    tiles = -(-(-(-L // S)) // scan_rows(D, bf16)) + 1
    zs = scale * torch.einsum('rd,rld->rl', qd, bd)
    p = torch.softmax(zs, 1)
    z = zs - zs.max(1, keepdim=True).values
    ds = sum_bound(D // 256 + 13, abs(scale) * torch.einsum('rd,rld->rl', qd.abs(), bd.abs()))
    rng = zs.max(1, keepdim=True).values - zs.min(1, keepdim=True).values
    rel = (ds + (p * ds).sum(1, keepdim=True) + tiles * (C_EXP * 2.0 ** -22 + 2 * U) * 2 + C_ARG * U * (z.abs() + rng) * 2
           + C_SUM * (L + S + 4) * U)
    ref = torch.einsum('rl,rld->rd', p, bd)
    pb = p.unsqueeze(2) * bd.abs()
    bound = torch.einsum('rl,rld->rd', rel, pb) + C_SUM * (L + S + 4) * U * pb.sum(1)
    if tf32_out:
        bound = bound + ulp_tf32(ref)
    return dict(out=(ref, bound), prob=(p, p * rel))


# ----------------------------------------------------------------------------------------------- builders
BUILD = {}


def builder(*names):
    def reg(f):
        for n in names:
            BUILD[n] = f
        return f
    return reg


EW_ARGS = {                     # wrapper -> (input parameters, output parameter)
    'relu_fwd': (('x',), 'y'), 'relu_bwd': (('dy', 'y'), 'dx'), 'axpby': (('x', 'y'), 'out'), 'fill': ((), 'x'),
    'round_tf32': (('x',), 'y'), 'add_tf32': (('x', 'y'), 'out'), 'relu_tf32': (('x',), 'y'),
    'add_relu_bwd_tf32': (('a', 'b', 'y'), 'out'), 'relu_bits': (('x',), 'bits'), 'relu_bwd_tf32': (('dy', 'y'), 'dx'),
    'sigmoid_fwd': (('x',), 'y')}


@builder(*EW_ARGS)
def _ew(P, gen):
    """Exact elementwise ops compare bit for bit (fp32 reference on the device).  axpby: two roundings of
    |a x| + |b y| (k = 2, n = 0).  sigmoid = 1 / (1 + __expf(-x)): the exp's relative error (C_EXP 2^-22 + C_ARG |x| u)
    moves the result by sigma (1 - sigma) times it, plus three roundings of sigma."""
    c = P.case
    fn, a = c['fn'], c['args']
    ins, outn = EW_ARGS[fn]
    off = c.get('off', 0)
    kind = c.get('content', 'randn')
    X = {}
    for nm in ins:
        if a.get(nm) is None:
            X[nm] = None
            continue
        X[nm] = content(a[nm]['shape'], gen, kind if nm in ('x', 'a', 'dy') else 'randn')
    shape = a[outn]['shape']
    f = lambda t: t.to(P.dev)
    s0, s1, v = c.get('s0', 0.75), c.get('s1', -1.5), c.get('v', 3.25)
    bound = None
    if fn == 'relu_fwd':
        ref = f(X['x']).clamp(min=0)
    elif fn == 'relu_bwd':
        ref = torch.where(f(X['y']) > 0, f(X['dy']), torch.zeros((), device=P.dev))
    elif fn == 'axpby':
        if X['y'] is None:                  # y = NULL needs b = 0
            s1 = 0.0
        yv = torch.zeros((), dtype=torch.float64, device=P.dev) if X['y'] is None else f(X['y']).double()
        ref, bound = axpby_ref(f(X['x']).double(), s0, yv, s1)
    elif fn == 'fill':
        ref = torch.full(tuple(shape), v, device=P.dev)
    elif fn == 'round_tf32':
        ref = tf32_round(f(X['x']))
    elif fn == 'add_tf32':
        ref = tf32_round(f(X['x']) + f(X['y']))
    elif fn == 'relu_tf32':
        ref = tf32_round(f(X['x']).clamp(min=0))
    elif fn == 'add_relu_bwd_tf32':
        s = tf32_round(f(X['a']) + f(X['b']))
        ref = s if X['y'] is None else torch.where(f(X['y']) > 0, s, torch.zeros((), device=P.dev))
    elif fn == 'relu_bits':
        ref = pack_sign_bits(f(X['x']))
    elif fn == 'relu_bwd_tf32':
        ref = torch.where(f(X['y']) > 0, tf32_round(f(X['dy'])), torch.zeros((), device=P.dev))
    else:
        ref, bound = sigmoid_ref(f(X['x']).double())
    alias = c.get('alias')
    if alias:                   # out is one of the inputs: its buffer is that input's
        n = int(np.prod(shape))
        buf = nan_buffer(GUARD + n + off + TAIL, P.dev)
        index = torch.arange(n, device=P.dev).view(shape) + GUARD + off
        buf[index.reshape(-1)] = X[alias].reshape(-1).to(P.dev)
        T_ = {alias: buf[GUARD + off:GUARD + off + n].view(shape)}
        add_out(P, outn, buf, index, ref, bound)
        out = T_[alias]
    else:
        T_ = {}
        out = place(P, outn, shape, ref, bound, dtype=torch.int32 if fn == 'relu_bits' else torch.float32, off=off)
    args = {}
    for nm in ins:
        args[nm] = None if X[nm] is None else T_.get(nm, inp(P, X[nm], off))
    args[outn] = out
    if fn == 'axpby':
        args.update(a=s0, b=s1)
    if fn == 'fill':
        args['v'] = v
    P.call = lambda K: getattr(K, fn)(**args)
    P.det = True


@builder('dropout')
def _dropout(P, gen):
    """Bit-exact: the keep mask of the numpy Philox reference, kept elements x * fp32(1 / (1 - ratio))."""
    c = P.case
    a = c['args']
    n = int(np.prod(a['x']['shape']))
    ratio, seed, offset, stepv = c.get('ratio', 0.25), c.get('seed_', 1234567), c.get('offset', 77), c.get('step', 0)
    x = content(a['x']['shape'], gen, 'randn')
    keep = torch.from_numpy(dropout_keep(n, ratio, seed, offset, stepv if a.get('step') is not None else 0))
    inv = np.float32(1.0) / (np.float32(1.0) - np.float32(ratio))
    ref = torch.where(keep.view(x.shape), x * float(inv), torch.zeros(())).to(P.dev)
    y = place(P, 'y', a['y']['shape'], ref, off=c.get('off', 0))
    xd = inp(P, x, c.get('off', 0))
    st = None if a.get('step') is None else inp(P, torch.tensor([stepv], dtype=torch.int64))
    P.call = lambda K: K.dropout(xd, y, ratio, seed, offset, st)
    P.det = True
    P.mask = keep


@builder('copy2d')
def _copy2d(P, gen):
    """Bit-exact without accumulate; with accumulate one rounding of |prev| + |src| (n = 1)."""
    c = P.case
    a = c['args']
    rows, cols, lds, ldd = a['rows'], a['cols'], a['lds'], a['ldd']
    so, do = a['src_off'], a['dst_off']
    src = randn(a['src']['shape'], gen)
    nd = int(np.prod(a['dst']['shape']))
    r_, c_ = torch.meshgrid(torch.arange(rows), torch.arange(cols), indexing='ij')
    sidx = so + r_ * lds + c_
    didx = GUARD + do + r_ * ldd + c_
    v = src.reshape(-1)[sidx]
    buf = nan_buffer(GUARD + nd + TAIL, P.dev)
    if a['accumulate']:
        prev = randn((rows, cols), gen)
        buf[didx.reshape(-1).to(P.dev)] = prev.reshape(-1).to(P.dev)
        ref = (prev.double() + v.double()).to(P.dev)
        add_out(P, 'dst', buf, didx.to(P.dev), ref, sum_bound(1, (prev.double().abs() + v.double().abs()).to(P.dev), k=0))
    else:
        add_out(P, 'dst', buf, didx.to(P.dev), v.to(P.dev))
    dst = buf[GUARD:GUARD + nd].view(a['dst']['shape'])
    sd = inp(P, src)
    P.call = lambda K: K.copy2d(sd, lds, dst, ldd, rows, cols, a['accumulate'], so, do)
    P.det = True


@builder('nc_to_cl', 'cl_to_nc')
def _layout(P, gen):
    """Bit-exact transposes (TF32-rounded where tf32_out); the pad channels Cpad > C are written as zeros by nc_to_cl
    and the pad pixels of the pitched form are guard."""
    c = P.case
    a = c['args']
    n, C, inner, cpad = a['n'], a['c'], a['inner'], a['cpad'] or a['c']
    if c['fn'] == 'cl_to_nc':
        src = content((n, inner, cpad), gen, c.get('content', 'randn'))
        ref = src[:, :, :C].permute(0, 2, 1).contiguous().to(P.dev)
        dst = place(P, 'dst', a['dst']['shape'], ref)
        sd = inp(P, src.view(a['src']['shape']))
        P.call = lambda K: K.cl_to_nc(sd, dst, n, C, inner, a['cpad'])
    else:
        src = content((n, C, inner), gen, c.get('content', 'randn'))
        v = torch.zeros((n, inner, cpad))
        v[:, :, :C] = src.permute(0, 2, 1)
        if a['tf32_out']:
            v = tf32_round(v)
        nd = int(np.prod(a['dst']['shape']))
        if a['pitch']:
            W, pitch, left = a['width'], a['pitch'], a['left']
            pix = torch.arange(n * inner)
            rowi, wi = pix // W, pix % W
            base = GUARD + (rowi * pitch + left + wi) * cpad
            index = (base.view(-1, 1) + torch.arange(cpad).view(1, -1)).view(n, inner, cpad)
        else:
            index = GUARD + torch.arange(n * inner * cpad).view(n, inner, cpad)
        buf = nan_buffer(GUARD + nd + TAIL, P.dev)
        add_out(P, 'dst', buf, index.to(P.dev), v.to(P.dev))
        dst = buf[GUARD:GUARD + nd].view(a['dst']['shape'])
        sd = inp(P, src.view(a['src']['shape']))
        P.call = lambda K: K.nc_to_cl(sd, dst, n, C, inner, a['cpad'], a['tf32_out'], a['width'], a['pitch'], a['left'])
    P.det = True


@builder('weight_transpose', 'weight_transpose_multi')
def _wt(P, gen):
    """Bit-exact: wt[ci][tap][co] = tf32_round(fp32(w[co][tap][ci] * scale[co]))."""
    c = P.case
    a = c['args']
    jobs = [(j[0], j[1], j[2]) for j in a['jobs']] if c['fn'] == 'weight_transpose_multi' else \
        [(a['w'], a['wt'], a['scale'])]
    dj = []
    for w_s, wt_s, s_s in jobs:
        w = randn(w_s['shape'], gen, 0.1)
        co, ci = w.shape[0], w.shape[-1]
        taps = w.numel() // (co * ci)
        w3 = w.reshape(co, taps, ci)
        s = None
        if s_s is not None:
            s = torch.rand(co, generator=gen) + 0.5
            w3 = w3 * s.view(-1, 1, 1)
        ref = tf32_round(w3.permute(2, 1, 0).contiguous()).view(wt_s['shape']).to(P.dev)
        wt = place(P, 'wt', wt_s['shape'], ref)
        dj.append((inp(P, w), wt, None if s is None else inp(P, s)))
    if c['fn'] == 'weight_transpose':
        P.call = lambda K: K.weight_transpose(*dj[0])
    else:
        P.call = lambda K: K.weight_transpose_multi(dj, {})
    P.det = True


@builder('softmax_fwd')
def _softmax_fwd(P, gen):
    """p_j = __expf(fl(scale x_j) - max) / sum.  Relative to each probability: the sum of cols terms (C_SUM (cols + 4) u,
    incl. the reciprocal and two products), the exp (C_EXP 2^-22 + C_ARG |z_j| u, z_j = scale x_j - max), the rounding of
    scale x_j (|scale x_j| u: it does not cancel against the max) and the same exp errors of the other terms carried
    by the normaliser (their p-weighted mean, zbar).  tf32_out adds one TF32 ulp."""
    c = P.case
    a = c['args']
    cols = a['x']['shape'][-1]
    scale = c.get('scale', 0.125)
    x = randn(a['x']['shape'], gen, c.get('spread', 3.0))
    ref, bound = softmax_fwd_ref(x.double().to(P.dev), scale, a['tf32_out'])
    p = place(P, 'p', a['p']['shape'], ref, bound, tol=6e-4 if a['tf32_out'] else 2e-5)
    xd = inp(P, x)
    P.call = lambda K: K.softmax_fwd(xd, p, scale, a['tf32_out'])
    P.det = True


def softmax_bwd_ref(p, dp, scale, dot=True):
    d = (p * dp).sum(-1, keepdim=True) if dot else 0.0
    return scale * p * (dp - d)


@builder('softmax_bwd')
def _softmax_bwd(P, gen):
    """dx = scale p (dp - sum p dp): a dot product of cols terms, one difference and two products:
    C_SUM (cols + 4) u scale p_j (|dp_j| + sum |p dp|).  tf32_out adds one TF32 ulp."""
    c = P.case
    a = c['args']
    cols = a['p']['shape'][-1]
    scale = c.get('scale', 0.125)
    z = randn(a['p']['shape'], gen, 3.0)
    p = torch.softmax(z, -1)
    dp = randn(a['dp']['shape'], gen)
    pd, dpd = p.double().to(P.dev), dp.double().to(P.dev)
    ref, bound = softmax_bwd_refb(pd, dpd, scale, a['tf32_out'])
    dx = place(P, 'dx', a['dx']['shape'], ref, bound, tol=6e-4 if a['tf32_out'] else 1e-4)
    p_, dp_ = inp(P, p), inp(P, dp)
    P.call = lambda K: K.softmax_bwd(p_, dp_, dx, scale, a['tf32_out'])
    P.det = True


@builder('layernorm_fwd')
def _layernorm_fwd(P, gen):
    """One warp per row: a lane sums every 32nd column and 5 shuffle levels combine the lanes, so a chain has
    n = ceil(cols / 32) + 5 terms.  mean: such a sum and a division (k = 2) of sum |x| / cols.  var: the same for (x - mean)^2 plus the
    mean's error times 2 mean|x - mean|; std = sqrt(var + eps) carries half the relative error of var + eps and one
    rounding.  y = (x - mean) / std: (dmean + u |x - mean|) / std + |y| (dstd / std + u)."""
    c = P.case
    a = c['args']
    cols, eps = a['cols'], c.get('eps', 1e-5)
    x = randn(a['x']['shape'], gen)
    rows = x.numel() // cols
    x = x.view(rows, cols)
    if c.get('content') == 'const_and_offset':             # constant rows (std = sqrt(eps)) and mean >> std rows
        x[0::3] = x[0::3, :1]
        x[1::3] = x[1::3] * 0.01 + 300.0
    ref, bound, mu, dmu, sd, dsd = layernorm_fwd_ref(x.double().to(P.dev), eps)
    y = place(P, 'y', (rows, cols), ref, bound)
    if c.get('content') == 'const_and_offset':
        # x - mean loses log2(|mean| / std) ~ 15 bits on the mean >> std rows, so their error is ~1e-3 of |y| (inside the
        # elementwise bound); the global check of the older suite applies to the well-conditioned random rows
        P.outs[-1]['tol_rows'] = (torch.arange(rows, device=P.dev) % 3 == 2).view(-1, 1).expand(rows, cols)
    mean = place(P, 'mean', (rows,), mu.view(-1), dmu.view(-1))
    std = place(P, 'std', (rows,), sd.view(-1), dsd.view(-1))
    xd_ = inp(P, x)
    P.call = lambda K: K.layernorm_fwd(xd_, y, mean, std, cols, eps)
    P.det = True


def layernorm_bwd_ref(dy, y, sd, yterm=True):
    m1 = dy.mean(1, keepdim=True)
    m2 = (dy * y).mean(1, keepdim=True) if yterm else 0.0
    return (dy - m1 - y * m2) / sd


@builder('layernorm_bwd')
def _layernorm_bwd(P, gen):
    """dx = (dy - mean dy - y mean(dy y)) / std: two sums of cols terms, then three roundings and a reciprocal:
    C_SUM (cols + 6) u (|dy| + mean|dy| + |y| mean|dy y|) / std."""
    c = P.case
    a = c['args']
    cols = a['cols']
    rows = int(np.prod(a['dy']['shape'])) // cols
    y = randn((rows, cols), gen)
    y = (y - y.mean(1, keepdim=True)) / y.std(1, unbiased=False, keepdim=True).clamp(min=1e-3)
    dy = randn((rows, cols), gen)
    sd = torch.rand(rows, generator=gen) + 0.5
    yd, dyd, sdd = y.double().to(P.dev), dy.double().to(P.dev), sd.double().to(P.dev).view(-1, 1)
    ref, bound = layernorm_bwd_refb(dyd, yd, sdd)
    dx = place(P, 'dx', (rows, cols), ref, bound, tol=1e-4)
    y_, dy_, sd_ = inp(P, y), inp(P, dy), inp(P, sd)
    P.call = lambda K: K.layernorm_bwd(dy_, y_, sd_, dx, cols)
    P.det = True


def colsum_terms(rows, cols):
    """Terms per fp32 chain of vlfb_colsum: a thread sums every 8th row of its slab, 8 partials are added, and the
    slabs are combined by atomics (the host's slab count of ops.cu vlfb_colsum)."""
    cb = -(-cols // 32)
    slabs = min((2 * 132 + cb - 1) // cb, (rows + 63) // 64)
    slabs = max(slabs, 1)
    rpb = -(-rows // slabs)
    return -(-rpb // 8) + 8 + slabs, slabs, rpb


@builder('colsum')
def _colsum(P, gen):
    """out[c] (+)= sum_r x[r ld + c]: C_SUM (n + 2) u (sum |x| + |prev|), n = the terms of one chain (colsum_terms)."""
    c = P.case
    a = c['args']
    rows, cols, ld = a['rows'], a['cols'], a['ld']
    x = randn(a['x']['shape'], gen)
    xs = x.reshape(-1)[:rows * ld].view(rows, ld)[:, :cols].double().to(P.dev)
    prev = randn((cols,), gen).to(P.dev) if a['accumulate'] else None
    n, _, _ = colsum_terms(rows, cols)
    ref, bound = colsum_ref(xs, None if prev is None else prev.double(), n)
    out = place(P, 'out', a['out']['shape'], ref, bound, prev=prev, tol=2e-5)
    x_ = inp(P, x)
    P.call = lambda K: K.colsum(x_, ld, out, rows, cols, a['accumulate'])


def _conv_geom_obj(g):
    from vlfb import libvlfb as L
    o = L.ConvGeom()
    for f in GEOM_FIELDS:
        setattr(o, f, int(g[f]))
    return o


def _nc(x, g):       # [N,T,H,W,C] -> [N,C,T,H,W]
    return x.permute(0, 4, 1, 2, 3)


def maxpool_ref(x_cl, g, last_tie=False):
    """(values [N,To,Ho,Wo,C], argmax = ((n T + t) H + h) W + w with torch's first-index rule)."""
    import torch.nn.functional as F
    xd = _nc(x_cl.double(), g)
    if last_tie:                                      # the mirrored scan order picks the last of equal maxima
        xd = xd.flip(2, 3, 4)
    y, idx = F.max_pool3d(xd, (g['kT'], g['kH'], g['kW']), (g['sT'], g['sH'], g['sW']), (g['pT'], g['pH'], g['pW']),
                          return_indices=True)
    if last_tie:
        thw = g['T'] * g['H'] * g['W']
        t, h, w = idx // (g['H'] * g['W']), (idx // g['W']) % g['H'], idx % g['W']
        idx = ((g['T'] - 1 - t) * g['H'] + (g['H'] - 1 - h)) * g['W'] + (g['W'] - 1 - w)
        y, idx = y.flip(2, 3, 4), idx.flip(2, 3, 4)
        assert thw > 0
    n = torch.arange(g['N'], device=idx.device).view(-1, 1, 1, 1, 1)
    arg = idx + n * g['T'] * g['H'] * g['W']
    return y.permute(0, 2, 3, 4, 1), arg.permute(0, 2, 3, 4, 1).to(torch.int32)


def _pool_input(P, gen, g, kind):
    shape = (g['N'], g['T'], g['H'], g['W'], g['C'])
    x = content(shape, gen, kind)
    if kind == 'neg':                                    # all negative: the padding must lose against every value
        x = -x.abs() - 0.5
    return x


@builder('maxpool_fwd')
def _maxpool_fwd(P, gen):
    """Bit-exact values and argmax (torch's first index among equal maxima, -inf padding)."""
    c = P.case
    g = c['args']['g']
    x = _pool_input(P, gen, g, c.get('content', 'int'))
    y, arg = maxpool_ref(x.to(P.dev), g)
    yo = place(P, 'y', c['args']['y']['shape'], y.float())
    ao = place(P, 'argmax', c['args']['argmax']['shape'], arg, dtype=torch.int32) if c['args']['argmax'] else None
    x_, go = inp(P, x), _conv_geom_obj(g)
    P.call = lambda K: K.maxpool_fwd(x_, yo, ao, go)
    P.det = True


def _scatter_windows(g, arg, dy, keep=None):
    """sum over pool windows of dy at the window's argmax: (value, sum |terms|, max terms per element)."""
    n_in = g['N'] * g['T'] * g['H'] * g['W']
    C = g['C']
    d = dy.double() if keep is None else torch.where(keep, dy.double(), torch.zeros((), dtype=torch.float64, device=dy.device))
    flat = (arg.long() * C + torch.arange(C, device=arg.device)).reshape(-1)
    v = torch.zeros(n_in * C, dtype=torch.float64, device=dy.device).index_add_(0, flat, d.reshape(-1))
    m = torch.zeros(n_in * C, dtype=torch.float64, device=dy.device).index_add_(0, flat, d.abs().reshape(-1))
    return v.view(g['N'], g['T'], g['H'], g['W'], C), m.view(g['N'], g['T'], g['H'], g['W'], C)


@builder('maxpool_bwd', 'maxpool_bwd_gather')
def _maxpool_bwd(P, gen):
    """dx = sum of dy over the windows whose argmax the element is (the gather form: windows with y <= 0 pass nothing,
    tf32_out rounds).  n = kT kH kW windows at most per element; the scatter form adds them to finite contents |prev|
    by atomics (k = 2).  tf32_out adds one TF32 ulp."""
    c = P.case
    a = c['args']
    g = a['g']
    x = _pool_input(P, gen, g, c.get('content', 'int'))
    if c.get('relu_zero'):                               # a ReLU output: many windows whose maximum is exactly 0
        x = x.clamp(min=0)
    xd = x.to(P.dev)
    y, arg = maxpool_ref(xd, g)
    dy = randn(a['dy']['shape'], gen).to(P.dev)
    go = _conv_geom_obj(g)
    arg_ = inp(P, arg)
    dy_ = inp(P, dy)
    if c['fn'] == 'maxpool_bwd':
        prev = randn(a['dx']['shape'], gen).to(P.dev)
        ref, bound = maxpool_bwd_refb(g, arg, dy, prev=prev.double())
        dx = place(P, 'dx', a['dx']['shape'], ref, bound, prev=prev, tol=2e-5)
        P.call = lambda K: K.maxpool_bwd(dy_, arg_, dx, go)
        return
    keep = (y > 0) if a['y'] is not None else None
    ref, bound = maxpool_bwd_refb(g, arg, dy, keep, tf32_out=a['tf32_out'])
    dx = place(P, 'dx', a['dx']['shape'], ref, bound, tol=6e-4 if a['tf32_out'] else 2e-5)
    y_ = inp(P, y.float()) if a['y'] is not None else None
    P.call = lambda K: K.maxpool_bwd_gather(dy_, arg_, y_, dx, go, a['tf32_out'])
    P.det = True


def avgpool_bwd_ref(dy, g, drop_window=False):
    import torch.nn.functional as F
    shape = (g['N'], g['C'], g['T'], g['H'], g['W'])
    d = _nc(dy.double(), g)
    if drop_window:                                       # one border window (the last along W) missing
        d = d.clone()
        d[..., -1] = 0
    x = torch.zeros(shape, dtype=torch.float64, device=dy.device, requires_grad=True)
    y = F.avg_pool3d(x, (g['kT'], g['kH'], g['kW']), (g['sT'], g['sH'], g['sW']))
    (gx,) = torch.autograd.grad(y, x, d)
    return gx.permute(0, 2, 3, 4, 1)


@builder('avgpool_fwd', 'avgpool_bwd')
def _avgpool(P, gen):
    """A sum of n = kT kH kW terms times fp32(1/n): C_SUM (n + 3) u sum |terms| (k = 3: the reciprocal, the product and
    the accumulate flag's addition of |prev|)."""
    c = P.case
    a = c['args']
    g = a['g']
    go = _conv_geom_obj(g)
    if c['fn'] == 'avgpool_fwd':
        x = randn((g['N'], g['T'], g['H'], g['W'], g['C']), gen).to(P.dev)
        ref, bound = avgpool_fwd_ref(x.double(), g)
        y = place(P, 'y', a['y']['shape'], ref, bound)
        x_ = inp(P, x)
        P.call = lambda K: K.avgpool_fwd(x_, y, go)
    else:
        dy = randn(a['dy']['shape'], gen).to(P.dev)
        prev = randn(a['dx']['shape'], gen).to(P.dev) if a['accumulate'] else None
        ref, bound = avgpool_bwd_refb(dy, g, None if prev is None else prev.double())
        dx = place(P, 'dx', a['dx']['shape'], ref, bound, prev=prev)
        dy_ = inp(P, dy)
        P.call = lambda K: K.avgpool_bwd(dy_, dx, go, a['accumulate'])
    P.det = True


@builder('affine_fwd', 'affine_bwd')
def _affine(P, gen):
    """y = x s (+ b): one fused multiply-add, at most two roundings of |x s| + |b|."""
    c = P.case
    a = c['args']
    x = randn((a['x'] if c['fn'] == 'affine_fwd' else a['dy'])['shape'], gen)
    s = randn(a['s']['shape'], gen)
    b = randn(a['b']['shape'], gen) if c['fn'] == 'affine_fwd' else torch.zeros(a['s']['shape'])
    xd, sd, bd = x.double().to(P.dev), s.double().to(P.dev), b.double().to(P.dev)
    ref, bound = affine_ref(xd, sd, bd)
    x_, s_ = inp(P, x), inp(P, s)
    if c['fn'] == 'affine_fwd':
        y, b_ = place(P, 'y', a['y']['shape'], ref, bound), inp(P, b)
        P.call = lambda K: K.affine_fwd(x_, s_, b_, y)
    else:
        dx = place(P, 'dx', a['dx']['shape'], ref, bound)
        P.call = lambda K: K.affine_bwd(x_, s_, dx)
    P.det = True


def roi_matrix(rois, N, H, W, PH, PW, scale, sr, swap_clamped=False):
    """[R PH PW, N H W] fp64 matrix of the bilinear weights / sample count (oracle/roi_align_np.py sample table: the
    fp32 index arithmetic of the kernel), and the number of samples per bin.  swap_clamped: two weights of one sample
    on the clamp branch exchanged (a planted error)."""
    from oracle import roi_align_np
    tab = roi_align_np.sample_table(rois.cpu().numpy(), H, W, PH, PW, scale, sr)
    R = len(tab)
    M = torch.zeros((R * PH * PW, N * H * W), dtype=torch.float64)
    nmax = 1
    for r, t in enumerate(tab):
        cnt = t['grid_h'] * t['grid_w']
        nmax = max(nmax, 4 * cnt)
        pos, w = t['pos'], t['w'].astype(np.float64)
        if swap_clamped:
            hit = np.argwhere((pos[..., 0] == pos[..., 2]) & (pos[..., 0] >= 0) & (w[..., 0] != w[..., 1]))
            if len(hit):
                i = tuple(hit[0])
                w[i + (0,)], w[i + (1,)] = w[i + (1,)], w[i + (0,)]
        base = t['batch'] * H * W
        for ph in range(PH):
            for pw in range(PW):
                row = (r * PH + ph) * PW + pw
                for iy in range(t['grid_h']):
                    for ix in range(t['grid_w']):
                        for k in range(4):
                            if pos[ph, pw, iy, ix, k] >= 0:
                                M[row, base + pos[ph, pw, iy, ix, k]] += w[ph, pw, iy, ix, k] / cnt
    return M, nmax


def make_rois(gen, R, N, H, W, scale, kind='random'):
    """(R, 5) boxes in input pixels: random ones inside the map, plus with kind='edges' a box partly outside, one fully
    outside, one on the last row / column (the clamp branch), a degenerate one and a full-frame one."""
    Himg, Wimg = H / scale, W / scale
    b = torch.randint(0, N, (R,), generator=gen).float()
    x1 = torch.rand(R, generator=gen) * Wimg * 0.7
    y1 = torch.rand(R, generator=gen) * Himg * 0.7
    x2 = x1 + torch.rand(R, generator=gen) * Wimg * 0.3 + 2
    y2 = y1 + torch.rand(R, generator=gen) * Himg * 0.3 + 2
    rois = torch.stack([b, x1, y1, x2, y2], 1)
    if kind == 'edges':
        e = [[N - 1, -40.3, -25.1, 60.2, 70.7], [N - 1, Wimg + 30.0, Himg + 50.0, Wimg + 90.0, Himg + 99.0],
             [0, Wimg - 20.2, Himg - 12.6, Wimg - 0.5, Himg - 0.25], [N - 1, 33.3, 44.4, 33.9, 45.0],
             [0, 0.0, 0.0, Wimg - 1, Himg - 1], [N - 1, Wimg * 0.5, Himg - 30.0, Wimg + 40.0, Himg + 20.0]]
        rois[:len(e)] = torch.tensor(e, dtype=torch.float32)
    return rois


@builder('roi_align_fwd', 'roi_align_bwd')
def _roi_align(P, gen):
    """out = sum over 4 gh gw bilinear terms / cnt (weights bit-exact from the fp32 sample table): C_SUM (n + 2) u
    sum |w feat| / cnt.  The backward adds n' <= 4 gh gw terms per RoI to finite dfeat contents by atomics."""
    c = P.case
    a = c['args']
    scale, sr = c.get('spatial_scale', 1.0 / 16), a['sampling_ratio']
    if c['fn'] == 'roi_align_fwd':
        N, H, W, C = a['feat']['shape']
        R, PH, PW, _ = a['out']['shape']
    else:
        N, H, W, C = a['dfeat']['shape']
        R, PH, PW, _ = a['dout']['shape']
    rois = make_rois(gen, R, N, H, W, scale, c.get('content', 'random'))
    M, nmax = roi_matrix(rois, N, H, W, PH, PW, scale, sr)
    M = M.to(P.dev)
    rois_ = inp(P, rois)
    if c['fn'] == 'roi_align_fwd':
        feat = randn((N, H, W, C), gen).to(P.dev)
        f2 = feat.double().view(N * H * W, C)
        ref, bound = roi_align_fwd_ref(M, nmax, f2)
        out = place(P, 'out', a['out']['shape'], ref.view(R, PH, PW, C), bound.view(R, PH, PW, C))
        feat_ = inp(P, feat)
        P.call = lambda K: K.roi_align_fwd(feat_, rois_, out, scale, sr)
        P.det = True
    else:
        dout = randn((R, PH, PW, C), gen).to(P.dev)
        d2 = dout.double().view(R * PH * PW, C)
        prev = randn((N, H, W, C), gen).to(P.dev)
        ref, bound = roi_align_bwd_ref(M, d2, prev.double().view(N * H * W, C))
        dfeat = place(P, 'dfeat', a['dfeat']['shape'], ref.view(N, H, W, C), bound.view(N, H, W, C), prev=prev)
        dout_ = inp(P, dout)
        P.call = lambda K: K.roi_align_bwd(dout_, rois_, dfeat, scale, sr)


@builder('sigmoid_ce_fwd', 'sigmoid_ce_bwd')
def _sigmoid_ce(P, gen):
    """fwd: loss = scale sum_valid l_i / max(cnt, 1e-5); each l_i = log1p(__expf(.)) - ... carries the exp's error
    (C_EXP 2^-22 + C_ARG |x| u) times its derivative (< 1) and a few roundings of |x|: a sum of n terms of magnitude
    |l_i| + (|x_i| + 2) 2^-21.  bwd: dx = k (sigma(x) - t), k = scale dloss / cnt: the exp's error times
    sigma (1 - sigma) plus three roundings of |sigma| + |t|, and one of k."""
    c = P.case
    a = c['args']
    shape = a['logits']['shape']
    scale = c.get('scale', 1.0)
    x = randn(shape, gen, 3.0)
    t = torch.randint(0, 2, tuple(shape), generator=gen).int()
    t[torch.rand(tuple(shape), generator=gen) < 0.2] = -1
    if c.get('content') == 'all_ignored':
        t[:] = -1
    xd, td = x.double().to(P.dev), t.to(P.dev)
    x_, t_ = inp(P, x), inp(P, t)
    if c['fn'] == 'sigmoid_ce_fwd':
        ref, bound = sigmoid_ce_fwd_ref(xd, td, scale)
        loss = place(P, 'loss', (1,), ref, bound)
        P.call = lambda K: K.sigmoid_ce_fwd(x_, t_, loss, scale)
    else:
        dl = 0.5 if a['dloss'] is not None else 1.0
        ref, bound = sigmoid_ce_bwd_ref(xd, td, scale, dl)
        dx = place(P, 'dlogits', shape, ref, bound)
        dl_ = inp(P, torch.tensor([dl])) if a['dloss'] is not None else None
        P.call = lambda K: K.sigmoid_ce_bwd(x_, t_, dl_, dx, scale)
    P.det = True


@builder('sgd_nesterov')
def _sgd(P, gen):
    """g' = g + wd p; m' = mu m + lr g'; step = (1 + mu) m' - mu m (nesterov) or m'; p' = p - step: every line is one
    or two roundings (fused or not) of its terms plus the propagated error of its inputs.  p_tf32 must be exactly
    tf32_round(p')."""
    c = P.case
    a = c['args']
    n = a['p']['shape']
    mu, wd, lr = (float(np.float32(v)) for v in (0.9, 1e-4, 0.01))      # the fp32 values the kernel uses
    p, g, m = randn(n, gen), randn(n, gen, 0.1), randn(n, gen, 0.05)
    pd, gd, md = p.double().to(P.dev), g.double().to(P.dev), m.double().to(P.dev)
    r = sgd_ref(pd, gd, md, lr, mu, wd, a['nesterov'])
    (p2, ep), (st, es), (m2, em) = r['p'], r['g'], r['m']
    pb, gb, mb = (nan_buffer(GUARD + int(np.prod(n)) + TAIL, P.dev) for _ in range(3))
    idx = torch.arange(int(np.prod(n)), device=P.dev).view(n) + GUARD
    for b_, v in ((pb, p), (gb, g), (mb, m)):
        b_[idx.reshape(-1)] = v.reshape(-1).to(P.dev)
    add_out(P, 'p', pb, idx, p2, ep)
    add_out(P, 'g', gb, idx, st, es)
    add_out(P, 'm', mb, idx, m2, em)
    view = lambda b_: b_[GUARD:GUARD + int(np.prod(n))].view(n)
    pt = place(P, 'p_tf32', n, p2, ep + ulp_tf32(p2), tol=6e-4) if a['p_tf32'] is not None else None
    lr_ = inp(P, torch.tensor([lr]))
    P.call = lambda K: K.sgd_nesterov(view(pb), view(gb), view(mb), lr_, mu, wd, a['nesterov'], pt)
    P.pt_of_p = pt is not None
    P.det = True


def fbo_ref(a0, bp, Ws, scale, pre_act_ln, keeps, inv_keep, eps=1e-5):
    """As-written NLLayers / NLCore (lfb_helper.py:170-292) in fp64, phi and g formed; keeps[i] = the dropout keep mask
    of layer i's output (None: no dropout)."""
    import torch.nn.functional as F
    A = a0
    outs = []
    for W, keep in zip(Ws, keeps):
        theta = A @ W['w_theta'].t() + W['b_theta']
        phi = bp @ W['w_phi'].t() + W['b_phi']
        g = bp @ W['w_g'].t() + W['b_g']
        aff = torch.einsum('rd,rld->rl', theta, phi) * scale
        if aff.requires_grad:
            aff.retain_grad()
        p = torch.softmax(aff, dim=1)
        t = torch.einsum('rl,rld->rd', p, g)
        x = F.layer_norm(t, (t.shape[1],), eps=eps) if pre_act_ln else t
        out = torch.relu(x) @ W['w_out'].t() + W['b_out']
        A = A + (out if keep is None else out * keep * inv_keep)
        outs.append(dict(theta=theta, prob=p, t=t, xhat=x, out=out, a_out=A, aff=aff))
    return A, outs


FBO_W = ('w_theta', 'b_theta', 'w_phi', 'b_phi', 'w_g', 'b_g', 'w_out', 'b_out')
FBO_SAVED = ('theta', 'prob', 't', 'xhat', 'out', 'a_out')


@builder('fbo_nl_fwd', 'fbo_nl_bwd')
def _fbo_nl(P, gen):
    """Every saved activation (fwd) and every gradient (bwd).  The stack chains per layer a dot product of dA terms
    (theta), of d and dB terms (u, scores), a softmax over L, a weighted sum over L, LayerNorm over d and products of d
    terms; the error of an element is bounded by C_SUM (dA + d + dB + L + 8) u per layer, relative to the element's
    own magnitude plus its row's mean magnitude (the dot products that feed it are of the row's scale).  This bound is
    a mixed relative one, not derived term by term like the streaming families.  The dropout masks of the reference
    come from the numpy Philox generator, so a mask that differs in one element fails by the element's full value."""
    c = P.case
    a = c['args']
    cf = a['cfgd']
    R, L, dA, d, dB = cf['R'], cf['L'], cf['dA'], cf['d'], cf['dB']
    nl = len(a['layers'])
    ratio = 0.2 if cf['drop_ratio'] else 0.0
    seed, stepv = 4242, c.get('step', 3)
    scale = d ** -0.5
    rn = lambda *s, sc=1.0: torch.randn(*s, generator=gen) * sc
    a0, bp = rn(R, dA), rn(R, L, dB, sc=0.7)
    Ws = [dict(w_theta=rn(d, dA, sc=0.05), b_theta=rn(d, sc=0.1), w_phi=rn(d, dB, sc=0.08), b_phi=rn(d, sc=0.1),
               w_g=rn(d, dB, sc=0.05), b_g=rn(d, sc=0.1), w_out=rn(dA, d, sc=0.05), b_out=rn(dA, sc=0.1))
          for _ in range(nl)]
    offs = [1000 + 7919 * i for i in range(nl)]
    st = stepv if cf.get('step') is not None else 0
    keeps = [torch.from_numpy(dropout_keep(R * dA, ratio, seed, o + (st << 32), 0)).view(R, dA).double().to(P.dev)
             if ratio > 0 else None for o in offs]
    inv = float(np.float32(1.0) / (np.float32(1.0) - np.float32(ratio)))
    a64 = a0.double().to(P.dev).requires_grad_(True)
    b64 = bp.double().to(P.dev).requires_grad_(True)
    W64 = [dict((k, v.double().to(P.dev).requires_grad_(True)) for k, v in W.items()) for W in Ws]
    A_ref, outs = fbo_ref(a64, b64, W64, scale, cf['pre_act_ln'], keeps, inv)
    tau = fbo_tau(L, dA, d, dB, nl)
    bnd = lambda ref: fbo_bound(ref, tau)
    dev = lambda t: inp(P, t.float())
    lay = []
    for i, W in enumerate(Ws):
        ld = dict((k, dev(W[k])) for k in FBO_W if a['layers'][i].get(k) is not None)
        ld['drop_offset'] = offs[i]
        lay.append(ld)
    cfgd = dict(R=R, L=L, dA=dA, d=d, dB=dB, scale=scale, pre_act_ln=cf['pre_act_ln'], drop_ratio=ratio, seed=seed,
                step=inp(P, torch.tensor([stepv], dtype=torch.int64)) if cf.get('step') is not None else None)
    a0_, bp_ = dev(a0), dev(bp)
    shapes = dict(theta=(R, d), prob=(R, L), s=(R, dB), t=(R, d), xhat=(R, d), ln_mean=(R,), ln_std=(R,), out=(R, dA),
                  a_out=(R, dA))
    if c['fn'] == 'fbo_nl_fwd':
        for i, ld in enumerate(lay):
            for k, shp in shapes.items():
                if k in FBO_SAVED:
                    ref = outs[i][k].detach()
                    ld[k] = place(P, 'L%d.%s' % (i, k), shp, ref, bnd(ref), tol=1e-4)
                else:
                    ld[k] = inp(P, torch.empty(shp))
        P.call = lambda K: K.fbo_nl_fwd(cfgd, lay, a0_, bp_)
        P.det = True
        P.keeps = keeps
        return
    dlast = rn(R, dA)
    (A_ref * dlast.double().to(P.dev)).sum().backward()
    # the saved activations of the forward, from the reference (fp32), as the backward reads them
    for i, ld in enumerate(lay):
        o = outs[i]
        x_ = o['t'].detach()
        mu = x_.mean(1)
        sd = (x_.var(1, unbiased=False) + 1e-5).sqrt()
        s_ = torch.einsum('rl,rld->rd', o['prob'].detach(), b64.detach())
        for k, v in dict(theta=o['theta'], prob=o['prob'], s=s_, t=o['t'], xhat=o['xhat'], ln_mean=mu, ln_std=sd,
                         out=o['out'], a_out=o['a_out']).items():
            ld[k] = inp(P, v.detach().float())
        for k in FBO_W:
            if a['layers'][i].get('g' + k) is None or k not in ld:
                continue
            prev = torch.full(Ws[i][k].shape, 0.25, device=P.dev)
            grad = W64[i][k].grad.detach()
            b_ = bnd(grad)
            if k == 'b_phi':        # exactly 0: theta_o sum_j dscore_j, where the sum cancels to rounding noise
                b_ = fbo_b_phi_bound(o['theta'], o['aff'].grad, tau)
            ld['g' + k] = place(P, 'L%d.g%s' % (i, k), tuple(Ws[i][k].shape), grad + 0.25, b_ + 2 * U * 0.25,
                                prev=prev, tol=1e-4)
    da0 = place(P, 'da0', (R, dA), a64.grad.detach(), bnd(a64.grad), tol=5e-5)
    dbp = place(P, 'dbp', (R, L, dB), b64.grad.detach(), bnd(b64.grad), tol=5e-5)
    dl_ = dev(dlast)
    P.call = lambda K: K.fbo_nl_bwd(cfgd, lay, a0_, bp_, dl_, da0, dbp)
    P.det = True
    P.keeps = keeps


def bn_chain(rows, C):
    """Terms of one fp32 chain of the SpatialBN reductions (bn.cu reduce_dims): a thread sums every 8th row of its slab;
    the 8 partials and the slabs are then combined in fp64."""
    cb = -(-C // 32)
    slabs = max(min((4 * 132 + cb - 1) // cb, (rows + 127) // 128), 1)
    return -(-(-(-rows // slabs)) // 8)


def _f32v(v):
    return float(np.float32(v))


@builder('spatial_bn_fwd', 'spatial_bn_infer')
def _bn_fwd(P, gen):
    """Training forward.  d = mean(x - x0) (pivot x0 = row 0) is a sum of n = bn_chain fp32 terms, each with one rounding
    of the difference (k = 2): dd = C_SUM (n + 2) u mean|x - x0|; mean = x0 + d stored in fp32 (+ u |mean|).
    E2 = mean (x - x0)^2 likewise (k = 3: the difference's rounding doubles in the square); var = E2 - d^2 in fp64:
    dvar = dE2 + 2 |d| dd + dd^2.  inv_std = 1 / sqrt(var + eps): half the relative error of var + eps, plus its fp32
    store; fs = fp32(scale inv_std).  y = (x - mean) fs + b: |fs| (dmean + u |x - mean|) + |x - mean| dfs + two roundings
    of |(x - mean) fs| + |b|.  Running statistics: (1 - momentum) times the error of mean / unbiased var, plus two
    roundings.  Inference: fs = scale / sqrtf(var + eps) has three fp32 roundings; y as above with the given mean."""
    c = P.case
    a = c['args']
    rows, C = int(np.prod(a['x']['shape'][:-1])), a['x']['shape'][-1]
    eps, mom = _f32v(c.get('eps', 1e-5)), _f32v(c.get('momentum', 0.9))
    center = torch.randn(C, generator=gen) * c.get('offset_', 1000.0)     # mean ~ 10^3 std: what the pivot is for
    x = center + randn((rows, C), gen)
    s, b = torch.rand(C, generator=gen) + 0.5, randn((C,), gen)
    rm0, rv0 = randn((C,), gen), torch.rand(C, generator=gen) + 0.5
    xd, sd_, bd = x.double().to(P.dev), s.double().to(P.dev), b.double().to(P.dev)
    rmd, rvd = rm0.double().to(P.dev), rv0.double().to(P.dev)
    x_, s_, b_ = inp(P, x.view(a['x']['shape'])), inp(P, s), inp(P, b)
    if c['fn'] == 'spatial_bn_infer':
        ref, bound = bn_infer_ref(xd, sd_, bd, rmd, rvd, eps)
        y = place(P, 'y', a['y']['shape'], ref.view(a['y']['shape']), bound.view(a['y']['shape']))
        rm_, rv_ = inp(P, rm0), inp(P, rv0)
        P.call = lambda K: K.spatial_bn_infer(x_, s_, b_, rm_, rv_, y, eps)
        P.det = True
        return
    r = bn_fwd_ref(xd, sd_, bd, bn_chain(rows, C), eps, *((rmd, rvd, mom) if a['rm'] is not None else ()))
    ref, bound = r['y']
    y = place(P, 'y', a['y']['shape'], ref.view(a['y']['shape']), bound.view(a['y']['shape']))
    sm = place(P, 'saved_mean', (C,), *r['sm'])
    siv = place(P, 'saved_inv_std', (C,), *r['siv'])
    rm = rv = None
    if a['rm'] is not None:
        rm = place(P, 'running_mean', (C,), *r['rm'], prev=rm0.to(P.dev))
        rv = place(P, 'running_var', (C,), *r['rv'], prev=rv0.to(P.dev))
    P.call = lambda K: K.spatial_bn_fwd(x_, s_, b_, rm, rv, sm, siv, y, eps, mom)
    P.det = True


def bn_bwd_ref(dy, x, s, sm, siv, bx=True):
    """dx = A dy + B x + C of SpatialBN's backward (bx=False: without the B x term, a planted error)."""
    m = dy.shape[0]
    s1, s2 = dy.sum(0), (dy * (x - sm)).sum(0)
    A, B = s * siv, -s * siv ** 3 * s2 / m
    Cc = -A * s1 / m - B * sm
    return A * dy + (B * x if bx else 0) + Cc


@builder('spatial_bn_bwd')
def _bn_bwd(P, gen):
    """s1 = sum dy and s2 = sum dy (x - mean) are fp32 chains of n = bn_chain terms (k = 2, 3); A = fp32(s inv_std),
    B = fp32(-s inv_std^3 s2 / m), C = fp32(-A s1 / m - B mean) carry those errors and one rounding each; dx = A dy + B x
    + C adds |dy| dA + |x| dB + dC and three roundings of |A dy| + |B x| + |C|.  dscale += fp32(s2 inv_std),
    dbias += fp32(s1): the chains' errors plus two roundings of the accumulated values."""
    c = P.case
    a = c['args']
    rows, C = int(np.prod(a['x']['shape'][:-1])), a['x']['shape'][-1]
    center = torch.randn(C, generator=gen) * 1000.0
    x = center + randn((rows, C), gen)
    dy = randn((rows, C), gen)
    s = torch.rand(C, generator=gen) + 0.5
    sm = (x.double().mean(0)).float()
    siv = (1.0 / (x.double().var(0, unbiased=False) + 1e-5).sqrt()).float()
    xd, dyd, sd_ = x.double().to(P.dev), dy.double().to(P.dev), s.double().to(P.dev)
    smd, sivd = sm.double().to(P.dev), siv.double().to(P.dev)
    p_s, p_b = randn((C,), gen).to(P.dev), randn((C,), gen).to(P.dev)
    r = bn_bwd_refb(dyd, xd, sd_, smd, sivd, bn_chain(rows, C), p_s.double() if a['ds'] is not None else None,
                    p_b.double() if a['db'] is not None else None)
    ref, bound = r['dx']
    dx = place(P, 'dx', a['dx']['shape'], ref.view(a['dx']['shape']), bound.view(a['dx']['shape']))
    ds = db = None
    if a['ds'] is not None:
        ds = place(P, 'dscale', (C,), *r['ds'], prev=p_s)
    if a['db'] is not None:
        db = place(P, 'dbias', (C,), *r['db'], prev=p_b)
    x_, dy_, s_, sm_, siv_ = (inp(P, t) for t in (x.view(a['x']['shape']), dy.view(a['dy']['shape']), s, sm, siv))
    P.call = lambda K: K.spatial_bn_bwd(dy_, x_, s_, sm_, siv_, dx, ds, db)
    P.det = True


@builder('softmax_ce_fwd', 'softmax_ce_bwd')
def _softmax_ce(P, gen):
    """One 256-thread block walks the rows.  prob: as softmax_fwd with scale 1 over chains of n = ceil(cols / 256) + 10
    terms (a thread's columns, then the block reduction).  loss = scale / rows sum_r (mx + log s - x[label]): each row
    term carries log's error (2^-21 absolute for __logf, plus the relative error of s) and two roundings of its parts;
    the rows are then summed in fp32.  bwd: dx = (prob - [c == label]) scale / rows: three roundings."""
    c = P.case
    a = c['args']
    rows, cols = (a['logits'] if c['fn'] == 'softmax_ce_fwd' else a['prob'])['shape']
    scale = c.get('scale', 1.0)
    x = randn((rows, cols), gen, 4.0)
    lab = torch.randint(0, cols, (rows,), generator=gen).int()
    lab[0], lab[-1] = 0, cols - 1
    lab_ = inp(P, lab)
    labd = lab.long().to(P.dev)
    if c['fn'] == 'softmax_ce_bwd':
        prob = torch.softmax(x, 1)
        ref, bound = softmax_ce_bwd_ref(prob.double().to(P.dev), labd, scale)
        dx = place(P, 'dlogits', (rows, cols), ref, bound)
        p_ = inp(P, prob)
        P.call = lambda K: K.softmax_ce_bwd(p_, lab_, dx, scale)
        P.det = True
        return
    r = softmax_ce_fwd_ref(x.double().to(P.dev), labd, scale)
    prob = place(P, 'prob', (rows, cols), *r['prob'])
    loss = place(P, 'loss', (1,), *r['loss'])
    x_ = inp(P, x)
    P.call = lambda K: K.softmax_ce_fwd(x_, lab_, prob, loss, scale)
    P.det = True


def scan_rows(D, bf16):
    if bf16:
        return {4096: 4, 2048: 4}[D]
    return {4096: 4, 2048: 8, 1024: 8}[D]


def scan_splits(R, L, D, bf16):
    """vlfb_fbo_bank_scan_splits_dt (fbo.cu): the split of a RoI's L rows over CTAs, replicated."""
    rows = scan_rows(D, bf16)
    best, best_cost = 1, 1e30
    for s in range(1, min((L + rows - 1) // rows, 1024) + 1):
        per = (L + s - 1) // s
        if (s - 1) * per >= L:
            continue
        cost = ((R * s + 263) // 264) * ((per + rows - 1) // rows + 0.5)
        if cost < best_cost - 1e-9:
            best_cost, best = cost, s
    return best


@builder('fbo_bank_scan')
def _bank_scan(P, gen):
    """out = sum_j p_j b_j, p = softmax(scale q . b_j), online over S splits of ceil(L / S) rows in tiles.
    A score is a dot product of D terms in chains of D / 256 per thread, 5 shuffle and 8 warp levels (n_s = D / 256 + 13):
    ds_j = C_SUM (n_s + 2) u scale sum |q b_j|.  Relative error of p_j: ds_j + sum_k p_k ds_k (the normaliser), the exps of
    the scores and of every tile's rescaling (C_EXP 2^-22 + 2 u per tile of the split, and of the combine), their
    arguments (C_ARG u (|z_j| + the score range): the rescaling arguments telescope to the range), and the sums of
    L + S terms (C_SUM (L + S + 4) u).  out: sum_j p_j |b_j| times that relative error plus the weighted sum's own
    C_SUM (L + S + 4) u.  prob: p_j times the relative error.  tf32_out adds one TF32 ulp."""
    c = P.case
    a = c['args']
    R, L, D = a['bank']['shape']
    bf16 = a['bank']['dtype'] == 'bfloat16'
    scale = c.get('scale', D ** -0.5)
    bank = randn((R, L, D), gen)
    if bf16:
        bank = bank.to(torch.bfloat16)
    q = randn((R, D), gen)
    S = scan_splits(R, L, D, bf16)
    P.splits = S
    r = bank_scan_ref(bank.double().to(P.dev), q.double().to(P.dev), scale, S, bf16, a['tf32_out'])
    out = place(P, 'out', (R, D), *r['out'], tol=6e-4 if a['tf32_out'] else 1e-4)
    prob = place(P, 'prob', (R, L), *r['prob']) if a['prob'] is not None else None
    b_, q_ = inp(P, bank), inp(P, q)
    P.call = lambda K: K.fbo_bank_scan(b_, q_, out, scale, prob, a['tf32_out'])
    P.det = True


@builder('lfb_gather')
def _lfb_gather(P, gen):
    """Bit-exact: out[i] = bank[idx[i]] (TF32-rounded with tf32_out) for 0 <= idx < bank_rows, zeros for idx < 0 and
    for idx >= bank_rows."""
    c = P.case
    a = c['args']
    nb, D = a['bank']['shape']
    rows = a['idx']['shape'][0]
    bank = randn((nb, D), gen)
    idx = torch.randint(-1, nb + 1, (rows,), generator=gen).int()
    idx[:4] = torch.tensor([-1, 0, nb - 1, nb], dtype=torch.int32)[:min(4, rows)]
    ok = (idx >= 0) & (idx < nb)
    ref = torch.where(ok.view(-1, 1), bank[idx.long().clamp(0, nb - 1)], torch.zeros(()))
    if a['tf32_out']:
        ref = tf32_round(ref)
    out = place(P, 'out', (rows, D), ref.to(P.dev))
    b_, i_ = inp(P, bank), inp(P, idx)
    P.call = lambda K: K.lfb_gather(b_, i_, out, a['tf32_out'])
    P.det = True


@builder('cast_bf16')
def _cast_bf16(P, gen):
    """Bit-exact: round to nearest, ties to even (half-way values with an even and an odd bf16 mantissa, both signs,
    and a carry into the next binade)."""
    c = P.case
    a = c['args']
    n = a['x']['shape'][0]
    x = randn((n,), gen)
    i = x.view(torch.int32).clone()
    sel = torch.arange(n) % 3 != 2
    i[sel] = (i[sel] & ~0xFFFF) | 0x8000
    car = torch.arange(n) % 11 == 0
    i[car] = (i[car] & ~0x7FFFFF) | 0x7F8000
    x = i.view(torch.float32)
    ref = bf16_rne(x).to(torch.int16).view(torch.bfloat16).to(P.dev)
    y = place(P, 'y', (n,), ref, dtype=torch.bfloat16)
    x_ = inp(P, x)
    P.call = lambda K: K.cast_bf16(x_, y)
    P.det = True


# ----------------------------------------------------------------------------------------------- the case table
CASES = []


def _add(name, fn, seed, **kw):
    args = kw.pop('args')
    CASES.append(dict(name=name, fn=fn, seed=seed, args=args, **kw))


def _ew_args(fn, n, y_none=False):
    ins, outn = EW_ARGS[fn]
    a = dict((k, T(n)) for k in ins)
    a[outn] = T(n // 32, dtype='int32') if fn == 'relu_bits' else T(n)
    if y_none:
        a['y'] = None
    return a


BIG = CAP_ITEMS * 4 + 4 * 1000 + 1           # above the cap of the 4-per-thread grids: several grid-stride rounds
for i, fn in enumerate(sorted(EW_ARGS)):
    sizes = [32, 4 * 1024] if fn == 'relu_bits' else [0, 1, 3, 4 * 1001 + 1]
    for n in sizes:
        _add('%s_n%d' % (fn, n), fn, 10 + i, args=_ew_args(fn, n))
    if fn != 'relu_bits':
        for off in (1, 2, 3):                  # pointers 4-12 bytes past a 16-byte boundary: the scalar loop
            _add('%s_off%d' % (fn, off), fn, 40 + i, args=_ew_args(fn, 1027), off=off)
        _add('%s_big' % fn, fn, 70 + i, args=_ew_args(fn, BIG))
    else:
        _add('%s_big' % fn, fn, 70 + i, args=_ew_args(fn, CAP_ITEMS * 32 + 1024))
for fn in ('round_tf32', 'add_tf32', 'relu_tf32', 'add_relu_bwd_tf32', 'relu_bwd_tf32'):
    _add('%s_ties' % fn, fn, 90, args=_ew_args(fn, 4099), content='ties')
for al in ('a', 'b'):
    _add('add_relu_bwd_tf32_alias_%s' % al, 'add_relu_bwd_tf32', 91, args=_ew_args('add_relu_bwd_tf32', 40001), alias=al)
    _add('add_relu_bwd_tf32_alias_%s_off' % al, 'add_relu_bwd_tf32', 92, args=_ew_args('add_relu_bwd_tf32', 4001),
         alias=al, off=1)
_add('add_relu_bwd_tf32_no_mask', 'add_relu_bwd_tf32', 93, args=_ew_args('add_relu_bwd_tf32', 4001, y_none=True))
_add('add_relu_bwd_tf32_no_mask_alias_b', 'add_relu_bwd_tf32', 94,
     args=_ew_args('add_relu_bwd_tf32', 4001, y_none=True), alias='b')

for n, st in ((1, False), (3, True), (4 * 1001 + 1, False), (4 * 1001 + 3, True), (CAP_ITEMS * 4 + 4 * 77 + 2, True)):
    _add('dropout_n%d%s' % (n, '_step' if st else ''), 'dropout', 100,
         args=dict(x=T(n), y=T(n), step=T(1, dtype='int64') if st else None), step=5 if st else 0)
_add('dropout_off1', 'dropout', 101, args=dict(x=T(1001), y=T(1001), step=None), off=1)


def _copy_args(rows, cols, lds, ldd, so=0, do=0, acc=False):
    return dict(src=T(so + rows * lds), lds=lds, dst=T(do + rows * ldd), ldd=ldd, rows=rows, cols=cols,
                accumulate=acc, src_off=so, dst_off=do)


_add('copy2d_gaps', 'copy2d', 110, args=_copy_args(37, 29, 40, 35, 3, 5))
_add('copy2d_accumulate', 'copy2d', 111, args=_copy_args(37, 29, 40, 35, 0, 2, True))
_add('copy2d_big', 'copy2d', 112, args=_copy_args(2000, 300, 301, 310, 1, 0))
for C_, inner, cpad, tf in ((1, 37, 4, False), (2, 64, 4, True), (3, 1003, 4, True), (4, 40, 4, False),
                            (3, 41, 8, False), (70, 999, 72, True), (3, 2 * CAP_ITEMS + 4 * 333, 4, True)):
    _add('nc_to_cl_c%d_i%d_p%d' % (C_, inner, cpad), 'nc_to_cl', 120,
         args=dict(src=T(2, C_, inner), dst=T(2, inner, cpad), n=2, c=C_, inner=inner, cpad=cpad, tf32_out=tf, width=0,
                   pitch=0, left=0), content='ties' if tf else 'randn')
_add('nc_to_cl_pitched', 'nc_to_cl', 121,
     args=dict(src=T(2, 3, 5 * 16), dst=T(2, 5 * 24, 4), n=2, c=3, inner=80, cpad=4, tf32_out=True, width=16, pitch=24,
               left=3))
_add('nc_to_cl_pitched_big', 'nc_to_cl', 123,          # a 2 x 3 x 16 x 224 x 224 clip: > CAP_ITEMS pixel quads
     args=dict(src=T(2, 3, 16 * 224 * 224), dst=T(2, 16 * 224 * 232, 4), n=2, c=3, inner=16 * 224 * 224, cpad=4,
               tf32_out=True, width=224, pitch=232, left=4))
for C_, inner, cpad in ((3, 37, 4), (70, 999, 72), (64, CAP_ITEMS // 32, 64)):
    _add('cl_to_nc_c%d_i%d' % (C_, inner), 'cl_to_nc', 122,
         args=dict(src=T(2, inner, cpad), dst=T(2, C_, inner), n=2, c=C_, inner=inner, cpad=cpad))
_add('weight_transpose_tails', 'weight_transpose', 130, args=dict(w=T(70, 3, 3, 3, 45), wt=T(45, 27, 70), scale=T(70)))
_add('weight_transpose_no_scale', 'weight_transpose', 131, args=dict(w=T(33, 1, 1, 1, 65), wt=T(65, 1, 33), scale=None))

for cols in (1, 31, 33, 784, 3136, 3600):
    _add('softmax_fwd_c%d' % cols, 'softmax_fwd', 140, args=dict(x=T(5, cols), p=T(5, cols), tf32_out=cols == 784),
         spread=80.0 if cols in (33, 3600) else 3.0)
    _add('softmax_bwd_c%d' % cols, 'softmax_bwd', 141, args=dict(p=T(5, cols), dp=T(5, cols), dx=T(5, cols),
                                                                 tf32_out=cols == 3136))
_add('softmax_fwd_rows_big', 'softmax_fwd', 142, args=dict(x=T(132 * 16 * 8 + 77, 33), p=T(132 * 16 * 8 + 77, 33),
                                                          tf32_out=False))
_add('softmax_bwd_rows_big', 'softmax_bwd', 143, args=dict(p=T(132 * 16 * 8 + 77, 33), dp=T(132 * 16 * 8 + 77, 33),
                                                           dx=T(132 * 16 * 8 + 77, 33), tf32_out=False))
for cols in (1, 31, 33, 784, 3136, 3600):
    _add('layernorm_fwd_c%d' % cols, 'layernorm_fwd', 150, args=dict(x=T(6, cols), y=T(6, cols), mean=T(6), std=T(6),
                                                                    cols=cols), content='const_and_offset')
    _add('layernorm_bwd_c%d' % cols, 'layernorm_bwd', 151, args=dict(dy=T(6, cols), y=T(6, cols), std=T(6),
                                                                    dx=T(6, cols), cols=cols))
_add('layernorm_fwd_rows_big', 'layernorm_fwd', 152, args=dict(x=T(132 * 16 * 8 + 5, 64), y=T(132 * 16 * 8 + 5, 64),
                                                              mean=T(132 * 16 * 8 + 5), std=T(132 * 16 * 8 + 5), cols=64))
_add('layernorm_bwd_rows_big', 'layernorm_bwd', 153, args=dict(dy=T(132 * 16 * 8 + 5, 64), y=T(132 * 16 * 8 + 5, 64),
                                                              std=T(132 * 16 * 8 + 5), dx=T(132 * 16 * 8 + 5, 64),
                                                              cols=64))
for rows, cols, ld, acc in ((5, 37, 40, False), (63, 100, 128, True), (1200, 512, 512, True), (3000, 2050, 2053, False)):
    _add('colsum_r%d_c%d_ld%d' % (rows, cols, ld), 'colsum', 160,
         args=dict(x=T(rows * ld), ld=ld, out=T(cols), rows=rows, cols=cols, accumulate=acc))

_G_TIES = geom(2, 5, 9, 11, 8, (3, 3, 3), (2, 2, 2), (1, 1, 1))          # overlapping windows, padding, integer ties
_G_T2 = geom(2, 6, 7, 7, 12, (2, 1, 1), (2, 1, 1), (0, 0, 0))
_G_BIG = geom(2, 8, 72, 72, 128, (1, 3, 3), (1, 2, 2), (0, 1, 1))       # > CAP_ITEMS work items in all three kernels


def _pool_args(g, fn):
    xs, ys = T(g['N'], g['T'], g['H'], g['W'], g['C']), T(g['N'], g['To'], g['Ho'], g['Wo'], g['C'])
    if fn == 'maxpool_fwd':
        return dict(x=xs, y=ys, argmax=T(*ys['shape'], dtype='int32'), g=g)
    if fn == 'maxpool_bwd':
        return dict(dy=ys, argmax=T(*ys['shape'], dtype='int32'), dx=xs, g=g)
    if fn == 'maxpool_bwd_gather':
        return dict(dy=ys, argmax=T(*ys['shape'], dtype='int32'), y=ys, dx=xs, g=g, tf32_out=True)
    if fn == 'avgpool_fwd':
        return dict(x=xs, y=ys, g=g)
    return dict(dy=ys, dx=xs, g=g, accumulate=True)


for nm, g in (('ties', _G_TIES), ('t2', _G_T2), ('big', _G_BIG)):
    for fn in ('maxpool_fwd', 'maxpool_bwd', 'maxpool_bwd_gather'):
        _add('%s_%s' % (fn, nm), fn, 170, args=_pool_args(g, fn))
_add('maxpool_fwd_negative_vs_padding', 'maxpool_fwd', 171, args=_pool_args(_G_TIES, 'maxpool_fwd'), content='neg')
_add('maxpool_bwd_gather_relu_zero_max', 'maxpool_bwd_gather', 172, args=_pool_args(_G_TIES, 'maxpool_bwd_gather'),
     relu_zero=True)
_a = _pool_args(_G_TIES, 'maxpool_bwd_gather')
_a.update(y=None, tf32_out=False)
_add('maxpool_bwd_gather_no_mask', 'maxpool_bwd_gather', 173, args=_a)
for nm, g in (('s2_overlap', geom(2, 7, 9, 9, 8, (3, 3, 3), (2, 2, 2), (0, 0, 0))),
              ('k4_t', geom(2, 4, 7, 7, 64, (4, 1, 1), (1, 1, 1), (0, 0, 0))),
              ('big', geom(2, 8, 64, 64, 512, (2, 2, 2), (2, 2, 2), (0, 0, 0)))):
    _add('avgpool_fwd_%s' % nm, 'avgpool_fwd', 180, args=_pool_args(g, 'avgpool_fwd'))
    _add('avgpool_bwd_%s' % nm, 'avgpool_bwd', 181, args=_pool_args(g, 'avgpool_bwd'))

for fn in ('roi_align_fwd', 'roi_align_bwd'):
    for nm, (N, H, W, C, R, PH, PW, sr, kind) in dict(
            edges=(2, 14, 14, 2048, 9, 7, 7, 0, 'edges'), sr2_ph_ne_pw=(3, 10, 12, 64, 11, 5, 3, 2, 'edges'),
            big=(2, 16, 16, 512, 100, 7, 7, 0, 'random')).items():
        a = dict(rois=T(R, 5), sampling_ratio=sr)
        if fn == 'roi_align_fwd':
            a.update(feat=T(N, H, W, C), out=T(R, PH, PW, C))
        else:
            a.update(dout=T(R, PH, PW, C), dfeat=T(N, H, W, C))
        _add('%s_%s' % (fn, nm), fn, 190, args=a, content=kind)

_add('sigmoid_ce_fwd_all_ignored', 'sigmoid_ce_fwd', 200, args=dict(logits=T(4, 80), targets=T(4, 80, dtype='int32'),
                                                                   loss=T(1)), content='all_ignored')
_add('sigmoid_ce_fwd_big', 'sigmoid_ce_fwd', 201, args=dict(logits=T(3000, 81), targets=T(3000, 81, dtype='int32'),
                                                           loss=T(1)))
_add('sigmoid_ce_bwd_dloss', 'sigmoid_ce_bwd', 202, args=dict(logits=T(37, 80), targets=T(37, 80, dtype='int32'),
                                                             dloss=T(1), dlogits=T(37, 80)))
_add('sigmoid_ce_bwd_all_ignored', 'sigmoid_ce_bwd', 203, args=dict(logits=T(4, 80), targets=T(4, 80, dtype='int32'),
                                                                   dloss=None, dlogits=T(4, 80)), content='all_ignored')
for nest in (True, False):
    for pt in (True, False):
        _add('sgd_nesterov%d_tf32%d' % (nest, pt), 'sgd_nesterov', 210,
             args=dict(p=T(4 * 1001 + 3), g=T(4 * 1001 + 3), m=T(4 * 1001 + 3), lr=T(1), nesterov=nest,
                       p_tf32=T(4 * 1001 + 3) if pt else None))
_add('sgd_big', 'sgd_nesterov', 211, args=dict(p=T(CAP_ITEMS * 4 + 9), g=T(CAP_ITEMS * 4 + 9), m=T(CAP_ITEMS * 4 + 9),
                                               lr=T(1), nesterov=True, p_tf32=T(CAP_ITEMS * 4 + 9)))
_add('affine_fwd_big', 'affine_fwd', 220, args=dict(x=T(6000, 512), s=T(512), b=T(512), y=T(6000, 512)))
_add('affine_bwd_big', 'affine_bwd', 221, args=dict(dy=T(6000, 512), s=T(512), dx=T(6000, 512)))

for rows, C, run in ((1, 4, True), (7, 4, True), (8 * 5 + 3, 4, False), (8 * 131 + 3, 64, True),
                     (8 * 5003 + 3, 64, True)):
    _add('spatial_bn_fwd_r%d_c%d' % (rows, C), 'spatial_bn_fwd', 240,
         args=dict(x=T(rows, C), s=T(C), b=T(C), rm=T(C) if run else None, rv=T(C) if run else None, sm=T(C), siv=T(C),
                   y=T(rows, C)))
    if rows > 1:
        _add('spatial_bn_bwd_r%d_c%d' % (rows, C), 'spatial_bn_bwd', 241,
             args=dict(dy=T(rows, C), x=T(rows, C), s=T(C), sm=T(C), siv=T(C), dx=T(rows, C), ds=T(C) if run else None,
                       db=T(C)))
    _add('spatial_bn_infer_r%d_c%d' % (rows, C), 'spatial_bn_infer', 242,
         args=dict(x=T(rows, C), s=T(C), b=T(C), rm=T(C), rv=T(C), y=T(rows, C)))
for rows, cols in ((4, 157), (37, 157), (3, 1000), (4000, 157)):
    _add('softmax_ce_fwd_r%d_c%d' % (rows, cols), 'softmax_ce_fwd', 250,
         args=dict(logits=T(rows, cols), labels=T(rows, dtype='int32'), prob=T(rows, cols), loss=T(1)))
    _add('softmax_ce_bwd_r%d_c%d' % (rows, cols), 'softmax_ce_bwd', 251,
         args=dict(prob=T(rows, cols), labels=T(rows, dtype='int32'), dlogits=T(rows, cols)))
# bank scans: (R, L) pairs whose split counts (scan_splits) range from 1 to many, with a partial last split and tile
for R, L, D, dt, tf, pr in ((1, 1, 2048, 'float32', False, True), (4, 300, 2048, 'float32', True, True),
                            (3, 301, 1024, 'float32', False, True), (300, 37, 2048, 'float32', False, False),
                            (5, 61, 4096, 'float32', True, True), (2, 2000, 2048, 'float32', False, True),
                            (4, 300, 2048, 'bfloat16', True, True), (3, 97, 4096, 'bfloat16', False, True)):
    _add('fbo_bank_scan_r%d_l%d_d%d_%s' % (R, L, D, dt), 'fbo_bank_scan', 260,
         args=dict(bank=T(R, L, D, dtype=dt), q=T(R, D), out=T(R, D), prob=T(R, L) if pr else None, tf32_out=tf))
for nb, rows, D, tf in ((10, 7, 64, False), (1000, 600, 2048, True), (50, 4800, 2048, False)):
    _add('lfb_gather_b%d_r%d_d%d' % (nb, rows, D), 'lfb_gather', 270,
         args=dict(bank=T(nb, D), idx=T(rows, dtype='int32'), out=T(rows, D), tf32_out=tf))
for n in (8, 8 * 1001, 8 * CAP_ITEMS + 8 * 123):
    _add('cast_bf16_n%d' % n, 'cast_bf16', 280, args=dict(x=T(n), y=T(n, dtype='bfloat16')))


def _fbo_args(fn, R, L, dA, d, dB, layers, ln=True, drop=True, step=True):
    lay = []
    for _ in range(layers):
        ld = dict((k, T(1)) for k in FBO_W)
        ld.update(dict(('g' + k, T(1)) for k in FBO_W))
        lay.append(ld)
    a = dict(cfgd=dict(R=R, L=L, dA=dA, d=d, dB=dB, pre_act_ln=ln, drop_ratio=drop,
                       step=T(1, dtype='int64') if step else None), layers=lay, a0=T(R, dA), bp=T(R, L, dB))
    if fn == 'fbo_nl_bwd':
        a.update(da_last=T(R, dA), da0=T(R, dA), dbp=T(R, L, dB))
    return a


for fn in ('fbo_nl_fwd', 'fbo_nl_bwd'):
    for nm, shp in dict(L1=(2, 1, 512, 512, 512, 1), L513_4layers=(3, 513, 512, 512, 512, 4),
                        L2000=(2, 2000, 512, 512, 512, 1), dA4096=(2, 40, 4096, 512, 512, 2),
                        dB600=(2, 37, 512, 600, 600, 2), R64=(64, 30, 512, 512, 512, 1)).items():
        _add('%s_%s' % (fn, nm), fn, 230, args=_fbo_args(fn, *shp))


# production launches (tests/golden/streaming_launches_config2.json, scripts/record_streaming_launches.py): one case per
# recorded signature, at the recorded shapes (every fp64 reference fits in the H100's memory, so none is scaled down)
PROD_FIXTURE = os.path.join(HERE, 'golden', 'streaming_launches_config2.json')


def production_signatures():
    import json
    with open(PROD_FIXTURE) as f:
        return json.load(f)['launches']


for _i, _r in enumerate(production_signatures()):
    _add('prod_%s_%d' % (_r['fn'], _i), _r['fn'], 300 + _i, args=_r['args'], prod=True)


def work_items(c):
    """(work items, items above which the grid-stride loop of the launch runs more than once) of a case, from the launch
    code in ops.cu / fbo.cu / bn.cu (stream_grid caps a grid at 132 * 16 blocks); None for kernels without such a loop
    (2-D tiled grids, one block or one CTA per row / RoI)."""
    fn, a = c['fn'], c['args']
    n = lambda k: int(np.prod(a[k]['shape']))
    g = a.get('g')
    if fn in EW_ARGS:
        return (n('x') if fn == 'relu_bits' else n(EW_ARGS[fn][1]), CAP_ITEMS if fn == 'relu_bits' else 4 * CAP_ITEMS)
    if fn in ('sgd_nesterov',):
        return n('p'), 4 * CAP_ITEMS
    if fn == 'dropout':
        return (n('x') + 3) // 4, CAP_ITEMS
    if fn == 'copy2d':
        return a['rows'] * a['cols'], CAP_ITEMS
    if fn == 'nc_to_cl':
        return (a['n'] * a['inner'] // 4, CAP_ITEMS) if (a['cpad'] == 4 and a['inner'] % 4 == 0) or a['pitch'] else None
    if fn in ('affine_fwd', 'affine_bwd'):
        return n('x' if fn == 'affine_fwd' else 'dy') // 4, CAP_ITEMS
    if fn in ('softmax_fwd', 'softmax_bwd', 'layernorm_fwd', 'layernorm_bwd'):
        x = a['x'] if 'x' in a else a['p'] if 'p' in a else a['dy']
        cols = x['shape'][-1] if fn.startswith('softmax') else a['cols']
        return int(np.prod(x['shape'])) // cols, CAP_ITEMS // 32          # one warp per row
    if fn in ('maxpool_fwd', 'avgpool_fwd'):
        return g['N'] * g['To'] * g['Ho'] * g['Wo'] * g['C'] // 4, CAP_ITEMS
    if fn == 'maxpool_bwd':
        return g['N'] * g['To'] * g['Ho'] * g['Wo'] * g['C'], CAP_ITEMS
    if fn in ('maxpool_bwd_gather', 'avgpool_bwd'):
        return g['N'] * g['T'] * g['H'] * g['W'] * g['C'] // 4, CAP_ITEMS
    if fn in ('roi_align_fwd', 'roi_align_bwd'):
        return n('out' if fn == 'roi_align_fwd' else 'dout') // 4, CAP_ITEMS
    if fn in ('spatial_bn_fwd', 'spatial_bn_infer', 'spatial_bn_bwd'):
        return n('x') // 4, CAP_ITEMS                                      # the apply pass
    if fn == 'softmax_ce_bwd':
        return n('prob'), CAP_ITEMS
    if fn == 'lfb_gather':
        return n('out') // 4, 4 * CAP_ITEMS
    if fn == 'cast_bf16':
        return n('x') // 8, CAP_ITEMS
    return None


def case_signature(c):
    return dict(fn=c['fn'], args=c['args'])


def case_by_name(name):
    return next(c for c in CASES if c['name'] == name)


# ----------------------------------------------------------------------------------------------- running / comparison
def prepare(c, dev):
    gen = torch.Generator().manual_seed(5000 + c['seed'])
    P = Prepared(c, dev)
    BUILD[c['fn']](P, gen)
    return P


def _results(P):
    return [o['buf'].view(-1)[o['index'].reshape(-1)].view(o['ref'].shape) for o in P.outs]


def check_case(K, c, dev):
    """Runs one case; returns its record (errors, worst bound ratio)."""
    rec = dict(case=c['name'], fn=c['fn'], errors=[], worst_ratio=0.0)
    P = prepare(c, dev)
    P.call(K)
    torch.cuda.synchronize()
    got = _results(P)
    for o, g in zip(P.outs, got):
        cmp = compare(g, o['ref'], o['bound'], o['tol'], o.get('tol_rows'))
        rec['worst_ratio'] = max(rec['worst_ratio'], cmp['worst_ratio'])
        if not cmp['ok']:
            rec['errors'].append('%s: %d elements outside the bound (worst %.3g x), rel_err %.3g' % (
                o['name'], cmp['nbad'], cmp['worst_ratio'], cmp['rel_err']))
        t = guard_touched(o['buf'], o['index'])
        if t:
            rec['errors'].append('%s: %d guard elements overwritten' % (o['name'], t))
    if getattr(P, 'pt_of_p', False):
        if not torch.equal(tf32_round(got[0].float().contiguous()), got[3].float()):
            rec['errors'].append('p_tf32 is not tf32_round(p)')
    if P.det and not rec['errors']:
        P2 = prepare(c, dev)
        P2.call(K)
        torch.cuda.synchronize()
        for o, a_, b_ in zip(P.outs, got, _results(P2)):
            bits = lambda t: t.contiguous().view(-1).view(BITS[t.dtype]) if t.dtype in BITS else t
            if not torch.equal(bits(a_), bits(b_)):
                rec['errors'].append('%s differs between two runs' % o['name'])
    rec['ok'] = not rec['errors']
    return rec
