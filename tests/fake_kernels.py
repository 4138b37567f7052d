"""TEST-ONLY stand-in for vlfb.kernels implemented with torch CPU ops.

It lets the host-side logic (net recording, lowering, fusion, autograd tape, ParamStore,
optimizer plan, data-parallel plumbing) be exercised on a machine without a GPU.  It lives
under tests/ on purpose: the product package has no CPU path and fails loudly without
libvlfb.so + CUDA.  Semantics mirror include/vlfb.h; TF32 rounding is the identity here.
"""
import torch
import torch.nn.functional as F

from vlfb import libvlfb as L
from vlfb.kernels import conv_geom, out_shape, _is_pointwise  # noqa: F401  (pure python helpers)
from util import pack_sign_bits, tf32_round


EMULATE_TF32 = False     # True: perform the TF32 roundings of the CUDA path (in whatever dtype the tensors have)


def _q(t, on=True):
    return tf32_round(t.detach()) if (EMULATE_TF32 and on) else t


def set_gemm_backend(name):
    pass


def _nc(x):     # [N,T,H,W,C] -> (N,C,T,H,W)
    return x.permute(0, 4, 1, 2, 3)


def _w_nc(w):   # [Co,kT,kH,kW,Ci] -> (Co,Ci,kT,kH,kW)
    return w.permute(0, 4, 1, 2, 3)


def _conv(x, w, g):
    return F.conv3d(_nc(x), w, None, (g.sT, g.sH, g.sW), (g.pT, g.pH, g.pW), (g.dT, g.dH, g.dW))


def _stem_w(w, g):
    return w[:, :, :, :g.kW, :3].permute(0, 4, 1, 2, 3)


def _unpack_bits(bits, shape):
    v = bits.to(torch.int64) & 0xFFFFFFFF
    return ((v.view(-1, 1) >> torch.arange(32, dtype=torch.int64)) & 1).reshape(shape) > 0


def relu_bits(x, bits):
    bits.copy_(pack_sign_bits(x))


def conv_fwd(x, w, y, g, scale=None, bias=None, residual=None, relu=False, tf32_out=False, relu_bits=None):
    if g.C == 4:
        o = F.conv3d(_nc(x)[:, :3], _stem_w(w, g), None, (g.sT, g.sH, g.sW), (g.pT, g.pH, g.pW))
    else:
        o = _conv(x, _w_nc(w.view(g.Co, g.kT, g.kH, g.kW, g.C)), g)
    o = o.permute(0, 2, 3, 4, 1)
    if scale is not None:
        o = o * scale
    if bias is not None:
        o = o + bias
    if residual is not None:
        o = o + residual
    if relu:
        o = torch.relu(o)
    y.copy_(_q(o, tf32_out))
    if relu_bits is not None:
        assert relu
        relu_bits.copy_(pack_sign_bits(y))


def conv_dgrad(dy, wt, dx, g, accumulate=False, residual=None, relu_mask=None, tf32_out=False, relu_mask_bits=None):
    taps = g.kT * g.kH * g.kW
    w = wt.view(g.C, taps, g.Co).permute(2, 1, 0).reshape(g.Co, g.kT, g.kH, g.kW, g.C)
    x = torch.zeros((g.N, g.C, g.T, g.H, g.W), dtype=dy.dtype, requires_grad=True)
    y = F.conv3d(x, _w_nc(w), None, (g.sT, g.sH, g.sW), (g.pT, g.pH, g.pW), (g.dT, g.dH, g.dW))
    y.backward(_nc(dy))
    r = x.grad.permute(0, 2, 3, 4, 1)
    if accumulate:
        r = r + dx
    if residual is not None:
        r = r + residual
    if relu_mask is not None:
        r = torch.where(relu_mask > 0, r, torch.zeros_like(r))
    if relu_mask_bits is not None:
        r = torch.where(_unpack_bits(relu_mask_bits, r.shape), r, torch.zeros_like(r))
    dx.copy_(_q(r, tf32_out))


def conv_wgrad(dy, x, dw, g, row_scale=None, col_mask=None):
    if g.C == 4:
        w = torch.zeros((g.Co, 3, g.kT, g.kH, g.kW), dtype=dy.dtype, requires_grad=True)
        y = F.conv3d(_nc(x)[:, :3], w, None, (g.sT, g.sH, g.sW), (g.pT, g.pH, g.pW))
        y.backward(_nc(dy))
        gw = torch.zeros_like(dw)
        gw[:, :, :, :g.kW, :3] = w.grad.permute(0, 2, 3, 4, 1)
    else:
        w = torch.zeros((g.Co, g.C, g.kT, g.kH, g.kW), dtype=dy.dtype, requires_grad=True)
        y = _conv(x, w, g)
        y.backward(_nc(dy))
        gw = w.grad.permute(0, 2, 3, 4, 1).reshape(dw.shape)
    if row_scale is not None:
        gw = gw * row_scale.view([-1] + [1] * (gw.dim() - 1))
    dw.add_(gw)


def weight_transpose(w, wt, scale=None):
    co, ci = w.shape[0], w.shape[-1]
    taps = w.numel() // (co * ci)
    s = w.reshape(co, taps, ci)
    if scale is not None:
        s = s * scale.view(-1, 1, 1)
    wt.copy_(_q(s.permute(2, 1, 0).reshape(wt.shape)))


def weight_transpose_multi(jobs, cache):
    for w, wt, s in jobs:
        weight_transpose(w, wt, s)


def _check_addressable(a, b, d):
    """Run the real wrapper's operand analysis so layout problems surface in the CPU tests."""
    from vlfb import kernels as RK
    if not RK._dim_ok(d.stride(2), d.shape[2]):
        assert RK._dim_ok(d.stride(1), d.shape[1])
        return _check_addressable(b.transpose(1, 2), a.transpose(1, 2), d.transpose(1, 2))
    RK._mat_operand(a, 1, 2)
    RK._mat_operand(b, 2, 1)


def matmul(a, b, d, alpha=1.0, accumulate=False, bias=None, tf32_out=False, tf32_optional=False):
    from vlfb import kernels as RK
    _check_addressable(a, b, d)
    Bt, M, K = a.shape
    N = b.shape[2]
    if not RK._dim_ok(d.stride(2), N):          # the wrapper computes d^T = b^T a^T
        M, N = N, M
    # as kernels.matmul: a product split over K accumulates atomically, so with tf32_optional it declines the rounding
    if tf32_out and tf32_optional and Bt * ((M + 127) // 128) * ((N + 255) // 256) <= RK.NUM_SMS // 2 and K >= 1024:
        tf32_out = False
    r = torch.bmm(a, b) * alpha
    if bias is not None:
        r = r + bias
    if accumulate:
        r = d + r
    d.copy_(_q(r, tf32_out))                    # the epilogue rounds an accumulated result too
    return bool(tf32_out)


def affine_fwd(x, s, b, y):
    y.copy_(x * s + b)


def affine_bwd(dy, s, dx):
    dx.copy_(dy * s)


def spatial_bn_fwd(x, s, b, rm, rv, sm, siv, y, eps, momentum):
    c = x.shape[-1]
    x2 = x.reshape(-1, c).double()
    m = x2.shape[0]
    mean, var = x2.mean(0), x2.var(0, unbiased=False)
    inv = 1.0 / torch.sqrt(var + eps)
    sm.copy_(mean.to(sm.dtype))
    siv.copy_(inv.to(siv.dtype))
    if rm is not None:
        rm.copy_((rm.double() * momentum + mean * (1.0 - momentum)).to(rm.dtype))
        rv.copy_((rv.double() * momentum + var * (m / max(m - 1.0, 1.0)) * (1.0 - momentum)).to(rv.dtype))
    y.copy_((((x2 - mean) * inv) * s.double() + b.double()).to(y.dtype).view(y.shape))


def spatial_bn_infer(x, s, b, rm, rv, y, eps):
    y.copy_((x - rm) * (s / torch.sqrt(rv + eps)) + b)


def spatial_bn_bwd(dy, x, s, sm, siv, dx, ds, db):
    c = x.shape[-1]
    x2, d2 = x.reshape(-1, c).double(), dy.reshape(-1, c).double()
    m = x2.shape[0]
    xh = (x2 - sm.double()) * siv.double()
    s1, s2 = d2.sum(0), (d2 * xh).sum(0)
    if ds is not None:
        ds.add_(s2.to(ds.dtype))
    if db is not None:
        db.add_(s1.to(db.dtype))
    dx.copy_(((s.double() * siv.double() / m) * (m * d2 - s1 - xh * s2)).to(dx.dtype).view(dx.shape))


def _pool_args(g):
    return (g.kT, g.kH, g.kW), (g.sT, g.sH, g.sW), (g.pT, g.pH, g.pW)


def maxpool_fwd(x, y, argmax, g):
    k, s, p = _pool_args(g)
    o, idx = F.max_pool3d(_nc(x), k, s, p, return_indices=True)
    y.copy_(o.permute(0, 2, 3, 4, 1))
    if argmax is not None:
        # F returns per-(n,c) flat THW indices; convert to global position index n*THW + idx
        n = torch.arange(g.N).view(-1, 1, 1, 1, 1) * (g.T * g.H * g.W)
        argmax.copy_((idx + n).permute(0, 2, 3, 4, 1).to(torch.int32))


def maxpool_bwd(dy, argmax, dx, g):
    c = dy.shape[-1]
    flat = dx.view(-1, c)
    idx = argmax.view(-1, c).long()
    flat.scatter_add_(0, idx, dy.reshape(-1, c))


def maxpool_bwd_gather(dy, argmax, y, dx, g, tf32_out=False):
    c = dy.shape[-1]
    d = dy.reshape(-1, c)
    if y is not None:
        d = d * (y.reshape(-1, c) > 0).to(d.dtype)
    dx.zero_()
    dx.view(-1, c).scatter_add_(0, argmax.view(-1, c).long(), d)
    if tf32_out:
        dx.copy_(_q(dx))


def avgpool_fwd(x, y, g):
    k, s, p = _pool_args(g)
    y.copy_(F.avg_pool3d(_nc(x), k, s, p).permute(0, 2, 3, 4, 1))


def avgpool_bwd(dy, dx, g, accumulate=False):
    k, s, p = _pool_args(g)
    x = torch.zeros((g.N, g.C, g.T, g.H, g.W), dtype=dy.dtype, requires_grad=True)
    F.avg_pool3d(x, k, s, p).backward(_nc(dy))
    r = x.grad.permute(0, 2, 3, 4, 1)
    if accumulate:
        dx.add_(r)
    else:
        dx.copy_(r)


# RoIAlign samples like the fp64 oracle (torchvision), in fp64 whatever the tensors' dtype: in fp32 torchvision rounds its
# sample coordinates differently from the kernel's fp32 sample table, by more than a summation bound allows.
def roi_align_fwd(feat, rois, out, spatial_scale, sampling_ratio=0):
    import torchvision
    o = torchvision.ops.roi_align(feat.permute(0, 3, 1, 2).double(), rois.double(), (out.shape[1], out.shape[2]),
                                  spatial_scale, sampling_ratio, False)
    out.copy_(o.permute(0, 2, 3, 1))


def roi_align_bwd(dout, rois, dfeat, spatial_scale, sampling_ratio=0):
    import torchvision
    f = torch.zeros(dfeat.permute(0, 3, 1, 2).shape, dtype=torch.float64, requires_grad=True)
    o = torchvision.ops.roi_align(f, rois.double(), (dout.shape[1], dout.shape[2]), spatial_scale, sampling_ratio, False)
    o.backward(dout.permute(0, 3, 1, 2).double())
    dfeat.copy_(dfeat.double() + f.grad.permute(0, 2, 3, 1))


def softmax_fwd(x, p, scale=1.0, tf32_out=False):
    p.copy_(_q(torch.softmax(x * scale, dim=-1), tf32_out))


def softmax_bwd(p, dp, dx, scale=1.0, tf32_out=False):
    dot = (p * dp).sum(-1, keepdim=True)
    dx.copy_(_q(scale * p * (dp - dot), tf32_out))


def layernorm_fwd(x, y, mean, std, cols, eps=1e-5):
    x2 = x.view(-1, cols)
    mu = x2.mean(1, keepdim=True)
    sd = torch.sqrt(((x2 - mu) ** 2).mean(1, keepdim=True) + eps)
    y.view(-1, cols).copy_((x2 - mu) / sd)
    if mean is not None:
        mean.copy_(mu.view(-1))
    if std is not None:
        std.copy_(sd.view(-1))


def layernorm_bwd(dy, y, std, dx, cols):
    d2, y2 = dy.view(-1, cols), y.view(-1, cols)
    a = d2.mean(1, keepdim=True)
    b = (d2 * y2).mean(1, keepdim=True)
    dx.view(-1, cols).copy_((d2 - a - y2 * b) / std.view(-1, 1))


def relu_fwd(x, y):
    y.copy_(torch.relu(x))


def relu_tf32(x, y):
    y.copy_(_q(torch.relu(x)))


def relu_bwd(dy, y, dx):
    dx.copy_(dy * (y > 0))


def add_relu_bwd_tf32(a, b, y, out):
    r = a + b
    if y is not None:
        r = torch.where(y > 0, r, torch.zeros_like(r))
    out.copy_(_q(r))


def relu_bwd_tf32(dy, y, dx):
    dx.copy_(_q(dy * (y > 0)))


def axpby(x, a, y, b, out):
    r = a * x
    if y is not None and b != 0.0:
        r = r + b * y
    out.copy_(r)


def add_tf32(x, y, out):
    out.copy_(_q(x + y))


def fill(x, v):
    x.fill_(v)


def round_tf32(x, y):
    if EMULATE_TF32:
        y.copy_(tf32_round(x.detach()))
    elif y.data_ptr() != x.data_ptr():
        y.copy_(x)


def colsum(x, ld, out, rows, cols, accumulate=False):
    r = x.reshape(-1)[:rows * ld].view(rows, ld)[:, :cols].sum(0)
    if accumulate:
        out.view(-1).add_(r)
    else:
        out.view(-1).copy_(r)


def sigmoid_fwd(x, y):
    y.copy_(torch.sigmoid(x))


def dropout(x, y, ratio, seed, offset, step=None):
    g = torch.Generator().manual_seed(int(seed) * 1000003 + int(offset) + (int(step.item()) << 20 if step is not None else 0))
    mask = (torch.rand(x.shape, generator=g) >= ratio).to(x.dtype)
    y.copy_(x * mask / (1.0 - ratio))


def copy2d(src, lds, dst, ldd, rows, cols, accumulate=False, src_off=0, dst_off=0):
    s = torch.as_strided(src, (rows, cols), (lds, 1), src.storage_offset() + src_off)
    d = torch.as_strided(dst, (rows, cols), (ldd, 1), dst.storage_offset() + dst_off)
    if accumulate:
        d.add_(s)
    else:
        d.copy_(s)


def nc_to_cl(src, dst, n, c, inner, cpad=None, tf32_out=False):
    cpad = cpad or c
    d = dst.view(n, inner, cpad)
    d.zero_()
    d[:, :, :c] = _q(src.reshape(n, c, inner).permute(0, 2, 1), tf32_out)


def cl_to_nc(src, dst, n, c, inner, cpad=None):
    cpad = cpad or c
    dst.view(n, c, inner).copy_(src.view(n, inner, cpad)[:, :, :c].permute(0, 2, 1))


def _sce(x, t, scale):
    from oracle import ops as O
    return O.sigmoid_cross_entropy_loss(x, t, scale)


def sigmoid_ce_fwd(logits, targets, loss, scale):
    loss.copy_(_sce(logits, targets, scale).view(1))


def sigmoid_ce_bwd(logits, targets, dloss, dlogits, scale):
    x = logits.detach().clone().requires_grad_(True)
    _sce(x, targets, scale).backward()
    g = x.grad
    if dloss is not None:
        g = g * dloss.view(())
    dlogits.copy_(g)


def softmax_ce_fwd(logits, labels, prob, loss, scale):
    from oracle import ops as O
    p, l = O.softmax_with_loss(logits, labels, scale)
    prob.copy_(p)
    loss.copy_(l.view(1))


def softmax_ce_bwd(prob, labels, dlogits, scale):
    onehot = torch.zeros_like(prob)
    onehot[torch.arange(prob.shape[0]), labels.long()] = 1.0
    dlogits.copy_((prob - onehot) * scale / prob.shape[0])


def sgd_nesterov(p, g, m, lr, momentum, wd, nesterov=True, p_tf32=None):
    lr = float(lr.view(-1)[0])
    gi = g + wd * p
    mn = momentum * m + lr * gi
    ng = (1 + momentum) * mn - momentum * m if nesterov else mn
    m.copy_(mn)
    g.copy_(ng)
    p.sub_(ng)
    if p_tf32 is not None:
        p_tf32.copy_(_q(p))


def fbo_bank_scan(bank, q, out, scale, prob=None, tf32_out=False):
    bank = bank.to(q.dtype)                      # a bf16 bank is a storage type: the arithmetic is the query's
    assert bank.is_contiguous() and q.is_contiguous() and out.is_contiguous()
    assert bank.shape[2] in (1024, 2048, 4096), 'csrc/fbo.cu supports D in {1024, 2048, 4096}'
    p = torch.softmax(torch.einsum('rld,rd->rl', bank, q) * scale, dim=1)
    if prob is not None:
        prob.copy_(p)
    out.copy_(_q(torch.einsum('rl,rld->rd', p, bank), tf32_out))


def _fbo_nl_forward(cfgd, layers, a0, bp):
    """Folded NLLayers forward (csrc/fbo.cu section 3) in torch; returns the final A and the per-layer activations."""
    A = a0
    acts = []
    for ld in layers:
        theta = A @ ld['w_theta'].t() + (ld['b_theta'] if ld.get('b_theta') is not None else 0)
        u = theta @ ld['w_phi']                                               # W_phi^T theta
        const = (theta * ld['b_phi']).sum(1, keepdim=True) if ld.get('b_phi') is not None else 0
        p = torch.softmax((torch.einsum('rd,rld->rl', u, bp) + const) * cfgd['scale'], dim=1)
        s = torch.einsum('rl,rld->rd', p, bp)
        t = s @ ld['w_g'].t() + (ld['b_g'] if ld.get('b_g') is not None else 0)
        if cfgd['pre_act_ln']:
            mean = t.mean(1, keepdim=True)
            std = torch.sqrt(((t - mean) ** 2).mean(1, keepdim=True) + cfgd.get('ln_eps', 1e-5))
            xhat = (t - mean) / std
        else:
            mean, std = torch.zeros_like(t[:, :1]), torch.ones_like(t[:, :1])
            xhat = t
        out = torch.relu(xhat) @ ld['w_out'].t() + (ld['b_out'] if ld.get('b_out') is not None else 0)
        o = out
        if cfgd.get('drop_ratio', 0.0) > 0.0:
            step = cfgd.get('step')
            g = torch.Generator().manual_seed(int(cfgd.get('seed', 0)) * 1000003 + int(ld.get('drop_offset', 0)) +
                                              (int(step.item()) << 20 if step is not None else 0))
            mask = (torch.rand(out.shape, generator=g) >= cfgd['drop_ratio']).to(out.dtype)
            o = out * mask / (1.0 - cfgd['drop_ratio'])
        A = A + o
        acts.append(dict(theta=theta, prob=p, s=s, t=t, xhat=xhat, ln_mean=mean[:, 0], ln_std=std[:, 0], out=out, a_out=A))
    return A, acts


def fbo_nl_fwd(cfgd, layers, a0, bp):
    with torch.no_grad():
        _, acts = _fbo_nl_forward(cfgd, layers, a0, bp)
    for ld, ac in zip(layers, acts):
        for k, v in ac.items():
            ld[k].copy_(v)


def fbo_nl_bwd(cfgd, layers, a0, bp, da_last, da0, dbp):
    a = a0.detach().clone().requires_grad_(True)
    b = bp.detach().clone().requires_grad_(True)
    wk = ('w_theta', 'b_theta', 'w_phi', 'b_phi', 'w_g', 'b_g', 'w_out', 'b_out')
    lay = [dict(ld, **dict((k, ld[k].detach().clone().requires_grad_(True)) for k in wk if ld.get(k) is not None))
           for ld in layers]
    A, _ = _fbo_nl_forward(cfgd, lay, a, b)
    (A * da_last).sum().backward()
    da0.copy_(a.grad)
    dbp.copy_(b.grad)
    for ld, l2 in zip(layers, lay):
        for k in wk:
            if ld.get('g' + k) is not None and l2.get(k) is not None and l2[k].grad is not None:
                ld['g' + k].add_(l2[k].grad)


def cast_bf16(x, y):
    y.copy_(x.to(torch.bfloat16))


def lfb_gather(bank, idx, out, tf32_out=False):
    assert idx.dtype == torch.int32
    flat_out = out.view(-1, out.shape[-1])
    rows = bank.view(-1, bank.shape[-1])
    i = idx.view(-1).long()
    ok = (i >= 0) & (i < rows.shape[0])
    flat_out.zero_()
    flat_out[ok] = _q(rows[i[ok]], tf32_out)


def install():
    """Route vlfb.executor / vlfb.workspace onto this module and the CPU device."""
    import sys
    from vlfb import executor
    executor.set_backend(sys.modules[__name__], 'cpu', torch.float64)


def uninstall():
    from vlfb import executor, kernels
    executor.set_backend(kernels, 'cuda', torch.float32)
