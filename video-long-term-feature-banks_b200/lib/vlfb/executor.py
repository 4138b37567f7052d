"""Lowers a recorded net (vlfb.net.Net) onto the sm_90a kernels and runs forward / backward /
optimizer.  Replaces the Caffe2 `dag` executor behind `workspace.RunNet`
(reference tools/train_net.py:152) for the hot path.

Representation
  * a blob is a torch tensor used as a strided *logical* view (reference NCTHW shape) over
    channels-last storage; Transpose/Reshape/Squeeze are metadata-only (so the reference's
    grouped-NL transposes, nonlocal_helper.py:191-211, and NTC_to_NCT11, lfb_helper.py:43-53,
    cost nothing), compute ops assert the layout their kernel needs;
  * Conv -> AffineNd -> [Sum] -> [Relu] chains are fused into one tensor-core GEMM with an
    epilogue (the reference runs 3-4 kernels, model_builder_video.py:211-219,
    resnet_helper.py:112-117); Scale -> Softmax likewise;
  * every tensor that feeds a tensor-core GEMM is rounded to TF32 (round-to-nearest) by its
    producer, because kind::tf32 MMAs truncate fp32 operands -- except in a B200.COMPUTE 'tf32x3' net, whose GEMMs
    multiply unrounded fp32 operands with split-TF32 products (precision=PREC_X3) and which rounds nothing.
"""
import collections
import functools
import math
import os

import torch

from . import kernels as K_default
from . import libvlfb as L
from .libvlfb import VlfbError

K = K_default          # tests may swap in a torch-CPU kernel set (tests/fake_kernels.py)
DEVICE = 'cuda'
DTYPE = torch.float32      # the CUDA kernels are fp32-only; the CPU test stand-in may run the host logic in fp64
STATS = {'fused_grad_finish': 0}
LAZY_GRAD_SUM = os.environ.get('VLFB_LAZY_GRAD_SUM', '1') != '0'   # defer residual + dgrad sums into the consumer's mask/round pass
# Fold the ReLU backward + TF32 rounding of a conv's incoming gradient (and the sum of its earlier contributions)
# into the epilogue of the dgrad GEMM that delivers the last contribution.  Exact (tests run both ways); removes 44
# streaming launches per step.  ON by default, VLFB_FUSE_GRAD_FINISH=0 disables.
FUSE_GRAD_FINISH = os.environ.get('VLFB_FUSE_GRAD_FINISH', '1') == '1'
# ... with the mask read as sign bits written by the producing conv's epilogue instead of the fp32 activation
RELU_BITS = os.environ.get('VLFB_RELU_BITS', '1') == '1'
# max-pool backward in gather form (no fill, no atomics, pool1 folds conv1's ReLU backward + rounding); '0' = the scatter
# form (zero fill + one atomic per output element + the separate ReLU-backward pass)
POOL_GATHER = int(os.environ.get('VLFB_POOL_GATHER', '1'))     # 2 = gather form only for non-overlapping windows
# the per-RoI inputs of an AVA net (model_builder_video.py), suffixed like 'proposals{sfx}': B200.ROI_CAPACITY buffers
ROI_INPUTS = ('proposals', 'labels', 'original_boxes', 'metadata', 'lfb')
COMPUTE_MODES = ('tf32', 'tf32x3')     # B200.COMPUTE values CreateNet accepts


def _mm(ctx):
    """The matmul of this net: the deterministic form in a B200.DETERMINISTIC net, split-TF32 in a 'tf32x3' net."""
    mm = K.matmul_det if ctx.net.det else K.matmul
    return functools.partial(mm, **ctx.prec) if ctx.prec else mm


def _live_kw(ctx, blob):
    """{'live_rows': device count} when `blob` is RoI-indexed in a B200.ROI_CAPACITY net, else {} (all rows)."""
    live = ctx.net.live_rows(blob)
    return {} if live is None else {'live_rows': live}


def set_backend(kernels_module, device, dtype=torch.float32):
    global K, DEVICE, DTYPE
    K = kernels_module
    DEVICE = device
    DTYPE = dtype


def empty(shape, dtype=None):
    return torch.empty(tuple(int(s) for s in shape), dtype=dtype or DTYPE, device=DEVICE)


def empty_like_strided(t):
    return torch.empty_strided(t.shape, t.stride(), dtype=t.dtype, device=t.device)


def cl_alloc(logical_shape):
    """Allocate channels-last storage for a logical (N, C, spatial...) shape; returns the logical view."""
    n, c = logical_shape[0], logical_shape[1]
    spatial = list(logical_shape[2:])
    phys = empty([n] + spatial + [c])
    return phys.permute([0, len(spatial) + 1] + list(range(1, len(spatial) + 1)))


def phys(t):
    """Physical channels-last view [N, spatial..., C] of a logical (N, C, spatial...) tensor."""
    if t.dim() <= 2:
        assert t.is_contiguous()
        return t
    p = t.permute([0] + list(range(2, t.dim())) + [1])
    if not p.is_contiguous() and t.dim() == 5 and t.shape[1] == 4 and p.stride(4) == 1 and p.stride(3) == 4:
        return p            # the fed clip: rows padded in W (workspace._feed_activation), conv1's TMA-staged operand
    assert p.is_contiguous(), 'blob is not channels-last contiguous: shape %s strides %s' % (
        tuple(t.shape), tuple(t.stride()))
    return p


def is_cl(t):
    """True when phys(t) would succeed."""
    if t.dim() <= 2:
        return t.is_contiguous()
    return t.permute([0] + list(range(2, t.dim())) + [1]).is_contiguous()


def flat(t):
    """1-D view of a dense tensor in storage order."""
    order = sorted(range(t.dim()), key=lambda d: (-t.stride(d), d))
    p = t.permute(order)
    if not p.is_contiguous():
        # size-1 dims can carry arbitrary strides; drop them
        keep = [d for d in order if t.shape[d] != 1]
        p = t.permute(keep + [d for d in order if t.shape[d] == 1])
    assert p.is_contiguous(), 'tensor is not dense: shape %s strides %s' % (tuple(t.shape), tuple(t.stride()))
    return p.reshape(-1)


def as5d(p):
    """[N, spatial..., C] physical tensor -> 5-D [N,T,H,W,C] (missing dims = 1)."""
    while p.dim() < 5:
        p = p.unsqueeze(1)
    return p


class Step(object):
    """One lowered kernel group.  fwd(ctx) computes outputs; bwd(ctx) consumes output grads."""
    params = ()

    def __init__(self, op, in_keys, out_keys):
        self.op = op
        self.in_keys = in_keys
        self.out_keys = out_keys

    def fwd(self, ctx):
        raise NotImplementedError(self.op.type)

    def bwd(self, ctx):
        raise NotImplementedError(self.op.type + ' backward')


# ======================================================================================
class Ctx(object):
    """Per-run state: blob tensors by name, gradients by (name, version) key."""

    def __init__(self, ws, net):
        self.ws = ws
        self.net = net
        self.grads = {}
        self.owned = {}
        self.saved = {}
        # gradient-finalisation fusion: `counts` = contributions each key received so far in this run;
        # net.contrib (recorded by the first run of the net) = how many it receives in total, so the LAST
        # contributor can be recognised; `final` = keys whose gradient already got its producer's ReLU mask
        # and TF32 rounding from that last contributor's GEMM epilogue.
        self.counts = {}
        self.final = set()
        self.relu_bits = {}      # conv + ReLU output key -> its sign bits (int32, 1 bit per element)
        self.grad_rounded = set()   # keys whose (single-contribution) gradient was stored TF32-rounded by its producer
        # lazy two-term sums: grads[key] (owned) + pending[key] (an alias of somebody else's gradient, e.g. the
        # residual branch).  A conv that owns `key` folds the sum into its ReLU-backward / rounding pass.
        self.pending = {}
        self.bound = {}          # blob name -> rounded flag of everything this run bound (re-installed after a graph replay)
        # B200.COMPUTE: `tf32` = GEMM operands are TF32-rounded where they are produced; False in a 'tf32x3' net, whose
        # GEMM calls all carry `prec` (precision=PREC_X3) and whose tensors are never rounded
        self.tf32 = not net.x3
        self.prec = {'precision': L.PREC_X3} if net.x3 else {}

    # ---- blobs
    def get(self, name):
        return self.ws.blobs[name]

    def put(self, name, t, rounded=False):
        self.ws.blobs[name] = t
        self.bound[name] = bool(rounded)
        if rounded:
            self.ws.rounded.add(name)
        else:
            self.ws.rounded.discard(name)

    def rounded(self, name):
        """Blob `name` as a GEMM operand: TF32-rounded (a parameter's Pt copy), or the blob itself in a 'tf32x3' net."""
        if not self.tf32:
            return self.ws.params.phys(name) if self.ws.params.has(name) else self.ws.blobs[name]
        t = self.ws.blobs[name]
        if name in self.ws.rounded or self.ws.params.has(name):
            return self.ws.params.tf32(name) if self.ws.params.has(name) else t
        r = empty_like_strided(t)
        K.round_tf32(flat(t), flat(r))
        return r

    def weight(self, name):
        """Parameter `name` as a GEMM operand: its TF32-rounded copy Pt, or the fp32 master P in a 'tf32x3' net."""
        return self.ws.params.tf32(name) if self.tf32 else self.ws.params.phys(name)

    # ---- grads
    def is_last_contribution(self, key):
        total = self.net.contrib.get(key) if self.net.contrib is not None else None
        return total is not None and self.counts.get(key, 0) == total - 1

    def set_final_grad(self, key, g):
        """The last contribution, already summed with the earlier ones, masked and rounded."""
        self.counts[key] = self.counts.get(key, 0) + 1
        self.grads[key] = g
        self.owned[key] = True
        self.final.add(key)

    def sole(self, key):
        """True when `key` receives exactly one gradient contribution (known after the first eager run) and the step
        that consumes this gradient -- the blob's producer, through views -- feeds it to GEMMs, i.e. would round it to
        TF32 anyway: the kernel that computes the gradient then stores it rounded, and the consumer's copy + rounding
        passes disappear.  (A pooling / ReLU / LayerNorm backward keeps receiving the unrounded fp32 values.)"""
        if self.net.contrib is None or self.net.det or not self.tf32:
            return False
        while True:
            if self.net.contrib.get(key) != 1:
                return False
            st = self.net.producer.get(key)
            if isinstance(st, (ReshapeStep, TransposeStep, SqueezeStep)):
                key = st.in_keys[0]
                continue
            return isinstance(st, (ConvStep, BatchMatMulStep))

    def add_grad(self, key, g, owned, rounded=False):
        if not self.net.requires.get(key, False):
            return
        assert key not in self.final, 'gradient of %s was finalised before its last contribution' % (key,)
        self.counts[key] = self.counts.get(key, 0) + 1
        cur = self.grads.get(key)
        if cur is None:
            self.grads[key] = g
            self.owned[key] = owned
            if rounded:
                self.grad_rounded.add(key)
        else:
            self.grad_rounded.discard(key)
            if self.owned[key]:
                K.axpby(flat(cur), 1.0, flat(g), 1.0, flat(cur))
            elif (LAZY_GRAD_SUM and owned and key not in self.pending and cur.shape == g.shape
                  and cur.stride() == g.stride()):
                self.pending[key] = cur          # summed when the gradient is consumed
                self.grads[key] = g
                self.owned[key] = True
            else:
                s = empty_like_strided(cur)
                K.axpby(flat(cur), 1.0, flat(g), 1.0, flat(s))
                self.grads[key] = s
                self.owned[key] = True

    def _settle(self, key):
        """Materialise a deferred two-term sum in place."""
        pend = self.pending.pop(key, None)
        if pend is not None:
            cur = self.grads[key]
            K.axpby(flat(cur), 1.0, flat(pend), 1.0, flat(cur))

    def pop_grad_finished(self, key, y):
        """Gradient of a conv output, ready to be a GEMM operand: summed, masked by the conv's ReLU (y = its
        output, or None) and TF32-rounded -- in one pass when a deferred sum is pending.  A 'tf32x3' net sums and masks
        only."""
        if not self.tf32:
            if y is None:
                return self.pop_grad(key)             # read-only operand: nothing to mask or round
            g = self.pop_grad_owned(key)
            if g is not None:
                K.relu_bwd(flat(g), flat(y), flat(g))
            return g
        pend = self.pending.pop(key, None)
        if pend is None:
            if y is None and key in self.grad_rounded:
                return self.pop_grad(key)            # complete and rounded by its producer: a read-only operand
            g = self.pop_grad_owned(key)
            if g is not None:
                if y is not None:
                    K.relu_bwd_tf32(flat(g), flat(y), flat(g))
                else:
                    K.round_tf32(flat(g), flat(g))
            return g
        self.owned.pop(key, None)
        g = self.grads.pop(key)
        K.add_relu_bwd_tf32(flat(g), flat(pend), None if y is None else flat(y), flat(g))
        return g

    def pop_grad(self, key):
        self._settle(key)
        self.owned.pop(key, None)
        self.grad_rounded.discard(key)
        return self.grads.pop(key, None)

    def pop_grad_meta(self, key):
        """(gradient, owned, rounded) for steps that pass a view of it on."""
        owned, rounded = self.owned.get(key, False), key in self.grad_rounded
        return self.pop_grad(key), owned, rounded

    def pop_grad_owned(self, key):
        """Gradient that may be modified in place."""
        self._settle(key)
        self.grad_rounded.discard(key)
        own = self.owned.pop(key, False)
        g = self.grads.pop(key, None)
        if g is not None and not own:
            c = empty_like_strided(g)
            K.axpby(flat(g), 1.0, None, 0.0, flat(c))
            g = c
        return g


# ====================================================================================== steps
def _pads3(pads, n):
    return list(pads[:n])


class ConvStep(Step):
    """Conv [+bias] [+AffineNd] [+Sum residual] [+Relu] as one gathered tensor-core GEMM."""

    def __init__(self, op, in_keys, out_keys, affine=None, residual_key=None, relu=False, out_name=None):
        Step.__init__(self, op, in_keys, out_keys)
        self.x, self.w = op.inputs[0], op.inputs[1]
        self.b = op.inputs[2] if len(op.inputs) > 2 else None
        self.affine = affine              # (scale_name, bias_name) or None
        self.res_key = residual_key
        self.relu = relu
        self.out = out_name or op.outputs[0]
        self.params = [self.w] + ([self.b] if self.b else [])
        self.round_out = True             # False: the consumer is not a GEMM (SpatialBN) and wants the fp32 sums
        self.groups = int(op.args.get('group', 1))      # Caffe2 grouped Conv (ResNeXt branch2b): csrc/gconv.cu
        self.gkw = {'groups': self.groups} if self.groups > 1 else {}     # kernel-wrapper keyword of grouped convs

    def _geom(self, ctx, xp):
        a = self.op.args
        k = list(a['kernels'])
        assert len(k) == 3
        wshape = ctx.ws.params.logical_shape(self.w)
        return K.conv_geom(xp.shape, wshape[0], k, a['strides'], _pads3(a['pads'], 3), a['dilations'])

    def fwd(self, ctx):
        x = ctx.rounded(self.x)
        xp = as5d(phys(x))
        g = self._geom(ctx, xp)
        w = ctx.weight(self.w)
        y = cl_alloc((g.N, g.Co, g.To, g.Ho, g.Wo))
        scale = bias = None
        if self.affine:
            scale = ctx.ws.params.phys(self.affine[0])
            bias = ctx.ws.params.phys(self.affine[1])
            if self.b:                      # (conv + b) * s + bb  ==  conv * s + (b * s + bb)
                eb = empty((1, g.Co))
                K.affine_fwd(ctx.ws.params.phys(self.b).view(1, -1), scale, bias, eb)
                bias = eb.view(-1)
        elif self.b:
            bias = ctx.ws.params.phys(self.b)
        res = None
        if self.res_key is not None:
            res = phys(ctx.get(self.res_key[0]))
        bits = None
        if id(self) in ctx.net.want_relu_bits and (g.Co & 31) == 0 and g.C != 4:
            # sign bits of the ReLU output: the backward mask the consumer's dgrad epilogue reads (1/32 of the bytes)
            bits = empty((y.numel() // 32,), torch.int32)
            ctx.relu_bits[self.out_keys[0]] = bits
        round_out = self.round_out and ctx.tf32
        K.conv_fwd(xp, w, phys(y), g, scale=scale, bias=bias, residual=res, relu=self.relu, tf32_out=round_out,
                   relu_bits=bits, **self.gkw, **ctx.prec)
        ctx.saved[id(self)] = (xp, g)
        ctx.put(self.out, y, rounded=round_out)

    def bwd(self, ctx):
        # the gradient is a GEMM operand of dgrad/wgrad: mask (ReLU) and round it to TF32 in one pass
        okey = self.out_keys[0]
        if okey in ctx.final:
            # masked + rounded by the dgrad GEMM that delivered the last contribution
            ctx.final.discard(okey)
            gy = ctx.pop_grad(okey)
            xp, g = ctx.saved.pop(id(self))
            gp = as5d(phys(gy))
        else:
            gy = ctx.pop_grad_finished(okey, ctx.get(self.out) if self.relu else None)
            if gy is None:
                return
            xp, g = ctx.saved.pop(id(self))
            gp = as5d(phys(gy))
        if self.res_key is not None:
            ctx.add_grad(self.res_key, gy, owned=False, rounded=ctx.tf32)       # gy is masked (+ rounded) already
        scale = ctx.ws.params.phys(self.affine[0]) if self.affine else None
        store = ctx.ws.params
        if store.trainable(self.w):
            mask = store.stem_mask() if g.C == 4 else None
            wgrad = K.conv_wgrad_det if ctx.net.det else K.conv_wgrad
            wgrad(gp, xp, store.grad(self.w), g, row_scale=scale, col_mask=mask, **self.gkw, **ctx.prec)
        if self.b and store.trainable(self.b):
            db = store.grad(self.b)
            rows = gp.numel() // g.Co
            colsum = K.colsum_det if ctx.net.det else K.colsum
            if scale is None:
                colsum(gp, g.Co, db, rows, g.Co, accumulate=True)
            else:
                t = empty((1, g.Co))
                colsum(gp, g.Co, t, rows, g.Co, accumulate=False)
                K.affine_bwd(t, scale, t)
                K.axpby(db, 1.0, t.view(-1), 1.0, db)
        xkey = self.in_keys[0]
        if ctx.net.requires.get(xkey, False):
            assert g.C != 4, 'the stem never propagates a gradient to the input clip'
            taps = g.kT * g.kH * g.kW
            wt = ctx.net.wt_buffers.get(id(self))                 # filled for all convs by one launch (_prepare_wt)
            if wt is None:
                # (a 'tf32x3' net must not get here: the unrounded transpose uploads a job table per call)
                assert ctx.tf32, 'tf32x3: dgrad weight operand of %s missing from _prepare_wt' % self.out
                wt = empty((g.C, taps, g.Co // self.groups))
                K.weight_transpose(store.phys(self.w), wt, scale, **self.gkw)     # wt = round_tf32(w * s)
            cur = ctx.grads.get(xkey)
            prod = ctx.net.producer.get(xkey)
            if (isinstance(prod, ConvStep) and ctx.is_last_contribution(xkey) and FUSE_GRAD_FINISH and not ctx.net.det
                    and (cur is None or (is_cl(cur) and as5d(phys(cur)).shape == xp.shape))):
                # Last contribution to the gradient of a conv output: sum the earlier contributions, apply that
                # conv's ReLU backward (mask = its output = our input xp) and the TF32 rounding its own
                # dgrad / wgrad GEMMs need (none in a 'tf32x3' net) -- all in this GEMM's epilogue (saves ~6 passes
                # over the tensor).
                mask = xp if prod.relu else None
                mbits = ctx.relu_bits.get(xkey) if prod.relu else None
                if mbits is not None:
                    mask = None
                ctx._settle(xkey)                 # a deferred sum must be complete before the gradient is finalised
                if cur is not None and ctx.owned.get(xkey, False):
                    dx = cur
                    K.conv_dgrad(gp, wt, as5d(phys(cur)), g, accumulate=True, relu_mask=mask, relu_mask_bits=mbits,
                                 tf32_out=ctx.tf32, **self.gkw, **ctx.prec)
                else:
                    dx = cl_alloc((g.N, g.C, g.T, g.H, g.W))
                    if dx.shape != ctx.get(self.x).shape:
                        dx = dx.view(ctx.get(self.x).shape)
                    K.conv_dgrad(gp, wt, as5d(phys(dx)), g, residual=None if cur is None else as5d(phys(cur)),
                                 relu_mask=mask, relu_mask_bits=mbits, tf32_out=ctx.tf32, **self.gkw, **ctx.prec)
                ctx.set_final_grad(xkey, dx)
                STATS['fused_grad_finish'] += 1
            elif cur is not None and ctx.owned.get(xkey, False):
                ctx.counts[xkey] = ctx.counts.get(xkey, 0) + 1
                K.conv_dgrad(gp, wt, as5d(phys(cur)), g, accumulate=True, **self.gkw, **ctx.prec)
            else:
                dx = cl_alloc((g.N, g.C, g.T, g.H, g.W))
                sole = ctx.sole(xkey)
                K.conv_dgrad(gp, wt, phys(dx), g, accumulate=False, tf32_out=sole, **self.gkw, **ctx.prec)
                ctx.add_grad(xkey, dx.view(ctx.get(self.x).shape) if dx.shape != ctx.get(self.x).shape else dx,
                             owned=True, rounded=sole)


class AffineStep(Step):
    """Stand-alone AffineNd (reference caffe2_customized_ops/video/affine_nd_op.cu:62-104)."""

    def fwd(self, ctx):
        x = ctx.get(self.op.inputs[0])
        y = empty_like_strided(x)
        s, b = ctx.ws.params.phys(self.op.inputs[1]), ctx.ws.params.phys(self.op.inputs[2])
        K.affine_fwd(phys(x), s, b, phys(y))
        ctx.put(self.op.outputs[0], y)

    def bwd(self, ctx):
        gy = ctx.pop_grad(self.out_keys[0])
        if gy is None:
            return
        dx = empty_like_strided(gy)
        K.affine_bwd(phys(gy), ctx.ws.params.phys(self.op.inputs[1]), phys(dx))
        ctx.add_grad(self.in_keys[0], dx, owned=True)


class SpatialBNStep(Step):
    """Trainable batch normalisation (Caffe2 SpatialBN as emitted by model_builder_video.py:186-190): batch statistics in
    a training net (outputs y, '_sm', '_siv'; running '_rm' / '_riv' updated in place in the ParamStore), running
    statistics in a test net.  Two streaming passes forward, two backward (csrc/bn.cu)."""

    def __init__(self, op, in_keys, out_keys):
        Step.__init__(self, op, in_keys, out_keys)
        self.x, self.s, self.b, self.rm, self.riv = op.inputs
        self.is_test = bool(op.args.get('is_test', False))
        self.eps = float(op.args.get('epsilon', 1e-5))
        self.momentum = float(op.args.get('momentum', 0.9))
        self.params = [self.s, self.b]

    def fwd(self, ctx):
        x = ctx.get(self.x)
        xp = phys(x)
        y = empty_like_strided(x)
        st = ctx.ws.params
        if self.is_test:
            K.spatial_bn_infer(xp, st.phys(self.s), st.phys(self.b), st.phys(self.rm), st.phys(self.riv), phys(y), self.eps)
        else:
            c = xp.shape[-1]
            v = ctx.net.gpus_per_step
            if v > 1:
                # B200.GPUS_PER_STEP: statistics per virtual GPU (its contiguous rows); the running statistics and the
                # '_sm' / '_siv' blobs are virtual GPU 0's, the other segments' statistics stay in this scratch
                if (xp.numel() // c) % v:
                    raise VlfbError('%s: %d rows do not split into B200.GPUS_PER_STEP = %d virtual GPUs'
                                    % (self.op.outputs[0], xp.numel() // c, v))
                sm, siv = empty((v, c)), empty((v, c))
                K.spatial_bn_seg_fwd(xp, st.phys(self.s), st.phys(self.b), st.phys(self.rm), st.phys(self.riv), sm, siv,
                                     phys(y), self.eps, self.momentum, v, det=ctx.net.det)
                ctx.put(self.op.outputs[3], sm[0])
                ctx.put(self.op.outputs[4], siv[0])
            else:
                sm, siv = empty((c,)), empty((c,))
                bn_fwd = K.spatial_bn_fwd_det if ctx.net.det else K.spatial_bn_fwd
                bn_fwd(xp, st.phys(self.s), st.phys(self.b), st.phys(self.rm), st.phys(self.riv), sm, siv, phys(y),
                       self.eps, self.momentum)
                ctx.put(self.op.outputs[3], sm)
                ctx.put(self.op.outputs[4], siv)
            ctx.saved[id(self)] = (xp, sm, siv)
        ctx.put(self.op.outputs[0], y)

    def bwd(self, ctx):
        gy = ctx.pop_grad(self.out_keys[0])
        if gy is None:
            return
        assert not self.is_test, 'a test-mode SpatialBN has no backward'
        xp, sm, siv = ctx.saved.pop(id(self))
        gp = phys(gy)
        assert gp.shape == xp.shape, 'gradient layout differs from the SpatialBN input'
        st = ctx.ws.params
        need_dx = ctx.net.requires.get(self.in_keys[0], False)
        dx = empty_like_strided(gy)
        ds = st.grad(self.s) if st.trainable(self.s) else None
        db = st.grad(self.b) if st.trainable(self.b) else None
        if sm.dim() == 2:                                   # B200.GPUS_PER_STEP: each segment's own statistics
            K.spatial_bn_seg_bwd(gp, xp, st.phys(self.s), sm, siv, phys(dx), ds, db, sm.shape[0], det=ctx.net.det)
        else:
            bn_bwd = K.spatial_bn_bwd_det if ctx.net.det else K.spatial_bn_bwd
            bn_bwd(gp, xp, st.phys(self.s), sm, siv, phys(dx), ds, db)
        if need_dx:
            ctx.add_grad(self.in_keys[0], dx, owned=True)


class ReluStep(Step):
    def fwd(self, ctx):
        x = ctx.get(self.op.inputs[0])
        y = x if self.op.outputs[0] == self.op.inputs[0] else empty_like_strided(x)
        (K.relu_tf32 if ctx.tf32 else K.relu_fwd)(flat(x), flat(y))
        ctx.put(self.op.outputs[0], y, rounded=ctx.tf32)

    def bwd(self, ctx):
        gy = ctx.pop_grad_owned(self.out_keys[0])
        if gy is None:
            return
        K.relu_bwd(flat(gy), flat(ctx.get(self.op.outputs[0])), flat(gy))
        ctx.add_grad(self.in_keys[0], gy, owned=True)


class SumStep(Step):
    def fwd(self, ctx):
        ins = [ctx.get(n) for n in self.op.inputs]
        assert len(ins) == 2 and ins[0].shape == ins[1].shape and ins[0].stride() == ins[1].stride()
        y = ins[0] if self.op.outputs[0] == self.op.inputs[0] else empty_like_strided(ins[0])
        if ctx.tf32:
            K.add_tf32(flat(ins[0]), flat(ins[1]), flat(y))
        else:
            K.axpby(flat(ins[0]), 1.0, flat(ins[1]), 1.0, flat(y))
        ctx.put(self.op.outputs[0], y, rounded=ctx.tf32)

    def bwd(self, ctx):
        gy = ctx.pop_grad(self.out_keys[0])
        if gy is None:
            return
        for k in self.in_keys:
            ctx.add_grad(k, gy, owned=False)


class ScaleStep(Step):
    def fwd(self, ctx):
        x = ctx.get(self.op.inputs[0])
        y = x if self.op.outputs[0] == self.op.inputs[0] else empty_like_strided(x)
        K.axpby(flat(x), self.op.args['scale'], None, 0.0, flat(y))
        ctx.put(self.op.outputs[0], y)

    def bwd(self, ctx):
        gy = ctx.pop_grad(self.out_keys[0])
        if gy is None:
            return
        dx = empty_like_strided(gy)
        K.axpby(flat(gy), self.op.args['scale'], None, 0.0, flat(dx))
        ctx.add_grad(self.in_keys[0], dx, owned=True)


class SoftmaxStep(Step):
    """Softmax over the last axis with an optional fused pre-scale (Scale -> Softmax chain)."""

    def __init__(self, op, in_keys, out_keys, scale=1.0, src=None):
        Step.__init__(self, op, in_keys, out_keys)
        self.scale = scale
        self.src = src or op.inputs[0]

    def fwd(self, ctx):
        x = ctx.get(self.src)
        assert x.is_contiguous() and self.op.args.get('axis', 1) == x.dim() - 1
        p = empty(x.shape)
        K.softmax_fwd(x, p, self.scale, tf32_out=ctx.tf32)
        ctx.put(self.op.outputs[0], p, rounded=ctx.tf32)

    def bwd(self, ctx):
        gp = ctx.pop_grad(self.out_keys[0])
        if gp is None:
            return
        p = ctx.get(self.op.outputs[0])
        if not gp.is_contiguous():
            gp = gp.contiguous()
        dx = empty(p.shape)
        sole = ctx.sole(self.in_keys[0])
        K.softmax_bwd(p, gp, dx, self.scale, tf32_out=sole)
        ctx.add_grad(self.in_keys[0], dx, owned=True, rounded=sole)


class PoolStep(Step):
    """MaxPool / AveragePool on channels-last storage (3-D windows; 2-D windows on 4-D blobs)."""

    def _geom(self, x):
        a = self.op.args
        k, s, p = list(a['kernels']), list(a['strides']), list(a['pads'])
        nd = len(k)
        p = p[:nd]
        k = [1] * (3 - nd) + k
        s = [1] * (3 - nd) + s
        p = [0] * (3 - nd) + p
        xp = as5d(phys(x))
        return xp, K.conv_geom(xp.shape, xp.shape[-1], k, s, p)

    def fwd(self, ctx):
        xname = self.op.inputs[0]
        x = ctx.get(xname)
        xp, g = self._geom(x)
        spatial = [g.To, g.Ho, g.Wo][5 - x.dim():]
        y = cl_alloc([g.N, g.C] + spatial)
        yp = as5d(phys(y))
        if self.op.type == 'MaxPool':
            arg = empty(yp.shape, torch.int32) if ctx.net.train else None
            K.maxpool_fwd(xp, yp, arg, g)
            ctx.saved[id(self)] = (g, arg, x.shape, x.stride(), yp)
        else:
            K.avgpool_fwd(xp, yp, g)
            ctx.saved[id(self)] = (g, None, x.shape, x.stride(), None)
        ctx.put(self.op.outputs[0], y, rounded=(self.op.type == 'MaxPool' and xname in ctx.ws.rounded))

    def bwd(self, ctx):
        gy = ctx.pop_grad(self.out_keys[0])
        if gy is None:
            return
        g, arg, xshape, xstride, yp = ctx.saved.pop(id(self))
        dx = torch.empty_strided(xshape, xstride, dtype=DTYPE, device=DEVICE)
        gp = as5d(phys(gy))
        xkey = self.in_keys[0]
        overlap = g.kT > g.sT or g.kH > g.sH or g.kW > g.sW
        # (a deterministic net always takes the gather form: the scatter form adds with atomics)
        if self.op.type == 'MaxPool' and not ctx.net.det and (POOL_GATHER == 0 or (POOL_GATHER == 2 and overlap)):
            K.fill(flat(dx), 0.0)
            K.maxpool_bwd(gp, arg, as5d(phys(dx)), g)
        elif self.op.type == 'MaxPool':
            # gather form: every dx element is written once (no zero fill, no atomics).  When the pooled blob is a
            # conv + ReLU output that nothing else reads (pool1), the ReLU backward (mask from the pool OUTPUT: the
            # winner of a window is positive iff the window's maximum is) and the TF32 rounding of the conv's wgrad
            # operand are folded in and the conv receives a finished gradient.
            prod = ctx.net.producer.get(xkey)
            fuse = (FUSE_GRAD_FINISH and not ctx.net.det and isinstance(prod, ConvStep) and prod.relu and ctx.net.contrib is not None
                    and ctx.net.contrib.get(xkey) == 1)
            K.maxpool_bwd_gather(gp, arg, yp if fuse else None, as5d(phys(dx)), g, tf32_out=fuse and ctx.tf32)
            if fuse:
                ctx.set_final_grad(xkey, dx)
                STATS['fused_grad_finish'] += 1
                return
        else:
            K.avgpool_bwd(gp, as5d(phys(dx)), g, accumulate=False)
        ctx.add_grad(xkey, dx, owned=True)


class ReshapeStep(Step):
    def fwd(self, ctx):
        x = ctx.get(self.op.inputs[0])
        if 'shape' in self.op.args:
            shape = [int(v) for v in self.op.args['shape']]
        else:
            shape = list(ctx.get(self.op.inputs[1]))
        y = x.view(shape)        # metadata only; raises if a copy would be needed
        ctx.put(self.op.outputs[0], y, rounded=self.op.inputs[0] in ctx.ws.rounded)
        if len(self.op.outputs) > 1:
            ctx.put(self.op.outputs[1], tuple(x.shape))
        ctx.saved[id(self)] = tuple(x.shape)

    def bwd(self, ctx):
        gy, owned, rounded = ctx.pop_grad_meta(self.out_keys[0])
        if gy is None:
            return
        ctx.add_grad(self.in_keys[0], gy.view(ctx.saved.pop(id(self))), owned=owned, rounded=rounded)


class TransposeStep(Step):
    def fwd(self, ctx):
        x = ctx.get(self.op.inputs[0])
        ctx.put(self.op.outputs[0], x.permute(self.op.args['axes']), rounded=self.op.inputs[0] in ctx.ws.rounded)

    def bwd(self, ctx):
        gy, _, rounded = ctx.pop_grad_meta(self.out_keys[0])
        if gy is None:
            return
        axes = self.op.args['axes']
        inv = [0] * len(axes)
        for i, a in enumerate(axes):
            inv[a] = i
        ctx.add_grad(self.in_keys[0], gy.permute(inv), owned=False, rounded=rounded)


class SqueezeStep(Step):
    def fwd(self, ctx):
        x = ctx.get(self.op.inputs[0])
        y = x
        for d in sorted(self.op.args['dims'], reverse=True):
            y = y.squeeze(d)
        ctx.put(self.op.outputs[0], y, rounded=self.op.inputs[0] in ctx.ws.rounded)
        ctx.saved[id(self)] = tuple(x.shape)

    def bwd(self, ctx):
        gy, _, rounded = ctx.pop_grad_meta(self.out_keys[0])
        if gy is None:
            return
        ctx.add_grad(self.in_keys[0], gy.view(ctx.saved.pop(id(self))), owned=False, rounded=rounded)


class StopGradientStep(Step):
    def fwd(self, ctx):
        if self.op.outputs[0] != self.op.inputs[0]:
            ctx.put(self.op.outputs[0], ctx.get(self.op.inputs[0]), rounded=self.op.inputs[0] in ctx.ws.rounded)

    def bwd(self, ctx):
        ctx.pop_grad(self.out_keys[0])


class NoopStep(Step):
    def fwd(self, ctx):
        pass

    def bwd(self, ctx):
        pass


class BatchMatMulStep(Step):
    """BatchMatMul([a, b], trans_a=, trans_b=) on strided views (nonlocal_helper.py:94-95,121)."""

    def _views(self, a, b):
        A = a.transpose(1, 2) if self.op.args.get('trans_a', 0) else a
        B = b.transpose(1, 2) if self.op.args.get('trans_b', 0) else b
        return A, B

    def fwd(self, ctx):
        a, b = ctx.rounded(self.op.inputs[0]), ctx.rounded(self.op.inputs[1])
        A, B = self._views(a, b)
        Bt, M, N = A.shape[0], A.shape[1], B.shape[2]
        if A.stride(1) == 1 and M > 1:        # rows of the output are "channels": keep channels-last
            d = empty((Bt, N, M)).transpose(1, 2)
        else:
            d = empty((Bt, M, N))
        _mm(ctx)(A, B, d, tf32_out=ctx.tf32)
        ctx.saved[id(self)] = (a, b)
        ctx.put(self.op.outputs[0], d, rounded=ctx.tf32)

    def bwd(self, ctx):
        if self.out_keys[0] in ctx.grad_rounded or not ctx.tf32:
            g = ctx.pop_grad(self.out_keys[0])       # stored rounded by its producer ('tf32x3': unrounded): read-only
            if g is None:
                return
        else:
            g = ctx.pop_grad_owned(self.out_keys[0])
            if g is None:
                return
            K.round_tf32(flat(g), flat(g))
        a, b = ctx.saved.pop(id(self))
        A, B = self._views(a, b)
        ta, tb = self.op.args.get('trans_a', 0), self.op.args.get('trans_b', 0)
        if ctx.net.requires.get(self.in_keys[0], False):
            da = empty_like_strided(a)
            dA = da.transpose(1, 2) if ta else da
            sole = _mm(ctx)(g, B.transpose(1, 2), dA, tf32_out=ctx.sole(self.in_keys[0]), tf32_optional=True)
            ctx.add_grad(self.in_keys[0], da, owned=True, rounded=sole)
        if ctx.net.requires.get(self.in_keys[1], False):
            db = empty_like_strided(b)
            dB = db.transpose(1, 2) if tb else db
            sole = _mm(ctx)(A.transpose(1, 2), g, dB, tf32_out=ctx.sole(self.in_keys[1]), tf32_optional=True)
            ctx.add_grad(self.in_keys[1], db, owned=True, rounded=sole)


class FboFoldStep(Step):
    """Inference-mode FBO-NL layer folded onto the RAW bank (csrc/fbo.cu header; SURVEY 8d "eval mode").

    Replaces Conv lfb_1x1 -> {Conv phi, Conv g} -> Reshape x2 -> BatchMatMul(theta, phi, trans_a) -> Scale ->
    Softmax -> BatchMatMul(g, p, trans_b) of lfb_helper.py:320-338,175-234 when the graph has no dropout between
    them (test / val nets) and one query per RoI:
        u = theta W_phi ; q = u W_1 ; s = sum_j softmax_j(scale q.b_j) b_j ; t = s W_1^T + c_1 ; y = t W_g^T + c_g.
    The four R-row matmuls run on the tensor-core GEMM; the bank pass is the HBM-bound kernel fbo_bank_scan.  The
    intermediate blobs of the replaced operators (lfb_1x1, *_phi, *_g, *_affinity) are not materialised;
    *_affinity_prob is (it is what visualisation code fetches).  B200.FBO_FOLD False keeps the as-written graph."""

    def __init__(self, op, in_keys, out_keys, theta, bank, w1, b1, wphi, wg, bg, scale, prob_name):
        Step.__init__(self, op, in_keys, out_keys)
        self.theta, self.bank = theta, bank
        self.w1, self.b1, self.wphi, self.wg, self.bg = w1, b1, wphi, wg, bg
        self.scale, self.prob_name = float(scale), prob_name

    def fwd(self, ctx):
        P = ctx.ws.params
        theta = ctx.rounded(self.theta)
        assert theta.dim() == 3 and theta.shape[2] == 1, 'FBO fold needs one query per RoI'
        R, d = int(theta.shape[0]), int(theta.shape[1])
        bank = phys(ctx.get(self.bank))                         # [R, L, 1, 1, D] over the fed (R, L, D) blob
        L_, D = int(bank.shape[1]), int(bank.shape[-1])
        bank = bank.reshape(R, L_, D)
        b16 = self._bf16_bank(ctx)
        if b16 is not None and tuple(b16.shape) == (R, L_, D):
            bank = b16                                          # B200.LFB_DTYPE 'bf16': half the bytes per pass
        w1 = ctx.weight(self.w1).view(1, -1, D)                 # [d1][D]
        d1 = int(w1.shape[1])
        wphi = ctx.weight(self.wphi).view(1, d, d1)             # [d][d1]
        wg = ctx.weight(self.wg).view(1, -1, d1)                # [dg][d1]
        dg = int(wg.shape[1])
        u = empty((1, R, d1))
        _mm(ctx)(flat(theta).view(1, R, d), wphi, u, tf32_out=ctx.tf32)
        q = empty((1, R, D))
        _mm(ctx)(u, w1, q)
        s = empty((R, D))
        prob = empty((R, L_)) if self.prob_name else None
        K.fbo_bank_scan(bank, q.view(R, D), s, self.scale, prob=prob, tf32_out=ctx.tf32, **_live_kw(ctx, self.theta))
        t = empty((1, R, d1))
        _mm(ctx)(s.view(1, R, D), w1.transpose(1, 2), t, bias=None if self.b1 is None else P.phys(self.b1),
                 tf32_out=ctx.tf32)
        y = empty((1, R, dg))
        _mm(ctx)(t, wg.transpose(1, 2), y, bias=None if self.bg is None else P.phys(self.bg), tf32_out=ctx.tf32)
        if prob is not None:
            ctx.put(self.prob_name, prob.view(R, 1, L_))
        ctx.put(self.op.outputs[0], y.view(R, dg, 1), rounded=ctx.tf32)

    def _bf16_bank(self, ctx):
        """The bf16 copy of the bank made when it was fed (workspace.bank_companion), found through the view chain
        (Transpose / Reshape of lfb_helper.NTC_to_NCT11) that leads from the fed blob to this step's bank input."""
        from core.config import config as cfg
        if cfg.B200.get('LFB_DTYPE', 'f32') != 'bf16':
            return None
        key = self.in_keys[1]
        for _ in range(8):
            t = ctx.ws.blobs.get(key[0] + '@bf16')
            if t is not None:
                return t
            st = ctx.net.producer.get(key)
            if not isinstance(st, (ReshapeStep, TransposeStep, SqueezeStep)):
                return None
            key = st.in_keys[0]
        return None

    def bwd(self, ctx):
        raise NotImplementedError('FboFoldStep is an inference-mode lowering')


class FboStackStep(Step):
    """Training-mode FBO-NL stack: every layer of lfb_helper.NLLayers in one launch per direction (the builder emits
    one 'FboNLStack' operator when B200.FBO_STACK is on; cnn.CNNModelHelper.FboNLStack).  phi and g are folded onto
    the shared projected bank B' (csrc/fbo.cu section 3): the as-written graph spends 4 GEMMs forward + 8 backward
    per layer on R*L = 1200 rows plus ~35 streaming launches; this step is 1 + 2 kernels whatever the layer count."""
    PARTS = ('theta', 'phi', 'g', 'out')

    def __init__(self, op, in_keys, out_keys):
        Step.__init__(self, op, in_keys, out_keys)
        a = op.args
        self.n = a['num_layers']
        names = list(op.inputs[2:])
        self.layer_params = []
        for _ in range(self.n):
            lp = {}
            for part, nb in zip(self.PARTS, a['no_bias']):
                lp['w_' + part] = names.pop(0)
                lp['b_' + part] = None if nb else names.pop(0)
            self.layer_params.append(lp)
        assert not names
        self.params = list(op.inputs[2:])

    def _cfg(self, ctx, R, L_, dropout):
        a = self.op.args
        return dict(R=R, L=L_, dA=a['dim_a'], d=a['latent_dim'], dB=a['dim_b'], scale=a['scale'], pre_act_ln=a['pre_act_ln'],
                    ln_eps=1e-5, drop_ratio=a['ratio'] if dropout else 0.0, seed=ctx.ws.rng_seed,
                    step=ctx.ws.step_tensor() if dropout else None)

    def fwd(self, ctx):
        a = self.op.args
        P = ctx.ws.params
        A = ctx.get(self.op.inputs[0])
        B = ctx.get(self.op.inputs[1])
        R, dA, d, dB = int(A.shape[0]), a['dim_a'], a['latent_dim'], a['dim_b']
        a0 = flat(A).view(R, dA)
        bp = phys(B).reshape(R, -1, dB)                       # channels-last storage of (R, dB, L, 1, 1) = [R][L][dB]
        L_ = int(bp.shape[1])
        assert L_ == a['num_feat2']
        dropout = a['ratio'] > 0.0 and ctx.ws.dropout_enabled and ctx.net.train
        layers = []
        for li, lp in enumerate(self.layer_params):
            ld = dict((k, None if n is None else P.phys(n).view(-1) if k.startswith('b_') else P.phys(n).view(P.phys(n).shape[0], -1))
                      for k, n in lp.items())
            ld.update(theta=empty((R, d)), prob=empty((R, L_)), s=empty((R, dB)), t=empty((R, d)), xhat=empty((R, d)),
                      ln_mean=empty((R,)), ln_std=empty((R,)), out=empty((R, dA)), a_out=empty((R, dA)))
            ld['drop_offset'] = ctx.ws.next_rng(R * dA)[1] if dropout else 0
            layers.append(ld)
        cfgd = self._cfg(ctx, R, L_, dropout)
        cfgd.update(_live_kw(ctx, self.op.inputs[0]))
        K.fbo_nl_fwd(cfgd, layers, a0, bp)
        outs = self.op.outputs
        for li, ld in enumerate(layers):
            th, pr, y, out, sm = outs[5 * li:5 * li + 5]
            ctx.put(th, ld['theta'].view(R, d, 1))
            ctx.put(pr, ld['prob'].view(R, 1, L_))
            ctx.put(y, ld['t'].view(R, d, 1, 1, 1))
            ctx.put(out, ld['out'].view(R, dA, 1, 1, 1))
            ctx.put(sm, ld['a_out'].view(R, dA, 1, 1, 1))
        ctx.saved[id(self)] = (cfgd, layers, a0, bp, A.shape, B.shape, B.stride())

    def bwd(self, ctx):
        for k in self.out_keys[:-1]:
            assert ctx.pop_grad(k) is None, 'only the last sum of an FBO-NL stack is consumed downstream'
        gy = ctx.pop_grad(self.out_keys[-1])
        if gy is None:
            return
        cfgd, layers, a0, bp, ashape, bshape, bstride = ctx.saved.pop(id(self))
        store = ctx.ws.params
        for ld, lp in zip(layers, self.layer_params):
            for k, n in lp.items():
                ld['g' + k] = None
                if n is not None and store.trainable(n):
                    g = store.grad(n)
                    ld['g' + k] = g.view(-1) if k.startswith('b_') else g.view(g.shape[0], -1)
        R = cfgd['R']
        da0 = empty((R, cfgd['dA']))
        dbl = torch.empty_strided(bshape, bstride, dtype=DTYPE, device=DEVICE)       # gradient of B in B's own layout
        dbp = phys(dbl).reshape(R, -1, cfgd['dB'])
        gyf = flat(gy).view(R, cfgd['dA'])
        if not gyf.is_contiguous():
            gyf = gyf.contiguous()
        K.fbo_nl_bwd(cfgd, layers, a0, bp, gyf, da0, dbp)
        ctx.add_grad(self.in_keys[0], da0.view(ashape), owned=True)
        ctx.add_grad(self.in_keys[1], dbl, owned=True)


class LayerNormStep(Step):
    def fwd(self, ctx):
        x = ctx.get(self.op.inputs[0])
        assert self.op.args.get('axis', 1) == 1
        rows = x.shape[0]
        cols = x.numel() // rows
        xf = flat(x)
        y = empty_like_strided(x)
        mean, std = empty((rows,)), empty((rows,))
        K.layernorm_fwd(xf, flat(y), mean, std, cols, self.op.args.get('epsilon', 1e-5))
        outs = self.op.outputs
        ctx.put(outs[0], y)
        if len(outs) > 1:
            ctx.put(outs[1], mean.view(rows, 1))
        if len(outs) > 2:
            ctx.put(outs[2], std.view(rows, 1))
        ctx.saved[id(self)] = (std, cols)

    def bwd(self, ctx):
        gy = ctx.pop_grad(self.out_keys[0])
        if gy is None:
            return
        std, cols = ctx.saved.pop(id(self))
        y = ctx.get(self.op.outputs[0])
        dx = empty_like_strided(y)
        K.layernorm_bwd(flat(gy), flat(y), std, flat(dx), cols)
        ctx.add_grad(self.in_keys[0], dx, owned=True)


class DropoutStep(Step):
    def fwd(self, ctx):
        x = ctx.get(self.op.inputs[0])
        ratio = self.op.args.get('ratio', 0.5)
        if self.op.args.get('is_test', False) or ratio <= 0.0 or not ctx.ws.dropout_enabled:
            ctx.put(self.op.outputs[0], x, rounded=self.op.inputs[0] in ctx.ws.rounded)
            ctx.saved[id(self)] = None
            return
        y = empty_like_strided(x)
        seed, offset = ctx.ws.next_rng(x.numel())
        K.dropout(flat(x), flat(y), ratio, seed, offset, ctx.ws.step_tensor())
        ctx.saved[id(self)] = (ratio, seed, offset)
        ctx.put(self.op.outputs[0], y)

    def bwd(self, ctx):
        gy = ctx.pop_grad(self.out_keys[0])
        if gy is None:
            return
        st = ctx.saved.pop(id(self))
        if st is None:
            ctx.add_grad(self.in_keys[0], gy, owned=False)
            return
        dx = empty_like_strided(gy)
        K.dropout(flat(gy), flat(dx), st[0], st[1], st[2], ctx.ws.step_tensor())
        ctx.add_grad(self.in_keys[0], dx, owned=True)


class FCStep(Step):
    def __init__(self, op, in_keys, out_keys):
        Step.__init__(self, op, in_keys, out_keys)
        self.params = [op.inputs[1], op.inputs[2]]

    def fwd(self, ctx):
        x = ctx.rounded(self.op.inputs[0])
        x2 = flat(x).view(x.shape[0], -1)
        w = ctx.weight(self.op.inputs[1])
        b = ctx.ws.params.phys(self.op.inputs[2])
        y = empty((x2.shape[0], w.shape[0]))
        _mm(ctx)(x2.unsqueeze(0), w.t().unsqueeze(0), y.unsqueeze(0), bias=b)
        ctx.saved[id(self)] = (x2, x.shape, x.stride())
        ctx.put(self.op.outputs[0], y)

    def bwd(self, ctx):
        gy = ctx.pop_grad_owned(self.out_keys[0]) if ctx.tf32 else ctx.pop_grad(self.out_keys[0])
        if gy is None:
            return
        if ctx.tf32:
            K.round_tf32(flat(gy), flat(gy))
        x2, xshape, xstride = ctx.saved.pop(id(self))
        store = ctx.ws.params
        wname, bname = self.op.inputs[1], self.op.inputs[2]
        if store.trainable(wname):
            _mm(ctx)(gy.t().unsqueeze(0), x2.unsqueeze(0), store.grad(wname).unsqueeze(0), accumulate=True)
        if store.trainable(bname):
            colsum = K.colsum_det if ctx.net.det else K.colsum
            colsum(gy, gy.shape[1], store.grad(bname), gy.shape[0], gy.shape[1], accumulate=True)
        if ctx.net.requires.get(self.in_keys[0], False):
            dx = torch.empty_strided(xshape, xstride, dtype=DTYPE, device=DEVICE)
            _mm(ctx)(gy.unsqueeze(0), ctx.weight(wname).unsqueeze(0), flat(dx).view(1, x2.shape[0], -1))
            ctx.add_grad(self.in_keys[0], dx, owned=True)


class ConcatStep(Step):
    def fwd(self, ctx):
        ins = [ctx.get(n) for n in self.op.inputs]
        assert self.op.args.get('axis', 1) == 1
        rows = ins[0].shape[0]
        cols = [t.numel() // rows for t in ins]
        for t, c in zip(ins, cols):
            assert t.shape[1] == c, 'Concat expects (R, C, 1, 1, 1) heads'
        total = sum(cols)
        y = cl_alloc([rows, total] + list(ins[0].shape[2:]))
        yp = flat(y)
        off = 0
        for t, c in zip(ins, cols):
            K.copy2d(flat(t), c, yp, total, rows, c, dst_off=off)
            off += c
        ctx.put(self.op.outputs[0], y)
        ctx.saved[id(self)] = (cols, [(t.shape, t.stride()) for t in ins])

    def bwd(self, ctx):
        gy = ctx.pop_grad(self.out_keys[0])
        if gy is None:
            return
        cols, metas = ctx.saved.pop(id(self))
        total = sum(cols)
        rows = gy.shape[0]
        gp = flat(gy)
        off = 0
        for key, c, (shape, stride) in zip(self.in_keys, cols, metas):
            d = torch.empty_strided(shape, stride, dtype=DTYPE, device=DEVICE)
            K.copy2d(gp, total, flat(d), c, rows, c, src_off=off)
            ctx.add_grad(key, d, owned=True)
            off += c


class RoIAlignStep(Step):
    def fwd(self, ctx):
        feat = ctx.get(self.op.inputs[0])
        rois = ctx.get(self.op.inputs[1])
        a = self.op.args
        fp = phys(feat)                               # [N,H,W,C]
        r = rois.shape[0]
        y = cl_alloc((r, feat.shape[1], a['pooled_h'], a['pooled_w']))
        live = _live_kw(ctx, self.op.inputs[1])
        K.roi_align_fwd(fp, rois, phys(y), a['spatial_scale'], a['sampling_ratio'], **live)
        ctx.put(self.op.outputs[0], y)
        ctx.saved[id(self)] = (rois, feat.shape, feat.stride(), live)

    def bwd(self, ctx):
        gy = ctx.pop_grad(self.out_keys[0])
        if gy is None:
            return
        rois, shape, stride, live = ctx.saved.pop(id(self))
        a = self.op.args
        d = torch.empty_strided(shape, stride, dtype=DTYPE, device=DEVICE)
        K.fill(flat(d), 0.0)
        roi_bwd = K.roi_align_bwd_det if ctx.net.det else K.roi_align_bwd
        roi_bwd(phys(gy), rois, phys(d), a['spatial_scale'], a['sampling_ratio'], **live)
        ctx.add_grad(self.in_keys[0], d, owned=True)


class SigmoidStep(Step):
    def fwd(self, ctx):
        x = ctx.get(self.op.inputs[0])
        y = empty_like_strided(x)
        K.sigmoid_fwd(flat(x), flat(y))
        ctx.put(self.op.outputs[0], y)

    def bwd(self, ctx):
        assert ctx.pop_grad(self.out_keys[0]) is None, 'Sigmoid(prob) is an output head without gradient'


class SigmoidCELossStep(Step):
    """B200.GPUS_PER_STEP = v > 1: the loss is the sum of the v virtual GPUs' losses, each normalised by its own count of
    targets != -1, over the row segments CompiledNet.loss_segments gives (RoI rows of an AVA net, clips otherwise)."""

    def fwd(self, ctx):
        x, t = ctx.get(self.op.inputs[0]), ctx.get(self.op.inputs[1])
        loss = empty((1,))
        seg = ctx.net.loss_segments()
        if seg is None:
            K.sigmoid_ce_fwd(x, t, loss, self.op.args['scale'])
        else:
            K.sigmoid_ce_seg_fwd(x, t, seg, loss, self.op.args['scale'])
        ctx.put(self.op.outputs[0], loss)

    def bwd(self, ctx):
        gl = ctx.pop_grad(self.out_keys[0])
        x, t = ctx.get(self.op.inputs[0]), ctx.get(self.op.inputs[1])
        dx = empty(x.shape)
        seg = ctx.net.loss_segments()
        if seg is None:
            K.sigmoid_ce_bwd(x, t, gl, dx, self.op.args['scale'])
        else:
            K.sigmoid_ce_seg_bwd(x, t, seg, gl, dx, self.op.args['scale'])
        ctx.add_grad(self.in_keys[0], dx, owned=True)


class SoftmaxCELossStep(Step):
    """B200.GPUS_PER_STEP = v: every virtual GPU has the same number of rows, so the sum of their mean losses is the
    mean over all rows times v -- the existing kernels with scale v x scale."""

    def fwd(self, ctx):
        x, t = ctx.get(self.op.inputs[0]), ctx.get(self.op.inputs[1])
        prob, loss = empty(x.shape), empty((1,))
        K.softmax_ce_fwd(x, t.view(-1), prob, loss, self.op.args['scale'] * ctx.net.gpus_per_step)
        ctx.put(self.op.outputs[0], prob)
        ctx.put(self.op.outputs[1], loss)

    def bwd(self, ctx):
        ctx.pop_grad(self.out_keys[0])
        ctx.pop_grad(self.out_keys[1])
        prob, t = ctx.get(self.op.outputs[0]), ctx.get(self.op.inputs[1])
        dx = empty(prob.shape)
        K.softmax_ce_bwd(prob, t.view(-1), dx, self.op.args['scale'] * ctx.net.gpus_per_step)
        ctx.add_grad(self.in_keys[0], dx, owned=True)


STEP_TYPES = {
    'AffineNd': AffineStep, 'Relu': ReluStep, 'Sum': SumStep, 'Scale': ScaleStep, 'Softmax': SoftmaxStep,
    'MaxPool': PoolStep, 'AveragePool': PoolStep, 'Reshape': ReshapeStep, 'Transpose': TransposeStep,
    'Squeeze': SqueezeStep, 'StopGradient': StopGradientStep, 'BatchMatMul': BatchMatMulStep,
    'LayerNorm': LayerNormStep, 'Dropout': DropoutStep, 'FC': FCStep, 'Concat': ConcatStep,
    'RoIAlign': RoIAlignStep, 'Sigmoid': SigmoidStep, 'SigmoidCrossEntropyLoss': SigmoidCELossStep,
    'SoftmaxWithLoss': SoftmaxCELossStep, 'DequeueBlobs': NoopStep, 'FboNLStack': FboStackStep,
    'SpatialBN': SpatialBNStep,
}
OPTIMIZER_OPS = ('WeightedSum', 'MomentumSGDUpdate')


# ====================================================================================== lowering
class CompiledNet(object):
    def __init__(self, model, ws):
        from core.config import config as cfg
        self.model = model
        self.ws = ws
        self.name = model.net.Proto().name
        # B200.COMPUTE, read once, when the net is created: 'tf32' rounds every GEMM operand to TF32 where it is produced;
        # 'tf32x3' rounds nothing and runs every tensor-core GEMM with split-TF32 products (precision=PREC_X3, DESIGN.md
        # 4.7).  Any other value (the reserved 'fp32' included) is refused rather than run as one of these.
        compute = cfg.B200.get('COMPUTE', 'tf32')
        if compute not in COMPUTE_MODES:
            raise VlfbError("%s: B200.COMPUTE = %r is not supported; nets lower with %s" % (
                self.name, compute, ' or '.join(repr(m) for m in COMPUTE_MODES)))
        self.compute = compute
        self.x3 = compute == 'tf32x3'
        if self.x3 and cfg.B200.get('LFB_DTYPE', 'f32') == 'bf16':
            raise VlfbError("%s: B200.COMPUTE = 'tf32x3' with B200.LFB_DTYPE = 'bf16': a bf16 feature bank would undo the "
                            "fp32 accuracy the mode computes at" % self.name)
        # read once, when the net is created.  A deterministic net also skips everything the first run's record of
        # gradient contributions (self.contrib) switches on later -- the grad-finish fusion, producer-side rounding of
        # sole gradients -- so that its first eager run computes exactly what every later run and graph replay does, and a
        # run resumed from a checkpoint in a fresh net continues the interrupted one bit for bit.
        self.det = bool(cfg.B200.get('DETERMINISTIC', False))
        self._rng_base = None        # deterministic nets: the workspace's dropout offset at the first run
        ops = [op for op in model.net.ops if op.type not in OPTIMIZER_OPS]
        self.update_ops = [op for op in model.net.ops if op.type in OPTIMIZER_OPS]
        self.losses = list(getattr(model, '_losses', []) or [])
        self.train = bool(self.losses) and bool(self.update_ops or getattr(model, '_want_grads', False))
        self._setup_iter_size(cfg)
        self._version(ops)
        self._setup_gpus_per_step(cfg, ops)
        self.steps = self._lower(ops)
        self.requires = {}
        self.trainable = []
        if self.losses:
            self._analyse()
        self.num_launch_groups = len(self.steps)
        self.producer = {}
        for st in self.steps:
            for k in st.out_keys:
                self.producer[k] = st
        # conv + ReLU outputs whose backward mask a consumer conv's dgrad epilogue may apply (grad-finish fusion): they
        # also emit their sign bits
        self.want_relu_bits = set()
        if self.train and FUSE_GRAD_FINISH and RELU_BITS and not self.det:
            for st in self.steps:
                if isinstance(st, ConvStep) and self.requires.get(st.in_keys[0], False):
                    pr = self.producer.get(st.in_keys[0])
                    if isinstance(pr, ConvStep) and pr.relu:
                        self.want_relu_bits.add(id(pr))
        self.contrib = None          # key -> number of gradient contributions, recorded by the first eager run
        self.wt_buffers = {}         # id(ConvStep) -> persistent [Ci][taps][Co] dgrad weight operand
        self._wt_jobs = None
        self._wt_cache = {}
        produced = set()
        self.external_inputs = []
        for op in ops:
            if op.type == 'DequeueBlobs':
                # the data loader's blobs are fed from outside (FeedBlob / EnqueueBlobs): they are inputs of the step,
                # and their shapes / addresses (e.g. the RoI count of an AVA batch) select the captured graph
                for n in op.outputs:
                    if n not in self.external_inputs:
                        self.external_inputs.append(n)
                continue
            for n in op.inputs:
                if n not in produced and n not in self.external_inputs and n not in model.params and \
                        n not in model.computed_params:
                    self.external_inputs.append(n)
            produced.update(op.outputs)
        self._graphs = collections.OrderedDict()     # input signature -> captured step (LRU)
        self._eager_runs = {}                        # input signature -> eager runs so far (two before capture)
        self._setup_roi_capacity(int(cfg.B200.get('ROI_CAPACITY', 0)), ops)
        self._register_inputs(ops)

    # ---- B200.ITER_SIZE (DESIGN.md 4.8)
    def _setup_iter_size(self, cfg):
        """k = B200.ITER_SIZE micro-steps per iteration for a training net with update ops (1 for every other net).  The
        k micro-batches of the NUM_GPUS = k x world_size 'virtual GPUs' of an iteration are spread over the processes."""
        k = cfg.B200.get('ITER_SIZE', 1)
        if isinstance(k, bool) or not isinstance(k, int) or k < 1:
            raise VlfbError('%s: B200.ITER_SIZE = %r; it must be an integer >= 1' % (self.name, k))
        v = cfg.B200.get('GPUS_PER_STEP', 1)
        if isinstance(v, bool) or not isinstance(v, int) or v < 1:
            raise VlfbError('%s: B200.GPUS_PER_STEP = %r; it must be an integer >= 1' % (self.name, v))
        self.iter_size = k if (self.train and self.update_ops) else 1
        self.gpus_per_step = v if (self.train and self.update_ops) else 1
        self.micro = 0                      # micro-steps of the current iteration run so far
        if self.iter_size > 1 or self.gpus_per_step > 1:
            from . import dist as vdist
            world = vdist.world_size()
            v = self.gpus_per_step
            if cfg.NUM_GPUS != v * k * world:
                if v == 1:
                    raise VlfbError('%s: B200.ITER_SIZE = %d on %d process(es) trains NUM_GPUS = %d virtual GPUs, but '
                                    'NUM_GPUS = %d' % (self.name, k, world, k * world, cfg.NUM_GPUS))
                raise VlfbError('%s: B200.GPUS_PER_STEP = %d x B200.ITER_SIZE = %d on %d process(es) trains NUM_GPUS = %d '
                                'virtual GPUs, but NUM_GPUS = %d' % (self.name, v, k, world, v * k * world, cfg.NUM_GPUS))

    # ---- B200.GPUS_PER_STEP (DESIGN.md 4.9)
    def _setup_gpus_per_step(self, cfg, ops):
        """v = self.gpus_per_step virtual GPUs of b = TRAIN.BATCH_SIZE / NUM_GPUS clips each in one packed batch.  The
        net's recorded batch must be v x b.  The sigmoid loss of an AVA net (RoIAlign on 'proposals{sfx}') is segmented by
        the RoI row offsets the workspace derives from every 'proposals' feed; any other sigmoid loss by the fixed clip
        offsets j x b."""
        v = self.gpus_per_step
        self.seg_rois, self._clip_seg = None, None
        if v == 1:
            return
        b = int(cfg.TRAIN.BATCH_SIZE / cfg.NUM_GPUS)
        rec = getattr(self.model, 'recorded_batch_size', None)
        if rec is not None and rec != v * b:
            raise VlfbError('%s: recorded with a batch of %d clips; B200.GPUS_PER_STEP = %d needs %d x %d = %d (build the '
                            'net while the setting is in force)' % (self.name, rec, v, v, b, v * b))
        rois = [op.inputs[1] for op in ops if op.type == 'RoIAlign' and op.inputs[1].startswith('proposals')]
        if rois:
            self.seg_rois = rois[0]
            if self.ws is not None:
                self.ws.gpus_per_step[self.seg_rois] = (v, b)
        else:
            self._clip_seg = torch.arange(0, v * b + 1, b, dtype=torch.int32).to(DEVICE)

    def loss_segments(self):
        """The device int32 [v + 1] row offsets of the virtual GPUs' loss rows, or None for a one-GPU step."""
        if self.gpus_per_step == 1:
            return None
        if self.seg_rois is None:
            return self._clip_seg
        return self.ws.roi_segments[self.seg_rois]

    def _check_segments(self):
        """The RoIs of this step were fed through the workspace's checks for this net's v and b."""
        ent = self.ws.seg_fed.get(self.seg_rois)
        if ent != self.ws.gpus_per_step.get(self.seg_rois):
            raise VlfbError('%s: not fed as a packed batch of B200.GPUS_PER_STEP = %d virtual GPUs (fed before net %s '
                            'was created?); feed it again' % (self.seg_rois, self.gpus_per_step, self.name))

    # ---- B200.COMPUTE of the fed inputs
    def _register_inputs(self, ops):
        """Register this net's float external inputs with the workspace under its compute mode: feeds of the names a
        'tf32x3' net reads are stored unrounded (workspace._feed_activation, DeviceLfb.feed).  A name registered by a net
        of the other mode is refused: one stored copy cannot be both TF32-rounded and unrounded."""
        targets = set(op.inputs[1] for op in ops if op.type in ('SigmoidCrossEntropyLoss', 'SoftmaxWithLoss'))
        self.float_inputs = [n for n in self.external_inputs if n not in targets]
        if self.ws is None:
            return                                            # the builder's gradient analysis (data_parallel.py)
        for n in self.float_inputs:
            other = self.ws.input_compute.get(n)
            if other is not None and other[0] != self.compute:
                raise VlfbError("%s: input %s is read by net %s with B200.COMPUTE = %r; net %s cannot read it with %r"
                                % (self.name, n, other[1], other[0], self.name, self.compute))
        for n in self.float_inputs:
            self.ws.input_compute[n] = (self.compute, self.name)

    def _check_unrounded_inputs(self):
        """A 'tf32x3' net must not read an input that was stored TF32-rounded (fed before the net was created)."""
        for n in self.float_inputs:
            if n in self.ws.rounded:
                raise VlfbError("%s: input %s holds TF32-rounded values (fed before B200.COMPUTE = 'tf32x3' net %s was "
                                "created?); feed it again" % (self.name, n, self.name))

    # ---- B200.ROI_CAPACITY (DESIGN.md 4.6)
    def _setup_roi_capacity(self, cap, ops):
        """A net with a RoIAlign on 'proposals{sfx}' is lowered at C = cap RoI rows: its per-RoI inputs are registered
        with the workspace (fed into C-row buffers, with a device live count r), and every blob computed from them along
        the leading dimension is marked RoI-indexed (the kernels that can skip padding rows get the live count; FetchBlob
        returns the r live rows)."""
        self.roi_capacity, self.roi_inputs, self.roi_sfx, self.roi_blobs = 0, [], None, set()
        rois = [op.inputs[1] for op in ops if op.type == 'RoIAlign' and op.inputs[1].startswith('proposals')]
        if cap <= 0 or not rois:
            return
        sfx = rois[0][len('proposals'):]
        for op in ops:
            if op.type == 'SoftmaxWithLoss':
                raise VlfbError('%s: B200.ROI_CAPACITY = %d on a net with SoftmaxWithLoss (%s), whose mean over rows would '
                                'count the padding rows' % (self.name, cap, op.outputs[-1]))
        names = set(p + sfx for p in ROI_INPUTS)
        self.roi_capacity, self.roi_sfx = cap, sfx
        self.roi_inputs = [n for n in self.external_inputs if n in names]
        marked = set(self.roi_inputs)
        for st in self.steps:
            if isinstance(st, (SigmoidCELossStep, SoftmaxCELossStep)):
                continue                                      # a reduction over all rows
            ins = [k[0] for k in st.in_keys] + ([st.res_key[0]] if isinstance(st, ConvStep) and st.res_key else [])
            if not any(n in marked for n in ins):
                continue
            outs = [k[0] for k in st.out_keys]
            marked.update(outs[:1] if isinstance(st, SpatialBNStep) else outs)   # not the per-channel statistics
            if isinstance(st, FboFoldStep) and st.prob_name:
                marked.add(st.prob_name)
        self.roi_blobs = marked
        self._roi_marks = dict((n, (cap, sfx)) for n in marked)
        if self.ws is None:
            return                                            # the builder's gradient analysis (data_parallel.py)
        for n in self.roi_inputs:
            self.ws.roi_capacity[n] = (cap, sfx)
        self.ws.roi_blobs.update(self._roi_marks)

    def live_rows(self, blob):
        """The device live count when `blob` is RoI-indexed in this net, else None."""
        if blob not in self.roi_blobs:
            return None
        return self.ws.roi_live[self.roi_sfx][0]

    def _check_roi_rows(self):
        """Every per-RoI input holds C rows and was fed the same number of live rows for this step."""
        ws = self.ws
        fed = {}
        for n in self.roi_inputs:
            t = ws.blobs.get(n)
            if not isinstance(t, torch.Tensor):
                continue
            if int(t.shape[0]) != self.roi_capacity or n not in ws.roi_fed:
                raise VlfbError('%s: %d rows, not a B200.ROI_CAPACITY = %d buffer (fed before net %s was created?)'
                                % (n, int(t.shape[0]), self.roi_capacity, self.name))
            fed[n] = ws.roi_fed[n]
        if len(set(fed.values())) > 1:
            raise VlfbError('per-RoI inputs of one step fed with different RoI counts: %s'
                            % ', '.join('%s %d' % kv for kv in sorted(fed.items())))

    # ---- SSA-style versioning of in-place blobs
    def _version(self, ops):
        ver = {}
        self.in_keys, self.out_keys = [], []
        self.consumers = {}
        for i, op in enumerate(ops):
            ik = [(n, ver.get(n, 0)) for n in op.inputs]
            for k in ik:
                self.consumers.setdefault(k, []).append(i)
            ok = []
            for n in op.outputs:
                ver[n] = ver.get(n, 0) + 1
                ok.append((n, ver[n]))
            self.in_keys.append(ik)
            self.out_keys.append(ok)
        self.final_ver = ver

    def _sole_consumer(self, key, ops, type_, taken=()):
        c = self.consumers.get(key, [])
        if len(c) == 1 and ops[c[0]].type == type_ and c[0] not in taken:
            return c[0]
        return None

    def _producer_index(self, key, ops):
        for i in range(len(ops)):
            if key in self.out_keys[i]:
                return i
        return None

    def _match_fbo_fold(self, ops, consumed, placed):
        """Find Conv(1x1x1 'lfb_1x1') whose consumers are the phi / g projections of single-query NL layers and
        replace each layer's bank-side operators by a FboFoldStep (test-mode graphs only: no Dropout in between)."""
        def pointwise(op):
            return op.type == 'Conv' and list(op.args.get('kernels', [])) == [1, 1, 1] and \
                list(op.args.get('strides', [1, 1, 1])) == [1, 1, 1]

        for i, c1 in enumerate(ops):
            if i in consumed or not pointwise(c1) or c1.outputs[0] in self.losses:
                continue
            # the bank-scan kernel handles rows of 1024 / 2048 / 4096 floats (csrc/fbo.cu); any other LFB_DIM keeps the
            # as-written Conv / BatchMatMul lowering, which works for every width
            if self.ws.params.has(c1.inputs[1]) and int(self.ws.params.logical_shape(c1.inputs[1])[1]) not in (1024, 2048, 4096):
                continue
            users = self.consumers.get(self.out_keys[i][0], [])
            if len(users) < 2 or len(users) % 2 or not all(pointwise(ops[j]) and j not in consumed for j in users):
                continue
            layers = []
            for j in users:                                     # phi: Conv -> Reshape -> BatchMatMul(theta, ., trans_a=1)
                jr = self._sole_consumer(self.out_keys[j][0], ops, 'Reshape', consumed)
                if jr is None:
                    continue
                jb = self._sole_consumer(self.out_keys[jr][0], ops, 'BatchMatMul', consumed)
                if jb is None or not ops[jb].args.get('trans_a', 0) or ops[jb].args.get('trans_b', 0) or \
                        self.in_keys[jb][1] != self.out_keys[jr][0]:
                    continue
                theta_key = self.in_keys[jb][0]
                tp = self._producer_index(theta_key, ops)
                if tp is None or ops[tp].type != 'Reshape' or list(ops[tp].args.get('shape', [0]))[-1] != 1:
                    continue
                key, chain, scale = self.out_keys[jb][0], [j, jr, jb], 1.0
                js = self._sole_consumer(key, ops, 'Scale', consumed)
                if js is not None:
                    scale = float(ops[js].args['scale'])
                    chain.append(js)
                    key = self.out_keys[js][0]
                jsm = self._sole_consumer(key, ops, 'Softmax', consumed)
                if jsm is None or ops[jsm].args.get('axis', 1) != 2:
                    continue
                chain.append(jsm)
                prob_key = self.out_keys[jsm][0]
                jy = self._sole_consumer(prob_key, ops, 'BatchMatMul', consumed)
                if jy is None or not ops[jy].args.get('trans_b', 0) or ops[jy].args.get('trans_a', 0) or \
                        self.in_keys[jy][1] != prob_key:
                    continue
                gr = self._producer_index(self.in_keys[jy][0], ops)          # g: Conv -> Reshape -> BatchMatMul input 0
                if gr is None or ops[gr].type != 'Reshape' or gr in consumed:
                    continue
                gc = self._producer_index(self.in_keys[gr][0], ops)
                if gc not in users or gc == j or len(self.consumers.get(self.out_keys[gc][0], [])) != 1 or \
                        len(self.consumers.get(self.out_keys[gr][0], [])) != 1:
                    continue
                layers.append((chain + [gc, gr, jy], theta_key, ops[j], ops[gc], scale, prob_key, jy))
            if 2 * len(layers) != len(users):
                continue
            consumed.add(i)
            for chain, theta_key, phi, g, scale, prob_key, jy in layers:
                consumed.update(chain)
                placed[jy] = FboFoldStep(
                    ops[jy], [theta_key, self.in_keys[i][0]], self.out_keys[jy], theta=theta_key[0], bank=c1.inputs[0],
                    w1=c1.inputs[1], b1=c1.inputs[2] if len(c1.inputs) > 2 else None, wphi=phi.inputs[1],
                    wg=g.inputs[1], bg=g.inputs[2] if len(g.inputs) > 2 else None, scale=scale, prob_name=prob_key[0])

    def _lower(self, ops):
        from core.config import config as cfg
        consumed = set()
        placed = {}                     # op index where a fused step is emitted -> step
        if not self.train and not self.losses and cfg.B200.get('FBO_FOLD', True):
            self._match_fbo_fold(ops, consumed, placed)
        for i, op in enumerate(ops):
            if i in consumed or i in placed:
                continue
            if op.type == 'Conv':
                chain = [i]
                key = self.out_keys[i][0]
                affine = None
                j = self._sole_consumer(key, ops, 'AffineNd', consumed)
                if j is not None and ops[j].inputs[0] == key[0]:
                    affine = (ops[j].inputs[1], ops[j].inputs[2])
                    chain.append(j)
                    key = self.out_keys[j][0]
                res_key = None
                j = self._sole_consumer(key, ops, 'Sum', consumed)
                if j is not None and len(ops[j].inputs) == 2 and self._safe_to_move(ops, i, j, op.inputs[0]):
                    other = [k for k in self.in_keys[j] if k != key]
                    if len(other) == 1:
                        res_key = other[0]
                        chain.append(j)
                        key = self.out_keys[j][0]
                relu = False
                j = self._sole_consumer(key, ops, 'Relu', consumed)
                if j is not None and self._safe_to_move(ops, i, j, op.inputs[0]):
                    relu = True
                    chain.append(j)
                    key = self.out_keys[j][0]
                consumed.update(chain)
                placed[chain[-1]] = ConvStep(op, self.in_keys[i], [key], affine, res_key, relu, key[0])
                if len(chain) == 1 and self._sole_consumer(key, ops, 'SpatialBN') is not None:
                    placed[i].round_out = False
            elif op.type == 'Scale':
                key = self.out_keys[i][0]
                j = self._sole_consumer(key, ops, 'Softmax', consumed)
                if j is not None:
                    consumed.update([i, j])
                    placed[j] = SoftmaxStep(ops[j], self.in_keys[i], self.out_keys[j], op.args['scale'],
                                            src=op.inputs[0])
        steps = []
        for i, op in enumerate(ops):
            if i in placed:
                steps.append(placed[i])
            elif i in consumed:
                continue
            elif op.type == 'Conv':
                steps.append(ConvStep(op, self.in_keys[i], self.out_keys[i]))
            else:
                cls = STEP_TYPES.get(op.type)
                if cls is None:
                    raise NotImplementedError('op type %s has no GPU lowering' % op.type)
                steps.append(cls(op, self.in_keys[i], self.out_keys[i]))
        return steps

    def _safe_to_move(self, ops, i, j, xname):
        """The conv at position i is executed at position j: its input must not be overwritten in between."""
        for k in range(i + 1, j + 1):
            if xname in ops[k].outputs:
                return False
        return True

    # ---- which keys need gradients / which params are trainable
    def _analyse(self):
        store_frozen = self.model.frozen_params
        loss_keys = set((n, self.final_ver.get(n, 1)) for n in self.losses)
        # backward reachability from the losses
        reach = set(loss_keys)
        for st in reversed(self.steps):
            if isinstance(st, StopGradientStep):
                continue
            if any(k in reach for k in st.out_keys):
                for k in st.in_keys:
                    reach.add(k)
                if isinstance(st, ConvStep) and st.res_key is not None:
                    reach.add(st.res_key)
        trainable = []
        for st in self.steps:
            if st.params and any(k in reach for k in st.out_keys):
                for p in st.params:
                    if p not in store_frozen and p not in trainable:
                        trainable.append(p)
        self.trainable = trainable
        # forward propagation of "requires grad"
        req = {}
        pset = set(trainable)
        for st in self.steps:
            if isinstance(st, StopGradientStep):
                for k in st.out_keys:
                    req[k] = False
                continue
            ins = list(st.in_keys) + ([st.res_key] if isinstance(st, ConvStep) and st.res_key else [])
            r = any(req.get(k, False) for k in ins) or any(p in pset for p in st.params)
            for k in st.out_keys:
                req[k] = r and (k in reach)
        self.requires = req
        self.model.param_to_grad = dict((p, p + '_grad') for p in trainable)

    # ---- execution
    def _input_key(self):
        """Shapes + addresses of every external input and the run-mode switches the lowering reads: a captured
        graph is only valid for these."""
        key = [('dropout', bool(self.ws.dropout_enabled))]
        for name in self.external_inputs:
            t = self.ws.blobs.get(name)
            if isinstance(t, torch.Tensor):
                key.append((name, tuple(t.shape), t.data_ptr()))
        return tuple(key)

    def _forward_backward(self, ctx):
        for st in self.steps:
            K.LABEL = st.out_keys[0][0] if st.out_keys else ''
            st.fwd(ctx)
        if not self.train:
            return
        if self.iter_size == 1:
            self.ws.params.begin_step(self.trainable)
        self._prepare_wt(ctx)
        red = self._reducer()
        if red is not None:
            red.begin()
        for n in self.losses:
            ctx.grads[(n, self.final_ver.get(n, 1))] = None
        for st in reversed(self.steps):
            K.LABEL = st.out_keys[0][0] if st.out_keys else ''
            if isinstance(st, (SigmoidCELossStep, SoftmaxCELossStep)):
                st.bwd(ctx)
            elif any(k in ctx.grads for k in st.out_keys):
                st.bwd(ctx)
            if red is not None:
                for pn in st.params:                   # this step's gradients are complete: their buckets may go
                    red.param_done(pn)
        if red is not None:
            red.finish()
        if self.contrib is None:
            self.contrib = dict(ctx.counts)
        else:
            assert self.contrib == ctx.counts, 'gradient contribution counts changed between runs'

    def _reducer(self):
        """The overlapped gradient all-reduce of a data-parallel training net (None: single process, or disabled)."""
        ws = self.ws
        if not (self.train and ws.allreduce is not None and getattr(ws, 'overlap_allreduce', False)):
            return None
        if self.iter_size > 1:
            return None               # only the boundary micro-step all-reduces, eagerly between the two graphs
        from core.config import config as cfg
        if not cfg.B200.get('OVERLAP_ALLREDUCE', True):
            return None
        if ws.reducer is None or ws.reducer.store is not ws.params or len(ws.reducer.store.chunks) != len(ws.params.chunks):
            from . import dist as vdist
            ws.params._ensure_state()
            ws.reducer = vdist.GradReducer(ws.params)
        return ws.reducer

    def _prepare_wt(self, ctx):
        """Transposed, affine-scaled, TF32-rounded ('tf32x3': unrounded) weights of every conv whose input needs a gradient: persistent
        buffers (static addresses -> one device job table) filled by ONE launch per step instead of one per conv."""
        if self._wt_jobs is None:
            store = self.ws.params
            jobs = []
            for st in self.steps:
                if isinstance(st, ConvStep) and self.requires.get(st.in_keys[0], False) and \
                        any(self.requires.get(k, False) for k in st.out_keys):
                    w = store.phys(st.w)
                    co, ci = w.shape[0], w.shape[-1]
                    if ci == 4 and st.groups == 1:
                        continue                                # the stem never propagates a gradient
                    taps = w.numel() // (co * ci)
                    wt = empty((ci * st.groups, taps, co // st.groups))      # grouped: [C][taps][Cog], one job per group
                    self.wt_buffers[id(st)] = wt
                    jobs.extend(K_default.grouped_wt_slices(w, wt, store.phys(st.affine[0]) if st.affine else None, st.groups))
            self._wt_jobs = jobs
        if self._wt_jobs:
            K.weight_transpose_multi(self._wt_jobs, self._wt_cache, **ctx.prec)

    MAX_GRAPHS = 4          # captured steps kept per net (each owns its activation memory): LRU over input signatures

    def run(self):
        """One pass.  Eager for the first runs of a given input signature; after that the whole
        step (forward + backward [+ SGD]) is replayed from a captured CUDA graph, which removes the
        per-launch host cost of the ~600 kernels of a step.  The gradient all-reduce (N > 1) stays
        eager between the two captured halves.  Graphs are cached per input signature (e.g. per RoI count).
        B200.ITER_SIZE = k > 1: the pass is one micro-step; only the k-th of an iteration all-reduces and updates."""
        from core.config import config as cfg
        ws = self.ws
        if self.roi_capacity:
            self._check_roi_rows()
            ws.roi_blobs.update(self._roi_marks)        # names shared with another net (train / test) are this net's now
        if self.x3:
            self._check_unrounded_inputs()
        if self.seg_rois is not None:
            self._check_segments()
        ws.begin_run()
        if self.det:
            # every run draws the dropout offsets its first run drew, as a graph replay does (the step counter varies
            # the masks), so the masks of a step depend on the step counter only, not on how many eager runs preceded
            if self._rng_base is None:
                self._rng_base = ws.rng_offset
            ws.rng_offset = self._rng_base
        boundary = self._micro_step()
        use_graph = (DEVICE != 'cpu' and cfg.B200.CUDA_GRAPH and not ws.force_eager and K is K_default)
        key = self._input_key() if use_graph else None
        if use_graph:
            entry = self._graphs.get(key)
            if entry is not None:
                self._graphs.move_to_end(key)
                return self._replay(entry, boundary)
            if self._eager_runs.get(key, 0) >= 2:
                entry = self._capture()
                self._graphs[key] = entry
                while len(self._graphs) > self.MAX_GRAPHS:
                    self._graphs.popitem(last=False)
                return self._replay(entry, boundary)
            self._eager_runs[key] = self._eager_runs.get(key, 0) + 1
            while len(self._eager_runs) > 4 * self.MAX_GRAPHS:
                self._eager_runs.pop(next(iter(self._eager_runs)))
        ctx = Ctx(ws, self)
        self._forward_backward(ctx)
        if not self.train or not boundary:
            return
        if ws.allreduce is not None and self._reducer() is None:
            ws.allreduce(ws.params)
        if self.update_ops:
            self._update(ws.params)

    def _micro_step(self):
        """B200.ITER_SIZE = k > 1: before micro-step 0 of an iteration, zero the gradients (a few fills, eager, outside
        any captured graph, whose backward then only adds into them) and hold the parameter store for this net until the
        boundary.  Returns True when this run ends an iteration (always for k = 1)."""
        if self.iter_size == 1:
            return True
        ws = self.ws
        if self.micro == 0:
            ws.params.begin_step(self.trainable)
            ws.open_iteration = self
        self.micro += 1
        if self.micro < self.iter_size:
            return False
        self.micro = 0
        ws.open_iteration = None
        return True

    def _capture(self):
        """Capture the step for the current input signature.  Returns (g1, g2, n1, n2, written, rounded, split):
        `written` = every blob the captured run bound (tensors and shape tuples), `rounded` = which of them are
        TF32-rounded; both are re-installed after every replay, because ws.blobs is shared by all nets and an eager run
        of another net (or of this one with another signature) rebinds the same names in between.  Data parallel: with
        the all-reduce overlapped (stream-ordered NCCL issued inside backward, vlfb.dist.GradReducer) the whole step
        is ONE graph; otherwise (`split`) two graphs with the eager all-reduce between them."""
        ws = self.ws
        torch.cuda.synchronize()
        if self._reducer() is not None:
            try:
                return self._capture_graphs(False)
            except Exception as exc:                                  # e.g. a NCCL build that cannot be captured
                import sys
                sys.stderr.write('vlfb: capturing the overlapped all-reduce failed (%r); falling back to the split step\n' % (exc,))
                ws.overlap_allreduce = False
                torch.cuda.synchronize()
        return self._capture_graphs(self.train and (ws.allreduce is not None or self.iter_size > 1))

    def _capture_graphs(self, split):
        ws = self.ws
        n0 = K.LAUNCHES
        g1 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g1):
            ctx = Ctx(ws, self)
            self._forward_backward(ctx)
            if self.train and self.update_ops and not split:
                self._update(ws.params)
        n1 = K.LAUNCHES - n0
        g2, n2 = None, 0
        if split and self.update_ops:
            g2 = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g2):
                self._update(ws.params)
            n2 = K.LAUNCHES - n0 - n1
        K.LAUNCHES = n0
        written = dict((k, ws.blobs[k]) for k in ctx.bound)
        rounded = set(k for k, r in ctx.bound.items() if r)
        return (g1, g2, n1, n2, written, rounded, split)

    def _replay(self, entry, boundary=True):
        """Replay a captured step; a non-boundary micro-step (B200.ITER_SIZE > 1) replays the forward + backward only."""
        g1, g2, n1, n2, written, rounded, split = entry
        ws = self.ws
        g1.replay()
        K.LAUNCHES += n1
        if boundary:
            if split and ws.allreduce is not None:
                ws.allreduce(ws.params)
            if g2 is not None:
                g2.replay()
                K.LAUNCHES += n2
        ws.blobs.update(written)
        ws.rounded.difference_update(written)
        ws.rounded.update(rounded)

    def _update(self, store):
        from core.config import config as cfg
        lr = self.ws.blobs['lr']
        wd_map = {}
        for op in self.update_ops:
            if op.type == 'WeightedSum':
                wd_map[op.inputs[2]] = op.inputs[3]
        mom = nesterov = None
        for op in self.update_ops:
            if op.type == 'MomentumSGDUpdate':
                mom, nesterov = op.args.get('momentum', 0.9), op.args.get('nesterov', 1)
        wd_val = {'weight_decay': cfg.SOLVER.WEIGHT_DECAY, 'weight_decay_bn': cfg.SOLVER.WEIGHT_DECAY_BN}
        store.sgd(self.trainable, lr, mom, bool(nesterov),
                  dict((p, wd_val.get(wd_map.get(p, 'weight_decay'), 0.0)) for p in self.trainable))
