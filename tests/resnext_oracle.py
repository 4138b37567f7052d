"""ResNeXt-I3D support of the test oracles: Caffe2's grouped Conv (`group`) in the fp64 oracle graph, and a torch-CPU
kernel stand-in whose conv wrappers take `groups` (the CPU engine tests run a ResNeXt net through it).

The reference builds the 1x3x3 `branch2b` conv of every bottleneck with `group=cfg.RESNETS.NUM_GROUPS`
(resnet_helper.py bottleneck_transformation_3d); its weight has the Caffe2 shape [dim_out, dim_in / group, kT, kH, kW].
`GroupedGraph` is `oracle.model.Graph` with exactly that change; with NUM_GROUPS 1 it is the same graph.  `grouped()`
makes `oracle.model.param_spec / make_params / forward` build it for the duration of a `with` block, so helpers that
call the oracle module (tests/test_gpu_model.py `_train_case`) run the ResNeXt graph unchanged.
"""
import contextlib
import sys

import torch
import torch.nn.functional as F

import fake_kernels as FK
from fake_kernels import *  # noqa: F401,F403  (every other kernel of the stand-in)
from oracle import model as OM


class GroupedGraph(OM.Graph):
    def conv(self, x, name, cin, cout, kernels, strides=(1, 1, 1), pads=(0, 0, 0),
             dilations=(1, 1, 1), no_bias=1, kind='msra', round_out=True, group=1):
        if group == 1:
            return super().conv(x, name, cin, cout, kernels, strides, pads, dilations, no_bias, kind, round_out)
        w = self._p(name + '_w', (cout, cin // group) + tuple(kernels), kind)
        b = None if no_bias else self._p(name + '_b', (cout,), 'zero')
        if not self.run:
            return None
        y = F.conv3d(self.q(x), self.q(w), b, tuple(strides), tuple(pads), tuple(dilations), groups=group)
        if round_out:
            y = self.q(y)
        self.blobs[name] = y
        return y

    def conv_affine(self, x, prefix, cin, cout, kernels, strides, pads, dilations=(1, 1, 1), group=1):
        if not self.cfg.MODEL.USE_AFFINE:
            dilations = (1, 1, 1)
        y = self.conv(x, prefix, cin, cout, kernels, strides, pads, dilations, no_bias=1, round_out=False, group=group)
        return self.norm(y, prefix + '_bn', cout)

    def bottleneck(self, x, dim_in, dim_out, stride, prefix, dim_inner, tc, ts):
        """bottleneck_transformation_3d (resnet_helper.py:35-72), with branch2b's `group=NUM_GROUPS`."""
        d = self.dilations
        y = self.conv_affine(x, prefix + '_branch2a', dim_in, dim_inner, (1 + 2 * tc, 1, 1), (ts, 1, 1), (tc, 0, 0))
        y = self.relu(y)
        y = self.conv_affine(y, prefix + '_branch2b', dim_inner, dim_inner, (1, 3, 3), (1, stride, stride), (0, d, d),
                             (1, d, d), group=int(self.cfg.RESNETS.NUM_GROUPS))
        y = self.relu(y)
        return self.conv_affine(y, prefix + '_branch2c', dim_inner, dim_out, (1, 1, 1), (1, 1, 1), (0, 0, 0))


@contextlib.contextmanager
def grouped():
    """oracle.model builds GroupedGraph inside the block."""
    saved = OM.Graph
    OM.Graph = GroupedGraph
    try:
        yield OM
    finally:
        OM.Graph = saved


# ------------------------------------------------------------------------------ torch-CPU kernels with `groups`
def _grouped_w(w, g, groups):          # [Co,kT,kH,kW,Cig] -> (Co,Cig,kT,kH,kW)
    return w.view(g.Co, g.kT, g.kH, g.kW, g.C // groups).permute(0, 4, 1, 2, 3)


def _conv_g(x, w_nc, g, groups):
    return F.conv3d(FK._nc(x), w_nc, None, (g.sT, g.sH, g.sW), (g.pT, g.pH, g.pW), (g.dT, g.dH, g.dW), groups=groups)


def conv_fwd(x, w, y, g, scale=None, bias=None, residual=None, relu=False, tf32_out=False, relu_bits=None, groups=1):
    if groups <= 1:
        return FK.conv_fwd(x, w, y, g, scale, bias, residual, relu, tf32_out, relu_bits)
    o = _conv_g(x, _grouped_w(w, g, groups), g, groups).permute(0, 2, 3, 4, 1)
    if scale is not None:
        o = o * scale
    if bias is not None:
        o = o + bias
    if residual is not None:
        o = o + residual
    if relu:
        o = torch.relu(o)
    y.copy_(FK._q(o, tf32_out))
    if relu_bits is not None:
        assert relu
        relu_bits.copy_(FK.pack_sign_bits(y))


def conv_dgrad(dy, wt, dx, g, accumulate=False, residual=None, relu_mask=None, tf32_out=False, relu_mask_bits=None,
               groups=1):
    if groups <= 1:
        return FK.conv_dgrad(dy, wt, dx, g, accumulate, residual, relu_mask, tf32_out, relu_mask_bits)
    taps, cig, cog = g.kT * g.kH * g.kW, g.C // groups, g.Co // groups
    # wt [C][taps][Cog], group-major rows -> w [Co][taps][Cig]
    w = wt.reshape(groups, cig, taps, cog).permute(0, 3, 2, 1).reshape(g.Co, g.kT, g.kH, g.kW, cig)
    x = torch.zeros((g.N, g.C, g.T, g.H, g.W), dtype=dy.dtype, requires_grad=True)
    y = F.conv3d(x, w.permute(0, 4, 1, 2, 3), None, (g.sT, g.sH, g.sW), (g.pT, g.pH, g.pW), (g.dT, g.dH, g.dW),
                 groups=groups)
    y.backward(FK._nc(dy))
    r = x.grad.permute(0, 2, 3, 4, 1)
    if accumulate:
        r = r + dx
    if residual is not None:
        r = r + residual
    if relu_mask is not None:
        r = torch.where(relu_mask > 0, r, torch.zeros_like(r))
    if relu_mask_bits is not None:
        r = torch.where(FK._unpack_bits(relu_mask_bits, r.shape), r, torch.zeros_like(r))
    dx.copy_(FK._q(r, tf32_out))


def conv_wgrad(dy, x, dw, g, row_scale=None, col_mask=None, groups=1):
    if groups <= 1:
        return FK.conv_wgrad(dy, x, dw, g, row_scale, col_mask)
    w = torch.zeros((g.Co, g.C // groups, g.kT, g.kH, g.kW), dtype=dy.dtype, requires_grad=True)
    _conv_g(x, w, g, groups).backward(FK._nc(dy))
    gw = w.grad.permute(0, 2, 3, 4, 1).reshape(dw.shape)
    if row_scale is not None:
        gw = gw * row_scale.view([-1] + [1] * (gw.dim() - 1))
    dw.add_(gw)


def weight_transpose(w, wt, scale=None, groups=1):
    from vlfb.kernels import grouped_wt_slices
    for w_, wt_, s_ in grouped_wt_slices(w, wt, scale, groups):
        FK.weight_transpose(w_, wt_, s_)


def install():
    """Route vlfb.executor / vlfb.workspace onto this module (fake_kernels plus `groups`) and the CPU device."""
    from vlfb import executor
    executor.set_backend(sys.modules[__name__], 'cpu', torch.float64)


def uninstall():
    FK.uninstall()
