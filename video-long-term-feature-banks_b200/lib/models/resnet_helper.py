"""Residual stages (CUDA re-implementation of the reference's lib/models/resnet_helper.py).

Signatures, blob names and semantics follow the reference (bottleneck :35-72, shortcut :75-89,
residual block :92-119, stages :122-194): temporal conv in branch2a, stride/dilation on the
1x3x3 branch2b, in-place Sum + ReLU into `{prefix}_branch2c_bn`.  vlfb.executor fuses each
conv -> affine -> (sum) -> relu chain into a single tensor-core GEMM epilogue.
"""
import logging

import numpy as np

from core.config import config as cfg
import models.nonlocal_helper as nonlocal_helper

logger = logging.getLogger(__name__)


def _conv_op(model):
    return model.Conv3dAffine if cfg.MODEL.USE_AFFINE else model.Conv3dBN


def bottleneck_transformation_3d(model, blob_in, dim_in, dim_out, stride, prefix, dim_inner, group=1,
                                 use_temp_conv=1, temp_stride=1):
    """(1+2tc)x1x1 -> 1x3x3 (stride, dilation) -> 1x1x1; the last conv has no ReLU."""
    conv = _conv_op(model)
    dil = cfg.DILATIONS
    a = conv(blob_in, prefix + '_branch2a', dim_in, dim_inner, [1 + 2 * use_temp_conv, 1, 1],
             strides=[temp_stride, 1, 1], pads=[use_temp_conv, 0, 0] * 2, inplace_affine=False)
    a = model.Relu_(a)
    b = conv(a, prefix + '_branch2b', dim_inner, dim_inner, [1, 3, 3], strides=[1, stride, stride],
             pads=[0, dil, dil] * 2, group=group, inplace_affine=False, dilations=[1, dil, dil])
    logger.info('%s using dilation %d', prefix, dil)
    b = model.Relu_(b)
    return conv(b, prefix + '_branch2c', dim_inner, dim_out, [1, 1, 1], strides=[1, 1, 1], pads=[0, 0, 0] * 2,
                inplace_affine=False, bn_init=cfg.MODEL.BN_INIT_GAMMA)


def _add_shortcut_3d(model, blob_in, prefix, dim_in, dim_out, stride, temp_stride=1):
    """Type-B shortcut: identity when shapes agree, else a strided 1x1x1 projection."""
    if dim_in == dim_out and temp_stride == 1 and stride == 1:
        return blob_in
    return _conv_op(model)(blob_in, prefix, dim_in, dim_out, [1, 1, 1], strides=[temp_stride, stride, stride],
                           pads=[0, 0, 0] * 2, group=1, inplace_affine=False)


def _generic_residual_block_3d(model, blob_in, dim_in, dim_out, stride, prefix, dim_inner, group=1,
                               use_temp_conv=0, temp_stride=1, trans_func=None):
    """relu(F(x) + shortcut(x)); the sum is written in place into F's output blob."""
    if trans_func is None:
        trans_func = globals()[cfg.RESNETS.TRANS_FUNC]
    transformed = trans_func(model, blob_in, dim_in, dim_out, stride, prefix, dim_inner, group=group,
                             use_temp_conv=use_temp_conv, temp_stride=temp_stride)
    shortcut = _add_shortcut_3d(model, blob_in, prefix + '_branch1', dim_in, dim_out, stride,
                                temp_stride=temp_stride)
    out_name = transformed if cfg.MODEL.ALLOW_INPLACE_SUM else prefix + '_sum'
    summed = model.net.Sum([transformed, shortcut], out_name)
    return model.Relu_(summed)


def _pad_schedules(num_blocks, use_temp_convs, temp_strides):
    tc = list(use_temp_convs) if use_temp_convs is not None else list(np.zeros(num_blocks).astype(int))
    ts = list(temp_strides) if temp_strides is not None else list(np.ones(num_blocks).astype(int))
    while len(tc) < num_blocks:
        tc.append(0)
        ts.append(1)
    return tc, ts


def _stage(model, blob_in, dim_in, dim_out, stride, num_blocks, prefix, dim_inner, group, use_temp_convs,
           temp_strides, add_nl, nonlocal_mod):
    tc, ts = _pad_schedules(num_blocks, use_temp_convs, temp_strides)
    for idx in range(num_blocks):
        blob_in = _generic_residual_block_3d(
            model, blob_in, dim_in, dim_out, 2 if (idx == 0 and stride == 2) else 1,
            '{}_{}'.format(prefix, idx), dim_inner, group, tc[idx], ts[idx])
        dim_in = dim_out
        if idx % nonlocal_mod == nonlocal_mod - 1:
            blob_in = add_nl(blob_in, dim_in, idx)
    return blob_in, dim_in


def res_stage_nonlocal(model, block_fn, blob_in, dim_in, dim_out, stride, num_blocks, prefix, dim_inner=None,
                       group=None, use_temp_convs=None, temp_strides=None, batch_size=None, nonlocal_name=None,
                       nonlocal_mod=1000):
    """A ResNet stage with an optional NL block after every `nonlocal_mod`-th residual block."""
    def add_nl(blob, dim, idx):
        return nonlocal_helper.add_nonlocal(model, blob, dim, dim, batch_size,
                                            nonlocal_name + '_{}'.format(idx), int(dim / 2))
    return _stage(model, blob_in, dim_in, dim_out, stride, num_blocks, prefix, dim_inner, group, use_temp_convs,
                  temp_strides, add_nl, nonlocal_mod)


def res_stage_nonlocal_group(model, block_fn, blob_in, dim_in, dim_out, stride, num_blocks, prefix, dim_inner=None,
                             group=None, use_temp_convs=None, temp_strides=None, batch_size=None, pool_stride=None,
                             spatial_dim=None, group_size=None, nonlocal_name=None, nonlocal_mod=1000):
    """Like res_stage_nonlocal, with the NL blocks restricted to groups of `group_size` frames."""
    def add_nl(blob, dim, idx):
        return nonlocal_helper.add_nonlocal_group(model, blob, dim, dim, batch_size, pool_stride, spatial_dim,
                                                  spatial_dim, group_size, nonlocal_name + '_{}'.format(idx),
                                                  int(dim / 2))
    return _stage(model, blob_in, dim_in, dim_out, stride, num_blocks, prefix, dim_inner, group, use_temp_convs,
                  temp_strides, add_nl, nonlocal_mod)
