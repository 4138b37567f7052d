"""Space-time non-local block (CUDA re-implementation of the reference's
lib/models/nonlocal_helper.py; arXiv:1711.07971).

`spacetime_nonlocal` (reference :29-160) records theta/phi/g 1x1x1 convs, the 1x2x2 max pool
in front of phi/g, BatchMatMul(theta^T, phi) -> Scale(C^-1/2) -> Softmax(axis=2) ->
BatchMatMul(g, p^T), the zero-initialised output conv and its AffineNd; `add_nonlocal`
(:163-171) adds the residual; `add_nonlocal_group` (:174-213) regroups the clip into groups
of `group_size` consecutive frames.  On channels-last storage the Reshape/Transpose ops are
views, so vlfb.executor runs the block as 4 conv-GEMMs + 2 batched GEMMs + 1 softmax pass.
"""
from core.config import config as cfg


def _pointwise(model, blob_in, name, dim_in, dim_out, zero_init=False):
    """1x1x1 conv with bias (NONLOCAL.NO_BIAS) and Gaussian / zero weight init."""
    if zero_init:
        w_init = ('ConstantFill', {'value': 0.})
    else:
        w_init = ('GaussianFill', {'std': cfg.NONLOCAL.CONV_INIT_STD})
    return model.ConvNd(blob_in, name, dim_in, dim_out, [1, 1, 1], strides=[1, 1, 1], pads=[0, 0, 0] * 2,
                        weight_init=w_init, bias_init=('ConstantFill', {'value': 0.}),
                        no_bias=cfg.NONLOCAL.NO_BIAS)


def _flatten_spacetime(model, blob, batch_size, dim):
    """(B, C, T, H, W) -> (B, C, THW) with explicit batch; returns (blob, saved 5-d shape blob)."""
    target = blob if cfg.MODEL.ALLOW_INPLACE_RESHAPE else blob + '_re'
    return model.Reshape(blob, [target, blob + '_shape5d'], shape=(batch_size, dim, -1))


def spacetime_nonlocal(model, blob_in, dim_in, dim_out, batch_size, prefix, dim_inner, is_test,
                       max_pool_stride=2):
    """The non-local operator without its residual connection."""
    theta = _pointwise(model, blob_in, prefix + '_theta', dim_in, dim_inner)
    # keys / values at half spatial resolution, e.g. (8, 1024, 4, 14, 14) -> (8, 1024, 4, 7, 7)
    pooled = blob_in
    if cfg.NONLOCAL.USE_MAXPOOL is True:
        pooled = model.MaxPool(blob_in, prefix + '_pool', kernels=[1, max_pool_stride, max_pool_stride],
                               strides=[1, max_pool_stride, max_pool_stride], pads=[0, 0, 0] * 2)
    phi = _pointwise(model, pooled, prefix + '_phi', dim_in, dim_inner)
    g = _pointwise(model, pooled, prefix + '_g', dim_in, dim_inner)

    theta, theta_shape_5d = _flatten_spacetime(model, theta, batch_size, dim_inner)
    phi, _ = _flatten_spacetime(model, phi, batch_size, dim_inner)
    g, _ = _flatten_spacetime(model, g, batch_size, dim_inner)

    # (B, C, M) x (B, C, K) -> (B, M, K)
    theta_phi = model.net.BatchMatMul([theta, phi], prefix + '_affinity', trans_a=1)
    if cfg.NONLOCAL.USE_SOFTMAX is True:
        scores = theta_phi
        if cfg.NONLOCAL.USE_SCALE is True:
            scores = model.Scale(theta_phi, theta_phi, scale=dim_inner ** -.5)
        p = model.Softmax(scores, theta_phi + '_prob', engine='CUDNN', axis=2)   # rows sum to 1 over K
    else:
        # dot-product variant: divide by the number of keys (unused by the shipped configs)
        ones = model.net.ConstantFill([theta_phi], [theta_phi + '_ones'], value=1.)
        ones = model.net.ReduceBackSum([ones], [theta_phi + '_const'])
        zeros = model.net.ConstantFill([theta_phi], [theta_phi + '_zeros'], value=0.)
        denom = model.net.Add([zeros, ones], [theta_phi + '_denom'], broadcast=1, axis=0)
        model.StopGradient(denom, denom)
        p = model.net.Div([theta_phi, denom], [theta_phi + '_sc'])

    # g (B, C, K) x p^T (B, K, M) -> (B, C, M), then back to (B, C, T, H, W)
    t = model.net.BatchMatMul([g, p], prefix + '_y', trans_b=1)
    t_re, _ = model.Reshape([t, theta_shape_5d],
                            [t if cfg.MODEL.ALLOW_INPLACE_RESHAPE else t + '_re', t + '_shape3d'])

    blob_out = _pointwise(model, t_re, prefix + '_out', dim_inner, dim_out,
                          zero_init=cfg.NONLOCAL.USE_ZERO_INIT_CONV)
    if cfg.NONLOCAL.USE_BN:
        blob_out = model.SpatialBN(blob_out, prefix + '_bn', dim_out, epsilon=cfg.NONLOCAL.BN_EPSILON,
                                   momentum=cfg.NONLOCAL.BN_MOMENTUM, is_test=is_test)
        model.param_init_net.ConstantFill([prefix + '_bn_s'], prefix + '_bn_s', value=cfg.NONLOCAL.BN_INIT_GAMMA)
    if cfg.NONLOCAL.USE_AFFINE is True:
        blob_out = model.AffineNd(blob_out, prefix + '_bn', dim_out)
    return blob_out


def add_nonlocal(model, blob_in, dim_in, dim_out, batch_size, prefix, dim_inner):
    """x + NL(x)."""
    is_test = model.split in ['test', 'val']
    nl = spacetime_nonlocal(model, blob_in, dim_in, dim_out, batch_size, prefix, dim_inner, is_test)
    return model.net.Sum([blob_in, nl], prefix + '_sum')


def _swap_time_and_channels(model, blob):
    return model.Transpose(blob, blob + '_trans', axes=(0, 2, 1, 3, 4))


def add_nonlocal_group(model, blob_in, dim_in, dim_out, batch_size, pool_stride, height, width, group_size,
                       prefix, dim_inner):
    """Non-local attention inside temporal groups of `group_size` frames (batch B -> B * T/group_size)."""
    is_test = model.split in ['test', 'val']
    assert pool_stride % group_size == 0
    group_num = int(pool_stride / group_size)
    blob_in_5d = None
    if group_num > 1:
        blob_in = _swap_time_and_channels(model, blob_in)
        blob_in, blob_in_5d = model.Reshape(
            blob_in, [blob_in if cfg.MODEL.ALLOW_INPLACE_RESHAPE else blob_in + '_re', blob_in + '_shape5d'],
            shape=(batch_size * group_num, group_size, dim_in, height, width))
        blob_in = _swap_time_and_channels(model, blob_in)

    nl = spacetime_nonlocal(model, blob_in, dim_in, dim_out, batch_size * group_num, prefix, dim_inner, is_test)
    blob_out = model.net.Sum([blob_in, nl], prefix + '_sum')

    if group_num > 1:
        blob_out = _swap_time_and_channels(model, blob_out)
        blob_out, _ = model.Reshape(
            [blob_out, blob_in_5d],
            [blob_out if cfg.MODEL.ALLOW_INPLACE_RESHAPE else blob_out + '_re', blob_out + '_shape5d'])
        blob_out = _swap_time_and_channels(model, blob_out)
    return blob_out
