"""Feature-bank operators (CUDA re-implementation of the reference's lib/models/lfb_helper.py).

FBO-NL (`add_fbo_nl_head`, reference :78-103): the RoI / clip feature A attends over the L
long-term bank features B with `FBO_NL.NUM_LAYERS` stacked single-query non-local layers
(`NLLayers` :266-292, `NLCore` :170-263); the projected bank is shared by all layers.
FBO-Avg / FBO-Max (:106-127) pool the bank.  `RoIFeatureTransform` (:130-152) wraps the legacy
RoIAlign.  The NTC -> NCT11 transposes (:43-53) are free views on channels-last storage.
"""
import logging
import os

from core.config import config as cfg

logger = logging.getLogger(__name__)

# The reference captures these at import time, i.e. before any YAML is merged (SURVEY.md
# section 5): theta/phi/g always use the default std / bias settings, `out` is zero-initialised.
init_params1 = {
    'weight_init': ('GaussianFill', {'std': cfg.NONLOCAL.CONV_INIT_STD}),
    'bias_init': ('ConstantFill', {'value': 0.}),
    'no_bias': cfg.NONLOCAL.NO_BIAS}
init_params2 = {
    'weight_init': ('ConstantFill', {'value': 0.}),
    'bias_init': ('ConstantFill', {'value': 0.}),
    'no_bias': cfg.NONLOCAL.NO_BIAS}

_UNIT = dict(strides=[1, 1, 1], pads=[0, 0, 0] * 2)


def NTC_to_NCT11(model, blob_in, dim, num_feat, name=''):
    """(N, T, C) bank -> (N, C, T, 1, 1) so that 1x1x1 convs act as per-feature linear layers."""
    blob_in = model.Transpose(blob_in, blob_in + '_tr' + name, axes=(0, 2, 1))
    blob_in, _ = model.Reshape(blob_in, [blob_in + '_rs' + name, blob_in + '_rs_shape' + name],
                               shape=(-1, dim, num_feat, 1, 1))
    return blob_in


def add_fbo_head(model, blob_in, dim_in, num_lfb_feat, test_mode, suffix):
    """Dispatch on LFB.FBO_TYPE."""
    kind = cfg.LFB.FBO_TYPE
    if kind == 'avg':
        return add_fbo_avg_head(model, num_lfb_feat, 'fbo_avg_out', suffix)
    if kind == 'max':
        return add_fbo_max_head(model, num_lfb_feat, 'fbo_max_out', suffix)
    if kind == 'nl':
        return add_fbo_nl_head(model, blob_in, dim_in=dim_in, num_lfb_feat=num_lfb_feat, test_mode=test_mode,
                               suffix=suffix)
    raise NotImplementedError


def add_fbo_nl_head(model, blob_in, dim_in, num_lfb_feat, test_mode, suffix):
    """ "Non-local" feature bank operator: returns (blob (N, C, 1, 1, 1), C)."""
    query, query_dim = prepare_nl_input(model, blob_in, dim_in, '_fbonl', test_mode)
    bank = get_lfb_blob(model, num_lfb_feat, suffix)
    bank, bank_dim = prepare_lfb(model, bank, test_mode, suffix)
    out = NLLayers(model, A=query, B=bank, in_dim1=query_dim, in_dim2=bank_dim,
                   latent_dim=cfg.FBO_NL.LATENT_DIM, num_feat1=1, num_feat2=num_lfb_feat, prefix='lfb',
                   test_mode=test_mode)
    return out, query_dim


def _pool_bank(model, pool, num_lfb_feat, out_name, suffix):
    bank = get_lfb_blob(model, num_lfb_feat, suffix)               # (N, lfb_dim, L, 1, 1)
    return pool(bank, out_name, kernels=[num_lfb_feat, 1, 1], strides=[1, 1, 1],
                pads=[0, 0, 0] * 2), cfg.LFB.LFB_DIM


def add_fbo_avg_head(model, num_lfb_feat, out_name, suffix):
    """ "Avg pooling" feature bank operator."""
    return _pool_bank(model, model.AveragePool, num_lfb_feat, out_name, suffix)


def add_fbo_max_head(model, num_lfb_feat, out_name, suffix):
    """ "Max pooling" feature bank operator."""
    return _pool_bank(model, model.MaxPool, num_lfb_feat, out_name, suffix)


def RoIFeatureTransform(model, blobs_in, blob_out, blob_rois='proposals', resolution=7, spatial_scale=1. / 16.,
                        sampling_ratio=0):
    """RoIAlign (legacy Caffe2 semantics) of `blobs_in` at the boxes `blob_rois`."""
    xform_out = model.RoIAlign([blobs_in, blob_rois], [blob_out], pooled_w=resolution, pooled_h=resolution,
                               spatial_scale=spatial_scale, sampling_ratio=sampling_ratio)
    return xform_out[0] if isinstance(xform_out, tuple) else xform_out


def get_lfb_blob(model, num_lfb_feat, suffix):
    return NTC_to_NCT11(model, 'lfb{}'.format(suffix), cfg.LFB.LFB_DIM, num_lfb_feat)


def pre_act(model, x):
    """Pre-activation non-linearity: LayerNorm (no affine) then ReLU."""
    if cfg.FBO_NL.PRE_ACT_LN:
        x = model.LayerNorm(x, [x + '_ln', x + '_ln_mean', x + '_ln_std'])[0]
    return model.Relu(x, x + '_relu')


def _linear(model, blob, name, dim_in, dim_out, init):
    return model.ConvNd(blob, name, dim_in, dim_out, [1, 1, 1], **dict(_UNIT, **init))


def NLCore(model, in_blob1, in_blob2, in_dim1, in_dim2, latent_dim, num_feat1, num_feat2, prefix, test_mode):
    """One non-local layer: softmax(theta(A)^T phi(B) / sqrt(d)) applied to g(B), then out()."""
    theta = _linear(model, in_blob1, prefix + '_theta', in_dim1, latent_dim, init_params1)
    phi = _linear(model, in_blob2, prefix + '_phi', in_dim2, latent_dim, init_params1)
    g = _linear(model, in_blob2, prefix + '_g', in_dim2, latent_dim, init_params1)

    inplace = cfg.MODEL.ALLOW_INPLACE_RESHAPE
    theta, theta_shape_5d = model.Reshape(theta, [theta if inplace else theta + '_re', theta + '_shape5d'],
                                          shape=(-1, latent_dim, num_feat1))
    phi, _ = model.Reshape(phi, [phi if inplace else phi + '_re', phi + '_shape5d'],
                           shape=(-1, latent_dim, num_feat2))
    g, _ = model.Reshape(g, [g + '_re', g + '_shape5d'], shape=(-1, latent_dim, num_feat2))

    # (N, C, F1) x (N, C, F2) -> (N, F1, F2)
    theta_phi = model.net.BatchMatMul([theta, phi], prefix + '_affinity', trans_a=1)
    if cfg.FBO_NL.SCALE:
        theta_phi = model.Scale(theta_phi, theta_phi, scale=latent_dim ** -.5)
    p = model.Softmax(theta_phi, theta_phi + '_prob', engine='CUDNN', axis=2)
    # (N, C, F2) x (N, F1, F2)^T -> (N, C, F1)
    t = model.net.BatchMatMul([g, p], prefix + '_y', trans_b=1)
    blob_out, _ = model.Reshape([t, theta_shape_5d], [t if inplace else t + '_re', t + '_shape3d'])

    if cfg.FBO_NL.PRE_ACT:
        blob_out = pre_act(model, blob_out)
    blob_out = _linear(model, blob_out, prefix + '_out', latent_dim, in_dim1, init_params2)
    if not cfg.FBO_NL.PRE_ACT:
        blob_out = model.LayerNorm(blob_out, [prefix + '_ln', prefix + '_ln_mean', prefix + '_ln_std'])[0]
    if cfg.FBO_NL.LFB_DROPOUT_ON and not test_mode:
        blob_out = model.Dropout(blob_out, blob_out + '_drop', ratio=cfg.FBO_NL.DROPOUT_RATE, is_test=False)
    return blob_out


def NLLayers(model, A, B, in_dim1, in_dim2, latent_dim, num_feat1, num_feat2, prefix, test_mode):
    """Stack FBO_NL.NUM_LAYERS residual NL layers; only A is updated between layers."""
    if (cfg.B200.get('FBO_STACK', True) and os.environ.get('VLFB_FBO_STACK', '1') != '0' and not test_mode and num_feat1 == 1 and cfg.FBO_NL.PRE_ACT
            and cfg.FBO_NL.NUM_LAYERS <= 4 and in_dim2 == latent_dim):
        # training graphs, one query per RoI: all layers in one launch per direction, phi / g folded onto the shared
        # projected bank (same parameters, same output blobs; B200.FBO_STACK False keeps the as-written operators)
        drop = cfg.FBO_NL.DROPOUT_RATE if cfg.FBO_NL.LFB_DROPOUT_ON else 0.0
        return model.FboNLStack(A, B, prefix, in_dim1, in_dim2, latent_dim, num_feat2, cfg.FBO_NL.NUM_LAYERS,
                                init_params1, init_params2, scale=latent_dim ** -.5 if cfg.FBO_NL.SCALE else 1.0,
                                pre_act_ln=cfg.FBO_NL.PRE_ACT_LN, dropout_ratio=drop)
    nl_out = None
    for layer in range(cfg.FBO_NL.NUM_LAYERS):
        name = prefix + '_nl%d' % layer
        nl_out = NLCore(model, in_blob1=A, in_blob2=B, in_dim1=in_dim1, in_dim2=in_dim2, latent_dim=latent_dim,
                        num_feat1=num_feat1, num_feat2=num_feat2, prefix=name, test_mode=test_mode)
        nl_out = model.net.Sum([nl_out, A], name + '_sum')
        if not cfg.FBO_NL.PRE_ACT:
            nl_out = model.Relu(nl_out, name + '_relu')
        A = nl_out
    return nl_out


def _fc_like_init():
    return {'weight_init': ('GaussianFill', {'std': cfg.MODEL.FC_INIT_STD}),
            'bias_init': ('ConstantFill', {'value': 0.}), 'no_bias': cfg.NONLOCAL.NO_BIAS}


def prepare_nl_input(model, blob, dim_in, prefix, test_mode):
    """Query-side pre-processing: optional 2048 -> LATENT_DIM reduction and dropout."""
    new_dim = dim_in
    if cfg.FBO_NL.INPUT_REDUCE_DIM:
        blob = _linear(model, blob, blob + prefix + '_reduc', dim_in, cfg.FBO_NL.LATENT_DIM, _fc_like_init())
        new_dim = cfg.FBO_NL.LATENT_DIM
    if cfg.FBO_NL.INPUT_DROPOUT_ON and not test_mode:
        blob = model.Dropout(blob, blob + prefix + '_drop', ratio=cfg.FBO_NL.DROPOUT_RATE, is_test=False)
    return blob, new_dim


def prepare_lfb(model, lfb, test_mode, suffix):
    """Bank-side pre-processing: LFB_DIM -> LATENT_DIM projection ('lfb_1x1') and dropout."""
    lfb = _linear(model, lfb, 'lfb_1x1', cfg.LFB.LFB_DIM, cfg.FBO_NL.LATENT_DIM, _fc_like_init())
    if cfg.FBO_NL.LFB_DROPOUT_ON and not test_mode:
        lfb = model.Dropout(lfb, lfb + '_drop', ratio=cfg.FBO_NL.DROPOUT_RATE, is_test=False)
    return lfb, cfg.FBO_NL.LATENT_DIM
