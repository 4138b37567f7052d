"""Output heads (CUDA re-implementation of the reference's lib/models/head_helper.py).

`add_roi_head` (AVA, box-level; reference :61-85 with `roi_pool` :88-123): temporal average
pool -> Squeeze -> legacy RoIAlign 7x7 -> 7x7 max pool -> `box_pooled` (R, 2048, 1, 1, 1),
optionally concatenated with the feature-bank operator output into `pool5`.
`add_basic_head` (Charades / EPIC, clip-level; reference :32-58): global average pool.
"""
from core.config import config as cfg
import models.lfb_helper as lfb_helper


def _with_fbo(model, feat, dim_in, num_lfb_feat, suffix, lfb_infer_only, test_mode):
    """Concat([feat, FBO(feat, bank)]) -> 'pool5' when the bank is enabled."""
    heads, dims = [feat], [dim_in]
    if cfg.LFB.ENABLED and not lfb_infer_only:
        fbo_out, fbo_dim = lfb_helper.add_fbo_head(model, feat, dim_in, num_lfb_feat=num_lfb_feat,
                                                   test_mode=test_mode, suffix=suffix)
        heads.append(fbo_out)
        dims.append(fbo_dim)
    return model.net.Concat(heads, ['pool5', 'pool5_concat_info'], axis=1)[0], sum(dims)


def add_basic_head(model, blob_in, dim_in, pool_stride, out_spatial_dim, suffix, lfb_infer_only, test_mode):
    """Clip-level head: (B, 2048, T, S, S) -> (B, 2048, 1, 1, 1)."""
    pooled = model.AveragePool(blob_in, blob_in + '_pooled',
                               kernels=[pool_stride, out_spatial_dim, out_spatial_dim],
                               strides=[1, 1, 1], pads=[0, 0, 0] * 2)
    return _with_fbo(model, pooled, dim_in, cfg.LFB.WINDOW_SIZE, suffix, lfb_infer_only, test_mode)


def add_roi_head(model, blob_in, dim_in, pool_stride, out_spatial_dim, suffix, lfb_infer_only, test_mode):
    """Box-level head: (B, 2048, 16, 14, 14) + proposals (R, 5) -> (R, 2048, 1, 1, 1)."""
    roi_feat = roi_pool(model, blob_in, dim_in, out_spatial_dim, suffix)
    return _with_fbo(model, roi_feat, dim_in, cfg.LFB.WINDOW_SIZE * cfg.AVA.LFB_MAX_NUM_FEAT_PER_STEP, suffix,
                     lfb_infer_only, test_mode)


def roi_pool(model, blob_in, dim_in, out_spatial_dim, suffix):
    """Temporal mean, RoIAlign and spatial max over each box."""
    pooled = model.AveragePool(blob_in, 'blob_pooled', kernels=[cfg.TRAIN.VIDEO_LENGTH // 2, 1, 1],
                               strides=[1, 1, 1], pads=[0, 0, 0] * 2)
    pooled = model.Squeeze(pooled, pooled + '_4d', dims=[2])               # (B, C, 1, H, W) -> (B, C, H, W)
    resolution = cfg.ROI.XFORM_RESOLUTION
    roi_feat = lfb_helper.RoIFeatureTransform(
        model, pooled, 'roi_feat_3d', blob_rois='proposals{}'.format(suffix), resolution=resolution,
        spatial_scale=(1.0 / cfg.ROI.SCALE_FACTOR))
    if resolution > 1:
        roi_feat = model.MaxPool(roi_feat, 'roi_feat_1d', kernels=[resolution, resolution], strides=[1, 1],
                                 pads=[0, 0] * 2)
    roi_feat, _ = model.Reshape(roi_feat, ['box_pooled', 'roi_feat_re2_shape'], shape=(-1, dim_in, 1, 1, 1))
    return roi_feat
