"""Full-model builder (CUDA re-implementation of the reference's lib/models/resnet_video.py).

Same public surface -- `obtain_arc(arc_type)`, `create_model(model, data, labels, split,
lfb_infer_only, suffix='')`, `BLOCK_CONFIG` -- same blob names and YAML keys, so the graph a
driver obtains is the one the reference builds (stem conv1 5x7x7 -> pool1 -> res2 -> pool2 ->
res3(+grouped NL) -> res4(+NL) -> res5(dilated) -> head -> dropout -> pred -> loss; reference
lib/models/resnet_video.py:133-351).  The ops are recorded on a vlfb model helper and later
lowered onto fused sm_90a kernels by vlfb.executor.
"""
import logging

from core.config import config as cfg
from utils.misc import get_batch_size
import models.head_helper as head_helper
import models.resnet_helper as resnet_helper

logger = logging.getLogger(__name__)

# blocks per stage (res2..res5) by depth (reference :33-36)
BLOCK_CONFIG = {50: (3, 4, 6, 3), 101: (3, 4, 23, 3)}

# Temporal-kernel tables: arc -> per-stage list of `use_temp_conv` flags (kernel T = 1 + 2*flag).
_ALTERNATING_23 = [1 if i % 2 == 0 else 0 for i in range(23)]
_ARC_TEMP_CONVS = {
    1: ([0], [0] * 3, [0] * 4, [0] * 6, [0] * 3),                       # C2D R50
    2: ([2], [1, 1, 1], [1, 0, 1, 0], [1, 0, 1, 0, 1, 0], [0, 1, 0]),   # I3D R50
    3: ([0], [0] * 3, [0] * 4, [0] * 23, [0] * 3),                      # C2D R101
    4: ([2], [1, 1, 1], [1, 0, 1, 0], _ALTERNATING_23, [0, 1, 0]),      # I3D R101
}


def obtain_arc(arc_type):
    """Temporal kernel radii, temporal strides (all 1) and the temporal pooling stride
    for an architecture id (reference :39-130)."""
    pool_stride = 1
    table = _ARC_TEMP_CONVS.get(arc_type)
    assert table is not None, 'unknown MODEL.VIDEO_ARC_CHOICE {}'.format(arc_type)
    use_temp_convs_set = [list(stage) for stage in table]
    temp_strides_set = [[1] * len(stage) for stage in table]
    pool_stride = int(cfg.TRAIN.VIDEO_LENGTH / 2)
    return use_temp_convs_set, temp_strides_set, pool_stride


def _nonlocal_period(stage):
    """Insert an NL block after every `period`-th residual block of res3 / res4 (reference :213-217,267-271)."""
    period = cfg.NONLOCAL.LAYER_MOD
    if stage == 3:
        if cfg.MODEL.DEPTH == 101:
            period = 2
        return period if cfg.NONLOCAL.CONV3_NONLOCAL else 1000
    if cfg.MODEL.DEPTH == 101:
        period = period * 4 - 1
    return period if cfg.NONLOCAL.CONV4_NONLOCAL else 1000


def create_model(model, data, labels, split, lfb_infer_only, suffix=''):
    """Record the whole network on `model`; returns (model, prob, loss)."""
    cfg.DILATIONS = 1
    assert cfg.MODEL.DEPTH in BLOCK_CONFIG, 'Block config is not defined for specified model depth.'
    blocks = BLOCK_CONFIG[cfg.MODEL.DEPTH]
    group, width = cfg.RESNETS.NUM_GROUPS, cfg.RESNETS.WIDTH_PER_GROUP
    dim_inner = group * width
    # a net that gets update ops packs B200.GPUS_PER_STEP virtual GPUs per step; precise-BN and other forward-only
    # training-split nets keep one GPU's clips
    packed = (split == 'train' and not lfb_infer_only and getattr(model, 'train', False)
              and not getattr(model, 'force_fw_only', False))
    batch_size = get_batch_size(split, packed)
    model.recorded_batch_size = batch_size           # CreateNet checks it against B200.GPUS_PER_STEP
    test_mode = split in ('test', 'val')
    crop_size = cfg.TRAIN.CROP_SIZE if (split == 'train' and not lfb_infer_only) else cfg.TEST.CROP_SIZE
    logger.info('ResNet-%d %dx%dd %s, dataset %s, split %s, infer LFB %s, suffix "%s"',
                cfg.MODEL.DEPTH, group, width, cfg.RESNETS.TRANS_FUNC, cfg.DATASET, split, lfb_infer_only, suffix)

    tconvs, tstrides, pool_stride = obtain_arc(cfg.MODEL.VIDEO_ARC_CHOICE)
    res_block = resnet_helper._generic_residual_block_3d

    # ---- stem: conv1 (kT x 7 x 7, stride 1,2,2) -> affine/BN -> ReLU -> 1x3x3 max pool
    kt1 = 1 + 2 * tconvs[0][0]
    stem = model.ConvNd(data, 'conv1', 3, 64, [kt1, 7, 7], strides=[tstrides[0][0], 2, 2],
                        pads=[tconvs[0][0], 3, 3] * 2, weight_init=('MSRAFill', {}),
                        bias_init=('ConstantFill', {'value': 0.}), no_bias=1)
    if cfg.MODEL.USE_AFFINE:
        stem = model.AffineNd(stem, 'res_conv1_bn', 64)
    else:
        stem = model.SpatialBN(stem, 'res_conv1_bn', 64, epsilon=cfg.MODEL.BN_EPSILON,
                               momentum=cfg.MODEL.BN_MOMENTUM, is_test=test_mode)
    stem = model.Relu(stem, stem)
    blob = model.MaxPool(stem, 'pool1', kernels=[1, 3, 3], strides=[1, 2, 2], pads=[0, 1, 1] * 2)

    # ---- res2, temporal pool2
    blob, dim = resnet_helper.res_stage_nonlocal(
        model, res_block, blob, 64, 256, stride=1, num_blocks=blocks[0], prefix='res2',
        dim_inner=dim_inner, group=group, use_temp_convs=tconvs[1], temp_strides=tstrides[1])
    blob = model.MaxPool(blob, 'pool2', kernels=[2, 1, 1], strides=[2, 1, 1], pads=[0, 0, 0] * 2)

    # ---- res3: the affine (frozen-BN) nets run the NL blocks on groups of 4 frames
    res3_common = dict(stride=2, num_blocks=blocks[1], prefix='res3', dim_inner=dim_inner * 2, group=group,
                       use_temp_convs=tconvs[2], temp_strides=tstrides[2], batch_size=batch_size,
                       nonlocal_name='nonlocal_conv3', nonlocal_mod=_nonlocal_period(3))
    if cfg.MODEL.USE_AFFINE:
        blob, dim = resnet_helper.res_stage_nonlocal_group(
            model, res_block, blob, dim, 512, pool_stride=pool_stride, spatial_dim=int(crop_size / 8),
            group_size=4, **res3_common)
    else:
        blob, dim = resnet_helper.res_stage_nonlocal(model, res_block, blob, dim, 512, **res3_common)

    # ---- res4
    blob, dim = resnet_helper.res_stage_nonlocal(
        model, res_block, blob, dim, 1024, stride=2, num_blocks=blocks[2], prefix='res4',
        dim_inner=dim_inner * 4, group=group, use_temp_convs=tconvs[3], temp_strides=tstrides[3],
        batch_size=batch_size, nonlocal_name='nonlocal_conv4', nonlocal_mod=_nonlocal_period(4))

    # ---- res5: stride 1, dilation 2 on the 3x3
    if cfg.MODEL.DILATIONS_AFTER_CONV5:
        cfg.DILATIONS = 2
    blob, dim = resnet_helper.res_stage_nonlocal(
        model, res_block, blob, dim, 2048, stride=1, num_blocks=blocks[3], prefix='res5',
        dim_inner=dim_inner * 8, group=group, use_temp_convs=tconvs[4], temp_strides=tstrides[4])
    if cfg.MODEL.FREEZE_BACKBONE:
        model.StopGradient(blob, blob)

    # ---- head
    heads = {'ava': head_helper.add_roi_head, 'charades': head_helper.add_basic_head,
             'epic': head_helper.add_basic_head}
    if cfg.DATASET not in heads:
        raise NotImplementedError('Unknown dataset {}'.format(cfg.DATASET))
    blob, dim = heads[cfg.DATASET](model, blob, dim, pool_stride, crop_size // 16, suffix, lfb_infer_only, test_mode)
    if lfb_infer_only:
        return model, None, None

    if cfg.TRAIN.DROPOUT_RATE > 0 and not test_mode:
        blob = model.Dropout(blob, blob + '_dropout', ratio=cfg.TRAIN.DROPOUT_RATE, is_test=False)
    logits = model.FC(blob, 'pred', dim, cfg.MODEL.NUM_CLASSES,
                      weight_init=('GaussianFill', {'std': cfg.MODEL.FC_INIT_STD}),
                      bias_init=('ConstantFill', {'value': 0.}))

    loss_scale = 1. / cfg.NUM_GPUS     # gradients are SUMMED across replicas (reference :333-341)
    loss = None
    if cfg.MODEL.MULTI_LABEL:
        if split == 'train':
            prob = model.Sigmoid(logits, 'prob')
            loss = model.SigmoidCrossEntropyLoss([logits, labels], ['loss'], scale=loss_scale)
        else:
            prob = model.Sigmoid(logits, 'prob', engine='CUDNN')
    elif split == 'train':
        prob, loss = model.SoftmaxWithLoss([logits, labels], ['prob', 'loss'], scale=loss_scale)
    else:
        prob = model.Softmax(logits, 'prob')
    return model, prob, loss
