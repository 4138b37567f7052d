"""Model builder abstraction (CUDA re-implementation of the reference's
lib/models/model_builder_video.py).

`ModelBuilder` keeps the reference's constructor kwargs, methods and attributes (:66-314) but
derives from vlfb.cnn.CNNModelHelper, so the builder functions record a net that vlfb.executor
lowers onto sm_90a kernels.  The data loader side (`get_input_db` / `DataLoader`, :98-117) is
out of scope: inputs are fed with workspace.FeedBlob under the reference's blob names.
"""
import logging

import numpy as np

from core.config import config as cfg
from models import resnet_video
import utils.lr_policy as lr_policy
import utils.misc as misc
from vlfb import cnn, data_parallel, workspace

logger = logging.getLogger(__name__)

model_creator_map = {
    'resnet_video': resnet_video,
    'resnet_video_org': resnet_video,      # alias named by BASELINE.json; no such module upstream
}

# blob names the reference's datasets enqueue (lib/datasets/ava.py:139-146, charades.py:51-55)
_INPUT_BLOBS = {
    'ava': ['data', 'labels', 'proposals', 'original_boxes', 'metadata', 'lfb'],
    'charades': ['data', 'labels', 'lfb'],
    'epic': ['data', 'labels', 'lfb'],
}


class _BlobFeeder(object):
    """Minimal stand-in for the reference DataLoader's naming interface (dataloader.py:67)."""

    def __init__(self, split, suffix, lfb_enabled):
        names = list(_INPUT_BLOBS.get(cfg.DATASET, ['data', 'labels']))
        if not lfb_enabled and 'lfb' in names:
            names.remove('lfb')
        self._names = [n + suffix for n in names]
        self._blobs_queue_name = 'blobs_queue_{}{}'.format(split, suffix)

    def get_blob_names(self):
        return list(self._names)


class ModelBuilder(cnn.CNNModelHelper):

    def __init__(self, **kwargs):
        kwargs['order'] = 'NCHW'
        self.train = kwargs.pop('train', False)
        self.split = kwargs.pop('split', 'train')
        self.force_fw_only = kwargs.pop('force_fw_only', False)
        super(ModelBuilder, self).__init__(**kwargs)
        self.do_not_update_params = []
        self.data_loader = None
        self.input_db = None
        self.current_lr = 0
        self.SetCurrentLr(0)

    def TrainableParams(self, scope=''):
        """Parameters that receive a gradient (AffineNd scale/bias never do, reference :91-95,223-250)."""
        scope = str(scope)
        return [p for p in self.params
                if p in self.param_to_grad and p not in self.do_not_update_params
                and (scope == '' or scope.startswith('gpu_') or str(p).find(scope) == 0)]

    def build_model(self, suffix, lfb=None, lfb_infer_only=False, shift=1, node_id=0):
        self.crop_size = misc.get_crop_size(self.split)
        self.data_loader = _BlobFeeder(self.split, suffix, cfg.LFB.ENABLED and not lfb_infer_only)
        self.create_data_parallel_model(
            model=self, db_loader=self.data_loader, split=self.split, node_id=node_id, train=self.train,
            force_fw_only=self.force_fw_only, suffix=suffix, lfb_infer_only=lfb_infer_only)

    def create_data_parallel_model(self, model, db_loader, split, node_id, train=True, force_fw_only=False,
                                   suffix='', lfb_infer_only=False):
        forward_fun = create_model(model=self, split=split, suffix=suffix, lfb_infer_only=lfb_infer_only)
        input_fun = add_inputs(model=model, data_loader=db_loader, suffix=suffix)
        update_fun = add_parameter_update_ops(model=model) if (train and not force_fw_only) else None
        data_parallel.Parallelize_GPU(
            model, input_builder_fun=input_fun, forward_pass_builder_fun=forward_fun,
            param_update_builder_fun=update_fun, devices=[cfg.ROOT_GPU_ID], rendezvous=None,
            broadcast_computed_params=False, optimize_gradient_memory=cfg.MODEL.MEMONGER,
            use_nccl=not cfg.DEBUG)

    def start_data_loader(self):
        logger.info('inputs are fed with workspace.FeedBlob; no loader threads to start')

    def shutdown_data_loader(self):
        pass

    # ---- op wrappers ---------------------------------------------------------------------
    def Relu_(self, blob_in):
        """ReLU, in place when MODEL.ALLOW_INPLACE_RELU."""
        return self.Relu(blob_in, blob_in if cfg.MODEL.ALLOW_INPLACE_RELU else blob_in + '_relu')

    def Conv3dBN(self, blob_in, prefix, dim_in, dim_out, kernels, strides, pads, group=1, bn_init=None, **kwargs):
        conv = self.ConvNd(blob_in, prefix, dim_in, dim_out, kernels, strides=strides, pads=pads, group=group,
                           weight_init=('MSRAFill', {}), bias_init=('ConstantFill', {'value': 0.}), no_bias=1)
        out = self.SpatialBN(conv, prefix + '_bn', dim_out, epsilon=cfg.MODEL.BN_EPSILON,
                             momentum=cfg.MODEL.BN_MOMENTUM, is_test=self.split in ['test', 'val'])
        if bn_init is not None and bn_init != 1.0:
            self.param_init_net.ConstantFill([prefix + '_bn_s'], prefix + '_bn_s', value=bn_init)
        return out

    def Conv3dAffine(self, blob_in, prefix, dim_in, dim_out, kernels, strides, pads, group=1, suffix='_bn',
                     inplace_affine=False, dilations=None, **kwargs):
        """conv (MSRA init, no bias) followed by the frozen-BN affine; fused into one kernel at lowering."""
        conv = self.ConvNd(blob_in, prefix, dim_in, dim_out, kernels, strides=strides, pads=pads, group=group,
                           weight_init=('MSRAFill', {}), bias_init=('ConstantFill', {'value': 0.}), no_bias=1,
                           dilations=dilations if dilations is not None else [1, 1, 1])
        return self.AffineNd(conv, prefix + suffix, dim_out, inplace=inplace_affine)

    def AffineNd(self, blob_in, blob_out, dim_in, share_with=None, inplace=False):
        """y = x * s[c] + b[c] with s, b frozen (the custom op caffe2_customized_ops/video/affine_nd_op.cu)."""
        blob_out = blob_out or self.net.NextName()
        owner = blob_out if share_with is None else share_with
        scale = self.param_init_net.ConstantFill([], owner + '_s', shape=[dim_in], value=1.)
        bias = self.param_init_net.ConstantFill([], owner + '_b', shape=[dim_in], value=0.)
        if share_with is None:
            self.net.Proto().external_input.extend([str(scale), str(bias)])
            self.params.extend([scale, bias])
            self.weights.append(scale)
            self.biases.append(bias)
        self.frozen_params.update([scale, bias])
        return self.net.AffineNd([blob_in, scale, bias], blob_in if inplace else blob_out)

    # ---- learning rate ---------------------------------------------------------------------
    def SetCurrentLr(self, cur_iter):
        self.current_lr = lr_policy.get_lr_at_iter(cur_iter)

    def UpdateWorkspaceLr(self, cur_iter):
        new_lr = lr_policy.get_lr_at_iter(cur_iter)
        if new_lr != self.current_lr:
            if _get_lr_change_ratio(self.current_lr, new_lr) > 1.1:
                logger.info('Setting learning rate to {:.6f} at iteration {}'.format(new_lr, cur_iter))
            self._SetNewLr(self.current_lr, new_lr)

    def _SetNewLr(self, cur_lr, new_lr):
        assert cur_lr > 0
        workspace.FeedBlob('gpu_{}/lr'.format(cfg.ROOT_GPU_ID), np.array(new_lr, dtype=np.float32))
        ratio = _get_lr_change_ratio(cur_lr, new_lr)
        if cfg.SOLVER.SCALE_MOMENTUM and cur_lr > 1e-7 and ratio > cfg.SOLVER.SCALE_MOMENTUM_THRESHOLD:
            self._CorrectMomentum(new_lr / cur_lr)
        self.current_lr = new_lr

    def _CorrectMomentum(self, correction):
        """MomentumSGDUpdate stores V = mu*V + lr*grad, so V is rescaled when lr jumps (reference :286-314)."""
        if correction < 0.9 or correction > 1.1:
            logger.info('Scaling update history by {:.6f} (new/old lr)'.format(correction))
        workspace.current().params.scale_momentum(self.TrainableParams(), float(correction))


def create_model(model, split, suffix, lfb_infer_only):
    model_name = cfg.MODEL.MODEL_NAME
    assert model_name in model_creator_map, 'Unknown model_type {}'.format(model_name)

    def model_creator(model, loss_scale):
        model, softmax, loss = model_creator_map[model_name].create_model(
            model=model, data='data{}'.format(suffix), labels='labels{}'.format(suffix), split=split,
            suffix=suffix, lfb_infer_only=lfb_infer_only)
        return [loss]
    return model_creator


def add_inputs(model, data_loader, suffix):
    blob_names = data_loader.get_blob_names()
    queue_name = data_loader._blobs_queue_name

    def input_fn(model):
        model.DequeueBlobs(queue_name, blob_names)
        model.StopGradient('data{}'.format(suffix), 'data{}'.format(suffix))
    return input_fn


def add_parameter_update_ops(model):
    def param_update_ops(model):
        fill = model.param_init_net.ConstantFill
        lr = fill([], 'lr', shape=[1], value=float(model.current_lr))
        weight_decay = fill([], 'weight_decay', shape=[1], value=cfg.SOLVER.WEIGHT_DECAY)
        weight_decay_bn = fill([], 'weight_decay_bn', shape=[1], value=cfg.SOLVER.WEIGHT_DECAY_BN)
        one = fill([], 'ONE', shape=[1], value=1.0)
        trainable = set(model.TrainableParams())
        assert len(model.GetParams()) > 0, 'No trainable params found in model'
        for param in model.GetParams():
            if param not in trainable:
                continue
            grad = model.param_to_grad[param]                # already summed over replicas
            momentum = fill([param], param + '_momentum', value=0.0)
            wd = weight_decay_bn if '_bn' in str(param) else weight_decay
            model.WeightedSum([grad, one, param, wd], grad)
            model.net.MomentumSGDUpdate([grad, momentum, lr, param], [grad, momentum, param],
                                        momentum=cfg.SOLVER.MOMENTUM, nesterov=cfg.SOLVER.NESTEROV)
    return param_update_ops


def _get_lr_change_ratio(cur_lr, new_lr):
    eps = 1e-10
    return np.max((new_lr / np.max((cur_lr, eps)), cur_lr / np.max((new_lr, eps))))
