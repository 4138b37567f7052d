"""Precise batch-norm statistics (CUDA re-implementation of the reference's lib/utils/bn_helper.py:60-221).

Before testing / checkpointing a SpatialBN model (`MODEL.USE_AFFINE False`), the running statistics kept by the
momentum update are replaced by the exact population statistics of `TRAIN.ITER_COMPUTE_PRECISE_BN` training batches:
an auxiliary forward-only training-mode net (batch statistics, no backward, no update) is run that many times, every
layer's batch mean `_bn_sm` and inverse std `_bn_siv` (outputs of vlfb_spatial_bn_fwd) are turned into E[x] and E[x^2],
averaged, and written to `_bn_rm` / `_bn_riv` (`riv` holds a VARIANCE, reference :216-219).

One process drives one GPU here, so the reference's loop over `gpu_{i}/` scopes (:164,213) covers the local device;
with torchrun data parallelism the per-rank E[x] / E[x^2] are additionally averaged over the ranks, which is what the
reference's division by `ITER * NUM_GPUS` (:186) does inside its single process.
"""
import logging

import numpy as np

from core.config import config as cfg
from models import model_builder_video
from vlfb import workspace

logger = logging.getLogger(__name__)


class BatchNormHelper(object):

    def __init__(self):
        self._model = None
        self._bn_layers = None
        self._meanX_dict = {}      # becomes '_bn_rm'
        self._meanX2_dict = {}
        self._var_dict = {}        # becomes '_bn_riv'
        self._last_update_iter = -1

    def create_bn_aux_model(self, node_id=0, suffix=None):
        """A net that is 'train' for its data and its BN mode (only training-mode BN emits sm / siv) and 'test' in that
        it neither back-propagates nor updates (reference :73-103)."""
        self._model = model_builder_video.ModelBuilder(
            name='{}_bn_aux'.format(cfg.MODEL.MODEL_NAME), train=True, use_cudnn=True, cudnn_exhaustive_search=True,
            ws_nbytes_limit=(cfg.get('CUDNN_WORKSPACE_LIMIT', 256) * 1024 * 1024), split=cfg.TRAIN.DATA_TYPE,
            use_mem_cache=False, force_fw_only=True)
        self._model.build_model(suffix='_{}'.format(cfg.TRAIN.DATA_TYPE) if suffix is None else suffix, node_id=node_id)
        # like the reference (:94), the aux net's param_init_net is NOT run: it shares the training net's parameters
        workspace.CreateNet(self._model.net)
        self._find_bn_layers()
        self._clean_and_reset_buffer()

    def compute_and_update_bn_stats(self, curr_iter=None, feed_fn=None):
        """Recompute when `curr_iter` changed since the last call, else only re-install the cached statistics
        (reference :105-136).  `feed_fn(i)`, when given, feeds batch i (the reference's loader threads do that)."""
        if curr_iter is None or curr_iter != self._last_update_iter:
            logger.info('Computing and updating BN stats at iter: {}'.format(-1 if curr_iter is None else curr_iter + 1))
            self._last_update_iter = curr_iter
            self._clean_and_reset_buffer()
            name = self._model.net.Proto().name
            for i in range(cfg.TRAIN.ITER_COMPUTE_PRECISE_BN):
                if feed_fn is not None:
                    feed_fn(i)
                workspace.RunNet(name)
                self._collect_bn_stats()
            self._finalize_bn_stats()
        else:
            logger.info('BN of iter {} computed. Update to GPU only.'.format(curr_iter + 1))
        self._update_bn_stats_gpu()

    def _find_bn_layers(self):
        self._bn_layers = []
        for blob in self._model.params:
            blob = str(blob)
            if blob.endswith('_bn_s') and (blob[:-2] + '_riv') in self._model.computed_params:
                if blob[:-5] not in self._bn_layers:
                    self._bn_layers.append(blob[:-5])

    def _clean_and_reset_buffer(self):
        self._meanX_dict = dict((layer, 0) for layer in self._bn_layers)
        self._meanX2_dict = dict((layer, 0) for layer in self._bn_layers)

    def _collect_bn_stats(self):
        """sm = mean(x), siv = 1 / sqrt(var(x) + eps) of the current batch; E[x] and E[x^2] are additive over
        batches (reference :154-182)."""
        eps = cfg.MODEL.BN_EPSILON
        for layer in self._bn_layers:
            mean = workspace.FetchBlob('gpu_{}/{}_bn_sm'.format(cfg.ROOT_GPU_ID, layer)).astype(np.float64)
            inv_std = workspace.FetchBlob('gpu_{}/{}_bn_siv'.format(cfg.ROOT_GPU_ID, layer)).astype(np.float64)
            var = (1. / inv_std) ** 2 - eps
            self._meanX_dict[layer] = self._meanX_dict[layer] + mean
            self._meanX2_dict[layer] = self._meanX2_dict[layer] + (var + mean ** 2)

    def _finalize_bn_stats(self):
        n = float(cfg.TRAIN.ITER_COMPUTE_PRECISE_BN)
        self._var_dict = {}
        for layer in self._bn_layers:
            ex, ex2 = self._meanX_dict[layer] / n, self._meanX2_dict[layer] / n
            ex, ex2 = _mean_over_ranks(ex), _mean_over_ranks(ex2)
            var = ex2 - ex ** 2
            assert (var > 0.).all(), 'layer: {} var < 0'.format(layer)
            self._meanX_dict[layer], self._meanX2_dict[layer], self._var_dict[layer] = ex, ex2, var

    def _update_bn_stats_gpu(self):
        """The blobs a test net reads are 'rm' and 'riv'; riv is the running VARIANCE (reference :198-221)."""
        for layer in self._bn_layers:
            scope = 'gpu_{}/{}'.format(cfg.ROOT_GPU_ID, layer)
            workspace.FeedBlob(scope + '_bn_rm', np.array(self._meanX_dict[layer], dtype=np.float32))
            workspace.FeedBlob(scope + '_bn_riv', np.array(self._var_dict[layer], dtype=np.float32))


def _mean_over_ranks(a):
    import torch
    if not (torch.distributed.is_available() and torch.distributed.is_initialized()) or torch.distributed.get_world_size() == 1:
        return a
    t = torch.as_tensor(np.asarray(a, dtype=np.float64))
    if torch.distributed.get_backend() == 'nccl':
        t = t.cuda()
    torch.distributed.all_reduce(t)
    return (t / torch.distributed.get_world_size()).cpu().numpy()
