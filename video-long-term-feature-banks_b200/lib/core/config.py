"""Global config tree -- py3 re-implementation of the reference's lib/core/config.py.

Same key names, same defaults (reference lib/core/config.py:52-364), same YAML /
command-line merge semantics (merge_dicts :394-420, cfg_from_file :423-428,
cfg_from_list :431-451, assert_and_infer_cfg :373-391) so every shipped
configs/*.yaml loads unchanged.  Differences forced by py3: string defaults are
`str` (the reference's are py2 byte strings) and YAML is read with safe_load.
"""
from ast import literal_eval

import yaml

from utils.collections import AttrDict


def _tree(d):
    return AttrDict({k: _tree(v) if isinstance(v, dict) else v for k, v in d.items()})


__C = _tree({
    'DEBUG': False,
    'DATALOADER': {'MAX_BAD_IMAGES': 100},
    'DATA_MEAN': [0.45, 0.45, 0.45],
    'DATA_STD': [0.225, 0.225, 0.225],
    'TRAIN': {
        'PARAMS_FILE': '', 'DATA_TYPE': 'train', 'BATCH_SIZE': 64,
        'RESUME_FROM_BATCH_SIZE': -1, 'RESET_START_ITER': False,
        'JITTER_SCALES': [256, 480], 'CROP_SIZE': 224, 'USE_COLOR_AUGMENTATION': False,
        'PCA_EIGVAL': [0.225, 0.224, 0.229],
        'PCA_EIGVEC': [[-0.5675, 0.7192, 0.4009], [-0.5808, -0.0045, -0.8140],
                       [-0.5836, -0.6948, 0.4203]],
        'COMPUTE_PRECISE_BN': True, 'ITER_COMPUTE_PRECISE_BN': 200, 'EVAL_PERIOD': 4000,
        'DATASET_SIZE': 0, 'VIDEO_LENGTH': 32, 'SAMPLE_RATE': 2, 'DROPOUT_RATE': 0.0,
        'TEST_AFTER_TRAIN': True,
    },
    'MODEL': {
        'NUM_CLASSES': -1, 'MODEL_NAME': '', 'VIDEO_ARC_CHOICE': 2, 'DEPTH': 50,
        'BN_MOMENTUM': 0.9, 'BN_EPSILON': 1.0000001e-5, 'BN_INIT_GAMMA': 1.0,
        'FC_INIT_STD': 0.01, 'MEAN': 114.75, 'STD': 57.375,
        'ALLOW_INPLACE_SUM': True, 'ALLOW_INPLACE_RELU': True, 'ALLOW_INPLACE_RESHAPE': True,
        'MEMONGER': True, 'USE_BGR': False, 'USE_AFFINE': False, 'SAMPLE_THREADS': 8,
        'MULTI_LABEL': True, 'DILATIONS_AFTER_CONV5': True, 'FREEZE_BACKBONE': False,
    },
    'RESNETS': {'NUM_GROUPS': 1, 'WIDTH_PER_GROUP': 64, 'STRIDE_1X1': False,
                'TRANS_FUNC': 'bottleneck_transformation'},
    'TEST': {
        'PARAMS_FILE': '', 'DATA_TYPE': '', 'BATCH_SIZE': 64, 'SCALE': 256, 'CROP_SIZE': 256,
        'DATASET_SIZE': 0, 'VIDEO_LENGTH': 32, 'SAMPLE_RATE': 2, 'CROP_SHIFT': 1,
    },
    'SOLVER': {
        'NESTEROV': True, 'WEIGHT_DECAY': 0.0001, 'WEIGHT_DECAY_BN': 0.0001, 'MOMENTUM': 0.9,
        'LR_POLICY': 'steps_with_relative_lrs', 'BASE_LR': 0.1,
        'STEP_SIZES': [100000, 20000, 20000], 'LRS': [1, 0.1, 0.01], 'MAX_ITER': 140000,
        'STEPS': None, 'GAMMA': 0.1, 'SCALE_MOMENTUM': False, 'SCALE_MOMENTUM_THRESHOLD': 1.1,
        'WARMUP': {'WARMUP_ON': False, 'WARMUP_START_LR': 0.1, 'WARMUP_END_ITER': 5000},
    },
    'CHECKPOINT': {'CHECKPOINT_MODEL': True, 'CHECKPOINT_PERIOD': -1, 'RESUME': True,
                   'DIR': '.', 'CONVERT_MODEL': False},
    'NONLOCAL': {
        'CONV_INIT_STD': 0.01, 'NO_BIAS': 0, 'USE_MAXPOOL': True, 'USE_SOFTMAX': True,
        'USE_ZERO_INIT_CONV': False, 'USE_BN': True, 'USE_SCALE': True, 'USE_AFFINE': False,
        'BN_MOMENTUM': 0.9, 'BN_EPSILON': 1.0000001e-5, 'BN_INIT_GAMMA': 0.0,
        'LAYER_MOD': 2, 'CONV3_NONLOCAL': True, 'CONV4_NONLOCAL': True,
    },
    'DATADIR': '', 'DATASET': '', 'ROOT_GPU_ID': 0, 'NUM_GPUS': 8,
    'CUDNN_WORKSPACE_LIMIT': 256, 'RNG_SEED': 2, 'USE_CYTHON': False, 'LOG_PERIOD': 10,
    'PROF_DAG': False, 'INTERPOLATION': 'INTER_LINEAR', 'MINIBATCH_QUEUE_SIZE': 64,
    'AVA': {
        'FRAME_LIST_DIR': 'data/ava/frame_lists', 'ANNOTATION_DIR': 'data/ava/annotations',
        'FPS': 30, 'FULL_EVAL_DURING_TRAINING': False, 'DETECTION_SCORE_THRESH_TRAIN': 0.9,
        'DETECTION_SCORE_THRESH_EVAL': [0.85], 'LFB_DETECTION_SCORE_THRESH': 0.9,
        'TRAIN_ON_TRAIN_VAL': False, 'TEST_ON_TEST_SET': False,
        'TRAIN_LISTS': ['train.csv'], 'TEST_LISTS': ['val.csv'],
        'TRAIN_BOX_LISTS': ['ava_train_v2.1.csv', 'ava_train_predicted_boxes.csv'],
        'TEST_BOX_LISTS': ['ava_val_predicted_boxes.csv'],
        'TRAIN_LFB_BOX_LISTS': ['ava_train_predicted_boxes.csv'],
        'TEST_LFB_BOX_LISTS': ['ava_val_predicted_boxes.csv'],
        'TEST_MULTI_CROP': False, 'TEST_MULTI_CROP_SCALES': [224, 256, 320],
        'FORCE_TEST_FLIP': False, 'LFB_MAX_NUM_FEAT_PER_STEP': 5,
    },
    'EPIC': {
        'FRAME_LIST_DIR': 'data/epic/frame_lists', 'ANNOTATION_DIR': 'data/epic/annotations',
        'TRAIN_LISTS': ['train.csv'], 'TEST_LISTS': ['val.csv'],
        'ANNOTATIONS': 'EPIC_train_action_labels.csv', 'FPS': 30, 'CLASS_TYPE': '',
        'VERB_LFB_CLIPS_PER_SECOND': 1, 'NOUN_LFB_FRAMES_PER_SECOND': 1,
        'MAX_NUM_FEATS_PER_NOUN_LFB_FRAME': 10,
    },
    'CHARADES': {
        'FRAME_LIST_DIR': 'data/charades/frame_lists', 'TRAIN_LISTS': ['train.csv'],
        'TEST_LISTS': ['val.csv'], 'FPS': 24, 'NUM_TEST_CLIPS_DURING_TRAINING': 9,
        'NUM_TEST_CLIPS_FINAL_EVAL': 30, 'LFB_CLIPS_PER_SECOND': 2,
    },
    'ROI': {'SCALE_FACTOR': 16, 'XFORM_RESOLUTION': 7},
    'LFB': {'ENABLED': False, 'MODEL_PARAMS_FILE': '', 'WRITE_LFB': False, 'LOAD_LFB': False,
            'LOAD_LFB_PATH': '', 'LFB_DIM': 2048, 'WINDOW_SIZE': 100, 'FBO_TYPE': 'nl'},
    'FBO_NL': {'NUM_LAYERS': 2, 'PRE_ACT': True, 'PRE_ACT_LN': True, 'SCALE': True,
               'LATENT_DIM': 512, 'INPUT_REDUCE_DIM': True, 'DROPOUT_RATE': 0.2,
               'INPUT_DROPOUT_ON': True, 'LFB_DROPOUT_ON': True, 'NL_DROPOUT_ON': True},
    'IMG_LOAD_RETRY': 10,
    'GET_TRAIN_LFB': False,
    # ---- additions of this implementation (not in the reference) -------------
    # B200.COMPUTE: 'tf32' = parity mode (fp32 storage, GEMM operands rounded to TF32 where they are produced, tensor-core
    #   tf32 MMA, fp32 accumulate); 'tf32x3' = nothing rounded, every tensor-core GEMM on split-TF32 products (3xTF32,
    #   about 2x the step time; DESIGN.md 4.7).  Any other value raises VlfbError: 'fp32' is reserved for a mode whose
    #   products are fp32 FMAs, which split-TF32 products are not.
    # B200.FBO_FOLD: inference nets run each FBO-NL layer as one pass over the raw bank (vlfb.executor.FboFoldStep).
    # B200.LFB_DTYPE: 'f32' | 'bf16' = storage type of the feature-bank windows the folded inference FBO scans (a bf16
    #   copy is made when the bank is fed; scores / softmax / sums stay fp32; parity tolerance 1e-2 instead of 1e-3).
    # B200.DETERMINISTIC: nets created while it is True run every cross-thread float reduction in a fixed order (no float
    #   atomics with more than one contribution per element), so that two runs of the same calls from the same state are
    #   bitwise identical on one GPU model and library build (DESIGN.md 4.5).  A guarantee, not a speed: off by default.
    # B200.ROI_CAPACITY: C > 0 = nets created while it is set that have a RoIAlign on 'proposals{sfx}' (AVA train, test and
    #   lfb_infer_only nets) keep their per-RoI inputs (proposals, labels, original_boxes, metadata, lfb) in buffers of C
    #   rows, so a batch with any number r <= C of boxes replays the same captured step; a device-side count tells the
    #   kernels which rows are real, and FetchBlob returns the r live rows.  C is a memory and compute budget the data
    #   pipeline chooses (clips per GPU x boxes per clip after the detection threshold).  0 = the RoI count is part of
    #   the captured graph's key, as before (DESIGN.md 4.6).
    # B200.ITER_SIZE: k > 1 = training nets (with update ops) created while it is set accumulate gradients over k RunNet
    #   calls (micro-steps, one micro-batch each) and all-reduce + apply SGD once, at the k-th; NUM_GPUS must equal k x
    #   the number of processes, so that an iteration computes the update of NUM_GPUS GPUs of the reference on fewer
    #   H100s.  Test, val, lfb_infer_only, precise-BN and gradient-only nets ignore it.  1 = one update per RunNet
    #   (DESIGN.md 4.8).
    # B200.GPUS_PER_STEP: v > 1 = training nets (with update ops) created while it is set run v of the recipe's virtual
    #   GPUs in one RunNet, as one packed batch of v x (TRAIN.BATCH_SIZE / NUM_GPUS) clips: clips [j b, (j+1) b) and the
    #   RoIs with batch index in that range are virtual GPU j's.  The sigmoid loss is normalised per virtual GPU and
    #   SpatialBN takes batch statistics per virtual GPU; NUM_GPUS must equal v x ITER_SIZE x the number of processes.
    #   Test, val, lfb_infer_only, precise-BN and gradient-only nets ignore it.  1 = one virtual GPU per step
    #   (DESIGN.md 4.9).
    'B200': {'COMPUTE': 'tf32', 'GEMM_BACKEND': 'tcgen05', 'CUDA_GRAPH': True, 'FBO_FOLD': True, 'FBO_STACK': True,
             'LFB_DTYPE': 'f32', 'DETERMINISTIC': False, 'ROI_CAPACITY': 0, 'ITER_SIZE': 1,
             'GPUS_PER_STEP': 1},
})
config = __C
_DEFAULTS = None


def reset_cfg():
    """Restore the defaults (handy for tests; the reference has no equivalent)."""
    import copy
    global _DEFAULTS
    if _DEFAULTS is None:
        _DEFAULTS = copy.deepcopy(dict(__C))
    else:
        __C.clear()
        __C.update(_tree(copy.deepcopy(_DEFAULTS)))


reset_cfg()


def print_cfg():
    import logging
    import pprint
    logging.getLogger(__name__).info('Config:\n' + pprint.pformat(__C))


def assert_and_infer_cfg():
    """reference lib/core/config.py:373-391."""
    if __C.SOLVER.STEPS is None:
        steps = [0]
        for size in __C.SOLVER.STEP_SIZES:
            steps.append(size + steps[-1])
        __C.SOLVER.STEPS = steps
    assert __C.TRAIN.BATCH_SIZE % __C.NUM_GPUS == 0, \
        'Train batch size should be multiple of num_gpus.'
    assert __C.TEST.BATCH_SIZE % __C.NUM_GPUS == 0, \
        'Test batch size should be multiple of num_gpus.'
    __C.LFB.NUM_LFB_FEAT = __C.AVA.LFB_MAX_NUM_FEAT_PER_STEP * __C.LFB.WINDOW_SIZE


def _same_type(old, new):
    if old is None or new is None:
        return True
    if isinstance(old, bool) or isinstance(new, bool):
        return isinstance(old, bool) and isinstance(new, bool)
    if isinstance(old, (int, float)) and isinstance(new, (int, float)):
        # the reference insists on identical types; YAML '1' vs default 1.0 only
        # differs by spelling, so int<->float is tolerated here.
        return True
    return type(old) is type(new) or (isinstance(old, dict) and isinstance(new, dict))


def merge_dicts(dict_a, dict_b):
    """Merge dict_a into dict_b with key and type checking (reference :394-420)."""
    for key, value in dict_a.items():
        if key not in dict_b:
            raise KeyError('Invalid key in config file: {}'.format(key))
        if isinstance(value, dict):
            value = _tree(value)
        if isinstance(value, str):
            try:
                value = literal_eval(value)
            except BaseException:
                pass
        if not _same_type(dict_b[key], value):
            raise ValueError('Type mismatch ({} vs. {}) for config key: {}'.format(
                type(dict_b[key]), type(value), key))
        if isinstance(value, AttrDict):
            try:
                merge_dicts(value, dict_b[key])
            except BaseException:
                raise Exception('Error under config key: {}'.format(key))
        else:
            dict_b[key] = value


def cfg_from_file(filename):
    """Load a YAML config and merge it into the defaults (reference :423-428)."""
    with open(filename, 'r') as fopen:
        yaml_config = _tree(yaml.safe_load(fopen))
    merge_dicts(yaml_config, __C)


def cfg_from_list(args_list):
    """Set config keys from a flat KEY VALUE list (reference :431-451)."""
    assert len(args_list) % 2 == 0, 'Specify values or keys for args'
    for key, value in zip(args_list[0::2], args_list[1::2]):
        key_list = key.split('.')
        cfg = __C
        for subkey in key_list[:-1]:
            assert subkey in cfg, 'Config key {} not found'.format(subkey)
            cfg = cfg[subkey]
        subkey = key_list[-1]
        assert subkey in cfg, 'Config key {} not found'.format(subkey)
        val = value
        if isinstance(value, str):
            try:
                val = literal_eval(value)
            except BaseException:
                val = value
        assert _same_type(cfg[subkey], val), 'type {} does not match original type {}'.format(
            type(val), type(cfg[subkey]))
        cfg[subkey] = val
