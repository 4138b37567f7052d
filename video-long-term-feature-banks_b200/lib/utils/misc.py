"""Small helpers that are part of the builder boundary (reference lib/utils/misc.py:68-79)."""
from core.config import config as cfg


def get_batch_size(split, packed=False):
    """Per-GPU batch size (reference lib/utils/misc.py:68-72).  packed: the clips of one step of a training net with
    update ops, which packs B200.GPUS_PER_STEP = v virtual GPUs (DESIGN.md 4.9) and gets v times the per-GPU size;
    every other net (feature-bank inference, test, precise-BN, gradient-only) keeps the per-GPU size.  (An invalid v is
    left for CreateNet to refuse.)"""
    if split in ['test', 'val']:
        return int(cfg.TEST.BATCH_SIZE / cfg.NUM_GPUS)
    elif split == 'train':
        b = int(cfg.TRAIN.BATCH_SIZE / cfg.NUM_GPUS)
        v = cfg.B200.get('GPUS_PER_STEP', 1)
        if not packed or isinstance(v, bool) or not isinstance(v, int) or v < 1:
            return b
        return b * v


def get_crop_size(split):
    """reference lib/utils/misc.py:75-79."""
    if split in ['test', 'val']:
        return cfg.TEST.CROP_SIZE
    elif split == 'train':
        return cfg.TRAIN.CROP_SIZE
