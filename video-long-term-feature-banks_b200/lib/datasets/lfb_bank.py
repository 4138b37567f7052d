"""Device-resident long-term feature bank (SURVEY.md 8f rank 1).

The reference keeps the bank as a nested python dict of numpy rows in host RAM (tools/lfb_loader.py:51-152,
pickle format {video_idx: {sec_or_frame: feature(s)}}), re-assembles each example's (L x 2048) window with python
loops (lib/datasets/ava.py:300-323, charades.py:251-276, epic.py:310-331) and ships it host->device every step:
2.46 MB per RoI at L=300, duplicated for every box of a clip.  Here the bank is packed ONCE into a [rows, LFB_DIM]
tensor in HBM; per step the host only computes an int32 row-index table with the reference's own sampling rules
(same np.random call sequence, so the same rows are drawn for the same seed) and `vlfb_lfb_gather` assembles the
windows on the device straight into the net's `lfb{suffix}` input blob (zero rows where the table holds -1).
The on-disk pickle format of the reference is kept (load_lfb / write_lfb).
"""
import pickle

import numpy as np
import torch

FPS = 24     # lib/datasets/charades.py / epic.py


# ---- construction / serialisation: same dict formats as tools/lfb_loader.py -------------------------------------
def construct_ava_lfb(all_features, all_metadata):
    """[iter][gpu] feature arrays (R, 2048[,1,1,1]) + metadata (R, 4) = (video_id, sec, ., .) -> {video: {sec: [rows]}}
    (tools/lfb_loader.py:82-113)."""
    lfb = {}
    for iter_features, iter_metadata in zip(all_features, all_metadata):
        for feats, meta in zip(iter_features, iter_metadata):
            assert feats.shape[0] == meta.shape[0]
            ids = np.round(np.asarray(meta)[:, :2]).astype(np.int64)
            for i in range(feats.shape[0]):
                lfb.setdefault(int(ids[i, 0]), {}).setdefault(int(ids[i, 1]), []).append(np.squeeze(feats[i]))
    return lfb


def construct_frame_level_lfb(all_features, all_metadata):
    """Charades / EPIC: one feature per sampled frame -> {video: {frame: row}} (tools/lfb_loader.py:51-79)."""
    lfb = {}
    n = 0
    for iter_features in all_features:
        for feats in iter_features:
            for i in range(feats.shape[0]):
                if n >= len(all_metadata):
                    break
                md = all_metadata[n]
                video_id, frame_id = (md[0], md[1]) if len(md) == 2 else (md[1], md[2])
                n += 1
                lfb.setdefault(video_id, {})[frame_id] = np.squeeze(feats[i])
    return lfb


def load_lfb(path):
    """Pickle written by the reference (python 2) or by write_lfb."""
    with open(path, 'rb') as f:
        return pickle.load(f, encoding='latin1')


def write_lfb(lfb, path):
    with open(path, 'wb') as f:
        pickle.dump(lfb, f, 2)           # protocol 2: readable by the reference's python 2


# ---- the device bank ------------------------------------------------------------------------------------------------
class DeviceLfb(object):
    """Packs {video: {key: row | [rows]}} into one [rows, dim] device tensor; `start[video][key] = (first_row, count)`."""

    def __init__(self, lfb, dim, device=None, dtype=None):
        from vlfb import executor as X
        self.dim = int(dim)
        self.start = {}
        rows = []
        n = 0
        for video in lfb:
            per = {}
            for key, val in lfb[video].items():
                feats = val if isinstance(val, list) else ([] if (isinstance(val, np.ndarray) and val.size == 0) else
                                                           (list(val) if np.ndim(val) == 2 else [val]))
                per[key] = (n, len(feats))
                for f in feats:
                    rows.append(np.asarray(f, dtype=np.float32).reshape(self.dim))
                n += len(feats)
            self.start[video] = per
        host = torch.from_numpy(np.stack(rows) if rows else np.zeros((0, self.dim), np.float32))
        self.rows = n
        self.bank = host.to(dtype or X.DTYPE).to(device or X.DEVICE)
        self._idx_dev = {}

    def nbytes(self):
        return self.bank.numel() * self.bank.element_size()

    # -- index tables: the reference's sampling rules, emitting bank row numbers instead of copying rows
    def sample_indices_ava(self, video_idx, sec, window_size, max_feat_per_step):
        """lib/datasets/ava.py:300-323 (np.random.choice per occupied second, in window order)."""
        K = int(max_feat_per_step)
        out = np.full((window_size * K,), -1, dtype=np.int32)
        video = self.start[video_idx]
        lower = sec - (window_size // 2)
        for j, si in enumerate(range(lower, lower + window_size)):
            if si in video:
                first, num_feat = video[si]
                used = min(num_feat, K)
                chosen = np.random.choice(range(num_feat), used, replace=False)
                out[j * K:j * K + used] = first + chosen
        return out

    def sample_indices_charades(self, video_idx, center_idx, window_size, clips_per_second):
        """lib/datasets/charades.py:251-276 (first WINDOW_SIZE stored frames inside the window, zero padded)."""
        video = self.start[video_idx]
        assert len(video) > 0
        secs = window_size // clips_per_second
        begin = int(np.round(center_idx - (float(secs) / 2.0 * FPS)))
        end = begin + secs * FPS
        out = np.full((window_size,), -1, dtype=np.int32)
        k = 0
        for frame_idx in range(begin, end + 1):
            if frame_idx in video and k < window_size:
                out[k] = video[frame_idx][0]
                k += 1
        return out

    def sample_indices_epic_verb(self, video_key, center_idx, window_size):
        """lib/datasets/epic.py:310-331."""
        video = self.start[video_key]
        half_len = (window_size * FPS) // 2
        out = np.full((window_size,), -1, dtype=np.int32)
        k = 0
        for frame_idx in range(center_idx - half_len, center_idx + half_len + 1):
            if frame_idx in video and k < window_size:
                out[k] = video[frame_idx][0]
                k += 1
        return out

    def sample_indices_epic_noun(self, video_key, center_idx, window_size, max_num_feat_per_frame, frames_per_second):
        """lib/datasets/epic.py:338-374: up to `max_num_feat_per_frame` detections of every stored frame inside the
        window, in frame order, until `window_size` rows are collected."""
        video = self.start[video_key]
        secs = float(window_size) / (max_num_feat_per_frame * frames_per_second)
        lower = int(center_idx - (secs / 2) * FPS)
        upper = int(lower + secs * FPS)
        out = np.full((window_size,), -1, dtype=np.int32)
        k = 0
        for frame_idx in range(lower, upper + 1):
            if frame_idx in video and video[frame_idx][1] > 0:
                first, count = video[frame_idx]
                take = min(max_num_feat_per_frame, count)
                fit = min(take, window_size - k)
                out[k:k + fit] = first + np.arange(fit, dtype=np.int32)
                k += take
                if k >= window_size:
                    break
        return out

    # -- device side
    def gather(self, index_table, out=None, tf32_out=False):
        """index_table int32 [R, L] (host numpy / tensor) -> device tensor [R, L, dim]."""
        from vlfb import executor as X
        idx = torch.as_tensor(np.ascontiguousarray(index_table), dtype=torch.int32)
        key = tuple(idx.shape)
        dev = self._idx_dev.get(key)
        if dev is None:
            dev = torch.empty(idx.shape, dtype=torch.int32, device=self.bank.device)
            self._idx_dev[key] = dev
        dev.copy_(idx, non_blocking=True)
        if out is None:
            out = torch.empty(tuple(idx.shape) + (self.dim,), dtype=self.bank.dtype, device=self.bank.device)
        X.K.lfb_gather(self.bank, dev.view(-1), out.view(-1, self.dim), tf32_out=tf32_out)
        return out

    def feed(self, blob_name, index_table):
        """Assemble the windows directly into the net's `lfb{suffix}` input blob (what FeedBlob(name, windows) would
        have produced, TF32 rounding of the GEMM operand included unless a B200.COMPUTE 'tf32x3' net reads it) -- R*L*4
        bytes cross PCIe instead of R*L*dim*4.
        In a B200.ROI_CAPACITY net the table is extended to C rows with -1 (zero windows), as FeedBlob pads."""
        from vlfb import workspace
        name = workspace._unscoped(blob_name)
        cap = workspace._roi_rows(name, np.shape(index_table))
        rows = int(np.shape(index_table)[0]) if cap is not None else None
        if cap is not None:
            table = np.full((cap,) + tuple(np.shape(index_table)[1:]), -1, dtype=np.int32)
            table[:rows] = np.asarray(index_table)
            index_table = table
        shape = tuple(np.shape(index_table)) + (self.dim,)
        dst = workspace._static(name, shape, self.bank.dtype)
        rnd = not workspace.feeds_unrounded(name)
        self.gather(index_table, out=dst, tf32_out=rnd)
        workspace.bank_companion(name, dst)                  # B200.LFB_DTYPE 'bf16': the scan operand of the folded FBO
        if cap is not None:
            workspace.set_live_rows(name, rows)
        ws = workspace.current()
        ws.blobs[name] = dst
        workspace._mark_rounded(name, rnd)
        return dst
