"""TEST-ONLY: CPU stand-ins for the segmented kernels of B200.GPUS_PER_STEP (include/vlfb_seg.h), added to a torch-CPU
kernel module (tests/fake_kernels.py, or resnext_oracle's) without editing it.

Each stand-in runs the base module's unsegmented function once per segment, which is what the CUDA kernels compute:
the sigmoid loss per row segment (seg = int [S + 1] row offsets; the first segment also owns the rows before seg[1],
the last the rows up to the end), SpatialBN per segment of rows // S rows with the running statistics taken from
segment 0, and dscale / dbias added one segment at a time."""
import types

import torch


def _bounds(seg, rows):
    s = [int(v) for v in seg.tolist()]
    s[0], s[-1] = 0, rows
    return [(min(max(s[j], 0), rows), min(max(s[j + 1], s[j]), rows)) for j in range(len(s) - 1)]


def kernels(base):
    """A module with every function of `base` and the segmented kernels."""
    mod = types.ModuleType(base.__name__ + '_seg')
    mod.__dict__.update(vars(base))

    def sigmoid_ce_seg_fwd(logits, targets, seg, loss, scale):
        total = torch.zeros(1, dtype=loss.dtype)
        part = torch.empty(1, dtype=loss.dtype)
        for r0, r1 in _bounds(seg, logits.shape[0]):
            if r1 > r0:
                base.sigmoid_ce_fwd(logits[r0:r1], targets[r0:r1], part, scale)
            else:
                part.zero_()
            total += part
        loss.copy_(total)

    def sigmoid_ce_seg_bwd(logits, targets, seg, dloss, dlogits, scale):
        for r0, r1 in _bounds(seg, logits.shape[0]):
            if r1 > r0:
                base.sigmoid_ce_bwd(logits[r0:r1], targets[r0:r1], dloss, dlogits[r0:r1], scale)

    def _rows(t, S):
        c = t.shape[-1]
        t2 = t.reshape(-1, c)
        assert t2.shape[0] % S == 0
        return t2, t2.shape[0] // S

    def spatial_bn_seg_fwd(x, s, b, rm, rv, sm, siv, y, eps, momentum, segments, det=False):
        x2, n = _rows(x, segments)
        y2 = torch.empty_like(x2)
        for j in range(segments):
            keep = j == 0
            base.spatial_bn_fwd(x2[j * n:(j + 1) * n], s, b, rm if keep else None, rv if keep else None, sm[j], siv[j],
                                y2[j * n:(j + 1) * n], eps, momentum)
        y.copy_(y2.view(y.shape))

    def spatial_bn_seg_bwd(dy, x, s, sm, siv, dx, ds, db, segments, det=False):
        x2, n = _rows(x, segments)
        d2, _ = _rows(dy.contiguous(), segments)
        dx2 = torch.empty_like(x2)
        for j in range(segments):
            base.spatial_bn_bwd(d2[j * n:(j + 1) * n], x2[j * n:(j + 1) * n], s, sm[j], siv[j], dx2[j * n:(j + 1) * n],
                                ds, db)
        dx.copy_(dx2.view(dx.shape))

    mod.sigmoid_ce_seg_fwd, mod.sigmoid_ce_seg_bwd = sigmoid_ce_seg_fwd, sigmoid_ce_seg_bwd
    mod.spatial_bn_seg_fwd, mod.spatial_bn_seg_bwd = spatial_bn_seg_fwd, spatial_bn_seg_bwd
    return mod


def install(base):
    """Route vlfb.executor onto kernels(base) and the CPU device (fp64); returns that module."""
    from vlfb import executor
    mod = kernels(base)
    executor.set_backend(mod, 'cpu', torch.float64)
    return mod
