"""Launch audit (tests/launch_audit.py) of B200.GPUS_PER_STEP nets: the same audit, extended to the segmented kernels
of include/vlfb_seg.h, which a packed training step calls in place of the sigmoid loss and SpatialBN.  Each segmented
call is held, segment by segment, to the fp64 reference and bound of its unsegmented twin:
  * sigmoid_ce_seg_fwd: the sum of the segments' losses, with the segments' bounds plus the fp32 additions;
  * sigmoid_ce_seg_bwd: each segment's rows against that segment's reference;
  * spatial_bn_seg_fwd / _bwd: each segment's rows and statistics against the reference over that segment alone (chain
    length = the segment's rows, which bounds the default form's slab order and the fixed-order form alike); the
    running statistics against segment 0's; ds / db against the segments' terms added in order.
Every other call is audited exactly as launch_audit.py audits it.

    python tests/launch_audit_seg.py --net NAME --out FILE      (NAME: a net of NETS below)
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import launch_audit as LA  # noqa: E402
import streaming_cases as SC  # noqa: E402

SEG_WRAPPERS = ('sigmoid_ce_seg_fwd', 'sigmoid_ce_seg_bwd', 'spatial_bn_seg_fwd', 'spatial_bn_seg_bwd')
# two virtual GPUs of one clip each, the two clips launch_audit.run_net feeds (their RoIs: batch indices 0, 0, 1, 1)
PACKED = ['NUM_GPUS', 2, 'TRAIN.BATCH_SIZE', 2, 'B200.GPUS_PER_STEP', 2]
SEG_LOSS = {'sigmoid_ce_seg_fwd', 'sigmoid_ce_seg_bwd'}
BN_SEG = {'spatial_bn_seg_fwd', 'spatial_bn_seg_bwd'}
AVA_PACKED_WRAPPERS = (LA.AVA_TRAIN_WRAPPERS - {'sigmoid_ce_fwd', 'sigmoid_ce_bwd'}) | SEG_LOSS

# name -> (yaml, overrides, split, runs, wrappers the net must reach, extra settings), as launch_audit.NETS
NETS = {
    'ava_train_packed': ('ava_r50_lfb_nl.yaml', LA.TINY + PACKED, 'train', 2, AVA_PACKED_WRAPPERS, {}),
    'ava_train_packed_capacity': ('ava_r50_lfb_nl.yaml', LA.TINY + PACKED + ['B200.ROI_CAPACITY', 8], 'train', 2,
                                  AVA_PACKED_WRAPPERS, {}),
    'resnext_bn_train_packed': ('ava_r50_lfb_nl.yaml', LA.TINY + LA.RESNEXT + PACKED, 'train', 2,
                                {'conv_fwd', 'conv_dgrad', 'conv_wgrad', 'sgd_nesterov'} | SEG_LOSS | BN_SEG,
                                {'grouped': True}),
    'resnext_bn_train_packed_det': ('ava_r50_lfb_nl.yaml', LA.TINY + LA.RESNEXT + PACKED + ['B200.DETERMINISTIC', True],
                                    'train', 2, {'conv_fwd', 'conv_dgrad', 'conv_wgrad_det', 'colsum_det',
                                                 'sgd_nesterov'} | SEG_LOSS | BN_SEG, {'grouped': True}),
}

OUT = {
    'sigmoid_ce_seg_fwd': ((), ('loss',)), 'sigmoid_ce_seg_bwd': ((), ('dlogits',)),
    'spatial_bn_seg_fwd': (('rm', 'rv'), ('sm', 'siv', 'y')), 'spatial_bn_seg_bwd': (('ds', 'db'), ('dx',)),
}


def _segments(seg, rows):
    """Row ranges of the segments, as the kernels take them: the first from row 0, the last to the end."""
    s = [int(v) for v in seg.view(-1).tolist()]
    s[0], s[-1] = 0, rows
    out = []
    for j in range(len(s) - 1):
        r0 = min(max(s[j], 0), rows)
        out.append((r0, min(max(s[j + 1], r0), rows)))
    return out


def _sigmoid_ce_seg(c):
    b, a = c.b, c.a
    x, t, scale = LA._d(b['logits']), b['targets'], float(b['scale'])
    x2, t2 = x.reshape(x.shape[0], -1), t.reshape(t.shape[0], -1)
    parts = [(r0, r1) for r0, r1 in _segments(b['seg'], x.shape[0]) if r1 > r0]
    if c.fn == 'sigmoid_ce_seg_fwd':
        total = torch.zeros(1, dtype=x.dtype, device=x.device)
        bound = torch.zeros_like(total)
        for r0, r1 in parts:
            r, bd = SC.sigmoid_ce_fwd_ref(x2[r0:r1], t2[r0:r1], scale)
            bound = bound + bd + SC.U * (total.abs() + r.abs())       # one fp32 addition per segment
            total = total + r
        return [('loss', a['loss'].reshape(-1)[:1], total, bound)]
    dl = float(b['dloss'].view(-1)[0]) if b['dloss'] is not None else 1.0
    out = []
    for j, (r0, r1) in enumerate(parts):
        r, bd = SC.sigmoid_ce_bwd_ref(x2[r0:r1], t2[r0:r1], scale, dl)
        out.append(('dlogits[seg %d]' % j, a['dlogits'].reshape(x2.shape)[r0:r1], r, bd))
    return out


def _bn_seg_fwd(c):
    b, a = c.b, c.a
    C_, S = b['x'].shape[-1], int(b['segments'])
    xd = LA._d(b['x']).reshape(-1, C_)
    n = xd.shape[0] // S
    eps, mom = float(np.float32(b['eps'])), float(np.float32(b['momentum']))
    y = a['y'].reshape(-1, C_)
    out = []
    for j in range(S):
        run = (LA._d(b['rm']), LA._d(b['rv']), mom) if (j == 0 and b['rm'] is not None) else ()
        r = SC.bn_fwd_ref(xd[j * n:(j + 1) * n], LA._d(b['s']), LA._d(b['b']), n, eps, *run)
        out += [('y[seg %d]' % j, y[j * n:(j + 1) * n], *r['y']), ('sm[seg %d]' % j, a['sm'][j], *r['sm']),
                ('siv[seg %d]' % j, a['siv'][j], *r['siv'])]
        out += [(k, a[k], *r[k]) for k in ('rm', 'rv') if k in r]
    return out


def _bn_seg_bwd(c):
    b, a = c.b, c.a
    C_, S = b['x'].shape[-1], int(b['segments'])
    xd, dyd = LA._d(b['x']).reshape(-1, C_), LA._d(b['dy']).reshape(-1, C_)
    n = xd.shape[0] // S
    dx = a['dx'].reshape(-1, C_)
    ds = None if b['ds'] is None else LA._d(b['ds'])
    db = None if b['db'] is None else LA._d(b['db'])
    dsb = dbb = 0.0
    out = []
    for j in range(S):
        sl = slice(j * n, (j + 1) * n)
        r = SC.bn_bwd_refb(dyd[sl], xd[sl], LA._d(b['s']), LA._d(b['sm'][j]), LA._d(b['siv'][j]), n, ds, db)
        out.append(('dx[seg %d]' % j, dx[sl], *r['dx']))
        if ds is not None:
            ds, dsb = r['ds'][0], dsb + r['ds'][1]
        if db is not None:
            db, dbb = r['db'][0], dbb + r['db'][1]
    if ds is not None:
        out.append(('ds', a['ds'], ds, dsb))
    if db is not None:
        out.append(('db', a['db'], db, dbb))
    return out


def install(patch=setattr):
    """Extend launch_audit in place (patch(obj, name, value): setattr, or a test's monkeypatch.setattr)."""
    patch(LA, 'AUDITED', LA.AUDITED + SEG_WRAPPERS)
    patch(LA, '_OUT', dict(LA._OUT, **OUT))
    patch(LA, 'REF', dict(LA.REF, sigmoid_ce_seg_fwd=_sigmoid_ce_seg, sigmoid_ce_seg_bwd=_sigmoid_ce_seg,
                          spatial_bn_seg_fwd=_bn_seg_fwd, spatial_bn_seg_bwd=_bn_seg_bwd))
    patch(LA, 'NETS', dict(LA.NETS, **NETS))


if __name__ == '__main__':
    install()
    sys.exit(LA.main())
