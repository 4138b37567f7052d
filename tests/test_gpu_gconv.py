"""Grouped convolution on the GPU (csrc/gconv.cu through vlfb_gemm with groups > 1): the case table of
tests/gconv_cases.py elementwise against fp64, and ResNeXt-50 32x4d (RESNETS.NUM_GROUPS 32, WIDTH_PER_GROUP 4) nets
through the builder API against the fp64 oracle, with the tolerances of tests/test_gpu_model.py."""
import numpy as np
import pytest
import torch

import harness as H
import resnext_oracle as RO
from test_gpu_model import FULL, TINY, _oracle, _train_case, ws  # noqa: F401  (ws: the fixture)
from util import run_worker

pytestmark = pytest.mark.gpu

RESNEXT = ['RESNETS.NUM_GROUPS', 32, 'RESNETS.WIDTH_PER_GROUP', 4]


def test_case_table():
    """Every case of the table in its own process (VLFB_DEBUG is read once per process): bound, guard bands, sign
    bits and the path record.  Prints each case's bound ratio (max |got - ref| / bound) and the worst per family."""
    proc, recs = run_worker('gconv_cases.py', [], timeout=1800)
    assert proc.returncode == 0, proc.stderr[-4000:]
    import gconv_cases as GC
    assert len(recs) == len(GC.CASES)
    worst = {}
    for r in recs:
        print('%-34s ratio %.3f %s' % (r['name'], r['ratio'], '' if r['ok'] else 'FAIL %s' % r))
        if r['ratio'] > worst.get(r['family'], (-1, ''))[0]:
            worst[r['family']] = (r['ratio'], r['name'])
    for fam, (ratio, name) in sorted(worst.items()):
        print('worst %-12s %.3f (%s)' % (fam, ratio, name))
    bad = [r['name'] for r in recs if not r['ok']]
    assert not bad, bad


def test_tiny_resnext_fbo_nl_train_step(ws):  # noqa: F811
    with RO.grouped():
        _train_case(ws, 'ava_r50_lfb_nl.yaml', TINY + RESNEXT, 64, 8, 2)


def test_tiny_resnext_gradients_vs_tf32_emulating_oracle(ws):  # noqa: F811
    """The same step against the oracle that rounds operands at the engine's TF32 points (test_gpu_model's
    tolerances: TF32 noise still flips ReLUs, so norms are bounded, not bit patterns)."""
    from test_gpu_model import FWD_TOL, GRAD_COS_TOL, GRAD_L2_TOL, GRAD_MEDIAN_L2_TOL
    ov = TINY + RESNEXT
    with RO.grouped() as OM:
        H.setup_cfg('ava_r50_lfb_nl.yaml', ov)
        ocfg = H.oracle_cfg('ava_r50_lfb_nl.yaml', ov)
        params = OM.make_params(ocfg, seed=2)
        inputs = OM.make_inputs(ocfg, n_clips=2, rois_per_clip=2, crop=64, frames=8)
        model, sfx = H.build('train', True)
        H.feed_params(params)
        H.feed_inputs(inputs, sfx)
        p64, blobs, loss = _oracle(ocfg, params, inputs, 'train', True, emulate_tf32=True)
    net = ws.current().nets[model.net.Proto().name]
    upd, net.update_ops = net.update_ops, []
    ws.RunNet(model.net.Proto().name)
    torch.cuda.synchronize()
    net.update_ops = upd
    assert H.rel(ws.FetchBlob('gpu_0/loss'), loss.item()) < FWD_TOL
    assert H.rel(ws.FetchBlob('gpu_0/pred'), blobs['pred'].detach().numpy()) < FWD_TOL
    errs = []
    for name in model.TrainableParams():
        ref = p64[name].grad.numpy()
        nref = float(np.linalg.norm(ref))
        if nref < 1e-7:
            continue
        g = ws.FetchBlob('gpu_0/' + name + '_grad').astype(np.float64)
        e = float(np.linalg.norm(g - ref) / nref)
        cos = float((g * ref).sum() / (np.linalg.norm(g) * nref + 1e-30))
        assert e < GRAD_L2_TOL and cos > GRAD_COS_TOL, (name, e, cos)
        errs.append(e)
    print('\nResNeXt vs TF32-emulating oracle: median grad rel-L2 %.2e, worst %.2e' % (np.median(errs), max(errs)))
    assert float(np.median(errs)) < GRAD_MEDIAN_L2_TOL


def test_tiny_resnext_spatial_bn_variant(ws):  # noqa: F811
    """SpatialBN nets: the grouped conv stores fp32 sums (no fused affine / ReLU) for the batch norm that follows.  A
    batch-normalised random net amplifies TF32-level noise about 100x where the Affine net damps it, so the bounds are
    those of test_spatial_bn.test_tiny_bn_train_step_on_gpu (loss 5e-3, last blobs 6e-2, gradient cosine)."""
    bn = ['MODEL.USE_AFFINE', False, 'NONLOCAL.USE_AFFINE', False, 'NONLOCAL.USE_BN', True,
          'MODEL.DILATIONS_AFTER_CONV5', False]
    ov = TINY + RESNEXT + bn
    with RO.grouped() as OM:
        H.setup_cfg('ava_r50_lfb_nl.yaml', ov)
        ocfg = H.oracle_cfg('ava_r50_lfb_nl.yaml', ov)
        params = OM.make_params(ocfg, seed=2)
        inputs = OM.make_inputs(ocfg, n_clips=2, rois_per_clip=2, crop=64, frames=8)
        model, sfx = H.build('train', True)
        H.feed_params(params)
        H.feed_inputs(inputs, sfx)
        p64, blobs, loss = _oracle(ocfg, params, inputs, 'train', True)
    net = ws.current().nets[model.net.Proto().name]
    upd, net.update_ops = net.update_ops, []
    ws.RunNet(model.net.Proto().name)
    torch.cuda.synchronize()
    net.update_ops = upd
    rep = dict((b, H.rel(ws.FetchBlob('gpu_0/' + b), blobs[b].detach().numpy()))
               for b in ('res2_2_branch2c_bn', 'res5_2_branch2c_bn', 'box_pooled', 'pred'))
    cos = []
    for name in model.TrainableParams():
        g = ws.FetchBlob('gpu_0/' + name + '_grad').astype(np.float64).ravel()
        ref = p64[name].grad.numpy().ravel()
        if np.abs(ref).max() < 1e-12:
            continue
        cos.append(float(g @ ref / (np.linalg.norm(g) * np.linalg.norm(ref) + 1e-300)))
    print('\nResNeXt SpatialBN: loss %.1e, %s; gradient cosine min %.4f median %.5f' % (
        H.rel(ws.FetchBlob('gpu_0/loss'), loss.item()), ' '.join('%s=%.1e' % kv for kv in rep.items()), min(cos),
        float(np.median(cos))))
    assert H.rel(ws.FetchBlob('gpu_0/loss'), loss.item()) < 5e-3
    assert rep['res2_2_branch2c_bn'] < 4e-3 and all(v < 6e-2 for v in rep.values()), rep
    assert min(cos) > 0.9 and float(np.median(cos)) > 0.95, (min(cos), float(np.median(cos)))


def test_tiny_resnext_val_split_with_folded_fbo(ws):  # noqa: F811
    from core.config import config as cfg
    from vlfb import executor as X
    ov = TINY + RESNEXT
    with RO.grouped() as OM:
        H.setup_cfg('ava_r50_lfb_nl.yaml', ov)
        ocfg = H.oracle_cfg('ava_r50_lfb_nl.yaml', ov)
        params = OM.make_params(ocfg, seed=2, split='val')
        inputs = OM.make_inputs(ocfg, n_clips=2, rois_per_clip=3, crop=64, frames=8)
        p64 = dict((k, v.double()) for k, v in params.items())
        i64 = dict((k, (v.double() if v.dtype == torch.float32 else v)) for k, v in inputs.items())
        blobs, _, _ = OM.forward(ocfg, p64, i64, 'val')
    assert cfg.B200.get('FBO_FOLD', True)
    model, sfx = H.build('val', False)
    H.feed_params(params)
    H.feed_inputs(inputs, sfx)
    ws.RunNet(model.net.Proto().name)
    net = ws.current().nets[model.net.Proto().name]
    assert any(isinstance(st, X.FboFoldStep) for st in net.steps)
    assert any(isinstance(st, X.ConvStep) and st.groups == 32 for st in net.steps)
    for b in ('box_pooled', 'pred', 'prob'):
        assert H.rel(ws.FetchBlob('gpu_0/' + b), blobs[b].numpy()) < 1e-3, b


def test_full_size_resnext50_32x4d_forward_backward(ws):  # noqa: F811
    """2 clips of 32 x 224^2 through ResNeXt-50 32x4d + FBO-NL: every branch2b conv runs on csrc/gconv.cu."""
    with RO.grouped():
        _train_case(ws, 'ava_r50_lfb_nl.yaml', FULL + RESNEXT, 224, 32, 2, check_all_grads=False)
