"""B200.COMPUTE 'tf32x3' on the fp64 CPU engine (tests/fake_kernels.py with EMULATE_TF32 on, so that every TF32 rounding
the CUDA path makes is performed; its GEMM wrappers take `precision` through tests/fake_kernels_x3.py).  A 'tf32x3' net rounds nothing and passes precision = PREC_X3 to every tensor-core
GEMM, so under the stand-in (exact products) its step must equal the PLAIN fp64 oracle -- the bounds of
test_engine_cpu._run: loss and blobs 1e-9, every gradient 1e-7, in both gradient-sum schedules -- where the same step of a
'tf32' net misses.  Also: the calls such a net makes (and a 'tf32' net does not), the errors CreateNet / RunNet raise,
and the other B200 options combined with the mode."""
import inspect

import numpy as np
import pytest
import torch

import harness as H
import test_engine_cpu as E

TINY = E.TINY
X3 = ['B200.COMPUTE', 'tf32x3']
YAML = 'ava_r50_lfb_nl.yaml'
CHARADES = TINY + ['MODEL.NUM_CLASSES', 157]
EPIC = TINY + ['DATASET', 'epic', 'MODEL.NUM_CLASSES', 125, 'MODEL.MULTI_LABEL', False]
AVA_BLOBS = ['pool1', 'res2_2_branch2c_bn', 'nonlocal_conv3_1_sum', 'res3_3_branch2c_bn', 'nonlocal_conv4_1_sum',
             'res5_2_branch2c_bn', 'blob_pooled', 'roi_feat_3d', 'box_pooled', 'lfb_1x1', 'lfb_nl0_affinity_prob',
             'lfb_nl1_sum', 'pool5', 'pred', 'prob']
GEMMS = ('conv_fwd', 'conv_dgrad', 'conv_wgrad', 'conv_wgrad_det', 'matmul', 'matmul_det')
ROUNDING = ('round_tf32', 'add_tf32', 'relu_tf32', 'relu_bwd_tf32', 'add_relu_bwd_tf32')
RECORDED = GEMMS + ROUNDING + ('weight_transpose_multi', 'nc_to_cl', 'lfb_gather', 'softmax_fwd',
                               'softmax_bwd', 'maxpool_bwd_gather', 'fbo_bank_scan')
SGD_PARAMS = ['conv1_w', 'res4_3_branch2b_w', 'nonlocal_conv4_1_theta_b', 'lfb_nl1_out_w', 'pred_w', 'pred_b']
DET = {'conv_wgrad': 'conv_wgrad_det', 'matmul': 'matmul_det', 'colsum': 'colsum_det',
       'roi_align_bwd': 'roi_align_bwd_det', 'spatial_bn_fwd': 'spatial_bn_fwd_det', 'spatial_bn_bwd': 'spatial_bn_bwd_det'}


@pytest.fixture
def fake(monkeypatch):
    import fake_kernels
    import fake_kernels_x3
    from vlfb import workspace
    monkeypatch.setattr(fake_kernels, 'EMULATE_TF32', True)
    mod = fake_kernels_x3.install(fake_kernels)
    for base, det in DET.items():              # the deterministic stand-ins compute the same function
        monkeypatch.setattr(mod, det, getattr(mod, base), raising=False)
    workspace.ResetWorkspace()
    yield mod
    workspace.ResetWorkspace()
    fake_kernels.uninstall()


def _record(monkeypatch, mod):
    """calls: [(wrapper, explicit keyword arguments, every argument bound with the defaults)] of the RECORDED wrappers."""
    calls = []

    def wrap(name, f):
        sig = inspect.signature(f)

        def g(*a, **kw):
            b = sig.bind(*a, **kw)
            b.apply_defaults()
            calls.append((name, dict(kw), dict(b.arguments)))
            return f(*a, **kw)
        return g
    for name in RECORDED:
        f = getattr(mod, name, None)
        if f is not None:
            monkeypatch.setattr(mod, name, wrap(name, f))
    return calls


def _oracle(yaml_name, ov, split='train', lfb_infer_only=False, rois_per_clip=2):
    from oracle import model as OM
    ocfg = H.oracle_cfg(yaml_name, ov)
    params = OM.make_params(ocfg, seed=2) if split == 'train' else \
        OM.make_params(ocfg, seed=2, split=split, lfb_infer_only=lfb_infer_only)
    inputs = OM.make_inputs(ocfg, n_clips=2, rois_per_clip=rois_per_clip, crop=64, frames=8)
    p64 = dict((k, v.double().requires_grad_(split == 'train')) for k, v in params.items())
    i64 = dict((k, (v.double() if v.dtype == torch.float32 else v)) for k, v in inputs.items())
    blobs, _, loss = OM.forward(ocfg, p64, i64, split, lfb_infer_only=lfb_infer_only)
    if split == 'train':
        loss.backward()
    return params, inputs, p64, blobs, loss


def _worst_grad(model, p64):
    from vlfb import workspace
    worst = 0.0
    for name in model.TrainableParams():
        ref = p64[name].grad.numpy()
        g = workspace.FetchBlob('gpu_0/' + name + '_grad')
        worst = max(worst, float(np.abs(g - ref).max() / max(np.abs(ref).max(), 1e-5)))
    return worst


# ------------------------------------------------------------------------------------------------ exactness
def _sgd_matches(model, params, p64):
    from core.config import config as cfg
    from oracle import ops as O
    from vlfb import workspace
    model.UpdateWorkspaceLr(10)
    lr = float(workspace.FetchBlob('gpu_0/lr'))
    workspace.RunNet(model.net.Proto().name)
    names = [n for n in SGD_PARAMS if n in model.TrainableParams()]
    assert names
    for name in names:                              # the parameters and bounds of test_engine_cpu's SGD check
        p_ref, m_ref = O.nesterov_update(params[name].double(), p64[name].grad, torch.zeros_like(p64[name]), lr,
                                         cfg.SOLVER.MOMENTUM, cfg.SOLVER.WEIGHT_DECAY)
        assert H.rel(workspace.FetchBlob('gpu_0/' + name), p_ref.detach().numpy()) < 1e-5, name
        assert H.rel(workspace.FetchBlob('gpu_0/' + name + '_momentum'), m_ref.detach().numpy()) < 1e-4, name


@pytest.mark.parametrize('case', ['ava', 'ava_no_stack', 'charades', 'epic_softmax'])
def test_x3_train_step_equals_the_plain_fp64_oracle(fake, case):
    """Forward blobs, loss and every gradient of both runs (lazy sums; the grad-finish fusion), then one SGD step."""
    yaml_name, ov, blobs = {'ava': (YAML, TINY, AVA_BLOBS), 'ava_no_stack': (YAML, TINY + ['B200.FBO_STACK', False], AVA_BLOBS),
                            'charades': ('charades_r50_lfb_nl.yaml', CHARADES, ['pool5', 'pred']),
                            'epic_softmax': ('charades_r50_lfb_nl.yaml', EPIC, ['pool5', 'pred'])}[case]
    model, params, p64, worst = E._run(yaml_name, ov + X3, fake, blobs, reps=2)
    print('%s: worst gradient error %.2e' % (case, worst))
    _sgd_matches(model, params, p64)


def test_tf32_train_step_misses_the_plain_oracle(fake):
    """Negative control: the same step of a 'tf32' net, roundings emulated, is TF32-accurate only."""
    from vlfb import workspace
    params, inputs, p64, _, loss = _oracle(YAML, TINY)
    H.setup_cfg(YAML, TINY)
    model, sfx = H.build('train', True)
    H.feed_params(params)
    H.feed_inputs(inputs, sfx)
    workspace.current().nets[model.net.Proto().name].update_ops = []
    workspace.RunNet(model.net.Proto().name)
    worst = _worst_grad(model, p64)
    print('tf32: loss error %.2e, worst gradient error %.2e' % (H.rel(workspace.FetchBlob('gpu_0/loss'), loss.item()), worst))
    assert worst > 1e-7


@pytest.mark.parametrize('infer_only', [False, True], ids=['val_fold', 'lfb_infer_only'])
def test_x3_test_nets_equal_the_plain_fp64_oracle(fake, infer_only):
    from vlfb import executor as X
    from vlfb import workspace
    params, inputs, _, blobs, _ = _oracle(YAML, TINY, 'val', infer_only, rois_per_clip=3)
    H.setup_cfg(YAML, TINY + X3)
    model, sfx = H.build('val', False, lfb_infer_only=infer_only)
    H.feed_params(dict((k, v) for k, v in params.items() if workspace.HasBlob(k)))
    H.feed_inputs(inputs, sfx)
    net = workspace.current().nets[model.net.Proto().name]
    assert sum(isinstance(s, X.FboFoldStep) for s in net.steps) == (0 if infer_only else 2)
    workspace.RunNet(model.net.Proto().name)
    names = ['box_pooled'] if infer_only else ['box_pooled', 'lfb_nl0_affinity_prob', 'lfb_nl1_sum', 'pred', 'prob']
    for b in names:
        got = workspace.FetchBlob('gpu_0/' + b).reshape(-1)
        assert H.rel(got, blobs[b].detach().numpy().reshape(-1)) < 1e-9, b


# ------------------------------------------------------------------------------------------------ call record
def _feed_bank(sfx, inputs):
    """The AVA bank through DeviceLfb.feed (the device gather) instead of FeedBlob."""
    from datasets.lfb_bank import DeviceLfb
    R, L_, D = inputs['lfb'].shape
    rows = inputs['lfb'].reshape(-1, D).double().numpy()
    bank = DeviceLfb({0: dict((i, rows[i]) for i in range(rows.shape[0]))}, D)
    bank.feed('gpu_0/lfb' + sfx, np.arange(R * L_, dtype=np.int32).reshape(R, L_))


def _record_steps(fake, monkeypatch, compute):
    """Every recorded call of: a train net (as-written FBO-NL graph: BatchMatMul / Softmax steps) fed the bank through
    DeviceLfb, two runs and an SGD step, then a val net with the folded FBO."""
    from vlfb import workspace
    calls = _record(monkeypatch, fake)
    params, inputs, _, _, _ = _oracle(YAML, TINY)
    H.setup_cfg(YAML, TINY + ['B200.FBO_STACK', False, 'B200.COMPUTE', compute])
    model, sfx = H.build('train', True)
    H.feed_params(params)
    H.feed_inputs(inputs, sfx)
    _feed_bank(sfx, inputs)
    model.UpdateWorkspaceLr(10)
    for _ in range(3):
        workspace.RunNet(model.net.Proto().name)
    vparams, vinputs, _, _, _ = _oracle(YAML, TINY, 'val')
    vmodel, vsfx = H.build('val', False)
    H.feed_params(dict((k, v) for k, v in vparams.items() if workspace.HasBlob(k)))
    H.feed_inputs(vinputs, vsfx)
    workspace.RunNet(vmodel.net.Proto().name)
    return calls


def test_x3_net_calls(fake, monkeypatch):
    from vlfb import libvlfb as L
    calls = _record_steps(fake, monkeypatch, 'tf32x3')
    names = set(c[0] for c in calls)
    assert {'conv_fwd', 'conv_dgrad', 'conv_wgrad', 'matmul', 'weight_transpose_multi', 'nc_to_cl', 'lfb_gather',
            'softmax_fwd', 'fbo_bank_scan'} <= names, names
    assert not _rounding_calls(calls), set(c[0] for c in _rounding_calls(calls))
    assert sum(c[0] == 'weight_transpose_multi' for c in calls) == 3       # one per step: no per-conv transposes
    for name, kw, args in calls:
        if name in GEMMS or name == 'weight_transpose_multi':
            assert args['precision'] == L.PREC_X3, (name, kw)
        if 'tf32_out' in args:
            assert not args['tf32_out'], (name, kw)


def _rounding_calls(calls):
    """Calls of the rounding wrappers, except the ParamStore's refresh of its TF32 copy Pt (a fed parameter)."""
    from vlfb import workspace
    pt = set(ch['Pt'].untyped_storage().data_ptr() for ch in workspace.current().params.chunks)
    return [c for c in calls if c[0] in ROUNDING and not (c[0] == 'round_tf32' and
                                                          c[2]['y'].untyped_storage().data_ptr() in pt)]


def test_tf32_net_calls_carry_no_precision(fake, monkeypatch):
    calls = _record_steps(fake, monkeypatch, 'tf32')
    assert calls and not [c for c in calls if 'precision' in c[1]]
    assert {'round_tf32', 'relu_bwd_tf32'} <= set(c[0] for c in calls)


# ------------------------------------------------------------------------------------------------ errors
def test_input_fed_before_the_x3_net_was_created_is_refused(fake):
    from vlfb import workspace
    from vlfb.libvlfb import VlfbError
    params, inputs, _, _, _ = _oracle(YAML, TINY)
    H.setup_cfg(YAML, TINY + X3)
    H.feed_inputs(inputs, '_train')                 # stored TF32-rounded: no net has registered the names yet
    model, sfx = H.build('train', True)
    H.feed_params(params)
    with pytest.raises(VlfbError, match='data_train'):
        workspace.RunNet(model.net.Proto().name)
    H.feed_inputs(inputs, sfx)                      # fed again after CreateNet: unrounded
    workspace.RunNet(model.net.Proto().name)


@pytest.mark.parametrize('first', ['tf32', 'tf32x3'])
def test_input_read_by_nets_of_both_modes_is_refused(fake, first):
    from vlfb.libvlfb import VlfbError
    second = 'tf32' if first == 'tf32x3' else 'tf32x3'
    H.setup_cfg(YAML, TINY + ['B200.COMPUTE', first])
    H.build('train', True)
    H.setup_cfg(YAML, TINY + ['B200.COMPUTE', second])
    with pytest.raises(VlfbError, match="data_train.*B200.COMPUTE = '%s'" % first):
        H.build('train', True)
    H.build('val', False)                           # other inputs ('_test' suffix): no conflict


def test_bf16_bank_is_refused(fake):
    from vlfb.libvlfb import VlfbError
    H.setup_cfg(YAML, TINY + X3 + ['B200.LFB_DTYPE', 'bf16'])
    with pytest.raises(VlfbError, match='LFB_DTYPE'):
        H.build('val', False)


def test_fp32_stays_refused(fake):
    from vlfb.libvlfb import VlfbError
    H.setup_cfg(YAML, TINY + ['B200.COMPUTE', 'fp32'])
    with pytest.raises(VlfbError, match="'tf32' or 'tf32x3'"):
        H.build('train', True)


# ------------------------------------------------------------------------------------------------ combinations
def _train_vs_oracle(ov, runs=2, grouped=False):
    """Loss, pred and every gradient of `runs` runs of the tiny AVA train net against the plain fp64 oracle."""
    import contextlib
    import resnext_oracle as RO
    from vlfb import workspace
    with RO.grouped() if grouped else contextlib.nullcontext():
        params, inputs, p64, blobs, loss = _oracle(YAML, TINY + ov)
    H.setup_cfg(YAML, TINY + X3 + ov)
    model, sfx = H.build('train', True)
    net = workspace.current().nets[model.net.Proto().name]
    net.update_ops = []
    H.feed_params(params)
    H.feed_inputs(inputs, sfx)
    for _ in range(runs):
        workspace.RunNet(model.net.Proto().name)
        assert H.rel(workspace.FetchBlob('gpu_0/loss'), loss.item()) < 1e-9
        assert H.rel(workspace.FetchBlob('gpu_0/pred'), blobs['pred'].detach().numpy()) < 1e-9
        assert _worst_grad(model, p64) < 1e-7
    return net


def test_x3_deterministic(fake, monkeypatch):
    calls = _record(monkeypatch, fake)
    net = _train_vs_oracle(['B200.DETERMINISTIC', True])
    assert net.det and net.x3
    names = set(c[0] for c in calls)
    assert {'conv_wgrad_det', 'matmul_det'} <= names and not _rounding_calls(calls)


def test_x3_roi_capacity(fake, monkeypatch):
    """C = 8 RoI rows, 4 fed: the step still equals the oracle's on the 4 boxes."""
    import fake_kernels
    import fake_kernels_x3
    import fake_live_rows
    fake_live_rows.install(monkeypatch)
    fake_kernels_x3.install(fake_kernels)            # again: with the live-row wrappers
    net = _train_vs_oracle(['B200.ROI_CAPACITY', 8])
    assert net.roi_capacity == 8 and net.x3


def test_x3_resnext_with_spatial_bn(fake, monkeypatch):
    import launch_audit as LA
    from vlfb import executor as X
    import fake_kernels_x3
    import resnext_oracle as RO
    mod = fake_kernels_x3.install(RO)                # resnext_oracle's stand-in: conv wrappers with `groups`
    calls = _record(monkeypatch, mod)
    net = _train_vs_oracle(LA.RESNEXT, grouped=True)
    assert any(isinstance(st, X.SpatialBNStep) for st in net.steps) and net.x3
    assert not _rounding_calls(calls)
    assert any(c[1].get('groups', 1) > 1 for c in calls if c[0] == 'conv_fwd')


# ------------------------------------------------------------------------------------------------ launch audit
def test_x3_launch_audit_on_the_stand_in(monkeypatch):
    """tests/launch_audit_x3.py without a GPU: the tiny 'tf32x3' train and val nets through the interposer on the fp32
    stand-in (TF32 roundings emulated, so the exactness check is live for every call but the split-TF32 ones).  Every
    call passes; every GEMM call and the weight transposes are PREC_X3 calls; no step reaches a rounding wrapper."""
    import fake_kernels
    import fake_kernels_x3
    import launch_audit as LA
    import launch_audit_x3 as LAX
    from vlfb import executor, libvlfb as L, workspace
    monkeypatch.setattr(fake_kernels, 'EMULATE_TF32', True)
    mod = fake_kernels_x3.kernels(fake_kernels)
    executor.set_backend(mod, 'cpu', torch.float32)       # the kernels' dtype: the fp32 bounds are meaningful
    LAX.install(monkeypatch.setattr)
    try:
        for net in ('ava_train_x3', 'ava_val_fold_f32_x3'):
            workspace.ResetWorkspace()
            audit = LA.Audit(mod, 'fake_tf32')
            assert not LA.run_net(audit, net)
            bad = audit.failures()
            assert not bad, '\n'.join(e for r in bad[:10] for e in r['errors'])
            gemm = [r for r in audit.records if r['wrapper'] in LA.GEMM_WRAPPERS + ('weight_transpose_multi',)]
            assert gemm and all(r['signature']['precision'] == L.PREC_X3 for r in gemm)
            assert not [r for r in audit.records if r['run'] > 0 and r['wrapper'] in LAX.ROUNDING_WRAPPERS]
    finally:
        workspace.ResetWorkspace()
        fake_kernels.uninstall()
