"""B200.GPUS_PER_STEP on the fp64 CPU engine (tests/fake_kernels.py with the segmented stand-ins of
tests/fake_kernels_seg.py): a training net created with GPUS_PER_STEP = v runs v virtual GPUs of b clips each as one
packed batch of v x b clips.  Its update must be the update of B200.ITER_SIZE = v over the same micro-batches -- per
virtual GPU loss normalisation and SpatialBN statistics, the 1/NUM_GPUS loss scale, summed gradients -- and, where the
GPU boundary matters, differ from the plain concatenated-batch step."""
import contextlib
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import harness as H

HERE = os.path.dirname(os.path.abspath(__file__))
AVA = 'ava_r50_lfb_nl.yaml'
CHARADES = 'charades_r50_lfb_nl.yaml'
TINY = ['TRAIN.CROP_SIZE', 32, 'TRAIN.VIDEO_LENGTH', 8, 'TEST.CROP_SIZE', 32, 'TEST.VIDEO_LENGTH', 8,
        'LFB.WINDOW_SIZE', 2, 'TRAIN.DROPOUT_RATE', 0.0, 'FBO_NL.INPUT_DROPOUT_ON', False, 'FBO_NL.LFB_DROPOUT_ON', False]
RESNEXT = ['RESNETS.NUM_GROUPS', 32, 'RESNETS.WIDTH_PER_GROUP', 4, 'MODEL.USE_AFFINE', False, 'NONLOCAL.USE_AFFINE', False,
           'NONLOCAL.USE_BN', True, 'MODEL.DILATIONS_AFTER_CONV5', False]
CASES = {
    'ava': (AVA, []),
    'charades': (CHARADES, ['MODEL.NUM_CLASSES', 157]),
    'epic_softmax': (CHARADES, ['DATASET', 'epic', 'MODEL.NUM_CLASSES', 125, 'MODEL.MULTI_LABEL', False]),
    'resnext_bn': (AVA, RESNEXT),
}


def _ov(extra, num_gpus, clips_per_gpu, k=1, v=1):
    return TINY + extra + ['NUM_GPUS', num_gpus, 'TRAIN.BATCH_SIZE', num_gpus * clips_per_gpu,
                           'TEST.BATCH_SIZE', num_gpus, 'B200.ITER_SIZE', k, 'B200.GPUS_PER_STEP', v]


def _clips(inputs, lo, hi):
    """The inputs of clips [lo, hi), their RoIs renumbered from batch index 0."""
    if 'proposals' not in inputs:
        return dict((n, t[lo:hi]) for n, t in inputs.items())
    rois = inputs['proposals']
    sel = (rois[:, 0] >= lo) & (rois[:, 0] < hi)
    out = {'data': inputs['data'][lo:hi], 'labels': inputs['labels'][sel], 'lfb': inputs['lfb'][sel]}
    pr = rois[sel].clone()
    pr[:, 0] -= lo
    out['proposals'] = pr
    return out


def _grouped(case):
    import resnext_oracle as RO
    return RO.grouped() if case == 'resnext_bn' else contextlib.nullcontext()


def _make(case, n_clips, rois=None, ignored=()):
    """Oracle parameters and n_clips clips (2 RoIs each, or rois[c] for clip c); the RoIs of the clips in `ignored` get
    label -1 everywhere."""
    from oracle import model as OM
    yaml, extra = CASES[case]
    ocfg = H.oracle_cfg(yaml, _ov(extra, 1, n_clips))
    with _grouped(case):
        params = OM.make_params(ocfg, seed=2)
    inputs = OM.make_inputs(ocfg, n_clips=n_clips, rois_per_clip=2, crop=32, frames=8)
    if rois is not None:
        assert sum(rois) == 2 * n_clips
        inputs['proposals'][:, 0] = torch.arange(n_clips).repeat_interleave(torch.tensor(rois)).to(torch.float32)
    for c in ignored:
        inputs['labels'][inputs['proposals'][:, 0] == c] = -1
    return params, inputs


@pytest.fixture
def fake():
    import fake_kernels
    import fake_kernels_seg
    from vlfb import workspace
    fake_kernels_seg.install(fake_kernels)
    workspace.ResetWorkspace()
    yield fake_kernels
    workspace.ResetWorkspace()
    fake_kernels.uninstall()


def _install(case):
    import fake_kernels
    import fake_kernels_seg
    import resnext_oracle as RO
    fake_kernels_seg.install(RO if case == 'resnext_bn' else fake_kernels)


def _run(case, ov, params, batches, between=None):
    """Fresh workspace and train net under `ov`; one RunNet per batch.  Returns (losses, {trainable param: (value,
    momentum)}, net)."""
    from vlfb import workspace
    workspace.ResetWorkspace()
    H.setup_cfg(CASES[case][0], ov)
    model, sfx = H.build('train', True)
    H.feed_params(params)
    model.UpdateWorkspaceLr(10)
    net = workspace.current().nets[model.net.Proto().name]
    losses = []
    for j, mb in enumerate(batches):
        H.feed_inputs(mb, sfx)
        workspace.RunNet(model.net.Proto().name)
        losses.append(float(workspace.FetchBlob('gpu_0/loss')))
        if between is not None:
            between(j, net)
    state = dict((n, (workspace.FetchBlob('gpu_0/' + n).copy(), workspace.FetchBlob('gpu_0/' + n + '_momentum').copy()))
                 for n in net.trainable)
    return losses, state, net


def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-30))


def _worst(got, ref):
    """Worst difference of parameters and momenta, relative to each tensor's magnitude but at least 1e-3 of the largest
    momentum (a gradient that cancels to roundoff, e.g. behind a zero-initialised BN scale, has no relative accuracy)."""
    floor = 1e-3 * max(np.abs(ref[n][1]).max() for n in ref)
    return max(max(np.abs(got[n][i] - ref[n][i]).max() / max(np.abs(ref[n][i]).max(), floor) for i in (0, 1))
               for n in ref)


def _packed_vs_iter_size(case, v, k=1, rois=None, ignored=(), extra=()):
    """v x k virtual GPUs of one clip each: GPUS_PER_STEP = v with ITER_SIZE = k against ITER_SIZE = v x k."""
    _install(case)
    n = v * k
    params, inputs = _make(case, n, rois, ignored)
    ex = CASES[case][1] + list(extra)
    micro = [_clips(inputs, c, c + 1) for c in range(n)]
    ref_l, ref, ref_net = _run(case, _ov(ex, n, 1, k=n), params, micro)
    packs = [_clips(inputs, j * v, (j + 1) * v) for j in range(k)]
    got_l, got, net = _run(case, _ov(ex, n, 1, k=k, v=v), params, packs)
    assert net.gpus_per_step == v and net.iter_size == k and ref_net.gpus_per_step == 1
    assert abs(sum(got_l) - sum(ref_l)) <= 1e-9 * abs(sum(ref_l))
    assert _worst(got, ref) < 1e-9
    moved = [n_ for n_ in ref if np.abs(ref[n_][0] - params[n_].numpy()).max() > 0] if case != 'resnext_bn' else list(ref)
    assert moved
    return params, inputs, ref


@pytest.mark.parametrize('case,v', [('ava', 2), ('charades', 2), ('epic_softmax', 4)])
def test_packed_step_equals_iter_size(fake, case, v):
    _packed_vs_iter_size(case, v)


def test_unequal_rois_and_an_ignored_gpu_match_iter_size_and_not_the_concatenated_step(fake):
    """Virtual GPUs of 1, 3, 2 and 2 RoIs, the third with every label -1 (count 0: the 1e-5 floor, no loss, no gradient);
    the concatenated 4-clip step normalises over all boxes together and computes another update."""
    params, inputs, ref = _packed_vs_iter_size('ava', 4, rois=[1, 3, 2, 2], ignored=(2,))
    _, cat, _ = _run('ava', _ov([], 1, 4), params, [inputs])
    assert max(_rel(cat[n][1], ref[n][1]) for n in ref) > 1e-2


def test_spatial_bn_statistics_are_per_virtual_gpu(fake):
    """ResNeXt with SpatialBN: the packed step equals ITER_SIZE = 2; the running statistics are virtual GPU 0's (those of
    ITER_SIZE's first micro-step); the concatenated step (statistics over both clips) is another update."""
    from vlfb import workspace
    params, inputs, ref = _packed_vs_iter_size('resnext_bn', 2)
    seen = {}

    def first(j, net):
        if j == 0:
            st = workspace.current().params
            seen.update((n, workspace.FetchBlob('gpu_0/' + n).copy()) for n in st.index if n.endswith('_rm') or n.endswith('_riv'))

    _run('resnext_bn', _ov(RESNEXT, 2, 1, k=2), params, [_clips(inputs, 0, 1), _clips(inputs, 1, 2)], between=first)
    _, _, net = _run('resnext_bn', _ov(RESNEXT, 2, 1, v=2), params, [inputs])
    assert seen and any(type(st).__name__ == 'SpatialBNStep' for st in net.steps)
    for n, val in seen.items():
        assert _rel(workspace.FetchBlob('gpu_0/' + n), val) < 1e-9, n
    _, cat, _ = _run('resnext_bn', _ov(RESNEXT, 1, 2), params, [inputs])
    assert max(_rel(cat[n][1], ref[n][1]) for n in ref) > 1e-2


def test_gpus_per_step_times_iter_size(fake):
    _packed_vs_iter_size('ava', 2, k=2, rois=[3, 1, 2, 2])


def test_with_roi_capacity(fake, monkeypatch):
    """C = 12 RoI rows for 2 virtual GPUs of 1 and 3 RoIs: the padded rows carry label -1 and count nowhere."""
    import fake_kernels
    import fake_live_rows
    fake_live_rows.install(monkeypatch)
    import fake_kernels_seg
    fake_kernels_seg.install(fake_kernels)                  # again: on top of the live-row wrappers
    params, inputs = _make('ava', 2, rois=[1, 3])
    micro = [_clips(inputs, 0, 1), _clips(inputs, 1, 2)]
    _, ref, _ = _run('ava', _ov([], 2, 1, k=2), params, micro)
    _, got, net = _run('ava', _ov(['B200.ROI_CAPACITY', 12], 2, 1, v=2), params, [inputs])
    assert net.roi_capacity == 12
    assert _worst(got, ref) < 1e-9


def test_with_deterministic(fake, monkeypatch):
    """The deterministic forms (the stand-in's sums are exact, so its _det names are its plain functions)."""
    import fake_kernels
    for det in ('conv_wgrad_det', 'matmul_det', 'colsum_det', 'roi_align_bwd_det', 'spatial_bn_fwd_det',
                'spatial_bn_bwd_det'):
        if not hasattr(fake_kernels, det):
            monkeypatch.setattr(fake_kernels, det, getattr(fake_kernels, det[:-4]), raising=False)
    _packed_vs_iter_size('ava', 2, rois=[3, 1], extra=['B200.DETERMINISTIC', True])


def test_error_cases(fake):
    from core.config import config as cfg
    from utils.misc import get_batch_size
    from vlfb import workspace
    from vlfb.libvlfb import VlfbError
    for bad in (0, -1, 1.5):
        workspace.ResetWorkspace()
        H.setup_cfg(AVA, _ov([], 1, 2, v=bad))
        with pytest.raises(VlfbError, match='GPUS_PER_STEP'):
            H.build('train', True)
    workspace.ResetWorkspace()
    H.setup_cfg(AVA, _ov([], 4, 1, v=2))                  # 2 virtual GPUs per step on 1 process train 2, not 4
    with pytest.raises(VlfbError, match='NUM_GPUS = 4'):
        H.build('train', True)
    workspace.ResetWorkspace()
    H.setup_cfg(AVA, _ov([], 4, 1, k=2, v=1))             # v = 1: the ITER_SIZE check as before
    with pytest.raises(VlfbError, match='ITER_SIZE = 2 on 1 process'):
        H.build('train', True)
    # the recorded batch must be v x b
    from models import model_builder_video
    workspace.ResetWorkspace()
    H.setup_cfg(AVA, _ov([], 2, 1, v=1))
    m = model_builder_video.ModelBuilder(train=True, use_cudnn=True, cudnn_exhaustive_search=True,
                                         ws_nbytes_limit=256 * 1024 * 1024, split='train', name='train_net')
    m.build_model(suffix='_train', lfb=None, lfb_infer_only=False)
    workspace.RunNetOnce(m.param_init_net)
    cfg.B200.GPUS_PER_STEP = 2
    with pytest.raises(VlfbError, match='batch of 1 clips'):
        workspace.CreateNet(m.net)
    # get_batch_size: v x b for the packed step of a net with update ops only
    assert get_batch_size('train', packed=True) == 2 and get_batch_size('train') == 1
    assert get_batch_size('test', packed=True) == int(cfg.TEST.BATCH_SIZE / cfg.NUM_GPUS)
    # a forward-only training-split net (precise-BN's aux net) is built at one GPU's clips and ignores the setting
    aux = model_builder_video.ModelBuilder(train=True, use_cudnn=True, cudnn_exhaustive_search=True,
                                           ws_nbytes_limit=256 * 1024 * 1024, split='train', name='bn_aux',
                                           force_fw_only=True)
    aux.build_model(suffix='_train', lfb=None, lfb_infer_only=False)
    workspace.CreateNet(aux.net)
    assert aux.recorded_batch_size == 1 and workspace.current().nets['bn_aux'].gpus_per_step == 1
    # nets without update ops ignore the setting
    workspace.ResetWorkspace()
    H.setup_cfg(AVA, _ov([], 2, 1, v=2))
    model, _ = H.build('val', False)
    assert workspace.current().nets[model.net.Proto().name].gpus_per_step == 1
    # feeds that break the packed batch's rules
    params, inputs = _make('ava', 2)
    workspace.ResetWorkspace()
    H.setup_cfg(AVA, _ov([], 2, 1, v=2))
    H.feed_inputs(inputs, '_train')                        # before the net exists: not checked
    model, sfx = H.build('train', True)
    H.feed_params(params)
    model.UpdateWorkspaceLr(10)
    with pytest.raises(VlfbError, match='proposals_train: not fed as a packed batch'):
        workspace.RunNet(model.net.Proto().name)
    bad = inputs['proposals'].clone()
    bad[:, 0] = torch.tensor([1.0, 1.0, 0.0, 0.0])
    with pytest.raises(VlfbError, match='proposals_train: batch indices decrease'):
        workspace.FeedBlob('gpu_0/proposals_train', bad.numpy())
    bad[:, 0] = torch.tensor([0.0, 0.0, 1.0, 2.0])
    with pytest.raises(VlfbError, match=r'proposals_train: batch indices must be integers in \[0, 2\)'):
        workspace.FeedBlob('gpu_0/proposals_train', bad.numpy())
    H.feed_inputs(inputs, sfx)
    workspace.RunNet(model.net.Proto().name)
    assert np.array_equal(workspace.current().roi_segments['proposals_train'].numpy(), [0, 2, 4])
    # a feed that fails after the check leaves the offsets of the last feed that landed
    workspace.current().roi_capacity['proposals_train'] = (3, '_train')
    with pytest.raises(VlfbError, match='ROI_CAPACITY = 3'):
        workspace.FeedBlob('gpu_0/proposals_train', inputs['proposals'][[0, 0, 1, 1]].numpy())
    assert np.array_equal(workspace.current().roi_segments['proposals_train'].numpy(), [0, 2, 4])


# ------------------------------------------------------------------------------------------- two processes (gloo)
def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, v, inputs, params, ret):
    sys.path.insert(0, HERE)
    import conftest  # noqa: F401  (sys.path setup)
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.set_num_threads(2)
    from core import config as C
    C.reset_cfg()
    import fake_kernels
    import fake_kernels_seg
    from vlfb import dist as vdist
    from vlfb import workspace
    vdist.init_from_env('gloo')
    fake_kernels_seg.install(fake_kernels)
    workspace.ResetWorkspace()
    H.setup_cfg(AVA, _ov([], world * v, 1, v=v))
    model, sfx = H.build('train', True)
    if rank == 0:
        H.feed_params(params)
    vdist.install(workspace.current())
    vdist.broadcast_params(workspace.current().params)
    model.UpdateWorkspaceLr(10)
    H.feed_inputs(_clips(inputs, rank * v, (rank + 1) * v), sfx)
    workspace.RunNet(model.net.Proto().name)
    names = workspace.current().nets[model.net.Proto().name].trainable
    ret[rank] = dict((n, (workspace.FetchBlob('gpu_0/' + n).copy(), workspace.FetchBlob('gpu_0/' + n + '_momentum').copy()))
                     for n in names)
    torch.distributed.destroy_process_group()


def test_two_ranks_of_two_virtual_gpus_equal_one_rank_of_four(fake):
    params, inputs = _make('ava', 4, rois=[1, 2, 4, 1])
    _, one, _ = _run('ava', _ov([], 4, 1, v=4), params, [inputs])
    port = _free_port()
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, port, 2, inputs, params, ret), nprocs=2, join=True)
    a, b = ret[0], ret[1]
    for n in one:
        assert np.array_equal(a[n][0], b[n][0]) and np.array_equal(a[n][1], b[n][1]), n
        assert _rel(a[n][0], one[n][0]) < 1e-9 and _rel(a[n][1], one[n][1]) < 1e-9, n


def test_launch_audit_of_packed_nets_on_the_stand_in(monkeypatch):
    """tests/launch_audit_seg.py without a GPU: packed AVA and ResNeXt + SpatialBN train nets through the interposer on
    the fp32 stand-in (TF32 roundings emulated).  Every call passes, the segmented ones included."""
    import fake_kernels
    import fake_kernels_seg
    import launch_audit as LA
    import launch_audit_seg as LAS
    import resnext_oracle as RO
    from vlfb import executor, workspace
    monkeypatch.setattr(fake_kernels, 'EMULATE_TF32', True)
    LAS.install(monkeypatch.setattr)
    try:
        for net, base in (('ava_train_packed', fake_kernels), ('resnext_bn_train_packed', RO)):
            mod = fake_kernels_seg.kernels(base)
            executor.set_backend(mod, 'cpu', torch.float32)
            workspace.ResetWorkspace()
            audit = LA.Audit(mod, 'fake_tf32')
            assert not LA.run_net(audit, net)
            bad = audit.failures()
            assert not bad, '\n'.join(e for r in bad[:10] for e in r['errors'])
            assert set(LAS.SEG_WRAPPERS) & set(audit.calls)
    finally:
        workspace.ResetWorkspace()
        fake_kernels.uninstall()
