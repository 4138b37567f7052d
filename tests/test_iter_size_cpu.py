"""B200.ITER_SIZE on the fp64 CPU engine (tests/fake_kernels.py): a training net created with ITER_SIZE = k runs k
micro-steps (RunNet calls, one micro-batch each) per iteration, sums their gradients and applies weight decay + Nesterov
SGD once, at the k-th.  With NUM_GPUS = k x world_size, an iteration computes the update of NUM_GPUS data-parallel GPUs
of one micro-batch each: per-micro-batch loss normalisation, the 1/NUM_GPUS loss scale, summed gradients."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import harness as H

HERE = os.path.dirname(os.path.abspath(__file__))
YAML = 'ava_r50_lfb_nl.yaml'
TINY = ['TRAIN.CROP_SIZE', 32, 'TRAIN.VIDEO_LENGTH', 8, 'TEST.CROP_SIZE', 32, 'TEST.VIDEO_LENGTH', 8,
        'LFB.WINDOW_SIZE', 2, 'TRAIN.DROPOUT_RATE', 0.0, 'FBO_NL.INPUT_DROPOUT_ON', False, 'FBO_NL.LFB_DROPOUT_ON', False]
CHECK = ['conv1_w', 'res3_1_branch2b_w', 'nonlocal_conv4_1_out_w', 'lfb_1x1_w', 'lfb_nl1_theta_b', 'pred_w', 'pred_b']


def _ov(num_gpus, clips_per_gpu, k):
    return TINY + ['NUM_GPUS', num_gpus, 'TRAIN.BATCH_SIZE', num_gpus * clips_per_gpu, 'TEST.BATCH_SIZE', num_gpus,
                   'B200.ITER_SIZE', k]


def _clips(inputs, lo, hi):
    """The inputs of clips [lo, hi), their RoIs renumbered from batch index 0."""
    rois = inputs['proposals']
    sel = (rois[:, 0] >= lo) & (rois[:, 0] < hi)
    out = {'data': inputs['data'][lo:hi], 'labels': inputs['labels'][sel], 'lfb': inputs['lfb'][sel]}
    pr = rois[sel].clone()
    pr[:, 0] -= lo
    out['proposals'] = pr
    return out


def _make(n_clips, rois=None):
    """Oracle parameters and n_clips clips of 2 RoIs each; `rois` = RoIs per clip instead (same 2 * n_clips boxes)."""
    from oracle import model as OM
    ocfg = H.oracle_cfg(YAML, _ov(1, n_clips, 1))
    params = OM.make_params(ocfg, seed=2)
    inputs = OM.make_inputs(ocfg, n_clips=n_clips, rois_per_clip=2, crop=32, frames=8)
    if rois is not None:
        assert sum(rois) == 2 * n_clips
        inputs['proposals'][:, 0] = torch.arange(n_clips).repeat_interleave(torch.tensor(rois)).to(torch.float32)
    return params, inputs


def _state(names):
    from vlfb import workspace
    return (dict((n, workspace.FetchBlob('gpu_0/' + n).copy()) for n in names),
            dict((n, workspace.FetchBlob('gpu_0/' + n + '_momentum').copy()) for n in names))


def _iteration(ov, params, micro_batches, lrs=None, between=None, before=None):
    """Fresh workspace and net under `ov` (before() called once the net exists, before the parameters are fed); one
    RunNet per micro-batch (lrs[j] fed before micro-step j; between(j, net) called after it).  Returns (losses, params,
    momenta) of CHECK after the last."""
    from vlfb import workspace
    workspace.ResetWorkspace()
    H.setup_cfg(YAML, ov)
    model, sfx = H.build('train', True)
    if before is not None:
        before()
    H.feed_params(params)
    model.UpdateWorkspaceLr(10)
    net = workspace.current().nets[model.net.Proto().name]
    losses = []
    for j, mb in enumerate(micro_batches):
        if lrs is not None:
            workspace.FeedBlob('gpu_0/lr', np.array(lrs[j], dtype=np.float32))
        H.feed_inputs(mb, sfx)
        workspace.RunNet(model.net.Proto().name)
        losses.append(float(workspace.FetchBlob('gpu_0/loss')))
        if between is not None:
            between(j, net)
    p, m = _state(CHECK)
    return losses, p, m


@pytest.fixture
def fake():
    import fake_kernels
    from vlfb import workspace
    fake_kernels.install()
    workspace.ResetWorkspace()
    yield fake_kernels
    workspace.ResetWorkspace()
    fake_kernels.uninstall()


def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-30))


def test_two_micro_steps_equal_the_two_clip_step(fake):
    params, inputs = _make(2)
    single, p1, m1 = _iteration(_ov(1, 2, 1), params, [inputs])
    micro, pk, mk = _iteration(_ov(2, 1, 2), params, [_clips(inputs, 0, 1), _clips(inputs, 1, 2)])
    assert abs(sum(micro) - single[0]) < 1e-9 * abs(single[0])
    for n in CHECK:
        assert _rel(pk[n], p1[n]) < 1e-9, n
        assert _rel(mk[n], m1[n]) < 1e-9, n
        assert np.abs(p1[n] - params[n].numpy()).max() > 0, n          # the step moved the weights


def test_unequal_roi_counts_match_the_per_micro_batch_oracle(fake):
    """Micro-batches of 1 and 3 RoIs: each normalises its loss over its own boxes, as one reference GPU does; the
    concatenated 2-clip step normalises over all 4 and computes a different update."""
    from core.config import config as cfg
    from oracle import model as OM
    from oracle import ops as O
    from vlfb import workspace
    params, inputs = _make(2, rois=[1, 3])
    mbs = [_clips(inputs, 0, 1), _clips(inputs, 1, 2)]
    assert [int(mb['proposals'].shape[0]) for mb in mbs] == [1, 3]
    _, pk, mk = _iteration(_ov(2, 1, 2), params, mbs)
    lr = float(workspace.FetchBlob('gpu_0/lr'))
    mom, wd = cfg.SOLVER.MOMENTUM, cfg.SOLVER.WEIGHT_DECAY
    _, pc, _ = _iteration(_ov(1, 2, 1), params, [inputs])
    ocfg = H.oracle_cfg(YAML, _ov(2, 1, 2))
    gsum = dict((n, torch.zeros_like(params[n], dtype=torch.float64)) for n in CHECK)
    for mb in mbs:
        p64 = dict((k, v.double().requires_grad_(True)) for k, v in params.items())
        i64 = dict((k, (v.double() if v.dtype == torch.float32 else v)) for k, v in mb.items())
        _, _, loss = OM.forward(ocfg, p64, i64, 'train')
        loss.backward()
        for n in CHECK:
            gsum[n] += p64[n].grad
    for n in CHECK:
        p0 = params[n].double()
        p_ref, m_ref = O.nesterov_update(p0, gsum[n], torch.zeros_like(p0), lr, mom, wd)
        d_ref = (p_ref - p0).numpy()
        assert _rel(pk[n] - p0.numpy(), d_ref) < 1e-7, n
        assert _rel(mk[n], m_ref.numpy()) < 1e-7, n
        assert _rel(pc[n] - p0.numpy(), d_ref) > 1e-2, n                 # the concatenated step is another update


def test_parameters_hold_until_the_boundary_and_use_its_lr(fake):
    params, inputs = _make(2)
    mbs = [_clips(inputs, 0, 1), _clips(inputs, 1, 2)]
    p0 = dict((n, params[n].numpy()) for n in CHECK)

    def unchanged(j, net):
        if j == 0:
            p, m = _state(CHECK)
            assert net.micro == 1
            for n in CHECK:
                assert np.array_equal(p[n], p0[n]), n
                assert not m[n].any(), n

    _, pa, ma = _iteration(_ov(2, 1, 2), params, mbs, lrs=[0.5, 0.01], between=unchanged)
    _, pb, mb = _iteration(_ov(2, 1, 2), params, mbs, lrs=[0.01, 0.01])
    _, pc, _ = _iteration(_ov(2, 1, 2), params, mbs, lrs=[0.01, 0.5])
    for n in CHECK:
        assert np.array_equal(pa[n], pb[n]) and np.array_equal(ma[n], mb[n]), n
        assert not np.array_equal(pa[n], pc[n]), n


def test_test_net_may_run_mid_iteration(fake):
    from vlfb import workspace
    params, inputs = _make(2)
    mbs = [_clips(inputs, 0, 1), _clips(inputs, 1, 2)]
    _, ref, _ = _iteration(_ov(2, 1, 2), params, mbs)
    seen = {}

    def build_val():
        seen['val'] = H.build('val', False)          # (its parameter initialisation runs before the parameters are fed)

    def run_val(j, net):
        if j == 0:
            model, sfx = seen['val']
            assert workspace.current().nets[model.net.Proto().name].iter_size == 1 and net.iter_size == 2
            H.feed_inputs(_clips(inputs, 0, 1), sfx)
            workspace.RunNet(model.net.Proto().name)
            seen['pred'] = workspace.FetchBlob('gpu_0/pred')

    _, got, _ = _iteration(_ov(2, 1, 2), params, mbs, between=run_val, before=build_val)
    assert seen['pred'].shape[0] == 2
    for n in CHECK:
        assert np.array_equal(got[n], ref[n]), n


def test_error_cases(fake):
    from vlfb import workspace
    from vlfb.libvlfb import VlfbError
    for bad in (0, -1):
        workspace.ResetWorkspace()
        H.setup_cfg(YAML, _ov(1, 2, bad))
        with pytest.raises(VlfbError, match='ITER_SIZE'):
            H.build('train', True)
    workspace.ResetWorkspace()
    H.setup_cfg(YAML, _ov(4, 1, 2))                     # 2 micro-steps on 1 process train 2 virtual GPUs, not 4
    with pytest.raises(VlfbError, match='NUM_GPUS = 4'):
        H.build('train', True)
    # nets without update ops ignore the setting
    workspace.ResetWorkspace()
    H.setup_cfg(YAML, _ov(1, 2, 3))
    model, _ = H.build('val', False)
    assert workspace.current().nets[model.net.Proto().name].iter_size == 1
    # another training net on the same parameters before the boundary
    params, inputs = _make(2)
    workspace.ResetWorkspace()
    H.setup_cfg(YAML, _ov(2, 1, 2))
    model, sfx = H.build('train', True)
    from models import model_builder_video
    m2 = model_builder_video.ModelBuilder(train=True, use_cudnn=True, cudnn_exhaustive_search=True,
                                          ws_nbytes_limit=256 * 1024 * 1024, split='train', name='train_net_b')
    m2.build_model(suffix=sfx, lfb=None, lfb_infer_only=False)
    workspace.RunNetOnce(m2.param_init_net)
    workspace.CreateNet(m2.net)
    H.feed_params(params)
    model.UpdateWorkspaceLr(10)
    H.feed_inputs(_clips(inputs, 0, 1), sfx)
    workspace.RunNet(model.net.Proto().name)
    with pytest.raises(VlfbError, match='micro-step 1 of 2'):
        workspace.RunNet(m2.net.Proto().name)
    workspace.RunNet(model.net.Proto().name)           # the boundary
    workspace.RunNet(m2.net.Proto().name)              # the iteration is complete: runs


# ------------------------------------------------------------------------------------------- two processes (gloo)
def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, k, inputs, params, ret):
    sys.path.insert(0, HERE)
    import conftest  # noqa: F401  (sys.path setup)
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.set_num_threads(2)
    from core import config as C
    C.reset_cfg()
    import fake_kernels
    from vlfb import dist as vdist
    from vlfb import workspace
    vdist.init_from_env('gloo')
    fake_kernels.install()
    workspace.ResetWorkspace()
    H.setup_cfg(YAML, _ov(world * k, 1, k))
    model, sfx = H.build('train', True)
    if rank == 0:
        H.feed_params(params)
    vdist.install(workspace.current())
    vdist.broadcast_params(workspace.current().params)
    model.UpdateWorkspaceLr(10)
    for j in range(k):
        c = rank * k + j
        H.feed_inputs(_clips(inputs, c, c + 1), sfx)
        workspace.RunNet(model.net.Proto().name)
    ret[rank] = _state(CHECK)
    torch.distributed.destroy_process_group()


def test_two_ranks_of_two_micro_steps_equal_one_rank_of_four(fake):
    params, inputs = _make(4)
    _, p1, m1 = _iteration(_ov(4, 1, 4), params, [_clips(inputs, c, c + 1) for c in range(4)])
    port = _free_port()
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, port, 2, inputs, params, ret), nprocs=2, join=True)
    (pa, ma), (pb, mb) = ret[0], ret[1]
    for n in CHECK:
        assert np.array_equal(pa[n], pb[n]) and np.array_equal(ma[n], mb[n]), n        # replicas stay in sync
        assert _rel(pa[n], p1[n]) < 1e-9 and _rel(ma[n], m1[n]) < 1e-9, n
        assert np.abs(p1[n] - params[n].numpy()).max() > 0, n
