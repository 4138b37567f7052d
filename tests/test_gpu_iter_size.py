"""B200.ITER_SIZE on the H100: gradient accumulation over micro-steps through the tensor-core kernels and the captured
step.  Every gradient writer must add into G (a writer that overwrote it would leave half the accumulated gradient); an
iteration of k micro-steps must compute the update of k data-parallel GPUs (fp64 oracle); non-boundary replays run the
forward + backward graph only; the memory of a k > 1 step is that of a k = 1 step."""
import contextlib
import gc
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import harness as H

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
YAML = 'ava_r50_lfb_nl.yaml'
TINY = ['TRAIN.CROP_SIZE', 64, 'TRAIN.VIDEO_LENGTH', 8, 'LFB.WINDOW_SIZE', 4, 'TRAIN.DROPOUT_RATE', 0.0,
        'FBO_NL.INPUT_DROPOUT_ON', False, 'FBO_NL.LFB_DROPOUT_ON', False]
RESNEXT = ['RESNETS.NUM_GROUPS', 32, 'RESNETS.WIDTH_PER_GROUP', 4, 'MODEL.USE_AFFINE', False, 'NONLOCAL.USE_AFFINE', False,
           'NONLOCAL.USE_BN', True, 'MODEL.DILATIONS_AFTER_CONV5', False]
MODES = {'tf32': [], 'deterministic': ['B200.DETERMINISTIC', True], 'tf32x3': ['B200.COMPUTE', 'tf32x3']}
# test_gpu_model.py's bounds for TF32-level differences of gradients
GRAD_L2_TOL, GRAD_COS_TOL, GRAD_MEDIAN_L2_TOL = 0.15, 0.98, 2e-2


def _ov(num_gpus, k, extra=()):
    return TINY + ['NUM_GPUS', num_gpus, 'TRAIN.BATCH_SIZE', 2 * num_gpus, 'TEST.BATCH_SIZE', num_gpus,
                   'B200.ITER_SIZE', k] + list(extra)


@pytest.fixture
def ws():
    from vlfb import kernels, workspace
    assert torch.cuda.is_available()
    kernels.set_gemm_backend('tcgen05')
    workspace.ResetWorkspace()
    yield workspace
    workspace.ResetWorkspace()


def _net(ws, ov, grouped=False, n_clips=2, rois=2):
    """Fresh workspace, config `ov`, the train net with oracle parameters fed.  Returns (model, sfx, net, params, inputs)."""
    import resnext_oracle as RO
    from oracle import model as OM
    ws.ResetWorkspace()
    H.setup_cfg(YAML, ov)
    ocfg = H.oracle_cfg(YAML, ov)
    with (RO.grouped() if grouped else contextlib.nullcontext(OM)) as OMg:
        params = OMg.make_params(ocfg, seed=2)
    inputs = OM.make_inputs(ocfg, n_clips=n_clips, rois_per_clip=rois, crop=64, frames=8)
    model, sfx = H.build('train', True)
    H.feed_params(params)
    model.UpdateWorkspaceLr(10)
    return model, sfx, ws.current().nets[model.net.Proto().name], params, inputs


def _grads(ws, names):
    torch.cuda.synchronize()
    return dict((n, ws.FetchBlob('gpu_0/' + n + '_grad').astype(np.float64)) for n in names)


@pytest.mark.parametrize('net_kind', ['ava_fbo_nl', 'resnext'])
@pytest.mark.parametrize('mode', sorted(MODES))
def test_every_gradient_writer_accumulates(ws, net_kind, mode):
    """k = 3; micro-steps 0 and 1 of the second iteration get the same inputs, so G after micro-step 1 is 2 g0.  The first
    iteration runs at lr 0 (no update) and makes the measured micro-steps graph replays.  A writer that overwrote G
    would leave |G - 2 g0| / |2 g0| near 0.5.  In deterministic mode G is 2 g0 bit for bit.  Elsewhere float atomics
    (split-K, fp64 SpatialBN statistics) reorder between the two runs (measured: up to 4e-6 on weights, 6e-5 on the
    non-local output biases in front of a SpatialBN), so the bound there is 1e-4.  Tensors whose gradient is below 1e-3
    of the median tensor's are skipped: mathematically zero gradients (e.g. a non-local g bias under the softmax-weighted
    sum), whose rounding noise differs between two runs by as much as itself."""
    grouped = net_kind == 'resnext'
    model, sfx, net, _, inputs = _net(ws, _ov(3, 3, MODES[mode] + (RESNEXT if grouped else [])), grouped=grouped)
    if grouped:
        assert any(getattr(s, 'groups', 1) > 1 for s in net.steps)
        assert any(type(s).__name__ == 'SpatialBNStep' for s in net.steps)
    name, names = model.net.Proto().name, model.TrainableParams()
    H.feed_inputs(inputs, sfx)
    ws.FeedBlob('gpu_0/lr', np.array(0.0, dtype=np.float32))
    for _ in range(3):
        ws.RunNet(name)
    ws.RunNet(name)
    g0 = _grads(ws, names)
    ws.RunNet(name)
    g = _grads(ws, names)
    assert len(net._graphs) == 1 and net.micro == 2
    err = {}
    floor = 1e-3 * float(np.median([np.linalg.norm(g0[n]) for n in names]))
    for n in names:
        if mode == 'deterministic':
            assert np.array_equal(g[n], 2.0 * g0[n]), n
        ref = 2.0 * g0[n]
        nref = float(np.linalg.norm(ref))
        if nref < 2.0 * floor:
            continue                                    # a mathematically zero gradient
        err[n] = float(np.linalg.norm(g[n] - ref)) / nref
    worst = sorted(err.items(), key=lambda kv: -kv[1])[:3]
    print('%s %s: |G - 2 g0| / |2 g0| worst %s' % (net_kind, mode, ' '.join('%s=%.2e' % kv for kv in worst)))
    for n, e in err.items():
        assert e <= 1e-4, (n, e)


def _micro(inputs, c, r):
    """Clip c with its first r RoIs, renumbered to batch index 0."""
    rois = inputs['proposals']
    sel = torch.nonzero(rois[:, 0] == c).view(-1)[:r]
    out = {'data': inputs['data'][c:c + 1], 'labels': inputs['labels'][sel], 'lfb': inputs['lfb'][sel]}
    pr = rois[sel].clone()
    pr[:, 0] = 0
    out['proposals'] = pr
    return out


@pytest.mark.parametrize('cap', [0, 4])
def test_iteration_matches_the_fp64_oracle(ws, cap):
    """k = NUM_GPUS = 3 micro-steps of one clip with 1, 2 and 4 RoIs: the update against Nesterov SGD of the summed fp64
    per-micro-batch gradients, held to test_gpu_model.py's gradient bounds.  Momentum starts at zero, so the new momentum
    is the update divided by (1 + momentum); it is compared rather than P_new - P, which fp32 quantises for the tensors
    whose update is far below their parameters' ulp (e.g. a non-local theta weight at this step's warm-up lr)."""
    from core.config import config as cfg
    from oracle import model as OM
    from oracle import ops as O
    ov = TINY + ['NUM_GPUS', 3, 'TRAIN.BATCH_SIZE', 3, 'TEST.BATCH_SIZE', 3, 'B200.ITER_SIZE', 3, 'B200.ROI_CAPACITY', cap]
    model, sfx, net, params, inputs = _net(ws, ov, n_clips=3, rois=4)
    mbs = [_micro(inputs, c, r) for c, r in enumerate((1, 2, 4))]
    name, names = model.net.Proto().name, model.TrainableParams()
    for mb in mbs:
        H.feed_inputs(mb, sfx)
        ws.RunNet(name)
    torch.cuda.synchronize()
    if cap:
        assert len(net._graphs) == 1                    # the third micro-step replayed the graph of the first two
    lr = float(ws.FetchBlob('gpu_0/lr'))
    ocfg = H.oracle_cfg(YAML, ov)
    gsum = {}
    for mb in mbs:
        p64 = dict((k, v.double().requires_grad_(True)) for k, v in params.items())
        i64 = dict((k, (v.double() if v.dtype == torch.float32 else v)) for k, v in mb.items())
        _, _, loss = OM.forward(ocfg, p64, i64, 'train')
        loss.backward()
        for n in names:
            gsum[n] = gsum.get(n, 0.0) + p64[n].grad
    err, cos = {}, {}
    for n in names:
        p0 = params[n].double()
        _, m_ref = O.nesterov_update(p0, gsum[n], torch.zeros_like(p0), lr, cfg.SOLVER.MOMENTUM, cfg.SOLVER.WEIGHT_DECAY)
        ref = m_ref.numpy()
        got = ws.FetchBlob('gpu_0/' + n + '_momentum').astype(np.float64)
        nref = float(np.linalg.norm(ref))
        if float(np.linalg.norm(gsum[n].numpy())) < 1e-7:
            continue
        err[n] = float(np.linalg.norm(got - ref) / nref)
        cos[n] = float((got * ref).sum() / (np.linalg.norm(got) * nref + 1e-30))
    med = float(np.median(list(err.values())))
    print('cap %d: update vs oracle median rel-L2 %.2e, worst %.2e, min cos %.5f' % (
        cap, med, max(err.values()), min(cos.values())))
    assert med < GRAD_MEDIAN_L2_TOL, med
    for n in err:
        assert err[n] < GRAD_L2_TOL and cos[n] > GRAD_COS_TOL, (n, err[n], cos[n])


def _three_iterations(ws, ov, k):
    """3 iterations of k micro-steps at one input signature.  Returns (net, per-run (launches, params changed), state)."""
    from vlfb import kernels as K
    model, sfx, net, _, inputs = _net(ws, ov)
    name, names = model.net.Proto().name, model.TrainableParams()
    H.feed_inputs(inputs, sfx)
    runs = []
    for _ in range(3 * k):
        before = dict((n, ws.FetchBlob('gpu_0/' + n)) for n in names[:4])
        n0 = K.LAUNCHES
        ws.RunNet(name)
        torch.cuda.synchronize()
        moved = any(not np.array_equal(before[n], ws.FetchBlob('gpu_0/' + n)) for n in before)
        runs.append((K.LAUNCHES - n0, moved))
    state = (ws.FetchBlob('gpu_0/loss').copy(), dict((n, ws.FetchBlob('gpu_0/' + n).copy()) for n in names),
             dict((n, ws.FetchBlob('gpu_0/' + n + '_momentum').copy()) for n in names))
    return net, runs, state


def test_graph_replays_and_memory(ws, monkeypatch):
    from vlfb import executor as X
    captures = []
    capture = X.CompiledNet._capture
    monkeypatch.setattr(X.CompiledNet, '_capture', lambda self: captures.append(1) or capture(self))
    k = 3
    det = ['B200.DETERMINISTIC', True]
    net, runs, graphed = _three_iterations(ws, _ov(k, k, det), k)
    assert len(captures) == 1 and len(net._graphs) == 1
    _, _, n1, n2, _, _, split = next(iter(net._graphs.values()))
    assert split and n2 > 0
    fills = len([c for c in ws.current().params.chunks if c['n_nonfrozen']])      # micro-step 0 zeroes G, eagerly
    for i, (launches, moved) in enumerate(runs):
        boundary = i % k == k - 1
        assert moved == boundary, i
        if i >= 2:                                      # graph replays
            expect = n1 + (fills if i % k == 0 else 0) + (n2 if boundary else 0)
            assert launches == expect, (i, launches, n1, n2, fills)
    _, _, eager = _three_iterations(ws, _ov(k, k, det + ['B200.CUDA_GRAPH', False]), k)
    assert np.array_equal(graphed[0], eager[0])
    for a, b in zip(graphed[1:], eager[1:]):
        for n in a:
            assert np.array_equal(a[n], b[n]), n
    peaks = {}
    for kk in (1, k):
        ws.ResetWorkspace()
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        _three_iterations(ws, _ov(kk, kk), kk)
        peaks[kk] = torch.cuda.max_memory_allocated()
    print('peak memory: k = 1 %.1f MiB, k = %d %.1f MiB' % (peaks[1] / 2 ** 20, k, peaks[k] / 2 ** 20))
    assert abs(peaks[k] - peaks[1]) <= 16 * 2 ** 20, peaks


def _worker(rank, world, port, k, inputs, params, ret):
    sys.path.insert(0, HERE)
    import conftest  # noqa: F401  (sys.path setup)
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    from core import config as C
    C.reset_cfg()
    from vlfb import dist as vdist
    vdist.init_from_env('nccl')
    ret[rank] = _run_ranks(rank, world, k, inputs, params)
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


CHECK = ['conv1_w', 'res2_0_branch2a_w', 'res3_1_branch2b_w', 'res5_2_branch2c_w', 'nonlocal_conv4_1_out_w', 'lfb_1x1_w',
         'lfb_nl1_theta_b', 'lfb_nl0_out_w', 'pred_w', 'pred_b']


def _run_ranks(rank, world, k, inputs, params):
    """One iteration of k micro-steps on this rank: clips rank * k .. rank * k + k - 1, one each."""
    from vlfb import dist as vdist
    from vlfb import kernels, workspace
    kernels.set_gemm_backend('tcgen05')
    workspace.ResetWorkspace()
    H.setup_cfg(YAML, TINY + ['NUM_GPUS', world * k, 'TRAIN.BATCH_SIZE', world * k, 'TEST.BATCH_SIZE', world * k,
                              'B200.ITER_SIZE', k])
    model, sfx = H.build('train', True)
    if rank == 0:
        H.feed_params(params)
    vdist.install(workspace.current())
    vdist.broadcast_params(workspace.current().params)
    model.UpdateWorkspaceLr(10)
    for j in range(k):
        H.feed_inputs(_micro(inputs, rank * k + j, 2), sfx)
        workspace.RunNet(model.net.Proto().name)
    torch.cuda.synchronize()
    out = dict((n, workspace.FetchBlob('gpu_0/' + n).copy()) for n in CHECK)
    workspace.ResetWorkspace()
    return out


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_gpus_of_two_micro_steps_equal_one_gpu_of_four():
    from oracle import model as OM
    ocfg = H.oracle_cfg(YAML, TINY + ['NUM_GPUS', 1, 'TRAIN.BATCH_SIZE', 4])
    params = OM.make_params(ocfg, seed=2)
    inputs = OM.make_inputs(ocfg, n_clips=4, rois_per_clip=2, crop=64, frames=8)
    port = _free_port()
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, port, 2, inputs, params, ret), nprocs=2, join=True)
    single = _run_ranks(0, 1, 4, inputs, params)
    for n in CHECK:
        assert np.array_equal(ret[0][n], ret[1][n]), n                     # replicas stay in sync, bit for bit
        moved = np.abs(single[n] - params[n].numpy()).max()
        d = np.abs(ret[0][n] - single[n]).max()
        assert moved > 0 and d < 2e-2 * moved + 1e-7, (n, d, moved)          # test_gpu_dist.py's bound
