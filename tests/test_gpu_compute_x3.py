"""B200.COMPUTE 'tf32x3' on the H100: every GEMM of the step on split-TF32 products of unrounded fp32 operands.

  * Launch audit (tests/launch_audit_x3.py) of the mode's tiny nets: every call against fp64 from its own tensors, a
    PREC_X3 GEMM at tau_x3(K) from its unrounded operands; every tensor-core record says prec=1, and no step reaches a
    rounding wrapper.
  * End to end: test_gpu_model's TINY step (seed 2), forward blobs, loss and gradients against the PLAIN fp64 oracle in
    both modes, on the tensor cores and (tf32x3, plain fp32) on the SIMT engine; config 2 at full size.
  * A DETERMINISTIC 'tf32x3' net: eager runs and graph replays bitwise identical.

Bounds (max|a-b|/max|b| forward and loss; per-tensor relative L2 and its median over the tensors for gradients) were
set from the errors measured on an H100 80GB HBM3 (700 W power limit), seed 2:
                              forward   loss      gradient median   worst gradient
  tiny, tf32                  5.3e-4    4.1e-6    1.1e-2            6.7e-2 (conv1_w)
  tiny, tf32x3                4.0e-5    6.0e-6    1.5e-3            6.8e-3 (conv1_w)
  tiny, tf32x3 on SIMT        9.8e-7    2.0e-8    5.2e-7            2.3e-4 (conv1_w)
  config 2, tf32x3            5.9e-5    7.3e-6    1.1e-3            2.2e-2 (conv1_w)
The forward error of the split products is 13x below TF32's.  The gradients gain less (7x in the median, 10x in the
worst tensor): their error is dominated by the ReLUs and max-pool arg-maxes that a forward perturbation flips, and
their number shrinks with the perturbation, not to zero.  The loss, a mean over all logits, is within 1e-5 in both
modes and is bounded, not compared."""
import numpy as np
import pytest
import torch

import harness as H
import launch_audit as LA
import launch_audit_x3 as LAX
from util import run_worker

pytestmark = pytest.mark.gpu

TINY = LA.TINY
FULL = ['NUM_GPUS', 1, 'TRAIN.BATCH_SIZE', 2, 'TEST.BATCH_SIZE', 2,
        'TRAIN.DROPOUT_RATE', 0.0, 'FBO_NL.INPUT_DROPOUT_ON', False, 'FBO_NL.LFB_DROPOUT_ON', False]
FWD_BLOBS = ['box_pooled', 'pool5', 'pred', 'prob']
FULL_GRADS = ['pred_w', 'lfb_1x1_w', 'lfb_nl1_out_w', 'res5_2_branch2c_w', 'res4_3_branch2b_w',
              'nonlocal_conv4_1_theta_w', 'nonlocal_conv3_1_out_w', 'res2_0_branch2a_w', 'conv1_w']
# committed 'tf32x3' bounds: (forward blobs, gradient median, worst gradient tensor), about 2.5x the measured errors
X3_TINY = (1e-4, 4e-3, 2e-2)
X3_FULL = (1.5e-4, 3e-3, 5e-2)
X3_LOSS = 3e-5
# the least gain of tf32x3 over tf32 in the same run: forward blobs, gradient median, worst gradient tensor
GAIN = (10.0, 5.0, 5.0)
X3_NETS = sorted(LAX.NETS)


@pytest.fixture
def ws():
    from vlfb import kernels, workspace
    assert torch.cuda.is_available()
    kernels.set_gemm_backend('tcgen05')
    workspace.ResetWorkspace()
    yield workspace
    workspace.ResetWorkspace()
    kernels.set_gemm_backend('tcgen05')


# ------------------------------------------------------------------------------------------------ launch audit
@pytest.mark.parametrize('net', X3_NETS)
def test_every_launch_of_a_tiny_x3_net_matches_fp64(net):
    from vlfb import libvlfb as L
    p, recs = run_worker('launch_audit_x3.py', ['--net', net], timeout=1200, tag='launch_audit')
    print('\n[%s]\n%s' % (net, p.stdout[-3000:]))
    assert p.returncode == 0, p.stderr[-4000:]
    *recs, tail = recs
    assert not tail['missing'], 'wrappers the net never reached: %s' % tail['missing']
    bad = [r for r in recs if not r['ok']]
    assert not bad, '\n'.join(e for r in bad[:20] for e in r['errors'])
    assert {r['run'] for r in recs} - {0} == set(range(1, LAX.NETS[net][3] + 1))
    gemm = [r for r in recs if r['wrapper'] in LA.GEMM_WRAPPERS]
    assert gemm and all(r['signature']['precision'] == L.PREC_X3 for r in gemm)
    tc = [q for r in gemm for q in r.get('paths', []) if q.get('path') != 'gconv']
    assert tc and all(q.get('prec') == 1 for q in tc), [q for q in tc if q.get('prec') != 1][:3]
    steps = [r for r in recs if r['run'] > 0]
    assert not [r['wrapper'] for r in steps if r['wrapper'] in LAX.ROUNDING_WRAPPERS]
    wt = [r for r in steps if r['wrapper'] == 'weight_transpose_multi']
    assert all(r['signature']['precision'] == L.PREC_X3 for r in wt)
    feeds = [r for r in recs if r['wrapper'] in ('nc_to_cl', 'lfb_gather')]
    assert feeds and not [r for r in feeds if r['signature']['tf32_out']]


# ------------------------------------------------------------------------------------------------ end to end
def _step_errors(ws, compute, backend='tcgen05', full=False):
    """Errors of one train step (no update) against the plain fp64 oracle: ({blob: max-norm}, {param: rel L2})."""
    from oracle import model as OM
    from vlfb import kernels
    kernels.set_gemm_backend(backend)
    ws.ResetWorkspace()
    ov = (FULL if full else TINY) + ['B200.COMPUTE', compute]
    H.setup_cfg('ava_r50_lfb_nl.yaml', ov)
    ocfg = H.oracle_cfg('ava_r50_lfb_nl.yaml', ov)
    params = OM.make_params(ocfg, seed=2)
    inputs = OM.make_inputs(ocfg, n_clips=2, rois_per_clip=2, crop=224 if full else 64, frames=32 if full else 8)
    model, sfx = H.build('train', True)
    H.feed_params(params)
    H.feed_inputs(inputs, sfx)
    p64 = dict((k, v.double().requires_grad_(True)) for k, v in params.items())
    i64 = dict((k, (v.double() if v.dtype == torch.float32 else v)) for k, v in inputs.items())
    blobs, _, loss = OM.forward(ocfg, p64, i64, 'train')
    loss.backward()
    ws.current().nets[model.net.Proto().name].update_ops = []
    ws.RunNet(model.net.Proto().name)
    torch.cuda.synchronize()
    fwd = {}
    loss_err = H.rel(ws.FetchBlob('gpu_0/loss'), loss.item())
    for b in FWD_BLOBS:
        fwd[b] = H.rel(ws.FetchBlob('gpu_0/' + b), blobs[b].detach().numpy())
    grads = {}
    for name in (FULL_GRADS if full else model.TrainableParams()):
        ref = p64[name].grad.numpy()
        nref = float(np.linalg.norm(ref))
        if nref < 1e-7:
            continue                                    # e.g. phi_b: mathematically zero gradient
        grads[name] = float(np.linalg.norm(ws.FetchBlob('gpu_0/' + name + '_grad').astype(np.float64) - ref) / nref)
    summary = (max(fwd.values()), float(np.median(list(grads.values()))), max(grads.values()))
    print('\n[%s %s%s] loss %.2e forward %s | gradients median %.2e worst %.2e (%s)' % (
        compute, backend, ' full' if full else '', loss_err, ' '.join('%s=%.2e' % kv for kv in fwd.items()), summary[1],
        summary[2], max(grads, key=grads.get)))
    return summary, loss_err


def _within(summary, bounds):
    return all(v < b for v, b in zip(summary, bounds))


def test_tiny_x3_step_beats_tf32(ws):
    """tf32x3 within its bounds and GAIN below the TF32 errors of the same step, which miss every one of those bounds."""
    tf32, _ = _step_errors(ws, 'tf32')
    x3, loss = _step_errors(ws, 'tf32x3')
    assert _within(x3, X3_TINY) and loss < X3_LOSS, (x3, loss)
    assert not any(v < b for v, b in zip(tf32, X3_TINY)), tf32
    for a, b, gain in zip(x3, tf32, GAIN):
        assert a * gain <= b, (x3, tf32)


def test_tiny_x3_step_on_the_simt_engine(ws):
    """On the SIMT engine `precision` changes nothing: the tf32x3 step is plain fp32."""
    x3, loss = _step_errors(ws, 'tf32x3', backend='simt')
    assert _within(x3, X3_TINY) and loss < X3_LOSS, (x3, loss)


def test_full_size_config2_x3_forward_backward(ws):
    """BASELINE config 2 (2 clips of 32 x 224^2, R = 4, L = 300) under tf32x3 against the plain fp64 oracle."""
    x3, loss = _step_errors(ws, 'tf32x3', full=True)
    assert _within(x3, X3_FULL) and loss < X3_LOSS, (x3, loss)


# ------------------------------------------------------------------------------------------------ replay
def test_deterministic_x3_replays_are_bitwise_identical(ws):
    """Eager runs 1 and 2, the capture (run 3) and a replay (run 4) from the same state: the same bits."""
    from oracle import model as OM
    ov = TINY + ['B200.COMPUTE', 'tf32x3', 'B200.DETERMINISTIC', True]
    H.setup_cfg('ava_r50_lfb_nl.yaml', ov)
    ocfg = H.oracle_cfg('ava_r50_lfb_nl.yaml', ov)
    model, sfx = H.build('train', True)
    H.feed_params(OM.make_params(ocfg, seed=2))
    H.feed_inputs(OM.make_inputs(ocfg, n_clips=2, rois_per_clip=2, crop=64, frames=8), sfx)
    net = ws.current().nets[model.net.Proto().name]
    assert net.x3 and net.det
    net.update_ops = []                         # every run starts from the same state
    runs = []
    for _ in range(5):
        ws.RunNet(model.net.Proto().name)
        torch.cuda.synchronize()
        out = dict((n, ws.FetchBlob('gpu_0/' + n + '_grad').copy()) for n in model.TrainableParams())
        out.update(loss=np.asarray(ws.FetchBlob('gpu_0/loss')).copy(), pred=ws.FetchBlob('gpu_0/pred').copy())
        runs.append(out)
    assert len(net._graphs) == 1
    for r in runs[1:]:
        for n in runs[0]:
            assert np.array_equal(r[n].reshape(-1).view(np.uint32), runs[0][n].reshape(-1).view(np.uint32)), n
