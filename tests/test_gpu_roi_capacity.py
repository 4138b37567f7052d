"""B200.ROI_CAPACITY on the H100: the kernels that take a live row count (RoIAlign forward / backward / deterministic
backward, the training FBO-NL stack, the inference bank scan) against fp64 and against a launch over the live rows only,
and the tiny AVA training net captured once at C RoI rows against the same steps run at C = 0."""
import numpy as np
import pytest
import torch

import harness as H
import streaming_cases as SC
from test_gpu_model import FULL, TINY, _train_case, ws  # noqa: F401  (ws: the fixture)

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _live(n):
    return torch.tensor([n], dtype=torch.int32, device=DEV)


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-30))


# ------------------------------------------------------------------------------------------------------ RoIAlign
def _roi_case(R, live, N=2, H=14, W=14, C=64, PH=7, PW=7, scale=1.0 / 16, sr=2, pad='zeros'):
    gen = torch.Generator().manual_seed(11)
    rois = SC.make_rois(gen, R, N, H, W, scale, 'edges')
    if pad == 'zeros':
        rois[live:] = 0.0
    elif pad == 'nan':
        rois[live:] = float('nan')
    else:                                                   # boxes far outside the image
        rois[live:] = torch.tensor([N - 1, 5000.0, 6000.0, 5100.0, 6100.0])
    feat = torch.randn((N, H, W, C), generator=gen)
    dout = torch.randn((R, PH, PW, C), generator=gen)
    dout[live:] = float('nan')                              # padded gradient rows are never read either
    return rois, feat, dout, (N, H, W, C, PH, PW, scale, sr)


@pytest.mark.parametrize('pad', ['zeros', 'nan', 'outside'])
def test_roi_align_live_rows(pad):
    from vlfb import kernels as K
    R, live = 12, 5
    rois, feat, dout, (N, H, W, C, PH, PW, scale, sr) = _roi_case(R, live, pad=pad)
    M, _ = SC.roi_matrix(rois[:live], N, H, W, PH, PW, scale, sr)
    r_d, f_d, d_d = rois.to(DEV), feat.to(DEV), dout.to(DEV)
    # forward: live rows vs fp64 and bitwise vs an R = live launch; padded rows exactly 0
    out = torch.full((R, PH, PW, C), float('nan'), device=DEV)
    K.roi_align_fwd(f_d, r_d, out, scale, sr, live_rows=_live(live))
    ref = (M @ feat.double().view(N * H * W, C)).view(live, PH, PW, C)
    assert _rel(out[:live], ref) < SC.TOL
    assert torch.count_nonzero(out[live:]) == 0
    exact = torch.empty((live, PH, PW, C), device=DEV)
    K.roi_align_fwd(f_d, r_d[:live].contiguous(), exact, scale, sr)
    assert torch.equal(out[:live], exact)
    # backward (atomic): the scatter of the live rows only
    gref = (M.t() @ dout[:live].double().reshape(live * PH * PW, C)).view(N, H, W, C)
    dfeat = torch.zeros((N, H, W, C), device=DEV)
    K.roi_align_bwd(d_d, r_d, dfeat, scale, sr, live_rows=_live(live))
    assert torch.isfinite(dfeat).all() and _rel(dfeat, gref) < SC.TOL
    # deterministic backward: also bitwise equal to the R = live launch
    det = torch.zeros((N, H, W, C), device=DEV)
    K.roi_align_bwd_det(d_d, r_d, det, scale, sr, live_rows=_live(live))
    det_exact = torch.zeros((N, H, W, C), device=DEV)
    K.roi_align_bwd_det(d_d[:live].contiguous(), r_d[:live].contiguous(), det_exact, scale, sr)
    assert _rel(det, gref) < SC.TOL and torch.equal(det, det_exact)


# ------------------------------------------------------------------------------------------------------ FBO-NL stack
def _fbo_setup(R, L, dA, d, dB, n, gen):
    Ws = []
    for _ in range(n):
        W = dict(w_theta=torch.randn((d, dA), generator=gen) * dA ** -0.5, b_theta=torch.randn(d, generator=gen) * 0.1,
                 w_phi=torch.randn((d, dB), generator=gen) * dB ** -0.5, b_phi=torch.randn(d, generator=gen) * 0.1,
                 w_g=torch.randn((d, dB), generator=gen) * dB ** -0.5, b_g=torch.randn(d, generator=gen) * 0.1,
                 w_out=torch.randn((dA, d), generator=gen) * d ** -0.5, b_out=torch.randn(dA, generator=gen) * 0.1)
        Ws.append(W)
    return Ws


def _fbo_layers(Ws, R, L, dA, d, dB):
    layers = []
    for W in Ws:
        ld = dict((k, v.to(DEV)) for k, v in W.items())
        for k, shape in (('theta', (R, d)), ('prob', (R, L)), ('s', (R, dB)), ('t', (R, d)), ('xhat', (R, d)),
                         ('ln_mean', (R,)), ('ln_std', (R,)), ('out', (R, dA)), ('a_out', (R, dA))):
            ld[k] = torch.full(shape, float('nan'), device=DEV)
        for k in SC.FBO_W:
            ld['g' + k] = torch.zeros_like(ld[k])
        layers.append(ld)
    return layers


def test_fbo_nl_stack_live_rows():
    from vlfb import kernels as K
    R, live, L, dA, d, dB, n = 12, 5, 24, 128, 64, 64, 2
    gen = torch.Generator().manual_seed(3)
    Ws = _fbo_setup(R, L, dA, d, dB, n, gen)
    a0 = torch.randn((R, dA), generator=gen)
    bp = torch.randn((R, L, dB), generator=gen)
    da = torch.randn((R, dA), generator=gen)
    a0[live:], bp[live:], da[live:] = float('nan'), float('nan'), float('nan')
    cfgd = dict(R=R, L=L, dA=dA, d=d, dB=dB, scale=d ** -0.5, pre_act_ln=True, live_rows=_live(live))
    layers = _fbo_layers(Ws, R, L, dA, d, dB)
    a0_d, bp_d, da_d = a0.to(DEV), bp.to(DEV), da.to(DEV)
    K.fbo_nl_fwd(cfgd, layers, a0_d, bp_d)
    da0 = torch.full((R, dA), float('nan'), device=DEV)
    dbp = torch.full((R, L, dB), float('nan'), device=DEV)
    K.fbo_nl_bwd(cfgd, layers, a0_d, bp_d, da_d, da0, dbp)
    # fp64 as-written graph over the live rows
    W64 = [dict((k, v.double().requires_grad_(True)) for k, v in W.items()) for W in Ws]
    a64 = a0[:live].double().requires_grad_(True)
    b64 = bp[:live].double().requires_grad_(True)
    A, outs = SC.fbo_ref(a64, b64, W64, d ** -0.5, True, [None] * n, 1.0)
    (A * da[:live].double()).sum().backward()
    for ld, o in zip(layers, outs):
        for k in SC.FBO_SAVED:
            assert _rel(ld[k][:live], o[k].detach()) < SC.TOL, k
        for k in ('theta', 'prob', 's', 't', 'xhat', 'ln_mean', 'ln_std', 'out', 'a_out'):
            assert torch.count_nonzero(ld[k][live:]) == 0, k
    assert _rel(da0[:live], a64.grad) < SC.TOL and _rel(dbp[:live], b64.grad) < SC.TOL
    assert torch.count_nonzero(da0[live:]) == 0 and torch.count_nonzero(dbp[live:]) == 0
    for ld, W in zip(layers, W64):
        for k in SC.FBO_W:
            if k != 'b_phi':                                # mathematically zero: theta * sum_j dscore_j
                assert _rel(ld['g' + k], W[k].grad) < SC.TOL, k
    # bitwise equal to the launch over the live rows only
    ex = _fbo_layers(Ws, live, L, dA, d, dB)
    cfg_ex = dict(cfgd, R=live)
    del cfg_ex['live_rows']
    a_ex, b_ex = a0_d[:live].contiguous(), bp_d[:live].contiguous()
    K.fbo_nl_fwd(cfg_ex, ex, a_ex, b_ex)
    da0_ex, dbp_ex = torch.empty((live, dA), device=DEV), torch.empty((live, L, dB), device=DEV)
    K.fbo_nl_bwd(cfg_ex, ex, a_ex, b_ex, da_d[:live].contiguous(), da0_ex, dbp_ex)
    for ld, le in zip(layers, ex):
        for k in ('theta', 'prob', 's', 't', 'xhat', 'ln_mean', 'ln_std', 'out', 'a_out'):
            assert torch.equal(ld[k][:live], le[k]), k
        for k in SC.FBO_W:
            assert torch.equal(ld['g' + k], le['g' + k]), k
    assert torch.equal(da0[:live], da0_ex) and torch.equal(dbp[:live], dbp_ex)


# ------------------------------------------------------------------------------------------------------ bank scan
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_fbo_bank_scan_live_rows(dtype):
    from vlfb import kernels as K, libvlfb as L
    R, live, Lb, D = 16, 5, 60, 2048
    dt = L.DT_BF16 if dtype == torch.bfloat16 else L.DT_F32
    lib = L.load()
    assert lib.vlfb_fbo_bank_scan_splits_dt(R, Lb, D, dt) == lib.vlfb_fbo_bank_scan_splits_dt(live, Lb, D, dt)
    gen = torch.Generator().manual_seed(9)
    bank = (torch.randn((R, Lb, D), generator=gen) * 0.5)
    q = torch.randn((R, D), generator=gen) * D ** -0.5
    bank[live:], q[live:] = float('nan'), float('nan')
    bank_d = bank.to(DEV).to(dtype).contiguous()
    q_d = q.to(DEV)
    out = torch.full((R, D), float('nan'), device=DEV)
    prob = torch.full((R, Lb), float('nan'), device=DEV)
    K.fbo_bank_scan(bank_d, q_d, out, 0.7, prob=prob, live_rows=_live(live))
    b64 = bank_d[:live].double().cpu()
    p64 = torch.softmax(torch.einsum('rld,rd->rl', b64, q[:live].double()) * 0.7, dim=1)
    assert _rel(out[:live], torch.einsum('rl,rld->rd', p64, b64)) < SC.TOL
    assert _rel(prob[:live], p64) < SC.TOL
    assert torch.count_nonzero(out[live:]) == 0 and torch.count_nonzero(prob[live:]) == 0
    out_ex, prob_ex = torch.empty((live, D), device=DEV), torch.empty((live, Lb), device=DEV)
    K.fbo_bank_scan(bank_d[:live].contiguous(), q_d[:live].contiguous(), out_ex, 0.7, prob=prob_ex)
    assert torch.equal(out[:live], out_ex) and torch.equal(prob[:live], prob_ex)


# ------------------------------------------------------------------------------------------------------ model level
SEQ = (5, 2, 16, 9, 5, 5, 12)
CAP = 16


def _sequence(ws, cap, extra=()):
    """The tiny AVA FBO-NL training net with SGD, fed r = SEQ rows per step: per-step losses, the parameters after every
    step, and how many graphs the net captured."""
    from oracle import model as OM
    H.setup_cfg('ava_r50_lfb_nl.yaml', TINY + ['B200.ROI_CAPACITY', cap] + list(extra))
    ws.ResetWorkspace()
    ocfg = H.oracle_cfg('ava_r50_lfb_nl.yaml', TINY)
    model, sfx = H.build('train', True)
    H.feed_params(OM.make_params(ocfg, seed=2))
    model.UpdateWorkspaceLr(10)
    name = model.net.Proto().name
    net = ws.current().nets[name]
    captures = [0]
    capture = net._capture

    def counted():
        captures[0] += 1
        return capture()
    net._capture = counted
    losses, params = [], []
    for i, r in enumerate(SEQ):
        inputs = OM.make_inputs(ocfg, n_clips=2, rois_per_clip=CAP // 2, crop=64, frames=8, seed=100 + i)
        for k in ('proposals', 'labels', 'lfb'):
            inputs[k] = inputs[k][:r]
        H.feed_inputs(inputs, sfx)
        ws.RunNet(name)
        assert ws.FetchBlob('gpu_0/pred').shape[0] == r
        losses.append(float(ws.FetchBlob('gpu_0/loss')))
        params.append(dict((n, ws.FetchBlob('gpu_0/' + n).copy()) for n in model.TrainableParams()))
    torch.cuda.synchronize()
    return losses, params, net, captures[0]


def test_one_captured_graph_matches_exact_row_steps(ws):
    """Deterministic mode on both sides: in the default mode float atomics let two runs of the same SGD sequence drift
    apart (TF32 rounding boundaries amplify last-bit differences from the second step on), so only here is the capacity
    the one difference between the two sequences."""
    det = ['B200.DETERMINISTIC', True]
    got, got_p, net, captures = _sequence(ws, CAP, det)
    assert len(net._graphs) == 1 and captures == 1
    want, want_p, net0, captures0 = _sequence(ws, 0, det)
    print('C = 0: %d captures, %d graphs kept (each new r moves the input buffers: a new graph key)' % (
        captures0, len(net0._graphs)))
    for i, (a, b) in enumerate(zip(got, want)):
        print('step %d r=%d loss %.7f vs %.7f' % (i, SEQ[i], a, b))
        assert abs(a - b) <= 1e-6 * abs(b), (i, a, b)          # test_gpu_model: two device runs of one step
    for i, (pa, pb) in enumerate(zip(got_p, want_p)):
        for n in pb:
            assert np.abs(pa[n] - pb[n]).max() <= 1e-5 * np.abs(pb[n]).max(), (i, n)


def test_default_mode_captures_once_and_matches_the_first_step(ws):
    """Default mode: one captured graph for every r, finite losses, and the first step (same state on both sides)
    equal to the C = 0 net's within test_gpu_model's two-run bound."""
    got, _, net, captures = _sequence(ws, CAP)
    assert len(net._graphs) == 1 and captures == 1
    assert all(np.isfinite(got))
    want, _, _, _ = _sequence(ws, 0)
    assert abs(got[0] - want[0]) <= 1e-6 * abs(want[0])


def test_deterministic_capacity_sequence_is_bitwise_reproducible(ws):
    a, pa, net, captures = _sequence(ws, CAP, ['B200.DETERMINISTIC', True])
    assert len(net._graphs) == 1 and captures == 1
    b, pb, _, _ = _sequence(ws, CAP, ['B200.DETERMINISTIC', True])
    assert a == b
    for x, y in zip(pa, pb):
        for n in x:
            assert np.array_equal(x[n], y[n]), n


def test_full_size_config2_at_capacity(ws):
    """Config 2 (2 clips of 32x224x224, L = 300) with C = 8 RoI rows of which r = 4 are live: forward and gradients
    against the fp64 oracle at test_gpu_model's bounds."""
    _train_case(ws, 'ava_r50_lfb_nl.yaml', FULL + ['B200.ROI_CAPACITY', 8], 224, 32, 2, check_all_grads=False)
    assert ws.current().blobs['pred'].shape[0] == 8 and ws.FetchBlob('gpu_0/pred').shape[0] == 4
