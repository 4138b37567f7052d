"""B200.DETERMINISTIC on the GPU.

Kernel level (in a worker process: the library reads VLFB_DEBUG once, when it loads):
    VLFB_DEBUG=1 python tests/test_gpu_deterministic.py
every deterministic entry point at production shapes and at shapes built to collide (long-K wgrads, many identical
RoIs) against fp64, twice on the same inputs with bitwise-identical results, and each GEMM launch's record showing a
schedule with one contribution per element (split 1; stream-K only with the fix-up).
Model level: the same sequence of steps (eager runs, graph replays, SGD) from the same state twice gives identical
losses, gradients and parameters; deterministic and default mode agree; a checkpoint resumes exactly.
"""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
for _p in (HERE, os.path.dirname(HERE), os.path.join(os.path.dirname(HERE), 'video-long-term-feature-banks_b200', 'lib')):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import harness as H  # noqa: E402
from util import capture_fd2, parse_record, run_worker  # noqa: E402

pytestmark = pytest.mark.gpu

TINY = ['NUM_GPUS', 1, 'TRAIN.BATCH_SIZE', 2, 'TRAIN.CROP_SIZE', 64, 'TRAIN.VIDEO_LENGTH', 8,
        'TEST.BATCH_SIZE', 2, 'TEST.CROP_SIZE', 64, 'TEST.VIDEO_LENGTH', 8, 'LFB.WINDOW_SIZE', 4,
        'TRAIN.DROPOUT_RATE', 0.0, 'FBO_NL.INPUT_DROPOUT_ON', False, 'FBO_NL.LFB_DROPOUT_ON', False]
DET = ['B200.DETERMINISTIC', True]


# ------------------------------------------------------------------------------------------------ kernel level
def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _twice(fn, out):
    """fn() accumulates into / writes `out` from the state `out` has now: run it twice from that state and return both."""
    start = out.clone()
    fn()
    first = out.clone()
    out.copy_(start)
    fn()
    torch.cuda.synchronize()
    return first, out.clone()


def _gemm_records(text):
    recs = [parse_record(l) for l in text.splitlines()]
    return [r for r in recs if r]


def _check_wgrad(K, label, shape, co, ker, st, pd, dil, tol, expect=None):
    dev = 'cuda'
    gen = torch.Generator(device='cpu').manual_seed(7)
    g = K.conv_geom(shape, co, ker, st, pd, dil)
    x = torch.randn(shape, generator=gen).to(dev)
    if g.C == 4:
        x[..., 3] = 0
    dy = torch.randn((g.N, g.To, g.Ho, g.Wo, co), generator=gen).to(dev)
    xr = x.clone(); K.round_tf32(x, xr)
    dyr = dy.clone(); K.round_tf32(dy, dyr)
    if g.C == 4:
        dw = torch.zeros((co, g.kT, g.kH, 8, 4), device=dev)
        mask = torch.tensor([1.0, 1.0, 1.0, 0.0] * 8, device=dev)
    else:
        dw = torch.zeros((co, g.kT, g.kH, g.kW, g.C), device=dev)
        mask = None
    (a, b), text = capture_fd2(lambda: _twice(lambda: K.conv_wgrad_det(dyr, xr, dw, g, col_mask=mask), dw))
    assert torch.equal(a, b), label
    recs = [r for r in _gemm_records(text) if r.get('det') == 1]
    assert recs, (label, text[-500:])
    for r in recs:
        assert r['split'] == 1 and (r['sk'] == 0 or r['fix'] == 1), (label, r)
        for k, v in (expect or {}).items():
            assert r[k] == v, (label, k, r)
    # fp64 reference: dw[co, kt, kh, kw, ci] = sum over positions of dy * x
    xc = xr.double().permute(0, 4, 1, 2, 3)
    dyc = dyr.double().permute(0, 4, 1, 2, 3)
    if g.C == 4:
        xpad = torch.nn.functional.pad(xc[:, :3], (0, 0, 0, 0, 0, 0))
        ref = torch.nn.grad.conv3d_weight(xpad, (co, 3, g.kT, g.kH, g.kW), dyc, stride=(g.sT, g.sH, g.sW),
                                          padding=(g.pT, g.pH, g.pW), dilation=(g.dT, g.dH, g.dW))
        got = a[:, :, :, :g.kW, :3].permute(0, 4, 1, 2, 3).double()
    else:
        ref = torch.nn.grad.conv3d_weight(xc, (co, g.C, g.kT, g.kH, g.kW), dyc, stride=(g.sT, g.sH, g.sW),
                                          padding=(g.pT, g.pH, g.pW), dilation=(g.dT, g.dH, g.dW))
        got = a.permute(0, 4, 1, 2, 3).double()
    err = _rel(got, ref)
    print('[deterministic] wgrad %-32s rel %.2e  %s' % (label, err, ' '.join('cp=%d sk=%d fix=%d bn=%d wide=%d' % (
        r['cp'], r['sk'], r['fix'], r['bn'], r.get('wide', 0)) for r in recs)))
    assert err < tol, (label, err)
    return recs


def kernel_checks():
    from vlfb import kernels as K
    import wgrad_cases as WC
    dev = 'cuda'
    gen = torch.Generator(device='cpu').manual_seed(3)
    # weight gradients: every production geometry, plus a grouped one
    for label, shape, co, ker, st, pd, dil, _ in WC.PRODUCTION:
        # conv1 (Co 64, 25088 K chunks per tile): 64 x 2BN wide tiles of the cp.async build, reduced by gemm_fixup_kernel
        expect = dict(cp=1, wide=1, sk=1, fix=1) if label.startswith('conv1') else None
        _check_wgrad(K, label, shape, co, ker, st, pd, dil, 1e-4, expect)
    # long-K split matmuls (the non-local gradient products, the classifier), rounded and not
    for (M, N, Kd, tf32) in [(784, 784, 3136, False), (512, 1024, 3136, True), (4, 80, 2560, False), (80, 2560, 8, False)]:
        a = torch.randn((1, M, Kd), generator=gen).to(dev)
        b = torch.randn((1, Kd, N), generator=gen).to(dev)
        ar, br = a.clone(), b.clone()
        K.round_tf32(a, ar), K.round_tf32(b, br)
        d = torch.empty((1, M, N), device=dev)
        (x, y), text = capture_fd2(lambda: _twice(lambda: K.matmul_det(ar, br, d, tf32_out=tf32), d))
        assert torch.equal(x, y)
        for r in _gemm_records(text):
            assert r['split'] == 1 and (r['sk'] == 0 or r['fix'] == 1), r
        err = _rel(x, ar.double() @ br.double())
        print('[deterministic] matmul_det %dx%dx%d tf32=%d rel %.2e' % (M, N, Kd, tf32, err))
        assert err < (1e-3 if tf32 else 1e-4)
    # bias gradients
    for rows, cols in [(100352, 64), (40, 2048), (7, 80)]:
        x = torch.randn((rows, cols), generator=gen).to(dev)
        out = torch.randn(cols, generator=gen).to(dev)
        o0 = out.clone()
        a, b = _twice(lambda: K.colsum_det(x, cols, out, rows, cols, accumulate=True), out)
        assert torch.equal(a, b)
        err = _rel(a - o0, x.double().sum(0))
        print('[deterministic] colsum_det %dx%d rel %.2e' % (rows, cols, err))
        assert err < 1e-5
    # RoIAlign backward against the fp64 sample-table reference of tests/streaming_cases.py: the res5 width (C 2048)
    # with boxes on the map's edges, 100 random boxes, and 32 identical boxes (every sample collides)
    import streaming_cases as SC
    for N, Hh, Ww, C, R, PH, sr, kind in [(2, 14, 14, 2048, 9, 7, 0, 'edges'), (2, 16, 16, 512, 100, 7, 0, 'random'),
                                          (2, 14, 14, 2048, 32, 7, 2, 'same')]:
        scale = 1.0 / 16
        rois = SC.make_rois(gen, R, N, Hh, Ww, scale, 'random' if kind == 'same' else kind)
        if kind == 'same':
            rois[:] = rois[0]
        M, _ = SC.roi_matrix(rois, N, Hh, Ww, PH, PH, scale, sr)
        M = M.to(dev)
        rois_d = rois.to(dev)
        dout = torch.randn((R, PH, PH, C), generator=gen).to(dev)
        dfeat = torch.randn((N, Hh, Ww, C), generator=gen).to(dev)
        ref = (M.t() @ dout.double().view(R * PH * PH, C)).view(N, Hh, Ww, C) + dfeat.double()
        mag = (M.abs().t() @ dout.double().abs().view(R * PH * PH, C)).view(N, Hh, Ww, C) + dfeat.double().abs()
        terms = int((M != 0).sum(0).max()) + 1
        a, b = _twice(lambda: K.roi_align_bwd_det(dout, rois_d, dfeat, scale, sr), dfeat)
        assert torch.equal(a, b)
        excess = float(((a.double() - ref).abs() - terms * 2.0 ** -23 * 2 * mag).max())
        print('[deterministic] roi_align_bwd_det %s R=%d C=%d: max |err| - bound %.2e' % (kind, R, C, excess))
        assert excess <= 0, kind
    # SpatialBN statistics
    rows, C = 2 * 8 * 28 * 28, 128
    x = (torch.randn((rows, C), generator=gen) * 3 + 1).to(dev)
    s, bb = torch.rand(C, generator=gen).to(dev) + 0.5, torch.randn(C, generator=gen).to(dev)
    rm, rv = torch.zeros(C, device=dev), torch.ones(C, device=dev)
    sm, siv, y = torch.empty(C, device=dev), torch.empty(C, device=dev), torch.empty_like(x)
    a, b = _twice(lambda: K.spatial_bn_fwd_det(x, s, bb, rm, rv, sm, siv, y, 1e-5, 0.9), y)
    assert torch.equal(a, b)
    xd = x.double()
    ref = (xd - xd.mean(0)) / torch.sqrt(xd.var(0, unbiased=False) + 1e-5) * s.double() + bb.double()
    assert _rel(a, ref) < 1e-5, _rel(a, ref)
    dy = torch.randn((rows, C), generator=gen).to(dev)
    dx = torch.empty_like(x)
    ds, db = torch.zeros(C, device=dev), torch.zeros(C, device=dev)
    a, b = _twice(lambda: K.spatial_bn_bwd_det(dy, x, s, sm, siv, dx, ds, db), dx)
    assert torch.equal(a, b)
    xr = xd.clone().requires_grad_(True)
    yr = (xr - xr.mean(0)) / torch.sqrt(xr.var(0, unbiased=False) + 1e-5) * s.double() + bb.double()
    yr.backward(dy.double())
    assert _rel(a, xr.grad) < 1e-4, _rel(a, xr.grad)
    print('[deterministic] spatial_bn det fwd / bwd ok')
    # grouped weight gradient (ResNeXt branch2b), split over positions into workspace slabs
    import gconv_cases as GC  # noqa: F401  (the grouped geometries' conventions)
    g = K.conv_geom((2, 8, 28, 28, 256), 256, (3, 3, 3), (1, 1, 1), (1, 1, 1))
    x = torch.randn((2, 8, 28, 28, 256), generator=gen).to(dev)
    dy = torch.randn((2, g.To, g.Ho, g.Wo, 256), generator=gen).to(dev)
    dw = torch.zeros((256, 3, 3, 3, 8), device=dev)
    (a, b), text = capture_fd2(lambda: _twice(lambda: K.conv_wgrad_det(dy, x, dw, g, groups=32), dw))
    assert torch.equal(a, b)
    rec = [l for l in text.splitlines() if 'vlfb gconv:' in l and 'dir=wgrad' in l]
    assert rec and 'det=1' in rec[-1], text[-300:]
    fields = dict(kv.split('=') for kv in rec[-1].split()[2:])
    assert int(fields['grid'].split(',')[0]) >= 2 and int(fields['slabs']) >= 2, rec[-1]     # partial slabs + sum pass
    ref = torch.nn.grad.conv3d_weight(x.double().permute(0, 4, 1, 2, 3), (256, 8, 3, 3, 3),
                                      dy.double().permute(0, 4, 1, 2, 3), padding=(1, 1, 1), groups=32)
    err = _rel(a.permute(0, 4, 1, 2, 3), ref)
    print('[deterministic] grouped wgrad det rel %.2e' % err)
    assert err < 1e-5
    print('KERNEL CHECKS OK')


def forced_cp_checks():
    """Every wgrad runs in the cp.async build (both operands are MN-major), on 128 x BN tiles when Co > 64: the fix-up
    of gemm_fixup_kernel on narrow tiles."""
    from vlfb import kernels as K
    import wgrad_cases as WC
    seen = 0
    for label, shape, co, ker, st, pd, dil, _ in WC.PRODUCTION:
        if co < 128 or co > 256:
            continue
        recs = _check_wgrad(K, label, shape, co, ker, st, pd, dil, 1e-4, dict(cp=1, wide=0))
        seen += sum(1 for r in recs if r['sk'] == 1 and r['fix'] == 1)
    assert seen > 0, 'no 128 x BN cp.async launch took the fix-up'
    print('FORCED CP CHECKS OK')


def _worker(args, ok):
    r, _ = run_worker('test_gpu_deterministic.py', args, timeout=1800, tag='deterministic', jsonl=False)
    print(r.stdout[-6000:])
    assert r.returncode == 0 and ok in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def test_deterministic_kernels():
    _worker([], 'KERNEL CHECKS OK')


def test_deterministic_wgrad_fixup_on_128_row_cp_async_tiles():
    _worker(['--forced-cp'], 'FORCED CP CHECKS OK')


# ------------------------------------------------------------------------------------------------ model level
@pytest.fixture
def ws():
    from vlfb import kernels, workspace
    assert torch.cuda.is_available()
    kernels.set_gemm_backend('tcgen05')
    workspace.ResetWorkspace()
    yield workspace
    workspace.ResetWorkspace()


def _session(ws, yaml_name, overrides, steps=4, crop=64, frames=8, rois=2, seed=2, grouped=False):
    """Fresh workspace, same parameters and inputs; `steps` training steps with SGD (eager, eager, then graph replays).
    Returns [(loss, {param: value}, {param: grad})] per step."""
    import contextlib
    import resnext_oracle as RO
    with (RO.grouped() if grouped else contextlib.nullcontext()) as OMg:
        return _session_in(ws, yaml_name, overrides, steps, crop, frames, rois, seed, OMg)


def _session_in(ws, yaml_name, overrides, steps, crop, frames, rois, seed, OMg):
    from oracle import model as OM
    OM = OMg or OM
    ws.ResetWorkspace()
    H.setup_cfg(yaml_name, overrides)
    ocfg = H.oracle_cfg(yaml_name, overrides)
    params = OM.make_params(ocfg, seed=seed)
    inputs = OM.make_inputs(ocfg, n_clips=2, rois_per_clip=rois, crop=crop, frames=frames)
    model, sfx = H.build('train', True)
    H.feed_params(params)
    H.feed_inputs(inputs, sfx)
    model.UpdateWorkspaceLr(10)
    out = []
    names = model.TrainableParams()
    for _ in range(steps):
        ws.RunNet(model.net.Proto().name)
        torch.cuda.synchronize()
        out.append(_state(ws, names))
    net = ws.current().nets[model.net.Proto().name]
    return out, net, model


def _state(ws, names):
    """(loss, {param}, {grad}, {momentum}) after a step."""
    return (ws.FetchBlob('gpu_0/loss').copy(),
            dict((n, ws.FetchBlob('gpu_0/' + n).copy()) for n in names),
            dict((n, ws.FetchBlob('gpu_0/' + n + '_grad').copy()) for n in names),
            dict((n, ws.FetchBlob('gpu_0/' + n + '_momentum').copy()) for n in names))


def _assert_identical(r1, r2):
    assert len(r1) == len(r2)
    for step, ((l1, p1, g1, m1), (l2, p2, g2, m2)) in enumerate(zip(r1, r2)):
        assert np.array_equal(l1, l2), step
        for n in p1:
            assert np.array_equal(g1[n], g2[n]), (step, n, 'grad')
            assert np.array_equal(m1[n], m2[n]), (step, n, 'momentum')
            assert np.array_equal(p1[n], p2[n]), (step, n, 'param')


def test_tiny_ava_fbo_nl_steps_are_bitwise_reproducible(ws):
    r1, net, _ = _session(ws, 'ava_r50_lfb_nl.yaml', TINY + DET)
    assert net.det and len(net._graphs) == 1, 'the later steps should be graph replays'
    r2, _, _ = _session(ws, 'ava_r50_lfb_nl.yaml', TINY + DET)
    _assert_identical(r1, r2)


def test_tiny_resnext_spatial_bn_steps_are_bitwise_reproducible(ws):
    """Grouped convolutions (ResNeXt 32x4d) and trainable SpatialBN in one net."""
    ov = TINY + DET + ['RESNETS.NUM_GROUPS', 32, 'RESNETS.WIDTH_PER_GROUP', 4, 'MODEL.USE_AFFINE', False,
                       'NONLOCAL.USE_AFFINE', False, 'NONLOCAL.USE_BN', True, 'MODEL.DILATIONS_AFTER_CONV5', False]
    r1, net, _ = _session(ws, 'ava_r50_lfb_nl.yaml', ov, grouped=True)
    assert any(getattr(s, 'groups', 1) > 1 for s in net.steps)
    assert any(type(s).__name__ == 'SpatialBNStep' for s in net.steps)
    r2, _, _ = _session(ws, 'ava_r50_lfb_nl.yaml', ov, grouped=True)
    _assert_identical(r1, r2)


def test_deterministic_and_default_mode_compute_the_same_step(ws):
    det, _, _ = _session(ws, 'ava_r50_lfb_nl.yaml', TINY + DET, steps=1)
    dflt, _, _ = _session(ws, 'ava_r50_lfb_nl.yaml', TINY, steps=1)
    (l1, _, g1, _), (l2, _, g2, _) = det[0], dflt[0]
    assert abs(float(l1) - float(l2)) < 1e-5 * abs(float(l2))
    # the two modes round the non-local gradient products at different points (TF32-level differences), which flips
    # near-zero ReLUs: test_gpu_model.py's gradient bounds for TF32-level perturbations apply
    err, cos = {}, {}
    for k in g1:
        a, b = g1[k].astype(np.float64), g2[k].astype(np.float64)
        nb = float(np.linalg.norm(b))
        if nb < 1e-7:
            continue
        err[k] = float(np.linalg.norm(a - b) / nb)
        cos[k] = float((a * b).sum() / (np.linalg.norm(a) * nb + 1e-30))
    print('deterministic vs default: median rel-L2 %.2e, worst %.2e, min cos %.5f' % (
        float(np.median(list(err.values()))), max(err.values()), min(cos.values())))
    assert float(np.median(list(err.values()))) < 2e-2
    for k in err:
        assert err[k] < 0.15 and cos[k] > 0.98, (k, err[k], cos[k])


def test_resume_from_a_checkpoint_is_exact(ws, tmp_path):
    """Save after step k = 3, continue to step 6; a fresh workspace loads the checkpoint, sets the step counter (the
    dropout masks' counter) to k and runs steps 4-6.  Both sides run eager steps and graph replays (the continued run
    replays its captured graph; the resumed net runs eager twice, then captures), with dropout on.  Every loss, gradient,
    momentum and parameter must be equal bit for bit."""
    from oracle import model as OM
    from utils import checkpoints as CK
    ov = TINY[:-6] + DET                   # the TINY overrides without the ones that switch dropout off
    k, more = 3, 3
    ws.ResetWorkspace()
    H.setup_cfg('ava_r50_lfb_nl.yaml', ov)
    ocfg = H.oracle_cfg('ava_r50_lfb_nl.yaml', ov)
    params = OM.make_params(ocfg, seed=2)
    inputs = OM.make_inputs(ocfg, n_clips=2, rois_per_clip=2, crop=64, frames=8)
    model, sfx = H.build('train', True)
    H.feed_params(params)
    H.feed_inputs(inputs, sfx)
    model.UpdateWorkspaceLr(10)
    name, names = model.net.Proto().name, model.TrainableParams()
    for _ in range(k):
        ws.RunNet(name)
    torch.cuda.synchronize()
    assert ws.current().step == k
    path = os.path.join(str(tmp_path), 'c2_model_iter%d.pkl' % k)
    CK.save_model_params(model, path, k - 1)
    cont = []
    for _ in range(more):
        ws.RunNet(name)
        torch.cuda.synchronize()
        cont.append(_state(ws, names))
    assert len(ws.current().nets[name]._graphs) == 1
    ws.ResetWorkspace()
    H.setup_cfg('ava_r50_lfb_nl.yaml', ov)
    model2, sfx2 = H.build('train', True)
    it, _ = CK.initialize_params_from_file(model2, path)
    assert it == k
    ws.current().step = k
    H.feed_inputs(inputs, sfx2)
    model2.UpdateWorkspaceLr(10)
    res = []
    for _ in range(more):
        ws.RunNet(model2.net.Proto().name)
        torch.cuda.synchronize()
        res.append(_state(ws, names))
    assert len(ws.current().nets[model2.net.Proto().name]._graphs) == 1
    _assert_identical(cont, res)


def test_full_size_benchmark_config_is_bitwise_reproducible(ws):
    full = ['NUM_GPUS', 1, 'TRAIN.BATCH_SIZE', 2, 'TRAIN.DROPOUT_RATE', 0.0, 'FBO_NL.INPUT_DROPOUT_ON', False,
            'FBO_NL.LFB_DROPOUT_ON', False] + DET
    r1, _, _ = _session(ws, 'ava_r50_lfb_nl.yaml', full, steps=3, crop=224, frames=32, rois=2)
    r2, _, _ = _session(ws, 'ava_r50_lfb_nl.yaml', full, steps=3, crop=224, frames=32, rois=2)
    _assert_identical(r1, r2)


if __name__ == '__main__':
    if os.environ.get('VLFB_DEBUG') != '1':
        raise SystemExit('the path records need VLFB_DEBUG=1')
    if '--forced-cp' in sys.argv:
        forced_cp_checks()
    else:
        kernel_checks()
