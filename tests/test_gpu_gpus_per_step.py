"""B200.GPUS_PER_STEP on the H100: the segmented loss and SpatialBN kernels (include/vlfb_seg.h) against fp64 at
production shapes, their S = 1 forms against the existing kernels, their deterministic forms for repeatability; packed
tiny AVA and ResNeXt + SpatialBN training steps against ITER_SIZE = 4, eager against replay, one capture for every RoI
distribution, and the launch audit of packed nets (tests/launch_audit_seg.py)."""
import contextlib

import numpy as np
import pytest
import torch

import harness as H
import launch_audit as LA
import streaming_cases as SC
from util import run_worker

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def K():
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from vlfb import kernels
    return kernels


def _seg_rows(S, rows, gen):
    """Unequal row offsets over `rows` rows, with an empty segment when S > 2."""
    cuts = sorted(torch.randint(0, rows + 1, (S - 1,), generator=gen).tolist())
    if S > 2:
        cuts[1] = cuts[0]
    return [0] + cuts + [rows]


@pytest.mark.parametrize('S', [1, 2, 4, 8])
def test_sigmoid_ce_seg_against_fp64(K, S):
    gen = torch.Generator().manual_seed(S)
    rows, cols, live = 16 * S, 80, 13 * S           # 3S padded rows (label -1) at the end, as ROI_CAPACITY feeds them
    x = torch.randn(rows, cols, generator=gen) * 3
    t = (torch.rand(rows, cols, generator=gen) < 0.1).to(torch.int32)
    t[live:] = -1
    t[1, :7] = -1
    offs = _seg_rows(S, live, gen)
    seg = torch.tensor(offs, dtype=torch.int32).cuda()
    xd, scale = x.double(), 0.125
    loss = torch.empty(1, device='cuda')
    K.sigmoid_ce_seg_fwd(x.cuda(), t.cuda(), seg, loss, scale)
    dl = torch.tensor([0.75], device='cuda')
    dx = torch.full((rows, cols), float('nan'), device='cuda')
    K.sigmoid_ce_seg_bwd(x.cuda(), t.cuda(), seg, dl, dx, scale)
    ref, bound = torch.zeros(1, dtype=torch.float64), torch.zeros(1, dtype=torch.float64)
    dref, dbound = torch.zeros_like(xd), torch.zeros_like(xd)
    ends = offs[:-1] + [rows]
    for j in range(S):
        r0, r1 = offs[j], ends[j + 1]
        if r1 == r0:
            continue
        l, b = SC.sigmoid_ce_fwd_ref(xd[r0:r1], t[r0:r1], scale)
        ref, bound = ref + l, bound + b + SC.U * (ref.abs() + l.abs())
        g, gb = SC.sigmoid_ce_bwd_ref(xd[r0:r1], t[r0:r1], scale, 0.75)
        dref[r0:r1], dbound[r0:r1] = g, gb
    assert (loss.cpu().double() - ref).abs().item() <= bound.item() + 1e-12
    err = (dx.cpu().double() - dref).abs()
    assert bool((err <= dbound + 1e-30).all()), float((err - dbound).max())
    if S == 1:                                      # the unsegmented kernels, bit for bit
        l1, d1 = torch.empty(1, device='cuda'), torch.empty(rows, cols, device='cuda')
        K.sigmoid_ce_fwd(x.cuda(), t.cuda(), l1, scale)
        K.sigmoid_ce_bwd(x.cuda(), t.cuda(), dl, d1, scale)
        assert torch.equal(l1, loss) and torch.equal(d1, dx)


def _bn_inputs(S, C, seg_rows, seed):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(S * seg_rows, C, generator=gen) * 2 + torch.randn(C, generator=gen) * 3
    x.view(S, seg_rows, C).add_(torch.randn(S, 1, C, generator=gen))       # every virtual GPU its own statistics
    dy = torch.randn(S * seg_rows, C, generator=gen)
    s, b = torch.rand(C, generator=gen) + 0.5, torch.randn(C, generator=gen)
    rm, rv = torch.randn(C, generator=gen), torch.rand(C, generator=gen) + 0.5
    return x, dy, s, b, rm, rv


def _bn_run(K, x, dy, s, b, rm, rv, S, det, ds0, db0):
    C = x.shape[1]
    sm, siv = torch.empty(S, C, device='cuda'), torch.empty(S, C, device='cuda')
    y, dx = torch.empty_like(x).cuda(), torch.empty_like(x).cuda()
    rmg, rvg, ds, db = rm.cuda(), rv.cuda(), ds0.cuda(), db0.cuda()
    K.spatial_bn_seg_fwd(x.cuda(), s.cuda(), b.cuda(), rmg, rvg, sm, siv, y, 1e-5, 0.9, S, det=det)
    K.spatial_bn_seg_bwd(dy.cuda(), x.cuda(), s.cuda(), sm, siv, dx, ds, db, S, det=det)
    return dict(y=y, sm=sm, siv=siv, rm=rmg, rv=rvg, dx=dx, ds=ds, db=db)


@pytest.mark.parametrize('det', [False, True])
@pytest.mark.parametrize('S', [1, 2, 4, 8])
def test_spatial_bn_seg_against_fp64(K, S, det):
    """res4-sized activations: 2 clips x 4 x 14 x 14 rows per virtual GPU, C = 256."""
    C, n = 256, 2 * 4 * 14 * 14
    x, dy, s, b, rm, rv = _bn_inputs(S, C, n, 10 * S + det)
    ds0, db0 = torch.randn(C), torch.randn(C)
    got = _bn_run(K, x, dy, s, b, rm, rv, S, det, ds0, db0)
    xd, dyd, sd, bd = x.double(), dy.double(), s.double(), b.double()
    ds_ref, db_ref = ds0.double(), db0.double()
    for j in range(S):
        sl = slice(j * n, (j + 1) * n)
        f = SC.bn_fwd_ref(xd[sl], sd, bd, n, 1e-5, rm.double() if j == 0 else None, rv.double() if j == 0 else None, 0.9)
        checks = [('y', got['y'][sl], f['y']), ('sm', got['sm'][j], f['sm']), ('siv', got['siv'][j], f['siv'])]
        if j == 0:
            checks += [('rm', got['rm'], f['rm']), ('rv', got['rv'], f['rv'])]
        bw = SC.bn_bwd_refb(dyd[sl], xd[sl], sd, got['sm'][j].cpu().double(), got['siv'][j].cpu().double(), n,
                            ds_ref, db_ref)
        checks.append(('dx', got['dx'][sl], bw['dx']))
        ds_ref, db_ref = bw['ds'][0], bw['db'][0]
        dsb = bw['ds'][1] if j == 0 else dsb + bw['ds'][1]
        dbb = bw['db'][1] if j == 0 else dbb + bw['db'][1]
        for name, val, (ref, bound) in checks:
            err = (val.cpu().double() - ref).abs()
            assert bool((err <= bound + 1e-30).all()), (name, j, float((err - bound).max()))
    assert bool(((got['ds'].cpu().double() - ds_ref).abs() <= dsb).all())
    assert bool(((got['db'].cpu().double() - db_ref).abs() <= dbb).all())


def test_spatial_bn_seg_with_one_segment_is_the_existing_kernel(K):
    C, n = 256, 2 * 4 * 14 * 14
    x, dy, s, b, rm, rv = _bn_inputs(1, C, n, 3)
    ds0, db0 = torch.randn(C), torch.randn(C)
    for det in (False, True):
        got = _bn_run(K, x, dy, s, b, rm, rv, 1, det, ds0, db0)
        sm, siv = torch.empty(C, device='cuda'), torch.empty(C, device='cuda')
        y, dx = torch.empty_like(x).cuda(), torch.empty_like(x).cuda()
        rmg, rvg, ds, db = rm.cuda(), rv.cuda(), ds0.cuda(), db0.cuda()
        (K.spatial_bn_fwd_det if det else K.spatial_bn_fwd)(x.cuda(), s.cuda(), b.cuda(), rmg, rvg, sm, siv, y, 1e-5, 0.9)
        (K.spatial_bn_bwd_det if det else K.spatial_bn_bwd)(dy.cuda(), x.cuda(), s.cuda(), sm, siv, dx, ds, db)
        pairs = [(got['y'], y), (got['sm'][0], sm), (got['siv'][0], siv), (got['rm'], rmg), (got['rv'], rvg),
                 (got['dx'], dx), (got['ds'], ds), (got['db'], db)]
        for a, e in pairs:
            if det:
                assert torch.equal(a, e)
            else:                               # the spread of the fp64 atomic ordering, rounded to fp32
                assert float((a - e).abs().max()) <= 4e-6 * float(e.abs().max()) + 1e-30


def test_deterministic_forms_repeat_bitwise(K):
    C, n, S = 256, 2 * 4 * 14 * 14, 4
    x, dy, s, b, rm, rv = _bn_inputs(S, C, n, 7)
    ds0, db0 = torch.zeros(C), torch.zeros(C)
    a = _bn_run(K, x, dy, s, b, rm, rv, S, True, ds0, db0)
    for _ in range(2):
        c = _bn_run(K, x, dy, s, b, rm, rv, S, True, ds0, db0)
        assert all(torch.equal(a[k], c[k]) for k in a)


# --------------------------------------------------------------------------------------------- whole steps
YAML = 'ava_r50_lfb_nl.yaml'
TINY = ['TRAIN.CROP_SIZE', 64, 'TRAIN.VIDEO_LENGTH', 8, 'LFB.WINDOW_SIZE', 4, 'TRAIN.DROPOUT_RATE', 0.0,
        'FBO_NL.INPUT_DROPOUT_ON', False, 'FBO_NL.LFB_DROPOUT_ON', False]


RESNEXT = LA.RESNEXT
# no weight decay: the momentum after one update from zero is lr x the summed gradient, one fp32 rounding
NO_WD = ['SOLVER.WEIGHT_DECAY', 0.0, 'SOLVER.WEIGHT_DECAY_BN', 0.0]
# test_gpu_model.py's bounds on TF32 gradients: relative L2 and cosine per tensor, median relative L2 over tensors
GRAD_L2_TOL, GRAD_COS_TOL, GRAD_MEDIAN_L2_TOL = 0.15, 0.98, 2e-2


def _ov(extra, k=1, v=1):
    return TINY + extra + ['NUM_GPUS', 4, 'TRAIN.BATCH_SIZE', 4, 'TEST.BATCH_SIZE', 4, 'B200.ITER_SIZE', k,
                           'B200.GPUS_PER_STEP', v]


def _inputs(rois, grouped=False):
    import resnext_oracle as RO
    from oracle import model as OM
    ocfg = H.oracle_cfg(YAML, _ov(RESNEXT if grouped else []))
    with (RO.grouped() if grouped else contextlib.nullcontext(OM)) as OMg:
        params = OMg.make_params(ocfg, seed=2)
    inputs = OM.make_inputs(ocfg, n_clips=4, rois_per_clip=2, crop=64, frames=8)
    inputs['proposals'][:, 0] = torch.arange(4).repeat_interleave(torch.tensor(rois)).to(torch.float32)
    return params, inputs


def _clips(inputs, lo, hi):
    rois = inputs['proposals']
    sel = (rois[:, 0] >= lo) & (rois[:, 0] < hi)
    pr = rois[sel].clone()
    pr[:, 0] -= lo
    return {'data': inputs['data'][lo:hi], 'labels': inputs['labels'][sel], 'lfb': inputs['lfb'][sel], 'proposals': pr}


def _train(ov, params, batches, runs=1, after_first=None):
    from vlfb import workspace
    workspace.ResetWorkspace()
    H.setup_cfg(YAML, ov)
    model, sfx = H.build('train', True)
    H.feed_params(params)
    model.UpdateWorkspaceLr(10)
    name = model.net.Proto().name
    net = workspace.current().nets[name]
    losses = []
    for _ in range(runs):
        for mb in batches:
            H.feed_inputs(mb, sfx)
            workspace.RunNet(name)
            losses.append(float(workspace.FetchBlob('gpu_0/loss')))
            if after_first is not None and len(losses) == 1:
                after_first()
    mom = dict((n, workspace.FetchBlob('gpu_0/' + n + '_momentum').copy()) for n in net.trainable)
    return losses, mom, net


def _grad_bounds(got, ref):
    """Every tensor's relative L2 error and cosine, and the median relative L2, within test_gpu_model.py's bounds (which
    likewise skip mathematically zero gradients)."""
    errs, coss = {}, {}
    top = max(np.linalg.norm(ref[n].astype(np.float64)) for n in ref)
    for n in ref:
        g, r = got[n].astype(np.float64).ravel(), ref[n].astype(np.float64).ravel()
        nr = np.linalg.norm(r)
        if nr < 1e-4 * top:
            # a mathematically zero gradient (e.g. a bias that a softmax or a normalisation cancels, the phi_b / g_b /
            # out_b of a non-local block): both sides are rounding noise, held to an absolute bound instead
            assert np.linalg.norm(g - r) < 1e-4 * top, (n, np.linalg.norm(g - r), top)
            continue
        errs[n] = float(np.linalg.norm(g - r) / nr)
        coss[n] = float(g @ r / (np.linalg.norm(g) * nr + 1e-300))
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:3]
    print('packed vs ITER_SIZE: median rel-L2 %.2e, worst %s, min cos %.5f' % (
        float(np.median(list(errs.values()))), worst, min(coss.values())))
    assert float(np.median(list(errs.values()))) < GRAD_MEDIAN_L2_TOL
    for n in errs:
        assert errs[n] < GRAD_L2_TOL and coss[n] > GRAD_COS_TOL, (n, errs[n], coss[n])


@pytest.mark.parametrize('net_kind', ['ava_fbo_nl', 'resnext_bn'])
def test_packed_step_matches_iter_size(net_kind):
    """GPUS_PER_STEP = 4 against ITER_SIZE = 4 on the same four clips (virtual GPUs of 1, 3, 2 and 2 RoIs), compared
    through the momentum after the update (lr x the summed gradient, with no weight decay).  The two differ by TF32
    rounding of differently shaped GEMMs only.  On ResNeXt the step runs the segmented SpatialBN kernels and the running
    statistics are virtual GPU 0's: those of ITER_SIZE's first micro-step, within the same TF32 noise."""
    from vlfb import executor as X
    from vlfb import workspace
    grouped = net_kind == 'resnext_bn'
    extra = NO_WD + (RESNEXT if grouped else [])
    params, inputs = _inputs([1, 3, 2, 2], grouped)
    first = {}

    def after_first():
        st = workspace.current().params
        first.update((n, workspace.FetchBlob('gpu_0/' + n).copy()) for n in st.index if n.endswith(('_rm', '_riv')))

    ref_l, ref, _ = _train(_ov(extra, k=4), params, [_clips(inputs, c, c + 1) for c in range(4)], after_first=after_first)
    got_l, got, net = _train(_ov(extra, v=4), params, [inputs])
    assert net.gpus_per_step == 4
    assert any(isinstance(st, X.SpatialBNStep) for st in net.steps) == grouped
    assert abs(got_l[0] - sum(ref_l)) < 1e-3 * abs(sum(ref_l))
    _grad_bounds(got, ref)
    if grouped:
        assert first
        for n, r in first.items():
            g = workspace.FetchBlob('gpu_0/' + n).astype(np.float64)
            assert np.linalg.norm(g - r) <= 2e-2 * np.linalg.norm(r) + 1e-6, n       # TF32 noise of the forward


def test_deterministic_replay_equals_eager():
    from core.config import config as cfg
    params, inputs = _inputs([1, 3, 2, 2])
    _, eager, _ = _train(_ov(['B200.DETERMINISTIC', True, 'B200.CUDA_GRAPH', False], v=4), params, [inputs], runs=4)
    _, replay, net = _train(_ov(['B200.DETERMINISTIC', True], v=4), params, [inputs], runs=4)
    assert cfg.B200.CUDA_GRAPH and len(net._graphs) == 1
    for n in eager:
        assert np.array_equal(eager[n], replay[n]), n


def test_roi_capacity_replays_one_capture_for_every_roi_distribution():
    params, inputs = _inputs([2, 2, 2, 2])
    dists = [[2, 2, 2, 2], [1, 3, 2, 2], [4, 0, 1, 3], [0, 0, 8, 0], [2, 2, 2, 2]]
    from vlfb import workspace
    workspace.ResetWorkspace()
    H.setup_cfg(YAML, _ov(['B200.ROI_CAPACITY', 12], v=4))
    model, sfx = H.build('train', True)
    H.feed_params(params)
    model.UpdateWorkspaceLr(10)
    name = model.net.Proto().name
    net = workspace.current().nets[name]
    for d in dists:
        inputs['proposals'][:, 0] = torch.arange(4).repeat_interleave(torch.tensor(d)).to(torch.float32)
        H.feed_inputs(inputs, sfx)
        workspace.RunNet(name)
        offs = np.concatenate([[0], np.cumsum(d)])
        assert np.array_equal(workspace.current().roi_segments['proposals' + sfx].cpu().numpy(), offs)
        assert np.isfinite(float(workspace.FetchBlob('gpu_0/loss')))
    assert len(net._graphs) == 1


@pytest.mark.parametrize('net', sorted(__import__('launch_audit_seg').NETS))
def test_every_launch_of_a_packed_net_matches_fp64(net):
    """tests/launch_audit_seg.py: every kernel call of two eager steps of a packed net, the segmented ones included,
    against fp64 from its own tensors."""
    import launch_audit_seg as LAS
    p, recs = run_worker('launch_audit_seg.py', ['--net', net], timeout=1200)
    print('\n[%s]\n%s' % (net, p.stdout[-3000:]))
    assert p.returncode == 0, p.stderr[-4000:]
    *recs, tail = recs
    assert not tail['missing'], 'wrappers the net never reached: %s' % tail['missing']
    bad = [r for r in recs if not r['ok']]
    assert not bad, '\n'.join(e for r in bad[:20] for e in r['errors'])
    seg = [r for r in recs if r['wrapper'] in LAS.SEG_WRAPPERS]
    assert seg and {r['run'] for r in seg} == {1, 2}
