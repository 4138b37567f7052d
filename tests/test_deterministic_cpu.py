"""B200.DETERMINISTIC without a GPU: the schedules vlfb_gemm_plan reports for deterministic launches, the ABI's argument
rules, the compiled fix-up instantiations, and the executor's routing onto the deterministic kernel wrappers."""
import ctypes
import os
import re
import subprocess

import pytest
import torch

import harness as H
import wgrad_cases as WC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'video-long-term-feature-banks_b200', 'csrc')
TINY = ['NUM_GPUS', 1, 'TRAIN.BATCH_SIZE', 2, 'TRAIN.CROP_SIZE', 64, 'TRAIN.VIDEO_LENGTH', 8,
        'TEST.BATCH_SIZE', 2, 'TEST.CROP_SIZE', 64, 'TEST.VIDEO_LENGTH', 8, 'LFB.WINDOW_SIZE', 4,
        'TRAIN.DROPOUT_RATE', 0.0, 'FBO_NL.INPUT_DROPOUT_ON', False, 'FBO_NL.LFB_DROPOUT_ON', False]
WS_PTR = 1 << 20          # never dereferenced: plans and argument checks are host-only


def _wgrad_params(L, shape, co, ker, st, pd, dil, det, ws=True):
    from vlfb import kernels as K
    g = K.conv_geom(shape, co, ker, st, pd, dil)
    p = L.GemmParams()
    p.a.ptr, p.a.kind, p.a.ld = 256, L.OP_DENSE_MN, co
    if g.C == 4:
        p.b.ptr, p.b.kind, n = 256, L.OP_STEM_MN, g.kH * 32
    elif K._is_pointwise(g):
        p.b.ptr, p.b.kind, p.b.ld, n = 256, L.OP_DENSE_MN, g.C, g.C
    else:
        p.b.ptr, p.b.kind, n = 256, L.OP_CONV_MN, g.kH * g.kW * g.C
    p.g = g
    p.M, p.N, p.K = co, n, g.N * g.To * g.Ho * g.Wo
    p.batch, p.taps, p.split_k = 1, (1 if K._is_pointwise(g) else g.kT), 0
    p.d, p.ldd, p.d_tap_stride, p.alpha = 256, p.taps * n, n, 1.0
    p.flags = L.EPI_ATOMIC
    p.deterministic = int(det)
    if ws:
        p.workspace, p.workspace_bytes = WS_PTR, int(L.load().vlfb_gemm_workspace_bytes())
    return p


def _matmul_params(L, M, N, K_, det):
    p = L.GemmParams()
    p.a.ptr, p.a.kind, p.a.ld = 256, L.OP_DENSE_K, K_
    p.b.ptr, p.b.kind, p.b.ld = 256, L.OP_DENSE_MN, N
    p.M, p.N, p.K, p.batch, p.taps, p.split_k = M, N, K_, 1, 1, 0
    p.d, p.ldd, p.alpha, p.flags, p.deterministic = 256, N, 1.0, L.EPI_ATOMIC, int(det)
    p.workspace, p.workspace_bytes = WS_PTR, int(L.load().vlfb_gemm_workspace_bytes())
    return p


def _plan(L, p, lib=None):
    pl = L.GemmPlan()
    assert (lib or L.load()).vlfb_gemm_plan(ctypes.byref(p), 132, ctypes.byref(pl)) == 0
    return pl


GOLDEN_PLANS = os.path.join(ROOT, 'tests', 'golden', 'gemm_plans_default.json')


def default_plan_rows(lib=None):
    """Plans of the default (deterministic = 0) mode for every production wgrad and split matmul, with and without a
    workspace: [(label, ws, [tile_n, split_k, pair, stream_k, tiles, units])].  tests/golden/gemm_plans_default.json
    holds these rows as the library computed them before the deterministic field existed (regenerate with
    `python tests/test_deterministic_cpu.py LIBRARY.so`)."""
    from vlfb import libvlfb as L
    rows = []
    for ws in (True, False):
        for label, shape, co, ker, st, pd, dil, _ in WC.PRODUCTION:
            pl = _plan(L, _wgrad_params(L, shape, co, ker, st, pd, dil, False, ws=ws), lib)
            rows.append(['wgrad ' + label, ws, [getattr(pl, f) for f, _ in L.GemmPlan._fields_]])
        for M, N, K_, label in SPLIT_MATMULS:
            p = _matmul_params(L, M, N, K_, False)
            if not ws:
                p.workspace, p.workspace_bytes = None, 0
            pl = _plan(L, p, lib)
            rows.append(['matmul ' + label, ws, [getattr(pl, f) for f, _ in L.GemmPlan._fields_]])
    return rows


# the long-K products kernels.matmul splits in the benchmarked step: non-local affinity gradients (K = 3136 / 784
# positions), the classifier and its weight gradient
SPLIT_MATMULS = [(784, 784, 1024, 'nl res4 dA'), (512, 512, 3136, 'nl res3 dtheta'), (4, 80, 2560, 'classifier'),
                 (80, 2560, 4, 'classifier wgrad'), (1024, 1024, 1568, 'nl res4 dphi')]


@pytest.mark.parametrize('case', WC.PRODUCTION, ids=[c[0] for c in WC.PRODUCTION])
def test_deterministic_wgrad_plans_never_split(case):
    from vlfb import libvlfb as L
    label, shape, co, ker, st, pd, dil, _ = case
    det = _plan(L, _wgrad_params(L, shape, co, ker, st, pd, dil, True))
    assert det.split_k == 1
    assert det.stream_k in (0, 1)
    # without a workspace stream-K is not available: split 1
    nows = _plan(L, _wgrad_params(L, shape, co, ker, st, pd, dil, True, ws=False))
    assert nows.split_k == 1 and nows.stream_k == 0


def test_default_mode_plans_are_unchanged():
    """deterministic = 0 plans every production wgrad and split matmul as the library did before the field existed."""
    import json
    with open(GOLDEN_PLANS) as f:
        golden = json.load(f)['rows']
    now = default_plan_rows()
    assert len(now) == len(golden)
    for (label, ws, plan), (glabel, gws, gplan) in zip(now, golden):
        assert (label, ws) == (glabel, gws)
        assert plan == gplan, (label, ws, plan, gplan)


def test_default_mode_still_splits_long_wgrads():
    from vlfb import libvlfb as L
    label, shape, co, ker, st, pd, dil, _ = WC.PRODUCTION[0]            # conv1: 25088 K chunks per tile
    dflt = _plan(L, _wgrad_params(L, shape, co, ker, st, pd, dil, False))
    assert dflt.split_k > 1 or dflt.stream_k == 1
    det = _plan(L, _wgrad_params(L, shape, co, ker, st, pd, dil, True))
    assert det.split_k == 1 and det.stream_k == 1, 'the long-K conv1 wgrad should take the stream-K fix-up'


@pytest.mark.parametrize('M,N,K_,label', SPLIT_MATMULS)
def test_deterministic_split_matmul_plans(M, N, K_, label):
    from vlfb import libvlfb as L
    pl = _plan(L, _matmul_params(L, M, N, K_, True))
    assert pl.split_k == 1, label


def test_deterministic_atomic_launch_needs_a_workspace():
    from vlfb import libvlfb as L
    lib = L.load()
    label, shape, co, ker, st, pd, dil, _ = WC.PRODUCTION[3]
    p = _wgrad_params(L, shape, co, ker, st, pd, dil, True, ws=False)
    assert lib.vlfb_gemm(ctypes.byref(p), None) == -4 and b'workspace' in lib.vlfb_last_error()
    p.workspace, p.workspace_bytes = WS_PTR, int(lib.vlfb_gemm_workspace_bytes()) - 16
    assert lib.vlfb_gemm(ctypes.byref(p), None) == -4
    p.workspace, p.workspace_bytes = WS_PTR + 4, int(lib.vlfb_gemm_workspace_bytes())
    assert lib.vlfb_gemm(ctypes.byref(p), None) == -4
    # grouped wgrad follows the same rule
    from vlfb import kernels as K
    g = K.conv_geom((2, 8, 14, 14, 128), 128, (3, 3, 3), (1, 1, 1), (1, 1, 1))
    q = L.GemmParams()
    q.a.ptr, q.a.kind, q.a.ld = 256, L.OP_DENSE_MN, 128
    q.b.ptr, q.b.kind = 256, L.OP_CONV_MN
    q.g, q.groups = g, 32
    q.M, q.N, q.K, q.batch, q.taps = 128, 9 * 4, g.N * g.To * g.Ho * g.Wo, 1, 3
    q.d, q.ldd, q.d_tap_stride, q.alpha, q.flags, q.deterministic = 256, 3 * 36, 36, 1.0, L.EPI_ATOMIC, 1
    assert lib.vlfb_gemm(ctypes.byref(q), None) == -4
    # a deterministic launch is never split by request either
    p.workspace, p.workspace_bytes, p.split_k = WS_PTR, int(lib.vlfb_gemm_workspace_bytes()), 4
    assert lib.vlfb_gemm(ctypes.byref(p), None) == -1
    p.split_k, p.deterministic = 0, 2
    assert lib.vlfb_gemm(ctypes.byref(p), None) == -1


def test_deterministic_entry_points_are_exported():
    from vlfb import libvlfb as L
    lib = L.load()
    src = open(os.path.join(ROOT, 'include', 'vlfb_det.h')).read()
    names = sorted(set(re.findall(r'\b(vlfb_[a-z0-9_]+)\s*\(', src)))
    assert names == sorted(L.DET_SIGNATURES)
    for n in names:
        assert hasattr(lib, n), n
    assert lib.vlfb_roi_align_bwd_det_scratch_bytes(3, 14, 14, 2048) == 3 * 14 * 14 * 2048 * 4
    assert lib.vlfb_colsum_det(None, 4, None, 4, 4, 0, None) == -1
    assert lib.vlfb_roi_align_bwd_det(256, 256, 256, 1, 14, 14, 64, 2, 7, 7, 0.0625, 0, None, 0, None) == -4


def _res_usage(obj):
    out = subprocess.run(['cuobjdump', '-res-usage', obj], capture_output=True, text=True, check=True).stdout
    usage = {}
    name = None
    for line in out.splitlines():
        m = re.search(r'Function (\S+):', line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r'REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)', line)
        if m and name:
            usage[name] = tuple(int(v) for v in m.groups())
    return usage


def test_cp_async_fixup_instantiations_have_no_spills():
    """The MN x MN cp.async builds with the fix-up compiled in (A = DENSE_MN; B = DENSE_MN, STEM_MN, CONV_MN) and the
    fix-up kernel: no local memory (spills) and no stack at the 128-register cap of the 16-warp build."""
    obj = os.path.join(CSRC, 'gemm_tc.o')
    if not os.path.exists(obj):
        pytest.skip('gemm_tc.o not built (run __graft_entry__.build())')
    usage = _res_usage(obj)
    want = ['_ZN4vlfb2tc14gemm_tc_kernelILi1ELi%dELb0ELb1ELb1EEEv' % b for b in (1, 6, 4)]
    for w in want:
        hits = [k for k in usage if k.startswith(w[:-3])]
        assert hits, w
        for k in hits:
            reg, stack, local = usage[k]
            assert reg <= 128 and stack == 0 and local == 0, (k, usage[k])
    fix = [k for k in usage if 'gemm_fixup_kernel' in k]
    assert fix and all(usage[k][1] == 0 and usage[k][2] == 0 for k in fix)
    # no other cp.async build carries the fix-up
    others = [k for k in usage if re.search(r'gemm_tc_kernelILi\dELi\dELb\dELb1ELb1E', k) and
              not re.search(r'ILi1ELi[164]ELb0ELb1ELb1E', k)]
    assert not others, others


@pytest.fixture
def fake():
    import fake_kernels
    from vlfb import workspace
    fake_kernels.install()
    workspace.ResetWorkspace()
    yield fake_kernels
    workspace.ResetWorkspace()
    fake_kernels.uninstall()


DET_WRAPPERS = {'conv_wgrad': 'conv_wgrad_det', 'matmul': 'matmul_det', 'colsum': 'colsum_det',
                'roi_align_bwd': 'roi_align_bwd_det', 'spatial_bn_fwd': 'spatial_bn_fwd_det',
                'spatial_bn_bwd': 'spatial_bn_bwd_det'}


def _run_tiny(fake, monkeypatch, det):
    """One forward + backward of the tiny AVA FBO-NL net on the CPU engine; returns the calls of each wrapper."""
    from oracle import model as OM
    from vlfb import workspace
    calls = dict((k, 0) for k in list(DET_WRAPPERS) + list(DET_WRAPPERS.values()) + ['maxpool_bwd'])

    def count(name, fn):
        def f(*a, **kw):
            calls[name] += 1
            return fn(*a, **kw)
        return f
    for base, detname in DET_WRAPPERS.items():
        fn = getattr(fake, base)
        monkeypatch.setattr(fake, base, count(base, fn))
        # the deterministic stand-ins compute the same function as the default ones
        monkeypatch.setattr(fake, detname, count(detname, fn), raising=False)
    monkeypatch.setattr(fake, 'maxpool_bwd', count('maxpool_bwd', fake.maxpool_bwd))
    H.setup_cfg('ava_r50_lfb_nl.yaml', TINY + ['B200.DETERMINISTIC', det])
    ocfg = H.oracle_cfg('ava_r50_lfb_nl.yaml', TINY)
    params = OM.make_params(ocfg, seed=2)
    inputs = OM.make_inputs(ocfg, n_clips=2, rois_per_clip=2, crop=64, frames=8)
    model, sfx = H.build('train', True)
    H.feed_params(params)
    H.feed_inputs(inputs, sfx)
    net = workspace.current().nets[model.net.Proto().name]
    assert net.det == det
    net.update_ops = []
    workspace.RunNet(model.net.Proto().name)
    return calls, float(workspace.FetchBlob('gpu_0/loss'))


def test_executor_routes_a_deterministic_net_to_the_deterministic_wrappers(fake, monkeypatch):
    from vlfb import executor as X
    monkeypatch.setattr(X, 'POOL_GATHER', 0)          # the deterministic net takes the gather form anyway
    calls, loss_det = _run_tiny(fake, monkeypatch, True)
    for base, detname in DET_WRAPPERS.items():
        assert calls[base] == 0, (base, calls)
    for detname in ('conv_wgrad_det', 'matmul_det', 'colsum_det', 'roi_align_bwd_det'):
        assert calls[detname] > 0, (detname, calls)
    assert calls['maxpool_bwd'] == 0


def test_executor_never_calls_the_deterministic_wrappers_by_default(fake, monkeypatch):
    calls, _ = _run_tiny(fake, monkeypatch, False)
    for base, detname in DET_WRAPPERS.items():
        assert calls[detname] == 0, (detname, calls)
    for base in ('conv_wgrad', 'matmul', 'colsum', 'roi_align_bwd'):
        assert calls[base] > 0, (base, calls)


def test_deterministic_range_is_checked_for_grouped_launches_too():
    from vlfb import libvlfb as L
    from vlfb import kernels as K
    lib = L.load()
    g = K.conv_geom((2, 8, 14, 14, 128), 128, (3, 3, 3), (1, 1, 1), (1, 1, 1))
    q = L.GemmParams()
    q.a.ptr, q.a.kind, q.a.ld = 256, L.OP_DENSE_MN, 128
    q.b.ptr, q.b.kind = 256, L.OP_CONV_MN
    q.g, q.groups = g, 32
    q.M, q.N, q.K, q.batch, q.taps = 128, 9 * 4, g.N * g.To * g.Ho * g.Wo, 1, 3
    q.d, q.ldd, q.d_tap_stride, q.alpha, q.flags, q.deterministic = 256, 3 * 36, 36, 1.0, L.EPI_ATOMIC, 2
    q.workspace, q.workspace_bytes = WS_PTR, int(lib.vlfb_gemm_workspace_bytes())
    assert lib.vlfb_gemm(ctypes.byref(q), None) == -1


def test_roi_align_bwd_det_needs_aligned_vectors():
    from vlfb import libvlfb as L
    lib = L.load()
    nb = int(lib.vlfb_roi_align_bwd_det_scratch_bytes(2, 14, 14, 64))
    # dfeat 4 bytes off a 16-byte boundary: rejected before any launch
    assert lib.vlfb_roi_align_bwd_det(256, 256, 260, 1, 14, 14, 64, 2, 7, 7, 0.0625, 0, 4096, nb, None) == -1


def test_deterministic_config_defaults_off():
    from core.config import config as cfg
    H.setup_cfg('ava_r50_lfb_nl.yaml', TINY)
    assert cfg.B200.DETERMINISTIC is False
    assert torch is not None


if __name__ == '__main__':
    # python tests/test_deterministic_cpu.py LIBRARY.so: write the golden default-mode plans computed by that library
    import json
    import sys
    sys.path.insert(0, os.path.join(ROOT, 'video-long-term-feature-banks_b200', 'lib'))
    lib = ctypes.CDLL(sys.argv[1])
    lib.vlfb_gemm_plan.restype = ctypes.c_int
    with open(GOLDEN_PLANS, 'w') as f:
        f.write('{"rows": [\n' + ',\n'.join(json.dumps(r) for r in default_plan_rows(lib)) + '\n]}\n')
