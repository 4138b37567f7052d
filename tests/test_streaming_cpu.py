"""The streaming case table (tests/streaming_cases.py) without a GPU: the entry points it covers, the production
launches it matches, the numpy Philox generator, and that every comparison rejects a planted error."""
import re

import numpy as np
import pytest
import torch

import streaming_cases as SC

ROOT = SC.ROOT

# Exported entry points of include/vlfb.h that launch a kernel but have no case here, with the reason.
EXEMPT = {
    'vlfb_gemm': 'tensor-core GEMM: tests/gemm_paths.py',
    'vlfb_roi_align_table': 'bit-exact against oracle/roi_align_np.py in test_gpu_kernels.py; the RoIAlign cases use '
                            'that table as their reference',
}
# wrapper of vlfb.kernels -> the entry points it calls
WRAPS = {
    'affine_fwd': ['vlfb_affine_nd_fwd'], 'affine_bwd': ['vlfb_affine_nd_bwd'], 'maxpool_fwd': ['vlfb_maxpool3d_fwd'],
    'maxpool_bwd': ['vlfb_maxpool3d_bwd'], 'maxpool_bwd_gather': ['vlfb_maxpool3d_bwd_gather'],
    'avgpool_fwd': ['vlfb_avgpool3d_fwd'], 'avgpool_bwd': ['vlfb_avgpool3d_bwd'], 'roi_align_fwd': ['vlfb_roi_align_fwd'],
    'roi_align_bwd': ['vlfb_roi_align_bwd'], 'softmax_fwd': ['vlfb_softmax_fwd'], 'softmax_bwd': ['vlfb_softmax_bwd'],
    'layernorm_fwd': ['vlfb_layernorm_fwd'], 'layernorm_bwd': ['vlfb_layernorm_bwd'], 'relu_fwd': ['vlfb_relu_fwd'],
    'relu_bwd': ['vlfb_relu_bwd'], 'axpby': ['vlfb_axpby'], 'fill': ['vlfb_fill'], 'round_tf32': ['vlfb_round_tf32'],
    'add_tf32': ['vlfb_add_tf32'], 'relu_tf32': ['vlfb_relu_tf32'], 'relu_bits': ['vlfb_relu_bits'],
    'relu_bwd_tf32': ['vlfb_relu_bwd_tf32'], 'add_relu_bwd_tf32': ['vlfb_add_relu_bwd_tf32'], 'colsum': ['vlfb_colsum'],
    'sigmoid_fwd': ['vlfb_sigmoid_fwd'], 'dropout': ['vlfb_dropout_fwd'], 'copy2d': ['vlfb_copy2d'],
    'nc_to_cl': ['vlfb_nc_to_cl_round', 'vlfb_nc_to_cl_pitched'], 'cl_to_nc': ['vlfb_cl_to_nc'],
    'weight_transpose': ['vlfb_weight_transpose'], 'weight_transpose_multi': ['vlfb_weight_transpose_multi'],
    'sigmoid_ce_fwd': ['vlfb_sigmoid_ce_fwd'], 'sigmoid_ce_bwd': ['vlfb_sigmoid_ce_bwd'],
    'sgd_nesterov': ['vlfb_sgd_nesterov'], 'fbo_nl_fwd': ['vlfb_fbo_nl_fwd'], 'fbo_nl_bwd': ['vlfb_fbo_nl_bwd'],
    'spatial_bn_fwd': ['vlfb_spatial_bn_fwd'], 'spatial_bn_infer': ['vlfb_spatial_bn_infer'],
    'spatial_bn_bwd': ['vlfb_spatial_bn_bwd'], 'softmax_ce_fwd': ['vlfb_softmax_ce_fwd'],
    'softmax_ce_bwd': ['vlfb_softmax_ce_bwd'], 'fbo_bank_scan': ['vlfb_fbo_bank_scan_dt'],
    'lfb_gather': ['vlfb_lfb_gather'], 'cast_bf16': ['vlfb_cast_f32_to_bf16'],
}
# host-only queries (no launch)
HOST_ONLY = {'vlfb_version', 'vlfb_last_error', 'vlfb_gemm_plan', 'vlfb_gemm_workspace_bytes',
             'vlfb_spatial_bn_workspace_bytes', 'vlfb_fbo_bank_scan_splits', 'vlfb_fbo_bank_scan_workspace',
             'vlfb_fbo_bank_scan_splits_dt', 'vlfb_fbo_bank_scan_workspace_dt', 'vlfb_fbo_nl_scratch_floats'}
# entry points that only forward to another one (the wrapper calls the one they forward to)
FORWARDERS = {'vlfb_nc_to_cl': 'vlfb_nc_to_cl_round', 'vlfb_fbo_bank_scan': 'vlfb_fbo_bank_scan_dt'}


def _exported():
    with open(SC.os.path.join(ROOT, 'include', 'vlfb.h')) as f:
        src = f.read()
    return sorted(set(re.findall(r'^\s*(?:int|size_t|const char\*)\s+(vlfb_\w+)\s*\(', src, re.M)))


def test_every_launching_entry_point_has_a_case_or_an_exemption():
    covered = set()
    for c in SC.CASES:
        covered.update(WRAPS[c['fn']])
    missing = []
    for e in _exported():
        if e in HOST_ONLY or e in EXEMPT:
            continue
        if FORWARDERS.get(e, e) not in covered:
            missing.append(e)
    assert not missing, 'entry points with neither a case nor an exemption: %s' % missing
    assert not (set(EXEMPT) & covered), 'exempted but covered: %s' % (set(EXEMPT) & covered)


def test_every_case_has_a_builder_and_a_unique_name():
    names = [c['name'] for c in SC.CASES]
    assert len(names) == len(set(names))
    assert all(c['fn'] in SC.BUILD and c['fn'] in WRAPS for c in SC.CASES)


def test_every_production_signature_is_matched_by_a_case():
    sigs = SC.production_signatures()
    assert len(sigs) > 0
    table = [SC.case_signature(c) for c in SC.CASES]
    for s in sigs:
        assert dict(fn=s['fn'], args=s['args']) in table, s['fn']


def test_every_grid_stride_kernel_has_a_case_above_the_grid_cap():
    """Each family whose launch is a grid-stride loop over a capped grid has a case whose work exceeds the cap, so the
    loop takes a second iteration."""
    over = {}
    for c in SC.CASES:
        w = SC.work_items(c)
        if w is not None:
            over[c['fn']] = over.get(c['fn'], False) or w[0] > w[1]
    assert over and not [fn for fn, ok in over.items() if not ok], \
        'no case above the grid cap: %s' % sorted(fn for fn, ok in over.items() if not ok)
    grid_stride = set(SC.EW_ARGS) | {'sgd_nesterov', 'dropout', 'copy2d', 'nc_to_cl', 'affine_fwd', 'affine_bwd',
                                     'softmax_fwd', 'softmax_bwd', 'layernorm_fwd', 'layernorm_bwd', 'maxpool_fwd',
                                     'maxpool_bwd', 'maxpool_bwd_gather', 'avgpool_fwd', 'avgpool_bwd', 'roi_align_fwd',
                                     'roi_align_bwd', 'spatial_bn_fwd', 'spatial_bn_infer', 'spatial_bn_bwd',
                                     'softmax_ce_bwd', 'lfb_gather', 'cast_bf16'}
    assert grid_stride <= set(over)


def test_production_cases_cover_the_recorded_step():
    prod = set(c['fn'] for c in SC.CASES if c.get('prod'))
    assert {'softmax_fwd', 'softmax_bwd', 'maxpool_fwd', 'maxpool_bwd_gather', 'roi_align_fwd', 'roi_align_bwd',
            'fbo_nl_fwd', 'fbo_nl_bwd', 'dropout', 'colsum', 'sgd_nesterov', 'nc_to_cl'} <= prod


def test_bank_scan_cases_reach_one_and_many_splits_with_a_partial_last_split():
    splits = []
    for c in SC.CASES:
        if c['fn'] == 'fbo_bank_scan':
            R, L, D = c['args']['bank']['shape']
            S = SC.scan_splits(R, L, D, c['args']['bank']['dtype'] == 'bfloat16')
            splits.append((S, L % -(-L // S) != 0))
    assert {S for S, _ in splits} >= {1} and max(S for S, _ in splits) >= 8 and any(p for _, p in splits)


def test_philox_known_answer():
    """Random123 kat_vectors: philox4x32 10 rounds, counter 0, key 0 -> 6627e8d5 e169c58d bc57ac4c 9b00dbd8 (the same
    value curand's Philox4_32_10 produces for that counter and key)."""
    got = SC.philox4x32_10([0], 0)[0]
    assert [int(v) for v in got] == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]


def test_dropout_keep_mask_uses_word_j_mod_4_of_block_j_div_4():
    r = SC.philox4x32_10(np.arange(10, 13, dtype=np.uint64) + (np.uint64(3) << np.uint64(32)), 99).reshape(-1)
    u = (r >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)
    assert np.array_equal(SC.dropout_keep(11, 0.3, 99, 10, 3), u[:11] >= np.float32(0.3))


def _prep(name):
    return SC.prepare(SC.case_by_name(name), 'cpu')


def _out(P, name):
    return next(o for o in P.outs if o['name'] == name)


def _rejects(o, bad):
    assert SC.compare(o['ref'].to(bad.dtype) if o['bound'] is None else o['ref'], o['ref'], o['bound'], o['tol'])['ok']
    assert not SC.compare(bad, o['ref'], o['bound'], o['tol'])['ok']


def test_planted_softmax_bwd_without_dot():
    P = _prep('softmax_bwd_c784')
    c = P.case
    o = _out(P, 'dx')
    p = [t for t in P.keep if t.shape == tuple(c['args']['p']['shape'])]
    bad = SC.softmax_bwd_ref(p[0].double(), p[1].double(), 0.125, dot=False)
    _rejects(o, bad)


def test_planted_layernorm_bwd_without_y_term():
    P = _prep('layernorm_bwd_c784')
    y, dy, sd = P.keep[0].double(), P.keep[1].double(), P.keep[2].double().view(-1, 1)
    _rejects(_out(P, 'dx'), SC.layernorm_bwd_ref(dy, y, sd, yterm=False))


def test_planted_avgpool_bwd_missing_border_window():
    P = _prep('avgpool_bwd_s2_overlap')
    o = _out(P, 'dx')
    g = P.case['args']['g']
    dy = P.keep[0]
    prev = o['ref'] - SC.avgpool_bwd_ref(dy, g)
    _rejects(o, SC.avgpool_bwd_ref(dy, g, drop_window=True) + prev)


def test_planted_roi_align_swapped_weights_on_a_clamped_sample():
    c = SC.case_by_name('roi_align_fwd_edges')
    P = SC.prepare(c, 'cpu')
    o = _out(P, 'out')
    rois, feat = P.keep[0], P.keep[1]
    N, H, W, C = feat.shape
    R, PH, PW, _ = o['ref'].shape
    M, _ = SC.roi_matrix(rois, N, H, W, PH, PW, 1.0 / 16, 0, swap_clamped=True)
    _rejects(o, (M @ feat.double().view(-1, C)).view(R, PH, PW, C))


def test_planted_colsum_missing_last_slab():
    P = _prep('colsum_r1200_c512_ld512')
    o = _out(P, 'out')
    a = P.case['args']
    _, slabs, rpb = SC.colsum_terms(a['rows'], a['cols'])
    assert slabs > 1
    x = P.keep[0].view(a['rows'], a['ld'])[:, :a['cols']].double()
    _rejects(o, o['ref'] - x[(slabs - 1) * rpb:].sum(0))


def test_planted_dropout_mask_shifted_by_one():
    P = _prep('dropout_n4005')
    o = _out(P, 'y')
    x = P.keep[0]
    shifted = torch.roll(P.mask, 1)
    inv = float(np.float32(1) / (np.float32(1) - np.float32(0.25)))
    _rejects(o, torch.where(shifted, x * inv, torch.zeros(())))


def test_planted_maxpool_argmax_last_tie():
    P = _prep('maxpool_fwd_ties')
    o = _out(P, 'argmax')
    g = P.case['args']['g']
    _, last = SC.maxpool_ref(P.keep[0], g, last_tie=True)
    _rejects(o, last)


def test_planted_fbo_dropout_mask_shifted():
    """The FBO-NL stack's a_out with its dropout mask shifted by one element fails the bound."""
    P = _prep('fbo_nl_fwd_L1')
    o = _out(P, 'L0.a_out')
    out = _out(P, 'L0.out')['ref']
    keep = P.keeps[0]
    inv = float(np.float32(1) / (np.float32(1) - np.float32(0.2)))
    a0 = o['ref'] - out * keep * inv
    bad = a0 + out * torch.roll(keep.reshape(-1), 1).view(keep.shape) * inv
    _rejects(o, bad)


def test_planted_bn_dx_without_the_bx_term():
    P = _prep('spatial_bn_bwd_r1051_c64')
    o = _out(P, 'dx')
    x, dy, s, sm, siv = (t.double() for t in P.keep[:5])
    _rejects(o, SC.bn_bwd_ref(dy, x, s, sm, siv, bx=False))


def test_planted_layernorm_one_pass_variance_on_mean_far_above_std():
    """E[x^2] - E[x]^2 loses the variance of the mean >> std rows; their bound is tight enough to see it."""
    P = _prep('layernorm_fwd_c784')
    o = _out(P, 'y')
    x = P.keep[0].double()
    mu = x.mean(1, keepdim=True)
    var = ((x.float() * x.float()).mean(1, keepdim=True) - (x.float().mean(1, keepdim=True)) ** 2).double().clamp(min=0)
    _rejects(o, (x - mu) / (var + 1e-5).sqrt())


def test_planted_guard_write():
    P = _prep('copy2d_gaps')
    o = _out(P, 'dst')
    buf = o['buf'].clone()
    buf[o['index'].reshape(-1)] = o['ref'].reshape(-1).float()
    assert SC.guard_touched(buf, o['index']) == 0
    a = P.case['args']
    buf[SC.GUARD + a['dst_off'] + a['cols']] = 0.0               # the first element of the gap after row 0
    assert SC.guard_touched(buf, o['index']) == 1


@pytest.mark.parametrize('name', [c['name'] for c in SC.CASES if not c.get('prod') and not c['name'].endswith('_big')])
def test_case_builds_and_its_reference_passes_its_own_check(name):
    P = SC.prepare(SC.case_by_name(name), 'cpu')
    assert P.outs and P.call is not None
    for o in P.outs:
        r = o['ref']
        assert bool(torch.isfinite(r.double()).all()) if r.is_floating_point() else True
        assert SC.compare(r.to(torch.float32) if o['bound'] is None and r.is_floating_point() else r, r, o['bound'])['ok']
