"""Path matrix of the tensor-core GEMM (csrc/gemm_tc.cu): a table of seeded, self-describing cases, each ONE vlfb_gemm call
whose result is checked elementwise against an fp64 PyTorch reference, and whose path record (the VLFB_DEBUG line of
launch()) is compared with the path the case declares.

The loader / schedule switches of the library (VLFB_TMA, VLFB_IM2COL, ...) are read once per process, so every
configuration runs in its own process:

    python tests/gemm_paths.py --config NAME --out FILE

writes one JSON record per case that lists NAME among its configurations.  tests/test_gpu_gemm_paths.py drives it;
tests/test_gemm_paths_cpu.py checks the table and the comparison itself without a GPU.  Besides the path cases, the
default configuration runs the weight gradient at every production geometry of tests/wgrad_cases.py, the wide-tile
forms and the conv1 column mask.

Every output lives inside a NaN-filled buffer with a guard band (a lead-in, rows past M, ldd > N where the caller
controls ldd, gaps between batches): after the call each in-range element must be finite and within the bound of
`compare`, and every other element must still be the NaN it was filled with, bit for bit.
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (os.path.join(ROOT, 'video-long-term-feature-banks_b200', 'lib'), HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import wgrad_cases as WC  # noqa: E402
from util import (capture_fd2, compare, guard_touched, nan_buffer, pack_sign_bits, parse_record,  # noqa: E402,F401
                  tf32_round, ulp_tf32)

# Tolerance of the accumulation, relative to sum_k |A[m,k]| |B[n,k]| (the operands are TF32-exact, so every product
# is exact and only the fp32 additions err).  The wgmma accumulator adds each k8 step to the running fp32 sum with at
# most one ulp (2^-23, truncation allowed) of a partial sum bounded by sum |A||B|, so over ceil(K/8) steps plus the
# in-MMA reduction the error is below (ceil(K/8) + 8) 2^-23 sum |A||B|.  tau(K) is that bound times TAU_SAFETY (the
# split-K / stream-K partial sums add a few more roundings of the same size).  A missing 32-wide K chunk of a random
# tile shifts an element by ~sqrt(32) times a typical |A||B| term, far above tau(K) sum |A||B| (test_gemm_paths_cpu.py
# shows the check rejects it at the largest K of the table).
TAU_SAFETY = 4.0
# The table's K stays in the range the worker's fp64 references handle quickly, and where the suite's global relative
# check holds; only the weight gradients marked long_k (the production geometries, K = N To Ho Wo) go beyond it.
KMAX = 16000


def tau(K):
    return TAU_SAFETY * (-(-K // 8) + 8) * 2.0 ** -23

# the fp32 epilogue (scale, bias, residual, accumulate) rounds a few times: 2^-22 of the magnitudes it adds
EPS32 = 2.0 ** -22
GUARD = 64                     # lead-in guard floats (keeps d 16-byte aligned)

CONFIGS = {
    'default': {},
    'tma0': {'VLFB_TMA': '0'},
    'im2col0': {'VLFB_IM2COL': '0'},
    'nopatch': {'VLFB_NO_PATCH': '1'},
    'nopar': {'VLFB_NO_PAR': '1'},
}

OP_DENSE_K, OP_DENSE_MN, OP_CONV_K, OP_DGRAD_K, OP_CONV_MN, OP_STEM_K, OP_STEM_MN = range(7)


# ----------------------------------------------------------------------------------------------- path records
def matches(rec, expect):
    """Fields of `expect` that the record contradicts ([] = it took the declared path).  An expected value '>N'
    means greater than N."""
    bad = []
    for k, want in expect.items():
        got = rec.get(k)
        if isinstance(want, str) and want.startswith('>'):
            ok = got is not None and got > int(want[1:])
        else:
            ok = tuple(got) == tuple(want) if isinstance(want, (tuple, list)) else got == want
        if not ok:
            bad.append('%s=%r (declared %r)' % (k, got, want))
    return bad


# ----------------------------------------------------------------------------------------------- the case table
def G(N, T, H, W, C, Co, ker, st=(1, 1, 1), pd=(0, 0, 0), dil=(1, 1, 1)):
    return dict(N=N, T=T, H=H, W=W, C=C, Co=Co, ker=ker, st=st, pd=pd, dil=dil)


def _case(name, op, seed, runs, **kw):
    c = dict(name=name, op=op, seed=seed, runs=runs, opts=kw.pop('opts', {}))
    c.update(kw)
    return c


# runs: configuration -> the path fields the case must take there (kinds / mask / tma / cp / bn / sk / fix / lean /
# bits2 / patch / par / split as printed by VLFB_DEBUG).  Kinds: 0 DENSE_K, 1 DENSE_MN, 2 CONV_K, 3 DGRAD_K, 4 CONV_MN,
# 5 STEM_K, 6 STEM_MN.  tma_a: 0 cp.async, 1 TMA tiled, 2 im2col, 3 stem; tma_b: 0 cp.async, 1 TMA tiled.  MN-major
# operands always report 0.
CASES = []


def _add(*a, **kw):
    CASES.append(_case(*a, **kw))


# ---- convolution forward (kernels.conv_fwd): CONV_K x DENSE_K
_add('fwd_3x3_res_relu_bits', 'conv_fwd', 1, geom=G(2, 3, 9, 10, 32, 64, (1, 3, 3), pd=(0, 1, 1)),
     epi=dict(scale=True, bias=True, residual=True, relu=True, bits=True),
     runs={'default': dict(kinds=(2, 0), mask=0, tma=(2, 1), cp=0, lean=1, bits2=0),
           'im2col0': dict(kinds=(2, 0), tma=(0, 1), cp=1, lean=0, bits2=1),
           'tma0': dict(kinds=(2, 0), tma=(0, 0), cp=1, bits2=1)})
_add('fwd_dilated_t96', 'conv_fwd', 2, geom=G(1, 2, 14, 14, 64, 112, (1, 3, 3), pd=(0, 2, 2), dil=(1, 2, 2)),
     epi=dict(bias=True, tf32=True), opts=dict(tile_n=96),
     runs={'default': dict(kinds=(2, 0), tma=(2, 1), cp=0, bn=96),
           'im2col0': dict(kinds=(2, 0), tma=(0, 1), cp=1, bn=96)})
_add('fwd_strided_t32_ntail', 'conv_fwd', 3, geom=G(2, 2, 14, 14, 32, 80, (1, 3, 3), st=(1, 2, 2), pd=(0, 1, 1)),
     epi=dict(scale=True, relu=True), opts=dict(tile_n=32),
     runs={'default': dict(kinds=(2, 0), tma=(2, 1), cp=0, bn=32),
           'im2col0': dict(kinds=(2, 0), tma=(0, 1), cp=1, bn=32)})
_add('fwd_temporal_t128', 'conv_fwd', 4, geom=G(1, 4, 7, 7, 256, 288, (3, 1, 1), pd=(1, 0, 0)),
     epi=dict(bias=True), opts=dict(tile_n=128),
     runs={'default': dict(kinds=(2, 0), tma=(2, 1), cp=0, bn=128),
           'tma0': dict(kinds=(2, 0), tma=(0, 0), cp=1, bn=128)})
# ---- conv1 stem forward (STEM_K x DENSE_K): patch tiles, TMA rows without patches, cp.async on a dense clip
_add('stem_fwd_patch', 'conv_fwd', 5, geom=G(1, 4, 32, 32, 4, 64, (5, 7, 7), st=(1, 2, 2), pd=(2, 3, 3)), pitched=True,
     epi=dict(scale=True, bias=True, relu=True, bits=True),
     runs={'default': dict(kinds=(5, 0), tma=(3, 1), patch=1, cp=0, lean=1, bits2=0),
           'nopatch': dict(kinds=(5, 0), tma=(3, 1), patch=0, cp=0),
           'tma0': dict(kinds=(5, 0), tma=(0, 0), patch=0, cp=1, bits2=1)})
_add('stem_fwd_rows_ho18', 'conv_fwd', 6, geom=G(1, 4, 36, 64, 4, 64, (5, 7, 7), st=(1, 2, 2), pd=(2, 3, 3)),
     pitched=True, epi=dict(bias=True),
     runs={'default': dict(kinds=(5, 0), tma=(3, 1), patch=0, cp=0)})
# a requested tile wider than N leaves B without a tensor map, so the launch is a cp.async build with the general
# epilogue: conv1 must then stage A as TMA rows, not as 16 x 8 patch tiles, whose rows only the lean epilogue maps back
# (the patch tiles stored each tile's rows in the wrong places)
_add('stem_fwd_patch_needs_tma_b', 'conv_fwd', 35, geom=G(1, 2, 48, 64, 4, 96, (5, 7, 7), st=(1, 2, 2), pd=(2, 3, 3)),
     pitched=True, epi=dict(scale=True, bias=True, relu=True, tf32=True), opts=dict(tile_n=128, stream_k=1),
     runs={'default': dict(kinds=(5, 0), tma=(3, 0), patch=0, cp=1, bn=128, lean=0)})
_add('stem_fwd_dense_clip', 'conv_fwd', 7, geom=G(2, 3, 20, 20, 4, 64, (5, 7, 7), st=(1, 2, 2), pd=(2, 3, 3)),
     epi=dict(relu=True),
     runs={'default': dict(kinds=(5, 0), tma=(0, 1), patch=0, cp=1)})
# ---- convolution dgrad (kernels.conv_dgrad): DGRAD_K x DENSE_K, parity classes, strided gather, ReLU masks
_add('dgrad_unit_accum', 'conv_dgrad', 8, geom=G(1, 3, 9, 10, 64, 32, (1, 3, 3), pd=(0, 1, 1)),
     epi=dict(accum=True),
     runs={'default': dict(kinds=(3, 0), mask=0, tma=(2, 1), cp=0, par=0),
           'im2col0': dict(kinds=(3, 0), mask=0, tma=(0, 1), cp=1),
           'tma0': dict(kinds=(3, 0), mask=0, tma=(0, 0), cp=1)})
_add('dgrad_parity_bits_tf32', 'conv_dgrad', 9, geom=G(2, 2, 30, 30, 64, 128, (1, 3, 3), st=(1, 2, 2), pd=(0, 1, 1)),
     epi=dict(residual=True, mask_bits=True, tf32=True),
     runs={'default': dict(kinds=(3, 0), mask=1, tma=(2, 1), cp=0, par='>0'),
           'nopar': dict(kinds=(3, 0), mask=1, tma=(0, 1), cp=1, par=0),
           'im2col0': dict(kinds=(3, 0), mask=1, tma=(0, 1), cp=1, par=0)})
_add('dgrad_parity_plain', 'conv_dgrad', 10, geom=G(3, 2, 20, 12, 128, 64, (1, 1, 1), st=(1, 2, 2)),
     epi=dict(),
     runs={'default': dict(kinds=(3, 0), mask=0, tma=(2, 1), cp=0, par='>0')})
_add('dgrad_strided_gather', 'conv_dgrad', 11, geom=G(1, 2, 15, 15, 32, 64, (1, 3, 3), st=(1, 2, 2), pd=(0, 1, 1)),
     epi=dict(residual=True),
     runs={'default': dict(kinds=(3, 0), tma=(0, 1), cp=1, par=0)})
_add('dgrad_pointwise_float_mask', 'conv_dgrad', 12, geom=G(2, 3, 6, 6, 64, 160, (1, 1, 1)),
     epi=dict(residual=True, mask_float=True, tf32=True),
     runs={'default': dict(kinds=(0, 0), mask=1, tma=(1, 1), cp=0, lean=1),
           'tma0': dict(kinds=(0, 0), mask=1, tma=(0, 0), cp=1)})
# ---- convolution wgrad (kernels.conv_wgrad): DENSE_MN x CONV_MN / STEM_MN, atomic, split or stream-K.  Both operands
# are MN-major, so every wgrad is staged by the cp.async gather loaders (cp=1, tma=0,0) whatever the switches say.
_add('wgrad_3x3', 'conv_wgrad', 13, geom=G(2, 3, 9, 10, 32, 64, (1, 3, 3), pd=(0, 1, 1)),
     epi=dict(row_scale=True),
     runs={'default': dict(kinds=(1, 4), tma=(0, 0), cp=1),
           'tma0': dict(kinds=(1, 4), tma=(0, 0), cp=1)})
_add('wgrad_temporal_pointwise_taps', 'conv_wgrad', 14, geom=G(2, 4, 8, 8, 64, 64, (3, 1, 1), pd=(1, 0, 0)),
     epi=dict(row_scale=True),
     runs={'default': dict(kinds=(1, 4), tma=(0, 0), cp=1, z=3)})
_add('wgrad_c36', 'conv_wgrad', 15, geom=G(1, 2, 6, 6, 36, 64, (1, 3, 3), pd=(0, 1, 1)),
     epi=dict(),
     runs={'default': dict(kinds=(1, 4), tma=(0, 0), cp=1)})
_add('wgrad_stream_k_atomic', 'conv_wgrad', 16, geom=G(2, 8, 14, 14, 64, 64, (1, 3, 3), pd=(0, 1, 1)),
     epi=dict(), opts=dict(stream_k=1),
     runs={'default': dict(kinds=(1, 4), cp=1, sk=1, fix=0)})
# conv1 wgrad 1x3x3 / stride (1, 2, 2) on a W-padded clip with Wo = 16 and Ho even: N = 32 kH fits one tile; the
# requested 96-wide tile becomes 64 (pow2_only) because the cp.async loader of the MN-major B operand needs a
# power-of-two width
_add('stem_wgrad_1x3x3_t128', 'conv_wgrad', 17, geom=G(1, 2, 32, 32, 4, 64, (1, 3, 3), st=(1, 2, 2), pd=(0, 1, 1)),
     pitched=True, epi=dict(row_scale=True), opts=dict(tile_n=128),
     runs={'default': dict(kinds=(1, 6), tma=(0, 0), patch=0, cp=1, bn=128),
           'nopatch': dict(kinds=(1, 6), tma=(0, 0), patch=0, cp=1, bn=128)})
_add('stem_wgrad_1x3x3_t96', 'conv_wgrad', 18, geom=G(1, 2, 32, 32, 4, 64, (1, 3, 3), st=(1, 2, 2), pd=(0, 1, 1)),
     pitched=True, epi=dict(), opts=dict(tile_n=96),
     runs={'default': dict(kinds=(1, 6), tma=(0, 0), patch=0, cp=1, bn=64)})
_add('stem_wgrad_7x7', 'conv_wgrad', 19, geom=G(1, 4, 36, 64, 4, 64, (5, 7, 7), st=(1, 2, 2), pd=(2, 3, 3)),
     pitched=True, epi=dict(),
     runs={'default': dict(kinds=(1, 6), tma=(0, 0), patch=0, cp=1)})
_add('stem_wgrad_dense_clip', 'conv_wgrad', 20, geom=G(2, 3, 20, 20, 4, 64, (5, 7, 7), st=(1, 2, 2), pd=(2, 3, 3)),
     epi=dict(),
     runs={'default': dict(kinds=(1, 6), tma=(0, 0), cp=1)})
# ---- dense GEMMs through kernels.matmul
# the Charades classifier: 4 x 157 x 2048, B = the transposed view of a contiguous [157, 2048] weight (K-major), split-K
# atomic into an output whose ldd (159) and N are not multiples of 4: the scalar epilogue of run_blocks
_add('fc_157_split_scalar', 'matmul', 21, Z=1, M=4, N=157, K=2048, a_mn=False, b_mn=False, b_weight=True, lib_split=True,
     gn=2, epi=dict(bias=True),
     runs={'default': dict(kinds=(0, 0), tma=(0, 1), cp=1, split='>1', sk=0, lean=0)})      # 4 rows: no 128-row TMA box
_add('mm_stream_k_fix_general', 'matmul', 22, Z=1, M=1000, N=200, K=1024, a_mn=False, b_mn=False, gn=4,
     epi=dict(tf32=True), opts=dict(stream_k=1),
     runs={'default': dict(kinds=(0, 0), tma=(1, 1), cp=0, sk=1, fix=1, lean=0),
           'tma0': dict(kinds=(0, 0), tma=(0, 0), cp=1, sk=0, fix=0)})
# ---- dense GEMMs with every field set directly (vlfb_gemm_params_t)
_add('raw_kk_t32_tails', 'raw', 23, Z=2, M=129, N=100, K=300, a_mn=False, b_mn=False, gn=3, gm=5,
     epi=dict(alpha=0.5, bias=True), opts=dict(tile_n=32),
     runs={'default': dict(kinds=(0, 0), tma=(1, 1), cp=0, bn=32),
           'tma0': dict(kinds=(0, 0), tma=(0, 0), cp=1, bn=32)})
_add('raw_kmn_t96', 'raw', 24, Z=1, M=192, N=160, K=256, a_mn=False, b_mn=True, gn=4, gm=3,
     epi=dict(scale=True, bias=True, relu=True), opts=dict(tile_n=96),
     runs={'default': dict(kinds=(0, 1), tma=(1, 0), cp=1, bn=64)})          # pow2_only: MN-major B by cp.async
_add('raw_mnk_t64_k32', 'raw', 25, Z=3, M=236, N=72, K=32, a_mn=True, b_mn=False, gn=4, gm=2,
     epi=dict(bias=True, residual=True), opts=dict(tile_n=64),
     runs={'default': dict(kinds=(1, 0), tma=(0, 1), cp=1, bn=64)})
_add('raw_mnmn_t128_accum', 'raw', 26, Z=2, M=256, N=200, K=200, a_mn=True, b_mn=True, gn=4, gm=1,
     epi=dict(accum=True), opts=dict(tile_n=128),
     runs={'default': dict(kinds=(1, 1), tma=(0, 0), cp=1, bn=128)})
_add('raw_k16_big_bias', 'raw', 27, Z=1, M=127, N=48, K=16, a_mn=False, b_mn=False, gn=4, gm=1,
     epi=dict(bias=True, bias_scale=64.0),
     runs={'default': dict(kinds=(0, 0), tma=(0, 0), cp=1)})
_add('raw_split3_row_scale', 'raw', 28, Z=1, M=300, N=96, K=1000, a_mn=False, b_mn=False, gn=4, gm=2, split_k=3,
     epi=dict(atomic=True, scale=True, bias=True, row_scale=True),
     runs={'default': dict(kinds=(0, 0), tma=(1, 1), cp=0, split=3, sk=0),
           'tma0': dict(kinds=(0, 0), tma=(0, 0), cp=1, split=3, sk=0)})
_add('raw_accum_residual_tf32', 'raw', 29, Z=1, M=130, N=64, K=96, a_mn=False, b_mn=False, gn=4, gm=2,
     epi=dict(accum=True, residual=True, relu=True, tf32=True),
     runs={'default': dict(kinds=(0, 0), tma=(1, 1), cp=0, lean=0)})
_add('raw_float_mask', 'raw', 30, Z=1, M=200, N=64, K=128, a_mn=False, b_mn=False, gn=4, gm=2,
     epi=dict(mask_float=True, bias=True),
     runs={'default': dict(kinds=(0, 0), mask=1, tma=(1, 1), cp=0),
           'tma0': dict(kinds=(0, 0), mask=1, tma=(0, 0), cp=1)})
_add('raw_stream_k_fix_lean', 'raw', 31, Z=1, M=1000, N=256, K=1024, a_mn=False, b_mn=False, gn=4, gm=2,
     epi=dict(bias=True, relu=True), opts=dict(stream_k=1),
     runs={'default': dict(kinds=(0, 0), tma=(1, 1), cp=0, sk=1, fix=1, lean=1)})
_add('raw_stream_k_fix_accum', 'raw', 32, Z=1, M=1000, N=256, K=1024, a_mn=False, b_mn=False, gn=4, gm=2,
     epi=dict(accum=True), opts=dict(stream_k=1),
     runs={'default': dict(kinds=(0, 0), tma=(1, 1), cp=0, sk=1, fix=1, lean=1)})

_add('raw_stream_k_atomic', 'raw', 33, Z=1, M=1000, N=256, K=1024, a_mn=False, b_mn=False, gn=4, gm=2, split_k=0,
     epi=dict(atomic=True, bias=True), opts=dict(stream_k=1),
     runs={'default': dict(kinds=(0, 0), tma=(1, 1), cp=0, sk=1, fix=0),
           'tma0': dict(kinds=(0, 0), tma=(0, 0), cp=1, sk=1, fix=0)})
# split_k = 0 on a stored (non-atomic) output means one split on both engines (include/vlfb.h); it was rejected, and the
# SIMT engine would have split K = 4096 four ways, each split overwriting the others' partial sums
_add('raw_split0_stored_residual_tf32', 'raw', 34, Z=1, M=200, N=96, K=4096, a_mn=False, b_mn=False, gn=4, gm=2,
     split_k=0, epi=dict(residual=True, tf32=True),
     runs={'default': dict(kinds=(0, 0), split=1, sk=0)})
_add('raw_split0_stored_residual_tf32_simt', 'raw', 34, Z=1, M=200, N=96, K=4096, a_mn=False, b_mn=False, gn=4, gm=2,
     split_k=0, engine='simt', epi=dict(residual=True, tf32=True),
     runs={'default': {}})


# ---- weight gradients at every production geometry of R50-I3D-NL at 2 clips (tests/wgrad_cases.py) and at small ragged
# ones: K (positions) not a multiple of 64, Co = 4, 32, 64 and 68, N tails, stream-K / split-K of each operand form.
# These launches stage both operands by cp.async and publish each chunk by the completion of its copies
# (cp.async.mbarrier.arrive), so the producers run ahead of the MMAs by the whole ring.  A case with Co <= 64 runs
# 64 x 2bn wide tiles, warpgroup w computing columns [w bn, (w + 1) bn) of the 64 rows (csrc/gemm_tc.cu, Launch::wide).
def _wgrad(name, seed, shape, co, ker, st=(1, 1, 1), pd=(0, 0, 0), dil=(1, 1, 1), opts=None, epi=None, long_k=False,
           col_mask=False, **expect):
    """A conv_wgrad case run under the default configuration only (check_case compares the record's kinds with
    describe() for every case).  long_k: K = N To Ho Wo may exceed KMAX.  col_mask: conv1 with the optimiser's 32-lane
    column mask."""
    n, t, h, w, c = shape
    run = dict(tma=(0, 0), cp=1)
    if c == 4:
        run['patch'] = 0
    run.update(expect)
    _add(name, 'conv_wgrad', seed, {'default': run}, opts=opts or {}, epi=epi or {}, long_k=long_k, col_mask=col_mask,
         geom=G(n, t, h, w, c, co, tuple(ker), st=tuple(st), pd=tuple(pd), dil=tuple(dil)))


_RS = dict(row_scale=True)
for _i, (_label, _shape, _co, _ker, _st, _pd, _dil, _) in enumerate(WC.PRODUCTION):
    _wgrad('wgrad prod ' + _label, 500 + _i, _shape, _co, _ker, _st, _pd, _dil, long_k=True)
_wgrad('wgrad ragged M=4 3x3', 601, (1, 2, 6, 6, 32), 4, (1, 3, 3), pd=(0, 1, 1))
_wgrad('wgrad ragged M=32 3x3 N tail', 602, (2, 3, 5, 7, 64), 32, (1, 3, 3), pd=(0, 1, 1))
_wgrad('wgrad ragged M=64 3x1x1', 603, (1, 3, 10, 10, 32), 64, (3, 1, 1), pd=(1, 0, 0))
_wgrad('wgrad ragged M=68 1x1', 604, (2, 2, 9, 9, 64), 68, (1, 1, 1))
_wgrad('wgrad ragged M=68 3x3 N tail', 605, (1, 3, 7, 9, 32), 68, (1, 3, 3), pd=(0, 1, 1))
_wgrad('wgrad ragged stem 5x7x7', 606, (1, 3, 20, 20, 4), 64, (5, 7, 7), st=(1, 2, 2), pd=(2, 3, 3))
# stream-K (atomic, no fix-up) of each operand form
_wgrad('wgrad stream-K 3x3', 611, (2, 8, 14, 14, 128), 128, (1, 3, 3), pd=(0, 1, 1), opts=dict(stream_k=1), sk=1, fix=0)
_wgrad('wgrad stream-K 1x1', 612, (2, 16, 14, 14, 256), 128, (1, 1, 1), opts=dict(stream_k=1), sk=1, fix=0)
_wgrad('wgrad stream-K stem', 613, (1, 4, 36, 64, 4), 64, (5, 7, 7), st=(1, 2, 2), pd=(2, 3, 3), opts=dict(stream_k=1),
       sk=1, fix=0)
# wide tiles: every Co = 64 production geometry, and one Co = 128 that stays narrow
for _i, (_label, _shape, _co, _ker, _st, _pd, _dil, _) in enumerate(WC.PRODUCTION):
    if _co <= 64 or _label == 'res3_x_2b 1x3x3 128->128':
        _wgrad('wide prod ' + _label, 700 + _i, _shape, _co, _ker, _st, _pd, _dil, long_k=True, wide=int(_co <= 64))
# M against the 64-row wide tile (Co % 4 == 0: 16-byte dY rows)
_wgrad('wide M=4 3x3', 801, (1, 2, 6, 6, 32), 4, (1, 3, 3), pd=(0, 1, 1), epi=_RS, wide=1)
_wgrad('wide M=32 3x3', 802, (2, 3, 5, 7, 64), 32, (1, 3, 3), pd=(0, 1, 1), wide=1)
_wgrad('wide M=60 3x1x1 N=32', 803, (1, 3, 8, 8, 32), 60, (3, 1, 1), pd=(1, 0, 0), epi=_RS, wide=1)
_wgrad('wide M=64 1x1', 804, (2, 2, 9, 9, 64), 64, (1, 1, 1), wide=1)
_wgrad('wide M=68 3x3', 805, (1, 3, 7, 9, 32), 68, (1, 3, 3), pd=(0, 1, 1), wide=0)
# N tails against bn and 2 bn, with the tile width forced
_wgrad('wide N=96 <= bn=128 1x1', 811, (2, 2, 8, 8, 96), 64, (1, 1, 1), opts=dict(tile_n=128), epi=_RS, wide=1, bn=128)
_wgrad('wide bn=64 < N=108 < 128 3x3', 812, (1, 3, 6, 6, 12), 48, (1, 3, 3), pd=(0, 1, 1), opts=dict(tile_n=64), wide=1,
       bn=64)
_wgrad('wide N=144 = 2 x 64 + 16, bn=32 1x1', 813, (1, 4, 6, 6, 144), 64, (1, 1, 1), opts=dict(tile_n=32), epi=_RS,
       wide=1, bn=32)
_wgrad('wide N=144 = 128 + 16, bn=64 3x3', 814, (1, 3, 6, 6, 16), 64, (1, 3, 3), pd=(0, 1, 1), opts=dict(tile_n=64),
       wide=1, bn=64)
_wgrad('wide N=224 bn=128 stem', 815, (1, 3, 20, 20, 4), 64, (5, 7, 7), st=(1, 2, 2), pd=(2, 3, 3),
       opts=dict(tile_n=128), wide=1, bn=128)
# split-K (few wide tiles, long K) and stream-K (atomic, no fix-up) for each B operand kind
_wgrad('wide split-K CONV_MN', 821, (2, 8, 14, 14, 64), 64, (1, 3, 3), pd=(0, 1, 1), epi=_RS, wide=1, split='>1', sk=0)
_wgrad('wide split-K STEM_MN', 822, (1, 4, 36, 64, 4), 64, (5, 7, 7), st=(1, 2, 2), pd=(2, 3, 3), wide=1, split='>1',
       sk=0)
_wgrad('wide split-K DENSE_MN', 823, (2, 8, 14, 14, 64), 64, (1, 1, 1), wide=1, split='>1', sk=0)
_wgrad('wide stream-K CONV_MN', 831, (2, 8, 14, 14, 64), 64, (1, 3, 3), pd=(0, 1, 1), opts=dict(stream_k=1), wide=1,
       sk=1, fix=0)
_wgrad('wide stream-K STEM_MN', 832, (1, 4, 36, 64, 4), 64, (5, 7, 7), st=(1, 2, 2), pd=(2, 3, 3),
       opts=dict(stream_k=1), epi=_RS, wide=1, sk=1, fix=0)
_wgrad('wide stream-K DENSE_MN', 833, (2, 16, 28, 28, 64), 64, (1, 1, 1), opts=dict(stream_k=1), long_k=True, wide=1,
       sk=1, fix=0)
# conv1 with the optimiser's column mask (padding lanes px >= kW and the fourth channel zeroed) and a row scale
_wgrad('wide stem col_mask', 841, (1, 4, 36, 64, 4), 64, (5, 7, 7), st=(1, 2, 2), pd=(2, 3, 3), epi=_RS, col_mask=True,
       wide=1)
# transposed x transposed matmul, M <= 64, plain stores with ACCUM (read-modify-write of D by exactly one warp: no
# reduction across warpgroups)
_add('wide raw MNxMN M=48 accum', 'raw', 851, Z=2, M=48, N=200, K=300, a_mn=True, b_mn=True, gn=4, gm=2,
     epi=dict(accum=True, scale=True, bias=True, row_scale=True),
     runs={'default': dict(kinds=(OP_DENSE_MN, OP_DENSE_MN), tma=(0, 0), cp=1, wide=1, sk=0, split=1)})


def case_by_name(name):
    return next(c for c in CASES if c['name'] == name)


# ----------------------------------------------------------------------------------------------- GEMM view of a case
def out_dims(g):
    To = (g['T'] + 2 * g['pd'][0] - g['dil'][0] * (g['ker'][0] - 1) - 1) // g['st'][0] + 1
    Ho = (g['H'] + 2 * g['pd'][1] - g['dil'][1] * (g['ker'][1] - 1) - 1) // g['st'][1] + 1
    Wo = (g['W'] + 2 * g['pd'][2] - g['dil'][2] * (g['ker'][2] - 1) - 1) // g['st'][2] + 1
    return To, Ho, Wo


def _pointwise(g):
    return tuple(g['ker']) == (1, 1, 1) and tuple(g['st']) == (1, 1, 1) and tuple(g['pd']) == (0, 0, 0)


def describe(c):
    """The vlfb_gemm call a case makes, as (kinds, M, N, K, batch, taps, flags): what kernels.py builds for the conv /
    matmul wrappers and what _run_raw sets.  The GPU worker checks the launch's record against it."""
    e = c.get('epi', {})
    if c['op'] in ('matmul', 'raw'):
        # lib_split: kernels.matmul itself picks split-K with atomic accumulation (few tiles, long K) and zero-fills d
        flags = dict(accum=bool(e.get('accum')), atomic=bool(e.get('atomic') or c.get('lib_split')),
                     residual=bool(e.get('residual')), relu=bool(e.get('relu')), tf32=bool(e.get('tf32')),
                     mask=bool(e.get('mask_float') or e.get('mask_bits')),
                     split_k=0 if c.get('lib_split') else c.get('split_k', 1))
        return dict(kinds=(OP_DENSE_MN if c['a_mn'] else OP_DENSE_K, OP_DENSE_MN if c['b_mn'] else OP_DENSE_K),
                    M=c['M'], N=c['N'], K=c['K'], batch=c['Z'], taps=1, flags=flags)
    g = c['geom']
    To, Ho, Wo = out_dims(g)
    kT, kH, kW = g['ker']
    stem = g['C'] == 4
    flags = dict(accum=bool(e.get('accum')), atomic=c['op'] == 'conv_wgrad', residual=bool(e.get('residual')),
                 relu=bool(e.get('relu')), tf32=bool(e.get('tf32')),
                 mask=bool(e.get('mask_float') or e.get('mask_bits')), split_k=0 if c['op'] == 'conv_wgrad' else 1)
    if c['op'] == 'conv_fwd':
        ak = OP_STEM_K if stem else (OP_DENSE_K if _pointwise(g) else OP_CONV_K)
        K = kT * kH * 32 if stem else kT * kH * kW * g['C']
        return dict(kinds=(ak, OP_DENSE_K), M=g['N'] * To * Ho * Wo, N=g['Co'], K=K, batch=1, taps=1, flags=flags)
    if c['op'] == 'conv_dgrad':
        ak = OP_DENSE_K if _pointwise(g) else OP_DGRAD_K
        return dict(kinds=(ak, OP_DENSE_K), M=g['N'] * g['T'] * g['H'] * g['W'], N=g['C'], K=kT * kH * kW * g['Co'],
                    batch=1, taps=1, flags=flags)
    bk = OP_STEM_MN if stem else (OP_DENSE_MN if _pointwise(g) else OP_CONV_MN)
    n = kH * 32 if stem else (g['C'] if _pointwise(g) else kH * kW * g['C'])
    return dict(kinds=(OP_DENSE_MN, bk), M=g['Co'], N=n, K=g['N'] * To * Ho * Wo, batch=1,
                taps=1 if _pointwise(g) else kT, flags=flags)


# ----------------------------------------------------------------------------------------------- the C ABI's rules
def effective_split_k(c):
    """split_k as vlfb_gemm resolves it before validation: 0 means 1 unless the epilogue is atomic."""
    f = describe(c)['flags']
    return 1 if f['split_k'] == 0 and not f['atomic'] else f['split_k']


def abi_errors(c):
    """The rules of include/vlfb.h (as validate_gemm in csrc/api.cu applies them, and the tensor-core engine's own
    rejections) for the call the case makes: [] when vlfb_gemm accepts it."""
    d = describe(c)
    f = d['flags']
    ak, bk = d['kinds']
    M, N, K = d['M'], d['N'], d['K']
    e = c.get('epi', {})
    sk = effective_split_k(c)
    det = bool(c.get('deterministic'))
    err = []
    if not (M > 0 and N > 0 and K > 0):
        err.append('M, N, K must be > 0')
    if sk < 0 or (sk != 1 and not f['atomic']):
        err.append('split_k != 1 needs VLFB_EPI_ATOMIC')
    if det and sk > 1:
        err.append('a deterministic call is never split')
    if (sk > 1 if det else sk != 1) and (f['residual'] or f['mask'] or f['relu'] or f['tf32']):
        err.append('split-K with a non-linear epilogue')
    if det and f['atomic'] and not c.get('workspace', True):
        err.append('a deterministic atomic call needs the workspace')
    ldd = c.get('ldd', N + c.get('gn', 0)) if c['op'] in ('raw', 'matmul') else N
    if e.get('bits') and not (f['relu'] and not f['atomic'] and sk == 1 and d['batch'] == 1 and d['taps'] == 1 and
                              ldd == N and N % 32 == 0):
        err.append('relu_bits_out needs RELU, no atomic, one batch, ldd == N, N % 32 == 0')
    if e.get('mask_float') and e.get('mask_bits'):
        err.append('relu_mask and relu_mask_bits together')
    if f['mask'] and engine(c) == 'tc' and (ak, bk) not in ((OP_DGRAD_K, OP_DENSE_K), (OP_DENSE_K, OP_DENSE_K)):
        err.append('relu_mask on the tensor-core engine needs DGRAD_K / DENSE_K x DENSE_K')
    tile_n = c.get('opts', {}).get('tile_n', 0)
    if not (tile_n == 0 or (32 <= tile_n <= 256 and tile_n % 32 == 0)):
        err.append('tile_n')
    g = c.get('geom')
    if g is not None:
        kT, kH, kW = g['ker']
        if ak == OP_CONV_K and not (g['C'] % 32 == 0 and K == kT * kH * kW * g['C']):
            err.append('CONV_K needs C % 32 == 0')
        if ak == OP_DGRAD_K and not (g['Co'] % 32 == 0 and K == kT * kH * kW * g['Co']):
            err.append('DGRAD_K needs Co % 32 == 0')
        if bk == OP_CONV_MN and not (N == kH * kW * g['C'] and g['C'] % 4 == 0 and d['taps'] == kT and kH <= 8 and kW <= 8):
            err.append('CONV_MN extents')
        if OP_STEM_K in (ak, bk) or OP_STEM_MN in (ak, bk):
            if not (g['C'] == 4 and kW <= 8 and tuple(g['dil']) == (1, 1, 1)):
                err.append('stem geometry')
            if bk == OP_STEM_MN and not (N == 32 * kH and kH <= 8 and d['taps'] == kT):
                err.append('STEM_MN extents')
            if ak == OP_STEM_K and K != kT * kH * 32:
                err.append('STEM_K extents')
        To, Ho, Wo = out_dims(g)
        if min(To, Ho, Wo) < 1:
            err.append('empty output')
    return err


def engine(c):
    """'tc' or 'simt': the engine vlfb_gemm runs the case's call on -- SIMT when the case asks for it, or when an
    operand is not 16-byte addressable for the tensor-core loaders (validate_gemm's tc_ok)."""
    if c.get('engine') == 'simt':
        return 'simt'
    d = describe(c)
    if c['op'] == 'raw':
        ops = [(w, d['kinds'][i], c['M'] if w == 'a' else c['N']) + operand_layout(c, w) for i, w in enumerate('ab')]
    elif c['op'] == 'matmul':
        return 'tc'
    else:
        g = c['geom']
        rows_a = {'conv_fwd': d['M'], 'conv_dgrad': d['M'], 'conv_wgrad': g['Co']}[c['op']]
        ld_a = {'conv_fwd': g['C'], 'conv_dgrad': g['Co'], 'conv_wgrad': g['Co']}[c['op']]
        ld_b = d['K'] if d['kinds'][1] == OP_DENSE_K else g['C']
        ops = [('a', d['kinds'][0], rows_a, ld_a, 0, 0), ('b', d['kinds'][1], d['N'], ld_b, 0, 0)]
    for _, kind, extent, ld, bs, off in ops:
        if off % 4:
            return 'simt'
        if kind == OP_DENSE_K and (ld % 4 or bs % 4 or d['K'] % 4):
            return 'simt'
        if kind == OP_DENSE_MN and (ld % 4 or bs % 4 or extent % 4):
            return 'simt'
    return 'tc'


# ----------------------------------------------------------------------------------------------- comparison
def finish(acc, mag, epi, K):
    """fp64 epilogue of vlfb_gemm (common.cuh epilogue_store, element by element) and the error bound of each element.
    acc / mag: [Z, M, N] sum_k A B and sum_k |A| |B| over the call's K; epi: alpha, cs [N], cb [N], rs [M],
    res / prev / keep [Z, M, N], relu, tf32, atomic.  prev is the d the call adds to: an ACCUM epilogue reads it before
    the ReLU, the mask and the rounding; an atomic one (atomic=True) adds its finished value to it.  Returns (ref,
    bound)."""
    Z, M, N = acc.shape
    one = torch.ones((), dtype=torch.float64, device=acc.device)
    cs = epi.get('cs', one).view(1, 1, -1) if epi.get('cs') is not None else one
    cb = epi.get('cb').view(1, 1, -1) if epi.get('cb') is not None else 0 * one
    rs = epi.get('rs').view(1, -1, 1) if epi.get('rs') is not None else one
    s = epi.get('alpha', 1.0) * cs * rs
    v = acc * s + cb * rs
    extra = (cb * rs).abs()
    after = epi.get('prev') if epi.get('atomic') else None
    for k in ('res', 'prev'):
        if epi.get(k) is not None and not (k == 'prev' and after is not None):
            v = v + epi[k]
            extra = extra + epi[k].abs()
    if epi.get('relu'):
        v = v.clamp(min=0)
    if epi.get('keep') is not None:
        v = torch.where(epi['keep'], v, torch.zeros_like(v))
    bound = tau(K) * s.abs() * mag + EPS32 * (s.abs() * mag + extra)
    if epi.get('tf32'):
        bound = bound + ulp_tf32(v)
    if after is not None:
        v = v + after
        bound = bound + EPS32 * after.abs()
    return v, bound.expand_as(v)


# ----------------------------------------------------------------------------------------------- case inputs / references
def rnd(shape, gen, scale=1.0):
    return tf32_round(torch.randn(shape, generator=gen) * scale)


def _to_cl(x):
    return x.permute(0, 2, 3, 4, 1).contiguous()


def _stem_ext_input(x, g, To, Ho, Wo):
    """conv1 as the library defines it: every K row spans 8 pixels x 4 channels, so the reference is a (kT, kH, 8)
    convolution over the zero-padded clip, trimmed to the extents the To x Ho x Wo outputs read."""
    kT, kH, _ = g['ker']
    (sT, sH, sW), (pT, pH, pW) = g['st'], g['pd']
    nt, nh, nw = (To - 1) * sT + kT, (Ho - 1) * sH + kH, (Wo - 1) * sW + 8
    xp = F.pad(x, (pW, max(0, nw - pW - g['W']), pH, max(0, nh - pH - g['H']), pT, max(0, nt - pT - g['T'])))
    return xp[:, :, :nt, :nh, :nw]


def conv_refs(c, x, w, dy, dev):
    """fp64 (acc, mag) of the case's convolution GEMM in its output layout [Z, M, N] (independent of libvlfb): x NCTHW,
    w [Co, C, kT, kH, kW] (stem: [Co, 4, kT, kH, 8]), dy [N, Co, To, Ho, Wo]."""
    g = c['geom']
    To, Ho, Wo = out_dims(g)
    stem = g['C'] == 4
    x, w, dy = x.to(dev).double(), w.to(dev).double(), dy.to(dev).double()
    res = []
    for sgn in (False, True):
        xs, ws, dys = (x.abs(), w.abs(), dy.abs()) if sgn else (x, w, dy)
        if stem:                                                     # (no conv1 dgrad: the clip needs no gradient)
            xi = _stem_ext_input(xs, g, To, Ho, Wo)
            wi = ws.clone().requires_grad_(True)
            y = F.conv3d(xi, wi, None, g['st'])
        else:
            xi = xs.clone().requires_grad_(True)
            wi = ws.clone().requires_grad_(True)
            y = F.conv3d(xi, wi, None, g['st'], g['pd'], g['dil'])
        if c['op'] == 'conv_fwd':
            r = y.detach().permute(0, 2, 3, 4, 1).reshape(1, -1, g['Co'])
        elif c['op'] == 'conv_dgrad':
            y.backward(dys)
            r = xi.grad.permute(0, 2, 3, 4, 1).reshape(1, -1, g['C'])
        else:
            y.backward(dys)
            kT = g['ker'][0]
            r = wi.grad.permute(2, 0, 3, 4, 1)                       # [kT, Co, kH, kW(8), C]
            r = r.reshape(kT, g['Co'], -1)
        res.append(r.detach())
    return res[0], res[1]


def _col_mask(kH):
    """conv1's column mask over the kH x 32 lanes of a wgrad row: lane px * 4 + ch is real when px < kW (7) and
    ch < 3.  conv_wgrad takes the first 32 lanes and repeats them."""
    m = torch.zeros(32)
    for px in range(7):
        m[px * 4:px * 4 + 3] = 1
    return m.repeat(kH)


class Prepared:
    """Inputs, output buffers, the call and the fp64 reference of one case."""


def prepare(c, dev):
    """Build the case on `dev` (the kernel call needs CUDA; the reference and bound work on any device)."""
    gen = torch.Generator().manual_seed(1000 + c['seed'])
    P = Prepared()
    P.case = c
    e = c.get('epi', {})
    if c['op'] in ('matmul', 'raw'):
        Z, M, N, K = c['Z'], c['M'], c['N'], c['K']
        A = rnd((Z, M, K), gen)
        B = rnd((Z, N, K), gen)
        for X, w in ((A, 'a'), (B, 'b')):
            if Z > 1 and c.get(w + '_shared'):                      # batch_stride 0: every batch reads batch 0
                X[1:] = X[:1]
        P.A, P.B = A, B
        Ad, Bd = A.to(dev).double(), B.to(dev).double()
        acc = torch.bmm(Ad, Bd.transpose(1, 2))
        mag = torch.bmm(Ad.abs(), Bd.abs().transpose(1, 2))
        gm, gn = c.get('gm', 0), c.get('gn', 0)
        ldd = c.get('ldd', N + gn)
        dbs = (M + gm) * ldd + (c.get('d_gap', 8) if Z > 1 else 0)      # a gap between batches
        d0 = GUARD + c.get('d_off', 0)                                  # d (and residual, mask) at float d0 of the buffer
        size = d0 + Z * dbs + gm * ldd + 64
        zz, mm, nn = torch.meshgrid(torch.arange(Z), torch.arange(M), torch.arange(N), indexing='ij')
        P.index = d0 + zz * dbs + mm * ldd + nn
        P.layout = dict(ldd=ldd, dbs=dbs if Z > 1 else 0, size=size, d0=d0)
    else:
        g = c['geom']
        To, Ho, Wo = out_dims(g)
        kT, kH, kW = g['ker']
        stem = g['C'] == 4
        Ci = 3 if stem else g['C']
        x = rnd((g['N'], Ci, g['T'], g['H'], g['W']), gen)
        if stem:
            x = torch.cat([x, torch.zeros_like(x[:, :1])], 1)           # the fourth (pad) channel is zero
            w = torch.zeros((g['Co'], 4, kT, kH, 8))
            w[:, :3, :, :, :kW] = rnd((g['Co'], 3, kT, kH, kW), gen, 0.1)
        else:
            w = rnd((g['Co'], g['C'], kT, kH, kW), gen, 0.1)
        dy = rnd((g['N'], g['Co'], To, Ho, Wo), gen)
        P.x, P.w, P.dy = x, w, dy
        acc, mag = conv_refs(c, x, w, dy, dev)
        Z, M, N = acc.shape
        P.layout = dict(size=GUARD + Z * M * N + 96)
        P.index = GUARD + torch.arange(Z * M * N).view(Z, M, N)
        if c['op'] == 'conv_wgrad':                                     # dw [Co][kT][n]: tap z at column z * n
            zz, mm, nn = torch.meshgrid(torch.arange(Z), torch.arange(M), torch.arange(N), indexing='ij')
            P.index = GUARD + mm * (Z * N) + zz * N + nn
    Z, M, N = acc.shape
    epi = dict(alpha=e.get('alpha', 1.0), relu=e.get('relu', False), tf32=e.get('tf32', False))
    if e.get('scale'):
        epi['cs'] = (torch.rand(N, generator=gen) + 0.5).double()
    if c.get('col_mask'):
        epi['cs'] = _col_mask(c['geom']['ker'][1]).double()
    if e.get('bias'):
        epi['cb'] = (torch.randn(N, generator=gen) * e.get('bias_scale', 1.0)).double()
    if e.get('row_scale'):
        epi['rs'] = (torch.rand(M, generator=gen) + 0.5).double()
    if e.get('residual'):
        epi['res'] = torch.randn((Z, M, N), generator=gen).double()
    if e.get('accum') or e.get('atomic') or c['op'] == 'conv_wgrad':
        # calls that add to d (ACCUM, atomic split / stream-K, the wgrad): d starts at prev; every other output starts
        # as the NaN fill, so an element the kernel never writes stays NaN
        epi['prev'] = torch.randn((Z, M, N), generator=gen).double()
        epi['atomic'] = not e.get('accum')
    if e.get('mask_float') or e.get('mask_bits'):
        epi['maskv'] = torch.randn((Z, M, N), generator=gen)
        epi['keep'] = epi['maskv'] > 0
    P.epi = dict((k, (v.to(dev) if torch.is_tensor(v) else v)) for k, v in epi.items())
    P.acc, P.mag = acc.to(dev), mag.to(dev)
    P.K = describe(c)['K']
    P.ref, P.bound = finish(P.acc, P.mag, P.epi, P.K)
    P.index = P.index.to(dev)
    return P


# ----------------------------------------------------------------------------------------------- running a case (GPU)
def _opts(K, c):
    K.GEMM_OPTS.update(dict(tile_n=0, pair=0, stream_k=0))
    K.GEMM_OPTS.update(c.get('opts', {}))


def _stem_input(K, P, dev):
    """[N,T,H,W,4] conv1 operand: dense, or a view of a W-padded zero buffer (the TMA stem path)."""
    c = P.case
    g = c['geom']
    x_cl = _to_cl(P.x).to(dev)
    if not c.get('pitched'):
        return x_cl
    pW = g['pd'][2]
    To, Ho, Wo = out_dims(g)
    pitch = max(pW + g['W'], (Wo - 1) * g['st'][2] + 8)
    pitch = (pitch + 3) // 4 * 4
    buf = torch.zeros((g['N'], g['T'], g['H'], pitch, 4), device=dev)
    buf[:, :, :, pW:pW + g['W'], :] = x_cl
    return buf[:, :, :, pW:pW + g['W'], :]


def run_case(K, P, dev):
    """Runs the case's one vlfb_gemm call; returns (buffer, bits or None, bits guard info)."""
    from vlfb import libvlfb as L
    import ctypes
    c = P.case
    e = c.get('epi', {})
    Z, M, N = P.ref.shape
    buf = nan_buffer(P.layout['size'], dev)
    flat = buf.view(-1)
    if 'prev' in P.epi:
        flat[P.index.reshape(-1)] = P.epi['prev'].reshape(-1).float()
    cs = P.epi['cs'].float() if 'cs' in P.epi else None
    cb = P.epi['cb'].float() if 'cb' in P.epi else None
    rs = P.epi['rs'].float() if 'rs' in P.epi else None
    bits = None
    _opts(K, c)
    K.set_gemm_backend('simt' if c.get('engine') == 'simt' else 'tcgen05')
    try:
        if c['op'] in ('conv_fwd', 'conv_dgrad', 'conv_wgrad'):
            g = c['geom']
            geo = K.conv_geom((g['N'], g['T'], g['H'], g['W'], g['C']), g['Co'], g['ker'], g['st'], g['pd'], g['dil'])
            n_out = Z * M * N
            out = flat[GUARD:GUARD + n_out]
            res = None
            if 'res' in P.epi:
                rbuf = torch.zeros_like(flat)
                rbuf[P.index.reshape(-1)] = P.epi['res'].reshape(-1).float()
                res = rbuf[GUARD:GUARD + n_out]
            if c['op'] == 'conv_fwd':
                x = _stem_input(K, P, dev) if g['C'] == 4 else _to_cl(P.x).to(dev)
                w = P.w.permute(0, 2, 3, 4, 1).contiguous().to(dev)      # [Co, kT, kH, kW(8), C]
                y = out.view(K.out_shape(geo))
                if e.get('bits'):
                    bits = torch.full((n_out // 32 + 8,), 0x5A5A5A5A, dtype=torch.int32, device=dev)
                K.conv_fwd(x, w, y, geo, scale=cs, bias=cb, residual=None if res is None else res.view(y.shape),
                           relu=bool(e.get('relu')), tf32_out=bool(e.get('tf32')),
                           relu_bits=None if bits is None else bits[:n_out // 32])
            elif c['op'] == 'conv_dgrad':
                taps = g['ker'][0] * g['ker'][1] * g['ker'][2]
                w_cl = P.w.permute(0, 2, 3, 4, 1).contiguous().to(dev)
                wt = torch.empty((g['C'], taps, g['Co']), device=dev)
                K.weight_transpose(w_cl, wt)
                dx = out.view(g['N'], g['T'], g['H'], g['W'], g['C'])
                mask = mbits = None
                if 'maskv' in P.epi:
                    mv = P.epi['maskv'].reshape(dx.shape).float().contiguous()
                    if e.get('mask_bits'):
                        mbits = pack_sign_bits(mv)
                    else:
                        mask = mv
                K.conv_dgrad(_to_cl(P.dy).to(dev), wt, dx, geo, accumulate=bool(e.get('accum')),
                             residual=None if res is None else res.view(dx.shape), relu_mask=mask,
                             tf32_out=bool(e.get('tf32')), relu_mask_bits=mbits)
            else:
                x = _stem_input(K, P, dev) if g['C'] == 4 else _to_cl(P.x).to(dev)
                dw = out.view((g['Co'],) + tuple(g['ker'][:2]) + (8 if g['C'] == 4 else g['ker'][2], g['C']))
                wgrad = K.conv_wgrad_det if c.get('deterministic') else K.conv_wgrad
                mask = P.epi['cs'][:32].float() if c.get('col_mask') else None
                wgrad(_to_cl(P.dy).to(dev), x, dw, geo, row_scale=rs, col_mask=mask)
        elif c['op'] == 'matmul':
            A = P.A.to(dev)
            if c.get('b_weight'):
                Bm = P.B[0].contiguous().to(dev).t().unsqueeze(0)              # [1, K, N] view of a [N, K] weight
            else:
                Bm = P.B.to(dev).transpose(1, 2)
            ldd, dbs = P.layout['ldd'], P.layout['dbs']
            d = torch.as_strided(flat, (Z, M, N), (dbs if Z > 1 else M * ldd, ldd, 1), GUARD)
            K.matmul(A, Bm, d, bias=cb, tf32_out=bool(e.get('tf32')))
        else:
            bits = _run_raw(K, L, ctypes, P, flat, cs, cb, rs, dev)
        torch.cuda.synchronize()
    finally:
        _opts(K, {'opts': {}})
        K.set_gemm_backend('tcgen05')
    return buf, bits


def operand_layout(c, w):
    """(ld, batch_stride, offset in floats from a 16-byte aligned base) of raw operand w ('a' or 'b').  Optional case
    fields: w_pad (floats after each row), w_gap (floats between batches), w_shared (batch_stride 0), w_off.  Without
    them: packed rows (ld = K, or the extent when MN-major) and packed batches."""
    Z, K = c['Z'], c['K']
    rows = c['M'] if w == 'a' else c['N']
    ld = (rows if c[w + '_mn'] else K) + c.get(w + '_pad', 0)
    span = (K if c[w + '_mn'] else rows) * ld
    bs = 0 if Z == 1 or c.get(w + '_shared') else span + c.get(w + '_gap', 0)
    return ld, bs, c.get(w + '_off', 0)


def _run_raw(K, L, ctypes, P, flat, cs, cb, rs, dev):
    """The case's vlfb_gemm call with every field set directly; returns the sign-bit buffer (or None)."""
    c = P.case
    e = c.get('epi', {})
    Z, M, N, Kd = c['Z'], c['M'], c['N'], c['K']
    keep = []

    def operand(X, w, rows):                                   # X logical [Z, rows, K]
        o = L.Operand()
        mn = c[w + '_mn']
        ld, bs, off = operand_layout(c, w)
        o.kind, o.ld, o.batch_stride = (L.OP_DENSE_MN if mn else L.OP_DENSE_K), ld, bs
        s = X.transpose(1, 2) if mn else X                     # MN-major: [Z, K, rows], rows contiguous
        zs = 1 if bs == 0 else Z
        # padding and gaps hold NaN: an element read outside the described matrix poisons the result
        st = torch.full((off + (zs - 1) * bs + s.shape[1] * ld + 16,), float('nan'), device=dev)
        torch.as_strided(st, (zs, s.shape[1], s.shape[2]), (bs, ld, 1), off).copy_(s[:zs])
        o.ptr = st.data_ptr() + off * 4
        keep.append(st)
        return o

    p = L.GemmParams()
    p.a = operand(P.A, 'a', M)
    p.b = operand(P.B, 'b', N)
    p.M, p.N, p.K, p.batch, p.taps = M, N, Kd, Z, 1
    p.split_k = c.get('split_k', 1)
    d0 = P.layout['d0']
    p.d = flat.data_ptr() + d0 * 4
    p.ldd, p.d_batch_stride, p.d_tap_stride = P.layout['ldd'], P.layout['dbs'], 0
    p.alpha = float(e.get('alpha', 1.0))
    for name, t in (('col_scale', cs), ('col_bias', cb), ('row_scale', rs)):
        if t is not None:
            t = t.contiguous().to(dev)
            keep.append(t)
            setattr(p, name, t.data_ptr())
    if 'res' in P.epi:
        rbuf = torch.zeros_like(flat)
        rbuf[P.index.reshape(-1)] = P.epi['res'].reshape(-1).float()
        keep.append(rbuf)
        p.residual = rbuf.data_ptr() + d0 * 4
    if 'maskv' in P.epi:
        mbuf = torch.zeros_like(flat)
        mbuf[P.index.reshape(-1)] = P.epi['maskv'].reshape(-1).float()
        if e.get('mask_bits'):                                 # bit (off & 31) of word off >> 5, off counted from d
            region = mbuf[d0:]
            region = torch.cat([region, region.new_zeros(-region.numel() % 32)])
            mbits = pack_sign_bits(region)
            keep.append(mbits)
            p.relu_mask_bits = mbits.data_ptr()
        else:
            keep.append(mbuf)
            p.relu_mask = mbuf.data_ptr() + d0 * 4
    bits = None
    if e.get('bits'):
        bits = torch.full((M * N // 32 + 8,), 0x5A5A5A5A, dtype=torch.int32, device=dev)
        p.relu_bits_out = bits.data_ptr()
    p.flags = ((L.EPI_RELU if e.get('relu') else 0) | (L.EPI_ACCUM if e.get('accum') else 0) |
               (L.EPI_ATOMIC if e.get('atomic') else 0) | (L.EPI_TF32 if e.get('tf32') else 0))
    if c.get('workspace', True):
        ws = K.gemm_workspace(flat.device)
        p.workspace, p.workspace_bytes = ws.data_ptr(), ws.numel() * 4
    p.deterministic = int(c.get('deterministic', 0))
    p.engine = L.ENGINE_SIMT if c.get('engine') == 'simt' else L.ENGINE_TCGEN05
    p.tile_n, p.pair, p.stream_k = K.GEMM_OPTS['tile_n'], K.GEMM_OPTS['pair'], K.GEMM_OPTS['stream_k']
    L.check(L.load().vlfb_gemm(ctypes.byref(p), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), 'vlfb_gemm')
    torch.cuda.synchronize()
    return bits


def check_case(K, c, config, dev, declared=True):
    """Runs one case under the current process's configuration; returns its JSON record.  The launch must take the
    engine abi_errors / engine() predict (one gemm_tc record, or none on the SIMT engine) and, with `declared`, the
    path the case declares for `config`.  A deterministic case runs twice and must give the same bits."""
    rec = dict(case=c['name'], config=config, errors=[], engine=engine(c))
    P = prepare(c, dev)
    (buf, bits), text = capture_fd2(lambda: run_case(K, P, dev))
    paths = [r for r in (parse_record(l) for l in text.splitlines()) if r is not None]
    rec['paths'] = [dict((k, list(v) if isinstance(v, tuple) else v) for k, v in r.items()) for r in paths]
    rec['flags'] = describe(c)['flags']
    if rec['engine'] == 'simt':
        if paths:
            rec['errors'].append('expected the SIMT engine, got %d tensor-core launch records' % len(paths))
    elif len(paths) != 1:
        rec['errors'].append('expected one tensor-core launch record, got %d' % len(paths))
    else:
        r = paths[0]
        want = describe(c)
        for k in ('M', 'N', 'K'):
            if r[k] != want[k]:
                rec['errors'].append('record %s=%d, case describes %d' % (k, r[k], want[k]))
        if tuple(r['kinds']) != tuple(want['kinds']):
            rec['errors'].append('record kinds=%r, case describes %r' % (r['kinds'], want['kinds']))
        bad = matches(r, c['runs'][config]) if declared else []
        if bad:
            rec['errors'].append('path: ' + ', '.join(bad))
    if c.get('deterministic'):
        (buf2, bits2), _ = capture_fd2(lambda: run_case(K, P, dev))
        if not (torch.equal(buf.view(torch.int32), buf2.view(torch.int32)) and
                (bits is None or torch.equal(bits, bits2))):
            rec['errors'].append('deterministic call: a second run gave other bits')
    d = buf.view(-1)[P.index.reshape(-1)].view(P.ref.shape)
    cmp = compare(d, P.ref, P.bound)
    rec.update(worst_ratio=cmp['worst_ratio'], worst_at=cmp['worst_at'], rel_err=cmp['rel_err'], tau=tau(P.K))
    if not cmp['ok']:
        rec['errors'].append('values: %d elements outside the bound, %d not finite, worst %.3g x bound at %s' % (
            cmp['nbad'], cmp['nonfinite'], cmp['worst_ratio'], cmp['worst_at']))
    tol = 6e-4 if c.get('epi', {}).get('tf32') else 2e-5
    if not declared:
        # a drawn call may sum up to KMAX products, most of them zero taps: its rounding grows like sqrt(K) against the
        # largest output (the elementwise bound above stays the rigorous check)
        tol *= max(1.0, (P.K / 2048.0) ** 0.5)
    # beyond KMAX the fp32 accumulation error of a K-long sum grows with K: the elementwise bound above is the check
    # that scales
    if P.K <= KMAX and not cmp['rel_err'] < tol:
        rec['errors'].append('global rel_err %.3g >= %g' % (cmp['rel_err'], tol))
    touched = guard_touched(buf, P.index)
    if touched:
        rec['errors'].append('%d guard elements overwritten' % touched)
    if bits is not None:
        n = P.ref.numel() // 32
        want_bits = pack_sign_bits(d.float())
        if not torch.equal(bits[:n], want_bits):
            rec['errors'].append('sign bits differ from the output in %d words' % int((bits[:n] != want_bits).sum()))
        if not bool((bits[n:] == 0x5A5A5A5A).all()):
            rec['errors'].append('sign-bit words past the output overwritten')
    cnt = K.gemm_workspace(buf.device)[:16384].view(torch.int32)
    if int(cnt.abs().sum()) != 0:
        rec['errors'].append('stream-K arrival counters not zero after the launch')
        cnt.zero_()
    rec['ok'] = not rec['errors']
    return rec


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--config', required=True, choices=sorted(CONFIGS))
    ap.add_argument('--out', required=True)
    args = ap.parse_args(argv)
    for k, v in CONFIGS[args.config].items():
        if os.environ.get(k) != v:
            raise SystemExit('configuration %s needs %s=%s in the environment' % (args.config, k, v))
    if os.environ.get('VLFB_DEBUG') != '1':
        raise SystemExit('the path records need VLFB_DEBUG=1')
    from vlfb import kernels as K
    dev = torch.device('cuda')
    K.set_gemm_backend('tcgen05')
    with open(args.out, 'w') as f:
        for c in CASES:
            if args.config not in c['runs']:
                continue
            print('[gemm_paths] config=%s case=%s' % (args.config, c['name']), flush=True)
            try:
                rec = check_case(K, c, args.config, dev)
            except Exception as ex:                       # a failing call is a result of the case, not of the run
                rec = dict(case=c['name'], config=args.config, ok=False, paths=[], errors=['%s: %s' % (type(ex).__name__, ex)])
            f.write(json.dumps(rec) + '\n')
            f.flush()
            torch.cuda.empty_cache()
    print('[gemm_paths] config=%s done' % args.config, flush=True)


if __name__ == '__main__':
    main()
