/*
 * vlfb_det.h -- deterministic forms of the streaming reductions of libvlfb.so (included by vlfb.h; same conventions).
 *
 * The default entry points of vlfb.h combine float partial sums with atomics in whatever order the hardware picks, so
 * two identical calls may differ in the last bits.  Each function below computes the same sum as its default twin in a
 * fixed order: two calls with the same inputs (and the same output contents where the output is accumulated) give
 * bitwise-identical results on the same GPU model and library build.  The GEMM's deterministic form is the
 * vlfb_gemm_params_t.deterministic field (vlfb.h).  DESIGN.md 4.5 lists every cross-thread float reduction of a step.
 */
#ifndef VLFB_DET_H_
#define VLFB_DET_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* RoIAlign backward, deterministic: dfeat += the sum vlfb_roi_align_bwd adds.  Pass 1: one thread per (RoI, 4
 * channels) walks that RoI's bins and samples in order into the RoI's slab [H][W][C] of `scratch` (every slab is
 * written completely: no zero fill needed).  Pass 2: each feature element adds the slabs of its map's RoIs in RoI
 * order.  scratch: >= vlfb_roi_align_bwd_det_scratch_bytes(R, H, W, C) bytes (R H W C floats), 16-byte aligned,
 * owned by the caller; VLFB_E_WORKSPACE if smaller.  dout and dfeat are accessed as 16-byte vectors and must be 16-byte
 * aligned (VLFB_E_BADARG), unlike vlfb_roi_align_bwd's dfeat, which takes scalar atomics.  Other arguments as
 * vlfb_roi_align_bwd. */
size_t vlfb_roi_align_bwd_det_scratch_bytes(int R, int H, int W, int C);
int vlfb_roi_align_bwd_det(const float* dout, const float* rois, float* dfeat /* accumulated */, int N, int H, int W,
                           int C, int R, int PH, int PW, float spatial_scale, int sampling_ratio, void* scratch,
                           size_t scratch_bytes, void* stream);

/* out[c] (+)= sum_r x[r*ld + c], deterministic: one block per 32-column strip reduces all rows in a fixed order (8 row
 * lanes, then their sum in lane order) and adds the result to out once.  Arguments and `accumulate` as vlfb_colsum. */
int vlfb_colsum_det(const float* x, int64_t ld, float* out, int64_t rows, int cols, int accumulate, void* stream);
/* (One block per strip keeps these reductions short of the bandwidth of the default forms on narrow tensors: a
 * 64-channel strip over 10^5-10^6 rows runs on two blocks.) */

/* SpatialBN training forward / backward with reproducible batch statistics: one block per 32-channel strip reduces all
 * rows (fp32 per row lane, fp64 across the 8 lanes in lane order), so every fp64 accumulator receives a single
 * contribution.  Arguments, outputs and workspace (vlfb_spatial_bn_workspace_bytes) as vlfb_spatial_bn_fwd / _bwd. */
int vlfb_spatial_bn_fwd_det(const float* x, const float* scale, const float* bias, float* running_mean,
                            float* running_var, float* saved_mean, float* saved_inv_std, float* y, int64_t rows, int C,
                            float eps, float momentum, void* workspace, size_t workspace_bytes, void* stream);
int vlfb_spatial_bn_bwd_det(const float* dy, const float* x, const float* scale, const float* saved_mean,
                            const float* saved_inv_std, float* dx, float* dscale, float* dbias, int64_t rows, int C,
                            void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VLFB_DET_H_ */
