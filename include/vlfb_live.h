/*
 * vlfb_live.h -- entry points with a live row count (included by vlfb.h; same conventions).
 *
 * B200.ROI_CAPACITY (DESIGN.md 4.6): a net's RoI rows are a fixed capacity R, captured once, of which the first
 * *live_rows are real; the rest are padding that the data feed rewrites at every step.  live_rows is a device int32
 * scalar read in stream order (so a captured CUDA graph sees the count of each replay), or NULL = all R rows.  Each
 * function computes what its twin without the suffix computes over rows [0, *live_rows), bit for bit where noted, and
 * never reads the inputs of a padded row.  The training FBO-NL stack takes the count as vlfb_fbo_cfg_t.live_rows.
 */
#ifndef VLFB_LIVE_H_
#define VLFB_LIVE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* vlfb_roi_align_fwd (executor.RoIAlignStep): rows >= *live_rows are written as zeros and their boxes are never read.
 * The live rows equal the R = *live_rows launch bit for bit. */
int vlfb_roi_align_fwd_live(const float* feat, const float* rois, float* out, int N, int H, int W, int C, int R, int PH,
                            int PW, float spatial_scale, int sampling_ratio, const int32_t* live_rows, void* stream);
/* vlfb_roi_align_bwd (executor.RoIAlignStep backward): rows >= *live_rows are neither read nor scattered. */
int vlfb_roi_align_bwd_live(const float* dout, const float* rois, float* dfeat /* accumulated */, int N, int H, int W,
                            int C, int R, int PH, int PW, float spatial_scale, int sampling_ratio,
                            const int32_t* live_rows, void* stream);
/* vlfb_roi_align_bwd_det (vlfb_det.h; the backward of a B200.DETERMINISTIC net): rows >= *live_rows are neither read
 * nor scattered, and the result equals the R = *live_rows launch bit for bit.  Scratch as for R rows. */
int vlfb_roi_align_bwd_det_live(const float* dout, const float* rois, float* dfeat /* accumulated */, int N, int H, int W,
                                int C, int R, int PH, int PW, float spatial_scale, int sampling_ratio, void* scratch,
                                size_t scratch_bytes, const int32_t* live_rows, void* stream);
/* vlfb_fbo_bank_scan_dt (executor.FboFoldStep, the inference FBO-NL over the raw bank): rows >= *live_rows are not
 * scanned and get out = 0 and prob = 0.  The splits and workspace are those of R rows, so a live row equals the
 * R = *live_rows launch bit for bit when both launches pick the same split (vlfb_fbo_bank_scan_splits_dt). */
int vlfb_fbo_bank_scan_live(const void* bank, int bank_dtype, const float* q, float scale, float* out, float* prob, int R,
                            int L, int D, int tf32_out, void* workspace, size_t workspace_bytes, const int32_t* live_rows,
                            void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VLFB_LIVE_H_ */
