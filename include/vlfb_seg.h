/*
 * vlfb_seg.h -- segmented entry points (included by vlfb.h; same conventions).
 *
 * B200.GPUS_PER_STEP (DESIGN.md 4.9): one training step runs S virtual GPUs as one batch.  The rows of a tensor are cut
 * into S contiguous segments, segment j being virtual GPU j's rows, and the two operations whose result depends on the
 * GPU boundary -- the sigmoid cross-entropy's per-GPU normalisation and SpatialBN's batch statistics -- compute per
 * segment.  Every function here with S = 1 computes what its unsegmented twin computes: bit for bit for the losses and
 * the _det forms, within the fp64 atomic-ordering spread for the default SpatialBN form.
 */
#ifndef VLFB_SEG_H_
#define VLFB_SEG_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Sigmoid cross-entropy of logits / targets [rows][cols] in S row segments: seg[0..S] is a device int32 array of row
 * offsets (seg[0] = 0, non-decreasing, seg[S] = rows), read in stream order so a captured graph sees each replay's
 * segments.  loss[0] = sum_j scale * CE_j / max(count_j, 1e-5), count_j = segment j's targets != -1, summed in segment
 * order; padded rows carry target -1 and count nowhere.  One block per segment: deterministic by construction. */
int vlfb_sigmoid_ce_seg_fwd(const float* logits, const int32_t* targets, const int32_t* seg, int S, int64_t rows,
                            int cols, float* loss, float scale, float* scratch /* S floats */, void* stream);
/* dlogits of the above: each row scaled by its own segment's count (times *dloss when dloss != NULL). */
int vlfb_sigmoid_ce_seg_bwd(const float* logits, const int32_t* targets, const int32_t* seg, int S, int64_t rows,
                            int cols, const float* dloss, float* dlogits, float scale, void* stream);

/* Training-mode SpatialBN of channels-last x [rows][C] with batch statistics per segment of rows / S contiguous rows
 * (rows % S == 0).  saved_mean / saved_inv_std are [S][C]; the running statistics (NULL: left alone) are updated from
 * segment 0's statistics only.  The workspace is vlfb_spatial_bn_seg_workspace_bytes(C, S). */
size_t vlfb_spatial_bn_seg_workspace_bytes(int C, int S);
int vlfb_spatial_bn_seg_fwd(const float* x, const float* scale, const float* bias, float* running_mean,
                            float* running_var, float* saved_mean, float* saved_inv_std, float* y, int64_t rows, int C,
                            int S, float eps, float momentum, void* workspace, size_t workspace_bytes, void* stream);
/* dx uses each segment's own statistics; dscale += sum_j sum dy * xhat_j and dbias += sum_j sum dy, added one segment
 * at a time in segment order (either may be NULL). */
int vlfb_spatial_bn_seg_bwd(const float* dy, const float* x, const float* scale, const float* saved_mean,
                            const float* saved_inv_std, float* dx, float* dscale, float* dbias, int64_t rows, int C,
                            int S, void* workspace, size_t workspace_bytes, void* stream);
/* The reproducible forms: one slab per (segment, 32-channel strip), so every sum has a fixed order. */
int vlfb_spatial_bn_seg_fwd_det(const float* x, const float* scale, const float* bias, float* running_mean,
                                float* running_var, float* saved_mean, float* saved_inv_std, float* y, int64_t rows,
                                int C, int S, float eps, float momentum, void* workspace, size_t workspace_bytes,
                                void* stream);
int vlfb_spatial_bn_seg_bwd_det(const float* dy, const float* x, const float* scale, const float* saved_mean,
                                const float* saved_inv_std, float* dx, float* dscale, float* dbias, int64_t rows, int C,
                                int S, void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VLFB_SEG_H_ */
