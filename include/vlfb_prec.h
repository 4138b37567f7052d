/*
 * vlfb_prec.h -- entry points of the split-TF32 GEMM precision (vlfb_gemm_params_t.precision = VLFB_PREC_X3, DESIGN.md
 * 4.7).  Included by vlfb.h; same conventions.
 */
#ifndef VLFB_PREC_H_
#define VLFB_PREC_H_

#ifdef __cplusplus
extern "C" {
#endif

/* The jobs of vlfb_weight_transpose_multi without the rounding: wt[ci][tap][co] = w[co][tap][ci] * (scale ? scale[co] : 1),
 * the dgrad B operand of a VLFB_PREC_X3 GEMM. */
int vlfb_weight_scale_transpose_multi(const vlfb_wt_job_t* jobs, int njobs, int total_blocks, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VLFB_PREC_H_ */
