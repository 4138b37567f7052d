// C-ABI surface of libvlfb.so: argument validation + dispatch (see include/vlfb.h).
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace vlfb {

static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// tc_ok = false: a dense operand is not 16-byte addressable for the tensor-core loaders (odd row
// strides / extents such as a 157-class FC); such (tiny) problems run on the SIMT engine.
static int validate_gemm(const vlfb_gemm_params_t& p, bool& tc_ok) {
  tc_ok = true;
  VLFB_CHECK_ARG(p.a.ptr && p.b.ptr && p.d);
  VLFB_CHECK_ARG(p.M > 0 && p.N > 0 && p.K > 0);      // K = 0 (an empty sum) is rejected by both engines alike
  VLFB_CHECK_ARG(p.batch >= 1 && p.taps >= 1 && p.split_k >= 0);          // split_k 0 = chosen by the library
  VLFB_CHECK_ARG(!(p.taps > 1 && p.batch > 1));
  VLFB_CHECK_ARG(p.engine == VLFB_ENGINE_TCGEN05 || p.engine == VLFB_ENGINE_SIMT);
  VLFB_CHECK_ARG(p.tile_n == 0 || (p.tile_n >= 32 && p.tile_n <= 256 && p.tile_n % 32 == 0));
  VLFB_CHECK_ARG(p.split_k == 1 || (p.flags & VLFB_EPI_ATOMIC));
  VLFB_CHECK_ARG(!(p.split_k != 1 && (p.residual || p.relu_mask || p.relu_mask_bits || (p.flags & (VLFB_EPI_RELU | VLFB_EPI_TF32)))));
  VLFB_CHECK_ARG(!(p.relu_mask && p.relu_mask_bits));
  if (p.relu_bits_out) {
    if (!((p.flags & VLFB_EPI_RELU) && !(p.flags & VLFB_EPI_ATOMIC) && p.split_k == 1 && p.batch == 1 && p.taps == 1 &&
          p.ldd == p.N && (p.N & 31) == 0 && (reinterpret_cast<uintptr_t>(p.relu_bits_out) & 3) == 0)) {
      set_error("vlfb_gemm: relu_bits_out needs VLFB_EPI_RELU and a dense, non-atomic, unsplit output with N %% 32 == 0");
      return VLFB_E_BADARG;
    }
  }
  if (!(aligned16(p.a.ptr) && aligned16(p.b.ptr))) tc_ok = false;
  const vlfb_operand_t* ops[2] = {&p.a, &p.b};
  for (int i = 0; i < 2; ++i) {
    const vlfb_operand_t& o = *ops[i];
    const int extent = (i == 0) ? p.M : p.N;
    switch (o.kind) {
      case VLFB_OP_DENSE_K:
        if (!((o.ld & 3) == 0 && (o.batch_stride & 3) == 0 && (p.K & 3) == 0)) tc_ok = false;
        break;
      case VLFB_OP_DENSE_MN:
        if (!((o.ld & 3) == 0 && (o.batch_stride & 3) == 0 && (extent & 3) == 0)) tc_ok = false;
        break;
      case VLFB_OP_CONV_K:
        VLFB_CHECK_ARG(i == 0 && p.g.C % 32 == 0 && p.K == p.g.kT * p.g.kH * p.g.kW * p.g.C);
        VLFB_CHECK_ARG((int64_t)p.M == (int64_t)p.g.N * p.g.To * p.g.Ho * p.g.Wo);
        break;
      case VLFB_OP_DGRAD_K:
        VLFB_CHECK_ARG(i == 0 && p.g.Co % 32 == 0 && p.K == p.g.kT * p.g.kH * p.g.kW * p.g.Co);
        VLFB_CHECK_ARG((int64_t)p.M == (int64_t)p.g.N * p.g.T * p.g.H * p.g.W);
        break;
      case VLFB_OP_CONV_MN:
        VLFB_CHECK_ARG(i == 1 && p.N == p.g.kH * p.g.kW * p.g.C && (p.g.C & 3) == 0 && p.taps == p.g.kT);
        VLFB_CHECK_ARG((int64_t)p.K == (int64_t)p.g.N * p.g.To * p.g.Ho * p.g.Wo);
        VLFB_CHECK_ARG(p.g.kH <= 8 && p.g.kW <= 8);      // per-row validity bits of the gather loader
        break;
      case VLFB_OP_STEM_K:
        VLFB_CHECK_ARG(i == 0 && p.g.C == 4 && p.g.kW <= 8 && p.K == p.g.kT * p.g.kH * 32);
        VLFB_CHECK_ARG(p.g.dT == 1 && p.g.dH == 1 && p.g.dW == 1);
        VLFB_CHECK_ARG((int64_t)p.M == (int64_t)p.g.N * p.g.To * p.g.Ho * p.g.Wo);
        break;
      case VLFB_OP_STEM_MN:
        VLFB_CHECK_ARG(i == 1 && p.g.C == 4 && p.g.kW <= 8 && p.g.kH <= 8 && p.N == 32 * p.g.kH && p.taps == p.g.kT);
        VLFB_CHECK_ARG(p.g.dT == 1 && p.g.dH == 1 && p.g.dW == 1);
        VLFB_CHECK_ARG((int64_t)p.K == (int64_t)p.g.N * p.g.To * p.g.Ho * p.g.Wo);
        break;
      default:
        set_error("vlfb_gemm: unknown operand kind %d", o.kind);
        return VLFB_E_BADARG;
    }
  }
  if (p.a.kind >= VLFB_OP_CONV_K || p.b.kind >= VLFB_OP_CONV_K) {
    // the gather loaders keep element offsets in 32 bits
    const int64_t in_elems = (int64_t)p.g.N * p.g.T * p.g.H * p.g.W * p.g.C;
    const int64_t out_elems = (int64_t)p.g.N * p.g.To * p.g.Ho * p.g.Wo * p.g.Co;
    if (in_elems >= (1ll << 31) || out_elems >= (1ll << 31)) {
      set_error("vlfb_gemm: conv tensors of >= 2^31 elements are not supported (split the batch)");
      return VLFB_E_BADARG;
    }
  }
  return VLFB_OK;
}

}  // namespace vlfb

using namespace vlfb;

extern "C" {

int vlfb_version(void) { return 100; }
const char* vlfb_last_error(void) { return g_err; }
int vlfb_gemm_plan(const vlfb_gemm_params_t* p, int num_sms, vlfb_gemm_plan_t* plan) {
  VLFB_CHECK_ARG(p && plan && p->M > 0 && p->N > 0 && p->K > 0);
  gemm_tc_plan(*p, num_sms > 0 ? num_sms : 132, plan);
  return VLFB_OK;
}

size_t vlfb_gemm_workspace_bytes(void) { return gemm_tc_workspace_bytes(); }

#ifdef VLFB_TRACE
/* diagnostic build only (libvlfb_trace.so, scripts/trace_gemm.py): device buffer of 64 x gridDim clock64 slots */
int vlfb_debug_set_trace(void* buf) { vlfb::gemm_tc_set_trace(buf); return VLFB_OK; }
#endif

int vlfb_gemm(const vlfb_gemm_params_t* p, void* stream) {
  VLFB_CHECK_ARG(p != nullptr);
  bool tc_ok = true;
  int rc = validate_gemm(*p, tc_ok);
  if (rc != VLFB_OK) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (p->engine == VLFB_ENGINE_SIMT || !tc_ok) {
    // the cross-check engine stores element by element: the sign bits are a second pass over the dense output
    vlfb_gemm_params_t q = *p;
    q.relu_bits_out = nullptr;
    rc = gemm_simt(q, s);
    if (rc == VLFB_OK && p->relu_bits_out) rc = relu_bits(p->d, p->relu_bits_out, (int64_t)p->M * p->N, s);
    return rc;
  }
  return gemm_tc(*p, s);
}

}  // extern "C"
