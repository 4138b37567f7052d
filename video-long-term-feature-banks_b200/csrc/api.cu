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
  VLFB_CHECK_ARG(p.batch >= 1 && p.taps >= 1 && p.split_k >= 0);          // split_k 0 (atomic) = chosen by the library
  VLFB_CHECK_ARG(!(p.taps > 1 && p.batch > 1));
  VLFB_CHECK_ARG(p.engine == VLFB_ENGINE_TCGEN05 || p.engine == VLFB_ENGINE_SIMT);
  VLFB_CHECK_ARG(p.tile_n == 0 || (p.tile_n >= 32 && p.tile_n <= 256 && p.tile_n % 32 == 0));
  VLFB_CHECK_ARG(p.split_k == 1 || (p.flags & VLFB_EPI_ATOMIC));
  VLFB_CHECK_ARG(p.deterministic == 0 || p.deterministic == 1);
  VLFB_CHECK_ARG(p.precision == VLFB_PREC_TF32 || p.precision == VLFB_PREC_X3);
  VLFB_CHECK_ARG(!(p.deterministic && p.split_k > 1));   // a deterministic launch is never split (split_k 0 = 1)
  const bool split = p.deterministic ? p.split_k > 1 : p.split_k != 1;
  VLFB_CHECK_ARG(!(split && (p.residual || p.relu_mask || p.relu_mask_bits || (p.flags & (VLFB_EPI_RELU | VLFB_EPI_TF32)))));
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

// groups > 1: the grouped-convolution forms of include/vlfb.h (fwd, dgrad, wgrad), run by gconv.cu.
#define GCONV_REQUIRE(cond, code, ...)  \
  do {                                  \
    if (!(cond)) {                      \
      set_error(__VA_ARGS__);           \
      return code;                      \
    }                                   \
  } while (0)

static int validate_gconv(const vlfb_gemm_params_t& p) {
  const vlfb_conv_geom_t& g = p.g;
  const int G = p.groups;
  VLFB_CHECK_ARG(p.a.ptr && p.b.ptr && p.d);
  VLFB_CHECK_ARG(p.M > 0 && p.N > 0 && p.K > 0);
  VLFB_CHECK_ARG(p.deterministic == 0 || p.deterministic == 1);
  VLFB_CHECK_ARG(p.precision == VLFB_PREC_TF32 || p.precision == VLFB_PREC_X3);   // fp32 products either way
  GCONV_REQUIRE(p.batch == 1, VLFB_E_UNSUPPORTED, "vlfb_gemm: groups > 1 needs batch == 1");
  GCONV_REQUIRE(p.split_k == 0 || p.split_k == 1, VLFB_E_UNSUPPORTED, "vlfb_gemm: groups > 1 needs split_k <= 1");
  GCONV_REQUIRE(p.a.kind != VLFB_OP_STEM_K && p.a.kind != VLFB_OP_STEM_MN && p.b.kind != VLFB_OP_STEM_K &&
                    p.b.kind != VLFB_OP_STEM_MN,
                VLFB_E_UNSUPPORTED, "vlfb_gemm: groups > 1 is not defined for the STEM_* operands");
  GCONV_REQUIRE(!(p.a.kind == VLFB_OP_DENSE_K), VLFB_E_UNSUPPORTED,
                "vlfb_gemm: groups > 1 with a DENSE_K A operand (a pointwise conv) is not supported");
  GCONV_REQUIRE(g.C > 0 && g.Co > 0 && g.C % G == 0 && g.Co % G == 0, VLFB_E_BADARG,
                "vlfb_gemm: groups = %d must divide C = %d and Co = %d", G, g.C, g.Co);
  const int Cig = g.C / G, Cog = g.Co / G;
  GCONV_REQUIRE(Cig % 4 == 0 && Cig >= 4 && Cig <= 64 && Cog % 4 == 0 && Cog >= 4 && Cog <= 64, VLFB_E_UNSUPPORTED,
                "vlfb_gemm: grouped conv widths Cig = %d, Cog = %d must be multiples of 4 in [4, 64]", Cig, Cog);
  VLFB_CHECK_ARG(g.N > 0 && g.T > 0 && g.H > 0 && g.W > 0 && g.To > 0 && g.Ho > 0 && g.Wo > 0);
  VLFB_CHECK_ARG(g.kT > 0 && g.kH > 0 && g.kW > 0 && g.sT > 0 && g.sH > 0 && g.sW > 0);
  VLFB_CHECK_ARG(g.pT >= 0 && g.pH >= 0 && g.pW >= 0 && g.dT > 0 && g.dH > 0 && g.dW > 0);
  const int64_t in_elems = (int64_t)g.N * g.T * g.H * g.W * g.C;
  const int64_t out_elems = (int64_t)g.N * g.To * g.Ho * g.Wo * g.Co;
  GCONV_REQUIRE(in_elems < (1ll << 31) && out_elems < (1ll << 31), VLFB_E_BADARG,
                "vlfb_gemm: conv tensors of >= 2^31 elements are not supported (split the batch)");
  const int taps = g.kT * g.kH * g.kW;
  const int64_t in_pos = (int64_t)g.N * g.T * g.H * g.W, out_pos = (int64_t)g.N * g.To * g.Ho * g.Wo;
  const uintptr_t mis = reinterpret_cast<uintptr_t>(p.a.ptr) | reinterpret_cast<uintptr_t>(p.b.ptr);
  VLFB_CHECK_ARG(!(p.relu_mask && p.relu_mask_bits));
  if (p.a.kind == VLFB_OP_DENSE_MN) {          // wgrad
    GCONV_REQUIRE(p.b.kind == VLFB_OP_CONV_MN && p.a.ld == g.Co && p.M == g.Co && p.N == g.kH * g.kW * Cig &&
                      p.taps == g.kT && (int64_t)p.K == out_pos,
                  VLFB_E_BADARG, "vlfb_gemm: grouped wgrad needs a = DENSE_MN dy (ld = Co), b = CONV_MN x, M = Co, "
                  "N = kH*kW*Cig, taps = kT, K = N*To*Ho*Wo");
    GCONV_REQUIRE((p.flags & VLFB_EPI_ATOMIC) && !(p.flags & (VLFB_EPI_RELU | VLFB_EPI_ACCUM | VLFB_EPI_TF32)) &&
                      !p.col_bias && !p.residual && !p.relu_mask && !p.relu_mask_bits && !p.relu_bits_out,
                  VLFB_E_BADARG, "vlfb_gemm: grouped wgrad accumulates (VLFB_EPI_ATOMIC) with alpha, col_scale and "
                  "row_scale only");
    GCONV_REQUIRE((mis & 15) == 0, VLFB_E_BADARG, "vlfb_gemm: grouped conv operands must be 16-byte aligned");
    return VLFB_OK;
  }
  const bool dgrad = p.a.kind == VLFB_OP_DGRAD_K;
  GCONV_REQUIRE(p.a.kind == VLFB_OP_CONV_K || dgrad, VLFB_E_BADARG,
                "vlfb_gemm: groups > 1 needs A = CONV_K (fwd), DGRAD_K (dgrad) or DENSE_MN (wgrad)");
  GCONV_REQUIRE(p.b.kind == VLFB_OP_DENSE_K && p.b.ld >= p.K, VLFB_E_BADARG,
                "vlfb_gemm: grouped fwd / dgrad needs b = DENSE_K weights with ld >= K");
  if (dgrad)
    GCONV_REQUIRE(p.N == g.C && p.K == taps * Cog && (int64_t)p.M == in_pos, VLFB_E_BADARG,
                  "vlfb_gemm: grouped dgrad needs M = N*T*H*W, N = C, K = taps*Cog");
  else
    GCONV_REQUIRE(p.N == g.Co && p.K == taps * Cig && (int64_t)p.M == out_pos, VLFB_E_BADARG,
                  "vlfb_gemm: grouped fwd needs M = N*To*Ho*Wo, N = Co, K = taps*Cig");
  GCONV_REQUIRE(!(p.flags & VLFB_EPI_ATOMIC), VLFB_E_UNSUPPORTED,
                "vlfb_gemm: grouped fwd / dgrad store their output (no VLFB_EPI_ATOMIC)");
  const uintptr_t out_mis = reinterpret_cast<uintptr_t>(p.a.ptr) | reinterpret_cast<uintptr_t>(p.d) |
                            reinterpret_cast<uintptr_t>(p.residual) | reinterpret_cast<uintptr_t>(p.relu_mask) |
                            reinterpret_cast<uintptr_t>(p.col_scale) | reinterpret_cast<uintptr_t>(p.col_bias);
  GCONV_REQUIRE((out_mis & 15) == 0 && p.ldd >= p.N && (p.ldd & 3) == 0, VLFB_E_BADARG,
                "vlfb_gemm: grouped fwd / dgrad need 16-byte aligned x / dy, d, residual, relu_mask, col_scale, "
                "col_bias and ldd %% 4 == 0");
  if (p.relu_bits_out)
    GCONV_REQUIRE((p.flags & VLFB_EPI_RELU) && p.ldd == p.N && (p.N & 31) == 0 &&
                      (reinterpret_cast<uintptr_t>(p.relu_bits_out) & 3) == 0,
                  VLFB_E_BADARG, "vlfb_gemm: relu_bits_out needs VLFB_EPI_RELU and a dense output with N %% 32 == 0");
  return VLFB_OK;
}
#undef GCONV_REQUIRE

}  // namespace vlfb

using namespace vlfb;

extern "C" {

int vlfb_version(void) { return 100; }
const char* vlfb_last_error(void) { return g_err; }
int vlfb_gemm_plan(const vlfb_gemm_params_t* p, int num_sms, vlfb_gemm_plan_t* plan) {
  VLFB_CHECK_ARG(p && plan && p->M > 0 && p->N > 0 && p->K > 0);
  VLFB_CHECK_ARG(p->precision == VLFB_PREC_TF32 || p->precision == VLFB_PREC_X3);
  if (p->groups > 1) {
    set_error("vlfb_gemm_plan: grouped convolutions (groups > 1) run on CUDA cores and have no tile plan");
    return VLFB_E_UNSUPPORTED;
  }
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
  VLFB_CHECK_ARG(p->groups >= 0);
  if (p->deterministic && (p->flags & VLFB_EPI_ATOMIC) &&
      !(p->workspace && p->workspace_bytes >= gemm_tc_workspace_bytes() && (reinterpret_cast<uintptr_t>(p->workspace) & 15) == 0)) {
    set_error("vlfb_gemm: a deterministic VLFB_EPI_ATOMIC launch needs a 16-byte aligned workspace of >= %zu bytes",
              gemm_tc_workspace_bytes());
    return VLFB_E_WORKSPACE;
  }
  if (p->groups > 1) {                 // Caffe2 grouped Conv: CUDA-core kernels, `engine` does not apply
    const int rc = validate_gconv(*p);
    return rc != VLFB_OK ? rc : gconv(*p, static_cast<cudaStream_t>(stream));
  }
  // split_k = 0 is the library's choice: a split for atomic epilogues, none for a stored output (each engine would
  // otherwise pick its own split, and a stored split overwrites its partial sums)
  vlfb_gemm_params_t q = *p;
  if (q.split_k == 0 && !(q.flags & VLFB_EPI_ATOMIC)) q.split_k = 1;
  bool tc_ok = true;
  int rc = validate_gemm(q, tc_ok);
  if (rc != VLFB_OK) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (q.engine == VLFB_ENGINE_SIMT || !tc_ok) {
    // the cross-check engine stores element by element: the sign bits are a second pass over the dense output
    uint32_t* bits = q.relu_bits_out;
    q.relu_bits_out = nullptr;
    rc = gemm_simt(q, s);
    if (rc == VLFB_OK && bits) rc = relu_bits(q.d, bits, (int64_t)q.M * q.N, s);
    return rc;
  }
  return gemm_tc(q, s);
}

}  // extern "C"
