// Feature-bank kernels that work on the RAW long-term bank (HBM-bound scans / gathers), sm_90a.
//
// 1. fbo_bank_scan / fbo_bank_combine: the inference-mode Feature-Bank Operator.  Without dropout between
//    'lfb_1x1' and the phi/g projections (lfb_helper.py:320-338 with test_mode), one FBO-NL layer with a single
//    query per RoI (lfb_helper.NLCore :170-263, num_feat1 == 1) folds algebraically:
//        score_j  = theta . (W_phi (W_1 b_j + c_1) + c_phi) = (W_1^T W_phi^T theta) . b_j + const   (const drops
//                   out of the softmax),
//        sum_j p_j g_j = W_g (W_1 (sum_j p_j b_j) + c_1) + c_g                                      (sum_j p_j = 1),
//    so the layer is ONE pass over the raw bank rows b_j (R x L x D fp32): q . b_j, online softmax, weighted row
//    sum.  The (R*L x D x d) projections of the as-written graph (314.6 MMAC per RoI at L=300 + 157 MMAC per
//    layer, SURVEY 8a a14/a15) disappear; what is left are four R-row matmuls per layer on the tensor-core GEMM.
//    Roofline: HBM.  Algorithmic bytes per launch = R*L*D*4 (every bank element is read exactly once).
// 2. lfb_gather: builds the per-sample (L x D) bank windows on the device from a resident bank tensor and a host
//    computed row-index table (tools/lfb_loader.py:51-152 + lib/datasets/ava.py:300-323: -1 = zero padding).
#include <float.h>
#include <limits.h>
#include <string.h>

#include "common.cuh"

namespace vlfb {
namespace {

constexpr int SCAN_TPB = 256;
// bf16 bank rows (2048 elements = 4 KB): rows per tile / resident CTAs per SM of the scan.  4 rows at 4 CTAs per SM
// (64 registers, no spills): the unpacked rows cost registers, so occupancy is favoured over tile depth.  A build
// parameter; not re-tuned on the H100.
#ifndef VLFB_SCAN16_ROWS
#define VLFB_SCAN16_ROWS 4
#endif
#ifndef VLFB_SCAN16_MINB
#define VLFB_SCAN16_MINB 4
#endif
#ifndef VLFB_SCAN16_VOLATILE
#define VLFB_SCAN16_VOLATILE 0
#endif

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ uint4 ldg_stream_u4(const uint4* p) {   // read-once data: do not keep it in L1
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}
// 16 bytes of bank row -> EPL floats: 4 fp32, or 8 bf16 (element 2i in the low half of word i)
template <int EPL>
__device__ __forceinline__ void unpack16(const uint4& u, float (&f)[EPL]) {
  if (EPL == 4) {
    f[0] = __uint_as_float(u.x); f[1] = __uint_as_float(u.y); f[2] = __uint_as_float(u.z); f[3] = __uint_as_float(u.w);
  } else {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#if VLFB_SCAN16_VOLATILE      // forces the second use (weighted sum) to unpack again instead of keeping 8 floats per row live
      uint32_t lo, hi;
      asm volatile("shl.b32 %0, %1, 16;" : "=r"(lo) : "r"(w[i]));
      asm volatile("and.b32 %0, %1, 0xffff0000;" : "=r"(hi) : "r"(w[i]));
#else
      const uint32_t lo = w[i] << 16, hi = w[i] & 0xffff0000u;
#endif
      f[(2 * i) % EPL] = __uint_as_float(lo);
      f[(2 * i + 1) % EPL] = __uint_as_float(hi);
    }
  }
}

// One CTA = rows [row_begin, row_end) of one RoI.  EPL = bank elements per 16-byte load (4: fp32 bank, 8: bf16 bank),
// V = 16-byte loads per thread per row (D = 256 * V * EPL), ROWS = rows per tile: ROWS*V independent 16-byte loads per
// thread are in flight before the first use (fp32: 64 KB per CTA, two CTAs per SM; bf16: 16 KB, four CTAs per SM).  Per tile: partial dots -> warp
// shuffles -> one shared-memory exchange between the 8 warps (double buffered: one __syncthreads per tile) -> every
// thread redoes the tiny online-softmax update and rescales / accumulates its V*EPL columns from the registers that
// still hold the rows.  Scores, softmax and the weighted sum are fp32 whatever the bank's storage type.
template <int EPL, int V, int ROWS>
__global__ void __launch_bounds__(SCAN_TPB, (EPL == 8 && V == 1) ? VLFB_SCAN16_MINB : 2)
fbo_bank_scan_k(const void* __restrict__ bank, const float* __restrict__ q, float scale, float* __restrict__ part_acc,
                float* __restrict__ part_ml, float* __restrict__ scores, int L, int S, int rows_per_split,
                const int32_t* __restrict__ live) {
  constexpr int D = SCAN_TPB * V * EPL;
  constexpr int NW = SCAN_TPB / 32;
  __shared__ float xch[2][NW][ROWS];
  const int r = blockIdx.x / S, sp = blockIdx.x % S;
  if (live != nullptr && r >= *live) return;          // padding row: fbo_bank_combine_k writes its zeros
  const int row_begin = sp * rows_per_split;
  const int row_end = min(L, row_begin + rows_per_split);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint4* brow = reinterpret_cast<const uint4*>(bank) + (int64_t)r * L * (SCAN_TPB * V);
  const float* qr = q + (int64_t)r * D;
  float qv[V][EPL], acc[V][EPL];
#pragma unroll
  for (int v = 0; v < V; ++v) {
#pragma unroll
    for (int e = 0; e < EPL; e += 4) {
      const float4 t = *reinterpret_cast<const float4*>(qr + (v * SCAN_TPB + tid) * EPL + e);
      qv[v][e] = t.x; qv[v][e + 1] = t.y; qv[v][e + 2] = t.z; qv[v][e + 3] = t.w;
    }
#pragma unroll
    for (int e = 0; e < EPL; ++e) acc[v][e] = 0.f;
  }
  float m = -FLT_MAX, l = 0.f;
  int buf = 0;
  for (int j0 = row_begin; j0 < row_end; j0 += ROWS, buf ^= 1) {
    uint4 x[ROWS][V];
#pragma unroll
    for (int i = 0; i < ROWS; ++i) {
      const bool ok = j0 + i < row_end;
#pragma unroll
      for (int v = 0; v < V; ++v)
        x[i][v] = ok ? ldg_stream_u4(brow + (int64_t)(j0 + i) * (SCAN_TPB * V) + v * SCAN_TPB + tid) : make_uint4(0u, 0u, 0u, 0u);
    }
    float part[ROWS];
#pragma unroll
    for (int i = 0; i < ROWS; ++i) {
      float s = 0.f;
#pragma unroll
      for (int v = 0; v < V; ++v) {
        float f[EPL];
        unpack16<EPL>(x[i][v], f);
#pragma unroll
        for (int e = 0; e < EPL; ++e) s += f[e] * qv[v][e];
      }
      part[i] = warp_sum_f(s);
    }
    if (lane == 0) {
#pragma unroll
      for (int i = 0; i < ROWS; ++i) xch[buf][warp][i] = part[i];
    }
    __syncthreads();
    float sc[ROWS], mx = m;
#pragma unroll
    for (int i = 0; i < ROWS; ++i) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < NW; ++w) s += xch[buf][w][i];
      s = (j0 + i < row_end) ? s * scale : -FLT_MAX;
      sc[i] = s;
      mx = fmaxf(mx, s);
    }
    if (scores != nullptr && tid < ROWS && j0 + tid < row_end) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < NW; ++w) s += xch[buf][w][tid];
      scores[(int64_t)r * L + j0 + tid] = s * scale;
    }
    const float corr = __expf(m - mx);      // m == -FLT_MAX on the first tile: exp(-huge) == 0 and acc, l are 0
    l *= corr;
#pragma unroll
    for (int v = 0; v < V; ++v) {
#pragma unroll
      for (int e = 0; e < EPL; ++e) acc[v][e] *= corr;
    }
#pragma unroll
    for (int i = 0; i < ROWS; ++i) {
      const float p = (j0 + i < row_end) ? __expf(sc[i] - mx) : 0.f;
      l += p;
#pragma unroll
      for (int v = 0; v < V; ++v) {
        float f[EPL];
        unpack16<EPL>(x[i][v], f);
#pragma unroll
        for (int e = 0; e < EPL; ++e) acc[v][e] += p * f[e];
      }
    }
    m = mx;
  }
  float* pa = part_acc + ((int64_t)r * S + sp) * D;
#pragma unroll
  for (int v = 0; v < V; ++v) {
#pragma unroll
    for (int e = 0; e < EPL; e += 4)
      *reinterpret_cast<float4*>(pa + (v * SCAN_TPB + tid) * EPL + e) =
          make_float4(acc[v][e], acc[v][e + 1], acc[v][e + 2], acc[v][e + 3]);
  }
  if (tid == 0) {
    part_ml[((int64_t)r * S + sp) * 2 + 0] = m;
    part_ml[((int64_t)r * S + sp) * 2 + 1] = l;
  }
}

// y = bf16(x), round to nearest even (the storage type of a bf16 feature bank); 8 elements per thread and iteration
__global__ void f32_to_bf16_k(const float4* __restrict__ x, uint4* __restrict__ y, int64_t n8) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 a = x[2 * i], b = x[2 * i + 1];
    const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    uint32_t h[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const uint32_t u = __float_as_uint(f[k]);
      h[k] = (u + 0x7fffu + ((u >> 16) & 1u)) >> 16;          // NaN payloads aside (banks are finite features)
    }
    y[i] = make_uint4(h[0] | (h[1] << 16), h[2] | (h[3] << 16), h[4] | (h[5] << 16), h[6] | (h[7] << 16));
  }
}

// s[r][:] = sum_sp w_sp acc_sp[:] / sum_sp w_sp l_sp, w_sp = exp(m_sp - max m); optional TF32 rounding (the result is
// the A operand of the W_1 matmul).  prob[r][j] = exp(score - M) / lsum when the scores were kept.
__global__ void fbo_bank_combine_k(const float* __restrict__ part_acc, const float* __restrict__ part_ml,
                                   float* __restrict__ out, float* __restrict__ scores_prob, int S, int D, int L,
                                   int tf32_out, const int32_t* __restrict__ live) {
  const int r = blockIdx.y;
  if (live != nullptr && r >= *live) {                 // padding row: out = 0, prob = 0
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < D) out[(int64_t)r * D + c] = 0.f;
    if (scores_prob != nullptr)
      for (int j = c; j < L; j += gridDim.x * blockDim.x) scores_prob[(int64_t)r * L + j] = 0.f;
    return;
  }
  float M = -FLT_MAX;
  for (int s = 0; s < S; ++s)
    if (part_ml[((int64_t)r * S + s) * 2 + 1] > 0.f) M = fmaxf(M, part_ml[((int64_t)r * S + s) * 2]);
  float lsum = 0.f;
  for (int s = 0; s < S; ++s) {
    const float ls = part_ml[((int64_t)r * S + s) * 2 + 1];
    if (ls > 0.f) lsum += ls * __expf(part_ml[((int64_t)r * S + s) * 2] - M);
  }
  const float inv = lsum > 0.f ? 1.f / lsum : 0.f;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < D) {
    float a = 0.f;
    for (int s = 0; s < S; ++s) {
      const float ls = part_ml[((int64_t)r * S + s) * 2 + 1];
      if (ls > 0.f) a += part_acc[((int64_t)r * S + s) * D + c] * __expf(part_ml[((int64_t)r * S + s) * 2] - M);
    }
    a *= inv;
    out[(int64_t)r * D + c] = tf32_out ? round_tf32(a) : a;
  }
  if (scores_prob != nullptr) {
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < L; j += gridDim.x * blockDim.x)
      scores_prob[(int64_t)r * L + j] = __expf(scores_prob[(int64_t)r * L + j] - M) * inv;
  }
}

// out[i][:] = idx[i] >= 0 ? bank[idx[i]][:] : 0   (rows of D floats, D % 4 == 0); one warp-wide float4 lane per 16 B.
__global__ void lfb_gather_k(const float4* __restrict__ bank, const int32_t* __restrict__ idx, float4* __restrict__ out,
                             int64_t rows, int d4, int64_t bank_rows, int tf32_out) {
  const int64_t total = rows * d4;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / d4;
    const int c = (int)(i - row * d4);
    const int32_t src = idx[row];
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (src >= 0 && src < bank_rows) v = bank[(int64_t)src * d4 + c];
    if (tf32_out) { v.x = round_tf32(v.x); v.y = round_tf32(v.y); v.z = round_tf32(v.z); v.w = round_tf32(v.w); }
    out[i] = v;
  }
}


// ---------------------------------------------------------------------------------------------------------------
// 3. fbo_nl_fwd / fbo_nl_bwd: the TRAINING-mode FBO-NL stack (lfb_helper.NLLayers :266-292 over NLCore :170-263) with
//    one query per RoI, as ONE launch per direction.  Dropout sits between 'lfb_1x1' and the phi / g projections
//    (prepare_lfb :320-338), so the raw-bank fold of the inference graph is not valid -- but the SAME algebra applies
//    one step later, on the projected (and dropped-out) bank B' [R][L][dB] that all layers share:
//        score_j = theta . (W_phi B'_j + b_phi) = (W_phi^T theta) . B'_j + const       (const drops out of the softmax)
//        sum_j p_j (W_g B'_j + b_g) = W_g (sum_j p_j B'_j) + b_g                        (sum_j p_j = 1)
//    i.e. phi and g (2 x R*L x dB x d MACs per layer forward, 4 more GEMMs backward) are never formed: a layer is four
//    d x d mat-vecs and two passes over B' per RoI.  The as-written graph spends 41 GEMM launches + ~70 streaming
//    launches on R*L = 1200 rows; here one CTA per RoI walks all
//    layers.  Gradients: exact (the b_phi / theta terms that multiply sum_j dscore_j = 0 are kept for parity with the
//    reference's autograd); the rank-R weight gradients are accumulated by fbo_nl_outer_k from the per-RoI vectors.
constexpr int NL_TPB = 512;
constexpr int NL_MAX_LAYERS = 4;

struct NlParams {
  vlfb_fbo_cfg_t c;
  vlfb_fbo_layer_t l[NL_MAX_LAYERS];
  const float* a0;       // [R][dA] query input of layer 0
  const float* bp;       // [R][L][dB] projected bank (after dropout)
  const float* da_last;  // bwd: gradient of the last layer's sum [R][dA]
  float* da0;            // bwd: gradient of a0
  float* dbp;            // bwd: gradient of bp (overwritten)
  float* scratch;        // bwd: per layer [R][dA + d + dB + d + 4]: do, dt, du, dtheta, sum_j dscore_j
};

__device__ __forceinline__ float block_sum_nl(float v, float* red) {
  v = warp_sum_f(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = (threadIdx.x < NL_TPB / 32) ? red[threadIdx.x] : 0.f;
  if (threadIdx.x < 32) {
    t = warp_sum_f(t);
    if (threadIdx.x == 0) red[0] = t;
  }
  __syncthreads();
  return red[0];
}
__device__ __forceinline__ float block_max_nl(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = (threadIdx.x < NL_TPB / 32) ? red[threadIdx.x] : -FLT_MAX;
  if (threadIdx.x < 32) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t = fmaxf(t, __shfl_xor_sync(0xffffffffu, t, o));
    if (threadIdx.x == 0) red[0] = t;
  }
  __syncthreads();
  return red[0];
}
// One CTA streams ~5 MB of weights / bank rows per layer from L2: the loads must be deep enough in flight to hide the
// L2 latency (Little's law): 4 scalar loads per thread in flight would leave a CTA latency-bound -- hence 4 rows per
// warp (matvec_rows: 16 x 16-byte loads per lane) and 8 rows x 16 bytes per thread (colsum_w) below.
// out[row] = bias[row] + sum_c W[row][c] x[c]   (one warp per 4 rows, 128-bit lanes; cols % 4 == 0)
__device__ __forceinline__ void matvec_rows(const float* __restrict__ W, const float* x, float* out,
                                            const float* __restrict__ bias, int rows, int cols) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c4n = cols >> 2;
  for (int row0 = warp * 4; row0 < rows; row0 += 4 * (NL_TPB / 32)) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int c = lane; c < c4n; c += 32) {
      const float4 b = *reinterpret_cast<const float4*>(x + 4 * c);
      float4 a[4];
#pragma unroll
      for (int r = 0; r < 4; ++r)
        a[r] = (row0 + r < rows) ? reinterpret_cast<const float4*>(W + (int64_t)(row0 + r) * cols)[c] : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[r] += a[r].x * b.x + a[r].y * b.y + a[r].z * b.z + a[r].w * b.w;
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const float v = warp_sum_f(acc[r]);
      if (lane == 0 && row0 + r < rows) out[row0 + r] = v + (bias ? bias[row0 + r] : 0.f);
    }
  }
}
// out[c] = sum_r w[r] M[r][c]  (M row-major [rows][cols], cols % 4 == 0; w, out in shared memory; `part` = scratch of
// NL_TPB float4).  Thread groups of cols/4 threads own disjoint row sets; each thread keeps 8 rows x 16 bytes in flight.
// Ends with a __syncthreads(); the caller synchronises before (w ready) as usual.
__device__ __forceinline__ void colsum_w(const float* __restrict__ M, int rows, int cols, const float* w, float* out,
                                         float4* part) {
  const int c4n = cols >> 2;
  const int G = NL_TPB / c4n > 0 ? NL_TPB / c4n : 1;            // row groups (cols = 512: 4; cols = 2048: 1)
  for (int cbase = 0; cbase < c4n; cbase += NL_TPB) {            // cols > 4 * NL_TPB: several column passes
    const int tg = G > 1 ? threadIdx.x / c4n : 0;
    const int c4 = G > 1 ? threadIdx.x - tg * c4n : cbase + threadIdx.x;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c4 < c4n && tg < G) {
      const float4* m4 = reinterpret_cast<const float4*>(M) + c4;
      int r = tg;
      for (; r + 7 * G < rows; r += 8 * G) {
        float4 v[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) v[q] = m4[(int64_t)(r + q * G) * c4n];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float ww = w[r + q * G];
          acc.x += ww * v[q].x; acc.y += ww * v[q].y; acc.z += ww * v[q].z; acc.w += ww * v[q].w;
        }
      }
      for (; r < rows; r += G) {
        const float4 v = m4[(int64_t)r * c4n];
        const float ww = w[r];
        acc.x += ww * v.x; acc.y += ww * v.y; acc.z += ww * v.z; acc.w += ww * v.w;
      }
    }
    if (G > 1) {
      part[threadIdx.x] = acc;
      __syncthreads();
      if (threadIdx.x < c4n) {
        float4 t = part[threadIdx.x];
        for (int g = 1; g < G; ++g) {
          const float4 u = part[g * c4n + threadIdx.x];
          t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w;
        }
        *reinterpret_cast<float4*>(out + 4 * threadIdx.x) = t;
      }
      __syncthreads();
      return;                                                    // G > 1 implies a single column pass
    }
    if (c4 < c4n) *reinterpret_cast<float4*>(out + 4 * c4) = acc;
  }
  __syncthreads();
}
// out[c] = sum_row W[row][c] x[row]   (= W^T x)
__device__ __forceinline__ void matvec_cols(const float* __restrict__ W, const float* x, float* out, int rows, int cols,
                                            float4* part) {
  colsum_w(W, rows, cols, x, out, part);
}
// the generator of vlfb_dropout_fwd (csrc/ops.cu): element idx keeps iff u(idx) >= ratio, scaled by 1 / (1 - ratio)
__device__ __forceinline__ float philox_keep(uint64_t seed, uint64_t offset, int64_t idx, float ratio) {
  const uint64_t ctr = offset + (uint64_t)(idx >> 2);
  uint32_t c0 = (uint32_t)ctr, c1 = (uint32_t)(ctr >> 32), c2 = 0u, c3 = 0u;
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t h0 = __umulhi(0xD2511F53u, c0), l0 = 0xD2511F53u * c0;
    const uint32_t h1 = __umulhi(0xCD9E8D57u, c2), l1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = h1 ^ c1 ^ k0, n1 = l1, n2 = h0 ^ c3 ^ k1, n3 = l0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  const uint32_t rr[4] = {c0, c1, c2, c3};
  const float u = (float)(rr[idx & 3] >> 8) * (1.0f / 16777216.0f);
  return (u >= ratio) ? 1.f / (1.f - ratio) : 0.f;
}

// smem: part[NL_TPB float4] | sA[dA] | sTh[d] | sU[dB] | sS[dB] | sT[d] | sAct[d] | sO[dA] | sE[L] | red[32]
__global__ void __launch_bounds__(NL_TPB, 1) fbo_nl_fwd_k(const NlParams P) {
  extern __shared__ float sm[];
  const vlfb_fbo_cfg_t& c = P.c;
  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float4* part = reinterpret_cast<float4*>(sm);
  float* sA = sm + 4 * NL_TPB;
  float* sTh = sA + c.dA;
  float* sU = sTh + c.d;
  float* sS = sU + c.dB;
  float* sT = sS + c.dB;
  float* sAct = sT + c.d;
  float* sO = sAct + c.d;
  float* sE = sO + c.dA;
  float* red = sE + ((c.L + 3) & ~3);
  const float* B = P.bp + (int64_t)r * c.L * c.dB;
  if (c.live_rows != nullptr && r >= *c.live_rows) {            // padding row: zeros in every per-row output
    for (int li = 0; li < c.layers; ++li) {
      const vlfb_fbo_layer_t& l = P.l[li];
      for (int i = tid; i < c.d; i += NL_TPB) {
        l.theta[(int64_t)r * c.d + i] = 0.f; l.t[(int64_t)r * c.d + i] = 0.f; l.xhat[(int64_t)r * c.d + i] = 0.f;
      }
      for (int i = tid; i < c.dB; i += NL_TPB) l.s[(int64_t)r * c.dB + i] = 0.f;
      for (int j = tid; j < c.L; j += NL_TPB) l.prob[(int64_t)r * c.L + j] = 0.f;
      for (int i = tid; i < c.dA; i += NL_TPB) { l.out[(int64_t)r * c.dA + i] = 0.f; l.a_out[(int64_t)r * c.dA + i] = 0.f; }
      if (tid == 0) { l.ln_mean[r] = 0.f; l.ln_std[r] = 0.f; }
    }
    return;
  }
  for (int i = tid; i < c.dA; i += NL_TPB) sA[i] = P.a0[(int64_t)r * c.dA + i];
  __syncthreads();
  uint64_t step_off = c.step ? ((uint64_t)c.step[0] << 32) : 0ull;
  for (int li = 0; li < c.layers; ++li) {
    const vlfb_fbo_layer_t& l = P.l[li];
    matvec_rows(l.w_theta, sA, sTh, l.b_theta, c.d, c.dA);
    __syncthreads();
    for (int i = tid; i < c.d; i += NL_TPB) l.theta[(int64_t)r * c.d + i] = sTh[i];
    matvec_cols(l.w_phi, sTh, sU, c.d, c.dB, part);
    for (int j = warp; j < c.L; j += NL_TPB / 32) {             // scores (the theta . b_phi constant is dropped)
      const float4* b4 = reinterpret_cast<const float4*>(B + (int64_t)j * c.dB);
      float acc = 0.f;
      for (int q = lane; q < (c.dB >> 2); q += 32) {
        const float4 a = b4[q];
        const float4 u = *reinterpret_cast<const float4*>(sU + 4 * q);
        acc += a.x * u.x + a.y * u.y + a.z * u.z + a.w * u.w;
      }
      acc = warp_sum_f(acc);
      if (lane == 0) sE[j] = acc * c.scale;
    }
    __syncthreads();
    float mx = -FLT_MAX;
    for (int j = tid; j < c.L; j += NL_TPB) mx = fmaxf(mx, sE[j]);
    mx = block_max_nl(mx, red);
    float sum = 0.f;
    for (int j = tid; j < c.L; j += NL_TPB) { const float e = __expf(sE[j] - mx); sE[j] = e; sum += e; }
    sum = block_sum_nl(sum, red);
    const float inv = 1.f / sum;
    for (int j = tid; j < c.L; j += NL_TPB) { const float pv = sE[j] * inv; sE[j] = pv; l.prob[(int64_t)r * c.L + j] = pv; }
    __syncthreads();
    colsum_w(B, c.L, c.dB, sE, sS, part);                       // s = sum_j p_j B'_j
    for (int i = tid; i < c.dB; i += NL_TPB) l.s[(int64_t)r * c.dB + i] = sS[i];
    matvec_rows(l.w_g, sS, sT, l.b_g, c.d, c.dB);
    __syncthreads();
    for (int i = tid; i < c.d; i += NL_TPB) l.t[(int64_t)r * c.d + i] = sT[i];
    // pre-activation: LayerNorm over the d channels (no affine, biased variance) then ReLU
    float mean = 0.f, rstd = 1.f;
    if (c.pre_act_ln) {
      float a = 0.f;
      for (int i = tid; i < c.d; i += NL_TPB) a += sT[i];
      mean = block_sum_nl(a, red) / (float)c.d;
      float v = 0.f;
      for (int i = tid; i < c.d; i += NL_TPB) { const float dlt = sT[i] - mean; v += dlt * dlt; }
      const float var = block_sum_nl(v, red) / (float)c.d;
      const float sd = sqrtf(var + c.ln_eps);
      rstd = 1.f / sd;
      if (tid == 0) { l.ln_std[r] = sd; l.ln_mean[r] = mean; }
    }
    for (int i = tid; i < c.d; i += NL_TPB) {
      const float xh = (sT[i] - mean) * rstd;
      l.xhat[(int64_t)r * c.d + i] = xh;
      sAct[i] = fmaxf(xh, 0.f);
    }
    __syncthreads();
    matvec_rows(l.w_out, sAct, sO, l.b_out, c.dA, c.d);
    __syncthreads();
    for (int i = tid; i < c.dA; i += NL_TPB) {                  // out -> dropout -> residual sum
      float o = sO[i];
      l.out[(int64_t)r * c.dA + i] = o;
      if (c.drop_ratio > 0.f) o *= philox_keep(c.seed, l.drop_offset + step_off, (int64_t)r * c.dA + i, c.drop_ratio);
      const float a = sA[i] + o;
      sA[i] = a;
      l.a_out[(int64_t)r * c.dA + i] = a;
    }
    __syncthreads();
  }
}

// smem: part[NL_TPB float4] | sA[dA] | sTh[d] | sU[dB] | sS[dB] | sX[d] (xhat) | sV1[max(dA,d,dB)] | sV2[max] | sV3[max] | sDA[dA] | sP[L] | sD[L] | red
__global__ void __launch_bounds__(NL_TPB, 1) fbo_nl_bwd_k(const NlParams P) {
  extern __shared__ float sm[];
  const vlfb_fbo_cfg_t& c = P.c;
  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int mx3 = max(c.dA, max(c.d, c.dB));
  float4* part = reinterpret_cast<float4*>(sm);
  float* sA = sm + 4 * NL_TPB;
  float* sTh = sA + c.dA;
  float* sU = sTh + c.d;
  float* sS = sU + c.dB;
  float* sX = sS + c.dB;
  float* sV1 = sX + c.d;
  float* sV2 = sV1 + mx3;
  float* sV3 = sV2 + mx3;
  float* sDA = sV3 + mx3;
  float* sP = sDA + c.dA;
  float* sD = sP + ((c.L + 3) & ~3);
  float* red = sD + ((c.L + 3) & ~3);
  const float* B = P.bp + (int64_t)r * c.L * c.dB;
  float* dB = P.dbp + (int64_t)r * c.L * c.dB;
  const int per_roi = c.dA + c.d + c.dB + c.d + 4;
  if (c.live_rows != nullptr && r >= *c.live_rows) {            // padding row: zero gradients, no scratch (outer_k skips it)
    for (int i = tid; i < c.dA; i += NL_TPB) P.da0[(int64_t)r * c.dA + i] = 0.f;
    float4* dB4 = reinterpret_cast<float4*>(dB);
    for (int64_t e = tid; e < (int64_t)c.L * (c.dB >> 2); e += NL_TPB) dB4[e] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  for (int i = tid; i < c.dA; i += NL_TPB) sDA[i] = P.da_last[(int64_t)r * c.dA + i];
  __syncthreads();
  const uint64_t step_off = c.step ? ((uint64_t)c.step[0] << 32) : 0ull;
  for (int li = c.layers - 1; li >= 0; --li) {
    const vlfb_fbo_layer_t& l = P.l[li];
    float* scr = P.scratch + ((int64_t)li * c.R + r) * per_roi;
    float* g_do = scr;
    float* g_dt = g_do + c.dA;
    float* g_du = g_dt + c.d;
    float* g_dth = g_du + c.dB;
    float* g_sum = g_dth + c.d;
    const float* a_in = li == 0 ? P.a0 : P.l[li - 1].a_out;
    for (int i = tid; i < c.dA; i += NL_TPB) sA[i] = a_in[(int64_t)r * c.dA + i];
    for (int i = tid; i < c.d; i += NL_TPB) { sTh[i] = l.theta[(int64_t)r * c.d + i]; sX[i] = l.xhat[(int64_t)r * c.d + i]; }
    for (int i = tid; i < c.dB; i += NL_TPB) sS[i] = l.s[(int64_t)r * c.dB + i];
    for (int j = tid; j < c.L; j += NL_TPB) sP[j] = l.prob[(int64_t)r * c.L + j];
    // d(out) = dropout backward of the residual branch; the identity branch keeps sDA
    for (int i = tid; i < c.dA; i += NL_TPB) {
      float v = sDA[i];
      if (c.drop_ratio > 0.f) v *= philox_keep(c.seed, l.drop_offset + step_off, (int64_t)r * c.dA + i, c.drop_ratio);
      sV1[i] = v;
      g_do[i] = v;
    }
    __syncthreads();
    matvec_cols(l.w_out, sV1, sV2, c.dA, c.d, part);            // d(act) = W_out^T d(out)
    // ReLU + LayerNorm backward: dt = (dy - mean(dy) - xhat mean(dy xhat)) / std, dy = d(act) where xhat > 0
    float m1 = 0.f, m2 = 0.f;
    for (int i = tid; i < c.d; i += NL_TPB) {
      const float dy = sX[i] > 0.f ? sV2[i] : 0.f;
      sV2[i] = dy;
      m1 += dy; m2 += dy * sX[i];
    }
    if (c.pre_act_ln) {
      m1 = block_sum_nl(m1, red) / (float)c.d;
      m2 = block_sum_nl(m2, red) / (float)c.d;
      const float rstd = 1.f / l.ln_std[r];
      for (int i = tid; i < c.d; i += NL_TPB) sV2[i] = (sV2[i] - m1 - sX[i] * m2) * rstd;
    }
    __syncthreads();
    for (int i = tid; i < c.d; i += NL_TPB) g_dt[i] = sV2[i];
    matvec_cols(l.w_g, sV2, sV1, c.d, c.dB, part);               // ds = W_g^T dt
    matvec_cols(l.w_phi, sTh, sU, c.d, c.dB, part);              // u (recomputed)
    for (int j = warp; j < c.L; j += NL_TPB / 32) {              // dp_j = ds . B'_j
      const float4* b4 = reinterpret_cast<const float4*>(B + (int64_t)j * c.dB);
      float acc = 0.f;
      for (int q = lane; q < (c.dB >> 2); q += 32) {
        const float4 a = b4[q];
        const float4 v = *reinterpret_cast<const float4*>(sV1 + 4 * q);
        acc += a.x * v.x + a.y * v.y + a.z * v.z + a.w * v.w;
      }
      acc = warp_sum_f(acc);
      if (lane == 0) sD[j] = acc;
    }
    __syncthreads();
    float dot = 0.f;
    for (int j = tid; j < c.L; j += NL_TPB) dot += sP[j] * sD[j];
    dot = block_sum_nl(dot, red);
    float sds = 0.f;
    for (int j = tid; j < c.L; j += NL_TPB) { const float v = c.scale * sP[j] * (sD[j] - dot); sD[j] = v; sds += v; }
    sds = block_sum_nl(sds, red);                                // sum_j dscore_j (= 0 up to rounding)
    if (tid == 0) g_sum[0] = sds;
    // du = sum_j dscore_j B'_j ; dB'_j (+)= p_j ds + dscore_j u
    colsum_w(B, c.L, c.dB, sD, sV3, part);
    for (int i = tid; i < c.dB; i += NL_TPB) g_du[i] = sV3[i];
    {
      const bool first = li == c.layers - 1;                     // the last layer (first visited) overwrites dB'
      const int c4n = c.dB >> 2;
      float4* dB4 = reinterpret_cast<float4*>(dB);
      for (int64_t e = tid; e < (int64_t)c.L * c4n; e += NL_TPB) {
        const int j = (int)(e / c4n), q = (int)(e - (int64_t)j * c4n);
        const float4 dsv = *reinterpret_cast<const float4*>(sV1 + 4 * q);
        const float4 uv = *reinterpret_cast<const float4*>(sU + 4 * q);
        const float pj = sP[j], dj = sD[j];
        float4 gq = make_float4(pj * dsv.x + dj * uv.x, pj * dsv.y + dj * uv.y, pj * dsv.z + dj * uv.z, pj * dsv.w + dj * uv.w);
        if (!first) { const float4 o = dB4[e]; gq.x += o.x; gq.y += o.y; gq.z += o.z; gq.w += o.w; }
        dB4[e] = gq;
      }
    }
    __syncthreads();
    matvec_rows(l.w_phi, sV3, sV2, nullptr, c.d, c.dB);          // dtheta = W_phi du (+ b_phi sum_j dscore_j)
    __syncthreads();
    for (int i = tid; i < c.d; i += NL_TPB) {
      const float v = sV2[i] + (l.b_phi ? l.b_phi[i] * sds : 0.f);
      sV2[i] = v;
      g_dth[i] = v;
    }
    __syncthreads();
    matvec_cols(l.w_theta, sV2, sV1, c.d, c.dA, part);           // dA += W_theta^T dtheta
    for (int i = tid; i < c.dA; i += NL_TPB) sDA[i] += sV1[i];
    __syncthreads();
  }
  for (int i = tid; i < c.dA; i += NL_TPB) P.da0[(int64_t)r * c.dA + i] = sDA[i];
}

// Weight gradients of all layers: dW[o][i] += sum_r left[r][o] right[r][i]; biases: sum_r left[r][o].
// grid = (row blocks, 4 * layers); which: 0 = out (do x act), 1 = g (dt x s), 2 = phi (theta x du), 3 = theta (dtheta x a_in)
__global__ void __launch_bounds__(256) fbo_nl_outer_k(const NlParams P) {
  const vlfb_fbo_cfg_t& c = P.c;
  const int li = blockIdx.y >> 2, which = blockIdx.y & 3;
  const vlfb_fbo_layer_t& l = P.l[li];
  const int per_roi = c.dA + c.d + c.dB + c.d + 4;
  const int R = c.live_rows != nullptr ? min(c.R, *c.live_rows) : c.R;     // padding rows add nothing
  const float* scr = P.scratch + (int64_t)li * c.R * per_roi;
  const float* left;
  const float* right;
  int rows, cols, lstride, rstride;
  float* gw;
  float* gb;
  const float* a_in = li == 0 ? P.a0 : P.l[li - 1].a_out;
  if (which == 0) { left = scr; lstride = per_roi; right = l.xhat; rstride = c.d; rows = c.dA; cols = c.d; gw = l.gw_out; gb = l.gb_out; }
  else if (which == 1) { left = scr + c.dA; lstride = per_roi; right = l.s; rstride = c.dB; rows = c.d; cols = c.dB; gw = l.gw_g; gb = l.gb_g; }
  else if (which == 2) { left = l.theta; lstride = c.d; right = scr + c.dA + c.d; rstride = per_roi; rows = c.d; cols = c.dB; gw = l.gw_phi; gb = l.gb_phi; }
  else { left = scr + c.dA + c.d + c.dB; lstride = per_roi; right = a_in; rstride = c.dA; rows = c.d; cols = c.dA; gw = l.gw_theta; gb = l.gb_theta; }
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    if (gw) {
      for (int i = threadIdx.x; i < cols; i += blockDim.x) {
        float acc = 0.f;
        for (int r = 0; r < R; ++r) {
          float rv = right[(int64_t)r * rstride + i];
          if (which == 0) rv = fmaxf(rv, 0.f);                   // act = relu(xhat)
          acc += left[(int64_t)r * lstride + row] * rv;
        }
        gw[(int64_t)row * cols + i] += acc;
      }
    }
    if (gb && threadIdx.x == 0) {
      float acc = 0.f;
      for (int r = 0; r < R; ++r) {
        float lv = left[(int64_t)r * lstride + row];
        if (which == 2) lv *= scr[(int64_t)r * per_roi + c.dA + c.d + c.dB + c.d];   // theta_o * sum_j dscore_j
        acc += lv;
      }
      gb[row] += acc;
    }
  }
}

}  // namespace
}  // namespace vlfb

using namespace vlfb;
#define ST(s) static_cast<cudaStream_t>(s)

extern "C" {

/* Rows per tile of the scan kernel for a bank of `D`-element rows stored as `dt` (0 = unsupported). */
static int scan_rows(int D, int dt) {
  if (dt == VLFB_DT_F32) return D == 4096 ? 4 : (D == 1024 || D == 2048) ? 8 : 0;
  if (dt == VLFB_DT_BF16) return D == 4096 ? 4 : D == 2048 ? VLFB_SCAN16_ROWS : 0;
  return 0;
}

/* Split of the L bank rows of every RoI over `S` CTAs: minimise waves x (tiles per CTA + partial-result cost) with
 * 2 resident CTAs per SM (264 per wave on H100). */
int vlfb_fbo_bank_scan_splits_dt(int R, int L, int D, int bank_dtype) {
  const int rows = scan_rows(D, bank_dtype);
  if (R <= 0 || L <= 0 || rows == 0) return 0;
  const int max_s = (L + rows - 1) / rows;
  const int wave = 264;
  int best = 1;
  double best_cost = 1e30;
  for (int s = 1; s <= max_s && s <= 1024; ++s) {
    const int per = (L + s - 1) / s;
    if ((int64_t)(s - 1) * per >= L) continue;                 /* an empty trailing split */
    const int tiles = (per + rows - 1) / rows;
    const double waves = (double)(((int64_t)R * s + wave - 1) / wave);
    const double cost = waves * (tiles + 0.5);
    if (cost < best_cost - 1e-9) { best_cost = cost; best = s; }
  }
  return best;
}
int vlfb_fbo_bank_scan_splits(int R, int L, int D) { return vlfb_fbo_bank_scan_splits_dt(R, L, D, VLFB_DT_F32); }

size_t vlfb_fbo_bank_scan_workspace_dt(int R, int L, int D, int bank_dtype) {
  const int S = vlfb_fbo_bank_scan_splits_dt(R, L, D, bank_dtype);
  if (S <= 0) return 0;
  return ((size_t)R * S * D + (size_t)R * S * 2) * sizeof(float);
}
size_t vlfb_fbo_bank_scan_workspace(int R, int L, int D) { return vlfb_fbo_bank_scan_workspace_dt(R, L, D, VLFB_DT_F32); }

int vlfb_fbo_bank_scan_dt(const void* bank, int bank_dtype, const float* q, float scale, float* out, float* prob, int R,
                          int L, int D, int tf32_out, void* workspace, size_t workspace_bytes, void* stream) {
  return vlfb_fbo_bank_scan_live(bank, bank_dtype, q, scale, out, prob, R, L, D, tf32_out, workspace, workspace_bytes,
                                 nullptr, stream);
}

int vlfb_fbo_bank_scan_live(const void* bank, int bank_dtype, const float* q, float scale, float* out, float* prob, int R,
                            int L, int D, int tf32_out, void* workspace, size_t workspace_bytes, const int32_t* live_rows,
                            void* stream) {
  VLFB_CHECK_ARG(bank && q && out && R >= 0 && L > 0);
  VLFB_CHECK_ARG(bank_dtype == VLFB_DT_F32 || bank_dtype == VLFB_DT_BF16);
  VLFB_CHECK_ARG(scan_rows(D, bank_dtype) > 0);
  VLFB_CHECK_ARG((reinterpret_cast<uintptr_t>(bank) & 15) == 0 && (reinterpret_cast<uintptr_t>(q) & 15) == 0);
  if (R == 0) return VLFB_OK;
  const int S = vlfb_fbo_bank_scan_splits_dt(R, L, D, bank_dtype);
  VLFB_CHECK_ARG(S > 0 && (int64_t)R * S < (1ll << 31));
  const size_t need = vlfb_fbo_bank_scan_workspace_dt(R, L, D, bank_dtype);
  if (workspace == nullptr || workspace_bytes < need) {
    set_error("vlfb_fbo_bank_scan: workspace of %zu bytes needed, %zu given", need, workspace_bytes);
    return VLFB_E_WORKSPACE;
  }
  float* part_acc = static_cast<float*>(workspace);
  float* part_ml = part_acc + (size_t)R * S * D;
  const int per = (L + S - 1) / S;
  const dim3 grid((unsigned)(R * S));
#define VLFB_SCAN(EPL, V, ROWS) \
  launch_k(fbo_bank_scan_k<EPL, V, ROWS>, grid, SCAN_TPB, 0, ST(stream), bank, q, scale, part_acc, part_ml, prob, L, S, per, \
           live_rows)
  if (bank_dtype == VLFB_DT_F32) {
    if (D == 1024) VLFB_SCAN(4, 1, 8);
    else if (D == 2048) VLFB_SCAN(4, 2, 8);
    else VLFB_SCAN(4, 4, 4);
  } else {
    if (D == 2048) VLFB_SCAN(8, 1, VLFB_SCAN16_ROWS);
    else VLFB_SCAN(8, 2, 4);
  }
#undef VLFB_SCAN
  VLFB_CHECK_LAUNCH();
  launch_k(fbo_bank_combine_k, dim3((unsigned)(D / 256), (unsigned)R), 256, 0, ST(stream), (const float*)part_acc,
           (const float*)part_ml, out, prob, S, D, L, tf32_out, live_rows);
  VLFB_CHECK_LAUNCH();
  return VLFB_OK;
}
int vlfb_fbo_bank_scan(const float* bank, const float* q, float scale, float* out, float* prob, int R, int L, int D,
                       int tf32_out, void* workspace, size_t workspace_bytes, void* stream) {
  return vlfb_fbo_bank_scan_dt(bank, VLFB_DT_F32, q, scale, out, prob, R, L, D, tf32_out, workspace, workspace_bytes, stream);
}

int vlfb_cast_f32_to_bf16(const float* x, void* y, int64_t n, void* stream) {
  VLFB_CHECK_ARG(x && y && n >= 0 && (n & 7) == 0);
  VLFB_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0);
  if (n == 0) return VLFB_OK;
  launch_k(f32_to_bf16_k, stream_grid(n / 8, 256), 256, 0, ST(stream), (const float4*)x, (uint4*)y, n / 8);
  VLFB_CHECK_LAUNCH();
  return VLFB_OK;
}

static int nl_validate(const vlfb_fbo_cfg_t* c, const vlfb_fbo_layer_t* layers) {
  VLFB_CHECK_ARG(c && layers);
  VLFB_CHECK_ARG(c->R >= 1 && c->L >= 1 && c->layers >= 1 && c->layers <= NL_MAX_LAYERS);
  VLFB_CHECK_ARG(c->dA >= 4 && c->d >= 4 && c->dB >= 4 && (c->dA & 3) == 0 && (c->d & 3) == 0 && (c->dB & 3) == 0);
  VLFB_CHECK_ARG(c->pre_act == 1 && c->drop_ratio >= 0.f && c->drop_ratio < 1.f);
  for (int i = 0; i < c->layers; ++i) {
    const vlfb_fbo_layer_t& l = layers[i];
    VLFB_CHECK_ARG(l.w_theta && l.w_phi && l.w_g && l.w_out && l.theta && l.prob && l.s && l.t && l.xhat && l.ln_mean &&
                   l.ln_std && l.out && l.a_out);
  }
  return VLFB_OK;
}

static void nl_fill(NlParams& P, const vlfb_fbo_cfg_t* c, const vlfb_fbo_layer_t* layers) {
  memset(&P, 0, sizeof(P));
  P.c = *c;
  for (int i = 0; i < c->layers; ++i) P.l[i] = layers[i];
}

size_t vlfb_fbo_nl_scratch_floats(const vlfb_fbo_cfg_t* c) {
  if (!c || c->R < 1 || c->layers < 1) return 0;
  return (size_t)c->layers * c->R * (size_t)(c->dA + c->d + c->dB + c->d + 4);
}

int vlfb_fbo_nl_fwd(const vlfb_fbo_cfg_t* c, const vlfb_fbo_layer_t* layers, const float* a0, const float* bp,
                    void* stream) {
  const int rc = nl_validate(c, layers);
  if (rc != VLFB_OK) return rc;
  VLFB_CHECK_ARG(a0 && bp);
  NlParams P;
  nl_fill(P, c, layers);
  P.a0 = a0; P.bp = bp;
  const size_t smem = ((size_t)4 * NL_TPB + 2 * c->dA + 3 * c->d + 2 * c->dB + ((c->L + 3) & ~3) + 32) * sizeof(float);
  VLFB_CHECK_ARG(smem <= 200 * 1024);
  static size_t attr = 0;
  if (smem > 48 * 1024 && smem > attr) {
    if (cudaFuncSetAttribute(fbo_nl_fwd_k, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) != cudaSuccess) {
      set_error("fbo_nl_fwd: cudaFuncSetAttribute failed");
      return VLFB_E_CUDA;
    }
    attr = 200 * 1024;
  }
  launch_k(fbo_nl_fwd_k, dim3(c->R), dim3(NL_TPB), smem, ST(stream), P);
  VLFB_CHECK_LAUNCH();
  return VLFB_OK;
}

int vlfb_fbo_nl_bwd(const vlfb_fbo_cfg_t* c, const vlfb_fbo_layer_t* layers, const float* a0, const float* bp,
                    const float* da_last, float* da0, float* dbp, float* scratch, size_t scratch_floats, void* stream) {
  const int rc = nl_validate(c, layers);
  if (rc != VLFB_OK) return rc;
  VLFB_CHECK_ARG(a0 && bp && da_last && da0 && dbp && scratch);
  if (scratch_floats < vlfb_fbo_nl_scratch_floats(c)) {
    set_error("vlfb_fbo_nl_bwd: scratch of %zu floats, %zu needed", scratch_floats, vlfb_fbo_nl_scratch_floats(c));
    return VLFB_E_WORKSPACE;
  }
  NlParams P;
  nl_fill(P, c, layers);
  P.a0 = a0; P.bp = bp; P.da_last = da_last; P.da0 = da0; P.dbp = dbp; P.scratch = scratch;
  const int mx3 = c->dA > c->d ? (c->dA > c->dB ? c->dA : c->dB) : (c->d > c->dB ? c->d : c->dB);
  const size_t smem = ((size_t)4 * NL_TPB + 2 * c->dA + 2 * c->d + 2 * c->dB + 3 * mx3 + 2 * ((c->L + 3) & ~3) + 32) * sizeof(float);
  VLFB_CHECK_ARG(smem <= 200 * 1024);
  static size_t attr = 0;
  if (smem > 48 * 1024 && smem > attr) {
    if (cudaFuncSetAttribute(fbo_nl_bwd_k, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) != cudaSuccess) {
      set_error("fbo_nl_bwd: cudaFuncSetAttribute failed");
      return VLFB_E_CUDA;
    }
    attr = 200 * 1024;
  }
  launch_k(fbo_nl_bwd_k, dim3(c->R), dim3(NL_TPB), smem, ST(stream), P);
  VLFB_CHECK_LAUNCH();
  launch_k(fbo_nl_outer_k, dim3(128, 4 * c->layers), dim3(256), 0, ST(stream), P);
  VLFB_CHECK_LAUNCH();
  return VLFB_OK;
}

int vlfb_lfb_gather(const float* bank, int64_t bank_rows, const int32_t* idx, float* out, int64_t rows, int D,
                    int tf32_out, void* stream) {
  VLFB_CHECK_ARG(rows >= 0 && bank_rows >= 0 && D > 0 && (D & 3) == 0);
  if (rows == 0) return VLFB_OK;            /* an empty table: nothing to write (pointers may be NULL) */
  VLFB_CHECK_ARG(idx && out && (bank || bank_rows == 0));
  launch_k(lfb_gather_k, stream_grid(rows * (D >> 2), 256, 4), 256, 0, ST(stream), (const float4*)bank, idx, (float4*)out,
           rows, D >> 2, bank_rows, tf32_out);
  VLFB_CHECK_LAUNCH();
  return VLFB_OK;
}

}  // extern "C"
