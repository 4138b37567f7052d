// SpatialBN (trainable batch normalisation; SURVEY 8f rank 4) of channels-last activations [rows][C].
// Replaces Caffe2's SpatialBN / SpatialBNGradient as called by the reference (model_builder_video.py:176-197
// Conv3dBN, resnet_video.py:185-188, nonlocal_helper.py:146-155) and produces the `_bn_sm` / `_bn_siv` blobs
// lib/utils/bn_helper.py:170-173 reads for precise-BN.  HBM-bound streaming kernels:
//   training forward  = one reduction pass (per-channel sum / sum of squares about a pivot, fp32 per thread,
//                       fp64 across blocks) + one apply pass y = (x - mean[c]) * fs[c] + b[c]
//   training backward = one reduction pass (sum dy, sum dy * (x - mean)) + one apply pass dx = A dy + B x + C
//   inference         = y = (x - mean) * s / sqrt(var + eps) + b: one apply pass
// Bytes per unit: forward 2 reads + 1 write of the tensor, backward 4 reads + 1 write.
#include "common.cuh"

namespace vlfb {
namespace {

constexpr int TPB = 256;

// MODE 0: s0 = sum (x - pivot), s1 = sum (x - pivot)^2  with pivot[c] = x[0][c]  (a = x, b unused)
// MODE 1: s0 = sum dy,          s1 = sum dy * (x - pivot) with pivot = batch mean (a = dy, b = x)
// block = 32 channels x 8 row lanes over a slab of rows; 4 independent rows in flight per thread.
template <int MODE>
__global__ void bn_reduce_k(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ pivot,
                            int64_t rows, int C, int64_t rows_per_block, double* __restrict__ acc) {
  __shared__ float p0[8][33], p1[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const int64_t r0 = (int64_t)blockIdx.y * rows_per_block;
  const int64_t r1 = min(rows, r0 + rows_per_block);
  float s0 = 0.f, s1 = 0.f;
  if (c < C) {
    const float pv = pivot[c];
    int64_t r = r0 + threadIdx.y;
    for (; r + 24 < r1; r += 32) {
      float u[4], v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        u[j] = a[(r + 8 * j) * C + c];
        if (MODE == 1) v[j] = b[(r + 8 * j) * C + c];
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (MODE == 0) { const float d = u[j] - pv; s0 += d; s1 += d * d; }
        else { s0 += u[j]; s1 += u[j] * (v[j] - pv); }
      }
    }
    for (; r < r1; r += 8) {
      const float u = a[r * C + c];
      if (MODE == 0) { const float d = u - pv; s0 += d; s1 += d * d; }
      else { s0 += u; s1 += u * (b[r * C + c] - pv); }
    }
  }
  p0[threadIdx.y][threadIdx.x] = s0;
  p1[threadIdx.y][threadIdx.x] = s1;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    double t0 = 0.0, t1 = 0.0;
#pragma unroll
    for (int j = 0; j < 8; ++j) { t0 += (double)p0[j][threadIdx.x]; t1 += (double)p1[j][threadIdx.x]; }
    atomicAdd(acc + c, t0);
    atomicAdd(acc + C + c, t1);
  }
}

// Batch statistics -> saved mean / inverse std, running statistics (Caffe2: running = running * momentum +
// batch * (1 - momentum), running variance from the unbiased batch variance), fused scale / bias of the apply pass.
__global__ void bn_finalize_fwd_k(const double* __restrict__ acc, const float* __restrict__ x0, int64_t rows, int C, float eps,
                                  float momentum, const float* __restrict__ scale, const float* __restrict__ bias,
                                  float* __restrict__ run_mean, float* __restrict__ run_var, float* __restrict__ saved_mean,
                                  float* __restrict__ saved_inv_std, float* __restrict__ fs) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double m = (double)rows;
  const double d = acc[c] / m;
  const double mean = (double)x0[c] + d;
  double var = acc[C + c] / m - d * d;
  if (var < 0.0) var = 0.0;
  const double inv_std = 1.0 / sqrt(var + (double)eps);
  saved_mean[c] = (float)mean;
  saved_inv_std[c] = (float)inv_std;
  if (run_mean) {
    const double unbiased = rows > 1 ? var * m / (m - 1.0) : var;
    run_mean[c] = (float)((double)run_mean[c] * momentum + mean * (1.0 - (double)momentum));
    run_var[c] = (float)((double)run_var[c] * momentum + unbiased * (1.0 - (double)momentum));
  }
  fs[c] = (float)((double)scale[c] * inv_std);           // apply pass: y = (x - saved_mean) * fs + bias
}

__global__ void bn_infer_params_k(const float* __restrict__ scale, const float* __restrict__ var, float eps, int C,
                                  float* __restrict__ fs) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) fs[c] = scale[c] / sqrtf(var[c] + eps);
}

// dscale += sum dy * xhat, dbias += sum dy; coefficients of dx = A dy + B x + Cc:
//   dx = (s * inv_std / m) * (m dy - sum dy - xhat * sum dy xhat),  xhat = (x - mean) * inv_std
__global__ void bn_finalize_bwd_k(const double* __restrict__ acc, int64_t rows, int C, const float* __restrict__ scale,
                                  const float* __restrict__ saved_mean, const float* __restrict__ saved_inv_std,
                                  float* __restrict__ dscale, float* __restrict__ dbias, float* __restrict__ cA,
                                  float* __restrict__ cB, float* __restrict__ cC) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double m = (double)rows, s1 = acc[c], s2 = acc[C + c];
  const double is = (double)saved_inv_std[c], mu = (double)saved_mean[c], g = (double)scale[c];
  if (dscale) dscale[c] += (float)(s2 * is);
  if (dbias) dbias[c] += (float)s1;
  const double A = g * is;
  const double B = -g * is * is * is * s2 / m;
  cA[c] = (float)A;
  cB[c] = (float)B;
  cC[c] = (float)(-A * s1 / m - B * mu);
}

// y = (x - m[c]) * s[c] + b[c]  (u == nullptr; m may be nullptr = 0)   or   y = x * s[c] + u * t[c] + b[c]
// (the forward subtracts the mean BEFORE scaling: x * (s inv_std) + (b - mean s inv_std) cancels badly when inv_std is large)
__global__ void bn_apply_k(const float4* __restrict__ x, const float4* __restrict__ m, const float4* __restrict__ s,
                           const float4* __restrict__ u, const float4* __restrict__ t, const float4* __restrict__ b,
                           float4* __restrict__ y, int64_t n4, int c4) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % c4);
    float4 v = x[i];
    const float4 sc = s[c], bi = b[c];
    if (m) {
      const float4 mc = m[c];
      v.x -= mc.x; v.y -= mc.y; v.z -= mc.z; v.w -= mc.w;
    }
    float4 o = make_float4(v.x * sc.x + bi.x, v.y * sc.y + bi.y, v.z * sc.z + bi.z, v.w * sc.w + bi.w);
    if (u) {
      const float4 w = u[i], tc = t[c];
      o.x += w.x * tc.x; o.y += w.y * tc.y; o.z += w.z * tc.z; o.w += w.w * tc.w;
    }
    y[i] = o;
  }
}

struct Ws {
  double* acc;            // [2][C]
  float *f0, *f1, *f2;    // [C] each
};
inline Ws carve(void* workspace, int C) {
  Ws w;
  w.acc = static_cast<double*>(workspace);
  w.f0 = reinterpret_cast<float*>(w.acc + 2 * (size_t)C);
  w.f1 = w.f0 + C;
  w.f2 = w.f1 + C;
  return w;
}
// det: one slab (block) per 32-channel strip, so each accumulator receives a single atomicAdd onto its zero: the sums are
// reproducible bit for bit (the deterministic entry points of include/vlfb_det.h)
inline void reduce_dims(int64_t rows, int C, dim3* grid, int64_t* rpb, bool det = false) {
  const int cb = ceil_div(C, 32);
  int slabs = det ? 1 : (4 * 132 + cb - 1) / cb;            // ~4 blocks of 256 threads per SM
  const int64_t max_slabs = (rows + 127) / 128;
  if (slabs > max_slabs) slabs = (int)max_slabs;
  if (slabs < 1) slabs = 1;
  *rpb = (rows + slabs - 1) / slabs;
  *grid = dim3(cb, slabs);
}

// ---- segmented forms (include/vlfb_seg.h, B200.GPUS_PER_STEP): S segments of seg_rows contiguous rows, statistics per
// (segment, channel).  Each kernel is its unsegmented twin run on blockIdx.z's (or the thread's) segment, with the same
// loops and arithmetic, so S = 1 computes what the twin computes.
// pivot: MODE 0 = x (segment j's pivot row is its first row, pstride = seg_rows * C); MODE 1 = saved_mean [S][C]
// (pstride = C).  acc = [S][2][C].
template <int MODE>
__global__ void bn_seg_reduce_k(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ pivot,
                                int64_t pstride, int64_t seg_rows, int C, int64_t rows_per_block, double* __restrict__ acc) {
  __shared__ float p0[8][33], p1[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const int64_t base = (int64_t)blockIdx.z * seg_rows;
  const int64_t r0 = base + (int64_t)blockIdx.y * rows_per_block;
  const int64_t r1 = min(base + seg_rows, r0 + rows_per_block);
  float s0 = 0.f, s1 = 0.f;
  if (c < C) {
    const float pv = pivot[blockIdx.z * pstride + c];
    int64_t r = r0 + threadIdx.y;
    for (; r + 24 < r1; r += 32) {
      float u[4], v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        u[j] = a[(r + 8 * j) * C + c];
        if (MODE == 1) v[j] = b[(r + 8 * j) * C + c];
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (MODE == 0) { const float d = u[j] - pv; s0 += d; s1 += d * d; }
        else { s0 += u[j]; s1 += u[j] * (v[j] - pv); }
      }
    }
    for (; r < r1; r += 8) {
      const float u = a[r * C + c];
      if (MODE == 0) { const float d = u - pv; s0 += d; s1 += d * d; }
      else { s0 += u; s1 += u * (b[r * C + c] - pv); }
    }
  }
  p0[threadIdx.y][threadIdx.x] = s0;
  p1[threadIdx.y][threadIdx.x] = s1;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    double t0 = 0.0, t1 = 0.0;
#pragma unroll
    for (int j = 0; j < 8; ++j) { t0 += (double)p0[j][threadIdx.x]; t1 += (double)p1[j][threadIdx.x]; }
    double* as = acc + (size_t)blockIdx.z * 2 * C;
    atomicAdd(as + c, t0);
    atomicAdd(as + C + c, t1);
  }
}

// one thread per (segment, channel); only segment 0 updates the running statistics (the reference keeps gpu_0's)
__global__ void bn_seg_finalize_fwd_k(const double* __restrict__ acc, const float* __restrict__ x, int64_t seg_rows, int C,
                                      int S, float eps, float momentum, const float* __restrict__ scale,
                                      float* __restrict__ run_mean, float* __restrict__ run_var,
                                      float* __restrict__ saved_mean, float* __restrict__ saved_inv_std,
                                      float* __restrict__ fs) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= S * C) return;
  const int j = i / C, c = i - j * C;
  const double* as = acc + (size_t)j * 2 * C;
  const double m = (double)seg_rows;
  const double d = as[c] / m;
  const double mean = (double)x[(int64_t)j * seg_rows * C + c] + d;
  double var = as[C + c] / m - d * d;
  if (var < 0.0) var = 0.0;
  const double inv_std = 1.0 / sqrt(var + (double)eps);
  saved_mean[i] = (float)mean;
  saved_inv_std[i] = (float)inv_std;
  if (run_mean && j == 0) {
    const double unbiased = seg_rows > 1 ? var * m / (m - 1.0) : var;
    run_mean[c] = (float)((double)run_mean[c] * momentum + mean * (1.0 - (double)momentum));
    run_var[c] = (float)((double)run_var[c] * momentum + unbiased * (1.0 - (double)momentum));
  }
  fs[i] = (float)((double)scale[c] * inv_std);
}

// one thread per channel: the segments' dscale / dbias terms are added in segment order, as S consecutive unsegmented
// backward passes would add them; the dx coefficients are per (segment, channel)
__global__ void bn_seg_finalize_bwd_k(const double* __restrict__ acc, int64_t seg_rows, int C, int S,
                                      const float* __restrict__ scale, const float* __restrict__ saved_mean,
                                      const float* __restrict__ saved_inv_std, float* __restrict__ dscale,
                                      float* __restrict__ dbias, float* __restrict__ cA, float* __restrict__ cB,
                                      float* __restrict__ cC) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double m = (double)seg_rows, g = (double)scale[c];
  for (int j = 0; j < S; ++j) {
    const int i = j * C + c;
    const double* as = acc + (size_t)j * 2 * C;
    const double s1 = as[c], s2 = as[C + c];
    const double is = (double)saved_inv_std[i], mu = (double)saved_mean[i];
    if (dscale) dscale[c] += (float)(s2 * is);
    if (dbias) dbias[c] += (float)s1;
    const double A = g * is;
    const double B = -g * is * is * is * s2 / m;
    cA[i] = (float)A;
    cB[i] = (float)B;
    cC[i] = (float)(-A * s1 / m - B * mu);
  }
}

// bn_apply_k over segment blockIdx.y: m / s / t are [S][C] (segment rows), b is [C] (b_seg = 0) or [S][C] (b_seg = 1)
__global__ void bn_seg_apply_k(const float4* __restrict__ x, const float4* __restrict__ m, const float4* __restrict__ s,
                               const float4* __restrict__ u, const float4* __restrict__ t, const float4* __restrict__ b,
                               int b_seg, float4* __restrict__ y, int64_t seg_n4, int c4) {
  const int64_t off = (int64_t)blockIdx.y * seg_n4;
  const int po = blockIdx.y * c4;
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < seg_n4; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = off + k;
    const int c = (int)(k % c4);
    float4 v = x[i];
    const float4 sc = s[po + c], bi = b[(b_seg ? po : 0) + c];
    if (m) {
      const float4 mc = m[po + c];
      v.x -= mc.x; v.y -= mc.y; v.z -= mc.z; v.w -= mc.w;
    }
    float4 o = make_float4(v.x * sc.x + bi.x, v.y * sc.y + bi.y, v.z * sc.z + bi.z, v.w * sc.w + bi.w);
    if (u) {
      const float4 w = u[i], tc = t[po + c];
      o.x += w.x * tc.x; o.y += w.y * tc.y; o.z += w.z * tc.z; o.w += w.w * tc.w;
    }
    y[i] = o;
  }
}

inline Ws carve_seg(void* workspace, int C, int S) {
  Ws w;
  w.acc = static_cast<double*>(workspace);
  w.f0 = reinterpret_cast<float*>(w.acc + 2 * (size_t)S * C);
  w.f1 = w.f0 + (size_t)S * C;
  w.f2 = w.f1 + (size_t)S * C;
  return w;
}
// reduce_dims per segment: the default form spreads the unsegmented form's slab count over the segments, slabs never
// straddle a segment; det = one slab per (segment, strip)
inline void seg_reduce_dims(int64_t seg_rows, int C, int S, dim3* grid, int64_t* rpb, bool det) {
  const int cb = ceil_div(C, 32);
  int slabs = det ? 1 : ((4 * 132 + cb - 1) / cb + S - 1) / S;
  const int64_t max_slabs = (seg_rows + 127) / 128;
  if (slabs > max_slabs) slabs = (int)max_slabs;
  if (slabs < 1) slabs = 1;
  *rpb = (seg_rows + slabs - 1) / slabs;
  *grid = dim3(cb, slabs, S);
}
inline dim3 seg_apply_grid(int64_t seg_n4, int S) {
  int gx = (stream_grid(seg_n4 * S, TPB) + S - 1) / S;
  return dim3(gx < 1 ? 1 : gx, S);
}

}  // namespace
}  // namespace vlfb

using namespace vlfb;
#define ST(s) static_cast<cudaStream_t>(s)

extern "C" {

size_t vlfb_spatial_bn_workspace_bytes(int C) { return C > 0 ? (size_t)C * 28 + 32 : 0; }

static int spatial_bn_fwd(const float* x, const float* scale, const float* bias, float* running_mean, float* running_var,
                          float* saved_mean, float* saved_inv_std, float* y, int64_t rows, int C, float eps, float momentum,
                          void* workspace, size_t workspace_bytes, void* stream, bool det) {
  VLFB_CHECK_ARG(x && scale && bias && saved_mean && saved_inv_std && y && rows > 0 && C > 0 && (C & 3) == 0);
  VLFB_CHECK_ARG((running_mean == nullptr) == (running_var == nullptr));
  VLFB_CHECK_ARG(workspace && workspace_bytes >= vlfb_spatial_bn_workspace_bytes(C) &&
                 (reinterpret_cast<uintptr_t>(workspace) & 15) == 0);
  const Ws w = carve(workspace, C);
  if (cudaMemsetAsync(w.acc, 0, 2 * (size_t)C * sizeof(double), ST(stream)) != cudaSuccess) {
    set_error("vlfb_spatial_bn_fwd: cudaMemsetAsync failed");
    return VLFB_E_CUDA;
  }
  dim3 grid;
  int64_t rpb;
  reduce_dims(rows, C, &grid, &rpb, det);
  launch_k(bn_reduce_k<0>, grid, dim3(32, 8), 0, ST(stream), x, (const float*)nullptr, x, rows, C, rpb, w.acc);
  VLFB_CHECK_LAUNCH();
  launch_k(bn_finalize_fwd_k, dim3(ceil_div(C, 128)), dim3(128), 0, ST(stream), (const double*)w.acc, x, rows, C, eps, momentum,
           scale, bias, running_mean, running_var, saved_mean, saved_inv_std, w.f0);
  VLFB_CHECK_LAUNCH();
  const int64_t n4 = rows * (C >> 2);
  launch_k(bn_apply_k, stream_grid(n4, TPB), TPB, 0, ST(stream), (const float4*)x, (const float4*)saved_mean,
           (const float4*)w.f0, (const float4*)nullptr, (const float4*)nullptr, (const float4*)bias, (float4*)y, n4, C >> 2);
  VLFB_CHECK_LAUNCH();
  return VLFB_OK;
}

int vlfb_spatial_bn_infer(const float* x, const float* scale, const float* bias, const float* running_mean,
                          const float* running_var, float* y, int64_t rows, int C, float eps, void* workspace,
                          size_t workspace_bytes, void* stream) {
  VLFB_CHECK_ARG(x && scale && bias && running_mean && running_var && y && rows >= 0 && C > 0 && (C & 3) == 0);
  VLFB_CHECK_ARG(workspace && workspace_bytes >= vlfb_spatial_bn_workspace_bytes(C) &&
                 (reinterpret_cast<uintptr_t>(workspace) & 15) == 0);
  if (rows == 0) return VLFB_OK;
  const Ws w = carve(workspace, C);
  launch_k(bn_infer_params_k, dim3(ceil_div(C, 128)), dim3(128), 0, ST(stream), scale, running_var, eps, C, w.f0);
  VLFB_CHECK_LAUNCH();
  const int64_t n4 = rows * (C >> 2);
  launch_k(bn_apply_k, stream_grid(n4, TPB), TPB, 0, ST(stream), (const float4*)x, (const float4*)running_mean,
           (const float4*)w.f0, (const float4*)nullptr, (const float4*)nullptr, (const float4*)bias, (float4*)y, n4, C >> 2);
  VLFB_CHECK_LAUNCH();
  return VLFB_OK;
}

static int spatial_bn_bwd(const float* dy, const float* x, const float* scale, const float* saved_mean,
                          const float* saved_inv_std, float* dx, float* dscale, float* dbias, int64_t rows, int C,
                          void* workspace, size_t workspace_bytes, void* stream, bool det) {
  VLFB_CHECK_ARG(dy && x && scale && saved_mean && saved_inv_std && dx && rows > 0 && C > 0 && (C & 3) == 0);
  VLFB_CHECK_ARG(workspace && workspace_bytes >= vlfb_spatial_bn_workspace_bytes(C) &&
                 (reinterpret_cast<uintptr_t>(workspace) & 15) == 0);
  const Ws w = carve(workspace, C);
  if (cudaMemsetAsync(w.acc, 0, 2 * (size_t)C * sizeof(double), ST(stream)) != cudaSuccess) {
    set_error("vlfb_spatial_bn_bwd: cudaMemsetAsync failed");
    return VLFB_E_CUDA;
  }
  dim3 grid;
  int64_t rpb;
  reduce_dims(rows, C, &grid, &rpb, det);
  launch_k(bn_reduce_k<1>, grid, dim3(32, 8), 0, ST(stream), dy, x, saved_mean, rows, C, rpb, w.acc);
  VLFB_CHECK_LAUNCH();
  launch_k(bn_finalize_bwd_k, dim3(ceil_div(C, 128)), dim3(128), 0, ST(stream), (const double*)w.acc, rows, C, scale, saved_mean,
           saved_inv_std, dscale, dbias, w.f0, w.f1, w.f2);
  VLFB_CHECK_LAUNCH();
  const int64_t n4 = rows * (C >> 2);
  launch_k(bn_apply_k, stream_grid(n4, TPB), TPB, 0, ST(stream), (const float4*)dy, (const float4*)nullptr,
           (const float4*)w.f0, (const float4*)x, (const float4*)w.f1, (const float4*)w.f2, (float4*)dx, n4, C >> 2);
  VLFB_CHECK_LAUNCH();
  return VLFB_OK;
}

}  // extern "C"

extern "C" {

int vlfb_spatial_bn_fwd(const float* x, const float* scale, const float* bias, float* running_mean, float* running_var,
                        float* saved_mean, float* saved_inv_std, float* y, int64_t rows, int C, float eps, float momentum,
                        void* workspace, size_t workspace_bytes, void* stream) {
  return spatial_bn_fwd(x, scale, bias, running_mean, running_var, saved_mean, saved_inv_std, y, rows, C, eps, momentum,
                        workspace, workspace_bytes, stream, false);
}

int vlfb_spatial_bn_bwd(const float* dy, const float* x, const float* scale, const float* saved_mean,
                        const float* saved_inv_std, float* dx, float* dscale, float* dbias, int64_t rows, int C,
                        void* workspace, size_t workspace_bytes, void* stream) {
  return spatial_bn_bwd(dy, x, scale, saved_mean, saved_inv_std, dx, dscale, dbias, rows, C, workspace, workspace_bytes,
                        stream, false);
}

int vlfb_spatial_bn_fwd_det(const float* x, const float* scale, const float* bias, float* running_mean, float* running_var,
                            float* saved_mean, float* saved_inv_std, float* y, int64_t rows, int C, float eps,
                            float momentum, void* workspace, size_t workspace_bytes, void* stream) {
  return spatial_bn_fwd(x, scale, bias, running_mean, running_var, saved_mean, saved_inv_std, y, rows, C, eps, momentum,
                        workspace, workspace_bytes, stream, true);
}

int vlfb_spatial_bn_bwd_det(const float* dy, const float* x, const float* scale, const float* saved_mean,
                            const float* saved_inv_std, float* dx, float* dscale, float* dbias, int64_t rows, int C,
                            void* workspace, size_t workspace_bytes, void* stream) {
  return spatial_bn_bwd(dy, x, scale, saved_mean, saved_inv_std, dx, dscale, dbias, rows, C, workspace, workspace_bytes,
                        stream, true);
}

}  // extern "C"

// ---- segmented forms (include/vlfb_seg.h)
static int spatial_bn_seg_fwd(const float* x, const float* scale, const float* bias, float* running_mean,
                              float* running_var, float* saved_mean, float* saved_inv_std, float* y, int64_t rows, int C,
                              int S, float eps, float momentum, void* workspace, size_t workspace_bytes, void* stream,
                              bool det) {
  VLFB_CHECK_ARG(x && scale && bias && saved_mean && saved_inv_std && y && rows > 0 && C > 0 && (C & 3) == 0);
  VLFB_CHECK_ARG(S > 0 && S <= 65535 && rows % S == 0);
  VLFB_CHECK_ARG((running_mean == nullptr) == (running_var == nullptr));
  VLFB_CHECK_ARG(workspace && workspace_bytes >= vlfb_spatial_bn_seg_workspace_bytes(C, S) &&
                 (reinterpret_cast<uintptr_t>(workspace) & 15) == 0);
  const Ws w = carve_seg(workspace, C, S);
  const int64_t seg_rows = rows / S;
  if (cudaMemsetAsync(w.acc, 0, 2 * (size_t)S * C * sizeof(double), ST(stream)) != cudaSuccess) {
    set_error("vlfb_spatial_bn_seg_fwd: cudaMemsetAsync failed");
    return VLFB_E_CUDA;
  }
  dim3 grid;
  int64_t rpb;
  seg_reduce_dims(seg_rows, C, S, &grid, &rpb, det);
  launch_k(bn_seg_reduce_k<0>, grid, dim3(32, 8), 0, ST(stream), x, (const float*)nullptr, x, seg_rows * C, seg_rows, C,
           rpb, w.acc);
  VLFB_CHECK_LAUNCH();
  launch_k(bn_seg_finalize_fwd_k, dim3(ceil_div(S * C, 128)), dim3(128), 0, ST(stream), (const double*)w.acc, x, seg_rows,
           C, S, eps, momentum, scale, running_mean, running_var, saved_mean, saved_inv_std, w.f0);
  VLFB_CHECK_LAUNCH();
  const int64_t seg_n4 = seg_rows * (C >> 2);
  launch_k(bn_seg_apply_k, seg_apply_grid(seg_n4, S), TPB, 0, ST(stream), (const float4*)x, (const float4*)saved_mean,
           (const float4*)w.f0, (const float4*)nullptr, (const float4*)nullptr, (const float4*)bias, 0, (float4*)y, seg_n4,
           C >> 2);
  VLFB_CHECK_LAUNCH();
  return VLFB_OK;
}

static int spatial_bn_seg_bwd(const float* dy, const float* x, const float* scale, const float* saved_mean,
                              const float* saved_inv_std, float* dx, float* dscale, float* dbias, int64_t rows, int C, int S,
                              void* workspace, size_t workspace_bytes, void* stream, bool det) {
  VLFB_CHECK_ARG(dy && x && scale && saved_mean && saved_inv_std && dx && rows > 0 && C > 0 && (C & 3) == 0);
  VLFB_CHECK_ARG(S > 0 && S <= 65535 && rows % S == 0);
  VLFB_CHECK_ARG(workspace && workspace_bytes >= vlfb_spatial_bn_seg_workspace_bytes(C, S) &&
                 (reinterpret_cast<uintptr_t>(workspace) & 15) == 0);
  const Ws w = carve_seg(workspace, C, S);
  const int64_t seg_rows = rows / S;
  if (cudaMemsetAsync(w.acc, 0, 2 * (size_t)S * C * sizeof(double), ST(stream)) != cudaSuccess) {
    set_error("vlfb_spatial_bn_seg_bwd: cudaMemsetAsync failed");
    return VLFB_E_CUDA;
  }
  dim3 grid;
  int64_t rpb;
  seg_reduce_dims(seg_rows, C, S, &grid, &rpb, det);
  launch_k(bn_seg_reduce_k<1>, grid, dim3(32, 8), 0, ST(stream), dy, x, saved_mean, (int64_t)C, seg_rows, C, rpb, w.acc);
  VLFB_CHECK_LAUNCH();
  launch_k(bn_seg_finalize_bwd_k, dim3(ceil_div(C, 128)), dim3(128), 0, ST(stream), (const double*)w.acc, seg_rows, C, S,
           scale, saved_mean, saved_inv_std, dscale, dbias, w.f0, w.f1, w.f2);
  VLFB_CHECK_LAUNCH();
  const int64_t seg_n4 = seg_rows * (C >> 2);
  launch_k(bn_seg_apply_k, seg_apply_grid(seg_n4, S), TPB, 0, ST(stream), (const float4*)dy, (const float4*)nullptr,
           (const float4*)w.f0, (const float4*)x, (const float4*)w.f1, (const float4*)w.f2, 1, (float4*)dx, seg_n4, C >> 2);
  VLFB_CHECK_LAUNCH();
  return VLFB_OK;
}

extern "C" {

size_t vlfb_spatial_bn_seg_workspace_bytes(int C, int S) {
  return (C > 0 && S > 0) ? (size_t)S * C * 28 + 32 : 0;
}

int vlfb_spatial_bn_seg_fwd(const float* x, const float* scale, const float* bias, float* running_mean,
                            float* running_var, float* saved_mean, float* saved_inv_std, float* y, int64_t rows, int C,
                            int S, float eps, float momentum, void* workspace, size_t workspace_bytes, void* stream) {
  return spatial_bn_seg_fwd(x, scale, bias, running_mean, running_var, saved_mean, saved_inv_std, y, rows, C, S, eps,
                            momentum, workspace, workspace_bytes, stream, false);
}

int vlfb_spatial_bn_seg_bwd(const float* dy, const float* x, const float* scale, const float* saved_mean,
                            const float* saved_inv_std, float* dx, float* dscale, float* dbias, int64_t rows, int C,
                            int S, void* workspace, size_t workspace_bytes, void* stream) {
  return spatial_bn_seg_bwd(dy, x, scale, saved_mean, saved_inv_std, dx, dscale, dbias, rows, C, S, workspace,
                            workspace_bytes, stream, false);
}

int vlfb_spatial_bn_seg_fwd_det(const float* x, const float* scale, const float* bias, float* running_mean,
                                float* running_var, float* saved_mean, float* saved_inv_std, float* y, int64_t rows,
                                int C, int S, float eps, float momentum, void* workspace, size_t workspace_bytes,
                                void* stream) {
  return spatial_bn_seg_fwd(x, scale, bias, running_mean, running_var, saved_mean, saved_inv_std, y, rows, C, S, eps,
                            momentum, workspace, workspace_bytes, stream, true);
}

int vlfb_spatial_bn_seg_bwd_det(const float* dy, const float* x, const float* scale, const float* saved_mean,
                                const float* saved_inv_std, float* dx, float* dscale, float* dbias, int64_t rows, int C,
                                int S, void* workspace, size_t workspace_bytes, void* stream) {
  return spatial_bn_seg_bwd(dy, x, scale, saved_mean, saved_inv_std, dx, dscale, dbias, rows, C, S, workspace,
                            workspace_bytes, stream, true);
}

}  // extern "C"
