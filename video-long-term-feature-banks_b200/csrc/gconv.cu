// Grouped 3-D convolution (Caffe2 Conv with group > 1: the ResNeXt branch2b conv) on CUDA cores, sm_90a.
//
// vlfb_gemm routes here when vlfb_gemm_params_t.groups > 1 (include/vlfb.h documents the three forms).  Per-group
// widths are 4..64 channels, far below the 128 x 32 tiles of the tensor-core GEMM, so the work runs as fp32 FMAs on
// operands that are already TF32-rounded: products of TF32 values are exact in fp32, so the result is the tensor-core
// path's definition up to summation order (DESIGN.md 4.4).
//
//   fwd / dgrad  gconv_kernel<DGRAD>: a CTA owns 64 output pixels x 64 output channels.  The CTA's weights of a chunk
//                of taps sit in shared memory as [tap][r][co] (r = reduction channel of the group); each thread keeps
//                4 pixels x 4 channels in registers, reads its input channels as float4 and stores float4.  dgrad
//                gathers dy through a per-tap stride-parity test, with dilation.  Deterministic.
//   wgrad        gconv_wgrad_kernel: a thread owns 4 output channels x 4 (tap, 4 input channels) pairs of dw, one CTA
//                a range of output positions; the partial sums go to dw with red.global.add.f32.
#include <stdlib.h>

#include <algorithm>

#include "common.cuh"

namespace vlfb {

namespace {

constexpr int GC_THREADS = 256;
constexpr int GC_QUADS = 16;                       // output-channel quads per CTA (64 channels)
constexpr int GC_CB = 4 * GC_QUADS;
constexpr int GC_PPT = 4;                          // pixels per thread
constexpr int GC_TILE_P = (GC_THREADS / GC_QUADS) * GC_PPT;   // 64 output pixels per CTA
constexpr int GC_WS_LD = GC_CB + 4;                // shared row pitch: the transposing stores hit 8 banks, not 1
constexpr int GC_SMEM_FLOATS = 12288;              // 48 KB of weights per tap chunk
constexpr int GW_PAIRS = 4;                        // wgrad: (tap, 4 input channels) pairs per thread

struct GconvGeom {
  int Ts, Hs, Ws, Cs;      // gathered source tensor: x (fwd) or dy (dgrad)
  int Td, Hd, Wd, Cd;      // destination = the GEMM's D: y (fwd) or dx (dgrad)
  int kT, kH, kW, sT, sH, sW, pT, pH, pW, dT, dH, dW;
  int R;                   // reduction channels per tap (Cig fwd, Cog dgrad)
  int outg;                // destination channels per group (Cog fwd, Cig dgrad)
  int taps, tchunk;
  int M;                   // destination pixels
};

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// q = a / s for a >= 0; false when s does not divide a.  Strides 1 and 2 (every ResNeXt conv) avoid the integer
// division, which would otherwise cost more than the FMAs of a narrow group.
__device__ __forceinline__ bool div_stride(int a, int s, int& q) {
  if (s == 1) { q = a; return true; }
  if (s == 2) { q = a >> 1; return (a & 1) == 0; }
  q = a / s;
  return a % s == 0;
}

template <bool DGRAD>
__global__ void __launch_bounds__(GC_THREADS, 2) gconv_kernel(const vlfb_gemm_params_t p, const GconvGeom g) {
  __shared__ __align__(16) float ws[GC_SMEM_FLOATS];
  const int tid = threadIdx.x;
  const int q = tid % GC_QUADS, pl = tid / GC_QUADS;
  const int cb = blockIdx.y * GC_CB;
  const int co = cb + 4 * q;                                   // first of the thread's 4 destination channels
  const bool co_ok = co < g.Cd;
  const int cbase = (co / g.outg) * g.R;                       // first source channel of its group
  const int64_t m0 = (int64_t)blockIdx.x * GC_TILE_P;
  const float* src = p.a.ptr;
  const float* wgt = p.b.ptr;

  int pn[GC_PPT], pt[GC_PPT], ph[GC_PPT], pw[GC_PPT];
#pragma unroll
  for (int i = 0; i < GC_PPT; ++i) {
    int64_t m = m0 + pl + (GC_THREADS / GC_QUADS) * i;
    if (m < g.M) {
      pw[i] = (int)(m % g.Wd); m /= g.Wd;
      ph[i] = (int)(m % g.Hd); m /= g.Hd;
      pt[i] = (int)(m % g.Td);
      pn[i] = (int)(m / g.Td);
    } else {
      pn[i] = -1; pt[i] = ph[i] = pw[i] = 0;
    }
  }
  float acc[GC_PPT][4];
#pragma unroll
  for (int i = 0; i < GC_PPT; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int t0 = 0; t0 < g.taps; t0 += g.tchunk) {
    const int tc = min(g.tchunk, g.taps - t0);
    const int span = tc * g.R;
    __syncthreads();                                           // the previous chunk's readers are done
    for (int idx = tid; idx < span * GC_CB; idx += GC_THREADS) {
      const int kk = idx % span, cl = idx / span;
      ws[kk * GC_WS_LD + cl] = (cb + cl < g.Cd) ? __ldg(wgt + (int64_t)(cb + cl) * p.b.ld + t0 * g.R + kk) : 0.f;
    }
    __syncthreads();
    for (int tl = 0; tl < tc; ++tl) {
      int kt, kh, kw;
      decode_tap(t0 + tl, g.kH, g.kW, kt, kh, kw);
      int off[GC_PPT];
      bool any = false;
#pragma unroll
      for (int i = 0; i < GC_PPT; ++i) {
        int ts, hs, wsx;
        bool ok = pn[i] >= 0;
        if (DGRAD) {           // dy position o with o*s - p + k*d == i: the stride parity decides whether the tap hits
          const int a = pt[i] + g.pT - kt * g.dT, b = ph[i] + g.pH - kh * g.dH, c = pw[i] + g.pW - kw * g.dW;
          ok = ok && a >= 0 && b >= 0 && c >= 0;
          ok = div_stride(a, g.sT, ts) && ok;
          ok = div_stride(b, g.sH, hs) && ok;
          ok = div_stride(c, g.sW, wsx) && ok;
        } else {
          ts = pt[i] * g.sT - g.pT + kt * g.dT;
          hs = ph[i] * g.sH - g.pH + kh * g.dH;
          wsx = pw[i] * g.sW - g.pW + kw * g.dW;
          ok = ok && ts >= 0 && hs >= 0 && wsx >= 0;
        }
        ok = ok && ts < g.Ts && hs < g.Hs && wsx < g.Ws;
        off[i] = ok ? (((pn[i] * g.Ts + ts) * g.Hs + hs) * g.Ws + wsx) * g.Cs + cbase : -1;
        any = any || ok;
      }
      if (!any || !co_ok) continue;
      const float* wrow = ws + tl * g.R * GC_WS_LD + 4 * q;
      for (int r = 0; r < g.R; r += 4) {
        float4 xv[GC_PPT];
#pragma unroll
        for (int i = 0; i < GC_PPT; ++i) xv[i] = off[i] >= 0 ? ldg4(src + off[i] + r) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float4 w0 = *reinterpret_cast<const float4*>(wrow + (r + 0) * GC_WS_LD);
        const float4 w1 = *reinterpret_cast<const float4*>(wrow + (r + 1) * GC_WS_LD);
        const float4 w2 = *reinterpret_cast<const float4*>(wrow + (r + 2) * GC_WS_LD);
        const float4 w3 = *reinterpret_cast<const float4*>(wrow + (r + 3) * GC_WS_LD);
#pragma unroll
        for (int i = 0; i < GC_PPT; ++i) {
          acc[i][0] = fmaf(xv[i].x, w0.x, acc[i][0]); acc[i][1] = fmaf(xv[i].x, w0.y, acc[i][1]);
          acc[i][2] = fmaf(xv[i].x, w0.z, acc[i][2]); acc[i][3] = fmaf(xv[i].x, w0.w, acc[i][3]);
          acc[i][0] = fmaf(xv[i].y, w1.x, acc[i][0]); acc[i][1] = fmaf(xv[i].y, w1.y, acc[i][1]);
          acc[i][2] = fmaf(xv[i].y, w1.z, acc[i][2]); acc[i][3] = fmaf(xv[i].y, w1.w, acc[i][3]);
          acc[i][0] = fmaf(xv[i].z, w2.x, acc[i][0]); acc[i][1] = fmaf(xv[i].z, w2.y, acc[i][1]);
          acc[i][2] = fmaf(xv[i].z, w2.z, acc[i][2]); acc[i][3] = fmaf(xv[i].z, w2.w, acc[i][3]);
          acc[i][0] = fmaf(xv[i].w, w3.x, acc[i][0]); acc[i][1] = fmaf(xv[i].w, w3.y, acc[i][1]);
          acc[i][2] = fmaf(xv[i].w, w3.z, acc[i][2]); acc[i][3] = fmaf(xv[i].w, w3.w, acc[i][3]);
        }
      }
    }
  }

  // epilogue, in the order of epilogue_store (common.cuh), on float4s
  float4 cs = make_float4(1.f, 1.f, 1.f, 1.f), bb = make_float4(0.f, 0.f, 0.f, 0.f);
  if (co_ok && p.col_scale) cs = ldg4(p.col_scale + co);
  if (co_ok && p.col_bias) bb = ldg4(p.col_bias + co);
  const int lane = tid & 31;
#pragma unroll
  for (int i = 0; i < GC_PPT; ++i) {
    const int64_t m = m0 + pl + (GC_THREADS / GC_QUADS) * i;
    const bool ok = co_ok && pn[i] >= 0;
    const int64_t o = m * p.ldd + co;
    float v[4] = {acc[i][0], acc[i][1], acc[i][2], acc[i][3]};
    uint32_t bits = 0;
    if (ok) {
      const float rs = p.row_scale ? __ldg(p.row_scale + m) : 1.f;
      const float c4[4] = {cs.x, cs.y, cs.z, cs.w}, b4[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        v[j] *= p.alpha;
        if (p.col_scale) v[j] *= c4[j];
        if (p.col_bias) v[j] += b4[j];
        v[j] *= rs;
      }
      if (p.residual) {
        const float4 r = ldg4(p.residual + o);
        v[0] += r.x; v[1] += r.y; v[2] += r.z; v[3] += r.w;
      }
      if (p.flags & VLFB_EPI_ACCUM) {
        const float4 r = *reinterpret_cast<const float4*>(p.d + o);
        v[0] += r.x; v[1] += r.y; v[2] += r.z; v[3] += r.w;
      }
      if (p.flags & VLFB_EPI_RELU)
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = fmaxf(v[j], 0.f);
      if (p.relu_mask) {
        const float4 r = ldg4(p.relu_mask + o);
        if (!(r.x > 0.f)) v[0] = 0.f;
        if (!(r.y > 0.f)) v[1] = 0.f;
        if (!(r.z > 0.f)) v[2] = 0.f;
        if (!(r.w > 0.f)) v[3] = 0.f;
      }
      if (p.relu_mask_bits) {
        const uint32_t w = __ldg(p.relu_mask_bits + (o >> 5)) >> (o & 31);   // o % 4 == 0: 4 bits of one word
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (!((w >> j) & 1u)) v[j] = 0.f;
      }
      if (p.flags & VLFB_EPI_TF32)
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = round_tf32(v[j]);
      *reinterpret_cast<float4*>(p.d + o) = make_float4(v[0], v[1], v[2], v[3]);
#pragma unroll
      for (int j = 0; j < 4; ++j) bits |= (v[j] > 0.f ? 1u : 0u) << j;
    }
    if (p.relu_bits_out) {
      // 8 neighbouring lanes hold 32 consecutive elements of one row (cb % 64 == 0, ldd == N, N % 32 == 0)
      bits <<= 4 * (lane & 7);
      bits |= __shfl_xor_sync(0xffffffffu, bits, 1);
      bits |= __shfl_xor_sync(0xffffffffu, bits, 2);
      bits |= __shfl_xor_sync(0xffffffffu, bits, 4);
      if (ok && (lane & 7) == 0) p.relu_bits_out[o >> 5] = bits;
    }
  }
}

struct GwGeom {
  int T, H, W, C, To, Ho, Wo, Co;
  int kT, kH, kW, sT, sH, sW, pT, pH, pW, dT, dH, dW;
  int Cig, Cog;
  int pairs;               // taps * Cig / 4
  int units;               // (Co / 4) * ceil(pairs / GW_PAIRS)
  int per_cta;             // output positions per CTA
  int K;                   // output positions
  float* part;             // deterministic form: [CTA column][kT][Co][N] partial dw slabs, or nullptr (red.global.add)
};

__global__ void __launch_bounds__(GC_THREADS, 2) gconv_wgrad_kernel(const vlfb_gemm_params_t p, const GwGeom g) {
  const int u = blockIdx.y * blockDim.x + threadIdx.x;
  if (u >= g.units) return;
  const int nq = g.Co / 4;
  const int co = 4 * (u % nq), jb = u / nq;
  const int cx = (co / g.Cog) * g.Cig;                         // first input channel of the group
  const int cq = g.Cig / 4;
  int dt[GW_PAIRS], dh[GW_PAIRS], dw[GW_PAIRS], ci[GW_PAIRS];
  bool pv[GW_PAIRS];
#pragma unroll
  for (int s = 0; s < GW_PAIRS; ++s) {
    const int j = jb * GW_PAIRS + s;
    pv[s] = j < g.pairs;
    const int tap = pv[s] ? j / cq : 0;
    ci[s] = pv[s] ? (j % cq) * 4 : 0;
    int kt, kh, kw;
    decode_tap(tap, g.kH, g.kW, kt, kh, kw);
    dt[s] = kt * g.dT - g.pT; dh[s] = kh * g.dH - g.pH; dw[s] = kw * g.dW - g.pW;
  }
  float acc[GW_PAIRS][4][4];
#pragma unroll
  for (int s = 0; s < GW_PAIRS; ++s)
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) acc[s][a][b] = 0.f;

  const int k0 = blockIdx.x * g.per_cta, k1 = min(g.K, k0 + g.per_cta);
  int ow = k0 % g.Wo, r = k0 / g.Wo;
  int oh = r % g.Ho;
  r /= g.Ho;
  int ot = r % g.To, on = r / g.To;
  const float* dy = p.a.ptr;
  const float* x = p.b.ptr;
  for (int k = k0; k < k1; ++k) {
    const float4 d4 = ldg4(dy + (int64_t)k * p.a.ld + co);
    const float dv[4] = {d4.x, d4.y, d4.z, d4.w};
    const int tb = ot * g.sT, hb = oh * g.sH, wb = ow * g.sW;
#pragma unroll
    for (int s = 0; s < GW_PAIRS; ++s) {
      const int ti = tb + dt[s], hi = hb + dh[s], wi = wb + dw[s];
      if (!pv[s] || ti < 0 || ti >= g.T || hi < 0 || hi >= g.H || wi < 0 || wi >= g.W) continue;
      const float4 x4 = ldg4(x + ((((int64_t)on * g.T + ti) * g.H + hi) * g.W + wi) * g.C + cx + ci[s]);
      const float xv[4] = {x4.x, x4.y, x4.z, x4.w};
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[s][a][b] = fmaf(dv[a], xv[b], acc[s][a][b]);
    }
    if (++ow == g.Wo) {
      ow = 0;
      if (++oh == g.Ho) {
        oh = 0;
        if (++ot == g.To) { ot = 0; ++on; }
      }
    }
  }
  if (k0 >= k1) return;
#pragma unroll
  for (int s = 0; s < GW_PAIRS; ++s) {
    if (!pv[s]) continue;
    const int j = jb * GW_PAIRS + s;
    const int tap = j / cq;
    const int kt = tap / (g.kH * g.kW), hw = tap % (g.kH * g.kW);
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const float rs = p.row_scale ? __ldg(p.row_scale + co + a) : 1.f;
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const int n = hw * g.Cig + ci[s] + b;                  // GEMM column: (kh, kw, ci)
        float v = acc[s][a][b] * p.alpha;
        if (p.col_scale) v *= __ldg(p.col_scale + n);
        v *= rs;
        if (g.part) {
          g.part[(((int64_t)blockIdx.x * g.kT + kt) * g.Co + co + a) * p.N + n] = v;
          continue;
        }
        float* dst = p.d + (int64_t)kt * p.d_tap_stride + (int64_t)(co + a) * p.ldd + n;
        asm volatile("red.global.add.f32 [%0], %1;" ::"l"(dst), "f"(v) : "memory");
      }
    }
  }
}

// deterministic grouped wgrad, second pass: dw[kt][co][n] += sum of the `splits` partial slabs in split order
__global__ void gconv_wgrad_sum_k(const vlfb_gemm_params_t p, const float* __restrict__ part, int kT, int splits) {
  const int64_t slab = (int64_t)kT * p.M * p.N;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < slab; e += (int64_t)gridDim.x * blockDim.x) {
    float v = 0.f;
    for (int s = 0; s < splits; ++s) v += part[s * slab + e];
    const int n = (int)(e % p.N);
    const int64_t r = e / p.N;
    const int co = (int)(r % p.M), kt = (int)(r / p.M);
    p.d[(int64_t)kt * p.d_tap_stride + (int64_t)co * p.ldd + n] += v;
  }
}

bool debug_on() {
  static const int on = [] { const char* e = getenv("VLFB_DEBUG"); return e ? atoi(e) : 0; }();
  return on != 0;
}

}  // namespace

int gconv(const vlfb_gemm_params_t& p, cudaStream_t stream) {
  const vlfb_conv_geom_t& c = p.g;
  const int G = p.groups, Cig = c.C / G, Cog = c.Co / G;
  const bool dgrad = p.a.kind == VLFB_OP_DGRAD_K, wgrad = p.a.kind == VLFB_OP_DENSE_MN;
  dim3 grid;
  unsigned slabs = 0;                  // deterministic grouped wgrad: partial dw slabs summed by gconv_wgrad_sum_k
  if (wgrad) {
    GwGeom w;
    w.T = c.T; w.H = c.H; w.W = c.W; w.C = c.C; w.To = c.To; w.Ho = c.Ho; w.Wo = c.Wo; w.Co = c.Co;
    w.kT = c.kT; w.kH = c.kH; w.kW = c.kW; w.sT = c.sT; w.sH = c.sH; w.sW = c.sW;
    w.pT = c.pT; w.pH = c.pH; w.pW = c.pW; w.dT = c.dT; w.dH = c.dH; w.dW = c.dW;
    w.Cig = Cig; w.Cog = Cog;
    w.pairs = c.kT * c.kH * c.kW * Cig / 4;
    w.units = (c.Co / 4) * ceil_div(w.pairs, GW_PAIRS);
    w.K = p.K;
    const int block = w.units < GC_THREADS ? (w.units + 31) / 32 * 32 : GC_THREADS;
    const int gy = ceil_div(w.units, block);
    // Positions are split until about 4 CTAs' worth of threads per SM are in flight (fewer splits = fewer atomics),
    // with at least 32 positions per CTA.  gy <= 65535 holds for every valid shape (Co <= 2^31 / positions).
    const int64_t want = (132LL * 4 * GC_THREADS) / ((int64_t)gy * block);
    int64_t splits = std::max<int64_t>(1, std::min<int64_t>(want, ceil_div(w.K, 32)));
    // deterministic: the partial slabs live in the partial-tile area of the GEMM workspace (api.cu checked its size);
    // as many splits as slabs fit there, and one split writes dw directly
    const int64_t slab = (int64_t)c.kT * p.M * p.N;
    float* part = nullptr;
    size_t part_floats = 0;
    if (p.deterministic) {
      part = gemm_tc_partials(p.workspace, p.workspace_bytes, &part_floats);
      splits = std::min<int64_t>(splits, (int64_t)(part_floats / (size_t)slab));
      if (splits < 2) { splits = 1; part = nullptr; }
    }
    w.per_cta = ceil_div(w.K, splits);
    w.part = part;
    grid = dim3(ceil_div(w.K, w.per_cta), gy, 1);
    if (gy > 65535) {
      set_error("vlfb_gemm: grouped wgrad with %d output-channel units needs more than 65535 CTA rows", w.units);
      return VLFB_E_UNSUPPORTED;
    }
    launch_k(gconv_wgrad_kernel, grid, block, 0, stream, p, w);
    if (part) {
      slabs = grid.x;
      VLFB_CHECK_LAUNCH();
      launch_k(gconv_wgrad_sum_k, dim3((unsigned)std::min<int64_t>(ceil_div(slab, 256), 132 * 8)), 256, 0, stream, p,
               (const float*)part, c.kT, (int)grid.x);
    }
  } else {
    GconvGeom g;
    if (dgrad) {
      g.Ts = c.To; g.Hs = c.Ho; g.Ws = c.Wo; g.Cs = c.Co;
      g.Td = c.T; g.Hd = c.H; g.Wd = c.W; g.Cd = c.C;
      g.R = Cog; g.outg = Cig;
    } else {
      g.Ts = c.T; g.Hs = c.H; g.Ws = c.W; g.Cs = c.C;
      g.Td = c.To; g.Hd = c.Ho; g.Wd = c.Wo; g.Cd = c.Co;
      g.R = Cig; g.outg = Cog;
    }
    g.kT = c.kT; g.kH = c.kH; g.kW = c.kW; g.sT = c.sT; g.sH = c.sH; g.sW = c.sW;
    g.pT = c.pT; g.pH = c.pH; g.pW = c.pW; g.dT = c.dT; g.dH = c.dH; g.dW = c.dW;
    g.taps = c.kT * c.kH * c.kW;
    g.tchunk = std::max(1, std::min(g.taps, GC_SMEM_FLOATS / (g.R * GC_WS_LD)));
    g.M = p.M;
    grid = dim3(ceil_div(p.M, GC_TILE_P), ceil_div(g.Cd, GC_CB), 1);
    if (dgrad) launch_k(gconv_kernel<true>, grid, GC_THREADS, 0, stream, p, g);
    else launch_k(gconv_kernel<false>, grid, GC_THREADS, 0, stream, p, g);
  }
  // VLFB_DEBUG: one record per launch, space-separated key=value like gemm_tc's (tests/gconv_cases.py parses it)
  if (debug_on())
    fprintf(stderr, "vlfb gconv: path=gconv dir=%s groups=%d cig=%d cog=%d M=%d N=%d K=%d grid=%u,%u,%u det=%d slabs=%u\n",
            wgrad ? "wgrad" : (dgrad ? "dgrad" : "fwd"), G, Cig, Cog, p.M, p.N, p.K, grid.x, grid.y, grid.z,
            p.deterministic ? 1 : 0, slabs);
  VLFB_CHECK_LAUNCH();
  return VLFB_OK;
}

}  // namespace vlfb
