// Probe of the TMA im2col mode (cuTensorMapEncodeIm2col + cp.async.bulk.tensor.5d...im2col) on sm_90a: which pixel
// lands in which shared-memory row for given tensor coordinates / filter offsets / traversal strides.  The
// tensor holds value n*1000 + d*100 + h*10 + w (+ c/100), so every row of the dump names its source pixel.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -o diag_im2col scripts/diag_im2col.cu -lcuda
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

__global__ void probe(const __grid_constant__ CUtensorMap tm, int c, int w, int h, int d, int n, int ow, int oh, int od,
                      int pixels, int chans, float* out) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ __align__(8) uint64_t bar;
  uint32_t sbase = (uint32_t)__cvta_generic_to_shared(smem);
  sbase = (sbase + 1023u) & ~1023u;
  uint32_t bar_a = (uint32_t)__cvta_generic_to_shared(&bar);
  float* sm = reinterpret_cast<float*>(smem + (sbase - (uint32_t)__cvta_generic_to_shared(smem)));
  for (int i = threadIdx.x; i < pixels * 32; i += blockDim.x) sm[i] = -7.f;
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  asm volatile("fence.proxy.async;" ::: "memory");
  if (threadIdx.x == 0) {
    uint32_t bytes = (uint32_t)pixels * chans * 4;
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bytes) : "memory");
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7], {%8, %9, %10};"
        ::"r"(sbase), "l"(reinterpret_cast<uint64_t>(&tm)), "r"(c), "r"(w), "r"(h), "r"(d), "r"(n), "r"(bar_a),
          "h"((uint16_t)ow), "h"((uint16_t)oh), "h"((uint16_t)od)
        : "memory");
  }
  // bounded wait
  uint32_t done = 0;
  for (long it = 0; it < 20000000 && !done; ++it)
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(bar_a) : "memory");
  __syncthreads();
  for (int i = threadIdx.x; i < pixels * 32; i += blockDim.x) out[i] = sm[i];
  if (threadIdx.x == 0) out[pixels * 32] = done ? 1.f : 0.f;
}

int main() {
  const int N = 2, D = 2, H = 4, W = 5, C = 32;
  std::vector<float> hx((size_t)N * D * H * W * C);
  for (int n = 0; n < N; ++n) for (int d = 0; d < D; ++d) for (int h = 0; h < H; ++h) for (int w = 0; w < W; ++w)
    for (int c = 0; c < C; ++c) hx[((((size_t)n * D + d) * H + h) * W + w) * C + c] = n * 1000 + d * 100 + h * 10 + w + c / 100.f;
  float *dx, *dout;
  CK(cudaMalloc(&dx, hx.size() * 4));
  CK(cudaMemcpy(dx, hx.data(), hx.size() * 4, cudaMemcpyHostToDevice));
  const int MAXP = 64;
  CK(cudaMalloc(&dout, (MAXP * 32 + 1) * 4));
  void* fp = nullptr;
  cudaDriverEntryPointQueryResult q;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fp, cudaEnableDefault, &q));
  if (!fp) { printf("no cuTensorMapEncodeIm2col\n"); return 1; }
  EncodeIm2colFn enc = (EncodeIm2colFn)fp;
  CK(cudaFuncSetAttribute(probe, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));

  struct Case { const char* name; int lo[3], hi[3]; unsigned es[5]; int pixels; int c, w, h, d, n, ow, oh, od; };
  // corners are {W, H, D} order (innermost first), like the tensor dims {C, W, H, D, N}
  Case cases[] = {
    {"A pad1 k3 s1: coords(-1,-1,-1) off(0,0,0)", {-1,-1,-1}, {-1,-1,-1}, {1,1,1,1,1}, 24, 0,-1,-1,-1,0, 0,0,0},
    {"B pad1 k3 s1: coords(0,0,0) off(0,0,0)",    {-1,-1,-1}, {-1,-1,-1}, {1,1,1,1,1}, 24, 0,0,0,0,0, 0,0,0},
    {"C pad1 k3 s1: coords(-1,-1,-1) off(1,1,1)", {-1,-1,-1}, {-1,-1,-1}, {1,1,1,1,1}, 24, 0,-1,-1,-1,0, 1,1,1},
    {"D pad1 k3 s1: coords(-1,-1,-1) off(2,2,2)", {-1,-1,-1}, {-1,-1,-1}, {1,1,1,1,1}, 24, 0,-1,-1,-1,0, 2,2,2},
    {"E pad1 k3 s1: start w=2,h=2,d=0,n=1 off(1,1,1) (tail of tensor)", {-1,-1,-1}, {-1,-1,-1}, {1,1,1,1,1}, 24, 0,2,2,0,1, 1,1,1},
    {"F k(1,3,3) pad(0,1,1) s(1,2,2): coords(-1,-1,0) off(1,1,0)", {-1,-1,0}, {-1,-1,0}, {1,2,2,1,1}, 16, 0,-1,-1,0,0, 1,1,0},
    {"G k(1,3,3) pad(0,1,1) s(1,2,2): coords(-1,-1,0) off(0,0,0)", {-1,-1,0}, {-1,-1,0}, {1,2,2,1,1}, 16, 0,-1,-1,0,0, 0,0,0},
    {"H same as F but start at 2nd output pixel: coords(1,-1,0)", {-1,-1,0}, {-1,-1,0}, {1,2,2,1,1}, 16, 0,1,-1,0,0, 1,1,0},
    {"I k1 no pad: coords(0,0,0) c=0 pixels 48 (runs past the tensor end?)", {0,0,0}, {0,0,0}, {1,1,1,1,1}, 48, 0,2,3,1,1, 0,0,0},
    {"J dil2 k3 pad2: coords(-2,-2,0) off(4,4,0)", {-2,-2,0}, {-2,-2,0}, {1,1,1,1,1}, 16, 0,-2,-2,0,0, 4,4,0},
  };
  for (const Case& cs : cases) {
    alignas(64) CUtensorMap tm;
    cuuint64_t gdim[5] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)D, (cuuint64_t)N};
    cuuint64_t gstr[4] = {(cuuint64_t)C * 4, (cuuint64_t)C * 4 * W, (cuuint64_t)C * 4 * W * H, (cuuint64_t)C * 4 * W * H * D};
    CUresult r = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, dx, gdim, gstr, cs.lo, cs.hi, 32, (cuuint32_t)cs.pixels, cs.es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    printf("== %s : encode rc=%d\n", cs.name, (int)r);
    if (r != CUDA_SUCCESS) continue;
    probe<<<1, 128, 48 * 1024>>>(tm, cs.c, cs.w, cs.h, cs.d, cs.n, cs.ow, cs.oh, cs.od, cs.pixels, 32, dout);
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { printf("   kernel error: %s\n", cudaGetErrorString(e)); return 2; }
    std::vector<float> ho(MAXP * 32 + 1);
    CK(cudaMemcpy(ho.data(), dout, (cs.pixels * 32 + 1) * 4, cudaMemcpyDeviceToHost));
    printf("   completed=%d rows:", (int)ho[cs.pixels * 32]);
    for (int p = 0; p < cs.pixels; ++p) {
      const int chunk = (0 ^ (p & 7));                 // channel 0..3 live in logical 16-byte chunk 0
      printf(" %g", ho[p * 32 + chunk * 4]);
    }
    printf("\n");
  }
  return 0;
}
