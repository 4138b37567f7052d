// Hopper (sm_90a) warpgroup-MMA gathered GEMM.
//
//   D[m,n] = epi( sum_k A[m,k] * B[n,k] ),  fp32 storage, wgmma tf32 MMA, fp32 accumulate in registers.
//
// Persistent kernel: grid = min(#tiles, #SMs), one CTA per SM walks a static sequence of 128 x BN output
// tiles (BN <= 128; 64 x 2 BN "wide" tiles when both operands are MN-major and M <= 64, Launch::wide):
//   PRODUCERS  -- the A/B K-chunks (32 fp32 = one 128-byte swizzle row) go straight from NDHWC tensors into
//              swizzled shared-memory tiles, never through an im2col buffer: dense K-major operands by TMA
//              tiled boxes (SWIZZLE_128B), convolution gathers by TMA im2col copies (conv fwd, unit-stride
//              dgrad), the conv1 stem by overlapping-window TMA boxes (one thread issues), and MN-major operands
//              and what TMA cannot express (strided dgrad outside the parity classes, unaligned operands) by
//              16-byte cp.async with zero-fill = padding (8 warps; a TMA-only build has one producer warpgroup);
//   CONSUMERS  -- two warpgroups; warpgroup w issues wgmma.m64nBNk8 for tile rows [64 w, 64 w + 64) (wide tiles:
//              columns [w BN, w BN + BN) of the 64 rows) and then
//              runs the epilogue of those rows from its registers: smem transpose -> fused affine /
//              residual / ReLU / TF32 rounding -> coalesced 128-bit global stores (or atomics for split-K).
// wgmma reads tf32 operands K-major only, so an MN-major stage tile (wgrad, transposed matmul operands) is
// first rewritten by the consumers into a K-major image in shared memory.  The smem ring (full[s]/empty[s]
// mbarriers) runs continuously across tiles, so the producers load the next tile during the epilogue.
//
// Operand kinds are described in include/vlfb.h; their element-level definition is
// operand_elem() in common.cuh, which the SIMT engine evaluates literally and the tests
// compare this kernel against.
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

#include <type_traits>

#include "common.cuh"

#ifndef VLFB_EPI_DEPTH
#define VLFB_EPI_DEPTH 2
#endif
namespace vlfb {
namespace tc {

constexpr int BM = 128;        // tile rows (two wgmma M = 64 warpgroups)
constexpr int BN_MAX = 128;    // widest tile: a warpgroup holds 64 x BN fp32 accumulators = BN / 2 registers per thread
constexpr int KC = 32;         // fp32 per K chunk (128 B)
constexpr int NPROD = 256;     // 8 cp.async producer warps = 2 per scheduler, so the address-generation latency of
                               // one warp hides behind the other
constexpr int RSTEP = NPROD / 8;   // rows covered by one pass of the K-major loaders
constexpr int NEPI = 256;          // 2 consumer warpgroups (MMA + epilogue); warp w of a warpgroup owns 16 tile rows
constexpr int NPROD_TMA = 128;     // producer threads of a TMA-only build: one warpgroup, so the consumers are warpgroup-aligned
constexpr int EPC = 16;            // accumulator columns per epilogue step
constexpr int EROWS = 2;           // tile rows per lane in the epilogue: (lane >> 2) + 8 i of the warp's 16
constexpr int EPITCH = BN_MAX + 4; // padded accumulator staging row (floats): a consumer warp's 16 rows x the tile
constexpr int EPI_COLV = 2 * BN_MAX;  // per-warp column scale + bias of the tile's columns (floats)
constexpr int EPI_WARP_FLOATS = 16 * EPITCH + EPI_COLV;
constexpr int EPI_STAGE_BYTES = (NEPI / 32) * EPI_WARP_FLOATS * 4;
constexpr int A_TILE_BYTES = BM * KC * 4;  // 16 KB
constexpr int MAX_STAGES = 8;
constexpr int WM = 64;                     // rows of a wide tile (Launch::wide): one wgmma M
// a wide launch's K-major images (one WM-row A, two 2 BN-row B) live in the epilogue staging tiles
static_assert(WM * KC * 4 + 2 * (2 * BN_MAX) * KC * 4 <= EPI_STAGE_BYTES, "wide images must fit the epilogue staging");

// ---------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok;
}
// Bounded wait: a protocol bug traps (kernel error) instead of hanging the GPU.  The clock is only read
// every 4096 polls so that the spin loop stays 3 instructions long (try_wait suspends in hardware).  No printf:
// a call inside the consumers' K loop would make ptxas serialize the wgmma pipeline.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = 0;
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0xFFFu) == 0) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 8000000000LL) {
        __trap();
      }
    }
  }
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  // ignore-src predicate => 16 bytes of zeros (conv padding / tails); one LDGSTS.ZFILL, no size arithmetic
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.eq.u32 p, %2, 0;\n\t"
      "cp.async.cg.shared.global [%0], [%1], 16, p;\n\t}"
      ::"r"(dst), "l"(src), "r"((uint32_t)valid) : "memory");
}
// TMA: one thread arms the stage barrier with the byte count, then issues the bulk tensor copy; the copy
// engine writes the box into shared memory in the SWIZZLE_128B pattern and completes the transaction.
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* tm, int c0, int c1, int c2, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* tm, int c0, int c1, int c2, int c3, int c4,
                                            uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4), "r"(bar)
      : "memory");
}
// Arrive on the mbarrier once every cp.async this thread has issued so far has landed (noinc: the arrival is one of the
// barrier's expected arrivals), without waiting for them.
__device__ __forceinline__ void cp_async_mbar_arrive(uint32_t bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void cp_async_wait_dyn(int n) {
  switch (n) {
    case 0: cp_async_wait<0>(); break;
    case 1: cp_async_wait<1>(); break;
    case 2: cp_async_wait<2>(); break;
    case 3: cp_async_wait<3>(); break;
    case 4: cp_async_wait<4>(); break;
    default: cp_async_wait<5>(); break;
  }
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// the 256 consumer threads (named barrier 1; barrier 0 is __syncthreads)
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, %0;" ::"n"(NEPI) : "memory"); }
// wgmma m64nNk8, tf32 x tf32 -> f32, both operands K-major SWIZZLE_128B in shared memory; d[0, N/2) accumulates
// (scale-d = 0 on the first MMA of a tile overwrites it).
template <int N>
__device__ __forceinline__ void wgmma_tf32(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (N == 32) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(accumulate));
  } else if constexpr (N == 64) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(accumulate));
  } else if constexpr (N == 96) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
        : "l"(da), "l"(db), "r"(accumulate));
  } else if constexpr (N == 128) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(accumulate));
  }
}
// wgmma shared-memory matrix descriptor: K-major SWIZZLE_128B, 8-row groups 1024 B apart (SBO), LBO unused (1).
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);                 // [0,14)  start address
  d |= (uint64_t)1 << 16;                                  // [16,30) leading byte offset (unused by 128B swizzle)
  d |= (uint64_t)(1024 >> 4) << 32;                        // [32,46) stride byte offset
  d |= (uint64_t)1 << 62;                                  // [62,64) 1 = SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void red_add_f4(float* p, const float4& v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float4 ld_cg_f4(const float* p) {
  float4 v;
  asm volatile("ld.global.cg.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}
// residual / accumulate reads: plain (coherent) 128-bit loads -- D may have been written by an earlier launch
// on the same stream, never by this one
__device__ __forceinline__ float4 ld_nc_f4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ uint32_t ld_nc_u16(const unsigned short* p) {
  unsigned short v;
  asm volatile("ld.global.nc.u16 %0, [%1];" : "=h"(v) : "l"(p));
  return (uint32_t)v;
}
__device__ __forceinline__ void prefetch_l2(const void* p) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}

// Split-TF32 (VLFB_PREC_X3): x = hi + lo with hi = x with its low 13 mantissa bits cleared (what the tensor core reads of
// an fp32 operand: it truncates) and lo = x - hi, which is exact in fp32.
__device__ __forceinline__ float tf32_lo(float x) { return x - __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }

// Consumer-side rewrite of an MN-major stage tile into the K-major SWIZZLE_128B image [row][128 B] that wgmma reads
// (tf32 operands in shared memory must be K-major).  Source: `rows` x 32 k as [atom of 32 elements][k-row][128 B]
// (MNLoader), 16-byte chunk c of k-row k at byte (16 c) ^ (32 (k & 3)), k-rows 128 B and atoms 4 KB apart.
// Image: element (n, k) at n * 128 + 16 ((k / 4) ^ (n % 8)) + 4 (k % 4).
// Unit u = t + NEPI j moves a 4 n x 4 k block: k-quad kq = u % 8, source chunk c = kq ^ ((u / 8) % 8) of atom u / 64.
// It reads chunk c of k-rows 4 kq .. 4 kq + 3 (four v4 loads), transposes in registers and writes rows n = 32 atom +
// 4 c + q, q = 0..3, at k-quad kq (four v4 stores).  A 16-byte access is served in four phases of 8 lanes, and a phase
// is conflict-free when its 8 addresses fall in 8 distinct 16-byte slots of the 128-byte bank window.  The 8 lanes of
// a phase have kq = 0..7 and one value of (u / 8) % 8 = b:
//   loads:  slot = c ^ 2 (k & 3) = kq ^ b ^ 2 r for load r  -> 8 distinct slots;
//   stores: slot = kq ^ (n % 8) = kq ^ 4 ((kq ^ b) & 1) ^ q  -> kq ^ const on even kq, kq ^ (const ^ 4) on odd kq, a
//           bijection of 0..7 (bit 0 is kept) -> 8 distinct slots.
// LO (split TF32, DESIGN.md 4.7): the same pass also writes the lo image of every element to `dst_lo`, in the image's layout.
template <bool LO = false>
__device__ __forceinline__ void mn_to_kmajor(uint32_t src, uint32_t dst, int rows, int ctid, uint32_t dst_lo = 0) {
  for (int u = ctid; u < rows * 2; u += NEPI) {
    const int kq = u & 7, c = kq ^ ((u >> 3) & 7), atom = u >> 6;
    float v[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int k = 4 * kq + r;
      asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                   : "=f"(v[r][0]), "=f"(v[r][1]), "=f"(v[r][2]), "=f"(v[r][3])
                   : "r"(src + (uint32_t)(atom * 4096 + k * 128) + (uint32_t)((c * 16) ^ (r << 5)))
                   : "memory");
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int n = atom * 32 + 4 * c + q;
      asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};"
                   ::"r"(dst + (uint32_t)(n * 128 + ((kq ^ (n & 7)) << 4))), "f"(v[0][q]), "f"(v[1][q]), "f"(v[2][q]), "f"(v[3][q])
                   : "memory");
      if constexpr (LO)
        asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};"
                     ::"r"(dst_lo + (uint32_t)(n * 128 + ((kq ^ (n & 7)) << 4))), "f"(tf32_lo(v[0][q])), "f"(tf32_lo(v[1][q])),
                       "f"(tf32_lo(v[2][q])), "f"(tf32_lo(v[3][q]))
                     : "memory");
    }
  }
}

// lo image of a K-major stage tile of `bytes` bytes: elementwise, so it keeps the tile's SWIZZLE_128B layout and the
// wgmma descriptors of the tile address it at the same offsets.  Consecutive 16-byte units per thread: conflict-free.
__device__ __forceinline__ void kmajor_lo(uint32_t src, uint32_t dst, uint32_t bytes, int ctid) {
  for (uint32_t o = (uint32_t)ctid * 16u; o < bytes; o += NEPI * 16u) {
    float v0, v1, v2, v3;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v0), "=f"(v1), "=f"(v2), "=f"(v3) : "r"(src + o) : "memory");
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};"
                 ::"r"(dst + o), "f"(tf32_lo(v0)), "f"(tf32_lo(v1)), "f"(tf32_lo(v2)), "f"(tf32_lo(v3)) : "memory");
  }
}

__host__ __device__ constexpr bool is_mn(int kind) { return kind == VLFB_OP_DENSE_MN || kind == VLFB_OP_CONV_MN || kind == VLFB_OP_STEM_MN; }

// ---------------------------------------------------------------- fast integer division
// q = x / d for 0 <= x < 2^31 with a precomputed multiplier (the gather loaders decode an output
// position per 16-byte copy; 64-bit hardware division there cost more than the copy itself).
struct FastDiv { uint32_t mul, shr, d; };
inline FastDiv make_fastdiv(int d) {
  FastDiv f;
  f.d = (uint32_t)d;
  if (d <= 1) { f.mul = 0; f.shr = 0; return f; }
  int lg = 31 - __builtin_clz((unsigned)d);
  if (d & (d - 1)) ++lg;                       // ceil(log2 d)
  const int p = 31 + lg;
  f.mul = (uint32_t)(((1ull << p) + (uint64_t)d - 1) / (uint64_t)d);
  f.shr = (uint32_t)(p - 32);
  return f;
}
__device__ __forceinline__ void fd_divmod(uint32_t x, const FastDiv& f, uint32_t& q, uint32_t& r) {
  q = (f.d <= 1) ? x : (__umulhi(x, f.mul) >> f.shr);
  r = x - q * f.d;
}
struct PosDiv { FastDiv w, h, t; };
__device__ __forceinline__ Pos4 decode_pos_fast(uint32_t idx, const PosDiv& pd) {
  Pos4 p;
  uint32_t q, r;
  fd_divmod(idx, pd.w, q, r); p.w = (int)r;
  fd_divmod(q, pd.h, q, r); p.h = (int)r;
  fd_divmod(q, pd.t, q, r); p.t = (int)r;
  p.n = (int)q;
  return p;
}

// TMA im2col mode: the 5-D map of an NDHWC tensor walks
// `pixelsPerColumn` window origins in W -> H -> D -> N order inside the bounding box [lower, dim-1+upper] with the
// convolution strides as traversal strides; {w,h,d} = origin of the first window (= out*stride - pad), the u16
// offsets select the filter tap (tap*dilation); out-of-range pixels (padding, tensor tail) read as zeros.
__device__ __forceinline__ void tma_load_im2col(uint32_t dst, const CUtensorMap* tm, int c, int w, int h, int d, int n,
                                                int ow, int oh, int od, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%2, %3, %4, %5, %6}], [%7], {%8, %9, %10};"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(c), "r"(w), "r"(h), "r"(d), "r"(n), "r"(bar),
        "h"((uint16_t)ow), "h"((uint16_t)oh), "h"((uint16_t)od)
      : "memory");
}

// ---------------------------------------------------------------- K-major loaders
// Tile = `rows` rows x 128 B.  Thread t copies the 16-byte chunk (t & 7) of rows (t >> 3) + RSTEP j.
template <int KIND, int MAXR>
struct KLoader {
  const float* base;
  int64_t ld;
  int nrow;          // rows of this tile handled per thread (rows / RSTEP)
  int kend;          // DENSE_K: K limit for the 16-byte tail predicate
  int row0;
  // per owned row: decoded position (conv kinds) and the swizzled shared-memory offset of its 16-byte chunk
  int s_n[MAXR], s_t[MAXR], s_hw[MAXR];
  uint32_t dst[MAXR];
  uint32_t rowmask;  // DENSE_K: bit j set when row j is inside the matrix
  // Filter-tap cursor.  Chunks are issued in order, so the tap advances incrementally (no division per
  // chunk) and the gathered element offset / validity of every owned row is recomputed only when the
  // tap changes (per-chunk divisions and 64-bit address math would make the producers instruction-bound).
  int cpt, tc, kt, kh, kw;
  int off[MAXR];
  uint32_t okmask;

  __device__ __forceinline__ void init(const vlfb_gemm_params_t& p, const vlfb_operand_t& op, int row0_, int rows,
                                       int limit, int batch, const PosDiv& pdo, const PosDiv& pdi, int kc_first) {
    const int tid = threadIdx.x;
    const int c = tid & 7;
    nrow = rows / RSTEP;
    base = op.ptr;
    ld = op.ld;
    if (KIND == VLFB_OP_STEM_K && ld <= 0) ld = p.g.W;
    kend = p.K;
    rowmask = 0;
    row0 = row0_;
    const vlfb_conv_geom_t& g = p.g;
    if (KIND == VLFB_OP_DENSE_K) base += (int64_t)batch * op.batch_stride;
#pragma unroll
    for (int j = 0; j < MAXR; ++j) {
      if (j >= nrow) break;
      const int r = (tid >> 3) + RSTEP * j;
      const int row = row0 + r;
      const bool ok = row < limit;
      dst[j] = (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4));
      if (KIND == VLFB_OP_DENSE_K) {
        if (ok) rowmask |= 1u << j;
      } else if (KIND == VLFB_OP_CONV_K || KIND == VLFB_OP_STEM_K) {
        Pos4 o = decode_pos_fast(ok ? (uint32_t)row : 0u, pdo);
        s_n[j] = o.n * g.T;
        s_t[j] = ok ? o.t * g.sT - g.pT : -100000;
        s_hw[j] = ((o.h * g.sH - g.pH) << 16) | ((o.w * g.sW - g.pW) & 0xFFFF);
      } else {  // DGRAD_K: rows are input positions
        Pos4 i = decode_pos_fast(ok ? (uint32_t)row : 0u, pdi);
        s_n[j] = i.n * g.To;
        s_t[j] = ok ? i.t + g.pT : -100000;
        s_hw[j] = ((i.h + g.pH) << 16) | ((i.w + g.pW) & 0xFFFF);
      }
    }
    if (KIND == VLFB_OP_CONV_K || KIND == VLFB_OP_DGRAD_K) {
      cpt = (KIND == VLFB_OP_CONV_K ? g.C : g.Co) / KC;
      const int tap = kc_first / cpt;              // one division per tile
      tc = kc_first - tap * cpt;
      decode_tap(tap, g.kH, g.kW, kt, kh, kw);
      compute_tap(g);
    } else if (KIND == VLFB_OP_STEM_K) {
      kt = kc_first / g.kH;
      kh = kc_first - kt * g.kH;
    }
  }

  __device__ __forceinline__ void compute_tap(const vlfb_conv_geom_t& g) {
    okmask = 0;
    const int dt = kt * g.dT, dh = kh * g.dH, dw = kw * g.dW;
#pragma unroll
    for (int j = 0; j < MAXR; ++j) {
      if (j >= nrow) break;
      if (KIND == VLFB_OP_CONV_K) {
        const int ti = s_t[j] + dt, hi = (s_hw[j] >> 16) + dh, wi = (int)(short)(s_hw[j] & 0xFFFF) + dw;
        const bool ok = (unsigned)ti < (unsigned)g.T && (unsigned)hi < (unsigned)g.H && (unsigned)wi < (unsigned)g.W;
        off[j] = ok ? (((s_n[j] + ti) * g.H + hi) * g.W + wi) * g.C : 0;
        if (ok) okmask |= 1u << j;
      } else {  // DGRAD_K
        const int a = s_t[j] - dt, b = (s_hw[j] >> 16) - dh, cc = (int)(short)(s_hw[j] & 0xFFFF) - dw;
        bool ok = a >= 0 && b >= 0 && cc >= 0;
        int to = a, ho = b, wo = cc;
        if (g.sT != 1) { ok = ok && (a % g.sT == 0); to = a / g.sT; }
        if (g.sH != 1) { ok = ok && (b % g.sH == 0); ho = b / g.sH; }
        if (g.sW != 1) { ok = ok && (cc % g.sW == 0); wo = cc / g.sW; }
        ok = ok && to < g.To && ho < g.Ho && wo < g.Wo;
        off[j] = ok ? (((s_n[j] + to) * g.Ho + ho) * g.Wo + wo) * g.Co : 0;
        if (ok) okmask |= 1u << j;
      }
    }
  }

  // Issue the cp.asyncs of the NEXT K chunk (`kc` = its global index, used by DENSE_K only) into `tile`.
  __device__ __forceinline__ void issue(const vlfb_gemm_params_t& p, int kc, uint32_t tile) {
    const int c = threadIdx.x & 7;
    const vlfb_conv_geom_t& g = p.g;
    if (KIND == VLFB_OP_DENSE_K) {
      const int k = kc * KC + c * 4;
      const bool kok = k < kend;
      const int r0 = threadIdx.x >> 3;
#pragma unroll
      for (int j = 0; j < MAXR; ++j) {
        if (j >= nrow) break;
        const bool ok = kok && ((rowmask >> j) & 1u);
        const float* src = ok ? base + (int64_t)(row0 + r0 + RSTEP * j) * ld + k : base;
        cp_async16(tile + dst[j], src, ok);
      }
    } else if (KIND == VLFB_OP_CONV_K || KIND == VLFB_OP_DGRAD_K) {
      const int c0 = tc * KC + c * 4;
#pragma unroll
      for (int j = 0; j < MAXR; ++j) {
        if (j >= nrow) break;
        const bool ok = (okmask >> j) & 1u;
        cp_async16(tile + dst[j], base + (off[j] + c0), ok);
      }
      if (++tc == cpt) {          // next tap
        tc = 0;
        if (++kw == g.kW) { kw = 0; if (++kh == g.kH) { kh = 0; ++kt; } }
        compute_tap(g);
      }
    } else {  // STEM_K: chunk = one (kt,kh) filter row of 8 pixels x 4 channels; this thread's pixel = c
#pragma unroll
      for (int j = 0; j < MAXR; ++j) {
        if (j >= nrow) break;
        const int ti = s_t[j] + kt, hi = (s_hw[j] >> 16) + kh, wi = (int)(short)(s_hw[j] & 0xFFFF) + c;
        const bool ok = (unsigned)ti < (unsigned)g.T && (unsigned)hi < (unsigned)g.H && (unsigned)wi < (unsigned)g.W;
        const int o = ok ? (((s_n[j] + ti) * g.H + hi) * (int)ld + wi) * 4 : 0;      // ld = row pitch in pixels
        cp_async16(tile + dst[j], base + o, ok);
      }
      if (++kh == g.kH) { kh = 0; ++kt; }
    }
  }
};

// ---------------------------------------------------------------- MN-major loaders
// Tile = 32 k-rows, each `rows`*4 bytes of the m (or n) extent, stored as
// [atom of 32 elements][32 k-rows][128 B] (the consumers rewrite it K-major before the MMAs, mn_to_kmajor).
template <int KIND>
struct MNLoader {
  static constexpr int SGRP = (32 * (BN_MAX / 4)) / NPROD;   // copies per thread per chunk at a 128-row tile (the
                                                             // 256-row B tile of a wide launch takes two groups)
  const float* base;
  int64_t ld;
  int tapz, nslot;
  // A thread copies the SAME 16-byte column chunk c of the k-rows kk0, kk0 + kstep, ... (NPROD is a multiple of
  // the chunks per k-row), so everything that depends on the column -- bounds, filter tap (kh,kw), channel,
  // swizzled shared-memory offset -- is one scalar per tile, and the per-chunk work per copy is two shuffles,
  // a bit test and an add.
  int mn, kk0, kstep;
  bool colok;
  uint32_t dst0, dstep;
  int slotoff;       // conv kinds: element offset of (kh,kw,ci) relative to the k-row's window origin
  int sh, sw;        // bit positions of this column's kh / kw in the k-row's validity word

  __device__ __forceinline__ void init(const vlfb_gemm_params_t& p, const vlfb_operand_t& op, int row0, int rows,
                                       int limit, int batch, int tap, const FastDiv& cdiv, const FastDiv& kwdiv) {
    const vlfb_conv_geom_t& g = p.g;
    base = op.ptr;
    if (KIND == VLFB_OP_DENSE_MN) base += (int64_t)batch * op.batch_stride;
    ld = op.ld;
    tapz = tap;
    const int cpr = rows >> 2;            // 16-byte chunks per k-row (8, 16, 32 or 64; power of two)
    const int lcpr = 31 - __clz(cpr);
    nslot = (KC * cpr) / NPROD;
    kstep = NPROD >> lcpr;
    kk0 = threadIdx.x >> lcpr;
    const int c = threadIdx.x & (cpr - 1);
    mn = row0 + c * 4;
    colok = mn < limit;
    // atom-major tile [atom of 32 elements][32 k-rows][128 B], 32-byte units of a k-row XOR (k & 3).
    // kstep is a multiple of 4 whenever a thread owns more than one copy, so the XOR term is per-thread.
    const int r = kk0 & 3, cc8 = c & 7;
    dst0 = (uint32_t)((c >> 3) * 4096 + kk0 * 128 + ((((cc8 >> 1) ^ r) << 5) | ((cc8 & 1) << 4)));
    dstep = (uint32_t)(kstep * 128);
    slotoff = 0; sh = 0; sw = 8;
    if (KIND == VLFB_OP_CONV_MN) {
      uint32_t tap_hw, cc, qh, qw;
      fd_divmod((uint32_t)(colok ? mn : 0), cdiv, tap_hw, cc);     // n = (kh*kW + kw) * C + ci
      fd_divmod(tap_hw, kwdiv, qh, qw);
      slotoff = ((int)qh * g.dH * g.W + (int)qw * g.dW) * g.C + (int)cc;
      sh = (int)qh; sw = 8 + (int)qw;
    } else if (KIND == VLFB_OP_STEM_MN) {            // n = kh*32 + px*4 (+ch); ld = row pitch in pixels (0 = W)
      if (ld <= 0) ld = g.W;
      const int qh = mn >> 5, qw = (mn & 31) >> 2;
      slotoff = (qh * (int)ld + qw) * 4;
      sh = qh; sw = 8 + qw;
    }
  }

  // k0 = first k of this chunk, kend = exclusive k limit of this CTA's K range.
  // Conv kinds (wgrad B operand): the N extent spans ALL (kh,kw) taps of one kt slice, so one pass over dY
  // feeds up to 256 (tap, ci) columns.  Each lane decodes ONE of the 32 k-rows (output positions) of the
  // chunk into (element offset of its window origin, validity bits per kh and per kw); the copies fetch the
  // row they need with warp shuffles.
  __device__ __forceinline__ void issue(const vlfb_gemm_params_t& p, const PosDiv& pd, int k0, int kend, uint32_t tile) const {
    const vlfb_conv_geom_t& g = p.g;
    int info_a = 0, info_b = 0;
    if (KIND != VLFB_OP_DENSE_MN) {
      const int k = k0 + (threadIdx.x & 31);
      const bool okr = k < kend;
      const Pos4 o = decode_pos_fast(okr ? (uint32_t)k : 0u, pd);
      const int t0 = o.t * g.sT - g.pT + tapz * g.dT;          // z slice = temporal tap
      const bool okt = okr && (unsigned)t0 < (unsigned)g.T;
      const int h0 = o.h * g.sH - g.pH, w0 = o.w * g.sW - g.pW;
      info_a = (((o.n * g.T + t0) * g.H + h0) * (KIND == VLFB_OP_STEM_MN ? (int)ld : g.W) + w0) * g.C;
      const int nh = g.kH, nw = (KIND == VLFB_OP_STEM_MN) ? 8 : g.kW;
      const int dh = (KIND == VLFB_OP_STEM_MN) ? 1 : g.dH, dw = (KIND == VLFB_OP_STEM_MN) ? 1 : g.dW;
      int hm = 0, wm = 0;
      for (int q = 0, h = h0; q < nh; ++q, h += dh) hm |= ((unsigned)h < (unsigned)g.H) ? (1 << q) : 0;
      for (int q = 0, w = w0; q < nw; ++q, w += dw) wm |= ((unsigned)w < (unsigned)g.W) ? (256 << q) : 0;
      info_b = okt ? (hm | wm) : 0;
    }
    int lane_src = kk0;
    uint32_t d = tile + dst0;
    // groups of SGRP copies: one pass up to the 128-row tiles, two for a wide launch's 256-row B tile (a body unrolled
    // over all MAXS copies slows the producers of every MN-major launch)
    for (int j0 = 0; j0 < nslot; j0 += SGRP) {
#pragma unroll
      for (int j = 0; j < SGRP; ++j) {
        if (j0 + j >= nslot) break;
        bool ok = colok;
        const float* src = base;
        if (KIND == VLFB_OP_DENSE_MN) {
          const int k = k0 + lane_src;
          ok = ok && k < kend;
          if (ok) src = base + (int64_t)k * ld + mn;
        } else {
          const int ra = __shfl_sync(0xffffffffu, info_a, lane_src);
          const int rb = __shfl_sync(0xffffffffu, info_b, lane_src);
          ok = ok && (((rb >> sh) & (rb >> sw) & 1) != 0);
          if (ok) src = base + (ra + slotoff);
        }
        // columns beyond the matrix are never copied: whatever shared memory holds there only reaches accumulator
        // columns >= N, which the epilogue does not store (k tails of real columns ARE zero-filled)
        if (colok) cp_async16(d, src, ok);
        lane_src += kstep;
        d += dstep;
      }
    }
  }
};

// ---------------------------------------------------------------- the kernel
// Timeline instrumentation of the diagnostic build (-DVLFB_TRACE, scripts/trace_gemm.py): per CTA 64 clock64 slots.
//   0 entry, 1 globaltimer at entry, 2 prologue done, 3 exit; producer 8+2i / 9+2i = work item i first / last copy issued;
//   MMA 16+2i first chunk landed, 17+2i last MMA issued; epilogue warp 0: 24+4i accumulator ready, 25+4i blocks done,
//   26+4i piece counted, 27+4i fix-up done.
#ifdef VLFB_TRACE
unsigned long long* g_trace_buf = nullptr;
#define TR(slot) do { if (L.trace) L.trace[(size_t)blockIdx.x * 64 + (slot)] = (unsigned long long)clock64(); } while (0)
#else
#define TR(slot) do { } while (0)
#endif
constexpr int MAX_UNITS = 160;       // >= #SMs: CTAs of the persistent grid
constexpr int SK_CNT_INTS = 16384;   // arrival counters at the head of the stream-K workspace (tile x consumer warp)

// the lean epilogue addresses D / residual / sign bits with 32-bit element offsets
__host__ __device__ inline bool span32_ok(const vlfb_gemm_params_t& p) {
  const long long z = p.taps > 1 ? (long long)(p.taps - 1) * p.d_tap_stride : (long long)(p.batch - 1) * p.d_batch_stride;
  return z >= 0 && p.ldd > 0 && (long long)p.M * p.ldd + z < (1ll << 32);
}

struct ParCls { short nh, nw, rh, rw, ph, pw; int nk; };   // taps per dim, first tap, parity, K chunks of the class

struct Launch {
  int bn;        // tile N (32/64/96/128) = wgmma N
  // Wide tiles (both operands MN-major and M <= 64: every wgrad with Co <= 64): a tile is 64 rows x 2 bn columns
  // instead of 128 x bn, and warpgroup w computes columns [w bn, (w + 1) bn) of the 64 rows, so no warpgroup multiplies
  // padding rows.  Both warpgroups read one 64-row A image; each reads its half of a 2 bn-row B image.  Staged by the
  // cp.async loaders only; the K-major images alias the epilogue staging tiles, so bn = 128 keeps 3 stages, bn = 64 six.
  int wide;
  int stages;
  PosDiv out;    // fast divisors of the conv OUTPUT extents (Wo, Ho, To)
  PosDiv in;     // ... and of the INPUT extents (W, H, T) for the dgrad row decode
  FastDiv cdiv;  // input channels C (wgrad: n -> (tap, ci))
  FastDiv kwdiv; // kW
  int tma_a, tma_b;  // loader of each operand (K-major only; MN-major operands are always 0): 0 = cp.async, 1 = dense
                     // tiled boxes, 2 = im2col (conv gathers, A only), 3 = conv1 stem rows (A only): {8 px x 4 ch =
                     // 128 B, 16 output positions} boxes of the overlapping-window view of a W-padded clip (make_tmap_stem)
  int lag;           // cp.async groups kept in flight before a stage is published (< stages)
  int tiles_m, tiles_n, total_tiles;
  int stem_patch;    // conv1 forward: an M tile = a 16 (wo) x 8 (ho) patch of one output frame instead of 128 consecutive
                     // positions, so that ONE strided TMA box stages the whole A tile of a K chunk (tile row r =
                     // (ho0 + r / 16, wo0 + r % 16)); the fast epilogue maps rows back (patch_row)
  int patch_wb, patch_hb;   // patches per output row / per frame column: Wo / 16, Ho / 8
  // Strided conv dgrad (A = DGRAD_K, sH / sW = 2) as sH * sW PARITY CLASSES: the input positions (h, w) = (sH h' + ph,
  // sW w' + pw) of one class receive only the filter taps kh = rh + sH j, kw = rw + sW i (rh = (ph + pH) % sH ...), i.e.
  // each class is a unit-stride convolution over dY with nh x nw taps (3x3 stride 2: 1 + 2 + 2 + 4 = 9 taps for the four
  // classes instead of 4 x 9 with three quarters of the gathered operand zero).  The class is the tile's z index: M
  // tiles run over the class's sub-grid (W / sW, H / sH, T, N), A is one im2col box over dY per chunk, B the chunk of
  // the transposed weights at the ORIGINAL tap, and the epilogue maps sub-grid rows back to dX rows (par_row).
  int par;           // number of parity classes (0 = off)
  int par_m;         // rows of one class = N T (H / sH) (W / sW)
  int par_lo[2];     // im2col origin offset (w, h) shared by the classes: (p + ph) / s - (taps - 1)
  PosDiv sub;        // fast divisors of the sub-grid extents
  ParCls par_cls[4];
  // Stream-K: the linear space (tile, K chunk) is cut into one contiguous range per unit (CTA), so every
  // SM gets the same number of chunks whatever the tile count.  A tile whose chunks span several units is reduced
  // through the workspace by the LAST unit to arrive at its counter (no unit ever waits for another).
  int sk;
  int nkt;           // K chunks per tile
  float* ws_tiles;   // partial-sum slots: [unit][2][128][bn]
  int* ws_cnt;       // arrival counters [tile][consumer warp], zero between launches
  unsigned long long* trace;   // diagnostic build only
  int bounds[MAX_UNITS + 1];
};

struct TileInfo {
  int m0, n0, batch, tap, k_begin, k_end, nk;
  int tile;          // linear tile index
  // stream-K: units sharing this tile, packed to keep the epilogue's register budget:
  //   bits 0-7 npieces (1 = whole tile here), 8-15 first unit, 16 = workspace slot (0/1) of that first unit's piece
  //   (every later piece is in slot 0), 17 = this unit's slot
  int pinfo;
  __device__ __forceinline__ int npieces() const { return pinfo & 0xFF; }
  __device__ __forceinline__ int ufirst() const { return (pinfo >> 8) & 0xFF; }
  __device__ __forceinline__ int first_slot() const { return (pinfo >> 16) & 1; }
  __device__ __forceinline__ int slot() const { return (pinfo >> 17) & 1; }
};

// Linear tile index -> (m tile fastest, n tile, z = batch|tap x split): CTAs that run concurrently share the
// same weight (B) tile in L2.
__device__ __forceinline__ void decode_tile(const vlfb_gemm_params_t& p, const Launch& L, int t, int split_k, TileInfo& ti) {
  const int mt = t % L.tiles_m;
  const int r = t / L.tiles_m;
  const int nt = r % L.tiles_n;
  const int z = r / L.tiles_n;
  const int split = z % split_k, zz = z / split_k;
  ti.batch = (p.taps > 1) ? 0 : zz;
  ti.tap = (p.taps > 1) ? zz : 0;
  ti.m0 = mt * BM;
  ti.n0 = nt * (L.bn << L.wide);       // (a wide launch has one M tile: m0 = 0)
  int kper = (p.K + split_k - 1) / split_k;
  kper = (kper + KC - 1) / KC * KC;
  ti.k_begin = split * kper;
  ti.k_end = min(p.K, ti.k_begin + kper);
  ti.nk = (ti.k_end > ti.k_begin) ? (ti.k_end - ti.k_begin + KC - 1) / KC : 0;
  if (L.par) {                     // z = parity class: its own K extent (possibly zero: epilogue-only tiles)
    ti.k_begin = 0;
    ti.nk = L.par_cls[zz].nk;
    ti.k_end = ti.nk * KC;
  }
  ti.tile = t;
  ti.pinfo = 1;
}

// strided-dgrad parity classes: dX row of sub-grid row m of class c
__device__ __forceinline__ int par_row(const vlfb_gemm_params_t& p, const Launch& L, int cls, int m) {
  const Pos4 o = decode_pos_fast((uint32_t)m, L.sub);
  const ParCls& c = L.par_cls[cls];
  return ((o.n * p.g.T + o.t) * p.g.H + o.h * p.g.sH + c.ph) * p.g.W + o.w * p.g.sW + c.pw;
}

// conv1 patch tiles: linear output position of tile row r of M tile `mt`
__device__ __forceinline__ int patch_row(const vlfb_gemm_params_t& p, const Launch& L, int mt, int r) {
  const int wb = mt % L.patch_wb, q = mt / L.patch_wb;
  const int hb = q % L.patch_hb, rest = q / L.patch_hb;            // rest = n * To + to
  return (rest * p.g.Ho + hb * 8 + (r >> 4)) * p.g.Wo + wb * 16 + (r & 15);
}

// Every role of a CTA walks the same work sequence.  cur/lim = next tile index / tile
// count (static loop, stride = #units) or next / end position in the (tile, K chunk) space (stream-K).
struct Sched { int cur, lim; };
__device__ __forceinline__ void sched_init(Sched& s, const Launch& L, int unit) {
  s.cur = L.sk ? L.bounds[unit] : unit;
  s.lim = L.sk ? L.bounds[unit + 1] : L.total_tiles;
}
__device__ __forceinline__ bool sched_next(const vlfb_gemm_params_t& p, const Launch& L, Sched& s, int unit, int nunits,
                                           TileInfo& ti) {
  if (L.sk) {
    if (s.cur >= s.lim) return false;
    const int tile = s.cur / L.nkt;
    const int c0 = s.cur - tile * L.nkt;
    const int len = min(L.nkt - c0, s.lim - s.cur);
    decode_tile(p, L, tile, 1, ti);
    ti.k_begin = c0 * KC;
    ti.k_end = min(p.K, (c0 + len) * KC);
    ti.nk = len;
    if (len != L.nkt && L.ws_tiles != nullptr) {
      const int s0 = tile * L.nkt, e0 = s0 + L.nkt;
      int uf = unit, ul = unit;
      while (L.bounds[uf] > s0) --uf;
      while (L.bounds[ul + 1] < e0) ++ul;
      const int first_slot = (L.bounds[uf] < s0) ? 1 : 0;
      const int slot = (unit == uf) ? first_slot : 0;
      ti.pinfo = (ul - uf + 1) | (uf << 8) | (first_slot << 16) | (slot << 17);
    }
    s.cur += len;
    return true;
  }
  while (s.cur < s.lim) {
    decode_tile(p, L, s.cur, p.split_k, ti);
    s.cur += nunits;
    if (ti.nk != 0 || L.par) return true;
  }
  return false;
}

// Persistent, warp-specialised: grid = min(#tiles, #SMs) CTAs; every role walks the same work sequence (Sched).  The
// smem ring (full/empty) runs continuously across tiles, so the producers stage the next tile while the consumers
// run the epilogue of the current one.
// CP = false: both operands are K-major and staged by TMA, so one producer warpgroup (one issuing thread) suffices and
// the CTA is 12 warps with up to 168 registers per thread; the 16-warp CP = true build (8 cp.async gather warps:
// MN-major operands, conv1 stem on a dense clip, strided dgrad, operands TMA cannot address) is capped at 128.
// FIX: the stream-K fix-up (a piece of a shared tile through the workspace) is compiled in; only the launches that plan
// fix-ups use these instantiations.  Its last-arriver decision is per warp, so the K loop must leave no MMA in flight
// when it ends on any path (ptxas would otherwise serialise every wgmma of the kernel, tests/test_gemm_pipeline_cpu.py).
// X3: split-TF32 products (gemm_tc3_kernel, DESIGN.md 4.7).  The consumers build a lo image of every operand chunk
// (double-buffered like the B images) and issue A_hi B_hi + A_hi B_lo + A_lo B_hi per k8 step; the stage tiles and the
// K-major images of MN-major operands are the hi operands as they stand (the tensor core truncates fp32 to TF32).
template <int AK, int BK, bool MASK, bool CP, bool FIX>
__global__ void __launch_bounds__((CP ? NPROD : NPROD_TMA) + NEPI, 1) gemm_tc_kernel(const vlfb_gemm_params_t p, const Launch L,
                                                              const __grid_constant__ CUtensorMap tmA,
                                                              const __grid_constant__ CUtensorMap tmB) {
  constexpr bool X3 = false;
#include "gemm_tc_body.inc"
}
// split-TF32 products (VLFB_PREC_X3): the same roles, loaders, schedules and epilogue
template <int AK, int BK, bool MASK, bool CP, bool FIX>
__global__ void __launch_bounds__((CP ? NPROD : NPROD_TMA) + NEPI, 1) gemm_tc3_kernel(const vlfb_gemm_params_t p, const Launch L,
                                                               const __grid_constant__ CUtensorMap tmA,
                                                               const __grid_constant__ CUtensorMap tmB) {
  constexpr bool X3 = true;
#include "gemm_tc_body.inc"
}


// Second half of a cp.async stream-K launch with fix-ups (deterministic atomic MN x MN launches): CTA t sums the
// workspace slots of tile t's pieces in piece order and applies d = epi(sum) (with VLFB_EPI_ATOMIC: d += epi(sum)) once
// per element.  Tiles that one unit ran whole were stored by the GEMM kernel itself.
__global__ void __launch_bounds__(256) gemm_fixup_kernel(const vlfb_gemm_params_t p, const Launch L) {
  const int t = blockIdx.x;
  const int s0 = t * L.nkt, e0 = s0 + L.nkt;
  int uf = 0, ul;
  while (L.bounds[uf + 1] <= s0) ++uf;                  // the unit whose range holds the tile's first chunk
  for (ul = uf; L.bounds[ul + 1] < e0; ++ul) {}         // ... and its last
  if (ul == uf) return;
  const int first_slot = L.bounds[uf] < s0 ? 1 : 0;     // as sched_next assigns the slots
  TileInfo ti;
  decode_tile(p, L, t, 1, ti);
  const int rows = L.wide ? WM : BM, tcols = L.bn << L.wide;
  const size_t tile_floats = (size_t)BM * L.bn;
  for (int idx = threadIdx.x; idx < rows * tcols; idx += blockDim.x) {
    const int r = idx / tcols, c = idx - r * tcols;
    const int m = ti.m0 + r, n = ti.n0 + c;
    if (m >= p.M || n >= p.N) continue;
    float v = 0.f;
    for (int u = uf; u <= ul; ++u)
      v += L.ws_tiles[(size_t)(u * 2 + (u == uf ? first_slot : 0)) * tile_floats + idx];
    epilogue_store(p, ti.batch, ti.tap, m, n, v, true);
  }
}

// ---------------------------------------------------------------- host dispatch
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
    const char* e = getenv("VLFB_TMA");
    if (e && atoi(e) == 0) fn = nullptr;
  }
  return fn;
}

// 3-D tensor map {K, rows, batch} of a dense K-major fp32 matrix; box = {32 floats (one 128-byte swizzle
// row), box_rows, 1}; out-of-range rows / K tail read as zeros.
static bool make_tmap(CUtensorMap* tm, const vlfb_operand_t& op, int rows, int K, int batch, int box_rows) {
  EncodeTiledFn enc = encode_fn();
  if (!enc || op.kind != VLFB_OP_DENSE_K || K < KC || rows < box_rows) return false;
  cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)rows, (cuuint64_t)(batch > 1 ? batch : 1)};
  cuuint64_t strides[2] = {(cuuint64_t)op.ld * 4,
                           (cuuint64_t)(batch > 1 ? op.batch_stride : (int64_t)rows * op.ld) * 4};
  if ((strides[0] & 15) || (strides[1] & 15) || strides[1] == 0) return false;
  cuuint32_t box[3] = {(cuuint32_t)KC, (cuuint32_t)box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  return enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(op.ptr), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// 5-D im2col map of an NDHWC fp32 tensor [N, D, H, W, C]: `pixels` window origins x 32 channels per copy.
// lower/upper = bounding-box corners {W, H, D}; strides = traversal strides {W, H, D}.
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);
static bool make_tmap_im2col(CUtensorMap* tm, const float* base, int N, int D, int H, int W, int C, const int lower[3],
                             const int upper[3], const int strides[3], int pixels) {
  static EncodeIm2colFn enc = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (encode_fn() && cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      enc = reinterpret_cast<EncodeIm2colFn>(ptr);
  }
  if (!enc || (C % KC) != 0 || (reinterpret_cast<uintptr_t>(base) & 15)) return false;
  for (int i = 0; i < 3; ++i)
    if (lower[i] < -16 || lower[i] > 15 || upper[i] < -16 || upper[i] > 15 || strides[i] < 1 || strides[i] > 8) return false;
  cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)D, (cuuint64_t)N};
  cuuint64_t gstr[4] = {(cuuint64_t)C * 4, (cuuint64_t)C * 4 * W, (cuuint64_t)C * 4 * W * H, (cuuint64_t)C * 4 * W * H * D};
  cuuint32_t estr[5] = {1, (cuuint32_t)strides[0], (cuuint32_t)strides[1], (cuuint32_t)strides[2], 1};
  return enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, const_cast<float*>(base), dims, gstr, lower, upper,
             (cuuint32_t)KC, (cuuint32_t)pixels, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// conv1 stem (C padded to 4, 16-byte pixels): overlapping-window view of a clip whose rows are stored with `pitch`
// >= pW + W + right pad pixels, the pad pixels zero.  dim0 = the 8 px x 4 ch = 32 floats of one filter row starting
// at padded pixel wo * sW (i.e. real pixel wo * sW - pW), dim1 = wo (stride sW pixels: consecutive windows OVERLAP),
// dim2 / dim3 = input row / frame (their out-of-range coordinates read as zeros = the H / T padding), dim4 = clip.
// One box = 16 consecutive output positions of one output row.
static bool make_tmap_stem(CUtensorMap* tm, const float* ptr, const vlfb_conv_geom_t& g, int64_t pitch, int box_rows = 1) {
  EncodeTiledFn enc = encode_fn();
  if (!enc || g.C != 4 || (g.Wo & 15) || g.dT != 1 || g.dH != 1 || g.dW != 1 || g.kW > 8) return false;
  if (pitch < g.pW + g.W || pitch < (int64_t)(g.Wo - 1) * g.sW + 8 || (reinterpret_cast<uintptr_t>(ptr) & 15)) return false;
  const float* base = ptr - (int64_t)g.pW * 4;                     // padded pixel 0 of row 0
  cuuint64_t dims[5] = {32, (cuuint64_t)g.Wo, (cuuint64_t)g.H, (cuuint64_t)g.T, (cuuint64_t)g.N};
  cuuint64_t gstr[4] = {(cuuint64_t)g.sW * 16, (cuuint64_t)pitch * 16, (cuuint64_t)pitch * 16 * g.H,
                        (cuuint64_t)pitch * 16 * g.H * g.T};
  // box_rows > 1: that many input rows `sH` apart (= consecutive OUTPUT rows) in one box: boxDim = rows * stride with
  // elementStride = stride loads ceil(boxDim / stride) = rows elements (cuTensorMapEncodeTiled)
  cuuint32_t box[5] = {32, 16, (cuuint32_t)(box_rows > 1 ? box_rows * g.sH : 1), 1, 1};
  cuuint32_t estr[5] = {1, 1, (cuuint32_t)(box_rows > 1 ? g.sH : 1), 1, 1};
  if (box[2] > 256 || estr[2] > 8) return false;
  return enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, const_cast<float*>(base), dims, gstr, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// tuning overrides, read once (scripts/tune_gemm.py); the per-call fields of vlfb_gemm_params_t take precedence
struct Env { int bn, stages, lag, sk, debug, no_patch, no_par; bool im2col; };
static Env read_env() {
  Env e;
  auto geti = [](const char* name, int dflt) { const char* v = getenv(name); return v ? atoi(v) : dflt; };
  e.bn = geti("VLFB_BN", 0);
  e.stages = geti("VLFB_STAGES", 0);
  e.lag = geti("VLFB_LAG", 0);
  e.sk = geti("VLFB_SK", 0);
  e.debug = geti("VLFB_DEBUG", 0);
  e.no_patch = geti("VLFB_NO_PATCH", 0);
  e.no_par = geti("VLFB_NO_PAR", 0);
  e.im2col = geti("VLFB_IM2COL", 1) != 0;
  return e;
}
static const Env& env() {
  static const Env e = read_env();
  return e;
}

// ---- plan: tile width x schedule, chosen together by a cycle model of one SM -----------------------------------
// A K chunk (32 fp32 of K) of a 128 x bn tile costs max(tensor pipe, operand delivery):
//   tensor   = 128 x bn x 32 MACs / 1024 tf32 MAC/clk (dense H100 SM) = 4 bn clocks;
//   delivery = (128 + bn) x 128 B through the SM's L2 port at a model rate of 64 B/clk.
// A wide chunk (64 x 2 bn, Launch::wide) issues the MMAs of a 128 x bn one and delivers (64 + 2 bn) x 128 B, plus a
// fixed latency the two terms leave out: the consumers' rewrite of the stage tiles between two 256-thread barriers.
// (Fitted to the Co = 64 wgrads of the benchmarked network, that term is worth 20-200 model clocks; with it a wide
// launch takes the wider tile when both widths pad N alike.)
// A tile adds a fixed fill + epilogue cost (~8 chunks' worth); a stream-K launch adds the fix-up of the shared tiles.
// A split-TF32 chunk (x3) issues three times the MMAs and adds the consumers' lo-image pass: the chunk's operand bytes
// read and written once through shared memory (128 B/clk) between two barriers (the same fixed latency as a wide rewrite).
// The constants rank tile widths against each other; they are model values, not measurements.
static double chunk_cost(int bn, bool wide, bool x3 = false) {
  const double tensor = (x3 ? 12.0 : 4.0) * bn;
  const double port = (wide ? 128.0 * (WM + 2 * bn) : 16384.0 + 128.0 * bn) / 64.0;
  const double lo = x3 ? 2.0 * (wide ? WM + 2 * bn : BM + bn) + (wide ? 0.0 : 128.0) : 0.0;
  return (tensor > port ? tensor : port) + (wide ? 128.0 : 0.0) + lo;
}

// Pipeline stages that fit shared memory next to the epilogue staging, the K-major images of MN-major operands (A, 2 x B;
// a wide launch keeps them in the epilogue staging) and, split-TF32, the lo images (2 x (A + B)); at most 6.
static int fit_stages(int bn, bool wide, bool ta, bool tb, bool x3) {
  const int a_tile_bytes = (wide ? WM : BM) * KC * 4, b_tile_bytes = (bn << (wide ? 1 : 0)) * KC * 4;
  const int stage_bytes = a_tile_bytes + b_tile_bytes;
  const int img_bytes = wide ? 0 : (ta ? a_tile_bytes : 0) + (tb ? 2 * b_tile_bytes : 0);
  const int lo_bytes = x3 ? 2 * stage_bytes : 0;
  const int s = (227 * 1024 - EPI_STAGE_BYTES - img_bytes - lo_bytes - 2048) / stage_bytes;
  return s > 6 ? 6 : s;
}

// Wide tiles: both operands MN-major (their K-major images are built by the consumers, so the tile shape is free) and
// at most one wgmma M of rows.
static bool wide_tiles(const vlfb_gemm_params_t& p) {
  return is_mn(p.a.kind) && is_mn(p.b.kind) && p.M <= WM;
}

struct Plan { int bn, split_k, pair, sk; int tiles, units; double cost; };

// sk_ok = what the workspace allows; pow2_only: a 96-wide request becomes 64 (the cp.async MN-major loader, which
// stages every MN-major B, needs a power-of-two tile width).  p.pair is accepted and ignored: Hopper has no CTA-pair MMA (pair is always 0).
// Deterministic atomic launches (p.deterministic): no plain split-K and no atomic stream-K.  Their schedule is split 1 or
// stream-K with the workspace fix-up (pieces summed in piece order), the latter weighed by the cost model unless
// p.stream_k = -1, since it replaces the split-K that such a launch would otherwise take.
static Plan make_plan(const vlfb_gemm_params_t& p, int num_sms, bool sk_ok, bool pow2_only = false) {
  const int zbase = p.taps > 1 ? p.taps : p.batch;
  const bool atomic = (p.flags & VLFB_EPI_ATOMIC) != 0;
  const bool det = atomic && p.deterministic != 0;
  int want_bn = p.tile_n > 0 ? p.tile_n : env().bn;
  if (want_bn > BN_MAX) want_bn = BN_MAX;                                      // wider requests get the widest tile
  if (pow2_only && want_bn == 96) want_bn = 64;                                // (the one width not a power of two)
  const int want_sk = p.stream_k != 0 ? p.stream_k : env().sk;
  // split-TF32: a width whose lo images would leave fewer than 3 stages is not planned; a narrower tile is
  const bool x3 = p.precision == VLFB_PREC_X3;
  const bool ta = is_mn(p.a.kind), tb = is_mn(p.b.kind);
  if (x3)
    while (want_bn > 32 && fit_stages(want_bn, wide_tiles(p), ta, tb, true) < 3) want_bn = want_bn == 96 ? 64 : want_bn / 2;
  Plan best, best_sk;
  best.cost = 1e30; best.bn = 32; best.split_k = p.split_k > 0 ? p.split_k : 1; best.pair = 0; best.sk = 0;
  best.tiles = 0; best.units = 0;
  best_sk = best;
  static const int kWidths[] = {128, 96, 64, 32};
  // Stream-K is opt-in (p.stream_k = 1, VLFB_SK): its fix-up pass costs more than it saves unless the tile count
  // leaves many SMs idle.
  const int U = num_sms;
  const bool wide = wide_tiles(p);
  for (int wi = 0; wi < 4; ++wi) {
    const int bn = kWidths[wi];
    const int tn = wide ? 2 * bn : bn;                                          // tile columns
    if (want_bn > 0 ? bn != want_bn : ((bn & (bn - 1)) != 0)) continue;       // 96 only on request
    if (want_bn <= 0 && bn > 32 && p.N <= tn / 2) continue;                   // do not pad N by 2x
    if (x3 && fit_stages(bn, wide, ta, tb, true) < 3) continue;
    const int tiles_m = wide ? 1 : ceil_div(p.M, BM);
    const int64_t T = (int64_t)tiles_m * ceil_div(p.N, tn) * zbase;
    const int nkt = ceil_div(p.K, KC);
    const double cc = chunk_cost(bn, wide, x3);
    const double fixed = 8.0 * cc;
    // (a) static tile loop, optional plain split-K (atomic epilogues only)
    const int smax = det ? 1 : p.split_k > 0 ? p.split_k : (atomic && p.K >= 512 ? (p.K / 256 < 128 ? p.K / 256 : 128) : 1);
    for (int sp = (p.split_k > 0 ? p.split_k : 1); sp <= smax; ++sp) {
      const int64_t tiles = T * sp;
      const double rounds = (double)((tiles + U - 1) / U);
      const double cost = rounds * (ceil_div(ceil_div(p.K, sp), KC) * cc + fixed);
      if (cost < best.cost * 0.999) {
        best.cost = cost; best.bn = bn; best.split_k = sp; best.pair = 0; best.sk = 0;
        best.tiles = (int)tiles; best.units = (int)(tiles < U ? tiles : U);
      }
    }
    // (b) stream-K: equal chunk ranges; shared tiles reduced through the workspace (or by atomics)
    const int64_t total = T * nkt;
    const bool sk_legal = (det ? sk_ok && want_sk >= 0 : (atomic ? p.split_k != 1 : (sk_ok && p.split_k <= 1)) && want_sk > 0) &&
                          nkt >= 2 && total >= 2 * (int64_t)U && T * (NEPI / 32) <= SK_CNT_INTS && U <= MAX_UNITS;
    if (sk_legal && (T % U) != 0) {
      const double per_unit = (double)((total + U - 1) / U);
      const double cost = per_unit * cc + fixed * (double)((T + U - 1) / U) + (atomic && !det ? 1.0 : 2.0) * fixed;
      if (cost < best_sk.cost * 0.999) {
        best_sk.cost = cost; best_sk.bn = bn; best_sk.split_k = 1; best_sk.pair = 0; best_sk.sk = 1;
        best_sk.tiles = (int)T; best_sk.units = U;
      }
    }
  }
  if (best_sk.cost < 1e29 && (want_sk > 0 || best_sk.cost < best.cost * 0.999)) return best_sk;
  return best;
}

// Chunk ranges of the stream-K units.  A boundary that would leave a piece of fewer than `minp` chunks at either end
// of a tile is moved onto the tile boundary.
static void make_bounds(int* b, int U, int64_t T, int nkt) {
  const int64_t total = T * nkt;
  const int minp = nkt >= 16 ? 4 : (nkt >= 8 ? 2 : 1);
  for (int u = 0; u <= U; ++u) {
    int64_t x = (int64_t)u * total / U;
    const int r = (int)(x % nkt);
    if (r && r < minp) x -= r;
    else if (r && nkt - r < minp) x += nkt - r;
    b[u] = (int)x;
  }
  b[0] = 0; b[U] = (int)total;
  bool ok = true;
  for (int u = 0; u < U; ++u) if (b[u + 1] <= b[u]) ok = false;
  if (!ok) for (int u = 0; u <= U; ++u) b[u] = (int)((int64_t)u * total / U);
}

size_t gemm_tc_workspace_bytes() {
  return (size_t)SK_CNT_INTS * 4 + (size_t)MAX_UNITS * 2 * BM * 256 * 4;
}

template <int AK, int BK, bool MASK, bool CP, bool FIX, bool X3>
static int launch_variant(const cudaLaunchConfig_t& cfg, const vlfb_gemm_params_t& p, const Launch& L, const CUtensorMap& tmA,
                          const CUtensorMap& tmB) {
  constexpr auto kernel = X3 ? gemm_tc3_kernel<AK, BK, MASK, CP, FIX> : gemm_tc_kernel<AK, BK, MASK, CP, FIX>;
  static bool attr_done = false;
  cudaError_t e;
  if (!attr_done) {
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(smem): %s", cudaGetErrorString(e));
      return VLFB_E_CUDA;
    }
    attr_done = true;
  }
  e = cudaLaunchKernelEx(&cfg, kernel, p, L, tmA, tmB);
  if (e != cudaSuccess) {
    set_error("gemm_tc launch: %s", cudaGetErrorString(e));
    return VLFB_E_CUDA;
  }
  VLFB_CHECK_LAUNCH();
  return VLFB_OK;
}

template <int AK, int BK, bool MASK>
int launch(const vlfb_gemm_params_t& p_in, cudaStream_t stream) {
  vlfb_gemm_params_t p = p_in;       // split_k == 0 is resolved below
  Launch L;
  memset(&L, 0, sizeof(L));
  L.out.w = make_fastdiv(p.g.Wo);
  L.out.h = make_fastdiv(p.g.Ho);
  L.out.t = make_fastdiv(p.g.To);
  L.in.w = make_fastdiv(p.g.W);
  L.in.h = make_fastdiv(p.g.H);
  L.in.t = make_fastdiv(p.g.T);
  L.cdiv = make_fastdiv(p.g.C);
  L.kwdiv = make_fastdiv(p.g.kW);
  static int num_sms = 0;
  if (num_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || num_sms <= 0) num_sms = 132;
    if (num_sms > MAX_UNITS) num_sms = MAX_UNITS;
  }
  const Env& ev = env();
  const vlfb_conv_geom_t& g = p.g;
  const bool unit_dgrad = g.sT == 1 && g.sH == 1 && g.sW == 1;
  bool sk_ws = p.workspace != nullptr && p.workspace_bytes >= gemm_tc_workspace_bytes() &&
                     (reinterpret_cast<uintptr_t>(p.workspace) & 15) == 0;
  alignas(64) CUtensorMap tmA, tmB;
  // Strided dgrad as parity classes (see Launch::par): needs whole strides in H / W, unit temporal stride and dilation,
  // both operands addressable by TMA, the lean epilogue (16-byte rows, whole 16-column blocks), and one im2col origin
  // offset shared by all classes that have taps (true for the networks' 3x3 / pad 1 and 1x1 / pad 0 stride-2 layers).
  int par_lo[3] = {0, 0, 0}, par_hi[3] = {0, 0, 0};
  if (AK == VLFB_OP_DGRAD_K && BK == VLFB_OP_DENSE_K && !unit_dgrad && !ev.no_par && ev.im2col && encode_fn() != nullptr &&
      g.sT == 1 && g.sH <= 2 && g.sW <= 2 && g.dT == 1 && g.dH == 1 && g.dW == 1 && (g.H % g.sH) == 0 && (g.W % g.sW) == 0 &&
      (g.Co % KC) == 0 && p.batch == 1 && p.taps <= 1 && p.split_k == 1 && !p.row_scale && !(p.flags & VLFB_EPI_ATOMIC) &&
      (p.N & 15) == 0 && (p.ldd & 3) == 0 && (reinterpret_cast<uintptr_t>(p.d) & 15) == 0 &&
      (!p.residual || ((reinterpret_cast<uintptr_t>(p.residual) & 15) == 0 && !(p.flags & VLFB_EPI_ACCUM))) &&
      !p.relu_mask && (!p.relu_mask_bits || (p.ldd & 15) == 0)) {
    const int Hs = g.H / g.sH, Ws = g.W / g.sW;
    bool ok = true, have_lo = false;
    int ncls = 0;
    ParCls cls[4];
    for (int ph = 0; ph < g.sH; ++ph)
      for (int pw = 0; pw < g.sW; ++pw) {
        ParCls c;
        c.ph = (short)ph; c.pw = (short)pw;
        c.rh = (short)((ph + g.pH) % g.sH); c.rw = (short)((pw + g.pW) % g.sW);
        c.nh = (short)(c.rh < g.kH ? (g.kH - 1 - c.rh) / g.sH + 1 : 0);
        c.nw = (short)(c.rw < g.kW ? (g.kW - 1 - c.rw) / g.sW + 1 : 0);
        if (c.nh == 0 || c.nw == 0) c.nh = c.nw = 0;
        c.nk = g.kT * c.nh * c.nw * (g.Co / KC);
        if (c.nk) {
          const int lw = (pw + g.pW) / g.sW - (c.nw - 1), lh = (ph + g.pH) / g.sH - (c.nh - 1);
          if (have_lo && (lw != par_lo[0] || lh != par_lo[1])) ok = false;
          par_lo[0] = lw; par_lo[1] = lh; have_lo = true;
        }
        cls[ncls++] = c;
      }
    if (ok && have_lo && (int64_t)g.N * g.T * Hs * Ws < (1ll << 31)) {
      // heaviest classes first: the static tile loop hands tiles out round-robin
      for (int i = 0; i < ncls; ++i)
        for (int j = i + 1; j < ncls; ++j)
          if (cls[j].nk > cls[i].nk) { const ParCls t = cls[i]; cls[i] = cls[j]; cls[j] = t; }
      L.par = ncls;
      L.par_m = g.N * g.T * Hs * Ws;
      L.par_lo[0] = par_lo[0]; L.par_lo[1] = par_lo[1];
      for (int i = 0; i < ncls; ++i) L.par_cls[i] = cls[i];
      L.sub.w = make_fastdiv(Ws); L.sub.h = make_fastdiv(Hs); L.sub.t = make_fastdiv(g.T);
      par_lo[2] = g.pT - (g.kT - 1);
      par_hi[0] = par_lo[0] + Ws - g.Wo; par_hi[1] = par_lo[1] + Hs - g.Ho; par_hi[2] = par_lo[2] + g.T - g.To;
      sk_ws = false;
    }
  }
  L.wide = wide_tiles(p) ? 1 : 0;
  const bool det = (p.flags & VLFB_EPI_ATOMIC) && p.deterministic;
  // a deterministic atomic launch whose operands are both MN-major may run its fix-ups in the cp.async build
  constexpr bool cp_fix = is_mn(AK) && is_mn(BK) && !MASK;
  Plan plan;
  // MN-major operands have no tensor map (sm_90 has no swizzle mode for their atom layout): the cp.async loaders stage
  // them, and the MN-major B loader needs a power-of-two tile width
  constexpr bool pow2_only = is_mn(BK);
  for (int attempt = 0; attempt < 4; ++attempt) {
    if (L.par) {                       // plan for the class sub-problems: M' rows, one z slice per class
      vlfb_gemm_params_t pp = p;
      pp.M = L.par_m; pp.batch = L.par; pp.K = L.par_cls[0].nk * KC;
      plan = make_plan(pp, num_sms, false, pow2_only);
      plan.split_k = 1;
    } else {
      plan = make_plan(p, num_sms, sk_ws, pow2_only);
    }
    L.bn = plan.bn;
    p.split_k = plan.split_k;
    memset(&tmA, 0, sizeof(tmA));
    memset(&tmB, 0, sizeof(tmB));
    L.tma_a = AK == VLFB_OP_DENSE_K && make_tmap(&tmA, p.a, p.M, p.K, p.batch, BM) ? 1 : 0;
    L.tma_b = BK == VLFB_OP_DENSE_K && make_tmap(&tmB, p.b, p.N, p.K, p.batch, L.bn) ? 1 : 0;
    if (ev.im2col) {
      // conv gathers as TMA im2col copies: one instruction per K chunk instead of 1024 16-byte cp.asyncs
      const int pad_lo[3] = {-g.pW, -g.pH, -g.pT};
      const int pad_hi[3] = {g.pW - (g.kW - 1) * g.dW, g.pH - (g.kH - 1) * g.dH, g.pT - (g.kT - 1) * g.dT};
      const int cstr[3] = {g.sW, g.sH, g.sT};
      const int ones[3] = {1, 1, 1};
      if (AK == VLFB_OP_CONV_K &&
          make_tmap_im2col(&tmA, p.a.ptr, g.N, g.T, g.H, g.W, g.C, pad_lo, pad_hi, cstr, BM))
        L.tma_a = 2;
      if (AK == VLFB_OP_DGRAD_K && unit_dgrad) {
        const int lo[3] = {g.pW - (g.kW - 1) * g.dW, g.pH - (g.kH - 1) * g.dH, g.pT - (g.kT - 1) * g.dT};
        const int hi[3] = {-g.pW, -g.pH, -g.pT};
        if (make_tmap_im2col(&tmA, p.a.ptr, g.N, g.To, g.Ho, g.Wo, g.Co, lo, hi, ones, BM))
          L.tma_a = 2;
      }
      if (AK == VLFB_OP_DGRAD_K && L.par) {
        if (L.tma_b && make_tmap_im2col(&tmA, p.a.ptr, g.N, g.To, g.Ho, g.Wo, g.Co, par_lo, par_hi, ones, BM))
          L.tma_a = 2;
        else { L.par = 0; continue; }   // not addressable: plan again for the cp.async gather path (any geometry)
      }
      if (AK == VLFB_OP_STEM_K && p.a.ld > 0) {
        // patch tiles need the lean epilogue's row mapping: a TMA-only build (B by TMA too: a cp.async build stores
        // through the general epilogue, which maps tile rows linearly), whole 16-column blocks, 16-byte addressable
        // rows, no mask
        const bool fast_ok = L.tma_b && (p.N & 15) == 0 && (p.ldd & 3) == 0 && (p.d_batch_stride & 3) == 0 && (p.d_tap_stride & 3) == 0 &&
                             (reinterpret_cast<uintptr_t>(p.d) & 15) == 0 && !p.relu_mask && !MASK &&
                             (!p.residual || ((reinterpret_cast<uintptr_t>(p.residual) & 15) == 0 && !(p.flags & VLFB_EPI_ACCUM)));
        L.stem_patch = 0;
        if (fast_ok && (g.Ho & 7) == 0 && (g.Wo & 15) == 0 && !ev.no_patch &&
            make_tmap_stem(&tmA, p.a.ptr, g, p.a.ld, 8)) {
          L.tma_a = 3;
          L.stem_patch = 1;
          L.patch_wb = g.Wo / 16;
          L.patch_hb = g.Ho / 8;
        } else if (make_tmap_stem(&tmA, p.a.ptr, g, p.a.ld)) {
          L.tma_a = 3;
        }
      }
    }
    const bool fixup = plan.sk && (!(p.flags & VLFB_EPI_ATOMIC) || det);
    if (!fixup || (L.tma_a && L.tma_b) || (cp_fix && det)) break;
    sk_ws = false;                     // an operand fell back to cp.async: plan again without fix-ups
  }
  const int zbase = L.par ? L.par : (p.taps > 1 ? p.taps : p.batch);
  L.tiles_m = L.wide ? 1 : ceil_div(L.par ? L.par_m : p.M, BM);
  L.tiles_n = ceil_div(p.N, L.bn << L.wide);
  L.total_tiles = (int)((int64_t)L.tiles_m * L.tiles_n * zbase * p.split_k);
  // (the kernel computes the same stage layout)
  const int a_tile_bytes = (L.wide ? WM : BM) * KC * 4, b_tile_bytes = (L.bn << L.wide) * KC * 4;
  const int stage_bytes = a_tile_bytes + b_tile_bytes;
  // K-major images: A, 2 x B; a wide launch keeps them in the epilogue staging tiles.  Split TF32: 2 x (A + B) lo images.
  const bool x3 = p.precision == VLFB_PREC_X3;
  const int img_bytes = L.wide ? 0 : (is_mn(AK) ? a_tile_bytes : 0) + (is_mn(BK) ? 2 * b_tile_bytes : 0);
  const int lo_bytes = x3 ? 2 * stage_bytes : 0;
  L.stages = fit_stages(L.bn, L.wide != 0, is_mn(AK), is_mn(BK), x3);
  if (x3 && L.bn == BN_MAX) {          // make_plan rules it out (2 stages at most): the split builds have no such K loop
    set_error("gemm_tc: split-TF32 launch planned at tile width %d", L.bn);
    return VLFB_E_UNSUPPORTED;
  }
  if (ev.stages >= 3 && ev.stages <= L.stages) L.stages = ev.stages;
  // The consumers release chunk c's stage after they have waited for chunk c + 1, and a cp.async producer publishes
  // chunk c only after the free-stage wait of chunk c + lag - stages.  lag <= stages - 2 keeps that wait behind a
  // release that does not depend on chunk c itself (no cycle); stages >= 3 always (the smem budget above gives >= 3).
  L.lag = L.stages - 2 < 2 ? L.stages - 2 : 2;
  if (ev.lag >= 1 && ev.lag <= L.stages - 2 && ev.lag <= 5) L.lag = ev.lag;
  const int cap = num_sms;
  int units = L.total_tiles < cap ? L.total_tiles : cap;
#ifdef VLFB_TRACE
  L.trace = g_trace_buf;
#endif
  L.sk = 0;
  if (plan.sk) {
    L.sk = 1;
    L.nkt = ceil_div(p.K, KC);
    units = cap;
    make_bounds(L.bounds, units, (int64_t)L.total_tiles, L.nkt);
    if (!(p.flags & VLFB_EPI_ATOMIC) || det) {
      L.ws_cnt = reinterpret_cast<int*>(p.workspace);
      L.ws_tiles = reinterpret_cast<float*>(reinterpret_cast<char*>(p.workspace) + (size_t)SK_CNT_INTS * 4);
    }
  }
  const int smem = L.stages * stage_bytes + img_bytes + lo_bytes + EPI_STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
  const bool cp = is_mn(AK) || is_mn(BK) || !(L.tma_a && L.tma_b);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)units);
  cfg.blockDim = dim3((unsigned)((cp ? NPROD : NPROD_TMA) + NEPI));
  cfg.dynamicSmemBytes = (size_t)smem;
  cfg.stream = stream;
  // ReLU sign bits are emitted by the lean epilogue; any other path writes them in a second pass over the dense output
  const bool lean = !cp && (p.ldd & 3) == 0 && (p.N & 15) == 0 && span32_ok(p) && (reinterpret_cast<uintptr_t>(p.d) & 15) == 0 &&
                    (!p.residual || ((reinterpret_cast<uintptr_t>(p.residual) & 15) == 0 && !(p.flags & VLFB_EPI_ACCUM)));
  uint32_t* bits_after = nullptr;
  if (p.relu_bits_out && (!lean || MASK)) { bits_after = p.relu_bits_out; p.relu_bits_out = nullptr; }
  // VLFB_DEBUG: one record per launch, space-separated key=value (tests/gemm_paths.py parses it; keep the keys stable)
  if (ev.debug)
    fprintf(stderr, "vlfb gemm_tc: kinds=%d,%d mask=%d M=%d N=%d K=%d z=%d bn=%d sk=%d split=%d tiles=%d units=%d stages=%d "
            "lag=%d tma=%d,%d cap=%d patch=%d par=%d cp=%d fix=%d lean=%d bits2=%d wide=%d det=%d prec=%d\n",
            AK, BK, MASK ? 1 : 0, p.M, p.N, p.K, zbase, L.bn, L.sk, p.split_k, L.total_tiles, units, L.stages, L.lag, L.tma_a,
            L.tma_b, cap, L.stem_patch, L.par, cp ? 1 : 0, L.ws_tiles != nullptr ? 1 : 0, lean ? 1 : 0, bits_after ? 1 : 0,
            L.wide, det ? 1 : 0, x3 ? 1 : 0);
  int rc = VLFB_OK;
  // (cp.async fix-ups exist only in the MN x MN builds, for deterministic atomic launches: the planning loop above
  // gives any other cp.async launch no workspace)
  if (cp && L.ws_tiles) {
    if constexpr (cp_fix) {
      rc = x3 ? launch_variant<AK, BK, MASK, true, true, true>(cfg, p, L, tmA, tmB)
              : launch_variant<AK, BK, MASK, true, true, false>(cfg, p, L, tmA, tmB);
      if (rc == VLFB_OK) {
        launch_k(gemm_fixup_kernel, dim3((unsigned)L.total_tiles), 256, 0, stream, p, L);
        VLFB_CHECK_LAUNCH();
      }
    } else {
      set_error("gemm_tc: stream-K fix-up planned for a cp.async build without one (kinds %d, %d)", AK, BK);
      return VLFB_E_UNSUPPORTED;
    }
  } else if (cp) {
    rc = x3 ? launch_variant<AK, BK, MASK, true, false, true>(cfg, p, L, tmA, tmB)
            : launch_variant<AK, BK, MASK, true, false, false>(cfg, p, L, tmA, tmB);
  } else if constexpr (!is_mn(AK) && !is_mn(BK)) {       // TMA-only builds exist for K-major pairs only
    if (L.ws_tiles) rc = x3 ? launch_variant<AK, BK, MASK, false, true, true>(cfg, p, L, tmA, tmB)
                            : launch_variant<AK, BK, MASK, false, true, false>(cfg, p, L, tmA, tmB);
    else rc = x3 ? launch_variant<AK, BK, MASK, false, false, true>(cfg, p, L, tmA, tmB)
                 : launch_variant<AK, BK, MASK, false, false, false>(cfg, p, L, tmA, tmB);
  }
  if (rc == VLFB_OK && bits_after) rc = relu_bits(p.d, bits_after, (int64_t)p.M * p.N, stream);
  return rc;
}

}  // namespace tc

void gemm_tc_plan(const vlfb_gemm_params_t& p, int num_sms, vlfb_gemm_plan_t* out) {
  // host-only view of the plan
  bool sk_ws = p.workspace != nullptr && p.workspace_bytes >= tc::gemm_tc_workspace_bytes();
  const tc::Plan pl = tc::make_plan(p, num_sms, sk_ws);
  out->tile_n = pl.bn; out->split_k = pl.split_k; out->pair = pl.pair; out->stream_k = pl.sk;
  out->tiles = pl.tiles; out->units = pl.units;
}

size_t gemm_tc_workspace_bytes() { return tc::gemm_tc_workspace_bytes(); }
float* gemm_tc_partials(void* workspace, size_t workspace_bytes, size_t* floats) {
  const size_t head = (size_t)tc::SK_CNT_INTS * 4;
  *floats = workspace && workspace_bytes > head ? (workspace_bytes - head) / 4 : 0;
  return *floats ? reinterpret_cast<float*>(static_cast<char*>(workspace) + head) : nullptr;
}
#ifdef VLFB_TRACE
void gemm_tc_set_trace(void* buf) { tc::g_trace_buf = reinterpret_cast<unsigned long long*>(buf); }
#endif

int gemm_tc(const vlfb_gemm_params_t& p, cudaStream_t stream) {
  const int ak = p.a.kind, bk = p.b.kind;
  if (p.relu_mask || p.relu_mask_bits) {
    // ReLU-backward mask: only the dgrad shapes need it (two more instantiations, not eighteen)
    if (ak == VLFB_OP_DGRAD_K && bk == VLFB_OP_DENSE_K) return tc::launch<VLFB_OP_DGRAD_K, VLFB_OP_DENSE_K, true>(p, stream);
    if (ak == VLFB_OP_DENSE_K && bk == VLFB_OP_DENSE_K) return tc::launch<VLFB_OP_DENSE_K, VLFB_OP_DENSE_K, true>(p, stream);
    set_error("vlfb_gemm: relu_mask is supported for DGRAD_K/DENSE_K x DENSE_K operands only (tensor-core engine)");
    return VLFB_E_BADARG;
  }
#define VLFB_TC_CASE(A, B) if (ak == A && bk == B) return tc::launch<A, B, false>(p, stream)
  VLFB_TC_CASE(VLFB_OP_CONV_K, VLFB_OP_DENSE_K);
  VLFB_TC_CASE(VLFB_OP_STEM_K, VLFB_OP_DENSE_K);
  VLFB_TC_CASE(VLFB_OP_DGRAD_K, VLFB_OP_DENSE_K);
  VLFB_TC_CASE(VLFB_OP_DENSE_MN, VLFB_OP_CONV_MN);
  VLFB_TC_CASE(VLFB_OP_DENSE_MN, VLFB_OP_STEM_MN);
  VLFB_TC_CASE(VLFB_OP_DENSE_K, VLFB_OP_DENSE_K);
  VLFB_TC_CASE(VLFB_OP_DENSE_K, VLFB_OP_DENSE_MN);
  VLFB_TC_CASE(VLFB_OP_DENSE_MN, VLFB_OP_DENSE_K);
  VLFB_TC_CASE(VLFB_OP_DENSE_MN, VLFB_OP_DENSE_MN);
#undef VLFB_TC_CASE
  set_error("gemm_tc: unsupported operand kinds (%d, %d)", ak, bk);
  return VLFB_E_UNSUPPORTED;
}

}  // namespace vlfb
