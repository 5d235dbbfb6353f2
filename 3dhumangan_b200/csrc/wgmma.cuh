// sm_90a primitives shared by every tensor-core kernel in this library: mbarrier, bulk-copy (TMA engine, 1-D),
// warpgroup MMA (wgmma) with register accumulators, and the 128B-swizzled K-major operand layout.
//
// Operand layout (both A and B): "K-major, SWIZZLE_128B" canonical wgmma layout.  A tile of
// R rows x 64 bf16 (= 128 B per row) is stored as R/8 groups of 8 rows; a group is 1024 B; inside
// a group row r (0..7) occupies 128 B and its 16-byte chunk c (0..7) sits at chunk slot (c ^ r).
//     byte(r, k) = (r/8)*1024 + (r%8)*128 + (((k/8) ^ (r%8)) * 16) + (k%8)*2          (k < 64)
// Matrix descriptor: start>>4, LBO=1 (ignored for swizzled K-major), SBO=1024>>4, base_offset=0,
// layout=SWIZZLE_128B(1).  One wgmma consumes K=16 (32 B): advance the start address by 32 B.
// The swizzle is a function of the absolute shared-memory address bits: tiles are 1024-byte aligned, and a descriptor may
// start at any whole 128-byte row of such a tile (the haloed convolutions address their filter taps that way).
//
// Accumulators: a warpgroup (4 consecutive warps, 128 threads) owns an M = 64 row block.  For m64nNk16 with fp32
// accumulation, thread t = 32 w + l of the warpgroup holds d[4 j + 2 i + e] = D[16 w + l/4 + 8 i][8 j + 2 (l%4) + e]
// (i, e in {0, 1}, j < N/8): see frag_row / frag_col.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace hg {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// latency-critical waits: plain try_wait loop
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// waits that are expected to block for a while: a short sleep between polls frees issue slots for the other warps
// on the same scheduler
__device__ __forceinline__ void mbar_wait_sleep(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) __nanosleep(32);
}
// producer threads run far ahead of their consumers: back off between polls so that their spin loops do not steal
// issue slots from the warps that do the arithmetic
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) __nanosleep(128);
}

// ---------------------------------------------------------------- named barriers
// bar.sync id, n: ids 1..15 (0 is __syncthreads); n a multiple of 32
__device__ __forceinline__ void named_barrier(uint32_t id, uint32_t n) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory");
}

// ---------------------------------------------------------------- register budget per warpgroup
// A CTA of three warpgroups (two MMA warpgroups + one producer warpgroup) is compiled for 168 registers per thread; the
// producer group gives most of its share to the MMA groups, whose [64 x 256] fp32 accumulators take 128 registers alone.
// Executed by every warp of a warpgroup.
template <uint32_t kRegs>
__device__ __forceinline__ void regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs)); }
template <uint32_t kRegs>
__device__ __forceinline__ void regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs)); }
constexpr uint32_t kMmaRegs = 232, kProducerRegs = 40;     // 2 x 128 x 232 + 128 x 40 <= 65536

// ---------------------------------------------------------------- explicit shared-space accesses
// (pointers that went through integer alignment arithmetic compile to GENERIC LD/ST, which cost extra
//  latency on the hot operand paths; these keep them LDS/STS)
__device__ __forceinline__ float lds_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}
// Operand-tile store: volatile but WITHOUT a "memory" clobber (which serialised every 8-element group behind the previous
// store); ordering against the consumers comes from fence_proxy_async_smem().
__device__ __forceinline__ void sts_b32x4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d));
}
// Makes the compiler forget what it knows about a register: loads whose address derives from it cannot be
// hoisted above this point (used after a barrier / table refresh in front of NON-volatile table loads).
__device__ __forceinline__ void opaque(uint32_t& r) { asm volatile("" : "+r"(r)); }
// 8 consecutive fp32 entries of a read-mostly shared-memory TABLE (two LDS.128), non-volatile so that they can be batched;
// callers pass an address made `opaque` after the last point at which the table may have changed.
__device__ __forceinline__ void lds8(uint32_t a, float (&o)[8]) {
  float4 x, y;
  asm("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(x.x), "=f"(x.y), "=f"(x.z), "=f"(x.w) : "r"(a));
  asm("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(y.x), "=f"(y.y), "=f"(y.z), "=f"(y.w) : "r"(a + 16));
  o[0] = x.x; o[1] = x.y; o[2] = x.z; o[3] = x.w;
  o[4] = y.x; o[5] = y.y; o[6] = y.z; o[7] = y.w;
}

// One fp32 entry of such a table (same contract as lds8).
__device__ __forceinline__ float lds1(uint32_t a) {
  float v;
  asm("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a));
  return v;
}

// ---------------------------------------------------------------- proxies / fences
// generic-proxy writes (st.shared) -> visible to the async proxy (wgmma operand reads / bulk copies)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---------------------------------------------------------------- bulk copy global -> shared (TMA engine, 1-D)
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---------------------------------------------------------------- warpgroup MMA
// K-major (or, for an MN-major B of 64 columns, MN-major) SW128 matrix descriptor for a tile whose 8-row groups are
// 1024 B apart.
__device__ __forceinline__ uint64_t wg_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);  // start address
  d |= static_cast<uint64_t>(1) << 16;                    // LBO (unused for swizzled K-major)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;            // SBO: 8 rows * 128 B
  d |= static_cast<uint64_t>(1) << 62;                    // SWIZZLE_128B
  return d;
}

// D[64 x N] (+)= A[64 x 16] . B[N x 16]^T with A, B read from shared memory through descriptors; kTransB = 1 reads B
// MN-major.  Issued by all 128 threads of a warpgroup; completes asynchronously (wgmma_commit / wgmma_wait).
template <int N, int kTransB = 0>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t accumulate);

// The accumulator operands of m64nNk16 (N/2 fp32 registers per thread) as asm operand lists.
#define HG_ACC4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define HG_ACC16(i) HG_ACC4(i), HG_ACC4(i + 4), HG_ACC4(i + 8), HG_ACC4(i + 12)
#define HG_ACC32 HG_ACC16(0), HG_ACC16(16)
#define HG_ACC64 HG_ACC32, HG_ACC16(32), HG_ACC16(48)
#define HG_ACC128 HG_ACC64, HG_ACC16(64), HG_ACC16(80), HG_ACC16(96), HG_ACC16(112)
#define HG_REGS32 \
  "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
  "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
#define HG_REGS64 \
  HG_REGS32 ", %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, " \
  "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define HG_REGS128 \
  HG_REGS64 ", %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, " \
  "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, " \
  "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, " \
  "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
// kN, kTransB, accumulator registers, the operand index of the first descriptor ("%<n>") and of the scale-d flag
#define HG_WGMMA(kN, kTransB, NREG, REGS, ACC, DA, FLAG)                                                        \
  template <>                                                                                                 \
  __device__ __forceinline__ void wgmma_bf16<kN, kTransB>(float (&d)[NREG], uint64_t da, uint64_t db,          \
                                                          uint32_t accumulate) {                              \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, " FLAG ", 0;\n\t"                                     \
                 "wgmma.mma_async.sync.aligned.m64n" #kN "k16.f32.bf16.bf16 {" REGS "}, " DA ", p, 1, 1, 0, " #kTransB \
                 ";\n\t}"                                                                                    \
                 : ACC                                                                                        \
                 : "l"(da), "l"(db), "r"(accumulate));                                                        \
  }
HG_WGMMA(64, 0, 32, HG_REGS32, HG_ACC32, "%32, %33", "%34")
HG_WGMMA(128, 0, 64, HG_REGS64, HG_ACC64, "%64, %65", "%66")
HG_WGMMA(256, 0, 128, HG_REGS128, HG_ACC128, "%128, %129", "%130")
HG_WGMMA(64, 1, 32, HG_REGS32, HG_ACC32, "%32, %33", "%34")
#undef HG_WGMMA

// Orders this warpgroup's register / shared-memory accesses before the wgmma that follows.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// Waits until at most kPending committed groups of this warpgroup are still in flight.
template <int kPending>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory");
}
// Keeps the compiler from moving accesses of the accumulator registers across wgmma_wait.
template <int kN>
__device__ __forceinline__ void acc_fence(float (&d)[kN]) {
#pragma unroll
  for (int i = 0; i < kN; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// One K-chunk of 64: four K=16 wgmmas.  a_tile: shared address of this warpgroup's [64 x 64] rows of a SW128 tile
// (1024-byte aligned or a whole row inside one); b_tile: the [N x 64] B tile (kTransB = 0).
template <int N>
__device__ __forceinline__ void wg_k64(float (&d)[N / 2], uint32_t a_tile, uint32_t b_tile, bool accumulate) {
  const uint64_t da = wg_desc_sw128(a_tile);
  const uint64_t db = wg_desc_sw128(b_tile);
#pragma unroll
  for (uint32_t k = 0; k < 4; ++k) {
    // +32 B per K=16 step inside the 128 B swizzle atom (address field is in 16 B units)
    wgmma_bf16<N>(d, da + 2 * k, db + 2 * k, (accumulate || k > 0) ? 1u : 0u);
  }
}

// Fragment coordinates of accumulator entry d[4 j + 2 i + e] for thread `t` (0..127) of the warpgroup.
__device__ __forceinline__ int frag_row(int t, int i) { return ((t >> 5) << 4) + ((t & 31) >> 2) + 8 * i; }
__device__ __forceinline__ int frag_col(int t, int j, int e) { return 8 * j + 2 * (t & 3) + e; }

// ---------------------------------------------------------------- operand packing
// byte offset of element (row, k) inside a [rows x 64] bf16 SW128 tile
__host__ __device__ __forceinline__ uint32_t sw128_offset(uint32_t row, uint32_t k) {
  return (row >> 3) * 1024u + (row & 7u) * 128u + ((((k >> 3) ^ row) & 7u) << 4) + ((k & 7u) << 1);
}

// split two fp32 into (hi, lo) bf16x2 pairs: x ~= hi + lo with |lo| <= 2^-9 |hi|.  The residual x - float(hi) is one FMA
// per value (hi * -1 + x: a single rounding, the same value as the subtraction), the unpack a shift and a mask.
__device__ __forceinline__ void split_bf16x2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  __nv_bfloat162 h = __floats2bfloat162_rn(x0, x1);
  const uint32_t hb = *reinterpret_cast<uint32_t*>(&h);
  const float2 hf = make_float2(__uint_as_float(hb << 16), __uint_as_float(hb & 0xffff0000u));
  const float2 r = ffma2(hf, make_float2(-1.f, -1.f), make_float2(x0, x1));
  __nv_bfloat162 l = __floats2bfloat162_rn(r.x, r.y);
  hi = hb;
  lo = *reinterpret_cast<uint32_t*>(&l);
}

// y[j] = LeakyReLU_slope(x[j] * g1[j] + g0[j]) for 8 values: max(v, slope * v) is the LeakyReLU for 0 <= slope <= 1 (0.2,
// the identity 1 and ReLU 0 are the slopes this library uses), bit-identical to the compare-and-select form for every
// finite and infinite v (and NaN stays NaN).
__device__ __forceinline__ void affine_lrelu8(const float* __restrict__ x, const float (&g1)[8], const float (&g0)[8], float slope,
                                              float (&y)[8]) {
  const float2 sl = make_float2(slope, slope);
#pragma unroll
  for (int j = 0; j < 8; j += 2) {
    const float2 v = ffma2(make_float2(x[j], x[j + 1]), make_float2(g1[j], g1[j + 1]), make_float2(g0[j], g0[j + 1]));
    const float2 s = fmul2(v, sl);
    y[j] = fmaxf(v.x, s.x);
    y[j + 1] = fmaxf(v.y, s.y);
  }
}

// Write 8 consecutive-k fp32 values (k0 % 8 == 0) of one row into the hi (and lo) operand tiles.
template <bool kSplit>
__device__ __forceinline__ void store_a8(uint8_t* tile_hi, uint8_t* tile_lo, uint32_t row, uint32_t k0,
                                         const float (&x)[8]) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) split_bf16x2(x[2 * i], x[2 * i + 1], h[i], l[i]);
  const uint32_t off = sw128_offset(row, k0);
  sts_b32x4(smem_u32(tile_hi) + off, h[0], h[1], h[2], h[3]);
  if (kSplit) sts_b32x4(smem_u32(tile_lo) + off, l[0], l[1], l[2], l[3]);
}

}  // namespace hg
