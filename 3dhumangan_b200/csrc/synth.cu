// SPADE synthesis backbone: one kernel launch per SPADE half-block
//     x_out = Conv1x1_SN( lrelu_0.2( BN(x) * (1 + gamma) + beta ) ) + b  [+ x_skip]  [-> ToRGB accumulate]
// (SPADE2d.forward lib/components/map3d_layers.py:176-190, SPADEBlock.forward :218-238,
//  ToRGB :346-352, SynthesisNetwork.forward lib/generators/map3d_generator.py:58-97.)
//
// Activations live in HBM as fp32 in a tile-blocked planar layout [B, T, C=256, 128] (T = ceil(HW/128)
// tiles of 128 consecutive pixels): the 128 KB a CTA reads / writes per tile are CONTIGUOUS, and every
// 32-channel slice of a tile is one contiguous 16 KB block (one cp.async.bulk).
//
// Per CTA (384 threads), persistent over tiles of 128 pixels of one image: warpgroup g (warps 4g..4g+3) builds the bf16
// hi/lo operand rows of pixels 64g..64g+63 (BN, SPADE modulation, LeakyReLU fused), issues their wgmmas ([64 x 256] fp32
// accumulator in registers) and runs the epilogue (bias, residual, ToRGB, next-BatchNorm statistics, plane stores); warps
// 8 and 9 stream the weights and the staging slices with cp.async.bulk.  The const-style forward's staging ring carries
// each tile's activation slices, then its residual slices, in the order the warpgroups take them, so the residual of an
// epilogue loads up to 5 slices ahead; the backward and the pixel-style kernel keep a separate residual ring streamed by
// warp 10 (one producer per ring, since a single producer of two rings couples them by program order and deadlocks).
//
// Two variants:
//   const-style : gamma/beta are per-sample vectors (blocks whose style map is spatially constant, 12 of 18
//                 half-blocks in 'mixed'/'isolated' mode).
//   pixel-style : gamma/beta come from a second GEMM on relu(bilinear_up(P_lr)) where
//                 P_lr = W_shared . feature_maps + b at RENDER resolution (W_shared commutes with the bilinear
//                 up-sample), so the 28x larger up-sampled style map of map3d_generator.py:244-245 is never
//                 materialised.  Per conv K chunk the [gamma | beta] GEMM of its 64 channels runs first (N = 128).
//
// The const-style kernel doubles as the library's blocked 1x1-convolution engine (runtime fields at the end of SpadeArgs):
// K of 64..512 input channels from one or two sources, LeakyReLU / sine / identity operand transform, and -- template
// flag kBwd -- the data-gradient form: the operand is the incoming gradient (optionally scaled per sample and channel),
// the weight image is W^T and the epilogue multiplies by the activation derivative rebuilt from the forward input that
// arrives through the residual ring, adds a rank-k term (the renderer's sigma / rgb heads) and accumulates the
// per-(sample, channel) sums the BatchNorm / FiLM gradients need (DESIGN.md "Backward").
//
// Ring protocol note: every consumer warp of a staging ring waits for and releases EVERY slice in order
// (see ring_take / ring_release).
#include "common.cuh"
#include "wgmma.cuh"

namespace hg {

constexpr int kC = 256;             // channels (hidden_dim == feature_dim == 256)
constexpr int kSynThreads = 384;
constexpr int kSynStages = 2;       // weight stages
constexpr int kASlots = 2;          // operand ring
constexpr int kXSlots = 5;          // const-style staging slots in total: forward, one ring of activation slices, each
                                    // tile's followed by its residual slices; backward, 3 activation + 2 residual slots
constexpr uint32_t kAChunk = 128 * 128;   // [128 x 64] bf16
constexpr uint32_t kBStage = 256 * 128;   // [256 x 64] bf16
constexpr uint32_t kXSlice = 32 * 128 * 4;  // 32 channels x 128 pixels fp32

struct SpadeArgs {
  const float* x;        // [B or 1, T, C, 128] tile-blocked
  long x_bstride;        // T*C*128, or 0 when x is shared by the whole batch (synthesis input)
  const float* mod;      // const-style: [B,2,C] (g1, g0): y = lrelu(x*g1 + g0)
  const float* scsh;     // pixel-style: [2,C] BN scale, shift
  const float* p_lr;     // pixel-style: [B, Rh*Rw, p_stride>=128] pre-activation of mlp_shared at render res
  long p_stride;         //              row stride of p_lr in floats (multiple of 4)
  const float* p_bias;   // pixel-style: [B,128] per-sample constant added after interpolation (or null)
  const uint8_t* wgb;    // pixel-style: packed [512 x 128] gamma/beta weights (2 N-blocks, interleaved)
  const float* bgb;      // pixel-style: [512] bias in the same interleaved order (gamma part includes +1)
  const uint8_t* wimg;   // packed conv weight [256 x 256] (already divided by sigma)
  const float* bias;     // [C]
  const float* skip;     // [B,T,C,128] residual or null   (backward: the forward input x of the half-block)
  long skip_bstride;     // T*C*128, or 0 when shared by the whole batch
  float* out;            // [B,T,C,128]
  double* stats;         // [2,C] accumulated sum / sumsq of out, or null
  const float* rgb_w;    // [3,C] or null
  const float* rgb_b;    // [3]
  const float* rgb_in;   // [B,3,HW] or null
  float* rgb_out;        // [B,3,HW]
  int B, HW, Hg, Wg, Rh, Rw;
  // generalisations used by the backward schedule (defaults reproduce the forward half-block):
  int nkc;               // K chunks of 64 input channels per tile: 2, 4 or 8
  int xC;                // channels per source tile (128 or 256); chunks beyond xC/64 come from x2
  const float* x2;       // second source [B,T,xC,128] (K = 512 products) or null
  float slope;           // operand LeakyReLU slope (1 = identity); backward epilogue: slope of the mask (0.2 / 0 = ReLU)
  int cout;              // output channels written by the epilogue: 256 or 128 (the MMA always runs N = 256)
  int out_pm;            // backward epilogue: write pixel-major [B,HW,cout] instead of tile-blocked
  int act;               // 0: LeakyReLU(slope) (SPADE), 1: sine (FiLM-SIREN layers of the renderer: y = sin(x*g1 + g0))
  const float* ascale;   // backward operand: per-(b,c) scale [B,C] applied to the incoming gradient ([B,2C] with x2), or null
  const float* rk_v;     // backward epilogue: rank-k term  acc += sum_j rgb_w[j][c] * rk_v[b][j][pixel]  (k = rk_n <= 3)
  int rk_n;
  const float* mod2;     // forward, K = 512: [B,2,C] table of the SECOND source's channels (null: the first table serves both,
                         // as for the renderer's first FiLM layer); lets a 512-channel layer (hidden_dim 384 / 420 zero-padded
                         // to 2 x 256) be modulated per channel
};

struct SynSmem {
  uint8_t* a_hi;   // operand chunks: const-style a 2-slot ring; pixel-style A1 (2 chunks) + one y chunk
  uint8_t* a_lo;
  uint8_t* b_st;
  float* x_st;     // staging slots [32][128]: activation ring, then residual ring
  int xs_n, ss_n;  // slots of the activation ring (0..xs_n-1) and of the residual ring after it; ss_n = 0: the residual
                   // slices follow each tile's activation slices through the activation ring
  float* tab_g1;   // [C]  (const: g1 | pixel: bn scale)
  float* tab_g0;   // [C]  (const: g0 | pixel: bn shift)
  float* tab_bias; // [C]
  float* tab_rgbw; // [3*C]
  float* tab_bgb;  // [512]
  float* tab_as;   // [C]  backward operand scale
  float* st_sum;   // [C]
  float* st_sq;    // [C]
  uint64_t* bars;
};

// const-style: 2 operand slots, one 5-slot staging ring (kOneRing) or 3 + 2 staging slots; pixel-style: 3 operand chunks,
// 2 + 1 staging slots
template <bool kPixel, bool kOneRing = false>
__device__ __forceinline__ SynSmem carve(uint8_t* raw) {
  constexpr int kA = kPixel ? 3 : kASlots, kX = kPixel ? 3 : kXSlots;
  uint8_t* s = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~uintptr_t(1023));
  SynSmem m;
  m.a_hi = s;
  m.a_lo = s + kA * kAChunk;
  m.b_st = s + 2 * kA * kAChunk;
  m.x_st = reinterpret_cast<float*>(m.b_st + kSynStages * kBStage);
  m.xs_n = kPixel ? 2 : kOneRing ? kXSlots : 3;
  m.ss_n = kPixel ? 1 : kOneRing ? 0 : 2;
  float* f = m.x_st + kX * (kXSlice / 4);
  m.tab_g1 = f; f += kC;
  m.tab_g0 = f; f += kC;
  m.tab_bias = f; f += kC;
  m.tab_rgbw = f; f += 3 * kC;
  m.tab_bgb = f; f += 512;
  m.tab_as = f; f += kC;
  m.st_sum = f; f += kC;
  m.st_sq = f; f += kC;
  m.bars = reinterpret_cast<uint64_t*>(f);
  return m;
}
constexpr uint32_t kSynSmemBytes = 2 * kASlots * kAChunk + kSynStages * kBStage + kXSlots * kXSlice +
                                   (kC * 9 + 512) * 4 + 24 * 8 + 1024;
constexpr uint32_t kPixSmemBytes = 2 * 3 * kAChunk + kSynStages * kBStage + 3 * kXSlice + (kC * 9 + 512) * 4 + 24 * 8 + 1024;
static_assert(kSynSmemBytes <= 232448 && kPixSmemBytes <= 232448, "shared memory budget");

// The pixel-style kernel divides the same weight ring into 16 KB units: a [gamma | beta] stage ([128 x 64]) takes one, a
// conv stage ([256 x 64]) two adjacent ones.
constexpr int kPixUnits = 4;
constexpr uint32_t kPixUnit = kBStage / 2;
static_assert(kPixUnits * kPixUnit == kSynStages * kBStage, "the pixel-style units tile the weight ring");

// barrier slots (const-style uses the first kSynStages of each weight pair, pixel-style all kPixUnits)
enum { B_FULL = 0 /*4*/, B_EMPTY = 4 /*4*/, X_FULL = 8 /*5*/, X_EMPTY = 13 /*5*/ };

__device__ __forceinline__ void rows_barrier() { named_barrier(1, 256); }

// Phase profile of the const-style forward, off by default: built with -DHG_SPADE_PROFILE, thread 0 of each MMA warpgroup
// sums %globaltimer intervals per phase over its walk and adds them to g_spade_prof (read and cleared by
// hg_spade_profile_read; slot kProfPhases counts warpgroup-tiles).  Without the macro every HG_PROF_* expands to nothing.
#ifdef HG_SPADE_PROFILE
enum { PROF_XRING, PROF_BUILD, PROF_WRING, PROF_MMA, PROF_DRAIN, PROF_EPI, PROF_TABLE, kProfPhases };
__device__ unsigned long long g_spade_prof[kProfPhases + 1];
__device__ __forceinline__ uint64_t prof_now() {
  uint64_t v;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(v));
  return v;
}
#define HG_PROF_BEGIN uint64_t prof_t = prof_now(), prof_acc[kProfPhases + 1] = {}
#define HG_PROF(k)                      \
  do {                                  \
    const uint64_t prof_n = prof_now(); \
    prof_acc[k] += prof_n - prof_t;     \
    prof_t = prof_n;                    \
  } while (0)
#define HG_PROF_TILE ++prof_acc[kProfPhases]
#define HG_PROF_END(t)                                                                          \
  do {                                                                                          \
    if ((t) == 0)                                                                               \
      for (int k = 0; k <= kProfPhases; ++k) atomicAdd(&g_spade_prof[k], static_cast<unsigned long long>(prof_acc[k])); \
  } while (0)
#else
#define HG_PROF_BEGIN
#define HG_PROF(k)
#define HG_PROF_TILE
#define HG_PROF_END(t)
#endif

__device__ __forceinline__ float lrelu02(float v) { return v > 0.f ? v : 0.2f * v; }

// sin / cos for |t| up to a few thousand: two-term Cody-Waite reduction by 2*pi, then the SFU (abs error ~2^-21);
// the same evaluation as the fused renderer (csrc/render.cu), so that forward and backward agree.
__device__ __forceinline__ float reduce_2pi(float t) {
  const float y = t * 0.15915494309189535f;
  const float k = (y + 12582912.f) - 12582912.f;
  float r = fmaf(-k, 6.2831854820251465f, t);
  return fmaf(-k, -1.7484555314695172e-07f, r);
}
__device__ __forceinline__ float sin_red(float t) { return __sinf(reduce_2pi(t)); }
__device__ __forceinline__ float cos_red(float t) { return __cosf(reduce_2pi(t)); }
// the same reduction on a pair (identical operations per lane)
__device__ __forceinline__ float2 reduce_2pi2(float2 t) {
  const float2 y = fmul2(t, make_float2(0.15915494309189535f, 0.15915494309189535f));
  const float2 k = fadd2(fadd2(y, make_float2(12582912.f, 12582912.f)), make_float2(-12582912.f, -12582912.f));
  const float2 r = ffma2(k, make_float2(-6.2831854820251465f, -6.2831854820251465f), t);
  return ffma2(k, make_float2(1.7484555314695172e-07f, 1.7484555314695172e-07f), r);
}
__device__ __forceinline__ float2 sin_red2(float2 t) { const float2 r = reduce_2pi2(t); return make_float2(__sinf(r.x), __sinf(r.y)); }
__device__ __forceinline__ float2 cos_red2(float2 t) { const float2 r = reduce_2pi2(t); return make_float2(__cosf(r.x), __cosf(r.y)); }

struct TileMap {
  int T, first, stride, count;
  __device__ __forceinline__ void get(int it, int& b, int& ti) const {
    const int tile = first + it * stride;
    b = tile / T;
    ti = tile - b * T;
  }
};

// ------------------------------------------------------------------------------------------
// common setup
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void init_common(const SpadeArgs& a, const SynSmem& m, int weight_slots) {
  for (int i = threadIdx.x; i < kC; i += blockDim.x) {
    m.tab_bias[i] = a.bias[i];
    m.st_sum[i] = 0.f;
    m.st_sq[i] = 0.f;
  }
  if (a.rgb_w)
    for (int i = threadIdx.x; i < 3 * kC; i += blockDim.x) m.tab_rgbw[i] = a.rgb_w[i];
  if (threadIdx.x == 0) {
    for (int i = 0; i < weight_slots; ++i) {
      mbar_init(m.bars + B_FULL + i, 1);
      mbar_init(m.bars + B_EMPTY + i, 2);             // one arrival per warpgroup
    }
    for (int i = 0; i < m.xs_n + m.ss_n; ++i) {
      mbar_init(m.bars + X_FULL + i, 1);
      mbar_init(m.bars + X_EMPTY + i, 8);             // every warp of both warpgroups
    }
    fence_mbar_init();
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------
// warp 8: weight stages.  Every tile consumes the same sequence: for each image `nstages` tiles of [256 x 64]
// in storage order (kc-major, hi then lo); the lo tiles are skipped in 1-pass mode.
// ------------------------------------------------------------------------------------------
template <int kPasses>
__device__ __forceinline__ void weight_producer_loop(const SynSmem& m, const uint8_t* img, int nstages, int num_my_tiles) {
  uint32_t st = 0, ph = 0;
  for (int t = 0; t < num_my_tiles; ++t)
    for (int s = 0; s < nstages; ++s) {
      if (kPasses == 1 && (s & 1)) continue;
      mbar_wait_backoff(m.bars + B_EMPTY + st, ph ^ 1);
      mbar_arrive_expect_tx(m.bars + B_FULL + st, kBStage);
      bulk_g2s(m.b_st + st * kBStage, img + static_cast<size_t>(s) * kBStage, kBStage, m.bars + B_FULL + st);
      if (++st == kSynStages) { st = 0; ph ^= 1; }
    }
}

// Weight-stage pipe of one warpgroup: wait for a stage, issue, and release the stage consumed one step earlier once its
// wgmmas are done (both warpgroups release every stage).
struct Pipe {
  uint32_t st = 0, ph = 0, prev = ~0u;
};
template <int N, int kPasses>
__device__ __forceinline__ void pipe_chunk(const SynSmem& m, Pipe& p, float (&d)[N / 2], uint32_t a_hi, uint32_t a_lo, bool accumulate,
                                           int t) {
#pragma unroll
  for (int part = 0; part < (kPasses == 3 ? 2 : 1); ++part) {
    mbar_wait(m.bars + B_FULL + p.st, p.ph);
    acc_fence(d);
    wgmma_fence();
    const uint32_t bt = smem_u32(m.b_st + p.st * kBStage);
    if (part == 0) {
      wg_k64<N>(d, a_hi, bt, accumulate);
      if (kPasses == 3) wg_k64<N>(d, a_lo, bt, true);
    } else {
      wg_k64<N>(d, a_hi, bt, true);
    }
    wgmma_commit();
    wgmma_wait<1>();
    acc_fence(d);
    if (p.prev != ~0u && t == 0) mbar_arrive(m.bars + B_EMPTY + p.prev);
    p.prev = p.st;
    if (++p.st == kSynStages) { p.st = 0; p.ph ^= 1; }
  }
}
template <int N>
__device__ __forceinline__ void pipe_drain(const SynSmem& m, Pipe& p, float (&d)[N / 2], int t) {
  wgmma_wait<0>();
  acc_fence(d);
  if (p.prev != ~0u && t == 0) mbar_arrive(m.bars + B_EMPTY + p.prev);
  p.prev = ~0u;
}

// ------------------------------------------------------------------------------------------
// warp 9: activation slices (const-style forward: followed by each tile's residual slices in the same ring), warp 10:
// residual slices in a ring of their own (backward, pixel-style).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void ring_emit(const SynSmem& m, uint32_t& g, int base, int slots, const float* src) {
  const uint32_t slot = base + g % slots;
  mbar_wait_backoff(m.bars + X_EMPTY + slot, ((g / slots) & 1) ^ 1);
  mbar_arrive_expect_tx(m.bars + X_FULL + slot, kXSlice);
  bulk_g2s(m.x_st + slot * (kXSlice / 4), src, kXSlice, m.bars + X_FULL + slot);
  ++g;
}
__device__ __forceinline__ void x_producer_loop(const SpadeArgs& a, const SynSmem& m, const TileMap& tm) {
  uint32_t g = 0;
  for (int it = 0; it < tm.count; ++it) {
    int b, ti;
    tm.get(it, b, ti);
    const int per_src = a.xC / 32;                 // 32-channel slices per source tile
    const float* base = a.x + static_cast<long>(b) * a.x_bstride + static_cast<long>(ti) * a.xC * 128;
    const float* base2 = a.x2 ? a.x2 + (static_cast<long>(b) * tm.T + ti) * a.xC * 128 : nullptr;
    for (int j = 0; j < 2 * a.nkc; ++j)
      ring_emit(m, g, 0, m.xs_n, (j < per_src ? base : base2 - per_src * 32 * 128) + j * 32 * 128);
    if (m.ss_n == 0 && a.skip) {   // one ring: the residual slices the epilogue takes after this tile's operand
      const float* sbase = a.skip + static_cast<long>(b) * a.skip_bstride + static_cast<long>(ti) * a.cout * 128;
      for (int j = 0; j < a.cout / 32; ++j) ring_emit(m, g, 0, m.xs_n, sbase + j * 32 * 128);
    }
  }
}
__device__ __forceinline__ void skip_producer_loop(const SpadeArgs& a, const SynSmem& m, const TileMap& tm) {
  if (!a.skip || m.ss_n == 0) return;
  uint32_t g = 0;
  for (int it = 0; it < tm.count; ++it) {
    int b, ti;
    tm.get(it, b, ti);
    const float* base = a.skip + static_cast<long>(b) * a.skip_bstride + static_cast<long>(ti) * a.cout * 128;
    for (int j = 0; j < a.cout / 32; ++j) ring_emit(m, g, m.xs_n, m.ss_n, base + j * 32 * 128);
  }
}

// Ring protocol: every warp of both warpgroups waits for and releases EVERY slice in order (a warp reads only what it
// needs).  With per-half arrivals a slot of an odd-sized ring alternates between halves, a fast half gets two phases
// ahead and the parity wait succeeds on a stale phase.
__device__ __forceinline__ uint32_t ring_take(const SynSmem& m, uint32_t g, int base, int slots) {
  const uint32_t slot = base + g % slots;
  mbar_wait_sleep(m.bars + X_FULL + slot, (g / slots) & 1);
  return slot;
}
__device__ __forceinline__ void ring_release(const SynSmem& m, uint32_t slot) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(m.bars + X_EMPTY + slot);
}

// Operand-side read of a chunk's two activation slices in the row layout: half h reads slice 2kc+h.
__device__ __forceinline__ void take_x_pair(const SynSmem& m, uint32_t& xg, int h, int row, float (&dst)[32]) {
#pragma unroll
  for (int hh = 0; hh < 2; ++hh, ++xg) {
    const uint32_t xslot = ring_take(m, xg, 0, m.xs_n);
    if (hh == h) {
      const uint32_t xs = smem_u32(m.x_st + xslot * (kXSlice / 4)) + row * 4;
#pragma unroll
      for (int j = 0; j < 32; ++j) dst[j] = lds_f32(xs + j * 512);
    }
    ring_release(m, xslot);
  }
}

// Column sums over the 64 rows of a warpgroup's fragments, folded into the CTA's shared sums: v[jj][e] holds this
// thread's two rows of column 8 jj + 2 (t%4) + e; lanes with equal t%4 hold the same columns, one per row group
// r = (t%32)/4.  A transposing reduction over r (lane bits 2..4: each step keeps half of the values and adds the partner's
// copy of the same half) leaves lane r the total of value k = r, i.e. column 8 (r/2) + 2 (t%4) + r%2: 7 shuffles and one
// warp-wide shared atomic instead of 24 shuffles and 8 atomics from 4 lanes (a float atomic on shared memory is a
// compare-and-swap loop, so every atomic instruction is a serial retry loop).  The atomic is issued on the shared
// window explicitly: through a generic pointer it compiles to a run-time dispatch over global and shared atomics.
__device__ __forceinline__ void column_sums(float* st, int c0, const float (&v)[4][2]) {
  const int lane = threadIdx.x & 31, r = lane >> 2;
  const bool b2 = r & 4, b1 = r & 2, b0 = r & 1;
  float w[4], u[2];
#pragma unroll
  for (int i = 0; i < 4; ++i) {   // k = i + 4 b2
    const float lo = v[i >> 1][i & 1], hi = v[(i + 4) >> 1][i & 1];
    w[i] = (b2 ? hi : lo) + __shfl_xor_sync(0xffffffffu, b2 ? lo : hi, 16);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i)     // k = i + 2 b1 + 4 b2
    u[i] = (b1 ? w[i + 2] : w[i]) + __shfl_xor_sync(0xffffffffu, b1 ? w[i] : w[i + 2], 8);
  const float x = (b0 ? u[1] : u[0]) + __shfl_xor_sync(0xffffffffu, b0 ? u[0] : u[1], 4);   // k = r
  asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(smem_u32(st + c0 + 8 * (r >> 1) + 2 * (lane & 3) + (r & 1))), "f"(x)
               : "memory");
}

// ------------------------------------------------------------------------------------------
// Forward epilogue of one tile from the fragments of warpgroup g.  The residual is a compile-time variant; ToRGB and the
// statistics are warp-uniform branches (eight fully unrolled variants took ptxas ten minutes for this file).
// ------------------------------------------------------------------------------------------
template <bool kSkip>
__device__ __forceinline__ void epilogue_fwd(const SpadeArgs& a, const SynSmem& m, const float (&d)[128], int b, int ti, int T,
                                             int g, int t, uint32_t& sg) {
  const int HW = a.HW, cout = a.cout;
  const bool kRgb = a.rgb_w != nullptr, kStats = a.stats != nullptr;
  int row[2];
  bool valid[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    row[i] = g * 64 + frag_row(t, i);
    valid[i] = ti * 128 + row[i] < HW;
  }
  float* const otile = a.out + (static_cast<long>(b) * T + ti) * cout * 128;
  float r[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
  // tables and slices are read through the shared window (LDS): through the generic pointers of SynSmem every read is a
  // generic load.  The tables are fixed after init_common.
  uint32_t tbias = smem_u32(m.tab_bias), trgbw = smem_u32(m.tab_rgbw);
  opaque(tbias);
  opaque(trgbw);
#pragma unroll
  for (int cg = 0; cg < 8; ++cg) {
    if (cg * 32 >= cout) break;
    float sk[2][4][2];
    if (kSkip) {
      const uint32_t slot = m.ss_n ? ring_take(m, sg, m.xs_n, m.ss_n) : ring_take(m, sg, 0, m.xs_n);
      const uint32_t xs = smem_u32(m.x_st + slot * (kXSlice / 4));
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int jj = 0; jj < 4; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e) sk[i][jj][e] = lds_f32(xs + ((frag_col(t, jj, e)) * 128 + row[i]) * 4);
      ring_release(m, slot);
      ++sg;
    }
    float s1[4][2], s2[4][2];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int j = cg * 4 + jj, c = frag_col(t, j, e);
        const float bc = lds1(tbias + c * 4);
        float wk[3];
        if (kRgb) {
#pragma unroll
          for (int k = 0; k < 3; ++k) wk[k] = lds1(trgbw + (k * kC + c) * 4);
        }
        s1[jj][e] = 0.f;
        s2[jj][e] = 0.f;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float v = d[4 * j + 2 * i + e] + bc;
          if (kSkip) v += sk[i][jj][e];
          if (valid[i]) otile[c * 128 + row[i]] = v;
          else v = 0.f;
          if (kRgb) {
#pragma unroll
            for (int k = 0; k < 3; ++k) r[i][k] = fmaf(v, wk[k], r[i][k]);
          }
          s1[jj][e] += v;
          s2[jj][e] = fmaf(v, v, s2[jj][e]);
        }
      }
    if (kStats) {
      column_sums(m.st_sum, cg * 32, s1);
      column_sums(m.st_sq, cg * 32, s2);
    }
  }
  if (kRgb) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        r[i][k] += __shfl_xor_sync(0xffffffffu, r[i][k], 1);
        r[i][k] += __shfl_xor_sync(0xffffffffu, r[i][k], 2);
      }
      if ((t & 3) == 0 && valid[i]) {
        const int pix = ti * 128 + row[i];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const long idx = (static_cast<long>(b) * 3 + k) * HW + pix;
          float o = r[i][k] + a.rgb_b[k];
          if (a.rgb_in) o += a.rgb_in[idx];
          a.rgb_out[idx] = o;
        }
      }
    }
  }
}

// warp-uniform dispatch on the launch's flags
__device__ __forceinline__ void epilogue_fwd_any(const SpadeArgs& a, const SynSmem& m, const float (&d)[128], int b, int ti, int T,
                                                 int g, int t, uint32_t& sg) {
  if (a.skip) epilogue_fwd<true>(a, m, d, b, ti, T, g, t, sg);
  else epilogue_fwd<false>(a, m, d, b, ti, T, g, t, sg);
}

// the forward statistics of the CTA -> the launch's [2,C] fp64 sums (after every tile's column_sums)
__device__ __forceinline__ void flush_fwd_stats(const SpadeArgs& a, const SynSmem& m) {
  rows_barrier();
  if (a.stats)
    for (int c = threadIdx.x; c < kC; c += 256) {
      atomicAdd(a.stats + c, static_cast<double>(m.st_sum[c]));
      atomicAdd(a.stats + kC + c, static_cast<double>(m.st_sq[c]));
    }
}

// ------------------------------------------------------------------------------------------
// Epilogue of the BACKWARD (data-gradient) variant.  The accumulator holds dL/dy = W^T dL/dout for the 128
// pixels of the tile; the forward input x of the half-block arrives through the residual ring, so that
//     pre = x*g1[b,c] + g0[b,c]            (the folded BatchNorm + SPADE modulation of the forward pass)
//     dpre = dL/dy * lrelu'(pre)           -> stored (tile-blocked, like every activation)
//     S1[b,c] += dpre,  S2[b,c] += dpre*x  -> everything BatchNorm / gamma / beta need (DESIGN.md "Backward")
// Compile-time variants (straight-line per-element code):
//   kSine  activation derivative cos(pre) (FiLM-SIREN) instead of the LeakyReLU / ReLU mask
//   kRk    rank-3 term from the renderer's heads (rows beyond rk_n of the [3,C] weight table are zero)
//   kPm    pixel-major [B,HW,cout] output
// The per-sample tables tab_g1 / tab_g0 and sums st_sum / st_sq are managed by the caller.
// ------------------------------------------------------------------------------------------
template <bool kSine, bool kRk, bool kPm>
__device__ __forceinline__ void epilogue_bwd(const SpadeArgs& a, const SynSmem& m, const float (&d)[128], int b, int ti, int T, int g,
                                             int t, uint32_t& sg) {
  const int HW = a.HW, cout = a.cout, rk_n = a.rk_n;
  const float mslope = a.slope;
  int row[2];
  bool valid[2];
  float rv[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    row[i] = g * 64 + frag_row(t, i);
    valid[i] = ti * 128 + row[i] < HW;
    if (kRk && valid[i]) {
      const float* rp = a.rk_v + static_cast<long>(b) * rk_n * HW + ti * 128 + row[i];
      rv[i][0] = rp[0];
      if (rk_n > 1) rv[i][1] = rp[HW];
      if (rk_n > 2) rv[i][2] = rp[2 * static_cast<long>(HW)];
    }
  }
  float* const otile = a.out + (static_cast<long>(b) * T + ti) * cout * 128;
#pragma unroll
  for (int cg = 0; cg < 8; ++cg) {
    if (cg * 32 >= cout) break;
    float xv[2][4][2];
    {
      const uint32_t slot = ring_take(m, sg, m.xs_n, m.ss_n);
      const float* xs = m.x_st + slot * (kXSlice / 4);
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int jj = 0; jj < 4; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e)   // rows past the image (last, partial tile only): the slice holds whatever the padding holds
            xv[i][jj][e] = valid[i] ? xs[frag_col(t, jj, e) * 128 + row[i]] : 0.f;
      ring_release(m, slot);
      ++sg;
    }
    float s1[4][2], s2[4][2];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int j = cg * 4 + jj, c = frag_col(t, j, e);
        const float t1 = m.tab_g1[c], t0 = m.tab_g0[c];
        s1[jj][e] = 0.f;
        s2[jj][e] = 0.f;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const float x = xv[i][jj][e];
          const float pre = fmaf(x, t1, t0);
          float acc = d[4 * j + 2 * i + e];       // 0 for rows past the image
          if (kRk)
            acc = fmaf(rv[i][2], m.tab_rgbw[2 * kC + c], fmaf(rv[i][1], m.tab_rgbw[kC + c], fmaf(rv[i][0], m.tab_rgbw[c], acc)));
          const float mask = kSine ? cos_red(pre) : (pre > 0.f ? 1.f : mslope);
          const float dd = acc * mask;
          if (valid[i]) {
            if (kPm) a.out[(static_cast<long>(b) * HW + ti * 128 + row[i]) * cout + c] = dd;
            else otile[c * 128 + row[i]] = dd;
          }
          s1[jj][e] += dd;
          s2[jj][e] = fmaf(dd, x, s2[jj][e]);
        }
      }
    column_sums(m.st_sum, cg * 32, s1);
    column_sums(m.st_sq, cg * 32, s2);
  }
}

__device__ __forceinline__ void epilogue_bwd_any(const SpadeArgs& a, const SynSmem& m, const float (&d)[128], int b, int ti, int T,
                                                 int g, int t, uint32_t& sg) {
  // warp-uniform dispatch to a straight-line variant (the host side rejects the other combinations)
  if (a.act == 1) {
    if (a.rk_v) epilogue_bwd<true, true, false>(a, m, d, b, ti, T, g, t, sg);
    else epilogue_bwd<true, false, false>(a, m, d, b, ti, T, g, t, sg);
  } else {
    if (a.out_pm) epilogue_bwd<false, false, true>(a, m, d, b, ti, T, g, t, sg);
    else epilogue_bwd<false, false, false>(a, m, d, b, ti, T, g, t, sg);
  }
}

// per-sample sums of the backward variant -> stats [B,2,cout] (fp64), then cleared
__device__ __forceinline__ void flush_bwd_sums(const SpadeArgs& a, const SynSmem& m, int b) {
  for (int c = threadIdx.x; c < a.cout; c += 256) {
    atomicAdd(a.stats + (static_cast<long>(b) * 2 + 0) * a.cout + c, static_cast<double>(m.st_sum[c]));
    atomicAdd(a.stats + (static_cast<long>(b) * 2 + 1) * a.cout + c, static_cast<double>(m.st_sq[c]));
    m.st_sum[c] = 0.f;
    m.st_sq[c] = 0.f;
  }
}

// ------------------------------------------------------------------------------------------
// const-style variant (384 threads).  Warpgroup g (warps 4g..4g+3) builds rows 64g..64g+63 of each K chunk in a 2-slot
// ring (warp (q, h): rows 32q.., channels 32h.. of the chunk), issues their wgmmas ([64 x 256] fp32 accumulator in
// registers) and runs the epilogue; warp 8 streams the weights, warp 9 the activation slices (forward: and behind each
// tile's, its residual slices, through one 5-slot ring), warp 10 the backward's residual slices.
// kBwd: data gradient of the same half-block: the operand is dL/dout passed through unchanged (optionally scaled), the
// weight image is W^T, the epilogue is `epilogue_bwd`.
// ------------------------------------------------------------------------------------------
template <int kPasses, bool kBwd>
__global__ void __launch_bounds__(kSynThreads, 1) spade_const_kernel(SpadeArgs a) {
  extern __shared__ uint8_t smem_raw[];
  const SynSmem m = carve<false, !kBwd>(smem_raw);   // the backward's epilogue spills with the single ring
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  init_common(a, m, kSynStages);
  TileMap tm;
  tm.T = (a.HW + 127) / 128;
  tm.first = blockIdx.x;
  tm.stride = gridDim.x;
  tm.count = (a.B * tm.T - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);

  if (warp < 8) {
    regs_inc<kMmaRegs>();
    const int g = warp >> 2, t = threadIdx.x & 127;
    const int q = 2 * g + (warp & 1), h = (warp >> 1) & 1;
    const int row = q * 32 + lane;
    int cur_b = -1;
    uint32_t acnt = 0;   // operand chunks produced (2-slot ring)
    uint32_t xg = 0, sg = 0;   // slices taken from the activation ring (forward: and the residual slices behind them)
                               // and from the backward's residual ring
    Pipe p;
    float d[128];
    HG_PROF_BEGIN;
    for (int it = 0; it < tm.count; ++it) {
      int b, ti;
      tm.get(it, b, ti);
      HG_PROF_TILE;
      if (b != cur_b) {  // refresh the per-sample tables (and, backward, flush the previous sample's sums)
        rows_barrier();
        if (kBwd && cur_b >= 0) flush_bwd_sums(a, m, cur_b);
        for (int i = threadIdx.x; i < kC; i += 256) {
          if (kBwd) {
            if (a.ascale) {    // K = 512: columns kC.. scale g2; they live in the (pixel-style only) gamma/beta bias table
              const long ld = a.x2 ? 2 * kC : kC;
              m.tab_as[i] = a.ascale[static_cast<long>(b) * ld + i];
              if (a.x2) m.tab_bgb[i] = a.ascale[static_cast<long>(b) * ld + kC + i];
            }
            if (i < a.cout) {
              m.tab_g1[i] = a.mod ? a.mod[(static_cast<long>(b) * 2 + 0) * a.cout + i] : 1.f;
              m.tab_g0[i] = a.mod ? a.mod[(static_cast<long>(b) * 2 + 1) * a.cout + i] : 0.f;
            }
          } else {   // no table = identity (plain 1x1 convolution)
            m.tab_g1[i] = a.mod ? a.mod[(static_cast<long>(b) * 2 + 0) * kC + i] : 1.f;
            m.tab_g0[i] = a.mod ? a.mod[(static_cast<long>(b) * 2 + 1) * kC + i] : 0.f;
            if (a.mod2) {      // second source's table lives in the (otherwise pixel-style only) gamma/beta bias table
              m.tab_bgb[i] = a.mod2[(static_cast<long>(b) * 2 + 0) * kC + i];
              m.tab_bgb[kC + i] = a.mod2[(static_cast<long>(b) * 2 + 1) * kC + i];
            }
          }
        }
        rows_barrier();
        cur_b = b;
      }
      const bool valid = ti * 128 + row < a.HW;
      uint32_t tg1a = smem_u32(kBwd ? m.tab_as : m.tab_g1), tg0a = smem_u32(m.tab_g0);
      uint32_t tg1b = smem_u32(m.tab_bgb), tg0b = smem_u32(m.tab_bgb + kC);
      opaque(tg1a);   // the tables may just have been refreshed: no table load may move above this point
      opaque(tg0a);
      opaque(tg1b);
      opaque(tg0b);
      const float slope = a.slope;
      const bool sine = a.act == 1, scaled = kBwd && a.ascale != nullptr;
      const bool two_tables = kBwd ? (scaled && a.x2 != nullptr) : a.mod2 != nullptr;
#pragma unroll 1
      for (int kc = 0; kc < a.nkc; ++kc, ++acnt) {
        const int c0 = (kc * 64 + h * 32) & (kC - 1);
        const bool second = two_tables && kc * 64 >= kC;
        const uint32_t tg1 = second ? tg1b : tg1a, tg0 = second ? tg0b : tg0a;
        float cur[32];
        HG_PROF(PROF_TABLE);
        take_x_pair(m, xg, h, row, cur);
        HG_PROF(PROF_XRING);
        // the slot was last read by chunk acnt - 2, whose wgmmas pipe_chunk has seen complete
        const uint32_t slot = acnt & 1;
#pragma unroll
        for (int gi = 0; gi < 4; ++gi) {
          float y[8], t1[8], t0[8];
          if (!kBwd || scaled) lds8(tg1 + (c0 + gi * 8) * 4, t1);
          if (!kBwd) lds8(tg0 + (c0 + gi * 8) * 4, t0);
          if (kBwd) {
#pragma unroll
            for (int j = 0; j < 8; ++j) y[j] = scaled ? cur[gi * 8 + j] * t1[j] : cur[gi * 8 + j];
          } else if (sine) {
#pragma unroll
            for (int j = 0; j < 8; j += 2) {
              const float2 sv = sin_red2(ffma2(make_float2(cur[gi * 8 + j], cur[gi * 8 + j + 1]), make_float2(t1[j], t1[j + 1]),
                                               make_float2(t0[j], t0[j + 1])));
              y[j] = sv.x;
              y[j + 1] = sv.y;
            }
          } else {
            affine_lrelu8(cur + gi * 8, t1, t0, slope, y);
          }
          if (!valid) {   // only the last, partial tile of an image
#pragma unroll
            for (int j = 0; j < 8; ++j) y[j] = 0.f;
          }
          store_a8<kPasses == 3>(m.a_hi + slot * kAChunk, m.a_lo + slot * kAChunk, row, h * 32 + gi * 8, y);
        }
        fence_proxy_async_smem();
        named_barrier(2 + g, 128);
        HG_PROF(PROF_BUILD);
#ifdef HG_SPADE_PROFILE
        mbar_wait(m.bars + B_FULL + p.st, p.ph);   // pipe_chunk's first wait then returns at once
        HG_PROF(PROF_WRING);
#endif
        pipe_chunk<256, kPasses>(m, p, d, smem_u32(m.a_hi + slot * kAChunk) + g * 64 * 128,
                                 smem_u32(m.a_lo + slot * kAChunk) + g * 64 * 128, kc > 0, t);
        HG_PROF(PROF_MMA);
      }
      pipe_drain<256>(m, p, d, t);
      HG_PROF(PROF_DRAIN);
      if (kBwd) epilogue_bwd_any(a, m, d, b, ti, tm.T, g, t, sg);
      else epilogue_fwd_any(a, m, d, b, ti, tm.T, g, t, xg);
      HG_PROF(PROF_EPI);
    }
    HG_PROF_END(t);
    if (kBwd) {
      rows_barrier();
      if (cur_b >= 0) flush_bwd_sums(a, m, cur_b);
    } else {
      flush_fwd_stats(a, m);
    }
  } else {
    regs_dec<kProducerRegs>();
    if (lane == 0) {
      if (warp == 8) weight_producer_loop<kPasses>(m, a.wimg, 2 * a.nkc, tm.count);
      else if (warp == 9) x_producer_loop(a, m, tm);
      else if (warp == 10) skip_producer_loop(a, m, tm);
    }
  }
}

// ------------------------------------------------------------------------------------------
// pixel-style variant
// ------------------------------------------------------------------------------------------
// PyTorch's bilinear source index (align_corners=False): src = max(scale*(dst+0.5)-0.5, 0)
__device__ __forceinline__ void bilin(int dst, int in_size, float scale, int& i0, int& i1, float& l0, float& l1) {
  float src = scale * (static_cast<float>(dst) + 0.5f) - 0.5f;
  src = src < 0.f ? 0.f : src;
  i0 = static_cast<int>(src);
  i1 = i0 + (i0 < in_size - 1 ? 1 : 0);
  l1 = src - static_cast<float>(i0);
  l0 = 1.f - l1;
}

// Weight stages of one pixel-style tile: per conv K chunk kc, the [gamma | beta] rows of channels 64kc.. (128 rows of
// gamma/beta block kc/2) for both K chunks of A1, then the conv chunk kc.  Each 16 KB unit of the ring is filled in turn;
// a conv stage is two units.  Per K chunk fp32x3 fills 8 units (gb k0 hi / lo, k1 hi / lo, conv hi, conv lo) and bf16 4
// (gb k0, k1, conv), so a conv stage always starts on unit 0 or 2 and its image is contiguous in shared memory.
template <int kPasses>
__device__ __forceinline__ void pixel_weight_producer_loop(const SpadeArgs& a, const SynSmem& m, int num_my_tiles) {
  uint32_t n = 0;   // units filled
  auto emit = [&](const uint8_t* src) {
    const uint32_t u = n % kPixUnits;
    mbar_wait_backoff(m.bars + B_EMPTY + u, ((n / kPixUnits) & 1) ^ 1);
    mbar_arrive_expect_tx(m.bars + B_FULL + u, kPixUnit);
    bulk_g2s(m.b_st + u * kPixUnit, src, kPixUnit, m.bars + B_FULL + u);
    ++n;
  };
  for (int t = 0; t < num_my_tiles; ++t)
    for (int kc = 0; kc < 4; ++kc) {
      for (int k = 0; k < 2; ++k)
        for (int part = 0; part < (kPasses == 3 ? 2 : 1); ++part)
          emit(a.wgb + static_cast<size_t>(((kc >> 1) * 2 + k) * 2 + part) * kBStage + (kc & 1) * kPixUnit);
      for (int part = 0; part < (kPasses == 3 ? 2 : 1); ++part) {
        const uint8_t* src = a.wimg + static_cast<size_t>(kc * 2 + part) * kBStage;
        emit(src);
        emit(src + kPixUnit);
      }
    }
}

// Consumer side of the unit ring, per warpgroup: a stage of N = 128 takes one unit, N = 256 two.  Like `pipe_chunk`, a
// stage's units are released (by both warpgroups) once the wgmmas of the NEXT stage have been issued and the stage's own
// have completed.
struct PixPipe {
  uint32_t n = 0;          // units consumed
  uint32_t prev = 0;       // first unit of the stage awaiting release
  uint32_t prev_units = 0; // its units (0: none)
};
__device__ __forceinline__ void pix_release(const SynSmem& m, PixPipe& p, int t) {
  if (t == 0)
    for (uint32_t j = 0; j < p.prev_units; ++j) mbar_arrive(m.bars + B_EMPTY + (p.prev + j) % kPixUnits);
  p.prev_units = 0;
}
// One weight stage (part 0: hi weights, A hi [+ A lo]; part 1: lo weights, A hi) into accumulator d.
template <int N, int kPasses>
__device__ __forceinline__ void pix_part(const SynSmem& m, PixPipe& p, float (&d)[N / 2], uint32_t a_hi, uint32_t a_lo, int part,
                                         bool accumulate, int t) {
  constexpr uint32_t kUnits = N == 256 ? 2 : 1;
  const uint32_t u = p.n % kPixUnits;
#pragma unroll
  for (uint32_t j = 0; j < kUnits; ++j) mbar_wait(m.bars + B_FULL + u + j, ((p.n + j) / kPixUnits) & 1);
  acc_fence(d);
  wgmma_fence();
  const uint32_t bt = smem_u32(m.b_st + u * kPixUnit);
  if (part == 0) {
    wg_k64<N>(d, a_hi, bt, accumulate);
    if (kPasses == 3) wg_k64<N>(d, a_lo, bt, true);
  } else {
    wg_k64<N>(d, a_hi, bt, true);
  }
  wgmma_commit();
  wgmma_wait<1>();
  acc_fence(d);
  pix_release(m, p, t);
  p.prev = u;
  p.prev_units = kUnits;
  p.n += kUnits;
}
template <int N>
__device__ __forceinline__ void pix_drain(const SynSmem& m, PixPipe& p, float (&d)[N / 2], int t) {
  wgmma_wait<0>();
  acc_fence(d);
  pix_release(m, p, t);
}

// A1 = relu(bilinear(P_lr) + c) of tile (b, ti) into the two A1 chunks: column half h builds K chunk h (the previous
// tile's wgmmas are complete).  Fully unrolled, so that all 64 + 16 loads of a thread are in flight at once: the caller
// runs it while neither accumulator is live.
template <int kPasses>
__device__ __forceinline__ void build_a1(const SpadeArgs& a, const SynSmem& m, int b, int ti, int row, int h, int g, float sy,
                                         float sx) {
  const int pix = ti * 128 + row;
  const bool valid = pix < a.HW;
  const int py = valid ? pix / a.Wg : 0, px = valid ? pix % a.Wg : 0;
  int y0, y1, x0, x1;
  float ly0, ly1, lx0, lx1;
  bilin(py, a.Rh, sy, y0, y1, ly0, ly1);
  bilin(px, a.Rw, sx, x0, x1, lx0, lx1);
  const float* base = a.p_lr + static_cast<long>(b) * a.Rh * a.Rw * a.p_stride;
  const float4* n00 = reinterpret_cast<const float4*>(base + (static_cast<long>(y0) * a.Rw + x0) * a.p_stride);
  const float4* n01 = reinterpret_cast<const float4*>(base + (static_cast<long>(y0) * a.Rw + x1) * a.p_stride);
  const float4* n10 = reinterpret_cast<const float4*>(base + (static_cast<long>(y1) * a.Rw + x0) * a.p_stride);
  const float4* n11 = reinterpret_cast<const float4*>(base + (static_cast<long>(y1) * a.Rw + x1) * a.p_stride);
  const float4* pb = a.p_bias ? reinterpret_cast<const float4*>(a.p_bias + static_cast<long>(b) * 128) : nullptr;
  const float2 lx0p = make_float2(lx0, lx0), lx1p = make_float2(lx1, lx1), ly0p = make_float2(ly0, ly0), ly1p = make_float2(ly1, ly1);
#pragma unroll
  for (int gi = 0; gi < 8; ++gi) {
    float y[8];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int f4 = h * 16 + gi * 2 + u;
      const float4 v00 = __ldg(n00 + f4), v01 = __ldg(n01 + f4), v10 = __ldg(n10 + f4), v11 = __ldg(n11 + f4);
      // same association as upsample_bilinear2d: ly0*(lx0*a + lx1*b) + ly1*(lx0*c + lx1*d), on channel pairs
      auto lerp2 = [&](float2 a, float2 b, float2 c, float2 d) {
        const float2 top = ffma2(b, lx1p, fmul2(a, lx0p));
        const float2 bot = ffma2(d, lx1p, fmul2(c, lx0p));
        return ffma2(top, ly0p, fmul2(bot, ly1p));
      };
      float2 lo2 = lerp2(make_float2(v00.x, v00.y), make_float2(v01.x, v01.y), make_float2(v10.x, v10.y), make_float2(v11.x, v11.y));
      float2 hi2 = lerp2(make_float2(v00.z, v00.w), make_float2(v01.z, v01.w), make_float2(v10.z, v10.w), make_float2(v11.z, v11.w));
      if (pb) {
        const float4 c4 = __ldg(pb + f4);
        lo2 = fadd2(lo2, make_float2(c4.x, c4.y));
        hi2 = fadd2(hi2, make_float2(c4.z, c4.w));
      }
      y[u * 4 + 0] = lo2.x; y[u * 4 + 1] = lo2.y; y[u * 4 + 2] = hi2.x; y[u * 4 + 3] = hi2.y;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) y[j] = valid ? fmaxf(y[j], 0.f) : 0.f;
    store_a8<kPasses == 3>(m.a_hi + h * kAChunk, m.a_lo + h * kAChunk, row, gi * 8, y);
  }
  fence_proxy_async_smem();
  named_barrier(2 + g, 128);
}

// Per tile: A1 = relu(bilinear(P_lr) + c) (K = 128, two chunks); then per conv K chunk kc: [gamma | beta] of channels
// 64kc.. = A1 . Wgb (a [64 x 128] accumulator per warpgroup), y = lrelu(BN(x)*(1+gamma)+beta) -> the y chunk, conv
// accumulate.  The 28x larger up-sampled style map of map3d_generator.py:244-245 is never materialised.
// The A1 gather and the epilogue run with the tensor pipe idle, but while the weight producer refills the ring for the
// next tile; DESIGN.md section 8 item 1 records what moving them under the wgmmas measured.
template <int kPasses>
__global__ void __launch_bounds__(kSynThreads, 1) spade_pixel_kernel(SpadeArgs a) {
  extern __shared__ uint8_t smem_raw[];
  const SynSmem m = carve<true>(smem_raw);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < kC; i += blockDim.x) {
    m.tab_g1[i] = a.scsh[i];
    m.tab_g0[i] = a.scsh[kC + i];
  }
  for (int i = threadIdx.x; i < 512; i += blockDim.x) m.tab_bgb[i] = a.bgb[i];
  init_common(a, m, kPixUnits);
  TileMap tm;
  tm.T = (a.HW + 127) / 128;
  tm.first = blockIdx.x;
  tm.stride = gridDim.x;
  tm.count = (a.B * tm.T - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);
  const float sy = static_cast<float>(a.Rh) / static_cast<float>(a.Hg);
  const float sx = static_cast<float>(a.Rw) / static_cast<float>(a.Wg);

  if (warp < 8) {
    regs_inc<kMmaRegs>();
    const int g = warp >> 2, t = threadIdx.x & 127;
    const int q = 2 * g + (warp & 1), h = (warp >> 1) & 1;
    const int row = q * 32 + lane;
    uint8_t* const y_hi = m.a_hi + 2 * kAChunk;
    uint8_t* const y_lo = m.a_lo + 2 * kAChunk;
    constexpr int kParts = kPasses == 3 ? 2 : 1;
    uint32_t xg = 0, sg = 0;
    PixPipe p;
    float d[128], e[64];
    for (int it = 0; it < tm.count; ++it) {
      int b, ti;
      tm.get(it, b, ti);
      build_a1<kPasses>(a, m, b, ti, row, h, g, sy, sx);
      // The first wgmma into each accumulator in a tile runs with scale-d = 0 and ignores its input; defining both here
      // tells the compiler so (the wgmma operands are read-write), and frees their 192 registers for the epilogue and
      // the A1 gather above.  Without it the gather could only run 2 iterations deep, and the kernel spilled.
#pragma unroll
      for (int i = 0; i < 128; ++i) d[i] = 0.f;
#pragma unroll
      for (int i = 0; i < 64; ++i) e[i] = 0.f;
      int frow[2];
      bool fvalid[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        frow[i] = g * 64 + frag_row(t, i);
        fvalid[i] = ti * 128 + frow[i] < a.HW;
      }
#pragma unroll 1
      for (int kc = 0; kc < 4; ++kc) {
        // ---- [gamma | beta] of channels 64kc.. (waits for the previous conv chunk too: the y chunk is free afterwards)
#pragma unroll
        for (int s = 0; s < 2 * kParts; ++s) {
          const int k = s / kParts;
          pix_part<128, kPasses>(m, p, e, smem_u32(m.a_hi + k * kAChunk) + g * 64 * 128, smem_u32(m.a_lo + k * kAChunk) + g * 64 * 128,
                                 s % kParts, s > 0, t);
        }
        pix_drain<128>(m, p, e, t);
        // ---- y = lrelu(BN(x)*(1+gamma)+beta) straight from the fragments; x from the chunk's two activation slices
        const uint32_t s0 = ring_take(m, xg, 0, m.xs_n), s1 = ring_take(m, xg + 1, 0, m.xs_n);
        xg += 2;
        const float* xs0 = m.x_st + s0 * (kXSlice / 4);
        const float* xs1 = m.x_st + s1 * (kXSlice / 4);
        const int col = (kc >> 1) * 256 + (kc & 1) * 128;       // this chunk's gamma columns in the bias table
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c = frag_col(t, j, 0), ch = kc * 64 + c;
          const float* xs = j < 4 ? xs0 : xs1;
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            float y2[2];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              const float gam = e[4 * j + 2 * i + u] + m.tab_bgb[col + c + u];               // 1 + gamma
              const float bet = e[4 * (j + 8) + 2 * i + u] + m.tab_bgb[col + 64 + c + u];    // beta
              const float xn = fmaf(xs[((c + u) & 31) * 128 + frow[i]], m.tab_g1[ch + u], m.tab_g0[ch + u]);
              const float v = fmaf(xn, gam, bet);
              y2[u] = fvalid[i] ? fmaxf(v, 0.2f * v) : 0.f;
            }
            uint32_t hb, lb;
            split_bf16x2(y2[0], y2[1], hb, lb);
            const uint32_t off = sw128_offset(frow[i], c);
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(smem_u32(y_hi) + off), "r"(hb));
            if (kPasses == 3) asm volatile("st.shared.b32 [%0], %1;" ::"r"(smem_u32(y_lo) + off), "r"(lb));
          }
        }
        ring_release(m, s0);
        ring_release(m, s1);
        fence_proxy_async_smem();
        named_barrier(2 + g, 128);
#pragma unroll
        for (int part = 0; part < kParts; ++part)
          pix_part<256, kPasses>(m, p, d, smem_u32(y_hi) + g * 64 * 128, smem_u32(y_lo) + g * 64 * 128, part, kc > 0, t);
      }
      pix_drain<256>(m, p, d, t);
      epilogue_fwd_any(a, m, d, b, ti, tm.T, g, t, sg);
    }
    flush_fwd_stats(a, m);
  } else {
    regs_dec<kProducerRegs>();
    if (lane == 0) {
      if (warp == 8) pixel_weight_producer_loop<kPasses>(a, m, tm.count);
      else if (warp == 9) x_producer_loop(a, m, tm);
      else if (warp == 10) skip_producer_loop(a, m, tm);
    }
  }
}

// ------------------------------------------------------------------------------------------
// BatchNorm finalisation: batch (or running) statistics -> scale/shift (+ fused per-sample modulation)
// ------------------------------------------------------------------------------------------
// nn.SyncBatchNorm semantics (map3d_layers.py:162): biased variance for normalisation, unbiased for
// the running estimate, momentum 0.1, eps 1e-5.
__global__ void bn_finalize_kernel(const double* __restrict__ stats, double count_in, const double* __restrict__ count_ptr,
                                   const float* __restrict__ weight,
                                   const float* __restrict__ bias, float* running_mean, float* running_var,
                                   int training, float eps, float momentum, const float* __restrict__ gb, int B,
                                   float* __restrict__ scsh, float* __restrict__ mod) {
  const int c = threadIdx.x;
  float mean, var;
  const double count = count_ptr ? count_ptr[0] : count_in;
  if (training) {
    const double mu = stats[c] / count;
    double v = stats[kC + c] / count - mu * mu;
    v = v < 0 ? 0 : v;
    mean = static_cast<float>(mu);
    var = static_cast<float>(v);
    if (running_mean) {
      const double unb = count > 1 ? v * count / (count - 1) : v;
      running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
      running_var[c] = (1.f - momentum) * running_var[c] + momentum * static_cast<float>(unb);
    }
  } else {
    mean = running_mean[c];
    var = running_var[c];
  }
  const float sc = weight[c] * rsqrtf(var + eps);
  const float sh = bias[c] - mean * sc;
  if (scsh) {
    scsh[c] = sc;
    scsh[kC + c] = sh;
  }
  if (mod && gb) {
    for (int b = 0; b < B; ++b) {
      const float G = gb[(static_cast<long>(b) * 2 + 0) * kC + c];   // 1 + gamma
      const float Bt = gb[(static_cast<long>(b) * 2 + 1) * kC + c];  // beta
      mod[(static_cast<long>(b) * 2 + 0) * kC + c] = sc * G;
      mod[(static_cast<long>(b) * 2 + 1) * kC + c] = fmaf(sh, G, Bt);
    }
  }
}

// ------------------------------------------------------------------------------------------
// synthesis input x0 = sin(W [i, j]^T + b)  (map3d_layers.py:260-275), shared by the whole batch,
// written in the tile-blocked layout [T, C, 128], with its BatchNorm statistics.
// ------------------------------------------------------------------------------------------
__global__ void synth_input_kernel(const float* __restrict__ w, const float* __restrict__ bias,
                                   const float* __restrict__ ic, const float* __restrict__ jc, int Hg, int Wg,
                                   float* __restrict__ x0, double* __restrict__ stats, double batch_mult) {
  // grid: (ceil(HW/256), C); one channel per blockIdx.y
  const int c = blockIdx.y;
  const int HW = Hg * Wg;
  const float w0 = w[c * 2 + 0], w1 = w[c * 2 + 1], bb = bias[c];
  float s1 = 0.f, s2 = 0.f;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += gridDim.x * blockDim.x) {
    const float v = sinf(fmaf(w1, jc[p % Wg], fmaf(w0, ic[p / Wg], bb)));
    x0[(static_cast<long>(p >> 7) * kC + c) * 128 + (p & 127)] = v;
    s1 += v;
    s2 += v * v;
  }
  __shared__ float r1[8], r2[8];
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  if ((threadIdx.x & 31) == 0) { r1[threadIdx.x >> 5] = s1; r2[threadIdx.x >> 5] = s2; }
  __syncthreads();
  if (threadIdx.x == 0 && stats) {
    float t1 = 0.f, t2 = 0.f;
    for (int i = 0; i < static_cast<int>(blockDim.x >> 5); ++i) { t1 += r1[i]; t2 += r2[i]; }
    atomicAdd(stats + c, static_cast<double>(t1) * batch_mult);
    atomicAdd(stats + kC + c, static_cast<double>(t2) * batch_mult);
  }
}

}  // namespace hg

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
extern "C" {

int hg_spade_conv(const float* x, long x_bstride, const float* mod, const float* scsh, const float* p_lr,
                  long p_stride, const float* p_bias, const void* wgb, const float* bgb, const void* wimg, const float* bias, const float* skip,
                  float* out, double* stats, const float* rgb_w, const float* rgb_b, const float* rgb_in,
                  float* rgb_out, int B, int C, int Hg, int Wg, int Rh, int Rw, int passes, void* stream) {
  HG_REQUIRE(C == hg::kC, "hg_spade_conv: only %d channels are supported (got %d)", hg::kC, C);
  HG_REQUIRE(x && wimg && bias && out, "hg_spade_conv: null pointer");
  HG_REQUIRE((mod != nullptr) != (p_lr != nullptr), "hg_spade_conv: give exactly one of mod (const style) / p_lr (pixel style)");
  HG_REQUIRE(passes == 1 || passes == 3, "hg_spade_conv: passes must be 1 or 3");
  HG_REQUIRE(B > 0 && Hg > 0 && Wg > 0, "hg_spade_conv: bad shape");
  HG_REQUIRE(!rgb_w || (rgb_b && rgb_out), "hg_spade_conv: rgb_b / rgb_out missing");
  if (p_lr) {
    HG_REQUIRE(scsh && wgb && bgb && Rh > 0 && Rw > 0, "hg_spade_conv: pixel-style arguments missing");
    HG_REQUIRE((reinterpret_cast<uintptr_t>(p_lr) & 15) == 0 && p_stride >= 128 && (p_stride & 3) == 0,
               "hg_spade_conv: p_lr must be 16-byte aligned with a row stride >= 128 that is a multiple of 4");
    HG_REQUIRE(!p_bias || (reinterpret_cast<uintptr_t>(p_bias) & 15) == 0, "hg_spade_conv: p_bias must be 16-byte aligned");
  }
  hg::SpadeArgs a{x, x_bstride, mod, scsh, p_lr, p_stride, p_bias, static_cast<const uint8_t*>(wgb), bgb,
                  static_cast<const uint8_t*>(wimg), bias, skip,
                  static_cast<long>((Hg * Wg + 127) / 128) * hg::kC * 128, out, stats, rgb_w, rgb_b, rgb_in, rgb_out,
                  B, Hg * Wg, Hg, Wg, Rh, Rw};
  a.nkc = 4; a.xC = hg::kC; a.x2 = nullptr; a.slope = 0.2f; a.cout = hg::kC; a.out_pm = 0;
  const int tiles = B * ((Hg * Wg + 127) / 128);
  const int grid = tiles < hg::num_sms() ? tiles : hg::num_sms();
  auto st = static_cast<cudaStream_t>(stream);
#define HG_LAUNCH(KERNEL, SMEM)                                                                                   \
  do {                                                                                                            \
    cudaError_t e = cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);               \
    if (e != cudaSuccess) { hg::set_error("hg_spade_conv: smem opt-in failed: %s", cudaGetErrorString(e)); return 2; } \
    KERNEL<<<grid, hg::kSynThreads, SMEM, st>>>(a);                                                               \
  } while (0)
  if (mod) {
    if (passes == 3) HG_LAUNCH((hg::spade_const_kernel<3, false>), hg::kSynSmemBytes); else HG_LAUNCH((hg::spade_const_kernel<1, false>), hg::kSynSmemBytes);
  } else {
    if (passes == 3) HG_LAUNCH(hg::spade_pixel_kernel<3>, hg::kPixSmemBytes); else HG_LAUNCH(hg::spade_pixel_kernel<1>, hg::kPixSmemBytes);
  }
#undef HG_LAUNCH
  return hg::check_launch("hg_spade_conv");
}

static int launch_blocked_gemm(const hg::SpadeArgs& a, int passes, bool bwd, cudaStream_t st, const char* who) {
  const int tiles = a.B * ((a.HW + 127) / 128);
  const int grid = tiles < hg::num_sms() ? tiles : hg::num_sms();
  cudaError_t e;
#define HG_LAUNCH_G(KERNEL)                                                                             \
  do {                                                                                                  \
    e = cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, hg::kSynSmemBytes);   \
    if (e == cudaSuccess) KERNEL<<<grid, hg::kSynThreads, hg::kSynSmemBytes, st>>>(a);                   \
  } while (0)
  if (bwd) {
    if (passes == 3) HG_LAUNCH_G((hg::spade_const_kernel<3, true>)); else HG_LAUNCH_G((hg::spade_const_kernel<1, true>));
  } else {
    if (passes == 3) HG_LAUNCH_G((hg::spade_const_kernel<3, false>)); else HG_LAUNCH_G((hg::spade_const_kernel<1, false>));
  }
#undef HG_LAUNCH_G
  if (e != cudaSuccess) { hg::set_error("%s: smem opt-in failed: %s", who, cudaGetErrorString(e)); return 2; }
  return hg::check_launch(who);
}

int hg_spade_bwd_dgrad(const float* dout, const float* x, long x_bstride, const float* mod, const void* wimg_t, float* dpre,
                       double* sums, int B, int C, int Hg, int Wg, int passes, void* stream) {
  HG_REQUIRE(C == hg::kC, "hg_spade_bwd_dgrad: only %d channels are supported (got %d)", hg::kC, C);
  HG_REQUIRE(dout && x && mod && wimg_t && dpre && sums, "hg_spade_bwd_dgrad: null pointer");
  HG_REQUIRE(passes == 1 || passes == 3, "hg_spade_bwd_dgrad: passes must be 1 or 3");
  HG_REQUIRE(B > 0 && Hg > 0 && Wg > 0, "hg_spade_bwd_dgrad: bad shape");
  const long T = (Hg * Wg + 127) / 128;
  hg::SpadeArgs a{};
  a.x = dout;
  a.x_bstride = T * hg::kC * 128;
  a.mod = mod;
  a.wimg = static_cast<const uint8_t*>(wimg_t);
  a.bias = mod;            // unused by the backward epilogue; init_common reads C floats
  a.skip = x;
  a.skip_bstride = x_bstride;
  a.out = dpre;
  a.stats = sums;
  a.B = B; a.HW = Hg * Wg; a.Hg = Hg; a.Wg = Wg;
  a.nkc = 4; a.xC = hg::kC; a.slope = 0.2f; a.cout = hg::kC;
  return launch_blocked_gemm(a, passes, true, static_cast<cudaStream_t>(stream), "hg_spade_bwd_dgrad");
}

int hg_conv1x1_blocked(const float* x, int Cin, const void* wimg, const float* bias, float* out, int B, int Hg, int Wg,
                       int passes, void* stream) {
  HG_REQUIRE(x && wimg && bias && out, "hg_conv1x1_blocked: null pointer");
  HG_REQUIRE(Cin == 64 || Cin == 128 || Cin == 256, "hg_conv1x1_blocked: Cin must be 64, 128 or 256 (got %d)", Cin);
  HG_REQUIRE(passes == 1 || passes == 3, "hg_conv1x1_blocked: passes must be 1 or 3");
  HG_REQUIRE(B > 0 && Hg > 0 && Wg > 0, "hg_conv1x1_blocked: bad shape");
  const long T = (Hg * Wg + 127) / 128;
  hg::SpadeArgs a{};
  a.x = x;
  a.x_bstride = T * Cin * 128;
  a.wimg = static_cast<const uint8_t*>(wimg);
  a.bias = bias;
  a.skip_bstride = T * hg::kC * 128;
  a.out = out;
  a.B = B; a.HW = Hg * Wg; a.Hg = Hg; a.Wg = Wg;
  a.nkc = Cin / 64; a.xC = Cin; a.slope = 1.f; a.cout = hg::kC;
  return launch_blocked_gemm(a, passes, false, static_cast<cudaStream_t>(stream), "hg_conv1x1_blocked");
}

int hg_act_conv1x1_blocked(const float* x, const float* x2, const float* mod, int act, const void* wimg, const float* bias,
                           float* out, int B, int Hg, int Wg, int passes, void* stream) {
  HG_REQUIRE(x && mod && wimg && bias && out, "hg_act_conv1x1_blocked: null pointer");
  HG_REQUIRE(act == 0 || act == 1, "hg_act_conv1x1_blocked: act must be 0 (LeakyReLU 0.2) or 1 (sine)");
  HG_REQUIRE(passes == 1 || passes == 3, "hg_act_conv1x1_blocked: passes must be 1 or 3");
  HG_REQUIRE(B > 0 && Hg > 0 && Wg > 0, "hg_act_conv1x1_blocked: bad shape");
  const long T = (Hg * Wg + 127) / 128;
  hg::SpadeArgs a{};
  a.x = x;
  a.x_bstride = T * hg::kC * 128;
  a.x2 = x2;
  a.mod = mod;
  a.wimg = static_cast<const uint8_t*>(wimg);
  a.bias = bias;
  a.skip_bstride = T * hg::kC * 128;
  a.out = out;
  a.B = B; a.HW = Hg * Wg; a.Hg = Hg; a.Wg = Wg;
  a.nkc = x2 ? 8 : 4; a.xC = hg::kC; a.slope = 0.2f; a.cout = hg::kC; a.act = act;
  return launch_blocked_gemm(a, passes, false, static_cast<cudaStream_t>(stream), "hg_act_conv1x1_blocked");
}

int hg_blocked_conv_wide(const float* x, const float* x2, const float* mod, const float* mod2, int act, float slope,
                         const void* wimg, const float* bias, const float* skip, float* out, double* stats,
                         const float* rgb_w, const float* rgb_b, const float* rgb_in, float* rgb_out, int B, int Hg, int Wg,
                         int passes, void* stream) {
  HG_REQUIRE(x && wimg && bias && out, "hg_blocked_conv_wide: null pointer");
  HG_REQUIRE(act == 0 || act == 1, "hg_blocked_conv_wide: act must be 0 (LeakyReLU(slope)) or 1 (sine)");
  HG_REQUIRE(!mod2 || (mod && x2), "hg_blocked_conv_wide: mod2 needs mod and a second source");
  HG_REQUIRE(!rgb_w || (rgb_b && rgb_out), "hg_blocked_conv_wide: rgb_b / rgb_out missing");
  HG_REQUIRE(passes == 1 || passes == 3, "hg_blocked_conv_wide: passes must be 1 or 3");
  HG_REQUIRE(B > 0 && Hg > 0 && Wg > 0, "hg_blocked_conv_wide: bad shape");
  const long T = (Hg * Wg + 127) / 128;
  hg::SpadeArgs a{};
  a.x = x;
  a.x_bstride = T * hg::kC * 128;
  a.x2 = x2;
  a.mod = mod;
  a.mod2 = mod2;
  a.wimg = static_cast<const uint8_t*>(wimg);
  a.bias = bias;
  a.skip = skip;
  a.skip_bstride = T * hg::kC * 128;
  a.out = out;
  a.stats = stats;
  a.rgb_w = rgb_w; a.rgb_b = rgb_b; a.rgb_in = rgb_in; a.rgb_out = rgb_out;
  a.B = B; a.HW = Hg * Wg; a.Hg = Hg; a.Wg = Wg;
  a.nkc = x2 ? 8 : 4; a.xC = hg::kC; a.slope = slope; a.cout = hg::kC; a.act = act;
  return launch_blocked_gemm(a, passes, false, static_cast<cudaStream_t>(stream), "hg_blocked_conv_wide");
}

int hg_conv1x1_blocked_bwd(const float* g, const float* g2, const float* aux, const float* mod, const void* wimg_t,
                           float* out, double* sums, int Cout, float slope, int pixel_major, int act, const float* ascale,
                           const float* rk_w, const float* rk_v, int rk_n, int B, int Hg, int Wg, int passes,
                           void* stream) {
  HG_REQUIRE(act == 0 || act == 1, "hg_conv1x1_blocked_bwd: act must be 0 (LeakyReLU/ReLU mask) or 1 (cosine)");
  HG_REQUIRE(!rk_v || (rk_w && rk_n >= 1 && rk_n <= 3 && Cout == 256), "hg_conv1x1_blocked_bwd: bad rank-k term");
  HG_REQUIRE(g && aux && wimg_t && out && sums, "hg_conv1x1_blocked_bwd: null pointer");
  HG_REQUIRE(Cout == 128 || Cout == 256, "hg_conv1x1_blocked_bwd: Cout must be 128 or 256 (got %d)", Cout);
  HG_REQUIRE(!pixel_major || Cout == 128, "hg_conv1x1_blocked_bwd: the pixel-major output is built for Cout == 128");
  HG_REQUIRE(!(act == 1 && pixel_major) && !(act == 0 && rk_v),
             "hg_conv1x1_blocked_bwd: compiled epilogues are sine [+ rank-k term] / LeakyReLU [+ pixel-major output]");
  HG_REQUIRE(passes == 1 || passes == 3, "hg_conv1x1_blocked_bwd: passes must be 1 or 3");
  HG_REQUIRE(B > 0 && Hg > 0 && Wg > 0, "hg_conv1x1_blocked_bwd: bad shape");
  const long T = (Hg * Wg + 127) / 128;
  hg::SpadeArgs a{};
  a.x = g;
  a.x_bstride = T * hg::kC * 128;
  a.x2 = g2;
  a.mod = mod;
  a.wimg = static_cast<const uint8_t*>(wimg_t);
  a.bias = static_cast<const float*>(wimg_t);   // unused by the backward epilogue; init_common reads C floats
  a.skip = aux;
  a.skip_bstride = T * Cout * 128;
  a.out = out;
  a.stats = sums;
  a.B = B; a.HW = Hg * Wg; a.Hg = Hg; a.Wg = Wg;
  a.nkc = g2 ? 8 : 4; a.xC = hg::kC; a.slope = slope; a.cout = Cout; a.out_pm = pixel_major;
  a.act = act; a.ascale = ascale; a.rgb_w = rk_v ? rk_w : nullptr; a.rk_v = rk_v; a.rk_n = rk_n;
  return launch_blocked_gemm(a, passes, true, static_cast<cudaStream_t>(stream), "hg_conv1x1_blocked_bwd");
}

#ifdef HG_SPADE_PROFILE
// nanoseconds per phase summed over the warpgroups of every const-style launch since the last read, then the count of
// warpgroup-tiles; clears the sums
int hg_spade_profile_read(unsigned long long* host) {
  unsigned long long zero[hg::kProfPhases + 1] = {};
  if (cudaMemcpyFromSymbol(host, hg::g_spade_prof, sizeof(zero)) != cudaSuccess ||
      cudaMemcpyToSymbol(hg::g_spade_prof, zero, sizeof(zero)) != cudaSuccess)
    return 1;
  return 0;
}
#endif

int hg_bn_finalize(const double* stats, double count, const double* count_dev, const float* weight, const float* bias, float* running_mean,
                   float* running_var, int training, float eps, float momentum, const float* gb, int B, int C,
                   float* scsh, float* mod, void* stream) {
  HG_REQUIRE(C == hg::kC, "hg_bn_finalize: only %d channels are supported (got %d)", hg::kC, C);
  HG_REQUIRE(weight && bias && (scsh || mod), "hg_bn_finalize: null pointer");
  HG_REQUIRE(training ? (stats != nullptr && (count > 0 || count_dev)) : (running_mean && running_var),
             "hg_bn_finalize: statistics missing");
  hg::bn_finalize_kernel<<<1, hg::kC, 0, static_cast<cudaStream_t>(stream)>>>(
      stats, count, count_dev, weight, bias, running_mean, running_var, training, eps, momentum, gb, B, scsh, mod);
  return hg::check_launch("hg_bn_finalize");
}

int hg_synth_input(const float* w, const float* bias, const float* ic, const float* jc, int C, int Hg, int Wg,
                   float* x0, double* stats, int batch, void* stream) {
  HG_REQUIRE(C == hg::kC, "hg_synth_input: only %d channels are supported (got %d)", hg::kC, C);
  HG_REQUIRE(w && bias && ic && jc && x0, "hg_synth_input: null pointer");
  const int HW = Hg * Wg;
  int bx = (HW + 255) / 256;
  if (bx > 32) bx = 32;
  dim3 grid(bx, C);
  hg::synth_input_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(w, bias, ic, jc, Hg, Wg, x0, stats,
                                                                              static_cast<double>(batch));
  return hg::check_launch("hg_synth_input");
}

}  // extern "C"
