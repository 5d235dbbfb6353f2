// Fused pose-mapping renderer: per-point FiLM-SIREN MLP + alpha compositing along each ray.
//
// Replaces (reference file:line):
//   COORDCONCATSIREN.forward        lib/implicit_funcitions/modulated.py:41-75
//   SineLayer / FiLMLayer           lib/components/pigan_layers.py:63-87
//   vr.ray_integration              lib/generators/volume_rendering.py:12-56
//   the [B,N,F+4] / [B,N,256..512] intermediates of Map3DGenerator.render (map3d_generator.py:427-515)
//
// A CTA owns tiles of 128 sample points = (128/S) whole rays; warpgroup g owns points 64g..64g+63 and runs the MLP for them
// on wgmma with the activations never leaving the SM (accumulator -> sin(F*acc + P) -> bf16 hi/lo operand -> next wgmma),
// while warp 8 streams the weight tiles from L2.  FiLM frequency/phase, bias and the x30 of the sine layers are folded into
// one (F, P) table per layer and sample (host side); only [rays, 256 feat + 3 rgb + depth] ever reaches HBM.
//
// Layer schedule per tile (one [64 x 256] fp32 accumulator per warpgroup; the weight blob holds the stages in this order):
//   L0c  rec[K=64: xyz*s, geo31, 0] x W01(coord)               -> acc -> kept in per-thread local memory (coord pre-act)
//   L0g  rec x W01(geo)                                         -> acc
//   E1   g = sin(30*(acc+b))                                    -> operand
//   L1b  g x Wn0[:, 256:512]                                    -> acc
//   E0   a = sin(30*(coord pre-act + b))                        -> operand
//   L1a  a x Wn0[:, 0:256]                                      -> acc (accumulate)
//   E2..E4  x = sin(F*(acc+b)+P) ; L: network.1..3             -> acc
//   E5   x4 (+ sigma head) ; L: color_layer_sine[:, 3:]        -> acc       (view-direction term in P)
//   E6   c (+ rgb head)    ; L: feature_layer_linear           -> acc
//   E7   feat + compositing
#include "common.cuh"
#include "wgmma.cuh"

namespace hg {

constexpr int kRH = 256;           // hidden_dim == feature_dim
constexpr int kRenThreads = 384;   // warpgroups 0-1 rows, warp 8 weight producer
constexpr int kRenStages = 2;
constexpr uint32_t kRA = 128 * 128;   // operand chunk [128 x 64] bf16
constexpr uint32_t kRB = 256 * 128;   // weight stage  [256 x 64] bf16
constexpr int kFilmLayers = 7;        // coord, geo, network.0..3, color
constexpr int kWeightStages = 60;     // per tile, hi+lo (see schedule above)
constexpr int kRayOut = 260;          // floats per ray: 256 feat, 3 rgb, depth
constexpr int kScr = 65;              // row stride (floats) of the compositing scratch

struct RenderArgs {
  const float* rec;      // [B,N,36] point records (geo.cu)
  const float* z_vals;   // [B,N]
  const float* noise;    // [B,N] N(0,1) draws or null
  const float* film;     // [B,7,2,256]: per layer F (multiplier) and P (offset): x = sin(F*acc + P)
  const uint8_t* wblob;  // 60 packed weight stages in schedule order
  const float* w_sigma;  // [256]
  const float* w_rgb;    // [3,256]
  const float* b_feat;   // [256]
  const float* heads_b;  // [4]: b_sigma, b_rgb[3]
  float* ray_out;        // [B,R,260]
  float* weights_out;    // [B,N] or null
  float* raw_out;        // [B,N,260] per-point (rgb 3, feat 256, sigma) instead of compositing, or null
  int B, R, S;           // rays per image, samples per ray (power of two <= 128)
  float noise_std;
  int white_back, last_back, clamp_softplus;
};

struct RenSmem {
  uint8_t* a_hi;
  uint8_t* a_lo;
  uint8_t* b_st;
  float* film;     // [7][2][256]
  float* w_sigma;  // [256]
  float* w_rgb;    // [3][256]
  float* b_feat;   // [256]
  float* part;     // [128][4] sigma / rgb dots per point
  float* tr;       // [128] 1 - alpha + 1e-12
  float* wgt;      // [128] compositing weights
  float* zs;       // [128]
  float* rayw;     // [128] per-ray sum of weights (first rays_per_tile entries)
  uint64_t* bars;
};
constexpr uint32_t kRenFloats = kFilmLayers * 2 * kRH + kRH + 3 * kRH + kRH + 128 * 4 + 4 * 128;
constexpr uint32_t kRenSmemBytes = 8 * kRA + kRenStages * kRB + kRenFloats * 4 + 16 * 8 + 1024;

__device__ __forceinline__ RenSmem ren_carve(uint8_t* raw) {
  uint8_t* s = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~uintptr_t(1023));
  RenSmem m;
  m.a_hi = s;
  m.a_lo = s + 4 * kRA;
  m.b_st = s + 8 * kRA;
  float* f = reinterpret_cast<float*>(m.b_st + kRenStages * kRB);
  m.film = f; f += kFilmLayers * 2 * kRH;
  m.w_sigma = f; f += kRH;
  m.w_rgb = f; f += 3 * kRH;
  m.b_feat = f; f += kRH;
  m.part = f; f += 128 * 4;
  m.tr = f; f += 128;
  m.wgt = f; f += 128;
  m.zs = f; f += 128;
  m.rayw = f; f += 128;
  m.bars = reinterpret_cast<uint64_t*>(f);
  return m;
}
enum { RB_FULL = 0 /*2*/, RB_EMPTY = 2 /*2*/ };

__device__ __forceinline__ void ren_rows_barrier() { named_barrier(1, 256); }

// sin(t) for |t| up to a few thousand: two-term Cody-Waite reduction by 2*pi, then the SFU sine on
// [-pi, pi] (abs error ~2^-21).  The reference path evaluates torch.sin on fp32 tensors.
__device__ __forceinline__ float sin_reduced(float t) {
  const float y = t * 0.15915494309189535f;
  const float k = (y + 12582912.f) - 12582912.f;  // round to nearest integer (|y| < 2^22)
  float r = fmaf(-k, 6.2831854820251465f, t);
  r = fmaf(-k, -1.7484555314695172e-07f, r);
  return __sinf(r);
}

// the same evaluation on a pair
__device__ __forceinline__ float2 sin_reduced2(float2 t) {
  const float2 y = fmul2(t, make_float2(0.15915494309189535f, 0.15915494309189535f));
  const float2 big = make_float2(12582912.f, 12582912.f), nbig = make_float2(-12582912.f, -12582912.f);
  const float2 k = fadd2(fadd2(y, big), nbig);
  float2 r = ffma2(k, make_float2(-6.2831854820251465f, -6.2831854820251465f), t);
  r = ffma2(k, make_float2(1.7484555314695172e-07f, 1.7484555314695172e-07f), r);
  return make_float2(__sinf(r.x), __sinf(r.y));
}

// two consecutive-k fp32 values (k even) of one row -> the hi (and lo) operand tiles
template <bool kSplit>
__device__ __forceinline__ void store_a2(uint8_t* tile_hi, uint8_t* tile_lo, uint32_t row, uint32_t k, float x0, float x1) {
  uint32_t h, l;
  split_bf16x2(x0, x1, h, l);
  const uint32_t off = sw128_offset(row, k);
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(smem_u32(tile_hi) + off), "r"(h));
  if (kSplit) asm volatile("st.shared.b32 [%0], %1;" ::"r"(smem_u32(tile_lo) + off), "r"(l));
}

// per-thread spill slot of one accumulator (the coord pre-activation waits there while the geo half of network.0 runs)
__device__ __forceinline__ void stash_store(float* slot, const float (&d)[128]) {
  const uint32_t base = static_cast<uint32_t>(__cvta_generic_to_local(slot));
#pragma unroll
  for (int i = 0; i < 128; i += 4)
    asm volatile("st.local.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(base + i * 4), "f"(d[i]), "f"(d[i + 1]), "f"(d[i + 2]), "f"(d[i + 3])
                 : "memory");
}
__device__ __forceinline__ float4 stash_load4(const float* slot, int i) {
  float4 v;
  asm volatile("ld.local.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "r"(static_cast<uint32_t>(__cvta_generic_to_local(slot)) + i * 4)
               : "memory");
  return v;
}

// Activation epilogue of one layer for warpgroup g: accumulator fragments -> x = sin(F*acc + P) -> bf16 hi/lo operand.
// kHead: 0 none, 1 sigma dot (1 value), 2 rgb dots (3 values) of each point -> part[row][*].  kStash: the fragments come
// from the per-thread stash instead of `d` (which is left untouched).
template <int kPasses, int kHead, bool kStash = false>
__device__ __forceinline__ void film_epilogue(const RenSmem& m, const float (&d)[128], const float* stash, int layer, int g, int t) {
  uint32_t F = smem_u32(m.film + (layer * 2 + 0) * kRH);
  uint32_t P = smem_u32(m.film + (layer * 2 + 1) * kRH);
  opaque(F);   // the per-sample FiLM table is refreshed between tiles: table loads stay inside this call
  opaque(P);
  float dots[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int c = frag_col(t, j, 0);
    float f2[2], p2[2];
    asm("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(f2[0]), "=f"(f2[1]) : "r"(F + c * 4));
    asm("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(p2[0]), "=f"(p2[1]) : "r"(P + c * 4));
    float v[4] = {d[4 * j], d[4 * j + 1], d[4 * j + 2], d[4 * j + 3]};
    if (kStash) {
      const float4 q = stash_load4(stash, 4 * j);
      v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float2 x = sin_reduced2(ffma2(make_float2(f2[0], f2[1]), make_float2(v[2 * i], v[2 * i + 1]),
                                          make_float2(p2[0], p2[1])));
      if (kHead == 1) dots[i][0] = fmaf(x.y, m.w_sigma[c + 1], fmaf(x.x, m.w_sigma[c], dots[i][0]));
      if (kHead == 2) {
#pragma unroll
        for (int h = 0; h < 3; ++h) dots[i][h] = fmaf(x.y, m.w_rgb[h * kRH + c + 1], fmaf(x.x, m.w_rgb[h * kRH + c], dots[i][h]));
      }
      const int kc = c >> 6;
      store_a2<kPasses == 3>(m.a_hi + kc * kRA, m.a_lo + kc * kRA, g * 64 + frag_row(t, i), c & 63, x.x, x.y);
    }
  }
  if (kHead != 0) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
      for (int h = 0; h < 3; ++h) {
        if (kHead == 1 && h > 0) break;
        float v = dots[i][h];
        v += __shfl_xor_sync(0xffffffffu, v, 1);
        v += __shfl_xor_sync(0xffffffffu, v, 2);
        if ((t & 3) == 0) m.part[(g * 64 + frag_row(t, i)) * 4 + (kHead == 1 ? 0 : 1 + h)] = v;
      }
    }
  }
  fence_proxy_async_smem();
  named_barrier(2 + g, 128);
}

template <int kPasses>
__global__ void __launch_bounds__(kRenThreads, 1) render_mlp_kernel(RenderArgs a) {
  extern __shared__ uint8_t smem_raw[];
  const RenSmem m = ren_carve(smem_raw);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < kRH; i += blockDim.x) {
    m.w_sigma[i] = a.w_sigma[i];
    m.b_feat[i] = a.b_feat[i];
  }
  for (int i = threadIdx.x; i < 3 * kRH; i += blockDim.x) m.w_rgb[i] = a.w_rgb[i];
  if (threadIdx.x == 0) {
    for (int i = 0; i < kRenStages; ++i) {
      mbar_init(m.bars + RB_FULL + i, 1);
      mbar_init(m.bars + RB_EMPTY + i, 2);     // one arrival per warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int S = a.S;
  const int rpt = 128 / S;                               // rays per tile
  const int tiles_per_img = (a.R + rpt - 1) / rpt;
  const int num_tiles = a.B * tiles_per_img;
  const int my_tiles = (num_tiles - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);
  const long N = static_cast<long>(a.R) * S;

  if (warp < 8) {
    regs_inc<kMmaRegs>();
    const int g = warp >> 2, t = threadIdx.x & 127;
    const int tid = threadIdx.x;                         // 0..255: per-point scalar work uses point row = tid (< 128)
    float d[128];
    __align__(16) float stash[128];
    uint32_t st = 0, ph = 0;
    // one weight stage: wait, issue on this warpgroup's 64 rows, release the previous stage once its wgmmas are done
    uint32_t prev = ~0u;
    auto stage = [&](uint32_t a_tile, uint32_t a_tile2, bool two, bool accumulate) {
      mbar_wait(m.bars + RB_FULL + st, ph);
      acc_fence(d);
      wgmma_fence();
      const uint32_t bt = smem_u32(m.b_st + st * kRB);
      wg_k64<256>(d, a_tile, bt, accumulate);
      if (two) wg_k64<256>(d, a_tile2, bt, true);
      wgmma_commit();
      wgmma_wait<1>();
      acc_fence(d);
      if (prev != ~0u && t == 0) mbar_arrive(m.bars + RB_EMPTY + prev);
      prev = st;
      if (++st == kRenStages) { st = 0; ph ^= 1; }
    };
    // one GEMM of K = 64 * nk over operand chunks k0.. into the accumulator
    auto layer = [&](int k0, int nk, bool accumulate) {
      for (int kc = k0; kc < k0 + nk; ++kc) {
        const uint32_t ahi = smem_u32(m.a_hi + kc * kRA) + g * 64 * 128, alo = smem_u32(m.a_lo + kc * kRA) + g * 64 * 128;
        stage(ahi, alo, kPasses == 3, accumulate || kc > k0);
        if (kPasses == 3) stage(ahi, ahi, false, true);
      }
      wgmma_wait<0>();
      acc_fence(d);
      if (t == 0) mbar_arrive(m.bars + RB_EMPTY + prev);
      prev = ~0u;
    };
    int cur_b = -1;
    for (int it = 0; it < my_tiles; ++it) {
      const int tile = blockIdx.x + it * gridDim.x;
      const int b = tile / tiles_per_img;
      const int ray0 = (tile % tiles_per_img) * rpt;
      if (b != cur_b) {
        ren_rows_barrier();
        for (int i = tid; i < kFilmLayers * 2 * kRH; i += 256)
          m.film[i] = a.film[static_cast<long>(b) * kFilmLayers * 2 * kRH + i];
        cur_b = b;
        ren_rows_barrier();
      }
      // ---- A0: point record -> operand chunk 0 (K = 64: 36 values + zeros); thread t: row 64g + t/2, k half t&1
      {
        const int row = g * 64 + (t >> 1), kh = t & 1;
        const int rl = row / S, s = row % S;
        const int ray = ray0 + rl;
        const bool valid = ray < a.R;
        const long gp = static_cast<long>(b) * N + static_cast<long>(ray) * S + s;
        float x[8];
        const float4* rp = reinterpret_cast<const float4*>(a.rec + gp * 36);
#pragma unroll
        for (int gi = 0; gi < 4; ++gi) {
          const int k0 = kh * 32 + gi * 8;
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int f4 = (k0 >> 2) + u;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (valid && f4 < 9) v = __ldg(rp + f4);
            x[u * 4 + 0] = v.x; x[u * 4 + 1] = v.y; x[u * 4 + 2] = v.z; x[u * 4 + 3] = v.w;
          }
          store_a8<kPasses == 3>(m.a_hi, m.a_lo, row, k0, x);
        }
        if (kh == 0) m.zs[row] = (valid && a.z_vals) ? a.z_vals[gp] : 0.f;
        fence_proxy_async_smem();
        named_barrier(2 + g, 128);
      }
      // ---- MLP
      layer(0, 1, false);                                   // L0c
      stash_store(stash, d);
      layer(0, 1, false);                                   // L0g
      film_epilogue<kPasses, 0>(m, d, stash, 1, g, t);      // E1
      layer(0, 4, false);                                   // L1b
      film_epilogue<kPasses, 0, true>(m, d, stash, 0, g, t);  // E0 (coord pre-activation from the stash)
      layer(0, 4, true);                                    // L1a, accumulating onto L1b
      film_epilogue<kPasses, 0>(m, d, stash, 2, g, t);      // E2
      layer(0, 4, false);                                   // network.1
      film_epilogue<kPasses, 0>(m, d, stash, 3, g, t);      // E3
      layer(0, 4, false);                                   // network.2
      film_epilogue<kPasses, 0>(m, d, stash, 4, g, t);      // E4
      layer(0, 4, false);                                   // network.3
      film_epilogue<kPasses, 1>(m, d, stash, 5, g, t);      // E5 + sigma head
      layer(0, 4, false);                                   // color
      film_epilogue<kPasses, 2>(m, d, stash, 6, g, t);      // E6 + rgb heads
      layer(0, 4, false);                                   // feature

      ren_rows_barrier();                                   // heads of both warpgroups in part[], operands no longer read
      if (a.raw_out) {
        // ---- per-point outputs of COORDCONCATSIREN.forward (modulated.py:70-73): [rgb, feat, sigma]
        if (tid < 128) {
          const int row = tid, rl = row / S, s = row % S, ray = ray0 + rl;
          const long gp = static_cast<long>(b) * N + static_cast<long>(ray) * S + s;
          if (ray < a.R) {
            float* po = a.raw_out + gp * kRayOut;
            po[259] = m.part[row * 4] + a.heads_b[0];
            for (int j = 0; j < 3; ++j) {
              const float dot = m.part[row * 4 + 1 + j] + a.heads_b[1 + j];
              po[j] = 1.f / (1.f + expf(-dot));
            }
          }
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int row = g * 64 + frag_row(t, i), rl = row / S, s = row % S, ray = ray0 + rl;
          if (ray >= a.R) continue;
          float* po = a.raw_out + (static_cast<long>(b) * N + static_cast<long>(ray) * S + s) * kRayOut + 3;
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const int c = frag_col(t, j, 0);
            po[c] = d[4 * j + 2 * i] + m.b_feat[c];
            po[c + 1] = d[4 * j + 2 * i + 1] + m.b_feat[c + 1];
          }
        }
        ren_rows_barrier();
        continue;
      }
      // ---- compositing weights (volume_rendering.py:12-38)
      float alpha = 0.f;
      if (tid < 128) {
        const int row = tid, rl = row / S, s = row % S, ray = ray0 + rl;
        const long gp = static_cast<long>(b) * N + static_cast<long>(ray) * S + s;
        const bool valid = ray < a.R;
        const float sigma = m.part[row * 4] + a.heads_b[0];
        const float delta = (s == S - 1) ? 1e9f : m.zs[row + 1] - m.zs[row];
        float pre = sigma;
        if (a.noise) pre += (valid ? a.noise[gp] : 0.f) * a.noise_std;
        const float dens = a.clamp_softplus ? (pre > 20.f ? pre : log1pf(expf(pre))) : fmaxf(pre, 0.f);
        alpha = 1.f - expf(-delta * dens);
        m.tr[row] = 1.f - alpha + 1e-12f;
      }
      ren_rows_barrier();
      if (tid < 128) {
        const int row = tid, rl = row / S, s = row % S;
        float T = 1.f;
        for (int k = 0; k < s; ++k) T *= m.tr[rl * S + k];
        m.wgt[row] = ray0 + rl < a.R ? alpha * T : 0.f;
      }
      ren_rows_barrier();
      if (tid < rpt) {
        float W = 0.f;
        for (int k = 0; k < S; ++k) W += m.wgt[tid * S + k];
        m.rayw[tid] = W;
      }
      ren_rows_barrier();
      if (tid < 128) {
        const int row = tid, rl = row / S, s = row % S, ray = ray0 + rl;
        const float Wsum = m.rayw[rl];
        float w = m.wgt[row];
        const float w_depth = w + ((s == S - 1) ? 1.f - Wsum : 0.f);
        if (a.last_back) w = w_depth;
        if (a.weights_out && ray < a.R) a.weights_out[static_cast<long>(b) * N + static_cast<long>(ray) * S + s] = w;
        m.tr[row] = w;                                     // the weight actually applied (tr is free again)
        m.wgt[row] = w_depth;
      }
      ren_rows_barrier();

      // ---- E7: weighted feature sum over each ray, 64 columns at a time through a [128 x 65] scratch (operand buffer)
      float* scratch = reinterpret_cast<float*>(m.a_hi);
      const float wr[2] = {m.tr[g * 64 + frag_row(t, 0)], m.tr[g * 64 + frag_row(t, 1)]};
#pragma unroll
      for (int cg = 0; cg < 4; ++cg) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int row = g * 64 + frag_row(t, i);
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = cg * 8 + jj, c = frag_col(t, j, 0);
            scratch[row * kScr + (c & 63)] = wr[i] * (d[4 * j + 2 * i] + m.b_feat[c]);
            scratch[row * kScr + (c & 63) + 1] = wr[i] * (d[4 * j + 2 * i + 1] + m.b_feat[c + 1]);
          }
        }
        ren_rows_barrier();
        {
          const int col = tid & 63;
          for (int r2 = tid >> 6; r2 < rpt; r2 += 4) {
            float acc = 0.f;
            const float* src = scratch + (r2 * S) * kScr + col;
            for (int k = 0; k < S; ++k) acc += src[k * kScr];
            if (ray0 + r2 < a.R)
              a.ray_out[(static_cast<long>(b) * a.R + ray0 + r2) * kRayOut + cg * 64 + col] =
                  acc + (a.white_back ? 1.f - m.rayw[r2] : 0.f);
          }
        }
        ren_rows_barrier();
      }
      // rgb and depth: per point into the scratch, then one thread per ray
      if (tid < 128) {
        const int row = tid;
        const float w = m.tr[row];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          const float dot = m.part[row * 4 + 1 + j] + a.heads_b[1 + j];
          scratch[row * kScr + j] = w / (1.f + expf(-dot));
        }
        scratch[row * kScr + 3] = m.wgt[row] * m.zs[row];
      }
      ren_rows_barrier();
      if (tid < rpt && ray0 + tid < a.R) {
        float e[4] = {0.f, 0.f, 0.f, 0.f};
        for (int k = 0; k < S; ++k)
#pragma unroll
          for (int j = 0; j < 4; ++j) e[j] += scratch[(tid * S + k) * kScr + j];
        const float back = a.white_back ? 1.f - m.rayw[tid] : 0.f;
        float* ro = a.ray_out + (static_cast<long>(b) * a.R + ray0 + tid) * kRayOut;
        ro[256] = e[0] + back; ro[257] = e[1] + back; ro[258] = e[2] + back; ro[259] = e[3];
      }
      ren_rows_barrier();   // scratch is the next tile's operand buffer
    }
  } else {
    regs_dec<kProducerRegs>();
    if (warp == 8 && lane == 0) {
      uint32_t st = 0, ph = 0;
      for (int it = 0; it < my_tiles; ++it)
        for (int sidx = 0; sidx < kWeightStages; ++sidx) {
          if (kPasses == 1 && (sidx & 1)) continue;
          mbar_wait_backoff(m.bars + RB_EMPTY + st, ph ^ 1);
          mbar_arrive_expect_tx(m.bars + RB_FULL + st, kRB);
          bulk_g2s(m.b_st + st * kRB, a.wblob + static_cast<size_t>(sidx) * kRB, kRB, m.bars + RB_FULL + st);
          if (++st == kRenStages) { st = 0; ph ^= 1; }
        }
    }
  }
}

}  // namespace hg

extern "C" {

size_t hg_render_weight_blob_bytes(void) { return static_cast<size_t>(hg::kWeightStages) * hg::kRB; }

int hg_render_mlp(const float* rec, const float* z_vals, const float* noise, const float* film, const void* wblob,
                  const float* w_sigma, const float* w_rgb, const float* b_feat, const float* heads_b, float* ray_out,
                  float* weights_out, float* raw_out, int B, int R, int S, int hidden, float noise_std, int white_back, int last_back,
                  int clamp_softplus, int passes, void* stream) {
  HG_REQUIRE(hidden == hg::kRH, "hg_render_mlp: only hidden_dim == %d is supported (got %d)", hg::kRH, hidden);
  HG_REQUIRE(rec && film && wblob && w_sigma && w_rgb && b_feat && heads_b, "hg_render_mlp: null pointer");
  HG_REQUIRE(raw_out || (ray_out && z_vals), "hg_render_mlp: need ray_out + z_vals (compositing) or raw_out (per-point)");
  HG_REQUIRE(B > 0 && R > 0, "hg_render_mlp: bad shape");
  HG_REQUIRE(S >= 2 && S <= 128 && (S & (S - 1)) == 0, "hg_render_mlp: samples per ray must be a power of two in [2,128] (got %d)", S);
  HG_REQUIRE(passes == 1 || passes == 3, "hg_render_mlp: passes must be 1 or 3");
  HG_REQUIRE((reinterpret_cast<uintptr_t>(rec) & 15) == 0 && (reinterpret_cast<uintptr_t>(wblob) & 15) == 0,
             "hg_render_mlp: rec / wblob must be 16-byte aligned");
  hg::RenderArgs a{rec, z_vals, noise, film, static_cast<const uint8_t*>(wblob), w_sigma, w_rgb, b_feat, heads_b,
                   ray_out, weights_out, raw_out, B, R, S, noise_std, white_back, last_back, clamp_softplus};
  const int rpt = 128 / S;
  const int tiles = B * ((R + rpt - 1) / rpt);
  const int grid = tiles < hg::num_sms() ? tiles : hg::num_sms();
  auto st = static_cast<cudaStream_t>(stream);
  cudaError_t e;
  if (passes == 3) {
    e = cudaFuncSetAttribute(hg::render_mlp_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, hg::kRenSmemBytes);
    if (e != cudaSuccess) { hg::set_error("hg_render_mlp: smem opt-in failed: %s", cudaGetErrorString(e)); return 2; }
    hg::render_mlp_kernel<3><<<grid, hg::kRenThreads, hg::kRenSmemBytes, st>>>(a);
  } else {
    e = cudaFuncSetAttribute(hg::render_mlp_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, hg::kRenSmemBytes);
    if (e != cudaSuccess) { hg::set_error("hg_render_mlp: smem opt-in failed: %s", cudaGetErrorString(e)); return 2; }
    hg::render_mlp_kernel<1><<<grid, hg::kRenThreads, hg::kRenSmemBytes, st>>>(a);
  }
  return hg::check_launch("hg_render_mlp");
}

}  // extern "C"
