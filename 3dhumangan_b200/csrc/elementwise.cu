// bias_act and upfirdn2d: the two StyleGAN3 native ops the reference ships as CUDA plugins
// (lib/components/ops/bias_act.cu:24-165, lib/components/ops/upfirdn2d.cu:29-375), rebuilt as
// vectorised HBM-streaming kernels for sm_90a.  Both are bandwidth-bound (<= 10 FLOP/B).
#include <cuda.h>
#include <cudaTypedefs.h>
#include <string.h>
#include "common.cuh"
#include "wgmma.cuh"

namespace hg {

// activation ids follow bias_act.cpp / bias_act.py:22-32: 1 linear, 2 relu, 3 lrelu, 4 tanh, 5 sigmoid,
// 6 elu, 7 selu, 8 softplus, 9 swish
__device__ __forceinline__ float act_apply(float x, int act, float alpha) {
  switch (act) {
    case 2: return x > 0.f ? x : 0.f;
    case 3: return x > 0.f ? x : x * alpha;
    case 4: return tanhf(x);
    case 5: return 1.f / (1.f + expf(-x));
    case 6: return x > 0.f ? x : expm1f(x);
    case 7: return 1.0507009873554805f * (x > 0.f ? x : 1.6732632423543772f * expm1f(x));
    case 8: return x > 20.f ? x : log1pf(expf(x));
    case 9: return x / (1.f + expf(-x));
    default: return x;
  }
}

// One float4 per lane and iteration, two iterations in flight; Idx = uint32_t whenever the tensor has < 2^32
// elements (a 64-bit division per element costs more than the activation).  kVecBias: stepB % 4 == 0, so the
// four lanes of a float4 share one bias element.
template <typename Idx, bool kVecBias>
__global__ void __launch_bounds__(256) bias_act_kernel(const float* __restrict__ x, const float* __restrict__ b,
                                                       float* __restrict__ y, long n, Idx stepB, Idx sizeB, int act,
                                                       float alpha, float gain, float clamp) {
  const Idx nvec = static_cast<Idx>(n >> 2);
  const Idx stride = static_cast<Idx>(gridDim.x) * blockDim.x;
  const float4* x4 = reinterpret_cast<const float4*>(x);
  float4* y4 = reinterpret_cast<float4*>(y);
  auto apply = [&](float4 t, Idx i) {
    float v[4] = {t.x, t.y, t.z, t.w};
    if (b) {
      const Idx e = i * 4;
      if (kVecBias) {
        const float bb = __ldg(b + (e / stepB) % sizeB);
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] += bb;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] += __ldg(b + ((e + j) / stepB) % sizeB);
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float u = act_apply(v[j], act, alpha) * gain;
      if (clamp >= 0.f) u = fminf(fmaxf(u, -clamp), clamp);
      v[j] = u;
    }
    return make_float4(v[0], v[1], v[2], v[3]);
  };
  Idx i = static_cast<Idx>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (; i + stride < nvec; i += 2 * stride) {
    const float4 t0 = __ldcs(x4 + i), t1 = __ldcs(x4 + i + stride);
    __stcs(y4 + i, apply(t0, i));
    __stcs(y4 + i + stride, apply(t1, i + stride));
  }
  if (i < nvec) __stcs(y4 + i, apply(__ldcs(x4 + i), i));
  // tail (n % 4 elements)
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long e = (n & ~3L) + threadIdx.x;
    float u = x[e];
    if (b) u += b[(e / static_cast<long>(stepB)) % static_cast<long>(sizeB)];
    u = act_apply(u, act, alpha) * gain;
    if (clamp >= 0.f) u = fminf(fmaxf(u, -clamp), clamp);
    y[e] = u;
  }
}

// First / second derivative of act at the pre-activation t, written in terms of the saved forward OUTPUT
// (yy = y / gain) wherever the function allows it, so that backward never needs the forward input
// (bias_act.py:22-32 `ref='y'`; swish is the one activation that needs t itself).  order 1: act'(t), 2: act''(t).
__device__ __forceinline__ float act_derivative(float t, float yy, int act, float alpha, int order) {
  const float kS = 1.0507009873554805f, kSA = 1.0507009873554805f * 1.6732632423543772f;
  if (order == 1) {
    switch (act) {
      case 2: return yy > 0.f ? 1.f : 0.f;
      case 3: return yy > 0.f ? 1.f : alpha;
      case 4: return 1.f - yy * yy;
      case 5: return yy * (1.f - yy);
      case 6: return yy >= 0.f ? 1.f : yy + 1.f;
      case 7: return yy >= 0.f ? kS : yy + kSA;
      case 8: return 1.f - expf(-yy);
      case 9: { const float s = 1.f / (1.f + expf(-t)); return s * (1.f + t * (1.f - s)); }
      default: return 1.f;
    }
  }
  switch (act) {
    case 4: return (1.f - yy * yy) * (-2.f * yy);
    case 5: return yy * (1.f - yy) * (1.f - 2.f * yy);
    case 6: return yy >= 0.f ? 0.f : yy + 1.f;
    case 7: return yy >= 0.f ? 0.f : yy + kSA;
    case 8: { const float c = expf(-yy); return c * (1.f - c); }
    case 9: { const float s = 1.f / (1.f + expf(-t)); const float q = s * (1.f - s); return 2.f * q + t * q * (1.f - 2.f * s); }
    default: return 0.f;
  }
}

// out = g * gain * act^(order)(xref + b) * dy, zero where the forward output was clamped.
template <typename Idx>
__global__ void __launch_bounds__(256) bias_act_grad_kernel(const float* __restrict__ g, const float* __restrict__ b,
                                     const float* __restrict__ xref, const float* __restrict__ yref,
                                     const float* __restrict__ dy, float* __restrict__ out, long n, Idx stepB, Idx sizeB,
                                     int order, int act, float alpha, float gain, float clamp) {
  const float inv_gain = gain != 0.f ? 1.f / gain : 0.f;
  auto one = [&](float gv, float t, float y, float d) {
    if (act == 9) y = act_apply(t, 9, alpha) * gain;       // swish keeps x, not y: rebuild y for the clamp mask
    float v = gv * gain * act_derivative(t, y * inv_gain, act, alpha, order) * d;
    if (clamp >= 0.f && !(y > -clamp && y < clamp)) v = 0.f;
    return v;
  };
  const Idx nvec = static_cast<Idx>(n >> 2);
  const Idx stride = static_cast<Idx>(gridDim.x) * blockDim.x;
  const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f), one4 = make_float4(1.f, 1.f, 1.f, 1.f);
  for (Idx i = static_cast<Idx>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    const float4 g4 = __ldcs(reinterpret_cast<const float4*>(g) + i);
    float4 t4 = xref ? __ldcs(reinterpret_cast<const float4*>(xref) + i) : zero4;
    const float4 y4 = yref ? __ldcs(reinterpret_cast<const float4*>(yref) + i) : zero4;
    const float4 d4 = dy ? __ldcs(reinterpret_cast<const float4*>(dy) + i) : one4;
    if (b) {
      const Idx e = i * 4;
      t4.x += __ldg(b + (e / stepB) % sizeB);
      t4.y += __ldg(b + ((e + 1) / stepB) % sizeB);
      t4.z += __ldg(b + ((e + 2) / stepB) % sizeB);
      t4.w += __ldg(b + ((e + 3) / stepB) % sizeB);
    }
    __stcs(reinterpret_cast<float4*>(out) + i,
           make_float4(one(g4.x, t4.x, y4.x, d4.x), one(g4.y, t4.y, y4.y, d4.y), one(g4.z, t4.z, y4.z, d4.z),
                       one(g4.w, t4.w, y4.w, d4.w)));
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long e = (n & ~3L) + threadIdx.x;
    float t = xref ? xref[e] : 0.f;
    if (b) t += b[(e / static_cast<long>(stepB)) % static_cast<long>(sizeB)];
    out[e] = one(g[e], t, yref ? yref[e] : 0.f, dy ? dy[e] : 1.f);
  }
}

// out[n,c,oy,ox] = sum_{ky,kx} xup[oy*downy + ky - pady0, ox*downx + kx - padx0] * g[ky,kx]
// where xup is x with (up-1) zeros inserted and g is the (optionally pre-flipped) filter.  Polyphase form: only
// the taps with (o*down + k - pad0) % up == 0 touch a sample, i.e. k = k0, k0+up, ... with consecutive
// input indices, so the inner loops carry no division.  One thread per output, x fastest (coalesced loads and
// stores; tap re-use is served by L1/L2).  grid: (ceil(outW/128), outH chunks, NC chunks).
__global__ void __launch_bounds__(128) upfirdn2d_kernel(const float* __restrict__ x, const float* __restrict__ f,
                                                        float* __restrict__ y, int NC, int inH, int inW, int outH,
                                                        int outW, int fH, int fW, int upx, int upy, int downx, int downy,
                                                        int padx0, int pady0, int flip, float gain) {
  extern __shared__ float sf[];
  for (int i = threadIdx.x; i < fH * fW; i += blockDim.x) {
    // conv2d is a cross-correlation: the reference flips the filter unless flip_filter (upfirdn2d.py:200-203)
    const int ky = i / fW, kx = i % fW;
    sf[i] = (flip ? f[i] : f[(fH - 1 - ky) * fW + (fW - 1 - kx)]) * gain;
  }
  __syncthreads();
  const int ox = blockIdx.x * blockDim.x + threadIdx.x;
  if (ox >= outW) return;
  // horizontal phase of this column: first tap kx0 >= 0 with (ox*downx + kx0 - padx0) % upx == 0
  const int bx = ox * downx - padx0;
  int kx0 = ((-bx) % upx + upx) % upx;
  int ix0 = (bx + kx0) / upx;                        // exact division (may be negative)
  if (ix0 < 0) { kx0 += -ix0 * upx; ix0 = 0; }
  int nx = kx0 < fW ? (fW - kx0 + upx - 1) / upx : 0;
  if (ix0 + nx > inW) nx = inW - ix0;
  for (int nc = blockIdx.z; nc < NC; nc += gridDim.z) {
    const float* xp = x + static_cast<long>(nc) * inH * inW;
    float* yp = y + static_cast<long>(nc) * outH * outW;
    // a contiguous band of rows per block: consecutive output rows re-read the same input rows (L1 hits)
    const int band = (outH + gridDim.y - 1) / gridDim.y;
    const int oy_end = min(outH, static_cast<int>(blockIdx.y + 1) * band);
    for (int oy = blockIdx.y * band; oy < oy_end; ++oy) {
      const int by = oy * downy - pady0;
      int ky0 = ((-by) % upy + upy) % upy;
      int iy0 = (by + ky0) / upy;
      if (iy0 < 0) { ky0 += -iy0 * upy; iy0 = 0; }
      int ny = ky0 < fH ? (fH - ky0 + upy - 1) / upy : 0;
      if (iy0 + ny > inH) ny = inH - iy0;
      float acc = 0.f;
      for (int a = 0; a < ny; ++a) {
        const float* row = xp + static_cast<long>(iy0 + a) * inW + ix0;
        const float* frow = sf + (ky0 + a * upy) * fW + kx0;
        for (int c = 0; c < nx; ++c) acc = fmaf(__ldg(row + c), frow[c * upx], acc);
      }
      yp[static_cast<long>(oy) * outW + ox] = acc;
    }
  }
}


// ---------------------------------------------------------------------------------------------------------------------
// Fused separable 2x resampler: BOTH 1-D passes of a separable up-by-2 or down-by-2 FIR in one kernel, the intermediate
// in shared memory.  These are the reference's only upfirdn2d call shapes (augment.py:314,325: `upsample2d(x, sym6, up=2)`,
// `downsample2d(x, sym6, down=2)` with the 12-tap sym6 filter, executed there as two 1-D passes, upfirdn2d.py:243-244).
// HBM traffic = read x + write y (the two-pass form also writes and re-reads an intermediate of the larger size).
//
// Per CTA: an output tile TOH x TOW.  (1) the input tile it depends on is staged in shared memory (zero outside the
// image: that IS the padding); (2) horizontal pass -> `mid` [input rows x TOW]; (3) vertical pass -> global.  In (2) and
// (3) a thread produces 4 consecutive outputs from one register window (T/2+2 values for up, T+6 for down), so a
// shared-memory word is read ~1/3 as often as a scalar tap loop would; all register indices are compile-time constants
// (T is a template parameter, the polyphase selection depends only on the parity of the padding: one uniform branch).
//   up  : y[o] = sum_t g[e + 2t] * x[i0 + t],  e = (pad0 - o) & 1, i0 = (o + e - pad0) / 2        (zero-insertion skipped)
//   down: y[o] = sum_k g[k] * x[2o + k - pad0]
// g = filter flipped unless flip_filter (upfirdn2d.py:200-203), times sqrt(gain) per axis.
// ---------------------------------------------------------------------------------------------------------------------
//
// Design (a first version was issue bound on index arithmetic and FMAs):
//   * staging is ONE cp.async.bulk.tensor (TMA, 3-D box [1, TIH, PIN] of the [planes, H, W] tensor, out-of-bounds = zero fill =
//     the padding) per tile instead of ~1 500 4-byte cp.async with their bounds checks (used when W % 4 == 0 and x is
//     16-byte aligned; the cp.async path is kept for everything else);
//   * the vertical pass runs on column PAIRS (float2 arithmetic, one pair per tap);
//   * a horizontal item makes 8 outputs from float4-aligned window reads, so its index arithmetic is amortised twice as far.
template <int T, bool kUp>
struct SepGeom {
  static constexpr int TOW = 64;
  static constexpr int TOH = kUp ? 64 : 32;
  static constexpr int NV = kUp ? T / 2 + 2 : T + 6;                 // register window for 4 outputs
  static constexpr int NV8 = kUp ? T / 2 + 4 : T + 14;               // ... for 8 outputs
  static constexpr int NVR = (NV8 + 3 + 3) & ~3;                      // read as float4, from up to 3 columns before the window
  static constexpr int NV2 = T + 2;                                   // down, 2 outputs (vertical pass)
  static constexpr int TIW = kUp ? TOW / 2 + T / 2 + 1 : 2 * TOW + T - 2;
  static constexpr int TIH = kUp ? TOH / 2 + T / 2 + 1 : 2 * TOH + T - 2;
  // staged row: the tile may start up to 3 columns early, so that the innermost coordinate of every TMA box is a multiple
  // of 4 floats (16 bytes)
  static constexpr int PIN = (TIW + 3 + 3) & ~3;
  static constexpr int PMID = TOW + 4;
  static constexpr int IN_BYTES = TIH * PIN * 4;
  static constexpr int IN_STRIDE = (IN_BYTES + 127) & ~127;           // TMA destinations are 128-byte aligned
  static constexpr int NBUF = kUp ? 3 : 2;                            // input tiles in flight (down: 43 KB each, two CTAs per SM)
  static constexpr int MID_OFF = NBUF * IN_STRIDE;
  static constexpr int GS_OFF = MID_OFF + TIH * PMID * 4;
  static constexpr int BAR_OFF = (GS_OFF + T * 4 + 7) & ~7;
  static constexpr int SMEM = BAR_OFF + NBUF * 8;
  // threads: one item each in the vertical pass (256); the horizontal pass has TIH * 8 items -- with 39 rows (up) a 256-thread CTA
  // left 56 items to a second, mostly empty iteration that every warp then waited for at the barrier
  static constexpr int THREADS = 320;                                 // down: 74 rows x 8 = 592 items = 2 balanced iterations
};

// first input index touched by output o (floor semantics for negative values)
template <bool kUp>
__device__ __forceinline__ int sep_first(int o, int pad0) {
  if (kUp) return (o - pad0 + 1) >> 1;      // ceil((o - pad0) / 2)
  return 2 * o - pad0;
}

// NQ (4, or 2 for down) outputs from a register window v[]; `odd` = parity of (o0 - pad0) (up only)
template <int T, bool kUp, int NQ = 4>
__device__ __forceinline__ void sep_fir4(const float* __restrict__ v, const float* __restrict__ g, bool odd, float (&o)[NQ]) {
#pragma unroll
  for (int q = 0; q < NQ; ++q) o[q] = 0.f;
  if (kUp) {
    // c = o - pad0.  c even: e = 0, start (c/2 - b);  c odd: e = 1, start ((c+1)/2 - b);  b = ceil(c0 / 2)
    if (!odd) {       // c0 even: b = c0/2; q=0: e0 s0 | q=1: e1 s1 | q=2: e0 s1 | q=3: e1 s2
#pragma unroll
      for (int t = 0; t < T / 2; ++t) {
        o[0] = fmaf(g[2 * t], v[t], o[0]);
        o[1] = fmaf(g[2 * t + 1], v[t + 1], o[1]);
        o[2] = fmaf(g[2 * t], v[t + 1], o[2]);
        o[3] = fmaf(g[2 * t + 1], v[t + 2], o[3]);
      }
    } else {          // c0 odd: b = (c0+1)/2; q=0: e1 s0 | q=1: e0 s0 | q=2: e1 s1 | q=3: e0 s1
#pragma unroll
      for (int t = 0; t < T / 2; ++t) {
        o[0] = fmaf(g[2 * t + 1], v[t], o[0]);
        o[1] = fmaf(g[2 * t], v[t], o[1]);
        o[2] = fmaf(g[2 * t + 1], v[t + 1], o[2]);
        o[3] = fmaf(g[2 * t], v[t + 1], o[3]);
      }
    }
  } else {
#pragma unroll
    for (int k = 0; k < T; ++k) {
#pragma unroll
      for (int q = 0; q < NQ; ++q) o[q] = fmaf(g[k], v[2 * q + k], o[q]);
    }
  }
}

// the same on two adjacent columns at once (float2): v[j] = (column c, column c+1) of window row j
template <int T, bool kUp, int NQ>
__device__ __forceinline__ void sep_fir_pair(const float2* __restrict__ v, const float* __restrict__ g, bool odd, float2 (&o)[NQ]) {
#pragma unroll
  for (int q = 0; q < NQ; ++q) o[q] = make_float2(0.f, 0.f);
  if (kUp) {
    if (!odd) {
#pragma unroll
      for (int t = 0; t < T / 2; ++t) {
        const float2 ge = make_float2(g[2 * t], g[2 * t]), go = make_float2(g[2 * t + 1], g[2 * t + 1]);
        o[0] = ffma2(ge, v[t], o[0]);
        o[1] = ffma2(go, v[t + 1], o[1]);
        o[2] = ffma2(ge, v[t + 1], o[2]);
        o[3] = ffma2(go, v[t + 2], o[3]);
      }
    } else {
#pragma unroll
      for (int t = 0; t < T / 2; ++t) {
        const float2 ge = make_float2(g[2 * t], g[2 * t]), go = make_float2(g[2 * t + 1], g[2 * t + 1]);
        o[0] = ffma2(go, v[t], o[0]);
        o[1] = ffma2(ge, v[t], o[1]);
        o[2] = ffma2(go, v[t + 1], o[2]);
        o[3] = ffma2(ge, v[t + 1], o[3]);
      }
    }
  } else {
#pragma unroll
    for (int k = 0; k < T; ++k) {
      const float2 gk = make_float2(g[k], g[k]);
#pragma unroll
      for (int q = 0; q < NQ; ++q) o[q] = ffma2(gk, v[2 * q + k], o[q]);
    }
  }
}

template <int T, bool kUp, int SH>
__device__ __forceinline__ void sep_hpass(const float* __restrict__ in_s, float* __restrict__ mid, const float (&g)[T], bool oddx, int tid) {
  using G = SepGeom<T, kUp>;
  constexpr int NW = (G::NV8 + SH + 3) & ~3;
  constexpr int NITEMS = G::TIH * (G::TOW / 8);
  static_assert((kUp ? 4 : 16) * (G::TOW / 8 - 1) + NW <= G::PIN, "an 8-output window leaves the staged row");
  if constexpr (kUp) {
    for (int i = tid; i < NITEMS; i += G::THREADS) {
      const int a = i & (G::TOW / 8 - 1), r = i / (G::TOW / 8);
      const float* wsrc = in_s + r * G::PIN + 4 * a;
      float w[NW];
#pragma unroll
      for (int j = 0; j < NW / 4; ++j) {
        const float4 t4 = *reinterpret_cast<const float4*>(wsrc + 4 * j);
        w[4 * j] = t4.x; w[4 * j + 1] = t4.y; w[4 * j + 2] = t4.z; w[4 * j + 3] = t4.w;
      }
      float o0[4], o1[4];
      sep_fir4<T, kUp>(w + SH, g, oddx, o0);
      sep_fir4<T, kUp>(w + SH + 2, g, oddx, o1);
      float4* m4 = reinterpret_cast<float4*>(mid + r * G::PMID + 8 * a);
      m4[0] = make_float4(o0[0], o0[1], o0[2], o0[3]);
      m4[1] = make_float4(o1[0], o1[1], o1[2], o1[3]);
    }
  } else {
    // y[q] = sum_k g[k] * w[SH + 2q + k]: with the window read as pairs W2[i] = (w[2i], w[2i+1]) and the taps as pairs
    // G2[j] = (g'[M0 + 2j], g'[M0 + 2j + 1]), g'[m] = g[m - SH] (0 outside), M0 = SH & ~1, it is one ffma2 per tap PAIR and
    // a final x + y, all register pairs naturally aligned.
    constexpr int M0 = SH & ~1, NP = T / 2 + (SH & 1);
    static_assert(2 * (7 + M0 / 2 + NP) <= NW, "pair window");
    float2 G2[NP];
#pragma unroll
    for (int j = 0; j < NP; ++j) {
      const int ka = M0 + 2 * j - SH, kb = ka + 1;
      G2[j] = make_float2(ka >= 0 && ka < T ? g[ka] : 0.f, kb >= 0 && kb < T ? g[kb] : 0.f);
    }
    // item -> (column group a, row r) with r FASTEST: the 8 threads of an LDS.128 phase then read 8 consecutive rows (pitch
    // 148 floats = 20 banks apart: conflict-free); with the column group fastest their windows start 16 floats apart -- two
    // bank groups for 8 threads, a 4-way conflict on every window load
    for (int i = tid; i < NITEMS; i += G::THREADS) {
      const int a = i / G::TIH, r = i - a * G::TIH;
      const float* wsrc = in_s + r * G::PIN + 16 * a;
      float2 W2[NW / 2];
#pragma unroll
      for (int j = 0; j < NW / 4; ++j) {
        const float4 t4 = *reinterpret_cast<const float4*>(wsrc + 4 * j);
        W2[2 * j] = make_float2(t4.x, t4.y);
        W2[2 * j + 1] = make_float2(t4.z, t4.w);
      }
      float o[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        float2 acc = fmul2(G2[0], W2[q + M0 / 2]);
#pragma unroll
        for (int j = 1; j < NP; ++j) acc = ffma2(G2[j], W2[q + M0 / 2 + j], acc);
        o[q] = acc.x + acc.y;
      }
      float4* m4 = reinterpret_cast<float4*>(mid + r * G::PMID + 8 * a);
      m4[0] = make_float4(o[0], o[1], o[2], o[3]);
      m4[1] = make_float4(o[4], o[5], o[6], o[7]);
    }
  }
}

template <int T, bool kUp, bool kTma>
__global__ void __launch_bounds__(SepGeom<T, kUp>::THREADS, kUp ? 1 : 2) upfirdn2d_sep_kernel(const float* __restrict__ x, const __grid_constant__ CUtensorMap tmap,
                                                            const float* __restrict__ f, float* __restrict__ y, int inH, int inW,
                                                            int outH, int outW, int padx0, int pady0, int flip, float gain_axis,
                                                            int tiles_x, int tiles_y, long nplanes) {
  using G = SepGeom<T, kUp>;
  // no static shared memory in this kernel: the dynamic window starts at offset 0 and honours the declared alignment (pointer
  // arithmetic through integers would turn every access into a generic LD / ST)
  extern __shared__ __align__(1024) uint8_t sep_raw[];
  uint8_t* const sbase = sep_raw;
  float* mid = reinterpret_cast<float*>(sbase + G::MID_OFF);            // [TIH][PMID]
  float* gs = reinterpret_cast<float*>(sbase + G::GS_OFF);              // [T]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sbase + G::BAR_OFF);     // [NBUF]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int NWARPS = G::THREADS / 32;
  if (tid < T) gs[tid] = (flip ? f[tid] : f[T - 1 - tid]) * gain_axis;
  if (kTma && tid == 0) {
    for (int i = 0; i < G::NBUF; ++i) mbar_init(bars + i, 1);
    fence_mbar_init();
  }
  const long ntiles = static_cast<long>(nplanes) * tiles_x * tiles_y;
  // columns staged in front of the tile so that the box starts on a 16-byte boundary; the same for every tile (a tile step is
  // 32 / 128 input columns)
  const int sh = kTma ? (sep_first<kUp>(0, padx0) & 3) : 0;
  // ---- (1) stage an input tile (zero outside the image = the padding).  The NEXT tile is prefetched while this one is
  //      filtered and stored.
  auto prefetch = [&](int tx, int ty, long plane, int buf) {
    const int ix0 = sep_first<kUp>(tx * G::TOW, padx0) - sh, iy0 = sep_first<kUp>(ty * G::TOH, pady0);
    float* dst = reinterpret_cast<float*>(sbase + buf * G::IN_STRIDE);
    if (kTma) {
      if (tid == 0) {
        mbar_arrive_expect_tx(bars + buf, G::IN_BYTES);
        const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(dst));
        const uint32_t mb = static_cast<uint32_t>(__cvta_generic_to_shared(bars + buf));
        asm volatile(
            "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
            ::"r"(d), "l"(reinterpret_cast<uint64_t>(&tmap)), "r"(ix0), "r"(iy0), "r"(static_cast<int>(plane)), "r"(mb)
            : "memory");
      }
    } else {      // 4-byte cp.async: a warp walks rows, lanes walk columns (coalesced)
      const float* xp = x + plane * inH * inW;
      for (int r = warp; r < G::TIH; r += NWARPS) {
        const int gy = iy0 + r;
        const bool rowok = gy >= 0 && gy < inH;
        const float* src = xp + static_cast<long>(rowok ? gy : 0) * inW;
#pragma unroll
        for (int c0 = 0; c0 < G::PIN; c0 += 32) {
          const int c = c0 + lane;
          if (c < G::PIN) {
            const int gx = ix0 + c;
            const bool ok = rowok && c < G::TIW && gx >= 0 && gx < inW;
            const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(dst + r * G::PIN + c));
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(d), "l"(src + (ok ? gx : 0)), "r"(ok ? 4 : 0) : "memory");
          }
        }
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
    }
  };
  __syncthreads();                                   // filter taps + barriers initialised
  // tile -> (plane, ty, tx) is carried incrementally: the 64-bit divisions of the first version cost more instructions per
  // tile than the two filter passes
  const int per_plane = tiles_x * tiles_y;
  const int step_p = static_cast<int>(gridDim.x) / per_plane, step_r = static_cast<int>(gridDim.x) % per_plane;
  const int step_y = step_r / tiles_x, step_x = step_r % tiles_x;
  struct TileAt { int tx, ty; long plane; };
  TileAt at{static_cast<int>(blockIdx.x) % tiles_x, (static_cast<int>(blockIdx.x) % per_plane) / tiles_x,
            static_cast<long>(blockIdx.x) / per_plane};
  TileAt pf = at;                                     // the next tile to prefetch (runs NBUF - 1 tiles ahead)
  auto advance = [&](TileAt& t) {
    t.tx += step_x;
    if (t.tx >= tiles_x) { t.tx -= tiles_x; ++t.ty; }
    t.ty += step_y;
    if (t.ty >= tiles_y) { t.ty -= tiles_y; ++t.plane; }
    t.plane += step_p;
  };
  long pf_tile = blockIdx.x;
  auto prefetch_next = [&](int buf) {                 // every thread calls it: the cp.async path counts commit groups
    if (pf_tile < ntiles) prefetch(pf.tx, pf.ty, pf.plane, buf);
    else if (!kTma) asm volatile("cp.async.commit_group;" ::: "memory");
    pf_tile += gridDim.x;
    advance(pf);
  };
#pragma unroll
  for (int i = 0; i < G::NBUF - 1; ++i) prefetch_next(i);
  float g[T];
#pragma unroll
  for (int k = 0; k < T; ++k) g[k] = gs[k];
  uint32_t it = 0;
  for (long tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
    const int tx = at.tx, ty = at.ty;
    const long plane = at.plane;
    advance(at);
    const int cur = static_cast<int>(it % G::NBUF);
    const int ox0 = tx * G::TOW, oy0 = ty * G::TOH;
    const float* in_s = reinterpret_cast<const float*>(sbase + cur * G::IN_STRIDE);
    if (kTma) mbar_wait(bars + cur, (it / G::NBUF) & 1);
    else asm volatile("cp.async.wait_group %0;" ::"n"(G::NBUF - 2) : "memory");
    __syncthreads();                                  // this tile's input has landed; everybody is done with the previous buffer
    prefetch_next(static_cast<int>((it + G::NBUF - 1) % G::NBUF));
    const bool oddx = ((ox0 - padx0) & 1) != 0, oddy = ((oy0 - pady0) & 1) != 0;
    // ---- (2) horizontal: item = (input row, group of 8 output columns).  Its window starts `sh` columns after column 4a
    //      (up) / 16a (down) of the staged row: aligned float4 reads, the shift is a compile-time register offset.
    switch (sh) {
      case 0: sep_hpass<T, kUp, 0>(in_s, mid, g, oddx, tid); break;
      case 1: sep_hpass<T, kUp, 1>(in_s, mid, g, oddx, tid); break;
      case 2: sep_hpass<T, kUp, 2>(in_s, mid, g, oddx, tid); break;
      default: sep_hpass<T, kUp, 3>(in_s, mid, g, oddx, tid); break;
    }
    __syncthreads();
    // ---- (3) vertical: item = (group of 4 output columns, group of NQ output rows) on two column pairs (float2): float4
    //      columns of `mid`, float4 stores (rows of the output are 16-byte aligned when outW % 4 == 0)
    constexpr int NQ = kUp ? 4 : 2;                   // 16 x 16 items (up, 64 rows) / 16 x 16 items (down, 32 rows)
    constexpr int NW = kUp ? G::NV : G::NV2;
    float* yp = y + plane * outH * outW;
    const bool vec_ok = (outW & 3) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0;
    const bool vec2_ok = (outW & 1) == 0 && (reinterpret_cast<uintptr_t>(y) & 7) == 0;
    for (int i = tid; i < (G::TOW / 4) * (G::TOH / NQ); i += G::THREADS) {
      const int c4 = i & (G::TOW / 4 - 1), a = i / (G::TOW / 4);
      const float* wsrc = mid + (kUp ? 2 * a : 2 * NQ * a) * G::PMID + 4 * c4;
      float2 lo[NW], hi[NW];
#pragma unroll
      for (int j = 0; j < NW; ++j) {
        const float4 t4 = *reinterpret_cast<const float4*>(wsrc + j * G::PMID);
        lo[j] = make_float2(t4.x, t4.y);
        hi[j] = make_float2(t4.z, t4.w);
      }
      float2 ol[NQ], oh[NQ];
      sep_fir_pair<T, kUp, NQ>(lo, g, oddy, ol);
      sep_fir_pair<T, kUp, NQ>(hi, g, oddy, oh);
      const int ox = ox0 + 4 * c4;
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const int oy = oy0 + NQ * a + q;
        if (oy >= outH) continue;
        float* dst = yp + static_cast<long>(oy) * outW + ox;
        if (vec_ok && ox + 3 < outW) {
          __stcs(reinterpret_cast<float4*>(dst), make_float4(ol[q].x, ol[q].y, oh[q].x, oh[q].y));
        } else if (vec2_ok && ox + 3 < outW) {      // even row length (1024 -> 506): rows are 8-byte aligned
          __stcs(reinterpret_cast<float2*>(dst), ol[q]);
          __stcs(reinterpret_cast<float2*>(dst) + 1, oh[q]);
        } else {
          if (ox < outW) __stcs(dst, ol[q].x);
          if (ox + 1 < outW) __stcs(dst + 1, ol[q].y);
          if (ox + 2 < outW) __stcs(dst + 2, oh[q].x);
          if (ox + 3 < outW) __stcs(dst + 3, oh[q].y);
        }
      }
    }
  }   // tile loop
}

// cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time dependency on libcuda)
static PFN_cuTensorMapEncodeTiled_v12000 tensor_map_encoder() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }
  return fn;
}

template <int T, bool kUp>
static int launch_sep_dir(const float* x, const float* f, float* y, long planes, int inH, int inW, int outH, int outW, int padx0,
                          int pady0, int flip, float ga, cudaStream_t st) {
  using G = SepGeom<T, kUp>;
  const int txn = (outW + G::TOW - 1) / G::TOW, tyn = (outH + G::TOH - 1) / G::TOH;
  const long nt = planes * txn * tyn, cap = static_cast<long>(num_sms()) * (kUp ? 6 : 2);
  const unsigned grid = static_cast<unsigned>(nt < cap ? nt : cap);
  CUtensorMap tmap;
  memset(&tmap, 0, sizeof(tmap));
  bool tma = (inW & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && planes < (1L << 31) && tensor_map_encoder() != nullptr;
  if (tma) {
    const cuuint64_t dims[3] = {static_cast<cuuint64_t>(inW), static_cast<cuuint64_t>(inH), static_cast<cuuint64_t>(planes)};
    const cuuint64_t strides[2] = {static_cast<cuuint64_t>(inW) * 4, static_cast<cuuint64_t>(inW) * inH * 4};
    const cuuint32_t box[3] = {static_cast<cuuint32_t>(G::PIN), static_cast<cuuint32_t>(G::TIH), 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    tma = tensor_map_encoder()(&tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(x), dims, strides, box, estr,
                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
  }
  if (tma) {
    cudaFuncSetAttribute(upfirdn2d_sep_kernel<T, kUp, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, G::SMEM);
    upfirdn2d_sep_kernel<T, kUp, true><<<grid, G::THREADS, G::SMEM, st>>>(x, tmap, f, y, inH, inW, outH, outW, padx0, pady0, flip, ga, txn,
                                                                    tyn, planes);
  } else {
    cudaFuncSetAttribute(upfirdn2d_sep_kernel<T, kUp, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, G::SMEM);
    upfirdn2d_sep_kernel<T, kUp, false><<<grid, G::THREADS, G::SMEM, st>>>(x, tmap, f, y, inH, inW, outH, outW, padx0, pady0, flip, ga, txn,
                                                                     tyn, planes);
  }
  return check_launch("hg_upfirdn2d_sep2");
}

template <int T>
static int launch_sep(bool up, const float* x, const float* f, float* y, long planes, int inH, int inW, int outH, int outW,
                      int padx0, int pady0, int flip, float gain, cudaStream_t st) {
  const float ga = sqrtf(gain);
  if (up) return launch_sep_dir<T, true>(x, f, y, planes, inH, inW, outH, outW, padx0, pady0, flip, ga, st);
  return launch_sep_dir<T, false>(x, f, y, planes, inH, inW, outH, outW, padx0, pady0, flip, ga, st);
}

// 2x2 average pooling / nearest-neighbour 2x up-sampling with a scale factor (each is the other's adjoint up to the
// scale: d avgpool = 0.25 * up(dy), d up = 4 * avgpool(dy)).  The discriminator's ResBlocks use them between
// convolutions (unet_discriminators.py:30,60-70); pure streaming, one float2 / float4 per lane.
__global__ void __launch_bounds__(256) pool2x_kernel(const float* __restrict__ x, float* __restrict__ y, long planes,
                                                     int oH, int oW, float scale) {
  const int ow2 = oW >> 1;                              // output float2 per row (oW even)
  const long total = planes * oH * ow2;
  for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int cx = static_cast<int>(i % ow2);
    const long r = i / ow2;                             // plane * oH + oy
    const long plane = r / oH;
    const int oy = static_cast<int>(r - plane * oH);
    const float* src = x + (plane * (2 * oH) + 2 * oy) * (2L * oW) + 4 * cx;
    const float4 a = __ldcs(reinterpret_cast<const float4*>(src));
    const float4 b = __ldcs(reinterpret_cast<const float4*>(src + 2 * oW));
    __stcs(reinterpret_cast<float2*>(y + r * oW) + cx, make_float2(((a.x + a.y) + (b.x + b.y)) * scale, ((a.z + a.w) + (b.z + b.w)) * scale));
  }
}

__global__ void __launch_bounds__(256) up2x_kernel(const float* __restrict__ x, float* __restrict__ y, long planes, int iH,
                                                   int iW, float scale) {
  const int iw2 = iW >> 1;
  const long total = planes * iH * iw2;
  for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int cx = static_cast<int>(i % iw2);
    const long r = i / iw2;                             // plane * iH + iy
    const long plane = r / iH;
    const int iy = static_cast<int>(r - plane * iH);
    const float2 v = __ldcs(reinterpret_cast<const float2*>(x + r * iW) + cx);
    const float4 o = make_float4(v.x * scale, v.x * scale, v.y * scale, v.y * scale);
    float* dst = y + (plane * (2 * iH) + 2 * iy) * (2L * iW) + 4 * cx;
    __stcs(reinterpret_cast<float4*>(dst), o);
    __stcs(reinterpret_cast<float4*>(dst + 2 * iW), o);
  }
}

}  // namespace hg

extern "C" {

int hg_bias_act(const float* x, const float* b, float* y, long n, int stepB, int sizeB, int act, float alpha,
                float gain, float clamp, void* stream) {
  HG_REQUIRE(x && y, "hg_bias_act: null pointer");
  HG_REQUIRE(act >= 1 && act <= 9, "hg_bias_act: unknown activation id %d", act);
  HG_REQUIRE(!b || (stepB > 0 && sizeB > 0), "hg_bias_act: bad bias geometry");
  HG_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0,
             "hg_bias_act: x / y must be 16-byte aligned");
  if (n <= 0) return 0;
  const long nvec = (n + 3) / 4;
  long blocks = (nvec + 511) / 512;                    // two float4 per thread and pass
  const long cap = static_cast<long>(hg::num_sms()) * 32;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  auto st = static_cast<cudaStream_t>(stream);
  const bool vec_bias = b && (stepB % 4 == 0);
  const unsigned grid = static_cast<unsigned>(blocks);
  if (n < (1L << 32)) {
    const uint32_t sB = b ? static_cast<uint32_t>(stepB) : 1u, zB = b ? static_cast<uint32_t>(sizeB) : 1u;
    if (vec_bias) hg::bias_act_kernel<uint32_t, true><<<grid, 256, 0, st>>>(x, b, y, n, sB, zB, act, alpha, gain, clamp);
    else hg::bias_act_kernel<uint32_t, false><<<grid, 256, 0, st>>>(x, b, y, n, sB, zB, act, alpha, gain, clamp);
  } else {
    const unsigned long long sB = b ? stepB : 1, zB = b ? sizeB : 1;
    if (vec_bias) hg::bias_act_kernel<unsigned long long, true><<<grid, 256, 0, st>>>(x, b, y, n, sB, zB, act, alpha, gain, clamp);
    else hg::bias_act_kernel<unsigned long long, false><<<grid, 256, 0, st>>>(x, b, y, n, sB, zB, act, alpha, gain, clamp);
  }
  return hg::check_launch("hg_bias_act");
}

int hg_bias_act_grad(const float* g, const float* b, const float* xref, const float* yref, const float* dy, float* out,
                     long n, int stepB, int sizeB, int order, int act, float alpha, float gain, float clamp,
                     void* stream) {
  HG_REQUIRE(g && out, "hg_bias_act_grad: null pointer");
  HG_REQUIRE(act >= 1 && act <= 9, "hg_bias_act_grad: unknown activation id %d", act);
  HG_REQUIRE(order == 1 || order == 2, "hg_bias_act_grad: derivative order must be 1 or 2 (got %d)", order);
  HG_REQUIRE(!b || (stepB > 0 && sizeB > 0), "hg_bias_act_grad: bad bias geometry");
  HG_REQUIRE(act == 1 || (act == 9 ? xref != nullptr : yref != nullptr),
             "hg_bias_act_grad: activation %d needs its saved %s", act, act == 9 ? "input (xref)" : "output (yref)");
  HG_REQUIRE(clamp < 0.f || act == 9 || yref, "hg_bias_act_grad: clamp needs the saved output (yref)");
  for (const float* ptr : {g, xref, yref, dy, static_cast<const float*>(out)})
    HG_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "hg_bias_act_grad: tensors must be 16-byte aligned");
  if (n <= 0) return 0;
  long blocks = ((n + 3) / 4 + 255) / 256;
  const long cap = static_cast<long>(hg::num_sms()) * 32;
  if (blocks > cap) blocks = cap;
  auto st = static_cast<cudaStream_t>(stream);
  if (n < (1L << 32))
    hg::bias_act_grad_kernel<uint32_t><<<static_cast<unsigned>(blocks), 256, 0, st>>>(
        g, b, xref, yref, dy, out, n, b ? static_cast<uint32_t>(stepB) : 1u, b ? static_cast<uint32_t>(sizeB) : 1u, order,
        act, alpha, gain, clamp);
  else
    hg::bias_act_grad_kernel<unsigned long long><<<static_cast<unsigned>(blocks), 256, 0, st>>>(
        g, b, xref, yref, dy, out, n, b ? stepB : 1, b ? sizeB : 1, order, act, alpha, gain, clamp);
  return hg::check_launch("hg_bias_act_grad");
}

int hg_upfirdn2d(const float* x, const float* f, float* y, int NC, int inH, int inW, int outH, int outW, int fH, int fW,
                 int upx, int upy, int downx, int downy, int padx0, int pady0, int flip_filter, float gain,
                 void* stream) {
  HG_REQUIRE(x && f && y, "hg_upfirdn2d: null pointer");
  HG_REQUIRE(upx >= 1 && upy >= 1 && downx >= 1 && downy >= 1, "hg_upfirdn2d: up/down factors must be >= 1");
  HG_REQUIRE(fH >= 1 && fW >= 1 && fH * fW <= 4096, "hg_upfirdn2d: filter too large");
  if (NC <= 0 || outH <= 0 || outW <= 0) return 0;
  const int gx = (outW + 127) / 128;
  int gy = (outH + 15) / 16;                       // >= 16 rows per block amortise the per-block filter setup
  const int want = hg::num_sms() * 16;             // enough blocks to fill the machine
  int gz = NC < 65535 ? NC : 65535;
  while (gy > 1 && static_cast<long>(gx) * gy * gz > 4L * want && gz > 1) gz = (gz + 1) / 2;
  dim3 grid(gx, gy, gz);
  hg::upfirdn2d_kernel<<<grid, 128, fH * fW * sizeof(float), static_cast<cudaStream_t>(stream)>>>(
      x, f, y, NC, inH, inW, outH, outW, fH, fW, upx, upy, downx, downy, padx0, pady0, flip_filter, gain);
  return hg::check_launch("hg_upfirdn2d");
}

int hg_upfirdn2d_sep2(const float* x, const float* f, float* y, long planes, int inH, int inW, int outH, int outW, int taps,
                      int up, int padx0, int pady0, int flip_filter, float gain, void* stream) {
  HG_REQUIRE(x && f && y, "hg_upfirdn2d_sep2: null pointer");
  HG_REQUIRE(planes > 0 && inH > 0 && inW > 0 && outH > 0 && outW > 0, "hg_upfirdn2d_sep2: bad shape");
  HG_REQUIRE(gain >= 0.f, "hg_upfirdn2d_sep2: gain must be non-negative");
  HG_REQUIRE(planes * ((outW + 63) / 64) * ((outH + 31) / 32) < (1L << 31), "hg_upfirdn2d_sep2: too many tiles");
  auto st = static_cast<cudaStream_t>(stream);
  switch (taps) {
    case 4: return hg::launch_sep<4>(up != 0, x, f, y, planes, inH, inW, outH, outW, padx0, pady0, flip_filter, gain, st);
    case 6: return hg::launch_sep<6>(up != 0, x, f, y, planes, inH, inW, outH, outW, padx0, pady0, flip_filter, gain, st);
    case 8: return hg::launch_sep<8>(up != 0, x, f, y, planes, inH, inW, outH, outW, padx0, pady0, flip_filter, gain, st);
    case 12: return hg::launch_sep<12>(up != 0, x, f, y, planes, inH, inW, outH, outW, padx0, pady0, flip_filter, gain, st);
    case 16: return hg::launch_sep<16>(up != 0, x, f, y, planes, inH, inW, outH, outW, padx0, pady0, flip_filter, gain, st);
    default: break;
  }
  hg::set_error("hg_upfirdn2d_sep2: taps must be one of 4, 6, 8, 12, 16 (got %d)", taps);
  return 1;
}

int hg_resample2x(const float* x, float* y, long planes, int inH, int inW, int up, float scale, void* stream) {
  HG_REQUIRE(x && y && planes > 0 && inH > 0 && inW > 0, "hg_resample2x: bad arguments");
  HG_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0, "hg_resample2x: tensors must be 16-byte aligned");
  auto st = static_cast<cudaStream_t>(stream);
  long total;
  if (up) {
    HG_REQUIRE(inW % 2 == 0, "hg_resample2x: up-sampling needs an even input width (got %d)", inW);
    total = planes * inH * (inW / 2);
  } else {
    HG_REQUIRE(inH % 2 == 0 && inW % 4 == 0, "hg_resample2x: pooling needs even height and a width that is a multiple of 4 (got %dx%d)", inH, inW);
    total = planes * (inH / 2) * (inW / 4);
  }
  long blocks = (total + 255) / 256;
  const long cap = static_cast<long>(hg::num_sms()) * 32;
  if (blocks > cap) blocks = cap;
  if (up) hg::up2x_kernel<<<static_cast<unsigned>(blocks), 256, 0, st>>>(x, y, planes, inH, inW, scale);
  else hg::pool2x_kernel<<<static_cast<unsigned>(blocks), 256, 0, st>>>(x, y, planes, inH / 2, inW / 2, scale);
  return hg::check_launch("hg_resample2x");
}

}  // extern "C"
