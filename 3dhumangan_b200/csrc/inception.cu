// FID Inception-v3 (pytorch-fid's fid_inception_v3, torchvision's Inception3 layout) and the feature statistics of FID.
//
//   hg_conv2d_general   every one of the network's 94 convolutions: an implicit GEMM on wgmma for any kh x kw <= 7 x 7 filter,
//                       stride 1 or 2, zero padding (ph, pw), any Cin and Cout <= 448, with bias + ReLU in the epilogue
//                       (BatchNorm is folded into the weights and the bias on the host).  The output lands in the channel
//                       window [c0, c0 + Cout) of a [B, Ctot, Ho, Wo] buffer, so an Inception block's concatenation is free.
//   hg_pool3x3          3x3 max (stride 2 pad 0, or stride 1 pad 1) and average (stride 1 pad 1, count_include_pad=False)
//                       pooling, also into a channel window.
//   hg_global_avgpool   the mean of every plane (8x8 -> [B, 2048]), a fixed-order warp reduction.
//   hg_feature_moments  sum += sum_i x_i and gram += sum_i x_i x_i^T in fp64 over features [n, D], in a fixed order without
//                       atomics (repeats are bit-identical); tiles above the diagonal only, each mirrored.
//
// GEMM view of the convolution: M = 128 consecutive output pixels of the flattened [B, Ho, Wo] grid (a tile may span images,
// so the 8x8 and 17x17 layers waste no rows), N = one block of <= 128 output channels, K = kh * kw * Cin in chunks of 64 in
// the order of the packed weight [Cout, kh, kw, Cin].  A thread builds 32 consecutive K entries of one row: it locates its
// first (tap, channel) once and then walks channels, moving to the next tap when one is exhausted, so Cin = 3 (K = 27, one
// chunk) and Cin = 48 / 80 need no per-tap padding.  Warpgroups 0-1 build the operand tiles in a 4-slot ring and issue the
// wgmmas (bf16x3 when passes == 3), warp 8 streams the packed weight tiles with bulk copies.
#include "common.cuh"
#include "wgmma.cuh"

namespace hg {

constexpr int kGcThreads = 384;
constexpr int kGcStages = 2;
constexpr uint32_t kGcA = 128 * 128;
constexpr uint32_t kGcB = 128 * 128;
constexpr int kGcMaxCout = 448;
constexpr uint32_t kGcSmem = 8 * kGcA + kGcStages * kGcB + 512 * 4 + 16 * 8 + 1024;

struct GConvArgs {
  const float* x;
  int B, Cin, H, W;
  int kh, kw, stride, ph, pw, Ho, Wo;
  const uint8_t* wimg;
  int Cout, Nb, nblocks, kchunks;
  const float* bias;
  float* out;
  int Ctot, c0;
};

template <int kPasses, int N>
__global__ void __launch_bounds__(kGcThreads, 1) conv_general_kernel(GConvArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_hi = smem;
  uint8_t* a_lo = smem + 4 * kGcA;
  uint8_t* b_st = smem + 8 * kGcA;
  float* tab_bias = reinterpret_cast<float*>(b_st + kGcStages * kGcB);   // [512]
  uint64_t* bars = reinterpret_cast<uint64_t*>(tab_bias + 512);
  uint64_t* b_full = bars;                  // [kGcStages]
  uint64_t* b_empty = bars + kGcStages;     // [kGcStages]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < 512; i += blockDim.x) tab_bias[i] = (a.bias && i < a.Cout) ? a.bias[i] : 0.f;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kGcStages; ++i) { mbar_init(b_full + i, 1); mbar_init(b_empty + i, 2); }
    fence_mbar_init();
  }
  __syncthreads();

  const int HWo = a.Ho * a.Wo;
  const long HW = static_cast<long>(a.H) * a.W;
  const long M = static_cast<long>(a.B) * HWo;
  const int tiles = static_cast<int>((M + 127) / 128);
  const int num_items = tiles * a.nblocks;
  const int my_items = (num_items - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);
  const int nchunks = a.kchunks;
  const uint32_t stage_bytes = static_cast<uint32_t>(a.Nb) * 128;

  if (warp < 8) {
    // ------------------------------------------------------------------ operand producer + wgmma + epilogue
    regs_inc<kMmaRegs>();
    // warp (g, q, h): rows q*32.. (q = 2g or 2g+1, inside warpgroup g's 64) and K entries h*32.. of every chunk
    const int g = warp >> 2, q = 2 * g + (warp & 1), h = (warp >> 1) & 1, t = threadIdx.x & 127;
    const int row = q * 32 + lane;
    const uint32_t a_off = g * 64 * 128;
    uint32_t cnt = 0;   // running chunk counter (ring position)
    uint32_t st = 0, ph = 0;
    float d[N / 2];
    for (int it = 0; it < my_items; ++it) {
      const int item = blockIdx.x + it * gridDim.x;
      const int tile = item / a.nblocks, nb = item % a.nblocks;
      const long m = static_cast<long>(tile) * 128 + row;
      const bool valid = m < M;
      const int b = valid ? static_cast<int>(m / HWo) : 0;
      const int pix = valid ? static_cast<int>(m - static_cast<long>(b) * HWo) : 0;
      const int iy0 = (pix / a.Wo) * a.stride - a.ph, ix0 = (pix % a.Wo) * a.stride - a.pw;
      const float* xb = a.x + static_cast<long>(b) * a.Cin * HW;

      // K entries ck*64 + h*32 .. +31 of this row; zero outside the image and past K (ky == kh)
      auto issue = [&](float (&dst)[32], int ck) {
        const int k0 = ck * 64 + h * 32;
        const int tap = k0 / a.Cin;
        int ci = k0 - tap * a.Cin, ky = tap / a.kw, kx = tap - ky * a.kw;
        bool ok;
        const float* p;
        auto locate = [&]() {
          const int sy = iy0 + ky, sx = ix0 + kx;
          ok = valid && ky < a.kh && sy >= 0 && sy < a.H && sx >= 0 && sx < a.W;
          p = ok ? xb + static_cast<long>(ci) * HW + static_cast<long>(sy) * a.W + sx : xb;
        };
        locate();
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          float v;
          asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(v) : "l"(p));
          dst[j] = ok ? v : 0.f;
          if (++ci == a.Cin) {            // warp-uniform: every lane walks the same (tap, channel) sequence
            ci = 0;
            if (++kx == a.kw) { kx = 0; ++ky; }
            locate();
          } else if (ok) {
            p += HW;
          }
        }
      };
      // one weight stage: wait, issue, and release the stage consumed one step earlier once its wgmmas are done
      uint32_t prev = ~0u;
      auto stage = [&](uint32_t a_tile, uint32_t a_tile2, bool two, bool accumulate) {
        mbar_wait(b_full + st, ph);
        acc_fence(d);
        wgmma_fence();
        const uint32_t bt = smem_u32(b_st + st * kGcB);
        wg_k64<N>(d, a_tile, bt, accumulate);
        if (two) wg_k64<N>(d, a_tile2, bt, true);
        wgmma_commit();
        wgmma_wait<1>();
        acc_fence(d);
        if (prev != ~0u && t == 0) mbar_arrive(b_empty + prev);
        prev = st;
        if (++st == kGcStages) { st = 0; ph ^= 1; }
      };
      // a ring slot is rewritten four chunks later: by then every warp of the group has seen its wgmmas complete
      auto convert = [&](float (&cur)[32], int ck) {
        const uint32_t slot = cnt & 3;
#pragma unroll
        for (int gi = 0; gi < 4; ++gi) {
          float y[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) y[j] = cur[gi * 8 + j];
          store_a8<kPasses == 3>(a_hi + slot * kGcA, a_lo + slot * kGcA, row, h * 32 + gi * 8, y);
        }
        fence_proxy_async_smem();
        named_barrier(1 + g, 128);
        const uint32_t ahi = smem_u32(a_hi + slot * kGcA) + a_off, alo = smem_u32(a_lo + slot * kGcA) + a_off;
        stage(ahi, alo, kPasses == 3, ck > 0);
        if (kPasses == 3) stage(ahi, ahi, false, true);
        ++cnt;
      };
      float xa[32], xb2[32];
      issue(xa, 0);
      for (int ck = 0; ck < nchunks; ck += 2) {
        if (ck + 1 < nchunks) issue(xb2, ck + 1);
        convert(xa, ck);
        if (ck + 1 < nchunks) {
          if (ck + 2 < nchunks) issue(xa, ck + 2);
          convert(xb2, ck + 1);
        }
      }

      // ---- epilogue straight from the fragments: bias + ReLU into channel c0 + nb*Nb + frag_col of the window
      wgmma_wait<0>();
      acc_fence(d);
      if (t == 0) mbar_arrive(b_empty + prev);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const long em = static_cast<long>(tile) * 128 + g * 64 + frag_row(t, i);
        if (em >= M) continue;
        const int eb = static_cast<int>(em / HWo), epix = static_cast<int>(em - static_cast<long>(eb) * HWo);
        float* ob = a.out + (static_cast<long>(eb) * a.Ctot + a.c0) * HWo + epix;
#pragma unroll
        for (int j = 0; j < N / 8; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = frag_col(t, j, e), ch = nb * a.Nb + c;
            if (c >= a.Nb || ch >= a.Cout) continue;
            ob[static_cast<long>(ch) * HWo] = fmaxf(d[4 * j + 2 * i + e] + tab_bias[ch], 0.f);
          }
      }
    }
  } else {
    // ------------------------------------------------------------------ weight producer
    regs_dec<kProducerRegs>();
    if (warp == 8 && lane == 0) {
      uint32_t st = 0, ph = 0;
      for (int it = 0; it < my_items; ++it) {
        const int nb = (blockIdx.x + it * gridDim.x) % a.nblocks;
        for (int ck = 0; ck < nchunks; ++ck)
          for (int part = 0; part < (kPasses == 3 ? 2 : 1); ++part) {
            mbar_wait_backoff(b_empty + st, ph ^ 1);
            mbar_arrive_expect_tx(b_full + st, stage_bytes);
            bulk_g2s(b_st + st * kGcB, a.wimg + (static_cast<size_t>(nb * nchunks + ck) * 2 + part) * stage_bytes, stage_bytes,
                     b_full + st);
            if (++st == kGcStages) { st = 0; ph ^= 1; }
          }
      }
    }
  }
}

template <int kPasses, int N>
static int launch_conv_general(int grid, cudaStream_t st, const GConvArgs& a) {
  const cudaError_t e = cudaFuncSetAttribute(conv_general_kernel<kPasses, N>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGcSmem);
  if (e != cudaSuccess) { set_error("hg_conv2d_general: smem opt-in failed: %s", cudaGetErrorString(e)); return 2; }
  conv_general_kernel<kPasses, N><<<grid, kGcThreads, kGcSmem, st>>>(a);
  return check_launch("hg_conv2d_general");
}

// torch's max_pool2d rule (the first maximum, NaN propagates; padding never wins) and avg_pool2d with count_include_pad=False
__global__ void __launch_bounds__(256) pool3x3_kernel(const float* __restrict__ x, int C, int H, int W, int stride, int pad,
                                                      int avg, float* __restrict__ out, int Ctot, int c0, int Ho, int Wo,
                                                      long total) {
  for (long e = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total; e += static_cast<long>(gridDim.x) * blockDim.x) {
    const int ox = static_cast<int>(e % Wo);
    const int oy = static_cast<int>((e / Wo) % Ho);
    const int c = static_cast<int>((e / (static_cast<long>(Wo) * Ho)) % C);
    const long b = e / (static_cast<long>(C) * Ho * Wo);
    const float* plane = x + (b * C + c) * static_cast<long>(H) * W;
    const int y0 = oy * stride - pad, x0 = ox * stride - pad;
    float m = -INFINITY, s = 0.f;
    int n = 0;
    for (int dy = 0; dy < 3; ++dy) {
      const int yy = y0 + dy;
      if (yy < 0 || yy >= H) continue;
      for (int dx = 0; dx < 3; ++dx) {
        const int xx = x0 + dx;
        if (xx < 0 || xx >= W) continue;
        const float v = __ldg(plane + static_cast<long>(yy) * W + xx);
        if (v > m || isnan(v)) m = v;
        s += v;
        ++n;
      }
    }
    out[((b * Ctot + c0 + c) * Ho + oy) * static_cast<long>(Wo) + ox] = avg ? s / static_cast<float>(n) : m;
  }
}

// one warp per plane: lane-strided sums, then a fixed butterfly
__global__ void __launch_bounds__(256) global_avgpool_kernel(const float* __restrict__ x, long planes, int HW, float* __restrict__ out) {
  const long warps = static_cast<long>(gridDim.x) * (blockDim.x >> 5);
  for (long pl = static_cast<long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); pl < planes; pl += warps) {
    const float* p = x + pl * HW;
    float s = 0.f;
    for (int i = threadIdx.x & 31; i < HW; i += 32) s += __ldg(p + i);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) out[pl] = s / static_cast<float>(HW);
  }
}

__global__ void __launch_bounds__(256) feature_sum_kernel(const float* __restrict__ f, int n, int D, double* __restrict__ sum) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= D) return;
  double s = 0.0;
  for (int i = 0; i < n; ++i) s += static_cast<double>(__ldg(f + static_cast<long>(i) * D + j));
  sum[j] += s;
}

// 64 x 64 tile (bi, bj), bi <= bj, of the Gram matrix: thread (ty, tx) owns rows 4ty.. and columns 4tx.., each entry a sum over
// i = 0..n-1 in order; the tile and, above the diagonal, its transpose are added to gram.
constexpr int kMomTile = 64, kMomRows = 32;
__global__ void __launch_bounds__(256) feature_gram_kernel(const float* __restrict__ f, int n, int D, double* __restrict__ gram) {
  const int bi = blockIdx.y, bj = blockIdx.x;
  if (bi > bj) return;
  __shared__ double sa[kMomRows][kMomTile], sb[kMomRows][kMomTile];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  double acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 0.0;
  for (int i0 = 0; i0 < n; i0 += kMomRows) {
    for (int e = threadIdx.x; e < kMomRows * kMomTile; e += blockDim.x) {
      const int r = e / kMomTile, c = e % kMomTile, i = i0 + r;
      const int ca = bi * kMomTile + c, cb = bj * kMomTile + c;
      sa[r][c] = (i < n && ca < D) ? static_cast<double>(__ldg(f + static_cast<long>(i) * D + ca)) : 0.0;
      sb[r][c] = (i < n && cb < D) ? static_cast<double>(__ldg(f + static_cast<long>(i) * D + cb)) : 0.0;
    }
    __syncthreads();
    for (int k = 0; k < kMomRows; ++k) {
      double va[4], vb[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) va[r] = sa[k][4 * ty + r];
#pragma unroll
      for (int c = 0; c < 4; ++c) vb[c] = sb[k][4 * tx + c];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = fma(va[r], vb[c], acc[r][c]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int gr = bi * kMomTile + 4 * ty + r, gc = bj * kMomTile + 4 * tx + c;
      if (gr >= D || gc >= D) continue;
      gram[static_cast<long>(gr) * D + gc] += acc[r][c];
      if (bi != bj) gram[static_cast<long>(gc) * D + gr] += acc[r][c];
    }
}

inline unsigned stream_grid(long total, int per_sm) {
  const long blocks = (total + 255) / 256, cap = static_cast<long>(num_sms()) * per_sm;
  return static_cast<unsigned>(blocks < cap ? blocks : cap);
}

}  // namespace hg

extern "C" {

int hg_conv2d_general(const float* x, int B, int Cin, int H, int W, int kh, int kw, int stride, int ph, int pw, const void* wimg,
                      int Cout, int Nb, const float* bias, float* out, int Ctot, int c0, int passes, void* stream) {
  HG_REQUIRE(x && wimg && out, "hg_conv2d_general: null pointer");
  HG_REQUIRE(B > 0 && Cin > 0 && H > 0 && W > 0, "hg_conv2d_general: bad input shape");
  HG_REQUIRE(kh >= 1 && kh <= 7 && kw >= 1 && kw <= 7, "hg_conv2d_general: filter %dx%d (at most 7x7)", kh, kw);
  HG_REQUIRE(stride == 1 || stride == 2, "hg_conv2d_general: stride must be 1 or 2 (got %d)", stride);
  HG_REQUIRE(ph >= 0 && pw >= 0 && ph < kh && pw < kw, "hg_conv2d_general: padding (%d,%d) for a %dx%d filter", ph, pw, kh, kw);
  HG_REQUIRE(Cout > 0 && Cout <= hg::kGcMaxCout, "hg_conv2d_general: Cout=%d (1..448)", Cout);
  HG_REQUIRE(Nb >= 16 && Nb <= 128 && Nb % 16 == 0, "hg_conv2d_general: Nb=%d must be a multiple of 16 in [16,128]", Nb);
  HG_REQUIRE(passes == 1 || passes == 3, "hg_conv2d_general: passes must be 1 or 3");
  HG_REQUIRE(c0 >= 0 && c0 + Cout <= Ctot, "hg_conv2d_general: window [%d,%d) outside %d channels", c0, c0 + Cout, Ctot);
  const int Ho = (H + 2 * ph - kh) / stride + 1, Wo = (W + 2 * pw - kw) / stride + 1;
  HG_REQUIRE(H + 2 * ph >= kh && W + 2 * pw >= kw, "hg_conv2d_general: %dx%d input smaller than the %dx%d filter", H, W, kh, kw);
  const long K = static_cast<long>(kh) * kw * Cin;
  HG_REQUIRE(K <= (1L << 20), "hg_conv2d_general: K=%ld too large", K);
  const long M = static_cast<long>(B) * Ho * Wo;
  const int nblocks = (Cout + Nb - 1) / Nb;
  const long items = (M + 127) / 128 * nblocks;
  HG_REQUIRE(items < (1L << 31), "hg_conv2d_general: %ld work items", items);
  hg::GConvArgs a{x, B, Cin, H, W, kh, kw, stride, ph, pw, Ho, Wo, static_cast<const uint8_t*>(wimg), Cout, Nb, nblocks,
                  static_cast<int>((K + 63) / 64), bias, out, Ctot, c0};
  const int grid = items < hg::num_sms() ? static_cast<int>(items) : hg::num_sms();
  auto st = static_cast<cudaStream_t>(stream);
  // wgmma N: 64 or 128, whichever covers a block (columns past Nb are computed and dropped).  Blocks of at most 128 channels
  // leave the [64 x 128] accumulator and two 32-entry operand prefetches room in the registers without spilling.
  if (passes == 3) return Nb <= 64 ? hg::launch_conv_general<3, 64>(grid, st, a) : hg::launch_conv_general<3, 128>(grid, st, a);
  return Nb <= 64 ? hg::launch_conv_general<1, 64>(grid, st, a) : hg::launch_conv_general<1, 128>(grid, st, a);
}

int hg_pool3x3(const float* x, int B, int C, int H, int W, int stride, int pad, int avg, float* out, int Ctot, int c0,
               void* stream) {
  HG_REQUIRE(x && out, "hg_pool3x3: null pointer");
  HG_REQUIRE(B > 0 && C > 0 && H > 0 && W > 0, "hg_pool3x3: bad shape");
  HG_REQUIRE((stride == 2 && pad == 0 && !avg) || (stride == 1 && pad == 1),
             "hg_pool3x3: max at stride 2 / pad 0, or max / average at stride 1 / pad 1 (got stride %d pad %d avg %d)", stride,
             pad, avg);
  HG_REQUIRE(H + 2 * pad >= 3 && W + 2 * pad >= 3, "hg_pool3x3: %dx%d input smaller than the window", H, W);
  HG_REQUIRE(c0 >= 0 && c0 + C <= Ctot, "hg_pool3x3: window [%d,%d) outside %d channels", c0, c0 + C, Ctot);
  const int Ho = (H + 2 * pad - 3) / stride + 1, Wo = (W + 2 * pad - 3) / stride + 1;
  const long total = static_cast<long>(B) * C * Ho * Wo;
  hg::pool3x3_kernel<<<hg::stream_grid(total, 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, C, H, W, stride, pad, avg, out,
                                                                                               Ctot, c0, Ho, Wo, total);
  return hg::check_launch("hg_pool3x3");
}

int hg_global_avgpool(const float* x, long planes, int HW, float* out, void* stream) {
  HG_REQUIRE(x && out, "hg_global_avgpool: null pointer");
  HG_REQUIRE(planes > 0 && HW > 0, "hg_global_avgpool: bad shape");
  hg::global_avgpool_kernel<<<hg::stream_grid(planes * 32, 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, planes, HW, out);
  return hg::check_launch("hg_global_avgpool");
}

int hg_feature_moments(const float* feat, int n, int D, double* sum, double* gram, void* stream) {
  HG_REQUIRE(feat && sum && gram, "hg_feature_moments: null pointer");
  HG_REQUIRE(n > 0 && D > 0 && D <= 65536, "hg_feature_moments: bad shape n=%d D=%d", n, D);
  auto st = static_cast<cudaStream_t>(stream);
  hg::feature_sum_kernel<<<(D + 255) / 256, 256, 0, st>>>(feat, n, D, sum);
  int rc = hg::check_launch("hg_feature_moments(sum)");
  if (rc) return rc;
  const unsigned T = static_cast<unsigned>((D + hg::kMomTile - 1) / hg::kMomTile);
  hg::feature_gram_kernel<<<dim3(T, T), 256, 0, st>>>(feat, n, D, gram);
  return hg::check_launch("hg_feature_moments(gram)");
}

}  // extern "C"
