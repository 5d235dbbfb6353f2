// U-Net discriminator convolutions as implicit GEMMs on wgmma.
//
// Replaces the cuDNN conv2d calls behind ResBlock / UNetDiscriminator
// (lib/discriminators/unet_discriminators.py:7-72, 82-160): 3x3 (pad 1) and 1x1 convolutions over NCHW
// fp32 planes with everything around them folded into the operand producer or the epilogue:
//   * LeakyReLU(0.2) in front of the conv (:24,29,34)           -> applied while building the A operand
//   * nn.Upsample(scale_factor=2, nearest) in front (:26,41)    -> source pixel (y>>1, x>>1)
//   * torch.cat((skip, x), dim=1) (:147)                        -> two source tensors, split by channel
//   * bias, residual add `x_s + dx` (:54)                       -> epilogue
// GEMM view: M = 128 consecutive output pixels of one image, N = one Cout block (<= 256 channels; a work item is one
// pixel tile x one block, so that the [128 x 256] fp32 accumulator fits the registers of two warpgroups),
// K = taps x Cin in chunks of 64 (one tap, 64 channels).  Warpgroup g (warps 4g..4g+3) builds rows 64g..64g+63 of each
// operand chunk in a 4-slot ring and issues their wgmmas while it builds the next chunk; warp 8 streams the weight
// tiles.  Weights are pre-packed as [Cout, tap, Cin] (hg_pack_weight).
// AvgPool2d(2) of the down path is a separate streaming kernel (hg_pool_add).
#include <stdlib.h>
#include "common.cuh"
#include "wgmma.cuh"

namespace hg {

constexpr int kDcThreads = 384;   // warpgroups 0-1: operands + wgmma + epilogue, warp 8: weight stages
constexpr int kDcStages = 2;
constexpr uint32_t kDcA = 128 * 128;
constexpr uint32_t kDcB = 256 * 128;
constexpr uint32_t kDcSmem = 8 * kDcA + kDcStages * kDcB + 512 * 4 + 16 * 8 + 16 + 1024;

struct ConvArgs {
  const float* x1;
  const float* x2;
  int C1, C2;
  int B, H, W;          // output (= conv input after the optional up-sample) size
  int up2, pre_lrelu, ksize;
  const uint8_t* wimg;
  int Cout, Nb, nblocks, kchunks;
  const float* bias;
  const float* residual;
  float* out;
  int small_cin;        // taps * Cin <= 64: a single K chunk holding (tap, channel) pairs
  int res_up2;          // residual is [B,Cout,H/2,W/2] and nearest-up-sampled on the fly (identity shortcut of an up block)
};

enum { DB_FULL = 0 /*2*/, DB_EMPTY = 2 /*2*/ };

template <int kPasses, int N>
__global__ void __launch_bounds__(kDcThreads, 1) conv_kernel(ConvArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_hi = smem;
  uint8_t* a_lo = smem + 4 * kDcA;
  uint8_t* b_st = smem + 8 * kDcA;
  float* tab_bias = reinterpret_cast<float*>(b_st + kDcStages * kDcB);   // [512]
  uint64_t* bars = reinterpret_cast<uint64_t*>(tab_bias + 512);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // LeakyReLU in front of the convolution as max(v, slope * v), slope 1 = none: no run-time flag inside the unrolled loops
  const float lslope = a.pre_lrelu ? 0.2f : 1.f;
  for (int i = threadIdx.x; i < 512; i += blockDim.x) tab_bias[i] = (a.bias && i < a.Cout) ? a.bias[i] : 0.f;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kDcStages; ++i) { mbar_init(bars + DB_FULL + i, 1); mbar_init(bars + DB_EMPTY + i, 2); }
    fence_mbar_init();
  }
  __syncthreads();

  const int HW = a.H * a.W;
  const int Hs = a.up2 ? a.H >> 1 : a.H, Ws = a.up2 ? a.W >> 1 : a.W;
  const long HWs = static_cast<long>(Hs) * Ws;
  const int Cin = a.C1 + a.C2;
  const int taps = a.ksize * a.ksize;
  const int tiles_per_img = (HW + 127) / 128;
  const int num_items = a.B * tiles_per_img * a.nblocks;
  const int my_items = (num_items - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);
  const int nchunks = a.kchunks;
  const int cblocks = a.small_cin ? 1 : Cin / 64;
  const uint32_t stage_bytes = static_cast<uint32_t>(a.Nb) * 128;

  if (warp < 8) {
    // ------------------------------------------------------------------ operand producer + epilogue
    regs_inc<kMmaRegs>();
    // warp (g, q, h): rows q*32.. (q = 2g or 2g+1, inside warpgroup g's 64) and channels h*32.. of every chunk
    const int g = warp >> 2, q = 2 * g + (warp & 1), h = (warp >> 1) & 1, t = threadIdx.x & 127;
    const int row = q * 32 + lane;
    const uint32_t a_off = g * 64 * 128;
    uint32_t cnt = 0;   // running chunk counter (ring position)
    uint32_t st = 0, ph = 0;
    float d[N / 2];
    for (int it = 0; it < my_items; ++it) {
      const int item = blockIdx.x + it * gridDim.x;
      const int tile = item / a.nblocks, nb = item % a.nblocks;
      const int b = tile / tiles_per_img, p0 = (tile % tiles_per_img) * 128;
      const int pix = p0 + row;
      const bool valid = pix < HW;
      const int py = valid ? pix / a.W : 0, px = valid ? pix % a.W : 0;

      // returns false when the tap falls outside the image (zero padding); src = offset into an Hs x Ws plane
      auto tap_src = [&](int tap, long& off) {
        const int dy = a.ksize == 3 ? tap / 3 - 1 : 0, dx = a.ksize == 3 ? tap % 3 - 1 : 0;
        int sy = py + dy, sx = px + dx;
        const bool in = valid && sy >= 0 && sy < a.H && sx >= 0 && sx < a.W;
        sy = in ? sy : 0;
        sx = in ? sx : 0;
        if (a.up2) { sy >>= 1; sx >>= 1; }
        off = static_cast<long>(sy) * Ws + sx;
        return in;
      };
      auto issue = [&](float (&dst)[32], int ck, bool& in) {
        if (a.small_cin) {
          in = true;
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const int kk = h * 32 + j;
            const int tap = kk / Cin, c = kk - tap * Cin;
            long off = 0;
            const bool ok = kk < taps * Cin && tap_src(tap, off);
            const float* src = a.x1 + (static_cast<long>(b) * a.C1 + (ok ? c : 0)) * HWs + (ok ? off : 0);
            float v;
            asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(v) : "l"(src));
            dst[j] = ok ? v : 0.f;
          }
        } else {
          const int tap = ck / cblocks, c0 = (ck - tap * cblocks) * 64 + h * 32;
          long off = 0;
          in = tap_src(tap, off);
          const float* src = c0 < a.C1 ? a.x1 + (static_cast<long>(b) * a.C1 + c0) * HWs + off
                                       : a.x2 + (static_cast<long>(b) * a.C2 + (c0 - a.C1)) * HWs + off;
#pragma unroll
          for (int j = 0; j < 32; ++j) asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(dst[j]) : "l"(src + j * HWs));
        }
      };
      // one weight stage: wait, issue, and release the stage consumed one step earlier once its wgmmas are done
      uint32_t prev = ~0u;
      auto stage = [&](uint32_t a_tile, uint32_t a_tile2, bool two, bool accumulate) {
        mbar_wait(bars + DB_FULL + st, ph);
        acc_fence(d);
        wgmma_fence();
        const uint32_t bt = smem_u32(b_st + st * kDcB);
        wg_k64<N>(d, a_tile, bt, accumulate);
        if (two) wg_k64<N>(d, a_tile2, bt, true);
        wgmma_commit();
        wgmma_wait<1>();
        acc_fence(d);
        if (prev != ~0u && t == 0) mbar_arrive(bars + DB_EMPTY + prev);
        prev = st;
        if (++st == kDcStages) { st = 0; ph ^= 1; }
      };
      // a ring slot is rewritten four chunks later: by then every warp of the group has seen its wgmmas complete
      auto convert = [&](float (&cur)[32], bool in, int ck) {
        const uint32_t slot = cnt & 3;
#pragma unroll
        for (int gi = 0; gi < 4; ++gi) {
          float y[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            float v = in ? cur[gi * 8 + j] : 0.f;
            v = fmaxf(v, lslope * v);
            y[j] = v;
          }
          store_a8<kPasses == 3>(a_hi + slot * kDcA, a_lo + slot * kDcA, row, h * 32 + gi * 8, y);
        }
        fence_proxy_async_smem();
        named_barrier(1 + g, 128);
        const uint32_t ahi = smem_u32(a_hi + slot * kDcA) + a_off, alo = smem_u32(a_lo + slot * kDcA) + a_off;
        stage(ahi, alo, kPasses == 3, ck > 0);
        if (kPasses == 3) stage(ahi, ahi, false, true);
        ++cnt;
      };
      float xa[32], xb[32];
      bool ina = false, inb = false;
      issue(xa, 0, ina);
      for (int ck = 0; ck < nchunks; ck += 2) {
        if (ck + 1 < nchunks) issue(xb, ck + 1, inb);
        convert(xa, ina, ck);
        if (ck + 1 < nchunks) {
          if (ck + 2 < nchunks) issue(xa, ck + 2, ina);
          convert(xb, inb, ck + 1);
        }
      }

      // ---- epilogue straight from the fragments: rows 64g + frag_row, channels nb*Nb + frag_col
      wgmma_wait<0>();
      acc_fence(d);
      if (t == 0) mbar_arrive(bars + DB_EMPTY + prev);
      const long rHW = a.res_up2 ? static_cast<long>(a.H >> 1) * (a.W >> 1) : HW;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int epix = p0 + g * 64 + frag_row(t, i);
        if (epix >= HW) continue;
        const int ey = epix / a.W, ex = epix % a.W;
        const long robase = a.res_up2 ? static_cast<long>(ey >> 1) * (a.W >> 1) + (ex >> 1) : epix;
#pragma unroll
        for (int j = 0; j < N / 8; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = frag_col(t, j, e), ch = nb * a.Nb + c;
            if (c >= a.Nb || ch >= a.Cout) continue;
            float v = d[4 * j + 2 * i + e] + tab_bias[ch];
            if (a.residual) v += __ldg(a.residual + (static_cast<long>(b) * a.Cout + ch) * rHW + robase);
            a.out[(static_cast<long>(b) * a.Cout + ch) * HW + epix] = v;
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
              mbar_wait_backoff(bars + DB_EMPTY + st, ph ^ 1);
              mbar_arrive_expect_tx(bars + DB_FULL + st, stage_bytes);
              bulk_g2s(b_st + st * kDcB,
                       a.wimg + (static_cast<size_t>(nb * nchunks + ck) * 2 + part) * stage_bytes, stage_bytes,
                       bars + DB_FULL + st);
              if (++st == kDcStages) { st = 0; ph ^= 1; }
            }
      }
    }
  }
}

template <int kPasses, int N>
static int launch_conv(int grid, cudaStream_t st, const ConvArgs& a) {
  const cudaError_t e = cudaFuncSetAttribute(conv_kernel<kPasses, N>, cudaFuncAttributeMaxDynamicSharedMemorySize, kDcSmem);
  if (e != cudaSuccess) { set_error("hg_conv2d: smem opt-in failed: %s", cudaGetErrorString(e)); return 2; }
  conv_kernel<kPasses, N><<<grid, kDcThreads, kDcSmem, st>>>(a);
  return check_launch("hg_conv2d");
}

// out[B,C,H,W] = P_a(a) + P_b(b) with P = 2x2 average pooling when the flag is set (source 2H x 2W),
// identity otherwise; b may be null.  (AvgPool2d(2) + residual add of the down blocks, :42-44, :52-54.)
__global__ void pool_add_kernel(const float* __restrict__ a, int pool_a, const float* __restrict__ b, int pool_b,
                                float* __restrict__ out, long planes, int H, int W) {
  const long total = planes * H * W;
  for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % W), y = static_cast<int>((i / W) % H);
    const long pl = i / (static_cast<long>(W) * H);
    auto fetch = [&](const float* s, int pool) {
      if (!pool) return s[i];
      const float* p = s + (pl * 2 * H + 2 * y) * 2 * W + 2 * x;
      return ((p[0] + p[1]) + (p[2 * W] + p[2 * W + 1])) * 0.25f;
    };
    float v = fetch(a, pool_a);
    if (b) v += fetch(b, pool_b);
    out[i] = v;
  }
}

// Full-extent convolution == dense layer (latent_layer, :117-118, :135): out[b,o] = bias[o] + <W[o,:], x[b,:]>
__global__ void dense_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                             float* __restrict__ out, int B, int K, int O) {
  const int o = blockIdx.x;
  __shared__ float red[8][33];
  for (int b0 = 0; b0 < B; b0 += 8) {
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
      const float wv = w[static_cast<long>(o) * K + k];
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (b0 + i < B) acc[i] = fmaf(wv, x[static_cast<long>(b0 + i) * K + k], acc[i]);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      for (int s = 16; s > 0; s >>= 1) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], s);
      if ((threadIdx.x & 31) == 0) red[i][threadIdx.x >> 5] = acc[i];
    }
    __syncthreads();
    if (threadIdx.x < 8 && b0 + threadIdx.x < B) {
      float t = 0.f;
      for (int i = 0; i < static_cast<int>(blockDim.x >> 5); ++i) t += red[threadIdx.x][i];
      out[static_cast<long>(b0 + threadIdx.x) * O + o] = t + (bias ? bias[o] : 0.f);
    }
    __syncthreads();
  }
}

}  // namespace hg

// dconv_halo.cu
int hg_conv3x3_halo_launch(const float* x1, int C1, const float* x2, int C2, int B, int H, int W, int up2, int pre_lrelu,
                           const void* wimg, int Cout, int Nb, const float* bias, const float* residual, int res_up2,
                           float* out, int passes, void* stream);
bool hg_conv3x3_halo_eligible(int C1, int C2, int H, int W, int ksize, int Cout, int Nb);
// dconv_small.cu
int hg_conv_small_launch(const float* x, int Cin, int B, int H, int W, int up2, int pre_lrelu, int ksize, const void* wimg, int Cout,
                         int Nb, const float* bias, const float* residual, int res_up2, float* out, void* stream);

static bool halo_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("HG3D_CONV_HALO");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v == 1;
}

extern "C" {

int hg_conv2d(const float* x1, int C1, const float* x2, int C2, int B, int H, int W, int up2, int pre_lrelu, int ksize,
              const void* wimg, int Cout, int Nb, const float* bias, const float* residual, int res_up2, float* out,
              int passes, void* stream) {
  HG_REQUIRE(x1 && wimg && out, "hg_conv2d: null pointer");
  HG_REQUIRE(ksize == 1 || ksize == 3, "hg_conv2d: kernel size must be 1 or 3 (got %d)", ksize);
  HG_REQUIRE(B > 0 && H > 0 && W > 0 && C1 > 0 && C2 >= 0 && Cout > 0, "hg_conv2d: bad shape");
  HG_REQUIRE((C2 == 0) == (x2 == nullptr), "hg_conv2d: x2 / C2 mismatch");
  HG_REQUIRE(!up2 || (H % 2 == 0 && W % 2 == 0), "hg_conv2d: up2 needs even output size");
  HG_REQUIRE(passes == 1 || passes == 3, "hg_conv2d: passes must be 1 or 3");
  HG_REQUIRE(Nb >= 16 && Nb <= 256 && Nb % 16 == 0, "hg_conv2d: Nb=%d must be a multiple of 16 in [16,256]", Nb);
  const int Cin = C1 + C2, taps = ksize * ksize;
  // single-chunk contractions: the 3-channel stem and the 64 -> 1 / 26 heads.  A 64 -> 256 1x1 layer (the data gradient of an
  // up-sampling shortcut) also has taps * Cin == 64 but is an ordinary K = 64, N = 256 GEMM: tensor-core path (the SIMT kernel
  // re-read x once per 32 output channels)
  const int small = (taps * Cin <= 64 && !(Cin % 64 == 0 && Cout > 32)) ? 1 : 0;
  HG_REQUIRE(small || (C1 % 64 == 0 && C2 % 64 == 0), "hg_conv2d: channel counts must be multiples of 64 (or taps*Cin <= 64)");
  HG_REQUIRE(!small || C2 == 0, "hg_conv2d: the small-Cin path takes a single input");
  const int nblocks = (Cout + Nb - 1) / Nb;
  HG_REQUIRE(nblocks <= 2, "hg_conv2d: at most two N blocks (Cout <= 2*Nb)");
  // tiny contractions (3-channel stem, 64 -> 27 heads): fp32 SIMT kernel, memory bound (dconv_small.cu)
  if (small && halo_enabled()) {
    const int rc = hg_conv_small_launch(x1, C1, B, H, W, up2, pre_lrelu, ksize, wimg, Cout, Nb, bias, residual, res_up2, out, stream);
    if (rc >= 0) return rc;
  }
  // 3x3 convolutions on rows of >= 128 pixels (84 % of the discriminator's FLOPs): one haloed operand tile per K chunk,
  // nine taps by descriptor offset (dconv_halo.cu)
  if (!small && halo_enabled() && hg_conv3x3_halo_eligible(C1, C2, H, W, ksize, Cout, Nb))
    return hg_conv3x3_halo_launch(x1, C1, x2, C2, B, H, W, up2, pre_lrelu, wimg, Cout, Nb, bias, residual, res_up2, out,
                                  passes, stream);
  hg::ConvArgs a{x1, x2, C1, C2, B, H, W, up2, pre_lrelu, ksize, static_cast<const uint8_t*>(wimg), Cout, Nb, nblocks,
                 small ? 1 : taps * Cin / 64, bias, residual, out, small, res_up2};
  const int items = B * ((H * W + 127) / 128) * nblocks;
  const int grid = items < hg::num_sms() ? items : hg::num_sms();
  auto st = static_cast<cudaStream_t>(stream);
  // wgmma N: the smallest of 64 / 128 / 256 that covers a block (columns past Nb are computed and dropped)
  const int n = Nb <= 64 ? 64 : Nb <= 128 ? 128 : 256;
  if (passes == 3) {
    if (n == 64) return hg::launch_conv<3, 64>(grid, st, a);
    if (n == 128) return hg::launch_conv<3, 128>(grid, st, a);
    return hg::launch_conv<3, 256>(grid, st, a);
  }
  if (n == 64) return hg::launch_conv<1, 64>(grid, st, a);
  if (n == 128) return hg::launch_conv<1, 128>(grid, st, a);
  return hg::launch_conv<1, 256>(grid, st, a);
}

int hg_pool_add(const float* a, int pool_a, const float* b, int pool_b, float* out, long planes, int H, int W,
                void* stream) {
  HG_REQUIRE(a && out && planes > 0 && H > 0 && W > 0, "hg_pool_add: bad arguments");
  const long total = planes * H * W;
  long blocks = (total + 255) / 256;
  const long cap = static_cast<long>(hg::num_sms()) * 16;
  if (blocks > cap) blocks = cap;
  hg::pool_add_kernel<<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, pool_a, b, pool_b, out,
                                                                                                    planes, H, W);
  return hg::check_launch("hg_pool_add");
}

int hg_dense(const float* x, const float* w, const float* bias, float* out, int B, int K, int O, void* stream) {
  HG_REQUIRE(x && w && out && B > 0 && K > 0 && O > 0, "hg_dense: bad arguments");
  hg::dense_kernel<<<O, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, w, bias, out, B, K, O);
  return hg::check_launch("hg_dense");
}

}  // extern "C"
