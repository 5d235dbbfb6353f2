// 3x3 'same' convolution of the U-Net discriminator as an implicit GEMM over ONE haloed operand tile per K chunk.
//
// The first version (dconv.cu, still used for 1x1 / small maps / the 3-channel stem) builds nine shifted copies of every
// [128 pixels x 64 channels] operand tile, one per filter tap: 9x the global loads and 9x the fp32 -> bf16 hi/lo
// conversion work.
//
// Here a CTA owns one image row of 128 output pixels (an M = 128 tile).  For one chunk of 64 input channels it converts the
// 3 x (128+2) haloed pixel block ONCE into the K-major SWIZZLE_128B operand layout (row = pixel, 390 rows) and issues all
// nine taps by moving the START ADDRESS of the A descriptor: tap (dy, dx) reads rows (dy + 1) * 130 + dx + 1 ... + 127.
// The swizzle of that layout is a function of the absolute shared-memory address bits, so a descriptor that starts at any
// whole row (a multiple of 128 bytes, base_offset = 0) addresses the rows that were written with the swizzle of their
// absolute row index.  Zero rows (outside the image) are the convolution's padding.
//
// Folded in, exactly as in dconv.cu (unet_discriminators.py:20-54): LeakyReLU(0.2) and nearest 2x up-sampling in front of
// the convolution, channel concatenation of two sources, bias, residual add (optionally of a half-resolution tensor).
//
// Warp roles (384 threads): warpgroups 0-1 convert the operand block together, then warpgroup g issues the wgmmas of
// pixels 64g..64g+63 (nsub <= 2 sub-blocks of <= 128 output channels, fp32 accumulators in registers) and stores them;
// warp 8 streams the weight stages.
#include "common.cuh"
#include "wgmma.cuh"

namespace hg {

constexpr int kHcThreads = 384;
constexpr int kHcSeg = 130;                       // pixels per haloed row segment
constexpr int kHcSegs = 3;                        // input rows y-1, y, y+1
constexpr uint32_t kHcA = 50 * 1024;              // 390 * 128 B rounded up to the 1024-byte swizzle pattern
constexpr int kHcBStages = 4;
constexpr uint32_t kHcB = 128 * 128;              // [128 x 64] bf16
constexpr uint32_t kHcSmem = 2 * kHcA + kHcBStages * kHcB + 256 * 4 + 32 * 8 + 1024;
static_assert(kHcSmem <= 232448, "shared memory budget");

struct HaloArgs {
  const float* x1;
  const float* x2;
  int C1, C2;
  int B, H, W;            // output size (= conv input after the optional up-sample)
  int up2, pre_lrelu;
  const uint8_t* wimg;    // packed [nblocks][kchunks][hi,lo][Nb x 64], K = tap-major (tap * Cin + c)
  int Cout, Nb, kchunks;  // kchunks = 9 * Cin / 64
  int nsub, nsubw;        // sub-blocks of `nsubw` (<= 128) output channels
  const float* bias;
  const float* residual;
  int res_up2;
  float* out;
};

enum { HB_FULL = 0 /*4*/, HB_EMPTY = 4 /*4*/ };

// kN: wgmma N of one sub-block (>= nsubw)
template <int kPasses, int kN>
__global__ void __launch_bounds__(kHcThreads, 1) conv3x3_halo_kernel(HaloArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_hi = smem;
  uint8_t* a_lo = smem + kHcA;
  uint8_t* b_st = smem + 2 * kHcA;
  float* tab_bias = reinterpret_cast<float*>(b_st + kHcBStages * kHcB);   // [256]
  uint64_t* bars = reinterpret_cast<uint64_t*>(tab_bias + 256);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // LeakyReLU in front of the convolution as max(v, slope * v), slope 1 = none: no run-time flag inside the unrolled loops
  const float lslope = a.pre_lrelu ? 0.2f : 1.f;
  for (int i = threadIdx.x; i < 256; i += blockDim.x) tab_bias[i] = (a.bias && i < a.Cout) ? a.bias[i] : 0.f;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kHcBStages; ++i) { mbar_init(bars + HB_FULL + i, 1); mbar_init(bars + HB_EMPTY + i, 2); }
    fence_mbar_init();
  }
  __syncthreads();

  const int HW = a.H * a.W;
  const int Hs = a.up2 ? a.H >> 1 : a.H, Ws = a.up2 ? a.W >> 1 : a.W;
  const long HWs = static_cast<long>(Hs) * Ws;
  const int Cin = a.C1 + a.C2;
  const int cblocks = Cin / 64;
  const int xtiles = a.W / 128;
  const int num_tiles = a.B * a.H * xtiles;
  const int my_tiles = (num_tiles - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);
  const uint32_t stage_bytes = static_cast<uint32_t>(a.nsubw) * 128;

  if (warp < 8) {
    regs_inc<kMmaRegs>();
    const int t = threadIdx.x;                 // 0..255
    const int g = t >> 7, t128 = t & 127;
    const int px = t & 127, half = t >> 7;     // one interior pixel, 32 of the chunk's 64 channels (two batches of 16)
    const int hside = t >> 3, hg8 = t & 7;     // threads 0..15: halo pixel (left / right), 8 channels
    float d[2][kN / 2];
    uint32_t st = 0, ph = 0, prev = ~0u;
    // the operand block is single-buffered: both warpgroups' wgmmas of the previous chunk are complete before it is rebuilt
    auto operands_free = [&]() {
      wgmma_wait<0>();
      acc_fence(d[0]);
      acc_fence(d[1]);
      if (prev != ~0u && t128 == 0) mbar_arrive(bars + HB_EMPTY + prev);
      prev = ~0u;
      named_barrier(1, 256);
    };
    for (int it = 0; it < my_tiles; ++it) {
      const int tile = blockIdx.x + it * gridDim.x;
      const int xb = tile % xtiles, y0 = (tile / xtiles) % a.H, b = tile / (xtiles * a.H);
      const int x0 = xb * 128;
      const int sx = a.up2 ? (x0 + px) >> 1 : x0 + px;
      const int hx = hside ? x0 + 128 : x0 - 1;
      const bool hxok = t < 16 && hx >= 0 && hx < a.W;
      const int hsx = hxok ? (a.up2 ? hx >> 1 : hx) : 0;
      for (int cb = 0; cb < cblocks; ++cb) {
        const int c0 = cb * 64;
        const float* plane = c0 < a.C1 ? a.x1 + (static_cast<long>(b) * a.C1 + c0) * HWs
                                       : a.x2 + (static_cast<long>(b) * a.C2 + (c0 - a.C1)) * HWs;
        float v[2][16];
        auto rowinfo = [&](int s, bool& ok, long& off) {
          const int y = y0 - 1 + s;
          ok = y >= 0 && y < a.H;
          off = static_cast<long>(ok ? (a.up2 ? y >> 1 : y) : 0) * Ws;
        };
        auto issue = [&](float (&dst)[16], int bi) {             // batch bi = segment * 2 + quarter
          bool ok;
          long off;
          rowinfo(bi >> 1, ok, off);
          const float* src = plane + static_cast<long>(half * 32 + (bi & 1) * 16) * HWs + off + sx;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(dst[j]) : "l"(src));
            src += HWs;
          }
        };
        auto convert = [&](const float (&cur)[16], int bi) {
          bool ok;
          long off;
          rowinfo(bi >> 1, ok, off);
          const uint32_t row = (bi >> 1) * kHcSeg + 1 + px;
#pragma unroll
          for (int gi = 0; gi < 2; ++gi) {
            float y[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              float val = ok ? cur[gi * 8 + j] : 0.f;
              val = fmaxf(val, lslope * val);
              y[j] = val;
            }
            store_a8<kPasses == 3>(a_hi, a_lo, row, half * 32 + (bi & 1) * 16 + gi * 8, y);
          }
        };
        issue(v[0], 0);
        issue(v[1], 1);
#pragma unroll
        for (int s = 0; s < kHcSegs; ++s) {
          // halo pixels of this segment (threads 0..15), loaded before the wait like the batches above
          float hv[8];
          bool hok = false;
          if (t < 16) {
            bool ok;
            long off;
            rowinfo(s, ok, off);
            hok = ok && hxok;
            const float* src = plane + static_cast<long>(hg8 * 8) * HWs + off + hsx;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(hv[j]) : "l"(src));
              src += HWs;
            }
          }
          if (s == 0) operands_free();
          convert(v[0], 2 * s);
          if (s < kHcSegs - 1) issue(v[0], 2 * s + 2);
          convert(v[1], 2 * s + 1);
          if (s < kHcSegs - 1) issue(v[1], 2 * s + 3);
          if (t < 16) {
            float y[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              float val = hok ? hv[j] : 0.f;
              val = fmaxf(val, lslope * val);
              y[j] = val;
            }
            store_a8<kPasses == 3>(a_hi, a_lo, s * kHcSeg + (hside ? kHcSeg - 1 : 0), hg8 * 8, y);
          }
        }
        fence_proxy_async_smem();
        named_barrier(1, 256);
        // ---- nine taps x nsub sub-blocks: warpgroup g reads pixel rows 64g.. of each tap's shifted window
        const uint32_t ahi = smem_u32(a_hi) + g * 64 * 128, alo = smem_u32(a_lo) + g * 64 * 128;
        for (int tap = 0; tap < 9; ++tap) {
          const int dy = tap / 3 - 1, dx = tap % 3 - 1;
          const uint32_t r0 = static_cast<uint32_t>((dy + 1) * kHcSeg + dx + 1) * 128u;
          const bool first = cb == 0 && tap == 0;
#pragma unroll
          for (int sb = 0; sb < 2; ++sb) {
            if (sb >= a.nsub) continue;
            // one weight stage: wait, issue, and release the stage consumed one step earlier once its wgmmas are done
            auto stage = [&](uint32_t a_tile, uint32_t a_tile2, bool two, bool accumulate) {
              mbar_wait(bars + HB_FULL + st, ph);
              acc_fence(d[sb]);
              wgmma_fence();
              const uint32_t bt = smem_u32(b_st + st * kHcB);
              wg_k64<kN>(d[sb], a_tile, bt, accumulate);
              if (two) wg_k64<kN>(d[sb], a_tile2, bt, true);
              wgmma_commit();
              wgmma_wait<1>();
              acc_fence(d[0]);
              acc_fence(d[1]);
              if (prev != ~0u && t128 == 0) mbar_arrive(bars + HB_EMPTY + prev);
              prev = st;
              if (++st == kHcBStages) { st = 0; ph ^= 1; }
            };
            stage(ahi + r0, alo + r0, kPasses == 3, !first);
            if (kPasses == 3) stage(ahi + r0, ahi + r0, false, true);
          }
        }
      }
      operands_free();
      // ---- epilogue straight from the fragments: pixel x0 + 64g + frag_row, channel sb * nsubw + frag_col
      const long pixrow = static_cast<long>(y0) * a.W;
#pragma unroll
      for (int sb = 0; sb < 2; ++sb) {
        if (sb >= a.nsub) continue;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int x = x0 + g * 64 + frag_row(t128, i);
          const long pix = pixrow + x;
          const long rpix = a.res_up2 ? static_cast<long>(y0 >> 1) * (a.W >> 1) + (x >> 1) : pix;
          const long rHW = a.res_up2 ? static_cast<long>(a.H >> 1) * (a.W >> 1) : HW;
#pragma unroll
          for (int j = 0; j < kN / 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int c = frag_col(t128, j, e), ch = sb * a.nsubw + c;
              if (c >= a.nsubw || ch >= a.Cout) continue;
              float val = d[sb][4 * j + 2 * i + e] + tab_bias[ch];
              if (a.residual) val += __ldg(a.residual + (static_cast<long>(b) * a.Cout + ch) * rHW + rpix);
              a.out[(static_cast<long>(b) * a.Cout + ch) * HW + pix] = val;
            }
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ weight producer
    regs_dec<kProducerRegs>();
    if (warp == 8 && lane == 0) {
      uint32_t st = 0, ph = 0;
      const size_t tile_bytes = static_cast<size_t>(a.Nb) * 128;       // one packed [Nb x 64] part
      for (int it = 0; it < my_tiles; ++it)
        for (int cb = 0; cb < cblocks; ++cb)
          for (int tap = 0; tap < 9; ++tap) {
            const int kc = tap * cblocks + cb;
            for (int sb = 0; sb < a.nsub; ++sb) {
              // sub-block sb of width nsubw: block nb = (sb * nsubw) / Nb of the packed image, row offset inside it
              const int nb = (sb * a.nsubw) / a.Nb, rowoff = (sb * a.nsubw) % a.Nb;
              for (int part = 0; part < (kPasses == 3 ? 2 : 1); ++part) {
                mbar_wait_backoff(bars + HB_EMPTY + st, ph ^ 1);
                mbar_arrive_expect_tx(bars + HB_FULL + st, stage_bytes);
                bulk_g2s(b_st + st * kHcB,
                         a.wimg + (static_cast<size_t>(nb * a.kchunks + kc) * 2 + part) * tile_bytes + static_cast<size_t>(rowoff) * 128,
                         stage_bytes, bars + HB_FULL + st);
                if (++st == kHcBStages) { st = 0; ph ^= 1; }
              }
            }
          }
    }
  }
}

template <int kPasses, int kN>
static int launch_halo(int grid, cudaStream_t st, const HaloArgs& a) {
  const cudaError_t e = cudaFuncSetAttribute(conv3x3_halo_kernel<kPasses, kN>, cudaFuncAttributeMaxDynamicSharedMemorySize, kHcSmem);
  if (e != cudaSuccess) { set_error("hg_conv2d (halo): smem opt-in failed: %s", cudaGetErrorString(e)); return 2; }
  conv3x3_halo_kernel<kPasses, kN><<<grid, kHcThreads, kHcSmem, st>>>(a);
  return check_launch("hg_conv2d (halo)");
}

}  // namespace hg

// Called by hg_conv2d (dconv.cu) for the shapes this kernel covers; not an exported entry point of its own.
int hg_conv3x3_halo_launch(const float* x1, int C1, const float* x2, int C2, int B, int H, int W, int up2, int pre_lrelu,
                           const void* wimg, int Cout, int Nb, const float* bias, const float* residual, int res_up2,
                           float* out, int passes, void* stream) {
  const int Cin = C1 + C2;
  // sub-blocks of <= 128 output channels: a packed [256 x 64] tile is two [128 x 64] tiles back to back
  const int nsubw = Nb > 128 ? 128 : Nb;
  const int nsub = (Cout + nsubw - 1) / nsubw;
  hg::HaloArgs a{x1, x2, C1, C2, B, H, W, up2, pre_lrelu, static_cast<const uint8_t*>(wimg), Cout, Nb, 9 * Cin / 64,
                 nsub, nsubw, bias, residual, res_up2, out};
  const int tiles = B * H * (W / 128);
  const int grid = tiles < hg::num_sms() ? tiles : hg::num_sms();
  auto st = static_cast<cudaStream_t>(stream);
  if (passes == 3) return nsubw <= 64 ? hg::launch_halo<3, 64>(grid, st, a) : hg::launch_halo<3, 128>(grid, st, a);
  return nsubw <= 64 ? hg::launch_halo<1, 64>(grid, st, a) : hg::launch_halo<1, 128>(grid, st, a);
}

// shapes the haloed kernel covers (everything else stays on dconv.cu's kernel)
bool hg_conv3x3_halo_eligible(int C1, int C2, int H, int W, int ksize, int Cout, int Nb) {
  if (ksize != 3 || W % 128 != 0) return false;
  if (C1 % 64 != 0 || C2 % 64 != 0) return false;
  if (Cout > 256) return false;
  const int nsubw = Nb > 128 ? 128 : Nb;
  if (Nb > 128 && Nb != 256) return false;
  if (nsubw % 16 != 0) return false;
  return (Cout + nsubw - 1) / nsubw <= 2;
}
