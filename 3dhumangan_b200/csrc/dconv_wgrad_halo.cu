// Weight gradient of the discriminator's 3x3 convolutions over haloed operand rows (rows of >= 128 pixels):
//     dW[co, ci, ky, kx] = sum_{b,y,x} dy[b, co, y, x] * x[b, ci, y + ky - 1, x + kx - 1]
// GEMM view per filter tap: D_tap[co, ci] += A[co, K = pixels] . B_tap[ci, K = pixels]^T.
//
// The first version (dconv_bwd.cu) rebuilds the B operand (rows = input channels, K-major along the pixels) once PER TAP from
// global memory through the tap's shift: nine times the loads and conversions, B single-buffered, and many launches per
// training iteration.
//
// Here the input is converted ONCE per image-row segment into the operand image the forward kernel uses (dconv_halo.cu):
// row = pixel (x0-1 .. x0+128), 128-byte row = 64 channels, SWIZZLE_128B.  Read as an MN-MAJOR B operand (wgmma with B
// transposed) that image has K = pixel rows and N = channels contiguous, so a filter tap is again nothing but a ROW offset of
// the descriptor start ((dy) selects the ring slot of image row y + dy, (dx) moves the start by one row).  A = dy rows are
// K-major as stored in NCHW.  A CTA walks down strips of image rows with a 4-slot ring of input rows (each input row is
// converted once and used by the three output rows around it) and double-buffered 64-pixel chunks of dy.  Two warpgroups
// build the operands together; warpgroup g issues the wgmmas of output channels 64g..64g+63 and keeps their
// [ntaps x 64 x 64] fp32 accumulators in registers for the CTA's lifetime (at most 4 taps per launch: a 3x3 filter takes
// three launches, one per filter row, per (128 output, 64 input)-channel block); per-CTA partials are reduced in fp64 in a
// fixed order (deterministic).
#include "common.cuh"
#include "wgmma.cuh"

namespace hg {

constexpr int kWhThreads = 256;                   // two warpgroups: operands, wgmma, drain
constexpr int kWhMaxTaps = 4;
constexpr int kWhSeg = 130;
constexpr uint32_t kWhX = 66 * 1024;              // 4 slots x 130 rows x 128 B, rounded to the swizzle pattern
constexpr uint32_t kWhDy = 128 * 128;             // [128 co x 64 px] bf16
constexpr uint32_t kWhSmem = 2 * kWhX + 4 * kWhDy + 32 * 8 + 16 + 1024;
static_assert(kWhSmem <= 232448, "shared memory budget");

struct WgHaloArgs {
  const float* dy;       // [B,Cout,H,W]
  const float* x;        // [B,Cin,H,W]
  float* part_w;         // [grid, ntaps, 128, 64]
  float* part_b;         // [grid, 128]
  int B, H, W, Cout, Cin;
  int co0, nco;          // <= 128 rows of dy
  int ci0, nci;          // <= 64 rows of x
  int ntaps;             // <= kWhMaxTaps
  int tdy[kWhMaxTaps], tdx[kWhMaxTaps];    // tap t reads x at (y + tdy, x + tdx)
  int strip;             // image rows per work unit
};

template <int kPasses>
__global__ void __launch_bounds__(kWhThreads, 1) conv3x3_wgrad_halo_kernel(WgHaloArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* x_hi = smem;
  uint8_t* x_lo = smem + kWhX;
  uint8_t* d_hi = smem + 2 * kWhX;               // 2 chunk buffers
  uint8_t* d_lo = d_hi + 2 * kWhDy;
  const int g = threadIdx.x >> 7, t128 = threadIdx.x & 127;

  const int HW = a.H * a.W;
  const int xtiles = a.W / 128, ystrips = a.H / a.strip;
  const int units = a.B * xtiles * ystrips;
  const int my_units = (units - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);
  const int S = a.strip;

  float d[kWhMaxTaps][32];
  // Operands are rewritten only after both warpgroups' wgmmas have completed (the ring slot / dy buffer that is refilled was
  // read two output rows / two chunks earlier; waiting for all of them keeps the protocol to two barriers per fill).
  auto operands_free = [&]() {
    wgmma_wait<0>();
#pragma unroll
    for (int tp = 0; tp < kWhMaxTaps; ++tp) acc_fence(d[tp]);
    named_barrier(1, 256);
  };
  auto operands_ready = [&]() {
    fence_proxy_async_smem();
    named_barrier(1, 256);
  };
  {
    // ------------------------------------------------------------------ producers + wgmma
    const int t = threadIdx.x;
    const int px = t & 127, half = t >> 7;       // x rows: one pixel, 32 channels
    const int sub = t & 7, rsub = t >> 3;        // dy: 8-pixel group, output-channel row (+ 32 i)
    float bsum[4] = {0.f, 0.f, 0.f, 0.f};
    uint32_t xcnt = 0, dcnt = 0, xbase = 0;
    bool started = false;
    for (int u = 0; u < my_units; ++u) {
      const int unit = blockIdx.x + u * gridDim.x;
      const int xb = unit % xtiles, ys = (unit / xtiles) % ystrips, b = unit / (xtiles * ystrips);
      const int x0 = xb * 128, y0 = ys * S;
      const float* xplane = a.x + (static_cast<long>(b) * a.Cin + a.ci0) * HW;
      const float* dplane = a.dy + (static_cast<long>(b) * a.Cout + a.co0) * HW;

      auto fill_x = [&](int y) {                 // image row y -> ring slot xcnt & 3
        const uint32_t slot = xcnt & 3;
        const bool rowok = y >= 0 && y < a.H;
        const long off = static_cast<long>(rowok ? y : 0) * a.W + x0 + px;
        float v[2][16];
        auto issue = [&](float (&dst)[16], int q) {
          const int c0 = half * 32 + q * 16;
          const float* src = xplane + static_cast<long>(c0) * HW + off;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            if (rowok && c0 + j < a.nci) asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(dst[j]) : "l"(src));
            else dst[j] = 0.f;
            src += HW;
          }
        };
        issue(v[0], 0);
        issue(v[1], 1);
        // halo pixels x0 - 1 and x0 + 128: threads 0..15 take 8 channels each
        float hv[8];
        const int hside = t >> 3, hg8 = t & 7;
        const int hx = hside ? x0 + 128 : x0 - 1;
        const bool hok = t < 16 && rowok && hx >= 0 && hx < a.W;
        if (t < 16) {
          const float* src = xplane + static_cast<long>(hg8 * 8) * HW + static_cast<long>(rowok ? y : 0) * a.W + (hok ? hx : 0);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            if (hok && hg8 * 8 + j < a.nci) asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(hv[j]) : "l"(src));
            else hv[j] = 0.f;
            src += HW;
          }
        }
        operands_free();
        const uint32_t row = slot * kWhSeg + 1 + px;
#pragma unroll
        for (int q = 0; q < 2; ++q) {
#pragma unroll
          for (int g = 0; g < 2; ++g) {
            float yv[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) yv[j] = v[q][g * 8 + j];
            store_a8<kPasses == 3>(x_hi, x_lo, row, half * 32 + q * 16 + g * 8, yv);
          }
        }
        if (t < 16) store_a8<kPasses == 3>(x_hi, x_lo, slot * kWhSeg + (hside ? kWhSeg - 1 : 0), hg8 * 8, hv);
        operands_ready();
        ++xcnt;
      };
      auto fill_dy = [&](int y, int c) {         // 64 pixels x0 + 64 c .. of image row y -> chunk buffer dcnt & 1
        const uint32_t buf = dcnt & 1;
        const long off = static_cast<long>(y) * a.W + x0 + c * 64 + sub * 8;
        float4 va[8];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int row = rsub + 32 * i;
          if (row < a.nco) {
            const float4* src = reinterpret_cast<const float4*>(dplane + static_cast<long>(row) * HW + off);
            va[2 * i] = __ldcs(src);
            va[2 * i + 1] = __ldcs(src + 1);
          } else {
            va[2 * i] = va[2 * i + 1] = make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
        operands_free();
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float yv[8] = {va[2 * i].x, va[2 * i].y, va[2 * i].z, va[2 * i].w,
                               va[2 * i + 1].x, va[2 * i + 1].y, va[2 * i + 1].z, va[2 * i + 1].w};
          bsum[i] += ((yv[0] + yv[1]) + (yv[2] + yv[3])) + ((yv[4] + yv[5]) + (yv[6] + yv[7]));
          store_a8<kPasses == 3>(d_hi + buf * kWhDy, d_lo + buf * kWhDy, rsub + 32 * i, sub * 8, yv);
        }
        operands_ready();
        ++dcnt;
      };
      // output row i, pixel chunk c: every tap of this launch on dy chunk buffer (dcnt - 1) & 1
      auto mma = [&](int i, int c) {
        const uint32_t buf = (dcnt - 1) & 1;
        const uint32_t ah = smem_u32(d_hi + buf * kWhDy) + g * 64 * 128, al = smem_u32(d_lo + buf * kWhDy) + g * 64 * 128;
        const uint32_t xh = smem_u32(x_hi), xl = smem_u32(x_lo);
#pragma unroll
        for (int tp = 0; tp < kWhMaxTaps; ++tp) {
          if (tp >= a.ntaps) continue;
          const uint32_t slot = (xbase + i + 1 + a.tdy[tp]) & 3;
          const uint32_t brow = (slot * kWhSeg + 1 + a.tdx[tp] + c * 64) * 128u;
          acc_fence(d[tp]);
          wgmma_fence();
#pragma unroll
          for (uint32_t ks = 0; ks < 4; ++ks) {
            const uint64_t da_h = wg_desc_sw128(ah) + 2 * ks, da_l = wg_desc_sw128(al) + 2 * ks;
            const uint64_t db_h = wg_desc_sw128(xh + brow + ks * 2048u), db_l = wg_desc_sw128(xl + brow + ks * 2048u);
            wgmma_bf16<64, 1>(d[tp], da_h, db_h, (started || ks > 0) ? 1u : 0u);
            if (kPasses == 3) {
              wgmma_bf16<64, 1>(d[tp], da_l, db_h, 1u);
              wgmma_bf16<64, 1>(d[tp], da_h, db_l, 1u);
            }
          }
        }
        wgmma_commit();
        started = true;
      };

      fill_x(y0 - 1);
      fill_x(y0);
      for (int i = 0; i < S; ++i) {
        fill_x(y0 + i + 1);
        fill_dy(y0 + i, 0);
        mma(i, 0);
        fill_dy(y0 + i, 1);
        mma(i, 1);
      }
      xbase += S + 2;
    }
    // bias gradient partials: rows rsub + 32 i, summed over the 8 pixel-group threads of a row
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float v = bsum[i];
      v += __shfl_xor_sync(0xffffffffu, v, 1);
      v += __shfl_xor_sync(0xffffffffu, v, 2);
      v += __shfl_xor_sync(0xffffffffu, v, 4);
      if (sub == 0) a.part_b[static_cast<long>(blockIdx.x) * 128 + rsub + 32 * i] = v;
    }
  }
  operands_free();
  // ---- drain: tap tp, output channel 64g + frag_row, input channel frag_col
  {
    float* dst0 = a.part_w + static_cast<long>(blockIdx.x) * a.ntaps * 128 * 64;
    if (my_units > 0) {
#pragma unroll
      for (int tp = 0; tp < kWhMaxTaps; ++tp) {
        if (tp >= a.ntaps) continue;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float* dst = dst0 + (static_cast<long>(tp) * 128 + g * 64 + frag_row(t128, i)) * 64;
#pragma unroll
          for (int j = 0; j < 8; ++j)
            *reinterpret_cast<float2*>(dst + frag_col(t128, j, 0)) = make_float2(d[tp][4 * j + 2 * i], d[tp][4 * j + 2 * i + 1]);
        }
      }
    } else {
      for (int i = threadIdx.x; i < a.ntaps * 128 * 64; i += kWhThreads) dst0[i] = 0.f;
      for (int i = threadIdx.x; i < 128; i += kWhThreads) a.part_b[static_cast<long>(blockIdx.x) * 128 + i] = 0.f;
    }
  }
}

__global__ void conv_wgrad_halo_reduce_kernel(const float* __restrict__ part_w, const float* __restrict__ part_b, int nparts,
                                              int nw, float* __restrict__ dw, float* __restrict__ db) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nw) {
    double acc = 0.0;
    for (int p = 0; p < nparts; ++p) acc += static_cast<double>(part_w[static_cast<long>(p) * nw + i]);
    dw[i] = static_cast<float>(acc);
  }
  if (db && i < 128) {
    double acc = 0.0;
    for (int p = 0; p < nparts; ++p) acc += static_cast<double>(part_b[static_cast<long>(p) * 128 + i]);
    db[i] = static_cast<float>(acc);
  }
}

}  // namespace hg

extern "C" {

// per CTA: kWhMaxTaps taps x 128 x 64 floats + 128 bias partials
size_t hg_conv3x3_wgrad_halo_workspace_bytes(void) {
  return static_cast<size_t>(hg::num_sms()) * (hg::kWhMaxTaps * 128 * 64 + 128) * sizeof(float);
}

// dw [ntaps, 128, 64] (rows >= nco and columns >= nci are zero), dbias [128] or null.  Requires W % 128 == 0.
int hg_conv3x3_wgrad_halo(const float* dy, const float* x, float* dw, float* dbias, void* workspace, int B, int H, int W,
                          int Cout, int Cin, int co0, int nco, int ci0, int nci, int ntaps, const int* tdy, const int* tdx,
                          int passes, void* stream) {
  HG_REQUIRE(dy && x && dw && workspace && tdy && tdx, "hg_conv3x3_wgrad_halo: null pointer");
  HG_REQUIRE(B > 0 && H > 0 && W > 0 && W % 128 == 0, "hg_conv3x3_wgrad_halo: the image width must be a multiple of 128 (got %d)", W);
  HG_REQUIRE(nco >= 1 && nco <= 128 && co0 >= 0 && co0 + nco <= Cout, "hg_conv3x3_wgrad_halo: bad output-channel block");
  HG_REQUIRE(nci >= 1 && nci <= 64 && ci0 >= 0 && ci0 + nci <= Cin, "hg_conv3x3_wgrad_halo: bad input-channel block");
  HG_REQUIRE(ntaps >= 1 && ntaps <= hg::kWhMaxTaps, "hg_conv3x3_wgrad_halo: 1..%d taps per launch (register accumulators)",
             hg::kWhMaxTaps);
  HG_REQUIRE(passes == 1 || passes == 3, "hg_conv3x3_wgrad_halo: passes must be 1 or 3");
  HG_REQUIRE(((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(workspace) | reinterpret_cast<uintptr_t>(dw)) & 15) == 0,
             "hg_conv3x3_wgrad_halo: dy / dw / workspace must be 16-byte aligned");
  hg::WgHaloArgs a{};
  for (int t = 0; t < ntaps; ++t) {
    HG_REQUIRE(tdy[t] >= -1 && tdy[t] <= 1 && tdx[t] >= -1 && tdx[t] <= 1, "hg_conv3x3_wgrad_halo: tap shift out of range");
    a.tdy[t] = tdy[t];
    a.tdx[t] = tdx[t];
  }
  int strip = 32;
  while (strip > 1 && H % strip != 0) strip >>= 1;
  a.dy = dy; a.x = x;
  a.B = B; a.H = H; a.W = W; a.Cout = Cout; a.Cin = Cin;
  a.co0 = co0; a.nco = nco; a.ci0 = ci0; a.nci = nci; a.ntaps = ntaps; a.strip = strip;
  const int units = B * (W / 128) * (H / strip);
  const int grid = units < hg::num_sms() ? units : hg::num_sms();
  a.part_w = static_cast<float*>(workspace);
  a.part_b = a.part_w + static_cast<size_t>(hg::num_sms()) * hg::kWhMaxTaps * 128 * 64;
  auto st = static_cast<cudaStream_t>(stream);
  cudaError_t e;
  if (passes == 3) {
    e = cudaFuncSetAttribute(hg::conv3x3_wgrad_halo_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, hg::kWhSmem);
    if (e == cudaSuccess) hg::conv3x3_wgrad_halo_kernel<3><<<grid, hg::kWhThreads, hg::kWhSmem, st>>>(a);
  } else {
    e = cudaFuncSetAttribute(hg::conv3x3_wgrad_halo_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, hg::kWhSmem);
    if (e == cudaSuccess) hg::conv3x3_wgrad_halo_kernel<1><<<grid, hg::kWhThreads, hg::kWhSmem, st>>>(a);
  }
  if (e != cudaSuccess) { hg::set_error("hg_conv3x3_wgrad_halo: smem opt-in failed: %s", cudaGetErrorString(e)); return 2; }
  int rc = hg::check_launch("hg_conv3x3_wgrad_halo");
  if (rc) return rc;
  const int nw = ntaps * 128 * 64;
  hg::conv_wgrad_halo_reduce_kernel<<<(nw + 255) / 256, 256, 0, st>>>(a.part_w, a.part_b, grid, nw, dw, dbias);
  return hg::check_launch("hg_conv3x3_wgrad_halo(reduce)");
}

}  // extern "C"
