// Weight gradient of the discriminator's 3x3 / 1x1 convolutions (autograd through nn.Conv2d in
// lib/discriminators/unet_discriminators.py:21-38), one launch per GROUP of filter taps and per output-channel chunk
// (as many taps as fit the register accumulators: ntaps * M-halves * N <= 256 with N = the Cin chunk rounded up to 64, 128
// or 256, so dy is read once per group):
//     dW[co, ci, ky, kx] = sum_{b,h,w} dy[b, co, h, w] * x[b, ci, h + ky - pad, w + kx - pad]
// Same machine as the SPADE weight gradient (csrc/synth_bwd.cu): K = pixels, both operands are K-major as stored
// (NCHW planes are contiguous along W), the operand warps convert rows of 64 pixels into bf16 hi/lo SW128 images --
// the x rows read through the tap's shift with zero padding at the image border.  Warpgroup g issues the wgmmas of output
// rows 64g..64g+63 of every M half; its fp32 accumulators stay in registers for the CTA's lifetime; per-CTA partials are
// reduced in fp64 in a fixed order.
#include "common.cuh"
#include "wgmma.cuh"

namespace hg {

constexpr int kDwThreads = 256;   // two warpgroups: operands, wgmma, drain
constexpr int kDwCo = 128;        // output channels per work item of the whole-layer mode
constexpr int kDwMaxTiles = 64;   // whole-layer mode: 128-pixel tiles summed by one CTA (bounds the fp32 accumulation)
constexpr uint32_t kDwImg = 256 * 128;
constexpr uint32_t kDwSmemBytes = 4 * kDwImg + 8 * 8 + 16 + 1024;

struct ConvWgradArgs {
  const float* dy;       // [B,Cout,H,W]
  const float* x;        // [B,Cin,H,W]
  float* part_w;         // [grid,256,nq]
  float* part_b;         // [grid,256]
  int B, H, W, Cout, Cin;
  int co0, nco;          // rows of dy handled by this launch (nco <= 256)
  int ci0, nci, nq;      // rows of x (nci valid, nq = nci rounded up to 32, <= 256)
  int ntaps;             // taps of this launch; tap t reads x at (h + oy[t], w + ox[t])
  int oy[9], ox[9];
  // whole-layer mode (hg_conv2d_wgrad_layer): blockIdx.y enumerates (256-row chunk of dy, 256-row chunk of x, group of `per`
  // taps) and the fields above are derived from it; every item owns `item_stride` floats of part_w (gridDim.x partials)
  int layer, ksize, per;
  long item_stride;
};

// item index -> chunk / tap-group geometry, shared by the GEMM kernel and its reduction
struct ConvWgradItem {
  int co0, nco, ci0, nci, nq, ntaps, t0;
};
__device__ __forceinline__ ConvWgradItem conv_wgrad_item(int idx, int Cout, int Cin, int ksize, int per) {
  const int kk = ksize * ksize;
  const int ngrp = (kk + per - 1) / per, nci_chunks = (Cin + 255) / 256;
  const int grp = idx % ngrp, cii = (idx / ngrp) % nci_chunks, coi = idx / (ngrp * nci_chunks);
  ConvWgradItem it;
  it.co0 = coi * kDwCo;
  it.nco = Cout - it.co0 < kDwCo ? Cout - it.co0 : kDwCo;
  it.ci0 = cii * 256;
  it.nci = Cin - it.ci0 < 256 ? Cin - it.ci0 : 256;
  it.nq = (it.nci + 31) / 32 * 32;
  it.t0 = grp * per;
  it.ntaps = kk - it.t0 < per ? kk - it.t0 : per;
  return it;
}

// wgmma N for a chunk of nq input channels
__host__ __device__ __forceinline__ int wgrad_n(int nq) { return nq <= 64 ? 64 : nq <= 128 ? 128 : 256; }

// kN: wgmma N (>= nq); kNAcc = 256 / kN accumulators of [64 x kN] per warpgroup, one per (tap, M half)
template <int kPasses, int kN>
__global__ void __launch_bounds__(kDwThreads, 1) conv_wgrad_kernel(ConvWgradArgs a) {
  constexpr int kNAcc = 256 / kN;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* s = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_hi = s;
  uint8_t* a_lo = s + kDwImg;
  uint8_t* b_hi = s + 2 * kDwImg;
  uint8_t* b_lo = s + 3 * kDwImg;
  const int g = threadIdx.x >> 7, t128 = threadIdx.x & 127;

  if (a.layer) {
    const ConvWgradItem it = conv_wgrad_item(blockIdx.y, a.Cout, a.Cin, a.ksize, a.per);
    a.co0 = it.co0; a.nco = it.nco; a.ci0 = it.ci0; a.nci = it.nci; a.nq = it.nq; a.ntaps = it.ntaps;
    const int pad = a.ksize >> 1;
    for (int t = 0; t < it.ntaps; ++t) {
      a.oy[t] = (it.t0 + t) / a.ksize - pad;
      a.ox[t] = (it.t0 + t) % a.ksize - pad;
    }
    a.part_w += static_cast<long>(blockIdx.y) * a.item_stride;
    a.part_b += static_cast<long>(blockIdx.y) * gridDim.x * 256;
  }
  const int HW = a.H * a.W, T = (HW + 127) / 128;
  const int total = a.B * T;
  const int count = (total - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);
  const int nmh = a.nco > 128 ? 2 : 1;          // M halves that carry rows
  const int nst_a = (a.nco + 31) >> 5, nst_b = a.nq >> 5;

  float d[kNAcc][kN / 2];
  // the operand images are single-buffered: both warpgroups' wgmmas that read them are complete before they are rewritten
  auto images_free = [&]() {
    wgmma_wait<0>();
#pragma unroll
    for (int ai = 0; ai < kNAcc; ++ai) acc_fence(d[ai]);
    named_barrier(1, 256);
  };
  auto images_ready = [&]() {
    fence_proxy_async_smem();
    named_barrier(1, 256);
  };
  {
    const int sub = threadIdx.x & 7, rsub = threadIdx.x >> 3;
    float bsum[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) bsum[i] = 0.f;
    uint32_t chunk = 0;
    for (int it = 0; it < count; ++it) {
      const int tile = blockIdx.x + it * gridDim.x;
      const int b = tile / T, ti = tile - b * T;
      const float* dbase = a.dy + (static_cast<long>(b) * a.Cout + a.co0) * HW;
      const float* xbase = a.x + (static_cast<long>(b) * a.Cin + a.ci0) * HW;
#pragma unroll 1
      for (int kc = 0; kc < 2; ++kc, ++chunk) {
        const int g0 = ti * 128 + kc * 64 + sub * 8;        // first pixel of this thread's 8
        const int nvalid = HW - g0;
        float4 va[16];
#pragma unroll
        for (int st = 0; st < 8; ++st) {
          const int row = st * 32 + rsub;
          if (st < nst_a && row < a.nco && nvalid >= 8) {
            const float4* src = reinterpret_cast<const float4*>(dbase + static_cast<long>(row) * HW + g0);
            va[2 * st] = __ldcs(src);
            va[2 * st + 1] = __ldcs(src + 1);
          } else {
            va[2 * st] = va[2 * st + 1] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (st < nst_a && row < a.nco && nvalid > 0) {      // ragged end of the image
              const float* src = dbase + static_cast<long>(row) * HW + g0;
              float t[8];
#pragma unroll
              for (int j = 0; j < 8; ++j) t[j] = j < nvalid ? src[j] : 0.f;
              va[2 * st] = make_float4(t[0], t[1], t[2], t[3]);
              va[2 * st + 1] = make_float4(t[4], t[5], t[6], t[7]);
            }
          }
        }
        images_free();
#pragma unroll
        for (int st = 0; st < 8; ++st) {
          if (st >= nmh * 4) break;
          const float y[8] = {va[2 * st].x, va[2 * st].y, va[2 * st].z, va[2 * st].w,
                              va[2 * st + 1].x, va[2 * st + 1].y, va[2 * st + 1].z, va[2 * st + 1].w};
          bsum[st] += ((y[0] + y[1]) + (y[2] + y[3])) + ((y[4] + y[5]) + (y[6] + y[7]));
          store_a8<kPasses == 3>(a_hi, a_lo, st * 32 + rsub, sub * 8, y);
        }
        // ---- x rows through each tap's shift (zero padding outside the image); re-reads hit L1/L2
        int ph[8], pw[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int g = g0 + j;
          ph[j] = g / a.W;
          pw[j] = g - ph[j] * a.W;
        }
#pragma unroll 1
        for (int t = 0; t < a.ntaps; ++t) {
          const int oy = a.oy[t], ox = a.ox[t];
          bool ok[8];
#pragma unroll
          for (int j = 0; j < 8; ++j)
            ok[j] = j < nvalid && ph[j] + oy >= 0 && ph[j] + oy < a.H && pw[j] + ox >= 0 && pw[j] + ox < a.W;
          const int shift = oy * a.W + ox;
          // all loads of this tap first (registers only), so that they overlap the MMAs of the previous tap;
          // the shared image is touched only after the EMPTY wait
          float yq[8][8];
#pragma unroll
          for (int st = 0; st < 8; ++st) {
            const int row = st * 32 + rsub;
            if (st < nst_b && row < a.nci) {
              const float* src = xbase + static_cast<long>(row) * HW + g0 + shift;
#pragma unroll
              for (int j = 0; j < 8; ++j) yq[st][j] = ok[j] ? __ldg(src + j) : 0.f;
            } else {
#pragma unroll
              for (int j = 0; j < 8; ++j) yq[st][j] = 0.f;
            }
          }
          if (t > 0) images_free();
#pragma unroll
          for (int st = 0; st < 8; ++st) {
            if (st >= nst_b) break;
            store_a8<kPasses == 3>(b_hi, b_lo, st * 32 + rsub, sub * 8, yq[st]);
          }
          images_ready();
          // accumulator ai = t * nmh + mh: rows mh*128 + 64g.. of A against every row of B
#pragma unroll
          for (int ai = 0; ai < kNAcc; ++ai) {
            if (ai / nmh != t) continue;
            const int mh = ai % nmh;
            const uint32_t ah = smem_u32(a_hi) + mh * (kDwImg / 2) + g * 64 * 128, al = ah + kDwImg;
            acc_fence(d[ai]);
            wgmma_fence();
            wg_k64<kN>(d[ai], ah, smem_u32(b_hi), chunk > 0);
            if (kPasses == 3) {
              wg_k64<kN>(d[ai], al, smem_u32(b_hi), true);
              wg_k64<kN>(d[ai], ah, smem_u32(b_lo), true);
            }
          }
          wgmma_commit();
        }
      }
    }
#pragma unroll
    for (int st = 0; st < 8; ++st) {
      float v = bsum[st];
      v += __shfl_xor_sync(0xffffffffu, v, 1);
      v += __shfl_xor_sync(0xffffffffu, v, 2);
      v += __shfl_xor_sync(0xffffffffu, v, 4);
      if (sub == 0) a.part_b[static_cast<long>(blockIdx.x) * 256 + st * 32 + rsub] = v;
    }
  }
  images_free();
  // ---- drain: accumulator (tap t, M half mh) -> rows mh*128 + 64g + frag_row of the [256 x nq] partial of tap t
  {
    float* dst0 = a.part_w + static_cast<long>(blockIdx.x) * a.ntaps * 256 * a.nq;
    if (count > 0) {
#pragma unroll
      for (int ai = 0; ai < kNAcc; ++ai) {
        if (ai >= a.ntaps * nmh) continue;
        const int t = ai / nmh, mh = ai % nmh;
        float* dst = dst0 + static_cast<long>(t) * 256 * a.nq;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int co = mh * 128 + g * 64 + frag_row(t128, i);
#pragma unroll
          for (int j = 0; j < kN / 8; ++j) {
            const int c = frag_col(t128, j, 0);
            if (c < a.nq) *reinterpret_cast<float2*>(dst + static_cast<long>(co) * a.nq + c) = make_float2(d[ai][4 * j + 2 * i], d[ai][4 * j + 2 * i + 1]);
          }
        }
      }
      if (nmh == 1)     // rows 128..255 of every tap are zero
        for (int t = 0; t < a.ntaps; ++t)
          for (int i = threadIdx.x; i < 128 * a.nq; i += kDwThreads) dst0[static_cast<long>(t) * 256 * a.nq + 128 * a.nq + i] = 0.f;
    } else {
      for (int i = threadIdx.x; i < a.ntaps * 256 * a.nq; i += kDwThreads) dst0[i] = 0.f;
      for (int i = threadIdx.x; i < 256; i += kDwThreads) a.part_b[static_cast<long>(blockIdx.x) * 256 + i] = 0.f;
    }
  }
}

__global__ void conv_wgrad_reduce_kernel(const float* __restrict__ part_w, const float* __restrict__ part_b, int nparts,
                                         int nw, float* __restrict__ dw, float* __restrict__ db) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nw) {
    double acc = 0.0;
    for (int p = 0; p < nparts; ++p) acc += static_cast<double>(part_w[static_cast<long>(p) * nw + i]);
    dw[i] = static_cast<float>(acc);
  }
  if (db && i < 256) {
    double acc = 0.0;
    for (int p = 0; p < nparts; ++p) acc += static_cast<double>(part_b[static_cast<long>(p) * 256 + i]);
    db[i] = static_cast<float>(acc);
  }
}

// whole-layer reduction: item partials -> dW [Cout, Cin, k, k] (and dbias from the items of the first x chunk / tap group), fp64,
// partials in ascending CTA order (deterministic)
__global__ void conv_wgrad_reduce_layer_kernel(const float* __restrict__ part_w, const float* __restrict__ part_b, int nparts,
                                               long item_stride, int Cout, int Cin, int ksize, int per, float* __restrict__ dW,
                                               float* __restrict__ db) {
  const ConvWgradItem it = conv_wgrad_item(blockIdx.y, Cout, Cin, ksize, per);
  const int nw = it.ntaps * 256 * it.nq;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const float* pw = part_w + static_cast<long>(blockIdx.y) * item_stride;
  if (i < nw) {
    const int t = i / (256 * it.nq), r = (i / it.nq) % 256, c = i % it.nq;
    if (r < it.nco && c < it.nci) {
      double acc = 0.0;
      for (int p = 0; p < nparts; ++p) acc += static_cast<double>(pw[static_cast<long>(p) * nw + i]);
      dW[(static_cast<long>(it.co0 + r) * Cin + it.ci0 + c) * (ksize * ksize) + it.t0 + t] = static_cast<float>(acc);
    }
  }
  if (db && it.ci0 == 0 && it.t0 == 0 && i < it.nco) {
    const float* pb = part_b + static_cast<long>(blockIdx.y) * nparts * 256;
    double acc = 0.0;
    for (int p = 0; p < nparts; ++p) acc += static_cast<double>(pb[static_cast<long>(p) * 256 + i]);
    db[it.co0 + i] = static_cast<float>(acc);
  }
}

template <int kPasses, int kN>
static cudaError_t launch_conv_wgrad_n(dim3 grid, cudaStream_t st, const ConvWgradArgs& a) {
  const cudaError_t e = cudaFuncSetAttribute(conv_wgrad_kernel<kPasses, kN>, cudaFuncAttributeMaxDynamicSharedMemorySize, kDwSmemBytes);
  if (e == cudaSuccess) conv_wgrad_kernel<kPasses, kN><<<grid, kDwThreads, kDwSmemBytes, st>>>(a);
  return e;
}
static cudaError_t launch_conv_wgrad(int passes, int n, dim3 grid, cudaStream_t st, const ConvWgradArgs& a) {
  if (passes == 3)
    return n == 64 ? launch_conv_wgrad_n<3, 64>(grid, st, a) : n == 128 ? launch_conv_wgrad_n<3, 128>(grid, st, a)
                                                              : launch_conv_wgrad_n<3, 256>(grid, st, a);
  return n == 64 ? launch_conv_wgrad_n<1, 64>(grid, st, a) : n == 128 ? launch_conv_wgrad_n<1, 128>(grid, st, a)
                                                            : launch_conv_wgrad_n<1, 256>(grid, st, a);
}

}  // namespace hg

extern "C" {

// worst case per CTA: ntaps * 256 * nq floats with ntaps * nq <= 512 (one M half), plus the bias partial
size_t hg_conv2d_wgrad_workspace_bytes(void) {
  return static_cast<size_t>(hg::num_sms()) * (512 * 256 + 256) * sizeof(float);
}

int hg_conv2d_wgrad_taps(const float* dy, const float* x, float* dw, float* dbias, void* workspace, int B, int H, int W,
                         int Cout, int Cin, int co0, int nco, int ci0, int nci, int ntaps, const int* oy, const int* ox,
                         int passes, void* stream) {
  HG_REQUIRE(dy && x && dw && workspace && oy && ox, "hg_conv2d_wgrad_taps: null pointer");
  HG_REQUIRE(B > 0 && H > 0 && W > 0 && (H * W) % 4 == 0, "hg_conv2d_wgrad_taps: bad image shape (H*W must be a multiple of 4)");
  HG_REQUIRE(nco >= 1 && nco <= 256 && co0 >= 0 && co0 + nco <= Cout, "hg_conv2d_wgrad_taps: bad output-channel chunk");
  HG_REQUIRE(nci >= 1 && nci <= 256 && ci0 >= 0 && ci0 + nci <= Cin, "hg_conv2d_wgrad_taps: bad input-channel chunk");
  HG_REQUIRE(passes == 1 || passes == 3, "hg_conv2d_wgrad_taps: passes must be 1 or 3");
  HG_REQUIRE(((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(workspace)) & 15) == 0,
             "hg_conv2d_wgrad_taps: dy / workspace must be 16-byte aligned");
  const int nq = (nci + 31) / 32 * 32;
  const int nmh = nco > 128 ? 2 : 1;
  HG_REQUIRE(ntaps >= 1 && ntaps <= 9 && ntaps * nmh * hg::wgrad_n(nq) <= 256,
             "hg_conv2d_wgrad_taps: %d taps x %d M-halves x %d columns do not fit the 256 accumulator columns", ntaps, nmh,
             hg::wgrad_n(nq));
  hg::ConvWgradArgs a{};
  for (int t = 0; t < ntaps; ++t) {
    HG_REQUIRE(oy[t] >= -1 && oy[t] <= 1 && ox[t] >= -1 && ox[t] <= 1, "hg_conv2d_wgrad_taps: tap shift out of range");
    a.oy[t] = oy[t];
    a.ox[t] = ox[t];
  }
  const int T = (H * W + 127) / 128;
  const int tiles = B * T;
  const int grid = tiles < hg::num_sms() ? tiles : hg::num_sms();
  float* part_w = static_cast<float*>(workspace);
  float* part_b = part_w + static_cast<size_t>(hg::num_sms()) * 512 * 256;
  a.dy = dy; a.x = x; a.part_w = part_w; a.part_b = part_b;
  a.B = B; a.H = H; a.W = W; a.Cout = Cout; a.Cin = Cin;
  a.co0 = co0; a.nco = nco; a.ci0 = ci0; a.nci = nci; a.nq = nq; a.ntaps = ntaps;
  auto st = static_cast<cudaStream_t>(stream);
  const cudaError_t e = hg::launch_conv_wgrad(passes, hg::wgrad_n(nq), dim3(grid), st, a);
  if (e != cudaSuccess) { hg::set_error("hg_conv2d_wgrad_taps: smem opt-in failed: %s", cudaGetErrorString(e)); return 2; }
  int rc = hg::check_launch("hg_conv2d_wgrad_taps");
  if (rc) return rc;
  // dw [ntaps, 256, nq] (rows >= nco and columns >= nci are zero), dbias [256]
  const int nw = ntaps * 256 * nq;
  hg::conv_wgrad_reduce_kernel<<<(nw + 255) / 256, 256, 0, st>>>(part_w, part_b, grid, nw, dw, dbias);
  return hg::check_launch("hg_conv2d_wgrad_taps(reduce)");
}

// ---- one launch per layer: every (dy chunk, x chunk, tap group) as blockIdx.y of the same grid.  The low-resolution layers
// (16^2 .. 64^2 pixels: 2 .. 32 tiles per image) needed 9 .. 36 launches of 16-128 CTAs each with hg_conv2d_wgrad_taps.
static void wgrad_layer_geometry(int B, int H, int W, int Cout, int Cin, int ksize, int* per, int* nitems, int* gx, long* item_stride) {
  const int kk = ksize * ksize;
  const int nq_max = ((Cin < 256 ? Cin : 256) + 31) / 32 * 32;
  *per = 256 / hg::wgrad_n(nq_max);        // one M half per item (kDwCo output channels)
  if (*per > kk) *per = kk;
  const int ngrp = (kk + *per - 1) / *per;
  *nitems = ((Cout + hg::kDwCo - 1) / hg::kDwCo) * ((Cin + 255) / 256) * ngrp;
  const int tiles = B * ((H * W + 127) / 128);
  // CTAs in flight: one per SM for a single item (every extra CTA is one more partial to drain and reduce), ~4 waves when the
  // grid is many small items of different cost
  int g = *nitems == 1 ? hg::num_sms() : 4 * hg::num_sms() / *nitems;
  if (g < 1) g = 1;
  // at most kDwMaxTiles tiles per CTA: each CTA sums its tiles in fp32 wgmma accumulators before the fp64 reduction, and the
  // bf16x3 product's error grows with that length (a 3x3 256 -> 64 layer at 512x512, B = 4, measured 6.3e-5 relative L2 with
  // 141 tiles per CTA, 3.2e-5 with 70)
  const int cap = (B * ((H * W + 127) / 128) + hg::kDwMaxTiles - 1) / hg::kDwMaxTiles;
  if (g < cap) g = cap;
  *gx = tiles < g ? tiles : g;
  *item_stride = static_cast<long>(*gx) * *per * 256 * nq_max;
}

size_t hg_conv2d_wgrad_layer_workspace_bytes(int B, int H, int W, int Cout, int Cin, int ksize) {
  int per, nitems, gx;
  long stride;
  wgrad_layer_geometry(B, H, W, Cout, Cin, ksize, &per, &nitems, &gx, &stride);
  return (static_cast<size_t>(nitems) * stride + static_cast<size_t>(nitems) * gx * 256) * sizeof(float);
}

int hg_conv2d_wgrad_layer(const float* dy, const float* x, float* dW, float* dbias, void* workspace, size_t workspace_bytes, int B,
                          int H, int W, int Cout, int Cin, int ksize, int passes, void* stream) {
  HG_REQUIRE(dy && x && dW && workspace, "hg_conv2d_wgrad_layer: null pointer");
  HG_REQUIRE(ksize == 1 || ksize == 3, "hg_conv2d_wgrad_layer: kernel size must be 1 or 3");
  HG_REQUIRE(B > 0 && H > 0 && W > 0 && (H * W) % 4 == 0, "hg_conv2d_wgrad_layer: bad image shape (H*W must be a multiple of 4)");
  HG_REQUIRE(Cout > 0 && Cin > 0, "hg_conv2d_wgrad_layer: bad channel counts");
  HG_REQUIRE(passes == 1 || passes == 3, "hg_conv2d_wgrad_layer: passes must be 1 or 3");
  HG_REQUIRE(((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(workspace)) & 15) == 0,
             "hg_conv2d_wgrad_layer: dy / workspace must be 16-byte aligned");
  int per, nitems, gx;
  long stride;
  wgrad_layer_geometry(B, H, W, Cout, Cin, ksize, &per, &nitems, &gx, &stride);
  HG_REQUIRE(workspace_bytes >= hg_conv2d_wgrad_layer_workspace_bytes(B, H, W, Cout, Cin, ksize),
             "hg_conv2d_wgrad_layer: workspace too small (%zu bytes)", workspace_bytes);
  HG_REQUIRE(nitems <= 65535, "hg_conv2d_wgrad_layer: too many work items");
  hg::ConvWgradArgs a{};
  float* part_w = static_cast<float*>(workspace);
  float* part_b = part_w + static_cast<size_t>(nitems) * stride;
  a.dy = dy; a.x = x; a.part_w = part_w; a.part_b = part_b;
  a.B = B; a.H = H; a.W = W; a.Cout = Cout; a.Cin = Cin;
  a.layer = 1; a.ksize = ksize; a.per = per; a.item_stride = stride;
  auto st = static_cast<cudaStream_t>(stream);
  const dim3 grid(gx, nitems);
  const int nq_max = ((Cin < 256 ? Cin : 256) + 31) / 32 * 32;
  const cudaError_t e = hg::launch_conv_wgrad(passes, hg::wgrad_n(nq_max), grid, st, a);
  if (e != cudaSuccess) { hg::set_error("hg_conv2d_wgrad_layer: smem opt-in failed: %s", cudaGetErrorString(e)); return 2; }
  int rc = hg::check_launch("hg_conv2d_wgrad_layer");
  if (rc) return rc;
  const int nw_max = per * 256 * 256;
  hg::conv_wgrad_reduce_layer_kernel<<<dim3((nw_max + 255) / 256, nitems), 256, 0, st>>>(part_w, part_b, gx, stride, Cout, Cin, ksize,
                                                                                          per, dW, dbias);
  return hg::check_launch("hg_conv2d_wgrad_layer(reduce)");
}

}  // extern "C"
