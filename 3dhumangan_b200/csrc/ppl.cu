// Perceptual path length: the LPIPS (VGG, v0.1) distance heads and the input stage of StyleGAN2-ADA's PPL.  The VGG16 trunk
// runs on hg_conv2d / hg_bias_act / hg_maxpool2x2.
//
//   hg_lpips_input  out = (box mean of x over f x f windows - shift) / scale, per channel: StyleGAN2-ADA's integer-factor
//                   downsampling (`reshape(..., H/f, f, W/f, f).mean([3, 5])`) and LPIPS's scaling layer in one pass.
//   hg_lpips_level  one LPIPS level of B pairs: per pixel the channel norms of both endpoints, the normalised difference and
//                   its lin-weighted square sum, all in fp64, averaged over the H x W pixels into a per-pair fp64 accumulator.
//
// hg_lpips_level is launched once per level.  The level's features are read exactly once, and each launch reads tens of
// megabytes at the sizes PPL runs, so one launch per level costs nothing measurable over a fused launch, while it lets the
// caller consume and free each level's features as soon as the level ends.  The order of every sum is fixed and no float
// atomic is used, so repeated calls are bit-identical; the number of CTAs per pair is a constant, so a pair's value also does
// not depend on the other pairs of the batch.
#include "../../include/hg3d.h"
#include "common.cuh"

namespace hg {

constexpr int kLpThreads = 256;
constexpr int kLpPix = kLpThreads / 32;   // pixels per tile: one warp per pixel
constexpr int kLpCtasPerPair = 32;        // CTAs per pair and level (fewer when the level has fewer tiles)
constexpr int kLpMaxC = 1024;

// xor butterfly: a + b == b + a bit for bit, so every lane ends with the same sum
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
  return v;
}

// grid (CTAs per pair, B).  A tile is kLpPix consecutive pixels of one pair: both endpoints' [C] channel vectors are staged in
// shared memory as [pixel][C + 1] fp32 (read once from HBM), then warp w reduces pixel w over its channels in fp64.  Each CTA
// walks tiles blockIdx.x, blockIdx.x + gridDim.x, ... and stores its pixel sum at part[b * gridDim.x + blockIdx.x].
__global__ void __launch_bounds__(kLpThreads) lpips_level_kernel(const float* __restrict__ f0, const float* __restrict__ f1,
                                                                 const float* __restrict__ w, int C, int HW, double* __restrict__ part) {
  extern __shared__ float lp_smem[];
  __shared__ double red[kLpPix];
  const int stride = C + 1;
  float* sa = lp_smem;
  float* sb = lp_smem + kLpPix * stride;
  const long base = static_cast<long>(blockIdx.y) * C * HW;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles = (HW + kLpPix - 1) / kLpPix;
  double total = 0.0;
  for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int p0 = tile * kLpPix;
    __syncthreads();                       // the previous tile's reads of sa / sb are done
#pragma unroll 4
    for (int e = threadIdx.x; e < C * kLpPix; e += kLpThreads) {
      const int c = e / kLpPix, p = e % kLpPix;
      const bool in = p0 + p < HW;
      const long off = base + static_cast<long>(c) * HW + p0 + p;
      sa[p * stride + c] = in ? __ldg(f0 + off) : 0.f;
      sb[p * stride + c] = in ? __ldg(f1 + off) : 0.f;
    }
    __syncthreads();
    const float* pa = sa + warp * stride;
    const float* pb = sb + warp * stride;
    double na = 0.0, nb = 0.0;
    for (int c = lane; c < C; c += 32) {
      const double x = pa[c], y = pb[c];
      na = fma(x, x, na);
      nb = fma(y, y, nb);
    }
    const double ia = 1.0 / (sqrt(warp_sum(na)) + 1e-10), ib = 1.0 / (sqrt(warp_sum(nb)) + 1e-10);
    double d = 0.0;
    for (int c = lane; c < C; c += 32) {
      // both products rounded before the subtraction: a contracted fma would leave the rounding error of one product, so
      // two equal endpoints would not be exactly 0 apart
      const double diff = __dsub_rn(__dmul_rn(pa[c], ia), __dmul_rn(pb[c], ib));
      d = fma(static_cast<double>(__ldg(w + c)), diff * diff, d);
    }
    d = warp_sum(d);
    if (lane == 0) red[warp] = p0 + warp < HW ? d : 0.0;
    __syncthreads();
    if (threadIdx.x == 0)
      for (int p = 0; p < kLpPix; ++p) total += red[p];
  }
  if (threadIdx.x == 0) part[static_cast<long>(blockIdx.y) * gridDim.x + blockIdx.x] = total;
}

__global__ void lpips_finalize_kernel(const double* __restrict__ part, int ctas, int B, int HW, double* __restrict__ acc) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  double s = 0.0;
  for (int j = 0; j < ctas; ++j) s += part[static_cast<long>(b) * ctas + j];
  acc[b] += s / static_cast<double>(HW);
}

__global__ void __launch_bounds__(256) lpips_input_kernel(const float* __restrict__ x, int H, int W, int f,
                                                          const float* __restrict__ shift, const float* __restrict__ scale,
                                                          float* __restrict__ out, long total) {
  const int Ho = H / f, Wo = W / f;
  const double inv = 1.0 / (static_cast<double>(f) * f);
  for (long e = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total; e += static_cast<long>(gridDim.x) * blockDim.x) {
    const int ox = static_cast<int>(e % Wo);
    const int oy = static_cast<int>((e / Wo) % Ho);
    const long plane = e / (static_cast<long>(Wo) * Ho);      // b * 3 + c
    const int c = static_cast<int>(plane % 3);
    const float* src = x + plane * H * W + static_cast<long>(oy) * f * W + static_cast<long>(ox) * f;
    double s = 0.0;
    for (int i = 0; i < f; ++i)
      for (int j = 0; j < f; ++j) s += __ldg(src + static_cast<long>(i) * W + j);
    out[e] = (static_cast<float>(s * inv) - __ldg(shift + c)) / __ldg(scale + c);
  }
}

}  // namespace hg

extern "C" {

size_t hg_lpips_workspace_bytes(int B) {
  return B > 0 ? static_cast<size_t>(B) * hg::kLpCtasPerPair * sizeof(double) : 0;
}

int hg_lpips_level(const float* f0, const float* f1, const float* w, int B, int C, int HW, double* acc, double* workspace,
                   size_t workspace_bytes, void* stream) {
  HG_REQUIRE(f0 && f1 && w && acc && workspace, "hg_lpips_level: null pointer");
  HG_REQUIRE(B >= 1 && B <= 65535 && C >= 1 && C <= hg::kLpMaxC && HW >= 1, "hg_lpips_level: bad shape B=%d C=%d HW=%d (B <= 65535, "
             "C <= %d)", B, C, HW, hg::kLpMaxC);
  HG_REQUIRE(workspace_bytes >= hg_lpips_workspace_bytes(B), "hg_lpips_level: workspace of %zu bytes, %zu needed", workspace_bytes,
             hg_lpips_workspace_bytes(B));
  auto st = static_cast<cudaStream_t>(stream);
  const int tiles = (HW + hg::kLpPix - 1) / hg::kLpPix;
  const int ctas = tiles < hg::kLpCtasPerPair ? tiles : hg::kLpCtasPerPair;
  const size_t smem = 2 * hg::kLpPix * static_cast<size_t>(C + 1) * sizeof(float);
  if (smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(hg::lpips_level_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) { hg::set_error("hg_lpips_level: shared memory of %zu bytes refused: %s", smem, cudaGetErrorString(e)); return 2; }
  }
  hg::lpips_level_kernel<<<dim3(ctas, B), hg::kLpThreads, smem, st>>>(f0, f1, w, C, HW, workspace);
  const int rc = hg::check_launch("hg_lpips_level");
  if (rc) return rc;
  hg::lpips_finalize_kernel<<<(B + 127) / 128, 128, 0, st>>>(workspace, ctas, B, HW, acc);
  return hg::check_launch("hg_lpips_level(finalize)");
}

int hg_lpips_input(const float* x, int B, int H, int W, int f, const float* shift, const float* scale, float* out, void* stream) {
  HG_REQUIRE(x && shift && scale && out, "hg_lpips_input: null pointer");
  HG_REQUIRE(B >= 1 && H >= 1 && W >= 1 && f >= 1, "hg_lpips_input: bad shape B=%d H=%d W=%d f=%d", B, H, W, f);
  HG_REQUIRE(H % f == 0 && W % f == 0, "hg_lpips_input: %d x %d is not divisible by the factor %d", H, W, f);
  const long total = static_cast<long>(B) * 3 * (H / f) * (W / f);
  const long want = (total + 255) / 256;
  const int grid = static_cast<int>(want < 65535 ? want : 65535);
  hg::lpips_input_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, H, W, f, shift, scale, out, total);
  return hg::check_launch("hg_lpips_input");
}

}  // extern "C"
