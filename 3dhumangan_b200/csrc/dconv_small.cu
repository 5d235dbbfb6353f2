// Convolutions with a tiny contraction (taps * Cin <= 64): the discriminator's 3-channel stem (3 -> 128, 3x3; and 3 -> 128, 1x1
// shortcut) and its heads (64 -> 1 + 26, 1x1) at full resolution (unet_discriminators.py:96-118, 139-152).  Their tensor-core
// tiles would be almost empty (K = 27 of 64) and the layers are bound by the 0.5-1 GB they write / read, so they run as a plain
// fp32 SIMT kernel: a thread owns one output pixel and 32 output channels, the K <= 64 inputs of its patch live in registers,
// the weights of the channel group in shared memory (fp32 rebuilt from the packed bf16 hi + lo image: 2^-17 relative, products
// and sums in fp32) are read as broadcast float4.  Same fused options (LeakyReLU / nearest 2x up-sampling in front, bias, residual).
#include <cuda_bf16.h>
#include "common.cuh"
#include "wgmma.cuh"

namespace hg {

struct SmallConvArgs {
  const float* x;
  int Cin, B, H, W, up2, pre_lrelu, ksize;
  const uint8_t* wimg;   // packed [nblocks][1][hi,lo][Nb x 64], K index = tap * Cin + c
  int Cout, Nb;
  const float* bias;
  const float* residual;
  int res_up2;
  float* out;
};

// KS / CIN are compile-time: the (tap, channel) decomposition of k must not cost integer divisions per load
template <int KS, int CIN>
__global__ void __launch_bounds__(128) conv_small_kernel(SmallConvArgs a) {
  constexpr int K = KS * KS * CIN;
  static_assert(K <= 64, "single K chunk");
  __shared__ __align__(16) float ws[K][32];    // [k][co within the group]
  __shared__ float bs[32];
  const int co0 = blockIdx.y * 32;
  for (int i = threadIdx.x; i < K * 32; i += 128) {
    const int k = i >> 5, c = i & 31, n = co0 + c;
    float w = 0.f;
    if (n < a.Cout) {
      const int nb = n / a.Nb, r = n % a.Nb;
      const uint8_t* hi = a.wimg + static_cast<size_t>(nb) * 2 * a.Nb * 128;
      const uint8_t* lo = hi + static_cast<size_t>(a.Nb) * 128;
      const uint32_t off = sw128_offset(r, k);
      w = __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(hi + off)) +
          __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(lo + off));
    }
    ws[k][c] = w;
  }
  if (threadIdx.x < 32) bs[threadIdx.x] = (a.bias && co0 + threadIdx.x < a.Cout) ? a.bias[co0 + threadIdx.x] : 0.f;
  __syncthreads();
  const long HW = static_cast<long>(a.H) * a.W;
  const long npix = static_cast<long>(a.B) * HW;
  // persistent over pixel blocks: the weights of the channel group are staged once per CTA, not once per 128 pixels
  for (long pix = static_cast<long>(blockIdx.x) * 128 + threadIdx.x; pix < npix; pix += static_cast<long>(gridDim.x) * 128) {
  const int b = static_cast<int>(pix / HW);
  const long q = pix - b * HW;
  const int py = static_cast<int>(q / a.W), px = static_cast<int>(q - static_cast<long>(py) * a.W);
  const int Hs = a.up2 ? a.H >> 1 : a.H, Ws = a.up2 ? a.W >> 1 : a.W;
  const long HWs = static_cast<long>(Hs) * Ws;
  const float* xb = a.x + static_cast<long>(b) * CIN * HWs;
  float v[K];
  constexpr int pad = KS >> 1;
#pragma unroll
  for (int tap = 0; tap < KS * KS; ++tap) {
    int sy = py + tap / KS - pad, sx = px + tap % KS - pad;
    const bool in = sy >= 0 && sy < a.H && sx >= 0 && sx < a.W;
    if (a.up2) { sy >>= 1; sx >>= 1; }
    const float* src = xb + static_cast<long>(sy) * Ws + sx;
#pragma unroll
    for (int c = 0; c < CIN; ++c) {
      float val = in ? __ldg(src + c * HWs) : 0.f;
      if (a.pre_lrelu) val = val > 0.f ? val : 0.2f * val;
      v[tap * CIN + c] = val;
    }
  }
  float acc[32];
#pragma unroll
  for (int c = 0; c < 32; ++c) acc[c] = bs[c];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    {
#pragma unroll
      for (int c4 = 0; c4 < 8; ++c4) {
        const float4 w = *reinterpret_cast<const float4*>(&ws[k][c4 * 4]);
        acc[c4 * 4 + 0] = fmaf(v[k], w.x, acc[c4 * 4 + 0]);
        acc[c4 * 4 + 1] = fmaf(v[k], w.y, acc[c4 * 4 + 1]);
        acc[c4 * 4 + 2] = fmaf(v[k], w.z, acc[c4 * 4 + 2]);
        acc[c4 * 4 + 3] = fmaf(v[k], w.w, acc[c4 * 4 + 3]);
      }
    }
  }
  const long rHW = a.res_up2 ? static_cast<long>(a.H >> 1) * (a.W >> 1) : HW;
  const long rq = a.res_up2 ? static_cast<long>(py >> 1) * (a.W >> 1) + (px >> 1) : q;
#pragma unroll
  for (int c = 0; c < 32; ++c) {
    const int n = co0 + c;
    if (n < a.Cout) {
      float o = acc[c];
      if (a.residual) o += __ldg(a.residual + (static_cast<long>(b) * a.Cout + n) * rHW + rq);
      a.out[(static_cast<long>(b) * a.Cout + n) * HW + q] = o;
    }
  }
  }
}

}  // namespace hg

// called by hg_conv2d for taps * Cin <= 64 (single source)
int hg_conv_small_launch(const float* x, int Cin, int B, int H, int W, int up2, int pre_lrelu, int ksize, const void* wimg, int Cout,
                         int Nb, const float* bias, const float* residual, int res_up2, float* out, void* stream) {
  hg::SmallConvArgs a{x, Cin, B, H, W, up2, pre_lrelu, ksize, static_cast<const uint8_t*>(wimg), Cout, Nb, bias, residual, res_up2, out};
  const long pixels = static_cast<long>(B) * H * W;
  const unsigned groups = static_cast<unsigned>((Cout + 31) / 32);
  const long blocks = (pixels + 127) / 128;
  const long per_group = (static_cast<long>(hg::num_sms()) * 8 + groups - 1) / groups;      // ~8 resident CTAs per SM in total
  dim3 grid(static_cast<unsigned>(blocks < per_group ? blocks : per_group), groups);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (ksize == 3 && Cin == 3) hg::conv_small_kernel<3, 3><<<grid, 128, 0, st>>>(a);
  else if (ksize == 1 && Cin == 3) hg::conv_small_kernel<1, 3><<<grid, 128, 0, st>>>(a);
  else if (ksize == 1 && Cin == 64) hg::conv_small_kernel<1, 64><<<grid, 128, 0, st>>>(a);
  else return -1;      // not a compiled shape: the caller falls back to the tensor-core kernel
  return hg::check_launch("hg_conv2d (small contraction)");
}
