// Everything of the VGG16 perceptual loss (lib/components/perceptual_loss.py) that is not a convolution or a ReLU; those run on
// hg_conv2d (fp32x3) and hg_bias_act / hg_bias_act_grad.
//
//   hg_vgg_input          1 -> 3 channel repeat, (x - mean) / std and the bilinear resize to Ho x Wo (align_corners=False, no
//                         antialias: torch's upsample_bilinear2d arithmetic) in one pass.  Ho x Wo == H x W is no resize.
//   hg_vgg_input_adjoint  its transpose as a gather: every input pixel sums the output pixels whose bilinear footprint covers it,
//                         in a fixed order and without atomics, so the gradient repeats bit for bit.
//   hg_maxpool2x2         MaxPool2d(2, 2) with torch's floor semantics (a ragged last row / column is dropped).
//   hg_vgg_level_bwd      the backward at the end of a block l:  d pre_l = [y_l > 0] * (unpool(d pooled_{l+1}) +
//                         g_l / n_l * clamp(y_l - t_l, -1, 1)), the argmax of every window recomputed from the saved y_l.
//   hg_smooth_l1          mean over n elements of smooth_l1(a - b), beta = 1: fp64 block partials summed in a fixed order.
// Everything is HBM-bound streaming.
#include "common.cuh"

namespace hg {

// area_pixel_compute_source_index (align_corners=False) and the two taps of upsample_bilinear2d, in its float arithmetic
__device__ __forceinline__ void bilinear_taps(int dst, float scale, int in, int& i0, int& i1, float& l1) {
  float src = scale * (static_cast<float>(dst) + 0.5f) - 0.5f;
  if (src < 0.f) src = 0.f;
  i0 = static_cast<int>(src);
  if (i0 > in - 1) i0 = in - 1;
  i1 = i0 < in - 1 ? i0 + 1 : i0;
  l1 = src - static_cast<float>(i0);
}

__global__ void __launch_bounds__(256) vgg_input_kernel(const float* __restrict__ x, int C, int H, int W,
                                                        const float* __restrict__ mean, const float* __restrict__ stdv,
                                                        float* __restrict__ out, int Ho, int Wo, long total) {
  const bool resize = Ho != H || Wo != W;
  const float sy = static_cast<float>(H) / static_cast<float>(Ho), sx = static_cast<float>(W) / static_cast<float>(Wo);
  for (long e = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total; e += static_cast<long>(gridDim.x) * blockDim.x) {
    const int ox = static_cast<int>(e % Wo);
    const int oy = static_cast<int>((e / Wo) % Ho);
    const int c = static_cast<int>((e / (static_cast<long>(Wo) * Ho)) % 3);
    const long b = e / (3L * Ho * Wo);
    const float* plane = x + (b * C + (C == 1 ? 0 : c)) * static_cast<long>(H) * W;
    const float m = __ldg(mean + c), s = __ldg(stdv + c);
    if (!resize) {
      out[e] = (__ldg(plane + static_cast<long>(oy) * W + ox) - m) / s;
      continue;
    }
    int y0, y1, x0, x1;
    float ly, lx;
    bilinear_taps(oy, sy, H, y0, y1, ly);
    bilinear_taps(ox, sx, W, x0, x1, lx);
    const float n00 = (__ldg(plane + static_cast<long>(y0) * W + x0) - m) / s;
    const float n01 = (__ldg(plane + static_cast<long>(y0) * W + x1) - m) / s;
    const float n10 = (__ldg(plane + static_cast<long>(y1) * W + x0) - m) / s;
    const float n11 = (__ldg(plane + static_cast<long>(y1) * W + x1) - m) / s;
    out[e] = (1.f - ly) * ((1.f - lx) * n00 + lx * n01) + ly * ((1.f - lx) * n10 + lx * n11);
  }
}

// weight of input index `i` in output `o` (both taps, which coincide on the clamped last row)
__device__ __forceinline__ float bilinear_weight(int o, float scale, int in, int i) {
  int i0, i1;
  float l1;
  bilinear_taps(o, scale, in, i0, i1, l1);
  return (i0 == i ? 1.f - l1 : 0.f) + (i1 == i ? l1 : 0.f);
}

// output rows that may read input row i: src(o) = scale (o + 0.5) - 0.5 lies in [i - 1, i + 1); one row of slack each side
__device__ __forceinline__ void footprint(int i, float scale, int out, int& lo, int& hi) {
  lo = static_cast<int>(floorf((static_cast<float>(i) - 0.5f) / scale - 0.5f)) - 1;
  hi = static_cast<int>(ceilf((static_cast<float>(i) + 1.5f) / scale - 0.5f)) + 1;
  if (lo < 0) lo = 0;
  if (hi > out - 1) hi = out - 1;
}

__global__ void __launch_bounds__(256) vgg_input_adjoint_kernel(const float* __restrict__ dout, int Ho, int Wo,
                                                                const float* __restrict__ stdv, float* __restrict__ dx, int C,
                                                                int H, int W, long total) {
  const bool resize = Ho != H || Wo != W;
  const float sy = static_cast<float>(H) / static_cast<float>(Ho), sx = static_cast<float>(W) / static_cast<float>(Wo);
  for (long e = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total; e += static_cast<long>(gridDim.x) * blockDim.x) {
    const int ix = static_cast<int>(e % W);
    const int iy = static_cast<int>((e / W) % H);
    const int ci = static_cast<int>((e / (static_cast<long>(W) * H)) % C);
    const long b = e / (static_cast<long>(C) * H * W);
    int ylo = iy, yhi = iy, xlo = ix, xhi = ix;
    if (resize) {
      footprint(iy, sy, Ho, ylo, yhi);
      footprint(ix, sx, Wo, xlo, xhi);
    }
    float acc = 0.f;
    for (int c = (C == 1 ? 0 : ci); c <= (C == 1 ? 2 : ci); ++c) {       // a 1-channel input feeds all three
      const float* plane = dout + (b * 3 + c) * static_cast<long>(Ho) * Wo;
      float sum = 0.f;
      for (int oy = ylo; oy <= yhi; ++oy) {
        const float wy = resize ? bilinear_weight(oy, sy, H, iy) : 1.f;
        if (wy == 0.f) continue;
        float row = 0.f;
        for (int ox = xlo; ox <= xhi; ++ox) {
          const float wx = resize ? bilinear_weight(ox, sx, W, ix) : 1.f;
          if (wx != 0.f) row = fmaf(wx, __ldg(plane + static_cast<long>(oy) * Wo + ox), row);
        }
        sum = fmaf(wy, row, sum);
      }
      acc += sum / __ldg(stdv + c);
    }
    dx[e] = acc;
  }
}

__global__ void __launch_bounds__(256) maxpool2x2_kernel(const float* __restrict__ x, float* __restrict__ y, int H, int W, long total) {
  const int Ho = H / 2, Wo = W / 2;
  for (long e = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total; e += static_cast<long>(gridDim.x) * blockDim.x) {
    const int ox = static_cast<int>(e % Wo);
    const int oy = static_cast<int>((e / Wo) % Ho);
    const float* p = x + (e / (static_cast<long>(Wo) * Ho)) * H * W + static_cast<long>(2 * oy) * W + 2 * ox;
    float m = __ldg(p);
    const float v[3] = {__ldg(p + 1), __ldg(p + W), __ldg(p + W + 1)};
    for (int i = 0; i < 3; ++i)
      if (v[i] > m || isnan(v[i])) m = v[i];          // torch's rule: the first maximum, NaN propagates
    y[e] = m;
  }
}

// d pre_l at one element of the block output y_l [planes,H,W].  The gradient of a window of the following max-pool goes to its
// first maximum in row-major order (strict '>'), recomputed from y_l.  y_l is a ReLU output, so two equal entries of a window are
// (but for a measure-zero coincidence) zeros, and a window that ties is all zero: the ReLU mask [y_l > 0] zeroes every element
// of it whichever one the rule picks, so the tie rule never shows in the gradient.
__global__ void __launch_bounds__(256) vgg_level_bwd_kernel(const float* __restrict__ y, const float* __restrict__ t,
                                                            const float* __restrict__ dpool, const float* __restrict__ gscale,
                                                            float inv_n, float* __restrict__ dpre, int H, int W, long total) {
  const int Ho = H / 2, Wo = W / 2;
  const float lam = (t && gscale) ? __ldg(gscale) * inv_n : 0.f;
  for (long e = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total; e += static_cast<long>(gridDim.x) * blockDim.x) {
    const float v = __ldg(y + e);
    float g = 0.f;
    if (v > 0.f) {
      const int w = static_cast<int>(e % W);
      const int h = static_cast<int>((e / W) % H);
      const long plane = e / (static_cast<long>(W) * H);
      const int ph = h >> 1, pw = w >> 1;
      if (dpool && ph < Ho && pw < Wo) {
        const float* p = y + plane * H * W + static_cast<long>(2 * ph) * W + 2 * pw;
        int arg = 0;
        float m = __ldg(p);
        const float c[3] = {__ldg(p + 1), __ldg(p + W), __ldg(p + W + 1)};
        for (int i = 0; i < 3; ++i)
          if (c[i] > m) { m = c[i]; arg = i + 1; }
        if (arg == (h & 1) * 2 + (w & 1)) g = __ldg(dpool + (plane * Ho + ph) * Wo + pw);
      }
      if (t) g += lam * fminf(fmaxf(v - __ldg(t + e), -1.f), 1.f);
    }
    dpre[e] = g;
  }
}

__global__ void __launch_bounds__(256) smooth_l1_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                        double* __restrict__ partials, long n) {
  __shared__ double red[8];
  double acc = 0.0;
  for (long e = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; e < n; e += static_cast<long>(gridDim.x) * blockDim.x) {
    const float d = __ldg(a + e) - __ldg(b + e);
    const float ad = fabsf(d);
    acc += static_cast<double>(ad < 1.f ? 0.5f * d * d : ad - 0.5f);
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < 8; ++i) s += red[i];
    partials[blockIdx.x] = s;
  }
}

__global__ void smooth_l1_reduce_kernel(const double* __restrict__ partials, int n, double scale, float* __restrict__ out) {
  double s = 0.0;                                   // single thread, fixed order
  for (int i = 0; i < n; ++i) s += partials[i];
  out[0] = static_cast<float>(s * scale);
}

inline unsigned stream_blocks(long total, int per_sm) {
  long blocks = (total + 255) / 256;
  const long cap = static_cast<long>(num_sms()) * per_sm;
  return static_cast<unsigned>(blocks < cap ? blocks : cap);
}

}  // namespace hg

extern "C" {

int hg_vgg_input(const float* x, int C, int B, int H, int W, const float* mean, const float* stdv, float* out, int Ho, int Wo,
                 void* stream) {
  HG_REQUIRE(x && mean && stdv && out, "hg_vgg_input: null pointer");
  HG_REQUIRE(C == 1 || C == 3, "hg_vgg_input: 1 or 3 input channels (got %d)", C);
  HG_REQUIRE(B > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0, "hg_vgg_input: bad shape");
  const long total = static_cast<long>(B) * 3 * Ho * Wo;
  hg::vgg_input_kernel<<<hg::stream_blocks(total, 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, C, H, W, mean, stdv, out,
                                                                                                     Ho, Wo, total);
  return hg::check_launch("hg_vgg_input");
}

int hg_vgg_input_adjoint(const float* dout, int B, int Ho, int Wo, const float* stdv, float* dx, int C, int H, int W, void* stream) {
  HG_REQUIRE(dout && stdv && dx, "hg_vgg_input_adjoint: null pointer");
  HG_REQUIRE(C == 1 || C == 3, "hg_vgg_input_adjoint: 1 or 3 input channels (got %d)", C);
  HG_REQUIRE(B > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0, "hg_vgg_input_adjoint: bad shape");
  const long total = static_cast<long>(B) * C * H * W;
  hg::vgg_input_adjoint_kernel<<<hg::stream_blocks(total, 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(dout, Ho, Wo, stdv, dx,
                                                                                                             C, H, W, total);
  return hg::check_launch("hg_vgg_input_adjoint");
}

int hg_maxpool2x2(const float* x, float* y, long planes, int H, int W, void* stream) {
  HG_REQUIRE(x && y, "hg_maxpool2x2: null pointer");
  HG_REQUIRE(planes > 0 && H >= 2 && W >= 2, "hg_maxpool2x2: bad shape (H and W must be >= 2)");
  const long total = planes * (H / 2) * (W / 2);
  hg::maxpool2x2_kernel<<<hg::stream_blocks(total, 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, y, H, W, total);
  return hg::check_launch("hg_maxpool2x2");
}

int hg_vgg_level_bwd(const float* y, const float* t, const float* dpool, const float* gscale, float inv_n, float* dpre, long planes,
                     int H, int W, void* stream) {
  HG_REQUIRE(y && dpre, "hg_vgg_level_bwd: null pointer");
  HG_REQUIRE((t == nullptr) == (gscale == nullptr), "hg_vgg_level_bwd: the target and the loss's incoming gradient go together");
  HG_REQUIRE(planes > 0 && H > 0 && W > 0 && (!dpool || (H >= 2 && W >= 2)), "hg_vgg_level_bwd: bad shape");
  const long total = planes * H * W;
  hg::vgg_level_bwd_kernel<<<hg::stream_blocks(total, 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(y, t, dpool, gscale, inv_n,
                                                                                                         dpre, H, W, total);
  return hg::check_launch("hg_vgg_level_bwd");
}

int hg_smooth_l1(const float* a, const float* b, long n, float* loss, double* workspace, void* stream) {
  HG_REQUIRE(a && b && loss && workspace, "hg_smooth_l1: null pointer");
  HG_REQUIRE(n > 0, "hg_smooth_l1: empty input");
  auto st = static_cast<cudaStream_t>(stream);
  const unsigned blocks = hg::stream_blocks(n, 2);
  hg::smooth_l1_kernel<<<blocks, 256, 0, st>>>(a, b, workspace, n);
  int rc = hg::check_launch("hg_smooth_l1");
  if (rc) return rc;
  hg::smooth_l1_reduce_kernel<<<1, 1, 0, st>>>(workspace, static_cast<int>(blocks), 1.0 / static_cast<double>(n), loss);
  return hg::check_launch("hg_smooth_l1(reduce)");
}

}  // extern "C"
