// Training-mode pieces of the pose-mapping renderer that are not GEMMs (the FiLM-SIREN layers themselves run on the
// blocked 1x1-convolution kernels of csrc/synth.cu / synth_bwd.cu with the sine activation mode):
//   heads     sigma = w_sigma . h4 + b,  rgb_pre = W_rgb . c + b        (COORDCONCATSIREN.forward, modulated.py:62-73)
//   composite volume integration of a ray and its exact gradient        (vr.ray_integration, volume_rendering.py:12-56)
// Layout: points of a sample are p = ray*S + s; per-point activations are tile-blocked [B, T, 256, 128] (T = N/128)
// like every activation of the synthesis network, per-point scalars are planes [B, N] / [B, 3, N].
#include "common.cuh"

namespace hg {

constexpr int kRC = 256;

__device__ __forceinline__ float rt_red(float t) {          // Cody-Waite by 2*pi, as csrc/render.cu `sin_reduced`
  const float y = t * 0.15915494309189535f;
  const float k = (y + 12582912.f) - 12582912.f;
  float r = fmaf(-k, 6.2831854820251465f, t);
  return fmaf(-k, -1.7484555314695172e-07f, r);
}
__device__ __forceinline__ float rt_sin(float t) { return __sinf(rt_red(t)); }

// ---------------------------------------------------------------------------------------------------------
// heads: one block per tile, one thread per point
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) heads_fwd_kernel(const float* __restrict__ out3, const float* __restrict__ linc,
                                                        const float* __restrict__ mod3, const float* __restrict__ w_sigma,
                                                        const float* __restrict__ w_rgb, const float* __restrict__ heads_b,
                                                        float* __restrict__ sig, float* __restrict__ rgbp, int B, int N) {
  __shared__ float sf[kRC], sp[kRC], ws[kRC], wr[3 * kRC];
  const int T = (N + 127) / 128;
  const int tile = blockIdx.x, b = tile / T, ti = tile - b * T;
  for (int i = threadIdx.x; i < kRC; i += 128) {
    sf[i] = mod3[(static_cast<long>(b) * 2 + 0) * kRC + i];
    sp[i] = mod3[(static_cast<long>(b) * 2 + 1) * kRC + i];
    ws[i] = w_sigma[i];
  }
  for (int i = threadIdx.x; i < 3 * kRC; i += 128) wr[i] = w_rgb[i];
  __syncthreads();
  const int p = ti * 128 + threadIdx.x;
  const float* o3 = out3 + static_cast<long>(tile) * kRC * 128 + threadIdx.x;
  const float* lc = linc + static_cast<long>(tile) * kRC * 128 + threadIdx.x;
  float d0 = 0.f, d1 = 0.f, d2 = 0.f, d3 = 0.f;
#pragma unroll 4
  for (int c = 0; c < kRC; ++c) {
    const float h4 = rt_sin(fmaf(sf[c], o3[c * 128], sp[c]));
    const float cc = rt_sin(fmaf(sf[c], lc[c * 128], sp[c]));
    d0 = fmaf(h4, ws[c], d0);
    d1 = fmaf(cc, wr[c], d1);
    d2 = fmaf(cc, wr[kRC + c], d2);
    d3 = fmaf(cc, wr[2 * kRC + c], d3);
  }
  if (p < N) {
    sig[static_cast<long>(b) * N + p] = d0 + heads_b[0];
    rgbp[(static_cast<long>(b) * 3 + 0) * N + p] = d1 + heads_b[1];
    rgbp[(static_cast<long>(b) * 3 + 1) * N + p] = d2 + heads_b[2];
    rgbp[(static_cast<long>(b) * 3 + 2) * N + p] = d3 + heads_b[3];
  }
}

// d w_sigma[c] = sum dsig*h4,  d W_rgb[j,c] = sum drgbp[j]*c,  d b = sums; acc [4,C] + [4] fp64 (accumulated).
// Warp w owns channels w, w+8, ...; a lane owns 4 points of the tile.
__global__ void __launch_bounds__(256) heads_bwd_kernel(const float* __restrict__ out3, const float* __restrict__ linc,
                                                        const float* __restrict__ mod3, const float* __restrict__ dsig,
                                                        const float* __restrict__ drgbp, double* __restrict__ acc, int B,
                                                        int N) {
  __shared__ float s_acc[4 * kRC];
  __shared__ float s_b[4];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < 4 * kRC; i += 256) s_acc[i] = 0.f;
  if (threadIdx.x < 4) s_b[threadIdx.x] = 0.f;
  __syncthreads();
  const int T = (N + 127) / 128;
  float bsum[4] = {0.f, 0.f, 0.f, 0.f};
  for (int tile = blockIdx.x; tile < B * T; tile += gridDim.x) {
    const int b = tile / T, ti = tile - b * T;
    const int p = ti * 128 + lane * 4;
    float4 g[4];
    const bool full = p + 3 < N;
    for (int j = 0; j < 4; ++j) {
      const float* src = (j == 0 ? dsig + static_cast<long>(b) * N : drgbp + (static_cast<long>(b) * 3 + (j - 1)) * N) + p;
      g[j] = full ? *reinterpret_cast<const float4*>(src)
                  : make_float4(p < N ? src[0] : 0.f, p + 1 < N ? src[1] : 0.f, p + 2 < N ? src[2] : 0.f, 0.f);
      if (warp == 0) bsum[j] += (g[j].x + g[j].y) + (g[j].z + g[j].w);
    }
    const long off = static_cast<long>(tile) * kRC * 128 + lane * 4;
#pragma unroll 2
    for (int c = warp; c < kRC; c += 8) {
      const float f = mod3[(static_cast<long>(b) * 2 + 0) * kRC + c], ph = mod3[(static_cast<long>(b) * 2 + 1) * kRC + c];
      const float4 o = __ldcs(reinterpret_cast<const float4*>(out3 + off + c * 128));
      const float4 l = __ldcs(reinterpret_cast<const float4*>(linc + off + c * 128));
      const float4 h4 = make_float4(rt_sin(fmaf(f, o.x, ph)), rt_sin(fmaf(f, o.y, ph)), rt_sin(fmaf(f, o.z, ph)), rt_sin(fmaf(f, o.w, ph)));
      const float4 cc = make_float4(rt_sin(fmaf(f, l.x, ph)), rt_sin(fmaf(f, l.y, ph)), rt_sin(fmaf(f, l.z, ph)), rt_sin(fmaf(f, l.w, ph)));
      float t[4];
      t[0] = (g[0].x * h4.x + g[0].y * h4.y) + (g[0].z * h4.z + g[0].w * h4.w);
#pragma unroll
      for (int j = 1; j < 4; ++j) t[j] = (g[j].x * cc.x + g[j].y * cc.y) + (g[j].z * cc.z + g[j].w * cc.w);
#pragma unroll
      for (int o2 = 16; o2 > 0; o2 >>= 1) {
#pragma unroll
        for (int j = 0; j < 4; ++j) t[j] += __shfl_xor_sync(0xffffffffu, t[j], o2);
      }
      if (lane == 0) {
#pragma unroll
        for (int j = 0; j < 4; ++j) s_acc[j * kRC + c] += t[j];
      }
    }
  }
  if (warp == 0) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float v = bsum[j];
      for (int o2 = 16; o2 > 0; o2 >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o2);
      if (lane == 0) s_b[j] = v;
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 4 * kRC; i += 256) atomicAdd(acc + i, static_cast<double>(s_acc[i]));
  if (threadIdx.x < 4) atomicAdd(acc + 4 * kRC + threadIdx.x, static_cast<double>(s_b[threadIdx.x]));
}

// ---------------------------------------------------------------------------------------------------------
// compositing.  One block per tile of 128 points = 128/S whole rays (S must divide 128).
//   delta_s = z_{s+1} - z_s (1e9 for the last), dens = relu|softplus(sigma + eps*noise_std), alpha = 1 - exp(-delta*dens),
//   T_s = prod_{k<s} (1 - alpha_k + 1e-12), w = alpha*T; out[c] = sum_s w_s v_s[c] (+ 1 - sum w if white_back);
//   v = [feat(256), sigmoid(rgb_pre)(3)]; depth = sum (w_s + [s = S-1](1 - sum w)) z_s.
//   last_back: w_{S-1} += 1 - sum w before the sums (volume_rendering.py:38-41), so with g = d out
//   d v_{S-1} gains (1 - sum w) g and every d w_s gains -<g, v_{S-1}>; the suffix sums of d alpha are unchanged.
// ray_out [B,R,260] = feat | rgb | depth, exactly the layout of the fused forward kernel (csrc/render.cu).
// ---------------------------------------------------------------------------------------------------------
struct CompArgs {
  const float* sig;      // [B,N]
  const float* z;        // [B,N]
  const float* noise;    // [B,N] or null
  const float* rgbp;     // [B,3,N]
  const float* feat;     // [B,T,256,128]
  float* ray_out;        // fwd: [B,R,260]
  float* w_out;          // fwd: [B,N] compositing weights as vr.ray_integration returns them (last_back: absorbed)
  const float* dray;     // bwd: [B,R,260]
  float* dfeat;          // bwd: [B,T,256,128]
  float* drgbp;          // bwd: [B,3,N]
  float* dsig;           // bwd: [B,N]
  int B, R, S;
  float noise_std;
  int white_back, softplus;
  int last_back;         // the last sample of a ray absorbs the remaining transmittance (volume_rendering.py:38-41)
};

__device__ __forceinline__ float comp_alpha(const CompArgs& a, long gp, int s, const float* zs, int row, float& dens_grad) {
  const float delta = (s == a.S - 1) ? 1e9f : zs[row + 1] - zs[row];
  float pre = a.sig[gp];
  if (a.noise) pre += a.noise[gp] * a.noise_std;
  float dens;
  if (a.softplus) {
    dens = pre > 20.f ? pre : log1pf(expf(pre));
    dens_grad = 1.f / (1.f + expf(-pre));
  } else {
    dens = fmaxf(pre, 0.f);
    dens_grad = pre > 0.f ? 1.f : 0.f;
  }
  const float e = expf(-delta * dens);
  dens_grad *= delta * e;                 // d alpha / d sigma
  return 1.f - e;
}

template <bool kBwd>
__global__ void __launch_bounds__(128) composite_kernel(CompArgs a) {
  __shared__ float zs[129], tr[128], wg[128], qs[128], rayw[128], sdr[16 * 260];
  const int N = a.R * a.S, T = N / 128;
  const int tile = blockIdx.x, b = tile / T, ti = tile - b * T;
  const int row = threadIdx.x, warp = row >> 5, lane = row & 31;
  const int S = a.S, rpt = 128 / S;          // rays per tile
  const int rl = row / S, s = row - rl * S;
  const int ray0 = ti * rpt;
  const long gp = static_cast<long>(b) * N + ti * 128 + row;
  zs[row] = a.z[gp];
  if (row == 0) zs[128] = 0.f;
  __syncthreads();
  float dgrad;
  const float alpha = comp_alpha(a, gp, s, zs, row, dgrad);
  tr[row] = 1.f - alpha + 1e-12f;
  __syncthreads();
  float Tr = 1.f;
  for (int k = 0; k < s; ++k) Tr *= tr[rl * S + k];
  const float w = alpha * Tr;
  wg[row] = w;
  __syncthreads();
  if (s == 0) {
    float W = 0.f;
    for (int k = 0; k < S; ++k) W += wg[rl * S + k];
    rayw[rl] = W;
  }
  __syncthreads();
  const float back = a.white_back ? 1.f : 0.f;
  const float* ft = a.feat + static_cast<long>(tile) * kRC * 128;

  if (!kBwd) {
    a.w_out[gp] = (a.last_back && s == S - 1) ? w + (1.f - rayw[rl]) : w;    // as csrc/render.cu's weights_out
    // weighted sums: warp w handles channels w, w+4, ...; lane l holds points l, l+32, l+64, l+96
    for (int c = warp; c < kRC + 4; c += 4) {
      auto value = [&](int p) {
        if (c < kRC) return ft[c * 128 + p];
        if (c < kRC + 3) return 1.f / (1.f + expf(-a.rgbp[(static_cast<long>(b) * 3 + (c - kRC)) * N + ti * 128 + p]));
        return zs[p];                                 // depth
      };
      float part[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int p = lane + 32 * i;
        part[i] = wg[p] * value(p);
      }
      if (S >= 32) {
        // every 32-point group lies inside one ray: full warp reduction, then add the groups of a ray
#pragma unroll
        for (int i = 0; i < 4; ++i)
          for (int o = 16; o > 0; o >>= 1) part[i] += __shfl_xor_sync(0xffffffffu, part[i], o);
        if (lane == 0) {
          const int gpr = S / 32;                     // groups per ray
          for (int r = 0; r < rpt; ++r) {
            float v = 0.f;
            for (int i = 0; i < gpr; ++i) v += part[r * gpr + i];
            float* ro = a.ray_out + (static_cast<long>(b) * a.R + ray0 + r) * 260;
            if (a.last_back && c < kRC + 3) v += (1.f - rayw[r]) * value(r * S + S - 1);
            if (c < kRC + 3) ro[c] = v + back * (1.f - rayw[r]);
            else ro[259] = v + (1.f - rayw[r]) * zs[r * S + S - 1];
          }
        }
      } else {
        // S < 32: segments of S lanes
#pragma unroll
        for (int i = 0; i < 4; ++i)
          for (int o = S >> 1; o > 0; o >>= 1) part[i] += __shfl_xor_sync(0xffffffffu, part[i], o);
        if ((lane & (S - 1)) == 0) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int r = (lane + 32 * i) / S;
            float* ro = a.ray_out + (static_cast<long>(b) * a.R + ray0 + r) * 260;
            if (a.last_back && c < kRC + 3) part[i] += (1.f - rayw[r]) * value(r * S + S - 1);
            if (c < kRC + 3) ro[c] = part[i] + back * (1.f - rayw[r]);
            else ro[259] = part[i] + (1.f - rayw[r]) * zs[r * S + S - 1];
          }
        }
      }
    }
  } else {
    // ---- backward: d ray_out of this tile's rays -> shared
    for (int i = row; i < rpt * 260; i += 128) sdr[i] = a.dray[(static_cast<long>(b) * a.R + ray0) * 260 + i];
    __syncthreads();
    const float* dr = sdr + rl * 260;
    // q = d out / d w_s = <dout, v_s - back (- v_{S-1} with last_back)> over the 259 composited channels
    const int last = rl * S + S - 1;
    const float lb = a.last_back ? 1.f : 0.f;
    float q = 0.f;
#pragma unroll 4
    for (int c = 0; c < kRC; ++c) q = fmaf(dr[c], ft[c * 128 + row] - back - lb * ft[c * 128 + last], q);
    float sgm[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const float* rp = a.rgbp + (static_cast<long>(b) * 3 + j) * N + ti * 128;
      sgm[j] = 1.f / (1.f + expf(-rp[row]));
      const float vl = a.last_back ? 1.f / (1.f + expf(-rp[last])) : 0.f;
      q = fmaf(dr[kRC + j], sgm[j] - back - vl, q);
    }
    qs[row] = q * w;
    __syncthreads();
    float suffix = 0.f;
    for (int k = s + 1; k < S; ++k) suffix += qs[rl * S + k];
    const float dalpha = q * Tr - suffix / tr[row];
    a.dsig[gp] = dalpha * dgrad;
    const float wv = (a.last_back && s == S - 1) ? w + (1.f - rayw[rl]) : w;      // d out / d v_s
#pragma unroll
    for (int j = 0; j < 3; ++j) a.drgbp[(static_cast<long>(b) * 3 + j) * N + ti * 128 + row] = wv * dr[kRC + j] * sgm[j] * (1.f - sgm[j]);
    float* df = a.dfeat + static_cast<long>(tile) * kRC * 128 + row;
#pragma unroll 4
    for (int c = 0; c < kRC; ++c) df[c * 128] = wv * dr[c];
  }
}

}  // namespace hg

extern "C" {

int hg_render_heads(const float* out3, const float* linc, const float* mod3, const float* w_sigma, const float* w_rgb,
                    const float* heads_b, float* sig, float* rgbp, int B, int N, void* stream) {
  HG_REQUIRE(out3 && linc && mod3 && w_sigma && w_rgb && heads_b && sig && rgbp, "hg_render_heads: null pointer");
  HG_REQUIRE(B > 0 && N > 0 && N % 128 == 0, "hg_render_heads: points per sample must be a positive multiple of 128 (got %d)", N);
  hg::heads_fwd_kernel<<<B * (N / 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(out3, linc, mod3, w_sigma, w_rgb, heads_b,
                                                                                   sig, rgbp, B, N);
  return hg::check_launch("hg_render_heads");
}

int hg_render_heads_bwd(const float* out3, const float* linc, const float* mod3, const float* dsig, const float* drgbp,
                        double* acc, int B, int N, void* stream) {
  HG_REQUIRE(out3 && linc && mod3 && dsig && drgbp && acc, "hg_render_heads_bwd: null pointer");
  HG_REQUIRE(B > 0 && N > 0 && N % 128 == 0, "hg_render_heads_bwd: points per sample must be a positive multiple of 128");
  int grid = hg::num_sms() * 4;
  if (grid > B * (N / 128)) grid = B * (N / 128);
  hg::heads_bwd_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(out3, linc, mod3, dsig, drgbp, acc, B, N);
  return hg::check_launch("hg_render_heads_bwd");
}

static int comp_check(int B, int R, int S, const char* who) {
  HG_REQUIRE(B > 0 && R > 0 && S > 0, "%s: bad shape", who);
  HG_REQUIRE(128 % S == 0 && S >= 8 && (R * S) % 128 == 0,
             "%s: the training compositing kernel needs samples/ray in {8,16,32,64,128} and rays*samples a multiple of 128 "
             "(got R=%d S=%d)", who, R, S);
  return 0;
}

int hg_render_composite(const float* sig, const float* z, const float* noise, const float* rgbp, const float* feat,
                        float* ray_out, float* weights, int B, int R, int S, float noise_std, int white_back,
                        int clamp_softplus, int last_back, void* stream) {
  HG_REQUIRE(sig && z && rgbp && feat && ray_out && weights, "hg_render_composite: null pointer");
  if (int rc = comp_check(B, R, S, "hg_render_composite")) return rc;
  hg::CompArgs a{};
  a.sig = sig; a.z = z; a.noise = noise; a.rgbp = rgbp; a.feat = feat; a.ray_out = ray_out; a.w_out = weights;
  a.B = B; a.R = R; a.S = S; a.noise_std = noise_std; a.white_back = white_back; a.softplus = clamp_softplus;
  a.last_back = last_back;
  hg::composite_kernel<false><<<B * (R * S / 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(a);
  return hg::check_launch("hg_render_composite");
}

int hg_render_composite_bwd(const float* sig, const float* z, const float* noise, const float* rgbp, const float* feat,
                            const float* dray, float* dfeat, float* drgbp, float* dsig, int B, int R, int S,
                            float noise_std, int white_back, int clamp_softplus, int last_back, void* stream) {
  HG_REQUIRE(sig && z && rgbp && feat && dray && dfeat && drgbp && dsig, "hg_render_composite_bwd: null pointer");
  if (int rc = comp_check(B, R, S, "hg_render_composite_bwd")) return rc;
  hg::CompArgs a{};
  a.sig = sig; a.z = z; a.noise = noise; a.rgbp = rgbp; a.feat = feat; a.dray = dray; a.dfeat = dfeat; a.drgbp = drgbp;
  a.dsig = dsig;
  a.B = B; a.R = R; a.S = S; a.noise_std = noise_std; a.white_back = white_back; a.softplus = clamp_softplus;
  a.last_back = last_back;
  hg::composite_kernel<true><<<B * (R * S / 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(a);
  return hg::check_launch("hg_render_composite_bwd");
}

}  // extern "C"
