// Importance sampling of the hierarchical renderer (hierarchical_sample=True).
//
// Replaces (reference file:line):
//   the coarse vr.ray_integration of the weights   lib/generators/map3d_generator.py:450-453
//                                                  (lib/generators/volume_rendering.py:12-38)
//   vr.sample_pdf                                  volume_rendering.py:261-303, called at map3d_generator.py:455-461
//   fine points = origin + direction * fine z      map3d_generator.py:463-465 (origins / directions: :150-170)
//   torch.sort + gather of cat([fine, coarse])     map3d_generator.py:500-505
//
// Gradients never flow through the fine depths (the reference computes them under no_grad and detaches them), so the
// hierarchical render is an ordinary render over 2S samples per ray whose point records come from hg_merge_samples.
//
// Both kernels run one warp per ray.  The scans (transmittance, pdf normaliser, cdf) are sequential per lane over at
// most 64 samples and accumulate in double, as torch's CPU cumprod / cumsum do, so the cdf knots are the oracle's to
// fp32 rounding.
#include "common.cuh"

namespace hg {

constexpr int kSampleMaxS = 64;   // 2S <= 128: the merged render runs on hg_render_mlp at 2S samples per ray
constexpr int kSampleWarps = 4;
constexpr int kRecStride = 36;    // point record of hg_geo_features (geo.cu)

struct SampleArgs {
  const float* sigma;     // [B*R*S] raw sigma (before noise), element stride sigma_stride
  int sigma_stride;
  const float* z_vals;    // [B,R*S] jittered coarse depths
  const float* noise;     // [B,R*S] N(0,1) draws or null
  const float* u_pdf;     // [B*R,S] uniform draws of sample_pdf
  float noise_std;
  int clamp_softplus;
  const float* xs;        // [Rw]
  const float* ys;        // [Rh]
  const float* focals;    // [B]
  const float* cam2world; // [B,4,4]
  int B, Rw, Rh, S;
  float* fine_z;          // [B,R*S]
  float* fine_points;     // [B,R*S,3]
};

__global__ void __launch_bounds__(kSampleWarps * 32) sample_fine_kernel(SampleArgs a) {
  __shared__ float s_tr[kSampleWarps][kSampleMaxS];
  __shared__ float s_wt[kSampleWarps][kSampleMaxS];
  __shared__ float s_cdf[kSampleWarps][kSampleMaxS];
  __shared__ float s_bin[kSampleWarps][kSampleMaxS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int R = a.Rw * a.Rh, S = a.S;
  const long ray = static_cast<long>(blockIdx.x) * kSampleWarps + warp;
  if (ray >= static_cast<long>(a.B) * R) return;
  const long base = ray * S;
  float* tr = s_tr[warp];
  float* wt = s_wt[warp];
  float* cdf = s_cdf[warp];
  float* bin = s_bin[warp];

  // coarse weights, ray_integration with white_back / last_back off (volume_rendering.py:19-35)
  float alpha[kSampleMaxS / 32];
#pragma unroll
  for (int k = 0; k < kSampleMaxS / 32; ++k) {
    const int s = lane + 32 * k;
    alpha[k] = 0.f;
    if (s < S) {
      const float z0 = a.z_vals[base + s];
      const float delta = s == S - 1 ? 1e9f : __fsub_rn(a.z_vals[base + s + 1], z0);
      float pre = a.sigma[(base + s) * a.sigma_stride];
      if (a.noise) pre = __fadd_rn(pre, __fmul_rn(a.noise[base + s], a.noise_std));
      const float dens = a.clamp_softplus ? (pre > 20.f ? pre : log1pf(expf(pre))) : fmaxf(pre, 0.f);
      alpha[k] = 1.f - expf(-__fmul_rn(delta, dens));
      tr[s] = __fadd_rn(1.f - alpha[k], 1e-12f);
      if (s < S - 1) bin[s] = 0.5f * __fadd_rn(z0, a.z_vals[base + s + 1]);   // z_vals_mid (map3d_generator.py:457)
    }
  }
  __syncwarp();
  // weights + 1e-5 (map3d_generator.py:454), [:, 1:-1] + eps (volume_rendering.py:280): wt[i] for coarse sample i + 1
#pragma unroll
  for (int k = 0; k < kSampleMaxS / 32; ++k) {
    const int s = lane + 32 * k;
    if (s >= 1 && s <= S - 2) {
      double T = 1.0;
      for (int i = 0; i < s; ++i) T *= static_cast<double>(tr[i]);
      const float w = __fmul_rn(alpha[k], static_cast<float>(T));
      wt[s - 1] = __fadd_rn(__fadd_rn(w, 1e-5f), 1e-5f);
    }
  }
  __syncwarp();
  // pdf and cdf = [0, cumsum(pdf)] (volume_rendering.py:281-283): S - 1 knots
  const int nw = S - 2;
  double total = 0.0;
  for (int i = 0; i < nw; ++i) total += static_cast<double>(wt[i]);
  const float tot = static_cast<float>(total);
#pragma unroll
  for (int k = 0; k < kSampleMaxS / 32; ++k) {
    const int c = lane + 32 * k;
    if (c < S - 1) {
      double acc = 0.0;
      for (int i = 0; i < c; ++i) acc += static_cast<double>(__fdiv_rn(wt[i], tot));
      cdf[c] = static_cast<float>(acc);
    }
  }
  __syncwarp();

  // the ray: direction normalize(x, y, focal) in camera space, rotated by cam2world; origin = cam2world . (0,0,0,1)
  const int b = static_cast<int>(ray / R), r = static_cast<int>(ray % R);
  const float* m = a.cam2world + static_cast<long>(b) * 16;
  const float vx = a.xs[r % a.Rw], vy = a.ys[r / a.Rw], vz = a.focals[b];
  const float nrm = sqrtf(vx * vx + vy * vy + vz * vz) + 1e-12f;
  const float dx = vx / nrm, dy = vy / nrm, dz = vz / nrm;
  const float wx = m[0] * dx + m[1] * dy + m[2] * dz;
  const float wy = m[4] * dx + m[5] * dy + m[6] * dz;
  const float wz = m[8] * dx + m[9] * dy + m[10] * dz;

  // inverse cdf (volume_rendering.py:290-303): searchsorted (left), clamped bin, denom < eps -> 1
#pragma unroll
  for (int k = 0; k < kSampleMaxS / 32; ++k) {
    const int j = lane + 32 * k;
    if (j >= S) continue;
    const float u = a.u_pdf[base + j];
    int lo = 0, hi = S - 1;                      // first knot >= u in [0, S-1); S-1 when none
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (cdf[mid] < u) lo = mid + 1; else hi = mid;
    }
    const int below = lo - 1 > 0 ? lo - 1 : 0;
    const int above = lo < nw ? lo : nw;
    const float c0 = cdf[below];
    float denom = __fsub_rn(cdf[above], c0);
    if (denom < 1e-5f) denom = 1.f;
    const float t = __fdiv_rn(__fsub_rn(u, c0), denom);
    const float z = __fadd_rn(bin[below], __fmul_rn(t, __fsub_rn(bin[above], bin[below])));
    a.fine_z[base + j] = z;
    float* p = a.fine_points + (base + j) * 3;
    p[0] = __fadd_rn(m[3], __fmul_rn(wx, z));
    p[1] = __fadd_rn(m[7], __fmul_rn(wy, z));
    p[2] = __fadd_rn(m[11], __fmul_rn(wz, z));
  }
}

// Stable ascending sort of each ray's 2S depths in cat([fine, coarse]) order -- on equal depths the fine sample first --
// by rank counting, then a gather of the point records.
__global__ void __launch_bounds__(kSampleWarps * 32) merge_samples_kernel(
    const float4* __restrict__ fine_rec, const float* __restrict__ fine_z, const float4* __restrict__ coarse_rec,
    const float* __restrict__ coarse_z, long rays, int S, float4* __restrict__ rec_out, float* __restrict__ z_out,
    int* __restrict__ perm_out) {
  __shared__ float s_z[kSampleWarps][2 * kSampleMaxS];
  __shared__ int s_src[kSampleWarps][2 * kSampleMaxS];
  constexpr int kQ = kRecStride / 4;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long ray = static_cast<long>(blockIdx.x) * kSampleWarps + warp;
  if (ray >= rays) return;
  const int n = 2 * S;
  float* zs = s_z[warp];
  int* src = s_src[warp];
  for (int e = lane; e < n; e += 32) zs[e] = e < S ? fine_z[ray * S + e] : coarse_z[ray * S + e - S];
  __syncwarp();
  // rank in the total order of torch.sort: every number before NaN, equal keys (NaN with NaN included) by position.
  // The ranks are then a permutation of [0, n) for any input, so every slot of src is written exactly once.
  for (int e = lane; e < n; e += 32) {
    const float v = zs[e];
    const bool vnan = isnan(v);
    int rank = 0;
    for (int k = 0; k < n; ++k) {
      const float w = zs[k];
      const bool wnan = isnan(w);
      const bool less = vnan ? !wnan : (w < v);
      const bool same = vnan ? wnan : (w == v);
      rank += less || (same && k < e);
    }
    src[rank] = e;
  }
  __syncwarp();
  const long out0 = ray * n;
  for (int o = lane; o < n; o += 32) {
    const int e = src[o];
    z_out[out0 + o] = zs[e];
    if (perm_out) perm_out[out0 + o] = e;
  }
  for (int i = lane; i < n * kQ; i += 32) {
    const int o = i / kQ, q = i - o * kQ;
    const int e = src[o];
    const float4* row = e < S ? fine_rec + (ray * S + e) * kQ : coarse_rec + (ray * S + e - S) * kQ;
    rec_out[(out0 + o) * kQ + q] = row[q];
  }
}

}  // namespace hg

extern "C" {

// See include/hg3d.h for the argument contract.
int hg_sample_fine(const float* sigma, int sigma_stride, const float* z_vals, const float* noise, const float* u_pdf,
                   float noise_std, int clamp_softplus, const float* xs, const float* ys, const float* focals,
                   const float* cam2world, int B, int Rw, int Rh, int S, float* fine_z, float* fine_points, void* stream) {
  HG_REQUIRE(sigma && z_vals && u_pdf && xs && ys && focals && cam2world && fine_z && fine_points,
             "hg_sample_fine: null pointer");
  HG_REQUIRE(B > 0 && Rw > 0 && Rh > 0, "hg_sample_fine: bad shape B=%d Rw=%d Rh=%d", B, Rw, Rh);
  HG_REQUIRE(S >= 3 && S <= hg::kSampleMaxS, "hg_sample_fine: need 3 <= num_steps <= %d (got %d)", hg::kSampleMaxS, S);
  HG_REQUIRE(sigma_stride >= 1, "hg_sample_fine: sigma_stride must be >= 1 (got %d)", sigma_stride);
  HG_REQUIRE(clamp_softplus == 0 || clamp_softplus == 1, "hg_sample_fine: clamp_softplus must be 0 or 1");
  hg::SampleArgs a{sigma, sigma_stride, z_vals, noise, u_pdf, noise_std, clamp_softplus, xs, ys, focals, cam2world,
                   B, Rw, Rh, S, fine_z, fine_points};
  const long rays = static_cast<long>(B) * Rw * Rh;
  const long blocks = (rays + hg::kSampleWarps - 1) / hg::kSampleWarps;
  HG_REQUIRE(blocks <= 0x7fffffffL, "hg_sample_fine: too many rays (%ld)", rays);
  hg::sample_fine_kernel<<<static_cast<unsigned>(blocks), hg::kSampleWarps * 32, 0, static_cast<cudaStream_t>(stream)>>>(a);
  return hg::check_launch("hg_sample_fine");
}

int hg_merge_samples(const float* fine_rec, const float* fine_z, const float* coarse_rec, const float* coarse_z, int B,
                     int R, int S, float* rec_out, float* z_out, int* perm_out, void* stream) {
  HG_REQUIRE(fine_rec && fine_z && coarse_rec && coarse_z && rec_out && z_out, "hg_merge_samples: null pointer");
  HG_REQUIRE(B > 0 && R > 0, "hg_merge_samples: bad shape B=%d R=%d", B, R);
  HG_REQUIRE(S >= 1 && S <= hg::kSampleMaxS, "hg_merge_samples: need 1 <= samples per ray <= %d (got %d)", hg::kSampleMaxS, S);
  HG_REQUIRE(((reinterpret_cast<uintptr_t>(fine_rec) | reinterpret_cast<uintptr_t>(coarse_rec) |
               reinterpret_cast<uintptr_t>(rec_out)) & 15) == 0, "hg_merge_samples: point records must be 16-byte aligned");
  const long rays = static_cast<long>(B) * R;
  const long blocks = (rays + hg::kSampleWarps - 1) / hg::kSampleWarps;
  HG_REQUIRE(blocks <= 0x7fffffffL, "hg_merge_samples: too many rays (%ld)", rays);
  hg::merge_samples_kernel<<<static_cast<unsigned>(blocks), hg::kSampleWarps * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const float4*>(static_cast<const void*>(fine_rec)), fine_z,
      static_cast<const float4*>(static_cast<const void*>(coarse_rec)), coarse_z, rays, S,
      static_cast<float4*>(static_cast<void*>(rec_out)), z_out, perm_out);
  return hg::check_launch("hg_merge_samples");
}

}  // extern "C"
