// Conditional (reconstruction) phases of the reference's trainer (lib/trainers/phase_trainer.py:344-553):
//
//   hg_latent_pool_gather / hg_latent_pool_grad   `LatentPool.forward` = `latents[indices]` (lib/components/util.py:18-29) and
//        the dense [P,L] gradient of the pool parameter that autograd's index backward produces.  No atomics: each touched row
//        is summed (fp64, batch order) by the one block that owns the row's first occurrence, so repeated indices sum the same
//        way on every run.
//   hg_latent_loss   mean SL1_beta(n(pred) - n(target)) with n = normalize_2nd_moment (lib/components/util.py:58), the latent
//        regression of phase_trainer.py:425-437 and :493-506, and d loss / d pred through the normalisation's Jacobian.
#include "common.cuh"

namespace hg {

__global__ void __launch_bounds__(128) latent_pool_gather_kernel(const float* __restrict__ pool, long P, int L,
                                                                 const long* __restrict__ idx, float* __restrict__ out) {
  const long i = idx[blockIdx.x];
  float* dst = out + static_cast<long>(blockIdx.x) * L;
  const bool ok = i >= 0 && i < P;
  for (int j = threadIdx.x; j < L; j += blockDim.x) dst[j] = ok ? pool[i * L + j] : __int_as_float(0x7fc00000);
}

__global__ void __launch_bounds__(128) latent_pool_grad_kernel(const float* __restrict__ dz, const long* __restrict__ idx, int B,
                                                               int L, long P, float* __restrict__ dpool) {
  const int b = blockIdx.x;
  const long i = idx[b];
  if (i < 0 || i >= P) return;
  int seen = 0;
  for (int k = threadIdx.x; k < b; k += blockDim.x) seen |= idx[k] == i;
  if (__syncthreads_or(seen)) return;             // an earlier block owns this row
  for (int j = threadIdx.x; j < L; j += blockDim.x) {
    double acc = 0.0;
    for (int k = b; k < B; ++k)
      if (idx[k] == i) acc += static_cast<double>(dz[static_cast<long>(k) * L + j]);
    dpool[i * L + j] = static_cast<float>(acc);
  }
}

__device__ __forceinline__ double warp_sum(double v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One block of 32 warps; warp w owns rows w, w + 32, ...  Per row: the two second moments, then the loss terms and
// dot = sum_j g_j n(p)_j, then (optionally) d loss / d p_k = s * r_p * (g_k - n(p)_k * dot / L).
constexpr int kLatentWarps = 32;
__global__ void __launch_bounds__(kLatentWarps * 32) latent_loss_kernel(const float* __restrict__ pred, const float* __restrict__ target,
                                                                        int B, int L, float beta, const float* __restrict__ gscale,
                                                                        float* __restrict__ dpred, float* __restrict__ loss) {
  __shared__ double red[kLatentWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float inv_n = 1.f / (static_cast<float>(B) * static_cast<float>(L));
  const float s = (gscale ? gscale[0] : 1.f) * inv_n;
  double acc = 0.0;
  for (int b = warp; b < B; b += kLatentWarps) {
    const float* p = pred + static_cast<long>(b) * L;
    const float* t = target + static_cast<long>(b) * L;
    double sp = 0.0, st = 0.0;
    for (int j = lane; j < L; j += 32) {
      sp += static_cast<double>(p[j]) * p[j];
      st += static_cast<double>(t[j]) * t[j];
    }
    sp = warp_sum(sp);
    st = warp_sum(st);
    const float rp = static_cast<float>(1.0 / sqrt(sp / L + 1e-8));
    const float rt = static_cast<float>(1.0 / sqrt(st / L + 1e-8));
    double row = 0.0, dot = 0.0;
    for (int j = lane; j < L; j += 32) {
      const float np = p[j] * rp;
      const float d = np - t[j] * rt;
      const float z = fabsf(d);
      float rho, g;
      if (z < beta) {
        rho = 0.5f * z * z / beta;
        g = d / beta;
      } else {
        rho = z - 0.5f * beta;
        g = d > 0.f ? 1.f : -1.f;
      }
      row += static_cast<double>(rho);
      dot += static_cast<double>(g) * np;
    }
    acc += warp_sum(row);
    if (dpred) {
      const float c = static_cast<float>(warp_sum(dot) / L);
      for (int j = lane; j < L; j += 32) {
        const float np = p[j] * rp;
        const float d = np - t[j] * rt;
        const float g = fabsf(d) < beta ? d / beta : (d > 0.f ? 1.f : -1.f);
        dpred[static_cast<long>(b) * L + j] = s * rp * (g - np * c);
      }
    }
  }
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0 && loss) {
    double tot = 0.0;
    for (int w = 0; w < kLatentWarps; ++w) tot += red[w];
    loss[0] = static_cast<float>(tot / (static_cast<double>(B) * L));
  }
}

}  // namespace hg

extern "C" {

// out[b,:] = pool[idx[b],:]; a row whose index lies outside [0, P) is written as NaN (torch's indexing would assert).
int hg_latent_pool_gather(const float* pool, long P, int L, const long* idx, int B, float* out, void* stream) {
  HG_REQUIRE(pool && idx && out, "hg_latent_pool_gather: null pointer");
  HG_REQUIRE(P > 0 && L > 0 && B > 0, "hg_latent_pool_gather: bad shape (P %ld, L %d, B %d)", P, L, B);
  hg::latent_pool_gather_kernel<<<B, 128, 0, static_cast<cudaStream_t>(stream)>>>(pool, P, L, idx, out);
  return hg::check_launch("hg_latent_pool_gather");
}

// dpool [P,L] = 0 except rows idx[b], which hold the sum over the b' with idx[b'] == idx[b] of dz[b'] in batch order (fp64,
// rounded once).  Indices outside [0, P) contribute nothing.
int hg_latent_pool_grad(const float* dz, const long* idx, int B, int L, long P, float* dpool, void* stream) {
  HG_REQUIRE(dz && idx && dpool, "hg_latent_pool_grad: null pointer");
  HG_REQUIRE(P > 0 && L > 0 && B > 0, "hg_latent_pool_grad: bad shape (P %ld, L %d, B %d)", P, L, B);
  auto st = static_cast<cudaStream_t>(stream);
  cudaMemsetAsync(dpool, 0, sizeof(float) * static_cast<size_t>(P) * L, st);
  int rc = hg::check_launch("hg_latent_pool_grad(zero)");
  if (rc) return rc;
  hg::latent_pool_grad_kernel<<<B, 128, 0, st>>>(dz, idx, B, L, P, dpool);
  return hg::check_launch("hg_latent_pool_grad");
}

// loss[0] = mean over B*L of SL1_beta(n(pred) - n(target)), n(x) = x * rsqrt(mean(x^2, row) + 1e-8); dpred (optional) =
// gscale[0] * d loss / d pred (gscale NULL: 1).  fp64 row sums added in a fixed order: the value repeats bit for bit.
int hg_latent_loss(const float* pred, const float* target, int B, int L, float beta, const float* gscale, float* dpred, float* loss,
                   void* stream) {
  HG_REQUIRE(pred && target && (loss || dpred), "hg_latent_loss: null pointer");
  HG_REQUIRE(B > 0 && L > 0 && beta > 0.f, "hg_latent_loss: bad arguments (B %d, L %d, beta %g)", B, L, static_cast<double>(beta));
  hg::latent_loss_kernel<<<1, hg::kLatentWarps * 32, 0, static_cast<cudaStream_t>(stream)>>>(pred, target, B, L, beta, gscale, dpred,
                                                                                               loss);
  return hg::check_launch("hg_latent_loss");
}

}  // extern "C"
