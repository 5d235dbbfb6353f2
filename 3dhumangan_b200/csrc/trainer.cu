// Loss + optimiser tail of a training iteration (SURVEY.md 8f-1): the reference's trainer spends it in ~10 passes over the
// [B,26,H,W] logits (one_hot, cross_entropy(reduction='none'), weighting, mean and their backward) and ~600 small per-tensor
// kernels (clip_grad_norm_, Adam for 5 + 1 parameter groups, the EMA of the generator).
//
//   hg_label_histogram / hg_seg_ce_coef / hg_seg_ce   class-balanced cross entropy of PhaseTrainer._calculate_segmentation_loss
//        (lib/trainers/phase_trainer.py:203-256, mode 'cross_entropy_balanced'): ONE pass over the logits produces the loss and
//        d loss / d logits; per-class coefficients from a label histogram, all on the device (the reference's
//        `torch.any(gt > 0)` host branch becomes a device-side select).
//   hg_mt_sumsq / hg_mt_clip_coef / hg_mt_adam         multi-tensor global-norm clipping (torch.nn.utils.clip_grad_norm_,
//        phase_trainer.py:314,336), Adam with per-group learning rates (:57-76; torch.optim.Adam arithmetic: lerp, addcmul,
//        sqrt / bias_correction2_sqrt + eps, addcdiv) and the generator's EMA (lib/components/ema.py:29-48) in one launch each
//        over a table of tensors.
// Everything is HBM-bound streaming; all reductions run in a fixed order (deterministic).
#include "common.cuh"

namespace hg {

// ------------------------------------------------------------------------------------------------------------------
// class-balanced cross entropy
// ------------------------------------------------------------------------------------------------------------------
__global__ void label_hist_kernel(const long* __restrict__ labels, long n, int L, int* __restrict__ hist) {
  __shared__ int sh[64];
  for (int i = threadIdx.x; i < 64; i += blockDim.x) sh[i] = 0;
  __syncthreads();
  for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const long v = labels[i];
    if (v >= 0 && v < L) atomicAdd(&sh[static_cast<int>(v)], 1);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < L; i += blockDim.x)
    if (sh[i]) atomicAdd(&hist[i], sh[i]);          // integer atomics: order-independent
}

// coef[c] = numel / (occ[c] * n_occ) * prior[c] / mean(prior) for the classes c >= 1 that occur (phase_trainer.py:231-239),
// 0 for the background class and for absent classes; all ones when no foreground label occurs (:242-243, plain mean CE).
__global__ void seg_ce_coef_kernel(const int* __restrict__ hist, const float* __restrict__ prior, int L, double numel,
                                   float* __restrict__ coef) {
  __shared__ int n_occ;
  __shared__ float pmean;
  if (threadIdx.x == 0) {
    int c = 0;
    float s = 0.f;
    for (int i = 0; i < L; ++i) {
      if (i >= 1 && hist[i] > 0) ++c;
      s += prior ? prior[i] : 1.f;
    }
    n_occ = c;
    pmean = s / L;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < L; i += blockDim.x) {
    float v;
    if (n_occ == 0) v = 1.f;
    else if (i == 0 || hist[i] == 0) v = 0.f;
    else v = static_cast<float>(numel / (static_cast<double>(hist[i]) * n_occ)) * ((prior ? prior[i] : 1.f) / pmean);
    coef[i] = v;
  }
}

// one thread per pixel; logits [B,L,HW] planes (a warp reads 32 consecutive pixels of one class: coalesced)
template <int kMaxL>
__global__ void __launch_bounds__(256) seg_ce_kernel(const float* __restrict__ logits, const long* __restrict__ labels,
                                                     const float* __restrict__ coef, float scale, float* __restrict__ dlogits,
                                                     double* __restrict__ partials, int B, int L, long HW) {
  __shared__ float scoef[kMaxL];
  __shared__ double red[8];
  if (threadIdx.x < kMaxL) scoef[threadIdx.x] = threadIdx.x < L ? coef[threadIdx.x] : 0.f;
  __syncthreads();
  const long total = static_cast<long>(B) * HW;
  double acc = 0.0;
  for (long p = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; p < total; p += static_cast<long>(gridDim.x) * blockDim.x) {
    const long b = p / HW, q = p - b * HW;
    const float* src = logits + b * L * HW + q;
    float v[kMaxL];
    float m = -INFINITY;
#pragma unroll
    for (int c = 0; c < kMaxL; ++c) {
      v[c] = c < L ? __ldcs(src + c * HW) : -INFINITY;
      m = fmaxf(m, v[c]);
    }
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < kMaxL; ++c) {
      v[c] = c < L ? __expf(v[c] - m) : 0.f;
      s += v[c];
    }
    const int gt = static_cast<int>(labels[p]);
    const float w = scoef[gt];
    float xg = 0.f;
#pragma unroll
    for (int c = 0; c < kMaxL; ++c)
      if (c == gt) xg = __ldg(src + c * HW);
    acc += static_cast<double>(w * (m + __logf(s) - xg));
    if (dlogits) {
      float* dst = dlogits + b * L * HW + q;
      const float k = w * scale / s;
#pragma unroll
      for (int c = 0; c < kMaxL; ++c)
        if (c < L) __stcs(dst + c * HW, k * v[c] - (c == gt ? w * scale : 0.f));
    }
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < 8; ++i) t += red[i];
    partials[blockIdx.x] = t;
  }
}

__global__ void sum_partials_kernel(const double* __restrict__ partials, int n, double scale, float* __restrict__ out) {
  double t = 0.0;                                   // single thread, fixed order
  for (int i = 0; i < n; ++i) t += partials[i];
  out[0] = static_cast<float>(t * scale);
}

// ------------------------------------------------------------------------------------------------------------------
// image reconstruction loss: mean over the B*3*HW elements of m[b,p] * rho(pred - target), rho(d) = d^2 (mode 0), the
// Charbonnier sqrt(d^2 + eps^2) (mode 1; eps -> 0 is L1) or smooth L1 with beta = eps (mode 2: the photometric loss of
// phase_trainer.py:525-527), and its gradient, in one pass.  fp64 partial per block.
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) image_loss_kernel(const float* __restrict__ pred, const float* __restrict__ target,
                                                         const float* __restrict__ mask, int mode, float eps, float scale,
                                                         float* __restrict__ dpred, double* __restrict__ partials, long total,
                                                         long HW) {
  __shared__ double red[8];
  double acc = 0.0;
  for (long e = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total; e += static_cast<long>(gridDim.x) * blockDim.x) {
    const float d = __ldcs(pred + e) - __ldcs(target + e);
    const float m = mask ? __ldg(mask + (e / (3 * HW)) * HW + e % HW) : 1.f;
    float rho, drho;
    if (mode == 0) {
      rho = d * d;
      drho = 2.f * d;
    } else if (mode == 1) {
      rho = sqrtf(fmaf(d, d, eps * eps));
      drho = d / rho;
    } else {                                        // F.smooth_l1_loss(beta = eps)
      const float z = fabsf(d);
      if (z < eps) {
        rho = 0.5f * z * z / eps;
        drho = d / eps;
      } else {
        rho = z - 0.5f * eps;
        drho = d > 0.f ? 1.f : -1.f;
      }
    }
    acc += static_cast<double>(m * rho);
    if (dpred) __stcs(dpred + e, m * drho * scale);
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < 8; ++i) t += red[i];
    partials[blockIdx.x] = t;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// multi-tensor clip / Adam / EMA
// ------------------------------------------------------------------------------------------------------------------
struct MtEntry {          // 48 bytes
  float* p;
  float* g;
  float* m;               // exp_avg
  float* v;               // exp_avg_sq
  float* ema;             // shadow parameter or null
  long n;                 // elements; the low 8 bits of `group` index the per-group scalars
};
struct MtChunk {          // 16 bytes: one block's work
  int tensor;
  int group;
  long offset;
};
constexpr int kMtChunk = 4096;
constexpr int kMtGroups = 8;
struct MtScalars {
  float lr[kMtGroups], beta1[kMtGroups], beta2[kMtGroups], eps[kMtGroups], wd[kMtGroups], bc1[kMtGroups], bc2s[kMtGroups];
  float ema_one_minus_decay;
};

__global__ void __launch_bounds__(256) mt_sumsq_kernel(const MtEntry* __restrict__ table, const MtChunk* __restrict__ chunks,
                                                       double* __restrict__ partials) {
  __shared__ double red[8];
  const MtChunk ch = chunks[blockIdx.x];
  const MtEntry e = table[ch.tensor];
  const long end = min(e.n, ch.offset + kMtChunk);
  double acc = 0.0;
  if (e.g)
    for (long i = ch.offset + threadIdx.x; i < end; i += 256) {
      const float g = e.g[i];
      acc += static_cast<double>(g) * g;
    }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < 8; ++i) t += red[i];
    partials[blockIdx.x] = t;
  }
}

// out[0] = total norm, out[1] = clip coefficient min(1, max_norm / (norm + 1e-6))  (torch.nn.utils.clip_grad_norm_)
__global__ void mt_clip_coef_kernel(const double* __restrict__ partials, int n, float max_norm, float* __restrict__ out) {
  double t = 0.0;
  for (int i = 0; i < n; ++i) t += partials[i];
  const float norm = static_cast<float>(sqrt(t));
  out[0] = norm;
  const float c = max_norm / (norm + 1e-6f);
  out[1] = max_norm > 0.f ? fminf(c, 1.f) : 1.f;
}

__global__ void __launch_bounds__(256) mt_adam_kernel(const MtEntry* __restrict__ table, const MtChunk* __restrict__ chunks,
                                                      const float* __restrict__ clip, MtScalars s, int write_grad) {
  const MtChunk ch = chunks[blockIdx.x];
  const MtEntry e = table[ch.tensor];
  const long end = min(e.n, ch.offset + kMtChunk);
  if (!e.g) {               // no gradient this step: torch.optim skips the parameter; the EMA still follows it (ema.py:44-45)
    if (e.ema)
      for (long i = ch.offset + threadIdx.x; i < end; i += 256) {
        const float sh = e.ema[i];
        e.ema[i] = sh - s.ema_one_minus_decay * (sh - e.p[i]);
      }
    return;
  }
  const int gi = ch.group;
  const float coef = clip ? clip[1] : 1.f;
  const float lr = s.lr[gi], b1 = s.beta1[gi], b2 = s.beta2[gi], eps = s.eps[gi], wd = s.wd[gi];
  const float step_size = lr / s.bc1[gi], bc2s = s.bc2s[gi];
  const float w1 = 1.f - b1;
  for (long i = ch.offset + threadIdx.x; i < end; i += 256) {
    float g = e.g[i] * coef;
    if (write_grad) e.g[i] = g;
    float p = e.p[i];
    if (wd != 0.f) g = fmaf(wd, p, g);
    float m = e.m[i], v = e.v[i];
    m = w1 < 0.5f ? m + w1 * (g - m) : g - (g - m) * (1.f - w1);      // exp_avg.lerp_(grad, 1 - beta1), ATen's two-sided form
    v = fmaf(v, b2, (1.f - b2) * g * g);              // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
    const float denom = sqrtf(v) / bc2s + eps;
    p = p - step_size * (m / denom);
    e.m[i] = m;
    e.v[i] = v;
    e.p[i] = p;
    if (e.ema) {
      const float sh = e.ema[i];
      e.ema[i] = sh - s.ema_one_minus_decay * (sh - p);          // ema.py:45
    }
  }
}

}  // namespace hg

extern "C" {

int hg_label_histogram(const long* labels, long n, int L, int* hist, void* stream) {
  HG_REQUIRE(labels && hist && n > 0 && L >= 1 && L <= 64, "hg_label_histogram: bad arguments (1 <= classes <= 64)");
  auto st = static_cast<cudaStream_t>(stream);
  cudaMemsetAsync(hist, 0, sizeof(int) * L, st);
  long blocks = (n + 255) / 256;
  if (blocks > hg::num_sms() * 8) blocks = hg::num_sms() * 8;
  hg::label_hist_kernel<<<static_cast<unsigned>(blocks), 256, 0, st>>>(labels, n, L, hist);
  return hg::check_launch("hg_label_histogram");
}

int hg_seg_ce_coef(const int* hist, const float* prior, int L, double numel, float* coef, void* stream) {
  HG_REQUIRE(hist && coef && L >= 1 && L <= 64 && numel > 0, "hg_seg_ce_coef: bad arguments");
  hg::seg_ce_coef_kernel<<<1, 64, 0, static_cast<cudaStream_t>(stream)>>>(hist, prior, L, numel, coef);
  return hg::check_launch("hg_seg_ce_coef");
}

// loss[0] = mean over pixels of coef[gt] * CE(logits, gt); dlogits (optional) = d loss / d logits.  workspace: >= 8 * (2 * #SMs) bytes.
int hg_seg_ce(const float* logits, const long* labels, const float* coef, float* dlogits, float* loss, double* workspace, int B,
              int L, long HW, void* stream) {
  HG_REQUIRE(logits && labels && coef && loss && workspace, "hg_seg_ce: null pointer");
  HG_REQUIRE(B > 0 && HW > 0 && L >= 1 && L <= 32, "hg_seg_ce: 1 <= classes <= 32 (got %d)", L);
  auto st = static_cast<cudaStream_t>(stream);
  const long total = static_cast<long>(B) * HW;
  long blocks = (total + 255) / 256;
  if (blocks > hg::num_sms() * 2) blocks = hg::num_sms() * 2;
  const float scale = 1.f / static_cast<float>(total);
  hg::seg_ce_kernel<32><<<static_cast<unsigned>(blocks), 256, 0, st>>>(logits, labels, coef, scale, dlogits, workspace, B, L, HW);
  int rc = hg::check_launch("hg_seg_ce");
  if (rc) return rc;
  hg::sum_partials_kernel<<<1, 1, 0, st>>>(workspace, static_cast<int>(blocks), 1.0 / static_cast<double>(total), loss);
  return hg::check_launch("hg_seg_ce(reduce)");
}

// loss[0] = mean over the B*3*HW elements of mask[b,p] * rho(pred - target); dpred (optional) = d loss / d pred.  The block
// partials are summed by one thread in block order, so the value repeats bit for bit.  workspace: >= 8 * (2 * #SMs) bytes.
int hg_image_loss(const float* pred, const float* target, const float* mask, float* dpred, float* loss, double* workspace,
                  int B, long HW, int mode, float eps, void* stream) {
  HG_REQUIRE(pred && target && loss && workspace, "hg_image_loss: null pointer");
  HG_REQUIRE(B > 0 && HW > 0, "hg_image_loss: bad shape");
  HG_REQUIRE(mode == 0 || ((mode == 1 || mode == 2) && eps > 0.f),
             "hg_image_loss: mode 0 (L2), 1 (Charbonnier, eps > 0) or 2 (smooth L1, beta = eps > 0)");
  auto st = static_cast<cudaStream_t>(stream);
  const long total = static_cast<long>(B) * 3 * HW;
  long blocks = (total + 255) / 256;
  if (blocks > hg::num_sms() * 2) blocks = hg::num_sms() * 2;
  hg::image_loss_kernel<<<static_cast<unsigned>(blocks), 256, 0, st>>>(pred, target, mask, mode, eps, 1.f / static_cast<float>(total),
                                                                      dpred, workspace, total, HW);
  int rc = hg::check_launch("hg_image_loss");
  if (rc) return rc;
  hg::sum_partials_kernel<<<1, 1, 0, st>>>(workspace, static_cast<int>(blocks), 1.0 / static_cast<double>(total), loss);
  return hg::check_launch("hg_image_loss(reduce)");
}

int hg_mt_entry_bytes(void) { return static_cast<int>(sizeof(hg::MtEntry)); }
int hg_mt_chunk_bytes(void) { return static_cast<int>(sizeof(hg::MtChunk)); }
int hg_mt_chunk_elems(void) { return hg::kMtChunk; }

// norm_clip[0] = global gradient norm, norm_clip[1] = clip coefficient (1 when max_norm <= 0); partials: nchunks doubles
int hg_mt_grad_norm(const void* table, const void* chunks, int nchunks, float max_norm, double* partials, float* norm_clip,
                    void* stream) {
  HG_REQUIRE(table && chunks && partials && norm_clip && nchunks > 0, "hg_mt_grad_norm: bad arguments");
  auto st = static_cast<cudaStream_t>(stream);
  hg::mt_sumsq_kernel<<<nchunks, 256, 0, st>>>(static_cast<const hg::MtEntry*>(table), static_cast<const hg::MtChunk*>(chunks), partials);
  int rc = hg::check_launch("hg_mt_grad_norm");
  if (rc) return rc;
  hg::mt_clip_coef_kernel<<<1, 1, 0, st>>>(partials, nchunks, max_norm, norm_clip);
  return hg::check_launch("hg_mt_grad_norm(finalize)");
}

// scalars: 7 arrays of `ngroups` floats (lr, beta1, beta2, eps, weight_decay, bias_correction1, sqrt(bias_correction2)), host memory
int hg_mt_adam(const void* table, const void* chunks, int nchunks, const float* norm_clip, const float* scalars, int ngroups,
               float ema_one_minus_decay, int write_clipped_grad, void* stream) {
  HG_REQUIRE(table && chunks && scalars && nchunks > 0, "hg_mt_adam: bad arguments");
  HG_REQUIRE(ngroups >= 1 && ngroups <= hg::kMtGroups, "hg_mt_adam: 1..%d parameter groups (got %d)", hg::kMtGroups, ngroups);
  hg::MtScalars s{};
  for (int i = 0; i < ngroups; ++i) {
    s.lr[i] = scalars[0 * ngroups + i]; s.beta1[i] = scalars[1 * ngroups + i]; s.beta2[i] = scalars[2 * ngroups + i];
    s.eps[i] = scalars[3 * ngroups + i]; s.wd[i] = scalars[4 * ngroups + i]; s.bc1[i] = scalars[5 * ngroups + i];
    s.bc2s[i] = scalars[6 * ngroups + i];
  }
  s.ema_one_minus_decay = ema_one_minus_decay;
  hg::mt_adam_kernel<<<nchunks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const hg::MtEntry*>(table), static_cast<const hg::MtChunk*>(chunks), norm_clip, s, write_clipped_grad);
  return hg::check_launch("hg_mt_adam");
}

}  // extern "C"
