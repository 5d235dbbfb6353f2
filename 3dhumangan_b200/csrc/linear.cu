// Weight packing + the generic row-major linear layer  Y[M,N] = X[M,K] . W[N,K]^T + b  on wgmma.
//
// Used for (a) the low-resolution SPADE style projections (SURVEY.md §8a a13: W_s . feature_maps
// is linear, so it commutes with the bilinear up-sample and runs at render resolution), and
// (b) as the smallest complete user of the tensor-core primitives in wgmma.cuh (self-test target).
//
// Precision modes: passes == 1  plain bf16 operands, fp32 accumulate;
//                  passes == 3  bf16x3 split (A_hi.B_hi + A_lo.B_hi + A_hi.B_lo), ~2^-16 relative,
//                               the mode that meets the 1e-3-of-fp32 parity contract.
#include "common.cuh"
#include "wgmma.cuh"

namespace hg {

// ------------------------------------------------------------------------------------------
// Packed weight image:  [nblocks][kchunks][part: hi, lo][Nb x 64 bf16, K-major SW128]
// Every [Nb x 64] tile is Nb*128 contiguous bytes = the exact shared-memory image a single
// cp.async.bulk drops next to the A operand.
// ------------------------------------------------------------------------------------------
__global__ void pack_weight_kernel(const float* __restrict__ W, int N, int K, int ldw,
                                   const float* __restrict__ scale_ptr, float scale, int Nb, int nblocks,
                                   int kchunks, uint8_t* __restrict__ out) {
  const long total = static_cast<long>(nblocks) * Nb * kchunks * 8;
  const long idx = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int k8 = static_cast<int>(idx % (kchunks * 8));
  const int n = static_cast<int>(idx / (kchunks * 8));
  const int nb = n / Nb, r = n % Nb, kc = k8 / 8, c = k8 % 8;
  const float s = scale_ptr ? scale * scale_ptr[0] : scale;
  float x[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int k = k8 * 8 + i;
    x[i] = (n < N && k < K) ? W[static_cast<long>(n) * ldw + k] * s : 0.f;
  }
  const size_t tile_bytes = static_cast<size_t>(Nb) * 128;
  uint8_t* hi = out + (static_cast<size_t>(nb * kchunks + kc) * 2 + 0) * tile_bytes;
  uint8_t* lo = hi + tile_bytes;
  uint32_t h4[4], l4[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) split_bf16x2(x[2 * i], x[2 * i + 1], h4[i], l4[i]);
  const uint32_t off = sw128_offset(r, c * 8);
  *reinterpret_cast<uint4*>(hi + off) = make_uint4(h4[0], h4[1], h4[2], h4[3]);
  *reinterpret_cast<uint4*>(lo + off) = make_uint4(l4[0], l4[1], l4[2], l4[3]);
}

// ------------------------------------------------------------------------------------------
// linear kernel: warps 0-7 are two warpgroups; warpgroup g loads rows 64g..64g+63 of the X tile, issues the wgmmas of those
// rows (accumulator [64 x N] in registers) and stores them; warp 8 streams the weight tiles.
// ------------------------------------------------------------------------------------------
constexpr int kLinThreads = 288;
constexpr int kLinStages = 3;
constexpr uint32_t kChunkBytesA = 128 * 128;  // one [128 x 64] bf16 tile
constexpr uint32_t kStageBytesB = 256 * 128;  // one [256 x 64] bf16 tile (max)
constexpr uint32_t kLinSmem = 8 * kChunkBytesA + kLinStages * kStageBytesB + 256 + 1024;

template <int kPasses, int N>
__global__ void __launch_bounds__(kLinThreads, 1)
linear_kernel(const float* __restrict__ X, int ldx, int M, int K, const uint8_t* __restrict__ Wimg, int Nb,
              int nblocks, int N_, const float* __restrict__ bias, float* __restrict__ Y, int ldy) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_hi = smem;
  uint8_t* a_lo = smem + 4 * kChunkBytesA;
  uint8_t* b_st = smem + 8 * kChunkBytesA;
  uint64_t* bars = reinterpret_cast<uint64_t*>(b_st + kLinStages * kStageBytesB);
  uint64_t* b_full = bars;                      // [kLinStages]
  uint64_t* b_empty = bars + kLinStages;        // [kLinStages]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kchunks = (K + 63) / 64;
  const int num_tiles = (M + 127) / 128;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kLinStages; ++i) {
      mbar_init(b_full + i, 1);
      mbar_init(b_empty + i, 2);     // one arrival per warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < 8) {
    const int g = warp >> 2, t = threadIdx.x & 127;
    const uint32_t a_off = g * 64 * 128;           // this warpgroup's rows inside every [128 x 64] chunk
    uint32_t st = 0, ph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      // ------------------------------------------------------------ X rows 64g.. -> A (the previous tile's wgmmas are done)
      for (int r = g * 64 + (warp & 3); r < g * 64 + 64; r += 4) {
        const long grow = static_cast<long>(tile) * 128 + r;
        for (int kb = lane * 8; kb < kchunks * 64; kb += 256) {
          float x[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) x[i] = 0.f;
          if (grow < M) {
            if (kb + 8 <= K && (ldx & 3) == 0) {
              const float4 v0 = *reinterpret_cast<const float4*>(X + grow * ldx + kb);
              const float4 v1 = *reinterpret_cast<const float4*>(X + grow * ldx + kb + 4);
              x[0] = v0.x; x[1] = v0.y; x[2] = v0.z; x[3] = v0.w;
              x[4] = v1.x; x[5] = v1.y; x[6] = v1.z; x[7] = v1.w;
            } else {
#pragma unroll
              for (int i = 0; i < 8; ++i)
                if (kb + i < K) x[i] = X[grow * ldx + kb + i];
            }
          }
          const int kc = kb >> 6;
          store_a8<kPasses == 3>(a_hi + kc * kChunkBytesA, a_lo + kc * kChunkBytesA, r, kb & 63, x);
        }
      }
      fence_proxy_async_smem();
      named_barrier(1 + g, 128);

      for (int nb = 0; nb < nblocks; ++nb) {
        float d[N / 2];
        // one weight stage: wait, issue, and release the stage consumed one step earlier once its wgmmas are done
        uint32_t prev = ~0u;
        auto stage = [&](uint32_t a_tile, uint32_t a_tile2, bool two, bool accumulate) {
          mbar_wait(b_full + st, ph);
          acc_fence(d);
          wgmma_fence();
          const uint32_t bt = smem_u32(b_st + st * kStageBytesB);
          wg_k64<N>(d, a_tile, bt, accumulate);
          if (two) wg_k64<N>(d, a_tile2, bt, true);
          wgmma_commit();
          wgmma_wait<1>();
          acc_fence(d);
          if (prev != ~0u && t == 0) mbar_arrive(b_empty + prev);
          prev = st;
          if (++st == kLinStages) { st = 0; ph ^= 1; }
        };
        for (int kc = 0; kc < kchunks; ++kc) {
          const uint32_t ahi = smem_u32(a_hi + kc * kChunkBytesA) + a_off, alo = smem_u32(a_lo + kc * kChunkBytesA) + a_off;
          stage(ahi, alo, kPasses == 3, kc > 0);
          if (kPasses == 3) stage(ahi, ahi, false, true);
        }
        wgmma_wait<0>();
        acc_fence(d);
        if (t == 0) mbar_arrive(b_empty + prev);
        // ---------------------------------------------------------- epilogue straight from the fragments
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const long grow = static_cast<long>(tile) * 128 + g * 64 + frag_row(t, i);
          if (grow >= M) continue;
#pragma unroll
          for (int j = 0; j < N / 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int c = frag_col(t, j, e), n = nb * Nb + c;
              if (c < Nb && n < N_) Y[grow * ldy + n] = d[4 * j + 2 * i + e] + (bias ? bias[n] : 0.f);
            }
        }
      }
      named_barrier(1 + g, 128);     // every warp of the group is done reading before the next tile overwrites A
    }
  } else {
    // ------------------------------------------------------------ weight producer (bulk copies from L2)
    if (lane == 0) {
      const uint32_t tile_bytes = static_cast<uint32_t>(Nb) * 128;
      uint32_t st = 0, ph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        for (int nb = 0; nb < nblocks; ++nb)
          for (int kc = 0; kc < kchunks; ++kc)
            for (int part = 0; part < (kPasses == 3 ? 2 : 1); ++part) {
              mbar_wait_backoff(b_empty + st, ph ^ 1);
              mbar_arrive_expect_tx(b_full + st, tile_bytes);
              bulk_g2s(b_st + st * kStageBytesB,
                       Wimg + (static_cast<size_t>(nb * kchunks + kc) * 2 + part) * tile_bytes, tile_bytes,
                       b_full + st);
              if (++st == kLinStages) { st = 0; ph ^= 1; }
            }
      }
    }
  }
}

template <int kPasses, int N>
static int launch_linear(int grid, cudaStream_t st, const float* X, int ldx, int M, int K, const uint8_t* img, int Nb, int nblocks,
                         int N_, const float* bias, float* Y, int ldy) {
  const cudaError_t e = cudaFuncSetAttribute(linear_kernel<kPasses, N>, cudaFuncAttributeMaxDynamicSharedMemorySize, kLinSmem);
  if (e != cudaSuccess) { set_error("hg_linear: smem opt-in failed: %s", cudaGetErrorString(e)); return 2; }
  linear_kernel<kPasses, N><<<grid, kLinThreads, kLinSmem, st>>>(X, ldx, M, K, img, Nb, nblocks, N_, bias, Y, ldy);
  return check_launch("hg_linear");
}

}  // namespace hg

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
extern "C" {

size_t hg_packed_weight_bytes(int N, int K, int Nb) {
  if (N <= 0 || K <= 0 || Nb <= 0) return 0;
  const size_t nblocks = (N + Nb - 1) / Nb, kchunks = (K + 63) / 64;
  return nblocks * kchunks * 2 * static_cast<size_t>(Nb) * 128;
}

int hg_pack_weight(const float* W, int N, int K, int ldw, const float* scale_dev, float scale, int Nb,
                   void* out_img, size_t out_bytes, void* stream) {
  HG_REQUIRE(W && out_img, "hg_pack_weight: null pointer");
  HG_REQUIRE(Nb >= 16 && Nb <= 256 && Nb % 16 == 0, "hg_pack_weight: Nb=%d must be a multiple of 16 in [16,256]", Nb);
  HG_REQUIRE(N > 0 && K > 0 && ldw >= K, "hg_pack_weight: bad shape N=%d K=%d ldw=%d", N, K, ldw);
  HG_REQUIRE(out_bytes >= hg_packed_weight_bytes(N, K, Nb), "hg_pack_weight: output buffer too small");
  HG_REQUIRE((reinterpret_cast<uintptr_t>(out_img) & 15) == 0, "hg_pack_weight: output must be 16-byte aligned");
  const int nblocks = (N + Nb - 1) / Nb, kchunks = (K + 63) / 64;
  const long total = static_cast<long>(nblocks) * Nb * kchunks * 8;
  hg::pack_weight_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      W, N, K, ldw, scale_dev, scale, Nb, nblocks, kchunks, static_cast<uint8_t*>(out_img));
  return hg::check_launch("hg_pack_weight");
}

int hg_linear(const float* X, int ldx, int M, int K, const void* Wimg, int Nb, int N, const float* bias, float* Y,
              int ldy, int passes, void* stream) {
  HG_REQUIRE(X && Wimg && Y, "hg_linear: null pointer");
  HG_REQUIRE(M > 0 && K > 0 && K <= 256 && N > 0, "hg_linear: need 0 < K <= 256 (got %d), M=%d N=%d", K, M, N);
  HG_REQUIRE(Nb >= 16 && Nb <= 256 && Nb % 16 == 0, "hg_linear: Nb=%d must be a multiple of 16 in [16,256]", Nb);
  HG_REQUIRE(passes == 1 || passes == 3, "hg_linear: passes must be 1 (bf16) or 3 (bf16x3)");
  HG_REQUIRE(ldx >= K && ldy >= N, "hg_linear: leading dimensions too small");
  const int nblocks = (N + Nb - 1) / Nb;
  const int num_tiles = (M + 127) / 128;
  const int grid = num_tiles < hg::num_sms() ? num_tiles : hg::num_sms();
  auto st = static_cast<cudaStream_t>(stream);
  const auto* img = static_cast<const uint8_t*>(Wimg);
  // wgmma N: the smallest of 64 / 128 / 256 that covers a block (columns past Nb are computed and dropped)
  if (passes == 3) {
    if (Nb <= 64) return hg::launch_linear<3, 64>(grid, st, X, ldx, M, K, img, Nb, nblocks, N, bias, Y, ldy);
    if (Nb <= 128) return hg::launch_linear<3, 128>(grid, st, X, ldx, M, K, img, Nb, nblocks, N, bias, Y, ldy);
    return hg::launch_linear<3, 256>(grid, st, X, ldx, M, K, img, Nb, nblocks, N, bias, Y, ldy);
  }
  if (Nb <= 64) return hg::launch_linear<1, 64>(grid, st, X, ldx, M, K, img, Nb, nblocks, N, bias, Y, ldy);
  if (Nb <= 128) return hg::launch_linear<1, 128>(grid, st, X, ldx, M, K, img, Nb, nblocks, N, bias, Y, ldy);
  return hg::launch_linear<1, 256>(grid, st, X, ldx, M, K, img, Nb, nblocks, N, bias, Y, ldy);
}

}  // extern "C"
