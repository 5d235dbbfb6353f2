// Sample-quality metrics on feature sets: KID and k-NN precision / recall, on one fp64 pairwise engine.
//
//   hg_row_sqnorms     ||x_i||^2 = x_i . x_i on the engine below, so that two equal rows are at d^2 = 0 exactly.
//   hg_knn_radii       rho_k^2(x_i, X): the k-th smallest ||x_i - x_j||^2 over j != i (excluded by index, so a duplicate of x_i
//                      at another index counts at distance 0).
//   hg_ball_coverage   both directions of the k-NN coverage test in one sweep of the G x R matrix: row g is flagged when some
//                      r has d^2(g, r) <= rho_R^2[r] (precision), column r when some g has d^2(g, r) <= rho_G^2[g] (recall).
//   hg_kid             per subset s, the unbiased MMD^2 with the cubic polynomial kernel k(a, b) = (a.b / D + 1)^3 over rows
//                      gathered by index.
//
// Engine: a CTA owns 64 rows and sweeps every 64-column tile in a fixed order.  Each 32-wide K chunk of both operands is read
// as fp32 (rows past the set and entries past D read as zero), widened to fp64 and staged in shared memory; the next chunk
// waits in registers while the current one is multiplied.  Four warps each own a 32 x 32 sub-tile as 2 x 4 fragments of
// mma.sync.m16n8k16.f64 (DMMA), so every product and every sum is fp64.  d^2 = ||a||^2 + ||b||^2 - 2 a.b, clamped at 0.
// No n x n matrix reaches global memory, and no value is decided by a float atomic: repeats are bit-identical.
#include "../../include/hg3d.h"
#include "common.cuh"

namespace hg {

constexpr int kPwThreads = 128;
constexpr int kPwTile = 64;          // rows and columns of a CTA tile
constexpr int kPwK = 32;             // K chunk
constexpr int kPwStride = kPwK + 4;  // shared row stride in doubles: a fragment load touches each bank pair at most twice
constexpr int kPwLoads = kPwTile * kPwK / kPwThreads;   // fp32 values one thread stages per operand per chunk
constexpr int kTopK = 8;             // hg_knn_radii keeps the 8 smallest distances of a row; rho_k^2 is the k-th
constexpr int kDtStride = kPwTile + 1;

struct PwOperands {
  double a[kPwTile * kPwStride];
  double b[kPwTile * kPwStride];
};

struct PwSmem {
  union {
    PwOperands op;
    double dt[kPwTile * kDtStride];   // hg_knn_radii: the d^2 tile, written after the tile's last chunk is consumed
  };
  long row_a[kPwTile];                // element offset of each operand row, -1 for a zero row
  long row_b[kPwTile];
};

// d += a * b on one 16 x 8 x 16 fp64 fragment.  PTX layout, g = lane / 4, t = lane % 4: a_i at (g + 8 (i & 1), t + 4 (i >> 1)),
// b_i at (t + 4 i, g), d_i at (g + 8 (i >> 1), 2 t + (i & 1)).
__device__ __forceinline__ void dmma16816(double (&d)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, "
      "{%0,%1,%2,%3};"
      : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]), "d"(b[2]),
        "d"(b[3]));
}

// Offset of row `i` of a set of `count` rows of x [n, D], gathered through idx when it is set; -1 (a zero row) past the set or
// for an index outside [0, n).
__device__ __forceinline__ long row_offset(const long* idx, int i, int count, int n, int D) {
  if (i >= count) return -1;
  const long r = idx ? idx[i] : i;
  return (r >= 0 && r < n) ? r * D : -1;
}

// thread (warp w, lane l) stages rows w + 4 j, column l of the chunk: a warp reads 32 consecutive floats of one row
__device__ __forceinline__ void load_chunk(float (&v)[kPwLoads], const float* __restrict__ x, const long* rows, int D, int k0) {
  const int warp = threadIdx.x >> 5, k = k0 + (threadIdx.x & 31);
#pragma unroll
  for (int j = 0; j < kPwLoads; ++j) {
    const long off = rows[warp + 4 * j];
    v[j] = (off >= 0 && k < D) ? __ldg(x + off + k) : 0.f;
  }
}

__device__ __forceinline__ void store_chunk(const float (&v)[kPwLoads], double* s) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < kPwLoads; ++j) s[(warp + 4 * j) * kPwStride + lane] = static_cast<double>(v[j]);
}

// acc[mi][ni] = the dot products of the 64 x 64 tile (rows sm.row_a of xa, columns sm.row_b of xb) over all D, in fp64.
// Thread (warp wm wn, g, t) holds rows wm*32 + mi*16 + g + 8 (i >> 1) and columns wn*32 + ni*8 + 2 t + (i & 1) in acc[mi][ni][i].
// Starts and ends with a barrier, so the caller may rewrite sm.row_b and sm.dt around it.
__device__ __forceinline__ void tile_dots(double (&acc)[2][4][4], const float* __restrict__ xa, const float* __restrict__ xb, int D,
                                          PwSmem& sm) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wm = warp >> 1, wn = warp & 1, g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[mi][ni][i] = 0.0;
  float va[kPwLoads], vb[kPwLoads];
  __syncthreads();
  load_chunk(va, xa, sm.row_a, D, 0);
  load_chunk(vb, xb, sm.row_b, D, 0);
  for (int k0 = 0; k0 < D; k0 += kPwK) {
    __syncthreads();
    store_chunk(va, sm.op.a);
    store_chunk(vb, sm.op.b);
    __syncthreads();
    if (k0 + kPwK < D) {
      load_chunk(va, xa, sm.row_a, D, k0 + kPwK);
      load_chunk(vb, xb, sm.row_b, D, k0 + kPwK);
    }
#pragma unroll
    for (int ks = 0; ks < kPwK; ks += 16) {
      double a[2][8], b[4][4];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int i = 0; i < 8; ++i)
          a[mi][i] = sm.op.a[(wm * 32 + mi * 16 + g + 8 * (i & 1)) * kPwStride + ks + t + 4 * (i >> 1)];
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int i = 0; i < 4; ++i) b[ni][i] = sm.op.b[(wn * 32 + ni * 8 + g) * kPwStride + ks + t + 4 * i];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) dmma16816(acc[mi][ni], a[mi], b[ni]);
    }
  }
  __syncthreads();
}

__device__ __forceinline__ int frag_r(int mi, int i) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  return (warp >> 1) * 32 + mi * 16 + (lane >> 2) + 8 * (i >> 1);
}
__device__ __forceinline__ int frag_c(int ni, int i) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  return (warp & 1) * 32 + ni * 8 + 2 * (lane & 3) + (i & 1);
}

// The diagonal of each row tile's own product: ||x_i||^2 = x_i . x_i through the same DMMA sequence as every pairwise product,
// so d^2 of two equal rows is exactly 0 (and the norm expansion carries no rounding mismatch between norms and products).
__global__ void __launch_bounds__(kPwThreads) row_sqnorms_kernel(const float* __restrict__ x, int n, int D, double* __restrict__ out) {
  __shared__ PwSmem sm;
  const int r0 = blockIdx.x * kPwTile;
  if (threadIdx.x < kPwTile) sm.row_a[threadIdx.x] = sm.row_b[threadIdx.x] = row_offset(nullptr, r0 + threadIdx.x, n, n, D);
  double acc[2][4][4];
  tile_dots(acc, x, x, D, sm);
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int rl = frag_r(mi, i);
        if (rl == frag_c(ni, i) && r0 + rl < n) out[r0 + rl] = acc[mi][ni][i];
      }
}

// CTA = 64 rows of X.  After each column tile the clamped d^2 (j == i and columns past n as +inf) go to shared memory, and
// thread (row tid / 2, half tid % 2) folds its 32 columns into a sorted list of the 8 smallest; the two halves of a row are
// merged at the end.  The k-th smallest of a row is a property of the multiset, so the result does not depend on the order.
__global__ void __launch_bounds__(kPwThreads) knn_radii_kernel(const float* __restrict__ x, const double* __restrict__ sqn, int n,
                                                               int D, int k, double* __restrict__ rho2) {
  __shared__ PwSmem sm;
  const int r0 = blockIdx.x * kPwTile;
  if (threadIdx.x < kPwTile) sm.row_a[threadIdx.x] = row_offset(nullptr, r0 + threadIdx.x, n, n, D);
  const int my_row = threadIdx.x >> 1, half = threadIdx.x & 1;
  double L[kTopK];
#pragma unroll
  for (int j = 0; j < kTopK; ++j) L[j] = INFINITY;
  double acc[2][4][4];
  const int tiles = (n + kPwTile - 1) / kPwTile;
  for (int ct = 0; ct < tiles; ++ct) {
    const int c0 = ct * kPwTile;
    if (threadIdx.x < kPwTile) sm.row_b[threadIdx.x] = row_offset(nullptr, c0 + threadIdx.x, n, n, D);
    tile_dots(acc, x, x, D, sm);
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int rl = frag_r(mi, i), cl = frag_c(ni, i), gi = r0 + rl, gj = c0 + cl;
          double v = INFINITY;
          if (gi < n && gj < n && gi != gj) v = fmax(sqn[gi] + sqn[gj] - 2.0 * acc[mi][ni][i], 0.0);
          sm.dt[rl * kDtStride + cl] = v;
        }
    __syncthreads();
    for (int c = 0; c < 32; ++c) {
      const double v = sm.dt[my_row * kDtStride + half * 32 + c];
      if (v < L[kTopK - 1]) {
        L[kTopK - 1] = v;
#pragma unroll
        for (int j = kTopK - 1; j > 0; --j)
          if (L[j] < L[j - 1]) {
            const double s = L[j];
            L[j] = L[j - 1];
            L[j - 1] = s;
          }
      }
    }
  }
  __syncthreads();   // the last tile's scan still reads sm.dt, which the lists now reuse
#pragma unroll
  for (int j = 0; j < kTopK; ++j) sm.dt[threadIdx.x * kTopK + j] = L[j];
  __syncthreads();
  if (half == 0 && r0 + my_row < n) {
    const double* p = sm.dt + threadIdx.x * kTopK;
    const double* q = p + kTopK;
    int a = 0, b = 0;
    double v = INFINITY;
    for (int j = 0; j < k; ++j) v = (b >= kTopK || (a < kTopK && p[a] <= q[b])) ? p[a++] : q[b++];
    rho2[r0 + my_row] = v;
  }
}

// CTA = 64 rows of G sweeping every column tile of R.  Row flags gather in shared memory; a column flag is a plain store of 1
// to global memory (every writer stores the same value).
__global__ void __launch_bounds__(kPwThreads) ball_coverage_kernel(const float* __restrict__ g, const double* __restrict__ sqn_g,
                                                                   const double* __restrict__ rho2_g, int ng,
                                                                   const float* __restrict__ r, const double* __restrict__ sqn_r,
                                                                   const double* __restrict__ rho2_r, int nr, int D,
                                                                   uint8_t* __restrict__ row_flag, uint8_t* __restrict__ col_flag) {
  __shared__ PwSmem sm;
  __shared__ uint8_t flag[kPwTile];
  const int r0 = blockIdx.x * kPwTile;
  if (threadIdx.x < kPwTile) {
    sm.row_a[threadIdx.x] = row_offset(nullptr, r0 + threadIdx.x, ng, ng, D);
    flag[threadIdx.x] = 0;
  }
  double acc[2][4][4];
  const int tiles = (nr + kPwTile - 1) / kPwTile;
  for (int ct = 0; ct < tiles; ++ct) {
    const int c0 = ct * kPwTile;
    if (threadIdx.x < kPwTile) sm.row_b[threadIdx.x] = row_offset(nullptr, c0 + threadIdx.x, nr, nr, D);
    tile_dots(acc, g, r, D, sm);
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int rl = frag_r(mi, i), gi = r0 + rl, gj = c0 + frag_c(ni, i);
          if (gi >= ng || gj >= nr) continue;
          const double d2 = fmax(sqn_g[gi] + sqn_r[gj] - 2.0 * acc[mi][ni][i], 0.0);
          if (d2 <= rho2_r[gj]) flag[rl] = 1;
          if (d2 <= rho2_g[gi]) col_flag[gj] = 1;
        }
  }
  __syncthreads();
  if (threadIdx.x < kPwTile && r0 + static_cast<int>(threadIdx.x) < ng) row_flag[r0 + threadIdx.x] = flag[threadIdx.x];
}

// counts[0] = sum of row_flag, counts[1] = sum of col_flag: one CTA, each thread a strided range, then a fixed tree
__global__ void __launch_bounds__(1024) flag_count_kernel(const uint8_t* __restrict__ row_flag, int ng,
                                                          const uint8_t* __restrict__ col_flag, int nr, long* __restrict__ counts) {
  __shared__ long s[2][1024];
  long a = 0, b = 0;
  for (int i = threadIdx.x; i < ng; i += blockDim.x) a += row_flag[i];
  for (int i = threadIdx.x; i < nr; i += blockDim.x) b += col_flag[i];
  s[0][threadIdx.x] = a;
  s[1][threadIdx.x] = b;
  __syncthreads();
  for (int w = 512; w > 0; w >>= 1) {
    if (static_cast<int>(threadIdx.x) < w) {
      s[0][threadIdx.x] += s[0][threadIdx.x + w];
      s[1][threadIdx.x] += s[1][threadIdx.x + w];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    counts[0] = s[0][0];
    counts[1] = s[1][0];
  }
}

// grid (row tiles, 3 blocks, S subsets).  Block 0 = G x G, 1 = R x R (both without the diagonal, by position in the subset),
// 2 = G x R.  Each thread sums its kernel values in a fixed order, the CTA sums its threads in order, and the partial lands at
// part[(s * 3 + blk) * tiles + tile].
__global__ void __launch_bounds__(kPwThreads) kid_blocks_kernel(const float* __restrict__ g, int ng, const float* __restrict__ r, int nr,
                                                                int D, const long* __restrict__ idx_g, const long* __restrict__ idx_r,
                                                                int m, double* __restrict__ part) {
  __shared__ PwSmem sm;
  __shared__ double red[kPwThreads];
  const int blk = blockIdx.y, s = blockIdx.z, r0 = blockIdx.x * kPwTile;
  const float* xa = blk == 1 ? r : g;
  const float* xb = blk == 0 ? g : r;
  const long* ia = (blk == 1 ? idx_r : idx_g) + static_cast<long>(s) * m;
  const long* ib = (blk == 0 ? idx_g : idx_r) + static_cast<long>(s) * m;
  const int na = blk == 1 ? nr : ng, nb = blk == 0 ? ng : nr;
  if (threadIdx.x < kPwTile) sm.row_a[threadIdx.x] = row_offset(ia, r0 + threadIdx.x, m, na, D);
  const double inv_d = 1.0 / D;
  double sum = 0.0, acc[2][4][4];
  const int tiles = (m + kPwTile - 1) / kPwTile;
  for (int ct = 0; ct < tiles; ++ct) {
    const int c0 = ct * kPwTile;
    if (threadIdx.x < kPwTile) sm.row_b[threadIdx.x] = row_offset(ib, c0 + threadIdx.x, m, nb, D);
    tile_dots(acc, xa, xb, D, sm);
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int gi = r0 + frag_r(mi, i), gj = c0 + frag_c(ni, i);
          if (gi >= m || gj >= m || (blk < 2 && gi == gj)) continue;
          const double u = fma(acc[mi][ni][i], inv_d, 1.0);
          sum += u * u * u;
        }
  }
  red[threadIdx.x] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0.0;
    for (int i = 0; i < kPwThreads; ++i) tot += red[i];
    part[(static_cast<long>(s) * 3 + blk) * gridDim.x + blockIdx.x] = tot;
  }
}

__global__ void kid_finalize_kernel(const double* __restrict__ part, int tiles, int S, int m, double* __restrict__ t) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  double b[3];
  for (int blk = 0; blk < 3; ++blk) {
    double v = 0.0;
    for (int i = 0; i < tiles; ++i) v += part[(static_cast<long>(s) * 3 + blk) * tiles + i];
    b[blk] = v;
  }
  const double md = static_cast<double>(m);
  t[s] = (b[0] + b[1]) / (md * (md - 1.0)) - 2.0 * b[2] / (md * md);
}

}  // namespace hg

extern "C" {

int hg_row_sqnorms(const float* x, int n, int D, double* out, void* stream) {
  HG_REQUIRE(x && out, "hg_row_sqnorms: null pointer");
  HG_REQUIRE(n > 0 && D > 0, "hg_row_sqnorms: bad shape n=%d D=%d", n, D);
  hg::row_sqnorms_kernel<<<(n + hg::kPwTile - 1) / hg::kPwTile, hg::kPwThreads, 0, static_cast<cudaStream_t>(stream)>>>(x, n, D, out);
  return hg::check_launch("hg_row_sqnorms");
}

int hg_knn_radii(const float* x, const double* sqn, int n, int D, int k, double* rho2, void* stream) {
  HG_REQUIRE(x && sqn && rho2, "hg_knn_radii: null pointer");
  HG_REQUIRE(n > 0 && D > 0, "hg_knn_radii: bad shape n=%d D=%d", n, D);
  HG_REQUIRE(k >= 1 && k <= hg::kTopK, "hg_knn_radii: k=%d (1..%d)", k, hg::kTopK);
  HG_REQUIRE(k < n, "hg_knn_radii: k=%d needs more than k rows (n=%d)", k, n);
  hg::knn_radii_kernel<<<(n + hg::kPwTile - 1) / hg::kPwTile, hg::kPwThreads, 0, static_cast<cudaStream_t>(stream)>>>(x, sqn, n, D, k,
                                                                                                                       rho2);
  return hg::check_launch("hg_knn_radii");
}

int hg_ball_coverage(const float* g, const double* sqn_g, const double* rho2_g, int ng, const float* r, const double* sqn_r,
                     const double* rho2_r, int nr, int D, unsigned char* row_flag, unsigned char* col_flag, long* counts, void* stream) {
  HG_REQUIRE(g && sqn_g && rho2_g && r && sqn_r && rho2_r && row_flag && col_flag && counts, "hg_ball_coverage: null pointer");
  HG_REQUIRE(ng > 0 && nr > 0 && D > 0, "hg_ball_coverage: bad shape ng=%d nr=%d D=%d", ng, nr, D);
  auto st = static_cast<cudaStream_t>(stream);
  const cudaError_t e = cudaMemsetAsync(col_flag, 0, static_cast<size_t>(nr), st);
  if (e != cudaSuccess) { hg::set_error("hg_ball_coverage: clearing the column flags failed: %s", cudaGetErrorString(e)); return 2; }
  hg::ball_coverage_kernel<<<(ng + hg::kPwTile - 1) / hg::kPwTile, hg::kPwThreads, 0, st>>>(g, sqn_g, rho2_g, ng, r, sqn_r, rho2_r, nr,
                                                                                         D, row_flag, col_flag);
  const int rc = hg::check_launch("hg_ball_coverage");
  if (rc) return rc;
  hg::flag_count_kernel<<<1, 1024, 0, st>>>(row_flag, ng, col_flag, nr, counts);
  return hg::check_launch("hg_ball_coverage(count)");
}

size_t hg_kid_workspace_bytes(int S, int m) {
  if (S <= 0 || m <= 0) return 0;
  return static_cast<size_t>(S) * 3 * ((m + hg::kPwTile - 1) / hg::kPwTile) * sizeof(double);
}

int hg_kid(const float* g, int ng, const float* r, int nr, int D, const long* idx_g, const long* idx_r, int S, int m, double* t,
           double* workspace, size_t workspace_bytes, void* stream) {
  HG_REQUIRE(g && r && idx_g && idx_r && t && workspace, "hg_kid: null pointer");
  HG_REQUIRE(ng > 0 && nr > 0 && D > 0, "hg_kid: bad shape ng=%d nr=%d D=%d", ng, nr, D);
  HG_REQUIRE(S >= 1 && S <= 65535, "hg_kid: S=%d subsets (1..65535)", S);
  HG_REQUIRE(m >= 2 && m <= ng && m <= nr, "hg_kid: subset size m=%d must be in [2, min(ng=%d, nr=%d)]", m, ng, nr);
  HG_REQUIRE(workspace_bytes >= hg_kid_workspace_bytes(S, m), "hg_kid: workspace of %zu bytes, %zu needed", workspace_bytes,
             hg_kid_workspace_bytes(S, m));
  auto st = static_cast<cudaStream_t>(stream);
  const int tiles = (m + hg::kPwTile - 1) / hg::kPwTile;
  hg::kid_blocks_kernel<<<dim3(tiles, 3, S), hg::kPwThreads, 0, st>>>(g, ng, r, nr, D, idx_g, idx_r, m, workspace);
  const int rc = hg::check_launch("hg_kid");
  if (rc) return rc;
  hg::kid_finalize_kernel<<<(S + 127) / 128, 128, 0, st>>>(workspace, tiles, S, m, t);
  return hg::check_launch("hg_kid(finalize)");
}

}  // extern "C"
