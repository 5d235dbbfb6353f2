// Ray sampling against the posed SMPL mesh + the 31-d geometry feature of every sample point.
//
// Replaces (reference file:line):
//   vr.get_initial_rays_weak_perspective   lib/generators/volume_rendering.py:86-110
//   vr.perturb_points / transform_sampled_points   volume_rendering.py:124-170
//   get_geo_features                        lib/components/smpl.py:210-249
//     (cdist to 24 joints, inverse(fk) blended by LBS weights, K=1 nearest posed vertex
//      [pytorch3d.ops.knn_points], canonicalisation, nearest distance)
//
// One thread = one sample point.  The 6890 posed vertices of the point's body are staged in
// shared memory as float4 (110 KB); the distance is evaluated exactly as the oracle defines it --
// (dx*dx + dy*dy) + dz*dz with one fp32 rounding per operation (no FMA contraction), lowest index
// on ties -- which makes the nearest index bit-exact for identical input points.
//
// Exact pruning (hg_knn_prep): vertices are Morton-sorted per body and cut into clusters of 32 with
// an axis-aligned box each.  A point first measures the first vertex of every cluster (a real
// candidate), then scans only clusters whose box distance -- computed with the SAME rounded
// operations, hence a true lower bound of every member's computed distance -- does not exceed the
// running best.  The result is identical to the brute-force scan (ties: explicit lowest original
// index) at ~1/8 of the instructions.
//
// Output record per point (kPointStride floats, 16-byte aligned rows):
//   [0..2]  xyz * input_scaler        (input of first_layer_coord, modulated.py:44,56)
//   [3..33] 31 geometry features      (order per legacy_mode, smpl.py:239-242)
//   [34,35] zero padding
#include "common.cuh"

namespace hg {

constexpr int kPointStride = 36;
constexpr int kJoints = 24;

// -------------------------------------------------------------------------------------------
// vertex_ik[b,v] = sum_j lbs[b,v,j] * inverse(fk[b,j])        (smpl.py:217-218)
// -------------------------------------------------------------------------------------------
__device__ void invert4x4(const float* m, float* out) {
  // Gauss-Jordan with partial pivoting on [m | I]
  float a[4][8];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      a[i][j] = m[i * 4 + j];
      a[i][4 + j] = (i == j) ? 1.f : 0.f;
    }
  for (int c = 0; c < 4; ++c) {
    int piv = c;
    float best = fabsf(a[c][c]);
    for (int r = c + 1; r < 4; ++r)
      if (fabsf(a[r][c]) > best) { best = fabsf(a[r][c]); piv = r; }
    if (piv != c)
      for (int j = 0; j < 8; ++j) { float t = a[c][j]; a[c][j] = a[piv][j]; a[piv][j] = t; }
    const float inv = 1.f / a[c][c];
    for (int j = 0; j < 8; ++j) a[c][j] *= inv;
    for (int r = 0; r < 4; ++r) {
      if (r == c) continue;
      const float f = a[r][c];
      for (int j = 0; j < 8; ++j) a[r][j] = fmaf(-f, a[c][j], a[r][j]);
    }
  }
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) out[i * 4 + j] = a[i][4 + j];
}

__global__ void vertex_ik_kernel(const float* __restrict__ fk, const float* __restrict__ lbs, int V,
                                 float* __restrict__ vertex_ik) {
  __shared__ float ik[kJoints * 16];
  const int b = blockIdx.y;
  if (threadIdx.x < kJoints) invert4x4(fk + (static_cast<long>(b) * kJoints + threadIdx.x) * 16, ik + threadIdx.x * 16);
  __syncthreads();
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const float* w = lbs + (static_cast<long>(b) * V + v) * kJoints;
  float acc[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = 0.f;
  for (int j = 0; j < kJoints; ++j) {
    const float wj = w[j];
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = fmaf(wj, ik[j * 16 + i], acc[i]);
  }
  float4* o = reinterpret_cast<float4*>(vertex_ik + (static_cast<long>(b) * V + v) * 16);
#pragma unroll
  for (int i = 0; i < 4; ++i) o[i] = make_float4(acc[4 * i], acc[4 * i + 1], acc[4 * i + 2], acc[4 * i + 3]);
}


// -------------------------------------------------------------------------------------------
// KNN preparation: Morton sort + cluster boxes (one CTA per body)
// -------------------------------------------------------------------------------------------
constexpr int kSortN = 8192;      // >= V, power of two
constexpr int kCluster = 32;

__device__ __forceinline__ uint32_t spread10(uint32_t v) {
  v &= 1023u;
  v = (v | (v << 16)) & 0x030000FFu;
  v = (v | (v << 8)) & 0x0300F00Fu;
  v = (v | (v << 4)) & 0x030C30C3u;
  v = (v | (v << 2)) & 0x09249249u;
  return v;
}

__global__ void __launch_bounds__(1024, 1) knn_prep_kernel(const float* __restrict__ vertices, int V, int Vp,
                                                           float4* __restrict__ sorted, float4* __restrict__ boxes) {
  extern __shared__ unsigned long long keys[];   // [kSortN]
  __shared__ float red[6][32];
  __shared__ float bb[6];
  const int b = blockIdx.x;
  const float* vp = vertices + static_cast<long>(b) * V * 3;
  float lo[3] = {3e38f, 3e38f, 3e38f}, hi[3] = {-3e38f, -3e38f, -3e38f};
  for (int v = threadIdx.x; v < V; v += blockDim.x)
    for (int d = 0; d < 3; ++d) {
      const float c = vp[v * 3 + d];
      lo[d] = fminf(lo[d], c);
      hi[d] = fmaxf(hi[d], c);
    }
  for (int d = 0; d < 3; ++d) {
    for (int o = 16; o > 0; o >>= 1) {
      lo[d] = fminf(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
      hi[d] = fmaxf(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
    }
    if ((threadIdx.x & 31) == 0) { red[d][threadIdx.x >> 5] = lo[d]; red[3 + d][threadIdx.x >> 5] = hi[d]; }
  }
  __syncthreads();
  if (threadIdx.x < 6) {
    float r = red[threadIdx.x][0];
    for (int i = 1; i < 32; ++i) r = threadIdx.x < 3 ? fminf(r, red[threadIdx.x][i]) : fmaxf(r, red[threadIdx.x][i]);
    bb[threadIdx.x] = r;
  }
  __syncthreads();
  for (int v = threadIdx.x; v < kSortN; v += blockDim.x) {
    unsigned long long key = ~0ull;
    if (v < V) {
      uint32_t code = 0;
      for (int d = 0; d < 3; ++d) {
        const float ext = fmaxf(bb[3 + d] - bb[d], 1e-20f);
        int qd = static_cast<int>((vp[v * 3 + d] - bb[d]) / ext * 1023.f);
        qd = qd < 0 ? 0 : (qd > 1023 ? 1023 : qd);
        code |= spread10(static_cast<uint32_t>(qd)) << d;
      }
      key = (static_cast<unsigned long long>(code) << 13) | static_cast<unsigned long long>(v);
    }
    keys[v] = key;
  }
  __syncthreads();
  for (int k = 2; k <= kSortN; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < kSortN; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = keys[i], c = keys[ixj];
          const bool up = (i & k) == 0;
          if ((a > c) == up) { keys[i] = c; keys[ixj] = a; }
        }
      }
      __syncthreads();
    }
  float4* out = sorted + static_cast<long>(b) * Vp;
  for (int i = threadIdx.x; i < Vp; i += blockDim.x) {
    const int src = i < V ? i : V - 1;   // pad with copies of the last vertex (same index: harmless)
    const int v = static_cast<int>(keys[src] & 8191ull);
    out[i] = make_float4(vp[v * 3], vp[v * 3 + 1], vp[v * 3 + 2], __int_as_float(v));
  }
  __syncthreads();
  const int M = Vp / kCluster;
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    float l[3] = {3e38f, 3e38f, 3e38f}, h[3] = {-3e38f, -3e38f, -3e38f};
    for (int i = 0; i < kCluster; ++i) {
      const int src = (m * kCluster + i) < V ? (m * kCluster + i) : V - 1;
      const int v = static_cast<int>(keys[src] & 8191ull);
      for (int d = 0; d < 3; ++d) {
        l[d] = fminf(l[d], vp[v * 3 + d]);
        h[d] = fmaxf(h[d], vp[v * 3 + d]);
      }
    }
    boxes[(static_cast<long>(b) * M + m) * 2 + 0] = make_float4(l[0], l[1], l[2], 0.f);
    boxes[(static_cast<long>(b) * M + m) * 2 + 1] = make_float4(h[0], h[1], h[2], 0.f);
  }
}

// -------------------------------------------------------------------------------------------
// rays + KNN + features
// -------------------------------------------------------------------------------------------
struct GeoArgs {
  // ray grid (tiny host-prepared tables so that the linspace arithmetic is torch's own)
  const float* xs;  // [Rw]  linspace(-Rw/Rh, Rw/Rh, Rw)
  const float* ys;  // [Rh]  linspace(-1, 1, Rh)
  const float* zs;  // [S]   linspace(ray_start, ray_end, S)
  const float* focals;     // [B]
  const float* scales;     // [B]
  const float* cam2world;  // [B,4,4]
  const float* jitter;     // [B,R,S] uniform draws, or null (no perturbation)
  const float* points_in;  // [B,N,3] world points; when non-null the ray stage is skipped
  const float* skeletons;  // [B,24,3]
  const float* vertices;   // [B,V,3]
  const float* tpose;      // [B,V,3]
  const float* vertex_ik;  // [B,V,16]
  const float4* sorted;    // [B,Vp] Morton-sorted (x,y,z,index) or null -> brute force over `vertices`
  const float4* boxes;     // [B,Vp/32,2] cluster boxes (lo, hi)
  int Vp;
  int B, Rw, Rh, S, V;
  int n_points;  // per body: Rw*Rh*S, or N when points_in is given
  float input_scaler;
  int legacy_mode;
  // outputs
  float* rec;       // [B,N,36]
  float* z_vals;    // [B,N] jittered depths (null when points_in)
  float* points;    // [B,N,3] optional world points
  int* nearest;     // [B,N] optional nearest vertex index
  float* nearest_d2;  // [B,N] optional squared distance
};

constexpr int kGeoThreads = 512;

// value barrier for a packed fp32 pair: keeps ptxas from contracting a packed product with the packed sum that follows
__device__ __forceinline__ float2 keep2(float2 v) {
  unsigned long long u = (static_cast<unsigned long long>(__float_as_uint(v.y)) << 32) | __float_as_uint(v.x);
  asm volatile("" : "+l"(u));
  return make_float2(__uint_as_float(static_cast<uint32_t>(u)), __uint_as_float(static_cast<uint32_t>(u >> 32)));
}

__global__ void __launch_bounds__(kGeoThreads, 1) geo_kernel(GeoArgs a) {
  extern __shared__ float4 sv[];  // [Vn] posed vertices (x,y,z,index), then [M][2] cluster boxes
  __shared__ float sk[kJoints * 3];
  __shared__ float c2w[16];
  const int b = blockIdx.y;
  const int Vn = a.sorted ? a.Vp : a.V;
  const int M = a.sorted ? a.Vp / kCluster : 0;
  float4* sbox = sv + Vn;
  if (a.sorted) {
    // pair layout for the packed-fp32 distance loop: vertices 2p, 2p+1 -> sv[2p] = (x0, x1, y0, y1), sv[2p+1] = (z0, z1, i0, i1)
    // (Vp is a multiple of the cluster size 32)
    for (int v = threadIdx.x; v < Vn; v += blockDim.x) {
      const float4 q = a.sorted[static_cast<long>(b) * Vn + v];
      float* pr = reinterpret_cast<float*>(sv + (v & ~1));
      const int e = v & 1;
      pr[0 + e] = q.x;
      pr[2 + e] = q.y;
      pr[4 + e] = q.z;
      pr[6 + e] = q.w;
    }
    for (int v = threadIdx.x; v < 2 * M; v += blockDim.x) sbox[v] = a.boxes[static_cast<long>(b) * 2 * M + v];
  } else {
    for (int v = threadIdx.x; v < a.V; v += blockDim.x) {
      const float* p = a.vertices + (static_cast<long>(b) * a.V + v) * 3;
      sv[v] = make_float4(p[0], p[1], p[2], __int_as_float(v));
    }
  }
  if (threadIdx.x < kJoints * 3) sk[threadIdx.x] = a.skeletons[static_cast<long>(b) * kJoints * 3 + threadIdx.x];
  if (threadIdx.x < 16 && a.cam2world) c2w[threadIdx.x] = a.cam2world[b * 16 + threadIdx.x];
  __syncthreads();

  const int N = a.n_points;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
    const long gp = static_cast<long>(b) * N + p;
    float px, py, pz;
    if (a.points_in) {
      px = a.points_in[gp * 3 + 0];
      py = a.points_in[gp * 3 + 1];
      pz = a.points_in[gp * 3 + 2];
    } else {
      // volume_rendering.py:86-110: ray r = h*Rw + w, sample s fastest
      const int s = p % a.S, r = p / a.S;
      const int w = r % a.Rw, h = r / a.Rw;
      const float focal = a.focals[b];
      const float vx = a.xs[w], vy = a.ys[h], vz = focal;
      const float nrm = sqrtf(vx * vx + vy * vy + vz * vz) + 1e-12f;
      const float dx = vx / nrm, dy = vy / nrm, dz = vz / nrm;
      const float zc = focal / a.scales[b];
      float z = a.zs[s] + zc;
      float cx = dx * z, cy = dy * z, cz = dz * z;
      if (a.jitter) {  // volume_rendering.py:124-130
        const float delta = (a.zs[1] + zc) - (a.zs[0] + zc);
        const float off = (a.jitter[gp] - 0.5f) * delta;
        z = z + off;
        cx = cx + off * dx;
        cy = cy + off * dy;
        cz = cz + off * dz;
      }
      // volume_rendering.py:150-155: world = cam2world . [p; 1]
      px = c2w[0] * cx + c2w[1] * cy + c2w[2] * cz + c2w[3];
      py = c2w[4] * cx + c2w[5] * cy + c2w[6] * cz + c2w[7];
      pz = c2w[8] * cx + c2w[9] * cy + c2w[10] * cz + c2w[11];
      if (a.z_vals) a.z_vals[gp] = z;
    }
    if (a.points) {
      a.points[gp * 3 + 0] = px;
      a.points[gp * 3 + 1] = py;
      a.points[gp * 3 + 2] = pz;
    }

    // K=1 nearest posed vertex (smpl.py:220), exact oracle arithmetic.  best starts at +inf so that a d2 which
    // overflows to inf is still a candidate (lowest index on the tie); only a NaN d2 is never taken.
    float best = INFINITY;
    int bi = 0x7fffffff;
    auto consider = [&](const float4 q) {
      const float ex = __fsub_rn(px, q.x), ey = __fsub_rn(py, q.y), ez = __fsub_rn(pz, q.z);
      const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(ez, ez));
      const int vi = __float_as_int(q.w);
      if (d2 < best || (d2 == best && vi < bi)) { best = d2; bi = vi; }
    };
    if (M == 0) {
#pragma unroll 4
      for (int v = 0; v < Vn; ++v) consider(sv[v]);
    } else {
      // two vertices per step on fp32 pairs (ffma2 / fmul2 / fadd2 are the same IEEE operations as the scalar ones:
      // p - q as fma(q, -1, p) rounds the exact difference once, like the subtraction; products and sums are NOT contracted),
      // candidates still examined in index order: bit-identical distances and the same tie-breaking as `consider`
      const float2 px2 = make_float2(px, px), py2 = make_float2(py, py), pz2 = make_float2(pz, pz), neg1 = make_float2(-1.f, -1.f);
      auto consider2 = [&](const float4 xy, const float4 zw) {
        const float2 ex = ffma2(make_float2(xy.x, xy.y), neg1, px2);
        const float2 ey = ffma2(make_float2(xy.z, xy.w), neg1, py2);
        const float2 ez = ffma2(make_float2(zw.x, zw.y), neg1, pz2);
        // the products go through an opaque register so that they are rounded before the sums, as in the oracle
        const float2 d2 = fadd2(fadd2(keep2(fmul2(ex, ex)), keep2(fmul2(ey, ey))), keep2(fmul2(ez, ez)));
        const int v0 = __float_as_int(zw.z), v1 = __float_as_int(zw.w);
        if (d2.x < best || (d2.x == best && v0 < bi)) { best = d2.x; bi = v0; }
        if (d2.y < best || (d2.y == best && v1 < bi)) { best = d2.y; bi = v1; }
      };
      // pass 1: one real candidate per cluster tightens the bound
#pragma unroll 4
      for (int m = 0; m < M; ++m) {
        const float4 xy = sv[m * kCluster], zw = sv[m * kCluster + 1];
        consider(make_float4(xy.x, xy.z, zw.x, zw.z));
      }
      // pass 2: scan the clusters whose box can still contain a vertex at distance <= best.  The box
      // distance uses the same rounded operations as `consider`, so it never exceeds a member's d2.
      for (int m = 0; m < M; ++m) {
        const float4 lo = sbox[2 * m], hi = sbox[2 * m + 1];
        const float bx = fmaxf(fmaxf(__fsub_rn(lo.x, px), __fsub_rn(px, hi.x)), 0.f);
        const float by = fmaxf(fmaxf(__fsub_rn(lo.y, py), __fsub_rn(py, hi.y)), 0.f);
        const float bz = fmaxf(fmaxf(__fsub_rn(lo.z, pz), __fsub_rn(pz, hi.z)), 0.f);
        const float lb = __fadd_rn(__fadd_rn(__fmul_rn(bx, bx), __fmul_rn(by, by)), __fmul_rn(bz, bz));
        if (lb <= best) {
#pragma unroll 8
          for (int i = 0; i < kCluster; i += 2) consider2(sv[m * kCluster + i], sv[m * kCluster + i + 1]);
        }
      }
    }
    // a NaN point took no candidate: index 0 and d2 NaN, as knn_points' min / first-argmin gives, and never a row
    // index from the sentinel below
    if (bi == 0x7fffffff) { bi = 0; best = __int_as_float(0x7fffffff); }
    if (a.nearest) a.nearest[gp] = bi;
    if (a.nearest_d2) a.nearest_d2[gp] = best;

    float* o = a.rec + gp * kPointStride;
    o[0] = px * a.input_scaler;
    o[1] = py * a.input_scaler;
    o[2] = pz * a.input_scaler;
    float* geo = o + 3;
    const int o_cano = a.legacy_mode ? kJoints : 0;
    const int o_jd = a.legacy_mode ? 0 : 3;
    // joint distances / 2.4 (smpl.py:215)
#pragma unroll
    for (int j = 0; j < kJoints; ++j) {
      const float ex = px - sk[3 * j], ey = py - sk[3 * j + 1], ez = pz - sk[3 * j + 2];
      geo[o_jd + j] = sqrtf(ex * ex + ey * ey + ez * ez) / 2.4f;
    }
    // canonical point through the blended inverse transform of the nearest vertex (smpl.py:222-231)
    const float4* ik = reinterpret_cast<const float4*>(a.vertex_ik + (static_cast<long>(b) * a.V + bi) * 16);
    const float4 r0 = ik[0], r1 = ik[1], r2 = ik[2];
    const float cx = r0.x * px + r0.y * py + r0.z * pz + r0.w;
    const float cy = r1.x * px + r1.y * py + r1.z * pz + r1.w;
    const float cz = r2.x * px + r2.y * py + r2.z * pz + r2.w;
    geo[o_cano + 0] = cx / 2.f;
    geo[o_cano + 1] = (cy + 0.2f) / 2.f;
    geo[o_cano + 2] = cz / 1.3f;
    // canonical (T-pose) nearest vertex (smpl.py:233-235)
    const float* tv = a.tpose + (static_cast<long>(b) * a.V + bi) * 3;
    geo[27] = tv[0];
    geo[28] = tv[1];
    geo[29] = tv[2] / 0.2f;
    geo[30] = sqrtf(best) / 1.3f;  // smpl.py:237
    o[34] = 0.f;
    o[35] = 0.f;
  }
}

}  // namespace hg

extern "C" {

int hg_vertex_ik(const float* fk, const float* lbs, int B, int V, float* vertex_ik, void* stream) {
  HG_REQUIRE(fk && lbs && vertex_ik, "hg_vertex_ik: null pointer");
  HG_REQUIRE(B > 0 && V > 0, "hg_vertex_ik: bad shape B=%d V=%d", B, V);
  HG_REQUIRE((reinterpret_cast<uintptr_t>(vertex_ik) & 15) == 0, "hg_vertex_ik: output must be 16-byte aligned");
  dim3 grid((V + 127) / 128, B);
  hg::vertex_ik_kernel<<<grid, 128, 0, static_cast<cudaStream_t>(stream)>>>(fk, lbs, V, vertex_ik);
  return hg::check_launch("hg_vertex_ik");
}

// Morton-sort the posed vertices of every body and box them in clusters of 32 (exact KNN pruning).
// sorted: [B, Vp] float4, boxes: [B, Vp/32, 2] float4 with Vp = hg_knn_padded(V).
int hg_knn_padded(int V) { return (V + hg::kCluster - 1) / hg::kCluster * hg::kCluster; }

int hg_knn_prep(const float* vertices, int B, int V, void* sorted, void* boxes, void* stream) {
  HG_REQUIRE(vertices && sorted && boxes, "hg_knn_prep: null pointer");
  HG_REQUIRE(B > 0 && V > 0 && V <= hg::kSortN, "hg_knn_prep: need 0 < V <= %d (got %d)", hg::kSortN, V);
  HG_REQUIRE((reinterpret_cast<uintptr_t>(sorted) & 15) == 0 && (reinterpret_cast<uintptr_t>(boxes) & 15) == 0,
             "hg_knn_prep: outputs must be 16-byte aligned");
  const int smem = hg::kSortN * 8;
  cudaError_t e = cudaFuncSetAttribute(hg::knn_prep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) { hg::set_error("hg_knn_prep: smem opt-in failed: %s", cudaGetErrorString(e)); return 2; }
  hg::knn_prep_kernel<<<B, 1024, smem, static_cast<cudaStream_t>(stream)>>>(
      vertices, V, hg_knn_padded(V), static_cast<float4*>(sorted), static_cast<float4*>(boxes));
  return hg::check_launch("hg_knn_prep");
}

// See include/hg3d.h for the argument contract.
int hg_geo_features(const float* xs, const float* ys, const float* zs, const float* focals, const float* scales,
                    const float* cam2world, const float* jitter, const float* points_in, const float* skeletons,
                    const float* vertices, const float* tpose, const float* vertex_ik, const void* knn_sorted,
                    const void* knn_boxes, int B, int Rw, int Rh, int S,
                    int V, int n_points, float input_scaler, int legacy_mode, float* rec, float* z_vals,
                    float* points, int* nearest, float* nearest_d2, void* stream) {
  HG_REQUIRE(skeletons && vertices && tpose && vertex_ik && rec, "hg_geo_features: null pointer");
  HG_REQUIRE(B > 0 && V > 0 && n_points > 0, "hg_geo_features: bad shape B=%d V=%d N=%d", B, V, n_points);
  HG_REQUIRE(static_cast<size_t>(V) * 17 <= 200 * 1024, "hg_geo_features: V=%d does not fit in shared memory", V);
  if (!points_in) {
    HG_REQUIRE(xs && ys && zs && focals && scales && cam2world, "hg_geo_features: ray tables missing");
    HG_REQUIRE(Rw > 0 && Rh > 0 && S > 1 && n_points == Rw * Rh * S, "hg_geo_features: n_points != Rw*Rh*S");
  }
  HG_REQUIRE((reinterpret_cast<uintptr_t>(vertex_ik) & 15) == 0, "hg_geo_features: vertex_ik must be 16-byte aligned");
  HG_REQUIRE((knn_sorted == nullptr) == (knn_boxes == nullptr), "hg_geo_features: knn_sorted and knn_boxes go together");
  const int Vp = hg_knn_padded(V);
  hg::GeoArgs a{xs, ys, zs, focals, scales, cam2world, jitter, points_in, skeletons, vertices, tpose, vertex_ik,
                static_cast<const float4*>(knn_sorted), static_cast<const float4*>(knn_boxes), Vp,
                B, Rw, Rh, S, V, n_points, input_scaler, legacy_mode, rec, z_vals, points, nearest, nearest_d2};
  const size_t smem = knn_sorted ? (static_cast<size_t>(Vp) + 2 * (Vp / hg::kCluster)) * sizeof(float4)
                                 : static_cast<size_t>(V) * sizeof(float4);
  cudaError_t e = cudaFuncSetAttribute(hg::geo_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e != cudaSuccess) { hg::set_error("hg_geo_features: smem opt-in failed: %s", cudaGetErrorString(e)); return 2; }
  int bx = (n_points + hg::kGeoThreads - 1) / hg::kGeoThreads;
  const int per_body = hg::num_sms() / B > 0 ? hg::num_sms() / B : 1;   // one CTA per SM in total
  if (bx > per_body) bx = per_body;
  dim3 grid(bx, B);
  hg::geo_kernel<<<grid, hg::kGeoThreads, smem, static_cast<cudaStream_t>(stream)>>>(a);
  return hg::check_launch("hg_geo_features");
}

}  // extern "C"
