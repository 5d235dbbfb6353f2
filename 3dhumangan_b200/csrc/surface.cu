// Iso-surface of a scalar lattice by marching tetrahedra over the Kuhn (Freudenthal) split of every cell -- the
// geometry extractor of pi-GAN-style generators (density lattice -> mesh), here for `surface.extract_mesh`.
//
//   hg_iso_count   per lattice point the 7-bit crossing mask of the edges it owns, per cell the triangle count, then the
//                  int64 exclusive scans of both (reduce / scan of block sums / apply) and the two totals
//   hg_iso_emit    vertices + normals in (point, edge slot) order and faces in (cell, tet, triangle) order
//
// Output positions come from the scans only (no atomics), so two calls write the same bits.  The rule is restated in numpy
// by tests/surface_oracle.py; the header (include/hg3d.h) states it in full.
#include "common.cuh"

namespace hg {

constexpr int kIsoThreads = 256;
constexpr int kIsoPerThread = 16;
constexpr int kIsoTile = kIsoThreads * kIsoPerThread;    // elements per scan block
constexpr int kIsoScanThreads = 1024;

// edge slot of a 0/1 direction given as bits (x = 1, y = 2, z = 4): x, y, z, x+y, x+z, y+z, x+y+z
__device__ __constant__ int8_t kSlotOfBits[8] = {-1, 0, 1, 3, 2, 4, 5, 6};
__device__ __constant__ int8_t kBitsOfSlot[7] = {1, 2, 4, 3, 5, 6, 7};
// Kuhn tets: axis permutations in lexicographic order (0 = x, 1 = y, 2 = z) and their parities (+1 even)
__device__ __constant__ int8_t kTetPerm[6][2] = {{0, 1}, {0, 2}, {1, 0}, {1, 2}, {2, 0}, {2, 1}};
__device__ __constant__ int8_t kTetSign[6] = {1, -1, -1, 1, 1, -1};

struct IsoDims {
  int nx, ny, nz;
  long n;   // nx * ny * nz
};

__device__ __forceinline__ bool iso_in(const float* lat, long i, float level) { return lat[i] > level; }

// inside bits of the 8 corners of the cell at (x, y, z), corner k = (k & 1, k >> 1 & 1, k >> 2 & 1)
__device__ __forceinline__ int corner_bits(const float* lat, const IsoDims& d, int x, int y, int z, float level) {
  const long sx = 1, sy = d.nx, sz = static_cast<long>(d.nx) * d.ny;
  const long base = z * sz + y * sy + x;
  int bits = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k)
    bits |= static_cast<int>(iso_in(lat, base + (k & 1) * sx + (k >> 1 & 1) * sy + (k >> 2 & 1) * sz, level)) << k;
  return bits;
}

// corner (bits x=1 y=2 z=4) of vertex v of tet t: u0 = 0, u1 = e_a, u2 = e_a + e_b, u3 = (1,1,1)
__device__ __forceinline__ int tet_corner(int t, int v) {
  const int ea = 1 << kTetPerm[t][0], eb = 1 << kTetPerm[t][1];
  return v == 0 ? 0 : v == 1 ? ea : v == 2 ? (ea | eb) : 7;
}

__device__ __forceinline__ int tri_count(int cbits) {
  int n = 0;
#pragma unroll
  for (int t = 0; t < 6; ++t) {
    int k = 0;
#pragma unroll
    for (int v = 0; v < 4; ++v) k += cbits >> tet_corner(t, v) & 1;
    n += (k == 1 || k == 3) ? 1 : (k == 2 ? 2 : 0);
  }
  return n;
}

__global__ void __launch_bounds__(kIsoThreads) iso_count_kernel(const float* __restrict__ lat, IsoDims d, float level,
                                                                uint8_t* __restrict__ mask, uint8_t* __restrict__ tcount) {
  for (long p = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; p < d.n; p += static_cast<long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(p % d.nx);
    const long r = p / d.nx;
    const int y = static_cast<int>(r % d.ny), z = static_cast<int>(r / d.ny);
    const bool a = iso_in(lat, p, level);
    int m = 0;
#pragma unroll
    for (int s = 0; s < 7; ++s) {
      const int b = kBitsOfSlot[s];
      const int dx = b & 1, dy = b >> 1 & 1, dz = b >> 2 & 1;
      if (x + dx < d.nx && y + dy < d.ny && z + dz < d.nz) {
        const long q = p + dx + static_cast<long>(dy) * d.nx + static_cast<long>(dz) * d.nx * d.ny;
        m |= static_cast<int>(a != iso_in(lat, q, level)) << s;
      }
    }
    mask[p] = static_cast<uint8_t>(m);
    int tc = 0;
    if (x + 1 < d.nx && y + 1 < d.ny && z + 1 < d.nz) {
      const int cb = corner_bits(lat, d, x, y, z, level);
      if (cb != 0 && cb != 255) tc = tri_count(cb);
    }
    tcount[p] = static_cast<uint8_t>(tc);
  }
}

// ---- int64 exclusive scan of popcount(mask) and tcount: block sums, one-block scan of the sums, apply ----------------
__device__ __forceinline__ int2 iso_vals(const uint8_t* mask, const uint8_t* tcount, long i, long n) {
  return i < n ? make_int2(__popc(mask[i]), tcount[i]) : make_int2(0, 0);
}

// exclusive block scan of one int per thread (values small: a tile holds at most 12 * 4096 triangles)
__device__ __forceinline__ int2 block_exclusive(int2 v, int2* warp_tot, int2& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int2 inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int ax = __shfl_up_sync(0xffffffffu, inc.x, o), ay = __shfl_up_sync(0xffffffffu, inc.y, o);
    if (lane >= o) inc.x += ax, inc.y += ay;
  }
  if (lane == 31) warp_tot[warp] = inc;
  __syncthreads();
  int2 before = make_int2(0, 0);
  total = make_int2(0, 0);
  for (int w = 0; w < nw; ++w) {
    if (w < warp) before.x += warp_tot[w].x, before.y += warp_tot[w].y;
    total.x += warp_tot[w].x, total.y += warp_tot[w].y;
  }
  __syncthreads();
  return make_int2(before.x + inc.x - v.x, before.y + inc.y - v.y);
}

__global__ void __launch_bounds__(kIsoThreads) iso_scan_reduce_kernel(const uint8_t* __restrict__ mask, const uint8_t* __restrict__ tcount,
                                                                      long n, long long* __restrict__ bsum) {
  __shared__ int2 warp_tot[kIsoThreads / 32];
  const long base = static_cast<long>(blockIdx.x) * kIsoTile + static_cast<long>(threadIdx.x) * kIsoPerThread;
  int2 s = make_int2(0, 0);
#pragma unroll
  for (int i = 0; i < kIsoPerThread; ++i) {
    const int2 v = iso_vals(mask, tcount, base + i, n);
    s.x += v.x, s.y += v.y;
  }
  int2 total;
  block_exclusive(s, warp_tot, total);
  if (threadIdx.x == 0) {
    bsum[2 * blockIdx.x] = total.x;
    bsum[2 * blockIdx.x + 1] = total.y;
  }
}

// one block: exclusive scan of the nblk (vertex, triangle) block sums in place; totals[0..1] = (V, F)
__global__ void __launch_bounds__(kIsoScanThreads) iso_scan_blocks_kernel(long long* __restrict__ bsum, long nblk,
                                                                          long long* __restrict__ totals) {
  __shared__ long long wv[kIsoScanThreads / 32], wt[kIsoScanThreads / 32];
  __shared__ long long carry[2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry[0] = carry[1] = 0;
  __syncthreads();
  for (long c0 = 0; c0 < nblk; c0 += kIsoScanThreads) {
    const long i = c0 + threadIdx.x;
    const long long v = i < nblk ? bsum[2 * i] : 0, t = i < nblk ? bsum[2 * i + 1] : 0;
    long long iv = v, it = t;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long av = __shfl_up_sync(0xffffffffu, iv, o), at = __shfl_up_sync(0xffffffffu, it, o);
      if (lane >= o) iv += av, it += at;
    }
    if (lane == 31) wv[warp] = iv, wt[warp] = it;
    __syncthreads();
    long long bv = carry[0], bt = carry[1], sv = 0, st = 0;
    for (int w = 0; w < kIsoScanThreads / 32; ++w) {
      if (w < warp) bv += wv[w], bt += wt[w];
      sv += wv[w], st += wt[w];
    }
    if (i < nblk) {
      bsum[2 * i] = bv + iv - v;
      bsum[2 * i + 1] = bt + it - t;
    }
    __syncthreads();
    if (threadIdx.x == 0) carry[0] += sv, carry[1] += st;
    __syncthreads();
  }
  if (threadIdx.x == 0) totals[0] = carry[0], totals[1] = carry[1];
}

__global__ void __launch_bounds__(kIsoThreads) iso_scan_apply_kernel(const uint8_t* __restrict__ mask, const uint8_t* __restrict__ tcount,
                                                                     long n, const long long* __restrict__ bsum,
                                                                     long long* __restrict__ voff, long long* __restrict__ toff) {
  __shared__ int2 warp_tot[kIsoThreads / 32];
  const long base = static_cast<long>(blockIdx.x) * kIsoTile + static_cast<long>(threadIdx.x) * kIsoPerThread;
  int2 vals[kIsoPerThread];
  int2 s = make_int2(0, 0);
#pragma unroll
  for (int i = 0; i < kIsoPerThread; ++i) {
    vals[i] = iso_vals(mask, tcount, base + i, n);
    s.x += vals[i].x, s.y += vals[i].y;
  }
  int2 total;
  const int2 ex = block_exclusive(s, warp_tot, total);
  long long ov = bsum[2 * blockIdx.x] + ex.x, ot = bsum[2 * blockIdx.x + 1] + ex.y;
#pragma unroll
  for (int i = 0; i < kIsoPerThread; ++i) {
    if (base + i < n) {
      voff[base + i] = ov;
      toff[base + i] = ot;
    }
    ov += vals[i].x, ot += vals[i].y;
  }
}

// ---- emit ------------------------------------------------------------------------------------------------------------
// -grad by central differences in index units (one-sided at the border), every operation rounded on its own
__device__ __forceinline__ float3 iso_grad(const float* lat, const IsoDims& d, int x, int y, int z) {
  const long sy = d.nx, sz = static_cast<long>(d.nx) * d.ny;
  const long p = z * sz + y * sy + x;
  auto diff = [&](int c, int n, long st) {
    if (c == 0) return __fsub_rn(lat[p + st], lat[p]);
    if (c == n - 1) return __fsub_rn(lat[p], lat[p - st]);
    return __fmul_rn(__fsub_rn(lat[p + st], lat[p - st]), 0.5f);
  };
  return make_float3(diff(x, d.nx, 1), diff(y, d.ny, sy), diff(z, d.nz, sz));
}

__device__ __forceinline__ float lerp_rn(float a, float b, float t) { return __fadd_rn(a, __fmul_rn(t, __fsub_rn(b, a))); }

// vertex index of the tet edge (u_i, u_j), i < j: owned by corner u_i, direction u_j - u_i
__device__ __forceinline__ long long edge_vertex(int t, int i, int j, const int* owner_mask, const long long* owner_off) {
  const int ci = tet_corner(t, i), cj = tet_corner(t, j);
  const int slot = kSlotOfBits[cj & ~ci];
  return owner_off[ci] + __popc(owner_mask[ci] & ((1 << slot) - 1));
}

__global__ void __launch_bounds__(kIsoThreads) iso_emit_kernel(const float* __restrict__ lat, IsoDims d, float3 origin, float h,
                                                               float level, const uint8_t* __restrict__ mask,
                                                               const uint8_t* __restrict__ tcount, const long long* __restrict__ voff,
                                                               const long long* __restrict__ toff, float* __restrict__ verts,
                                                               float* __restrict__ normals, int* __restrict__ faces) {
  for (long p = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; p < d.n; p += static_cast<long>(gridDim.x) * blockDim.x) {
    const int m = mask[p], tc = tcount[p];
    if (m == 0 && tc == 0) continue;
    const int x = static_cast<int>(p % d.nx);
    const long r = p / d.nx;
    const int y = static_cast<int>(r % d.ny), z = static_cast<int>(r / d.ny);
    const long sy = d.nx, sz = static_cast<long>(d.nx) * d.ny;
    if (m) {
      const float va = lat[p];
      const float3 ga = iso_grad(lat, d, x, y, z);
      long long o = voff[p];
      for (int s = 0; s < 7; ++s) {
        if (!(m >> s & 1)) continue;
        const int b = kBitsOfSlot[s];
        const int dx = b & 1, dy = b >> 1 & 1, dz = b >> 2 & 1;
        const float vb = lat[p + dx + dy * sy + dz * sz];
        const float t = __fdiv_rn(__fsub_rn(level, va), __fsub_rn(vb, va));
        const float3 gb = iso_grad(lat, d, x + dx, y + dy, z + dz);
        float* vo = verts + 3 * o;
        vo[0] = __fadd_rn(origin.x, __fmul_rn(h, dx ? __fadd_rn(static_cast<float>(x), t) : static_cast<float>(x)));
        vo[1] = __fadd_rn(origin.y, __fmul_rn(h, dy ? __fadd_rn(static_cast<float>(y), t) : static_cast<float>(y)));
        vo[2] = __fadd_rn(origin.z, __fmul_rn(h, dz ? __fadd_rn(static_cast<float>(z), t) : static_cast<float>(z)));
        const float nx = lerp_rn(ga.x, gb.x, t), ny = lerp_rn(ga.y, gb.y, t), nz = lerp_rn(ga.z, gb.z, t);
        const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(nx, nx), __fmul_rn(ny, ny)), __fmul_rn(nz, nz)));
        float* no = normals + 3 * o;
        no[0] = len > 0.f ? -__fdiv_rn(nx, len) : 0.f;
        no[1] = len > 0.f ? -__fdiv_rn(ny, len) : 0.f;
        no[2] = len > 0.f ? -__fdiv_rn(nz, len) : 0.f;
        ++o;
      }
    }
    if (tc) {
      const int cb = corner_bits(lat, d, x, y, z, level);
      // masks / offsets of the corners that own tet edges (u0, u1, u2 of every tet: every corner but (1,1,1))
      int cmask[7];
      long long coff[7];
#pragma unroll
      for (int k = 0; k < 7; ++k) {
        const long q = p + (k & 1) + (k >> 1 & 1) * sy + (k >> 2 & 1) * sz;
        cmask[k] = mask[q];
        coff[k] = voff[q];
      }
      long long f = toff[p];
      for (int t = 0; t < 6; ++t) {
        int in[4], out[4], ni = 0, no = 0;
        for (int v = 0; v < 4; ++v) {
          if (cb >> tet_corner(t, v) & 1) in[ni++] = v;
          else out[no++] = v;
        }
        if (ni == 0 || ni == 4) continue;
        auto ev = [&](int a, int b) {
          return static_cast<int>(a < b ? edge_vertex(t, a, b, cmask, coff) : edge_vertex(t, b, a, cmask, coff));
        };
        int* fo = faces + 3 * f;
        if (ni == 2) {
          // (a, b, c, d) = (in ascending, out ascending); its parity times the tet's orientation fixes the winding
          const int a = in[0], b = in[1], c = out[0], e = out[1];
          int inv = 0;
          const int seq[4] = {a, b, c, e};
          for (int i = 0; i < 4; ++i)
            for (int j = i + 1; j < 4; ++j) inv += seq[i] > seq[j];
          const int sgn = kTetSign[t] * ((inv & 1) ? -1 : 1);
          const int q0 = ev(a, c), q1 = ev(a, e), q2 = ev(b, e), q3 = ev(b, c);
          if (sgn > 0) {
            fo[0] = q0, fo[1] = q1, fo[2] = q2, fo[3] = q0, fo[4] = q2, fo[5] = q3;
          } else {
            fo[0] = q0, fo[1] = q2, fo[2] = q1, fo[3] = q0, fo[4] = q3, fo[5] = q2;
          }
          f += 2;
        } else {
          // the lone vertex i (inside when ni == 1, outside when ni == 3), the others j < k < l: (i, j, k, l) has parity i
          const int i = ni == 1 ? in[0] : out[0];
          const int* rest = ni == 1 ? out : in;
          const int sgn = kTetSign[t] * ((i & 1) ? -1 : 1) * (ni == 1 ? 1 : -1);
          const int e0 = ev(i, rest[0]), e1 = ev(i, rest[1]), e2 = ev(i, rest[2]);
          fo[0] = e0;
          fo[1] = sgn > 0 ? e1 : e2;
          fo[2] = sgn > 0 ? e2 : e1;
          f += 1;
        }
      }
    }
  }
}

inline int iso_grid(long n) {
  const long want = (n + kIsoThreads - 1) / kIsoThreads;
  const long cap = static_cast<long>(num_sms()) * 16;
  return static_cast<int>(want < cap ? want : cap);
}

struct IsoWorkspace {
  long long* voff;
  long long* toff;
  long long* bsum;
  uint8_t* mask;
  uint8_t* tcount;
};

inline long iso_blocks(long n) { return (n + kIsoTile - 1) / kIsoTile; }

inline size_t iso_workspace_bytes(long n) {
  return static_cast<size_t>(8 * (2 * n + 2 * iso_blocks(n)) + ((2 * n + 15) & ~15L));
}

inline IsoWorkspace iso_carve(void* ws, long n) {
  auto* w = static_cast<long long*>(ws);
  IsoWorkspace c;
  c.voff = w;
  c.toff = w + n;
  c.bsum = w + 2 * n;
  c.mask = reinterpret_cast<uint8_t*>(c.bsum + 2 * iso_blocks(n));
  c.tcount = c.mask + n;
  return c;
}

constexpr long kIsoMaxPoints = 1L << 30;

}  // namespace hg

extern "C" {

size_t hg_iso_workspace_bytes(int nz, int ny, int nx) {
  if (nz < 2 || ny < 2 || nx < 2) return 0;
  const long n = static_cast<long>(nz) * ny * nx;
  return n > hg::kIsoMaxPoints ? 0 : hg::iso_workspace_bytes(n);
}

int hg_iso_count(const float* lattice, int nz, int ny, int nx, float level, void* workspace, size_t workspace_bytes,
                 long long* totals, void* stream) {
  HG_REQUIRE(lattice && workspace && totals, "hg_iso_count: null pointer");
  HG_REQUIRE(nz >= 2 && ny >= 2 && nx >= 2, "hg_iso_count: every lattice axis needs >= 2 points (got %d x %d x %d)", nz, ny, nx);
  const long n = static_cast<long>(nz) * ny * nx;
  HG_REQUIRE(n <= hg::kIsoMaxPoints, "hg_iso_count: %ld lattice points, at most 2^30 are supported", n);
  HG_REQUIRE(workspace_bytes >= hg::iso_workspace_bytes(n), "hg_iso_count: workspace of %zu bytes, %zu needed", workspace_bytes,
             hg::iso_workspace_bytes(n));
  HG_REQUIRE(level == level, "hg_iso_count: level is NaN");
  auto st = static_cast<cudaStream_t>(stream);
  const hg::IsoDims d{nx, ny, nz, n};
  const hg::IsoWorkspace w = hg::iso_carve(workspace, n);
  hg::iso_count_kernel<<<hg::iso_grid(n), hg::kIsoThreads, 0, st>>>(lattice, d, level, w.mask, w.tcount);
  int rc = hg::check_launch("hg_iso_count(count)");
  if (rc) return rc;
  const long nblk = hg::iso_blocks(n);
  hg::iso_scan_reduce_kernel<<<static_cast<unsigned>(nblk), hg::kIsoThreads, 0, st>>>(w.mask, w.tcount, n, w.bsum);
  if ((rc = hg::check_launch("hg_iso_count(reduce)"))) return rc;
  hg::iso_scan_blocks_kernel<<<1, hg::kIsoScanThreads, 0, st>>>(w.bsum, nblk, totals);
  if ((rc = hg::check_launch("hg_iso_count(scan)"))) return rc;
  hg::iso_scan_apply_kernel<<<static_cast<unsigned>(nblk), hg::kIsoThreads, 0, st>>>(w.mask, w.tcount, n, w.bsum, w.voff, w.toff);
  return hg::check_launch("hg_iso_count(apply)");
}

int hg_iso_emit(const float* lattice, int nz, int ny, int nx, float ox, float oy, float oz, float spacing, float level,
                const void* workspace, size_t workspace_bytes, long long n_vertices, float* vertices, float* normals, int* faces,
                void* stream) {
  HG_REQUIRE(lattice && workspace, "hg_iso_emit: null pointer");
  HG_REQUIRE(nz >= 2 && ny >= 2 && nx >= 2, "hg_iso_emit: every lattice axis needs >= 2 points (got %d x %d x %d)", nz, ny, nx);
  const long n = static_cast<long>(nz) * ny * nx;
  HG_REQUIRE(n <= hg::kIsoMaxPoints, "hg_iso_emit: %ld lattice points, at most 2^30 are supported", n);
  HG_REQUIRE(workspace_bytes >= hg::iso_workspace_bytes(n), "hg_iso_emit: workspace of %zu bytes, %zu needed", workspace_bytes,
             hg::iso_workspace_bytes(n));
  HG_REQUIRE(n_vertices >= 0 && n_vertices < (1LL << 31), "hg_iso_emit: %lld vertices do not fit int32 face indices", n_vertices);
  HG_REQUIRE(n_vertices == 0 || (vertices && normals && faces), "hg_iso_emit: null output pointer");
  HG_REQUIRE(spacing > 0.f, "hg_iso_emit: spacing must be positive (got %g)", static_cast<double>(spacing));
  if (n_vertices == 0) return 0;
  auto st = static_cast<cudaStream_t>(stream);
  const hg::IsoDims d{nx, ny, nz, n};
  const hg::IsoWorkspace c = hg::iso_carve(const_cast<void*>(workspace), n);
  hg::iso_emit_kernel<<<hg::iso_grid(n), hg::kIsoThreads, 0, st>>>(lattice, d, make_float3(ox, oy, oz), spacing, level, c.mask,
                                                                    c.tcount, c.voff, c.toff, vertices, normals, faces);
  return hg::check_launch("hg_iso_emit");
}

}  // extern "C"
