// SMPL label-map rasteriser: the segmentation targets of a training step, in place of pytorch3d's MeshRasterizer
// (`SHHQPreprocessor._forward_rasterize`, lib/data/preprocessor.py:138-176).  The contract restated here (pytorch3d 0.6.2,
// blur_radius = 0, faces_per_pixel = 1, no culling, perspective-correct barycentrics) is written out in oracle/raster_port.py,
// which reproduces every rounding below with one fp32 operation per step; DESIGN.md lists which parts are unpinned.
//   hg_raster_project  per vertex: X_view = X @ R + T (row vector), x_ndc = f X / Z, y_ndc = f Y / Z, keep view z
//   hg_raster_faces    per face (large boxes spread over the warp): z-buffer by one 64-bit atomicMin on
//                      (float bits of pz) << 32 | face -- nearest wins, ties to the lowest face, independent of launch order
//   hg_raster_resolve  per pixel: decode the face, recompute its barycentrics, first-maximum vertex, labels / semantics
#include "common.cuh"

namespace hg {

constexpr float kRasterEps = 1e-8f;       // pytorch3d's kEpsilon
constexpr int kRasterSmallBox = 32;       // boxes with more pixels are rasterised by the whole warp
constexpr unsigned long long kRasterEmpty = ~0ull;

// pixel index -> NDC centre: the shorter side spans [-1, 1], the longer +-(long / short)
__device__ __forceinline__ float raster_pix_ndc(int i, int S1, int S2) {
  float range = 2.0f;
  if (S1 > S2) range = __fdiv_rn(__fmul_rn(static_cast<float>(S1), range), static_cast<float>(S2));
  const float offset = __fdiv_rn(range, 2.0f);
  return __fadd_rn(-offset, __fdiv_rn(__fadd_rn(__fmul_rn(range, static_cast<float>(i)), offset), static_cast<float>(S1)));
}

// (p - v0) x (v1 - v0) in pytorch3d's operand order
__device__ __forceinline__ float raster_edge(float px, float py, float ax, float ay, float bx, float by) {
  return __fsub_rn(__fmul_rn(__fsub_rn(px, ax), __fsub_rn(by, ay)), __fmul_rn(__fsub_rn(py, ay), __fsub_rn(bx, ax)));
}

struct RasterTri {
  float x0, y0, z0, x1, y1, z1, x2, y2, z2;
};

// perspective-corrected barycentrics of the pixel centre (px, py); returns pz
__device__ __forceinline__ float raster_bary(const RasterTri& t, float px, float py, float& w0, float& w1, float& w2) {
  const float area = __fadd_rn(raster_edge(t.x2, t.y2, t.x0, t.y0, t.x1, t.y1), kRasterEps);
  const float b0 = __fdiv_rn(raster_edge(px, py, t.x1, t.y1, t.x2, t.y2), area);
  const float b1 = __fdiv_rn(raster_edge(px, py, t.x2, t.y2, t.x0, t.y0), area);
  const float b2 = __fdiv_rn(raster_edge(px, py, t.x0, t.y0, t.x1, t.y1), area);
  const float t0 = __fmul_rn(__fmul_rn(b0, t.z1), t.z2);
  const float t1 = __fmul_rn(__fmul_rn(t.z0, b1), t.z2);
  const float t2 = __fmul_rn(__fmul_rn(t.z0, t.z1), b2);
  const float denom = fmaxf(__fadd_rn(__fadd_rn(t0, t1), t2), kRasterEps);
  w0 = __fdiv_rn(t0, denom);
  w1 = __fdiv_rn(t1, denom);
  w2 = __fdiv_rn(t2, denom);
  return __fadd_rn(__fadd_rn(__fmul_rn(w0, t.z0), __fmul_rn(w1, t.z1)), __fmul_rn(w2, t.z2));
}

__device__ __forceinline__ RasterTri raster_load(const float* __restrict__ proj, const long long* __restrict__ faces, int b, int f, int V,
                                                 bool& ok) {
  RasterTri t;
  float* o = &t.x0;
  ok = true;
  for (int k = 0; k < 3; ++k) {
    const long long v = faces[static_cast<long>(f) * 3 + k];
    ok &= v >= 0 && v < V;
    const float* p = proj + (static_cast<long>(b) * V + (ok ? v : 0)) * 3;
    o[k * 3 + 0] = p[0];
    o[k * 3 + 1] = p[1];
    o[k * 3 + 2] = p[2];
  }
  return t;
}

__global__ void __launch_bounds__(256) raster_project_kernel(const float* __restrict__ verts, const float* __restrict__ R,
                                                             const float* __restrict__ T, float focal, float* __restrict__ proj,
                                                             int V) {
  const int b = blockIdx.y, v = blockIdx.x * 256 + threadIdx.x;
  if (v >= V) return;
  const float* X = verts + (static_cast<long>(b) * V + v) * 3;
  const float* r = R + b * 9;
  const float* t = T + b * 3;
  float xv[3];
#pragma unroll
  for (int j = 0; j < 3; ++j)
    xv[j] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(X[0], r[j]), __fmul_rn(X[1], r[3 + j])), __fmul_rn(X[2], r[6 + j])), t[j]);
  float* o = proj + (static_cast<long>(b) * V + v) * 3;
  o[0] = __fdiv_rn(__fmul_rn(focal, xv[0]), xv[2]);
  o[1] = __fdiv_rn(__fmul_rn(focal, xv[1]), xv[2]);
  o[2] = xv[2];
}

// one pixel of one face: bbox test, barycentrics, inside (strict), pz >= 0, z-buffer
__device__ __forceinline__ void raster_pixel(const RasterTri& t, float xmin, float xmax, float ymin, float ymax, int f, int yi, int xi,
                                             int H, int W, unsigned long long* __restrict__ zrow) {
  const float px = raster_pix_ndc(W - 1 - xi, W, H), py = raster_pix_ndc(H - 1 - yi, H, W);
  if (px > xmax || px < xmin || py > ymax || py < ymin) return;
  float w0, w1, w2;
  float pz = raster_bary(t, px, py, w0, w1, w2);
  if (pz < 0.f || !(w0 > 0.f && w1 > 0.f && w2 > 0.f)) return;
  if (pz == 0.f) pz = 0.f;                                      // -0 -> +0: non-negative floats order as their bits
  atomicMin(zrow + static_cast<long>(yi) * W + xi, (static_cast<unsigned long long>(__float_as_uint(pz)) << 32) | static_cast<unsigned>(f));
}

// conservative column / row range of [lo, hi] in NDC (one pixel of margin; raster_pixel applies the exact test)
__device__ __forceinline__ void raster_span(float lo, float hi, int S1, int S2, int& a, int& b) {
  const float range = S1 > S2 ? 2.0f * S1 / S2 : 2.0f;
  const float off = 0.5f * range;
  float ilo = floorf(((lo + off) * S1 - off) / range) - 1.f;    // NDC index i (increasing with the coordinate)
  float ihi = ceilf(((hi + off) * S1 - off) / range) + 1.f;
  ilo = fminf(fmaxf(ilo, 0.f), static_cast<float>(S1));
  ihi = fminf(fmaxf(ihi, -1.f), static_cast<float>(S1 - 1));
  // pixel index = S1 - 1 - i (+X left, +Y up)
  a = S1 - 1 - static_cast<int>(ihi);
  b = S1 - 1 - static_cast<int>(ilo);
}

__global__ void __launch_bounds__(256) raster_faces_kernel(const float* __restrict__ proj, const long long* __restrict__ faces, int V,
                                                           int F, int H, int W, unsigned long long* __restrict__ zkey) {
  const int b = blockIdx.y, f = blockIdx.x * 256 + threadIdx.x;
  const int lane = threadIdx.x & 31;
  unsigned long long* zrow = zkey + static_cast<long>(b) * H * W;
  RasterTri t{};
  bool ok = false;
  float xmin = 0.f, xmax = 0.f, ymin = 0.f, ymax = 0.f;
  int xa = 0, xb = -1, ya = 0, yb = -1;
  if (f < F) {
    t = raster_load(proj, faces, b, f, V, ok);
    const float zmax = fmaxf(t.z0, fmaxf(t.z1, t.z2));
    const float area = raster_edge(t.x0, t.y0, t.x1, t.y1, t.x2, t.y2);
    xmin = fminf(t.x0, fminf(t.x1, t.x2));
    xmax = fmaxf(t.x0, fmaxf(t.x1, t.x2));
    ymin = fminf(t.y0, fminf(t.y1, t.y2));
    ymax = fmaxf(t.y0, fmaxf(t.y1, t.y2));
    // behind the camera, zero area (|area| <= eps), or a non-finite box (no pixel can pass the barycentric test)
    ok &= !(zmax < 0.f) && !(area <= kRasterEps && area >= -kRasterEps) && isfinite(xmin) && isfinite(xmax) && isfinite(ymin) &&
          isfinite(ymax) && isfinite(area);
    if (ok) {
      raster_span(xmin, xmax, W, H, xa, xb);
      raster_span(ymin, ymax, H, W, ya, yb);
    }
  }
  const int nx = xb - xa + 1, ny = yb - ya + 1;
  const int count = (ok && nx > 0 && ny > 0) ? nx * ny : 0;
  if (count > 0 && count <= kRasterSmallBox) {
    for (int yi = ya; yi <= yb; ++yi)
      for (int xi = xa; xi <= xb; ++xi) raster_pixel(t, xmin, xmax, ymin, ymax, f, yi, xi, H, W, zrow);
  }
  unsigned big = __ballot_sync(0xffffffffu, count > kRasterSmallBox);
  while (big) {
    const int src = __ffs(big) - 1;
    big &= big - 1;
    RasterTri s;
    float* so = &s.x0;
    const float* to = &t.x0;
#pragma unroll
    for (int k = 0; k < 9; ++k) so[k] = __shfl_sync(0xffffffffu, to[k], src);
    const float sxmin = __shfl_sync(0xffffffffu, xmin, src), sxmax = __shfl_sync(0xffffffffu, xmax, src);
    const float symin = __shfl_sync(0xffffffffu, ymin, src), symax = __shfl_sync(0xffffffffu, ymax, src);
    const int sf = __shfl_sync(0xffffffffu, f, src), sxa = __shfl_sync(0xffffffffu, xa, src);
    const int sya = __shfl_sync(0xffffffffu, ya, src), snx = __shfl_sync(0xffffffffu, nx, src);
    const int scount = __shfl_sync(0xffffffffu, count, src);
    for (int p = lane; p < scount; p += 32) raster_pixel(s, sxmin, sxmax, symin, symax, sf, sya + p / snx, sxa + p % snx, H, W, zrow);
  }
}

__global__ void __launch_bounds__(256) raster_resolve_kernel(const float* __restrict__ proj, const long long* __restrict__ faces,
                                                             const long long* __restrict__ labels, const float* __restrict__ tpose0,
                                                             const unsigned long long* __restrict__ zkey, int V, int F, int H, int W,
                                                             long long* __restrict__ segments, float* __restrict__ semantics,
                                                             long long* __restrict__ pix_to_face, float* __restrict__ zbuf,
                                                             float* __restrict__ bary) {
  const int b = blockIdx.y, pix = blockIdx.x * 256 + threadIdx.x;
  const int HW = H * W;
  if (pix >= HW) return;
  const long o = static_cast<long>(b) * HW + pix;
  const unsigned long long key = zkey[o];
  float* sem = semantics + static_cast<long>(b) * 3 * HW + pix;
  if (key == kRasterEmpty) {
    segments[o] = 1;
    sem[0] = sem[HW] = sem[2 * HW] = 0.f;
    if (pix_to_face) pix_to_face[o] = -1;
    if (zbuf) zbuf[o] = -1.f;
    if (bary) bary[o * 3] = bary[o * 3 + 1] = bary[o * 3 + 2] = -1.f;
    return;
  }
  const int f = static_cast<int>(key & 0xffffffffu);
  bool ok;
  const RasterTri t = raster_load(proj, faces, b, f, V, ok);
  const int yi = pix / W, xi = pix - yi * W;
  float w[3];
  raster_bary(t, raster_pix_ndc(W - 1 - xi, W, H), raster_pix_ndc(H - 1 - yi, H, W), w[0], w[1], w[2]);
  int j = 0;                                                     // first maximum (torch.argmax)
  if (w[1] > w[j]) j = 1;
  if (w[2] > w[j]) j = 2;
  const long long vert = faces[static_cast<long>(f) * 3 + j];
  segments[o] = labels[f] + 2;
  sem[0] = tpose0[vert * 3 + 0];
  sem[HW] = tpose0[vert * 3 + 1];
  sem[2 * HW] = tpose0[vert * 3 + 2];
  if (pix_to_face) pix_to_face[o] = static_cast<long long>(b) * F + f;
  if (zbuf) zbuf[o] = __uint_as_float(static_cast<unsigned>(key >> 32));
  if (bary) {
    bary[o * 3] = w[0];
    bary[o * 3 + 1] = w[1];
    bary[o * 3 + 2] = w[2];
  }
}

}  // namespace hg

extern "C" {

// proj [B,V,3] = (f X/Z, f Y/Z, Z) of X_view = verts [B,V,3] @ R [B,3,3] + T [B,3]
int hg_raster_project(const float* verts, const float* R, const float* T, float focal, float* proj, int B, int V, void* stream) {
  HG_REQUIRE(verts && R && T && proj, "hg_raster_project: null pointer");
  HG_REQUIRE(B > 0 && V > 0, "hg_raster_project: bad sizes");
  dim3 grid((V + 255) / 256, B);
  hg::raster_project_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(verts, R, T, focal, proj, V);
  return hg::check_launch("hg_raster_project");
}

// zkey [B,H,W] u64 is cleared here, then holds (pz bits << 32 | face) of the nearest covering face, or ~0 for background
int hg_raster_faces(const float* proj, const long long* faces, int B, int V, int F, int H, int W, unsigned long long* zkey, void* stream) {
  HG_REQUIRE(proj && faces && zkey, "hg_raster_faces: null pointer");
  HG_REQUIRE(B > 0 && V > 0 && F > 0 && H > 0 && W > 0 && static_cast<long>(H) * W <= (1l << 30), "hg_raster_faces: bad sizes");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaMemsetAsync(zkey, 0xff, static_cast<size_t>(B) * H * W * sizeof(unsigned long long), s);
  if (e != cudaSuccess) { hg::set_error("hg_raster_faces: clearing the z-buffer failed: %s", cudaGetErrorString(e)); return 2; }
  dim3 grid((F + 255) / 256, B);
  hg::raster_faces_kernel<<<grid, 256, 0, s>>>(proj, faces, V, F, H, W, zkey);
  return hg::check_launch("hg_raster_faces");
}

// segments [B,H,W] int64 = labels[face] + 2 (1 = background); semantics [B,3,H,W] = tpose0[vertex of the largest barycentric]
// (0 = background); pix_to_face [B,H,W] int64 (b*F + face, -1), zbuf [B,H,W], bary [B,H,W,3] (-1 on background) may be NULL
int hg_raster_resolve(const float* proj, const long long* faces, const long long* faces_to_labels, const float* tpose0,
                      const unsigned long long* zkey, int B, int V, int F, int H, int W, long long* segments, float* semantics,
                      long long* pix_to_face, float* zbuf, float* bary, void* stream) {
  HG_REQUIRE(proj && faces && faces_to_labels && tpose0 && zkey && segments && semantics, "hg_raster_resolve: null pointer");
  HG_REQUIRE(B > 0 && V > 0 && F > 0 && H > 0 && W > 0 && static_cast<long>(H) * W <= (1l << 30), "hg_raster_resolve: bad sizes");
  dim3 grid((H * W + 255) / 256, B);
  hg::raster_resolve_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(proj, faces, faces_to_labels, tpose0, zkey, V, F, H, W,
                                                                                 segments, semantics, pix_to_face, zbuf, bary);
  return hg::check_launch("hg_raster_resolve");
}

}  // extern "C"
