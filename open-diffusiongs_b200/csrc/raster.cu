// raster.cu -- batched differentiable 3D-Gaussian-splatting rasterizer for sm_90a (H100).
//
// One launch set renders ALL (sample, view) pairs of a step: projection -> scan -> key emission ->
// one global radix sort keyed (view, tile, depth) -> tile ranges -> per-tile alpha blend; the backward
// walks the SAME sorted tile lists back-to-front (no re-render), reduces gradients inside the warp and
// the CTA before touching global memory, and folds camera construction and the exp / normalize /
// sigmoid activations (and their Jacobians) into the per-Gaussian kernels.
//
// Numerical specification = the reference rasterizer (DGR = submodules/diff-gaussian-rasterization):
//   projection   DGR/cuda_rasterizer/forward.cu:155-256, auxiliary.h:41-95,139-164
//   binning      DGR/cuda_rasterizer/rasterizer_impl.cu:70-138,277-317 (stable (tile,depth) order)
//   blend fwd    DGR/cuda_rasterizer/forward.cu:261-374
//   blend bwd    DGR/cuda_rasterizer/backward.cu:399-557
//   geometry bwd DGR/cuda_rasterizer/backward.cu:20-139,144-274,278-396
//   camera/activations  diffusionGS/models/gsrenderer/gs_core.py:277-316,330-334,545-570,874-945
// This file is an independent implementation (SoA float4 state, no glm, batched, fused); it shares
// only the math with the reference.
#include <cub/cub.cuh>

#include <cstring>
#include <type_traits>

#include "dgs_internal.h"
#include "sm90_ptx.cuh"

namespace dgs {

constexpr int TILE = 16;            // DGR/cuda_rasterizer/config.h:16-17
constexpr int TILE_PIX = TILE * TILE;
constexpr float NEAR_Z = 0.2f;      // auxiliary.h:154
constexpr float ALPHA_MIN = 1.0f / 255.0f;
constexpr float T_EPS = 0.0001f;

struct Camera {
  float view[16];  // [4c+r] = W2C[r][c]
  float proj[16];  // [4c+r] = (P W2C)[r][c]
  float campos[3];
  float tanx, tany, fx, fy;
  float pad;
};

struct Problem {
  int NV, V, P, D, M, W, H, gx, gy, tiles;
  int raw;  // 1: inputs are raw renderer tensors -> apply exp / normalize / sigmoid in-kernel
  int near_log2;  // > 0: two-phase binning, phase A = the nearest P >> near_log2 Gaussians of every view
  float mod;
  const float* means;
  const float* shs;
  const float* colors_pre;
  const float* opac;
  const float* scales;
  const float* rots;
  const float* cov_pre;
  float bg[3];
};

// Counters of one forward, written by the binning and blend kernels and read back by the host at its syncs
struct BinTotals {
  uint32_t R;              // instances of the batch (32-bit scan: R64 tells whether it wrapped)
  uint32_t R_near;         // two-phase: phase-A instances at the first near fraction (1/2^near_log2, adaptive 1/8)
  uint32_t unfinished;     // two-phase: tiles that still have an unsaturated pixel after phase A
  uint32_t longest;        // small-scene path: longest tile list
  unsigned long long R64;  // exact instance count
  uint32_t R_near_b;       // adaptive two-phase: phase-A instances at 1/16
  uint32_t pad;
};

struct GeomState {
  float4* g0;       // {x_pix, y_pix, depth, radius (int bits)}
  float4* g1;        // {conic A, B, C, opacity}
  float4* g2;        // {r, g, b, clamped bits}
  uint32_t* tiles;   // tiles touched, indexed by (view, Gaussian)
  // depth pre-sort: slot k of view v holds the k-th nearest Gaussian of that view (ties in index order)
  uint64_t* dkey_in;   // (view << 32) | depth bits
  uint64_t* dkey;      // sorted
  uint32_t* perm_in;   // Gaussian index (iota per view)
  uint32_t* perm;      // sorted: Gaussian index at each depth rank
  uint32_t* tiles_sorted;  // tiles touched in depth-rank order
  uint32_t* offsets;       // inclusive scan of tiles_sorted
  uint32_t* open_counts;   // phase B: open tiles touched per depth rank (0 for the near ranks) ...
  uint32_t* open_offsets;  // ... and their inclusive scan
  uint32_t* view_meta;     // [2][NV][2] two-phase binning, per candidate near fraction and view: where its near
                           // instances start in the global scan and in the compact phase-A buffer
  BinTotals* totals;
  Camera* cams;
  void* scan_temp;
  size_t scan_bytes;
  static GeomState carve(void* base, int NV, int P, size_t* total) {
    GeomState s;
    Carver c(base);
    size_t N = (size_t)NV * P;
    s.g0 = c.take<float4>(N);
    s.g1 = c.take<float4>(N);
    s.g2 = c.take<float4>(N);
    s.tiles = c.take<uint32_t>(N);
    s.dkey_in = c.take<uint64_t>(N);
    s.dkey = c.take<uint64_t>(N);
    s.perm_in = c.take<uint32_t>(N);
    s.perm = c.take<uint32_t>(N);
    s.tiles_sorted = c.take<uint32_t>(N);
    s.offsets = c.take<uint32_t>(N);
    s.open_counts = c.take<uint32_t>(N);
    s.open_offsets = c.take<uint32_t>(N);
    s.view_meta = c.take<uint32_t>((size_t)NV * 4);
    s.totals = c.take<BinTotals>(1);
    s.cams = c.take<Camera>(NV);
    size_t scan_b = 0, sort_b = 0;
    cub::DeviceScan::InclusiveSum(nullptr, scan_b, s.tiles_sorted, s.offsets, (int)N);
    cub::DeviceRadixSort::SortPairs(nullptr, sort_b, s.dkey_in, s.dkey, s.perm_in, s.perm, (int)N);
    s.scan_bytes = scan_b > sort_b ? scan_b : sort_b;  // shared temp: the two library calls run back to back
    s.scan_temp = c.take<char>(s.scan_bytes);
    if (total) *total = c.bytes();
    return s;
  }
};

struct BinState {
  uint32_t* keys_in;   // view * tiles + tile, emitted in (view, depth rank, tile) order
  uint32_t* keys;      // after the stable sort by tile
  uint32_t* vals_in;
  uint32_t* point_list;
  void* sort_temp;
  size_t sort_bytes;
  static BinState carve(void* base, long long R, size_t* total) {
    BinState s;
    Carver c(base);
    size_t n = (size_t)(R > 0 ? R : 1);
    s.point_list = c.take<uint32_t>(n);
    s.keys = c.take<uint32_t>(n);
    s.keys_in = c.take<uint32_t>(n);
    s.vals_in = c.take<uint32_t>(n);
    s.sort_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, s.sort_bytes, s.keys_in, s.keys, s.vals_in, s.point_list, (int)n);
    s.sort_temp = c.take<char>(s.sort_bytes);
    if (total) *total = c.bytes();
    return s;
  }
};

struct ImgState {
  float* final_T;
  uint32_t* n_contrib;
  uint2* ranges;
  uint2* ranges_b;     // phase-B tile ranges (two-phase binning)
  float4* acc;         // per-pixel blend state between the phases: {C.r, C.g, C.b, T}
  uint32_t* contrib;   // entries visited so far | (finished << 31)
  uint32_t* tile_open; // [views * tiles] 1 = the tile still has an unsaturated pixel after phase A
  static ImgState carve(void* base, int NV, int W, int H, size_t* total) {
    ImgState s;
    Carver c(base);
    size_t npix = (size_t)NV * W * H;
    size_t ntiles = (size_t)NV * ceil_div(W, TILE) * ceil_div(H, TILE);
    s.final_T = c.take<float>(npix);
    s.n_contrib = c.take<uint32_t>(npix);
    s.ranges = c.take<uint2>(ntiles);
    s.ranges_b = c.take<uint2>(ntiles);
    s.acc = c.take<float4>(npix);
    s.contrib = c.take<uint32_t>(npix);
    s.tile_open = c.take<uint32_t>(ntiles);
    if (total) *total = c.bytes();
    return s;
  }
};

// ---------------------------------------------------------------------------------------------
// device math shared by forward and backward
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float ndc_to_pix(float v, int S) {
  // auxiliary.h:41-44: the reference's literals are double, so this is evaluated in fp64
  return (float)((((double)v + 1.0) * (double)S - 1.0) * 0.5);
}

__device__ __forceinline__ void tile_rect(float px, float py, int radius, int gx, int gy, int& x0,
                                          int& y0, int& x1, int& y1) {  // auxiliary.h:46-56
  x0 = min(gx, max(0, (int)((px - radius) / TILE)));
  y0 = min(gy, max(0, (int)((py - radius) / TILE)));
  x1 = min(gx, max(0, (int)((px + radius + TILE - 1) / TILE)));
  y1 = min(gy, max(0, (int)((py + radius + TILE - 1) / TILE)));
}

__device__ __forceinline__ float3 xform43(const float* m, float3 p) {
  return make_float3(m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12], m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13],
                     m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14]);
}
__device__ __forceinline__ float4 xform44(const float* m, float3 p) {
  return make_float4(m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12], m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13],
                     m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14], m[3] * p.x + m[7] * p.y + m[11] * p.z + m[15]);
}

__device__ __forceinline__ void quat_to_rot(float4 q, float R[3][3]) {  // (r,x,y,z), not re-normalised
  float r = q.x, x = q.y, y = q.z, z = q.w;
  R[0][0] = 1.f - 2.f * (y * y + z * z); R[0][1] = 2.f * (x * y - r * z); R[0][2] = 2.f * (x * z + r * y);
  R[1][0] = 2.f * (x * y + r * z); R[1][1] = 1.f - 2.f * (x * x + z * z); R[1][2] = 2.f * (y * z - r * x);
  R[2][0] = 2.f * (x * z - r * y); R[2][1] = 2.f * (y * z + r * x); R[2][2] = 1.f - 2.f * (x * x + y * y);
}

__device__ __forceinline__ void quat_to_rot_d(float4 qf, double R[3][3]) {  // quat_to_rot in fp64
  const double r = qf.x, x = qf.y, y = qf.z, z = qf.w;
  R[0][0] = 1.0 - 2.0 * (y * y + z * z); R[0][1] = 2.0 * (x * y - r * z); R[0][2] = 2.0 * (x * z + r * y);
  R[1][0] = 2.0 * (x * y + r * z); R[1][1] = 1.0 - 2.0 * (x * x + z * z); R[1][2] = 2.0 * (y * z - r * x);
  R[2][0] = 2.0 * (x * z - r * y); R[2][1] = 2.0 * (y * z + r * x); R[2][2] = 1.0 - 2.0 * (x * x + y * y);
}

// Sigma = Rq diag(mod*s)^2 Rq^T, upper triangle (forward.cu:118-152)
__device__ __forceinline__ void cov3d_from_scale_rot(float3 s, float mod, float4 q, float c6[6]) {
  float R[3][3], M[3][3];
  quat_to_rot(q, R);
  float sv[3] = {mod * s.x, mod * s.y, mod * s.z};
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) M[i][j] = sv[i] * R[j][i];
  int k = 0;
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int b = a; b < 3; b++) c6[k++] = M[0][a] * M[0][b] + M[1][a] * M[1][b] + M[2][a] * M[2][b];
}

struct Ewa {
  float A[2][3];  // J * Rw (screen-space Jacobian times world->view rotation)
  float3 t;       // view-space mean, x/y clamped to the 1.3*tanfov frustum
  float txtz, tytz, limx, limy;
};

__device__ __forceinline__ void ewa_setup(float3 mean, const Camera& cam, Ewa& e) {  // forward.cu:74-97
  e.t = xform43(cam.view, mean);
  e.limx = 1.3f * cam.tanx;
  e.limy = 1.3f * cam.tany;
  e.txtz = e.t.x / e.t.z;
  e.tytz = e.t.y / e.t.z;
  e.t.x = fminf(e.limx, fmaxf(-e.limx, e.txtz)) * e.t.z;
  e.t.y = fminf(e.limy, fmaxf(-e.limy, e.tytz)) * e.t.z;
  float tz = e.t.z;
  float j00 = cam.fx / tz, j02 = -(cam.fx * e.t.x) / (tz * tz);
  float j11 = cam.fy / tz, j12 = -(cam.fy * e.t.y) / (tz * tz);
#pragma unroll
  for (int k = 0; k < 3; k++) {
    e.A[0][k] = cam.view[4 * k + 0] * j00 + cam.view[4 * k + 2] * j02;
    e.A[1][k] = cam.view[4 * k + 1] * j11 + cam.view[4 * k + 2] * j12;
  }
}

__device__ __forceinline__ void sym6(const float c[6], float V[3][3]) {
  V[0][0] = c[0]; V[0][1] = V[1][0] = c[1]; V[0][2] = V[2][0] = c[2];
  V[1][1] = c[3]; V[1][2] = V[2][1] = c[4]; V[2][2] = c[5];
}

__device__ __forceinline__ void cov2d(const Ewa& e, const float c6[6], float& a, float& b, float& c) {
  float V[3][3], va0[3], va1[3];
  sym6(c6, V);
#pragma unroll
  for (int k = 0; k < 3; k++) {
    va0[k] = V[k][0] * e.A[0][0] + V[k][1] * e.A[0][1] + V[k][2] * e.A[0][2];
    va1[k] = V[k][0] * e.A[1][0] + V[k][1] * e.A[1][1] + V[k][2] * e.A[1][2];
  }
  a = e.A[0][0] * va0[0] + e.A[0][1] * va0[1] + e.A[0][2] * va0[2] + 0.3f;  // forward.cu:110-111
  b = e.A[0][0] * va1[0] + e.A[0][1] * va1[1] + e.A[0][2] * va1[2];
  c = e.A[1][0] * va1[0] + e.A[1][1] * va1[1] + e.A[1][2] * va1[2] + 0.3f;
}

// real SH basis (degree <= 3) and its gradient w.r.t. the unit direction; public constants.
__constant__ float kSH1 = 0.4886025119029199f;
__constant__ float kSH2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                              -1.0925484305920792f, 0.5462742152960396f};
__constant__ float kSH3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                              0.3731763325901154f,  -0.4570457994644658f, 1.445305721320277f,
                              -0.5900435899266435f};
constexpr float kSH0 = 0.28209479177387814f;

template <bool GRAD>
__device__ inline void sh_basis(int deg, float x, float y, float z, float b[16], float db[16][3]) {
  if (GRAD) {
#pragma unroll
    for (int k = 0; k < 16; k++) db[k][0] = db[k][1] = db[k][2] = 0.f;
  }
  b[0] = kSH0;
  if (deg > 0) {
    b[1] = -kSH1 * y; b[2] = kSH1 * z; b[3] = -kSH1 * x;
    if (GRAD) { db[1][1] = -kSH1; db[2][2] = kSH1; db[3][0] = -kSH1; }
  }
  if (deg > 1) {
    float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    b[4] = kSH2[0] * xy; b[5] = kSH2[1] * yz; b[6] = kSH2[2] * (2.0f * zz - xx - yy);
    b[7] = kSH2[3] * xz; b[8] = kSH2[4] * (xx - yy);
    if (GRAD) {
      db[4][0] = kSH2[0] * y; db[4][1] = kSH2[0] * x;
      db[5][1] = kSH2[1] * z; db[5][2] = kSH2[1] * y;
      db[6][0] = kSH2[2] * 2.f * -x; db[6][1] = kSH2[2] * 2.f * -y; db[6][2] = kSH2[2] * 2.f * 2.f * z;
      db[7][0] = kSH2[3] * z; db[7][2] = kSH2[3] * x;
      db[8][0] = kSH2[4] * 2.f * x; db[8][1] = kSH2[4] * 2.f * -y;
    }
    if (deg > 2) {
      b[9] = kSH3[0] * y * (3.0f * xx - yy);
      b[10] = kSH3[1] * xy * z;
      b[11] = kSH3[2] * y * (4.0f * zz - xx - yy);
      b[12] = kSH3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy);
      b[13] = kSH3[4] * x * (4.0f * zz - xx - yy);
      b[14] = kSH3[5] * z * (xx - yy);
      b[15] = kSH3[6] * x * (xx - 3.0f * yy);
      if (GRAD) {
        db[9][0] = kSH3[0] * 3.f * 2.f * xy; db[9][1] = kSH3[0] * 3.f * (xx - yy);
        db[10][0] = kSH3[1] * yz; db[10][1] = kSH3[1] * xz; db[10][2] = kSH3[1] * xy;
        db[11][0] = kSH3[2] * -2.f * xy; db[11][1] = kSH3[2] * (-3.f * yy + 4.f * zz - xx); db[11][2] = kSH3[2] * 4.f * 2.f * yz;
        db[12][0] = kSH3[3] * -3.f * 2.f * xz; db[12][1] = kSH3[3] * -3.f * 2.f * yz; db[12][2] = kSH3[3] * 3.f * (2.f * zz - xx - yy);
        db[13][0] = kSH3[4] * (-3.f * xx + 4.f * zz - yy); db[13][1] = kSH3[4] * -2.f * xy; db[13][2] = kSH3[4] * 4.f * 2.f * xz;
        db[14][0] = kSH3[5] * 2.f * xz; db[14][1] = kSH3[5] * -2.f * yz; db[14][2] = kSH3[5] * (xx - yy);
        db[15][0] = kSH3[6] * 3.f * (xx - yy); db[15][1] = kSH3[6] * -3.f * 2.f * xy;
      }
    }
  }
}

// Activations of the reference's GaussianModel (gs_core.py:330-334,545-570)
__device__ __forceinline__ float3 act_scale(float3 s) { return make_float3(expf(s.x), expf(s.y), expf(s.z)); }
__device__ __forceinline__ float act_opacity(float o) { return 1.0f / (1.0f + expf(-o)); }
__device__ __forceinline__ float4 act_rot(float4 q, float* inv_norm) {  // F.normalize, eps 1e-12
  float n = sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
  float inv = 1.0f / fmaxf(n, 1e-12f);
  if (inv_norm) *inv_norm = inv;
  return make_float4(q.x * inv, q.y * inv, q.z * inv, q.w * inv);
}

__device__ __forceinline__ float3 ld3(const float* p, size_t i) { return make_float3(p[3 * i], p[3 * i + 1], p[3 * i + 2]); }
__device__ __forceinline__ float4 ld4(const float* p, size_t i) {
  return *reinterpret_cast<const float4*>(p + 4 * i);
}

// ---------------------------------------------------------------------------------------------
// cameras
// ---------------------------------------------------------------------------------------------
// Batched: Camera(C2W, fxfycxcy, h, w) of gs_core.py:277-316, one thread per view.
__global__ void build_cameras_kernel(int NV, const float* __restrict__ c2w, const float* __restrict__ fxfycxcy,
                                     int W, int H, Camera* __restrict__ cams) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= NV) return;
  // general 4x4 inverse (torch `C2W.inverse()`), Gauss-Jordan with partial pivoting in fp64
  double a[4][8];
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) {
      a[r][c] = (double)c2w[16 * v + 4 * r + c];
      a[r][4 + c] = (r == c) ? 1.0 : 0.0;
    }
  for (int col = 0; col < 4; col++) {
    int piv = col;
    double best = fabs(a[col][col]);
    for (int r = col + 1; r < 4; r++)
      if (fabs(a[r][col]) > best) { best = fabs(a[r][col]); piv = r; }
    if (piv != col)
      for (int c = 0; c < 8; c++) { double t = a[col][c]; a[col][c] = a[piv][c]; a[piv][c] = t; }
    double inv = 1.0 / a[col][col];
    for (int c = 0; c < 8; c++) a[col][c] *= inv;
    for (int r = 0; r < 4; r++)
      if (r != col) {
        double f = a[r][col];
        for (int c = 0; c < 8; c++) a[r][c] -= f * a[col][c];
      }
  }
  float w2c[4][4];
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) w2c[r][c] = (float)a[r][4 + c];
  const float fx = fxfycxcy[4 * v + 0], fy = fxfycxcy[4 * v + 1], cx = fxfycxcy[4 * v + 2], cy = fxfycxcy[4 * v + 3];
  const float zn = 0.01f, zf = 100.0f;  // gs_core.py:286-287
  float Pm[4][4] = {{0}};
  Pm[0][0] = 2 * fx / W;
  Pm[1][1] = 2 * fy / H;
  Pm[0][2] = 2 * (cx / W) - 1;
  Pm[1][2] = 2 * (cy / H) - 1;
  Pm[2][2] = -(zf + zn) / (zf - zn);
  Pm[3][2] = 1.0f;
  Pm[2][3] = -(2 * zf * zn) / (zf - zn);
  Camera cam;
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) {
      cam.view[4 * c + r] = w2c[r][c];
      float s = 0.f;
      for (int k = 0; k < 4; k++) s += Pm[r][k] * w2c[k][c];
      cam.proj[4 * c + r] = s;
    }
  cam.campos[0] = c2w[16 * v + 3];
  cam.campos[1] = c2w[16 * v + 7];
  cam.campos[2] = c2w[16 * v + 11];
  cam.tanx = W / (2 * fx);
  cam.tany = H / (2 * fy);
  cam.fx = W / (2.0f * cam.tanx);  // rasterizer_impl.cu:222-223
  cam.fy = H / (2.0f * cam.tany);
  cam.pad = 0.f;
  cams[v] = cam;
}

// Single view: matrices already on the device (GaussianRasterizationSettings), tan(fov) from the host.
__global__ void pack_camera_kernel(const float* __restrict__ view, const float* __restrict__ proj,
                                   const float* __restrict__ campos, float tanx, float tany, int W, int H,
                                   Camera* __restrict__ cam) {
  int t = threadIdx.x;
  if (t < 16) { cam->view[t] = view[t]; cam->proj[t] = proj[t]; }
  if (t < 3) cam->campos[t] = campos[t];
  if (t == 0) {
    cam->tanx = tanx; cam->tany = tany;
    cam->fx = W / (2.0f * tanx); cam->fy = H / (2.0f * tany);
    cam->pad = 0.f;
  }
}

// ---------------------------------------------------------------------------------------------
// K1: projection, one thread per (view, Gaussian)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) project_kernel(Problem pb, GeomState gs, int* __restrict__ radii_out) {
  __shared__ Camera cam;
  const int view = blockIdx.y;
  {
    const float* src = reinterpret_cast<const float*>(gs.cams + view);
    float* dst = reinterpret_cast<float*>(&cam);
    for (int t = threadIdx.x; t < (int)(sizeof(Camera) / 4); t += blockDim.x) dst[t] = src[t];
  }
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= pb.P) return;
  const size_t n = (size_t)view * pb.P + i;
  const size_t si = (size_t)(view / pb.V) * pb.P + i;  // index into the per-sample parameter tensors

  uint32_t tiles = 0;
  float4 o0 = make_float4(0.f, 0.f, 0.f, 0.f), o1 = o0, o2 = o0;
  int radius_i = 0;
  do {
    const float3 p = ld3(pb.means, si);
    const float3 pv = xform43(cam.view, p);
    if (pv.z <= NEAR_Z) break;  // in_frustum, auxiliary.h:139-164
    const float4 ph = xform44(cam.proj, p);
    const float pw = 1.0f / (ph.w + 0.0000001f);
    const float projx = ph.x * pw, projy = ph.y * pw;

    float c6[6];
    if (pb.cov_pre) {
#pragma unroll
      for (int k = 0; k < 6; k++) c6[k] = pb.cov_pre[6 * si + k];
    } else {
      float3 s = ld3(pb.scales, si);
      float4 q = ld4(pb.rots, si);
      if (pb.raw) { s = act_scale(s); q = act_rot(q, nullptr); }
      cov3d_from_scale_rot(s, pb.mod, q, c6);
    }
    Ewa e;
    ewa_setup(p, cam, e);
    float a, b, c;
    cov2d(e, c6, a, b, c);
    const float det = a * c - b * b;
    if (det == 0.0f) break;
    const float det_inv = 1.f / det;
    const float mid = 0.5f * (a + c);
    const float l1 = mid + sqrtf(fmaxf(0.1f, mid * mid - det));
    const float l2 = mid - sqrtf(fmaxf(0.1f, mid * mid - det));
    const float radius = ceilf(3.f * sqrtf(fmaxf(l1, l2)));
    const float px = ndc_to_pix(projx, pb.W), py = ndc_to_pix(projy, pb.H);
    int x0, y0, x1, y1;
    tile_rect(px, py, (int)radius, pb.gx, pb.gy, x0, y0, x1, y1);
    if ((x1 - x0) * (y1 - y0) == 0) break;

    float rgb[3];
    int clamped = 0;
    if (pb.colors_pre) {
      rgb[0] = pb.colors_pre[3 * si]; rgb[1] = pb.colors_pre[3 * si + 1]; rgb[2] = pb.colors_pre[3 * si + 2];
    } else {
      const float* sh = pb.shs + si * pb.M * 3;
      if (pb.D == 0) {
#pragma unroll
        for (int ch = 0; ch < 3; ch++) rgb[ch] = kSH0 * sh[ch];
      } else {
        float dx = p.x - cam.campos[0], dy = p.y - cam.campos[1], dz = p.z - cam.campos[2];
        float len = sqrtf(dx * dx + dy * dy + dz * dz);
        float bs[16];
        sh_basis<false>(pb.D, dx / len, dy / len, dz / len, bs, nullptr);
        const int nb = (pb.D + 1) * (pb.D + 1);
#pragma unroll
        for (int ch = 0; ch < 3; ch++) rgb[ch] = 0.f;
        for (int k = 0; k < nb; k++)
#pragma unroll
          for (int ch = 0; ch < 3; ch++) rgb[ch] += bs[k] * sh[3 * k + ch];
      }
#pragma unroll
      for (int ch = 0; ch < 3; ch++) {
        rgb[ch] += 0.5f;
        if (rgb[ch] < 0.f) clamped |= (1 << ch);
        rgb[ch] = fmaxf(rgb[ch], 0.0f);
      }
    }
    float op = pb.opac[si];
    if (pb.raw) op = act_opacity(op);
    radius_i = (int)radius;
    o0 = make_float4(px, py, pv.z, __int_as_float(radius_i));
    o1 = make_float4(c * det_inv, -b * det_inv, a * det_inv, op);
    o2 = make_float4(rgb[0], rgb[1], rgb[2], __int_as_float(clamped));
    tiles = (uint32_t)((y1 - y0) * (x1 - x0));
  } while (false);
  gs.g0[n] = o0;
  gs.g1[n] = o1;
  gs.g2[n] = o2;
  gs.tiles[n] = tiles;
  gs.dkey_in[n] = ((uint64_t)view << 32) | __float_as_uint(o0.z);  // depth > 0.2: bit pattern is monotonic
  gs.perm_in[n] = (uint32_t)i;
  if (radii_out) radii_out[n] = radius_i;
}

// tiles touched in depth-rank order (input of the instance-offset scan)
// Also accumulates the EXACT instance count in 64 bits (totals->R64): the 32-bit scan below wraps silently beyond
// 2^32 instances, and the host must be able to tell "too many for one batch" from a small wrapped number.
__global__ void gather_tiles_kernel(size_t N, int P, GeomState gs) {
  const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t t = 0;
  if (k < N) {
    const size_t view = k / P;
    t = gs.tiles[view * P + gs.perm[k]];
    gs.tiles_sorted[k] = t;
  }
  unsigned long long sum = t;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0 && sum) atomicAdd(&gs.totals->R64, sum);
}

// ---------------------------------------------------------------------------------------------
// Walking a Gaussian's tile rect, shared by every binning kernel that visits tiles one by one.
// walk_rect visits the tiles of [x0,x1) x [y0,y1) in row-major order as visit(tile, rank, payload), tile = y * gx + x.
// A rect under DUP_COOP_THRESHOLD tiles is walked by its own thread; larger ones (a few big splats would otherwise
// serialise a thread for hundreds of tiles) lane-parallel by the whole warp, one rect after another, with the owner's
// payload broadcast.  keep(tile) drops tiles (KeepAll: none); rank is the tile's position among the kept tiles of its
// rect, counted by the thread or, on the warp path, by a ballot prefix over each 32-tile step, so ranks stay in
// row-major order.  Every lane of the warp must call it; an empty rect visits nothing.
// ---------------------------------------------------------------------------------------------
constexpr int DUP_COOP_THRESHOLD = 32;
struct KeepAll {};

template <typename Keep, typename Visit>
__device__ __forceinline__ void walk_rect(int x0, int y0, int x1, int y1, int gx, uint2 payload, Keep keep, Visit visit) {
  constexpr bool kFilter = !std::is_same<Keep, KeepAll>::value;
  const int lane = threadIdx.x & 31;
  const int w = x1 - x0, area = w * (y1 - y0);
  if (area > 0 && area < DUP_COOP_THRESHOLD) {
    uint32_t rank = 0;
    for (int y = y0; y < y1; y++)
      for (int x = x0; x < x1; x++) {
        const int t = y * gx + x;
        if constexpr (kFilter) {
          if (!keep(t)) continue;
        }
        visit(t, rank++, payload);
      }
  }
  unsigned big = __ballot_sync(0xffffffffu, area >= DUP_COOP_THRESHOLD);
  while (big) {
    const int src = __ffs(big) - 1;
    big &= big - 1;
    const int bx0 = __shfl_sync(0xffffffffu, x0, src), by0 = __shfl_sync(0xffffffffu, y0, src);
    const int bw = __shfl_sync(0xffffffffu, w, src), barea = __shfl_sync(0xffffffffu, area, src);
    const uint2 bp = make_uint2(__shfl_sync(0xffffffffu, payload.x, src), __shfl_sync(0xffffffffu, payload.y, src));
    if constexpr (kFilter) {
      uint32_t rank = 0;
      for (int t0 = 0; t0 < barea; t0 += 32) {
        const int t = t0 + lane;
        int tile = 0;
        bool kept = false;
        if (t < barea) {
          tile = (by0 + t / bw) * gx + bx0 + t % bw;
          kept = keep(tile);
        }
        const unsigned m = __ballot_sync(0xffffffffu, kept);
        if (kept) visit(tile, rank + __popc(m & ((1u << lane) - 1u)), bp);
        rank += __popc(m);
      }
    } else {
      for (uint32_t t = lane; t < (uint32_t)barea; t += 32) visit((by0 + (int)(t / bw)) * gx + bx0 + (int)(t % bw), t, bp);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// K3: instance emission in DEPTH-RANK order.  The reference sorts 64-bit (tile | depth) keys globally
// (rasterizer_impl.cu:70-111, 300-308).  Here each view's Gaussians are first ranked by (depth bits, index)
// (a sort of P elements), instances are emitted in that order, and the big per-instance sort only has to be a
// STABLE sort by the 32-bit tile id (2 radix passes over 8-byte pairs instead of 6 over 12-byte pairs).
// The resulting order -- tile, then depth, ties by Gaussian index -- is identical.
// ---------------------------------------------------------------------------------------------

// Two-phase binning bookkeeping for one near fraction: per view, where its near instances (ranks < Pn) start in the
// global scan and in the compact phase-A buffer (near_meta[2v], near_meta[2v + 1]); *r_near = their total, totals->R =
// every instance.  One thread: NV is small.
__global__ void chunk_meta_kernel(int NV, int P, int Pn, const uint32_t* __restrict__ offsets,
                                  uint32_t* __restrict__ near_meta, BinTotals* __restrict__ totals,
                                  uint32_t* __restrict__ r_near) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  uint32_t base = 0;
  for (int v = 0; v < NV; v++) {
    const size_t k0 = (size_t)v * P;
    const uint32_t start = (k0 == 0) ? 0u : offsets[k0 - 1];
    near_meta[2 * v + 0] = start;
    near_meta[2 * v + 1] = base;
    base += offsets[k0 + Pn - 1] - start;
  }
  totals->R = offsets[(size_t)NV * P - 1];
  *r_near = base;
}

// Ranks [rank_lo, rank_hi) of every view.  OPEN = false: every tile of the rect, at the rank's exclusive scan position
// in `offsets`, rebased per view into the compact phase-A buffer when near_meta is given.  OPEN = true (phase B): only
// the tiles still open after phase A, at the rank's exclusive scan position in `open_offsets`.
template <bool OPEN>
__global__ void __launch_bounds__(256) emit_keys_kernel(Problem pb, GeomState gs, const uint32_t* __restrict__ tile_open,
                                                        const uint32_t* __restrict__ near_meta,
                                                        uint32_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                                        int rank_lo, int rank_hi) {
  const int view = blockIdx.y;
  const int r = rank_lo + blockIdx.x * blockDim.x + threadIdx.x;  // depth rank inside the view
  const bool in_range = r < rank_hi;
  const size_t k = (size_t)view * pb.P + (in_range ? r : rank_lo);
  const uint32_t cnt = !in_range ? 0u : OPEN ? gs.open_counts[k] : gs.tiles_sorted[k];
  uint32_t off = 0, id = 0;
  int x0 = 0, y0 = 0, x1 = 0, y1 = 0;
  if (cnt) {
    if (OPEN) {
      off = gs.open_offsets[k] - cnt;  // inclusive scan
    } else {
      off = (k == 0) ? 0u : gs.offsets[k - 1];
      if (near_meta) off = off - near_meta[2 * view] + near_meta[2 * view + 1];
    }
    id = gs.perm[k];
    const float4 g = gs.g0[(size_t)view * pb.P + id];
    tile_rect(g.x, g.y, __float_as_int(g.w), pb.gx, pb.gy, x0, y0, x1, y1);
  }
  const uint32_t tile_base = (uint32_t)(view * pb.tiles);
  auto emit = [&](int tile, uint32_t rank, uint2 p) {
    keys[p.x + rank] = tile_base + (uint32_t)tile;
    vals[p.x + rank] = p.y;
  };
  if constexpr (OPEN) {
    const uint32_t* open = tile_open + (size_t)view * pb.tiles;
    walk_rect(x0, y0, x1, y1, pb.gx, make_uint2(off, id), [&](int tile) { return open[tile] != 0u; }, emit);
  } else {
    walk_rect(x0, y0, x1, y1, pb.gx, make_uint2(off, id), KeepAll(), emit);
  }
}

// Phase B of the two-phase binning only serves the tiles that are still OPEN after phase A (tile_open): per far rank,
// count the open tiles of its rect (near ranks: 0) -- the scan of these counts gives the compact phase-B offsets.
__global__ void __launch_bounds__(256) count_open_kernel(Problem pb, GeomState gs, const uint32_t* __restrict__ tile_open,
                                                         int Pn) {
  const int view = blockIdx.y;
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= pb.P) return;
  const size_t k = (size_t)view * pb.P + r;
  uint32_t cnt = 0;
  if (r >= Pn && gs.tiles_sorted[k]) {
    const float4 g = gs.g0[(size_t)view * pb.P + gs.perm[k]];
    int x0, y0, x1, y1;
    tile_rect(g.x, g.y, __float_as_int(g.w), pb.gx, pb.gy, x0, y0, x1, y1);
    const uint32_t* op = tile_open + (size_t)view * pb.tiles;
    for (int y = y0; y < y1; y++)
      for (int x = x0; x < x1; x++) cnt += op[y * pb.gx + x];
  }
  gs.open_counts[k] = cnt;
}

// ---------------------------------------------------------------------------------------------
// Small-scene binning: when a batch has few view-Gaussians the global machinery above (depth ranking sort, scan,
// key emission, tile sort: ~12 launches) costs more than the work.  Instead: the projection counts instances per tile,
// ONE block turns the counts into tile ranges, a fill kernel drops (depth bits, id) into each tile's bucket in arrival
// order, and every tile sorts its own bucket in shared memory by (depth bits, Gaussian index) -- the reference's order
// (stable radix sort of tile | depth keys emitted in index order, rasterizer_impl.cu:70-111, 300-308).  point_list and
// ranges come out exactly as from the global path; the blend kernels do not know the difference.
// ---------------------------------------------------------------------------------------------
constexpr int SMALL_TILE_CAP = 4096;      // longest tile list the shared-memory sort takes (32 KB of keys)
constexpr int SMALL_MAX_N = 1 << 18;      // view-Gaussians
constexpr int SMALL_MAX_TILES = 1 << 15;  // views * tiles (one block scans them)

// counts[t] -> ranges[t] = [start, end), cursor[t] = start; totals->R = R, totals->longest = longest list
__global__ void __launch_bounds__(1024) tile_scan_kernel(int ntiles, const uint32_t* __restrict__ counts, uint2* __restrict__ ranges,
                                                         uint2* __restrict__ cursor, BinTotals* __restrict__ totals) {
  __shared__ uint32_t s_warp[32];
  __shared__ uint32_t s_carry, s_max;
  if (threadIdx.x == 0) { s_carry = 0; s_max = 0; }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < ntiles; base += 1024) {
    const int t = base + threadIdx.x;
    const uint32_t c = t < ntiles ? counts[t] : 0u;
    uint32_t incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    uint32_t mx = c;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 31) s_warp[warp] = incl;
    if (lane == 0) atomicMax(&s_max, mx);
    __syncthreads();
    if (warp == 0) {
      uint32_t w = s_warp[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += v;
      }
      s_warp[lane] = w;  // inclusive over warps
    }
    __syncthreads();
    const uint32_t start = s_carry + (warp ? s_warp[warp - 1] : 0u) + incl - c;
    if (t < ntiles) {
      ranges[t] = make_uint2(start, start + c);
      cursor[t] = make_uint2(start, 0u);
    }
    __syncthreads();
    if (threadIdx.x == 0) s_carry += s_warp[31];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    totals->R = s_carry;
    totals->longest = s_max;
  }
}

// COUNT: every (view, Gaussian) adds 1 to each tile of its rect.  FILL: it drops one (depth bits, id) record into each of
// those tiles at the tile's cursor.
template <bool FILL>
__global__ void __launch_bounds__(256) tile_count_fill_kernel(Problem pb, GeomState gs, uint32_t* __restrict__ counts,
                                                              uint2* __restrict__ cursor, uint32_t* __restrict__ depth_out,
                                                              uint32_t* __restrict__ id_out) {
  const int view = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int x0 = 0, y0 = 0, x1 = 0, y1 = 0;
  uint32_t depth = 0;
  if (i < pb.P) {
    const size_t n = (size_t)view * pb.P + i;
    if (gs.tiles[n]) {
      const float4 g = gs.g0[n];
      tile_rect(g.x, g.y, __float_as_int(g.w), pb.gx, pb.gy, x0, y0, x1, y1);
      depth = __float_as_uint(g.z);
    }
  }
  const size_t tbase = (size_t)view * pb.tiles;
  walk_rect(x0, y0, x1, y1, pb.gx, make_uint2(depth, (uint32_t)i), KeepAll(), [&](int tile, uint32_t, uint2 p) {
    if (FILL) {
      const uint32_t pos = atomicAdd(&cursor[tbase + tile].x, 1u);
      depth_out[pos] = p.x;
      id_out[pos] = p.y;
    } else {
      atomicAdd(counts + tbase + tile, 1u);
    }
  });
}

// one CTA per (view, tile): bitonic sort of the bucket's 64-bit (depth bits << 32 | id) keys in shared memory
__global__ void __launch_bounds__(256) tile_sort_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ depth_in,
                                                        const uint32_t* __restrict__ id_in, uint32_t* __restrict__ point_list) {
  extern __shared__ unsigned long long s_key[];
  const uint2 r = ranges[blockIdx.x];
  const int n = (int)(r.y - r.x);
  if (n == 0) return;
  if (n == 1) {
    if (threadIdx.x == 0) point_list[r.x] = id_in[r.x];
    return;
  }
  int m = 2;
  while (m < n) m <<= 1;
  for (int k = threadIdx.x; k < m; k += blockDim.x)
    s_key[k] = k < n ? (((unsigned long long)depth_in[r.x + k] << 32) | id_in[r.x + k]) : ~0ull;
  __syncthreads();
  for (int size = 2; size <= m; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int k = threadIdx.x; k < (m >> 1); k += blockDim.x) {
        const int lo = ((k / stride) * stride << 1) + (k % stride), hi = lo + stride;
        const bool up = ((lo & size) == 0);
        const unsigned long long a = s_key[lo], b = s_key[hi];
        if ((a > b) == up) { s_key[lo] = b; s_key[hi] = a; }
      }
      __syncthreads();
    }
  }
  for (int k = threadIdx.x; k < n; k += blockDim.x) point_list[r.x + k] = (uint32_t)s_key[k];
}

// K5: tile ranges from the sorted keys (rasterizer_impl.cu:116-138)
__global__ void tile_ranges_kernel(long long R, const uint32_t* __restrict__ keys, uint2* __restrict__ ranges) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= R) return;
  uint32_t cur = keys[idx];
  if (idx == 0) ranges[cur].x = 0;
  else {
    uint32_t prev = keys[idx - 1];
    if (cur != prev) { ranges[prev].y = (uint32_t)idx; ranges[cur].x = (uint32_t)idx; }
  }
  if (idx == R - 1) ranges[cur].y = (uint32_t)R;
}

// The Gaussian falloff G = exp(power), power = -0.5 (A dx^2 + C dy^2) - B dx dy (forward.cu:326-329), is evaluated as
// ex2(power * log2 e) on the MUFU pipe with the conic pre-scaled by -0.5 log2 e / -log2 e (5 FMA-pipe ops + 1 MUFU
// instead of the 7 + ~10 of expf).  Forward and backward call the SAME two functions with explicitly rounded
// intrinsics, so they take bit-identical contribute / skip decisions for every (pixel, Gaussian) pair.
constexpr float kLog2e = 1.4426950408889634f;
__device__ __forceinline__ float4 conic_log2(float4 co) {
  return make_float4(__fmul_rn(co.x, -0.5f * kLog2e), __fmul_rn(co.y, -kLog2e), __fmul_rn(co.z, -0.5f * kLog2e), co.w);
}
__device__ __forceinline__ float pair_power2(float4 c2, float dx, float dy) {
  return __fmaf_rn(dx, __fmaf_rn(c2.x, dx, __fmul_rn(c2.y, dy)), __fmul_rn(__fmul_rn(c2.z, dy), dy));
}
__device__ __forceinline__ float ex2_mufu(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Exact footprint of a Gaussian at the alpha >= 1/255 level: alpha = o exp(power) with
// power = -0.5 (A dx^2 + C dy^2) - B dx dy;  for a fixed dy the largest power over dx is -0.5 dy^2 det / A, so the pair can
// only pass the alpha test when dy^2 <= 2 ln(255 o) A / det (and dx^2 <= 2 ln(255 o) C / det).  The blend kernels use these
// half-extents to skip, per WARP (two pixel rows of the tile), staged list entries that cannot contribute to any of its
// pixels: a skipped entry is one the reference's own `alpha < 1/255` test rejects for every pixel of the warp, so images,
// n_contrib, final_T and gradients are unchanged (it still counts as a visited entry).  The sparse regimes spend 85-94 %
// of their pair evaluations on such rejections.  Margins (0.1 % + 0.01 px) keep the bound conservative against
// fp32 rounding; a conic that is not positive definite gets +inf (never skipped), an opacity <= 1/255 gets -1 (always).
__device__ __forceinline__ float2 alpha_extent(float4 q /* A, B, C, opacity */) {
  const float det = q.x * q.z - q.y * q.y;
  if (!(q.x > 0.f && q.z > 0.f && det > 0.f)) return make_float2(INFINITY, INFINITY);
  const float lv = 2.0f * __logf(255.0f * q.w);
  if (!(lv > 0.f)) return make_float2(-1.f, -1.f);
  const float s = lv / det;
  return make_float2(sqrtf(s * q.z) * 1.001f + 0.01f, sqrtf(s * q.x) * 1.001f + 0.01f);  // (x half-extent, y half-extent)
}
constexpr float SKIP_WORTH = 13.0f;  // a y half-extent below this can miss at least one warp of a 16-row tile

// Fused image loss (LossComputer.forward's l2 term, diffusionGS/utils/losses.py:280-284): the blend
// forward accumulates sum (render - target)^2 per sample while the pixel is still in registers, and the blend backward
// forms dL/dpix = [upstream gradient image] + coef[sample] * (render - target) itself, so the MSE never materialises a
// per-element loss or gradient image.  target [NV, tc, H, W] (tc = 3, or 4 = rgb + mask whose plane is skipped,
// losses.py:274-276).
struct MseFwd {
  const float* target = nullptr;
  int tc = 3;
  double* loss = nullptr;  // [samples]
};
struct MseBwd {
  const float* target = nullptr;
  int tc = 3;
  const float* images = nullptr;  // the forward's output [NV,3,H,W]
  const float* coef = nullptr;    // [samples] device
};

// Depth and alpha maps (the blend kernels' AUX instantiations).  depth = sum_i w_i z_i with w_i = alpha_i T_i the colour's
// blend weight and z_i the view-space depth in g0.z (background 0); alpha = 1 - final T.  Both are linear in the same
// weights as the colour, so the backward adds one accumulator, folds dL/dalpha into the background term and reduces one
// more per-Gaussian component, dL/dz, which the geometry backward pushes through W2C's third row.
struct AuxFwd {
  float* depth = nullptr;  // [NV,1,H,W]; two-phase: phase A leaves its partial sum here for phase B
  float* alpha = nullptr;  // [NV,1,H,W]
};
// Video frames (the FRAMES instantiations): each pixel leaves the kernel as the reference's uint8 frame value,
// (image * 255).clip(0, 255).astype(uint8) of the fp32 colour (gs_core.py:1215-1216), HWC [NV,H,W,3]; no fp32 image is
// written.  The frames pointer travels in out_color's slot, so the other instantiations keep their parameters (and code).
struct FramesFwd {
  // the product rounded on its own (no FMA contraction with the blend); fmaxf maps NaN to 0; the cast truncates
  __device__ __forceinline__ static uint8_t quantise(float c) {
    return (uint8_t)fminf(fmaxf(__fmul_rn(c, 255.f), 0.f), 255.f);
  }
};
struct AuxBwd {
  const float* ddepth = nullptr;  // [NV,1,H,W] or null
  const float* dalpha = nullptr;  // [NV,1,H,W] or null
  float* dz = nullptr;            // [N] out: dL/dz per (view, Gaussian)
};
// ---------------------------------------------------------------------------------------------
// K6: per-tile front-to-back alpha blend (forward.cu:261-374), one CTA per (view, tile)
// ---------------------------------------------------------------------------------------------
// MODE 0: the whole list in one pass.  MODE 1: phase A of two (the nearest Gaussians); saves the per-pixel blend state
// and counts the tiles that still have unfinished pixels.  MODE 2: phase B, continues from that state.
// AUX: also the depth and alpha maps; z rides in the .w of s_rgb (the clamped bits the blend does not read).
// FRAMES: out_color points to uint8 frames (see FramesFwd), written wherever the fp32 image would be.
template <int MODE, bool AUX = false, bool FRAMES = false>
__global__ void __launch_bounds__(TILE_PIX) blend_forward_kernel(Problem pb, GeomState gs, ImgState im,
                                                                 const uint32_t* __restrict__ point_list,
                                                                 float* __restrict__ out_color, MseFwd mse, AuxFwd aux) {
  const int tile_g = blockIdx.x;
  const int view = tile_g / pb.tiles, tile = tile_g - view * pb.tiles;
  const int tx = tile % pb.gx, ty = tile / pb.gx;
  const int lx = threadIdx.x & (TILE - 1), ly = threadIdx.x >> 4;
  const int x = tx * TILE + lx, y = ty * TILE + ly;
  const bool inside = x < pb.W && y < pb.H;
  const float pxf = (float)x, pyf = (float)y;
  const uint2 range = (MODE == 2) ? im.ranges_b[tile_g] : im.ranges[tile_g];
  const size_t gbase = (size_t)view * pb.P;
  const size_t pix_g = (size_t)view * pb.W * pb.H + (size_t)y * pb.W + x;

  __shared__ float4 s_xy[TILE_PIX];  // x, y, x half-extent, y half-extent (alpha_extent)
  __shared__ float4 s_co[TILE_PIX];
  __shared__ float4 s_rgb[TILE_PIX];
  __shared__ uint8_t s_list[TILE_PIX / 32][TILE_PIX];  // per-warp compacted entry indices of a sparse chunk
  const float wy0 = (float)(ty * TILE + (threadIdx.x >> 5) * 2);  // this warp's first pixel row
  const float tx0 = (float)(tx * TILE);

  bool done = !inside;
  float T = 1.0f, C0 = 0.f, C1 = 0.f, C2 = 0.f, D = 0.f;
  uint32_t contributor = 0, last = 0;
  if (MODE == 2 && inside) {
    const float4 a = im.acc[pix_g];
    const uint32_t cb = im.contrib[pix_g];
    C0 = a.x; C1 = a.y; C2 = a.z; T = a.w;
    contributor = cb & 0x7fffffffu;
    done = (cb >> 31) != 0;
    last = im.n_contrib[pix_g];
    if constexpr (AUX) D = aux.depth[pix_g];
  }
  // visits before this kernel's list: 0, or (phase B) the phase-A list length, which every unfinished pixel has visited fully
  const uint32_t contrib0 = (MODE == 2) ? (im.ranges[tile_g].y - im.ranges[tile_g].x) : 0u;
  int todo = (int)(range.y - range.x);
  for (uint32_t start = range.x; start < range.y; start += TILE_PIX, todo -= TILE_PIX) {
    if (__syncthreads_count(done) == TILE_PIX) break;
    const uint32_t e = start + threadIdx.x;
    int small = 0;
    if (e < range.y) {
      const size_t g = gbase + point_list[e];
      const float4 a0 = gs.g0[g];
      const float4 q = gs.g1[g];
      const float2 ext = alpha_extent(q);
      s_xy[threadIdx.x] = make_float4(a0.x, a0.y, ext.x, ext.y);
      s_co[threadIdx.x] = conic_log2(q);
      if constexpr (AUX) {
        const float4 c = gs.g2[g];
        s_rgb[threadIdx.x] = make_float4(c.x, c.y, c.z, a0.z);
      } else {
        s_rgb[threadIdx.x] = gs.g2[g];
      }
      small = ext.y < SKIP_WORTH;
    }
    const int use_skip = __syncthreads_or(small);  // dense chunks (every footprint covers the tile) keep the plain loop
    const int nb = min(TILE_PIX, todo);
    // Sparse chunks: every warp first compacts the staged entries whose footprint can reach its two pixel rows (and the
    // tile's 16 columns) into its own index list -- 8 tests per lane, ballot-compacted, order preserved -- and then runs the
    // SAME branch-free body over that list only.  A dropped entry is one the alpha test rejects for every pixel of the warp.
    int nw = nb;
    if (use_skip) {
      const int w_ = threadIdx.x >> 5, lane_ = threadIdx.x & 31;
      int cnt = 0;
#pragma unroll
      for (int r = 0; r < TILE_PIX / 32; r++) {
        const int j = r * 32 + lane_;
        bool hit = false;
        if (j < nb) {
          const float4 xy = s_xy[j];
          const float dyc = xy.y - wy0, dxc = xy.x - tx0;
          hit = !(dyc > 1.0f + xy.w || dyc < -xy.w || dxc > 15.0f + xy.z || dxc < -xy.z);
        }
        const unsigned m = __ballot_sync(0xffffffffu, hit);
        if (hit) s_list[w_][cnt + __popc(m & ((1u << lane_) - 1u))] = (uint8_t)j;
        cnt += __popc(m);
      }
      nw = cnt;
      __syncwarp();
    }
    // Branch-free body (the reference's three `continue`s become predicates): every lane evaluates every listed entry
    // until its whole warp is done; ~28 instructions per (pixel, entry) pair instead of 24 (rejected) / 54 (blended).
    // `contributor` (entries visited before the pixel was done, forward.cu:333) is positional: entry j of this chunk is
    // visit number cbase + j + 1 whether or not the warp evaluated the entries before it.
    const uint32_t cbase = contrib0 + (start - range.x);
    const uint8_t* lst = s_list[threadIdx.x >> 5];
    for (int k = 0; k < nw; k++) {
      if ((k & 3) == 0 && __all_sync(0xffffffffu, done)) break;
      const int j = use_skip ? (int)lst[k] : k;
      const float4 xy = s_xy[j];
      const float4 co = s_co[j];
      const float4 col = s_rgb[j];
      const float dx = xy.x - pxf, dy = xy.y - pyf;
      const float power2 = pair_power2(co, dx, dy);
      const float alpha = fminf(0.99f, co.w * ex2_mufu(power2));
      const uint32_t visit = cbase + (uint32_t)j + 1u;
      bool ok = !done && power2 <= 0.0f && alpha >= ALPHA_MIN;
      const float test_T = T * (1 - alpha);
      const bool sat = ok && test_T < T_EPS;
      contributor = sat ? visit : contributor;
      done |= sat;
      ok = ok && !sat;
      const float w = ok ? alpha * T : 0.f;
      C0 = fmaf(col.x, w, C0); C1 = fmaf(col.y, w, C1); C2 = fmaf(col.z, w, C2);
      if constexpr (AUX) D = fmaf(col.w, w, D);
      T = ok ? test_T : T;
      last = ok ? visit : last;
    }
    if (!done) contributor = cbase + (uint32_t)nb;  // every entry of the chunk was visited (an early break needs all done)
  }
  int unfinished = 0;
  if (MODE == 1) {
    // a pixel that ran out of phase-A entries without saturating must continue in phase B
    if (inside) {
      im.acc[pix_g] = make_float4(C0, C1, C2, T);
      im.contrib[pix_g] = contributor | (done ? 0x80000000u : 0u);
    }
    unfinished = __syncthreads_or(!done);
    if (threadIdx.x == 0) {
      im.tile_open[tile_g] = unfinished ? 1u : 0u;
      if (unfinished) atomicAdd(&gs.totals->unfinished, 1u);
    }
  }
  if (inside) {
    const size_t pid = (size_t)y * pb.W + x;
    const size_t ibase = (size_t)view * pb.W * pb.H;
    im.final_T[ibase + pid] = T;
    im.n_contrib[ibase + pid] = last;
    if constexpr (FRAMES) {
      uint8_t* px = reinterpret_cast<uint8_t*>(out_color) + 3 * (ibase + pid);
      px[0] = FramesFwd::quantise(C0 + T * pb.bg[0]);
      px[1] = FramesFwd::quantise(C1 + T * pb.bg[1]);
      px[2] = FramesFwd::quantise(C2 + T * pb.bg[2]);
    } else {
      float* oc = out_color + 3 * ibase;
      const size_t plane = (size_t)pb.W * pb.H;
      oc[pid] = C0 + T * pb.bg[0];
      oc[plane + pid] = C1 + T * pb.bg[1];
      oc[2 * plane + pid] = C2 + T * pb.bg[2];
    }
    if constexpr (AUX) {
      aux.depth[ibase + pid] = D;
      aux.alpha[ibase + pid] = 1.0f - T;
    }
  }
  if (mse.target) {
    // every pixel's FINAL colour is counted exactly once: phase A counts the tiles it finished, phase B the open ones
    const bool count = MODE == 0 ? true : MODE == 1 ? !unfinished : (im.tile_open[tile_g] != 0u);
    float e = 0.f;
    if (inside && count) {
      const size_t plane = (size_t)pb.W * pb.H, pid = (size_t)y * pb.W + x;
      const float* t = mse.target + (size_t)view * mse.tc * plane + pid;
      const float d0 = (C0 + T * pb.bg[0]) - t[0], d1 = (C1 + T * pb.bg[1]) - t[plane], d2 = (C2 + T * pb.bg[2]) - t[2 * plane];
      e = d0 * d0 + d1 * d1 + d2 * d2;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
    __shared__ float s_loss[TILE_PIX / 32];
    if ((threadIdx.x & 31) == 0) s_loss[threadIdx.x >> 5] = e;
    __syncthreads();
    if (threadIdx.x == 0 && count) {
      float tot = 0.f;
#pragma unroll
      for (int w = 0; w < TILE_PIX / 32; w++) tot += s_loss[w];
      atomicAdd(mse.loss + view / pb.V, (double)tot);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// K7: per-tile back-to-front gradient replay (backward.cu:399-557).
// Differences from the reference's data flow (not its math): starts at the deepest contributor of the
// tile instead of the end of the list; per-(pixel, Gaussian) terms are summed across the warp with
// shuffles, then across the CTA's 8 warps in shared memory, and only ONE atomic per gradient component
// per (tile, Gaussian) instance reaches L2 (the reference issues 9 atomics per contributing pair).
// ---------------------------------------------------------------------------------------------
using ptx::warp_sum;

constexpr int BWD_CHUNK = 64;  // Gaussians staged per round in the backward

// AUX: the depth / alpha gradients as well (see AuxFwd): a tenth reduced component, dL/dz, into aux.dz.
template <bool AUX = false>
__global__ void __launch_bounds__(TILE_PIX) blend_backward_kernel(Problem pb, GeomState gs, ImgState im,
                                                                  const uint32_t* __restrict__ point_list,
                                                                  const uint32_t* __restrict__ point_list_b,
                                                                  const float* __restrict__ dL_dpix, MseBwd mse,
                                                                  float* __restrict__ dmean2D /*[N,3]*/,
                                                                  float* __restrict__ dconic /*[N,4]*/,
                                                                  float* __restrict__ dopac /*[N]*/,
                                                                  float* __restrict__ dcolor /*[N,3]*/, AuxBwd aux) {
  constexpr int NC = AUX ? 10 : 9;  // reduced components per staged Gaussian
  const int tile_g = blockIdx.x;
  const int view = tile_g / pb.tiles, tile = tile_g - view * pb.tiles;
  const int tx = tile % pb.gx, ty = tile / pb.gx;
  const int lx = threadIdx.x & (TILE - 1), ly = threadIdx.x >> 4;
  const int x = tx * TILE + lx, y = ty * TILE + ly;
  const bool inside = x < pb.W && y < pb.H;
  const float pxf = (float)x, pyf = (float)y;
  const uint2 range = im.ranges[tile_g];
  const size_t gbase = (size_t)view * pb.P;
  const size_t ibase = (size_t)view * pb.W * pb.H;
  const size_t pid = (size_t)y * pb.W + x;
  const size_t plane = (size_t)pb.W * pb.H;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float wy0 = (float)(ty * TILE + warp * 2);  // this warp's first pixel row
  const float tx0 = (float)(tx * TILE);

  __shared__ uint32_t s_id[BWD_CHUNK];
  __shared__ float4 s_xy[BWD_CHUNK];  // x, y, x half-extent, y half-extent (alpha_extent)
  __shared__ float4 s_co[BWD_CHUNK];
  __shared__ float4 s_rgb[BWD_CHUNK];
  __shared__ float s_acc[BWD_CHUNK][NC];  // CTA-level partial sums per staged Gaussian
  __shared__ uint8_t s_list[TILE_PIX / 32][BWD_CHUNK];  // per-warp compacted slot indices
  __shared__ uint32_t s_max;

  const float T_final = inside ? im.final_T[ibase + pid] : 0.f;
  const uint32_t last = inside ? im.n_contrib[ibase + pid] : 0u;
  float dp0 = 0.f, dp1 = 0.f, dp2 = 0.f;
  if (inside) {
    if (dL_dpix) {
      const float* d = dL_dpix + 3 * ibase;
      dp0 = d[pid]; dp1 = d[plane + pid]; dp2 = d[2 * plane + pid];
    }
    if (mse.target) {  // + coef[sample] * (render - target): the MSE gradient, never stored as an image
      const float k = mse.coef[view / pb.V];
      const float* c = mse.images + 3 * ibase + pid;
      const float* t = mse.target + (size_t)view * mse.tc * plane + pid;
      dp0 = fmaf(k, c[0] - t[0], dp0); dp1 = fmaf(k, c[plane] - t[plane], dp1); dp2 = fmaf(k, c[2 * plane] - t[2 * plane], dp2);
    }
  }
  float dD = 0.f, dA = 0.f;
  if constexpr (AUX) {
    if (inside && aux.ddepth) dD = aux.ddepth[ibase + pid];
    if (inside && aux.dalpha) dA = aux.dalpha[ibase + pid];
  }
  if (threadIdx.x == 0) s_max = 0;
  __syncthreads();
  {
    uint32_t m = last;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) atomicMax(&s_max, m);
  }
  __syncthreads();
  const uint32_t deepest = s_max;  // entries [0, deepest) of this tile's list matter
  if (deepest == 0) return;
  const uint32_t len_a = range.y - range.x;
  const uint2 range_b = point_list_b ? im.ranges_b[tile_g] : make_uint2(0u, 0u);

  float T = T_final;
  float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, lc0 = 0.f, lc1 = 0.f, lc2 = 0.f, last_alpha = 0.f;
  float accD = 0.f, lz = 0.f;
  float bg_dot = pb.bg[0] * dp0 + pb.bg[1] * dp1 + pb.bg[2] * dp2;
  // alpha = 1 - T_final has d/dalpha_i = T_final / (1 - alpha_i): the background term's factor with the opposite sign
  if constexpr (AUX) bg_dot -= dA;
  const float ddelx_dx = 0.5f * pb.W, ddely_dy = 0.5f * pb.H;

  // walk positions deepest-1 ... 0 in chunks; within a chunk slot j holds position (top - j)
  for (int top = (int)deepest - 1; top >= 0; top -= BWD_CHUNK) {
    const int nb = min(BWD_CHUNK, top + 1);
    __syncthreads();  // previous chunk's s_acc fully flushed, staging buffers free
    if (threadIdx.x < nb) {
      // position in the tile's full depth-ordered list = phase-A entries followed by phase-B entries
      const uint32_t pos_t = (uint32_t)(top - (int)threadIdx.x);
      const uint32_t id = (pos_t < len_a) ? point_list[range.x + pos_t] : point_list_b[range_b.x + (pos_t - len_a)];
      const size_t g = gbase + id;
      s_id[threadIdx.x] = id;
      const float4 a0 = gs.g0[g];
      const float4 q = gs.g1[g];
      const float2 ext = alpha_extent(q);
      s_xy[threadIdx.x] = make_float4(a0.x, a0.y, ext.x, ext.y);
      s_co[threadIdx.x] = q;
      if constexpr (AUX) {
        const float4 c = gs.g2[g];
        s_rgb[threadIdx.x] = make_float4(c.x, c.y, c.z, a0.z);
      } else {
        s_rgb[threadIdx.x] = gs.g2[g];
      }
    }
    for (int t = threadIdx.x; t < nb * NC; t += TILE_PIX) (&s_acc[0][0])[t] = 0.f;
    __syncthreads();
    // per-warp compaction of the staged slots whose footprint can reach this warp's pixels (see alpha_extent and the
    // forward kernel); 2 tests per lane, order preserved
    int nw = 0;
    {
#pragma unroll
      for (int r = 0; r < BWD_CHUNK / 32; r++) {
        const int j = r * 32 + lane;
        bool hit = false;
        if (j < nb) {
          const float4 xy = s_xy[j];
          const float dyc = xy.y - wy0, dxc = xy.x - tx0;
          hit = !(dyc > 1.0f + xy.w || dyc < -xy.w || dxc > 15.0f + xy.z || dxc < -xy.z);
        }
        const unsigned m = __ballot_sync(0xffffffffu, hit);
        if (hit) s_list[warp][nw + __popc(m & ((1u << lane) - 1u))] = (uint8_t)j;
        nw += __popc(m);
      }
      __syncwarp();
    }
    for (int k = 0; k < nw; k++) {
      const int j = (int)s_list[warp][k];
      const uint32_t pos = (uint32_t)(top - j);  // 0-based position in the tile list
      float g_c0 = 0.f, g_c1 = 0.f, g_c2 = 0.f, g_mx = 0.f, g_my = 0.f, g_ca = 0.f, g_cb = 0.f, g_cc = 0.f, g_op = 0.f;
      float g_z = 0.f;
      bool active = false;
      const float4 xy = s_xy[j];
      if (pos < last) {
        const float dx = xy.x - pxf, dy = xy.y - pyf;
        const float4 co = s_co[j];
        const float power2 = pair_power2(conic_log2(co), dx, dy);  // same bits as the forward's decision
        if (power2 <= 0.0f) {
          const float G = ex2_mufu(power2);
          const float alpha = fminf(0.99f, co.w * G);
          if (alpha >= ALPHA_MIN) {
            active = true;
            T = T / (1.f - alpha);
            const float dch = alpha * T;
            const float4 col = s_rgb[j];
            acc0 = last_alpha * lc0 + (1.f - last_alpha) * acc0; lc0 = col.x;
            acc1 = last_alpha * lc1 + (1.f - last_alpha) * acc1; lc1 = col.y;
            acc2 = last_alpha * lc2 + (1.f - last_alpha) * acc2; lc2 = col.z;
            float dL_dalpha = (col.x - acc0) * dp0 + (col.y - acc1) * dp1 + (col.z - acc2) * dp2;
            if constexpr (AUX) {
              accD = last_alpha * lz + (1.f - last_alpha) * accD; lz = col.w;
              dL_dalpha += (col.w - accD) * dD;
              g_z = dch * dD;
            }
            g_c0 = dch * dp0; g_c1 = dch * dp1; g_c2 = dch * dp2;
            dL_dalpha *= T;
            last_alpha = alpha;
            dL_dalpha += (-T_final / (1.f - alpha)) * bg_dot;
            const float dL_dG = co.w * dL_dalpha;
            const float gdx = G * dx, gdy = G * dy;
            const float dG_ddelx = -gdx * co.x - gdy * co.y;
            const float dG_ddely = -gdy * co.z - gdx * co.y;
            g_mx = dL_dG * dG_ddelx * ddelx_dx;
            g_my = dL_dG * dG_ddely * ddely_dy;
            g_ca = -0.5f * gdx * dx * dL_dG;
            g_cb = -0.5f * gdx * dy * dL_dG;
            g_cc = -0.5f * gdy * dy * dL_dG;
            g_op = G * dL_dalpha;
          }
        }
      }
      if (__any_sync(0xffffffffu, active)) {
        // 9 sums over the 32 pixels of this warp.  Eight of them go through a halving butterfly (each step a lane
        // keeps half of its values and receives the partner's partial sums of that half): 4 + 2 + 1 + 1 + 1 shuffles
        // instead of 8 x 5; the ninth is a plain 5-step reduction.  14 shuffles instead of 45.
        float a0 = g_mx, a1 = g_my, a2 = g_ca, a3 = g_cb, a4 = g_cc, a5 = g_op, a6 = g_c0, a7 = g_c1;
        {
          const bool hi = lane & 16;
          const float s0 = hi ? a0 : a4, s1 = hi ? a1 : a5, s2 = hi ? a2 : a6, s3 = hi ? a3 : a7;
          a0 = (hi ? a4 : a0) + __shfl_xor_sync(0xffffffffu, s0, 16);
          a1 = (hi ? a5 : a1) + __shfl_xor_sync(0xffffffffu, s1, 16);
          a2 = (hi ? a6 : a2) + __shfl_xor_sync(0xffffffffu, s2, 16);
          a3 = (hi ? a7 : a3) + __shfl_xor_sync(0xffffffffu, s3, 16);
        }
        {
          const bool hi = lane & 8;
          const float s0 = hi ? a0 : a2, s1 = hi ? a1 : a3;
          a0 = (hi ? a2 : a0) + __shfl_xor_sync(0xffffffffu, s0, 8);
          a1 = (hi ? a3 : a1) + __shfl_xor_sync(0xffffffffu, s1, 8);
        }
        {
          const bool hi = lane & 4;
          const float s0 = hi ? a0 : a1;
          a0 = (hi ? a1 : a0) + __shfl_xor_sync(0xffffffffu, s0, 4);
        }
        a0 += __shfl_xor_sync(0xffffffffu, a0, 2);
        a0 += __shfl_xor_sync(0xffffffffu, a0, 1);
        g_c2 = warp_sum(g_c2);
        // lane L (L % 4 == 0) now holds component ((L>>4)&1)*4 + ((L>>3)&1)*2 + ((L>>2)&1) of
        // {mean.x, mean.y, conic.a, conic.b, conic.c, opacity, colour.r, colour.g}
        if ((lane & 3) == 0) atomicAdd(&s_acc[j][((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1)], a0);
        if (lane == 1) atomicAdd(&s_acc[j][8], g_c2);
        if constexpr (AUX) {
          g_z = warp_sum(g_z);
          if (lane == 2) atomicAdd(&s_acc[j][9], g_z);
        }
      }
    }
    __syncthreads();
    // flush: one global atomic per component per staged Gaussian
    for (int t = threadIdx.x; t < nb * NC; t += TILE_PIX) {
      const int j = t / NC, c = t - NC * j;
      const float v = s_acc[j][c];
      if (v != 0.f) {
        const size_t g = gbase + s_id[j];
        float* dst;
        switch (c) {
          case 0: dst = dmean2D + 3 * g; break;
          case 1: dst = dmean2D + 3 * g + 1; break;
          case 2: dst = dconic + 4 * g; break;
          case 3: dst = dconic + 4 * g + 1; break;
          case 4: dst = dconic + 4 * g + 3; break;
          case 5: dst = dopac + g; break;
          default: dst = dcolor + 3 * g + (c - 6); break;
        }
        if constexpr (AUX) {
          if (c == 9) dst = aux.dz + g;
        }
        atomicAdd(dst, v);
      }
    }
  }
  (void)warp;
}

// ---------------------------------------------------------------------------------------------
// K8 + K9 fused, plus (raw mode) the activation Jacobians and the sum over a sample's views.
// One thread per (sample, Gaussian); loops over that sample's V views.
// ---------------------------------------------------------------------------------------------
struct GeomGradOut {
  float* dmeans;   // [S*P,3]
  float* dcov3d;   // [S*P,6] or null (single-view API only)
  float* dsh;      // [S*P,M,3] or null
  float* dscale;   // [S*P,3] or null
  float* drot;     // [S*P,4] or null
  float* dopac_raw;  // [S*P] raw-opacity gradient (batched mode) or null
};

// AUX: plus dL/dz (blend_backward_kernel<true>'s tenth component) through z = W2C[2] . (mean, 1)
template <bool AUX = false>
__global__ void __launch_bounds__(256) geometry_backward_kernel(Problem pb, GeomState gs, const int* __restrict__ radii_in,
                                                                const float* __restrict__ dmean2D,
                                                                const float* __restrict__ dconic,
                                                                const float* __restrict__ dopac,
                                                                const float* __restrict__ dcolor, GeomGradOut out,
                                                                const float* __restrict__ dz) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int s = blockIdx.y;
  if (i >= pb.P) return;
  const size_t si = (size_t)s * pb.P + i;
  const float3 mean = ld3(pb.means, si);
  float3 scale = make_float3(0.f, 0.f, 0.f);
  float4 q = make_float4(0.f, 0.f, 0.f, 0.f), q_raw = q;
  float inv_norm = 1.f;
  const bool has_sr = pb.scales != nullptr;
  if (has_sr) {
    scale = ld3(pb.scales, si);
    q_raw = ld4(pb.rots, si);
    q = q_raw;
    if (pb.raw) { scale = act_scale(scale); q = act_rot(q_raw, &inv_norm); }
  }
  // The covariance chain (cov3D -> cov2D -> conic and back to scale / rotation) runs in fp64: for a needle-shaped
  // Gaussian the 2D covariance is close to singular (a c ~ b^2), and in fp32 the cancellation in its determinant and
  // in the rotation gradient (differences of nearly equal terms) costs up to ~1e-2 relative on that Gaussian.
  double c6d[6];
  if (pb.cov_pre) {
#pragma unroll
    for (int k = 0; k < 6; k++) c6d[k] = pb.cov_pre[6 * si + k];
  } else {
    double R[3][3];
    quat_to_rot_d(q, R);
    const double sv[3] = {(double)pb.mod * scale.x, (double)pb.mod * scale.y, (double)pb.mod * scale.z};
    double S[3][3];
#pragma unroll
    for (int r_ = 0; r_ < 3; r_++)
#pragma unroll
      for (int k = 0; k < 3; k++)
        S[r_][k] = R[r_][0] * sv[0] * sv[0] * R[k][0] + R[r_][1] * sv[1] * sv[1] * R[k][1] + R[r_][2] * sv[2] * sv[2] * R[k][2];
    c6d[0] = S[0][0]; c6d[1] = S[0][1]; c6d[2] = S[0][2]; c6d[3] = S[1][1]; c6d[4] = S[1][2]; c6d[5] = S[2][2];
  }
  double V[3][3];
  V[0][0] = c6d[0]; V[0][1] = V[1][0] = c6d[1]; V[0][2] = V[2][0] = c6d[2];
  V[1][1] = c6d[3]; V[1][2] = V[2][1] = c6d[4]; V[2][2] = c6d[5];
  const int nb = (pb.D + 1) * (pb.D + 1);
  const bool sh_general = pb.shs && pb.D > 0;
  float* dsh_out = (pb.shs && out.dsh) ? out.dsh + si * pb.M * 3 : nullptr;
  if (sh_general)
    for (int k = 0; k < pb.M * 3; k++) dsh_out[k] = 0.f;

  float dm[3] = {0.f, 0.f, 0.f}, dsh0[3] = {0.f, 0.f, 0.f};
  double dc6[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  float dop_sum = 0.f;

  for (int v = 0; v < pb.V; v++) {
    const int view = s * pb.V + v;
    const size_t n = (size_t)view * pb.P + i;
    const int radius = radii_in ? radii_in[n] : __float_as_int(gs.g0[n].w);
    if (!(radius > 0)) continue;
    const Camera& cam = gs.cams[view];
    // ---- conic -> cov2D -> cov3D & mean (backward.cu:144-274) ----
    Ewa e;
    ewa_setup(mean, cam, e);  // the frustum clamp decisions, as in the forward
    const float xmul = (e.txtz < -e.limx || e.txtz > e.limx) ? 0.f : 1.f;
    const float ymul = (e.tytz < -e.limy || e.tytz > e.limy) ? 0.f : 1.f;
    // view-space mean and the EWA Jacobian times the view rotation, in fp64
    const float* vm = cam.view;
    double tv[3];
#pragma unroll
    for (int k = 0; k < 3; k++) tv[k] = (double)vm[k] * mean.x + (double)vm[4 + k] * mean.y + (double)vm[8 + k] * mean.z + vm[12 + k];
    if (!xmul) tv[0] = (e.txtz < 0.f ? -(double)e.limx : (double)e.limx) * tv[2];
    if (!ymul) tv[1] = (e.tytz < 0.f ? -(double)e.limy : (double)e.limy) * tv[2];
    const double j00 = cam.fx / tv[2], j02 = -(cam.fx * tv[0]) / (tv[2] * tv[2]);
    const double j11 = cam.fy / tv[2], j12 = -(cam.fy * tv[1]) / (tv[2] * tv[2]);
    double A[2][3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
      A[0][k] = vm[4 * k + 0] * j00 + vm[4 * k + 2] * j02;
      A[1][k] = vm[4 * k + 1] * j11 + vm[4 * k + 2] * j12;
    }
    double a, b, c;
    {
      double va0[3], va1[3];
#pragma unroll
      for (int k = 0; k < 3; k++) {
        va0[k] = V[k][0] * A[0][0] + V[k][1] * A[0][1] + V[k][2] * A[0][2];
        va1[k] = V[k][0] * A[1][0] + V[k][1] * A[1][1] + V[k][2] * A[1][2];
      }
      a = A[0][0] * va0[0] + A[0][1] * va0[1] + A[0][2] * va0[2] + 0.3;
      b = A[0][0] * va1[0] + A[0][1] * va1[1] + A[0][2] * va1[2];
      c = A[1][0] * va1[0] + A[1][1] * va1[1] + A[1][2] * va1[2] + 0.3;
    }
    const double dcx = dconic[4 * n], dcy = dconic[4 * n + 1], dcz = dconic[4 * n + 3];
    const double denom = a * c - b * b;
    double da = 0.0, db = 0.0, dc = 0.0;
    const double denom2inv = 1.0 / ((denom * denom) + (double)0.0000001f);
    if (denom2inv != 0) {
      da = denom2inv * (-c * c * dcx + 2 * b * c * dcy + (denom - a * c) * dcz);
      dc = denom2inv * (-a * a * dcz + 2 * a * b * dcy + (denom - a * c) * dcx);
      db = denom2inv * 2 * (b * c * dcx - (denom + 2 * b * b) * dcy + a * b * dcz);
      dc6[0] += A[0][0] * A[0][0] * da + A[0][0] * A[1][0] * db + A[1][0] * A[1][0] * dc;
      dc6[3] += A[0][1] * A[0][1] * da + A[0][1] * A[1][1] * db + A[1][1] * A[1][1] * dc;
      dc6[5] += A[0][2] * A[0][2] * da + A[0][2] * A[1][2] * db + A[1][2] * A[1][2] * dc;
      dc6[1] += 2 * A[0][0] * A[0][1] * da + (A[0][0] * A[1][1] + A[0][1] * A[1][0]) * db + 2 * A[1][0] * A[1][1] * dc;
      dc6[2] += 2 * A[0][0] * A[0][2] * da + (A[0][0] * A[1][2] + A[0][2] * A[1][0]) * db + 2 * A[1][0] * A[1][2] * dc;
      dc6[4] += 2 * A[0][2] * A[0][1] * da + (A[0][1] * A[1][2] + A[0][2] * A[1][1]) * db + 2 * A[1][1] * A[1][2] * dc;
    }
    double dA0[3], dA1[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const double va0 = A[0][0] * V[k][0] + A[0][1] * V[k][1] + A[0][2] * V[k][2];
      const double va1 = A[1][0] * V[k][0] + A[1][1] * V[k][1] + A[1][2] * V[k][2];
      dA0[k] = 2 * va0 * da + va1 * db;
      dA1[k] = 2 * va1 * dc + va0 * db;
    }
    const double dJ00 = vm[0] * dA0[0] + vm[4] * dA0[1] + vm[8] * dA0[2];
    const double dJ02 = vm[2] * dA0[0] + vm[6] * dA0[1] + vm[10] * dA0[2];
    const double dJ11 = vm[1] * dA1[0] + vm[5] * dA1[1] + vm[9] * dA1[2];
    const double dJ12 = vm[2] * dA1[0] + vm[6] * dA1[1] + vm[10] * dA1[2];
    const double tz = 1.0 / tv[2], tz2 = tz * tz, tz3 = tz2 * tz;
    const double dtx = xmul * -cam.fx * tz2 * dJ02;
    const double dty = ymul * -cam.fy * tz2 * dJ12;
    const double dtz = -cam.fx * tz2 * dJ00 - cam.fy * tz2 * dJ11 + (2 * cam.fx * tv[0]) * tz3 * dJ02 +
                       (2 * cam.fy * tv[1]) * tz3 * dJ12;
    float dmv[3];
    dmv[0] = (float)(vm[0] * dtx + vm[1] * dty + vm[2] * dtz);
    dmv[1] = (float)(vm[4] * dtx + vm[5] * dty + vm[6] * dtz);
    dmv[2] = (float)(vm[8] * dtx + vm[9] * dty + vm[10] * dtz);
    // ---- mean2D -> mean3D (backward.cu:366-387) ----
    const float* pm = cam.proj;
    const float4 mh = xform44(pm, mean);
    const float mw = 1.0f / (mh.w + 0.0000001f);
    const float mul1 = mh.x * mw * mw, mul2 = mh.y * mw * mw;
    const float gx2 = dmean2D[3 * n], gy2 = dmean2D[3 * n + 1];
    dmv[0] += (pm[0] * mw - pm[3] * mul1) * gx2 + (pm[1] * mw - pm[3] * mul2) * gy2;
    dmv[1] += (pm[4] * mw - pm[7] * mul1) * gx2 + (pm[5] * mw - pm[7] * mul2) * gy2;
    dmv[2] += (pm[8] * mw - pm[11] * mul1) * gx2 + (pm[9] * mw - pm[11] * mul2) * gy2;
    if constexpr (AUX) {
      const float gz = dz[n];
      dmv[0] += vm[2] * gz; dmv[1] += vm[6] * gz; dmv[2] += vm[10] * gz;
    }
    // ---- colour -> SH (backward.cu:20-139) ----
    if (pb.shs) {
      const int clamped = __float_as_int(gs.g2[n].w);
      float g[3];
#pragma unroll
      for (int ch = 0; ch < 3; ch++) g[ch] = dcolor[3 * n + ch] * ((clamped >> ch) & 1 ? 0.f : 1.f);
      if (!sh_general) {
#pragma unroll
        for (int ch = 0; ch < 3; ch++) dsh0[ch] += kSH0 * g[ch];
      } else {
        const float ox = mean.x - cam.campos[0], oy = mean.y - cam.campos[1], oz = mean.z - cam.campos[2];
        const float len = sqrtf(ox * ox + oy * oy + oz * oz);
        float bs[16], dbs[16][3];
        sh_basis<true>(pb.D, ox / len, oy / len, oz / len, bs, dbs);
        const float* sh = pb.shs + si * pb.M * 3;
        float ddir[3] = {0.f, 0.f, 0.f};
        for (int k = 0; k < nb; k++) {
          float dot = 0.f;
#pragma unroll
          for (int ch = 0; ch < 3; ch++) {
            dsh_out[3 * k + ch] += bs[k] * g[ch];
            dot += sh[3 * k + ch] * g[ch];
          }
#pragma unroll
          for (int ax = 0; ax < 3; ax++) ddir[ax] += dbs[k][ax] * dot;
        }
        const float s2 = ox * ox + oy * oy + oz * oz;  // dnormvdv, auxiliary.h:107-117
        const float inv32 = 1.0f / sqrtf(s2 * s2 * s2);
        dmv[0] += ((+s2 - ox * ox) * ddir[0] - oy * ox * ddir[1] - oz * ox * ddir[2]) * inv32;
        dmv[1] += (-ox * oy * ddir[0] + (s2 - oy * oy) * ddir[1] - oz * oy * ddir[2]) * inv32;
        dmv[2] += (-ox * oz * ddir[0] - oy * oz * ddir[1] + (s2 - oz * oz) * ddir[2]) * inv32;
      }
    }
    dm[0] += dmv[0]; dm[1] += dmv[1]; dm[2] += dmv[2];
    dop_sum += dopac[n];
  }

  out.dmeans[3 * si] = dm[0]; out.dmeans[3 * si + 1] = dm[1]; out.dmeans[3 * si + 2] = dm[2];
  if (out.dcov3d) {
#pragma unroll
    for (int k = 0; k < 6; k++) out.dcov3d[6 * si + k] = (float)dc6[k];
  }
  if (dsh_out && !sh_general) {
    dsh_out[0] = dsh0[0]; dsh_out[1] = dsh0[1]; dsh_out[2] = dsh0[2];
    for (int k = 3; k < pb.M * 3; k++) dsh_out[k] = 0.f;
  }
  if (out.dopac_raw) {
    const float o = act_opacity(pb.opac[si]);
    out.dopac_raw[si] = dop_sum * o * (1.f - o);
  }
  // ---- cov3D -> scale / rotation (backward.cu:278-341), fp64; linear in dL/dcov3D, so the per-view sum is
  // pushed through once ----
  if (has_sr && out.dscale) {
    double R[3][3], Mm[3][3], dS[3][3], dM[3][3], E[3][3];
    quat_to_rot_d(q, R);
    const double sv[3] = {(double)pb.mod * scale.x, (double)pb.mod * scale.y, (double)pb.mod * scale.z};
#pragma unroll
    for (int r_ = 0; r_ < 3; r_++)
#pragma unroll
      for (int k = 0; k < 3; k++) Mm[r_][k] = sv[r_] * R[k][r_];
    dS[0][0] = dc6[0]; dS[0][1] = dS[1][0] = 0.5 * dc6[1]; dS[0][2] = dS[2][0] = 0.5 * dc6[2];
    dS[1][1] = dc6[3]; dS[1][2] = dS[2][1] = 0.5 * dc6[4]; dS[2][2] = dc6[5];
#pragma unroll
    for (int r_ = 0; r_ < 3; r_++)
#pragma unroll
      for (int k = 0; k < 3; k++) dM[r_][k] = 2.0 * (Mm[r_][0] * dS[0][k] + Mm[r_][1] * dS[1][k] + Mm[r_][2] * dS[2][k]);
    double dsc[3];
#pragma unroll
    for (int r_ = 0; r_ < 3; r_++) dsc[r_] = R[0][r_] * dM[r_][0] + R[1][r_] * dM[r_][1] + R[2][r_] * dM[r_][2];
#pragma unroll
    for (int a_ = 0; a_ < 3; a_++)
#pragma unroll
      for (int b_ = 0; b_ < 3; b_++) E[a_][b_] = sv[b_] * dM[b_][a_];
    const double r = q.x, x = q.y, y = q.z, z = q.w;
    double dq[4];
    dq[0] = 2 * z * (E[1][0] - E[0][1]) + 2 * y * (E[0][2] - E[2][0]) + 2 * x * (E[2][1] - E[1][2]);
    dq[1] = 2 * y * (E[0][1] + E[1][0]) + 2 * z * (E[0][2] + E[2][0]) + 2 * r * (E[2][1] - E[1][2]) - 4 * x * (E[2][2] + E[1][1]);
    dq[2] = 2 * x * (E[0][1] + E[1][0]) + 2 * r * (E[0][2] - E[2][0]) + 2 * z * (E[2][1] + E[1][2]) - 4 * y * (E[2][2] + E[0][0]);
    dq[3] = 2 * r * (E[1][0] - E[0][1]) + 2 * x * (E[0][2] + E[2][0]) + 2 * y * (E[2][1] + E[1][2]) - 4 * z * (E[1][1] + E[0][0]);
    // dsc is dL/d(mod * scale), the reference rasterizer's convention (backward.cu:295-325), which the activated
    // (single-view) path returns as it is.  The raw (batched) path follows GaussianModel.get_scaling instead:
    // S = exp(s_raw) * mod outside a rasterizer run with mod = 1, so d/ds_raw = d/dS * mod * exp(s_raw).
    if (pb.raw) {
      // exp: d/ds_raw = d/d(mod scale) * mod * scale ; normalize: (dq - q (q.dq)) / max(|q_raw|, eps)
      dsc[0] *= (double)pb.mod * scale.x; dsc[1] *= (double)pb.mod * scale.y; dsc[2] *= (double)pb.mod * scale.z;
      const double dot = r * dq[0] + x * dq[1] + y * dq[2] + z * dq[3];
      dq[0] = (dq[0] - r * dot) * inv_norm; dq[1] = (dq[1] - x * dot) * inv_norm;
      dq[2] = (dq[2] - y * dot) * inv_norm; dq[3] = (dq[3] - z * dot) * inv_norm;
    }
    out.dscale[3 * si] = (float)dsc[0]; out.dscale[3 * si + 1] = (float)dsc[1]; out.dscale[3 * si + 2] = (float)dsc[2];
    *reinterpret_cast<float4*>(out.drot + 4 * si) = make_float4((float)dq[0], (float)dq[1], (float)dq[2], (float)dq[3]);
  }
}

__global__ void mark_visible_kernel(int P, const float* __restrict__ means, const float* __restrict__ view,
                                    uint8_t* __restrict__ present) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  float3 pv = xform43(view, ld3(means, i));
  present[i] = pv.z > NEAR_Z;
}

__global__ void export_geom_kernel(size_t N, GeomState gs, float* xy, float* depth, float* conic_opacity,
                                   float* rgb, uint32_t* tiles) {
  size_t n = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float4 a = gs.g0[n], b = gs.g1[n], c = gs.g2[n];
  bool vis = __float_as_int(a.w) > 0;
  if (xy) { xy[2 * n] = a.x; xy[2 * n + 1] = a.y; }
  if (depth) depth[n] = a.z;
  if (conic_opacity) { conic_opacity[4 * n] = b.x; conic_opacity[4 * n + 1] = b.y; conic_opacity[4 * n + 2] = b.z; conic_opacity[4 * n + 3] = b.w; }
  if (rgb) { rgb[3 * n] = vis ? c.x : 0.f; rgb[3 * n + 1] = vis ? c.y : 0.f; rgb[3 * n + 2] = vis ? c.z : 0.f; }
  if (tiles) tiles[n] = gs.tiles[n];
}

// ---------------------------------------------------------------------------------------------
// host-side pipeline
// ---------------------------------------------------------------------------------------------
static int bits_for(uint32_t n) {  // smallest b with (n >> b) == 0  (getHigherMsb, rasterizer_impl.cu:35-50)
  int b = 0;
  while (b < 32 && (n >> b)) b++;
  return b;
}

struct Allocators {  // the caller's arena callbacks: geometry, binning (once per bin pass) and image state
  dgs_alloc_fn geom; void* geom_user;
  dgs_alloc_fn bin; void* bin_user;
  dgs_alloc_fn img; void* img_user;
};

// Batched: C2W and fxfycxcy per view (build_cameras_kernel).  Single view (c2w == nullptr): the view and projection
// matrices, camera position and tan(fov) of GaussianRasterizationSettings (pack_camera_kernel).
struct CameraInput {
  const float* c2w = nullptr;
  const float* fxfycxcy = nullptr;
  const float* view = nullptr;
  const float* proj = nullptr;
  const float* campos = nullptr;
  float tanx = 0.f, tany = 0.f;
};

struct Forward {  // one forward's problem, arenas and launch context, shared by its stages
  Problem pb;
  GeomState gs;
  ImgState im;
  Allocators al;
  float* out_color;
  MseFwd mse;
  AuxFwd aux;
  uint8_t* frames;   // set: uint8 frames [NV,H,W,3] instead of out_color
  cudaStream_t st;
  int debug;
  size_t N, ntiles;  // view-Gaussians, view-tiles
  dim3 pgrid() const { return dim3(ceil_div(pb.P, 256), pb.NV); }
};

static int alloc_binning(const Forward& f, long long R, BinState* bs) {
  size_t bytes = 0;
  BinState::carve(nullptr, R, &bytes);
  void* buf = f.al.bin(bytes, f.al.bin_user);
  if (!buf) { set_error("binning allocator returned NULL"); return DGS_ERR_ALLOC; }
  *bs = BinState::carve(buf, R, nullptr);
  return DGS_OK;
}

template <int MODE>
static int blend_forward(const Forward& f, const uint32_t* point_list) {
  ProfScope ps(f.st, PROF_RASTER_BLEND_FWD);
  if (f.frames)
    blend_forward_kernel<MODE, false, true><<<(unsigned)f.ntiles, TILE_PIX, 0, f.st>>>(
        f.pb, f.gs, f.im, point_list, reinterpret_cast<float*>(f.frames), f.mse, f.aux);
  else if (!f.aux.depth)
    blend_forward_kernel<MODE><<<(unsigned)f.ntiles, TILE_PIX, 0, f.st>>>(f.pb, f.gs, f.im, point_list, f.out_color, f.mse,
                                                                          f.aux);
  else
    blend_forward_kernel<MODE, true><<<(unsigned)f.ntiles, TILE_PIX, 0, f.st>>>(f.pb, f.gs, f.im, point_list, f.out_color,
                                                                                f.mse, f.aux);
  DGS_LAUNCH_OK(f.st, f.debug);
  return DGS_OK;
}

static int project(const Forward& f, const CameraInput& cam, int* radii) {
  if (cam.c2w) {
    build_cameras_kernel<<<ceil_div(f.pb.NV, 64), 64, 0, f.st>>>(f.pb.NV, cam.c2w, cam.fxfycxcy, f.pb.W, f.pb.H, f.gs.cams);
  } else {
    pack_camera_kernel<<<1, 32, 0, f.st>>>(cam.view, cam.proj, cam.campos, cam.tanx, cam.tany, f.pb.W, f.pb.H, f.gs.cams);
  }
  DGS_LAUNCH_OK(f.st, f.debug);
  ProfScope ps(f.st, PROF_RASTER_PROJECT);
  project_kernel<<<f.pgrid(), 256, 0, f.st>>>(f.pb, f.gs, radii);
  DGS_LAUNCH_OK(f.st, f.debug);
  return DGS_OK;
}

// Small-scene binning and blend.  *done = false: a tile list is longer than the shared-memory sort takes, and the
// caller bins globally instead (the projection's outputs stand).
static int bin_small(const Forward& f, long long* R_out, bool* done) {
  // no phase B on this path: its image arrays hold the per-tile instance counts and the fill cursors
  uint32_t* tile_counts = f.im.tile_open;
  uint2* fill_cursor = f.im.ranges_b;
  BinTotals tot;
  DGS_CUDA_OK(cudaMemsetAsync(tile_counts, 0, f.ntiles * sizeof(uint32_t), f.st));
  {
    ProfScope ps(f.st, PROF_RASTER_SCAN);
    tile_count_fill_kernel<false><<<f.pgrid(), 256, 0, f.st>>>(f.pb, f.gs, tile_counts, nullptr, nullptr, nullptr);
    DGS_LAUNCH_OK(f.st, f.debug);
    tile_scan_kernel<<<1, 1024, 0, f.st>>>((int)f.ntiles, tile_counts, f.im.ranges, fill_cursor, f.gs.totals);
    DGS_LAUNCH_OK(f.st, f.debug);
    DGS_CUDA_OK(cudaMemcpyAsync(&tot, f.gs.totals, sizeof(tot), cudaMemcpyDeviceToHost, f.st));
    DGS_CUDA_OK(cudaStreamSynchronize(f.st));  // the one host sync of the batch
  }
  *done = tot.longest <= (uint32_t)SMALL_TILE_CAP;
  if (!*done) return DGS_OK;
  const long long R = (long long)tot.R;
  *R_out = R;
  BinState bs;
  int rc = alloc_binning(f, R, &bs);
  if (rc) return rc;
  if (R > 0) {
    {
      ProfScope ps(f.st, PROF_RASTER_EMIT);
      tile_count_fill_kernel<true><<<f.pgrid(), 256, 0, f.st>>>(f.pb, f.gs, nullptr, fill_cursor, bs.keys_in, bs.vals_in);
      DGS_LAUNCH_OK(f.st, f.debug);
    }
    ProfScope ps(f.st, PROF_RASTER_SORT);
    int cap = 2;
    while (cap < (int)tot.longest) cap <<= 1;
    static bool configured = false;
    if (!configured) {
      DGS_CUDA_OK(cudaFuncSetAttribute(tile_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMALL_TILE_CAP * 8));
      configured = true;
    }
    tile_sort_kernel<<<(unsigned)f.ntiles, 256, (size_t)cap * 8, f.st>>>(f.im.ranges, bs.keys_in, bs.vals_in, bs.point_list);
    DGS_LAUNCH_OK(f.st, f.debug);
  }
  return blend_forward<0>(f, bs.point_list);
}

// per-view depth ranking of the Gaussians, and the instance offsets in rank order
static int rank_and_scan(const Forward& f) {
  ProfScope ps(f.st, PROF_RASTER_SCAN);
  GeomState gs = f.gs;  // (cub takes the temp size by reference)
  const int depth_end_bit = 32 + bits_for((uint32_t)f.pb.NV);
  DGS_CUDA_OK(cub::DeviceRadixSort::SortPairs(gs.scan_temp, gs.scan_bytes, gs.dkey_in, gs.dkey, gs.perm_in, gs.perm,
                                              (int)f.N, 0, depth_end_bit, f.st));
  DGS_CUDA_OK(cudaMemsetAsync(gs.totals, 0, sizeof(BinTotals), f.st));
  gather_tiles_kernel<<<(unsigned)((f.N + 255) / 256), 256, 0, f.st>>>(f.N, f.pb.P, gs);
  DGS_LAUNCH_OK(f.st, f.debug);
  DGS_CUDA_OK(cub::DeviceScan::InclusiveSum(gs.scan_temp, gs.scan_bytes, gs.tiles_sorted, gs.offsets, (int)f.N, f.st));
  return DGS_OK;
}

struct Split {                // how the global path bins
  long long R;                // instances of the batch
  long long RA;               // instances of the first (or only) bin pass
  int Pn;                     // two-phase: near ranks per view binned in phase A; 0: one pass over every rank
  const uint32_t* near_meta;  // two-phase: chunk_meta_kernel's output for Pn
};

// The split decision, after the one host sync of the global path.  near_log2 > 0: phase A = the nearest P >> near_log2
// Gaussians of every view; 0: single pass; < 0 adaptive: the splits at 1/8 and 1/16 are both prepared and the host picks
// 1/16 when its near lists are still long enough to saturate the pixels (>= 2048 entries per tile on average: the dense
// random-init step), 1/8 otherwise (sparser lists leave the near pass short of work).  Phase A must be a real saving:
// at most half of the instances, in a batch of at least 2^21.
static int plan_split(const Forward& f, Split* sp) {
  const Problem& pb = f.pb;
  const GeomState& gs = f.gs;
  const bool adaptive = pb.near_log2 < 0;
  const int k_a = adaptive ? 3 : pb.near_log2;
  int Pn = (k_a > 0) ? (pb.P >> k_a) : 0;
  const int Pn_b = adaptive ? (pb.P >> 4) : 0;
  const bool may_split = Pn >= 1024;
  const bool two_cands = adaptive && Pn_b >= 1024;
  uint32_t* const meta_b = gs.view_meta + (size_t)pb.NV * 2;
  BinTotals tot = {};
  if (may_split) {
    chunk_meta_kernel<<<1, 32, 0, f.st>>>(pb.NV, pb.P, Pn, gs.offsets, gs.view_meta, gs.totals, &gs.totals->R_near);
    if (two_cands) chunk_meta_kernel<<<1, 32, 0, f.st>>>(pb.NV, pb.P, Pn_b, gs.offsets, meta_b, gs.totals, &gs.totals->R_near_b);
    DGS_LAUNCH_OK(f.st, f.debug);
    DGS_CUDA_OK(cudaMemcpyAsync(&tot, gs.totals, sizeof(tot), cudaMemcpyDeviceToHost, f.st));
  } else {
    DGS_CUDA_OK(cudaMemcpyAsync(&tot.R, gs.offsets + f.N - 1, sizeof(tot.R), cudaMemcpyDeviceToHost, f.st));
    DGS_CUDA_OK(cudaMemcpyAsync(&tot.R64, &gs.totals->R64, sizeof(tot.R64), cudaMemcpyDeviceToHost, f.st));
  }
  DGS_CUDA_OK(cudaStreamSynchronize(f.st));  // the one host sync per batch (two-phase: a second, after phase A)
  if (tot.R64 >= (unsigned long long)INT32_MAX) {
    set_error("instance count %lld exceeds 2^31-1 (render the views in smaller batches)", (long long)tot.R64);
    return DGS_ERR_OVERFLOW;
  }
  const long long R = (long long)tot.R;
  uint32_t R_near = tot.R_near;
  const uint32_t* near_meta = gs.view_meta;
  if (two_cands && (unsigned long long)tot.R_near_b >= 2048ull * (unsigned long long)pb.NV * pb.tiles) {
    Pn = Pn_b;
    R_near = tot.R_near_b;
    near_meta = meta_b;
  }
  const bool split = may_split && R >= (1ll << 21) && 2ll * R_near <= R && R_near > 0;
  sp->R = R;
  sp->RA = split ? (long long)R_near : R;
  sp->Pn = split ? Pn : 0;
  sp->near_meta = split ? near_meta : nullptr;
  return DGS_OK;
}

struct Emission {             // which instances a bin pass emits
  int rank_lo, rank_hi;       // depth ranks of every view
  bool open_only;             // phase B: only the tiles still open after phase A
  const uint32_t* near_meta;  // phase A: rebase into the compact near buffer (Split::near_meta)
};

// One binning pass into its own arena: allocate -> zero the ranges -> emit -> stable sort by tile -> tile ranges
static int bin_pass(const Forward& f, long long R, const Emission& e, uint2* ranges, BinState* bs) {
  int rc = alloc_binning(f, R, bs);
  if (rc) return rc;
  DGS_CUDA_OK(cudaMemsetAsync(ranges, 0, f.ntiles * sizeof(uint2), f.st));
  if (R == 0) return DGS_OK;
  {
    ProfScope ps(f.st, PROF_RASTER_EMIT);
    const dim3 grid(ceil_div(e.rank_hi - e.rank_lo, 256), f.pb.NV);
    if (e.open_only)
      emit_keys_kernel<true><<<grid, 256, 0, f.st>>>(f.pb, f.gs, f.im.tile_open, nullptr, bs->keys_in, bs->vals_in,
                                                     e.rank_lo, e.rank_hi);
    else
      emit_keys_kernel<false><<<grid, 256, 0, f.st>>>(f.pb, f.gs, nullptr, e.near_meta, bs->keys_in, bs->vals_in,
                                                      e.rank_lo, e.rank_hi);
    DGS_LAUNCH_OK(f.st, f.debug);
  }
  {
    ProfScope ps(f.st, PROF_RASTER_SORT);  // tile ids only: depth order is already in the emission order
    DGS_CUDA_OK(cub::DeviceRadixSort::SortPairs(bs->sort_temp, bs->sort_bytes, bs->keys_in, bs->keys, bs->vals_in,
                                                bs->point_list, (int)R, 0, bits_for((uint32_t)f.ntiles), f.st));
  }
  ProfScope ps(f.st, PROF_RASTER_RANGES);
  tile_ranges_kernel<<<(unsigned)((R + 255) / 256), 256, 0, f.st>>>(R, bs->keys, ranges);
  DGS_LAUNCH_OK(f.st, f.debug);
  return DGS_OK;
}

// Two-phase binning.  Phase A: the nearest Pn Gaussians of every view.  In dense scenes every pixel saturates here and
// the remaining instances are never emitted, sorted or read.  Phase B: everything behind the near ranks, for the OPEN
// tiles only, continuing from the saved per-pixel state.  A tile that saturated in phase A never looks at its far
// entries, so they are neither counted, emitted nor sorted; an open tile gets every far Gaussian of its rect, in the
// same (depth, index) order as the single-pass list.
static int bin_two_phase(const Forward& f, const Split& sp, long long* R_far) {
  BinState bsa, bsb;
  int rc = bin_pass(f, sp.RA, Emission{0, sp.Pn, false, sp.near_meta}, f.im.ranges, &bsa);
  if (rc) return rc;
  rc = blend_forward<1>(f, bsa.point_list);
  if (rc) return rc;
  uint32_t unfinished = 0, rb = 0;
  DGS_CUDA_OK(cudaMemcpyAsync(&unfinished, &f.gs.totals->unfinished, sizeof(uint32_t), cudaMemcpyDeviceToHost, f.st));
  DGS_CUDA_OK(cudaStreamSynchronize(f.st));
  if (unfinished == 0) return DGS_OK;
  {
    ProfScope ps(f.st, PROF_RASTER_SCAN);
    count_open_kernel<<<f.pgrid(), 256, 0, f.st>>>(f.pb, f.gs, f.im.tile_open, sp.Pn);
    DGS_LAUNCH_OK(f.st, f.debug);
    size_t scan_bytes = f.gs.scan_bytes;
    DGS_CUDA_OK(cub::DeviceScan::InclusiveSum(f.gs.scan_temp, scan_bytes, f.gs.open_counts, f.gs.open_offsets, (int)f.N,
                                              f.st));
    DGS_CUDA_OK(cudaMemcpyAsync(&rb, f.gs.open_offsets + f.N - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, f.st));
    DGS_CUDA_OK(cudaStreamSynchronize(f.st));
  }
  rc = bin_pass(f, rb, Emission{sp.Pn, f.pb.P, true, nullptr}, f.im.ranges_b, &bsb);
  if (rc) return rc;
  *R_far = rb;
  return blend_forward<2>(f, bsb.point_list);
}

// projection -> small-scene binning, or depth ranking and scan -> split decision -> bin pass(es) + blend
static int run_forward(Problem pb, const CameraInput& cam, const Allocators& al, float* out_color, int* radii,
                       long long* R_out, long long chunk_R[2], cudaStream_t st, int debug, MseFwd mse = MseFwd(),
                       AuxFwd aux = AuxFwd(), uint8_t* frames = nullptr) {
  Forward f;
  f.pb = pb; f.al = al; f.out_color = out_color; f.mse = mse; f.aux = aux; f.frames = frames; f.st = st; f.debug = debug;
  f.N = (size_t)pb.NV * pb.P;
  f.ntiles = (size_t)pb.NV * pb.tiles;
  DGS_REQUIRE(f.N < (size_t)INT32_MAX, "n_views * P = %zu does not fit the 32-bit scan", f.N);
  size_t gbytes = 0, ibytes = 0;
  GeomState::carve(nullptr, pb.NV, pb.P, &gbytes);
  ImgState::carve(nullptr, pb.NV, pb.W, pb.H, &ibytes);
  void* gbuf = al.geom(gbytes, al.geom_user);
  void* ibuf = al.img(ibytes, al.img_user);
  if (!gbuf || !ibuf) { set_error("arena allocator returned NULL"); return DGS_ERR_ALLOC; }
  f.gs = GeomState::carve(gbuf, pb.NV, pb.P, nullptr);
  f.im = ImgState::carve(ibuf, pb.NV, pb.W, pb.H, nullptr);

  int rc = project(f, cam, radii);
  if (rc) return rc;
  chunk_R[1] = 0;
  if (f.N <= (size_t)SMALL_MAX_N && f.ntiles <= (size_t)SMALL_MAX_TILES) {
    bool done = false;
    rc = bin_small(f, R_out, &done);
    if (rc || done) {
      chunk_R[0] = *R_out;
      return rc;
    }
  }
  rc = rank_and_scan(f);
  if (rc) return rc;
  Split sp;
  rc = plan_split(f, &sp);
  if (rc) return rc;
  *R_out = sp.R;
  chunk_R[0] = sp.RA;
  if (sp.Pn > 0) return bin_two_phase(f, sp, &chunk_R[1]);
  BinState bs;
  rc = bin_pass(f, sp.R, Emission{0, pb.P, false, nullptr}, f.im.ranges, &bs);
  if (rc) return rc;
  return blend_forward<0>(f, bs.point_list);
}

static Problem make_problem(int NV, int V, int P, int D, int M, int W, int H, int raw, float mod) {
  Problem pb;
  memset(&pb, 0, sizeof(pb));
  pb.NV = NV; pb.V = V; pb.P = P; pb.D = D; pb.M = M; pb.W = W; pb.H = H;
  pb.gx = ceil_div(W, TILE); pb.gy = ceil_div(H, TILE); pb.tiles = pb.gx * pb.gy;
  pb.raw = raw; pb.mod = mod; pb.near_log2 = 0;
  return pb;
}

}  // namespace dgs

using namespace dgs;

// =============================================================================================
// C ABI
// =============================================================================================
extern "C" {

size_t dgs_raster_geom_bytes(int n_views, int P) {
  size_t b = 0;
  GeomState::carve(nullptr, n_views, P, &b);
  return b;
}
size_t dgs_raster_binning_bytes(long long R) {
  size_t b = 0;
  BinState::carve(nullptr, R, &b);
  return b;
}
size_t dgs_raster_image_bytes(int n_views, int W, int H) {
  size_t b = 0;
  ImgState::carve(nullptr, n_views, W, H, &b);
  return b;
}

static int check_single_args(const dgs_raster_args* a) {
  DGS_REQUIRE(a != nullptr, "args is NULL");
  DGS_REQUIRE(a->P >= 0 && a->W > 0 && a->H > 0, "bad sizes P=%d W=%d H=%d", a->P, a->W, a->H);
  DGS_REQUIRE(a->D >= 0 && a->D <= 3, "SH degree %d not in 0..3", a->D);
  DGS_REQUIRE((a->shs != nullptr) != (a->colors_precomp != nullptr),
              "Please provide exactly one of either SHs or precomputed colors!");
  DGS_REQUIRE(((a->scales != nullptr && a->rotations != nullptr) != (a->cov3D_precomp != nullptr)) &&
                  ((a->scales != nullptr) == (a->rotations != nullptr)),
              "Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!");
  DGS_REQUIRE(a->shs == nullptr || a->M >= (a->D + 1) * (a->D + 1), "M=%d too small for SH degree %d", a->M, a->D);
  return DGS_OK;
}

static Problem single_problem(const dgs_raster_args* a, float bg[3]) {
  Problem pb = make_problem(1, 1, a->P, a->D, a->M, a->W, a->H, 0, a->scale_modifier);
  pb.means = a->means3D; pb.shs = a->shs; pb.colors_pre = a->colors_precomp; pb.opac = a->opacities;
  pb.scales = a->scales; pb.rots = a->rotations; pb.cov_pre = a->cov3D_precomp;
  pb.bg[0] = bg[0]; pb.bg[1] = bg[1]; pb.bg[2] = bg[2];
  return pb;
}

int dgs_raster_forward(const dgs_raster_args* a, dgs_alloc_fn geom_alloc, void* geom_user, dgs_alloc_fn bin_alloc,
                       void* bin_user, dgs_alloc_fn img_alloc, void* img_user, float* out_color, int* radii,
                       int* num_rendered, void* stream) {
  int rc = check_single_args(a);
  if (rc) return rc;
  DGS_REQUIRE(geom_alloc && bin_alloc && img_alloc && out_color && num_rendered, "NULL output/allocator");
  cudaStream_t st = (cudaStream_t)stream;
  *num_rendered = 0;
  if (a->P == 0) return DGS_OK;  // legal: the caller's zero-filled outputs stand (rasterize_points.cu:81)
  float bg[3];
  DGS_CUDA_OK(cudaMemcpyAsync(bg, a->background, sizeof(bg), cudaMemcpyDeviceToHost, st));
  DGS_CUDA_OK(cudaStreamSynchronize(st));
  Problem pb = single_problem(a, bg);
  long long R = 0, chunk_R[2] = {0, 0};
  CameraInput cam;
  cam.view = a->viewmatrix; cam.proj = a->projmatrix; cam.campos = a->campos;
  cam.tanx = a->tan_fovx; cam.tany = a->tan_fovy;
  const Allocators al = {geom_alloc, geom_user, bin_alloc, bin_user, img_alloc, img_user};
  rc = run_forward(pb, cam, al, out_color, radii, &R, chunk_R, st, a->debug);
  *num_rendered = (int)R;
  return rc;
}

int dgs_raster_backward(const dgs_raster_args* a, int R, const int* radii, const void* geom_buffer,
                        const void* binning_buffer, const void* image_buffer, const float* dL_dpix,
                        float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                        float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot,
                        void* stream) {
  int rc = check_single_args(a);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (a->P == 0) return DGS_OK;
  DGS_REQUIRE(geom_buffer && binning_buffer && image_buffer && dL_dpix, "NULL state buffer");
  DGS_REQUIRE(dL_dmean2D && dL_dconic && dL_dopacity && dL_dcolor && dL_dmean3D, "NULL gradient buffer");
  float bg[3];
  DGS_CUDA_OK(cudaMemcpyAsync(bg, a->background, sizeof(bg), cudaMemcpyDeviceToHost, st));
  DGS_CUDA_OK(cudaStreamSynchronize(st));
  Problem pb = single_problem(a, bg);
  GeomState gs = GeomState::carve(const_cast<void*>(geom_buffer), 1, a->P, nullptr);
  ImgState im = ImgState::carve(const_cast<void*>(image_buffer), 1, a->W, a->H, nullptr);
  BinState bs = BinState::carve(const_cast<void*>(binning_buffer), R, nullptr);
  if (R > 0) {
    blend_backward_kernel<false><<<pb.tiles, TILE_PIX, 0, st>>>(pb, gs, im, bs.point_list, nullptr, dL_dpix, MseBwd(),
                                                                 dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolor, AuxBwd());
    DGS_LAUNCH_OK(st, a->debug);
  }
  GeomGradOut out;
  out.dmeans = dL_dmean3D; out.dcov3d = dL_dcov3D; out.dsh = dL_dsh; out.dscale = dL_dscale; out.drot = dL_drot;
  out.dopac_raw = nullptr;
  geometry_backward_kernel<false><<<dim3(ceil_div(a->P, 256), 1), 256, 0, st>>>(pb, gs, radii, dL_dmean2D, dL_dconic,
                                                                                 dL_dopacity, dL_dcolor, out, nullptr);
  DGS_LAUNCH_OK(st, a->debug);
  return DGS_OK;
}

int dgs_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                     uint8_t* present, void* stream) {
  (void)projmatrix;
  DGS_REQUIRE(P >= 0, "bad P");
  if (P == 0) return DGS_OK;
  DGS_REQUIRE(means3D && viewmatrix && present, "NULL pointer");
  mark_visible_kernel<<<ceil_div(P, 256), 256, 0, (cudaStream_t)stream>>>(P, means3D, viewmatrix, present);
  DGS_LAUNCH_OK((cudaStream_t)stream, 0);
  return DGS_OK;
}

static int check_batch_args(const dgs_render_batch_args* a) {
  DGS_REQUIRE(a != nullptr, "args is NULL");
  DGS_REQUIRE(a->B > 0 && a->V > 0 && a->P > 0 && a->W > 0 && a->H > 0, "bad sizes");
  DGS_REQUIRE(a->D >= 0 && a->D <= 3 && a->M >= (a->D + 1) * (a->D + 1), "bad SH degree/M");
  DGS_REQUIRE(a->xyz && a->features && a->scaling && a->rotation && a->opacity && a->c2w && a->fxfycxcy, "NULL input");
  return DGS_OK;
}

static Problem batch_problem(const dgs_render_batch_args* a) {
  Problem pb = make_problem(a->B * a->V, a->V, a->P, a->D, a->M, a->W, a->H, 1, a->scale_modifier);
  pb.means = a->xyz; pb.shs = a->features; pb.opac = a->opacity; pb.scales = a->scaling; pb.rots = a->rotation;
  pb.bg[0] = a->bg[0]; pb.bg[1] = a->bg[1]; pb.bg[2] = a->bg[2];
  pb.near_log2 = a->near_log2;  // > 0 fixed fraction 1/2^k, 0 single pass, < 0 adaptive (1/8 or 1/16)
  return pb;
}

int dgs_render_batch_forward(const dgs_render_batch_args* a, dgs_alloc_fn geom_alloc, void* geom_user,
                             dgs_alloc_fn bin_alloc, void* bin_user, dgs_alloc_fn img_alloc, void* img_user,
                             float* out_images, long long* num_rendered, long long* chunk_instances,
                             const dgs_render_mse* mse, const dgs_render_aux* aux, void* stream) {
  int rc = check_batch_args(a);
  if (rc) return rc;
  DGS_REQUIRE(geom_alloc && bin_alloc && img_alloc && out_images && num_rendered && chunk_instances,
              "NULL output/allocator");
  MseFwd mf;
  if (mse) {
    DGS_REQUIRE(mse->target && mse->loss_sum && (mse->target_channels == 3 || mse->target_channels == 4),
                "mse: target / loss_sum NULL or target_channels not 3|4");
    mf.target = mse->target; mf.tc = mse->target_channels; mf.loss = mse->loss_sum;
  }
  AuxFwd af;
  if (aux) {
    DGS_REQUIRE(aux->depth && aux->alpha, "aux: depth / alpha output NULL");
    af.depth = aux->depth; af.alpha = aux->alpha;
  }
  Problem pb = batch_problem(a);
  CameraInput cam;
  cam.c2w = a->c2w; cam.fxfycxcy = a->fxfycxcy;
  const Allocators al = {geom_alloc, geom_user, bin_alloc, bin_user, img_alloc, img_user};
  return run_forward(pb, cam, al, out_images, nullptr, num_rendered, chunk_instances, (cudaStream_t)stream, a->debug,
                     mf, af);
}

int dgs_render_frames(const dgs_render_batch_args* a, dgs_alloc_fn geom_alloc, void* geom_user, dgs_alloc_fn bin_alloc,
                      void* bin_user, dgs_alloc_fn img_alloc, void* img_user, uint8_t* frames, long long* num_rendered,
                      void* stream) {
  DGS_REQUIRE(a != nullptr, "args is NULL");
  // P == 0 is legal: the caller's zero-filled frames stand, the reference's image of an empty model
  // (rasterize_points.cu:68,81)
  if (a->P == 0) {
    DGS_REQUIRE(a->B > 0 && a->V > 0 && a->W > 0 && a->H > 0, "bad sizes");
    DGS_REQUIRE(frames && num_rendered, "NULL output");
    *num_rendered = 0;
    return DGS_OK;
  }
  int rc = check_batch_args(a);
  if (rc) return rc;
  DGS_REQUIRE(geom_alloc && bin_alloc && img_alloc && frames && num_rendered, "NULL output/allocator");
  Problem pb = batch_problem(a);
  CameraInput cam;
  cam.c2w = a->c2w; cam.fxfycxcy = a->fxfycxcy;
  const Allocators al = {geom_alloc, geom_user, bin_alloc, bin_user, img_alloc, img_user};
  long long chunk_R[2] = {0, 0};
  return run_forward(pb, cam, al, nullptr, nullptr, num_rendered, chunk_R, (cudaStream_t)stream, a->debug, MseFwd(),
                     AuxFwd(), frames);
}

int dgs_render_batch_backward(const dgs_render_batch_args* a, long long R, const long long* chunk_instances,
                              const void* geom_buffer, const void* binning_buffer, const void* binning_buffer_b,
                              const void* image_buffer, const float* dL_dimages, const dgs_render_mse* mse,
                              const dgs_render_aux* aux, float* d_xyz, float* d_features, float* d_scaling,
                              float* d_rotation, float* d_opacity, dgs_alloc_fn scratch_alloc, void* scratch_user,
                              void* stream) {
  int rc = check_batch_args(a);
  if (rc) return rc;
  const bool has_aux = aux && (aux->dL_ddepth || aux->dL_dalpha);  // no aux gradient: the plain kernels
  DGS_REQUIRE(geom_buffer && binning_buffer && image_buffer && (dL_dimages || mse || has_aux) && scratch_alloc &&
                  chunk_instances,
              "NULL state buffer");
  MseBwd mb;
  if (mse) {
    DGS_REQUIRE(mse->target && mse->coef && mse->images && (mse->target_channels == 3 || mse->target_channels == 4),
                "mse: target / coef / images NULL or target_channels not 3|4");
    mb.target = mse->target; mb.tc = mse->target_channels; mb.images = mse->images; mb.coef = mse->coef;
  }
  DGS_REQUIRE(chunk_instances[1] == 0 || binning_buffer_b, "phase-B binning buffer missing");
  DGS_REQUIRE(d_xyz && d_features && d_scaling && d_rotation && d_opacity, "NULL gradient buffer");
  cudaStream_t st = (cudaStream_t)stream;
  Problem pb = batch_problem(a);
  GeomState gs = GeomState::carve(const_cast<void*>(geom_buffer), pb.NV, pb.P, nullptr);
  ImgState im = ImgState::carve(const_cast<void*>(image_buffer), pb.NV, pb.W, pb.H, nullptr);
  BinState bs = BinState::carve(const_cast<void*>(binning_buffer), chunk_instances[0], nullptr);
  const uint32_t* list_b = nullptr;
  if (chunk_instances[1] > 0)
    list_b = BinState::carve(const_cast<void*>(binning_buffer_b), chunk_instances[1], nullptr).point_list;
  // per-(view, Gaussian) screen-space gradient records: mean2D[3] conic[4] opacity[1] colour[3], and with aux gradients z[1]
  const size_t N = (size_t)pb.NV * pb.P;
  Carver c(nullptr);
  c.take<float>(N * 3); c.take<float>(N * 4); c.take<float>(N); c.take<float>(N * 3);
  if (has_aux) c.take<float>(N);
  const size_t sbytes = c.bytes();
  void* sbuf = scratch_alloc(sbytes, scratch_user);
  if (!sbuf) { set_error("scratch allocator returned NULL"); return DGS_ERR_ALLOC; }
  Carver cc(sbuf);
  float* dmean2D = cc.take<float>(N * 3);
  float* dconic = cc.take<float>(N * 4);
  float* dopac = cc.take<float>(N);
  float* dcolor = cc.take<float>(N * 3);
  AuxBwd ab;
  if (has_aux) {
    ab.ddepth = aux->dL_ddepth; ab.dalpha = aux->dL_dalpha;
    ab.dz = cc.take<float>(N);
  }
  DGS_CUDA_OK(cudaMemsetAsync(sbuf, 0, sbytes, st));
  if (R > 0) {
    ProfScope ps(st, PROF_RASTER_BLEND_BWD);
    const unsigned grid = (unsigned)((size_t)pb.NV * pb.tiles);
    if (has_aux)
      blend_backward_kernel<true><<<grid, TILE_PIX, 0, st>>>(pb, gs, im, bs.point_list, list_b, dL_dimages, mb, dmean2D,
                                                             dconic, dopac, dcolor, ab);
    else
      blend_backward_kernel<false><<<grid, TILE_PIX, 0, st>>>(pb, gs, im, bs.point_list, list_b, dL_dimages, mb, dmean2D,
                                                              dconic, dopac, dcolor, ab);
    DGS_LAUNCH_OK(st, a->debug);
  }
  GeomGradOut out;
  out.dmeans = d_xyz; out.dcov3d = nullptr; out.dsh = d_features; out.dscale = d_scaling; out.drot = d_rotation;
  out.dopac_raw = d_opacity;
  {
    ProfScope ps(st, PROF_RASTER_GEOM_BWD);
    const dim3 grid(ceil_div(a->P, 256), a->B);
    if (has_aux)
      geometry_backward_kernel<true><<<grid, 256, 0, st>>>(pb, gs, nullptr, dmean2D, dconic, dopac, dcolor, out, ab.dz);
    else
      geometry_backward_kernel<false><<<grid, 256, 0, st>>>(pb, gs, nullptr, dmean2D, dconic, dopac, dcolor, out, nullptr);
    DGS_LAUNCH_OK(st, a->debug);
  }
  return DGS_OK;
}

int dgs_raster_export_state(int n_views, int P, int W, int H, long long R, const void* geom_buffer,
                            const void* binning_buffer, const void* image_buffer, float* xy, float* depth,
                            float* conic_opacity, float* rgb, uint32_t* tiles_touched, uint32_t* point_list,
                            uint32_t* ranges, float* final_T, uint32_t* n_contrib, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  DGS_REQUIRE(geom_buffer && image_buffer, "NULL state buffer");
  GeomState gs = GeomState::carve(const_cast<void*>(geom_buffer), n_views, P, nullptr);
  ImgState im = ImgState::carve(const_cast<void*>(image_buffer), n_views, W, H, nullptr);
  const size_t N = (size_t)n_views * P;
  if (N) {
    export_geom_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(N, gs, xy, depth, conic_opacity, rgb, tiles_touched);
    DGS_LAUNCH_OK(st, 0);
  }
  const size_t npix = (size_t)n_views * W * H, ntiles = (size_t)n_views * ceil_div(W, TILE) * ceil_div(H, TILE);
  if (point_list && R > 0) {
    DGS_REQUIRE(binning_buffer, "NULL binning buffer");
    BinState bs = BinState::carve(const_cast<void*>(binning_buffer), R, nullptr);
    DGS_CUDA_OK(cudaMemcpyAsync(point_list, bs.point_list, R * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
  }
  if (ranges) DGS_CUDA_OK(cudaMemcpyAsync(ranges, im.ranges, ntiles * sizeof(uint2), cudaMemcpyDeviceToDevice, st));
  if (final_T) DGS_CUDA_OK(cudaMemcpyAsync(final_T, im.final_T, npix * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (n_contrib) DGS_CUDA_OK(cudaMemcpyAsync(n_contrib, im.n_contrib, npix * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
  return DGS_OK;
}

}  // extern "C"
