// poisson.cu -- surface reconstruction from oriented points: the reference's poisson_mesh_reconstruction
// (utils/mesh_utils.py:5-41: Open3D's statistical outlier removal, normal estimation, screened Poisson at depth 9 and
// the 10 % density trim), as one exact contract that oracle/poisson.py restates serially.  Compiled with -fmad=false.
//
// points fp32 [P, 3] (finite), normals NULL or fp32 [P, 3]; k = nb_neighbors in [1, 32], P >= k.
//   1. Outliers (Open3D's RemoveStatisticalOutliers as recalled; Open3D was not available to check it against):
//      a_i = the fp64 mean, in neighbour order, of the square roots of point i's k nearest squared distances (dgs_knn,
//      itself included).  The mean m and the sample standard deviation s of the a_i > 0 are fp64 sums of per-CTA
//      partials in a fixed order; point i is an inlier iff 0 < a_i < m + std_ratio s (s = 0 when fewer than two a_i
//      are > 0).  The N inliers keep their input order.
//   2. Normals: given, each inlier's normal over its length (fp64, rounded to fp32); a zero or non-finite normal
//      anywhere in the input is an error.  Otherwise the eigenvector of the smallest eigenvalue of the fp64 covariance
//      (1 / n sum (q - mean)(q - mean)^T) of the inlier's k nearest inliers (dgs_knn over the inliers; fewer when
//      N < k), by cyclic Jacobi, oriented so that n . (p - c) >= 0 for the inliers' fp64 centroid c.  Open3D leaves
//      the sign arbitrary, which gives Poisson no inside; orienting away from the centroid is this pass's departure,
//      right for star-shaped objects.
//   3. Grid: the inliers' bounding cube (its largest extent, about the box centre) scaled by `scale` (>= 1, so every
//      point lies inside); R = 2^depth + 1 nodes per axis, h = side / (R - 1).  Everything below is in grid units
//      g = (p - origin) / h (fp64).  A point's cell is floor(g) clamped to [0, R - 2]; its eight trilinear weights
//      w_ij (fp64 products, rounded to fp32) are stored once.
//   4. Splat, in gather form: the inliers sorted by cell (radix sort, so the input order within a cell); every node
//      sums over its eight cells' ranges in sorted order D_j = sum_i w_ij and V_j = (R^2 / N) sum_i w_ij n_i (fp32).
//   5. System: (L + point_weight (R^2 / N) B^T B) chi = -div V on the interior nodes, chi = 0 on the outer layer.  L is
//      the 7-point negative Laplacian, div V the central difference, B trilinear interpolation at the inliers;
//      B^T B is applied as interpolation at the points, then a gather over the same ranges (no scatter).
//   6. Solver: conjugate gradients (fp32 vectors) preconditioned by one V-cycle of geometric multigrid on L: levels
//      of 2^l + 1 nodes down to 5^3, red-black Gauss-Seidel with 2 pre-sweeps (red, black) and 2 post-sweeps (black,
//      red), full-weighting restriction, trilinear prolongation, and 4 symmetric sweep pairs on 5^3; the cycle is a
//      symmetric operator.  Dot products are fp64 per-CTA partials over a fixed grid, summed by one fixed-order
//      finalize; the one read-back per iteration is ||r||^2.  It stops when ||r|| / ||b|| <= tol or after max_iters.
//   7. Surface: iso = the fp64 mean of chi interpolated at the inliers.  chi is about -1 inside and 0 outside (for
//      outward normals), so dgs_marching_cubes runs on -chi at -iso and its faces come out oriented outwards.
//      Vertices map back by origin + h v (fp64, rounded to fp32).
//   8. Trim (density_quantile > 0): each vertex's density is D interpolated at it (fp32); the threshold is
//      numpy.quantile(densities, density_quantile) ('linear', in fp32) over the cub-sorted densities; vertices with a
//      smaller density go, with every face that touches one; the other vertices keep their order (unreferenced ones
//      stay: Open3D's remove_vertices_by_mask) and the faces are renumbered.
// No floating-point atomics: the result is the same bits on every run.
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "dgs_internal.h"
#include "sorted_ranges.cuh"

namespace dgs {
namespace {

constexpr int T = 256;
constexpr int kParts = 1024;  // CTAs of every reduction: a fixed grid, so a fixed summation order
constexpr unsigned kFull = 0xffffffffu;

__host__ __device__ __forceinline__ unsigned fkey(float x) {
  unsigned u;
  memcpy(&u, &x, sizeof(u));
  return (u & 0x80000000u) ? ~u : u | 0x80000000u;
}
__host__ __device__ __forceinline__ float fval(unsigned k) {
  const unsigned u = (k & 0x80000000u) ? k & 0x7fffffffu : ~k;
  float x;
  memcpy(&x, &u, sizeof(x));
  return x;
}

// Device scalars of the solver and the reductions.
struct Scal {
  double sum[4];  // finalized sums
  double rz, alpha, beta;
  unsigned box[6];
  int bad;
};

// ------------------------------------------------------------------------------------------------------ reductions
// part[blockIdx.x * W + w] = this CTA's sum of f(i, w) for w < W over a grid-stride loop; f returns W values.
template <int W, class F>
__device__ __forceinline__ void block_partials(long long n, F f, double* __restrict__ part) {
  typedef cub::BlockReduce<double, T> BR;
  __shared__ typename BR::TempStorage tmp;
  double acc[W];
  for (int w = 0; w < W; w++) acc[w] = 0.0;
  for (long long i = (long long)blockIdx.x * T + threadIdx.x; i < n; i += (long long)gridDim.x * T) f(i, acc);
  for (int w = 0; w < W; w++) {
    const double s = BR(tmp).Sum(acc[w]);
    if (threadIdx.x == 0) part[blockIdx.x * W + w] = s;
    __syncthreads();
  }
}

// s->sum[w] = the sum of the kParts partials of value w, in a fixed order; op then updates the solver scalars:
// 1: alpha = rz / sum[0];  2: beta = sum[0] / rz, rz = sum[0];  3: rz = sum[0]
__global__ void __launch_bounds__(1024) finalize_kernel(const double* __restrict__ part, int W, int op,
                                                        Scal* __restrict__ s) {
  typedef cub::BlockReduce<double, 1024> BR;
  __shared__ typename BR::TempStorage tmp;
  for (int w = 0; w < W; w++) {
    const double v = BR(tmp).Sum(part[threadIdx.x * W + w]);
    if (threadIdx.x == 0) s->sum[w] = v;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    if (op == 1) s->alpha = s->rz / s->sum[0];
    if (op == 2) { s->beta = s->sum[0] / s->rz; s->rz = s->sum[0]; }
    if (op == 3) s->rz = s->sum[0];
  }
}

template <int W, class F>
__global__ void __launch_bounds__(T) partials_kernel(long long n, F f, double* __restrict__ part) {
  block_partials<W>(n, f, part);
}

// ------------------------------------------------------------------------------------------- outliers and normals
__global__ void mean_dist_kernel(int P, int k, const float* __restrict__ d2, double* __restrict__ a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  double s = 0.0;
  for (int j = 0; j < k; j++) s += sqrt((double)d2[(size_t)i * k + j]);
  a[i] = s / k;
}

__global__ void inlier_kernel(int P, const double* __restrict__ a, double thr, uint8_t* __restrict__ mask) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P) mask[i] = a[i] > 0.0 && a[i] < thr;
}

__global__ void normal_check_kernel(int P, const float* __restrict__ n, Scal* __restrict__ s) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool bad = false;
  if (i < P) {
    const double x = n[3 * i], y = n[3 * i + 1], z = n[3 * i + 2];
    const double l2 = (x * x + y * y) + z * z;
    bad = !(l2 > 0.0) || !isfinite(l2);
  }
  const unsigned c = __popc(__ballot_sync(kFull, bad));
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s->bad, (int)c);
}

__global__ void normalize_kernel(int N, float3* __restrict__ n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const double x = n[i].x, y = n[i].y, z = n[i].z;
  const double l = sqrt((x * x + y * y) + z * z);
  n[i] = make_float3((float)(x / l), (float)(y / l), (float)(z / l));
}

// Eigenvector of the smallest eigenvalue of the symmetric 3 x 3 matrix a (cyclic Jacobi, destroys a).
__device__ void smallest_eigvec(double a[3][3], double out[3]) {
  double v[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  for (int sweep = 0; sweep < 32; sweep++) {
    const double off = fabs(a[0][1]) + fabs(a[0][2]) + fabs(a[1][2]);
    const double diag = fabs(a[0][0]) + fabs(a[1][1]) + fabs(a[2][2]);
    if (off == 0.0 || off <= 1e-300 || off < 1e-17 * diag) break;
    for (int p = 0; p < 2; p++)
      for (int q = p + 1; q < 3; q++) {
        if (a[p][q] == 0.0) continue;
        const double theta = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int r = 0; r < 3; r++) {  // a = J^T a J
          const double arp = a[r][p], arq = a[r][q];
          a[r][p] = c * arp - s * arq;
          a[r][q] = s * arp + c * arq;
        }
        for (int r = 0; r < 3; r++) {
          const double apr = a[p][r], aqr = a[q][r];
          a[p][r] = c * apr - s * aqr;
          a[q][r] = s * apr + c * aqr;
        }
        for (int r = 0; r < 3; r++) {
          const double vrp = v[r][p], vrq = v[r][q];
          v[r][p] = c * vrp - s * vrq;
          v[r][q] = s * vrp + c * vrq;
        }
      }
  }
  int m = 0;
  if (a[1][1] < a[m][m]) m = 1;
  if (a[2][2] < a[m][m]) m = 2;
  for (int r = 0; r < 3; r++) out[r] = v[r][m];
}

__global__ void pca_kernel(int N, int k, const float3* __restrict__ pts, const int* __restrict__ idx,
                           const Scal* __restrict__ s, float3* __restrict__ nrm) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  double m[3] = {0, 0, 0};
  int cnt = 0;
  for (int j = 0; j < k; j++) {
    const int q = idx[(size_t)i * k + j];
    if (q < 0) continue;
    m[0] += pts[q].x; m[1] += pts[q].y; m[2] += pts[q].z;
    cnt++;
  }
  for (int r = 0; r < 3; r++) m[r] /= cnt;
  double a[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  for (int j = 0; j < k; j++) {
    const int q = idx[(size_t)i * k + j];
    if (q < 0) continue;
    const double d[3] = {pts[q].x - m[0], pts[q].y - m[1], pts[q].z - m[2]};
    for (int r = 0; r < 3; r++)
      for (int c = r; c < 3; c++) a[r][c] += d[r] * d[c];
  }
  for (int r = 0; r < 3; r++)
    for (int c = r; c < 3; c++) { a[r][c] /= cnt; a[c][r] = a[r][c]; }
  double n[3];
  smallest_eigvec(a, n);
  const double c[3] = {s->sum[0] / N, s->sum[1] / N, s->sum[2] / N};
  const double o = (n[0] * (pts[i].x - c[0]) + n[1] * (pts[i].y - c[1])) + n[2] * (pts[i].z - c[2]);
  const double sg = o < 0.0 ? -1.0 : 1.0;
  const double l = sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]);
  nrm[i] = make_float3((float)(sg * n[0] / l), (float)(sg * n[1] / l), (float)(sg * n[2] / l));
}

__global__ void box_kernel(int N, const float3* __restrict__ p, Scal* __restrict__ s) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned lo[3] = {kFull, kFull, kFull}, hi[3] = {0u, 0u, 0u};
  if (i < N) {
    lo[0] = hi[0] = fkey(p[i].x);
    lo[1] = hi[1] = fkey(p[i].y);
    lo[2] = hi[2] = fkey(p[i].z);
  }
  for (int k = 0; k < 3; k++) {
    lo[k] = __reduce_min_sync(kFull, lo[k]);
    hi[k] = __reduce_max_sync(kFull, hi[k]);
  }
  if ((threadIdx.x & 31) == 0)
    for (int k = 0; k < 3; k++) {
      atomicMin(&s->box[k], lo[k]);
      atomicMax(&s->box[3 + k], hi[k]);
    }
}

// ------------------------------------------------------------------------------------------------------------ grid
struct PGrid {
  double origin[3], h;
  int R;  // nodes per axis; R - 1 cells
};

__global__ void cell_kernel(int N, const float3* __restrict__ p, PGrid g, uint32_t* __restrict__ keys,
                            uint32_t* __restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int C = g.R - 1;
  const double q[3] = {((double)p[i].x - g.origin[0]) / g.h, ((double)p[i].y - g.origin[1]) / g.h,
                       ((double)p[i].z - g.origin[2]) / g.h};
  int c[3];
  for (int k = 0; k < 3; k++) c[k] = (int)fmin(fmax(floor(q[k]), 0.0), (double)(C - 1));
  keys[i] = ((uint32_t)c[0] * C + c[1]) * C + c[2];
  vals[i] = i;
}

// Sorted point s: its normal and its eight weights, corner c = 4 dx + 2 dy + dz of its cell.
__global__ void weights_kernel(int N, const float3* __restrict__ p, const float3* __restrict__ n, PGrid g,
                               const uint32_t* __restrict__ keys, const uint32_t* __restrict__ vals,
                               float3* __restrict__ sn, float* __restrict__ w) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= N) return;
  const int i = (int)vals[s];
  const int C = g.R - 1;
  const uint32_t key = keys[s];
  const int c[3] = {(int)(key / ((uint32_t)C * C)), (int)((key / C) % C), (int)(key % C)};
  const double q[3] = {((double)p[i].x - g.origin[0]) / g.h, ((double)p[i].y - g.origin[1]) / g.h,
                       ((double)p[i].z - g.origin[2]) / g.h};
  double f[3];
  for (int k = 0; k < 3; k++) f[k] = q[k] - c[k];
  for (int cc = 0; cc < 8; cc++) {
    const double wx = (cc & 4) ? f[0] : 1.0 - f[0], wy = (cc & 2) ? f[1] : 1.0 - f[1], wz = (cc & 1) ? f[2] : 1.0 - f[2];
    w[8 * (size_t)s + cc] = (float)((wx * wy) * wz);
  }
  sn[s] = n[i];
}

__device__ __forceinline__ void node_xyz(long long j, int R, int& x, int& y, int& z) {
  x = (int)(j / ((long long)R * R));
  y = (int)((j / R) % R);
  z = (int)(j % R);
}
__device__ __forceinline__ bool interior(int x, int y, int z, int R) {
  return x > 0 && y > 0 && z > 0 && x < R - 1 && y < R - 1 && z < R - 1;
}

// Visits the points of node (x, y, z)'s eight cells in a fixed order: f(sorted point, corner of the node in its cell).
template <class F>
__device__ __forceinline__ void for_node_points(int x, int y, int z, int R, const uint2* __restrict__ ranges, F f) {
  const int C = R - 1;
  for (int c = 0; c < 8; c++) {
    const int cx = x - ((c >> 2) & 1), cy = y - ((c >> 1) & 1), cz = z - (c & 1);
    if (cx < 0 || cy < 0 || cz < 0 || cx >= C || cy >= C || cz >= C) continue;
    const uint2 rg = ranges[((size_t)cx * C + cy) * C + cz];
    for (uint32_t s = rg.x; s < rg.y; s++) f(s, c);
  }
}

__global__ void splat_kernel(int R, const uint2* __restrict__ ranges, const float* __restrict__ w,
                             const float3* __restrict__ sn, float vscale, float* __restrict__ D, float* __restrict__ Vx,
                             float* __restrict__ Vy, float* __restrict__ Vz) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= (long long)R * R * R) return;
  int x, y, z;
  node_xyz(j, R, x, y, z);
  float d = 0.f, vx = 0.f, vy = 0.f, vz = 0.f;
  for_node_points(x, y, z, R, ranges, [&](uint32_t s, int c) {
    const float ws = w[8 * (size_t)s + c];
    const float3 n = sn[s];
    d += ws;
    vx += ws * n.x;
    vy += ws * n.y;
    vz += ws * n.z;
  });
  D[j] = d;
  Vx[j] = vscale * vx;
  Vy[j] = vscale * vy;
  Vz[j] = vscale * vz;
}

// b = -div V (central differences) on the interior, 0 on the outer layer
__global__ void rhs_kernel(int R, const float* __restrict__ Vx, const float* __restrict__ Vy,
                           const float* __restrict__ Vz, float* __restrict__ b) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= (long long)R * R * R) return;
  int x, y, z;
  node_xyz(j, R, x, y, z);
  if (!interior(x, y, z, R)) { b[j] = 0.f; return; }
  const long long sx = (long long)R * R, sy = R;
  const float div = ((0.5f * (Vx[j + sx] - Vx[j - sx]) + 0.5f * (Vy[j + sy] - Vy[j - sy])) + 0.5f * (Vz[j + 1] - Vz[j - 1]));
  b[j] = -div;
}

// u[s] = (B chi)[s]: the sorted point's trilinear interpolation of the field
__global__ void interp_kernel(int N, int R, const uint32_t* __restrict__ keys, const float* __restrict__ w,
                              const float* __restrict__ f, float* __restrict__ u) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= N) return;
  const int C = R - 1;
  const uint32_t key = keys[s];
  const int cx = (int)(key / ((uint32_t)C * C)), cy = (int)((key / C) % C), cz = (int)(key % C);
  float acc = 0.f;
  for (int c = 0; c < 8; c++)
    acc += w[8 * (size_t)s + c] * f[((size_t)(cx + ((c >> 2) & 1)) * R + cy + ((c >> 1) & 1)) * R + cz + (c & 1)];
  u[s] = acc;
}

__device__ __forceinline__ float lap(const float* __restrict__ p, long long j, int R) {
  const long long sx = (long long)R * R, sy = R;
  return 6.f * p[j] - (((p[j - sx] + p[j + sx]) + (p[j - sy] + p[j + sy])) + (p[j - 1] + p[j + 1]));
}

// Ap = L p + sw B^T u on the interior (0 on the outer layer), with the partials of p . Ap
struct ApplyOp {
  int R;
  float sw;
  const float* p;
  const float* u;
  const float* w;
  const uint2* ranges;
  float* Ap;
  __device__ void operator()(long long j, double* acc) const {
    int x, y, z;
    node_xyz(j, R, x, y, z);
    float v = 0.f;
    if (interior(x, y, z, R)) {
      float g = 0.f;
      for_node_points(x, y, z, R, ranges, [&](uint32_t s, int c) { g += w[8 * (size_t)s + c] * u[s]; });
      v = lap(p, j, R) + sw * g;
    }
    Ap[j] = v;
    acc[0] += (double)p[j] * (double)v;
  }
};

// x += alpha p, r -= alpha Ap, with the partials of r . r
struct UpdateOp {
  const Scal* s;
  const float* p;
  const float* Ap;
  float* x;
  float* r;
  __device__ void operator()(long long j, double* acc) const {
    const float a = (float)s->alpha;
    x[j] += a * p[j];
    const float rv = r[j] - a * Ap[j];
    r[j] = rv;
    acc[0] += (double)rv * (double)rv;
  }
};

struct DotOp {
  const float* a;
  const float* b;
  __device__ void operator()(long long j, double* acc) const { acc[0] += (double)a[j] * (double)b[j]; }
};

// p = z + beta p
__global__ void direction_kernel(long long n, const Scal* __restrict__ s, const float* __restrict__ z,
                                 float* __restrict__ p) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) p[j] = z[j] + (float)s->beta * p[j];
}

// ----------------------------------------------------------------------------------------------------------- V-cycle
// One red (color 0) or black (color 1) Gauss-Seidel half-sweep of stencil e = f on the interior of an n^3 level.
__global__ void gs_kernel(int n, int color, const float* __restrict__ f, float* __restrict__ e) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= (long long)n * n * n) return;
  int x, y, z;
  node_xyz(j, n, x, y, z);
  if (!interior(x, y, z, n) || ((x + y + z) & 1) != color) return;
  const long long sx = (long long)n * n, sy = n;
  e[j] = (f[j] + (((e[j - sx] + e[j + sx]) + (e[j - sy] + e[j + sy])) + (e[j - 1] + e[j + 1]))) * (1.f / 6.f);
}

__global__ void residual_kernel(int n, const float* __restrict__ f, const float* __restrict__ e, float* __restrict__ res) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= (long long)n * n * n) return;
  int x, y, z;
  node_xyz(j, n, x, y, z);
  res[j] = interior(x, y, z, n) ? f[j] - lap(e, j, n) : 0.f;
}

// coarse f = 4 * full weighting of the fine residual (the coarse stencil is in units of its own spacing 2h)
__global__ void restrict_kernel(int nc, const float* __restrict__ res, float* __restrict__ fc) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= (long long)nc * nc * nc) return;
  int X, Y, Z;
  node_xyz(j, nc, X, Y, Z);
  if (!interior(X, Y, Z, nc)) { fc[j] = 0.f; return; }
  const int nf = 2 * nc - 1;
  float acc = 0.f;
  for (int dx = -1; dx <= 1; dx++)
    for (int dy = -1; dy <= 1; dy++)
      for (int dz = -1; dz <= 1; dz++) {
        const float wgt = (float)(1 << (3 - abs(dx) - abs(dy) - abs(dz))) * (1.f / 64.f);
        acc += wgt * res[((long long)(2 * X + dx) * nf + 2 * Y + dy) * nf + 2 * Z + dz];
      }
  fc[j] = 4.f * acc;
}

// e += trilinear prolongation of the coarse correction, on the fine interior
__global__ void prolong_kernel(int nf, const float* __restrict__ ec, float* __restrict__ e) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= (long long)nf * nf * nf) return;
  int x, y, z;
  node_xyz(j, nf, x, y, z);
  if (!interior(x, y, z, nf)) return;
  const int nc = (nf + 1) / 2;
  const int X0 = x >> 1, Y0 = y >> 1, Z0 = z >> 1, X1 = X0 + (x & 1), Y1 = Y0 + (y & 1), Z1 = Z0 + (z & 1);
  auto at = [&](int X, int Y, int Z) { return ec[((long long)X * nc + Y) * nc + Z]; };
  const float v = (((at(X0, Y0, Z0) + at(X1, Y0, Z0)) + (at(X0, Y1, Z0) + at(X1, Y1, Z0))) +
                   ((at(X0, Y0, Z1) + at(X1, Y0, Z1)) + (at(X0, Y1, Z1) + at(X1, Y1, Z1)))) * 0.125f;
  e[j] += v;
}

// --------------------------------------------------------------------------------------------------- surface, trim
struct IsoOp {
  int R;
  const uint32_t* keys;
  const float* w;
  const float* chi;
  __device__ void operator()(long long s, double* acc) const {
    const int C = R - 1;
    const uint32_t key = keys[s];
    const int cx = (int)(key / ((uint32_t)C * C)), cy = (int)((key / C) % C), cz = (int)(key % C);
    double v = 0.0;
    for (int c = 0; c < 8; c++)
      v += (double)w[8 * s + c] *
           (double)chi[((size_t)(cx + ((c >> 2) & 1)) * R + cy + ((c >> 1) & 1)) * R + cz + (c & 1)];
    acc[0] += v;
  }
};

__global__ void negate_kernel(long long n, const float* __restrict__ a, float* __restrict__ b) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) b[j] = -a[j];
}

// the density D at each marching-cubes vertex (index coordinates), trilinear in fp32
__global__ void vertex_density_kernel(int V, int R, const float* __restrict__ v, const float* __restrict__ D,
                                      float* __restrict__ dens) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= V) return;
  int c[3];
  float f[3];
  for (int k = 0; k < 3; k++) {
    const float q = v[3 * i + k];
    c[k] = min(max((int)floorf(q), 0), R - 2);
    f[k] = q - (float)c[k];
  }
  float acc = 0.f;
  for (int cc = 0; cc < 8; cc++) {
    const float wx = (cc & 4) ? f[0] : 1.f - f[0], wy = (cc & 2) ? f[1] : 1.f - f[1], wz = (cc & 1) ? f[2] : 1.f - f[2];
    acc += ((wx * wy) * wz) * D[((size_t)(c[0] + ((cc >> 2) & 1)) * R + c[1] + ((cc >> 1) & 1)) * R + c[2] + (cc & 1)];
  }
  dens[i] = acc;
}

__global__ void keep_vertex_kernel(int V, const float* __restrict__ dens, float thr, uint32_t* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < V) keep[i] = !(dens[i] < thr);
}

// output vertices (back in the input frame) and faces renumbered through the inclusive scan of the kept vertices
__global__ void emit_vertices_kernel(int V, const float* __restrict__ v, const uint32_t* __restrict__ keep,
                                     const uint32_t* __restrict__ scan, PGrid g, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= V || !keep[i]) return;
  const uint32_t o = scan[i] - 1;
  for (int k = 0; k < 3; k++) out[3 * (size_t)o + k] = (float)(g.origin[k] + g.h * (double)v[3 * i + k]);
}

__global__ void face_flags_kernel(int F, const int3* __restrict__ f, const uint32_t* __restrict__ keep,
                                  const uint32_t* __restrict__ scan, int3* __restrict__ remapped,
                                  uint8_t* __restrict__ flag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= F) return;
  const int3 t = f[i];
  flag[i] = keep[t.x] && keep[t.y] && keep[t.z];
  remapped[i] = make_int3((int)scan[t.x] - 1, (int)scan[t.y] - 1, (int)scan[t.z] - 1);
}

inline unsigned blocks(long long n) { return (unsigned)((n + T - 1) / T); }

// ----------------------------------------------------------------------------------------------------------- driver
struct Level {
  int n;
  float *e, *f, *res;
};

struct Solver {
  std::vector<Level> lv;
  cudaStream_t st;

  cudaError_t gs(const Level& L, int color) {
    gs_kernel<<<blocks((long long)L.n * L.n * L.n), T, 0, st>>>(L.n, color, L.f, L.e);
    g_kernel_launches++;
    return cudaGetLastError();
  }
  // e_l = V-cycle(f_l), the symmetric multigrid preconditioner of L
  cudaError_t vcycle(size_t l) {
    const Level& L = lv[l];
    const long long n3 = (long long)L.n * L.n * L.n;
    cudaError_t e = cudaMemsetAsync(L.e, 0, n3 * sizeof(float), st);
    if (e != cudaSuccess) return e;
    if (l + 1 == lv.size()) {
      for (int s = 0; s < 8; s++)
        if ((e = gs(L, (s % 4 == 0 || s % 4 == 3) ? 0 : 1)) != cudaSuccess) return e;
      return cudaSuccess;
    }
    for (int s = 0; s < 4; s++)
      if ((e = gs(L, s & 1)) != cudaSuccess) return e;
    residual_kernel<<<blocks(n3), T, 0, st>>>(L.n, L.f, L.e, L.res);
    g_kernel_launches++;
    const Level& Cl = lv[l + 1];
    restrict_kernel<<<blocks((long long)Cl.n * Cl.n * Cl.n), T, 0, st>>>(Cl.n, L.res, Cl.f);
    g_kernel_launches++;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    if ((e = vcycle(l + 1)) != cudaSuccess) return e;
    prolong_kernel<<<blocks(n3), T, 0, st>>>(L.n, Cl.e, L.e);
    g_kernel_launches++;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    for (int s = 0; s < 4; s++)
      if ((e = gs(L, 1 - (s & 1))) != cudaSuccess) return e;
    return cudaSuccess;
  }
};

template <int W, class F>
cudaError_t reduce(long long n, F f, double* part, int op, Scal* s, cudaStream_t st) {
  partials_kernel<W><<<kParts, T, 0, st>>>(n, f, part);
  finalize_kernel<<<1, 1024, 0, st>>>(part, W, op, s);
  g_kernel_launches += 2;
  return cudaGetLastError();
}

struct Summer {  // fixed-order fp64 sums of a device array
  const double* a;
  int n;
  double m;
  int mode;  // 0: (sum of a > 0, count of a > 0);  1: sum of (a - m)^2 over a > 0
  __device__ void operator()(long long i, double* acc) const {
    const double v = a[i];
    if (!(v > 0.0)) return;
    if (mode == 0) { acc[0] += v; acc[1] += 1.0; }
    else { acc[0] += (v - m) * (v - m); }
  }
};

struct CentroidOp {
  const float3* p;
  __device__ void operator()(long long i, double* acc) const {
    acc[0] += p[i].x;
    acc[1] += p[i].y;
    acc[2] += p[i].z;
  }
};

struct Timer {
  cudaEvent_t ev[7] = {};
  bool on;
  int n = 0;
  cudaStream_t st;
  Timer(bool on_, cudaStream_t s) : on(on_), st(s) {
    if (on)
      for (auto& e : ev) cudaEventCreate(&e);
  }
  ~Timer() {
    if (on)
      for (auto& e : ev) cudaEventDestroy(e);
  }
  void mark(int i) {
    if (on) { cudaEventRecord(ev[i], st); n = std::max(n, i + 1); }
  }
  void read(double* ms) {
    if (!on) return;
    cudaEventSynchronize(ev[n - 1]);
    for (int i = 0; i + 1 < n; i++) {
      float t = 0.f;
      cudaEventElapsedTime(&t, ev[i], ev[i + 1]);
      ms[i] = t;
    }
  }
};

}  // namespace
}  // namespace dgs

using namespace dgs;

extern "C" int dgs_poisson_reconstruct(const float* points, long long num_points, const float* normals, int depth,
                                       int nb_neighbors, double std_ratio, double scale, double point_weight,
                                       double density_quantile, double tol, int max_iters, dgs_alloc_fn alloc,
                                       void* alloc_user, float** out_vertices, int** out_faces,
                                       long long* out_num_vertices, long long* out_num_faces,
                                       dgs_poisson_stats* stats, const dgs_poisson_trace* trace, void* stream) {
  const char* name = "poisson";
  DGS_REQUIRE(alloc && out_vertices && out_faces && out_num_vertices && out_num_faces,
              "poisson: alloc and the four outputs must not be NULL");
  DGS_REQUIRE(nb_neighbors >= 1 && nb_neighbors <= 32, "poisson: nb_neighbors must be in [1, 32] (got %d)", nb_neighbors);
  DGS_REQUIRE(num_points >= nb_neighbors && num_points <= (1LL << 26),
              "poisson: need nb_neighbors = %d to 2^26 points (got %lld)", nb_neighbors, num_points);
  DGS_REQUIRE(points, "poisson: points must not be NULL");
  DGS_REQUIRE(depth >= 4 && depth <= 9, "poisson: depth must be in [4, 9] (got %d)", depth);
  DGS_REQUIRE(std::isfinite(std_ratio) && std::isfinite(point_weight) && point_weight >= 0,
              "poisson: std_ratio and point_weight must be finite, point_weight >= 0");
  DGS_REQUIRE(std::isfinite(scale) && scale >= 1.0, "poisson: scale must be finite and >= 1 (got %g)", scale);
  DGS_REQUIRE(density_quantile >= 0.0 && density_quantile <= 1.0, "poisson: density_quantile must be in [0, 1] (got %g)",
              density_quantile);
  DGS_REQUIRE(std::isfinite(tol) && tol >= 0 && max_iters >= 1, "poisson: need tol >= 0 and max_iters >= 1");
  *out_vertices = nullptr;
  *out_faces = nullptr;
  *out_num_vertices = *out_num_faces = 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int P = (int)num_points, k = nb_neighbors, R = (1 << depth) + 1, C = R - 1;
  const long long R3 = (long long)R * R * R, C3 = (long long)C * C * C;
  Timer tm(stats != nullptr, st);
  dgs_poisson_stats hs;
  memset(&hs, 0, sizeof(hs));

  // ---- points: kNN, outliers, normals
  size_t sel_bytes = 0, sort_bytes = 0;
  {
    float3* nf3 = nullptr;
    uint8_t* nu8 = nullptr;
    int* ni = nullptr;
    uint32_t* nu = nullptr;
    DGS_CUDA_OK(cub::DeviceSelect::Flagged(nullptr, sel_bytes, nf3, nu8, nf3, ni, P));
    DGS_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, nu, nu, nu, nu, P, 0, 27));
  }
  Carver pc(nullptr);
  auto carve_points = [&](Carver& cv, Scal** s, double** part, int** idx, float** d2, double** a, uint8_t** mask,
                          float3** ip, float3** in, int** cnt, void** temp) {
    *s = cv.take<Scal>(1);
    *part = cv.take<double>(3 * kParts);
    *idx = cv.take<int>((size_t)P * k);
    *d2 = cv.take<float>((size_t)P * k);
    *a = cv.take<double>(P);
    *mask = cv.take<uint8_t>(P);
    *ip = cv.take<float3>(P);
    *in = cv.take<float3>(P);
    *cnt = cv.take<int>(2);
    *temp = cv.take<char>(std::max(sel_bytes, sort_bytes));
  };
  Scal* s;
  double* part;
  int *idx, *cnt;
  float* d2;
  double* a;
  uint8_t* mask;
  float3 *ip, *in;
  void* temp;
  carve_points(pc, &s, &part, &idx, &d2, &a, &mask, &ip, &in, &cnt, &temp);
  {
    void* buf = alloc(pc.bytes(), alloc_user);
    if (!buf) { set_error("%s: scratch allocation failed (%zu bytes)", name, pc.bytes()); return DGS_ERR_ALLOC; }
    Carver cv(buf);
    carve_points(cv, &s, &part, &idx, &d2, &a, &mask, &ip, &in, &cnt, &temp);
  }
  DGS_CUDA_OK(cudaMemsetAsync(s, 0, sizeof(Scal), st));
  if (normals) {
    normal_check_kernel<<<ceil_div(P, T), T, 0, st>>>(P, normals, s);
    DGS_POST_LAUNCH();
  }
  tm.mark(0);
  {
    const int rc = dgs_knn(points, P, k, idx, d2, alloc, alloc_user, stream);  // rejects non-finite points
    if (rc != DGS_OK) return rc;
  }
  if (normals) {
    int bad = 0;
    DGS_CUDA_OK(cudaMemcpyAsync(&bad, &s->bad, sizeof(int), cudaMemcpyDeviceToHost, st));
    DGS_CUDA_OK(cudaStreamSynchronize(st));
    DGS_REQUIRE(bad == 0, "poisson: %d normals are zero or not finite", bad);
  }
  tm.mark(1);
  mean_dist_kernel<<<ceil_div(P, T), T, 0, st>>>(P, k, d2, a);
  DGS_POST_LAUNCH();
  DGS_CUDA_OK(reduce<2>(P, Summer{a, P, 0.0, 0}, part, 0, s, st));
  double sums[2];
  DGS_CUDA_OK(cudaMemcpyAsync(sums, s->sum, sizeof(sums), cudaMemcpyDeviceToHost, st));
  DGS_CUDA_OK(cudaStreamSynchronize(st));
  const double nvalid = sums[1], mean = nvalid > 0 ? sums[0] / nvalid : 0.0;
  double sd = 0.0;
  if (nvalid >= 2) {
    DGS_CUDA_OK(reduce<1>(P, Summer{a, P, mean, 1}, part, 0, s, st));
    DGS_CUDA_OK(cudaMemcpyAsync(sums, s->sum, sizeof(double), cudaMemcpyDeviceToHost, st));
    DGS_CUDA_OK(cudaStreamSynchronize(st));
    sd = std::sqrt(sums[0] / (nvalid - 1.0));
  }
  inlier_kernel<<<ceil_div(P, T), T, 0, st>>>(P, a, mean + std_ratio * sd, mask);
  DGS_POST_LAUNCH();
  if (trace && trace->inliers)
    DGS_CUDA_OK(cudaMemcpyAsync(trace->inliers, mask, P, cudaMemcpyDeviceToDevice, st));
  DGS_CUDA_OK(cub::DeviceSelect::Flagged(temp, sel_bytes, reinterpret_cast<const float3*>(points), mask, ip, cnt, P, st));
  if (normals)
    DGS_CUDA_OK(cub::DeviceSelect::Flagged(temp, sel_bytes, reinterpret_cast<const float3*>(normals), mask, in, cnt, P,
                                           st));
  int N = 0;
  DGS_CUDA_OK(cudaMemcpyAsync(&N, cnt, sizeof(int), cudaMemcpyDeviceToHost, st));
  DGS_CUDA_OK(cudaStreamSynchronize(st));  // the inlier count sizes everything below
  hs.inliers = N;
  if (stats) *stats = hs;
  DGS_REQUIRE(N > 0, "poisson: no point is an inlier");
  DGS_CUDA_OK(reduce<3>(N, CentroidOp{ip}, part, 0, s, st));
  if (normals) {
    normalize_kernel<<<ceil_div(N, T), T, 0, st>>>(N, in);
    DGS_POST_LAUNCH();
  } else {
    const int rc = dgs_knn(reinterpret_cast<const float*>(ip), N, k, idx, d2, alloc, alloc_user, stream);
    if (rc != DGS_OK) return rc;
    pca_kernel<<<ceil_div(N, T), T, 0, st>>>(N, k, ip, idx, s, in);
    DGS_POST_LAUNCH();
  }
  if (trace && trace->normals)
    DGS_CUDA_OK(cudaMemcpyAsync(trace->normals, in, (size_t)N * sizeof(float3), cudaMemcpyDeviceToDevice, st));
  tm.mark(2);

  // ---- grid and splat
  DGS_CUDA_OK(cudaMemsetAsync(s->box, 0xff, 3 * sizeof(unsigned), st));
  DGS_CUDA_OK(cudaMemsetAsync(s->box + 3, 0, 3 * sizeof(unsigned), st));
  box_kernel<<<ceil_div(N, T), T, 0, st>>>(N, ip, s);
  DGS_POST_LAUNCH();
  unsigned box[6];
  DGS_CUDA_OK(cudaMemcpyAsync(box, s->box, sizeof(box), cudaMemcpyDeviceToHost, st));
  DGS_CUDA_OK(cudaStreamSynchronize(st));  // the box places the grid
  PGrid g;
  g.R = R;
  double side = 0.0, ctr[3];
  for (int q = 0; q < 3; q++) {
    const double lo = fval(box[q]), hi = fval(box[3 + q]);
    ctr[q] = 0.5 * (lo + hi);
    side = std::max(side, hi - lo);
  }
  DGS_REQUIRE(side > 0, "poisson: the inliers are all one point");
  side *= scale;
  g.h = side / C;
  for (int q = 0; q < 3; q++) g.origin[q] = ctr[q] - 0.5 * side;

  size_t gsort = 0;
  {
    uint32_t* nu = nullptr;
    DGS_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, gsort, nu, nu, nu, nu, N, 0, 3 * depth));
  }
  Solver sv;
  sv.st = st;
  auto carve_grid = [&](Carver& cv, uint32_t** kin, uint32_t** keys, uint32_t** vin, uint32_t** vals, float3** sn,
                        float** w, float** u, uint2** ranges, float** f, void** gt) {
    *kin = cv.take<uint32_t>(N);
    *keys = cv.take<uint32_t>(N);
    *vin = cv.take<uint32_t>(N);
    *vals = cv.take<uint32_t>(N);
    *sn = cv.take<float3>(N);
    *w = cv.take<float>(8 * (size_t)N);
    *u = cv.take<float>(N);
    *ranges = cv.take<uint2>(C3);
    for (int q = 0; q < 10; q++) f[q] = cv.take<float>(R3);
    *gt = cv.take<char>(gsort);
    sv.lv.clear();
    sv.lv.push_back(Level{R, nullptr, nullptr, nullptr});
    for (int n = (R + 1) / 2; n >= 5; n = (n + 1) / 2) {
      const long long n3 = (long long)n * n * n;
      sv.lv.push_back(Level{n, cv.take<float>(n3), cv.take<float>(n3), cv.take<float>(n3)});
    }
  };
  uint32_t *kin, *keys, *vin, *vals;
  float3* sn;
  float *w, *u;
  uint2* ranges;
  float* f[10];
  void* gt;
  Carver gp(nullptr);
  carve_grid(gp, &kin, &keys, &vin, &vals, &sn, &w, &u, &ranges, f, &gt);
  {
    void* buf = alloc(gp.bytes(), alloc_user);
    if (!buf) { set_error("%s: grid allocation failed (%zu bytes)", name, gp.bytes()); return DGS_ERR_ALLOC; }
    Carver cv(buf);
    carve_grid(cv, &kin, &keys, &vin, &vals, &sn, &w, &u, &ranges, f, &gt);
  }
  float *x = f[0], *b = f[1], *r = f[2], *z = f[3], *p = f[4], *Ap = f[5], *D = f[6], *Vx = f[7], *Vy = f[8],
        *Vz = f[9];
  cell_kernel<<<ceil_div(N, T), T, 0, st>>>(N, ip, g, kin, vin);
  DGS_POST_LAUNCH();
  DGS_CUDA_OK(cub::DeviceRadixSort::SortPairs(gt, gsort, kin, keys, vin, vals, N, 0, 3 * depth, st));
  DGS_CUDA_OK(cudaMemsetAsync(ranges, 0, (size_t)C3 * sizeof(uint2), st));
  ranges_kernel<<<ceil_div(N, T), T, 0, st>>>(N, keys, ranges);
  DGS_POST_LAUNCH();
  weights_kernel<<<ceil_div(N, T), T, 0, st>>>(N, ip, in, g, keys, vals, sn, w);
  DGS_POST_LAUNCH();
  const double r2n = (double)R * R / N;
  splat_kernel<<<blocks(R3), T, 0, st>>>(R, ranges, w, sn, (float)r2n, D, Vx, Vy, Vz);
  DGS_POST_LAUNCH();
  rhs_kernel<<<blocks(R3), T, 0, st>>>(R, Vx, Vy, Vz, b);
  DGS_POST_LAUNCH();
  tm.mark(3);

  // ---- solve: PCG with the V-cycle; Vx is the finest level's residual scratch once b is formed
  sv.lv[0].f = r;
  sv.lv[0].e = z;
  sv.lv[0].res = Vx;
  const float sw = (float)(point_weight * r2n);
  DGS_CUDA_OK(cudaMemsetAsync(x, 0, R3 * sizeof(float), st));
  DGS_CUDA_OK(cudaMemcpyAsync(r, b, R3 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  DGS_CUDA_OK(reduce<1>(R3, DotOp{b, b}, part, 0, s, st));
  double bb = 0.0;
  DGS_CUDA_OK(cudaMemcpyAsync(&bb, s->sum, sizeof(double), cudaMemcpyDeviceToHost, st));
  DGS_CUDA_OK(cudaStreamSynchronize(st));
  int iters = 0;
  double rel = 0.0;
  if (bb > 0) {
    DGS_CUDA_OK(sv.vcycle(0));
    DGS_CUDA_OK(reduce<1>(R3, DotOp{r, z}, part, 3, s, st));
    DGS_CUDA_OK(cudaMemcpyAsync(p, z, R3 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    rel = 1.0;
    while (iters < max_iters) {
      interp_kernel<<<ceil_div(N, T), T, 0, st>>>(N, R, keys, w, p, u);
      DGS_POST_LAUNCH();
      DGS_CUDA_OK(reduce<1>(R3, ApplyOp{R, sw, p, u, w, ranges, Ap}, part, 1, s, st));
      DGS_CUDA_OK(reduce<1>(R3, UpdateOp{s, p, Ap, x, r}, part, 0, s, st));
      double rr = 0.0;
      DGS_CUDA_OK(cudaMemcpyAsync(&rr, s->sum, sizeof(double), cudaMemcpyDeviceToHost, st));
      DGS_CUDA_OK(cudaStreamSynchronize(st));  // the one read-back of the iteration: the stopping test
      iters++;
      rel = std::sqrt(rr / bb);
      if (!(rel > tol) || iters >= max_iters) break;
      DGS_CUDA_OK(sv.vcycle(0));
      DGS_CUDA_OK(reduce<1>(R3, DotOp{r, z}, part, 2, s, st));
      direction_kernel<<<blocks(R3), T, 0, st>>>(R3, s, z, p);
      DGS_POST_LAUNCH();
    }
  }
  hs.iterations = iters;
  hs.residual = rel;
  if (trace && trace->chi) DGS_CUDA_OK(cudaMemcpyAsync(trace->chi, x, R3 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  tm.mark(4);

  // ---- surface
  DGS_CUDA_OK(reduce<1>(N, IsoOp{R, keys, w, x}, part, 0, s, st));
  double iso_sum = 0.0;
  DGS_CUDA_OK(cudaMemcpyAsync(&iso_sum, s->sum, sizeof(double), cudaMemcpyDeviceToHost, st));
  negate_kernel<<<blocks(R3), T, 0, st>>>(R3, x, z);
  DGS_POST_LAUNCH();
  DGS_CUDA_OK(cudaStreamSynchronize(st));
  hs.iso = iso_sum / N;
  float* mv = nullptr;
  int* mf = nullptr;
  long long V = 0, F = 0;
  {
    const int rc = dgs_marching_cubes(z, R, R, R, (float)(-hs.iso), alloc, alloc_user, &mv, &mf, &V, &F, stream);
    if (rc != DGS_OK) return rc;
  }
  hs.vertices_before = V;
  hs.faces_before = F;
  tm.mark(5);

  // ---- trim
  long long NV = V, NF = F;
  if (V > 0) {
    size_t tb = 0, t2 = 0, t3 = 0;
    {
      float* nfl = nullptr;
      uint32_t* nu = nullptr;
      int3* n3 = nullptr;
      uint8_t* n8 = nullptr;
      int* ni = nullptr;
      DGS_CUDA_OK(cub::DeviceRadixSort::SortKeys(nullptr, tb, nfl, nfl, (int)V));
      DGS_CUDA_OK(cub::DeviceScan::InclusiveSum(nullptr, t2, nu, nu, (int)V));
      DGS_CUDA_OK(cub::DeviceSelect::Flagged(nullptr, t3, n3, n8, n3, ni, (int)std::max(F, 1LL)));
      tb = std::max(tb, std::max(t2, t3));
    }
    auto carve_trim = [&](Carver& cv, float** dens, float** sorted, uint32_t** keep, uint32_t** scan, int3** remap,
                          uint8_t** flag, int3** fout, void** tt) {
      *dens = cv.take<float>(V);
      *sorted = cv.take<float>(V);
      *keep = cv.take<uint32_t>(V);
      *scan = cv.take<uint32_t>(V);
      *remap = cv.take<int3>(std::max(F, 1LL));
      *flag = cv.take<uint8_t>(std::max(F, 1LL));
      *fout = cv.take<int3>(std::max(F, 1LL));
      *tt = cv.take<char>(tb);
    };
    float *dens, *sorted;
    uint32_t *keep, *scan;
    int3 *remap, *fout;
    uint8_t* flag;
    void* tt;
    Carver tp(nullptr);
    carve_trim(tp, &dens, &sorted, &keep, &scan, &remap, &flag, &fout, &tt);
    void* buf = alloc(tp.bytes(), alloc_user);
    if (!buf) { set_error("%s: trim allocation failed (%zu bytes)", name, tp.bytes()); return DGS_ERR_ALLOC; }
    Carver cv(buf);
    carve_trim(cv, &dens, &sorted, &keep, &scan, &remap, &flag, &fout, &tt);
    const int Vi = (int)V, Fi = (int)F;
    vertex_density_kernel<<<ceil_div(Vi, T), T, 0, st>>>(Vi, R, mv, D, dens);
    DGS_POST_LAUNCH();
    if (trace && trace->density && trace->density_capacity > 0)
      DGS_CUDA_OK(cudaMemcpyAsync(trace->density, dens, (size_t)std::min(V, trace->density_capacity) * sizeof(float),
                                  cudaMemcpyDeviceToDevice, st));
    float thr = -INFINITY;
    if (density_quantile > 0) {
      // numpy.quantile(densities, q) ('linear') on fp32 data: virtual index q (V - 1), lerp in fp32
      DGS_CUDA_OK(cub::DeviceRadixSort::SortKeys(tt, tb, dens, sorted, Vi, 0, 32, st));
      const double vi = density_quantile * (double)(V - 1);
      const long long lo = std::min((long long)std::floor(vi), V - 1), hi = std::min(lo + 1, V - 1);
      float ab[2];
      DGS_CUDA_OK(cudaMemcpyAsync(&ab[0], sorted + lo, sizeof(float), cudaMemcpyDeviceToHost, st));
      DGS_CUDA_OK(cudaMemcpyAsync(&ab[1], sorted + hi, sizeof(float), cudaMemcpyDeviceToHost, st));
      DGS_CUDA_OK(cudaStreamSynchronize(st));
      const float t = (float)(vi - (double)lo);
      const volatile float diff = ab[1] - ab[0];
      if (t >= 0.5f) {
        const volatile float m = diff * (1.f - t);
        thr = ab[1] - m;
      } else {
        const volatile float m = diff * t;
        thr = ab[0] + m;
      }
    }
    keep_vertex_kernel<<<ceil_div(Vi, T), T, 0, st>>>(Vi, dens, thr, keep);
    DGS_POST_LAUNCH();
    DGS_CUDA_OK(cub::DeviceScan::InclusiveSum(tt, tb, keep, scan, Vi, st));
    if (Fi > 0) {
      face_flags_kernel<<<ceil_div(Fi, T), T, 0, st>>>(Fi, reinterpret_cast<const int3*>(mf), keep, scan, remap, flag);
      DGS_POST_LAUNCH();
      DGS_CUDA_OK(cub::DeviceSelect::Flagged(tt, tb, remap, flag, fout, cnt, Fi, st));
    } else {
      DGS_CUDA_OK(cudaMemsetAsync(cnt, 0, sizeof(int), st));
    }
    uint32_t nv = 0;
    int nf = 0;
    DGS_CUDA_OK(cudaMemcpyAsync(&nv, scan + V - 1, sizeof(nv), cudaMemcpyDeviceToHost, st));
    DGS_CUDA_OK(cudaMemcpyAsync(&nf, cnt, sizeof(nf), cudaMemcpyDeviceToHost, st));
    DGS_CUDA_OK(cudaStreamSynchronize(st));  // the counts size the outputs
    NV = nv;
    NF = nf;
    float* ov = NV ? reinterpret_cast<float*>(alloc((size_t)NV * 3 * sizeof(float), alloc_user)) : nullptr;
    int* of = NF ? reinterpret_cast<int*>(alloc((size_t)NF * 3 * sizeof(int), alloc_user)) : nullptr;
    if ((NV && !ov) || (NF && !of)) { set_error("%s: output allocation failed", name); return DGS_ERR_ALLOC; }
    emit_vertices_kernel<<<ceil_div(Vi, T), T, 0, st>>>(Vi, mv, keep, scan, g, ov);
    DGS_POST_LAUNCH();
    if (NF) DGS_CUDA_OK(cudaMemcpyAsync(of, fout, (size_t)NF * sizeof(int3), cudaMemcpyDeviceToDevice, st));
    *out_vertices = ov;
    *out_faces = of;
  }
  *out_num_vertices = NV;
  *out_num_faces = NF;
  hs.vertices = NV;
  hs.faces = NF;
  tm.mark(6);
  if (stats) {
    tm.read(hs.stage_ms);
    *stats = hs;
  }
  return DGS_OK;
}
