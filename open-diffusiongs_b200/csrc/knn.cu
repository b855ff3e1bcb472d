// knn.cu -- exact k-nearest neighbours of a point cloud (k <= 32): the neighbour search under
// dgs_poisson_reconstruct's outlier removal and normal estimation, and under simple_knn's distCUDA2.
//
// Contract (include/dgs_b200.h, dgs_knn): every point's k nearest points of the cloud, itself included at distance 0
// (as Open3D's SearchKNN), duplicates included; the squared distance of p and q is the fp32 (dx*dx + dy*dy) + dz*dz
// with dx = q.x - p.x, rounded product by product (this file is compiled with -fmad=false); the order is by
// (squared distance, index), so ties go to the smaller index.  Slots beyond P get index -1 and distance +inf.
//
// Method: a uniform grid over the cloud's bounding box.  It starts at about cbrt(P / 4) cells along the longest axis
// (a volume-filling cloud then holds about 4 points per cell) and doubles while the occupied cells hold more than 8
// points on average (a cloud on a surface or a curve occupies far fewer cells than the box holds), up to 16 P + 64
// cells in all and 1024 per axis.  Each round radix-sorts the points by cell key and counts the occupied cells; the
// last round's order and per-cell ranges (sorted_ranges.cuh) are the grid.  Then one warp per point searches rings of
// cells outwards from the point's cell; lane j holds the j-th best (distance, index) so far, and a candidate that beats
// the k-th best is inserted by one shift of the lanes above its place.  The search stops when the k-th best distance
// is below the distance from the point to the cells not yet searched, less a margin for the rounding of the cell
// indices (the rule of mesh_remesh.cu's closest-point query), or when the rings cover the grid.
//
// No floating-point atomics (the bounding box is taken over order-preserving integer keys): the same bits on every
// run.  Non-finite coordinates are rejected.
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>

#include "dgs_internal.h"
#include "sorted_ranges.cuh"

namespace dgs {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxAxis = 1024;  // cells per axis
constexpr int kNone = 0x7fffffff;
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

struct Check {
  unsigned box[6];  // order-preserving keys: min x y z, max x y z
  int nonfinite;
  unsigned long long occupied;
};

struct KGrid {
  double mn[3], h;
  int n[3];
};

__device__ __forceinline__ int cell_of(const KGrid& g, float x, int k) {
  const double c = floor(((double)x - g.mn[k]) / g.h);
  return (int)fmin(fmax(c, 0.0), (double)(g.n[k] - 1));
}

__global__ void box_kernel(int P, const float* __restrict__ pts, Check* __restrict__ chk) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned lo[3] = {kFull, kFull, kFull}, hi[3] = {0u, 0u, 0u};
  bool bad = false;
  if (i < P) {
    for (int k = 0; k < 3; k++) {
      const float x = pts[3 * i + k];
      bad |= !isfinite(x);
      lo[k] = fkey(x);
      hi[k] = lo[k];
    }
  }
  for (int k = 0; k < 3; k++) {
    lo[k] = __reduce_min_sync(kFull, lo[k]);
    hi[k] = __reduce_max_sync(kFull, hi[k]);
  }
  const unsigned nbad = __popc(__ballot_sync(kFull, bad));
  if ((threadIdx.x & 31) == 0) {
    for (int k = 0; k < 3; k++) {
      atomicMin(&chk->box[k], lo[k]);
      atomicMax(&chk->box[3 + k], hi[k]);
    }
    if (nbad) atomicAdd(&chk->nonfinite, (int)nbad);
  }
}

__global__ void key_kernel(int P, const float* __restrict__ pts, KGrid g, uint32_t* __restrict__ keys,
                           uint32_t* __restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const int x = cell_of(g, pts[3 * i], 0), y = cell_of(g, pts[3 * i + 1], 1), z = cell_of(g, pts[3 * i + 2], 2);
  keys[i] = ((uint32_t)x * g.n[1] + y) * g.n[2] + z;
  vals[i] = i;
}

// occupied cells: the heads of the runs of the sorted keys (integer atomics only)
__global__ void occupied_kernel(int P, const uint32_t* __restrict__ keys, Check* __restrict__ chk) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool head = i < P && (i == 0 || keys[i] != keys[i - 1]);
  const unsigned n = __popc(__ballot_sync(kFull, head));
  if ((threadIdx.x & 31) == 0 && n) atomicAdd(&chk->occupied, (unsigned long long)n);
}

__global__ void gather_kernel(int P, const float* __restrict__ pts, const uint32_t* __restrict__ vals,
                              float4* __restrict__ spts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const int j = (int)vals[i];
  spts[i] = make_float4(pts[3 * j], pts[3 * j + 1], pts[3 * j + 2], __int_as_float(j));
}

__device__ __forceinline__ bool less(float da, int ia, float db, int ib) { return da < db || (da == db && ia < ib); }

// One warp per point, in cell order; lane j keeps the j-th best (d, i) of the point.
__global__ void __launch_bounds__(kThreads) knn_kernel(int P, int k, KGrid g, const float4* __restrict__ spts,
                                                       const uint2* __restrict__ ranges, int* __restrict__ out_idx,
                                                       float* __restrict__ out_d2) {
  const int lane = threadIdx.x & 31;
  const int s = blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (s >= P) return;
  const float4 q = spts[s];
  const int self = __float_as_int(q.w);
  const int c[3] = {cell_of(g, q.x, 0), cell_of(g, q.y, 1), cell_of(g, q.z, 2)};
  float bd = INFINITY;
  int bi = kNone;
  float kd = INFINITY;  // the k-th best, lane k - 1's
  int ki = kNone;
  const double tol = 1e-6 * g.h;
  for (int r = 0;; r++) {
    for (int dx = -r; dx <= r; dx++) {
      const int x = c[0] + dx;
      if (x < 0 || x >= g.n[0]) continue;
      for (int dy = -r; dy <= r; dy++) {
        const int y = c[1] + dy;
        if (y < 0 || y >= g.n[1]) continue;
        const int step = (abs(dx) == r || abs(dy) == r) ? 1 : max(2 * r, 1);
        for (int dz = -r; dz <= r; dz += step) {
          const int z = c[2] + dz;
          if (z < 0 || z >= g.n[2]) continue;
          const uint2 rg = ranges[((uint32_t)x * g.n[1] + y) * g.n[2] + z];
          for (uint32_t base = rg.x; base < rg.y; base += 32) {
            const uint32_t j = base + lane;
            float cd = INFINITY;
            int ci = kNone;
            if (j < rg.y) {
              const float4 p = spts[j];
              const float ex = p.x - q.x, ey = p.y - q.y, ez = p.z - q.z;
              cd = (ex * ex + ey * ey) + ez * ez;
              ci = __float_as_int(p.w);
            }
            unsigned m = __ballot_sync(kFull, j < rg.y && less(cd, ci, kd, ki));
            while (m) {
              const int src = __ffs(m) - 1;
              const float nd = __shfl_sync(kFull, cd, src);
              const int ni = __shfl_sync(kFull, ci, src);
              const int pos = __popc(__ballot_sync(kFull, less(bd, bi, nd, ni)));
              const float ud = __shfl_up_sync(kFull, bd, 1);
              const int ui = __shfl_up_sync(kFull, bi, 1);
              if (lane == pos) { bd = nd; bi = ni; }
              else if (lane > pos) { bd = ud; bi = ui; }
              kd = __shfl_sync(kFull, bd, k - 1);
              ki = __shfl_sync(kFull, bi, k - 1);
              m &= ~(1u << src);
              m &= __ballot_sync(kFull, less(cd, ci, kd, ki));
            }
          }
        }
      }
    }
    bool covered = true;
    double dmin = INFINITY;
    const float qc[3] = {q.x, q.y, q.z};
    for (int a = 0; a < 3; a++) {
      if (c[a] - r > 0) { covered = false; dmin = fmin(dmin, (double)qc[a] - (g.mn[a] + (c[a] - r) * g.h)); }
      if (c[a] + r < g.n[a] - 1) { covered = false; dmin = fmin(dmin, g.mn[a] + (c[a] + r + 1) * g.h - (double)qc[a]); }
    }
    if (covered || (ki != kNone && sqrt((double)kd) * (1.0 + 1e-5) + tol < dmin)) break;
  }
  if (lane < k) {
    const size_t o = (size_t)self * k + lane;
    out_idx[o] = bi == kNone ? -1 : bi;
    out_d2[o] = bi == kNone ? INFINITY : bd;
  }
}

}  // namespace
}  // namespace dgs

using namespace dgs;

extern "C" int dgs_knn(const float* points, long long num_points, int k, int* out_idx, float* out_d2,
                       dgs_alloc_fn alloc, void* alloc_user, void* stream) {
  DGS_REQUIRE(k >= 1 && k <= 32, "knn: k must be in [1, 32] (got %d)", k);
  DGS_REQUIRE(num_points >= 0 && num_points <= 0x7fffffffLL / 32, "knn: %lld points is not in [0, 2^26)", num_points);
  DGS_REQUIRE(alloc && (num_points == 0 || (points && out_idx && out_d2)),
              "knn: alloc, points and the outputs must not be NULL");
  if (num_points == 0) return DGS_OK;
  const int P = (int)num_points;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long max_cells = std::min(16LL * P + 64, 1LL << 27);
  size_t sort_bytes = 0;
  {
    uint32_t* nul = nullptr;
    DGS_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, nul, nul, nul, nul, P, 0, 32));
  }
  auto carve = [&](Carver& cv, Check** chk, uint32_t** k_in, uint32_t** keys, uint32_t** v_in, uint32_t** vals,
                   float4** spts, uint2** ranges, void** temp) {
    *chk = cv.take<Check>(1);
    *k_in = cv.take<uint32_t>(P);
    *keys = cv.take<uint32_t>(P);
    *v_in = cv.take<uint32_t>(P);
    *vals = cv.take<uint32_t>(P);
    *spts = cv.take<float4>(P);
    *ranges = cv.take<uint2>(max_cells);
    *temp = cv.take<char>(sort_bytes);
  };
  Check* chk;
  uint32_t *k_in, *keys, *v_in, *vals;
  float4* spts;
  uint2* ranges;
  void* temp;
  Carver probe(nullptr);
  carve(probe, &chk, &k_in, &keys, &v_in, &vals, &spts, &ranges, &temp);
  void* buf = alloc(probe.bytes(), alloc_user);
  if (!buf) { set_error("knn: scratch allocation failed (%zu bytes)", probe.bytes()); return DGS_ERR_ALLOC; }
  Carver cv(buf);
  carve(cv, &chk, &k_in, &keys, &v_in, &vals, &spts, &ranges, &temp);

  Check h;
  DGS_CUDA_OK(cudaMemsetAsync(chk, 0xff, 3 * sizeof(unsigned), st));
  DGS_CUDA_OK(cudaMemsetAsync(chk->box + 3, 0, sizeof(Check) - 3 * sizeof(unsigned), st));
  box_kernel<<<ceil_div(P, kThreads), kThreads, 0, st>>>(P, points, chk);
  DGS_POST_LAUNCH();
  DGS_CUDA_OK(cudaMemcpyAsync(&h, chk, sizeof(h), cudaMemcpyDeviceToHost, st));
  DGS_CUDA_OK(cudaStreamSynchronize(st));  // the box sizes the grid
  DGS_REQUIRE(h.nonfinite == 0, "knn: %d points have a non-finite coordinate", h.nonfinite);

  KGrid g;
  double ext[3], emax = 0.0;
  for (int a = 0; a < 3; a++) {
    g.mn[a] = (double)fval(h.box[a]);
    ext[a] = (double)fval(h.box[3 + a]) - g.mn[a];
    emax = std::max(emax, ext[a]);
  }
  int cells = std::max(1, (int)std::ceil(std::cbrt(P / 4.0)));
  for (;;) {
    g.h = emax > 0 ? emax / cells : 1.0;
    for (int a = 0; a < 3; a++) g.n[a] = std::min((int)std::floor(ext[a] / g.h) + 1, kMaxAxis);
    key_kernel<<<ceil_div(P, kThreads), kThreads, 0, st>>>(P, points, g, k_in, v_in);
    DGS_POST_LAUNCH();
    const int bits = std::max(1, (int)std::ceil(std::log2((double)g.n[0] * g.n[1] * g.n[2] + 1)));
    DGS_CUDA_OK(cub::DeviceRadixSort::SortPairs(temp, sort_bytes, k_in, keys, v_in, vals, P, 0, bits, st));
    // the next size: twice the cells per axis, when the occupied cells are crowded and the grid may grow
    const int next = 2 * cells;
    long long next_total = 1;
    for (int a = 0; a < 3; a++)
      next_total *= std::min((long long)std::floor(ext[a] / (emax > 0 ? emax / next : 1.0)) + 1, (long long)kMaxAxis);
    if (emax == 0 || next > kMaxAxis || next_total > max_cells) break;
    DGS_CUDA_OK(cudaMemsetAsync(&chk->occupied, 0, sizeof(unsigned long long), st));
    occupied_kernel<<<ceil_div(P, kThreads), kThreads, 0, st>>>(P, keys, chk);
    DGS_POST_LAUNCH();
    unsigned long long occ = 0;
    DGS_CUDA_OK(cudaMemcpyAsync(&occ, &chk->occupied, sizeof(occ), cudaMemcpyDeviceToHost, st));
    DGS_CUDA_OK(cudaStreamSynchronize(st));  // the occupancy decides whether the grid is refined
    if ((double)P <= 8.0 * (double)occ) break;
    cells = next;
  }
  const long long total = (long long)g.n[0] * g.n[1] * g.n[2];
  DGS_CUDA_OK(cudaMemsetAsync(ranges, 0, (size_t)total * sizeof(uint2), st));
  ranges_kernel<<<ceil_div(P, kThreads), kThreads, 0, st>>>(P, keys, ranges);
  DGS_POST_LAUNCH();
  gather_kernel<<<ceil_div(P, kThreads), kThreads, 0, st>>>(P, points, vals, spts);
  DGS_POST_LAUNCH();
  knn_kernel<<<ceil_div(P, kWarps), kThreads, 0, st>>>(P, k, g, spts, ranges, out_idx, out_d2);
  DGS_POST_LAUNCH();
  return DGS_OK;
}
