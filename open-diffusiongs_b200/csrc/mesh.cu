// mesh.cu -- mesh extraction from Gaussians: the block-truncated opacity field of GaussianModel.extract_fields
// (gs_core.py:786-852) and marching cubes over a dense field (what extract_mesh gets from PyMCubes, gs_core.py:855-869).
//
// Field: the per-block Gaussian lists of mesh_field.cuh (in Gaussian order), and each block's points summed over its
// list in that fixed order: no atomics, the same bits on every run.
//
// Marching cubes: a classify pass over grid points (sign-changing edges owned by the point, case of the voxel it is
// the origin of), in-place scans of the vertex and triangle counts, one read-back of the two totals, and an emit pass.
// Vertex order is by owning edge (grid point, then axis), triangle order by voxel, then case-table order.
// The masked instantiation (the TSDF extraction of tsdf.cu) keeps only what observed points support: a voxel emits
// triangles only when its 8 corners are observed, and an edge a vertex only when both its ends are observed and a voxel
// containing it is, so every vertex is referenced and no face touches an unobserved point.
#include <cub/cub.cuh>

#include "dgs_internal.h"
#include "mc_tables.h"
#define DGS_MESH_FIELD_LISTS  // the one file that compiles the list build
#include "mesh_field.cuh"

namespace dgs {
namespace {

// ---------------------------------------------------------------------------------------------------- opacity field
constexpr int kEvalWarps = 8;

// One warp per grid block, eight blocks per CTA.  At the default 4^3 points per block a warp holds the block's 64
// points two per lane, so every warp sums its points over the whole list itself: no reduction across warps and no
// CTA barrier, and an SM keeps 64 blocks in flight.  The list is staged 32 records at a time in the warp's shared
// slice; larger blocks (e.g. 8^3 at resolution 128 / 16 blocks) take their points 64 at a time.
__global__ void __launch_bounds__(32 * kEvalWarps) field_eval_kernel(Grid grid, const uint2* __restrict__ ranges,
                                                                     const uint32_t* __restrict__ vals,
                                                                     const GaussRec* __restrict__ rec,
                                                                     float* __restrict__ occ, int* __restrict__ counts) {
  __shared__ float4 stage[kEvalWarps][3][32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int nc = grid.nc, R = grid.R, split = grid.split;
  const long long blk = (long long)blockIdx.x * kEvalWarps + wid;
  if (blk >= (long long)nc * nc * nc) return;
  const uint2 rg = ranges[blk];
  const int n = (int)(rg.y - rg.x);
  if (counts && lane == 0) counts[blk] = n;
  if (n == 0) return;  // the field was zeroed: blocks without Gaussians stay 0
  const int bx = (int)(blk / ((long long)nc * nc)), by = (int)((blk / nc) % nc), bz = (int)(blk % nc);
  const int x0 = bx * split, y0 = by * split, z0 = bz * split;
  const int lx = min(split, R - x0), ly = min(split, R - y0), lz = min(split, R - z0), npts = lx * ly * lz;
  float4(&sa)[32] = stage[wid][0];
  float4(&sb)[32] = stage[wid][1];
  float4(&sc)[32] = stage[wid][2];
  for (int base = 0; base < npts; base += 64) {
    float px[2], py[2], pz[2], acc[2] = {0.f, 0.f};
    size_t out[2];
    bool live[2];
    for (int u = 0; u < 2; u++) {
      const int q = base + lane + 32 * u;
      live[u] = q < npts;
      const int qq = live[u] ? q : 0;
      const int ix = qq / (ly * lz), iy = (qq / lz) % ly, iz = qq % lz;
      px[u] = grid.lin[x0 + ix];
      py[u] = grid.lin[y0 + iy];
      pz[u] = grid.lin[z0 + iz];
      out[u] = ((size_t)(x0 + ix) * R + (y0 + iy)) * R + (z0 + iz);
    }
    for (int s0 = 0; s0 < n; s0 += 32) {
      const int m = min(32, n - s0);
      __syncwarp();
      if (lane < m) {
        const GaussRec gr = rec[vals[rg.x + s0 + lane]];
        sa[lane] = gr.a;
        sb[lane] = gr.b;
        sc[lane] = gr.c;
      }
      __syncwarp();
      for (int j = 0; j < m; j++) {
        const float4 A = sa[j], B = sb[j], Cc = sc[j];
#pragma unroll
        for (int u = 0; u < 2; u++) {
          const float dx = px[u] - A.x, dy = py[u] - A.y, dz = pz[u] - A.z;
          const float pw = dx * (B.x * dx + B.w * dy + Cc.x * dz) + dy * (B.y * dy + Cc.y * dz) + B.z * dz * dz;
          acc[u] += pw > 0.f ? 0.f : A.w * exp2f(pw);
        }
      }
    }
    for (int u = 0; u < 2; u++)
      if (live[u]) occ[out[u]] = acc[u];
  }
}

// ---------------------------------------------------------------------------------------------------- marching cubes
// Bit (dx + 1) + 3 (dy + 1) + 9 (dz + 1) of the 27-bit neighbourhood mask; whether all 8 corners of the voxel whose
// origin is offset (ox, oy, oz) in {-1, 0}^3 from the centre are set.
__device__ __forceinline__ int nb_bit(int dx, int dy, int dz) { return (dx + 1) + 3 * (dy + 1) + 9 * (dz + 1); }
__device__ __forceinline__ bool voxel_full(uint32_t nb, int ox, int oy, int oz) {
#pragma unroll
  for (int c = 0; c < 8; c++)
    if (!((nb >> nb_bit(ox + (c & 1), oy + ((c >> 1) & 1), oz + (c >> 2))) & 1)) return false;
  return true;
}

// kMasked: only points with weight > 0 are observed (the rules in the header); weight is unused otherwise.
template <bool kMasked>
__global__ void mc_classify_kernel(const float* __restrict__ f, int nx, int ny, int nz, float iso,
                                   uint8_t* __restrict__ ecode, uint8_t* __restrict__ cases, uint32_t* __restrict__ vscan,
                                   uint32_t* __restrict__ tscan, const int* __restrict__ weight) {
  const long long N = (long long)nx * ny * nz;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int x = (int)(i / ((long long)ny * nz)), y = (int)((i / nz) % ny), z = (int)(i % nz);
  const long long sx = (long long)ny * nz, sy = nz;
  const bool in = f[i] > iso;
  uint32_t e = 0;
  if (x + 1 < nx && (f[i + sx] > iso) != in) e |= 1;
  if (y + 1 < ny && (f[i + sy] > iso) != in) e |= 2;
  if (z + 1 < nz && (f[i + 1] > iso) != in) e |= 4;
  uint32_t cs = 0, nt = 0;
  if (x + 1 < nx && y + 1 < ny && z + 1 < nz) {
#pragma unroll
    for (int c = 0; c < 8; c++)
      if (f[i + (c & 1) * sx + ((c >> 1) & 1) * sy + (c >> 2)] > iso) cs |= 1u << c;
    nt = kMcNumTris[cs];
  }
  if constexpr (kMasked) {
    uint32_t nb = 0;  // observed points of the 3 x 3 x 3 neighbourhood; points outside the grid are not observed
    for (int dz = -1; dz <= 1; dz++)
      for (int dy = -1; dy <= 1; dy++)
        for (int dx = -1; dx <= 1; dx++) {
          const int qx = x + dx, qy = y + dy, qz = z + dz;
          if (qx >= 0 && qx < nx && qy >= 0 && qy < ny && qz >= 0 && qz < nz && weight[i + dx * sx + dy * sy + dz] > 0)
            nb |= 1u << nb_bit(dx, dy, dz);
        }
    // an edge along axis a lies in the 4 voxels with origin offset 0 along a and -1 or 0 along the other two axes
    const bool fx = voxel_full(nb, 0, -1, -1) || voxel_full(nb, 0, 0, -1) || voxel_full(nb, 0, -1, 0) ||
                    voxel_full(nb, 0, 0, 0);
    const bool fy = voxel_full(nb, -1, 0, -1) || voxel_full(nb, 0, 0, -1) || voxel_full(nb, -1, 0, 0) ||
                    voxel_full(nb, 0, 0, 0);
    const bool fz = voxel_full(nb, -1, -1, 0) || voxel_full(nb, 0, -1, 0) || voxel_full(nb, -1, 0, 0) ||
                    voxel_full(nb, 0, 0, 0);
    const bool here = (nb >> nb_bit(0, 0, 0)) & 1;
    if (!(here && ((nb >> nb_bit(1, 0, 0)) & 1) && fx)) e &= ~1u;
    if (!(here && ((nb >> nb_bit(0, 1, 0)) & 1) && fy)) e &= ~2u;
    if (!(here && ((nb >> nb_bit(0, 0, 1)) & 1) && fz)) e &= ~4u;
    if (!voxel_full(nb, 0, 0, 0)) cs = nt = 0;
  }
  ecode[i] = (uint8_t)e;
  cases[i] = (uint8_t)cs;
  vscan[i] = __popc(e);
  tscan[i] = nt;
}

__global__ void mc_emit_kernel(const float* __restrict__ f, int nx, int ny, int nz, float iso,
                               const uint8_t* __restrict__ ecode, const uint8_t* __restrict__ cases,
                               const uint32_t* __restrict__ vscan, const uint32_t* __restrict__ tscan,
                               float* __restrict__ verts, int* __restrict__ tris) {
  const long long N = (long long)nx * ny * nz;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const long long sx = (long long)ny * nz, sy = nz;
  const uint32_t e = ecode[i];
  if (e) {
    const int x = (int)(i / sx), y = (int)((i / nz) % ny), z = (int)(i % nz);
    const float va = f[i];
    uint32_t v = vscan[i] - __popc(e);
    for (int a = 0; a < 3; a++) {
      if (!((e >> a) & 1)) continue;
      const float vb = f[i + (a == 0 ? sx : a == 1 ? sy : 1)];
      const float t = (iso - va) / (vb - va);
      verts[3 * (size_t)v + 0] = (float)x + (a == 0 ? t : 0.f);
      verts[3 * (size_t)v + 1] = (float)y + (a == 1 ? t : 0.f);
      verts[3 * (size_t)v + 2] = (float)z + (a == 2 ? t : 0.f);
      v++;
    }
  }
  const int cs = cases[i], nt = kMcNumTris[cs];
  if (nt == 0) return;
  uint32_t t = tscan[i] - nt;
  for (int k = 0; k < 3 * nt; k++) {
    const int edge = kMcTriEdges[cs][k], c0 = kMcEdgeCorners[edge][0], a = edge >> 2;
    const long long q = i + (c0 & 1) * sx + ((c0 >> 1) & 1) * sy + (c0 >> 2);
    const uint32_t eq = ecode[q];
    tris[3 * (size_t)t + k] = (int)(vscan[q] - __popc(eq) + __popc(eq & ((1u << a) - 1)));
  }
}

}  // namespace
}  // namespace dgs

using namespace dgs;

extern "C" {

int dgs_mesh_field(int P, const float* xyz, const float* scaling, const float* rotation, const float* opacity,
                   float scale_modifier, const float* center, float scale, int resolution, int num_blocks,
                   double relax_ratio, const float* lin, float* occ, int* block_counts, long long* num_pairs,
                   dgs_alloc_fn scratch_alloc, void* scratch_user, void* stream) {
  DGS_REQUIRE(P >= 0, "mesh field: P must be >= 0 (got %d)", P);
  DGS_REQUIRE(resolution >= 1 && resolution <= 4096, "mesh field: resolution must be in [1, 4096] (got %d)", resolution);
  DGS_REQUIRE(num_blocks >= 1 && num_blocks <= resolution,
              "mesh field: num_blocks must be in [1, resolution] (got %d at resolution %d)", num_blocks, resolution);
  DGS_REQUIRE(lin && occ && scratch_alloc, "mesh field: lin, occ and scratch_alloc must not be NULL");
  DGS_REQUIRE(P == 0 || (xyz && scaling && rotation && opacity && center),
              "mesh field: xyz, scaling, rotation, opacity and center must not be NULL");
  const int split = resolution / num_blocks, nc = ceil_div(resolution, split);
  const long long nblocks = (long long)nc * nc * nc;
  DGS_REQUIRE(nblocks <= 0x7fffffffLL && nc < 0x8000, "mesh field: %d chunks per axis is too many", nc);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t R3 = (size_t)resolution * resolution * resolution;
  if (num_pairs) *num_pairs = 0;
  DGS_CUDA_OK(cudaMemsetAsync(occ, 0, R3 * sizeof(float), st));
  if (P == 0) {
    if (block_counts) DGS_CUDA_OK(cudaMemsetAsync(block_counts, 0, nblocks * sizeof(int), st));
    return DGS_OK;
  }
  Grid grid{lin, resolution, split, nc, (float)((2.0 / num_blocks) * relax_ratio)};
  FieldScratch fs;
  PairScratch ps;
  long long total = 0;
  const int rc = build_block_lists("mesh field", P, xyz, scaling, rotation, opacity, scale_modifier, center, scale,
                                   grid, nblocks, scratch_alloc, scratch_user, st, fs, ps, &total);
  if (num_pairs) *num_pairs = total;
  if (rc != DGS_OK) return rc;
  if (total > 0) {
    field_eval_kernel<<<(unsigned)((nblocks + kEvalWarps - 1) / kEvalWarps), 32 * kEvalWarps, 0, st>>>(
        grid, fs.ranges, ps.vals, fs.rec, occ, block_counts);
    DGS_POST_LAUNCH();
  } else if (block_counts) {
    DGS_CUDA_OK(cudaMemsetAsync(block_counts, 0, nblocks * sizeof(int), st));
  }
  return DGS_OK;
}

int dgs_marching_cubes(const float* field, int nx, int ny, int nz, float iso, dgs_alloc_fn alloc, void* alloc_user,
                       float** vertices, int** triangles, long long* num_vertices, long long* num_triangles,
                       void* stream) {
  return marching_cubes("marching cubes", field, nullptr, nx, ny, nz, iso, alloc, alloc_user, vertices, triangles,
                        num_vertices, num_triangles, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"

namespace dgs {

int marching_cubes(const char* name, const float* field, const int* weight, int nx, int ny, int nz, float iso,
                   dgs_alloc_fn alloc, void* alloc_user, float** vertices, int** triangles, long long* num_vertices,
                   long long* num_triangles, cudaStream_t st) {
  DGS_REQUIRE(field && alloc && vertices && triangles && num_vertices && num_triangles,
              "%s: field, alloc and the four outputs must not be NULL", name);
  DGS_REQUIRE(nx >= 2 && ny >= 2 && nz >= 2, "%s: the field must be at least 2 x 2 x 2 (got %d x %d x %d)", name,
              nx, ny, nz);
  const long long N = (long long)nx * ny * nz;
  DGS_REQUIRE(N * DGS_MC_MAX_TRIS <= 0x7fffffffLL, "%s: %d x %d x %d grid points is too many (at most %lld)", name,
              nx, ny, nz, 0x7fffffffLL / DGS_MC_MAX_TRIS);
  *vertices = nullptr;
  *triangles = nullptr;
  *num_vertices = *num_triangles = 0;
  size_t temp_bytes = 0;
  uint32_t* nul = nullptr;
  DGS_CUDA_OK(cub::DeviceScan::InclusiveSum(nullptr, temp_bytes, nul, nul, (int)N));
  auto carve = [&](void* base, uint8_t** ecode, uint8_t** cases, uint32_t** vscan, uint32_t** tscan, void** temp) {
    Carver cv(base);
    *ecode = cv.take<uint8_t>(N);
    *cases = cv.take<uint8_t>(N);
    *vscan = cv.take<uint32_t>(N);
    *tscan = cv.take<uint32_t>(N);
    *temp = cv.take<char>(temp_bytes);
    return cv.bytes();
  };
  uint8_t *ecode, *cases;
  uint32_t *vscan, *tscan;
  void* temp;
  void* buf = alloc(carve(nullptr, &ecode, &cases, &vscan, &tscan, &temp), alloc_user);
  if (!buf) { set_error("%s: scratch allocation failed", name); return DGS_ERR_ALLOC; }
  carve(buf, &ecode, &cases, &vscan, &tscan, &temp);
  const unsigned grid = (unsigned)((N + 255) / 256);
  if (weight)
    mc_classify_kernel<true><<<grid, 256, 0, st>>>(field, nx, ny, nz, iso, ecode, cases, vscan, tscan, weight);
  else
    mc_classify_kernel<false><<<grid, 256, 0, st>>>(field, nx, ny, nz, iso, ecode, cases, vscan, tscan, nullptr);
  DGS_POST_LAUNCH();
  DGS_CUDA_OK(cub::DeviceScan::InclusiveSum(temp, temp_bytes, vscan, vscan, (int)N, st));
  DGS_CUDA_OK(cub::DeviceScan::InclusiveSum(temp, temp_bytes, tscan, tscan, (int)N, st));
  uint32_t tot[2];
  DGS_CUDA_OK(cudaMemcpyAsync(&tot[0], vscan + N - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  DGS_CUDA_OK(cudaMemcpyAsync(&tot[1], tscan + N - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  DGS_CUDA_OK(cudaStreamSynchronize(st));  // the one host sync: the totals size the outputs
  if (tot[0] == 0) return DGS_OK;          // no sign change: no vertex and no triangle
  float* v = reinterpret_cast<float*>(alloc((size_t)tot[0] * 3 * sizeof(float), alloc_user));
  int* t = tot[1] ? reinterpret_cast<int*>(alloc((size_t)tot[1] * 3 * sizeof(int), alloc_user)) : nullptr;
  if (!v || (tot[1] && !t)) { set_error("%s: output allocation failed", name); return DGS_ERR_ALLOC; }
  mc_emit_kernel<<<grid, 256, 0, st>>>(field, nx, ny, nz, iso, ecode, cases, vscan, tscan, v, t);
  DGS_POST_LAUNCH();
  *vertices = v;
  *triangles = t;
  *num_vertices = tot[0];
  *num_triangles = tot[1];
  return DGS_OK;
}

}  // namespace dgs
