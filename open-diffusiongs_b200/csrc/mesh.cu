// mesh.cu -- mesh extraction from Gaussians: the block-truncated opacity field of GaussianModel.extract_fields
// (gs_core.py:786-852) and marching cubes over a dense field (what extract_mesh gets from PyMCubes, gs_core.py:855-869).
//
// Field: per-Gaussian records (normalised centre, opacity, inverse-covariance coefficients) are formed once, each
// Gaussian's box of grid blocks is emitted as (block, Gaussian) pairs in Gaussian order, the pairs are radix-sorted by
// block (stable, so every block's list stays in Gaussian order) and each block's points are summed over its list in
// that fixed order: no atomics, the same bits on every run.
//
// Marching cubes: a classify pass over grid points (sign-changing edges owned by the point, case of the voxel it is
// the origin of), in-place scans of the vertex and triangle counts, one read-back of the two totals, and an emit pass.
// Vertex order is by owning edge (grid point, then axis), triangle order by voxel, then case-table order.
#include <cub/cub.cuh>

#include "dgs_internal.h"
#include "mc_tables.h"
#include "sorted_ranges.cuh"

namespace dgs {
namespace {

// ---------------------------------------------------------------------------------------------------- opacity field
struct GaussRec {
  float4 a;  // normalised centre x, y, z; opacity
  float4 b;  // log2(e) * power coefficients: xx, yy, zz, xy
  float4 c;  // xz, yz, unused, unused
};

constexpr int kPrepThreads = 256;
constexpr int kEvalWarps = 8;

struct Grid {
  const float* lin;  // [R] the fp32 linspace(-1, 1, R)
  int R, split, nc;  // points per axis, points per chunk, chunks per axis
  float margin;      // fp32(block_size * relax_ratio)
  __device__ float vmin(int c) const { return __fsub_rn(lin[c * split], margin); }
  __device__ float vmax(int c) const { return __fadd_rn(lin[min((c + 1) * split, R) - 1], margin); }
  // [lo, hi) = the chunks with vmin < x < vmax (strict, as the reference's mask); empty for NaN
  __device__ int2 chunks(float x) const {
    int lo = 0, hi = nc;
    while (lo < hi) {  // first chunk with x < vmax
      const int m = (lo + hi) >> 1;
      if (x < vmax(m)) hi = m; else lo = m + 1;
    }
    int lo2 = 0, hi2 = nc;
    while (lo2 < hi2) {  // first chunk without vmin < x
      const int m = (lo2 + hi2) >> 1;
      if (vmin(m) < x) lo2 = m + 1; else hi2 = m;
    }
    return make_int2(lo, max(lo, lo2));
  }
};

// Per Gaussian: the reference's fp32 arithmetic op for op (separately rounded, in its evaluation order) for the
// normalised centre, the covariance (R S)(R S)^T with R from the raw quaternion over its Euclidean norm, and the
// cofactor inverse; then the block box and its pair count.
__global__ void __launch_bounds__(kPrepThreads) field_prep_kernel(
    int P, const float* __restrict__ xyz, const float* __restrict__ scaling, const float* __restrict__ rotation,
    const float* __restrict__ opacity, float smod, const float* __restrict__ center, float scale, Grid grid,
    GaussRec* __restrict__ rec, int4* __restrict__ box, unsigned long long* __restrict__ npairs) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= P) return;
  float p[3], s[3];
  for (int k = 0; k < 3; k++) {
    p[k] = __fmul_rn(__fsub_rn(xyz[3 * g + k], center[k]), scale);
    s[k] = __fmul_rn(__fmul_rn(expf(scaling[3 * g + k]), smod), scale);
  }
  const float r0 = rotation[4 * g], r1 = rotation[4 * g + 1], r2 = rotation[4 * g + 2], r3 = rotation[4 * g + 3];
  const float nrm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r0, r0), __fmul_rn(r1, r1)), __fmul_rn(r2, r2)),
                                         __fmul_rn(r3, r3)));
  const float r = __fdiv_rn(r0, nrm), x = __fdiv_rn(r1, nrm), y = __fdiv_rn(r2, nrm), z = __fdiv_rn(r3, nrm);
  float Rm[3][3];
  Rm[0][0] = __fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(__fmul_rn(y, y), __fmul_rn(z, z))));
  Rm[0][1] = __fmul_rn(2.f, __fsub_rn(__fmul_rn(x, y), __fmul_rn(r, z)));
  Rm[0][2] = __fmul_rn(2.f, __fadd_rn(__fmul_rn(x, z), __fmul_rn(r, y)));
  Rm[1][0] = __fmul_rn(2.f, __fadd_rn(__fmul_rn(x, y), __fmul_rn(r, z)));
  Rm[1][1] = __fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(__fmul_rn(x, x), __fmul_rn(z, z))));
  Rm[1][2] = __fmul_rn(2.f, __fsub_rn(__fmul_rn(y, z), __fmul_rn(r, x)));
  Rm[2][0] = __fmul_rn(2.f, __fsub_rn(__fmul_rn(x, z), __fmul_rn(r, y)));
  Rm[2][1] = __fmul_rn(2.f, __fadd_rn(__fmul_rn(y, z), __fmul_rn(r, x)));
  Rm[2][2] = __fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y))));
  float L[3][3];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) L[i][j] = __fmul_rn(Rm[i][j], s[j]);
  auto cov = [&](int i, int k) {
    return __fadd_rn(__fadd_rn(__fmul_rn(L[i][0], L[k][0]), __fmul_rn(L[i][1], L[k][1])), __fmul_rn(L[i][2], L[k][2]));
  };
  const float a = cov(0, 0), b = cov(0, 1), c = cov(0, 2), d = cov(1, 1), e = cov(1, 2), f = cov(2, 2);
  // gaussian_3d_coeff (gs_core.py:27-46)
  float det = __fmul_rn(__fmul_rn(a, d), f);
  det = __fadd_rn(det, __fmul_rn(__fmul_rn(__fmul_rn(2.f, e), c), b));
  det = __fsub_rn(det, __fmul_rn(__fmul_rn(e, e), a));
  det = __fsub_rn(det, __fmul_rn(__fmul_rn(c, c), d));
  det = __fsub_rn(det, __fmul_rn(__fmul_rn(b, b), f));
  const float inv_det = __fdiv_rn(1.f, __fadd_rn(det, 1e-24f));
  const float ia = __fmul_rn(__fsub_rn(__fmul_rn(d, f), __fmul_rn(e, e)), inv_det);
  const float ib = __fmul_rn(__fsub_rn(__fmul_rn(e, c), __fmul_rn(b, f)), inv_det);
  const float ic = __fmul_rn(__fsub_rn(__fmul_rn(e, b), __fmul_rn(c, d)), inv_det);
  const float id = __fmul_rn(__fsub_rn(__fmul_rn(a, f), __fmul_rn(c, c)), inv_det);
  const float ie = __fmul_rn(__fsub_rn(__fmul_rn(b, c), __fmul_rn(e, a)), inv_det);
  const float iff = __fmul_rn(__fsub_rn(__fmul_rn(a, d), __fmul_rn(b, b)), inv_det);
  // power = -0.5 (x^2 ia + y^2 id + z^2 if) - xy ib - xz ic - yz ie, evaluated in the log2 domain
  const float h = -0.5f * 1.4426950408889634f, l2e = -1.4426950408889634f;
  const float op = 1.f / (1.f + expf(-opacity[g]));
  GaussRec o;
  o.a = make_float4(p[0], p[1], p[2], op);
  o.b = make_float4(h * ia, h * id, h * iff, l2e * ib);
  o.c = make_float4(l2e * ic, l2e * ie, 0.f, 0.f);
  rec[g] = o;
  const int2 bx = grid.chunks(p[0]), by = grid.chunks(p[1]), bz = grid.chunks(p[2]);
  box[g] = make_int4(bx.x | (bx.y << 16), by.x | (by.y << 16), bz.x | (bz.y << 16), 0);
  npairs[g] = (unsigned long long)(bx.y - bx.x) * (by.y - by.x) * (bz.y - bz.x);
}

// (block, Gaussian) pairs of each Gaussian's box, at its offset in the inclusive scan of the pair counts
__global__ void __launch_bounds__(kPrepThreads) field_fill_kernel(int P, int nc, const int4* __restrict__ box,
                                                                  const unsigned long long* __restrict__ scan,
                                                                  uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= P) return;
  const int4 bb = box[g];
  const int x0 = bb.x & 0xffff, x1 = bb.x >> 16, y0 = bb.y & 0xffff, y1 = bb.y >> 16, z0 = bb.z & 0xffff,
            z1 = bb.z >> 16;
  const unsigned long long n = (unsigned long long)(x1 - x0) * (y1 - y0) * (z1 - z0);
  unsigned long long o = scan[g] - n;
  for (int bx = x0; bx < x1; bx++)
    for (int by = y0; by < y1; by++)
      for (int bz = z0; bz < z1; bz++, o++) {
        keys[o] = (uint32_t)((bx * nc + by) * nc + bz);
        vals[o] = (uint32_t)g;
      }
}

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

struct FieldScratch {
  GaussRec* rec;
  int4* box;
  unsigned long long* npairs;
  uint2* ranges;
  void* temp;
  size_t temp_bytes;
  size_t carve(void* base, int P, long long nblocks) {
    Carver cv(base);
    rec = cv.take<GaussRec>(P);
    box = cv.take<int4>(P);
    npairs = cv.take<unsigned long long>(P);
    ranges = cv.take<uint2>(nblocks);
    temp_bytes = 0;
    cub::DeviceScan::InclusiveSum(nullptr, temp_bytes, npairs, npairs, P);
    temp = cv.take<char>(temp_bytes);
    return cv.bytes();
  }
};

struct PairScratch {
  uint32_t *keys_in, *keys, *vals_in, *vals;
  void* temp;
  size_t temp_bytes;
  size_t carve(void* base, int n, int end_bit) {
    Carver cv(base);
    keys_in = cv.take<uint32_t>(n);
    keys = cv.take<uint32_t>(n);
    vals_in = cv.take<uint32_t>(n);
    vals = cv.take<uint32_t>(n);
    temp_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, temp_bytes, keys_in, keys, vals_in, vals, n, 0, end_bit);
    temp = cv.take<char>(temp_bytes);
    return cv.bytes();
  }
};

// ---------------------------------------------------------------------------------------------------- marching cubes
__global__ void mc_classify_kernel(const float* __restrict__ f, int nx, int ny, int nz, float iso,
                                   uint8_t* __restrict__ ecode, uint8_t* __restrict__ cases, uint32_t* __restrict__ vscan,
                                   uint32_t* __restrict__ tscan) {
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
  void* fbuf = scratch_alloc(fs.carve(nullptr, P, nblocks), scratch_user);
  if (!fbuf) { set_error("mesh field: scratch allocation failed"); return DGS_ERR_ALLOC; }
  fs.carve(fbuf, P, nblocks);
  field_prep_kernel<<<ceil_div(P, kPrepThreads), kPrepThreads, 0, st>>>(P, xyz, scaling, rotation, opacity,
                                                                         scale_modifier, center, scale, grid, fs.rec,
                                                                         fs.box, fs.npairs);
  DGS_POST_LAUNCH();
  DGS_CUDA_OK(cub::DeviceScan::InclusiveSum(fs.temp, fs.temp_bytes, fs.npairs, fs.npairs, P, st));
  unsigned long long total = 0;
  DGS_CUDA_OK(cudaMemcpyAsync(&total, fs.npairs + P - 1, sizeof(total), cudaMemcpyDeviceToHost, st));
  DGS_CUDA_OK(cudaStreamSynchronize(st));  // the one host sync: the pair count sizes the sort
  if (num_pairs) *num_pairs = (long long)total;
  if (total > 0x7fffffffULL) {
    set_error("mesh field: %llu (block, Gaussian) pairs do not fit 32 bits", total);
    return DGS_ERR_OVERFLOW;
  }
  DGS_CUDA_OK(cudaMemsetAsync(fs.ranges, 0, nblocks * sizeof(uint2), st));
  const int n = (int)total;
  if (n > 0) {
    int end_bit = 1;
    while (end_bit < 32 && (1LL << end_bit) < nblocks) end_bit++;
    PairScratch ps;
    void* pbuf = scratch_alloc(ps.carve(nullptr, n, end_bit), scratch_user);
    if (!pbuf) { set_error("mesh field: pair allocation failed (%d pairs)", n); return DGS_ERR_ALLOC; }
    ps.carve(pbuf, n, end_bit);
    field_fill_kernel<<<ceil_div(P, kPrepThreads), kPrepThreads, 0, st>>>(P, nc, fs.box, fs.npairs, ps.keys_in,
                                                                          ps.vals_in);
    DGS_POST_LAUNCH();
    DGS_CUDA_OK(cub::DeviceRadixSort::SortPairs(ps.temp, ps.temp_bytes, ps.keys_in, ps.keys, ps.vals_in, ps.vals, n, 0,
                                                end_bit, st));
    ranges_kernel<<<ceil_div(n, 256), 256, 0, st>>>(n, ps.keys, fs.ranges);
    DGS_POST_LAUNCH();
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
  DGS_REQUIRE(field && alloc && vertices && triangles && num_vertices && num_triangles,
              "marching cubes: field, alloc and the four outputs must not be NULL");
  DGS_REQUIRE(nx >= 2 && ny >= 2 && nz >= 2, "marching cubes: the field must be at least 2 x 2 x 2 (got %d x %d x %d)",
              nx, ny, nz);
  const long long N = (long long)nx * ny * nz;
  DGS_REQUIRE(N * DGS_MC_MAX_TRIS <= 0x7fffffffLL, "marching cubes: %d x %d x %d grid points is too many (at most %lld)",
              nx, ny, nz, 0x7fffffffLL / DGS_MC_MAX_TRIS);
  *vertices = nullptr;
  *triangles = nullptr;
  *num_vertices = *num_triangles = 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
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
  if (!buf) { set_error("marching cubes: scratch allocation failed"); return DGS_ERR_ALLOC; }
  carve(buf, &ecode, &cases, &vscan, &tscan, &temp);
  const unsigned grid = (unsigned)((N + 255) / 256);
  mc_classify_kernel<<<grid, 256, 0, st>>>(field, nx, ny, nz, iso, ecode, cases, vscan, tscan);
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
  if (!v || (tot[1] && !t)) { set_error("marching cubes: output allocation failed"); return DGS_ERR_ALLOC; }
  mc_emit_kernel<<<grid, 256, 0, st>>>(field, nx, ny, nz, iso, ecode, cases, vscan, tscan, v, t);
  DGS_POST_LAUNCH();
  *vertices = v;
  *triangles = t;
  *num_vertices = tot[0];
  *num_triangles = tot[1];
  return DGS_OK;
}

}  // extern "C"
