// mesh_field.cuh -- the per-block Gaussian lists of the opacity field (GaussianModel.extract_fields,
// gs_core.py:786-852), shared by mesh.cu's field and mesh_color.cu's vertex colours so both sum the same Gaussians, with
// the same records, in the same order.
//
// Per-Gaussian records (normalised centre, opacity, inverse-covariance coefficients) are formed once, each Gaussian's
// box of grid blocks is emitted as (block, Gaussian) pairs in Gaussian order, and the pairs are radix-sorted by block
// (stable, so every block's list stays in Gaussian order) and cut into one range per block.  The kernels and
// build_block_lists are compiled once, in mesh.cu (which defines DGS_MESH_FIELD_LISTS), with the field's flags: a thin
// Gaussian's cofactor inverse turns one ulp of a scale into about 1e-3 of its power, so records formed under another
// file's flags (mesh_color.cu's -fmad=false changes expf's code) would not be the field's.
#pragma once
#include <cub/cub.cuh>

#include "dgs_internal.h"
#include "sorted_ranges.cuh"

namespace dgs {

struct GaussRec {
  float4 a;  // normalised centre x, y, z; opacity
  float4 b;  // log2(e) * power coefficients: xx, yy, zz, xy
  float4 c;  // xz, yz, unused, unused
};

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
  // The chunk of the grid point at or below x: the largest i with lin[i] <= x, clamped to [0, R - 1] (0 for NaN and
  // below -1), over split.
  __device__ int chunk_of(float x) const {
    int lo = 0, hi = R;
    while (lo < hi) {  // first point with x < lin[i] (NaN: none is passed over)
      const int m = (lo + hi) >> 1;
      if (lin[m] <= x) lo = m + 1; else hi = m;
    }
    return max(lo - 1, 0) / split;
  }
};

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

// The bits of a block index below nblocks: the width of the radix sorts keyed by block.
inline int block_bits(long long nblocks) {
  int end_bit = 1;
  while (end_bit < 32 && (1LL << end_bit) < nblocks) end_bit++;
  return end_bit;
}

// The lists of P > 0 Gaussians: fs.rec the records, fs.ranges[block] the block's run of ps.vals (Gaussian ids in
// Gaussian order), *num_pairs the total (also when it is too many).  scratch_alloc is called for fs, then, after the one host sync that reads the
// pair count, for ps when there are pairs (ps is left unset when there are none).  Errors are reported under `name`.
int build_block_lists(const char* name, int P, const float* xyz, const float* scaling, const float* rotation,
                      const float* opacity, float scale_modifier, const float* center, float scale,
                      const Grid& grid, long long nblocks, dgs_alloc_fn scratch_alloc, void* scratch_user,
                      cudaStream_t st, FieldScratch& fs, PairScratch& ps, long long* num_pairs);

}  // namespace dgs

#ifdef DGS_MESH_FIELD_LISTS
namespace dgs {
namespace {

constexpr int kPrepThreads = 256;

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

}  // namespace

int build_block_lists(const char* name, int P, const float* xyz, const float* scaling, const float* rotation,
                      const float* opacity, float scale_modifier, const float* center, float scale,
                      const Grid& grid, long long nblocks, dgs_alloc_fn scratch_alloc, void* scratch_user,
                      cudaStream_t st, FieldScratch& fs, PairScratch& ps, long long* num_pairs) {
  void* fbuf = scratch_alloc(fs.carve(nullptr, P, nblocks), scratch_user);
  if (!fbuf) { set_error("%s: scratch allocation failed", name); return DGS_ERR_ALLOC; }
  fs.carve(fbuf, P, nblocks);
  field_prep_kernel<<<ceil_div(P, kPrepThreads), kPrepThreads, 0, st>>>(P, xyz, scaling, rotation, opacity,
                                                                  scale_modifier, center, scale, grid, fs.rec,
                                                                  fs.box, fs.npairs);
  DGS_POST_LAUNCH();
  DGS_CUDA_OK(cub::DeviceScan::InclusiveSum(fs.temp, fs.temp_bytes, fs.npairs, fs.npairs, P, st));
  unsigned long long total = 0;
  DGS_CUDA_OK(cudaMemcpyAsync(&total, fs.npairs + P - 1, sizeof(total), cudaMemcpyDeviceToHost, st));
  DGS_CUDA_OK(cudaStreamSynchronize(st));  // the one host sync: the pair count sizes the sort
  *num_pairs = (long long)total;
  if (total > 0x7fffffffULL) {
    set_error("%s: %llu (block, Gaussian) pairs do not fit 32 bits", name, total);
    return DGS_ERR_OVERFLOW;
  }
  DGS_CUDA_OK(cudaMemsetAsync(fs.ranges, 0, nblocks * sizeof(uint2), st));
  const int n = (int)total;
  if (n == 0) return DGS_OK;
  const int end_bit = block_bits(nblocks);
  void* pbuf = scratch_alloc(ps.carve(nullptr, n, end_bit), scratch_user);
  if (!pbuf) { set_error("%s: pair allocation failed (%d pairs)", name, n); return DGS_ERR_ALLOC; }
  ps.carve(pbuf, n, end_bit);
  field_fill_kernel<<<ceil_div(P, kPrepThreads), kPrepThreads, 0, st>>>(P, grid.nc, fs.box, fs.npairs, ps.keys_in,
                                                                 ps.vals_in);
  DGS_POST_LAUNCH();
  DGS_CUDA_OK(cub::DeviceRadixSort::SortPairs(ps.temp, ps.temp_bytes, ps.keys_in, ps.keys, ps.vals_in, ps.vals, n, 0,
                                       end_bit, st));
  ranges_kernel<<<ceil_div(n, 256), 256, 0, st>>>(n, ps.keys, fs.ranges);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

}  // namespace dgs
#endif  // DGS_MESH_FIELD_LISTS
