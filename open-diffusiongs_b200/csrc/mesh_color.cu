// mesh_color.cu -- per-vertex normals and colours of an extracted mesh from the Gaussians that produced it
// (include/dgs_b200.h, dgs_mesh_vertex_colors).
//
// Normals: the vertex -> face lists of mesh_common.cuh (face order), each vertex's face normals summed in fp64.  This
// file is compiled with -fmad=false so that sum is the one oracle/mesh_color.py makes, bit for bit.
// Colours: the opacity field's own per-block Gaussian lists and records (mesh_field.cuh's build_block_lists, compiled
// in mesh.cu with the field's flags); the vertices are radix-sorted by the block of their grid point (stable, so in
// index order within a block), and one warp per occupied block takes its vertices 32 at a time, one per lane, against
// the block's list staged 32 records at a time in shared memory.  Every sum runs in a fixed order with no
// floating-point atomics: a vertex's result does not depend on the run or on where the vertex sits in the array.
#include <cub/cub.cuh>

#include "mesh_common.cuh"
#include "mesh_field.cuh"

namespace dgs {
namespace {

constexpr int kColorWarps = 4;

// The real SH basis of the 3DGS rasterizer (public constants), degree <= 3.
constexpr float kC0 = 0.28209479177387814f, kC1 = 0.4886025119029199f;
__constant__ float kC2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f, -1.0925484305920792f,
                          0.5462742152960396f};
__constant__ float kC3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f, 0.3731763325901154f,
                          -0.4570457994644658f, 1.445305721320277f, -0.5900435899266435f};

template <int DEG>
__device__ __forceinline__ void sh_basis(float x, float y, float z, float b[(DEG + 1) * (DEG + 1)]) {
  b[0] = kC0;
  if (DEG > 0) {
    b[1] = -kC1 * y; b[2] = kC1 * z; b[3] = -kC1 * x;
  }
  if (DEG > 1) {
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    b[4] = kC2[0] * xy; b[5] = kC2[1] * yz; b[6] = kC2[2] * (2.0f * zz - xx - yy);
    b[7] = kC2[3] * xz; b[8] = kC2[4] * (xx - yy);
    if (DEG > 2) {
      b[9] = kC3[0] * y * (3.0f * xx - yy);
      b[10] = kC3[1] * xy * z;
      b[11] = kC3[2] * y * (4.0f * zz - xx - yy);
      b[12] = kC3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy);
      b[13] = kC3[4] * x * (4.0f * zz - xx - yy);
      b[14] = kC3[5] * z * (xx - yy);
      b[15] = kC3[6] * x * (xx - 3.0f * yy);
    }
  }
}

// Per vertex: the fp64 sum of (b - a) x (c - a) over its faces in face order, over its length, rounded to fp32; 0
// without faces or for a zero sum.
__global__ void vertex_normal_kernel(int V, const float* __restrict__ pos, const int3* __restrict__ faces,
                                     const uint32_t* __restrict__ vfaces, const uint2* __restrict__ vrange,
                                     float* __restrict__ normals) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const uint2 r = vrange[v];
  double3 s = make_double3(0.0, 0.0, 0.0);
  for (uint32_t i = r.x; i < r.y; i++) {
    const int3 f = faces[vfaces[i]];
    const double3 a = load(pos, f.x);
    const double3 n = cross(sub(load(pos, f.y), a), sub(load(pos, f.z), a));
    s = make_double3(s.x + n.x, s.y + n.y, s.z + n.z);
  }
  const double len = sqrt(dot(s, s));
  float3 o = make_float3(0.f, 0.f, 0.f);
  if (len > 0.0) o = make_float3((float)(s.x / len), (float)(s.y / len), (float)(s.z / len));
  normals[3 * (size_t)v] = o.x;
  normals[3 * (size_t)v + 1] = o.y;
  normals[3 * (size_t)v + 2] = o.z;
}

// Per vertex: its block (the chunk of its grid point on each axis) as the sort key, its index as the value.
__global__ void vertex_block_kernel(int V, const float* __restrict__ pos, Grid grid, uint32_t* __restrict__ keys,
                                    uint32_t* __restrict__ vals) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int bx = grid.chunk_of(pos[3 * v]), by = grid.chunk_of(pos[3 * v + 1]), bz = grid.chunk_of(pos[3 * v + 2]);
  keys[v] = (uint32_t)((bx * grid.nc + by) * grid.nc + bz);
  vals[v] = (uint32_t)v;
}

// One warp per block with vertices, one vertex per lane, 32 at a time.  Each lane forms the SH basis of its direction
// -n once; each (vertex, Gaussian) pair then costs its power (in fp64), one exp2f and 3 (DEG + 1)^2 FMAs, skipped
// when the weight is 0.
// The opacity enters as log2 of it in the staged record's unused third slot of c.
// glist / gvals are the block lists (glist NULL: no Gaussians).
template <int DEG>
__global__ void __launch_bounds__(32 * kColorWarps) vertex_color_kernel(
    long long nblocks, const uint2* __restrict__ vlist, const uint32_t* __restrict__ vsorted,
    const float* __restrict__ pos, const float* __restrict__ normals, const uint2* __restrict__ glist,
    const uint32_t* __restrict__ gvals, const GaussRec* __restrict__ rec, const float* __restrict__ features,
    float* __restrict__ rgb, unsigned long long* __restrict__ unweighted) {
  constexpr int NB = (DEG + 1) * (DEG + 1), NCO = 3 * NB;
  __shared__ float4 stage[kColorWarps][3][32];
  __shared__ float shs[kColorWarps][32 * NCO];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const long long blk = (long long)blockIdx.x * kColorWarps + wid;
  if (blk >= nblocks) return;
  const uint2 vr = vlist[blk];
  if (vr.x == vr.y) return;
  const uint2 gr = glist ? glist[blk] : make_uint2(0u, 0u);
  const int n = (int)(gr.y - gr.x);
  float4(&sa)[32] = stage[wid][0];
  float4(&sb)[32] = stage[wid][1];
  float4(&sc)[32] = stage[wid][2];
  float* sh = shs[wid];
  for (uint32_t base = vr.x; base < vr.y; base += 32) {
    const bool live = base + lane < vr.y;
    const int v = (int)vsorted[live ? base + lane : vr.x];
    const float px = pos[3 * v], py = pos[3 * v + 1], pz = pos[3 * v + 2];
    float y[NB];
    sh_basis<DEG>(-normals[3 * v], -normals[3 * v + 1], -normals[3 * v + 2], y);
    // the sums are kept relative to the largest weight so far (2^top), so no weight underflows: a vertex far from
    // its list's Gaussians gets their colours as precisely as a near one
    float acc[3] = {0.f, 0.f, 0.f}, wsum = 0.f, top = -INFINITY;
    for (int s0 = 0; s0 < n; s0 += 32) {
      const int m = min(32, n - s0);
      __syncwarp();
      if (lane < m) {
        const GaussRec g = rec[gvals[gr.x + s0 + lane]];
        sa[lane] = g.a;
        sb[lane] = g.b;
        sc[lane] = make_float4(g.c.x, g.c.y, log2f(g.a.w), 0.f);  // -inf for opacity 0
      }
      for (int t = lane; t < m * NCO; t += 32) {
        const int j = t / NCO;
        sh[t] = features[(size_t)gvals[gr.x + s0 + j] * NCO + (t - j * NCO)];
      }
      __syncwarp();
      for (int j = 0; j < m; j++) {
        const float4 A = sa[j], B = sb[j], Cc = sc[j];
        // the power in fp64: the quadratic form of a thin Gaussian cancels, and fp32 would lose its low digits
        const double dx = (double)px - A.x, dy = (double)py - A.y, dz = (double)pz - A.z;
        const double pw = dx * (B.x * dx + B.w * dy + Cc.x * dz) + dy * (B.y * dy + Cc.y * dz) + B.z * dz * dz;
        const float lw = (float)pw + Cc.z;  // log2 of the weight
        if (pw > 0.0 || !(lw > -INFINITY)) continue;  // a zero weight
        if (lw > top) {
          const float r = exp2f(top - lw);
          acc[0] *= r; acc[1] *= r; acc[2] *= r; wsum *= r;
          top = lw;
        }
        const float w = exp2f(lw - top);
        const float* c = sh + j * NCO;
#pragma unroll
        for (int ch = 0; ch < 3; ch++) {
          float col = y[0] * c[ch];
#pragma unroll
          for (int k = 1; k < NB; k++) col = fmaf(y[k], c[3 * k + ch], col);
          acc[ch] = fmaf(w, fmaxf(col + 0.5f, 0.f), acc[ch]);
        }
        wsum += w;
      }
    }
    const bool white = !(wsum > 0.f);
    if (live) {
      for (int ch = 0; ch < 3; ch++)
        rgb[3 * (size_t)v + ch] = white ? 1.f : fminf(fmaxf(acc[ch] / wsum, 0.f), 1.f);
    }
    const unsigned nw = __popc(__ballot_sync(kFull, live && white));
    if (lane == 0 && nw) atomicAdd(unweighted, (unsigned long long)nw);
  }
}

struct Scratch : MeshScratch {
  unsigned long long* unweighted;
  FaceCheck* chk;
  float* normals;  // when the caller gives none
  uint32_t *vkey_in, *vkey, *vval_in, *vval;
  uint2* vlist;

  size_t carve(void* base, int V, int F, long long nblocks, bool own_normals) {
    Carver cv(base);
    unweighted = cv.take<unsigned long long>(1);
    chk = cv.take<FaceCheck>(1);
    carve_mesh(cv, V, F, V);
    normals = cv.take<float>(own_normals ? 3 * (size_t)V : 0);
    vkey_in = cv.take<uint32_t>(V);
    vkey = cv.take<uint32_t>(V);
    vval_in = cv.take<uint32_t>(V);
    vval = cv.take<uint32_t>(V);
    vlist = cv.take<uint2>(nblocks);
    size_t t = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, t, vkey_in, vkey, vval_in, vval, V, 0, block_bits(nblocks));
    need(t);
    carve_temp(cv);
    return cv.bytes();
  }
};

template <int DEG>
cudaError_t launch_colors(long long nblocks, const Scratch& s, const float* pos, const float* normals,
                          const uint2* glist, const uint32_t* gvals, const GaussRec* rec, const float* features,
                          float* rgb, cudaStream_t st) {
  vertex_color_kernel<DEG><<<(unsigned)((nblocks + kColorWarps - 1) / kColorWarps), 32 * kColorWarps, 0, st>>>(
      nblocks, s.vlist, s.vval, pos, normals, glist, gvals, rec, features, rgb, s.unweighted);
  g_kernel_launches++;
  return cudaGetLastError();
}

}  // namespace
}  // namespace dgs

using namespace dgs;

extern "C" {

int dgs_mesh_vertex_colors(int P, const float* xyz, const float* features, int sh_degree, const float* scaling,
                           const float* rotation, const float* opacity, float scale_modifier, const float* center,
                           float scale, int resolution, int num_blocks, double relax_ratio, const float* lin,
                           const float* vertices, long long num_vertices, const int* faces, long long num_faces,
                           float* out_rgb, float* out_normals, long long* num_unweighted, dgs_alloc_fn alloc,
                           void* alloc_user, void* stream) {
  const char* name = "mesh vertex colors";
  const int rc0 = check_mesh_input(name, vertices, num_vertices, faces, num_faces,
                                   num_vertices <= 0x7fffffffLL && 3 * num_faces <= 0x7fffffffLL,
                                   "V and 3F must be at most 2^31 - 1");
  if (rc0 != DGS_OK) return rc0;
  DGS_REQUIRE(P >= 0, "%s: P must be >= 0 (got %d)", name, P);
  DGS_REQUIRE(sh_degree >= 0 && sh_degree <= 3, "%s: sh_degree must be in [0, 3] (got %d)", name, sh_degree);
  DGS_REQUIRE(resolution >= 1 && resolution <= 4096, "%s: resolution must be in [1, 4096] (got %d)", name, resolution);
  DGS_REQUIRE(num_blocks >= 1 && num_blocks <= resolution,
              "%s: num_blocks must be in [1, resolution] (got %d at resolution %d)", name, num_blocks, resolution);
  DGS_REQUIRE(lin && alloc && (num_vertices == 0 || out_rgb), "%s: lin, alloc and out_rgb must not be NULL", name);
  DGS_REQUIRE(P == 0 || (xyz && features && scaling && rotation && opacity && center),
              "%s: xyz, features, scaling, rotation, opacity and center must not be NULL", name);
  const int split = resolution / num_blocks, nc = ceil_div(resolution, split);
  const long long nblocks = (long long)nc * nc * nc;
  DGS_REQUIRE(nblocks <= 0x7fffffffLL && nc < 0x8000, "%s: %d chunks per axis is too many", name, nc);
  if (num_unweighted) *num_unweighted = 0;
  if (num_vertices == 0 && num_faces == 0) return DGS_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int V = (int)num_vertices, F = (int)num_faces;
  Scratch s;
  void* buf = alloc(s.carve(nullptr, V, F, nblocks, !out_normals), alloc_user);
  if (!buf) { set_error("%s: scratch allocation failed", name); return DGS_ERR_ALLOC; }
  s.carve(buf, V, F, nblocks, !out_normals);
  float* normals = out_normals ? out_normals : s.normals;
  const int3* in_faces = reinterpret_cast<const int3*>(faces);
  FaceCheck h;
  const int rc1 = check_faces(name, vertices, V, in_faces, F, false, nullptr, s.chk, h, st);
  if (rc1 != DGS_OK) return rc1;
  if (V == 0) return DGS_OK;

  // 1. normals
  if (F > 0) {
    DGS_CUDA_OK(cudaMemcpyAsync(s.faces, in_faces, (size_t)F * sizeof(int3), cudaMemcpyDeviceToDevice, st));
    DGS_CUDA_OK(s.vertex_faces(F, V, st));
  } else {
    DGS_CUDA_OK(cudaMemsetAsync(s.vrange, 0, (size_t)V * sizeof(uint2), st));
  }
  vertex_normal_kernel<<<ceil_div(V, kThreads), kThreads, 0, st>>>(V, vertices, s.faces, s.vfaces, s.vrange, normals);
  DGS_POST_LAUNCH();

  // 2. the field's block lists
  Grid grid{lin, resolution, split, nc, (float)((2.0 / num_blocks) * relax_ratio)};
  FieldScratch fs;
  PairScratch ps{};
  long long pairs = 0;
  if (P > 0) {
    const int rc2 = build_block_lists(name, P, xyz, scaling, rotation, opacity, scale_modifier, center, scale, grid,
                                      nblocks, alloc, alloc_user, st, fs, ps, &pairs);
    if (rc2 != DGS_OK) return rc2;
  }

  // 3. vertices grouped by block
  vertex_block_kernel<<<ceil_div(V, kThreads), kThreads, 0, st>>>(V, vertices, grid, s.vkey_in, s.vval_in);
  DGS_POST_LAUNCH();
  DGS_CUDA_OK(cub::DeviceRadixSort::SortPairs(s.temp, s.temp_bytes, s.vkey_in, s.vkey, s.vval_in, s.vval, V, 0,
                                              block_bits(nblocks), st));
  DGS_CUDA_OK(cudaMemsetAsync(s.vlist, 0, nblocks * sizeof(uint2), st));
  ranges_kernel<<<ceil_div(V, kThreads), kThreads, 0, st>>>(V, s.vkey, s.vlist);
  DGS_POST_LAUNCH();

  // 4. colours
  DGS_CUDA_OK(cudaMemsetAsync(s.unweighted, 0, sizeof(unsigned long long), st));
  const uint2* glist = P > 0 ? fs.ranges : nullptr;
  const uint32_t* gvals = pairs > 0 ? ps.vals : nullptr;
  const GaussRec* rec = P > 0 ? fs.rec : nullptr;
  switch (sh_degree) {
    case 0: DGS_CUDA_OK(launch_colors<0>(nblocks, s, vertices, normals, glist, gvals, rec, features, out_rgb, st)); break;
    case 1: DGS_CUDA_OK(launch_colors<1>(nblocks, s, vertices, normals, glist, gvals, rec, features, out_rgb, st)); break;
    case 2: DGS_CUDA_OK(launch_colors<2>(nblocks, s, vertices, normals, glist, gvals, rec, features, out_rgb, st)); break;
    default: DGS_CUDA_OK(launch_colors<3>(nblocks, s, vertices, normals, glist, gvals, rec, features, out_rgb, st));
  }
  unsigned long long nw = 0;
  DGS_CUDA_OK(cudaMemcpyAsync(&nw, s.unweighted, sizeof(nw), cudaMemcpyDeviceToHost, st));
  DGS_CUDA_OK(cudaStreamSynchronize(st));  // the count of white vertices
  if (num_unweighted) *num_unweighted = (long long)nw;
  return DGS_OK;
}

}  // extern "C"
