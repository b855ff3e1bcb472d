// mesh_edges.cuh -- the connectivity passes mesh_decimate.cu and mesh_clean.cu share over a face list int3 [F]:
// half-edges sorted into unique undirected edges, and the vertex -> face incidence lists.
#pragma once
#include <cub/cub.cuh>

#include "dgs_internal.h"

namespace dgs {
namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ int corner(int3 f, int k) { return k == 0 ? f.x : k == 1 ? f.y : f.z; }

// (vertex, face) incidences in face order; a stable sort by vertex makes each vertex's faces one run in face order
__global__ void incidence_kernel(int n, const int3* __restrict__ faces, uint32_t* __restrict__ keys,
                                 uint32_t* __restrict__ vals) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= n) return;
  keys[h] = (uint32_t)corner(faces[h / 3], h % 3);
  vals[h] = (uint32_t)(h / 3);
}

__global__ void ranges_kernel(int n, const uint32_t* __restrict__ keys, uint2* __restrict__ ranges) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t k = keys[i];
  if (i == 0 || keys[i - 1] != k) ranges[k].x = i;
  if (i == n - 1 || keys[i + 1] != k) ranges[k].y = i + 1;
}

// half-edge h = 3 f + k runs from corner k to corner k + 1 of face f; its key is (min, max) of the two
__global__ void halfedge_kernel(int n, const int3* __restrict__ faces, int vbits, unsigned long long* __restrict__ keys,
                                uint32_t* __restrict__ vals) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= n) return;
  const int3 f = faces[h / 3];
  const int u = corner(f, h % 3), w = corner(f, (h % 3 + 1) % 3);
  keys[h] = ((unsigned long long)min(u, w) << vbits) | (unsigned long long)max(u, w);
  vals[h] = (uint32_t)h;
}

__global__ void edge_heads_kernel(int n, const unsigned long long* __restrict__ keys, uint32_t* __restrict__ heads) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  heads[i] = i == 0 || keys[i] != keys[i - 1];
}

// The n = 3F half-edges of faces sorted by undirected edge: keys[i] / vals[i] (half-edge ids) in (min, max) order, in
// half-edge order within an edge; scan[i] = 1 + the edge id of sorted half-edge i (edges numbered in key order).
// keys_in / vals_in are overwritten; temp must hold SortPairs(n, 2 vbits bits) and InclusiveSum(n).
inline cudaError_t sort_edges(int n, const int3* faces, int vbits, unsigned long long* keys_in,
                              unsigned long long* keys, uint32_t* vals_in, uint32_t* vals, uint32_t* scan, void* temp,
                              size_t temp_bytes, cudaStream_t st) {
  const int g = ceil_div(n, kThreads);
  halfedge_kernel<<<g, kThreads, 0, st>>>(n, faces, vbits, keys_in, vals_in);
  g_kernel_launches++;
  cudaError_t e = cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys_in, keys, vals_in, vals, n, 0, 2 * vbits, st);
  if (e != cudaSuccess) return e;
  edge_heads_kernel<<<g, kThreads, 0, st>>>(n, keys, scan);
  g_kernel_launches++;
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  return cub::DeviceScan::InclusiveSum(temp, temp_bytes, scan, scan, n, st);
}

// The vertex -> face lists of F faces over V vertices: vfaces[vrange[v].x, vrange[v].y) in face order, with the
// vertex of sorted incidence i in ikey[i].  ikey_in / ival_in are overwritten; temp must hold SortPairs(3F, vbits bits).
inline cudaError_t vertex_faces(int F, int V, const int3* faces, int vbits, uint32_t* ikey_in, uint32_t* ikey,
                                uint32_t* ival_in, uint32_t* vfaces, uint2* vrange, void* temp, size_t temp_bytes,
                                cudaStream_t st) {
  const int n = 3 * F;
  incidence_kernel<<<ceil_div(n, kThreads), kThreads, 0, st>>>(n, faces, ikey_in, ival_in);
  g_kernel_launches++;
  cudaError_t e = cub::DeviceRadixSort::SortPairs(temp, temp_bytes, ikey_in, ikey, ival_in, vfaces, n, 0, vbits, st);
  if (e != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(vrange, 0, (size_t)V * sizeof(uint2), st)) != cudaSuccess) return e;
  ranges_kernel<<<ceil_div(n, kThreads), kThreads, 0, st>>>(n, ikey, vrange);
  g_kernel_launches++;
  return cudaGetLastError();
}

}  // namespace
}  // namespace dgs
