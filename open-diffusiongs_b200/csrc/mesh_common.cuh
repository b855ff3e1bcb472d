// mesh_common.cuh -- what the mesh passes (mesh_decimate.cu, mesh_clean.cu, mesh_remesh.cu) share over a face list
// int3 [F]: the entry points' argument checks and output contract, the face check, half-edges sorted into unique
// undirected edges, the vertex -> face incidence lists, the removal of dead faces, and the finish that keeps the
// referenced vertices.  Everything here is instantiated in each file that includes it, so its floating-point code is
// compiled with that file's flags (mesh_clean.cu and mesh_remesh.cu use -fmad=false).
#pragma once
#include <cub/cub.cuh>

#include <algorithm>
#include <cstring>

#include "dgs_internal.h"
#include "sorted_ranges.cuh"

namespace dgs {
namespace {

constexpr int kThreads = 256;
constexpr unsigned long long kNoKey = ~0ull;
constexpr unsigned kFull = 0xffffffffu;

// The bits of a vertex index below V (at least 1): the width of the radix sorts keyed by vertex.
inline int bits_for(int V) {
  int b = 1;
  while (b < 31 && (1LL << b) < V) b++;
  return b;
}

// Order-preserving uint key of a float, and back (the host reads boxes too).
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

__device__ __forceinline__ double3 sub(double3 u, double3 v) { return make_double3(u.x - v.x, u.y - v.y, u.z - v.z); }
__device__ __forceinline__ double dot(double3 u, double3 v) { return u.x * v.x + u.y * v.y + u.z * v.z; }
__device__ __forceinline__ double3 cross(double3 u, double3 v) {
  return make_double3(u.y * v.z - u.z * v.y, u.z * v.x - u.x * v.z, u.x * v.y - u.y * v.x);
}
__device__ __forceinline__ double3 load(const float* __restrict__ pos, int v) {
  return make_double3(pos[3 * v], pos[3 * v + 1], pos[3 * v + 2]);
}
__device__ __forceinline__ double3 round_f32(double3 v) {
  return make_double3((double)(float)v.x, (double)(float)v.y, (double)(float)v.z);
}
__device__ __forceinline__ bool has(int3 f, int x) { return f.x == x || f.y == x || f.z == x; }
__device__ __forceinline__ int corner(int3 f, int k) { return k == 0 ? f.x : k == 1 ? f.y : f.z; }

// A box in order-preserving keys, grown one vertex at a time.
struct Box {
  unsigned lo[3] = {kFull, kFull, kFull}, hi[3] = {0u, 0u, 0u};
  __device__ void add(const float* __restrict__ pos, int v) {
    for (int k = 0; k < 3; k++) {
      const unsigned q = fkey(pos[3 * v + k]);
      lo[k] = min(lo[k], q);
      hi[k] = max(hi[k], q);
    }
  }
};

// --------------------------------------------------------------------------------------------------------- arguments
// Where an entry point puts its result: the allocator and the four outputs of include/dgs_b200.h.
struct MeshOut {
  dgs_alloc_fn alloc;
  void* alloc_user;
  float** vertices;
  int** faces;
  long long *num_vertices, *num_faces;

  void set(float* v, int* f, long long nv, long long nf) const {
    *vertices = v;
    *faces = f;
    *num_vertices = nv;
    *num_faces = nf;
  }
  // One scratch allocation of `bytes`; nullptr (with the error set) when it fails.
  void* scratch(const char* name, size_t bytes) const {
    void* buf = alloc(bytes, alloc_user);
    if (!buf) set_error("%s: scratch allocation failed (%zu bytes)", name, bytes);
    return buf;
  }
};

// The checks of an input mesh, in this order; size_ok is the pass's own size limit, described by `limit`.
inline int check_mesh_input(const char* name, const float* vertices, long long V, const int* faces, long long F,
                            bool size_ok, const char* limit) {
  DGS_REQUIRE(V >= 0 && F >= 0, "%s: negative size (%lld vertices, %lld faces)", name, V, F);
  DGS_REQUIRE(size_ok, "%s: %lld vertices / %lld faces is too many (%s)", name, V, F, limit);
  DGS_REQUIRE((V == 0 || vertices) && (F == 0 || faces), "%s: vertices and faces must not be NULL", name);
  return DGS_OK;
}

// The checks every mesh entry point that returns a mesh makes, in this order, before its own and before any CUDA call.
inline int check_mesh_args(const char* name, const float* vertices, long long V, const int* faces, long long F,
                           bool size_ok, const char* limit, const MeshOut& out) {
  DGS_REQUIRE(out.alloc && out.vertices && out.faces && out.num_vertices && out.num_faces,
              "%s: alloc and the four outputs must not be NULL", name);
  return check_mesh_input(name, vertices, V, faces, F, size_ok, limit);
}

// -------------------------------------------------------------------------------------------------------- face check
// The smallest bad face (kNoKey if none) and the order-preserving keys of the box of the vertices the good faces
// reference: min x y z, max x y z.
struct FaceCheck {
  unsigned long long bad_face;
  unsigned box[6];
};

// A face is bad when an index is outside [0, V) or, with reject_repeated, repeated.  With used, the vertices of the
// faces with indices in range are marked.  The box is warp-reduced before its atomics.
__global__ void validate_kernel(int F, int V, const int3* __restrict__ faces, const float* __restrict__ pos,
                                bool reject_repeated, FaceCheck* __restrict__ chk, uint32_t* __restrict__ used) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  Box b;
  if (f < F) {
    const int3 t = faces[f];
    const bool in_range = t.x >= 0 && t.x < V && t.y >= 0 && t.y < V && t.z >= 0 && t.z < V;
    if (!in_range || (reject_repeated && (t.x == t.y || t.y == t.z || t.x == t.z))) {
      atomicMin(&chk->bad_face, (unsigned long long)f);
    } else {
      b.add(pos, t.x); b.add(pos, t.y); b.add(pos, t.z);
    }
    if (used && in_range) used[t.x] = used[t.y] = used[t.z] = 1;
  }
  for (int k = 0; k < 3; k++) {
    b.lo[k] = __reduce_min_sync(kFull, b.lo[k]);
    b.hi[k] = __reduce_max_sync(kFull, b.hi[k]);
  }
  if ((threadIdx.x & 31) == 0)
    for (int k = 0; k < 3; k++) {
      atomicMin(&chk->box[k], b.lo[k]);
      atomicMax(&chk->box[3 + k], b.hi[k]);
    }
}

// Checks every face on the device (validate_kernel; used, when given, is zeroed first) and reads the result into h
// with one synchronise.  A bad face is DGS_ERR_INVALID_ARGUMENT naming it.
inline int check_faces(const char* name, const float* vertices, int V, const int3* faces, int F, bool reject_repeated,
                       uint32_t* used, FaceCheck* chk, FaceCheck& h, cudaStream_t st) {
  DGS_CUDA_OK(cudaMemsetAsync(chk, 0xff, sizeof(FaceCheck), st));
  DGS_CUDA_OK(cudaMemsetAsync(chk->box + 3, 0, 3 * sizeof(unsigned), st));
  if (used) DGS_CUDA_OK(cudaMemsetAsync(used, 0, (size_t)V * sizeof(uint32_t), st));
  if (F > 0) {
    validate_kernel<<<ceil_div(F, kThreads), kThreads, 0, st>>>(F, V, faces, vertices, reject_repeated, chk, used);
    DGS_POST_LAUNCH();
  }
  DGS_CUDA_OK(cudaMemcpyAsync(&h, chk, sizeof(h), cudaMemcpyDeviceToHost, st));
  DGS_CUDA_OK(cudaStreamSynchronize(st));  // indices must be valid before any kernel follows them
  if (h.bad_face == kNoKey) return DGS_OK;
  int t[3] = {0, 0, 0};
  DGS_CUDA_OK(cudaMemcpyAsync(t, faces + h.bad_face, sizeof(t), cudaMemcpyDeviceToHost, st));
  DGS_CUDA_OK(cudaStreamSynchronize(st));
  set_error("%s: face %llu = (%d, %d, %d) has an index outside [0, %d)%s", name, h.bad_face, t[0], t[1], t[2], V,
            reject_repeated ? " or a repeated index" : "");
  return DGS_ERR_INVALID_ARGUMENT;
}

// The input returned as it is, for a pass with nothing to do: the faces are checked (no repeated index) with a
// scratch of one FaceCheck, then copied with the vertices into a new output.
inline int copy_unchanged(const char* name, const float* vertices, int V, const int* faces, int F, const MeshOut& out,
                          cudaStream_t st) {
  FaceCheck* chk = reinterpret_cast<FaceCheck*>(out.scratch(name, sizeof(FaceCheck)));
  if (!chk) return DGS_ERR_ALLOC;
  FaceCheck h;
  const int rc = check_faces(name, vertices, V, reinterpret_cast<const int3*>(faces), F, true, nullptr, chk, h, st);
  if (rc != DGS_OK) return rc;
  float* v = V ? reinterpret_cast<float*>(out.alloc(3 * (size_t)V * sizeof(float), out.alloc_user)) : nullptr;
  int* f = F ? reinterpret_cast<int*>(out.alloc(3 * (size_t)F * sizeof(int), out.alloc_user)) : nullptr;
  if ((V && !v) || (F && !f)) { set_error("%s: output allocation failed", name); return DGS_ERR_ALLOC; }
  if (V) DGS_CUDA_OK(cudaMemcpyAsync(v, vertices, 3 * (size_t)V * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (F) DGS_CUDA_OK(cudaMemcpyAsync(f, faces, 3 * (size_t)F * sizeof(int), cudaMemcpyDeviceToDevice, st));
  out.set(v, f, V, F);
  return DGS_OK;
}

// ------------------------------------------------------------------------------------------------------ connectivity
// (vertex, face) incidences in face order; a stable sort by vertex makes each vertex's faces one run in face order
__global__ void incidence_kernel(int n, const int3* __restrict__ faces, uint32_t* __restrict__ keys,
                                 uint32_t* __restrict__ vals) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= n) return;
  keys[h] = (uint32_t)corner(faces[h / 3], h % 3);
  vals[h] = (uint32_t)(h / 3);
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

// Faces re-indexed through `to` (to[v] >= 0 renames v); a face that now repeats a vertex is not alive.
__global__ void remap_kernel(int F, int3* __restrict__ faces, const int* __restrict__ to, uint8_t* __restrict__ alive) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  int3 t = faces[f];
  if (to[t.x] >= 0) t.x = to[t.x];
  if (to[t.y] >= 0) t.y = to[t.y];
  if (to[t.z] >= 0) t.z = to[t.z];
  faces[f] = t;
  alive[f] = t.x != t.y && t.y != t.z && t.x != t.z;
}

// ---------------------------------------------------------------------------------------------------------- finish
__global__ void used_kernel(int n, const int* __restrict__ fv, uint32_t* __restrict__ used) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < n) used[fv[c]] = 1;
}

// Vertex i < NV goes to vscan[i] - 1 when used (a vertex i >= V is a copy of src[i - V]); faces are renumbered.
__global__ void emit_kernel(int V, int NV, int F, const float* __restrict__ pos, const int* __restrict__ src,
                            const int3* __restrict__ faces, const uint32_t* __restrict__ used,
                            const uint32_t* __restrict__ vscan, float* __restrict__ out_v, int3* __restrict__ out_f) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < NV && used[i]) {
    const uint32_t o = vscan[i] - 1;
    const int s = i < V ? i : src[i - V];
    out_v[3 * o] = pos[3 * s];
    out_v[3 * o + 1] = pos[3 * s + 1];
    out_v[3 * o + 2] = pos[3 * s + 2];
  }
  if (i < F) {
    const int3 t = faces[i];
    out_f[i] = make_int3((int)vscan[t.x] - 1, (int)vscan[t.y] - 1, (int)vscan[t.z] - 1);
  }
}

// The buffers of the connectivity passes and the finish, for V vertices (NV used / vscan entries: the finish may see
// vertex copies) and F faces, n = 3F half-edges.  Each pass's Scratch derives from it, carves its own buffers after
// carve_mesh and adds what its own cub calls need (need) before carve_temp.
struct MeshScratch {
  int3 *faces, *faces_alt;
  uint8_t* keep;  // per face: kept by the next compact
  unsigned long long *hkey_in, *hkey;
  uint32_t *hval_in, *hval, *heads, *edge_of, *ikey_in, *ikey, *ival_in, *vfaces, *used, *vscan;
  uint2* vrange;
  void* temp;
  size_t temp_bytes;

  void carve_mesh(Carver& cv, int V, int F, int NV) {
    const int n = 3 * F, vbits = bits_for(V);
    faces = cv.take<int3>(F);
    faces_alt = cv.take<int3>(F);
    keep = cv.take<uint8_t>(F);
    hkey_in = cv.take<unsigned long long>(n);
    hkey = cv.take<unsigned long long>(n);
    hval_in = cv.take<uint32_t>(n);
    hval = cv.take<uint32_t>(n);
    heads = cv.take<uint32_t>(n);
    edge_of = cv.take<uint32_t>(n);
    ikey_in = cv.take<uint32_t>(n);
    ikey = cv.take<uint32_t>(n);
    ival_in = cv.take<uint32_t>(n);
    vfaces = cv.take<uint32_t>(n);
    used = cv.take<uint32_t>(NV);
    vscan = cv.take<uint32_t>(NV);
    vrange = cv.take<uint2>(V);
    temp_bytes = 0;
    size_t t = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, t, hkey_in, hkey, hval_in, hval, n, 0, 2 * vbits);
    need(t);
    cub::DeviceRadixSort::SortPairs(nullptr, t, ikey_in, ikey, ival_in, vfaces, n, 0, vbits);
    need(t);
    cub::DeviceScan::InclusiveSum(nullptr, t, heads, heads, std::max(n, NV));
    need(t);
    cub::DeviceSelect::Flagged(nullptr, t, faces, keep, faces_alt, static_cast<int*>(nullptr), F);
    need(t);
  }
  void need(size_t t) { temp_bytes = std::max(temp_bytes, t); }
  void carve_temp(Carver& cv) { temp = cv.take<char>(temp_bytes); }

  // The 3F half-edges of the first F faces over V vertices sorted by undirected edge: hkey[i] / hval[i] (half-edge
  // ids) in (min, max) order, in half-edge order within an edge; heads[i] = 1 + the edge id of sorted half-edge i
  // (edges numbered in key order).
  cudaError_t sort_edges(int F, int V, cudaStream_t st) {
    const int n = 3 * F, g = ceil_div(n, kThreads), vbits = bits_for(V);
    halfedge_kernel<<<g, kThreads, 0, st>>>(n, faces, vbits, hkey_in, hval_in);
    g_kernel_launches++;
    cudaError_t e =
        cub::DeviceRadixSort::SortPairs(temp, temp_bytes, hkey_in, hkey, hval_in, hval, n, 0, 2 * vbits, st);
    if (e != cudaSuccess) return e;
    edge_heads_kernel<<<g, kThreads, 0, st>>>(n, hkey, heads);
    g_kernel_launches++;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    return cub::DeviceScan::InclusiveSum(temp, temp_bytes, heads, heads, n, st);
  }

  // The vertex -> face lists of the first F faces over V vertices: vfaces[vrange[v].x, vrange[v].y) in face order,
  // with the vertex of sorted incidence i in ikey[i].
  cudaError_t vertex_faces(int F, int V, cudaStream_t st) {
    const int n = 3 * F;
    incidence_kernel<<<ceil_div(n, kThreads), kThreads, 0, st>>>(n, faces, ikey_in, ival_in);
    g_kernel_launches++;
    cudaError_t e =
        cub::DeviceRadixSort::SortPairs(temp, temp_bytes, ikey_in, ikey, ival_in, vfaces, n, 0, bits_for(V), st);
    if (e != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(vrange, 0, (size_t)V * sizeof(uint2), st)) != cudaSuccess) return e;
    ranges_kernel<<<ceil_div(n, kThreads), kThreads, 0, st>>>(n, ikey, vrange);
    g_kernel_launches++;
    return cudaGetLastError();
  }

  // Keeps the first F faces flagged in keep, in face order, as the faces; their number goes to *count on the device
  // (the caller reads it back at its next synchronise).
  cudaError_t compact(int F, int* count, cudaStream_t st) {
    const cudaError_t e = cub::DeviceSelect::Flagged(temp, temp_bytes, faces, keep, faces_alt, count, F, st);
    if (e == cudaSuccess) std::swap(faces, faces_alt);
    return e;
  }
};

// The finish of every pass: the vertices of [0, NV) that the F faces reference, in index order (pos for i < V, a copy
// of src[i - V] above), and the faces renumbered onto them.  Nothing is allocated when F == 0; otherwise the output's
// vertices, then its faces, after all scratch (dgs_b200.mesh reads them back in that order).  live, when given, is the
// device's own count of the faces, which must be F.
inline int emit_mesh(const char* name, MeshScratch& s, int V, int NV, int F, const float* pos, const int* src,
                     const int* live, const MeshOut& out, cudaStream_t st) {
  DGS_CUDA_OK(cudaMemsetAsync(s.used, 0, (size_t)NV * sizeof(uint32_t), st));
  if (F > 0) {
    used_kernel<<<ceil_div(3 * F, kThreads), kThreads, 0, st>>>(3 * F, reinterpret_cast<const int*>(s.faces), s.used);
    DGS_POST_LAUNCH();
  }
  DGS_CUDA_OK(cub::DeviceScan::InclusiveSum(s.temp, s.temp_bytes, s.used, s.vscan, NV, st));
  uint32_t nv = 0;
  int dev_live = F;
  DGS_CUDA_OK(cudaMemcpyAsync(&nv, s.vscan + NV - 1, sizeof(nv), cudaMemcpyDeviceToHost, st));
  if (live) DGS_CUDA_OK(cudaMemcpyAsync(&dev_live, live, sizeof(int), cudaMemcpyDeviceToHost, st));
  DGS_CUDA_OK(cudaStreamSynchronize(st));  // the vertex count sizes the output
  if (dev_live != F) {
    set_error("%s: internal error, %d live faces where %d were expected", name, dev_live, F);
    return DGS_ERR_CUDA;
  }
  if (F == 0) return DGS_OK;
  float* v = reinterpret_cast<float*>(out.alloc((size_t)nv * 3 * sizeof(float), out.alloc_user));
  int* f = reinterpret_cast<int*>(out.alloc((size_t)F * 3 * sizeof(int), out.alloc_user));
  if (!v || !f) { set_error("%s: output allocation failed", name); return DGS_ERR_ALLOC; }
  emit_kernel<<<ceil_div(std::max(NV, F), kThreads), kThreads, 0, st>>>(V, NV, F, pos, src, s.faces, s.used, s.vscan,
                                                                          v, reinterpret_cast<int3*>(f));
  DGS_POST_LAUNCH();
  out.set(v, f, nv, F);
  return DGS_OK;
}

}  // namespace
}  // namespace dgs
