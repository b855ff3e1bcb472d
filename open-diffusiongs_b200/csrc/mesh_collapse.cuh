// mesh_collapse.cuh -- what mesh_decimate.cu and mesh_remesh.cu share to collapse edges in parallel rounds: the link
// condition, the fold-over test, and the two-hop minimum (m1, m2) that selects independent edges.  Both files are
// compiled with the same helpers, so a collapse test means the same thing in each.
#pragma once
#include "mesh_common.cuh"

namespace dgs {
namespace {

struct Edge {
  int a, b;  // a < b
  int c, d;  // the apexes of its two faces; -1 unless it has exactly two
};

// Moving v to p keeps the orientation of every face around v that does not contain `other` (those die): its normal
// after the move has a positive dot product with its normal before.  Faces with zero area before are exempt.
__device__ bool keeps_orientation(int v, int other, double3 p, const float* __restrict__ pos,
                                  const int3* __restrict__ faces, const uint2* __restrict__ vrange,
                                  const uint32_t* __restrict__ vfaces) {
  const uint2 r = vrange[v];
  for (uint32_t i = r.x; i < r.y; i++) {
    const int3 f = faces[vfaces[i]];
    if (has(f, other)) continue;
    double3 p0 = load(pos, f.x), p1 = load(pos, f.y), p2 = load(pos, f.z);
    const double3 n0 = cross(sub(p1, p0), sub(p2, p0));
    if (n0.x == 0.0 && n0.y == 0.0 && n0.z == 0.0) continue;
    if (f.x == v) p0 = p; else if (f.y == v) p1 = p; else p2 = p;
    if (!(dot(n0, cross(sub(p1, p0), sub(p2, p0))) > 0.0)) return false;
  }
  return true;
}

// The link condition of edge (a, b) with apexes c, d: no common neighbour besides c and d, and not both of the faces
// (a, c, d) and (b, c, d) (the tetrahedron, which the collapse would fold onto itself).
__device__ bool link_ok(Edge e, const int3* __restrict__ faces, const uint2* __restrict__ vrange,
                        const uint32_t* __restrict__ vfaces) {
  if (e.c == e.d) return false;
  const uint2 ra = vrange[e.a], rb = vrange[e.b];
  bool acd = false, bcd = false;
  for (uint32_t i = ra.x; i < ra.y; i++) {
    const int3 f = faces[vfaces[i]];
    if (has(f, e.c) && has(f, e.d) && !has(f, e.b)) acd = true;
    for (int k = 0; k < 3; k++) {
      const int x = corner(f, k);
      if (x == e.a || x == e.b || x == e.c || x == e.d) continue;
      for (uint32_t j = rb.x; j < rb.y; j++)
        if (has(faces[vfaces[j]], x)) return false;
    }
  }
  for (uint32_t j = rb.x; j < rb.y; j++) {
    const int3 g = faces[vfaces[j]];
    if (has(g, e.c) && has(g, e.d) && !has(g, e.a)) bcd = true;
  }
  return !(acd && bcd);
}

// m1[v] = the smallest key of v's edges (the two edges of each of v's faces that contain v)
__global__ void m1_kernel(int V, const int3* __restrict__ faces, const uint2* __restrict__ vrange,
                          const uint32_t* __restrict__ vfaces, const uint32_t* __restrict__ edge_of,
                          const unsigned long long* __restrict__ ekey, unsigned long long* __restrict__ m1) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  unsigned long long m = kNoKey;
  const uint2 r = vrange[v];
  for (uint32_t i = r.x; i < r.y; i++) {
    const uint32_t f = vfaces[i];
    const int3 t = faces[f];
    const int k = t.x == v ? 0 : t.y == v ? 1 : 2;
    m = min(m, min(ekey[edge_of[3 * f + k]], ekey[edge_of[3 * f + (k + 2) % 3]]));
  }
  m1[v] = m;
}

// m2[v] = the smallest m1 over v and its neighbours (the vertices of its faces)
__global__ void m2_kernel(int V, const int3* __restrict__ faces, const uint2* __restrict__ vrange,
                          const uint32_t* __restrict__ vfaces, const unsigned long long* __restrict__ m1,
                          unsigned long long* __restrict__ m2) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  unsigned long long m = m1[v];
  const uint2 r = vrange[v];
  for (uint32_t i = r.x; i < r.y; i++) {
    const int3 t = faces[vfaces[i]];
    m = min(m, min(m1[t.x], min(m1[t.y], m1[t.z])));
  }
  m2[v] = m;
}

}  // namespace
}  // namespace dgs
