// mesh_remesh.cu -- isotropic remeshing of a welded triangle mesh towards a target edge length L: VCG's
// IsotropicRemeshing as pymeshlab's meshing_isotropic_explicit_remeshing runs it inside the reference's clean_mesh
// (utils/mesh_utils.py:88-147, remesh=True), as the exact contract of include/dgs_b200.h (dgs_mesh_remesh) that
// oracle/mesh_remesh.py restates serially.  Every decision and every new position is computed in fp64 from the fp32
// positions; this file is compiled with -fmad=false, so each product and sum is rounded on its own, as in the oracle.
// The only atomics are integer ones whose result does not depend on their order (min of keys, counts, flags), so the
// output is the same bits on every run.
//
// Per iteration: the edges (mesh_common.cuh sort_edges) give the locks; split (one pass, one read-back for the counts;
// scratch grows here when the mesh outgrows it); collapse rounds (the key / m1 / m2 selection of mesh_decimate.cu
// through mesh_collapse.cuh, one read-back per round); flip rounds (each vertex keeps the smallest (-gain, edge) key of
// the candidates that touch it, one read-back per round); one Jacobi pass of tangential smoothing; reprojection onto the
// input surface through a uniform grid of its triangle boxes (cell -> triangle pairs radix-sorted once per call).
// Collapse and flip stages stop after kRoundCap rounds each; that is reported in the stats, never an error.
#include <cmath>

#include "mesh_collapse.cuh"

namespace dgs {
namespace {

constexpr int kRoundCap = 256;        // rounds per collapse / flip stage and iteration
constexpr int kMaxCells = 1024;       // grid cells per axis (10 bits of the cell key each)

struct Counters {
  FaceCheck chk;
  int num_edges, selected, num_faces;
};

// An undirected edge (a < b) of the current faces; h0 < h1 are its first two half-edges (3 f + k runs from corner k
// to k + 1), c and d the apexes of their faces.  blocked: not exactly two faces running it in opposite directions
// (boundary, non-manifold) or a feature edge; such an edge is never collapsed or flipped and locks its ends.
struct REdge {
  int a, b, c, d, h0, h1, nf, blocked;
};

// The input surface S and its grid: triangle t is listed in every cell its box touches, (cell key, t) sorted by key.
struct Surface {
  const float* pos;
  const int3* faces;
  const uint32_t* keys;
  const uint32_t* tris;
  int npairs;
  double mn[3], h;
  int n[3];
};

__device__ __forceinline__ double3 add(double3 u, double3 v) { return make_double3(u.x + v.x, u.y + v.y, u.z + v.z); }
__device__ __forceinline__ double3 scale(double s, double3 v) { return make_double3(s * v.x, s * v.y, s * v.z); }
__device__ __forceinline__ double dist(double3 p, double3 q) { return sqrt(dot(sub(q, p), sub(q, p))); }
__device__ __forceinline__ double3 normal(double3 p0, double3 p1, double3 p2) { return cross(sub(p1, p0), sub(p2, p0)); }
__device__ __forceinline__ double3 face_normal(const float* __restrict__ pos, int3 f) {
  return normal(load(pos, f.x), load(pos, f.y), load(pos, f.z));
}
__device__ __forceinline__ void store(float* __restrict__ pos, int v, double3 p) {
  pos[3 * v] = (float)p.x;
  pos[3 * v + 1] = (float)p.y;
  pos[3 * v + 2] = (float)p.z;
}
__device__ __forceinline__ double comp(double3 v, int k) { return k == 0 ? v.x : k == 1 ? v.y : v.z; }

// Ericson's ClosestPtPointTriangle (Real-Time Collision Detection, 5.1.5), regions in the book's order.
__device__ double3 closest_on_triangle(double3 p, double3 a, double3 b, double3 c) {
  const double3 ab = sub(b, a), ac = sub(c, a), ap = sub(p, a);
  const double d1 = dot(ab, ap), d2 = dot(ac, ap);
  if (d1 <= 0.0 && d2 <= 0.0) return a;
  const double3 bp = sub(p, b);
  const double d3 = dot(ab, bp), d4 = dot(ac, bp);
  if (d3 >= 0.0 && d4 <= d3) return b;
  const double vc = d1 * d4 - d3 * d2;
  if (vc <= 0.0 && d1 >= 0.0 && d3 <= 0.0) return add(a, scale(d1 / (d1 - d3), ab));
  const double3 cp = sub(p, c);
  const double d5 = dot(ab, cp), d6 = dot(ac, cp);
  if (d6 >= 0.0 && d5 <= d6) return c;
  const double vb = d5 * d2 - d1 * d6;
  if (vb <= 0.0 && d2 >= 0.0 && d6 <= 0.0) return add(a, scale(d2 / (d2 - d6), ac));
  const double va = d3 * d6 - d5 * d4;
  const double e43 = d4 - d3, e56 = d5 - d6;
  if (va <= 0.0 && e43 >= 0.0 && e56 >= 0.0) return add(b, scale(e43 / (e43 + e56), sub(c, b)));
  const double denom = 1.0 / (va + vb + vc);
  return add(add(a, scale(vb * denom, ab)), scale(vc * denom, ac));
}

// The closest point of S to p: the smallest (squared distance, face) over S.  Rings of cells around p's cell are
// searched outwards until the best distance is below the distance from p to the unsearched cells (less a margin that
// covers the rounding of cell indices), or the rings cover the grid.  *d2_out receives the squared distance and
// *face_out (when given) the face.
__device__ double3 closest(const Surface& S, double3 p, double* d2_out, int* face_out = nullptr) {
  int c[3];
  for (int k = 0; k < 3; k++) {
    const double x = floor((comp(p, k) - S.mn[k]) / S.h);
    c[k] = (int)fmin(fmax(x, 0.0), (double)(S.n[k] - 1));
  }
  double best = INFINITY;
  int bestf = 0x7fffffff;
  double3 bq = p;
  const double tol = 1e-6 * S.h;
  for (int r = 0;; r++) {
    for (int dx = -r; dx <= r; dx++) {
      const int x = c[0] + dx;
      if (x < 0 || x >= S.n[0]) continue;
      for (int dy = -r; dy <= r; dy++) {
        const int y = c[1] + dy;
        if (y < 0 || y >= S.n[1]) continue;
        const int step = (abs(dx) == r || abs(dy) == r) ? 1 : max(2 * r, 1);
        for (int dz = -r; dz <= r; dz += step) {
          const int z = c[2] + dz;
          if (z < 0 || z >= S.n[2]) continue;
          const uint32_t key = ((uint32_t)x << 20) | ((uint32_t)y << 10) | (uint32_t)z;
          int lo = 0, hi = S.npairs;  // lower bound of key
          while (lo < hi) {
            const int m = (lo + hi) >> 1;
            if (S.keys[m] < key) lo = m + 1; else hi = m;
          }
          for (int j = lo; j < S.npairs && S.keys[j] == key; j++) {
            const int t = (int)S.tris[j];
            const int3 f = S.faces[t];
            const double3 q = closest_on_triangle(p, load(S.pos, f.x), load(S.pos, f.y), load(S.pos, f.z));
            const double3 dq = sub(p, q);
            const double d2 = dot(dq, dq);
            if (d2 < best || (d2 == best && t < bestf)) { best = d2; bestf = t; bq = q; }
          }
        }
      }
    }
    bool covered = true;
    double dmin = INFINITY;
    for (int k = 0; k < 3; k++) {
      if (c[k] - r > 0) { covered = false; dmin = fmin(dmin, comp(p, k) - (S.mn[k] + (c[k] - r) * S.h)); }
      if (c[k] + r < S.n[k] - 1) { covered = false; dmin = fmin(dmin, S.mn[k] + (c[k] + r + 1) * S.h - comp(p, k)); }
    }
    if (covered || (bestf != 0x7fffffff && sqrt(best) + tol < dmin)) break;
  }
  *d2_out = best;
  if (face_out) *face_out = bestf;
  return bq;
}

__device__ __forceinline__ bool near_surface(const Surface& S, double3 p, double max_dist) {
  double d2;
  closest(S, p, &d2);
  return !(sqrt(d2) > max_dist);
}

// ---------------------------------------------------------------------------------------------------------- setup
__device__ __forceinline__ void cell_range(const Surface& S, const float* __restrict__ pos, int3 f, int* lo, int* hi) {
  for (int k = 0; k < 3; k++) {
    const double x0 = pos[3 * f.x + k], x1 = pos[3 * f.y + k], x2 = pos[3 * f.z + k];
    const double a = floor((fmin(x0, fmin(x1, x2)) - S.mn[k]) / S.h), b = floor((fmax(x0, fmax(x1, x2)) - S.mn[k]) / S.h);
    lo[k] = (int)fmin(fmax(a, 0.0), (double)(S.n[k] - 1));
    hi[k] = (int)fmin(fmax(b, 0.0), (double)(S.n[k] - 1));
  }
}
__global__ void grid_count_kernel(int F, Surface S, unsigned long long* __restrict__ cnt) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  int lo[3], hi[3];
  cell_range(S, S.pos, S.faces[f], lo, hi);
  cnt[f] = (unsigned long long)(hi[0] - lo[0] + 1) * (hi[1] - lo[1] + 1) * (hi[2] - lo[2] + 1);
}
__global__ void grid_fill_kernel(int F, Surface S, const unsigned long long* __restrict__ cnt,
                                 const unsigned long long* __restrict__ scan, uint32_t* __restrict__ keys,
                                 uint32_t* __restrict__ tris) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  int lo[3], hi[3];
  cell_range(S, S.pos, S.faces[f], lo, hi);
  unsigned long long o = scan[f] - cnt[f];
  for (int x = lo[0]; x <= hi[0]; x++)
    for (int y = lo[1]; y <= hi[1]; y++)
      for (int z = lo[2]; z <= hi[2]; z++, o++) {
        keys[o] = ((uint32_t)x << 20) | ((uint32_t)y << 10) | (uint32_t)z;
        tris[o] = (uint32_t)f;
      }
}

// ---------------------------------------------------------------------------------------------------------- edges
// One thread per sorted half-edge: its edge id; the run's first thread writes the edge (and, with lock, the locks).
__global__ void edge_kernel(int n, const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ vals,
                            const uint32_t* __restrict__ scan, const int3* __restrict__ faces,
                            const float* __restrict__ pos, int vbits, double cos_t, REdge* __restrict__ edges,
                            uint32_t* __restrict__ edge_of, uint8_t* __restrict__ lock, Counters* __restrict__ ctr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t eid = scan[i] - 1;
  edge_of[vals[i]] = eid;
  if (i == n - 1) ctr->num_edges = (int)scan[i];
  const unsigned long long key = keys[i];
  if (i > 0 && keys[i - 1] == key) return;
  int j = i + 1;
  while (j < n && keys[j] == key) j++;
  REdge e;
  e.a = (int)(key >> vbits);
  e.b = (int)(key & ((1ull << vbits) - 1));
  e.nf = j - i;
  e.h0 = (int)vals[i];
  e.h1 = (int)vals[min(i + 1, n - 1)];
  const int3 f0 = faces[e.h0 / 3], f1 = faces[e.h1 / 3];
  e.c = corner(f0, (e.h0 % 3 + 2) % 3);
  e.d = corner(f1, (e.h1 % 3 + 2) % 3);
  bool blocked = !(e.nf == 2 && corner(f0, e.h0 % 3) == corner(f1, (e.h1 % 3 + 1) % 3));
  if (!blocked) {
    const double3 n0 = face_normal(pos, f0), n1 = face_normal(pos, f1);
    blocked = dot(n0, n1) < cos_t * sqrt(dot(n0, n0)) * sqrt(dot(n1, n1));  // a feature edge
  }
  e.blocked = blocked;
  if (lock && blocked) lock[e.a] = lock[e.b] = 1;
  edges[eid] = e;
}

__device__ __forceinline__ double edge_length(const float* __restrict__ pos, const REdge& e) {
  return dist(load(pos, e.a), load(pos, e.b));
}

// ---------------------------------------------------------------------------------------------------------- split
__global__ void split_flag_kernel(int n, const Counters* __restrict__ ctr, const REdge* __restrict__ edges,
                                  const float* __restrict__ pos, double hi, uint32_t* __restrict__ flag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  flag[i] = i < ctr->num_edges && edge_length(pos, edges[i]) > hi;
}
__global__ void split_count_kernel(int F, const uint32_t* __restrict__ edge_of, const uint32_t* __restrict__ flag,
                                   uint32_t* __restrict__ cnt) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  cnt[f] = flag[edge_of[3 * f]] + flag[edge_of[3 * f + 1]] + flag[edge_of[3 * f + 2]];
}
// Split edge i gets vertex V + (its rank among split edges) at its fp32 midpoint, locked iff the edge is blocked.
__global__ void split_vertex_kernel(int n, int V, const Counters* __restrict__ ctr, const REdge* __restrict__ edges,
                                    const uint32_t* __restrict__ flag, const uint32_t* __restrict__ rank,
                                    float* __restrict__ pos, uint8_t* __restrict__ lock) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || i >= ctr->num_edges || !flag[i]) return;
  const REdge e = edges[i];
  const int v = V + (int)rank[i] - 1;
  store(pos, v, scale(0.5, add(load(pos, e.a), load(pos, e.b))));
  lock[v] = (uint8_t)e.blocked;
}
// Face f (v0, v1, v2), with m_k the midpoint of edge k (corner k -> k + 1), is re-triangulated in place, its extra
// faces going to F + (extras of earlier faces).  One split (a, b) opposite c: (a, m, c), (m, b, c).  Two, with (c, a)
// not split: (m_ab, b, m_bc), then the quad (a, m_ab, m_bc, c) cut along its strictly shorter diagonal, (a, m_bc) on a
// tie.  Three: (v0, m0, m2), (m0, v1, m1), (m2, m1, v2), (m0, m1, m2).
__global__ void split_face_kernel(int F, int V, const uint32_t* __restrict__ edge_of, const uint32_t* __restrict__ flag,
                                  const uint32_t* __restrict__ rank, const uint32_t* __restrict__ cnt,
                                  const uint32_t* __restrict__ scan, const float* __restrict__ pos,
                                  int3* __restrict__ faces) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F || cnt[f] == 0) return;
  const int3 t = faces[f];
  int m[3];
  for (int k = 0; k < 3; k++) {
    const uint32_t e = edge_of[3 * f + k];
    m[k] = flag[e] ? V + (int)rank[e] - 1 : -1;
  }
  int3 out[4];
  const int n = (int)cnt[f];
  if (n == 1) {
    const int k = m[0] >= 0 ? 0 : m[1] >= 0 ? 1 : 2;
    const int a = corner(t, k), b = corner(t, (k + 1) % 3), c = corner(t, (k + 2) % 3);
    out[0] = make_int3(a, m[k], c);
    out[1] = make_int3(m[k], b, c);
  } else if (n == 2) {
    const int k = m[0] < 0 ? 0 : m[1] < 0 ? 1 : 2;
    const int c = corner(t, k), a = corner(t, (k + 1) % 3), b = corner(t, (k + 2) % 3);
    const int mab = m[(k + 1) % 3], mbc = m[(k + 2) % 3];
    out[0] = make_int3(mab, b, mbc);
    if (dist(load(pos, mab), load(pos, c)) < dist(load(pos, a), load(pos, mbc))) {
      out[1] = make_int3(a, mab, c);
      out[2] = make_int3(mab, mbc, c);
    } else {
      out[1] = make_int3(a, mab, mbc);
      out[2] = make_int3(a, mbc, c);
    }
  } else {
    out[0] = make_int3(t.x, m[0], m[2]);
    out[1] = make_int3(m[0], t.y, m[1]);
    out[2] = make_int3(m[2], m[1], t.z);
    out[3] = make_int3(m[0], m[1], m[2]);
  }
  faces[f] = out[0];
  const int o = F + (int)scan[f] - n;
  for (int j = 0; j < n; j++) faces[o + j] = out[1 + j];
}

// ---------------------------------------------------------------------------------------------------------- collapse
// Edge i is a candidate when it is not blocked, shorter than lo and not locked at both ends.  It moves both ends to
// the locked end, or to the fp32 midpoint.  Rejected when the link condition fails, a face around a or b flips, an
// edge longer than hi would appear, or the new position is farther than max_dist from S.
__global__ void collapse_cost_kernel(const Counters* __restrict__ ctr, const REdge* __restrict__ edges,
                                     const float* __restrict__ pos, const uint8_t* __restrict__ lock,
                                     const int3* __restrict__ faces, const uint2* __restrict__ vrange,
                                     const uint32_t* __restrict__ vfaces, double lo, double hi, double max_dist,
                                     Surface S, unsigned long long* __restrict__ ekey, float3* __restrict__ eplace) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ctr->num_edges) return;
  ekey[i] = kNoKey;
  const REdge e = edges[i];
  if (e.blocked || (lock[e.a] && lock[e.b])) return;
  const double3 pa = load(pos, e.a), pb = load(pos, e.b);
  const double len = dist(pa, pb);
  if (!(len < lo)) return;
  const double3 p = lock[e.a] ? pa : lock[e.b] ? pb : round_f32(scale(0.5, add(pa, pb)));
  Edge le;
  le.a = e.a; le.b = e.b; le.c = e.c; le.d = e.d;
  if (!link_ok(le, faces, vrange, vfaces)) return;
  if (!keeps_orientation(e.a, e.b, p, pos, faces, vrange, vfaces) ||
      !keeps_orientation(e.b, e.a, p, pos, faces, vrange, vfaces))
    return;
  for (int s = 0; s < 2; s++) {
    const uint2 r = vrange[s ? e.b : e.a];
    for (uint32_t j = r.x; j < r.y; j++) {
      const int3 t = faces[vfaces[j]];
      for (int k = 0; k < 3; k++) {
        const int x = corner(t, k);
        if (x != e.a && x != e.b && dist(p, load(pos, x)) > hi) return;
      }
    }
  }
  if (!near_surface(S, p, max_dist)) return;
  ekey[i] = ((unsigned long long)__float_as_uint((float)len) << 32) | (unsigned)i;
  eplace[i] = make_float3((float)p.x, (float)p.y, (float)p.z);
}

// Taken iff key == m2[a] == m2[b] (the independence argument of mesh_decimate.cu select_kernel): b retires into a,
// which moves to the new position and inherits b's lock.
__global__ void collapse_apply_kernel(Counters* __restrict__ ctr, const REdge* __restrict__ edges,
                                      const unsigned long long* __restrict__ ekey,
                                      const unsigned long long* __restrict__ m2, const float3* __restrict__ eplace,
                                      float* __restrict__ pos, uint8_t* __restrict__ lock, int* __restrict__ to) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ctr->num_edges) return;
  const unsigned long long key = ekey[i];
  const REdge e = edges[i];
  if (key == kNoKey || m2[e.a] != key || m2[e.b] != key) return;
  const float3 p = eplace[i];
  pos[3 * e.a] = p.x;
  pos[3 * e.a + 1] = p.y;
  pos[3 * e.a + 2] = p.z;
  lock[e.a] |= lock[e.b];
  to[e.b] = e.a;
  atomicAdd(&ctr->selected, 1);
}

// ---------------------------------------------------------------------------------------------------------- flip
__global__ void valence_kernel(const Counters* __restrict__ ctr, const REdge* __restrict__ edges, int* __restrict__ val,
                               uint8_t* __restrict__ bnd) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ctr->num_edges) return;
  const REdge e = edges[i];
  atomicAdd(&val[e.a], 1);
  atomicAdd(&val[e.b], 1);
  if (e.nf == 1) bnd[e.a] = bnd[e.b] = 1;
}

__device__ __forceinline__ int sq_dev(const int* __restrict__ val, const uint8_t* __restrict__ bnd, int x, int dv) {
  const int y = val[x] + dv - (bnd[x] ? 4 : 6);
  return y * y;
}

// Edge (a, b) with faces (u, w, c) and (w, u, d) becomes (c, d) when it is not blocked, (c, d) is not an edge yet,
// both new faces face the way both old ones do, the midpoint of (c, d) is within max_dist of S and the valence energy
// sum (valence - target)^2 over a, b, c, d drops.  Key (2^31 - 1 - gain) << 32 | edge; every end keeps the smallest.
__global__ void flip_cost_kernel(const Counters* __restrict__ ctr, const REdge* __restrict__ edges,
                                 const float* __restrict__ pos, const int3* __restrict__ faces,
                                 const uint2* __restrict__ vrange, const uint32_t* __restrict__ vfaces,
                                 const int* __restrict__ val, const uint8_t* __restrict__ bnd, double max_dist, Surface S,
                                 unsigned long long* __restrict__ ekey, unsigned long long* __restrict__ vmin) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ctr->num_edges) return;
  ekey[i] = kNoKey;
  const REdge e = edges[i];
  if (e.blocked || e.c == e.d) return;
  const uint2 r = vrange[e.c];
  for (uint32_t j = r.x; j < r.y; j++)
    if (has(faces[vfaces[j]], e.d)) return;
  const int gain = sq_dev(val, bnd, e.a, 0) + sq_dev(val, bnd, e.b, 0) + sq_dev(val, bnd, e.c, 0) +
                   sq_dev(val, bnd, e.d, 0) -
                   (sq_dev(val, bnd, e.a, -1) + sq_dev(val, bnd, e.b, -1) + sq_dev(val, bnd, e.c, 1) +
                    sq_dev(val, bnd, e.d, 1));
  if (gain <= 0) return;
  const int3 f0 = faces[e.h0 / 3], f1 = faces[e.h1 / 3];
  const int u = corner(f0, e.h0 % 3), w = corner(f0, (e.h0 % 3 + 1) % 3);
  const double3 n0 = face_normal(pos, f0), n1 = face_normal(pos, f1);
  const double3 pc = load(pos, e.c), pd = load(pos, e.d);
  const double3 m0 = normal(pc, load(pos, u), pd), m1 = normal(pd, load(pos, w), pc);
  if (!(dot(m0, n0) > 0.0 && dot(m0, n1) > 0.0 && dot(m1, n0) > 0.0 && dot(m1, n1) > 0.0)) return;
  if (!near_surface(S, scale(0.5, add(pc, pd)), max_dist)) return;
  const unsigned long long key = ((unsigned long long)(0x7fffffffu - (unsigned)gain) << 32) | (unsigned)i;
  ekey[i] = key;
  atomicMin(&vmin[e.a], key);
  atomicMin(&vmin[e.b], key);
  atomicMin(&vmin[e.c], key);
  atomicMin(&vmin[e.d], key);
}

// Taken iff the key is the smallest at all four vertices, so the flips of a round share no vertex.
__global__ void flip_apply_kernel(Counters* __restrict__ ctr, const REdge* __restrict__ edges,
                                  const unsigned long long* __restrict__ ekey,
                                  const unsigned long long* __restrict__ vmin, int3* __restrict__ faces) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ctr->num_edges) return;
  const unsigned long long key = ekey[i];
  const REdge e = edges[i];
  if (key == kNoKey || vmin[e.a] != key || vmin[e.b] != key || vmin[e.c] != key || vmin[e.d] != key) return;
  const int3 f0 = faces[e.h0 / 3];
  const int u = corner(f0, e.h0 % 3), w = corner(f0, (e.h0 % 3 + 1) % 3);
  faces[e.h0 / 3] = make_int3(e.c, u, e.d);
  faces[e.h1 / 3] = make_int3(e.d, w, e.c);
  atomicAdd(&ctr->selected, 1);
}

// ---------------------------------------------------------------------------------------------------------- smooth
// Jacobi: every free vertex reads the old positions.  c = the mean of the other two corners of its faces (each
// neighbour of a manifold vertex counted twice), n = the normalised sum of its faces' (p1 - p0) x (p2 - p0), both in
// face order; p + (d - (d . n) n) with d = c - p.
__global__ void smooth_kernel(int V, const float* __restrict__ pos, const int3* __restrict__ faces,
                              const uint2* __restrict__ vrange, const uint32_t* __restrict__ vfaces,
                              const uint8_t* __restrict__ lock, float* __restrict__ out) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const double3 p = load(pos, v);
  const uint2 r = vrange[v];
  double3 q = p;
  if (!lock[v] && r.y > r.x) {
    double3 s = make_double3(0.0, 0.0, 0.0), ns = s;
    for (uint32_t i = r.x; i < r.y; i++) {
      const int3 t = faces[vfaces[i]];
      const int k = t.x == v ? 0 : t.y == v ? 1 : 2;
      s = add(s, load(pos, corner(t, (k + 1) % 3)));
      s = add(s, load(pos, corner(t, (k + 2) % 3)));
      ns = add(ns, face_normal(pos, t));
    }
    const double nl = sqrt(dot(ns, ns));
    if (nl > 0.0) {
      const double m = 2.0 * (double)(r.y - r.x);
      const double3 c = make_double3(s.x / m, s.y / m, s.z / m), n = make_double3(ns.x / nl, ns.y / nl, ns.z / nl);
      const double3 d = sub(c, p);
      const double t = dot(d, n);
      q = add(p, sub(d, scale(t, n)));
    }
  }
  store(out, v, q);
}

__global__ void reproject_kernel(int V, float* __restrict__ pos, const uint2* __restrict__ vrange, Surface S) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const uint2 r = vrange[v];
  if (r.y == r.x) return;
  double d2;
  store(pos, v, closest(S, load(pos, v), &d2));
}

// The mesh being remeshed and the per-round scratch, sized for Vc vertices and Fc faces (n = 3 Fc half-edges, at
// most n edges).  A split that outgrows it gets a new one; the mesh is copied over.
struct Scratch : MeshScratch {
  int Vc = 0, Fc = 0;
  Counters* ctr;
  float *pos, *pos_alt;
  uint8_t *lock, *bnd;
  int *to, *val;
  unsigned long long *m1, *m2, *ekey;
  uint32_t *xcnt, *xscan, *eflag, *erank;
  REdge* edges;
  float3* eplace;

  size_t carve(void* base, int V, int F) {
    Vc = std::max(V, 1);
    Fc = std::max(F, 1);
    const int n = 3 * Fc;
    Carver cv(base);
    ctr = cv.take<Counters>(1);
    carve_mesh(cv, Vc, Fc, Vc);
    pos = cv.take<float>(3 * (size_t)Vc);
    pos_alt = cv.take<float>(3 * (size_t)Vc);
    lock = cv.take<uint8_t>(Vc);
    bnd = cv.take<uint8_t>(Vc);
    to = cv.take<int>(Vc);
    val = cv.take<int>(Vc);
    m1 = cv.take<unsigned long long>(Vc);
    m2 = cv.take<unsigned long long>(Vc);
    ekey = cv.take<unsigned long long>(n);
    xcnt = cv.take<uint32_t>(Fc);
    xscan = cv.take<uint32_t>(Fc);
    eflag = cv.take<uint32_t>(n);
    erank = cv.take<uint32_t>(n);
    edges = cv.take<REdge>(n);
    eplace = cv.take<float3>(n);
    size_t t = 0;
    cub::DeviceScan::InclusiveSum(nullptr, t, hkey_in, hkey, Fc);  // build_surface's scan of the grid counts
    need(t);
    carve_temp(cv);
    return cv.bytes();
  }
};

// Edges of the first F faces (and, with lock, the iteration's locks); then the vertex -> face lists when vf is set.
cudaError_t edge_pass(Scratch& s, int F, int V, double cos_t, uint8_t* lock, bool vf, cudaStream_t st) {
  const int n = 3 * F;
  cudaError_t e = s.sort_edges(F, V, st);
  if (e != cudaSuccess) return e;
  edge_kernel<<<ceil_div(n, kThreads), kThreads, 0, st>>>(n, s.hkey, s.hval, s.heads, s.faces, s.pos, bits_for(V),
                                                           cos_t, s.edges, s.edge_of, lock, s.ctr);
  g_kernel_launches++;
  if ((e = cudaGetLastError()) != cudaSuccess || !vf) return e;
  return s.vertex_faces(F, V, st);
}

// The grid of the surface (F > 0 checked faces, box in h): about sqrt(F) / 2 cells along the longest axis, so a
// marching-cubes triangle touches a few cells.  cnt and scan are scratch of F entries, temp holds an InclusiveSum of F
// of them; the (cell, triangle) pairs get an allocation of their own.
int build_surface(const char* name, const float* vertices, const int3* faces, int F, const FaceCheck& h,
                  unsigned long long* cnt, unsigned long long* scan, void* temp, size_t temp_bytes, dgs_alloc_fn alloc,
                  void* alloc_user, cudaStream_t st, Surface& S) {
  double ext[3], ext_max = 0.0;
  S.pos = vertices;
  S.faces = faces;
  for (int k = 0; k < 3; k++) {
    S.mn[k] = (double)fval(h.box[k]);
    ext[k] = (double)fval(h.box[3 + k]) - S.mn[k];
    ext_max = std::max(ext_max, ext[k]);
  }
  const int cells = std::min(std::max((int)std::ceil(std::sqrt((double)F) / 2.0), 1), kMaxCells);
  S.h = ext_max > 0 ? ext_max / cells : 1.0;
  for (int k = 0; k < 3; k++) S.n[k] = std::min((int)std::floor(ext[k] / S.h) + 1, kMaxCells);
  S.keys = S.tris = nullptr;
  S.npairs = 0;
  grid_count_kernel<<<ceil_div(F, kThreads), kThreads, 0, st>>>(F, S, cnt);
  DGS_POST_LAUNCH();
  DGS_CUDA_OK(cub::DeviceScan::InclusiveSum(temp, temp_bytes, cnt, scan, F, st));
  unsigned long long npairs = 0;
  DGS_CUDA_OK(cudaMemcpyAsync(&npairs, scan + F - 1, sizeof(npairs), cudaMemcpyDeviceToHost, st));
  DGS_CUDA_OK(cudaStreamSynchronize(st));  // the pair count sizes the grid
  if (npairs > 0x7fffffffULL) {
    set_error("%s: the surface grid needs %llu (cell, triangle) pairs, more than 2^31 - 1", name, npairs);
    return DGS_ERR_INVALID_ARGUMENT;
  }
  const int np = (int)npairs;
  uint32_t *gk_in = nullptr, *gk = nullptr, *gt_in = nullptr, *gt = nullptr;
  size_t sort_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, gk_in, gk, gt_in, gt, np, 0, 30);
  Carver probe(nullptr);
  for (int k = 0; k < 4; k++) probe.take<uint32_t>(np);
  probe.take<char>(sort_bytes);
  void* buf = alloc(probe.bytes(), alloc_user);
  if (!buf) { set_error("%s: grid allocation failed (%zu bytes)", name, probe.bytes()); return DGS_ERR_ALLOC; }
  Carver cv(buf);
  gk_in = cv.take<uint32_t>(np);
  gk = cv.take<uint32_t>(np);
  gt_in = cv.take<uint32_t>(np);
  gt = cv.take<uint32_t>(np);
  void* sort_temp = cv.take<char>(sort_bytes);
  grid_fill_kernel<<<ceil_div(F, kThreads), kThreads, 0, st>>>(F, S, cnt, scan, gk_in, gt_in);
  DGS_POST_LAUNCH();
  DGS_CUDA_OK(cub::DeviceRadixSort::SortPairs(sort_temp, sort_bytes, gk_in, gk, gt_in, gt, np, 0, 30, st));
  S.keys = gk;
  S.tris = gt;
  S.npairs = np;
  return DGS_OK;
}

__global__ void closest_kernel(int Q, const double* __restrict__ queries, Surface S, double* __restrict__ points,
                               double* __restrict__ d2, int* __restrict__ face) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Q) return;
  const double3 p = make_double3(queries[3 * i], queries[3 * i + 1], queries[3 * i + 2]);
  double best;
  int f;
  const double3 q = closest(S, p, &best, &f);
  points[3 * i] = q.x;
  points[3 * i + 1] = q.y;
  points[3 * i + 2] = q.z;
  d2[i] = best;
  face[i] = f;
}

}  // namespace
}  // namespace dgs

using namespace dgs;

extern "C" {

int dgs_mesh_remesh(const float* vertices, long long num_vertices, const int* faces, long long num_faces,
                    double target_len, int iterations, double feature_deg, double max_surf_dist, dgs_alloc_fn alloc,
                    void* alloc_user, float** out_vertices, int** out_faces, long long* out_num_vertices,
                    long long* out_num_faces, long long* stats, void* stream) {
  const char* name = "mesh remesh";
  const MeshOut out{alloc, alloc_user, out_vertices, out_faces, out_num_vertices, out_num_faces};
  const int rc = check_mesh_args(name, vertices, num_vertices, faces, num_faces,
                                 num_vertices <= 0x7fffffffLL && 3 * num_faces <= 0x7fffffffLL,
                                 "at most 2^31 - 1 vertices and half-edges", out);
  if (rc != DGS_OK) return rc;
  DGS_REQUIRE(std::isfinite(target_len) && target_len > 0, "mesh remesh: target_len must be finite and > 0 (got %g)",
              target_len);
  DGS_REQUIRE(iterations >= 0, "mesh remesh: iterations must be >= 0 (got %d)", iterations);
  DGS_REQUIRE(std::isfinite(feature_deg) && std::isfinite(max_surf_dist),
              "mesh remesh: feature_deg and max_surf_dist must be finite");
  out.set(nullptr, nullptr, 0, 0);
  if (stats)
    for (long long k = 0; k < 4LL * iterations; k++) stats[k] = 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int V = (int)num_vertices, F = (int)num_faces;
  const int T = kThreads;
  if (iterations == 0) return copy_unchanged(name, vertices, V, faces, F, out, st);  // the input, bit for bit
  const int3* in_faces = reinterpret_cast<const int3*>(faces);
  Scratch s;
  {
    void* buf = out.scratch(name, s.carve(nullptr, V, F));
    if (!buf) return DGS_ERR_ALLOC;
    s.carve(buf, V, F);
  }
  Counters h;
  {
    const int rc = check_faces(name, vertices, V, in_faces, F, true, nullptr, &s.ctr->chk, h.chk, st);
    if (rc != DGS_OK) return rc;
  }
  if (F == 0) return DGS_OK;  // nothing is referenced: the result is empty

  const double L = target_len, lo = 4.0 * L / 5.0, hi = 4.0 * L / 3.0;
  const double cos_t = std::cos(feature_deg * (M_PI / 180.0));
  if (max_surf_dist < 0) {
    double d2 = 0.0;
    for (int k = 0; k < 3; k++) {
      const double e = (double)fval(h.chk.box[3 + k]) - (double)fval(h.chk.box[k]);
      d2 += e * e;
    }
    max_surf_dist = std::sqrt(d2) / 100.0;
  }
  Surface S;
  {
    const int rc = build_surface(name, vertices, in_faces, F, h.chk, s.hkey_in, s.hkey, s.temp, s.temp_bytes, alloc,
                                 alloc_user, st, S);
    if (rc != DGS_OK) return rc;
  }
  DGS_CUDA_OK(cudaMemcpyAsync(s.pos, vertices, 3 * (size_t)V * sizeof(float), cudaMemcpyDeviceToDevice, st));
  DGS_CUDA_OK(cudaMemcpyAsync(s.faces, in_faces, (size_t)F * sizeof(int3), cudaMemcpyDeviceToDevice, st));

  for (int it = 0; it < iterations && F > 0; it++) {
    long long* row = stats ? stats + 4LL * it : nullptr;
    // locks, then split
    DGS_CUDA_OK(cudaMemsetAsync(s.lock, 0, (size_t)V, st));
    DGS_CUDA_OK(edge_pass(s, F, V, cos_t, s.lock, false, st));
    const int n = 3 * F;
    split_flag_kernel<<<ceil_div(n, T), T, 0, st>>>(n, s.ctr, s.edges, s.pos, hi, s.eflag);
    DGS_POST_LAUNCH();
    DGS_CUDA_OK(cub::DeviceScan::InclusiveSum(s.temp, s.temp_bytes, s.eflag, s.erank, n, st));
    split_count_kernel<<<ceil_div(F, T), T, 0, st>>>(F, s.edge_of, s.eflag, s.xcnt);
    DGS_POST_LAUNCH();
    DGS_CUDA_OK(cub::DeviceScan::InclusiveSum(s.temp, s.temp_bytes, s.xcnt, s.xscan, F, st));
    uint32_t counts[2] = {0, 0};
    DGS_CUDA_OK(cudaMemcpyAsync(&counts[0], s.erank + n - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    DGS_CUDA_OK(cudaMemcpyAsync(&counts[1], s.xscan + F - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    DGS_CUDA_OK(cudaStreamSynchronize(st));  // the split counts size the grown mesh
    const long long V2 = (long long)V + counts[0], F2 = (long long)F + counts[1];
    if (V2 > 0x7fffffffLL || 3 * F2 > 0x7fffffffLL) {
      set_error("mesh remesh: the split mesh (%lld vertices, %lld faces) is too large", V2, F2);
      return DGS_ERR_INVALID_ARGUMENT;
    }
    if (counts[0] > 0) {
      Scratch w = s;  // the split reads this round's edges from the scratch they were built in
      if (V2 > s.Vc || F2 > s.Fc) {
        const int vc = (int)std::min(V2 + V2 / 2, 0x7fffffffLL), fc = (int)std::min(F2 + F2 / 2, 0x7fffffffLL / 3);
        Scratch g;
        void* buf = out.scratch(name, g.carve(nullptr, vc, fc));
        if (!buf) return DGS_ERR_ALLOC;
        g.carve(buf, vc, fc);
        DGS_CUDA_OK(cudaMemcpyAsync(g.pos, s.pos, 3 * (size_t)V * sizeof(float), cudaMemcpyDeviceToDevice, st));
        DGS_CUDA_OK(cudaMemcpyAsync(g.lock, s.lock, (size_t)V, cudaMemcpyDeviceToDevice, st));
        DGS_CUDA_OK(cudaMemcpyAsync(g.faces, s.faces, (size_t)F * sizeof(int3), cudaMemcpyDeviceToDevice, st));
        s = g;
      }
      split_vertex_kernel<<<ceil_div(n, T), T, 0, st>>>(n, V, w.ctr, w.edges, w.eflag, w.erank, s.pos, s.lock);
      DGS_POST_LAUNCH();
      split_face_kernel<<<ceil_div(F, T), T, 0, st>>>(F, V, w.edge_of, w.eflag, w.erank, w.xcnt, w.xscan, s.pos,
                                                      s.faces);
      DGS_POST_LAUNCH();
      V = (int)V2;
      F = (int)F2;
    }
    if (row) row[0] = F;

    // collapse rounds
    bool collapsed = false;
    for (int r = 0; r < kRoundCap && F > 0; r++) {
      const int gn = ceil_div(3 * F, T), gv = ceil_div(V, T);
      DGS_CUDA_OK(edge_pass(s, F, V, cos_t, nullptr, true, st));
      collapse_cost_kernel<<<gn, T, 0, st>>>(s.ctr, s.edges, s.pos, s.lock, s.faces, s.vrange, s.vfaces, lo, hi,
                                             max_surf_dist, S, s.ekey, s.eplace);
      DGS_POST_LAUNCH();
      m1_kernel<<<gv, T, 0, st>>>(V, s.faces, s.vrange, s.vfaces, s.edge_of, s.ekey, s.m1);
      DGS_POST_LAUNCH();
      m2_kernel<<<gv, T, 0, st>>>(V, s.faces, s.vrange, s.vfaces, s.m1, s.m2);
      DGS_POST_LAUNCH();
      DGS_CUDA_OK(cudaMemsetAsync(&s.ctr->selected, 0, sizeof(int), st));
      DGS_CUDA_OK(cudaMemsetAsync(s.to, 0xff, (size_t)V * sizeof(int), st));
      collapse_apply_kernel<<<gn, T, 0, st>>>(s.ctr, s.edges, s.ekey, s.m2, s.eplace, s.pos, s.lock, s.to);
      DGS_POST_LAUNCH();
      DGS_CUDA_OK(cudaMemcpyAsync(&h, s.ctr, sizeof(h), cudaMemcpyDeviceToHost, st));
      DGS_CUDA_OK(cudaStreamSynchronize(st));  // the one read-back of the round: how many edges were taken
      if (r > 0 && h.num_faces != F) {
        set_error("mesh remesh: internal error, %d faces where %d were expected", h.num_faces, F);
        return DGS_ERR_CUDA;
      }
      if (h.selected == 0) break;
      remap_kernel<<<ceil_div(F, T), T, 0, st>>>(F, s.faces, s.to, s.keep);
      DGS_POST_LAUNCH();
      DGS_CUDA_OK(s.compact(F, &s.ctr->num_faces, st));
      F -= 2 * h.selected;  // the link condition leaves exactly the two faces of each collapsed edge degenerate
      collapsed = true;
      if (row) row[1]++;
    }
    // flip rounds
    for (int r = 0; r < kRoundCap && F > 0; r++) {
      const int gn = ceil_div(3 * F, T);
      DGS_CUDA_OK(edge_pass(s, F, V, cos_t, nullptr, true, st));
      DGS_CUDA_OK(cudaMemsetAsync(s.val, 0, (size_t)V * sizeof(int), st));
      DGS_CUDA_OK(cudaMemsetAsync(s.bnd, 0, (size_t)V, st));
      DGS_CUDA_OK(cudaMemsetAsync(s.m1, 0xff, (size_t)V * sizeof(unsigned long long), st));
      valence_kernel<<<gn, T, 0, st>>>(s.ctr, s.edges, s.val, s.bnd);
      DGS_POST_LAUNCH();
      flip_cost_kernel<<<gn, T, 0, st>>>(s.ctr, s.edges, s.pos, s.faces, s.vrange, s.vfaces, s.val, s.bnd,
                                         max_surf_dist, S, s.ekey, s.m1);
      DGS_POST_LAUNCH();
      DGS_CUDA_OK(cudaMemsetAsync(&s.ctr->selected, 0, sizeof(int), st));
      flip_apply_kernel<<<gn, T, 0, st>>>(s.ctr, s.edges, s.ekey, s.m1, s.faces);
      DGS_POST_LAUNCH();
      DGS_CUDA_OK(cudaMemcpyAsync(&h, s.ctr, sizeof(h), cudaMemcpyDeviceToHost, st));
      DGS_CUDA_OK(cudaStreamSynchronize(st));  // the one read-back of the round: how many edges were flipped
      // the last collapse round's compaction is checked here (flips keep the face count), so every later stage runs
      // on the face count the collapses left
      if (r == 0 && collapsed && h.num_faces != F) {
        set_error("mesh remesh: internal error, %d faces where %d were expected", h.num_faces, F);
        return DGS_ERR_CUDA;
      }
      if (h.selected == 0) break;
      if (row) row[2]++;
    }
    if (row) row[3] = row[1] == kRoundCap || row[2] == kRoundCap;
    if (F == 0) break;
    // tangential smoothing, then reprojection of the referenced vertices onto S
    const int gv = ceil_div(V, T);
    DGS_CUDA_OK(s.vertex_faces(F, V, st));
    smooth_kernel<<<gv, T, 0, st>>>(V, s.pos, s.faces, s.vrange, s.vfaces, s.lock, s.pos_alt);
    DGS_POST_LAUNCH();
    std::swap(s.pos, s.pos_alt);
    reproject_kernel<<<gv, T, 0, st>>>(V, s.pos, s.vrange, S);
    DGS_POST_LAUNCH();
  }

  // finish: referenced vertices in index order, faces remapped
  return emit_mesh(name, s, V, V, F, s.pos, nullptr, nullptr, out, st);
}

int dgs_mesh_closest_points(const float* vertices, long long num_vertices, const int* faces, long long num_faces,
                            const double* queries, long long num_queries, double* out_points, double* out_d2,
                            int* out_faces, dgs_alloc_fn alloc, void* alloc_user, void* stream) {
  DGS_REQUIRE(alloc, "mesh closest points: alloc must not be NULL");
  DGS_REQUIRE(num_vertices >= 0 && num_faces > 0 && num_queries >= 0,
              "mesh closest points: need faces and non-negative sizes (%lld vertices, %lld faces, %lld queries)",
              num_vertices, num_faces, num_queries);
  DGS_REQUIRE(num_vertices <= 0x7fffffffLL && num_faces <= 0x7fffffffLL && num_queries <= 0x7fffffffLL,
              "mesh closest points: %lld vertices / %lld faces / %lld queries is too many (at most 2^31 - 1 each)",
              num_vertices, num_faces, num_queries);
  DGS_REQUIRE(vertices && faces && (num_queries == 0 || (queries && out_points && out_d2 && out_faces)),
              "mesh closest points: vertices, faces, queries and the outputs must not be NULL");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int V = (int)num_vertices, F = (int)num_faces, Q = (int)num_queries;
  const int3* in_faces = reinterpret_cast<const int3*>(faces);
  size_t scan_bytes = 0;
  cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, static_cast<unsigned long long*>(nullptr),
                                static_cast<unsigned long long*>(nullptr), F);
  Carver probe(nullptr);
  probe.take<FaceCheck>(1);
  probe.take<unsigned long long>(F);
  probe.take<unsigned long long>(F);
  probe.take<char>(scan_bytes);
  void* buf = alloc(probe.bytes(), alloc_user);
  if (!buf) { set_error("mesh closest points: scratch allocation failed (%zu bytes)", probe.bytes()); return DGS_ERR_ALLOC; }
  Carver cv(buf);
  FaceCheck* chk = cv.take<FaceCheck>(1);
  unsigned long long* cnt = cv.take<unsigned long long>(F);
  unsigned long long* scan = cv.take<unsigned long long>(F);
  void* temp = cv.take<char>(scan_bytes);
  FaceCheck h;
  int rc = check_faces("mesh closest points", vertices, V, in_faces, F, true, nullptr, chk, h, st);
  if (rc != DGS_OK) return rc;
  Surface S;
  rc = build_surface("mesh closest points", vertices, in_faces, F, h, cnt, scan, temp, scan_bytes, alloc, alloc_user, st,
                     S);
  if (rc != DGS_OK) return rc;
  if (Q > 0) {
    closest_kernel<<<ceil_div(Q, kThreads), kThreads, 0, st>>>(Q, queries, S, out_points, out_d2, out_faces);
    DGS_POST_LAUNCH();
  }
  return DGS_OK;
}

}  // extern "C"
