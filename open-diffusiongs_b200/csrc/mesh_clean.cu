// mesh_clean.cu -- cleaning of an extracted triangle mesh: the reference's clean_mesh (utils/mesh_utils.py:88-147) with
// remesh=False, i.e. pymeshlab's remove-unreferenced-vertices, merge-close-vertices, remove-duplicate-faces,
// remove-null-faces, remove-small-components (by diameter, then by face count) and the non-manifold edge and vertex
// repairs, as nine stages with an exact contract (include/dgs_b200.h, dgs_mesh_clean) that oracle/mesh_clean.py restates
// serially.  Every geometric decision is made in fp64 from the fp32 positions; this file is compiled with -fmad=false,
// so each product and sum is rounded on its own, as in the oracle.  The only atomics are integer ones whose result does
// not depend on their order (min / max of order-preserving float keys, counts, union-find hooks of the larger root
// under the smaller), so the output is the same bits on every run.
//
// Merge: the lexicographically-first maximal independent set of the radius graph, in rounds.  Referenced vertices are
// radix-sorted by the key of their grid cell (cell size >= r); each undecided vertex finds the lowest-index neighbour
// within r in its 27 cells that is not merged (in the previous round's states): a seed -> merge into it; undecided ->
// wait; none -> seed.  The lowest undecided vertex always decides, so the rounds end; one read-back per round.
// Components (stages 5, 6) and fans (stage 8) are lock-free union-find over the sorted half-edges; a root is the
// smallest member, i.e. the component's lowest face / the fan's corner in its lowest face.  Stage 7 walks its sorted
// candidates in one thread.
#include <cmath>

#include "mesh_common.cuh"

namespace dgs {
namespace {

constexpr int kCellBits = 21;

struct Counters {
  FaceCheck chk;                // stage 1's, then its box is stage 4's (the box of what is left)
  int selected;                 // faces kept by the last compaction
  int undecided;                // vertices left undecided by the last merge round
  int counted;                  // faces left by the stage before a combined compaction (3 before 4, 5 before 6)
  int candidates;               // stage 7's faces with an edge of more than two faces
};

// |(b - a) x (c - a)| (fp64, no contraction)
__device__ double doubled_area(const float* __restrict__ pos, int3 f) {
  const double3 a = load(pos, f.x), b = load(pos, f.y), c = load(pos, f.z);
  const double ux = b.x - a.x, uy = b.y - a.y, uz = b.z - a.z, wx = c.x - a.x, wy = c.y - a.y, wz = c.z - a.z;
  const double n0 = uy * wz - uz * wy, n1 = uz * wx - ux * wz, n2 = ux * wy - uy * wx;
  return sqrt(n0 * n0 + n1 * n1 + n2 * n2);
}

// The norm of max - min of a box in keys (6 consecutive: min x y z, max x y z).
__host__ __device__ __forceinline__ double box_diag(const unsigned* b) {
  const double dx = (double)fval(b[3]) - (double)fval(b[0]), dy = (double)fval(b[4]) - (double)fval(b[1]),
               dz = (double)fval(b[5]) - (double)fval(b[2]);
  return sqrt(dx * dx + dy * dy + dz * dz);
}

// Merges the lane's box (and one to *size) into boxes[6 key] for key >= 0.  Every lane of the warp calls it; when the
// warp's valid lanes share one key (the common case: neighbouring faces in one component) the warp reduces first.
__device__ void flush(unsigned* __restrict__ boxes, int* __restrict__ size, int key, const Box& b) {
  const int k0 = __shfl_sync(kFull, key, 0);
  if (__all_sync(kFull, key == k0 || key < 0)) {
    unsigned r[6];
    for (int k = 0; k < 3; k++) {
      r[k] = __reduce_min_sync(kFull, b.lo[k]);
      r[3 + k] = __reduce_max_sync(kFull, b.hi[k]);
    }
    const int n = __popc(__ballot_sync(kFull, key >= 0));
    if ((threadIdx.x & 31) == 0 && k0 >= 0) {
      for (int k = 0; k < 3; k++) {
        atomicMin(&boxes[6 * k0 + k], r[k]);
        atomicMax(&boxes[6 * k0 + 3 + k], r[3 + k]);
      }
      if (size) atomicAdd(&size[k0], n);
    }
  } else if (key >= 0) {
    for (int k = 0; k < 3; k++) {
      atomicMin(&boxes[6 * key + k], b.lo[k]);
      atomicMax(&boxes[6 * key + 3 + k], b.hi[k]);
    }
    if (size) atomicAdd(&size[key], 1);
  }
}

// Adds the warp's number of true predicates to *ctr (every lane calls it).
__device__ __forceinline__ void warp_count(int* ctr, bool pred) {
  const unsigned b = __ballot_sync(kFull, pred);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(ctr, __popc(b));
}

// Union-find: p[x] <= x always, so a root is the smallest member of its set.  Path halving only ever writes an
// ancestor, and a root changes only by the CAS that hooks it, so concurrent finds and unions are safe.
__device__ int uf_find(int* p, int x) {
  volatile int* vp = p;
  while (true) {
    const int y = vp[x];
    if (y == x) return x;
    const int z = vp[y];
    if (z != y) vp[x] = z;
    x = z;
  }
}
__device__ void uf_unite(int* p, int a, int b) {
  while (true) {
    a = uf_find(p, a);
    b = uf_find(p, b);
    if (a == b) return;
    if (a > b) { const int t = a; a = b; b = t; }
    if (atomicCAS(&p[b], b, a) == b) return;
  }
}

__global__ void iota_kernel(int n, int* __restrict__ p) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = i;
}
// After the unions: p[i] = the root of i.  The walk does not compress paths: a halving store of another thread could
// land after this thread's store and leave p[i] at an ancestor that is not the root.
__global__ void flatten_kernel(int n, int* __restrict__ p) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  volatile int* vp = p;
  int r = i, y;
  while ((y = vp[r]) != r) r = y;
  vp[i] = r;
}
__global__ void box_init_kernel(int n, unsigned* __restrict__ boxes) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 6 * n) boxes[i] = i % 6 < 3 ? kFull : 0u;
}

// ----------------------------------------------------------------------------------------- stage 2: merge
struct Grid {
  double mn[3], cell, r;
  int n[3];
};

__global__ void cell_key_kernel(int V, const float* __restrict__ pos, const uint32_t* __restrict__ used, Grid g,
                                unsigned long long* __restrict__ keys, uint32_t* __restrict__ vals) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  unsigned long long key = kNoKey;
  if (used[v]) {
    key = 0;
    for (int k = 0; k < 3; k++) {
      const int c = min(max((int)floor(((double)pos[3 * v + k] - g.mn[k]) / g.cell), 0), g.n[k] - 1);
      key = (key << kCellBits) | (unsigned long long)c;
    }
  }
  keys[v] = key;
  vals[v] = (uint32_t)v;
}

// rep: -1 undecided, v a seed, s < v merged into seed s.  Reads the previous round's states only.
__global__ void merge_round_kernel(int V, const float* __restrict__ pos, Grid g,
                                   const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ vals,
                                   const int* __restrict__ rep_in, int* __restrict__ rep_out, Counters* __restrict__ ctr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= V) return;
  const unsigned long long key = keys[i];
  if (key == kNoKey) return;
  const int v = (int)vals[i];
  if (rep_in[v] >= 0) { rep_out[v] = rep_in[v]; return; }
  const double3 p = load(pos, v);
  const int mask = (1 << kCellBits) - 1;
  const int c[3] = {(int)(key >> (2 * kCellBits)) & mask, (int)(key >> kCellBits) & mask, (int)key & mask};
  int best = v;
  for (int dx = -1; dx <= 1; dx++)
    for (int dy = -1; dy <= 1; dy++)
      for (int dz = -1; dz <= 1; dz++) {
        const int x = c[0] + dx, y = c[1] + dy, z = c[2] + dz;
        if (x < 0 || y < 0 || z < 0 || x >= g.n[0] || y >= g.n[1] || z >= g.n[2]) continue;
        const unsigned long long k =
            ((unsigned long long)x << (2 * kCellBits)) | ((unsigned long long)y << kCellBits) | (unsigned long long)z;
        int lo = 0, hi = V;  // lower bound of k
        while (lo < hi) {
          const int m = (lo + hi) >> 1;
          if (keys[m] < k) lo = m + 1; else hi = m;
        }
        for (int j = lo; j < V && keys[j] == k; j++) {
          const int u = (int)vals[j];
          if (u >= best) continue;
          const int ru = rep_in[u];
          if (ru >= 0 && ru != u) continue;  // merged
          const double3 q = load(pos, u);
          const double ex = q.x - p.x, ey = q.y - p.y, ez = q.z - p.z;
          if (sqrt(ex * ex + ey * ey + ez * ez) < g.r) best = u;
        }
      }
  int out = v;  // no unmerged lower neighbour: a seed
  if (best != v) out = rep_in[best] == best ? best : -1;
  rep_out[v] = out;
  if (out < 0) atomicAdd(&ctr->undecided, 1);
}

// ----------------------------------------------------------------------------------------- stages 3, 4
// LSD sort of the sorted triples (a <= b <= c): by c, then stably by (a, b); ties stay in face order.
__global__ void dup_key_c_kernel(int F, const int3* __restrict__ faces, uint32_t* __restrict__ keys,
                                 uint32_t* __restrict__ vals) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int3 t = faces[f];
  keys[f] = (uint32_t)max(t.x, max(t.y, t.z));
  vals[f] = (uint32_t)f;
}
__global__ void dup_key_ab_kernel(int F, const int3* __restrict__ faces, const uint32_t* __restrict__ perm, int vbits,
                                  unsigned long long* __restrict__ keys, uint32_t* __restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= F) return;
  const uint32_t f = perm[i];
  const int3 t = faces[f];
  const int a = min(t.x, min(t.y, t.z)), b = max(min(t.x, t.y), min(max(t.x, t.y), t.z));
  keys[i] = ((unsigned long long)a << vbits) | (unsigned long long)b;
  vals[i] = f;
}
__global__ void dup_flag_kernel(int F, const int3* __restrict__ faces, const unsigned long long* __restrict__ keys,
                                const uint32_t* __restrict__ vals, uint8_t* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= F) return;
  const int3 t = faces[vals[i]];
  bool first = true;
  if (i > 0 && keys[i - 1] == keys[i]) {
    const int3 s = faces[vals[i - 1]];
    first = max(s.x, max(s.y, s.z)) != max(t.x, max(t.y, t.z));
  }
  keep[vals[i]] = first;
}
// Stage 3's survivors are counted, then null faces dropped from them; the box of what is left sizes stage 5.
__global__ void null_kernel(int F, const int3* __restrict__ faces, const float* __restrict__ pos,
                            uint8_t* __restrict__ keep, Counters* __restrict__ ctr) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  bool nondup = false, ok = false;
  Box b;
  if (f < F) {
    nondup = keep[f];
    const int3 t = faces[f];
    ok = nondup && doubled_area(pos, t) != 0.0;
    keep[f] = ok;
    if (ok) { b.add(pos, t.x); b.add(pos, t.y); b.add(pos, t.z); }
  }
  warp_count(&ctr->counted, nondup);
  flush(ctr->chk.box, nullptr, ok ? 0 : -1, b);
}

// ----------------------------------------------------------------------------------------- stages 5, 6
// Two faces are joined when they share an edge: each sorted half-edge with its predecessor in the same edge.
__global__ void face_union_kernel(int n, const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ vals,
                                  int* __restrict__ parent) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 1 || i >= n || keys[i] != keys[i - 1]) return;
  uf_unite(parent, (int)(vals[i] / 3), (int)(vals[i - 1] / 3));
}
__global__ void comp_stats_kernel(int F, const int3* __restrict__ faces, const float* __restrict__ pos,
                                  const int* __restrict__ comp, unsigned* __restrict__ boxes, int* __restrict__ size) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  Box b;
  int key = -1;
  if (f < F) {
    const int3 t = faces[f];
    b.add(pos, t.x); b.add(pos, t.y); b.add(pos, t.z);
    key = comp[f];
  }
  flush(boxes, size, key, b);
}
__global__ void comp_flag_kernel(int F, const int* __restrict__ comp, const unsigned* __restrict__ boxes,
                                 const int* __restrict__ size, double min_diag, long long min_f,
                                 uint8_t* __restrict__ keep, Counters* __restrict__ ctr) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  bool k5 = false, k6 = false;
  if (f < F) {
    const int c = comp[f];
    k5 = !(box_diag(boxes + 6 * c) < min_diag);
    k6 = k5 && !(size[c] < min_f);
    keep[f] = k6;
  }
  warp_count(&ctr->counted, k5);
}

// ----------------------------------------------------------------------------------------- stage 7
// Per sorted half-edge: its edge; the first of each edge writes the edge's face count.
__global__ void edge_count_kernel(int n, const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ vals,
                                  const uint32_t* __restrict__ scan, uint32_t* __restrict__ edge_of,
                                  int* __restrict__ live) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  edge_of[vals[i]] = scan[i] - 1;
  if (i > 0 && keys[i - 1] == keys[i]) return;
  int j = i + 1;
  while (j < n && keys[j] == keys[i]) j++;
  live[scan[i] - 1] = j - i;
}
// Candidates sort first, by (doubled area, face); the rest get kNoKey.
__global__ void candidate_kernel(int F, const int3* __restrict__ faces, const float* __restrict__ pos,
                                 const uint32_t* __restrict__ edge_of, const int* __restrict__ live,
                                 unsigned long long* __restrict__ keys, uint32_t* __restrict__ vals,
                                 Counters* __restrict__ ctr) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  bool cand = false;
  if (f < F) {
    cand = live[edge_of[3 * f]] > 2 || live[edge_of[3 * f + 1]] > 2 || live[edge_of[3 * f + 2]] > 2;
    keys[f] = cand ? (unsigned long long)__double_as_longlong(doubled_area(pos, faces[f])) : kNoKey;
    vals[f] = (uint32_t)f;
  }
  warp_count(&ctr->candidates, cand);
}
// The serial walk: a candidate goes iff one of its edges still has more than two live faces.
__global__ void nonmanifold_walk_kernel(const Counters* __restrict__ ctr, const uint32_t* __restrict__ order,
                                        const uint32_t* __restrict__ edge_of, int* __restrict__ live,
                                        uint8_t* __restrict__ keep) {
  const int n = ctr->candidates;
  for (int i = 0; i < n; i++) {
    const uint32_t f = order[i];
    const uint32_t e0 = edge_of[3 * f], e1 = edge_of[3 * f + 1], e2 = edge_of[3 * f + 2];
    if (live[e0] > 2 || live[e1] > 2 || live[e2] > 2) {
      live[e0]--; live[e1]--; live[e2]--;
      keep[f] = 0;
    }
  }
}

// ----------------------------------------------------------------------------------------- stage 8
// Corners 3 f + k.  The two half-edges of an edge join the corners of each of its two vertices.
__global__ void fan_union_kernel(int n, const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ vals,
                                 const int* __restrict__ fv, int* __restrict__ parent) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 1 || i >= n || keys[i] != keys[i - 1]) return;
  const int h0 = (int)vals[i - 1], h1 = (int)vals[i];
  const int n0 = 3 * (h0 / 3) + (h0 % 3 + 1) % 3, n1 = 3 * (h1 / 3) + (h1 % 3 + 1) % 3;
  const bool same = fv[h0] == fv[h1];
  uf_unite(parent, h0, same ? h1 : n1);
  uf_unite(parent, n0, same ? n1 : h1);
}
// Over the sorted incidences (vertex, face): a fan root that is not in the vertex's lowest face gets a copy.
__global__ void copy_flag_kernel(int n, const uint32_t* __restrict__ ikey, const uint32_t* __restrict__ vfaces,
                                 const uint2* __restrict__ vrange, const int3* __restrict__ faces,
                                 const int* __restrict__ fan, uint32_t* __restrict__ flag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int v = (int)ikey[i], f = (int)vfaces[i];
  const int3 t = faces[f];
  const int c = 3 * f + (t.x == v ? 0 : t.y == v ? 1 : 2);
  flag[i] = fan[c] == c && (uint32_t)i != vrange[v].x;
}
__global__ void copy_assign_kernel(int n, int V, const uint32_t* __restrict__ ikey, const uint32_t* __restrict__ vfaces,
                                   const int3* __restrict__ faces, const uint32_t* __restrict__ flag,
                                   const uint32_t* __restrict__ scan, int* __restrict__ copy_id,
                                   int* __restrict__ src) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !flag[i]) return;
  const int v = (int)ikey[i], f = (int)vfaces[i];
  const int3 t = faces[f];
  const int c = 3 * f + (t.x == v ? 0 : t.y == v ? 1 : 2);
  const int k = (int)scan[i] - 1;
  copy_id[c] = V + k;
  src[k] = v;
}
__global__ void reindex_kernel(int n, int* __restrict__ fv, const int* __restrict__ fan,
                               const int* __restrict__ copy_id) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n) return;
  const int id = copy_id[fan[c]];
  if (id >= 0) fv[c] = id;
}

// All scratch, sized once from V and F (n = 3F half-edges / corners; at most n vertex copies).
struct Scratch : MeshScratch {
  Counters* ctr;
  int *rep_a, *rep_b, *parent, *copy_id, *src, *live, *csize;
  uint32_t *cval_in, *cval;
  unsigned long long *ckey_in, *ckey;
  unsigned* cbox;

  size_t carve(void* base, int V, int F) {
    const int n = 3 * F;
    Carver cv(base);
    ctr = cv.take<Counters>(1);
    carve_mesh(cv, V, F, V + n);
    rep_a = cv.take<int>(V);
    rep_b = cv.take<int>(V);
    parent = cv.take<int>(n);
    copy_id = cv.take<int>(n);
    src = cv.take<int>(n);
    live = cv.take<int>(n);
    csize = cv.take<int>(F);
    cval_in = cv.take<uint32_t>(V);
    cval = cv.take<uint32_t>(V);
    ckey_in = cv.take<unsigned long long>(V);
    ckey = cv.take<unsigned long long>(V);
    cbox = cv.take<unsigned>(6 * (size_t)F);
    size_t t = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, t, ckey_in, ckey, cval_in, cval, V, 0, 3 * kCellBits);
    need(t);
    cub::DeviceRadixSort::SortPairs(nullptr, t, hkey_in, hkey, hval_in, hval, n, 0, 64);
    need(t);
    carve_temp(cv);
    return cv.bytes();
  }
};

}  // namespace
}  // namespace dgs

using namespace dgs;

// Keeps the faces flagged in s.keep (face order) as s.faces and reads their number back.
#define CLEAN_COMPACT(F)                                                          \
  do {                                                                            \
    DGS_CUDA_OK(s.compact(F, &s.ctr->selected, st));                              \
    DGS_CUDA_OK(cudaMemcpyAsync(&h, s.ctr, sizeof(h), cudaMemcpyDeviceToHost, st)); \
    DGS_CUDA_OK(cudaStreamSynchronize(st));                                       \
    F = h.selected;                                                               \
  } while (0)

extern "C" {

int dgs_mesh_clean(const float* vertices, long long num_vertices, const int* faces, long long num_faces, double v_pct,
                   long long min_f, double min_d, int repair, dgs_alloc_fn alloc, void* alloc_user,
                   float** out_vertices, int** out_faces, long long* out_num_vertices, long long* out_num_faces,
                   int* merge_rounds, long long* stage_faces, void* stream) {
  const char* name = "mesh clean";
  const MeshOut out{alloc, alloc_user, out_vertices, out_faces, out_num_vertices, out_num_faces};
  const int rc = check_mesh_args(name, vertices, num_vertices, faces, num_faces,
                                 num_vertices + 3 * num_faces <= 0x7fffffffLL, "V + 3F must be at most 2^31 - 1", out);
  if (rc != DGS_OK) return rc;
  DGS_REQUIRE(std::isfinite(v_pct) && std::isfinite(min_d), "mesh clean: v_pct and min_d must be finite");
  out.set(nullptr, nullptr, 0, 0);
  if (merge_rounds) *merge_rounds = 0;
  if (stage_faces)
    for (int k = 0; k < 9; k++) stage_faces[k] = 0;
  if (num_faces == 0) return DGS_OK;  // nothing is referenced: the result is empty
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int V = (int)num_vertices, vbits = bits_for(V);
  int F = (int)num_faces;
  Scratch s;
  void* buf = out.scratch(name, s.carve(nullptr, V, F));
  if (!buf) return DGS_ERR_ALLOC;
  s.carve(buf, V, F);
  const int3* in_faces = reinterpret_cast<const int3*>(faces);
  long long counts[9];
  Counters h;
  const int T = kThreads;

  // 1. check the indices; the box of the referenced vertices
  DGS_CUDA_OK(cudaMemcpyAsync(s.faces, in_faces, (size_t)F * sizeof(int3), cudaMemcpyDeviceToDevice, st));
  {
    const int rc = check_faces(name, vertices, V, in_faces, F, false, s.used, &s.ctr->chk, h.chk, st);
    if (rc != DGS_OK) return rc;
  }
  counts[0] = F;

  // 2. merge close vertices
  int rounds = 0;
  if (v_pct > 0) {
    const double r = (v_pct / 100.0) * box_diag(h.chk.box);
    const int gv = ceil_div(V, T);
    if (r > 0) {
      Grid g;
      double ext = 0.0;
      for (int k = 0; k < 3; k++) {
        g.mn[k] = (double)fval(h.chk.box[k]);
        ext = std::max(ext, (double)fval(h.chk.box[3 + k]) - g.mn[k]);
      }
      // a margin over r keeps every pair closer than r within adjacent cells; at most 2^21 - 1 cells per axis
      g.cell = std::max(r * (1.0 + 0x1p-20), ext / ((1 << kCellBits) - 2));
      g.r = r;
      for (int k = 0; k < 3; k++)
        g.n[k] =
            std::min((int)std::floor(((double)fval(h.chk.box[3 + k]) - g.mn[k]) / g.cell) + 1, (1 << kCellBits) - 1);
      cell_key_kernel<<<gv, T, 0, st>>>(V, vertices, s.used, g, s.ckey_in, s.cval_in);
      DGS_POST_LAUNCH();
      DGS_CUDA_OK(cub::DeviceRadixSort::SortPairs(s.temp, s.temp_bytes, s.ckey_in, s.ckey, s.cval_in, s.cval, V, 0, 64,
                                                  st));
      DGS_CUDA_OK(cudaMemsetAsync(s.rep_a, 0xff, (size_t)V * sizeof(int), st));
      while (true) {
        DGS_CUDA_OK(cudaMemsetAsync(&s.ctr->undecided, 0, sizeof(int), st));
        merge_round_kernel<<<gv, T, 0, st>>>(V, vertices, g, s.ckey, s.cval, s.rep_a, s.rep_b, s.ctr);
        DGS_POST_LAUNCH();
        std::swap(s.rep_a, s.rep_b);
        rounds++;
        DGS_CUDA_OK(cudaMemcpyAsync(&h, s.ctr, sizeof(h), cudaMemcpyDeviceToHost, st));
        DGS_CUDA_OK(cudaStreamSynchronize(st));  // the one read-back of the round: how many are still undecided
        if (h.undecided == 0) break;
      }
    } else {
      iota_kernel<<<gv, T, 0, st>>>(V, s.rep_a);
      DGS_POST_LAUNCH();
    }
    remap_kernel<<<ceil_div(F, T), T, 0, st>>>(F, s.faces, s.rep_a, s.keep);
    DGS_POST_LAUNCH();
    CLEAN_COMPACT(F);
  }
  counts[1] = F;

  // 3, 4. duplicate faces, then null faces (one compaction; stage 3's count comes from the flags)
  if (F > 0) {
    const int g = ceil_div(F, T);
    dup_key_c_kernel<<<g, T, 0, st>>>(F, s.faces, s.ikey_in, s.ival_in);
    DGS_POST_LAUNCH();
    DGS_CUDA_OK(cub::DeviceRadixSort::SortPairs(s.temp, s.temp_bytes, s.ikey_in, s.ikey, s.ival_in, s.vfaces, F, 0,
                                                vbits, st));
    dup_key_ab_kernel<<<g, T, 0, st>>>(F, s.faces, s.vfaces, vbits, s.hkey_in, s.hval_in);
    DGS_POST_LAUNCH();
    DGS_CUDA_OK(cub::DeviceRadixSort::SortPairs(s.temp, s.temp_bytes, s.hkey_in, s.hkey, s.hval_in, s.hval, F, 0,
                                                2 * vbits, st));
    dup_flag_kernel<<<g, T, 0, st>>>(F, s.faces, s.hkey, s.hval, s.keep);
    DGS_POST_LAUNCH();
    DGS_CUDA_OK(cudaMemsetAsync(&s.ctr->counted, 0, sizeof(int), st));
    box_init_kernel<<<1, 32, 0, st>>>(1, s.ctr->chk.box);
    DGS_POST_LAUNCH();
    null_kernel<<<g, T, 0, st>>>(F, s.faces, vertices, s.keep, s.ctr);
    DGS_POST_LAUNCH();
    CLEAN_COMPACT(F);
    counts[2] = h.counted;
  } else {
    counts[2] = 0;
  }
  counts[3] = F;

  // 5, 6. small components by diameter, then by face count (one compaction)
  counts[4] = F;
  if (F > 0 && (min_d > 0 || min_f > 0)) {
    const int n = 3 * F, g = ceil_div(F, T);
    DGS_CUDA_OK(s.sort_edges(F, V, st));
    iota_kernel<<<g, T, 0, st>>>(F, s.parent);
    DGS_POST_LAUNCH();
    face_union_kernel<<<ceil_div(n, T), T, 0, st>>>(n, s.hkey, s.hval, s.parent);
    DGS_POST_LAUNCH();
    flatten_kernel<<<g, T, 0, st>>>(F, s.parent);
    DGS_POST_LAUNCH();
    box_init_kernel<<<ceil_div(6 * F, T), T, 0, st>>>(F, s.cbox);
    DGS_POST_LAUNCH();
    DGS_CUDA_OK(cudaMemsetAsync(s.csize, 0, (size_t)F * sizeof(int), st));
    comp_stats_kernel<<<g, T, 0, st>>>(F, s.faces, vertices, s.parent, s.cbox, s.csize);
    DGS_POST_LAUNCH();
    const double min_diag = min_d > 0 ? (min_d / 100.0) * box_diag(h.chk.box) : -1.0;
    DGS_CUDA_OK(cudaMemsetAsync(&s.ctr->counted, 0, sizeof(int), st));
    comp_flag_kernel<<<g, T, 0, st>>>(F, s.parent, s.cbox, s.csize, min_diag, min_f > 0 ? min_f : 0, s.keep, s.ctr);
    DGS_POST_LAUNCH();
    CLEAN_COMPACT(F);
    counts[4] = h.counted;
  }
  counts[5] = F;

  // 7. non-manifold edges
  if (repair && F > 0) {
    const int n = 3 * F, g = ceil_div(F, T);
    DGS_CUDA_OK(s.sort_edges(F, V, st));
    edge_count_kernel<<<ceil_div(n, T), T, 0, st>>>(n, s.hkey, s.hval, s.heads, s.edge_of, s.live);
    DGS_POST_LAUNCH();
    DGS_CUDA_OK(cudaMemsetAsync(&s.ctr->candidates, 0, sizeof(int), st));
    candidate_kernel<<<g, T, 0, st>>>(F, s.faces, vertices, s.edge_of, s.live, s.hkey_in, s.hval_in, s.ctr);
    DGS_POST_LAUNCH();
    DGS_CUDA_OK(cub::DeviceRadixSort::SortPairs(s.temp, s.temp_bytes, s.hkey_in, s.hkey, s.hval_in, s.hval, F, 0, 64,
                                                st));
    DGS_CUDA_OK(cudaMemsetAsync(s.keep, 1, (size_t)F, st));
    nonmanifold_walk_kernel<<<1, 1, 0, st>>>(s.ctr, s.hval, s.edge_of, s.live, s.keep);
    DGS_POST_LAUNCH();
    CLEAN_COMPACT(F);
  }
  counts[6] = F;

  // 8. non-manifold vertices
  int copies = 0;
  if (repair && F > 0) {
    const int n = 3 * F, gn = ceil_div(n, T);
    int* fv = reinterpret_cast<int*>(s.faces);
    DGS_CUDA_OK(s.sort_edges(F, V, st));
    iota_kernel<<<gn, T, 0, st>>>(n, s.parent);
    DGS_POST_LAUNCH();
    fan_union_kernel<<<gn, T, 0, st>>>(n, s.hkey, s.hval, fv, s.parent);
    DGS_POST_LAUNCH();
    flatten_kernel<<<gn, T, 0, st>>>(n, s.parent);
    DGS_POST_LAUNCH();
    DGS_CUDA_OK(s.vertex_faces(F, V, st));
    copy_flag_kernel<<<gn, T, 0, st>>>(n, s.ikey, s.vfaces, s.vrange, s.faces, s.parent, s.heads);
    DGS_POST_LAUNCH();
    DGS_CUDA_OK(cub::DeviceScan::InclusiveSum(s.temp, s.temp_bytes, s.heads, s.vscan, n, st));
    uint32_t total = 0;
    DGS_CUDA_OK(cudaMemcpyAsync(&total, s.vscan + n - 1, sizeof(total), cudaMemcpyDeviceToHost, st));
    DGS_CUDA_OK(cudaStreamSynchronize(st));  // the copy count sizes the vertex range of stage 9
    copies = (int)total;
    if (copies > 0) {
      DGS_CUDA_OK(cudaMemsetAsync(s.copy_id, 0xff, (size_t)n * sizeof(int), st));
      copy_assign_kernel<<<gn, T, 0, st>>>(n, V, s.ikey, s.vfaces, s.faces, s.heads, s.vscan, s.copy_id, s.src);
      DGS_POST_LAUNCH();
      reindex_kernel<<<gn, T, 0, st>>>(n, fv, s.parent, s.copy_id);
      DGS_POST_LAUNCH();
    }
  }
  counts[7] = counts[8] = F;

  // 9. compact: referenced vertices (copies last) in index order, faces remapped
  if (merge_rounds) *merge_rounds = rounds;
  if (stage_faces)
    for (int k = 0; k < 9; k++) stage_faces[k] = counts[k];
  return emit_mesh(name, s, V, V + copies, F, vertices, s.src, nullptr, out, st);
}

}  // extern "C"
