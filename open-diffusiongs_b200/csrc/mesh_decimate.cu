// mesh_decimate.cu -- quadric edge-collapse decimation of a welded triangle mesh to a target face count: the reference's
// decimate_mesh (utils/mesh_utils.py:44-85, pymeshlab's meshing_decimation_quadric_edge_collapse with
// optimalplacement=True), as deterministic rounds of parallel Garland-Heckbert collapses.
//
// Setup: every index is checked on the device (one flag, read at the first host sync).  Each face's plane quadric
// K_f = A_f p p^T (p = (n, -n.x0), unit normal n, area A_f) is formed in fp64; each vertex's quadric Q_v is the sum of
// its faces' K_f in face order, over a stable radix sort of the (vertex, face) incidences.  No floating-point atomics
// anywhere, so the output is the same bits on every run.
//
// Round: unique undirected edges come from a radix sort of the live faces' half-edges by (min, max) and a run-length
// pass, with each edge's two apex vertices when it has exactly two faces; the vertex -> face lists come from a stable
// sort of the incidences (a vertex's neighbours are read through its faces).  Both endpoints of an edge whose face
// count is not 2 (boundary or non-manifold) are locked for the rest of the call, so open surfaces keep their boundary
// loops exactly (pymeshlab's preserve_border behaviour, not its default).  A collapse never creates such an edge, so
// the locks are those of the input.  Per edge (a, b), in fp64: Q = Q_a + Q_b, the optimal position solves the 3 x 3
// system; it falls back to the best of a, b and their midpoint when the system is singular or ill-conditioned, when
// the solution is not finite, or when it lies farther than |a - b| from the midpoint (the spikes the reference warns
// about); cost = v^T Q v.  An edge is not collapsible when an endpoint is locked, when the link condition fails (the
// common neighbours of a and b are not exactly its apexes c != d, or faces (a,c,d) and (b,c,d) both exist), or when
// the move flips a face around a or b (new normal . old normal <= 0, which also rejects a face the move makes
// degenerate; faces that already had zero area are exempt, so coincident marching-cubes vertices collapse cleanly).
// Selection: key = (fp32 bits of cost) << 32 | edge, m1[v] = min key over v's edges, m2[v] = min m1 over v and its
// neighbours, and an edge is taken iff key == m2[a] == m2[b] (see select_kernel for why the taken edges are
// independent).  One read-back per round gives the count; if taking all would pass the target, only the smallest keys
// are kept.  Apply: the lower index survives at the new position with Q_a += Q_b, b becomes a in every face (winding
// kept), the two faces with both die and the faces are compacted in order.  Rounds stop at F <= target or when no
// edge can be taken.  Finish: referenced vertices are compacted in index order and the faces remapped.
#include "mesh_collapse.cuh"

namespace dgs {
namespace {

constexpr double kMaxCondition = 1e7;  // Frobenius condition number above which the 3 x 3 system is not solved

struct Quadric {
  double q[10];  // xx xy xz xw yy yz yw zz zw ww of the symmetric 4 x 4 form
};

struct Counters {
  FaceCheck chk;
  int num_edges, num_selected, num_faces;
};

__device__ Quadric face_quadric(const float* __restrict__ pos, int3 f) {
  const double3 p0 = load(pos, f.x);
  const double3 n = cross(sub(load(pos, f.y), p0), sub(load(pos, f.z), p0));
  const double len = sqrt(dot(n, n));
  Quadric K;
  if (!(len > 0.0) || !isfinite(len)) {
    for (int i = 0; i < 10; i++) K.q[i] = 0.0;
    return K;
  }
  const double w = 0.5 * len;
  const double p[4] = {n.x / len, n.y / len, n.z / len, -(n.x * p0.x + n.y * p0.y + n.z * p0.z) / len};
  int k = 0;
  for (int i = 0; i < 4; i++)
    for (int j = i; j < 4; j++) K.q[k++] = w * p[i] * p[j];
  return K;
}

__device__ __forceinline__ double quadric_cost(const double* q, double3 v) {
  return v.x * (q[0] * v.x + 2.0 * (q[1] * v.y + q[2] * v.z + q[3])) + v.y * (q[4] * v.y + 2.0 * (q[5] * v.z + q[6])) +
         v.z * (q[7] * v.z + 2.0 * q[8]) + q[9];
}

// The fp32 position the collapse of (pa, pb) moves to under quadric q, and its cost there.
__device__ double3 placement(const double* q, double3 pa, double3 pb, double& cost) {
  const double3 mid = round_f32(make_double3(0.5 * (pa.x + pb.x), 0.5 * (pa.y + pb.y), 0.5 * (pa.z + pb.z)));
  const double a00 = q[0], a01 = q[1], a02 = q[2], a11 = q[4], a12 = q[5], a22 = q[7];
  const double c00 = a11 * a22 - a12 * a12, c01 = a02 * a12 - a01 * a22, c02 = a01 * a12 - a02 * a11;
  const double c11 = a00 * a22 - a02 * a02, c12 = a01 * a02 - a00 * a12, c22 = a00 * a11 - a01 * a01;
  const double det = a00 * c00 + a01 * c01 + a02 * c02;
  const double nA = sqrt(a00 * a00 + a11 * a11 + a22 * a22 + 2.0 * (a01 * a01 + a02 * a02 + a12 * a12));
  const double nC = sqrt(c00 * c00 + c11 * c11 + c22 * c22 + 2.0 * (c01 * c01 + c02 * c02 + c12 * c12));
  if (det != 0.0 && nA * nC <= kMaxCondition * fabs(det)) {  // A v = -b by the adjugate (A symmetric)
    const double b0 = q[3], b1 = q[6], b2 = q[8];
    const double3 v = round_f32(make_double3(-(c00 * b0 + c01 * b1 + c02 * b2) / det,
                                             -(c01 * b0 + c11 * b1 + c12 * b2) / det,
                                             -(c02 * b0 + c12 * b1 + c22 * b2) / det));
    const double3 dm = sub(v, mid), ab = sub(pa, pb);
    if (isfinite(v.x) && isfinite(v.y) && isfinite(v.z) && dot(dm, dm) <= dot(ab, ab)) {
      cost = quadric_cost(q, v);
      return v;
    }
  }
  double3 best = mid;
  cost = quadric_cost(q, mid);
  const double ca = quadric_cost(q, pa), cb = quadric_cost(q, pb);
  if (ca < cost) { best = pa; cost = ca; }
  if (cb < cost) { best = pb; cost = cb; }
  return best;
}

// ---------------------------------------------------------------------------------------------------------- setup
__global__ void vertex_quadric_kernel(int V, const float* __restrict__ pos, const int3* __restrict__ faces,
                                      const uint2* __restrict__ vrange, const uint32_t* __restrict__ vfaces,
                                      Quadric* __restrict__ Q) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  Quadric s;
  for (int i = 0; i < 10; i++) s.q[i] = 0.0;
  const uint2 r = vrange[v];
  for (uint32_t i = r.x; i < r.y; i++) {
    const Quadric K = face_quadric(pos, faces[vfaces[i]]);
    for (int k = 0; k < 10; k++) s.q[k] += K.q[k];
  }
  Q[v] = s;
}

// ---------------------------------------------------------------------------------------------------------- edges
// One thread per sorted half-edge: its edge id; the run's first thread writes the edge, its apexes and the locks.
__global__ void edge_build_kernel(int n, const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ vals,
                                  const uint32_t* __restrict__ scan, const int3* __restrict__ faces, int vbits,
                                  Edge* __restrict__ edges, uint32_t* __restrict__ edge_of, uint8_t* __restrict__ lock,
                                  Counters* __restrict__ ctr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t eid = scan[i] - 1;
  edge_of[vals[i]] = eid;
  if (i == n - 1) ctr->num_edges = (int)scan[i];
  const unsigned long long key = keys[i];
  if (i > 0 && keys[i - 1] == key) return;
  int j = i + 1;
  while (j < n && keys[j] == key) j++;
  Edge e;
  e.a = (int)(key >> vbits);
  e.b = (int)(key & ((1ull << vbits) - 1));
  e.c = e.d = -1;
  if (j - i == 2) {
    const uint32_t h0 = vals[i], h1 = vals[i + 1];
    e.c = corner(faces[h0 / 3], (h0 % 3 + 2) % 3);
    e.d = corner(faces[h1 / 3], (h1 % 3 + 2) % 3);
  } else {
    lock[e.a] = 1;
    lock[e.b] = 1;
  }
  edges[eid] = e;
}

__global__ void cost_kernel(const Counters* __restrict__ ctr, const Edge* __restrict__ edges,
                            const float* __restrict__ pos, const Quadric* __restrict__ Q, const uint8_t* __restrict__ lock,
                            const int3* __restrict__ faces, const uint2* __restrict__ vrange,
                            const uint32_t* __restrict__ vfaces, unsigned long long* __restrict__ ekey,
                            float3* __restrict__ eplace) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ctr->num_edges) return;
  const Edge e = edges[i];
  ekey[i] = kNoKey;
  if (e.c < 0 || lock[e.a] || lock[e.b] || !link_ok(e, faces, vrange, vfaces)) return;
  double q[10];
  for (int k = 0; k < 10; k++) q[k] = Q[e.a].q[k] + Q[e.b].q[k];
  double cost;
  const double3 v = placement(q, load(pos, e.a), load(pos, e.b), cost);
  if (!isfinite(cost)) return;
  if (!keeps_orientation(e.a, e.b, v, pos, faces, vrange, vfaces) ||
      !keeps_orientation(e.b, e.a, v, pos, faces, vrange, vfaces))
    return;
  const float c = cost > 0.0 ? (float)cost : 0.f;
  ekey[i] = ((unsigned long long)__float_as_uint(c) << 32) | (unsigned)i;
  eplace[i] = make_float3((float)v.x, (float)v.y, (float)v.z);
}

// Edge (a, b) is taken iff key == m2[a] == m2[b]: its key is the smallest over every edge touching the closed
// neighbourhoods of a and b.  If another taken edge (a', b') had an endpoint, say a', in N[a] (a or a neighbour), then
// key' = m2[a'] <= m1[a] <= key and key = m2[a] <= m1[a'] <= key', so key == key' and, keys holding the edge index, the
// edges are the same.  So the endpoints of two taken edges are at least two hops apart: no face contains endpoints of
// both, and no vertex whose position or faces one collapse reads (the link and fold-over tests read a, b, their faces
// and those faces' vertices) is moved or renamed by the other.  The collapses of a round are independent, and each
// one's tests hold after all of them are applied.
__global__ void select_kernel(Counters* __restrict__ ctr, const Edge* __restrict__ edges,
                              const unsigned long long* __restrict__ ekey, const unsigned long long* __restrict__ m2,
                              unsigned long long* __restrict__ skey) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ctr->num_edges) return;
  const unsigned long long key = ekey[i];
  const Edge e = edges[i];
  const bool take = key != kNoKey && m2[e.a] == key && m2[e.b] == key;
  skey[i] = take ? key : kNoKey;
  if (take) atomicAdd(&ctr->num_selected, 1);
}

// The taken edges with key <= *thr (every taken edge when thr is NULL): b retires into a.
__global__ void apply_kernel(const Counters* __restrict__ ctr, const Edge* __restrict__ edges,
                             const unsigned long long* __restrict__ skey, const unsigned long long* __restrict__ thr,
                             const float3* __restrict__ eplace, float* __restrict__ pos, Quadric* __restrict__ Q,
                             int* __restrict__ to) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ctr->num_edges) return;
  const unsigned long long key = skey[i];
  if (key == kNoKey || (thr && key > *thr)) return;
  const Edge e = edges[i];
  const float3 p = eplace[i];
  pos[3 * e.a] = p.x;
  pos[3 * e.a + 1] = p.y;
  pos[3 * e.a + 2] = p.z;
  for (int k = 0; k < 10; k++) Q[e.a].q[k] += Q[e.b].q[k];
  to[e.b] = e.a;
}

// All scratch, sized once from V and F (n = 3F half-edges, at most n edges).
struct Scratch : MeshScratch {
  Counters* ctr;
  float* pos;
  Quadric* Q;
  uint8_t* lock;
  int* to;
  unsigned long long *m1, *m2, *skey, *skey_sorted, *ekey;
  Edge* edges;
  float3* eplace;

  size_t carve(void* base, int V, int F) {
    const int n = 3 * F;
    Carver cv(base);
    ctr = cv.take<Counters>(1);
    carve_mesh(cv, V, F, V);
    pos = cv.take<float>(3 * (size_t)V);
    Q = cv.take<Quadric>(V);
    lock = cv.take<uint8_t>(V);
    to = cv.take<int>(V);
    m1 = cv.take<unsigned long long>(V);
    m2 = cv.take<unsigned long long>(V);
    skey = cv.take<unsigned long long>(n);
    skey_sorted = cv.take<unsigned long long>(n);
    ekey = cv.take<unsigned long long>(n);
    edges = cv.take<Edge>(n);
    eplace = cv.take<float3>(n);
    size_t t = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, t, skey, skey_sorted, n);
    need(t);
    carve_temp(cv);
    return cv.bytes();
  }
};

}  // namespace
}  // namespace dgs

using namespace dgs;

extern "C" {

int dgs_mesh_decimate(const float* vertices, long long num_vertices, const int* faces, long long num_faces,
                      long long target_faces, dgs_alloc_fn alloc, void* alloc_user, float** out_vertices,
                      int** out_faces, long long* out_num_vertices, long long* out_num_faces, int* rounds,
                      void* stream) {
  const char* name = "mesh decimate";
  const MeshOut out{alloc, alloc_user, out_vertices, out_faces, out_num_vertices, out_num_faces};
  const int rc = check_mesh_args(name, vertices, num_vertices, faces, num_faces,
                                 num_vertices <= 0x7fffffffLL && 3 * num_faces <= 0x7fffffffLL,
                                 "at most 2^31 - 1 vertices and half-edges", out);
  if (rc != DGS_OK) return rc;
  DGS_REQUIRE(target_faces >= 0, "mesh decimate: target_faces must be >= 0 (got %lld)", target_faces);
  out.set(nullptr, nullptr, 0, 0);
  if (rounds) *rounds = 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int V = (int)num_vertices, F = (int)num_faces, vbits = bits_for(V);
  if (num_faces <= target_faces) return copy_unchanged(name, vertices, V, faces, F, out, st);
  Scratch s;
  void* buf = out.scratch(name, s.carve(nullptr, V, F));
  if (!buf) return DGS_ERR_ALLOC;
  s.carve(buf, V, F);
  const int3* in_faces = reinterpret_cast<const int3*>(faces);
  DGS_CUDA_OK(cudaMemcpyAsync(s.pos, vertices, 3 * (size_t)V * sizeof(float), cudaMemcpyDeviceToDevice, st));
  DGS_CUDA_OK(cudaMemcpyAsync(s.faces, in_faces, (size_t)F * sizeof(int3), cudaMemcpyDeviceToDevice, st));
  Counters h;
  {
    const int rc = check_faces(name, vertices, V, in_faces, F, true, nullptr, &s.ctr->chk, h.chk, st);
    if (rc != DGS_OK) return rc;
  }

  // setup: vertex quadrics over the vertex -> face lists (face order), no locks yet
  DGS_CUDA_OK(s.vertex_faces(F, V, st));
  vertex_quadric_kernel<<<ceil_div(V, kThreads), kThreads, 0, st>>>(V, s.pos, s.faces, s.vrange, s.vfaces, s.Q);
  DGS_POST_LAUNCH();
  DGS_CUDA_OK(cudaMemsetAsync(s.lock, 0, (size_t)V, st));

  int live = F, applied_rounds = 0;
  while (live > (long long)target_faces) {
    const int n = 3 * live, gn = ceil_div(n, kThreads), gv = ceil_div(V, kThreads);
    DGS_CUDA_OK(s.sort_edges(live, V, st));
    edge_build_kernel<<<gn, kThreads, 0, st>>>(n, s.hkey, s.hval, s.heads, s.faces, vbits, s.edges, s.edge_of, s.lock,
                                               s.ctr);
    DGS_POST_LAUNCH();
    if (applied_rounds > 0) DGS_CUDA_OK(s.vertex_faces(live, V, st));  // setup built the first round's
    cost_kernel<<<gn, kThreads, 0, st>>>(s.ctr, s.edges, s.pos, s.Q, s.lock, s.faces, s.vrange, s.vfaces, s.ekey,
                                         s.eplace);
    DGS_POST_LAUNCH();
    m1_kernel<<<gv, kThreads, 0, st>>>(V, s.faces, s.vrange, s.vfaces, s.edge_of, s.ekey, s.m1);
    DGS_POST_LAUNCH();
    m2_kernel<<<gv, kThreads, 0, st>>>(V, s.faces, s.vrange, s.vfaces, s.m1, s.m2);
    DGS_POST_LAUNCH();
    DGS_CUDA_OK(cudaMemsetAsync(&s.ctr->num_selected, 0, sizeof(int), st));
    select_kernel<<<gn, kThreads, 0, st>>>(s.ctr, s.edges, s.ekey, s.m2, s.skey);
    DGS_POST_LAUNCH();
    DGS_CUDA_OK(cudaMemcpyAsync(&h, s.ctr, sizeof(h), cudaMemcpyDeviceToHost, st));
    DGS_CUDA_OK(cudaStreamSynchronize(st));  // the one read-back of the round: how many edges were taken
    if (applied_rounds > 0 && h.num_faces != live) {
      set_error("mesh decimate: internal error, %d live faces where %d were expected", h.num_faces, live);
      return DGS_ERR_CUDA;
    }
    if (h.num_selected == 0) break;
    // every collapse removes exactly the two faces of its edge; round up so that the result is target or target - 1
    const int want = (int)((live - target_faces + 1) / 2), take = std::min(h.num_selected, want);
    const unsigned long long* thr = nullptr;
    if (take < h.num_selected) {
      DGS_CUDA_OK(cub::DeviceRadixSort::SortKeys(s.temp, s.temp_bytes, s.skey, s.skey_sorted, h.num_edges, 0, 64, st));
      thr = s.skey_sorted + (take - 1);
    }
    DGS_CUDA_OK(cudaMemsetAsync(s.to, 0xff, (size_t)V * sizeof(int), st));
    apply_kernel<<<gn, kThreads, 0, st>>>(s.ctr, s.edges, s.skey, thr, s.eplace, s.pos, s.Q, s.to);
    DGS_POST_LAUNCH();
    remap_kernel<<<ceil_div(live, kThreads), kThreads, 0, st>>>(live, s.faces, s.to, s.keep);
    DGS_POST_LAUNCH();
    DGS_CUDA_OK(s.compact(live, &s.ctr->num_faces, st));
    live -= 2 * take;
    applied_rounds++;
  }

  // finish: referenced vertices in index order, faces remapped
  if (rounds) *rounds = applied_rounds;
  return emit_mesh(name, s, V, V, live, s.pos, nullptr, applied_rounds > 0 ? &s.ctr->num_faces : nullptr, out, st);
}

}  // extern "C"
