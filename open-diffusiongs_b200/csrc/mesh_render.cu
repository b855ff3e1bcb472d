// mesh_render.cu -- depth-tested triangle rasterization of a mesh into face id, depth, alpha, normal and colour maps,
// with silhouette antialiasing (include/dgs_b200.h, dgs_mesh_render; the serial specification is oracle/mesh_render.py).
//
// Per chunk of views: setup per (view, face) -> coverage of the triangles whose pixel box fits one 8 x 8 tile, one
// thread each, and of the larger ones as (triangle, tile) work items found by a scan -> resolve per pixel ->
// antialias per pixel (gather).  The depth test is a 64-bit atomicMin on (depth key << 32 | face), so every output is
// the same bits on every run.  Compiled with -fmad=false: every fp32 product and sum is rounded as the oracle rounds it.
#include <cub/cub.cuh>

#include "mesh_common.cuh"

namespace dgs {
namespace {

constexpr int kTile = 8;        // a thread's pixel box: kTile x kTile
constexpr float kSub = 256.f;   // snapped screen positions, in 1/256 pixel
constexpr int kMaxSize = 8192;  // largest H and W
// Guard band, in pixels beyond each side of the image.  After clipping every screen coordinate lies in
// [-kGuard, kMaxSize + kGuard] (to within fp32 rounding), so a snapped coordinate is below 2^22 in magnitude, a
// difference of two below 2^23, and an edge function (two products of such differences) below 2^47: int64 is exact.
constexpr float kGuard = 8192.f;
constexpr int kMaxPoly = 8;     // a triangle clipped by 5 planes

struct Hom {  // a vertex in screen-homogeneous coordinates: screen position (X / w, Y / w), clip w
  float X, Y, w;
};

// Row-major world -> clip matrix M; X = (clip x + w) W / 2, Y = (clip y + w) H / 2, so pixel (i, j) has its centre at
// X / w = i + 0.5, Y / w = j + 0.5.
__device__ __forceinline__ Hom transform(const float* __restrict__ M, const float* __restrict__ pos, int v, float hw,
                                         float hh) {
  const float x = pos[3 * v], y = pos[3 * v + 1], z = pos[3 * v + 2];
  const float cx = ((M[0] * x + M[1] * y) + M[2] * z) + M[3];
  const float cy = ((M[4] * x + M[5] * y) + M[6] * z) + M[7];
  const float cw = ((M[12] * x + M[13] * y) + M[14] * z) + M[15];
  return Hom{(cx + cw) * hw, (cy + cw) * hh, cw};
}

struct Frame {
  int W, H;
  float hw, hh, near, gx, gy;  // gx = W + kGuard, gy = H + kGuard
};

// Signed distance of v to clip plane p (inside: >= 0): w >= near, then the four sides of the guard band.
__device__ __forceinline__ float plane_dist(const Frame& fr, int p, const Hom& v) {
  switch (p) {
    case 0: return v.w - fr.near;
    case 1: return v.X + kGuard * v.w;
    case 2: return fr.gx * v.w - v.X;
    case 3: return v.Y + kGuard * v.w;
    default: return fr.gy * v.w - v.Y;
  }
}

// The clipped, snapped polygon of one triangle and its pixel box.
struct Prim {
  int n;  // 0: culled
  int x[kMaxPoly], y[kMaxPoly];
  int i0, i1, j0, j1;
  __device__ int tiles_x() const { return (i1 - i0) / kTile + 1; }
  __device__ int tiles() const { return tiles_x() * ((j1 - j0) / kTile + 1); }
};

// Sutherland-Hodgman against the 5 planes in order.  The crossing of an edge is computed from its inside end to its
// outside end, so the two faces sharing an edge make the same point.
__device__ Prim setup_prim(const Frame& fr, const Hom t[3]) {
  Hom a[kMaxPoly + 1], b[kMaxPoly + 1];
  int n = 3;
  a[0] = t[0]; a[1] = t[1]; a[2] = t[2];
  Prim pr;
  pr.n = 0;
  for (int p = 0; p < 5; p++) {
    float d[kMaxPoly + 1];
    bool any_out = false;
    for (int k = 0; k < n; k++) {
      d[k] = plane_dist(fr, p, a[k]);
      any_out |= !(d[k] >= 0.f);
    }
    if (!any_out) continue;
    int m = 0;
    for (int k = 0; k < n; k++) {
      const int k1 = k + 1 == n ? 0 : k + 1;
      const bool in0 = d[k] >= 0.f, in1 = d[k1] >= 0.f;
      // a convex polygon gains at most one corner per plane (8 at most); rounding that alternates the signs of d on
      // a near-degenerate face could make more, and such a face is culled
      if (m + (int)in0 + (int)(in0 != in1) > kMaxPoly) return pr;
      if (in0) b[m++] = a[k];
      if (in0 != in1) {
        const Hom& I = in0 ? a[k] : a[k1];
        const Hom& O = in0 ? a[k1] : a[k];
        const float di = in0 ? d[k] : d[k1], dout = in0 ? d[k1] : d[k];
        const float s = di / (di - dout);
        b[m++] = Hom{I.X + s * (O.X - I.X), I.Y + s * (O.Y - I.Y), I.w + s * (O.w - I.w)};
      }
    }
    n = m;
    for (int k = 0; k < n; k++) a[k] = b[k];
    if (n < 3) return pr;
  }
  long long area = 0;
  int xmin = INT_MAX, xmax = INT_MIN, ymin = INT_MAX, ymax = INT_MIN;
  for (int k = 0; k < n; k++) {
    pr.x[k] = (int)rintf((a[k].X / a[k].w) * kSub);
    pr.y[k] = (int)rintf((a[k].Y / a[k].w) * kSub);
    xmin = min(xmin, pr.x[k]); xmax = max(xmax, pr.x[k]);
    ymin = min(ymin, pr.y[k]); ymax = max(ymax, pr.y[k]);
  }
  for (int k = 0; k < n; k++) {
    const int k1 = k + 1 == n ? 0 : k + 1;
    area += (long long)pr.x[k] * pr.y[k1] - (long long)pr.x[k1] * pr.y[k];
  }
  if (area == 0) return pr;
  if (area < 0)  // make the inside the positive side of every edge function
    for (int k = 0; k < n / 2; k++) {
      const int tx = pr.x[k], ty = pr.y[k];
      pr.x[k] = pr.x[n - 1 - k]; pr.y[k] = pr.y[n - 1 - k];
      pr.x[n - 1 - k] = tx; pr.y[n - 1 - k] = ty;
    }
  // pixel i is a candidate when its centre 256 i + 128 lies in [min, max]
  pr.i0 = max((xmin - 128 + 255) >> 8, 0);
  pr.i1 = min((xmax - 128) >> 8, fr.W - 1);
  pr.j0 = max((ymin - 128 + 255) >> 8, 0);
  pr.j1 = min((ymax - 128) >> 8, fr.H - 1);
  if (pr.i0 > pr.i1 || pr.j0 > pr.j1) return pr;
  pr.n = n;
  return pr;
}

// Top-left rule: a centre on an edge belongs to the face whose edge is a top edge (horizontal, inside below) or a
// left edge (inside to the right); zero-length edges are skipped.
__device__ __forceinline__ bool covers(const Prim& pr, int i, int j) {
  const long long px = 256LL * i + 128, py = 256LL * j + 128;
  for (int k = 0; k < pr.n; k++) {
    const int k1 = k + 1 == pr.n ? 0 : k + 1;
    const long long dx = pr.x[k1] - pr.x[k], dy = pr.y[k1] - pr.y[k];
    if (dx == 0 && dy == 0) continue;
    const long long e = dx * (py - pr.y[k]) - dy * (px - pr.x[k]);
    const bool top_left = dy < 0 || (dy == 0 && dx > 0);
    if (e < (top_left ? 0 : 1)) return false;
  }
  return true;
}

// b[k]: the homogeneous edge function of the edge opposite corner k at screen point (px, py); u = b / sum(b) are the
// perspective-correct barycentrics of the unclipped face.  Returns the sum (0: no barycentrics).
__device__ __forceinline__ float edge_fns(const Hom t[3], float px, float py, float b[3]) {
  float ex[3], ey[3];
  for (int k = 0; k < 3; k++) {
    ex[k] = t[k].X - px * t[k].w;
    ey[k] = t[k].Y - py * t[k].w;
  }
  b[0] = ex[1] * ey[2] - ex[2] * ey[1];
  b[1] = ex[2] * ey[0] - ex[0] * ey[2];
  b[2] = ex[0] * ey[1] - ex[1] * ey[0];
  return (b[0] + b[1]) + b[2];
}

__device__ __forceinline__ bool bary(const Hom t[3], int i, int j, float u[3]) {
  float b[3];
  const float d = edge_fns(t, (float)i + 0.5f, (float)j + 0.5f, b);
  if (!(d != 0.f)) return false;
  u[0] = b[0] / d; u[1] = b[1] / d; u[2] = b[2] / d;
  return true;
}

__device__ __forceinline__ float lerp3(const float u[3], float a, float b, float c) {
  return (u[0] * a + u[1] * b) + u[2] * c;
}

struct Mesh {
  const float* pos;
  const int3* faces;
  int F;
  const float* clip;  // [views, 4, 4]
};

__device__ __forceinline__ void face_hom(const Mesh& m, const Frame& fr, int view, int f, Hom t[3]) {
  const float* M = m.clip + 16 * (size_t)view;
  const int3 c = m.faces[f];
  t[0] = transform(M, m.pos, c.x, fr.hw, fr.hh);
  t[1] = transform(M, m.pos, c.y, fr.hw, fr.hh);
  t[2] = transform(M, m.pos, c.z, fr.hw, fr.hh);
}

// Depth-tests face f at pixel (i, j); keys is its view's key image.
__device__ __forceinline__ void shade(const Frame& fr, const Hom t[3], int f, int i, int j,
                                      unsigned long long* __restrict__ keys) {
  float u[3];
  if (!bary(t, i, j, u)) return;
  const float depth = lerp3(u, t[0].w, t[1].w, t[2].w);
  atomicMin(keys + (size_t)j * fr.W + i, ((unsigned long long)fkey(depth) << 32) | (unsigned)f);
}

__device__ __forceinline__ void walk(const Frame& fr, const Prim& pr, const Hom t[3], int f, int ti,
                                     unsigned long long* __restrict__ keys) {
  const int tx = ti % pr.tiles_x(), ty = ti / pr.tiles_x();
  const int ia = pr.i0 + tx * kTile, ja = pr.j0 + ty * kTile;
  const int ib = min(ia + kTile - 1, pr.i1), jb = min(ja + kTile - 1, pr.j1);
  for (int j = ja; j <= jb; j++)
    for (int i = ia; i <= ib; i++)
      if (covers(pr, i, j)) shade(fr, t, f, i, j, keys);
}

// Per (view, face): the number of tiles when more than one (0 otherwise), and the facing: the sign of the homogeneous
// determinant of the unclipped face, defined for faces crossing the near plane too.
__global__ void setup_kernel(long long n, Mesh m, Frame fr, int view0, unsigned long long* __restrict__ tiles,
                             int8_t* __restrict__ facing) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const int vs = (int)(idx / m.F), f = (int)(idx - (long long)vs * m.F);
  Hom t[3];
  face_hom(m, fr, view0 + vs, f, t);
  const float det = (t[0].X * (t[1].Y * t[2].w - t[1].w * t[2].Y) - t[0].Y * (t[1].X * t[2].w - t[1].w * t[2].X)) +
                    t[0].w * (t[1].X * t[2].Y - t[1].Y * t[2].X);
  facing[idx] = (int8_t)((det > 0.f) - (det < 0.f));
  const Prim pr = setup_prim(fr, t);
  tiles[idx] = pr.n && pr.tiles() > 1 ? (unsigned long long)pr.tiles() : 0ull;
}

// One thread per (view, face) whose box is one tile.
__global__ void cover_small_kernel(long long n, Mesh m, Frame fr, int view0, const unsigned long long* __restrict__ tiles,
                                   unsigned long long* __restrict__ keys) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n || tiles[idx]) return;
  const int vs = (int)(idx / m.F), f = (int)(idx - (long long)vs * m.F);
  Hom t[3];
  face_hom(m, fr, view0 + vs, f, t);
  const Prim pr = setup_prim(fr, t);
  if (pr.n) walk(fr, pr, t, f, 0, keys + (size_t)vs * fr.H * fr.W);
}

// One thread per (large triangle, tile): item it belongs to the first (view, face) whose inclusive tile sum exceeds it.
__global__ void cover_tiles_kernel(long long n, unsigned long long total, Mesh m, Frame fr, int view0,
                                   const unsigned long long* __restrict__ incl, unsigned long long* __restrict__ keys) {
  for (unsigned long long it = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; it < total;
       it += (unsigned long long)gridDim.x * blockDim.x) {
    long long lo = 0, hi = n - 1;
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      if (incl[mid] > it) hi = mid; else lo = mid + 1;
    }
    const unsigned long long first = lo ? incl[lo - 1] : 0ull;
    const int vs = (int)(lo / m.F), f = (int)(lo - (long long)vs * m.F);
    Hom t[3];
    face_hom(m, fr, view0 + vs, f, t);
    const Prim pr = setup_prim(fr, t);
    walk(fr, pr, t, f, (int)(it - first), keys + (size_t)vs * fr.H * fr.W);
  }
}

struct Attrs {
  const float* normals;  // [V, 3] or NULL
  const float* colors;
  float nbg[3], cbg[3];
};

// Per pixel: face id and depth to the outputs, the normal and colour before antialiasing to pre [pixel][6].
__global__ void resolve_kernel(long long n, Mesh m, Frame fr, int view0, Attrs at,
                               const unsigned long long* __restrict__ keys, float* __restrict__ pre,
                               int* __restrict__ out_id, float* __restrict__ out_depth) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const long long hw = (long long)fr.H * fr.W;
  const int vs = (int)(idx / hw);
  const int pix = (int)(idx - vs * hw), j = pix / fr.W, i = pix - j * fr.W;
  const unsigned long long key = keys[idx];
  const size_t o = (size_t)view0 * hw + idx;
  float* p = pre + 6 * (size_t)idx;
  if (key == kNoKey) {
    if (out_id) out_id[o] = -1;
    if (out_depth) out_depth[o] = 0.f;
    for (int c = 0; c < 3; c++) { p[c] = at.nbg[c]; p[3 + c] = at.cbg[c]; }
    return;
  }
  const int f = (int)(unsigned)key;
  Hom t[3];
  face_hom(m, fr, view0 + vs, f, t);
  float u[3];
  bary(t, i, j, u);  // non-zero sum: the coverage pass tested it
  if (out_id) out_id[o] = f;
  if (out_depth) out_depth[o] = lerp3(u, t[0].w, t[1].w, t[2].w);
  const int3 c = m.faces[f];
  for (int k = 0; k < 3; k++) { p[k] = at.nbg[k]; p[3 + k] = at.cbg[k]; }  // without normals / colours
  if (at.normals) {
    const float* N = at.normals;
    float v[3];
    for (int k = 0; k < 3; k++) v[k] = lerp3(u, N[3 * c.x + k], N[3 * c.y + k], N[3 * c.z + k]);
    const float len = sqrtf((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]);
    for (int k = 0; k < 3; k++) p[k] = len > 0.f ? v[k] / len : 0.f;
  }
  if (at.colors) {
    const float* Cc = at.colors;
    for (int k = 0; k < 3; k++) p[3 + k] = lerp3(u, Cc[3 * c.x + k], Cc[3 * c.y + k], Cc[3 * c.z + k]);
  }
}

// The antialiasing weight of pixel `self` from its pair with neighbour `other` (horizontal: left/right): the
// occluder o (smaller key) finds the first edge of its face the segment to the far pixel's centre leaves through; if
// that edge is a silhouette edge of the pair's class, at distance t from the occluder's centre, the far pixel moves
// t - 1/2 towards the occluder when t > 1/2 and the occluder 1/2 - t towards the far pixel when t < 1/2.
__device__ float aa_weight(const Mesh& m, const Frame& fr, int view, int vs, const int* __restrict__ opp,
                           const int8_t* __restrict__ facing, unsigned long long kself, unsigned long long kother,
                           int si, int sj, int oi, int oj, bool horizontal) {
  const bool self_occ = kself < kother;
  const unsigned long long ko = self_occ ? kself : kother;
  const int f = (int)(unsigned)ko;
  const int ci = self_occ ? si : oi, cj = self_occ ? sj : oj;  // occluder centre
  const int fi = self_occ ? oi : si, fj = self_occ ? oj : sj;  // far centre
  Hom t[3];
  face_hom(m, fr, view, f, t);
  float bo[3], bf[3];
  const float d = edge_fns(t, (float)ci + 0.5f, (float)cj + 0.5f, bo);
  edge_fns(t, (float)fi + 0.5f, (float)fj + 0.5f, bf);
  int ke = -1;
  float te = 0.f;
  for (int k = 0; k < 3; k++) {
    const bool out_f = d > 0.f ? bf[k] < 0.f : bf[k] > 0.f;
    const bool in_o = d > 0.f ? bo[k] >= 0.f : bo[k] <= 0.f;
    if (!(out_f && in_o)) continue;
    const float tk = bo[k] / (bo[k] - bf[k]);
    if (ke < 0 || tk < te) { ke = k; te = tk; }
  }
  if (ke < 0) return 0.f;
  const Hom& p = t[(ke + 1) % 3];
  const Hom& q = t[(ke + 2) % 3];
  const float a = q.w * p.Y - p.w * q.Y;  // d b / d px
  const float b = p.w * q.X - q.w * p.X;  // d b / d py
  if ((fabsf(a) > fabsf(b)) != horizontal) return 0.f;
  const int nb = opp[3 * f + (ke + 1) % 3];
  const int8_t* fc = facing + (size_t)vs * m.F;
  if (nb >= 0 && fc[nb] == fc[f]) return 0.f;
  if (self_occ) return te < 0.5f ? 0.5f - te : 0.f;
  return te > 0.5f ? te - 0.5f : 0.f;
}

// Per pixel: alpha, normal and colour, each moved by its up-to-four pair weights (left, right, up, down, in this order)
// towards the neighbour's value before antialiasing.
__global__ void antialias_kernel(long long n, Mesh m, Frame fr, int view0, const int* __restrict__ opp,
                                 const int8_t* __restrict__ facing, const unsigned long long* __restrict__ keys,
                                 const float* __restrict__ pre, float* __restrict__ out_alpha,
                                 float* __restrict__ out_normal, float* __restrict__ out_rgb) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const long long hw = (long long)fr.H * fr.W;
  const int vs = (int)(idx / hw);
  const int pix = (int)(idx - vs * hw), j = pix / fr.W, i = pix - j * fr.W;
  const unsigned long long key = keys[idx];
  const float* p = pre + 6 * (size_t)idx;
  const float a0 = key != kNoKey ? 1.f : 0.f;
  float acc[7] = {a0, p[0], p[1], p[2], p[3], p[4], p[5]};
  const int di[4] = {-1, 1, 0, 0}, dj[4] = {0, 0, -1, 1};
  for (int s = 0; s < 4; s++) {
    const int qi = i + di[s], qj = j + dj[s];
    if (qi < 0 || qi >= fr.W || qj < 0 || qj >= fr.H) continue;
    const long long q = idx + (long long)dj[s] * fr.W + di[s];
    const unsigned long long kq = keys[q];
    if ((unsigned)kq == (unsigned)key) continue;  // same face, or both background
    const float wgt = aa_weight(m, fr, view0 + vs, vs, opp, facing, key, kq, i, j, qi, qj, s < 2);
    if (wgt == 0.f) continue;
    const float* pq = pre + 6 * (size_t)q;
    const float aq = kq != kNoKey ? 1.f : 0.f;
    acc[0] = acc[0] + wgt * (aq - a0);
    for (int c = 0; c < 6; c++) acc[1 + c] = acc[1 + c] + wgt * (pq[c] - p[c]);
  }
  const size_t o = (size_t)view0 * hw + idx;
  if (out_alpha) out_alpha[o] = acc[0];
  if (out_normal)
    for (int c = 0; c < 3; c++) out_normal[3 * o + c] = acc[1 + c];
  if (out_rgb)
    for (int c = 0; c < 3; c++) out_rgb[3 * o + c] = acc[4 + c];
}

// The face across each half-edge: the other half-edge of its undirected edge when the edge has exactly two, else -1.
__global__ void opposite_kernel(int n, const uint32_t* __restrict__ heads, const uint32_t* __restrict__ hval,
                                int* __restrict__ opp) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t e = heads[i];
  auto same = [&](int j) { return j >= 0 && j < n && heads[j] == e; };
  int partner = -1;
  if (same(i + 1) && !same(i - 1) && !same(i + 2)) partner = i + 1;
  if (same(i - 1) && !same(i + 1) && !same(i - 2)) partner = i - 1;
  opp[hval[i]] = partner >= 0 ? (int)(hval[partner] / 3) : -1;
}

// Only the buffers MeshScratch::sort_edges uses (faces, half-edge keys and values, edge ids, temp) are carved.
struct Scratch : MeshScratch {
  FaceCheck* chk;
  int* opp;
  unsigned long long *tiles, *keys;
  int8_t* facing;
  float* pre;

  size_t carve(void* base, int V, int F, int H, int W, int views) {
    Carver cv(base);
    const int n = 3 * F, vbits = bits_for(V);
    chk = cv.take<FaceCheck>(1);
    faces = cv.take<int3>(F);
    hkey_in = cv.take<unsigned long long>(n);
    hkey = cv.take<unsigned long long>(n);
    hval_in = cv.take<uint32_t>(n);
    hval = cv.take<uint32_t>(n);
    heads = cv.take<uint32_t>(n);
    opp = cv.take<int>(n);
    const size_t vf = (size_t)views * F, px = (size_t)views * H * W;
    tiles = cv.take<unsigned long long>(vf);
    facing = cv.take<int8_t>(vf);
    keys = cv.take<unsigned long long>(px);
    pre = cv.take<float>(6 * px);
    temp_bytes = 0;
    size_t t = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, t, hkey_in, hkey, hval_in, hval, n, 0, 2 * vbits);
    need(t);
    cub::DeviceScan::InclusiveSum(nullptr, t, heads, heads, n);
    need(t);
    cub::DeviceScan::InclusiveSum(nullptr, t, tiles, tiles, (int)vf);
    need(t);
    carve_temp(cv);
    return cv.bytes();
  }
};

}  // namespace
}  // namespace dgs

using namespace dgs;

extern "C" {

int dgs_mesh_render(const float* vertices, long long num_vertices, const int* faces, long long num_faces,
                    const float* normals, const float* colors, const float* clip, int n_views, int H, int W,
                    float near, const float* normal_bg, const float* color_bg, size_t max_arena_bytes,
                    int* out_face_id, float* out_depth, float* out_alpha, float* out_normal, float* out_rgb,
                    dgs_alloc_fn alloc, void* alloc_user, void* stream) {
  const char* name = "mesh render";
  const int rc0 = check_mesh_input(name, vertices, num_vertices, faces, num_faces,
                                   num_vertices <= 0x7fffffffLL && 3 * num_faces <= 0x7fffffffLL,
                                   "V and 3F must be at most 2^31 - 1");
  if (rc0 != DGS_OK) return rc0;
  DGS_REQUIRE(n_views >= 0, "%s: n_views must be >= 0 (got %d)", name, n_views);
  DGS_REQUIRE(H >= 1 && H <= kMaxSize && W >= 1 && W <= kMaxSize, "%s: H and W must be in [1, %d] (got %d x %d)", name,
              kMaxSize, H, W);
  DGS_REQUIRE(near > 0.f && near < INFINITY, "%s: near must be finite and > 0 (got %g)", name, near);
  DGS_REQUIRE(alloc && (n_views == 0 || clip), "%s: alloc and clip must not be NULL", name);
  DGS_REQUIRE(!out_normal || normals, "%s: a normal map needs vertex normals", name);
  DGS_REQUIRE(!out_rgb || colors, "%s: a colour map needs vertex colours", name);
  if (n_views == 0) return DGS_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int V = (int)num_vertices, F = (int)num_faces;
  // views per chunk: as many as max_arena_bytes holds (at least 1), with (views x faces) and pixels below 2^31
  Scratch s;
  const size_t fixed = s.carve(nullptr, V, F, H, W, 0);
  const size_t per_view = s.carve(nullptr, V, F, H, W, 1) - fixed + 512;
  long long chunk = max_arena_bytes > fixed ? (long long)((max_arena_bytes - fixed) / per_view) : 1;
  chunk = std::max(1LL, std::min<long long>(chunk, n_views));
  chunk = std::max(1LL, std::min(chunk, 0x7fffffffLL / std::max(1LL, std::max((long long)F, (long long)H * W))));
  const int C = (int)chunk;
  void* buf = alloc(s.carve(nullptr, V, F, H, W, C), alloc_user);
  if (!buf) { set_error("%s: scratch allocation failed", name); return DGS_ERR_ALLOC; }
  s.carve(buf, V, F, H, W, C);
  const int3* in_faces = reinterpret_cast<const int3*>(faces);
  FaceCheck h;
  const int rc1 = check_faces(name, vertices, V, in_faces, F, false, nullptr, s.chk, h, st);
  if (rc1 != DGS_OK) return rc1;

  // the face across each half-edge, from the sorted half-edges
  if (F > 0) {
    DGS_CUDA_OK(cudaMemcpyAsync(s.faces, in_faces, (size_t)F * sizeof(int3), cudaMemcpyDeviceToDevice, st));
    DGS_CUDA_OK(s.sort_edges(F, V, st));
    opposite_kernel<<<ceil_div(3 * F, kThreads), kThreads, 0, st>>>(3 * F, s.heads, s.hval, s.opp);
    DGS_POST_LAUNCH();
  }
  const Mesh m{vertices, in_faces, F, clip};
  const Frame fr{W, H, 0.5f * (float)W, 0.5f * (float)H, near, (float)W + kGuard, (float)H + kGuard};
  Attrs at{normals, colors, {0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
  for (int c = 0; c < 3; c++) {
    if (normal_bg) at.nbg[c] = normal_bg[c];
    if (color_bg) at.cbg[c] = color_bg[c];
  }
  for (int v0 = 0; v0 < n_views; v0 += C) {
    const int nv = std::min(C, n_views - v0);
    const long long nvf = (long long)nv * F, npx = (long long)nv * H * W;
    DGS_CUDA_OK(cudaMemsetAsync(s.keys, 0xff, (size_t)npx * sizeof(unsigned long long), st));
    if (nvf > 0) {
      const unsigned g = (unsigned)((nvf + kThreads - 1) / kThreads);
      setup_kernel<<<g, kThreads, 0, st>>>(nvf, m, fr, v0, s.tiles, s.facing);
      DGS_POST_LAUNCH();
      cover_small_kernel<<<g, kThreads, 0, st>>>(nvf, m, fr, v0, s.tiles, s.keys);
      DGS_POST_LAUNCH();
      DGS_CUDA_OK(cub::DeviceScan::InclusiveSum(s.temp, s.temp_bytes, s.tiles, s.tiles, (int)nvf, st));
      unsigned long long total = 0;
      DGS_CUDA_OK(cudaMemcpyAsync(&total, s.tiles + nvf - 1, sizeof(total), cudaMemcpyDeviceToHost, st));
      DGS_CUDA_OK(cudaStreamSynchronize(st));  // the number of tile items sizes the next launch
      if (total) {
        const unsigned g2 = (unsigned)std::min<unsigned long long>((total + kThreads - 1) / kThreads, 1u << 20);
        cover_tiles_kernel<<<g2, kThreads, 0, st>>>(nvf, total, m, fr, v0, s.tiles, s.keys);
        DGS_POST_LAUNCH();
      }
    }
    const unsigned gp = (unsigned)((npx + kThreads - 1) / kThreads);
    resolve_kernel<<<gp, kThreads, 0, st>>>(npx, m, fr, v0, at, s.keys, s.pre, out_face_id, out_depth);
    DGS_POST_LAUNCH();
    if (out_alpha || out_normal || out_rgb) {
      antialias_kernel<<<gp, kThreads, 0, st>>>(npx, m, fr, v0, s.opp, s.facing, s.keys, s.pre, out_alpha, out_normal,
                                                out_rgb);
      DGS_POST_LAUNCH();
    }
  }
  return DGS_OK;
}

}  // extern "C"
