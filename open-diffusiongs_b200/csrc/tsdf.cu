// tsdf.cu -- mesh extraction by TSDF fusion: rendered depth, alpha and colour maps fused into a truncated signed
// distance volume (dgs_tsdf_integrate), its zero crossing marched where it was observed (dgs_tsdf_extract), and vertex
// colours read back from the volume (dgs_tsdf_colors).  Compiled with -fmad=false: every product and sum below is
// rounded on its own, in the order written, and oracle/tsdf.py restates each step operation for operation in numpy fp32.
//
// Volume.  R points per axis at lin = linspace(-1, 1, R) (the opacity field's grid), indexed [x][y][z], with per point
// tsdf_sum fp32, weight int32, rgb_sum fp32 x 3 and rgb_weight int32, all zero before the first view.
//
// Integration, per point p = (lin[x], lin[y], lin[z]) and per view, in view order.  t is the camera centre and c0, c1,
// c2 the columns of the c2w rotation (OpenCV: x right, y down, z forward); d = p - t.
//   xc = (c0.x * d.x + c0.y * d.y) + c0.z * d.z, yc and zc likewise from c1 and c2.  zc <= 0.2 (the rasterizer's near
//     plane): skipped.
//   u = fx * xc / zc + cx, v = fy * yc / zc + cy, each evaluated left to right.  The sample is pixel (floor(u), floor(v)):
//     the rasterizer puts pixel x's centre at pinhole coordinate x + 1/2 (its projection has Pm[0][2] = 2 cx / W - 1 and
//     ndc2Pix subtracts 1/2, and it blends at pxf = x).  Outside the image (u < 0, u >= W, v < 0 or v >= H): skipped.
//   a = alpha[pixel].  a < alpha_thresh (background): tsdf_sum += 1, weight += 1 -- free space is carved.
//   Otherwise depth = D / a (D the accumulated depth) and sdf = depth - zc.  sdf < -trunc: no update.  Else
//     tsdf_sum += min(1, sdf / trunc), weight += 1, and when also sdf < trunc, per channel
//     rgb_sum += (I - (1 - a)) / a (the blend's colour without its white background) and rgb_weight += 1.
// One thread per point holds its four values in registers over the chunk's views, whose cameras are staged in shared
// memory.  Updates go in view order: the volume is the same bits whatever the chunk size, and there are no atomics.
//
// Extraction.  f = -(tsdf_sum / weight) where weight > 0 (0 elsewhere, never read) goes through mesh.cu's marching
// cubes at iso 0 with weight > 0 as the observed mask: a voxel emits triangles only when its 8 corners are observed, and
// an edge a vertex only when it changes sign, both its ends are observed and a voxel containing it is.  Every vertex is
// referenced, no face touches an unobserved point, and faces are oriented outwards (f > 0 is inside the surface).
// Vertices are in index coordinates, as dgs_marching_cubes returns them.
//
// Colours, per vertex position q (in the grid's [-1, 1] frame):
//   g = (q + 1) * s with s = (R - 1) * 0.5, clamped to [0, R - 1]; i0 = min(floor(g), R - 2); t = g - i0 (per axis).
//   Corner c in 0..7 (x = c & 1, y = (c >> 1) & 1, z = c >> 2) weighs w = (wx * wy) * wz, wx = t.x if x else 1 - t.x.
//   Over the corners with rgb_weight > 0, in corner order: acc += w * (rgb_sum / rgb_weight) per channel, wsum += w.
//   rgb = clamp(acc / wsum, 0, 1); white when wsum == 0 (no coloured corner).
#include "mesh_common.cuh"

namespace dgs {
namespace {

constexpr int kCamBatch = 64;  // cameras staged in shared memory at a time
constexpr float kNearZ = 0.2f;  // the rasterizer's NEAR_Z

// Per view: t.xyz, c0.xyz, c1.xyz, c2.xyz, fx, fy, cx, cy.
struct TsdfCam {
  float t[3], c0[3], c1[3], c2[3], fx, fy, cx, cy;
};

__global__ void tsdf_cams_kernel(int n, const float* __restrict__ c2w, const float* __restrict__ fxfycxcy,
                                 TsdfCam* __restrict__ cams) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const float* m = c2w + 16 * k;  // row-major 4 x 4
  TsdfCam c;
  for (int r = 0; r < 3; r++) {
    c.t[r] = m[4 * r + 3];
    c.c0[r] = m[4 * r + 0];
    c.c1[r] = m[4 * r + 1];
    c.c2[r] = m[4 * r + 2];
  }
  c.fx = fxfycxcy[4 * k + 0];
  c.fy = fxfycxcy[4 * k + 1];
  c.cx = fxfycxcy[4 * k + 2];
  c.cy = fxfycxcy[4 * k + 3];
  cams[k] = c;
}

__global__ void __launch_bounds__(kThreads) tsdf_integrate_kernel(
    int n_views, const TsdfCam* __restrict__ cams, int H, int W, const float* __restrict__ image,
    const float* __restrict__ depth, const float* __restrict__ alpha, const float* __restrict__ lin, int R, float trunc,
    float alpha_thresh, float* __restrict__ tsdf_sum, int* __restrict__ weight, float* __restrict__ rgb_sum,
    int* __restrict__ rgb_weight) {
  __shared__ TsdfCam sc[kCamBatch];
  const long long N = (long long)R * R * R;
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  const bool live = i < N;
  const long long ii = live ? i : 0;
  const int x = (int)(ii / ((long long)R * R)), y = (int)((ii / R) % R), z = (int)(ii % R);
  const float px = lin[x], py = lin[y], pz = lin[z];
  float ts = 0.f, r0 = 0.f, r1 = 0.f, r2 = 0.f;
  int w = 0, rw = 0;
  if (live) {
    ts = tsdf_sum[i];
    w = weight[i];
    r0 = rgb_sum[3 * i + 0];
    r1 = rgb_sum[3 * i + 1];
    r2 = rgb_sum[3 * i + 2];
    rw = rgb_weight[i];
  }
  const size_t HW = (size_t)H * W;
  for (int b0 = 0; b0 < n_views; b0 += kCamBatch) {
    const int nb = min(kCamBatch, n_views - b0);
    __syncthreads();
    for (int k = threadIdx.x; k < nb * (int)(sizeof(TsdfCam) / 4); k += kThreads)
      reinterpret_cast<float*>(sc)[k] = reinterpret_cast<const float*>(cams + b0)[k];
    __syncthreads();
    if (!live) continue;
    for (int k = 0; k < nb; k++) {
      const TsdfCam& c = sc[k];
      const float dx = px - c.t[0], dy = py - c.t[1], dz = pz - c.t[2];
      const float zc = (c.c2[0] * dx + c.c2[1] * dy) + c.c2[2] * dz;
      if (zc <= kNearZ) continue;
      const float xc = (c.c0[0] * dx + c.c0[1] * dy) + c.c0[2] * dz;
      const float yc = (c.c1[0] * dx + c.c1[1] * dy) + c.c1[2] * dz;
      const float u = c.fx * xc / zc + c.cx, v = c.fy * yc / zc + c.cy;
      if (!(u >= 0.f && u < (float)W && v >= 0.f && v < (float)H)) continue;
      const int iu = (int)floorf(u), iv = (int)floorf(v);
      const size_t view = (size_t)(b0 + k), pix = (size_t)iv * W + iu;
      const float a = alpha[view * HW + pix];
      if (a < alpha_thresh) {
        ts = ts + 1.f;
        w++;
        continue;
      }
      const float sdf = depth[view * HW + pix] / a - zc;
      if (sdf < -trunc) continue;
      ts = ts + fminf(1.f, sdf / trunc);
      w++;
      if (sdf < trunc) {
        const float* I = image + view * 3 * HW + pix;
        const float bg = 1.f - a;
        r0 = r0 + (I[0] - bg) / a;
        r1 = r1 + (I[HW] - bg) / a;
        r2 = r2 + (I[2 * HW] - bg) / a;
        rw++;
      }
    }
  }
  if (!live) return;
  tsdf_sum[i] = ts;
  weight[i] = w;
  rgb_sum[3 * i + 0] = r0;
  rgb_sum[3 * i + 1] = r1;
  rgb_sum[3 * i + 2] = r2;
  rgb_weight[i] = rw;
}

__global__ void tsdf_field_kernel(long long N, const float* __restrict__ tsdf_sum, const int* __restrict__ weight,
                                  float* __restrict__ f) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= N) return;
  const int w = weight[i];
  f[i] = w > 0 ? -(tsdf_sum[i] / (float)w) : 0.f;
}

__global__ void tsdf_colors_kernel(long long V, const float* __restrict__ verts, int R, const float* __restrict__ rgb_sum,
                                   const int* __restrict__ rgb_weight, float* __restrict__ out) {
  const long long v = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (v >= V) return;
  const float s = (float)(R - 1) * 0.5f, hi = (float)(R - 1);
  int i0[3];
  float t[3];
  for (int k = 0; k < 3; k++) {
    const float g = fminf(fmaxf((verts[3 * v + k] + 1.f) * s, 0.f), hi);
    i0[k] = min((int)floorf(g), R - 2);
    t[k] = g - (float)i0[k];
  }
  float acc[3] = {0.f, 0.f, 0.f}, wsum = 0.f;
  for (int c = 0; c < 8; c++) {
    const int cx = c & 1, cy = (c >> 1) & 1, cz = c >> 2;
    const size_t q = ((size_t)(i0[0] + cx) * R + (i0[1] + cy)) * R + (i0[2] + cz);
    const int rw = rgb_weight[q];
    if (rw <= 0) continue;
    const float wx = cx ? t[0] : 1.f - t[0], wy = cy ? t[1] : 1.f - t[1], wz = cz ? t[2] : 1.f - t[2];
    const float w = (wx * wy) * wz;
    for (int ch = 0; ch < 3; ch++) acc[ch] = acc[ch] + w * (rgb_sum[3 * q + ch] / (float)rw);
    wsum = wsum + w;
  }
  for (int ch = 0; ch < 3; ch++)
    out[3 * v + ch] = wsum == 0.f ? 1.f : fminf(fmaxf(acc[ch] / wsum, 0.f), 1.f);
}

int check_volume(const char* name, int R, const void* a, const void* b, const void* c, const void* d) {
  DGS_REQUIRE(R >= 2 && R <= 512, "%s: resolution must be in [2, 512] (got %d)", name, R);
  DGS_REQUIRE(a && b && c && d, "%s: the four volume arrays must not be NULL", name);
  return DGS_OK;
}

}  // namespace
}  // namespace dgs

using namespace dgs;

extern "C" {

int dgs_tsdf_integrate(int n_views, const float* c2w, const float* fxfycxcy, int H, int W, const float* image,
                       const float* depth, const float* alpha, const float* lin, int resolution, float trunc,
                       float alpha_thresh, float* tsdf_sum, int* weight, float* rgb_sum, int* rgb_weight,
                       dgs_alloc_fn alloc, void* alloc_user, void* stream) {
  const char* name = "tsdf integrate";
  DGS_REQUIRE(n_views >= 0, "%s: n_views must be >= 0 (got %d)", name, n_views);
  DGS_REQUIRE(H >= 1 && W >= 1 && (long long)H * W <= (1LL << 28), "%s: bad image size %d x %d", name, H, W);
  if (int rc = check_volume(name, resolution, tsdf_sum, weight, rgb_sum, rgb_weight)) return rc;
  DGS_REQUIRE(lin && alloc, "%s: lin and alloc must not be NULL", name);
  DGS_REQUIRE(n_views == 0 || (c2w && fxfycxcy && image && depth && alpha),
              "%s: cameras and maps must not be NULL", name);
  DGS_REQUIRE(trunc > 0.f && trunc <= 1e30f, "%s: trunc must be finite and > 0 (got %g)", name, (double)trunc);
  DGS_REQUIRE(alpha_thresh > 0.f && alpha_thresh <= 1.f, "%s: alpha_thresh must be in (0, 1] (got %g)", name,
              (double)alpha_thresh);
  if (n_views == 0) return DGS_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  TsdfCam* cams = reinterpret_cast<TsdfCam*>(alloc(sizeof(TsdfCam) * (size_t)n_views, alloc_user));
  if (!cams) { set_error("%s: scratch allocation failed", name); return DGS_ERR_ALLOC; }
  tsdf_cams_kernel<<<ceil_div(n_views, 64), 64, 0, st>>>(n_views, c2w, fxfycxcy, cams);
  DGS_POST_LAUNCH();
  const long long N = (long long)resolution * resolution * resolution;
  tsdf_integrate_kernel<<<(unsigned)((N + kThreads - 1) / kThreads), kThreads, 0, st>>>(
      n_views, cams, H, W, image, depth, alpha, lin, resolution, trunc, alpha_thresh, tsdf_sum, weight, rgb_sum,
      rgb_weight);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

int dgs_tsdf_extract(const float* tsdf_sum, const int* weight, int resolution, dgs_alloc_fn alloc, void* alloc_user,
                     float** out_vertices, int** out_faces, long long* out_num_vertices, long long* out_num_faces,
                     void* stream) {
  const char* name = "tsdf extract";
  DGS_REQUIRE(resolution >= 2 && resolution <= 512, "%s: resolution must be in [2, 512] (got %d)", name, resolution);
  DGS_REQUIRE(tsdf_sum && weight && alloc && out_vertices && out_faces && out_num_vertices && out_num_faces,
              "%s: the volume, alloc and the four outputs must not be NULL", name);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long N = (long long)resolution * resolution * resolution;
  float* f = reinterpret_cast<float*>(alloc((size_t)N * sizeof(float), alloc_user));
  if (!f) { set_error("%s: scratch allocation failed", name); return DGS_ERR_ALLOC; }
  tsdf_field_kernel<<<(unsigned)((N + kThreads - 1) / kThreads), kThreads, 0, st>>>(N, tsdf_sum, weight, f);
  DGS_POST_LAUNCH();
  return marching_cubes(name, f, weight, resolution, resolution, resolution, 0.f, alloc, alloc_user, out_vertices,
                        out_faces, out_num_vertices, out_num_faces, st);
}

int dgs_tsdf_colors(const float* rgb_sum, const int* rgb_weight, int resolution, const float* vertices,
                    long long num_vertices, float* out_rgb, void* stream) {
  const char* name = "tsdf colors";
  DGS_REQUIRE(resolution >= 2 && resolution <= 512, "%s: resolution must be in [2, 512] (got %d)", name, resolution);
  if (int rc = check_mesh_input(name, vertices, num_vertices, nullptr, 0, num_vertices < (1LL << 40), "at most 2^40"))
    return rc;
  DGS_REQUIRE(rgb_sum && rgb_weight && (num_vertices == 0 || out_rgb), "%s: the volume and out_rgb must not be NULL",
              name);
  if (num_vertices == 0) return DGS_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  tsdf_colors_kernel<<<(unsigned)((num_vertices + kThreads - 1) / kThreads), kThreads, 0, st>>>(
      num_vertices, vertices, resolution, rgb_sum, rgb_weight, out_rgb);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

}  // extern "C"
