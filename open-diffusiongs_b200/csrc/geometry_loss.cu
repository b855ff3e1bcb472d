// geometry_loss.cu -- the two geometry terms of the training loss on the pixel-aligned Gaussian centres
// img [B, V, 3, H, W] (diffusionGS/utils/losses.py:286-291, 323-364), and their gradient w.r.t. img.
//
//   dist = |img - o|,  per view (b, v): mean and unbiased std of dist over its H W pixels,
//   trgt = (dist - mean) / (std + 1e-8) * 0.5 + |o|           (detached; |o| per pixel)
//   pointsdist[b] = mean over (v, h, w) of (dist - trgt)^2
//   l2_xyz = sum (img m - gt m)^2 / sum m                       (m [B, V, 1, H, W] broadcast over the 3 channels)
//
// Per-pixel arithmetic is fp32 as in the reference; every sum is fp64.  Each view is cut into PARTS CTAs that stride over
// its pixels, so a CTA's pixels, and the order in which it adds them, depend only on (H, W).  Pass 1 writes per-CTA
// partials of the shifted distance moments (shifted by the view's first distance: a constant view sums exact zeros)
// and of the masked residual / mask sums; a one-warp kernel turns each view's partials into (mean, std); pass 2 writes
// per-CTA partials of (dist - trgt)^2; the last kernel adds each sample's partials in a fixed order.  No atomics: the
// results are the same bits on every run, and pointsdist[b] does not depend on the other samples.
//
// Backward, one thread per pixel:
//   d_img = g_pd[b] 2 (dist - trgt) / (V H W) (img - o) / dist  +  g_xyz 2 m (img m - gt m) / sum m
// with the pointsdist part 0 where dist == 0 (torch's norm backward).
#include "dgs_internal.h"

namespace dgs {
namespace {

constexpr int NT = 256, PARTS = 64;

__device__ __forceinline__ float pixel_dist(const float* img, const float* o, size_t i, size_t plane) {
  const float x = __fsub_rn(img[i], o[i]), y = __fsub_rn(img[i + plane], o[i + plane]);
  const float z = __fsub_rn(img[i + 2 * plane], o[i + 2 * plane]);
  return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
}

__device__ __forceinline__ float pixel_target(float dist, float mean, float std_, const float* o, size_t i, size_t plane) {
  const float n = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(o[i], o[i]), __fmul_rn(o[i + plane], o[i + plane])),
                                       __fmul_rn(o[i + 2 * plane], o[i + 2 * plane])));
  return __fadd_rn(__fmul_rn(__fdiv_rn(__fsub_rn(dist, mean), __fadd_rn(std_, 1e-8f)), 0.5f), n);
}

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// the CTA's K sums in a fixed warp / CTA tree order -> out[0..K) (thread 0)
template <int K>
__device__ __forceinline__ void block_sum_f64(double (&v)[K], double* out) {
  __shared__ double red[K][NT / 32];
#pragma unroll
  for (int k = 0; k < K; k++) v[k] = warp_sum_f64(v[k]);
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < K; k++) red[k][threadIdx.x >> 5] = v[k];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < K; k++) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < NT / 32; w++) s += red[k][w];
      out[k] = s;
    }
  }
}

// part1[(bv * PARTS + part) * 4 + {0..3}] = sum (dist - shift), sum (dist - shift)^2, sum (img m - gt m)^2, sum m
__global__ void __launch_bounds__(NT) geo_moments_kernel(const float* __restrict__ img, const float* __restrict__ o,
                                                         const float* __restrict__ gt, const float* __restrict__ m,
                                                         int HW, int want_pd, double* __restrict__ part1) {
  const int bv = blockIdx.y;
  const size_t plane = (size_t)HW, base = (size_t)bv * 3 * plane;
  const float* I = img + base;
  const float* O = o + base;
  const float shift = want_pd ? pixel_dist(I, O, 0, plane) : 0.f;
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (int i = blockIdx.x * NT + threadIdx.x; i < HW; i += PARTS * NT) {
    if (want_pd) {
      const double e = (double)pixel_dist(I, O, i, plane) - (double)shift;
      acc[0] += e;
      acc[1] += e * e;
    }
    if (gt) {
      const float w = m[(size_t)bv * plane + i];
#pragma unroll
      for (int c = 0; c < 3; c++) {
        const float r = __fsub_rn(__fmul_rn(I[c * plane + i], w), __fmul_rn(gt[base + c * plane + i], w));
        acc[2] += (double)__fmul_rn(r, r);
      }
      acc[3] += (double)w;
    }
  }
  block_sum_f64<4>(acc, part1 + ((size_t)bv * PARTS + blockIdx.x) * 4);
}

// one warp per view: stats[bv] = (mean, unbiased std) of dist, in fp32
__global__ void __launch_bounds__(32) geo_view_stats_kernel(const float* __restrict__ img, const float* __restrict__ o,
                                                            int HW, const double* __restrict__ part1,
                                                            float* __restrict__ stats) {
  const int bv = blockIdx.x, lane = threadIdx.x;
  const double* p = part1 + (size_t)bv * PARTS * 4;
  double s1 = 0.0, s2 = 0.0;
  for (int k = lane; k < PARTS; k += 32) {
    s1 += p[4 * k];
    s2 += p[4 * k + 1];
  }
  s1 = warp_sum_f64(s1);
  s2 = warp_sum_f64(s2);
  if (lane == 0) {
    const size_t base = (size_t)bv * 3 * HW;
    const double n = (double)HW, shift = (double)pixel_dist(img + base, o + base, 0, HW);
    const double var = (s2 - s1 * s1 / n) / (n - 1.0);  // H W == 1: 0 / 0 = NaN, as torch.std
    stats[2 * bv] = (float)(shift + s1 / n);
    stats[2 * bv + 1] = (float)sqrt(var < 0.0 ? 0.0 : var);
  }
}

// part2[bv * PARTS + part] = sum (dist - trgt)^2
__global__ void __launch_bounds__(NT) geo_residual_kernel(const float* __restrict__ img, const float* __restrict__ o,
                                                          int HW, const float* __restrict__ stats,
                                                          double* __restrict__ part2) {
  const int bv = blockIdx.y;
  const size_t plane = (size_t)HW, base = (size_t)bv * 3 * plane;
  const float* I = img + base;
  const float* O = o + base;
  const float mean = stats[2 * bv], std_ = stats[2 * bv + 1];
  double acc[1] = {0.0};
  for (int i = blockIdx.x * NT + threadIdx.x; i < HW; i += PARTS * NT) {
    const float d = pixel_dist(I, O, i, plane);
    const float r = __fsub_rn(d, pixel_target(d, mean, std_, O, i, plane));
    acc[0] += (double)__fmul_rn(r, r);
  }
  block_sum_f64<1>(acc, part2 + (size_t)bv * PARTS + blockIdx.x);
}

// blocks 0..nb_pd-1: pointsdist[b] from sample b's V * PARTS partials; the last block (if l2_xyz): sum r^2 / sum m over
// every view, and sum m into msum for the backward
__global__ void __launch_bounds__(NT) geo_finalize_kernel(const double* __restrict__ part1,
                                                          const double* __restrict__ part2, int nb_pd, int BV, int V,
                                                          double inv_count, float* __restrict__ pointsdist,
                                                          float* __restrict__ l2_xyz, float* __restrict__ msum) {
  double acc[2] = {0.0, 0.0};
  if ((int)blockIdx.x < nb_pd) {
    const double* p = part2 + (size_t)blockIdx.x * V * PARTS;
    for (int k = threadIdx.x; k < V * PARTS; k += NT) acc[0] += p[k];
  } else {
    for (int k = threadIdx.x; k < BV * PARTS; k += NT) {
      acc[0] += part1[4 * (size_t)k + 2];
      acc[1] += part1[4 * (size_t)k + 3];
    }
  }
  __shared__ double out[2];
  block_sum_f64<2>(acc, out);
  if (threadIdx.x == 0) {
    if ((int)blockIdx.x < nb_pd) {
      pointsdist[blockIdx.x] = (float)(out[0] * inv_count);
    } else {
      *l2_xyz = (float)(out[0] / out[1]);  // an all-zero mask: 0 / 0 = NaN, as in the reference
      *msum = (float)out[1];
    }
  }
}

__global__ void __launch_bounds__(NT) geo_backward_kernel(const float* __restrict__ img, const float* __restrict__ o,
                                                          const float* __restrict__ gt, const float* __restrict__ m,
                                                          int V, int HW, const float* __restrict__ stats,
                                                          const float* __restrict__ g_pd,
                                                          const float* __restrict__ g_xyz, float inv_count,
                                                          float* __restrict__ d_img) {
  const int i = blockIdx.x * NT + threadIdx.x;
  if (i >= HW) return;
  const int bv = blockIdx.y;
  const size_t plane = (size_t)HW, base = (size_t)bv * 3 * plane;
  const float* I = img + base;
  float g[3] = {0.f, 0.f, 0.f};
  if (g_pd) {
    const float* O = o + base;
    const float d = pixel_dist(I, O, i, plane);
    if (d != 0.f) {
      const float t = pixel_target(d, stats[2 * bv], stats[2 * bv + 1], O, i, plane);
      const float coef = 2.f * (d - t) * (g_pd[bv / V] * inv_count) / d;
#pragma unroll
      for (int c = 0; c < 3; c++) g[c] = coef * (I[c * plane + i] - O[c * plane + i]);
    }
  }
  if (g_xyz) {
    const float w = m[(size_t)bv * plane + i];
    const float s = 2.f * (*g_xyz / stats[2 * (size_t)gridDim.y]) * w;  // stats[2 B V] = sum m
#pragma unroll
    for (int c = 0; c < 3; c++) g[c] += s * (I[c * plane + i] * w - gt[base + c * plane + i] * w);
  }
#pragma unroll
  for (int c = 0; c < 3; c++) d_img[base + c * plane + i] = g[c];
}

int check_shape(const char* fn, int B, int V, int H, int W) {
  DGS_REQUIRE(B > 0 && V > 0 && H > 0 && W > 0, "%s: B, V, H and W must be > 0 (got %d, %d, %d, %d)", fn, B, V, H, W);
  DGS_REQUIRE((long long)B * V <= 65535, "%s: B * V must be <= 65535 (got %lld)", fn, (long long)B * V);
  DGS_REQUIRE((long long)H * W <= (1LL << 30), "%s: H * W must be <= 2^30 (got %lld)", fn, (long long)H * W);
  return DGS_OK;
}

}  // namespace
}  // namespace dgs

using namespace dgs;

extern "C" {

size_t dgs_geometry_loss_workspace_bytes(int B, int V) {
  if (B <= 0 || V <= 0) return 0;
  Carver cv(nullptr);
  cv.take<double>((size_t)B * V * PARTS * 4);
  cv.take<double>((size_t)B * V * PARTS);
  return cv.bytes();
}

int dgs_geometry_loss_forward(int B, int V, int H, int W, const float* img_xyz, const float* ray_o, const float* gt_xyz,
                              const float* masks, float* pointsdist, float* l2_xyz, float* state, void* workspace,
                              size_t workspace_bytes, void* stream) {
  int rc = check_shape("geometry loss forward", B, V, H, W);
  if (rc) return rc;
  DGS_REQUIRE(img_xyz && state, "geometry loss forward: img_xyz and state must not be NULL");
  DGS_REQUIRE(!pointsdist || ray_o, "geometry loss forward: pointsdist needs ray_o");
  DGS_REQUIRE(!l2_xyz || (gt_xyz && masks), "geometry loss forward: l2_xyz needs gt_xyz and masks");
  const size_t need = dgs_geometry_loss_workspace_bytes(B, V);
  DGS_REQUIRE(workspace != nullptr && workspace_bytes >= need,
              "geometry loss forward: workspace too small (%zu bytes, need %zu)", workspace_bytes, need);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int BV = B * V, HW = H * W;
  Carver cv(workspace);
  double* part1 = cv.take<double>((size_t)BV * PARTS * 4);
  double* part2 = cv.take<double>((size_t)BV * PARTS);
  const dim3 grid(PARTS, BV);
  const bool pd = pointsdist != nullptr, xyz = l2_xyz != nullptr;
  if (!pd && !xyz) return DGS_OK;
  geo_moments_kernel<<<grid, NT, 0, st>>>(img_xyz, ray_o, xyz ? gt_xyz : nullptr, masks, HW, pd, part1);
  DGS_POST_LAUNCH();
  if (pd) {
    geo_view_stats_kernel<<<BV, 32, 0, st>>>(img_xyz, ray_o, HW, part1, state);
    DGS_POST_LAUNCH();
    geo_residual_kernel<<<grid, NT, 0, st>>>(img_xyz, ray_o, HW, state, part2);
    DGS_POST_LAUNCH();
  }
  const int nb_pd = pd ? B : 0;
  geo_finalize_kernel<<<nb_pd + (xyz ? 1 : 0), NT, 0, st>>>(part1, part2, nb_pd, BV, V, 1.0 / ((double)V * HW),
                                                            pointsdist, l2_xyz, state + 2 * (size_t)BV);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

int dgs_geometry_loss_backward(int B, int V, int H, int W, const float* img_xyz, const float* ray_o, const float* gt_xyz,
                               const float* masks, const float* state, const float* g_pointsdist, const float* g_l2_xyz,
                               float* d_img_xyz, void* stream) {
  int rc = check_shape("geometry loss backward", B, V, H, W);
  if (rc) return rc;
  DGS_REQUIRE(img_xyz && state && d_img_xyz, "geometry loss backward: img_xyz, state and d_img_xyz must not be NULL");
  DGS_REQUIRE(!g_pointsdist || ray_o, "geometry loss backward: g_pointsdist needs ray_o");
  DGS_REQUIRE(!g_l2_xyz || (gt_xyz && masks), "geometry loss backward: g_l2_xyz needs gt_xyz and masks");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int HW = H * W;
  const dim3 grid(ceil_div(HW, NT), B * V);
  geo_backward_kernel<<<grid, NT, 0, st>>>(img_xyz, ray_o, gt_xyz, masks, V, HW, state, g_pointsdist, g_l2_xyz,
                                           (float)(1.0 / ((double)V * HW)), d_img_xyz);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

}  // extern "C"
