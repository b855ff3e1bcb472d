// ssim.cu -- SSIM (11-tap Gaussian window, sigma 1.5) per image, its gradient w.r.t. the first image, and PSNR.
//
//   S = (2 mx my + C1)(2 sxy + C2) / ((mx^2 + my^2 + C1)(sx^2 + sy^2 + C2)),   ssim[n] = mean over 3 channels and the
//   (H-10) x (W-10) valid pixels of S
//
// with the moments mx = W*x, my = W*y, sx^2 = k (W*(x x) - mx^2), sy^2 = k (W*(y y) - my^2), sxy = k (W*(x y) - mx my)
// taken by the valid separable 11 x 11 window W.  k = 1 is pytorch_msssim's SSIM (the training loss); k = 121/120 is
// skimage's structural_similarity(gaussian_weights=True), whose reflect-padded filter only reaches the border in the
// 5-pixel frame it crops, so it is the same valid-window mean.
//
// Forward: one CTA per (image, 32 x 32 output tile), all 3 channels.  Each channel's tile plus its 10-pixel halo of x
// and y is read into shared memory with plain coalesced loads (chosen for simplicity; no TMA variant has been measured), the
// horizontal 11-tap pass writes the 5 moments of every halo row to shared memory, and the vertical pass accumulates in
// registers.  Each CTA writes one partial sum of S (and, for PSNR, of the clamped squared differences of the pixels it
// owns: border tiles own the 5-pixel frame) in a fixed warp / CTA tree order; a second kernel adds each image's partials
// in fp64 in tile order.  A training forward also stores, per channel and valid pixel, the coefficients
//   alpha = dS/dmx = S (2my/A1 - 2mx/B1 + 2k mx/B2 - 2k my/A2),  beta = dS/dE[xx] = -k S/B2,  gamma = dS/dE[xy] = 2k S/A2
// (A1, A2, B1, B2 the four factors of S above; formed without dividing by A1 or A2, which may be 0), and the backward
// is one stencil over them:
//   dx(p) = s [(W^T alpha)(p) + 2 x(p) (W^T beta)(p) + y(p) (W^T gamma)(p)],   s = dout / (3 (H-10)(W-10)).
// No atomics: every result is independent of n and of whether a training state is written, bit for bit.
#include "dgs_internal.h"
#include "sm90_ptx.cuh"

namespace dgs {
namespace {

constexpr int WIN = 11, HALO = WIN - 1, RAD = HALO / 2;
constexpr int TH = 32, TW = 32, LH = TH + HALO, LW = TW + HALO, NT = 256;

struct Win { float g[WIN]; };

using ptx::warp_sum;

// partial[(img * tiles + tile) * 2 + {0, 1}] = sum of S over the tile's valid pixels and 3 channels, and (want_psnr)
// the sum of (clamp(x) - clamp(y))^2 over the image pixels the tile owns.  maps (training): [n, 3 ch, 3, Hv, Wv].
__global__ void __launch_bounds__(NT) ssim_fwd_kernel(const float* __restrict__ x, const float* __restrict__ y, int H,
                                                      int W, Win win, float C1, float C2, float k, int want_psnr,
                                                      float* __restrict__ partial, float* __restrict__ maps) {
  __shared__ float sx[LH][LW], sy[LH][LW];
  __shared__ float hs[5][LH][TW];
  __shared__ float red[2][NT / 32];
  const int tid = threadIdx.x, img = blockIdx.z;
  const int oy = blockIdx.y * TH, ox = blockIdx.x * TW;
  const int Hv = H - HALO, Wv = W - HALO;
  const size_t HW = (size_t)H * W, HWv = (size_t)Hv * Wv;
  // image pixels this tile owns for PSNR: rows [r0, r1), cols [c0, c1) -- all inside the loaded halo tile
  const int r0 = blockIdx.y == 0 ? 0 : oy + RAD, r1 = blockIdx.y == gridDim.y - 1 ? H : oy + TH + RAD;
  const int c0 = blockIdx.x == 0 ? 0 : ox + RAD, c1 = blockIdx.x == gridDim.x - 1 ? W : ox + TW + RAD;
  float s_acc = 0.f, e_acc = 0.f;
  for (int ch = 0; ch < 3; ch++) {
    const float* xc = x + ((size_t)img * 3 + ch) * HW;
    const float* yc = y + ((size_t)img * 3 + ch) * HW;
    __syncthreads();  // the previous channel is done with sx / sy / hs
    for (int i = tid; i < LH * LW; i += NT) {
      const int r = i / LW, c = i - r * LW, gy = oy + r, gx = ox + c;
      const bool in = gy < H && gx < W;
      const float a = in ? xc[(size_t)gy * W + gx] : 0.f, b = in ? yc[(size_t)gy * W + gx] : 0.f;
      sx[r][c] = a;
      sy[r][c] = b;
      if (want_psnr && gy >= r0 && gy < r1 && gx >= c0 && gx < c1) {
        const float d = __fsub_rn(fminf(fmaxf(a, 0.f), 1.f), fminf(fmaxf(b, 0.f), 1.f));
        e_acc = __fmaf_rn(d, d, e_acc);
      }
    }
    __syncthreads();
    for (int i = tid; i < LH * TW; i += NT) {
      const int r = i / TW, c = i - r * TW;
      float m[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int t = 0; t < WIN; t++) {
        const float a = sx[r][c + t], b = sy[r][c + t], w = win.g[t];
        m[0] = __fmaf_rn(w, a, m[0]);
        m[1] = __fmaf_rn(w, b, m[1]);
        m[2] = __fmaf_rn(w, __fmul_rn(a, a), m[2]);
        m[3] = __fmaf_rn(w, __fmul_rn(b, b), m[3]);
        m[4] = __fmaf_rn(w, __fmul_rn(a, b), m[4]);
      }
#pragma unroll
      for (int j = 0; j < 5; j++) hs[j][r][c] = m[j];
    }
    __syncthreads();
    for (int i = tid; i < TH * TW; i += NT) {
      const int r = i / TW, c = i - r * TW;
      if (oy + r >= Hv || ox + c >= Wv) continue;
      float m[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int t = 0; t < WIN; t++) {
        const float w = win.g[t];
#pragma unroll
        for (int j = 0; j < 5; j++) m[j] = __fmaf_rn(w, hs[j][r + t][c], m[j]);
      }
      // explicit rounding: the loop may be specialised on `maps`, and S must not depend on which copy runs
      const float mx = m[0], my = m[1];
      const float mx2 = __fmul_rn(mx, mx), my2 = __fmul_rn(my, my), mxy = __fmul_rn(mx, my);
      const float vx = __fmul_rn(k, __fsub_rn(m[2], mx2)), vy = __fmul_rn(k, __fsub_rn(m[3], my2));
      const float vxy = __fmul_rn(k, __fsub_rn(m[4], mxy));
      const float A1 = __fadd_rn(__fmul_rn(2.f, mxy), C1), A2 = __fadd_rn(__fmul_rn(2.f, vxy), C2);
      const float B1 = __fadd_rn(__fadd_rn(mx2, my2), C1), B2 = __fadd_rn(__fadd_rn(vx, vy), C2);
      const float l = __fdiv_rn(A1, B1), cs = __fdiv_rn(A2, B2);
      const float S = __fmul_rn(l, cs);
      s_acc = __fadd_rn(s_acc, S);
      if (maps) {
        // alpha and gamma with S/A1 = cs/B1 and S/A2 = l/B2 substituted: B1 >= C1 > 0 and B2 ~ C2 > 0, while A1 or A2
        // may round to 0 (then S = 0 and S/A2 would be 0 * inf)
        const float alpha = 2.f * (my * cs - mx * S) / B1 + 2.f * k * (mx * S - my * l) / B2;
        const float beta = -k * S / B2, gamma = 2.f * k * l / B2;
        float* mp = maps + ((size_t)img * 3 + ch) * 3 * HWv + (size_t)(oy + r) * Wv + (ox + c);
        mp[0] = alpha;
        mp[HWv] = beta;
        mp[2 * HWv] = gamma;
      }
    }
  }
  s_acc = warp_sum(s_acc);
  e_acc = warp_sum(e_acc);
  if ((tid & 31) == 0) {
    red[0][tid >> 5] = s_acc;
    red[1][tid >> 5] = e_acc;
  }
  __syncthreads();
  if (tid == 0) {
    float s = 0.f, e = 0.f;
#pragma unroll
    for (int w = 0; w < NT / 32; w++) {
      s += red[0][w];
      e += red[1][w];
    }
    const size_t slot = ((size_t)img * gridDim.x * gridDim.y + (size_t)blockIdx.y * gridDim.x + blockIdx.x) * 2;
    partial[slot] = s;
    partial[slot + 1] = e;
  }
}

// one block per image: the tiles' partial sums in fp64, in a fixed order -> ssim[img], psnr[img] (if psnr)
__global__ void __launch_bounds__(NT) ssim_finalize_kernel(const float* __restrict__ partial, int tiles, double inv_valid,
                                                           double inv_pixels, float* __restrict__ ssim,
                                                           float* __restrict__ psnr) {
  __shared__ double red[2][NT];
  const float* p = partial + (size_t)blockIdx.x * tiles * 2;
  double s = 0.0, e = 0.0;
  for (int t = threadIdx.x; t < tiles; t += NT) {
    s += (double)p[2 * t];
    e += (double)p[2 * t + 1];
  }
  red[0][threadIdx.x] = s;
  red[1][threadIdx.x] = e;
  __syncthreads();
  for (int o = NT / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      red[0][threadIdx.x] += red[0][threadIdx.x + o];
      red[1][threadIdx.x] += red[1][threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    ssim[blockIdx.x] = (float)(red[0][0] * inv_valid);
    if (psnr) psnr[blockIdx.x] = (float)(-10.0 * log10(red[1][0] * inv_pixels));  // mse 0 -> +inf
  }
}

// d_x over one 32 x 32 tile of image pixels: the transposed stencil of the three coefficient maps (zero outside the
// valid domain), then dx = s (W^T alpha + 2 x W^T beta + y W^T gamma).
__global__ void __launch_bounds__(NT) ssim_bwd_kernel(const float* __restrict__ x, const float* __restrict__ y,
                                                      const float* __restrict__ maps, const float* __restrict__ dout,
                                                      int H, int W, Win win, float* __restrict__ dx) {
  __shared__ float sm[3][LH][LW];
  __shared__ float hs[3][LH][TW];
  const int tid = threadIdx.x, img = blockIdx.z;
  const int py0 = blockIdx.y * TH, px0 = blockIdx.x * TW;
  const int Hv = H - HALO, Wv = W - HALO;
  const size_t HW = (size_t)H * W, HWv = (size_t)Hv * Wv;
  const float s = dout[img] / (3.f * (float)Hv * (float)Wv);
  for (int ch = 0; ch < 3; ch++) {
    const float* mp = maps + ((size_t)img * 3 + ch) * 3 * HWv;
    __syncthreads();
    // map rows [py0 - 10, py0 + TH), cols [px0 - 10, px0 + TW)
    for (int i = tid; i < LH * LW; i += NT) {
      const int r = i / LW, c = i - r * LW, qy = py0 - HALO + r, qx = px0 - HALO + c;
      const bool in = qy >= 0 && qy < Hv && qx >= 0 && qx < Wv;
      const size_t q = in ? (size_t)qy * Wv + qx : 0;
#pragma unroll
      for (int j = 0; j < 3; j++) sm[j][r][c] = in ? mp[j * HWv + q] : 0.f;
    }
    __syncthreads();
    // (W^T m)(py, px) = sum_{u,v} g[10-u] g[10-v] m(py - 10 + u, px - 10 + v): smem row r + u, col c + v
    for (int i = tid; i < LH * TW; i += NT) {
      const int r = i / TW, c = i - r * TW;
      float a[3] = {0.f, 0.f, 0.f};
#pragma unroll
      for (int v = 0; v < WIN; v++) {
        const float w = win.g[HALO - v];
#pragma unroll
        for (int j = 0; j < 3; j++) a[j] += w * sm[j][r][c + v];
      }
#pragma unroll
      for (int j = 0; j < 3; j++) hs[j][r][c] = a[j];
    }
    __syncthreads();
    for (int i = tid; i < TH * TW; i += NT) {
      const int r = i / TW, c = i - r * TW, py = py0 + r, px = px0 + c;
      if (py >= H || px >= W) continue;
      float a[3] = {0.f, 0.f, 0.f};
#pragma unroll
      for (int u = 0; u < WIN; u++) {
        const float w = win.g[HALO - u];
#pragma unroll
        for (int j = 0; j < 3; j++) a[j] += w * hs[j][r + u][c];
      }
      const size_t o = ((size_t)img * 3 + ch) * HW + (size_t)py * W + px;
      dx[o] = s * (a[0] + 2.f * x[o] * a[1] + y[o] * a[2]);
    }
  }
}

Win make_window() {
  double g[WIN], sum = 0.0;
  for (int i = 0; i < WIN; i++) {
    const double d = i - RAD;
    g[i] = exp(-d * d / (2.0 * 1.5 * 1.5));
    sum += g[i];
  }
  Win w;
  for (int i = 0; i < WIN; i++) w.g[i] = (float)(g[i] / sum);
  return w;
}

inline int tiles_x(int W) { return ceil_div(W - HALO, TW); }
inline int tiles_y(int H) { return ceil_div(H - HALO, TH); }
inline bool shape_ok(int n, int H, int W) { return n > 0 && H >= WIN && W >= WIN; }

int check_shape(const char* fn, int n, int H, int W) {
  DGS_REQUIRE(n > 0 && n <= 65535, "%s: need n > 0 and n <= 65535 (got %d)", fn, n);
  DGS_REQUIRE(H >= WIN && W >= WIN, "%s: H and W must be at least 11, the window size (got %dx%d)", fn, H, W);
  return DGS_OK;
}

}  // namespace
}  // namespace dgs

using namespace dgs;

extern "C" {

size_t dgs_ssim_workspace_bytes(int n, int H, int W) {
  if (!shape_ok(n, H, W)) return 0;
  Carver cv(nullptr);
  cv.take<float>((size_t)n * tiles_x(W) * tiles_y(H) * 2);
  return cv.bytes();
}

size_t dgs_ssim_state_bytes(int n, int H, int W) {
  if (!shape_ok(n, H, W)) return 0;
  Carver cv(nullptr);
  cv.take<float>((size_t)n * 9 * (H - HALO) * (W - HALO));
  return cv.bytes();
}

int dgs_ssim_forward(int n, int H, int W, const float* x, const float* y, float data_range, int sample_covariance,
                     float* ssim, float* psnr, void* state, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_shape("ssim forward", n, H, W);
  if (rc) return rc;
  DGS_REQUIRE(x && y && ssim, "ssim forward: x, y and ssim must not be NULL");
  DGS_REQUIRE(data_range > 0.f, "ssim forward: data_range must be > 0 (got %g)", (double)data_range);
  const size_t need = dgs_ssim_workspace_bytes(n, H, W);
  DGS_REQUIRE(workspace != nullptr && workspace_bytes >= need, "ssim forward: workspace too small (%zu bytes, need %zu)",
              workspace_bytes, need);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const double R = data_range;
  const float C1 = (float)((0.01 * R) * (0.01 * R)), C2 = (float)((0.03 * R) * (0.03 * R));
  const float k = sample_covariance ? (float)(121.0 / 120.0) : 1.f;
  const dim3 grid(tiles_x(W), tiles_y(H), n);
  float* partial = reinterpret_cast<float*>(workspace);
  ssim_fwd_kernel<<<grid, NT, 0, st>>>(x, y, H, W, make_window(), C1, C2, k, psnr != nullptr, partial,
                                       reinterpret_cast<float*>(state));
  DGS_POST_LAUNCH();
  const double valid = 3.0 * (H - HALO) * (double)(W - HALO), pixels = 3.0 * H * (double)W;
  ssim_finalize_kernel<<<n, NT, 0, st>>>(partial, (int)(grid.x * grid.y), 1.0 / valid, 1.0 / pixels, ssim, psnr);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

int dgs_ssim_backward(int n, int H, int W, const float* x, const float* y, const void* state, const float* dout,
                      float* d_x, void* stream) {
  int rc = check_shape("ssim backward", n, H, W);
  if (rc) return rc;
  DGS_REQUIRE(state != nullptr, "ssim backward: state is NULL (the forward must be given a training state)");
  DGS_REQUIRE(x && y && dout && d_x, "ssim backward: x, y, dout and d_x must not be NULL");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const dim3 grid(ceil_div(W, TW), ceil_div(H, TH), n);
  ssim_bwd_kernel<<<grid, NT, 0, st>>>(x, y, reinterpret_cast<const float*>(state), dout, H, W, make_window(), d_x);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

}  // extern "C"
