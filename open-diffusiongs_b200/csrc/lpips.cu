// lpips.cu -- the LPIPS-VGG perceptual distance (lpips 0.1, net="vgg", eval mode) and its gradient w.r.t. the first input.
//
//   d[n] = sum_k mean_hw sum_c lin_k[c] (f0 - f1)^2,   f = a / (sqrt(sum_c a^2) + 1e-10)
//
// a = the post-ReLU VGG16 activations relu1_2, relu2_2, relu3_3, relu4_3, relu5_3 of the ScalingLayer-normalised
// inputs (x - shift) / scale.  Activations are NHWC bf16.  Each 3x3 convolution is one call of the wgmma GEMM
// (gemm_sm90.cu) on a materialised im2col operand: M = pixels, N = C_out, K = 9 C_in laid out (ky, kx, c), with the
// bias + ReLU + bf16 rounding fused into the GEMM epilogue (EPI_BIAS_RELU_BF16).  conv1_1 reads its 3 input channels
// padded to 8 (K = 72).
//
// Backward: the distance is one scalar per image, so the forward already writes G_k = d d[n] / d a0 at every tap (fp32)
// and the backward only scales it by dout[n].  Walking the convolutions in reverse, the gather that builds the next
// im2col operand forms dz = (da + dout G_k) * [a > 0] (rounded to bf16) while it reads, and da of the layer below is
// one more GEMM against the flipped, transposed weights Wt[c_in, (ky, kx, c_out)] = W[c_out, c_in, 2-ky, 2-kx]
// (fp32 output).  The max-pool backward sends each gradient to the first maximum of its window in row-major order, as
// torch's max_pool2d does.  No atomics anywhere: the results do not depend on the chunking or the batch size.
#include <cuda_bf16.h>

#include "dgs_internal.h"
#include "dit_kernels.h"
#include "sm90_ptx.cuh"

namespace dgs {
namespace {

using namespace ptx;

struct ConvSpec { int cin, cout, level, tap; bool pool_before; };
constexpr int NCONV = 13, NTAP = 5, COL_K_MAX = 9 * 64, WT0_ROWS = 32;
// torchvision vgg16().features[0:30]: conv indices 0,2 | 5,7 | 10,12,14 | 17,19,21 | 24,26,28; conv1_1's C_in padded to 8
constexpr ConvSpec kConv[NCONV] = {
    {8, 64, 0, -1, false},    {64, 64, 0, 0, false},
    {64, 128, 1, -1, true},   {128, 128, 1, 1, false},
    {128, 256, 2, -1, true},  {256, 256, 2, -1, false}, {256, 256, 2, 2, false},
    {256, 512, 3, -1, true},  {512, 512, 3, -1, false}, {512, 512, 3, 3, false},
    {512, 512, 4, -1, true},  {512, 512, 4, -1, false}, {512, 512, 4, 4, false}};
constexpr int kTapConv[NTAP] = {1, 3, 6, 9, 12};

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const float2 t = __bfloat1622float2(h[i]);
    f[2 * i] = t.x; f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  return make_uint4(pack2_bf16(f[0], f[1]), pack2_bf16(f[2], f[3]), pack2_bf16(f[4], f[5]), pack2_bf16(f[6], f[7]));
}

// NCHW fp32 [c, 3, H, W] -> ScalingLayer -> NHWC bf16 [c, H, W, 8] (channels 3..7 zero)
__global__ void input_stage_kernel(const float* __restrict__ in, const float* __restrict__ shift,
                                   const float* __restrict__ scale, int c, int HW, __nv_bfloat16* __restrict__ out) {
  const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (size_t)c * HW) return;
  const size_t img = p / HW, q = p - img * HW;
  const float* x = in + img * 3 * HW + q;
  float f[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int ch = 0; ch < 3; ch++) f[ch] = (x[(size_t)ch * HW] - shift[ch]) / scale[ch];
  reinterpret_cast<uint4*>(out)[p] = pack8(f);
}

// im2col of a 3x3, pad-1 convolution over NHWC bf16 [c, h, w, C]: col [c*h*w, 9*C], column = (ky*3 + kx)*C + ch.
// One thread per 8 channels of one (pixel, tap).  DZ: the source is dz = (da + dout[img] * G) * [a > 0] formed on the
// fly from a (bf16 post-ReLU activation), da (fp32 or NULL) and G (fp32 or NULL), rounded to bf16.
template <bool DZ>
__global__ void im2col_kernel(const __nv_bfloat16* __restrict__ a, const float* __restrict__ da,
                              const float* __restrict__ G, const float* __restrict__ dout, int c, int h, int w, int C,
                              __nv_bfloat16* __restrict__ col) {
  const int C8 = C >> 3;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)c * h * w * 9 * C8;
  if (idx >= total) return;
  const int j = (int)(idx % C8);
  const size_t r = idx / C8;
  const int t = (int)(r % 9);
  const size_t p = r / 9;
  const int hw = h * w;
  const int img = (int)(p / hw), yx = (int)(p - (size_t)img * hw);
  const int yy = yx / w + t / 3 - 1, xx = yx % w + t % 3 - 1;
  uint4 v = make_uint4(0u, 0u, 0u, 0u);
  if (yy >= 0 && yy < h && xx >= 0 && xx < w) {
    const size_t off = ((size_t)img * hw + (size_t)yy * w + xx) * C + j * 8;
    v = *reinterpret_cast<const uint4*>(a + off);
    if constexpr (DZ) {
      float f[8], g[8];
      unpack8(v, f);
#pragma unroll
      for (int i = 0; i < 8; i++) g[i] = 0.f;
      if (da) {
        const float4 d0 = *reinterpret_cast<const float4*>(da + off), d1 = *reinterpret_cast<const float4*>(da + off + 4);
        g[0] = d0.x; g[1] = d0.y; g[2] = d0.z; g[3] = d0.w; g[4] = d1.x; g[5] = d1.y; g[6] = d1.z; g[7] = d1.w;
      }
      if (G) {
        const float s = dout[img];
        const float4 g0 = *reinterpret_cast<const float4*>(G + off), g1 = *reinterpret_cast<const float4*>(G + off + 4);
        g[0] += s * g0.x; g[1] += s * g0.y; g[2] += s * g0.z; g[3] += s * g0.w;
        g[4] += s * g1.x; g[5] += s * g1.y; g[6] += s * g1.z; g[7] += s * g1.w;
      }
#pragma unroll
      for (int i = 0; i < 8; i++) g[i] = f[i] > 0.f ? g[i] : 0.f;
      v = pack8(g);
    }
  }
  reinterpret_cast<uint4*>(col)[idx] = v;
}

// 2x2 / 2 max-pool, NHWC bf16 [c, h, w, C] -> [c, h/2, w/2, C]
__global__ void maxpool_kernel(const __nv_bfloat16* __restrict__ in, int c, int h, int w, int C,
                               __nv_bfloat16* __restrict__ out) {
  const int C8 = C >> 3, ho = h >> 1, wo = w >> 1;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)c * ho * wo * C8) return;
  const int j = (int)(idx % C8);
  const size_t p = idx / C8;
  const int img = (int)(p / ((size_t)ho * wo)), yx = (int)(p - (size_t)img * ho * wo);
  const int y = 2 * (yx / wo), x = 2 * (yx % wo);
  const __nv_bfloat16* base = in + (((size_t)img * h + y) * w + x) * C + j * 8;
  uint4 m = *reinterpret_cast<const uint4*>(base);
  const size_t offs[3] = {(size_t)C, (size_t)w * C, (size_t)w * C + C};
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const uint4 u = *reinterpret_cast<const uint4*>(base + offs[k]);
    __nv_bfloat162* mm = reinterpret_cast<__nv_bfloat162*>(&m);
    const __nv_bfloat162* uu = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; i++) mm[i] = __hmax2(mm[i], uu[i]);
  }
  reinterpret_cast<uint4*>(out)[idx] = m;
}

// max-pool backward: g [c, h/2, w/2, C] fp32 -> da [c, h, w, C] fp32, each gradient to the FIRST maximum of its window
// in row-major order (torch's max_pool2d), every other entry 0.  a = the pool's bf16 input.
__global__ void maxpool_bwd_kernel(const __nv_bfloat16* __restrict__ a, const float* __restrict__ g, int c, int h, int w,
                                   int C, float* __restrict__ da) {
  const int C8 = C >> 3, ho = h >> 1, wo = w >> 1;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)c * ho * wo * C8) return;
  const int j = (int)(idx % C8);
  const size_t p = idx / C8;
  const int img = (int)(p / ((size_t)ho * wo)), yx = (int)(p - (size_t)img * ho * wo);
  const int y = 2 * (yx / wo), x = 2 * (yx % wo);
  const size_t offs[4] = {0, (size_t)C, (size_t)w * C, (size_t)w * C + C};
  const size_t base = (((size_t)img * h + y) * w + x) * C + j * 8;
  float v[4][8];
#pragma unroll
  for (int k = 0; k < 4; k++) unpack8(*reinterpret_cast<const uint4*>(a + base + offs[k]), v[k]);
  float gg[8];
  {
    const float4 g0 = *reinterpret_cast<const float4*>(g + p * C + j * 8);
    const float4 g1 = *reinterpret_cast<const float4*>(g + p * C + j * 8 + 4);
    gg[0] = g0.x; gg[1] = g0.y; gg[2] = g0.z; gg[3] = g0.w; gg[4] = g1.x; gg[5] = g1.y; gg[6] = g1.z; gg[7] = g1.w;
  }
  int arg[8];
#pragma unroll
  for (int i = 0; i < 8; i++) {
    arg[i] = 0;
    float best = v[0][i];
#pragma unroll
    for (int k = 1; k < 4; k++)
      if (v[k][i] > best) { best = v[k][i]; arg[i] = k; }
  }
#pragma unroll
  for (int k = 0; k < 4; k++) {
    float o[8];
#pragma unroll
    for (int i = 0; i < 8; i++) o[i] = arg[i] == k ? gg[i] : 0.f;
    float4* d = reinterpret_cast<float4*>(da + base + offs[k]);
    d[0] = make_float4(o[0], o[1], o[2], o[3]);
    d[1] = make_float4(o[4], o[5], o[6], o[7]);
  }
}

// LPIPS head of one tap: one warp per pixel over both inputs' activations [npix, C] (C = 64 * VP).
//   dpix[p] = sum_c lin[c] (f0 - f1)^2 ;  G (optional) = d (inv_hw * dpix summed over the image) / d a0:
//   with g = 2 inv_hw lin (f0 - f1), r = |a0|, s = r + 1e-10:   G = g / s - a0 (g . a0) / (s^2 r)   (0 at r = 0)
template <int VP>
__global__ void __launch_bounds__(256) head_kernel(const __nv_bfloat16* __restrict__ a0, const __nv_bfloat16* __restrict__ a1,
                                                   const float* __restrict__ lin, int npix, float inv_hw,
                                                   float* __restrict__ dpix, float* __restrict__ G) {
  constexpr int C = 64 * VP;
  const int p = (int)(((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (p >= npix) return;
  const __nv_bfloat162* x0 = reinterpret_cast<const __nv_bfloat162*>(a0 + (size_t)p * C);
  const __nv_bfloat162* x1 = reinterpret_cast<const __nv_bfloat162*>(a1 + (size_t)p * C);
  float2 u[VP], v[VP];
  float r0 = 0.f, r1 = 0.f;
#pragma unroll
  for (int i = 0; i < VP; i++) {
    u[i] = __bfloat1622float2(x0[i * 32 + lane]);
    v[i] = __bfloat1622float2(x1[i * 32 + lane]);
    r0 += u[i].x * u[i].x + u[i].y * u[i].y;
    r1 += v[i].x * v[i].x + v[i].y * v[i].y;
  }
  r0 = sqrtf(warp_sum(r0));
  r1 = sqrtf(warp_sum(r1));
  const float s0 = r0 + 1e-10f, s1 = r1 + 1e-10f;
  float2 df[VP], wl[VP];
  float d = 0.f;
#pragma unroll
  for (int i = 0; i < VP; i++) {
    wl[i] = *reinterpret_cast<const float2*>(lin + 2 * (i * 32 + lane));
    df[i] = make_float2(u[i].x / s0 - v[i].x / s1, u[i].y / s0 - v[i].y / s1);
    d += wl[i].x * df[i].x * df[i].x + wl[i].y * df[i].y * df[i].y;
  }
  d = warp_sum(d);
  if (lane == 0) dpix[p] = d;
  if (G == nullptr) return;
  float2 g[VP];
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < VP; i++) {
    g[i] = make_float2(2.f * inv_hw * wl[i].x * df[i].x, 2.f * inv_hw * wl[i].y * df[i].y);
    t += g[i].x * u[i].x + g[i].y * u[i].y;
  }
  t = warp_sum(t);
  const float coef = r0 > 0.f ? t / (s0 * s0 * r0) : 0.f;
  float2* Gp = reinterpret_cast<float2*>(G + (size_t)p * C);
#pragma unroll
  for (int i = 0; i < VP; i++) Gp[i * 32 + lane] = make_float2(g[i].x / s0 - u[i].x * coef, g[i].y / s0 - u[i].y * coef);
}

// out[img] (+)= inv_hw * sum of dpix over the image's hw pixels: one block per image, fixed summation order
__global__ void __launch_bounds__(256) image_sum_kernel(const float* __restrict__ dpix, int hw, float inv_hw,
                                                        float* __restrict__ out, int accumulate) {
  __shared__ float red[256];
  const float* d = dpix + (size_t)blockIdx.x * hw;
  float s = 0.f;
  for (int i = threadIdx.x; i < hw; i += 256) s += d[i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[blockIdx.x] = (accumulate ? out[blockIdx.x] : 0.f) + red[0] * inv_hw;
}

// conv1_1's input gradient [c*HW, 32] fp32 (channels 0..2 real) -> d in0 NCHW fp32 [c, 3, H, W], through the ScalingLayer
__global__ void input_grad_kernel(const float* __restrict__ dx, const float* __restrict__ scale, int c, int HW,
                                  float* __restrict__ d_in) {
  const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (size_t)c * HW) return;
  const size_t img = p / HW, q = p - img * HW;
#pragma unroll
  for (int ch = 0; ch < 3; ch++) d_in[(img * 3 + ch) * HW + q] = dx[p * WT0_ROWS + ch] / scale[ch];
}

inline unsigned blocks_for(size_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

// ---- buffers ----
struct State {  // per layer / tap, all n images contiguous
  __nv_bfloat16* act[NCONV];  // in0's post-ReLU activations [n, h_l, w_l, C_out]
  float* G[NTAP];             // d d[n] / d a0 at each tap [n, h_k, w_k, C_k]
};
State carve_state(void* base, int n, int H, int W, size_t* bytes) {
  Carver cv(base);
  State s;
  const size_t HW = (size_t)H * W;
  for (int l = 0; l < NCONV; l++) s.act[l] = cv.take<__nv_bfloat16>((size_t)n * (HW >> (2 * kConv[l].level)) * kConv[l].cout);
  for (int k = 0; k < NTAP; k++) {
    const ConvSpec& cs = kConv[kTapConv[k]];
    s.G[k] = cv.take<float>((size_t)n * (HW >> (2 * cs.level)) * cs.cout);
  }
  if (bytes) *bytes = cv.bytes();
  return s;
}

// Workspace for a chunk of c images.  The backward reuses the forward's activation buffers: x0a|x0b as fp32 da_a and
// x1a|x1b as fp32 da_b (each pair is contiguous: the sizes are multiples of 256 bytes because H*W is).
struct Work {
  __nv_bfloat16* col;                   // im2col operand [c*HW, 576]
  __nv_bfloat16 *x0a, *x0b, *x1a, *x1b; // ping-pong activations of in0 / in1 [c*HW, 64]
  float* dpix;                          // head: per-pixel distance [c*HW]
};
Work carve_work(void* base, int c, int H, int W, size_t* bytes) {
  Carver cv(base);
  Work w;
  const size_t px = (size_t)c * H * W;
  w.col = cv.take<__nv_bfloat16>(px * COL_K_MAX);
  w.x0a = cv.take<__nv_bfloat16>(px * 64);
  w.x0b = cv.take<__nv_bfloat16>(px * 64);
  w.x1a = cv.take<__nv_bfloat16>(px * 64);
  w.x1b = cv.take<__nv_bfloat16>(px * 64);
  w.dpix = cv.take<float>(px);
  if (bytes) *bytes = cv.bytes();
  return w;
}
size_t work_bytes(int c, int H, int W) {
  size_t b = 0;
  carve_work(nullptr, c, H, W, &b);
  return b;
}
size_t state_bytes(int n, int H, int W) {
  size_t b = 0;
  carve_state(nullptr, n, H, W, &b);
  return b;
}

int check_args(const dgs_lpips_weights* w, int n, int H, int W, const void* workspace, size_t workspace_bytes, int* chunk) {
  DGS_REQUIRE(w != nullptr, "lpips: weights are NULL");
  DGS_REQUIRE(n > 0, "lpips: need n > 0 (got %d)", n);
  DGS_REQUIRE(H >= 16 && W >= 16 && H % 16 == 0 && W % 16 == 0,
              "lpips: H and W must be multiples of 16 and at least 16 (got %dx%d)", H, W);
  DGS_REQUIRE(workspace != nullptr && workspace_bytes >= work_bytes(1, H, W),
              "lpips: workspace too small (%zu bytes, one image needs %zu)", workspace_bytes, work_bytes(1, H, W));
  int c = (int)(workspace_bytes / work_bytes(1, H, W));
  c = c < n ? c : n;
  while (c > 1 && work_bytes(c, H, W) > workspace_bytes) c--;
  *chunk = c;
  return DGS_OK;
}

inline __nv_bfloat16* other(__nv_bfloat16* cur, __nv_bfloat16* a, __nv_bfloat16* b) { return cur == a ? b : a; }

int conv_fwd(const dgs_lpips_weights* w, int l, const __nv_bfloat16* in, __nv_bfloat16* col, __nv_bfloat16* out, int c,
             int h, int wd, cudaStream_t st) {
  const ConvSpec& cs = kConv[l];
  const size_t n8 = (size_t)c * h * wd * 9 * (cs.cin / 8);
  im2col_kernel<false><<<blocks_for(n8, 256), 256, 0, st>>>(in, nullptr, nullptr, nullptr, c, h, wd, cs.cin, col);
  DGS_POST_LAUNCH();
  GemmEpilogue ep;
  ep.out = out;
  ep.ldc = cs.cout;
  ep.bias = w->conv_b[l];
  return gemm_bf16(col, w->conv_w[l], c * h * wd, cs.cout, 9 * cs.cin, EPI_BIAS_RELU_BF16, ep, st);
}

int pool_fwd(const __nv_bfloat16* in, __nv_bfloat16* out, int c, int h, int wd, int C, cudaStream_t st) {
  const size_t n8 = (size_t)c * (h / 2) * (wd / 2) * (C / 8);
  maxpool_kernel<<<blocks_for(n8, 256), 256, 0, st>>>(in, c, h, wd, C, out);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

int head(const dgs_lpips_weights* w, int k, const __nv_bfloat16* a0, const __nv_bfloat16* a1, int c, int hw, float* dpix,
         float* G, float* out, cudaStream_t st) {
  const int C = kConv[kTapConv[k]].cout, npix = c * hw;
  const float inv_hw = 1.0f / (float)hw;
  const unsigned grid = blocks_for((size_t)npix * 32, 256);
  switch (C / 64) {
    case 1: head_kernel<1><<<grid, 256, 0, st>>>(a0, a1, w->lin[k], npix, inv_hw, dpix, G); break;
    case 2: head_kernel<2><<<grid, 256, 0, st>>>(a0, a1, w->lin[k], npix, inv_hw, dpix, G); break;
    case 4: head_kernel<4><<<grid, 256, 0, st>>>(a0, a1, w->lin[k], npix, inv_hw, dpix, G); break;
    default: head_kernel<8><<<grid, 256, 0, st>>>(a0, a1, w->lin[k], npix, inv_hw, dpix, G); break;
  }
  DGS_POST_LAUNCH();
  image_sum_kernel<<<c, 256, 0, st>>>(dpix, hw, inv_hw, out, k > 0);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

}  // namespace
}  // namespace dgs

using namespace dgs;

extern "C" {

size_t dgs_lpips_workspace_bytes(int n, int H, int W) { return n > 0 && H > 0 && W > 0 ? work_bytes(n, H, W) : 0; }
size_t dgs_lpips_state_bytes(int n, int H, int W) { return n > 0 && H > 0 && W > 0 ? state_bytes(n, H, W) : 0; }

int dgs_lpips_forward(const dgs_lpips_weights* w, int n, int H, int W, const float* in0, const float* in1, float* out,
                      void* state, void* workspace, size_t workspace_bytes, void* stream) {
  int c = 0;
  int rc = check_args(w, n, H, W, workspace, workspace_bytes, &c);
  if (rc) return rc;
  DGS_REQUIRE(in0 && in1 && out, "lpips: in0, in1 and out must not be NULL");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int HW = H * W;
  State s = carve_state(state, n, H, W, nullptr);
  Work wk = carve_work(workspace, c, H, W, nullptr);
  for (int i0 = 0; i0 < n; i0 += c) {
    const int cc = n - i0 < c ? n - i0 : c;
    input_stage_kernel<<<blocks_for((size_t)cc * HW, 256), 256, 0, st>>>(in0 + (size_t)i0 * 3 * HW, w->shift, w->scale, cc,
                                                                          HW, wk.x0a);
    DGS_POST_LAUNCH();
    input_stage_kernel<<<blocks_for((size_t)cc * HW, 256), 256, 0, st>>>(in1 + (size_t)i0 * 3 * HW, w->shift, w->scale, cc,
                                                                          HW, wk.x1a);
    DGS_POST_LAUNCH();
    __nv_bfloat16 *cur0 = wk.x0a, *cur1 = wk.x1a;
    for (int l = 0; l < NCONV; l++) {
      const ConvSpec& cs = kConv[l];
      const int h = H >> cs.level, wd = W >> cs.level, hw = h * wd;
      if (cs.pool_before) {
        __nv_bfloat16* p0 = other(cur0, wk.x0a, wk.x0b);
        __nv_bfloat16* p1 = other(cur1, wk.x1a, wk.x1b);
        if ((rc = pool_fwd(cur0, p0, cc, 2 * h, 2 * wd, cs.cin, st))) return rc;
        if ((rc = pool_fwd(cur1, p1, cc, 2 * h, 2 * wd, cs.cin, st))) return rc;
        cur0 = p0; cur1 = p1;
      }
      __nv_bfloat16* o0 = state ? s.act[l] + (size_t)i0 * hw * cs.cout : other(cur0, wk.x0a, wk.x0b);
      __nv_bfloat16* o1 = other(cur1, wk.x1a, wk.x1b);
      if ((rc = conv_fwd(w, l, cur0, wk.col, o0, cc, h, wd, st))) return rc;
      if ((rc = conv_fwd(w, l, cur1, wk.col, o1, cc, h, wd, st))) return rc;
      cur0 = o0; cur1 = o1;
      if (cs.tap >= 0) {
        float* G = state ? s.G[cs.tap] + (size_t)i0 * hw * cs.cout : nullptr;
        if ((rc = head(w, cs.tap, cur0, cur1, cc, hw, wk.dpix, G, out + i0, st))) return rc;
      }
    }
  }
  return DGS_OK;
}

int dgs_lpips_backward(const dgs_lpips_weights* w, int n, int H, int W, const void* state, const float* dout,
                       float* d_in0, void* workspace, size_t workspace_bytes, void* stream) {
  int c = 0;
  int rc = check_args(w, n, H, W, workspace, workspace_bytes, &c);
  if (rc) return rc;
  DGS_REQUIRE(state != nullptr, "lpips backward: state is NULL (the forward must be given a training state)");
  DGS_REQUIRE(dout && d_in0, "lpips backward: dout and d_in0 must not be NULL");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int HW = H * W;
  State s = carve_state(const_cast<void*>(state), n, H, W, nullptr);
  Work wk = carve_work(workspace, c, H, W, nullptr);
  float* da_a = reinterpret_cast<float*>(wk.x0a);  // [c*HW, 64] fp32 each (see Work)
  float* da_b = reinterpret_cast<float*>(wk.x1a);
  for (int i0 = 0; i0 < n; i0 += c) {
    const int cc = n - i0 < c ? n - i0 : c;
    const float* da = nullptr;
    for (int l = NCONV - 1; l >= 0; l--) {
      const ConvSpec& cs = kConv[l];
      const int h = H >> cs.level, wd = W >> cs.level, hw = h * wd;
      const __nv_bfloat16* a = s.act[l] + (size_t)i0 * hw * cs.cout;
      const float* G = cs.tap >= 0 ? s.G[cs.tap] + (size_t)i0 * hw * cs.cout : nullptr;
      const size_t n8 = (size_t)cc * hw * 9 * (cs.cout / 8);
      im2col_kernel<true><<<blocks_for(n8, 256), 256, 0, st>>>(a, da, G, dout + i0, cc, h, wd, cs.cout, wk.col);
      DGS_POST_LAUNCH();
      const int N = l == 0 ? WT0_ROWS : cs.cin;
      GemmEpilogue ep;
      ep.out = da_a;
      ep.ldc = N;
      if ((rc = gemm_bf16(wk.col, w->conv_wt[l], cc * hw, N, 9 * cs.cout, EPI_F32, ep, st))) return rc;
      if (l == 0) {
        input_grad_kernel<<<blocks_for((size_t)cc * HW, 256), 256, 0, st>>>(da_a, w->scale, cc, HW,
                                                                             d_in0 + (size_t)i0 * 3 * HW);
        DGS_POST_LAUNCH();
      } else if (cs.pool_before) {
        const ConvSpec& below = kConv[l - 1];
        const size_t n8p = (size_t)cc * hw * (cs.cin / 8);
        maxpool_bwd_kernel<<<blocks_for(n8p, 256), 256, 0, st>>>(s.act[l - 1] + (size_t)i0 * 4 * hw * below.cout, da_a, cc,
                                                                 2 * h, 2 * wd, cs.cin, da_b);
        DGS_POST_LAUNCH();
        da = da_b;
      } else {
        da = da_a;
      }
    }
  }
  return DGS_OK;
}

}  // extern "C"
