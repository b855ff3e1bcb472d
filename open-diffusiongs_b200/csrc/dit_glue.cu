// dit_glue.cu -- the memory-bound glue kernels of the DiT denoiser (everything that is not a GEMM or the attention),
// forward and backward, ordered by operation with each backward right after its forward: LayerNorm (+ adaLN modulate),
// the input stage (posed-image patchify, token assembly), the skinny (batch-row) linears of the timestep / adaLN MLPs
// and the tiny free-token head linear, the Gaussian heads' epilogue (to_gs + pixel alignment), the gate / transpose /
// column-sum kernels around the weight-gradient GEMMs, and the fused AdamW update.
// Spec: diffusionGS/models/denoiser/denoiser.py:26-72,76-164,306-416 and denoiser_scene.py:314-429,
//       diffusionGS/models/transformers/utils_transformer.py:26-27,246-290.  The reference gets the backward from torch
// autograd; the backward formulas below are the derivatives of the forward kernels here and in gemm_sm90.cu.
#include "dgs_internal.h"
#include "dit_kernels.h"
#include "sm90_ptx.cuh"

namespace dgs {

namespace {

using ptx::warp_sum;

// ---- fp32 / bf16 element loads of the kernels that take either input type ----
__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
// 4 consecutive elements -> fp32
__device__ __forceinline__ void load4_f32(const float* p, float* o) {
  const float4 v = *reinterpret_cast<const float4*>(p);
  o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
}
__device__ __forceinline__ void load4_f32(const __nv_bfloat16* p, float* o) {
  const uint2 v = *reinterpret_cast<const uint2*>(p);
  const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v.x));
  const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v.y));
  o[0] = a.x; o[1] = a.y; o[2] = b.x; o[3] = b.y;
}
// 16 consecutive elements -> bf16 (two 16-byte vectors)
__device__ __forceinline__ void load16_bf16(const __nv_bfloat16* src, uint4& lo, uint4& hi) {
  lo = *reinterpret_cast<const uint4*>(src);
  hi = *reinterpret_cast<const uint4*>(src + 8);
}
__device__ __forceinline__ void load16_bf16(const float* src, uint4& lo, uint4& hi) {
  using ptx::pack2_bf16;
  const float4 a = *reinterpret_cast<const float4*>(src), b = *reinterpret_cast<const float4*>(src + 4);
  const float4 c = *reinterpret_cast<const float4*>(src + 8), d = *reinterpret_cast<const float4*>(src + 12);
  lo = make_uint4(pack2_bf16(a.x, a.y), pack2_bf16(a.z, a.w), pack2_bf16(b.x, b.y), pack2_bf16(b.z, b.w));
  hi = make_uint4(pack2_bf16(c.x, c.y), pack2_bf16(c.z, c.w), pack2_bf16(d.x, d.y), pack2_bf16(d.z, d.w));
}

// The column reductions of 256-thread CTAs over 64 columns: thread t adds up rows of column t % 64 in quarter t / 64
// and stores its partial sum to red[(t / 64) * 64 + t % 64] (+ a multiple of 256 per quantity); after a barrier,
// column c's total is
__device__ __forceinline__ float quarter_sum(const float* red, int c) {
  return red[c] + red[64 + c] + red[128 + c] + red[192 + c];
}

__device__ __forceinline__ float silu(float v) { return v / (1.0f + __expf(-v)); }

}  // namespace

// ---------------------------------------------------------------------------------------------
// LayerNorm (+ optional weight) + adaLN modulate.  One warp per row, D = 32 * 4 * VEC.
// Two-pass statistics in registers (mean, then centred variance) = torch's LayerNorm numerics.
// ---------------------------------------------------------------------------------------------
namespace {

// one warp loads row xr into v (lane l holds float4 number i of the row at columns 4 (32 i + l) .. + 3), centres it on
// the row mean and returns 1 / sqrt(var + eps)
template <int D>
__device__ __forceinline__ float ln_row_stats(const float* xr, int lane, float (&v)[D / 32], float eps,
                                              float& mean) {
  constexpr int PER_LANE = D / 32;
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < PER_LANE / 4; i++) {
    const float4 t = *reinterpret_cast<const float4*>(xr + (i * 32 + lane) * 4);
    v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
    s += t.x + t.y + t.z + t.w;
  }
  mean = warp_sum(s) * (1.0f / D);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < PER_LANE; i++) { v[i] -= mean; q += v[i] * v[i]; }
  return rsqrtf(warp_sum(q) * (1.0f / D) + eps);
}

// Output row r (0 .. B * rows_out) is  y = LN(x row b * rows_in + row_off + r % rows_out) [* lnw], b = r / rows_out,
// stored as OUT (LnOut): y * (1 + scale[b]) + shift[b] as bf16, split bf16 or e4m3, or y itself as fp32.  LN_F32 writes
// in place (out == x): a row is stored only after all of it was loaded and reduced.
template <int D, LnOut OUT>
__global__ void __launch_bounds__(256) ln_kernel(const float* __restrict__ x, const float* __restrict__ lnw,
                                                 const float* __restrict__ shift, const float* __restrict__ scale,
                                                 int mod_stride, void* __restrict__ out, float* __restrict__ q_scale,
                                                 int lds, int B, int rows_in, int row_off, int rows_out, float eps) {
  constexpr int PER_LANE = D / 32;  // 32 for D = 1024
  constexpr bool ALWAYS_W = OUT == LN_F32, NEVER_W = OUT == LN_E4M3;  // LnOut: whether lnw may be null
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  ptx::griddep_launch_dependents();  // PDL: launched via launch_pdl (LN_F32: a plain launch, where these are no-ops)
  ptx::griddep_wait();
  if (warp >= B * rows_out) return;
  const int b = warp / rows_out, r = warp - b * rows_out;
  float v[PER_LANE];
  float mean;
  const float rstd = ln_row_stats<D>(x + ((size_t)b * rows_in + row_off + r) * D, lane, v, eps, mean);
  const float* sh = shift + (size_t)b * mod_stride;
  const float* sc = scale + (size_t)b * mod_stride;
#pragma unroll
  for (int i = 0; i < PER_LANE / 4; i++) {
    const int c = (i * 32 + lane) * 4;
    float4 w4 = make_float4(1.f, 1.f, 1.f, 1.f);  // x * 1.0f is exact: no weight = weight 1
    if (ALWAYS_W || (!NEVER_W && lnw)) w4 = __ldg(reinterpret_cast<const float4*>(lnw + c));
    float o0 = v[4 * i] * rstd * w4.x, o1 = v[4 * i + 1] * rstd * w4.y;
    float o2 = v[4 * i + 2] * rstd * w4.z, o3 = v[4 * i + 3] * rstd * w4.w;
    if constexpr (OUT == LN_F32) {  // no modulate: y * (1 + 0) + 0 would turn -0 into +0
      *reinterpret_cast<float4*>(static_cast<float*>(out) + (size_t)warp * D + c) = make_float4(o0, o1, o2, o3);
      continue;
    }
    const float4 s4 = __ldg(reinterpret_cast<const float4*>(sc + c));
    const float4 h4 = __ldg(reinterpret_cast<const float4*>(sh + c));
    o0 = o0 * (1.f + s4.x) + h4.x;
    o1 = o1 * (1.f + s4.y) + h4.y;
    o2 = o2 * (1.f + s4.z) + h4.z;
    o3 = o3 * (1.f + s4.w) + h4.w;
    if constexpr (OUT == LN_E4M3) {
      // lane l's float4 number i lies in 128-column group i, so each group's amax is one warp reduction
      float amax = fmaxf(fmaxf(fabsf(o0), fabsf(o1)), fmaxf(fabsf(o2), fabsf(o3)));
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
      const int e = ptx::e4m3_scale_exp(amax);
      const float inv = ptx::exp2_int(-e);
      const uint32_t packed =
          (uint32_t)ptx::pack2_e4m3(o0 * inv, o1 * inv) | ((uint32_t)ptx::pack2_e4m3(o2 * inv, o3 * inv) << 16);
      *reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(out) + (size_t)warp * D + c) = packed;
      if (lane == 0) q_scale[(size_t)i * lds + warp] = ptx::exp2_int(e);
    } else {
      __nv_bfloat16* hr = static_cast<__nv_bfloat16*>(out) + (size_t)warp * D * (OUT == LN_SPLIT_BF16 ? 3 : 1);
      __nv_bfloat162 p0 = __floats2bfloat162_rn(o0, o1), p1 = __floats2bfloat162_rn(o2, o3);
      uint2 pk;
      pk.x = *reinterpret_cast<uint32_t*>(&p0);
      pk.y = *reinterpret_cast<uint32_t*>(&p1);
      *reinterpret_cast<uint2*>(hr + c) = pk;
      if constexpr (OUT == LN_SPLIT_BF16) {  // [hi | lo | hi]: y = hi + lo to ~2^-17 relative (split-bf16 operand)
        const float2 f0 = __bfloat1622float2(p0), f1 = __bfloat1622float2(p1);
        __nv_bfloat162 q0 = __floats2bfloat162_rn(o0 - f0.x, o1 - f0.y), q1 = __floats2bfloat162_rn(o2 - f1.x, o3 - f1.y);
        uint2 lo;
        lo.x = *reinterpret_cast<uint32_t*>(&q0);
        lo.y = *reinterpret_cast<uint32_t*>(&q1);
        *reinterpret_cast<uint2*>(hr + D + c) = lo;
        *reinterpret_cast<uint2*>(hr + 2 * D + c) = pk;
      }
    }
  }
}

}  // namespace

int ln_forward(LnOut kind, const float* x, const float* ln_weight, const float* shift, const float* scale,
               int mod_stride, void* out, float* out_scale, int B, int rows_in, int row_off, int rows_out, int D,
               float eps, cudaStream_t st) {
  static const char* const name[] = {"ln_modulate", "ln_modulate", "ln_modulate_fp8", "ln_weight"};
  DGS_REQUIRE(D == 1024, "%s: width %d not supported (1024 only)", name[kind], D);
  DGS_REQUIRE(kind != LN_E4M3 || (B > 0 && rows_out > 0), "ln_modulate_fp8: bad shape B=%d rows=%d", B, rows_out);
  const int blocks = (int)(((long long)B * rows_out * 32 + 255) / 256);
  const int lds = kind == LN_E4M3 ? fp8_scale_stride(B * rows_out) : 0;
  auto launch = [&](auto kern) {
    return launch_pdl(kern, dim3(blocks), dim3(256), 0, st, x, ln_weight, shift, scale, mod_stride, out, out_scale,
                      lds, B, rows_in, row_off, rows_out, eps);
  };
  switch (kind) {
    case LN_BF16: DGS_CUDA_OK(launch(ln_kernel<1024, LN_BF16>)); break;
    case LN_SPLIT_BF16: DGS_CUDA_OK(launch(ln_kernel<1024, LN_SPLIT_BF16>)); break;
    case LN_E4M3: DGS_CUDA_OK(launch(ln_kernel<1024, LN_E4M3>)); break;
    case LN_F32:
      ln_kernel<1024, LN_F32><<<blocks, 256, 0, st>>>(x, ln_weight, shift, scale, mod_stride, out, out_scale, lds, B,
                                                      rows_in, row_off, rows_out, eps);
      break;
  }
  DGS_POST_LAUNCH();
  return DGS_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Backward of  h = (LN(x; eps) [* w]) * (1 + scale[b]) + shift[b]   (ln_kernel), two kernels:
//  rows:  one warp per row:  dx (+)= rstd (dxh - mean(dxh) - xhat mean(dxh xhat)),  dxh = g (1+scale) w;  keeps (mean, rstd)
//  cols:  64-column x 128-row tiles:  dshift[b] += sum g ; dscale[b] += sum g xhat w ; dw += sum g (1+scale) xhat
// (the fused single-kernel version needed 96 accumulator registers per lane -> 255 registers, 8 warps per SM)
// ---------------------------------------------------------------------------------------------------------------
namespace {

template <typename TG>
__global__ void __launch_bounds__(256) ln_bwd_rows_kernel(const float* __restrict__ x, const TG* __restrict__ dh,
                                                          const float* __restrict__ lnw, const float* __restrict__ scale,
                                                          int mod_stride, int rows_in, int row_off, int rows_out, float eps,
                                                          float* __restrict__ dx, int accumulate,
                                                          float2* __restrict__ stats) {
  constexpr int D = 1024, PER = 32;
  ptx::griddep_launch_dependents();  // PDL: launched via launch_pdl
  ptx::griddep_wait();
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= rows_out) return;
  const size_t xrow = ((size_t)b * rows_in + row_off + r) * D;
  const TG* gr = dh + ((size_t)b * rows_out + r) * D;
  float v[PER], g[PER];
#pragma unroll
  for (int i = 0; i < PER / 4; i++) load4_f32(gr + (i * 32 + lane) * 4, g + 4 * i);
  float mean;
  const float rstd = ln_row_stats<D>(x + xrow, lane, v, eps, mean);
  if (lane == 0) stats[(size_t)b * rows_out + r] = make_float2(mean, rstd);
  float m1 = 0.f, m2 = 0.f;
#pragma unroll
  for (int i = 0; i < PER / 4; i++) {
    const int c = (i * 32 + lane) * 4;
    float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f), w4 = make_float4(1.f, 1.f, 1.f, 1.f);
    if (scale) s4 = __ldg(reinterpret_cast<const float4*>(scale + (size_t)b * mod_stride + c));
    if (lnw) w4 = __ldg(reinterpret_cast<const float4*>(lnw + c));
    const float sv[4] = {s4.x, s4.y, s4.z, s4.w}, wv[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
    for (int e = 0; e < 4; e++) {
      const int k = 4 * i + e;
      const float xh = v[k] * rstd;
      const float dxh = g[k] * (1.0f + sv[e]) * wv[e];
      v[k] = xh;
      g[k] = dxh;
      m1 += dxh;
      m2 += dxh * xh;
    }
  }
  m1 = warp_sum(m1) * (1.0f / D);
  m2 = warp_sum(m2) * (1.0f / D);
#pragma unroll
  for (int i = 0; i < PER / 4; i++) {
    const int c = (i * 32 + lane) * 4;
    float4 o;
    o.x = rstd * (g[4 * i] - m1 - v[4 * i] * m2);
    o.y = rstd * (g[4 * i + 1] - m1 - v[4 * i + 1] * m2);
    o.z = rstd * (g[4 * i + 2] - m1 - v[4 * i + 2] * m2);
    o.w = rstd * (g[4 * i + 3] - m1 - v[4 * i + 3] * m2);
    float4* dst = reinterpret_cast<float4*>(dx + xrow + c);
    if (accumulate) {
      const float4 p = *dst;
      o.x += p.x; o.y += p.y; o.z += p.z; o.w += p.w;
    }
    *dst = o;
  }
}

template <typename TG>
__global__ void __launch_bounds__(256) ln_bwd_cols_kernel(const float* __restrict__ x, const TG* __restrict__ dh,
                                                          const float* __restrict__ lnw, const float* __restrict__ scale,
                                                          int mod_stride, int rows_in, int row_off, int rows_out,
                                                          const float2* __restrict__ stats, float* __restrict__ dshift,
                                                          float* __restrict__ dscale, float* __restrict__ dlnw) {
  constexpr int D = 1024, ROWS = 128;
  __shared__ float red[3 * 4 * 64];
  ptx::griddep_launch_dependents();  // PDL: launched via launch_pdl
  ptx::griddep_wait();
  const int b = blockIdx.z, c = blockIdx.x * 64 + (threadIdx.x & 63), rq = threadIdx.x >> 6;
  const int r0 = blockIdx.y * ROWS;
  const float w = lnw ? __ldg(lnw + c) : 1.0f;
  const float sc1 = scale ? 1.0f + __ldg(scale + (size_t)b * mod_stride + c) : 1.0f;
  float a0 = 0.f, a1 = 0.f;
  const int r_end = min(rows_out, r0 + ROWS);
#pragma unroll 4
  for (int r = r0 + rq; r < r_end; r += 4) {
    const float2 st = __ldg(stats + (size_t)b * rows_out + r);
    const float g = to_f(dh[((size_t)b * rows_out + r) * D + c]);
    const float xh = (x[((size_t)b * rows_in + row_off + r) * D + c] - st.x) * st.y;
    a0 += g;
    a1 += g * xh;
  }
  red[rq * 64 + (threadIdx.x & 63)] = a0;
  red[256 + rq * 64 + (threadIdx.x & 63)] = a1;
  __syncthreads();
  if (threadIdx.x < 64) {
    const int t = threadIdx.x;
    const float sg = quarter_sum(red, t);
    const float sgx = quarter_sum(red, 256 + t);
    if (dshift) {
      atomicAdd(dshift + (size_t)b * mod_stride + c, sg);
      atomicAdd(dscale + (size_t)b * mod_stride + c, sgx * w);  // sum g * y, y = xhat * w
    }
    if (dlnw) atomicAdd(dlnw + c, sgx * sc1);                     // sum g (1 + scale) xhat
  }
}

}  // namespace

template <typename TG>
int ln_modulate_bwd(const float* x, const TG* dh, const float* lnw, const float* scale, int mod_stride, int B,
                    int rows_in, int row_off, int rows_out, int D, float eps, float* dx, int accumulate, float* dshift,
                    float* dscale, float* dlnw, float* stats /* scratch: 2 * B * rows_out floats */, cudaStream_t st) {
  DGS_REQUIRE(D == 1024, "ln_modulate_bwd: width %d not supported (1024 only)", D);
  DGS_REQUIRE((scale != nullptr) == (dshift != nullptr && dscale != nullptr), "ln_modulate_bwd: scale/dshift/dscale mismatch");
  DGS_REQUIRE((lnw != nullptr) == (dlnw != nullptr), "ln_modulate_bwd: lnw/dlnw mismatch");
  DGS_REQUIRE(stats != nullptr, "ln_modulate_bwd: stats scratch is NULL");
  float2* s2 = reinterpret_cast<float2*>(stats);
  DGS_CUDA_OK(launch_pdl(ln_bwd_rows_kernel<TG>, dim3((rows_out + 7) / 8, B), dim3(256), 0, st, x, dh, lnw, scale,
                         mod_stride, rows_in, row_off, rows_out, eps, dx, accumulate, s2));
  DGS_POST_LAUNCH();
  if (dshift != nullptr || dlnw != nullptr) {
    DGS_CUDA_OK(launch_pdl(ln_bwd_cols_kernel<TG>, dim3(D / 64, (rows_out + 127) / 128, B), dim3(256), 0, st, x, dh, lnw,
                           scale, mod_stride, rows_in, row_off, rows_out, (const float2*)s2, dshift, dscale, dlnw));
    DGS_POST_LAUNCH();
  }
  return DGS_OK;
}
template int ln_modulate_bwd(const float*, const float*, const float*, const float*, int, int, int, int, int, int, float,
                             float*, int, float*, float*, float*, float*, cudaStream_t);
template int ln_modulate_bwd(const float*, const __nv_bfloat16*, const float*, const float*, int, int, int, int, int, int,
                             float, float*, int, float*, float*, float*, float*, cudaStream_t);

// One block per row: amax, then the row times 2^-e rounded to e4m3 (the FP8 weight format, one scale per row).
namespace {
__global__ void __launch_bounds__(256) quantize_rows_e4m3_kernel(const float* __restrict__ x, int cols,
                                                                 uint8_t* __restrict__ q, float* __restrict__ scale) {
  __shared__ float red[8];
  const float* xr = x + (size_t)blockIdx.x * cols;
  float amax = 0.f;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) amax = fmaxf(amax, fabsf(xr[c]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = amax;
  __syncthreads();
  amax = red[0];
#pragma unroll
  for (int w = 1; w < 8; w++) amax = fmaxf(amax, red[w]);
  const int e = ptx::e4m3_scale_exp(amax);
  const float inv = ptx::exp2_int(-e);
  uint8_t* qr = q + (size_t)blockIdx.x * cols;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) qr[c] = (uint8_t)(ptx::pack2_e4m3(xr[c] * inv, 0.f) & 0xffu);
  if (threadIdx.x == 0) scale[blockIdx.x] = ptx::exp2_int(e);
}
}  // namespace

int quantize_rows_e4m3(const float* x, int rows, int cols, uint8_t* q, float* scale, cudaStream_t st) {
  DGS_REQUIRE(rows > 0 && cols > 0, "quantize_rows_e4m3: bad shape %dx%d", rows, cols);
  quantize_rows_e4m3_kernel<<<rows, 256, 0, st>>>(x, cols, q, scale);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

// ---------------------------------------------------------------------------------------------
// Input stage: posed image (rgb*2-1 | ray channels) + patchify "b v c (hh ph) (ww pw) -> (b v)(hh ww)(ph pw c)",
// token assembly, and the position embedding's backward.
// ---------------------------------------------------------------------------------------------
namespace {

// Entry q of the token-major enumeration (bv, hh, ww, ph, pw) of BV images of H x W in p x p patches (the order of the
// patchified tokens and of the image head's outputs): image bv, pixel row y, pixel column x.
struct PatchPixel { int bv, y, x; };
__device__ __forceinline__ PatchPixel patch_pixel(long long q, int H, int W, int p) {
  const int hh_n = H / p, ww_n = W / p;
  const int pw = (int)(q % p);
  long long r = q / p;
  const int ph = (int)(r % p); r /= p;
  const int ww = (int)(r % ww_n); r /= ww_n;
  const int hh = (int)(r % hh_n);
  return {(int)(r / hh_n), hh * p + ph, ww * p + pw};
}

// one thread per (token, ph, pw): writes its 9 channels contiguously (18 B) -- output-coalesced.
__global__ void __launch_bounds__(256) posed_patchify_kernel(const float* __restrict__ img,
                                                             const float* __restrict__ ray_o,
                                                             const float* __restrict__ ray_d,
                                                             __nv_bfloat16* __restrict__ tokens, int BV, int H, int W,
                                                             int p, int img_c, int mode) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)BV * H * W;
  if (idx >= total) return;
  const PatchPixel px = patch_pixel(idx, H, W, p);  // idx enumerates (bv, hh, ww, ph, pw) in output order
  const size_t plane = (size_t)H * W, pix = (size_t)px.y * W + px.x;
  const float* ip = img + (size_t)px.bv * img_c * plane + pix;
  const float* op = ray_o + (size_t)px.bv * 3 * plane + pix;
  const float* dp = ray_d + (size_t)px.bv * 3 * plane + pix;
  const float o0 = op[0], o1 = op[plane], o2 = op[2 * plane];
  const float d0 = dp[0], d1 = dp[plane], d2 = dp[2 * plane];
  float c[9];
  c[0] = ip[0] * 2.0f - 1.0f; c[1] = ip[plane] * 2.0f - 1.0f; c[2] = ip[2 * plane] * 2.0f - 1.0f;
  if (mode == 0) {  // 'relative_plk' (denoiser.py:312-323)
    const float odd = -o0 * d0 + -o1 * d1 + -o2 * d2;
    c[3] = d0; c[4] = d1; c[5] = d2;
    c[6] = o0 + odd * d0; c[7] = o1 + odd * d1; c[8] = o2 + odd * d2;
  } else {  // 'plk' (denoiser.py:324-333): o x d, d
    c[3] = o1 * d2 - o2 * d1; c[4] = o2 * d0 - o0 * d2; c[5] = o0 * d1 - o1 * d0;
    c[6] = d0; c[7] = d1; c[8] = d2;
  }
  // split-bf16 token row [hi | lo | hi] (K = 3 * p*p*9): the tokenizer GEMM then computes
  // x_hi W_hi + x_lo W_hi + x_hi W_lo, i.e. an fp32-accurate product on the bf16 tensor-core path
  const int Kt = p * p * 9;
  const long long token = idx / (p * p);
  const int inner = (int)(idx % (p * p)) * 9;
  __nv_bfloat16* o = tokens + token * 3 * Kt + inner;
#pragma unroll
  for (int k = 0; k < 9; k++) {
    const __nv_bfloat16 hi = __float2bfloat16_rn(c[k]);
    o[k] = hi;
    o[Kt + k] = __float2bfloat16_rn(c[k] - __bfloat162float(hi));
    o[2 * Kt + k] = hi;
  }
}

__global__ void assemble_tokens_kernel(const float* __restrict__ tok, const float* __restrict__ pos,
                                       float* __restrict__ x, int B, int G, int T, int D4) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)B * (G + T) * D4;
  if (idx >= total) return;
  const int c = (int)(idx % D4);
  const long long r = idx / D4;
  const int n = (int)(r % (G + T)), b = (int)(r / (G + T));
  const float4* src = (n < G) ? reinterpret_cast<const float4*>(pos) + (size_t)n * D4 + c
                              : reinterpret_cast<const float4*>(tok) + ((size_t)b * T + (n - G)) * D4 + c;
  reinterpret_cast<float4*>(x)[idx] = *src;
}

// dpos[g, :] = sum_b dx[b, g, :]   (the learned Gaussian tokens sit at rows 0..G of every sample)
__global__ void pos_embed_bwd_kernel(const float* __restrict__ dx, float* __restrict__ dpos, int B, int G, int N, int D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G * D) return;
  const int g = i / D, c = i - g * D;
  float s = 0.f;
  for (int b = 0; b < B; b++) s += dx[((size_t)b * N + g) * D + c];
  dpos[i] = s;
}

}  // namespace

int posed_patchify(const float* images, const float* ray_o, const float* ray_d, __nv_bfloat16* tokens, int B, int V,
                   int H, int W, int patch, int plucker_mode, cudaStream_t st) {
  DGS_REQUIRE(H % patch == 0 && W % patch == 0, "image size %dx%d not divisible by patch %d", H, W, patch);
  const long long total = (long long)B * V * H * W;
  posed_patchify_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(images, ray_o, ray_d, tokens, B * V, H, W,
                                                                          patch, 3, plucker_mode);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

int assemble_tokens(const float* tok, const float* pos_embed, float* x, int B, int G, int T, int D, cudaStream_t st) {
  const long long total = (long long)B * (G + T) * (D / 4);
  assemble_tokens_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(tok, pos_embed, x, B, G, T, D / 4);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

int pos_embed_bwd(const float* dx, float* dpos, int B, int G, int N, int D, cudaStream_t st) {
  if (G == 0) return DGS_OK;
  pos_embed_bwd_kernel<<<ceil_div(G * D, 256), 256, 0, st>>>(dx, dpos, B, G, N, D);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

// ---------------------------------------------------------------------------------------------
// Conditioning: the sinusoidal timestep embedding and the skinny linear
//   out[b, n] = act(in[b, :]) . W[n, :] + bias[n] for b < B <= 8.  HBM-bound on W
// (each fp32 weight row read once, 16-byte loads); one warp per output column n, all B rows at once.
// fp32 weights: the conditioning (shift / scale / gate of every block) multiplies every activation, so
// bf16-rounding it would put a 1e-3 relative error on the whole network for a saving of ~50 us.
// Used for the timestep MLP and for the adaLN modulation of ALL 24 blocks + 2 heads in one launch
// (the conditioning vector is layer-invariant).
// ---------------------------------------------------------------------------------------------
namespace {

constexpr int SKINNY_MAXB = 8;

// denoiser.py:44-66 (cos | sin, max_period 1e4)
__global__ void timestep_embedding_kernel(const float* __restrict__ t, float* __restrict__ out, int B, int dim) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int half = dim / 2;
  if (idx >= B * half) return;
  const int b = idx / half, i = idx - b * half;
  const float freq = expf(-logf(10000.0f) * (float)i / (float)half);
  const float a = t[b] * freq;
  out[(size_t)b * dim + i] = cosf(a);
  out[(size_t)b * dim + half + i] = sinf(a);
}

__global__ void __launch_bounds__(256) skinny_linear_kernel(const float* __restrict__ in,
                                                            const float* __restrict__ W,
                                                            const float* __restrict__ bias, float* __restrict__ out,
                                                            int B, int N, int K, int act_in, int act_out) {
  extern __shared__ float s_in[];  // [B, K] activated input
  for (int t = threadIdx.x; t < B * K; t += blockDim.x) {
    float v = in[t];
    s_in[t] = act_in ? silu(v) : v;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x * (blockDim.x >> 5) + warp;
  if (n >= N) return;
  float acc[SKINNY_MAXB];
#pragma unroll
  for (int b = 0; b < SKINNY_MAXB; b++) acc[b] = 0.f;
  const float* wr = W + (size_t)n * K;
  for (int k = lane * 8; k < K; k += 256) {
    const float4 wa = __ldg(reinterpret_cast<const float4*>(wr + k));
    const float4 wb = __ldg(reinterpret_cast<const float4*>(wr + k + 4));
    const float w[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w};
#pragma unroll
    for (int b = 0; b < SKINNY_MAXB; b++) {
      if (b < B) {
        const float* xi = s_in + b * K + k;
#pragma unroll
        for (int j = 0; j < 8; j++) acc[b] += w[j] * xi[j];
      }
    }
  }
#pragma unroll
  for (int b = 0; b < SKINNY_MAXB; b++) {
    if (b < B) {
      float v = warp_sum(acc[b]);
      if (lane == 0) {
        v += bias ? bias[n] : 0.f;
        out[(size_t)b * N + n] = act_out ? silu(v) : v;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Backward of the skinny linear  out[b, n] = a[b, :] . W[n, :] + bias[n],  a = act_in(in)  (skinny_linear_kernel):
//   dW[n, k] = sum_b dout[b, n] a[b, k]     dbias[n] = sum_b dout[b, n]     da[b, k] += sum_n dout[b, n] W[n, k]
// One CTA per SKB_ROWS output rows n; a thread owns 4 consecutive k.  W is read once, dW written once.  Each CTA writes
// its partial da to part[cta] and skinny_da_reduce_kernel adds the partials into da in CTA order, so da does not depend
// on the order in which the CTAs finish (fp32 atomics did: run-to-run noise in every gradient behind da).
// ---------------------------------------------------------------------------------------------------------------
constexpr int SKB_ROWS = 128;

__global__ void __launch_bounds__(256) skinny_linear_bwd_kernel(const float* __restrict__ in, const float* __restrict__ W,
                                                                const float* __restrict__ dout, int ldo, int B, int N,
                                                                int K, int act_in, SkinnySegs segs,
                                                                float* __restrict__ part) {
  extern __shared__ float sm[];
  float* s_a = sm;               // [B, K]
  float* s_do = sm + B * K;      // [B, SKB_ROWS]
  const int n0 = blockIdx.x * SKB_ROWS, nrows = min(SKB_ROWS, N - n0);
  // destination of this CTA's rows: regular segments (one per DiT block) then up to two tail segments (the heads)
  float* dW;
  float* dbias;
  {
    const int reg_rows = segs.seg_rows * segs.n_seg;
    if (n0 < reg_rows) {
      const int sg = n0 / segs.seg_rows, r0 = n0 - sg * segs.seg_rows;
      dW = segs.dW0 + (size_t)sg * segs.seg_stride + (size_t)r0 * K;
      dbias = segs.db0 ? segs.db0 + (size_t)sg * segs.seg_stride + r0 : nullptr;
    } else {
      int r0 = n0 - reg_rows, t = 0;
      if (r0 >= segs.tail_rows[0]) { r0 -= segs.tail_rows[0]; t = 1; }
      dW = segs.tail_dW[t] + (size_t)r0 * K;
      dbias = segs.tail_db[t] ? segs.tail_db[t] + r0 : nullptr;
    }
  }
  for (int t = threadIdx.x; t < B * K; t += 256) {
    const float v = in[t];
    s_a[t] = act_in ? silu(v) : v;
  }
  for (int t = threadIdx.x; t < B * SKB_ROWS; t += 256) {
    const int b = t / SKB_ROWS, r = t - b * SKB_ROWS;
    s_do[t] = r < nrows ? dout[(size_t)b * ldo + n0 + r] : 0.f;
  }
  __syncthreads();
  if (dbias && threadIdx.x < nrows) {
    float s = 0.f;
    for (int b = 0; b < B; b++) s += s_do[b * SKB_ROWS + threadIdx.x];
    dbias[threadIdx.x] = s;
  }
  for (int k = threadIdx.x * 4; k < K; k += 1024) {
    float acc[SKINNY_MAXB][4];
    float a[SKINNY_MAXB][4];
#pragma unroll
    for (int b = 0; b < SKINNY_MAXB; b++) {
#pragma unroll
      for (int e = 0; e < 4; e++) { acc[b][e] = 0.f; a[b][e] = b < B ? s_a[b * K + k + e] : 0.f; }
    }
    for (int r = 0; r < nrows; r++) {
      const float4 w4 = __ldg(reinterpret_cast<const float4*>(W + (size_t)(n0 + r) * K + k));
      float4 g4 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int b = 0; b < SKINNY_MAXB; b++) {
        if (b < B) {
          const float d = s_do[b * SKB_ROWS + r];
          g4.x += d * a[b][0]; g4.y += d * a[b][1]; g4.z += d * a[b][2]; g4.w += d * a[b][3];
          acc[b][0] += d * w4.x; acc[b][1] += d * w4.y; acc[b][2] += d * w4.z; acc[b][3] += d * w4.w;
        }
      }
      *reinterpret_cast<float4*>(dW + (size_t)r * K + k) = g4;
    }
    if (part) {
      float* pc = part + (size_t)blockIdx.x * B * K;
#pragma unroll
      for (int b = 0; b < SKINNY_MAXB; b++) {
        if (b < B) *reinterpret_cast<float4*>(pc + (size_t)b * K + k) = make_float4(acc[b][0], acc[b][1], acc[b][2], acc[b][3]);
      }
    }
  }
}

// da[i] += sum_c part[c][i], c = 0 .. n_part-1 in order (i < n = B*K)
__global__ void skinny_da_reduce_kernel(const float* __restrict__ part, int n_part, int n, float* __restrict__ da) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int c = 0; c < n_part; c++) s += part[(size_t)c * n + i];
  da[i] += s;
}

// dpre = dpost * silu'(pre)  (elementwise, in place on dpost)
__global__ void silu_bwd_kernel(float* __restrict__ d, const float* __restrict__ pre, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = pre[i];
  const float sg = 1.0f / (1.0f + __expf(-x));
  d[i] *= sg * (1.0f + x * (1.0f - sg));
}

}  // namespace

int timestep_embedding(const float* t, float* out, int B, int dim, cudaStream_t st) {
  DGS_REQUIRE(dim % 2 == 0, "timestep_embedding: odd dim");
  timestep_embedding_kernel<<<ceil_div(B * dim / 2, 128), 128, 0, st>>>(t, out, B, dim);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

int skinny_linear(const float* in, const float* W, const float* bias, float* out, int B, int N, int K,
                  int act_in, int act_out_silu, cudaStream_t st) {
  DGS_REQUIRE(B >= 1 && K % 8 == 0, "skinny_linear: bad shape B=%d K=%d", B, K);
  for (int b0 = 0; b0 < B; b0 += SKINNY_MAXB) {
    const int nb = (B - b0) < SKINNY_MAXB ? (B - b0) : SKINNY_MAXB;
    const size_t smem = (size_t)nb * K * sizeof(float);
    skinny_linear_kernel<<<ceil_div(N, 8), 256, smem, st>>>(in + (size_t)b0 * K, W, bias, out + (size_t)b0 * N, nb, N,
                                                            K, act_in, act_out_silu);
    DGS_POST_LAUNCH();
  }
  return DGS_OK;
}

int skinny_linear_bwd_segs(const float* in, const float* W, const float* dout, int ldo, int B, int N, int K, int act_in,
                           const SkinnySegs& segs, float* da, float* part, cudaStream_t st) {
  DGS_REQUIRE(B >= 1 && B <= SKINNY_MAXB && K % 4 == 0, "skinny_linear_bwd: bad shape B=%d K=%d (B <= 8)", B, K);
  DGS_REQUIRE(!da || part, "skinny_linear_bwd: da needs the partial-sum scratch");
  DGS_REQUIRE(segs.seg_rows % SKB_ROWS == 0 && segs.tail_rows[0] % SKB_ROWS == 0 &&
                  segs.seg_rows * segs.n_seg + segs.tail_rows[0] + segs.tail_rows[1] == N,
              "skinny_linear_bwd: segments must be multiples of %d rows and cover N", SKB_ROWS);
  const size_t smem = ((size_t)B * K + (size_t)B * SKB_ROWS) * sizeof(float);
  static bool configured = false;
  if (!configured) {
    DGS_CUDA_OK(cudaFuncSetAttribute(skinny_linear_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    configured = true;
  }
  DGS_REQUIRE(smem <= 96 * 1024, "skinny_linear_bwd: B*K too large");
  const int n_part = ceil_div(N, SKB_ROWS);
  skinny_linear_bwd_kernel<<<n_part, 256, smem, st>>>(in, W, dout, ldo, B, N, K, act_in, segs, da ? part : nullptr);
  DGS_POST_LAUNCH();
  if (da) {
    skinny_da_reduce_kernel<<<ceil_div(B * K, 256), 256, 0, st>>>(part, n_part, B * K, da);
    DGS_POST_LAUNCH();
  }
  return DGS_OK;
}

size_t skinny_linear_bwd_part_floats(int B, int N, int K) { return (size_t)ceil_div(N, SKB_ROWS) * B * K; }

int skinny_linear_bwd(const float* in, const float* W, const float* dout, int ldo, int B, int N, int K, int act_in,
                      float* dW, float* dbias, float* da, float* part, cudaStream_t st) {
  SkinnySegs segs;
  segs.seg_rows = N; segs.n_seg = 1; segs.seg_stride = 0; segs.dW0 = dW; segs.db0 = dbias;
  if (N % SKB_ROWS) {  // a single ragged segment: express it as a tail (no alignment requirement on the last one)
    segs.seg_rows = 0; segs.n_seg = 0; segs.tail_rows[0] = 0; segs.tail_rows[1] = N; segs.tail_dW[1] = dW; segs.tail_db[1] = dbias;
  }
  return skinny_linear_bwd_segs(in, W, dout, ldo, B, N, K, act_in, segs, da, part, st);
}

int silu_bwd_inplace(float* d, const float* pre, int n, cudaStream_t st) {
  silu_bwd_kernel<<<ceil_div(n, 256), 256, 0, st>>>(d, pre, n);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

// ---------------------------------------------------------------------------------------------
// The tiny linear of the free Gaussian tokens' head (rows = B*G, N = C channels), forward and backward.
// ---------------------------------------------------------------------------------------------
namespace {

__global__ void tiny_linear_kernel(const __nv_bfloat16* __restrict__ h, const __nv_bfloat16* __restrict__ W,
                                   float* __restrict__ out, int rows, int N, int K) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows * N) return;
  const int r = warp / N, n = warp - r * N;
  float acc = 0.f;
  for (int k = lane; k < K; k += 32) acc += __bfloat162float(h[(size_t)r * K + k]) * __bfloat162float(W[(size_t)n * K + k]);
  acc = warp_sum(acc);
  if (lane == 0) out[(size_t)r * N + n] = acc;
}

// dh[r, k] = sum_n dy[r, n] W[n, k] (bf16 out), dW[n, k] = sum_r dy[r, n] h[r, k]  with h = hi + lo of the split-bf16
// operand [rows, 3K].
__global__ void tiny_linear_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ W,
                                       const __nv_bfloat16* __restrict__ h3, __nv_bfloat16* __restrict__ dh,
                                       float* __restrict__ dW, int rows, int N, int K) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  for (int r = 0; r < rows; r++) {
    float s = 0.f;
    for (int n = 0; n < N; n++) s += dy[r * N + n] * W[(size_t)n * K + k];
    dh[(size_t)r * K + k] = __float2bfloat16_rn(s);
  }
  for (int n = 0; n < N; n++) {
    float s = 0.f;
    for (int r = 0; r < rows; r++)
      s += dy[r * N + n] * (__bfloat162float(h3[(size_t)r * 3 * K + k]) + __bfloat162float(h3[(size_t)r * 3 * K + K + k]));
    dW[(size_t)n * K + k] = s;
  }
}

}  // namespace

int tiny_linear_bf16(const __nv_bfloat16* h, const __nv_bfloat16* W, float* out, int rows, int N, int K,
                     cudaStream_t st) {
  tiny_linear_kernel<<<ceil_div(rows * N * 32, 256), 256, 0, st>>>(h, W, out, rows, N, K);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

int tiny_linear_bwd(const float* dy, const float* W, const __nv_bfloat16* h3, __nv_bfloat16* dh, float* dW, int rows,
                    int N, int K, cudaStream_t st) {
  tiny_linear_bwd_kernel<<<ceil_div(K, 128), 128, 0, st>>>(dy, W, h3, dh, dW, rows, N, K);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

// ---------------------------------------------------------------------------------------------
// Gaussian heads' epilogue: to_gs + pixel alignment (denoiser.py:103-120, 362-413), one thread per Gaussian, and its
// backward: gradients w.r.t. the renderer-ready tensors -> gradients of the raw C-channel head outputs (free tokens
// fp32, image tokens bf16).  Both are templated on the SH degree SH: a Gaussian's raw row is
// C = 11 + 3 (SH+1)^2 channels [xyz 3 | features NF = 3 (SH+1)^2 | scaling 3 | rotation 4 | opacity 1], kept in
// registers whole (C <= 59: no spills).
// ---------------------------------------------------------------------------------------------
namespace {

template <int SH>
struct GsLayout {
  static constexpr int NF = 3 * (SH + 1) * (SH + 1);  // feature channels, coefficient-major, RGB-minor
  static constexpr int SC = 3 + NF, ROT = SC + 3, OP = ROT + 4, C = OP + 1;
};

// An image Gaussian sits at o + t d on its pixel's ray, with t a function of sg = sigmoid(mean of its 3 xyz channels):
//   scene 1: sg * (far - near) + near                 (denoiser_scene.py:263,406-410)
//   scene 2: sg                                       (denoiser.py:381-388 with ray_pe_type == 'plk')
//   scene 0: (2 sg - 1) * 1.8 - o . d                 (denoiser.py:382-392)
constexpr float OBJ_DEPTH_HALF_RANGE = 1.8f;
__device__ __forceinline__ float pixel_depth(int scene, float sg, float near_, float far_, float3 o, float3 d) {
  if (scene == 1) return sg * (far_ - near_) + near_;
  if (scene == 2) return sg;
  return (2.0f * sg - 1.0f) * OBJ_DEPTH_HALF_RANGE + (-o.x * d.x + -o.y * d.y + -o.z * d.z);
}
// d pixel_depth / d m, m the sigmoid's argument
__device__ __forceinline__ float pixel_depth_dm(int scene, float sg, float near_, float far_) {
  return (scene == 1 ? (far_ - near_) : scene == 2 ? 1.0f : 2.0f * OBJ_DEPTH_HALF_RANGE) * sg * (1.0f - sg);
}

template <int SH>
__global__ void __launch_bounds__(256) gaussians_epilogue_kernel(const float* __restrict__ gs_tok,
                                                                 const float* __restrict__ img_gs,
                                                                 const float* __restrict__ ray_o,
                                                                 const float* __restrict__ ray_d, GsOut out, int B,
                                                                 int G, int V, int H, int W, int p, int scene,
                                                                 float near_, float far_) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long per_b = (long long)G + (long long)V * H * W;
  if (idx >= (long long)B * per_b) return;
  const int b = (int)(idx / per_b);
  const long long g = idx - (long long)b * per_b;
  using Ly = GsLayout<SH>;
  constexpr int C = Ly::C;
  float a[C];
  float xyz[3];
  if (g < G) {
    const float* s = gs_tok + ((size_t)b * G + g) * C;
#pragma unroll
    for (int k = 0; k < C; k++) a[k] = s[k];
    xyz[0] = a[0]; xyz[1] = a[1]; xyz[2] = a[2];
  } else {
    const long long q = g - G;  // (v, hh, ww, ph, pw) order == img_gs memory order
    const float* s = img_gs + ((size_t)b * V * H * W + q) * C;  // scalar loads: rows of odd C are not 8-byte aligned
#pragma unroll
    for (int k = 0; k < C; k++) a[k] = s[k];
    const PatchPixel px = patch_pixel(q, H, W, p);
    const size_t plane = (size_t)H * W, pix = (size_t)px.y * W + px.x;
    const size_t base = ((size_t)b * V + px.bv) * 3 * plane + pix;
    const float3 o = make_float3(ray_o[base], ray_o[base + plane], ray_o[base + 2 * plane]);
    const float3 d = make_float3(ray_d[base], ray_d[base + plane], ray_d[base + 2 * plane]);
    const float m = (a[0] + a[1] + a[2]) / 3.0f;
    const float sg = 1.0f / (1.0f + expf(-m));
    const float t = pixel_depth(scene, sg, near_, far_, o, d);
    xyz[0] = o.x + t * d.x; xyz[1] = o.y + t * d.y; xyz[2] = o.z + t * d.z;
    if (out.img_aligned_xyz) {
      out.img_aligned_xyz[base] = xyz[0];
      out.img_aligned_xyz[base + plane] = xyz[1];
      out.img_aligned_xyz[base + 2 * plane] = xyz[2];
    }
  }
  const size_t o = (size_t)idx;
  out.xyz[3 * o] = xyz[0]; out.xyz[3 * o + 1] = xyz[1]; out.xyz[3 * o + 2] = xyz[2];
#pragma unroll
  for (int k = 0; k < Ly::NF; k++) out.features[Ly::NF * o + k] = a[3 + k];  // [.., (SH+1)^2, 3]: a plain copy
  out.scaling[3 * o] = fminf(a[Ly::SC] - 2.3f, -1.2f);  // denoiser.py:118
  out.scaling[3 * o + 1] = fminf(a[Ly::SC + 1] - 2.3f, -1.2f);
  out.scaling[3 * o + 2] = fminf(a[Ly::SC + 2] - 2.3f, -1.2f);
  *reinterpret_cast<float4*>(out.rotation + 4 * o) = make_float4(a[Ly::ROT], a[Ly::ROT + 1], a[Ly::ROT + 2], a[Ly::ROT + 3]);
  out.opacity[o] = a[Ly::OP] - 2.0f;  // denoiser.py:119
}

// img_xyz: NULL, or the gradient of img_aligned_xyz [B,V,3,H,W] -- the image Gaussians' xyz in the pixel layout, so it
// adds to their d xyz exactly
struct GsGrad {
  const float* xyz; const float* features; const float* scaling; const float* rotation; const float* opacity;
  const float* img_xyz;
};

template <int SH>
__global__ void __launch_bounds__(256) gaussians_epilogue_bwd_kernel(const float* __restrict__ gs_tok,
                                                                     const float* __restrict__ img_gs,
                                                                     const float* __restrict__ ray_d, GsGrad d,
                                                                     float* __restrict__ d_gs_tok,
                                                                     __nv_bfloat16* __restrict__ d_img_gs, int B, int G,
                                                                     int V, int H, int W, int p, int scene, float near_,
                                                                     float far_) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long per_b = (long long)G + (long long)V * H * W;
  if (idx >= (long long)B * per_b) return;
  const int b = (int)(idx / per_b);
  const long long g = idx - (long long)b * per_b;
  const size_t o = (size_t)idx;
  using Ly = GsLayout<SH>;
  constexpr int C = Ly::C;
  float da[C];
  const float* src = (g < G) ? gs_tok + ((size_t)b * G + g) * C : img_gs + ((size_t)b * V * H * W + (g - G)) * C;
  float gx = d.xyz[3 * o], gy = d.xyz[3 * o + 1], gz = d.xyz[3 * o + 2];
  if (g < G) {
    da[0] = gx; da[1] = gy; da[2] = gz;
  } else {
    const PatchPixel px = patch_pixel(g - G, H, W, p);
    const size_t plane = (size_t)H * W, pix = (size_t)px.y * W + px.x;
    const size_t base = ((size_t)b * V + px.bv) * 3 * plane + pix;
    if (d.img_xyz) {
      gx += d.img_xyz[base];
      gy += d.img_xyz[base + plane];
      gz += d.img_xyz[base + 2 * plane];
    }
    const float d0 = ray_d[base], d1 = ray_d[base + plane], d2 = ray_d[base + 2 * plane];
    const float m = (src[0] + src[1] + src[2]) / 3.0f;
    const float sg = 1.0f / (1.0f + expf(-m));
    const float dt = gx * d0 + gy * d1 + gz * d2;  // xyz = o + t d
    da[0] = da[1] = da[2] = dt * pixel_depth_dm(scene, sg, near_, far_) * (1.0f / 3.0f);
  }
#pragma unroll
  for (int k = 0; k < Ly::NF; k++) da[3 + k] = d.features[Ly::NF * o + k];
#pragma unroll
  for (int k = 0; k < 3; k++)
    da[Ly::SC + k] = (src[Ly::SC + k] - 2.3f <= -1.2f) ? d.scaling[3 * o + k] : 0.f;  // clamp(max=-1.2)
  const float4 dr = *reinterpret_cast<const float4*>(d.rotation + 4 * o);
  da[Ly::ROT] = dr.x; da[Ly::ROT + 1] = dr.y; da[Ly::ROT + 2] = dr.z; da[Ly::ROT + 3] = dr.w;
  da[Ly::OP] = d.opacity[o];
  if (g < G) {
    float* dst = d_gs_tok + ((size_t)b * G + g) * C;
#pragma unroll
    for (int k = 0; k < C; k++) dst[k] = da[k];
  } else {
    __nv_bfloat16* dst = d_img_gs + ((size_t)b * V * H * W + (g - G)) * C;
    if constexpr (C % 2 == 0) {
#pragma unroll
      for (int k = 0; k < C; k += 2) {
        __nv_bfloat162 pk = __floats2bfloat162_rn(da[k], da[k + 1]);
        *reinterpret_cast<__nv_bfloat162*>(dst + k) = pk;
      }
    } else {  // odd C: every other row starts on a 2-byte boundary, so no pair stores.  Consecutive threads write
              // consecutive rows, so a warp's stores still fill whole sectors of one contiguous 32 C * 2-byte range.
#pragma unroll
      for (int k = 0; k < C; k++) dst[k] = __float2bfloat16_rn(da[k]);
    }
  }
}

}  // namespace

int gaussians_epilogue(const float* gs_tokens, const float* img_gs, const float* ray_o, const float* ray_d, GsOut out,
                       int B, int G, int V, int H, int W, int patch, int sh_degree, int scene_mode, float near_,
                       float far_, cudaStream_t st) {
  const long long total = (long long)B * ((long long)G + (long long)V * H * W);
  const dim3 grid((unsigned)((total + 255) / 256));
  switch (sh_degree) {
    case 0: gaussians_epilogue_kernel<0><<<grid, 256, 0, st>>>(gs_tokens, img_gs, ray_o, ray_d, out, B, G, V, H, W, patch,
                                                                scene_mode, near_, far_); break;
    case 1: gaussians_epilogue_kernel<1><<<grid, 256, 0, st>>>(gs_tokens, img_gs, ray_o, ray_d, out, B, G, V, H, W, patch,
                                                                scene_mode, near_, far_); break;
    case 2: gaussians_epilogue_kernel<2><<<grid, 256, 0, st>>>(gs_tokens, img_gs, ray_o, ray_d, out, B, G, V, H, W, patch,
                                                                scene_mode, near_, far_); break;
    case 3: gaussians_epilogue_kernel<3><<<grid, 256, 0, st>>>(gs_tokens, img_gs, ray_o, ray_d, out, B, G, V, H, W, patch,
                                                                scene_mode, near_, far_); break;
    default: DGS_REQUIRE(false, "gaussians_epilogue: sh_degree %d out of [0, 3]", sh_degree);
  }
  DGS_POST_LAUNCH();
  return DGS_OK;
}

int gaussians_epilogue_bwd(const float* gs_tok, const float* img_gs, const float* ray_d, const float* dxyz,
                           const float* dfeatures, const float* dscaling, const float* drotation, const float* dopacity,
                           const float* d_img_xyz, float* d_gs_tok, __nv_bfloat16* d_img_gs, int B, int G, int V, int H,
                           int W, int patch, int sh_degree, int scene_mode, float near_, float far_, cudaStream_t st) {
  GsGrad d{dxyz, dfeatures, dscaling, drotation, dopacity, d_img_xyz};
  const long long total = (long long)B * ((long long)G + (long long)V * H * W);
  const dim3 grid((unsigned)((total + 255) / 256));
  switch (sh_degree) {
    case 0: gaussians_epilogue_bwd_kernel<0><<<grid, 256, 0, st>>>(gs_tok, img_gs, ray_d, d, d_gs_tok, d_img_gs, B, G, V,
                                                                    H, W, patch, scene_mode, near_, far_); break;
    case 1: gaussians_epilogue_bwd_kernel<1><<<grid, 256, 0, st>>>(gs_tok, img_gs, ray_d, d, d_gs_tok, d_img_gs, B, G, V,
                                                                    H, W, patch, scene_mode, near_, far_); break;
    case 2: gaussians_epilogue_bwd_kernel<2><<<grid, 256, 0, st>>>(gs_tok, img_gs, ray_d, d, d_gs_tok, d_img_gs, B, G, V,
                                                                    H, W, patch, scene_mode, near_, far_); break;
    case 3: gaussians_epilogue_bwd_kernel<3><<<grid, 256, 0, st>>>(gs_tok, img_gs, ray_d, d, d_gs_tok, d_img_gs, B, G, V,
                                                                    H, W, patch, scene_mode, near_, far_); break;
    default: DGS_REQUIRE(false, "gaussians_epilogue_bwd: sh_degree %d out of [0, 3]", sh_degree);
  }
  DGS_POST_LAUNCH();
  return DGS_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Around the weight-gradient GEMMs: operand transposes (+ bias gradients), the gate / residual backward and the column
// sums of bf16 gradients.
// ---------------------------------------------------------------------------------------------------------------
namespace {

constexpr int TP = 72;  // smem tile pitch in bf16 elements (144 B: 16-byte aligned rows)

// The read-out of the 64 x 64 bf16 tile (m0, c0) in shared memory (row pitch TP) by 256 threads: thread t reads column
// c = t % 64 over rows mc = 16 (t / 64) .. + 15 (the lanes run along the columns: conflict-free), calls per_row(r) for
// each of those tile rows r in the same loop, stores the 16 values to the transposed matrix outT [C, ldT] (unless
// null) at outT[c0 + c, m0 + mc ..] (32 contiguous bytes) and returns their fp32 sum.
template <typename PerRow>
__device__ __forceinline__ float tile_column(const __nv_bfloat16* tile, int t, __nv_bfloat16* outT, int c0, int m0,
                                             int ldT, PerRow per_row) {
  const int c = t & 63, mc = (t >> 6) * 16;
  __align__(16) __nv_bfloat16 o[16];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 16; i++) {
    o[i] = tile[(mc + i) * TP + c];
    s += __bfloat162float(o[i]);
    per_row(mc + i);
  }
  if (outT) {
    __nv_bfloat16* dst = outT + (size_t)(c0 + c) * ldT + m0 + mc;
    *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(o);
    *reinterpret_cast<uint4*>(dst + 8) = *reinterpret_cast<const uint4*>(o + 8);
  }
  return s;
}

// out[c, m] = bf16(in[row(m), c]),  m = b * rows_out + j  ->  input row  b * rows_in + row_off + j;  out is [C, Mp]
// (Mp = round_up(M, 64), pad columns zero-filled: they are the K tail of the weight-gradient GEMM).
// colsum[c] += sum_m in[row(m), c]  (bias gradient), optional.
// 64 x 64 tile per CTA: 16-byte global loads -> smem -> tile_column -> 32-byte global stores.
template <typename TI>
__global__ void __launch_bounds__(256) transpose_kernel(const TI* __restrict__ in, int ldi, int rows_in, int row_off,
                                                        int rows_out, int M, int Mp, __nv_bfloat16* __restrict__ out,
                                                        float* __restrict__ colsum, __nv_bfloat16* __restrict__ out_rm,
                                                        int C, size_t in_bstride, size_t out_bstride, size_t rm_bstride) {
  __shared__ __align__(16) __nv_bfloat16 tile[64 * TP];
  __shared__ float red[4 * 64];
  const int m0 = blockIdx.x * 64, c0 = blockIdx.y * 64, t = threadIdx.x;
  ptx::griddep_launch_dependents();  // PDL: launched via launch_pdl
  ptx::griddep_wait();
  in += (size_t)blockIdx.z * in_bstride;   // batched use (weight refresh): one matrix per blockIdx.z
  out += (size_t)blockIdx.z * out_bstride;
  {
    const int lr = t >> 2, lc = (t & 3) * 16;
    const int m = m0 + lr;
    uint4 lo = make_uint4(0, 0, 0, 0), hi = lo;
    if (m < M) {
      const int b = m / rows_out, j = m - b * rows_out;
      load16_bf16(in + ((size_t)b * rows_in + row_off + j) * ldi + c0 + lc, lo, hi);
      if (out_rm) {  // optional plain (row-major) bf16 copy of the same tile
        __nv_bfloat16* rm = out_rm + (size_t)blockIdx.z * rm_bstride + (size_t)m * C + c0 + lc;
        *reinterpret_cast<uint4*>(rm) = lo;
        *reinterpret_cast<uint4*>(rm + 8) = hi;
      }
    }
    *reinterpret_cast<uint4*>(tile + lr * TP + lc) = lo;
    *reinterpret_cast<uint4*>(tile + lr * TP + lc + 8) = hi;
  }
  __syncthreads();
  const int c = t & 63, mq = t >> 6;
  const float s = tile_column(tile, t, out, c0, m0, Mp, [](int) {});
  if (colsum) {
    red[mq * 64 + c] = s;
    __syncthreads();
    if (t < 64) atomicAdd(colsum + c0 + t, quarter_sum(red, t));
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Backward of  x_out = x_in + gate[b] * y   (y = branch output incl. bias, saved pre-gate in bf16):
//   dy = gate[b] * dx  (bf16, row-major AND transposed [C, Mp]),  dgate[b, c] += sum_rows dx * y,  dbias[c] += sum dy
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) gate_bwd_kernel(const float* __restrict__ dx, const __nv_bfloat16* __restrict__ y,
                                                       const float* __restrict__ gate, int gate_stride,
                                                       int rows_per_sample, int M, int Mp, int C,
                                                       __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ dyT,
                                                       float* __restrict__ dgate, float* __restrict__ dbias) {
  __shared__ __align__(16) __nv_bfloat16 tile[64 * TP];
  __shared__ float prod[64 * 65];
  __shared__ float red[3 * 4 * 64];
  const int m0 = blockIdx.x * 64, c0 = blockIdx.y * 64, t = threadIdx.x;
  ptx::griddep_launch_dependents();  // PDL: launched via launch_pdl
  ptx::griddep_wait();
  {
    const int lr = t >> 2, lc = (t & 3) * 16;
    const int m = m0 + lr;
    if (m < M) {
      const int b = m / rows_per_sample;
      const float* g = gate + (size_t)b * gate_stride + c0 + lc;
      const float* dxr = dx + (size_t)m * C + c0 + lc;
      uint4 ylo, yhi;
      load16_bf16(y + (size_t)m * C + c0 + lc, ylo, yhi);
      const uint32_t yw[8] = {ylo.x, ylo.y, ylo.z, ylo.w, yhi.x, yhi.y, yhi.z, yhi.w};
      uint32_t pk[8];
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const float4 d4 = *reinterpret_cast<const float4*>(dxr + 4 * q);
        const float4 g4 = __ldg(reinterpret_cast<const float4*>(g + 4 * q));
        const float2 y0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&yw[2 * q]));
        const float2 y1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&yw[2 * q + 1]));
        pk[2 * q] = ptx::pack2_bf16(d4.x * g4.x, d4.y * g4.y);
        pk[2 * q + 1] = ptx::pack2_bf16(d4.z * g4.z, d4.w * g4.w);
        float* pr = prod + lr * 65 + lc + 4 * q;
        pr[0] = d4.x * y0.x; pr[1] = d4.y * y0.y; pr[2] = d4.z * y1.x; pr[3] = d4.w * y1.y;
      }
      const uint4 lo = make_uint4(pk[0], pk[1], pk[2], pk[3]), hi = make_uint4(pk[4], pk[5], pk[6], pk[7]);
      *reinterpret_cast<uint4*>(tile + lr * TP + lc) = lo;
      *reinterpret_cast<uint4*>(tile + lr * TP + lc + 8) = hi;
      __nv_bfloat16* o = dy + (size_t)m * C + c0 + lc;
      *reinterpret_cast<uint4*>(o) = lo;
      *reinterpret_cast<uint4*>(o + 8) = hi;
    } else {
#pragma unroll
      for (int i = 0; i < 16; i++) prod[lr * 65 + lc + i] = 0.f;
      *reinterpret_cast<uint4*>(tile + lr * TP + lc) = make_uint4(0, 0, 0, 0);
      *reinterpret_cast<uint4*>(tile + lr * TP + lc + 8) = make_uint4(0, 0, 0, 0);
    }
  }
  __syncthreads();
  const int c = t & 63, mq = t >> 6;
  const int b_first = m0 / rows_per_sample;
  const int split = (b_first + 1) * rows_per_sample - m0;  // tile rows >= split belong to sample b_first + 1
  float g0 = 0.f, g1 = 0.f;
  // dyT: the transposed copy, only for the K-major weight-gradient path
  const float s = tile_column(tile, t, dyT, c0, m0, Mp, [&](int r) {
    const float p = prod[r * 65 + c];
    if (r < split) g0 += p; else g1 += p;
  });
  red[mq * 64 + c] = s;
  red[256 + mq * 64 + c] = g0;
  red[512 + mq * 64 + c] = g1;
  __syncthreads();
  if (t < 64) {
    const float ss = quarter_sum(red, t);
    const float s0 = quarter_sum(red, 256 + t);
    const float s1 = quarter_sum(red, 512 + t);
    if (dbias) atomicAdd(dbias + c0 + t, ss);
    atomicAdd(dgate + (size_t)b_first * gate_stride + c0 + t, s0);
    if (split < 64 && m0 + split < M) atomicAdd(dgate + (size_t)(b_first + 1) * gate_stride + c0 + t, s1);
  }
}

// colsum[c] += sum_m in[m, c]  (bias gradient of a linear whose output gradient `in` is [M, C] bf16)
// A CTA owns 256 columns x COLSUM_ROWS rows: every lane reads 8 consecutive columns with ONE 16-byte load (512 contiguous
// bytes per warp and row; the first version read 2 bytes per thread = 64 bytes per warp instruction and ran at 30 % of the
// HBM bandwidth: 61 us for the [16392, 3072] qkv gradient), the 8 warps take rows r0 + warp, r0 + warp + 8, ...
constexpr int COLSUM_ROWS = 512;
__global__ void __launch_bounds__(256) colsum_kernel(const __nv_bfloat16* __restrict__ in, int M, int C,
                                                     float* __restrict__ colsum) {
  __shared__ float red[8][256];
  ptx::griddep_launch_dependents();  // PDL: launched via launch_pdl
  ptx::griddep_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = blockIdx.x * 256 + lane * 8;
  const int r0 = blockIdx.y * COLSUM_ROWS, r_end = min(M, r0 + COLSUM_ROWS);
  float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (c0 < C) {  // C % 64 == 0 and 8 columns per lane: a lane is either fully inside or fully outside
#pragma unroll 4
    for (int r = r0 + warp; r < r_end; r += 8) {
      const uint4 v = *reinterpret_cast<const uint4*>(in + (size_t)r * C + c0);
      const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const float2 f = __bfloat1622float2(p[i]);
        a[2 * i] += f.x;
        a[2 * i + 1] += f.y;
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; i++) red[warp][lane * 8 + i] = a[i];
  __syncthreads();
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c < C) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; w++) t += red[w][threadIdx.x];
    atomicAdd(colsum + c, t);
  }
}

}  // namespace

template <typename TI>
int transpose_to_bf16(const TI* in, int ldi, int B, int rows_in, int row_off, int rows_out, int C, __nv_bfloat16* out,
                      float* colsum, cudaStream_t st) {
  DGS_REQUIRE(C % 64 == 0 && ldi % 8 == 0, "transpose: need C %% 64 == 0 (C=%d ldi=%d)", C, ldi);
  const int M = B * rows_out, Mp = (M + 63) / 64 * 64;
  DGS_CUDA_OK(launch_pdl(transpose_kernel<TI>, dim3(Mp / 64, C / 64), dim3(256), 0, st, in, ldi, rows_in, row_off,
                         rows_out, M, Mp, out, colsum, (__nv_bfloat16*)nullptr, C, (size_t)0, (size_t)0, (size_t)0));
  DGS_POST_LAUNCH();
  return DGS_OK;
}
template int transpose_to_bf16(const float*, int, int, int, int, int, int, __nv_bfloat16*, float*, cudaStream_t);
template int transpose_to_bf16(const __nv_bfloat16*, int, int, int, int, int, int, __nv_bfloat16*, float*, cudaStream_t);

// batch x [M, C] fp32 (matrix i at in + i * in_bstride) -> bf16 copies [batch, M, C] and/or transposed [batch, C, M]
int cast_transpose_f32(const float* in, long long in_bstride, int batch, int M, int C, __nv_bfloat16* out_rm,
                       __nv_bfloat16* outT, cudaStream_t st) {
  DGS_REQUIRE(M % 64 == 0 && C % 64 == 0 && outT != nullptr, "cast_transpose: need M, C multiples of 64 and outT");
  dim3 grid(M / 64, C / 64, batch);
  DGS_CUDA_OK(launch_pdl(transpose_kernel<float>, grid, dim3(256), 0, st, in, C, M, 0, M, M, M, outT, (float*)nullptr, out_rm, C,
                         (size_t)in_bstride, (size_t)M * C, (size_t)M * C));
  DGS_POST_LAUNCH();
  return DGS_OK;
}

int gate_bwd(const float* dx, const __nv_bfloat16* y, const float* gate, int gate_stride, int rows_per_sample, int M,
             int C, __nv_bfloat16* dy, __nv_bfloat16* dyT, float* dgate, float* dbias, cudaStream_t st) {
  DGS_REQUIRE(C % 64 == 0 && rows_per_sample >= 64, "gate_bwd: need C %% 64 == 0 and >= 64 rows per sample");
  const int Mp = (M + 63) / 64 * 64;
  DGS_CUDA_OK(launch_pdl(gate_bwd_kernel, dim3(Mp / 64, C / 64), dim3(256), 0, st, dx, y, gate, gate_stride, rows_per_sample, M,
                         Mp, C, dy, dyT, dgate, dbias));
  DGS_POST_LAUNCH();
  return DGS_OK;
}

int colsum_bf16(const __nv_bfloat16* in, int M, int C, float* colsum, cudaStream_t st) {
  DGS_REQUIRE(C % 64 == 0, "colsum: need C %% 64 == 0");
  DGS_REQUIRE(((uintptr_t)in % 16) == 0, "colsum: input must be 16-byte aligned");
  DGS_CUDA_OK(launch_pdl(colsum_kernel, dim3(ceil_div(C, 256), ceil_div(M, COLSUM_ROWS)), dim3(256), 0, st, in, M, C, colsum));
  DGS_POST_LAUNCH();
  return DGS_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// AdamW (torch.optim.AdamW semantics: decoupled weight decay, bias-corrected moments), fp32 master weights
// ---------------------------------------------------------------------------------------------------------------
namespace {
__global__ void adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                             float* __restrict__ v, size_t n, float lr, float b1, float b2, float eps, float wd,
                             float bc1, float bc2_sqrt, float grad_scale, const float* __restrict__ grad_scale_dev,
                             float* __restrict__ ema, float ema_decay) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (grad_scale_dev) grad_scale *= __ldg(grad_scale_dev);  // e.g. the clip factor, computed on the device
  const float gi = g[i] * grad_scale;
  const float mi = b1 * m[i] + (1.0f - b1) * gi;
  const float vi = b2 * v[i] + (1.0f - b2) * gi * gi;
  m[i] = mi;
  v[i] = vi;
  float pi = p[i] * (1.0f - lr * wd);
  pi -= (lr / bc1) * mi / (sqrtf(vi) / bc2_sqrt + eps);
  p[i] = pi;
  if (ema) ema[i] = ema_decay * ema[i] + (1.0f - ema_decay) * pi;  // ema.py:82-101 (multi_tensor_axpby form)
}
}  // namespace

int adamw_step(float* p, const float* g, float* m, float* v, size_t n, float lr, float b1, float b2, float eps, float wd,
               int step, float grad_scale, const float* grad_scale_dev, cudaStream_t st, float* ema, float ema_decay) {
  if (n == 0) return DGS_OK;
  const float bc1 = 1.0f - powf(b1, (float)step), bc2 = 1.0f - powf(b2, (float)step);
  adamw_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(p, g, m, v, n, lr, b1, b2, eps, wd, bc1, sqrtf(bc2),
                                                            grad_scale, grad_scale_dev, ema, ema_decay);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

}  // namespace dgs
