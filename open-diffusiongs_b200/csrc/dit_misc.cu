// dit_misc.cu -- the memory-bound glue kernels of the DiT denoiser (everything that is not a GEMM or the
// attention): posed-image patchify, token assembly + input LayerNorm, LayerNorm+adaLN modulate, the skinny
// (batch-row) linears of the timestep / adaLN MLPs, the Gaussian heads' epilogue (to_gs + pixel alignment).
// Spec: diffusionGS/models/denoiser/denoiser.py:26-72,76-164,306-416 and denoiser_scene.py:314-429,
//       diffusionGS/models/transformers/utils_transformer.py:26-27,246-290.
#include "dgs_internal.h"
#include "dit_kernels.h"
#include "sm90_ptx.cuh"

namespace dgs {

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------------------------------------
// LayerNorm (+ optional weight) + adaLN modulate -> bf16.  One warp per row, D = 32 * 4 * VEC.
// Two-pass statistics in registers (mean, then centred variance) = torch's LayerNorm numerics.
// ---------------------------------------------------------------------------------------------
// one warp loads row xr into v (lane l holds float4 number i of the row at columns 4 (32 i + l) .. + 3) and returns
// its mean and 1 / sqrt(var + eps)
template <int D>
__device__ __forceinline__ void ln_row_stats(const float* xr, int lane, float (&v)[D / 32], float eps, float& mean,
                                             float& rstd) {
  constexpr int PER_LANE = D / 32;
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < PER_LANE / 4; i++) {
    const float4 t = *reinterpret_cast<const float4*>(xr + (i * 32 + lane) * 4);
    v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
    s += t.x + t.y + t.z + t.w;
  }
  mean = warp_sum_f(s) * (1.0f / D);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < PER_LANE; i++) { const float d = v[i] - mean; q += d * d; }
  rstd = rsqrtf(warp_sum_f(q) * (1.0f / D) + eps);
}

template <int D>
__global__ void __launch_bounds__(256) ln_modulate_kernel(const float* __restrict__ x, const float* __restrict__ lnw,
                                                          const float* __restrict__ shift,
                                                          const float* __restrict__ scale, int mod_stride,
                                                          __nv_bfloat16* __restrict__ h, int B, int rows_in,
                                                          int row_off, int rows_out, float eps, int split) {
  constexpr int PER_LANE = D / 32;  // 32 for D = 1024
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");  // PDL (sm90_ptx.cuh): launched via launch_pdl
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (warp >= B * rows_out) return;
  const int b = warp / rows_out, r = warp - b * rows_out;
  const float* xr = x + ((size_t)b * rows_in + row_off + r) * D;
  float v[PER_LANE];
  float mean, rstd;
  ln_row_stats<D>(xr, lane, v, eps, mean, rstd);
  const float* sh = shift + (size_t)b * mod_stride;
  const float* sc = scale + (size_t)b * mod_stride;
  __nv_bfloat16* hr = h + (size_t)warp * D * (split ? 3 : 1);
#pragma unroll
  for (int i = 0; i < PER_LANE / 4; i++) {
    const int c = (i * 32 + lane) * 4;
    const float4 s4 = __ldg(reinterpret_cast<const float4*>(sc + c));
    const float4 h4 = __ldg(reinterpret_cast<const float4*>(sh + c));
    float4 w4 = make_float4(1.f, 1.f, 1.f, 1.f);
    if (lnw) w4 = __ldg(reinterpret_cast<const float4*>(lnw + c));
    const float o0 = (v[4 * i] - mean) * rstd * w4.x * (1.f + s4.x) + h4.x;
    const float o1 = (v[4 * i + 1] - mean) * rstd * w4.y * (1.f + s4.y) + h4.y;
    const float o2 = (v[4 * i + 2] - mean) * rstd * w4.z * (1.f + s4.z) + h4.z;
    const float o3 = (v[4 * i + 3] - mean) * rstd * w4.w * (1.f + s4.w) + h4.w;
    __nv_bfloat162 p0 = __floats2bfloat162_rn(o0, o1), p1 = __floats2bfloat162_rn(o2, o3);
    uint2 pk;
    pk.x = *reinterpret_cast<uint32_t*>(&p0);
    pk.y = *reinterpret_cast<uint32_t*>(&p1);
    *reinterpret_cast<uint2*>(hr + c) = pk;
    if (split) {  // [hi | lo | hi]: x = hi + lo to ~2^-17 relative (split-bf16 operand of the head GEMMs)
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

int ln_modulate(const float* x, const float* ln_weight, const float* shift, const float* scale, int mod_stride,
                __nv_bfloat16* h, int B, int rows_in, int row_off, int rows_out, int D, float eps, int split,
                cudaStream_t st) {
  DGS_REQUIRE(D == 1024, "ln_modulate: width %d not supported (1024 only)", D);
  const long long warps = (long long)B * rows_out;
  const int blocks = (int)((warps * 32 + 255) / 256);
  DGS_CUDA_OK(launch_pdl(ln_modulate_kernel<1024>, dim3(blocks), dim3(256), 0, st, x, ln_weight, shift, scale, mod_stride, h,
                         B, rows_in, row_off, rows_out, eps, split));
  DGS_POST_LAUNCH();
  return DGS_OK;
}

// LayerNorm + modulate -> e4m3 with 1 x 128 group scales (the FP8 GEMMs' A operand).  The LayerNorm and modulate
// arithmetic is ln_modulate_kernel's; lane l's float4 number i lies in column group i, so each group's amax is one warp
// reduction.
template <int D>
__global__ void __launch_bounds__(256) ln_modulate_fp8_kernel(const float* __restrict__ x,
                                                              const float* __restrict__ shift,
                                                              const float* __restrict__ scale, int mod_stride,
                                                              uint8_t* __restrict__ q, float* __restrict__ q_scale,
                                                              int lds, int B, int rows, float eps) {
  constexpr int PER_LANE = D / 32, GROUPS = D / 128;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (warp >= B * rows) return;
  const int b = warp / rows;
  float v[PER_LANE];
  float mean, rstd;
  ln_row_stats<D>(x + (size_t)warp * D, lane, v, eps, mean, rstd);
  const float* sh = shift + (size_t)b * mod_stride;
  const float* sc = scale + (size_t)b * mod_stride;
  uint8_t* qr = q + (size_t)warp * D;
#pragma unroll
  for (int i = 0; i < GROUPS; i++) {
    const int c = (i * 32 + lane) * 4;
    const float4 s4 = __ldg(reinterpret_cast<const float4*>(sc + c));
    const float4 h4 = __ldg(reinterpret_cast<const float4*>(sh + c));
    const float o0 = (v[4 * i] - mean) * rstd * (1.f + s4.x) + h4.x;
    const float o1 = (v[4 * i + 1] - mean) * rstd * (1.f + s4.y) + h4.y;
    const float o2 = (v[4 * i + 2] - mean) * rstd * (1.f + s4.z) + h4.z;
    const float o3 = (v[4 * i + 3] - mean) * rstd * (1.f + s4.w) + h4.w;
    float amax = fmaxf(fmaxf(fabsf(o0), fabsf(o1)), fmaxf(fabsf(o2), fabsf(o3)));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const int e = ptx::e4m3_scale_exp(amax);
    const float inv = ptx::exp2_int(-e);
    const uint32_t packed = (uint32_t)ptx::pack2_e4m3(o0 * inv, o1 * inv) | ((uint32_t)ptx::pack2_e4m3(o2 * inv, o3 * inv) << 16);
    *reinterpret_cast<uint32_t*>(qr + c) = packed;
    if (lane == 0) q_scale[(size_t)i * lds + warp] = ptx::exp2_int(e);
  }
}

int ln_modulate_fp8(const float* x, const float* shift, const float* scale, int mod_stride, uint8_t* q, float* q_scale,
                    int B, int rows, int D, float eps, cudaStream_t st) {
  DGS_REQUIRE(D == 1024, "ln_modulate_fp8: width %d not supported (1024 only)", D);
  DGS_REQUIRE(B > 0 && rows > 0, "ln_modulate_fp8: bad shape B=%d rows=%d", B, rows);
  const long long warps = (long long)B * rows;
  const int blocks = (int)((warps * 32 + 255) / 256);
  DGS_CUDA_OK(launch_pdl(ln_modulate_fp8_kernel<1024>, dim3(blocks), dim3(256), 0, st, x, shift, scale, mod_stride, q,
                         q_scale, fp8_scale_stride(B * rows), B, rows, eps));
  DGS_POST_LAUNCH();
  return DGS_OK;
}

// One block per row: amax, then the row times 2^-e rounded to e4m3 (the FP8 weight format, one scale per row).
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

int quantize_rows_e4m3(const float* x, int rows, int cols, uint8_t* q, float* scale, cudaStream_t st) {
  DGS_REQUIRE(rows > 0 && cols > 0, "quantize_rows_e4m3: bad shape %dx%d", rows, cols);
  quantize_rows_e4m3_kernel<<<rows, 256, 0, st>>>(x, cols, q, scale);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

template <int D>
__global__ void __launch_bounds__(256) ln_weight_kernel(float* __restrict__ x, const float* __restrict__ w, int rows,
                                                        float eps) {
  constexpr int PER_LANE = D / 32;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  float* xr = x + (size_t)warp * D;
  float v[PER_LANE];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < PER_LANE / 4; i++) {
    const float4 t = *reinterpret_cast<const float4*>(xr + (i * 32 + lane) * 4);
    v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
    s += t.x + t.y + t.z + t.w;
  }
  const float mean = warp_sum_f(s) * (1.0f / D);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < PER_LANE; i++) { const float d = v[i] - mean; q += d * d; }
  const float rstd = rsqrtf(warp_sum_f(q) * (1.0f / D) + eps);
#pragma unroll
  for (int i = 0; i < PER_LANE / 4; i++) {
    const int c = (i * 32 + lane) * 4;
    const float4 w4 = __ldg(reinterpret_cast<const float4*>(w + c));
    *reinterpret_cast<float4*>(xr + c) =
        make_float4((v[4 * i] - mean) * rstd * w4.x, (v[4 * i + 1] - mean) * rstd * w4.y,
                    (v[4 * i + 2] - mean) * rstd * w4.z, (v[4 * i + 3] - mean) * rstd * w4.w);
  }
}

int ln_weight_inplace(float* x, const float* w, int rows, int D, float eps, cudaStream_t st) {
  DGS_REQUIRE(D == 1024, "ln_weight: width %d not supported (1024 only)", D);
  ln_weight_kernel<1024><<<(int)(((long long)rows * 32 + 255) / 256), 256, 0, st>>>(x, w, rows, eps);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

// ---------------------------------------------------------------------------------------------
// Skinny linear: out[b, n] = act(in[b, :]) . W[n, :] + bias[n] for b < B <= 8.  HBM-bound on W
// (each fp32 weight row read once, 16-byte loads); one warp per output column n, all B rows at once.
// fp32 weights: the conditioning (shift / scale / gate of every block) multiplies every activation, so
// bf16-rounding it would put a 1e-3 relative error on the whole network for a saving of ~50 us.
// Used for the timestep MLP and for the adaLN modulation of ALL 24 blocks + 2 heads in one launch
// (the conditioning vector is layer-invariant).
// ---------------------------------------------------------------------------------------------
constexpr int SKINNY_MAXB = 8;

__device__ __forceinline__ float silu(float v) { return v / (1.0f + __expf(-v)); }

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
      float v = warp_sum_f(acc[b]);
      if (lane == 0) {
        v += bias ? bias[n] : 0.f;
        out[(size_t)b * N + n] = act_out ? silu(v) : v;
      }
    }
  }
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

int timestep_embedding(const float* t, float* out, int B, int dim, cudaStream_t st) {
  DGS_REQUIRE(dim % 2 == 0, "timestep_embedding: odd dim");
  timestep_embedding_kernel<<<ceil_div(B * dim / 2, 128), 128, 0, st>>>(t, out, B, dim);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

// ---------------------------------------------------------------------------------------------
// posed image (rgb*2-1 | ray channels) + patchify "b v c (hh ph) (ww pw) -> (b v)(hh ww)(ph pw c)"
// one thread per (token, ph, pw): writes its 9 channels contiguously (18 B) -- output-coalesced.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) posed_patchify_kernel(const float* __restrict__ img,
                                                             const float* __restrict__ ray_o,
                                                             const float* __restrict__ ray_d,
                                                             __nv_bfloat16* __restrict__ tokens, int BV, int H, int W,
                                                             int p, int img_c, int mode) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int hh_n = H / p, ww_n = W / p;
  const long long total = (long long)BV * H * W;
  if (idx >= total) return;
  // idx enumerates (bv, hh, ww, ph, pw) in output order
  int pw = (int)(idx % p);
  long long r = idx / p;
  int ph = (int)(r % p); r /= p;
  int ww = (int)(r % ww_n); r /= ww_n;
  int hh = (int)(r % hh_n);
  int bv = (int)(r / hh_n);
  const int y = hh * p + ph, x = ww * p + pw;
  const size_t plane = (size_t)H * W, pix = (size_t)y * W + x;
  const float* ip = img + (size_t)bv * img_c * plane + pix;
  const float* op = ray_o + (size_t)bv * 3 * plane + pix;
  const float* dp = ray_d + (size_t)bv * 3 * plane + pix;
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

int posed_patchify(const float* images, const float* ray_o, const float* ray_d, __nv_bfloat16* tokens, int B, int V,
                   int H, int W, int patch, int plucker_mode, cudaStream_t st) {
  DGS_REQUIRE(H % patch == 0 && W % patch == 0, "image size %dx%d not divisible by patch %d", H, W, patch);
  const long long total = (long long)B * V * H * W;
  posed_patchify_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(images, ray_o, ray_d, tokens, B * V, H, W,
                                                                          patch, 3, plucker_mode);
  DGS_POST_LAUNCH();
  return DGS_OK;
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

int assemble_tokens(const float* tok, const float* pos_embed, float* x, int B, int G, int T, int D, cudaStream_t st) {
  const long long total = (long long)B * (G + T) * (D / 4);
  assemble_tokens_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(tok, pos_embed, x, B, G, T, D / 4);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

__global__ void tiny_linear_kernel(const __nv_bfloat16* __restrict__ h, const __nv_bfloat16* __restrict__ W,
                                   float* __restrict__ out, int rows, int N, int K) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows * N) return;
  const int r = warp / N, n = warp - r * N;
  float acc = 0.f;
  for (int k = lane; k < K; k += 32) acc += __bfloat162float(h[(size_t)r * K + k]) * __bfloat162float(W[(size_t)n * K + k]);
  acc = warp_sum_f(acc);
  if (lane == 0) out[(size_t)r * N + n] = acc;
}

int tiny_linear_bf16(const __nv_bfloat16* h, const __nv_bfloat16* W, float* out, int rows, int N, int K,
                     cudaStream_t st) {
  tiny_linear_kernel<<<ceil_div(rows * N * 32, 256), 256, 0, st>>>(h, W, out, rows, N, K);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

// ---------------------------------------------------------------------------------------------
// to_gs + pixel alignment: one thread per Gaussian.
// ---------------------------------------------------------------------------------------------
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
  float a[14];
  float xyz[3];
  if (g < G) {
    const float* s = gs_tok + ((size_t)b * G + g) * 14;
#pragma unroll
    for (int k = 0; k < 14; k++) a[k] = s[k];
    xyz[0] = a[0]; xyz[1] = a[1]; xyz[2] = a[2];
  } else {
    const long long q = g - G;  // (v, hh, ww, ph, pw) order == img_gs memory order
    const float* s = img_gs + ((size_t)b * V * H * W + q) * 14;
#pragma unroll
    for (int k = 0; k < 14; k++) a[k] = s[k];
    const int hh_n = H / p, ww_n = W / p;
    int pw = (int)(q % p);
    long long r = q / p;
    int ph = (int)(r % p); r /= p;
    int ww = (int)(r % ww_n); r /= ww_n;
    int hh = (int)(r % hh_n);
    int v = (int)(r / hh_n);
    const int y = hh * p + ph, x = ww * p + pw;
    const size_t plane = (size_t)H * W, pix = (size_t)y * W + x;
    const size_t base = ((size_t)b * V + v) * 3 * plane + pix;
    const float o0 = ray_o[base], o1 = ray_o[base + plane], o2 = ray_o[base + 2 * plane];
    const float d0 = ray_d[base], d1 = ray_d[base + plane], d2 = ray_d[base + 2 * plane];
    const float m = (a[0] + a[1] + a[2]) / 3.0f;
    const float sg = 1.0f / (1.0f + expf(-m));
    float t;
    if (scene == 1) t = sg * (far_ - near_) + near_;                  // denoiser_scene.py:263,406-410
    else if (scene == 2) t = sg;                                      // denoiser.py:381-388 with ray_pe_type == 'plk'
    else t = (2.0f * sg - 1.0f) * 1.8f + (-o0 * d0 + -o1 * d1 + -o2 * d2);  // denoiser.py:382-392
    xyz[0] = o0 + t * d0; xyz[1] = o1 + t * d1; xyz[2] = o2 + t * d2;
    if (out.img_aligned_xyz) {
      out.img_aligned_xyz[base] = xyz[0];
      out.img_aligned_xyz[base + plane] = xyz[1];
      out.img_aligned_xyz[base + 2 * plane] = xyz[2];
    }
  }
  const size_t o = (size_t)idx;
  out.xyz[3 * o] = xyz[0]; out.xyz[3 * o + 1] = xyz[1]; out.xyz[3 * o + 2] = xyz[2];
  out.features[3 * o] = a[3]; out.features[3 * o + 1] = a[4]; out.features[3 * o + 2] = a[5];
  out.scaling[3 * o] = fminf(a[6] - 2.3f, -1.2f);  // denoiser.py:118
  out.scaling[3 * o + 1] = fminf(a[7] - 2.3f, -1.2f);
  out.scaling[3 * o + 2] = fminf(a[8] - 2.3f, -1.2f);
  *reinterpret_cast<float4*>(out.rotation + 4 * o) = make_float4(a[9], a[10], a[11], a[12]);
  out.opacity[o] = a[13] - 2.0f;  // denoiser.py:119
}

int gaussians_epilogue(const float* gs_tokens, const float* img_gs, const float* ray_o, const float* ray_d, GsOut out,
                       int B, int G, int V, int H, int W, int patch, int scene_mode, float near_, float far_,
                       cudaStream_t st) {
  const long long total = (long long)B * ((long long)G + (long long)V * H * W);
  gaussians_epilogue_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(gs_tokens, img_gs, ray_o, ray_d, out, B, G,
                                                                              V, H, W, patch, scene_mode, near_, far_);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

__global__ void f32_to_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = __float2bfloat16_rn(in[i]);
}

int f32_to_bf16(const float* in, __nv_bfloat16* out, size_t n, cudaStream_t st) {
  if (n == 0) return DGS_OK;
  f32_to_bf16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(in, out, n);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

}  // namespace dgs
