// dit_bwd_misc.cu -- the memory-bound kernels of the DiT denoiser BACKWARD (everything that is not a GEMM or the
// attention backward): operand transposes for the weight-gradient GEMMs (+ bias gradients), the gate/residual
// backward, LayerNorm+adaLN-modulate backward, the skinny conditioning linears' backward, the Gaussian heads'
// epilogue backward, and the fused AdamW update.
// The reference gets all of this from torch autograd over denoiser.py:306-416 / utils_transformer.py:246-290; the
// formulas below are the derivatives of the forward kernels in dit_misc.cu / gemm_sm90.cu.
#include "dgs_internal.h"
#include "dit_kernels.h"

namespace dgs {

namespace {

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }

constexpr int TP = 72;  // smem tile pitch in bf16 elements (144 B: 16-byte aligned rows)

// 16 consecutive elements of a row -> bf16 (two 16-byte vectors)
__device__ __forceinline__ void load16_bf16(const __nv_bfloat16* src, uint4& lo, uint4& hi) {
  lo = *reinterpret_cast<const uint4*>(src);
  hi = *reinterpret_cast<const uint4*>(src + 8);
}
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ void load16_bf16(const float* src, uint4& lo, uint4& hi) {
  const float4 a = *reinterpret_cast<const float4*>(src), b = *reinterpret_cast<const float4*>(src + 4);
  const float4 c = *reinterpret_cast<const float4*>(src + 8), d = *reinterpret_cast<const float4*>(src + 12);
  lo = make_uint4(pack_bf16x2(a.x, a.y), pack_bf16x2(a.z, a.w), pack_bf16x2(b.x, b.y), pack_bf16x2(b.z, b.w));
  hi = make_uint4(pack_bf16x2(c.x, c.y), pack_bf16x2(c.z, c.w), pack_bf16x2(d.x, d.y), pack_bf16x2(d.z, d.w));
}

// ---------------------------------------------------------------------------------------------------------------
// out[c, m] = bf16(in[row(m), c]),  m = b * rows_out + j  ->  input row  b * rows_in + row_off + j;  out is [C, Mp]
// (Mp = round_up(M, 64), pad columns zero-filled: they are the K tail of the weight-gradient GEMM).
// colsum[c] += sum_m in[row(m), c]  (bias gradient), optional.
// 64 x 64 tile per CTA: 16-byte global loads -> smem -> column reads with the lanes along c (conflict-free) ->
// 32-byte global stores.
// ---------------------------------------------------------------------------------------------------------------
template <typename TI>
__global__ void __launch_bounds__(256) transpose_kernel(const TI* __restrict__ in, int ldi, int rows_in, int row_off,
                                                        int rows_out, int M, int Mp, __nv_bfloat16* __restrict__ out,
                                                        float* __restrict__ colsum, __nv_bfloat16* __restrict__ out_rm,
                                                        int C, size_t in_bstride, size_t out_bstride, size_t rm_bstride) {
  __shared__ __align__(16) __nv_bfloat16 tile[64 * TP];
  __shared__ float red[4 * 64];
  const int m0 = blockIdx.x * 64, c0 = blockIdx.y * 64, t = threadIdx.x;
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");  // PDL: launched via launch_pdl
  asm volatile("griddepcontrol.wait;" ::: "memory");
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
  const int c = t & 63, mq = t >> 6, mc = mq * 16;
  __align__(16) __nv_bfloat16 o[16];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 16; i++) {
    o[i] = tile[(mc + i) * TP + c];
    s += __bfloat162float(o[i]);
  }
  __nv_bfloat16* dst = out + (size_t)(c0 + c) * Mp + m0 + mc;
  *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(o);
  *reinterpret_cast<uint4*>(dst + 8) = *reinterpret_cast<const uint4*>(o + 8);
  if (colsum) {
    red[mq * 64 + c] = s;
    __syncthreads();
    if (t < 64) atomicAdd(colsum + c0 + t, red[t] + red[64 + t] + red[128 + t] + red[192 + t]);
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
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");  // PDL: launched via launch_pdl
  asm volatile("griddepcontrol.wait;" ::: "memory");
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
        pk[2 * q] = pack_bf16x2(d4.x * g4.x, d4.y * g4.y);
        pk[2 * q + 1] = pack_bf16x2(d4.z * g4.z, d4.w * g4.w);
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
  const int c = t & 63, mq = t >> 6, mc = mq * 16;
  __align__(16) __nv_bfloat16 o[16];
  const int b_first = m0 / rows_per_sample;
  const int split = (b_first + 1) * rows_per_sample - m0;  // tile rows >= split belong to sample b_first + 1
  float s = 0.f, g0 = 0.f, g1 = 0.f;
#pragma unroll
  for (int i = 0; i < 16; i++) {
    o[i] = tile[(mc + i) * TP + c];
    s += __bfloat162float(o[i]);
    const float p = prod[(mc + i) * 65 + c];
    if (mc + i < split) g0 += p; else g1 += p;
  }
  if (dyT) {  // transposed copy (only the K-major weight-gradient path wants it)
    __nv_bfloat16* dst = dyT + (size_t)(c0 + c) * Mp + m0 + mc;
    *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(o);
    *reinterpret_cast<uint4*>(dst + 8) = *reinterpret_cast<const uint4*>(o + 8);
  }
  red[mq * 64 + c] = s;
  red[256 + mq * 64 + c] = g0;
  red[512 + mq * 64 + c] = g1;
  __syncthreads();
  if (t < 64) {
    const float ss = red[t] + red[64 + t] + red[128 + t] + red[192 + t];
    const float s0 = red[256 + t] + red[320 + t] + red[384 + t] + red[448 + t];
    const float s1 = red[512 + t] + red[576 + t] + red[640 + t] + red[704 + t];
    if (dbias) atomicAdd(dbias + c0 + t, ss);
    atomicAdd(dgate + (size_t)b_first * gate_stride + c0 + t, s0);
    if (split < 64 && m0 + split < M) atomicAdd(dgate + (size_t)(b_first + 1) * gate_stride + c0 + t, s1);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Backward of  h = (LN(x; eps) [* w]) * (1 + scale[b]) + shift[b]   (ln_modulate_kernel / ln_weight_kernel), two kernels:
//  rows:  one warp per row:  dx (+)= rstd (dxh - mean(dxh) - xhat mean(dxh xhat)),  dxh = g (1+scale) w;  keeps (mean, rstd)
//  cols:  64-column x 128-row tiles:  dshift[b] += sum g ; dscale[b] += sum g xhat w ; dw += sum g (1+scale) xhat
// (the fused single-kernel version needed 96 accumulator registers per lane -> 255 registers, 8 warps per SM)
// ---------------------------------------------------------------------------------------------------------------
template <typename TG>
__device__ __forceinline__ void load4_f32(const TG* p, float* o);
template <>
__device__ __forceinline__ void load4_f32<float>(const float* p, float* o) {
  const float4 v = *reinterpret_cast<const float4*>(p);
  o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
}
template <>
__device__ __forceinline__ void load4_f32<__nv_bfloat16>(const __nv_bfloat16* p, float* o) {
  const uint2 v = *reinterpret_cast<const uint2*>(p);
  const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v.x));
  const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v.y));
  o[0] = a.x; o[1] = a.y; o[2] = b.x; o[3] = b.y;
}

template <typename TG>
__global__ void __launch_bounds__(256) ln_bwd_rows_kernel(const float* __restrict__ x, const TG* __restrict__ dh,
                                                          const float* __restrict__ lnw, const float* __restrict__ scale,
                                                          int mod_stride, int rows_in, int row_off, int rows_out, float eps,
                                                          float* __restrict__ dx, int accumulate,
                                                          float2* __restrict__ stats) {
  constexpr int D = 1024, PER = 32;
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");  // PDL: launched via launch_pdl
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= rows_out) return;
  const size_t xrow = ((size_t)b * rows_in + row_off + r) * D;
  const TG* gr = dh + ((size_t)b * rows_out + r) * D;
  float v[PER], g[PER];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < PER / 4; i++) {
    const int c = (i * 32 + lane) * 4;
    const float4 t4 = *reinterpret_cast<const float4*>(x + xrow + c);
    v[4 * i] = t4.x; v[4 * i + 1] = t4.y; v[4 * i + 2] = t4.z; v[4 * i + 3] = t4.w;
    s += t4.x + t4.y + t4.z + t4.w;
    load4_f32<TG>(gr + c, g + 4 * i);
  }
  const float mean = wsum(s) * (1.0f / D);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < PER; i++) { v[i] -= mean; q += v[i] * v[i]; }
  const float rstd = rsqrtf(wsum(q) * (1.0f / D) + eps);
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
  m1 = wsum(m1) * (1.0f / D);
  m2 = wsum(m2) * (1.0f / D);
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
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");  // PDL: launched via launch_pdl
  asm volatile("griddepcontrol.wait;" ::: "memory");
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
    const float sg = red[t] + red[64 + t] + red[128 + t] + red[192 + t];
    const float sgx = red[256 + t] + red[320 + t] + red[384 + t] + red[448 + t];
    if (dshift) {
      atomicAdd(dshift + (size_t)b * mod_stride + c, sg);
      atomicAdd(dscale + (size_t)b * mod_stride + c, sgx * w);  // sum g * y, y = xhat * w
    }
    if (dlnw) atomicAdd(dlnw + c, sgx * sc1);                     // sum g (1 + scale) xhat
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
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");  // PDL: launched via launch_pdl
  asm volatile("griddepcontrol.wait;" ::: "memory");
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

// ---------------------------------------------------------------------------------------------------------------
// Backward of the skinny linear  out[b, n] = a[b, :] . W[n, :] + bias[n],  a = act_in(in)  (skinny_linear_kernel):
//   dW[n, k] = sum_b dout[b, n] a[b, k]     dbias[n] = sum_b dout[b, n]     da[b, k] += sum_n dout[b, n] W[n, k]
// One CTA per SKB_ROWS output rows n; a thread owns 4 consecutive k.  W is read once, dW written once.  Each CTA writes
// its partial da to part[cta] and skinny_da_reduce_kernel adds the partials into da in CTA order, so da does not depend
// on the order in which the CTAs finish (fp32 atomics did: run-to-run noise in every gradient behind da).
// ---------------------------------------------------------------------------------------------------------------
constexpr int SKB_MAXB = 8, SKB_ROWS = 128;
__device__ __forceinline__ float silu_f(float v) { return v / (1.0f + __expf(-v)); }

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
    s_a[t] = act_in ? silu_f(v) : v;
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
    float acc[SKB_MAXB][4];
    float a[SKB_MAXB][4];
#pragma unroll
    for (int b = 0; b < SKB_MAXB; b++) {
#pragma unroll
      for (int e = 0; e < 4; e++) { acc[b][e] = 0.f; a[b][e] = b < B ? s_a[b * K + k + e] : 0.f; }
    }
    for (int r = 0; r < nrows; r++) {
      const float4 w4 = __ldg(reinterpret_cast<const float4*>(W + (size_t)(n0 + r) * K + k));
      float4 g4 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int b = 0; b < SKB_MAXB; b++) {
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
      for (int b = 0; b < SKB_MAXB; b++) {
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

// ---------------------------------------------------------------------------------------------------------------
// Backward of gaussians_epilogue_kernel (to_gs + pixel alignment, denoiser.py:103-120, 362-413): gradients w.r.t. the
// renderer-ready tensors -> gradients of the raw 14-channel head outputs (free tokens fp32, image tokens bf16).
// ---------------------------------------------------------------------------------------------------------------
struct GsGrad { const float* xyz; const float* features; const float* scaling; const float* rotation; const float* opacity; };

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
  float da[14];
  const float* src = (g < G) ? gs_tok + ((size_t)b * G + g) * 14 : img_gs + ((size_t)b * V * H * W + (g - G)) * 14;
  const float gx = d.xyz[3 * o], gy = d.xyz[3 * o + 1], gz = d.xyz[3 * o + 2];
  if (g < G) {
    da[0] = gx; da[1] = gy; da[2] = gz;
  } else {
    const long long q = g - G;
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
    const float d0 = ray_d[base], d1 = ray_d[base + plane], d2 = ray_d[base + 2 * plane];
    const float m = (src[0] + src[1] + src[2]) / 3.0f;
    const float sg = 1.0f / (1.0f + expf(-m));
    const float dt = gx * d0 + gy * d1 + gz * d2;  // xyz = o + t d
    const float dtdm = (scene == 1 ? (far_ - near_) : scene == 2 ? 1.0f : 3.6f) * sg * (1.0f - sg);
    da[0] = da[1] = da[2] = dt * dtdm * (1.0f / 3.0f);
  }
  da[3] = d.features[3 * o]; da[4] = d.features[3 * o + 1]; da[5] = d.features[3 * o + 2];
#pragma unroll
  for (int k = 0; k < 3; k++) da[6 + k] = (src[6 + k] - 2.3f <= -1.2f) ? d.scaling[3 * o + k] : 0.f;  // clamp(max=-1.2)
  const float4 dr = *reinterpret_cast<const float4*>(d.rotation + 4 * o);
  da[9] = dr.x; da[10] = dr.y; da[11] = dr.z; da[12] = dr.w;
  da[13] = d.opacity[o];
  if (g < G) {
    float* dst = d_gs_tok + ((size_t)b * G + g) * 14;
#pragma unroll
    for (int k = 0; k < 14; k++) dst[k] = da[k];
  } else {
    __nv_bfloat16* dst = d_img_gs + ((size_t)b * V * H * W + (g - G)) * 14;
#pragma unroll
    for (int k = 0; k < 14; k += 2) {
      __nv_bfloat162 pk = __floats2bfloat162_rn(da[k], da[k + 1]);
      *reinterpret_cast<__nv_bfloat162*>(dst + k) = pk;
    }
  }
}

// Backward of the free-token head linear (rows = B*G, N = 14): dh[r, k] = sum_n dy[r, n] W[n, k] (bf16 out),
// dW[n, k] = sum_r dy[r, n] h[r, k]  with h = hi + lo of the split-bf16 operand [rows, 3K].
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

// dpos[g, :] = sum_b dx[b, g, :]   (the learned Gaussian tokens sit at rows 0..G of every sample)
__global__ void pos_embed_bwd_kernel(const float* __restrict__ dx, float* __restrict__ dpos, int B, int G, int N, int D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G * D) return;
  const int g = i / D, c = i - g * D;
  float s = 0.f;
  for (int b = 0; b < B; b++) s += dx[((size_t)b * N + g) * D + c];
  dpos[i] = s;
}

// AdamW (torch.optim.AdamW semantics: decoupled weight decay, bias-corrected moments), fp32 master weights
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

// ---------------------------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------------------------
int transpose_to_bf16(const void* in, int in_is_f32, int ldi, int B, int rows_in, int row_off, int rows_out, int C,
                      __nv_bfloat16* out, float* colsum, cudaStream_t st) {
  DGS_REQUIRE(C % 64 == 0 && ldi % 8 == 0, "transpose: need C %% 64 == 0 (C=%d ldi=%d)", C, ldi);
  const int M = B * rows_out, Mp = (M + 63) / 64 * 64;
  dim3 grid(Mp / 64, C / 64);
  if (in_is_f32)
    DGS_CUDA_OK(launch_pdl(transpose_kernel<float>, grid, dim3(256), 0, st, (const float*)in, ldi, rows_in, row_off, rows_out,
                           M, Mp, out, colsum, (__nv_bfloat16*)nullptr, C, (size_t)0, (size_t)0, (size_t)0));
  else
    DGS_CUDA_OK(launch_pdl(transpose_kernel<__nv_bfloat16>, grid, dim3(256), 0, st, (const __nv_bfloat16*)in, ldi, rows_in,
                           row_off, rows_out, M, Mp, out, colsum, (__nv_bfloat16*)nullptr, C, (size_t)0, (size_t)0, (size_t)0));
  DGS_POST_LAUNCH();
  return DGS_OK;
}

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

int ln_modulate_bwd(const float* x, const void* dh, int dh_is_f32, const float* lnw, const float* scale, int mod_stride,
                    int B, int rows_in, int row_off, int rows_out, int D, float eps, float* dx, int accumulate,
                    float* dshift, float* dscale, float* dlnw, float* stats /* scratch: 2 * B * rows_out floats */,
                    cudaStream_t st) {
  DGS_REQUIRE(D == 1024, "ln_modulate_bwd: width %d not supported (1024 only)", D);
  DGS_REQUIRE((scale != nullptr) == (dshift != nullptr && dscale != nullptr), "ln_modulate_bwd: scale/dshift/dscale mismatch");
  DGS_REQUIRE((lnw != nullptr) == (dlnw != nullptr), "ln_modulate_bwd: lnw/dlnw mismatch");
  DGS_REQUIRE(stats != nullptr, "ln_modulate_bwd: stats scratch is NULL");
  float2* s2 = reinterpret_cast<float2*>(stats);
  const dim3 grid_r((rows_out + 7) / 8, B), grid_c(D / 64, (rows_out + 127) / 128, B);
  const bool cols = dshift != nullptr || dlnw != nullptr;
  if (dh_is_f32) {
    DGS_CUDA_OK(launch_pdl(ln_bwd_rows_kernel<float>, grid_r, dim3(256), 0, st, x, (const float*)dh, lnw, scale, mod_stride,
                           rows_in, row_off, rows_out, eps, dx, accumulate, s2));
    DGS_POST_LAUNCH();
    if (cols) {
      DGS_CUDA_OK(launch_pdl(ln_bwd_cols_kernel<float>, grid_c, dim3(256), 0, st, x, (const float*)dh, lnw, scale, mod_stride,
                             rows_in, row_off, rows_out, (const float2*)s2, dshift, dscale, dlnw));
      DGS_POST_LAUNCH();
    }
  } else {
    DGS_CUDA_OK(launch_pdl(ln_bwd_rows_kernel<__nv_bfloat16>, grid_r, dim3(256), 0, st, x, (const __nv_bfloat16*)dh, lnw, scale,
                           mod_stride, rows_in, row_off, rows_out, eps, dx, accumulate, s2));
    DGS_POST_LAUNCH();
    if (cols) {
      DGS_CUDA_OK(launch_pdl(ln_bwd_cols_kernel<__nv_bfloat16>, grid_c, dim3(256), 0, st, x, (const __nv_bfloat16*)dh, lnw, scale,
                             mod_stride, rows_in, row_off, rows_out, (const float2*)s2, dshift, dscale, dlnw));
      DGS_POST_LAUNCH();
    }
  }
  return DGS_OK;
}

int skinny_linear_bwd_segs(const float* in, const float* W, const float* dout, int ldo, int B, int N, int K, int act_in,
                           const SkinnySegs& segs, float* da, float* part, cudaStream_t st) {
  DGS_REQUIRE(B >= 1 && B <= SKB_MAXB && K % 4 == 0, "skinny_linear_bwd: bad shape B=%d K=%d (B <= 8)", B, K);
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

int gaussians_epilogue_bwd(const float* gs_tok, const float* img_gs, const float* ray_d, const float* dxyz,
                           const float* dfeatures, const float* dscaling, const float* drotation, const float* dopacity,
                           float* d_gs_tok, __nv_bfloat16* d_img_gs, int B, int G, int V, int H, int W, int patch,
                           int scene_mode, float near_, float far_, cudaStream_t st) {
  GsGrad d{dxyz, dfeatures, dscaling, drotation, dopacity};
  const long long total = (long long)B * ((long long)G + (long long)V * H * W);
  gaussians_epilogue_bwd_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(gs_tok, img_gs, ray_d, d, d_gs_tok,
                                                                                  d_img_gs, B, G, V, H, W, patch,
                                                                                  scene_mode, near_, far_);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

int tiny_linear_bwd(const float* dy, const float* W, const __nv_bfloat16* h3, __nv_bfloat16* dh, float* dW, int rows,
                    int N, int K, cudaStream_t st) {
  tiny_linear_bwd_kernel<<<ceil_div(K, 128), 128, 0, st>>>(dy, W, h3, dh, dW, rows, N, K);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

int pos_embed_bwd(const float* dx, float* dpos, int B, int G, int N, int D, cudaStream_t st) {
  if (G == 0) return DGS_OK;
  pos_embed_bwd_kernel<<<ceil_div(G * D, 256), 256, 0, st>>>(dx, dpos, B, G, N, D);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

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
