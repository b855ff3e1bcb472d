// dit_kernels.h -- internal launchers of the DiT denoiser kernels (host side, C++).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <cstdint>

namespace dgs {

enum GemmEpi { EPI_BIAS_BF16 = 0, EPI_BIAS_GELU_BF16 = 1, EPI_GATE_RESID_F32 = 2, EPI_F32 = 3, EPI_DGELU_BF16 = 4,
               EPI_BIAS_RELU_BF16 = 5, EPI_BIAS_GELU_E4M3 = 6 };

struct GemmEpilogue {
  void* out = nullptr;          // bf16 or fp32 [M, ldc]
  int ldc = 0;
  const float* bias = nullptr;  // [N] or null
  const float* gate = nullptr;  // EPI_GATE_RESID_F32: gate vector of sample b at gate + b * gate_stride
  int gate_stride = 0;
  int rows_per_sample = 1;      // sample index of a row = row / rows_per_sample
  // training-mode extras (all optional):
  void* aux = nullptr;          // bf16 [M, ldc]: EPI_BIAS_GELU_BF16 -> also store the pre-activation (acc + b);
                                //                EPI_GATE_RESID_F32 -> also store the pre-gate branch output (acc + b);
                                //                EPI_DGELU_BF16     -> INPUT: the saved pre-activation u (out = acc * gelu'(u))
  const float* resid = nullptr; // EPI_GATE_RESID_F32: residual source [M, ldc] (null: in place, = out)
  int lda = 0, ldb = 0;         // row strides of A / W in elements (0 = K): lets K-padded (transposed) operands be used
};

// C = epi(A[M,K] * W[N,K]^T), bf16 operands, fp32 accumulate (gemm_sm90.cu)
int gemm_bf16(const void* A, const void* W, int M, int N, int K, int epi, const GemmEpilogue& ep, cudaStream_t st);

// C[M,N] fp32 = A^T W for A [K,M], W [K,N] bf16 row-major (MN-major wgmma operands; ep.lda/ldb = row strides, 0 = M/N)
int gemm_bf16_tn(const void* A, const void* W, int M, int N, int K, const GemmEpilogue& ep, cudaStream_t st);

// FP8 operands (gemm_sm90.cu): A e4m3 [M, K] with group scales sa [K/128][fp8_scale_stride(M)] (one per row and
// 128-column group), W e4m3 [N, K] with per-row scales sw [N].  C = epi(sw[n] * sum_kb sa[kb][m] * (A_kb W_kb^T)).
// epi: EPI_BIAS_BF16, EPI_GATE_RESID_F32 (in place only), EPI_F32, or EPI_BIAS_GELU_E4M3 (out e4m3 [M, ldc] plus its
// group scales out_scale [N/128][fp8_scale_stride(M)]).  K % 128 == 0, N % 128 == 0.
inline int fp8_scale_stride(int M) { return (M + 3) / 4 * 4; }
int gemm_fp8(const void* A, const float* sa, const void* W, const float* sw, int M, int N, int K, int epi,
             const GemmEpilogue& ep, float* out_scale, cudaStream_t st);


// softmax(Q K^T / sqrt(64)) V over qkv [B, N, 3, H, 64] (bf16) -> out [B, N, H*64] (bf16) (attention_sm90.cu)
// lse2 (optional, training): [B, H, attention_lse_stride(N)] fp32, log2-domain log-sum-exp of the scaled scores
int attention_fwd(const void* qkv, void* out, float* lse2, int B, int N, int H, cudaStream_t st);
inline int attention_lse_stride(int N) { return (N + 127) / 128 * 128; }
// FP8 inference attention (attention_sm90.cu; layouts in include/dgs_b200.h): the quantize pass qkv -> q8 / k8 [B, N, H,
// 64], vt8 [B, H, 64, Nk] (Nk = attention_lse_stride(N)) with scales sq [B, H, N], sk / sv [B, H, Nk/128]; then the
// attention forward on those operands -> out [B, N, H*64] (bf16)
int attention_quantize_e4m3(const void* qkv, uint8_t* q8, uint8_t* k8, uint8_t* vt8, float* sq, float* sk, float* sv,
                            int B, int N, int H, cudaStream_t st);
int attention_fwd_e4m3(const uint8_t* q8, const uint8_t* k8, const uint8_t* vt8, const float* sq, const float* sk,
                       const float* sv, void* out, int B, int N, int H, cudaStream_t st);
// backward (attention_bwd_sm90.cu): dqkv [B, N, 3, H, 64] (bf16) from qkv, out (= O), lse2 and dout [B, N, H*64] (bf16);
// dsum = scratch [B, H, attention_lse_stride(N)] fp32.  Fills the pad entries of lse2 (+inf) as a side effect.
int attention_bwd(const void* qkv, const void* out, const void* dout, float* lse2, float* dsum, void* dqkv, int B, int N,
                  int H, cudaStream_t st);

// ---- dit_glue.cu: forward ----------------------------------------------------------------------
// LayerNorm [* w] + adaLN modulate: output row r (0..B*rows_out) normalises x row  b*rows_in + row_off + (r % rows_out),
// b = r / rows_out, to y = LN(x; eps) [* w] and stores  y * (1 + scale[b,:]) + shift[b,:]  as
enum LnOut {
  LN_BF16,        // bf16 [B*rows_out, D]
  LN_SPLIT_BF16,  // bf16 [B*rows_out, 3*D] = [hi | lo | hi] with value = hi + lo (split-bf16 operand)
  LN_E4M3,        // e4m3 [B*rows_out, D] with one power-of-two scale per row and 128-column group,
                  // out_scale [D/128][fp8_scale_stride(B*rows_out)]; no LN weight (ln_weight ignored)
  LN_F32,         // fp32, out = y (no modulate: shift / scale unused); in place (out == x); needs ln_weight
};
int ln_forward(LnOut kind, const float* x, const float* ln_weight, const float* shift, const float* scale,
               int mod_stride, void* out, float* out_scale, int B, int rows_in, int row_off, int rows_out, int D,
               float eps, cudaStream_t st);
// q [rows, cols] e4m3 = x / scale[r] with one power-of-two scale per row (the FP8 weight format)
int quantize_rows_e4m3(const float* x, int rows, int cols, uint8_t* q, float* scale, cudaStream_t st);
// out[b, n] = act_in(in[b,:]) . W[n,:] + bias[n], W fp32 [N,K]; act_in: 0 none, 1 SiLU
int skinny_linear(const float* in, const float* W, const float* bias, float* out, int B, int N, int K,
                  int act_in, int act_out_silu, cudaStream_t st);
// sinusoidal timestep embedding (denoiser.py:44-66): out [B, 256] = [cos(t f), sin(t f)]
int timestep_embedding(const float* t, float* out, int B, int dim, cudaStream_t st);
// Plücker-style posed image + patchify (denoiser.py:312-334, 210-216) -> split-bf16 tokens
// [B*V*hh*ww, 3*p*p*9] = [hi | lo | hi]
int posed_patchify(const float* images, const float* ray_o, const float* ray_d, __nv_bfloat16* tokens, int B, int V,
                   int H, int W, int patch, int plucker_mode, cudaStream_t st);
// x[b, 0:G] = pos_embed ; x[b, G:] = tok[b] ; (then the caller applies the input LayerNorm)
int assemble_tokens(const float* tok, const float* pos_embed, float* x, int B, int G, int T, int D, cudaStream_t st);
// small-M linear for the 2 free Gaussian tokens: out[r, n] = h[r,:] . W[n,:]   (N = C head channels)
int tiny_linear_bf16(const __nv_bfloat16* h, const __nv_bfloat16* W, float* out, int rows, int N, int K,
                     cudaStream_t st);
// to_gs + pixel alignment (denoiser.py:103-120, 362-413): raw head outputs -> renderer tensors
struct GsOut { float* xyz; float* features; float* scaling; float* rotation; float* opacity; float* img_aligned_xyz; };
// C = 11 + 3 (sh_degree+1)^2 raw channels per Gaussian, sh_degree 0..3; features out [B, P, (sh_degree+1)^2, 3]
int gaussians_epilogue(const float* gs_tokens /*[B,G,C]*/, const float* img_gs /*[B*V*hh*ww, p*p*C]*/,
                       const float* ray_o, const float* ray_d, GsOut out, int B, int G, int V, int H, int W, int patch,
                       int sh_degree, int scene_mode, float near_, float far_, cudaStream_t st);

// ---- dit_glue.cu: backward ---------------------------------------------------------------------
// out[c, m] = bf16(in[row(m), c]); m = b*rows_out + j -> input row b*rows_in + row_off + j; out [C, round_up(M,64)]
// TI: float or __nv_bfloat16
template <typename TI>
int transpose_to_bf16(const TI* in, int ldi, int B, int rows_in, int row_off, int rows_out, int C, __nv_bfloat16* out,
                      float* colsum, cudaStream_t st);
int gate_bwd(const float* dx, const __nv_bfloat16* y, const float* gate, int gate_stride, int rows_per_sample, int M,
             int C, __nv_bfloat16* dy, __nv_bfloat16* dyT, float* dgate, float* dbias, cudaStream_t st);
// backward of ln_forward (TG, the type of dh: float or __nv_bfloat16)
template <typename TG>
int ln_modulate_bwd(const float* x, const TG* dh, const float* lnw, const float* scale, int mod_stride, int B,
                    int rows_in, int row_off, int rows_out, int D, float eps, float* dx, int accumulate, float* dshift,
                    float* dscale, float* dlnw, float* stats /* scratch [B*rows_out*2] */, cudaStream_t st);
// Where the weight/bias gradient rows of a (stacked) skinny linear go: n_seg regular segments of seg_rows rows each
// (segment i at dW0 + i*seg_stride floats, its bias gradient at db0 + i*seg_stride), then two tail segments.
struct SkinnySegs {
  int seg_rows = 0, n_seg = 0;
  long long seg_stride = 0;
  float* dW0 = nullptr; float* db0 = nullptr;
  int tail_rows[2] = {0, 0};
  float* tail_dW[2] = {nullptr, nullptr}; float* tail_db[2] = {nullptr, nullptr};
};
int colsum_bf16(const __nv_bfloat16* in, int M, int C, float* colsum, cudaStream_t st);
// da (optional) += dout W, summed in a fixed order through `part`, a scratch of skinny_linear_bwd_part_floats(B, N, K)
int skinny_linear_bwd_segs(const float* in, const float* W, const float* dout, int ldo, int B, int N, int K, int act_in,
                           const SkinnySegs& segs, float* da, float* part, cudaStream_t st);
size_t skinny_linear_bwd_part_floats(int B, int N, int K);
// dout [B, ldo] (row stride ldo >= N): rows n of this linear are columns [0, N) of dout
int skinny_linear_bwd(const float* in, const float* W, const float* dout, int ldo, int B, int N, int K, int act_in,
                      float* dW, float* dbias, float* da, float* part, cudaStream_t st);
int silu_bwd_inplace(float* d, const float* pre, int n, cudaStream_t st);
int gaussians_epilogue_bwd(const float* gs_tok, const float* img_gs, const float* ray_d, const float* dxyz,
                           const float* dfeatures, const float* dscaling, const float* drotation, const float* dopacity,
                           const float* d_img_xyz /* [B,V,3,H,W] or NULL */, float* d_gs_tok, __nv_bfloat16* d_img_gs,
                           int B, int G, int V, int H, int W, int patch, int sh_degree, int scene_mode, float near_,
                           float far_, cudaStream_t st);
int tiny_linear_bwd(const float* dy, const float* W, const __nv_bfloat16* h3, __nv_bfloat16* dh, float* dW, int rows,
                    int N, int K, cudaStream_t st);
int pos_embed_bwd(const float* dx, float* dpos, int B, int G, int N, int D, cudaStream_t st);
int adamw_step(float* p, const float* g, float* m, float* v, size_t n, float lr, float b1, float b2, float eps, float wd,
               int step, float grad_scale, const float* grad_scale_dev, cudaStream_t st, float* ema = nullptr, float ema_decay = 0.f);
int cast_transpose_f32(const float* in, long long in_bstride, int batch, int M, int C, __nv_bfloat16* out_rm,
                       __nv_bfloat16* outT, cudaStream_t st);

}  // namespace dgs
