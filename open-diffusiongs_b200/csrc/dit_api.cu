// dit_api.cu -- C ABI of the DiT denoiser forward (include/dgs_b200.h, section B2): orchestrates the
// wgmma GEMMs, the wgmma attention and the glue kernels into DGSDenoiser.image_to_gaussians
// (diffusionGS/models/denoiser/denoiser.py:306-416).
#include "dgs_internal.h"
#include "dit_kernels.h"

using namespace dgs;

namespace {

struct DitWorkspace {
  __nv_bfloat16* tokens;  // [B*T, 3*p*p*9] split-bf16
  float* tok;             // [B*T, w]
  float* x;               // [B*N, w]   fp32 residual stream
  __nv_bfloat16* h;       // [B*N, w]
  __nv_bfloat16* qkv;     // [B*N, 3w]
  __nv_bfloat16* attn;    // [B*N, w]
  __nv_bfloat16* u;       // [B*N, 4w]
  float* temb0;           // [B, 256]
  float* temb1;           // [B, w]
  float* c;               // [B, w]
  float* mod;             // [B, L*6w + 4w]
  __nv_bfloat16* hg;      // [B*G, 3w] split-bf16
  float* gs_tok;          // [B*G, 14]
  float* img_gs;          // [B*T, p*p*14]
  size_t bytes;
  DitWorkspace(void* base, const dgs_dit_weights* w, int B, int V, int H, int W) {
    const size_t T = (size_t)V * (H / w->patch) * (W / w->patch), N = T + w->n_gaussians, D = w->width;
    Carver c_(base);
    tokens = c_.take<__nv_bfloat16>((size_t)B * T * 3 * w->patch * w->patch * 9);
    tok = c_.take<float>((size_t)B * T * D);
    x = c_.take<float>((size_t)B * N * D);
    h = c_.take<__nv_bfloat16>((size_t)B * N * D);
    qkv = c_.take<__nv_bfloat16>((size_t)B * N * 3 * D);
    attn = c_.take<__nv_bfloat16>((size_t)B * N * D);
    u = c_.take<__nv_bfloat16>((size_t)B * N * w->mlp_hidden);
    temb0 = c_.take<float>((size_t)B * 256);
    temb1 = c_.take<float>((size_t)B * D);
    c = c_.take<float>((size_t)B * D);
    mod = c_.take<float>((size_t)B * ((size_t)w->layers * 6 * D + 4 * D));
    hg = c_.take<__nv_bfloat16>((size_t)B * w->n_gaussians * 3 * D);
    gs_tok = c_.take<float>((size_t)B * w->n_gaussians * 14);
    img_gs = c_.take<float>((size_t)B * T * w->patch * w->patch * 14);
    bytes = c_.bytes();
  }
};

// Everything the backward needs from the forward (training mode), plus the backward's own scratch.  Per-layer tensors
// are stacked along a leading L axis.  M = B*N rows, Mp = round_up(M, 64), Mt = B*T image-token rows.
// Recompute mode (io->train_mode == DGS_TRAIN_RECOMPUTE; the reference's torch.utils.checkpoint around every block,
// denoiser.py:348-354): only the residual stream entering each block (x_all) survives the forward; the per-layer tensors
// have ONE slot that the backward refills by re-running block l's forward right before differentiating it.
struct TrainState {
  float* x_pre;             // [M, w]      assembled tokens before the input LayerNorm
  float* x_all;             // [L+1][M, w] residual stream entering block l (x_all[L] = final)
  float* x_mid;             // [L][M, w]   after the attention branch
  __nv_bfloat16* h1;        // [L][M, w]   LN1+modulate output (A of qkv)
  __nv_bfloat16* h2;        // [L][M, w]   LN2+modulate output (A of fc1)
  __nv_bfloat16* qkv;       // [L][M, 3w]
  __nv_bfloat16* attn;      // [L][M, w]
  float* lse;               // [L][B, heads, Np]
  __nv_bfloat16* proj_out;  // [L][M, w]   attention branch output before the gate
  __nv_bfloat16* fc2_out;   // [L][M, w]   MLP branch output before the gate
  __nv_bfloat16* u_pre;     // [L][M, 4w]  fc1 + bias (pre-GELU)
  __nv_bfloat16* u;         // [L][M, 4w]  GELU output (A of fc2)
  __nv_bfloat16* hdec;      // [Mt, 3w]    decoder-head operand (split-bf16)
  // ---- backward scratch ----
  float* dx;                // [M, w]      gradient of the residual stream
  float* dx_pre;            // [M, w]
  float* dmod;              // [B, mod_stride]
  float* dsum;              // [B, heads, Np]
  float* dcond;             // [3][B, w]   dsilu(c) / dtemb1 / pre1
  float* ln_stats;          // [M, 2]      (mean, rstd) of the LayerNorm being differentiated
  float* d_gs_tok;          // [B*G, 14]
  __nv_bfloat16* dyb;       // [M, w]      gated branch gradient / generic [M, w] bf16
  __nv_bfloat16* dh;        // [M, w]
  __nv_bfloat16* big0;      // [M, 4w]     du / dqkv / d_img_gs
  __nv_bfloat16* bigT0;     // [w, Mp]     transposed token gradient (tokenizer weight gradient only)
  __nv_bfloat16* bigT1;     // [w, Mp]     transposed patches        (tokenizer weight gradient only)
  size_t bytes;
  size_t lk;  // slots of the per-layer tensors: L (store mode) or 1 (recompute mode: only x_all is kept per layer)
  TrainState(void* base, const dgs_dit_weights* w, int B, int V, int H, int W, int mode) {
    const size_t T = (size_t)V * (H / w->patch) * (W / w->patch), N = T + w->n_gaussians, D = w->width;
    const size_t Lx = w->layers, L = mode == DGS_TRAIN_RECOMPUTE ? 1 : Lx;
    lk = L;
    const size_t M = (size_t)B * N, Mp = (M + 63) / 64 * 64, U = w->mlp_hidden;
    const size_t Np = (size_t)attention_lse_stride((int)N);
    const size_t mod_stride = Lx * 6 * D + 4 * D;
    const size_t wide = U > 3 * D ? U : 3 * D;
    Carver c(base);
    x_pre = c.take<float>(M * D);
    x_all = c.take<float>((Lx + 1) * M * D);
    x_mid = c.take<float>(L * M * D);
    h1 = c.take<__nv_bfloat16>(L * M * D);
    h2 = c.take<__nv_bfloat16>(L * M * D);
    qkv = c.take<__nv_bfloat16>(L * M * 3 * D);
    attn = c.take<__nv_bfloat16>(L * M * D);
    lse = c.take<float>(L * B * w->heads * Np);
    proj_out = c.take<__nv_bfloat16>(L * M * D);
    fc2_out = c.take<__nv_bfloat16>(L * M * D);
    u_pre = c.take<__nv_bfloat16>(L * M * U);
    u = c.take<__nv_bfloat16>(L * M * U);
    hdec = c.take<__nv_bfloat16>((size_t)B * T * 3 * D);
    dx = c.take<float>(M * D);
    dx_pre = c.take<float>(M * D);
    dmod = c.take<float>((size_t)B * mod_stride);
    dsum = c.take<float>((size_t)B * w->heads * Np);
    dcond = c.take<float>((size_t)3 * B * D);
    ln_stats = c.take<float>(2 * M);
    d_gs_tok = c.take<float>((size_t)B * w->n_gaussians * 14 + 16);
    dyb = c.take<__nv_bfloat16>(M * D);
    dh = c.take<__nv_bfloat16>(M * D);
    big0 = c.take<__nv_bfloat16>(M * wide);
    bigT0 = c.take<__nv_bfloat16>(D * Mp);
    bigT1 = c.take<__nv_bfloat16>(D * Mp);
    bytes = c.bytes();
  }
};

int check_dit(const dgs_dit_weights* w, int B, int V, int H, int W) {
  DGS_REQUIRE(w != nullptr, "weights is NULL");
  DGS_REQUIRE(w->width == 1024 && w->heads * 64 == w->width, "unsupported width/heads %d/%d (1024/16 only)", w->width, w->heads);
  DGS_REQUIRE(w->layers > 0 && w->patch > 0 && w->n_gaussians >= 0 && w->mlp_hidden % 256 == 0, "bad DiT config");
  DGS_REQUIRE(B > 0 && V > 0 && H % w->patch == 0 && W % w->patch == 0, "bad input shape B=%d V=%d H=%d W=%d", B, V, H, W);
  DGS_REQUIRE((w->patch * w->patch * 14) % 32 == 0 && (w->patch * w->patch * 9) % 8 == 0, "patch %d unsupported", w->patch);
  DGS_REQUIRE(w->mlp_hidden >= 3 * w->width, "mlp_hidden must be >= 3*width (decoder head re-uses that buffer)");
  return DGS_OK;
}

#define DGS_TRY(expr)       \
  do {                      \
    int _rc = (expr);       \
    if (_rc) return _rc;    \
  } while (0)

// Buffers of ONE DiTBlock forward (utils_transformer.py:270-290).  Inference: every block re-uses the workspace and the
// residual stream is updated in place (x_in == x_mid == x_out, TMA reduce-add epilogue).  Training: x_in / x_mid / x_out
// are distinct fp32 tensors and the pre-gate branch outputs / pre-GELU values are kept for the backward.
struct BlockBufs {
  const float* x_in; float* x_mid; float* x_out;
  __nv_bfloat16 *h1, *h2, *qkv, *attn, *u;
  __nv_bfloat16 *proj_out, *fc2_out, *u_pre;  // training only (NULL: not stored)
  float* lse;                                  // training only
  bool distinct;                               // x_in / x_mid / x_out are separate buffers
};

int block_forward(const dgs_dit_weights* w, int l, const float* m, int mod_stride, int B, int N, const BlockBufs& b,
                  cudaStream_t st) {
  const int D = w->width;
  {
    ProfScope ps(st, PROF_DIT_LN);
    DGS_TRY(ln_modulate(b.x_in, nullptr, m, m + D, mod_stride, b.h1, B, N, 0, N, D, 1e-6f, 0, st));
  }
  {
    ProfScope ps(st, PROF_DIT_GEMM_QKV);
    GemmEpilogue ep;
    ep.out = b.qkv; ep.ldc = 3 * D; ep.bias = w->qkv_b + (size_t)l * 3 * D;
    DGS_TRY(gemm_bf16(b.h1, (const __nv_bfloat16*)w->qkv_w + (size_t)l * 3 * D * D, B * N, 3 * D, D, EPI_BIAS_BF16, ep, st));
  }
  {
    ProfScope ps(st, PROF_DIT_ATTN);
    DGS_TRY(attention_fwd(b.qkv, b.attn, b.lse, B, N, w->heads, st));
  }
  {
    ProfScope ps(st, PROF_DIT_GEMM_PROJ);
    GemmEpilogue ep;
    ep.out = b.x_mid; ep.ldc = D; ep.bias = w->proj_b + (size_t)l * D;
    ep.gate = m + 2 * D; ep.gate_stride = mod_stride; ep.rows_per_sample = N;
    if (b.distinct) { ep.resid = b.x_in; ep.aux = b.proj_out; }
    DGS_TRY(gemm_bf16(b.attn, (const __nv_bfloat16*)w->proj_w + (size_t)l * D * D, B * N, D, D, EPI_GATE_RESID_F32, ep, st));
  }
  {
    ProfScope ps(st, PROF_DIT_LN);
    DGS_TRY(ln_modulate(b.x_mid, nullptr, m + 3 * D, m + 4 * D, mod_stride, b.h2, B, N, 0, N, D, 1e-6f, 0, st));
  }
  {
    ProfScope ps(st, PROF_DIT_GEMM_FC1);
    GemmEpilogue ep;
    ep.out = b.u; ep.ldc = w->mlp_hidden; ep.bias = w->fc1_b + (size_t)l * w->mlp_hidden;
    ep.aux = b.u_pre;
    DGS_TRY(gemm_bf16(b.h2, (const __nv_bfloat16*)w->fc1_w + (size_t)l * w->mlp_hidden * D, B * N, w->mlp_hidden, D,
                      EPI_BIAS_GELU_BF16, ep, st));
  }
  {
    ProfScope ps(st, PROF_DIT_GEMM_FC2);
    GemmEpilogue ep;
    ep.out = b.x_out; ep.ldc = D; ep.bias = w->fc2_b + (size_t)l * D;
    ep.gate = m + 5 * D; ep.gate_stride = mod_stride; ep.rows_per_sample = N;
    if (b.distinct) { ep.resid = b.x_mid; ep.aux = b.fc2_out; }
    DGS_TRY(gemm_bf16(b.u, (const __nv_bfloat16*)w->fc2_w + (size_t)l * D * w->mlp_hidden, B * N, D, w->mlp_hidden,
                      EPI_GATE_RESID_F32, ep, st));
  }
  return DGS_OK;
}

// FP8 inference: the activation scales of the e4m3 copies of h (LN outputs, [w/128][Ms]) and u (GELU output,
// [4w/128][Ms]), carved after the bf16 workspace; the e4m3 activations themselves live in h / u.
struct Fp8Workspace {
  float* sa_h;
  float* sa_u;
  size_t bytes;
  Fp8Workspace(void* base, const dgs_dit_weights* w, int B, int V, int H, int W) {
    const size_t T = (size_t)V * (H / w->patch) * (W / w->patch), N = T + w->n_gaussians;
    const size_t Ms = (size_t)fp8_scale_stride((int)(B * N));
    Carver c(base);
    sa_h = c.take<float>((size_t)(w->width / 128) * Ms);
    sa_u = c.take<float>((size_t)(w->mlp_hidden / 128) * Ms);
    bytes = c.bytes();
  }
};

// One DiTBlock on the FP8 path (inference, residual stream x updated in place): LN -> e4m3, qkv (FP8) -> bf16,
// attention and attn.proj as in block_forward, LN -> e4m3, fc1 (FP8) + GELU -> e4m3, fc2 (FP8) gated into x.
int block_forward_fp8(const dgs_dit_weights* w, const dgs_dit_weights_fp8* w8, int l, const float* m, int mod_stride,
                      int B, int N, float* x, uint8_t* h8, float* sa_h, __nv_bfloat16* qkv, __nv_bfloat16* attn,
                      uint8_t* u8, float* sa_u, cudaStream_t st) {
  const int D = w->width, U = w->mlp_hidden, M = B * N;
  {
    ProfScope ps(st, PROF_DIT_LN);
    DGS_TRY(ln_modulate_fp8(x, m, m + D, mod_stride, h8, sa_h, B, N, D, 1e-6f, st));
  }
  {
    ProfScope ps(st, PROF_DIT_GEMM_QKV);
    GemmEpilogue ep;
    ep.out = qkv; ep.ldc = 3 * D; ep.bias = w->qkv_b + (size_t)l * 3 * D;
    DGS_TRY(gemm_fp8(h8, sa_h, (const uint8_t*)w8->qkv_w + (size_t)l * 3 * D * D, w8->qkv_s + (size_t)l * 3 * D, M, 3 * D,
                     D, EPI_BIAS_BF16, ep, nullptr, st));
  }
  {
    ProfScope ps(st, PROF_DIT_ATTN);
    DGS_TRY(attention_fwd(qkv, attn, nullptr, B, N, w->heads, st));
  }
  {
    ProfScope ps(st, PROF_DIT_GEMM_PROJ);
    GemmEpilogue ep;
    ep.out = x; ep.ldc = D; ep.bias = w->proj_b + (size_t)l * D;
    ep.gate = m + 2 * D; ep.gate_stride = mod_stride; ep.rows_per_sample = N;
    DGS_TRY(gemm_bf16(attn, (const __nv_bfloat16*)w->proj_w + (size_t)l * D * D, M, D, D, EPI_GATE_RESID_F32, ep, st));
  }
  {
    ProfScope ps(st, PROF_DIT_LN);
    DGS_TRY(ln_modulate_fp8(x, m + 3 * D, m + 4 * D, mod_stride, h8, sa_h, B, N, D, 1e-6f, st));
  }
  {
    ProfScope ps(st, PROF_DIT_GEMM_FC1);
    GemmEpilogue ep;
    ep.out = u8; ep.ldc = U; ep.bias = w->fc1_b + (size_t)l * U;
    DGS_TRY(gemm_fp8(h8, sa_h, (const uint8_t*)w8->fc1_w + (size_t)l * U * D, w8->fc1_s + (size_t)l * U, M, U, D,
                     EPI_BIAS_GELU_E4M3, ep, sa_u, st));
  }
  {
    ProfScope ps(st, PROF_DIT_GEMM_FC2);
    GemmEpilogue ep;
    ep.out = x; ep.ldc = D; ep.bias = w->fc2_b + (size_t)l * D;
    ep.gate = m + 5 * D; ep.gate_stride = mod_stride; ep.rows_per_sample = N;
    DGS_TRY(gemm_fp8(u8, sa_u, (const uint8_t*)w8->fc2_w + (size_t)l * D * U, w8->fc2_s + (size_t)l * D, M, D, U,
                     EPI_GATE_RESID_F32, ep, nullptr, st));
  }
  return DGS_OK;
}

// the training-mode buffers of block l: slice l of the stacked tensors (store mode) or the single slot (recompute mode);
// `keep_aux` = false drops the stores only the backward reads (recompute-mode forward pass)
BlockBufs train_bufs(const TrainState& ts, const dgs_dit_weights* w, int l, size_t MD, size_t MU, int B, int N, bool keep_aux) {
  const size_t s = ts.lk == 1 ? 0 : (size_t)l;
  BlockBufs b;
  b.x_in = ts.x_all + (size_t)l * MD; b.x_mid = ts.x_mid + s * MD; b.x_out = ts.x_all + (size_t)(l + 1) * MD;
  b.h1 = ts.h1 + s * MD; b.h2 = ts.h2 + s * MD; b.qkv = ts.qkv + s * 3 * MD; b.attn = ts.attn + s * MD; b.u = ts.u + s * MU;
  b.proj_out = keep_aux ? ts.proj_out + s * MD : nullptr;
  b.fc2_out = keep_aux ? ts.fc2_out + s * MD : nullptr;
  b.u_pre = keep_aux ? ts.u_pre + s * MU : nullptr;
  b.lse = ts.lse + s * B * w->heads * attention_lse_stride(N);
  b.distinct = true;
  return b;
}

// dgs_dit_forward (w8 == NULL) and dgs_dit_forward_fp8 (w8 != NULL: inference with the FP8 block GEMMs)
int dit_forward(const dgs_dit_weights* w, const dgs_dit_weights_fp8* w8, const dgs_dit_io* io, void* workspace,
                size_t workspace_bytes, cudaStream_t st) {
  DGS_REQUIRE(io != nullptr, "io is NULL");
  DGS_TRY(check_dit(w, io->B, io->V, io->H, io->W));
  DGS_REQUIRE(io->images && io->ray_o && io->ray_d && io->t, "NULL input");
  DGS_REQUIRE(io->xyz && io->features && io->scaling && io->rotation && io->opacity, "NULL output");
  const int B = io->B, V = io->V, H = io->H, W = io->W, D = w->width, L = w->layers, G = w->n_gaussians, p = w->patch;
  const int T = V * (H / p) * (W / p), N = T + G, Kin = p * p * 9, Ndec = p * p * 14;
  DitWorkspace ws(workspace, w, B, V, H, W);
  Fp8Workspace ws8(workspace ? (char*)workspace + ws.bytes : nullptr, w, B, V, H, W);
  const size_t need = ws.bytes + (w8 ? ws8.bytes : 0);
  DGS_REQUIRE(workspace && workspace_bytes >= need, "workspace too small: %zu < %zu", workspace_bytes, need);
  const int mod_stride = L * 6 * D + 4 * D;
  const bool train = io->train_state != nullptr;
  const bool recompute = train && io->train_mode == DGS_TRAIN_RECOMPUTE;
  DGS_REQUIRE(io->train_mode == DGS_TRAIN_STORE || io->train_mode == DGS_TRAIN_RECOMPUTE, "bad train_mode %d", io->train_mode);
  TrainState ts(io->train_state, w, B, V, H, W, io->train_mode);
  const size_t MD = (size_t)B * N * D, MU = (size_t)B * N * w->mlp_hidden;
  float* x0 = (train && !recompute) ? ts.x_all : ws.x;  // residual stream entering block 0

  // ---- input stage: posed image -> tokens -> tokenizer GEMM -> [pos tokens | image tokens] -> LayerNorm(weight) ----
  if (g_prof_on) prof_begin(st, PROF_DIT_INPUT);
  DGS_TRY(posed_patchify(io->images, io->ray_o, io->ray_d, ws.tokens, B, V, H, W, p, io->plucker_mode, st));
  {
    GemmEpilogue ep;
    ep.out = ws.tok; ep.ldc = D;
    DGS_TRY(gemm_bf16(ws.tokens, w->tokenizer_w, B * T, D, 3 * Kin, EPI_F32, ep, st));  // split-bf16: K = 3*576
  }
  DGS_TRY(assemble_tokens(ws.tok, w->pos_embed, x0, B, G, T, D, st));
  if (train) DGS_CUDA_OK(cudaMemcpyAsync(ts.x_pre, x0, MD * sizeof(float), cudaMemcpyDeviceToDevice, st));
  DGS_TRY(ln_weight_inplace(x0, w->in_ln_w, B * N, D, 1e-5f, st));  // nn.LayerNorm default eps (denoiser.py:234-236)
  if (g_prof_on) { prof_end(st, PROF_DIT_INPUT); prof_begin(st, PROF_DIT_COND); }

  // ---- conditioning: timestep MLP, then the adaLN modulation of ALL blocks and both heads in one launch ----
  DGS_TRY(timestep_embedding(io->t, ws.temb0, B, 256, st));
  DGS_TRY(skinny_linear(ws.temb0, w->t0_w, w->t0_b, ws.temb1, B, D, 256, 0, 1, st));
  DGS_TRY(skinny_linear(ws.temb1, w->t2_w, w->t2_b, ws.c, B, D, D, 0, 0, st));
  DGS_TRY(skinny_linear(ws.c, w->adaln_w, w->adaln_b, ws.mod, B, mod_stride, D, 1, 0, st));
  if (g_prof_on) prof_end(st, PROF_DIT_COND);

  // ---- L x DiTBlock (utils_transformer.py:270-290) ----
  for (int l = 0; l < L; l++) {
    const float* m = ws.mod + (size_t)l * 6 * D;  // shift_msa | scale_msa | gate_msa | shift_mlp | scale_mlp | gate_mlp
    BlockBufs bb;
    if (train && !recompute) {
      bb = train_bufs(ts, w, l, MD, MU, B, N, /*keep_aux=*/true);
    } else {  // inference / recompute mode: one set of buffers, residual stream updated in place (TMA reduce-add epilogues);
              // recompute mode snapshots the stream entering every block (all the backward keeps per layer)
      if (recompute) DGS_CUDA_OK(cudaMemcpyAsync(ts.x_all + (size_t)l * MD, ws.x, MD * sizeof(float), cudaMemcpyDeviceToDevice, st));
      bb.x_in = ws.x; bb.x_mid = ws.x; bb.x_out = ws.x;
      bb.h1 = ws.h; bb.h2 = ws.h; bb.qkv = ws.qkv; bb.attn = ws.attn; bb.u = ws.u;
      bb.proj_out = bb.fc2_out = bb.u_pre = nullptr; bb.lse = nullptr; bb.distinct = false;
    }
    if (w8)
      DGS_TRY(block_forward_fp8(w, w8, l, m, mod_stride, B, N, ws.x, (uint8_t*)ws.h, ws8.sa_h, ws.qkv, ws.attn,
                                (uint8_t*)ws.u, ws8.sa_u, st));
    else
      DGS_TRY(block_forward(w, l, m, mod_stride, B, N, bb, st));
  }
  float* x_fin = (train && !recompute) ? ts.x_all + (size_t)L * MD : ws.x;
  if (recompute) DGS_CUDA_OK(cudaMemcpyAsync(ts.x_all + (size_t)L * MD, ws.x, MD * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (io->tokens_out)
    DGS_CUDA_OK(cudaMemcpyAsync(io->tokens_out, x_fin, (size_t)B * N * D * sizeof(float), cudaMemcpyDeviceToDevice, st));

  // ---- heads (denoiser.py:76-164): LN(weight) + modulate + Linear ----
  ProfScope ps_heads(st, PROF_DIT_HEADS);
  const float* mu = ws.mod + (size_t)L * 6 * D;  // upsampler: shift | scale
  const float* md = mu + 2 * D;                  // image_token_decoder: shift | scale
  if (G > 0) {
    DGS_TRY(ln_modulate(x_fin, w->ups_ln_w, mu, mu + D, mod_stride, ws.hg, B, N, 0, G, D, 1e-5f, 1, st));
    DGS_TRY(tiny_linear_bf16(ws.hg, (const __nv_bfloat16*)w->ups_w, ws.gs_tok, B * G, 14, 3 * D, st));
  }
  // the decoder head runs split-bf16 (K = 3*width) so the Gaussian parameters are fp32-accurate functions of the
  // residual stream; its A operand re-uses the (now free) MLP hidden buffer
  __nv_bfloat16* hdec = train ? ts.hdec : ws.u;
  DGS_TRY(ln_modulate(x_fin, w->dec_ln_w, md, md + D, mod_stride, hdec, B, N, G, T, D, 1e-5f, 1, st));
  {
    GemmEpilogue ep;
    ep.out = ws.img_gs; ep.ldc = Ndec;
    DGS_TRY(gemm_bf16(hdec, w->dec_w, B * T, Ndec, 3 * D, EPI_F32, ep, st));
  }
  GsOut go;
  go.xyz = io->xyz; go.features = io->features; go.scaling = io->scaling; go.rotation = io->rotation;
  go.opacity = io->opacity; go.img_aligned_xyz = io->img_aligned_xyz;
  DGS_TRY(gaussians_epilogue(ws.gs_tok, ws.img_gs, io->ray_o, io->ray_d, go, B, G, V, H, W, p, io->scene_depth,
                             io->range_near, io->range_far, st));
  return DGS_OK;
}

}  // namespace

extern "C" {

size_t dgs_dit_workspace_bytes(const dgs_dit_weights* w, int B, int V, int H, int W) {
  if (check_dit(w, B, V, H, W)) return 0;
  return DitWorkspace(nullptr, w, B, V, H, W).bytes;
}

int dgs_dit_forward(const dgs_dit_weights* w, const dgs_dit_io* io, void* workspace, size_t workspace_bytes,
                    void* stream) {
  return dit_forward(w, nullptr, io, workspace, workspace_bytes, (cudaStream_t)stream);
}

size_t dgs_dit_workspace_bytes_fp8(const dgs_dit_weights* w, int B, int V, int H, int W) {
  if (check_dit(w, B, V, H, W)) return 0;
  return DitWorkspace(nullptr, w, B, V, H, W).bytes + Fp8Workspace(nullptr, w, B, V, H, W).bytes;
}

int dgs_dit_forward_fp8(const dgs_dit_weights* w, const dgs_dit_weights_fp8* w8, const dgs_dit_io* io, void* workspace,
                        size_t workspace_bytes, void* stream) {
  DGS_REQUIRE(w8 && w8->qkv_w && w8->qkv_s && w8->fc1_w && w8->fc1_s && w8->fc2_w && w8->fc2_s, "NULL FP8 weight or scale");
  DGS_REQUIRE(io == nullptr || io->train_state == nullptr,
              "dgs_dit_forward_fp8 is inference only (io->train_state must be NULL; training runs bf16)");
  return dit_forward(w, w8, io, workspace, workspace_bytes, (cudaStream_t)stream);
}

int dgs_quantize_rows_e4m3(const float* x, int rows, int cols, void* q, float* scale, void* stream) {
  DGS_REQUIRE(x && q && scale, "NULL pointer");
  return quantize_rows_e4m3(x, rows, cols, (uint8_t*)q, scale, (cudaStream_t)stream);
}

int dgs_ln_modulate_fp8(const float* x, const float* shift, const float* scale, int mod_stride, void* q, float* q_scale,
                        int B, int rows, int width, float eps, void* stream) {
  DGS_REQUIRE(x && shift && scale && q && q_scale, "NULL pointer");
  return ln_modulate_fp8(x, shift, scale, mod_stride, (uint8_t*)q, q_scale, B, rows, width, eps, (cudaStream_t)stream);
}

int dgs_gemm_fp8(const void* A, const float* sa, const void* W, const float* sw, const float* bias, const float* gate,
                 void* out, float* out_scale, int M, int N, int K, int epi, int ldc, int gate_stride,
                 int rows_per_sample, void* stream) {
  DGS_REQUIRE(epi != EPI_GATE_RESID_F32 || (gate && rows_per_sample > 0), "gate epilogue needs gate and rows_per_sample");
  GemmEpilogue ep;
  ep.out = out; ep.ldc = ldc; ep.bias = bias; ep.gate = gate; ep.gate_stride = gate_stride;
  ep.rows_per_sample = rows_per_sample > 0 ? rows_per_sample : 1;
  return gemm_fp8(A, sa, W, sw, M, N, K, epi, ep, out_scale, (cudaStream_t)stream);
}

size_t dgs_dit_train_state_bytes(const dgs_dit_weights* w, int B, int V, int H, int W) {
  return dgs_dit_train_state_bytes_ex(w, B, V, H, W, DGS_TRAIN_STORE);
}

size_t dgs_dit_train_state_bytes_ex(const dgs_dit_weights* w, int B, int V, int H, int W, int train_mode) {
  if (check_dit(w, B, V, H, W)) return 0;
  if (train_mode != DGS_TRAIN_STORE && train_mode != DGS_TRAIN_RECOMPUTE) {
    set_error("bad train_mode %d", train_mode);
    return 0;
  }
  return TrainState(nullptr, w, B, V, H, W, train_mode).bytes;
}

int dgs_dit_export_state(const dgs_dit_weights* w, int B, int V, int H, int W, int train_mode, const void* train_state,
                         int layer, float* x, float* x_mid, void* h1, void* qkv, void* attn, float* lse, void* proj_out,
                         void* h2, void* u_pre, void* u, void* fc2_out, void* stream) {
  DGS_TRY(check_dit(w, B, V, H, W));
  DGS_REQUIRE(train_mode == DGS_TRAIN_STORE || train_mode == DGS_TRAIN_RECOMPUTE, "bad train_mode %d", train_mode);
  DGS_REQUIRE(train_state != nullptr, "train_state is NULL");
  const int L = w->layers;
  DGS_REQUIRE(layer >= 0 && layer <= L, "layer %d out of range [0, %d]", layer, L);
  const bool per_layer = x_mid || h1 || qkv || attn || lse || proj_out || h2 || u_pre || u || fc2_out;
  DGS_REQUIRE(!per_layer || train_mode == DGS_TRAIN_STORE,
              "per-layer tensors are kept only in DGS_TRAIN_STORE mode (recompute mode keeps the residual stream alone)");
  DGS_REQUIRE(!per_layer || layer < L, "per-layer tensors exist for layers [0, %d), not %d", L, layer);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t T = (size_t)V * (H / w->patch) * (W / w->patch), N = T + w->n_gaussians, D = w->width;
  const size_t MD = (size_t)B * N * D, MU = (size_t)B * N * w->mlp_hidden;
  const size_t LS = (size_t)B * w->heads * attention_lse_stride((int)N);
  TrainState ts(const_cast<void*>(train_state), w, B, V, H, W, train_mode);
  const size_t l = (size_t)layer;
  auto copy = [&](void* dst, const void* src, size_t bytes) -> int {
    if (dst) DGS_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st));
    return DGS_OK;
  };
  const size_t f4 = sizeof(float), b2 = sizeof(__nv_bfloat16);
  DGS_TRY(copy(x, ts.x_all + l * MD, MD * f4));
  if (!per_layer) return DGS_OK;
  DGS_TRY(copy(x_mid, ts.x_mid + l * MD, MD * f4));
  DGS_TRY(copy(h1, ts.h1 + l * MD, MD * b2));
  DGS_TRY(copy(qkv, ts.qkv + l * 3 * MD, 3 * MD * b2));
  DGS_TRY(copy(attn, ts.attn + l * MD, MD * b2));
  DGS_TRY(copy(lse, ts.lse + l * LS, LS * f4));
  DGS_TRY(copy(proj_out, ts.proj_out + l * MD, MD * b2));
  DGS_TRY(copy(h2, ts.h2 + l * MD, MD * b2));
  DGS_TRY(copy(u_pre, ts.u_pre + l * MU, MU * b2));
  DGS_TRY(copy(u, ts.u + l * MU, MU * b2));
  DGS_TRY(copy(fc2_out, ts.fc2_out + l * MD, MD * b2));
  return DGS_OK;
}

int dgs_dit_export_ends(const dgs_dit_weights* w, int B, int V, int H, int W, int train_mode, const void* train_state,
                        const void* workspace, size_t workspace_bytes, float* x_pre, float* c, float* mod, float* gs_tok,
                        float* img_gs, float* dx0, float* dx_pre, float* dmod, float* dc, float* d_gs_tok, void* stream) {
  DGS_TRY(check_dit(w, B, V, H, W));
  DGS_REQUIRE(train_mode == DGS_TRAIN_STORE || train_mode == DGS_TRAIN_RECOMPUTE, "bad train_mode %d", train_mode);
  DGS_REQUIRE(train_state != nullptr, "train_state is NULL");
  DitWorkspace ws(const_cast<void*>(workspace), w, B, V, H, W);
  DGS_REQUIRE(workspace && workspace_bytes >= ws.bytes, "workspace too small: %zu < %zu", workspace_bytes, ws.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t T = (size_t)V * (H / w->patch) * (W / w->patch), N = T + w->n_gaussians, D = w->width;
  const size_t MD = (size_t)B * N * D, mod_n = (size_t)B * ((size_t)w->layers * 6 * D + 4 * D);
  TrainState ts(const_cast<void*>(train_state), w, B, V, H, W, train_mode);
  auto copy = [&](void* dst, const void* src, size_t n) -> int {
    if (dst) DGS_CUDA_OK(cudaMemcpyAsync(dst, src, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return DGS_OK;
  };
  // none of these is written again after the pass that produces it: the forward's by the later forward stages, the
  // backward's by the later backward stages (dx is final once block 0 is differentiated, dcond slice 0 once silu_bwd ran)
  DGS_TRY(copy(x_pre, ts.x_pre, MD));
  DGS_TRY(copy(c, ws.c, (size_t)B * D));
  DGS_TRY(copy(mod, ws.mod, mod_n));
  DGS_TRY(copy(gs_tok, ws.gs_tok, (size_t)B * w->n_gaussians * 14));
  DGS_TRY(copy(img_gs, ws.img_gs, (size_t)B * T * w->patch * w->patch * 14));
  DGS_TRY(copy(dx0, ts.dx, MD));
  DGS_TRY(copy(dx_pre, ts.dx_pre, MD));
  DGS_TRY(copy(dmod, ts.dmod, mod_n));
  DGS_TRY(copy(dc, ts.dcond, (size_t)B * D));
  DGS_TRY(copy(d_gs_tok, ts.d_gs_tok, (size_t)B * w->n_gaussians * 14));
  return DGS_OK;
}

int dgs_dit_backward(const dgs_dit_weights* w, const dgs_dit_weights_t* wT, const dgs_dit_io* io,
                     const dgs_dit_out_grads* dout, const dgs_dit_grads* g, void* workspace, size_t workspace_bytes,
                     void* stream) {
  return dgs_dit_backward_ex(w, wT, io, dout, g, nullptr, workspace, workspace_bytes, stream);
}

int dgs_dit_backward_ex(const dgs_dit_weights* w, const dgs_dit_weights_t* wT, const dgs_dit_io* io,
                        const dgs_dit_out_grads* dout, const dgs_dit_grads* g, const dgs_dit_bwd_opts* opts,
                        void* workspace, size_t workspace_bytes, void* stream) {
  DGS_REQUIRE(io != nullptr && wT != nullptr && dout != nullptr && g != nullptr, "NULL argument");
  DGS_TRY(check_dit(w, io->B, io->V, io->H, io->W));
  DGS_REQUIRE(io->train_state, "dgs_dit_backward: io->train_state is NULL (the forward must run in training mode)");
  DGS_REQUIRE(dout->d_xyz && dout->d_features && dout->d_scaling && dout->d_rotation && dout->d_opacity, "NULL output gradient");
  DGS_REQUIRE(wT->qkv_wT && wT->proj_wT && wT->fc1_wT && wT->fc2_wT && wT->dec_wT && wT->ups_w, "NULL transposed weight");
  cudaStream_t st = (cudaStream_t)stream;
  const int B = io->B, V = io->V, H = io->H, W = io->W, D = w->width, L = w->layers, G = w->n_gaussians, p = w->patch;
  const int T = V * (H / p) * (W / p), N = T + G, Kin = p * p * 9, Ndec = p * p * 14, U = w->mlp_hidden;
  const int M = B * N, Mp = (M + 63) / 64 * 64, Mt = B * T, Mtp = (Mt + 63) / 64 * 64;
  DGS_REQUIRE(B <= 8, "dgs_dit_backward: per-call batch %d > 8 (split the batch)", B);
  DGS_REQUIRE(N >= 64, "dgs_dit_backward: needs at least 64 tokens per sample");
  DitWorkspace ws(workspace, w, B, V, H, W);
  DGS_REQUIRE(workspace && workspace_bytes >= ws.bytes, "workspace too small: %zu < %zu", workspace_bytes, ws.bytes);
  DGS_REQUIRE(io->train_mode == DGS_TRAIN_STORE || io->train_mode == DGS_TRAIN_RECOMPUTE, "bad train_mode %d", io->train_mode);
  const bool recompute = io->train_mode == DGS_TRAIN_RECOMPUTE;
  TrainState ts(io->train_state, w, B, V, H, W, io->train_mode);
  const int mod_stride = L * 6 * D + 4 * D;
  const size_t MD = (size_t)M * D, MU = (size_t)M * U;
  const int Np = attention_lse_stride(N);
  void** done_ev = opts ? opts->block_done : nullptr;

  // gradients accumulated by atomics start from zero; GEMM-produced ones are overwritten
  DGS_CUDA_OK(cudaMemsetAsync(ts.dmod, 0, (size_t)B * mod_stride * sizeof(float), st));
  DGS_CUDA_OK(cudaMemsetAsync(ts.dcond, 0, (size_t)3 * B * D * sizeof(float), st));
  const size_t LS = (size_t)g->layer_stride;
  for (int l = 0; l < L; l++) {
    DGS_CUDA_OK(cudaMemsetAsync(g->qkv_b + l * LS, 0, (size_t)3 * D * sizeof(float), st));
    DGS_CUDA_OK(cudaMemsetAsync(g->proj_b + l * LS, 0, (size_t)D * sizeof(float), st));
    DGS_CUDA_OK(cudaMemsetAsync(g->fc1_b + l * LS, 0, (size_t)U * sizeof(float), st));
    DGS_CUDA_OK(cudaMemsetAsync(g->fc2_b + l * LS, 0, (size_t)D * sizeof(float), st));
  }
  DGS_CUDA_OK(cudaMemsetAsync(g->in_ln_w, 0, D * sizeof(float), st));
  DGS_CUDA_OK(cudaMemsetAsync(g->ups_ln_w, 0, D * sizeof(float), st));
  DGS_CUDA_OK(cudaMemsetAsync(g->dec_ln_w, 0, D * sizeof(float), st));

  auto wgrad = [&](const __nv_bfloat16* dyT, const __nv_bfloat16* xT, float* dW, int n_out, int n_in, int kp) -> int {
    GemmEpilogue ep;  // dW[n_out, n_in] = dY^T [n_out, kp] x (X^T [n_in, kp])^T   (K = padded row count, pads are zero)
    ep.out = dW; ep.ldc = n_in;
    return gemm_bf16(dyT, xT, n_out, n_in, kp, EPI_F32, ep, st);
  };
  auto wgrad_tn = [&](const __nv_bfloat16* dy, int ld_dy, const __nv_bfloat16* x, int ld_x, float* dW, int n_out, int n_in,
                      int rows) -> int {
    GemmEpilogue ep;  // dW[n_out, n_in] = dY[rows, n_out]^T X[rows, n_in]: MN-major operands, nothing transposed in memory
    ep.out = dW; ep.ldc = n_in; ep.lda = ld_dy; ep.ldb = ld_x;
    return gemm_bf16_tn(dy, x, n_out, n_in, rows, ep, st);
  };
  auto dgrad = [&](const __nv_bfloat16* dy, const void* wt, __nv_bfloat16* dxo, int rows, int n_in, int n_out, int epi,
                   void* aux) -> int {
    GemmEpilogue ep;  // dX[rows, n_in] = dY [rows, n_out] x (W^T [n_in, n_out])^T
    ep.out = dxo; ep.ldc = n_in; ep.aux = aux;
    return gemm_bf16(dy, wt, rows, n_in, n_out, epi, ep, st);
  };

  const float* x_fin = ts.x_all + (size_t)L * MD;
  const float* mu = ws.mod + (size_t)L * 6 * D;
  const float* md = mu + 2 * D;
  float* dmu = ts.dmod + (size_t)L * 6 * D;
  float* dmd = dmu + 2 * D;
  {  // ---- heads ----
    ProfScope ps(st, PROF_DIT_BWD_ELEM);
    __nv_bfloat16* d_img = ts.big0;  // [Mt, Ndec]
    DGS_TRY(gaussians_epilogue_bwd(ws.gs_tok, ws.img_gs, io->ray_d, dout->d_xyz, dout->d_features, dout->d_scaling,
                                   dout->d_rotation, dout->d_opacity, ts.d_gs_tok, d_img, B, G, V, H, W, p,
                                   io->scene_depth, io->range_near, io->range_far, st));
    // image_token_decoder: dh = d_img W, dW = d_img^T h
    DGS_TRY(dgrad(d_img, wT->dec_wT, ts.dh, Mt, D, Ndec, EPI_BIAS_BF16, nullptr));
    DGS_TRY(wgrad_tn(d_img, Ndec, ts.hdec, 3 * D, g->dec_w, Ndec, D, Mt));  // hi part of the [hi|lo|hi] operand
    DGS_TRY(ln_modulate_bwd(x_fin, ts.dh, 0, w->dec_ln_w, md + D, mod_stride, B, N, G, T, D, 1e-5f, ts.dx, 0, dmd, dmd + D,
                            g->dec_ln_w, ts.ln_stats, st));
    if (G > 0) {  // upsampler (the free Gaussian tokens, rows 0..G of every sample)
      DGS_TRY(tiny_linear_bwd(ts.d_gs_tok, wT->ups_w, ws.hg, ts.dyb, g->ups_w, B * G, 14, D, st));
      DGS_TRY(ln_modulate_bwd(x_fin, ts.dyb, 0, w->ups_ln_w, mu + D, mod_stride, B, N, 0, G, D, 1e-5f, ts.dx, 0, dmu, dmu + D,
                              g->ups_ln_w, ts.ln_stats, st));
    }
  }

  // ---- L x DiTBlock, reversed ----
  for (int l = L - 1; l >= 0; l--) {
    const float* m = ws.mod + (size_t)l * 6 * D;
    float* dm = ts.dmod + (size_t)l * 6 * D;
    const size_t sl = recompute ? 0 : (size_t)l;  // slot of the per-layer tensors
    if (recompute) {  // refill the single slot: block l's forward from the saved residual stream (denoiser.py:348-354)
      BlockBufs bb = train_bufs(ts, w, l, MD, MU, B, N, /*keep_aux=*/true);
      bb.x_out = ts.dx_pre;  // the block's output is not needed again; dx_pre is free until the input stage
      DGS_TRY(block_forward(w, l, m, mod_stride, B, N, bb, st));
    }
    const float* x_in = ts.x_all + (size_t)l * MD;
    const float* x_mid = ts.x_mid + sl * MD;
    // -- MLP branch: x_out = x_mid + gate_mlp * (fc2(gelu(fc1(h2))) )
    {
      ProfScope ps(st, PROF_DIT_BWD_ELEM);
      DGS_TRY(gate_bwd(ts.dx, ts.fc2_out + sl * MD, m + 5 * D, mod_stride, N, M, D, ts.dyb, nullptr, dm + 5 * D,
                       g->fc2_b + l * LS, st));
    }
    {
      ProfScope ps(st, PROF_DIT_BWD_WGRAD);
      DGS_TRY(wgrad_tn(ts.dyb, D, ts.u + sl * MU, U, g->fc2_w + l * LS, D, U, M));
    }
    {
      ProfScope ps(st, PROF_DIT_BWD_DGRAD);
      DGS_TRY(dgrad(ts.dyb, (const __nv_bfloat16*)wT->fc2_wT + (size_t)l * D * U, ts.big0, M, U, D, EPI_DGELU_BF16,
                    ts.u_pre + sl * MU));  // du_pre = (dy W2) * gelu'(u_pre)
    }
    {
      ProfScope ps(st, PROF_DIT_BWD_ELEM);
      DGS_TRY(colsum_bf16(ts.big0, M, U, g->fc1_b + l * LS, st));
    }
    {
      ProfScope ps(st, PROF_DIT_BWD_WGRAD);
      DGS_TRY(wgrad_tn(ts.big0, U, ts.h2 + sl * MD, D, g->fc1_w + l * LS, U, D, M));
    }
    {
      ProfScope ps(st, PROF_DIT_BWD_DGRAD);
      DGS_TRY(dgrad(ts.big0, (const __nv_bfloat16*)wT->fc1_wT + (size_t)l * D * U, ts.dh, M, D, U, EPI_BIAS_BF16, nullptr));
    }
    {
      ProfScope ps(st, PROF_DIT_BWD_ELEM);
      DGS_TRY(ln_modulate_bwd(x_mid, ts.dh, 0, nullptr, m + 4 * D, mod_stride, B, N, 0, N, D, 1e-6f, ts.dx, 1, dm + 3 * D,
                              dm + 4 * D, nullptr, ts.ln_stats, st));
      // -- attention branch: x_mid = x_in + gate_msa * proj(attn(qkv(h1)))
      DGS_TRY(gate_bwd(ts.dx, ts.proj_out + sl * MD, m + 2 * D, mod_stride, N, M, D, ts.dyb, nullptr, dm + 2 * D,
                       g->proj_b + l * LS, st));
    }
    {
      ProfScope ps(st, PROF_DIT_BWD_WGRAD);
      DGS_TRY(wgrad_tn(ts.dyb, D, ts.attn + sl * MD, D, g->proj_w + l * LS, D, D, M));
    }
    {
      ProfScope ps(st, PROF_DIT_BWD_DGRAD);
      DGS_TRY(dgrad(ts.dyb, (const __nv_bfloat16*)wT->proj_wT + (size_t)l * D * D, ts.dh, M, D, D, EPI_BIAS_BF16, nullptr));
    }
    {
      ProfScope ps(st, PROF_DIT_BWD_ATTN);
      DGS_TRY(attention_bwd(ts.qkv + sl * 3 * MD, ts.attn + sl * MD, ts.dh,
                            ts.lse + sl * B * w->heads * Np, ts.dsum, ts.big0, B, N, w->heads, st));
    }
    {
      ProfScope ps(st, PROF_DIT_BWD_ELEM);
      DGS_TRY(colsum_bf16(ts.big0, M, 3 * D, g->qkv_b + l * LS, st));
    }
    {
      ProfScope ps(st, PROF_DIT_BWD_WGRAD);
      DGS_TRY(wgrad_tn(ts.big0, 3 * D, ts.h1 + sl * MD, D, g->qkv_w + l * LS, 3 * D, D, M));
    }
    {
      ProfScope ps(st, PROF_DIT_BWD_DGRAD);
      DGS_TRY(dgrad(ts.big0, (const __nv_bfloat16*)wT->qkv_wT + (size_t)l * 3 * D * D, ts.dh, M, D, 3 * D, EPI_BIAS_BF16, nullptr));
    }
    {
      ProfScope ps(st, PROF_DIT_BWD_ELEM);
      DGS_TRY(ln_modulate_bwd(x_in, ts.dh, 0, nullptr, m + D, mod_stride, B, N, 0, N, D, 1e-6f, ts.dx, 1, dm, dm + D, nullptr, ts.ln_stats, st));
      // this block's adaLN linear (6w x w, a third of the block's parameters): d mod_l is complete now, so its weight /
      // bias gradient is produced HERE -- every gradient of block l is final at this point and its all-reduce can start
      // while blocks l-1 .. 0 are still being differentiated (block_done event); d silu(c) accumulates across blocks
      DGS_TRY(skinny_linear_bwd(ws.c, w->adaln_w + (size_t)l * 6 * D * D, dm, mod_stride, B, 6 * D, D, 1, g->adaln_w + l * LS,
                                g->adaln_b + l * LS, ts.dcond, st));
    }
    if (done_ev && done_ev[l]) DGS_CUDA_OK(cudaEventRecord((cudaEvent_t)done_ev[l], st));
  }

  ProfScope ps_in(st, PROF_DIT_BWD_ELEM);
  // ---- input stage: LayerNorm(weight) -> [pos tokens | tokenizer GEMM] ----
  DGS_TRY(ln_modulate_bwd(ts.x_pre, ts.dx, 1, w->in_ln_w, nullptr, 0, B, N, 0, N, D, 1e-5f, ts.dx_pre, 0, nullptr, nullptr,
                          g->in_ln_w, ts.ln_stats, st));
  DGS_TRY(pos_embed_bwd(ts.dx_pre, g->pos_embed, B, G, N, D, st));
  DGS_TRY(transpose_to_bf16(ts.dx_pre, 1, D, B, N, G, T, D, ts.bigT0, nullptr, st));          // d tok^T [D, Mtp]
  DGS_TRY(transpose_to_bf16(ws.tokens, 0, 3 * Kin, 1, Mt, 0, Mt, Kin, ts.bigT1, nullptr, st));  // hi part of the patches
  DGS_TRY(wgrad(ts.bigT0, ts.bigT1, g->tokenizer_w, D, Kin, Mtp));

  // ---- conditioning: adaLN modulation of all blocks + heads, then the timestep MLP ----
  float* dsc = ts.dcond;                       // d silu(c), then dc
  float* dt1 = ts.dcond + (size_t)B * D;       // d temb1, then d pre1
  float* pre1 = ts.dcond + (size_t)2 * B * D;  // t0 pre-activation (recomputed)
  {  // the two heads' adaLN linears in one launch (the blocks' ones were differentiated inside the block loop)
    SkinnySegs segs;
    segs.seg_rows = 0; segs.n_seg = 0; segs.seg_stride = 0; segs.dW0 = nullptr; segs.db0 = nullptr;
    segs.tail_rows[0] = 2 * D; segs.tail_dW[0] = g->ups_adaln_w; segs.tail_db[0] = g->ups_adaln_b;
    segs.tail_rows[1] = 2 * D; segs.tail_dW[1] = g->dec_adaln_w; segs.tail_db[1] = g->dec_adaln_b;
    DGS_TRY(skinny_linear_bwd_segs(ws.c, w->adaln_w + (size_t)L * 6 * D * D, ts.dmod + (size_t)L * 6 * D, mod_stride, B, 4 * D, D,
                                   1, segs, dsc, st));
  }
  DGS_TRY(silu_bwd_inplace(dsc, ws.c, B * D, st));
  DGS_TRY(skinny_linear_bwd(ws.temb1, w->t2_w, dsc, D, B, D, D, 0, g->t2_w, g->t2_b, dt1, st));
  DGS_TRY(skinny_linear(ws.temb0, w->t0_w, w->t0_b, pre1, B, D, 256, 0, 0, st));
  DGS_TRY(silu_bwd_inplace(dt1, pre1, B * D, st));
  DGS_TRY(skinny_linear_bwd(ws.temb0, w->t0_w, dt1, D, B, D, 256, 0, g->t0_w, g->t0_b, nullptr, st));
  if (done_ev && done_ev[L]) DGS_CUDA_OK(cudaEventRecord((cudaEvent_t)done_ev[L], st));
  return DGS_OK;
}

int dgs_event_create(void** ev) {
  DGS_REQUIRE(ev != nullptr, "NULL pointer");
  cudaEvent_t e;
  DGS_CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  *ev = (void*)e;
  return DGS_OK;
}

int dgs_event_destroy(void* ev) {
  if (ev) DGS_CUDA_OK(cudaEventDestroy((cudaEvent_t)ev));
  return DGS_OK;
}

int dgs_stream_wait_event(void* stream, void* ev) {
  DGS_REQUIRE(ev != nullptr, "NULL event");
  DGS_CUDA_OK(cudaStreamWaitEvent((cudaStream_t)stream, (cudaEvent_t)ev, 0));
  return DGS_OK;
}

int dgs_transpose_bf16(const void* in, int in_is_f32, int M, int C, void* out, float* colsum, void* stream) {
  DGS_REQUIRE(in && out && M > 0, "NULL pointer / bad shape");
  return transpose_to_bf16(in, in_is_f32, C, 1, M, 0, M, C, (__nv_bfloat16*)out, colsum, (cudaStream_t)stream);
}

int dgs_adamw_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, size_t n, float lr, float beta1,
                   float beta2, float eps, float weight_decay, int step, float grad_scale, const float* grad_scale_dev,
                   void* stream) {
  DGS_REQUIRE(param && grad && exp_avg && exp_avg_sq && step >= 1, "bad AdamW arguments");
  return adamw_step(param, grad, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, step, grad_scale,
                    grad_scale_dev, (cudaStream_t)stream);
}

int dgs_adamw_ema_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, float* ema, size_t n, float lr,
                       float beta1, float beta2, float eps, float weight_decay, int step, float grad_scale,
                       const float* grad_scale_dev, float ema_decay, void* stream) {
  DGS_REQUIRE(param && grad && exp_avg && exp_avg_sq && step >= 1, "bad AdamW arguments");
  DGS_REQUIRE(!ema || (ema_decay >= 0.f && ema_decay <= 1.f), "EMA decay must be in [0, 1]");  // ema.py:56-57
  return adamw_step(param, grad, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, step, grad_scale,
                    grad_scale_dev, (cudaStream_t)stream, ema, ema_decay);
}

int dgs_cast_transpose_f32(const float* in, long long in_batch_stride, int batch, int M, int C, void* out_bf16,
                           void* outT_bf16, void* stream) {
  DGS_REQUIRE(in && outT_bf16 && batch > 0, "bad arguments");
  return cast_transpose_f32(in, in_batch_stride, batch, M, C, (__nv_bfloat16*)out_bf16, (__nv_bfloat16*)outT_bf16,
                            (cudaStream_t)stream);
}

int dgs_attention_fwd_train(const void* qkv, void* out, float* lse2, int B, int N, int heads, void* stream) {
  DGS_REQUIRE(qkv && out && lse2, "NULL pointer");
  return attention_fwd(qkv, out, lse2, B, N, heads, (cudaStream_t)stream);
}

int dgs_attention_bwd(const void* qkv, const void* out, const void* dout, float* lse2, float* dsum, void* dqkv, int B,
                      int N, int heads, void* stream) {
  DGS_REQUIRE(qkv && out && dout && lse2 && dsum && dqkv, "NULL pointer");
  return attention_bwd(qkv, out, dout, lse2, dsum, dqkv, B, N, heads, (cudaStream_t)stream);
}

int dgs_gemm_bf16_ex(const void* A, const void* Wt, const float* bias, const float* gate, void* out, void* aux,
                     const float* resid, int M, int N, int K, int lda, int ldb, int epi, int ldc, int gate_stride,
                     int rows_per_sample, void* stream) {
  DGS_REQUIRE(A && Wt && out, "NULL pointer");
  DGS_REQUIRE(epi != EPI_GATE_RESID_F32 || (gate && rows_per_sample > 0), "gate epilogue needs gate and rows_per_sample");
  GemmEpilogue ep;
  ep.out = out; ep.ldc = ldc; ep.bias = bias; ep.gate = gate; ep.gate_stride = gate_stride;
  ep.rows_per_sample = rows_per_sample > 0 ? rows_per_sample : 1;
  ep.aux = aux; ep.resid = resid; ep.lda = lda; ep.ldb = ldb;
  return gemm_bf16(A, Wt, M, N, K, epi, ep, (cudaStream_t)stream);
}

int dgs_gemm_bf16_tn(const void* A, const void* W, float* out, int M, int N, int K, int lda, int ldb, int ldc, void* stream) {
  DGS_REQUIRE(A && W && out, "NULL pointer");
  GemmEpilogue ep;
  ep.out = out; ep.ldc = ldc; ep.lda = lda; ep.ldb = ldb;
  return gemm_bf16_tn(A, W, M, N, K, ep, (cudaStream_t)stream);
}

int dgs_ln_modulate_bwd(const float* x, const void* dh, int dh_is_f32, const float* ln_w, const float* scale,
                        int mod_stride, int B, int rows, int width, float eps, float* dx, int accumulate, float* dshift,
                        float* dscale, float* dln_w, float* stats, void* stream) {
  DGS_REQUIRE(x && dh && dx && stats, "NULL pointer");
  return ln_modulate_bwd(x, dh, dh_is_f32, ln_w, scale, mod_stride, B, rows, 0, rows, width, eps, dx, accumulate, dshift,
                         dscale, dln_w, stats, (cudaStream_t)stream);
}

int dgs_gate_bwd(const float* dx, const void* y, const float* gate, int gate_stride, int rows_per_sample, int M, int C,
                 void* dy, void* dyT, float* dgate, float* dbias, void* stream) {
  DGS_REQUIRE(dx && y && gate && dy && dgate, "NULL pointer");
  return gate_bwd(dx, (const __nv_bfloat16*)y, gate, gate_stride, rows_per_sample, M, C, (__nv_bfloat16*)dy,
                  (__nv_bfloat16*)dyT, dgate, dbias, (cudaStream_t)stream);
}

int dgs_gemm_bf16(const void* A, const void* Wt, const float* bias, const float* gate, void* out, int M, int N, int K,
                  int epi, int ldc, int gate_stride, int rows_per_sample, void* stream) {
  DGS_REQUIRE(A && Wt && out, "NULL pointer");
  DGS_REQUIRE(epi != EPI_GATE_RESID_F32 || (gate && rows_per_sample > 0), "gate epilogue needs gate and rows_per_sample");
  GemmEpilogue ep;
  ep.out = out; ep.ldc = ldc; ep.bias = bias; ep.gate = gate; ep.gate_stride = gate_stride;
  ep.rows_per_sample = rows_per_sample > 0 ? rows_per_sample : 1;
  return gemm_bf16(A, Wt, M, N, K, epi, ep, (cudaStream_t)stream);
}

int dgs_attention_fwd(const void* qkv, void* out, int B, int N, int heads, void* stream) {
  DGS_REQUIRE(qkv && out, "NULL pointer");
  return attention_fwd(qkv, out, nullptr, B, N, heads, (cudaStream_t)stream);
}

int dgs_ln_modulate(const float* x, const float* ln_w, const float* shift, const float* scale, int mod_stride, void* h,
                    int B, int rows, int width, float eps, void* stream) {
  DGS_REQUIRE(x && shift && scale && h, "NULL pointer");
  return ln_modulate(x, ln_w, shift, scale, mod_stride, (__nv_bfloat16*)h, B, rows, 0, rows, width, eps, 0,
                     (cudaStream_t)stream);
}

}  // extern "C"
