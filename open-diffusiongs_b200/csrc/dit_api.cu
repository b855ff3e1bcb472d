// dit_api.cu -- C ABI of the DiT denoiser forward (include/dgs_b200.h, section B2): orchestrates the
// wgmma GEMMs, the wgmma attention and the glue kernels into DGSDenoiser.image_to_gaussians
// (diffusionGS/models/denoiser/denoiser.py:306-416).
#include <algorithm>

#include "dgs_internal.h"
#include "dit_kernels.h"

using namespace dgs;

namespace {

// Channels per Gaussian of both heads (denoiser.py:94-98, 145-149): xyz 3, SH features 3 (d+1)^2, scaling 3, rotation 4,
// opacity 1.
int head_channels(int sh_degree) { return 11 + 3 * (sh_degree + 1) * (sh_degree + 1); }

// The shapes of one DiT call, from the weights' config and the input size B x V x H x W: T image tokens and G free
// Gaussian tokens per sample, N = T + G, M = B*N rows, Mt = B*T image-token rows; Mp / Mtp round them up to 64.
struct DitDims {
  int B, T, G, N, M, Mp, Mt, Mtp;
  int D, U;          // width, mlp_hidden
  int heads;
  int C;             // raw head channels per Gaussian, 11 + 3 (sh_degree+1)^2
  int Kin, Ndec;     // patch*patch*9 tokenizer inputs, patch*patch*C decoder outputs per token
  int mod_stride;    // L*6w + 4w: the adaLN modulation of every block and of both heads, per sample
  size_t MD, MU;     // elements of an [M, w] and an [M, mlp_hidden] tensor
  size_t lse_n;      // floats of one block's attention log-sum-exp, [B, heads, attention_lse_stride(N)]
  DitDims(const dgs_dit_weights* w, int B_, int V, int H, int W)
      : B(B_), T(V * (H / w->patch) * (W / w->patch)), G(w->n_gaussians), N(T + G), M(B * N), Mp((M + 63) / 64 * 64),
        Mt(B * T), Mtp((Mt + 63) / 64 * 64), D(w->width), U(w->mlp_hidden), C(head_channels(w->sh_degree)),
        Kin(w->patch * w->patch * 9), Ndec(w->patch * w->patch * C), heads(w->heads),
        mod_stride(w->layers * 6 * D + 4 * D), MD((size_t)M * D), MU((size_t)M * U),
        lse_n((size_t)B * w->heads * attention_lse_stride(N)) {}
};

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
  float* gs_tok;          // [B*G, C]
  float* img_gs;          // [B*T, p*p*C]
  // FP8 inference only, carved after the bf16 workspace: the activation scales of the e4m3 copies of h (LN outputs,
  // [w/128][Ms]) and u (GELU output, [4w/128][Ms]); the e4m3 activations themselves live in h / u.
  float* sa_h;
  float* sa_u;
  // DGS_FP8_ATTENTION only, carved after those: the e4m3 attention operands of one block and their scales
  uint8_t *q8, *k8, *vt8;
  float *sq, *sk, *sv;
  size_t bytes;          // without the FP8 scales
  size_t bytes_fp8;      // with them
  size_t bytes_fp8_att;  // with the FP8 attention operands as well
  DitWorkspace(void* base, const DitDims& d) {
    Carver c_(base);
    tokens = c_.take<__nv_bfloat16>((size_t)d.Mt * 3 * d.Kin);
    tok = c_.take<float>((size_t)d.Mt * d.D);
    x = c_.take<float>(d.MD);
    h = c_.take<__nv_bfloat16>(d.MD);
    qkv = c_.take<__nv_bfloat16>(3 * d.MD);
    attn = c_.take<__nv_bfloat16>(d.MD);
    u = c_.take<__nv_bfloat16>(d.MU);
    temb0 = c_.take<float>((size_t)d.B * 256);
    temb1 = c_.take<float>((size_t)d.B * d.D);
    c = c_.take<float>((size_t)d.B * d.D);
    mod = c_.take<float>((size_t)d.B * d.mod_stride);
    hg = c_.take<__nv_bfloat16>((size_t)d.B * d.G * 3 * d.D);
    gs_tok = c_.take<float>((size_t)d.B * d.G * d.C);
    img_gs = c_.take<float>((size_t)d.Mt * d.Ndec);
    bytes = c_.bytes();
    const size_t Ms = (size_t)fp8_scale_stride(d.M);
    sa_h = c_.take<float>((size_t)(d.D / 128) * Ms);
    sa_u = c_.take<float>((size_t)(d.U / 128) * Ms);
    bytes_fp8 = c_.bytes();
    const size_t Nk = attention_lse_stride(d.N), BH = (size_t)d.B * d.heads;
    q8 = c_.take<uint8_t>(d.MD);
    k8 = c_.take<uint8_t>(d.MD);
    vt8 = c_.take<uint8_t>(BH * 64 * Nk);
    sq = c_.take<float>(BH * d.N);
    sk = c_.take<float>(BH * Nk / 128);
    sv = c_.take<float>(BH * Nk / 128);
    bytes_fp8_att = c_.bytes();
  }
};

// Everything the backward needs from the forward (training mode), plus the backward's own scratch.  Per-layer tensors
// are stacked along a leading L axis.
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
  float* skb_part;          // per-CTA partial sums of the adaLN / timestep-MLP input gradients (skinny_linear_bwd)
  float* d_gs_tok;          // [B*G, C]
  __nv_bfloat16* dyb;       // [M, w]      gated branch gradient / generic [M, w] bf16
  __nv_bfloat16* dh;        // [M, w]
  __nv_bfloat16* big0;      // [M, max(4w, 3w, Ndec)]  du / dqkv / d_img_gs [Mt, Ndec]
  __nv_bfloat16* bigT0;     // [w, Mp]     transposed token gradient (tokenizer weight gradient only)
  __nv_bfloat16* bigT1;     // [w, Mp]     transposed patches        (tokenizer weight gradient only)
  size_t bytes;
  TrainState(void* base, const dgs_dit_weights* w, const DitDims& d, int mode) {
    const size_t Lx = w->layers, L = mode == DGS_TRAIN_RECOMPUTE ? 1 : Lx;  // slots of the per-layer tensors
    const size_t MD = d.MD, MU = d.MU, D = d.D;
    const size_t wide = std::max({d.U, 3 * d.D, d.Ndec});
    Carver c(base);
    x_pre = c.take<float>(MD);
    x_all = c.take<float>((Lx + 1) * MD);
    x_mid = c.take<float>(L * MD);
    h1 = c.take<__nv_bfloat16>(L * MD);
    h2 = c.take<__nv_bfloat16>(L * MD);
    qkv = c.take<__nv_bfloat16>(L * 3 * MD);
    attn = c.take<__nv_bfloat16>(L * MD);
    lse = c.take<float>(L * d.lse_n);
    proj_out = c.take<__nv_bfloat16>(L * MD);
    fc2_out = c.take<__nv_bfloat16>(L * MD);
    u_pre = c.take<__nv_bfloat16>(L * MU);
    u = c.take<__nv_bfloat16>(L * MU);
    hdec = c.take<__nv_bfloat16>((size_t)d.Mt * 3 * D);
    dx = c.take<float>(MD);
    dx_pre = c.take<float>(MD);
    dmod = c.take<float>((size_t)d.B * d.mod_stride);
    dsum = c.take<float>(d.lse_n);
    dcond = c.take<float>((size_t)3 * d.B * D);
    ln_stats = c.take<float>(2 * (size_t)d.M);
    skb_part = c.take<float>(skinny_linear_bwd_part_floats(d.B, 6 * d.D, d.D));  // the widest: a block's 6w rows
    d_gs_tok = c.take<float>((size_t)d.B * d.G * d.C + 16);
    dyb = c.take<__nv_bfloat16>(MD);
    dh = c.take<__nv_bfloat16>(MD);
    big0 = c.take<__nv_bfloat16>((size_t)d.M * wide);
    bigT0 = c.take<__nv_bfloat16>(D * d.Mp);
    bigT1 = c.take<__nv_bfloat16>(D * d.Mp);
    bytes = c.bytes();
  }
};

int check_dit(const dgs_dit_weights* w, int B, int V, int H, int W) {
  DGS_REQUIRE(w != nullptr, "weights is NULL");
  DGS_REQUIRE(w->width == 1024 && w->heads * 64 == w->width, "unsupported width/heads %d/%d (1024/16 only)", w->width, w->heads);
  DGS_REQUIRE(w->layers > 0 && w->patch > 0 && w->n_gaussians >= 0 && w->mlp_hidden % 256 == 0, "bad DiT config");
  DGS_REQUIRE(B > 0 && V > 0 && H % w->patch == 0 && W % w->patch == 0, "bad input shape B=%d V=%d H=%d W=%d", B, V, H, W);
  DGS_REQUIRE(w->sh_degree >= 0 && w->sh_degree <= 3, "sh_degree %d unsupported (0..3, as the rasterizer evaluates)",
              w->sh_degree);
  DGS_REQUIRE((w->patch * w->patch * 9) % 8 == 0, "patch %d unsupported", w->patch);
  DGS_REQUIRE((w->patch * w->patch * head_channels(w->sh_degree)) % 32 == 0,
              "patch %d with sh_degree %d: the decoder head's patch^2 * %d outputs per token must be a multiple of 32 "
              "(the GEMM's N %% 32 rule)", w->patch, w->sh_degree, head_channels(w->sh_degree));
  DGS_REQUIRE(w->mlp_hidden >= 3 * w->width, "mlp_hidden must be >= 3*width (decoder head re-uses that buffer)");
  return DGS_OK;
}

int check_train_mode(int mode) {
  DGS_REQUIRE(mode == DGS_TRAIN_STORE || mode == DGS_TRAIN_RECOMPUTE, "bad train_mode %d", mode);
  return DGS_OK;
}

#define DGS_TRY(expr)       \
  do {                      \
    int _rc = (expr);       \
    if (_rc) return _rc;    \
  } while (0)

// Buffers of ONE DiTBlock (utils_transformer.py:270-290).  Inference: every block re-uses the workspace and the
// residual stream is updated in place (x_in == x_mid == x_out, TMA reduce-add epilogue).  Training: x_in / x_mid / x_out
// are distinct fp32 tensors and the pre-gate branch outputs / pre-GELU values are kept for the backward.
struct BlockBufs {
  float* x_in; float* x_mid; float* x_out;
  float* x_save;                               // NULL, or where the stream entering the block is snapshot
  __nv_bfloat16 *h1, *h2, *qkv, *attn, *u;     // h1 / h2 / u hold e4m3 on the FP8 path
  __nv_bfloat16 *proj_out, *fc2_out, *u_pre;  // training only (NULL: not stored)
  float* lse;                                  // training only
  float *sa_h, *sa_u;                          // FP8 only: the activation scales of h1 / h2 and of u
  uint8_t *q8, *k8, *vt8;                      // DGS_FP8_ATTENTION only: the e4m3 attention operands ...
  float *sq, *sk, *sv;                         // ... and their scales
};

enum BlockPlan { PLAN_INFER, PLAN_STORE, PLAN_RECOMPUTE, PLAN_REFILL };

// The buffers of block l for each way a block runs; the one place that knows the train state's per-layer slots.
//   PLAN_INFER      inference, bf16 or FP8: the workspace, residual stream updated in place (TMA reduce-add epilogues);
//   PLAN_STORE      store-mode training forward: slice l of the stacked tensors, with the stores the backward reads;
//   PLAN_RECOMPUTE  recompute-mode training forward: PLAN_INFER, plus a snapshot of the stream entering the block into
//                   x_all[l] (all the backward keeps per layer);
//   PLAN_REFILL     recompute-mode backward: block l's forward re-run from x_all[l] into the single slot, with the
//                   stores; its output is not needed again, so it goes to dx_pre, which is free until the input stage.
// The backward and dgs_dit_export_state read block l's forward tensors through PLAN_STORE / PLAN_REFILL.  l == L
// addresses the stream leaving the last block: x_in (and x_save for PLAN_RECOMPUTE).
BlockBufs block_bufs(BlockPlan plan, int l, const DitDims& d, const DitWorkspace& ws, const TrainState& ts) {
  BlockBufs b = {};
  if (plan == PLAN_INFER || plan == PLAN_RECOMPUTE) {
    b.x_in = b.x_mid = b.x_out = ws.x;
    b.h1 = b.h2 = ws.h; b.qkv = ws.qkv; b.attn = ws.attn; b.u = ws.u;
    b.sa_h = ws.sa_h; b.sa_u = ws.sa_u;
    b.q8 = ws.q8; b.k8 = ws.k8; b.vt8 = ws.vt8; b.sq = ws.sq; b.sk = ws.sk; b.sv = ws.sv;
    if (plan == PLAN_RECOMPUTE) b.x_save = ts.x_all + (size_t)l * d.MD;
    return b;
  }
  const size_t s = plan == PLAN_STORE ? (size_t)l : 0;
  b.x_in = ts.x_all + (size_t)l * d.MD;
  b.x_mid = ts.x_mid + s * d.MD;
  b.x_out = plan == PLAN_STORE ? ts.x_all + (size_t)(l + 1) * d.MD : ts.dx_pre;
  b.h1 = ts.h1 + s * d.MD; b.h2 = ts.h2 + s * d.MD; b.qkv = ts.qkv + s * 3 * d.MD; b.attn = ts.attn + s * d.MD;
  b.u = ts.u + s * d.MU;
  b.proj_out = ts.proj_out + s * d.MD; b.fc2_out = ts.fc2_out + s * d.MD; b.u_pre = ts.u_pre + s * d.MU;
  b.lse = ts.lse + s * d.lse_n;
  return b;
}

// One DiTBlock forward.  w8 != NULL: the LayerNorms emit e4m3 and qkv, fc1 and fc2 run on the FP8 weights (inference
// only); attn.proj is the bf16 path's either way, attention too unless fp8_flags has DGS_FP8_ATTENTION (then the qkv
// output is quantized to e4m3 and attention runs on it).
int block_forward(const dgs_dit_weights* w, const dgs_dit_weights_fp8* w8, int fp8_flags, int l, const float* m,
                  const DitDims& d, const BlockBufs& b, cudaStream_t st) {
  const int B = d.B, N = d.N, M = d.M, D = d.D, U = d.U, ms = d.mod_stride;
  {
    ProfScope ps(st, PROF_DIT_LN);
    DGS_TRY(ln_forward(w8 ? LN_E4M3 : LN_BF16, b.x_in, nullptr, m, m + D, ms, b.h1, b.sa_h, B, N, 0, N, D, 1e-6f, st));
  }
  {
    ProfScope ps(st, PROF_DIT_GEMM_QKV);
    GemmEpilogue ep;
    ep.out = b.qkv; ep.ldc = 3 * D; ep.bias = w->qkv_b + (size_t)l * 3 * D;
    if (w8)
      DGS_TRY(gemm_fp8(b.h1, b.sa_h, (const uint8_t*)w8->qkv_w + (size_t)l * 3 * D * D, w8->qkv_s + (size_t)l * 3 * D, M,
                       3 * D, D, EPI_BIAS_BF16, ep, nullptr, st));
    else
      DGS_TRY(gemm_bf16(b.h1, (const __nv_bfloat16*)w->qkv_w + (size_t)l * 3 * D * D, M, 3 * D, D, EPI_BIAS_BF16, ep, st));
  }
  {
    ProfScope ps(st, PROF_DIT_ATTN);
    if (fp8_flags & DGS_FP8_ATTENTION) {
      DGS_TRY(attention_quantize_e4m3(b.qkv, b.q8, b.k8, b.vt8, b.sq, b.sk, b.sv, B, N, w->heads, st));
      DGS_TRY(attention_fwd_e4m3(b.q8, b.k8, b.vt8, b.sq, b.sk, b.sv, b.attn, B, N, w->heads, st));
    } else {
      DGS_TRY(attention_fwd(b.qkv, b.attn, b.lse, B, N, w->heads, st));
    }
  }
  {
    ProfScope ps(st, PROF_DIT_GEMM_PROJ);
    GemmEpilogue ep;
    ep.out = b.x_mid; ep.ldc = D; ep.bias = w->proj_b + (size_t)l * D;
    ep.gate = m + 2 * D; ep.gate_stride = ms; ep.rows_per_sample = N;
    ep.resid = b.x_in == b.x_mid ? nullptr : b.x_in; ep.aux = b.proj_out;  // resid NULL: reduce-add into out in place
    DGS_TRY(gemm_bf16(b.attn, (const __nv_bfloat16*)w->proj_w + (size_t)l * D * D, M, D, D, EPI_GATE_RESID_F32, ep, st));
  }
  {
    ProfScope ps(st, PROF_DIT_LN);
    DGS_TRY(ln_forward(w8 ? LN_E4M3 : LN_BF16, b.x_mid, nullptr, m + 3 * D, m + 4 * D, ms, b.h2, b.sa_h, B, N, 0, N, D,
                       1e-6f, st));
  }
  {
    ProfScope ps(st, PROF_DIT_GEMM_FC1);
    GemmEpilogue ep;
    ep.out = b.u; ep.ldc = U; ep.bias = w->fc1_b + (size_t)l * U;
    ep.aux = b.u_pre;
    if (w8)
      DGS_TRY(gemm_fp8(b.h2, b.sa_h, (const uint8_t*)w8->fc1_w + (size_t)l * U * D, w8->fc1_s + (size_t)l * U, M, U, D,
                       EPI_BIAS_GELU_E4M3, ep, b.sa_u, st));
    else
      DGS_TRY(gemm_bf16(b.h2, (const __nv_bfloat16*)w->fc1_w + (size_t)l * U * D, M, U, D, EPI_BIAS_GELU_BF16, ep, st));
  }
  {
    ProfScope ps(st, PROF_DIT_GEMM_FC2);
    GemmEpilogue ep;
    ep.out = b.x_out; ep.ldc = D; ep.bias = w->fc2_b + (size_t)l * D;
    ep.gate = m + 5 * D; ep.gate_stride = ms; ep.rows_per_sample = N;
    ep.resid = b.x_mid == b.x_out ? nullptr : b.x_mid; ep.aux = b.fc2_out;
    if (w8)
      DGS_TRY(gemm_fp8(b.u, b.sa_u, (const uint8_t*)w8->fc2_w + (size_t)l * D * U, w8->fc2_s + (size_t)l * D, M, D, U,
                       EPI_GATE_RESID_F32, ep, nullptr, st));
    else
      DGS_TRY(gemm_bf16(b.u, (const __nv_bfloat16*)w->fc2_w + (size_t)l * D * U, M, D, U, EPI_GATE_RESID_F32, ep, st));
  }
  return DGS_OK;
}

// dgs_dit_forward (w8 == NULL) and dgs_dit_forward_fp8_ex (w8 != NULL: inference with the FP8 block GEMMs, plus the
// FP8 attention with fp8_flags = DGS_FP8_ATTENTION)
int dit_forward(const dgs_dit_weights* w, const dgs_dit_weights_fp8* w8, int fp8_flags, const dgs_dit_io* io,
                void* workspace, size_t workspace_bytes, cudaStream_t st) {
  DGS_REQUIRE(io != nullptr, "io is NULL");
  DGS_TRY(check_dit(w, io->B, io->V, io->H, io->W));
  DGS_REQUIRE(io->images && io->ray_o && io->ray_d && io->t, "NULL input");
  DGS_REQUIRE(io->xyz && io->features && io->scaling && io->rotation && io->opacity, "NULL output");
  const DitDims d(w, io->B, io->V, io->H, io->W);
  const int B = d.B, T = d.T, N = d.N, G = d.G, D = d.D, L = w->layers, p = w->patch, mod_stride = d.mod_stride;
  DitWorkspace ws(workspace, d);
  const size_t need = !w8 ? ws.bytes : (fp8_flags & DGS_FP8_ATTENTION) ? ws.bytes_fp8_att : ws.bytes_fp8;
  DGS_REQUIRE(workspace && workspace_bytes >= need, "workspace too small: %zu < %zu", workspace_bytes, need);
  const bool train = io->train_state != nullptr;
  DGS_TRY(check_train_mode(io->train_mode));
  TrainState ts(io->train_state, w, d, io->train_mode);
  const BlockPlan plan = !train ? PLAN_INFER : io->train_mode == DGS_TRAIN_RECOMPUTE ? PLAN_RECOMPUTE : PLAN_STORE;
  float* x0 = block_bufs(plan, 0, d, ws, ts).x_in;  // residual stream entering block 0

  // ---- input stage: posed image -> tokens -> tokenizer GEMM -> [pos tokens | image tokens] -> LayerNorm(weight) ----
  if (g_prof_on) prof_begin(st, PROF_DIT_INPUT);
  DGS_TRY(posed_patchify(io->images, io->ray_o, io->ray_d, ws.tokens, B, io->V, io->H, io->W, p, io->plucker_mode, st));
  {
    GemmEpilogue ep;
    ep.out = ws.tok; ep.ldc = D;
    DGS_TRY(gemm_bf16(ws.tokens, w->tokenizer_w, d.Mt, D, 3 * d.Kin, EPI_F32, ep, st));  // split-bf16: K = 3*576
  }
  DGS_TRY(assemble_tokens(ws.tok, w->pos_embed, x0, B, G, T, D, st));
  if (train) DGS_CUDA_OK(cudaMemcpyAsync(ts.x_pre, x0, d.MD * sizeof(float), cudaMemcpyDeviceToDevice, st));
  // in place, nn.LayerNorm's default eps (denoiser.py:234-236)
  DGS_TRY(ln_forward(LN_F32, x0, w->in_ln_w, nullptr, nullptr, 0, x0, nullptr, 1, d.M, 0, d.M, D, 1e-5f, st));
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
    const BlockBufs bb = block_bufs(plan, l, d, ws, ts);
    if (bb.x_save) DGS_CUDA_OK(cudaMemcpyAsync(bb.x_save, bb.x_in, d.MD * sizeof(float), cudaMemcpyDeviceToDevice, st));
    DGS_TRY(block_forward(w, w8, fp8_flags, l, m, d, bb, st));
  }
  const BlockBufs fin = block_bufs(plan, L, d, ws, ts);  // the stream leaving the last block
  if (fin.x_save) DGS_CUDA_OK(cudaMemcpyAsync(fin.x_save, fin.x_in, d.MD * sizeof(float), cudaMemcpyDeviceToDevice, st));
  const float* x_fin = fin.x_in;
  if (io->tokens_out)
    DGS_CUDA_OK(cudaMemcpyAsync(io->tokens_out, x_fin, d.MD * sizeof(float), cudaMemcpyDeviceToDevice, st));

  // ---- heads (denoiser.py:76-164): LN(weight) + modulate + Linear ----
  ProfScope ps_heads(st, PROF_DIT_HEADS);
  const float* mu = ws.mod + (size_t)L * 6 * D;  // upsampler: shift | scale
  const float* md = mu + 2 * D;                  // image_token_decoder: shift | scale
  if (G > 0) {
    DGS_TRY(ln_forward(LN_SPLIT_BF16, x_fin, w->ups_ln_w, mu, mu + D, mod_stride, ws.hg, nullptr, B, N, 0, G, D, 1e-5f, st));
    DGS_TRY(tiny_linear_bf16(ws.hg, (const __nv_bfloat16*)w->ups_w, ws.gs_tok, B * G, d.C, 3 * D, st));
  }
  // the decoder head runs split-bf16 (K = 3*width) so the Gaussian parameters are fp32-accurate functions of the
  // residual stream; its A operand re-uses the (now free) MLP hidden buffer
  __nv_bfloat16* hdec = train ? ts.hdec : ws.u;
  DGS_TRY(ln_forward(LN_SPLIT_BF16, x_fin, w->dec_ln_w, md, md + D, mod_stride, hdec, nullptr, B, N, G, T, D, 1e-5f, st));
  {
    GemmEpilogue ep;
    ep.out = ws.img_gs; ep.ldc = d.Ndec;
    DGS_TRY(gemm_bf16(hdec, w->dec_w, d.Mt, d.Ndec, 3 * D, EPI_F32, ep, st));
  }
  GsOut go;
  go.xyz = io->xyz; go.features = io->features; go.scaling = io->scaling; go.rotation = io->rotation;
  go.opacity = io->opacity; go.img_aligned_xyz = io->img_aligned_xyz;
  DGS_TRY(gaussians_epilogue(ws.gs_tok, ws.img_gs, io->ray_o, io->ray_d, go, B, G, io->V, io->H, io->W, p,
                             w->sh_degree, io->scene_depth, io->range_near, io->range_far, st));
  return DGS_OK;
}

// ---- backward ----

// trace read-out: slice `slice` of the stacked caller buffer `base` <- `bytes` of src (NULL field: nothing)
int trace_out(void* base, int slice, const void* src, size_t bytes, cudaStream_t st) {
  if (base) DGS_CUDA_OK(cudaMemcpyAsync((char*)base + (size_t)slice * bytes, src, bytes, cudaMemcpyDeviceToDevice, st));
  return DGS_OK;
}

// dW[n_out, n_in] = dY[rows, n_out]^T X[rows, n_in]: MN-major operands, nothing transposed in memory
int wgrad_tn(const __nv_bfloat16* dy, int ld_dy, const __nv_bfloat16* x, int ld_x, float* dW, int n_out, int n_in,
             int rows, cudaStream_t st) {
  GemmEpilogue ep;
  ep.out = dW; ep.ldc = n_in; ep.lda = ld_dy; ep.ldb = ld_x;
  return gemm_bf16_tn(dy, x, n_out, n_in, rows, ep, st);
}

// dX[rows, n_in] = dY [rows, n_out] x (W^T [n_in, n_out])^T, epilogue epi (aux: its input, if any)
int dgrad(const __nv_bfloat16* dy, const void* wt, __nv_bfloat16* dxo, int rows, int n_in, int n_out, int epi,
          void* aux, cudaStream_t st) {
  GemmEpilogue ep;
  ep.out = dxo; ep.ldc = n_in; ep.aux = aux;
  return gemm_bf16(dy, wt, rows, n_in, n_out, epi, ep, st);
}

// Backward of the two heads and of to_gs: the gradient of the final stream x_fin into ts.dx, the heads' d mod into
// their slices of ts.dmod.
int heads_backward(const dgs_dit_weights* w, const dgs_dit_weights_t* wT, const dgs_dit_io* io,
                   const dgs_dit_out_grads* dout, const dgs_dit_grads* g, const DitDims& d, const DitWorkspace& ws,
                   const TrainState& ts, const float* x_fin, cudaStream_t st) {
  const int B = d.B, N = d.N, T = d.T, G = d.G, D = d.D, L = w->layers;
  const float* mu = ws.mod + (size_t)L * 6 * D;
  const float* md = mu + 2 * D;
  float* dmu = ts.dmod + (size_t)L * 6 * D;
  float* dmd = dmu + 2 * D;
  ProfScope ps(st, PROF_DIT_BWD_ELEM);
  __nv_bfloat16* d_img = ts.big0;  // [Mt, Ndec]
  DGS_TRY(gaussians_epilogue_bwd(ws.gs_tok, ws.img_gs, io->ray_d, dout->d_xyz, dout->d_features, dout->d_scaling,
                                 dout->d_rotation, dout->d_opacity, dout->d_img_aligned_xyz, ts.d_gs_tok, d_img, B, G,
                                 io->V, io->H, io->W, w->patch, w->sh_degree, io->scene_depth, io->range_near,
                                 io->range_far, st));
  // image_token_decoder: dh = d_img W, dW = d_img^T h
  DGS_TRY(dgrad(d_img, wT->dec_wT, ts.dh, d.Mt, D, d.Ndec, EPI_BIAS_BF16, nullptr, st));
  DGS_TRY(wgrad_tn(d_img, d.Ndec, ts.hdec, 3 * D, g->dec_w, d.Ndec, D, d.Mt, st));  // hi part of the [hi|lo|hi] operand
  DGS_TRY(ln_modulate_bwd(x_fin, ts.dh, w->dec_ln_w, md + D, d.mod_stride, B, N, G, T, D, 1e-5f, ts.dx, 0, dmd,
                          dmd + D, g->dec_ln_w, ts.ln_stats, st));
  if (G > 0) {  // upsampler (the free Gaussian tokens, rows 0..G of every sample)
    DGS_TRY(tiny_linear_bwd(ts.d_gs_tok, wT->ups_w, ws.hg, ts.dyb, g->ups_w, B * G, d.C, D, st));
    DGS_TRY(ln_modulate_bwd(x_fin, ts.dyb, w->ups_ln_w, mu + D, d.mod_stride, B, N, 0, G, D, 1e-5f, ts.dx, 0, dmu,
                            dmu + D, g->ups_ln_w, ts.ln_stats, st));
  }
  return DGS_OK;
}

// Backward of block l, the mirror of block_forward: reads the block's forward tensors from b and the gradient of its
// output from ts.dx, leaves the gradient of its input in ts.dx, accumulates d mod_l into dm and writes every parameter
// gradient of block l.  c: the conditioning (the adaLN linear's input).
int block_backward(const dgs_dit_weights* w, const dgs_dit_weights_t* wT, const dgs_dit_grads* g,
                   const dgs_dit_bwd_trace& tr, int l, const float* c, const float* m, float* dm, const DitDims& d,
                   const BlockBufs& b, const TrainState& ts, cudaStream_t st) {
  const int B = d.B, N = d.N, M = d.M, D = d.D, U = d.U, ms = d.mod_stride;
  const size_t LS = (size_t)g->layer_stride, MD = d.MD, MU = d.MU, f4 = sizeof(float), b2 = sizeof(__nv_bfloat16);
  // -- MLP branch: x_out = x_mid + gate_mlp * (fc2(gelu(fc1(h2))) )
  {
    ProfScope ps(st, PROF_DIT_BWD_ELEM);
    DGS_TRY(gate_bwd(ts.dx, b.fc2_out, m + 5 * D, ms, N, M, D, ts.dyb, nullptr, dm + 5 * D, g->fc2_b + l * LS, st));
  }
  DGS_TRY(trace_out(tr.d_fc2_out, l, ts.dyb, MD * b2, st));
  {
    ProfScope ps(st, PROF_DIT_BWD_WGRAD);
    DGS_TRY(wgrad_tn(ts.dyb, D, b.u, U, g->fc2_w + l * LS, D, U, M, st));
  }
  {
    ProfScope ps(st, PROF_DIT_BWD_DGRAD);
    DGS_TRY(dgrad(ts.dyb, (const __nv_bfloat16*)wT->fc2_wT + (size_t)l * D * U, ts.big0, M, U, D, EPI_DGELU_BF16,
                  b.u_pre, st));  // du_pre = (dy W2) * gelu'(u_pre)
  }
  DGS_TRY(trace_out(tr.du_pre, l, ts.big0, MU * b2, st));
  {
    ProfScope ps(st, PROF_DIT_BWD_ELEM);
    DGS_TRY(colsum_bf16(ts.big0, M, U, g->fc1_b + l * LS, st));
  }
  {
    ProfScope ps(st, PROF_DIT_BWD_WGRAD);
    DGS_TRY(wgrad_tn(ts.big0, U, b.h2, D, g->fc1_w + l * LS, U, D, M, st));
  }
  {
    ProfScope ps(st, PROF_DIT_BWD_DGRAD);
    DGS_TRY(dgrad(ts.big0, (const __nv_bfloat16*)wT->fc1_wT + (size_t)l * D * U, ts.dh, M, D, U, EPI_BIAS_BF16, nullptr,
                  st));
  }
  DGS_TRY(trace_out(tr.dh2, l, ts.dh, MD * b2, st));
  {
    ProfScope ps(st, PROF_DIT_BWD_ELEM);
    DGS_TRY(ln_modulate_bwd(b.x_mid, ts.dh, nullptr, m + 4 * D, ms, B, N, 0, N, D, 1e-6f, ts.dx, 1, dm + 3 * D,
                            dm + 4 * D, nullptr, ts.ln_stats, st));
    DGS_TRY(trace_out(tr.dx_mid, l, ts.dx, MD * f4, st));
    // -- attention branch: x_mid = x_in + gate_msa * proj(attn(qkv(h1)))
    DGS_TRY(gate_bwd(ts.dx, b.proj_out, m + 2 * D, ms, N, M, D, ts.dyb, nullptr, dm + 2 * D, g->proj_b + l * LS, st));
  }
  DGS_TRY(trace_out(tr.d_proj_out, l, ts.dyb, MD * b2, st));
  {
    ProfScope ps(st, PROF_DIT_BWD_WGRAD);
    DGS_TRY(wgrad_tn(ts.dyb, D, b.attn, D, g->proj_w + l * LS, D, D, M, st));
  }
  {
    ProfScope ps(st, PROF_DIT_BWD_DGRAD);
    DGS_TRY(dgrad(ts.dyb, (const __nv_bfloat16*)wT->proj_wT + (size_t)l * D * D, ts.dh, M, D, D, EPI_BIAS_BF16, nullptr,
                  st));
  }
  DGS_TRY(trace_out(tr.d_attn, l, ts.dh, MD * b2, st));
  {
    ProfScope ps(st, PROF_DIT_BWD_ATTN);
    DGS_TRY(attention_bwd(b.qkv, b.attn, ts.dh, b.lse, ts.dsum, ts.big0, B, N, w->heads, st));
  }
  DGS_TRY(trace_out(tr.dsum, l, ts.dsum, d.lse_n * f4, st));
  DGS_TRY(trace_out(tr.dqkv, l, ts.big0, 3 * MD * b2, st));
  {
    ProfScope ps(st, PROF_DIT_BWD_ELEM);
    DGS_TRY(colsum_bf16(ts.big0, M, 3 * D, g->qkv_b + l * LS, st));
  }
  {
    ProfScope ps(st, PROF_DIT_BWD_WGRAD);
    DGS_TRY(wgrad_tn(ts.big0, 3 * D, b.h1, D, g->qkv_w + l * LS, 3 * D, D, M, st));
  }
  {
    ProfScope ps(st, PROF_DIT_BWD_DGRAD);
    DGS_TRY(dgrad(ts.big0, (const __nv_bfloat16*)wT->qkv_wT + (size_t)l * 3 * D * D, ts.dh, M, D, 3 * D, EPI_BIAS_BF16,
                  nullptr, st));
  }
  DGS_TRY(trace_out(tr.dh1, l, ts.dh, MD * b2, st));
  {
    ProfScope ps(st, PROF_DIT_BWD_ELEM);
    DGS_TRY(ln_modulate_bwd(b.x_in, ts.dh, nullptr, m + D, ms, B, N, 0, N, D, 1e-6f, ts.dx, 1, dm, dm + D, nullptr,
                            ts.ln_stats, st));
    DGS_TRY(trace_out(tr.dx, l, ts.dx, MD * f4, st));
    // this block's adaLN linear (6w x w, a third of the block's parameters): d mod_l is complete now, so its weight /
    // bias gradient is produced HERE -- every gradient of block l is final at this point and its all-reduce can start
    // while blocks l-1 .. 0 are still being differentiated (block_done event); d silu(c) accumulates across blocks
    DGS_TRY(skinny_linear_bwd(c, w->adaln_w + (size_t)l * 6 * D * D, dm, ms, B, 6 * D, D, 1, g->adaln_w + l * LS,
                              g->adaln_b + l * LS, ts.dcond, ts.skb_part, st));
  }
  return DGS_OK;
}

// Backward of the input stage (LayerNorm(weight) -> [pos tokens | tokenizer GEMM]) from ts.dx, then of the
// conditioning (the heads' adaLN linears, the timestep MLP; the blocks' adaLN linears ran in block_backward).
int input_cond_backward(const dgs_dit_weights* w, const dgs_dit_grads* g, const DitDims& d, const DitWorkspace& ws,
                        const TrainState& ts, cudaStream_t st) {
  const int B = d.B, N = d.N, T = d.T, G = d.G, D = d.D, L = w->layers;
  DGS_TRY(ln_modulate_bwd(ts.x_pre, ts.dx, w->in_ln_w, nullptr, 0, B, N, 0, N, D, 1e-5f, ts.dx_pre, 0, nullptr, nullptr,
                          g->in_ln_w, ts.ln_stats, st));
  DGS_TRY(pos_embed_bwd(ts.dx_pre, g->pos_embed, B, G, N, D, st));
  DGS_TRY(transpose_to_bf16(ts.dx_pre, D, B, N, G, T, D, ts.bigT0, nullptr, st));                  // d tok^T [D, Mtp]
  DGS_TRY(transpose_to_bf16(ws.tokens, 3 * d.Kin, 1, d.Mt, 0, d.Mt, d.Kin, ts.bigT1, nullptr, st));  // hi part of the patches
  {
    GemmEpilogue ep;  // dW[D, Kin] = d tok^T [D, Mtp] x (patches^T [Kin, Mtp])^T   (K = padded row count, pads are zero)
    ep.out = g->tokenizer_w; ep.ldc = d.Kin;
    DGS_TRY(gemm_bf16(ts.bigT0, ts.bigT1, D, d.Kin, d.Mtp, EPI_F32, ep, st));
  }

  float* dsc = ts.dcond;                       // d silu(c), then dc
  float* dt1 = ts.dcond + (size_t)B * D;       // d temb1, then d pre1
  float* pre1 = ts.dcond + (size_t)2 * B * D;  // t0 pre-activation (recomputed)
  {  // the two heads' adaLN linears in one launch
    SkinnySegs segs;
    segs.seg_rows = 0; segs.n_seg = 0; segs.seg_stride = 0; segs.dW0 = nullptr; segs.db0 = nullptr;
    segs.tail_rows[0] = 2 * D; segs.tail_dW[0] = g->ups_adaln_w; segs.tail_db[0] = g->ups_adaln_b;
    segs.tail_rows[1] = 2 * D; segs.tail_dW[1] = g->dec_adaln_w; segs.tail_db[1] = g->dec_adaln_b;
    DGS_TRY(skinny_linear_bwd_segs(ws.c, w->adaln_w + (size_t)L * 6 * D * D, ts.dmod + (size_t)L * 6 * D, d.mod_stride, B,
                                   4 * D, D, 1, segs, dsc, ts.skb_part, st));
  }
  DGS_TRY(silu_bwd_inplace(dsc, ws.c, B * D, st));
  DGS_TRY(skinny_linear_bwd(ws.temb1, w->t2_w, dsc, D, B, D, D, 0, g->t2_w, g->t2_b, dt1, ts.skb_part, st));
  DGS_TRY(skinny_linear(ws.temb0, w->t0_w, w->t0_b, pre1, B, D, 256, 0, 0, st));
  DGS_TRY(silu_bwd_inplace(dt1, pre1, B * D, st));
  DGS_TRY(skinny_linear_bwd(ws.temb0, w->t0_w, dt1, D, B, D, 256, 0, g->t0_w, g->t0_b, nullptr, nullptr, st));
  return DGS_OK;
}

// the GemmEpilogue of the GEMM ABI calls (rows_per_sample <= 0: one sample)
int abi_epilogue(int epi, void* out, int ldc, const float* bias, const float* gate, int gate_stride, int rows_per_sample,
                 GemmEpilogue& ep) {
  DGS_REQUIRE(epi != EPI_GATE_RESID_F32 || (gate && rows_per_sample > 0), "gate epilogue needs gate and rows_per_sample");
  ep.out = out; ep.ldc = ldc; ep.bias = bias; ep.gate = gate; ep.gate_stride = gate_stride;
  ep.rows_per_sample = rows_per_sample > 0 ? rows_per_sample : 1;
  return DGS_OK;
}

}  // namespace

extern "C" {

size_t dgs_dit_workspace_bytes(const dgs_dit_weights* w, int B, int V, int H, int W) {
  if (check_dit(w, B, V, H, W)) return 0;
  return DitWorkspace(nullptr, DitDims(w, B, V, H, W)).bytes;
}

int dgs_dit_forward(const dgs_dit_weights* w, const dgs_dit_io* io, void* workspace, size_t workspace_bytes,
                    void* stream) {
  return dit_forward(w, nullptr, 0, io, workspace, workspace_bytes, (cudaStream_t)stream);
}

size_t dgs_dit_workspace_bytes_fp8(const dgs_dit_weights* w, int B, int V, int H, int W) {
  return dgs_dit_workspace_bytes_fp8_ex(w, B, V, H, W, 0);
}

size_t dgs_dit_workspace_bytes_fp8_ex(const dgs_dit_weights* w, int B, int V, int H, int W, int flags) {
  if (check_dit(w, B, V, H, W)) return 0;
  if (flags & ~DGS_FP8_ATTENTION) {
    set_error("unknown FP8 flags 0x%x", flags);
    return 0;
  }
  const DitWorkspace ws(nullptr, DitDims(w, B, V, H, W));
  return (flags & DGS_FP8_ATTENTION) ? ws.bytes_fp8_att : ws.bytes_fp8;
}

int dgs_dit_forward_fp8(const dgs_dit_weights* w, const dgs_dit_weights_fp8* w8, const dgs_dit_io* io, void* workspace,
                        size_t workspace_bytes, void* stream) {
  return dgs_dit_forward_fp8_ex(w, w8, io, 0, workspace, workspace_bytes, stream);
}

int dgs_dit_forward_fp8_ex(const dgs_dit_weights* w, const dgs_dit_weights_fp8* w8, const dgs_dit_io* io, int flags,
                           void* workspace, size_t workspace_bytes, void* stream) {
  DGS_REQUIRE(w8 && w8->qkv_w && w8->qkv_s && w8->fc1_w && w8->fc1_s && w8->fc2_w && w8->fc2_s, "NULL FP8 weight or scale");
  DGS_REQUIRE(io == nullptr || io->train_state == nullptr,
              "dgs_dit_forward_fp8 is inference only (io->train_state must be NULL; training runs bf16)");
  DGS_REQUIRE((flags & ~DGS_FP8_ATTENTION) == 0, "unknown FP8 flags 0x%x", flags);
  return dit_forward(w, w8, flags, io, workspace, workspace_bytes, (cudaStream_t)stream);
}

int dgs_attention_quantize_e4m3(const void* qkv, void* q8, void* k8, void* vt8, float* sq, float* sk, float* sv, int B,
                                int N, int heads, void* stream) {
  DGS_REQUIRE(qkv && q8 && k8 && vt8 && sq && sk && sv, "NULL pointer");
  return attention_quantize_e4m3(qkv, (uint8_t*)q8, (uint8_t*)k8, (uint8_t*)vt8, sq, sk, sv, B, N, heads,
                                 (cudaStream_t)stream);
}

int dgs_attention_fwd_fp8(const void* q8, const void* k8, const void* vt8, const float* sq, const float* sk,
                          const float* sv, void* out, int B, int N, int heads, void* stream) {
  DGS_REQUIRE(q8 && k8 && vt8 && sq && sk && sv && out, "NULL pointer");
  return attention_fwd_e4m3((const uint8_t*)q8, (const uint8_t*)k8, (const uint8_t*)vt8, sq, sk, sv, out, B, N, heads,
                            (cudaStream_t)stream);
}

int dgs_quantize_rows_e4m3(const float* x, int rows, int cols, void* q, float* scale, void* stream) {
  DGS_REQUIRE(x && q && scale, "NULL pointer");
  return quantize_rows_e4m3(x, rows, cols, (uint8_t*)q, scale, (cudaStream_t)stream);
}

int dgs_ln_modulate_fp8(const float* x, const float* shift, const float* scale, int mod_stride, void* q, float* q_scale,
                        int B, int rows, int width, float eps, void* stream) {
  DGS_REQUIRE(x && shift && scale && q && q_scale, "NULL pointer");
  return ln_forward(LN_E4M3, x, nullptr, shift, scale, mod_stride, q, q_scale, B, rows, 0, rows, width, eps,
                    (cudaStream_t)stream);
}

int dgs_gemm_fp8(const void* A, const float* sa, const void* W, const float* sw, const float* bias, const float* gate,
                 void* out, float* out_scale, int M, int N, int K, int epi, int ldc, int gate_stride,
                 int rows_per_sample, void* stream) {
  GemmEpilogue ep;
  DGS_TRY(abi_epilogue(epi, out, ldc, bias, gate, gate_stride, rows_per_sample, ep));
  return gemm_fp8(A, sa, W, sw, M, N, K, epi, ep, out_scale, (cudaStream_t)stream);
}

size_t dgs_dit_train_state_bytes(const dgs_dit_weights* w, int B, int V, int H, int W) {
  return dgs_dit_train_state_bytes_ex(w, B, V, H, W, DGS_TRAIN_STORE);
}

size_t dgs_dit_train_state_bytes_ex(const dgs_dit_weights* w, int B, int V, int H, int W, int train_mode) {
  if (check_dit(w, B, V, H, W) || check_train_mode(train_mode)) return 0;
  return TrainState(nullptr, w, DitDims(w, B, V, H, W), train_mode).bytes;
}

int dgs_dit_export_state(const dgs_dit_weights* w, int B, int V, int H, int W, int train_mode, const void* train_state,
                         int layer, float* x, float* x_mid, void* h1, void* qkv, void* attn, float* lse, void* proj_out,
                         void* h2, void* u_pre, void* u, void* fc2_out, void* stream) {
  DGS_TRY(check_dit(w, B, V, H, W));
  DGS_TRY(check_train_mode(train_mode));
  DGS_REQUIRE(train_state != nullptr, "train_state is NULL");
  const int L = w->layers;
  DGS_REQUIRE(layer >= 0 && layer <= L, "layer %d out of range [0, %d]", layer, L);
  const bool per_layer = x_mid || h1 || qkv || attn || lse || proj_out || h2 || u_pre || u || fc2_out;
  DGS_REQUIRE(!per_layer || train_mode == DGS_TRAIN_STORE,
              "per-layer tensors are kept only in DGS_TRAIN_STORE mode (recompute mode keeps the residual stream alone)");
  DGS_REQUIRE(!per_layer || layer < L, "per-layer tensors exist for layers [0, %d), not %d", L, layer);
  cudaStream_t st = (cudaStream_t)stream;
  const DitDims d(w, B, V, H, W);
  const TrainState ts(const_cast<void*>(train_state), w, d, train_mode);
  const BlockBufs b = block_bufs(train_mode == DGS_TRAIN_STORE ? PLAN_STORE : PLAN_REFILL, layer, d,
                                 DitWorkspace(nullptr, d), ts);  // the train-state plans read no workspace
  auto copy = [&](void* dst, const void* src, size_t bytes) -> int {
    if (dst) DGS_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st));
    return DGS_OK;
  };
  const size_t MD = d.MD, MU = d.MU, f4 = sizeof(float), b2 = sizeof(__nv_bfloat16);
  DGS_TRY(copy(x, b.x_in, MD * f4));
  if (!per_layer) return DGS_OK;
  DGS_TRY(copy(x_mid, b.x_mid, MD * f4));
  DGS_TRY(copy(h1, b.h1, MD * b2));
  DGS_TRY(copy(qkv, b.qkv, 3 * MD * b2));
  DGS_TRY(copy(attn, b.attn, MD * b2));
  DGS_TRY(copy(lse, b.lse, d.lse_n * f4));
  DGS_TRY(copy(proj_out, b.proj_out, MD * b2));
  DGS_TRY(copy(h2, b.h2, MD * b2));
  DGS_TRY(copy(u_pre, b.u_pre, MU * b2));
  DGS_TRY(copy(u, b.u, MU * b2));
  DGS_TRY(copy(fc2_out, b.fc2_out, MD * b2));
  return DGS_OK;
}

int dgs_dit_export_ends(const dgs_dit_weights* w, int B, int V, int H, int W, int train_mode, const void* train_state,
                        const void* workspace, size_t workspace_bytes, float* x_pre, float* c, float* mod, float* gs_tok,
                        float* img_gs, float* dx0, float* dx_pre, float* dmod, float* dc, float* d_gs_tok, void* stream) {
  DGS_TRY(check_dit(w, B, V, H, W));
  DGS_TRY(check_train_mode(train_mode));
  DGS_REQUIRE(train_state != nullptr, "train_state is NULL");
  const DitDims d(w, B, V, H, W);
  DitWorkspace ws(const_cast<void*>(workspace), d);
  DGS_REQUIRE(workspace && workspace_bytes >= ws.bytes, "workspace too small: %zu < %zu", workspace_bytes, ws.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t mod_n = (size_t)B * d.mod_stride;
  TrainState ts(const_cast<void*>(train_state), w, d, train_mode);
  auto copy = [&](void* dst, const void* src, size_t n) -> int {
    if (dst) DGS_CUDA_OK(cudaMemcpyAsync(dst, src, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return DGS_OK;
  };
  // none of these is written again after the pass that produces it: the forward's by the later forward stages, the
  // backward's by the later backward stages (dx is final once block 0 is differentiated, dcond slice 0 once silu_bwd ran)
  DGS_TRY(copy(x_pre, ts.x_pre, d.MD));
  DGS_TRY(copy(c, ws.c, (size_t)B * d.D));
  DGS_TRY(copy(mod, ws.mod, mod_n));
  DGS_TRY(copy(gs_tok, ws.gs_tok, (size_t)B * d.G * d.C));
  DGS_TRY(copy(img_gs, ws.img_gs, (size_t)d.Mt * d.Ndec));
  DGS_TRY(copy(dx0, ts.dx, d.MD));
  DGS_TRY(copy(dx_pre, ts.dx_pre, d.MD));
  DGS_TRY(copy(dmod, ts.dmod, mod_n));
  DGS_TRY(copy(dc, ts.dcond, (size_t)B * d.D));
  DGS_TRY(copy(d_gs_tok, ts.d_gs_tok, (size_t)B * d.G * d.C));
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
  const DitDims d(w, io->B, io->V, io->H, io->W);
  const int B = d.B, D = d.D, L = w->layers;
  DGS_REQUIRE(B <= 8, "dgs_dit_backward: per-call batch %d > 8 (split the batch)", B);
  DGS_REQUIRE(d.N >= 64, "dgs_dit_backward: needs at least 64 tokens per sample");
  DitWorkspace ws(workspace, d);
  DGS_REQUIRE(workspace && workspace_bytes >= ws.bytes, "workspace too small: %zu < %zu", workspace_bytes, ws.bytes);
  DGS_TRY(check_train_mode(io->train_mode));
  const bool recompute = io->train_mode == DGS_TRAIN_RECOMPUTE;
  TrainState ts(io->train_state, w, d, io->train_mode);
  void** done_ev = opts ? opts->block_done : nullptr;
  const dgs_dit_bwd_trace no_trace = {};
  const dgs_dit_bwd_trace& tr = opts && opts->trace ? *opts->trace : no_trace;

  // gradients accumulated by atomics start from zero; GEMM-produced ones are overwritten
  DGS_CUDA_OK(cudaMemsetAsync(ts.dmod, 0, (size_t)B * d.mod_stride * sizeof(float), st));
  DGS_CUDA_OK(cudaMemsetAsync(ts.dcond, 0, (size_t)3 * B * D * sizeof(float), st));
  const size_t LS = (size_t)g->layer_stride;
  for (int l = 0; l < L; l++) {
    DGS_CUDA_OK(cudaMemsetAsync(g->qkv_b + l * LS, 0, (size_t)3 * D * sizeof(float), st));
    DGS_CUDA_OK(cudaMemsetAsync(g->proj_b + l * LS, 0, (size_t)D * sizeof(float), st));
    DGS_CUDA_OK(cudaMemsetAsync(g->fc1_b + l * LS, 0, (size_t)d.U * sizeof(float), st));
    DGS_CUDA_OK(cudaMemsetAsync(g->fc2_b + l * LS, 0, (size_t)D * sizeof(float), st));
  }
  DGS_CUDA_OK(cudaMemsetAsync(g->in_ln_w, 0, D * sizeof(float), st));
  DGS_CUDA_OK(cudaMemsetAsync(g->ups_ln_w, 0, D * sizeof(float), st));
  DGS_CUDA_OK(cudaMemsetAsync(g->dec_ln_w, 0, D * sizeof(float), st));

  const BlockPlan plan = recompute ? PLAN_REFILL : PLAN_STORE;
  DGS_TRY(heads_backward(w, wT, io, dout, g, d, ws, ts, block_bufs(plan, L, d, ws, ts).x_in, st));
  DGS_TRY(trace_out(tr.dx, L, ts.dx, d.MD * sizeof(float), st));
  for (int l = L - 1; l >= 0; l--) {  // ---- L x DiTBlock, reversed ----
    const float* m = ws.mod + (size_t)l * 6 * D;
    float* dm = ts.dmod + (size_t)l * 6 * D;
    const BlockBufs b = block_bufs(plan, l, d, ws, ts);
    if (recompute) DGS_TRY(block_forward(w, nullptr, 0, l, m, d, b, st));  // refill the slot (denoiser.py:348-354)
    DGS_TRY(block_backward(w, wT, g, tr, l, ws.c, m, dm, d, b, ts, st));
    if (done_ev && done_ev[l]) DGS_CUDA_OK(cudaEventRecord((cudaEvent_t)done_ev[l], st));
  }
  ProfScope ps_in(st, PROF_DIT_BWD_ELEM);
  DGS_TRY(input_cond_backward(w, g, d, ws, ts, st));
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
  __nv_bfloat16* o = (__nv_bfloat16*)out;
  cudaStream_t st = (cudaStream_t)stream;
  return in_is_f32 ? transpose_to_bf16((const float*)in, C, 1, M, 0, M, C, o, colsum, st)
                   : transpose_to_bf16((const __nv_bfloat16*)in, C, 1, M, 0, M, C, o, colsum, st);
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
  GemmEpilogue ep;
  DGS_TRY(abi_epilogue(epi, out, ldc, bias, gate, gate_stride, rows_per_sample, ep));
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
  cudaStream_t st = (cudaStream_t)stream;
  return dh_is_f32 ? ln_modulate_bwd(x, (const float*)dh, ln_w, scale, mod_stride, B, rows, 0, rows, width, eps, dx,
                                     accumulate, dshift, dscale, dln_w, stats, st)
                   : ln_modulate_bwd(x, (const __nv_bfloat16*)dh, ln_w, scale, mod_stride, B, rows, 0, rows, width, eps,
                                     dx, accumulate, dshift, dscale, dln_w, stats, st);
}

int dgs_gate_bwd(const float* dx, const void* y, const float* gate, int gate_stride, int rows_per_sample, int M, int C,
                 void* dy, void* dyT, float* dgate, float* dbias, void* stream) {
  DGS_REQUIRE(dx && y && gate && dy && dgate, "NULL pointer");
  return gate_bwd(dx, (const __nv_bfloat16*)y, gate, gate_stride, rows_per_sample, M, C, (__nv_bfloat16*)dy,
                  (__nv_bfloat16*)dyT, dgate, dbias, (cudaStream_t)stream);
}

int dgs_gemm_bf16(const void* A, const void* Wt, const float* bias, const float* gate, void* out, int M, int N, int K,
                  int epi, int ldc, int gate_stride, int rows_per_sample, void* stream) {
  return dgs_gemm_bf16_ex(A, Wt, bias, gate, out, nullptr, nullptr, M, N, K, 0, 0, epi, ldc, gate_stride,
                          rows_per_sample, stream);
}

int dgs_attention_fwd(const void* qkv, void* out, int B, int N, int heads, void* stream) {
  DGS_REQUIRE(qkv && out, "NULL pointer");
  return attention_fwd(qkv, out, nullptr, B, N, heads, (cudaStream_t)stream);
}

int dgs_gaussians_epilogue(const float* gs_tok, const float* img_gs, const float* ray_o, const float* ray_d, float* xyz,
                           float* features, float* scaling, float* rotation, float* opacity, float* img_aligned_xyz,
                           int B, int G, int V, int H, int W, int patch, int sh_degree, int scene_depth, float near_,
                           float far_, void* stream) {
  DGS_REQUIRE((G == 0 || gs_tok) && img_gs && ray_o && ray_d && xyz && features && scaling && rotation && opacity,
              "NULL pointer");
  DGS_REQUIRE(B > 0 && G >= 0 && V > 0 && patch > 0 && H % patch == 0 && W % patch == 0, "bad shape");
  GsOut go;
  go.xyz = xyz; go.features = features; go.scaling = scaling; go.rotation = rotation; go.opacity = opacity;
  go.img_aligned_xyz = img_aligned_xyz;
  return gaussians_epilogue(gs_tok, img_gs, ray_o, ray_d, go, B, G, V, H, W, patch, sh_degree, scene_depth, near_, far_,
                            (cudaStream_t)stream);
}

int dgs_gaussians_epilogue_bwd(const float* gs_tok, const float* img_gs, const float* ray_d, const float* d_xyz,
                               const float* d_features, const float* d_scaling, const float* d_rotation,
                               const float* d_opacity, float* d_gs_tok, void* d_img_gs, int B, int G, int V, int H,
                               int W, int patch, int sh_degree, int scene_depth, float near_, float far_, void* stream) {
  DGS_REQUIRE((G == 0 || (gs_tok && d_gs_tok)) && img_gs && ray_d && d_xyz && d_features && d_scaling && d_rotation &&
                  d_opacity && d_img_gs, "NULL pointer");
  DGS_REQUIRE(B > 0 && G >= 0 && V > 0 && patch > 0 && H % patch == 0 && W % patch == 0, "bad shape");
  return gaussians_epilogue_bwd(gs_tok, img_gs, ray_d, d_xyz, d_features, d_scaling, d_rotation, d_opacity, nullptr,
                                d_gs_tok, (__nv_bfloat16*)d_img_gs, B, G, V, H, W, patch, sh_degree, scene_depth, near_,
                                far_, (cudaStream_t)stream);
}

int dgs_ln_modulate(const float* x, const float* ln_w, const float* shift, const float* scale, int mod_stride, void* h,
                    int B, int rows, int width, float eps, void* stream) {
  DGS_REQUIRE(x && shift && scale && h, "NULL pointer");
  return ln_forward(LN_BF16, x, ln_w, shift, scale, mod_stride, h, nullptr, B, rows, 0, rows, width, eps,
                    (cudaStream_t)stream);
}

}  // extern "C"
