/*
 * dgs_b200.h -- C ABI of libdgs_b200.so: the H100-native (sm_90a) hot path of Open-DiffusionGS.
 *
 * Plain C: raw DEVICE pointers, sizes, a cudaStream_t passed as void*.  No torch types, no C++
 * exceptions cross this boundary; every entry point returns a status code and
 * dgs_last_error() gives the message.  Each entry point cites the reference interface it
 * replaces (paths relative to the reference repo; DGR = submodules/diff-gaussian-rasterization).
 *
 * All kernels are enqueued on the caller's stream.  Only the rasterizer forward synchronises
 * that stream once (to read the instance count R that sizes the binning arena), exactly like
 * the reference's cudaMemcpy at DGR/cuda_rasterizer/rasterizer_impl.cu:281 -- but ONCE PER BATCH
 * of (sample, view) pairs instead of once per view.
 */
#ifndef DGS_B200_H_INCLUDED
#define DGS_B200_H_INCLUDED

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DGS_VERSION 100

typedef enum {
  DGS_OK = 0,
  DGS_ERR_INVALID_ARGUMENT = 1, /* replaces AT_ERROR / std::runtime_error, rasterize_points.cu:57-59 */
  DGS_ERR_CUDA = 2,             /* replaces CHECK_CUDA's throw, auxiliary.h:166-173 */
  DGS_ERR_ALLOC = 3,            /* allocator callback returned NULL */
  DGS_ERR_OVERFLOW = 4          /* instance count does not fit 32 bits */
} dgs_status;

/* Arena allocator callback: must return DEVICE memory of at least `bytes` bytes (256-B aligned)
 * that stays valid until the matching backward has run.  Replaces the reference's
 * std::function<char*(size_t)> resize callbacks (DGR/cuda_rasterizer/rasterizer.h:31-34,
 * DGR/rasterize_points.cu:27-33). */
typedef void* (*dgs_alloc_fn)(size_t bytes, void* user);

int dgs_version(void);
const char* dgs_last_error(void);
/* Kernels of this library launched so far by the calling process (for bench.py's `gpu_launches`). */
unsigned long long dgs_kernel_launch_count(void);
/* Optional per-kernel-family device timing: when enabled, every entry point records CUDA events on the
 * caller's stream around each kernel family it launches.  dgs_profile_read() waits for the recorded spans,
 * writes the summed milliseconds and span counts per family (order: raster project, scan, emit_keys, sort,
 * tile_ranges, blend_fwd, blend_bwd, geometry_bwd; dit input, conditioning, ln_modulate, gemm_qkv, attention,
 * gemm_proj, gemm_fc1, gemm_fc2, heads), clears the record and returns the number of families. */
int dgs_profile_enable(int on);
int dgs_profile_read(float* ms_sum, int* span_count, int n_families);

/* ------------------------------------------------------------------------------------------------
 * B1a. Single-view rasterizer: what `_C.rasterize_gaussians`, `_C.rasterize_gaussians_backward`
 * and `_C.mark_visible` bind (DGR/ext.cpp:15-19; DGR/rasterize_points.h:18-66;
 * CudaRasterizer::Rasterizer::{forward,backward,markVisible}, DGR/cuda_rasterizer/rasterizer.h:24-85).
 * Inputs are the ACTIVATED tensors the reference binding receives (post-exp scales, normalised
 * quaternions, post-sigmoid opacities).  NULL == "not provided" (the reference's empty tensor).
 * viewmatrix / projmatrix are the 16 floats of the reference's transposed matrices
 * (element [4*c + r] = row r, column c; DGR/cuda_rasterizer/auxiliary.h:58-77).
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int P;            /* number of Gaussians                     */
  int D;            /* active SH degree (0..3)                 */
  int M;            /* SH coefficients per Gaussian in `shs`   */
  int W, H;         /* image size                              */
  const float* background;     /* [3]      */
  const float* means3D;        /* [P,3]    */
  const float* shs;            /* [P,M,3] or NULL */
  const float* colors_precomp; /* [P,3]   or NULL */
  const float* opacities;      /* [P]      */
  const float* scales;         /* [P,3]   or NULL */
  const float* rotations;      /* [P,4]   or NULL */
  const float* cov3D_precomp;  /* [P,6]   or NULL */
  const float* viewmatrix;     /* [16]     */
  const float* projmatrix;     /* [16]     */
  const float* campos;         /* [3]      */
  float scale_modifier;
  float tan_fovx, tan_fovy;
  int prefiltered;  /* accepted for signature parity; culled points are skipped either way */
  int debug;        /* non-zero: synchronise and check for CUDA errors after every stage */
} dgs_raster_args;

/* Sizes of the three opaque arenas (geometry: per Gaussian, binning: per instance, image: per pixel)
 * -- the equivalents of required<GeometryState/BinningState/ImageState>() (rasterizer_impl.h:67-73). */
size_t dgs_raster_geom_bytes(int n_views, int P);
size_t dgs_raster_binning_bytes(long long R);
size_t dgs_raster_image_bytes(int n_views, int W, int H);

/* Forward (rasterizer_impl.cu:198-336).  out_color [3,H,W] and radii [P] are caller-allocated;
 * the three arenas are obtained through the callbacks and must be handed back to the backward.
 * *num_rendered receives R (the reference's return value). */
int dgs_raster_forward(const dgs_raster_args* args, dgs_alloc_fn geom_alloc, void* geom_user,
                       dgs_alloc_fn binning_alloc, void* binning_user, dgs_alloc_fn image_alloc,
                       void* image_user, float* out_color, int* radii, int* num_rendered,
                       void* stream);

/* Backward (rasterizer_impl.cu:340-434).  The nine gradient buffers are caller-allocated and
 * ZERO-initialised (rasterize_points.cu:151-159): dL_dmean2D [P,3], dL_dconic [P,2,2],
 * dL_dopacity [P,1], dL_dcolor [P,3], dL_dmean3D [P,3], dL_dcov3D [P,6], dL_dsh [P,M,3],
 * dL_dscale [P,3], dL_drot [P,4]. */
int dgs_raster_backward(const dgs_raster_args* args, int R, const int* radii, const void* geom_buffer,
                        const void* binning_buffer, const void* image_buffer, const float* dL_dpix,
                        float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                        float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale,
                        float* dL_drot, void* stream);

/* markVisible (rasterizer_impl.cu:54-66,141-153): present[i] = view-space z > 0.2 */
int dgs_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                     uint8_t* present, void* stream);

/* ------------------------------------------------------------------------------------------------
 * B1b. Batched renderer: one call for ALL (sample, view) pairs of `Renderer.forward`
 * (diffusionGS/models/gsrenderer/renderer.py:34-92) = DeferredGaussianRender.forward/backward
 * (gs_core.py:949-1060) + render_opencv_cam (874-945) + Camera (277-316) + the GaussianModel
 * activations (330-334,545-570), fused.  Inputs are the RAW per-sample parameter tensors
 * (fp32, contiguous): xyz [B,P,3], features [B,P,M,3], scaling [B,P,3], rotation [B,P,4],
 * opacity [B,P,1], C2W [B,V,4,4] row-major, fxfycxcy [B,V,4].  Output [B,V,3,H,W].
 * The forward keeps its sorted tile lists in the arenas; the backward re-uses them (no re-render,
 * unlike gs_core.py:1041-1056) and returns gradients w.r.t. the raw tensors, summed over views.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int B, V, P, M, D, W, H;
  const float* xyz;
  const float* features;
  const float* scaling;
  const float* rotation;
  const float* opacity;
  const float* c2w;
  const float* fxfycxcy;
  float scale_modifier; /* 1.0 when the reference passes scaling_modifier=None */
  float bg[3];          /* (1,1,1) in render_opencv_cam, gs_core.py:880 */
  int debug;
  int near_log2;        /* 0: one binning pass over all instances.  k < 0: adaptive (1/8, or 1/16 when those near lists still
                           average >= 2048 entries per tile).  k > 0: two-phase binning -- phase A bins and blends
                           only the nearest P >> k Gaussians of every view; if every pixel saturates there (dense scenes)
                           the remaining instances are never emitted or sorted, otherwise phase B continues from the
                           saved per-pixel state.  Same images, final_T, n_contrib and gradients either way. */
} dgs_render_batch_args;

int dgs_render_batch_forward(const dgs_render_batch_args* args, dgs_alloc_fn geom_alloc, void* geom_user,
                             dgs_alloc_fn binning_alloc, void* binning_user, dgs_alloc_fn image_alloc,
                             void* image_user, float* out_images, long long* num_rendered,
                             long long* chunk_instances /* out [2]: instances binned in phase A / phase B */,
                             void* stream);

/* d_* are caller-allocated, same shapes as the inputs; they are fully overwritten.  scratch_alloc
 * provides the per-(view, Gaussian) screen-space gradient records (44 B each), free after the call. */
int dgs_render_batch_backward(const dgs_render_batch_args* args, long long R,
                              const long long* chunk_instances /* [2] from the forward */, const void* geom_buffer,
                              const void* binning_buffer /* 1st binning_alloc result */,
                              const void* binning_buffer_b /* 2nd (phase B) or NULL */, const void* image_buffer,
                              const float* dL_dimages, float* d_xyz, float* d_features,
                              float* d_scaling, float* d_rotation, float* d_opacity,
                              dgs_alloc_fn scratch_alloc, void* scratch_user, void* stream);

/* The same pair with the image-space MSE of the training loss fused in (LossComputer.forward's l2 term,
 * diffusionGS/utils/losses.py:261-284: l2_loss[b] = mean over (v,3,h,w) of (rendering - target)^2, later averaged over b and
 * weighted by lambda_diffusion, diffusion_gs_system.py:94-124).  Forward: the blend kernel adds sum (render - target)^2 of
 * sample b into loss_sum[b] (caller-zeroed, fp64) while the pixel is in registers.  Backward: the blend-backward kernel forms
 * dL/dpix = dL_dimages (may be NULL) + coef[b] * (render - target) itself, with coef[b] = dL/dl2_loss[b] * 2 / (V*3*H*W)
 * computed by the caller on the device -- no per-element loss or gradient image exists.  mse == NULL: the plain pair. */
typedef struct {
  const float* target;   /* [B,V,target_channels,H,W] fp32 in (0,1)                                       */
  int target_channels;   /* 3, or 4 = rgb + mask (the mask plane is skipped, losses.py:274-276)           */
  double* loss_sum;      /* forward:  out [B]                                                              */
  const float* coef;     /* backward: in  [B] (device)                                                     */
  const float* images;   /* backward: in  the forward's out_images                                         */
} dgs_render_mse;
int dgs_render_batch_forward_mse(const dgs_render_batch_args* args, dgs_alloc_fn geom_alloc, void* geom_user,
                                 dgs_alloc_fn binning_alloc, void* binning_user, dgs_alloc_fn image_alloc,
                                 void* image_user, float* out_images, long long* num_rendered, long long* chunk_instances,
                                 const dgs_render_mse* mse, void* stream);
int dgs_render_batch_backward_mse(const dgs_render_batch_args* args, long long R, const long long* chunk_instances,
                                  const void* geom_buffer, const void* binning_buffer, const void* binning_buffer_b,
                                  const void* image_buffer, const float* dL_dimages, const dgs_render_mse* mse,
                                  float* d_xyz, float* d_features, float* d_scaling, float* d_rotation, float* d_opacity,
                                  dgs_alloc_fn scratch_alloc, void* scratch_user, void* stream);

/* Introspection used by the parity tests: copies of per-(view, Gaussian) / per-pixel forward state
 * out of the opaque arenas into caller DEVICE buffers (any may be NULL):
 * xy [N,2], depth [N], conic_opacity [N,4], rgb [N,3], tiles_touched [N] (N = n_views*P),
 * point_list [R], ranges [n_views*tiles,2], final_T / n_contrib [n_views*H*W].  point_list / ranges describe a
 * single-pass binning (near_log2 == 0); the per-pixel and per-Gaussian outputs are valid in both modes. */
int dgs_raster_export_state(int n_views, int P, int W, int H, long long R, const void* geom_buffer,
                            const void* binning_buffer, const void* image_buffer, float* xy,
                            float* depth, float* conic_opacity, float* rgb, uint32_t* tiles_touched,
                            uint32_t* point_list, uint32_t* ranges, float* final_T,
                            uint32_t* n_contrib, void* stream);

/* ------------------------------------------------------------------------------------------------
 * B2. DiT denoiser forward: DGSDenoiser.image_to_gaussians
 * (diffusionGS/models/denoiser/denoiser.py:306-416; scene twin denoiser_scene.py:314-429), i.e.
 * posed-image patchify + tokenizer -> +2 learned tokens -> LayerNorm -> L x DiTBlock
 * (utils_transformer.py:246-290 around timm Attention/Mlp) -> GaussiansUpsampler / ImageTokenDecoder
 * heads -> to_gs + pixel alignment.  GEMMs and attention run on wgmma (bf16 in, fp32 accumulate),
 * the residual stream, LayerNorm statistics and softmax stay fp32.
 * Weights: GEMM matrices are bf16 row-major [out, in] (nn.Linear layout), per-layer tensors stacked
 * along a leading L axis; vectors fp32.  state_dict key -> field mapping is in dgs_b200/denoiser.py.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int width, heads, layers, patch, n_gaussians, mlp_hidden; /* 1024, 16, 24, 8, 2, 4096 */
  const void* tokenizer_w;  /* image_tokenizer.1.weight, split-bf16 [width, 3*patch*patch*9] = [hi|hi|lo] */
  const float* pos_embed;   /* gaussians_pos_embedding             fp32 [n_gaussians, width]          */
  const float* in_ln_w;     /* transformer_input_layernorm.weight  fp32 [width]                       */
  const float* t0_w; const float* t0_b; /* t_embedder.mlp.0  fp32 [width,256], fp32 [width]          */
  const float* t2_w; const float* t2_b; /* t_embedder.mlp.2  fp32 [width,width], fp32 [width]        */
  const float* adaln_w;     /* all adaLN_modulation.1.weight stacked: L x [6*width] rows, then upsampler
                               [2*width], then image_token_decoder [2*width]; fp32 [.., width]        */
  const float* adaln_b;     /* same stacking, fp32                                                    */
  const void* qkv_w;  const float* qkv_b;   /* transformer.{i}.attn.qkv   bf16 [L,3w,w], fp32 [L,3w] */
  const void* proj_w; const float* proj_b;  /* transformer.{i}.attn.proj  bf16 [L,w,w],  fp32 [L,w]  */
  const void* fc1_w;  const float* fc1_b;   /* transformer.{i}.mlp.fc1    bf16 [L,4w,w], fp32 [L,4w] */
  const void* fc2_w;  const float* fc2_b;   /* transformer.{i}.mlp.fc2    bf16 [L,w,4w], fp32 [L,w]  */
  const float* ups_ln_w; const void* ups_w; /* upsampler.layernorm.weight fp32 [w]; upsampler.linear.weight split-bf16 [14,3w] */
  const float* dec_ln_w; const void* dec_w; /* image_token_decoder.*: fp32 [w]; split-bf16 [patch*patch*14, 3w]
     "split-bf16 [n, 3k] = [hi|hi|lo]": hi = bf16(W), lo = bf16(W - hi); paired with activations laid out
     [hi|lo|hi] the bf16 MMA then yields x_hi W_hi + x_lo W_hi + x_hi W_lo (fp32-accurate) -- used for the two
     small GEMMs at the ends of the network whose rounding would otherwise dominate the output error. */
} dgs_dit_weights;

typedef struct {
  int B, V, H, W;
  int plucker_mode;          /* 0 = 'relative_plk' (object model), 1 = 'plk' (scene model)            */
  int scene_depth;           /* 0: depth=(2s-1)*1.8 + (-o.d) (object model, 'relative_plk'); 1: depth=s*(far-near)+near
                                (scene model); 2: depth=s (object model with ray_pe_type 'plk', denoiser.py:381-388) */
  float range_near, range_far;
  const float* images;       /* [B,V,3,H,W] fp32 (view 0 clean, others noised)                        */
  const float* ray_o;        /* [B,V,3,H,W]                                                           */
  const float* ray_d;        /* [B,V,3,H,W]                                                           */
  const float* t;            /* [B] timesteps as fp32                                                 */
  float* xyz;                /* out [B,P,3],  P = n_gaussians + V*H*W                                 */
  float* features;           /* out [B,P,1,3]                                                         */
  float* scaling;            /* out [B,P,3]                                                           */
  float* rotation;           /* out [B,P,4]                                                           */
  float* opacity;            /* out [B,P,1]                                                           */
  float* img_aligned_xyz;    /* out [B,V,3,H,W] or NULL                                               */
  float* tokens_out;         /* optional debug out: final residual stream [B,N,width] fp32, or NULL   */
  void* train_state;         /* NULL: inference.  Else a caller buffer of dgs_dit_train_state_bytes[_ex](): what the
                                backward needs from the forward lives there; it must stay untouched, together with
                                `workspace`, until dgs_dit_backward has run.                              */
  int train_mode;            /* DGS_TRAIN_STORE (0): every activation is kept (4 GB per sample at N=4098; forward + 2x
                                backward FLOPs).  DGS_TRAIN_RECOMPUTE (1): only the fp32 residual stream entering each
                                block is kept (0.6 GB per sample) and the backward re-runs each block's forward before
                                differentiating it -- the reference's torch.utils.checkpoint around every block
                                (denoiser.py:348-354; grad_checkpoint_every = 1), for the yaml batch sizes.           */
} dgs_dit_io;
#define DGS_TRAIN_STORE 0
#define DGS_TRAIN_RECOMPUTE 1

size_t dgs_dit_workspace_bytes(const dgs_dit_weights* w, int B, int V, int H, int W);
int dgs_dit_forward(const dgs_dit_weights* w, const dgs_dit_io* io, void* workspace, size_t workspace_bytes,
                    void* stream);

/* ---- opt-in FP8 (e4m3) inference: the qkv, mlp.fc1 and mlp.fc2 GEMMs of every block on e4m3 operands ----
 * Weights: e4m3 [L, N, K] row-major with one fp32 scale per output channel, [L, N].  Activations: e4m3 [M, K] with
 * one fp32 scale per row and 128-column group, stored transposed as [K/128][round_up(M, 4)].  Every scale is a power
 * of two, 2^ceil(log2(amax / 448)) (1 for an all-zero group), so quantizing is an exact scaling and one
 * round-to-nearest-even: q = e4m3(x / s).  A GEMM computes sw[n] * sum over k-blocks of sa[kb][m] * (qa qw^T)_kb, then
 * the bf16 path's epilogue.  Everything else (input stage, conditioning, attention, attn.proj, heads) is the bf16 path;
 * there is no FP8 training. */
typedef struct {
  const void* qkv_w; const float* qkv_s;  /* e4m3 [L, 3w, w], fp32 [L, 3w] */
  const void* fc1_w; const float* fc1_s;  /* e4m3 [L, 4w, w], fp32 [L, 4w] */
  const void* fc2_w; const float* fc2_s;  /* e4m3 [L, w, 4w], fp32 [L, w]  */
} dgs_dit_weights_fp8;
/* dgs_dit_workspace_bytes plus the activation scale arrays */
size_t dgs_dit_workspace_bytes_fp8(const dgs_dit_weights* w, int B, int V, int H, int W);
/* dgs_dit_forward with the three GEMMs above on FP8 (w8); w supplies every other weight.  Inference only: a non-NULL
 * io->train_state is DGS_ERR_INVALID_ARGUMENT. */
int dgs_dit_forward_fp8(const dgs_dit_weights* w, const dgs_dit_weights_fp8* w8, const dgs_dit_io* io, void* workspace,
                        size_t workspace_bytes, void* stream);
/* Building blocks of the FP8 forward (the same kernels it launches), for the unit tests and weight packing:
 * q [rows, cols] e4m3, scale [rows] = x [rows, cols] fp32 with one power-of-two scale per row (the weight format). */
int dgs_quantize_rows_e4m3(const float* x, int rows, int cols, void* q, float* scale, void* stream);
/* dgs_ln_modulate (no LayerNorm weight) -> q e4m3 [B*rows, width] and q_scale [width/128][round_up(B*rows, 4)] */
int dgs_ln_modulate_fp8(const float* x, const float* shift, const float* scale, int mod_stride, void* q, float* q_scale,
                        int B, int rows, int width, float eps, void* stream);
/* FP8 GEMM, A e4m3 [M, K] with group scales sa, W e4m3 [N, K] with channel scales sw; K % 128 == 0, N % 128 == 0,
 * 16-byte aligned pointers.  epi: 0 = (acc + bias) -> bf16; 2 = out(fp32) += gate[row / rows_per_sample] * (acc + bias),
 * in place; 3 = (acc + bias) -> fp32; 6 = GELU(tanh)(acc + bias) -> e4m3 out [M, ldc] with its group scales out_scale
 * [N/128][round_up(M, 4)].  ldc: output row stride in elements. */
int dgs_gemm_fp8(const void* A, const float* sa, const void* W, const float* sw, const float* bias, const float* gate,
                 void* out, float* out_scale, int M, int N, int K, int epi, int ldc, int gate_stride,
                 int rows_per_sample, void* stream);

/* ---- training: backward of dgs_dit_forward (what torch autograd derives for denoiser.py:306-416 in the reference) ----
 * dgrad GEMMs read TRANSPOSED bf16 copies of the block weights (W^T, [in, out] row-major) so that every GEMM of the
 * backward runs on the same K-major wgmma kernel as the forward; the caller refreshes them after each optimizer step
 * (dgs_transpose_bf16).  Gradients are fp32, in the state_dict layout of the fp32 master parameters. */
typedef struct {
  const void* qkv_wT;   /* bf16 [L, w, 3w]   */
  const void* proj_wT;  /* bf16 [L, w, w]    */
  const void* fc1_wT;   /* bf16 [L, w, 4w]   */
  const void* fc2_wT;   /* bf16 [L, 4w, w]   */
  const void* dec_wT;   /* bf16 [w, patch*patch*14]  (image_token_decoder.linear.weight^T)             */
  const float* ups_w;   /* fp32 [14, w]      (upsampler.linear.weight, master copy)                    */
} dgs_dit_weights_t;

typedef struct {  /* all fp32, OVERWRITTEN by dgs_dit_backward */
  float* tokenizer_w;  /* [w, patch*patch*9] */
  float* pos_embed;    /* [n_gaussians, w]   */
  float* in_ln_w;      /* [w]                */
  float* t0_w; float* t0_b; float* t2_w; float* t2_b;
  /* per-block tensors: the pointer addresses block 0; block l lives layer_stride floats further.  This is the layout
     of a flat gradient arena in module.parameters() order (dgs_b200/dist.py GradArena: one contiguous bucket per
     block, all-reduced in reverse order as the backward finishes them); a stacked [L, ...] layout is not expressible */
  long long layer_stride;
  float* qkv_w; float* qkv_b; float* proj_w; float* proj_b; float* fc1_w; float* fc1_b; float* fc2_w; float* fc2_b;
  float* adaln_w; float* adaln_b;          /* block 0: [6w, w], [6w] */
  float* ups_ln_w; float* ups_w;           /* [w], [14, w]               */
  float* ups_adaln_w; float* ups_adaln_b;  /* [2w, w], [2w]              */
  float* dec_ln_w; float* dec_w;           /* [w], [patch*patch*14, w]   */
  float* dec_adaln_w; float* dec_adaln_b;  /* [2w, w], [2w]              */
} dgs_dit_grads;

typedef struct {  /* gradients w.r.t. the outputs of dgs_dit_forward (what dgs_render_batch_backward returns) */
  const float* d_xyz; const float* d_features; const float* d_scaling; const float* d_rotation; const float* d_opacity;
} dgs_dit_out_grads;

size_t dgs_dit_train_state_bytes(const dgs_dit_weights* w, int B, int V, int H, int W); /* DGS_TRAIN_STORE */
size_t dgs_dit_train_state_bytes_ex(const dgs_dit_weights* w, int B, int V, int H, int W, int train_mode);
/* io / workspace / io->train_state: exactly what the matching dgs_dit_forward call was given. */
int dgs_dit_backward(const dgs_dit_weights* w, const dgs_dit_weights_t* wT, const dgs_dit_io* io,
                     const dgs_dit_out_grads* dout, const dgs_dit_grads* grads, void* workspace, size_t workspace_bytes,
                     void* stream);
/* Same, with a completion hook for the data-parallel gradient exchange (what torch DDP's autograd hooks give the
 * reference, diffusionGS_rel.yaml:80): block_done[l], l = layers-1 .. 0, is recorded on `stream` as soon as EVERY
 * parameter gradient of transformer block l is final (the blocks are differentiated in reverse order), block_done[layers]
 * when the remaining gradients (tokenizer, embedder, heads) are.  A side stream that waits on block_done[l]
 * (dgs_stream_wait_event) can all-reduce block l's contiguous bucket while blocks l-1 .. 0 are still running.
 * Entries may be NULL; events come from dgs_event_create.
 *
 * trace (NULL: none) reads out the backward's per-block gradients for the per-block parity tests: each field is NULL or
 * the DEVICE base of a caller buffer stacked over the layers (slice l of a [layers, ...] field belongs to block l), which
 * the backward fills by cudaMemcpyAsync on `stream` at the point where that tensor is final.  M = B*N rows,
 * Np = round_up(N, 128).  The names are the gradients of the tensors dgs_dit_export_state reads out:
 *   dx [layers + 1, M, width] fp32: the gradient of the residual stream; slice layers right after the heads, slice l
 *   once block l is differentiated (the gradient of the stream entering it);
 *   dx_mid [layers, M, width] fp32: of x_mid (after the MLP branch's LayerNorm + modulate backward);
 *   d_fc2_out, d_proj_out [layers, M, width] bf16: gate * dx of the two branches (the pre-gate branch outputs);
 *   du_pre [layers, M, mlp_hidden] bf16: of u_pre (the fc2 dgrad times gelu'(u_pre));
 *   dh2, dh1 [layers, M, width] bf16: of h2 / h1 (the fc1 / qkv dgrad);
 *   d_attn [layers, M, width] bf16: of attn (the attn.proj dgrad);
 *   dsum [layers, B, heads, Np] fp32: rowsum(attn * d_attn) per head (pad entries 0);  dqkv [layers, M, 3*width] bf16.
 * Kernels and results do not depend on the trace. */
typedef struct {
  float* dx; float* dx_mid;
  void* d_fc2_out; void* du_pre; void* dh2; void* d_proj_out; void* d_attn;
  float* dsum; void* dqkv; void* dh1;
} dgs_dit_bwd_trace;
typedef struct {
  void** block_done;                /* NULL or [layers + 1] events */
  const dgs_dit_bwd_trace* trace;   /* NULL or the per-block read-out above */
} dgs_dit_bwd_opts;
int dgs_dit_backward_ex(const dgs_dit_weights* w, const dgs_dit_weights_t* wT, const dgs_dit_io* io,
                        const dgs_dit_out_grads* dout, const dgs_dit_grads* grads, const dgs_dit_bwd_opts* opts,
                        void* workspace, size_t workspace_bytes, void* stream);
/* Introspection used by the per-block parity tests: copies of what a training forward (dgs_dit_forward with
 * io->train_state) left in the train state for block `layer` into caller DEVICE buffers (any may be NULL).
 * M = B*N rows, Np = round_up(N, 128):
 *   x [M, width] fp32: the residual stream entering block `layer` (0 <= layer <= layers; layer == layers is the final
 *   stream), in both modes.  Recompute mode takes it around the inference block (in-place residual), store mode around
 *   the training block (separate residual buffers).
 *   Store mode only, 0 <= layer < layers: x_mid [M, width] fp32 (after the attention branch), h1 / h2 [M, width] bf16
 *   (LayerNorm + modulate outputs), qkv [M, 3*width] bf16, attn [M, width] bf16, lse [B, heads, Np] fp32 (log2-domain
 *   log-sum-exp of the scaled scores; pad entries undefined), proj_out / fc2_out [M, width] bf16 (branch outputs + bias,
 *   before the gate), u_pre / u [M, mlp_hidden] bf16 (fc1 + bias, and its GELU).
 * An out-of-range layer, or a per-layer tensor requested in recompute mode, is DGS_ERR_INVALID_ARGUMENT. */
int dgs_dit_export_state(const dgs_dit_weights* w, int B, int V, int H, int W, int train_mode, const void* train_state,
                         int layer, float* x, float* x_mid, void* h1, void* qkv, void* attn, float* lse, void* proj_out,
                         void* h2, void* u_pre, void* u, void* fc2_out, void* stream);
/* Introspection used by the end-stage parity tests: copies of the tensors on either side of the blocks into caller
 * DEVICE buffers (any may be NULL), all fp32.  M = B*N rows, T image tokens per sample, G = n_gaussians.
 * Left by the last training forward (dgs_dit_forward with io->train_state; c, mod, gs_tok and img_gs by the last
 * forward that used `workspace`, training or not):
 *   x_pre [M, width]: the assembled tokens [pos embedding | tokenizer output] before the input LayerNorm;
 *   c [B, width]: the conditioning t_embedder(t), before the adaLN SiLU;
 *   mod [B, layers*6*width + 4*width]: the adaLN table (block l at l*6*width; upsampler then decoder shift | scale);
 *   gs_tok [B*G, 14] and img_gs [B*T, patch*patch*14]: the raw head outputs, before the Gaussian epilogue.
 * Left by dgs_dit_backward(_ex) on the same train state and workspace (undefined before a backward):
 *   dx0 [M, width]: the gradient of the residual stream entering block 0 (the input LayerNorm's output);
 *   dx_pre [M, width]: the gradient of x_pre;
 *   dmod [B, layers*6*width + 4*width]: the gradient of the adaLN table;
 *   dc [B, width]: the gradient of c (after the SiLU backward);
 *   d_gs_tok [B*G, 14]: the gradient of gs_tok.
 * A NULL train state, a bad mode or a workspace smaller than dgs_dit_workspace_bytes is DGS_ERR_INVALID_ARGUMENT. */
int dgs_dit_export_ends(const dgs_dit_weights* w, int B, int V, int H, int W, int train_mode, const void* train_state,
                        const void* workspace, size_t workspace_bytes, float* x_pre, float* c, float* mod, float* gs_tok,
                        float* img_gs, float* dx0, float* dx_pre, float* dmod, float* dc, float* d_gs_tok, void* stream);
int dgs_event_create(void** event);                 /* cudaEventCreateWithFlags(DisableTiming) */
int dgs_event_destroy(void* event);
int dgs_stream_wait_event(void* stream, void* event);
/* out[c, m] = bf16(in[m, c]) for in [M, C] (fp32 if in_is_f32 else bf16), out [C, round_up(M, 64)] zero padded;
 * colsum (optional, fp32 [C]) += column sums.  Used for the transposed weight copies and inside the backward. */
int dgs_transpose_bf16(const void* in, int in_is_f32, int M, int C, void* out, float* colsum, void* stream);
/* fused AdamW on fp32 master parameters (torch.optim.AdamW semantics; diffusionGS_rel.yaml:57-62), step >= 1.
 * The gradient is multiplied by grad_scale * (grad_scale_dev ? *grad_scale_dev : 1): the clip factor stays on the device */
int dgs_adamw_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, size_t n, float lr, float beta1,
                   float beta2, float eps, float weight_decay, int step, float grad_scale, const float* grad_scale_dev,
                   void* stream);
/* Same update with the exponential moving average of the parameters folded in (the reference's EMA callback,
 * diffusionGS/utils/ema.py:82-101 with decay 0.9999, launch.py:227): after the AdamW update of p,
 * ema = ema_decay * ema + (1 - ema_decay) * p, in the same pass over the arena.  ema == NULL: plain dgs_adamw_step. */
int dgs_adamw_ema_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, float* ema, size_t n, float lr,
                       float beta1, float beta2, float eps, float weight_decay, int step, float grad_scale,
                       const float* grad_scale_dev, float ema_decay, void* stream);
/* weight refresh after an optimizer step: `batch` fp32 matrices [M, C] (matrix i at in + i*in_batch_stride floats) ->
 * bf16 copies [batch, M, C] (optional) and transposed bf16 copies [batch, C, M]; M, C multiples of 64 */
int dgs_cast_transpose_f32(const float* in, long long in_batch_stride, int batch, int M, int C, void* out_bf16,
                           void* outT_bf16, void* stream);

/* Building blocks, exported for the unit parity tests (same kernels dgs_dit_forward launches).
 * epi: 0 = bias -> bf16, 1 = bias + GELU(tanh) -> bf16, 2 = out(fp32) += gate[row / rows_per_sample] * (acc + bias),
 *      3 = (acc + bias) -> fp32.   A [M,K], W [N,K] bf16 row-major. */
int dgs_gemm_bf16(const void* A, const void* W, const float* bias, const float* gate, void* out, int M, int N,
                  int K, int epi, int ldc, int gate_stride, int rows_per_sample, void* stream);
/* qkv [B,N,3,heads,64] bf16 -> out [B,N,heads*64] bf16 = softmax(q k^T / 8) v */
int dgs_attention_fwd(const void* qkv, void* out, int B, int N, int heads, void* stream);
/* training pair: the forward also writes lse2 [B, heads, round_up(N,128)] fp32; the backward turns (qkv, out, lse2,
 * dout [B,N,heads*64] bf16) into dqkv [B,N,3,heads,64] bf16; dsum = scratch of the lse2 size. */
int dgs_attention_fwd_train(const void* qkv, void* out, float* lse2, int B, int N, int heads, void* stream);
int dgs_attention_bwd(const void* qkv, const void* out, const void* dout, float* lse2, float* dsum, void* dqkv, int B,
                      int N, int heads, void* stream);
/* extended GEMM entry (training epilogues): epi 4 = out(bf16) = acc * gelu'(aux);  aux (bf16 [M,ldc]): epi 1/2 also
 * store acc + bias there;  resid: residual source of epi 2 (NULL = in place);  lda/ldb: operand row strides (0 = K) */
int dgs_gemm_bf16_ex(const void* A, const void* W, const float* bias, const float* gate, void* out, void* aux,
                     const float* resid, int M, int N, int K, int lda, int ldb, int epi, int ldc, int gate_stride,
                     int rows_per_sample, void* stream);
/* out[M,N] (fp32, row stride ldc) = A^T W for A [K,M], W [K,N] bf16 row-major with row strides lda / ldb (0 = M / N):
 * the weight-gradient GEMM (K = tokens) on MN-major wgmma operands -- no transposed copies */
int dgs_gemm_bf16_tn(const void* A, const void* W, float* out, int M, int N, int K, int lda, int ldb, int ldc, void* stream);
/* backward of dgs_ln_modulate: dx (+)= ..., dshift/dscale [B, mod_stride] += ..., dln_w += ... (NULL where absent);
 * stats = scratch of 2*B*rows floats (per-row mean / rstd handed from the row kernel to the column kernel) */
int dgs_ln_modulate_bwd(const float* x, const void* dh, int dh_is_f32, const float* ln_w, const float* scale,
                        int mod_stride, int B, int rows, int width, float eps, float* dx, int accumulate, float* dshift,
                        float* dscale, float* dln_w, float* stats, void* stream);
/* backward of x_out = x_in + gate[b] * y: dy (bf16 [M,C]), dyT (bf16 [C, round_up(M,64)]), dgate += , dbias += */
int dgs_gate_bwd(const float* dx, const void* y, const float* gate, int gate_stride, int rows_per_sample, int M, int C,
                 void* dy, void* dyT, float* dgate, float* dbias, void* stream);
/* h = (LN(x; eps) [* ln_w]) * (1 + scale[b]) + shift[b] -> bf16 ; x fp32 [B, rows, width] */
int dgs_ln_modulate(const float* x, const float* ln_w, const float* shift, const float* scale, int mod_stride,
                    void* h, int B, int rows, int width, float eps, void* stream);

/* ------------------------------------------------------------------------------------------------
 * B2b. LPIPS-VGG perceptual distance, the lpips term of LossComputer (diffusionGS/utils/losses.py:243-309, which calls
 * lpips.LPIPS(net="vgg") in eval mode): ScalingLayer (x - shift) / scale, torchvision VGG16 features[0:30] (13 conv3x3
 * + ReLU, 4 max-pools), channel-normalised taps relu1_2 .. relu5_3, 1x1 `lin` weights, spatial mean, sum over taps.
 * Inputs NCHW fp32 [n, 3, H, W] in [-1, 1]; out [n] fp32.  Activations are bf16, GEMMs accumulate in fp32.
 * H and W must be multiples of 16 and at least 16, n > 0; anything else is DGS_ERR_INVALID_ARGUMENT.
 * The images are processed in chunks of as many as the workspace holds (dgs_lpips_workspace_bytes(c, H, W) bytes run
 * c images at a time; at least c = 1); the results do not depend on the chunking.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  /* conv l = 0..12 (torchvision features indices 0,2,5,7,10,12,14,17,19,21,24,26,28):
     conv_w[l]  bf16 [C_out, 9*C_in] with K ordered (ky, kx, c_in); conv1_1's C_in is zero-padded from 3 to 8;
     conv_wt[l] bf16 [C_in, 9*C_out] = W flipped in both spatial axes and transposed: Wt[ci, (ky, kx, co)] =
                W[co, ci, 2-ky, 2-kx]; conv1_1's copy has 32 rows, rows 3..31 zero (the input gradient's GEMM);
     conv_b[l]  fp32 [C_out] */
  const void* conv_w[13];
  const void* conv_wt[13];
  const float* conv_b[13];
  const float* lin[5];   /* lin{k}.model.1.weight, fp32 [C_k] = 64, 128, 256, 512, 512 */
  const float* shift;    /* scaling_layer.shift, fp32 [3] */
  const float* scale;    /* scaling_layer.scale, fp32 [3] */
} dgs_lpips_weights;

/* Workspace for c images at a time (about 109 MB per image at 256 x 256, most of it the im2col operand). */
size_t dgs_lpips_workspace_bytes(int n, int H, int W);
/* Training state for n images: in0's post-ReLU activations of all 13 convolutions in bf16 (35 MB per image at 256 x 256)
 * and the gradient of the distance w.r.t. in0's activations at the 5 taps in fp32 (32 MB per image).  The second
 * input's activations are never kept. */
size_t dgs_lpips_state_bytes(int n, int H, int W);
/* out[i] = LPIPS(in0[i], in1[i]).  state: NULL for inference, else a buffer of dgs_lpips_state_bytes(n, H, W) that must
 * stay untouched until dgs_lpips_backward has run.  Inference and training forwards give the same out, bit for bit. */
int dgs_lpips_forward(const dgs_lpips_weights* w, int n, int H, int W, const float* in0, const float* in1, float* out,
                      void* state /* NULL = inference */, void* workspace, size_t workspace_bytes, void* stream);
/* d_in0 [n, 3, H, W] fp32 (overwritten) = dout[i] * d out[i] / d in0[i], dout = device fp32 [n].  The gradient w.r.t. in1
 * is not computed.  The workspace need not be the forward's. */
int dgs_lpips_backward(const dgs_lpips_weights* w, int n, int H, int W, const void* state, const float* dout,
                       float* d_in0, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * B2c. SSIM with an 11-tap Gaussian window (sigma 1.5), C1 = (0.01 R)^2, C2 = (0.03 R)^2, R = data_range, per image
 * the mean over the 3 channels and the (H-10) x (W-10) valid pixels; optionally PSNR of the images clamped to [0, 1].
 *   sample_covariance = 0: pytorch_msssim.SSIM(win_size=11, win_sigma=1.5, channel=3), the ssim term of LossComputer
 *                          (diffusionGS/utils/losses.py:216-234, 314-318);
 *   sample_covariance = 1: skimage structural_similarity(gaussian_weights=True, win_size=11, channel_axis=0) of
 *                          MetricComputer.compute_ssim (losses.py:373-473): variances scaled by 121/120.  Its
 *                          reflect-padded filter is only read inside the valid window, so the value is the same mean.
 * Images NCHW fp32 [n, 3, H, W]; 0 < n <= 65535, H and W >= 11, data_range > 0, else DGS_ERR_INVALID_ARGUMENT.
 * No atomics: results do not depend on n or on whether a training state is written, bit for bit.
 * ---------------------------------------------------------------------------------------------- */
/* Workspace of one forward: one partial sum pair per (image, 32 x 32 output tile). */
size_t dgs_ssim_workspace_bytes(int n, int H, int W);
/* Training state: 3 coefficient maps x 3 channels x (H-10)(W-10) fp32 per image. */
size_t dgs_ssim_state_bytes(int n, int H, int W);
/* ssim[i] = SSIM(x[i], y[i]) (device fp32 [n]); psnr[i] = -10 log10(mean (clamp(x) - clamp(y))^2) when psnr != NULL
 * (+inf for identical images).  state: NULL for inference, else a buffer of dgs_ssim_state_bytes(n, H, W) that must stay
 * untouched until dgs_ssim_backward has run. */
int dgs_ssim_forward(int n, int H, int W, const float* x, const float* y, float data_range, int sample_covariance,
                     float* ssim /* [n] */, float* psnr /* [n] or NULL */, void* state /* NULL = inference */,
                     void* workspace, size_t workspace_bytes, void* stream);
/* d_x [n, 3, H, W] fp32 (overwritten) = dout[i] * d ssim[i] / d x[i], dout = device fp32 [n] (the gradient of ssim, not of
 * 1 - ssim).  x and y are the forward's images.  The gradient w.r.t. y is not computed. */
int dgs_ssim_backward(int n, int H, int W, const float* x, const float* y, const void* state, const float* dout,
                      float* d_x, void* stream);

/* ------------------------------------------------------------------------------------------------
 * B2d. Mesh extraction after the sampler loop: GaussianModel.extract_fields / extract_mesh
 * (diffusionGS/models/gsrenderer/gs_core.py:786-869).
 * ---------------------------------------------------------------------------------------------- */
/* The block-truncated opacity field of extract_fields(resolution, num_blocks, relax_ratio).  Inputs are the RAW fp32
 * tensors xyz [P,3], scaling [P,3], rotation [P,4] (not normalised), opacity [P,1]; scale_modifier is 1 when the model
 * has none; center (device fp32 [3]) and scale are the caller's mesh_center and fp32 mesh_scale; lin (device fp32
 * [resolution]) is torch.linspace(-1, 1, resolution), whose values decide membership.  Each axis is cut into chunks of
 * resolution / num_blocks points (the last one shorter); a Gaussian belongs to a block of three chunks iff on every axis
 * vmin < (x - center) * scale < vmax, with vmin / vmax the chunk's first / last coordinate -/+ fp32((2 / num_blocks) *
 * relax_ratio), all fp32 as in the reference.  occ [resolution^3] (x-major, fp32) = per point the sum over the block's
 * Gaussians, in Gaussian order, of opacity * exp(power) (0 where power > 0); blocks without Gaussians are 0.  The sum
 * order is fixed: the result does not change from run to run.
 * block_counts (NULL, or device int [chunks^3]) receives each block's number of Gaussians; *num_pairs (NULL or host)
 * the total.  scratch_alloc is called once for per-Gaussian and per-block scratch and, after the one host sync that
 * reads the pair count, once more for the pairs (16 B each plus the sort's temporary storage); both are free after
 * the call.  More than 2^31 - 1 pairs is DGS_ERR_OVERFLOW. */
int dgs_mesh_field(int P, const float* xyz, const float* scaling, const float* rotation, const float* opacity,
                   float scale_modifier, const float* center, float scale, int resolution, int num_blocks,
                   double relax_ratio, const float* lin, float* occ, int* block_counts, long long* num_pairs,
                   dgs_alloc_fn scratch_alloc, void* scratch_user, void* stream);
/* Marching cubes over field [nx, ny, nz] (C order, fp32, every size >= 2).  A grid point is inside iff value > iso; every
 * grid edge with exactly one inside end gets one vertex, at a + (iso - va) / (vb - va) (b - a) in index coordinates,
 * shared by the triangles of the (up to four) voxels around it, so the mesh is welded.  Vertices are ordered by owning
 * edge (grid point in C order, then axis x, y, z), triangles by voxel, then case-table order (mc_tables.h, generated by
 * gen_mc_tables.py); each triangle's right-hand-rule normal points from inside to outside.  On faces with two diagonally
 * opposite inside corners the inside corners are kept apart, so the surface is closed.
 * alloc is called once for scratch (10 B per grid point plus the scans' temporary storage, free after the call), then,
 * after the one host sync that reads the totals, for *vertices (fp32 [V, 3]) and *triangles (int32 [F, 3]) when V > 0.
 * An empty surface returns V = F = 0 and NULL outputs. */
int dgs_marching_cubes(const float* field, int nx, int ny, int nz, float iso, dgs_alloc_fn alloc, void* alloc_user,
                       float** vertices, int** triangles, long long* num_vertices, long long* num_triangles,
                       void* stream);

/* ------------------------------------------------------------------------------------------------
 * B3. The elementwise callers either side of the path.
 * ---------------------------------------------------------------------------------------------- */
/* TransformInput (diffusionGS/systems/utils.py:621-757, patch_size=None): per-pixel world-space rays.
 * c2w [n_views,4,4] row-major, fxfycxcy [n_views,4] -> ray_o, ray_d [n_views,3,H,W] (ray_d normalised). */
int dgs_rays_from_cameras(const float* c2w, const float* fxfycxcy, int n_views, int H, int W, float* ray_o,
                          float* ray_d, void* stream);
/* GaussianDiffusion.q_sample (gaussian_diffusion.py:268-284): out = sqrt_ac[t[b]]*x_start + sqrt_1mac[t[b]]*noise.
 * Tables are DEVICE fp32 arrays indexed by timestep; t is int64 [B]; per_sample = elements per batch item. */
int dgs_q_sample(const float* x_start, const float* noise, const float* sqrt_alphas_cumprod,
                 const float* sqrt_one_minus_alphas_cumprod, const long long* t, int B, long long per_sample,
                 float* out, void* stream);
/* One ancestral step of p_sample with x0-prediction and FIXED_LARGE variance (gaussian_diffusion.py:291-312,
 * 380-392, 505-516): out = coef1[t]*pred_xstart + coef2[t]*x_t + (t != 0) * exp(0.5*log_var[t]) * noise. */
int dgs_p_sample_step(const float* pred_xstart, const float* x_t, const float* noise, const float* posterior_mean_coef1,
                      const float* posterior_mean_coef2, const float* model_log_variance, const long long* t, int B,
                      long long per_sample, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DGS_B200_H_INCLUDED */
