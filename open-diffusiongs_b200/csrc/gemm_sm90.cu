// gemm_sm90.cu -- persistent, warp-specialised wgmma GEMM for the DiT linears (sm_90a).
//
//   C[M,N] = epilogue( A[M,K] (bf16, row-major) x W[N,K]^T (bf16, row-major = nn.Linear weight) )
//
// One CTA per SM, 384 threads: warps 0..7 = two consumer warpgroups (64 rows of the 128-row tile each, fp32
// accumulators in registers), warp 8 = TMA producer (its warpgroup gives its registers to the consumers).  Operands are
// staged by TMA into a 128-byte-swizzled shared-memory ring (a k-block of K = one 128-byte swizzle row) that runs
// continuously across the CTA's tiles, so the producer loads the next tile while the consumers run the epilogue of the
// current one.  Tile = 128 x BN (BN = 256 or 128),
// wgmma m64nBNk16, one k-block group kept in flight while the next is issued.  The inference epilogues stage the
// finished tile in shared memory and hand it to the TMA unit (a store, or for the in-place residual update a reduce-add
// in L2), so the consumers go on to the next tile's mainloop while the tile is written out.  The two consumer
// warpgroups run their epilogues at the same time, so the tensor cores idle for as long as an epilogue takes: it loads
// the bias and gate values of eight column groups at once before using them, rather than waiting for each load in turn
// (one memory latency per column pair cost qkv and mlp.fc1 a fifth of their time at 4098 tokens).
//
// Operand modes (GemmOp): bf16 K-major (the forward and dgrad GEMMs), bf16 MN-major (the weight gradients, gemm_bf16_tn)
// and e4m3 (the FP8 inference path, gemm_fp8).  The e4m3 mode is the K-major kernel at BN = 128 with a k-block of 128
// e4m3 elements, the k-block's 128 activation row scales loaded with each stage, four wgmma m64n128k32 per k-block into
// a fresh partial tile that is added into the accumulator times its rows' scales, and the per-channel weight scale
// applied before the epilogue.
//
// Fused epilogues = the elementwise tails of the reference DiT block
// (diffusionGS/models/transformers/utils_transformer.py:270-290, timm Attention/Mlp):
//   EPI_BIAS_BF16       y = acc + b                         (qkv)
//   EPI_BIAS_GELU_BF16  y = gelu_tanh(acc + b)              (mlp.fc1 + act)
//   EPI_GATE_RESID_F32  x += gate[sample] * (acc + b)       (attn.proj / mlp.fc2 + gate + residual, fp32 stream)
//   EPI_F32             y = acc (+ b), fp32                 (tokenizer, decoder head, weight gradients)
//   EPI_DGELU_BF16      y = acc * gelu'(u)                  (backward of mlp.fc2 -> act: u = saved pre-activation)
//   EPI_BIAS_RELU_BF16  y = max(acc + b, 0)                 (the LPIPS VGG convolutions, lpips.cu)
//   EPI_BIAS_GELU_E4M3  y = e4m3(gelu_tanh(acc + b)) + scales (FP8 mlp.fc1 -> fc2's operand; e4m3 mode only)
// Training mode (GemmEpilogue::aux / resid): fc1 also stores its pre-activation, the gate epilogues also store the
// pre-gate branch output and may read the residual from a different buffer than they write.
#include <cstdlib>
#include <cstring>

#include "dgs_internal.h"
#include "dit_kernels.h"
#include "sm90_ptx.cuh"

namespace dgs {

using namespace ptx;

// ---------------------------------------------------------------------------------------------
// host: tensor maps
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int make_tmap(CUtensorMap* out, CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims,
              const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swizzle) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled not available (no CUDA driver?)"); return DGS_ERR_CUDA; }
  cuuint64_t gdim[5], gstr[5];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; i++) { gdim[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i + 1 < rank; i++) gstr[i] = strides_bytes[i];
  CUresult r = fn(out, dtype, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r); return DGS_ERR_CUDA; }
  return DGS_OK;
}

// ---------------------------------------------------------------------------------------------
// device
// ---------------------------------------------------------------------------------------------
constexpr int BM = 128, BK = 64, BK8 = 128;  // BK / BK8: the bf16 / e4m3 elements of a k-block (one 128-byte row)
constexpr int GEMM_THREADS = WS_THREADS;

enum GemmOp { OP_BF16_K = 0, OP_BF16_MN = 1, OP_E4M3 = 2 };

// OUT_BYTES: element size of the output tile staged in shared memory for the TMA-store epilogue (0: the epilogue
// writes from registers).  The staging buffer takes what would otherwise be operand stages.  It holds RING column
// blocks (128 bytes x 64 rows, 8 KB) per consumer warpgroup: the whole 64 x BN fragment of a 128 x 128 tile, and two
// column blocks at a time of a 128 x 256 tile (staged whole, a bf16 tile would leave three operand stages and an fp32
// tile two), which keeps four stages.  SCALE_BYTES: the row scales a stage carries besides its operands (e4m3: BM fp32,
// else 0).
template <int BN, int OUT_BYTES, int SCALE_BYTES>
struct GemmCfg {
  static constexpr int SMEM_LIMIT = 227 * 1024;
  static constexpr int S_BYTES = SCALE_BYTES;
  static constexpr int A_BYTES = BM * 128;
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int OUT_BLOCKS = BN * OUT_BYTES / 128;  // column blocks of a warpgroup's fragment
  static constexpr int RING = BN == 256 && OUT_BLOCKS > 2 ? 2 : OUT_BLOCKS;
  static constexpr int OUT_TILE_BYTES = 2 * RING * 8192;
  static constexpr int EXTRA = 1024 /*align slack*/ + 256 /*barriers*/;
  static constexpr int FIT = (SMEM_LIMIT - EXTRA - OUT_TILE_BYTES) / (STAGE_BYTES + S_BYTES);
  static constexpr int STAGES = FIT < (BN == 256 ? 4 : 6) ? FIT : (BN == 256 ? 4 : 6);
  static constexpr int SMEM_BYTES = STAGES * (STAGE_BYTES + S_BYTES) + OUT_TILE_BYTES + EXTRA;
  static_assert(STAGES >= 3 && SMEM_BYTES <= SMEM_LIMIT, "GEMM configuration does not fit in shared memory");
  static_assert(S_BYTES % 16 == 0, "the row scales are one bulk copy per stage: 16-byte multiples");
};
static_assert(GemmCfg<256, 4, 0>::RING == 2 && GemmCfg<256, 4, 0>::STAGES == 4 && GemmCfg<256, 2, 0>::RING == 2 &&
                  GemmCfg<256, 2, 0>::STAGES == 4,
              "the bf16 stores and the in-place gate + residual update on 128 x 256 tiles keep four operand stages");
static_assert(GemmCfg<128, 1, BM * 4>::STAGES == 6 && GemmCfg<128, 4, BM * 4>::STAGES == 4,
              "FP8 stage counts: 6 for fc1 (e4m3 out), 4 for fc2 (in-place fp32)");

// The element size of the output tile of each epilogue when it is staged for a TMA store (see epilogue_tma).
constexpr int epi_out_bytes(int epi) {
  return (epi == EPI_GATE_RESID_F32 || epi == EPI_F32) ? 4 : (epi == EPI_BIAS_GELU_E4M3 ? 1 : 2);
}

// FP8 scales (gemm_fp8; unused in the bf16 modes)
struct Fp8Scales {
  const float* sa = nullptr;         // [K/128][lds] activation group scales
  const float* sw = nullptr;         // [N] weight scales
  float* out_scale = nullptr;        // EPI_BIAS_GELU_E4M3: [N/128][lds] group scales of the output
  int lds = 0;                       // fp8_scale_stride(M)
};

__device__ __forceinline__ float epi_gelu_tanh(float x) {  // nn.GELU(approximate="tanh"), tanh on the MUFU pipe
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  const float u = k0 * (x + k1 * x * x * x);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
  return 0.5f * x * (1.0f + t);
}
__device__ __forceinline__ float epi_dgelu_tanh(float x) {  // d/dx of the above
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  const float x2 = x * x;
  const float u = k0 * (x + k1 * x * x2);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
  const float du = k0 * (1.0f + 3.0f * k1 * x2);
  return 0.5f * (1.0f + t) + 0.5f * x * (1.0f - t * t) * du;
}

// The GELU or ReLU of the epilogues that have one.
template <int EPI>
__device__ __forceinline__ float2 epi_act(float2 v) {
  if (EPI == EPI_BIAS_GELU_BF16 || EPI == EPI_BIAS_GELU_E4M3) { v.x = epi_gelu_tanh(v.x); v.y = epi_gelu_tanh(v.y); }
  if (EPI == EPI_BIAS_RELU_BF16) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); }
  return v;
}

// The per-element part every epilogue shares, on one thread's column pair (n, n+1) of output row offset ro: acc + b
// (with keep_pre, training mode, also stored to ep.aux as bf16), then the GELU or ReLU of the epilogues that have one.
template <int EPI>
__device__ __forceinline__ float2 epi_bias_act(const GemmEpilogue& ep, float2 v, int n, bool keep_pre = false,
                                               size_t ro = 0) {
  if (ep.bias) {
    const float2 b = __ldg(reinterpret_cast<const float2*>(ep.bias + n));
    v.x += b.x; v.y += b.y;
  }
  if (keep_pre) *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(ep.aux) + ro + n) = pack2_bf16(v.x, v.y);
  return epi_act<EPI>(v);
}

template <int BN, bool MN>
__device__ __forceinline__ void wg_mma_k16(float (&acc)[BN / 2], uint64_t da, uint64_t db) {
  if constexpr (BN == 256) wgmma_m64n256_ss<MN, MN>(acc, da, db);
  else wgmma_m64n128_ss<MN, MN>(acc, da, db);
}

// Fused epilogue of one 64 x BN accumulator fragment (see sm90_ptx.cuh for the fragment layout).  Every thread owns
// column pairs (n, n+1) of two rows.  reduce: EPI_F32 only -- add into the output (split-K partial sums).
template <int EPI, int BN>
__device__ __forceinline__ void epilogue_fragment(const GemmEpilogue& ep, const float (&acc)[BN / 2], int row0, int n0,
                                                  int M, int N, bool reduce) {
#pragma unroll
  for (int i = 0; i < 2; i++) {
    const int row = row0 + 8 * i;
    if (row >= M) continue;
    const float* gate_row =
        EPI == EPI_GATE_RESID_F32 ? ep.gate + (size_t)(row / ep.rows_per_sample) * ep.gate_stride : nullptr;
    const size_t ro = (size_t)row * ep.ldc;
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
      const int n = n0 + 8 * j;
      if (n >= N) break;  // N % 32 == 0: whole 8-column groups are in or out
      const bool keep_pre = (EPI == EPI_BIAS_GELU_BF16 || EPI == EPI_GATE_RESID_F32) && ep.aux;
      float2 v = epi_bias_act<EPI>(ep, make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]), n, keep_pre, ro);
      if (EPI == EPI_BIAS_BF16 || EPI == EPI_BIAS_GELU_BF16 || EPI == EPI_DGELU_BF16 || EPI == EPI_BIAS_RELU_BF16) {
        if (EPI == EPI_DGELU_BF16) {
          const __nv_bfloat162 u = *reinterpret_cast<const __nv_bfloat162*>(reinterpret_cast<const __nv_bfloat16*>(ep.aux) + ro + n);
          const float2 uf = __bfloat1622float2(u);
          v.x *= epi_dgelu_tanh(uf.x); v.y *= epi_dgelu_tanh(uf.y);
        }
        *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(ep.out) + ro + n) = pack2_bf16(v.x, v.y);
      } else if (EPI == EPI_GATE_RESID_F32) {
        float* x = reinterpret_cast<float*>(ep.out) + ro + n;
        const float2 r = *reinterpret_cast<const float2*>(ep.resid ? ep.resid + ro + n : x);
        const float2 g = __ldg(reinterpret_cast<const float2*>(gate_row + n));
        // r + round(g v), not fmaf: the same value as the in-place TMA reduce-add of epilogue_tma
        *reinterpret_cast<float2*>(x) = make_float2(__fadd_rn(r.x, __fmul_rn(g.x, v.x)), __fadd_rn(r.y, __fmul_rn(g.y, v.y)));
      } else {  // EPI_F32
        float2* o = reinterpret_cast<float2*>(reinterpret_cast<float*>(ep.out) + ro + n);
        if (reduce) atomicAdd(o, v);
        else *o = v;
      }
    }
  }
}

// Epilogue of one warpgroup's 64 x BN fragment through shared memory: the values are computed in registers as in
// epilogue_fragment, written to this warpgroup's staging buffer, and one thread hands the buffer to the TMA unit, which
// writes it out while the warpgroup goes on with its next tile's mainloop.  Rows >= M and columns >= N are clipped by
// the TMA unit.  The staging buffer holds column blocks of 128 bytes (64 bf16 / 32 fp32 / 128 e4m3 columns) x 64 rows,
// 8 KB each, 128-byte swizzled like the TMA box that stores it: the 16-byte chunk c of row r sits at chunk c ^ (r % 8),
// which also makes the fragment writes free of bank conflicts.
// EPI_GATE_RESID_F32 (in place, no ep.resid) stages gate * (acc + b) and adds it into x with a TMA reduce-add, so x is
// never read by the SM.  The result is x + round(g * v) rather than fmaf(g, v, x): one more fp32 rounding per update.
// EPI_BIAS_GELU_E4M3 (BN = 128): the tile's 128 columns are one scale group, so a row's amax is a reduction over the 4
// lanes that hold the row; a pass over the row applies bias + GELU and writes the row's scale straight to out_scale
// before the row is staged.
// RING < the fragment's column blocks: the fragment goes out in batches of RING blocks, each written once the previous
// batch's stores have read the buffer.
template <int EPI, int BN, int RING>
__device__ __forceinline__ void epilogue_tma(const GemmEpilogue& ep, const Fp8Scales& fs, float (&acc)[BN / 2],
                                             uint8_t* stage, const CUtensorMap* tmC, int m0, int n0, int M, int N, int wg,
                                             int wq, int lane) {
  constexpr int OB = epi_out_bytes(EPI);
  constexpr int COLS = 128 / OB;            // columns per staging row
  constexpr int JB = RING * COLS / 8;       // 8-column groups per batch
  constexpr bool WHOLE = EPI == EPI_BIAS_GELU_E4M3;  // gemm_fp8 checks N % 128 == 0: the tile has no columns >= N
  constexpr int PJ = JB < 8 ? JB : 8;       // 8-column groups whose bias and gate are loaded ahead at once
  static_assert(JB % PJ == 0, "whole load groups per batch");
  const bool leader = wq == 0 && lane == 0;
  float2 bias_v[PJ], gate_v[PJ];
  const float* gate_row[2] = {nullptr, nullptr};
  if (EPI == EPI_GATE_RESID_F32) {
#pragma unroll
    for (int i = 0; i < 2; i++) {
      const int row = min(m0 + 16 * wq + (lane >> 2) + 8 * i, M - 1);  // rows >= M are clipped by the store, but must
      gate_row[i] = ep.gate + (size_t)(row / ep.rows_per_sample) * ep.gate_stride;  // not index past the gates
    }
  }
#pragma unroll
  for (int j0 = 0; j0 < BN / 8; j0 += JB) {
    if (!WHOLE && n0 + 8 * j0 >= N) break;
    if (leader) bulk_wait_read<0>();  // the stores of the previous batch (or tile) have read the buffer
    named_bar_sync(1 + wg, 128);
#pragma unroll
    for (int i = 0; i < 2; i++) {
      const int r = 16 * wq + (lane >> 2) + 8 * i;  // row in the warpgroup's 64-row slice; r % 8 == lane / 4
      float inv;  // EPI_BIAS_GELU_E4M3: 1 / the row's scale
      if constexpr (EPI == EPI_BIAS_GELU_E4M3) {  // bias + GELU into acc, then the row's amax and scale
        static_assert(BN == 128 && JB == BN / 8, "one e4m3 scale group per tile row, staged in one batch");
        float amax = 0.f;
#pragma unroll
        for (int j = 0; j < BN / 8; j++) {
          const float2 v = epi_bias_act<EPI>(ep, make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]),
                                             n0 + 8 * j + 2 * (lane & 3));
          acc[4 * j + 2 * i] = v.x; acc[4 * j + 2 * i + 1] = v.y;
          amax = fmaxf(amax, fmaxf(fabsf(v.x), fabsf(v.y)));
        }
        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
        const int e = e4m3_scale_exp(amax);
        inv = exp2_int(-e);
        if ((lane & 3) == 0 && m0 + r < M) fs.out_scale[(size_t)(n0 / 128) * fs.lds + m0 + r] = exp2_int(e);
      }
#pragma unroll
      for (int j = j0; j < j0 + JB; j++) {
        // The bias and gate column pairs of the next PJ groups are loaded together before the first is used, so that
        // the fragment waits for one memory latency per PJ groups rather than one per group.  Columns >= N (only in
        // the last tile column when N % BN != 0) read the pair N - 2 instead: they are staged, and clipped by the store.
        const int jp = (j - j0) % PJ;
        if (!WHOLE && jp == 0) {
#pragma unroll
          for (int q = 0; q < PJ; q++) {
            const int n = min(n0 + 8 * (j + q) + 2 * (lane & 3), N - 2);
            if (ep.bias) bias_v[q] = __ldg(reinterpret_cast<const float2*>(ep.bias + n));
            if (EPI == EPI_GATE_RESID_F32) gate_v[q] = __ldg(reinterpret_cast<const float2*>(gate_row[i] + n));
          }
        }
        float2 v = make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
        if constexpr (EPI == EPI_BIAS_GELU_E4M3) {
          v.x *= inv; v.y *= inv;
        } else {
          if (ep.bias) { v.x += bias_v[jp].x; v.y += bias_v[jp].y; }
          v = epi_act<EPI>(v);
        }
        if (EPI == EPI_GATE_RESID_F32) { v.x *= gate_v[jp].x; v.y *= gate_v[jp].y; }
        const int byte = ((8 * j) % COLS + 2 * (lane & 3)) * OB;  // within the 128-byte staging row
        uint8_t* p = stage + (8 * j / COLS % RING) * 8192 + r * 128 + ((((byte >> 4) ^ (lane >> 2)) << 4) | (byte & 15));
        if (OB == 1) *reinterpret_cast<uint16_t*>(p) = pack2_e4m3(v.x, v.y);
        else if (OB == 2) *reinterpret_cast<uint32_t*>(p) = pack2_bf16(v.x, v.y);
        else *reinterpret_cast<float2*>(p) = v;
      }
    }
    fence_proxy_async();  // make the generic-proxy writes visible to the TMA unit
    named_bar_sync(1 + wg, 128);
    if (leader) {
#pragma unroll
      for (int b = 8 * j0 / COLS; b < 8 * j0 / COLS + RING; b++) {
        if (!WHOLE && n0 + b * COLS >= N) break;
        if (EPI == EPI_GATE_RESID_F32) tma_reduce_add_2d(tmC, stage + (b % RING) * 8192, n0 + b * COLS, m0);
        else tma_store_2d(tmC, stage + (b % RING) * 8192, n0 + b * COLS, m0);
      }
      bulk_commit();
    }
  }
}

// OP = OP_BF16_K:  C = A[M,K] x W[N,K]^T, both operands K-major (rows of 64 K elements = one 128-byte swizzle row).
// OP = OP_BF16_MN: C = A^T x W   for A [K, M], W [K, N] row-major, i.e. both operands MN-major (the weight-gradient
//              GEMM dW = dY^T X with K = tokens: neither operand has to be transposed in memory).  A stage then holds
//              BM/64 (resp. BN/64) swizzle atoms of [64 K rows x 64 M/N elements]; the descriptors use LBO = 8192 B
//              (atom to atom along M/N), SBO = 1024 B (8 K rows), and step 16 K rows = 2048 B per wgmma.
// OP = OP_E4M3:    C = sw[n] * sum_kb sa[kb][m] * (A_kb W_kb^T), e4m3 operands K-major (rows of 128 K elements), BN = 128
//              (a 128 x 256 tile would need 128 + 128 accumulator registers per thread: over the consumers' 232).  The
//              partial tile of each k-block keeps the tensor core's reduced-precision FP8 accumulation to one 128-term sum.
// splits > 1 (split-K, bf16 EPI_F32 only): work unit u = (tile u % num_tiles, K range u / num_tiles); every unit adds
// its partial product into the (pre-zeroed) output.
// TMA_EPI: the epilogue goes through shared memory and a TMA store into tmC (epilogue_tma); otherwise it writes from
// registers (epilogue_fragment) and tmC is unused.
template <int BN, int EPI, int OP, bool TMA_EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
            const __grid_constant__ CUtensorMap tmC, GemmEpilogue ep, int M, int N, int K, int splits, Fp8Scales fs) {
  constexpr bool MN = OP == OP_BF16_MN, E4M3 = OP == OP_E4M3;
  constexpr int KB = E4M3 ? BK8 : BK;
  static_assert(!E4M3 || BN == 128, "the e4m3 mode runs 128 x 128 tiles");
  using Cfg = GemmCfg<BN, TMA_EPI ? epi_out_bytes(EPI) : 0, E4M3 ? BM * 4 : 0>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  uint8_t* sA = smem;
  uint8_t* sB = smem + Cfg::STAGES * Cfg::A_BYTES;
  uint8_t* sC = smem + Cfg::STAGES * Cfg::STAGE_BYTES;  // TMA_EPI: one 64 x BN staging buffer per consumer warpgroup
  float* sS = reinterpret_cast<float*>(sC + Cfg::OUT_TILE_BYTES);  // e4m3: [STAGES][BM] row scales of the k-block
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sC + Cfg::OUT_TILE_BYTES + Cfg::STAGES * Cfg::S_BYTES);
  uint64_t* empty_bar = full_bar + Cfg::STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_m = (M + BM - 1) / BM, num_n = (N + BN - 1) / BN;
  const int num_tiles = num_m * num_n, num_k = (K + KB - 1) / KB;
  const int num_units = num_tiles * splits, kpb = (num_k + splits - 1) / splits;  // k-blocks per unit

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    for (int s = 0; s < Cfg::STAGES; s++) { mbar_init(full_bar + s, 1); mbar_init(empty_bar + s, 8); }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_launch_dependents();  // PDL: see sm90_ptx.cuh
  griddep_wait();

  if (warp >= 8) {
    // ===================== TMA producer =====================
    ws_producer_regs();
    if (warp == 8 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int unit = blockIdx.x; unit < num_units; unit += gridDim.x) {
        const int tile = E4M3 ? unit : unit % num_tiles;  // the e4m3 mode does not split K
        const int kb0 = E4M3 ? 0 : (unit / num_tiles) * kpb, kb1 = E4M3 ? num_k : min(num_k, kb0 + kpb);
        const int m0 = (tile / num_n) * BM, n0 = (tile % num_n) * BN;
        // e4m3: the scale rows [m0, min(m0 + 128, lds)): lds % 4 == 0, so a multiple of 16 bytes that stays inside sa
        const uint32_t sbytes = E4M3 ? (uint32_t)min(BM, fs.lds - m0) * 4u : 0u;
        for (int kb = kb0; kb < kb1; kb++) {
          mbar_wait(empty_bar + stage, phase ^ 1);
          mbar_arrive_expect_tx(full_bar + stage, Cfg::STAGE_BYTES + sbytes);
          if (!MN) {
            tma_load_2d(sA + stage * Cfg::A_BYTES, &tmA, full_bar + stage, kb * KB, m0);
            tma_load_2d(sB + stage * Cfg::B_BYTES, &tmB, full_bar + stage, kb * KB, n0);
          } else {  // one [64 K x 64 MN] box per swizzle atom
#pragma unroll
            for (int a = 0; a < BM / 64; a++)
              tma_load_2d(sA + stage * Cfg::A_BYTES + a * 8192, &tmA, full_bar + stage, m0 + a * 64, kb * BK);
#pragma unroll
            for (int a = 0; a < BN / 64; a++)
              tma_load_2d(sB + stage * Cfg::B_BYTES + a * 8192, &tmB, full_bar + stage, n0 + a * 64, kb * BK);
          }
          if constexpr (E4M3) bulk_load_1d(sS + stage * BM, fs.sa + (size_t)kb * fs.lds + m0, sbytes, full_bar + stage);
          if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumer warpgroups 0, 1: rows [64 wg, 64 wg + 64) of each tile =====================
    ws_consumer_regs();
    const int wg = warp >> 2;
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    for (int unit = blockIdx.x; unit < num_units; unit += gridDim.x) {
      const int tile = E4M3 ? unit : unit % num_tiles;  // the e4m3 mode does not split K
      const int kb0 = E4M3 ? 0 : (unit / num_tiles) * kpb, kb1 = E4M3 ? num_k : min(num_k, kb0 + kpb);
      const int m0 = (tile / num_n) * BM, n0 = (tile % num_n) * BN;
#pragma unroll
      for (int i = 0; i < BN / 2; i++) acc[i] = 0.f;
      int prev = -1;
      for (int kb = kb0; kb < kb1; kb++) {
        mbar_wait(full_bar + stage, phase);
        // K-major: this warpgroup's 64 rows start 64 x 128 B into the A tile; MN-major: they are the wg-th atom
        const uint64_t adesc = wg_desc_sw128(smem_u32(sA + stage * Cfg::A_BYTES + wg * 8192), MN ? 8192 : 16, 1024);
        const uint64_t bdesc = wg_desc_sw128(smem_u32(sB + stage * Cfg::B_BYTES), MN ? 8192 : 16, 1024);
        wg_fence();
        if constexpr (E4M3) {
          // k32 steps (32 bytes along the swizzle row) into a fresh partial tile, which is added into acc times its
          // rows' activation scales once it is complete; the stage is released as soon as the scales are read
          float part[64];
#pragma unroll
          for (int k = 0; k < BK8 / 32; k++) wgmma_m64n128k32_e4m3(part, adesc + 2 * k, bdesc + 2 * k, k);
          wg_commit();
          wg_wait<0>();
          wg_fence_regs(part);
          const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // the thread's rows r0, r0 + 8 of the tile
          const float s0 = sS[stage * BM + r0], s1 = sS[stage * BM + r0 + 8];
          __syncwarp();
          if (lane == 0) mbar_arrive(empty_bar + stage);
#pragma unroll
          for (int j = 0; j < 16; j++) {
            acc[4 * j] = fmaf(s0, part[4 * j], acc[4 * j]);
            acc[4 * j + 1] = fmaf(s0, part[4 * j + 1], acc[4 * j + 1]);
            acc[4 * j + 2] = fmaf(s1, part[4 * j + 2], acc[4 * j + 2]);
            acc[4 * j + 3] = fmaf(s1, part[4 * j + 3], acc[4 * j + 3]);
          }
        } else {
#pragma unroll
          for (int k = 0; k < BK / 16; k++) {
            // K-major: 16 bf16 = 32 bytes along the swizzle row (+2 in the >>4 address field); MN-major: 16 K rows = 2048 B
            const uint64_t adv = MN ? (uint64_t)(128 * k) : (uint64_t)(2 * k);
            wg_mma_k16<BN, MN>(acc, adesc + adv, bdesc + adv);
          }
          wg_commit();
          wg_wait<1>();  // the group of the previous k-block has retired: its stage may be refilled
          if (prev >= 0 && lane == 0) mbar_arrive(empty_bar + prev);
          prev = stage;
        }
        if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
      }
      if constexpr (E4M3) {  // the per-output-channel weight scales
#pragma unroll
        for (int j = 0; j < 16; j++) {
          const float2 w = __ldg(reinterpret_cast<const float2*>(fs.sw + n0 + 8 * j + 2 * (lane & 3)));
          acc[4 * j] *= w.x; acc[4 * j + 1] *= w.y; acc[4 * j + 2] *= w.x; acc[4 * j + 3] *= w.y;
        }
      } else {  // the last k-block's group is still in flight
        wg_wait<0>();
        wg_fence_regs(acc);
        if (prev >= 0 && lane == 0) mbar_arrive(empty_bar + prev);
      }
      if constexpr (TMA_EPI) {
        epilogue_tma<EPI, BN, Cfg::RING>(ep, fs, acc, sC + wg * (Cfg::OUT_TILE_BYTES / 2), &tmC, m0 + wg * 64, n0, M, N,
                                         wg, warp & 3, lane);
      } else {
        const int row0 = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
        epilogue_fragment<EPI, BN>(ep, acc, row0, n0 + 2 * (lane & 3), M, N, splits > 1);
      }
    }
    if (TMA_EPI && (warp & 3) == 0 && lane == 0) bulk_wait<0>();  // the output is written before the grid completes
  }
}

// ---------------------------------------------------------------------------------------------
// host launcher
// ---------------------------------------------------------------------------------------------
static int num_sms() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
      n = 0;
  }
  return n;
}

// A tensor map over a row-major [rows, cols] matrix of elem_bytes-byte elements with a row stride of ld elements, read
// or written in boxes of box_rows x box_cols (box_cols x elem_bytes = 128 bytes: one swizzle row).
static int tmap_2d(CUtensorMap* m, const void* base, int elem_bytes, int rows, int cols, int ld, int box_rows,
                   int box_cols) {
  const CUtensorMapDataType type = elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                   : (elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8);
  uint64_t dims[2] = {(uint64_t)cols, (uint64_t)rows}, str[1] = {(uint64_t)ld * elem_bytes};
  uint32_t box[2] = {(uint32_t)box_cols, (uint32_t)box_rows};
  return make_tmap(m, type, base, 2, dims, str, box);
}

template <int BN, int EPI, int OP, bool TMA_EPI>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const GemmEpilogue& ep,
                       int M, int N, int K, cudaStream_t st, int splits = 1, const Fp8Scales& fs = Fp8Scales()) {
  using Cfg = GemmCfg<BN, TMA_EPI ? epi_out_bytes(EPI) : 0, OP == OP_E4M3 ? BM * 4 : 0>;
  auto kern = gemm_kernel<BN, EPI, OP, TMA_EPI>;
  static bool configured = false;
  if (!configured) {
    DGS_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    configured = true;
  }
  const int sms = num_sms();
  DGS_REQUIRE(sms > 0, "gemm: cannot query the device's SM count");
  const int units = ceil_div(M, BM) * ceil_div(N, BN) * splits;
  const int grid = units < sms ? units : sms;
  DGS_CUDA_OK(launch_pdl(kern, dim3(grid), dim3(GEMM_THREADS), Cfg::SMEM_BYTES, st, tmA, tmB, tmC, ep, M, N, K, splits,
                         fs));
  DGS_POST_LAUNCH();
  return DGS_OK;
}

template <int EPI>
static int launch_epi(bool wide, bool tma_epi, const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC,
                      const GemmEpilogue& ep, int M, int N, int K, cudaStream_t st) {
  if constexpr (EPI != EPI_DGELU_BF16) {  // dGELU reads the saved pre-activation per element: register epilogue only
    if (tma_epi) {
      if constexpr (epi_out_bytes(EPI) == 2 || EPI == EPI_GATE_RESID_F32)
        if (wide) return launch_gemm<256, EPI, OP_BF16_K, true>(tmA, tmB, tmC, ep, M, N, K, st);
      return launch_gemm<128, EPI, OP_BF16_K, true>(tmA, tmB, tmC, ep, M, N, K, st);
    }
  }
  return wide ? launch_gemm<256, EPI, OP_BF16_K, false>(tmA, tmB, tmC, ep, M, N, K, st)
              : launch_gemm<128, EPI, OP_BF16_K, false>(tmA, tmB, tmC, ep, M, N, K, st);
}

int gemm_bf16(const void* A, const void* W, int M, int N, int K, int epi, const GemmEpilogue& ep, cudaStream_t st) {
  DGS_REQUIRE(M > 0 && N > 0 && K > 0, "gemm: bad shape %dx%dx%d", M, N, K);
  DGS_REQUIRE(N % 32 == 0, "gemm: need N %% 32 == 0 (got N=%d)", N);
  DGS_REQUIRE((ep.lda ? ep.lda : K) % 8 == 0 && (ep.ldb ? ep.ldb : K) % 8 == 0,
              "gemm: operand row strides must be multiples of 8 elements (K=%d lda=%d ldb=%d)", K, ep.lda, ep.ldb);
  DGS_REQUIRE(epi != EPI_DGELU_BF16 || ep.aux, "gemm: EPI_DGELU_BF16 needs aux = saved pre-activation");
  DGS_REQUIRE(((uintptr_t)A % 16) == 0 && ((uintptr_t)W % 16) == 0, "gemm: operands must be 16-byte aligned");
  // every thread stores column pairs (n, n + 1) of a row, n even: the pairs of every row are aligned when ldc is even
  DGS_REQUIRE(ep.ldc % 2 == 0, "gemm: the output row stride must be even (got ldc=%d)", ep.ldc);
  // a row stride below the row length would make rows overlap (and the last row run past an M x ldc buffer)
  DGS_REQUIRE(ep.ldc >= N, "gemm: ldc=%d must be >= N=%d", ep.ldc, N);
  DGS_REQUIRE(ep.lda == 0 || ep.lda >= K, "gemm: lda=%d must be >= K=%d (or 0)", ep.lda, K);
  DGS_REQUIRE(ep.ldb == 0 || ep.ldb >= K, "gemm: ldb=%d must be >= K=%d (or 0)", ep.ldb, K);
  const int sms = num_sms();
  DGS_REQUIRE(sms > 0, "gemm: cannot query the device's SM count");
  // The epilogue stages the tile in shared memory for a TMA store (or, in place, a TMA reduce-add) when the output rows
  // meet the TMA's 16-byte alignment.  The training variants (aux stores, a separate residual source), dGELU and
  // unaligned outputs write from registers.
  const int ob = epi_out_bytes(epi);
  const bool out_f32 = ob == 4;
  const bool tma_epi = epi != EPI_DGELU_BF16 && !ep.aux && !ep.resid && ep.ldc >= N && ((size_t)ep.ldc * ob) % 16 == 0 &&
                       ((uintptr_t)ep.out % 16) == 0;
  // 128 x 256 tiles when every CTA of the persistent grid gets at least two of them, so that each tile's epilogue
  // drains under the next tile's mainloop; else 128 x 128 tiles.  The in-place gate + residual update (staged two column
  // blocks at a time, four operand stages) takes 128 x 256 tiles at any M: at attn.proj / mlp.fc2 (4098 tokens, one
  // tile per CTA) they are faster than two 128 x 128 tiles per CTA, which stream 1.33x the operand bytes per FLOP from
  // L2.  Other staged fp32 outputs (whole 128 x 256 tiles would leave two operand stages) use 128 x 128 tiles.
  const bool gate_tma = tma_epi && epi == EPI_GATE_RESID_F32;
  const bool wide = (N % 256 == 0) && (gate_tma || (ceil_div(M, BM) * (N / 256) >= 2 * sms && !(tma_epi && out_f32)));
  const int BN = wide ? 256 : 128;
  CUtensorMap tmA, tmB, tmC;
  memset(&tmC, 0, sizeof(tmC));
  int rc = tmap_2d(&tmA, A, 2, M, K, ep.lda ? ep.lda : K, BM, BK);
  if (!rc) rc = tmap_2d(&tmB, W, 2, N, K, ep.ldb ? ep.ldb : K, BN, BK);
  // one box = one 128-byte column block x the 64 rows of a consumer warpgroup
  if (!rc && tma_epi) rc = tmap_2d(&tmC, ep.out, ob, M, N, ep.ldc, 64, 128 / ob);
  if (rc) return rc;
#define DGS_GEMM_CASE(E) \
  case E: return launch_epi<E>(wide, tma_epi, tmA, tmB, tmC, ep, M, N, K, st);
  switch (epi) {
    DGS_GEMM_CASE(EPI_BIAS_BF16)
    DGS_GEMM_CASE(EPI_BIAS_GELU_BF16)
    DGS_GEMM_CASE(EPI_GATE_RESID_F32)
    DGS_GEMM_CASE(EPI_F32)
    DGS_GEMM_CASE(EPI_DGELU_BF16)
    DGS_GEMM_CASE(EPI_BIAS_RELU_BF16)
    default:
      set_error("gemm: unknown epilogue %d", epi);
      return DGS_ERR_INVALID_ARGUMENT;
  }
#undef DGS_GEMM_CASE
}

// C[M, N] (fp32) = A^T W for A [K, M], W [K, N] bf16 row-major (lda / ldb = row strides in elements, 0 = M / N):
// the weight-gradient GEMM  dW[n_out, n_in] = dY[tokens, n_out]^T  X[tokens, n_in]  without transposed copies.
int gemm_bf16_tn(const void* A, const void* W, int M, int N, int K, const GemmEpilogue& ep, cudaStream_t st) {
  DGS_REQUIRE(M > 0 && N > 0 && K > 0, "gemm_tn: bad shape %dx%dx%d", M, N, K);
  const int lda = ep.lda ? ep.lda : M, ldb = ep.ldb ? ep.ldb : N, ldc = ep.ldc ? ep.ldc : N;
  DGS_REQUIRE(N % 32 == 0 && lda % 8 == 0 && ldb % 8 == 0, "gemm_tn: need N %% 32 == 0 and row strides %% 8 == 0");
  DGS_REQUIRE(((uintptr_t)A % 16) == 0 && ((uintptr_t)W % 16) == 0, "gemm_tn: operands must be 16-byte aligned");
  DGS_REQUIRE(lda >= M, "gemm_tn: lda=%d must be >= M=%d (or 0)", lda, M);
  DGS_REQUIRE(ldb >= N, "gemm_tn: ldb=%d must be >= N=%d (or 0)", ldb, N);
  DGS_REQUIRE(ldc >= N, "gemm_tn: ldc=%d must be >= N=%d (or 0)", ldc, N);
  const int sms = num_sms();
  const bool wide = (N % 256 == 0) && (ceil_div(M, BM) * (N / 256) >= sms);
  const int BN = wide ? 256 : 128;
  CUtensorMap tmA, tmB, tmC;
  memset(&tmC, 0, sizeof(tmC));  // unused: split-K partial sums are added from registers
  // [64 contiguous M/N elements (128 B) x 64 K rows]
  int rc = tmap_2d(&tmA, A, 2, K, M, lda, BK, 64);
  if (!rc) rc = tmap_2d(&tmB, W, 2, K, N, ldb, BK, 64);
  if (rc) return rc;
  // Split-K: the weight gradients have few output tiles (attn.proj: 64 of 128 x 128) but K = tokens is long, so K is cut
  // until the work units fill the SMs; every unit adds its partial sum into the zeroed output (fp32 atomics).
  const int tiles = ceil_div(M, BM) * ceil_div(N, BN), num_k = ceil_div(K, BK);
  int splits = 1;
  if (!ep.bias && tiles < sms && num_k >= 16 && (ldc % 2) == 0 && ((uintptr_t)ep.out % 8) == 0) {
    splits = ceil_div(sms, tiles);                      // ~1 wave of work units
    if (splits > num_k / 8) splits = num_k / 8;         // at least 8 k-blocks per unit
    splits = ceil_div(num_k, ceil_div(num_k, splits));  // no empty unit
  }
  GemmEpilogue e2 = ep;
  e2.ldc = ldc;
  if (splits > 1) DGS_CUDA_OK(cudaMemset2DAsync(ep.out, (size_t)ldc * 4, 0, (size_t)N * 4, (size_t)M, st));
  return wide ? launch_gemm<256, EPI_F32, OP_BF16_MN, false>(tmA, tmB, tmC, e2, M, N, K, st, splits)
              : launch_gemm<128, EPI_F32, OP_BF16_MN, false>(tmA, tmB, tmC, e2, M, N, K, st, splits);
}

int gemm_fp8(const void* A, const float* sa, const void* W, const float* sw, int M, int N, int K, int epi,
             const GemmEpilogue& ep, float* out_scale, cudaStream_t st) {
  DGS_REQUIRE(M > 0 && N > 0 && K > 0, "gemm_fp8: bad shape %dx%dx%d", M, N, K);
  DGS_REQUIRE(K % 128 == 0 && N % 128 == 0, "gemm_fp8: need K %% 128 == 0 and N %% 128 == 0 (got N=%d K=%d)", N, K);
  DGS_REQUIRE(epi == EPI_BIAS_BF16 || epi == EPI_GATE_RESID_F32 || epi == EPI_F32 || epi == EPI_BIAS_GELU_E4M3,
              "gemm_fp8: unsupported epilogue %d (0 bias -> bf16, 2 gate + residual, 3 fp32, 6 bias + GELU -> e4m3)", epi);
  DGS_REQUIRE(A && W && ep.out, "gemm_fp8: NULL operand or output");
  DGS_REQUIRE(sa && sw, "gemm_fp8: NULL scales (activation group scales and weight scales are required)");
  DGS_REQUIRE(epi != EPI_BIAS_GELU_E4M3 || out_scale, "gemm_fp8: the GELU -> e4m3 epilogue needs out_scale");
  DGS_REQUIRE(epi != EPI_GATE_RESID_F32 || (ep.gate && !ep.resid && !ep.aux),
              "gemm_fp8: the gate epilogue needs gate and runs in place only");
  DGS_REQUIRE(((uintptr_t)A % 16) == 0 && ((uintptr_t)W % 16) == 0 && ((uintptr_t)sa % 16) == 0 &&
                  ((uintptr_t)(out_scale) % 16) == 0 && ((uintptr_t)ep.out % 16) == 0,
              "gemm_fp8: operands, scales and output must be 16-byte aligned");
  const bool tma_epi = epi != EPI_F32;
  const int ob = epi_out_bytes(epi);
  DGS_REQUIRE(ep.ldc >= N && ((size_t)ep.ldc * ob) % 16 == 0, "gemm_fp8: output row stride %d must be >= N and 16-byte "
              "aligned", ep.ldc);
  const int sms = num_sms();
  DGS_REQUIRE(sms > 0, "gemm_fp8: cannot query the device's SM count");
  Fp8Scales fs;
  fs.sa = sa; fs.sw = sw; fs.out_scale = out_scale; fs.lds = fp8_scale_stride(M);
  CUtensorMap tmA, tmB, tmC;
  memset(&tmC, 0, sizeof(tmC));
  int rc = tmap_2d(&tmA, A, 1, M, K, K, BM, BK8);
  if (!rc) rc = tmap_2d(&tmB, W, 1, N, K, K, 128, BK8);
  if (!rc && tma_epi) rc = tmap_2d(&tmC, ep.out, ob, M, N, ep.ldc, 64, 128 / ob);
  if (rc) return rc;
  switch (epi) {
    case EPI_BIAS_BF16: return launch_gemm<128, EPI_BIAS_BF16, OP_E4M3, true>(tmA, tmB, tmC, ep, M, N, K, st, 1, fs);
    case EPI_GATE_RESID_F32: return launch_gemm<128, EPI_GATE_RESID_F32, OP_E4M3, true>(tmA, tmB, tmC, ep, M, N, K, st, 1, fs);
    case EPI_BIAS_GELU_E4M3: return launch_gemm<128, EPI_BIAS_GELU_E4M3, OP_E4M3, true>(tmA, tmB, tmC, ep, M, N, K, st, 1, fs);
    default: return launch_gemm<128, EPI_F32, OP_E4M3, false>(tmA, tmB, tmC, ep, M, N, K, st, 1, fs);
  }
}

}  // namespace dgs
