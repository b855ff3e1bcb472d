// attention_sm90.cu -- non-causal multi-head attention forward on wgmma (sm_90a), head_dim 64.
//
//   out[b, n, h*64:(h+1)*64] = softmax(q k^T / 8) v      (timm Attention.forward -> F.scaled_dot_product_attention,
//                                                         instantiated at utils_transformer.py:254-256)
// reading q/k/v straight out of the fused qkv GEMM output [B, N, 3, H, 64] (bf16) through ONE 3-D TMA tensor
// map (no head-major re-layout), N arbitrary (4098 = 32*128 + 2: the tail is zero-filled by TMA and masked).
//
// One CTA per (128-query block, head, sample), 384 threads:
//   warps 0..7  two consumer warpgroups, 64 query rows each.  Per 128-key block: S = Q K^T (wgmma, both operands from
//               shared memory, fp32 accumulators in registers) -> online softmax in registers (a row lives in the 4
//               threads of a quad) -> the bf16 probabilities are repacked into the A-operand fragments of the P V
//               wgmma (A from registers, V read MN-major from the same shared-memory tile layout as K), so P never
//               touches shared memory.  O accumulates in registers.  The loop is software-pipelined (the softmax of
//               block j runs while P_{j-1} V_{j-1} is in the tensor cores) and the two warpgroups issue their wgmma
//               in turns (ping-pong), so one warpgroup's softmax overlaps the other's MMAs.
//   warp 8      TMA producer: Q once, K/V blocks through a 3-stage ring with separate K and V release barriers
//               (warps 9..11 only give their registers away).
//
// Operand mode ATT_E4M3 (FP8 inference, dgs_attention_fwd_fp8): the same producer, ring, turns and pipelined loop on the
// e4m3 operands of attention_quantize_e4m3 (layouts in include/dgs_b200.h): S = Q K^T is two wgmma k32 steps on
// 64-byte-swizzled Q / K tiles, the softmax folds the scales into its one fmaf per score (c = sq[r] sk[j] / 8 * log2 e)
// and emits P = 2^(x c - m + 8) in [0, 256] straight into e4m3 A fragments (the +8 keeps small probabilities out of
// e4m3's subnormals and cancels in the final division), and P V reads the transposed, key-permuted V tile.  O is kept in
// units of the current block's V scale: the per-block rescale is alpha * sv[j-1] / sv[j], exact for powers of two.
#include "dgs_internal.h"
#include "dit_kernels.h"
#include "sm90_ptx.cuh"

namespace dgs {

using namespace ptx;

constexpr int ATT_BM = 128, ATT_BN = 128, ATT_HD = 64, ATT_KV_STAGES = 3, ATT_THREADS = WS_THREADS;
constexpr int ATT_Q_BYTES = ATT_BM * ATT_HD * 2;    // [128 x 64] bf16
constexpr int ATT_KV_BYTES = ATT_BN * ATT_HD * 2;   // [128 x 64] bf16 (one K or V block)
constexpr int ATT_SMEM_BYTES = ATT_Q_BYTES + 2 * ATT_KV_STAGES * ATT_KV_BYTES + 1024 + 256;
enum AttOperands { ATT_BF16 = 0, ATT_E4M3 = 1 };
// e4m3: Q / K tiles [128 x 64 B] (64-byte swizzle), V^T tiles [64 x 128 B] (128-byte swizzle), all 8 KB
constexpr int ATT8_TILE_BYTES = ATT_BM * ATT_HD;
// Every exponential of the e4m3 softmax runs on the MUFU pipe: moving a quarter or a half of them to a cubic polynomial
// on the FMA pipe was measured slower on the H100 (README, "FP8 attention"): the loop is bound by issue, not by MUFU.
constexpr int ATT8_SMEM_BYTES = 7 * ATT8_TILE_BYTES + 1024 + 256;

// What the e4m3 mode reads besides the Q map (the bf16 mode: nothing).
template <int OP>
struct AttExtra {};
template <>
struct AttExtra<ATT_E4M3> {
  CUtensorMap tm_k;   // k8 [B, N, H*64], 64-byte swizzle, box 64 x 128
  CUtensorMap tm_vt;  // vt8 [B*H*64, Nk], 128-byte swizzle, box 128 x 64
  const float* sq;    // [B, H, N]
  const float* sk;    // [B, H, Nk/128]
  const float* sv;    // [B, H, Nk/128]
  int nkb;            // Nk / 128
};

// Scores of one 128-key block -> online-softmax update of the row state, the probabilities overwrite the scores (fp32).
// Rows i = 0 (r0) and 1 (r0 + 8) of this thread: sc[4 jj + 2 i + e].  Returns alpha = 2^((m_old - m_new) * sl2), the
// factor O is rescaled by.
__device__ __forceinline__ void att_softmax(float (&sc)[64], float (&m_run)[2], float (&l_run)[2], float (&alpha)[2],
                                            int kv_valid, int quad_col, float sl2) {
  if (kv_valid < ATT_BN) {  // mask the zero-filled tail keys (last block only)
#pragma unroll
    for (int jj = 0; jj < 16; jj++)
#pragma unroll
      for (int e = 0; e < 4; e++)
        if (8 * jj + quad_col + (e & 1) >= kv_valid) sc[4 * jj + e] = -INFINITY;
  }
  float moff[2];
#pragma unroll
  for (int i = 0; i < 2; i++) {
    float mx = -INFINITY;
#pragma unroll
    for (int jj = 0; jj < 16; jj++) mx = fmaxf(mx, fmaxf(sc[4 * jj + 2 * i], sc[4 * jj + 2 * i + 1]));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    const float m_new = fmaxf(m_run[i], mx);           // finite: every block has at least one valid key
    alpha[i] = ex2_approx((m_run[i] - m_new) * sl2);   // 0 on the first block (m_run = -inf)
    m_run[i] = m_new;
    moff[i] = m_new * sl2;
  }
  float ls[2] = {0.f, 0.f};
#pragma unroll
  for (int kk = 0; kk < 8; kk++) {
#pragma unroll
    for (int q = 0; q < 4; q++) {  // fragment register q: row i = q & 1, keys 16 kk + 8 (q >> 1) + quad_col + {0, 1}
      const int idx = 8 * kk + 4 * (q >> 1) + 2 * (q & 1);
      const float p0 = ex2_approx(fmaf(sc[idx], sl2, -moff[q & 1]));
      const float p1 = ex2_approx(fmaf(sc[idx + 1], sl2, -moff[q & 1]));
      ls[q & 1] += p0 + p1;  // row sums of the fp32 probabilities, before the bf16 rounding
      sc[idx] = p0;
      sc[idx + 1] = p1;
    }
  }
#pragma unroll
  for (int i = 0; i < 2; i++) l_run[i] = l_run[i] * alpha[i] + ls[i];
}
// P as the A fragments of the 8 k16 slices of the P V product: fragment register q of slice kk holds row q & 1, keys
// 16 kk + 8 (q >> 1) + quad_col + {0, 1}.
__device__ __forceinline__ void att_pack_p(const float (&sc)[64], uint32_t (&pa)[8][4]) {
#pragma unroll
  for (int kk = 0; kk < 8; kk++)
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const int idx = 8 * kk + 4 * (q >> 1) + 2 * (q & 1);
      pa[kk][q] = pack2_bf16(sc[idx], sc[idx + 1]);
    }
}

// att_softmax for raw e4m3 scores: the score of row i is sc * c[i] (log2 units), m_run is kept in the same units, and
// the probabilities are 2^(sc c - m + 8).  Returns alpha = 2^(m_old - m_new).
__device__ __forceinline__ void att_softmax_e4m3(float (&sc)[64], float (&m_run)[2], float (&l_run)[2],
                                                 float (&alpha)[2], int kv_valid, int quad_col, const float (&c)[2]) {
  if (kv_valid < ATT_BN) {
#pragma unroll
    for (int jj = 0; jj < 16; jj++)
#pragma unroll
      for (int e = 0; e < 4; e++)
        if (8 * jj + quad_col + (e & 1) >= kv_valid) sc[4 * jj + e] = -INFINITY;
  }
  float moff[2];
#pragma unroll
  for (int i = 0; i < 2; i++) {
    float mx = -INFINITY;
#pragma unroll
    for (int jj = 0; jj < 16; jj++) mx = fmaxf(mx, fmaxf(sc[4 * jj + 2 * i], sc[4 * jj + 2 * i + 1]));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    const float m_new = fmaxf(m_run[i], mx * c[i]);  // c > 0: the max of the scaled scores
    alpha[i] = ex2_approx(m_run[i] - m_new);
    m_run[i] = m_new;
    moff[i] = m_new - 8.0f;
  }
  float ls[2] = {0.f, 0.f};
#pragma unroll
  for (int jj = 0; jj < 16; jj++)
#pragma unroll
    for (int e = 0; e < 4; e++) {
      const int i = e >> 1;
      const float p = ex2_approx(fmaf(sc[4 * jj + e], c[i], -moff[i]));
      ls[i] += p;  // row sums of the fp32 probabilities, before the e4m3 rounding
      sc[4 * jj + e] = p;
    }
#pragma unroll
  for (int i = 0; i < 2; i++) l_run[i] = l_run[i] * alpha[i] + ls[i];
}
// P as the e4m3 A fragments of the 4 k32 slices.  The thread holds keys {2u, 2u+1, 8+2u, 9+2u} of every 16 (u = lane % 4)
// and register q of slice kk takes A's k = 4u..4u+3 of the 16-key group 2 kk + (q >> 1) for row q & 1: vt8 stores the
// keys of every 16 in that order (key_of_slot in attention_quantize_e4m3_kernel), so no quad shuffles are needed.
__device__ __forceinline__ void att_pack_p_e4m3(const float (&sc)[64], uint32_t (&pa)[4][4]) {
#pragma unroll
  for (int kk = 0; kk < 4; kk++)
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const int i0 = 4 * (4 * kk + 2 * (q >> 1)) + 2 * (q & 1);  // n8 block 2 g, then 2 g + 1 (4 registers on)
      pa[kk][q] = (uint32_t)pack2_e4m3(sc[i0], sc[i0 + 1]) | ((uint32_t)pack2_e4m3(sc[i0 + 4], sc[i0 + 5]) << 16);
    }
}

// OP = ATT_BF16: tm_qkv maps the bf16 qkv [B, N, 3, H, 64]; OP = ATT_E4M3: tm_qkv maps q8, x the rest (lse2 unused).
template <int OP>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_fwd_kernel(const __grid_constant__ CUtensorMap tm_qkv, __nv_bfloat16* __restrict__ out, float* __restrict__ lse2,
                     int Np, int N, int H, const __grid_constant__ AttExtra<OP> x) {
  constexpr bool E4M3 = OP == ATT_E4M3;
  constexpr int Q_BYTES = E4M3 ? ATT8_TILE_BYTES : ATT_Q_BYTES, KV_BYTES = E4M3 ? ATT8_TILE_BYTES : ATT_KV_BYTES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Q_BYTES;
  uint8_t* sV = sK + ATT_KV_STAGES * KV_BYTES;
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sV + ATT_KV_STAGES * KV_BYTES);
  uint64_t* k_full = q_full + 1;
  uint64_t* v_full = k_full + ATT_KV_STAGES;
  uint64_t* k_empty = v_full + ATT_KV_STAGES;  // K and V of a stage are consumed (and released) one block apart
  uint64_t* v_empty = k_empty + ATT_KV_STAGES;
  float2* kv_scale = reinterpret_cast<float2*>(v_empty + ATT_KV_STAGES);  // e4m3: (sk, sv) of the block in K stage s

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * ATT_BM, h = blockIdx.y, b = blockIdx.z;
  const int n_blocks = (N + ATT_BN - 1) / ATT_BN;
  const int D = H * ATT_HD;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tm_qkv);
    if constexpr (E4M3) {
      prefetch_tmap(&x.tm_k);
      prefetch_tmap(&x.tm_vt);
    }
    mbar_init(q_full, 1);
    for (int s = 0; s < ATT_KV_STAGES; s++) {
      mbar_init(k_full + s, 1); mbar_init(v_full + s, 1); mbar_init(k_empty + s, 8); mbar_init(v_empty + s, 8);
    }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_launch_dependents();  // programmatic dependent launch: the next kernel may start its prologue now ...
  griddep_wait();               // ... and this one touches global memory only after its predecessor has completed

  if (warp >= 8) {
    // ===================== TMA producer =====================
    ws_producer_regs();
    if constexpr (E4M3) {
      if (warp == 8 && lane == 0) {
        const size_t sb = ((size_t)b * H + h) * x.nkb;
        mbar_arrive_expect_tx(q_full, Q_BYTES);
        tma_load_3d(sQ, &tm_qkv, q_full, h * ATT_HD, q0, b);
        for (int j = 0; j < n_blocks; j++) {
          const int s = j % ATT_KV_STAGES;
          const uint32_t ph = ((uint32_t)(j / ATT_KV_STAGES) & 1) ^ 1;
          mbar_wait(k_empty + s, ph);
          kv_scale[s] = make_float2(x.sk[sb + j], x.sv[sb + j]);  // published by the k_full arrive (release)
          mbar_arrive_expect_tx(k_full + s, KV_BYTES);
          tma_load_3d(sK + s * KV_BYTES, &x.tm_k, k_full + s, h * ATT_HD, j * ATT_BN, b);
          mbar_wait(v_empty + s, ph);
          mbar_arrive_expect_tx(v_full + s, KV_BYTES);
          tma_load_2d(sV + s * KV_BYTES, &x.tm_vt, v_full + s, j * ATT_BN, (b * H + h) * ATT_HD);
        }
      }
      return;
    }
    if (warp == 8 && lane == 0) {
      mbar_arrive_expect_tx(q_full, ATT_Q_BYTES);
      tma_load_3d(sQ, &tm_qkv, q_full, h * ATT_HD, q0, b);
      for (int j = 0; j < n_blocks; j++) {
        const int s = j % ATT_KV_STAGES;
        const uint32_t ph = ((uint32_t)(j / ATT_KV_STAGES) & 1) ^ 1;
        mbar_wait(k_empty + s, ph);
        mbar_arrive_expect_tx(k_full + s, ATT_KV_BYTES);
        tma_load_3d(sK + s * ATT_KV_BYTES, &tm_qkv, k_full + s, D + h * ATT_HD, j * ATT_BN, b);
        mbar_wait(v_empty + s, ph);
        mbar_arrive_expect_tx(v_full + s, ATT_KV_BYTES);
        tma_load_3d(sV + s * ATT_KV_BYTES, &tm_qkv, v_full + s, 2 * D + h * ATT_HD, j * ATT_BN, b);
      }
    }
    return;
  }

  // ===================== consumers: warpgroup wg owns query rows [64 wg, 64 wg + 64) =====================
  // Software pipeline: iteration j issues S_j = Q K_j^T and O += P_{j-1} V_{j-1} back to back, then runs the softmax
  // of S_j while the tensor cores still work on P_{j-1} V_{j-1}.  On top of that the two warpgroups take turns to issue
  // (named barriers 1 and 2), so one warpgroup's softmax runs under the other's MMAs.  Every warpgroup walks all key
  // blocks, also when its rows are past N, so both take the same number of turns.
  ws_consumer_regs();
  const int wg = warp >> 2;
  const int quad_col = 2 * (lane & 3);                      // first key / dim column of this thread in every n8 block
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // rows r0 and r0 + 8 of the 128-query block
  const float sl2 = 0.125f * 1.4426950408889634f;           // 1/sqrt(64) * log2(e)
  const uint64_t qdesc = E4M3 ? wg_desc_sw64(smem_u32(sQ + wg * 4096), 512) : wg_desc_sw128(smem_u32(sQ + wg * 8192), 16, 1024);
  auto turn_wait = [&]() { named_bar_sync(1 + wg, 256); };   // my warpgroup may issue ...
  auto turn_pass = [&]() { named_bar_arrive(2 - wg, 256); }; // ... and now the other one may
  if (wg == 1) turn_pass();                                  // warpgroup 0 issues first
  auto issue_s = [&](float (&sc)[64], int s) {
    if constexpr (E4M3) {  // K = 64 e4m3 = two k32 steps; the first overwrites sc
      const uint64_t kdesc = wg_desc_sw64(smem_u32(sK + s * KV_BYTES), 512);
      wg_fence();
      wgmma_m64n128k32_e4m3(sc, qdesc, kdesc, 0);
      wgmma_m64n128k32_e4m3(sc, qdesc + 2, kdesc + 2, 1);
      wg_commit();
    } else {
#pragma unroll
      for (int i = 0; i < 64; i++) sc[i] = 0.f;
      const uint64_t kdesc = wg_desc_sw128(smem_u32(sK + s * ATT_KV_BYTES), 16, 1024);
      wg_fence();
#pragma unroll
      for (int k = 0; k < ATT_HD / 16; k++) wgmma_m64n128_ss<0, 0>(sc, qdesc + (uint64_t)(2 * k), kdesc + (uint64_t)(2 * k));
      wg_commit();
    }
  };
  // B = V MN-major: rows = keys (128 B of 64 dims each), 16 keys = 2 groups of 8 rows = 2048 B per k16 slice
  // e4m3: B = the V^T tile K-major, rows = head dims (128 B of 128 keys each), one k32 slice = 32 B along the row
  auto issue_pv = [&](float (&o)[32], const auto& pa, int s) {
    if constexpr (E4M3) {
      const uint64_t vdesc = wg_desc_sw128(smem_u32(sV + s * KV_BYTES), 16, 1024);
      wg_fence();
#pragma unroll
      for (int kk = 0; kk < 4; kk++) wgmma_m64n64k32_e4m3_rs(o, pa[kk], vdesc + (uint64_t)(2 * kk));
      wg_commit();
      return;
    }
    const uint64_t vdesc = wg_desc_sw128(smem_u32(sV + s * ATT_KV_BYTES), 8192, 1024);
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < 8; kk++) wgmma_m64n64_rs<1>(o, pa[kk], vdesc + (uint64_t)(128 * kk));
    wg_commit();
  };
  auto release = [&](uint64_t* bar) {
    __syncwarp();
    if (lane == 0) mbar_arrive(bar);
  };

  float o[32];
#pragma unroll
  for (int i = 0; i < 32; i++) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f}, alpha[2];
  uint32_t pa[E4M3 ? 4 : 8][4];  // P_{j-1}, the A operand of the P V product in flight
  // e4m3: the score factor of rows r0 / r0 + 8 without the block's K scale, and the V scale O is currently in units of
  float cq[2] = {0.f, 0.f}, sv_cur = 1.f;
  if constexpr (E4M3) {
#pragma unroll
    for (int i = 0; i < 2; i++) {
      const int q = q0 + r0 + 8 * i;
      cq[i] = (q < N ? x.sq[((size_t)b * H + h) * N + q] : 1.f) * sl2;
    }
  }
  // e4m3: this block's score factors and V scale, read before the K stage is released
  auto block_scales = [&](float (&c)[2], float& svj, int s) {
    const float2 ks = kv_scale[s];
    c[0] = cq[0] * ks.x; c[1] = cq[1] * ks.x;
    svj = ks.y;
  };
  mbar_wait(q_full, 0);
  {  // prologue: S_0 -> P_0
    float sc[64];
    turn_wait();
    mbar_wait(k_full, 0);
    issue_s(sc, 0);
    turn_pass();
    wg_wait<0>();
    wg_fence_regs(sc);
    if constexpr (E4M3) {
      float c[2];
      block_scales(c, sv_cur, 0);
      release(k_empty);
      att_softmax_e4m3(sc, m_run, l_run, alpha, N, quad_col, c);
      att_pack_p_e4m3(sc, pa);
    } else {
      release(k_empty);
      att_softmax(sc, m_run, l_run, alpha, N, quad_col, sl2);  // alpha = 0, O is still 0
      att_pack_p(sc, pa);
    }
  }
  for (int j = 1; j < n_blocks; j++) {
    const int s = j % ATT_KV_STAGES, sp = (j - 1) % ATT_KV_STAGES;
    float sc[64];
    turn_wait();
    mbar_wait(k_full + s, (uint32_t)(j / ATT_KV_STAGES) & 1);
    issue_s(sc, s);
    mbar_wait(v_full + sp, (uint32_t)((j - 1) / ATT_KV_STAGES) & 1);
    issue_pv(o, pa, sp);
    turn_pass();
    wg_wait<1>();  // S_j is ready; P_{j-1} V_{j-1} may still run
    wg_fence_regs(sc);
    if constexpr (E4M3) {
      float c[2], svj;
      block_scales(c, svj, s);
      release(k_empty + s);
      att_softmax_e4m3(sc, m_run, l_run, alpha, N - j * ATT_BN, quad_col, c);
      // O from units of sv[j-1] into units of sv[j]: sv[j-1] / sv[j] from the exponent bits (both are powers of two;
      // no division, whose slow path is a call that would serialise the wgmma pipeline)
      const float rebase = __int_as_float(__float_as_int(sv_cur) - __float_as_int(svj) + (127 << 23));
      alpha[0] *= rebase; alpha[1] *= rebase;
      sv_cur = svj;
    } else {
      release(k_empty + s);
      att_softmax(sc, m_run, l_run, alpha, N - j * ATT_BN, quad_col, sl2);
    }
    wg_wait<0>();  // P_{j-1} V_{j-1} is done: O and the P fragments may be rewritten
    wg_fence_regs(o);
    release(v_empty + sp);
#pragma unroll
    for (int jj = 0; jj < 8; jj++) {
      o[4 * jj + 0] *= alpha[0]; o[4 * jj + 1] *= alpha[0];
      o[4 * jj + 2] *= alpha[1]; o[4 * jj + 3] *= alpha[1];
    }
    if constexpr (E4M3) att_pack_p_e4m3(sc, pa);
    else att_pack_p(sc, pa);  // only now: redefining the A fragments of an in-flight wgmma makes ptxas serialise every wgmma
  }
  {  // epilogue: the last P V
    const int sl = (n_blocks - 1) % ATT_KV_STAGES;
    turn_wait();
    mbar_wait(v_full + sl, (uint32_t)((n_blocks - 1) / ATT_KV_STAGES) & 1);
    issue_pv(o, pa, sl);
    if (wg == 0) turn_pass();  // warpgroup 1 takes no further turn
    wg_wait<0>();
    wg_fence_regs(o);
    release(v_empty + sl);
  }
  // all blocks accumulated -> normalise and store
#pragma unroll
  for (int i = 0; i < 2; i++) {
    l_run[i] += __shfl_xor_sync(0xffffffffu, l_run[i], 1);
    l_run[i] += __shfl_xor_sync(0xffffffffu, l_run[i], 2);
  }
#pragma unroll
  for (int i = 0; i < 2; i++) {
    const int q = q0 + r0 + 8 * i;
    if (q >= N) continue;
    // training: log2-domain log-sum-exp of the scaled scores, consumed by attention_bwd_sm90.cu
    if (lse2 && (lane & 3) == 0) lse2[((size_t)b * H + h) * Np + q] = fmaf(m_run[i], sl2, log2f(l_run[i]));
    const float inv = E4M3 ? sv_cur / l_run[i] : 1.0f / l_run[i];
    __nv_bfloat16* dst = out + ((size_t)b * N + q) * D + h * ATT_HD + quad_col;
#pragma unroll
    for (int jj = 0; jj < 8; jj++)
      *reinterpret_cast<uint32_t*>(dst + 8 * jj) = pack2_bf16(o[4 * jj + 2 * i] * inv, o[4 * jj + 2 * i + 1] * inv);
  }
}

int attention_fwd(const void* qkv, void* out, float* lse2, int B, int N, int H, cudaStream_t st) {
  DGS_REQUIRE(B > 0 && N > 0 && H > 0, "attention: bad shape B=%d N=%d H=%d", B, N, H);
  const int D = H * ATT_HD;
  const int Np = attention_lse_stride(N);
  CUtensorMap tm_qkv;
  uint64_t dims[3] = {(uint64_t)(3 * D), (uint64_t)N, (uint64_t)B};
  uint64_t str[2] = {(uint64_t)(3 * D) * 2, (uint64_t)N * 3 * D * 2};
  uint32_t box[3] = {ATT_HD, ATT_BM, 1};  // = ATT_BN rows: one map serves the Q, K and V tiles
  int rc = make_tmap_bf16(&tm_qkv, qkv, 3, dims, str, box);
  if (rc) return rc;
  static bool configured = false;
  if (!configured) {
    DGS_CUDA_OK(cudaFuncSetAttribute(attention_fwd_kernel<ATT_BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     ATT_SMEM_BYTES));
    configured = true;
  }
  dim3 grid(ceil_div(N, ATT_BM), H, B);
  DGS_CUDA_OK(launch_pdl(attention_fwd_kernel<ATT_BF16>, grid, dim3(ATT_THREADS), ATT_SMEM_BYTES, st, tm_qkv,
                         reinterpret_cast<__nv_bfloat16*>(out), lse2, Np, N, H, AttExtra<ATT_BF16>{}));
  DGS_POST_LAUNCH();
  return DGS_OK;
}

// ---- FP8 (e4m3) operands --------------------------------------------------------------------------------------------
// Slot a of every 16 keys of vt8 holds key key_of_slot(a): the fp32 S accumulator gives a thread keys {2u, 2u+1, 8+2u,
// 9+2u} of every 16, the e4m3 A fragment wants k = 4u..4u+3 from it (wgmma .m64nNk32 register fragments), so slot 4u + v
// holds the v-th of those keys.  Permuting the contraction index on both sides of P V leaves the product exact.
__device__ __forceinline__ int key_of_slot(int a) { return 2 * (a >> 2) + (a & 1) + 8 * ((a >> 1) & 1); }

// One CTA per (128-token block, head, sample), 256 threads; thread t handles token t / 2, head dims 32 (t % 2) + [0, 32).
__global__ void __launch_bounds__(256)
attention_quantize_e4m3_kernel(const __nv_bfloat16* __restrict__ qkv, uint8_t* __restrict__ q8, uint8_t* __restrict__ k8,
                               uint8_t* __restrict__ vt8, float* __restrict__ sq, float* __restrict__ sk,
                               float* __restrict__ sv, int N, int H) {
  __shared__ float s_v[ATT_BN][ATT_HD + 1];
  __shared__ float s_red[2][8];
  const int blk = blockIdx.x, h = blockIdx.y, b = blockIdx.z, t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int row = t >> 1, c0 = 32 * (t & 1), n = blk * ATT_BN + row, D = H * ATT_HD, nkb = gridDim.x;
  const bool valid = n < N;
  float v[3][32];  // q, k, v (zeros past N)
  float amax[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int m = 0; m < 3; m++) {
    const __nv_bfloat16* src = qkv + ((size_t)b * N + n) * 3 * D + m * D + h * ATT_HD + c0;
#pragma unroll
    for (int c = 0; c < 32; c += 8) {
      uint4 u = make_uint4(0u, 0u, 0u, 0u);
      if (valid) u = *reinterpret_cast<const uint4*>(src + c);
      const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(&u);
#pragma unroll
      for (int i = 0; i < 8; i++) {
        v[m][c + i] = __bfloat162float(e[i]);
        amax[m] = fmaxf(amax[m], fabsf(v[m][c + i]));
      }
    }
  }
  auto store_row = [&](uint8_t* dst, const float (&x)[32], float inv) {  // 32 e4m3 bytes
    uint32_t w[8];
#pragma unroll
    for (int i = 0; i < 8; i++)
      w[i] = (uint32_t)pack2_e4m3(x[4 * i] * inv, x[4 * i + 1] * inv) |
             ((uint32_t)pack2_e4m3(x[4 * i + 2] * inv, x[4 * i + 3] * inv) << 16);
    reinterpret_cast<uint4*>(dst)[0] = make_uint4(w[0], w[1], w[2], w[3]);
    reinterpret_cast<uint4*>(dst)[1] = make_uint4(w[4], w[5], w[6], w[7]);
  };
  // q: one scale per (token, head)
  const int eq = e4m3_scale_exp(fmaxf(amax[0], __shfl_xor_sync(0xffffffffu, amax[0], 1)));
  if (valid) {
    if (c0 == 0) sq[((size_t)b * H + h) * N + n] = exp2_int(eq);
    store_row(q8 + ((size_t)b * N + n) * D + h * ATT_HD + c0, v[0], exp2_int(-eq));
  }
  // k, v: one scale per (128-key block, head) over the valid keys
#pragma unroll
  for (int m = 1; m < 3; m++) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax[m] = fmaxf(amax[m], __shfl_xor_sync(0xffffffffu, amax[m], o));
    if (lane == 0) s_red[m - 1][warp] = amax[m];
  }
#pragma unroll
  for (int c = 0; c < 32; c++) s_v[row][c0 + c] = v[2][c];
  __syncthreads();
  float bk = 0.f, bv = 0.f;
#pragma unroll
  for (int w = 0; w < 8; w++) { bk = fmaxf(bk, s_red[0][w]); bv = fmaxf(bv, s_red[1][w]); }
  const int ek = e4m3_scale_exp(bk), ev = e4m3_scale_exp(bv);
  if (t == 0) {
    sk[((size_t)b * H + h) * nkb + blk] = exp2_int(ek);
    sv[((size_t)b * H + h) * nkb + blk] = exp2_int(ev);
  }
  if (valid) store_row(k8 + ((size_t)b * N + n) * D + h * ATT_HD + c0, v[1], exp2_int(-ek));
  // vt8 row d = t / 4, slots 32 (t % 4) + [0, 32) of this block (pad keys are the zeros loaded above)
  const int d = t >> 2, a0 = 32 * (t & 3);
  float xv[32];
#pragma unroll
  for (int a = 0; a < 32; a++) xv[a] = s_v[a0 + (a & ~15) + key_of_slot(a & 15)][d];
  store_row(vt8 + (((size_t)b * H + h) * ATT_HD + d) * ((size_t)nkb * ATT_BN) + blk * ATT_BN + a0, xv, exp2_int(-ev));
}

int attention_quantize_e4m3(const void* qkv, uint8_t* q8, uint8_t* k8, uint8_t* vt8, float* sq, float* sk, float* sv,
                            int B, int N, int H, cudaStream_t st) {
  DGS_REQUIRE(B > 0 && N > 0 && H > 0, "attention quantize: bad shape B=%d N=%d H=%d", B, N, H);
  dim3 grid(ceil_div(N, ATT_BN), H, B);
  attention_quantize_e4m3_kernel<<<grid, 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(qkv), q8, k8, vt8, sq, sk,
                                                         sv, N, H);
  DGS_POST_LAUNCH();
  return DGS_OK;
}

int attention_fwd_e4m3(const uint8_t* q8, const uint8_t* k8, const uint8_t* vt8, const float* sq, const float* sk,
                       const float* sv, void* out, int B, int N, int H, cudaStream_t st) {
  DGS_REQUIRE(B > 0 && N > 0 && H > 0, "attention fp8: bad shape B=%d N=%d H=%d", B, N, H);
  const int D = H * ATT_HD, nkb = ceil_div(N, ATT_BN);
  CUtensorMap tm_q;
  AttExtra<ATT_E4M3> x;
  {
    uint64_t dims[3] = {(uint64_t)D, (uint64_t)N, (uint64_t)B};
    uint64_t str[2] = {(uint64_t)D, (uint64_t)N * D};
    uint32_t box[3] = {ATT_HD, ATT_BM, 1};
    int rc = make_tmap(&tm_q, CU_TENSOR_MAP_DATA_TYPE_UINT8, q8, 3, dims, str, box, CU_TENSOR_MAP_SWIZZLE_64B);
    if (rc) return rc;
    rc = make_tmap(&x.tm_k, CU_TENSOR_MAP_DATA_TYPE_UINT8, k8, 3, dims, str, box, CU_TENSOR_MAP_SWIZZLE_64B);
    if (rc) return rc;
  }
  {
    uint64_t dims[2] = {(uint64_t)nkb * ATT_BN, (uint64_t)B * H * ATT_HD};
    uint64_t str[1] = {(uint64_t)nkb * ATT_BN};
    uint32_t box[2] = {ATT_BN, ATT_HD};
    int rc = make_tmap(&x.tm_vt, CU_TENSOR_MAP_DATA_TYPE_UINT8, vt8, 2, dims, str, box);
    if (rc) return rc;
  }
  x.sq = sq; x.sk = sk; x.sv = sv; x.nkb = nkb;
  static bool configured = false;
  if (!configured) {
    DGS_CUDA_OK(cudaFuncSetAttribute(attention_fwd_kernel<ATT_E4M3>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     ATT8_SMEM_BYTES));
    configured = true;
  }
  dim3 grid(ceil_div(N, ATT_BM), H, B);
  DGS_CUDA_OK(launch_pdl(attention_fwd_kernel<ATT_E4M3>, grid, dim3(ATT_THREADS), ATT8_SMEM_BYTES, st, tm_q,
                         reinterpret_cast<__nv_bfloat16*>(out), (float*)nullptr, 0, N, H, x));
  DGS_POST_LAUNCH();
  return DGS_OK;
}

}  // namespace dgs
