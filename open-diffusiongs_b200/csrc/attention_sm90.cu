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
#include "dgs_internal.h"
#include "dit_kernels.h"
#include "sm90_ptx.cuh"

namespace dgs {

using namespace ptx;

constexpr int ATT_BM = 128, ATT_BN = 128, ATT_HD = 64, ATT_KV_STAGES = 3, ATT_THREADS = WS_THREADS;
constexpr int ATT_Q_BYTES = ATT_BM * ATT_HD * 2;    // [128 x 64] bf16
constexpr int ATT_KV_BYTES = ATT_BN * ATT_HD * 2;   // [128 x 64] bf16 (one K or V block)
constexpr int ATT_SMEM_BYTES = ATT_Q_BYTES + 2 * ATT_KV_STAGES * ATT_KV_BYTES + 1024 + 256;

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

__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_fwd_kernel(const __grid_constant__ CUtensorMap tm_qkv, __nv_bfloat16* __restrict__ out, float* __restrict__ lse2,
                     int Np, int N, int H) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + ATT_Q_BYTES;
  uint8_t* sV = sK + ATT_KV_STAGES * ATT_KV_BYTES;
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sV + ATT_KV_STAGES * ATT_KV_BYTES);
  uint64_t* k_full = q_full + 1;
  uint64_t* v_full = k_full + ATT_KV_STAGES;
  uint64_t* k_empty = v_full + ATT_KV_STAGES;  // K and V of a stage are consumed (and released) one block apart
  uint64_t* v_empty = k_empty + ATT_KV_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * ATT_BM, h = blockIdx.y, b = blockIdx.z;
  const int n_blocks = (N + ATT_BN - 1) / ATT_BN;
  const int D = H * ATT_HD;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tm_qkv);
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
  const uint64_t qdesc = wg_desc_sw128(smem_u32(sQ + wg * 8192), 16, 1024);
  auto turn_wait = [&]() { named_bar_sync(1 + wg, 256); };   // my warpgroup may issue ...
  auto turn_pass = [&]() { named_bar_arrive(2 - wg, 256); }; // ... and now the other one may
  if (wg == 1) turn_pass();                                  // warpgroup 0 issues first
  auto issue_s = [&](float (&sc)[64], int s) {
#pragma unroll
    for (int i = 0; i < 64; i++) sc[i] = 0.f;
    const uint64_t kdesc = wg_desc_sw128(smem_u32(sK + s * ATT_KV_BYTES), 16, 1024);
    wg_fence();
#pragma unroll
    for (int k = 0; k < ATT_HD / 16; k++) wgmma_m64n128_ss<0, 0>(sc, qdesc + (uint64_t)(2 * k), kdesc + (uint64_t)(2 * k));
    wg_commit();
  };
  // B = V MN-major: rows = keys (128 B of 64 dims each), 16 keys = 2 groups of 8 rows = 2048 B per k16 slice
  auto issue_pv = [&](float (&o)[32], const uint32_t (&pa)[8][4], int s) {
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
  uint32_t pa[8][4];  // P_{j-1}, the A operand of the P V product in flight
  mbar_wait(q_full, 0);
  {  // prologue: S_0 -> P_0
    float sc[64];
    turn_wait();
    mbar_wait(k_full, 0);
    issue_s(sc, 0);
    turn_pass();
    wg_wait<0>();
    wg_fence_regs(sc);
    release(k_empty);
    att_softmax(sc, m_run, l_run, alpha, N, quad_col, sl2);  // alpha = 0, O is still 0
    att_pack_p(sc, pa);
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
    release(k_empty + s);
    att_softmax(sc, m_run, l_run, alpha, N - j * ATT_BN, quad_col, sl2);
    wg_wait<0>();  // P_{j-1} V_{j-1} is done: O and the P fragments may be rewritten
    wg_fence_regs(o);
    release(v_empty + sp);
#pragma unroll
    for (int jj = 0; jj < 8; jj++) {
      o[4 * jj + 0] *= alpha[0]; o[4 * jj + 1] *= alpha[0];
      o[4 * jj + 2] *= alpha[1]; o[4 * jj + 3] *= alpha[1];
    }
    att_pack_p(sc, pa);  // only now: redefining the A fragments of an in-flight wgmma makes ptxas serialise every wgmma
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
    const float inv = 1.0f / l_run[i];
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
    DGS_CUDA_OK(cudaFuncSetAttribute(attention_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM_BYTES));
    configured = true;
  }
  dim3 grid(ceil_div(N, ATT_BM), H, B);
  DGS_CUDA_OK(launch_pdl(attention_fwd_kernel, grid, dim3(ATT_THREADS), ATT_SMEM_BYTES, st, tm_qkv,
                         reinterpret_cast<__nv_bfloat16*>(out), lse2, Np, N, H));
  DGS_POST_LAUNCH();
  return DGS_OK;
}

}  // namespace dgs
