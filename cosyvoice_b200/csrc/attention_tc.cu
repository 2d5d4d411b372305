// bf16 self-attention on Hopper tensor cores (wgmma) for the flow estimator (matcha transformer.py:243-316 via diffusers
// Attention; flow/decoder.py:439-449): head_dim 64, ragged sequences, full or block-causal (chunk) masking, and the conformer
// relative-position attention of the encoder.
#include "common.cuh"
#include "wgmma.cuh"
#include "tma.cuh"

namespace {

constexpr int AT_BQ = 128, AT_BK = 64, AT_HD = 64;    // 128 queries x 64-key tiles
constexpr int AT_KVST = 3;                             // K/V stages (one key tile each)
constexpr int AT_THREADS = 256;   // attn_wg_kernel: warpgroups 0-1, 64 queries each (MMA + softmax); thread 0 also issues the TMA loads
constexpr int RP_THREADS = 384;   // relpos_u_kernel: warp 0 TMA producer; warpgroups 1-2 consumers
constexpr uint32_t Q_BYTES = AT_BQ * AT_HD * 2;        // 16 KB
constexpr uint32_t K_BYTES = AT_BK * AT_HD * 2;        // 8 KB
constexpr uint32_t V_BYTES = AT_BK * AT_HD * 2;        // 8 KB
constexpr uint32_t KV_STAGE = K_BYTES + V_BYTES;       // 16 KB

constexpr uint32_t AT_SMEM = Q_BYTES + AT_KVST * KV_STAGE + 1024;   // 65 KB

// One CTA = 128 queries of one (sequence, head), 256 threads: warpgroups 0 and 1 own 64 queries each, and thread 0 also issues
// the TMA loads (Q once, then K/V 64-key tiles through a three-stage ring).  Without a producer warp the plain kernel fits in 128
// registers, so two CTAs share an SM and one CTA's softmax runs under the other's MMAs.  Per key tile a consumer warpgroup computes
// S = Q K^T (wgmma, 64 x 64 fp32 in registers), applies mask / bias and an online softmax in registers (the four threads of a
// quad share a row: row maxima and sums are quad shuffles), rescales its O accumulator and issues O += P V with P taken straight
// from the S registers (the accumulator layout of S is the register A-operand layout of the P V MMA) and V consumed MN-major
// from the TMA tile (transposed-B wgmma), so no transpose is ever materialised.
// BIAS: an additive score term read from global memory, bias(i, j) = ubias[((s0 + i) * H + h) * ldu + ucenter - i + j]: the
// relative-position term of the conformer attention (transformer/attention.py:249-330), where row t of U = (q + pos_bias_v) p[t]^T
// has been produced by relpos_u_kernel and the reference's rel_shift (attention.py:225-247) is the index map (i, j) -> center - (i - j).
// Work that cannot change a stored row is skipped: a warpgroup whose 64 rows all lie at or past L returns at once (the K/V stages
// are then released by the 4 warps that consume), and the key mask / -inf select run only on the key tiles that reach past the
// smallest key limit of the warp's 16 rows.  Every stored value goes through the same operations in the same order either way.
// The row sum takes the rescale and the tile's first P in one fma, lsum = fma(lsum, f, p) + p' + ...: the rounding this kernel
// has always had (the compiler contracted lsum * f + p), written out so that changes around it cannot move the contraction.
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 h2 = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h2);
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

template <bool BIAS>
__global__ void __launch_bounds__(AT_THREADS, BIAS ? 1 : 2)
attn_wg_kernel(const __grid_constant__ CUtensorMap tmq, const __grid_constant__ CUtensorMap tmk, const __grid_constant__ CUtensorMap tmv,
               const int* __restrict__ start, const int* __restrict__ len, int chunk, float scale_log2e, int kv_div,
               bf16* __restrict__ out, int ldo, const int* __restrict__ kstart, const int* __restrict__ klen, const int* __restrict__ qoff,
               const float* __restrict__ ubias, int ldu, int ucenter) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_q;
  __shared__ __align__(8) uint64_t bar_full[AT_KVST], bar_empty[AT_KVST];   // K/V stages

  const int b = blockIdx.z, h = blockIdx.y;
  const int L = len[b], s0 = start[b];            // query rows
  const int Lk = klen ? klen[b] : L, ks0 = kstart ? kstart[b] : s0, q0 = qoff ? qoff[b] : 0;   // key rows (cache geometry); position of query 0
  const int i0 = blockIdx.x * AT_BQ;
  if (i0 >= L) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = base, sKV = base + Q_BYTES;
  // keys visible to this query tile: all of the sequence, or up to the end of the last query's chunk
  const int i_last = q0 + min(i0 + AT_BQ, L) - 1;
  const int kmax = chunk > 0 ? min(Lk, (i_last / chunk + 1) * chunk) : Lk;
  const int G = (kmax + AT_BK - 1) / AT_BK;
  const int wg = threadIdx.x >> 7;      // warpgroup 0 always has a valid row (i0 < L); warpgroup 1 only if i0 + 64 < L

  if (threadIdx.x == 0) {
    mbar_init(smem_u32(&bar_q), 1);
    for (int s = 0; s < AT_KVST; ++s) {
      mbar_init(smem_u32(&bar_full[s]), 1);
      mbar_init(smem_u32(&bar_empty[s]), i0 + 64 < L ? 8 : 4);     // one arrival per consuming warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (i0 + wg * 64 >= L) return;        // all 64 rows padded: nothing of this warpgroup is stored

  // Thread 0 produces: Q once, then K/V tile t into stage t % AT_KVST once every consuming warp has released the tile t - AT_KVST
  // that used it.  It blocks on that release only when the consumers need tile t now (t == g); otherwise it tries again later.
  int nx = 0;                           // next K/V tile to load (thread 0)
  auto produce = [&](int g) {
    for (; nx < G && nx < g + AT_KVST; ++nx) {
      const int st = nx % AT_KVST;
      const uint32_t eb = smem_u32(&bar_empty[st]), par = (uint32_t)(((nx / AT_KVST) & 1) ^ 1);
      if (nx > g) {
        if (!mbar_test(eb, par)) break;
      } else {
        mbar_wait(eb, par);
      }
      const uint32_t fb = smem_u32(&bar_full[st]);
      mbar_expect_tx(fb, KV_STAGE);
      tma_load_2d(sKV + st * KV_STAGE, &tmk, fb, (h / kv_div) * AT_HD, ks0 + nx * AT_BK);
      tma_load_2d(sKV + st * KV_STAGE + K_BYTES, &tmv, fb, (h / kv_div) * AT_HD, ks0 + nx * AT_BK);
    }
  };
  if (threadIdx.x == 0) {
    mbar_expect_tx(smem_u32(&bar_q), Q_BYTES);
    tma_load_2d(sQ, &tmq, smem_u32(&bar_q), h * AT_HD, s0 + i0);
  }

  const int q = lane & 3;
  const int rbase = wg * 64 + (warp & 3) * 16 + (lane >> 2);     // tile rows rbase (h = 0) and rbase + 8 (h = 1)
  int ii[2], klim[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    ii[hh] = i0 + rbase + 8 * hh;
    klim[hh] = ii[hh] < L ? (chunk > 0 ? min(Lk, ((q0 + ii[hh]) / chunk + 1) * chunk) : Lk) : 0;
  }
  // key tiles that end at or before the smallest key limit of the warp's 16 rows need no mask (warp-uniform)
  const int kfree = __reduce_min_sync(0xffffffffu, min(klim[0], klim[1]));
  const uint64_t dq = wg_desc_sw128(sQ + (uint32_t)wg * (Q_BYTES / 2));
  float o[32], m_run[2] = {-INFINITY, -INFINITY}, lsum[2] = {0.f, 0.f};
#pragma unroll
  for (int e = 0; e < 32; ++e) o[e] = 0.f;
  mbar_wait(smem_u32(&bar_q), 0);
  for (int g = 0; g < G; ++g) {
    const int st = g % AT_KVST;
    const int j0 = g * AT_BK;
    const bool masked = j0 + AT_BK > kfree;
    if (threadIdx.x == 0) produce(g);
    __syncwarp();
    float bia[BIAS ? 32 : 1];
    if (BIAS) {       // issued before the score MMA: the two latencies overlap
#pragma unroll
      for (int e = 0; e < 32; ++e) {
        const int hh = (e >> 1) & 1, j = j0 + 8 * (e >> 2) + 2 * q + (e & 1);
        bia[e] = (ii[hh] < L && j < klim[hh])
                     ? __ldg(ubias + ((size_t)(s0 + ii[hh]) * gridDim.y + h) * ldu + (ucenter - (q0 + ii[hh]) + j)) : 0.f;
      }
    }
    mbar_wait(smem_u32(&bar_full[st]), (uint32_t)((g / AT_KVST) & 1));
    const uint32_t sK = sKV + st * KV_STAGE, sV = sK + K_BYTES;
    float s[32];
#pragma unroll
    for (int e = 0; e < 32; ++e) s[e] = 0.f;
    wg_fence();
    const uint64_t dk = wg_desc_sw128(sK);
#pragma unroll
    for (int k = 0; k < AT_HD / 16; ++k) wgmma_ss<64, 0>(s, dq + (uint64_t)(2 * k), dk + (uint64_t)(2 * k), 1);
    wg_commit();
    if (threadIdx.x == 0) produce(g);    // stages released meanwhile: never blocks here (tile g is already loaded)
    __syncwarp();
    wg_wait<0>();
    wg_touch<32>(s);
    // s[e]: row rbase + 8 ((e >> 1) & 1), key j0 + 8 (e >> 2) + 2 q + (e & 1)
    float tm[2] = {-INFINITY, -INFINITY};
    if (masked) {
#pragma unroll
      for (int e = 0; e < 32; ++e) {
        const int hh = (e >> 1) & 1, j = j0 + 8 * (e >> 2) + 2 * q + (e & 1);
        if (BIAS) s[e] += bia[e];
        if (j >= klim[hh]) s[e] = -INFINITY;
        tm[hh] = fmaxf(tm[hh], s[e]);
      }
    } else {
#pragma unroll
      for (int e = 0; e < 32; ++e) {
        const int hh = (e >> 1) & 1;
        if (BIAS) s[e] += bia[e];
        tm[hh] = fmaxf(tm[hh], s[e]);
      }
    }
    float f[2], mneg[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const float mt = quad_max(tm[hh]) * scale_log2e;     // scale > 0: max commutes with the scaling
      const float mn = fmaxf(m_run[hh], mt);
      f[hh] = m_run[hh] == -INFINITY ? 1.f : fast_ex2(m_run[hh] - mn);   // nothing accumulated yet: o and lsum are 0
      m_run[hh] = mn;
      mneg[hh] = mn == -INFINITY ? 0.f : -mn;
    }
    if (masked) {
#pragma unroll
      for (int e = 0; e < 32; ++e) {
        const int hh = (e >> 1) & 1;
        const float p = s[e] == -INFINITY ? 0.f : fast_ex2(fmaf(s[e], scale_log2e, mneg[hh]));
        s[e] = p;
        lsum[hh] = e < 4 && !(e & 1) ? fmaf(lsum[hh], f[hh], p) : lsum[hh] + p;   // rescale fused into the row's first add
        o[e] *= f[hh];
      }
    } else {      // no -inf from the mask here (an overflowed score of -inf still gives ex2(-inf) = +0)
#pragma unroll
      for (int e = 0; e < 32; ++e) {
        const int hh = (e >> 1) & 1;
        const float p = fast_ex2(fmaf(s[e], scale_log2e, mneg[hh]));
        s[e] = p;
        lsum[hh] = e < 4 && !(e & 1) ? fmaf(lsum[hh], f[hh], p) : lsum[hh] + p;   // rescale fused into the row's first add
        o[e] *= f[hh];
      }
    }
    uint32_t pa[4][4];      // P as the A operand of 4 K16 steps: rows rbase / rbase + 8, keys 16 kk + 2 q (+8)
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      pa[kk][0] = pack_bf16(s[8 * kk + 0], s[8 * kk + 1]);
      pa[kk][1] = pack_bf16(s[8 * kk + 2], s[8 * kk + 3]);
      pa[kk][2] = pack_bf16(s[8 * kk + 4], s[8 * kk + 5]);
      pa[kk][3] = pack_bf16(s[8 * kk + 6], s[8 * kk + 7]);
    }
    wg_fence();
    const uint64_t dv = wg_desc_sw128(sV);
#pragma unroll
    for (int kk = 0; kk < AT_BK / 16; ++kk) wgmma_rs_tb_m64n64(o, pa[kk], dv + (uint64_t)(128 * kk), 1);   // +2048 B per 16 keys
    wg_commit();
    wg_wait<0>();
    wg_touch<32>(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&bar_empty[st]));
  }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const float den = quad_sum(lsum[hh]);
    const float inv = den > 0.f ? 1.f / den : 0.f;
    if (ii[hh] < L) {
      bf16* op = out + (size_t)(s0 + ii[hh]) * ldo + h * AT_HD + 2 * q;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<uint32_t*>(op + 8 * jj) = pack_bf16(o[4 * jj + 2 * hh] * inv, o[4 * jj + 2 * hh + 1] * inv);
    }
  }
}

// ---- relative-position scores of the conformer attention ---------------------------------------------------------------------
// U[(s0 + i) * H + h][t] = (q_i + pos_bias_v)_h . p[t]_h for the table rows t that query tile i0 can address (t = center - (i - j),
// j < L): one CTA per (query tile, head, sequence), 64-row tiles of the position table through the same TMA / wgmma pipeline as
// the score MMA of the attention kernel; each consumer warpgroup writes the fp32 rows of its 64 queries.
__global__ void __launch_bounds__(RP_THREADS, 1)
relpos_u_kernel(const __grid_constant__ CUtensorMap tmq, const __grid_constant__ CUtensorMap tmp, const int* __restrict__ start,
                const int* __restrict__ len, int center, int pos_rows, float* __restrict__ U, int ldu) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_q;
  __shared__ __align__(8) uint64_t bar_full[AT_KVST], bar_empty[AT_KVST];
  const int b = blockIdx.z, h = blockIdx.y;
  const int L = len[b], s0 = start[b];
  const int i0 = blockIdx.x * AT_BQ;
  if (i0 >= L) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = base, sP = base + Q_BYTES;
  const int i_hi = min(i0 + AT_BQ, L) - 1;
  const int t_lo = max(center - i_hi, 0), t_hi = min(center - i0 + L - 1, pos_rows - 1);
  const int t0 = (t_lo / AT_BK) * AT_BK;
  const int G = (t_hi - t0) / AT_BK + 1;
  if (threadIdx.x == 0) {
    mbar_init(smem_u32(&bar_q), 1);
    for (int s = 0; s < AT_KVST; ++s) {
      mbar_init(smem_u32(&bar_full[s]), 1);
      mbar_init(smem_u32(&bar_empty[s]), 8);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (warp < 4) {
    if (warp == 0 && lane == 0) {
      mbar_expect_tx(smem_u32(&bar_q), Q_BYTES);
      tma_load_2d(sQ, &tmq, smem_u32(&bar_q), h * AT_HD, s0 + i0);
      for (int g = 0; g < G; ++g) {
        const int st = g % AT_KVST;
        mbar_wait(smem_u32(&bar_empty[st]), (uint32_t)(((g / AT_KVST) & 1) ^ 1));
        const uint32_t fb = smem_u32(&bar_full[st]);
        mbar_expect_tx(fb, K_BYTES);
        tma_load_2d(sP + st * K_BYTES, &tmp, fb, h * AT_HD, t0 + g * AT_BK);
      }
    }
    return;
  }
  const int wg = (threadIdx.x - 128) >> 7;
  const int q = lane & 3;
  const int rbase = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const uint64_t dq = wg_desc_sw128(sQ + (uint32_t)wg * (Q_BYTES / 2));
  mbar_wait(smem_u32(&bar_q), 0);
  for (int g = 0; g < G; ++g) {
    const int st = g % AT_KVST;
    mbar_wait(smem_u32(&bar_full[st]), (uint32_t)((g / AT_KVST) & 1));
    float s[32];
#pragma unroll
    for (int e = 0; e < 32; ++e) s[e] = 0.f;
    wg_fence();
    const uint64_t dp = wg_desc_sw128(sP + st * K_BYTES);
#pragma unroll
    for (int k = 0; k < AT_HD / 16; ++k) wgmma_ss<64, 0>(s, dq + (uint64_t)(2 * k), dp + (uint64_t)(2 * k), 1);
    wg_commit();
    wg_wait<0>();
    wg_touch<32>(s);
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&bar_empty[st]));
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int i = i0 + rbase + 8 * hh;
      if (i < L) {
        float* urow = U + ((size_t)(s0 + i) * gridDim.y + h) * ldu + t0 + g * AT_BK + 2 * q;     // ldu and t0 are even
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) *reinterpret_cast<float2*>(urow + 8 * jj) = make_float2(s[4 * jj + 2 * hh], s[4 * jj + 2 * hh + 1]);
      }
    }
  }
}

// bf16 operand [rows, cols]: 64-column boxes of box_rows rows
void make_map(cvk_ctx* ctx, CUtensorMap* m, const Mat& x, int box_rows) {
  const cuuint64_t dims[2] = {(cuuint64_t)x.cols, (cuuint64_t)x.rows};
  const cuuint64_t strides[1] = {(cuuint64_t)x.ld * 2};
  const cuuint32_t box[2] = {AT_HD, (cuuint32_t)box_rows};
  encode_tma_map(ctx, m, x.p, 2, dims, strides, box, DT_BF16, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "attention");
}

}  // namespace

void attention_tc_setup() {
  CVK_CHECK_CUDA(cudaFuncSetAttribute(attn_wg_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AT_SMEM));
  CVK_CHECK_CUDA(cudaFuncSetAttribute(attn_wg_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AT_SMEM));
  CVK_CHECK_CUDA(cudaFuncSetAttribute(relpos_u_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AT_SMEM));
  // the kernel relies on two co-resident CTAs per SM to hide its serial MMA -> softmax -> MMA chain: a register or shared
  // memory increase that loses the second CTA is an error, not a silent slowdown
  int per_sm = 0;
  CVK_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, attn_wg_kernel<false>, AT_THREADS, AT_SMEM));
  CVK_REQUIRE(per_sm >= 2, "attn_wg_kernel: " + std::to_string(per_sm) + " CTA(s) per SM, laid out for 2");
}

void attention_fwd_tc(cvk_ctx* ctx, cudaStream_t st, const Mat& q, const Mat& k, const Mat& v, const Seqs& s, int H, int chunk,
                      float scale, const Mat& out, int kv_div, const KvGeom* kg) {
  CVK_REQUIRE(q.dtype == DT_BF16 && out.dtype == DT_BF16, "attention_fwd_tc: bf16 only");
  CVK_REQUIRE(q.ld % 8 == 0 && k.ld % 8 == 0 && v.ld % 8 == 0 && out.ld % 8 == 0, "attention_fwd_tc: 16-byte row pitch required");
  CVK_REQUIRE((((uintptr_t)q.p | (uintptr_t)k.p | (uintptr_t)v.p | (uintptr_t)out.p) & 15) == 0, "attention_fwd_tc: 16-byte alignment required");
  CUtensorMap tq, tk, tv;
  make_map(ctx, &tq, q, AT_BQ);
  make_map(ctx, &tk, k, AT_BK);
  make_map(ctx, &tv, v, AT_BK);
  dim3 grid(ceil_div(s.max_len, AT_BQ), H, s.B);
  attn_wg_kernel<false><<<grid, AT_THREADS, AT_SMEM, st>>>(tq, tk, tv, s.d_start, s.d_len, chunk, scale * 1.4426950408889634f, kv_div, out.b16(), out.ld,
                                                           kg ? kg->d_kstart : nullptr, kg ? kg->d_klen : nullptr, kg ? kg->d_qoff : nullptr,
                                                           nullptr, 0, 0);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}

// Conformer relative-position attention on the tensor cores (bf16 operands): score(i, j) = ((q_i + u) . k_j + (q_i + v) . p[center - (i - j)]) * scale.
// qu = q + pos_bias_u and qv = q + pos_bias_v are materialised by the caller; U (fp32 [rows * H, ldu], workspace) receives the second
// term for every addressable table row, the attention kernel adds it as a bias.
void relpos_attention_fwd_tc(cvk_ctx* ctx, cudaStream_t st, const Mat& qu, const Mat& qv, const Mat& k, const Mat& v, const Mat& pos, int pos_rows,
                             int pos_center, const Seqs& s, int H, int chunk, float scale, const Mat& U, const Mat& out) {
  CVK_REQUIRE(qu.dtype == DT_BF16 && qv.dtype == DT_BF16 && k.dtype == DT_BF16 && v.dtype == DT_BF16 && pos.dtype == DT_BF16 && out.dtype == DT_BF16 &&
              U.dtype == DT_F32, "relpos_attention_fwd_tc: bf16 operands, fp32 workspace");
  CVK_REQUIRE(U.ld % 4 == 0 && U.ld >= round_up(pos_rows, AT_BK) && U.rows >= s.R * H, "relpos_attention_fwd_tc: workspace too small");
  CVK_REQUIRE(pos.rows >= round_up(pos_rows, AT_BK), "relpos_attention_fwd_tc: position table must be padded to a multiple of 64 rows");
  CUtensorMap tq, tqv, tk, tv, tp;
  make_map(ctx, &tq, qu, AT_BQ);
  make_map(ctx, &tqv, qv, AT_BQ);
  make_map(ctx, &tk, k, AT_BK);
  make_map(ctx, &tv, v, AT_BK);
  make_map(ctx, &tp, pos, AT_BK);
  dim3 grid(ceil_div(s.max_len, AT_BQ), H, s.B);
  relpos_u_kernel<<<grid, RP_THREADS, AT_SMEM, st>>>(tqv, tp, s.d_start, s.d_len, pos_center, pos_rows, U.f32(), U.ld);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  attn_wg_kernel<true><<<grid, AT_THREADS, AT_SMEM, st>>>(tq, tk, tv, s.d_start, s.d_len, chunk, scale * 1.4426950408889634f, 1, out.b16(), out.ld,
                                                          nullptr, nullptr, nullptr, U.f32(), U.ld, pos_center);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}
