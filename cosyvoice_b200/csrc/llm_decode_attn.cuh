// One (row, kv head) unit of the LM decode attention, shared by the per-op kernel (llm.cu attn_fused_kernel) and the
// persistent decode kernel (llm_mega.cu).
//
// qkv split-K reduction + bias + RoPE + KV-cache append + GQA decode attention (transformers Qwen2 attention,
// SURVEY.md Appendix C; cosyvoice/llm/llm.py:242-254 forward_one_step).  The attention itself is flash-decoding on
// warp-level tensor-core MMAs (m16n8k16, bf16 in / fp32 accumulate): the 7 query heads of the group are the M rows of the
// tile (7 of 16 used - wgmma's M >= 64 would waste 9/10 of the tile), each of the NW warps walks its own
// 16-key blocks with an online softmax held in registers, K and V fragments come straight from the cache with 4-byte loads
// (V's key pairs are formed with byte permutes, the output dims of a 16-dim block are assigned to the two n-tiles as evens /
// odds so that each lane ends up with 4 consecutive dims), P never leaves registers (the QK^T accumulator layout is the
// A-operand layout of the P V MMA), and the warps' partial (max, sum, O) are merged through shared memory.
#pragma once
#include "llm_internal.h"

namespace lm {

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 h2 = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h2);
}
__device__ __forceinline__ void mma_16816(float* c, uint32_t a0, uint32_t a2, uint32_t b0, uint32_t b1) {   // A rows 8..15 are zero
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(0u), "r"(a2), "r"(0u), "r"(b0), "r"(b1));
}
template <int BAR_ID, int NTHREADS>
__device__ __forceinline__ void attn_bar() {
  if (BAR_ID == 0) __syncthreads();
  else asm volatile("bar.sync %0, %1;" ::"n"(BAR_ID), "n"(NTHREADS) : "memory");
}

// shared memory floats needed by one unit
template <int NW>
__host__ __device__ constexpr int decode_attn_smem_floats() { return (NH / NKV + 2) * HD + NW * 8 * 2 + NW * (NH / NKV) * HD; }

// K / V fragments of one 16-key block (rows j0 .. j0+15, all below `L`), in the MMA operand layout used by decode_attn_unit
struct KvFrag {
  uint32_t kf[2][4][2], vw[4][4];
};
__device__ __forceinline__ void decode_attn_load_block(const bf16* __restrict__ kb, const bf16* __restrict__ vb, int j0, int L, int lane, KvFrag& f) {
  const int g = lane >> 2, t4 = lane & 3;
#pragma unroll
  for (int nt = 0; nt < 2; ++nt) {
    const uint32_t* kr = reinterpret_cast<const uint32_t*>(kb + (size_t)min(j0 + nt * 8 + g, L - 1) * HD);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      f.kf[nt][kk][0] = kr[kk * 8 + t4];
      f.kf[nt][kk][1] = kr[kk * 8 + 4 + t4];
    }
  }
  const uint32_t* v0 = reinterpret_cast<const uint32_t*>(vb + (size_t)min(j0 + t4 * 2, L - 1) * HD);
  const uint32_t* v1 = reinterpret_cast<const uint32_t*>(vb + (size_t)min(j0 + t4 * 2 + 1, L - 1) * HD);
  const uint32_t* v2 = reinterpret_cast<const uint32_t*>(vb + (size_t)min(j0 + 8 + t4 * 2, L - 1) * HD);
  const uint32_t* v3 = reinterpret_cast<const uint32_t*>(vb + (size_t)min(j0 + 9 + t4 * 2, L - 1) * HD);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    f.vw[q][0] = v0[q * 8 + g];
    f.vw[q][1] = v1[q * 8 + g];
    f.vw[q][2] = v2[q * 8 + g];
    f.vw[q][3] = v3[q * 8 + g];
  }
}

// tid / warp / lane: coordinates inside the group of NW warps that runs the unit (all NW*32 threads must call).
// partial [splits][rows][1152] fp32 split-K sums of the qkv projection of row b; kb / vb: this (row, kv head)'s cache
// [max_ctx][64]; out: bf16 [.. ldo], this row's attention output (columns of the kv group's 7 query heads).
// SPLITS > 0: compile-time split count - every partial-sum load of a thread is issued before the first add (ONE memory round
// trip instead of one per in-order add), read with ld.global.cg (the producers are other SMs of the same kernel).
template <int NW, int BAR_ID, int SPLITS = 0>
__device__ __forceinline__ void decode_attn_unit(float* __restrict__ sm_all, int tid, const float* __restrict__ partial, int splits, int rows,
                                                 int b, int kvh, const float* __restrict__ bias, bf16* __restrict__ kb, bf16* __restrict__ vb,
                                                 int pos, int max_ctx, const float* __restrict__ inv_freq, bf16* __restrict__ out_row,
                                                 KvFrag& fr /*fragment registers; if have_pre: this warp's first block, loaded early*/,
                                                 bool have_pre) {
  constexpr int G = NH / NKV;
  constexpr int NT = NW * 32;
  const int warp = tid >> 5, lane = tid & 31;
  float* stage = sm_all;
  float* ml = stage + (G + 2) * HD;
  float* po = ml + NW * 8 * 2;
  if (SPLITS > 0) {
    constexpr int PER = ((G + 2) * HD + NT - 1) / NT;
    constexpr int S = SPLITS > 0 ? SPLITS : 1;
    float ld[PER][S], bs[PER];
    const size_t stride = (size_t)rows * QKV_N;
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      const int e = tid + i * NT;
      const bool ok = e < (G + 2) * HD;
      const int vec = ok ? e / HD : 0, d = e % HD;
      const int col = vec < G ? (kvh * G + vec) * HD + d : (vec == G ? NH * HD + kvh * HD + d : NH * HD + NKV * HD + kvh * HD + d);
      const float* p = partial + (size_t)b * QKV_N + col;
      bs[i] = bias[col];
#pragma unroll
      for (int s2 = 0; s2 < S; ++s2) ld[i][s2] = ok ? __ldcg(p + (size_t)s2 * stride) : 0.f;
    }
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      const int e = tid + i * NT;
      float a = bs[i];
#pragma unroll
      for (int s2 = 0; s2 < S; ++s2) a += ld[i][s2];
      if (e < (G + 2) * HD) stage[e] = a;
    }
  } else {
    for (int e = tid; e < (G + 2) * HD; e += NT) {
      const int vec = e / HD, d = e % HD;
      const int col = vec < G ? (kvh * G + vec) * HD + d : (vec == G ? NH * HD + kvh * HD + d : NH * HD + NKV * HD + kvh * HD + d);
      const float* p = partial + (size_t)b * QKV_N + col;
      const size_t stride = (size_t)rows * QKV_N;
      float a0 = bias[col], a1 = 0.f, a2 = 0.f, a3 = 0.f;
      int s = 0;
      for (; s + 4 <= splits; s += 4) {      // independent loads in flight
        a0 += p[(size_t)s * stride];
        a1 += p[(size_t)(s + 1) * stride];
        a2 += p[(size_t)(s + 2) * stride];
        a3 += p[(size_t)(s + 3) * stride];
      }
      for (; s < splits; ++s) a0 += p[(size_t)s * stride];
      stage[e] = (a0 + a1) + (a2 + a3);
    }
  }
  attn_bar<BAR_ID, NT>();
  for (int e = tid; e < (G + 1) * (HD / 2); e += NT) {     // rotate the G query heads and k (half-split RoPE, theta 1e6)
    const int vec = e / (HD / 2), i = e % (HD / 2);
    const float fr = (float)pos * inv_freq[i];
    const float c = cosf(fr), sn = sinf(fr);
    float* p = stage + vec * HD;
    const float x1 = p[i], x2 = p[i + HD / 2];
    p[i] = x1 * c - x2 * sn;
    p[i + HD / 2] = x2 * c + x1 * sn;
  }
  attn_bar<BAR_ID, NT>();
  if (pos < max_ctx && tid < 2 * HD) {
    const int d = tid % HD;
    if (tid < HD) kb[(size_t)pos * HD + d] = __float2bfloat16_rn(stage[G * HD + d]);
    else vb[(size_t)pos * HD + d] = __float2bfloat16_rn(stage[(G + 1) * HD + d]);
  }
  attn_bar<BAR_ID, NT>();
  const int L = min(pos + 1, max_ctx);
  const int g = lane >> 2, t4 = lane & 3;        // MMA fragment coordinates: row / column group
  uint32_t qa[4][2];                             // Q as the A operand: [k step][dims t4*2.. | +8]; row g = query head g (row 7 unused)
#pragma unroll
  for (int kk = 0; kk < 4; ++kk)
#pragma unroll
    for (int hv = 0; hv < 2; ++hv) {
      const int d = kk * 16 + hv * 8 + t4 * 2;
      qa[kk][hv] = g < G ? pack_bf16x2(__bfloat162float(__float2bfloat16_rn(stage[g * HD + d])) * 0.125f,
                                       __bfloat162float(__float2bfloat16_rn(stage[g * HD + d + 1])) * 0.125f)
                         : 0u;
    }
  float o[4][2][4];
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int t = 0; t < 2; ++t)
#pragma unroll
      for (int e = 0; e < 4; ++e) o[q][t][e] = 0.f;
  float m_run = -INFINITY, l_run = 0.f;
  for (int j0 = warp * 16; j0 < L; j0 += NW * 16) {
    // every load of the block is issued before the first use: one memory round trip per 16 keys.  Rows past the end are
    // clamped to the last valid row (finite data), their probabilities are forced to zero below.
    if (!(have_pre && j0 == warp * 16)) decode_attn_load_block(kb, vb, j0, L, lane, fr);
    uint32_t (&kf)[2][4][2] = fr.kf;
    uint32_t (&vw)[4][4] = fr.vw;
    float s0[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      mma_16816(s0, qa[kk][0], qa[kk][1], kf[0][kk][0], kf[0][kk][1]);
      mma_16816(s1, qa[kk][0], qa[kk][1], kf[1][kk][0], kf[1][kk][1]);
    }
    // this lane: head g, keys j0 + 2 t4 + {0,1} (s0) and j0 + 8 + 2 t4 + {0,1} (s1)
    const int ka = j0 + t4 * 2;
    const bool va0 = ka < L, va1 = ka + 1 < L, vb0 = ka + 8 < L, vb1 = ka + 9 < L;
    float mx = fmaxf(fmaxf(va0 ? s0[0] : -INFINITY, va1 ? s0[1] : -INFINITY), fmaxf(vb0 ? s1[0] : -INFINITY, vb1 ? s1[1] : -INFINITY));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    const float m_new = fmaxf(m_run, mx);          // finite: key j0 itself is valid
    const float corr = __expf(m_run - m_new);      // exp(-inf) = 0 on the first block
    const float p0 = va0 ? __expf(s0[0] - m_new) : 0.f, p1 = va1 ? __expf(s0[1] - m_new) : 0.f;
    const float p2 = vb0 ? __expf(s1[0] - m_new) : 0.f, p3 = vb1 ? __expf(s1[1] - m_new) : 0.f;
    l_run = l_run * corr + ((p0 + p1) + (p2 + p3));
    m_run = m_new;
    const uint32_t pa0 = pack_bf16x2(p0, p1), pa2 = pack_bf16x2(p2, p3);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      o[q][0][0] *= corr; o[q][0][1] *= corr;
      o[q][1][0] *= corr; o[q][1][1] *= corr;
      // n-tile 0: even dims of the 16-dim block, n-tile 1: odd dims (low / high halves of the loaded words)
      mma_16816(o[q][0], pa0, pa2, __byte_perm(vw[q][0], vw[q][1], 0x5410), __byte_perm(vw[q][2], vw[q][3], 0x5410));
      mma_16816(o[q][1], pa0, pa2, __byte_perm(vw[q][0], vw[q][1], 0x7632), __byte_perm(vw[q][2], vw[q][3], 0x7632));
    }
  }
  l_run += __shfl_xor_sync(0xffffffffu, l_run, 1);
  l_run += __shfl_xor_sync(0xffffffffu, l_run, 2);
  if (g < G) {
    if (t4 == 0) {
      ml[(warp * 8 + g) * 2] = m_run;
      ml[(warp * 8 + g) * 2 + 1] = l_run;
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)     // dims 16 q + 4 t4 .. + 3
      *reinterpret_cast<float4*>(po + ((size_t)warp * G + g) * HD + q * 16 + t4 * 4) = make_float4(o[q][0][0], o[q][1][0], o[q][0][1], o[q][1][1]);
  }
  attn_bar<BAR_ID, NT>();
  for (int e = tid; e < G * HD; e += NT) {
    const int hq = e / HD, d = e % HD;
    float M = -INFINITY;
#pragma unroll
    for (int w2 = 0; w2 < NW; ++w2) M = fmaxf(M, ml[(w2 * 8 + hq) * 2]);
    float num = 0.f, den = 0.f;
#pragma unroll
    for (int w2 = 0; w2 < NW; ++w2) {
      const float wgt = __expf(ml[(w2 * 8 + hq) * 2] - M);    // warps without keys: exp(-inf) = 0
      den = fmaf(wgt, ml[(w2 * 8 + hq) * 2 + 1], den);
      num = fmaf(wgt, po[((size_t)w2 * G + hq) * HD + d], num);
    }
    out_row[(kvh * G + hq) * HD + d] = __float2bfloat16_rn(num / den);
  }
}

}  // namespace lm
