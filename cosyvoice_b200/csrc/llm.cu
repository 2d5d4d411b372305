// CosyVoice2 speech-token LM: Qwen2-0.5B-shaped decoder driven through inputs_embeds, KV-cached autoregressive
// decode, fused log-softmax + repetition-aware sampling + stop logic + next-embedding gather.
//
// Follows cosyvoice/llm/llm.py:458-502 (Qwen2LM.inference: prompt assembly), :536-549 (inference_wrapper decode
// loop), :150-160 (sampling_ids), cosyvoice/utils/common.py:138-167 (ras_sampling / nucleus_sampling /
// random_sampling).  The transformer arithmetic is transformers' Qwen2 (modeling_qwen2.py; SURVEY.md Appendix C):
// RMSNorm(1e-6) -> q/k/v (+bias) -> half-split RoPE(theta 1e6) -> GQA 14/2 x 64 -> o_proj -> +res -> RMSNorm ->
// SwiGLU(4864) -> +res, 24 layers, final RMSNorm.
//
// Batched over B independent rows (the reference decodes one utterance at a time).  One decode step for all rows is
// captured into a CUDA graph; the sampler advances per-row counters on the device, so the host only polls the
// number of live rows every few steps - no .item() style host round trip per token (common.py:155-161 has several).
#include "llm_decode_attn.cuh"
#include <math.h>
#include <algorithm>

using namespace lm;

namespace {

float* copy_param(cvk_ctx* ctx, const std::string& name) {
  const RawTensor& t = ctx->get_raw(name);
  return dev_copy_f32(ctx, t.p, (size_t)t.numel());
}

ConvW concat_linear(cvk_ctx* ctx, const std::vector<std::string>& wn, const std::vector<std::string>& bn) {
  int K = (int)ctx->get_raw(wn[0]).shape[1], N = 0;
  for (auto& n : wn) N += (int)ctx->get_raw(n).shape[0];
  ConvW w;
  w.N = N; w.K = K;
  w.w32 = (float*)ctx->dmalloc((size_t)N * K * sizeof(float));
  size_t off = 0;
  for (auto& n : wn) {
    const RawTensor& t = ctx->get_raw(n);
    CVK_CHECK_CUDA(cudaMemcpy(w.w32 + off, t.p, (size_t)t.numel() * sizeof(float), cudaMemcpyDeviceToDevice));
    off += t.numel();
  }
  if (!bn.empty()) {
    w.bias = (float*)ctx->dmalloc((size_t)N * sizeof(float));
    size_t bo = 0;
    for (auto& n : bn) {
      const RawTensor& t = ctx->get_raw(n);
      CVK_CHECK_CUDA(cudaMemcpy(w.bias + bo, t.p, (size_t)t.numel() * sizeof(float), cudaMemcpyDeviceToDevice));
      bo += t.numel();
    }
  }
  finish_convw(ctx, w);
  return w;
}

// ------------------------------------------------------------------------------------------------ kernels
// lm_input rows: [sos, embed(text...), task_id, speech_embedding(prompt...)] per sequence (llm.py:485-494)
__global__ void build_input_kernel(const int32_t* __restrict__ text, const int* __restrict__ text_off, const int* __restrict__ text_len,
                                   const int32_t* __restrict__ speech, const int* __restrict__ sp_off, const int* __restrict__ sp_len,
                                   const float* __restrict__ text_emb, const float* __restrict__ llm_emb, const float* __restrict__ speech_emb,
                                   const int* __restrict__ start, float* __restrict__ out) {
  int b = blockIdx.y;
  int nt = text_len[b], ns = sp_len[b];
  int L = 1 + nt + 1 + ns;
  for (int t = blockIdx.x; t < L; t += gridDim.x) {
    const float* src;
    if (t == 0) src = llm_emb;
    else if (t <= nt) src = text_emb + (size_t)text[text_off[b] + t - 1] * D;
    else if (t == nt + 1) src = llm_emb + D;
    else src = speech_emb + (size_t)speech[sp_off[b] + t - nt - 2] * D;
    float* dst = out + (size_t)(start[b] + t) * D;
    for (int c = threadIdx.x; c < D; c += blockDim.x) dst[c] = src[c];
  }
}

// half-split RoPE (modeling_qwen2.py rotate_half) on the q and k parts of a fused qkv row, in place; position =
// pos0[seq] + t.  Also appends k, v to the cache at that position.  With rowpos (ragged feed, rows_are_seqs = 1): qkv row
// blockIdx.y goes to cache row rowpos[.].x at position rowpos[.].y.
template <typename T>
__global__ void rope_append_kernel(T* __restrict__ qkv, int ld, const int* __restrict__ start, const int* __restrict__ len,
                                   const int* __restrict__ pos0, const float* __restrict__ inv_freq, T* __restrict__ kc, T* __restrict__ vc,
                                   int max_ctx, int rows_are_seqs, const int2* __restrict__ rowpos) {
  int b = blockIdx.y;
  int L = rows_are_seqs ? 1 : len[b];
  int base = rows_are_seqs ? b : start[b];
  const int cb = rowpos ? rowpos[b].x : b;
  const int p0 = rowpos ? rowpos[b].y : (pos0 ? pos0[b] : 0);
  for (int t = blockIdx.x; t < L; t += gridDim.x) {
    int pos = p0 + t;
    T* row = qkv + (size_t)(base + t) * ld;
    // 16 heads to rotate (14 q + 2 k), 32 pairs each
    for (int e = threadIdx.x; e < (NH + NKV) * (HD / 2); e += blockDim.x) {
      int h = e / (HD / 2), i = e % (HD / 2);
      float fr = (float)pos * inv_freq[i];
      float c = cosf(fr), s = sinf(fr);
      T* p = row + h * HD;
      float x1 = to_f32(p[i]), x2 = to_f32(p[i + HD / 2]);
      p[i] = from_f32<T>(x1 * c - x2 * s);
      p[i + HD / 2] = from_f32<T>(x2 * c + x1 * s);
    }
    __syncthreads();
    if (pos < max_ctx) {
      for (int e = threadIdx.x; e < NKV * HD; e += blockDim.x) {
        int h = e / HD, d = e % HD;
        size_t ci = (((size_t)cb * NKV + h) * max_ctx + pos) * HD + d;
        kc[ci] = row[NH * HD + e];
        vc[ci] = row[NH * HD + NKV * HD + e];
      }
    }
    __syncthreads();
  }
}

// decode attention: one CTA per (row, kv head), one warp per query head of the group (7 warps).  Phase A: one key per
// lane (full 64-dim dot product from a 128-byte cache row), scores to shared memory; softmax over the warp; phase B: one
// pair of output dims per lane, keys streamed with coalesced 128-byte rows.  Keys 0..ctx_len[b] (new token included).  With
// rowpos (ragged feed): query row b reads cache row rowpos[b].x, keys 0..rowpos[b].y.
template <typename T>
__global__ void __launch_bounds__((NH / NKV) * 32)
decode_attn_kernel(const T* __restrict__ qkv, int ld, const T* __restrict__ kc, const T* __restrict__ vc,
                   const int* __restrict__ ctx_len, int max_ctx, T* __restrict__ out, int ldo, const int2* __restrict__ rowpos) {
  extern __shared__ float sc_all[];            // [7][max_ctx]
  const int b = blockIdx.x, kvh = blockIdx.y;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = kvh * (NH / NKV) + w;
  const int cb = rowpos ? rowpos[b].x : b;
  const int L = min((rowpos ? rowpos[b].y : ctx_len[b]) + 1, max_ctx);
  float* sc = sc_all + (size_t)w * max_ctx;
  const T* q = qkv + (size_t)b * ld + h * HD;
  const T* kb = kc + ((size_t)cb * NKV + kvh) * max_ctx * HD;
  const T* vb = vc + ((size_t)cb * NKV + kvh) * max_ctx * HD;
  float qr[HD];
#pragma unroll
  for (int d = 0; d < HD; ++d) qr[d] = to_f32(q[d]) * 0.125f;
  float m = -INFINITY;
  for (int j = lane; j < L; j += 32) {
    const T* kr = kb + (size_t)j * HD;
    float s = 0.f;
    if (sizeof(T) == 2) {
      const uint4* k4 = reinterpret_cast<const uint4*>(kr);
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        uint4 u = k4[c];
        const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float2 f = __bfloat1622float2(h2[e]);
          s = fmaf(qr[c * 8 + 2 * e], f.x, s);
          s = fmaf(qr[c * 8 + 2 * e + 1], f.y, s);
        }
      }
    } else {
      const float4* k4 = reinterpret_cast<const float4*>(kr);
#pragma unroll
      for (int c = 0; c < 16; ++c) {
        float4 f = k4[c];
        s = fmaf(qr[c * 4], f.x, s);
        s = fmaf(qr[c * 4 + 1], f.y, s);
        s = fmaf(qr[c * 4 + 2], f.z, s);
        s = fmaf(qr[c * 4 + 3], f.w, s);
      }
    }
    sc[j] = s;
    m = fmaxf(m, s);
  }
  m = warp_max(m);
  float l = 0.f;
  for (int j = lane; j < L; j += 32) {
    float p = expf(sc[j] - m);
    sc[j] = p;
    l += p;
  }
  l = warp_sum(l);
  __syncwarp();
  float o0 = 0.f, o1 = 0.f;
  int j = 0;
  for (; j + 4 <= L; j += 4) {
    float p0 = sc[j], p1 = sc[j + 1], p2 = sc[j + 2], p3 = sc[j + 3];
    const T* v0 = vb + (size_t)j * HD;
    float a0 = to_f32(v0[lane]), a1 = to_f32(v0[lane + 32]);
    float b0 = to_f32(v0[HD + lane]), b1 = to_f32(v0[HD + lane + 32]);
    float c0 = to_f32(v0[2 * HD + lane]), c1 = to_f32(v0[2 * HD + lane + 32]);
    float d0 = to_f32(v0[3 * HD + lane]), d1 = to_f32(v0[3 * HD + lane + 32]);
    o0 = fmaf(p0, a0, o0); o1 = fmaf(p0, a1, o1);
    o0 = fmaf(p1, b0, o0); o1 = fmaf(p1, b1, o1);
    o0 = fmaf(p2, c0, o0); o1 = fmaf(p2, c1, o1);
    o0 = fmaf(p3, d0, o0); o1 = fmaf(p3, d1, o1);
  }
  for (; j < L; ++j) {
    float p = sc[j];
    o0 = fmaf(p, to_f32(vb[(size_t)j * HD + lane]), o0);
    o1 = fmaf(p, to_f32(vb[(size_t)j * HD + lane + 32]), o1);
  }
  T* op = out + (size_t)b * ldo + h * HD;
  float inv = 1.f / l;
  op[lane] = from_f32<T>(o0 * inv);
  op[lane + 32] = from_f32<T>(o1 * inv);
}

// qkv[b] = sum_s partial[s][b] + bias, in split order, rounded to the activation dtype: the split-K reduction of the per-op
// (unfused) decode path, cvk_op_decode_attention with lm_fused = 0
__global__ void qkv_reduce_kernel(const float* __restrict__ partial, int splits, int rows, const float* __restrict__ bias, bf16* __restrict__ qkv) {
  const size_t total = (size_t)rows * QKV_N;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int s = 0; s < splits; ++s) acc += partial[(size_t)s * total + i];
    qkv[i] = __float2bfloat16_rn(acc + bias[i % QKV_N]);
  }
}

// ---- fused decode kernels (bf16 path) -----------------------------------------------------------------------------
// x[b] += sum_s partial[s][b] (+bias); xn[b] = rmsnorm(x[b]) * gamma  - split-K reduction, residual add and the next
// RMSNorm (modeling_qwen2.py:258-263) in one pass; one CTA per row.
__global__ void __launch_bounds__(D) finish_rms_kernel(const float* __restrict__ partial, int splits, int rows, float* __restrict__ x,
                                                       const float* __restrict__ gamma, bf16* __restrict__ xn, long long* __restrict__ tl) {
  __shared__ float red[D / 32];
  pdl_trigger();
  tl_stamp(tl, 0);
  const int b = blockIdx.x, n = threadIdx.x;
  const float gam = gamma[n];            // constant: fetched before waiting for the producer of `partial`
  pdl_wait();
  tl_stamp(tl, 1);
  const float* p = partial + (size_t)b * D + n;
  const size_t stride = (size_t)rows * D;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  int s = 0;
  for (; s + 4 <= splits; s += 4) {      // independent loads in flight (a plain loop is one L2 round trip per split)
    a0 += p[(size_t)s * stride];
    a1 += p[(size_t)(s + 1) * stride];
    a2 += p[(size_t)(s + 2) * stride];
    a3 += p[(size_t)(s + 3) * stride];
  }
  for (; s < splits; ++s) a0 += p[(size_t)s * stride];
  const float v = x[(size_t)b * D + n] + ((a0 + a1) + (a2 + a3));
  x[(size_t)b * D + n] = v;
  float ss = warp_sum(v * v);
  if ((n & 31) == 0) red[n >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < D / 32; ++i) tot += red[i];
  xn[(size_t)b * D + n] = __float2bfloat16_rn(gam * (v * rsqrtf(tot / D + RMS_EPS)));
  tl_stamp(tl, 2);
}

// qkv split-K reduction + bias + RoPE + KV-cache append + GQA decode attention; one CTA per (row, kv head): see
// llm_decode_attn.cuh (the same unit runs inside the persistent decode kernel, llm_mega.cu).
// QK^T and P V run on mma.sync instead of CUDA-core FMAs (which would need a bf16->fp32 conversion + FMA per element, per head).
constexpr int AF_WARPS = 16;
__global__ void __launch_bounds__(32 * AF_WARPS)
attn_fused_kernel(const float* __restrict__ partial /*[S][rows][1152]*/, int splits, int rows, const float* __restrict__ bias,
                  bf16* __restrict__ kc, bf16* __restrict__ vc, const int* __restrict__ ctx_len, int max_ctx,
                  const float* __restrict__ inv_freq, bf16* __restrict__ out, int ldo, long long* __restrict__ tl) {
  extern __shared__ float sm_all[];            // [G+2][64] staging | [WARPS][8][2] max/sum | [WARPS][G][64] partial O
  const int b = blockIdx.x, kvh = blockIdx.y;
  pdl_trigger();
  tl_stamp(tl, 0);
  bf16* kb = kc + ((size_t)b * NKV + kvh) * max_ctx * HD;
  bf16* vb = vc + ((size_t)b * NKV + kvh) * max_ctx * HD;
  // Before waiting for the qkv projection: this warp's first 16-key block of OLD cache rows (written by earlier decode steps /
  // the prefill, i.e. by grids that completed long before this one could start) is pulled from HBM while the projection still
  // runs.  ctx_len[b] may be read mid-update by this step's sampler (it only grows by one per step): either value is a valid
  // lower bound of the number of finished rows, and only blocks entirely below it are preloaded.
  const int p0 = min(*reinterpret_cast<const volatile int*>(ctx_len + b), max_ctx);
  const int wj0 = (threadIdx.x >> 5) * 16;
  KvFrag pre;
  const bool have_pre = wj0 + 16 <= p0;
  if (have_pre) decode_attn_load_block(kb, vb, wj0, p0, threadIdx.x & 31, pre);
  pdl_wait();
  tl_stamp(tl, 1);
  decode_attn_unit<AF_WARPS, 0>(sm_all, threadIdx.x, partial, splits, rows, b, kvh, bias, kb, vb, ctx_len[b], max_ctx, inv_freq,
                                out + (size_t)b * ldo, pre, have_pre);
  tl_stamp(tl, 2);
}

__global__ void interleave_rows_kernel(const float* __restrict__ gu /*[2*F][K]: gate rows then up rows*/, float* __restrict__ out, int F, int K) {
  size_t total = (size_t)2 * F * K;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int k = i % K;
    int r = i / K;
    int src = (r & 1) ? F + (r >> 1) : (r >> 1);
    out[i] = gu[(size_t)src * K + k];
  }
}

// SwiGLU: silu(gate) * up; gu = [gate(4864) | up(4864)]
template <typename T>
__global__ void swiglu_kernel(const T* __restrict__ gu, int ld, int rows, T* __restrict__ out, int ldo) {
  size_t total = (size_t)rows * DFF;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int r = i / DFF, c = i % DFF;
    float g = to_f32(gu[(size_t)r * ld + c]), u = to_f32(gu[(size_t)r * ld + DFF + c]);
    out[(size_t)r * ldo + c] = from_f32<T>(g / (1.f + expf(-g)) * u);
  }
}

__global__ void gather_last_kernel(const float* __restrict__ x, const int* __restrict__ start, const int* __restrict__ len,
                                   float* __restrict__ out) {
  int b = blockIdx.x;
  const float* src = x + (size_t)(start[b] + len[b] - 1) * D;
  for (int c = threadIdx.x; c < D; c += blockDim.x) out[(size_t)b * D + c] = src[c];
}

// ---- ragged feed kernels (cvk_lm_feed_rows / cvk_lm_next_logp_rows) -------------------------------------------------------
// activation row m <- embedding of (kinds[m], ids[m]): 0 text (embed_tokens), 1 speech (speech_embedding), 2 llm_embedding row
__global__ void ragged_embed_kernel(const int* __restrict__ ids, const int* __restrict__ kinds, const float* __restrict__ text_emb,
                                    const float* __restrict__ llm_emb, const float* __restrict__ speech_emb, float* __restrict__ x) {
  const int m = blockIdx.x, kind = kinds[m], id = ids[m];
  const float* src = kind == 0 ? text_emb + (size_t)id * D : (kind == 1 ? speech_emb + (size_t)id * D : llm_emb + (size_t)id * D);
  for (int c = threadIdx.x; c < D; c += blockDim.x) x[(size_t)m * D + c] = src[c];
}

// per fed row i: hidden[row] <- x[its last activation row], ctx_len[row] += its position count (sc [n][3] = row, last row, count)
__global__ void feed_scatter_kernel(const int* __restrict__ sc, const float* __restrict__ x, float* __restrict__ hidden, int* __restrict__ ctx_len) {
  const int i = blockIdx.x, b = sc[3 * i], ml = sc[3 * i + 1];
  for (int c = threadIdx.x; c < D; c += blockDim.x) hidden[(size_t)b * D + c] = x[(size_t)ml * D + c];
  if (threadIdx.x == 0) ctx_len[b] += sc[3 * i + 2];
}

// out[i] <- hidden[rows[i]]
__global__ void gather_rows_kernel(const int* __restrict__ rows, const float* __restrict__ hidden, float* __restrict__ out) {
  const int i = blockIdx.x;
  for (int c = threadIdx.x; c < D; c += blockDim.x) out[(size_t)i * D + c] = hidden[(size_t)rows[i] * D + c];
}

__device__ __forceinline__ void mma_16816_full(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// Ragged cached GQA attention on tensor cores (bf16 KV).  One CTA per (tile, kv head); a tile is up to two consecutive positions
// of one session row: tiles[t] = (first activation row, session row, its cache position, 1 or 2).  The MMA's 16 rows are the 7
// query heads of the first position (rows 0..6) and of the second (rows 8..14), so both positions share every K / V fragment.
// Each query attends to its row's cache up to and including its own position: the appends of the whole pass ran before this
// kernel, so causality inside a feed is only the key bound.  The RA_WARPS warps walk interleaved 16-key blocks with an online
// softmax in registers (the decode unit's scheme, llm_decode_attn.cuh) and merge their partial (max, sum, O) in shared memory.
constexpr int RA_WARPS = 4;
__global__ void __launch_bounds__(32 * RA_WARPS)
ragged_attn_tc_kernel(const bf16* __restrict__ qkv, int ld, const bf16* __restrict__ kc, const bf16* __restrict__ vc, int max_ctx,
                      const int4* __restrict__ tiles, bf16* __restrict__ out, int ldo) {
  constexpr int G = NH / NKV;
  __shared__ float ml[RA_WARPS][16][2];
  __shared__ __align__(16) float po[RA_WARPS][16][HD];
  const int4 tl = tiles[blockIdx.x];
  const int m0 = tl.x, b = tl.y, pos0 = tl.z, n = tl.w, kvh = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t4 = lane & 3;
  const bf16* kb = kc + ((size_t)b * NKV + kvh) * max_ctx * HD;
  const bf16* vb = vc + ((size_t)b * NKV + kvh) * max_ctx * HD;
  const int L0 = pos0 + 1, L1 = pos0 + n;      // key bounds of MMA rows 0..7 and 8..15 (n == 1: rows 8..15 repeat the first query)
  const bf16* qa_row = qkv + (size_t)m0 * ld + (kvh * G + g) * HD;
  const bf16* qb_row = qkv + (size_t)(m0 + n - 1) * ld + (kvh * G + g) * HD;
  auto qpair = [&](const bf16* p, int d) -> uint32_t {   // two dims of one query head, pre-scaled by 1/sqrt(64) (exact in bf16)
    if (g >= G) return 0u;
    const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p + d));
    return pack_bf16x2(f.x * 0.125f, f.y * 0.125f);
  };
  uint32_t qf[4][4];
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const int d = kk * 16 + t4 * 2;
    qf[kk][0] = qpair(qa_row, d);
    qf[kk][1] = qpair(qb_row, d);
    qf[kk][2] = qpair(qa_row, d + 8);
    qf[kk][3] = qpair(qb_row, d + 8);
  }
  float o[4][2][4];
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int t = 0; t < 2; ++t)
#pragma unroll
      for (int e = 0; e < 4; ++e) o[q][t][e] = 0.f;
  float m_a = -INFINITY, l_a = 0.f, m_b = -INFINITY, l_b = 0.f;
  KvFrag fr;
  for (int j0 = warp * 16; j0 < L1; j0 += RA_WARPS * 16) {
    decode_attn_load_block(kb, vb, j0, L1, lane, fr);
    float s0[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      mma_16816_full(s0, qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3], fr.kf[0][kk][0], fr.kf[0][kk][1]);
      mma_16816_full(s1, qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3], fr.kf[1][kk][0], fr.kf[1][kk][1]);
    }
    // this lane: keys ka, ka + 1 (s0) and ka + 8, ka + 9 (s1); elements 0, 1 belong to MMA row g, elements 2, 3 to row g + 8
    const int ka = j0 + t4 * 2;
    const int key[4] = {ka, ka + 1, ka + 8, ka + 9};
    const float sa[4] = {s0[0], s0[1], s1[0], s1[1]}, sb[4] = {s0[2], s0[3], s1[2], s1[3]};
    float mxa = -INFINITY, mxb = -INFINITY;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (key[e] < L0) mxa = fmaxf(mxa, sa[e]);
      if (key[e] < L1) mxb = fmaxf(mxb, sb[e]);
    }
    mxa = fmaxf(mxa, __shfl_xor_sync(0xffffffffu, mxa, 1));
    mxa = fmaxf(mxa, __shfl_xor_sync(0xffffffffu, mxa, 2));
    mxb = fmaxf(mxb, __shfl_xor_sync(0xffffffffu, mxb, 1));
    mxb = fmaxf(mxb, __shfl_xor_sync(0xffffffffu, mxb, 2));
    // a block can hold no key of the first query (j0 == L0 when L1 = L0 + 1): keep its state, scale by 1, add nothing
    const float na = fmaxf(m_a, mxa), nb = fmaxf(m_b, mxb);
    const float ua = na == -INFINITY ? 0.f : na, ub = nb == -INFINITY ? 0.f : nb;
    const float ca = __expf(m_a - ua), cb = __expf(m_b - ub);
    float pa[4], pb[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      pa[e] = key[e] < L0 ? __expf(sa[e] - ua) : 0.f;
      pb[e] = key[e] < L1 ? __expf(sb[e] - ub) : 0.f;
    }
    l_a = l_a * ca + ((pa[0] + pa[1]) + (pa[2] + pa[3]));
    l_b = l_b * cb + ((pb[0] + pb[1]) + (pb[2] + pb[3]));
    m_a = na;
    m_b = nb;
    const uint32_t p0 = pack_bf16x2(pa[0], pa[1]), p1 = pack_bf16x2(pb[0], pb[1]), p2 = pack_bf16x2(pa[2], pa[3]), p3 = pack_bf16x2(pb[2], pb[3]);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        o[q][t][0] *= ca; o[q][t][1] *= ca;
        o[q][t][2] *= cb; o[q][t][3] *= cb;
      }
      // n-tile 0: even dims of the 16-dim block, n-tile 1: odd dims (as in decode_attn_unit)
      mma_16816_full(o[q][0], p0, p1, p2, p3, __byte_perm(fr.vw[q][0], fr.vw[q][1], 0x5410), __byte_perm(fr.vw[q][2], fr.vw[q][3], 0x5410));
      mma_16816_full(o[q][1], p0, p1, p2, p3, __byte_perm(fr.vw[q][0], fr.vw[q][1], 0x7632), __byte_perm(fr.vw[q][2], fr.vw[q][3], 0x7632));
    }
  }
  l_a += __shfl_xor_sync(0xffffffffu, l_a, 1);
  l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
  l_b += __shfl_xor_sync(0xffffffffu, l_b, 1);
  l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);
  if (g < G) {
    if (t4 == 0) {
      ml[warp][g][0] = m_a;
      ml[warp][g][1] = l_a;
      ml[warp][g + 8][0] = m_b;
      ml[warp][g + 8][1] = l_b;
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {     // dims 16 q + 4 t4 .. + 3
      *reinterpret_cast<float4*>(&po[warp][g][q * 16 + t4 * 4]) = make_float4(o[q][0][0], o[q][1][0], o[q][0][1], o[q][1][1]);
      *reinterpret_cast<float4*>(&po[warp][g + 8][q * 16 + t4 * 4]) = make_float4(o[q][0][2], o[q][1][2], o[q][0][3], o[q][1][3]);
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < n * G * HD; e += 32 * RA_WARPS) {
    const int r = e / (G * HD), hq = (e / HD) % G, d = e % HD, mr = r * 8 + hq;
    float M = -INFINITY;
#pragma unroll
    for (int w2 = 0; w2 < RA_WARPS; ++w2) M = fmaxf(M, ml[w2][mr][0]);
    float num = 0.f, den = 0.f;
#pragma unroll
    for (int w2 = 0; w2 < RA_WARPS; ++w2) {
      const float wgt = __expf(ml[w2][mr][0] - M);    // warps without keys: exp(-inf) = 0
      den = fmaf(wgt, ml[w2][mr][1], den);
      num = fmaf(wgt, po[w2][mr][d], num);
    }
    out[(size_t)(m0 + r) * ldo + (kvh * G + hq) * HD + d] = __float2bfloat16_rn(num / den);
  }
}

static inline size_t sampler_smem(int V) { return (size_t)2 * ((V + 3) & ~3) * sizeof(float); }   // probabilities + scores

// ---- block-wide helpers for the sampler (256 threads, contiguous segments of `per` entries per thread) ----
__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
  for (int i = 1; i < SAMPLER_THREADS / 32; ++i) r = fmaxf(r, red[i]);
  return r;
}
// float32 sum in the oracle's order (oracle/sampling.py hsum): per-thread contiguous segment left to right, then the
// 256 partials left to right by one thread.
__device__ __forceinline__ float block_hsum(float seg, float* part, float* total) {
  __syncthreads();
  part[threadIdx.x] = seg;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < SAMPLER_THREADS; ++i) t += part[i];
    *total = t;
  }
  __syncthreads();
  return *total;
}

// Fused head epilogue: [optional log-softmax of logits] -> eos mask -> softmax -> nucleus (top-p 0.8 / top-k 25,
// stable order) -> inverse-CDF draw on u1 -> repetition window test (win 10, tau_r 0.1) -> fallback draw on u2 from
// the full distribution with the repeated id removed -> stop / length logic -> append id, gather next embedding.
// Bit-for-bit restatement: oracle/sampling.py (ras_sample, nucleus_select, draw_index, softmax_f32).
// standalone mode (cvk_ras_sample): `scores` already holds log-probs, history given explicitly, no state update.
//
// The row lives in SHARED memory for the whole kernel (one coalesced read, one coalesced write-back of the log-probs with the
// reference's in-place -inf marks) instead of walking the global row with a 104-byte stride per lane in ~8 dependent passes.  The arithmetic (segment order of every
// float32 sum, stable tie-break of the nucleus) is unchanged.
__global__ void __launch_bounds__(SAMPLER_THREADS)
ras_sampler_kernel(float* __restrict__ scores, int V, int from_logits, const float* __restrict__ uniforms /*[..][B][2]*/, int B,
                   const int32_t* __restrict__ min_len, const int32_t* __restrict__ max_len, int32_t* __restrict__ out_ids, int out_ld,
                   int32_t* __restrict__ out_count, int32_t* __restrict__ done, int* __restrict__ ctx_len, const int* __restrict__ base_len,
                   int* __restrict__ live,
                   const float* __restrict__ speech_emb, float* __restrict__ next_x,
                   const int32_t* __restrict__ history, int hist_ld, const int32_t* __restrict__ hist_count,
                   const int32_t* __restrict__ ignore_eos_in, int32_t* __restrict__ ids_out, const float* __restrict__ ln_gamma,
                   bf16* __restrict__ xn_out, long long* __restrict__ tl, long long* __restrict__ dbg_fine) {
  extern __shared__ __align__(16) float sp_all[];   // [V4] probabilities | [V4] scores (log-probs), V4 = V rounded up to 4
  __shared__ float red[SAMPLER_THREADS / 32];
  __shared__ float part[SAMPLER_THREADS];
  __shared__ float tot;
  __shared__ int bi[2][SAMPLER_THREADS / 32];
  __shared__ float kept_p[TOPK];
  __shared__ int kept_i[TOPK];
  __shared__ int s_n, s_top;

  const int b = blockIdx.x, tid = threadIdx.x;
  const bool standalone = ids_out != nullptr;
  pdl_trigger();
  tl_stamp(tl, 0);
  pdl_wait();
  tl_stamp(tl, 1);
  long long* sf = (dbg_fine && b == 0 && tid == 0) ? dbg_fine : nullptr;      // stage stamps of CTA 0 (debug option chain_timeline)
  int sf_i = 0;
#define SF() do { if (sf) { long long t_; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t_)); sf[sf_i++] = t_; } } while (0)
  SF();
  if (!standalone && done[b]) { tl_stamp(tl, 2); return; }
  const int V4 = (V + 3) & ~3;
  float* sp = sp_all;
  float* x = sp_all + V4;
  float* xg = scores + (size_t)b * V;
  if ((V & 3) == 0) {
    for (int i = tid; i < V / 4; i += SAMPLER_THREADS) reinterpret_cast<float4*>(x)[i] = __ldcg(reinterpret_cast<const float4*>(xg) + i);
  } else {
    for (int i = tid; i < V; i += SAMPLER_THREADS) x[i] = __ldcg(xg + i);
  }
  const int per = (V + SAMPLER_THREADS - 1) / SAMPLER_THREADS;
  const int lo = tid * per, hi = min(lo + per, V);
  const int cnt = standalone ? hist_count[b] : out_count[b];
  const bool ignore_eos = standalone ? (ignore_eos_in[b] != 0) : (cnt < min_len[b]);
  const float u1 = standalone ? uniforms[b * 2] : uniforms[((size_t)cnt * B + b) * 2];
  const float u2 = standalone ? uniforms[b * 2 + 1] : uniforms[((size_t)cnt * B + b) * 2 + 1];
  __syncthreads();
  // The thread's contiguous segment (<= SAMPLER_PER entries) lives in REGISTERS from here on: every pass below is an unrolled
  // register loop (a shared-memory version would be a chain of dependent LDS per element).  Entries past
  // the segment hold -inf (scores) / -3 (probabilities) and are skipped by the ordered sums.
  float xr[SAMPLER_PER], pr[SAMPLER_PER];
#pragma unroll
  for (int i = 0; i < SAMPLER_PER; ++i) xr[i] = (i < per && lo + i < hi) ? x[lo + i] : -INFINITY;
  SF();

  // (1) log-softmax of the head output (llm.py:542): (x - max) - log(hsum(exp(x - max)))
  if (from_logits) {
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < SAMPLER_PER; ++i) mx = fmaxf(mx, xr[i]);
    mx = block_max(mx, red);
    float seg = 0.f;
#pragma unroll
    for (int i = 0; i < SAMPLER_PER; ++i)
      if (i < per && lo + i < hi) seg += expf(xr[i] - mx);
    float s = block_hsum(seg, part, &tot);
    float ls = logf(s);
#pragma unroll
    for (int i = 0; i < SAMPLER_PER; ++i)
      if (i < per && lo + i < hi) xr[i] = (xr[i] - mx) - ls;
  }
  SF();
  // (2) eos mask before min_len (llm.py:157-158: only index speech_token_size is masked)
  if (ignore_eos) {
#pragma unroll
    for (int i = 0; i < SAMPLER_PER; ++i)
      if (i < per && lo + i == EOS && lo + i < hi) xr[i] = -INFINITY;
  }
  // (3) softmax of the scores
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < SAMPLER_PER; ++i) mx = fmaxf(mx, xr[i]);
  mx = block_max(mx, red);
  {
    float seg = 0.f;
#pragma unroll
    for (int i = 0; i < SAMPLER_PER; ++i) {
      const bool ok = i < per && lo + i < hi;
      float e = (!ok || xr[i] == -INFINITY) ? 0.f : expf(xr[i] - mx);
      pr[i] = e;
      if (ok) seg += e;
    }
    float s = block_hsum(seg, part, &tot);
#pragma unroll
    for (int i = 0; i < SAMPLER_PER; ++i) pr[i] = (i < per && lo + i < hi) ? pr[i] / s : -3.f;
  }
  SF();
  // (4) nucleus: repeatedly take the largest remaining probability (ties -> lowest index == stable sort).  The 25 rounds are a
  // serial chain, so a round is kept short (instead of two 5-level shuffle trees + a 27-entry rescan by the owner): every
  // thread caches the three largest remaining entries of its segment (popped in O(1), rebuilt only when exhausted), the warp
  // winner comes from two redux.sync (probabilities are >= 0, so their bit patterns order like unsigned integers; +1 keeps 0.0
  // above "nothing left"), the 8 warp winners are double-buffered so that one barrier per round suffices, and every thread
  // reduces them itself (running count / cumulative probability are thread-uniform registers).
  float c_v[3];
  int c_i[3], c_n;
  auto rebuild = [&]() {
    c_v[0] = c_v[1] = c_v[2] = -1.f;
    c_i[0] = c_i[1] = c_i[2] = -1;
#pragma unroll
    for (int i = 0; i < SAMPLER_PER; ++i) {
      const float v = pr[i];               // removed entries hold -2, entries past the segment -3
      const int ix = lo + i;
      if (v > c_v[0]) { c_v[2] = c_v[1]; c_i[2] = c_i[1]; c_v[1] = c_v[0]; c_i[1] = c_i[0]; c_v[0] = v; c_i[0] = ix; }
      else if (v > c_v[1]) { c_v[2] = c_v[1]; c_i[2] = c_i[1]; c_v[1] = v; c_i[1] = ix; }
      else if (v > c_v[2]) { c_v[2] = v; c_i[2] = ix; }
    }
    c_n = (c_v[0] >= 0.f) + (c_v[1] >= 0.f) + (c_v[2] >= 0.f);
  };
  rebuild();
  __shared__ unsigned bk[2][SAMPLER_THREADS / 32];
  __shared__ int s_cnt[SAMPLER_THREADS / 32 + 1];
  __shared__ unsigned s_thr_key;
  int n_kept = 0;
  float cum = 0.f;
  // Fast exact selection (instead of 25 serial block-wide rounds): the 25 largest entries are all >= the 25th largest
  // of the 256 per-thread maxima, so (a) rank the thread maxima (every thread counts how many precede its own: one pass over 256
  // shared entries), (b) gather the entries >= that threshold into a candidate list (typically 25-60 of 6564), (c) rank the
  // candidates the same way - order (value desc, index asc) == the reference's stable descending sort.  If the candidate list
  // overflows (hundreds of exact ties at the threshold, e.g. a distribution with < 25 non-zero entries) the serial rounds below
  // run instead; both give the same kept list.
  constexpr int CAND_CAP = 512;
  unsigned* tk = reinterpret_cast<unsigned*>(sp);          // [256] keys of the thread maxima   (sp is free until the fallback draw)
  int* ti = reinterpret_cast<int*>(sp) + SAMPLER_THREADS;     // [256] their indices
  float* cv = sp + 2 * SAMPLER_THREADS;                       // [CAND_CAP] candidate values
  int* ci = reinterpret_cast<int*>(sp) + 2 * SAMPLER_THREADS + CAND_CAP;
  bool fast_done = false;
  {
    const unsigned mykey = c_n > 0 ? __float_as_uint(c_v[0]) + 1u : 0u;
    const int myidx = c_n > 0 ? c_i[0] : 0x7fffffff;
    tk[tid] = mykey;
    ti[tid] = myidx;
    __syncthreads();
    int rank = 0;
    for (int q = 0; q < SAMPLER_THREADS / 4; ++q) {
      const uint4 k4 = reinterpret_cast<const uint4*>(tk)[q];
      const int4 i4 = reinterpret_cast<const int4*>(ti)[q];
      rank += (k4.x > mykey || (k4.x == mykey && i4.x < myidx)) + (k4.y > mykey || (k4.y == mykey && i4.y < myidx)) +
              (k4.z > mykey || (k4.z == mykey && i4.z < myidx)) + (k4.w > mykey || (k4.w == mykey && i4.w < myidx));
    }
    if (tid == 0) s_thr_key = 0u;
    __syncthreads();
    if (rank == TOPK - 1) s_thr_key = mykey;                // unique: ranks are a permutation
    __syncthreads();
    const unsigned thr = s_thr_key;
    if (thr != 0u) {
      int cnt = 0;
#pragma unroll
      for (int i = 0; i < SAMPLER_PER; ++i) cnt += (pr[i] >= 0.f && __float_as_uint(pr[i]) + 1u >= thr) ? 1 : 0;
      // exclusive offsets: warp scan + warp totals
      int incl = cnt;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if ((tid & 31) >= o) incl += t;
      }
      if ((tid & 31) == 31) s_cnt[tid >> 5] = incl;
      __syncthreads();
      int base = 0, total = 0;
#pragma unroll
      for (int w = 0; w < SAMPLER_THREADS / 32; ++w) {
        if (w < (tid >> 5)) base += s_cnt[w];
        total += s_cnt[w];
      }
      if (total <= CAND_CAP) {
        int pos = base + incl - cnt;
#pragma unroll
        for (int i = 0; i < SAMPLER_PER; ++i)
          if (pr[i] >= 0.f && __float_as_uint(pr[i]) + 1u >= thr) { cv[pos] = pr[i]; ci[pos] = lo + i; ++pos; }
        __syncthreads();
        for (int j = tid; j < total; j += SAMPLER_THREADS) {
          const float vj = cv[j];
          const int ij = ci[j];
          int r = 0;
          for (int k = 0; k < total; ++k) r += (cv[k] > vj || (cv[k] == vj && ci[k] < ij)) ? 1 : 0;
          if (r < TOPK) { kept_p[r] = vj; kept_i[r] = ij; }
        }
        __syncthreads();
        const int avail = total < TOPK ? total : TOPK;
        while (n_kept < avail && cum < 0.8f) {               // thread-uniform: every thread walks the same shared list
          cum = cum + kept_p[n_kept];
          ++n_kept;
        }
        fast_done = true;
      }
    }
  }
  for (int round = 0; round < TOPK && !fast_done; ++round) {
    if (!(cum < 0.8f)) break;             // thread-uniform
    const unsigned key = c_n > 0 ? __float_as_uint(c_v[0]) + 1u : 0u;
    const unsigned wmax = __reduce_max_sync(0xffffffffu, key);
    const int widx = __reduce_min_sync(0xffffffffu, (key == wmax && wmax != 0u) ? c_i[0] : 0x7fffffff);
    const int pb = round & 1;
    if ((tid & 31) == 0) { bk[pb][tid >> 5] = wmax; bi[pb][tid >> 5] = widx; }
    __syncthreads();
    unsigned gk = bk[pb][0];
    int gi = bi[pb][0];
#pragma unroll
    for (int w = 1; w < SAMPLER_THREADS / 32; ++w) {
      const unsigned k2 = bk[pb][w];
      const int i2 = bi[pb][w];
      if (k2 > gk || (k2 == gk && i2 < gi)) { gk = k2; gi = i2; }
    }
    if (gk == 0u) break;                  // nothing left (cannot happen: V > TOPK)
    const float gv = __uint_as_float(gk - 1u);
    if (tid == 0) {
      kept_p[n_kept] = gv;
      kept_i[n_kept] = gi;
    }
    n_kept += 1;
    cum = cum + gv;
    if (gi >= lo && gi < hi) {            // owner removes it: mark the entry, pop the cache
#pragma unroll
      for (int i = 0; i < SAMPLER_PER; ++i)
        if (lo + i == gi) pr[i] = -2.f;
      c_v[0] = c_v[1]; c_i[0] = c_i[1];
      c_v[1] = c_v[2]; c_i[1] = c_i[2];
      c_v[2] = -1.f; c_i[2] = -1;
      if (--c_n == 0) rebuild();
    }
  }
  SF();
  // (5) inverse-CDF draw over the kept (unnormalised) probabilities
  if (tid == 0) {
    int n = n_kept;
    float total = 0.f;
    for (int i = 0; i < n; ++i) total += kept_p[i];
    float thr = u1 * total, acc = 0.f;
    int pick = -1, last = -1;
    for (int i = 0; i < n; ++i) {
      if (kept_p[i] > 0.f) last = i;
      acc += kept_p[i];
      if (pick < 0 && acc > thr && kept_p[i] > 0.f) pick = i;
    }
    if (pick < 0) pick = last;
    int top = kept_i[pick];
    // (6) repetition-aware fallback (common.py:140-143): count of top in the last WIN outputs >= WIN*tau_r = 1
    int rep = 0;
    const int32_t* hist = standalone ? history + (size_t)b * hist_ld : out_ids + (size_t)b * out_ld;
    for (int i = max(0, cnt - WIN); i < cnt; ++i) rep += hist[i] == top;
    s_top = top;
    s_n = rep >= 1 ? 1 : 0;
  }
  __syncthreads();
  SF();
  if (s_n) {
    int top = s_top;
#pragma unroll
    for (int i = 0; i < SAMPLER_PER; ++i)
      if (lo + i == top) xr[i] = -INFINITY;
    float m3 = -INFINITY;
#pragma unroll
    for (int i = 0; i < SAMPLER_PER; ++i) m3 = fmaxf(m3, xr[i]);
    m3 = block_max(m3, red);
    float seg = 0.f;
#pragma unroll
    for (int i = 0; i < SAMPLER_PER; ++i) {
      const bool ok = i < per && lo + i < hi;
      float e = (!ok || xr[i] == -INFINITY) ? 0.f : expf(xr[i] - m3);
      pr[i] = e;
      if (ok) seg += e;
    }
    float s = block_hsum(seg, part, &tot);
    seg = 0.f;
#pragma unroll
    for (int i = 0; i < SAMPLER_PER; ++i) {
      if (i < per && lo + i < hi) {
        pr[i] = pr[i] / s;
        seg += pr[i];
        sp[lo + i] = pr[i];                 // the walk below reads other threads' segments
      }
    }
    // hierarchical inverse CDF (oracle draw_index): segment sums -> sequential prefix -> walk inside the segment
    __syncthreads();
    part[tid] = seg;
    __syncthreads();
    if (tid == 0) {
      float pre = 0.f;
      for (int i = 0; i < SAMPLER_THREADS; ++i) pre += part[i];
      float thr = u2 * pre;
      float acc = 0.f;
      int segi = -1, lastseg = -1;
      float segbase = 0.f, lastbase = 0.f;
      for (int i = 0; i < SAMPLER_THREADS; ++i) {
        if (part[i] > 0.f) {
          lastseg = i;
          lastbase = acc;
          if (acc + part[i] > thr) { segi = i; segbase = acc; break; }
        }
        acc += part[i];
      }
      // walk (the oracle keeps scanning later segments if rounding leaves the chosen one without a hit).  Every segment the walk
      // enters starts from its own prefix sum, as draw_index does: the element-by-element running sum can end a few ulps below the
      // segment prefix, and carried over it would let a tiny first entry of the next segment fail the threshold.
      int pick = -1, last = -1;
      if (segi < 0) { segi = lastseg; segbase = lastbase; }
      float sgbase = segbase;              // prefix sum of segment sg (part[] summed in order)
      for (int sg = segi; sg >= 0 && sg < SAMPLER_THREADS && pick < 0; ++sg) {
        const float a0 = sgbase;
        sgbase += part[sg];
        if (sg > segi && !(part[sg] > 0.f)) continue;   // prefix[sg+1] > thr holds once an earlier segment exceeded it
        float a = a0;
        int l2 = sg * per, h2 = min(l2 + per, V);
        for (int i = l2; i < h2; ++i) {
          if (sp[i] > 0.f) last = i;
          a += sp[i];
          if (a > thr && sp[i] > 0.f) { pick = i; break; }
        }
      }
      if (pick < 0) pick = last;
      s_top = pick;
    }
    __syncthreads();
  }
  SF();
  // the scores with the reference's in-place marks go back to shared memory for the coalesced write-back
#pragma unroll
  for (int i = 0; i < SAMPLER_PER; ++i)
    if (i < per && lo + i < hi) x[lo + i] = xr[i];
  __syncthreads();
  const int top = s_top;
  // the log-probs with the reference's in-place marks (eos / repeated id = -inf) go back to the caller's buffer
  // (cvk_ras_sample modifies logp like common.py does; cvk_lm_last_logits reads them)
  if ((V & 3) == 0) {
    for (int i = tid; i < V / 4; i += SAMPLER_THREADS) reinterpret_cast<float4*>(xg)[i] = reinterpret_cast<const float4*>(x)[i];
  } else {
    for (int i = tid; i < V; i += SAMPLER_THREADS) xg[i] = x[i];
  }
  SF();
  if (standalone) {
    if (tid == 0) ids_out[b] = top;
    return;
  }
  // (7) stop / length logic (llm.py:544-549)
  const bool stop = top >= EOS;      // Qwen2LM: 6561..6563 (llm.py:297); CosyVoice3LM: 6561..6760 (llm.py:704); nothing else exists above 6560
  if (!stop) {
    float ss = 0.f;
    float ev[(D + SAMPLER_THREADS - 1) / SAMPLER_THREADS];
#pragma unroll
    for (int k = 0; k < (D + SAMPLER_THREADS - 1) / SAMPLER_THREADS; ++k) {
      const int c = tid + k * SAMPLER_THREADS;
      ev[k] = c < D ? speech_emb[(size_t)top * D + c] : 0.f;
    }
#pragma unroll
    for (int k = 0; k < (D + SAMPLER_THREADS - 1) / SAMPLER_THREADS; ++k) {
      const int c = tid + k * SAMPLER_THREADS;
      if (c < D) {
        next_x[(size_t)b * D + c] = ev[k];
        ss += ev[k] * ev[k];
      }
    }
    if (xn_out) {   // fused decode path: RMSNorm of the next layer-0 input (input_layernorm of layer 0)
      ss = warp_sum(ss);
      __syncthreads();
      if ((tid & 31) == 0) red[tid >> 5] = ss;
      __syncthreads();
      float t2 = 0.f;
      for (int i = 0; i < SAMPLER_THREADS / 32; ++i) t2 += red[i];
      const float r = rsqrtf(t2 / D + RMS_EPS);
#pragma unroll
      for (int k = 0; k < (D + SAMPLER_THREADS - 1) / SAMPLER_THREADS; ++k) {
        const int c = tid + k * SAMPLER_THREADS;
        if (c < D) xn_out[(size_t)b * D + c] = __float2bfloat16_rn(ln_gamma[c] * (ev[k] * r));
      }
    }
  }
  if (tid == 0) {
    bool fin = stop;
    if (!stop) {
      out_ids[(size_t)b * out_ld + cnt] = top;
      out_count[b] = cnt + 1;
      ctx_len[b] = base_len[b] + cnt;   // cache position of the token that is fed next
      if (cnt + 1 >= max_len[b]) fin = true;
    }
    if (fin) {
      done[b] = 1;
      atomicSub(live, 1);
    }
  }
  SF();
  tl_stamp(tl, 2);
#undef SF
}

__global__ void logsoftmax_rows_kernel(float* __restrict__ x, int V) {
  __shared__ float red[SAMPLER_THREADS / 32];
  __shared__ float part[SAMPLER_THREADS];
  __shared__ float tot;
  float* row = x + (size_t)blockIdx.x * V;
  const int per = (V + SAMPLER_THREADS - 1) / SAMPLER_THREADS;
  const int lo = threadIdx.x * per, hi = min(lo + per, V);
  float mx = -INFINITY;
  for (int i = lo; i < hi; ++i) mx = fmaxf(mx, row[i]);
  mx = block_max(mx, red);
  float seg = 0.f;
  for (int i = lo; i < hi; ++i) seg += expf(row[i] - mx);
  float s = block_hsum(seg, part, &tot);
  float ls = logf(s);
  for (int i = lo; i < hi; ++i) row[i] = (row[i] - mx) - ls;
}

__global__ void init_state_kernel(const int* __restrict__ len, int B, int* ctx_len, int* base_len, int* live) {
  int b = threadIdx.x;
  if (b < B) {
    ctx_len[b] = len[b];
    base_len[b] = len[b];
  }
  if (b == 0) *live = B;
}

int* upload(cvk_ctx* ctx, const std::vector<int>& v, cudaStream_t st) {
  int* d = (int*)ctx->arena.alloc(sizeof(int) * (v.size() ? v.size() : 1));
  if (!v.empty()) CVK_CHECK_CUDA(cudaMemcpyAsync(d, v.data(), sizeof(int) * v.size(), cudaMemcpyHostToDevice, st));
  return d;
}
std::vector<int> prefix(const int* lens, int B) {
  std::vector<int> off(B);
  int a = 0;
  for (int b = 0; b < B; ++b) { off[b] = a; a += lens[b]; }
  return off;
}

// GEMM of the LM: the weight-streaming split-K kernel when there are at most 64 activation rows (decode, small feeds) and a
// split-K scratch is given, else the tiled kernel
void lm_gemm(cvk_ctx* ctx, cudaStream_t st, const Mat& A, const ConvW& W, const Epilogue& e, float* scratch, size_t scratch_floats) {
  if (scratch && A.dtype == DT_BF16 && ctx->use_tc && ctx->use_skinny && e.out.rows <= 64 && W.w16)
    conv_gemm_skinny(ctx, st, A, W, e, scratch, scratch_floats);
  else
    conv_gemm(ctx, st, A, W, e);
}

// rows [r0, r0 + n) of a row-major view
static Mat row_slice(const Mat& a, int r0, int n) { return Mat((char*)a.p + (size_t)r0 * a.ld * a.esize(), a.dtype, n, a.cols, a.ld); }

// GEMM of the ragged feed calls: every activation row gets the same arithmetic whatever rows share the call.  lm_gemm's choice
// between the skinny and the tiled kernel (different summation orders in bf16) depends on the row count, so in bf16 the rows go
// through the weight-streaming kernel in slices of at most 64; its split count depends only on the weight, and the scratch covers
// that split count at 64 rows for every LM weight, so no slice falls back to fewer splits.  fp32 (SIMT GEMM) is row-independent.
void lm_gemm_rows(cvk_ctx* ctx, cudaStream_t st, const Mat& A, const ConvW& W, const Epilogue& e, float* scratch, size_t scratch_floats) {
  if (!(scratch && A.dtype == DT_BF16 && ctx->use_tc && ctx->use_skinny && W.w16)) {
    conv_gemm(ctx, st, A, W, e);
    return;
  }
  for (int r0 = 0; r0 < e.out.rows; r0 += 64) {
    const int n = std::min(64, e.out.rows - r0);
    Epilogue es = e;
    es.out = row_slice(e.out, r0, n);
    if (e.resid.p) es.resid = row_slice(e.resid, r0, n);
    conv_gemm_skinny(ctx, st, row_slice(A, r0, n), W, es, scratch, scratch_floats);
  }
}

// one pass of a ragged feed: where each activation row goes in the cache, and the attention tiles over them (llm_feed_rows)
struct RaggedPass {
  const int2* rowpos = nullptr;   // [M] (session row, cache position)
  const int4* tiles = nullptr;    // [ntiles] see ragged_attn_tc_kernel
  int ntiles = 0;
};

// one transformer layer on `rows` rows.  prefill: seqs geometry + causal attention over the qkv buffer;
// decode: rows == sequences, attention against the cache; ragged (rg != null): rows are fed positions placed by rg, attention
// against the cache.
void layer_forward(cvk_ctx* ctx, cudaStream_t st, const LlmModel* m, int li, const Mat& x, const Mat& xn, const Mat& qkv, const Mat& att,
                   const Mat& gu, const Mat& ffa, const Seqs* s, cvk_lm_session* sess, bool decode, const RaggedPass* rg = nullptr) {
  const LayerW& w = m->layers[li];
  const int rows = x.rows;
  float* scr = rg ? sess->fscratch : (decode ? sess->scratch : nullptr);
  const size_t scr_n = rg ? sess->fscratch_floats : (decode ? sess->scratch_floats : 0);
  rmsnorm(ctx, st, x, w.ln1, RMS_EPS, xn);
  {
    Epilogue e;
    e.out = qkv;
    (rg ? lm_gemm_rows : lm_gemm)(ctx, st, xn, w.qkv, e, scr, scr_n);
  }
  size_t es = qkv.dtype == DT_F32 ? 4 : 2;
  void* kc = sess ? (char*)sess->kcache + (size_t)li * sess->max_batch * NKV * sess->max_ctx * HD * es : nullptr;
  void* vc = sess ? (char*)sess->vcache + (size_t)li * sess->max_batch * NKV * sess->max_ctx * HD * es : nullptr;
  if (rg) {
    if (qkv.dtype == DT_F32) {
      rope_append_kernel<float><<<dim3(1, rows), 128, 0, st>>>(qkv.f32(), qkv.ld, nullptr, nullptr, nullptr, m->d_inv_freq, (float*)kc,
                                                               (float*)vc, sess->max_ctx, 1, rg->rowpos);
      decode_attn_kernel<float><<<dim3(rows, NKV), (NH / NKV) * 32, (NH / NKV) * sess->max_ctx * sizeof(float), st>>>(
          qkv.f32(), qkv.ld, (const float*)kc, (const float*)vc, nullptr, sess->max_ctx, att.f32(), att.ld, rg->rowpos);
    } else {
      rope_append_kernel<bf16><<<dim3(1, rows), 128, 0, st>>>(qkv.b16(), qkv.ld, nullptr, nullptr, nullptr, m->d_inv_freq, (bf16*)kc,
                                                              (bf16*)vc, sess->max_ctx, 1, rg->rowpos);
      ragged_attn_tc_kernel<<<dim3(rg->ntiles, NKV), 32 * RA_WARPS, 0, st>>>(qkv.b16(), qkv.ld, (const bf16*)kc, (const bf16*)vc, sess->max_ctx,
                                                                              rg->tiles, att.b16(), att.ld);
    }
    ctx->launches += 2;
    CVK_LAUNCH_CHECK();
  } else if (decode) {
    if (qkv.dtype == DT_F32) {
      rope_append_kernel<float><<<dim3(1, rows), 128, 0, st>>>(qkv.f32(), qkv.ld, nullptr, nullptr, sess->ctx_len, m->d_inv_freq, (float*)kc,
                                                               (float*)vc, sess->max_ctx, 1, nullptr);
      decode_attn_kernel<float><<<dim3(rows, NKV), (NH / NKV) * 32, (NH / NKV) * sess->max_ctx * sizeof(float), st>>>(qkv.f32(), qkv.ld, (const float*)kc, (const float*)vc, sess->ctx_len, sess->max_ctx,
                                                          att.f32(), att.ld, nullptr);
    } else {
      rope_append_kernel<bf16><<<dim3(1, rows), 128, 0, st>>>(qkv.b16(), qkv.ld, nullptr, nullptr, sess->ctx_len, m->d_inv_freq, (bf16*)kc,
                                                              (bf16*)vc, sess->max_ctx, 1, nullptr);
      decode_attn_kernel<bf16><<<dim3(rows, NKV), (NH / NKV) * 32, (NH / NKV) * sess->max_ctx * sizeof(float), st>>>(qkv.b16(), qkv.ld, (const bf16*)kc, (const bf16*)vc, sess->ctx_len, sess->max_ctx,
                                                         att.b16(), att.ld, nullptr);
    }
    ctx->launches += 2;
    CVK_LAUNCH_CHECK();
  } else {
    int bx = s->max_len < 256 ? s->max_len : 256;
    // without a session (teacher-forced parity path) the cache pointers are null: append is skipped via max_ctx = 0
    int mc = sess ? sess->max_ctx : 0;
    if (qkv.dtype == DT_F32)
      rope_append_kernel<float><<<dim3(bx, s->B), 128, 0, st>>>(qkv.f32(), qkv.ld, s->d_start, s->d_len, nullptr, m->d_inv_freq, (float*)kc,
                                                                (float*)vc, mc, 0, nullptr);
    else
      rope_append_kernel<bf16><<<dim3(bx, s->B), 128, 0, st>>>(qkv.b16(), qkv.ld, s->d_start, s->d_len, nullptr, m->d_inv_freq, (bf16*)kc,
                                                               (bf16*)vc, mc, 0, nullptr);
    ctx->launches++;
    CVK_LAUNCH_CHECK();
    // causal == block-causal with chunk 1; 7 query heads per kv head
    attention_fwd(ctx, st, qkv.slice(0, NH * HD), qkv.slice(NH * HD, NKV * HD), qkv.slice(NH * HD + NKV * HD, NKV * HD), *s, NH, 1, 0.125f,
                  att, NH / NKV);
  }
  {
    Epilogue e;
    e.resid = x;
    e.out = x;
    (rg ? lm_gemm_rows : lm_gemm)(ctx, st, att, w.o, e, scr, scr_n);
  }
  rmsnorm(ctx, st, x, w.ln2, RMS_EPS, xn);
  {
    Epilogue e;
    e.out = gu;
    (rg ? lm_gemm_rows : lm_gemm)(ctx, st, xn, w.gate_up, e, scr, scr_n);
  }
  {
    size_t total = (size_t)rows * DFF;
    int g = (int)((total + 255) / 256);
    if (g > 132 * 8) g = 132 * 8;
    if (gu.dtype == DT_F32) swiglu_kernel<float><<<g, 256, 0, st>>>(gu.f32(), gu.ld, rows, ffa.f32(), ffa.ld);
    else swiglu_kernel<bf16><<<g, 256, 0, st>>>(gu.b16(), gu.ld, rows, ffa.b16(), ffa.ld);
    ctx->launches++;
    CVK_LAUNCH_CHECK();
  }
  {
    Epilogue e;
    e.resid = x;
    e.out = x;
    (rg ? lm_gemm_rows : lm_gemm)(ctx, st, ffa, w.down, e, scr, scr_n);
  }
}

void head_logits(cvk_ctx* ctx, cudaStream_t st, const LlmModel* m, const Mat& hidden_f32, const Mat& xn_act, const Mat& logits,
                 cvk_lm_session* sess = nullptr) {
  rmsnorm(ctx, st, hidden_f32, m->final_norm, RMS_EPS, xn_act);
  Epilogue e;
  e.out = logits;
  lm_gemm(ctx, st, xn_act, m->head, e, sess ? sess->scratch : nullptr, sess ? sess->scratch_floats : 0);
}

// Let decode_attn_kernel hold the scores of max_ctx positions for its 7 query heads in shared memory.  The limit is per function,
// not per session: it is never lowered for a smaller context requested later.
void decode_attn_allow_ctx(int max_ctx) {
  static int decode_attn_smem = 0;
  const size_t need = (size_t)(NH / NKV) * max_ctx * sizeof(float);
  CVK_REQUIRE(need <= 200 * 1024, "session context too long for the decode attention kernel (max ~7300 positions)");
  if ((int)need > decode_attn_smem) {
    CVK_CHECK_CUDA(cudaFuncSetAttribute(decode_attn_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)need));
    CVK_CHECK_CUDA(cudaFuncSetAttribute(decode_attn_kernel<bf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)need));
    decode_attn_smem = (int)need;
  }
}

constexpr size_t ATTN_FUSED_SMEM = ((NH / NKV + 2) * HD + AF_WARPS * 8 * 2 + AF_WARPS * (NH / NKV) * HD) * sizeof(float);

}  // namespace

// RoPE frequencies of the half-split rotation (theta 1e6): the table every LM decode / prefill kernel reads
void lm_rope_inv_freq(float* out) {
  for (int i = 0; i < HD / 2; ++i) out[i] = 1.0f / powf(ROPE_THETA, (float)(2 * i) / (float)HD);
}

// One decode-attention step on a caller-supplied cache, without a loaded LM (cvk_op_decode_attention): the qkv split-K partial sums
// [splits][rows][1152] + bias -> RoPE at position ctx_len[b] -> append k, v to the cache -> GQA attention over positions
// 0..ctx_len[b].  The caches [rows][NKV][max_ctx][64] cross the call as fp32 and run as bf16, as in a session.  lm_fused selects
// attn_fused_kernel (the decode graph's kernel) or the per-op pair rope_append_kernel + decode_attn_kernel.
void llm_decode_attention_op(cvk_ctx* ctx, const float* partial, int splits, int rows, const float* bias, float* k_cache, float* v_cache,
                             const int* ctx_len_host, int max_ctx, float* out, cudaStream_t st) {
  decode_attn_allow_ctx(max_ctx);      // the context limit of a session, whichever kernel runs
  ctx->arena.reset();
  float inv[HD / 2];
  lm_rope_inv_freq(inv);
  float* d_inv = (float*)ctx->arena.alloc(sizeof(inv));
  CVK_CHECK_CUDA(cudaMemcpyAsync(d_inv, inv, sizeof(inv), cudaMemcpyHostToDevice, st));
  int* d_len = upload(ctx, std::vector<int>(ctx_len_host, ctx_len_host + rows), st);
  const int cache_rows = rows * NKV * max_ctx;
  Mat k32(k_cache, DT_F32, cache_rows, HD, HD), v32(v_cache, DT_F32, cache_rows, HD, HD);
  Mat kc = arena_mat(ctx, DT_BF16, cache_rows, HD, HD), vc = arena_mat(ctx, DT_BF16, cache_rows, HD, HD);
  Mat att = arena_mat(ctx, DT_BF16, rows, D, D);
  convert_mat(ctx, st, k32, kc);
  convert_mat(ctx, st, v32, vc);
  if (ctx->lm_fused) {
    launch_ex(attn_fused_kernel, dim3(rows, NKV), dim3(32 * AF_WARPS), ATTN_FUSED_SMEM, st, false, partial, splits, rows, bias, kc.b16(),
              vc.b16(), (const int*)d_len, max_ctx, (const float*)d_inv, att.b16(), att.ld, (long long*)nullptr);
    ctx->launches++;
  } else {
    Mat qkv = arena_mat(ctx, DT_BF16, rows, QKV_N, QKV_N);
    qkv_reduce_kernel<<<ceil_div(rows * QKV_N, 256), 256, 0, st>>>(partial, splits, rows, bias, qkv.b16());
    rope_append_kernel<bf16><<<dim3(1, rows), 128, 0, st>>>(qkv.b16(), qkv.ld, nullptr, nullptr, d_len, d_inv, kc.b16(), vc.b16(), max_ctx, 1, nullptr);
    decode_attn_kernel<bf16><<<dim3(rows, NKV), (NH / NKV) * 32, (NH / NKV) * max_ctx * sizeof(float), st>>>(
        qkv.b16(), qkv.ld, kc.b16(), vc.b16(), d_len, max_ctx, att.b16(), att.ld, nullptr);
    ctx->launches += 3;
  }
  CVK_LAUNCH_CHECK();
  convert_mat(ctx, st, kc, k32);
  convert_mat(ctx, st, vc, v32);
  convert_mat(ctx, st, att, Mat(out, DT_F32, rows, D, D));
  CVK_CHECK_CUDA(cudaStreamSynchronize(st));
}

// The tensor-core attention of a ragged feed on a caller-supplied cache, without a loaded LM (cvk_op_ragged_attention): q [M][896]
// (already rotated), caches [cache_rows][NKV][max_ctx][64], query m = (cache row rowpos[2m], position rowpos[2m+1]) attending to
// keys 0..position.  Consecutive queries of one row at consecutive positions share a tile, as in llm_feed_rows.  Everything crosses
// the call as fp32 and runs as bf16, as in a session.
void llm_ragged_attention_op(cvk_ctx* ctx, const float* q, const float* k_cache, const float* v_cache, int cache_rows, int max_ctx,
                             const int* rowpos, int M, float* out, cudaStream_t st) {
  for (int i = 0; i < M; ++i)
    CVK_REQUIRE(rowpos[2 * i] >= 0 && rowpos[2 * i] < cache_rows && rowpos[2 * i + 1] >= 0 && rowpos[2 * i + 1] < max_ctx,
                "cvk_op_ragged_attention: row or position out of range");
  std::vector<int> tiles;
  for (int i = 0; i < M;) {
    const int n = (i + 1 < M && rowpos[2 * i + 2] == rowpos[2 * i] && rowpos[2 * i + 3] == rowpos[2 * i + 1] + 1) ? 2 : 1;
    tiles.insert(tiles.end(), {i, rowpos[2 * i], rowpos[2 * i + 1], n});
    i += n;
  }
  ctx->arena.reset();
  const int ntiles = (int)tiles.size() / 4;
  int* d_tiles = upload(ctx, tiles, st);
  const int crows = cache_rows * NKV * max_ctx;
  Mat q16 = arena_mat(ctx, DT_BF16, M, D, D), kc = arena_mat(ctx, DT_BF16, crows, HD, HD), vc = arena_mat(ctx, DT_BF16, crows, HD, HD),
      att = arena_mat(ctx, DT_BF16, M, D, D);
  convert_mat(ctx, st, Mat(const_cast<float*>(q), DT_F32, M, D, D), q16);
  convert_mat(ctx, st, Mat(const_cast<float*>(k_cache), DT_F32, crows, HD, HD), kc);
  convert_mat(ctx, st, Mat(const_cast<float*>(v_cache), DT_F32, crows, HD, HD), vc);
  ragged_attn_tc_kernel<<<dim3(ntiles, NKV), 32 * RA_WARPS, 0, st>>>(q16.b16(), q16.ld, kc.b16(), vc.b16(), max_ctx,
                                                                     reinterpret_cast<const int4*>(d_tiles), att.b16(), att.ld);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  convert_mat(ctx, st, att, Mat(out, DT_F32, M, D, D));
  CVK_CHECK_CUDA(cudaStreamSynchronize(st));
}

// ================================================================================================ build / session
void llm_build(cvk_ctx* ctx, const int* cfg, int ncfg) {
  LlmModel* m = new LlmModel();
  if (ncfg >= 1) m->num_layers = cfg[0];
  const std::string P = "llm.";
  m->text_emb = copy_param(ctx, P + "llm.model.model.embed_tokens.weight");
  m->speech_emb = copy_param(ctx, P + "speech_embedding.weight");
  if (ctx->has_raw(P + "llm_embedding.weight")) {          // Qwen2LM (CosyVoice2)
    m->llm_emb = copy_param(ctx, P + "llm_embedding.weight");
    m->head = make_linear(ctx, P + "llm_decoder.weight", P + "llm_decoder.bias");
  } else {
    // CosyVoice3LM (llm.py:664-705): sos / task_id are rows 6561 / 6563 of speech_embedding; the head has 6761 outputs and no bias.
    // The head is padded to 6764 rows (16-byte logits pitch for the TMA epilogues); the 3 pad ids get a bias of -1e30, i.e.
    // probability exactly 0 after the softmax, so sampling, log-probs and the stop rule (id >= 6561) see the reference's vocabulary.
    const RawTensor& se = ctx->get_raw(P + "speech_embedding.weight");
    const RawTensor& hw = ctx->get_raw(P + "llm_decoder.weight");
    CVK_REQUIRE(se.shape[0] == VOUT3 && hw.shape[0] == VOUT3 && hw.shape[1] == D, "CosyVoice3LM: speech_embedding / llm_decoder must have 6761 rows");
    m->llm_emb = (float*)ctx->dmalloc(2 * D * sizeof(float));
    CVK_CHECK_CUDA(cudaMemcpy(m->llm_emb, se.p + (size_t)EOS * D, D * sizeof(float), cudaMemcpyDeviceToDevice));               // sos = 6561
    CVK_CHECK_CUDA(cudaMemcpy(m->llm_emb + D, se.p + (size_t)(EOS + 2) * D, D * sizeof(float), cudaMemcpyDeviceToDevice));     // task_id = 6563
    float* wpad = (float*)ctx->dmalloc((size_t)VOUT3_PAD * D * sizeof(float));
    CVK_CHECK_CUDA(cudaMemset(wpad, 0, (size_t)VOUT3_PAD * D * sizeof(float)));
    CVK_CHECK_CUDA(cudaMemcpy(wpad, hw.p, (size_t)VOUT3 * D * sizeof(float), cudaMemcpyDeviceToDevice));
    std::vector<float> hb(VOUT3_PAD, 0.f);
    for (int i = VOUT3; i < VOUT3_PAD; ++i) hb[i] = -1.0e30f;
    float* bpad = (float*)ctx->dmalloc(VOUT3_PAD * sizeof(float));
    CVK_CHECK_CUDA(cudaMemcpy(bpad, hb.data(), VOUT3_PAD * sizeof(float), cudaMemcpyHostToDevice));
    m->head = make_conv(ctx, wpad, bpad, VOUT3_PAD, D, 1, 1, 0);
    m->vout = VOUT3_PAD;
  }
  m->final_norm = copy_param(ctx, P + "llm.model.model.norm.weight");
  if (ctx->precision == CVK_PREC_BF16) skinny_tiled_weights(ctx, m->head);
  for (int i = 0; i < m->num_layers; ++i) {
    std::string L = P + "llm.model.model.layers." + std::to_string(i);
    LayerW w;
    w.ln1 = copy_param(ctx, L + ".input_layernorm.weight");
    w.ln2 = copy_param(ctx, L + ".post_attention_layernorm.weight");
    w.qkv = concat_linear(ctx, {L + ".self_attn.q_proj.weight", L + ".self_attn.k_proj.weight", L + ".self_attn.v_proj.weight"},
                          {L + ".self_attn.q_proj.bias", L + ".self_attn.k_proj.bias", L + ".self_attn.v_proj.bias"});
    w.o = make_linear(ctx, L + ".self_attn.o_proj.weight", "");
    w.gate_up = concat_linear(ctx, {L + ".mlp.gate_proj.weight", L + ".mlp.up_proj.weight"}, {});
    w.down = make_linear(ctx, L + ".mlp.down_proj.weight", "");
    if (ctx->precision == CVK_PREC_BF16) {
      w.gate_up_il.N = 2 * DFF; w.gate_up_il.K = D;
      w.gate_up_il.w32 = (float*)ctx->dmalloc((size_t)2 * DFF * D * sizeof(float));
      interleave_rows_kernel<<<132 * 8, 256>>>(w.gate_up.w32, w.gate_up_il.w32, DFF, D);
      CVK_LAUNCH_CHECK();
      finish_convw(ctx, w.gate_up_il);
    }
    if (ctx->precision == CVK_PREC_BF16) {
      skinny_tiled_weights(ctx, w.qkv); skinny_tiled_weights(ctx, w.o); skinny_tiled_weights(ctx, w.gate_up); skinny_tiled_weights(ctx, w.down);
      skinny_tiled_weights(ctx, w.gate_up_il);
      CVK_CHECK_CUDA(cudaFree(w.gate_up_il.w32));   // only the bf16 streaming copy is used
      for (auto it = ctx->owned.begin(); it != ctx->owned.end(); ++it) if (*it == (void*)w.gate_up_il.w32) { ctx->owned.erase(it); break; }
      w.gate_up_il.w32 = nullptr;
    }
    m->layers.push_back(w);
  }
  lm_rope_inv_freq(m->inv_freq);
  m->d_inv_freq = (float*)ctx->dmalloc(sizeof(m->inv_freq));
  CVK_CHECK_CUDA(cudaMemcpy(m->d_inv_freq, m->inv_freq, sizeof(m->inv_freq), cudaMemcpyHostToDevice));
  CVK_CHECK_CUDA(cudaDeviceSynchronize());
  ctx->llm = m;
  if (ctx->precision == CVK_PREC_BF16) lm_mega_build(ctx, m);
}

cvk_lm_session* llm_session_create(cvk_ctx* ctx, int max_batch, int max_context) {
  CVK_REQUIRE(ctx->llm, "llm stage not finalised");
  cvk_lm_session* s = new cvk_lm_session();
  s->max_batch = max_batch;
  s->max_ctx = max_context;
  s->kv_dtype = ctx->act_dtype;
  size_t es = s->kv_dtype == DT_F32 ? 4 : 2;
  auto alloc = [&](size_t bytes) {
    void* p = nullptr;
    CVK_CHECK_CUDA(cudaMalloc(&p, bytes ? bytes : 16));
    CVK_CHECK_CUDA(cudaMemset(p, 0, bytes));
    s->owned.push_back(p);
    return p;
  };
  size_t cache = (size_t)ctx->llm->num_layers * max_batch * NKV * max_context * HD * es;
  s->kcache = alloc(cache);
  s->vcache = alloc(cache);
  s->ctx_len = (int*)alloc(sizeof(int) * max_batch);
  s->base_len = (int*)alloc(sizeof(int) * max_batch);
  CVK_CHECK_CUDA(cudaFuncSetAttribute(ras_sampler_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sampler_smem(VOUT3_PAD)));
  CVK_REQUIRE((NH / NKV) * max_context * sizeof(float) <= 200 * 1024, "session context too long for the decode attention kernel");
  decode_attn_allow_ctx(max_context);
  // keep every kernel of the decode step on the same (maximum) shared-memory carveout: alternating carveouts between
  // consecutive kernels forces an SM reconfiguration (idle + several microseconds) at every boundary
  CVK_CHECK_CUDA(cudaFuncSetAttribute(attn_fused_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  CVK_CHECK_CUDA(cudaFuncSetAttribute(finish_rms_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  CVK_CHECK_CUDA(cudaFuncSetAttribute(ras_sampler_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  skinny_set_carveout();
  CVK_CHECK_CUDA(cudaFuncSetAttribute(attn_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ATTN_FUSED_SMEM));
  s->count = (int*)alloc(sizeof(int) * max_batch);
  s->done = (int*)alloc(sizeof(int) * max_batch);
  s->live = (int*)alloc(sizeof(int));
  s->x = (float*)alloc(sizeof(float) * max_batch * D);
  s->hidden = (float*)alloc(sizeof(float) * max_batch * D);
  s->logits = (float*)alloc(sizeof(float) * (size_t)max_batch * VOUT3_PAD);   // large enough for either head
  s->xn = alloc(es * max_batch * D);
  s->qkv = alloc(es * max_batch * QKV_N);
  s->att = alloc(es * max_batch * D);
  s->gu = alloc(es * (size_t)max_batch * 2 * DFF);
  s->ffa = alloc(es * (size_t)max_batch * DFF);
  s->scratch_floats = skinny_scratch_floats(max_batch, 2 * DFF);
  s->scratch = (float*)alloc(s->scratch_floats * sizeof(float));
  s->sel = (int*)alloc(sizeof(int) * max_batch);
  s->rows_fed.assign(max_batch, 0);
  lm_mega_session_init(ctx, s);
  return s;
}

void llm_session_destroy(cvk_ctx* ctx, cvk_lm_session* s) {
  cudaSetDevice(ctx->device);
  // the caller guarantees that no call on this session is in flight on the host; device work still queued on the caller's
  // stream is drained by cudaFree (it synchronises the device implicitly) before the buffers go away
  if (s->graph) cudaGraphExecDestroy(s->graph);
  for (void* p : s->owned) cudaFree(p);
  lm_mega_session_free(s);
  delete s;
}

// ================================================================================================ prefill
// full causal forward over packed rows; if sess != null also fills the KV cache
static Mat forward_packed(cvk_ctx* ctx, cudaStream_t st, const Seqs& s, const Mat& x, cvk_lm_session* sess) {
  const LlmModel* m = ctx->llm;
  const int adt = ctx->act_dtype;
  Mat xn = arena_mat(ctx, adt, s.R, D), qkv = arena_mat(ctx, adt, s.R, QKV_N), att = arena_mat(ctx, adt, s.R, D),
      gu = arena_mat(ctx, adt, s.R, 2 * DFF), ffa = arena_mat(ctx, adt, s.R, DFF);
  zero_mat(ctx, st, att);
  for (int li = 0; li < m->num_layers; ++li) layer_forward(ctx, st, m, li, x, xn, qkv, att, gu, ffa, &s, sess, false);
  return x;
}

void llm_prefill(cvk_ctx* ctx, cvk_lm_session* sess, const int32_t* text, const int* text_lens, const int32_t* speech,
                 const int* speech_lens, int B, cudaStream_t st) {
  const LlmModel* m = ctx->llm;
  CVK_REQUIRE(m, "llm stage not finalised");
  CVK_REQUIRE(B <= sess->max_batch, "batch larger than the session");
  ctx->arena.reset();
  std::vector<int> lens(B);
  for (int b = 0; b < B; ++b) {
    lens[b] = 1 + text_lens[b] + 1 + speech_lens[b];
    CVK_REQUIRE(lens[b] < sess->max_ctx, "prompt longer than the session context");
  }
  Seqs s = make_seqs(ctx, lens.data(), B, 0, 1, 0, st);
  Mat x = arena_mat(ctx, DT_F32, s.R, D, D);
  zero_mat(ctx, st, x);
  int* toff = upload(ctx, prefix(text_lens, B), st);
  int* tlen = upload(ctx, std::vector<int>(text_lens, text_lens + B), st);
  int* soff = upload(ctx, prefix(speech_lens, B), st);
  int* slen = upload(ctx, std::vector<int>(speech_lens, speech_lens + B), st);
  int bx = s.max_len < 512 ? s.max_len : 512;
  build_input_kernel<<<dim3(bx, B), 128, 0, st>>>(text, toff, tlen, speech, soff, slen, m->text_emb, m->llm_emb, m->speech_emb, s.d_start, x.f32());
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  if (sess->graph) {   // a new batch invalidates the captured decode graph (row count / output pointers may change)
    cudaGraphExecDestroy(sess->graph);
    sess->graph = nullptr;
  }
  forward_packed(ctx, st, s, x, sess);
  // the first decode step consumes the hidden state of the last prompt position: keep its pre-norm residual in x
  gather_last_kernel<<<B, 128, 0, st>>>(x.f32(), s.d_start, s.d_len, sess->hidden);
  CVK_REQUIRE(sess->max_batch <= 1024, "max_batch > 1024");
  init_state_kernel<<<1, sess->max_batch < 32 ? 32 : round_up(sess->max_batch, 32), 0, st>>>(s.d_len, B, sess->ctx_len, sess->base_len, sess->live);
  sess->fresh = true;
  sess->ragged = false;
  ctx->launches += 2;
  CVK_LAUNCH_CHECK();
  sess->B = B;
}

// ================================================================================================ decode
// One device step = head + sampler on the current hidden state (emits token k, gathers its embedding into x), then the
// 24 layers on x (position base_len + k) leaving the next hidden state.  The reference's loop (llm.py:538-549) is the
// same sequence rotated by half a step: its first iteration is the prefill.
static bool lm_fused_path(cvk_ctx* ctx, cvk_lm_session* s) {
  return s->kv_dtype == DT_BF16 && ctx->use_tc && ctx->use_skinny && ctx->lm_fused && s->g_B <= 64;
}

// The layers of a bf16 decode step on the fused path: x (residual stream) and xn = RMSNorm(x) ln1[0] in -> x, xn = the final-normed
// hidden state out; every layer appends its K / V row at ctx_len.  Persistent kernel when it can run, else the PDL chain of 7
// launches per layer.  decode_step_fused runs it after the sampler, cvk_op_lm_decode_layers on caller state.
static void decode_layers_fused(cvk_ctx* ctx, cudaStream_t st, cvk_lm_session* s) {
  const LlmModel* m = ctx->llm;
  const int B = s->g_B;
  if (lm_mega_usable(ctx, s, B)) {     // all layers in one persistent cooperative kernel (llm_mega.cu)
    lm_mega_layers(ctx, st, s, B);
    return;
  }
  const bool pdl = ctx->pdl != 0;
  Mat xn(s->xn, DT_BF16, B, D, D), att(s->att, DT_BF16, B, D, D), ffa(s->ffa, DT_BF16, B, DFF, DFF);
  for (int li = 0; li < m->num_layers; ++li) {
    const LayerW& w = m->layers[li];
    bf16* kc = (bf16*)s->kcache + (size_t)li * s->max_batch * NKV * s->max_ctx * HD;
    bf16* vc = (bf16*)s->vcache + (size_t)li * s->max_batch * NKV * s->max_ctx * HD;
    Epilogue none;
    int sp = conv_gemm_skinny_ex(ctx, st, xn, w.qkv, none, s->scratch, s->scratch_floats, 1);
    launch_ex(attn_fused_kernel, dim3(B, NKV), dim3(32 * AF_WARPS), ATTN_FUSED_SMEM, st, pdl, (const float*)s->scratch, sp, B,
              (const float*)w.qkv.bias, kc, vc, (const int*)s->ctx_len, s->max_ctx, (const float*)m->d_inv_freq, att.b16(), att.ld, ctx->tl_next());
    ctx->launches++;
    CVK_LAUNCH_CHECK();
    sp = conv_gemm_skinny_ex(ctx, st, att, w.o, none, s->scratch, s->scratch_floats, 1);
    launch_ex(finish_rms_kernel, dim3(B), dim3(D), 0, st, pdl, (const float*)s->scratch, sp, B, s->x, (const float*)w.ln2, xn.b16(), ctx->tl_next());
    ctx->launches++;
    CVK_LAUNCH_CHECK();
    {
      Epilogue e;
      e.out = ffa;
      conv_gemm_skinny_ex(ctx, st, xn, w.gate_up_il, e, s->scratch, s->scratch_floats, 2);
    }
    sp = conv_gemm_skinny_ex(ctx, st, ffa, w.down, none, s->scratch, s->scratch_floats, 1);
    const float* next_gamma = li + 1 < m->num_layers ? m->layers[li + 1].ln1 : m->final_norm;
    launch_ex(finish_rms_kernel, dim3(B), dim3(D), 0, st, pdl, (const float*)s->scratch, sp, B, s->x, next_gamma, xn.b16(), ctx->tl_next());
    ctx->launches++;
    CVK_LAUNCH_CHECK();
  }
}

// bf16 decode step with fused kernels: 2 + 7 launches per layer instead of 2 + 12
static void decode_step_fused(cvk_ctx* ctx, cudaStream_t st, cvk_lm_session* s) {
  const LlmModel* m = ctx->llm;
  const int B = s->g_B;
  const bool fused = true;
  ctx->tl_seq = 0;
  Mat xn(s->xn, DT_BF16, B, D, D), logits(s->logits, DT_F32, B, m->vout, m->vout);
  {
    Epilogue e;
    e.out = logits;
    conv_gemm_skinny_ex(ctx, st, xn, m->head, e, s->scratch, s->scratch_floats, 0);
  }
  const bool pdl = ctx->pdl != 0;
  launch_ex(ras_sampler_kernel, dim3(B), dim3(SAMPLER_THREADS), sampler_smem(m->vout), st, pdl, s->logits, m->vout, 1, s->g_uniforms, B, s->g_min,
            s->g_max, s->g_out_ids, s->g_out_ld, s->g_out_count, s->g_done, s->ctx_len, (const int*)s->base_len, s->live,
            (const float*)m->speech_emb, s->x, (const int32_t*)nullptr, 0, (const int32_t*)nullptr, (const int32_t*)nullptr, (int32_t*)nullptr,
            (const float*)(fused ? m->layers[0].ln1 : nullptr), fused ? (bf16*)s->xn : (bf16*)nullptr, ctx->tl_next(),
            ctx->tl ? (long long*)ctx->tl + 1024 : (long long*)nullptr);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  decode_layers_fused(ctx, st, s);
}

static void decode_step(cvk_ctx* ctx, cudaStream_t st, cvk_lm_session* s) {
  if (lm_fused_path(ctx, s)) {
    decode_step_fused(ctx, st, s);
    return;
  }
  const LlmModel* m = ctx->llm;
  const int adt = s->kv_dtype;
  const int B = s->g_B;
  const bool fused = false;
  Mat hid(s->hidden, DT_F32, B, D, D), x(s->x, DT_F32, B, D, D), xn(s->xn, adt, B, D, D), qkv(s->qkv, adt, B, QKV_N, QKV_N),
      att(s->att, adt, B, D, D), gu(s->gu, adt, B, 2 * DFF, 2 * DFF), ffa(s->ffa, adt, B, DFF, DFF), logits(s->logits, DT_F32, B, m->vout, m->vout);
  head_logits(ctx, st, m, hid, xn, logits, s);
  ras_sampler_kernel<<<B, SAMPLER_THREADS, sampler_smem(m->vout), st>>>(s->logits, m->vout, 1, s->g_uniforms, B, s->g_min, s->g_max, s->g_out_ids,
                                                                       s->g_out_ld, s->g_out_count, s->g_done, s->ctx_len, s->base_len, s->live,
                                                                       m->speech_emb, s->x, nullptr, 0, nullptr, nullptr, nullptr, fused ? m->layers[0].ln1 : nullptr,
                                                                       fused ? (bf16*)s->xn : nullptr, nullptr, nullptr);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  for (int li = 0; li < m->num_layers; ++li) layer_forward(ctx, st, m, li, x, xn, qkv, att, gu, ffa, nullptr, s, true);
  CVK_CHECK_CUDA(cudaMemcpyAsync(s->hidden, s->x, sizeof(float) * (size_t)B * D, cudaMemcpyDeviceToDevice, st));
}

void llm_decode(cvk_ctx* ctx, cvk_lm_session* s, int n_steps, const float* uniforms, const int32_t* min_len, const int32_t* max_len,
                int32_t* out_ids, int out_ld, int32_t* out_count, int32_t* done, int* live_host, cudaStream_t st) {
  const LlmModel* m = ctx->llm;
  CVK_REQUIRE(m && s->B > 0, "cvk_lm_prefill must run before cvk_lm_decode");
  const int B = s->B;
  s->ragged = false;   // the decode steps advance ctx_len on the device only
  const bool was_fresh = s->fresh;
  if (s->fresh) {
    CVK_CHECK_CUDA(cudaMemsetAsync(out_count, 0, sizeof(int32_t) * B, st));
    CVK_CHECK_CUDA(cudaMemsetAsync(done, 0, sizeof(int32_t) * B, st));
    s->fresh = false;
  }
  bool same = s->g_out_count == out_count && s->g_done == done && s->g_out_ids == out_ids && s->g_uniforms == uniforms &&
              s->g_min == min_len && s->g_max == max_len && s->g_out_ld == out_ld && s->g_B == B && s->g_pdl == ctx->pdl &&
              s->g_mega == ctx->lm_mega;
  if (!same) {
    if (s->graph) {
      cudaGraphExecDestroy(s->graph);
      s->graph = nullptr;
    }
    s->g_out_count = out_count; s->g_done = done; s->g_out_ids = out_ids; s->g_uniforms = uniforms; s->g_min = min_len; s->g_max = max_len;
    s->g_out_ld = out_ld; s->g_B = B; s->g_pdl = ctx->pdl; s->g_mega = ctx->lm_mega;
  }
  s->g_B = B;
  if (was_fresh && lm_fused_path(ctx, s)) {
    // the fused step expects the final-normed hidden state of the previous position in xn
    Mat hid(s->hidden, DT_F32, B, D, D), xn(s->xn, DT_BF16, B, D, D);
    rmsnorm(ctx, st, hid, m->final_norm, RMS_EPS, xn);
  }
  const bool can_graph = ctx->use_graph && st != nullptr && st != cudaStreamLegacy && st != cudaStreamPerThread;   // capture is illegal on the default streams
  if (can_graph && !s->graph) {
    cudaGraph_t graph = nullptr;
    CVK_CHECK_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    cvk_in_capture = 1;
    try {
      decode_step(ctx, st, s);
      cvk_in_capture = 0;
    } catch (...) {
      cvk_in_capture = 0;
      cudaStreamEndCapture(st, &graph);
      if (graph) cudaGraphDestroy(graph);
      throw;
    }
    CVK_CHECK_CUDA(cudaStreamEndCapture(st, &graph));
    // kernels of the step = kernel nodes of the graph (other threads launch concurrently, so the context counter cannot tell); the
    // captured launches were counted while capturing and are counted again at every replay
    size_t n_nodes = 0;
    CVK_CHECK_CUDA(cudaGraphGetNodes(graph, nullptr, &n_nodes));
    std::vector<cudaGraphNode_t> nodes(n_nodes);
    if (n_nodes) CVK_CHECK_CUDA(cudaGraphGetNodes(graph, nodes.data(), &n_nodes));
    int64_t kernels = 0;
    for (cudaGraphNode_t n : nodes) {
      cudaGraphNodeType t;
      CVK_CHECK_CUDA(cudaGraphNodeGetType(n, &t));
      kernels += t == cudaGraphNodeTypeKernel;
    }
    CVK_CHECK_CUDA(cudaGraphInstantiate(&s->graph, graph, 0));
    cudaGraphDestroy(graph);
    s->graph_kernels = kernels;
    ctx->launches -= kernels;
  }
  for (int i = 0; i < n_steps; ++i) {
    if (can_graph && s->graph) {
      CVK_CHECK_CUDA(cudaGraphLaunch(s->graph, st));
      ctx->launches += s->graph_kernels;
    } else {
      decode_step(ctx, st, s);
    }
  }
  if (live_host) {
    CVK_CHECK_CUDA(cudaMemcpyAsync(live_host, s->live, sizeof(int), cudaMemcpyDeviceToHost, st));
    CVK_CHECK_CUDA(cudaStreamSynchronize(st));
  }
}

// The layers of one decode step on caller state (cvk_op_lm_decode_layers), on a temporary session of B rows x max_ctx positions:
// the layer loop cvk_lm_decode runs after the sampler, on the path the step would take (decode_step: the fused chain or the persistent
// kernel, else the per-op loop).  x [B][896] fp32 in / out; the caches [layers][B][2][max_ctx][64] cross the call as fp32 and run as
// bf16, each layer appending its row at ctx_len_host[b]; xn_out [B][896] the bf16 final-normed row the step hands to the head;
// att_out [B][896] / ffa_out [B][4864] (nullable) the last layer's o_proj / down_proj operands, which every path leaves in the session's
// att / ffa buffers.  The entry xn = RMSNorm(x) ln1[0], which the sampler computes in a step, comes from the path's own norm kernel.
void llm_decode_layers_op(cvk_ctx* ctx, int B, const int* ctx_len_host, int max_ctx, float* x, float* k_cache, float* v_cache,
                          float* xn_out, float* att_out, float* ffa_out, cudaStream_t st) {
  const LlmModel* m = ctx->llm;
  ctx->arena.reset();
  cvk_lm_session* s = llm_session_create(ctx, B, max_ctx);
  try {
    s->B = s->g_B = B;
    const int cache_rows = m->num_layers * B * NKV * max_ctx;
    Mat k32(k_cache, DT_F32, cache_rows, HD, HD), v32(v_cache, DT_F32, cache_rows, HD, HD);
    Mat kc(s->kcache, DT_BF16, cache_rows, HD, HD), vc(s->vcache, DT_BF16, cache_rows, HD, HD);
    Mat xs(s->x, DT_F32, B, D, D), xn(s->xn, DT_BF16, B, D, D), att(s->att, DT_BF16, B, D, D), ffa(s->ffa, DT_BF16, B, DFF, DFF);
    CVK_CHECK_CUDA(cudaMemcpyAsync(s->ctx_len, ctx_len_host, sizeof(int) * B, cudaMemcpyHostToDevice, st));
    CVK_CHECK_CUDA(cudaMemcpyAsync(s->x, x, sizeof(float) * (size_t)B * D, cudaMemcpyDeviceToDevice, st));
    convert_mat(ctx, st, k32, kc);
    convert_mat(ctx, st, v32, vc);
    if (lm_fused_path(ctx, s)) {
      // no split to add: finish_rms_kernel is the plain RMSNorm of x
      launch_ex(finish_rms_kernel, dim3(B), dim3(D), 0, st, ctx->pdl != 0, (const float*)s->scratch, 0, B, s->x, (const float*)m->layers[0].ln1,
                xn.b16(), (long long*)nullptr);
      ctx->launches++;
      CVK_LAUNCH_CHECK();
      decode_layers_fused(ctx, st, s);
    } else {
      Mat qkv(s->qkv, DT_BF16, B, QKV_N, QKV_N), gu(s->gu, DT_BF16, B, 2 * DFF, 2 * DFF);
      for (int li = 0; li < m->num_layers; ++li) layer_forward(ctx, st, m, li, xs, xn, qkv, att, gu, ffa, nullptr, s, true);
      rmsnorm(ctx, st, xs, m->final_norm, RMS_EPS, xn);     // what head_logits does at the next step
    }
    CVK_CHECK_CUDA(cudaMemcpyAsync(x, s->x, sizeof(float) * (size_t)B * D, cudaMemcpyDeviceToDevice, st));
    convert_mat(ctx, st, kc, k32);
    convert_mat(ctx, st, vc, v32);
    convert_mat(ctx, st, xn, Mat(xn_out, DT_F32, B, D, D));
    if (att_out) convert_mat(ctx, st, att, Mat(att_out, DT_F32, B, D, D));
    if (ffa_out) convert_mat(ctx, st, ffa, Mat(ffa_out, DT_F32, B, DFF, DFF));
    CVK_CHECK_CUDA(cudaStreamSynchronize(st));
  } catch (...) {
    cudaStreamSynchronize(st);
    llm_session_destroy(ctx, s);
    throw;
  }
  llm_session_destroy(ctx, s);
}

// ---------------------------------------------------------------------------------------------- incremental feeding
// Primitives for the text-streaming LM (Qwen2LM.inference_bistream, llm.py:551-661), whose control flow (5 text : 15 speech
// interleaving, fill-token forcing) lives on the host: start an empty session, push arbitrary embeddings (text ids ->
// embed_tokens, speech ids -> speech_embedding, 0/1 -> llm_embedding sos/task) through the cached decode path one position at a
// time, read the log-probabilities of the next token.  Sampling is cvk_ras_sample.
namespace {
__global__ void feed_embed_kernel(int kind, int id, int B, const float* __restrict__ text_emb, const float* __restrict__ llm_emb,
                                  const float* __restrict__ speech_emb, float* __restrict__ x) {
  const float* src = kind == 0 ? text_emb + (size_t)id * D : (kind == 1 ? speech_emb + (size_t)id * D : llm_emb + (size_t)id * D);
  for (int b = 0; b < B; ++b)
    for (int c = threadIdx.x; c < D; c += blockDim.x) x[(size_t)b * D + c] = src[c];
}
__global__ void bump_ctx_kernel(int* __restrict__ ctx_len, int B) {
  if (threadIdx.x < B) ctx_len[threadIdx.x] += 1;
}
__global__ void zero_state_kernel(int* ctx_len, int* base_len, int* live, int n, int B) {
  if (threadIdx.x < n) {
    ctx_len[threadIdx.x] = 0;
    base_len[threadIdx.x] = 0;
  }
  if (threadIdx.x == 0) *live = B;
}
}  // namespace

void llm_session_begin(cvk_ctx* ctx, cvk_lm_session* s, int B, cudaStream_t st) {
  CVK_REQUIRE(ctx->llm, "llm stage not finalised");
  CVK_REQUIRE(B >= 1 && B <= s->max_batch && s->max_batch <= 1024, "cvk_lm_begin: bad batch");
  if (s->graph) {
    cudaGraphExecDestroy(s->graph);
    s->graph = nullptr;
  }
  zero_state_kernel<<<1, round_up(s->max_batch, 32), 0, st>>>(s->ctx_len, s->base_len, s->live, s->max_batch, B);
  CVK_CHECK_CUDA(cudaMemsetAsync(s->hidden, 0, sizeof(float) * (size_t)s->max_batch * D, st));
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  s->B = B;
  s->fresh = true;
  s->fed = 0;
  s->ragged = true;
  s->rows_fed.assign(s->max_batch, 0);
}

// ids / kinds: HOST arrays of n entries (kind 0 text id, 1 speech id, 2 llm_embedding row); every row of the session receives the
// same positions (the text-streaming path is one utterance per session)
void llm_feed(cvk_ctx* ctx, cvk_lm_session* s, const int32_t* ids, const int32_t* kinds, int n, cudaStream_t st) {
  const LlmModel* m = ctx->llm;
  CVK_REQUIRE(m && s->B > 0, "cvk_lm_begin or cvk_lm_prefill must run before cvk_lm_feed");
  CVK_REQUIRE(s->fed + n < s->max_ctx, "cvk_lm_feed: session context exhausted");
  const int adt = s->kv_dtype, B = s->B;
  Mat x(s->x, DT_F32, B, D, D), xn(s->xn, adt, B, D, D), qkv(s->qkv, adt, B, QKV_N, QKV_N), att(s->att, adt, B, D, D),
      gu(s->gu, adt, B, 2 * DFF, 2 * DFF), ffa(s->ffa, adt, B, DFF, DFF);
  for (int i = 0; i < n; ++i) {
    const int kind = kinds[i], id = ids[i];
    CVK_REQUIRE((kind == 0 && id >= 0 && id < 151936) || (kind == 1 && id >= 0 && id < m->vout) || (kind == 2 && id >= 0 && id < 2),
                "cvk_lm_feed: id out of range");
    feed_embed_kernel<<<1, 256, 0, st>>>(kind, id, B, m->text_emb, m->llm_emb, m->speech_emb, s->x);
    for (int li = 0; li < m->num_layers; ++li) layer_forward(ctx, st, m, li, x, xn, qkv, att, gu, ffa, nullptr, s, true);
    bump_ctx_kernel<<<1, round_up(B, 32), 0, st>>>(s->ctx_len, B);
    ctx->launches += 2;
    CVK_LAUNCH_CHECK();
  }
  CVK_CHECK_CUDA(cudaMemcpyAsync(s->hidden, s->x, sizeof(float) * (size_t)B * D, cudaMemcpyDeviceToDevice, st));
  s->fed += n;
  for (int b = 0; b < B; ++b) s->rows_fed[b] += n;
  s->fresh = false;      // the step-graph decode (cvk_lm_decode) is not mixed with host-driven feeding
}

// log_softmax(llm_decoder(final_norm(hidden))) of the last fed position -> logp [B][6564] (device)
void llm_next_logp(cvk_ctx* ctx, cvk_lm_session* s, float* logp, cudaStream_t st) {
  const LlmModel* m = ctx->llm;
  CVK_REQUIRE(m && s->B > 0 && s->fed > 0, "cvk_lm_feed must run before cvk_lm_next_logp");
  const int B = s->B;
  Mat hid(s->hidden, DT_F32, B, D, D), xn(s->xn, s->kv_dtype, B, D, D), logits(s->logits, DT_F32, B, m->vout, m->vout);
  head_logits(ctx, st, m, hid, xn, logits, s);
  logsoftmax_rows_kernel<<<B, SAMPLER_THREADS, 0, st>>>(s->logits, m->vout);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  CVK_CHECK_CUDA(cudaMemcpyAsync(logp, s->logits, sizeof(float) * (size_t)B * m->vout, cudaMemcpyDeviceToDevice, st));
}

// ---------------------------------------------------------------------------------------------- ragged feeding
// Several rows of one session, each with its own number of new positions, in one forward per layer over M = sum(counts) activation
// rows (the reference pushes a request's whole lm_input in one forward, llm.py:617-621; here the rows of several requests share it).
// Everything is checked against the host mirror rows_fed before any device work, so a refused call changes nothing.
static constexpr int FEED_CAP = 256;   // positions per forward pass; a larger feed runs as several passes in position order

static void feed_buffers(cvk_lm_session* s) {
  if (s->feed_cap) return;
  const size_t es = s->kv_dtype == DT_F32 ? 4 : 2, cap = FEED_CAP;
  auto alloc = [&](size_t bytes) {
    void* p = nullptr;
    CVK_CHECK_CUDA(cudaMalloc(&p, bytes));
    s->owned.push_back(p);
    return p;
  };
  s->fx = (float*)alloc(sizeof(float) * cap * D);
  s->fxn = alloc(es * cap * D);
  s->fqkv = alloc(es * cap * QKV_N);
  s->fatt = alloc(es * cap * D);
  s->fgu = alloc(es * cap * 2 * DFF);
  s->fffa = alloc(es * cap * DFF);
  s->fidx = (int*)alloc(sizeof(int) * (8 * cap + 3 * (size_t)s->max_batch));
  // the largest split-K partial sums of the feed GEMMs at 64 rows: the down projection (N = 896) at up to 32 splits
  s->fscratch_floats = skinny_scratch_floats(64, D);
  s->fscratch = (float*)alloc(s->fscratch_floats * sizeof(float));
  s->feed_cap = FEED_CAP;
}

static void check_id(const LlmModel* m, int kind, int id, const char* what) {
  CVK_REQUIRE((kind == 0 && id >= 0 && id < 151936) || (kind == 1 && id >= 0 && id < m->vout) || (kind == 2 && id >= 0 && id < 2), what);
}

void llm_feed_rows(cvk_ctx* ctx, cvk_lm_session* s, int n_rows, const int* rows, const int* counts, const int32_t* ids, const int32_t* kinds,
                   cudaStream_t st) {
  const LlmModel* m = ctx->llm;
  CVK_REQUIRE(m && s->B > 0 && s->ragged, "cvk_lm_begin must run before cvk_lm_feed_rows");
  CVK_REQUIRE(n_rows >= 1 && n_rows <= s->B, "cvk_lm_feed_rows: row count out of range");
  std::vector<char> seen(s->B, 0);
  int64_t total = 0;
  for (int r = 0; r < n_rows; ++r) {
    const int b = rows[r];
    CVK_REQUIRE(b >= 0 && b < s->B && !seen[b], "cvk_lm_feed_rows: duplicate or out-of-range row");
    seen[b] = 1;
    CVK_REQUIRE(counts[r] >= 1 && (int64_t)s->rows_fed[b] + counts[r] <= s->max_ctx, "cvk_lm_feed_rows: row context exhausted");
    total += counts[r];
  }
  for (int64_t i = 0; i < total; ++i) check_id(m, kinds[i], ids[i], "cvk_lm_feed_rows: id or kind out of range");
  feed_buffers(s);
  const int adt = s->kv_dtype, cap = s->feed_cap;
  // pass index tables, one upload per pass: ids [cap] | kinds [cap] | rowpos int2 [cap] | tiles int4 [cap] | scatter [max_batch][3]
  std::vector<int> h((size_t)8 * cap + 3 * (size_t)s->max_batch);
  int* h_ids = h.data();
  int* h_kinds = h_ids + cap;
  int* h_rowpos = h_kinds + cap;
  int* h_tiles = h_rowpos + 2 * cap;
  int* h_sc = h_tiles + 4 * cap;
  const int2* d_rowpos = reinterpret_cast<const int2*>(s->fidx + 2 * cap);
  const int4* d_tiles = reinterpret_cast<const int4*>(s->fidx + 4 * cap);
  const int* d_sc = s->fidx + 8 * cap;
  int r = 0, in_row = 0;           // next position to place: row index r of the call, its in_row-th position
  int64_t off = 0;
  while (off < total) {
    const int M = (int)std::min<int64_t>(cap, total - off);
    int mm = 0, ntiles = 0, nsc = 0;
    while (mm < M) {
      const int b = rows[r], take = std::min(counts[r] - in_row, M - mm), pos = s->rows_fed[b];
      for (int k = 0; k < take; ++k) {
        h_ids[mm + k] = ids[off + mm + k];
        h_kinds[mm + k] = kinds[off + mm + k];
        h_rowpos[2 * (mm + k)] = b;
        h_rowpos[2 * (mm + k) + 1] = pos + k;
      }
      for (int k = 0; k < take; k += 2) {
        int* t = h_tiles + 4 * ntiles++;
        t[0] = mm + k; t[1] = b; t[2] = pos + k; t[3] = std::min(2, take - k);
      }
      h_sc[3 * nsc] = b; h_sc[3 * nsc + 1] = mm + take - 1; h_sc[3 * nsc + 2] = take;
      ++nsc;
      s->rows_fed[b] += take;
      mm += take;
      in_row += take;
      if (in_row == counts[r]) { ++r; in_row = 0; }
    }
    CVK_CHECK_CUDA(cudaMemcpyAsync(s->fidx, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    Mat x(s->fx, DT_F32, M, D, D), xn(s->fxn, adt, M, D, D), qkv(s->fqkv, adt, M, QKV_N, QKV_N), att(s->fatt, adt, M, D, D),
        gu(s->fgu, adt, M, 2 * DFF, 2 * DFF), ffa(s->fffa, adt, M, DFF, DFF);
    ragged_embed_kernel<<<M, 128, 0, st>>>(s->fidx, s->fidx + cap, m->text_emb, m->llm_emb, m->speech_emb, s->fx);
    ctx->launches++;
    CVK_LAUNCH_CHECK();
    RaggedPass rg;
    rg.rowpos = d_rowpos;
    rg.tiles = d_tiles;
    rg.ntiles = ntiles;
    for (int li = 0; li < m->num_layers; ++li) layer_forward(ctx, st, m, li, x, xn, qkv, att, gu, ffa, nullptr, s, true, &rg);
    feed_scatter_kernel<<<nsc, 128, 0, st>>>(d_sc, s->fx, s->hidden, s->ctx_len);
    ctx->launches++;
    CVK_LAUNCH_CHECK();
    off += M;
  }
  s->fed = std::max(s->fed, *std::max_element(s->rows_fed.begin(), s->rows_fed.begin() + s->B));
  s->fresh = false;
}

// log_softmax(llm_decoder(final_norm(hidden))) of the listed rows -> logp [n_rows][V] (device)
void llm_next_logp_rows(cvk_ctx* ctx, cvk_lm_session* s, int n_rows, const int* rows, float* logp, cudaStream_t st) {
  const LlmModel* m = ctx->llm;
  CVK_REQUIRE(m && s->B > 0 && s->ragged, "cvk_lm_begin must run before cvk_lm_next_logp_rows");
  CVK_REQUIRE(n_rows >= 1 && n_rows <= s->B, "cvk_lm_next_logp_rows: row count out of range");
  std::vector<char> seen(s->B, 0);
  for (int r = 0; r < n_rows; ++r) {
    const int b = rows[r];
    CVK_REQUIRE(b >= 0 && b < s->B && !seen[b], "cvk_lm_next_logp_rows: duplicate or out-of-range row");
    CVK_REQUIRE(s->rows_fed[b] > 0, "cvk_lm_next_logp_rows: row has no fed position");
    seen[b] = 1;
  }
  CVK_CHECK_CUDA(cudaMemcpyAsync(s->sel, rows, sizeof(int) * n_rows, cudaMemcpyHostToDevice, st));
  gather_rows_kernel<<<n_rows, 128, 0, st>>>(s->sel, s->hidden, s->x);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  Mat hid(s->x, DT_F32, n_rows, D, D), xn(s->xn, s->kv_dtype, n_rows, D, D), logits(s->logits, DT_F32, n_rows, m->vout, m->vout);
  rmsnorm(ctx, st, hid, m->final_norm, RMS_EPS, xn);
  Epilogue e;
  e.out = logits;
  lm_gemm_rows(ctx, st, xn, m->head, e, s->scratch, s->scratch_floats);   // at most min(64, max_batch) rows per slice: within scratch
  logsoftmax_rows_kernel<<<n_rows, SAMPLER_THREADS, 0, st>>>(s->logits, m->vout);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  CVK_CHECK_CUDA(cudaMemcpyAsync(logp, s->logits, sizeof(float) * (size_t)n_rows * m->vout, cudaMemcpyDeviceToDevice, st));
}

int llm_vocab(cvk_ctx* ctx) { return ctx->llm ? ctx->llm->vout : 0; }

void llm_last_logits(cvk_ctx* ctx, cvk_lm_session* s, float* logits, cudaStream_t st) {
  CVK_REQUIRE(s->B > 0 && s->logits, "cvk_lm_last_logits: no decode step has run");
  CVK_REQUIRE(ctx->llm, "llm stage not finalised");
  CVK_CHECK_CUDA(cudaMemcpyAsync(logits, s->logits, sizeof(float) * (size_t)s->B * ctx->llm->vout, cudaMemcpyDeviceToDevice, st));
}

// teacher-forced log-probs for every position (parity tests)
void llm_forward_logp(cvk_ctx* ctx, const float* embeds, const int* lens, int B, float* logp, cudaStream_t st) {
  const LlmModel* m = ctx->llm;
  CVK_REQUIRE(m, "llm stage not finalised");
  ctx->arena.reset();
  Seqs s = make_seqs(ctx, lens, B, 0, 1, 0, st);
  Mat x = arena_mat(ctx, DT_F32, s.R, D, D);
  zero_mat(ctx, st, x);
  pack_rows(ctx, st, embeds, D, s, x);
  forward_packed(ctx, st, s, x, nullptr);
  Mat xn = arena_mat(ctx, ctx->act_dtype, s.R, D), logits = arena_mat(ctx, DT_F32, s.R, m->vout, m->vout);
  head_logits(ctx, st, m, x, xn, logits);
  logsoftmax_rows_kernel<<<s.R, SAMPLER_THREADS, 0, st>>>(logits.f32(), m->vout);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  unpack_rows(ctx, st, logits, s, 0, logp, m->vout);
}

void llm_ras_sample(cvk_ctx* ctx, float* logp, int B, int V, const int32_t* history, int hist_ld, const int32_t* hist_count,
                    const float* uniforms, const int32_t* ignore_eos, int32_t* out_ids, cudaStream_t st) {
  CVK_REQUIRE(V > EOS + 2 && V <= SAMPLER_PER * SAMPLER_THREADS, "vocabulary size out of range (6564 .. 6912 supported)");
  CVK_CHECK_CUDA(cudaFuncSetAttribute(ras_sampler_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)sampler_smem(V > VOUT3_PAD ? V : VOUT3_PAD)));   // per function, never lowered
  ras_sampler_kernel<<<B, SAMPLER_THREADS, sampler_smem(V), st>>>(logp, V, 0, uniforms, B, nullptr, nullptr, nullptr, 0, nullptr, nullptr, nullptr,
                                                                    nullptr, nullptr, nullptr, nullptr, history, hist_ld, hist_count, ignore_eos,
                                                                    out_ids, nullptr, nullptr, nullptr, nullptr);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}

// One decode-graph sampler step on caller data, without a loaded LM (cvk_op_sample_step): the kernel the decode step launches,
// with from_logits = 1 and the caller's state buffers.  With gamma, the fused layer-0 RMSNorm goes to a bf16 copy of xn that is
// widened back into the caller's fp32 xn (rows the kernel does not write come back rounded to bf16).
void llm_sample_step_op(cvk_ctx* ctx, float* logits, int B, int V, const float* uniforms, const int32_t* min_len, const int32_t* max_len,
                        int32_t* out_ids, int out_ld, int32_t* out_count, int32_t* done, int* ctx_len, const int* base_len, int* live,
                        const float* speech_emb, float* next_x, const float* gamma, float* xn, cudaStream_t st) {
  CVK_CHECK_CUDA(cudaFuncSetAttribute(ras_sampler_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)sampler_smem(V > VOUT3_PAD ? V : VOUT3_PAD)));   // per function, never lowered
  ctx->arena.reset();
  Mat xn16;
  if (gamma) {
    xn16 = arena_mat(ctx, DT_BF16, B, D, D);
    convert_mat(ctx, st, Mat(xn, DT_F32, B, D, D), xn16);
  }
  ras_sampler_kernel<<<B, SAMPLER_THREADS, sampler_smem(V), st>>>(logits, V, 1, uniforms, B, min_len, max_len, out_ids, out_ld, out_count,
                                                                    done, ctx_len, base_len, live, speech_emb, next_x, nullptr, 0, nullptr,
                                                                    nullptr, nullptr, gamma, gamma ? xn16.b16() : nullptr, nullptr, nullptr);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  if (gamma) convert_mat(ctx, st, xn16, Mat(xn, DT_F32, B, D, D));
}

// log_softmax of rows [rows][V] in place with the kernel of cvk_lm_next_logp / cvk_lm_forward_logp (cvk_op_log_softmax)
void llm_log_softmax_op(cvk_ctx* ctx, float* x, int rows, int V, cudaStream_t st) {
  logsoftmax_rows_kernel<<<rows, SAMPLER_THREADS, 0, st>>>(x, V);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}
