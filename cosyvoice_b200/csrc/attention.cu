// Multi-head attention over ragged time-major sequences, head_dim 64.
//
//  * estimator self-attention (matcha transformer.py:243-316 via diffusers Attention, flow/decoder.py:439-449):
//    full attention inside each sequence, or block-causal with chunk 50 when streaming
//    (utils/mask.py:127-158: key j visible from query i iff j < (i/chunk+1)*chunk) - the mask is a predicate
//    evaluated in the kernel, never a materialised [T,T] bias tensor.
//  * conformer relative-position attention (transformer/attention.py:249-330):
//    score = ((q+u).k + (q+v).p[i-j]) / sqrt(d), where p[r] = linear_pos(pe(r)) and the reference's rel_shift
//    (attention.py:225-247) is exactly the index map (i,j) -> r = i-j.
//
// This file holds the fp32-math flash-style kernel (online softmax, one CTA per 32 queries x head x sequence);
// it serves the parity mode and any operand dtype.  The tensor-core kernel for bf16 operands is in attention_tc.cu.
#include "common.cuh"

namespace {

constexpr int BQ = 32, BKEY = 32, HD = 64;

template <typename T, bool RELPOS>
__global__ void __launch_bounds__(128) attn_simt_kernel(const T* __restrict__ q, int ldq, const T* __restrict__ k, int ldk,
                                                        const T* __restrict__ v, int ldv, const T* __restrict__ pos, int ldp, int pos_rows, int pos_center,
                                                        const float* __restrict__ bias_u, const float* __restrict__ bias_v,
                                                        const int* __restrict__ start, const int* __restrict__ len, int chunk, float scale, int kv_div,
                                                        T* __restrict__ out, int ldo, const int* __restrict__ kstart, const int* __restrict__ klen,
                                                        const int* __restrict__ qoff) {
  __shared__ float Qs[BQ][HD + 1];
  __shared__ float Ks[BKEY][HD + 1];
  __shared__ float Vs[BKEY][HD + 1];
  __shared__ float Ps[BQ][BKEY + 1];
  __shared__ float Rs[RELPOS ? (BQ + BKEY - 1) : 1][HD + 1];
  __shared__ float dvu[HD];   // bias_v - bias_u: (q+v) = (q+u) + dvu

  const int b = blockIdx.z, h = blockIdx.y;
  const int L = len[b], s0 = start[b];               // query rows
  const int Lk = klen ? klen[b] : L, ks0 = kstart ? kstart[b] : s0, q0 = qoff ? qoff[b] : 0;   // key rows; absolute position of query 0
  const int i0 = blockIdx.x * BQ;
  if (i0 >= L) return;
  const int t = threadIdx.x, ty = t >> 4, tx = t & 15;

  for (int e = t; e < BQ * HD; e += 128) {
    int i = e >> 6, d = e & 63;
    float x = 0.f;
    if (i0 + i < L) x = to_f32(q[(size_t)(s0 + i0 + i) * ldq + h * HD + d]);
    if (RELPOS) x += bias_u[h * HD + d];
    Qs[i][d] = x;
  }
  if (RELPOS && t < HD) dvu[t] = bias_v[h * HD + t] - bias_u[h * HD + t];
  // highest visible key over the queries of this tile
  int i_last = q0 + min(i0 + BQ, L) - 1;
  int kmax = chunk > 0 ? min(Lk, (i_last / chunk + 1) * chunk) : Lk;

  float m_run[4], l_run[4], o[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    m_run[a] = -INFINITY;
    l_run[a] = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) o[a][c] = 0.f;
  }
  int klim[4];
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    int i = i0 + ty * 4 + a;
    klim[a] = chunk > 0 ? min(Lk, ((q0 + i) / chunk + 1) * chunk) : Lk;
    if (i >= L) klim[a] = 0;
  }

  for (int j0 = 0; j0 < kmax; j0 += BKEY) {
    __syncthreads();
    for (int e = t; e < BKEY * HD; e += 128) {
      int j = e >> 6, d = e & 63;
      float kv = 0.f, vv = 0.f;
      if (j0 + j < Lk) {
        kv = to_f32(k[(size_t)(ks0 + j0 + j) * ldk + (h / kv_div) * HD + d]);
        vv = to_f32(v[(size_t)(ks0 + j0 + j) * ldv + (h / kv_div) * HD + d]);
      }
      Ks[j][d] = kv;
      Vs[j][d] = vv;
    }
    if (RELPOS) {
      // relative positions r = i - j for i in [i0, i0+BQ), j in [j0, j0+BKEY): r in [i0-j0-(BKEY-1), i0-j0+BQ-1]
      int rbase = i0 - j0 - (BKEY - 1);
      for (int e = t; e < (BQ + BKEY - 1) * HD; e += 128) {
        int rr = e >> 6, d = e & 63;
        int row = pos_center - (rbase + rr);   // table row of relative position rbase+rr
        row = max(0, min(pos_rows - 1, row));  // only reachable for masked (i,j) pairs beyond the sequence end
        Rs[rr][d] = to_f32(pos[(size_t)row * ldp + h * HD + d]);
      }
    }
    __syncthreads();
    // scores: rows 4ty..4ty+3, keys 2tx, 2tx+1
    float s[4][2];
#pragma unroll
    for (int a = 0; a < 4; ++a) s[a][0] = s[a][1] = 0.f;
#pragma unroll 8
    for (int d = 0; d < HD; ++d) {
      float k0 = Ks[2 * tx][d], k1 = Ks[2 * tx + 1][d];
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        float qa = Qs[ty * 4 + a][d];
        s[a][0] = fmaf(qa, k0, s[a][0]);
        s[a][1] = fmaf(qa, k1, s[a][1]);
      }
    }
    if (RELPOS) {
#pragma unroll 8
      for (int d = 0; d < HD; ++d) {
        const float dv = dvu[d];
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          float qa = Qs[ty * 4 + a][d] + dv;
          int il = ty * 4 + a;
          // rr = (i - j) - rbase = il - jl + BKEY - 1
          s[a][0] = fmaf(qa, Rs[il - 2 * tx + BKEY - 1][d], s[a][0]);
          s[a][1] = fmaf(qa, Rs[il - 2 * tx - 1 + BKEY - 1][d], s[a][1]);
        }
      }
    }
    // online softmax per row (the 16 lanes tx=0..15 of a half-warp share a row group)
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      float v0 = (j0 + 2 * tx < klim[a]) ? s[a][0] * scale : -INFINITY;
      float v1 = (j0 + 2 * tx + 1 < klim[a]) ? s[a][1] * scale : -INFINITY;
      float mx = fmaxf(v0, v1);
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
      float m_new = fmaxf(m_run[a], mx);
      float corr = (m_new == -INFINITY) ? 1.f : expf(m_run[a] - m_new);
      float p0 = (v0 == -INFINITY) ? 0.f : expf(v0 - m_new);
      float p1 = (v1 == -INFINITY) ? 0.f : expf(v1 - m_new);
      float ps = p0 + p1;
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) ps += __shfl_xor_sync(0xffffffffu, ps, off);
      l_run[a] = l_run[a] * corr + ps;
      m_run[a] = m_new;
#pragma unroll
      for (int c = 0; c < 4; ++c) o[a][c] *= corr;
      Ps[ty * 4 + a][2 * tx] = p0;
      Ps[ty * 4 + a][2 * tx + 1] = p1;
    }
    __syncwarp();   // a row group's P values are produced and consumed by the same half-warp
#pragma unroll 8
    for (int j = 0; j < BKEY; ++j) {
      float vv[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) vv[c] = Vs[j][tx * 4 + c];
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        float p = Ps[ty * 4 + a][j];
#pragma unroll
        for (int c = 0; c < 4; ++c) o[a][c] = fmaf(p, vv[c], o[a][c]);
      }
    }
  }
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    int i = i0 + ty * 4 + a;
    if (i >= L) continue;
    float inv = 1.f / l_run[a];
#pragma unroll
    for (int c = 0; c < 4; ++c) out[(size_t)(s0 + i) * ldo + h * HD + tx * 4 + c] = from_f32<T>(o[a][c] * inv);
  }
}

}  // namespace

void attention_fwd_tc(cvk_ctx* ctx, cudaStream_t st, const Mat& q, const Mat& k, const Mat& v, const Seqs& s, int H, int chunk,
                      float scale, const Mat& out, int kv_div, const KvGeom* kg);

void attention_fwd(cvk_ctx* ctx, cudaStream_t st, const Mat& q, const Mat& k, const Mat& v, const Seqs& s, int H, int chunk,
                   float scale, const Mat& out, int kv_div, const KvGeom* kg) {
  const int* ks = kg ? kg->d_kstart : nullptr;
  const int* kl = kg ? kg->d_klen : nullptr;
  const int* qo = kg ? kg->d_qoff : nullptr;
  CVK_REQUIRE(!kg || (ks && kl && qo), "attention: incomplete key/value geometry");
  CVK_REQUIRE(q.dtype == k.dtype && q.dtype == v.dtype && q.dtype == out.dtype, "attention: mixed dtypes");
  dim3 grid(ceil_div(s.max_len, BQ), H, s.B);
  double fl = 0;
  for (int b = 0; b < s.B; ++b) fl += 4.0 * (double)s.len[b] * s.len[b] * 64 * H * (chunk > 0 ? 0.5 : 1.0);
  ProfScope ps(ctx, st, FAM_ATTN, fl, (double)s.sum_len * H * 64 * 4 * q.esize());
  if (q.dtype == DT_BF16 && ctx->use_tc_attn) {
    attention_fwd_tc(ctx, st, q, k, v, s, H, chunk, scale, out, kv_div, kg);
    return;
  }
  if (q.dtype == DT_F32)
    attn_simt_kernel<float, false><<<grid, 128, 0, st>>>(q.f32(), q.ld, k.f32(), k.ld, v.f32(), v.ld, nullptr, 0, 0, 0, nullptr, nullptr,
                                                         s.d_start, s.d_len, chunk, scale, kv_div, out.f32(), out.ld, ks, kl, qo);
  else
    attn_simt_kernel<bf16, false><<<grid, 128, 0, st>>>(q.b16(), q.ld, k.b16(), k.ld, v.b16(), v.ld, nullptr, 0, 0, 0, nullptr, nullptr,
                                                        s.d_start, s.d_len, chunk, scale, kv_div, out.b16(), out.ld, ks, kl, qo);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}

void relpos_attention_fwd_tc(cvk_ctx* ctx, cudaStream_t st, const Mat& qu, const Mat& qv, const Mat& k, const Mat& v, const Mat& pos, int pos_rows,
                             int pos_center, const Seqs& s, int H, int chunk, float scale, const Mat& U, const Mat& out);

namespace {
// qu = q + pos_bias_u, qv = q + pos_bias_v (transformer/attention.py:303-306), bf16
__global__ void add_pos_bias_kernel(const bf16* __restrict__ q, int ldq, const float* __restrict__ bu, const float* __restrict__ bv, int rows, int C,
                                    bf16* __restrict__ qu, bf16* __restrict__ qv, int ldo) {
  size_t total = (size_t)rows * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int r = i / C, c = i % C;
    const float x = __bfloat162float(q[(size_t)r * ldq + c]);
    qu[(size_t)r * ldo + c] = __float2bfloat16_rn(x + bu[c]);
    qv[(size_t)r * ldo + c] = __float2bfloat16_rn(x + bv[c]);
  }
}
}  // namespace

void relpos_attention_fwd(cvk_ctx* ctx, cudaStream_t st, const Mat& q, const Mat& k, const Mat& v, const Mat& pos, int pos_center,
                          const float* bias_u, const float* bias_v, const Seqs& s, int H, int chunk, float scale, const Mat& out) {
  CVK_REQUIRE(q.dtype == k.dtype && q.dtype == v.dtype && q.dtype == out.dtype && q.dtype == pos.dtype, "attention: mixed dtypes");
  CVK_REQUIRE(pos.rows >= 2 * s.max_len - 1 + 0 && pos_center >= s.max_len - 1 + 0, "relative position table too small");
  const int pos_rows = 2 * pos_center + 1;
  if (q.dtype == DT_BF16 && ctx->use_tc_attn && ctx->enc_tc_attn && pos.rows >= round_up(pos_rows, 64)) {
    // tensor-core path: the position term of every (query, table row) pair first (relpos_u_kernel), then the one-pass attention
    // kernel with that term as an additive bias (attention_tc.cu)
    double fl = 0;
    for (int b = 0; b < s.B; ++b) fl += 6.0 * (double)s.len[b] * s.len[b] * 64 * H * (chunk > 0 ? 0.5 : 1.0);
    ProfScope ps(ctx, st, FAM_ATTN, fl, (double)s.sum_len * H * 64 * 4 * q.esize());
    const size_t mark = ctx->arena.off;
    const int C = H * HD;
    Mat qu = arena_mat(ctx, DT_BF16, s.R, C), qv = arena_mat(ctx, DT_BF16, s.R, C);
    add_pos_bias_kernel<<<132 * 8, 256, 0, st>>>(q.b16(), q.ld, bias_u, bias_v, s.R, C, qu.b16(), qv.b16(), qu.ld);
    ctx->launches++;
    CVK_LAUNCH_CHECK();
    const int ldu = round_up(pos_rows, 64);
    Mat U = arena_mat(ctx, DT_F32, s.R * H, ldu, ldu);
    relpos_attention_fwd_tc(ctx, st, qu, qv, k, v, pos, pos_rows, pos_center, s, H, chunk, scale, U, out);
    ctx->arena.off = mark;
    return;
  }
  dim3 grid(ceil_div(s.max_len, BQ), H, s.B);
  if (q.dtype == DT_F32)
    attn_simt_kernel<float, true><<<grid, 128, 0, st>>>(q.f32(), q.ld, k.f32(), k.ld, v.f32(), v.ld, pos.f32(), pos.ld, pos.rows, pos_center, bias_u,
                                                        bias_v, s.d_start, s.d_len, chunk, scale, 1, out.f32(), out.ld, nullptr, nullptr, nullptr);
  else
    attn_simt_kernel<bf16, true><<<grid, 128, 0, st>>>(q.b16(), q.ld, k.b16(), k.ld, v.b16(), v.ld, pos.b16(), pos.ld, pos.rows, pos_center, bias_u,
                                                       bias_v, s.d_start, s.d_len, chunk, scale, 1, out.b16(), out.ld, nullptr, nullptr, nullptr);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}
