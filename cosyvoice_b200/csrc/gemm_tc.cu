// bf16 / fp16 conv-GEMM on Hopper tensor cores (wgmma.mma_async, fp32 accumulators in registers, operands staged by TMA).
//
//   out[r, n] = epilogue( sum_{j<taps} sum_{k<K} A[r + shift0 + j*dil, k] * W[n][j][k] ),  fp32 accumulate
//
// A convolution tap is just a row-shifted TMA box of the time-major activation matrix; rows outside the matrix and the K tail
// are zero-filled by the TMA unit, gap rows between ragged sequences hold zeros in memory.
//
// Reference ops served: every dense Linear / Conv1d of the flow estimator + encoder (flow/decoder.py,
// matcha transformer.py), the LM projections (transformers Qwen2, llm/llm.py:244-251) and the HiFT ResBlock /
// upsampling convolutions (hifigan/generator.py:110-117, 432-443).
#include "common.cuh"
#include "wgmma.cuh"
#include "tma.cuh"

namespace {

constexpr int TC_BM = 128;
constexpr int TC_BK = 64;   // 64 bf16 = 128 B = one SWIZZLE_128B atom row
constexpr int TC_THREADS = 384;   // warpgroup 0: TMA producer (one thread), warpgroups 1-2: wgmma + epilogue, 64 rows each

// 16 consecutive columns of one row through the fused epilogue (vector fast path + scalar tail).
__device__ __forceinline__ void epi_store16(const EpiDev& e, int r, int n0, int N, const float* acc) {
  if (n0 + 16 > N) {
    for (int i = 0; i < 16 && n0 + i < N; ++i) epi_store<true>(e, r, n0 + i, acc[i]);
    return;
  }
  int seq = 0;
  bool valid = true;
  if (e.row2seq) {
    seq = e.row2seq[r];
    valid = seq >= 0;
  }
  float v[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) v[i] = acc[i];
  if (e.bias) {
#pragma unroll
    for (int i = 0; i < 16; i += 4) {
      float4 b = *reinterpret_cast<const float4*>(e.bias + n0 + i);
      v[i] += b.x; v[i + 1] += b.y; v[i + 2] += b.z; v[i + 3] += b.w;
    }
  }
  if (e.rowvec && valid) {
    const float* rv = e.rowvec + (size_t)seq * e.rowvec_ld + n0;
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] += rv[i];
  }
  act16_fast(e.act1, v, e.act1_param, e.alpha1 ? e.alpha1 + n0 : nullptr);
  if (e.scale != 1.f) {
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] *= e.scale;
  }
  if (e.resid) {
    const float* rp = e.resid + (size_t)r * e.resid_ld + n0;
#pragma unroll
    for (int i = 0; i < 16; i += 4) {
      float4 b = *reinterpret_cast<const float4*>(rp + i);
      v[i] += b.x; v[i + 1] += b.y; v[i + 2] += b.z; v[i + 3] += b.w;
    }
  }
  if (!valid) {
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = 0.f;
  }
  size_t o = (size_t)r * e.out_ld + n0;
  if (e.out_dtype == DT_F32) {
    float* op = (float*)e.out + o;
    if (e.accumulate) {
#pragma unroll
      for (int i = 0; i < 16; i += 4) {
        float4 b = *reinterpret_cast<const float4*>(op + i);
        v[i] += b.x; v[i + 1] += b.y; v[i + 2] += b.z; v[i + 3] += b.w;
      }
    }
#pragma unroll
    for (int i = 0; i < 16; i += 4) *reinterpret_cast<float4*>(op + i) = make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]);
  } else {
    unsigned short* op = (unsigned short*)e.out + o;
    if (e.accumulate) {
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] += f16bits_to_f32(op[i], e.out_dtype);
    }
    __align__(16) unsigned short t[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) t[i] = f32_to_16(v[i], e.out_dtype);
    *reinterpret_cast<uint4*>(op) = *reinterpret_cast<uint4*>(t);
    *reinterpret_cast<uint4*>(op + 8) = *reinterpret_cast<uint4*>(t + 8);
  }
  if (e.out2) {
    float w[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) w[i] = v[i];
    act16_fast(e.act2, w, e.act2_param, e.alpha2 ? e.alpha2 + n0 : nullptr);
    if (!valid) {
#pragma unroll
      for (int i = 0; i < 16; ++i) w[i] = 0.f;
    }
    size_t o2 = (size_t)r * e.out2_ld + n0;
    if (e.out2_dtype == DT_F32) {
      float* op = (float*)e.out2 + o2;
#pragma unroll
      for (int i = 0; i < 16; i += 4) *reinterpret_cast<float4*>(op + i) = make_float4(w[i], w[i + 1], w[i + 2], w[i + 3]);
    } else {
      unsigned short* op = (unsigned short*)e.out2 + o2;
      __align__(16) unsigned short t[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) t[i] = f32_to_16(w[i], e.out2_dtype);
      *reinterpret_cast<uint4*>(op) = *reinterpret_cast<uint4*>(t);
      *reinterpret_cast<uint4*>(op + 8) = *reinterpret_cast<uint4*>(t + 8);
    }
  }
}

// values of 16 consecutive columns of one row (fused epilogue math, no stores); columns >= N yield 0
__device__ __forceinline__ void epi_math16(const EpiDev& e, int r, bool rin, int n0, int N, const float* acc, float* v, float* w2) {
  int seq = 0;
  bool valid = rin;
  if (rin && e.row2seq) {
    seq = e.row2seq[r];
    valid = seq >= 0;
  }
  const bool full = n0 + 16 <= N;
#pragma unroll
  for (int i = 0; i < 16; ++i) v[i] = acc[i];
  if (full) {
    if (e.bias) {
#pragma unroll
      for (int i = 0; i < 16; i += 4) {
        float4 b = *reinterpret_cast<const float4*>(e.bias + n0 + i);
        v[i] += b.x; v[i + 1] += b.y; v[i + 2] += b.z; v[i + 3] += b.w;
      }
    }
    if (e.rowvec && valid) {
      const float* rv = e.rowvec + (size_t)seq * e.rowvec_ld + n0;
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] += rv[i];
    }
    act16_fast(e.act1, v, e.act1_param, e.alpha1 ? e.alpha1 + n0 : nullptr);
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] *= e.scale;
    if (e.resid && rin) {
      const float* rp = e.resid + (size_t)r * e.resid_ld + n0;
#pragma unroll
      for (int i = 0; i < 16; i += 4) {
        float4 b = *reinterpret_cast<const float4*>(rp + i);
        v[i] += b.x; v[i + 1] += b.y; v[i + 2] += b.z; v[i + 3] += b.w;
      }
    }
  } else {
    for (int i = 0; i < 16; ++i) {
      const int n = n0 + i;
      float t = 0.f;
      if (n < N) {
        t = v[i] + (e.bias ? e.bias[n] : 0.f);
        if (e.rowvec && valid) t += e.rowvec[(size_t)seq * e.rowvec_ld + n];
        t = apply_act_fast(e.act1, t, e.act1_param, e.alpha1 ? e.alpha1[n] : 1.f) * e.scale;
        if (e.resid && rin) t += e.resid[(size_t)r * e.resid_ld + n];
      }
      v[i] = t;
    }
  }
  if (!valid) {
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = 0.f;
  }
  if (e.out2) {
    if (full) {
#pragma unroll
      for (int i = 0; i < 16; ++i) w2[i] = v[i];
      act16_fast(e.act2, w2, e.act2_param, e.alpha2 ? e.alpha2 + n0 : nullptr);
      if (!valid) {
#pragma unroll
        for (int i = 0; i < 16; ++i) w2[i] = 0.f;
      }
    } else {
      for (int i = 0; i < 16; ++i)
        w2[i] = (valid && n0 + i < N) ? apply_act_fast(e.act2, v[i], e.act2_param, e.alpha2 ? e.alpha2[n0 + i] : 1.f) : 0.f;
    }
  }
}

// epi_math16 for a full group of 16 columns: the row's sequence index has been resolved by the caller (loaded before the main
// loop) and the bias of the tile's columns sits in shared memory, so no dependent global load sits between the accumulator and
// the stores.
__device__ __forceinline__ void epi_math16p(const EpiDev& e, int r, bool rin, int seq, bool valid, const float* s_bias, int cl, int n0,
                                            const float* acc, float* v, float* w2) {
#pragma unroll
  for (int i = 0; i < 16; ++i) v[i] = acc[i];
  if (e.bias) {
#pragma unroll
    for (int i = 0; i < 16; i += 4) {
      const float4 b = *reinterpret_cast<const float4*>(s_bias + cl + i);
      v[i] += b.x; v[i + 1] += b.y; v[i + 2] += b.z; v[i + 3] += b.w;
    }
  }
  if (e.rowvec && valid) {
    const float* rv = e.rowvec + (size_t)seq * e.rowvec_ld + n0;
#pragma unroll
    for (int i = 0; i < 16; i += 4) {
      const float4 b = *reinterpret_cast<const float4*>(rv + i);
      v[i] += b.x; v[i + 1] += b.y; v[i + 2] += b.z; v[i + 3] += b.w;
    }
  }
  act16_fast(e.act1, v, e.act1_param, e.alpha1 ? e.alpha1 + n0 : nullptr);
#pragma unroll
  for (int i = 0; i < 16; ++i) v[i] *= e.scale;
  if (e.resid && rin) {
    const float* rp = e.resid + (size_t)r * e.resid_ld + n0;
#pragma unroll
    for (int i = 0; i < 16; i += 4) {
      const float4 b = *reinterpret_cast<const float4*>(rp + i);
      v[i] += b.x; v[i + 1] += b.y; v[i + 2] += b.z; v[i + 3] += b.w;
    }
  }
  if (!valid) {
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = 0.f;
  }
  if (e.out2) {
#pragma unroll
    for (int i = 0; i < 16; ++i) w2[i] = v[i];
    act16_fast(e.act2, w2, e.act2_param, e.alpha2 ? e.alpha2 + n0 : nullptr);
    if (!valid) {
#pragma unroll
      for (int i = 0; i < 16; ++i) w2[i] = 0.f;
    }
  }
}

// 16 consecutive columns of one tile row into a SWIZZLE_128B staging tile (128-byte wide sub-tiles of 128 rows, 16 KB each)
__device__ __forceinline__ void stage_store16(uint32_t stg, int dtype, int row, int c, const float* v) {
  if (dtype != DT_F32) {
    const uint32_t sub = stg + (uint32_t)(c >> 6) * 16384u + (uint32_t)row * 128u;
    const uint32_t ch = (uint32_t)((c & 63) >> 3);
    uint32_t pk[8];
    if (dtype == DT_BF16) {
#pragma unroll
      for (int i = 0; i < 16; i += 2) {
        __nv_bfloat162 h2 = __floats2bfloat162_rn(v[i], v[i + 1]);
        pk[i >> 1] = *reinterpret_cast<uint32_t*>(&h2);
      }
    } else {
#pragma unroll
      for (int i = 0; i < 16; i += 2) pk[i >> 1] = (uint32_t)f32_to_16(v[i], DT_F16) | ((uint32_t)f32_to_16(v[i + 1], DT_F16) << 16);
    }
    asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(sub + ((ch ^ (uint32_t)(row & 7)) << 4)), "r"(pk[0]), "r"(pk[1]), "r"(pk[2]), "r"(pk[3]) : "memory");
    asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(sub + (((ch + 1) ^ (uint32_t)(row & 7)) << 4)), "r"(pk[4]), "r"(pk[5]), "r"(pk[6]), "r"(pk[7]) : "memory");
  } else {
    const uint32_t sub = stg + (uint32_t)(c >> 5) * 16384u + (uint32_t)row * 128u;
    const uint32_t ch = (uint32_t)((c & 31) >> 2);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(sub + (((ch + j) ^ (uint32_t)(row & 7)) << 4)), "r"(__float_as_uint(v[4 * j])),
                   "r"(__float_as_uint(v[4 * j + 1])), "r"(__float_as_uint(v[4 * j + 2])), "r"(__float_as_uint(v[4 * j + 3]))
                   : "memory");
    }
  }
}

// ------------------------------------------------------------------------------------------------ fragment-native epilogue
// The functions above take 16 consecutive columns of one row, so the kernels first move each thread's accumulator values there with
// wg_frag_rows16 (12 shuffles and ~32 selects per 16 values).  Every epilogue operation is elementwise in (row, column), so the
// functions below (option "tc_epi_frag", default 1) apply them where the wgmma left the values: thread (warp w, lane l) of a
// warpgroup holds rows 16 w + l / 4 and + 8 of its 64, columns 8 j + 2 (l & 3) and + 1 - a 32-column block [cb, cb + 32) of the
// accumulator is a[4 j + 2 h + e] = (row + 8 h, column cb + 8 j + 2 (l & 3) + e), a = acc + cb / 2.  Each of the two rows has its own
// sequence and validity; bias, rowvec and resid are read as column pairs; the 16-bit results go to the staging tile with stmatrix.
// The operations, their order and the activation forms are those of epi_math16p / epi_math16 (the 16-wide fast forms for columns in a
// whole group of 16 columns, the scalar forms in the partial group at the end of N), so both epilogues give the same bits.
// Only the staged epilogue with 16-bit outputs takes this path: with an fp32 output (8-byte shared stores) and with direct stores
// (column-pair global stores) it was slower than the transposing epilogue on an H100 (the 40064 x 512 -> 256 projection with an fp32
// residual 82.5 against 76.3 us per launch, its accumulating direct-store form 112.4 against 72.5 us; H100 80GB HBM3, 700 W).
struct FragRows {
  int r[2], seq[2];
  bool rin[2], valid[2];
};

__device__ __forceinline__ FragRows frag_rows(const EpiDev& e, int r, int rowsOut) {
  FragRows f;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    f.r[h] = r + 8 * h;
    f.rin[h] = f.r[h] < rowsOut;
    f.seq[h] = (f.rin[h] && e.row2seq) ? e.row2seq[f.r[h]] : 0;
    f.valid[h] = f.rin[h] && (!e.row2seq || f.seq[h] >= 0);
  }
  return f;
}

// columns n and n + 1 of a row; WHOLE: both < N, otherwise those >= N read nothing and give 0
template <bool WHOLE> __device__ __forceinline__ float2 ld_pair(const float* p, int n, int N) {
  if (WHOLE) return *reinterpret_cast<const float2*>(p);
  return make_float2(n < N ? p[0] : 0.f, n + 1 < N ? p[1] : 0.f);
}

// act16_fast over the block's 16 values; Snake reads its per-column alpha[n + 8 j + e] (1 where alpha is null or beyond N)
template <bool WHOLE>
__device__ __forceinline__ void frag_act(int act, float param, const float* alpha, int n, int N, float* v) {
  if (act != ACT_SNAKE) {
    act16_fast(act, v, param, nullptr);
    return;
  }
  float al[16];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int c = n + 8 * j + e;
      al[4 * j + e] = al[4 * j + 2 + e] = (alpha && (WHOLE || c < N)) ? alpha[c] : 1.f;
    }
  act16_fast(ACT_SNAKE, v, param, al);
}

// v = act1(a + bias + rowvec) * scale + resid, zero in invalid rows, for the 32-column block [cb, cb + 32) of the tile at matrix column n0
// (s_bias: the tile's bias), q = lane & 3.  WHOLE: all 32 columns < N.  PLAIN: the epilogue has no activation, rowvec, residual or
// second output and scale 1 (frag_plain), so v = a + bias and nothing else is compiled in.
template <bool WHOLE, bool PLAIN = false>
__device__ __forceinline__ void frag_math(const EpiDev& e, const FragRows& f, const float* s_bias, int n0, int cb, int q, int N, const float* a,
                                          float* v) {
  const int cl = cb + 2 * q, n = n0 + cl;
#pragma unroll
  for (int i = 0; i < 16; ++i) v[i] = a[i];
  if (e.bias) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 b = *reinterpret_cast<const float2*>(s_bias + cl + 8 * j);
      v[4 * j] += b.x; v[4 * j + 1] += b.y; v[4 * j + 2] += b.x; v[4 * j + 3] += b.y;
    }
  }
  if (!PLAIN && e.rowvec) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!f.valid[h]) continue;
      const float* rv = e.rowvec + (size_t)f.seq[h] * e.rowvec_ld + n;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 b = ld_pair<WHOLE>(rv + 8 * j, n + 8 * j, N);
        v[4 * j + 2 * h] += b.x; v[4 * j + 2 * h + 1] += b.y;
      }
    }
  }
  if (!PLAIN) {
    frag_act<WHOLE>(e.act1, e.act1_param, e.alpha1, n, N, v);
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] *= e.scale;
  }
  if (!PLAIN && e.resid) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!f.rin[h]) continue;
      const float* rp = e.resid + (size_t)f.r[h] * e.resid_ld + n;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 b = ld_pair<WHOLE>(rp + 8 * j, n + 8 * j, N);
        v[4 * j + 2 * h] += b.x; v[4 * j + 2 * h + 1] += b.y;
      }
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h)
    if (!f.valid[h]) {
#pragma unroll
      for (int j = 0; j < 4; ++j) v[4 * j + 2 * h] = v[4 * j + 2 * h + 1] = 0.f;
    }
}

// v <- act2(v), zero in invalid rows
template <bool WHOLE>
__device__ __forceinline__ void frag_act2(const EpiDev& e, const FragRows& f, int n0, int cb, int q, int N, float* v) {
  frag_act<WHOLE>(e.act2, e.act2_param, e.alpha2, n0 + cb + 2 * q, N, v);
#pragma unroll
  for (int h = 0; h < 2; ++h)
    if (!f.valid[h]) {
#pragma unroll
      for (int j = 0; j < 4; ++j) v[4 * j + 2 * h] = v[4 * j + 2 * h + 1] = 0.f;
    }
}

// staged epilogue (epi_mode 2), out values of one 32-column block.  In the block at the end of N the columns of a partial 16-column
// group take epi_math16's scalar forms; columns >= N hold junk that the clipped TMA store never writes.
template <bool PLAIN>
__device__ __forceinline__ void frag_values(const EpiDev& e, const FragRows& f, const float* s_bias, int n0, int cb, int q, int N, const float* a,
                                            float* v) {
  if (n0 + cb + 32 <= N) {
    frag_math<true, PLAIN>(e, f, s_bias, n0, cb, q, N, a, v);
    return;
  }
  frag_math<false, PLAIN>(e, f, s_bias, n0, cb, q, N, a, v);
  const int n = n0 + cb + 2 * q;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (n0 + cb + 16 * (j >> 1) + 16 <= N) continue;   // a whole group of 16
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int x = 0; x < 2; ++x) {
        const int c = n + 8 * j + x;
        if (c >= N) continue;
        float t = a[4 * j + 2 * h + x] + (e.bias ? e.bias[c] : 0.f);
        if (e.rowvec && f.valid[h]) t += e.rowvec[(size_t)f.seq[h] * e.rowvec_ld + c];
        t = apply_act_fast(e.act1, t, e.act1_param, e.alpha1 ? e.alpha1[c] : 1.f) * e.scale;
        if (e.resid && f.rin[h]) t += e.resid[(size_t)f.r[h] * e.resid_ld + c];
        v[4 * j + 2 * h + x] = f.valid[h] ? t : 0.f;
      }
  }
}

// ... and its out2 values, in place over the out values
__device__ __forceinline__ void frag_values2(const EpiDev& e, const FragRows& f, int n0, int cb, int q, int N, float* v) {
  if (n0 + cb + 32 <= N) {
    frag_act2<true>(e, f, n0, cb, q, N, v);
    return;
  }
  float w[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) w[i] = v[i];
  frag_act2<false>(e, f, n0, cb, q, N, w);
  const int n = n0 + cb + 2 * q;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (n0 + cb + 16 * (j >> 1) + 16 <= N) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int x = 0; x < 2; ++x) {
        const int c = n + 8 * j + x, i = 4 * j + 2 * h + x;
        if (c < N) w[i] = f.valid[h] ? apply_act_fast(e.act2, v[i], e.act2_param, e.alpha2 ? e.alpha2[c] : 1.f) : 0.f;
      }
  }
#pragma unroll
  for (int i = 0; i < 16; ++i) v[i] = w[i];
}

// an epilogue that only adds the bias (no activation, rowvec, residual or second output, scale 1) - the estimator's qkv projection
// and most of the flow's convolutions: the kernels compile it without the other operations (EPI 2)
inline bool frag_plain(const EpiDev& e) {
  return e.act1 == ACT_NONE && !e.rowvec && !e.resid && e.scale == 1.f && !e.out2;
}

// one 32-column block of the fragment into a 16-bit staging tile (stage_store16's layout), one stmatrix per 16 x 16; row0 = the tile
// row of the warp's first row
__device__ __forceinline__ void frag_stage16(uint32_t stg, int dtype, int row0, int lane, int cb, const float* v) {
  uint32_t pk[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (dtype == DT_BF16) {
      __nv_bfloat162 h2 = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
      pk[i] = *reinterpret_cast<uint32_t*>(&h2);
    } else {
      pk[i] = (uint32_t)f32_to_16(v[2 * i], DT_F16) | ((uint32_t)f32_to_16(v[2 * i + 1], DT_F16) << 16);
    }
  }
#pragma unroll
  for (int k = 0; k < 2; ++k) stmatrix_x4(stg + stg_stmatrix_offset(row0, 0, lane, cb / 16 + k), pk[4 * k], pk[4 * k + 1], pk[4 * k + 2], pk[4 * k + 3]);
}

// One CTA computes 128 x BN output tiles: warp 0 (lane 0) is the TMA producer, warpgroups 1 and 2 each issue wgmma for 64 of the
// 128 rows and run the fused epilogue on their own accumulators.  With more tiles than CTAs (persistent launch, one CTA per SM)
// a CTA walks the tiles blockIdx.x, blockIdx.x + gridDim.x, ... (column tile fastest, so CTAs running at the same time share A
// rows in L2); the operand ring runs across tile boundaries, so the producer fetches the next tile's operands while the
// epilogue of the current one runs.  epi_mode 2: the tile is staged in SWIZZLE_128B sub-tiles of a dedicated 64 KB region and
// written by TMA stores (full 128-byte lines; rows / columns outside the matrix are clipped by the tensor map); the elected thread
// waits for a store to have read the staging tile only before the next tile is staged.  epi_mode 0: direct per-thread stores.
constexpr uint32_t TC_STG_BYTES = 65536;

template <int BN, int NSTG, int EPI>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_gemm_wg_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w,
                    const __grid_constant__ CUtensorMap tmap_o, const __grid_constant__ CUtensorMap tmap_o2, int N, int K, int taps,
                    int dil, int shift0, int rowsOut, EpiDev ep, int epi_mode, int ntn, int ntiles) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_full[NSTG];
  __shared__ __align__(8) uint64_t bar_empty[NSTG];
  __shared__ __align__(16) float s_bias[BN];
  constexpr uint32_t A_BYTES = TC_BM * TC_BK * 2;
  constexpr uint32_t B_BYTES = BN * TC_BK * 2;
  constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // SWIZZLE_128B needs 1024-B aligned tiles
  const uint32_t stg_base = smem_base + NSTG * STAGE_BYTES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kchunks = (K + TC_BK - 1) / TC_BK;
  const int iters = taps * kchunks;

  if (threadIdx.x == 0) {
    for (int s = 0; s < NSTG; ++s) {
      mbar_init(smem_u32(&bar_full[s]), 1);
      mbar_init(smem_u32(&bar_empty[s]), 8);     // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    if (warp == 0 && lane == 0) {
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int r0 = (tile / ntn) * TC_BM, n0 = (tile % ntn) * BN;
        for (int i = 0; i < iters; ++i, ++it) {
          const uint32_t s = it % NSTG, round = it / NSTG;
          mbar_wait(smem_u32(&bar_empty[s]), (round & 1u) ^ 1u);
          const int j = i / kchunks, kc = i - j * kchunks;
          const uint32_t sa = smem_base + s * STAGE_BYTES;
          const uint32_t fb = smem_u32(&bar_full[s]);
          mbar_expect_tx(fb, STAGE_BYTES);
          tma_load_2d(sa, &tmap_a, fb, kc * TC_BK, r0 + shift0 + j * dil);
          tma_load_3d(sa + A_BYTES, &tmap_w, fb, kc * TC_BK, j, n0);
        }
      }
    }
    return;
  }
  const int ct = threadIdx.x - 128;                   // consumer thread 0..255
  const int wg = ct >> 7;                             // rows [64 wg, 64 wg + 64) of the tile
  const int q = lane & 3;
  const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * (q & 1);   // the tile row this thread's epilogue owns
  const int cq = 16 * (q >> 1);                       // ... and its 16 columns of every 32
  const int frow0 = wg * 64 + (warp & 3) * 16;        // fragment epilogue: the warp's first tile row
  uint32_t it = 0;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int r0 = (tile / ntn) * TC_BM, n0 = (tile % ntn) * BN;
    const int r = r0 + row;
    const bool rin = r < rowsOut;
    // the previous tile's epilogue has read s_bias, and its TMA store has read the staging tile (thread 0 waited below)
    if (ct == 0 && epi_mode == 2) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    asm volatile("bar.sync 1, 256;" ::: "memory");
    for (int i = ct; i < BN; i += 256) s_bias[i] = (ep.bias && n0 + i < N) ? ep.bias[n0 + i] : 0.f;
    int seq = 0;
    bool valid = false;
    FragRows f;
    if (EPI) {
      f = frag_rows(ep, r0 + frow0 + (lane >> 2), rowsOut);
    } else {
      if (rin && ep.row2seq) seq = ep.row2seq[r];
      valid = rin && (!ep.row2seq || seq >= 0);
    }

    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int i = 0; i < iters; ++i, ++it) {
      const uint32_t s = it % NSTG, round = it / NSTG;
      mbar_wait(smem_u32(&bar_full[s]), round & 1u);
      const uint32_t sa = smem_base + s * STAGE_BYTES + (uint32_t)wg * (A_BYTES / 2);
      const uint32_t sb = smem_base + s * STAGE_BYTES + A_BYTES;
      const uint64_t da = wg_desc_sw128(sa), db = wg_desc_sw128(sb);
      wg_fence();
      if (ep.ab_f16) {
#pragma unroll
        for (int k = 0; k < TC_BK / 16; ++k) wgmma_ss<BN, 1>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), 1);
      } else {
#pragma unroll
        for (int k = 0; k < TC_BK / 16; ++k) wgmma_ss<BN, 0>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), 1);
      }
      wg_commit();
      // one group stays in flight: the stage of the previous iteration is released once its MMAs have completed
      wg_wait<1>();
      __syncwarp();
      if (i > 0 && lane == 0) mbar_arrive(smem_u32(&bar_empty[(it - 1) % NSTG]));
    }
    wg_wait<0>();
    wg_touch<BN / 2>(acc);
    __syncwarp();
    if (iters > 0 && lane == 0) mbar_arrive(smem_u32(&bar_empty[(it - 1) % NSTG]));
    asm volatile("bar.sync 1, 256;" ::: "memory");   // s_bias complete

    const uint32_t stg1 = stg_base;
    const uint32_t stg2 = stg_base + (uint32_t)TC_BM * BN * (ep.out_dtype == DT_F32 ? 4u : 2u);
    if (EPI) {
#pragma unroll
      for (int cb = 0; cb < BN; cb += 32) {
        if (n0 + cb >= N) break;
        float v[16];
        frag_values<EPI == 2>(ep, f, s_bias, n0, cb, q, N, acc + cb / 2, v);
        frag_stage16(stg1, ep.out_dtype, frow0, lane, cb, v);
        if (EPI == 1 && ep.out2) {
          frag_values2(ep, f, n0, cb, q, N, v);
          frag_stage16(stg2, ep.out2_dtype, frow0, lane, cb, v);
        }
      }
    } else {
#pragma unroll
      for (int cb = 0; cb < BN; cb += 32) {
        float a16[16], v[16], w2[16];
        wg_frag_rows16(acc + cb / 2, lane, a16);
        const int c = cb + cq;
        if (n0 + c < N) {
          if (epi_mode == 2) {
            if (n0 + c + 16 <= N) epi_math16p(ep, r, rin, seq, valid, s_bias, c, n0 + c, a16, v, w2);
            else epi_math16(ep, r, rin, n0 + c, N, a16, v, w2);
            stage_store16(stg1, ep.out_dtype, row, c, v);
            if (ep.out2) stage_store16(stg2, ep.out2_dtype, row, c, w2);
          } else if (rin) {
            epi_store16(ep, r, n0 + c, N, a16);
          }
        }
      }
    }
    if (epi_mode == 2) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (ct == 0) {
        const int w1 = ep.out_dtype == DT_F32 ? 32 : 64;
        for (int sb = 0; sb * w1 < BN && n0 + sb * w1 < N; ++sb) tma_store_2d(&tmap_o, stg1 + sb * 16384u, n0 + sb * w1, r0);
        if (ep.out2) {
          const int w2c = ep.out2_dtype == DT_F32 ? 32 : 64;
          for (int sb = 0; sb * w2c < BN && n0 + sb * w2c < N; ++sb) tma_store_2d(&tmap_o2, stg2 + sb * 16384u, n0 + sb * w2c, r0);
        }
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
    }
  }
  if (ct == 0 && epi_mode == 2) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

template <int BN, int NSTG>
constexpr size_t wg_smem() {
  return (size_t)NSTG * (TC_BM * TC_BK * 2 + BN * TC_BK * 2) + TC_STG_BYTES + 1024;
}

template <int BN, int NSTG, int EPI>
void launch_wg(cvk_ctx* ctx, cudaStream_t st, const CUtensorMap& ta, const CUtensorMap& tw, const CUtensorMap& to, const CUtensorMap& to2,
               const ConvW& W, int rowsOut, const EpiDev& e, int epi_mode) {
  constexpr size_t smem = wg_smem<BN, NSTG>();
  const int ntn = ceil_div(W.N, BN), ntiles = ntn * ceil_div(rowsOut, TC_BM);
  // more tiles than SMs: persistent CTAs (one per SM) unless switched off
  const int grid = (ctx->tc_persist && ntiles > ctx->num_sms) ? ctx->num_sms : ntiles;
  conv_gemm_wg_kernel<BN, NSTG, EPI><<<grid, TC_THREADS, smem, st>>>(ta, tw, to, to2, W.N, W.K, W.taps, W.dil, W.shift0, rowsOut, e, epi_mode,
                                                                     ntn, ntiles);
}

// ------------------------------------------------------------------------------------------------ row-panel GEMM, K = 256
// out[r, n] = epilogue(sum_k A[r + shift0, k] W[n][k]) for one tap, K = 256 and a wide N (the qkv projection of the flow estimator's
// transformer blocks: 256 -> 1536 on ~40 k rows; option "flow_qkv_panel").  At K = 256 a 128 x 128 tile of conv_gemm_wg_kernel has
// only four ring stages of work, refills 128 KB of operands for it, and nothing runs on the tensor cores under its epilogue.  Here a
// CTA keeps the 128 x 256 activation panel resident (64 KB, four SWIZZLE_128B sub-tiles [128 rows][64 channels], loaded once per
// work unit) and walks 128-column chunks of W ([128][256], 64 KB, all of K) that the producer thread streams through a two-stage ring.
// The two consumer warpgroups own 64 rows each and never wait for one another: each has two accumulator sets (setmaxnreg gives the
// consumers 232 registers), commits the 16 wgmma of chunk c + 1 into one set and runs the epilogue of chunk c from the other while
// they execute, stages its 64 x 128 tile in its own half of the staging region and issues its own TMA store, ordered by a
// 128-thread named barrier of its own.
// Shared memory: A 64 KB + 2 x 64 KB of W + 32 KB of staging = 224 KB (+ 1 KB alignment).  128-column chunks keep the generic
// kernel's m64n128k16 instruction and leave room for exactly two W stages; that suffices because a stage is released as soon as the
// chunk's MMAs complete, before its epilogue, so the refill has the whole epilogue to land.  64-column chunks would allow deeper
// rings but halve the work per wgmma and double the barrier traffic.  Staging 64 x 128 of a 16-bit type per warpgroup: 16-bit outputs only.
// A work unit is (panel, column group): group fastest, so the CTAs running together read the same W chunks from L2, and the CTA
// walks units blockIdx.x, blockIdx.x + gridDim.x, ...  The next unit's first W chunk is requested before its A panel; the panel load
// itself waits for the unit's last MMAs and lands under the last epilogue.
// Per output the MMAs are those of conv_gemm_wg_kernel (K sub-tiles ascending, four k16 steps each, one fp32 accumulator from zero)
// and the epilogue is its 16-bit staged one (frag_math / frag_stage16; epi_math16p / stage_store16 with tc_epi_frag 0), so the results
// agree bit for bit.
constexpr int QP_K = 256, QP_BN = 128, QP_NSTG = 2;
constexpr uint32_t QP_A_BYTES = TC_BM * QP_K * 2;
constexpr uint32_t QP_W_BYTES = QP_BN * QP_K * 2;
constexpr uint32_t QP_STG_BYTES = TC_BM * QP_BN * 2;
constexpr size_t QP_SMEM = QP_A_BYTES + QP_NSTG * QP_W_BYTES + QP_STG_BYTES + 1024;
// fewest panels the dispatch sends here: 3200 rows x 256 -> 1536, the smallest size timed, took 15.5 us against 21.5 us on the generic
// kernel (H100 80GB HBM3, 700 W); smaller launches, the streaming sessions' 50-frame chunks among them, have not been timed and stay there
constexpr int QP_MIN_PANELS = 25;

template <int EPI>
__global__ void __launch_bounds__(TC_THREADS, 1)
qkv_panel_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w,
                 const __grid_constant__ CUtensorMap tmap_o, int shift0, int rowsOut, EpiDev ep, int ngroups, int cpu, int nunits) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_full[QP_NSTG];
  __shared__ __align__(8) uint64_t bar_empty[QP_NSTG];
  __shared__ __align__(8) uint64_t bar_a_full, bar_a_empty;
  __shared__ __align__(16) float s_bias_all[2 * QP_BN];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t w_base = smem_base + QP_A_BYTES;
  const uint32_t stg_base = w_base + QP_NSTG * QP_W_BYTES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < QP_NSTG; ++s) {
      mbar_init(smem_u32(&bar_full[s]), 1);
      mbar_init(smem_u32(&bar_empty[s]), 8);     // one arrival per consumer warp
    }
    mbar_init(smem_u32(&bar_a_full), 1);
    mbar_init(smem_u32(&bar_a_empty), 8);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 0 && lane == 0) {
      uint32_t it = 0, ui = 0;
      for (int u = blockIdx.x; u < nunits; u += gridDim.x, ++ui) {
        const int r0 = (u / ngroups) * TC_BM, c0 = (u % ngroups) * cpu;
        for (int c = 0; c < cpu; ++c, ++it) {
          const uint32_t s = it % QP_NSTG, round = it / QP_NSTG;
          mbar_wait(smem_u32(&bar_empty[s]), (round & 1u) ^ 1u);
          const uint32_t sw = w_base + s * QP_W_BYTES;
          const uint32_t fb = smem_u32(&bar_full[s]);
          mbar_expect_tx(fb, QP_W_BYTES);
#pragma unroll
          for (int kt = 0; kt < QP_K / TC_BK; ++kt) tma_load_3d(sw + kt * (QP_BN * 128u), &tmap_w, fb, kt * TC_BK, 0, (c0 + c) * QP_BN);
          if (c == 0) {     // the panel, once the previous unit's MMAs have read theirs
            mbar_wait(smem_u32(&bar_a_empty), (ui & 1u) ^ 1u);
            const uint32_t fa = smem_u32(&bar_a_full);
            mbar_expect_tx(fa, QP_A_BYTES);
#pragma unroll
            for (int kt = 0; kt < QP_K / TC_BK; ++kt) tma_load_2d(smem_base + kt * (TC_BM * 128u), &tmap_a, fa, kt * TC_BK, r0 + shift0);
          }
        }
      }
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  const int ct = threadIdx.x - 128;                   // consumer thread 0..255
  const int wg = ct >> 7;                             // rows [64 wg, 64 wg + 64) of the panel
  const int wt = ct & 127;                            // thread of the warpgroup
  const int q = lane & 3;
  const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * (q & 1);   // the panel row this thread's epilogue owns
  const int cq = 16 * (q >> 1);                       // ... and its 16 columns of every 32
  const int frow0 = wg * 64 + (warp & 3) * 16;        // fragment epilogue: the warp's first panel row
  const uint32_t a_wg = smem_base + (uint32_t)wg * (64 * 128u);
  float* s_bias = s_bias_all + wg * QP_BN;
  EpiDev e = ep;
  e.out2 = nullptr;                                   // no second output on this path: its epilogue code folds away

  int r0 = 0, r = 0, seq = 0;
  bool rin = false, valid = false;
  FragRows f;
  // the 16 MMAs of one chunk: K sub-tiles ascending, four k16 steps each, into a zeroed accumulator
  auto issue = [&](float* acc, uint32_t it) {
    const uint32_t s = it % QP_NSTG;
    mbar_wait(smem_u32(&bar_full[s]), (it / QP_NSTG) & 1u);
    const uint32_t sw = w_base + s * QP_W_BYTES;
#pragma unroll
    for (int i = 0; i < QP_BN / 2; ++i) acc[i] = 0.f;
    wg_fence();
#pragma unroll
    for (int kt = 0; kt < QP_K / TC_BK; ++kt) {
      const uint64_t da = wg_desc_sw128(a_wg + kt * (TC_BM * 128u)), db = wg_desc_sw128(sw + kt * (QP_BN * 128u));
      if (e.ab_f16) {
#pragma unroll
        for (int k = 0; k < TC_BK / 16; ++k) wgmma_ss<QP_BN, 1>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), 1);
      } else {
#pragma unroll
        for (int k = 0; k < TC_BK / 16; ++k) wgmma_ss<QP_BN, 0>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), 1);
      }
    }
    wg_commit();
  };
  // chunk `it` has completed: free its W stage (and the panel after a unit's last chunk)
  auto release = [&](uint32_t it, bool last) {
    __syncwarp();
    if (lane == 0) {
      mbar_arrive(smem_u32(&bar_empty[it % QP_NSTG]));
      if (last) mbar_arrive(smem_u32(&bar_a_empty));
    }
  };
  // this warpgroup's 64 x 128 tile of columns [n0, n0 + 128): epilogue math, staging, one TMA store per 64 columns
  auto epilogue = [&](float* acc, int n0, float bv) {
    if (wt == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // the previous store has read the staging tile
    s_bias[wt] = bv;
    asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
    if (EPI) {
#pragma unroll
      for (int cb = 0; cb < QP_BN; cb += 32) {
        float v[16];
        frag_math<true, EPI == 2>(e, f, s_bias, n0, cb, q, n0 + QP_BN, acc + cb / 2, v);
        frag_stage16(stg_base, e.out_dtype, frow0, lane, cb, v);
      }
    } else {
#pragma unroll
      for (int cb = 0; cb < QP_BN; cb += 32) {
        float a16[16], v[16], w2[16];
        wg_frag_rows16(acc + cb / 2, lane, a16);
        const int c = cb + cq;
        epi_math16p(e, r, rin, seq, valid, s_bias, c, n0 + c, a16, v, w2);
        stage_store16(stg_base, e.out_dtype, row, c, v);
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
    if (wt == 0) {
#pragma unroll
      for (int sb = 0; sb < QP_BN / 64; ++sb)
        tma_store_2d(&tmap_o, stg_base + sb * 16384u + (uint32_t)wg * 8192u, n0 + sb * 64, r0 + wg * 64);
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
  };

  float acc0[QP_BN / 2], acc1[QP_BN / 2];
  uint32_t it = 0, ui = 0;
  for (int u = blockIdx.x; u < nunits; u += gridDim.x, ++ui) {
    r0 = (u / ngroups) * TC_BM;
    const int nb = (u % ngroups) * cpu * QP_BN;
    if (EPI) {
      f = frag_rows(e, r0 + frow0 + (lane >> 2), rowsOut);
    } else {
      r = r0 + row;
      rin = r < rowsOut;
      seq = 0;
      if (rin && e.row2seq) seq = e.row2seq[r];
      valid = rin && (!e.row2seq || seq >= 0);
    }
    mbar_wait(smem_u32(&bar_a_full), ui & 1u);
    issue(acc0, it);
    for (int c = 0; c < cpu; c += 2) {
      // chunk c is in flight in acc0
      float bv = e.bias ? e.bias[nb + c * QP_BN + wt] : 0.f;
      if (c + 1 < cpu) {
        issue(acc1, it + 1);
        wg_wait<1>();
      } else {
        wg_wait<0>();
      }
      wg_touch<QP_BN / 2>(acc0);
      release(it, c + 1 == cpu);
      epilogue(acc0, nb + c * QP_BN, bv);
      ++it;
      if (c + 1 == cpu) break;
      // chunk c + 1 is in flight in acc1
      bv = e.bias ? e.bias[nb + (c + 1) * QP_BN + wt] : 0.f;
      if (c + 2 < cpu) {
        issue(acc0, it + 1);
        wg_wait<1>();
      } else {
        wg_wait<0>();
      }
      wg_touch<QP_BN / 2>(acc1);
      release(it, c + 2 == cpu);
      epilogue(acc1, nb + (c + 1) * QP_BN, bv);
      ++it;
    }
  }
  if (wt == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

void launch_panel(cvk_ctx* ctx, cudaStream_t st, const CUtensorMap& ta, const CUtensorMap& tw, const CUtensorMap& to, const ConvW& W, int rowsOut,
                  const EpiDev& e) {
  // Column groups per panel: whole panels leave the last wave of CTAs partly idle (313 panels on 132 SMs: 3 waves of 12 chunks
  // where 2.4 are needed), more groups reload the panel more often.  Take the split with the fewest chunk times on the busiest SM,
  // a unit's panel load and its unpipelined first chunk counted as one more.
  const int panels = ceil_div(rowsOut, TC_BM), nch = W.N / QP_BN;
  int ngroups = 1;
  long best = -1;
  for (int g = 1; g <= 4; ++g) {
    if (nch % g) continue;
    const long cost = (long)ceil_div(panels * g, ctx->num_sms) * (nch / g + 1);
    if (best < 0 || cost < best) { best = cost; ngroups = g; }
  }
  const int nunits = panels * ngroups;
  const int grid = std::min(nunits, ctx->num_sms);
  const int epi = !ctx->tc_epi_frag ? 0 : frag_plain(e) ? 2 : 1;
  auto k = epi == 2 ? qkv_panel_kernel<2> : epi == 1 ? qkv_panel_kernel<1> : qkv_panel_kernel<0>;
  k<<<grid, TC_THREADS, QP_SMEM, st>>>(ta, tw, to, W.shift0, rowsOut, e, ngroups, nch / ngroups, nunits);
}

// ------------------------------------------------------------------------------------------------ fused feed-forward
// The feed-forward half of a flow-estimator transformer block in one launch (matcha transformer.py: x = x + ff(norm3(x))):
//   x <- valid(r) ? x + b2 + GELU(LN3(x) W1^T + b1) W2^T : 0,   C = 256 channels, 1024 hidden,
// followed by the bf16 operand the next launch reads: LN1 of the next block over the new x, or a plain bf16 copy of x (the stage's
// output activation).  One CTA owns 128 rows; the 1024-wide hidden activation never leaves the SM: per 64-wide hidden chunk a
// consumer warpgroup computes h = A W1c^T (wgmma, 64 x 64 fp32 in registers), adds the bias, applies the GELU and issues
// O += h W2c^T with h taken straight from its registers (the accumulator layout is the register A-operand layout).  The producer
// warp streams the W1 / W2 chunks through a two-stage ring.  Operations and their order are those of the unfused path
// (layernorm256_kernel, conv_gemm_wg_kernel with the GELU and the residual epilogues: same wgmma K steps in ascending order, same
// bf16 roundings), so the results agree bit for bit.
// With the attention output `att` (bf16 [rows, 512]) the launch first folds in the block's attention output projection and its residual
// (x <- valid(r) ? x + bo + att Wo^T : 0, the out conv-GEMM of the unfused path): the producer streams eight 64-wide K chunks, each the
// CTA's 128 x 64 att slice and a 256 x 64 Wo slice (48 KB), through the same ring ahead of the W1 / W2 chunks; each consumer warpgroup
// accumulates m64n256k16 over K = 512 in ascending order from zero (the conv-GEMM's MMAs), stages acc + bo in fp32 over the A tile
// region (free until LN3) in two 128-column halves, and adds the residual and the row mask per row (the conv-GEMM epilogue's order)
// as it writes x.  LN3 takes the new x from the registers of the lanes that wrote it, and the ring's first W1 / W2 chunks land meanwhile.
constexpr int FF_C = 256, FF_HID = 1024, FF_HC = 64, FF_NCH = FF_HID / FF_HC;
constexpr int FF_OK = 512, FF_OCH = FF_OK / 64;         // out projection: K = 512 (8 heads x 64) in 64-wide ring chunks
constexpr uint32_t FF_ATT_BYTES = TC_BM * 64 * 2;      // att chunk: [128 rows][64], one SWIZZLE_128B sub-tile
constexpr uint32_t FF_WO_BYTES = FF_C * 64 * 2;        // Wo chunk: [256 channels][64]
constexpr uint32_t FF_A_BYTES = TC_BM * FF_C * 2;      // LN3(x): four SWIZZLE_128B sub-tiles [128 rows][64 channels]
constexpr uint32_t FF_W1_BYTES = FF_HC * FF_C * 2;     // W1 chunk: four sub-tiles [64 hidden][64 channels]
constexpr uint32_t FF_W2_BYTES = FF_C * FF_HC * 2;     // W2 chunk: [256 channels][64 hidden]
constexpr uint32_t FF_STAGE_BYTES = FF_W1_BYTES + FF_W2_BYTES;
constexpr int FF_NSTG = 2;
constexpr int FF_OLD = FF_C + 8;                       // pitch (floats) of the fp32 output tile staged over the operand region
constexpr size_t FF_SMEM = FF_A_BYTES + FF_NSTG * FF_STAGE_BYTES + 1024;
static_assert((size_t)TC_BM * FF_OLD * 4 <= FF_A_BYTES + FF_NSTG * FF_STAGE_BYTES, "output staging tile must fit the operand region");
static_assert(FF_ATT_BYTES + FF_WO_BYTES <= FF_STAGE_BYTES, "an out-projection chunk must fit a ring stage");
static_assert((size_t)TC_BM * (FF_C / 2) * 4 <= FF_A_BYTES, "a half of the out-projection tile must fit the A tile region");

struct FfnDev {
  float* x;                      // [rows][ldx] fp32 residual stream, in place
  int ldx, rows;
  const int* row2seq;
  const float *ln3_g, *ln3_b, *b1, *b2;
  const float *ln_g, *ln_b;      // LN1 of the next block; null: out is a bf16 copy of x
  const float* bo;               // out-projection bias; null: no out-projection phase (x is taken as given)
  bf16* out;
  int ldo;
};

// byte address of (row, column c) of a warpgroup's 128-column half of the fp32 out-projection tile, laid over its own rows of the A tile
// (row `grow` of the CTA tile; 32 columns per 128-byte sub-tile row, 16-byte chunks XOR-swizzled so that the fragment stores and the
// row reads are free of bank conflicts).  LN3 later writes these same bytes from the same warpgroup's rows.
__device__ __forceinline__ uint32_t ff_stg_addr(uint32_t base, int grow, int c) {
  return base + (uint32_t)(c >> 5) * (TC_BM * 128u) + (uint32_t)grow * 128u + ((((uint32_t)(c & 31) >> 2) ^ ((uint32_t)(grow & 3) << 1)) << 4) +
         (uint32_t)(c & 3) * 4u;
}

__global__ void __launch_bounds__(TC_THREADS, 1)
ffn_fused_kernel(const __grid_constant__ CUtensorMap tmap_w1, const __grid_constant__ CUtensorMap tmap_w2,
                 const __grid_constant__ CUtensorMap tmap_att, const __grid_constant__ CUtensorMap tmap_wo, FfnDev p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_full[FF_NSTG];
  __shared__ __align__(8) uint64_t bar_empty[FF_NSTG];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t w_base = smem_base + FF_A_BYTES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = blockIdx.x * TC_BM;

  if (threadIdx.x == 0) {
    for (int s = 0; s < FF_NSTG; ++s) {
      mbar_init(smem_u32(&bar_full[s]), 1);
      mbar_init(smem_u32(&bar_empty[s]), 8);     // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int och = p.bo ? FF_OCH : 0;                  // ring chunks of the out projection, ahead of the FF chunks
  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 0 && lane == 0) {
      for (int g = 0; g < och + FF_NCH; ++g) {
        const uint32_t s = g % FF_NSTG, round = g / FF_NSTG;
        mbar_wait(smem_u32(&bar_empty[s]), (round & 1u) ^ 1u);
        const uint32_t sw = w_base + s * FF_STAGE_BYTES;
        const uint32_t fb = smem_u32(&bar_full[s]);
        if (g < och) {
          mbar_expect_tx(fb, FF_ATT_BYTES + FF_WO_BYTES);
          tma_load_2d(sw, &tmap_att, fb, g * 64, r0);
          tma_load_2d(sw + FF_ATT_BYTES, &tmap_wo, fb, g * 64, 0);
          continue;
        }
        const int c = g - och;
        mbar_expect_tx(fb, FF_STAGE_BYTES);
#pragma unroll
        for (int kt = 0; kt < FF_C / 64; ++kt) tma_load_2d(sw + kt * (FF_HC * 128u), &tmap_w1, fb, kt * 64, c * FF_HC);
        tma_load_2d(sw + FF_W1_BYTES, &tmap_w2, fb, c * FF_HC, 0);
      }
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  const int ct = threadIdx.x - 128;                   // consumer thread 0..255
  const int wg = ct >> 7;                             // rows [64 wg, 64 wg + 64) of the tile
  const int cw = ct >> 5;                             // consumer warp 0..7
  const int c0 = lane * 4, c1 = 128 + lane * 4;       // this lane's columns in the row-per-warp phases
  const int q = lane & 3;

  // this lane's columns c0 and c1 of x in the 16 rows of its warp (valid rows only), loaded together so that their latencies overlap;
  // with the out projection they become the new x, so LN3 takes them from registers
  float4 xa[16], xb[16];
  uint32_t okm = 0;                                   // bit i: row i of the warp is a valid (sequence) row
  auto load_x = [&](float4* xv, int c) {
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int r = r0 + cw * 16 + i;
      xv[i] = (okm >> i) & 1u ? *reinterpret_cast<const float4*>(p.x + (size_t)r * p.ldx + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int r = r0 + cw * 16 + i;
    if (r < p.rows && p.row2seq[r] >= 0) okm |= 1u << i;
  }

  if (och) {
    // out projection: acc = att Wo^T over the ring's first FF_OCH chunks, one MMA group in flight (conv_gemm_wg_kernel's loop)
    float acc[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    for (int g = 0; g < FF_OCH; ++g) {
      const uint32_t s = g % FF_NSTG;
      mbar_wait(smem_u32(&bar_full[s]), (uint32_t)(g / FF_NSTG) & 1u);
      const uint32_t sa = w_base + s * FF_STAGE_BYTES;
      const uint64_t da = wg_desc_sw128(sa + (uint32_t)wg * (64 * 128u)), db = wg_desc_sw128(sa + FF_ATT_BYTES);
      wg_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_ss<256, 0>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), 1);
      wg_commit();
      wg_wait<1>();
      __syncwarp();
      if (g > 0 && lane == 0) mbar_arrive(smem_u32(&bar_empty[(g - 1) % FF_NSTG]));
    }
    wg_wait<0>();
    wg_touch<128>(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&bar_empty[(FF_OCH - 1) % FF_NSTG]));
    // per 128-column half: acc + bo staged in fp32 over this warpgroup's rows of the A tile, then per row (one warp per row, the rows
    // LN3 gives the warp below) + residual and the row mask into x
    const int fr = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // tile row of acc[4 j], acc[4 j + 1]; + 8 for acc[4 j + 2], acc[4 j + 3]
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = 8 * j + 2 * q;
        const float* a = acc + 64 * hf + 4 * j;
        const float2 b = *reinterpret_cast<const float2*>(p.bo + 128 * hf + col);
        asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(ff_stg_addr(smem_base, fr, col)), "f"(a[0] + b.x), "f"(a[1] + b.y) : "memory");
        asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(ff_stg_addr(smem_base, fr + 8, col)), "f"(a[2] + b.x), "f"(a[3] + b.y) : "memory");
      }
      if (hf == 0) load_x(xa, c0);                    // the residual of this half, all 16 rows in flight at once
      else load_x(xb, c1);
      asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
      float4* xv = hf ? xb : xa;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int row = cw * 16 + i, r = r0 + row;
        if (r >= p.rows) break;
        float4 v;
        asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(ff_stg_addr(smem_base, row, c0)) : "memory");
        const float4 xr = xv[i];
        xv[i] = (okm >> i) & 1u ? make_float4(v.x + xr.x, v.y + xr.y, v.z + xr.z, v.w + xr.w) : make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4*>(p.x + (size_t)r * p.ldx + 128 * hf + c0) = xv[i];
      }
      asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");   // the half has been read: the region takes the next one, then LN3
    }
  } else {
    load_x(xa, c0);
    load_x(xb, c1);
  }

  // LN3 prologue, one warp per row as in layernorm256_kernel: bf16 rows of the A tile (gap rows and rows past the end are zero)
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int row = cw * 16 + i;
    float v[8] = {xa[i].x, xa[i].y, xa[i].z, xa[i].w, xb[i].x, xb[i].y, xb[i].z, xb[i].w};
    if ((okm >> i) & 1u) ln256_warp(v, p.ln3_g, p.ln3_b, 1e-5f, c0, c1);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int c = h ? c1 : c0;
      __nv_bfloat162 lo = __floats2bfloat162_rn(v[4 * h], v[4 * h + 1]), hi = __floats2bfloat162_rn(v[4 * h + 2], v[4 * h + 3]);
      const uint32_t addr = smem_base + (uint32_t)(c >> 6) * (TC_BM * 128u) + (uint32_t)row * 128u +
                            ((((uint32_t)(c & 63) >> 3) ^ (uint32_t)(row & 7)) << 4) + (uint32_t)(c & 7) * 2u;
      asm volatile("st.shared.v2.b32 [%0], {%1,%2};" ::"r"(addr), "r"(*reinterpret_cast<uint32_t*>(&lo)), "r"(*reinterpret_cast<uint32_t*>(&hi))
                   : "memory");
    }
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> wgmma operand reads
  asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");     // this warpgroup's 64 rows are complete

  float o[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) o[i] = 0.f;
  uint32_t hp[16];
  const uint32_t a_wg = smem_base + (uint32_t)wg * (64 * 128u);
  for (int c = 0; c < FF_NCH; ++c) {
    const uint32_t g = och + c;                       // ring chunk
    const uint32_t s = g % FF_NSTG;
    mbar_wait(smem_u32(&bar_full[s]), (g / FF_NSTG) & 1u);
    const uint32_t sw1 = w_base + s * FF_STAGE_BYTES, sw2 = sw1 + FF_W1_BYTES;
    float h[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) h[i] = 0.f;
    wg_fence();
#pragma unroll
    for (int kt = 0; kt < FF_C / 64; ++kt) {
      const uint64_t da = wg_desc_sw128(a_wg + kt * (TC_BM * 128u)), db = wg_desc_sw128(sw1 + kt * (FF_HC * 128u));
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_ss<64, 0>(h, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), 1);
    }
    wg_commit();
    wg_wait<0>();                                     // FF1 of this chunk and FF2 of the previous one have completed
    wg_touch<32>(h);
    __syncwarp();
    if (c > 0 && lane == 0) mbar_arrive(smem_u32(&bar_empty[(g - 1) % FF_NSTG]));
    // bias + GELU as the FF1 epilogue computes them (act16_fast), bf16 pairs in the register A-operand layout
    const float* b1 = p.b1 + c * FF_HC + 2 * q;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float2 b = *reinterpret_cast<const float2*>(b1 + 8 * j);
      h[4 * j] += b.x; h[4 * j + 1] += b.y; h[4 * j + 2] += b.x; h[4 * j + 3] += b.y;
    }
    gelu16_packed(h);
    gelu16_packed(h + 16);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      __nv_bfloat162 t = __floats2bfloat162_rn(h[2 * j], h[2 * j + 1]);
      hp[j] = *reinterpret_cast<uint32_t*>(&t);
    }
    const uint64_t d2 = wg_desc_sw128(sw2);
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < FF_HC / 16; ++kk) wgmma_rs_m64n256(o, hp + 4 * kk, d2 + (uint64_t)(2 * kk), 1);
    wg_commit();
  }
  wg_wait<0>();
  wg_touch<128>(o);
  asm volatile("bar.sync 1, 256;" ::: "memory");     // every MMA of the CTA has completed: the operand region is free

  // O + b2 -> fp32 staging tile [128][FF_OLD] over the operand region
  float* stg = reinterpret_cast<float*>(smem_raw + (smem_base - smem_u32(smem_raw)));
  {
    const int rb = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int col = 8 * j + 2 * q;
      const float2 b = *reinterpret_cast<const float2*>(p.b2 + col);
      *reinterpret_cast<float2*>(stg + rb * FF_OLD + col) = make_float2(o[4 * j] + b.x, o[4 * j + 1] + b.y);
      *reinterpret_cast<float2*>(stg + (rb + 8) * FF_OLD + col) = make_float2(o[4 * j + 2] + b.x, o[4 * j + 3] + b.y);
    }
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");

  // full rows, one warp per row: + residual, row mask, x out, then LN1 of the next block or the bf16 copy
  for (int i = 0; i < 16; ++i) {
    const int row = cw * 16 + i, r = r0 + row;
    if (r >= p.rows) break;
    const bool valid = p.row2seq[r] >= 0;
    float* xp = p.x + (size_t)r * p.ldx;
    const float* sp = stg + row * FF_OLD;
    const float4 sa = *reinterpret_cast<const float4*>(sp + c0), sb = *reinterpret_cast<const float4*>(sp + c1);
    const float4 xa = *reinterpret_cast<const float4*>(xp + c0), xb = *reinterpret_cast<const float4*>(xp + c1);
    float v[8] = {sa.x + xa.x, sa.y + xa.y, sa.z + xa.z, sa.w + xa.w, sb.x + xb.x, sb.y + xb.y, sb.z + xb.z, sb.w + xb.w};
    if (!valid) {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = 0.f;
    }
    *reinterpret_cast<float4*>(xp + c0) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(xp + c1) = make_float4(v[4], v[5], v[6], v[7]);
    if (p.ln_g && valid) ln256_warp(v, p.ln_g, p.ln_b, 1e-5f, c0, c1);
    bf16* op = p.out + (size_t)r * p.ldo;
    __nv_bfloat162 h0 = __floats2bfloat162_rn(v[0], v[1]), h1 = __floats2bfloat162_rn(v[2], v[3]);
    __nv_bfloat162 h2 = __floats2bfloat162_rn(v[4], v[5]), h3 = __floats2bfloat162_rn(v[6], v[7]);
    *reinterpret_cast<uint2*>(op + c0) = make_uint2(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1));
    *reinterpret_cast<uint2*>(op + c1) = make_uint2(*reinterpret_cast<uint32_t*>(&h2), *reinterpret_cast<uint32_t*>(&h3));
  }
}

}  // namespace

void conv_gemm_tc(cvk_ctx* ctx, cudaStream_t st, const Mat& A, const ConvW& W, const Epilogue& ep) {
  CVK_REQUIRE((A.dtype == DT_BF16 && W.w16 != nullptr) || (A.dtype == DT_F16 && W.wf16 != nullptr), "conv_gemm_tc: 16-bit operands (A and W of the same kind) required");
  const void* w16p = A.dtype == DT_F16 ? (const void*)W.wf16 : (const void*)W.w16;
  CVK_REQUIRE(A.cols >= W.K, "conv_gemm_tc: A has fewer columns than K");
  CVK_REQUIRE(W.K % 8 == 0 && A.ld % 8 == 0 && ((uintptr_t)A.p & 15) == 0, "conv_gemm_tc: operands must be 16-byte aligned");
  CVK_REQUIRE(ep.out.p != nullptr && ep.out.cols >= W.N, "conv_gemm_tc: bad output");
  const int BN = W.N > 64 ? 128 : 64;
  CUtensorMap ta, tw;
  {
    const cuuint64_t dims[2] = {(cuuint64_t)W.K, (cuuint64_t)A.rows};
    const cuuint64_t strides[1] = {(cuuint64_t)A.ld * 2};
    const cuuint32_t box[2] = {TC_BK, TC_BM};
    encode_tma_map(ctx, &ta, A.p, 2, dims, strides, box, A.dtype, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "A");
  }
  {
    const cuuint64_t dims[3] = {(cuuint64_t)W.K, (cuuint64_t)W.taps, (cuuint64_t)W.N};
    const cuuint64_t strides[2] = {(cuuint64_t)W.K * 2, (cuuint64_t)W.K * W.taps * 2};
    const cuuint32_t box[3] = {TC_BK, 1, (cuuint32_t)BN};
    encode_tma_map(ctx, &tw, w16p, 3, dims, strides, box, A.dtype, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "W");
  }
  EpiDev e = to_dev(ep);
  e.ab_f16 = A.dtype == DT_F16;
  if (!e.bias) e.bias = W.bias;
  int rowsOut = ep.out.rows;
  CVK_REQUIRE((ep.out.ld * ep.out.esize()) % 16 == 0 && ((uintptr_t)ep.out.p & 15) == 0, "conv_gemm_tc: output rows must be 16-byte aligned");
  CVK_REQUIRE(!ep.resid.p || (ep.resid.ld % 4 == 0 && ((uintptr_t)ep.resid.p & 15) == 0), "conv_gemm_tc: residual alignment");
  CVK_REQUIRE(!(ep.resid.p && ep.rowvec), "conv_gemm_tc: residual and per-sequence vector cannot be combined");
  CVK_REQUIRE(!ep.rowvec || (ep.rowvec_ld % 4 == 0 && ((uintptr_t)ep.rowvec & 15) == 0), "conv_gemm_tc: rowvec alignment");
  CVK_REQUIRE(!ep.out2.p || ((ep.out2.ld * ep.out2.esize()) % 16 == 0 && ((uintptr_t)ep.out2.p & 15) == 0), "conv_gemm_tc: out2 alignment");
  const double flops = 2.0 * rowsOut * (double)W.N * W.K * W.taps;
  const double bytes = (double)rowsOut * W.K * 2 + (double)W.N * W.K * W.taps * 2 + (double)rowsOut * W.N * ep.out.esize();
  ProfScope ps(ctx, st, FAM_GEMM_TC, flops, bytes);
  // epilogue mode: 2 = staged TMA stores (default when the output tile(s) fit the staging region and no read-modify-write of the
  // output is needed), otherwise direct per-thread stores
  int epi_mode = ctx->tc_epi == 2 ? 2 : 0;
  CUtensorMap to = ta, to2 = ta;
  if (epi_mode == 2) {
    const size_t need = (size_t)TC_BM * BN * ep.out.esize() + (ep.out2.p ? (size_t)TC_BM * BN * ep.out2.esize() : 0);
    // the TMA store of a tile whose last column ends inside a 16-byte chunk of the row also overwrote the columns past N (an H100
    // wrote the pad columns of N = 1 in pitch 4 and of N = 18 in pitch 24, fp32): such widths take the direct stores, which write [0, N) only
    const bool whole16 = (W.N * ep.out.esize()) % 16 == 0 && (!ep.out2.p || (W.N * ep.out2.esize()) % 16 == 0);
    if (ep.accumulate || need > TC_STG_BYTES || !whole16) epi_mode = 0;
  }
  // the row-panel kernel: one tap, K = 256, wide N in whole 128-column chunks, one 16-bit output through the staged stores, and at
  // least QP_MIN_PANELS 128-row panels (option 2: any row count)
  const bool panel = ctx->flow_qkv_panel && epi_mode == 2 && W.taps == 1 && W.K == QP_K && W.N % QP_BN == 0 && W.N >= 512 && !ep.out2.p &&
                     ep.out.esize() == 2 && (ctx->flow_qkv_panel == 2 || ceil_div(rowsOut, TC_BM) >= QP_MIN_PANELS);
  if (epi_mode == 2) {
    auto mk = [&](CUtensorMap* m, const Mat& o) {
      const cuuint64_t dims[2] = {(cuuint64_t)W.N, (cuuint64_t)rowsOut};
      const cuuint64_t strides[1] = {(cuuint64_t)o.ld * o.esize()};
      const cuuint32_t box[2] = {(cuuint32_t)(o.dtype == DT_F32 ? 32 : 64), (cuuint32_t)(panel ? TC_BM / 2 : TC_BM)};   // panel: a store per warpgroup
      encode_tma_map(ctx, m, o.p, 2, dims, strides, box, o.dtype, CU_TENSOR_MAP_L2_PROMOTION_NONE, "out");
    };
    mk(&to, ep.out);
    if (ep.out2.p) mk(&to2, ep.out2);
  }
  if (panel) launch_panel(ctx, st, ta, tw, to, W, rowsOut, e);
  else {
    // the fragment epilogue: staged stores of 16-bit outputs only (see frag_values)
    const bool frag = ctx->tc_epi_frag && epi_mode == 2 && ep.out.esize() == 2 && (!ep.out2.p || ep.out2.esize() == 2);
    const int epi = !frag ? 0 : frag_plain(e) ? 2 : 1;
    if (BN == 128) {
      if (epi == 2) launch_wg<128, 4, 2>(ctx, st, ta, tw, to, to2, W, rowsOut, e, epi_mode);
      else if (epi == 1) launch_wg<128, 4, 1>(ctx, st, ta, tw, to, to2, W, rowsOut, e, epi_mode);
      else launch_wg<128, 4, 0>(ctx, st, ta, tw, to, to2, W, rowsOut, e, epi_mode);
    } else {
      if (epi == 2) launch_wg<64, 4, 2>(ctx, st, ta, tw, to, to2, W, rowsOut, e, epi_mode);
      else if (epi == 1) launch_wg<64, 4, 1>(ctx, st, ta, tw, to, to2, W, rowsOut, e, epi_mode);
      else launch_wg<64, 4, 0>(ctx, st, ta, tw, to, to2, W, rowsOut, e, epi_mode);
    }
  }
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}

void ffn_fused(cvk_ctx* ctx, cudaStream_t st, const Mat& x, const Mat* att, const ConvW* wo, const int* row2seq, const float* ln3_g,
               const float* ln3_b, const ConvW& w1, const ConvW& w2, const float* ln_g, const float* ln_b, const Mat& out) {
  CVK_REQUIRE(x.dtype == DT_F32 && x.cols == FF_C && x.ld % 4 == 0 && ((uintptr_t)x.p & 15) == 0, "ffn_fused: x must be fp32 [rows, 256], 16-byte aligned rows");
  CVK_REQUIRE(!att == !wo, "ffn_fused: the out projection needs both att and its weights");
  if (att) {
    CVK_REQUIRE(att->dtype == DT_BF16 && att->cols == FF_OK && att->rows >= x.rows && att->ld % 8 == 0 && ((uintptr_t)att->p & 15) == 0,
                "ffn_fused: att must be bf16 [rows, 512], 16-byte aligned rows");
    CVK_REQUIRE(wo->N == FF_C && wo->K == FF_OK && wo->taps == 1 && wo->w16 && wo->bias && ((uintptr_t)wo->bias & 15) == 0,
                "ffn_fused: unexpected out-projection weights");
  }
  CVK_REQUIRE(out.dtype == DT_BF16 && out.cols == FF_C && out.rows >= x.rows && out.ld % 8 == 0 && ((uintptr_t)out.p & 15) == 0,
              "ffn_fused: out must be bf16 [rows, 256], 16-byte aligned rows");
  CVK_REQUIRE(w1.N == FF_HID && w1.K == FF_C && w1.taps == 1 && w1.w16 && w1.bias && w2.N == FF_C && w2.K == FF_HID && w2.taps == 1 && w2.w16 &&
                  w2.bias && row2seq && ln3_g && ln3_b && (!ln_g || ln_b),
              "ffn_fused: unexpected weights");
  CVK_REQUIRE((((uintptr_t)ln3_g | (uintptr_t)ln3_b | (uintptr_t)ln_g | (uintptr_t)ln_b | (uintptr_t)w1.bias | (uintptr_t)w2.bias) & 15) == 0,
              "ffn_fused: LayerNorm and bias vectors must be 16-byte aligned");
  CUtensorMap t1, t2;
  auto mk = [&](CUtensorMap* m, const bf16* w, int N, int K, int box_n) {
    const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)N};
    const cuuint64_t strides[1] = {(cuuint64_t)K * 2};
    const cuuint32_t box[2] = {64, (cuuint32_t)box_n};
    encode_tma_map(ctx, m, w, 2, dims, strides, box, DT_BF16, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "ffn weights");
  };
  mk(&t1, w1.w16, FF_HID, FF_C, FF_HC);
  mk(&t2, w2.w16, FF_C, FF_HID, FF_C);
  CUtensorMap ta = t1, two = t1;                      // not read without the out projection
  if (att) {
    const cuuint64_t dims[2] = {(cuuint64_t)FF_OK, (cuuint64_t)att->rows};
    const cuuint64_t strides[1] = {(cuuint64_t)att->ld * 2};
    const cuuint32_t box[2] = {64, TC_BM};
    encode_tma_map(ctx, &ta, att->p, 2, dims, strides, box, DT_BF16, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "att");
    mk(&two, wo->w16, FF_C, FF_OK, FF_C);
  }
  FfnDev p;
  p.x = x.f32(); p.ldx = x.ld; p.rows = x.rows; p.row2seq = row2seq;
  p.ln3_g = ln3_g; p.ln3_b = ln3_b; p.b1 = w1.bias; p.b2 = w2.bias; p.ln_g = ln_g; p.ln_b = ln_b;
  p.bo = att ? wo->bias : nullptr;
  p.out = out.b16(); p.ldo = out.ld;
  double flops = 4.0 * x.rows * (double)FF_C * FF_HID;
  double bytes = (double)x.rows * FF_C * (4 + 4 + 2) + 2.0 * FF_C * FF_HID * 2;
  if (att) {
    flops += 2.0 * x.rows * (double)FF_C * FF_OK;
    bytes += (double)x.rows * FF_OK * 2 + (double)FF_C * FF_OK * 2;
  }
  ProfScope ps(ctx, st, FAM_GEMM_TC, flops, bytes);
  ffn_fused_kernel<<<ceil_div(x.rows, TC_BM), TC_THREADS, FF_SMEM, st>>>(t1, t2, ta, two, p);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}

void gemm_tc_setup() {
  auto set = [](auto epi) {
    constexpr int E = decltype(epi)::value;
    CVK_CHECK_CUDA(cudaFuncSetAttribute(conv_gemm_wg_kernel<128, 4, E>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wg_smem<128, 4>()));
    CVK_CHECK_CUDA(cudaFuncSetAttribute(conv_gemm_wg_kernel<64, 4, E>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wg_smem<64, 4>()));
    CVK_CHECK_CUDA(cudaFuncSetAttribute(qkv_panel_kernel<E>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)QP_SMEM));
  };
  set(std::integral_constant<int, 0>());
  set(std::integral_constant<int, 1>());
  set(std::integral_constant<int, 2>());
  CVK_CHECK_CUDA(cudaFuncSetAttribute(ffn_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FF_SMEM));
}
