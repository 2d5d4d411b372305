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

namespace {

constexpr int TC_BM = 128;
constexpr int TC_BK = 64;   // 64 bf16 = 128 B = one SWIZZLE_128B atom row
constexpr int TC_THREADS = 384;   // warpgroup 0: TMA producer (one thread), warpgroups 1-2: wgmma + epilogue, 64 rows each

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// bounded spin: a broken pipeline traps (-> CUDA error in the host API) instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok = 0;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  if (ok) return;            // fast path without clock reads: the wait sits on the single MMA-issuing thread's instruction stream
  const long long t0 = clock64();
  for (;;) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    if (ok) return;
    if (clock64() - t0 > 4000000000ll) break;   // ~2 s at 2 GHz
  }
  __trap();
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(map), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
      "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

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
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(map), "r"(src), "r"(c0), "r"(c1) : "memory");
}

// One CTA computes 128 x BN output tiles: warp 0 (lane 0) is the TMA producer, warpgroups 1 and 2 each issue wgmma for 64 of the
// 128 rows and run the fused epilogue on their own accumulators.  With more tiles than CTAs (persistent launch, one CTA per SM)
// a CTA walks the tiles blockIdx.x, blockIdx.x + gridDim.x, ... (column tile fastest, so CTAs running at the same time share A
// rows in L2); the operand ring runs across tile boundaries, so the producer fetches the next tile's operands while the
// epilogue of the current one runs.  epi_mode 2: the tile is staged in SWIZZLE_128B sub-tiles of a dedicated 64 KB region and
// written by TMA stores (full 128-byte lines; rows / columns outside the matrix are clipped by the tensor map); the elected thread
// waits for a store to have read the staging tile only before the next tile is staged.  epi_mode 0: direct per-thread stores.
constexpr uint32_t TC_STG_BYTES = 65536;

template <int BN, int NSTG>
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
    if (rin && ep.row2seq) seq = ep.row2seq[r];
    const bool valid = rin && (!ep.row2seq || seq >= 0);

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

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode(cvk_ctx* ctx) {
  if (!ctx->encode_tiled) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    CVK_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    CVK_REQUIRE(fn != nullptr && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available");
    ctx->encode_tiled = fn;
  }
  return (EncodeTiledFn)ctx->encode_tiled;
}

template <int BN, int NSTG>
void launch_wg(cvk_ctx* ctx, cudaStream_t st, const CUtensorMap& ta, const CUtensorMap& tw, const CUtensorMap& to, const CUtensorMap& to2,
               const ConvW& W, int rowsOut, const EpiDev& e, int epi_mode) {
  constexpr size_t smem = (size_t)NSTG * (TC_BM * TC_BK * 2 + BN * TC_BK * 2) + TC_STG_BYTES + 1024;
  static bool attr_set = false;
  if (!attr_set) {
    CVK_CHECK_CUDA(cudaFuncSetAttribute(conv_gemm_wg_kernel<BN, NSTG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set = true;
  }
  const int ntn = ceil_div(W.N, BN), ntiles = ntn * ceil_div(rowsOut, TC_BM);
  // more tiles than SMs: persistent CTAs (one per SM) unless switched off
  const int grid = (ctx->tc_persist && ntiles > ctx->num_sms) ? ctx->num_sms : ntiles;
  conv_gemm_wg_kernel<BN, NSTG><<<grid, TC_THREADS, smem, st>>>(ta, tw, to, to2, W.N, W.K, W.taps, W.dil, W.shift0, rowsOut, e, epi_mode, ntn, ntiles);
}

}  // namespace

void conv_gemm_tc(cvk_ctx* ctx, cudaStream_t st, const Mat& A, const ConvW& W, const Epilogue& ep) {
  CVK_REQUIRE((A.dtype == DT_BF16 && W.w16 != nullptr) || (A.dtype == DT_F16 && W.wf16 != nullptr), "conv_gemm_tc: 16-bit operands (A and W of the same kind) required");
  const void* w16p = A.dtype == DT_F16 ? (const void*)W.wf16 : (const void*)W.w16;
  CVK_REQUIRE(A.cols >= W.K, "conv_gemm_tc: A has fewer columns than K");
  CVK_REQUIRE(W.K % 8 == 0 && A.ld % 8 == 0 && ((uintptr_t)A.p & 15) == 0, "conv_gemm_tc: operands must be 16-byte aligned");
  CVK_REQUIRE(ep.out.p != nullptr && ep.out.cols >= W.N, "conv_gemm_tc: bad output");
  EncodeTiledFn enc = get_encode(ctx);
  const int BN = W.N > 64 ? 128 : 64;
  CUtensorMap ta, tw;
  {
    cuuint64_t dims[2] = {(cuuint64_t)W.K, (cuuint64_t)A.rows};
    cuuint64_t strides[1] = {(cuuint64_t)A.ld * 2};
    cuuint32_t box[2] = {TC_BK, TC_BM};
    cuuint32_t es[2] = {1, 1};
    CUresult r = enc(&ta, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, A.p, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CVK_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(A) failed: " + std::to_string((int)r));
  }
  {
    cuuint64_t dims[3] = {(cuuint64_t)W.K, (cuuint64_t)W.taps, (cuuint64_t)W.N};
    cuuint64_t strides[2] = {(cuuint64_t)W.K * 2, (cuuint64_t)W.K * W.taps * 2};
    cuuint32_t box[3] = {TC_BK, 1, (cuuint32_t)BN};
    cuuint32_t es[3] = {1, 1, 1};
    CUresult r = enc(&tw, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(w16p), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CVK_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(W) failed: " + std::to_string((int)r));
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
  if (epi_mode == 2) {
    auto mk = [&](CUtensorMap* m, const Mat& o) {
      cuuint64_t dims[2] = {(cuuint64_t)W.N, (cuuint64_t)rowsOut};
      cuuint64_t strides[1] = {(cuuint64_t)o.ld * o.esize()};
      cuuint32_t box[2] = {(cuuint32_t)(o.dtype == DT_F32 ? 32 : 64), TC_BM};
      cuuint32_t es[2] = {1, 1};
      CUresult r = enc(m, o.dtype == DT_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, o.p, dims, strides, box, es,
                       CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      CVK_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(out) failed: " + std::to_string((int)r));
    };
    mk(&to, ep.out);
    if (ep.out2.p) mk(&to2, ep.out2);
  }
  if (BN == 128) launch_wg<128, 4>(ctx, st, ta, tw, to, to2, W, rowsOut, e, epi_mode);
  else launch_wg<64, 4>(ctx, st, ta, tw, to, to2, W, rowsOut, e, epi_mode);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}
