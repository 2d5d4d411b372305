// Persistent decode kernel of the speech-token LM: ALL transformer layers of one decode step (cosyvoice/llm/llm.py:536-549
// loop body -> Qwen2Encoder.forward_one_step :242-254 -> transformers Qwen2 decoder layers, SURVEY.md Appendix C) in ONE
// cooperative kernel instead of 7 PDL-chained kernels per layer.
//
// Why: the step is HBM-bound in principle (727.6 MB of bf16 weights per step shared by all rows, SURVEY.md §8d) but the
// per-op chain is latency-bound: 171 kernels per step, each a launch + a few dependent memory round trips.  Here
//   * one CTA per SM stays resident for the whole step; phases are separated by grid-wide barriers (one release-add + one
//     acquire-polled word in L2) instead of kernel boundaries;
//   * the weights are re-laid out once into PER-CTA STREAMS: the SWIZZLE_128B operand blocks ([64 .. 80 output rows] x [64 K],
//     8 - 10 KB) a CTA will consume, in the order it consumes them, across phases and layers.  Every projection is cut by OUTPUT
//     ROWS (and K ranges) so that all CTAs carry about the same bytes per layer and no unit exceeds the ring;
//     a dedicated producer warp walks the stream with plain bulk copies into a shared-memory ring of 10 KB slots and never
//     waits for a phase boundary, so HBM keeps streaming through the barriers and the latency-bound phases.  At most
//     MG_INFLIGHT blocks of a CTA are in flight at once: a deeper burst only queues in front of the latency-critical loads
//     and stores of the same SM;
//   * GEMMs are swap-AB wgmma (weights = the M side: two warpgroups read 64 rows each from the slot, rows past the block belong
//     to the next slot and produce accumulator rows nobody reads; the <= 64 batch rows = wgmma N) with fp32 accumulators in
//     registers; activations (the B operand) are gathered with ld.global.cg into the swizzled layout after the barrier;
//   * split-K partial sums go to a small fp32 scratch and are reduced in a fixed order (deterministic, no atomics) by the
//     attention unit (qkv) or by a per-row reduce + residual + RMSNorm phase (o_proj, down_proj).
// Phases per layer: qkv GEMM | bias + RoPE + cache append + attention | o GEMM | +res, RMSNorm | gate/up GEMM + SwiGLU |
// down GEMM | +res, RMSNorm.
#include "llm_decode_attn.cuh"
#include "wgmma.cuh"
#include <algorithm>
#include <type_traits>

using namespace lm;

namespace {

constexpr int MG_THREADS = 512;          // warp 0: weight producer; warps 1..15: workers (4..11: the two MMA warpgroups)
constexpr int MG_WORKERS = MG_THREADS - 32;
constexpr int MG_NW = MG_WORKERS / 32;   // 15
constexpr int MG_BK = 64;
constexpr int MG_MAXROWS = 80;           // output rows of a weight block (multiple of 8)
constexpr uint32_t MG_SLOT = MG_MAXROWS * 128;   // 10 KB ring slot (a 64-row block uses 8 KB of it)
constexpr int MG_MAX_STAGES = 16;
constexpr int MG_INFLIGHT = 3;           // bulk copies of one CTA in flight
constexpr int MG_KCH = D / MG_BK;        // 14 K chunks of the 896-wide activations
constexpr int MG_PH = 4;                 // GEMM phases per layer: qkv, o, gate_up, down
constexpr int MG_MAX_LAYERS = 32;
// static schedule constants shared by the host-side table builder and the kernel (compile-time split counts let every
// partial-sum load of a reduction be issued before the first add)
constexpr int MG_TILE = 64;                                          // output rows per unit of qkv / o / down
constexpr int MG_CPU_QKV = 2, MG_CPU_O = 2;                          // K chunks per unit
constexpr int MG_SPL_QKV = MG_KCH / MG_CPU_QKV;                      // 7
constexpr int MG_SPL_O = MG_KCH / MG_CPU_O;                          // 7
constexpr int MG_SPL_DOWN = 9;                                       // 76 K chunks -> 4 units of 9 + 5 of 8 per row tile

struct MegaUnit { int row0, nrows, kc0, nblk, split; };
struct MegaLayerDev { const float* qkv_bias; const float* ln2; const float* next_gamma; };

struct MegaParams {
  const uint8_t* wstream;
  const unsigned long long* cta_off;   // [G] byte offset of the CTA's stream
  const MegaUnit* units;               // [4][G]
  const MegaLayerDev* layers;          // [L]
  int num_layers, B, max_ctx;
  float* x; bf16* xn; bf16* att; bf16* ffa;
  float *part_qkv, *part_o, *part_down;
  bf16 *kcache, *vcache;
  unsigned long long kv_layer_stride;  // elements
  const int* ctx_len;
  const float* inv_freq;
  unsigned* bar;                       // [0] arrival counter (monotonic), [1] generation base of the next launch
  long long* tl;                       // optional phase timeline (CTA 0)
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok = 0;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  if (ok) return;                       // fast path: no clock reads on the MMA issuers' instruction stream
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
    if (clock64() - t0 > 4000000000ll) break;     // ~2 s: a protocol bug traps instead of hanging the GPU
  }
  __trap();
}
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void worker_bar() { asm volatile("bar.sync 1, %0;" ::"n"(MG_WORKERS) : "memory"); }
__device__ __forceinline__ void epi_bar() { asm volatile("bar.sync 2, 256;" ::: "memory"); }   // the two MMA warpgroups
__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_add(unsigned* p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ long long gtime() {
  long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

template <int BPAD>
__global__ void __launch_bounds__(MG_THREADS, 1)
lm_mega_kernel(const MegaParams p) {
  constexpr int NST = BPAD == 32 ? 16 : 10;
  constexpr uint32_t ACT_CHUNK = BPAD * 128;     // one 64-wide K chunk of the activations: [BPAD rows][128 B], SWIZZLE_128B
  constexpr int STG_LD = 40;                     // SwiGLU staging pitch (bf16): up to 40 channels, rows 8-byte aligned
  static_assert(decode_attn_smem_floats<MG_NW>() * 4 <= MG_KCH * ACT_CHUNK, "attention scratch must fit the activation buffer");
  static_assert(BPAD * STG_LD * 2 <= MG_KCH * ACT_CHUNK, "SwiGLU staging must fit the activation buffer");
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_full[MG_MAX_STAGES];
  __shared__ __align__(8) uint64_t bar_empty[MG_MAX_STAGES];
  __shared__ float red[16];
  __shared__ MegaUnit s_units[MG_PH];
  __shared__ MegaLayerDev s_layers[MG_MAX_LAYERS];

  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* sptr = smem_raw + (sbase - smem_u32(smem_raw));
  const uint32_t ring = sbase, act = sbase + NST * MG_SLOT;
  uint8_t* act_ptr = sptr + NST * MG_SLOT;
  float* attn_sm = reinterpret_cast<float*>(act_ptr);       // aliases the activation buffer (disjoint phases)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int cta = blockIdx.x, G = gridDim.x;
  const int B = p.B;

  if (threadIdx.x == 0) {
    for (int s = 0; s < NST; ++s) {
      mbar_init(smem_u32(&bar_full[s]), 1);
      mbar_init(smem_u32(&bar_empty[s]), 8);     // one arrival per MMA warp (warps 4..11)
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (threadIdx.x >= 64 && threadIdx.x < 64 + MG_PH) s_units[threadIdx.x - 64] = p.units[(threadIdx.x - 64) * G + cta];
  if (threadIdx.x >= 128 && threadIdx.x < 128 + p.num_layers) s_layers[threadIdx.x - 128] = p.layers[threadIdx.x - 128];
  __syncthreads();

  if (warp == 0) {
    // ---------------------------------------------------------------------------------------- weight producer
    if (lane == 0) {
      const uint8_t* src = p.wstream + p.cta_off[cta];
      int it = 0;
      for (int l = 0; l < p.num_layers; ++l)
        for (int ph = 0; ph < MG_PH; ++ph) {
          const int nblk = s_units[ph].nblk;
          const uint32_t bytes = (uint32_t)s_units[ph].nrows * 128u;
          for (int j = 0; j < nblk; ++j, ++it) {
            const int s = it % NST;
            if (it >= NST) mbar_wait(smem_u32(&bar_empty[s]), ((uint32_t)(it / NST) & 1u) ^ 1u);
            if (it >= MG_INFLIGHT) {     // block it - MG_INFLIGHT has landed: bounded burst in front of this SM's latency-critical traffic
              const int itp = it - MG_INFLIGHT;
              mbar_wait(smem_u32(&bar_full[itp % NST]), (uint32_t)(itp / NST) & 1u);
            }
            const uint32_t fb = smem_u32(&bar_full[s]);
            mbar_expect_tx(fb, bytes);
            bulk_load(ring + s * MG_SLOT, src, bytes, fb);
            src += bytes;
          }
        }
    }
    __syncwarp();
  } else {
    // ---------------------------------------------------------------------------------------- workers
    const int wt = threadIdx.x - 32;
    const int ww = warp - 1;
    unsigned bar_target = __ldcg(p.bar + 1);
    const unsigned gen0 = bar_target;
    int mma_it = 0, tl_i = 0;
    const bool stamp = p.tl != nullptr && cta == 0 && wt == 0;
    if (stamp) p.tl[tl_i++] = gtime();
    // fine-grained debug stamps of layer 1: CTA 0 -> tl[512..], CTA 100 -> tl[768..]
    int fs_i = 0;
    bool fs_on = false;
    long long* fs = p.tl ? p.tl + (cta == 0 ? 512 : 768) : nullptr;
    const bool fs_cta = p.tl != nullptr && (cta == 0 || cta == 100) && wt == 0;
#define FS() do { if (fs_cta && fs_on && fs_i < 250) fs[fs_i++] = gtime(); } while (0)

    // grid-wide barrier: every worker's global writes happen-before (bar.sync) the release-add of thread 0; the acquire-load that
    // sees the last arrival happens-before (bar.sync) every worker's following reads (which use ld.global.cg: L2 is the
    // coherence point, stale L1 lines of the previous layer's activations are never consulted)
    auto grid_sync = [&]() {
      bar_target += (unsigned)G;
      FS();
      worker_bar();
      if (wt == 0) {
        red_release_add(p.bar, 1u);
        FS();
        const long long t0 = clock64();
        while ((int)(ld_acquire(p.bar) - bar_target) < 0) {
          if (clock64() - t0 > 4000000000ll) __trap();
        }
        if (stamp) p.tl[tl_i++] = gtime();
        FS();
      }
      worker_bar();
    };

    // one GEMM phase: this CTA's unit = output rows [row0, row0 + nrows) of the weight, K chunks [kc0, kc0 + nblk) of the
    // activation matrix `actg` [B][K] bf16.  mode 0: fp32 partial sums -> out_f32[(split * B + b) * N + n]; mode 1: SwiGLU on
    // interleaved gate/up rows -> ffa
    auto gemm_phase = [&](int ph, const bf16* actg, int K, float* out_f32, int N, int mode) {
      const MegaUnit u = s_units[ph];
      if (u.nblk <= 0) return;
      {
        // activations -> shared memory in the K-major SWIZZLE_128B operand layout (what a TMA box {64, BPAD} would write): row b,
        // 16-byte chunk c of K chunk j at j*ACT_CHUNK + b*128 + ((c ^ (b & 7)) << 4).  All loads of a thread are issued before the
        // first store.  Rows >= B are left as they are: column b of the accumulator depends on row b only and is never stored.
        const int items = u.nblk * B * 8;
        constexpr int UN = 4;
        for (int i0 = wt; i0 < items; i0 += MG_WORKERS * UN) {
          uint4 v[UN];
#pragma unroll
          for (int q = 0; q < UN; ++q) {
            const int i = i0 + q * MG_WORKERS;
            if (i < items) {
              const int c = i & 7, b = (i >> 3) % B, j = (i >> 3) / B;
              v[q] = __ldcg(reinterpret_cast<const uint4*>(actg + (size_t)b * K + (size_t)(u.kc0 + j) * MG_BK) + c);
            }
          }
#pragma unroll
          for (int q = 0; q < UN; ++q) {
            const int i = i0 + q * MG_WORKERS;
            if (i < items) {
              const int c = i & 7, b = (i >> 3) % B, j = (i >> 3) / B;
              *reinterpret_cast<uint4*>(act_ptr + j * ACT_CHUNK + b * 128 + ((c ^ (b & 7)) << 4)) = v[q];
            }
          }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy smem writes -> visible to the MMA (async proxy)
        worker_bar();
        FS();
      }
      if (warp >= 4 && warp < 12) {
        // warpgroup wg: weight rows [64 wg, 64 wg + 64) of every block of the unit (rows past the block belong to the next slot and
        // produce accumulator rows nobody reads); both warpgroups walk every block so each stage sees its 8 warp arrivals
        const int wg = (warp - 4) >> 2, q = lane & 3;
        const bool active = wg * 64 < u.nrows;
        float acc[BPAD / 2];
#pragma unroll
        for (int e = 0; e < BPAD / 2; ++e) acc[e] = 0.f;
        for (int j = 0; j < u.nblk; ++j) {
          const int it = mma_it + j;
          const int s = it % NST;
          mbar_wait(smem_u32(&bar_full[s]), (uint32_t)(it / NST) & 1u);
          if (active) {
            const uint64_t da = wg_desc_sw128(ring + s * MG_SLOT + (uint32_t)wg * 8192u), db = wg_desc_sw128(act + j * ACT_CHUNK);
            wg_fence();
#pragma unroll
            for (int k = 0; k < MG_BK / 16; ++k) wgmma_ss<BPAD, 0>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), 1);
            wg_commit();
            wg_wait<0>();
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(smem_u32(&bar_empty[s]));
        }
        wg_touch<BPAD / 2>(acc);
        bf16* stage = reinterpret_cast<bf16*>(act_ptr);
        if (mode == 1) epi_bar();     // both warpgroups' MMAs have read the activations the staging tile aliases
        if (active) {
          // acc[e]: unit row r = 64 wg + 16 (warp & 3) + lane / 4 + 8 ((e >> 1) & 1), batch row b = 8 (e >> 2) + 2 q + (e & 1)
#pragma unroll
          for (int e = 0; e < BPAD / 2; ++e) {
            const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * ((e >> 1) & 1);
            const int b = 8 * (e >> 2) + 2 * q + (e & 1);
            if (mode == 1) {
              // rows of W are interleaved (2i = gate_i, 2i+1 = up_i): rows r and r + 1 sit in lanes l and l + 4, the even one forms
              // silu(g) * u (Qwen2 MLP act_fn(gate_proj(x)) * up_proj(x)) for channel (row0 + r) / 2 and parks it in the staging
              // tile [b][channel]
              const float other = __shfl_xor_sync(0xffffffffu, acc[e], 4);
              if (!((lane >> 2) & 1) && r < u.nrows && b < B) {
                const float g = acc[e];
                stage[b * STG_LD + (r >> 1)] = __float2bfloat16_rn(__fdividef(g, 1.f + fast_exp(-g)) * other);
              }
            } else if (r < u.nrows && b < B) {
              out_f32[((size_t)u.split * B + b) * N + u.row0 + r] = acc[e];
            }
          }
        }
        if (mode == 1) {
          // staging tile -> ffa[b][row0/2 .. + nrows/2) with 8-byte stores (each row's run is a multiple of 8 bytes, 8-byte aligned)
          epi_bar();
          const int nq = u.nrows >> 3;               // 8-byte chunks per row (4 channels each)
          const int ch0 = u.row0 >> 1;
          for (int i = threadIdx.x - 128; i < B * nq; i += 256) {
            const int b = i / nq, c4 = i % nq;
            *reinterpret_cast<uint2*>(p.ffa + (size_t)b * DFF + ch0 + c4 * 4) = *reinterpret_cast<const uint2*>(stage + b * STG_LD + c4 * 4);
          }
        }
      }
      mma_it += u.nblk;
    };

    // x[b] += sum_s part[s][b]; xn[b] = bf16(gamma * rmsnorm(x[b]))   (one row per CTA; fixed summation order; every load of a
    // thread in flight at once)
    auto reduce_norm = [&](const float* part, auto splits_tag, const float* gamma) {
      constexpr int S = decltype(splits_tag)::value;
      for (int b = cta; b < B; b += G) {
        float ld[2][S + 1];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int n = wt + h * MG_WORKERS;
          const bool ok = n < D;
          ld[h][0] = ok ? __ldcg(p.x + (size_t)b * D + n) : 0.f;
#pragma unroll
          for (int s = 0; s < S; ++s) ld[h][s + 1] = ok ? __ldcg(part + ((size_t)s * B + b) * D + n) : 0.f;
        }
        float v[2], ss = 0.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float a = 0.f;
#pragma unroll
          for (int s = 0; s < S; ++s) a += ld[h][s + 1];
          v[h] = ld[h][0] + a;
          const int n = wt + h * MG_WORKERS;
          if (n < D) {
            p.x[(size_t)b * D + n] = v[h];
            ss += v[h] * v[h];
          }
        }
        ss = warp_sum(ss);
        if (lane == 0) red[ww] = ss;
        FS();
        worker_bar();
        float tot = 0.f;
#pragma unroll
        for (int i = 0; i < MG_NW; ++i) tot += red[i];
        const float r = rsqrtf(tot / D + RMS_EPS);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int n = wt + h * MG_WORKERS;
          if (n < D) p.xn[(size_t)b * D + n] = __float2bfloat16_rn(gamma[n] * (v[h] * r));
        }
        worker_bar();
      }
    };

    for (int l = 0; l < p.num_layers; ++l) {
      const MegaLayerDev Lw = s_layers[l];
      fs_on = l == 1;
      bf16* kc_l = p.kcache + (size_t)l * p.kv_layer_stride;
      bf16* vc_l = p.vcache + (size_t)l * p.kv_layer_stride;
      if (cta < B * NKV && warp >= 8) {
        // this CTA's attention unit of the NEXT phase: pull its K / V rows (one 128-byte line per position) into L2 while the qkv
        // projection runs (the caches of 24 layers x 32 rows do not stay L2-resident between steps)
        const int b = cta / NKV, kvh = cta % NKV;
        const int L = min(p.ctx_len[b], p.max_ctx);
        const bf16* kb = kc_l + ((size_t)b * NKV + kvh) * p.max_ctx * HD;
        const bf16* vb = vc_l + ((size_t)b * NKV + kvh) * p.max_ctx * HD;
        for (int j = threadIdx.x - 256; j < L; j += MG_THREADS - 256) {
          prefetch_l2(kb + (size_t)j * HD);
          prefetch_l2(vb + (size_t)j * HD);
        }
      }
      gemm_phase(0, p.xn, D, p.part_qkv, QKV_N, 0);
      grid_sync();
      for (int u = cta; u < B * NKV; u += G) {
        const int b = u / NKV, kvh = u % NKV;
        bf16* kb = kc_l + ((size_t)b * NKV + kvh) * p.max_ctx * HD;
        bf16* vb = vc_l + ((size_t)b * NKV + kvh) * p.max_ctx * HD;
        KvFrag fr;
        decode_attn_unit<MG_NW, 1, MG_SPL_QKV>(attn_sm, wt, p.part_qkv, MG_SPL_QKV, B, b, kvh, Lw.qkv_bias, kb, vb, p.ctx_len[b], p.max_ctx,
                                               p.inv_freq, p.att + (size_t)b * D, fr, false);
        worker_bar();
      }
      grid_sync();
      gemm_phase(1, p.att, D, p.part_o, D, 0);
      grid_sync();
      reduce_norm(p.part_o, std::integral_constant<int, MG_SPL_O>(), Lw.ln2);
      grid_sync();
      gemm_phase(2, p.xn, D, nullptr, 2 * DFF, 1);
      grid_sync();
      gemm_phase(3, p.ffa, DFF, p.part_down, D, 0);
      grid_sync();
      reduce_norm(p.part_down, std::integral_constant<int, MG_SPL_DOWN>(), Lw.next_gamma);
      if (l + 1 < p.num_layers) grid_sync();
    }
    if (cta == 0 && wt == 0) {
      p.bar[1] = gen0 + (unsigned)G * (unsigned)(7 * p.num_layers - 1);    // generation base of the next launch
      if (stamp) p.tl[tl_i++] = gtime();
    }
  }
}

// one weight block: rows [row0, row0 + nrows) x K chunk kc of W [N][K] bf16 row-major -> the shared-memory image of a K-major
// SWIZZLE_128B operand tile (row r, 16-byte chunk c at r*128 + ((c ^ (r & 7)) << 4)); nrows*128 contiguous bytes in the stream
struct PackDesc { const bf16* w; int K, row0, nrows, kc; unsigned long long dst; };
__global__ void pack_blocks_kernel(const PackDesc* __restrict__ descs, int n, uint8_t* __restrict__ out) {
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    const PackDesc d = descs[i];
    for (int e = threadIdx.x; e < d.nrows * 8; e += blockDim.x) {
      const int r = e >> 3, c = e & 7;
      const uint4 v = *reinterpret_cast<const uint4*>(d.w + (size_t)(d.row0 + r) * d.K + (size_t)d.kc * MG_BK + c * 8);
      *reinterpret_cast<uint4*>(out + d.dst + r * 128 + ((c ^ (r & 7)) << 4)) = v;
    }
  }
}

template <int BPAD> constexpr size_t mega_smem() { return (size_t)(BPAD == 32 ? 16 : 10) * MG_SLOT + (size_t)MG_KCH * BPAD * 128 + 1024; }

}  // namespace

struct LmMega {
  int G = 0;
  int splits[MG_PH] = {0, 0, 0, 0};
  uint8_t* wstream = nullptr;
  unsigned long long* cta_off = nullptr;
  MegaUnit* units = nullptr;
  MegaLayerDev* layers = nullptr;
  size_t stream_bytes = 0;
};

struct MegaSession {
  float *part_qkv = nullptr, *part_o = nullptr, *part_down = nullptr;
  unsigned* bar = nullptr;
};

void lm_mega_build(cvk_ctx* ctx, LlmModel* m) {
  const int G = ctx->num_sms, L = m->num_layers;
  if (L > MG_MAX_LAYERS) return;
  // static schedule (identical for every layer): which output rows x K range of each projection a CTA owns.  Row-granular cuts
  // spread every projection over (nearly) all CTAs with about equal bytes, so no unit exceeds the ring and the aggregate HBM
  // stream is balanced; K splits (partial sums) only where the output is narrow (qkv 1152, o / down 896 rows).
  std::vector<MegaUnit> units((size_t)MG_PH * G, MegaUnit{0, 0, 0, 0, 0});
  auto put = [&](int ph, int c, MegaUnit u) {
    c = ((c % G) + G) % G;
    CVK_REQUIRE(units[(size_t)ph * G + c].nblk == 0, "lm mega: two units on one CTA in a phase");
    units[(size_t)ph * G + c] = u;
  };
  const int qkv_tiles = QKV_N / MG_TILE, o_tiles = D / MG_TILE, down_chunks = DFF / MG_BK;
  if (qkv_tiles * MG_SPL_QKV > G || o_tiles * MG_SPL_O > G || o_tiles * MG_SPL_DOWN > G) return;      // fewer SMs than the schedule assumes
  for (int t = 0; t < qkv_tiles; ++t)
    for (int s = 0; s < MG_SPL_QKV; ++s) put(0, t * MG_SPL_QKV + s, MegaUnit{t * MG_TILE, MG_TILE, s * MG_CPU_QKV, MG_CPU_QKV, s});
  for (int t = 0; t < o_tiles; ++t)
    for (int s = 0; s < MG_SPL_O; ++s) put(1, G - o_tiles * MG_SPL_O + t * MG_SPL_O + s, MegaUnit{t * MG_TILE, MG_TILE, s * MG_CPU_O, MG_CPU_O, s});
  {
    // gate|up (interleaved rows, whole K, SwiGLU in the epilogue): 9728 rows in groups of 8 dealt over all CTAs
    const int groups = 2 * DFF / 8, base = groups / G, extra = groups % G;
    if ((base + (extra ? 1 : 0)) * 8 > MG_MAXROWS || base < 1) return;
    int row = 0;
    for (int c = 0; c < G; ++c) {
      const int nr = (base + (c < extra ? 1 : 0)) * 8;
      put(2, c, MegaUnit{row, nr, 0, MG_KCH, 0});
      row += nr;
    }
  }
  {
    const int base = down_chunks / MG_SPL_DOWN, extra = down_chunks % MG_SPL_DOWN;       // 7, 6
    for (int t = 0; t < o_tiles; ++t) {
      int kc = 0;
      for (int s = 0; s < MG_SPL_DOWN; ++s) {
        const int nb = base + (s < extra ? 1 : 0);
        put(3, t * MG_SPL_DOWN + s, MegaUnit{t * MG_TILE, MG_TILE, kc, nb, s});
        kc += nb;
      }
    }
  }
  LmMega* mg = new LmMega();
  mg->G = G;
  mg->splits[0] = MG_SPL_QKV; mg->splits[1] = MG_SPL_O; mg->splits[2] = 1; mg->splits[3] = MG_SPL_DOWN;
  std::vector<unsigned> lbytes(G, 0);
  std::vector<unsigned long long> off(G, 0);
  size_t total = 0;
  for (int c = 0; c < G; ++c) {
    for (int ph = 0; ph < MG_PH; ++ph) lbytes[c] += (unsigned)(units[(size_t)ph * G + c].nblk * units[(size_t)ph * G + c].nrows * 128);
    off[c] = total;
    total += (size_t)lbytes[c] * L;
  }
  mg->stream_bytes = total;
  mg->wstream = (uint8_t*)ctx->dmalloc(total);
  std::vector<PackDesc> descs;
  for (int c = 0; c < G; ++c)
    for (int l = 0; l < L; ++l) {
      const LayerW& w = m->layers[l];
      const ConvW* Ws[MG_PH] = {&w.qkv, &w.o, &w.gate_up_il, &w.down};
      unsigned long long dst = off[c] + (unsigned long long)l * lbytes[c];
      for (int ph = 0; ph < MG_PH; ++ph) {
        const MegaUnit& u = units[(size_t)ph * G + c];
        CVK_REQUIRE(u.nblk == 0 || (Ws[ph]->w16 && u.row0 + u.nrows <= Ws[ph]->N && (u.kc0 + u.nblk) * MG_BK <= Ws[ph]->K), "lm mega: unit outside its weight");
        for (int j = 0; j < u.nblk; ++j) {
          descs.push_back(PackDesc{Ws[ph]->w16, Ws[ph]->K, u.row0, u.nrows, u.kc0 + j, dst});
          dst += (unsigned long long)u.nrows * 128;
        }
      }
    }
  {
    PackDesc* dd = nullptr;
    CVK_CHECK_CUDA(cudaMalloc((void**)&dd, descs.size() * sizeof(PackDesc)));
    CVK_CHECK_CUDA(cudaMemcpy(dd, descs.data(), descs.size() * sizeof(PackDesc), cudaMemcpyHostToDevice));
    pack_blocks_kernel<<<G * 8, 256>>>(dd, (int)descs.size(), mg->wstream);
    CVK_LAUNCH_CHECK();
    CVK_CHECK_CUDA(cudaDeviceSynchronize());
    cudaFree(dd);
  }
  std::vector<MegaLayerDev> lay(L);
  for (int l = 0; l < L; ++l) {
    lay[l].qkv_bias = m->layers[l].qkv.bias;
    lay[l].ln2 = m->layers[l].ln2;
    lay[l].next_gamma = l + 1 < L ? m->layers[l + 1].ln1 : m->final_norm;
  }
  auto up = [&](const void* h, size_t bytes) {
    void* d = ctx->dmalloc(bytes);
    CVK_CHECK_CUDA(cudaMemcpy(d, h, bytes, cudaMemcpyHostToDevice));
    return d;
  };
  mg->cta_off = (unsigned long long*)up(off.data(), off.size() * sizeof(unsigned long long));
  mg->units = (MegaUnit*)up(units.data(), units.size() * sizeof(MegaUnit));
  mg->layers = (MegaLayerDev*)up(lay.data(), lay.size() * sizeof(MegaLayerDev));
  CVK_CHECK_CUDA(cudaFuncSetAttribute(lm_mega_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)mega_smem<32>()));
  CVK_CHECK_CUDA(cudaFuncSetAttribute(lm_mega_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)mega_smem<64>()));
  m->mega = mg;
}

bool lm_mega_usable(cvk_ctx* ctx, const cvk_lm_session* s, int B) {
  return ctx->lm_mega && ctx->llm && ctx->llm->mega && s->kv_dtype == DT_BF16 && ctx->use_tc && B >= 1 && B <= 64 && s->mega_state;
}

void lm_mega_session_init(cvk_ctx* ctx, cvk_lm_session* s) {
  const LmMega* mg = ctx->llm ? ctx->llm->mega : nullptr;
  if (!mg || s->kv_dtype != DT_BF16 || s->max_batch > 64) return;
  MegaSession* ms = new MegaSession();
  auto alloc = [&](size_t bytes) {
    void* p = nullptr;
    CVK_CHECK_CUDA(cudaMalloc(&p, bytes));
    CVK_CHECK_CUDA(cudaMemset(p, 0, bytes));
    s->owned.push_back(p);
    return p;
  };
  ms->part_qkv = (float*)alloc((size_t)mg->splits[0] * s->max_batch * QKV_N * sizeof(float));
  ms->part_o = (float*)alloc((size_t)mg->splits[1] * s->max_batch * D * sizeof(float));
  ms->part_down = (float*)alloc((size_t)mg->splits[3] * s->max_batch * D * sizeof(float));
  ms->bar = (unsigned*)alloc(64);
  s->mega_state = ms;
}

void lm_mega_session_free(cvk_lm_session* s) {
  delete (MegaSession*)s->mega_state;
  s->mega_state = nullptr;
}

void lm_mega_layers(cvk_ctx* ctx, cudaStream_t st, cvk_lm_session* s, int B) {
  const LlmModel* m = ctx->llm;
  const LmMega* mg = m->mega;
  const MegaSession* ms = (const MegaSession*)s->mega_state;
  CVK_REQUIRE(mg && ms && B >= 1 && B <= 64 && m->num_layers <= MG_MAX_LAYERS, "lm mega: not initialised");
  const int bpad = B <= 32 ? 32 : 64;
  MegaParams p;
  p.wstream = mg->wstream; p.cta_off = mg->cta_off; p.units = mg->units; p.layers = mg->layers;
  p.num_layers = m->num_layers; p.B = B; p.max_ctx = s->max_ctx;
  p.x = s->x; p.xn = (bf16*)s->xn; p.att = (bf16*)s->att; p.ffa = (bf16*)s->ffa;
  p.part_qkv = ms->part_qkv; p.part_o = ms->part_o; p.part_down = ms->part_down;
  p.kcache = (bf16*)s->kcache; p.vcache = (bf16*)s->vcache;
  p.kv_layer_stride = (unsigned long long)s->max_batch * NKV * s->max_ctx * HD;
  p.ctx_len = s->ctx_len; p.inv_freq = m->d_inv_freq;
  p.bar = ms->bar;
  p.tl = ctx->tl ? (long long*)ctx->tl + 2048 : nullptr;   // second half of the chain-timeline buffer
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(mg->G);
  cfg.blockDim = dim3(MG_THREADS);
  cfg.dynamicSmemBytes = bpad == 32 ? mega_smem<32>() : mega_smem<64>();
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeCooperative;     // all CTAs co-resident: the grid barriers cannot deadlock against other work
  at[0].val.cooperative = 1;
  cfg.attrs = at;
  cfg.numAttrs = ctx->mega_coop ? 1 : 0;
  if (bpad == 32) CVK_CHECK_CUDA(cudaLaunchKernelEx(&cfg, lm_mega_kernel<32>, p));
  else CVK_CHECK_CUDA(cudaLaunchKernelEx(&cfg, lm_mega_kernel<64>, p));
  ctx->launches++;
}
