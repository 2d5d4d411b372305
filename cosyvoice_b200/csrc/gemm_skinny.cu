// Weight-streaming GEMM for the LM decode step (at most 64 activation rows): out[b, n] = sum_k x[b, k] * W[n, k].
//
// The step is HBM-bound on the weights (SURVEY.md §8d: 727.6 MB of bf16 weights per step shared by all rows), so the
// kernel is organised around memory-level parallelism, not MMA rate: operands are swapped (the wgmma M side holds 128 output
// features of W, 64 per warpgroup, the wgmma N dimension holds the <= 64 batch rows), K is split across CTAs so that ~all SMs
// stream disjoint weight slabs, and each CTA keeps 8 TMA stages (160 / 192 KB) in flight.  fp32 accumulation in registers;
// split-K partial sums go to a [splits][rows][N] scratch and are reduced in fixed order by a finishing kernel that
// applies the same fused epilogue as the big GEMM (deterministic - no atomics).
// Serves transformers' Qwen2 q/k/v/o/gate/up/down projections and the llm_decoder head at decode time
// (cosyvoice/llm/llm.py:244-251, 542).
#include "common.cuh"
#include "wgmma.cuh"
#include "tma.cuh"

namespace {

constexpr int SK_BM = 128;      // output features per CTA (wgmma M of two warpgroups)
constexpr int SK_BK = 64;
constexpr int SK_STAGES = 8;
constexpr int SK_THREADS = 384;   // warp 0: TMA producer; warpgroups 1-2: wgmma + epilogue, 64 features each

// W [N][K] bf16 row-major -> streaming layout: [N/128 tiles][K/64 chunks] blocks of 16 KB, each block being the exact
// shared-memory image of a K-major SWIZZLE_128B operand tile (row r, 16-byte chunk c stored at r*128 + ((c ^ (r & 7)) << 4)),
// so that one stage is ONE contiguous 16 KB bulk copy: DRAM sees perfectly sequential reads instead of 128 strided rows.
__global__ void tile_weights_kernel(const bf16* __restrict__ w, bf16* __restrict__ out, int N, int K, int tiles, int kchunks) {
  size_t total = (size_t)tiles * kchunks * SK_BM * 8;     // 16-byte chunks
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int c = i & 7;
    int r = (i >> 3) & (SK_BM - 1);
    size_t blk = i >> 10;
    int kc = blk % kchunks, nt = blk / kchunks;
    int n = nt * SK_BM + r, k = kc * SK_BK + c * 8;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (n < N && k + 8 <= K) v = *reinterpret_cast<const uint4*>(w + (size_t)n * K + k);
    else if (n < N && k < K) {
      __align__(16) bf16 t[8];
      for (int e = 0; e < 8; ++e) t[e] = k + e < K ? w[(size_t)n * K + k + e] : __float2bfloat16_rn(0.f);
      v = *reinterpret_cast<uint4*>(t);
    }
    *reinterpret_cast<uint4*>(reinterpret_cast<char*>(out) + blk * (SK_BM * SK_BK * 2) + r * 128 + ((c ^ (r & 7)) << 4)) = v;
  }
}

// grid: (N tiles, splits).  BPAD = padded batch (wgmma N): 32 or 64.  Warp 0 streams the stages; warpgroups 1 and 2 each
// accumulate 64 of the tile's 128 output features over the CTA's K chunks (fp32 in registers) and run the epilogue on them.
template <int BPAD>
__global__ void __launch_bounds__(SK_THREADS, 1)
skinny_gemm_kernel(const bf16* __restrict__ w_tiled, const __grid_constant__ CUtensorMap tmap_x, int N, int K, int rows,
                   int chunks_per_split, float* __restrict__ partial /*[splits][rows][N] or null*/, EpiDev ep, int swiglu,
                   long long* __restrict__ tl) {
  extern __shared__ uint8_t smem_raw[];
  pdl_trigger();
  tl_stamp(tl, 0);
  __shared__ __align__(8) uint64_t bar_full[SK_STAGES];
  __shared__ __align__(8) uint64_t bar_empty[SK_STAGES];
  constexpr uint32_t A_BYTES = SK_BM * SK_BK * 2;    // 16 KB of weights
  constexpr uint32_t B_BYTES = BPAD * SK_BK * 2;     // activations
  constexpr uint32_t STAGE = A_BYTES + B_BYTES;

  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * SK_BM;
  const int kchunks = (K + SK_BK - 1) / SK_BK;
  const int kc0 = blockIdx.y * chunks_per_split;
  const int kc1 = min(kchunks, kc0 + chunks_per_split);
  const int iters = kc1 - kc0;    // >= 1 by construction of the launch

  if (threadIdx.x == 0) {
    for (int s = 0; s < SK_STAGES; ++s) {
      mbar_init(smem_u32(&bar_full[s]), 1);
      mbar_init(smem_u32(&bar_empty[s]), 8);     // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    if (warp == 0 && lane == 0) {
      // The weights are written by no kernel of the chain: the first ring of weight slabs is requested BEFORE waiting for the
      // producer of the activations, so the HBM stream of this kernel overlaps the tail of the previous one.
      const int pre = min(iters, SK_STAGES);
      for (int it = 0; it < pre; ++it) {
        const uint32_t fb = smem_u32(&bar_full[it]);
        mbar_expect_tx(fb, STAGE);
        bulk_load(base + it * STAGE, w_tiled + ((size_t)blockIdx.x * kchunks + (kc0 + it)) * (SK_BM * SK_BK), A_BYTES, fb);
      }
      pdl_wait();
      tl_stamp(tl, 1);
      for (int it = 0; it < pre; ++it) tma_load_2d(base + it * STAGE + A_BYTES, &tmap_x, smem_u32(&bar_full[it]), (kc0 + it) * SK_BK, 0);
      for (int it = pre; it < iters; ++it) {
        const int s = it % SK_STAGES;
        const uint32_t round = (uint32_t)(it / SK_STAGES);
        mbar_wait(smem_u32(&bar_empty[s]), (round & 1u) ^ 1u);
        const uint32_t sa = base + s * STAGE, sb = sa + A_BYTES;
        const uint32_t fb = smem_u32(&bar_full[s]);
        mbar_expect_tx(fb, STAGE);
        bulk_load(sa, w_tiled + ((size_t)blockIdx.x * kchunks + (kc0 + it)) * (SK_BM * SK_BK), A_BYTES, fb);
        tma_load_2d(sb, &tmap_x, fb, (kc0 + it) * SK_BK, 0);
      }
    } else {
      pdl_wait();
    }
  } else {
    const int wg = (threadIdx.x - 128) >> 7;
    const int q = lane & 3;
    const int fr = wg * 64 + (warp & 3) * 16 + (lane >> 2);    // tile features fr (acc[4 j + 0/1]) and fr + 8 (acc[4 j + 2/3])
    float bias_n[2];                                           // fetched while the weights stream
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) bias_n[hh] = (!partial && !swiglu && ep.bias && n0 + fr + 8 * hh < N) ? ep.bias[n0 + fr + 8 * hh] : 0.f;
    pdl_wait();
    float acc[BPAD / 2];
#pragma unroll
    for (int e = 0; e < BPAD / 2; ++e) acc[e] = 0.f;
    for (int it = 0; it < iters; ++it) {
      const int s = it % SK_STAGES;
      mbar_wait(smem_u32(&bar_full[s]), (uint32_t)(it / SK_STAGES) & 1u);
      const uint32_t sa = base + s * STAGE + (uint32_t)wg * (A_BYTES / 2), sb = base + s * STAGE + A_BYTES;
      const uint64_t da = wg_desc_sw128(sa), db = wg_desc_sw128(sb);
      wg_fence();
#pragma unroll
      for (int k = 0; k < SK_BK / 16; ++k) wgmma_ss<BPAD, 0>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), 1);
      wg_commit();
      wg_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&bar_empty[s]));
    }
    wg_touch<BPAD / 2>(acc);
    const bool plain = ep.act1 == ACT_NONE && !ep.resid && !ep.rowvec && !ep.row2seq && !ep.accumulate && !ep.out2 && ep.scale == 1.f;
    // acc[e]: feature n0 + fr + 8 ((e >> 1) & 1), batch row 8 (e >> 2) + 2 q + (e & 1)
#pragma unroll
    for (int e = 0; e < BPAD / 2; ++e) {
      const int hh = (e >> 1) & 1;
      const int n = n0 + fr + 8 * hh, b = 8 * (e >> 2) + 2 * q + (e & 1);
      if (swiglu) {
        // rows of W are interleaved (2i = gate_i, 2i+1 = up_i): features n and n + 1 sit in lanes l and l + 4, the even one emits
        // silu(g) * u (Qwen2 MLP act_fn(gate_proj(x)) * up_proj(x), modeling_qwen2.py:46-48) into column n/2
        const float other = __shfl_xor_sync(0xffffffffu, acc[e], 4);
        if (!((lane >> 2) & 1) && n + 1 < N && b < rows) {
          const float g = acc[e];
          st_any(ep.out, ep.out_dtype, (size_t)b * ep.out_ld + (n >> 1), __fdividef(g, 1.f + fast_exp(-g)) * other);
        }
      } else if (n < N && b < rows) {
        if (partial) partial[((size_t)blockIdx.y * rows + b) * N + n] = acc[e];
        else if (plain) st_any(ep.out, ep.out_dtype, (size_t)b * ep.out_ld + n, acc[e] + bias_n[hh]);   // plain Linear (+bias): no loads in the store loop
        else epi_store(ep, b, n, acc[e]);
      }
    }
  }
  tl_stamp(tl, 2);
}

// out = epilogue(sum_s partial[s]) in fixed split order
__global__ void splitk_finish_kernel(const float* __restrict__ partial, int splits, int rows, int N, EpiDev ep, long long* __restrict__ tl) {
  pdl_trigger();
  tl_stamp(tl, 0);
  pdl_wait();
  tl_stamp(tl, 1);
  size_t total = (size_t)rows * N;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int s = 0; s < splits; ++s) acc += partial[(size_t)s * total + i];
    epi_store(ep, (int)(i / N), (int)(i % N), acc);
  }
  tl_stamp(tl, 2);
}

template <int BPAD>
constexpr size_t skinny_smem() {
  return (size_t)SK_STAGES * (SK_BM * SK_BK * 2 + BPAD * SK_BK * 2) + 1024;
}

template <int BPAD>
void launch(cudaStream_t st, dim3 grid, const bf16* tw, const CUtensorMap& tx, const ConvW& W, int rows, int cps, float* partial,
            const EpiDev& e, int swiglu, bool pdl, long long* tl) {
  launch_ex(skinny_gemm_kernel<BPAD>, grid, dim3(SK_THREADS), skinny_smem<BPAD>(), st, pdl, tw, tx, W.N, W.K, rows, cps, partial, e, swiglu, tl);
}

}  // namespace

// streaming-layout copy of a Linear weight, created once (llm_build calls this for every decode-time weight; creating it
// lazily inside a CUDA-graph capture would be illegal)
const bf16* skinny_tiled_weights(cvk_ctx* ctx, const ConvW& W) {
  auto it = ctx->tiled.find(W.w16);
  if (it != ctx->tiled.end()) return (const bf16*)it->second;
  CVK_REQUIRE(!cvk_in_capture, "skinny_tiled_weights: weight was not pre-tiled before graph capture");
  const int tiles = ceil_div(W.N, SK_BM), kchunks = ceil_div(W.K, SK_BK);
  bf16* out = (bf16*)ctx->dmalloc((size_t)tiles * kchunks * SK_BM * SK_BK * sizeof(bf16));
  tile_weights_kernel<<<ctx->num_sms * 8, 256>>>(W.w16, out, W.N, W.K, tiles, kchunks);
  CVK_LAUNCH_CHECK();
  CVK_CHECK_CUDA(cudaDeviceSynchronize());
  ctx->tiled[W.w16] = out;
  return out;
}

// scratch: device buffer of at least skinny_scratch_floats() floats, owned by the caller (LM session: stable across graph replays)
size_t skinny_scratch_floats(int rows, int maxN) { return (size_t)32 * rows * maxN; }

// mode 0: fused epilogue (split-K reduced by splitk_finish_kernel); mode 1: leave the split-K partial sums [splits][rows][N]
// in `scratch` for a fused consumer (returns the split count); mode 2: no split, SwiGLU epilogue on interleaved gate/up rows
int conv_gemm_skinny_ex(cvk_ctx* ctx, cudaStream_t st, const Mat& A, const ConvW& W, const Epilogue& ep, float* scratch, size_t scratch_floats,
                        int mode) {
  CVK_REQUIRE(A.dtype == DT_BF16 && W.w16 != nullptr && W.taps == 1, "conv_gemm_skinny: bf16 1-tap operands required");
  const int rows = mode == 1 ? A.rows : ep.out.rows;
  CVK_REQUIRE(rows <= 64 && A.rows >= rows, "conv_gemm_skinny: at most 64 rows");
  CVK_REQUIRE(W.K % 8 == 0 && A.ld % 8 == 0 && ((uintptr_t)A.p & 15) == 0, "conv_gemm_skinny: 16-byte aligned operands required");
  const int BPAD = rows <= 32 ? 32 : 64;
  CUtensorMap tx;
  const bf16* tw = skinny_tiled_weights(ctx, W);
  {
    const cuuint64_t dims[2] = {(cuuint64_t)W.K, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)A.ld * 2};
    const cuuint32_t box[2] = {SK_BK, (cuuint32_t)BPAD};
    encode_tma_map(ctx, &tx, A.p, 2, dims, strides, box, DT_BF16, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "skinny x");
  }
  const int tiles = ceil_div(W.N, SK_BM);
  const int kchunks = ceil_div(W.K, SK_BK);
  int splits = ctx->num_sms / tiles;
  if (splits > kchunks / 4) splits = kchunks / 4;   // at least 4 K chunks (64 KB of weights) per CTA
  if (splits > 32) splits = 32;
  if (splits < 1) splits = 1;
  int cps = ceil_div(kchunks, splits);
  splits = ceil_div(kchunks, cps);                   // no empty split
  if (mode == 2 || (splits > 1 && (scratch == nullptr || (size_t)splits * rows * W.N > scratch_floats))) {
    splits = 1;
    cps = kchunks;
  }
  CVK_REQUIRE(mode != 1 || (scratch != nullptr && (size_t)splits * rows * W.N <= scratch_floats), "conv_gemm_skinny: scratch too small");
  EpiDev e = to_dev(ep);
  if (!e.bias) e.bias = W.bias;
  const double flops = 2.0 * rows * (double)W.N * W.K;
  const double bytes = (double)W.N * W.K * 2 + (double)rows * W.K * 2 + (double)rows * W.N * 2;
  ProfScope ps(ctx, st, FAM_GEMM_TC, flops, bytes);
  dim3 grid(tiles, splits);
  float* partial = (splits > 1 || mode == 1) ? scratch : nullptr;
  long long* tl = ctx->tl_next();
  if (BPAD == 32) launch<32>(st, grid, tw, tx, W, rows, cps, partial, e, mode == 2, ctx->pdl != 0, tl);
  else launch<64>(st, grid, tw, tx, W, rows, cps, partial, e, mode == 2, ctx->pdl != 0, tl);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  if (splits > 1 && mode == 0) {
    size_t total = (size_t)rows * W.N;
    int g = (int)((total + 255) / 256);
    if (g > ctx->num_sms * 4) g = ctx->num_sms * 4;
    launch_ex(splitk_finish_kernel, dim3(g), dim3(256), 0, st, ctx->pdl != 0, (const float*)partial, splits, rows, W.N, e, ctx->tl_next());
    ctx->launches++;
    CVK_LAUNCH_CHECK();
  }
  return splits;
}

void conv_gemm_skinny(cvk_ctx* ctx, cudaStream_t st, const Mat& A, const ConvW& W, const Epilogue& ep, float* scratch, size_t scratch_floats) {
  conv_gemm_skinny_ex(ctx, st, A, W, ep, scratch, scratch_floats, 0);
}

// dynamic shared memory of both batch widths, and the maximum shared-memory carveout that every kernel of the LM decode chain
// keeps (see llm_session_create)
void skinny_setup() {
  CVK_CHECK_CUDA(cudaFuncSetAttribute(skinny_gemm_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)skinny_smem<32>()));
  CVK_CHECK_CUDA(cudaFuncSetAttribute(skinny_gemm_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)skinny_smem<64>()));
  CVK_CHECK_CUDA(cudaFuncSetAttribute(skinny_gemm_kernel<32>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  CVK_CHECK_CUDA(cudaFuncSetAttribute(skinny_gemm_kernel<64>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  CVK_CHECK_CUDA(cudaFuncSetAttribute(splitk_finish_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
}
