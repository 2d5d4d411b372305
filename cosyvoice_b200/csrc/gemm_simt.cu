// fp32 CUDA-core conv-GEMM: the parity path (CVK_PREC_FP32) and the kernel for the precision-critical layers
// (f0 predictor, mel DFT) in every mode; with use_tc = 0 it also takes the bf16 / fp16 operands of the tensor-core mode.
//
//   out[r, n] = epilogue( sum_{j<taps} sum_{k<K} A[r + shift0 + j*dil, k] * W[n][j][k] )
//
// A is a time-major activation matrix whose gap rows hold zeros, so a Conv1d / CausalConv1d / polyphase
// ConvTranspose1d over ragged sequences is this one kernel with different (taps, dil, shift0)
// (reference ops: flow/decoder.py:36-62 CausalConv1d, hifigan/generator.py:110-117 ResBlock convs, :432-443 ups).
#include "common.cuh"

namespace {

constexpr int BM = 64, BN = 64, BK = 16, TM = 4, TN = 4;

template <typename TA, typename TW>
__global__ void __launch_bounds__(256) conv_gemm_simt_kernel(const TA* __restrict__ A, int lda, int rowsA, const TW* __restrict__ W,
                                                             int N, int K, int taps, int dil, int shift0, int rowsOut, EpiDev ep) {
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid % 16, ty = tid / 16;
  const int r0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int Kt = taps * K;
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < Kt; k0 += BK) {
    // A tile: 64 rows x 16 k ; thread -> (row = tid/4, 4 consecutive k)
    {
      int row = tid >> 2, kq = (tid & 3) * 4;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        int kk = k0 + kq + q;
        float v = 0.f;
        if (kk < Kt) {
          int j = kk / K, k = kk - j * K;
          int rs = r0 + row + shift0 + j * dil;
          if (rs >= 0 && rs < rowsA) v = to_f32(A[(size_t)rs * lda + k]);
        }
        As[kq + q][row] = v;
      }
    }
    {
      int col = tid >> 2, kq = (tid & 3) * 4;
      int n = n0 + col;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        int kk = k0 + kq + q;
        float v = 0.f;
        if (kk < Kt && n < N) v = to_f32(W[(size_t)n * Kt + kk]);
        Bs[kq + q][col] = v;
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; ++i) a[i] = As[k][ty * TM + i];
#pragma unroll
      for (int j = 0; j < TN; ++j) b[j] = Bs[k][tx * TN + j];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int r = r0 + ty * TM + i;
    if (r >= rowsOut) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int n = n0 + tx * TN + j;
      if (n < N) epi_store(ep, r, n, acc[i][j]);
    }
  }
}

}  // namespace

void conv_gemm_simt(cvk_ctx* ctx, cudaStream_t st, const Mat& A, const ConvW& W, const Epilogue& ep) {
  CVK_REQUIRE(A.cols >= W.K, "conv_gemm: A has fewer columns than the weight's K");
  CVK_REQUIRE(ep.out.p != nullptr && ep.out.cols >= W.N, "conv_gemm: bad output");
  int rowsOut = ep.out.rows;
  dim3 grid(ceil_div(W.N, BN), ceil_div(rowsOut, BM));
  EpiDev e = to_dev(ep);
  if (!e.bias) e.bias = W.bias;
  ProfScope ps(ctx, st, FAM_GEMM_SIMT, 2.0 * rowsOut * (double)W.N * W.K * W.taps,
               (double)rowsOut * W.K * A.esize() + (double)W.N * W.K * W.taps * 4 + (double)rowsOut * W.N * ep.out.esize());
  if (A.dtype == DT_F32) {
    conv_gemm_simt_kernel<float, float><<<grid, 256, 0, st>>>(A.f32(), A.ld, A.rows, W.w32, W.N, W.K, W.taps, W.dil, W.shift0,
                                                              rowsOut, e);
  } else if (A.dtype == DT_F16) {
    // the vocoder's IEEE-half operands (use_tc = 0 in a bf16 context): its weights carry only the half copy
    CVK_REQUIRE(W.wf16 != nullptr, "conv_gemm: fp16 operand but no fp16 weights");
    conv_gemm_simt_kernel<__half, __half><<<grid, 256, 0, st>>>((const __half*)A.p, A.ld, A.rows, W.wf16, W.N, W.K, W.taps, W.dil,
                                                                W.shift0, rowsOut, e);
  } else {
    CVK_REQUIRE(W.w16 != nullptr, "conv_gemm: bf16 operand but no bf16 weights");
    conv_gemm_simt_kernel<bf16, bf16><<<grid, 256, 0, st>>>(A.b16(), A.ld, A.rows, W.w16, W.N, W.K, W.taps, W.dil, W.shift0,
                                                            rowsOut, e);
  }
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}

void conv_gemm(cvk_ctx* ctx, cudaStream_t st, const Mat& A, const ConvW& W, const Epilogue& ep) {
  if (A.dtype != DT_F32 && ctx->use_tc) conv_gemm_tc(ctx, st, A, W, ep);
  else conv_gemm_simt(ctx, st, A, W, ep);
}
