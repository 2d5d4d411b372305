// Geometry, weight repacking and the HBM-bound elementwise / normalisation kernels.
#include "common.cuh"

// ================================================================================================ geometry
namespace {
__global__ void fill_row2seq_kernel(const int* __restrict__ start, const int* __restrict__ len, int B, int* __restrict__ row2seq) {
  int b = blockIdx.y;
  int s = start[b], l = len[b];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < l; i += gridDim.x * blockDim.x) row2seq[s + i] = b;
}
}  // namespace

static void upload_seqs(cvk_ctx* ctx, Seqs& s, cudaStream_t st, bool with_row2seq) {
  s.d_start = (int*)ctx->arena.alloc(sizeof(int) * s.B);
  s.d_len = (int*)ctx->arena.alloc(sizeof(int) * s.B);
  CVK_CHECK_CUDA(cudaMemcpyAsync(s.d_start, s.start.data(), sizeof(int) * s.B, cudaMemcpyHostToDevice, st));
  CVK_CHECK_CUDA(cudaMemcpyAsync(s.d_len, s.len.data(), sizeof(int) * s.B, cudaMemcpyHostToDevice, st));
  if (!with_row2seq) return;
  s.d_row2seq = (int*)ctx->arena.alloc(sizeof(int) * (size_t)s.R);
  CVK_CHECK_CUDA(cudaMemsetAsync(s.d_row2seq, 0xFF, sizeof(int) * (size_t)s.R, st));
  int bx = ceil_div(s.max_len, 256);
  if (bx > 64) bx = 64;
  if (bx < 1) bx = 1;
  fill_row2seq_kernel<<<dim3(bx, s.B), 256, 0, st>>>(s.d_start, s.d_len, s.B, s.d_row2seq);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}

// lens: host lengths at the base rate.  Rows: [gap][seq0][gap][seq1]...[gap], total rounded up to 128.
// scale multiplies every coordinate (HiFT up-sampling levels); extra_front prepends rows to every sequence
// (the ReflectionPad1d((1,0)) sample of the last HiFT stage, generator.py:516-517).
Seqs make_seqs(cvk_ctx* ctx, const int* lens, int B, int gap, int scale, int extra_front, cudaStream_t st, bool with_row2seq) {
  CVK_REQUIRE(B > 0, "empty batch");
  Seqs s;
  s.B = B;
  s.start.resize(B);
  s.len.resize(B);
  int pos = gap;
  for (int b = 0; b < B; ++b) {
    CVK_REQUIRE(lens[b] > 0, "sequence of length 0");
    s.start[b] = pos * scale - extra_front;
    s.len[b] = lens[b] * scale + extra_front;
    if (s.len[b] > s.max_len) s.max_len = s.len[b];
    s.sum_len += s.len[b];
    pos += lens[b] + gap;
  }
  s.R = round_up(pos, 128) * scale;
  upload_seqs(ctx, s, st, with_row2seq);
  return s;
}

Seqs scale_seqs(cvk_ctx* ctx, const Seqs& b, int scale, int extra_front, cudaStream_t st, bool with_row2seq) {
  Seqs s;
  s.B = b.B;
  s.start.resize(b.B);
  s.len.resize(b.B);
  for (int i = 0; i < b.B; ++i) {
    s.start[i] = b.start[i] * scale - extra_front;
    s.len[i] = b.len[i] * scale + extra_front;
    if (s.len[i] > s.max_len) s.max_len = s.len[i];
    s.sum_len += s.len[i];
  }
  s.R = b.R * scale;
  upload_seqs(ctx, s, st, with_row2seq);
  return s;
}

// same rows, every sequence shortened by drop_tail rows at its end (flow look-ahead context, flow/flow.py:259-261)
Seqs shrink_seqs(cvk_ctx* ctx, const Seqs& b, int drop_tail, cudaStream_t st) {
  Seqs s;
  s.B = b.B;
  s.start = b.start;
  s.len.resize(b.B);
  for (int i = 0; i < b.B; ++i) {
    s.len[i] = b.len[i] - drop_tail;
    CVK_REQUIRE(s.len[i] > 0, "sequence shorter than the look-ahead context");
    if (s.len[i] > s.max_len) s.max_len = s.len[i];
    s.sum_len += s.len[i];
  }
  s.R = b.R;
  upload_seqs(ctx, s, st, true);
  return s;
}

// same rows, sequence b restricted to its first skip[b] rows (prompt part)
Seqs subseqs(cvk_ctx* ctx, const Seqs& b, const int* head_host, cudaStream_t st) {
  Seqs s;
  s.B = b.B;
  s.start = b.start;
  s.len.assign(head_host, head_host + b.B);
  for (int i = 0; i < b.B; ++i) {
    CVK_REQUIRE(s.len[i] >= 0 && s.len[i] <= b.len[i], "prefix longer than the sequence");
    if (s.len[i] > s.max_len) s.max_len = s.len[i];
    s.sum_len += s.len[i];
  }
  s.R = b.R;
  upload_seqs(ctx, s, st, false);
  return s;
}

// ================================================================================================ weights
namespace {
// torch Conv1d weight [N][K][taps] -> [N][taps][K]
__global__ void repack_conv_kernel(const float* __restrict__ w, float* __restrict__ o, int N, int K, int taps) {
  size_t total = (size_t)N * K * taps;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int k = i % K;
    int j = (i / K) % taps;
    int n = i / ((size_t)K * taps);
    o[i] = w[((size_t)n * K + k) * taps + j];
  }
}
__global__ void f32_to_bf16_kernel(const float* __restrict__ x, bf16* __restrict__ y, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    y[i] = __float2bfloat16_rn(x[i]);
}
__global__ void f32_to_f16_kernel(const float* __restrict__ x, __half* __restrict__ y, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    y[i] = from_f32<__half>(x[i]);
}
// weight_norm (dim 0): w[i, ...] = g[i] * v[i, ...] / ||v[i, ...]||_2   (one block per leading index)
__global__ void weight_norm_kernel(const float* __restrict__ g, const float* __restrict__ v, float* __restrict__ w, int inner) {
  __shared__ float red[32];
  int i = blockIdx.x;
  const float* vp = v + (size_t)i * inner;
  float s = 0.f;
  for (int j = threadIdx.x; j < inner; j += blockDim.x) s += vp[j] * vp[j];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) red[0] = t;
  }
  __syncthreads();
  float scale = g[i] / sqrtf(red[0]);
  for (int j = threadIdx.x; j < inner; j += blockDim.x) w[(size_t)i * inner + j] = vp[j] * scale;
}
}  // namespace

float* dev_copy_f32(cvk_ctx* ctx, const float* src_dev, size_t n) {
  float* p = (float*)ctx->dmalloc(n * sizeof(float));
  CVK_CHECK_CUDA(cudaMemcpy(p, src_dev, n * sizeof(float), cudaMemcpyDeviceToDevice));
  return p;
}

void finish_convw(cvk_ctx* ctx, ConvW& w) {
  if (ctx->precision == CVK_PREC_BF16 && w.K % 8 == 0 && ctx->build_f16) {      // vocoder stage on IEEE-half operands
    size_t n = (size_t)w.N * w.taps * w.K;
    w.wf16 = (__half*)ctx->dmalloc(n * sizeof(__half));
    f32_to_f16_kernel<<<256, 256>>>(w.w32, w.wf16, n);
    CVK_LAUNCH_CHECK();
    return;
  }
  if (ctx->precision == CVK_PREC_BF16 && w.K % 8 == 0) {
    size_t n = (size_t)w.N * w.taps * w.K;
    w.w16 = (bf16*)ctx->dmalloc(n * sizeof(bf16));
    f32_to_bf16_kernel<<<256, 256>>>(w.w32, w.w16, n);
    CVK_LAUNCH_CHECK();
  }
}

ConvW make_conv(cvk_ctx* ctx, const float* w_nkt, const float* bias, int N, int K, int taps, int dil, int shift0) {
  ConvW w;
  w.N = N; w.K = K; w.taps = taps; w.dil = dil; w.shift0 = shift0;
  size_t n = (size_t)N * K * taps;
  w.w32 = (float*)ctx->dmalloc(n * sizeof(float));
  if (taps == 1) CVK_CHECK_CUDA(cudaMemcpy(w.w32, w_nkt, n * sizeof(float), cudaMemcpyDeviceToDevice));
  else {
    repack_conv_kernel<<<256, 256>>>(w_nkt, w.w32, N, K, taps);
    CVK_LAUNCH_CHECK();
  }
  if (bias) w.bias = dev_copy_f32(ctx, bias, N);
  finish_convw(ctx, w);
  return w;
}

ConvW make_conv_named(cvk_ctx* ctx, const std::string& wname, const std::string& bname, int dil, int shift0) {
  const RawTensor& w = ctx->get_raw(wname);
  CVK_REQUIRE(w.shape.size() == 3 || w.shape.size() == 2, "conv/linear weight must be 2-D or 3-D: " + wname);
  int N = (int)w.shape[0], K = (int)w.shape[1], taps = w.shape.size() == 3 ? (int)w.shape[2] : 1;
  const float* b = nullptr;
  if (!bname.empty()) {
    const RawTensor& bt = ctx->get_raw(bname);
    CVK_REQUIRE(bt.numel() == N, "bias size mismatch: " + bname);
    b = bt.p;
  }
  return make_conv(ctx, w.p, b, N, K, taps, dil, shift0);
}

ConvW make_linear(cvk_ctx* ctx, const std::string& wname, const std::string& bname) {
  return make_conv_named(ctx, wname, bname, 1, 0);
}

// effective weight of a weight-normalised module "<prefix>.parametrizations.weight.original{0,1}" (or the legacy
// "<prefix>.weight_g/.weight_v" spelling, hifigan/generator.py:26-29).  Returns a temporary device buffer (owned by ctx).
float* fold_weight_norm(cvk_ctx* ctx, const std::string& prefix, int64_t* numel_out) {
  std::string gk = prefix + ".parametrizations.weight.original0", vk = prefix + ".parametrizations.weight.original1";
  if (!ctx->has_raw(gk)) { gk = prefix + ".weight_g"; vk = prefix + ".weight_v"; }
  const RawTensor& g = ctx->get_raw(gk);
  const RawTensor& v = ctx->get_raw(vk);
  int lead = (int)v.shape[0];
  int inner = (int)(v.numel() / lead);
  CVK_REQUIRE(g.numel() == lead, "weight-norm g/v mismatch: " + prefix);
  float* w = (float*)ctx->dmalloc(v.numel() * sizeof(float));
  weight_norm_kernel<<<lead, 256>>>(g.p, v.p, w, inner);
  CVK_LAUNCH_CHECK();
  if (numel_out) *numel_out = v.numel();
  return w;
}

// ================================================================================================ elementwise
namespace {

template <typename TO>
__global__ void zero_kernel(TO* __restrict__ p, int rows, int cols, int ld) {
  size_t total = (size_t)rows * cols;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int r = i / cols, c = i % cols;
    p[(size_t)r * ld + c] = from_f32<TO>(0.f);
  }
}

// LayerNorm over the channel dimension, one warp per row; optional activation, post-scale and row mask.
// torch.nn.LayerNorm: biased variance, eps inside the sqrt.
template <typename TO>
__global__ void layernorm_kernel(const float* __restrict__ x, int ldx, int rows, int C, const float* __restrict__ gamma,
                                 const float* __restrict__ beta, float eps, int act, float post_scale, const int* __restrict__ row2seq,
                                 TO* __restrict__ out, int ldo, const float* __restrict__ rowvec, int rowvec_ld) {
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const float* xp = x + (size_t)warp * ldx;
  TO* op = out + (size_t)warp * ldo;
  int seq = row2seq ? row2seq[warp] : 0;
  bool valid = seq >= 0;
  if (!valid) {
    for (int c = lane; c < C; c += 32) op[c] = from_f32<TO>(0.f);
    return;
  }
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += xp[c];
  float mean = warp_sum(s) / C;
  float v = 0.f;
  for (int c = lane; c < C; c += 32) {
    float d = xp[c] - mean;
    v += d * d;
  }
  float rstd = rsqrtf(warp_sum(v) / C + eps);
  for (int c = lane; c < C; c += 32) {
    float y = (xp[c] - mean) * rstd;
    if (gamma) y = y * gamma[c] + (beta ? beta[c] : 0.f);
    y = apply_act(act, y, 0.f, 1.f) * post_scale;
    if (rowvec) y += rowvec[(size_t)seq * rowvec_ld + c];
    op[c] = from_f32<TO>(y);
  }
}

// C == 256 (every LayerNorm of the flow estimator): the row lives in registers (two float4 per lane), read once with 16-byte
// loads, written with 8/16-byte stores; the activation dispatch is outside the element loop.  FAST = bf16 mode (hardware
// approximations, error two orders below the bf16 rounding of the stored result); the fp32 parity mode keeps libm.
template <typename TO, bool FAST>
__global__ void layernorm256_kernel(const float* __restrict__ x, int ldx, int rows, const float* __restrict__ gamma,
                                    const float* __restrict__ beta, float eps, int act, float post_scale, const int* __restrict__ row2seq,
                                    TO* __restrict__ out, int ldo, const float* __restrict__ rowvec, int rowvec_ld) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const float* xp = x + (size_t)warp * ldx;
  TO* op = out + (size_t)warp * ldo;
  const int seq = row2seq ? row2seq[warp] : 0;
  const int c0 = lane * 4, c1 = 128 + lane * 4;
  float v[8];
  if (seq < 0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = 0.f;
  } else {
    const float4 a = *reinterpret_cast<const float4*>(xp + c0), b = *reinterpret_cast<const float4*>(xp + c1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    const float mean = warp_sum(((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]))) * (1.f / 256.f);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      v[i] -= mean;
      q = fmaf(v[i], v[i], q);
    }
    const float rstd = rsqrtf(warp_sum(q) * (1.f / 256.f) + eps);
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] *= rstd;
    if (gamma) {
      const float4 ga = *reinterpret_cast<const float4*>(gamma + c0), gb = *reinterpret_cast<const float4*>(gamma + c1);
      v[0] *= ga.x; v[1] *= ga.y; v[2] *= ga.z; v[3] *= ga.w; v[4] *= gb.x; v[5] *= gb.y; v[6] *= gb.z; v[7] *= gb.w;
      if (beta) {
        const float4 ba = *reinterpret_cast<const float4*>(beta + c0), bb = *reinterpret_cast<const float4*>(beta + c1);
        v[0] += ba.x; v[1] += ba.y; v[2] += ba.z; v[3] += ba.w; v[4] += bb.x; v[5] += bb.y; v[6] += bb.z; v[7] += bb.w;
      }
    }
    if (act == ACT_MISH) {
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = FAST ? apply_act_fast(ACT_MISH, v[i], 0.f, 1.f) : apply_act(ACT_MISH, v[i], 0.f, 1.f);
    } else if (act != ACT_NONE) {
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = FAST ? apply_act_fast(act, v[i], 0.f, 1.f) : apply_act(act, v[i], 0.f, 1.f);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] *= post_scale;
    if (rowvec) {
      const float* rv = rowvec + (size_t)seq * rowvec_ld;
      const float4 ra = *reinterpret_cast<const float4*>(rv + c0), rb = *reinterpret_cast<const float4*>(rv + c1);
      v[0] += ra.x; v[1] += ra.y; v[2] += ra.z; v[3] += ra.w; v[4] += rb.x; v[5] += rb.y; v[6] += rb.z; v[7] += rb.w;
    }
  }
  if constexpr (sizeof(TO) == 4) {
    *reinterpret_cast<float4*>((float*)op + c0) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>((float*)op + c1) = make_float4(v[4], v[5], v[6], v[7]);
  } else {
    __nv_bfloat162 h0 = __floats2bfloat162_rn(v[0], v[1]), h1 = __floats2bfloat162_rn(v[2], v[3]);
    __nv_bfloat162 h2 = __floats2bfloat162_rn(v[4], v[5]), h3 = __floats2bfloat162_rn(v[6], v[7]);
    *reinterpret_cast<uint2*>((bf16*)op + c0) = make_uint2(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1));
    *reinterpret_cast<uint2*>((bf16*)op + c1) = make_uint2(*reinterpret_cast<uint32_t*>(&h2), *reinterpret_cast<uint32_t*>(&h3));
  }
}

// Qwen2 RMSNorm (modeling_qwen2.py:258-263): w * (x * rsqrt(mean(x^2) + eps))
template <typename TO>
__global__ void rmsnorm_kernel(const float* __restrict__ x, int ldx, int rows, int C, const float* __restrict__ gamma, float eps,
                               TO* __restrict__ out, int ldo) {
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const float* xp = x + (size_t)warp * ldx;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += xp[c] * xp[c];
  float r = rsqrtf(warp_sum(s) / C + eps);
  for (int c = lane; c < C; c += 32) out[(size_t)warp * ldo + c] = from_f32<TO>(gamma[c] * (xp[c] * r));
}

template <typename TI, typename TO>
__global__ void act_copy_kernel(const TI* __restrict__ x, int ldx, int rows, int C, int act, float param, const float* __restrict__ alpha,
                                float pre_scale, const int* __restrict__ row2seq, TO* __restrict__ out, int ldo) {
  size_t total = (size_t)rows * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int r = i / C, c = i % C;
    float v = 0.f;
    if (!row2seq || row2seq[r] >= 0) v = apply_act(act, to_f32(x[(size_t)r * ldx + c]) * pre_scale, param, alpha ? alpha[c] : 1.f);
    out[(size_t)r * ldo + c] = from_f32<TO>(v);
  }
}

// dense ragged [sum_len, C] fp32 -> packed rows (gap rows zero)
template <typename TO>
__global__ void pack_rows_kernel(const float* __restrict__ dense, int C, const int* __restrict__ start, const int* __restrict__ len,
                                 int B, TO* __restrict__ out, int ldo, const int* __restrict__ dense_off) {
  int b = blockIdx.y;
  int l = len[b], s = start[b];
  size_t total = (size_t)l * C;
  const float* src = dense + (size_t)dense_off[b] * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int t = i / C, c = i % C;
    out[(size_t)(s + t) * ldo + c] = from_f32<TO>(src[i]);
  }
}
template <typename TI>
__global__ void unpack_rows_kernel(const TI* __restrict__ in, int ldi, const int* __restrict__ start, const int* __restrict__ len,
                                   int skip_all, const int* __restrict__ skips, float* __restrict__ dense, int C,
                                   const int* __restrict__ dense_off) {
  int b = blockIdx.y;
  int skip = skips ? skips[b] : skip_all;
  int l = len[b] - skip, s = start[b] + skip;
  if (l <= 0) return;
  size_t total = (size_t)l * C;
  float* dst = dense + (size_t)dense_off[b] * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int t = i / C, c = i % C;
    dst[i] = to_f32(in[(size_t)(s + t) * ldi + c]);
  }
}
template <typename TO>
__global__ void bcast_rows_kernel(const float* __restrict__ vec, int C, int vec_ld, const int* __restrict__ row2seq, int rows,
                                  TO* __restrict__ out, int ldo) {
  size_t total = (size_t)rows * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int r = i / C, c = i % C;
    int sq = row2seq[r];
    out[(size_t)r * ldo + c] = from_f32<TO>(sq >= 0 ? vec[(size_t)sq * vec_ld + c] : 0.f);
  }
}

inline int grid_for(size_t total, int threads = 256) {
  size_t g = (total + threads - 1) / threads;
  if (g > 132 * 16) g = 132 * 16;
  if (g < 1) g = 1;
  return (int)g;
}
}  // namespace

void zero_mat(cvk_ctx* ctx, cudaStream_t st, const Mat& m) {
  if (m.ld == m.cols) {
    CVK_CHECK_CUDA(cudaMemsetAsync(m.p, 0, (size_t)m.rows * m.ld * m.esize(), st));
    return;
  }
  size_t total = (size_t)m.rows * m.cols;
  if (m.dtype == DT_F32) zero_kernel<float><<<grid_for(total), 256, 0, st>>>(m.f32(), m.rows, m.cols, m.ld);
  else zero_kernel<bf16><<<grid_for(total), 256, 0, st>>>(m.b16(), m.rows, m.cols, m.ld);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}

void layernorm(cvk_ctx* ctx, cudaStream_t st, const Mat& x, const float* gamma, const float* beta, float eps, int act,
               float post_scale, const int* row2seq, const Mat& out, const float* rowvec, int rowvec_ld) {
  CVK_REQUIRE(x.dtype == DT_F32, "layernorm input must be fp32");
  int rows = x.rows, C = x.cols;
  int blocks = ceil_div(rows, 8);
  const bool vec = C == 256 && x.ld % 4 == 0 && ((uintptr_t)x.p & 15) == 0 && (out.ld * out.esize()) % 16 == 0 && ((uintptr_t)out.p & 15) == 0 &&
                   (!rowvec || (rowvec_ld % 4 == 0 && ((uintptr_t)rowvec & 15) == 0)) && (!gamma || ((uintptr_t)gamma & 15) == 0) &&
                   (!beta || ((uintptr_t)beta & 15) == 0);
  if (vec) {
    const bool fast = ctx->precision == CVK_PREC_BF16;
    if (out.dtype == DT_F32) {
      if (fast) layernorm256_kernel<float, true><<<blocks, 256, 0, st>>>(x.f32(), x.ld, rows, gamma, beta, eps, act, post_scale, row2seq, out.f32(), out.ld, rowvec, rowvec_ld);
      else layernorm256_kernel<float, false><<<blocks, 256, 0, st>>>(x.f32(), x.ld, rows, gamma, beta, eps, act, post_scale, row2seq, out.f32(), out.ld, rowvec, rowvec_ld);
    } else {
      if (fast) layernorm256_kernel<bf16, true><<<blocks, 256, 0, st>>>(x.f32(), x.ld, rows, gamma, beta, eps, act, post_scale, row2seq, out.b16(), out.ld, rowvec, rowvec_ld);
      else layernorm256_kernel<bf16, false><<<blocks, 256, 0, st>>>(x.f32(), x.ld, rows, gamma, beta, eps, act, post_scale, row2seq, out.b16(), out.ld, rowvec, rowvec_ld);
    }
    ctx->launches++;
    CVK_LAUNCH_CHECK();
    return;
  }
  if (out.dtype == DT_F32)
    layernorm_kernel<float><<<blocks, 256, 0, st>>>(x.f32(), x.ld, rows, C, gamma, beta, eps, act, post_scale, row2seq, out.f32(), out.ld, rowvec, rowvec_ld);
  else
    layernorm_kernel<bf16><<<blocks, 256, 0, st>>>(x.f32(), x.ld, rows, C, gamma, beta, eps, act, post_scale, row2seq, out.b16(), out.ld, rowvec, rowvec_ld);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}

void rmsnorm(cvk_ctx* ctx, cudaStream_t st, const Mat& x, const float* gamma, float eps, const Mat& out) {
  CVK_REQUIRE(x.dtype == DT_F32, "rmsnorm input must be fp32");
  int blocks = ceil_div(x.rows, 8);
  if (out.dtype == DT_F32) rmsnorm_kernel<float><<<blocks, 256, 0, st>>>(x.f32(), x.ld, x.rows, x.cols, gamma, eps, out.f32(), out.ld);
  else rmsnorm_kernel<bf16><<<blocks, 256, 0, st>>>(x.f32(), x.ld, x.rows, x.cols, gamma, eps, out.b16(), out.ld);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}

void act_copy(cvk_ctx* ctx, cudaStream_t st, const Mat& x, int act, float param, const float* alpha, const int* row2seq,
              const Mat& out) {
  act_copy_scaled(ctx, st, x, 1.f, act, param, alpha, row2seq, out);
}

void act_copy_scaled(cvk_ctx* ctx, cudaStream_t st, const Mat& x, float pre_scale, int act, float param, const float* alpha,
                     const int* row2seq, const Mat& out) {
  size_t total = (size_t)x.rows * x.cols;
  int g = grid_for(total);
#define LAUNCH(TI, TO, xi, oo) \
  act_copy_kernel<TI, TO><<<g, 256, 0, st>>>(xi, x.ld, x.rows, x.cols, act, param, alpha, pre_scale, row2seq, oo, out.ld)
  if (x.dtype == DT_F32 && out.dtype == DT_F16) LAUNCH(float, __half, x.f32(), (__half*)out.p);
  else if (x.dtype == DT_F16 && out.dtype == DT_F32) LAUNCH(__half, float, (const __half*)x.p, out.f32());
  else if (x.dtype == DT_F16 && out.dtype == DT_F16) LAUNCH(__half, __half, (const __half*)x.p, (__half*)out.p);
  else if (x.dtype == DT_F16 || out.dtype == DT_F16) throw CvkError(CVK_ERR_INVALID, "act_copy: half <-> bf16 conversion is not provided");
  else if (x.dtype == DT_F32 && out.dtype == DT_F32) LAUNCH(float, float, x.f32(), out.f32());
  else if (x.dtype == DT_F32) LAUNCH(float, bf16, x.f32(), out.b16());
  else if (out.dtype == DT_F32) LAUNCH(bf16, float, x.b16(), out.f32());
  else LAUNCH(bf16, bf16, x.b16(), out.b16());
#undef LAUNCH
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}

void convert_mat(cvk_ctx* ctx, cudaStream_t st, const Mat& in, const Mat& out) {
  act_copy_scaled(ctx, st, in, 1.f, ACT_NONE, 0.f, nullptr, nullptr, out);
}

static int* dense_offsets(cvk_ctx* ctx, const Seqs& s, int skip, cudaStream_t st) {
  std::vector<int> off(s.B);
  int acc = 0;
  for (int b = 0; b < s.B; ++b) {
    off[b] = acc;
    acc += s.len[b] - skip;
  }
  int* d = (int*)ctx->arena.alloc(sizeof(int) * s.B);
  CVK_CHECK_CUDA(cudaMemcpyAsync(d, off.data(), sizeof(int) * s.B, cudaMemcpyHostToDevice, st));
  return d;
}

void pack_rows(cvk_ctx* ctx, cudaStream_t st, const float* dense, int C, const Seqs& s, const Mat& out) {
  int* off = dense_offsets(ctx, s, 0, st);
  int bx = grid_for((size_t)s.max_len * C);
  if (bx > 256) bx = 256;
  if (out.dtype == DT_F32) pack_rows_kernel<float><<<dim3(bx, s.B), 256, 0, st>>>(dense, C, s.d_start, s.d_len, s.B, out.f32(), out.ld, off);
  else pack_rows_kernel<bf16><<<dim3(bx, s.B), 256, 0, st>>>(dense, C, s.d_start, s.d_len, s.B, out.b16(), out.ld, off);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}

void unpack_rows(cvk_ctx* ctx, cudaStream_t st, const Mat& in, const Seqs& s, int skip, float* dense, int C) {
  int* off = dense_offsets(ctx, s, skip, st);
  int bx = grid_for((size_t)s.max_len * C);
  if (bx > 256) bx = 256;
  if (in.dtype == DT_F32) unpack_rows_kernel<float><<<dim3(bx, s.B), 256, 0, st>>>(in.f32(), in.ld, s.d_start, s.d_len, skip, nullptr, dense, C, off);
  else unpack_rows_kernel<bf16><<<dim3(bx, s.B), 256, 0, st>>>(in.b16(), in.ld, s.d_start, s.d_len, skip, nullptr, dense, C, off);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}

void unpack_rows_skip(cvk_ctx* ctx, cudaStream_t st, const Mat& in, const Seqs& s, const int* skip_host, float* dense, int C) {
  std::vector<int> off(s.B), sk(skip_host, skip_host + s.B);
  int acc = 0;
  for (int b = 0; b < s.B; ++b) {
    off[b] = acc;
    acc += s.len[b] - sk[b];
  }
  int* d_off = (int*)ctx->arena.alloc(sizeof(int) * s.B);
  int* d_sk = (int*)ctx->arena.alloc(sizeof(int) * s.B);
  CVK_CHECK_CUDA(cudaMemcpyAsync(d_off, off.data(), sizeof(int) * s.B, cudaMemcpyHostToDevice, st));
  CVK_CHECK_CUDA(cudaMemcpyAsync(d_sk, sk.data(), sizeof(int) * s.B, cudaMemcpyHostToDevice, st));
  int bx = grid_for((size_t)s.max_len * C);
  if (bx > 256) bx = 256;
  if (in.dtype == DT_F32) unpack_rows_kernel<float><<<dim3(bx, s.B), 256, 0, st>>>(in.f32(), in.ld, s.d_start, s.d_len, 0, d_sk, dense, C, d_off);
  else unpack_rows_kernel<bf16><<<dim3(bx, s.B), 256, 0, st>>>(in.b16(), in.ld, s.d_start, s.d_len, 0, d_sk, dense, C, d_off);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}

void bcast_rows(cvk_ctx* ctx, cudaStream_t st, const float* vec, int C, int vec_ld, const Seqs& s, const Mat& out) {
  size_t total = (size_t)s.R * C;
  if (out.dtype == DT_F32) bcast_rows_kernel<float><<<grid_for(total), 256, 0, st>>>(vec, C, vec_ld, s.d_row2seq, s.R, out.f32(), out.ld);
  else bcast_rows_kernel<bf16><<<grid_for(total), 256, 0, st>>>(vec, C, vec_ld, s.d_row2seq, s.R, out.b16(), out.ld);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}
