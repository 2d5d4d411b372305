// HiFT vocoder (CosyVoice2 config): mel -> f0 -> harmonic source -> STFT -> conv / ResBlock stack -> ISTFT.
// Follows cosyvoice/hifigan/generator.py:557-569 (inference), :507-539 (decode), :491-505 (_stft/_istft),
// :358-375 + :233-317 (SourceModuleHnNSF / SineGen2), f0_predictor.py:56-59; hyper-parameters of
// examples/libritts/cosyvoice2/conf/cosyvoice2.yaml:89-111.
//
// Layout: time-major ragged matrices at four rates (mel frame, x8, x40, x120) that share one row geometry scaled
// by the up-sampling factor, so that ConvTranspose1d(stride s) is a 3-tap convolution producing s*Cout columns
// whose output buffer [R, s*Cout] *is* the next level's [s*R, Cout] matrix (polyphase form, no scatter).
#include "common.cuh"

namespace {

constexpr int kUps[3] = {8, 5, 3};
constexpr int kUpK[3] = {16, 11, 7};
constexpr int kRbK[3] = {3, 7, 11};
constexpr int kSrcRbK[3] = {7, 7, 11};
constexpr int kDil[3] = {1, 3, 5};
constexpr int kCh[4] = {512, 256, 128, 64};
constexpr int kUpscale = 480;
constexpr int kStftLd = 24;   // 18 STFT channels padded to 24 so that strided views keep 16-byte row pitch

struct ResBlockW {
  ConvW c1[3], c2[3];
  float* a1[3];
  float* a2[3];
};

}  // namespace

struct HiftModel {
  bool half_weights = false;   // conv weights were finalised as IEEE half (wf16): the body runs on DT_F16 operands
  ConvW f0_conv[5];
  ConvW f0_cls;
  float* src_w = nullptr;   // [9]
  float* src_b = nullptr;   // [1]
  ConvW conv_pre, conv_post;
  ConvW ups[3];
  ConvW src_down[3];
  ResBlockW src_rb[3];
  ResBlockW rb[9];
};

namespace {

// ---------------------------------------------------------------------------------------------- weight repack
// ConvTranspose1d weight [Cin][Cout][k] (stride s, padding p) -> polyphase conv [s*Cout][3][Cin]:
//   out[t*s + ph, co] = sum_{m in {-1,0,1}} sum_ci x[t - m, ci] * w[ci][co][m*s + ph + p]
// tap jt reads input row t + (jt - 1), i.e. m = 1 - jt.
__global__ void polyphase_kernel(const float* __restrict__ w, float* __restrict__ o, int Cin, int Cout, int k, int s, int p) {
  size_t total = (size_t)s * Cout * 3 * Cin;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int ci = i % Cin;
    int jt = (i / Cin) % 3;
    int n = i / ((size_t)Cin * 3);
    int ph = n / Cout, co = n % Cout;
    int m = 1 - jt;
    int j = m * s + ph + p;
    o[i] = (j >= 0 && j < k) ? w[((size_t)ci * Cout + co) * k + j] : 0.f;
  }
}
__global__ void repeat_bias_kernel(const float* __restrict__ b, float* __restrict__ o, int Cout, int s) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < Cout * s) o[i] = b[i % Cout];
}
// strided Conv1d weight [N][18][k] (stride s, padding p) over the STFT matrix viewed as [R/s, s*24]:
//   level-3 row of tap j for output row r = s*r + j - (p+1)  ->  view row r + dq, view column pp*24 + c
__global__ void strided_view_fill_kernel(const float* __restrict__ w, float* __restrict__ o, int N, int C, int k, int s, int off) {
  int Kv = s * kStftLd;
  size_t total = (size_t)N * C * k;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int j = i % k;
    int c = (i / k) % C;
    int n = i / ((size_t)C * k);
    int jp = j - off;
    int dq = jp >= 0 ? jp / s : -((-jp + s - 1) / s);
    int pp = jp - dq * s;
    o[((size_t)n * 3 + (dq + 1)) * Kv + pp * kStftLd + c] = w[i];
  }
}

// ---------------------------------------------------------------------------------------------- source
// SineGen2 phase: per (sequence, harmonic) running sum over mel frames of rad = (f0*h/24000) mod 1, then
// (cum * 2) * pi * 480 exactly as generator.py:255-257.  torch's CPU cumsum accumulates float in double
// (at::acc_type<float,false>), mirrored here so the parity mode tracks the CPU reference.
__global__ void phase_kernel(const float* __restrict__ f0, int f0_ld, const int* __restrict__ start, const int* __restrict__ len,
                             float* __restrict__ phase /*[R0][9]*/) {
  int b = blockIdx.x;
  int h = threadIdx.x;
  if (h >= 9) return;
  int s = start[b], l = len[b];
  double cum = 0.0;
  const float harm = (float)(h + 1);
  const float pi_f = 3.14159265358979323846f;
  for (int t = 0; t < l; ++t) {
    float fn = f0[(size_t)(s + t) * f0_ld] * harm;
    float rad = fmodf(fn / 24000.f, 1.f);
    cum += (double)rad;
    float c = (float)cum;
    phase[(size_t)(s + t) * 9 + h] = ((c * 2.f) * pi_f) * 480.f;
  }
}

// one thread per output sample: linear x480 up-sampling of the phase (F.interpolate, align_corners=False),
// sin, voiced/unvoiced gating, additive noise, Linear(9->1) + tanh (generator.py:289-317, 358-375)
__global__ void source_kernel(const float* __restrict__ f0, int f0_ld, const float* __restrict__ phase, const int* __restrict__ start,
                              const int* __restrict__ len, const float* __restrict__ noise /*dense [sum 480T][9]*/,
                              const int* __restrict__ noise_off, const float* __restrict__ lw, const float* __restrict__ lb,
                              float* __restrict__ src /*[480*R0]*/) {
  int b = blockIdx.y;
  int T = len[b], s0 = start[b];
  int L = T * kUpscale;
  const float scale = (float)(1.0 / 480.0);
  for (int l = blockIdx.x * blockDim.x + threadIdx.x; l < L; l += gridDim.x * blockDim.x) {
    float srcf = scale * ((float)l + 0.5f) - 0.5f;
    if (srcf < 0.f) srcf = 0.f;
    int i0 = (int)srcf;
    int i1 = i0 + (i0 < T - 1 ? 1 : 0);
    float l1 = srcf - (float)i0, l0 = 1.f - l1;
    int t = l / kUpscale;
    float f = f0[(size_t)(s0 + t) * f0_ld];
    float uv = f > 10.f ? 1.f : 0.f;
    float noise_amp = uv * 0.003f + (1.f - uv) * 0.1f / 3.f;
    const float* p0 = phase + (size_t)(s0 + i0) * 9;
    const float* p1 = phase + (size_t)(s0 + i1) * 9;
    const float* nz = noise + ((size_t)noise_off[b] * kUpscale + l) * 9;
    float acc = 0.f;
#pragma unroll
    for (int h = 0; h < 9; ++h) {
      float ph = l0 * p0[h] + l1 * p1[h];
      float sw = (sinf(ph) * 0.1f) * uv + noise_amp * nz[h];
      acc += sw * lw[h];
    }
    src[(size_t)s0 * kUpscale + l] = tanhf(acc + lb[0]);
  }
}

__global__ void cache_source_kernel(const float* __restrict__ cache, const int* __restrict__ cache_off, const int* __restrict__ cache_len,
                                    const int* __restrict__ start, float* __restrict__ src) {
  int b = blockIdx.y;
  int n = cache_len[b];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    src[(size_t)start[b] * kUpscale + i] = cache[cache_off[b] + i];
}

// ---------------------------------------------------------------------------------------------- STFT / ISTFT (n_fft 16, hop 4)
__constant__ float c_win[16];
__constant__ float c_cos[16];   // cos(2*pi*i/16)
__constant__ float c_sin[16];

// frame f of sequence b -> 9 re + 9 im (torch.stft center=True, reflect), written to the level-3 matrix row
// start3[b] + f, columns [0,9) re, [9,18) im, [18,24) zero.
template <typename TO>
__global__ void stft16_kernel(const float* __restrict__ src, const int* __restrict__ start0, const int* __restrict__ len0,
                              const int* __restrict__ start3, TO* __restrict__ out, int ldo, const int* __restrict__ len_sig = nullptr) {
  int b = blockIdx.y;
  // len_sig (CosyVoice3 vocoder): sequence b's source is len_sig[b] frames long, only the first len0[b]*120 + 1 STFT frames are
  // kept.  A final utterance passes len_sig[b] == len0[b], which is the nullptr case.
  int L = (len_sig ? len_sig[b] : len0[b]) * kUpscale;
  int F = len_sig ? len0[b] * 120 + 1 : L / 4 + 1;
  const float* x = src + (size_t)start0[b] * kUpscale;
  for (int f = blockIdx.x * blockDim.x + threadIdx.x; f < F; f += gridDim.x * blockDim.x) {
    float xv[16];
#pragma unroll
    for (int n = 0; n < 16; ++n) {
      int m = 4 * f + n - 8;
      if (m < 0) m = -m;
      if (m >= L) m = 2 * (L - 1) - m;
      xv[n] = x[m] * c_win[n];
    }
    TO* op = out + (size_t)(start3[b] + f) * ldo;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      float re = 0.f, im = 0.f;
#pragma unroll
      for (int n = 0; n < 16; ++n) {
        int idx = (k * n) & 15;
        re += xv[n] * c_cos[idx];
        im -= xv[n] * c_sin[idx];
      }
      op[k] = from_f32<TO>(re);
      op[9 + k] = from_f32<TO>(im);
    }
#pragma unroll
    for (int k = 18; k < kStftLd; ++k) op[k] = from_f32<TO>(0.f);
  }
}

// conv_post output [R3, 18] -> magnitude = min(exp(x[:9]), 100), phase = sin(x[9:]) -> irfft(16) * window,
// overlap-add / window-envelope, trim 8, clamp +-0.99 (generator.py:533-538, torch.istft center=True).
// Block: 512 output samples, which need frames f_base-1 .. f_base+129.
__global__ void istft16_kernel(const float* __restrict__ xp, int ldx, const int* __restrict__ start3, const int* __restrict__ len0,
                               const int* __restrict__ out_off, float* __restrict__ wav, float limit,
                               const int* __restrict__ drop_tail = nullptr) {
  __shared__ float fr[131][17];   // frames f_base-1 .. f_base+129
  int b = blockIdx.y;
  int L = len0[b] * kUpscale;
  int F = L / 4 + 1;
  const int L_out = L - (drop_tail ? drop_tail[b] : 0);
  int f_base = blockIdx.x * 128;          // first frame whose leading 4 samples this block emits
  if (f_base * 4 >= L) return;
  for (int i = threadIdx.x; i < 131; i += blockDim.x) {
    int f = f_base - 1 + i;
    if (f < 0 || f >= F) {
#pragma unroll
      for (int n = 0; n < 16; ++n) fr[i][n] = 0.f;
      continue;
    }
    const float* p = xp + (size_t)(start3[b] + f) * ldx;
    float re[9], im[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      float mag = fminf(expf(p[k]), 100.f);
      float ph = sinf(p[9 + k]);
      re[k] = mag * cosf(ph);
      im[k] = mag * sinf(ph);
    }
#pragma unroll
    for (int n = 0; n < 16; ++n) {
      float acc = re[0] + ((n & 1) ? -re[8] : re[8]);   // DC and Nyquist (imaginary parts ignored by irfft)
#pragma unroll
      for (int k = 1; k < 8; ++k) {
        int idx = (k * n) & 15;
        acc += 2.f * (re[k] * c_cos[idx] - im[k] * c_sin[idx]);
      }
      fr[i][n] = acc * (1.f / 16.f) * c_win[n];
    }
  }
  __syncthreads();
  // output sample n (after trimming 8) lives at padded position p = n + 8; frames f with 4f <= p < 4f + 16
  for (int i = threadIdx.x; i < 512; i += blockDim.x) {
    int n = f_base * 4 + i;
    if (n >= L_out) break;        // drop_tail[b]: samples of the last look-ahead frame are not emitted (generator.py:709-710)
    int p = n + 8;
    int f_hi = p >> 2;
    float acc = 0.f, env = 0.f;
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      int f = f_hi - d;
      if (f < 0 || f >= F) continue;
      int m = p - 4 * f;
      acc += fr[f - (f_base - 1)][m];
      env += c_win[m] * c_win[m];
    }
    float y = acc / env;
    wav[(size_t)out_off[b] * kUpscale + n] = fminf(fmaxf(y, -limit), limit);
  }
}

// ReflectionPad1d((1,0)) at the last level: row start3[b] := row start3[b] + 2
__global__ void reflect_front_kernel(float* __restrict__ x, int ld, int C, const int* __restrict__ start3) {
  int b = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) x[(size_t)start3[b] * ld + c] = x[(size_t)(start3[b] + 2) * ld + c];
}

bool g_consts_ready = false;
void init_consts() {
  if (g_consts_ready) return;
  float win[16], cs[16], sn[16];
  const double PI = 3.14159265358979323846;
  for (int i = 0; i < 16; ++i) {
    win[i] = (float)(0.5 - 0.5 * cos(2.0 * PI * i / 16.0));   // scipy get_window('hann', 16, fftbins=True)
    cs[i] = (float)cos(2.0 * PI * i / 16.0);
    sn[i] = (float)sin(2.0 * PI * i / 16.0);
  }
  CVK_CHECK_CUDA(cudaMemcpyToSymbol(c_win, win, sizeof(win)));
  CVK_CHECK_CUDA(cudaMemcpyToSymbol(c_cos, cs, sizeof(cs)));
  CVK_CHECK_CUDA(cudaMemcpyToSymbol(c_sin, sn, sizeof(sn)));
  g_consts_ready = true;
}

// ---------------------------------------------------------------------------------------------- model build
ConvW wn_conv(cvk_ctx* ctx, const std::string& prefix, int dil, int shift0) {
  float* w = fold_weight_norm(ctx, prefix, nullptr);
  const RawTensor& v = ctx->has_raw(prefix + ".parametrizations.weight.original1") ? ctx->get_raw(prefix + ".parametrizations.weight.original1")
                                                                                     : ctx->get_raw(prefix + ".weight_v");
  const RawTensor& b = ctx->get_raw(prefix + ".bias");
  return make_conv(ctx, w, b.p, (int)v.shape[0], (int)v.shape[1], (int)v.shape[2], dil, shift0);
}

ResBlockW build_resblock(cvk_ctx* ctx, const std::string& p, int k) {
  ResBlockW r;
  for (int i = 0; i < 3; ++i) {
    int d = kDil[i];
    r.c1[i] = wn_conv(ctx, p + ".convs1." + std::to_string(i), d, -((k - 1) * d) / 2);
    r.c2[i] = wn_conv(ctx, p + ".convs2." + std::to_string(i), 1, -(k - 1) / 2);
    r.a1[i] = dev_copy_f32(ctx, ctx->get_raw(p + ".activations1." + std::to_string(i) + ".alpha").p, r.c1[i].K);
    r.a2[i] = dev_copy_f32(ctx, ctx->get_raw(p + ".activations2." + std::to_string(i) + ".alpha").p, r.c1[i].K);
  }
  return r;
}

}  // namespace

void hift_build(cvk_ctx* ctx) {
  init_consts();
  HiftModel* m = new HiftModel();
  m->half_weights = ctx->precision == CVK_PREC_BF16 && ctx->hift_f16;
  struct F16Scope { cvk_ctx* c; F16Scope(cvk_ctx* c_, bool on) : c(c_) { c->build_f16 = on; } ~F16Scope() { c->build_f16 = 0; } } f16scope(ctx, m->half_weights);
  const std::string P = "hift.";
  for (int i = 0; i < 5; ++i) {
    m->f0_conv[i] = wn_conv(ctx, P + "f0_predictor.condnet." + std::to_string(2 * i), 1, -1);
    m->f0_conv[i].w16 = nullptr;   // the f0 predictor always runs fp32 (phase accumulates f0 over the utterance)
    m->f0_conv[i].wf16 = nullptr;
  }
  m->f0_cls = make_linear(ctx, P + "f0_predictor.classifier.weight", P + "f0_predictor.classifier.bias");
  m->f0_cls.w16 = nullptr;
  m->f0_cls.wf16 = nullptr;
  m->src_w = dev_copy_f32(ctx, ctx->get_raw(P + "m_source.l_linear.weight").p, 9);
  m->src_b = dev_copy_f32(ctx, ctx->get_raw(P + "m_source.l_linear.bias").p, 1);
  m->conv_pre = wn_conv(ctx, P + "conv_pre", 1, -3);
  m->conv_post = wn_conv(ctx, P + "conv_post", 1, -3);
  for (int i = 0; i < 3; ++i) {
    // polyphase transposed convolution
    std::string pre = P + "ups." + std::to_string(i);
    float* w = fold_weight_norm(ctx, pre, nullptr);   // [Cin][Cout][k]
    int Cin = kCh[i], Cout = kCh[i + 1], k = kUpK[i], s = kUps[i], p = (k - s) / 2;
    ConvW c;
    c.N = s * Cout; c.K = Cin; c.taps = 3; c.dil = 1; c.shift0 = -1;
    c.w32 = (float*)ctx->dmalloc((size_t)c.N * 3 * Cin * sizeof(float));
    polyphase_kernel<<<256, 256>>>(w, c.w32, Cin, Cout, k, s, p);
    CVK_LAUNCH_CHECK();
    c.bias = (float*)ctx->dmalloc((size_t)c.N * sizeof(float));
    repeat_bias_kernel<<<ceil_div(c.N, 256), 256>>>(ctx->get_raw(pre + ".bias").p, c.bias, Cout, s);
    CVK_LAUNCH_CHECK();
    finish_convw(ctx, c);
    m->ups[i] = c;
  }
  {
    // source_downs: strided convs over the STFT matrix, expressed on its [R/s, s*24] view
    const int ds[3] = {15, 3, 1}, dk[3] = {30, 6, 1}, dp[3] = {7, 1, 0};
    for (int i = 0; i < 3; ++i) {
      std::string pre = P + "source_downs." + std::to_string(i);
      const RawTensor& w = ctx->get_raw(pre + ".weight");
      int N = (int)w.shape[0], C = (int)w.shape[1], k = (int)w.shape[2];
      CVK_REQUIRE(C == 18 && k == dk[i] && N == kCh[i + 1], "unexpected source_downs shape");
      ConvW c;
      c.N = N;
      c.bias = dev_copy_f32(ctx, ctx->get_raw(pre + ".bias").p, N);
      if (ds[i] == 1) {
        c.K = kStftLd; c.taps = 1; c.dil = 1; c.shift0 = 0;
        c.w32 = (float*)ctx->dmalloc((size_t)N * kStftLd * sizeof(float));
        CVK_CHECK_CUDA(cudaMemset(c.w32, 0, (size_t)N * kStftLd * sizeof(float)));
        CVK_CHECK_CUDA(cudaMemcpy2D(c.w32, kStftLd * sizeof(float), w.p, 18 * sizeof(float), 18 * sizeof(float), N, cudaMemcpyDeviceToDevice));
      } else {
        c.K = ds[i] * kStftLd; c.taps = 3; c.dil = 1; c.shift0 = -1;
        size_t n = (size_t)N * 3 * c.K;
        c.w32 = (float*)ctx->dmalloc(n * sizeof(float));
        CVK_CHECK_CUDA(cudaMemset(c.w32, 0, n * sizeof(float)));
        strided_view_fill_kernel<<<64, 256>>>(w.p, c.w32, N, C, k, ds[i], dp[i] + 1);
        CVK_LAUNCH_CHECK();
      }
      finish_convw(ctx, c);
      m->src_down[i] = c;
    }
  }
  for (int i = 0; i < 3; ++i) m->src_rb[i] = build_resblock(ctx, P + "source_resblocks." + std::to_string(i), kSrcRbK[i]);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) m->rb[i * 3 + j] = build_resblock(ctx, P + "resblocks." + std::to_string(i * 3 + j), kRbK[j]);
  CVK_CHECK_CUDA(cudaDeviceSynchronize());
  ctx->hift = m;
}

// ================================================================================================ forward pieces
struct HiftGeom {
  Seqs s0;      // mel rate
  Seqs lv[3];   // x8, x40, x120(+1 front row)
};

static HiftGeom hift_geom(cvk_ctx* ctx, const int* lens, int B, cudaStream_t st) {
  HiftGeom g;
  g.s0 = make_seqs(ctx, lens, B, 8, 1, 0, st);
  g.lv[0] = scale_seqs(ctx, g.s0, 8, 0, st);
  g.lv[1] = scale_seqs(ctx, g.s0, 40, 0, st);
  g.lv[2] = scale_seqs(ctx, g.s0, 120, 1, st);
  return g;
}

// mel32 packed [R0,80] fp32 -> f0 [R0] (ld 1)
static void hift_f0_packed(cvk_ctx* ctx, cudaStream_t st, const Seqs& s0, const Mat& mel32, const Mat& f0) {
  HiftModel* m = ctx->hift;
  Mat a = arena_mat(ctx, DT_F32, s0.R, 512), b = arena_mat(ctx, DT_F32, s0.R, 512);
  Mat cur = mel32;
  for (int i = 0; i < 5; ++i) {
    Epilogue e;
    e.act1 = ACT_ELU;
    e.row2seq = s0.d_row2seq;
    e.out = (i & 1) ? b : a;
    conv_gemm_simt(ctx, st, cur, m->f0_conv[i], e);
    cur = e.out;
  }
  Epilogue e;
  e.act1 = ACT_ABS;
  e.row2seq = s0.d_row2seq;
  e.out = f0;
  conv_gemm_simt(ctx, st, cur, m->f0_cls, e);
}

static int* upload_ints(cvk_ctx* ctx, const std::vector<int>& v, cudaStream_t st) {
  int* d = (int*)ctx->arena.alloc(sizeof(int) * v.size());
  CVK_CHECK_CUDA(cudaMemcpyAsync(d, v.data(), sizeof(int) * v.size(), cudaMemcpyHostToDevice, st));
  return d;
}

static std::vector<int> prefix_offsets(const int* lens, int B) {
  std::vector<int> off(B);
  int acc = 0;
  for (int b = 0; b < B; ++b) { off[b] = acc; acc += lens[b]; }
  return off;
}

// f0 [R0] -> packed source [480*R0] fp32 (zero in gaps).  noise: dense [sum 480T][9]
static void hift_source_packed(cvk_ctx* ctx, cudaStream_t st, const Seqs& s0, const int* lens, const Mat& f0, const float* noise,
                               float* src_packed) {
  HiftModel* m = ctx->hift;
  float* phase = (float*)ctx->arena.alloc(sizeof(float) * 9 * (size_t)s0.R);
  phase_kernel<<<s0.B, 32, 0, st>>>(f0.f32(), f0.ld, s0.d_start, s0.d_len, phase);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  CVK_CHECK_CUDA(cudaMemsetAsync(src_packed, 0, sizeof(float) * (size_t)s0.R * kUpscale, st));
  int* noff = upload_ints(ctx, prefix_offsets(lens, s0.B), st);
  int bx = ceil_div(s0.max_len * kUpscale, 256);
  if (bx > 512) bx = 512;
  source_kernel<<<dim3(bx, s0.B), 256, 0, st>>>(f0.f32(), f0.ld, phase, s0.d_start, s0.d_len, noise, noff, m->src_w, m->src_b, src_packed);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}

static void run_resblock(cvk_ctx* ctx, cudaStream_t st, const ResBlockW& rb, const Seqs& s, const Mat& x /*fp32 input*/,
                         const Mat& a /*act(x) with alpha a1[0], act dtype, consumed*/, const Mat& ya, const Mat& xr /*fp32 scratch*/,
                         const Mat& final_out, int final_accumulate) {
  for (int d = 0; d < 3; ++d) {
    Epilogue e1;
    e1.act1 = ACT_SNAKE;
    e1.alpha1 = rb.a2[d];
    e1.row2seq = s.d_row2seq;
    e1.out = ya;
    conv_gemm(ctx, st, a, rb.c1[d], e1);
    Epilogue e2;
    e2.resid = d == 0 ? x : xr;
    e2.row2seq = s.d_row2seq;
    if (d < 2) {
      e2.out = xr;
      e2.act2 = ACT_SNAKE;
      e2.alpha2 = rb.a1[d + 1];
      e2.out2 = a;
    } else {
      e2.out = final_out;
      e2.accumulate = final_accumulate;
    }
    conv_gemm(ctx, st, ya, rb.c2[d], e2);
  }
}

// mel packed + source packed -> conv_post output [R3, 18] fp32 (ld 24).
// hidden != nullptr (the test-only read-out cvk_hift_hidden): stop at read-out `unit` and write its sequence rows densely, widened to
// fp32, to `hidden`; the returned Mat is then empty.  Read-outs: 0 the source STFT (18 columns), 1 conv_pre + LReLU (xin); per level
// i: 2 + 6i the up-sampled xu (after the reflect pad at i = 2), 3 + 6i xu + the source branch, 4 + 6i .. 6 + 6i the running resblock
// sum xs, 7 + 6i the level output; 20 conv_post.
static Mat hift_body(cvk_ctx* ctx, cudaStream_t st, const HiftGeom& g, const Mat& mel32, const float* src_packed,
                     const HiftModel* m = nullptr, const int* d_len_sig = nullptr, int unit = -1, float* hidden = nullptr) {
  if (!m) m = ctx->hift;
  auto read_out = [&](int u, const Mat& x, const Seqs& s, int C) {
    if (!hidden || u != unit) return false;
    unpack_rows(ctx, st, x, s, 0, hidden, C);
    return true;
  };
  // tensor-core mode: IEEE-half operands (10-bit mantissa, the class of the TF32 convolutions the reference's "fp32" vocoder runs
  // on under cuDNN's defaults) unless the option hift_f16 is off (then bf16, 7 bits: narrower than the reference)
  const int adt = (ctx->act_dtype == DT_BF16 && m->half_weights) ? DT_F16 : ctx->act_dtype;
  const Seqs& s0 = g.s0;
  // STFT of the source at the x120 rate
  const Seqs& s3 = g.lv[2];
  Mat stft = arena_mat(ctx, adt, s3.R, kStftLd, kStftLd);
  zero_mat(ctx, st, stft);
  {
    int F = s0.max_len * 120 + 1;
    int bx = ceil_div(F, 128);
    if (bx > 1024) bx = 1024;
    if (adt == DT_F32) stft16_kernel<float><<<dim3(bx, s0.B), 128, 0, st>>>(src_packed, s0.d_start, s0.d_len, s3.d_start, stft.f32(), stft.ld, d_len_sig);
    else if (adt == DT_F16) stft16_kernel<__half><<<dim3(bx, s0.B), 128, 0, st>>>(src_packed, s0.d_start, s0.d_len, s3.d_start, (__half*)stft.p, stft.ld, d_len_sig);
    else stft16_kernel<bf16><<<dim3(bx, s0.B), 128, 0, st>>>(src_packed, s0.d_start, s0.d_len, s3.d_start, stft.b16(), stft.ld, d_len_sig);
    ctx->launches++;
    CVK_LAUNCH_CHECK();
  }
  if (read_out(0, stft, s3, 18)) return Mat();
  // conv_pre (+ leaky_relu 0.1 for ups[0])
  Mat mel_a = mel32;
  if (adt != DT_F32) {
    mel_a = arena_mat(ctx, adt, s0.R, 80);
    convert_mat(ctx, st, mel32, mel_a);
  }
  Mat xin = arena_mat(ctx, adt, s0.R, 512);
  {
    Epilogue e;
    e.act1 = ACT_LRELU;
    e.act1_param = 0.1f;
    e.row2seq = s0.d_row2seq;
    e.out = xin;
    conv_gemm(ctx, st, mel_a, m->conv_pre, e);
  }
  if (read_out(1, xin, s0, 512)) return Mat();
  const Seqs* sin_ = &s0;
  // ping-pong buffers for the activated level outputs, sized for the largest level (x120, 64 ch)
  const size_t lvl_elems = (size_t)g.lv[2].R * 64 > (size_t)g.lv[1].R * 128 ? (size_t)g.lv[2].R * 64 : (size_t)g.lv[1].R * 128;
  void* nxt_buf[2];
  nxt_buf[0] = ctx->arena.alloc(lvl_elems * (adt == DT_F32 ? 4 : 2));
  nxt_buf[1] = ctx->arena.alloc(lvl_elems * (adt == DT_F32 ? 4 : 2));
  for (int i = 0; i < 3; ++i) {
    const Seqs& sl = g.lv[i];
    const int C = kCh[i + 1];
    const size_t mark = ctx->arena.off;   // per-level scratch is released at the end of the level (stream-ordered reuse)
    // transposed conv (polyphase): [R_in, s*C] == [R_out, C]
    Mat xu_in(ctx->arena.alloc((size_t)sl.R * C * 4), DT_F32, sin_->R, kUps[i] * C, kUps[i] * C);
    {
      Epilogue e;
      e.row2seq = sin_->d_row2seq;
      e.out = xu_in;
      conv_gemm(ctx, st, xin, m->ups[i], e);
    }
    Mat xu(xu_in.p, DT_F32, sl.R, C, C);
    if (i == 2) {
      reflect_front_kernel<<<sl.B, 64, 0, st>>>(xu.f32(), xu.ld, C, sl.d_start);
      ctx->launches++;
      CVK_LAUNCH_CHECK();
    }
    if (read_out(2 + 6 * i, xu, sl, C)) return Mat();
    // source branch
    Mat si = arena_mat(ctx, DT_F32, sl.R, C);
    Mat a = arena_mat(ctx, adt, sl.R, C);
    Mat ya = arena_mat(ctx, adt, sl.R, C);
    Mat xr = arena_mat(ctx, DT_F32, sl.R, C);
    {
      const int ds[3] = {15, 3, 1};
      Mat view(stft.p, adt, s3.R / ds[i], ds[i] * kStftLd, ds[i] * kStftLd);
      Epilogue e;
      e.row2seq = sl.d_row2seq;
      e.out = si;
      e.act2 = ACT_SNAKE;
      e.alpha2 = m->src_rb[i].a1[0];
      e.out2 = a;
      conv_gemm(ctx, st, view, m->src_down[i], e);
    }
    run_resblock(ctx, st, m->src_rb[i], sl, si, a, ya, xr, xu, 1);   // xu += source_resblock(si)
    if (read_out(3 + 6 * i, xu, sl, C)) return Mat();
    // main resblocks, summed into xs
    Mat xs = arena_mat(ctx, DT_F32, sl.R, C);
    for (int j = 0; j < 3; ++j) {
      const ResBlockW& rb = m->rb[i * 3 + j];
      act_copy(ctx, st, xu, ACT_SNAKE, 0.f, rb.a1[0], sl.d_row2seq, a);
      run_resblock(ctx, st, rb, sl, xu, a, ya, xr, xs, j > 0);
      if (read_out(4 + 6 * i + j, xs, sl, C)) return Mat();
    }
    // x = xs / 3 ; leaky_relu (0.1 before the next ups, default 0.01 before conv_post, generator.py:513,532)
    Mat nxt(nxt_buf[i & 1], adt, sl.R, C, C);
    act_copy_scaled(ctx, st, xs, 1.f / 3.f, ACT_LRELU, i < 2 ? 0.1f : 0.01f, nullptr, sl.d_row2seq, nxt);
    if (read_out(7 + 6 * i, nxt, sl, C)) return Mat();
    xin = nxt;
    sin_ = &sl;
    ctx->arena.off = mark;
  }
  Mat xp = arena_mat(ctx, DT_F32, s3.R, 18, kStftLd);
  {
    Epilogue e;
    e.row2seq = s3.d_row2seq;
    e.out = xp;
    conv_gemm(ctx, st, xin, m->conv_post, e);
  }
  if (read_out(20, xp, s3, 18)) return Mat();
  return xp;
}

// lens: frames per utterance that define the OUTPUT offsets (sum 480*lens samples); d_drop_tail[b] samples at the end of utterance
// b are not written (device array; nullptr = none, 480 for a CosyVoice3 streaming utterance)
static void hift_istft(cvk_ctx* ctx, cudaStream_t st, const HiftGeom& g, const int* lens, const Mat& xp, float* wav_dense,
                       const int* d_drop_tail = nullptr) {
  const Seqs& s0 = g.s0;
  int* ooff = upload_ints(ctx, prefix_offsets(lens, s0.B), st);
  int bx = ceil_div(s0.max_len * kUpscale, 512);
  istft16_kernel<<<dim3(bx, s0.B), 128, 0, st>>>(xp.f32(), xp.ld, g.lv[2].d_start, s0.d_len, ooff, wav_dense, 0.99f, d_drop_tail);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}

__global__ void gather_f0_kernel(const float* __restrict__ f0, int ld, const int* __restrict__ start, const int* __restrict__ len,
                                 const int* __restrict__ off, float* __restrict__ out) {
  int b = blockIdx.y;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < len[b]; t += gridDim.x * blockDim.x) out[off[b] + t] = f0[(size_t)(start[b] + t) * ld];
}
__global__ void scatter_f0_kernel(const float* __restrict__ in, const int* __restrict__ start, const int* __restrict__ len,
                                  const int* __restrict__ off, float* __restrict__ f0, int ld) {
  int b = blockIdx.y;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < len[b]; t += gridDim.x * blockDim.x) f0[(size_t)(start[b] + t) * ld] = in[off[b] + t];
}
__global__ void copy_samples_kernel(const float* __restrict__ in, float* __restrict__ out, const int* __restrict__ start,
                                    const int* __restrict__ len, const int* __restrict__ off, int to_packed) {
  int b = blockIdx.y;
  int L = len[b] * kUpscale;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < L; i += gridDim.x * blockDim.x) {
    size_t pi = (size_t)start[b] * kUpscale + i, di = (size_t)off[b] * kUpscale + i;
    if (to_packed) out[pi] = in[di];
    else out[di] = in[pi];
  }
}

static Mat pack_mel(cvk_ctx* ctx, cudaStream_t st, const Seqs& s0, const float* mel) {
  Mat mel32 = arena_mat(ctx, DT_F32, s0.R, 80);
  zero_mat(ctx, st, mel32);
  pack_rows(ctx, st, mel, 80, s0, mel32);
  return mel32;
}

// ================================================================================================ entry points (called from api.cu)
void hift_f0(cvk_ctx* ctx, const float* mel, const int* lens, int B, float* f0_out, cudaStream_t st) {
  CVK_REQUIRE(ctx->hift, "hift stage not finalised");
  ctx->arena.reset();
  Seqs s0 = make_seqs(ctx, lens, B, 8, 1, 0, st);
  Mat mel32 = pack_mel(ctx, st, s0, mel);
  Mat f0 = arena_mat(ctx, DT_F32, s0.R, 1, 1);
  hift_f0_packed(ctx, st, s0, mel32, f0);
  int* off = upload_ints(ctx, prefix_offsets(lens, B), st);
  gather_f0_kernel<<<dim3(ceil_div(s0.max_len, 128), B), 128, 0, st>>>(f0.f32(), 1, s0.d_start, s0.d_len, off, f0_out);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}

void hift_source(cvk_ctx* ctx, const float* f0_dense, const int* lens, int B, const float* noise, float* source_out, cudaStream_t st) {
  CVK_REQUIRE(ctx->hift, "hift stage not finalised");
  ctx->arena.reset();
  Seqs s0 = make_seqs(ctx, lens, B, 8, 1, 0, st);
  Mat f0 = arena_mat(ctx, DT_F32, s0.R, 1, 1);
  zero_mat(ctx, st, f0);
  int* off = upload_ints(ctx, prefix_offsets(lens, B), st);
  scatter_f0_kernel<<<dim3(ceil_div(s0.max_len, 128), B), 128, 0, st>>>(f0_dense, s0.d_start, s0.d_len, off, f0.f32(), 1);
  ctx->launches++;
  float* src = (float*)ctx->arena.alloc(sizeof(float) * (size_t)s0.R * kUpscale);
  hift_source_packed(ctx, st, s0, lens, f0, noise, src);
  copy_samples_kernel<<<dim3(256, B), 256, 0, st>>>(src, source_out, s0.d_start, s0.d_len, off, 0);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
}

// unit / hidden: cvk_hift_hidden's read-out instead of the waveform (hift_body)
void hift_decode(cvk_ctx* ctx, const float* mel, const int* lens, int B, const float* source, float* wav, cudaStream_t st, int unit,
                 float* hidden) {
  CVK_REQUIRE(ctx->hift, "hift stage not finalised");
  ctx->arena.reset();
  HiftGeom g = hift_geom(ctx, lens, B, st);
  Mat mel32 = pack_mel(ctx, st, g.s0, mel);
  float* src = (float*)ctx->arena.alloc(sizeof(float) * (size_t)g.s0.R * kUpscale);
  CVK_CHECK_CUDA(cudaMemsetAsync(src, 0, sizeof(float) * (size_t)g.s0.R * kUpscale, st));
  int* off = upload_ints(ctx, prefix_offsets(lens, B), st);
  copy_samples_kernel<<<dim3(256, B), 256, 0, st>>>(source, src, g.s0.d_start, g.s0.d_len, off, 1);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  Mat xp = hift_body(ctx, st, g, mel32, src, nullptr, nullptr, unit, hidden);
  if (hidden) return;
  hift_istft(ctx, st, g, lens, xp, wav);
}

void hift_inference(cvk_ctx* ctx, const float* mel, const int* lens, int B, const float* noise, const float* cache_source,
                    const int* cache_lens, float* wav, float* source_out, cudaStream_t st) {
  CVK_REQUIRE(ctx->hift, "hift stage not finalised");
  ctx->arena.reset();
  HiftGeom g = hift_geom(ctx, lens, B, st);
  Mat mel32 = pack_mel(ctx, st, g.s0, mel);
  Mat f0 = arena_mat(ctx, DT_F32, g.s0.R, 1, 1);
  hift_f0_packed(ctx, st, g.s0, mel32, f0);
  float* src = (float*)ctx->arena.alloc(sizeof(float) * (size_t)g.s0.R * kUpscale);
  hift_source_packed(ctx, st, g.s0, lens, f0, noise, src);
  int* off = upload_ints(ctx, prefix_offsets(lens, B), st);
  if (cache_source && cache_lens) {
    std::vector<int> cl(cache_lens, cache_lens + B);
    int mx = 0;
    for (int b = 0; b < B; ++b) {
      CVK_REQUIRE(cl[b] <= lens[b] * kUpscale, "cache_source longer than the utterance");
      if (cl[b] > mx) mx = cl[b];
    }
    if (mx > 0) {
      int* coff = upload_ints(ctx, prefix_offsets(cache_lens, B), st);
      int* clen = upload_ints(ctx, cl, st);
      cache_source_kernel<<<dim3(ceil_div(mx, 256), B), 256, 0, st>>>(cache_source, coff, clen, g.s0.d_start, src);
      ctx->launches++;
      CVK_LAUNCH_CHECK();
    }
  }
  if (source_out) {
    copy_samples_kernel<<<dim3(256, B), 256, 0, st>>>(src, source_out, g.s0.d_start, g.s0.d_len, off, 0);
    ctx->launches++;
    CVK_LAUNCH_CHECK();
  }
  Mat xp = hift_body(ctx, st, g, mel32, src);
  hift_istft(ctx, st, g, lens, xp, wav);
}


// ================================================================================================ CosyVoice3 causal vocoder
// cosyvoice/hifigan/generator.py:572-726 (CausalHiFTGenerator), f0_predictor.py:60-103 (CausalConvRNNF0Predictor, float64 per
// generator.py:716-717), convolution.py:150-258 (causal convolutions), the causal branches of SineGen2 / SourceModuleHnNSF.
// The vocoder BODY is the CosyVoice2 one with different weights: every centred convolution becomes a left-padded one (a different
// row shift of the same conv-GEMM), conv_pre looks 4 frames to the right, the transposed convolutions become nearest-neighbour
// up-sampling + causal convolution (again a 3-tap polyphase conv-GEMM whose [R, u*C] output is the next level's [u*R, C]), and
// the strided source_downs pad left only.  The f0 predictor runs in float64 on the fp64 tensor cores (a few GFLOP per utterance;
// the reference insists on float64 so that streaming and offline f0 agree), the harmonic source uses nearest-neighbour phase
// up-sampling and the module's stored uniform noise instead of fresh Gaussian draws.
namespace {

struct F64Conv {
  double* w = nullptr;      // [taps][K][N]  (n fastest: 16-byte cp.async rows of the kernel's weight slabs)
  double* bias = nullptr;   // [N]
  int N = 0, K = 0, taps = 0, shift0 = 0;
};
struct Hift3Extra {
  F64Conv conv[5];
  double* cls_w = nullptr;  // [512]
  double cls_b = 0.0;
  float* rand_ini = nullptr;    // [9]  (SineGen2.rand_ini; without effect for upsample_scale 480, kept for the interface)
  float* noise = nullptr;       // [n][9]  SineGen2.sine_waves
  long long noise_n = 0;
};

__device__ __forceinline__ int floor_div(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// nn.Upsample(nearest, u) + left pad k-1 + Conv1d(k)  ==  3-tap polyphase conv on the un-upsampled input:
//   out[u m + p, co] = sum_{jt<3} sum_ci x[m + jt - 2, ci] * W[p][co][jt][ci],  W[p][co][jt] = sum_{j: floor((p-k+1+j)/u) == jt-2} w[co][ci][j]
__global__ void upsample_causal_poly_kernel(const float* __restrict__ w /*[Cout][Cin][k]*/, float* __restrict__ o /*[u*Cout][3][Cin]*/,
                                            int Cin, int Cout, int k, int u) {
  const size_t total = (size_t)u * Cout * 3 * Cin;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int ci = (int)(i % Cin);
    const int jt = (int)((i / Cin) % 3);
    const int n = (int)(i / ((size_t)Cin * 3));
    const int p = n / Cout, co = n % Cout;
    float acc = 0.f;
    for (int j = 0; j < k; ++j)
      if (floor_div(p - (k - 1) + j, u) == jt - 2) acc += w[((size_t)co * Cin + ci) * k + j];
    o[i] = acc;
  }
}

// weight norm folded in float64, as the reference's float64 predictor module computes it (generator.py:716-717 converts the module,
// so its parametrization runs in double): g [N], v [N][K][taps] fp32 -> w = g v / ||v|| as [taps][K][N] fp64.  One block per n.
__global__ void f64_weight_norm_kernel(const float* __restrict__ g, const float* __restrict__ v, double* __restrict__ o, int N, int K,
                                       int taps) {
  __shared__ double red[32];
  const int n = blockIdx.x, inner = K * taps;
  const float* vp = v + (size_t)n * inner;
  double s = 0.0;
  for (int i = threadIdx.x; i < inner; i += blockDim.x) s += (double)vp[i] * (double)vp[i];
  for (int o2 = 16; o2 > 0; o2 >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o2);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  double tot = 0.0;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
  const double scale = (double)g[n] / sqrt(tot);
  for (int i = threadIdx.x; i < inner; i += blockDim.x) {
    const int k = i / taps, j = i % taps;
    o[((size_t)j * K + k) * N + n] = (double)vp[i] * scale;
  }
}
__global__ void f64_copy_kernel(const float* __restrict__ a, double* __restrict__ o, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) o[i] = (double)a[i];
}

// f0 predictor convolution on the fp64 tensor cores (mma.sync m16n8k8 f64, SASS DMMA.16x8x8):
//   out[r, n] = ELU(bias[n] + sum_j sum_k A[r + shift0 + j, k] * w[j][k][n])
// One CTA computes an F0_BM x F0_BN output tile.  Per F0_BK-wide K slab it stages the tile's A rows plus the taps-1 halo rows
// once (tap j reads them at row offset j) and the taps' F0_BK x F0_BN weight slabs, in a cp.async ring of F0Stages slabs, so
// the weights are read once per row tile.  Every output sums its products in the same (slab, tap, k) order whatever tile or
// row it sits in, with no split-K, and rows outside [0, rows) read as zero like the zero gap rows between sequences: an
// utterance's f0 is bit-identical alone, in any ragged batch and as the prefix of a streaming call (the reason the reference
// runs this predictor in float64).  Rows outside every sequence (row2seq < 0) are written as zero: they are the zero padding
// (gap rows, streaming look-ahead rows) of the next layer.
constexpr int F0_BM = 128, F0_BN = 128, F0_BK = 16, F0_THREADS = 256;
constexpr int F0_LDA = F0_BK + 4, F0_LDW = F0_BN + 4;   // pitches of 4 mod 16 doubles: conflict-free fragment loads
template <int TAPS> struct F0Tile {
  static constexpr int kStages = TAPS == 3 ? 3 : 2;
  static constexpr int kArows = F0_BM + TAPS - 1;
  static constexpr int kStage = kArows * F0_LDA + TAPS * F0_BK * F0_LDW;   // doubles per stage (even: 16-byte aligned)
  static constexpr size_t kSmem = (size_t)kStages * kStage * sizeof(double);
};

__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool ok) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(ok ? 16 : 0) : "memory");
}
__device__ __forceinline__ void dmma16x8x8(double (&c)[4], const double (&a)[4], const double (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
               : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}

// A [rows][K], w [TAPS][K][N], out [rows][N]; K % F0_BK == 0, N % F0_BN == 0.  Grid (N / F0_BN, ceil(rows / F0_BM)): the
// column tiles of one row tile run side by side and share its A rows in L2.
template <int TAPS>
__global__ void __launch_bounds__(F0_THREADS, 1)
f0_conv_dmma_kernel(const double* __restrict__ A, int K, const double* __restrict__ w, const double* __restrict__ bias, int N, int shift0,
                    int rows, const int* __restrict__ row2seq, double* __restrict__ out) {
  using T = F0Tile<TAPS>;
  extern __shared__ __align__(16) double f0_smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int wm = (warp >> 2) * 64, wn = (warp & 3) * 32;     // 2 x 4 warps, 64 x 32 each
  const int n0 = blockIdx.x * F0_BN, r0 = blockIdx.y * F0_BM;
  const int nk = K / F0_BK;

  auto load = [&](int ks, int s) {
    double* sa = f0_smem + (size_t)s * T::kStage;
    double* sw = sa + T::kArows * F0_LDA;
    const int k0 = ks * F0_BK;
    for (int c = tid; c < T::kArows * (F0_BK / 2); c += F0_THREADS) {
      const int i = c / (F0_BK / 2), q = c % (F0_BK / 2);
      const int rr = r0 + shift0 + i;
      const bool ok = rr >= 0 && rr < rows;
      cp_async16(sa + i * F0_LDA + 2 * q, ok ? A + (size_t)rr * K + k0 + 2 * q : A, ok);
    }
    for (int c = tid; c < TAPS * F0_BK * (F0_BN / 2); c += F0_THREADS) {
      const int q = c % (F0_BN / 2), kk = (c / (F0_BN / 2)) % F0_BK, j = c / (F0_BK * (F0_BN / 2));
      cp_async16(sw + (j * F0_BK + kk) * F0_LDW + 2 * q, w + ((size_t)j * K + k0 + kk) * N + n0 + 2 * q, true);
    }
  };

  double acc[4][4][4];
#pragma unroll
  for (int mt = 0; mt < 4; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.0;

#pragma unroll
  for (int s = 0; s < T::kStages - 1; ++s) {
    if (s < nk) load(s, s);
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  for (int ks = 0; ks < nk; ++ks) {
    asm volatile("cp.async.wait_group %0;" ::"n"(T::kStages - 2) : "memory");
    __syncthreads();                                        // slab ks landed for all threads; slab ks-1's buffer is free
    if (ks + T::kStages - 1 < nk) load(ks + T::kStages - 1, (ks + T::kStages - 1) % T::kStages);
    asm volatile("cp.async.commit_group;" ::: "memory");
    const double* sa = f0_smem + (size_t)(ks % T::kStages) * T::kStage;
    const double* sw = sa + T::kArows * F0_LDA;
#pragma unroll
    for (int j = 0; j < TAPS; ++j) {
#pragma unroll
      for (int kk = 0; kk < F0_BK; kk += 8) {
        double a[4][4], b[4][2];
#pragma unroll
        for (int mt = 0; mt < 4; ++mt) {
          const double* p = sa + (wm + mt * 16 + g + j) * F0_LDA + kk + t;
          a[mt][0] = p[0];
          a[mt][1] = p[8 * F0_LDA];
          a[mt][2] = p[4];
          a[mt][3] = p[8 * F0_LDA + 4];
        }
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const double* p = sw + (j * F0_BK + kk + t) * F0_LDW + wn + nt * 8 + g;
          b[nt][0] = p[0];
          b[nt][1] = p[4 * F0_LDW];
        }
#pragma unroll
        for (int mt = 0; mt < 4; ++mt)
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) dmma16x8x8(acc[mt][nt], a[mt], b[nt]);
      }
    }
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");

#pragma unroll
  for (int mt = 0; mt < 4; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r0 + wm + mt * 16 + g + 8 * h;
      if (r >= rows) continue;
      const bool valid = row2seq[r] >= 0;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const int n = n0 + wn + nt * 8 + 2 * t;
        double2 v = make_double2(0.0, 0.0);
        if (valid) {
          v.x = acc[mt][nt][2 * h] + bias[n];
          v.y = acc[mt][nt][2 * h + 1] + bias[n + 1];
          v.x = v.x > 0.0 ? v.x : expm1(v.x);
          v.y = v.y > 0.0 ? v.y : expm1(v.y);
        }
        *reinterpret_cast<double2*>(out + (size_t)r * N + n) = v;
      }
    }
}
// f0 = |x . w + b| (f0_predictor.py:103), written as float32
__global__ void f0_head_f64_kernel(const double* __restrict__ x, const double* __restrict__ w, double b, int rows, const int* __restrict__ row2seq,
                                   float* __restrict__ f0) {
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  double acc = 0.0;
  if (row2seq[r] >= 0)
    for (int k = lane; k < 512; k += 32) acc = fma(x[(size_t)r * 512 + k], w[k], acc);
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) f0[r] = row2seq[r] >= 0 ? (float)fabs(acc + b) : 0.f;
}

// causal SineGen2 + SourceModuleHnNSF (generator.py:255-261 nearest up-sampling of the phase, :303-307 stored noise, :358-366)
__global__ void source_causal_kernel(const float* __restrict__ f0, int f0_ld, const float* __restrict__ phase, const int* __restrict__ start,
                                     const int* __restrict__ len, const float* __restrict__ noise /*[n][9], indexed from the utterance start*/,
                                     const float* __restrict__ lw, const float* __restrict__ lb, float* __restrict__ src) {
  const int b = blockIdx.y;
  const int T = len[b], s0 = start[b];
  const int L = T * kUpscale;
  for (int l = blockIdx.x * blockDim.x + threadIdx.x; l < L; l += gridDim.x * blockDim.x) {
    const int t = l / kUpscale;
    const float f = f0[(size_t)(s0 + t) * f0_ld];
    const float uv = f > 10.f ? 1.f : 0.f;
    const float noise_amp = uv * 0.003f + (1.f - uv) * 0.1f / 3.f;
    const float* p0 = phase + (size_t)(s0 + t) * 9;
    const float* nz = noise + (size_t)l * 9;
    float acc = 0.f;
#pragma unroll
    for (int h = 0; h < 9; ++h) acc += ((sinf(p0[h]) * 0.1f) * uv + noise_amp * nz[h]) * lw[h];
    src[(size_t)s0 * kUpscale + l] = tanhf(acc + lb[0]);
  }
}

ResBlockW build_resblock_causal(cvk_ctx* ctx, const std::string& p, int k) {
  ResBlockW r;
  for (int i = 0; i < 3; ++i) {
    const int d = kDil[i];
    r.c1[i] = wn_conv(ctx, p + ".convs1." + std::to_string(i), d, -(k - 1) * d);     // left padding (k-1)*d (convolution.py:172)
    r.c2[i] = wn_conv(ctx, p + ".convs2." + std::to_string(i), 1, -(k - 1));
    r.a1[i] = dev_copy_f32(ctx, ctx->get_raw(p + ".activations1." + std::to_string(i) + ".alpha").p, r.c1[i].K);
    r.a2[i] = dev_copy_f32(ctx, ctx->get_raw(p + ".activations2." + std::to_string(i) + ".alpha").p, r.c1[i].K);
  }
  return r;
}

}  // namespace

void hift3_build(cvk_ctx* ctx) {
  init_consts();
  HiftModel* m = new HiftModel();
  m->half_weights = ctx->precision == CVK_PREC_BF16 && ctx->hift_f16;
  struct F16Scope { cvk_ctx* c; F16Scope(cvk_ctx* c_, bool on) : c(c_) { c->build_f16 = on; } ~F16Scope() { c->build_f16 = 0; } } f16scope(ctx, m->half_weights);
  Hift3Extra* x = ctx->hift3_extra ? (Hift3Extra*)ctx->hift3_extra : new Hift3Extra();
  const std::string P = "hift3.";
  // float64 f0 predictor: conv0 k4 looking RIGHT (f0_predictor.py:71), then four causal k3 convolutions
  for (int i = 0; i < 5; ++i) {
    const std::string pre = P + "f0_predictor.condnet." + std::to_string(2 * i);
    ConvW c = wn_conv(ctx, pre, 1, i == 0 ? 0 : -2);
    CVK_CHECK_CUDA(cudaDeviceSynchronize());
    F64Conv& f = x->conv[i];
    f.N = c.N; f.K = c.K; f.taps = c.taps; f.shift0 = c.shift0;
    CVK_REQUIRE(f.K % F0_BK == 0 && f.N % F0_BN == 0 && f.taps == (i == 0 ? 4 : 3), "unexpected f0 predictor convolution shape");
    f.w = (double*)ctx->dmalloc((size_t)c.N * c.taps * c.K * sizeof(double));
    f.bias = (double*)ctx->dmalloc((size_t)c.N * sizeof(double));
    const bool pz = ctx->has_raw(pre + ".parametrizations.weight.original0");
    const RawTensor& wg = ctx->get_raw(pre + (pz ? ".parametrizations.weight.original0" : ".weight_g"));
    const RawTensor& wv = ctx->get_raw(pre + (pz ? ".parametrizations.weight.original1" : ".weight_v"));
    f64_weight_norm_kernel<<<c.N, 256>>>(wg.p, wv.p, f.w, c.N, c.K, c.taps);
    f64_copy_kernel<<<4, 256>>>(c.bias, f.bias, (size_t)c.N);
    CVK_LAUNCH_CHECK();
  }
  {
    const RawTensor& w = ctx->get_raw(P + "f0_predictor.classifier.weight");
    const RawTensor& b = ctx->get_raw(P + "f0_predictor.classifier.bias");
    x->cls_w = (double*)ctx->dmalloc(512 * sizeof(double));
    f64_copy_kernel<<<2, 256>>>(w.p, x->cls_w, 512);
    CVK_LAUNCH_CHECK();
    float bh = 0.f;
    CVK_CHECK_CUDA(cudaMemcpy(&bh, b.p, sizeof(float), cudaMemcpyDeviceToHost));
    x->cls_b = (double)bh;
  }
  m->src_w = dev_copy_f32(ctx, ctx->get_raw(P + "m_source.l_linear.weight").p, 9);
  m->src_b = dev_copy_f32(ctx, ctx->get_raw(P + "m_source.l_linear.bias").p, 1);
  m->conv_pre = wn_conv(ctx, P + "conv_pre", 1, 0);          // k5, 4 frames of look-ahead (convolution.py:183-184 'right')
  m->conv_post = wn_conv(ctx, P + "conv_post", 1, -6);       // k7 causal
  for (int i = 0; i < 3; ++i) {
    const std::string pre = P + "ups." + std::to_string(i);
    float* w = fold_weight_norm(ctx, pre, nullptr);          // Conv1d layout [Cout][Cin][k]
    const int Cin = kCh[i], Cout = kCh[i + 1], k = kUpK[i], u = kUps[i];
    ConvW c;
    c.N = u * Cout; c.K = Cin; c.taps = 3; c.dil = 1; c.shift0 = -2;
    c.w32 = (float*)ctx->dmalloc((size_t)c.N * 3 * Cin * sizeof(float));
    upsample_causal_poly_kernel<<<256, 256>>>(w, c.w32, Cin, Cout, k, u);
    CVK_LAUNCH_CHECK();
    c.bias = (float*)ctx->dmalloc((size_t)c.N * sizeof(float));
    repeat_bias_kernel<<<ceil_div(c.N, 256), 256>>>(ctx->get_raw(pre + ".bias").p, c.bias, Cout, u);
    CVK_LAUNCH_CHECK();
    finish_convw(ctx, c);
    m->ups[i] = c;
  }
  {
    // CausalConv1dDownSample(k = 2*stride, stride): left pad stride-1 -> STFT frame stride*r - (stride-1) + j for tap j
    const int ds[3] = {15, 3, 1}, dk[3] = {30, 6, 1};
    for (int i = 0; i < 3; ++i) {
      const std::string pre = P + "source_downs." + std::to_string(i);
      const RawTensor& w = ctx->get_raw(pre + ".weight");
      const int N = (int)w.shape[0], C = (int)w.shape[1], k = (int)w.shape[2];
      CVK_REQUIRE(C == 18 && k == dk[i] && N == kCh[i + 1], "unexpected source_downs shape");
      ConvW c;
      c.N = N;
      c.bias = dev_copy_f32(ctx, ctx->get_raw(pre + ".bias").p, N);
      if (ds[i] == 1) {
        c.K = kStftLd; c.taps = 1; c.dil = 1; c.shift0 = 0;
        c.w32 = (float*)ctx->dmalloc((size_t)N * kStftLd * sizeof(float));
        CVK_CHECK_CUDA(cudaMemset(c.w32, 0, (size_t)N * kStftLd * sizeof(float)));
        CVK_CHECK_CUDA(cudaMemcpy2D(c.w32, kStftLd * sizeof(float), w.p, 18 * sizeof(float), 18 * sizeof(float), N, cudaMemcpyDeviceToDevice));
      } else {
        c.K = ds[i] * kStftLd; c.taps = 3; c.dil = 1; c.shift0 = -1;
        const size_t n = (size_t)N * 3 * c.K;
        c.w32 = (float*)ctx->dmalloc(n * sizeof(float));
        CVK_CHECK_CUDA(cudaMemset(c.w32, 0, n * sizeof(float)));
        strided_view_fill_kernel<<<64, 256>>>(w.p, c.w32, N, C, k, ds[i], ds[i]);   // level-3 row = s*r + j - ((s-1) + 1)
        CVK_LAUNCH_CHECK();
      }
      finish_convw(ctx, c);
      m->src_down[i] = c;
    }
  }
  for (int i = 0; i < 3; ++i) m->src_rb[i] = build_resblock_causal(ctx, P + "source_resblocks." + std::to_string(i), kSrcRbK[i]);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) m->rb[i * 3 + j] = build_resblock_causal(ctx, P + "resblocks." + std::to_string(i * 3 + j), kRbK[j]);
  CVK_CHECK_CUDA(cudaDeviceSynchronize());
  ctx->hift3 = m;
  ctx->hift3_extra = x;
}

void hift3_setup() {
  CVK_CHECK_CUDA(cudaFuncSetAttribute(f0_conv_dmma_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)F0Tile<3>::kSmem));
  CVK_CHECK_CUDA(cudaFuncSetAttribute(f0_conv_dmma_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)F0Tile<4>::kSmem));
}

// SineGen2.rand_ini [9] and SineGen2.sine_waves [n][9] (generator.py:223-226): module attributes, not state_dict entries
void hift3_set_noise(cvk_ctx* ctx, const float* rand_ini, const float* sine_noise, long long n, int on_device) {
  Hift3Extra* x = ctx->hift3_extra ? (Hift3Extra*)ctx->hift3_extra : new Hift3Extra();
  const cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  x->rand_ini = (float*)ctx->dmalloc(9 * sizeof(float));
  CVK_CHECK_CUDA(cudaMemcpy(x->rand_ini, rand_ini, 9 * sizeof(float), kind));
  x->noise = (float*)ctx->dmalloc((size_t)n * 9 * sizeof(float));
  CVK_CHECK_CUDA(cudaMemcpy(x->noise, sine_noise, (size_t)n * 9 * sizeof(float), kind));
  x->noise_n = n;
  ctx->hift3_extra = x;
}

// generator.py:714-726 with a finalize flag per utterance.  mel dense [sum T, 80]; utterance b's outputs, back to back:
// finalize[b] != 0: wav 480 T, f0_out T, source_out 480 T (f0_out / source_out optional);
// finalize[b] == 0 (streaming): wav 480 (T-8), f0_out T-3, source_out 480 (T-3).
// unit / hidden: cvk_hift_hidden's read-out instead of the waveform (hift_body)
void hift3_inference(cvk_ctx* ctx, const float* mel, const int* lens, const int* finalize, int B, float* wav, float* f0_out,
                     float* source_out, cudaStream_t st, int unit, float* hidden) {
  const HiftModel* m = ctx->hift3;
  Hift3Extra* x = (Hift3Extra*)ctx->hift3_extra;
  CVK_REQUIRE(m && x && x->conv[0].w, "hift3 stage not finalised");
  CVK_REQUIRE(x->noise != nullptr, "cvk_hift3_set_noise has not been called");
  // Geometry.  A final utterance has one geometry of T frames.  A streaming utterance (generator.py:676-683, 709-710, 722-725;
  // f0_predictor.py:99-100): the f0 predictor consumes 3 frames of look-ahead (f0 / source have T-3 frames), conv_pre 4 more
  // (the body runs on T-7 frames, the source STFT is cut to its first 120(T-7)+1 frames) and the last 480 samples are dropped
  // (480(T-8) returned).  All geometries share the row starts of the T-frame one, so the look-ahead rows are simply read by the
  // right-looking convs, and each utterance's look-ahead is its own: one call serves streaming and final utterances together.
  std::vector<int> la_f0(B), la_body(B), drop(B), lens_src(B), lens_out(B);
  bool any_stream = false;
  for (int b = 0; b < B; ++b) {
    const bool fin = finalize[b] != 0;
    CVK_REQUIRE(lens[b] > 0, "cvk_hift3_inference: an utterance of 0 mel frames");
    CVK_REQUIRE(fin || lens[b] >= 9, "cvk_hift3_inference: a streaming utterance needs at least 9 mel frames");
    any_stream |= !fin;
    la_f0[b] = fin ? 0 : 3;
    la_body[b] = fin ? 0 : 3 + 4;
    drop[b] = fin ? 0 : kUpscale;
    lens_src[b] = lens[b] - la_f0[b];
    lens_out[b] = fin ? lens[b] : lens[b] - 8;
    CVK_REQUIRE((long long)lens_src[b] * kUpscale <= x->noise_n, "stored source noise shorter than the utterance");
  }
  ctx->arena.reset();
  HiftGeom g;
  Seqs sF = make_seqs(ctx, lens, B, 8, 1, 0, st);                             // all frames
  Seqs s0 = any_stream ? shrink_seqs(ctx, sF, la_f0.data(), st) : sF;         // f0 / source frames
  g.s0 = any_stream ? shrink_seqs(ctx, sF, la_body.data(), st) : sF;          // body frames
  g.lv[0] = scale_seqs(ctx, g.s0, 8, 0, st);
  g.lv[1] = scale_seqs(ctx, g.s0, 40, 0, st);
  g.lv[2] = scale_seqs(ctx, g.s0, 120, 1, st);
  Mat mel32 = pack_mel(ctx, st, sF, mel);
  // ---- f0 predictor in float64
  double* a = (double*)ctx->arena.alloc(sizeof(double) * (size_t)s0.R * 512);
  double* bb = (double*)ctx->arena.alloc(sizeof(double) * (size_t)s0.R * 512);
  double* mel64 = (double*)ctx->arena.alloc(sizeof(double) * (size_t)s0.R * 80);
  f64_copy_kernel<<<256, 256, 0, st>>>(mel32.f32(), mel64, (size_t)s0.R * 80);
  ctx->launches++;
  CVK_REQUIRE(mel32.ld == 80, "packed mel must be dense");
  const double* cur = mel64;
  for (int i = 0; i < 5; ++i) {
    const F64Conv& f = x->conv[i];
    double* o = (i & 1) ? bb : a;
    const dim3 grid(f.N / F0_BN, ceil_div(s0.R, F0_BM));
    if (f.taps == 4)
      f0_conv_dmma_kernel<4><<<grid, F0_THREADS, F0Tile<4>::kSmem, st>>>(cur, f.K, f.w, f.bias, f.N, f.shift0, s0.R, s0.d_row2seq, o);
    else
      f0_conv_dmma_kernel<3><<<grid, F0_THREADS, F0Tile<3>::kSmem, st>>>(cur, f.K, f.w, f.bias, f.N, f.shift0, s0.R, s0.d_row2seq, o);
    ctx->launches++;
    CVK_LAUNCH_CHECK();
    cur = o;
  }
  Mat f0 = arena_mat(ctx, DT_F32, s0.R, 1, 1);
  f0_head_f64_kernel<<<ceil_div(s0.R, 4), 128, 0, st>>>(cur, x->cls_w, x->cls_b, s0.R, s0.d_row2seq, f0.f32());
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  int* off = upload_ints(ctx, prefix_offsets(lens_src.data(), B), st);
  if (f0_out) {
    gather_f0_kernel<<<dim3(ceil_div(s0.max_len, 128), B), 128, 0, st>>>(f0.f32(), 1, s0.d_start, s0.d_len, off, f0_out);
    ctx->launches++;
    CVK_LAUNCH_CHECK();
  }
  // ---- harmonic source
  float* phase = (float*)ctx->arena.alloc(sizeof(float) * 9 * (size_t)s0.R);
  phase_kernel<<<s0.B, 32, 0, st>>>(f0.f32(), f0.ld, s0.d_start, s0.d_len, phase);
  float* src = (float*)ctx->arena.alloc(sizeof(float) * (size_t)s0.R * kUpscale);
  CVK_CHECK_CUDA(cudaMemsetAsync(src, 0, sizeof(float) * (size_t)s0.R * kUpscale, st));
  {
    int bx = ceil_div(s0.max_len * kUpscale, 256);
    if (bx > 512) bx = 512;
    source_causal_kernel<<<dim3(bx, s0.B), 256, 0, st>>>(f0.f32(), f0.ld, phase, s0.d_start, s0.d_len, x->noise, m->src_w, m->src_b, src);
  }
  ctx->launches += 2;
  CVK_LAUNCH_CHECK();
  if (source_out) {
    copy_samples_kernel<<<dim3(256, B), 256, 0, st>>>(src, source_out, s0.d_start, s0.d_len, off, 0);
    ctx->launches++;
    CVK_LAUNCH_CHECK();
  }
  // ---- vocoder body (shared with CosyVoice2) + ISTFT
  // per utterance: the source length the STFT reads and the samples the ISTFT drops (nullptr when every utterance is final)
  Mat xp = hift_body(ctx, st, g, mel32, src, m, any_stream ? s0.d_len : nullptr, unit, hidden);
  if (hidden) return;
  hift_istft(ctx, st, g, lens_out.data(), xp, wav, any_stream ? upload_ints(ctx, drop, st) : nullptr);
}
