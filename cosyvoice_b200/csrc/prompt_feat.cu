// Prompt-side acoustic features of the reference frontend on the GPU (SURVEY.md 8(f) rank 2: the step right before the hot path,
// CPU / single-threaded in the reference):
//
//  * whisper log-mel (cosyvoice/cli/frontend.py:95-98 -> whisper.log_mel_spectrogram(speech, n_mels=128), openai-whisper audio.py):
//    16 kHz, hann(400) periodic, n_fft 400, hop 160, center=True (reflect pad 200), |X|^2 of all frames but the last, 128-band
//    Slaney mel filterbank (librosa.filters.mel(sr=16000, n_fft=400, n_mels=128) = whisper's mel_filters.npz), log10(max(., 1e-10)),
//    floor at (utterance maximum - 8), (x + 4) / 4.
//  * kaldi fbank (frontend.py:108-113 -> torchaudio.compliance.kaldi.fbank(speech, num_mel_bins=80, dither=0,
//    sample_frequency=16000) and `feat - feat.mean(dim=0)`): 25 ms / 10 ms frames with snip_edges, per-frame DC removal,
//    pre-emphasis 0.97 (first sample against itself), povey window (hann(400, symmetric)^0.85), zero-padded 512-point power
//    spectrum, 80 triangular filters on the kaldi mel scale (1127 ln(1 + f/700)) between 20 Hz and Nyquist, log(max(., FLT_EPSILON)).
//
// Both are hop-160 framings of a 400-sample window: the signal viewed as rows of 160 samples makes a frame three consecutive rows
// (480 samples, the last 80 weighted by zero), so framing + window + DFT is ONE 3-tap conv-GEMM against a constant matrix - and
// for kaldi the per-frame DC removal and pre-emphasis, both linear in the frame, are folded into that matrix as well
// (M = DFT . diag(window) . P . (I - 11^T/400), built in double).  The speech tokenizer and the CAM++ speaker network that consume
// these features are opaque ONNX files outside the repository and stay with onnxruntime.
#include "common.cuh"
#include <math.h>

namespace {
constexpr int HOP = 160, WIN = 400, SR = 16000;
constexpr double PI = 3.14159265358979323846;
// whisper
constexpr int W_BINS = 201, W_MEL = 128, W_PAD = 200;
// kaldi
constexpr int K_FFT = 512, K_BINS = 257, K_MEL = 80;

struct PromptFeatModel {
  ConvW w_dft;    // [2*201][3][160]
  ConvW w_mel;    // [128][201]
  ConvW k_dft;    // [2*257][3][160]
  ConvW k_mel;    // [80][257]
};

// reflect-padded (pad 200 on both sides, torch.stft center=True) signal as rows of 160; only the (frames + 2) rows the kept frames
// read are written.  pad == 0: plain copy (kaldi, snip_edges).
__global__ void rows160_kernel(const float* __restrict__ wav, const int* __restrict__ off, const int* __restrict__ nsamp,
                               const int* __restrict__ start, const int* __restrict__ nrows, int pad, float* __restrict__ out) {
  const int b = blockIdx.y;
  const int N = nsamp[b];
  const int total = nrows[b] * HOP;
  const float* x = wav + off[b];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    int m = i - pad;
    if (m < 0) m = -m;
    if (m >= N) m = pad ? 2 * (N - 1) - m : -1;
    out[(size_t)start[b] * HOP + i] = (m >= 0 && m < N) ? x[m] : 0.f;
  }
}

__global__ void power_kernel(const float* __restrict__ spec, int lds, int rows, int bins, float* __restrict__ pw, int ldp) {
  size_t total = (size_t)rows * bins;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int r = i / bins, k = i % bins;
    float re = spec[(size_t)r * lds + k], im = spec[(size_t)r * lds + bins + k];
    pw[(size_t)r * ldp + k] = re * re + im * im;
  }
}

// whisper: x = log10(max(x, 1e-10)); x = max(x, max_over_utterance(x) - 8); x = (x + 4) / 4.   One CTA per utterance.
__global__ void whisper_log_kernel(float* __restrict__ x, int ld, const int* __restrict__ start, const int* __restrict__ len) {
  __shared__ float red[32];
  const int b = blockIdx.x, s0 = start[b], L = len[b];
  const size_t total = (size_t)L * W_MEL;
  float mx = -INFINITY;
  for (size_t i = threadIdx.x; i < total; i += blockDim.x) {
    float* p = x + (size_t)(s0 + i / W_MEL) * ld + i % W_MEL;
    const float v = log10f(fmaxf(*p, 1e-10f));
    *p = v;
    mx = fmaxf(mx, v);
  }
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w) mx = fmaxf(mx, red[w]);
  const float floor_v = mx - 8.0f;
  for (size_t i = threadIdx.x; i < total; i += blockDim.x) {
    float* p = x + (size_t)(s0 + i / W_MEL) * ld + i % W_MEL;
    *p = (fmaxf(*p, floor_v) + 4.0f) / 4.0f;
  }
}

// kaldi: x = log(max(x, FLT_EPSILON)); optionally minus the utterance's mean over frames (frontend.py:113).  One CTA per
// utterance, bin after bin: a column's sum runs over the frames in a fixed order per thread, then a tree over the threads.
__global__ void kaldi_log_cmn_kernel(float* __restrict__ x, int ld, const int* __restrict__ start, const int* __restrict__ len, int subtract_mean) {
  __shared__ float part[256];
  const int b = blockIdx.x, s0 = start[b], L = len[b];
  for (int c = 0; c < K_MEL; ++c) {
    float s = 0.f;
    for (int t = threadIdx.x; t < L; t += blockDim.x) {
      float* p = x + (size_t)(s0 + t) * ld + c;
      const float v = logf(fmaxf(*p, 1.1920928955078125e-07f));
      *p = v;
      s += v;
    }
    if (!subtract_mean) continue;
    part[threadIdx.x] = s;
    __syncthreads();
    for (int o = blockDim.x >> 1; o > 0; o >>= 1) {
      if ((int)threadIdx.x < o) part[threadIdx.x] += part[threadIdx.x + o];
      __syncthreads();
    }
    const float mean = part[0] / (float)L;
    __syncthreads();
    for (int t = threadIdx.x; t < L; t += blockDim.x) x[(size_t)(s0 + t) * ld + c] -= mean;
  }
}

double slaney_hz_to_mel(double f) {
  const double f_sp = 200.0 / 3, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = log(6.4) / 27.0;
  return f >= min_log_hz ? min_log_mel + log(f / min_log_hz) / logstep : f / f_sp;
}
double slaney_mel_to_hz(double m) {
  const double f_sp = 200.0 / 3, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = log(6.4) / 27.0;
  return m >= min_log_mel ? min_log_hz * exp(logstep * (m - min_log_mel)) : f_sp * m;
}

ConvW upload_w(cvk_ctx* ctx, const std::vector<float>& w, int N, int K, int taps) {
  ConvW c;
  c.N = N; c.K = K; c.taps = taps; c.dil = 1; c.shift0 = 0;
  c.w32 = (float*)ctx->dmalloc(w.size() * sizeof(float));
  CVK_CHECK_CUDA(cudaMemcpy(c.w32, w.data(), w.size() * sizeof(float), cudaMemcpyHostToDevice));
  return c;
}

PromptFeatModel* build(cvk_ctx* ctx) {
  PromptFeatModel* m = new PromptFeatModel();
  const int FR = 3 * HOP;     // 480 samples per frame view, the last 80 unused
  {   // whisper DFT: rows k2 < 201 -> hann[n] cos(2 pi k n / 400), else -hann[n] sin(.)
    std::vector<float> w((size_t)2 * W_BINS * FR, 0.f);
    for (int k2 = 0; k2 < 2 * W_BINS; ++k2) {
      const int k = k2 < W_BINS ? k2 : k2 - W_BINS;
      for (int n = 0; n < WIN; ++n) {
        const double win = 0.5 - 0.5 * cos(2.0 * PI * n / WIN);            // torch.hann_window(400), periodic
        const double ang = 2.0 * PI * (double)(((long long)k * n) % WIN) / WIN;
        w[(size_t)k2 * FR + n] = (float)(win * (k2 < W_BINS ? cos(ang) : -sin(ang)));
      }
    }
    m->w_dft = upload_w(ctx, w, 2 * W_BINS, HOP, 3);
  }
  {   // librosa.filters.mel(sr=16000, n_fft=400, n_mels=128): Slaney scale, Slaney (area) norm, fmin 0, fmax 8000
    std::vector<float> fb((size_t)W_MEL * W_BINS, 0.f);
    std::vector<double> mel_f(W_MEL + 2);
    const double m0 = slaney_hz_to_mel(0.0), m1 = slaney_hz_to_mel(SR / 2.0);
    for (int i = 0; i < W_MEL + 2; ++i) mel_f[i] = slaney_mel_to_hz(m0 + (m1 - m0) * i / (double)(W_MEL + 1));
    for (int i = 0; i < W_MEL; ++i) {
      const double enorm = 2.0 / (mel_f[i + 2] - mel_f[i]);
      for (int k = 0; k < W_BINS; ++k) {
        const double f = (double)SR / 2 * k / (double)(W_BINS - 1);
        const double lower = (f - mel_f[i]) / (mel_f[i + 1] - mel_f[i]), upper = (mel_f[i + 2] - f) / (mel_f[i + 2] - mel_f[i + 1]);
        const double v = lower < upper ? lower : upper;
        fb[(size_t)i * W_BINS + k] = (float)((v > 0 ? v : 0) * enorm);
      }
    }
    m->w_mel = upload_w(ctx, fb, W_MEL, W_BINS, 1);
  }
  {   // kaldi: rows of (DFT512 . diag(povey) . pre-emphasis . DC removal) over the 400 samples of a frame
    std::vector<float> w((size_t)2 * K_BINS * FR, 0.f);
    std::vector<double> r(WIN + 1), q(WIN);
    for (int k2 = 0; k2 < 2 * K_BINS; ++k2) {
      const int k = k2 < K_BINS ? k2 : k2 - K_BINS;
      for (int n = 0; n < WIN; ++n) {
        const double win = pow(0.5 - 0.5 * cos(2.0 * PI * n / (WIN - 1)), 0.85);     // povey: hann(400, periodic=False)^0.85
        const double ang = 2.0 * PI * (double)(((long long)k * n) % K_FFT) / K_FFT;
        r[n] = win * (k2 < K_BINS ? cos(ang) : -sin(ang));
      }
      r[WIN] = 0.0;
      // y[0] = x[0] - 0.97 x[0], y[j] = x[j] - 0.97 x[j-1]  =>  sum_j r[j] y[j] = sum_j x[j] (r[j] - 0.97 r[j+1]) - 0.97 r[0] x[0]
      double mean = 0.0;
      for (int j = 0; j < WIN; ++j) {
        q[j] = r[j] - 0.97 * r[j + 1];
        if (j == 0) q[j] -= 0.97 * r[0];
        mean += q[j];
      }
      mean /= WIN;
      for (int j = 0; j < WIN; ++j) w[(size_t)k2 * FR + j] = (float)(q[j] - mean);      // x - mean(x) first: (q . (I - 11^T/400))
    }
    m->k_dft = upload_w(ctx, w, 2 * K_BINS, HOP, 3);
  }
  {   // torchaudio.compliance.kaldi.get_mel_banks(80, 512, 16000, low 20, high 0 -> 8000): kaldi mel scale, no normalisation
    std::vector<float> fb((size_t)K_MEL * K_BINS, 0.f);
    auto mel = [](double f) { return 1127.0 * log(1.0 + f / 700.0); };
    const double bin_w = (double)SR / K_FFT, lo = mel(20.0), hi = mel(SR / 2.0), delta = (hi - lo) / (K_MEL + 1);
    for (int i = 0; i < K_MEL; ++i) {
      const double left = lo + i * delta, center = left + delta, right = center + delta;
      for (int k = 0; k < K_FFT / 2; ++k) {       // 256 bins; the Nyquist column stays zero (kaldi.py pads it)
        const double mk = mel(bin_w * k);
        const double up = (mk - left) / (center - left), down = (right - mk) / (right - center);
        const double v = up < down ? up : down;
        fb[(size_t)i * K_BINS + k] = (float)(v > 0 ? v : 0);
      }
    }
    m->k_mel = upload_w(ctx, fb, K_MEL, K_BINS, 1);
  }
  return m;      // every upload above is a blocking cudaMemcpy: nothing in flight, no device-wide synchronisation needed
}

// shared body: frames of 3 rows of 160 -> DFT conv-GEMM -> power -> filterbank; returns the [R, n_mel] matrix in geometry sf
Mat features(cvk_ctx* ctx, cudaStream_t st, const float* wav, const int* lens, const std::vector<int>& frames, int B, int pad, const ConvW& dft,
             int bins, const ConvW& fbank, int n_mel, Seqs* sf_out) {
  std::vector<int> rows(B), off(B), ns(lens, lens + B);
  int acc = 0;
  for (int b = 0; b < B; ++b) {
    rows[b] = frames[b] + 2;
    off[b] = acc;
    acc += lens[b];
  }
  Seqs sr = make_seqs(ctx, rows.data(), B, 4, 1, 0, st);
  Seqs sf = shrink_seqs(ctx, sr, 2, st);
  auto up = [&](const std::vector<int>& v) {
    int* d = (int*)ctx->arena.alloc(sizeof(int) * B);
    CVK_CHECK_CUDA(cudaMemcpyAsync(d, v.data(), sizeof(int) * B, cudaMemcpyHostToDevice, st));
    return d;
  };
  int *d_off = up(off), *d_ns = up(ns), *d_rows = up(rows);
  Mat x = arena_mat(ctx, DT_F32, sr.R, HOP, HOP);
  zero_mat(ctx, st, x);
  rows160_kernel<<<dim3(64, B), 256, 0, st>>>(wav, d_off, d_ns, sr.d_start, d_rows, pad, x.f32());
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  Mat spec = arena_mat(ctx, DT_F32, sr.R, 2 * bins, round_up(2 * bins, 8));
  {
    Epilogue e;
    e.row2seq = sf.d_row2seq;
    e.out = spec;
    conv_gemm_simt(ctx, st, x, dft, e);
  }
  Mat pw = arena_mat(ctx, DT_F32, sr.R, bins, round_up(bins, 8));
  power_kernel<<<132 * 4, 256, 0, st>>>(spec.f32(), spec.ld, sr.R, bins, pw.f32(), pw.ld);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  Mat out = arena_mat(ctx, DT_F32, sr.R, n_mel, n_mel);
  {
    Epilogue e;
    e.out = out;
    conv_gemm_simt(ctx, st, pw, fbank, e);
  }
  *sf_out = sf;
  return out;
}

PromptFeatModel* model(cvk_ctx* ctx) {
  if (!ctx->prompt_feat_model) ctx->prompt_feat_model = build(ctx);
  return (PromptFeatModel*)ctx->prompt_feat_model;
}
}  // namespace

// cvk_finalize(ctx, "prompt"): build the constant matrices at set-up time (otherwise they are built by the first feature call)
void prompt_feat_init(cvk_ctx* ctx) { model(ctx); }

// wav: the utterances back to back (16 kHz, float), lens[b] samples each (> 200: reflect padding); out [sum lens[b]/160, 128]
// time-major (the reference's [1, 128, T] transposed)
void whisper_log_mel(cvk_ctx* ctx, const float* wav, const int* lens, int B, float* out, cudaStream_t st) {
  PromptFeatModel* m = model(ctx);
  ctx->arena.reset();
  std::vector<int> frames(B);
  for (int b = 0; b < B; ++b) {
    CVK_REQUIRE(lens[b] > W_PAD, "whisper_log_mel: reflect padding by 200 needs more than 200 samples (torch.stft raises as well)");
    frames[b] = lens[b] / HOP;                      // 1 + N / 160 frames of torch.stft(center=True), the last one dropped
    CVK_REQUIRE(frames[b] > 0, "whisper_log_mel: utterance shorter than one hop");
  }
  Seqs sf;
  Mat o = features(ctx, st, wav, lens, frames, B, W_PAD, m->w_dft, W_BINS, m->w_mel, W_MEL, &sf);
  whisper_log_kernel<<<B, 1024, 0, st>>>(o.f32(), o.ld, sf.d_start, sf.d_len);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  unpack_rows(ctx, st, o, sf, 0, out, W_MEL);
}

// out [sum (1 + (lens[b] - 400) / 160), 80]; subtract_mean: the frontend's per-utterance mean normalisation (frontend.py:113)
void kaldi_fbank80(cvk_ctx* ctx, const float* wav, const int* lens, int B, int subtract_mean, float* out, cudaStream_t st) {
  PromptFeatModel* m = model(ctx);
  ctx->arena.reset();
  std::vector<int> frames(B);
  for (int b = 0; b < B; ++b) {
    CVK_REQUIRE(lens[b] >= WIN, "kaldi_fbank80: utterance shorter than one 25 ms frame");
    frames[b] = 1 + (lens[b] - WIN) / HOP;          // snip_edges
  }
  Seqs sf;
  Mat o = features(ctx, st, wav, lens, frames, B, 0, m->k_dft, K_BINS, m->k_mel, K_MEL, &sf);
  kaldi_log_cmn_kernel<<<B, 256, 0, st>>>(o.f32(), o.ld, sf.d_start, sf.d_len, subtract_mean);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  unpack_rows(ctx, st, o, sf, 0, out, K_MEL);
}
