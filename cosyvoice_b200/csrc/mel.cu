// Mel-spectrogram frontend (prompt features): reflect pad -> framed windowed DFT (n_fft 1920, hop 480) -> magnitude
// -> 80-band Slaney mel filterbank -> log(clamp(., 1e-5)).
// Follows third_party/Matcha-TTS/matcha/utils/audio.py:45-82 with the feat_extractor parameters of
// examples/libritts/cosyvoice2/conf/cosyvoice2.yaml:150-158 (fmin 0, fmax 8000, center False).  The filterbank is
// librosa 0.10.2 filters.mel (htk=False, norm='slaney'), restated from its published algorithm (librosa is not
// vendored in the reference).
//
// hop 480 divides n_fft 1920, so the padded signal viewed as a [N/480 + 3, 480] matrix turns framing into a 4-tap
// "convolution" and the DFT into the conv-GEMM with a [1922][4][480] windowed cos/sin weight - no FFT plan, fp32.
#include "common.cuh"
#include <math.h>

namespace {
constexpr int N_FFT = 1920, HOP = 480, N_BINS = 961, N_MEL = 80, SR = 24000;
constexpr int PAD = (N_FFT - HOP) / 2;   // 720
constexpr int BINS_LD = 968;

struct MelModel {
  ConvW dft;    // [2*961][4][480]
  ConvW mel;    // [80][961], fmax 8000 (cosyvoice2.yaml:150-158)
  ConvW mel_nyq;  // [80][961], fmax = sr/2 (CosyVoice3: `fmax: null`, cosyvoice3.yaml:140-147)
};

__global__ void dft_weight_kernel(float* __restrict__ w) {
  // w[(k2)][j][c], k2 < 1922: k2 < 961 -> cos row k2, else -sin row (k2-961); sample n = 480*j + c
  size_t total = (size_t)2 * N_BINS * N_FFT;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int n = i % N_FFT;
    int k2 = i / N_FFT;
    int k = k2 < N_BINS ? k2 : k2 - N_BINS;
    int m = (int)(((long long)k * n) % N_FFT);
    double ang = 2.0 * 3.14159265358979323846 * (double)m / (double)N_FFT;
    double win = 0.5 - 0.5 * cos(2.0 * 3.14159265358979323846 * (double)n / (double)N_FFT);   // torch.hann_window (periodic)
    double v = k2 < N_BINS ? cos(ang) : -sin(ang);
    w[i] = (float)(win * v);
  }
}

// reflect-pad each utterance by 720 (about sample 0 and about its TRUE last sample, torch.nn.functional.pad(mode="reflect") on
// the whole signal, audio.py:70-72) and lay the first (N/480 + 3) * 480 padded samples out as rows of 480: the center=False
// framing of audio.py:74-86 uses exactly those (frame f = padded samples [480 f, 480 f + 1920))
__global__ void frame_rows_kernel(const float* __restrict__ wav, const int* __restrict__ off, const int* __restrict__ nsamp,
                                  const int* __restrict__ start, float* __restrict__ out) {
  int b = blockIdx.y;
  int N = nsamp[b];
  int total = (N / HOP + 3) * HOP;
  const float* x = wav + off[b];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    int m = i - PAD;
    if (m < 0) m = -m;
    if (m >= N) m = 2 * (N - 1) - m;
    out[(size_t)start[b] * HOP + i] = x[m];
  }
}

__global__ void magnitude_kernel(const float* __restrict__ spec, int lds, int rows, float* __restrict__ mag, int ldm) {
  size_t total = (size_t)rows * N_BINS;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int r = i / N_BINS, k = i % N_BINS;
    float re = spec[(size_t)r * lds + k], im = spec[(size_t)r * lds + N_BINS + k];
    mag[(size_t)r * ldm + k] = sqrtf(re * re + im * im + 1e-9f);
  }
}
__global__ void log_clamp_kernel(float* __restrict__ x, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) x[i] = logf(fmaxf(x[i], 1e-5f));
}

double hz_to_mel(double f) {
  const double f_sp = 200.0 / 3, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = log(6.4) / 27.0;
  return f >= min_log_hz ? min_log_mel + log(f / min_log_hz) / logstep : f / f_sp;
}
double mel_to_hz(double m) {
  const double f_sp = 200.0 / 3, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = log(6.4) / 27.0;
  return m >= min_log_mel ? min_log_hz * exp(logstep * (m - min_log_mel)) : f_sp * m;
}
}  // namespace

void mel_init(cvk_ctx* ctx) {
  if (ctx->mel_model) return;
  MelModel* m = new MelModel();
  m->dft.N = 2 * N_BINS; m->dft.K = HOP; m->dft.taps = 4; m->dft.dil = 1; m->dft.shift0 = 0;
  m->dft.w32 = (float*)ctx->dmalloc((size_t)2 * N_BINS * N_FFT * sizeof(float));
  dft_weight_kernel<<<512, 256>>>(m->dft.w32);
  CVK_LAUNCH_CHECK();
  // librosa.filters.mel(sr=24000, n_fft=1920, n_mels=80, fmin=0, fmax): Slaney scale, Slaney (area) norm
  auto filterbank = [&](double fmax_hz) {
    std::vector<float> fb((size_t)N_MEL * N_BINS, 0.f);
    std::vector<double> mel_f(N_MEL + 2);
    double m0 = hz_to_mel(0.0), m1 = hz_to_mel(fmax_hz);
    for (int i = 0; i < N_MEL + 2; ++i) mel_f[i] = mel_to_hz(m0 + (m1 - m0) * (double)i / (double)(N_MEL + 1));
    for (int i = 0; i < N_MEL; ++i) {
      double enorm = 2.0 / (mel_f[i + 2] - mel_f[i]);
      for (int k = 0; k < N_BINS; ++k) {
        double f = (double)SR / 2 * (double)k / (double)(N_BINS - 1);
        double lower = (f - mel_f[i]) / (mel_f[i + 1] - mel_f[i]);
        double upper = (mel_f[i + 2] - f) / (mel_f[i + 2] - mel_f[i + 1]);
        double w = lower < upper ? lower : upper;
        if (w < 0) w = 0;
        fb[(size_t)i * N_BINS + k] = (float)(w * enorm);
      }
    }
    ConvW w;
    w.N = N_MEL; w.K = N_BINS;
    w.w32 = (float*)ctx->dmalloc(fb.size() * sizeof(float));
    CVK_CHECK_CUDA(cudaMemcpy(w.w32, fb.data(), fb.size() * sizeof(float), cudaMemcpyHostToDevice));
    return w;
  };
  m->mel = filterbank(8000.0);
  m->mel_nyq = filterbank((double)SR / 2);
  CVK_CHECK_CUDA(cudaDeviceSynchronize());
  ctx->mel_model = m;
}

// fmax_hz: 8000 (CosyVoice2) or 0 / 12000 (= sr/2: the reference's `fmax: null`, CosyVoice3).  lens[b] >= 721 samples (reflect
// padding by 720 needs more than 720 samples, as in torch); frames = lens[b] / 480 (integer division: the tail shorter than a hop
// only contributes through the frames that overlap it).
void mel_spectrogram(cvk_ctx* ctx, const float* wav, const int* lens, int B, int fmax_hz, float* mel, cudaStream_t st) {
  if (!ctx->mel_model) mel_init(ctx);
  MelModel* g_mel = (MelModel*)ctx->mel_model;
  ctx->arena.reset();
  std::vector<int> frames(B), rows(B), off(B), ns(lens, lens + B);
  int acc = 0;
  for (int b = 0; b < B; ++b) {
    CVK_REQUIRE(lens[b] > PAD, "mel_spectrogram: reflect padding by 720 needs at least 721 samples (torch raises as well)");
    frames[b] = lens[b] / HOP;
    rows[b] = frames[b] + 3;
    off[b] = acc;
    acc += lens[b];
  }
  Seqs sr = make_seqs(ctx, rows.data(), B, 4, 1, 0, st);
  Seqs sf = shrink_seqs(ctx, sr, 3, st);
  int* d_off = (int*)ctx->arena.alloc(sizeof(int) * B);
  int* d_ns = (int*)ctx->arena.alloc(sizeof(int) * B);
  CVK_CHECK_CUDA(cudaMemcpyAsync(d_off, off.data(), sizeof(int) * B, cudaMemcpyHostToDevice, st));
  CVK_CHECK_CUDA(cudaMemcpyAsync(d_ns, ns.data(), sizeof(int) * B, cudaMemcpyHostToDevice, st));
  Mat x = arena_mat(ctx, DT_F32, sr.R, HOP, HOP);
  zero_mat(ctx, st, x);
  frame_rows_kernel<<<dim3(64, B), 256, 0, st>>>(wav, d_off, d_ns, sr.d_start, x.f32());
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  Mat spec = arena_mat(ctx, DT_F32, sr.R, 2 * N_BINS, round_up(2 * N_BINS, 8));
  {
    Epilogue e;
    e.row2seq = sf.d_row2seq;
    e.out = spec;
    conv_gemm_simt(ctx, st, x, g_mel->dft, e);
  }
  Mat mag = arena_mat(ctx, DT_F32, sr.R, N_BINS, BINS_LD);
  magnitude_kernel<<<132 * 4, 256, 0, st>>>(spec.f32(), spec.ld, sr.R, mag.f32(), mag.ld);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  Mat out = arena_mat(ctx, DT_F32, sr.R, N_MEL, N_MEL);
  {
    Epilogue e;
    e.out = out;
    CVK_REQUIRE(fmax_hz == 8000 || fmax_hz == 0 || fmax_hz == SR / 2, "mel_spectrogram: fmax must be 8000 or sr/2 (0 = null)");
    conv_gemm_simt(ctx, st, mag, fmax_hz == 8000 ? g_mel->mel : g_mel->mel_nyq, e);
  }
  log_clamp_kernel<<<132, 256, 0, st>>>(out.f32(), (size_t)sr.R * N_MEL);
  ctx->launches++;
  CVK_LAUNCH_CHECK();
  unpack_rows(ctx, st, out, sf, 0, mel, N_MEL);
}
