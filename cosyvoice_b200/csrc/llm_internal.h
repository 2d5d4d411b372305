// Definitions shared by the LM translation units (llm.cu: model / session / per-op decode path; llm_mega.cu: the
// persistent one-kernel-per-step decode path).  Not part of the C ABI.
#pragma once
#include "common.cuh"

namespace lm {
constexpr int D = 896, NH = 14, NKV = 2, HD = 64, DFF = 4864, VOUT = 6564, EOS = 6561;
constexpr int VOUT3 = 6761, VOUT3_PAD = 6764;   // CosyVoice3LM head (llm.py:689), padded to a 16-byte row pitch
constexpr int QKV_N = NH * HD + 2 * NKV * HD;   // 1152
constexpr float ROPE_THETA = 1.0e6f, RMS_EPS = 1e-6f;
constexpr int SAMPLER_THREADS = 256, TOPK = 25, WIN = 10;
constexpr int SAMPLER_PER = (VOUT3_PAD + SAMPLER_THREADS - 1) / SAMPLER_THREADS;   // 27: largest per-thread segment of the sampler

struct LayerW {
  float *ln1, *ln2;
  ConvW qkv, o, gate_up, down;
  ConvW gate_up_il;   // rows interleaved (2i = gate_i, 2i+1 = up_i) for the SwiGLU epilogue of the decode GEMM
};
}  // namespace lm

struct LmMega;   // llm_mega.cu: per-model schedule + per-CTA weight streams of the persistent decode kernel

struct LlmModel {
  int num_layers = 24;
  int vout = lm::VOUT;           // width of the head / logits rows: 6564 (Qwen2LM) or 6764 (CosyVoice3LM: 6761 + 3 impossible pad ids)
  std::vector<lm::LayerW> layers;
  float* final_norm = nullptr;
  float* text_emb = nullptr;     // [151936][896]
  float* llm_emb = nullptr;      // [2][896]  sos, task_id
  float* speech_emb = nullptr;   // [6564][896]
  ConvW head;                    // llm_decoder 896 -> 6564
  float inv_freq[lm::HD / 2];
  float* d_inv_freq = nullptr;
  LmMega* mega = nullptr;        // bf16 mode: built by llm_build
};

struct cvk_lm_session {
  int max_batch = 0, max_ctx = 0, B = 0;
  int kv_dtype = DT_F32;
  void* kcache = nullptr;   // [layers][max_batch][NKV][max_ctx][HD]
  void* vcache = nullptr;
  int* ctx_len = nullptr;   // [max_batch] cache position of the token currently being fed
  int* base_len = nullptr;  // [max_batch] prompt length L0
  bool fresh = false;
  int fed = 0;              // positions pushed by cvk_lm_feed since cvk_lm_begin
  int64_t graph_kernels = 0;
  int* count = nullptr;     // [max_batch] tokens generated so far
  int* done = nullptr;      // [max_batch]
  int* live = nullptr;      // [1]
  float* x = nullptr;       // [max_batch][896] input embedding of the current step (fp32 residual stream)
  float* hidden = nullptr;  // [max_batch][896] final-normed hidden of the last position
  float* logits = nullptr;  // [max_batch][VOUT]
  void* xn = nullptr;       // act [max_batch][896]
  void* qkv = nullptr;      // act [max_batch][1152]
  void* att = nullptr;      // act [max_batch][896]
  void* gu = nullptr;       // act [max_batch][2*4864]
  void* ffa = nullptr;      // act [max_batch][4864]
  cudaGraphExec_t graph = nullptr;
  // arguments baked into the captured graph
  const float* g_uniforms = nullptr;
  const int32_t *g_min = nullptr, *g_max = nullptr;
  int32_t *g_out_ids = nullptr, *g_out_count = nullptr, *g_done = nullptr;
  int g_out_ld = 0, g_B = 0, g_pdl = -1, g_mega = -1;
  float* scratch = nullptr;      // split-K partial sums of the weight-streaming GEMM
  size_t scratch_floats = 0;
  void* mega_state = nullptr;    // llm_mega.cu: per-session device state of the persistent decode kernel (barrier words, layer table)
  // ragged feeding (cvk_lm_feed_rows / cvk_lm_next_logp_rows)
  bool ragged = false;           // set by cvk_lm_begin; rows_fed mirrors ctx_len only between a begin and the next prefill / decode
  std::vector<int> rows_fed;     // [max_batch] host mirror of ctx_len: positions fed to each row since cvk_lm_begin
  int* sel = nullptr;            // [max_batch] device: rows listed by cvk_lm_next_logp_rows
  int feed_cap = 0;              // positions per forward pass of the feed buffers below (0 until the first cvk_lm_feed_rows)
  float* fx = nullptr;           // [feed_cap][896] fp32 residual stream of the fed positions
  void *fxn = nullptr, *fqkv = nullptr, *fatt = nullptr, *fgu = nullptr, *fffa = nullptr;   // act [feed_cap][...]
  int* fidx = nullptr;           // device copy of a pass's index tables (see llm_feed_rows)
  float* fscratch = nullptr;     // split-K partial sums of the weight-streaming GEMM for up to 64 fed positions
  size_t fscratch_floats = 0;
  std::vector<void*> owned;
};

// ---- llm_mega.cu -------------------------------------------------------------------------------------------------
// build the schedule and the per-CTA weight streams from the (already pre-tiled) decode weights of the model
void lm_mega_build(cvk_ctx* ctx, LlmModel* m);
// true when the persistent kernel can run this session's decode step (bf16 KV, batch <= 64, option on)
bool lm_mega_usable(cvk_ctx* ctx, const cvk_lm_session* s, int B);
// one-time per-session state (called outside graph capture)
void lm_mega_session_init(cvk_ctx* ctx, cvk_lm_session* s);
void lm_mega_session_free(cvk_lm_session* s);
// all transformer layers of one decode step: x / xn (layer-0 input, normed) -> xn (final-normed hidden of this position)
void lm_mega_layers(cvk_ctx* ctx, cudaStream_t st, cvk_lm_session* s, int B);
