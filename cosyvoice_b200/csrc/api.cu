// extern "C" boundary of libcvk (include/cvk.h): argument checking, error translation, no exceptions across the ABI.
#include "common.cuh"
#include <string.h>
#include <algorithm>

// stage entry points implemented in hift.cu / flow.cu / llm.cu / mel.cu
void hift_build(cvk_ctx* ctx);
void hift_f0(cvk_ctx* ctx, const float* mel, const int* lens, int B, float* f0_out, cudaStream_t st);
void hift_source(cvk_ctx* ctx, const float* f0, const int* lens, int B, const float* noise, float* source_out, cudaStream_t st);
void hift_decode(cvk_ctx* ctx, const float* mel, const int* lens, int B, const float* source, float* wav, cudaStream_t st, int unit = -1,
                 float* hidden = nullptr);
void hift_inference(cvk_ctx* ctx, const float* mel, const int* lens, int B, const float* noise, const float* cache_source,
                    const int* cache_lens, float* wav, float* source_out, cudaStream_t st);
void flow_build(cvk_ctx* ctx, const int* cfg, int ncfg);
void flow_encoder(cvk_ctx* ctx, const int32_t* tokens, const int* lens, int B, int streaming, int context_len, float* h, cudaStream_t st,
                  int n_layers = 0, float* hidden = nullptr);
void flow_estimator(cvk_ctx* ctx, const float* x, const float* mu, const float* t, const float* spks, const float* cond, const int* lens,
                    int B, int streaming, float* out, cudaStream_t st, int n_units = 0,
                    float* hidden = nullptr);
void flow_cfm_solve(cvk_ctx* ctx, const float* mu, const float* spks, const float* cond, const int* lens, int B, const float* z,
                    int n_timesteps, float cfg_rate, int streaming, float* out, cudaStream_t st);
void flow_inference(cvk_ctx* ctx, const int32_t* tokens, const int* token_lens, const float* prompt_feat, const int* prompt_feat_lens,
                    const float* embedding, int B, int n_timesteps, int streaming, int finalize, float* mel, cudaStream_t st);
void flow_set_noise(cvk_ctx* ctx, const float* noise_tm, int T, int on_device);
void llm_build(cvk_ctx* ctx, const int* cfg, int ncfg);
cvk_lm_session* llm_session_create(cvk_ctx* ctx, int max_batch, int max_context);
void llm_session_destroy(cvk_ctx* ctx, cvk_lm_session* s);
void hift3_build(cvk_ctx* ctx);
void hift3_set_noise(cvk_ctx* ctx, const float* rand_ini, const float* sine_noise, long long n, int on_device);
void hift3_inference(cvk_ctx* ctx, const float* mel, const int* lens, const int* finalize, int B, float* wav, float* f0_out,
                     float* source_out, cudaStream_t st, int unit = -1, float* hidden = nullptr);
void dit_build(cvk_ctx* ctx, const int* cfg, int ncfg);
void dit_estimator(cvk_ctx* ctx, const float* x, const float* mu, const float* t, const float* spks, const float* cond, const int* lens,
                   int B, int streaming, float* out, cudaStream_t st, int n_blocks = 0, float* hidden = nullptr);
void flow3_inference(cvk_ctx* ctx, const int32_t* tokens, const int* token_lens, const float* prompt_feat, const int* prompt_feat_lens,
                     const float* embedding, int B, int n_timesteps, int streaming, int finalize, float* mel, cudaStream_t st);
void llm_prefill(cvk_ctx* ctx, cvk_lm_session* s, const int32_t* text, const int* text_lens, const int32_t* speech,
                 const int* speech_lens, int B, cudaStream_t st);
void llm_decode(cvk_ctx* ctx, cvk_lm_session* s, int n_steps, const float* uniforms, const int32_t* min_len, const int32_t* max_len,
                int32_t* out_ids, int out_ld, int32_t* out_count, int32_t* done, int* live_host, cudaStream_t st);
void llm_forward_logp(cvk_ctx* ctx, const float* embeds, const int* lens, int B, float* logp, cudaStream_t st);
void llm_last_logits(cvk_ctx* ctx, cvk_lm_session* s, float* logits, cudaStream_t st);
int llm_vocab(cvk_ctx* ctx);
void llm_session_begin(cvk_ctx* ctx, cvk_lm_session* s, int B, cudaStream_t st);
void llm_feed(cvk_ctx* ctx, cvk_lm_session* s, const int32_t* ids, const int32_t* kinds, int n, cudaStream_t st);
void llm_next_logp(cvk_ctx* ctx, cvk_lm_session* s, float* logp, cudaStream_t st);
void llm_feed_rows(cvk_ctx* ctx, cvk_lm_session* s, int n_rows, const int* rows, const int* counts, const int32_t* ids, const int32_t* kinds,
                   cudaStream_t st);
void llm_ragged_attention_op(cvk_ctx* ctx, const float* q, const float* k_cache, const float* v_cache, int cache_rows, int max_ctx,
                             const int* rowpos, int M, float* out, cudaStream_t st);
void llm_next_logp_rows(cvk_ctx* ctx, cvk_lm_session* s, int n_rows, const int* rows, float* logp, cudaStream_t st);
void llm_ras_sample(cvk_ctx* ctx, float* logp, int B, int V, const int32_t* history, int hist_ld, const int32_t* hist_count,
                    const float* uniforms, const int32_t* ignore_eos, int32_t* out_ids, cudaStream_t st);
void llm_decode_attention_op(cvk_ctx* ctx, const float* partial, int splits, int rows, const float* bias, float* k_cache, float* v_cache,
                             const int* ctx_len_host, int max_ctx, float* out, cudaStream_t st);
void llm_decode_layers_op(cvk_ctx* ctx, int B, const int* ctx_len_host, int max_ctx, float* x, float* k_cache, float* v_cache,
                          float* xn_out, float* att_out, float* ffa_out, cudaStream_t st);
void llm_sample_step_op(cvk_ctx* ctx, float* logits, int B, int V, const float* uniforms, const int32_t* min_len, const int32_t* max_len,
                        int32_t* out_ids, int out_ld, int32_t* out_count, int32_t* done, int* ctx_len, const int* base_len, int* live,
                        const float* speech_emb, float* next_x, const float* gamma, float* xn, cudaStream_t st);
void llm_log_softmax_op(cvk_ctx* ctx, float* x, int rows, int V, cudaStream_t st);
void mel_spectrogram(cvk_ctx* ctx, const float* wav, const int* lens, int B, int fmax_hz, float* mel, cudaStream_t st);
void mel_init(cvk_ctx* ctx);
void mel_resample(cvk_ctx* ctx, const float* mel, const int* lens, const int* out_lens, int B, float* out, cudaStream_t st);
void prompt_feat_init(cvk_ctx* ctx);

#define CVK_API_BEGIN            \
  if (!ctx) return CVK_ERR_INVALID; \
  try {                          \
    cudaSetDevice(ctx->device);
#define CVK_API_END                                  \
    return CVK_OK;                                   \
  } catch (const CvkError& e) {                      \
    ctx->last_error = e.what();                      \
    return e.code;                                   \
  } catch (const std::exception& e) {                \
    ctx->last_error = std::string("internal: ") + e.what(); \
    return CVK_ERR_INVALID;                          \
  }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

void encode_tma_map(cvk_ctx* ctx, CUtensorMap* map, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
                    const cuuint32_t* box, int dtype, CUtensorMapL2promotion l2, const char* what) {
  CVK_REQUIRE(rank == 2 || rank == 3, std::string("tensor map ") + what + ": rank 2 or 3");
  const cuuint32_t es[3] = {1, 1, 1};
  CUresult r = ((EncodeTiledFn)ctx->encode_tiled)(map, dtype == DT_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank,
                                                  const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                                  CU_TENSOR_MAP_SWIZZLE_128B, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  CVK_REQUIRE(r == CUDA_SUCCESS, std::string("cuTensorMapEncodeTiled(") + what + ") failed: " + std::to_string((int)r));
}

extern "C" {

const char* cvk_version(void) { return "libcvk 0.1 (sm_90a)"; }

int cvk_create(int device, int precision, size_t workspace_bytes, cvk_ctx** out) {
  if (!out) return CVK_ERR_INVALID;
  *out = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= device || device < 0) return CVK_ERR_CUDA;   // no CPU fallback
  if (precision != CVK_PREC_FP32 && precision != CVK_PREC_BF16) return CVK_ERR_INVALID;
  if (cudaSetDevice(device) != cudaSuccess) return CVK_ERR_CUDA;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return CVK_ERR_CUDA;
  if (prop.major != 9) return CVK_ERR_CUDA;    // sm_90a only: the wgmma/TMA kernels have no other code path
  void* encode = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &encode, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess || !encode)
    return CVK_ERR_CUDA;
  try {
    gemm_tc_setup();
    attention_tc_setup();
    skinny_setup();
    hift3_setup();
  } catch (const std::exception&) {
    return CVK_ERR_CUDA;
  }
  cvk_ctx* ctx = new cvk_ctx();
  ctx->device = device;
  ctx->precision = precision;
  ctx->act_dtype = precision == CVK_PREC_BF16 ? DT_BF16 : DT_F32;
  ctx->num_sms = prop.multiProcessorCount;
  ctx->encode_tiled = encode;
  if (workspace_bytes == 0) workspace_bytes = (size_t)4 << 30;
  void* p = nullptr;
  if (cudaMalloc(&p, workspace_bytes) != cudaSuccess) {
    delete ctx;
    return CVK_ERR_OOM;
  }
  ctx->arena.base = (char*)p;
  ctx->arena.cap = workspace_bytes;
  *out = ctx;
  return CVK_OK;
}

void cvk_destroy(cvk_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  for (auto& kv : ctx->raw) cudaFree(kv.second.p);
  for (void* p : ctx->owned) cudaFree(p);
  cudaFree(ctx->arena.base);
  delete ctx;
}

const char* cvk_last_error(cvk_ctx* ctx) { return ctx ? ctx->last_error.c_str() : "null context"; }
thread_local int cvk_in_capture = 0;
int64_t cvk_launch_count(cvk_ctx* ctx) { return ctx ? ctx->launches.load() : 0; }
int cvk_stream_create(cvk_ctx* ctx, void** out) {
  CVK_API_BEGIN
  CVK_REQUIRE(out != nullptr, "cvk_stream_create: bad arguments");
  cudaStream_t s = nullptr;
  CVK_CHECK_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  *out = (void*)s;
  CVK_API_END
}
void cvk_stream_destroy(cvk_ctx* ctx, void* stream) {
  if (!ctx || !stream) return;
  cudaSetDevice(ctx->device);
  cudaStreamDestroy((cudaStream_t)stream);
}
double cvk_last_op_ms(cvk_ctx* ctx) { return ctx ? ctx->op_ms : 0.0; }
int cvk_debug_read(cvk_ctx* ctx, long long* out, int n) {
  if (!ctx || !ctx->tl || !out || n != 4096) return CVK_ERR_INVALID;   // the LM-chain timeline ("chain_timeline")
  cudaSetDevice(ctx->device);
  if (cudaMemcpy(out, ctx->tl, 4096 * sizeof(long long), cudaMemcpyDeviceToHost) != cudaSuccess) return CVK_ERR_CUDA;
  return CVK_OK;
}

int cvk_set_option(cvk_ctx* ctx, const char* key, int value) {
  CVK_API_BEGIN
  std::string k(key ? key : "");
  if (k == "use_tc") ctx->use_tc = value;
  else if (k == "flow_fused_ff") ctx->flow_fused_ff = value;
  else if (k == "flow_qkv_panel") ctx->flow_qkv_panel = value;
  else if (k == "tc_epi") ctx->tc_epi = value;
  else if (k == "tc_persist") ctx->tc_persist = value;
  else if (k == "tc_epi_frag") ctx->tc_epi_frag = value;
  else if (k == "op_out_bf16") ctx->op_out_bf16 = value;
  else if (k == "op_iters") ctx->op_iters = value;
  else if (k == "use_graph") ctx->use_graph = value;
  else if (k == "use_tc_attn") ctx->use_tc_attn = value;
  else if (k == "use_skinny") ctx->use_skinny = value;
  else if (k == "lm_fused") ctx->lm_fused = value;
  else if (k == "pdl") ctx->pdl = value;
  else if (k == "enc_tc_attn") ctx->enc_tc_attn = value;
  else if (k == "hift_f16") ctx->hift_f16 = value;      // takes effect at the next cvk_finalize("hift" / "hift3")
  else if (k == "chain_timeline") {
    if (value && !ctx->tl) {
      ctx->tl = ctx->dmalloc(4096 * sizeof(long long));
      CVK_CHECK_CUDA(cudaMemset(ctx->tl, 0, 4096 * sizeof(long long)));
    }
    if (!value) ctx->tl = nullptr;
  }
  else throw CvkError(CVK_ERR_INVALID, "unknown option: " + k);
  CVK_API_END
}

int cvk_profile(cvk_ctx* ctx, int enable) {
  CVK_API_BEGIN
  CVK_CHECK_CUDA(cudaDeviceSynchronize());
  for (auto& r : ctx->prof) { ctx->event_pool.push_back(r.a); ctx->event_pool.push_back(r.b); }
  ctx->prof.clear();
  ctx->prof_on = enable;
  CVK_API_END
}

int cvk_profile_read(cvk_ctx* ctx, int family, double* ms, double* flops, double* bytes, int64_t* launches) {
  CVK_API_BEGIN
  CVK_REQUIRE(family >= 0 && family < FAM_COUNT && ms && flops && bytes && launches, "cvk_profile_read: bad arguments");
  CVK_CHECK_CUDA(cudaDeviceSynchronize());
  double t = 0, w = 0, by = 0;
  int64_t n = 0;
  for (auto& r : ctx->prof) {
    if (r.family != family) continue;
    float e = 0.f;
    CVK_CHECK_CUDA(cudaEventElapsedTime(&e, r.a, r.b));
    t += e; w += r.work; by += r.bytes; ++n;
  }
  *ms = t; *flops = w; *bytes = by; *launches = n;
  CVK_API_END
}

int cvk_set_tensor(cvk_ctx* ctx, const char* name, const float* data, int on_device, const int64_t* shape, int ndim) {
  CVK_API_BEGIN
  CVK_REQUIRE(name && data && shape && ndim >= 1 && ndim <= 4, "cvk_set_tensor: bad arguments");
  RawTensor t;
  t.shape.assign(shape, shape + ndim);
  size_t bytes = (size_t)t.numel() * sizeof(float);
  CVK_CHECK_CUDA(cudaMalloc((void**)&t.p, bytes));
  cudaError_t e = cudaMemcpy(t.p, data, bytes, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    cudaFree(t.p);
    throw CvkError(CVK_ERR_CUDA, std::string("cvk_set_tensor copy: ") + cudaGetErrorString(e));
  }
  auto it = ctx->raw.find(name);
  if (it != ctx->raw.end()) {
    cudaFree(it->second.p);
    ctx->raw.erase(it);
  }
  ctx->raw[name] = t;
  CVK_API_END
}

int cvk_finalize(cvk_ctx* ctx, const char* stage, const int* cfg, int ncfg) {
  CVK_API_BEGIN
  std::string s(stage ? stage : "");
  if (s == "hift") hift_build(ctx);
  else if (s == "flow") flow_build(ctx, cfg, ncfg);
  else if (s == "flow3") dit_build(ctx, cfg, ncfg);
  else if (s == "hift3") hift3_build(ctx);
  else if (s == "llm") llm_build(ctx, cfg, ncfg);
  else if (s == "mel") mel_init(ctx);
  else if (s == "prompt") prompt_feat_init(ctx);
  else throw CvkError(CVK_ERR_INVALID, "unknown stage: " + s);
  CVK_CHECK_CUDA(cudaDeviceSynchronize());
  // raw tensors of this stage are no longer needed
  std::string prefix = s + ".";
  for (auto it = ctx->raw.begin(); it != ctx->raw.end();) {
    if (it->first.compare(0, prefix.size(), prefix) == 0) {
      cudaFree(it->second.p);
      it = ctx->raw.erase(it);
    } else ++it;
  }
  CVK_API_END
}

// ---------------------------------------------------------------------------------------------- generic ops
int cvk_op_conv1d(cvk_ctx* ctx, const float* x, const int* lens, int B, int K, const float* w, const float* bias, int N, int taps,
                  int dil, int shift0, int act, float* out, void* stream) {
  CVK_API_BEGIN
  cudaStream_t st = (cudaStream_t)stream;
  CVK_REQUIRE(x && lens && w && out && B > 0 && N >= 1 && K >= 1 && taps >= 1 && dil >= 1, "cvk_op_conv1d: bad arguments");
  ctx->arena.reset();
  size_t owned_mark = ctx->owned.size();
  // Both kernels read rows r + shift0 + j*dil straight from the packed matrix and rely on zero gap rows between sequences: the gap
  // must cover the receptive field on either side, or a sequence convolves with its neighbour's edge.
  const int reach = std::max(-shift0, (taps - 1) * dil + shift0);
  int gap = std::max(32, round_up(reach, 8));
  Seqs s = make_seqs(ctx, lens, B, gap, 1, 0, st);
  ConvW W = make_conv(ctx, w, bias, N, K, taps, dil, shift0);
  CVK_CHECK_CUDA(cudaDeviceSynchronize());   // weight repack runs on the default stream
  Mat a = arena_mat(ctx, ctx->act_dtype, s.R, K);
  zero_mat(ctx, st, a);
  pack_rows(ctx, st, x, K, s, a);
  Mat o = arena_mat(ctx, ctx->op_out_bf16 ? DT_BF16 : DT_F32, s.R, N);
  Epilogue e;
  e.act1 = act;
  e.act1_param = 0.1f;
  e.row2seq = s.d_row2seq;
  e.out = o;
  if (a.dtype == DT_BF16 && W.w16 == nullptr) {   // K not TMA-able: fp32 path
    Mat a32 = arena_mat(ctx, DT_F32, s.R, K);
    zero_mat(ctx, st, a32);
    pack_rows(ctx, st, x, K, s, a32);
    conv_gemm_simt(ctx, st, a32, W, e);
  } else {
    conv_gemm(ctx, st, a, W, e);
    if (ctx->op_iters > 0) {
      cudaEvent_t e0, e1;
      cudaEventCreate(&e0); cudaEventCreate(&e1);
      cudaEventRecord(e0, st);
      for (int i = 0; i < ctx->op_iters; ++i) conv_gemm(ctx, st, a, W, e);
      cudaEventRecord(e1, st);
      CVK_CHECK_CUDA(cudaStreamSynchronize(st));
      float ms = 0.f;
      cudaEventElapsedTime(&ms, e0, e1);
      ctx->op_ms = ms / ctx->op_iters;
      cudaEventDestroy(e0); cudaEventDestroy(e1);
    }
  }
  unpack_rows(ctx, st, o, s, 0, out, N);
  CVK_CHECK_CUDA(cudaStreamSynchronize(st));
  for (size_t i = owned_mark; i < ctx->owned.size(); ++i) cudaFree(ctx->owned[i]);
  ctx->owned.resize(owned_mark);
  CVK_API_END
}

// out[b, n] = sum_k x[b,k] w[n,k] (+bias) through the LM decode weight-streaming kernel (bf16 mode, rows <= 64)
int cvk_op_linear_small(cvk_ctx* ctx, const float* x, int rows, int K, const float* w, const float* bias, int N, float* out, int iters,
                        float* ms_out, void* stream) {
  CVK_API_BEGIN
  cudaStream_t st = (cudaStream_t)stream;
  // every argument is checked before the first allocation or launch: the weight streaming layout needs K % 8 == 0 (finish_convw
  // makes no bf16 copy otherwise) and at least one K chunk and one output tile (the split count divides by both)
  CVK_REQUIRE(x && w && out && rows >= 1 && rows <= 64 && N >= 1 && K >= 8 && K % 8 == 0 && iters >= 0 &&
                  ctx->precision == CVK_PREC_BF16,
              "cvk_op_linear_small: bf16 context, 1 <= rows <= 64, N >= 1, K >= 8 and K % 8 == 0");
  ctx->arena.reset();
  size_t owned_mark = ctx->owned.size();
  ConvW W;
  auto release = [&]() {      // the weight copies live only for this call; a stale `tiled` entry would outlive its source buffer
    if (W.w16) ctx->tiled.erase(W.w16);
    for (size_t i = owned_mark; i < ctx->owned.size(); ++i) cudaFree(ctx->owned[i]);
    ctx->owned.resize(owned_mark);
  };
  try {
    W = make_conv(ctx, w, bias, N, K, 1, 1, 0);
    skinny_tiled_weights(ctx, W);
    CVK_CHECK_CUDA(cudaDeviceSynchronize());
    Mat a32((void*)x, DT_F32, rows, K, K);
    Mat a = arena_mat(ctx, DT_BF16, rows, K);
    convert_mat(ctx, st, a32, a);
    Mat o(out, DT_F32, rows, N, N);
    size_t sf = skinny_scratch_floats(rows, N);
    float* scratch = (float*)ctx->arena.alloc(sf * sizeof(float));
    Epilogue e;
    e.out = o;
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    conv_gemm_skinny(ctx, st, a, W, e, scratch, sf);
    cudaEventRecord(e0, st);
    for (int i = 0; i < iters; ++i) conv_gemm_skinny(ctx, st, a, W, e, scratch, sf);
    cudaEventRecord(e1, st);
    CVK_CHECK_CUDA(cudaStreamSynchronize(st));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    if (ms_out) *ms_out = iters > 0 ? ms / iters : 0.f;
    cudaEventDestroy(e0); cudaEventDestroy(e1);
  } catch (...) {
    release();
    throw;
  }
  release();
  CVK_API_END
}

int cvk_op_attention(cvk_ctx* ctx, const float* q, const float* k, const float* v, const int* lens, int B, int H, int chunk,
                     float scale, float* out, void* stream) {
  CVK_API_BEGIN
  cudaStream_t st = (cudaStream_t)stream;
  // scale > 0: the tensor-core kernel takes the row maximum of the unscaled scores
  CVK_REQUIRE(q && k && v && out && lens && B > 0 && H > 0 && chunk >= 0 && scale > 0.f, "cvk_op_attention: bad arguments");
  ctx->arena.reset();
  Seqs s = make_seqs(ctx, lens, B, 8, 1, 0, st);
  int C = H * 64;
  Mat mq = arena_mat(ctx, ctx->act_dtype, s.R, C), mk = arena_mat(ctx, ctx->act_dtype, s.R, C), mv = arena_mat(ctx, ctx->act_dtype, s.R, C);
  Mat mo = arena_mat(ctx, ctx->act_dtype, s.R, C);
  zero_mat(ctx, st, mq); zero_mat(ctx, st, mk); zero_mat(ctx, st, mv); zero_mat(ctx, st, mo);
  pack_rows(ctx, st, q, C, s, mq);
  pack_rows(ctx, st, k, C, s, mk);
  pack_rows(ctx, st, v, C, s, mv);
  attention_fwd(ctx, st, mq, mk, mv, s, H, chunk, scale, mo);
  unpack_rows(ctx, st, mo, s, 0, out, C);
  CVK_API_END
}

int cvk_op_attention_ex(cvk_ctx* ctx, const float* q, const float* k, const float* v, const int* q_lens, const int* k_lens,
                        const int* q_offset, int B, int H, int kv_heads, int chunk, float scale, float* out, void* stream) {
  CVK_API_BEGIN
  cudaStream_t st = (cudaStream_t)stream;
  CVK_REQUIRE(q && k && v && out && q_lens && k_lens && q_offset && B > 0 && H > 0 && kv_heads > 0 && H % kv_heads == 0 && chunk >= 0 &&
                  scale > 0.f,
              "cvk_op_attention_ex: bad arguments");
  for (int b = 0; b < B; ++b)
    CVK_REQUIRE(q_lens[b] >= 1 && k_lens[b] >= 1 && q_offset[b] >= 0, "cvk_op_attention_ex: empty sequence or negative offset");
  ctx->arena.reset();
  // queries and keys are packed separately, the keys addressed through a cache geometry: the layout of the LM prefill (GQA) and of
  // the streaming flow sessions (key cache longer than the new query rows)
  Seqs s = make_seqs(ctx, q_lens, B, 8, 1, 0, st);
  Seqs ks = make_seqs(ctx, k_lens, B, 8, 1, 0, st, false);
  int* d_qoff = (int*)ctx->arena.alloc(sizeof(int) * B);
  CVK_CHECK_CUDA(cudaMemcpyAsync(d_qoff, q_offset, sizeof(int) * B, cudaMemcpyHostToDevice, st));
  KvGeom kg;
  kg.d_kstart = ks.d_start;
  kg.d_klen = ks.d_len;
  kg.d_qoff = d_qoff;
  const int C = H * 64, Ck = kv_heads * 64;
  Mat mq = arena_mat(ctx, ctx->act_dtype, s.R, C), mo = arena_mat(ctx, ctx->act_dtype, s.R, C);
  Mat mk = arena_mat(ctx, ctx->act_dtype, ks.R, Ck), mv = arena_mat(ctx, ctx->act_dtype, ks.R, Ck);
  zero_mat(ctx, st, mq); zero_mat(ctx, st, mk); zero_mat(ctx, st, mv); zero_mat(ctx, st, mo);
  pack_rows(ctx, st, q, C, s, mq);
  pack_rows(ctx, st, k, Ck, ks, mk);
  pack_rows(ctx, st, v, Ck, ks, mv);
  attention_fwd(ctx, st, mq, mk, mv, s, H, chunk, scale, mo, H / kv_heads, &kg);
  unpack_rows(ctx, st, mo, s, 0, out, C);
  CVK_API_END
}

int cvk_op_decode_attention(cvk_ctx* ctx, const float* partial, int splits, int rows, const float* bias, float* k_cache, float* v_cache,
                            const int* ctx_len, int max_ctx, float* out, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(partial && bias && k_cache && v_cache && ctx_len && out && splits >= 1 && rows >= 1 && max_ctx >= 1 &&
                  ctx->precision == CVK_PREC_BF16,
              "cvk_op_decode_attention: bad arguments (bf16 context)");
  for (int b = 0; b < rows; ++b) CVK_REQUIRE(ctx_len[b] >= 0 && ctx_len[b] < max_ctx, "cvk_op_decode_attention: ctx_len outside [0, max_ctx)");
  llm_decode_attention_op(ctx, partial, splits, rows, bias, k_cache, v_cache, ctx_len, max_ctx, out, (cudaStream_t)stream);
  CVK_API_END
}

int cvk_op_lm_decode_layers(cvk_ctx* ctx, int B, const int* ctx_len_host, int max_ctx, float* x, float* k_cache, float* v_cache,
                            float* xn_out, float* att_out, float* ffa_out, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(ctx_len_host && x && k_cache && v_cache && xn_out && ctx->precision == CVK_PREC_BF16,
              "cvk_op_lm_decode_layers: bad arguments (bf16 context)");
  CVK_REQUIRE(ctx->llm, "cvk_op_lm_decode_layers: llm stage not finalised");
  CVK_REQUIRE(B >= 1 && B <= 64, "cvk_op_lm_decode_layers: B outside [1, 64]");
  // the decode attention kernel holds the scores of max_ctx positions for its 7 query heads in shared memory (decode_attn_allow_ctx)
  CVK_REQUIRE(max_ctx >= 1 && 7 * (size_t)max_ctx * sizeof(float) <= 200 * 1024, "cvk_op_lm_decode_layers: max_ctx beyond the decode attention limit");
  for (int b = 0; b < B; ++b) CVK_REQUIRE(ctx_len_host[b] >= 0 && ctx_len_host[b] < max_ctx, "cvk_op_lm_decode_layers: ctx_len outside [0, max_ctx)");
  llm_decode_layers_op(ctx, B, ctx_len_host, max_ctx, x, k_cache, v_cache, xn_out, att_out, ffa_out, (cudaStream_t)stream);
  CVK_API_END
}

int cvk_op_ragged_attention(cvk_ctx* ctx, const float* q, const float* k_cache, const float* v_cache, int cache_rows, int max_ctx,
                            const int* rowpos_host, int M, float* out, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(q && k_cache && v_cache && rowpos_host && out && M >= 1 && cache_rows >= 1 && max_ctx >= 1 && ctx->precision == CVK_PREC_BF16,
              "cvk_op_ragged_attention: bad arguments (bf16 context)");
  llm_ragged_attention_op(ctx, q, k_cache, v_cache, cache_rows, max_ctx, rowpos_host, M, out, (cudaStream_t)stream);
  CVK_API_END
}

int cvk_op_conv_gemm(cvk_ctx* ctx, const float* x, int rows, int K, int x_ld, int operand, const int* seq_start, const int* seq_len, int B,
                     const float* w, const float* bias, int N, int taps, int dil, int shift0, int act1, float act1_param, const float* alpha1,
                     const float* resid, int resid_ld, int resid_is_out, int accumulate, float* out, int out_dtype, int out_ld, int act2,
                     float act2_param, const float* alpha2, float* out2, int out2_dtype, int out2_ld, void* stream) {
  CVK_API_BEGIN
  cudaStream_t st = (cudaStream_t)stream;
  auto dt_ok = [](int d) { return d == DT_F32 || d == DT_BF16 || d == DT_F16; };
  auto act_ok = [](int a) { return a >= ACT_NONE && a <= ACT_GELU_TANH; };
  auto esize = [](int d) { return d == DT_F32 ? (size_t)4 : (size_t)2; };
  // every argument is checked before the first allocation or launch
  CVK_REQUIRE(x && seq_start && seq_len && w && out && B >= 1 && rows >= 1 && K >= 1 && x_ld >= K && N >= 1 && taps >= 1 && dil >= 1 &&
                  dt_ok(operand) && dt_ok(out_dtype) && out_ld >= N && act_ok(act1) && act_ok(act2) &&
                  (!out2 || (dt_ok(out2_dtype) && out2_ld >= N)) && (!resid || resid_ld >= N) && !(resid && resid_is_out) &&
                  (!resid_is_out || out_dtype == DT_F32),
              "cvk_op_conv_gemm: bad arguments");
  CVK_REQUIRE(operand == DT_F32 || (ctx->precision == CVK_PREC_BF16 && K % 8 == 0),
              "cvk_op_conv_gemm: a 16-bit operand needs a bf16 context and K % 8 == 0 (no 16-bit weight copy otherwise)");
  // output row r reads rows r + shift0 + j*dil, j < taps: a gap narrower than that reach lets a sequence see its neighbour
  const long long reach = std::max(0LL, std::max(-(long long)shift0, (long long)shift0 + (long long)(taps - 1) * dil));
  std::vector<int> order(B);
  for (int b = 0; b < B; ++b) {
    order[b] = b;
    CVK_REQUIRE(seq_len[b] >= 1 && seq_start[b] >= 0 && (long long)seq_start[b] + seq_len[b] <= rows,
                "cvk_op_conv_gemm: empty sequence or sequence outside [0, rows)");
  }
  std::sort(order.begin(), order.end(), [&](int a, int b) { return seq_start[a] < seq_start[b]; });
  for (int i = 1; i < B; ++i) {
    const long long gap = (long long)seq_start[order[i]] - ((long long)seq_start[order[i - 1]] + seq_len[order[i - 1]]);
    CVK_REQUIRE(gap >= reach, "cvk_op_conv_gemm: sequences overlap or are closer than the receptive field");
  }
  if (operand != DT_F32 && ctx->use_tc)
    CVK_REQUIRE(x_ld % 8 == 0 && ((size_t)out_ld * esize(out_dtype)) % 16 == 0 && (!out2 || ((size_t)out2_ld * esize(out2_dtype)) % 16 == 0) &&
                    (!resid || (resid_ld % 4 == 0 && ((uintptr_t)resid & 15) == 0)),
                "cvk_op_conv_gemm: the wgmma kernel needs 16-byte aligned rows of x, out, out2 and resid");
  ctx->arena.reset();
  const size_t owned_mark = ctx->owned.size();
  auto release = [&]() {      // the weight copies live only for this call
    for (size_t i = owned_mark; i < ctx->owned.size(); ++i) cudaFree(ctx->owned[i]);
    ctx->owned.resize(owned_mark);
  };
  try {
    ConvW W;
    {
      // fp16 operands: the IEEE-half weight copy the vocoder stage builds, instead of the bf16 one
      struct F16Scope { cvk_ctx* c; F16Scope(cvk_ctx* c_, bool on) : c(c_) { c->build_f16 = on; } ~F16Scope() { c->build_f16 = 0; } } f16scope(ctx, operand == DT_F16);
      W = make_conv(ctx, w, bias, N, K, taps, dil, shift0);
    }
    CVK_CHECK_CUDA(cudaDeviceSynchronize());   // weight repack runs on the default stream
    std::vector<int> row2seq(rows, -1);
    for (int b = 0; b < B; ++b)
      for (int i = 0; i < seq_len[b]; ++i) row2seq[seq_start[b] + i] = b;
    int* d_row2seq = (int*)ctx->arena.alloc(sizeof(int) * (size_t)rows);
    CVK_CHECK_CUDA(cudaMemcpyAsync(d_row2seq, row2seq.data(), sizeof(int) * (size_t)rows, cudaMemcpyHostToDevice, st));
    // the operand keeps x's pitch, so the columns [K, x_ld) travel with it and must stay unread
    Mat a((void*)x, DT_F32, rows, K, x_ld);
    if (operand != DT_F32) {
      Mat a16 = arena_mat(ctx, operand, rows, x_ld, x_ld);
      convert_mat(ctx, st, Mat((void*)x, DT_F32, rows, x_ld, x_ld), a16);
      a = Mat(a16.p, operand, rows, K, x_ld);
    }
    auto stage = [&](float* p, int dt, int ld) {      // the whole caller matrix, pad columns included, in the output dtype
      Mat m = arena_mat(ctx, dt, rows, ld, ld);
      convert_mat(ctx, st, Mat(p, DT_F32, rows, ld, ld), m);
      return m;
    };
    Mat o = stage(out, out_dtype, out_ld);
    Epilogue e;
    e.act1 = act1;
    e.act1_param = act1_param;
    e.alpha1 = alpha1;
    if (resid_is_out) e.resid = Mat(o.p, DT_F32, rows, N, out_ld);
    else if (resid) e.resid = Mat((void*)resid, DT_F32, rows, N, resid_ld);
    e.row2seq = d_row2seq;
    e.accumulate = accumulate;
    e.out = Mat(o.p, out_dtype, rows, N, out_ld);
    e.act2 = act2;
    e.act2_param = act2_param;
    e.alpha2 = alpha2;
    Mat o2;
    if (out2) {
      o2 = stage(out2, out2_dtype, out2_ld);
      e.out2 = Mat(o2.p, out2_dtype, rows, N, out2_ld);
    }
    if (operand == DT_F32) conv_gemm_simt(ctx, st, a, W, e);
    else conv_gemm(ctx, st, a, W, e);
    convert_mat(ctx, st, o, Mat(out, DT_F32, rows, out_ld, out_ld));
    if (out2) convert_mat(ctx, st, o2, Mat(out2, DT_F32, rows, out2_ld, out2_ld));
    CVK_CHECK_CUDA(cudaStreamSynchronize(st));
  } catch (...) {
    release();
    throw;
  }
  release();
  CVK_API_END
}

int cvk_op_flow_ff(cvk_ctx* ctx, float* x, int rows, const int* seq_start, const int* seq_len, int B, const float* ln3_g, const float* ln3_b,
                   const float* w1, const float* b1, const float* w2, const float* b2, const float* ln_g, const float* ln_b, const float* att,
                   const float* wo, const float* bo, float* out, void* stream) {
  CVK_API_BEGIN
  cudaStream_t st = (cudaStream_t)stream;
  CVK_REQUIRE(x && rows >= 1 && seq_start && seq_len && B >= 1 && ln3_g && ln3_b && w1 && b1 && w2 && b2 && (!ln_g) == (!ln_b) && out &&
                  ((uintptr_t)x & 15) == 0 && (!att) == (!wo) && (!att) == (!bo),
              "cvk_op_flow_ff: bad arguments");
  std::vector<int> row2seq(rows, -1);
  for (int b = 0; b < B; ++b) {
    CVK_REQUIRE(seq_len[b] >= 1 && seq_start[b] >= 0 && (long long)seq_start[b] + seq_len[b] <= rows,
                "cvk_op_flow_ff: empty sequence or sequence outside [0, rows)");
    for (int i = 0; i < seq_len[b]; ++i) {
      CVK_REQUIRE(row2seq[seq_start[b] + i] < 0, "cvk_op_flow_ff: sequences overlap");
      row2seq[seq_start[b] + i] = b;
    }
  }
  ctx->arena.reset();
  const size_t owned_mark = ctx->owned.size();
  auto release = [&]() {      // the weight copies live only for this call
    for (size_t i = owned_mark; i < ctx->owned.size(); ++i) cudaFree(ctx->owned[i]);
    ctx->owned.resize(owned_mark);
  };
  try {
    const ConvW W1 = make_conv(ctx, w1, b1, 1024, 256, 1, 1, 0), W2 = make_conv(ctx, w2, b2, 256, 1024, 1, 1, 0);
    ConvW Wo;
    if (att) Wo = make_conv(ctx, wo, bo, 256, 512, 1, 1, 0);
    CVK_CHECK_CUDA(cudaDeviceSynchronize());   // weight repack runs on the default stream
    int* d_row2seq = (int*)ctx->arena.alloc(sizeof(int) * (size_t)rows);
    CVK_CHECK_CUDA(cudaMemcpyAsync(d_row2seq, row2seq.data(), sizeof(int) * (size_t)rows, cudaMemcpyHostToDevice, st));
    const int adt = ctx->act_dtype;
    Mat o = arena_mat(ctx, adt, rows, 256), xn = arena_mat(ctx, adt, rows, 256), hid = arena_mat(ctx, adt, rows, 1024);
    Mat am;
    if (att) {
      am = arena_mat(ctx, adt, rows, 512);
      convert_mat(ctx, st, Mat(const_cast<float*>(att), DT_F32, rows, 512, 512), am);
    }
    const Mat xm(x, DT_F32, rows, 256, 256);
    flow_ff(ctx, st, xm, att ? &am : nullptr, att ? &Wo : nullptr, d_row2seq, ln3_g, ln3_b, W1, W2, ln_g, ln_b, o, xn, hid);
    convert_mat(ctx, st, o, Mat(out, DT_F32, rows, 256, 256));
    CVK_CHECK_CUDA(cudaStreamSynchronize(st));
  } catch (...) {
    release();
    throw;
  }
  release();
  CVK_API_END
}

int cvk_op_relpos_attention(cvk_ctx* ctx, const float* q, const float* k, const float* v, const float* pos, int center, const float* bias_u,
                            const float* bias_v, const int* lens, int B, int H, int chunk, float scale, float* out, void* stream) {
  CVK_API_BEGIN
  cudaStream_t st = (cudaStream_t)stream;
  // scale > 0: the tensor-core kernel takes the row maximum of the unscaled scores
  CVK_REQUIRE(q && k && v && pos && bias_u && bias_v && lens && out && B >= 1 && H >= 1 && chunk >= 0 && scale > 0.f && center < (1 << 24),
              "cvk_op_relpos_attention: bad arguments");
  int max_len = 0;
  for (int b = 0; b < B; ++b) {
    CVK_REQUIRE(lens[b] >= 1, "cvk_op_relpos_attention: empty sequence");
    max_len = std::max(max_len, lens[b]);
  }
  CVK_REQUIRE(center >= max_len - 1, "cvk_op_relpos_attention: the table must hold the relative positions -(max(lens)-1) .. max(lens)-1");
  ctx->arena.reset();
  Seqs s = make_seqs(ctx, lens, B, 8, 1, 0, st);
  const int C = H * 64, adt = ctx->act_dtype, pos_rows = 2 * center + 1;
  Mat mq = arena_mat(ctx, adt, s.R, C), mk = arena_mat(ctx, adt, s.R, C), mv = arena_mat(ctx, adt, s.R, C), mo = arena_mat(ctx, adt, s.R, C);
  zero_mat(ctx, st, mq); zero_mat(ctx, st, mk); zero_mat(ctx, st, mv); zero_mat(ctx, st, mo);
  pack_rows(ctx, st, q, C, s, mq);
  pack_rows(ctx, st, k, C, s, mk);
  pack_rows(ctx, st, v, C, s, mv);
  // zero rows up to a multiple of 128, as the encoder builds its table (flow.cu make_pe)
  Mat pe = arena_mat(ctx, adt, round_up(pos_rows, 128), C);
  zero_mat(ctx, st, pe);
  convert_mat(ctx, st, Mat((void*)pos, DT_F32, pos_rows, C, C), Mat(pe.p, adt, pos_rows, C, pe.ld));
  relpos_attention_fwd(ctx, st, mq, mk, mv, pe, center, bias_u, bias_v, s, H, chunk, scale, mo);
  unpack_rows(ctx, st, mo, s, 0, out, C);
  CVK_API_END
}

// ---------------------------------------------------------------------------------------------- HiFT
int cvk_hift_f0(cvk_ctx* ctx, const float* mel, const int* lens, int B, float* f0, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(mel && lens && f0 && B > 0, "cvk_hift_f0: bad arguments");
  hift_f0(ctx, mel, lens, B, f0, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_hift_source(cvk_ctx* ctx, const float* f0, const int* lens, int B, const float* noise, float* source, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(f0 && lens && noise && source && B > 0, "cvk_hift_source: bad arguments");
  hift_source(ctx, f0, lens, B, noise, source, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_hift_decode(cvk_ctx* ctx, const float* mel, const int* lens, int B, const float* source, float* wav, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(mel && lens && source && wav && B > 0, "cvk_hift_decode: bad arguments");
  hift_decode(ctx, mel, lens, B, source, wav, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_hift_inference(cvk_ctx* ctx, const float* mel, const int* lens, int B, const float* noise, const float* cache_source,
                       const int* cache_lens, float* wav, float* source, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(mel && lens && noise && wav && B > 0, "cvk_hift_inference: bad arguments");
  hift_inference(ctx, mel, lens, B, noise, cache_source, cache_lens, wav, source, (cudaStream_t)stream);
  CVK_API_END
}

// ---------------------------------------------------------------------------------------------- flow
int cvk_flow_encoder(cvk_ctx* ctx, const int32_t* tokens, const int* lens, int B, int streaming, int context_len, float* h, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(tokens && lens && h && B > 0 && (context_len == 0 || context_len == 3), "cvk_flow_encoder: bad arguments");
  flow_encoder(ctx, tokens, lens, B, streaming, context_len, h, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_flow_encoder_hidden(cvk_ctx* ctx, const int32_t* tokens, const int* lens, int B, int streaming, int context_len, int n_layers,
                            float* hidden, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(tokens && lens && hidden && B > 0 && (context_len == 0 || context_len == 3), "cvk_flow_encoder_hidden: bad arguments");
  flow_encoder(ctx, tokens, lens, B, streaming, context_len, nullptr, (cudaStream_t)stream, n_layers, hidden);
  CVK_API_END
}
int cvk_cfm_estimator(cvk_ctx* ctx, const float* x, const float* mu, const float* t, const float* spks, const float* cond, const int* lens,
                      int B, int streaming, float* out, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(x && mu && t && spks && cond && lens && out && B > 0, "cvk_cfm_estimator: bad arguments");
  flow_estimator(ctx, x, mu, t, spks, cond, lens, B, streaming, out, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_cfm_estimator_hidden(cvk_ctx* ctx, const float* x, const float* mu, const float* t, const float* spks, const float* cond,
                             const int* lens, int B, int streaming, int n_units, float* hidden, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(x && mu && t && spks && cond && lens && hidden && B > 0, "cvk_cfm_estimator_hidden: bad arguments");
  flow_estimator(ctx, x, mu, t, spks, cond, lens, B, streaming, nullptr, (cudaStream_t)stream, n_units, hidden);
  CVK_API_END
}
int cvk_cfm_estimator_inplace(cvk_ctx* ctx, float* x, const float* mu, const float* t, const float* spks, const float* cond, const int* lens,
                              int B, int streaming, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(x && mu && t && spks && cond && lens && B > 0, "cvk_cfm_estimator_inplace: bad arguments");
  flow_estimator(ctx, x, mu, t, spks, cond, lens, B, streaming, x, (cudaStream_t)stream);     // x is packed before the first write
  CVK_API_END
}
int cvk_workspace_bytes(cvk_ctx* ctx, size_t* capacity, size_t* high_water) {
  CVK_API_BEGIN
  CVK_REQUIRE(capacity && high_water, "cvk_workspace_bytes: bad arguments");
  *capacity = ctx->arena.cap;
  *high_water = ctx->arena.high;
  CVK_API_END
}
int cvk_cfm_solve(cvk_ctx* ctx, const float* mu, const float* spks, const float* cond, const int* lens, int B, const float* z,
                  int n_timesteps, float cfg_rate, int streaming, float* out, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(mu && spks && cond && lens && out && B > 0 && n_timesteps > 0, "cvk_cfm_solve: bad arguments");
  flow_cfm_solve(ctx, mu, spks, cond, lens, B, z, n_timesteps, cfg_rate, streaming, out, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_flow_inference(cvk_ctx* ctx, const int32_t* tokens, const int* token_lens, const float* prompt_feat, const int* prompt_feat_lens,
                       const float* embedding, int B, int n_timesteps, int streaming, int finalize, float* mel, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(tokens && token_lens && prompt_feat_lens && embedding && mel && B > 0, "cvk_flow_inference: bad arguments");
  flow_inference(ctx, tokens, token_lens, prompt_feat, prompt_feat_lens, embedding, B, n_timesteps, streaming, finalize, mel,
                 (cudaStream_t)stream);
  CVK_API_END
}
int cvk_flow_stream_create(cvk_ctx* ctx, int max_frames, int n_timesteps, cvk_flow_stream** out) {
  CVK_API_BEGIN
  CVK_REQUIRE(out != nullptr, "cvk_flow_stream_create: bad arguments");
  *out = flow_stream_create(ctx, 0, 1, max_frames, n_timesteps);
  CVK_API_END
}
int cvk_flow3_stream_create(cvk_ctx* ctx, int max_frames, int n_timesteps, cvk_flow_stream** out) {
  CVK_API_BEGIN
  CVK_REQUIRE(out != nullptr, "cvk_flow3_stream_create: bad arguments");
  *out = flow_stream_create(ctx, 1, 1, max_frames, n_timesteps);
  CVK_API_END
}
int cvk_flow_stream_create_slots(cvk_ctx* ctx, int kind, int slots, int max_frames, int n_timesteps, cvk_flow_stream** out) {
  CVK_API_BEGIN
  CVK_REQUIRE(out != nullptr && (kind == 0 || kind == 1) && slots >= 1, "cvk_flow_stream_create_slots: bad arguments");
  *out = flow_stream_create(ctx, kind, slots, max_frames, n_timesteps);
  CVK_API_END
}
void cvk_flow_stream_destroy(cvk_ctx* ctx, cvk_flow_stream* fs) {
  if (!ctx || !fs) return;
  try { cudaSetDevice(ctx->device); flow_stream_destroy(fs); } catch (...) {}
}
long long cvk_flow_stream_bytes(const cvk_flow_stream* fs) { return fs ? (long long)flow_stream_bytes(fs) : 0; }
int cvk_flow_stream_begin(cvk_ctx* ctx, cvk_flow_stream* fs, const float* prompt_feat, int prompt_frames, const float* embedding, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(fs && embedding && (prompt_feat || prompt_frames == 0), "cvk_flow_stream_begin: bad arguments");
  flow_stream_begin(ctx, fs, 0, prompt_feat, prompt_frames, embedding, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_flow_stream_begin_slot(cvk_ctx* ctx, cvk_flow_stream* fs, int slot, const float* prompt_feat, int prompt_frames, const float* embedding,
                               void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(fs && embedding && (prompt_feat || prompt_frames == 0), "cvk_flow_stream_begin_slot: bad arguments");
  flow_stream_begin(ctx, fs, slot, prompt_feat, prompt_frames, embedding, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_flow_stream_chunk(cvk_ctx* ctx, cvk_flow_stream* fs, const int32_t* tokens, int n_tokens, float* mel_out, int mel_capacity_frames,
                          int* n_frames_out, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(fs && tokens && mel_out && n_frames_out && n_tokens > 3, "cvk_flow_stream_chunk: bad arguments");
  const int slot0 = 0;
  flow_stream_chunk(ctx, fs, 1, &slot0, tokens, &n_tokens, mel_out, mel_capacity_frames, n_frames_out, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_flow_stream_chunk_batch(cvk_ctx* ctx, cvk_flow_stream* fs, int B, const int* slots_host, const int32_t* tokens, const int* token_lens_host,
                                float* mel_out, int mel_capacity_frames, int* n_frames_out_host, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(fs && B > 0 && slots_host && tokens && token_lens_host && mel_out && n_frames_out_host, "cvk_flow_stream_chunk_batch: bad arguments");
  flow_stream_chunk(ctx, fs, B, slots_host, tokens, token_lens_host, mel_out, mel_capacity_frames, n_frames_out_host, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_cfm_set_noise(cvk_ctx* ctx, const float* noise_tm, int T, int on_device) {
  CVK_API_BEGIN
  CVK_REQUIRE(noise_tm && T > 0, "cvk_cfm_set_noise: bad arguments");
  flow_set_noise(ctx, noise_tm, T, on_device);
  CVK_API_END
}

// ---------------------------------------------------------------------------------------------- LM
int cvk_hift3_set_noise(cvk_ctx* ctx, const float* rand_ini, const float* sine_noise, long long n, int on_device) {
  CVK_API_BEGIN
  CVK_REQUIRE(rand_ini && sine_noise && n > 0, "cvk_hift3_set_noise: bad arguments");
  hift3_set_noise(ctx, rand_ini, sine_noise, n, on_device);
  CVK_API_END
}
int cvk_hift3_inference(cvk_ctx* ctx, const float* mel, const int* lens_host, int B, int finalize, float* wav, float* f0_out,
                        float* source_out, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(mel && lens_host && wav && B > 0, "cvk_hift3_inference: bad arguments");
  const std::vector<int> flags(B, finalize);
  hift3_inference(ctx, mel, lens_host, flags.data(), B, wav, f0_out, source_out, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_hift3_inference_rows(cvk_ctx* ctx, const float* mel, const int* lens_host, const int* finalize_host, int B, float* wav,
                             float* f0_out, float* source_out, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(mel && lens_host && finalize_host && wav && B > 0, "cvk_hift3_inference_rows: bad arguments");
  hift3_inference(ctx, mel, lens_host, finalize_host, B, wav, f0_out, source_out, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_hift_hidden(cvk_ctx* ctx, int causal, const float* mel, const int* lens_host, const int* finalize_host, int B, const float* source,
                    int unit, float* out, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(mel && lens_host && out && B > 0 && (causal == 0 || causal == 1), "cvk_hift_hidden: bad arguments");
  CVK_REQUIRE(unit >= 0 && unit <= 20, "cvk_hift_hidden: unit outside [0, 20]");
  if (causal) {
    std::vector<int> flags(B, 1);
    if (finalize_host) flags.assign(finalize_host, finalize_host + B);
    hift3_inference(ctx, mel, lens_host, flags.data(), B, nullptr, nullptr, nullptr, (cudaStream_t)stream, unit, out);
  } else {
    CVK_REQUIRE(source != nullptr, "cvk_hift_hidden: stage \"hift\" reads the given source");
    hift_decode(ctx, mel, lens_host, B, source, nullptr, (cudaStream_t)stream, unit, out);
  }
  CVK_API_END
}
int cvk_dit_estimator(cvk_ctx* ctx, const float* x, const float* mu, const float* t, const float* spks, const float* cond,
                      const int* lens_host, int B, int streaming, float* out, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(x && mu && t && spks && cond && lens_host && out && B > 0, "cvk_dit_estimator: bad arguments");
  dit_estimator(ctx, x, mu, t, spks, cond, lens_host, B, streaming, out, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_dit_hidden(cvk_ctx* ctx, const float* x, const float* mu, const float* t, const float* spks, const float* cond,
                   const int* lens_host, int B, int streaming, int n_blocks, float* hidden, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(x && mu && t && spks && cond && lens_host && hidden && B > 0, "cvk_dit_hidden: bad arguments");
  dit_estimator(ctx, x, mu, t, spks, cond, lens_host, B, streaming, nullptr, (cudaStream_t)stream, n_blocks, hidden);
  CVK_API_END
}
int cvk_flow3_inference(cvk_ctx* ctx, const int32_t* tokens, const int* token_lens_host, const float* prompt_feat,
                        const int* prompt_feat_lens_host, const float* embedding, int B, int n_timesteps, int streaming, int finalize,
                        float* mel, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(tokens && token_lens_host && prompt_feat_lens_host && embedding && mel && B > 0 && n_timesteps > 0,
              "cvk_flow3_inference: bad arguments");
  flow3_inference(ctx, tokens, token_lens_host, prompt_feat, prompt_feat_lens_host, embedding, B, n_timesteps, streaming, finalize, mel,
                  (cudaStream_t)stream);
  CVK_API_END
}
int cvk_lm_session_create(cvk_ctx* ctx, int max_batch, int max_context, cvk_lm_session** out) {
  CVK_API_BEGIN
  CVK_REQUIRE(out && max_batch > 0 && max_context > 0, "cvk_lm_session_create: bad arguments");
  *out = llm_session_create(ctx, max_batch, max_context);
  CVK_API_END
}
void cvk_lm_session_destroy(cvk_ctx* ctx, cvk_lm_session* s) {
  if (!ctx || !s) return;
  try { llm_session_destroy(ctx, s); } catch (...) {}
}
int cvk_lm_prefill(cvk_ctx* ctx, cvk_lm_session* s, const int32_t* text, const int* text_lens, const int32_t* speech,
                   const int* speech_lens, int B, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(s && text && text_lens && speech_lens && B > 0, "cvk_lm_prefill: bad arguments");
  llm_prefill(ctx, s, text, text_lens, speech, speech_lens, B, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_lm_decode(cvk_ctx* ctx, cvk_lm_session* s, int n_steps, const float* uniforms, const int32_t* min_len, const int32_t* max_len,
                  int32_t* out_ids, int out_ld, int32_t* out_count, int32_t* done, int* live_host, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(s && uniforms && min_len && max_len && out_ids && out_count && done && n_steps >= 0, "cvk_lm_decode: bad arguments");
  llm_decode(ctx, s, n_steps, uniforms, min_len, max_len, out_ids, out_ld, out_count, done, live_host, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_lm_forward_logp(cvk_ctx* ctx, const float* embeds, const int* lens, int B, float* logp, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(embeds && lens && logp && B > 0, "cvk_lm_forward_logp: bad arguments");
  llm_forward_logp(ctx, embeds, lens, B, logp, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_lm_vocab(cvk_ctx* ctx) { return ctx ? llm_vocab(ctx) : 0; }
int cvk_lm_begin(cvk_ctx* ctx, cvk_lm_session* s, int B, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(s != nullptr, "cvk_lm_begin: bad arguments");
  llm_session_begin(ctx, s, B, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_lm_feed(cvk_ctx* ctx, cvk_lm_session* s, const int32_t* ids_host, const int32_t* kinds_host, int n, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(s && ids_host && kinds_host && n > 0, "cvk_lm_feed: bad arguments");
  llm_feed(ctx, s, ids_host, kinds_host, n, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_lm_next_logp(cvk_ctx* ctx, cvk_lm_session* s, float* logp, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(s && logp, "cvk_lm_next_logp: bad arguments");
  llm_next_logp(ctx, s, logp, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_lm_feed_rows(cvk_ctx* ctx, cvk_lm_session* s, int n_rows, const int* rows_host, const int* counts_host, const int32_t* ids_host,
                     const int32_t* kinds_host, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(s && rows_host && counts_host && ids_host && kinds_host, "cvk_lm_feed_rows: bad arguments");
  llm_feed_rows(ctx, s, n_rows, rows_host, counts_host, ids_host, kinds_host, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_lm_next_logp_rows(cvk_ctx* ctx, cvk_lm_session* s, int n_rows, const int* rows_host, float* logp, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(s && rows_host && logp, "cvk_lm_next_logp_rows: bad arguments");
  llm_next_logp_rows(ctx, s, n_rows, rows_host, logp, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_lm_last_logits(cvk_ctx* ctx, cvk_lm_session* s, float* logits, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(s && logits, "cvk_lm_last_logits: bad arguments");
  llm_last_logits(ctx, s, logits, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_ras_sample(cvk_ctx* ctx, float* logp, int B, int V, const int32_t* history, int hist_ld, const int32_t* hist_count,
                   const float* uniforms, const int32_t* ignore_eos, int32_t* out_ids, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(logp && history && hist_count && uniforms && ignore_eos && out_ids && B > 0 && V > 0 && hist_ld >= 0,
              "cvk_ras_sample: bad arguments");
  llm_ras_sample(ctx, logp, B, V, history, hist_ld, hist_count, uniforms, ignore_eos, out_ids, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_op_sample_step(cvk_ctx* ctx, float* logits, int B, int V, const float* uniforms, int steps, const int32_t* min_len,
                       const int32_t* max_len, int32_t* out_ids, int out_ld, int32_t* out_count, int32_t* done, int* ctx_len,
                       const int* base_len, int* live, const float* speech_emb, float* next_x, const float* gamma, float* xn, void* stream) {
  CVK_API_BEGIN
  cudaStream_t st = (cudaStream_t)stream;
  CVK_REQUIRE(logits && uniforms && min_len && max_len && out_ids && out_count && done && ctx_len && base_len && live && speech_emb &&
                  next_x && !gamma == !xn && B >= 1 && steps >= 1 && out_ld >= 1,
              "cvk_op_sample_step: bad arguments");
  CVK_REQUIRE(V >= 6564 && V <= 6912, "cvk_op_sample_step: vocabulary size out of range (6564 .. 6912 supported)");
  // a live row reads uniforms[count] and, unless it stops, writes out_ids[count]: both must lie inside the caller's buffers
  std::vector<int32_t> cnt(B), dn(B);
  CVK_CHECK_CUDA(cudaMemcpyAsync(cnt.data(), out_count, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, st));
  CVK_CHECK_CUDA(cudaMemcpyAsync(dn.data(), done, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, st));
  CVK_CHECK_CUDA(cudaStreamSynchronize(st));
  for (int b = 0; b < B; ++b)
    CVK_REQUIRE(dn[b] || (cnt[b] >= 0 && cnt[b] < steps && cnt[b] < out_ld), "cvk_op_sample_step: a live row's count is outside [0, min(steps, out_ld))");
  llm_sample_step_op(ctx, logits, B, V, uniforms, min_len, max_len, out_ids, out_ld, out_count, done, ctx_len, base_len, live, speech_emb,
                     next_x, gamma, xn, st);
  CVK_API_END
}
int cvk_op_log_softmax(cvk_ctx* ctx, float* x, int rows, int V, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(x && rows >= 1 && V >= 1, "cvk_op_log_softmax: bad arguments");
  llm_log_softmax_op(ctx, x, rows, V, (cudaStream_t)stream);
  CVK_API_END
}

// ---------------------------------------------------------------------------------------------- mel
int cvk_mel_spectrogram(cvk_ctx* ctx, const float* wav, const int* lens, int B, float* mel, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(wav && lens && mel && B > 0, "cvk_mel_spectrogram: bad arguments");
  mel_spectrogram(ctx, wav, lens, B, 8000, mel, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_mel_spectrogram_ex(cvk_ctx* ctx, const float* wav, const int* lens, int B, int fmax_hz, float* mel, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(wav && lens && mel && B > 0, "cvk_mel_spectrogram_ex: bad arguments");
  mel_spectrogram(ctx, wav, lens, B, fmax_hz, mel, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_mel_resample(cvk_ctx* ctx, const float* mel, const int* lens, const int* out_lens, int B, float* out, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(mel && lens && out_lens && out && B > 0 && B <= 65535, "cvk_mel_resample: bad arguments");
  CVK_REQUIRE(((uintptr_t)mel & 15) == 0 && ((uintptr_t)out & 15) == 0, "cvk_mel_resample: mel and out must be 16-byte aligned");
  mel_resample(ctx, mel, lens, out_lens, B, out, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_whisper_log_mel(cvk_ctx* ctx, const float* wav, const int* lens, int B, float* out, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(wav && lens && out && B > 0, "cvk_whisper_log_mel: bad arguments");
  whisper_log_mel(ctx, wav, lens, B, out, (cudaStream_t)stream);
  CVK_API_END
}
int cvk_kaldi_fbank(cvk_ctx* ctx, const float* wav, const int* lens, int B, int subtract_mean, float* out, void* stream) {
  CVK_API_BEGIN
  CVK_REQUIRE(wav && lens && out && B > 0, "cvk_kaldi_fbank: bad arguments");
  kaldi_fbank80(ctx, wav, lens, B, subtract_mean, out, (cudaStream_t)stream);
  CVK_API_END
}

}  // extern "C"
