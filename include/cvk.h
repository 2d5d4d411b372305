/* libcvk - C ABI of the H100-native CosyVoice2 hot path (LM decode -> CFM flow -> HiFT vocoder + mel frontend).
 *
 * This header is the drop-in boundary (SURVEY.md §8b).  The reference is pure Python, so there is no FFI to
 * mirror symbol-for-symbol; each entry point replaces one of the engine plug-in granularities the reference itself
 * swaps (TensorRT estimator, vLLM LM, TorchScript encoder) or one stage-model method, cited per function as
 * "replaces <file>:<lines>" relative to the reference tree.
 *
 * Conventions
 *  - Every pointer is a DEVICE pointer unless its name ends in _host.  Memory is owned by the caller (PyTorch
 *    allocates it); the library owns only its repacked weights, KV arena and workspace, all inside cvk_ctx.
 *  - Activations cross the ABI as *ragged time-major* fp32 matrices: the B sequences are concatenated along
 *    rows without padding, `lens_host[b]` rows each, channels contiguous ([sum(lens), C]).
 *  - Every data-path call takes an explicit cudaStream_t (passed as void*), never touches the default stream on its own
 *    and never calls cudaDeviceSynchronize (set-up calls - cvk_create / cvk_set_tensor / cvk_finalize / cvk_profile /
 *    cvk_destroy - repack weights on the default stream and block until done).
 *  - Threading: calls that use the ctx workspace (cvk_lm_prefill, cvk_lm_forward_logp, every flow / vocoder / mel / op
 *    call) must be serialised by the caller.  Calls that only touch an LM session (cvk_lm_decode, cvk_lm_begin,
 *    cvk_lm_feed, cvk_lm_next_logp, cvk_lm_feed_rows, cvk_lm_next_logp_rows, cvk_lm_last_logits) and cvk_ras_sample own no
 *    shared state: they may run
 *    concurrently with workspace calls and with each other on DISTINCT sessions and streams - this is the reference's
 *    own concurrency (LM side thread + side stream next to token2wav, cli/model.py:101-129, 268; several requests in
 *    flight, runtime/python/grpc/server.py:69).  One session is never used by two host threads at once.  Streaming-flow
 *    sessions (cvk_flow_stream_*) hold caches only: their begin / chunk calls use the workspace and are serialised like every
 *    other flow call.
 *  - Return value: 0 on success, a negative cvk_status otherwise; cvk_last_error(ctx) holds the message.  No C++
 *    exception crosses the ABI.  There is NO CPU fallback: without a CUDA device cvk_create fails.
 */
#ifndef CVK_H_
#define CVK_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct cvk_ctx cvk_ctx;

typedef enum {
  CVK_OK = 0,
  CVK_ERR_INVALID = -1,        /* bad argument / shape (reference: AssertionError / ValueError) */
  CVK_ERR_CUDA = -2,           /* CUDA runtime / driver error */
  CVK_ERR_OOM = -3,            /* workspace or KV arena exhausted */
  CVK_ERR_MISSING_WEIGHT = -4, /* a state_dict key required by cvk_finalize was not supplied */
  CVK_ERR_STATE = -5           /* stage not finalised / session misuse */
} cvk_status;

/* arithmetic of the tensor-core stages */
#define CVK_PREC_FP32 0 /* everything fp32 on CUDA cores: parity mode, tracks the CPU reference to ~1e-4 */
#define CVK_PREC_BF16 1 /* dense GEMM / conv operands bf16 on wgmma tensor cores, fp32 accumulate + residuals */

/* ---------------------------------------------------------------------------------------------- context */
/* Fails with CVK_ERR_CUDA when the device is not an sm_90 GPU, when the driver does not provide cuTensorMapEncodeTiled, or when the
 * tensor-core kernels cannot be configured on the device, including when the flow attention kernel no longer fits two CTAs per SM. */
int cvk_create(int device, int precision, size_t workspace_bytes, cvk_ctx** out);
void cvk_destroy(cvk_ctx* ctx);
const char* cvk_last_error(cvk_ctx* ctx);
const char* cvk_version(void);
/* kernels launched by this library since creation (bench.py "gpu_launches") */
int64_t cvk_launch_count(cvk_ctx* ctx);
/* A CUDA stream (non-blocking) of the context's device that belongs to the caller alone until cvk_stream_destroy.  For concurrent LM
 * sessions: the decode step graph is captured on the caller's stream, so two sessions, or a session and the workspace calls, must
 * never share one (pooled framework streams are reused round-robin and give no such guarantee). */
int cvk_stream_create(cvk_ctx* ctx, void** out);
void cvk_stream_destroy(cvk_ctx* ctx, void* stream);
/* mean device time (ms) of the kernel timed by the last cvk_op_* call when the "op_iters" option is > 0 (tools/gemm_probe.py) */
double cvk_last_op_ms(cvk_ctx* ctx);
/* debug: copy the LM decode-chain timeline (4 int64 slots per launch, n must be 4096) recorded while "chain_timeline" is on */
int cvk_debug_read(cvk_ctx* ctx, long long* out, int n);
/* workspace arena of the context (SURVEY.md §8b `cvk_workspace_bytes`): capacity given to cvk_create and the high-water mark of
 * the calls made so far - what a caller needs to size cvk_create for its largest batch. */
int cvk_workspace_bytes(cvk_ctx* ctx, size_t* capacity, size_t* high_water);
/* Test / measurement switches, NOT part of the drop-in surface (every default is the benchmarked configuration): kernel-variant
 * A/B ("use_tc", "tc_persist", "tc_epi", "tc_epi_frag", "use_tc_attn", "enc_tc_attn", "use_skinny", "flow_fused_ff", "flow_qkv_panel" (0 / 1 /
 * 2 = the row-panel GEMM never / from 25 panels of 128 rows up / at any row count), "lm_fused", "lm_mega", "mega_coop", "pdl", "use_graph", "hift_f16" - the last one takes effect at the next cvk_finalize("hift")),
 * probes ("op_iters", "op_out_bf16", "chain_timeline").  Unknown keys return CVK_ERR_INVALID. */
int cvk_set_option(cvk_ctx* ctx, const char* key, int value);

/* Per-kernel-family device timing for the roofline report of bench.py: CUDA events are recorded around every launch
 * of a family while enabled (family 0 = wgmma conv-GEMM, 1 = CUDA-core conv-GEMM, 2 = attention).  Launches inside
 * the captured LM decode graph are not instrumented.  cvk_profile_read sums elapsed ms, algorithmic FLOPs and bytes. */
int cvk_profile(cvk_ctx* ctx, int enable);
int cvk_profile_read(cvk_ctx* ctx, int family, double* ms, double* flops, double* bytes, int64_t* launches);

/* ---------------------------------------------------------------------------------------------- weights
 * replaces cosyvoice/cli/model.py:65-73 (CosyVoice2Model.load -> load_state_dict(strict=True)).
 * `name` = "<stage>." + reference state_dict key, stage in {"llm","flow","hift"}; data fp32, C-contiguous, on the
 * device (on_device=1) or host.  cvk_finalize(stage) folds weight-norm (g*v/||v||), repacks convolutions to
 * [Cout][tap][Cin], builds polyphase transposed-conv weights and bf16 copies, then drops the raw tensors.
 * cfg: hift: none; flow: {enc_blocks, enc_up_blocks, num_mid_blocks, n_blocks}; llm: {num_layers}. */
int cvk_set_tensor(cvk_ctx* ctx, const char* name, const float* data, int on_device, const int64_t* shape, int ndim);
int cvk_finalize(cvk_ctx* ctx, const char* stage, const int* cfg, int ncfg);

/* ---------------------------------------------------------------------------------------------- generic ops
 * exposed for per-op parity tests (tests/test_ops_gpu.py); same kernels the stages use. */
/* out[r,n] = act(bias[n] + sum_j sum_k x[r + shift0 + j*dil, k] * w[n,k,j]) for one zero-padded sequence per
 * entry of lens_host, at any receptive field (rows outside a sequence read as zero, never as a neighbouring sequence).
 * w is a torch Conv1d weight [N,K,taps] fp32 on the device; N, K, taps, dil >= 1. */
int cvk_op_conv1d(cvk_ctx* ctx, const float* x, const int* lens_host, int B, int K, const float* w, const float* bias,
                  int N, int taps, int dil, int shift0, int act, float* out, void* stream);
/* out[b,n] = bias[n] + sum_k x[b,k] w[n,k] through the LM decode weight-streaming kernel (bf16 context, 1 <= rows <= 64, N >= 1,
 * K >= 8 with K % 8 == 0; anything else is refused with CVK_ERR_INVALID before any device work); runs it `iters` more times and
 * reports the mean device time. */
int cvk_op_linear_small(cvk_ctx* ctx, const float* x, int rows, int K, const float* w, const float* bias, int N, float* out, int iters,
                        float* ms_out, void* stream);
/* block-causal / full multi-head attention over ragged sequences; q,k,v,out [sum(lens), H*64]; scale > 0 */
int cvk_op_attention(cvk_ctx* ctx, const float* q, const float* k, const float* v, const int* lens_host, int B, int H,
                     int chunk, float scale, float* out, void* stream);
/* the same kernels with grouped-query heads and a key cache, as the LM prefill and the streaming flow sessions run them:
 * q, out [sum q_lens, H*64], k, v [sum k_lens, kv_heads*64] (ragged, packed separately); query head h reads kv head h / (H / kv_heads).
 * Query row i of sequence b sits at absolute position q_offset_host[b] + i; key j of sequence b is visible iff j < k_lens_host[b] and,
 * when chunk > 0, j < ((q_offset_host[b] + i) / chunk + 1) * chunk.  With k_lens == q_lens and q_offset == 0 this is cvk_op_attention.
 * Requires H % kv_heads == 0, scale > 0, lengths >= 1. */
int cvk_op_attention_ex(cvk_ctx* ctx, const float* q, const float* k, const float* v, const int* q_lens_host, const int* k_lens_host,
                        const int* q_offset_host, int B, int H, int kv_heads, int chunk, float scale, float* out, void* stream);
/* One LM decode-attention step (Qwen2 GQA 14/2 x 64, half-split RoPE theta 1e6) on a caller-supplied cache, bf16 context only:
 * partial [splits][rows][1152] are the split-K sums of the qkv projection, bias [1152]; k_cache, v_cache [rows][2][max_ctx][64] fp32,
 * in / out (run as bf16, as in a session, and written back as fp32 with the new row appended); ctx_len_host[b] in [0, max_ctx) is the
 * position of the new token, i.e. the number of history rows; out [rows][896].  Option "lm_fused" selects the fused kernel of the
 * decode graph (default) or, at 0, the per-op reduction + RoPE/append + attention kernels.  max_ctx obeys the session limit. */
/* The cached GQA attention of cvk_lm_feed_rows (tensor-core kernel) on a caller-supplied cache, bf16 context only: q [M][896]
 * (14 query heads, already rotated), k_cache, v_cache [cache_rows][2][max_ctx][64]; query m belongs to cache row rowpos_host[2m] at
 * position rowpos_host[2m+1] and attends to that row's keys 0..position; out [M][896].  Consecutive queries of one row at consecutive
 * positions share a tensor-core tile, as in a feed.  Inputs cross as fp32 and run as bf16, as in a session. */
int cvk_op_ragged_attention(cvk_ctx* ctx, const float* q, const float* k_cache, const float* v_cache, int cache_rows, int max_ctx,
                            const int* rowpos_host, int M, float* out, void* stream);
int cvk_op_decode_attention(cvk_ctx* ctx, const float* partial, int splits, int rows, const float* bias, float* k_cache, float* v_cache,
                            const int* ctx_len_host, int max_ctx, float* out, void* stream);
/* Every layer of the finalised "llm" stage for one decode step on caller state, bf16 context only: the layer loop cvk_lm_decode runs
 * after the sampler, on a temporary session of B x max_ctx.  x [B][896] fp32 residual stream, in / out; k_cache, v_cache
 * [layers][B][2][max_ctx][64] fp32, in / out (run as bf16, as in a session; layer l appends row b at position ctx_len_host[b]);
 * xn_out [B][896] the bf16 final-normed row the step hands to the head; att_out [B][896] and ffa_out [B][4864] (nullable) the last
 * layer's attention output and SwiGLU output, the bf16 operands of its o_proj and down_proj.  The options choose the path as in
 * cvk_lm_decode: "lm_fused" 1 the fused chain ("lm_mega" 1: the persistent kernel), "lm_fused" 0 the per-op chain ("use_skinny" 0: the
 * tiled GEMMs); "pdl" is honoured.  The entry xn = RMSNorm(x) ln1[0] comes from the path's own norm kernel.  An fp32 context, an
 * unfinalised stage, B outside [1, 64], ctx_len outside [0, max_ctx) and max_ctx beyond the decode-attention limit are refused with
 * CVK_ERR_INVALID before any device work. */
int cvk_op_lm_decode_layers(cvk_ctx* ctx, int B, const int* ctx_len_host, int max_ctx, float* x, float* k_cache, float* v_cache,
                            float* xn_out, float* att_out, float* ffa_out, void* stream);
/* element types of the cvk_op_conv_gemm operand and outputs */
#define CVK_DT_F32 0
#define CVK_DT_BF16 1
#define CVK_DT_F16 2 /* IEEE half (the vocoder's operands in the bf16 context); stores saturate at +-65504 */
/* One conv-GEMM launch with the fused epilogue the stages use, on caller-packed matrices (tests):
 *   v    = act1(bias[n] + sum_j sum_k x[r + shift0 + j*dil, k] * w[n,k,j]; act1_param, alpha1[n]) (+ resid[r,n])
 *   v    = valid(r) ? v : 0,  out[r,n] = accumulate ? out[r,n] + v : v,  out2[r,n] = valid(r) ? act2(v; act2_param, alpha2[n]) : 0
 * x [rows, x_ld] fp32 (x_ld >= K; columns [K, x_ld) are never read) is converted to `operand` (CVK_DT_*; 16-bit operands need a bf16
 * context and K % 8 == 0; fp16 operands use the half weight copy the vocoder stage builds).  Rows outside [0, rows) read as zero.  Sequence b
 * occupies rows [seq_start_host[b], + seq_len_host[b]); every other row is a gap row (invalid) and must hold zeros in x.  Sequences must
 * lie inside [0, rows), not overlap, and be separated by gaps at least as wide as the receptive field (max(-shift0, shift0 +
 * (taps-1)*dil) rows).  w is a torch Conv1d weight [N,K,taps], bias [N] or NULL, alpha1 / alpha2 [N] or NULL (alpha 1).
 * resid [rows, resid_ld] fp32 or NULL; resid_is_out = 1 adds the fp32 out itself (in place; resid must be NULL).  out / out2 (out2 may be
 * NULL) are fp32 [rows, out_ld] / [rows, out2_ld] (ld >= N) in / out: their contents are rounded to out_dtype / out2_dtype to form the
 * device matrices (accumulate input, untouched pad columns [N, ld) and rows) and the whole matrices are converted back.
 * Path: fp32 operand -> CUDA-core kernel; 16-bit operand -> wgmma (options "tc_epi", "tc_persist") or, with "use_tc" 0, CUDA cores.
 * A wgmma launch needs 16-byte aligned rows of x (as `operand`), out and out2 (as their dtypes) and resid_ld % 4 == 0.  Every argument is
 * checked before any device work; a refusal returns CVK_ERR_INVALID. */
int cvk_op_conv_gemm(cvk_ctx* ctx, const float* x, int rows, int K, int x_ld, int operand, const int* seq_start_host,
                     const int* seq_len_host, int B, const float* w, const float* bias, int N, int taps, int dil, int shift0, int act1,
                     float act1_param, const float* alpha1, const float* resid, int resid_ld, int resid_is_out, int accumulate,
                     float* out, int out_dtype, int out_ld, int act2, float act2_param, const float* alpha2, float* out2, int out2_dtype,
                     int out2_ld, void* stream);
/* The feed-forward half of a flow-estimator transformer block with the first operand of the next block (tests), in place on
 * x [rows, 256] fp32 (device):
 *   x[r]   = valid(r) ? x[r] + b2 + GELU(LN3(x[r]) w1^T + b1) w2^T : 0,   LN3 = LayerNorm(eps 1e-5; ln3_g, ln3_b)
 *   out[r] = valid(r) ? LayerNorm(x[r]; ln_g, ln_b) : 0   (ln_g, ln_b NULL: out = x)
 * rounded to the activation dtype, returned as fp32 [rows, 256].  w1 [1024, 256], b1 [1024], w2 [256, 1024], b2 [256] (torch Linear).
 * Sequence b occupies rows [seq_start_host[b], + seq_len_host[b]) (inside [0, rows), not overlapping); every other row is a gap row.
 * bf16 context: one fused launch, or with option "flow_fused_ff" 0 the LayerNorm / GEMM launches the estimator otherwise runs. */
int cvk_op_flow_ff(cvk_ctx* ctx, float* x, int rows, const int* seq_start_host, const int* seq_len_host, int B, const float* ln3_g,
                   const float* ln3_b, const float* w1, const float* b1, const float* w2, const float* b2, const float* ln_g,
                   const float* ln_b, float* out, void* stream);
/* The conformer relative-position attention (tests): score(i, j) = ((q_i + bias_u) . k_j + (q_i + bias_v) . pos[center - (i - j)]) * scale
 * per head, block-causal when chunk > 0 (key j visible iff j < (i / chunk + 1) * chunk), softmax over the visible keys, times v.
 * q, k, v, out [sum lens, H*64] ragged; pos [2*center+1, H*64] (row t holds relative position center - t; the library pads it to a
 * multiple of 128 rows); bias_u, bias_v [H*64].  fp32 context: CUDA-core fp32 kernel; bf16 context: the wgmma pair, or the CUDA-core
 * kernel on bf16 operands when "enc_tc_attn" or "use_tc_attn" is 0.  Requires H >= 1, chunk >= 0, scale > 0, lengths >= 1 and
 * center >= max(lens) - 1. */
int cvk_op_relpos_attention(cvk_ctx* ctx, const float* q, const float* k, const float* v, const float* pos, int center, const float* bias_u,
                            const float* bias_v, const int* lens_host, int B, int H, int chunk, float scale, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------- HiFT vocoder
 * replaces cosyvoice/hifigan/generator.py:557-569 (HiFTGenerator.inference) and its parts. */
/* f0_predictor.py:56-59: mel [sum T,80] -> f0 [sum T] */
int cvk_hift_f0(cvk_ctx* ctx, const float* mel, const int* lens_host, int B, float* f0, void* stream);
/* generator.py:560-564 + SourceModuleHnNSF/SineGen2: f0 [sum T], noise [sum 480T, 9] (standard-normal draws, the
 * reference's randn_like) -> source [sum 480T] */
int cvk_hift_source(cvk_ctx* ctx, const float* f0, const int* lens_host, int B, const float* noise, float* source,
                    void* stream);
/* generator.py:507-539 (decode): mel [sum T,80], source [sum 480T] -> wav [sum 480T] (clamped to +-0.99) */
int cvk_hift_decode(cvk_ctx* ctx, const float* mel, const int* lens_host, int B, const float* source, float* wav,
                    void* stream);
/* whole inference(); cache_source (optional, may be NULL) [sum cache_lens] overwrites the head of each source
 * (generator.py:566-567, streaming glue).  Outputs wav [sum 480T], source [sum 480T]. */
int cvk_hift_inference(cvk_ctx* ctx, const float* mel, const int* lens_host, int B, const float* noise,
                       const float* cache_source, const int* cache_lens_host, float* wav, float* source, void* stream);

/* ---------------------------------------------------------------------------------------------- flow (token -> mel)
 * replaces cosyvoice/flow/flow.py:235-281 (CausalMaskedDiffWithXvec.inference) and the engine plug-in points
 * flow/flow_matching.py:126-153 (forward_estimator: the TensorRT swap point) and cli/model.py:277-279 (encoder). */
/* transformer/upsample_encoder.py:244-307 on token ids.  tokens [sum N] int32 (prompt ++ generated per sequence).
 * context_len: 0 (finalize) or 3 (the last 3 tokens of every sequence are look-ahead context only,
 * flow.py:259-261).  out h [sum 2*(N-context_len), 512]. */
int cvk_flow_encoder(cvk_ctx* ctx, const int32_t* tokens, const int* lens_host, int B, int streaming, int context_len,
                     float* h, void* stream);
/* flow/decoder.py:405-494 (CausalConditionalDecoder.forward) - same I/O contract as the TensorRT engine:
 * x, mu, cond [sum T,80]; t [B]; spks [B,80]; out [sum T,80]; mask = ones within each length. */
int cvk_cfm_estimator(cvk_ctx* ctx, const float* x, const float* mu, const float* t, const float* spks, const float* cond,
                      const int* lens_host, int B, int streaming, float* out, void* stream);
/* parity tests: the arguments of cvk_flow_encoder, but the call stops after the first n_layers units and writes the fp32 residual
 * stream to `hidden` instead of h.  Unit 0 is the token embedding, embed and the PreLookahead layer; units 1 .. enc_blocks the
 * conformer layers (hidden [sum (N - context_len), 512], token rate); unit enc_blocks + 1 up_layer and up_embed, each later one an
 * up layer (hidden [sum 2 (N - context_len), 512]).  after_norm is not applied.  An n_layers outside
 * [0, enc_blocks + 1 + enc_up_blocks] is refused before any device work. */
int cvk_flow_encoder_hidden(cvk_ctx* ctx, const int32_t* tokens, const int* lens_host, int B, int streaming, int context_len,
                            int n_layers, float* hidden, void* stream);
/* parity tests: the arguments of cvk_cfm_estimator, but the call stops after the first n_units units and writes the fp32 residual
 * stream [sum T, 256] to `hidden` instead of the estimator output.  A unit is one stage's resnet or one of its transformer blocks,
 * in execution order (down, mid 0 .. num_mid - 1, up); down_blocks.0.2 runs with the first mid-stage resnet.  An n_units outside
 * [1, (num_mid + 2) * (1 + n_blocks)] is refused before any device work. */
int cvk_cfm_estimator_hidden(cvk_ctx* ctx, const float* x, const float* mu, const float* t, const float* spks, const float* cond,
                             const int* lens_host, int B, int streaming, int n_units, float* hidden, void* stream);
/* the engine contract itself (flow/flow_matching.py:140-148: the last binding of the TensorRT context is x.data_ptr(), the
 * result overwrites x).  `out` of cvk_cfm_estimator may alias `x` as well: x is consumed before the first write. */
int cvk_cfm_estimator_inplace(cvk_ctx* ctx, float* x, const float* mu, const float* t, const float* spks, const float* cond,
                              const int* lens_host, int B, int streaming, void* stream);
/* flow/flow_matching.py:203-227 + 71-124: fixed seed-0 noise unless z given ([sum T,80]), cosine schedule, Euler,
 * CFG.  mu, cond [sum T,80]; spks [B,80]; out mel [sum T,80]. */
int cvk_cfm_solve(cvk_ctx* ctx, const float* mu, const float* spks, const float* cond, const int* lens_host, int B,
                  const float* z, int n_timesteps, float cfg_rate, int streaming, float* out, void* stream);
/* flow.py:235-281 end to end.  tokens [sum (P_b+N_b)] (prompt then generated), prompt_feat [sum Tp_b, 80],
 * embedding [B,192]; finalize=0 treats the last 3 tokens as look-ahead.  out mel [sum (2*(P+N-ctx) - Tp), 80]. */
int cvk_flow_inference(cvk_ctx* ctx, const int32_t* tokens, const int* token_lens_host, const float* prompt_feat,
                       const int* prompt_feat_lens_host, const float* embedding, int B, int n_timesteps, int streaming,
                       int finalize, float* mel, void* stream);

/* ---- incremental streaming flow (SURVEY 8(f) rank 1) -------------------------------------------------------------------------
 * The reference's streaming loop calls flow.inference(streaming=True, finalize=False) on the GROWING token prefix for every
 * chunk (cli/model.py:346-363) and keeps only the frames past token_offset.  Block-causal attention (utils/mask.py:127-158,
 * static chunk 50 frames) and causal convolutions (flow/decoder.py:25-62) make every complete chunk independent of later
 * frames, so a session object caches, per Euler step, the K/V rows of every estimator transformer block and the two-row
 * input tails of every causal convolution; a chunk call then computes its NEW frames only and returns exactly the rows the
 * reference call would (same noise rows of cvk_cfm_set_noise, same prompt conditioning).  Chunk ends must be multiples of
 * 50 frames (the reference's hop schedule guarantees it); the final, non-streaming call (finalize=True runs with
 * streaming=False in the reference, cli/model.py:372-378: full attention) stays cvk_flow_inference.
 * create: caches for up to max_frames mel frames (prompt included) and n_timesteps Euler steps; cvk_flow_stream_bytes reports
 * their size.  begin: new utterance - prompt_feat [prompt_frames,80], embedding [192] (device).  chunk: tokens = device
 * [n_tokens] prompt tokens + all speech tokens so far + the 3 look-ahead tokens; writes the frames
 * [max(done, prompt_frames), 2*(n_tokens-3)) to mel_out [mel_capacity_frames,80] and their count to *n_frames_out (host).
 * Calls on one session are serialised by the caller, like every workspace call of the context. */
typedef struct cvk_flow_stream cvk_flow_stream;
int cvk_flow_stream_create(cvk_ctx* ctx, int max_frames, int n_timesteps, cvk_flow_stream** out);
/* the same session for the CosyVoice3 DiT (stage "flow3", flow/flow.py:369-414 with streaming=True): K/V rows of the 22 blocks
 * (rotary positions absolute) and the 30-row input tails of the two grouped k31 position convolutions (DiT/modules.py:115-145);
 * begin / chunk / destroy / bytes are shared */
int cvk_flow3_stream_create(cvk_ctx* ctx, int max_frames, int n_timesteps, cvk_flow_stream** out);
void cvk_flow_stream_destroy(cvk_ctx* ctx, cvk_flow_stream* fs);
long long cvk_flow_stream_bytes(const cvk_flow_stream* fs);
int cvk_flow_stream_begin(cvk_ctx* ctx, cvk_flow_stream* fs, const float* prompt_feat, int prompt_frames, const float* embedding,
                          void* stream);
int cvk_flow_stream_chunk(cvk_ctx* ctx, cvk_flow_stream* fs, const int32_t* tokens, int n_tokens, float* mel_out,
                          int mel_capacity_frames, int* n_frames_out, void* stream);
/* Multi-slot sessions: `slots` independent utterances in one session (kind 0: U-Net "flow", 1: DiT "flow3").  All slots share one
 * cache allocation per Euler step ([n_blocks][2*slots*cap + 64][K|V]; CFG sequence c of slot s owns rows [(2s+c)*cap, (2s+c+1)*cap)),
 * so one chunk call serves several slots with one launch sequence per stage - the batched form of the reference's per-request
 * streaming loop (cli/model.py:346-363).  The calls above are the 1-slot session, slot 0.
 * begin_slot: new utterance in `slot`; the other slots are not touched.
 * chunk_batch: one chunk for each of B <= slots distinct, begun slots slots_host[0..B).  tokens [sum token_lens_host] ragged, per
 * slot the argument of cvk_flow_stream_chunk; mel_out receives the new frames of every slot back to back ([sum n_frames_out_host,
 * 80], capacity mel_capacity_frames rows), n_frames_out_host[b] their counts.  Every rule of cvk_flow_stream_chunk holds per slot;
 * all arguments are checked before any device work, so a refused call changes no slot's state.
 * Threading: like every flow call, begin_slot / chunk_batch use the workspace and are serialised by the caller. */
int cvk_flow_stream_create_slots(cvk_ctx* ctx, int kind, int slots, int max_frames, int n_timesteps, cvk_flow_stream** out);
int cvk_flow_stream_begin_slot(cvk_ctx* ctx, cvk_flow_stream* fs, int slot, const float* prompt_feat, int prompt_frames,
                               const float* embedding, void* stream);
int cvk_flow_stream_chunk_batch(cvk_ctx* ctx, cvk_flow_stream* fs, int B, const int* slots_host, const int32_t* tokens,
                                const int* token_lens_host, float* mel_out, int mel_capacity_frames, int* n_frames_out_host,
                                void* stream);

/* ---- CosyVoice3 vocoder (stage "hift3") ------------------------------------------------------------------------------------
 * cosyvoice/hifigan/generator.py:572-726 CausalHiFTGenerator (+ f0_predictor.py:60-103 in float64, generator.py:716-717).
 * cvk_hift3_set_noise hands over the module's constructor-time random tensors, which are not state_dict entries
 * (generator.py:223-226): rand_ini [9] (SineGen2.rand_ini) and sine_noise [n][9] (SineGen2.sine_waves, indexed from the start of
 * every utterance).  cvk_hift3_inference = CausalHiFTGenerator.inference (:714-726) for B utterances: mel [sum T, 80] ->
 * wav [sum 480 T]; f0_out [sum T] and source_out [sum 480 T] are optional (NULL).  finalize == 0 is the streaming call
 * (:676-683, :709-710, :722-725): 3 + 4 mel frames of look-ahead are consumed and the last frame's samples dropped, i.e.
 * wav [sum 480 (T-8)], f0_out [sum (T-3)], source_out [sum 480 (T-3)]; every utterance needs T >= 9.
 * cvk_hift3_inference_rows is the same call with a flag per utterance, finalize_host[B]: utterance b's outputs take, back to back,
 * 480 T / T / 480 T samples when its flag is set and 480 (T-8) / T-3 / 480 (T-3) when it is 0 (then T >= 9).  One call thus
 * vocodes streaming chunks and final utterances together, with the kernels of one homogeneous call of the same total size;
 * each utterance's outputs are bit-identical to a cvk_hift3_inference of it alone with its own flag.  cvk_hift3_inference is
 * the case where every flag equals `finalize`.  All arguments are checked before any device work. */
int cvk_hift3_set_noise(cvk_ctx* ctx, const float* rand_ini, const float* sine_noise, long long n, int on_device);
int cvk_hift3_inference(cvk_ctx* ctx, const float* mel, const int* lens_host, int B, int finalize, float* wav, float* f0_out,
                        float* source_out, void* stream);
int cvk_hift3_inference_rows(cvk_ctx* ctx, const float* mel, const int* lens_host, const int* finalize_host, int B, float* wav,
                             float* f0_out, float* source_out, void* stream);

/* ---- CosyVoice3 flow (stage "flow3", cvk_finalize cfg = {DiT depth}) -----------------------------------------------------------
 * cosyvoice/flow/DiT/dit.py:145-176 (DiT.forward, the CFM estimator of CosyVoice3; TensorRT swap point flow_matching.py:126-153):
 * same dense argument layout as cvk_cfm_estimator - x, mu, cond [sum T, 80] time-major, t [B], spks [B, 80] -> out [sum T, 80];
 * streaming != 0 selects the static 50-frame block-causal mask (dit.py:165-166). */
int cvk_dit_estimator(cvk_ctx* ctx, const float* x, const float* mu, const float* t, const float* spks, const float* cond,
                      const int* lens_host, int B, int streaming, float* out, void* stream);
/* parity tests: the arguments of cvk_dit_estimator, but the call stops after the input embedding and the first n_blocks DiT blocks
 * (0 <= n_blocks <= depth) and writes the fp32 residual stream x [sum T, 1024] (before norm_out) to `hidden` instead of the
 * estimator output.  An n_blocks outside [0, depth] is refused before any device work. */
int cvk_dit_hidden(cvk_ctx* ctx, const float* x, const float* mu, const float* t, const float* spks, const float* cond,
                   const int* lens_host, int B, int streaming, int n_blocks, float* hidden, void* stream);
/* cosyvoice/flow/flow.py:369-414 CausalMaskedDiffWithDiT.inference for B utterances: tokens = prompt tokens followed by the new
 * tokens of every utterance (token_lens_host), prompt_feat [sum Tp, 80], embedding [B, 192]; finalize == 0: the last 3 tokens of
 * every utterance are look-ahead context (flow.py:389-392).  mel receives 2 * (tokens - context) - Tp frames per utterance.
 * The CFM noise is the tensor given to cvk_cfm_set_noise. */
int cvk_flow3_inference(cvk_ctx* ctx, const int32_t* tokens, const int* token_lens_host, const float* prompt_feat,
                        const int* prompt_feat_lens_host, const float* embedding, int B, int n_timesteps, int streaming, int finalize,
                        float* mel, void* stream);
/* the fixed noise tensor of CausalConditionalCFM (flow_matching.py:199-200) must be supplied once: [15000,80]
 * time-major (it is torch's seed-0 randn stream; the library does not re-implement torch's Philox/MT generator) */
int cvk_cfm_set_noise(cvk_ctx* ctx, const float* noise_tm, int T, int on_device);

/* ---------------------------------------------------------------------------------------------- speech-token LM
 * replaces cosyvoice/llm/llm.py:458-549 (Qwen2LM.inference / inference_wrapper; the vLLM swap point :506-534). */
typedef struct cvk_lm_session cvk_lm_session;
int cvk_lm_session_create(cvk_ctx* ctx, int max_batch, int max_context, cvk_lm_session** out);
void cvk_lm_session_destroy(cvk_ctx* ctx, cvk_lm_session* s);
/* llm.py:474-494: assemble [sos, embed(text), task_id, speech_embedding(prompt)] for B rows and run the prefill.
 * text [sum Nt] (prompt_text ++ text per row), speech [sum Np].  After the call the session holds the KV cache and
 * the hidden state of the last prompt position of every row. */
int cvk_lm_prefill(cvk_ctx* ctx, cvk_lm_session* s, const int32_t* text, const int* text_lens_host,
                   const int32_t* speech, const int* speech_lens_host, int B, void* stream);
/* llm.py:536-549: run up to n_steps decode steps for all live rows: head -> log_softmax -> RAS sampling ->
 * stop test -> next embedding.  uniforms [max_steps][B][2] (u1 nucleus draw, u2 fallback draw) indexed by the
 * absolute step; min_len/max_len [B] (device int32).  out_ids [B][out_ld] receives the accepted ids, out_count [B]
 * their number, done [B] (1 once a row hit a stop id or max_len).  Returns the number of live rows via
 * *live_host after synchronising the stream when live_host != NULL. */
int cvk_lm_decode(cvk_ctx* ctx, cvk_lm_session* s, int n_steps, const float* uniforms, const int32_t* min_len,
                  const int32_t* max_len, int32_t* out_ids, int out_ld, int32_t* out_count, int32_t* done, int* live_host,
                  void* stream);
/* teacher-forced log-probs for parity tests: embeds [sum L, 896] -> logp [sum L, V], V = cvk_lm_vocab */
int cvk_lm_forward_logp(cvk_ctx* ctx, const float* embeds, const int* lens_host, int B, float* logp, void* stream);
/* Width V of the log-prob / logits rows of the loaded LM: 6564 for Qwen2LM (llm.py:281), 6764 for CosyVoice3LM (llm.py:689: 6761
 * outputs, padded by 3 ids whose probability is exactly 0); 0 before the "llm" stage is finalised.  The "llm" stage recognises a
 * CosyVoice3LM state_dict by the absence of llm_embedding.weight. */
int cvk_lm_vocab(cvk_ctx* ctx);
/* Text-streaming LM (Qwen2LM.inference_bistream, llm.py:551-661: the caller interleaves 5 text : 15 speech embeddings and forces
 * fill tokens; cli/model.py:113-123 drives it when `text` is a generator).  cvk_lm_begin empties the session (B rows, normally 1);
 * cvk_lm_feed pushes n positions through the KV-cached decode path (llm.py:617-621 forward_one_step): ids_host / kinds_host are
 * HOST arrays, kind 0 = text id (embed_tokens), 1 = speech id (speech_embedding), 2 = llm_embedding row (0 sos, 1 task_id);
 * cvk_lm_next_logp writes log_softmax(llm_decoder(y_pred[:, -1])) (llm.py:622) of the last position to logp [B][V] (device, V = cvk_lm_vocab).
 * The draw itself is cvk_ras_sample (llm.py:627 sampling_ids). */
int cvk_lm_begin(cvk_ctx* ctx, cvk_lm_session* s, int B, void* stream);
int cvk_lm_feed(cvk_ctx* ctx, cvk_lm_session* s, const int32_t* ids_host, const int32_t* kinds_host, int n, void* stream);
int cvk_lm_next_logp(cvk_ctx* ctx, cvk_lm_session* s, float* logp, void* stream);
/* Ragged feeding, for several text-streaming requests in one session (one row each, after cvk_lm_begin with B rows): row
 * rows_host[r] (n_rows distinct rows < B) receives counts_host[r] >= 1 new positions; ids_host / kinds_host hold them concatenated
 * in row order (kinds as in cvk_lm_feed).  Every position of every listed row goes through ONE forward per layer: row b's positions
 * take RoPE / cache positions fed_b .. fed_b + n - 1 (fed_b = positions fed to row b since cvk_lm_begin) and attend causally to
 * that row's cache.  A row's results are bit for bit the same whatever other rows and positions share the call (or split it into
 * passes).  Rows not listed keep their cache, context length and hidden state bit for bit.  Duplicate or out-of-range
 * rows, ids or kinds out of range, and a row whose context would pass the session's max_context are refused with CVK_ERR_INVALID
 * before any device work, so a refused call changes nothing.  A feed of more than 256 positions runs as several forward passes in
 * position order.  The session owns the feed buffers (allocated on first use); like cvk_lm_feed, the call touches no workspace.
 * cvk_lm_next_logp_rows writes the log-probs of the next id after the last fed position of each listed row (distinct rows that
 * have been fed) to logp [n_rows][V] (device, V = cvk_lm_vocab), in list order.  After cvk_lm_prefill or cvk_lm_decode both are
 * refused until the next cvk_lm_begin. */
int cvk_lm_feed_rows(cvk_ctx* ctx, cvk_lm_session* s, int n_rows, const int* rows_host, const int* counts_host, const int32_t* ids_host,
                     const int32_t* kinds_host, void* stream);
int cvk_lm_next_logp_rows(cvk_ctx* ctx, cvk_lm_session* s, int n_rows, const int* rows_host, float* logp, void* stream);
/* parity tests: the row the most recent decode step sampled from, copied to `logits` [B][V] (device): the log-probs
 * log_softmax(llm_decoder output) (llm.py:542) with the sampler's in-place marks, -inf at the eos id while it was masked (min_len) and
 * at the repeated id when the repetition fallback fired.  Rows already done before that step are not sampled and hold the raw head
 * logits. */
int cvk_lm_last_logits(cvk_ctx* ctx, cvk_lm_session* s, float* logits, void* stream);
/* utils/common.py:138-167 + llm.py:150-160 as one kernel.  logp [B,V] (modified in place like the reference),
 * history [B, hist_ld] (hist_ld >= 0) with hist_count [B] valid entries, uniforms [B,2], ignore_eos [B]; out ids [B]; 6564 <= V <= 6912. */
int cvk_ras_sample(cvk_ctx* ctx, float* logp, int B, int V, const int32_t* history, int hist_ld, const int32_t* hist_count,
                   const float* uniforms, const int32_t* ignore_eos, int32_t* out_ids, void* stream);
/* One decode-graph sampler step on caller data, without a loaded LM (tests): the kernel cvk_lm_decode runs after the head, with
 * log_softmax of the logits first.  All pointers are device memory.  logits [B][V] in / out (receives the log-probs with the sampler's
 * -inf marks, as cvk_lm_last_logits shows them); uniforms [steps][B][2] indexed by each row's count; min_len, max_len [B]; out_ids
 * [B][out_ld], out_count [B], done [B], ctx_len [B] (= base_len + count after an accepted id), base_len [B], live [1] as in a session.
 * A row with done != 0 is skipped.  speech_emb [V][896] fp32; next_x [B][896] receives the embedding row of an accepted id.  gamma [896]
 * or NULL: with gamma, xn [B][896] fp32 in / out receives RMSNorm(next_x) * gamma as the bf16 the decode step stores (rows the kernel
 * does not write come back rounded to bf16); gamma and xn are both NULL or both given.  Requires 6564 <= V <= 6912, B >= 1,
 * steps >= 1, out_ld >= 1 and, for every row not done, 0 <= count < min(steps, out_ld) (read back before the launch).  Any other
 * argument is refused with CVK_ERR_INVALID before the sampler runs.  Either precision of context. */
int cvk_op_sample_step(cvk_ctx* ctx, float* logits, int B, int V, const float* uniforms, int steps, const int32_t* min_len,
                       const int32_t* max_len, int32_t* out_ids, int out_ld, int32_t* out_count, int32_t* done, int* ctx_len,
                       const int* base_len, int* live, const float* speech_emb, float* next_x, const float* gamma, float* xn, void* stream);
/* x [rows][V] (device) <- log_softmax(x) per row, in place, with the kernel of cvk_lm_next_logp / cvk_lm_forward_logp (tests):
 * (x - max) - log(sum exp(x - max)), the sum in the sampler's segment order.  rows, V >= 1. */
int cvk_op_log_softmax(cvk_ctx* ctx, float* x, int rows, int V, void* stream);

/* ---------------------------------------------------------------------------------------------- mel frontend
 * replaces third_party/Matcha-TTS/matcha/utils/audio.py:45-82 with cosyvoice2.yaml:150-158 parameters (n_fft 1920, hop 480,
 * 80 mels, fmin 0, fmax 8000, center False).  wav [sum N_b] (24 kHz, any N_b >= 721: the reflect padding is taken about the true
 * last sample) -> mel [sum floor(N_b/480), 80] */
int cvk_mel_spectrogram(cvk_ctx* ctx, const float* wav, const int* lens_host, int B, float* mel, void* stream);
/* same with the filterbank's upper edge as a parameter: fmax_hz = 8000 (CosyVoice2) or 0 / 12000 = sr/2 (`fmax: null` of
 * examples/libritts/cosyvoice3/conf/cosyvoice3.yaml:140-147) */
int cvk_mel_spectrogram_ex(cvk_ctx* ctx, const float* wav, const int* lens_host, int B, int fmax_hz, float* mel, void* stream);
/* The `speed` time-stretch of an offline request: replaces the F.interpolate(tts_mel, size=int(T / speed), mode="linear") of
 * cosyvoice/cli/model.py:320-322 (CosyVoice2Model.token2wav) and :444-446 (CosyVoice3Model.token2wav) for B utterances in one launch.
 * mel [sum lens_host[b], 80] -> out [sum out_lens_host[b], 80], both time-major ragged fp32, 16-byte aligned, not overlapping.
 * Output row j of utterance b is torch's linear interpolation (align_corners=False, no scale factor) bit for bit: scale =
 * (float)T / T', src = max((j + 0.5) scale - 0.5, 0), i0 = (int)src, i1 = min(i0 + 1, T - 1), out = (1 - l) x[i0] + l x[i1] with
 * l = src - i0 (one fused multiply-add each for src and the blend, as torch's kernel rounds them); T' == T copies the rows.  Every
 * length must be >= 1 (torch refuses a size of 0); a refusal returns CVK_ERR_INVALID before any device work.  Uses the workspace. */
int cvk_mel_resample(cvk_ctx* ctx, const float* mel, const int* lens_host, const int* out_lens_host, int B, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------- prompt-side features (16 kHz)
 * SURVEY 8(f) rank 2: the two feature extractors the reference frontend runs on the CPU before its ONNX sessions.
 * cvk_whisper_log_mel replaces whisper.log_mel_spectrogram(speech, n_mels=128) at cosyvoice/cli/frontend.py:98 (hann 400 / hop 160,
 * center, 128 Slaney mels, log10, floor at max - 8, (x + 4) / 4): wav [sum N_b] (N_b > 200) -> out [sum floor(N_b/160), 128],
 * time-major (the reference tensor [1,128,T] transposed).
 * cvk_kaldi_fbank replaces kaldi.fbank(speech, num_mel_bins=80, dither=0, sample_frequency=16000) at frontend.py:108-112 and, with
 * subtract_mean != 0, the mean normalisation of :113: wav [sum N_b] (N_b >= 400) -> out [sum 1 + floor((N_b-400)/160), 80].
 * The speech tokenizer / CAM++ networks that consume them are ONNX files outside the repository and are not rebuilt.
 * cvk_finalize(ctx, "prompt", NULL, 0) builds the constant DFT / filterbank matrices at set-up time (else: on the first call). */
int cvk_whisper_log_mel(cvk_ctx* ctx, const float* wav, const int* lens_host, int B, float* out, void* stream);
int cvk_kaldi_fbank(cvk_ctx* ctx, const float* wav, const int* lens_host, int B, int subtract_mean, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CVK_H_ */
