"""Host-side mirror of the reference pipeline orchestrator, over libcvk.

``B200CosyVoice2Model`` exposes the constructor / ``load`` / ``tts`` / ``token2wav`` surface and the session attributes
of ``cosyvoice.cli.model.CosyVoice2Model`` (cosyvoice/cli/model.py:245-394) so it can be dropped in behind
``cosyvoice.cli.cosyvoice.CosyVoice2`` (``cosyvoice.model = B200CosyVoice2Model(...)``, see INTEGRATION.md), plus
``tts_batch`` for the batch-32 metric (the reference has no batched API; its batch is a Python loop).

All arithmetic happens in libcvk (hand-written sm_90a kernels); torch provides device memory, streams and the two
random streams the reference draws from the global RNG (sampling uniforms, SineGen noise).  No CPU fallback.
"""
import threading
import time
import uuid
from contextlib import contextmanager, nullcontext

import numpy as np
import torch

from . import cvk

TOKEN_MEL_RATIO = 2          # cosyvoice2.yaml:14
PRE_LOOKAHEAD = 3            # cosyvoice2.yaml:46
STREAM_CHUNK_FRAMES = 25 * TOKEN_MEL_RATIO     # cosyvoice2.yaml:16 static_chunk_size, in mel frames
SAMPLES_PER_FRAME = 480


# the streaming chunk schedule of tts(stream=True) (cli/model.py:346-364), shared by tts() and the batched poll loop
def _first_hop_pad(P, hop):
    """tokens added to the first hop so that a P-token prompt and the first hop end on the hop grid"""
    return int(np.ceil(P / hop) * hop - P)


def _this_hop(hop, pad, token_offset):
    """the tokens of the next chunk: the first one also takes the prompt's padding"""
    return hop + pad if token_offset == 0 else hop


def _hop_ready(n_tokens, token_offset, this_hop):
    """the next chunk's tokens and their look-ahead have arrived"""
    return n_tokens - token_offset >= this_hop + PRE_LOOKAHEAD


class SilentTokenFilter:
    """The silent-token rule of the reference's LM job (cli/model.py:102, 121-127) for one request: a silent token is dropped once
    more than MAX_RUN of them have come in a row.  CosyVoice2's list of silent tokens is empty, so it never drops anything."""
    MAX_RUN = 5

    def __init__(self, silent_tokens):
        self.silent_tokens = silent_tokens
        self.run = 0

    def keep(self, tok):
        """feed the request's next id: whether it is kept"""
        if tok in self.silent_tokens:
            self.run += 1
            return self.run <= self.MAX_RUN
        self.run = 0
        return True

    def filter(self, ids):
        """the kept ids of a whole sequence"""
        return [t for t in ids if self.keep(t)]


# tts()'s defaults for the request keys a frontend may leave out: inference_cross_lingual / inference_instruct2 delete prompt keys,
# inference_vc builds no text (cli/frontend.py:191-225)
_REQUEST_DEFAULTS = {k: torch.zeros(1, 0, dtype=torch.int32) for k in ("text", "prompt_text", "llm_prompt_speech_token",
                                                                        "flow_prompt_speech_token", "source_speech_token")}
_REQUEST_DEFAULTS.update(prompt_speech_feat=torch.zeros(1, 0, 80), flow_embedding=torch.zeros(0, 192))


def request_field(r, key):
    """request r's tts() argument `key`, or tts()'s default when r does not carry it"""
    v = r.get(key)
    return _REQUEST_DEFAULTS[key] if v is None else v


def is_vc_request(r):
    """a voice-conversion request (inference_vc): tts() runs token2wav on its source_speech_token and no LM (cli/model.py:336-339)"""
    return request_field(r, "source_speech_token").shape[1] > 0


def request_speed(r):
    """request r's `speed` (default 1.0) as a float; ValueError unless it is > 0"""
    s = float(r.get("speed", 1.0))
    if not s > 0:
        raise ValueError(f"speed must be > 0, got {s}")
    return s


class _LmStopped(Exception):
    """raised into a batched LM generation whose consumer has gone away"""


def _count(keys, prefix):
    idx = set()
    for k in keys:
        if k.startswith(prefix):
            idx.add(int(k[len(prefix):].split(".")[0]))
    return len(idx)


def infer_cfgs(llm_sd, flow_sd):
    """layer counts from state_dict keys (the reference builds these from yaml; cosyvoice2.yaml:23-87)"""
    nl = _count(llm_sd.keys(), "llm.model.model.layers.")
    fk = list(flow_sd.keys())
    flow_cfg = [_count(fk, "encoder.encoders."), _count(fk, "encoder.up_encoders."), _count(fk, "decoder.estimator.mid_blocks."),
                _count(fk, "decoder.estimator.down_blocks.0.1.")]
    return [nl], flow_cfg


def _state_dict(m):
    return m if isinstance(m, dict) else m.state_dict()


def _to_device(t, device):
    """a small host tensor on `device` without a host sync: staged in pinned memory and copied asynchronously on the current stream
    (a plain .to() from pageable memory waits for the stream's queued work)"""
    if device.type != "cuda" or t.device.type == "cuda":
        return t.to(device)
    return t.pin_memory().to(device, non_blocking=True)


class _BistreamRow:
    """The per-request control flow of the text-streaming LM (llm.py:551-661, Qwen2LM.inference_bistream), as a state machine that
    lm_generate_bistream and lm_generate_bistream_batch both drive.

    States: WAIT (needs the next text chunk, or the end of the text), DECODE (the inner decode loop of llm.py:614-640: every step is
    one model call on `lm_input` and one id, forced or drawn, until a fill token sends the row back to WAIT), FINAL (llm.py:642-661:
    decode until eos) and DONE.  A step in DECODE / FINAL is: feed `lm_input`, then, unless `forced()`, draw with
    `ignore_eos()` from the log-probs, then `take(id)`.

    `lm_input` has the reference variable's exact life cycle (list of (kind, id) positions): every model call pushes ALL of it, it is
    replaced after a yielded id and - like the reference - left untouched when a fill token ends a decode burst, so a final phase
    entered right after a fill token pushes that last input a second time (llm.py:634-637, 643)."""
    WAIT, DECODE, FINAL, DONE = range(4)
    MIX_TEXT, MIX_SPEECH = 5, 15
    TEXT, SPEECH, LLM = 0, 1, 2
    SPEECH_VOCAB = 6561

    def __init__(self, fill_token, eos_token, eop_token, prompt_text, prompt_speech_token, max_tokens=None):
        self.fill_token, self.eos_token, self.max_tokens = fill_token, eos_token, max_tokens
        ptext = [int(x) for x in prompt_text.reshape(-1).tolist()]
        lm_prefix = []
        if eop_token is not None:
            # llm.py:583-588: the prompt text up to and including <|endofprompt|> is fed ahead of the 5:15 interleaving
            if eop_token not in ptext:
                raise AssertionError("<|endofprompt|> not detected in CosyVoice3 prompt_text, check your input!")
            eop = ptext.index(eop_token)
            lm_prefix, ptext = [(self.TEXT, t) for t in ptext[:eop + 1]], ptext[eop + 1:]
        self.pspeech = [int(x) for x in prompt_speech_token.reshape(-1).tolist()]
        self.lm_input = [(self.LLM, 0)] + lm_prefix
        self.text_cache = list(ptext)
        self.out_tokens = []
        self.next_fill_index = (len(self.pspeech) // self.MIX_SPEECH + 1) * self.MIX_SPEECH - len(self.pspeech)
        self.fed = 0                       # positions pushed so far (the session's context)
        self.state = self.WAIT

    def add_text(self, ids):
        """one chunk of the text generator (llm.py:593-613): interleave prompt speech, then enter the decode loop if possible"""
        T, M = self.MIX_TEXT, self.MIX_SPEECH
        self.text_cache += [int(x) for x in ids]
        while self.pspeech:                                            # llm.py:595-604
            if len(self.text_cache) >= T:
                self.lm_input = self.lm_input + [(self.TEXT, t) for t in self.text_cache[:T]] + [(self.SPEECH, t) for t in self.pspeech[:M]]
                self.text_cache, self.pspeech = self.text_cache[T:], self.pspeech[M:]
            else:
                break
        if self.pspeech:
            return
        out = self.out_tokens                                          # llm.py:606-613
        if (out and out[-1] == self.fill_token) or (not out and len(self.lm_input) == 1):
            if len(self.text_cache) < T:
                return
            lm_text = [(self.TEXT, t) for t in self.text_cache[:T]]
            self.lm_input = lm_text if (out and out[-1] == self.fill_token) else self.lm_input + lm_text
            self.text_cache = self.text_cache[T:]
        self.state = self.DECODE

    def end_text(self):
        """the text generator is exhausted (llm.py:643)"""
        self.lm_input = self.lm_input + [(self.TEXT, t) for t in self.text_cache] + [(self.LLM, 1)]
        self.state = self.FINAL
        self._check_cap()

    def _check_cap(self):
        # benchmark aid (bistream_max_tokens): the final phase ends after this many ids
        if self.state == self.FINAL and self.max_tokens is not None and len(self.out_tokens) >= self.max_tokens:
            self.state = self.DONE

    def forced(self):
        """the id of this step is a forced fill token (llm.py:624-626); the reference still runs the model first"""
        return self.state == self.DECODE and self.next_fill_index != -1 and len(self.out_tokens) == self.next_fill_index

    def ignore_eos(self):
        return self.state == self.DECODE

    def take(self, top):
        """the id of this step (ignored when forced); returns the id to yield, or None.  Raises ValueError like the reference."""
        if self.state == self.DECODE:
            if self.forced():
                top = self.fill_token
                self.next_fill_index += self.MIX_SPEECH + 1
            if top == self.fill_token:
                self.next_fill_index = len(self.out_tokens) + self.MIX_SPEECH + 1
            self.out_tokens.append(top)
            if top >= self.SPEECH_VOCAB:
                if top == self.fill_token:
                    self.state = self.WAIT
                    return None
                raise ValueError(f"should not get token {top}")
        else:
            self.out_tokens.append(top)
            if top >= self.SPEECH_VOCAB:
                if top == self.eos_token:
                    self.state = self.DONE
                    return None
                raise ValueError(f"should not get token {top}")
        self.lm_input = [(self.SPEECH, top)]
        self._check_cap()
        return top


def cfm_rand_noise():
    """CausalConditionalCFM.rand_noise (flow/flow_matching.py:199-200): seed-0 torch.randn([1,80,15000]), time-major."""
    g = torch.Generator(device="cpu")
    g.manual_seed(0)
    return torch.randn([1, 80, 50 * 300], generator=g)[0].t().contiguous()


class B200CosyVoice2Model:
    # text-streaming LM constants: Qwen2LM (llm.py:275-277: eos = speech_token_size, fill = speech_token_size + 2, whole
    # prompt text goes into the text cache).  B200CosyVoice3Model overrides them (CosyVoice3LM, llm.py:681-684, 583-588).
    bistream_fill_token = 6563
    bistream_eos_token = 6561
    bistream_eop_token = None
    # benchmark aid only (None = the reference's behaviour: decode "until met eos", llm.py:642-661, without any cap): random-init
    # weights cannot be made to emit eos at a chosen time, so bench.py ends the text-streaming decode after this many ids
    bistream_max_tokens = None
    bistream_max_ctx = 4096              # positions of the text-streaming LM session (per request)
    # streaming synthesis: intermediate chunks through the cached flow session (cvk_flow_stream_*: each chunk computes only its new
    # frames) instead of the reference's prefix recompute (cli/model.py:346-363); same frames either way.  The U-Net estimator of
    # B200CosyVoice3Model uses the same sessions for its DiT.
    incremental_flow = True
    flow_stream_dit = False              # which estimator the sessions cache: the CosyVoice2 U-Net (stage "flow") or the CosyVoice3 DiT ("flow3")
    stream_cache_frames = 2048           # mel frames (prompt included) one streaming request can cache (41 s); ~2.3 MB per frame in bf16
    # tts_stream_batch: the most slots of the one multi-slot flow session the model creates on first use, each caching
    # stream_cache_frames frames (~2.3 MB per frame for the full-size U-Net in bf16: 16 x 2048 frames would be 75 GB).  The session
    # takes the largest of stream_batch_slots, /2, /4, ... that allocates and leaves stream_pool_headroom bytes of device memory free
    # for LM sessions and activations (8 slots next to a full-size model with the default 24 GB workspace on an 80 GB card);
    # `stream_slots` reports the outcome.  0 = no session.  Requests that find no free slot recompute their prefix like the reference.
    stream_batch_slots = 16
    stream_pool_headroom = 8 << 30
    stream_slots = None                  # slots of the session once tts_stream_batch has tried to create it (0: none fitted)
    _slot_pool = None                    # the multi-slot cvk_flow_stream handle, once created
    _free_slots = None                   # its free slot indices

    def __init__(self, llm=None, flow=None, hift=None, fp16=False, precision="bf16", device=0, workspace_gb=24.0):
        # attribute names follow cli/model.py:245-275
        self.device = torch.device("cuda", device)
        self.llm, self.flow, self.hift = llm, flow, hift
        self.fp16 = fp16
        self.token_hop_len = 25
        self.token_max_hop_len = 4 * self.token_hop_len
        self.stream_scale_factor = 2
        self.mel_cache_len = 8
        self.source_cache_len = int(self.mel_cache_len * 480)
        self.speech_window = np.hamming(2 * self.source_cache_len)
        self.lock = threading.Lock()
        self.tts_speech_token_dict = {}
        self.llm_end_dict = {}
        self.hift_cache_dict = {}
        self.silent_tokens = []
        self.ctx = cvk.Context(device, precision, workspace_gb)
        self.stream = torch.cuda.Stream(self.device)     # every library call of this model runs on this stream
        self.generator = torch.Generator(device=self.device)
        self.generator.manual_seed(1986)
        self._free_sessions = {}             # (B, ctx rounded to 256) -> idle cvk_lm_session handles (see _checkout_session)
        self._session_lru = []               # keys of idle sessions, least recently returned first
        self.max_idle_sessions = 4
        self._pool_lock = threading.Lock()
        self._lm_streams = []
        self._idle_lm_streams = []           # LM job streams not in use (see _lm_stream)
        self.flow_stream_dict = {}           # uuid -> cvk_flow_stream handle, or False once a request has left the chunk grid
        self._idle_flow_streams = []
        self.lm_chains = 1                   # independent decode chains run concurrently (see lm_generate)
        self._window = torch.from_numpy(self.speech_window).float().to(self.device)
        self.n_timesteps = 10
        self.min_token_text_ratio, self.max_token_text_ratio = 2.0, 20.0
        self.timings = {}
        # test hooks: explicit random streams instead of the device generator (the reference uses the global torch RNG)
        self.uniforms_override = None        # tensor [steps, B, 2]
        self.noise_fn = None                 # callable(n_samples) -> [n_samples, 9]
        if llm is not None and flow is not None and hift is not None:
            self.load_state_dicts(_state_dict(llm), _state_dict(flow), _state_dict(hift))

    # ---------------------------------------------------------------- weights (cli/model.py:65-73)
    def load(self, llm_model, flow_model, hift_model):
        llm_sd = torch.load(llm_model, map_location="cpu", weights_only=True)
        flow_sd = torch.load(flow_model, map_location="cpu", weights_only=True)
        hift_sd = {k.replace("generator.", ""): v for k, v in torch.load(hift_model, map_location="cpu", weights_only=True).items()}
        self.load_state_dicts(llm_sd, flow_sd, hift_sd)

    def load_state_dicts(self, llm_sd, flow_sd, hift_sd):
        llm_cfg, flow_cfg = infer_cfgs(llm_sd, flow_sd)
        self.ctx.load_state_dict("llm", llm_sd, llm_cfg)
        self.ctx.load_state_dict("flow", flow_sd, flow_cfg)
        self.ctx.load_state_dict("hift", hift_sd)
        self.ctx.set_cfm_noise(cfm_rand_noise())
        self.ctx.finalize("mel")

    # engine swap points of the reference are meaningless here; kept so that CosyVoice2.__init__ flags fail loudly
    def load_jit(self, *a, **k):
        raise RuntimeError("B200CosyVoice2Model has no TorchScript path (cli/model.py:277-279 swap point is replaced by libcvk)")

    def load_trt(self, *a, **k):
        raise RuntimeError("B200CosyVoice2Model has no TensorRT path (the estimator runs in libcvk)")

    def load_vllm(self, *a, **k):
        raise RuntimeError("B200CosyVoice2Model has no vLLM path (the LM runs in libcvk)")

    # ---------------------------------------------------------------- LM (llm/llm.py:458-549), batched
    def _checkout_session(self, B, ctx_len):
        """An LM session (KV cache + decode buffers + captured step graph) is owned by ONE generation from prefill to the last
        token: the reference keeps per-request state keyed by uuid (cli/model.py:334-337) and serves overlapping tts() calls
        from threads, so two requests of similar shape must never share a KV cache.  Idle sessions are kept for re-use
        (creating one allocates hundreds of MB at batch 32) and the idle pool is bounded (LRU, cvk_lm_session_destroy)."""
        key = (B, (ctx_len + 255) // 256 * 256)
        with self._pool_lock:
            free = self._free_sessions.get(key)
            if free:
                self._session_lru.remove(key)
                return key, free.pop()
        return key, self.ctx.lm_session(*key)

    @contextmanager
    def _lm_stream(self):
        """A stream that belongs to one LM job until it ends.  The decode step graph is captured on it, so it must never be the
        model's stream or another job's: torch's pooled streams are handed out round-robin from 32 per device and repeat after 32
        creations, so they come from cvk_stream_create instead and are recycled here."""
        if self.device.type != "cuda":
            yield None
            return
        with self._pool_lock:
            s = self._idle_lm_streams.pop() if self._idle_lm_streams else None
        if s is None:
            s = self.ctx.stream_create()
        try:
            yield s
        finally:
            s.synchronize()
            with self._pool_lock:
                self._idle_lm_streams.append(s)

    def _checkin_session(self, key, sess):
        evict = []
        with self._pool_lock:
            self._free_sessions.setdefault(key, []).append(sess)
            self._session_lru.append(key)
            while len(self._session_lru) > self.max_idle_sessions:
                k = self._session_lru.pop(0)
                evict.append(self._free_sessions[k].pop(0))
        for e in evict:
            self.ctx.lm_session_destroy(e)

    def lm_generate(self, texts, prompt_texts, prompt_speech_tokens, uniforms=None, steps_per_sync=32, on_progress=None, stream=None):
        """texts/prompt_texts/prompt_speech_tokens: lists of int32 tensors [1,n].  Returns a list of python id lists.

        `stream`: CUDA stream for this generation (default: the model's stream).  Only the prefill uses the shared workspace and
        takes `ctx.lock`; the decode calls touch nothing but their own session (include/cvk.h threading rules), so a request's
        LM job on its own stream overlaps another request's - or its own - flow / vocoder calls like the reference's LM thread
        does (cli/model.py:101-129, 268).

        `self.lm_chains > 1` splits the rows into independent groups, each with its own KV session, CUDA graph and stream (an
        experiment knob from the per-op decode chain).  Results are independent of the grouping (rows never interact; every row
        consumes its own uniforms)."""
        B = len(texts)
        d = self.device
        main = stream if stream is not None else self.stream
        chains = 1 if on_progress is not None else max(1, min(self.lm_chains, B))
        groups = [list(range(g, B, chains)) for g in range(chains)]
        mins = [int(t.shape[1] * self.min_token_text_ratio) for t in texts]      # llm.py:497-498
        maxs = [int(t.shape[1] * self.max_token_text_ratio) for t in texts]
        mx = max(maxs)
        st = []
        try:
            # The prefill uses the context's shared workspace arena, so it runs on the model's stream under ctx.lock like every other
            # workspace call (flow / vocoder): the lock orders the host calls, the common stream orders the device work.  Only the
            # decode steps - which touch nothing but their session - run on the generation's own stream.
            with torch.cuda.stream(self.stream):
                if uniforms is None and self.uniforms_override is not None:
                    uniforms = self.uniforms_override
                if uniforms is None:
                    with self.lock:                                  # one device generator shared by the request threads
                        uniforms = torch.rand(mx + 1, B, 2, device=d, generator=self.generator)
                uniforms = uniforms.to(d).float()
                for g, rows in enumerate(groups):
                    tl = [int(texts[r].shape[1] + prompt_texts[r].shape[1]) for r in rows]
                    sl = [int(prompt_speech_tokens[r].shape[1]) for r in rows]
                    tt = torch.cat([torch.cat([prompt_texts[r].reshape(-1).to(d, non_blocking=True), texts[r].reshape(-1).to(d, non_blocking=True)])
                                    for r in rows]).to(torch.int32)
                    ss = torch.cat([prompt_speech_tokens[r].reshape(-1).to(d, non_blocking=True) for r in rows]).to(torch.int32) if sum(sl) \
                        else torch.zeros(1, dtype=torch.int32, device=d)
                    key, sess = self._checkout_session(len(rows), max(a + b2 for a, b2 in zip(tl, sl)) + 2 + mx + 8)
                    c = dict(rows=rows, n=len(rows), key=key, sess=sess,
                             min_len=torch.tensor([mins[r] for r in rows], dtype=torch.int32, device=d),
                             max_len=torch.tensor([maxs[r] for r in rows], dtype=torch.int32, device=d),
                             max_len_host=torch.tensor([maxs[r] for r in rows], dtype=torch.int32),
                             out_ids=torch.zeros(len(rows), mx + 1, dtype=torch.int32, device=d),
                             out_count=torch.zeros(len(rows), dtype=torch.int32, device=d),
                             done=torch.zeros(len(rows), dtype=torch.int32, device=d),
                             U=uniforms[:, rows, :].contiguous(), live=len(rows))
                    st.append(c)
                    with self.ctx.lock:
                        self.ctx.lm_prefill(sess, tt, tl, ss, sl)
                        ready = torch.cuda.Event()
                        ready.record(self.stream)
                    c["ready"] = ready
            while len(self._lm_streams) < chains:
                self._lm_streams.append(self.ctx.stream_create())
            n = 0
            for c in st:
                c["left"] = mx                     # upper bound of the steps this chain still needs (refined after every block)
            while True:
                for g, c in enumerate(st):
                    if c["live"] == 0:
                        continue
                    s_g = main if chains == 1 else self._lm_streams[g]
                    with torch.cuda.stream(s_g):
                        if n == 0:
                            s_g.wait_event(c["ready"])
                        # never run past the longest possible remainder: the last block is cut to what the live rows can still emit
                        # (round 1 always ran whole blocks: 320 steps for rows that end at 300)
                        c["block"] = max(1, min(steps_per_sync, c["left"]))
                        self.ctx.lm_decode(c["sess"], c["block"], c["U"], c["min_len"], c["max_len"], c["out_ids"], c["out_count"], c["done"],
                                           want_live=False)
                for g, c in enumerate(st):
                    if c["live"] == 0:
                        continue
                    s_g = main if chains == 1 else self._lm_streams[g]
                    with torch.cuda.stream(s_g):
                        c["live"] = self.ctx.lm_decode(c["sess"], 0, c["U"], c["min_len"], c["max_len"], c["out_ids"], c["out_count"], c["done"])
                        if c["live"]:
                            cnt, dn = c["out_count"].cpu(), c["done"].cpu()
                            c["left"] = int(((c["max_len_host"] - cnt) * (dn == 0)).max())
                n += steps_per_sync
                if on_progress is not None:
                    on_progress(st[0]["out_ids"], st[0]["out_count"], st[0]["live"])
                if all(c["live"] == 0 for c in st) or n > mx + steps_per_sync:
                    break
            out = [None] * B
            for g, c in enumerate(st):
                with torch.cuda.stream(main if chains == 1 else self._lm_streams[g]):
                    cnt = c["out_count"].cpu().tolist()
                    ids = c["out_ids"].cpu()
                for i, r in enumerate(c["rows"]):
                    out[r] = ids[i, :cnt[i]].tolist()
            if chains > 1:
                for g in range(chains):
                    main.wait_stream(self._lm_streams[g])
            return out
        finally:
            main.synchronize()                     # the session goes back to the pool only when its last kernel has finished
            for c in st:
                self._checkin_session(c["key"], c["sess"])

    def lm_generate_bistream(self, text, prompt_text, prompt_speech_token, uniforms=None, stream=None):
        """llm/llm.py:551-661 (Qwen2LM.inference_bistream): `text` is a generator of int32 [1,k] chunks; speech ids are yielded
        as soon as they are decoded.  The interleaving (5 text : 15 speech), the forced / sampled fill tokens and the final
        'decode until eos' phase are the reference's control flow line for line; the arithmetic runs on the device through
        cvk_lm_begin / cvk_lm_feed / cvk_lm_next_logp / cvk_ras_sample.  uniforms [n,2]: row len(out_tokens) is consumed by the
        draw that produces that token (default: drawn from the model's generator)."""
        d = self.device
        row = self._bistream_row(prompt_text, prompt_speech_token)
        max_ctx = self.bistream_max_ctx
        lm_stream = stream if stream is not None else self.stream
        key, sess = self._checkout_session(1, max_ctx - 8)
        with torch.cuda.stream(lm_stream):
            self.ctx.lm_begin(sess, 1)
        if uniforms is None and self.uniforms_override is not None:
            uniforms = self.uniforms_override[:, 0, :]

        def step():
            """llm.py:617-627 / 648-650: push lm_input through the cached model, then the forced id or a draw (sampling_ids)"""
            with torch.cuda.stream(lm_stream):
                self._bistream_count_fed(row)
                self.ctx.lm_feed(sess, [i for _, i in row.lm_input], [k for k, _ in row.lm_input])
                if row.forced():                                      # the reference runs the model before overriding the draw
                    return row.take(None)
                logp = self.ctx.lm_next_logp(sess, 1)
                i = len(row.out_tokens)
                if uniforms is not None:
                    u = uniforms[i].reshape(1, 2)
                else:
                    with self.lock:
                        u = torch.rand(1, 2, device=d, generator=self.generator)
                hist, cnt = self._bistream_history([row])
                top = self.ctx.ras_sample(logp, hist, cnt, u, torch.tensor([1 if row.ignore_eos() else 0], dtype=torch.int32))
                return row.take(int(top.item()))

        try:
            for this_text in text:
                row.add_text(this_text.reshape(-1).tolist())
                while row.state == row.DECODE:
                    top = step()
                    if top is not None:
                        yield top
            row.end_text()
            while row.state == row.FINAL:
                top = step()
                if top is not None:
                    yield top
        finally:
            if lm_stream is not None:
                lm_stream.synchronize()
            self._checkin_session(key, sess)

    def _bistream_row(self, prompt_text, prompt_speech_token):
        return _BistreamRow(self.bistream_fill_token, self.bistream_eos_token, self.bistream_eop_token, prompt_text, prompt_speech_token,
                            self.bistream_max_tokens)

    def _bistream_count_fed(self, row):
        row.fed += len(row.lm_input)
        if row.fed >= self.bistream_max_ctx - 16:
            raise RuntimeError("text-streaming LM: session context exhausted")

    @staticmethod
    def _bistream_history(rows):
        """the rows' last 16 ids (zero-padded) and their counts: the repetition window of sampling_ids (common.py:138-149)"""
        hist = torch.tensor([(r.out_tokens[-16:] + [0] * 16)[:16] for r in rows], dtype=torch.int32)
        return hist, torch.tensor([min(len(r.out_tokens), 16) for r in rows], dtype=torch.int32)

    def lm_generate_bistream_batch(self, texts, prompt_texts, prompt_speech_tokens, uniforms=None, stream=None):
        """lm_generate_bistream for several requests in one LM session: a generator of (i, id) as request i's ids are decoded.

        `texts` are generators of int32 [1,k] chunks; one feeder thread per generator moves its chunks into a queue.  Every step
        makes one cvk_lm_feed_rows call for all rows whose state machine can advance (rows waiting for text sit the step out), one
        cvk_lm_next_logp_rows + one cvk_ras_sample call for the rows that draw (forced fill tokens do not), and one device-to-host
        copy of the drawn ids - the step's only host sync (the sampler's small inputs go through pinned memory).  uniforms [n, B, 2]: uniforms[k, i] is row i's draw for
        len(out_tokens) == k, as in lm_generate_bistream.  A row's ids depend only on its own chunks and uniforms, not on arrival
        timing or on which rows share a step.  A row error (ValueError for an unexpected special id, AssertionError for a CosyVoice3
        prompt without <|endofprompt|>) ends the whole generator; closing it stops within one step and returns the session."""
        import queue
        B = len(texts)
        d = self.device
        rows = [self._bistream_row(pt, ps) for pt, ps in zip(prompt_texts, prompt_speech_tokens)]
        if uniforms is None and self.uniforms_override is not None:
            uniforms = self.uniforms_override
        lm_stream = stream if stream is not None else self.stream
        arrivals = queue.Queue()               # (row, chunk ids) / (row, None) at the end / (row, exception)
        pending = [[] for _ in range(B)]
        stop = threading.Event()

        def feeder(i, gen):
            try:
                for chunk in gen:
                    if stop.is_set():
                        return
                    arrivals.put((i, chunk.reshape(-1).tolist()))
                arrivals.put((i, None))
            except BaseException as e:        # noqa: BLE001  (re-raised by the generator)
                arrivals.put((i, e))

        key, sess = self._checkout_session(B, self.bistream_max_ctx - 8)
        try:
            with torch.cuda.stream(lm_stream):
                self.ctx.lm_begin(sess, B)
            for i, gen in enumerate(texts):
                threading.Thread(target=feeder, args=(i, gen), name=f"cvk-bistream-text-{i}", daemon=True).start()
            while True:
                # take what has arrived (and block for more when no row can advance)
                while True:
                    try:
                        i, item = arrivals.get_nowait()
                    except queue.Empty:
                        break
                    pending[i].append(item)
                for i, r in enumerate(rows):
                    while r.state == r.WAIT and pending[i]:
                        item = pending[i].pop(0)
                        if isinstance(item, BaseException):
                            raise item
                        if item is None:
                            r.end_text()
                        else:
                            r.add_text(item)
                adv = [i for i, r in enumerate(rows) if r.state in (r.DECODE, r.FINAL)]
                if not adv:
                    if all(r.state == r.DONE for r in rows):
                        return
                    i, item = arrivals.get()
                    pending[i].append(item)
                    continue
                with torch.cuda.stream(lm_stream):
                    for i in adv:
                        self._bistream_count_fed(rows[i])
                    self.ctx.lm_feed_rows(sess, adv, [len(rows[i].lm_input) for i in adv],
                                          [t for i in adv for _, t in rows[i].lm_input], [k for i in adv for k, _ in rows[i].lm_input])
                    draw = [i for i in adv if not rows[i].forced()]
                    drawn = {}
                    if draw:
                        logp = self.ctx.lm_next_logp_rows(sess, draw)
                        if uniforms is not None:
                            u = _to_device(torch.stack([uniforms[len(rows[i].out_tokens), i] for i in draw]).reshape(len(draw), 2), d)
                        else:
                            with self.lock:
                                u = torch.rand(len(draw), 2, device=d, generator=self.generator)
                        hist, cnt = self._bistream_history([rows[i] for i in draw])
                        ign = torch.tensor([1 if rows[i].ignore_eos() else 0 for i in draw], dtype=torch.int32)
                        top = self.ctx.ras_sample(logp, _to_device(hist, d), _to_device(cnt, d), u, _to_device(ign, d)).cpu().tolist()
                        drawn = dict(zip(draw, top))
                for i in adv:
                    top = rows[i].take(drawn.get(i))
                    if top is not None:
                        yield i, top
        finally:
            stop.set()
            if lm_stream is not None:
                lm_stream.synchronize()
            self._checkin_session(key, sess)

    # ---------------------------------------------------------------- flow + vocoder
    def flow_batch(self, tokens, prompt_tokens, prompt_feats, embeddings, streaming=False, finalize=True):
        """lists per utterance: tokens [1,N] int, prompt_tokens [1,P], prompt_feats [1,Tp,80], embeddings [1,192]
        -> (mel [sum T,80] time-major on the device, lens)"""
        d = self.device
        tl = [int(t.shape[1] + p.shape[1]) for t, p in zip(tokens, prompt_tokens)]
        pl = [int(f.shape[1]) for f in prompt_feats]
        with torch.cuda.stream(self.stream), self.ctx.lock:
            toks = torch.cat([torch.cat([p.reshape(-1).to(d, non_blocking=True), t.reshape(-1).to(d, non_blocking=True)])
                              for t, p in zip(tokens, prompt_tokens)]).to(torch.int32)
            pf = torch.cat([f[0].to(d, non_blocking=True) for f in prompt_feats], 0) if sum(pl) else None
            emb = torch.cat([e.reshape(1, -1).to(d, non_blocking=True) for e in embeddings], 0)
            return self.ctx.flow_inference(toks, tl, pf, pl, emb, n_timesteps=self.n_timesteps, streaming=streaming, finalize=finalize)

    def _vocoder_noise(self, n, noise_fn=None):
        """vocoder noise for n samples: from noise_fn when given, else from the model's noise_fn hook or its generator"""
        noise_fn = noise_fn if noise_fn is not None else self.noise_fn
        if noise_fn is not None:
            return noise_fn(n).to(self.device)
        return torch.randn(n, 9, device=self.device, generator=self.generator)

    def hift_batch(self, mel_tm, lens, cache_source=None, cache_lens=None, noise=None):
        with torch.cuda.stream(self.stream), self.ctx.lock:
            if noise is None:
                noise = self._vocoder_noise(sum(lens) * SAMPLES_PER_FRAME)
            return self.ctx.hift_inference(mel_tm, lens, noise, cache_source, cache_lens)

    def tts_batch_device(self, inputs, uniforms=None, noise=None):
        """The batched pipeline with the result left on the device: returns (wav_flat, lens, stats) - wav_flat is the vocoder's
        output buffer (float32 [sum n_i], the utterances back to back in input order, empty ones skipped), lens[i] the sample
        count of input i (0 when the LM produced no token).  Used by tts_batch and by the multi-GPU gather (parallel.gather_flat).

        Every request kind tts() serves: a missing key takes tts()'s default; a voice-conversion request (non-empty
        source_speech_token) takes those tokens as its speech tokens, without the LM and without the silent-token rule, like vc_job;
        the LM runs over the other rows only (request i still draws uniforms[:, i]) and not at all when there are none.  `speed`
        (default 1) stretches a request's mel after the flow as token2wav does (mel_stretch, one call for the batch, made only when
        some request has speed != 1); the vocoder, its noise draw, the sample counts and stats["mel_frames"] follow the stretched
        lengths, stats["flow_frames"] holds the flow's.  A speed <= 0 is a ValueError before any device work."""
        speeds = [request_speed(r) for r in inputs]
        vc = [b for b, r in enumerate(inputs) if is_vc_request(r)]
        lm_rows = [b for b in range(len(inputs)) if b not in vc]
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        with torch.cuda.stream(self.stream):
            ev[0].record()
        ids = [None] * len(inputs)
        for b in vc:
            ids[b] = request_field(inputs[b], "source_speech_token").flatten().tolist()
        if lm_rows:
            if vc and uniforms is None:
                uniforms = self.uniforms_override
            if vc and uniforms is not None:
                uniforms = uniforms[:, lm_rows]
            lm_ids = self.lm_generate([request_field(inputs[b], "text") for b in lm_rows], [request_field(inputs[b], "prompt_text") for b in lm_rows],
                                      [request_field(inputs[b], "llm_prompt_speech_token") for b in lm_rows], uniforms)
            for b, x in zip(lm_rows, lm_ids):
                ids[b] = SilentTokenFilter(self.silent_tokens).filter(x)      # what tts() keeps of each request's ids
        with torch.cuda.stream(self.stream):
            ev[1].record()
        toks = [torch.tensor(x, dtype=torch.int32).unsqueeze(0) for x in ids]
        keep = [b for b, x in enumerate(ids) if len(x) > 0]
        mel, lens = self.flow_batch([toks[b] for b in keep], [request_field(inputs[b], "flow_prompt_speech_token") for b in keep],
                                    [request_field(inputs[b], "prompt_speech_feat") for b in keep],
                                    [request_field(inputs[b], "flow_embedding") for b in keep])
        flow_lens = list(lens)
        with torch.cuda.stream(self.stream):
            ev[2].record()
        if any(speeds[b] != 1.0 for b in keep):
            mel, lens = self.mel_stretch(mel, lens, [speeds[b] for b in keep])
        wav, _ = self.hift_batch(mel, lens, noise=noise)
        with torch.cuda.stream(self.stream):
            ev[3].record()
        n = [0] * len(inputs)
        for b, L in zip(keep, lens):
            n[b] = L * SAMPLES_PER_FRAME
        stats = {"ev": ev, "tokens": [len(x) for x in ids], "mel_frames": lens, "flow_frames": flow_lens}
        return wav, n, stats

    def mel_stretch(self, mel, lens, speeds):
        """token2wav's speed change (cli/model.py:320-322) for a ragged batch in one cvk_mel_resample call: utterance b's lens[b]
        frames of mel [sum lens, 80] are linearly resampled to int(lens[b] / speeds[b]) frames, the length tts() computes, bit for
        bit what F.interpolate(mode="linear") gives on the device (speed 1 copies).  Returns (mel, stretched lens); a stretched
        length of 0 is a ValueError before the call (F.interpolate refuses it too)."""
        out = [int(T / s) for T, s in zip(lens, speeds)]
        for T, s, n in zip(lens, speeds, out):
            if n < 1:
                raise ValueError(f"speed {s} stretches a mel of {T} frames to 0 frames")
        with torch.cuda.stream(self.stream), self.ctx.lock:
            return self.ctx.mel_resample(mel, lens, out), out

    def _stage_ms(self, stats):
        ev = stats.pop("ev")
        stats.update({"lm_ms": ev[0].elapsed_time(ev[1]), "flow_ms": ev[1].elapsed_time(ev[2]), "hift_ms": ev[2].elapsed_time(ev[3])})
        return stats

    def tts_batch(self, inputs, uniforms=None, noise=None, return_stats=False, to_host=True):
        """inputs: list of dicts with the kwargs of tts() (text, prompt_text, llm_prompt_speech_token,
        flow_prompt_speech_token, prompt_speech_feat, flow_embedding, source_speech_token, speed), any of them left out as tts()
        allows.  Each request gets what tts() gives it alone (tts_batch_device).  Returns a list of waveforms [1,N] (CPU tensors, or
        views of one device buffer when to_host=False)."""
        wav, n, stats = self.tts_batch_device(inputs, uniforms, noise)
        with torch.cuda.stream(self.stream):
            host = wav.cpu() if to_host else wav          # one D2H for the whole batch
        self.stream.synchronize()
        out, o = [], 0
        for k in n:
            out.append(host[o:o + k].unsqueeze(0) if k else torch.zeros(1, 0))
            o += k
        self.timings = self._stage_ms(stats)
        return (out, dict(self.timings)) if return_stats else out

    # ---------------------------------------------------------------- reference-shaped single-request API
    def _fade_in_out(self, fade_in, fade_out):
        """utils/common.py:170-178 without the CPU round trip."""
        n = self.source_cache_len
        fade_in = fade_in.clone()
        fade_in[..., :n] = fade_in[..., :n] * self._window[:n] + fade_out[..., -n:] * self._window[n:]
        return fade_in

    def _to_host(self, t):
        """D2H on the model's stream (the kernels that produced `t` were enqueued there, not on torch's current stream)."""
        with torch.cuda.stream(self.stream):
            h = t.cpu()
        self.stream.synchronize()
        return h

    def _session_chunk_ok(self, P, prompt_frames, n_tokens, token_offset, has_session):
        """Whether the streaming chunk of the first n_tokens speech tokens (look-ahead included) past token_offset can come from a
        cached flow session: it starts and ends on the STREAM_CHUNK_FRAMES grid, the prompt mel has TOKEN_MEL_RATIO frames per
        prompt token (P of them), its frames fit in stream_cache_frames, and the request has held a session since its first chunk."""
        total = TOKEN_MEL_RATIO * (P + n_tokens - PRE_LOOKAHEAD)
        done = TOKEN_MEL_RATIO * (P + token_offset) if token_offset else 0
        return (total % STREAM_CHUNK_FRAMES == 0 and done % STREAM_CHUNK_FRAMES == 0 and prompt_frames == TOKEN_MEL_RATIO * P
                and total <= self.stream_cache_frames and (has_session or token_offset == 0))

    def _flow_stream_chunk(self, token, prompt_token, prompt_feat, embedding, token_offset, uuid):
        """The frames of this streaming chunk from the request's cached flow session, or None when the request cannot use one
        (_session_chunk_ok): the caller then recomputes the prefix like the reference."""
        if not self.incremental_flow or uuid not in self.tts_speech_token_dict:
            return None
        fs = self.flow_stream_dict.get(uuid)
        if fs is False:
            return None
        if not self._session_chunk_ok(int(prompt_token.shape[1]), int(prompt_feat.shape[1]), int(token.shape[1]), token_offset,
                                      fs is not None):
            if fs:
                self._release_flow_stream(uuid)
            self.flow_stream_dict[uuid] = False
            return None
        d = self.device
        with torch.cuda.stream(self.stream), self.ctx.lock:
            if fs is None:
                with self._pool_lock:
                    fs = self._idle_flow_streams.pop() if self._idle_flow_streams else None
                if fs is None:
                    try:
                        fs = self.ctx.flow_stream(self.stream_cache_frames, self.n_timesteps, dit=self.flow_stream_dit)
                    except cvk.CvkError:
                        # no memory for another session's caches (several GB each): this request recomputes the prefix like the reference
                        self.flow_stream_dict[uuid] = False
                        return None
                self.flow_stream_dict[uuid] = fs
                self.ctx.flow_stream_begin(fs, prompt_feat[0].to(d, non_blocking=True), embedding.reshape(-1).to(d, non_blocking=True))
            toks = torch.cat([prompt_token.reshape(-1).to(d, non_blocking=True), token.reshape(-1).to(d, non_blocking=True)]).to(torch.int32)
            return self.ctx.flow_stream_chunk(fs, toks)

    def _release_flow_stream(self, uuid):
        fs = self.flow_stream_dict.pop(uuid, None)
        if fs:
            with self._pool_lock:
                if len(self._idle_flow_streams) < 2:
                    self._idle_flow_streams.append(fs)
                    fs = None
            if fs:
                self.stream.synchronize()
                self.ctx.flow_stream_destroy(fs)

    def _token2wav_mel(self, token, prompt_token, prompt_feat, embedding, token_offset, uuid, stream, finalize):
        """The flow half of token2wav: the mel frames past token_offset, from the request's cached flow session when a streaming
        chunk can use one (_flow_stream_chunk), else from the flow over the whole prefix like the reference (cli/model.py:294-303)."""
        token = token.to(torch.int32)
        mel = self._flow_stream_chunk(token, prompt_token, prompt_feat, embedding, token_offset, uuid) if (stream and not finalize) else None
        if mel is None:
            mel, _ = self.flow_batch([token], [prompt_token], [prompt_feat], [embedding], streaming=stream, finalize=finalize)
            mel = mel[token_offset * TOKEN_MEL_RATIO:]
        return mel

    def _vocode_cached(self, caches, mels, finals, noise_fns):
        """CosyVoice2's vocoder bookkeeping (cli/model.py:304-326) for several requests in one vocoder call.  Request k has its cache
        dict caches[k] (None before its first chunk), its new mel frames mels[k], finals[k] for its final call and its noise stream
        noise_fns[k] (None: _vocoder_noise's default).  Its cached mel frames are prepended, its cached source is passed to the
        vocoder and its waveform is cross-faded with its cached speech; unless final, its caches are renewed and the last
        source_cache_len samples are held back.  Returns (the requests' waveforms on the device, their caches)."""
        with torch.cuda.stream(self.stream):
            tts_mel = [torch.cat([c["mel"], m], 0) if c is not None else m for c, m in zip(caches, mels)]
            lens = [int(m.shape[0]) for m in tts_mel]
            noise = torch.cat([self._vocoder_noise(n * SAMPLES_PER_FRAME, fn) for n, fn in zip(lens, noise_fns)], 0)
            cached = [c for c in caches if c is not None]
            cache_lens = [int(c["source"].shape[0]) if c is not None else 0 for c in caches] if cached else None
            wav, src = self.hift_batch(torch.cat(tts_mel, 0), lens, torch.cat([c["source"] for c in cached]) if cached else None, cache_lens,
                                       noise)
            wavs, new_caches, o = [], [], 0
            for c, m, n, final in zip(caches, tts_mel, lens, finals):
                w, s = wav[o * SAMPLES_PER_FRAME:(o + n) * SAMPLES_PER_FRAME], src[o * SAMPLES_PER_FRAME:(o + n) * SAMPLES_PER_FRAME]
                o += n
                if c is not None:
                    w = self._fade_in_out(w, c["speech"])
                if not final:
                    c = {"mel": m[-self.mel_cache_len:].clone(), "source": s[-self.source_cache_len:].clone(),
                         "speech": w[-self.source_cache_len:].clone()}
                    w = w[:-self.source_cache_len]
                wavs.append(w)
                new_caches.append(c)
        return wavs, new_caches

    def token2wav(self, token, prompt_token, prompt_feat, embedding, token_offset, uuid, stream=False, finalize=False, speed=1.0):
        """cli/model.py:292-326"""
        mel = self._token2wav_mel(token, prompt_token, prompt_feat, embedding, token_offset, uuid, stream, finalize)
        cache = self.hift_cache_dict[uuid]
        if finalize and speed != 1.0:
            assert cache is None, "speed change only support non-stream inference mode"
            mel, _ = self.mel_stretch(mel, [mel.shape[0]], [speed])
        wavs, caches = self._vocode_cached([cache], [mel], [finalize], [None])
        self.hift_cache_dict[uuid] = caches[0]
        return wavs[0].unsqueeze(0)

    def llm_job(self, text, prompt_text, llm_prompt_speech_token, llm_embedding, uuid):
        """cli/model.py:101-129 (non-generator text).  Tokens are appended to the session list as they arrive."""
        if hasattr(text, "__next__") or (hasattr(text, "__iter__") and not torch.is_tensor(text)):
            # cli/model.py:113-123: text generator -> bi-stream decoding, tokens appended one by one
            silent = SilentTokenFilter(self.silent_tokens)
            with self._lm_stream() as lm_stream:
                for tok in self.lm_generate_bistream(iter(text), prompt_text, llm_prompt_speech_token, stream=lm_stream):
                    if silent.keep(tok):
                        self.tts_speech_token_dict[uuid].append(tok)
            self.llm_end_dict[uuid] = True
            return

        st = {"consumed": 0}
        silent = SilentTokenFilter(self.silent_tokens)

        def progress(out_ids, out_count, live):
            n = int(out_count[0].item())
            if n > st["consumed"]:
                for tok in out_ids[0, st["consumed"]:n].tolist():
                    if silent.keep(tok):
                        self.tts_speech_token_dict[uuid].append(tok)
                st["consumed"] = n
        # the LM job decodes on its own stream (cli/model.py:103: `with self.llm_context`, a side stream) while token2wav runs on
        # the model's stream
        with self._lm_stream() as lm_stream:
            self.lm_generate([text], [prompt_text], [llm_prompt_speech_token], steps_per_sync=8, on_progress=progress, stream=lm_stream)
        self.llm_end_dict[uuid] = True

    def vc_job(self, source_speech_token, uuid):
        self.tts_speech_token_dict[uuid] = source_speech_token.flatten().tolist()
        self.llm_end_dict[uuid] = True

    def _grow_hop(self, hop):
        """the hop after a streaming chunk (cli/model.py:362)"""
        return min(self.token_max_hop_len, hop * self.stream_scale_factor)

    def tts(self, text=torch.zeros(1, 0, dtype=torch.int32), flow_embedding=torch.zeros(0, 192), llm_embedding=torch.zeros(0, 192),
            prompt_text=torch.zeros(1, 0, dtype=torch.int32), llm_prompt_speech_token=torch.zeros(1, 0, dtype=torch.int32),
            flow_prompt_speech_token=torch.zeros(1, 0, dtype=torch.int32), prompt_speech_feat=torch.zeros(1, 0, 80),
            source_speech_token=torch.zeros(1, 0, dtype=torch.int32), stream=False, speed=1.0, **kwargs):
        """cli/model.py:328-394: same signature, same yielded dicts ({'tts_speech': float32 CPU [1,N]})."""
        this_uuid = str(uuid.uuid1())
        with self.lock:
            self.tts_speech_token_dict[this_uuid], self.llm_end_dict[this_uuid] = [], False
            self.hift_cache_dict[this_uuid] = None
        if source_speech_token.shape[1] == 0:
            p = threading.Thread(target=self.llm_job, args=(text, prompt_text, llm_prompt_speech_token, llm_embedding, this_uuid))
        else:
            p = threading.Thread(target=self.vc_job, args=(source_speech_token, this_uuid))
        p.start()
        if stream is True:
            # the hop lives on the instance, shared by concurrent requests, like the reference's self.token_hop_len
            token_offset = 0
            prompt_token_pad = _first_hop_pad(flow_prompt_speech_token.shape[1], self.token_hop_len)
            while True:
                time.sleep(0.005)
                this_hop = _this_hop(self.token_hop_len, prompt_token_pad, token_offset)
                toks = self.tts_speech_token_dict[this_uuid]
                if _hop_ready(len(toks), token_offset, this_hop):
                    this_tok = torch.tensor(toks[:token_offset + this_hop + PRE_LOOKAHEAD]).unsqueeze(0)
                    speech = self.token2wav(this_tok, flow_prompt_speech_token, prompt_speech_feat, flow_embedding, token_offset,
                                            this_uuid, stream=True, finalize=False)
                    token_offset += this_hop
                    self.token_hop_len = self._grow_hop(self.token_hop_len)
                    yield {"tts_speech": self._to_host(speech)}
                if self.llm_end_dict[this_uuid] is True and not _hop_ready(len(self.tts_speech_token_dict[this_uuid]), token_offset, this_hop):
                    break
            p.join()
            this_tok = torch.tensor(self.tts_speech_token_dict[this_uuid]).unsqueeze(0)
            speech = self.token2wav(this_tok, flow_prompt_speech_token, prompt_speech_feat, flow_embedding, token_offset, this_uuid,
                                    finalize=True)
            yield {"tts_speech": self._to_host(speech)}
        else:
            p.join()
            this_tok = torch.tensor(self.tts_speech_token_dict[this_uuid]).unsqueeze(0)
            speech = self.token2wav(this_tok, flow_prompt_speech_token, prompt_speech_feat, flow_embedding, 0, this_uuid, finalize=True,
                                    speed=speed)
            yield {"tts_speech": self._to_host(speech)}
        with self.lock:
            self.tts_speech_token_dict.pop(this_uuid)
            self.llm_end_dict.pop(this_uuid)
            self.hift_cache_dict.pop(this_uuid)
        self._release_flow_stream(this_uuid)
        self.stream.synchronize()

    # ---------------------------------------------------------------- batched streaming
    def _take_slot(self):
        """a free slot of the model's multi-slot flow session (created on first use), or None: no session configured, no memory
        for it, or every slot taken"""
        if not self.incremental_flow or self.stream_batch_slots <= 0:
            return None
        with torch.cuda.stream(self.stream), self.ctx.lock, self._pool_lock:     # the lock order of _flow_stream_chunk
            if self.stream_slots is None:
                self._create_slot_pool()
            return self._free_slots.pop(0) if self._free_slots else None

    def _create_slot_pool(self):
        """Once per model: the largest slot count of stream_batch_slots, /2, /4, ... whose session allocates and leaves
        stream_pool_headroom bytes free.  A model that fits none records 0 slots and is not retried."""
        import warnings
        n = self.stream_batch_slots
        while n >= 1:
            try:
                pool = self.ctx.flow_stream(self.stream_cache_frames, self.n_timesteps, dit=self.flow_stream_dit, slots=n)
            except cvk.CvkError:
                pool = None
            if pool is not None and self.device.type == "cuda" and torch.cuda.mem_get_info(self.device)[0] < self.stream_pool_headroom:
                self.ctx.flow_stream_destroy(pool)
                pool = None
            if pool is not None:
                break
            n //= 2
        self._slot_pool, self.stream_slots = pool, n if pool is not None else 0
        self._free_slots = list(range(self.stream_slots))
        if self.stream_slots < self.stream_batch_slots:
            warnings.warn(f"tts_stream_batch: {self.stream_slots} of {self.stream_batch_slots} streaming-flow slots of {self.stream_cache_frames} "
                          "frames fit in device memory; requests beyond them recompute their prefix", RuntimeWarning, stacklevel=4)

    def _give_slot(self, slot):
        with self._pool_lock:
            self._free_slots.append(slot)
            self._free_slots.sort()

    def tts_stream_batch(self, inputs, uniforms=None, noise_fns=None):
        """Streaming synthesis of several requests at once: a generator of (i, {'tts_speech': float32 CPU [1, n]}).

        `inputs` are tts() kwargs dicts with tensor `text`, as for tts_batch.  Each request gets exactly the chunks tts(stream=True)
        yields for it alone (cli/model.py:339-374: first hop token_hop_len + the prompt's padding to the hop grid, then x
        stream_scale_factor up to token_max_hop_len, 3 look-ahead tokens, a final non-streaming call); its chunks come out in order,
        requests interleave as their chunks become ready.  One LM generation decodes every row on a side stream (uniforms[:, i]
        for request i, as in tts_batch); every poll round then makes at most one call per stage for all requests that are ready:
        one cvk_flow_stream_chunk_batch for requests holding a slot of the model's multi-slot session, one prefix-recompute
        flow_inference for the others, one final flow_inference for requests that are finishing, and one vocoder call over all of
        them.  Request i's k-th vocoder call draws noise_fns[i](n) when given, so its audio does not depend on which other
        requests shared its rounds.  The instance's token_hop_len is not modified.  Closing the generator early (or an
        exception in it) gives the requests' slots back and ends the LM generation within one block of 8 decode steps.

        A voice-conversion request (non-empty source_speech_token, no text needed) has all its tokens at the first round, as with
        vc_job: the LM runs over the other rows only (still uniforms[:, i] for request i), not at all when every row is one, and the
        request finishes as soon as its own tokens are used up.  Refused when called, with ValueError: a speed other than 1 (the
        reference's streaming path asserts it away, cli/model.py:321) and a text generator (tts_bistream_batch serves those)."""
        vc = self._check_stream_requests(inputs)
        for i, r in enumerate(inputs):
            if i not in vc and not torch.is_tensor(r.get("text")):
                raise ValueError("tts_stream_batch takes token tensors as text; requests with a text generator go to tts_bistream_batch")
        lm_rows = [i for i in range(len(inputs)) if i not in vc]
        if vc:
            if uniforms is None:
                uniforms = self.uniforms_override
            if uniforms is not None:
                uniforms = uniforms[:, lm_rows]

        def lm_run(emit, lm_state):
            B = len(lm_rows)
            consumed = [0] * B

            def progress(out_ids, out_count, live):
                if lm_state["stop"]:
                    raise _LmStopped()                   # the generator was closed: end the decode at the next block
                cnt = out_count.cpu().tolist()
                ids = out_ids.cpu()
                for b in range(B):
                    if cnt[b] > consumed[b]:
                        for tok in ids[b, consumed[b]:cnt[b]].tolist():
                            emit(lm_rows[b], tok)
                        consumed[b] = cnt[b]
            with self._lm_stream() as lm_stream:
                self.lm_generate([inputs[i]["text"] for i in lm_rows], [request_field(inputs[i], "prompt_text") for i in lm_rows],
                                 [request_field(inputs[i], "llm_prompt_speech_token") for i in lm_rows], uniforms=uniforms, steps_per_sync=8,
                                 on_progress=progress, stream=lm_stream)
        return self._stream_batch(inputs, lm_run if lm_rows else None, noise_fns, vc)

    def tts_bistream_batch(self, inputs, uniforms=None, noise_fns=None):
        """tts_stream_batch for text-streaming requests: `inputs` are tts() kwargs dicts whose `text` is a generator of int32 [1,k]
        chunks.  Same contract and rounds as tts_stream_batch - (i, {'tts_speech': ...}) with each request's tts(stream=True) chunk
        schedule, the multi-slot flow session, vocoder caches and cross-fade - with the LM job replaced by one
        lm_generate_bistream_batch over all requests (uniforms[k, i] for request i's k-th draw).  Closing the generator early (or an
        exception in it) gives the requests' slots back and ends the LM generation at its next decoded id.  Refused when called,
        with ValueError: voice-conversion requests (they have no text to stream) and a speed other than 1."""
        if self._check_stream_requests(inputs):
            raise ValueError("tts_bistream_batch serves text-streaming requests; voice-conversion requests go to tts_stream_batch")

        def lm_run(emit, lm_state):
            with self._lm_stream() as lm_stream:
                gen = self.lm_generate_bistream_batch([iter(r["text"]) for r in inputs], [request_field(r, "prompt_text") for r in inputs],
                                                      [request_field(r, "llm_prompt_speech_token") for r in inputs], uniforms=uniforms,
                                                      stream=lm_stream)
                try:
                    for b, tok in gen:
                        if lm_state["stop"]:
                            break
                        emit(b, tok)
                finally:
                    gen.close()
        return self._stream_batch(inputs, lm_run, noise_fns)

    @staticmethod
    def _check_stream_requests(inputs):
        """the voice-conversion rows of a streaming batch; ValueError for a speed other than 1"""
        for r in inputs:
            if request_speed(r) != 1.0:
                raise ValueError("speed change only supports non-streaming inference (cli/model.py:321); use tts_batch")
        return [i for i, r in enumerate(inputs) if is_vc_request(r)]

    def _stream_batch(self, inputs, lm_run, noise_fns, vc=()):
        """the poll loop of tts_stream_batch / tts_bistream_batch.  lm_run(emit, lm_state) runs the LM job on a side thread and calls
        emit(i, id) for every id request i decodes; it ends early once lm_state["stop"] is set.  Rows in `vc` are voice-conversion
        requests: their source tokens are all there from the start and they end on their own; lm_run is None when every row is one."""
        B = len(inputs)
        req = [dict(ptok=request_field(r, "flow_prompt_speech_token"), pfeat=request_field(r, "prompt_speech_feat"),
                    emb=request_field(r, "flow_embedding")) for r in inputs]
        toks = [[] for _ in range(B)]
        own_end = [False] * B
        for i in vc:
            toks[i], own_end[i] = request_field(inputs[i], "source_speech_token").flatten().tolist(), True
        lm_state = {"end": lm_run is None, "err": None, "stop": False}
        silent = [SilentTokenFilter(self.silent_tokens) for _ in range(B)]

        def emit(b, tok):
            if silent[b].keep(tok):
                toks[b].append(tok)

        def llm_job():
            try:
                lm_run(emit, lm_state)
            except _LmStopped:
                pass
            except BaseException as e:                   # noqa: BLE001  (re-raised by the generator)
                lm_state["err"] = e
            finally:
                lm_state["end"] = True

        hop0 = self.token_hop_len
        st = []
        for r in req:
            P = int(r["ptok"].shape[1])
            st.append(dict(P=P, pad=_first_hop_pad(P, hop0), hop=hop0, offset=0, slot=None, eligible=True, cache=None, done=False))
        p = None
        if lm_run is not None:
            p = threading.Thread(target=llm_job, name="cvk-stream-batch-lm", daemon=True)
            p.start()
        try:
            while not all(s["done"] for s in st):
                end = lm_state["end"]                    # read first: once the LM has ended, the token lists are complete
                if lm_state["err"] is not None:
                    raise lm_state["err"]
                ready, finishing = [], []
                for i, s in enumerate(st):
                    if s["done"]:
                        continue
                    this_hop = _this_hop(s["hop"], s["pad"], s["offset"])
                    if _hop_ready(len(toks[i]), s["offset"], this_hop):
                        ready.append((i, this_hop))
                    elif end or own_end[i]:
                        finishing.append(i)
                if not ready and not finishing:
                    time.sleep(0.005)
                    continue
                for i, out in self._stream_round(req, st, toks, ready, finishing, noise_fns):
                    yield i, out
            if p is not None:
                p.join()
        finally:
            lm_state["stop"] = True                      # closed or failed early: the LM stops within one block of 8 steps
            for s in st:
                if s["slot"] is not None:
                    self._give_slot(s["slot"])
                    s["slot"] = None
            if self.stream is not None:
                self.stream.synchronize()

    def _stream_vocode(self, voc, mels, st, finishing, noise_fns):
        """the vocoder step of a poll round: requests `voc` (in order) with their new mel frames mels[i], in one vocoder call with
        token2wav's bookkeeping per request (_vocode_cached); requests in `finishing` make their final call.  Returns
        {i: float32 CPU [n]}, copied to the host in one D2H for the round."""
        wavs, caches = self._vocode_cached([st[i]["cache"] for i in voc], [mels[i] for i in voc], [i in finishing for i in voc],
                                           [noise_fns[i] if noise_fns is not None else None for i in voc])
        for i, c in zip(voc, caches):
            st[i]["cache"] = c
        return self._round_to_host(voc, wavs)

    def _round_to_host(self, voc, wavs):
        """{i: host copy of wavs[k]} for the requests i = voc[k], in one D2H"""
        with torch.cuda.stream(self.stream):
            flat = torch.cat(wavs).cpu()
        if self.stream is not None:
            self.stream.synchronize()
        return dict(zip(voc, flat.split([int(w.shape[0]) for w in wavs])))

    def _stream_round(self, req, st, toks, ready, finishing, noise_fns):
        """one poll round of tts_stream_batch: flow for every ready / finishing request (at most three calls), then one vocoder call
        with the model's token2wav bookkeeping per request (_stream_vocode)"""
        d = self.device
        slot_grp, prefix_grp = [], []
        for i, this_hop in ready:
            s = st[i]
            n_tok = s["offset"] + this_hop + PRE_LOOKAHEAD
            this_tok = torch.tensor(toks[i][:n_tok], dtype=torch.int32).unsqueeze(0)
            if s["eligible"]:
                ok = self._session_chunk_ok(s["P"], int(req[i]["pfeat"].shape[1]), n_tok, s["offset"], s["slot"] is not None)
                if ok and s["slot"] is None:
                    s["slot"] = self._take_slot()
                    s["begin"] = s["slot"] is not None
                    ok = s["slot"] is not None
                if not ok:
                    s["eligible"] = False
                    if s["slot"] is not None:
                        self._give_slot(s["slot"])
                        s["slot"] = None
            (slot_grp if s["eligible"] else prefix_grp).append((i, this_hop, this_tok))
        mels = {}
        if slot_grp:
            with torch.cuda.stream(self.stream), self.ctx.lock:
                for i, _, _ in slot_grp:
                    if st[i].pop("begin", False):
                        self.ctx.flow_stream_begin_slot(self._slot_pool, st[i]["slot"], req[i]["pfeat"][0].to(d, non_blocking=True),
                                                        req[i]["emb"].reshape(-1).to(d, non_blocking=True))
                token_list = [torch.cat([req[i]["ptok"].reshape(-1), t.reshape(-1)]).to(torch.int32) for i, _, t in slot_grp]
                mel, lens = self.ctx.flow_stream_chunk_batch(self._slot_pool, [st[i]["slot"] for i, _, _ in slot_grp], token_list)
            o = 0
            for (i, _, _), n in zip(slot_grp, lens):
                mels[i] = mel[o:o + n]
                o += n
        for grp, final in ((prefix_grp, False), ([(i, None, torch.tensor(toks[i], dtype=torch.int32).unsqueeze(0)) for i in finishing], True)):
            grp = [g for g in grp if g[2].shape[1] > 0]
            if not grp:
                continue
            mel, lens = self.flow_batch([t for _, _, t in grp], [req[i]["ptok"] for i, _, _ in grp], [req[i]["pfeat"] for i, _, _ in grp],
                                        [req[i]["emb"] for i, _, _ in grp], streaming=not final, finalize=final)
            o = 0
            for (i, _, _), n in zip(grp, lens):
                mels[i] = mel[o + st[i]["offset"] * TOKEN_MEL_RATIO:o + n]
                o += n
        # vocoder: every request of the round in one call
        order = [i for i, _ in ready] + finishing
        voc = [i for i in order if i in mels]
        outs = self._stream_vocode(voc, mels, st, finishing, noise_fns) if voc else {}
        for i, this_hop in ready:
            st[i]["offset"] += this_hop
            st[i]["hop"] = self._grow_hop(st[i]["hop"])
        results = []
        for i in order:
            results.append((i, {"tts_speech": outs[i].unsqueeze(0) if i in outs else torch.zeros(1, 0)}))
        for i in finishing:
            st[i]["done"] = True
            if st[i]["slot"] is not None:
                self._give_slot(st[i]["slot"])
                st[i]["slot"] = None
        return results
