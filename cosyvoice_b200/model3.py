"""Host-side mirror of the reference's CosyVoice3Model (cosyvoice/cli/model.py:397-450) over libcvk.

CosyVoice3Model inherits CosyVoice2Model.tts (thread-per-request LM job, chunk schedule hop 25 -> 50 -> 100 with 3 look-ahead
tokens) and replaces token2wav: the flow is the DiT one (stage "flow3", through the inherited flow half of token2wav with
``flow_batch`` below and DiT flow sessions), the vocoder is the causal one (stage "hift3"), and instead of the CosyVoice2 mel /
source / speech caches with a cross-fade it keeps ALL mel frames produced so far, re-runs the causal vocoder over them and emits
the samples beyond ``speech_offset``.  ``_append_mel`` and ``_new_speech`` keep that bookkeeping on a request's cache dict.

Offline requests also batch: the inherited ``tts_batch`` / ``tts_batch_device`` run the LM, the DiT flow and the causal vocoder
(``hift_batch`` below) once for the whole batch, and ``TtsBatcher`` serves CosyVoice3 offline requests through them.  Each request
gets what ``tts()`` gives it alone: the causal vocoder reads its stored noise from each utterance's start and its float64 f0
predictor sums in an order that does not depend on the batch.

Streaming requests batch too: ``tts_stream_batch`` / ``tts_bistream_batch`` run the inherited poll loop (multi-slot DiT flow
sessions, ``flow_batch`` for prefix recomputes and final calls) with the vocoder step replaced by ``_stream_vocode`` below, which
keeps token2wav's bookkeeping per request and vocodes every request of a round - streaming chunks and final calls together - in
one ``hift3_inference_rows`` call with a finalize flag per utterance.  ``TtsBatcher`` serves CosyVoice3 streaming requests
through them.

The class is checked on the CPU against the reference's own CosyVoice3Model.tts with the device primitives faked by the oracle
(tests/test_host_logic_cpu.py, tests/test_tts3_batch_cpu.py, tests/test_stream3_batch_cpu.py) and on the GPU against the
reference's waveform (tests/test_zz_model3_gpu.py, tests/test_zz_tts3_batch_gpu.py, tests/test_zz_stream3_batch_gpu.py)."""
import torch

from .model import B200CosyVoice2Model, SAMPLES_PER_FRAME, _count


class B200CosyVoice3Model(B200CosyVoice2Model):
    # CosyVoice3LM (llm.py:681-684): sos 6561 / eos 6562 / task_id 6563 / fill 6564; <|endofprompt|> = 151646 (llm.py:585)
    bistream_fill_token = 6564
    bistream_eos_token = 6562
    bistream_eop_token = 151646
    flow_stream_dit = True            # streaming chunks through cvk_flow3_stream_create sessions (DiT K/V + position-convolution tails)

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        # FSQ silent and breath tokens (cli/model.py:423)
        self.silent_tokens = [1, 2, 28, 29, 55, 248, 494, 2241, 2242, 2322, 2323]

    def tts_stream_batch(self, inputs, uniforms=None, noise_fns=None):
        """Streaming synthesis of several CosyVoice3 requests at once: a generator of (i, {'tts_speech': float32 CPU [1, n]}).

        `inputs` are tts() kwargs dicts with tensor `text`.  Each request gets the chunks tts(stream=True) gives it alone: the
        same chunk schedule and the same chunk lengths.  One LM generation decodes every row (uniforms[:, i] for request i); every
        poll round then makes at most one multi-slot DiT chunk call, one prefix-recompute and one final flow call, and one
        causal-vocoder call over every request of the round, streaming and finishing ones together (_stream_vocode).  The
        instance's token_hop_len is not modified.  Closing the generator early returns every slot to the pool.  Refused when
        called, before any work: `noise_fns` (ValueError: the causal vocoder draws its noise from its stored sine_waves, from
        each utterance's start) and a model without a libcvk context (NotImplementedError, see _check_stream_batch)."""
        self._check_stream_batch(noise_fns)
        return super().tts_stream_batch(inputs, uniforms)

    def tts_bistream_batch(self, inputs, uniforms=None, noise_fns=None):
        """tts_stream_batch for text-streaming CosyVoice3 requests: `inputs` are tts() kwargs dicts whose `text` is a generator of
        int32 [1,k] chunks, decoded by one lm_generate_bistream_batch (uniforms[k, i] for request i's k-th draw).  Each request
        gets the chunks tts(text=<generator>, stream=True) gives it alone: the same chunk schedule and the same chunk lengths.
        The instance's token_hop_len is not modified.  Closing the generator early returns every slot to the pool.  Refuses
        what tts_stream_batch refuses, when called."""
        self._check_stream_batch(noise_fns)
        return super().tts_bistream_batch(inputs, uniforms)

    def _check_stream_batch(self, noise_fns):
        """The batched streaming path vocodes each round with one cvk_hift3_inference_rows call (a finalize flag per utterance);
        a model whose context does not provide that call - no context loaded, or one without the entry point - cannot serve it,
        and says so before any LM or flow work is started rather than failing in the middle of a stream."""
        if noise_fns is not None:
            raise ValueError("the causal vocoder draws its noise from its stored sine_waves: noise_fns= is not accepted")
        if not callable(getattr(getattr(self, "ctx", None), "hift3_inference_rows", None)):
            raise NotImplementedError("batched CosyVoice3 streaming needs a libcvk context with cvk_hift3_inference_rows (one causal-vocoder "
                                      "call with a finalize flag per utterance); this model has none")

    # ---------------------------------------------------------------- weights
    def load_state_dicts(self, llm_sd, flow_sd, hift_sd, rand_ini=None, sine_noise=None):
        """llm_sd: CosyVoice3LM, flow_sd: CausalMaskedDiffWithDiT, hift_sd: CausalHiFTGenerator state_dicts.  rand_ini [1,9] /
        sine_noise [1,n,9]: the vocoder's constructor-time random tensors (SineGen2.rand_ini / .sine_waves, generator.py:223-226),
        which are module attributes and not part of the state_dict; drawn like the reference draws them when omitted."""
        from .model import cfm_rand_noise
        nl = _count(llm_sd.keys(), "llm.model.model.layers.")
        depth = _count(list(flow_sd.keys()), "decoder.estimator.transformer_blocks.")
        self.ctx.load_state_dict("llm", llm_sd, [nl])
        self.ctx.load_state_dict("flow3", flow_sd, [depth])
        self.ctx.load_state_dict("hift3", hift_sd)
        self.ctx.set_cfm_noise(cfm_rand_noise())
        if rand_ini is None:
            rand_ini = torch.rand(1, 9)
            rand_ini[:, 0] = 0
        if sine_noise is None:
            sine_noise = torch.rand(1, 300 * 24000, 9)
        self.ctx.hift3_set_noise(rand_ini, sine_noise.reshape(-1, 9))

    # ---------------------------------------------------------------- flow + vocoder
    def flow_batch(self, tokens, prompt_tokens, prompt_feats, embeddings, streaming=False, finalize=True):
        d = self.device
        tl = [int(t.shape[1] + p.shape[1]) for t, p in zip(tokens, prompt_tokens)]
        pl = [int(f.shape[1]) for f in prompt_feats]
        with torch.cuda.stream(self.stream), self.ctx.lock:
            toks = torch.cat([torch.cat([p.reshape(-1).to(d), t.reshape(-1).to(d)]) for t, p in zip(tokens, prompt_tokens)]).to(torch.int32)
            pf = torch.cat([f[0].to(d) for f in prompt_feats], 0) if sum(pl) else None
            emb = torch.cat([e.reshape(1, -1).to(d) for e in embeddings], 0)
            return self.ctx.flow3_inference(toks, tl, pf, pl, emb, n_timesteps=self.n_timesteps, streaming=streaming, finalize=finalize)

    def hift_batch(self, mel_tm, lens, cache_source=None, cache_lens=None, noise=None):
        """The causal vocoder over a ragged batch (finalize=True): mel [sum T, 80] -> (wav [sum 480 T], source [sum 480 T]), the pair
        the inherited tts_batch_device takes.  Its source noise is the module's stored sine_waves indexed from each utterance's start
        (generator.py:303-307), so a noise tensor or a source cache from the caller has no meaning here."""
        if noise is not None or cache_source is not None:
            raise ValueError("the causal vocoder draws its noise from its stored sine_waves: noise= and cache_source= are not accepted")
        with torch.cuda.stream(self.stream), self.ctx.lock:
            wav, _, src = self.ctx.hift3_inference(mel_tm, lens, finalize=True)
        return wav, src

    def _stream_vocode(self, voc, mels, st, finishing, noise_fns):
        """the vocoder step of a tts_stream_batch round with token2wav's bookkeeping (cli/model.py:425-450) per request: append the
        new mel to the request's history, re-run the causal vocoder over the whole history - one hift3_inference_rows call for
        the round, finalize for the requests in `finishing` - and emit the samples past its speech_offset.  Returns
        {i: float32 CPU [n]}, copied to the host in one D2H for the round.  noise_fns is always None here (refused by
        _check_stream_batch)."""
        with torch.cuda.stream(self.stream):
            for i in voc:
                st[i]["cache"] = self._append_mel(st[i]["cache"], mels[i])
            lens, fin = [int(st[i]["cache"]["mel"].shape[0]) for i in voc], [i in finishing for i in voc]
            with self.ctx.lock:
                wav, _, _ = self.ctx.hift3_inference_rows(torch.cat([st[i]["cache"]["mel"] for i in voc], 0), lens, fin)
            outs, o = [], 0
            for i, n, f in zip(voc, lens, fin):
                n_out = SAMPLES_PER_FRAME * (n if f else n - 8)
                outs.append(self._new_speech(st[i]["cache"], wav[o:o + n_out]))
                o += n_out
        return self._round_to_host(voc, outs)

    @staticmethod
    def _append_mel(cache, mel):
        """a request's cache dict (None before its first chunk) with `mel` appended to its mel history"""
        if cache is None:
            return {"mel": mel, "speech_offset": 0}
        cache["mel"] = torch.cat([cache["mel"], mel], 0)
        return cache

    @staticmethod
    def _new_speech(cache, wav):
        """the samples of `wav` (the vocoder over the request's whole mel history) past its speech_offset, which moves past them"""
        wav = wav[cache["speech_offset"]:]
        cache["speech_offset"] += wav.shape[0]
        return wav

    def token2wav(self, token, prompt_token, prompt_feat, embedding, token_offset, uuid, stream=False, finalize=False, speed=1.0):
        """cli/model.py:425-450"""
        mel = self._token2wav_mel(token, prompt_token, prompt_feat, embedding, token_offset, uuid, stream, finalize)
        with torch.cuda.stream(self.stream):
            cache = self.hift_cache_dict[uuid] = self._append_mel(self.hift_cache_dict[uuid], mel)
            tts_mel = cache["mel"]
            if speed != 1.0:
                assert token_offset == 0 and finalize is True, "speed change only support non-stream inference mode"
                tts_mel, _ = self.mel_stretch(tts_mel, [tts_mel.shape[0]], [speed])
            with self.ctx.lock:
                wav, _, _ = self.ctx.hift3_inference(tts_mel.contiguous(), [tts_mel.shape[0]], finalize=finalize)
        return self._new_speech(cache, wav).unsqueeze(0)
