"""GPU: batched streaming synthesis.

Multi-slot streaming-flow sessions (cvk_flow_stream_create_slots / _begin_slot / _chunk_batch) against the reference's schedule,
which re-runs flow.inference(streaming=True, finalize=False) on every request's growing prefix (cli/model.py:346-363), and the
host scheduler above them (B200CosyVoice2Model.tts_stream_batch, TtsBatcher.submit_stream) against single-request tts()."""
import numpy as np
import pytest
import torch

from gpu_util import maxdiff
from oracle import cases, dit, flow, hift, lm, weights
from oracle.make_golden import stream_noise

pytestmark = pytest.mark.gpu

UNET = {"small": dict(enc_blocks=2, enc_up_blocks=1, num_mid_blocks=2, n_blocks=2),
        "full": dict(enc_blocks=6, enc_up_blocks=4, num_mid_blocks=12, n_blocks=4)}
_c = {}


@pytest.fixture(scope="module", autouse=True)
def _release_contexts():
    """this module's contexts, models and slot caches go before the full-size modules build theirs"""
    yield
    for k in list(_c):
        obj = _c.pop(k)
        if hasattr(obj, "ctx"):                        # a model: its sessions and context, even if a failed test's traceback holds it
            for fs in obj._idle_flow_streams + ([obj._slot_pool] if obj._slot_pool else []):
                obj.ctx.flow_stream_destroy(fs)
            obj._idle_flow_streams, obj._slot_pool = [], None
            obj = obj.ctx
        if hasattr(obj, "close"):
            obj.close()
    torch.cuda.empty_cache()


def flow_ctx(precision, tag):
    """own context per precision (the shared one of gpu_util holds other modules' stages); tag: U-Net "small" / "full" or "dit2" """
    from cosyvoice_b200 import cvk
    if precision not in _c:
        _c[precision] = cvk.Context(0, precision, workspace_gb=6.0)
    c = _c[precision]
    if _c.get((precision, "tag")) != tag:
        if tag == "dit2":
            c.load_state_dict("flow3", weights.synth_state_dict(dit.flow_param_shapes(2), 1986, dit.SYNTH_GAINS), cfg=[2])
        else:
            cfg = flow.FlowCfg(**UNET[tag])
            c.load_state_dict("flow", weights.synth_state_dict(flow.param_shapes(cfg), 1986, flow.SYNTH_GAINS),
                              cfg=[cfg.enc_blocks, cfg.enc_up_blocks, cfg.num_mid_blocks, cfg.n_blocks])
        c.set_cfm_noise(flow.cfm_noise(15000)[0].t().contiguous())
        _c[(precision, "tag")] = tag
    return c


class Utt:
    """one streaming utterance: prompt of P tokens (prompt mel 2 frames per token), the reference's hop schedule (first hop padded
    to the 25-token grid, then x2 up to 100)"""

    def __init__(self, P, seed):
        g = torch.Generator().manual_seed(seed)
        self.P = P
        self.toks = torch.randint(0, 6561, (P + 400,), generator=g, dtype=torch.int32)
        self.pfeat = torch.rand(2 * P, 80, generator=g) * 13.5 - 11.5
        self.emb = torch.randn(1, 192, generator=g)
        self.restart()

    def restart(self):
        self.offset, self.hop = 0, 25

    def next_tokens(self):
        pad = int(np.ceil(self.P / 25) * 25 - self.P)
        this_hop = self.hop + pad if self.offset == 0 else self.hop
        return self.toks[:self.P + self.offset + this_hop + 3], this_hop

    def advance(self, this_hop):
        self.offset += this_hop
        self.hop = min(100, 2 * self.hop)

    def reference(self, c, dit_kind, toks):
        """frames of the prefix-recompute call that this chunk must reproduce"""
        fn = c.flow3_inference if dit_kind else c.flow_inference
        n = int(toks.numel())
        ref, lens = fn(toks, [n], self.pfeat, [2 * self.P], self.emb, streaming=True, finalize=False)
        done = 2 * (self.P + self.offset) if self.offset else 0
        return ref[max(done - 2 * self.P, 0):]


def run_round(c, fs, dit_kind, utts, group, slot_of, bound):
    """one chunk_batch call for the utterances in `group`; every slot's frames against its own prefix recompute"""
    steps = [utts[i].next_tokens() for i in group]
    mel, lens = c.flow_stream_chunk_batch(fs, [slot_of[i] for i in group], [t for t, _ in steps])
    assert len(lens) == len(group) and mel.shape[0] == sum(lens)
    o = 0
    for i, (toks, hop), n in zip(group, steps, lens):
        want = utts[i].reference(c, dit_kind, toks)
        assert n == want.shape[0], (i, n, want.shape)
        got = mel[o:o + n]
        assert torch.isfinite(got).all()
        d = maxdiff(got, want)
        assert d < bound, (i, hop, d)
        o += n
        utts[i].advance(hop)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("tag", ["small", "full", "dit2"])
def test_batched_chunks_equal_prefix_recompute(precision, tag):
    """Three utterances (prompts of 30, 9 and 50 tokens: first hops 45, 41 and 25) in slots 2, 0 and 3 of a 4-slot session, chunk
    calls in changing groupings.  Every row's arithmetic is the same sequence of operations as in the prefix recompute, so the
    bound is round-off (that of test_incremental_stream_equals_prefix_recompute)."""
    c = flow_ctx(precision, tag)
    dit_kind = tag == "dit2"
    bound = 1e-5 if precision == "fp32" else 1e-3
    utts = [Utt(30, 1), Utt(9, 2), Utt(50, 3)]
    slot_of = {0: 2, 1: 0, 2: 3}
    fs = c.flow_stream(max_frames=512, n_timesteps=10, dit=dit_kind, slots=4)
    try:
        assert c.flow_stream_bytes(fs) > 0
        for i, u in enumerate(utts):
            c.flow_stream_begin_slot(fs, slot_of[i], u.pfeat, u.emb)
        for group in ([0, 1, 2], [2, 0], [1], [1, 2], [0]):
            run_round(c, fs, dit_kind, utts, group, slot_of, bound)
        assert [u.offset for u in utts] == [45 + 50 + 100, 41 + 50 + 100, 25 + 50 + 100]
    finally:
        c.flow_stream_destroy(fs)


def test_slot_sessions_scale_with_slot_count():
    c = flow_ctx("fp32", "small")
    one = c.flow_stream(max_frames=512, n_timesteps=10)
    four = c.flow_stream(max_frames=512, n_timesteps=10, slots=4)
    try:
        b1, b4 = c.flow_stream_bytes(one), c.flow_stream_bytes(four)
        assert 3.5 * b1 < b4 < 4.0 * b1           # 64 spare key rows per block are shared by all slots
    finally:
        c.flow_stream_destroy(one)
        c.flow_stream_destroy(four)


@pytest.mark.parametrize("tag", ["small", "dit2"])
def test_refused_calls_leave_every_slot_intact(tag):
    from cosyvoice_b200.cvk import CvkError
    c = flow_ctx("fp32", tag)
    dit_kind = tag == "dit2"
    utts = [Utt(30, 11), Utt(9, 12), Utt(50, 13)]
    slot_of = {0: 0, 1: 1, 2: 2}
    fs = c.flow_stream(max_frames=512, n_timesteps=10, dit=dit_kind, slots=4)
    try:
        for i, u in enumerate(utts):
            c.flow_stream_begin_slot(fs, slot_of[i], u.pfeat, u.emb)
        run_round(c, fs, dit_kind, utts, [0, 1, 2], slot_of, 1e-5)
        t0, _ = utts[0].next_tokens()
        t1, _ = utts[1].next_tokens()
        with pytest.raises(CvkError):                  # one slot twice in one call
            c.flow_stream_chunk_batch(fs, [0, 0], [t0, t0])
        with pytest.raises(CvkError):                  # slot 1 off the 50-frame grid
            c.flow_stream_chunk_batch(fs, [0, 1], [t0, utts[1].toks[:t1.numel() + 10]])
        with pytest.raises(CvkError):                  # slot 3 was never begun
            c.flow_stream_chunk_batch(fs, [0, 3], [t0, t0])
        with pytest.raises(CvkError):                  # slot index out of range
            c.flow_stream_chunk_batch(fs, [0, 4], [t0, t0])
        with pytest.raises(CvkError):
            c.flow_stream_begin_slot(fs, 4, utts[0].pfeat, utts[0].emb)
        # nothing moved: the next valid call on every slot still equals the prefix recompute
        run_round(c, fs, dit_kind, utts, [2, 1, 0], slot_of, 1e-5)
        # a new utterance in slot 1 in the middle of the others' streams does not perturb slot 0
        utts[1] = Utt(20, 14)
        c.flow_stream_begin_slot(fs, 1, utts[1].pfeat, utts[1].emb)
        run_round(c, fs, dit_kind, utts, [0, 1], slot_of, 1e-5)
        run_round(c, fs, dit_kind, utts, [1, 2], slot_of, 1e-5)
    finally:
        c.flow_stream_destroy(fs)


# ------------------------------------------------------------------------------------------------ host scheduler
def small_model():
    if "m" not in _c:
        from cosyvoice_b200.model import B200CosyVoice2Model
        kw = dict(enc_blocks=2, enc_up_blocks=1, num_mid_blocks=2, n_blocks=2)
        m = B200CosyVoice2Model(precision="fp32", device=0, workspace_gb=4.0)
        m.load_state_dicts(lm.synth_state_dict(2), weights.synth_state_dict(flow.param_shapes(flow.FlowCfg(**kw)), 1986, flow.SYNTH_GAINS),
                           weights.synth_state_dict(hift.param_shapes(), 1986, hift.SYNTH_GAINS))
        m.stream_batch_slots, m.stream_cache_frames = 4, 1024
        m.stream_pool_headroom = 1 << 30              # the test process holds the contexts of the earlier GPU modules too
        _c["m"] = m
    return _c["m"]


def batch_case():
    """request 0 = the golden request of tests/test_model_gpu.py; request 1 with a different text length, request 2 with a
    different prompt (24 tokens: first hop 26)"""
    text, ptext, ptok, U = cases.lm_case()
    _, _, pfeat, emb = cases.flow_case(P=9)
    req0 = dict(text=text, flow_embedding=emb, llm_embedding=emb, prompt_text=ptext, llm_prompt_speech_token=ptok,
                flow_prompt_speech_token=ptok, prompt_speech_feat=pfeat[:, :18])
    g = torch.Generator().manual_seed(321)
    req1 = dict(req0, text=torch.randint(0, 151643, (1, 5), generator=g, dtype=torch.int32))
    _, ptok2, pfeat2, emb2 = cases.flow_case(P=24)
    req2 = dict(req0, flow_prompt_speech_token=ptok2, prompt_speech_feat=pfeat2[:, :48], flow_embedding=emb2)
    Ub = torch.rand(U.shape[0], 3, 2, generator=g)
    Ub[:, 0] = U
    return [req0, req1, req2], Ub


def noise_fns(B, device):
    """per-request vocoder noise streams: request i's k-th vocoder call draws stream_noise(1000 i + k, n)"""
    def make(i):
        st = {"k": 0}

        def fn(n):
            z = stream_noise(1000 * i + st["k"], n).to(device)
            st["k"] += 1
            return z
        return fn
    return [make(i) for i in range(B)]


def single_stream(m, req, U_row, i):
    """request i alone through tts(stream=True), with its uniforms row and its noise stream"""
    m.uniforms_override, m.noise_fn, m.token_hop_len = U_row[:, None, :], noise_fns(i + 1, m.device)[i], 25
    try:
        return [o["tts_speech"] for o in m.tts(**req, stream=True)]
    finally:
        m.uniforms_override, m.noise_fn = None, None
        m.token_hop_len = 25


def collect(gen, B):
    chunks = [[] for _ in range(B)]
    for i, out in gen:
        chunks[i].append(out["tts_speech"])
    return chunks


def check_against_singles(chunks, singles, golden_stream):
    g = golden_stream
    assert [c.shape[1] for c in chunks[0]] == g["stream_lens"].tolist()
    wav = torch.cat(chunks[0], 1)
    ref = torch.from_numpy(g["stream_wav"])
    assert maxdiff(wav[:, :24000], ref[:, :24000]) < 5e-3
    assert ((wav - ref).norm() / ref.norm()).item() < 0.05
    for i in range(len(chunks)):
        assert [c.shape[1] for c in chunks[i]] == [c.shape[1] for c in singles[i]], i
        assert all(c.device.type == "cpu" and c.dtype == torch.float32 and c.shape[0] == 1 for c in chunks[i])
        d = maxdiff(torch.cat(chunks[i], 1), torch.cat(singles[i], 1))
        assert d <= 1e-4, (i, d)


_singles = {}


def singles(m, reqs, Ub):
    if "s" not in _singles:
        _singles["s"] = [single_stream(m, r, Ub[:, i, :], i) for i, r in enumerate(reqs)]
    return _singles["s"]


def test_tts_stream_batch_equals_single_requests(golden):
    m = small_model()
    reqs, Ub = batch_case()
    want = singles(m, reqs, Ub)
    assert m.token_hop_len == 25
    launches = m.ctx.launch_count()
    chunks = collect(m.tts_stream_batch(reqs, uniforms=Ub, noise_fns=noise_fns(3, m.device)), 3)
    assert m.token_hop_len == 25                     # per-request hop state; the instance attribute is left alone
    check_against_singles(chunks, want, golden("stream_tts"))
    assert m._free_slots is not None and len(m._free_slots) == m.stream_batch_slots      # every slot went back to the pool
    print(f"tts_stream_batch: {m.ctx.launch_count() - launches} launches for 3 requests, chunk lengths "
          f"{[[c.shape[1] for c in ch] for ch in chunks]}")


@pytest.mark.parametrize("mode", ["no_slots", "one_ineligible"])
def test_tts_stream_batch_fallback_paths(mode, golden):
    m = small_model()
    reqs, Ub = batch_case()
    want = singles(m, reqs, Ub)
    if mode == "no_slots":
        m.stream_batch_slots = 0
    else:
        reqs = list(reqs)
        reqs[1] = dict(reqs[1], prompt_speech_feat=reqs[1]["prompt_speech_feat"][:, :17])   # not 2 frames per prompt token
    try:
        chunks = collect(m.tts_stream_batch(reqs, uniforms=Ub, noise_fns=noise_fns(3, m.device)), 3)
    finally:
        m.stream_batch_slots = 4
    if mode == "one_ineligible":
        # request 1 recomputes its prefix with a 17-frame prompt mel: its own reference is tts() with that prompt
        want = list(want)
        want[1] = single_stream(m, reqs[1], Ub[:, 1, :], 1)
    check_against_singles(chunks, want, golden("stream_tts"))


def test_tts_stream_batch_refuses_text_generator():
    m = small_model()
    reqs, Ub = batch_case()
    with pytest.raises(ValueError):
        list(m.tts_stream_batch([dict(reqs[0], text=iter([reqs[0]["text"]]))]))


def test_batcher_streams_and_keeps_offline_requests_apart(golden):
    """two streaming requests and one offline request submitted together: the streaming pair is one tts_stream_batch batch (same
    chunks as calling it directly), the offline request a batch of its own"""
    from cosyvoice_b200.batcher import TtsBatcher, pcm16
    m = small_model()
    reqs, Ub = batch_case()

    def hook():
        st = {"k": 0}

        def fn(n):
            z = stream_noise(500 + st["k"], n).to(m.device)
            st["k"] += 1
            return z
        return fn
    m.uniforms_override = Ub[:, :2]
    try:
        m.noise_fn = hook()
        want = collect(m.tts_stream_batch(reqs[:2]), 2)
        m.noise_fn = hook()
        with TtsBatcher(m, max_batch=4, max_wait_ms=2000) as b:
            s1 = b.submit_stream(**reqs[0])
            s2 = b.submit_stream_pcm(**reqs[1])
            f3 = b.submit(**reqs[2])
            got1 = list(s1)
            got2 = list(s2)
            w3 = f3.result(timeout=300)
        assert b.batches == [2, 1]
    finally:
        m.uniforms_override, m.noise_fn = None, None
    assert len(got1) == len(want[0]) and all(torch.equal(a, w) for a, w in zip(got1, want[0]))
    assert got2 == [pcm16(w) for w in want[1]]
    assert w3.shape[0] == 1 and w3.shape[1] > 0


def test_lm_job_streams_are_exclusive():
    """every LM job decodes (and captures its step graph) on a stream no other job and no workspace call uses: torch's pooled
    streams repeat after 32 creations, so concurrent jobs could land on the model's own stream"""
    from contextlib import ExitStack
    m = small_model()
    with ExitStack() as es:
        handles = [es.enter_context(m._lm_stream()).cuda_stream for _ in range(40)]
    assert len(set(handles)) == 40 and m.stream.cuda_stream not in handles
    with m._lm_stream() as s:
        assert s.cuda_stream in handles                  # recycled, not created anew
