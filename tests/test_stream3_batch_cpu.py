"""CPU: CosyVoice3 batched streaming (B200CosyVoice3Model.tts_stream_batch / tts_bistream_batch) with the device primitives faked
by the oracle: multi-slot DiT flow sessions, ragged flow3_inference and the per-utterance-flag vocoder call hift3_inference_rows.

Each request must get the chunks tts(stream=True) gives it alone, and every poll round must make at most one call per stage, with
streaming and finishing requests sharing the round's one vocoder call (the same class over the real library:
tests/test_zz_stream3_batch_gpu.py)."""
import numpy as np
import pytest
import torch

from oracle import cases, lm
from test_bistream_batch_cpu import RowsMixin
from test_tts3_batch_cpu import SILENT, FakeCtx3Batch, _model as _model3


class FakeStream3Ctx(FakeCtx3Batch):
    """FakeCtx3Batch (ragged LM session, flow3_inference) with multi-slot DiT flow sessions and hift3_inference_rows; the calls
    of the batched path are recorded in self.calls.  Its LM hands out every row's ids in its first decode call, so the poll
    rounds do not depend on thread timing."""

    def __init__(self, *a):
        super().__init__(*a)
        self.calls = []

    def _prefix_mel(self, fs, toks):
        """the streaming DiT call on the session's prefix; the prompt has 2 mel frames per prompt token"""
        assert fs["dit"]
        P = fs["pf"].shape[0] // 2
        return self.dit.inference(self.fsd, toks[None, P:], toks[None, :P], fs["pf"][None], fs["emb"], self.depth, 10, True, False)[0].t()

    # ---- multi-slot DiT session: per slot, the frames of the streaming flow call on the prefix not returned yet
    def flow_stream(self, max_frames, n_timesteps=10, dit=False, slots=1):
        if slots == 1:                                   # tts()'s own one-request sessions
            return super().flow_stream(max_frames, n_timesteps, dit)
        assert dit
        self.calls.append(("create", slots))
        return {"slots": [None] * slots, "cap": max_frames}

    def flow_stream_begin_slot(self, fs, slot, prompt_feat, embedding):
        fs["slots"][slot] = {"done": 0, "pf": prompt_feat, "emb": embedding.reshape(1, -1), "dit": True}

    def flow_stream_chunk_batch(self, fs, slots, token_list):
        self.calls.append(("chunk_batch", list(slots), [int(t.numel()) for t in token_list]))
        out, lens = [], []
        for s, toks in zip(slots, token_list):
            st = fs["slots"][s]
            mel = self._prefix_mel(st, toks)
            Tp = st["pf"].shape[0]
            new = mel[max(st["done"] - Tp, 0):]
            st["done"] = Tp + mel.shape[0]
            assert st["done"] % 50 == 0 and st["done"] <= fs["cap"]
            out.append(new)
            lens.append(new.shape[0])
        return torch.cat(out).contiguous(), lens

    def flow3_inference(self, toks, tl, pf, pl, emb, n_timesteps=10, streaming=False, finalize=True):
        self.calls.append(("flow", [int(n) for n in tl], bool(streaming), bool(finalize)))
        return super().flow3_inference(toks, tl, pf, pl, emb, n_timesteps, streaming, finalize)

    def hift3_inference_rows(self, mel, lens, finalize):
        """every utterance through the oracle on its own with its own flag: wav 480 T (final) or 480 (T-8) (streaming)"""
        self.calls.append(("hift_rows", [int(T) for T in lens], [bool(f) for f in finalize]))
        wavs, srcs, o = [], [], 0
        for T, f in zip(lens, finalize):
            assert f or T >= 9
            wav, src = self.hc.inference(self.hsd, mel[o:o + T].t()[None], self.rand_ini, self.sine_noise, bool(f))
            wavs.append(wav[0])
            srcs.append(src.reshape(-1))
            o += T
        return torch.cat(wavs), None, torch.cat(srcs)


def _model(monkeypatch, slots=3):
    m = _model3(monkeypatch)
    base = m.ctx
    ctx = FakeStream3Ctx(base.lsd, base.fsd, base.hsd, base.depth, base.rand_ini, base.sine_noise)
    m.ctx = ctx
    m.min_token_text_ratio, m.max_token_text_ratio = 2.0, 20.0         # the golden request's LM runs to 140 ids
    m.uniforms_override = None
    m.stream_batch_slots, m.stream_cache_frames, m.stream_slots, m._slot_pool = slots, 2048, None, None
    return m, ctx


def _requests():
    """request 0 = the golden request of tests/golden/stream3_tts.npz (prompt 9 tokens / 18 frames); request 1: prompt 6 tokens,
    5 text ids; request 2: prompt 12 tokens, 3 text ids.  Uniforms [n, 3, 2]: column i is request i's draws."""
    text, ptext, ptok, U = cases.lm3_case()
    _, _, pfeat, emb = cases.flow_case(P=9)
    _, ptok12, pfeat12, emb2 = cases.flow_case(P=12, seed=4)
    g = torch.Generator().manual_seed(77)
    r0 = dict(text=text, prompt_text=ptext, llm_prompt_speech_token=ptok, flow_prompt_speech_token=ptok, prompt_speech_feat=pfeat[:, :18],
              flow_embedding=emb, llm_embedding=emb)
    r1 = dict(r0, text=torch.randint(0, 151643, (1, 5), generator=g, dtype=torch.int32), llm_prompt_speech_token=ptok[:, :6],
              flow_prompt_speech_token=ptok[:, :6], prompt_speech_feat=pfeat[:, :12])
    r2 = dict(r0, text=torch.randint(0, 151643, (1, 3), generator=g, dtype=torch.int32), llm_prompt_speech_token=ptok12,
              flow_prompt_speech_token=ptok12, prompt_speech_feat=pfeat12, flow_embedding=emb2, llm_embedding=emb2)
    Ub = torch.rand(U.shape[0], 3, 2, generator=g)
    Ub[:, 0] = U
    return [r0, r1, r2], Ub


def _collect(gen, B):
    chunks = [[] for _ in range(B)]
    for i, out in gen:
        chunks[i].append(out["tts_speech"])
    return chunks


def _alone(m, reqs, Ub):
    out = []
    for i, r in enumerate(reqs):
        m.uniforms_override, m.token_hop_len = Ub[:, i:i + 1], 25
        try:
            out.append([o["tts_speech"] for o in m.tts(**r, stream=True)])
        finally:
            m.uniforms_override, m.token_hop_len = None, 25
    return out


def _rounds(calls):
    """calls grouped into poll rounds: a round ends with its one vocoder call"""
    out, cur = [], []
    for c in calls:
        if c[0] == "create":
            continue
        cur.append(c)
        if c[0] == "hift_rows":
            out.append(cur)
            cur = []
    assert not cur
    return out


def _check(chunks, alone, tol=1e-6):
    for i, (c, a) in enumerate(zip(chunks, alone)):
        assert [x.shape[1] for x in c] == [x.shape[1] for x in a], i
        assert all(x.dtype == torch.float32 and x.shape[0] == 1 for x in c)
        d = np.abs(torch.cat(c, 1).numpy() - torch.cat(a, 1).numpy()).max()
        assert d < tol, (i, d)


_cache = {}


def _singles(m, reqs, Ub):
    if "alone" not in _cache:
        _cache["alone"] = _alone(m, reqs, Ub)
    return _cache["alone"]


def test_stream3_batch_equals_tts_per_request(golden, monkeypatch):
    """a ragged batch of three requests with different prompt lengths: each request's chunks == tts(stream=True) alone (lengths
    identical, waveforms within 1e-6); request 0 reproduces the reference's own streaming output; every poll round makes at most
    one call per stage, and the round where request 2 finishes while 0 and 1 stream has one vocoder call with mixed flags"""
    g = golden("stream3_tts")
    m, ctx = _model(monkeypatch)
    reqs, Ub = _requests()
    alone = _singles(m, reqs, Ub)
    ctx.calls.clear()
    chunks = _collect(m.tts_stream_batch(reqs, uniforms=Ub), 3)
    _check(chunks, alone)
    assert [c.shape[1] for c in chunks[0]] == g["stream_lens"].tolist()
    d = np.abs(torch.cat(chunks[0], 1).numpy() - g["stream_wav"])
    assert d[:, :24000].max() < 2e-3 and d.max() < 1e-2
    assert m.token_hop_len == 25 and sorted(m._free_slots) == [0, 1, 2]
    rounds = _rounds(ctx.calls)
    for r in rounds:
        kinds = [c[0] if c[0] != "flow" else ("final" if c[3] else "prefix") for c in r]
        assert all(kinds.count(k) <= 1 for k in ("chunk_batch", "prefix", "final")) and kinds.count("hift_rows") == 1, kinds
        assert "prefix" not in kinds                     # every request holds a slot
    voc = [c for r in rounds for c in r if c[0] == "hift_rows"]
    # round 1: the three first chunks (hops 25 + prompt padding 16 / 19 / 13) in one DiT call and one streaming vocoder call
    assert rounds[0][0] == ("chunk_batch", [0, 1, 2], [9 + 41 + 3, 6 + 44 + 3, 12 + 38 + 3])
    assert voc[0][2] == [False, False, False] and voc[0][1] == [82, 88, 76]
    # round 2: requests 0 and 1 stream their second chunk, request 2 (60 ids) finishes: one call with per-utterance flags over
    # each request's whole mel so far
    assert voc[1][2] == [False, False, True] and voc[1][1] == [182, 188, 2 * 60]
    assert any(len(set(c[2])) == 2 for c in voc)


def test_stream3_batch_fallback_paths(monkeypatch):
    """no slots (prefix recompute for every chunk) and incremental_flow = False give the same chunks"""
    m, ctx = _model(monkeypatch)
    reqs, Ub = _requests()
    alone = _singles(m, reqs, Ub)
    for mode in ("no_slots", "no_incremental"):
        m, ctx = _model(monkeypatch, slots=0 if mode == "no_slots" else 3)
        m.incremental_flow = mode != "no_incremental"
        chunks = _collect(m.tts_stream_batch(reqs, uniforms=Ub), 3)
        _check(chunks, alone)
        rounds = _rounds(ctx.calls)
        assert not any(c[0] == "chunk_batch" for r in rounds for c in r)
        for r in rounds:
            kinds = [("final" if c[3] else "prefix") for c in r if c[0] == "flow"]
            assert all(kinds.count(k) <= 1 for k in ("prefix", "final")), (mode, kinds)


def test_stream3_batch_filters_silent_runs_like_tts(monkeypatch):
    """request 1's LM emits 8 silent ids in a row: the batch keeps 5 of them like tts() does, and its chunks equal tts()'s"""
    m, ctx = _model(monkeypatch)
    reqs, Ub = _requests()
    ctx.silent_row_len = reqs[1]["prompt_text"].shape[1] + reqs[1]["text"].shape[1]
    reqs, Ub = reqs[:2], Ub[:, :2].contiguous()
    alone = _alone(m, reqs, Ub)
    ctx.calls.clear()
    chunks = _collect(m.tts_stream_batch(reqs, uniforms=Ub), 2)
    _check(chunks, alone)
    # request 1's final flow call: its 6 prompt tokens and its 100 ids minus the 3 dropped silent ones
    assert any(c[0] == "flow" and c[3] and 6 + 97 in c[1] for c in ctx.calls)


def test_stream3_batch_refusals(monkeypatch):
    m, _ = _model(monkeypatch)
    reqs, Ub = _requests()
    with pytest.raises(ValueError):
        next(m.tts_stream_batch(reqs, uniforms=Ub, noise_fns=[lambda n: torch.zeros(n, 9)] * 3))
    with pytest.raises(ValueError):
        next(m.tts_bistream_batch([dict(reqs[0], text=iter([reqs[0]["text"]]))], noise_fns=[lambda n: torch.zeros(n, 9)]))
    with pytest.raises(ValueError):                      # text generators go to tts_bistream_batch (inherited check)
        next(m.tts_stream_batch([dict(reqs[0], text=iter([reqs[0]["text"]]))]))


def test_closing_the_generator_returns_every_slot(monkeypatch):
    m, _ = _model(monkeypatch)
    reqs, Ub = _requests()
    gen = m.tts_stream_batch(reqs, uniforms=Ub)
    i, out = next(gen)
    assert out["tts_speech"].shape[1] > 0
    assert len(m._free_slots) == 0                       # all three requests hold a slot mid-stream
    gen.close()
    assert sorted(m._free_slots) == [0, 1, 2]


class FakeBistream3Ctx(RowsMixin, FakeStream3Ctx):
    """FakeStream3Ctx with the ragged text-streaming LM session calls on a CosyVoice3LM state_dict"""

    def __init__(self, *a):
        super().__init__(*a)
        self.sd, self.nl, self.cv3, self.lm_calls = self.lsd, 2, True, []

    def lm_session(self, B, ctx_len):
        return {"B": B}


def test_tts_bistream3_batch_equals_tts_per_request(golden, monkeypatch):
    """tts_bistream_batch over cases.bistream3_case(): the text in its own chunks and re-chunked by 1 and 7 ids, each with its own
    flow prompt; each request == tts(text=iter(chunks), stream=True) alone, and the LM ids are the reference's"""
    from test_bistream_batch_cpu import _rechunk
    m, base = _model(monkeypatch)
    ctx = FakeBistream3Ctx(lm.bistream_state_dict3(2), base.fsd, base.hsd, base.depth, base.rand_ini, base.sine_noise)
    m.ctx = ctx
    m.bistream_max_tokens = 130
    m.silent_tokens = []          # the synthetic ids are uniform over the codebook: count every id
    chunks, ptext, ptok, U = cases.bistream3_case()
    reqs3, _ = _requests()
    texts = [chunks, _rechunk(chunks, 1), _rechunk(chunks, 7)]
    reqs = [dict(r, text=t, prompt_text=ptext, llm_prompt_speech_token=ptok) for r, t in zip(reqs3, texts)]
    Ub = torch.stack([U] * 3, 1)
    got = _collect(m.tts_bistream_batch([dict(r, text=iter(r["text"])) for r in reqs], uniforms=Ub), 3)
    assert sorted(m._free_slots) == [0, 1, 2] and m.token_hop_len == 25
    n_ids = len(golden("lm3_bistream_l2")["ids"])
    alone = []
    for i, r in enumerate(reqs):
        m.uniforms_override, m.token_hop_len = Ub[:, i:i + 1], 25
        try:
            alone.append([o["tts_speech"] for o in m.tts(**dict(r, text=iter(r["text"])), stream=True)])
        finally:
            m.uniforms_override, m.token_hop_len = None, 25
    _check(got, alone)
    for i, c in enumerate(got):                          # 960 samples per id of the reference's decode
        assert sum(x.shape[1] for x in c) == n_ids * 960, i


def test_batcher_serves_cosyvoice3_streaming_requests(monkeypatch):
    from cosyvoice_b200.batcher import TtsBatcher, pcm16
    m, _ = _model(monkeypatch)
    reqs, Ub = _requests()
    reqs, Ub = reqs[1:], Ub[:, 1:].contiguous()
    m.uniforms_override = Ub
    try:
        want = _collect(m.tts_stream_batch(reqs), 2)
        with TtsBatcher(m, max_batch=2, max_wait_ms=2000) as b:
            s1, s2 = b.submit_stream(**reqs[0]), b.submit_stream_pcm(**reqs[1])
            got1, got2 = list(s1), list(s2)
        assert b.batches == [2]
    finally:
        m.uniforms_override = None
    assert len(got1) == len(want[0]) and all(torch.equal(a, w) for a, w in zip(got1, want[0]))
    assert got2 == [pcm16(w) for w in want[1]]
