"""CPU: the host scheduler of B200CosyVoice2Model.tts_stream_batch over device primitives faked by the oracle - chunk schedule,
one call per stage per poll round, per-request vocoder caches, slot pool (the same method over the real library:
tests/test_stream_batch_gpu.py)."""
import threading

import numpy as np
import torch

from oracle import cases, flow, hift, lm, weights
from oracle.make_golden import stream_noise
from test_host_logic_cpu import FakeCtx2, _DummyEvent, _DummyStream, _pool


class FakeBatchCtx(FakeCtx2):
    """FakeCtx2 with B-row LM sessions, ragged flow / vocoder calls and multi-slot flow sessions; every call is recorded"""

    def __init__(self, *a):
        super().__init__(*a)
        self.calls = []

    # ---- LM: every row decodes its own oracle ids from its own uniforms column
    def lm_prefill(self, sess, tt, tl, ss, sl):
        rows, ot, os_ = [], 0, 0
        for a, b in zip(tl, sl):
            rows.append(dict(tt=tt[ot:ot + a].clone(), ss=ss[os_:os_ + b].clone()))
            ot, os_ = ot + a, os_ + b
        sess.update(rows=rows, ids=None, emitted=[0] * len(rows))

    def lm_decode(self, sess, n_steps, U, min_len, max_len, out_ids, out_count, done, want_live=True):
        if sess["ids"] is None:
            sess["ids"] = [self._run(r, U[:, b:b + 1], int(min_len[b]), int(max_len[b])) for b, r in enumerate(sess["rows"])]
        live = 0
        for b, ids in enumerate(sess["ids"]):
            n = sess["emitted"][b] = min(len(ids), sess["emitted"][b] + n_steps)
            out_ids[b, :n] = torch.tensor(ids[:n], dtype=torch.int32)
            out_count[b] = n
            done[b] = int(n == len(ids))
            live += n < len(ids)
        return live

    # ---- multi-slot flow session: per slot, the frames of the streaming flow call on the prefix not returned yet
    def flow_stream(self, max_frames, n_timesteps=10, dit=False, slots=1):
        if slots == 1:                                   # tts()'s own one-request sessions
            return super().flow_stream(max_frames, n_timesteps, dit)
        self.calls.append(("create", slots))
        return {"slots": [None] * slots, "cap": max_frames}

    def flow_stream_begin_slot(self, fs, slot, prompt_feat, embedding):
        fs["slots"][slot] = {"done": 0, "pf": prompt_feat, "emb": embedding.reshape(1, -1), "dit": False}

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

    def flow_inference(self, toks, tl, pf, pl, emb, n_timesteps=10, streaming=False, finalize=True):
        self.calls.append(("flow", [int(n) for n in tl], bool(streaming), bool(finalize)))
        out, lens, ot, op = [], [], 0, 0
        for b, (n, p) in enumerate(zip(tl, pl)):
            t = toks[ot:ot + n]
            mel = flow.inference(self.fsd, t[None, self._P:], t[None, :self._P], pf[op:op + p][None], emb[b:b + 1], self.fcfg, n_timesteps,
                                 streaming, finalize)
            out.append(mel[0].t())
            lens.append(mel.shape[2])
            ot, op = ot + n, op + p
        return torch.cat(out).contiguous(), lens

    def hift_inference(self, mel, lens, noise, cache_source=None, cache_lens=None):
        self.calls.append(("hift", list(lens), list(cache_lens) if cache_lens is not None else [0] * len(lens)))
        wavs, srcs, om, oc = [], [], 0, 0
        for b, T in enumerate(lens):
            cl = cache_lens[b] if cache_lens is not None else 0
            cs = cache_source[oc:oc + cl].reshape(1, 1, -1) if cl else None
            wav, src = hift.inference(self.hsd, mel[om:om + T].t()[None], noise[om * 480:(om + T) * 480][None], None, cs)
            wavs.append(wav[0])
            srcs.append(src.reshape(-1))
            om, oc = om + T, oc + cl
        return torch.cat(wavs), torch.cat(srcs)


def _model(monkeypatch):
    from cosyvoice_b200.model import B200CosyVoice2Model
    monkeypatch.setattr(torch.cuda, "Event", _DummyEvent)
    fcfg = flow.FlowCfg(enc_blocks=2, enc_up_blocks=1, num_mid_blocks=2, n_blocks=2)
    ctx = FakeBatchCtx(lm.synth_state_dict(2), weights.synth_state_dict(flow.param_shapes(fcfg), 1986, flow.SYNTH_GAINS),
                       weights.synth_state_dict(hift.param_shapes(), 1986, hift.SYNTH_GAINS), fcfg)
    ctx._P = 9
    m = object.__new__(B200CosyVoice2Model)
    m.ctx, m.stream, m.device = ctx, _DummyStream(), torch.device("cpu")
    m._lm_streams, m.lm_chains = [_DummyStream()], 1
    _pool(m)
    m.uniforms_override, m.noise_fn, m.generator = None, None, None
    m.tts_speech_token_dict, m.llm_end_dict, m.hift_cache_dict = {}, {}, {}
    m.silent_tokens = []
    m.token_hop_len, m.token_max_hop_len, m.stream_scale_factor = 25, 100, 2
    m.mel_cache_len, m.source_cache_len = 8, 8 * 480
    m._window = torch.from_numpy(np.hamming(2 * 8 * 480)).float()
    m.min_token_text_ratio, m.max_token_text_ratio, m.n_timesteps = 2.0, 20.0, 10
    m.stream_batch_slots, m.stream_cache_frames = 2, 2048
    return m, ctx


def _case():
    """request 0 = the golden request (tests/golden/stream_tts.npz), request 1 = a longer text with the same prompt"""
    text, ptext, ptok, U = cases.lm_case()
    _, _, pfeat, emb = cases.flow_case(P=9)
    r0 = dict(text=text, flow_embedding=emb, llm_embedding=emb, prompt_text=ptext, llm_prompt_speech_token=ptok, flow_prompt_speech_token=ptok,
              prompt_speech_feat=pfeat[:, :18])
    g = torch.Generator().manual_seed(5)
    r1 = dict(r0, text=torch.randint(0, 151643, (1, 11), generator=g, dtype=torch.int32))
    Ub = torch.rand(U.shape[0], 2, 2, generator=g)
    Ub[:, 0] = U
    return [r0, r1], Ub


def _noise_fns(B):
    def make(i):
        k = {"k": 0}

        def fn(n):
            z = stream_noise(1000 * i + k["k"], n)
            k["k"] += 1
            return z
        return fn
    return [make(i) for i in range(B)]


def _rounds(calls):
    """calls grouped into poll rounds: every round ends with its one vocoder call"""
    out, cur = [], []
    for c in calls:
        if c[0] == "create":
            continue
        cur.append(c)
        if c[0] == "hift":
            out.append(cur)
            cur = []
    assert not cur
    return out


def test_stream_batch_host_logic_matches_reference(golden, monkeypatch):
    g = golden("stream_tts")
    m, ctx = _model(monkeypatch)
    reqs, Ub = _case()
    chunks = [[], []]
    for i, out in m.tts_stream_batch(reqs, uniforms=Ub, noise_fns=_noise_fns(2)):
        chunks[i].append(out["tts_speech"])
    assert [c.shape[1] for c in chunks[0]] == g["stream_lens"].tolist()
    d = np.abs(torch.cat(chunks[0], 1).numpy() - g["stream_wav"])
    assert d[:, :24000].max() < 5e-3 and d.max() < 2e-2, (d[:, :24000].max(), d.max())
    assert m.token_hop_len == 25
    calls = list(ctx.calls)
    # request 1 alone through tts(stream=True), with its uniforms column and noise stream: the same chunks
    m.uniforms_override, m.noise_fn = Ub[:, 1:2, :], _noise_fns(2)[1]
    single = [o["tts_speech"] for o in m.tts(**reqs[1], stream=True)]
    m.uniforms_override, m.noise_fn, m.token_hop_len = None, None, 25
    assert [c.shape[1] for c in chunks[1]] == [c.shape[1] for c in single]
    assert np.abs(torch.cat(chunks[1], 1).numpy() - torch.cat(single, 1).numpy()).max() < 1e-5
    rounds = _rounds(calls)
    for r in rounds:
        kinds = [c[0] if c[0] != "flow" else ("final" if c[3] else "prefix") for c in r]
        assert all(kinds.count(k) <= 1 for k in ("chunk_batch", "prefix", "final", "hift")), kinds
        assert "prefix" not in kinds                     # both requests hold a slot
    batch = [c for r in rounds for c in r if c[0] == "chunk_batch"]
    # the first round serves both first chunks (hop 25 padded to 41, 3 look-ahead tokens) in one call, slots 0 and 1
    assert batch[0] == ("chunk_batch", [0, 1], [9 + 41 + 3, 9 + 41 + 3])
    # request 0's vocoder calls: no cached source on its first chunk, then 3840 cached samples every time
    assert [c[2][0] for c in [c for r in rounds for c in r if c[0] == "hift"]][:3] == [0, 3840, 3840]
    assert sorted(m._free_slots) == [0, 1]


def test_closing_the_generator_releases_the_slots(monkeypatch):
    m, ctx = _model(monkeypatch)
    reqs, Ub = _case()
    gen = m.tts_stream_batch(reqs, uniforms=Ub, noise_fns=_noise_fns(2))
    i, out = next(gen)
    assert out["tts_speech"].shape[1] > 0
    assert len(m._free_slots) == 0                       # both requests hold a slot mid-stream
    gen.close()
    assert sorted(m._free_slots) == [0, 1]


def test_stream_batch_refuses_text_generators_and_cosyvoice3(monkeypatch):
    import pytest
    from cosyvoice_b200.model3 import B200CosyVoice3Model
    m, _ = _model(monkeypatch)
    reqs, _ = _case()
    with pytest.raises(ValueError):
        next(m.tts_stream_batch([dict(reqs[0], text=iter([reqs[0]["text"]]))]))
    m3 = object.__new__(B200CosyVoice3Model)
    with pytest.raises(NotImplementedError):
        m3.tts_stream_batch(reqs)


def test_batcher_never_mixes_streaming_and_offline_requests():
    """admission: a batch is the run of same-kind requests at the head of the queue"""
    from cosyvoice_b200.batcher import TtsBatcher

    class Model:
        def __init__(self):
            self.gate = threading.Event()

        def tts_batch(self, inputs):
            self.gate.wait(5)
            return [torch.full((1, 3), float(r["text"])) for r in inputs]

        def tts_stream_batch(self, inputs):
            self.gate.wait(5)
            for k in range(2):
                for i, r in enumerate(inputs):
                    yield i, {"tts_speech": torch.full((1, 2), float(r["text"]) + k)}

    model = Model()
    with TtsBatcher(model, max_batch=8, max_wait_ms=200) as b:
        s1, s2 = b.submit_stream(text=1), b.submit_stream(text=2)
        f3 = b.submit(text=3)
        s4 = b.submit_stream_pcm(text=4)
        model.gate.set()
        assert [float(c[0, 0]) for c in s1] == [1.0, 2.0]
        assert [float(c[0, 0]) for c in s2] == [2.0, 3.0]
        assert float(f3.result(5)[0, 0]) == 3.0
        assert len(list(s4)) == 2
    assert b.batches == [2, 1, 1]


def test_slot_pool_takes_the_largest_slot_count_that_fits(monkeypatch):
    """a session of stream_batch_slots slots that cannot be allocated is retried with half as many; the outcome is reported
    once (warning, stream_slots) and kept: later requests do not retry the allocation"""
    import pytest
    from cosyvoice_b200.cvk import CvkError
    m, ctx = _model(monkeypatch)
    tried = []

    def flow_stream(max_frames, n_timesteps=10, dit=False, slots=1):
        tried.append(slots)
        if slots > 3:
            raise CvkError("libcvk status -3: out of memory")
        return {"slots": [None] * slots, "cap": max_frames}
    monkeypatch.setattr(ctx, "flow_stream", flow_stream)
    m.stream_batch_slots = 16
    with pytest.warns(RuntimeWarning, match="2 of 16"):
        assert m._take_slot() == 0
    assert tried == [16, 8, 4, 2] and m.stream_slots == 2
    assert m._take_slot() == 1 and m._take_slot() is None and tried == [16, 8, 4, 2]

    m2, ctx2 = _model(monkeypatch)
    monkeypatch.setattr(ctx2, "flow_stream", lambda *a, **k: (_ for _ in ()).throw(CvkError("out of memory")))
    with pytest.warns(RuntimeWarning, match="0 of 2"):
        assert m2._take_slot() is None
    assert m2.stream_slots == 0 and m2._take_slot() is None
