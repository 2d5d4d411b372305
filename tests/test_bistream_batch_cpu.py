"""CPU: the batched text-streaming LM (`lm_generate_bistream_batch`) and `tts_bistream_batch` with the ragged session calls
(cvk_lm_feed_rows / cvk_lm_next_logp_rows / cvk_ras_sample) faked by the oracle with one KV cache per row."""
import random
import time

import numpy as np
import pytest
import torch

from oracle import cases, lm, sampling
from test_host_logic_cpu import _model_with
from test_stream_batch_cpu import FakeBatchCtx, _model as _stream_model, _noise_fns


class RowsMixin:
    """per-row oracle KV caches behind the ragged session calls; every call is recorded in self.lm_calls"""

    def lm_begin(self, sess, B=1):
        sess.update(past=[None] * B, hidden=[None] * B)

    def _emb(self, i, k):
        if k == 2 and self.cv3:
            return self.sd["speech_embedding.weight"][(6561, 6563)[i]]
        return self.sd[{0: "llm.model.model.embed_tokens.weight", 1: "speech_embedding.weight", 2: "llm_embedding.weight"}[k]][i]

    def _head(self, y):
        if self.cv3:
            return torch.log_softmax(torch.nn.functional.linear(y, self.sd["llm_decoder.weight"]), -1)
        return lm.logprobs(self.sd, y)

    def lm_feed_rows(self, sess, rows, counts, ids, kinds):
        self.lm_calls.append(("feed", list(rows), list(counts)))
        assert len(set(rows)) == len(rows) and len(ids) == len(kinds) == sum(counts)
        o = 0
        for r, n in zip(rows, counts):
            x = torch.stack([self._emb(i, k) for i, k in zip(ids[o:o + n], kinds[o:o + n])])[None]
            y, sess["past"][r] = lm.qwen2_forward(self.sd, x, sess["past"][r], self.nl)
            sess["hidden"][r] = y[:, -1]
            o += n

    def lm_next_logp_rows(self, sess, rows):
        self.lm_calls.append(("logp", list(rows)))
        return torch.cat([self._head(sess["hidden"][r]) for r in rows])

    def lm_feed(self, sess, ids, kinds):                 # the single-request calls on row 0 (tts(text=generator))
        self.lm_feed_rows(sess, [0], [len(ids)], ids, kinds)

    def lm_next_logp(self, sess, B=1):
        return self.lm_next_logp_rows(sess, [0])

    def ras_sample(self, logp, history, hist_count, uniforms, ignore_eos):
        self.lm_calls.append(("sample", int(logp.shape[0])))
        return torch.tensor([sampling.ras_sample(logp[b].numpy(), history[b, :int(hist_count[b])].tolist(), float(uniforms[b, 0]),
                                                 float(uniforms[b, 1]), ignore_eos=bool(ignore_eos[b])) for b in range(logp.shape[0])],
                            dtype=torch.int32)


class FakeRowsCtx(RowsMixin):
    def __init__(self, sd, num_layers, cv3=False):
        import threading
        self.sd, self.nl, self.cv3 = sd, num_layers, cv3
        self.lock = threading.Lock()
        self.lm_calls, self.destroyed = [], 0

    def lm_session(self, B, ctx_len):
        return {"B": B}

    def lm_session_destroy(self, sess):
        self.destroyed += 1


def _rechunk(chunks, n):
    flat = torch.cat([c.reshape(-1) for c in chunks])
    return [flat[i:i + n].reshape(1, -1) for i in range(0, flat.numel(), n)]


def _batch_case():
    """row 0: the golden case; rows 1-3: the same text in one chunk, 1-id chunks and 7-id chunks; row 4: a different text with its
    own uniforms"""
    chunks, ptext, ptok, U = cases.bistream_case()
    other, _, _, U2 = cases.bistream_case(seed=12)
    texts = [chunks, _rechunk(chunks, 10 ** 6), _rechunk(chunks, 1), _rechunk(chunks, 7), other]
    Ub = torch.stack([U, U, U, U, U2], 1)
    return texts, ptext, ptok, Ub


def _delayed(chunks, rng):
    for c in chunks:
        time.sleep(rng.random() * 0.004)
        yield c


def _run(m, texts, ptext, ptok, Ub, rng=None):
    gens = [iter(t) if rng is None else _delayed(t, rng) for t in texts]
    out = [[] for _ in texts]
    for i, tok in m.lm_generate_bistream_batch(gens, [ptext] * len(texts), [ptok] * len(texts), uniforms=Ub):
        out[i].append(tok)
    return out


def test_batch_ids_match_the_oracle_row_by_row(golden):
    texts, ptext, ptok, Ub = _batch_case()
    sd = lm.bistream_state_dict(2)
    ctx = FakeRowsCtx(sd, 2)
    m = _model_with(ctx)
    out = _run(m, texts, ptext, ptok, Ub)
    assert out[0] == golden("lm_bistream_l2")["ids"].tolist()
    for i, t in enumerate(texts):
        assert out[i] == lm.inference_bistream(sd, t, ptext, ptok, Ub[:, i], num_layers=2), i
    # every step: one feed call, then at most one log-prob call and one sampler call for the rows that draw
    steps = []
    for c in ctx.lm_calls:
        if c[0] == "feed":
            steps.append([c])
        else:
            steps[-1].append(c)
    for s in steps:
        kinds = [c[0] for c in s]
        assert kinds in (["feed"], ["feed", "logp", "sample"]), kinds
        if len(s) == 3:
            assert set(s[1][1]) <= set(s[0][1]) and s[2][1] == len(s[1][1])
    assert max(len(s[0][1]) for s in steps) == len(texts)          # the rows do share steps
    # the session went back to the pool
    assert sum(len(v) for v in m._free_sessions.values()) == 1 and ctx.destroyed == 0


def test_arrival_timing_does_not_change_the_ids():
    texts, ptext, ptok, Ub = _batch_case()
    sd = lm.bistream_state_dict(2)
    m = _model_with(FakeRowsCtx(sd, 2))
    ref = _run(m, texts, ptext, ptok, Ub)
    for seed in (1, 2):
        assert _run(m, texts, ptext, ptok, Ub, rng=random.Random(seed)) == ref


def test_cosyvoice3_batch_ids_match_the_oracle(golden):
    from cosyvoice_b200.model3 import B200CosyVoice3Model
    chunks, ptext, ptok, U = cases.bistream3_case()
    sd = lm.bistream_state_dict3(2)
    ctx = FakeRowsCtx(sd, 2, cv3=True)
    m = object.__new__(B200CosyVoice3Model)
    m.ctx, m.stream, m.device = ctx, None, torch.device("cpu")
    m.uniforms_override, m.generator = None, None
    from test_host_logic_cpu import _pool
    _pool(m)
    texts = [chunks, _rechunk(chunks, 1), _rechunk(chunks, 7)]
    Ub = torch.stack([U] * 3, 1)
    out = _run(m, texts, ptext, ptok, Ub)
    assert out[0] == golden("lm3_bistream_l2")["ids"].tolist()
    for i, t in enumerate(texts):
        assert out[i] == lm.inference_bistream(sd, t, ptext, ptok, U, num_layers=2, variant="cv3"), i
    # without <|endofprompt|> in a row's prompt text the whole generator fails like the reference (llm.py:585)
    with pytest.raises(AssertionError):
        list(m.lm_generate_bistream_batch([iter(chunks), iter(chunks)], [ptext, ptext.clamp(max=151645)], [ptok, ptok], uniforms=Ub))


class _BadDrawCtx(FakeRowsCtx):
    """row 1's sampler draws 6562, which the Qwen2LM text-streaming loop does not expect"""

    def lm_next_logp_rows(self, sess, rows):
        self.rows_drawn = list(rows)
        return super().lm_next_logp_rows(sess, rows)

    def ras_sample(self, logp, history, hist_count, uniforms, ignore_eos):
        top = super().ras_sample(logp, history, hist_count, uniforms, ignore_eos)
        if 1 in self.rows_drawn:
            top[self.rows_drawn.index(1)] = 6562
        return top


def test_row_errors_end_the_generator_and_closing_returns_the_session():
    texts, ptext, ptok, Ub = _batch_case()
    sd = lm.bistream_state_dict(2)
    ctx = _BadDrawCtx(sd, 2)
    m = _model_with(ctx)
    with pytest.raises(ValueError):
        _run(m, texts[:2], ptext, ptok, Ub[:, :2])
    assert sum(len(v) for v in m._free_sessions.values()) == 1
    ctx = FakeRowsCtx(sd, 2)
    m = _model_with(ctx)
    gen = m.lm_generate_bistream_batch([iter(t) for t in texts], [ptext] * 5, [ptok] * 5, uniforms=Ub)
    next(gen)
    n = len(ctx.lm_calls)
    gen.close()
    assert len(ctx.lm_calls) == n                                  # no further step after the close
    assert sum(len(v) for v in m._free_sessions.values()) == 1 and ctx.destroyed == 0


class FakeBistreamCtx(RowsMixin, FakeBatchCtx):
    def __init__(self, *a):
        super().__init__(*a)
        self.sd, self.nl, self.cv3, self.lm_calls = self.lsd, 2, False, []

    def lm_session(self, B, ctx_len):
        return {"B": B}


def test_tts_bistream_batch_gives_each_request_its_single_request_chunks(monkeypatch):
    m, _ = _stream_model(monkeypatch)
    ctx = FakeBistreamCtx(m.ctx.lsd, m.ctx.fsd, m.ctx.hsd, m.ctx.fcfg)
    ctx._P = m.ctx._P
    m.ctx = ctx
    m.bistream_max_tokens = 130                        # synthetic weights: bound the 'decode until eos' phase like the benchmarks do
    chunks, ptext, ptok, U = cases.bistream_case()
    other, _, _, U2 = cases.bistream_case(seed=12)
    from test_stream_batch_cpu import _case
    (r0, _), _ = _case()
    texts = [chunks, other]
    reqs = [dict(r0, text=iter(t), prompt_text=ptext, llm_prompt_speech_token=ptok) for t in texts]
    Ub = torch.stack([U, U2], 1)
    got = [[], []]
    for i, out in m.tts_bistream_batch(reqs, uniforms=Ub, noise_fns=_noise_fns(2)):
        got[i].append(out["tts_speech"])
    assert sorted(m._free_slots) == [0, 1] and m.token_hop_len == 25
    for i, t in enumerate(texts):
        m.uniforms_override, m.noise_fn = Ub[:, i:i + 1, :], _noise_fns(2)[i]
        single = [o["tts_speech"] for o in m.tts(**dict(reqs[i], text=iter(t)), stream=True)]
        m.token_hop_len = 25
        assert [c.shape[1] for c in got[i]] == [c.shape[1] for c in single], i
        assert np.abs(torch.cat(got[i], 1).numpy() - torch.cat(single, 1).numpy()).max() < 1e-5
    m.uniforms_override, m.noise_fn = None, None


def test_cosyvoice3_refuses_tts_bistream_batch():
    from cosyvoice_b200.model3 import B200CosyVoice3Model
    m3 = object.__new__(B200CosyVoice3Model)
    with pytest.raises(NotImplementedError):
        m3.tts_bistream_batch([])
