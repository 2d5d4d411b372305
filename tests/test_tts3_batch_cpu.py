"""CPU: CosyVoice3 batched offline synthesis (B200CosyVoice3Model.tts_batch) with the device primitives faked by the oracle.

Each request of a ragged batch must get what tts() gives it alone, including the reference's silent-token rule
(cli/model.py:102, 121-127), which tts_batch_device applies to every row's ids through the same helper as tts()."""
import threading

import numpy as np
import pytest
import torch

from oracle import cases, dit, hift_causal as hc, lm, weights
from test_host_logic_cpu import FakeCtx3, _DummyEvent, _DummyStream, _pool

SILENT = [1, 2, 28, 29, 55, 248, 494, 2241, 2242, 2322, 2323]         # cli/model.py:423


class _TimedEvent(_DummyEvent):
    def elapsed_time(self, other):
        return 0.0


class FakeCtx3Batch(FakeCtx3):
    """FakeCtx3 whose LM session, flow3_inference and hift3_inference take ragged batches (every row through the oracle on its
    own).  The LM of a row whose prompt + text has `silent_row_len` ids emits 8 silent ids in place of its ids 2-9."""

    silent_row_len = None

    def lm_prefill(self, sess, tt, tl, ss, sl):
        ot, os_ = np.cumsum([0] + list(tl)), np.cumsum([0] + list(sl))
        sess.update(rows=[(tt[ot[b]:ot[b + 1]].clone(), ss[os_[b]:os_[b + 1]].clone()) for b in range(len(tl))], ids=None)

    def lm_decode(self, sess, n_steps, U, min_len, max_len, out_ids, out_count, done, want_live=True):
        if sess["ids"] is None:
            sess["ids"] = []
            for b, (tt, ss) in enumerate(sess["rows"]):
                ids = self._run({"tt": tt, "ss": ss}, U[:, b:b + 1], int(min_len[b]), int(max_len[b]))
                if len(tt) == self.silent_row_len:
                    ids = ids[:2] + [SILENT[0]] * 8 + ids[10:]
                sess["ids"].append(ids)
            self.last_ids = sess["ids"]
        for b, ids in enumerate(sess["ids"]):
            out_ids[b, :len(ids)] = torch.tensor(ids, dtype=torch.int32)
            out_count[b] = len(ids)
            done[b] = 1
        return 0

    def flow3_inference(self, toks, tl, pf, pl, emb, n_timesteps=10, streaming=False, finalize=True):
        mels, ot, of = [], 0, 0
        for b, (n, p) in enumerate(zip(tl, pl)):
            P = p // 2                                     # prompt mel = 2 frames per prompt token
            row = toks[ot:ot + n]
            mel = self.dit.inference(self.fsd, row[None, P:], row[None, :P], pf[of:of + p][None], emb[b:b + 1], self.depth, n_timesteps,
                                     streaming, finalize)
            mels.append(mel[0].t())
            ot, of = ot + n, of + p
        return torch.cat(mels, 0).contiguous(), [m.shape[0] for m in mels]

    def hift3_inference(self, mel, lens, finalize=True):
        wavs, srcs, o = [], [], 0
        for T in lens:
            self.hift_calls.append((int(T), bool(finalize)))
            wav, src = self.hc.inference(self.hsd, mel[o:o + T].t()[None], self.rand_ini, self.sine_noise, finalize)
            wavs.append(wav[0])
            srcs.append(src.reshape(-1))
            o += T
        return torch.cat(wavs), None, torch.cat(srcs)


def _model(monkeypatch):
    from cosyvoice_b200.model3 import B200CosyVoice3Model
    monkeypatch.setattr(torch.cuda, "Event", _TimedEvent)
    _, rand_ini, sine_noise = cases.hift_causal_case(T=400)
    ctx = FakeCtx3Batch(lm.synth_state_dict3(2), weights.synth_state_dict(dit.flow_param_shapes(2), 1986, dit.SYNTH_GAINS),
                        weights.synth_state_dict(hc.param_shapes(), 1986, hc.SYNTH_GAINS), 2, rand_ini, sine_noise)
    m = object.__new__(B200CosyVoice3Model)
    m.ctx, m.stream, m.device = ctx, _DummyStream(), torch.device("cpu")
    m._lm_streams, m.lm_chains = [_DummyStream()], 1
    _pool(m)
    m.noise_fn, m.generator = None, None
    m.lock = threading.Lock()
    m.tts_speech_token_dict, m.llm_end_dict, m.hift_cache_dict = {}, {}, {}
    m.silent_tokens = list(SILENT)
    m.token_hop_len, m.token_max_hop_len, m.stream_scale_factor = 25, 100, 2
    m.min_token_text_ratio, m.max_token_text_ratio, m.n_timesteps = 2.0, 8.0, 10
    m.incremental_flow = True
    return m


def test_tts3_batch_equals_tts_per_request(monkeypatch):
    """three requests of different text lengths in one tts_batch == each request's tts() alone (same length, values within 1e-5);
    the middle request's LM emits 8 silent ids in a row, of which both paths keep 5"""
    text, ptext, ptok, U = cases.lm3_case()
    _, _, pfeat, emb = cases.flow_case(P=9)
    pfeat = pfeat[:, :18]
    m = _model(monkeypatch)
    m.ctx.silent_row_len = ptext.shape[1] + 5
    m.uniforms_override = U[:, None, :]
    reqs = [dict(text=text[:, :n], prompt_text=ptext, llm_prompt_speech_token=ptok, flow_prompt_speech_token=ptok,
                 prompt_speech_feat=pfeat, flow_embedding=emb) for n in (7, 5, 3)]
    alone = []
    for r in reqs:
        chunks = [o["tts_speech"] for o in m.tts(llm_embedding=emb, stream=False, **r)]
        assert len(chunks) == 1
        alone.append(chunks[0])
    wavs, stats = m.tts_batch(reqs, uniforms=U[:, None, :].expand(-1, len(reqs), -1), return_stats=True)
    assert len({w.shape[1] for w in wavs}) == len(reqs)                     # the batch is ragged
    for i, (w, a) in enumerate(zip(wavs, alone)):
        assert w.shape == a.shape, (i, w.shape, a.shape)
        d = (w - a).abs().max().item()
        assert d < 1e-5, (i, d)
    # the LM's ids as they came; of the middle request's run of 8 silent ids the flow saw 5
    raw = m.ctx.last_ids
    assert raw[1][2:10] == [SILENT[0]] * 8 and raw[1][1] not in SILENT and raw[1][10] not in SILENT
    assert stats["tokens"] == [len(raw[0]), len(raw[1]) - 3, len(raw[2])]
    assert set(stats) >= {"lm_ms", "flow_ms", "hift_ms", "tokens", "mel_frames"}


def test_tts3_batch_refuses_noise(monkeypatch):
    m = _model(monkeypatch)
    with pytest.raises(ValueError):
        m.hift_batch(torch.zeros(10, 80), [10], noise=torch.zeros(4800, 9))
    with pytest.raises(ValueError):
        m.hift_batch(torch.zeros(10, 80), [10], cache_source=torch.zeros(480))


def _reference_rule(ids, silent_tokens):
    """cli/model.py:102, 121-127, transcribed"""
    out, cur_silent_token_num, max_silent_token_num = [], 0, 5
    for i in ids:
        if i in silent_tokens:
            cur_silent_token_num += 1
            if cur_silent_token_num > max_silent_token_num:
                continue
        else:
            cur_silent_token_num = 0
        out.append(i)
    return out


def test_silent_token_filter_matches_reference_rule():
    from cosyvoice_b200.model import SilentTokenFilter
    ids = [7, 1, 1, 2, 28, 29, 55, 248, 494, 9, 2241] + [2242] * 4 + [2322, 2323, 3, 1, 1, 1, 1, 1, 1, 1, 4, 5, 1]
    ref = _reference_rule(ids, SILENT)
    assert ref != ids
    assert SilentTokenFilter(SILENT).filter(ids) == ref
    f = SilentTokenFilter(SILENT)
    assert [t for t in ids if f.keep(t)] == ref
    assert SilentTokenFilter([]).filter(ids) == ids                        # CosyVoice2: nothing is dropped
