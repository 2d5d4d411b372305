"""CPU: every request kind of tts() in the batched paths - voice conversion (source_speech_token, no LM), requests without prompt
keys (cross-lingual, instruct2), per-request `speed` - with the device primitives faked by the oracle and a fake cvk_mel_resample
that calls F.interpolate per sequence (the kernel itself is held to F.interpolate bit for bit in tests/test_zz_vc_speed_batch_gpu.py).

Each request of a mixed batch must get what tts() gives it alone, offline for both models and streaming for CosyVoice2, and the
requests the batched paths refuse must be refused before any work."""
import threading

import pytest
import torch
import torch.nn.functional as F

from oracle import cases
from oracle.make_golden import stream_noise
import test_stream_batch_cpu as sb
import test_tts3_batch_cpu as t3


def fake_mel_resample(ctx):
    """cvk_mel_resample on the CPU: F.interpolate(mode="linear") per sequence; the calls are recorded in ctx.resample_calls"""
    ctx.resample_calls = []

    def mel_resample(mel, lens, out_lens):
        ctx.resample_calls.append((list(lens), list(out_lens)))
        out, o = [], 0
        for T, Tn in zip(lens, out_lens):
            out.append(F.interpolate(mel[o:o + T].t()[None], size=Tn, mode="linear")[0].t())
            o += T
        return torch.cat(out).contiguous()
    ctx.mel_resample = mel_resample


def mixed_requests(ptext, ptok, pfeat, emb, seed):
    """zero-shot, cross-lingual (prompt_text and llm_prompt_speech_token deleted), instruct2-shaped (llm_prompt_speech_token
    deleted), voice conversion (no text keys), zero-shot at speed 0.8 and voice conversion at speed 1.25 - the model inputs of
    cli/frontend.py:191-225"""
    g = torch.Generator().manual_seed(seed)

    def text(n):
        return torch.randint(0, 151643, (1, n), generator=g, dtype=torch.int32)
    flow_keys = dict(flow_prompt_speech_token=ptok, prompt_speech_feat=pfeat, flow_embedding=emb)
    zero_shot = dict(text=text(5), prompt_text=ptext, llm_prompt_speech_token=ptok, **flow_keys)
    cross = dict(text=text(4), **flow_keys)
    instruct = dict(text=text(3), prompt_text=text(6), **flow_keys)
    vc = dict(source_speech_token=torch.randint(0, 6561, (1, 23), generator=g, dtype=torch.int32), **flow_keys)
    slow = dict(zero_shot, text=text(4), speed=0.8)
    fast_vc = dict(vc, source_speech_token=torch.randint(0, 6561, (1, 31), generator=g, dtype=torch.int32), speed=1.25)
    return [zero_shot, cross, instruct, vc, slow, fast_vc]


def _alone(m, reqs, Ub, noise=True):
    """every request through tts() alone with its uniforms column and (CosyVoice2) its noise stream stream_noise(i, .)"""
    out = []
    for i, r in enumerate(reqs):
        m.uniforms_override = Ub[:, i:i + 1]
        if noise:
            m.noise_fn = lambda n, i=i: stream_noise(i, n)
        try:
            chunks = [o["tts_speech"] for o in m.tts(stream=False, **r)]
        finally:
            m.uniforms_override, m.noise_fn = None, None
        assert len(chunks) == 1
        out.append(chunks[0])
    return out


def _check(wavs, alone):
    for i, (w, a) in enumerate(zip(wavs, alone)):
        assert w.shape == a.shape, (i, w.shape, a.shape)
        d = (w - a).abs().max().item()
        assert d < 1e-5, (i, d)


def _model2(monkeypatch):
    m, ctx = sb._model(monkeypatch)
    monkeypatch.setattr(torch.cuda, "Event", t3._TimedEvent)          # tts_batch reads its stage times
    m.max_token_text_ratio = 6.0
    fake_mel_resample(ctx)
    return m, ctx


def _case2(B):
    text, ptext, ptok, U = cases.lm_case()
    _, _, pfeat, emb = cases.flow_case(P=9)
    reqs = mixed_requests(ptext, ptok, pfeat[:, :18], emb, seed=77)
    Ub = torch.rand(U.shape[0], B, 2, generator=torch.Generator().manual_seed(78))
    return reqs, Ub


def test_tts_batch_mixed_kinds_equals_tts(monkeypatch):
    """CosyVoice2: one tts_batch over the six request kinds == each request's tts() alone (length, values within 1e-5); the LM
    sees only the four LM rows, one mel_resample call stretches the batch"""
    m, ctx = _model2(monkeypatch)
    reqs, Ub = _case2(6)
    alone = _alone(m, reqs, Ub)
    ctx.calls.clear()
    ctx.resample_calls.clear()
    lens = [a.shape[1] for a in alone]
    noise = torch.cat([stream_noise(i, n) for i, n in enumerate(lens)], 0)
    wavs, stats = m.tts_batch(reqs, uniforms=Ub, noise=noise, return_stats=True)
    _check(wavs, alone)
    assert stats["tokens"][3] == 23 and stats["tokens"][5] == 31           # voice conversion: the source tokens, no LM
    assert len(ctx.resample_calls) == 1
    flow = stats["flow_frames"]
    assert ctx.resample_calls[0] == (flow, stats["mel_frames"])
    assert stats["mel_frames"][4] == int(flow[4] / 0.8) and stats["mel_frames"][5] == int(flow[5] / 1.25)
    assert [stats["mel_frames"][b] for b in (0, 1, 2, 3)] == [flow[b] for b in (0, 1, 2, 3)]
    assert [n * 480 for n in stats["mel_frames"]] == lens
    hift = [c for c in ctx.calls if c[0] == "hift"]
    assert len(hift) == 1 and hift[0][1] == stats["mel_frames"]


def test_vc_rows_and_lm_rows_do_not_depend_on_each_other(monkeypatch):
    """a VC row's waveform is the same alone and next to LM rows; an LM row's ids and waveform do not change when a VC row joins
    (request i keeps its uniforms column); a batch of VC rows only makes no LM call"""
    m, ctx = _model2(monkeypatch)
    reqs, Ub = _case2(6)
    zs, cross, vc = reqs[0], reqs[1], reqs[3]

    def run(rs, cols, seeds):
        ids = {}
        orig = ctx.lm_prefill

        def prefill(sess, tt, tl, ss, sl):
            ids["rows"] = len(tl)
            return orig(sess, tt, tl, ss, sl)
        ctx.lm_prefill = prefill
        try:
            # sample counts first (noise sized per request), then the real run
            _, st = m.tts_batch(rs, uniforms=Ub[:, cols], noise=torch.zeros(10 ** 6, 9), return_stats=True)
            noise = torch.cat([stream_noise(s, f * 480) for s, f in zip(seeds, st["mel_frames"])], 0)
            wavs, st = m.tts_batch(rs, uniforms=Ub[:, cols], noise=noise, return_stats=True)
        finally:
            ctx.lm_prefill = orig
        return wavs, st, ids.get("rows")

    w_lm, st_lm, rows_lm = run([zs, cross], [0, 1], [0, 1])
    w_mix, st_mix, rows_mix = run([zs, vc, cross], [0, 3, 1], [0, 3, 1])
    w_vc, st_vc, rows_vc = run([vc], [3], [3])
    assert rows_lm == 2 and rows_mix == 2 and rows_vc is None            # VC rows never reach the LM
    assert st_mix["tokens"] == [st_lm["tokens"][0], 23, st_lm["tokens"][1]]
    assert torch.equal(w_mix[0], w_lm[0]) and torch.equal(w_mix[2], w_lm[1])
    assert torch.equal(w_mix[1], w_vc[0])


def test_tts3_batch_mixed_kinds_equals_tts(monkeypatch):
    """CosyVoice3: the same six request kinds; a VC row keeps a run of 8 silent tokens (vc_job applies no silent-token rule)"""
    m = t3._model(monkeypatch)
    fake_mel_resample(m.ctx)
    text, ptext, ptok, U = cases.lm3_case()
    _, _, pfeat, emb = cases.flow_case(P=9)
    reqs = mixed_requests(ptext, ptok, pfeat[:, :18], emb, seed=79)
    src = reqs[3]["source_speech_token"].clone()
    src[0, 4:12] = t3.SILENT[0]
    reqs[3] = dict(reqs[3], source_speech_token=src)
    Ub = torch.rand(U.shape[0], 6, 2, generator=torch.Generator().manual_seed(80))
    alone = _alone(m, reqs, Ub, noise=False)
    m.ctx.resample_calls.clear()
    wavs, stats = m.tts_batch(reqs, uniforms=Ub, return_stats=True)
    _check(wavs, alone)
    assert stats["tokens"][3] == 23 and stats["tokens"][5] == 31
    assert len(m.ctx.resample_calls) == 1
    assert stats["mel_frames"][4] == int(stats["flow_frames"][4] / 0.8)


def test_tts_batch_refusals_come_before_any_work(monkeypatch):
    m, ctx = _model2(monkeypatch)
    reqs, Ub = _case2(6)
    for bad in (0.0, -1.0, float("nan")):
        ctx.calls.clear()
        with pytest.raises(ValueError):
            m.tts_batch([reqs[0], dict(reqs[3], speed=bad)], uniforms=Ub[:, :2])
        assert ctx.calls == []
    # a stretched length of 0: refused after the flow, before the stretch and the vocoder
    ctx.calls.clear()
    ctx.resample_calls.clear()
    with pytest.raises(ValueError):
        m.tts_batch([dict(reqs[3], speed=1e6)])
    assert ctx.resample_calls == [] and not [c for c in ctx.calls if c[0] == "hift"]


def test_stream_refusals(monkeypatch):
    m, _ = _model2(monkeypatch)
    reqs, Ub = _case2(6)
    with pytest.raises(ValueError):
        m.tts_stream_batch([reqs[0], dict(reqs[1], speed=0.8)])
    with pytest.raises(ValueError):
        m.tts_bistream_batch([dict(reqs[0], speed=1.25)])
    with pytest.raises(ValueError):
        m.tts_bistream_batch([dict(reqs[0], text=iter([reqs[0]["text"]])), reqs[3]])


def test_tts_stream_batch_with_vc_rows_equals_tts_stream(monkeypatch):
    """CosyVoice2: two LM rows and a VC row in one tts_stream_batch: each request gets tts(stream=True)'s chunks alone, and the VC
    row has finished before the LM generation ends (the LM holds back its last block until the VC row's last chunk is out)"""
    m, ctx = _model2(monkeypatch)
    m.max_token_text_ratio = 20.0
    (r0, r1), Ub = sb._case()
    vc = dict(source_speech_token=torch.randint(0, 6561, (1, 120), generator=torch.Generator().manual_seed(9), dtype=torch.int32),
              flow_prompt_speech_token=r0["flow_prompt_speech_token"], prompt_speech_feat=r0["prompt_speech_feat"],
              flow_embedding=r0["flow_embedding"])
    reqs = [r0, vc, r1]
    Ub3 = torch.stack([Ub[:, 0], torch.zeros_like(Ub[:, 0]), Ub[:, 1]], 1)
    fns = sb._noise_fns(3)
    singles = []
    for i, r in enumerate(reqs):
        m.uniforms_override, m.noise_fn, m.token_hop_len = Ub3[:, i:i + 1], sb._noise_fns(3)[i], 25
        try:
            singles.append([o["tts_speech"] for o in m.tts(**r, stream=True)])
        finally:
            m.uniforms_override, m.noise_fn, m.token_hop_len = None, None, 25
    vc_done, held = threading.Event(), {}
    orig = ctx.lm_decode

    def lm_decode(sess, n_steps, U, min_len, max_len, out_ids, out_count, done, want_live=True):
        live = orig(sess, n_steps, U, min_len, max_len, out_ids, out_count, done, want_live)
        if live == 0 and "waited" not in held:
            held["waited"] = vc_done.wait(60)
        return live
    ctx.lm_decode = lm_decode
    chunks = [[], [], []]
    try:
        for i, out in m.tts_stream_batch(reqs, uniforms=Ub3, noise_fns=fns):
            chunks[i].append(out["tts_speech"])
            if i == 1 and len(chunks[1]) == len(singles[1]):
                vc_done.set()
    finally:
        ctx.lm_decode = orig
    assert held.get("waited") is True
    assert len(singles[1]) == 3                       # two streaming chunks and the final call
    for i in range(3):
        assert [c.shape[1] for c in chunks[i]] == [c.shape[1] for c in singles[i]], i
        assert (torch.cat(chunks[i], 1) - torch.cat(singles[i], 1)).abs().max().item() < 1e-5, i
    assert sorted(m._free_slots) == [0, 1]


def test_tts_stream_batch_vc_only_runs_no_lm(monkeypatch):
    m, ctx = _model2(monkeypatch)
    reqs, _ = _case2(6)
    vc = dict(reqs[3], source_speech_token=torch.randint(0, 6561, (1, 60), generator=torch.Generator().manual_seed(3), dtype=torch.int32))
    m.noise_fn, m.token_hop_len = sb._noise_fns(1)[0], 25
    try:
        single = [o["tts_speech"] for o in m.tts(**vc, stream=True)]
    finally:
        m.noise_fn, m.token_hop_len = None, 25
    ctx.lm_prefill = lambda *a, **k: (_ for _ in ()).throw(AssertionError("no LM call for a batch of VC rows"))
    chunks = [o["tts_speech"] for _, o in m.tts_stream_batch([vc], noise_fns=sb._noise_fns(1))]
    assert [c.shape[1] for c in chunks] == [c.shape[1] for c in single] and len(chunks) == 2
    assert (torch.cat(chunks, 1) - torch.cat(single, 1)).abs().max().item() < 1e-5


def test_batcher_rejects_streaming_speed_at_submit():
    """submit_stream / submit_stream_pcm refuse speed != 1 and every submit refuses speed <= 0, in the caller's thread; the other
    requests are served as usual, and offline requests of every kind share a batch"""
    from cosyvoice_b200.batcher import TtsBatcher

    class Model:
        def __init__(self):
            self.seen = []

        def tts_batch(self, inputs):
            self.seen.append(inputs)
            return [torch.full((1, 3), float(r.get("speed", 1.0))) for r in inputs]

        def tts_stream_batch(self, inputs):
            for i, r in enumerate(inputs):
                yield i, {"tts_speech": torch.full((1, 2), float(r["text"]))}

    model = Model()
    with TtsBatcher(model, max_batch=8, max_wait_ms=300) as b:
        s1 = b.submit_stream(text=1)
        with pytest.raises(ValueError):
            b.submit_stream(text=2, speed=0.8)
        with pytest.raises(ValueError):
            b.submit_stream_pcm(text=3, speed=1.25)
        with pytest.raises(ValueError):
            b.submit(text=4, speed=0.0)
        s2 = b.submit_stream(text=5, speed=1.0)
        assert [float(c[0, 0]) for c in s1] == [1.0] and [float(c[0, 0]) for c in s2] == [5.0]
        f1 = b.submit(text=6, speed=0.8)
        f2 = b.submit(source_speech_token=torch.zeros(1, 4, dtype=torch.int32))
        f3 = b.submit(text=7)
        assert [float(f.result(5)[0, 0]) for f in (f1, f2, f3)] == pytest.approx([0.8, 1.0, 1.0])
    assert b.batches == [2, 3]
