"""GPU: the host-side mirror of cosyvoice/cli/model.py:245-394 (B200CosyVoice2Model.tts / token2wav / tts_batch) against
outputs of the reference CosyVoice2Model.tts itself (tests/golden/stream_tts.npz: offline and streaming runs on small
modules with the RNG streams injected) - chunk schedule, cache/fade bookkeeping and waveform."""
import numpy as np
import pytest
import torch

from gpu_util import maxdiff
from oracle import cases, flow, hift, lm, weights
from oracle.make_golden import stream_noise

pytestmark = pytest.mark.gpu
_m = {}


def model():
    if "m" not in _m:
        from cosyvoice_b200.model import B200CosyVoice2Model
        NL, kw = 2, dict(enc_blocks=2, enc_up_blocks=1, num_mid_blocks=2, n_blocks=2)
        m = B200CosyVoice2Model(precision="fp32", device=0, workspace_gb=4.0)
        m.load_state_dicts(lm.synth_state_dict(NL), weights.synth_state_dict(flow.param_shapes(flow.FlowCfg(**kw)), 1986, flow.SYNTH_GAINS),
                           weights.synth_state_dict(hift.param_shapes(), 1986, hift.SYNTH_GAINS))
        _m["m"] = m
    return _m["m"]


def request():
    text, ptext, ptok, U = cases.lm_case()
    _, _, pfeat, emb = cases.flow_case(P=9)
    return dict(text=text, flow_embedding=emb, llm_embedding=emb, prompt_text=ptext, llm_prompt_speech_token=ptok,
                flow_prompt_speech_token=ptok, prompt_speech_feat=pfeat[:, :18]), U


def hooks(m, U):
    st = {"k": 0}

    def noise_fn(n):
        z = stream_noise(st["k"], n).to(m.device)
        st["k"] += 1
        return z
    m.uniforms_override = U[:, None, :]
    m.noise_fn = noise_fn
    m.token_hop_len = 25


@pytest.mark.parametrize("stream", [False, True])
def test_tts_matches_reference_model(stream, golden):
    g = golden("stream_tts")
    m = model()
    req, U = request()
    hooks(m, U)
    try:
        chunks = [o["tts_speech"] for o in m.tts(**req, stream=stream)]
    finally:
        m.uniforms_override, m.noise_fn = None, None
    key = "stream" if stream else "offline"
    assert [c.shape[1] for c in chunks] == g[key + "_lens"].tolist()          # chunk schedule: bit-exact bookkeeping
    assert all(c.device.type == "cpu" and c.dtype == torch.float32 and c.shape[0] == 1 for c in chunks)
    wav = torch.cat(chunks, 1)
    ref = torch.from_numpy(g[key + "_wav"])
    # The excitation phase is 2*pi*480*cumsum(f0/sr), so fp32 summation-order differences in the f0 predictor grow along the
    # utterance (DESIGN.md §4): tight bound on the first second, looser on the rest.
    d_head = maxdiff(wav[:, :24000], ref[:, :24000])
    rel = ((wav - ref).norm() / ref.norm()).item()
    print(f"[{key}] max|d| first second {d_head:.3g}, relative L2 over {wav.shape[1]} samples {rel:.3g}, max|d| {maxdiff(wav, ref):.3g}")
    assert d_head < 5e-3, d_head
    assert rel < 0.05, rel
    if stream:
        assert m.token_hop_len == 100        # the reference leaves the doubled hop on the instance (cli/model.py:359-360)


def test_tts_batch_equals_single_requests(golden):
    g = golden("stream_tts")
    m = model()
    req, U = request()
    req2 = dict(req)
    g2 = torch.Generator().manual_seed(123)
    req2["text"] = torch.randint(0, 151643, (1, 5), generator=g2, dtype=torch.int32)
    st = {"k": 0}
    n1 = 140 * 960
    noise1 = stream_noise(0, n1)
    Ub = torch.rand(141, 2, 2, generator=g2)
    Ub[:, 0] = U[:141]
    ids = m.lm_generate([req["text"], req2["text"]], [req["prompt_text"]] * 2, [req["llm_prompt_speech_token"]] * 2, uniforms=Ub)
    n2 = len(ids[1]) * 960
    noise = torch.cat([noise1, torch.randn(n2, 9, generator=g2)], 0)
    wavs = m.tts_batch([req, req2], uniforms=Ub, noise=noise)
    assert wavs[0].shape[1] == n1 and wavs[1].shape[1] == n2
    ref = torch.from_numpy(g["offline_wav"])
    assert maxdiff(wavs[0][:, :24000], ref[:, :24000]) < 5e-3
    assert ((wavs[0] - ref).norm() / ref.norm()).item() < 0.05


def test_tts_with_text_generator_bistream(golden):
    """cli/model.py:113-123 + llm.py:551-661: `text` given as a generator -> the LM thread runs the text-streaming decode while
    the main thread streams audio chunks.  The speech ids equal the reference's (golden from Qwen2LM.inference_bistream), so the
    audio length is 960 samples per id and the chunk schedule is the deterministic hop 25 -> 50 -> 100 one."""
    from cosyvoice_b200.model import B200CosyVoice2Model
    g = golden("lm_bistream_l2")
    chunks, ptext, ptok, U = cases.bistream_case()
    kw = dict(enc_blocks=2, enc_up_blocks=1, num_mid_blocks=2, n_blocks=2)
    m = B200CosyVoice2Model(precision="fp32", device=0, workspace_gb=4.0)
    m.load_state_dicts(lm.bistream_state_dict(2), weights.synth_state_dict(flow.param_shapes(flow.FlowCfg(**kw)), 1986, flow.SYNTH_GAINS),
                       weights.synth_state_dict(hift.param_shapes(), 1986, hift.SYNTH_GAINS))
    _, _, pfeat, emb = cases.flow_case(P=9)
    ftok = ptok[:, :9]
    m.uniforms_override = U[:, None, :]
    m.token_hop_len = 25
    try:
        outs = [o["tts_speech"] for o in m.tts(text=iter(chunks), flow_embedding=emb, llm_embedding=emb, prompt_text=ptext,
                                               llm_prompt_speech_token=ptok, flow_prompt_speech_token=ftok,
                                               prompt_speech_feat=pfeat[:, :18], stream=True)]
    finally:
        m.uniforms_override = None
    n_ids = len(g["ids"])
    assert sum(o.shape[1] for o in outs) == n_ids * 960
    assert len(outs) >= 4 and all(torch.isfinite(o).all() for o in outs)
    # first chunk: hop 25 + pad to a multiple of 25 of the 9 prompt tokens (cli/model.py:347-350) = 41 tokens minus the 8-frame
    # mel cache kept back (3840 samples)
    assert outs[0].shape[1] == 41 * 960 - 3840


def test_overlapping_tts_requests_do_not_share_lm_sessions(golden):
    """The reference serves tts() from one thread per request with per-request state keyed by uuid (cli/model.py:334-337).  Two
    overlapping requests of the same shape must each own an LM session (KV cache + decode graph) from prefill to the last token:
    run two tts() calls from two threads at once and require both to reproduce the reference's audio.  (Round 1 cached sessions
    by shape, so the second prefill overwrote the first request's KV cache mid-decode.)"""
    import threading
    g = golden("stream_tts")
    m = model()
    req, U = request()
    m.uniforms_override = U[:, None, :]
    n = 140 * 960
    m.noise_fn = lambda k: stream_noise(0, n).to(m.device) if k == n else torch.randn(k, 9, device=m.device)
    outs, errs = {}, []

    def run(i):
        try:
            outs[i] = torch.cat([o["tts_speech"] for o in m.tts(**req, stream=False)], 1)
        except Exception as e:              # noqa: BLE001
            errs.append(e)
    try:
        ts = [threading.Thread(target=run, args=(i,)) for i in range(2)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
    finally:
        m.uniforms_override, m.noise_fn = None, None
    assert not errs, errs
    ref = torch.from_numpy(g["offline_wav"])
    for i in range(2):
        assert outs[i].shape == ref.shape
        assert maxdiff(outs[i][:, :24000], ref[:, :24000]) < 5e-3
    # the idle pool holds both sessions now and stays bounded
    assert sum(len(v) for v in m._free_sessions.values()) >= 2
    assert len(m._session_lru) <= m.max_idle_sessions


def test_batcher_over_tts_batch(golden):
    """cosyvoice_b200.batcher.TtsBatcher over the real model: requests submitted while the worker is busy are served as ragged batches
    and every request gets the waveform tts_batch gives for that batch (first request = the reference's offline waveform), as float
    tensors and as the servers' int16 PCM bytes."""
    from cosyvoice_b200.batcher import TtsBatcher, pcm16
    g = golden("stream_tts")
    m = model()
    req, U = request()
    req2 = dict(req)
    g2 = torch.Generator().manual_seed(123)
    req2["text"] = torch.randint(0, 151643, (1, 5), generator=g2, dtype=torch.int32)
    Ub = torch.rand(141, 2, 2, generator=g2)
    Ub[:, 0] = U[:141]
    m.uniforms_override = Ub
    m.noise_fn = lambda n: stream_noise(0, n).to(m.device)
    try:
        want = m.tts_batch([req, req2])
        with TtsBatcher(m, max_batch=2, max_wait_ms=2000) as b:
            f1, f2 = b.submit(**req), b.submit_pcm(**req2)
            w1, p2 = f1.result(timeout=120), f2.result(timeout=120)
        assert b.batches == [2]
    finally:
        m.uniforms_override, m.noise_fn = None, None
    assert torch.equal(w1, want[0]) and p2 == pcm16(want[1])
    ref = torch.from_numpy(g["offline_wav"])
    assert w1.shape == ref.shape and maxdiff(w1[:, :24000], ref[:, :24000]) < 5e-3
