"""GPU: CosyVoice3 batched streaming - the causal vocoder with a finalize flag per utterance (cvk_hift3_inference_rows) bit for
bit against cvk_hift3_inference one utterance at a time, and B200CosyVoice3Model.tts_stream_batch / tts_bistream_batch / TtsBatcher
against tts(stream=True) per request and the reference's own streaming waveform (tests/golden/stream3_tts.npz).

The file name sorts last so that a CUDA fault here cannot disturb the tests that share the process."""
import pytest
import torch

from gpu_util import maxdiff
from oracle import cases, dit, hift_causal as hc, lm, weights
from test_zz_hift3_gpu import model as vocoder
from test_zz_tts3_batch_gpu import _noise, model as small_model, requests

pytestmark = pytest.mark.gpu

LENS = [9, 3000, 10, 57, 400, 9, 3000]
FLAGS = [False, True, False, True, False, True, False]


def _mels(lens, seed=8):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(T, 80, generator=g) * 2 - 5 for T in lens]


def _cpu(*ts):
    torch.cuda.synchronize()
    return [t.cpu() for t in ts]


def _sizes(T, fin):
    return (480 * T, T, 480 * T) if fin else (480 * (T - 8), T - 3, 480 * (T - 3))


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_mixed_vocoder_call_is_each_utterance_alone(precision):
    """one call over 9 .. 3000 frames with mixed flags: every utterance's wav / f0 / source bit-identical to cvk_hift3_inference
    on it alone with its own flag; with all flags equal, bit-identical to cvk_hift3_inference on the whole batch"""
    c = vocoder(precision)
    rand_ini, noise = _noise(3000)
    c.hift3_set_noise(rand_ini, noise)
    mels = _mels(LENS)
    n0 = c.launch_count()
    got = _cpu(*c.hift3_inference_rows(torch.cat(mels, 0), LENS, FLAGS))
    n_mixed = c.launch_count() - n0
    offs = [0, 0, 0]
    for T, fin, mel in zip(LENS, FLAGS, mels):
        alone = _cpu(*c.hift3_inference(mel, [T], finalize=fin))
        for k, (a, n) in enumerate(zip(alone, _sizes(T, fin))):
            assert a.numel() == n
            assert torch.equal(got[k][offs[k]:offs[k] + n], a), (precision, T, fin, ("wav", "f0", "source")[k])
            offs[k] += n
    assert offs == [g.numel() for g in got]
    for fin in (True, False):
        n0 = c.launch_count()
        whole = _cpu(*c.hift3_inference(torch.cat(mels, 0), LENS, finalize=fin))
        if not fin:
            assert c.launch_count() - n0 == n_mixed             # a mixed call launches what a streaming call of its size does
        rows = _cpu(*c.hift3_inference_rows(torch.cat(mels, 0), LENS, [fin] * len(LENS)))
        assert all(torch.equal(a, b) for a, b in zip(whole, rows)), (precision, fin)
    print(f"[hift3 rows {precision}] {len(LENS)} utterances ({sum(LENS)} frames, mixed flags): bit-identical alone; {n_mixed} launches")


def test_streaming_utterance_of_8_frames_is_refused():
    from cosyvoice_b200.cvk import CvkError
    c = vocoder("fp32")
    rand_ini, noise = _noise(3000)
    c.hift3_set_noise(rand_ini, noise)
    mels = _mels([57, 8])
    before = _cpu(*c.hift3_inference(mels[0], [57], finalize=False))
    with pytest.raises(CvkError):
        c.hift3_inference_rows(torch.cat(mels, 0), [57, 8], [False, False])
    with pytest.raises(CvkError):
        c.hift3_inference_rows(torch.cat(mels, 0), [57, 3001], [True, True])          # longer than the stored noise
    after = _cpu(*c.hift3_inference_rows(torch.cat(mels, 0), [57, 8], [False, True]))  # a final 8-frame utterance is fine
    assert torch.equal(after[0][:480 * 49], before[0]) and after[0].numel() == 480 * (49 + 8)


# ---------------------------------------------------------------------------------------------------------- the model
def _model(precision):
    m = small_model(precision)
    m.stream_batch_slots, m.stream_cache_frames = 4, 768
    m.stream_pool_headroom = 1 << 30              # the test process holds the contexts of the earlier GPU modules too
    return m


def _collect(gen, B):
    chunks = [[] for _ in range(B)]
    for i, out in gen:
        chunks[i].append(out["tts_speech"])
    return chunks


_singles = {}


def _alone(m, precision, reqs, Ub):
    if precision not in _singles:
        out = []
        for i, r in enumerate(reqs):
            m.uniforms_override, m.token_hop_len = Ub[:, i:i + 1], 25
            try:
                out.append([o["tts_speech"] for o in m.tts(llm_embedding=r["flow_embedding"], stream=True, **r)])
            finally:
                m.uniforms_override, m.token_hop_len = None, 25
        _singles[precision] = out
    return _singles[precision]


BOUND = {"fp32": 1e-4, "bf16": 1e-3}


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_tts_stream_batch3_equals_tts(precision, golden):
    """three requests in one tts_stream_batch == each request's tts(stream=True) alone: same chunk lengths, waveforms within 1e-4
    in fp32 (the bound of the CosyVoice2 batched test) and 1e-3 in bf16.  Measured on an H100: 0 in both, i.e. bit-identical -
    the vocoder is bit-identical per utterance by construction and the slot-batched DiT computes every row as a one-slot session
    does.  Request 0 also matches the reference's own streaming waveform on its first second."""
    m = _model(precision)
    reqs, Ub = requests()
    want = _alone(m, precision, reqs, Ub)
    launches = m.ctx.launch_count()
    chunks = _collect(m.tts_stream_batch(reqs, uniforms=Ub), 3)
    print(f"[cv3 tts_stream_batch {precision}] {m.ctx.launch_count() - launches} launches, chunks {[[c.shape[1] for c in ch] for ch in chunks]}")
    assert m.token_hop_len == 25 and len(m._free_slots) == m.stream_slots > 0
    for i in range(3):
        assert [c.shape[1] for c in chunks[i]] == [c.shape[1] for c in want[i]], i
        w = torch.cat(chunks[i], 1)
        assert torch.isfinite(w).all()
        d = maxdiff(w, torch.cat(want[i], 1))
        print(f"[cv3 tts_stream_batch {precision}] request {i}: max|batch - tts(stream=True)| {d:.3g}")
        assert d <= BOUND[precision], (i, d)
    if precision == "fp32":
        g = golden("stream3_tts")
        assert [c.shape[1] for c in chunks[0]] == g["stream_lens"].tolist()
        d_head = maxdiff(torch.cat(chunks[0], 1)[:, :24000], torch.from_numpy(g["stream_wav"])[:, :24000])
        print(f"[cv3 tts_stream_batch fp32] request 0 vs reference: max|d| first second {d_head:.3g}")
        assert d_head < 5e-3


def test_closing_the_generator_returns_every_slot():
    m = _model("fp32")
    reqs, Ub = requests()
    gen = m.tts_stream_batch(reqs, uniforms=Ub)
    _, out = next(gen)
    assert out["tts_speech"].shape[1] > 0 and len(m._free_slots) < m.stream_slots       # the first chunk's request holds a slot
    gen.close()
    assert sorted(m._free_slots) == list(range(m.stream_slots))


def test_tts_bistream3_batch_equals_single_requests(golden):
    """config #4's call pattern batched: text generators, fp32.  The LM ids equal the reference's (lm3_bistream_l2), and each
    request's chunks equal tts(text=<generator>, stream=True) alone"""
    from cosyvoice_b200.model3 import B200CosyVoice3Model
    g = golden("lm3_bistream_l2")
    chunks, ptext, ptok, U = cases.bistream3_case()
    # the earlier GPU modules of the process keep their contexts: hand torch's cached blocks back to the driver and keep the
    # workspace small, so that this model's context fits beside them
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    print(f"[cv3 tts_bistream_batch] device memory free before the model: {free / 2**30:.1f} of {total / 2**30:.1f} GiB")
    m = B200CosyVoice3Model(precision="fp32", device=0, workspace_gb=1.0)
    _, rand_ini, sine_noise = cases.hift_causal_case(T=400)
    m.load_state_dicts(lm.bistream_state_dict3(2), weights.synth_state_dict(dit.flow_param_shapes(2), 1986, dit.SYNTH_GAINS),
                       weights.synth_state_dict(hc.param_shapes(), 1986, hc.SYNTH_GAINS), rand_ini=rand_ini, sine_noise=sine_noise)
    m.stream_batch_slots, m.stream_cache_frames, m.stream_pool_headroom = 4, 768, 1 << 30
    m.silent_tokens = []          # the synthetic ids are uniform over the codebook: count every id
    m.bistream_max_tokens = 130
    try:
        _, _, pfeat, emb = cases.flow_case(P=9)
        flat = torch.cat([c.reshape(-1) for c in chunks])
        texts = [chunks, [flat[i:i + 1].reshape(1, -1) for i in range(flat.numel())], [flat[i:i + 7].reshape(1, -1) for i in range(0, flat.numel(), 7)]]
        base = dict(flow_embedding=emb, llm_embedding=emb, prompt_text=ptext, llm_prompt_speech_token=ptok, flow_prompt_speech_token=ptok[:, :9],
                    prompt_speech_feat=pfeat[:, :18])
        Ub = torch.stack([U] * 3, 1)
        got = _collect(m.tts_bistream_batch([dict(base, text=iter(t)) for t in texts], uniforms=Ub), 3)
        assert m.token_hop_len == 25 and len(m._free_slots) == m.stream_slots
        for i, t in enumerate(texts):
            m.uniforms_override, m.token_hop_len = U[:, None, :], 25
            try:
                single = [o["tts_speech"] for o in m.tts(**dict(base, text=iter(t)), stream=True)]
            finally:
                m.uniforms_override, m.token_hop_len = None, 25
            d = maxdiff(torch.cat(got[i], 1), torch.cat(single, 1))
            print(f"[cv3 tts_bistream_batch fp32] request {i}: chunks {[c.shape[1] for c in got[i]]}, max|batch - tts()| {d:.3g}")
            assert [c.shape[1] for c in got[i]] == [c.shape[1] for c in single], i
            assert sum(c.shape[1] for c in got[i]) == len(g["ids"]) * 960      # every id of the reference's decode
            assert d <= 1e-4, (i, d)
    finally:
        torch.cuda.synchronize()
        for fs in m._idle_flow_streams + ([m._slot_pool] if m._slot_pool else []):
            m.ctx.flow_stream_destroy(fs)
        m._idle_flow_streams, m._slot_pool = [], None
        for sessions in m._free_sessions.values():
            for sess in sessions:
                m.ctx.lm_session_destroy(sess)
        m._free_sessions.clear()
        m.ctx.close()


def test_batcher_streams_cosyvoice3_requests():
    """TtsBatcher.submit_stream / submit_stream_pcm on a CosyVoice3 model: one streaming batch with tts_stream_batch's chunks"""
    from cosyvoice_b200.batcher import TtsBatcher, pcm16
    m = _model("fp32")
    reqs, Ub = requests()
    reqs, Ub = reqs[:2], Ub[:, :2].contiguous()
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
