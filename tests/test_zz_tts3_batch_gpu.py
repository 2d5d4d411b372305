"""GPU: CosyVoice3 batched offline synthesis - the float64 f0 predictor on the fp64 tensor cores (csrc/hift.cu f0_conv_dmma_kernel)
against the float64 oracle and bit-stable across batch composition and streaming prefixes, and B200CosyVoice3Model.tts_batch /
TtsBatcher against tts() per request and the reference's own offline waveform (tests/golden/stream3_tts.npz).

The file name sorts last so that a CUDA fault here cannot disturb the tests that share the process."""
import pytest
import torch

from gpu_util import maxdiff
from oracle import cases, dit, hift_causal as hc, lm, weights
from test_zz_hift3_gpu import model as vocoder

pytestmark = pytest.mark.gpu
_m = {}


def _hsd():
    return weights.synth_state_dict(hc.param_shapes(), 1986, hc.SYNTH_GAINS)


def _noise(T, seed=21):
    g = torch.Generator().manual_seed(seed)
    rand_ini = torch.rand(1, 9, generator=g)
    rand_ini[:, 0] = 0
    return rand_ini, torch.rand(T * 480, 9, generator=g)


def _f0(c, mel_tm, lens, finalize):
    _, f0, _ = c.hift3_inference(mel_tm, lens, finalize=finalize)
    torch.cuda.synchronize()
    return f0.cpu()


@pytest.mark.parametrize("finalize", [True, False])
def test_f0_dmma_matches_float64_oracle(finalize):
    """f0 against oracle.hift_causal.f0_predict (float64 throughout).  Both fold the weight norm in fp32, in different summation
    orders, so their weights differ by a few fp32 ulps per output channel; the bound is 4x the change of the oracle's f0 when its
    fold is done in float64 instead (the size of that rounding's effect) plus the float32 rounding of the written f0."""
    sd = _hsd()
    sd64 = {k: v.double() for k, v in sd.items()}
    c = vocoder("fp32")
    rand_ini, noise = _noise(3000)
    c.hift3_set_noise(rand_ini, noise)
    g = torch.Generator().manual_seed(3)
    for T in (1, 9, 57, 500, 3000):
        if not finalize and T < 9:
            continue                                           # a streaming call needs at least 9 frames
        mel = torch.randn(1, 80, T, generator=g) * 2 - 5
        got = _f0(c, mel[0].t().contiguous(), [T], finalize)
        ref = hc.f0_predict(sd, mel, finalize)[0]
        fold = (ref.double() - hc.f0_predict(sd64, mel, finalize)[0].double()).abs().max().item()
        bound = 4 * fold + 2.0 ** -22 * ref.abs().max().item()
        d = (got.double() - ref.double()).abs().max().item()
        print(f"[f0 T={T} finalize={finalize}] max|f0 - oracle| {d:.3g} (bound {bound:.3g}, fp32-fold effect {fold:.3g}, max f0 {ref.abs().max():.3g})")
        assert got.shape == ref.shape
        assert d <= bound, (T, d, bound)
        torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-2)


def test_f0_bit_identical_across_batches_prefixes_and_runs():
    c = vocoder("fp32")
    rand_ini, noise = _noise(3000)
    c.hift3_set_noise(rand_ini, noise)
    g = torch.Generator().manual_seed(4)
    # ~40 utterances of mixed lengths: 128-row tiles straddle sequences and the gap rows between them
    lens = [int(x) for x in torch.randint(1, 160, (40,), generator=g)] + [1, 2, 3, 300]
    mels = [torch.randn(T, 80, generator=g) * 2 - 5 for T in lens]
    batch = _f0(c, torch.cat(mels, 0), lens, True)
    o = 0
    for T, mel in zip(lens, mels):
        assert torch.equal(batch[o:o + T], _f0(c, mel, [T], True)), T
        o += T
    assert torch.equal(batch, _f0(c, torch.cat(mels, 0), lens, True))          # two runs
    # a streaming call on mel[:T] gives the first T-3 f0 of the offline call on the whole mel
    mel = torch.randn(700, 80, generator=g) * 2 - 5
    full = _f0(c, mel, [700], True)
    for T in (9, 57, 131, 500, 700):
        assert torch.equal(_f0(c, mel[:T].contiguous(), [T], False), full[:T - 3]), T
    # ... also when the prefixes are batched
    pre = [9, 130, 257]
    got = _f0(c, torch.cat([mel[:T] for T in pre], 0), pre, False)
    assert torch.equal(got, torch.cat([full[:T - 3] for T in pre]))


def model(precision="fp32"):
    if precision not in _m:
        from cosyvoice_b200.model3 import B200CosyVoice3Model
        m = B200CosyVoice3Model(precision=precision, device=0, workspace_gb=4.0)
        _, rand_ini, sine_noise = cases.hift_causal_case(T=400)
        m.load_state_dicts(lm.synth_state_dict3(2), weights.synth_state_dict(dit.flow_param_shapes(2), 1986, dit.SYNTH_GAINS),
                           _hsd(), rand_ini=rand_ini, sine_noise=sine_noise)
        _m[precision] = m
    return _m[precision]


def requests():
    """request 0 = the golden request of test_zz_model3_gpu.py; two more with shorter texts.  uniforms [n, 3, 2]: column i is
    request i's draws (column 0 the golden ones)."""
    text, ptext, ptok, U = cases.lm3_case()
    _, _, pfeat, emb = cases.flow_case(P=9)
    base = dict(text=text, prompt_text=ptext, llm_prompt_speech_token=ptok, flow_prompt_speech_token=ptok, prompt_speech_feat=pfeat[:, :18],
                flow_embedding=emb)
    g = torch.Generator().manual_seed(321)
    reqs = [base]
    for n in (5, 3):
        r = dict(base)
        r["text"] = torch.randint(0, 151643, (1, n), generator=g, dtype=torch.int32)
        reqs.append(r)
    Ub = torch.rand(U.shape[0], len(reqs), 2, generator=g)
    Ub[:, 0] = U
    return reqs, Ub


def _alone(m, reqs, Ub):
    out = []
    for i, r in enumerate(reqs):
        m.uniforms_override = Ub[:, i:i + 1]
        out.append(torch.cat([o["tts_speech"] for o in m.tts(llm_embedding=r["flow_embedding"], stream=False, **r)], 1))
    return out


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_tts3_batch_equals_tts(precision, golden):
    """tts_batch of three requests == each request's tts() alone.  fp32: same length, within 1e-3 (printed; the vocoder and flow
    compute every row independently of the batch, so the difference is expected to be zero).  bf16: printed.  Request 0 also
    matches the reference's own offline waveform to test_tts3_matches_reference_model's bounds."""
    m = model(precision)
    reqs, Ub = requests()
    try:
        alone = _alone(m, reqs, Ub)
        m.uniforms_override = None
        wavs, stats = m.tts_batch(reqs, uniforms=Ub, return_stats=True)
    finally:
        m.uniforms_override = None
    print(f"[cv3 tts_batch {precision}] tokens {stats['tokens']}, mel frames {stats['mel_frames']}, "
          f"lm {stats['lm_ms']:.1f} ms, flow {stats['flow_ms']:.1f} ms, vocoder {stats['hift_ms']:.1f} ms")
    for i, (w, a) in enumerate(zip(wavs, alone)):
        assert torch.isfinite(w).all()
        if w.shape == a.shape:
            print(f"[cv3 tts_batch {precision}] request {i}: {w.shape[1]} samples, max|batch - tts()| {maxdiff(w, a):.3g}, "
                  f"bit-identical {torch.equal(w, a)}")
        else:
            print(f"[cv3 tts_batch {precision}] request {i}: batch {w.shape[1]} samples, tts() {a.shape[1]} samples")
        if precision == "fp32":
            assert w.shape == a.shape, (i, w.shape, a.shape)
            assert maxdiff(w, a) < 1e-3, (i, maxdiff(w, a))
    if precision == "fp32":
        ref = torch.from_numpy(golden("stream3_tts")["offline_wav"])
        w = wavs[0]
        assert w.shape == ref.shape
        d_head = maxdiff(w[:, :24000], ref[:, :24000])
        rel = ((w - ref).norm() / ref.norm()).item()
        print(f"[cv3 tts_batch fp32] request 0 vs reference: max|d| first second {d_head:.3g}, relative L2 {rel:.3g}")
        assert d_head < 5e-3 and rel < 0.05, (d_head, rel)


def test_batcher_over_cosyvoice3_tts_batch():
    """TtsBatcher over B200CosyVoice3Model: requests submitted while the worker is busy are served as one batch and get tts_batch's
    waveforms, as float tensors and as int16 PCM bytes"""
    from cosyvoice_b200.batcher import TtsBatcher, pcm16
    m = model("fp32")
    reqs, Ub = requests()
    reqs, Ub = reqs[:2], Ub[:, :2].contiguous()
    m.uniforms_override = Ub
    try:
        want = m.tts_batch(reqs)
        with TtsBatcher(m, max_batch=2, max_wait_ms=2000) as b:
            f1, f2 = b.submit(**reqs[0]), b.submit_pcm(**reqs[1])
            w1, p2 = f1.result(timeout=120), f2.result(timeout=120)
        assert b.batches == [2]
    finally:
        m.uniforms_override = None
    assert torch.equal(w1, want[0]) and p2 == pcm16(want[1])
