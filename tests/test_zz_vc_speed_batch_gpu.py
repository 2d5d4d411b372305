"""GPU: the `speed` time-stretch kernel (cvk_mel_resample, csrc/mel.cu) against F.interpolate(mode="linear") - bit for bit on the
same device, within 2 fp32 ulps on the CPU - and every tts() request kind in the batched paths: tts_batch over zero-shot,
cross-lingual, instruct2-shaped, voice-conversion and speed-changed requests against each request's tts() alone (both models),
tts_stream_batch with voice-conversion rows against tts(source_speech_token=..., stream=True), tts() with speed != 1 against the
torch expression it replaces, and TtsBatcher over a mixed offline batch.

The file name sorts last so that a CUDA fault here cannot disturb the tests that share the process."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gpu_util import maxdiff
from oracle import cases, flow, hift, lm, weights
from oracle.make_golden import stream_noise
from test_vc_speed_batch_cpu import mixed_requests

pytestmark = pytest.mark.gpu

SPEEDS = (0.5, 0.75, 0.9, 0.999, 1.1, 1.25, 1.5, 2.0)
LENS = (1, 2, 7, 500, 3000)
_c = {}


@pytest.fixture(scope="module", autouse=True)
def _release_contexts():
    yield
    for k in list(_c):
        obj = _c.pop(k)
        if hasattr(obj, "ctx"):
            for fs in obj._idle_flow_streams + ([obj._slot_pool] if obj._slot_pool else []):
                obj.ctx.flow_stream_destroy(fs)
            obj._idle_flow_streams, obj._slot_pool = [], None
            obj = obj.ctx
        obj.close()
    torch.cuda.empty_cache()


def _ctx():
    from cosyvoice_b200 import cvk
    if "ctx" not in _c:
        _c["ctx"] = cvk.Context(0, "fp32", workspace_gb=0.25)
    return _c["ctx"]


def _stretch_cases():
    """(T, speed, T', mel [T, 80]) for every speed and length whose stretched length is not 0; log-mel-like values"""
    g = torch.Generator().manual_seed(31)
    out = []
    for T in LENS:
        for s in SPEEDS:
            Tn = int(T / s)
            if Tn == 0:
                continue                      # the ValueError case
            out.append((T, s, Tn, torch.randn(T, 80, generator=g) * 3 - 5))
    return out


def _interp(x, Tn):
    return F.interpolate(x.t()[None], size=Tn, mode="linear")[0].t()


# ------------------------------------------------------------------------------------------------ kernel
def test_mel_resample_bit_identical_to_torch_on_device():
    c = _ctx()
    cs = _stretch_cases()
    assert any(T == Tn for T, _, Tn, _ in cs) and any(Tn == 1 and T > 1 for T, _, Tn, _ in cs)       # copy and single-frame cases
    for T, s, Tn, x in cs:
        xd = x.cuda()
        ref = _interp(xd, Tn)
        got = c.mel_resample(xd, [T], [Tn])
        torch.cuda.synchronize()
        assert got.shape == (Tn, 80)
        assert torch.equal(got, ref), (T, s, Tn, maxdiff(got.cpu(), ref.cpu()))
    # one ragged call over every case (mixed speeds) == each sequence alone
    lens, out_lens = [T for T, _, _, _ in cs], [Tn for _, _, Tn, _ in cs]
    xs = torch.cat([x for _, _, _, x in cs]).cuda()
    got = c.mel_resample(xs, lens, out_lens)
    ref = torch.cat([_interp(x.cuda(), Tn) for _, _, Tn, x in cs])
    torch.cuda.synchronize()
    assert torch.equal(got, ref)


def test_mel_resample_within_two_ulps_of_torch_on_cpu():
    c = _ctx()
    worst = 0.0
    for T, s, Tn, x in _stretch_cases():
        ref = _interp(x, Tn).numpy()
        got = c.mel_resample(x.cuda(), [T], [Tn]).cpu().numpy()
        ulp = float(np.spacing(np.float32(np.abs(ref).max())))
        d = float(np.abs(got - ref).max())
        worst = max(worst, d / ulp)
        assert d <= 2 * ulp, (T, s, Tn, d, ulp)
    print(f"[mel_resample] worst difference from torch on the CPU: {worst:.2f} ulps of the output magnitude")


def test_mel_resample_refuses_empty_lengths():
    from cosyvoice_b200.cvk import _ints, _ptr, _stream
    c = _ctx()
    x = torch.zeros(4, 80, device="cuda")
    with pytest.raises(ValueError):
        c.mel_resample(x, [4], [0])
    out = torch.empty(4, 80, device="cuda")
    assert c.lib.cvk_mel_resample(c.h, _ptr(x), _ints([4]), _ints([0]), 1, _ptr(out), _stream()) == -1
    assert c.lib.cvk_mel_resample(c.h, _ptr(x), _ints([0]), _ints([4]), 1, _ptr(out), _stream()) == -1


# ------------------------------------------------------------------------------------------------ models
def _model2(precision):
    """the small CosyVoice2 model of tests/test_model_gpu.py in fp32 (the process already holds it when the whole suite runs, and
    device memory is short by then), an own one with a small workspace in bf16"""
    if precision == "fp32":
        from test_model_gpu import model
        m = model()
    else:
        if "cv2bf16" not in _c:
            from cosyvoice_b200.model import B200CosyVoice2Model
            torch.cuda.empty_cache()
            kw = dict(enc_blocks=2, enc_up_blocks=1, num_mid_blocks=2, n_blocks=2)
            m = B200CosyVoice2Model(precision="bf16", device=0, workspace_gb=1.0)
            m.load_state_dicts(lm.synth_state_dict(2), weights.synth_state_dict(flow.param_shapes(flow.FlowCfg(**kw)), 1986, flow.SYNTH_GAINS),
                               weights.synth_state_dict(hift.param_shapes(), 1986, hift.SYNTH_GAINS))
            _c["cv2bf16"] = m
        m = _c["cv2bf16"]
    if m.stream_slots is None:
        m.stream_batch_slots, m.stream_cache_frames, m.stream_pool_headroom = 4, 1024, 1 << 30
    return m


def _model3(precision):
    """the small CosyVoice3 models of tests/test_zz_tts3_batch_gpu.py"""
    from test_zz_tts3_batch_gpu import model
    m = model(precision)
    if m.stream_slots is None:
        m.stream_batch_slots, m.stream_cache_frames, m.stream_pool_headroom = 4, 768, 1 << 30
    return m


def _requests(cv3):
    text, ptext, ptok, U = cases.lm3_case() if cv3 else cases.lm_case()
    _, _, pfeat, emb = cases.flow_case(P=9)
    reqs = mixed_requests(ptext, ptok, pfeat[:, :18], emb, seed=81)
    Ub = torch.rand(U.shape[0], len(reqs), 2, generator=torch.Generator().manual_seed(82))
    return reqs, Ub


def _alone(m, reqs, Ub, noise):
    out = []
    for i, r in enumerate(reqs):
        m.uniforms_override = Ub[:, i:i + 1]
        m.noise_fn = (lambda n, i=i: stream_noise(i, n).to(m.device)) if noise else None
        try:
            out.append(torch.cat([o["tts_speech"] for o in m.tts(stream=False, **r)], 1))
        finally:
            m.uniforms_override, m.noise_fn = None, None
    return out


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("cv3", [False, True], ids=["cv2", "cv3"])
def test_tts_batch_mixed_kinds_equals_tts(cv3, precision):
    """one tts_batch over the six request kinds == each request's tts() alone.  fp32: same lengths, within 1e-4 per sample
    (CosyVoice2, the bound of the batched streaming test) / 1e-3 (CosyVoice3, the bound of its batched offline test); bf16:
    printed, as in those tests."""
    m = _model3(precision) if cv3 else _model2(precision)
    reqs, Ub = _requests(cv3)
    alone = _alone(m, reqs, Ub, noise=not cv3)
    noise = None if cv3 else torch.cat([stream_noise(i, a.shape[1]) for i, a in enumerate(alone)], 0)
    launches = m.ctx.launch_count()
    wavs, stats = m.tts_batch(reqs, uniforms=Ub, noise=noise, return_stats=True)
    tag = f"[{'cv3' if cv3 else 'cv2'} mixed tts_batch {precision}]"
    print(f"{tag} {m.ctx.launch_count() - launches} launches, tokens {stats['tokens']}, flow frames {stats['flow_frames']}, "
          f"stretched {stats['mel_frames']}")
    assert stats["tokens"][3] == 23 and stats["tokens"][5] == 31
    assert stats["mel_frames"][4] == int(stats["flow_frames"][4] / 0.8) and stats["mel_frames"][5] == int(stats["flow_frames"][5] / 1.25)
    diffs = []
    for i, (w, a) in enumerate(zip(wavs, alone)):
        assert torch.isfinite(w).all()
        d = maxdiff(w, a) if w.shape == a.shape else float("inf")
        diffs.append(d)
        print(f"{tag} request {i}: batch {w.shape[1]} samples, tts() {a.shape[1]}, max|batch - tts()| {d:.3g}, bit-identical {torch.equal(w, a)}")
    if precision == "fp32":
        bound = 1e-3 if cv3 else 1e-4
        assert all(d <= bound for d in diffs), diffs


@pytest.mark.parametrize("cv3", [False, True], ids=["cv2", "cv3"])
def test_tts_speed_equals_the_torch_interpolate_it_replaces(cv3, monkeypatch):
    """tts(speed=0.8) through cvk_mel_resample == the same request through token2wav's former torch expression
    (F.interpolate(tts_mel.t().unsqueeze(0), size=int(T / speed), mode="linear")), bit for bit"""
    m = _model3("fp32") if cv3 else _model2("fp32")
    reqs, Ub = _requests(cv3)
    r = dict(reqs[4])
    speed = r.pop("speed")

    def run():
        m.uniforms_override = Ub[:, 4:5]
        m.noise_fn = None if cv3 else (lambda n: stream_noise(4, n).to(m.device))
        try:
            return torch.cat([o["tts_speech"] for o in m.tts(stream=False, speed=speed, **r)], 1)
        finally:
            m.uniforms_override, m.noise_fn = None, None
    got = run()

    def torch_stretch(mel, lens, speeds):
        with torch.cuda.stream(m.stream):
            out = torch.nn.functional.interpolate(mel.t().unsqueeze(0), size=int(mel.shape[0] / speeds[0]), mode="linear")
        return out[0].t(), [out.shape[2]]
    monkeypatch.setattr(m, "mel_stretch", torch_stretch)
    want = run()
    assert got.shape == want.shape and torch.equal(got, want)


@pytest.mark.parametrize("cv3", [False, True], ids=["cv2", "cv3"])
def test_tts_stream_batch_with_vc_rows_equals_tts_stream(cv3):
    """an LM row and two voice-conversion rows in one tts_stream_batch: each request gets the chunks tts(stream=True) gives it
    alone, within 1e-4 (fp32, the bound of the batched streaming tests)"""
    m = _model3("fp32") if cv3 else _model2("fp32")
    reqs, Ub = _requests(cv3)
    g = torch.Generator().manual_seed(83)
    vc_a = dict(reqs[3], source_speech_token=torch.randint(0, 6561, (1, 120), generator=g, dtype=torch.int32))
    vc_b = dict(reqs[3], source_speech_token=torch.randint(0, 6561, (1, 70), generator=g, dtype=torch.int32))
    batch = [reqs[0], vc_a, vc_b]

    def fn(i):
        st = {"k": 0}

        def f(n):
            z = stream_noise(1000 * i + st["k"], n).to(m.device)
            st["k"] += 1
            return z
        return f
    singles = []
    for i, r in enumerate(batch):
        m.uniforms_override, m.token_hop_len = Ub[:, i:i + 1], 25
        m.noise_fn = None if cv3 else fn(i)
        try:
            singles.append([o["tts_speech"] for o in m.tts(stream=True, **r)])
        finally:
            m.uniforms_override, m.noise_fn, m.token_hop_len = None, None, 25
    chunks = [[], [], []]
    kw = {} if cv3 else dict(noise_fns=[fn(i) for i in range(3)])
    for i, out in m.tts_stream_batch(batch, uniforms=Ub[:, :3], **kw):
        chunks[i].append(out["tts_speech"])
    assert len(singles[1]) >= 3
    for i in range(3):
        assert [c.shape[1] for c in chunks[i]] == [c.shape[1] for c in singles[i]], i
        d = maxdiff(torch.cat(chunks[i], 1), torch.cat(singles[i], 1))
        print(f"[{'cv3' if cv3 else 'cv2'} tts_stream_batch with VC rows] request {i}: chunks {[c.shape[1] for c in chunks[i]]}, "
              f"max|batch - tts(stream=True)| {d:.3g}")
        assert d <= 1e-4, (i, d)
    assert len(m._free_slots) == m.stream_slots


def test_batcher_serves_a_mixed_offline_batch():
    """TtsBatcher: requests of every kind submitted together are served as one batch and get tts_batch's waveforms"""
    from cosyvoice_b200.batcher import TtsBatcher
    m = _model3("fp32")
    reqs, Ub = _requests(True)
    m.uniforms_override = Ub
    try:
        want = m.tts_batch(reqs)
        with TtsBatcher(m, max_batch=len(reqs), max_wait_ms=2000) as b:
            futs = [b.submit(**r) for r in reqs]
            got = [f.result(timeout=120) for f in futs]
        assert b.batches == [len(reqs)]
    finally:
        m.uniforms_override = None
    assert all(torch.equal(g_, w) for g_, w in zip(got, want))
