"""GPU: the CosyVoice2 vocoder (stage "hift") stage by stage against the fp64 vocoder of tests/kernel_refs.py, read through the
test-only cvk_hift_hidden (the 21 read-outs of the body: source STFT, conv_pre, per level the up-sampling, the source branch, the
three resblocks and the level output, conv_post):
 A. stage isolation in three modes - fp32 (against the exact reference), bf16 with hift_f16 = 1 (IEEE-half operands) and bf16 with
    hift_f16 = 0 (bf16 operands), both against the reference that rounds where the 16-bit path stores (kernel_refs.hift_body's
    `rounding`).  Every unit is fed the kernel's own read-outs of the units before it.  Long sequences are checked on windows of
    body frames (head, tail and the frames around every launch-grid seam: source_kernel's grid-stride seam at 131 072 samples =
    frame 273, stft16_kernel's at 131 072 STFT frames = frame 1092), each window computed from the kernel's rows with the unit's
    halo; f0, source, STFT and ISTFT are checked over the whole length.  Lengths 1 .. 3000 frames and a ragged batch.
 B. identities: each of 32 utterances of 400 .. 600 frames alone equals its rows of the batch bit for bit, for every read-out, the
    source and the waveform; two runs agree.

Ratios are the largest |error| over the rms of the reference row (kernel_refs.hift_ratio).  Bounds are kernel_refs.HIFT_TOL, where
the measurements they come from are listed; each case prints its ratios before anything is asserted.  Which defects the bounds
catch is pinned on the CPU by test_kernel_refs_cpu.py::test_hift_mutations_exceed_bounds.

The weights are kernel_refs.hift_test_state_dict(clip=True): conv_post's magnitude channels push some frames past ln 100 and some
samples past +-0.99, so the ISTFT's magnitude clip and the output clamp are compared too.  Each context is private to this module
and closed at its end."""
import pytest
import torch

import kernel_refs as kr

pytestmark = pytest.mark.gpu

SEED = 1987
MODES = ("fp32", "f16", "bf16")
ROUNDING = {"fp32": None, "f16": "fp16", "bf16": "bf16"}
SEAMS = (273, 274, 1092, 1093)
LAYOUTS = {"short": [[T] for T in (1, 2, 3, 7, 8, 9, 16, 24)], "tiles": [[127], [128], [129]], "seams": [[273], [274], [500]],
           "long": [[1092], [1093], [3000]], "ragged": [[1, 1093, 2, 274, 129]]}

_models = {}


def _model(mode):
    """(context, fp64 weights) per mode, closed at the end of the module.  One context is open at a time (the
    tests run mode by mode): three vocoder contexts at once would hold device memory that the tests of the process around them need"""
    if mode not in _models:
        _release()
        from cosyvoice_b200 import cvk
        c = cvk.Context(0, "fp32" if mode == "fp32" else "bf16", workspace_gb=6.0)
        if mode == "bf16":
            c.set_option("hift_f16", 0)
        sd = kr.hift_test_state_dict(SEED, False, clip=True)
        c.load_state_dict("hift", sd)
        _models[mode] = (c, kr.hift_weights(sd, False))
    return _models[mode]


def _release():
    for c, _ in _models.values():
        c.close()
    _models.clear()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", autouse=True)
def _release_models():
    yield
    _release()


def _mel(lens, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(sum(lens), 80, generator=g) * 2 - 5


def _f0(T, seed):
    """crafted f0 [T]: voiced stretches at 80 .. 400 Hz, an unvoiced run, f0 exactly at 10 and one fp32 ulp above, and f0 whose
    h f0 / 24000 lands on integers (3000 Hz: h = 8, 4800 Hz: h = 5)"""
    g = torch.Generator().manual_seed(seed)
    f = 80 + 320 * torch.rand(T, generator=g)
    special = torch.tensor([10.0, float(torch.nextafter(torch.tensor(10.0), torch.tensor(11.0))), 0.0, 3.0, 3000.0, 4800.0, 0.0, 9.5])
    n = min(T - T // 3, special.numel())
    f[T // 3:T // 3 + n] = special[:n]
    return f


def _source(lens, seed):
    """a source [sum 480 T] at full scale: +-1 at both ends of every utterance and within 1e-3 of it in between"""
    g = torch.Generator().manual_seed(seed)
    parts = []
    for T in lens:
        s = torch.tanh(3 * torch.randn(480 * T, generator=g)).clamp(-0.999, 0.999)
        s[0], s[-1], s[1], s[-2] = 1.0, -1.0, -1.0, 1.0
        parts.append(s)
    return torch.cat(parts)


def _split(x, sizes):
    return list(torch.split(x, sizes))


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("mode", MODES)
def test_hift_units(mode, layout):
    """every body read-out against its fp64 unit fed the kernel's read-outs; the STFT against the fp64 STFT of the injected source;
    the waveform against the fp64 ISTFT of the kernel's conv_post"""
    c, W = _model(mode)
    rnd = ROUNDING[mode]
    tol = kr.HIFT_TOL[mode]
    worst = {}
    fails = []
    for n, lens in enumerate(LAYOUTS[layout]):
        mel = _mel(lens, 11 + n)
        src = _source(lens, 17 + n)
        K = [_split(c.hift_hidden(mel, lens, u, source=src).cpu(), [120 * T + 1 if u in (0, 20) else
                    [T, 8 * T, 40 * T, 120 * T + 1][kr._unit_level(u) + 1] for T in lens]) for u in range(21)]
        wav = _split(c.hift_decode(mel, lens, src).cpu().double(), [480 * T for T in lens])
        for b, (T, m, s) in enumerate(zip(lens, _split(mel, lens), _split(src, [480 * T for T in lens]))):
            Kb = [K[u][b] for u in range(21)]
            checks = [("stft", kr.hift_stft(s, rnd), Kb[0]), ("istft", kr.hift_istft(Kb[20]), wav[b])]
            for win in kr.hift_unit_refs(W, Kb, m, T, kr.hift_windows(T, SEAMS), rnd):
                checks += [(kr.HIFT_UNIT_GROUP[u], ref, got) for u, (ref, got) in win.items()]
            for name, ref, got in checks:
                r = kr.hift_ratio(ref, got[:, None] if got.dim() == 1 else got) if name != "istft" else (got - ref).abs().max().item()
                worst[name] = max(worst.get(name, 0.0), r)
                if r > tol[name]:
                    fails.append((lens, b, name, r))
    print(f"[hift {mode} {layout}] largest ratio: " + ", ".join(f"{k} {v:.3g} (bound {tol[k]})" for k, v in worst.items()))
    assert not fails, fails[:10]


@pytest.mark.parametrize("mode", ["fp32", "bf16"])
def test_hift_f0(mode):
    """the f0 predictor (fp32 in every mode) against the fp64 predictor at every length; error over the utterance's f0 rms"""
    c, W = _model(mode)
    worst = 0.0
    for lens in ([1], [2], [3], [9], [127, 128, 129], [500], [3000], [1, 1093, 2, 274, 129]):
        mel = _mel(lens, 5 + len(lens))
        f0 = _split(c.hift_f0(mel, lens).cpu().double(), lens)
        for T, m, got in zip(lens, _split(mel, lens), f0):
            ref = kr.hift_f0(W, m)
            worst = max(worst, ((got - ref).abs().max() / ref.pow(2).mean().sqrt()).item())
    print(f"[hift f0 {mode}] largest error / f0 rms {worst:.3g} (bound {kr.HIFT_TOL[mode]['f0']})")
    assert worst <= kr.HIFT_TOL[mode]["f0"], worst


def test_hift_source():
    """hift_source on crafted f0 against the fp32-emulating source (phase_kernel's and source_kernel's fp32 rounding points):
    tight at every length, including past source_kernel's grid-stride seam and a steady 300 Hz over 3000 frames, where the phase
    reaches 2.7e7 rad and one fp32 ulp of it is 2 rad; against the exact fp64 source: printed and held to the effect of that
    ulp (kernel_refs.hift_source_ulp_bound)"""
    c, W = _model("fp32")
    fails = []
    for lens in ([1], [2], [8], [273], [274], [1093], [3000], [1, 274, 2, 1093]):
        f0 = torch.cat([_f0(T, 3 + T) for T in lens])
        if lens == [3000]:
            f0 = torch.full((3000,), 300.0)
        g = torch.Generator().manual_seed(len(lens) + lens[0])
        noise = torch.randn(480 * sum(lens), 9, generator=g)
        got = _split(c.hift_source(f0, lens, noise).cpu().double(), [480 * T for T in lens])
        o = 0
        for T, f, s in zip(lens, _split(f0, lens), got):
            nz = noise[480 * o:480 * (o + T)]
            e_emu = (s - kr.hift_source(W, f, nz, emulate=True)).abs().max().item()
            e_ex = (s - kr.hift_source(W, f, nz)).abs().max().item()
            bound_ex = kr.hift_source_ulp_bound(W, f)
            print(f"[hift source T={T}] vs fp32-emulating {e_emu:.3g} (bound {kr.HIFT_TOL['source']}), vs exact {e_ex:.3g} "
                  f"(bound {bound_ex:.3g})")
            if e_emu > kr.HIFT_TOL["source"] or e_ex > bound_ex:
                fails.append((T, e_emu, e_ex, bound_ex))
            o += T
    assert not fails, fails


def test_hift_cache_source():
    """a ragged hift_inference whose utterances carry cache lengths 0, 1 and 480 T: the cache replaces the head of each source, the
    rest is hift_source of the predicted f0, and the waveform is hift_decode's of that source, all bit for bit"""
    c, _ = _model("f16")
    lens = [24, 9, 40]
    cl = [0, 1, 480 * 40]
    mel = _mel(lens, 21)
    g = torch.Generator().manual_seed(22)
    noise = torch.randn(480 * sum(lens), 9, generator=g)
    cache = torch.rand(sum(cl), generator=g) * 2 - 1
    wav, src = c.hift_inference(mel, lens, noise, cache_source=cache, cache_lens=cl)
    plain = c.hift_source(c.hift_f0(mel, lens), lens, noise)
    o, oc = 0, 0
    for T, n in zip(lens, cl):
        assert torch.equal(src[o:o + n].cpu(), cache[oc:oc + n]), (T, n)
        assert torch.equal(src[o + n:o + 480 * T], plain[o + n:o + 480 * T]), (T, n)
        o, oc = o + 480 * T, oc + n
    assert torch.equal(wav, c.hift_decode(mel, lens, src))


def _batch_lens():
    g = torch.Generator().manual_seed(32)
    return torch.randint(400, 601, (32,), generator=g).tolist()


@pytest.mark.parametrize("mode", MODES)
def test_hift_batch_rows_bit_identical(mode):
    """32 utterances of 400 .. 600 frames (the benchmark's vocoder batch): every read-out, the source and the waveform of each
    utterance alone equal its rows of the batch bit for bit, and two batch runs agree bit for bit"""
    c, _ = _model(mode)
    lens = _batch_lens()
    mel = _mel(lens, 3232)
    f0 = torch.cat([_f0(T, T) for T in lens])
    g = torch.Generator().manual_seed(33)
    noise = torch.randn(480 * sum(lens), 9, generator=g)
    src = c.hift_source(f0, lens, noise)
    assert torch.equal(src, c.hift_source(f0, lens, noise)), "source: run to run"
    wav = c.hift_decode(mel, lens, src)
    assert torch.equal(wav, c.hift_decode(mel, lens, src)), "wav: run to run"
    mels, f0s, srcs = _split(mel, lens), _split(f0, lens), _split(src, [480 * T for T in lens])
    wavs = _split(wav, [480 * T for T in lens])
    noises = _split(noise, [480 * T for T in lens])
    for b, T in enumerate(lens):
        assert torch.equal(c.hift_source(f0s[b], [T], noises[b]), srcs[b]), (mode, b, T, "source")
        assert torch.equal(c.hift_decode(mels[b], [T], srcs[b]), wavs[b]), (mode, b, T, "wav")
    for u in range(21):
        hb = c.hift_hidden(mel, lens, u, source=src)
        assert torch.equal(hb, c.hift_hidden(mel, lens, u, source=src)), (mode, u, "run to run")
        rows = [120 * T + 1 if u in (0, 20) else [T, 8 * T, 40 * T, 120 * T + 1][kr._unit_level(u) + 1] for T in lens]
        for b, (T, h) in enumerate(zip(lens, _split(hb, rows))):
            assert torch.equal(c.hift_hidden(mels[b], [T], u, source=srcs[b]), h), (mode, u, b, T)


def test_hift_hidden_refuses_bad_arguments():
    """a unit outside [0, 20] and a missing source are refused before any device work"""
    from cosyvoice_b200.cvk import CvkError
    c, _ = _model("fp32")
    lens = [9]
    mel, src = _mel(lens, 1), _source(lens, 1)
    before = c.hift_hidden(mel, lens, 20, source=src)
    for u in (-1, 21):
        with pytest.raises(CvkError):
            c.hift_hidden(mel, lens, u, source=src)
    with pytest.raises(CvkError):
        c.hift_hidden(mel, lens, 5)
    assert torch.equal(before, c.hift_hidden(mel, lens, 20, source=src))
