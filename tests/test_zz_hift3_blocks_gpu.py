"""GPU: the CosyVoice3 causal vocoder (stage "hift3") stage by stage against the fp64 vocoder of tests/kernel_refs.py (causal=True),
read through the test-only cvk_hift_hidden and cvk_hift3_inference_rows:
 - f0 (f0_conv_dmma_kernel + f0_head_f64_kernel, float64) against the fp64 predictor with its weight norm folded in float64, as the
   reference's float64 module folds it: within one fp32 ulp (only the order of the fp64 sums differs), final and streaming (T - 3
   frames out, the look-ahead read), across the 128-row tiles, at 3000 frames and in a ragged batch of final and streaming rows;
 - the source, from the kernel's own f0, against the fp32-emulating causal source (nearest phase up-sampling, stored noise indexed
   from each utterance's start);
 - body read-outs 0 .. 20 and the waveform, final and streaming (the body on T - 7 frames, the STFT cut at 120 (T - 7) + 1 frames,
   the last 480 samples dropped), in the three modes of test_hift_blocks_gpu.py, with the bounds of kernel_refs.HIFT_TOL.

The file name sorts last, like the other hift3 files, so that a CUDA fault here cannot disturb the tests that share the process."""
import pytest
import torch

import kernel_refs as kr

pytestmark = pytest.mark.gpu

SEED = 1988
MODES = ("fp32", "f16", "bf16")
ROUNDING = {"fp32": None, "f16": "fp16", "bf16": "bf16"}
MAX_T = 3000
CASES = {"short": ([1, 4, 5, 9, 24], [1, 1, 1, 1, 1]), "stream": ([9, 10, 24, 129], [0, 0, 0, 0]),
         "tiles": ([127, 128, 129], [1, 0, 1]), "long": ([500, 3000], [0, 1]), "ragged": ([1, 130, 9, 274, 300], [1, 0, 0, 1, 0])}

_models = {}


def _model(mode):
    """(context, fp64 weights, stored noise [n, 9]) per mode, closed at the end of the module.  One context is open at a time (the
    tests run mode by mode): three vocoder contexts at once would hold device memory that the tests of the process around them need"""
    if mode not in _models:
        _release()
        from cosyvoice_b200 import cvk
        c = cvk.Context(0, "fp32" if mode == "fp32" else "bf16", workspace_gb=2.0)
        if mode == "bf16":
            c.set_option("hift_f16", 0)
        sd = kr.hift_test_state_dict(SEED, True, clip=True)
        c.load_state_dict("hift3", sd)
        g = torch.Generator().manual_seed(SEED)
        rand_ini = torch.rand(9, generator=g)
        rand_ini[0] = 0
        noise = torch.rand(480 * MAX_T, 9, generator=g)
        c.hift3_set_noise(rand_ini, noise)
        _models[mode] = (c, kr.hift_weights(sd, True), noise.double())
    return _models[mode]


def _release():
    for c, _, _ in _models.values():
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


def _split(x, sizes):
    return list(torch.split(x, sizes))


def _ulps(got, ref):
    """|got - ref| in fp32 ulps of ref"""
    r = ref.float().abs()
    ulp = (torch.nextafter(r, torch.full_like(r, float("inf"))) - r).double()
    return ((got.double() - ref.double()).abs() / ulp).max().item()


@pytest.mark.parametrize("case", list(CASES))
def test_hift3_f0_and_source(case):
    """f0 within one fp32 ulp of the fp64 predictor (fp64 weight-norm fold); the source against the fp32-emulating causal source"""
    c, W, noise = _model("fp32")
    lens, fin = CASES[case]
    mel = _mel(lens, 31 + len(lens))
    _, f0, src = c.hift3_inference_rows(mel, lens, fin)
    n_src = [T if f else T - 3 for T, f in zip(lens, fin)]
    f0s, srcs = _split(f0.cpu(), n_src), _split(src.cpu().double(), [480 * n for n in n_src])
    worst_u, worst_s = 0.0, 0.0
    for T, f, m, got_f0, got_s, n in zip(lens, fin, _split(mel, lens), f0s, srcs, n_src):
        ref = kr.hift_f0(W, m)[:n]
        worst_u = max(worst_u, _ulps(got_f0, ref))
        worst_s = max(worst_s, (got_s - kr.hift_source(W, got_f0, noise, emulate=True)).abs().max().item())
    print(f"[hift3 {case}] f0 largest error {worst_u:.3g} ulp (bound 1); source vs fp32-emulating {worst_s:.3g} "
          f"(bound {kr.HIFT_TOL['source']})")
    assert worst_u <= 1.0 and worst_s <= kr.HIFT_TOL["source"], (worst_u, worst_s)


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("mode", MODES)
def test_hift3_units(mode, case):
    """every body read-out against its fp64 unit fed the kernel's read-outs (the STFT against the fp64 STFT of the kernel's own
    source), and the waveform against the fp64 ISTFT of the kernel's conv_post, final and streaming"""
    c, W, _ = _model(mode)
    rnd = ROUNDING[mode]
    tol = kr.HIFT_TOL[mode]
    lens, fin = CASES[case]
    mel = _mel(lens, 41 + len(lens))
    wav, _, src = c.hift3_inference_rows(mel, lens, fin)
    tb = [T if f else T - 7 for T, f in zip(lens, fin)]
    n_src = [T if f else T - 3 for T, f in zip(lens, fin)]
    K = [_split(c.hift_hidden(mel, lens, u, causal=True, finalize=fin).cpu(),
                [120 * t + 1 if u in (0, 20) else [t, 8 * t, 40 * t, 120 * t + 1][kr._unit_level(u) + 1] for t in tb]) for u in range(21)]
    wavs = _split(wav.cpu().double(), [480 * (T if f else T - 8) for T, f in zip(lens, fin)])
    srcs = _split(src.cpu(), [480 * n for n in n_src])
    worst, fails = {}, []
    for b, (T, f, t, m) in enumerate(zip(lens, fin, tb, _split(mel, lens))):
        Kb = [K[u][b] for u in range(21)]
        checks = [("stft", kr.hift_stft(srcs[b], rnd)[:120 * t + 1], Kb[0]), ("istft", kr.hift_istft(Kb[20], 0 if f else 480), wavs[b])]
        for win in kr.hift_unit_refs(W, Kb, m, t, kr.hift_windows(t, (273, 274)), rnd):
            checks += [(kr.HIFT_UNIT_GROUP[u], ref, got) for u, (ref, got) in win.items()]
        for name, ref, got in checks:
            r = (got - ref).abs().max().item() if name == "istft" else kr.hift_ratio(ref, got)
            worst[name] = max(worst.get(name, 0.0), r)
            if r > tol[name]:
                fails.append((T, f, name, r))
    print(f"[hift3 {mode} {case}] largest ratio: " + ", ".join(f"{k} {v:.3g} (bound {tol[k]})" for k, v in worst.items()))
    assert not fails, fails[:10]
