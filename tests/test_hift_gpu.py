"""GPU: HiFT vocoder parity through the C ABI against the oracle (oracle/hift.py) and the committed reference
outputs (tests/golden/hift_*.npz).  fp32 mode: atol 1e-4/rtol 1e-2 per op, the reference's own export tolerance
(cosyvoice/bin/export_onnx.py:99-110); bf16 mode: stated bounds below."""
import numpy as np
import pytest
import torch

from gpu_util import ctx, from_tm, maxdiff, to_tm
from oracle import cases, hift, weights

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sd():
    return weights.synth_state_dict(hift.param_shapes(), 1986, hift.SYNTH_GAINS)


_loaded = set()


def model(precision, sd):
    c = ctx(precision)
    if precision not in _loaded:
        c.load_state_dict("hift", sd)
        _loaded.add(precision)
    return c


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_f0_and_source(precision, sd, golden):
    g = golden("hift_b2_t24")
    melx, noise, rand_ini = cases.hift_case()
    c = model(precision, sd)
    mel_tm, lens = to_tm(melx)
    f0 = c.hift_f0(mel_tm, lens).view(2, -1)
    # the f0 predictor always runs fp32 (its output is integrated into a phase)
    np.testing.assert_allclose(f0.cpu().numpy(), g["f0"], rtol=1e-4, atol=2e-2)
    src = c.hift_source(torch.from_numpy(g["f0"]).reshape(-1), lens, noise.reshape(-1, 9)).view(2, 1, -1)
    assert maxdiff(src, torch.from_numpy(g["source"])) < 2e-3


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_decode_golden(precision, sd, golden):
    g = golden("hift_b2_t24")
    melx, _, _ = cases.hift_case()
    c = model(precision, sd)
    mel_tm, lens = to_tm(melx)
    wav = c.hift_decode(mel_tm, lens, torch.from_numpy(g["source"]).reshape(-1)).view(2, -1)
    d = maxdiff(wav, torch.from_numpy(g["decode"]))
    # tensor-core mode: IEEE-half operands (TF32-class mantissa, like the reference's default cuDNN convolutions)
    print(f"[hift decode golden, {precision}] max |d| {d:.3g}")
    assert d < (1e-3 if precision == "fp32" else 4e-3), d


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_inference_ragged_batch_vs_oracle(precision, sd):
    """ragged batch (different lengths in one call) == per-utterance oracle"""
    c = model(precision, sd)
    lens = [17, 40, 9]
    g = torch.Generator().manual_seed(77)
    mels = [torch.randn(1, 80, T, generator=g) * 2 - 5 for T in lens]
    noises = [torch.randn(1, T * 480, 9, generator=g) for T in lens]
    mel_tm = torch.cat([m[0].t() for m in mels], 0)
    noise = torch.cat([n[0] for n in noises], 0)
    wav, src = c.hift_inference(mel_tm, lens, noise)
    o = 0
    for m, n, T in zip(mels, noises, lens):
        ow, osrc = hift.inference(sd, m, n)
        assert maxdiff(src[o:o + T * 480], osrc.reshape(-1)) < 3e-3
        # the vocoder body is compared with the oracle's source injected (phase conditioning, see DESIGN.md)
        w2 = c.hift_decode(m[0].t().contiguous(), [T], osrc.reshape(-1))
        assert maxdiff(w2, ow.reshape(-1)) < (1e-3 if precision == "fp32" else 4e-3)
        o += T * 480
    assert wav.abs().max().item() <= 0.99 + 1e-6


def test_inference_cuda_cores_in_bf16_context(sd):
    """use_tc 0 (the A/B switch to the CUDA-core conv-GEMM) in a bf16 context: the vocoder's IEEE-half operands and half weight copies
    run on the CUDA cores and give the default (wgmma) run's waveform within the bf16-mode bound above"""
    c = model("bf16", sd)
    lens = [17, 40]
    g = torch.Generator().manual_seed(78)
    mel_tm = torch.randn(sum(lens), 80, generator=g) * 2 - 5
    noise = torch.randn(sum(lens) * 480, 9, generator=g)
    wav_tc, src_tc = c.hift_inference(mel_tm, lens, noise)
    c.set_option("use_tc", 0)
    try:
        wav_cc, src_cc = c.hift_inference(mel_tm, lens, noise)
    finally:
        c.set_option("use_tc", 1)
    d = maxdiff(wav_cc, wav_tc)
    print(f"[hift inference, bf16 context, CUDA cores vs wgmma] max |d| {d:.3g}")
    assert maxdiff(src_cc, src_tc) < 2e-3       # the source path runs fp32 in both
    assert d < 4e-3, d


def test_cache_source_golden(sd, golden):
    g = golden("hift_cache_source")
    melx, noise, _ = cases.hift_case()
    c = model("fp32", sd)
    mel_tm, lens = to_tm(melx[:1])
    wav, src = c.hift_inference(mel_tm, lens, noise[:1].reshape(-1, 9), cache_source=torch.from_numpy(g["cache"]).reshape(-1),
                                cache_lens=[g["cache"].shape[-1]])
    assert maxdiff(src, torch.from_numpy(g["source"]).reshape(-1)) < 2e-3
    w2 = c.hift_decode(mel_tm, lens, torch.from_numpy(g["source"]).reshape(-1))
    assert maxdiff(w2, torch.from_numpy(g["wav"]).reshape(-1)) < 1e-3
