"""GPU: CosyVoice3 causal vocoder (SURVEY.md §8 row a16) through the C ABI against the committed outputs of the reference
CausalHiFTGenerator (tests/golden/hift_causal.npz, made by oracle/make_golden.py::gen_hift_causal).

The file name sorts last so that a CUDA fault here cannot disturb the tests that share the process."""
import numpy as np
import pytest
import torch

from gpu_util import ctx, maxdiff
from oracle import cases, hift_causal as hc, weights

pytestmark = pytest.mark.gpu
_loaded = set()


def model(precision):
    c = ctx(precision)
    if precision not in _loaded:
        c.load_state_dict("hift3", weights.synth_state_dict(hc.param_shapes(), 1986, hc.SYNTH_GAINS))
        _loaded.add(precision)
    return c


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_hift3_offline_golden(precision, golden):
    g = golden("hift_causal")
    mel, rand_ini, sine_noise = cases.hift_causal_case()
    c = model(precision)
    c.hift3_set_noise(rand_ini, sine_noise[0])
    wav, f0, src = c.hift3_inference(mel[0].t().contiguous(), [mel.shape[2]], finalize=True)
    np.testing.assert_allclose(f0.cpu().numpy(), g["f0_final"][0], rtol=1e-4, atol=1e-2)         # float64 predictor (weight-norm folded in fp32)
    assert maxdiff(src, torch.from_numpy(g["source_final"]).reshape(-1)) < 2e-3
    d = maxdiff(wav, torch.from_numpy(g["wav_final"]).reshape(-1))
    assert d < (2e-3 if precision == "fp32" else 8e-2), d


def test_hift3_ragged_batch_vs_oracle():
    """two utterances of different lengths in one call == the oracle one at a time"""
    c = model("fp32")
    sd = weights.synth_state_dict(hc.param_shapes(), 1986, hc.SYNTH_GAINS)
    g = torch.Generator().manual_seed(12)
    lens = [19, 33]
    mels = [torch.randn(1, 80, T, generator=g) * 2 - 5 for T in lens]
    rand_ini = torch.rand(1, 9, generator=g)
    rand_ini[:, 0] = 0
    noise = torch.rand(1, max(lens) * 480, 9, generator=g)
    c.hift3_set_noise(rand_ini, noise[0])
    wav, f0, src = c.hift3_inference(torch.cat([m[0].t() for m in mels], 0), lens, finalize=True)
    o = 0
    for m, T in zip(mels, lens):
        ow, osrc = hc.inference(sd, m, rand_ini, noise, True)
        assert maxdiff(src[o * 480:(o + T) * 480], osrc.reshape(-1)) < 3e-3
        assert maxdiff(wav[o * 480:(o + T) * 480], ow.reshape(-1)) < 5e-3
        o += T


def test_hift3_streaming_call_golden(golden):
    """finalize=False (generator.py:676-683, 709-710, 722-725): look-ahead frames consumed, tail dropped"""
    g = golden("hift_causal")
    mel, rand_ini, sine_noise = cases.hift_causal_case()
    c = model("fp32")
    c.hift3_set_noise(rand_ini, sine_noise[0])
    wav, f0, src = c.hift3_inference(mel[0].t().contiguous(), [mel.shape[2]], finalize=False)
    assert wav.numel() == g["wav_chunk"].shape[1] == (24 - 8) * 480
    np.testing.assert_allclose(f0.cpu().numpy(), g["f0_chunk"][0], rtol=1e-4, atol=1e-2)
    assert maxdiff(src, torch.from_numpy(g["source_chunk"]).reshape(-1)) < 2e-3
    assert maxdiff(wav, torch.from_numpy(g["wav_chunk"]).reshape(-1)) < 2e-3
