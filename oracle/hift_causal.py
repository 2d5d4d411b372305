"""Oracle (test infrastructure): CosyVoice3 causal vocoder restated in plain torch on CPU.

Follows cosyvoice/hifigan/generator.py:572-726 (CausalHiFTGenerator: __init__, decode :674-712, inference :714-726), the causal
branches of SineGen2 / SourceModuleHnNSF (:223-226, :243-244, :257-261, :303-307, :356-357, :369-372), ResBlock(causal=True)
(:45-117), cosyvoice/hifigan/f0_predictor.py:60-103 (CausalConvRNNF0Predictor, run in float64 by inference :716-717) and the
causal convolutions of cosyvoice/transformer/convolution.py:150-258, with the hyper-parameters of
examples/libritts/cosyvoice3/conf/cosyvoice3.yaml (upsample 8/5/3, kernels 16/11/7, conv_pre look-right 4).

The reference's "stored noise" (``SineGen2.rand_ini`` [1,9], ``SineGen2.sine_waves`` [1,300*24000,9] uniform, and
``SourceModuleHnNSF.uv``) is drawn from the global RNG in the constructors and is NOT part of the state_dict; here, as in the
non-causal oracle, it is an explicit input, and the golden generator overwrites the reference module's attributes with the same
tensors.  Pinned against the reference module by oracle/make_golden.py (tests/golden/hift_causal.npz).
"""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

from . import hift as H
from .hift import (AUDIO_LIMIT, BASE_CH, HOP, LRELU, N_FFT, NB_HARM, NOISE_STD, RB_DILS, RB_KERNELS, SINE_AMP, SR, SRC_RB_KERNELS,
                   UPS_KERNELS, UPS_RATES, UPSCALE, VOICED_THR, _w, _wn, _resblock_shapes, snake, stft16, istft16)

LOOK_RIGHT = 4          # conv_pre_look_right (cosyvoice3.yaml)
F0_LOOK_RIGHT = 3       # CausalConv1d(80, 512, kernel 4, 'right').causal_padding


def param_shapes():
    """state_dict keys / shapes of the reference CausalHiFTGenerator in module order."""
    s = OrderedDict()
    s["m_source.l_linear.weight"] = (1, NB_HARM + 1)
    s["m_source.l_linear.bias"] = (1,)
    _wn(s, "conv_pre", (BASE_CH, 80, LOOK_RIGHT + 1))
    for i, (u, k) in enumerate(zip(UPS_RATES, UPS_KERNELS)):
        # CausalConv1dUpsample is a Conv1d (not transposed): weight [out, in, k], bias [out]
        p = f"ups.{i}"
        cin, cout = BASE_CH // 2 ** i, BASE_CH // 2 ** (i + 1)
        s[p + ".bias"] = (cout,)
        s[p + ".parametrizations.weight.original0"] = (cout, 1, 1)
        s[p + ".parametrizations.weight.original1"] = (cout, cin, k)
    down = [30, 6, 1]       # CausalConv1dDownSample kernel = 2 * stride (15, 3); last level: CausalConv1d k1
    for i in range(3):
        ch = BASE_CH // 2 ** (i + 1)
        s[f"source_downs.{i}.weight"] = (ch, N_FFT + 2, down[i])
        s[f"source_downs.{i}.bias"] = (ch,)
    for i in range(3):
        _resblock_shapes(s, f"source_resblocks.{i}", BASE_CH // 2 ** (i + 1), SRC_RB_KERNELS[i])
    for i in range(3):
        for j, k in enumerate(RB_KERNELS):
            _resblock_shapes(s, f"resblocks.{i * 3 + j}", BASE_CH // 2 ** (i + 1), k)
    _wn(s, "conv_post", (N_FFT + 2, BASE_CH // 8, 7))
    _wn(s, "f0_predictor.condnet.0", (512, 80, 4))
    for i in range(1, 5):
        _wn(s, f"f0_predictor.condnet.{2 * i}", (512, 512, 3))
    s["f0_predictor.classifier.weight"] = (1, 512)
    s["f0_predictor.classifier.bias"] = (1,)
    return s


SYNTH_GAINS = H.SYNTH_GAINS


def causal_padding(k, d=1):
    """convolution.py:172"""
    return int((k * d - d) / 2) * 2 + (k + 1) % 2


def causal_conv(x, w, b, d=1, right=False, cache=None):
    """CausalConv1d.forward (convolution.py:176-187): zero (or cached) padding of causal_padding samples on the left
    ('left') or on the right ('right' = look-ahead)."""
    k = w.shape[2]
    pad = causal_padding(k, d)
    if cache is None:
        cache = torch.zeros(x.shape[0], x.shape[1], pad, dtype=x.dtype)
    assert cache.shape[2] == pad
    x = torch.cat([x, cache], dim=2) if right else torch.cat([cache, x], dim=2)
    y = F.conv1d(x, w, b, dilation=d)
    assert y.shape[2] == x.shape[2] - pad
    return y


def resblock_causal(sd, prefix, x, k):
    """ResBlock(causal=True): generator.py:110-117 over left-padded convolutions."""
    for i, d in enumerate(RB_DILS):
        xt = snake(x, sd[f"{prefix}.activations1.{i}.alpha"])
        xt = causal_conv(xt, _w(sd, f"{prefix}.convs1.{i}"), sd[f"{prefix}.convs1.{i}.bias"], d=d)
        xt = snake(xt, sd[f"{prefix}.activations2.{i}.alpha"])
        xt = causal_conv(xt, _w(sd, f"{prefix}.convs2.{i}"), sd[f"{prefix}.convs2.{i}.bias"])
        x = xt + x
    return x


def _w64(sd, prefix):
    """weight norm folded in float64: the reference converts the predictor module to float64 before its parametrization runs"""
    return H.weight_norm_effective(sd[prefix + ".parametrizations.weight.original0"].double(),
                                   sd[prefix + ".parametrizations.weight.original1"].double())


def f0_predict(sd, mel, finalize=True):
    """f0_predictor.py:95-103 in float64 (generator.py:716-717).  mel [B,80,T] -> f0 [B,T] (finalize) or [B,T-3]."""
    x = mel.double()
    w0, b0 = _w64(sd, "f0_predictor.condnet.0"), sd["f0_predictor.condnet.0.bias"].double()
    if finalize:
        x = causal_conv(x, w0, b0, right=True)
    else:
        x = causal_conv(x[:, :, :-F0_LOOK_RIGHT], w0, b0, right=True, cache=x[:, :, -F0_LOOK_RIGHT:])
    x = F.elu(x)
    for i in range(1, 5):
        p = f"f0_predictor.condnet.{2 * i}"
        x = F.elu(causal_conv(x, _w64(sd, p), sd[p + ".bias"].double()))
    x = x.transpose(1, 2)
    f0 = torch.abs(F.linear(x, sd["f0_predictor.classifier.weight"].double(), sd["f0_predictor.classifier.bias"].double()).squeeze(-1))
    return f0.float()


def sine_source(sd, f0, rand_ini, sine_noise):
    """generator.py:718-721 + causal SourceModuleHnNSF / SineGen2.  f0 [B,T]; rand_ini [1,9] (column 0 = 0); sine_noise
    [1, >=480T, 9] (the stored ``sine_waves`` tensor, uniform [0,1) in the reference).  Returns s [B,1,480T]."""
    B, T = f0.shape
    L = T * UPSCALE
    f0u = f0[:, :, None].repeat_interleave(UPSCALE, dim=1)
    harm = torch.arange(1, NB_HARM + 2, dtype=torch.float32).view(1, 1, -1)
    rad = (f0u * harm / SR) % 1
    rad[:, 0, :] = rad[:, 0, :] + rand_ini
    rad = F.interpolate(rad.transpose(1, 2), scale_factor=1 / UPSCALE, mode="linear").transpose(1, 2)
    phase = torch.cumsum(rad, dim=1) * 2 * np.pi
    phase = F.interpolate(phase.transpose(1, 2) * UPSCALE, scale_factor=UPSCALE, mode="nearest").transpose(1, 2)   # causal: nearest
    sines = torch.sin(phase) * SINE_AMP
    uv = (f0u > VOICED_THR).float()
    noise_amp = uv * NOISE_STD + (1 - uv) * SINE_AMP / 3
    sine_waves = sines * uv + noise_amp * sine_noise[:, :L]
    merged = torch.tanh(F.linear(sine_waves, sd["m_source.l_linear.weight"], sd["m_source.l_linear.bias"]))
    return merged.transpose(1, 2)


def decode(sd, mel, s, finalize=True, return_pre_istft=False):
    """generator.py:674-712.  finalize: mel [B,80,T], s [B,1,480T] -> wav [B,480T].  Streaming (finalize=False): the last
    LOOK_RIGHT mel frames are look-ahead for conv_pre only, the source STFT is cut accordingly and the last 480 samples of the
    waveform are dropped."""
    re, im = stft16(s.squeeze(1))
    wpre, bpre = _w(sd, "conv_pre"), sd["conv_pre.bias"]
    if finalize:
        x = causal_conv(mel, wpre, bpre, right=True)
    else:
        x = causal_conv(mel[:, :, :-LOOK_RIGHT], wpre, bpre, right=True, cache=mel[:, :, -LOOK_RIGHT:])
        cut = int(np.prod(UPS_RATES)) * LOOK_RIGHT
        re, im = re[:, :, :-cut], im[:, :, :-cut]
    s_stft = torch.cat([re, im], dim=1)
    strides = [15, 3, 1]
    for i in range(3):
        x = F.leaky_relu(x, LRELU)
        u, k = UPS_RATES[i], UPS_KERNELS[i]
        x = x.repeat_interleave(u, dim=2)                                           # nn.Upsample(nearest)
        x = F.conv1d(F.pad(x, (k - 1, 0)), _w(sd, f"ups.{i}"), sd[f"ups.{i}.bias"])  # CausalConv1dUpsample
        if i == 2:
            x = F.pad(x, (1, 0), mode="reflect")
        w, b = sd[f"source_downs.{i}.weight"], sd[f"source_downs.{i}.bias"]
        if strides[i] == 1:
            si = causal_conv(s_stft, w, b)                                           # k = 1: no padding
        else:
            si = F.conv1d(F.pad(s_stft, (strides[i] - 1, 0)), w, b, stride=strides[i])   # CausalConv1dDownSample
        si = resblock_causal(sd, f"source_resblocks.{i}", si, SRC_RB_KERNELS[i])
        x = x + si
        xs = None
        for j, k2 in enumerate(RB_KERNELS):
            r = resblock_causal(sd, f"resblocks.{i * 3 + j}", x, k2)
            xs = r if xs is None else xs + r
        x = xs / 3
    x = F.leaky_relu(x)
    x = causal_conv(x, _w(sd, "conv_post"), sd["conv_post.bias"])
    if return_pre_istft:
        return x
    mag = torch.exp(x[:, :N_FFT // 2 + 1])
    phase = torch.sin(x[:, N_FFT // 2 + 1:])
    y = istft16(mag, phase)
    if not finalize:
        y = y[:, :-int(np.prod(UPS_RATES) * HOP)]
    return torch.clamp(y, -AUDIO_LIMIT, AUDIO_LIMIT)


def inference(sd, mel, rand_ini, sine_noise, finalize=True):
    """generator.py:714-726.  Returns (wav, source [B,1,480 T'])."""
    f0 = f0_predict(sd, mel, finalize)
    s = sine_source(sd, f0, rand_ini, sine_noise)
    if finalize:
        return decode(sd, mel, s, True), s
    return decode(sd, mel[:, :, :-F0_LOOK_RIGHT], s, False), s
