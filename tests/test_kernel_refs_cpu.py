"""CPU: the fp64 references of test_kernel_edges_gpu.py (tests/kernel_refs.py) against independent formulations - torch's
scaled_dot_product_attention with an explicit mask and expanded K/V heads, and one KV-cached step of the oracle Qwen2 LM."""
import pytest
import torch
import torch.nn.functional as F

import kernel_refs as kr
from oracle import lm as olm


@pytest.mark.parametrize("H,kvh,chunk", [(14, 2, 1), (8, 8, 50), (16, 16, 0), (14, 2, 25)])
def test_attention_ref_equals_sdpa(H, kvh, chunk):
    g = torch.Generator().manual_seed(H * 100 + chunk)
    q_lens, k_lens, q_off = [5, 50, 1, 70], [5, 160, 300, 140], [0, 100, 299, 63]
    q = torch.randn(sum(q_lens), H * 64, generator=g, dtype=torch.float64)
    k = torch.randn(sum(k_lens), kvh * 64, generator=g, dtype=torch.float64)
    v = torch.randn(sum(k_lens), kvh * 64, generator=g, dtype=torch.float64)
    ref = kr.attention(q, k, v, q_lens, k_lens, q_off, H, kvh, chunk, 0.125)
    oq = ok = 0
    for Lq, Lk, off in zip(q_lens, k_lens, q_off):
        qq = q[oq:oq + Lq].view(Lq, H, 64).transpose(0, 1)[None]
        head_kv = torch.arange(H) // (H // kvh)                     # GQA: query head h reads kv head h // G
        kk = k[ok:ok + Lk].view(Lk, kvh, 64).transpose(0, 1)[head_kv][None]
        vv = v[ok:ok + Lk].view(Lk, kvh, 64).transpose(0, 1)[head_kv][None]
        pos_q = torch.arange(Lq)[:, None] + off
        mask = torch.arange(Lk)[None, :] < ((pos_q // chunk + 1) * chunk if chunk > 0 else Lk)
        o = F.scaled_dot_product_attention(qq, kk, vv, attn_mask=mask, scale=0.125)[0].transpose(0, 1).reshape(Lq, H * 64)
        assert (o - ref[oq:oq + Lq]).abs().max().item() < 1e-12
        oq += Lq
        ok += Lk


def _one_layer_sd(seed):
    """layer 0 of the Qwen2 decoder with o_proj = I and a zero MLP, so the layer output is x + attention(x): the attention output
    of the oracle's KV-cached step becomes observable through its hidden state"""
    g = torch.Generator().manual_seed(seed)
    p = "llm.model.model.layers.0"
    D = olm.D
    sd = {}
    for name, shape in olm.param_shapes(1, with_lm_head=False).items():
        if name.startswith(p):
            sd[name] = torch.randn(*shape, generator=g) * (0.05 if name.endswith("weight") and len(shape) == 2 else 0.5)
    sd[p + ".input_layernorm.weight"] = 1.0 + 0.1 * torch.randn(D, generator=g)
    sd[p + ".self_attn.o_proj.weight"] = torch.eye(D)
    for n in ("gate_proj", "up_proj", "down_proj"):
        sd[f"{p}.mlp.{n}.weight"].zero_()
    sd["llm.model.model.norm.weight"] = torch.ones(D)
    return sd


@pytest.mark.parametrize("past_len", [0, 1, 17, 300])
def test_decode_ref_equals_oracle_step(past_len):
    sd = _one_layer_sd(past_len + 7)
    p = "llm.model.model.layers.0"
    g = torch.Generator().manual_seed(past_len)
    x = torch.randn(1, 1, olm.D, generator=g)
    kp = torch.randn(1, olm.N_KV, past_len, 64, generator=g)
    vp = torch.randn(1, olm.N_KV, past_len, 64, generator=g)
    hid, new_past = olm.qwen2_forward(sd, x, [(kp, vp)] if past_len else None, num_layers=1)
    # the qkv projection as the split-K GEMM leaves it: 3 partial sums over disjoint K ranges, bias separate
    xn = olm.rmsnorm(x, sd[p + ".input_layernorm.weight"])[0].double()
    W = torch.cat([sd[f"{p}.self_attn.{n}_proj.weight"] for n in "qkv"]).double()
    bias = torch.cat([sd[f"{p}.self_attn.{n}_proj.bias"] for n in "qkv"]).double()
    cuts = [0, 300, 301, olm.D]
    partial = torch.stack([xn[:, a:b] @ W[:, a:b].t() for a, b in zip(cuts[:-1], cuts[1:])])     # [3, 1, 1152]
    q, k, v = kr.decode_qkv(partial, bias, [past_len], round_bf16=False)
    kc = torch.zeros(1, olm.N_KV, 512, 64, dtype=torch.float64)
    vc = torch.zeros_like(kc)
    kc[0, :, :past_len], vc[0, :, :past_len] = kp[0].double(), vp[0].double()
    o = kr.decode_attention(q, k, v, kc, vc, [past_len])
    # appended cache row == the oracle's rotated k / v of the new position (fp32 oracle vs fp64 reference)
    assert (new_past[0][0][0, :, past_len] - k[0]).abs().max().item() < 1e-5
    assert (new_past[0][1][0, :, past_len] - v[0]).abs().max().item() < 1e-5
    # hidden = rmsnorm(x + o) with unit norm weight
    h = x[0].double() + o
    want = h * torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + olm.RMS_EPS)
    assert (hid[0].double() - want).abs().max().item() < 1e-4


def test_rope_phase_table_matches_libm():
    """The LM kernels rotate by cosf / sinf of fp32(pos * inv_freq[i]) with inv_freq = 1 / powf(1e6, 2i / 64) (llm.cu
    lm_rope_inv_freq); oracle.lm.rope builds the same fp32 table, so the decode-attention bound of test_kernel_edges_gpu.py needs
    no allowance for a phase difference, only for the fp32 evaluation of the rotation."""
    import ctypes
    import ctypes.util
    import numpy as np
    libm = ctypes.CDLL(ctypes.util.find_library("m"))
    libm.powf.restype, libm.powf.argtypes = ctypes.c_float, [ctypes.c_float, ctypes.c_float]
    kern = np.array([np.float32(1.0) / np.float32(libm.powf(1.0e6, np.float32(2 * i) / np.float32(64))) for i in range(32)], np.float32)
    pos = torch.tensor([1])
    x = torch.zeros(1, 1, 1, 64, dtype=torch.float64)
    x[..., :32] = 1.0                                   # rope(x) first half = cos(pos * inv)
    want = torch.cos(torch.from_numpy(kern) * pos.float())
    assert torch.equal(olm.rope(x, pos)[0, 0, 0, :32].float(), want)


def test_bf16_helpers():
    x = torch.tensor([1.0, 1.0 + 2 ** -8, 1.0 + 2 ** -9, -3.0, 1e-3], dtype=torch.float64)
    assert torch.equal(kr.bf16_ulp(x), torch.tensor([2 ** -7, 2 ** -7, 2 ** -7, 2 ** -6, 2.0 ** (-10 - 7)], dtype=torch.float64))
    assert kr.near_bf16_tie(x, 1e-12).tolist() == [False, True, False, False, False]     # 1 + 2^-8 is a midpoint
