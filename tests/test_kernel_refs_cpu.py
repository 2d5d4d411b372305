"""CPU: the fp64 references of test_kernel_edges_gpu.py and test_kernel_epilogues_gpu.py (tests/kernel_refs.py) against independent
formulations - torch's scaled_dot_product_attention with an explicit mask and expanded K/V heads, one KV-cached step of the oracle
Qwen2 LM, F.conv1d with torch's activations, and the oracle conformer layer's relative-position attention."""
import pytest
import torch
import torch.nn.functional as F

import kernel_refs as kr
from oracle import flow as oflow, hift as ohift, lm as olm


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


@pytest.mark.parametrize("num_layers", [1, 2])
@pytest.mark.parametrize("past_len", [0, 5, 40])
def test_decode_layer_ref_equals_oracle_step(num_layers, past_len):
    """kr.decode_layer (rounding off), layer after layer, then the final RMSNorm == one KV-cached step of oracle.lm.qwen2_forward: the
    final-normed hidden state and every layer's new K / V row"""
    g = torch.Generator().manual_seed(num_layers * 100 + past_len)
    sd = {}
    for name, shape in olm.param_shapes(num_layers, with_lm_head=False).items():
        if name.startswith("llm.model.model.layers."):
            fan_in = shape[-1] if len(shape) == 2 else 1
            sd[name] = kr.bf16(torch.randn(*shape, generator=g) * (fan_in ** -0.5 if len(shape) == 2 else 0.1))
            if name.endswith("layernorm.weight"):
                sd[name] = 1.0 + 0.1 * torch.randn(*shape, generator=g)
    sd["llm.model.model.norm.weight"] = 1.0 + 0.1 * torch.randn(olm.D, generator=g)
    x = torch.randn(1, 1, olm.D, generator=g)
    past = [(torch.randn(1, olm.N_KV, past_len, 64, generator=g), torch.randn(1, olm.N_KV, past_len, 64, generator=g))
            for _ in range(num_layers)]
    hid, new_past = olm.qwen2_forward(sd, x, past if past_len else None, num_layers=num_layers)
    h = x[0].double()
    for i in range(num_layers):
        kc = torch.zeros(1, olm.N_KV, 64, 64, dtype=torch.float64)
        vc = torch.zeros_like(kc)
        kc[0, :, :past_len], vc[0, :, :past_len] = past[i][0][0].double(), past[i][1][0].double()
        st = kr.decode_layer(kr.layer_weights(sd, i), h, kc, vc, [past_len])
        # the oracle runs in fp32: ~1e-6 relative on O(1) values
        assert (new_past[i][0][0, :, past_len].double() - st["k"][0]).abs().max().item() < 1e-4, i
        assert (new_past[i][1][0, :, past_len].double() - st["v"][0]).abs().max().item() < 1e-4, i
        h = st["x_out"]
    want = kr.rms_norm(h, sd["llm.model.model.norm.weight"])
    assert (hid[0].double() - want).abs().max().item() < 1e-4


def test_decode_layer_rounding_points():
    """rounding "fused" / "per-op" rounds exactly the stored stages: every one of them is bf16-representable, the exact reference's
    fp32-kept stages are not (the per-op qkv and g / u), and without rounding nothing is"""
    g = torch.Generator().manual_seed(11)
    sd = {}
    for name, shape in olm.param_shapes(1, with_lm_head=False).items():
        if name.startswith("llm.model.model.layers."):
            sd[name] = kr.bf16(torch.randn(*shape, generator=g) * (shape[-1] ** -0.5 if len(shape) == 2 else 0.1))
    w = kr.layer_weights(sd, 0)
    x = torch.randn(3, olm.D, generator=g, dtype=torch.float64)
    kc = kr.bf16(torch.randn(3, olm.N_KV, 32, 64, generator=g, dtype=torch.float64))
    vc = kr.bf16(torch.randn(3, olm.N_KV, 32, 64, generator=g, dtype=torch.float64))
    is_b = lambda t: torch.equal(t, kr.bf16(t))
    for rounding, stored in [("fused", ("xn", "q", "k", "v", "att", "xn_mid", "ffa")),
                             ("per-op", ("xn", "qkv", "q", "k", "v", "att", "xn_mid", "g", "u", "ffa"))]:
        st = kr.decode_layer(w, x, kc, vc, [0, 7, 31], rounding)
        assert all(is_b(st[n]) for n in stored), rounding
        assert not any(is_b(st[n]) for n in set(("qkv", "g", "u", "x_mid", "x_out")) - set(stored)), rounding
    st = kr.decode_layer(w, x, kc, vc, [0, 7, 31])
    assert not any(is_b(st[n]) for n in ("xn", "qkv", "q", "k", "v", "att", "xn_mid", "g", "u", "ffa", "x_out"))


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


TORCH_ACTS = {
    "none": lambda x, a: x,
    "gelu": lambda x, a: F.gelu(x),
    "gelu_tanh": lambda x, a: F.gelu(x, approximate="tanh"),
    "silu": lambda x, a: F.silu(x),
    "mish": lambda x, a: F.mish(x),
    "elu": lambda x, a: F.elu(x),
    "lrelu": lambda x, a: F.leaky_relu(x, 0.1),
    "snake": lambda x, a: ohift.snake(x.t()[None], a)[0].t(),       # oracle vocoder Snake, channel-major
    "tanh": lambda x, a: torch.tanh(x),
    "abs": lambda x, a: x.abs(),
}


@pytest.mark.parametrize("act", list(TORCH_ACTS))
@pytest.mark.parametrize("taps,dil,shift0", [(1, 1, 0), (3, 1, -1), (7, 3, -9), (31, 1, -30)])
def test_conv_ref_equals_conv1d(taps, dil, shift0, act):
    """conv_rows + conv_epilogue on a packed matrix with gap rows == per-sequence F.conv1d (zero padding) + the torch activation;
    resid, accumulate and the second output follow the epilogue order"""
    g = torch.Generator().manual_seed(taps * 31 + dil)
    K, N = 12, 10
    lens, gap = [17, 1, 40], max(-shift0, shift0 + (taps - 1) * dil)
    starts, r = [], gap
    for L in lens:
        starts.append(r)
        r += L + gap
    rows = r
    x = torch.zeros(rows, K, dtype=torch.float64)
    valid = torch.zeros(rows, dtype=torch.bool)
    for s, L in zip(starts, lens):
        x[s:s + L] = torch.randn(L, K, generator=g, dtype=torch.float64) * 2
        valid[s:s + L] = True
    w = torch.randn(N, K, taps, generator=g, dtype=torch.float64) * (K * taps) ** -0.5
    bias = torch.randn(N, generator=g, dtype=torch.float64)
    alpha = torch.rand(N, generator=g, dtype=torch.float64) * 2 + 0.2
    resid = torch.randn(rows, N, generator=g, dtype=torch.float64)
    init = torch.randn(rows, N, generator=g, dtype=torch.float64)
    acc = kr.conv_rows(x, w, dil, shift0)
    out, out2 = kr.conv_epilogue(acc, valid, bias, act, 0.1, alpha, resid=resid, out_init=init, accumulate=True, act2=act,
                                 act2_param=0.1, alpha2=alpha.flip(0))
    plain, _ = kr.conv_epilogue(acc, valid, bias, act, 0.1, alpha)
    for s, L in zip(starts, lens):
        xs = x[s:s + L].t()[None]
        y = F.conv1d(F.pad(xs, (-shift0, shift0 + (taps - 1) * dil)), w, bias, dilation=dil)[0].t()
        y = TORCH_ACTS[act](y, alpha)
        assert (plain[s:s + L] - y).abs().max().item() < 1e-12
        v = init[s:s + L] + y + resid[s:s + L]
        assert (out[s:s + L] - v).abs().max().item() < 1e-12
        assert (out2[s:s + L] - TORCH_ACTS[act](v, alpha.flip(0))).abs().max().item() < 1e-12
    # gap rows: no output (the accumulate input comes back unchanged), no second output, whatever resid holds there
    assert torch.equal(plain[~valid], torch.zeros_like(plain[~valid]))
    assert torch.equal(out[~valid], init[~valid]) and torch.equal(out2[~valid], torch.zeros_like(out2[~valid]))


def _oracle_enc_layer_attention(x, qkv_w, qkv_b, pos_emb, u, v, chunk):
    """the attention term of oracle.flow._enc_layer: with linear_out = I, linear_pos = I and a zero feed-forward output the layer
    returns x + attention(x)"""
    D, H = oflow.D_ENC, oflow.H_ENC
    p, a = "L", "L.self_attn"
    sd = {p + ".norm_mha.weight": torch.ones(D), p + ".norm_mha.bias": torch.zeros(D),
          p + ".norm_ff.weight": torch.ones(D), p + ".norm_ff.bias": torch.zeros(D),
          a + ".linear_out.weight": torch.eye(D), a + ".linear_out.bias": torch.zeros(D), a + ".linear_pos.weight": torch.eye(D),
          a + ".pos_bias_u": u.view(H, 64), a + ".pos_bias_v": v.view(H, 64),
          p + ".feed_forward.w_1.weight": torch.zeros(4, D), p + ".feed_forward.w_1.bias": torch.zeros(4),
          p + ".feed_forward.w_2.weight": torch.zeros(D, 4), p + ".feed_forward.w_2.bias": torch.zeros(D)}
    for i, n in enumerate("qkv"):
        sd[f"{a}.linear_{n}.weight"] = qkv_w[i]
        sd[f"{a}.linear_{n}.bias"] = qkv_b[i]
    T = x.shape[0]
    mask = oflow.chunk_attention_mask(T, chunk).unsqueeze(0)
    return oflow._enc_layer(sd, p, x[None], mask, pos_emb[None])[0] - x


@pytest.mark.parametrize("chunk", [0, 25])
@pytest.mark.parametrize("extra", [0, 37])
def test_relpos_ref_equals_oracle_layer(extra, chunk):
    """kr.relpos_attention == the oracle conformer layer's attention for one sequence of length L, with the table the oracle builds
    (center = L-1) and with a larger table (center = L-1+extra) whose central 2L-1 rows are the oracle's"""
    D, H = oflow.D_ENC, oflow.H_ENC
    g = torch.Generator().manual_seed(extra + chunk)
    L = 70
    x = torch.randn(L, D, generator=g)
    qkv_w = torch.randn(3, D, D, generator=g) * D ** -0.5
    qkv_b = torch.randn(3, D, generator=g) * 0.1
    u, v = torch.randn(D, generator=g) * 0.5, torch.randn(D, generator=g) * 0.5
    center = L - 1 + extra
    pos = torch.randn(2 * center + 1, D, generator=g)
    att = _oracle_enc_layer_attention(x, qkv_w, qkv_b, pos[extra:extra + 2 * L - 1], u, v, chunk)
    xn = F.layer_norm(x, (D,), torch.ones(D), torch.zeros(D), 1e-12)
    q, k, vv = (F.linear(xn, qkv_w[i], qkv_b[i]) for i in range(3))
    ref = kr.relpos_attention(q, k, vv, pos, center, u, v, [L], H, chunk, 0.125)
    # the oracle runs in fp32: its scores (|s| ~ 10) carry ~1e-6 absolute rounding, the output ~1e-6 relative
    assert (att.double() - ref).abs().max().item() < 1e-4


def test_f16_rounding_saturates():
    x = torch.tensor([1.0, 1.0 + 2 ** -11, 65504.0, 65519.0, 1e6, -1e6, 2.0 ** -25], dtype=torch.float64)
    assert kr.f16(x).tolist() == [1.0, 1.0, 65504.0, 65504.0, 65504.0, -65504.0, 0.0]
