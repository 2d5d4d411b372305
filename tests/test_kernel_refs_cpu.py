"""CPU: the fp64 references of test_kernel_edges_gpu.py and test_kernel_epilogues_gpu.py (tests/kernel_refs.py) against independent
formulations - torch's scaled_dot_product_attention with an explicit mask and expanded K/V heads, one KV-cached step of the oracle
Qwen2 LM, F.conv1d with torch's activations, and the oracle conformer layer's relative-position attention."""
import numpy as np
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


# ================================================================================================ CosyVoice3 DiT references
from oracle import cases, dit as odit, weights as oweights  # noqa: E402


def _dit_sd(depth=2):
    return kr.dit_test_state_dict(depth, 31)


def _dit_case(lens, seed):
    g = torch.Generator().manual_seed(seed)
    R = sum(lens)
    x, mu, cond = (kr.bf16(torch.rand(R, 80, generator=g) * 2 - 1) for _ in range(3))
    return x, mu, cond, kr.bf16(torch.randn(len(lens), 80, generator=g)), torch.tensor([0.3, 0.7][:len(lens)], dtype=torch.float64)


def test_dit_modulation_ref_equals_oracle():
    """kr.dit_modulation == oracle.dit's time_embedding and every AdaLN linear on its SiLU, in float32"""
    sd = _dit_sd()
    W = kr.dit_weights(sd, 2)
    t = torch.tensor([0.05, 0.3, 0.95])
    te = odit.time_embedding(sd, "decoder.estimator.", t)
    mod = kr.dit_modulation(W, t.double())["mod"]
    for i, name in enumerate(["transformer_blocks.0.attn_norm", "transformer_blocks.1.attn_norm", "norm_out"]):
        p = f"decoder.estimator.{name}.linear."
        want = F.linear(F.silu(te), sd[p + "weight"], sd[p + "bias"]).double()
        # fp32 angles up to 950 rad: sin / cos good to ~1e-4 (1000 t e_i rounded to 24 bits); through the time MLP ~1e-4 of |mod| ~ 1
        assert (mod[:, i * 6144:i * 6144 + want.shape[1]] - want).abs().max().item() < 1e-3, name


def test_dit_input_embedding_ref_equals_oracle():
    """kr.dit_input_embedding (exact) == proj([x | cond | mu | spks]) + oracle.dit.conv_pos_embed, per sequence of a ragged pack"""
    sd = _dit_sd()
    W = kr.dit_weights(sd, 2)
    lens = [37, 1, 64]
    x, mu, cond, spks, _ = _dit_case(lens, 1)
    spks = torch.cat([spks, spks[:1]])
    got = kr.dit_input_embedding(W, x, mu, cond, spks, lens)["x0"]
    p, o = "decoder.estimator.", 0
    for b, L in enumerate(lens):
        h = F.linear(torch.cat([x[o:o + L], cond[o:o + L], mu[o:o + L], spks[b].expand(L, 80)], -1)[None], sd[p + "input_embed.proj.weight"],
                     sd[p + "input_embed.proj.bias"])
        want = (odit.conv_pos_embed(sd, p, h) + h)[0].double()
        assert (got[o:o + L] - want).abs().max().item() < 1e-4, (b, L)          # fp32 oracle on O(1) values
        o += L


@pytest.mark.parametrize("streaming", [False, True])
def test_dit_block_ref_equals_oracle(streaming):
    """kr.dit_block (exact) == oracle.dit.dit_block on every sequence of a ragged pack (per-sequence modulation, rotary positions
    from 0, the 50-frame block-causal mask when streaming)"""
    sd = _dit_sd()
    W = kr.dit_weights(sd, 2)
    lens = [120, 51]
    g = torch.Generator().manual_seed(2)
    x = torch.randn(sum(lens), 1024, generator=g)
    t = torch.tensor([0.2, 0.8])
    mod = kr.dit_modulation(W, t.double())["mod"]
    got = kr.dit_block(W, 1, x, mod, lens, 50 if streaming else 0)["x_out"]
    te = odit.time_embedding(sd, "decoder.estimator.", t)
    o = 0
    for b, L in enumerate(lens):
        m = odit._flow.chunk_attention_mask(L, 50)[None] if streaming else torch.ones(1, L, L, dtype=torch.bool)
        want = odit.dit_block(sd, "decoder.estimator.transformer_blocks.1.", x[o:o + L][None], te[b:b + 1], m.unsqueeze(1),
                              odit.rotary_freqs(L))[0].double()
        assert (got[o:o + L] - want).abs().max().item() < 2e-3 * want.abs().max().item(), (b, L)   # fp32 oracle, gates ~ 1
        o += L


def test_dit_ref_composed_equals_golden(golden):
    """the fp64 pieces composed (kr.dit_estimator) == the reference DiT's outputs in tests/golden/dit_small.npz (depth 2, the synthetic
    weights of test_flow3_gpu.py) within the export tolerance (rtol 1e-2, atol 1e-4)"""
    import numpy as np
    g = golden("dit_small")
    sd = oweights.synth_state_dict(odit.flow_param_shapes(2), 1986, odit.SYNTH_GAINS)
    W = kr.dit_weights(sd, 2)
    x, mask, mu, t, spks, cond = cases.estimator_case(T=130)
    tm = lambda a: a.transpose(1, 2).reshape(-1, a.shape[1])
    for streaming, key in ((False, "est_offline"), (True, "est_stream")):
        _, out = kr.dit_estimator(W, tm(x), tm(mu), tm(cond), spks, t.double(), [130, 130], streaming)
        np.testing.assert_allclose(out.numpy(), tm(torch.from_numpy(g[key])).double().numpy(), rtol=1e-2, atol=1e-4)


def test_dit_rounding_points():
    """rounding=True stores bf16 exactly at the DIT_ROUNDING points (and nowhere else); rounding=False nowhere"""
    sd = _dit_sd()
    W = kr.dit_weights(sd, 2)
    lens = [60]
    x, mu, cond, spks, t = _dit_case(lens, 4)
    is_b = lambda v: torch.equal(v, kr.bf16(v))
    mod = kr.dit_modulation(W, t[:1])["mod"]
    for rounding in (True, False):
        e = kr.dit_input_embedding(W, x, mu, cond, spks, lens, rounding)
        st = kr.dit_block(W, 0, e["x0"], mod, lens, 50, rounding)
        stored = [e["xa"], e["c1"], st["xn"], st["qkv"], st["qkv_rot"], st["att"], st["xn2"], st["h"]]
        assert all(is_b(v) == rounding for v in stored), rounding
        assert not any(is_b(v) for v in (e["h"], e["x0"], st["o"], st["x_mid"], st["f"], st["x_out"])), rounding


# share of the elements of the mutated result beyond the GPU bound (kr.DIT_TOL) that each mode claims; None: not caught in that mode.
# Measured on this case: fp32 >= 0.73 for every structural defect, 0.05 for the erf GELU, 0 for eps 1e-5; bf16 0.03 - 0.96 for the
# structural defects, 0 for the erf GELU and eps 1e-5.
DIT_CAUGHT = {
    "fp32": dict(rope_half=0.5, rope_all_heads=0.5, kpos_shift=0.5, adaln_swap=0.5, mod_neighbour=0.5, chunk48=0.5, chunk_edge=0.5,
                 silu_pos=0.5, time_div=0.5, gelu_erf=0.02, ln_eps=None),
    "bf16": dict(rope_half=0.1, rope_all_heads=0.3, kpos_shift=0.02, adaln_swap=0.5, mod_neighbour=0.5, chunk48=0.02, chunk_edge=0.01,
                 silu_pos=0.5, time_div=0.5, gelu_erf=None, ln_eps=None),
}


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_dit_mutations_exceed_bounds(precision):
    """each defect of kr.DIT_MUTATIONS, injected into the reference of its mode (exact for fp32, bf16-emulating for bf16), moves at
    least the stated share of the elements beyond the per-element bound test_dit_blocks_gpu.py holds the kernels to, on a ragged
    pair of 130 + 70 frames with the streaming mask; the defects a mode does not claim stay below a share of 0.1 there, so the claim
    list is exact.  The embedding defect is judged on x0, the others on block 0's output."""
    bf = precision == "bf16"
    sd = _dit_sd()
    W = kr.dit_weights(sd, 2)
    lens = [130, 70]
    x, mu, cond, spks, t = _dit_case(lens, 3)
    rms = lambda v: v.pow(2).mean(-1, keepdim=True).sqrt()
    tol = kr.DIT_TOL[precision]
    e = kr.dit_input_embedding(W, x, mu, cond, spks, lens, bf)
    mod = kr.dit_modulation(W, t)["mod"]
    st = kr.dit_block(W, 0, e["x0"], mod, lens, 50, bf)
    shares = {}
    for m in kr.DIT_MUTATIONS:
        if m == "silu_pos":
            d, scale, bound = kr.dit_input_embedding(W, x, mu, cond, spks, lens, bf, mutate=m)["x0"] - e["x0"], rms(e["x0"]), tol["embed"]
        else:
            mm = kr.dit_modulation(W, t, mutate=m)["mod"] if m == "time_div" else mod
            sm = kr.dit_block(W, 0, e["x0"], mm, lens, 50, bf, mutate=None if m == "time_div" else m)
            d, scale, bound = sm["x_out"] - st["x_out"], rms(st["x_out"] - st["x"]), tol["block"]
        shares[m] = ((d.abs() / scale) > bound).double().mean().item()
    print(precision, {k: round(v, 3) for k, v in shares.items()})
    for m, need in DIT_CAUGHT[precision].items():
        if need is None:
            assert shares[m] < 0.1, (m, shares[m])
        else:
            assert shares[m] >= need, (m, shares[m], need)


# ================================================================================================ CosyVoice2 flow references
FLOW_SMALL = oflow.FlowCfg(2, 2, 2, 2)


def _flow_w(cfg=FLOW_SMALL, seed=23):
    sd = kr.flow_test_state_dict(cfg, seed)
    return sd, kr.flow_weights(sd, cfg)


def _est_case(lens, seed):
    g = torch.Generator().manual_seed(seed)
    R = sum(lens)
    x, mu, cond = (kr.bf16(torch.rand(R, 80, generator=g) * 2 - 1) for _ in range(3))
    t = (0.05 + 0.9 * torch.rand(len(lens), generator=g)).double()
    return x, mu, cond, kr.bf16(torch.randn(len(lens), 80, generator=g)), t


@pytest.mark.parametrize("context_len", [0, 3])
@pytest.mark.parametrize("streaming", [False, True])
def test_flow_encoder_ref_equals_oracle(streaming, context_len):
    """kr.flow_encoder (exact; the units composed) == oracle.flow.encoder on every utterance of a ragged pack, with the look-ahead
    context passed to the oracle separately, as flow.py:259-261 passes it"""
    sd, W = _flow_w()
    lens = [37 + context_len, 5 + context_len, 60 + context_len]
    g = torch.Generator().manual_seed(3)
    tok = torch.randint(0, 6561, (sum(lens),), generator=g)
    _, got = kr.flow_encoder(W, tok, lens, streaming, context_len)
    o = oo = 0
    for L in lens:
        x = F.embedding(tok[o:o + L].long()[None], sd["input_embedding.weight"])
        Lo = L - context_len
        want = oflow.encoder(sd, x[:, :Lo], FLOW_SMALL, streaming, context=x[:, Lo:] if context_len else None)[0].double()
        assert (got[oo:oo + 2 * Lo] - want).abs().max().item() < 1e-4, L       # fp32 oracle, after_norm output of O(1)
        o += L
        oo += 2 * Lo


@pytest.mark.parametrize("streaming", [False, True])
def test_flow_estimator_ref_equals_oracle(streaming):
    """kr.flow_estimator (exact; the units, down_blocks.0.2, the skip and the tail composed) == oracle.flow.estimator on every sequence
    of a ragged pack, and a CFG pair (zero mu / spks / cond in its second sequence) sequence by sequence"""
    sd, W = _flow_w()
    lens = [70, 1, 51, 51]
    x, mu, cond, spks, t = _est_case(lens, 4)
    mu[-51:], cond[-51:], spks[-1] = 0.0, 0.0, 0.0
    x[-51:] = x[-102:-51]
    _, got = kr.flow_estimator(W, x, mu, cond, spks, t, lens, streaming)
    o = 0
    for b, L in enumerate(lens):
        cm = lambda a: a[o:o + L].t()[None]
        want = oflow.estimator(sd, cm(x), torch.ones(1, 1, L), cm(mu), t[b:b + 1].float(), spks[b:b + 1], cm(cond), FLOW_SMALL,
                               streaming)[0].t().double()
        assert (got[o:o + L] - want).abs().max().item() < 1e-4, (b, L)          # fp32 oracle on O(1) values
        o += L


@pytest.mark.parametrize("tag,cfg", [("small", oflow.FlowCfg(2, 1, 2, 2)), ("full", oflow.FlowCfg())])
def test_flow_ref_composed_equals_golden(golden, tag, cfg):
    """the fp64 pieces composed (kr.flow_encoder, kr.flow_estimator) == the reference flow's encoder and estimator outputs in
    tests/golden/flow_{small,full}.npz (the synthetic weights, cases.flow_case / cases.estimator_case) within the export tolerance
    (rtol 1e-2, atol 1e-4)"""
    import numpy as np
    gd = golden("flow_" + tag)
    sd = oweights.synth_state_dict(oflow.param_shapes(cfg), 1986, oflow.SYNTH_GAINS)
    W = kr.flow_weights(sd, cfg)
    token, ptok, _, _ = cases.flow_case()
    tok = torch.cat([ptok, token], 1)[0]
    _, h = kr.flow_encoder(W, tok, [tok.numel()], False)
    np.testing.assert_allclose(h.numpy(), gd["enc_offline"][0].astype(np.float64), rtol=1e-2, atol=1e-4)
    x, mask, mu, t, spks, cond = cases.estimator_case()
    T = x.shape[2]
    tm = lambda a: a.transpose(1, 2).reshape(-1, a.shape[1])
    for streaming, key in ((False, "est_offline"), (True, "est_stream")):
        _, out = kr.flow_estimator(W, tm(x), tm(mu), tm(cond), spks, t.double(), [T] * x.shape[0], streaming)
        np.testing.assert_allclose(out.numpy(), tm(torch.from_numpy(gd[key])).double().numpy(), rtol=1e-2, atol=1e-4)


def test_flow_rounding_points():
    """rounding=True stores bf16 exactly at the FLOW_ROUNDING points (and nowhere else); rounding=False nowhere"""
    sd, W = _flow_w()
    is_b = lambda v: torch.equal(v, kr.bf16(v))
    lens = [40, 9]
    x, mu, cond, spks, t = _est_case(lens, 5)
    temb = kr.est_time(W, t)["temb"]
    tok = torch.randint(0, 6561, (sum(lens),), generator=torch.Generator().manual_seed(6))
    for rounding in (True, False):
        inp = kr.est_pack(x + 1e-3, mu, cond, spks, lens, rounding)
        rn = kr.est_resnet(W, 0, inp, temb, lens, rounding)
        tb = kr.est_tblock(W, 0, 0, rn["x_out"], lens, 50, rounding)
        acts = {-1: inp, 0: kr.bf16(tb["x_out"]) if rounding else tb["x_out"]}
        xa = kr.est_stage_input(W, 1, acts, lens, rounding)
        stored = [inp, rn["h1"], tb["xn"], tb["qkv"], tb["att"], tb["xn3"], tb["ff"], xa]
        assert all(is_b(v) == rounding for v in stored), rounding
        assert not any(is_b(v) for v in (rn["c"], rn["h2"], rn["x_out"], tb["x_mid"], tb["x_out"], temb)), rounding
        e = kr.enc_embed(W, tok, lens, 3, rounding)
        el = kr.enc_layer(W, "encoder.encoders.0", e["x"], [37, 6], 25, rounding)
        up = kr.enc_upsample(W, el["x_out"], [37, 6], rounding)
        assert all(is_b(v) == rounding for v in (el["xn"], el["qkv"], el["pos"], el["att"], el["xn2"], el["ff"], up["up"])), rounding
        assert not any(is_b(v) for v in (e["h0"], e["x"], el["x_mid"], el["x_out"], up["y"])), rounding


def _flow_mutation_shares(precision):
    """share of the elements that each defect of kr.FLOW_MUTATIONS, injected into the reference of its mode (exact for fp32,
    bf16-emulating for bf16), moves beyond the per-element bound test_flow_blocks_gpu.py holds the kernels to (kr.FLOW_TOL), on a
    ragged pair with the streaming masks.  Each defect is judged on the unit it lives in, fed the unmutated reference's input, over
    the rms of that unit's contribution, as the GPU test judges the kernels."""
    bf = precision == "bf16"
    tol = kr.FLOW_TOL[precision]
    _, W = _flow_w()
    rms = lambda v: v.pow(2).mean(-1, keepdim=True).sqrt()
    share = lambda d, scale, bound: ((d.abs() / scale) > bound).double().mean().item()
    shares = {}
    # estimator: stage 1 (the first mid stage: down_blocks.0.2, resnet, block 0) and the up stage's resnet on the skip
    lens = [130, 70]
    x, mu, cond, spks, t = _est_case(lens, 3)
    temb = kr.est_time(W, t)["temb"]
    acts = {-1: kr.est_pack(x, mu, cond, spks, lens, bf)}
    g = torch.Generator().manual_seed(8)
    acts[0] = kr.bf16(torch.randn(sum(lens), 256, generator=g))
    acts[1], acts[2] = (kr.bf16(torch.randn(sum(lens), 256, generator=g)) for _ in range(2))
    nst = FLOW_SMALL.num_mid_blocks + 2
    for m in kr.FLOW_MUTATIONS["est"]:
        if m in ("chunk48", "chunk_edge", "gelu_tanh"):
            h = kr.est_resnet(W, 1, kr.est_stage_input(W, 1, acts, lens, bf), temb, lens, bf)["x_out"]
            ref, mut = (kr.est_tblock(W, 1, 0, h, lens, 50, bf, mutate=mm) for mm in (None, m))
            shares[m] = share(mut["x_out"] - ref["x_out"], rms(ref["x_out"] - ref["x"]), tol["est_block"])
        elif m == "skip_swap":
            ref, mut = (kr.est_resnet(W, nst - 1, kr.est_stage_input(W, nst - 1, acts, lens, bf, mutate=mm), temb, lens, bf)["x_out"]
                        for mm in (None, m))
            shares[m] = share(mut - ref, rms(ref), tol["est_resnet"])
        else:
            tm = kr.est_time(W, t, mutate=m)["temb"] if m == "time_div" else temb
            mm = None if m == "time_div" else m
            ref = kr.est_resnet(W, 1, kr.est_stage_input(W, 1, acts, lens, bf), temb, lens, bf)["x_out"]
            mut = kr.est_resnet(W, 1, kr.est_stage_input(W, 1, acts, lens, bf, mutate=mm), tm, lens, bf, mutate=mm)["x_out"]
            shares[m] = share(mut - ref, rms(ref), tol["est_resnet"])
    # encoder: the embedding, conformer layer 0 (token rate, chunk 25), the up-sampler
    tl = [60 + 3, 23 + 3]
    tok = torch.randint(0, 6561, (sum(tl),), generator=torch.Generator().manual_seed(9))
    lo = [60, 23]
    e = kr.enc_embed(W, tok, tl, 3, bf)["x"]
    for m in kr.FLOW_MUTATIONS["enc"]:
        if m in ("lookahead2", "no_sqrt"):
            mut = kr.enc_embed(W, tok, tl, 3, bf, mutate=m)["x"]
            shares["enc_" + m] = share(mut - e, rms(e), tol["enc_embed"])
        elif m == "up_pad3":
            ref, mut = (kr.enc_upsample(W, e, lo, bf, mutate=mm)["y"] for mm in (None, m))
            shares["enc_" + m] = share(mut - ref, rms(ref), tol["enc_up"])
        else:
            ref, mut = (kr.enc_layer(W, "encoder.encoders.0", e, lo, 25, bf, mutate=mm) for mm in (None, m))
            shares["enc_" + m] = share(mut["x_out"] - ref["x_out"], rms(ref["x_out"] - ref["x"]), tol["enc_layer"])
    return shares


# share of the elements beyond the GPU bound that each defect must move in each mode; None: not caught in that mode (its share stays
# under 0.1).  Measured on this case: fp32 0.6 - 1.0 for every structural defect and 0.94 for the tanh GELU, 0.002 and 0 for the
# LayerNorm eps changes; bf16 0.31 - 0.99 for the structural defects, 0 for the tanh GELU (the bf16 path's own GELU is the tanh form
# on a half-precision tanh, within 5e-4 of the erf) and for both eps changes.
FLOW_CAUGHT = {
    "fp32": dict(chunk48=0.5, chunk_edge=0.5, temb_neighbour=0.5, temb_before_mish=0.5, skip_swap=0.5, centred_pad=0.5, silu_for_mish=0.5,
                 gelu_tanh=0.5, time_div=0.5, ln_eps=None, enc_pos_bias_swap=0.5, enc_rel_shift=0.5, enc_chunk24=0.3, enc_lookahead2=0.5,
                 enc_up_pad3=0.5, enc_no_sqrt=0.5, enc_ln_eps=None),
    "bf16": dict(chunk48=0.2, chunk_edge=0.15, temb_neighbour=0.5, temb_before_mish=0.4, skip_swap=0.5, centred_pad=0.5, silu_for_mish=0.5,
                 gelu_tanh=None, time_div=0.4, ln_eps=None, enc_pos_bias_swap=0.5, enc_rel_shift=0.4, enc_chunk24=0.2, enc_lookahead2=0.5,
                 enc_up_pad3=0.5, enc_no_sqrt=0.5, enc_ln_eps=None),
}


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_flow_mutations_exceed_bounds(precision):
    """each defect of kr.FLOW_MUTATIONS moves at least the stated share of its unit's elements beyond the bound of its mode; the
    defects a mode does not claim stay under a share of 0.1, so the claim list is exact"""
    shares = _flow_mutation_shares(precision)
    print(precision, {k: round(v, 3) for k, v in shares.items()})
    assert set(FLOW_CAUGHT[precision]) == set(shares)
    for m, need in FLOW_CAUGHT[precision].items():
        if need is None:
            assert shares[m] < 0.1, (m, shares[m])
        else:
            assert shares[m] >= need, (m, shares[m], need)


# ------------------------------------------------------------------------------------------------ HiFT vocoders
def _hift_oracle_sd(causal):
    from oracle import hift_causal as ohc, weights as oweights
    return oweights.synth_state_dict((ohc if causal else ohift).param_shapes(), 1986, ohift.SYNTH_GAINS)


def test_hift_ref_composed_equals_oracle_and_goldens(golden):
    """the fp64 units composed (f0, source, body, ISTFT) against oracle.hift.decode and the reference's outputs hift_b2_t24 and
    hift_cache_source at fp32 tolerance; the fp32-emulating source against the goldens to 1e-7"""
    from oracle import cases
    sd = _hift_oracle_sd(False)
    W = kr.hift_weights(sd, False)
    g, gc = golden("hift_b2_t24"), golden("hift_cache_source")
    mel, noise, _ = cases.hift_case()
    for b in range(2):
        s = torch.from_numpy(g["source"][b, 0])
        outs, wav = kr.hift_decode(W, mel[b].t(), s)
        pre = ohift.decode(sd, mel[b:b + 1], s[None, None], return_pre_istft=True)[0].t().double()
        assert (outs[20] - pre).abs().max() < 5e-5
        assert (wav - ohift.decode(sd, mel[b:b + 1], s[None, None])[0].double()).abs().max() < 1e-5
        assert (wav - torch.from_numpy(g["decode"][b]).double()).abs().max() < 1e-5
        assert (kr.hift_f0(W, mel[b].t()) - torch.from_numpy(g["f0"][b]).double()).abs().max() < 2e-4
        f0 = torch.from_numpy(g["f0"][b])
        assert (kr.hift_source(W, f0, noise[b], emulate=True) - s.double()).abs().max() < 1e-7
        assert (kr.hift_source(W, f0, noise[b]) - s.double()).abs().max() < 1e-4
    _, wav = kr.hift_decode(W, mel[0].t(), torch.from_numpy(gc["source"][0, 0]))
    assert (wav - torch.from_numpy(gc["wav"][0]).double()).abs().max() < 1e-5


def test_hift3_ref_composed_equals_oracle_and_golden(golden):
    """the causal units against oracle.hift_causal.inference and the reference's hift_causal outputs, final and streaming; the
    fp64-fold f0 predictor equals the reference's float64 predictor to within fp32 rounding of its output"""
    from oracle import cases, hift_causal as ohc
    sd = _hift_oracle_sd(True)
    W = kr.hift_weights(sd, True)
    g = golden("hift_causal")
    mel, rand_ini, sine_noise = cases.hift_causal_case()
    m = mel[0].t()
    f0 = kr.hift_f0(W, m)
    assert (f0.float() - torch.from_numpy(g["f0_final"][0])).abs().max() == 0
    assert (f0[:21].float() - torch.from_numpy(g["f0_chunk"][0])).abs().max() == 0
    for fin, n, key in ((True, 24, "final"), (False, 21, "chunk")):
        s = kr.hift_source(W, torch.from_numpy(g[f"f0_{key}"][0]), sine_noise[0], emulate=True)
        assert s.shape[0] == 480 * n and (s - torch.from_numpy(g[f"source_{key}"][0, 0]).double()).abs().max() < 1e-7
        _, wav = kr.hift_decode(W, m, torch.from_numpy(g[f"source_{key}"][0, 0]), finalize=fin)
        assert (wav - torch.from_numpy(g[f"wav_{key}"][0]).double()).abs().max() < 2e-5, key
        ow, _ = ohc.inference(sd, mel, rand_ini, sine_noise, fin)
        assert (wav - ow[0].double()).abs().max() < 2e-5, key


def test_hift_windows_equal_whole_sequence():
    """a unit computed on a window of a sequence's rows widened by kernel_refs' halo equals the whole-sequence composition on the
    window's frames (head, tail, interior), final, causal and causal streaming; and a one-row defect in a read-out is seen"""
    for causal in (False, True):
        W = kr.hift_weights(kr.hift_test_state_dict(7, causal), causal)
        g = torch.Generator().manual_seed(3)
        T = 44
        mel = torch.randn(T, 80, generator=g) * 2 - 5
        s = torch.tanh(torch.randn(480 * T, generator=g))
        for fin in ((True, False) if causal else (True,)):
            Tb = T if fin else T - 7
            K = kr.hift_body(W, mel, s[:480 * (T if fin else T - 3)], Tb, "fp16")
            res = kr.hift_unit_refs(W, K, mel, Tb, kr.hift_windows(Tb, (20,), 6), "fp16")
            assert [sorted(w) for w in res] == [list(range(1, 21))] * 3
            assert max(kr.hift_ratio(r, k) for w in res for r, k in w.values()) == 0.0
            K[12] = K[12].clone()
            K[12][40 * 21] += 1.0                          # one row of level 1, frame 21
            res = kr.hift_unit_refs(W, K, mel, Tb, [(18, 24)], "fp16")
            assert kr.hift_ratio(*res[0][13]) > 1e-3


def test_hift_emulated_source_matches_oracle():
    """the fp32-emulating source equals oracle.hift.sine_source (torch's CPU arithmetic, which the kernel follows) to 1e-6 at every
    sample at T = 24, 500 and 1500 - no phase-ulp mismatch - while the separately rounded interpolation l0 p0 + l1 p1 (what the
    kernel would compute without FMA contraction) misses it on a growing number of samples and the exact fp64 source differs by up
    to the 1-ulp phase effect"""
    sd = _hift_oracle_sd(False)
    W = kr.hift_weights(sd, False)
    for T, n_unfused in ((24, 10000), (500, 300000), (1500, 1000000)):
        g = torch.Generator().manual_seed(T)
        f0 = 80 + 320 * torch.rand(T, generator=g)
        noise = torch.randn(480 * T, 9, generator=g)
        o = ohift.sine_source(sd, f0[None], noise[None])[0, 0].double()
        d = (o - kr.hift_source(W, f0, noise, emulate=True)).abs()
        assert int((d > 1e-6).sum()) == 0, (T, d.max().item())
        ph = kr.hift_phase(f0, emulate=True).numpy().astype(np.float32)
        i0, i1, l0, l1 = kr._interp_index(480 * T, T)
        sep = ((l0[:, None] * ph[i0]).astype(np.float32) + (l1[:, None] * ph[i1]).astype(np.float32)).astype(np.float32)
        fused = kr.hift_sample_phase(torch.from_numpy(ph.astype(np.float64)), False, emulate=True).numpy()
        n_diff = int((sep != fused).sum())
        print(f"T={T}: {n_diff} of {sep.size} phase samples differ without contraction; exact source differs by "
              f"{(o - kr.hift_source(W, f0, noise)).abs().max().item():.3g}")
        assert n_diff >= n_unfused, (T, n_diff)
        assert (o - kr.hift_source(W, f0, noise)).abs().max().item() <= kr.hift_source_ulp_bound(W, f0)


_HIFT_MUT_UNIT = dict(lrelu_post="level_out", no_reflect="ups", reflect_back="ups", down_pad="source_branch", poly_phase="ups",
                      snake_swap="resblock", dil1="resblock", no_div3="level_out", hann_sym="stft", no_env="istft", phase_x="source",
                      clip_first="istft", uv_ge="source", pre_left="conv_pre", f0_look2="f0")


def _hift_mutation_shares(mode):
    """share of the elements that each defect of kr.HIFT_MUTATIONS, injected into the reference of its mode (exact for fp32, rounding
    to IEEE half for f16, to bf16 for bf16), moves beyond the bound test_hift_blocks_gpu.py holds that unit to (kr.HIFT_TOL).  A
    defect lives in one unit, so the first read-out it changes is that unit fed the unmutated inputs; it is judged there, per element
    over the reference row's rms (istft and source: absolute; f0: in fp32 ulps, against one ulp)."""
    rnd = {"fp32": None, "f16": "fp16", "bf16": "bf16"}[mode]
    tol = kr.HIFT_TOL[mode]
    shares = {}
    g = torch.Generator().manual_seed(12)
    T = 14
    mel = torch.randn(T, 80, generator=g) * 2 - 5
    s = torch.tanh(3 * torch.randn(480 * T, generator=g))
    f0 = torch.full((T,), 10.0)
    f0[T // 2:] = 150.0
    noise = torch.randn(480 * T, 9, generator=g)
    for causal in (False, True):
        W = kr.hift_weights(kr.hift_test_state_dict(5, causal, clip=True), causal)
        ref, wav = kr.hift_decode(W, mel, s, rounding=rnd)
        for m in kr.HIFT_MUTATIONS:
            unit = _HIFT_MUT_UNIT[m]
            if (m in ("pre_left", "f0_look2")) != causal:
                continue
            if unit == "f0":
                a, b = kr.hift_f0(W, mel), kr.hift_f0(W, mel, mutate=m)
                r = a.float().abs()
                shares[m] = (((b - a).abs() / (torch.nextafter(r, r + 1) - r).double()) > 1.0).double().mean().item()
            elif unit == "source":
                a, b = kr.hift_source(W, f0, noise), kr.hift_source(W, f0, noise, mutate=m)
                shares[m] = ((b - a).abs() > kr.HIFT_TOL["source"]).double().mean().item()
            elif unit == "istft":
                a, b = kr.hift_istft(ref[20]), kr.hift_istft(ref[20], mutate=m)
                shares[m] = ((b - a).abs() > tol["istft"]).double().mean().item()
            else:
                mut, _ = kr.hift_decode(W, mel, s, rounding=rnd, mutate=m)
                u = next(i for i in range(21) if mut[i].shape != ref[i].shape or not torch.equal(mut[i], ref[i]))
                # a resblock defect shows first in the source branch, whose source resblock comes first
                assert kr.HIFT_UNIT_GROUP.get(u, "stft") in (unit, "source_branch" if unit == "resblock" else unit), (m, u)
                unit = kr.HIFT_UNIT_GROUP.get(u, "stft")
                a, b = ref[u], mut[u]
                if a.shape != b.shape:
                    n = min(a.shape[0], b.shape[0])
                    a, b = a[:n], b[:n]
                rms = a.pow(2).mean(-1, keepdim=True).sqrt().clamp_min(1e-30)
                shares[("c_" if causal else "") + m] = ((b - a).abs() / rms > tol[unit]).double().mean().item()
    return shares


# share of the elements beyond the GPU bound that each defect must move, in every mode (fp32, f16, bf16): all of them are caught in
# all three.  Measured on this case (fp32 / f16 / bf16): lrelu_post 0.52 / 0.50 / 0.44, reflect_back, down_pad, poly_phase, dil1,
# no_div3 0.94 - 1.0, snake_swap 1.0 / 0.98 / 0.84, hann_sym 0.89 / 0.85 / 0.59, causal pre_left 1.0 / 0.96 / 0.75; mode-independent:
# no_reflect 6e-4 (the one front row of 1681 it changes, changed beyond the bound), no_env 0.10 and clip_first 0.27 (most samples of
# the clip=True waveform sit on the +-0.99 clamp, where neither defect shows), phase_x and uv_ge 0.5 (the voiced half of the crafted
# f0; uv_ge on the frames at exactly 10 Hz), f0_look2 1.0 (in fp32 ulps of the fp64 predictor).
HIFT_CAUGHT = dict(lrelu_post=0.25, no_reflect=5e-4, reflect_back=0.5, down_pad=0.5, poly_phase=0.5, snake_swap=0.5, dil1=0.5,
                   no_div3=0.5, hann_sym=0.3, no_env=0.05, phase_x=0.25, clip_first=0.1, uv_ge=0.25, c_pre_left=0.3, f0_look2=0.5)


@pytest.mark.parametrize("mode", ["fp32", "f16", "bf16"])
def test_hift_mutations_exceed_bounds(mode):
    """each defect of kr.HIFT_MUTATIONS moves at least the stated share of its unit's elements beyond the bound of its mode"""
    shares = _hift_mutation_shares(mode)
    print(mode, {k: round(v, 4) for k, v in shares.items()})
    assert set(HIFT_CAUGHT) == set(shares)
    for m, need in HIFT_CAUGHT.items():
        assert shares[m] >= need, (m, shares[m], need)
