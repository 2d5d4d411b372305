"""GPU: per-op parity of the conv-GEMM kernels (fp32 CUDA-core and bf16 wgmma/TMA) and the attention kernel
against plain torch fp32 on the CPU, through the C ABI."""
import pytest
import torch
import torch.nn.functional as F

from gpu_util import ctx, maxdiff

pytestmark = pytest.mark.gpu


def _ref_conv(xs, w, b, dil, shift0, act):
    outs = []
    taps = w.shape[2]
    for x in xs:                                     # x [T,K]
        T = x.shape[0]
        left = -shift0
        right = (taps - 1) * dil + shift0
        xp = F.pad(x.t().unsqueeze(0), (max(left, 0), max(right, 0)))
        y = F.conv1d(xp, w, b, dilation=dil)
        y = y[0, :, max(-left, 0): max(-left, 0) + T].t() if left < 0 else y[0, :, :T].t()
        outs.append(y)
    y = torch.cat(outs, 0)
    return {"none": lambda v: v, "gelu": F.gelu, "silu": F.silu, "mish": F.mish, "elu": F.elu,
            "lrelu": lambda v: F.leaky_relu(v, 0.1), "tanh": torch.tanh}[act](y)


CASES = [
    # K, N, taps, dil, shift0, act, lens
    (256, 256, 3, 1, -2, "mish", [70, 129, 5]),        # estimator causal conv (flow/decoder.py:36-62)
    (320, 256, 1, 1, 0, "none", [200]),                # res_conv 1x1
    (256, 1024, 1, 1, 0, "gelu", [300, 17]),           # ff.net.0 (GELU)
    (1024, 256, 1, 1, 0, "none", [260]),
    (64, 64, 11, 5, -25, "none", [333, 64]),           # HiFT ResBlock k11 d5 (generator.py:63-76)
    (128, 128, 7, 3, -9, "silu", [500]),
    (80, 512, 7, 1, -3, "lrelu", [50, 31]),            # conv_pre (K=80: TMA zero-fills the K tail)
    (512, 80, 1, 1, 0, "none", [140]),                 # encoder_proj / final_proj (N=80)
    (896, 1152, 1, 1, 0, "none", [139]),               # LM qkv
    (512, 512, 4, 1, 0, "lrelu", [40, 9]),             # pre-lookahead conv1 (right-looking)
]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=[f"K{c[0]}N{c[1]}t{c[2]}d{c[3]}" for c in CASES])
def test_conv_gemm(precision, case):
    K, N, taps, dil, shift0, act, lens = case
    g = torch.Generator().manual_seed(K * 131 + N)
    xs = [torch.randn(T, K, generator=g) for T in lens]
    w = torch.randn(N, K, taps, generator=g) / (K * taps) ** 0.5
    b = torch.randn(N, generator=g) * 0.1
    ref = _ref_conv(xs, w, b, dil, shift0, act)
    c = ctx(precision)
    out = c.conv1d(torch.cat(xs, 0), lens, w, b, dil=dil, shift0=shift0, act=act)
    torch.cuda.synchronize()
    tol = 2e-4 if precision == "fp32" else 3e-2        # bf16 operands: 2^-8 relative per product, fp32 accumulate
    assert maxdiff(out, ref) < tol, (precision, case, maxdiff(out, ref))


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_conv_gemm_tc_matches_simt_on_same_operands(precision):
    """bf16 mode: the wgmma kernel and the CUDA-core kernel fed the same bf16 operands agree to fp32 rounding."""
    if precision == "fp32":
        pytest.skip("single path")
    c = ctx("bf16")
    g = torch.Generator().manual_seed(5)
    lens = [257, 40]
    x = torch.randn(sum(lens), 256, generator=g)
    w = torch.randn(512, 256, 3, generator=g) / 27
    b = torch.randn(512, generator=g)
    a = c.conv1d(x, lens, w, b, shift0=-2, act="none")
    c.set_option("use_tc", 0)
    try:
        s = c.conv1d(x, lens, w, b, shift0=-2, act="none")
    finally:
        c.set_option("use_tc", 1)
    assert maxdiff(a, s) < 1e-3


def _ref_attention(q, k, v, lens, H, chunk, scale):
    outs, o = [], 0
    for L in lens:
        qq, kk, vv = (t[o:o + L].view(L, H, 64).transpose(0, 1) for t in (q, k, v))
        s = qq @ kk.transpose(1, 2) * scale
        if chunk > 0:
            pos = torch.arange(L)
            m = pos[None, :] < ((pos // chunk + 1) * chunk)[:, None]
            s = s.masked_fill(~m[None], float("-inf"))
        outs.append((torch.softmax(s, -1) @ vv).transpose(0, 1).reshape(L, H * 64))
        o += L
    return torch.cat(outs, 0)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("chunk", [0, 50])
def test_attention(precision, chunk):
    g = torch.Generator().manual_seed(11)
    lens, H = [130, 33, 64], 8
    q, k, v = (torch.randn(sum(lens), H * 64, generator=g) for _ in range(3))
    ref = _ref_attention(q, k, v, lens, H, chunk, 0.125)
    out = ctx(precision).attention(q, k, v, lens, H, chunk, 0.125)
    torch.cuda.synchronize()
    assert maxdiff(out, ref) < (2e-5 if precision == "fp32" else 3e-2)


@pytest.mark.parametrize("chunk", [0, 50])
def test_attention_tcgen05_long_ragged(chunk):
    """bf16 mode runs the wgmma attention kernel: multi-tile sequences, ragged lengths, block-causal mask."""
    g = torch.Generator().manual_seed(13)
    lens, H = [650, 129, 300, 7], 8
    q, k, v = (torch.randn(sum(lens), H * 64, generator=g) for _ in range(3))
    q = q * 1.5
    ref = _ref_attention(q.bfloat16().float(), k.bfloat16().float(), v.bfloat16().float(), lens, H, chunk, 0.125)
    c = ctx("bf16")
    out = c.attention(q, k, v, lens, H, chunk, 0.125)
    c.set_option("use_tc_attn", 0)
    try:
        simt = c.attention(q, k, v, lens, H, chunk, 0.125)
    finally:
        c.set_option("use_tc_attn", 1)
    torch.cuda.synchronize()
    assert maxdiff(simt, ref) < 2e-2
    assert maxdiff(out, ref) < 2e-2, maxdiff(out, ref)      # P rounded to bf16 before P.V


@pytest.mark.parametrize("case", [(256, 384, 3, -2, "mish"), (256, 1024, 1, 0, "gelu"), (1024, 256, 1, 0, "none")],
                         ids=["K256N384t3", "K256N1024", "K1024N256"])
def test_conv_gemm_persistent_tiles(case):
    """More output tiles than SMs: the persistent wgmma kernel (one CTA per SM, operand ring running across tile boundaries)
    == the one-tile-per-CTA launch bit for bit, and == torch fp32 to bf16 operand rounding."""
    K, N, taps, shift0, act = case
    g = torch.Generator().manual_seed(K + N)
    lens = [5000, 3333, 4100, 129]                      # ~99 row tiles x 2-8 column tiles, ragged tails
    xs = [torch.randn(T, K, generator=g) for T in lens]
    w = torch.randn(N, K, taps, generator=g) / (K * taps) ** 0.5
    b = torch.randn(N, generator=g) * 0.1
    c = ctx("bf16")
    x = torch.cat(xs, 0)
    a = c.conv1d(x, lens, w, b, shift0=shift0, act=act)
    outs = []
    for mode in (0, 1):                                  # one tile per CTA; persistent with 8 epilogue warps (default: 16)
        c.set_option("tc_persist", mode)
        try:
            outs.append(c.conv1d(x, lens, w, b, shift0=shift0, act=act))
        finally:
            c.set_option("tc_persist", 2)
    assert torch.equal(a, outs[0]) and torch.equal(a, outs[1]), (maxdiff(a, outs[0]), maxdiff(a, outs[1]))
    assert maxdiff(a, _ref_conv(xs, w, b, 1, shift0, act)) < 3e-2
