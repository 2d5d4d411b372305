"""GPU: the fused feed-forward of the flow estimator's transformer blocks (ffn_fused_kernel, gemm_tc.cu; option "flow_fused_ff").

 A. cvk_op_flow_ff against an fp64 restatement of LN3 -> ff1 -> GELU -> ff2 -> residual -> next LN1 (or the plain bf16 copy), on ragged
    batches with gap rows, row counts that are not multiples of the 128-row tile and a single short sequence.  Gap rows of x carry
    large values: a tile that leaked them into a sequence would show an O(1) error, and they must come out exactly zero.
 B. the same op with the option off (the LayerNorm / conv-GEMM launches of the unfused path): identical bits.
The whole flow with the option on and off is compared in test_zz_flow_fused_gpu.py."""
import math

import pytest
import torch

import kernel_refs as kr
from gpu_util import ctx, maxdiff

pytestmark = pytest.mark.gpu

C, HID = 256, 1024
LAYOUTS = {                                   # rows, [(start, len)]
    "ragged": (300, [(3, 100), (110, 57), (175, 120)]),
    "multi_tile": (1000, [(8, 650), (666, 326)]),
    "short": (37, [(2, 30)]),
    "one_row": (5, [(4, 1)]),
}


def _operands(rows, seqs, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, C, generator=g) * 2.0 + 0.5
    valid = torch.zeros(rows, dtype=torch.bool)
    for s, n in seqs:
        valid[s:s + n] = True
    x[~valid] = 1e3 * torch.randn(int((~valid).sum()), C, generator=g)
    w = dict(ln3_g=1 + 0.1 * torch.randn(C, generator=g), ln3_b=0.1 * torch.randn(C, generator=g),
             w1=kr.bf16(torch.randn(HID, C, generator=g) * C ** -0.5), b1=0.1 * torch.randn(HID, generator=g),
             w2=kr.bf16(torch.randn(C, HID, generator=g) * HID ** -0.5), b2=0.1 * torch.randn(C, generator=g),
             ln_g=1 + 0.1 * torch.randn(C, generator=g), ln_b=0.1 * torch.randn(C, generator=g))
    return x, valid, w


def _ln64(x, g, b):
    m = x.mean(1, keepdim=True)
    v = ((x - m) ** 2).mean(1, keepdim=True)
    return (x - m) / torch.sqrt(v + 1e-5) * g.double() + b.double()


def _run(c, x, seqs, w, next_ln):
    kw = dict(ln_g=w["ln_g"], ln_b=w["ln_b"]) if next_ln else {}
    xo, out = c.flow_ff(x, [s for s, _ in seqs], [n for _, n in seqs], w["ln3_g"], w["ln3_b"], w["w1"], w["b1"], w["w2"], w["b2"], **kw)
    return xo.cpu(), out.cpu()


@pytest.mark.parametrize("next_ln", [True, False], ids=["ln1", "out2"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_flow_ff_vs_fp64(layout, next_ln):
    rows, seqs = LAYOUTS[layout]
    x, valid, w = _operands(rows, seqs, seed=rows + 7 * len(seqs))
    c = ctx("bf16")
    xo, out = _run(c, x, seqs, w, next_ln)
    assert torch.isfinite(xo).all() and torch.isfinite(out).all()
    assert (xo[~valid] == 0).all() and (out[~valid] == 0).all()
    xv = x[valid].double()
    xn = kr.bf16(_ln64(xv, w["ln3_g"], w["ln3_b"]))                 # the bf16 operand of ff1
    w1, w2 = w["w1"].double(), w["w2"].double()
    a = xn @ w1.t() + w["b1"].double()
    h = kr.bf16(0.5 * a * (1 + torch.erf(a / math.sqrt(2))))        # exact-erf GELU, rounded to the bf16 operand of ff2
    y = xv + h @ w2.t() + w["b2"].double()
    # Error budget of an element of y:
    #  - systematic: the kernel's tanh-form GELU on the half-precision tanh is within 5e-4 + 2.5e-4 |a| of the exact one
    #    (common.cuh), summed with |w2| over the 1024 hidden units;
    #  - roundings of independent sign: where the kernel's fp32 value of an xn or h element sits on the other side of a bf16 tie
    #    from the fp64 one, the two differ by one ulp (<= 2^-7 relative); counted as a standard deviation of 2^-8 relative per
    #    element, a hidden unit carries sigma_h = 2^-8 |h| + 1.13 (GELU slope) 2^-8 sqrt(xn^2 w1^2), and y is allowed six standard
    #    deviations sqrt(sigma_h^2 w2^2);
    #  - the fp32 accumulation of 1024 products and the two fp32 additions: 2^-16 (|h| |w2|^T) + 2^-22 |y|.
    # On these operands the bound is ~0.06 while a dropped 64-wide hidden chunk moves most outputs by more (median ~0.11).
    sh = 2.0 ** -8 * h.abs() + 1.13 * 2.0 ** -8 * torch.sqrt((xn ** 2) @ (w1 ** 2).t())
    bound = ((5e-4 + 2.5e-4 * a.abs()) @ w2.abs().t() + 6 * torch.sqrt((sh ** 2) @ (w2 ** 2).t()) + 2.0 ** -16 * (h.abs() @ w2.abs().t())
             + 2.0 ** -22 * y.abs() + 1e-6)
    d = (xo[valid].double() - y).abs()
    print(f"{layout} {'ln1' if next_ln else 'out2'}: x max |d| {d.max().item():.3g} (bound median {bound.median().item():.3g}), "
          f"mean |d| {d.mean().item():.3g}")
    assert (d <= bound).all(), (d - bound).max().item()
    # the second output is computed from the kernel's own x
    if next_ln:
        ref = _ln64(xo[valid].double(), w["ln_g"], w["ln_b"])
        # fp32 LayerNorm (error ~1e-6 |.|) rounded to bf16: within one bf16 ulp (2^-7 relative) of the fp64 value
        assert ((out[valid].double() - ref).abs() <= 2.0 ** -7 * ref.abs() + 1e-5).all()
    else:
        assert torch.equal(out, kr.bf16(xo))


@pytest.mark.parametrize("next_ln", [True, False], ids=["ln1", "out2"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_flow_ff_fused_equals_unfused(layout, next_ln):
    """the fused kernel performs the unfused path's operations in the same order: identical bits"""
    rows, seqs = LAYOUTS[layout]
    x, valid, w = _operands(rows, seqs, seed=3 * rows + len(seqs))
    c = ctx("bf16")
    res = {}
    for on in (1, 0):
        c.set_option("flow_fused_ff", on)
        try:
            res[on] = _run(c, x, seqs, w, next_ln)
        finally:
            c.set_option("flow_fused_ff", 1)
    assert torch.equal(res[1][0], res[0][0]), maxdiff(res[1][0], res[0][0])
    assert torch.equal(res[1][1], res[0][1]), maxdiff(res[1][1], res[0][1])
