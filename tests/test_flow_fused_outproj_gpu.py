"""GPU: the attention output projection folded into the fused feed-forward of the flow estimator's transformer blocks (ffn_fused_kernel,
gemm_tc.cu; option "flow_fused_ff").

cvk_op_flow_ff with att, wo and bo: x <- valid(r) ? x + bo + att wo^T : 0, then the feed-forward half of the block and the next block's
LN1 (or the plain bf16 copy).  The fused launch, the unfused path (out-projection conv-GEMM, LN3, ff1, ff2 launches) and the separate
out-projection conv-GEMM op followed by the feed-forward op all give identical bits: on ragged batches with gap rows, row counts that
are not multiples of the 128-row tile, sequences shorter than a tile and the streaming sessions' 50-row chunks behind 2 gap rows.  Gap
rows of x and att carry large values: a tile that leaked them into a sequence would show, and they must come out exactly zero.  The
feed-forward alone (no att) is tested in test_flow_fused_gpu.py, the whole flow with the option on and off in test_zz_flow_fused_gpu.py."""
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
    "stream_chunk": (8 * 52, [(52 * i + 2, 50) for i in range(8)]),
}


def _operands(rows, seqs, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, C, generator=g) * 2.0 + 0.5
    valid = torch.zeros(rows, dtype=torch.bool)
    for s, n in seqs:
        valid[s:s + n] = True
    x[~valid] = 1e3 * torch.randn(int((~valid).sum()), C, generator=g)
    att = torch.randn(rows, 2 * C, generator=g)
    att[~valid] = 1e3 * torch.randn(int((~valid).sum()), 2 * C, generator=g)   # whatever the attention left in gap rows must not leak
    w = dict(ln3_g=1 + 0.1 * torch.randn(C, generator=g), ln3_b=0.1 * torch.randn(C, generator=g),
             w1=kr.bf16(torch.randn(HID, C, generator=g) * C ** -0.5), b1=0.1 * torch.randn(HID, generator=g),
             w2=kr.bf16(torch.randn(C, HID, generator=g) * HID ** -0.5), b2=0.1 * torch.randn(C, generator=g),
             ln_g=1 + 0.1 * torch.randn(C, generator=g), ln_b=0.1 * torch.randn(C, generator=g),
             wo=kr.bf16(torch.randn(C, 2 * C, generator=g) * (2 * C) ** -0.5), bo=0.1 * torch.randn(C, generator=g))
    return x, att, valid, w


def _run(c, x, seqs, w, next_ln, att=None):
    kw = dict(ln_g=w["ln_g"], ln_b=w["ln_b"]) if next_ln else {}
    if att is not None:
        kw.update(att=att, wo=w["wo"], bo=w["bo"])
    xo, out = c.flow_ff(x, [s for s, _ in seqs], [n for _, n in seqs], w["ln3_g"], w["ln3_b"], w["w1"], w["b1"], w["w2"], w["b2"], **kw)
    return xo.cpu(), out.cpu()


@pytest.mark.parametrize("next_ln", [True, False], ids=["ln1", "out2"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_flow_ff_out_proj_fused_equals_unfused(layout, next_ln):
    """x + bo + att wo^T folded into the fused launch: the same bits as the out-projection conv-GEMM and the unfused feed-forward"""
    rows, seqs = LAYOUTS[layout]
    x, att, valid, w = _operands(rows, seqs, seed=5 * rows + len(seqs))
    c = ctx("bf16")
    res = {}
    for on in (1, 0):
        c.set_option("flow_fused_ff", on)
        try:
            res[on] = _run(c, x, seqs, w, next_ln, att)
        finally:
            c.set_option("flow_fused_ff", 1)
    # the two launches the fold replaces, as separate ops: out projection with the residual (bf16 operands, fp32 x), then the fused FF
    x1, _ = c.conv_gemm(att, [s for s, _ in seqs], [n for _, n in seqs], w["wo"][:, :, None], bias=w["bo"], operand="bf16", resid_is_out=True,
                        out=x, out_dtype="fp32")
    ref = _run(c, x1, seqs, w, next_ln)
    xo, out = res[1]
    assert torch.isfinite(xo).all() and torch.isfinite(out).all()
    assert (xo[~valid] == 0).all() and (out[~valid] == 0).all()
    assert not torch.equal(xo[valid], _run(c, x, seqs, w, next_ln)[0][valid])   # the projection did something
    for name, (rx, ro) in (("unfused", res[0]), ("conv_gemm + flow_ff", ref)):
        assert torch.equal(xo, rx), (name, maxdiff(xo, rx))
        assert torch.equal(out, ro), (name, maxdiff(out, ro))
