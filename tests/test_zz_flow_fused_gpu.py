"""GPU: the whole flow (encoder, 10 Euler steps of the estimator with CFG) on a ragged batch, small and full-size estimator, offline and
streaming, with the fused feed-forward of the estimator's transformer blocks (option "flow_fused_ff" = 1) and with the unfused
LayerNorm / conv-GEMM launches (= 0): identical mel.  Kept apart from test_flow_fused_gpu.py and named to run late, as the other
full-size tests: loading the full-size flow weights holds device memory for the rest of the session."""
import pytest
import torch

from test_flow_gpu import model

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("tag", ["small", "full"])
def test_flow_fused_ff_bit_identical(tag):
    """the whole flow (encoder, 10 Euler steps of the estimator with CFG) on a ragged batch, offline and streaming, with the fused
    feed-forward and with the unfused launches"""
    c, sd, cfg = model("bf16", tag)
    g = torch.Generator().manual_seed(5)
    n_tok = [130, 57, 211]
    toks = torch.cat([torch.randint(0, 6561, (n + 20,), generator=g, dtype=torch.int32) for n in n_tok])
    tl = [n + 20 for n in n_tok]
    pf = torch.randn(3 * 40, 80, generator=g)
    emb = torch.randn(3, 192, generator=g)
    for streaming in (False, True):
        outs = {}
        for on in (1, 0):
            c.set_option("flow_fused_ff", on)
            try:
                mel, lens = c.flow_inference(toks, tl, pf, [40] * 3, emb, streaming=streaming)
                outs[on] = mel.clone()
            finally:
                c.set_option("flow_fused_ff", 1)
        d = (outs[1] - outs[0]).abs()
        print(f"{tag} streaming={streaming}: mel {tuple(outs[1].shape)}, max |d| {d.max().item():.3g}, mean |d| {d.mean().item():.3g}")
        assert torch.isfinite(outs[1]).all()
        assert torch.equal(outs[1], outs[0]), (d.max().item(), d.mean().item())
