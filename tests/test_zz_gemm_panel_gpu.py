"""GPU: the whole flow (encoder, 10 Euler steps of the estimator with CFG) on a ragged batch, small and full-size estimator, offline and
chunk-50 streaming, with the estimator's qkv projections on the row-panel GEMM (option "flow_qkv_panel" = 2: at any row count; 1: by
the row count, the default) and on the generic conv-GEMM (= 0): identical mel.  Kept apart from test_gemm_panel_gpu.py and named to
run late, as the other full-size tests: loading the full-size flow weights holds device memory for the rest of the session."""
import pytest
import torch

from test_flow_gpu import model

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("tag", ["small", "full"])
def test_flow_qkv_panel_bit_identical(tag):
    c, sd, cfg = model("bf16", tag)
    g = torch.Generator().manual_seed(11)
    n_tok = [130, 57, 211]
    toks = torch.cat([torch.randint(0, 6561, (n + 20,), generator=g, dtype=torch.int32) for n in n_tok])
    tl = [n + 20 for n in n_tok]
    pf = torch.randn(3 * 40, 80, generator=g)
    emb = torch.randn(3, 192, generator=g)
    for streaming in (False, True):
        outs, launches = {}, {}
        for opt in (2, 1, 0):
            c.set_option("flow_qkv_panel", opt)
            try:
                n0 = c.launch_count()
                mel, lens = c.flow_inference(toks, tl, pf, [40] * 3, emb, streaming=streaming)
                launches[opt] = c.launch_count() - n0
                outs[opt] = mel.clone()
            finally:
                c.set_option("flow_qkv_panel", 1)
        assert torch.isfinite(outs[0]).all()
        assert launches[2] == launches[0] == launches[1]          # the panel kernel replaces launches one for one
        for opt in (2, 1):
            d = (outs[opt] - outs[0]).abs()
            print(f"{tag} streaming={streaming} flow_qkv_panel={opt}: mel {tuple(outs[0].shape)}, max |d| {d.max().item():.3g}")
            assert torch.equal(outs[opt], outs[0]), (opt, d.max().item(), d.mean().item())
