"""Timing probe of the LM decode weight-streaming GEMM: mean device time per launch and the weight bandwidth it implies."""
import os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cosyvoice_b200 import cvk
c = cvk.Context(0, "bf16", 2.0)
g = torch.Generator().manual_seed(0)
for (N, K) in ((1152, 896), (9728, 896), (896, 4864), (6564, 896)):
    x = torch.randn(32, K, generator=g)
    w = torch.randn(N, K, generator=g) / K ** 0.5
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        out, ms = c.linear_small(x, w, None, iters=20)
    ref = x.bfloat16().float() @ w.bfloat16().float().t()
    err = (out.cpu() - ref).abs().max().item()
    print(f"N={N} K={K}: {ms*1000:.1f} us/iter  ({N*K*2/ms/1e6:.0f} GB/s weights)  maxerr {err:.3g}")
