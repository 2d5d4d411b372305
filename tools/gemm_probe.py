"""Times the wgmma conv-GEMM on the estimator / HiFT shapes: one CTA per tile vs persistent CTAs (one per SM),
bf16 outputs.  CUDA events around `op_iters` back-to-back launches inside cvk_op_conv1d."""
import os, sys, itertools
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cosyvoice_b200 import cvk
c = cvk.Context(0, "bf16", 12.0)
c.set_option("op_iters", 10)
g = torch.Generator().manual_seed(0)
SHAPES = [  # name, rows, K, N, taps, dil, act
    ("est ff1 gelu", 40064, 256, 1024, 1, 1, "gelu"), ("est ff1 none", 40064, 256, 1024, 1, 1, "none"), ("est ff1 silu", 40064, 256, 1024, 1, 1, "silu"),
    ("est ff1 tanh", 40064, 256, 1024, 1, 1, "tanh"), ("est ff2", 40064, 1024, 256, 1, 1, "none"), ("est qkv", 40064, 256, 1536, 1, 1, "none"),
    ("est conv k3", 40064, 256, 256, 3, 1, "mish"), ("est to_out", 40064, 512, 256, 1, 1, "none"),
    ("hift L1 k7", 130000, 256, 256, 7, 3, "silu"), ("hift L2 k3", 650000, 128, 128, 3, 1, "none")]
only = sys.argv[1:]
for name, rows, K, N, taps, dil, act in SHAPES:
    if only and not any(o in name for o in only):
        continue
    x = torch.randn(rows, K, generator=g)
    w = torch.randn(N, K, taps, generator=g) / (K * taps) ** 0.5
    b = torch.randn(N, generator=g)
    res = []
    for obf, persist in itertools.product((1,), (0, 2)):
        c.set_option("op_out_bf16", obf); c.set_option("tc_persist", persist)
        st = torch.cuda.Stream()
        with torch.cuda.stream(st):
            c.conv1d(x, [rows], w, b, dil=dil, shift0=-(taps - 1) * dil // 2, act=act)
        ms = c.last_op_ms()
        res.append(f"{'bf16' if obf else 'f32 '} out persist={persist}: {ms*1000:6.1f} us {2*rows*N*K*taps/ms/1e9:5.0f} TF")
    print(f"{name:13s} M={rows} K={K} N={N} t={taps}: " + " | ".join(res), flush=True)
