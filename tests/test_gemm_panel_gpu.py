"""GPU: the row-panel wgmma GEMM for one tap, K = 256 and a wide N (qkv_panel_kernel, gemm_tc.cu; option "flow_qkv_panel": 1 = from
25 panels of 128 rows up, 2 = at any row count, 0 = conv_gemm_wg_kernel).

 A. one conv-GEMM launch (cvk_op_conv_gemm, 16-bit output) under the three option values: identical bits, for the estimator's qkv shape
    (N = 1536, no bias, no activation) and its ff1 shape (N = 1024, bias + GELU), bf16 and IEEE-half operands, on ragged layouts whose
    gap rows hold large values (a panel that leaked them into a sequence would show an O(1) error) and must come out exactly zero.
    Which kernel ran is read from a torch.profiler trace of the call, so a comparison of the generic kernel with itself cannot pass.
 B. the qkv shape on the new kernel against the fp64 product of the bf16 operands.
The whole flow with the option on and off is compared in test_zz_gemm_panel_gpu.py."""
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import kernel_refs as kr
from gpu_util import ctx, maxdiff

pytestmark = pytest.mark.gpu

K = 256
PANEL, GENERIC = "qkv_panel_kernel", "conv_gemm_wg_kernel"
SHAPES = {"qkv": (1536, False, "none"), "ff1": (1024, True, "gelu")}       # N, bias, activation
LAYOUTS = {                                   # rows, [(start, len)]
    "ragged": (300, [(3, 100), (110, 57), (175, 120)]),
    "multi_tile": (1000, [(8, 650), (666, 326)]),
    "short": (37, [(2, 30)]),
    "one_row": (5, [(4, 1)]),
}


@pytest.fixture(autouse=True)
def _release_cached_blocks():
    yield
    torch.cuda.empty_cache()


def _layout(name):
    """the named layout, or "every_sm": one more 128-row panel than the device has SMs (more work units than CTAs, and above the row
    threshold of option 1), the last one partial, in three sequences"""
    if name != "every_sm":
        return LAYOUTS[name]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rows = 128 * sms + 77
    a, b = rows // 3, 2 * rows // 3
    return rows, [(5, a - 40), (a, b - a - 3), (b, rows - b - 9)]


def _operands(rows, seqs, N, bias, seed):
    g = torch.Generator().manual_seed(seed)
    x = kr.bf16(torch.randn(rows, K, generator=g))
    valid = torch.zeros(rows, dtype=torch.bool)
    for s, n in seqs:
        valid[s:s + n] = True
    x[~valid] = kr.bf16(1e3 * torch.randn(int((~valid).sum()), K, generator=g))
    w = kr.bf16(torch.randn(N, K, 1, generator=g) * K ** -0.5)
    b = 0.1 * torch.randn(N, generator=g) if bias else None
    return x, valid, w, b


def _run(c, opt, x, seqs, w, b, act, operand):
    """(out, names of the kernels the call launched) under flow_qkv_panel = opt"""
    out0 = torch.full((x.shape[0], w.shape[0]), -1536.0)
    c.set_option("flow_qkv_panel", opt)
    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out, _ = c.conv_gemm(x, [s for s, _ in seqs], [n for _, n in seqs], w, bias=b, operand=operand, act1=act, out=out0,
                                 out_dtype=operand)
            torch.cuda.synchronize()
    finally:
        c.set_option("flow_qkv_panel", 1)
    return out.cpu(), [e.key for e in prof.key_averages()]


def _ran(names, kernel):
    return any(kernel in n for n in names)


@pytest.mark.parametrize("operand", ["bf16", "fp16"])
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("layout", list(LAYOUTS) + ["every_sm"])
def test_panel_equals_generic(layout, shape, operand):
    """the panel kernel issues the generic kernel's MMAs per output and runs its epilogue functions: identical bits"""
    rows, seqs = _layout(layout)
    N, bias, act = SHAPES[shape]
    x, valid, w, b = _operands(rows, seqs, N, bias, seed=rows + N)
    c = ctx("bf16")
    ref, names = _run(c, 0, x, seqs, w, b, act, operand)
    assert _ran(names, GENERIC) and not _ran(names, PANEL), names
    assert torch.isfinite(ref).all() and (ref[~valid] == 0).all() and ref[valid].abs().max() > 0.5
    forced, names = _run(c, 2, x, seqs, w, b, act, operand)
    assert _ran(names, PANEL) and not _ran(names, GENERIC), names
    assert torch.equal(forced, ref), maxdiff(forced, ref)
    auto, names = _run(c, 1, x, seqs, w, b, act, operand)
    assert _ran(names, PANEL if layout == "every_sm" else GENERIC), names      # by the row count
    assert not _ran(names, GENERIC if layout == "every_sm" else PANEL), names
    assert torch.equal(auto, ref), maxdiff(auto, ref)


def test_panel_shape_conditions():
    """shapes the panel kernel does not serve stay on the generic kernel even when forced: N not in whole 128-column chunks, N < 512,
    K != 256, an fp32 output"""
    rows, seqs = LAYOUTS["ragged"]
    c = ctx("bf16")
    g = torch.Generator().manual_seed(3)
    for N, Kx, odt in ((1600, 256, "bf16"), (384, 256, "bf16"), (1536, 512, "bf16"), (1536, 256, "fp32")):
        x = kr.bf16(torch.randn(rows, Kx, generator=g))
        w = kr.bf16(torch.randn(N, Kx, 1, generator=g) * Kx ** -0.5)
        c.set_option("flow_qkv_panel", 2)
        try:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                c.conv_gemm(x, [s for s, _ in seqs], [n for _, n in seqs], w, operand="bf16", out=torch.zeros(rows, N), out_dtype=odt)
                torch.cuda.synchronize()
        finally:
            c.set_option("flow_qkv_panel", 1)
        names = [e.key for e in prof.key_averages()]
        assert _ran(names, GENERIC) and not _ran(names, PANEL), (N, Kx, odt, names)


@pytest.mark.parametrize("layout", ["multi_tile", "every_sm"])
def test_panel_qkv_vs_fp64(layout):
    rows, seqs = _layout(layout)
    N = SHAPES["qkv"][0]
    x, valid, w, _ = _operands(rows, seqs, N, False, seed=7 * rows + 1)
    c = ctx("bf16")
    out, names = _run(c, 2, x, seqs, w, None, "none", "bf16")
    assert _ran(names, PANEL), names
    assert (out[~valid] == 0).all()
    xv, w2 = x[valid].double(), w[:, :, 0].double()
    y = xv @ w2.t()
    mag = xv.abs() @ w2.abs().t()
    # exact products of bf16 operands; fp32 accumulation of 256 products on the tensor cores: (256 2^-24 + 2^-16) sum|x w| (the bound of
    # test_kernel_epilogues_gpu.py); then one rounding to bf16 (8 significant bits), half an ulp: 2^-8 relative
    acc = (K * 2.0 ** -24 + 2.0 ** -16) * mag
    bound = acc + 2.0 ** -8 * (y.abs() + acc) + 2.0 ** -30
    d = (out[valid].double() - y).abs()
    print(f"{layout}: max |d| {d.max().item():.3g}, bound median {bound.median().item():.3g}, |y| median {y.abs().median().item():.3g}")
    assert (d <= bound).all(), (d - bound).max().item()
