"""GPU: the fragment-native epilogue of the wgmma conv-GEMM and the row-panel GEMM (option "tc_epi_frag": 1, the default = the epilogue
runs on the accumulator fragments; 0 = the fragments are first transposed to 16 consecutive columns of one row) gives the same bits.

The fragment epilogue serves the staged stores of 16-bit outputs; launches with an fp32 output or direct stores keep the transposing
epilogue under both values, and the cases below that reach them check that.  Bias-only epilogues take the fragment epilogue's plain
variant, the others its general one; both are covered.  One cvk_op_conv_gemm launch under both values, on the
generic kernel (BN = 128 and 64, staged TMA stores and direct stores, persistent and one-CTA-per-tile launches) and on the panel kernel
(forced by flow_qkv_panel = 2): every activation with and without a per-column
alpha, bias or none, a residual, the accumulate input, out2 with its own activation, bf16 / IEEE-half / fp32 outputs, bf16 and half
operands, N not a multiple of 16, 64 or 128, rows not a multiple of 128 with gap rows (row2seq = -1) holding large values, and taps with
dilation and a shift.  Which kernel ran is read from a torch.profiler trace.  The per-sequence rowvec and the scale are set only inside
the flow stages (tools/epi_ab.py compares the flow stage's mels and bench.py's waveforms under both values)."""
import pytest
import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile

import kernel_refs as kr
from gpu_util import ctx, maxdiff

pytestmark = pytest.mark.gpu

DEV = "cuda"
PANEL, GENERIC = "qkv_panel_kernel", "conv_gemm_wg_kernel"
ACTS = ["none", "gelu", "silu", "mish", "elu", "lrelu", "snake", "tanh", "abs", "gelu_tanh"]


@pytest.fixture(autouse=True)
def _release_cached_blocks():
    yield
    torch.cuda.empty_cache()


def _bits_equal(a, b):
    return torch.equal(a, b) or bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


class Case:
    def __init__(self, rows, seqs, N, K=256, taps=1, dil=1, shift0=0, act1="none", alpha1=False, bias=True, resid=False, accumulate=False,
                 act2=None, alpha2=False, out="bf16", out2="bf16", operand="bf16", out_ld=None, seed=0):
        g = torch.Generator().manual_seed(seed)
        self.seqs, self.N, self.dil, self.shift0 = seqs, N, dil, shift0
        self.act1, self.act2, self.out, self.out2, self.operand, self.accumulate = act1, act2, out, out2, operand, accumulate
        valid = torch.zeros(rows, dtype=torch.bool)
        for s, n in seqs:
            valid[s:s + n] = True
        x = kr.bf16(torch.randn(rows, K, generator=g))
        x[~valid] = 0.0
        self.x = x.to(DEV)
        self.w = kr.bf16(torch.randn(N, K, taps, generator=g) * (K * taps) ** -0.5).to(DEV)
        self.bias = (0.5 * torch.randn(N, generator=g)).to(DEV) if bias else None
        self.alpha1 = (torch.rand(N, generator=g) * 2.7 + 0.3).to(DEV) if alpha1 else None
        self.alpha2 = (torch.rand(N, generator=g) * 2.7 + 0.3).to(DEV) if alpha2 else None
        ld = out_ld or N
        self.out_init = torch.randn(rows, ld, generator=g).to(DEV)
        self.resid = None
        if resid:
            r = 1e6 * torch.ones(rows, N + 4)
            r[valid] = torch.randn(int(valid.sum()), N + 4, generator=g)
            self.resid = r.to(DEV)
        self.out2_init = torch.randn(rows, ld, generator=g).to(DEV) if act2 is not None else None
        self.valid = valid

    def run(self, frag, tc_epi=2, tc_persist=2, panel=0):
        c = ctx("bf16")
        c.set_option("tc_epi_frag", frag)
        c.set_option("tc_epi", tc_epi)
        c.set_option("tc_persist", tc_persist)
        c.set_option("flow_qkv_panel", panel)
        try:
            # the launch is deterministic, so a trace that came back without any device-side record (the profiler lost the window's
            # GPU activity, as it occasionally does on a shared device) is taken again; the caller still requires the kernel's name
            for _ in range(3):
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    out, out2 = c.conv_gemm(self.x, [s for s, _ in self.seqs], [n for _, n in self.seqs], self.w, self.bias, self.dil,
                                            self.shift0, self.operand, self.act1, 0.1, self.alpha1, self.resid, False, self.accumulate,
                                            self.out_init, self.out, self.act2 or "none", 0.2, self.alpha2, self.out2_init, self.out2)
                    torch.cuda.synchronize()
                if any(e.device_type == DeviceType.CUDA for e in prof.key_averages()):
                    break
        finally:
            c.set_option("tc_epi_frag", 1)
            c.set_option("tc_epi", 2)
            c.set_option("tc_persist", 2)
            c.set_option("flow_qkv_panel", 1)
        return out.cpu(), (out2.cpu() if out2 is not None else None), [e.key for e in prof.key_averages()]

    def check(self, kernel, **kw):
        ref, ref2, names = self.run(0, **kw)
        assert any(kernel in n for n in names), names
        assert torch.isfinite(ref).all()
        got, got2, names = self.run(1, **kw)
        assert any(kernel in n for n in names), names
        bad = (got != ref) & ~(torch.isnan(got) & torch.isnan(ref))
        assert not bad.any(), (kw, "out", maxdiff(got, ref), bad.nonzero()[:8].tolist(), self.valid[bad.nonzero()[:8, 0]].tolist())
        if ref2 is not None:
            bad2 = (got2 != ref2) & ~(torch.isnan(got2) & torch.isnan(ref2))
            assert not bad2.any(), (kw, "out2", maxdiff(got2, ref2), bad2.nonzero()[:8].tolist())


RAGGED = (1000, [(3, 300), (320, 417), (760, 229)])         # rows not a multiple of 128, gap rows between and after the sequences


@pytest.mark.parametrize("act,alpha", [(a, False) for a in ACTS] + [("snake", True)])
def test_activations(act, alpha):
    """every activation (Snake also with its per-column alpha), bias + out2 in bf16, at N = 200 (a partial 16-column group in the last
    128-column tile), staged and direct stores"""
    cs = Case(*RAGGED, N=200, act1=act, alpha1=alpha, act2="snake", alpha2=alpha, seed=ACTS.index(act))
    for tc_epi in (2, 0):
        cs.check(GENERIC, tc_epi=tc_epi)


EPILOGUES = {
    # name: Case keyword arguments
    "plain_bias_bf16": dict(N=200, out="bf16"),                  # bias only: the plain variant, a partial 16-column group
    "plain_nobias_k3_fp16": dict(N=256, bias=False, taps=3, shift0=-1, out="fp16", operand="fp16"),
    "plain_bn64_bf16": dict(N=56, out="bf16"),
    "nobias_fp32": dict(N=256, bias=False, out="fp32"),
    "resid_fp32": dict(N=256, K=512, resid=True, out="fp32"),
    "resid_gelu_bf16": dict(N=256, act1="gelu", resid=True, out="bf16"),
    "accumulate_fp32": dict(N=192, accumulate=True, out="fp32"),
    "accumulate_bf16": dict(N=72, accumulate=True, act1="lrelu", out="bf16"),
    "out2_fp32_bf16": dict(N=256, act1="silu", act2="gelu", out="fp32", out2="bf16"),
    "out2_fp16_fp32": dict(N=320, act1="tanh", act2="mish", out="fp16", out2="fp32"),
    "f16_operand_fp16": dict(N=160, K=192, operand="fp16", out="fp16", act1="snake", alpha1=True),
    "f16_operand_fp32": dict(N=96, K=64, operand="fp16", out="fp32", act1="elu", resid=True),
    "n72_fp32": dict(N=72, out="fp32", act1="gelu"),             # N % 16 = 8: staged fp32, direct 16-bit
    "n100_fp32": dict(N=100, out="fp32", act1="silu"),           # N % 8 = 4
    "n18_bf16": dict(N=18, out="bf16", act1="mish", act2="abs", out_ld=24),  # 16-bit N % 8 != 0: direct stores only
    "n1_fp32": dict(N=1, out="fp32", act1="gelu", out_ld=4),
    "n40_bf16": dict(N=40, out="bf16", act1="gelu", act2="gelu_tanh", out2="fp16"),  # BN = 64, a partial group
    "n64_ld_pad": dict(N=64, out="bf16", out_ld=72, act1="gelu"),
    "k3_dil2": dict(N=256, taps=3, dil=2, shift0=-2, act1="snake", alpha1=True, out="fp16", operand="fp16"),
    "k7_shift": dict(N=136, K=128, taps=7, dil=1, shift0=-3, act1="lrelu", out="fp32"),
}


@pytest.mark.parametrize("name", list(EPILOGUES))
def test_epilogues(name):
    cs = Case(*RAGGED, seed=len(name), **EPILOGUES[name])
    for kw in (dict(), dict(tc_epi=0), dict(tc_persist=0)):
        cs.check(GENERIC, **kw)


def test_persistent_many_tiles():
    """more tiles than SMs: the persistent CTAs walk several tiles each (staging reuse, the next tile's rows), against one CTA per tile"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rows = 64 * sms + 77
    cs = Case(rows, [(5, rows // 2), (rows // 2 + 40, rows // 2 - 60)], N=256, taps=3, shift0=-1, act1="gelu", act2="silu", out="bf16",
              out2="fp32", seed=5)
    for kw in (dict(), dict(tc_persist=0), dict(tc_epi=0)):
        cs.check(GENERIC, **kw)


@pytest.mark.parametrize("out", ["bf16", "fp16"])
@pytest.mark.parametrize("layout", ["ragged", "short", "every_sm"])
@pytest.mark.parametrize("shape", [(1536, False, "none"), (512, True, "gelu")])
def test_panel(shape, layout, out):
    """the row-panel kernel (16-bit outputs only): qkv shape without bias, a bias + GELU shape"""
    N, bias, act = shape
    if layout == "ragged":
        rows, seqs = RAGGED
    elif layout == "short":
        rows, seqs = 37, [(2, 30)]
    else:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        rows = 128 * sms + 77
        seqs = [(5, rows // 3), (rows // 3 + 9, rows // 3), (2 * rows // 3 + 20, rows - 2 * rows // 3 - 29)]
    cs = Case(rows, seqs, N=N, bias=bias, act1=act, out=out, operand=out, seed=N + rows)
    cs.check(PANEL, panel=2)
