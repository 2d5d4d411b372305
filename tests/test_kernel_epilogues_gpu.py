"""GPU: the conv-GEMM with the epilogues the stages ask of it, and the conformer relative-position attention, each against a plain fp64
reference (tests/kernel_refs.py) fed exactly the operands the kernel sees:
 A. one recipe per call site of the vocoder, the U-Net estimator and the DiT (Snake with per-column alpha as act1 and act2, residual from
    another matrix and in place, accumulate, a second output in fp32 / bf16 / fp16, ELU / ABS / TANH / GELU_TANH, column slices and pitches
    wider than N), on every operand path the stage meets plus the fp32 CUDA-core kernel, with both wgmma epilogue modes and with per-tile
    and persistent launches;
 B. the relative-position attention on its three paths (fp32 CUDA cores, the wgmma pair, CUDA cores on bf16 operands).
Gap rows of every operand carry large values where the kernel must not look (resid 1e6, every second attention sequence V * 1e4,
NaN in the columns of x past K), so that a leak shows up as a failure that names the field, row and column.  Every tolerance is derived
next to its assert, and each test prints its largest error / bound."""
import ctypes
import math
import zlib
from dataclasses import dataclass
from typing import Optional

import pytest
import torch

import kernel_refs as kr
from gpu_util import ctx

pytestmark = pytest.mark.gpu

ERR_INVALID = -1
SENTINEL = -1536.0           # exact in fp32, bf16 and fp16: pad columns and gap rows of the outputs start with it
DEV = "cuda"

# operand path -> (context precision, operand dtype, use_tc)
PATHS = {
    "fp16-tc": ("bf16", "fp16", 1),      # the vocoder in the tensor-core mode (hift_f16 on, the default)
    "bf16-tc": ("bf16", "bf16", 1),      # estimator / DiT / encoder, and the vocoder with hift_f16 off
    "fp16-simt": ("bf16", "fp16", 0),    # use_tc 0 on the vocoder's operands
    "bf16-simt": ("bf16", "bf16", 0),
    "fp32-simt": ("fp32", "fp32", 1),    # the fp32 mode, and the time MLPs / f0 predictor in every mode
}
VOC = ["fp16-tc", "bf16-tc", "fp16-simt", "fp32-simt"]
EST = ["bf16-tc", "bf16-simt", "fp32-simt"]
SIMT32 = ["fp32-simt", "bf16-tc"]        # called on the CUDA cores in fp32 by the stages; the wgmma run adds its fast activations


@pytest.fixture(autouse=True)
def _release_cached_blocks():
    """the recipes allocate matrices of up to ~18k x 1024 fp32: their cached blocks go back to the device after each test, so that later
    tests which size device pools from the free memory (tts_stream_batch's slot pool) see what they would see without this file"""
    yield
    torch.cuda.empty_cache()


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _ints(v):
    return (ctypes.c_int * len(v))(*[int(x) for x in v])


def _exact(*shape, g, scale=1.0):
    """values exact in bf16 and in IEEE half (8 significant bits, 0 or |x| >= 2^-14): every operand path sees the same numbers, and
    products of two of them are exact in fp32"""
    x = kr.bf16(torch.randn(*shape, generator=g) * scale)
    return torch.where(x.abs() < 2.0 ** -14, torch.zeros_like(x), x)


# ================================================================================================ A. conv-GEMM epilogue recipes
@dataclass
class Recipe:
    name: str
    paths: list
    K: int
    N: int
    taps: int = 1
    dil: int = 1
    shift0: int = 0
    act1: str = "none"
    p1: float = 0.0
    alpha1: bool = False
    resid: Optional[str] = None          # None, "other" (fp32 matrix of its own) or "inplace" (the fp32 out itself)
    accumulate: bool = False
    out: str = "fp32"                    # the output dtype of the call site
    act2: Optional[str] = None           # None: no second output
    p2: float = 0.0
    alpha2: bool = False
    out2: str = "fp32"
    x_ld: int = 0                        # 0: K
    out_ld: int = 0                      # 0: N
    out2_ld: int = 0


RECIPES = [
    # vocoder (hift.cu): level-3 widths (64 channels) so that a ragged batch gives more output tiles than SMs at moderate cost
    Recipe("vocoder-resblock-conv1", VOC, 64, 64, taps=11, dil=5, shift0=-25, act1="snake", alpha1=True, out="fp16"),
    Recipe("vocoder-resblock-conv2", VOC, 128, 128, taps=7, shift0=-3, resid="other", act2="snake", alpha2=True, out2="fp16"),
    Recipe("vocoder-last-resblock-conv2", VOC, 64, 64, taps=7, shift0=-3, resid="other", accumulate=True),
    Recipe("vocoder-source-down", VOC, 360, 256, taps=3, shift0=-1, act2="snake", alpha2=True, out2="fp16"),    # 15 STFT rows per row
    Recipe("vocoder-conv_pre", VOC, 80, 512, taps=7, shift0=-3, act1="lrelu", p1=0.1, out="fp16", x_ld=88),
    Recipe("vocoder-ups0", VOC, 512, 2048, taps=3, shift0=-1),                   # polyphase ConvTranspose1d, N = s * C
    Recipe("vocoder-ups1", VOC, 256, 640, taps=3, shift0=-1),
    Recipe("vocoder-ups2", VOC, 128, 192, taps=3, shift0=-1),
    Recipe("vocoder-conv_post", VOC, 64, 18, taps=7, shift0=-3, out_ld=24),
    Recipe("vocoder-f0-elu", SIMT32, 80, 512, taps=3, shift0=-1, act1="elu"),
    Recipe("vocoder-f0-abs", SIMT32, 512, 1, act1="abs", out_ld=4),
    # U-Net estimator (flow.cu)
    Recipe("estimator-time-mlp", SIMT32, 320, 1024, act1="silu", act2="mish"),
    Recipe("estimator-ff1", EST, 256, 1024, act1="gelu", out="bf16"),
    Recipe("estimator-ff2", EST, 1024, 256, resid="inplace", act2="none", out2="bf16"),
    Recipe("estimator-res-conv", EST, 320, 256, resid="other", x_ld=328),
    # DiT (flow.cu): the k31 causal position convolution on a 64-wide column slice of 1024-wide matrices, residual in place
    Recipe("dit-k31-position-conv", EST, 64, 64, taps=31, shift0=-30, act1="mish", resid="inplace", x_ld=1024, out_ld=1024),
    Recipe("dit-ff1", EST, 1024, 2048, act1="gelu_tanh", out="bf16"),
    Recipe("dit-time-silu", SIMT32, 256, 1024, act1="silu", act2="silu"),
    Recipe("tanh", EST, 72, 200, act1="tanh", out="bf16", x_ld=80),
    # no call site combines them, but the epilogue defines it: out2 = act2(out + v) on valid rows, 0 on gap rows (whose out is kept)
    Recipe("accumulate-with-out2", VOC, 64, 80, taps=3, shift0=-1, act1="snake", alpha1=True, resid="other", accumulate=True, act2="snake",
           alpha2=True, out2="fp16"),
]


def _reach(rec):
    return max(0, -rec.shift0, rec.shift0 + (rec.taps - 1) * rec.dil)


def _geometry(rec, sms):
    """ragged sequences packed with gaps of the receptive field + 3 rows; the first one starts at row 0 and the last one ends at the last
    row (their halos fall outside the matrix), and there are more output tiles (128 rows x BN columns) than SMs"""
    ntn = -(-rec.N // (128 if rec.N > 64 else 64))
    want = 128 * -(-(sms + 8) // ntn)
    gap = _reach(rec) + 3
    lens = [1, 2, 77, 128, 129, 300]
    total = sum(lens) + gap * (len(lens) - 1)
    if total < want:
        lens.append(max(1, want - total - gap))
    if (sum(lens) + gap * (len(lens) - 1)) % 128 == 0:
        lens[-1] += 1
    starts, r = [], 0
    for L in lens:
        starts.append(r)
        r += L + gap
    rows = r - gap
    assert ntn * -(-rows // 128) > sms and rows % 128
    return starts, lens, rows


class Case:
    """operands of one recipe (on the device) and its fp64 reference"""

    def __init__(self, rec, sms):
        g = torch.Generator().manual_seed(zlib.crc32(rec.name.encode()))
        self.starts, self.lens, rows = _geometry(rec, sms)
        self.rows = rows
        K, N = rec.K, rec.N
        valid = torch.zeros(rows, dtype=torch.bool)
        for s, L in zip(self.starts, self.lens):
            valid[s:s + L] = True
        nv = int(valid.sum())
        x = torch.full((rows, rec.x_ld or K), float("nan"))       # columns past K: must never be read
        x[:, :K] = 0.0
        x[valid, :K] = _exact(nv, K, g=g, scale=1.5)
        self.w = _exact(N, K, rec.taps, g=g, scale=(K * rec.taps) ** -0.5).to(DEV)
        self.bias = (torch.randn(N, generator=g) * 0.5).to(DEV)
        self.alpha1 = (torch.rand(N, generator=g) * 2.7 + 0.3).to(DEV) if rec.alpha1 else None
        self.alpha2 = (torch.rand(N, generator=g) * 2.7 + 0.3).to(DEV) if rec.alpha2 else None
        out_init = torch.full((rows, rec.out_ld or N), SENTINEL)
        out_init[valid, :N] = _exact(nv, N, g=g)                   # the accumulate input / the in-place residual
        if rec.resid == "inplace":
            out_init[~valid, :N] = 1e6
        self.resid = None
        if rec.resid == "other":
            resid = torch.full((rows, N + 4), float("nan"))         # pad columns: never read
            resid[:, :N] = 1e6                                      # gap rows: large, must not reach the output
            resid[valid, :N] = torch.randn(nv, N, generator=g)
            self.resid = resid.to(DEV)
        self.out2_init = torch.full((rows, rec.out2_ld or N), SENTINEL).to(DEV) if rec.act2 is not None else None
        self.x, self.out_init, self.valid = x.to(DEV), out_init.to(DEV), valid.to(DEV)
        # fp64 reference on the device (IEEE double GEMMs)
        x64 = self.x[:, :K].double()
        acc = kr.conv_rows(x64, self.w, rec.dil, rec.shift0)
        self.mag = kr.conv_rows(x64.abs(), self.w.abs(), rec.dil, rec.shift0)     # sum |x w|
        self.pre = acc + self.bias.double()[None]
        resid_ref = self.out_init[:, :N] if rec.resid == "inplace" else (self.resid[:, :N] if self.resid is not None else None)
        self.ref, self.ref2 = kr.conv_epilogue(acc, self.valid, self.bias, rec.act1, rec.p1, self.alpha1, resid_ref, self.out_init[:, :N],
                                               rec.accumulate, rec.act2, rec.p2, self.alpha2)
        self.tol, self.tol2 = _bounds(rec, self)

    def run(self, rec, path, out="fp32", out2="fp32", tc_epi=2, tc_persist=2, x=None):
        precision, operand, use_tc = PATHS[path]
        c = ctx(precision)
        c.set_option("use_tc", use_tc)
        c.set_option("tc_epi", tc_epi)
        c.set_option("tc_persist", tc_persist)
        try:
            return c.conv_gemm(self.x if x is None else x, self.starts, self.lens, self.w, self.bias, rec.dil, rec.shift0, operand, rec.act1,
                               rec.p1, self.alpha1, self.resid, rec.resid == "inplace", rec.accumulate, self.out_init, out, rec.act2 or "none",
                               rec.p2, self.alpha2, self.out2_init, out2)
        finally:
            c.set_option("use_tc", 1)
            c.set_option("tc_epi", 2)
            c.set_option("tc_persist", 2)


# Lipschitz constants of the activations (max |f'|): GELU 1.13, SiLU 1.10, Mish 1.09, Snake 1 + |sin(2 a x)| <= 2
LIP = dict(none=1.0, lrelu=1.0, abs=1.0, elu=1.0, tanh=1.0, gelu=1.13, gelu_tanh=1.13, silu=1.1, mish=1.1, snake=2.0)


def _act_err(name, x, alpha):
    """bound on the error of one activation evaluated in fp32 by the kernels at x (the fast forms of the wgmma epilogue, which also
    cover the libm forms of the CUDA-core kernel):
      lrelu: one product, 2^-24 |x|;  none / abs: exact;
      SiLU, Mish, ELU: ex2.approx (2^-22 relative), __fdividef (2 ulp) and a few roundings: 2^-20 (1 + |x|);
      tanh: tanh.approx.f32, relative error about 2^-11: 2^-10 |tanh x| + 2^-20;
      Snake: __sinf(a x) within 2^-19 (1 + |a x|) after its range reduction, so sin^2 / a within 2^-18 (1 + |a x|) / a, plus __fdividef and
        the fma: 2^-21 (|x| + 1/a);
      GELU_TANH: tanh of a half-rounded argument in half precision (tanh.approx.f16x2): |tanh error| <= 2^-9, times 0.5 |x|; the tail
        columns use tanh.approx.f32 (smaller);
      GELU: as GELU_TANH plus the distance of the tanh form from the erf form, computed here exactly."""
    ax = x.abs()
    if name in ("none", "abs"):
        return torch.zeros_like(x)
    if name == "lrelu":
        return 2.0 ** -24 * ax
    if name in ("silu", "mish", "elu"):
        return 2.0 ** -20 * (1 + ax)
    if name == "tanh":
        return 2.0 ** -10 * torch.tanh(ax) + 2.0 ** -20
    if name == "snake":
        a = alpha.double()[None]
        return 2.0 ** -18 * (1 + a * ax) / a + 2.0 ** -21 * (ax + 1 / a)
    if name == "gelu_tanh":
        return 2.0 ** -10 * ax
    if name == "gelu":
        return (kr.act("gelu", x) - kr.act("gelu_tanh", x)).abs() + 2.0 ** -10 * ax
    raise ValueError(name)


def _bounds(rec, cs):
    """per-element bounds on |out - ref| and |out2 - ref2| for fp32 outputs, propagated through the epilogue in its order:
      product: exact operands (bf16 / fp16 values), fp32 accumulation of n = K * taps products: n 2^-24 sum|x w| on the CUDA cores
        (sequential fma), 2^-16 sum|x w| on the tensor cores (see test_kernel_edges_gpu.py); their sum bounds both;
      + bias: one rounding, 2^-24 |pre|;
      act1: Lipschitz constant times the error so far, plus its own evaluation error (_act_err);
      + resid, + the accumulate input: one rounding each, 2^-24 |v|;
      gap rows: exactly 0 (or exactly the accumulate input);
      out2 = act2(v): Lipschitz constant of act2 times the error of v, plus act2's evaluation error."""
    n = rec.K * rec.taps
    d = (n * 2.0 ** -24 + 2.0 ** -16) * cs.mag + 2.0 ** -24 * cs.pre.abs()
    y = kr.act(rec.act1, cs.pre, rec.p1, cs.alpha1)
    d = LIP[rec.act1] * d + _act_err(rec.act1, cs.pre, cs.alpha1)
    d = d + 2.0 ** -24 * (int(rec.resid is not None) + int(rec.accumulate)) * (y.abs() + cs.ref.abs())
    d = torch.where(cs.valid[:, None], d * 1.01 + 2.0 ** -30, 0.0)
    d2 = None
    if rec.act2 is not None:
        d2 = LIP[rec.act2] * d + _act_err(rec.act2, cs.ref, cs.alpha2)
        d2 = torch.where(cs.valid[:, None], d2 * 1.01 + 2.0 ** -30, 0.0)
    return d, d2


def _check_ref(rec, cs, what, out, out2, worst):
    """out / out2 (fp32 runs) against the reference, pad columns against the sentinel; names field, row and column of a failure"""
    N = rec.N
    for field, got, ref, tol in (("out", out, cs.ref, cs.tol), ("out2", out2, cs.ref2, cs.tol2)):
        if ref is None:
            continue
        err = (got[:, :N].double() - ref).abs()
        ratio = torch.where(tol > 0, err / tol.clamp_min(1e-300), torch.where(err > 0, torch.inf, 0.0))
        ratio = torch.where(torch.isnan(err), torch.inf, ratio)
        r, c = divmod(int(ratio.argmax()), N)
        worst[field] = max(worst.get(field, 0.0), ratio.max().item())
        assert ratio.max().item() <= 1.0, (f"{rec.name} {what}: {field} row {r} ({'valid' if cs.valid[r] else 'gap'}) col {c}: "
                                           f"got {got[r, c].item():.7g} ref {ref[r, c].item():.7g} bound {tol[r, c].item():.3g}")
        pad = got[:, N:]
        assert bool((pad == SENTINEL).all()), f"{rec.name} {what}: {field} pad columns [{N}, {got.shape[1]}) overwritten"


def _bits_equal(a, b):
    return torch.equal(a, b) or bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


@pytest.mark.parametrize("rec", RECIPES, ids=[r.name for r in RECIPES])
def test_conv_gemm_epilogue_recipe(rec):
    """each call site's epilogue on every operand path it meets (+ fp32 CUDA cores), against the fp64 reference; then the identities:
    wgmma tc_epi 0 == 2 and persistent == per-tile launches, bit for bit; the call site's 16-bit out / out2 == the fp32 run's values
    rounded once (the epilogue rounds only at the store); junk in x[:, K:x_ld] changes nothing"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cs = Case(rec, sms)
    for path in rec.paths:
        worst = {}
        tc = PATHS[path][2] == 1 and PATHS[path][1] != "fp32"
        out, out2 = cs.run(rec, path)
        _check_ref(rec, cs, f"{path} default", out, out2, worst)
        variants = [dict(tc_epi=0), dict(tc_persist=0), dict(tc_epi=0, tc_persist=0)] if tc else []
        for v in variants:
            o, o2 = cs.run(rec, path, **v)
            assert _bits_equal(o, out), (rec.name, path, v, "out", (o - out).abs().max().item())
            assert out2 is None or _bits_equal(o2, out2), (rec.name, path, v, "out2", (o2 - out2).abs().max().item())
        if rec.out != "fp32" or (rec.act2 is not None and rec.out2 != "fp32"):
            for v in [dict()] + ([dict(tc_epi=0)] if tc else []):
                o, o2 = cs.run(rec, path, out=rec.out, out2=rec.out2, **v)
                assert _bits_equal(o, kr.round_to(out, rec.out)), (rec.name, path, v, rec.out, (o - kr.round_to(out, rec.out)).abs().max().item())
                if out2 is not None:
                    assert _bits_equal(o2, kr.round_to(out2, rec.out2)), (rec.name, path, v, rec.out2)
        if cs.x.shape[1] > rec.K:
            x0 = cs.x.clone()
            x0[:, rec.K:] = 0.0
            o, o2 = cs.run(rec, path, x=x0)
            assert _bits_equal(o, out) and (out2 is None or _bits_equal(o2, out2)), (rec.name, path, "junk columns of x were read")
        print(f"{rec.name} [{path}] rows {cs.rows} largest error / bound: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


@pytest.mark.parametrize("path", ["fp16-tc", "fp16-simt", "fp32-simt"])
def test_conv_gemm_fp16_store_saturates(path):
    """a value beyond the half range is stored as +-65504, not inf, in out and in out2 (from_f32<__half>), on both wgmma epilogues"""
    g = torch.Generator().manual_seed(11)
    rows, K, N = 300, 64, 72
    x = _exact(rows, K, g=g).to(DEV)
    w = _exact(N, K, 1, g=g, scale=K ** -0.5).to(DEV)
    bias = torch.tensor([1e5, -1e5, 7e4, -6.6e4, 3.0, 60000.0] * 12)[:N].to(DEV)
    precision, operand, use_tc = PATHS[path]
    c = ctx(precision)
    c.set_option("use_tc", use_tc)
    try:
        for epi in (2, 0):
            c.set_option("tc_epi", epi)
            out, out2 = c.conv_gemm(x, [0], [rows], w, bias, operand=operand, out=torch.zeros(rows, N), out_dtype="fp16", act2="none",
                                    out2=torch.zeros(rows, N), out2_dtype="fp16")
            ref, _ = kr.conv_epilogue(kr.conv_rows(x.double(), w), torch.ones(rows, dtype=torch.bool, device=DEV), bias)
            assert bool(torch.isfinite(out).all()) and bool(torch.isfinite(out2).all()), (path, epi)
            big = ref.abs() > 65520          # rounds past the largest half even before saturation
            assert big.any()
            for o in (out, out2):
                assert torch.equal(o[big], torch.sign(ref[big]).float() * 65504.0), (path, epi)
                # the rest: one half rounding of an fp32 value within 2^-16 sum|x w| + 2^-24 |v| of the reference
                d = (o[~big].double() - ref[~big]).abs()
                assert (d <= 2.0 ** -11 * ref[~big].abs() + 1e-3).all(), (path, epi, d.max().item())
    finally:
        c.set_option("use_tc", 1)
        c.set_option("tc_epi", 2)


def test_conv_gemm_refusals_leave_context_usable():
    """arguments the kernels cannot serve are refused before any allocation or launch, and the context still computes"""
    c = ctx("bf16")
    lib = c.lib
    rows, K, N = 64, 16, 16
    x = torch.zeros(rows, 24, device=DEV)
    w = torch.zeros(N * K * 3, device=DEV)
    out = torch.zeros(rows, 24, device=DEV)
    resid = torch.zeros(rows, 24, device=DEV)

    def call(K=K, x_ld=16, operand=1, starts=(0,), lens=(rows,), N=N, taps=3, dil=1, shift0=-1, act1=0, resid_p=None, resid_ld=0,
             inplace=0, out_dtype=0, out_ld=16, act2=0, out2=None, out2_dtype=0, out2_ld=0, lib=lib, h=c.h):
        return lib.cvk_op_conv_gemm(h, _p(x), rows, K, x_ld, operand, _ints(starts), _ints(lens), len(lens), _p(w), None, N, taps, dil, shift0,
                                    act1, 0.0, None, _p(resid_p), resid_ld, inplace, 0, _p(out), out_dtype, out_ld, act2, 0.0, None, _p(out2),
                                    out2_dtype, out2_ld, _stream())

    bad = [dict(N=0), dict(K=0), dict(taps=0), dict(dil=0), dict(x_ld=8), dict(out_ld=8), dict(operand=3), dict(out_dtype=5),
           dict(act1=10), dict(act2=-1), dict(K=12, x_ld=16),                      # 16-bit operand with K % 8 != 0
           dict(starts=(0, 30), lens=(32, 10)),                                     # overlapping sequences
           dict(starts=(0, 33), lens=(32, 10), taps=5, shift0=-2),                  # gap 1 < reach 2
           dict(starts=(60,), lens=(8,)), dict(starts=(-1,), lens=(8,)), dict(lens=(0,)),
           dict(resid_p=resid, resid_ld=16, inplace=1), dict(inplace=1, out_dtype=1),
           dict(x_ld=20),                                                           # wgmma: x rows of 40 bytes
           dict(out_dtype=1, out_ld=20),                                            # wgmma: bf16 out rows of 40 bytes
           dict(out2=out, out2_dtype=2, out2_ld=18),                                # wgmma: fp16 out2 rows of 36 bytes
           dict(resid_p=resid, resid_ld=18)]                                        # wgmma: resid_ld % 4 != 0
    for kw in bad:
        assert call(**kw) == ERR_INVALID, kw
    f = ctx("fp32")
    assert call(lib=f.lib, h=f.h) == ERR_INVALID                                   # 16-bit operand in an fp32 context
    assert call(lib=f.lib, h=f.h, operand=0, x_ld=20, out_ld=17) == 0              # the CUDA-core kernel takes any pitch
    g = torch.Generator().manual_seed(5)
    xe, we = _exact(rows, K, g=g).to(DEV), _exact(N, K, 3, g=g).to(DEV)
    got, _ = c.conv_gemm(xe, [0], [rows], we, shift0=-1, operand="bf16", out=torch.zeros(rows, N))
    ref = kr.conv_rows(xe.double(), we, 1, -1)
    assert ((got.double() - ref).abs() <= 2.0 ** -16 * kr.conv_rows(xe.double().abs(), we.abs(), 1, -1) + 1e-6).all()


# ================================================================================================ B. relative-position attention
RP_PATHS = [("fp32", 1), ("bf16", 1), ("bf16", 0)]       # CUDA cores fp32, wgmma pair, CUDA cores on bf16 operands (enc_tc_attn = 0)
RP_LENS = [1, 2, 63, 64, 65, 127, 128, 129, 300, 700]
RP_CHUNKS = [0, 1, 25, 50, 64]


def _grid16(*shape, g):
    """multiples of 1/16 with |x| < 4: q + bias_u and q + bias_v stay exact in bf16 (add_pos_bias_kernel rounds them)"""
    return torch.randint(-63, 64, shape, generator=g).float() / 16


def _rp_case(H, seed, lens=RP_LENS, extra=0):
    """operands of a ragged batch: the position table has independent random rows and the position term ((q + v) . p, std ~3 after the
    scale) outweighs the content term, so that an off-by-one table row is an O(1) error; every second sequence carries V * 1e4"""
    g = torch.Generator().manual_seed(seed)
    R, C = sum(lens), H * 64
    q = _grid16(R, C, g=g)
    bu, bv = _grid16(C, g=g), _grid16(C, g=g)
    k = kr.bf16(torch.randn(R, C, generator=g) * 0.5)
    v = kr.bf16(torch.randn(R, C, generator=g))
    o = 0
    for i, L in enumerate(lens):
        if i % 2:
            v[o:o + L] = kr.bf16(v[o:o + L] * 1e4)
        o += L
    center = max(lens) - 1 + extra
    pos = kr.bf16(torch.randn(2 * center + 1, C, generator=g))
    return q, k, v, pos, center, bu, bv


def _run_relpos(precision, tc, q, k, v, pos, center, bu, bv, lens, H, chunk):
    c = ctx(precision)
    if precision == "bf16" and not tc:
        c.set_option("enc_tc_attn", 0)
    try:
        return c.relpos_attention(q, k, v, pos, center, bu, bv, lens, H, chunk=chunk, scale=0.125).cpu().double()
    finally:
        c.set_option("enc_tc_attn", 1)


@pytest.mark.parametrize("chunk", RP_CHUNKS)
@pytest.mark.parametrize("H", [8, 4])
def test_relpos_attention(H, chunk):
    """every path against kr.relpos_attention (written from the reference layer's rel_shift, not from the kernels' index map)"""
    q, k, v, pos, center, bu, bv = _rp_case(H, H * 100 + chunk)
    ref = kr.relpos_attention(q, k, v, pos, center, bu, bv, RP_LENS, H, chunk, 0.125)
    pv = kr.relpos_attention(q, k, v.abs(), pos, center, bu, bv, RP_LENS, H, chunk, 0.125)       # sum_j p_j |v_j|
    for precision, tc in RP_PATHS:
        out = _run_relpos(precision, tc, q, k, v, pos, center, bu, bv, RP_LENS, H, chunk)
        worst, o = 0.0, 0
        for L in RP_LENS:
            # a score is a 128-term fp32 dot product of exact operands (64 content + 64 position terms; the wgmma pair adds the fp32 U
            # term to the fp32 content score): error <= 128 * 2^-24 * (|q+u||k| + |q+v||p|) times the scale (Cauchy-Schwarz over the
            # rows and heads of the sequence).  Every softmax weight moves by at most e^(+-2 ds), the output by (e^(2 ds) - 1) sum p|v|;
            # on top: fp32 1e-5 (exp / normalisation / accumulation), bf16 output 2^-8, wgmma P rounded to bf16 before P.V another
            # 2^-8 (as in test_kernel_edges_gpu.py _attn_tol).
            rows = slice(o, o + L)
            t = pos[center - (L - 1):center + L].view(-1, H, 64).norm(dim=-1).max().item()
            qu = (q[rows] + bu).view(L, H, 64).norm(dim=-1).max().item()
            qv = (q[rows] + bv).view(L, H, 64).norm(dim=-1).max().item()
            kn = k[rows].view(L, H, 64).norm(dim=-1).max().item()
            ds = 0.125 * 128 * 2.0 ** -24 * (qu * kn + qv * t)
            base = 1e-5 if precision == "fp32" else (2.0 ** -7 + 1e-5 if tc else 2.0 ** -8 + 1e-5)
            tol = (base + math.expm1(2 * ds)) * pv[rows] + 1e-7
            err = (out[rows] - ref[rows]).abs()
            ratio = err / tol
            worst = max(worst, ratio.max().item())
            i, col = divmod(int(ratio.argmax()), H * 64)
            assert (err <= tol).all(), (f"{precision} tc={tc} H={H} chunk={chunk} len {L}: row {i} head {col // 64} col {col % 64}: "
                                        f"out {out[o + i, col].item():.6g} ref {ref[o + i, col].item():.6g} ratio {ratio.max().item():.3g}")
            o += L
        print(f"relpos H={H} chunk={chunk} {precision}/tc{tc}: largest error / bound {worst:.3g}")


@pytest.mark.parametrize("precision,tc", RP_PATHS, ids=["fp32", "bf16-wgmma", "bf16-simt"])
def test_relpos_sequence_alone_equals_in_batch(precision, tc):
    """a sequence run alone with the table its own length gives (center L-1) equals the same sequence inside the ragged batch, where it
    reads the central rows of a larger table (center max(lens)-1+37): same operands, same tile order, bit for bit"""
    H = 8
    q, k, v, pos, center, bu, bv = _rp_case(H, 7, extra=37)
    for chunk in (0, 25):
        full = _run_relpos(precision, tc, q, k, v, pos, center, bu, bv, RP_LENS, H, chunk)
        o = 0
        for L in RP_LENS:
            if L in (1, 65, 129, 700):
                rows = slice(o, o + L)
                alone = _run_relpos(precision, tc, q[rows], k[rows], v[rows], pos[center - (L - 1):center + L], L - 1, bu, bv, [L], H, chunk)
                assert torch.equal(alone, full[rows]), (precision, tc, chunk, L, (alone - full[rows]).abs().max().item())
            o += L


def test_relpos_refusals_leave_context_usable():
    c = ctx("bf16")
    lib = c.lib
    H, L = 2, 8
    q = torch.zeros(L, H * 64, device=DEV)
    pos = torch.zeros(2 * L - 1, H * 64, device=DEV)
    b = torch.zeros(H * 64, device=DEV)
    out = torch.empty_like(q)
    for center, lens, h, chunk, scale in [(L - 2, [L], H, 0, 0.125), (L - 1, [L], H, 0, 0.0), (L - 1, [L], H, 0, -1.0), (L - 1, [L], 0, 0, 0.125),
                                          (L - 1, [L], H, -1, 0.125), (L - 1, [L, 0], H, 0, 0.125)]:
        rc = lib.cvk_op_relpos_attention(c.h, _p(q), _p(q), _p(q), _p(pos), center, _p(b), _p(b), _ints(lens), len(lens), h, chunk, scale,
                                         _p(out), _stream())
        assert rc == ERR_INVALID, (center, lens, h, chunk, scale)
    qq, k, v, p, center, bu, bv = _rp_case(H, 3, lens=[L])
    got = _run_relpos("bf16", 1, qq, k, v, p, center, bu, bv, [L], H, 0)
    ref = kr.relpos_attention(qq, k, v, p, center, bu, bv, [L], H, 0, 0.125)
    pv = kr.relpos_attention(qq, k, v.abs(), p, center, bu, bv, [L], H, 0, 0.125)
    assert ((got - ref).abs() <= 0.02 * pv + 1e-7).all()
