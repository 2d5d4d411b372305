"""GPU: the bf16 LM decode layers (cvk_op_lm_decode_layers: the layer loop of one cvk_lm_decode step on caller state) on every decode
path - the fused PDL chain, the per-op chain on the weight-streaming and on the tiled GEMMs - against an fp64 Qwen2 decoder layer
(tests/kernel_refs.py decode_layer):
 A. stage checks on a one-layer model: each stage is fed the kernel's own bf16 outputs, so every bound stays tight;
 B. stacks of 2 and 24 layers against the fp64 reference, exact and with the path's bf16 rounding points emulated;
 C. identities: run to run, pdl 0 / 1, a row against the other rows of its batch;
 D. refusals, each leaving the context usable.
Rows carry contexts that cross the 16-key blocks and the 256-key chunks up to 4000 keys, a dominant late key in the long rows, residual
rows of different scales and one row with outlier channels.  Every tolerance is derived next to its assert."""
import contextlib
import ctypes
import math

import pytest
import torch

import kernel_refs as kr
from oracle import lm as olm

pytestmark = pytest.mark.gpu

ERR_INVALID = -1
D, DFF, NKV = kr.LM_D, kr.LM_DFF, kr.NKV
CTX = [0, 1, 15, 16, 17, 255, 256, 257, 420, 1000, 4000]
BATCHES = [1, 7, 32, 33, 64]              # BPAD (padded batch of the decode GEMMs) 32 up to 32 rows, 64 above
PATHS = {                                 # the options that select each path, and the bf16 rounding points of its reference
    "fused": (dict(lm_fused=1, use_skinny=1), "fused"),
    "per-op": (dict(lm_fused=0, use_skinny=1), "per-op"),
    "per-op-tiled": (dict(lm_fused=0, use_skinny=0), "per-op"),
}
DEFAULTS = dict(lm_fused=1, use_skinny=1, pdl=1)
# fp32 RMSNorm (sum of 896 squares, rsqrtf, two products) against fp64: a few tens of fp32 roundings in the sum of positive terms, half
# of it through the square root, plus the rsqrtf and the products - < 2^-19 of |xn| with room to spare
NORM_EPS = 2.0 ** -19
GEMM_EPS = 2.0 ** -16                     # the decode GEMM bound of test_kernel_edges_gpu.py: 2^-16 sum |a||w| on exact bf16 operands


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _ints(v):
    return (ctypes.c_int * len(v))(*[int(x) for x in v])


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ================================================================================================ model and cases
def _state_dict(num_layers, seed):
    """a Qwen2LM state dict with bf16-representable projections (the kernels stream them as bf16, so the reference sees the kernels'
    weights), fan-in scaled; q/k/v twice as large so that the scores spread over a few units; RMSNorm weights 1 +- 0.1, each layer its
    own.  The decode layers read no embedding: the text table is a stub."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shape in olm.param_shapes(num_layers, with_lm_head=False).items():
        if name.endswith("layernorm.weight") or name == "llm.model.model.norm.weight":
            sd[name] = 1.0 + 0.1 * torch.randn(*shape, generator=g)
        elif name.endswith("_proj.bias"):
            sd[name] = 0.1 * torch.randn(*shape, generator=g)
        elif name == "llm.model.model.embed_tokens.weight":
            sd[name] = 0.5 * torch.randn(16, D, generator=g)
        elif "_proj.weight" in name:
            gain = 2.0 if any(f".{n}_proj" in name for n in "qkv") else 1.0
            sd[name] = kr.bf16(torch.randn(*shape, generator=g) * gain * shape[1] ** -0.5)
        else:
            sd[name] = kr.bf16(0.5 * torch.randn(*shape, generator=g))
    return sd


_models = {}


def _model(num_layers):
    """(context, per-layer weights, final norm weight); one context per model size, closed at the end of the module"""
    if num_layers not in _models:
        from cosyvoice_b200 import cvk
        c = cvk.Context(0, "bf16", workspace_gb=1.0)
        sd = _state_dict(num_layers, 1000 + num_layers)
        c.load_state_dict("llm", sd, cfg=[num_layers])
        _models[num_layers] = (c, [kr.layer_weights(sd, i) for i in range(num_layers)], sd["llm.model.model.norm.weight"])
    return _models[num_layers]


@pytest.fixture(scope="module", autouse=True)
def _release_models():
    yield
    for c, _, _ in _models.values():
        c.close()
    _models.clear()
    torch.cuda.empty_cache()


def _contexts(B):
    return [CTX[(b + 10) % len(CTX)] for b in range(B)]      # row 0 is the 4000-key row, so B = 1 is a long row


def _case(B, ws, seed):
    """x [B, 896] with row scales 0.3 / 1 / 3 / 10 and four outlier channels in row 2; bf16 caches [layers, B, 2, max_ctx, 64]; in the
    rows of 256 keys or more, layer 0 holds one dominant key 37 positions before the new one (as in _decode_case of
    test_kernel_edges_gpu.py): aligned with its group's mean query, so the warp that owns it holds the row maximum and the cross-warp
    merge decides the output; its value row is distinct"""
    g = torch.Generator().manual_seed(seed)
    ctx = _contexts(B)
    L, max_ctx = len(ws), max(ctx) + 1
    x = torch.randn(B, D, generator=g) * torch.tensor([(0.3, 1.0, 3.0, 10.0)[b % 4] for b in range(B)])[:, None]
    if B > 2:
        x[2, [7, 300, 301, 640]] = torch.tensor([60.0, -45.0, 80.0, -100.0])
    kc = kr.bf16(torch.randn(L, B, NKV, max_ctx, 64, generator=g) * 2.0)
    vc = kr.bf16(torch.randn(L, B, NKV, max_ctx, 64, generator=g))
    q = kr.decode_layer(ws[0], x, kc[0], vc[0], ctx, "fused")["q"]
    for b, n in enumerate(ctx):
        if n >= 256:
            for h in range(NKV):
                qm = q[b, h * 7:(h + 1) * 7].mean(0)
                kc[0, b, h, n - 37] = kr.bf16(qm * (80.0 / qm.dot(qm).clamp_min(1.0)) * 8).float()
                vc[0, b, h, n - 37] = 5.0
    return x, kc, vc, ctx


@contextlib.contextmanager
def _options(c, **opts):
    for k, v in opts.items():
        c.set_option(k, v)
    try:
        yield
    finally:
        for k in opts:
            c.set_option(k, DEFAULTS.get(k, 1))


def _run(c, path, x, kc, vc, ctx, **extra):
    """the op on `path`; caches go up once and come back as the new rows per layer [layers, B, 2, 64] after checking on the device that
    everything else is untouched (bf16-representable input: exact round trip)"""
    kg, vg = kc.cuda(), vc.cuda()
    with _options(c, **PATHS[path][0], **extra):
        x_out, k_out, v_out, (xn, att, ffa) = c.lm_decode_layers(x, kg, vg, ctx)
    rows = torch.arange(len(ctx))
    pos = torch.tensor(ctx)
    k_new, v_new = k_out[:, rows, :, pos].clone(), v_out[:, rows, :, pos].clone()      # [B, layers, 2, 64]
    k_out[:, rows, :, pos] = kg[:, rows, :, pos]
    v_out[:, rows, :, pos] = vg[:, rows, :, pos]
    assert torch.equal(k_out, kg) and torch.equal(v_out, vg), f"{path}: a cache row other than the new one changed"
    out = dict(x=x_out, xn=xn, att=att, ffa=ffa, k=k_new, v=v_new)
    return {k: v.cpu().double() for k, v in out.items()}


def _flip(exact, eps):
    """bound on |bf16(v) - bf16(exact)| for a kernel value v within eps of the fp64 value: 0 unless a rounding boundary lies within
    eps, else eps + one ulp (eps can exceed half an ulp of a small element: the GEMM bound is absolute)"""
    return torch.where(kr.near_bf16_tie(exact, eps), eps + kr.bf16_ulp(exact.abs() + eps), torch.zeros_like(exact))


def _pair(t):
    """|x1| + |x2| of every rotated pair (half-split RoPE: element i pairs with i + 32), for both elements"""
    s = t[..., :32] + t[..., 32:]
    return torch.cat([s, s], -1)


def _check(what, err, tol):
    ratio = (err / tol).max().item()
    if not (err <= tol).all():
        i = int((err - tol).flatten().argmax())
        raise AssertionError(f"{what}: element {i}: error {err.flatten()[i].item():.4g} > bound {tol.flatten()[i].item():.4g} "
                             f"(largest error / bound {ratio:.3g})")
    return ratio


# ================================================================================================ A. stage checks, one layer
def _stage_checks(path, x, kc, vc, ctx, out, w, g_final):
    """every stage of the single layer against fp64 fed the kernel's own outputs of the stage before; returns the largest
    error / bound per stage"""
    per_op = PATHS[path][1] == "per-op"
    B = len(ctx)
    W = {k: v.double() for k, v in w.items()}
    A = {k: v.abs() for k, v in W.items()}
    x = x.double()
    r = {}
    # entry xn = bf16(RMSNorm(x) ln1): elements within NORM_EPS of a tie may round the other way (a_xn)
    xn64 = kr.rms_norm(x, W["ln1"])
    xn_b = kr.bf16(xn64)
    a_xn = _flip(xn64, NORM_EPS * xn64.abs())
    # qkv: the GEMM bound on the rounded xn, plus the flips of xn through |W|, plus the bias add (one fp32 rounding)
    qkv64 = xn_b @ W["wqkv"].t() + W["bqkv"][None]
    e_qkv = GEMM_EPS * (xn_b.abs() @ A["wqkv"].t()) + a_xn @ A["wqkv"].t() + 2.0 ** -23 * qkv64.abs()
    if per_op:      # stored as bf16 before the rotation: equal to bf16(qkv64) except at a tie within e_qkv
        qkv_used = kr.bf16(qkv64)
        e_pre = _flip(qkv64, e_qkv)
    else:
        qkv_used, e_pre = qkv64, e_qkv
    q64, k64, v64 = kr.decode_qkv(qkv_used[None], torch.zeros(kr.QKV_N, dtype=torch.float64), ctx, round_bf16=False)
    # the rotation moves the input errors of a pair into both of its elements; the fp32 rotation adds < 2^-20 (|x1| + |x2|)
    ep = e_pre.view(B, 18, 64)
    e_rot = _pair(ep) + 2.0 ** -20 * _pair(qkv_used.abs().view(B, 18, 64))
    a_q = _flip(q64, e_rot[:, :14])
    a_k = _flip(k64, e_rot[:, 14:16])
    a_v = _flip(v64, ep[:, 16:18])
    # the appended K / V rows: bf16 of the fp64 values, exact unless a rounding boundary lies within the error of the kernel's fp32 value
    r["k_row"] = _check(f"{path}: appended k row", (out["k"][:, 0] - kr.bf16(k64)).abs(), a_k + 1e-30)
    r["v_row"] = _check(f"{path}: appended v row", (out["v"][:, 0] - kr.bf16(v64)).abs(), a_v + 1e-30)
    # attention on the kernel's own new K / V rows and bf16(q): in units of sum_j p_j |v_j|, 2^-8 for P in bf16 before P.V (fused)
    # + 2^-8 for the bf16 output + 1e-5 for __expf and the fp32 sums; a q element that may have flipped (a_q) moves score j by at most
    # 1/8 sum_d a_q |k_jd|, so every weight by a factor e^(+-2M) and the output by (e^(2M) - 1) sum p|v| (_decode_bound)
    q_b = kr.bf16(q64)
    k_new, v_new = out["k"][:, 0], out["v"][:, 0]
    ref = kr.decode_attention(q_b, k_new, v_new, kc[0], vc[0], ctx)
    pv = kr.decode_attention(q_b, k_new, v_new.abs(), kc[0], vc[0].abs(), ctx)
    scale = torch.empty(B, kr.NH, dtype=torch.float64)
    for b, n in enumerate(ctx):
        for h in range(kr.NH):
            keys = torch.cat([kc[0, b, h // 7, :n].double(), k_new[b, h // 7][None]]).abs()
            M = 0.125 * (keys @ a_q[b, h]).max().item()
            scale[b, h] = 2.0 ** -7 + 1e-5 + math.expm1(2 * M)
    tol = (scale[:, :, None] * pv.view(B, kr.NH, 64)).view(B, D) + 1e-7
    r["att"] = _check(f"{path}: attention", (out["att"] - ref).abs(), tol)
    # x_out = x + att_k Wo^T + ffa_k Wd^T: the two GEMM bounds on the kernel's own operands and the fp32 residual adds.  A lost or
    # doubled split, a wrong row or a missing residual moves an element by far more.
    att_k, ffa_k = out["att"], out["ffa"]
    x_mid = x + att_k @ W["wo"].t()
    e_mid = GEMM_EPS * (att_k.abs() @ A["wo"].t()) + 2.0 ** -23 * x_mid.abs()
    x_ref = x_mid + ffa_k @ W["wd"].t()
    r["x_out"] = _check(f"{path}: x_out", (out["x"] - x_ref).abs(), e_mid + GEMM_EPS * (ffa_k.abs() @ A["wd"].t()) + 2.0 ** -23 * x_ref.abs())
    # ffa = bf16(silu(g) u), g / u from xn_mid = bf16(RMSNorm(x_mid) ln2).  x_mid is the kernel's fp32 value within e_mid; through the
    # norm: |d xn| <= |ln2| r (e_mid + |x| mean(|x| e_mid) / mean(x^2)) + NORM_EPS |xn|, r = 1/rms
    ms = x_mid.pow(2).mean(-1, keepdim=True)
    rel = (x_mid.abs() * e_mid).mean(-1, keepdim=True) / ms
    xnm64 = kr.rms_norm(x_mid, W["ln2"])
    e_xnm = A["ln2"] * torch.rsqrt(ms + olm.RMS_EPS) * (e_mid + x_mid.abs() * rel) + NORM_EPS * xnm64.abs()
    xnm_b = kr.bf16(xnm64)
    a_xnm = _flip(xnm64, e_xnm)
    gu = {}
    for n in ("wg", "wu"):
        v64 = xnm_b @ W[n].t()
        e = GEMM_EPS * (xnm_b.abs() @ A[n].t()) + a_xnm @ A[n].t()
        gu[n] = (kr.bf16(v64), _flip(v64, e)) if per_op else (v64, e)       # per-op: stored as bf16 before the SwiGLU kernel
    (g, dg), (u, du) = gu["wg"], gu["wu"]
    silu = g / (1.0 + torch.exp(-g))
    f64 = silu * u
    # |silu'| <= 1.1; fast_exp / __fdividef (or expf and a division) and the product: 2^-20 relative
    e_f = 1.1 * u.abs() * dg + silu.abs() * du + 1.1 * dg * du + 2.0 ** -20 * f64.abs()
    r["ffa"] = _check(f"{path}: ffa", (ffa_k - kr.bf16(f64)).abs(), _flip(f64, e_f) + e_f + 1e-30)
    # the final-normed row the head reads: bf16(RMSNorm(x_out_k) g_final), exact unless a tie lies within NORM_EPS
    xf64 = kr.rms_norm(out["x"], g_final)
    r["xn_out"] = _check(f"{path}: xn_out", (out["xn"] - kr.bf16(xf64)).abs(), _flip(xf64, NORM_EPS * xf64.abs()) + 1e-30)
    return r


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("path", list(PATHS))
def test_decode_layer_stages(path, B):
    c, ws, g_final = _model(1)
    x, kc, vc, ctx = _case(B, ws, 7 * B)
    out = _run(c, path, x, kc, vc, ctx)
    r = _stage_checks(path, x, kc, vc, ctx, out, ws[0], g_final)
    print(f"[one layer, {path}, B={B}] largest error / bound: " + ", ".join(f"{k} {v:.3g}" for k, v in r.items()))


# ================================================================================================ B. stacks
def _stack_reference(ws, g_final, x, kc, vc, ctx, rounding):
    h, ks, vs = x.double(), [], []
    for l, w in enumerate(ws):
        st = kr.decode_layer(w, h, kc[l], vc[l], ctx, rounding)
        ks.append(st["k"])
        vs.append(st["v"])
        h = st["x_out"]
    xn = kr.rms_norm(h, g_final)
    return dict(x=h, xn=kr.bf16(xn) if rounding else xn, k=torch.stack(ks, 1), v=torch.stack(vs, 1))


def _stack_errors(out, ref):
    """largest error of the final-normed row (|xn| ~ 1), of the residual stream relative to its row's rms, and of the appended K / V
    rows relative to their row's rms"""
    rms = lambda t: t.pow(2).mean(-1, keepdim=True).sqrt()
    return dict(xn=(out["xn"] - ref["xn"]).abs().max().item(),
                x=((out["x"] - ref["x"]).abs() / rms(ref["x"])).max().item(),
                kv=max(((out[n] - ref[n]).abs() / rms(ref[n])).max().item() for n in ("k", "v")))


# Largest errors measured on an H100 80GB HBM3 (700 W power limit) over the three paths at B = 33, against the exact reference and
# against the one emulating the path's bf16 rounding points:
#   2 layers:  exact xn 0.053, x 0.050, kv 0.027;  emulated xn 0.023, x 0.021, kv 0.017
#   24 layers: exact xn 0.52,  x 0.45,  kv 0.45;   emulated xn 0.21,  x 0.20,  kv 0.22
# (this random 24-layer stack amplifies a bf16 rounding difference from layer to layer).  The bounds are twice those.  At 2 layers a
# wrong layer's RMSNorm weight moves xn by 0.85, a missing residual by 16; the stage checks above catch the single-stage defects at
# 50x - 10^5 their bounds.
STACK_BOUND = {2: (dict(xn=0.11, x=0.10, kv=0.055), dict(xn=0.047, x=0.042, kv=0.035)),
               24: (dict(xn=1.05, x=0.9, kv=0.9), dict(xn=0.42, x=0.4, kv=0.44))}


@pytest.mark.parametrize("num_layers", [2, 24])
def test_decode_layer_stacks(num_layers):
    c, ws, g_final = _model(num_layers)
    B = 33
    x, kc, vc, ctx = _case(B, ws, 100 + num_layers)
    refs = {None: _stack_reference(ws, g_final, x, kc, vc, ctx, None)}
    failures = []
    for path, (_, rounding) in PATHS.items():
        if rounding not in refs:
            refs[rounding] = _stack_reference(ws, g_final, x, kc, vc, ctx, rounding)
        out = _run(c, path, x, kc, vc, ctx)
        ex, em = _stack_errors(out, refs[None]), _stack_errors(out, refs[rounding])
        print(f"[{num_layers} layers, {path}, B={B}] exact reference: " + ", ".join(f"{k} {v:.3g}" for k, v in ex.items()) +
              f"; {rounding} rounding emulated: " + ", ".join(f"{k} {v:.3g}" for k, v in em.items()))
        for ref, err, bounds in (("exact", ex, STACK_BOUND[num_layers][0]), (rounding, em, STACK_BOUND[num_layers][1])):
            failures += [(path, ref, k, err[k], bound) for k, bound in bounds.items() if err[k] > bound]
    assert not failures, failures


# ================================================================================================ C. identities
@pytest.mark.parametrize("path", list(PATHS))
def test_decode_layer_repeatable_and_pdl_invariant(path):
    """two runs agree bit for bit, and so do pdl 0 and 1 (programmatic dependent launch only overlaps prologues)"""
    c, ws, _ = _model(2)
    x, kc, vc, ctx = _case(33, ws, 5)
    a = _run(c, path, x, kc, vc, ctx)
    b = _run(c, path, x, kc, vc, ctx)
    p0 = _run(c, path, x, kc, vc, ctx, pdl=0)
    for k in a:
        assert torch.equal(a[k], b[k]), (path, k, "run to run")
        assert torch.equal(a[k], p0[k]), (path, k, "pdl 0 vs 1")


@pytest.mark.parametrize("B", [7, 33])
@pytest.mark.parametrize("path", list(PATHS))
def test_decode_layer_row_independent_of_batch(path, B):
    """row 5 computes the same whatever the other rows of its batch hold (same BPAD class), bit for bit"""
    c, ws, _ = _model(1)
    x, kc, vc, ctx = _case(B, ws, 50 + B)
    x2, kc2, vc2, _ = _case(B, ws, 60 + B)
    keep = 5
    x2[keep], kc2[:, keep], vc2[:, keep] = x[keep], kc[:, keep], vc[:, keep]
    x2[torch.arange(B) != keep] *= 7.0
    b = _run(c, path, x2, kc2, vc2, ctx)
    a = _run(c, path, x, kc, vc, ctx)
    for k in a:
        assert torch.equal(a[k][keep], b[k][keep]), (path, B, k)


# ================================================================================================ D. refusals
def test_decode_layer_refusals_leave_context_usable():
    """refused before any device work, with CVK_ERR_INVALID: an fp32 context, a context without the llm stage, B outside [1, 64],
    ctx_len outside [0, max_ctx), max_ctx beyond the decode-attention limit (7 x max_ctx fp32 scores in 200 KB of shared memory);
    the options "lm_mega" and "mega_coop" are unknown keys (there is no persistent decode kernel to select); afterwards the same
    context computes what it computed before"""
    from cosyvoice_b200 import cvk
    c, ws, _ = _model(1)
    x, kc, vc, ctx = _case(7, ws, 3)
    before = _run(c, "fused", x, kc, vc, ctx)
    xg = torch.zeros(65, D, device="cuda")
    cache = torch.zeros(65 * NKV * 16 * 64, device="cuda")
    out = torch.zeros(65, DFF, device="cuda")
    lib = c.lib

    def call(h, B, ctx_len, max_ctx):
        return lib.cvk_op_lm_decode_layers(h, B, _ints(ctx_len), max_ctx, _p(xg), _p(cache), _p(cache), _p(out), _p(out), _p(out), _stream())

    for B, ctx_len, max_ctx in [(0, [0], 16), (65, [0] * 65, 16), (1, [-1], 16), (1, [16], 16), (2, [0, 16], 16), (1, [0], 0),
                                (1, [0], 8000)]:
        assert call(c.h, B, ctx_len, max_ctx) == ERR_INVALID, (B, ctx_len, max_ctx)
    f = cvk.Context(0, "fp32", workspace_gb=0.25)
    e = cvk.Context(0, "bf16", workspace_gb=0.25)
    try:
        assert call(f.h, 1, [0], 16) == ERR_INVALID
        assert call(e.h, 1, [0], 16) == ERR_INVALID        # no llm stage
    finally:
        f.close()
        e.close()
    for key, value in (("lm_mega", 1), ("mega_coop", 0)):
        with pytest.raises(cvk.CvkError):
            c.set_option(key, value)
    after = _run(c, "fused", x, kc, vc, ctx)
    for k in before:
        assert torch.equal(before[k], after[k]), k
