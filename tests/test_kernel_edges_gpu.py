"""GPU: the Hopper kernels at their edges, each against a plain fp64 CPU reference (tests/kernel_refs.py) fed the operands rounded
exactly as the kernel rounds them:
 A. the weight-streaming split-K decode GEMM (gemm_skinny.cu) at the LM's layer shapes and the split / tail extremes;
 B. the flash attention (SIMT fp32, wgmma bf16, SIMT bf16) with GQA, block-causal chunks and key-cache geometry;
 C. the LM decode attention (fused kernel and the per-op RoPE/append + attention pair);
 D. the conv-GEMM epilogue paths (direct vs TMA-staged stores, bf16 output) and ragged batches with a wide receptive field.
Neighbouring sequences of every ragged call carry large values, so that a tile load which leaks across a mask or a gap shows up
as an O(1) error.  Every tolerance is derived next to its assert."""
import ctypes
import math

import pytest
import torch

import kernel_refs as kr
from gpu_util import ctx
from test_ops_gpu import _ref_conv

pytestmark = pytest.mark.gpu

ERR_INVALID = -1


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _ints(v):
    return (ctypes.c_int * len(v))(*[int(x) for x in v])


def _bf16_randn(*shape, g, scale=1.0):
    """bf16-representable fp32 values: the kernel's operand rounding is then exact and the reference sees the kernel's operands"""
    return kr.bf16(torch.randn(*shape, generator=g) * scale)


# ================================================================================================ A. weight-streaming decode GEMM
SKINNY_SHAPES = [            # (N, K)
    (1152, 896),             # qkv
    (896, 896),              # o
    (9728, 896),             # gate_up: 76 tiles, 1 split
    (896, 4864),             # down: 16 splits of 5 K chunks, the last split holds 1 chunk (132 SMs)
    (6564, 896),             # Qwen2LM head: N tail of 36 in the last 128-feature tile
    (6764, 896),             # CosyVoice3LM head: N tail of 108
    (128, 8192),             # one tile, 32 splits
    (136, 904),              # N tail of 8, K tail of 8 inside the last 64-wide chunk
    (8, 64),                 # a single K chunk
]
SKINNY_ROWS = [1, 7, 31, 32, 33, 63, 64]      # BPAD (padded batch = wgmma N) is 32 up to 32 rows, 64 above


def skinny_splits(N, K, num_sms):
    """the split count of conv_gemm_skinny_ex (gemm_skinny.cu): ~all SMs busy, >= 4 K chunks per CTA, <= 32 splits, none empty"""
    tiles, kchunks = -(-N // 128), -(-K // 64)
    splits = max(1, min(num_sms // tiles, kchunks // 4, 32))
    cps = -(-kchunks // splits)
    return -(-kchunks // cps), cps, kchunks


@pytest.mark.parametrize("N,K", SKINNY_SHAPES, ids=[f"N{n}K{k}" for n, k in SKINNY_SHAPES])
def test_skinny_gemm(N, K):
    c = ctx("bf16")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    splits, cps, kchunks = skinny_splits(N, K, sms)
    print(f"N={N} K={K}: {splits} split(s) of {cps} K chunk(s), last split {kchunks - (splits - 1) * cps} chunk(s), {sms} SMs")
    g = torch.Generator().manual_seed(N * 7 + K)
    x = _bf16_randn(64, K, g=g)
    w = _bf16_randn(N, K, g=g, scale=K ** -0.5)
    bias = torch.randn(N, generator=g) * 0.1
    x64, w64 = x.double(), w.double()
    acc = x64 @ w64.t()
    # bf16 x bf16 products are exact in fp32; the fp32 accumulation (tensor-core internal order + split-K partial sums + the ordered
    # reduction) of K terms stays within 2^-16 of sum |x w| with room to spare for the tensor core's internal rounding (not IEEE fp32,
    # not measured here); adding the bias costs one more fp32 rounding (2^-24 |out|).  A lost or doubled split moves an output by
    # about sum|x w| / splits (>= 1/32 of it), a dropped 8-wide K tail by ~8/K of it: both > 100x this bound.
    bound = 2.0 ** -16 * (x64.abs() @ w64.abs().t()) + 1e-6
    worst = 0.0
    for rows in SKINNY_ROWS:
        for b in (None, bias):
            out, _ = c.linear_small(x[:rows], w, b)
            ref = acc[:rows] + (b.double()[None] if b is not None else 0.0)
            err = (out.cpu().double() - ref).abs()
            tol = bound[:rows] + 2.0 ** -24 * ref.abs()
            worst = max(worst, (err / tol).max().item())
            assert (err <= tol).all(), (rows, b is not None, err.max().item(), (err / tol).max().item())
    print(f"  largest error / bound: {worst:.3g}")
    # fixed split order: two calls agree bit for bit
    a1, _ = c.linear_small(x[:33], w, bias)
    a2, _ = c.linear_small(x[:33], w, bias)
    assert torch.equal(a1, a2)
    # a row's output does not depend on the other rows of the batch (same BPAD class: 33 rows -> 64, 7 rows -> 32)
    for rows in (7, 33):
        x2 = x[:rows].clone()
        x2[torch.arange(rows) != 5] = _bf16_randn(rows - 1, K, g=g, scale=30.0)
        b1, _ = c.linear_small(x[:rows], w, bias)
        b2, _ = c.linear_small(x2, w, bias)
        assert torch.equal(b1[5], b2[5]), rows


def test_skinny_gemm_refusals_leave_context_usable():
    """Arguments the weight-streaming GEMM cannot serve are refused before any allocation or launch (K % 8 != 0 has no bf16
    weight copy to stream; N = 0 / K = 0 would divide by zero in the split count); the same context then still computes."""
    c = ctx("bf16")
    g = torch.Generator().manual_seed(3)
    x = torch.randn(65, 64, generator=g).cuda()
    w = torch.randn(64, 64, generator=g).cuda()
    out = torch.empty(65, 64, device="cuda")
    ms = ctypes.c_float(0)
    lib = c.lib
    for rows, K, N in [(0, 64, 64), (65, 64, 64), (4, 12, 64), (4, 64, 0), (4, 0, 64), (4, 4, 64)]:
        rc = lib.cvk_op_linear_small(c.h, _p(x), rows, K, _p(w), None, N, _p(out), 0, ctypes.byref(ms), _stream())
        assert rc == ERR_INVALID, (rows, K, N, rc)
    f = ctx("fp32")
    assert f.lib.cvk_op_linear_small(f.h, _p(x), 4, 64, _p(w), None, 64, _p(out), 0, ctypes.byref(ms), _stream()) == ERR_INVALID
    torch.cuda.synchronize()
    xb, wb = kr.bf16(x[:9].cpu()), kr.bf16(w.cpu())
    got, _ = c.linear_small(xb, wb)
    ref = xb.double() @ wb.double().t()
    assert ((got.cpu().double() - ref).abs() <= 2.0 ** -16 * (xb.double().abs() @ wb.double().abs().t()) + 1e-6).all()


# ================================================================================================ B. prefill / flow attention
ATTN_PATHS = [("fp32", 1), ("bf16", 1), ("bf16", 0)]      # SIMT fp32, wgmma, SIMT on bf16 operands (use_tc_attn = 0)
HEADS = [(14, 2), (8, 8), (16, 16)]                      # LM prefill (GQA), U-Net estimator, DiT
CHUNKS = [0, 1, 25, 50, 64, 200]


def _run_attention(precision, tc, *args, **kw):
    c = ctx(precision)
    if precision == "bf16" and not tc:
        c.set_option("use_tc_attn", 0)
    try:
        return c.attention_ex(*args, **kw).cpu().double()
    finally:
        if precision == "bf16":
            c.set_option("use_tc_attn", 1)


def _attn_tol(precision, tc, ds):
    """bound on |o - ref| in units of sum_j p_j |v_j| (the attention output of |v|, per element), with ds the largest fp32 error of
    a score: a 64-term fp32 dot product of exact operands errs by <= 64 * 2^-24 sum_d |q_d k_d| (times the scale), so every softmax
    weight moves by at most a factor e^(+-2 ds) and o by (e^(2 ds) - 1) sum p|v|.  On top of that:
    fp32 SIMT: exp / normalisation / accumulation over <= 1000 keys, 1e-5 (a P-weighted mean: the rounding errors of positive
      weights do not align, far below 1000 * 2^-24);
    bf16 operands are exact (fed bf16 values); the output is stored as bf16 (8 significant bits, unit roundoff 2^-8):
      2^-8 |o| <= 2^-8 sum p|v|;
    wgmma: P is rounded to bf16 before P.V while the row sum uses the unrounded P: 2^-8 sum p|v| / sum p; the approximate exp2
      (~2^-22 relative) and the fp32 accumulation fit in another 1e-5."""
    base = 1e-5 if precision == "fp32" else (2.0 ** -7 + 1e-5 if tc else 2.0 ** -8 + 1e-5)
    return base + math.expm1(2 * ds)


def _check_attention(q, k, v, q_lens, k_lens, q_off, H, kvh, chunk, what, paths=ATTN_PATHS):
    ref = kr.attention(q, k, v, q_lens, k_lens, q_off, H, kvh, chunk, 0.125)
    pv = kr.attention(q, k, v.abs(), q_lens, k_lens, q_off, H, kvh, chunk, 0.125)     # sum_j p_j |v_j|
    worst = {}
    for precision, tc in paths:
        out = _run_attention(precision, tc, q, k, v, q_lens, k_lens, q_off, H, kvh, chunk=chunk)
        oq = ok = 0
        for Lq, Lk in zip(q_lens, k_lens):
            # sum_d |q_d k_d| <= |q|_2 |k|_2 (Cauchy-Schwarz), over every row / head of the sequence
            qn = q[oq:oq + Lq].view(Lq, H, 64).norm(dim=-1).max().item()
            kn = k[ok:ok + Lk].view(Lk, kvh, 64).norm(dim=-1).max().item()
            tol = _attn_tol(precision, tc, 0.125 * 64 * 2.0 ** -24 * qn * kn) * pv[oq:oq + Lq] + 1e-7
            err = (out[oq:oq + Lq] - ref[oq:oq + Lq]).abs()
            ratio = err / tol
            worst[(precision, tc)] = max(worst.get((precision, tc), 0.0), ratio.max().item())
            i, c = divmod(int(ratio.argmax()), H * 64)
            assert (err <= tol).all(), (f"{what} {precision} tc={tc} H={H}/{kvh} chunk={chunk} seq Lq={Lq} Lk={Lk}: row {i} col {c} "
                                        f"out {out[oq + i, c].item():.6g} ref {ref[oq + i, c].item():.6g} tol {tol[i, c].item():.3g} "
                                        f"ratio {ratio.max().item():.3g}")
            oq += Lq
            ok += Lk
    print(what, H, kvh, chunk, {f"{p}/tc{t}": f"{r:.3g}" for (p, t), r in worst.items()})


@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("H,kvh", HEADS, ids=[f"H{h}kv{k}" for h, k in HEADS])
def test_attention_ragged_self(H, kvh, chunk):
    """self attention (keys == queries) over ragged lengths crossing every 64-key and 128-query tile edge; every second sequence
    carries V * 1e4, so a key tile read past a sequence's end into its neighbour is an O(1) error for the small ones"""
    g = torch.Generator().manual_seed(H * 1000 + chunk)
    lens = [65, 700, 1, 128, 2, 257, 63, 129, 64, 127]
    R = sum(lens)
    q = _bf16_randn(R, H * 64, g=g)
    k = _bf16_randn(R, kvh * 64, g=g)
    v = _bf16_randn(R, kvh * 64, g=g)
    o = 0
    for i, L in enumerate(lens):
        if i % 2:
            v[o:o + L] = kr.bf16(v[o:o + L] * 1e4)
        o += L
    _check_attention(q, k, v, lens, lens, [0] * len(lens), H, kvh, chunk, "self")


@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("H,kvh", HEADS, ids=[f"H{h}kv{k}" for h, k in HEADS])
def test_attention_key_cache(H, kvh, chunk):
    """the streaming-session geometry: new query rows at offsets (multiples and non-multiples of the chunk and of 64) against a
    longer key cache, up to 1000 keys; keys past a query's chunk are in the cache but must stay invisible"""
    g = torch.Generator().manual_seed(H * 77 + chunk)
    q_lens = [50, 50, 75, 129, 1, 64]
    q_off = [100, 150, 925, 77, 999, 0]
    k_lens = [200, 200, 1000, 300, 1000, 65]
    q = _bf16_randn(sum(q_lens), H * 64, g=g)
    k = _bf16_randn(sum(k_lens), kvh * 64, g=g)
    v = _bf16_randn(sum(k_lens), kvh * 64, g=g)
    o = 0
    for i, L in enumerate(k_lens):
        if i % 2:
            v[o:o + L] = kr.bf16(v[o:o + L] * 1e4)
        o += L
    _check_attention(q, k, v, q_lens, k_lens, q_off, H, kvh, chunk, "cache")


@pytest.mark.parametrize("H,kvh,chunk", [(14, 2, 1), (8, 8, 50), (16, 16, 0)])
def test_attention_hard_scores(H, kvh, chunk):
    """(a) large scores: q * 8 (|s| up to ~100, softmax nearly one-hot); (b) the row maximum moves late: key norms grow along j,
    so every 64-key tile raises the running maximum and rescales the accumulator"""
    g = torch.Generator().manual_seed(H + chunk)
    lens = [300, 129, 700]
    R = sum(lens)
    q = _bf16_randn(R, H * 64, g=g, scale=8.0)
    k = _bf16_randn(R, kvh * 64, g=g)
    v = _bf16_randn(R, kvh * 64, g=g)
    _check_attention(q, k, v, lens, lens, [0] * len(lens), H, kvh, chunk, "large")
    q = _bf16_randn(R, H * 64, g=g)
    o = 0
    for L in lens:
        k[o:o + L] = kr.bf16(k[o:o + L] * torch.linspace(0.2, 4.0, L)[:, None])
        o += L
    _check_attention(q, k, v, lens, lens, [0] * len(lens), H, kvh, chunk, "late-max")


@pytest.mark.parametrize("precision,tc", ATTN_PATHS, ids=["fp32", "bf16-wgmma", "bf16-simt"])
def test_attention_query_slice_is_bit_identical(precision, tc):
    """what the streaming sessions rely on: rows [a, b) computed alone with q_offset = a against the full key set == rows [a, b)
    of the full computation, bit for bit (offsets not aligned to 64 or 128)"""
    g = torch.Generator().manual_seed(21)
    L = 700
    for H, kvh, chunk in [(8, 8, 50), (14, 2, 1), (16, 16, 0)]:
        q = _bf16_randn(L, H * 64, g=g)
        k = _bf16_randn(L, kvh * 64, g=g)
        v = _bf16_randn(L, kvh * 64, g=g)
        full = _run_attention(precision, tc, q, k, v, [L], [L], [0], H, kvh, chunk=chunk)
        for a, b in [(77, 211), (150, 200), (1, 2), (129, 700), (0, 63)]:
            part = _run_attention(precision, tc, q[a:b], k, v, [b - a], [L], [a], H, kvh, chunk=chunk)
            assert torch.equal(part, full[a:b]), (precision, tc, H, chunk, a, b, (part - full[a:b]).abs().max().item())


def test_attention_refusals():
    c = ctx("bf16")
    q = torch.zeros(8, 14 * 64, device="cuda")
    k = torch.zeros(8, 2 * 64, device="cuda")
    out = torch.empty_like(q)
    lens = _ints([8])
    for H, kvh, scale in [(14, 3, 0.125), (14, 2, 0.0), (14, 2, -0.125), (14, 0, 0.125)]:
        rc = c.lib.cvk_op_attention_ex(c.h, _p(q), _p(k), _p(k), lens, lens, _ints([0]), 1, H, kvh, 0, scale, _p(out), _stream())
        assert rc == ERR_INVALID, (H, kvh, scale)
    assert c.lib.cvk_op_attention(c.h, _p(q), _p(q), _p(q), lens, 1, 14, 0, -1.0, _p(out), _stream()) == ERR_INVALID


# ================================================================================================ C. decode attention
DEC_MAX_CTX = 4100
DEC_CTX = [0, 1, 15, 16, 17, 255, 256, 257, 511, 4000, DEC_MAX_CTX - 1]


def _decode_case(splits, seed):
    """partial sums on a 2^-10 grid with |value| < 2^3: every fp32 sum of <= 16 of them plus the bias is exact, so the kernels'
    reduced projection equals the fp64 one and only the RoPE arithmetic differs (fp32 in the kernels)"""
    g = torch.Generator().manual_seed(seed)
    rows = len(DEC_CTX)
    partial = torch.round(torch.randn(splits, rows, kr.QKV_N, generator=g).clamp(-4, 4) / splits ** 0.5 * 1024) / 1024
    bias = torch.round(torch.randn(kr.QKV_N, generator=g).clamp(-4, 4) * 0.2 * 1024) / 1024
    kc = _bf16_randn(rows, kr.NKV, DEC_MAX_CTX, 64, g=g)
    vc = _bf16_randn(rows, kr.NKV, DEC_MAX_CTX, 64, g=g)
    # one dominant key in a late 16-key block of two long rows: aligned with the group's mean query, so the warp that owns it holds
    # the row maximum and the cross-warp merge decides the output; its value row is distinct
    q, _, _ = kr.decode_qkv(partial, bias, DEC_CTX)
    for b in (DEC_CTX.index(511), DEC_CTX.index(4000)):
        j = DEC_CTX[b] - 37
        for h in range(kr.NKV):
            qm = q[b, h * 7:(h + 1) * 7].mean(0)
            kc[b, h, j] = kr.bf16(qm * (80.0 / qm.dot(qm).clamp_min(1.0)) * 8)
            vc[b, h, j] = 5.0
    return partial, bias, kc, vc


def _decode_bound(q, k_new, kc, q_ref64, k_ref64):
    """per (row, head) bound on |out - ref| (the reference is fed the kernel's exact projection, bf16-rounded first for the per-op
    path, see _decode_case):
    everything in units of sum_j p_j |v_j| (the attention output of |v|, per element);
    P in bf16 before P.V (row sum unrounded): <= 2^-8 (bf16 unit roundoff); bf16 output: 2^-8; __expf and the fp32 sums: 1e-5.
    q and k_new: the kernels rotate in fp32 by the same fp32 phase as oracle.lm.rope (test_kernel_refs_cpu.py checks the
    frequency table), the reference in fp64, so the rotated values differ by a few fp32 ulps: < 2^-20 (|x1| + |x2|) of the pair.  An
    element whose fp64 value lies that close to a bf16 rounding boundary may round the other way: one bf16 ulp.  With a_d = that ulp
    where it can happen (else 0) and c_d the same for k_new, score j moves by at most M = 1/8 max_j (sum_d a_d |k_jd| + [j new]
    sum_d (|q_d| + a_d) c_d); every softmax weight moves by at most a factor e^(+-2M), so o by (e^(2M) - 1) sum p|v|.  v_new is a
    plain rounding of an exact sum: no flip."""
    rows = q.shape[0]
    scale = torch.empty(rows, kr.NH)
    nflip = 0
    for b in range(rows):
        L = int(DEC_CTX[b])
        m_q = torch.cat([q_ref64[b, :, :32].abs() + q_ref64[b, :, 32:].abs()] * 2, -1)    # |x1| + |x2| of each rotated pair
        m_k = torch.cat([k_ref64[b, :, :32].abs() + k_ref64[b, :, 32:].abs()] * 2, -1)
        a = torch.where(kr.near_bf16_tie(q_ref64[b], 2.0 ** -20 * m_q), kr.bf16_ulp(q[b]), torch.zeros_like(q[b]))
        cc = torch.where(kr.near_bf16_tie(k_ref64[b], 2.0 ** -20 * m_k), kr.bf16_ulp(k_new[b]), torch.zeros_like(k_new[b]))
        nflip += int((a > 0).sum() + (cc > 0).sum())
        for h in range(kr.NH):
            kvh = h // 7
            M = (kc[b, kvh, :L].double().abs() @ a[h]).max().item() if L else 0.0
            M = 0.125 * max(M, ((k_new[b, kvh].abs() @ a[h]) + (q[b, h].abs() + a[h]) @ cc[kvh]).item())
            scale[b, h] = 2.0 ** -7 + 1e-5 + math.expm1(2 * M)
    return scale, nflip


@pytest.mark.parametrize("splits", [1, 3, 16])
@pytest.mark.parametrize("fused", [1, 0], ids=["fused", "per-op"])
def test_decode_attention(fused, splits):
    c = ctx("bf16")
    partial, bias, kc, vc = _decode_case(splits, splits * 10 + fused)
    c.set_option("lm_fused", fused)
    try:
        out, kc_out, vc_out = c.decode_attention(partial, bias, kc, vc, DEC_CTX)
    finally:
        c.set_option("lm_fused", 1)
    out, kc_out, vc_out = out.cpu().double(), kc_out.cpu(), vc_out.cpu()
    preround = not fused            # the per-op path stores the reduced projection as bf16 before the rotation
    q, k_new, v_new = kr.decode_qkv(partial, bias, DEC_CTX, preround=preround)
    q64, k64, _ = kr.decode_qkv(partial, bias, DEC_CTX, preround=preround, round_bf16=False)
    ref = kr.decode_attention(q, k_new, v_new, kc, vc, DEC_CTX)
    pv = kr.decode_attention(q, k_new, v_new.abs(), kc, vc.abs(), DEC_CTX)       # sum_j p_j |v_j|
    scale, nflip = _decode_bound(q, k_new, kc, q64, k64)
    tol = (scale[:, :, None] * pv.view(len(DEC_CTX), kr.NH, 64) + 1e-7).view(len(DEC_CTX), -1)
    err = (out - ref).abs()
    print(f"fused={fused} splits={splits}: largest error / bound {(err / tol).max().item():.3g}, "
          f"{nflip} q/k elements near a bf16 boundary, largest bound factor {scale.max().item():.3g}")
    bad = torch.nonzero(err > tol)
    assert len(bad) == 0, [(DEC_CTX[int(b)], int(d) // 64, err[b, d].item(), tol[b, d].item()) for b, d in bad[:8]]
    for b, L in enumerate(DEC_CTX):
        # the appended row: bf16(rope(k_new)) / bf16(v_new) within one bf16 ulp (the fp32 rotation may round the other way)
        assert ((kc_out[b, :, L].double() - k_new[b]).abs() <= kr.bf16_ulp(k_new[b])).all(), L
        assert ((vc_out[b, :, L].double() - v_new[b]).abs() <= kr.bf16_ulp(v_new[b])).all(), L
        # history and the rows after the new one: untouched (bf16-representable input, exact round trip)
        assert torch.equal(kc_out[b, :, :L], kc[b, :, :L]) and torch.equal(vc_out[b, :, :L], vc[b, :, :L]), L
        assert torch.equal(kc_out[b, :, L + 1:], kc[b, :, L + 1:]) and torch.equal(vc_out[b, :, L + 1:], vc[b, :, L + 1:]), L


def test_decode_attention_refusals():
    c = ctx("bf16")
    partial = torch.zeros(1, 1, kr.QKV_N, device="cuda")
    bias = torch.zeros(kr.QKV_N, device="cuda")
    cache = torch.zeros(1, 2, 16, 64, device="cuda")
    out = torch.empty(1, 896, device="cuda")
    lib = c.lib
    for splits, ctx_len, max_ctx in [(0, 0, 16), (1, 16, 16), (1, -1, 16), (1, 0, 8000)]:
        rc = lib.cvk_op_decode_attention(c.h, _p(partial), splits, 1, _p(bias), _p(cache), _p(cache), _ints([ctx_len]), max_ctx, _p(out), _stream())
        assert rc == ERR_INVALID, (splits, ctx_len, max_ctx)
    f = ctx("fp32")
    assert f.lib.cvk_op_decode_attention(f.h, _p(partial), 1, 1, _p(bias), _p(cache), _p(cache), _ints([0]), 16, _p(out), _stream()) == ERR_INVALID


# ================================================================================================ D. conv-GEMM epilogues
EPI_N = [8, 18, 48, 64, 80, 200, 1000]       # BN 64 (N <= 64) and 128; column tails inside a 16-column group and a tile
EPI_K = [8, 24, 72, 1000]                     # TMA K tail zero fill (K % 64 != 0)
EPI_TAPS = [(1, 0, "none"), (3, -2, "mish"), (7, -3, "lrelu")]


def _conv_with(c, x, lens, w, b, shift0, act, **opts):
    for k_, v_ in opts.items():
        c.set_option(k_, v_)
    try:
        return c.conv1d(x, lens, w, b, shift0=shift0, act=act).cpu()
    finally:
        c.set_option("tc_epi", 2)
        c.set_option("op_out_bf16", 0)


@pytest.mark.parametrize("K", EPI_K)
@pytest.mark.parametrize("N", EPI_N)
def test_conv_epilogue_paths_bit_identical(N, K):
    """the TMA-staged epilogue (tc_epi 2, the default) and the direct stores (tc_epi 0) compute the same values; with op_out_bf16 the
    output equals the fp32 output rounded to bf16 (the epilogue rounds once, at the store)"""
    c = ctx("bf16")
    g = torch.Generator().manual_seed(N * 13 + K)
    lens = [300, 45]
    x = _bf16_randn(sum(lens), K, g=g)
    for taps, shift0, act in EPI_TAPS:
        w = _bf16_randn(N, K, taps, g=g, scale=(K * taps) ** -0.5)
        b = torch.randn(N, generator=g) * 0.1
        staged = _conv_with(c, x, lens, w, b, shift0, act)
        direct = _conv_with(c, x, lens, w, b, shift0, act, tc_epi=0)
        assert torch.equal(staged, direct), (N, K, taps, act, (staged - direct).abs().max().item())
        for epi in (2, 0):
            o16 = _conv_with(c, x, lens, w, b, shift0, act, tc_epi=epi, op_out_bf16=1)
            assert torch.equal(o16, kr.bf16(staged)), (N, K, taps, act, epi, (o16 - kr.bf16(staged)).abs().max().item())
        ref = _ref_conv([t.double() for t in torch.split(x, lens)], w.double(), b.double(), 1, shift0, act)
        # bf16 operands exact, fp32 accumulation of K*taps products: 2^-16 sum|x w| (see the skinny GEMM bound); the activations are
        # 1.1-Lipschitz and their fast-exp forms add ~1e-6 relative
        xs = torch.split(x.double().abs(), lens)
        mag = _ref_conv(list(xs), w.double().abs(), None, 1, shift0, "none")
        tol = 1.1 * 2.0 ** -16 * mag + 1e-5 * ref.abs() + 1e-6
        assert ((staged.double() - ref).abs() <= tol).all(), (N, K, taps, act, (staged.double() - ref).abs().max().item())


WIDE_CASES = [(64, 64, 11, 7, -35), (64, 64, 9, 6, -48)]     # (K, N, taps, dil, shift0): reach 35 left / 35 right, 48 left (causal)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("case", WIDE_CASES, ids=["k11d7-centred", "k9d6-causal"])
def test_conv_receptive_field_wider_than_gap(precision, case):
    """ragged batch whose receptive field reaches further than 32 rows: every sequence still convolves with zeros outside itself.
    The middle sequence is 100x larger, so a read into a neighbour is an O(100) error."""
    K, N, taps, dil, shift0 = case
    g = torch.Generator().manual_seed(taps * dil)
    lens = [300, 200, 90]
    xs = [_bf16_randn(L, K, g=g, scale=100.0 if i == 1 else 1.0) for i, L in enumerate(lens)]
    w = _bf16_randn(N, K, taps, g=g, scale=(K * taps) ** -0.5)
    b = torch.randn(N, generator=g) * 0.1
    out = ctx(precision).conv1d(torch.cat(xs), lens, w, b, dil=dil, shift0=shift0).cpu().double()
    ref = _ref_conv([t.double() for t in xs], w.double(), b.double(), dil, shift0, "none")
    mag = _ref_conv([t.double().abs() for t in xs], w.double().abs(), None, dil, shift0, "none")
    # bf16-representable operands: products exact in both modes; fp32 accumulation of K*taps = 704 / 576 terms: n 2^-24 sum|x w| for
    # sequential fp32 sums, plus the 2^-16 tensor-core margin of the bf16 mode
    n = K * taps
    tol = (n * 2.0 ** -24 + 2.0 ** -16) * mag + 1e-6
    err = (out - ref).abs()
    o = 0
    for L in lens:
        print(f"{precision} {case} len {L}: max error {err[o:o + L].max().item():.3g}, max bound {tol[o:o + L].max().item():.3g}")
        o += L
    assert (err <= tol).all(), err.max().item()


def test_conv_refusals():
    c = ctx("bf16")
    x = torch.zeros(16, 8, device="cuda")
    w = torch.zeros(8 * 8 * 3, device="cuda")
    out = torch.empty(16, 8, device="cuda")
    for N, K, taps, dil in [(0, 8, 3, 1), (8, 0, 3, 1), (8, 8, 0, 1), (8, 8, 3, 0)]:
        rc = c.lib.cvk_op_conv1d(c.h, _p(x), _ints([16]), 1, K, _p(w), None, N, taps, dil, 0, 0, _p(out), _stream())
        assert rc == ERR_INVALID, (N, K, taps, dil)
