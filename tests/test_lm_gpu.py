"""GPU: speech-token LM through the C ABI - sampler bit-exactness, teacher-forced log-probs, KV-cached decode loop.

The sampler is integer bookkeeping over float32 probabilities: given identical log-probs and identical uniforms the
ids must be IDENTICAL to the reference's (tests/golden/sampling.npz, produced by cosyvoice/utils/common.py:138-167
with Tensor.multinomial fed from the same uniforms).  The decode loop in fp32 mode reproduces the reference's ids
token for token; in bf16 mode the log-probs are held to a stated bound instead (free-running ids legitimately
diverge once two candidates are within the bf16 noise)."""
import numpy as np
import pytest
import torch

from gpu_util import ctx, maxdiff
from oracle import cases, lm, sampling

pytestmark = pytest.mark.gpu
_state = {}


def model(precision, NL):
    c = ctx(precision)
    if _state.get(precision) != NL:
        sd = lm.synth_state_dict(NL)
        c.load_state_dict("llm", sd, cfg=[NL])
        _state[precision] = NL
        _state[(precision, "sd")] = sd
    return c, _state[(precision, "sd")]


def test_sampler_matches_reference_ids(golden):
    g = golden("sampling")
    logp, hist, U, ignore = cases.sampling_case()
    c = ctx("fp32")
    cnt = torch.full((logp.shape[0],), hist.shape[1], dtype=torch.int32)
    ids = c.ras_sample(logp, hist, cnt, U, ignore.int())
    assert ids.cpu().tolist() == g["ids"].tolist()


def test_sampler_edge_cases():
    c = ctx("fp32")
    V = 6564
    lp = torch.full((4, V), -float("inf"))
    lp[:, 7] = 0.0
    lp[:, 9] = -20.0
    lp[2:, :] = -30.0
    lp[2:, 6561] = 0.0
    lp[2:, 5] = -1.0
    hist = torch.zeros(4, 12, dtype=torch.int32)
    hist[1, 0] = 7
    cnt = torch.tensor([0, 1, 0, 0], dtype=torch.int32)
    U = torch.tensor([[0.3, 0.3], [0.3, 0.3], [0.0, 0.0], [0.0, 0.0]])
    ign = torch.tensor([0, 0, 1, 0], dtype=torch.int32)
    ids = c.ras_sample(lp, hist, cnt, U, ign).cpu().tolist()
    exp = [sampling.ras_sample(lp[i].numpy(), hist[i, :cnt[i]].tolist(), float(U[i, 0]), float(U[i, 1]), bool(ign[i])) for i in range(4)]
    assert ids == exp == [7, 9, 5, 6561]


@pytest.mark.parametrize("precision,NL", [("fp32", 2), ("bf16", 2), ("fp32", 24), ("bf16", 24)])
def test_teacher_forced_logp(precision, NL, golden):
    g = golden(f"lm_l{NL}")
    c, sd = model(precision, NL)
    text, ptext, ptok, U = cases.lm_case()
    lm_in = lm.build_lm_input(sd, text, ptext, ptok)
    ids = torch.from_numpy(g["ids"][:16]).long()
    full = torch.cat([lm_in, torch.nn.functional.embedding(ids[None], sd["speech_embedding.weight"])], 1)[0]
    logp = c.lm_forward_logp(full, [full.shape[0]])
    ref_rows = torch.from_numpy(g["logp_rows"])                      # reference HF model, last 4 positions, every 41st column
    d = maxdiff(logp[-4:, ::41], ref_rows)
    assert d < (2e-3 if precision == "fp32" else 0.25), d
    # ragged batch of two copies with different lengths == single
    two = c.lm_forward_logp(torch.cat([full, full[:11]], 0), [full.shape[0], 11])
    assert maxdiff(two[:full.shape[0]], logp) < 1e-4
    assert maxdiff(two[full.shape[0]:], logp[:11]) < (1e-3 if precision == "fp32" else 0.1)


def _decode(c, text, ptext, ptok, U, max_ratio=20.0, min_ratio=2.0, steps_per_call=16):
    """batch of rows -> list of id lists.  text/ptext/ptok: lists of [1,n] tensors; U [max_len, B, 2]"""
    B = len(text)
    tl = [int(t.shape[1] + p.shape[1]) for t, p in zip(text, ptext)]
    sl = [int(s.shape[1]) for s in ptok]
    tt = torch.cat([torch.cat([p, t], 1).reshape(-1) for t, p in zip(text, ptext)])
    ss = torch.cat([s.reshape(-1) for s in ptok])
    min_len = torch.tensor([int(t.shape[1] * min_ratio) for t in text], dtype=torch.int32, device=c.device)
    max_len = torch.tensor([int(t.shape[1] * max_ratio) for t in text], dtype=torch.int32, device=c.device)
    mx = int(max_len.max())
    sess = c.lm_session(B, max(tl) + max(sl) + 2 + mx + 8)
    out_ids = torch.zeros(B, mx + 1, dtype=torch.int32, device=c.device)
    out_count = torch.zeros(B, dtype=torch.int32, device=c.device)
    done = torch.zeros(B, dtype=torch.int32, device=c.device)
    Ud = U.to(c.device).float().contiguous()
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        c.lm_prefill(sess, tt, tl, ss, sl)
        n = 0
        while True:
            live = c.lm_decode(sess, steps_per_call, Ud, min_len, max_len, out_ids, out_count, done)
            n += steps_per_call
            if live == 0 or n > mx + steps_per_call:
                break
    torch.cuda.synchronize()
    c.lm_session_destroy(sess)
    cnt = out_count.cpu().tolist()
    return [out_ids[b, :cnt[b]].cpu().tolist() for b in range(B)]


@pytest.mark.parametrize("NL", [2, 24])
def test_decode_ids_match_reference_fp32(NL, golden):
    g = golden(f"lm_l{NL}")
    c, sd = model("fp32", NL)
    text, ptext, ptok, U = cases.lm_case()
    ids = _decode(c, [text], [ptext], [ptok], U[:, None, :])[0]
    assert ids == g["ids"].tolist()


def test_decode_graph_equals_eager():
    c, sd = model("fp32", 2)
    text, ptext, ptok, U = cases.lm_case()
    a = _decode(c, [text], [ptext], [ptok], U[:, None, :])[0]
    c.set_option("use_graph", 0)
    try:
        b = _decode(c, [text], [ptext], [ptok], U[:, None, :])[0]
    finally:
        c.set_option("use_graph", 1)
    assert a == b


def test_decode_ragged_batch_fp32():
    """three rows with different prompts/lengths decode together == the oracle one row at a time"""
    c, sd = model("fp32", 2)
    g = torch.Generator().manual_seed(21)
    rows = []
    for nt, npt, nps in ((5, 3, 7), (9, 4, 12), (3, 2, 0)):
        rows.append((torch.randint(0, 151643, (1, nt), generator=g, dtype=torch.int32), torch.randint(0, 151643, (1, npt), generator=g, dtype=torch.int32),
                     torch.randint(0, 6561, (1, nps), generator=g, dtype=torch.int32)))
    U = torch.rand(200, 3, 2, generator=g)
    got = _decode(c, [r[0] for r in rows], [r[1] for r in rows], [r[2] for r in rows], U, max_ratio=6.0)
    for b, (t, p, s) in enumerate(rows):
        exp = lm.inference(sd, t, p, s, U[:, b], 2, max_ratio=6.0)
        assert got[b] == exp, b


def test_decode_bf16_runs_and_first_token_matches(golden):
    g = golden("lm_l24")
    c, sd = model("bf16", 24)
    text, ptext, ptok, U = cases.lm_case()
    ids = _decode(c, [text], [ptext], [ptok], U[:, None, :])[0]
    assert len(ids) == len(g["ids"]) and all(0 <= i < 6561 for i in ids)
    assert ids[0] == int(g["ids"][0])


def test_decode_weight_streaming_gemm_vs_tiled_bf16():
    """bf16 decode: the split-K weight-streaming GEMM and the tiled wgmma GEMM see the same operands (both runs on the
    one-kernel-per-op attention path); the sampled ids agree until fp32 summation-order noise meets a near-tie (the first
    tokens are required to agree)."""
    c, sd = model("bf16", 2)
    text, ptext, ptok, U = cases.lm_case()
    c.set_option("lm_fused", 0)
    try:
        a = _decode(c, [text], [ptext], [ptok], U[:, None, :])[0]
        c.set_option("use_skinny", 0)
        try:
            b = _decode(c, [text], [ptext], [ptok], U[:, None, :])[0]
        finally:
            c.set_option("use_skinny", 1)
    finally:
        c.set_option("lm_fused", 1)
    n = min(len(a), len(b), 8)
    assert n >= 6 and a[:n] == b[:n], (a[:16], b[:16])


@pytest.mark.parametrize("n_prompt", [9, 420], ids=["short", "long-context"])
def test_decode_fused_kernels_vs_unfused_bf16(n_prompt):
    """bf16 decode: fused (split-K finish + RMSNorm, qkv finish + RoPE + cache append + tensor-core flash-decoding attention,
    SwiGLU epilogue) vs the one-kernel-per-op path (fp32-math attention) on the same weights: the first sampled ids agree
    (24-layer model).  The long prompt puts > 400 keys in the cache, so every warp of the decode attention owns key blocks
    and the cross-warp merge is exercised."""
    c, sd = model("bf16", 24)
    text, ptext, ptok, U = cases.lm_case()
    if n_prompt != ptok.shape[1]:
        ptok = torch.randint(0, 6561, (1, n_prompt), generator=torch.Generator().manual_seed(n_prompt), dtype=torch.int32)
    a = _decode(c, [text], [ptext], [ptok], U[:, None, :])[0]
    c.set_option("lm_fused", 0)
    try:
        b = _decode(c, [text], [ptext], [ptok], U[:, None, :])[0]
    finally:
        c.set_option("lm_fused", 1)
    # random-weight logits are nearly flat: fp32 summation-order noise re-rounded to bf16 flips a nucleus draw after a few tokens
    # (which token depends on the split-K / accumulator partition of the day); the numeric closeness of the two paths is held by
    # test_decode_attention_logits_fused_vs_unfused_bf16, here the first two sampled ids must agree
    n = min(len(a), len(b), 2)
    assert n >= 2 and a[:n] == b[:n], (a[:12], b[:12])


@pytest.mark.parametrize("n_prompt", [9, 150, 420])
def test_decode_attention_logits_fused_vs_unfused_bf16(n_prompt):
    """Numeric check of the tensor-core flash-decoding attention inside the fused decode step.  The log-probs of the SECOND
    decode step (the first token is the arg-max of the prefill distribution on every path; the second distribution is a function
    of every layer's decode attention over the n_prompt + few keys in the cache) are compared with the fp32 context (CUDA-core
    kernels, fp32 everything): the fused bf16 path (bf16 P on mma.sync) must be as close to fp32 as the one-kernel-per-op bf16
    path (fp32-math attention) is - bf16 rounding noise through 24 layers for both, while one
    misplaced fragment element moves the fused path by O(1).  Rows of a batch of 3 have different context lengths."""
    cb, _ = model("bf16", 24)
    cf, _ = model("fp32", 24)
    text, ptext, _, U = cases.lm_case()
    g = torch.Generator().manual_seed(n_prompt)
    ptoks = [torch.randint(0, 6561, (1, n), generator=g, dtype=torch.int32) for n in (n_prompt, max(1, n_prompt // 2), n_prompt + 5)]
    B = len(ptoks)
    tl = [int(text.shape[1] + ptext.shape[1])] * B
    sl = [int(p.shape[1]) for p in ptoks]
    tt = torch.cat([torch.cat([ptext, text], 1).reshape(-1)] * B)
    ss = torch.cat([p.reshape(-1) for p in ptoks])
    U2 = torch.rand(8, B, 2, generator=g)
    U2[:, :, 0] = 1e-4                                   # nucleus draw lands on the most probable id

    def run(c, fused):
        Ud = U2.to(c.device)
        mn = torch.full((B,), 100, dtype=torch.int32, device=c.device)        # no stop inside the 2 steps
        c.set_option("lm_fused", fused)
        try:
            sess = c.lm_session(B, max(tl) + max(sl) + 32)
            ids = torch.zeros(B, 8, dtype=torch.int32, device=c.device)
            cnt = torch.zeros(B, dtype=torch.int32, device=c.device)
            done = torch.zeros(B, dtype=torch.int32, device=c.device)
            st = torch.cuda.Stream()
            torch.cuda.synchronize()
            with torch.cuda.stream(st):
                c.lm_prefill(sess, tt, tl, ss, sl)
                c.lm_decode(sess, 2, Ud, mn, mn, ids, cnt, done)
                out = (c.lm_last_logits(sess, B).cpu(), ids.cpu().clone())
            torch.cuda.synchronize()
            c.lm_session_destroy(sess)
            return out
        finally:
            c.set_option("lm_fused", 1)
    (lt, it), (la, ia), (lb, ib) = run(cf, 0), run(cb, 1), run(cb, 0)
    assert torch.equal(ia[:, :1], it[:, :1]) and torch.equal(ib[:, :1], it[:, :1]), (it, ia, ib)   # same token fed back
    fin = torch.isfinite(lt) & torch.isfinite(la) & torch.isfinite(lb)      # the sampler leaves log-probs in place, -inf on masked ids
    assert fin.float().mean() > 0.99
    d_fused = (la - lt)[fin].abs().max().item()
    d_unfused = (lb - lt)[fin].abs().max().item()
    print(f"n_prompt={n_prompt}: max |logp - fp32| fused {d_fused:.4g}, unfused {d_unfused:.4g} (|logp| up to {lt[fin].abs().max().item():.3g})")
    assert d_fused < 1.5 * d_unfused + 0.05, (d_fused, d_unfused)


def test_bistream_ids_match_reference_fp32(golden):
    """§8 a7, text-streaming LM (llm.py:551-661) through cvk_lm_begin / cvk_lm_feed / cvk_lm_next_logp / cvk_ras_sample and the
    host control flow of B200CosyVoice2Model.lm_generate_bistream: ids identical to the reference's, token for token."""
    from cosyvoice_b200.model import B200CosyVoice2Model
    g = golden("lm_bistream_l2")
    chunks, ptext, ptok, U = cases.bistream_case()
    m = B200CosyVoice2Model(precision="fp32", device=0, workspace_gb=2.0)
    m.ctx.load_state_dict("llm", lm.bistream_state_dict(2), [2])            # LM stage only
    ids = list(m.lm_generate_bistream(iter(chunks), ptext, ptok, uniforms=U))
    assert ids == g["ids"].tolist()
