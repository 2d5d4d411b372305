"""GPU: ragged feeding of an LM session (cvk_lm_feed_rows / cvk_lm_next_logp_rows), lm_generate_bistream_batch and
tts_bistream_batch.

Bounds: fp32 mode reorders no sum that matters, so the ragged forward matches per-row cvk_lm_feed to 1e-4 in log-prob; bf16 mode is
held to the suite's teacher-forced bound, 0.25 (tests/test_lm_gpu.py::test_teacher_forced_logp), since the ragged path runs the
tiled GEMM and the tensor-core attention where cvk_lm_feed runs the weight-streaming GEMM and the CUDA-core decode attention."""
import numpy as np
import pytest
import torch

from gpu_util import maxdiff
from oracle import cases, lm

pytestmark = pytest.mark.gpu
BOUND = {"fp32": 1e-4, "bf16": 0.25}
_c, _m = {}, {}


@pytest.fixture(scope="module", autouse=True)
def _release_contexts():
    """this module's contexts, models and slot caches go before the later modules build theirs"""
    yield
    for k in list(_m):
        _close(_m.pop(k))
    for k in list(_c):
        _c.pop(k).close()
    torch.cuda.empty_cache()


def _close(m):
    """a model's flow sessions, pooled LM sessions and context"""
    torch.cuda.synchronize()
    for fs in m._idle_flow_streams + ([m._slot_pool] if m._slot_pool else []):
        m.ctx.flow_stream_destroy(fs)
    m._idle_flow_streams, m._slot_pool = [], None
    for sessions in m._free_sessions.values():
        for sess in sessions:
            m.ctx.lm_session_destroy(sess)
    m._free_sessions.clear()
    m.ctx.close()


def lm_ctx(precision):
    from cosyvoice_b200 import cvk
    if precision not in _c:
        c = cvk.Context(0, precision, workspace_gb=1.0)
        c.load_state_dict("llm", lm.synth_state_dict(2), cfg=[2])
        _c[precision] = c
    return _c[precision]


def _positions(n, seed):
    """n (id, kind) positions: sos first, then text and speech ids"""
    g = np.random.default_rng(seed)
    ids, kinds = [0], [2]
    for _ in range(n - 1):
        k = int(g.integers(0, 2))
        ids.append(int(g.integers(0, 151643 if k == 0 else 6561)))
        kinds.append(k)
    return ids, kinds


def _single(c, ids, kinds):
    """reference: one B = 1 session fed by cvk_lm_feed; log-probs after the whole feed and after one more speech position"""
    s = c.lm_session(1, 512)
    try:
        c.lm_begin(s, 1)
        c.lm_feed(s, ids, kinds)
        a = c.lm_next_logp(s, 1)
        c.lm_feed(s, [17], [1])
        b = c.lm_next_logp(s, 1)
        return a, b
    finally:
        torch.cuda.synchronize()
        c.lm_session_destroy(s)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("counts", [[1, 5, 20, 30], [1, 5, 20, 70, 130], [130, 70, 130]],
                         ids=["sum56_skinny", "sum226_tiled", "sum330_two_passes"])
def test_feed_rows_matches_per_row_feed(precision, counts):
    c = lm_ctx(precision)
    B = len(counts) + 1                                # the last row is never listed by the big feed
    feeds = [_positions(n, 100 + i) for i, n in enumerate(counts)]
    s = c.lm_session(B, 512)
    try:
        c.lm_begin(s, B)
        c.lm_feed_rows(s, [B - 1], [3], [0, 5, 6], [2, 1, 1])
        quiet = c.lm_next_logp_rows(s, [B - 1]).clone()
        rows = list(range(len(counts)))[::-1]          # listed in reverse order: placement follows the row ids, not the list order
        c.lm_feed_rows(s, rows, [counts[r] for r in rows], [i for r in rows for i in feeds[r][0]], [k for r in rows for k in feeds[r][1]])
        got = c.lm_next_logp_rows(s, list(range(B)))
        assert torch.equal(got[B - 1], quiet[0])        # the unlisted row: bit for bit
        # one more position per row reads every cached position of the feed: the cache contents must match too
        c.lm_feed_rows(s, list(range(B)), [1] * B, [17] * B, [1] * B)
        nxt = c.lm_next_logp_rows(s, list(range(B)))
        torch.cuda.synchronize()
    finally:
        c.lm_session_destroy(s)
    for r, (ids, kinds) in enumerate(feeds):
        a, b = _single(c, ids, kinds)
        da, db = maxdiff(got[r], a[0]), maxdiff(nxt[r], b[0])
        print(f"{precision} counts={counts} row {r} (n={counts[r]}): max |dlogp| {da:.3g}, after one more position {db:.3g}")
        assert da < BOUND[precision] and db < BOUND[precision], (r, da, db)
    a, b = _single(c, [0, 5, 6], [2, 1, 1])
    assert maxdiff(nxt[B - 1], b[0]) < BOUND[precision]


def test_refused_feeds_change_nothing():
    from cosyvoice_b200.cvk import CvkError
    c = lm_ctx("fp32")
    s = c.lm_session(3, 64)
    try:
        c.lm_begin(s, 3)
        c.lm_feed_rows(s, [0, 1, 2], [2, 3, 60], [0, 9] + [0, 9, 10] + [0] + [9] * 59, [2, 1] + [2, 1, 1] + [2] + [0] * 59)
        before = c.lm_next_logp_rows(s, [0, 1, 2]).clone()
        bad = [([0, 0], [1, 1], [5, 5], [1, 1]),             # duplicate row
               ([3], [1], [5], [1]),                          # row >= B
               ([-1], [1], [5], [1]),                         # negative row
               ([0], [0], [], []),                            # empty row
               ([0], [1], [151936], [0]),                     # text id out of range
               ([0], [1], [6564], [1]),                       # speech id out of range
               ([0], [1], [2], [2]),                          # llm_embedding row out of range
               ([0], [1], [5], [3]),                          # unknown kind
               ([0, 2], [1, 5], [5] * 6, [1] * 6)]            # row 2 would pass max_context (60 + 5 > 64)
        for rows, counts, ids, kinds in bad:
            with pytest.raises(CvkError, match="status -1"):
                c.lm_feed_rows(s, rows, counts, ids, kinds)
        for rows in ([1, 1], [3], []):
            with pytest.raises(CvkError, match="status -1"):
                c.lm_next_logp_rows(s, rows)
        after = c.lm_next_logp_rows(s, [0, 1, 2])
        assert torch.equal(before, after)
        c.lm_feed_rows(s, [0, 2], [1, 4], [5] * 5, [1] * 5)   # row 2 up to exactly max_context
        c.lm_begin(s, 2)
        with pytest.raises(CvkError, match="status -1"):
            c.lm_next_logp_rows(s, [0])                       # nothing fed since the begin
        torch.cuda.synchronize()
    finally:
        c.lm_session_destroy(s)


def test_launches_do_not_scale_with_rows():
    c = lm_ctx("bf16")
    s = c.lm_session(8, 256)
    try:
        n = {}
        for B in (1, 8):
            c.lm_begin(s, B)
            c.lm_feed_rows(s, list(range(B)), [4] * B, [0, 5, 6, 7] * B, [2, 1, 1, 1] * B)
            c.lm_next_logp_rows(s, list(range(B)))
            l0 = c.launch_count()
            c.lm_feed_rows(s, list(range(B)), [1] * B, [9] * B, [1] * B)
            c.lm_next_logp_rows(s, list(range(B)))
            n[B] = c.launch_count() - l0
        torch.cuda.synchronize()
    finally:
        c.lm_session_destroy(s)
    print(f"launches of one feed + next-logp step: {n[1]} for 1 row, {n[8]} for 8 rows")
    assert n[8] < 2 * n[1]


def _rechunk(chunks, k):
    flat = torch.cat([x.reshape(-1) for x in chunks])
    return [flat[i:i + k].reshape(1, -1) for i in range(0, flat.numel(), k)]


@pytest.mark.parametrize("variant", ["cosyvoice2", "cosyvoice3"])
def test_batch_ids_equal_single_request_ids_fp32(variant, golden):
    if variant == "cosyvoice2":
        from cosyvoice_b200.model import B200CosyVoice2Model as M
        chunks, ptext, ptok, U = cases.bistream_case()
        sd, g = lm.bistream_state_dict(2), golden("lm_bistream_l2")
    else:
        from cosyvoice_b200.model3 import B200CosyVoice3Model as M
        chunks, ptext, ptok, U = cases.bistream3_case()
        sd, g = lm.bistream_state_dict3(2), golden("lm3_bistream_l2")
    m = M(precision="fp32", device=0, workspace_gb=1.0)
    try:
        m.ctx.load_state_dict("llm", sd, [2])                               # LM stage only
        texts = [chunks, _rechunk(chunks, 1), _rechunk(chunks, 7), _rechunk(chunks, 100)]
        Ub = torch.stack([U] * 4, 1)
        out = [[] for _ in texts]
        for i, tok in m.lm_generate_bistream_batch([iter(t) for t in texts], [ptext] * 4, [ptok] * 4, uniforms=Ub):
            out[i].append(tok)
        assert out[0] == g["ids"].tolist()
        for i, t in enumerate(texts):
            assert out[i] == list(m.lm_generate_bistream(iter(t), ptext, ptok, uniforms=U)), i
    finally:
        _close(m)


def small_model(precision):
    if precision not in _m:
        from cosyvoice_b200.model import B200CosyVoice2Model
        from oracle import flow, hift, weights
        kw = dict(enc_blocks=2, enc_up_blocks=1, num_mid_blocks=2, n_blocks=2)
        m = B200CosyVoice2Model(precision=precision, device=0, workspace_gb=2.0)
        m.load_state_dicts(lm.synth_state_dict(2), weights.synth_state_dict(flow.param_shapes(flow.FlowCfg(**kw)), 1986, flow.SYNTH_GAINS),
                           weights.synth_state_dict(hift.param_shapes(), 1986, hift.SYNTH_GAINS))
        m.stream_batch_slots, m.stream_cache_frames = 4, 1024
        m.stream_pool_headroom = 1 << 30
        m.bistream_max_tokens = 130               # synthetic weights: bound the 'decode until eos' phase
        _m[precision] = m
    return _m[precision]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_tts_bistream_batch_equals_single_requests(precision):
    from test_stream_batch_gpu import noise_fns
    m = small_model(precision)
    _, ptok9, pfeat, emb = cases.flow_case(P=9)
    chunks, ptext, ptok, U = cases.bistream_case()
    other, _, _, U2 = cases.bistream_case(seed=12)
    texts = [chunks, other, _rechunk(chunks, 1)]
    base = dict(flow_embedding=emb, llm_embedding=emb, prompt_text=ptext, llm_prompt_speech_token=ptok, flow_prompt_speech_token=ptok9,
                prompt_speech_feat=pfeat[:, :18])
    Ub = torch.stack([U, U2, U], 1)
    got = [[] for _ in texts]
    for i, out in m.tts_bistream_batch([dict(base, text=iter(t)) for t in texts], uniforms=Ub, noise_fns=noise_fns(3, m.device)):
        got[i].append(out["tts_speech"])
    assert m.token_hop_len == 25 and len(m._free_slots) == m.stream_batch_slots
    for i, t in enumerate(texts):
        if precision == "fp32":
            # fp32: the batched ids equal the single-request ids, so the request alone through tts(stream=True) is the reference
            m.uniforms_override, m.noise_fn, m.token_hop_len = Ub[:, i:i + 1, :], noise_fns(i + 1, m.device)[i], 25
            try:
                single = [o["tts_speech"] for o in m.tts(**dict(base, text=iter(t)), stream=True)]
            finally:
                m.uniforms_override, m.noise_fn, m.token_hop_len = None, None, 25
            bound = 1e-4
        else:
            # bf16: the ragged feed and cvk_lm_feed round differently, so the ids may legitimately differ from tts()'s; a request's
            # ids do not depend on the rows beside it, so the request alone through tts_bistream_batch is the reference of the
            # batched flow / vocoder rounds
            single = [o["tts_speech"] for _, o in m.tts_bistream_batch([dict(base, text=iter(t))], uniforms=Ub[:, i:i + 1],
                                                                      noise_fns=[noise_fns(i + 1, m.device)[i]])]
            bound = 5e-3
        d = maxdiff(torch.cat(got[i], 1), torch.cat(single, 1))
        print(f"{precision} request {i}: chunks {[c.shape[1] for c in got[i]]} (alone {[c.shape[1] for c in single]}), max |dwav| {d:.3g}")
        assert [c.shape[1] for c in got[i]] == [c.shape[1] for c in single], i
        assert d <= bound, (i, d)


def test_bf16_row_results_do_not_depend_on_the_rows_beside_it():
    """a row fed alone and the same row fed beside others (the step's total over 64 and over one 256-position pass, its own positions
    split by the pass boundary) give bit-identical log-probs, and so do the one-position steps after it"""
    c = lm_ctx("bf16")
    ids, kinds = _positions(33, 7)
    big = [_positions(240, 8), _positions(100, 9)]
    out = {}
    for mode in ("alone", "beside"):
        s = c.lm_session(3, 512)
        try:
            c.lm_begin(s, 3)
            if mode == "alone":
                c.lm_feed_rows(s, [1], [33], ids, kinds)
            else:                                      # row 0 first: row 1's positions 16.. fall into the second pass
                c.lm_feed_rows(s, [0, 1, 2], [240, 33, 100], big[0][0] + ids + big[1][0], big[0][1] + kinds + big[1][1])
            a = c.lm_next_logp_rows(s, [1]).clone()
            rows = [1] if mode == "alone" else [0, 1, 2]
            c.lm_feed_rows(s, rows, [1] * len(rows), [17] * len(rows), [1] * len(rows))
            b = c.lm_next_logp_rows(s, [1]).clone()
            torch.cuda.synchronize()
            out[mode] = (a, b)
        finally:
            c.lm_session_destroy(s)
    assert torch.equal(out["alone"][0], out["beside"][0]) and torch.equal(out["alone"][1], out["beside"][1])


def test_bf16_batch_ids_equal_each_row_alone_and_steps_sync_once():
    from cosyvoice_b200.model import B200CosyVoice2Model
    chunks, ptext, ptok, U = cases.bistream_case()
    other, _, _, U2 = cases.bistream_case(seed=12)
    m = B200CosyVoice2Model(precision="bf16", device=0, workspace_gb=1.0)
    try:
        m.ctx.load_state_dict("llm", lm.bistream_state_dict(2), [2])
        texts = [chunks, _rechunk(chunks, 1), other, _rechunk(other, 7)]
        Ub = torch.stack([U, U, U2, U2], 1).to(m.device)
        calls = {"n": 0}
        logp_rows = m.ctx.lm_next_logp_rows

        def counted(*a):
            calls["n"] += 1
            return logp_rows(*a)
        m.ctx.lm_next_logp_rows = counted
        out = [[] for _ in texts]
        import warnings
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                for i, tok in m.lm_generate_bistream_batch([iter(t) for t in texts], [ptext] * 4, [ptok] * 4, uniforms=Ub):
                    out[i].append(tok)
            finally:
                torch.cuda.set_sync_debug_mode("default")
        syncs = sum("synchroniz" in str(x.message) for x in w)
        print(f"bf16 batch: {calls['n']} sampling steps, {syncs} synchronising torch operations")
        assert syncs <= calls["n"] + 4                 # one D2H copy of the drawn ids per step (+ the set-up and the end)
        del m.ctx.lm_next_logp_rows
        for i, t in enumerate(texts):
            alone = [tok for _, tok in m.lm_generate_bistream_batch([iter(t)], [ptext], [ptok], uniforms=Ub[:, i:i + 1])]
            assert out[i] == alone, i
    finally:
        _close(m)


def test_ragged_attention_kernel_matches_fp64():
    """cvk_op_ragged_attention (the tensor-core attention of a feed) against fp64 attention on the same bf16-rounded q / K / V: rows
    with 1..130 queries, paired and unpaired tiles, keys 0..position; position 0 must return v0 itself"""
    c = lm_ctx("bf16")
    g = torch.Generator().manual_seed(3)
    rows, max_ctx = 3, 160
    kc, vc = torch.randn(rows, 2, max_ctx, 64, generator=g), torch.randn(rows, 2, max_ctx, 64, generator=g)
    rowpos = [(0, p) for p in range(0, 5)] + [(1, 17)] + [(2, p) for p in range(20, 150)] + [(1, 40), (1, 41), (1, 42)]
    q = torch.randn(len(rowpos), 896, generator=g) * 2
    out = c.ragged_attention(q, kc, vc, rowpos).cpu().double()
    bf = lambda t: t.to(torch.bfloat16).double()
    qd, kd, vd = bf(q) * 0.125, bf(kc), bf(vc)
    ref = torch.empty_like(out)
    for m_, (r, p) in enumerate(rowpos):
        for h in range(14):
            kvh = h // 7
            s = kd[r, kvh, :p + 1] @ qd[m_, h * 64:(h + 1) * 64]
            ref[m_, h * 64:(h + 1) * 64] = torch.softmax(s, 0) @ vd[r, kvh, :p + 1]
    d = (out - ref).abs().max().item()
    print(f"ragged attention vs fp64: max |d| {d:.3g}")
    assert torch.equal(out[0].float(), bf(torch.cat([vc[0, 0, 0]] * 7 + [vc[0, 1, 0]] * 7)).float())
    assert d < 2e-2, d
