"""GPU: ras_sampler_kernel (llm.cu) bit for bit against the oracle (oracle/sampling.py) on both selection paths, in standalone mode
(cvk_ras_sample) and in the decode-graph mode (cvk_op_sample_step: log-softmax of logits, stop / length bookkeeping, next embedding and
the fused layer-0 RMSNorm), plus the log-prob kernel of the text-streaming path (cvk_op_log_softmax) against fp64.

Given identical log-probs and uniforms the ids must be identical.  The library's expf / logf are CUDA's (up to 2 ulp), the oracle's
are numpy's, so "identical" holds only where both see the same probabilities or where no decision is close:
 - the structured families (sampler_refs.families) use a few distinct x - max values.  Every float32 argument the oracle passes to
   exp is evaluated on the device with torch, and a row whose arguments do not all agree bit for bit is rebuilt from the next seed
   (up to 8).  Rows built from 0 and -120 only (exp exactly 1 and 0) always agree: they carry the exact ties, exact prefix sums and
   the cumulative sum landing on 0.8f.  A row that agrees must give the oracle's id;
 - every other row (the generic randn * T rows, structured rows that never agreed) is compared when the oracle's smallest decision
   margin (cum vs 0.8, acc vs thr, neighbouring probabilities among the 26 largest) is at least 8 ulps; the rows below are counted
   and printed.
The walk-divergence row is built on the device's exponential, so that the kernel's fallback probabilities are the construction's."""
import ctypes

import numpy as np
import pytest
import torch

import sampler_refs as sr
from gpu_util import ctx
from oracle import sampling

pytestmark = pytest.mark.gpu

ERR_INVALID = -1
WIDTHS = [6564, 6565, 6567, 6764, 6912]
D = 896
MARGIN_ULPS = 8
_rows = {}


def _dev():
    return torch.device("cuda", 0)


def _agree(args, fn_np, fn_t):
    if len(args) == 0:
        return True
    a = np.unique(np.asarray(args, np.float32))
    d = fn_t(torch.from_numpy(a).to(_dev())).cpu().numpy()
    return np.array_equal(fn_np(a).astype(np.float32).view(np.uint32), d.view(np.uint32))


def _same_math(t):
    """numpy and the device give bitwise-equal exp / log on every argument of this trace"""
    return _agree(t["exp_args"], np.exp, torch.exp) and _agree(t["log_args"], np.log, torch.log)


def _comparable(t):
    """the kernel must give the oracle's id: same probabilities (numpy and the device agree on every exp / log argument) or every
    decision at least MARGIN_ULPS away"""
    return _same_math(t) or t["margin"] >= MARGIN_ULPS


def structured(V):
    """every family of sampler_refs at width V, each row rebuilt from the next seed (up to 8) until the device and numpy agree on
    every exp argument of its standalone trace; a row that never agrees keeps its first seed and is compared under the margin rule.
    Returns a list of dicts(name, want, row, case, s (standalone trace), exact, seed)."""
    if V not in _rows:
        out = []
        for fi, (name, build, want) in enumerate(sr.families()):
            first = None
            for seed in range(8):
                row, case = build(V, np.random.default_rng(1000 * fi + seed))
                ts = sr.trace(row, case["hist"], case["u1"], case["u2"], case["ignore"])
                exact = _same_math(ts)
                first = first or (row, case, ts, seed)
                if exact:
                    break
            else:
                row, case, ts, seed = first
            out.append(dict(name=name, want=want, row=row, case=case, s=ts, exact=exact, seed=seed,
                            comparable=exact or ts["margin"] >= MARGIN_ULPS))
        _rows[V] = out
    return _rows[V]


def decode_oracle(ls, cases):
    """decode-mode expectations from the oracle run on the device's log-probs (cvk_op_log_softmax rows, which the decode step forms
    bit for bit as the write-back checks show): traces for the rows whose exp arguments agree, None for the others"""
    out = []
    for r, k in zip(ls, cases):
        t = sr.trace(r, k["hist"], k["u1"], k["u2"], k["ignore"])
        out.append(t if _comparable(t) else None)
    return out


def _hist_tensor(cases, junk):
    """history rows padded past each count with `junk` (hist_ld > cnt: the kernel must not read past cnt)"""
    ld = max(len(c["hist"]) for c in cases) + 12
    h = np.array([c["hist"] + [j] * (ld - len(c["hist"])) for c, j in zip(cases, junk)], dtype=np.int32)
    return torch.from_numpy(h), torch.tensor([len(c["hist"]) for c in cases], dtype=torch.int32)


def run_standalone(rows, cases):
    """cvk_ras_sample on all rows in one call; the history is padded with each row's own argmax"""
    c = ctx("fp32")
    x = torch.from_numpy(np.stack(rows))
    hist, cnt = _hist_tensor(cases, [int(np.argmax(r)) for r in rows])
    U = torch.tensor([[k["u1"], k["u2"]] for k in cases], dtype=torch.float32)
    ign = torch.tensor([int(k["ignore"]) for k in cases], dtype=torch.int32)
    logp = x.to(_dev()).contiguous()
    dev = [t.to(_dev()).contiguous() for t in (hist, cnt, U, ign)]        # held until the call has finished
    out = torch.empty(len(rows), dtype=torch.int32, device=_dev())
    p = [ctypes.c_void_p(t.data_ptr()) for t in dev]
    rc = c.lib.cvk_ras_sample(c.h, ctypes.c_void_p(logp.data_ptr()), len(rows), x.shape[1], p[0], hist.shape[1], p[1], p[2], p[3],
                              ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert rc == 0
    return out.cpu().numpy().tolist(), logp.cpu().numpy()


class Step:
    """device state of cvk_op_sample_step for B rows (int32 tensors on the device)"""

    def __init__(self, B, V, steps, out_ld, min_len, max_len, base_len, emb, gamma=None, seed=0):
        i32 = dict(dtype=torch.int32, device=_dev())
        g = torch.Generator().manual_seed(seed)
        self.B, self.V = B, V
        self.U = torch.rand(steps, B, 2, generator=g).to(_dev())
        self.min_len, self.max_len = torch.tensor(min_len, **i32), torch.tensor(max_len, **i32)
        self.base_len = torch.tensor(base_len, **i32)
        self.out_ids = torch.full((B, out_ld), -7, **i32)
        self.count, self.done = torch.zeros(B, **i32), torch.zeros(B, **i32)
        self.ctx_len = torch.full((B,), -5, **i32)
        self.live = torch.tensor([B], **i32)
        self.emb = emb.to(_dev()).contiguous()
        self.next_x = torch.zeros(B, D, device=_dev())
        self.gamma = gamma.to(_dev()).contiguous() if gamma is not None else None
        self.xn = torch.zeros(B, D, device=_dev()) if gamma is not None else None

    def run(self, c, logits):
        c.sample_step(logits, self.U, self.min_len, self.max_len, self.out_ids, self.count, self.done, self.ctx_len, self.base_len,
                      self.live, self.emb, self.next_x, self.gamma, self.xn)
        torch.cuda.synchronize()


def run_decode(rows, cases, junk=None):
    """one decode-mode step for rows whose state is the cases' history: count = len(hist), out_ids = history then junk, uniforms at
    [count][b], min_len = count + 1 where eos is ignored (count < min_len) else 0.  Returns (ids or -1 for a stop, written rows, step)."""
    c = ctx("fp32")
    B, V = len(rows), rows[0].shape[0]
    ld = max(len(k["hist"]) for k in cases) + 12
    emb = torch.randn(V, D, generator=torch.Generator().manual_seed(V))
    st = Step(B, V, ld, ld, [len(k["hist"]) + 1 if k["ignore"] else 0 for k in cases], [10 ** 6] * B, [3] * B, emb)
    junk = junk or [int(np.argmax(r)) for r in rows]
    for b, k in enumerate(cases):
        n = len(k["hist"])
        st.out_ids[b] = torch.tensor(k["hist"] + [junk[b]] * (ld - n), dtype=torch.int32)
        st.count[b] = n
        st.U[n, b] = torch.tensor([k["u1"], k["u2"]])
    logits = torch.from_numpy(np.stack(rows)).to(_dev()).contiguous()
    st.run(c, logits)
    cnt = st.count.cpu().numpy()
    out = st.out_ids.cpu().numpy()
    ids = [int(out[b, len(k["hist"])]) if cnt[b] == len(k["hist"]) + 1 else -1 for b, k in enumerate(cases)]
    return ids, logits.cpu().numpy(), st


def _expect_decode_id(t):
    return t["id"] if t["id"] < sr.EOS else -1


def _check_written_decode(ls, written, traces, sel):
    """decode mode writes cvk_op_log_softmax of the logits with the marks, bit for bit"""
    for b in sel:
        exp = ls[b].copy()
        exp[np.isneginf(traces[b]["written"])] = -np.inf
        assert np.array_equal(written[b].view(np.uint32), exp.view(np.uint32)), b
    return ls


@pytest.mark.parametrize("V", WIDTHS)
def test_structured_families(V):
    fam = structured(V)
    rows, cases = [f["row"] for f in fam], [f["case"] for f in fam]
    paths = {"fast": 0, "serial": 0}
    for f in fam:
        got = "serial" if f["s"]["path"]["serial"] else "fast"
        paths[got] += 1
        if f["want"] is not None:
            assert got == f["want"], (f["name"], f["s"]["path"])
    # rows built from 0 and -120 only (exp 1 and 0 on any implementation) decide at exact ties and prefix sums: always compared
    for f in fam:
        if f["name"].startswith(("draw exact prefix", "top-p reached exactly", "underflow k1 ", "ties top-k")):
            assert f["exact"], f["name"]
    ids, written = run_standalone(rows, cases)
    bad = [(f["name"], i, f["s"]["id"]) for f, i in zip(fam, ids) if f["comparable"] and i != f["s"]["id"]]
    assert not bad, bad
    for b, f in enumerate(fam):          # the input back, -inf at the ignored eos and at the id of the first draw when the fallback fired
        if f["comparable"]:
            assert np.array_equal(written[b].view(np.uint32), f["s"]["written"].view(np.uint32)), f["name"]
    ids_d, written_d, st = run_decode(rows, cases)
    ls = ctx("fp32").log_softmax(torch.from_numpy(np.stack(rows))).cpu().numpy()
    td = decode_oracle(ls, cases)
    sel = [b for b, t in enumerate(td) if t is not None]
    bad = [(fam[b]["name"], ids_d[b], td[b]["id"]) for b in sel if ids_d[b] != _expect_decode_id(td[b])]
    assert not bad, bad
    _check_written_decode(ls, written_d, td, sel)
    # cvk_lm_decode == cvk_lm_next_logp + cvk_ras_sample: the log-prob kernel's rows through the standalone sampler give the same ids
    ids_s2, _ = run_standalone(list(ls), cases)
    assert [i if i < sr.EOS else -1 for i in ids_s2] == ids_d
    print(f"V={V}: {len(fam)} structured rows, fast path {paths['fast']}, serial path {paths['serial']}, "
          f"exact exp {sum(f['exact'] for f in fam)}, compared by margin {sum(f['comparable'] and not f['exact'] for f in fam)}, "
          f"not compared {[f['name'] for f in fam if not f['comparable']]}; decode mode against the oracle on {len(sel)} rows")


@pytest.mark.parametrize("V", WIDTHS)
def test_generic_rows(V):
    rows, cases = sr.generic_rows(V, 32, seed=V)
    ts = [sr.trace(r, k["hist"], k["u1"], k["u2"], k["ignore"]) for r, k in zip(rows, cases)]
    td = [sr.trace(r, k["hist"], k["u1"], k["u2"], k["ignore"], from_logits=True) for r, k in zip(rows, cases)]
    keep_s = [b for b, t in enumerate(ts) if t["margin"] >= MARGIN_ULPS]
    keep_d = [b for b, t in enumerate(td) if t["margin"] >= MARGIN_ULPS]
    ids, written = run_standalone(rows, cases)
    assert [ids[b] for b in keep_s] == [ts[b]["id"] for b in keep_s]
    for b in keep_s:
        assert np.array_equal(written[b].view(np.uint32), ts[b]["written"].view(np.uint32)), b
    ids_d, written_d, _ = run_decode(rows, cases)
    assert [ids_d[b] for b in keep_d] == [_expect_decode_id(td[b]) for b in keep_d]
    ls = ctx("fp32").log_softmax(torch.from_numpy(np.stack(rows))).cpu().numpy()
    _check_written_decode(ls, written_d, td, keep_d)
    ids_s2, _ = run_standalone(list(ls), cases)
    assert [i if i < sr.EOS else -1 for i in ids_s2] == ids_d           # kernel against kernel: every row
    paths = sum(t["path"]["serial"] for t in ts)
    fb = sum(t["fallback"] for t in ts)
    print(f"V={V}: {len(rows)} generic rows, excluded by the {MARGIN_ULPS}-ulp margin rule: standalone {len(rows) - len(keep_s)}, "
          f"decode {len(rows) - len(keep_d)}; serial path {paths}, fast path {len(rows) - paths}, fallback {fb}")


@pytest.mark.parametrize("V", [6564, 6764])
def test_walk_divergence_row(V):
    """the fallback walk restarts every segment at its prefix sum (draw_index); carrying the running sum drew the next id"""
    # the row is built on the device's exponential: the kernel's fallback probabilities are then the ones the construction used
    dev_exp = lambda a: torch.exp(torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(_dev())).cpu().numpy()
    row, s, u2 = sr.walk_divergence_case(V, exp=dev_exp)
    sc = row.copy()
    sc[0] = -np.inf
    w = sr.softmax_with(sc, dev_exp)
    first = sr.softmax_with(row, dev_exp)
    assert sampling.nucleus_select(first)[0].tolist() == [0]           # id 0 alone is kept and drawn, then sent to the fallback
    t = dict(id=sampling.draw_index(w, u2), fallback=True)
    assert sr.kernel_walk(w, u2, restart=False) == t["id"] + 1
    per = sr.seg_len(V)
    assert t["fallback"] and t["id"] == (s + 1) * per
    ids, written = run_standalone([row], [dict(hist=[0], u1=0.5, u2=u2, ignore=False)])
    print(f"V={V}: segment {s}, u2={u2!r}: kernel {ids[0]}, oracle {t['id']}")
    assert ids[0] == t["id"]
    assert np.isneginf(written[0][0]) and np.isneginf(written[0]).sum() == 1


def test_cosyvoice3_pad_ids_never_drawn():
    """V = 6764: the 3 pad ids hold -1e30 (probability exactly 0).  A uniform fallback at u2 = 1 - 2^-24 takes the last possible id
    (6760), in decode mode a stop id"""
    V = 6764
    row = np.full(V, -120.0, np.float32)
    row[5] = 0.0
    row[6761:] = -1e30
    case = dict(hist=[5], u1=0.5, u2=1.0 - 2.0 ** -24, ignore=False)
    t = sr.trace(row, case["hist"], case["u1"], case["u2"], False)
    assert t["id"] == 6760
    ids, _ = run_standalone([row], [case])
    assert ids == [6760]
    ids_d, _, st = run_decode([row], [case])
    assert ids_d == [-1] and st.done.item() == 1 and st.live.item() == 0


@pytest.mark.parametrize("V", [6564, 6764])
def test_batch_equals_single(V):
    """64 rows mixed from every family in one call == each row alone, ids and write-back, both modes"""
    fam = structured(V)
    grows, gcases = sr.generic_rows(V, 64 - len(fam), seed=V + 1)
    rows = [f["row"] for f in fam] + grows
    cases = [f["case"] for f in fam] + gcases
    perm = np.random.default_rng(V).permutation(len(rows))[:64]
    rows, cases = [rows[i] for i in perm], [cases[i] for i in perm]
    assert len(rows) == 64
    ids, written = run_standalone(rows, cases)
    ids_d, written_d, st = run_decode(rows, cases)
    for b in range(64):
        i1, w1 = run_standalone([rows[b]], [cases[b]])
        assert i1[0] == ids[b] and np.array_equal(w1[0].view(np.uint32), written[b].view(np.uint32)), b
        i2, w2, _ = run_decode([rows[b]], [cases[b]], junk=[int(np.argmax(rows[b]))])
        assert i2[0] == ids_d[b] and np.array_equal(w2[0].view(np.uint32), written_d[b].view(np.uint32)), b


def _palette_row(g, V, top, pads):
    """a logits row with a dominant id `top` (probability ~0.985 after the log-softmax) over palette values"""
    x = sr._rest(g, V, np.float32(-4.0))
    x[top] = 8.0
    if pads:
        x[6761:] = -1e30
    return x


def _bf16(x):
    return torch.from_numpy(np.asarray(x, np.float32)).to(torch.bfloat16).float().numpy()


def test_decode_bookkeeping():
    """a scripted 6-step run of 5 rows at V = 6764 (CosyVoice3 width, pad ids impossible) against a Python model of llm.py:544-549:
    row 0 stops on id 6562 and row 1 on eos (masked until its min_len 3) in the same step (live drops by 2); row 2 ends on max_len 2;
    row 3 is done from the start (its logits row, ids and count stay untouched); row 4 runs on and stops on id 6760."""
    V, B, steps = 6764, 5, 6
    c = ctx("fp32")
    g = torch.Generator().manual_seed(11)
    emb = torch.randn(V, D, generator=g)
    gamma = torch.randn(D, generator=g)
    min_len, max_len, base = [0, 3, 0, 0, 0], [50, 50, 2, 50, 50], [17, 4, 9, 30, 1]
    st = Step(B, V, steps, 8, min_len, max_len, base, emb, gamma, seed=3)
    st.done[3] = 1
    st.live[0] = B - 1
    st.xn.copy_(torch.from_numpy(_bf16(np.random.default_rng(0).standard_normal((B, D)))).to(_dev()))
    ref_ids = [[] for _ in range(B)]
    done, live = [0, 0, 0, 1, 0], B - 1
    next_x = np.zeros((B, D), np.float32)
    xn = st.xn.cpu().numpy()
    Uh = st.U.cpu().numpy()
    rng = np.random.default_rng(5)
    # dominant id per (step, row): stop ids where the script wants them, eos as the argmax of row 1 from step 0
    script = {(3, 0): 6562, (0, 1): sr.EOS, (1, 1): sr.EOS, (2, 1): sr.EOS, (3, 1): sr.EOS, (5, 4): 6760}
    for step in range(steps):
        rows = []
        for b in range(B):
            top = script.get((step, b), int(rng.integers(0, sr.EOS)))
            x = _palette_row(np.random.default_rng(100 * step + 10 * b), V, top, pads=True)
            cnt = len(ref_ids[b])
            if not done[b]:
                t = sr.trace(x, ref_ids[b], Uh[cnt, b, 0], Uh[cnt, b, 1], cnt < min_len[b], from_logits=True)
                assert _comparable(t), (step, b)
            rows.append(x)
        logits = torch.from_numpy(np.stack(rows)).to(_dev()).contiguous()
        before_done = list(done)
        st.run(c, logits)
        stopped = 0
        for b in range(B):
            if done[b]:
                continue
            cnt = len(ref_ids[b])
            top = sampling.ras_sample(sampling.log_softmax_f32(rows[b]), ref_ids[b], Uh[cnt, b, 0], Uh[cnt, b, 1], cnt < min_len[b])
            assert top < 6761
            if top >= sr.EOS:
                done[b] = 1
                stopped += 1
                continue
            ref_ids[b].append(top)
            next_x[b] = emb[top].numpy()
            e = emb[top].double().numpy()
            r = 1.0 / np.sqrt(np.mean(e * e) + 1e-6)
            xn[b] = gamma.double().numpy() * e * r          # fp64 RMSNorm * gamma, compared within one bf16 ulp below
            if cnt + 1 >= max_len[b]:
                done[b] = 1
                stopped += 1
        live -= stopped
        got_ids, got_cnt = st.out_ids.cpu().numpy(), st.count.cpu().numpy()
        for b in range(B):
            assert got_cnt[b] == len(ref_ids[b]), (step, b)
            assert got_ids[b, :len(ref_ids[b])].tolist() == ref_ids[b], (step, b)
            assert (got_ids[b, len(ref_ids[b]):] == -7).all(), (step, b)
            if ref_ids[b]:
                assert st.ctx_len[b].item() == base[b] + len(ref_ids[b]) - 1, (step, b)
            else:
                assert st.ctx_len[b].item() == -5
        assert st.done.cpu().numpy().tolist() == done, step
        assert st.live.item() == live, step
        assert np.array_equal(st.next_x.cpu().numpy(), next_x), step
        got_xn = st.xn.cpu().numpy()
        for b in range(B):
            if before_done[b] or not ref_ids[b]:
                continue
            ulp = np.spacing(_bf16(np.abs(xn[b])).astype(np.float32)) * 2 ** 16          # bf16 ulp at the value
            assert (np.abs(got_xn[b] - xn[b]) <= ulp).all(), (step, b, np.abs(got_xn[b] - xn[b]).max())
        w = logits.cpu().numpy()
        assert np.array_equal(w[3].view(np.uint32), rows[3].view(np.uint32))          # the done row is not touched
        if step == 3:
            assert before_done[:2] == [0, 0] and done[:2] == [1, 1] and live == 1
    assert done == [1, 1, 1, 1, 1] and st.live.item() == 0
    assert len(ref_ids[2]) == 2 and len(ref_ids[1]) == 3 and ref_ids[1].count(sr.EOS) == 0


def test_log_softmax_against_fp64():
    """cvk_op_log_softmax against an fp64 log-softmax.  The kernel forms y = fl(fl(x - m) - L), L = logf(S), S the float32 sum of
    expf(x - m) in segment order.  Error terms: x - m is exact or within 0.5 ulp of itself; the last subtraction 0.5 ulp of y; S carries
    up to 2 ulp per expf term plus at most (27 + 256) roundings of 2^-24 relative in the two-level sum, which shift L by that relative
    amount (dL = dS / S); logf adds 1 ulp of L.  Bound per entry: ulp(x - m) + ulp(y) + (2 + 283) * 2^-24 + 2 ulp(L)."""
    c = ctx("fp32")
    g = np.random.default_rng(9)
    for V in (6564, 6567, 6764, 6912, 1000, 7):
        x = np.stack([(g.standard_normal(V) * T).astype(np.float32) for T in (0.5, 3.0, 20.0)])
        if V == 6764:
            x[:, 6761:] = -1e30
        y = c.log_softmax(torch.from_numpy(x)).cpu().numpy()
        xd = x.astype(np.float64)
        m = xd.max(1, keepdims=True)
        ref = (xd - m) - np.log(np.exp(xd - m).sum(1, keepdims=True))
        L = np.log(np.exp(xd - m).sum(1, keepdims=True))
        bound = (np.spacing(np.abs(x - m).astype(np.float32)) + np.spacing(np.abs(ref).astype(np.float32)) + 285 * 2.0 ** -24
                 + 2 * np.spacing(L.astype(np.float32)))
        err = np.abs(y - ref)
        fin = ref > -1e29
        assert (err[fin] <= bound[fin]).all(), (V, (err / bound)[fin].max())
        print(f"V={V}: largest error / bound {(err / bound)[fin].max():.3f}")


def test_refusals_leave_context_usable():
    c = ctx("fp32")
    i32 = dict(dtype=torch.int32, device=_dev())
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    for V in (6563, 6913):
        lp = torch.zeros(1, V, device=_dev())
        args = (p(lp), 1, V, p(torch.zeros(1, 4, **i32)), 4, p(torch.zeros(1, **i32)), p(torch.zeros(1, 2, device=_dev())),
                p(torch.zeros(1, **i32)), p(torch.zeros(1, **i32)), s)
        assert c.lib.cvk_ras_sample(c.h, *args) == ERR_INVALID
    V = 6564
    lp = torch.zeros(2, V, device=_dev())
    hist, cnt, U, ign, out = (torch.zeros(2, 4, **i32), torch.zeros(2, **i32), torch.zeros(2, 2, device=_dev()), torch.zeros(2, **i32),
                              torch.zeros(2, **i32))
    assert c.lib.cvk_ras_sample(c.h, p(lp), 0, V, p(hist), 4, p(cnt), p(U), p(ign), p(out), s) == ERR_INVALID
    assert c.lib.cvk_ras_sample(c.h, p(lp), 2, V, p(hist), -1, p(cnt), p(U), p(ign), p(out), s) == ERR_INVALID
    assert c.lib.cvk_ras_sample(c.h, p(lp), 2, V, None, 4, p(cnt), p(U), p(ign), p(out), s) == ERR_INVALID
    emb = torch.zeros(6913, D, device=_dev())
    for prec in ("fp32", "bf16"):
        cc = ctx(prec)
        for V, B, steps, ld, gamma_only, count in ((6563, 1, 4, 4, False, 0), (6913, 1, 4, 4, False, 0), (V, 0, 4, 4, False, 0),
                                                   (V, 1, 0, 4, False, 0), (V, 1, 4, 0, False, 0), (V, 1, 4, 4, True, 0),
                                                   (V, 1, 4, 4, False, 4), (V, 1, 8, 4, False, 4), (V, 1, 4, 4, False, -1)):
            st = Step(max(B, 1), V, max(steps, 1), max(ld, 1), [0], [9], [0], emb[:V], torch.ones(D) if gamma_only else None)
            st.count.fill_(count)
            rc = cc.lib.cvk_op_sample_step(
                cc.h, p(torch.zeros(1, V, device=_dev())), B, V, p(st.U), steps, p(st.min_len), p(st.max_len), p(st.out_ids), ld,
                p(st.count), p(st.done), p(st.ctx_len), p(st.base_len), p(st.live), p(st.emb), p(st.next_x),
                p(st.gamma) if gamma_only else None, None, s)
            assert rc == ERR_INVALID, (prec, V, B, steps, ld, gamma_only, count)
            assert st.count.item() == count and st.live.item() == 1          # nothing ran
        st = Step(1, 6564, 4, 4, [0], [9], [0], emb[:6564])
        rc = cc.lib.cvk_op_sample_step(cc.h, None, 1, 6564, p(st.U), 4, p(st.min_len), p(st.max_len), p(st.out_ids), 4, p(st.count),
                                       p(st.done), p(st.ctx_len), p(st.base_len), p(st.live), p(st.emb), p(st.next_x), None, None, s)
        assert rc == ERR_INVALID
        assert cc.lib.cvk_op_log_softmax(cc.h, None, 1, 10, s) == ERR_INVALID
        assert cc.lib.cvk_op_log_softmax(cc.h, p(lp), 0, 10, s) == ERR_INVALID
        # still usable: one decode step in this context, and a standalone draw
        st = Step(1, 6564, 4, 4, [0], [9], [0], emb[:6564], torch.ones(D))
        logits = torch.full((1, 6564), -5.0, device=_dev())
        logits[0, 42] = 10.0
        st.run(cc, logits)
        assert st.count.item() == 1 and st.out_ids[0, 0].item() == 42 and st.ctx_len.item() == 0
    ids = c.ras_sample(torch.where(torch.arange(6564) == 42, 0.0, -50.0)[None], torch.zeros(1, 1, dtype=torch.int32),
                       torch.zeros(1, dtype=torch.int32), torch.tensor([[0.5, 0.5]]), torch.zeros(1, dtype=torch.int32))
    assert ids.item() == 42
