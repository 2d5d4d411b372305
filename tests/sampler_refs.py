"""Python restatements and case builders for the repetition-aware sampler tests (test_sampler_cpu.py, test_sampler_gpu.py).

The yardstick for ids is the oracle (oracle/sampling.py).  This module adds what the oracle does not say:
 - which selection path ras_sampler_kernel (llm.cu) takes for a row: the fast candidate-list path or the serial rounds;
 - float32 restatements of the kernel's fallback walk before and after the prefix fix, and a row on which they differ;
 - a trace of the oracle that records every float32 argument it feeds to exp / log and its smallest decision margins;
 - the row families of the GPU test."""
import numpy as np

from oracle import sampling

SEG = sampling.SEG                 # 256 sampler threads, one contiguous segment each
TOPK = sampling.TOP_K
EOS = 6561
CAND_CAP = 512                     # candidate-list capacity of the fast path
F32 = np.float32


def seg_len(V):
    return (V + SEG - 1) // SEG


# ------------------------------------------------------------------------------------------------ selection path
def path_stats(prob):
    """The selection path of ras_sampler_kernel for probabilities `prob` [V] (after the eos mask and the softmax), restated from
    llm.cu (the block before `constexpr int CAND_CAP`): every thread's maximum key (float bits + 1, lowest index on ties), the key
    ranked 25th among the 256 (key desc, index asc), and the number of entries whose key is at or above it.  More than 512 such
    entries send the row to the serial rounds.  Returns dict(thr_key, count, serial)."""
    prob = np.asarray(prob, dtype=F32)
    V = prob.shape[0]
    per = seg_len(V)
    keys = prob.view(np.uint32).astype(np.int64) + 1
    tk = []
    for t in range(SEG):
        lo, hi = t * per, min(t * per + per, V)
        if lo >= hi:
            tk.append((0, 0x7FFFFFFF))
            continue
        j = lo + int(np.argmax(keys[lo:hi]))           # argmax returns the first (lowest) index of the maximum
        tk.append((int(keys[j]), j))
    ranked = sorted(tk, key=lambda kv: (-kv[0], kv[1]))
    thr = ranked[TOPK - 1][0]
    count = int((keys >= thr).sum()) if thr else 0
    return dict(thr_key=thr, count=count, serial=thr == 0 or count > CAND_CAP)


# ------------------------------------------------------------------------------------------------ fallback walk
def _segments(w):
    w = np.asarray(w, dtype=F32)
    V = w.shape[0]
    per = seg_len(V)
    part = np.zeros(SEG, dtype=F32)
    for s in range(SEG):
        a = F32(0)
        for i in range(s * per, min(s * per + per, V)):
            a = F32(a + w[i])
        part[s] = a
    return w, V, per, part


def kernel_walk(w, u, restart=True):
    """float32 restatement of the fallback draw of ras_sampler_kernel (thread 0 after the segment sums): find the first non-empty
    segment whose prefix sum exceeds thr = u * total, walk it, continue into later non-empty segments.  restart=True starts every
    segment at its own prefix sum (the kernel since the fix, == oracle draw_index); restart=False carries the element-by-element
    running sum across segments (the kernel before the fix)."""
    w, V, per, part = _segments(w)
    pre = F32(0)
    for s in range(SEG):
        pre = F32(pre + part[s])
    thr = F32(F32(u) * pre)
    acc, segi, lastseg, segbase, lastbase = F32(0), -1, -1, F32(0), F32(0)
    for s in range(SEG):
        if part[s] > 0:
            lastseg, lastbase = s, acc
            if F32(acc + part[s]) > thr:
                segi, segbase = s, acc
                break
        acc = F32(acc + part[s])
    if segi < 0:
        segi, segbase = lastseg, lastbase
    pick, last, sgbase, a = -1, -1, segbase, segbase
    for sg in range(segi, SEG):
        if pick >= 0:
            break
        a0 = sgbase
        sgbase = F32(sgbase + part[sg])
        if sg > segi and not part[sg] > 0:
            continue
        if restart:
            a = a0
        for i in range(sg * per, min(sg * per + per, V)):
            if w[i] > 0:
                last = i
            a = F32(a + w[i])
            if a > thr and w[i] > 0:
                pick = i
                break
    return pick if pick >= 0 else last


# ------------------------------------------------------------------------------------------------ margins
def ulps(a, b):
    """|a - b| in float32 ulps of the larger magnitude"""
    a, b = F32(a), F32(b)
    return float(abs(np.float64(a) - np.float64(b)) / np.spacing(max(abs(a), abs(b), F32(1e-38))))


def draw_margin(w, u):
    """smallest distance, in ulps, between thr = u * total and a running sum that draw_index compares with it: the segment prefix
    sums up to the chosen segment and the element sums inside it"""
    w, V, per, part = _segments(w)
    prefix = np.zeros(SEG + 1, dtype=F32)
    for s in range(SEG):
        prefix[s + 1] = F32(prefix[s] + part[s])
    thr = F32(F32(u) * prefix[SEG])
    m = float("inf")
    for s in range(SEG):
        if part[s] <= 0:
            continue
        m = min(m, ulps(prefix[s + 1], thr))
        if prefix[s + 1] > thr:
            a = prefix[s]
            for i in range(s * per, min(s * per + per, V)):
                a = F32(a + w[i])
                if w[i] > 0:
                    m = min(m, ulps(a, thr))
                if a > thr and w[i] > 0:
                    return m
    return m


def nucleus_margin(prob):
    """smallest |cum - 0.8| (ulps) over the nucleus's cum < top_p tests, and the smallest relative gap (ulps) between neighbours
    among the 26 largest probabilities (the order that decides which ids are kept)"""
    order = np.argsort(-prob.astype(np.float64), kind="stable")
    cum, m = F32(0), float("inf")
    for n, i in enumerate(order[:TOPK]):
        m = min(m, ulps(cum, sampling.TOP_P)) if cum > 0 else m
        if not cum < F32(sampling.TOP_P):
            break
        cum = F32(cum + prob[i])
    else:
        if cum > 0:
            m = min(m, ulps(cum, sampling.TOP_P))
    top = prob[order[:TOPK + 1]]
    gap = min((ulps(top[j], top[j + 1]) for j in range(len(top) - 1) if top[j] != top[j + 1]), default=float("inf"))
    return m, gap


# ------------------------------------------------------------------------------------------------ traced oracle
def trace(row, hist, u1, u2, ignore_eos, from_logits=False):
    """oracle.sampling.ras_sample on `row` (log-probs, or logits when from_logits, as the decode step takes them) with the
    float32 arguments it passes to exp and log, its smallest decision margin, the path of the first selection and the row the
    kernel writes back.  Returns a dict."""
    row = np.asarray(row, dtype=F32)
    exp_args, log_args = [], []
    if from_logits:
        d = (row - np.max(row)).astype(F32)
        exp_args.append(d)
        s = sampling.hsum(np.exp(d).astype(F32))
        log_args.append(np.array([s], dtype=F32))
        scores = sampling.log_softmax_f32(row)
    else:
        scores = row.copy()
    sc = scores.copy()
    if ignore_eos:
        sc[EOS] = -np.inf
    fin = ~np.isneginf(sc)
    exp_args.append((sc - np.max(sc)).astype(F32)[fin])
    prob = sampling.softmax_f32(sc)
    idx, pr = sampling.nucleus_select(prob)
    m_cut, m_gap = nucleus_margin(prob)
    m_draw = draw_margin(pr, u1)
    top = int(idx[sampling.draw_index(pr, u1)])
    rep = sum(1 for t in list(hist)[-sampling.WIN_SIZE:] if t == top)
    fallback = rep >= 1
    if fallback:
        sc[top] = -np.inf
        fin = ~np.isneginf(sc)
        exp_args.append((sc - np.max(sc)).astype(F32)[fin])
        p2 = sampling.softmax_f32(sc)
        m_draw = min(m_draw, draw_margin(p2, u2))
        top = int(sampling.draw_index(p2, u2))
    assert top == sampling.ras_sample(scores, list(hist), u1, u2, ignore_eos)
    return dict(id=top, exp_args=np.concatenate(exp_args), log_args=np.concatenate(log_args) if log_args else np.zeros(0, F32),
                margin=min(m_cut, m_gap, m_draw), path=path_stats(prob), fallback=fallback, written=sc)


# ------------------------------------------------------------------------------------------------ the walk-divergence row
def softmax_with(x, exp):
    """oracle.sampling.softmax_f32 with the exponential supplied (np.exp, or the device's, to build a row on the kernel's own
    probabilities)"""
    x = np.asarray(x, dtype=F32)
    e = np.asarray(exp((x - np.max(x)).astype(F32)), dtype=F32)
    e[np.isneginf(x)] = 0
    return (e / sampling.hsum(e)).astype(F32)


def walk_divergence_case(V, s=None, d_other=-4.6051702, d_tiny=-16.118095, exp=np.exp):
    """A standalone-mode row on which the pre-fix fallback walk and draw_index pick different ids.  Id 0 holds 12 (probability
    ~0.9994: the nucleus keeps it alone, it is drawn, and the history [0] sends the row to the fallback).  In the fallback
    distribution, segment s holds 1 (relative weight 1), the first entry of segment s + 1 holds d_tiny (weight ~1e-7, below half an
    ulp of the running sum) and every other entry d_other (weight ~1e-2).  u2 puts thr in [E, P), E being the element-by-element sum
    through segment s and P = prefix[s + 1]: draw_index restarts segment s + 1 at P and takes its first entry, the old walk carries E
    and takes the second.  Returns (row, s, u2) for the first s (from s on, default the middle) where such a u2 exists.  `exp` is the
    exponential the fallback probabilities are formed with."""
    per = seg_len(V)
    for seg in range(SEG // 2 if s is None else s, (V - 1) // per - 1):
        row = np.full(V, d_other, dtype=F32)
        row[seg * per:(seg + 1) * per] = 0.0
        row[(seg + 1) * per] = d_tiny
        row[0] = 12.0
        sc = row.copy()
        sc[0] = -np.inf
        w = softmax_with(sc, exp)
        w_, _, _, part = _segments(w)
        prefix = F32(0)
        for t in range(seg):
            prefix = F32(prefix + part[t])
        E = prefix
        for i in range(seg * per, (seg + 1) * per):
            E = F32(E + w[i])
        P = F32(prefix + part[seg])
        total = F32(0)
        for t in range(SEG):
            total = F32(total + part[t])
        if not (E < P and F32(E + w[(seg + 1) * per]) == E):
            continue
        u = F32(np.float64(E) / np.float64(total))
        for _ in range(64):
            thr = F32(u * total)
            if E <= thr < P:
                return row, seg, float(u)
            u = np.nextafter(u, F32(1) if thr < E else F32(0))
    raise AssertionError("no divergence row found")


# ------------------------------------------------------------------------------------------------ row families
# Every builder takes (V, rng) and returns (row, case); case = dict(hist, u1, u2, ignore).  Rows are built from a few distinct
# x - max values (multiples of 1/32, so that the float32 differences the sampler forms are exact), so the GPU test can check that
# numpy's exp / log and the device's agree on every argument and rebuild the row from another seed when they do not.
def _pal(g, n=6):
    return (g.choice(np.arange(1, 65), n, replace=False) * F32(-1 / 32)).astype(F32)


def _rest(g, V, base):
    return (base + g.choice(_pal(g), V)).astype(F32)


def _case(g, hist=(), u1=None, u2=None, ignore=False):
    return dict(hist=[int(h) for h in hist], u1=float(g.random() if u1 is None else u1), u2=float(g.random() if u2 is None else u2),
                ignore=bool(ignore))


def _case_fb(g, x, fallback, **kw):
    c = _case(g, **kw)
    if fallback:              # the id the first draw takes goes into the window
        c["hist"] = [sampling.ras_sample(x, [], c["u1"], c["u2"], False)]
    return c


def underflow(k, spread, fallback=False):
    """k entries near the maximum, all others below max - 110 (fp32 exp is exactly 0 there).  packed: k consecutive ids (fewer than
    25 segments: serial rounds); spread: one id per segment (fast path once k >= 25).  fallback: the maximum is in the window (k = 1:
    the fallback draws from a uniform distribution over the V - 1 others)."""
    def build(V, g):
        per = seg_len(V)
        x = np.full(V, -120.0, dtype=F32)
        if spread:
            ids = g.choice((V - 1) // per, size=k, replace=False) * per + g.integers(0, per, size=k)
        else:
            start = int(g.integers(0, V - k))
            ids = np.arange(start, start + k)
        vals = g.choice(np.append(_pal(g), F32(0)), size=k).astype(F32)
        vals[0] = 0.0
        x[ids] = vals
        return x, _case_fb(g, x, fallback)
    return build


def ties_topk(n_tie):
    """n_tie entries tied at the maximum, the rest at -3: top-k cuts inside the tie.  40 tied ids in 40 segments (the 25th thread
    maximum is the tie: 40 candidates, fast path, index tie-break); 600 tied ids every 10th id (600 > 512 candidates: serial)."""
    def build(V, g):
        per = seg_len(V)
        x = np.full(V, -3.0, dtype=F32)
        if n_tie <= 200:
            ids = np.sort(g.choice((V - 1) // per, size=n_tie, replace=False)) * per + per - 1     # last id of each chosen segment
        else:
            ids = np.arange(n_tie) * 10 + int(g.integers(0, 10))
        x[ids] = 0.0
        return x, _case(g)
    return build


def ties_topp(V, g):
    """16 tied ids straddling a segment boundary, rest at -9.25: top-p cuts inside the tied block"""
    per = seg_len(V)
    x = np.full(V, -9.25, dtype=F32)
    b0 = int(g.integers(2, 200)) * per - 8
    x[b0:b0 + 16] = 0.0
    return x, _case(g)


def ties_offset(V, g):
    """one maximum and 30 ids tied at x - max = -1.5, one per segment, across the 25th place"""
    per = seg_len(V)
    x = np.full(V, -6.0, dtype=F32)
    ids = np.arange(30) * per + per // 2 + int(g.integers(0, per // 2))
    x[ids] = -1.5
    x[int(g.integers(0, V))] = 0.0
    return x, _case(g)


def clustered(where, rest):
    """the 26 largest in one or two segments: ids 0..25, the last 26 ids, or across the boundary of segment 13.  rest 'flat': every
    other id equal (serial rounds, the owner's 3-deep cache rebuilt 8 times); 'spread': 30 more ids at -5.5, one in each of 30 other
    segments (fast path: 56 candidates, 26 of them in one or two threads)."""
    def build(V, g):
        per = seg_len(V)
        start = {"first": 0, "last": V - 26, "boundary": 13 * per - 13}[where]
        x = np.full(V, -6.0, dtype=F32)
        if rest == "spread":
            x[(np.arange(30) + 40) * per + int(g.integers(0, per))] = -5.5
        x[start:start + 26] = (np.arange(26) * F32(-1 / 16)).astype(F32)
        return x, _case(g, hist=[start + int(g.integers(0, 4))] if rest == "flat" else ())
    return build


def window(cnt, back):
    """the argmax (drawn with probability ~0.985) sits at position cnt - back of a cnt-long history: back 1 and 10 are inside the
    window of 10 (fallback), back 11 is not"""
    def build(V, g):
        x = _rest(g, V, F32(-4.0))
        top = int(g.integers(0, EOS))
        x[top] = 8.0
        hist = [int(h) if h != top else (top + 1) % EOS for h in g.integers(0, EOS, cnt)]
        if cnt:
            hist[cnt - back] = top
        return x, _case(g, hist=hist)
    return build


def eos_argmax(ignore):
    def build(V, g):
        x = _rest(g, V, F32(-4.0))
        x[EOS] = 6.0
        return x, _case(g, ignore=ignore)
    return build


def draw_edge(u, fallback):
    """u1 = u2 = u on a row with six ids near the maximum; fallback: the id of the first draw is in the window"""
    def build(V, g):
        x = _rest(g, V, F32(-5.0))
        x[:6] = np.array([0.0, -0.25, -0.5, -0.75, -1.0, -1.25], dtype=F32)
        return x, _case_fb(g, x, fallback, u1=u, u2=u)
    return build


def exact_prefix(u):
    """four ids at the maximum, every other impossible: kept weights 1/4 each, u * total = u lands exactly on a prefix sum and the
    strict test acc > thr takes the next id"""
    def build(V, g):
        x = np.full(V, -120.0, dtype=F32)
        x[[3, 300, 301, 4000]] = 0.0
        return x, _case(g, u1=u)
    return build


def exact_topp(n):
    """n ids at the maximum, every other impossible: probabilities 1/n, and for n = 5 and 15 the float32 cumulative sum reaches
    0.8f exactly (after 4 / 12 ids), where cum < 0.8 stops the nucleus.  u1 = 1 - 2^-24 draws the last kept id."""
    def build(V, g):
        x = np.full(V, -120.0, dtype=F32)
        x[np.arange(n) * 100 + 7] = 0.0
        return x, _case(g, u1=1.0 - 2.0 ** -24)
    return build


U_EDGES = (0.0, 2.0 ** -24, 0.5, 1.0 - 2.0 ** -24)


def families():
    """(name, builder, intended path: 'fast' / 'serial' / None)"""
    f = []
    for k in (1, 2, 24, 25, 26, 40):
        f.append((f"underflow k{k} packed", underflow(k, False), "serial"))
        f.append((f"underflow k{k} spread", underflow(k, True), "fast" if k >= TOPK else "serial"))
        f.append((f"underflow k{k} fallback", underflow(k, False, fallback=True), "serial"))
    f += [("ties top-k 40", ties_topk(40), "fast"), ("ties top-k 600", ties_topk(600), "serial"), ("ties top-p", ties_topp, "serial"),
          ("ties offset block", ties_offset, "fast")]
    for where in ("first", "last", "boundary"):
        f.append((f"clustered {where} flat", clustered(where, "flat"), "serial"))
        f.append((f"clustered {where} spread", clustered(where, "spread"), "fast"))
    for u in U_EDGES:
        f.append((f"draw u={u!r}", draw_edge(u, False), None))
        f.append((f"draw fallback u={u!r}", draw_edge(u, True), None))
    for u in (0.25, 0.5, 0.75):
        f.append((f"draw exact prefix u={u}", exact_prefix(u), "serial"))
    for n in (5, 15):
        f.append((f"top-p reached exactly n={n}", exact_topp(n), "serial"))
    for cnt in (0, 1, 9, 10, 11, 40):
        for back in ((1,) if cnt == 0 else tuple(b for b in (1, 10, 11) if b <= cnt)):
            f.append((f"window cnt{cnt} at cnt-{back}", window(cnt, back), None))
    f += [("eos argmax ignored", eos_argmax(True), None), ("eos argmax", eos_argmax(False), None)]
    return f


def generic_rows(V, n, seed):
    """family 1: randn * T log-probs, T from 0.5 to 6.5 (as the golden case, at any width); every other row carries one of its five
    most likely ids in the window, every third ignores eos"""
    g = np.random.default_rng(seed)
    rows, cases = [], []
    for r, T in enumerate(np.linspace(0.5, 6.5, n)):
        x = (g.standard_normal(V) * T).astype(F32)
        top5 = np.argsort(-x)[:5]
        cnt = int(g.integers(0, 30))
        hist = [int(v) for v in g.integers(0, EOS, cnt)]
        if r % 2 and cnt:
            hist[-1 - int(g.integers(0, min(cnt, 10)))] = int(top5[int(g.integers(0, 5))])
        rows.append(x)
        cases.append(_case(g, hist=hist, ignore=r % 3 == 0))
    return rows, cases
