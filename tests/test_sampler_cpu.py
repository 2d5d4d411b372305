"""CPU: the helpers of test_sampler_gpu.py (sampler_refs.py) before they judge ras_sampler_kernel - the selection-path classifier,
the float32 restatements of the fallback walk, the walk-divergence row and the decision-margin helpers."""
import numpy as np
import pytest

import sampler_refs as sr
from oracle import sampling

WIDTHS = [6564, 6565, 6567, 6764, 6912]


def _prob(x, ignore=False):
    x = np.array(x, dtype=np.float32)
    if ignore:
        x[sr.EOS] = -np.inf
    return sampling.softmax_f32(x)


def test_path_classifier_hand_rows():
    V = 6564                                           # 26 entries per thread, threads 253..255 empty
    flat = np.zeros(V, np.float32)                     # every entry ties: the 25th thread maximum is everyone's key
    st = sr.path_stats(_prob(flat))
    assert st["serial"] and st["count"] == V
    x = np.full(V, -5.0, np.float32)                   # 25 distinct maxima in 25 threads: exactly 25 candidates
    x[np.arange(25) * 26 + 7] = -np.arange(25, dtype=np.float32) * 0.01
    st = sr.path_stats(_prob(x))
    assert not st["serial"] and st["count"] == 25
    x[np.arange(25) * 26 + 7] = -1.0                   # a maximum at id 3 hides thread 0's tied id 7 from the thread maxima, but
    x[3] = 0.0                                         # the 25th-ranked key is still the tie: candidates = the maximum + 25 tied
    st = sr.path_stats(_prob(x))
    assert not st["serial"] and st["count"] == 26
    x = np.full(V, -5.0, np.float32)                   # 24 threads above the rest: the 25th key is the rest, 6540 candidates
    x[np.arange(24) * 26] = 0.0
    st = sr.path_stats(_prob(x))
    assert st["serial"] and st["count"] == V


@pytest.mark.parametrize("V", WIDTHS)
def test_families_reach_their_path(V):
    """each family meant for one selection path reaches it at every width (the GPU test asserts the same on the rows it runs)"""
    counts = {"fast": 0, "serial": 0}
    for name, build, want in sr.families():
        x, c = build(V, np.random.default_rng(7))
        st = sr.path_stats(_prob(x, c["ignore"]))
        counts["serial" if st["serial"] else "fast"] += 1
        if want is not None:
            assert st["serial"] == (want == "serial"), (name, st)
    print(V, counts)


@pytest.mark.parametrize("V", [6564, 6764])
def test_walk_divergence_row(V):
    """on the constructed row the pre-fix walk (running sum carried across segments) and draw_index disagree; the fixed walk agrees"""
    row, s, u2 = sr.walk_divergence_case(V)
    per = sr.seg_len(V)
    sc = row.copy()
    sc[0] = -np.inf
    w = sampling.softmax_f32(sc)
    want = sampling.draw_index(w, u2)
    assert want == (s + 1) * per                       # the tiny first entry of the next segment
    assert sr.kernel_walk(w, u2, restart=True) == want
    assert sr.kernel_walk(w, u2, restart=False) == want + 1
    # through the whole sampler: id 0 is drawn, it is in the window, the fallback draws with u2
    assert sampling.ras_sample(row, [0], 0.5, u2, False) == want
    print(f"V={V}: segment {s}, u2={u2!r}, draw_index {want}, old walk {want + 1}")


@pytest.mark.parametrize("V", [6564, 6567, 6912])
def test_fixed_walk_equals_draw_index(V):
    g = np.random.default_rng(V)
    for trial in range(12):
        w = np.exp(g.standard_normal(V) * (1 + trial)).astype(np.float32)
        w[g.random(V) < (0.2 if trial % 2 else 0.0)] = 0.0
        w = (w / sampling.hsum(w)).astype(np.float32)
        for u in (0.0, 2.0 ** -24, float(g.random()), 1.0 - 2.0 ** -24):
            assert sr.kernel_walk(w, u) == sampling.draw_index(w, u), (trial, u)


def test_margin_helpers_hand_rows():
    w = np.zeros(6564, np.float32)
    w[:4] = 0.25
    assert sr.draw_margin(w, 0.5) == 0.0                                 # thr == 0.5 == the prefix after two entries
    assert sr.draw_margin(w, 0.375) == 2.0 ** 21                         # |0.5 - 0.375| in ulps of 0.5 (2^-24)
    assert sr.ulps(np.float32(0.8), np.nextafter(np.float32(0.8), np.float32(1))) == 1.0
    p = np.zeros(6564, np.float32)
    p[:3] = [0.5, 0.25, 0.25]
    cut, gap = sr.nucleus_margin(p)
    assert cut == 13421773 - 12582912                                    # 0.8f - 0.75 in ulps of 0.8f (2^-24)
    assert gap == 2.0 ** 22                                              # 0.5 - 0.25 in ulps of 0.5


def test_trace_matches_oracle_and_records_arguments():
    V = 6564
    g = np.random.default_rng(3)
    x = (g.standard_normal(V) * 2).astype(np.float32)
    top = int(np.argmax(x))
    t = sr.trace(x, [top], 0.3, 0.6, True, from_logits=True)
    assert t["id"] == sampling.ras_sample(sampling.log_softmax_f32(x), [top], 0.3, 0.6, True)
    assert len(t["log_args"]) == 1 and len(t["exp_args"]) >= 2 * V - 2
    assert np.isneginf(t["written"][sr.EOS])
    if t["fallback"]:
        assert np.isneginf(t["written"]).sum() == 2


@pytest.mark.parametrize("n,kept", [(5, 4), (15, 12)])
def test_exact_topp_rows(n, kept):
    """the cumulative sum of the kept probabilities reaches 0.8f exactly: the strict test stops there"""
    x, c = sr.exact_topp(n)(6564, np.random.default_rng(0))
    p = _prob(x)
    idx, pr = sampling.nucleus_select(p)
    assert len(idx) == kept and np.float32(pr.sum(dtype=np.float32)) == np.float32(0.8)
    assert sampling.ras_sample(x, [], c["u1"], c["u2"], False) == idx[-1]
