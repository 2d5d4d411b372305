"""GPU: the CosyVoice3 DiT estimator (stage "flow3") block by block against the fp64 DiT of tests/kernel_refs.py, read through the
test-only cvk_dit_hidden (the fp32 residual stream after the input embedding and the first n blocks):
 A. stage isolation, fp32 and bf16, offline and streaming (block-causal, 50-frame chunks): hidden(0) against the fp64 input embedding,
    hidden(i+1) against fp64 block i fed the kernel's own hidden(i).  The fp32 context is held to the exact reference, the bf16 one
    to the reference that rounds to bf16 where the bf16 path stores bf16 (kernel_refs.DIT_ROUNDING) - both with the same t-dependent
    modulation vectors, computed in fp64 from t, so the single fp32 modulation GEMM and its SiLU output are checked on the way;
    single sequences of 1 .. 129 frames (the 50-frame chunk, the 64- and 128-row tiles), one sequence of 2000 frames (rotary
    positions up to 1999, many query and key tiles) and a ragged batch of six;
 B. identities: every sequence of a 64-sequence ragged batch (a CFG-doubled batch of 32) alone equals its rows of the batch bit for
    bit, in both precisions, for hidden(depth) and the estimator output; two runs agree bit for bit; an n_blocks outside
    [0, depth] is refused;
 C. the 22-block stack at T = 130 (two sequences) and T = 500 against both references.

The weights are kernel_refs.dit_test_state_dict: gates ~ 1, t different per sequence.  Each context is private to this module (the
shared gpu_util contexts keep the weights test_flow3_gpu.py loaded) and is closed at its end.

Bounds (kernel_refs.DIT_TOL, DIT_STACK_TOL, where the measurements are listed): an element's error over the rms of its row of the
stage's contribution - x0 for the embedding, x_out - x (the gated attention and feed-forward terms) for a block.  They are measured,
not derived: a worst-case propagation of the fp32 and bf16 roundings through two 1984-term convolutions, or through the three fp32
GEMMs of the time MLP into the gates, comes out at O(1) on values of O(1).  Each bound is about twice the largest ratio measured on an
H100 80GB HBM3 (700 W), and each case prints its own.  Which defects the bounds catch, per mode, is pinned on the CPU by
test_kernel_refs_cpu.py::test_dit_mutations_exceed_bounds:
  caught in fp32 and bf16: rotary on rotate-half pairs, rotary on all 16 heads, key positions shifted by one against the queries,
    AdaLN shift and scale swapped, the modulation row of the neighbouring sequence, block-causal chunk 48 instead of 50, a chunk
    edge one key late, SiLU in place of Mish in the position convolution, the time-embedding frequency divisor 128 instead of 127;
  caught in fp32 only: the exact-erf GELU in place of the tanh form (5 % of the elements);
  caught in neither: LayerNorm eps 1e-5 instead of 1e-6 (a 5e-6 relative change of the normalised rows)."""
import pytest
import torch

import kernel_refs as kr

pytestmark = pytest.mark.gpu

DEPTH = 2
SEED = 31
SINGLE = [1, 2, 49, 50, 51, 64, 65, 128, 129]
LAYOUTS = {"single": [[T] for T in SINGLE], "long": [[2000]], "ragged": [[37, 50, 51, 64, 65, 129]]}

_models = {}


def _model(precision, depth=DEPTH):
    """(context, fp64 weights); one private context per precision and depth, closed at the end of the module"""
    if (precision, depth) not in _models:
        from cosyvoice_b200 import cvk
        c = cvk.Context(0, precision, workspace_gb=4.0)
        sd = kr.dit_test_state_dict(depth, SEED)
        c.load_state_dict("flow3", sd, cfg=[depth])
        _models[(precision, depth)] = (c, kr.dit_weights(sd, depth))
    return _models[(precision, depth)]


@pytest.fixture(scope="module", autouse=True)
def _release_models():
    yield
    for c, _ in _models.values():
        c.close()
    _models.clear()
    torch.cuda.empty_cache()


def _case(lens, seed):
    """x, mu, cond [sum T, 80] in [-1, 1), spks [B, 80], all bf16-representable (the bf16 path packs them as bf16); t [B] distinct in
    [0.05, 0.95]"""
    g = torch.Generator().manual_seed(seed)
    R, B = sum(lens), len(lens)
    x, mu, cond = (kr.bf16(torch.rand(R, 80, generator=g) * 2 - 1) for _ in range(3))
    spks = kr.bf16(torch.randn(B, 80, generator=g))
    t = 0.05 + 0.9 * torch.rand(B, generator=g)
    return x, mu, cond, spks, t


def _row_rms(t):
    return t.pow(2).mean(-1, keepdim=True).sqrt()


def _ratio(err, scale, what):
    r = (err / scale).max().item()
    assert r == r, f"{what}: NaN"
    return r


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("streaming", [0, 1])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_dit_stages(precision, streaming, layout):
    c, W = _model(precision)
    bf = precision == "bf16"
    chunk = 50 if streaming else 0
    tol = kr.DIT_TOL[precision]
    worst = {}
    for n, lens in enumerate(LAYOUTS[layout]):
        x, mu, cond, spks, t = _case(lens, 100 * n + 7 * streaming + len(lens))
        hid = [c.dit_hidden(x, mu, t, spks, cond, lens, i, streaming=bool(streaming)).cpu().double() for i in range(DEPTH + 1)]
        mod = kr.dit_modulation(W, t.double())["mod"]
        emb = kr.dit_input_embedding(W, x, mu, cond, spks, lens, rounding=bf)["x0"]
        r = _ratio((hid[0] - emb).abs(), _row_rms(emb), "embedding")
        assert r <= tol["embed"], f"{precision} {layout} lens {lens}: embedding error / row rms {r:.3g} > {tol['embed']}"
        worst["embed"] = max(worst.get("embed", 0.0), r)
        for i in range(DEPTH):
            st = kr.dit_block(W, i, hid[i], mod, lens, chunk, rounding=bf)
            r = _ratio((hid[i + 1] - st["x_out"]).abs(), _row_rms(st["x_out"] - st["x"]), f"block {i}")
            assert r <= tol["block"], f"{precision} {layout} lens {lens}: block {i} error / row rms of its contribution {r:.3g} > {tol['block']}"
            worst["block"] = max(worst.get("block", 0.0), r)
    print(f"[{precision} streaming={streaming} {layout}] largest error / row rms: " +
          ", ".join(f"{k} {v:.3g} (bound {tol[k]})" for k, v in worst.items()))


def _batch_lens():
    """64 sequences: 32 lengths in [1, 300] (every tile and chunk edge class), each twice as the CFG doubling lays them out"""
    g = torch.Generator().manual_seed(64)
    half = torch.randint(1, 301, (32,), generator=g).tolist()
    half[:6] = [1, 50, 51, 64, 128, 129]
    return half + half


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_dit_batch_rows_bit_identical(precision):
    """each of 64 sequences computed alone equals its rows of the ragged batch, bit for bit (streaming and offline), and two batch
    runs agree bit for bit: no kernel on the path lets a row depend on its neighbours or on the batch size"""
    c, _ = _model(precision)
    lens = _batch_lens()
    x, mu, cond, spks, t = _case(lens, 640)
    for streaming in (True, False):
        hb = c.dit_hidden(x, mu, t, spks, cond, lens, DEPTH, streaming=streaming)
        ob = c.dit_estimator(x, mu, t, spks, cond, lens, streaming=streaming)
        assert torch.equal(hb, c.dit_hidden(x, mu, t, spks, cond, lens, DEPTH, streaming=streaming)), "hidden: run to run"
        assert torch.equal(ob, c.dit_estimator(x, mu, t, spks, cond, lens, streaming=streaming)), "estimator: run to run"
        o = 0
        for b, T in enumerate(lens):
            args = (x[o:o + T], mu[o:o + T], t[b:b + 1], spks[b:b + 1], cond[o:o + T], [T])
            assert torch.equal(c.dit_hidden(*args, DEPTH, streaming=streaming), hb[o:o + T]), (precision, streaming, b, T, "hidden")
            assert torch.equal(c.dit_estimator(*args, streaming=streaming), ob[o:o + T]), (precision, streaming, b, T, "estimator")
            o += T


def test_dit_hidden_refuses_n_blocks_out_of_range():
    """n_blocks < 0 or > depth is refused before any device work; the context then computes what it computed before"""
    from cosyvoice_b200.cvk import CvkError
    c, _ = _model("bf16")
    lens = [70, 33]
    x, mu, cond, spks, t = _case(lens, 5)
    before = c.dit_hidden(x, mu, t, spks, cond, lens, DEPTH, streaming=True)
    for n in (-1, DEPTH + 1):
        with pytest.raises(CvkError):
            c.dit_hidden(x, mu, t, spks, cond, lens, n, streaming=True)
    assert torch.equal(before, c.dit_hidden(x, mu, t, spks, cond, lens, DEPTH, streaming=True))


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_dit_stack_22_blocks(precision):
    """hidden(22) and the estimator output of the full-depth DiT against the exact and the bf16-emulating fp64 references.  Errors
    relative to the reference's rms (the residual stream's, the output's)."""
    c, W = _model(precision, 22)
    tol = kr.DIT_STACK_TOL[precision]
    for lens in ([130, 130], [500]):
        x, mu, cond, spks, t = _case(lens, 22 + len(lens))
        hid = c.dit_hidden(x, mu, t, spks, cond, lens, 22, streaming=True).cpu().double()
        out = c.dit_estimator(x, mu, t, spks, cond, lens, streaming=True).cpu().double()
        line = []
        for ref_name, rounding in (("exact", False), ("bf16-emulating", True)):
            h_ref, o_ref = kr.dit_estimator(W, x, mu, cond, spks, t, lens, True, rounding)
            eh = ((hid - h_ref).abs().max() / _row_rms(h_ref).mean()).item()
            eo = ((out - o_ref).abs().max() / _row_rms(o_ref).mean()).item()
            line.append(f"{ref_name}: hidden {eh:.3g} (bound {tol[ref_name][0]}), output {eo:.3g} (bound {tol[ref_name][1]})")
            assert eh <= tol[ref_name][0] and eo <= tol[ref_name][1], (precision, lens, ref_name, eh, eo)
        print(f"[22 blocks, {precision}, lens {lens}] largest error / rms: " + "; ".join(line))
