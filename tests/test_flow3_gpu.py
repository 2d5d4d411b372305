"""GPU: CosyVoice3 flow stage (DiT estimator + CausalMaskedDiffWithDiT.inference, SURVEY.md §8 row a16) through the C ABI against
the committed outputs of the reference modules (tests/golden/dit_*.npz, made by oracle/make_golden.py::gen_dit).

fp32 mode: the reference's export tolerance for an estimator (cosyvoice/bin/export_onnx.py:99-110, rtol 1e-2 / atol 1e-4);
bf16 mode: bounds of twice the largest error measured on an H100, stated and printed next to each assert."""
import numpy as np
import pytest
import torch

from gpu_util import ctx, maxdiff
from oracle import cases, dit, flow, weights

pytestmark = pytest.mark.gpu
_state = {}


def model(precision, depth):
    c = ctx(precision)
    if _state.get(precision) != depth:
        sd = weights.synth_state_dict(dit.flow_param_shapes(depth), 1986, dit.SYNTH_GAINS)
        c.load_state_dict("flow3", sd, cfg=[depth])
        c.set_cfm_noise(flow.cfm_noise(15000)[0].t().contiguous())
        _state[precision] = depth
    return c


def tm(x):          # [B,C,T] -> [B*T, C]
    return x.transpose(1, 2).reshape(-1, x.shape[1]).contiguous()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("tag,depth", [
    ("small", 2),
    ("full", 22),
])
def test_dit_estimator_golden(precision, tag, depth, golden):
    g = golden("dit_" + tag)
    c = model(precision, depth)
    x, mask, mu, t, spks, cond = cases.estimator_case(T=130)
    T = x.shape[2]
    for streaming, key in ((False, "est_offline"), (True, "est_stream")):
        out = c.dit_estimator(tm(x), tm(mu), t, spks, tm(cond), [T, T], streaming=streaming)
        ref = tm(torch.from_numpy(g[key]))
        if precision == "fp32":
            np.testing.assert_allclose(out.cpu().numpy(), ref.numpy(), rtol=1e-2, atol=1e-4)
        else:
            # |out| ~ 0.7; largest |d| measured on an H100 80GB HBM3 (700 W): 8.0e-3 (depth 2, streaming), 4.4e-3 (depth 22); twice
            d = maxdiff(out, ref)
            print(f"[estimator {precision} {tag} streaming={streaming}] max |d| {d:.4g} (bound 0.016)")
            assert d < 0.016, d


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_flow3_inference_golden(precision, golden):
    g = golden("dit_small")
    c = model(precision, 2)
    token, ptok, pfeat, emb = cases.flow_case()
    toks = torch.cat([ptok, token], 1).reshape(-1)
    n = toks.numel()
    for name, streaming, finalize in (("offline", False, True), ("stream_final", True, True), ("stream_chunk", True, False)):
        mel, lens = c.flow3_inference(toks, [n], pfeat[0], [pfeat.shape[1]], emb, streaming=streaming, finalize=finalize)
        ref = torch.from_numpy(g["mel_" + name])[0].t()
        assert lens == [ref.shape[0]]
        d = maxdiff(mel, ref)
        # |mel| ~ 3.7 after ten Euler steps; bf16: largest |d| measured on an H100 80GB HBM3 (700 W) 1.27e-2 (stream_final), twice
        bound = 2e-3 if precision == "fp32" else 0.025
        print(f"[flow3_inference {precision} {name}] max |d| {d:.4g} (bound {bound})")
        assert d < bound, (name, d)


def test_dit_ragged_batch_equals_single(golden):
    """three sequences of different lengths in one call == one call per sequence (32 gap rows isolate the 30-row causal
    position convolution)"""
    c = model("fp32", 2)
    g = torch.Generator().manual_seed(9)
    lens = [70, 131, 33]
    xs = [torch.rand(T, 80, generator=g) for T in lens]
    mus = [torch.rand(T, 80, generator=g) for T in lens]
    conds = [torch.rand(T, 80, generator=g) for T in lens]
    t = torch.rand(3, generator=g)
    spks = torch.rand(3, 80, generator=g)
    out = c.dit_estimator(torch.cat(xs), torch.cat(mus), t, spks, torch.cat(conds), lens, streaming=True)
    o = 0
    for b, T in enumerate(lens):
        single = c.dit_estimator(xs[b], mus[b], t[b:b + 1], spks[b:b + 1], conds[b], [T], streaming=True)
        assert torch.equal(out[o:o + T], single), (b, T, maxdiff(out[o:o + T], single))
        o += T


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("depth", [2, 22])
def test_dit_incremental_stream_equals_prefix_recompute(precision, depth):
    """cvk_flow3_stream_create + the shared session calls for the DiT estimator: K/V rows of every block (rotary positions absolute) and the
    30-row input tails of the two grouped k31 position convolutions per Euler step, against flow3_inference(streaming=True,
    finalize=False) re-run on the growing prefix (what CosyVoice3Model.tts does per chunk, cli/model.py:346-363, 425-450).  Same
    chunk schedule as the CosyVoice2 test: prompt 30 tokens, hops 45 / 25 / 50."""
    c = model(precision, depth)
    g = torch.Generator().manual_seed(78)
    P, hops = 30, (45, 25, 50)
    toks = torch.randint(0, 6561, (P + sum(hops) + 3,), generator=g, dtype=torch.int32)
    pfeat = torch.rand(2 * P, 80, generator=g) * 13.5 - 11.5
    emb = torch.randn(1, 192, generator=g)
    fs = c.flow_stream(max_frames=512, n_timesteps=10, dit=True)
    try:
        c.flow_stream_begin(fs, pfeat, emb)
        n, done = P, 0
        for hop in hops:
            n += hop
            ref, lens = c.flow3_inference(toks[:n + 3], [n + 3], pfeat, [2 * P], emb, streaming=True, finalize=False)
            new = c.flow_stream_chunk(fs, toks[:n + 3])
            want = ref[max(done - 2 * P, 0):]
            assert new.shape == want.shape, (new.shape, want.shape)
            assert torch.isfinite(new).all()
            d = maxdiff(new, want)
            assert d < (1e-5 if precision == "fp32" else 1e-3), (hop, d)
            done = 2 * n
    finally:
        c.flow_stream_destroy(fs)
