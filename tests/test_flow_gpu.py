"""GPU: flow stage (conformer encoder + CFM estimator + Euler/CFG) through the C ABI against the committed outputs
of the reference (tests/golden/flow_*.npz) and the oracle (oracle/flow.py).

Tolerances: fp32 mode follows the reference's own export check (cosyvoice/bin/export_onnx.py:99-110,
rtol 1e-2 / atol 1e-4 on the estimator); bf16 mode (tensor-core operands, fp32 accumulate and residual stream) is held
to the measured bounds stated next to each assert."""
import numpy as np
import pytest
import torch

from gpu_util import ctx, maxdiff
from oracle import cases, flow, weights

pytestmark = pytest.mark.gpu

CFGS = {"small": dict(enc_blocks=2, enc_up_blocks=1, num_mid_blocks=2, n_blocks=2),
        "full": dict(enc_blocks=6, enc_up_blocks=4, num_mid_blocks=12, n_blocks=4)}
_state = {}


def model(precision, tag):
    c = ctx(precision)
    if _state.get(precision) != tag:
        cfg = flow.FlowCfg(**CFGS[tag])
        sd = weights.synth_state_dict(flow.param_shapes(cfg), 1986, flow.SYNTH_GAINS)
        c.load_state_dict("flow", sd, cfg=[cfg.enc_blocks, cfg.enc_up_blocks, cfg.num_mid_blocks, cfg.n_blocks])
        c.set_cfm_noise(flow.cfm_noise(15000)[0].t().contiguous())
        _state[precision] = tag
        _state[(precision, "sd")] = sd
    return c, _state[(precision, "sd")], flow.FlowCfg(**CFGS[tag])


def tm(x):          # [B,C,T] -> [B*T, C]
    return x.transpose(1, 2).reshape(-1, x.shape[1]).contiguous()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("tag", ["small", "full"])
def test_estimator_golden(precision, tag, golden):
    g = golden("flow_" + tag)
    c, sd, cfg = model(precision, tag)
    x, mask, mu, t, spks, cond = cases.estimator_case()
    T = x.shape[2]
    for streaming, key in ((False, "est_offline"), (True, "est_stream")):
        out = c.cfm_estimator(tm(x), tm(mu), t, spks, tm(cond), [T, T], streaming=streaming)
        ref = tm(torch.from_numpy(g[key]))
        d = maxdiff(out, ref)
        if precision == "fp32":
            np.testing.assert_allclose(out.cpu().numpy(), ref.numpy(), rtol=1e-2, atol=1e-4)
        else:
            assert d < 0.15, d          # bf16 operands through 14 resnets + 56 transformer blocks (|out| ~ 3)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("tag", ["small", "full"])
def test_encoder_golden(precision, tag, golden):
    g = golden("flow_" + tag)
    c, sd, cfg = model(precision, tag)
    token, ptok, pfeat, emb = cases.flow_case()
    toks = torch.cat([ptok, token], 1).reshape(-1)
    h = c.flow_encoder(toks, [toks.numel()], streaming=False, context_len=0)
    ref = torch.from_numpy(g["enc_offline"])[0]
    d = maxdiff(h, ref)
    assert d < (2e-3 if precision == "fp32" else 0.25), d     # after_norm output, unit scale


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("tag", ["small", "full"])
def test_inference_golden(precision, tag, golden):
    g = golden("flow_" + tag)
    c, sd, cfg = model(precision, tag)
    token, ptok, pfeat, emb = cases.flow_case()
    toks = torch.cat([ptok, token], 1).reshape(-1)
    for name, streaming, finalize in (("offline", False, True), ("stream_final", True, True), ("stream_chunk", True, False)):
        if "mel_" + name not in g:
            continue
        mel, lens = c.flow_inference(toks, [toks.numel()], pfeat[0], [pfeat.shape[1]], emb, streaming=streaming, finalize=finalize)
        ref = torch.from_numpy(g["mel_" + name])[0].t()
        assert mel.shape == ref.shape
        d = maxdiff(mel, ref)
        assert d < (5e-3 if precision == "fp32" else 0.5), (name, d)      # mel after 10 Euler steps, |mel| ~ 5


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_ragged_batch_vs_oracle(precision):
    """three utterances of different length in one call == the oracle run one utterance at a time"""
    c, sd, cfg = model(precision, "small")
    g = torch.Generator().manual_seed(9)
    utts = []
    for N, P in ((17, 6), (40, 25), (9, 3)):
        utts.append((torch.randint(0, 6561, (1, N), generator=g, dtype=torch.int32), torch.randint(0, 6561, (1, P), generator=g, dtype=torch.int32),
                     torch.rand(1, 2 * P, 80, generator=g) * 13.5 - 11.5, torch.randn(1, 192, generator=g)))
    toks = torch.cat([torch.cat([p, t], 1).reshape(-1) for t, p, _, _ in utts])
    tl = [t.shape[1] + p.shape[1] for t, p, _, _ in utts]
    pf = torch.cat([f[0] for _, _, f, _ in utts], 0)
    pl = [f.shape[1] for _, _, f, _ in utts]
    emb = torch.cat([e for _, _, _, e in utts], 0)
    mel, lens = c.flow_inference(toks, tl, pf, pl, emb)
    o = 0
    for (t, p, f, e), L in zip(utts, lens):
        ref = flow.inference(sd, t, p, f, e, cfg)[0].t()
        assert L == ref.shape[0]
        d = maxdiff(mel[o:o + L], ref)
        assert d < (5e-3 if precision == "fp32" else 0.5), d
        o += L


def test_persistent_gemm_flow_bit_identical():
    """A batch large enough for the persistent wgmma GEMM path (tiles > SMs; bf16 and fp32 outputs, second outputs, residual /
    per-sequence-vector epilogues): the whole flow is bit-identical with the path switched off."""
    c, sd, cfg = model("bf16", "small")
    g = torch.Generator().manual_seed(31)
    B = 12
    n_tok = [int(x) for x in torch.randint(200, 330, (B,), generator=g)]
    toks = torch.cat([torch.randint(0, 6561, (n + 40,), generator=g, dtype=torch.int32) for n in n_tok])
    tl = [n + 40 for n in n_tok]
    pf = torch.randn(B * 80, 80, generator=g)
    emb = torch.randn(B, 192, generator=g)
    outs = []
    for on in (2, 0):
        c.set_option("tc_persist", on)
        try:
            mel, lens = c.flow_inference(toks, tl, pf, [80] * B, emb, n_timesteps=3)
            outs.append(mel.clone())
        finally:
            c.set_option("tc_persist", 2)
    assert lens == [2 * n for n in n_tok]
    assert torch.isfinite(outs[0]).all()
    assert torch.equal(outs[0], outs[1]), maxdiff(outs[0], outs[1])


@pytest.mark.parametrize("tag", ["small", "full"])
def test_encoder_relpos_attention_tensor_core_vs_cuda_core(tag):
    """the conformer relative-position attention on the wgmma kernels (position scores by relpos_u_kernel, added as a bias inside the
    one-pass attention kernel) against the CUDA-core flash kernel it replaces (same bf16 operands, fp32 math): ragged batch, offline
    and with the streaming chunk masks + look-ahead context.  Output = after_norm rows, unit scale."""
    c, sd, cfg = model("bf16", tag)
    g = torch.Generator().manual_seed(5)
    lens = [203, 77, 150]
    toks = torch.randint(0, 6561, (sum(lens),), generator=g, dtype=torch.int32)
    for streaming, ctxl in ((False, 0), (True, 3)):
        outs = []
        for on in (1, 0):
            c.set_option("enc_tc_attn", on)
            try:
                outs.append(c.flow_encoder(toks, lens, streaming=streaming, context_len=ctxl).clone())
            finally:
                c.set_option("enc_tc_attn", 1)
        assert torch.isfinite(outs[0]).all()
        d = maxdiff(outs[0], outs[1])
        assert d < 0.06, (streaming, d)          # bf16 re-rounding of P / of the intermediate activations through 3 (small) / 10 (full) layers


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("tag", ["small", "full"])
def test_incremental_stream_equals_prefix_recompute(precision, tag):
    """cvk_flow_stream_* (cached K/V + causal-conv tails per Euler step) against the reference's schedule, which re-runs
    flow.inference(streaming=True, finalize=False) on the growing prefix for every chunk (cli/model.py:346-363): same frames, chunk by
    chunk.  Prompt of 30 tokens -> first hop padded to the 25-token grid (45), then hops of 25 and 50; the first chunk's prompt
    rows are computed (they are attended to) but not returned.  Every row's arithmetic is the same sequence of operations in both
    schedules (row-independent GEMMs, keys visited in the same order), so the bound is round-off, not a model tolerance."""
    c, sd, cfg = model(precision, tag)
    g = torch.Generator().manual_seed(77)
    P, hops = 30, (45, 25, 50)
    toks = torch.randint(0, 6561, (P + sum(hops) + 3,), generator=g, dtype=torch.int32)
    pfeat = torch.rand(2 * P, 80, generator=g) * 13.5 - 11.5
    emb = torch.randn(1, 192, generator=g)
    fs = c.flow_stream(max_frames=512, n_timesteps=10)
    try:
        assert c.flow_stream_bytes(fs) > 0
        c.flow_stream_begin(fs, pfeat, emb)
        n, done = P, 0
        for hop in hops:
            n += hop
            ref, lens = c.flow_inference(toks[:n + 3], [n + 3], pfeat, [2 * P], emb, streaming=True, finalize=False)
            assert lens == [2 * n - 2 * P]
            new = c.flow_stream_chunk(fs, toks[:n + 3])
            want = ref[max(done - 2 * P, 0):]
            assert new.shape == want.shape, (new.shape, want.shape)
            assert torch.isfinite(new).all()
            d = maxdiff(new, want)
            assert d < (1e-5 if precision == "fp32" else 1e-3), (hop, d)
            done = 2 * n
        # a second utterance on the same session object: begin() resets the caches
        c.flow_stream_begin(fs, pfeat, emb)
        ref, _ = c.flow_inference(toks[:P + 45 + 3], [P + 45 + 3], pfeat, [2 * P], emb, streaming=True, finalize=False)
        new = c.flow_stream_chunk(fs, toks[:P + 45 + 3])
        assert maxdiff(new, ref) < (1e-5 if precision == "fp32" else 1e-3)
        # a chunk end off the 50-frame grid is refused (the caches would not be exact), and so is a call without new frames
        from cosyvoice_b200.cvk import CvkError
        with pytest.raises(CvkError):
            c.flow_stream_chunk(fs, toks[:P + 45 + 10 + 3])
        with pytest.raises(CvkError):
            c.flow_stream_chunk(fs, toks[:P + 45 + 3])
    finally:
        c.flow_stream_destroy(fs)


@pytest.mark.parametrize("precision", ["fp32"])
def test_engine_estimator_inplace_contract(precision, golden):
    """INTEGRATION.md §2 executed: cosyvoice_b200.engine.CvkEstimator at the reference's TensorRT swap point
    (flow_matching.py:126-153) - channel-major [2,80,T] tensors in, result written over x."""
    from cosyvoice_b200.engine import CvkEstimator
    g = golden("flow_small")
    c, sd, cfg = model(precision, "small")
    est = CvkEstimator(None, context=c)
    x, mask, mu, t, spks, cond = cases.estimator_case()
    xd = x.clone().cuda()
    ret = est(xd, mask.cuda(), mu.cuda(), t.cuda(), spks.cuda(), cond.cuda(), streaming=False)
    assert ret.data_ptr() == xd.data_ptr()
    np.testing.assert_allclose(xd.cpu().numpy(), g["est_offline"], rtol=1e-2, atol=1e-4)
    cap, high = c.workspace_bytes()
    assert 0 < high <= cap
