"""GPU: the CosyVoice2 flow (stage "flow") unit by unit against the fp64 flow of tests/kernel_refs.py, read through the test-only
cvk_flow_encoder_hidden and cvk_cfm_estimator_hidden (the fp32 residual stream after the first n units):
 A. stage isolation, fp32 and bf16, offline and streaming (block-causal: 25 tokens before the up-sampler, 50 frames after it and in
    the estimator), on the config (2, 2, 2, 2).  Each unit is fed the kernel's own read-out of the unit before and checked against
    the fp64 unit: the fp32 context against the exact reference, the bf16 one against the reference that rounds where the bf16 path
    stores bf16 (kernel_refs.FLOW_ROUNDING).  Encoder: unit 0 (embedding + PreLookahead) against enc_embed, each conformer layer, the
    up-sampler + up_embed, each up layer, and after_norm through cvk_flow_encoder; 1 .. 375 tokens with no and with 3 look-ahead
    tokens, and a ragged batch of very different lengths (the position table is sized by the longest).  Estimator: every resnet
    (the first mid one with down_blocks.0.2) and transformer block, and the tail through cvk_cfm_estimator; single sequences of 1 ..
    257 frames (the 50-frame chunk, the 64- and 128-row tiles), of 750 (the benchmark's longest) and 1500 frames (30 chunks), a
    ragged six, and a CFG pair laid out as cfm_solve_packed lays it out (zero mu / spks / cond in the second half);
 B. identities, bit for bit: each sequence of a 64-sequence estimator batch at the benchmark's lengths (550 .. 750 frames, CFG
    doubled) and of a 32-utterance encoder batch (275 .. 375 tokens) alone equals its rows of the batch, for every read-out and the
    output; two runs agree; an n outside its range is refused;
 C. the full config (6, 4, 12, 4) on 275 + 375 tokens and 550 + 750 frames: the whole encoder and the 70-unit estimator against
    both references.

The weights are kernel_refs.flow_test_state_dict.  Each context is private to this module (the shared gpu_util contexts keep the
weights test_flow_gpu.py loaded) and is closed at its end.  Bounds: kernel_refs.FLOW_TOL and FLOW_STACK_TOL, where the measurements
are listed; every case prints its ratios, and each test asserts after its cases have printed.  They are measured on an H100, not
derived, and set at about twice the largest ratio.  Which defects the bounds catch, per mode, is pinned on the CPU by
test_kernel_refs_cpu.py::test_flow_mutations_exceed_bounds:
  caught in fp32 and bf16: block-causal chunk 48 instead of 50 and a chunk edge one frame late in the estimator, chunk 24 instead of
    25 in the encoder, the neighbouring stage's time projection, the time projection added before Mish, the skip and x halves of the
    up stage swapped, a centred instead of causal k3 padding, SiLU for Mish, the time-embedding divisor 160 instead of 159,
    pos_bias_u / v swapped, rel_shift one position off, 2 look-ahead rows instead of 3, the up-sampler's left pad 3 instead of 4,
    the embedding without its x sqrt(512);
  caught in fp32 only: the tanh GELU in place of the exact erf (the bf16 path computes the tanh form itself);
  caught in neither: LayerNorm eps 1e-6 instead of 1e-5 in the estimator, or 1e-5 instead of 1e-12 in the encoder."""
import pytest
import torch

import kernel_refs as kr
from oracle import flow as oflow

pytestmark = pytest.mark.gpu

SMALL = (2, 2, 2, 2)
FULL = (6, 4, 12, 4)
SEED = 23
EST_SINGLE = [1, 2, 3, 49, 50, 51, 64, 65, 127, 128, 129, 257]
EST_LAYOUTS = {"single": [[T] for T in EST_SINGLE], "long": [[750], [1500]], "ragged": [[37, 50, 51, 64, 65, 129]], "cfg": [[200, 200]]}
ENC_SINGLE = [1, 2, 3, 4, 24, 25, 26, 50, 64, 65, 128, 129, 375]
ENC_LAYOUTS = {"single": [[T] for T in ENC_SINGLE], "ragged": [[4, 375, 26, 129]]}

_models = {}


def _model(precision, cfg=SMALL):
    """(context, fp64 weights); one private context per precision and config, closed at the end of the module"""
    if (precision, cfg) not in _models:
        from cosyvoice_b200 import cvk
        c = cvk.Context(0, precision, workspace_gb=6.0)
        sd = kr.flow_test_state_dict(oflow.FlowCfg(*cfg), SEED)
        c.load_state_dict("flow", sd, cfg=list(cfg))
        _models[(precision, cfg)] = (c, kr.flow_weights(sd, oflow.FlowCfg(*cfg)))
    return _models[(precision, cfg)]


@pytest.fixture(scope="module", autouse=True)
def _release_models():
    yield
    for c, _ in _models.values():
        c.close()
    _models.clear()
    torch.cuda.empty_cache()


def _est_case(lens, seed, cfg_pair=False):
    """x, mu, cond [sum T, 80] in [-1, 1), spks [B, 80], all bf16-representable (the bf16 path packs them as bf16); t [B] distinct in
    [0.05, 0.95].  cfg_pair: the second half of the batch repeats the first half's x with zero mu / spks / cond, as cfm_solve_packed
    lays out the two classifier-free-guidance branches"""
    g = torch.Generator().manual_seed(seed)
    R, B = sum(lens), len(lens)
    x, mu, cond = (kr.bf16(torch.rand(R, 80, generator=g) * 2 - 1) for _ in range(3))
    spks = kr.bf16(torch.randn(B, 80, generator=g))
    t = 0.05 + 0.9 * torch.rand(B, generator=g)
    if cfg_pair:
        h, Rh = B // 2, sum(lens[:B // 2])
        x[Rh:] = x[:Rh]
        mu[Rh:], cond[Rh:], spks[h:] = 0.0, 0.0, 0.0
    return x, mu, cond, spks, t


def _tokens(lens, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 6561, (sum(lens),), generator=g, dtype=torch.int32)


def _row_rms(t):
    return t.pow(2).mean(-1, keepdim=True).sqrt()


def _ratio(got, ref, scale, what):
    r = ((got - ref).abs() / scale).max().item()
    assert r == r, f"{what}: NaN"
    return r


def _report(tag, worst, tol):
    print(f"[{tag}] largest error / row rms: " + ", ".join(f"{k} {v:.3g} (bound {tol[k]})" for k, v in worst.items()))
    bad = {k: v for k, v in worst.items() if not v <= tol[k]}
    assert not bad, f"{tag}: over the bound: {bad}"


def _est_hidden_all(c, args, n_units, streaming):
    return [c.cfm_estimator_hidden(*args, n, streaming=streaming).cpu().double() for n in range(1, n_units + 1)]


@pytest.mark.parametrize("layout", list(EST_LAYOUTS))
@pytest.mark.parametrize("streaming", [0, 1])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_estimator_units(precision, streaming, layout):
    c, W = _model(precision)
    cfg = W["cfg"]
    bf = precision == "bf16"
    rd = kr.bf16 if bf else (lambda v: v)
    nst, per = cfg.num_mid_blocks + 2, 1 + cfg.n_blocks
    chunk = 50 if streaming else 0
    tol = kr.FLOW_TOL[precision]
    worst = dict(est_resnet=0.0, est_block=0.0, est_out=0.0)
    for n, lens in enumerate(EST_LAYOUTS[layout]):
        x, mu, cond, spks, t = _est_case(lens, 100 * n + 7 * streaming + len(lens), cfg_pair=layout == "cfg")
        args = (x, mu, t, spks, cond, lens)
        hid = _est_hidden_all(c, args, nst * per, bool(streaming))
        out = c.cfm_estimator(*args, streaming=bool(streaming)).cpu().double()
        temb = kr.est_time(W, t.double())["temb"]
        acts = {-1: kr.est_pack(x, mu, cond, spks, lens, bf)}
        line = {}
        for k in range(nst):
            u = k * per
            st = kr.est_resnet(W, k, kr.est_stage_input(W, k, acts, lens, bf), temb, lens, bf)
            r = _ratio(hid[u], st["x_out"], _row_rms(st["x_out"]), f"stage {k} resnet")
            line["est_resnet"] = max(line.get("est_resnet", 0.0), r)
            for j in range(cfg.n_blocks):
                st = kr.est_tblock(W, k, j, hid[u + j], lens, chunk, bf)
                r = _ratio(hid[u + j + 1], st["x_out"], _row_rms(st["x_out"] - st["x"]), f"stage {k} block {j}")
                line["est_block"] = max(line.get("est_block", 0.0), r)
            acts[k] = rd(hid[u + per - 1])
        ref = kr.est_tail(W, acts[nst - 1], lens, bf)
        line["est_out"] = _ratio(out, ref, _row_rms(ref), "tail")
        print(f"  {precision} streaming={streaming} lens {lens if len(lens) < 8 else len(lens)}: " +
              ", ".join(f"{k} {v:.3g}" for k, v in line.items()))
        for k, v in line.items():
            worst[k] = max(worst[k], v)
    _report(f"estimator {precision} streaming={streaming} {layout}", worst, tol)


@pytest.mark.parametrize("context_len", [0, 3])
@pytest.mark.parametrize("layout", list(ENC_LAYOUTS))
@pytest.mark.parametrize("streaming", [0, 1])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_encoder_units(precision, streaming, layout, context_len):
    c, W = _model(precision)
    cfg = W["cfg"]
    bf = precision == "bf16"
    ne = cfg.enc_blocks
    tol = kr.FLOW_TOL[precision]
    worst = dict(enc_embed=0.0, enc_layer=0.0, enc_up=0.0, enc_out=0.0)
    for n, out_lens in enumerate(ENC_LAYOUTS[layout]):
        lens = [L + context_len for L in out_lens]
        tok = _tokens(lens, 31 * n + streaming + 5 * context_len)
        hid = [c.flow_encoder_hidden(tok, lens, i, ne, streaming=bool(streaming), context_len=context_len).cpu().double()
               for i in range(ne + 2 + cfg.enc_up_blocks)]
        out = c.flow_encoder(tok, lens, streaming=bool(streaming), context_len=context_len).cpu().double()
        line = {}
        ref = kr.enc_embed(W, tok, lens, context_len, bf)["x"]
        line["enc_embed"] = _ratio(hid[0], ref, _row_rms(ref), "embedding")
        for i in range(ne):
            st = kr.enc_layer(W, f"encoder.encoders.{i}", hid[i], out_lens, 25 if streaming else 0, bf)
            r = _ratio(hid[i + 1], st["x_out"], _row_rms(st["x_out"] - st["x"]), f"layer {i}")
            line["enc_layer"] = max(line.get("enc_layer", 0.0), r)
        ref = kr.enc_upsample(W, hid[ne], out_lens, bf)["y"]
        line["enc_up"] = _ratio(hid[ne + 1], ref, _row_rms(ref), "up-sampler")
        lens2 = [2 * L for L in out_lens]
        for i in range(cfg.enc_up_blocks):
            st = kr.enc_layer(W, f"encoder.up_encoders.{i}", hid[ne + 1 + i], lens2, 50 if streaming else 0, bf)
            r = _ratio(hid[ne + 2 + i], st["x_out"], _row_rms(st["x_out"] - st["x"]), f"up layer {i}")
            line["enc_layer"] = max(line["enc_layer"], r)
        ref = kr.enc_after_norm(W, hid[-1])
        line["enc_out"] = _ratio(out, ref, _row_rms(ref), "after_norm")
        print(f"  {precision} streaming={streaming} context {context_len} tokens {out_lens}: " +
              ", ".join(f"{k} {v:.3g}" for k, v in line.items()))
        for k, v in line.items():
            worst[k] = max(worst[k], v)
    _report(f"encoder {precision} streaming={streaming} context {context_len} {layout}", worst, tol)


def _bench_frames(n, seed):
    """n token counts of the benchmark's requests (75 prompt tokens + 5 x (40 .. 60) text tokens: 275 .. 375), with 275 and 375"""
    g = torch.Generator().manual_seed(seed)
    toks = (275 + torch.randint(0, 101, (n,), generator=g)).tolist()
    toks[:2] = [275, 375]
    return toks


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_estimator_batch_rows_bit_identical(precision):
    """each of 64 sequences (32 benchmark lengths of 550 .. 750 frames, CFG doubled) computed alone equals its rows of the batch,
    bit for bit, for every read-out and the output, streaming and offline; two batch runs agree bit for bit"""
    c, W = _model(precision)
    cfg = W["cfg"]
    n_units = (cfg.num_mid_blocks + 2) * (1 + cfg.n_blocks)
    half = [2 * n for n in _bench_frames(32, 64)]
    lens = half + half
    x, mu, cond, spks, t = _est_case(lens, 640, cfg_pair=True)
    for streaming in (True, False):
        for n in list(range(1, n_units + 1)) + [None]:
            run = (lambda a, ls: c.cfm_estimator(*a, ls, streaming=streaming)) if n is None else \
                  (lambda a, ls: c.cfm_estimator_hidden(*a, ls, n, streaming=streaming))
            full = run((x, mu, t, spks, cond), lens)
            assert torch.equal(full, run((x, mu, t, spks, cond), lens)), (precision, streaming, n, "run to run")
            o = 0
            for b, T in enumerate(lens):
                alone = run((x[o:o + T], mu[o:o + T], t[b:b + 1], spks[b:b + 1], cond[o:o + T]), [T])
                assert torch.equal(alone, full[o:o + T]), (precision, streaming, n, b, T)
                o += T


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_encoder_batch_rows_bit_identical(precision):
    """each of 32 utterances (275 .. 375 tokens) encoded alone equals its rows of the batch, bit for bit, for every read-out and the
    output, streaming with 3 look-ahead tokens and offline without; two batch runs agree bit for bit"""
    c, W = _model(precision)
    cfg = W["cfg"]
    ne = cfg.enc_blocks
    lens0 = _bench_frames(32, 32)
    for streaming, ctxl in ((True, 3), (False, 0)):
        lens = [L + ctxl for L in lens0]
        tok = _tokens(lens, 320)
        for n in list(range(ne + 2 + cfg.enc_up_blocks)) + [None]:
            run = (lambda tk, ls: c.flow_encoder(tk, ls, streaming=streaming, context_len=ctxl)) if n is None else \
                  (lambda tk, ls: c.flow_encoder_hidden(tk, ls, n, ne, streaming=streaming, context_len=ctxl))
            full = run(tok, lens)
            assert torch.equal(full, run(tok, lens)), (precision, streaming, n, "run to run")
            rate = 1 if n is not None and n <= ne else 2
            o = ot = 0
            for b, L in enumerate(lens):
                rows = rate * (L - ctxl)
                alone = run(tok[ot:ot + L], [L])
                assert torch.equal(alone, full[o:o + rows]), (precision, streaming, n, b, L)
                o += rows
                ot += L


def test_flow_hidden_refuses_n_out_of_range():
    """n_layers outside [0, enc_blocks + 1 + enc_up_blocks] and n_units outside [1, n_stages * (1 + n_blocks)] are refused before any
    device work; the context then computes what it computed before"""
    from cosyvoice_b200.cvk import CvkError
    c, W = _model("bf16")
    cfg = W["cfg"]
    lens = [70, 33]
    x, mu, cond, spks, t = _est_case(lens, 5)
    n_units = (cfg.num_mid_blocks + 2) * (1 + cfg.n_blocks)
    before = c.cfm_estimator_hidden(x, mu, t, spks, cond, lens, n_units, streaming=True)
    for n in (-1, 0, n_units + 1):
        with pytest.raises(CvkError):
            c.cfm_estimator_hidden(x, mu, t, spks, cond, lens, n, streaming=True)
    assert torch.equal(before, c.cfm_estimator_hidden(x, mu, t, spks, cond, lens, n_units, streaming=True))
    tl = [40, 23]
    tok = _tokens(tl, 6)
    n_enc = cfg.enc_blocks + 1 + cfg.enc_up_blocks
    before = c.flow_encoder_hidden(tok, tl, n_enc, cfg.enc_blocks, streaming=True, context_len=3)
    for n in (-1, n_enc + 1):
        with pytest.raises(CvkError):
            c.flow_encoder_hidden(tok, tl, n, cfg.enc_blocks, streaming=True, context_len=3)
    assert torch.equal(before, c.flow_encoder_hidden(tok, tl, n_enc, cfg.enc_blocks, streaming=True, context_len=3))


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_flow_full_config(precision):
    """the (6, 4, 12, 4) encoder on 275 + 375 tokens and the 70-unit estimator on 550 + 750 frames, offline and streaming, against
    the exact and the bf16-emulating fp64 references.  Errors relative to the mean row rms of the reference."""
    c, W = _model(precision, FULL)
    cfg = W["cfg"]
    n_enc = cfg.enc_blocks + 1 + cfg.enc_up_blocks
    n_units = (cfg.num_mid_blocks + 2) * (1 + cfg.n_blocks)
    tol = kr.FLOW_STACK_TOL[precision]
    names = ("encoder hidden", "encoder output", "estimator hidden", "estimator output")
    bad = []
    for streaming in (False, True):
        ctxl = 3 if streaming else 0
        tl = [275 + ctxl, 375 + ctxl]
        tok = _tokens(tl, 11)
        lens = [550, 750]
        x, mu, cond, spks, t = _est_case(lens, 12)
        got = (c.flow_encoder_hidden(tok, tl, n_enc, cfg.enc_blocks, streaming=streaming, context_len=ctxl),
               c.flow_encoder(tok, tl, streaming=streaming, context_len=ctxl),
               c.cfm_estimator_hidden(x, mu, t, spks, cond, lens, n_units, streaming=streaming),
               c.cfm_estimator(x, mu, t, spks, cond, lens, streaming=streaming))
        got = [g.cpu().double() for g in got]
        line = []
        for ref_name, rounding in (("exact", False), ("bf16-emulating", True)):
            refs = kr.flow_encoder(W, tok, tl, streaming, ctxl, rounding) + \
                kr.flow_estimator(W, x, mu, cond, spks, t, lens, streaming, rounding)
            es = [((g - r).abs().max() / _row_rms(r).mean()).item() for g, r in zip(got, refs)]
            line.append(f"{ref_name}: " + ", ".join(f"{nm} {e:.3g} (bound {b})" for nm, e, b in zip(names, es, tol[ref_name])))
            bad += [(streaming, ref_name, nm, e) for nm, e, b in zip(names, es, tol[ref_name]) if not e <= b]
        print(f"[full config {precision} streaming={streaming}] largest error / rms: " + "; ".join(line))
    assert not bad, bad
