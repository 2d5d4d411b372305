"""Plain fp64 CPU references of the kernels checked by test_kernel_edges_gpu.py and test_kernel_epilogues_gpu.py.
test_kernel_refs_cpu.py checks them against torch's scaled_dot_product_attention, F.conv1d and activations, the oracle LM and the
oracle conformer layer, so that the yardsticks are trusted before they judge a kernel."""
import math

import torch

from oracle import lm as olm

HD = 64
NH, NKV = olm.N_HEAD, olm.N_KV              # 14 query heads, 2 kv heads
QKV_N = (NH + 2 * NKV) * HD                 # 1152


def bf16(x):
    """round to bf16 (nearest even), returned in x's dtype"""
    return x.to(torch.bfloat16).to(x.dtype)


def f16(x):
    """round to IEEE half (nearest even) with the kernels' saturation at +-65504 (common.cuh from_f32<__half>), in x's dtype"""
    return x.clamp(-65504.0, 65504.0).to(torch.float16).to(x.dtype)


def round_to(x, dtype):
    """x rounded to a storage dtype of the conv-GEMM ("fp32", "bf16" or "fp16"), in x's dtype"""
    return {"fp32": lambda t: t.float().to(t.dtype), "bf16": bf16, "fp16": f16}[dtype](x)


def bf16_ulp(x):
    """one bf16 ulp at |x| (8 significant bits): 2^(floor(log2|x|) - 7); the smallest normal's ulp at 0"""
    a = x.abs().double().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7).to(x.dtype)


def near_bf16_tie(x, eps):
    """True where x lies within eps of a bf16 rounding boundary: a perturbation of eps may round it the other way"""
    half = bf16_ulp(x) / 2
    return (half - (x - bf16(x)).abs()) <= eps


def visible(Lq, Lk, q_off, chunk):
    """[Lq, Lk] bool: key j visible from query i (absolute position q_off + i): j < Lk and, when chunk > 0, j < ((q_off+i)//chunk+1)*chunk"""
    i = torch.arange(Lq)[:, None] + q_off
    j = torch.arange(Lk)[None, :]
    m = torch.ones(Lq, Lk, dtype=torch.bool)
    if chunk > 0:
        m = j < (i // chunk + 1) * chunk
    return m


def attention(q, k, v, q_lens, k_lens, q_offset, H, kv_heads, chunk, scale):
    """cvk_op_attention_ex in fp64: q [sum q_lens, H*64], k / v [sum k_lens, kv_heads*64] ragged; query head h reads kv head
    h // (H // kv_heads).  Returns [sum q_lens, H*64] float64."""
    q, k, v = (t.double() for t in (q, k, v))
    G = H // kv_heads
    outs, oq, ok = [], 0, 0
    for Lq, Lk, off in zip(q_lens, k_lens, q_offset):
        qq = q[oq:oq + Lq].view(Lq, H, HD).transpose(0, 1)
        kk = k[ok:ok + Lk].view(Lk, kv_heads, HD).transpose(0, 1).repeat_interleave(G, 0)
        vv = v[ok:ok + Lk].view(Lk, kv_heads, HD).transpose(0, 1).repeat_interleave(G, 0)
        s = (qq @ kk.transpose(1, 2)) * scale
        s = s.masked_fill(~visible(Lq, Lk, off, chunk)[None], float("-inf"))
        outs.append((torch.softmax(s, -1) @ vv).transpose(0, 1).reshape(Lq, H * HD))
        oq += Lq
        ok += Lk
    return torch.cat(outs, 0)


def decode_qkv(partial, bias, ctx_len, preround=False, round_bf16=True):
    """The new token's q [rows,14,64], k [rows,2,64] (RoPE at position ctx_len[b], oracle.lm.rope) and v [rows,2,64] from the split-K
    partial sums [splits,rows,1152] + bias, in fp64.  round_bf16: q, k, v rounded to bf16 as the kernels store / feed them;
    preround: the qkv row is rounded to bf16 before the rotation (the per-op path stores the reduced projection as bf16 first)."""
    qkv = partial.double().sum(0) + bias.double()[None]
    if preround:
        qkv = bf16(qkv)
    rows = qkv.shape[0]
    q = qkv[:, :NH * HD].view(rows, NH, HD)
    k = qkv[:, NH * HD:(NH + NKV) * HD].view(rows, NKV, HD)
    v = qkv[:, (NH + NKV) * HD:].view(rows, NKV, HD)
    qr, kr = torch.empty_like(q), torch.empty_like(k)
    for b in range(rows):
        pos = torch.tensor([int(ctx_len[b])])
        qr[b] = olm.rope(q[b][None, :, None, :], pos)[0, :, 0]
        kr[b] = olm.rope(k[b][None, :, None, :], pos)[0, :, 0]
    if round_bf16:
        qr, kr, v = bf16(qr), bf16(kr), bf16(v)
    return qr, kr, v


def decode_attention(q, k_new, v_new, k_cache, v_cache, ctx_len):
    """One GQA decode step in fp64: q [rows,14,64] (already rotated), k_new / v_new [rows,2,64], caches [rows,2,max_ctx,64] holding
    ctx_len[b] history rows.  Keys 0..ctx_len[b] (the new one last), scale 1/8.  Returns out [rows, 896] float64."""
    rows = q.shape[0]
    out = torch.empty(rows, NH * HD, dtype=torch.float64)
    G = NH // NKV
    for b in range(rows):
        L = int(ctx_len[b])
        keys = torch.cat([k_cache[b, :, :L].double(), k_new[b, :, None].double()], 1)      # [2, L+1, 64]
        vals = torch.cat([v_cache[b, :, :L].double(), v_new[b, :, None].double()], 1)
        kk, vv = keys.repeat_interleave(G, 0), vals.repeat_interleave(G, 0)               # [14, L+1, 64]
        s = (q[b].double()[:, None, :] @ kk.transpose(1, 2))[:, 0] * 0.125                 # [14, L+1]
        out[b] = (torch.softmax(s, -1)[:, None, :] @ vv)[:, 0].reshape(-1)
    return out


# ------------------------------------------------------------------------------------------------ LM decode layer
LM_D, LM_DFF = olm.D, olm.D_FF              # 896, 4864
LAYER_ROUNDING = {
    # where a decode path stores a bf16 value that the next stage reads: the fused chain keeps the qkv and gate/up projections in
    # fp32 (split-K partial sums reduced by the attention unit, SwiGLU in the GEMM epilogue); the per-op chain stores both as bf16
    # first
    None: (),
    "fused": ("xn", "qkv_rot", "att", "ffa"),
    "per-op": ("xn", "qkv", "qkv_rot", "att", "gu", "ffa"),
}


def rms_norm(x, g):
    """RMSNorm (eps 1e-6) of the rows of x times g, in fp64"""
    x = x.double()
    return g.double() * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + olm.RMS_EPS))


def layer_weights(sd, i):
    """layer i of an oracle-style LM state dict, in the kernels' grouping: ln1, wqkv [1152, 896], bqkv, wo, ln2, wg, wu, wd"""
    p = f"llm.model.model.layers.{i}"
    return dict(ln1=sd[p + ".input_layernorm.weight"], ln2=sd[p + ".post_attention_layernorm.weight"],
                wqkv=torch.cat([sd[f"{p}.self_attn.{n}_proj.weight"] for n in "qkv"]),
                bqkv=torch.cat([sd[f"{p}.self_attn.{n}_proj.bias"] for n in "qkv"]),
                wo=sd[p + ".self_attn.o_proj.weight"], wg=sd[p + ".mlp.gate_proj.weight"], wu=sd[p + ".mlp.up_proj.weight"],
                wd=sd[p + ".mlp.down_proj.weight"])


def decode_layer(w, x, k_cache, v_cache, ctx_len, rounding=None):
    """One Qwen2 decoder layer (modeling_qwen2.py: RMSNorm -> q/k/v + bias -> RoPE -> GQA attention over the cache and the new row ->
    o_proj + residual -> RMSNorm -> SwiGLU -> down_proj + residual) for one decode step of `rows` independent rows, in fp64.
    w: layer_weights(...) (the kernels hold the weights as bf16: give bf16-representable ones); x [rows, 896] the residual stream;
    caches [rows, 2, max_ctx, 64] holding ctx_len[b] history rows (not modified: the new rows are returned); the new token sits at
    position ctx_len[b].  rounding: None (exact), "fused" or "per-op": the values that path stores as bf16 before the next stage reads
    them are rounded here too (LAYER_ROUNDING).  Returns every stage: xn, qkv, q, k, v (rotated; k, v are the cache rows), att, x_mid,
    xn_mid, g, u, ffa, x_out."""
    r = LAYER_ROUNDING[rounding]
    rd = lambda t, what: bf16(t) if what in r else t
    W = {k: v.double() for k, v in w.items()}
    xn = rd(rms_norm(x, W["ln1"]), "xn")
    qkv = rd(xn @ W["wqkv"].t() + W["bqkv"][None], "qkv")
    q, k, v = decode_qkv(qkv[None], torch.zeros(QKV_N, dtype=torch.float64), ctx_len, round_bf16="qkv_rot" in r)
    att = rd(decode_attention(q, k, v, k_cache, v_cache, ctx_len), "att")
    x_mid = x.double() + att @ W["wo"].t()
    xn_mid = rd(rms_norm(x_mid, W["ln2"]), "xn")
    g, u = rd(xn_mid @ W["wg"].t(), "gu"), rd(xn_mid @ W["wu"].t(), "gu")
    ffa = rd(g / (1.0 + torch.exp(-g)) * u, "ffa")
    x_out = x_mid + ffa @ W["wd"].t()
    return dict(xn=xn, qkv=qkv, q=q, k=k, v=v, att=att, x_mid=x_mid, xn_mid=xn_mid, g=g, u=u, ffa=ffa, x_out=x_out)


# ------------------------------------------------------------------------------------------------ conv-GEMM and its epilogue
def act(name, x, param=0.0, alpha=None):
    """the epilogue activations in x's dtype, written from their definitions: GELU with erf, GELU's tanh form
    (F.gelu(approximate='tanh')), SiLU, Mish, ELU (alpha 1), leaky ReLU (slope param), Snake x + sin^2(a x) / (a + 1e-9) with a per
    column (alpha [N], 1 when None; oracle/hift.py snake), tanh, |x|"""
    if name == "none":
        return x
    if name == "gelu":
        return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))
    if name == "gelu_tanh":
        return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))
    if name == "silu":
        return x / (1.0 + torch.exp(-x))
    if name == "mish":
        return x * torch.tanh(torch.log1p(torch.exp(x.clamp(max=40.0))))     # tanh(softplus(x)) == 1 in fp64 from x = 20 on
    if name == "elu":
        return torch.where(x > 0, x, torch.expm1(x))
    if name == "lrelu":
        return torch.where(x > 0, x, x * param)
    if name == "snake":
        a = torch.ones_like(x[0]) if alpha is None else alpha.to(x.dtype)
        return x + torch.sin(a * x) ** 2 / (a + 1e-9)
    if name == "tanh":
        return torch.tanh(x)
    if name == "abs":
        return x.abs()
    raise ValueError(name)


def conv_rows(x, w, dil=1, shift0=0):
    """the conv-GEMM product on a packed matrix in fp64: acc[r, n] = sum_j sum_k x[r + shift0 + j*dil, k] w[n, k, j], rows outside
    [0, rows) read as zero.  x [rows, K], w a torch Conv1d weight [N, K, taps] (on x's device)."""
    x, w = x.double(), w.double()
    rows = x.shape[0]
    N, K, taps = w.shape
    acc = torch.zeros(rows, N, dtype=torch.float64, device=x.device)
    for j in range(taps):
        s = shift0 + j * dil
        lo, hi = max(0, -s), min(rows, rows - s)          # output rows whose input row r + s lies inside the matrix
        if lo < hi:
            acc[lo:hi] += x[lo + s:hi + s] @ w[:, :, j].t()
    return acc


def conv_epilogue(acc, valid, bias=None, act1="none", act1_param=0.0, alpha1=None, resid=None, out_init=None, accumulate=False,
                  act2=None, act2_param=0.0, alpha2=None):
    """the fused epilogue of the conv-GEMM (struct Epilogue, cvk_internal.h) in fp64, in its order:
      v = act1(acc + bias) (+ resid);  v = 0 on invalid rows;  out = out_init + v if accumulate else v;
      out2 = act2(out) on valid rows (applied to the unrounded value), 0 on invalid rows.
    acc [rows, N], valid [rows] bool, bias / alpha [N], resid / out_init [rows, N].  Returns (out, out2 or None)."""
    v = acc.double() + (bias.double()[None] if bias is not None else 0.0)
    v = act(act1, v, act1_param, alpha1)
    if resid is not None:
        v = v + resid.double()
    v = torch.where(valid[:, None], v, 0.0)
    if accumulate:
        v = out_init.double() + v
    out2 = None
    if act2 is not None:
        out2 = torch.where(valid[:, None], act(act2, v, act2_param, alpha2), 0.0)
    return v, out2


# ------------------------------------------------------------------------------------------------ relative-position attention
def rel_shift(x):
    """the reference conformer's rel_shift (transformer/attention.py:225-247, oracle/flow.py _rel_shift) on [H, t, 2t-1] -> [H, t, t]"""
    h, t, n = x.shape
    xp = torch.cat([x.new_zeros(h, t, 1), x], -1).view(h, n + 1, t)
    return xp[:, 1:].reshape(h, t, n)[:, :, : n // 2 + 1]


def relpos_attention(q, k, v, pos, center, bias_u, bias_v, lens, H, chunk, scale):
    """cvk_op_relpos_attention in fp64, computed the way the reference conformer layer does (oracle/flow.py _enc_layer):
    ac = (q + u) k^T, bd = rel_shift((q + v) p^T), softmax((ac + bd) * scale) over the visible keys, times v.  A sequence of length L
    uses the 2L-1 central rows of the table, center - (L-1) .. center + (L-1) (relative positions L-1 .. -(L-1)), which is the table
    the reference builds for it.  q, k, v [sum lens, H*64], pos [2*center+1, H*64], bias_u / bias_v [H*64]."""
    q, k, v, pos = (t.double() for t in (q, k, v, pos))
    u, vb = bias_u.double().view(H, 1, HD), bias_v.double().view(H, 1, HD)
    outs, o = [], 0
    for L in lens:
        qq, kk, vv = (t[o:o + L].view(L, H, HD).transpose(0, 1) for t in (q, k, v))
        pp = pos[center - (L - 1):center + L].view(2 * L - 1, H, HD).transpose(0, 1)
        ac = (qq + u) @ kk.transpose(1, 2)
        bd = rel_shift((qq + vb) @ pp.transpose(1, 2))
        s = ((ac + bd) * scale).masked_fill(~visible(L, L, 0, chunk)[None], float("-inf"))
        outs.append((torch.softmax(s, -1) @ vv).transpose(0, 1).reshape(L, H * HD))
        o += L
    return torch.cat(outs, 0)


# ------------------------------------------------------------------------------------------------ CosyVoice3 DiT estimator
# The DiT of oracle/dit.py (dit.py:145-176 of the reference) restated on the packed time-major rows the kernels use, in fp64, one piece
# at a time: the time embedding and every AdaLN modulation vector (dit_modulation), the input embedding (dit_input_embedding), one
# block (dit_block) and norm_out + proj_out (dit_output).  rounding=True emulates the bf16 path: the values it stores as bf16 and
# reads again are rounded at the same points (DIT_ROUNDING), and the tensor-core weights are taken as bf16.  `mutate` applies one of
# DIT_MUTATIONS, the defects the sensitivity test of test_kernel_refs_cpu.py injects.
from oracle import dit as odit  # noqa: E402

DIT_D, DIT_FF, DIT_CK = odit.DIM, odit.FF, odit.CONV_K
DIT_ROUNDING = ("x_conv", "mish1", "xn", "qkv", "rot", "att", "ff")
DIT_MUTATIONS = ("rope_half", "rope_all_heads", "kpos_shift", "adaln_swap", "mod_neighbour", "chunk48", "chunk_edge", "silu_pos",
                 "time_div", "gelu_erf", "ln_eps")


def dit_weights(sd, depth, p="decoder.estimator."):
    """the estimator's weights in fp64, grouped the way the kernels hold them (qkv concatenated, every modulation linear in one matrix)"""
    g = lambda k: sd[p + k].double()
    blocks = []
    for i in range(depth):
        b = f"transformer_blocks.{i}."
        blocks.append(dict(qkv_w=torch.cat([g(b + f"attn.to_{n}.weight") for n in "qkv"]),
                           qkv_b=torch.cat([g(b + f"attn.to_{n}.bias") for n in "qkv"]),
                           out_w=g(b + "attn.to_out.0.weight"), out_b=g(b + "attn.to_out.0.bias"),
                           ff1_w=g(b + "ff.ff.0.0.weight"), ff1_b=g(b + "ff.ff.0.0.bias"),
                           ff2_w=g(b + "ff.ff.2.weight"), ff2_b=g(b + "ff.ff.2.bias")))
    mods = [f"transformer_blocks.{i}.attn_norm.linear." for i in range(depth)] + ["norm_out.linear."]
    return dict(depth=depth, blocks=blocks,
                t1_w=g("time_embed.time_mlp.0.weight"), t1_b=g("time_embed.time_mlp.0.bias"),
                t2_w=g("time_embed.time_mlp.2.weight"), t2_b=g("time_embed.time_mlp.2.bias"),
                mod_w=torch.cat([g(m + "weight") for m in mods]), mod_b=torch.cat([g(m + "bias") for m in mods]),
                in_w=g("input_embed.proj.weight"), in_b=g("input_embed.proj.bias"),
                c1_w=g("input_embed.conv_pos_embed.conv1.0.weight"), c1_b=g("input_embed.conv_pos_embed.conv1.0.bias"),
                c2_w=g("input_embed.conv_pos_embed.conv2.0.weight"), c2_b=g("input_embed.conv_pos_embed.conv2.0.bias"),
                proj_w=g("proj_out.weight"), proj_b=g("proj_out.bias"))


def _rd(rounding):
    return bf16 if rounding else (lambda t: t)


def _seq_ids(lens):
    return torch.repeat_interleave(torch.arange(len(lens)), torch.tensor(lens))


def _silu(x):
    return x / (1.0 + torch.exp(-x))


def dit_modulation(W, t, mutate=None):
    """TimestepEmbedding (modules.py:71-84, 606-616) and every AdaLN linear on SiLU of it, in fp64: t [B] -> dict(a (the sinusoid
    angles), sc, te1, te, ste, mod [B, depth*6144 + 2048]).  The fp32 CUDA-core GEMMs of the kernels have no bf16 rounding point."""
    half = 128
    div = half if mutate == "time_div" else half - 1
    e = torch.exp(torch.arange(half, dtype=torch.float64) * -(math.log(10000.0) / div))
    a = 1000.0 * t.double()[:, None] * e[None]
    sc = torch.cat([a.sin(), a.cos()], -1)
    te1 = _silu(sc @ W["t1_w"].t() + W["t1_b"])
    te = te1 @ W["t2_w"].t() + W["t2_b"]
    ste = _silu(te)
    return dict(a=a, sc=sc, te1=te1, te=te, ste=ste, mod=ste @ W["mod_w"].t() + W["mod_b"])


def _mish(x):
    return act("mish", x)


def _causal_grouped_conv(x, w, b, lens):
    """CausalConvPositionEmbedding's Conv1d (k31, 16 groups, 30 zero rows in front of every sequence) on packed rows [sum T, 1024]"""
    outs, o = [], 0
    for L in lens:
        y = torch.nn.functional.conv1d(torch.nn.functional.pad(x[o:o + L].t()[None], (DIT_CK - 1, 0)), w, b, groups=odit.CONV_GROUPS)
        outs.append(y[0].t())
        o += L
    return torch.cat(outs, 0)


def dit_input_embedding(W, x, mu, cond, spks, lens, rounding=False, mutate=None):
    """InputEmbedding (modules.py:87-112, 115-145): proj([x | cond | mu | spks]) -> two causal grouped k31 convolutions with Mish ->
    + proj.  x, mu, cond [sum T, 80], spks [B, 80] (one row per sequence).  Returns dict(h (the projection), xa (conv1's input),
    c1 (conv1 after Mish), acc2 (conv2 before Mish), x0 = the residual stream entering block 0)."""
    rd = _rd(rounding)
    wt = rd if rounding else (lambda t: t)
    inp = torch.cat([x.double(), cond.double(), mu.double(), spks.double()[_seq_ids(lens)]], -1)
    h = rd(inp) @ wt(W["in_w"]).t() + W["in_b"]                         # the bf16 path packs its input as bf16
    act_pos = _silu if mutate == "silu_pos" else _mish
    xa = rd(h)
    acc1 = _causal_grouped_conv(xa, wt(W["c1_w"]), W["c1_b"], lens)
    c1 = rd(act_pos(acc1))
    acc2 = _causal_grouped_conv(c1, wt(W["c2_w"]), W["c2_b"], lens)
    return dict(inp=rd(inp), h=h, xa=xa, acc1=acc1, c1=c1, acc2=acc2, x0=act_pos(acc2) + h)


def _layer_norm(x, eps=1e-6):
    mu = x.mean(-1, keepdim=True)
    v = x - mu
    return v * torch.rsqrt(v.pow(2).mean(-1, keepdim=True) + eps)


def rotary_angles(T, q_off=0):
    """the reference's fp32 rotary angles (oracle.dit.rotary_freqs: x_transformers' table, position * 10000^(-2i/64) in fp32) of
    positions q_off .. q_off + T - 1, in fp64: [T, 64], each angle in two adjacent channels"""
    return odit.rotary_freqs(T + q_off)[0, q_off:].double()


def _rotate(t, ang, half_split=False):
    """x_transformers' rotation of adjacent pairs (2i, 2i+1) -> (a cos - b sin, b cos + a sin) on the last dim (64); half_split: the
    rotate-half pairing (i, i + 32) instead"""
    if half_split:
        a, b = t[..., :32], t[..., 32:]
        c, s = ang[..., ::2].cos(), ang[..., ::2].sin()
        return torch.cat([a * c - b * s, b * c + a * s], -1)
    a2 = t.reshape(*t.shape[:-1], 32, 2)
    rot = torch.stack((-a2[..., 1], a2[..., 0]), -1).flatten(-2)
    return t * ang.cos() + rot * ang.sin()


def _dit_visible(T, chunk, edge=0):
    """[T, T] key j visible from query i: all keys, or the static block-causal mask of `chunk` frames (add_optional_chunk_mask),
    with the chunk's right edge moved by `edge`"""
    if chunk <= 0:
        return torch.ones(T, T, dtype=torch.bool)
    i = torch.arange(T)[:, None]
    return torch.arange(T)[None, :] < (i // chunk + 1) * chunk + edge


def dit_block(W, i, x, mod, lens, chunk, rounding=False, mutate=None):
    """DiTBlock i (modules.py:500-533) on packed rows x [sum T, 1024] (fp64), mod = dit_modulation(...)["mod"] [B, ...], chunk 0
    (offline) or 50 (streaming).  Returns every stage: n1 (the normalised rows), xn, qkv, qkv_rot (head 0 of q and k rotated), p
    (the attention weights per sequence), att, o, x_mid, n2, xn2, hpre, h, f, x_out (all fp64, rounded where DIT_ROUNDING says)."""
    rd = _rd(rounding)
    wt = bf16 if rounding else (lambda t: t)
    w = W["blocks"][i]
    x = x.double()
    B = len(lens)
    seq = _seq_ids(lens)
    m = mod[:, i * 6 * DIT_D:(i + 1) * 6 * DIT_D]
    if mutate == "mod_neighbour":
        m = m[(torch.arange(B) + 1) % B]
    sh1, sc1, g1, sh2, sc2, g2 = (t[seq] for t in m.split(DIT_D, -1))
    if mutate == "adaln_swap":
        sh1, sc1, sh2, sc2 = sc1, sh1, sc2, sh2
    eps = 1e-5 if mutate == "ln_eps" else 1e-6
    n1 = _layer_norm(x, eps)
    xn64 = n1 * (1 + sc1) + sh1
    xn = rd(xn64)
    qkv64 = xn @ wt(w["qkv_w"]).t() + w["qkv_b"]
    qkv = rd(qkv64)
    heads = 16 if mutate == "rope_all_heads" else 1
    rot64 = qkv.clone()
    outs, ps, o0 = [], [], 0
    for L in lens:
        ang = rotary_angles(L)
        for which in (0, 1):
            kang = rotary_angles(L, 1) if (which == 1 and mutate == "kpos_shift") else ang
            cols = slice(which * DIT_D, which * DIT_D + 64 * heads)
            blk = qkv[o0:o0 + L, cols].reshape(L, heads, 64)
            rot64[o0:o0 + L, cols] = _rotate(blk, kang[:, None], mutate == "rope_half").reshape(L, 64 * heads)
        o0 += L
    qkv_rot = rd(rot64)
    o0 = 0
    ch = 48 if mutate == "chunk48" else chunk
    for L in lens:
        q, k, v = (qkv_rot[o0:o0 + L, n * DIT_D:(n + 1) * DIT_D].reshape(L, 16, 64).transpose(0, 1) for n in range(3))
        s = (q @ k.transpose(1, 2)) * 0.125
        s = s.masked_fill(~_dit_visible(L, ch, 1 if mutate == "chunk_edge" else 0)[None], float("-inf"))
        p = torch.softmax(s, -1)
        ps.append(p)
        outs.append((p @ v).transpose(0, 1).reshape(L, DIT_D))
        o0 += L
    att64 = torch.cat(outs, 0)
    att = rd(att64)
    o = att @ wt(w["out_w"]).t() + w["out_b"]
    x_mid = x + g1 * o
    n2 = _layer_norm(x_mid, eps)
    xn2_64 = n2 * (1 + sc2) + sh2
    xn2 = rd(xn2_64)
    hpre = xn2 @ wt(w["ff1_w"]).t() + w["ff1_b"]
    h64 = act("gelu" if mutate == "gelu_erf" else "gelu_tanh", hpre)
    h = rd(h64)
    f = h @ wt(w["ff2_w"]).t() + w["ff2_b"]
    return dict(x=x, n1=n1, xn64=xn64, xn=xn, qkv64=qkv64, qkv=qkv, rot64=rot64, qkv_rot=qkv_rot, p=ps, att64=att64, att=att, o=o,
                x_mid=x_mid, n2=n2, xn2_64=xn2_64, xn2=xn2, hpre=hpre, h64=h64, h=h, f=f, x_out=x_mid + g2 * f,
                sc1=sc1, sh1=sh1, g1=g1, sc2=sc2, sh2=sh2, g2=g2)


def dit_output(W, x, mod, lens, rounding=False):
    """AdaLayerNormZero_Final + proj_out (modules.py:251-264, dit.py:174-175): x [sum T, 1024] -> [sum T, 80]"""
    depth = W["depth"]
    sc, sh = (t[_seq_ids(lens)] for t in mod[:, depth * 6 * DIT_D:].split(DIT_D, -1))
    xn = _rd(rounding)(_layer_norm(x.double()) * (1 + sc) + sh)
    return xn @ (bf16(W["proj_w"]) if rounding else W["proj_w"]).t() + W["proj_b"]


def dit_estimator(W, x, mu, cond, spks, t, lens, streaming, rounding=False, n_blocks=None):
    """the composed estimator on packed rows: returns (hidden after n_blocks blocks (all by default), output [sum T, 80])"""
    mod = dit_modulation(W, t)["mod"]
    h = dit_input_embedding(W, x, mu, cond, spks, lens, rounding)["x0"]
    for i in range(W["depth"] if n_blocks is None else n_blocks):
        h = dit_block(W, i, h, mod, lens, 50 if streaming else 0, rounding)["x_out"]
    return h, dit_output(W, h, mod, lens, rounding)


def dit_test_state_dict(depth, seed):
    """CosyVoice3 flow weights for the DiT checks (named as oracle.dit.flow_param_shapes names them): fan-in-scaled matrices,
    bf16-representable where the bf16 path streams them as bf16 (so both references see the kernels' weights), and AdaLN
    modulation vectors of O(1) - gates ~ 1, unlike oracle.dit.SYNTH_GAINS, which keep ten Euler steps tame with gates ~ 0.1 and so
    shrink each block's contribution under the residual."""
    from oracle import weights as oweights
    sd = oweights.synth_state_dict(odit.flow_param_shapes(depth), seed, {"attn_norm.linear.weight": 4.0, "norm_out.linear.weight": 4.0})
    est = "decoder.estimator."
    g = torch.Generator().manual_seed(seed)
    for k in ("input_embed.proj.weight", "time_embed.time_mlp.0.weight", "time_embed.time_mlp.2.weight"):
        w = sd[est + k]                                     # matrices, not embedding tables: fan-in scaled
        sd[est + k] = torch.randn(w.shape, generator=g) * w.shape[1] ** -0.5
    for k, v in sd.items():
        if v.dim() >= 2 and k.startswith(est) and "time_embed" not in k and ".linear." not in k:
            sd[k] = bf16(v)
    return sd


# bounds of test_dit_blocks_gpu.py: largest |kernel - reference| of a stage over the rms of that row's contribution (embedding: x0;
# block: x_out - x).  Largest ratios measured on an H100 80GB HBM3 (700 W) over every layout, both masks, in one run: fp32 embedding
# 7.6e-6, block 1.1e-4 (the fp32 sinusoid of t, angles up to 950 rad, carries ~6e-5 into the modulation vectors); bf16 (against the
# bf16-emulating reference) embedding 2.4e-3, block 2.4e-2.  Each bound is about twice that.
DIT_TOL = {"fp32": dict(embed=2e-5, block=2.5e-4), "bf16": dict(embed=5e-3, block=0.05)}
# 22-block stack: largest error over the mean row rms of the reference, (hidden, estimator output), per reference.  Measured, same run:
# fp32 vs exact 1.1e-4 / 8.3e-5, fp32 vs bf16-emulating 1.3e-2 / 1.1e-2, bf16 vs exact 1.2e-2 / 1.2e-2, bf16 vs bf16-emulating
# 1.3e-2 / 1.2e-2.  Bounds about twice that.
DIT_STACK_TOL = {"fp32": {"exact": (2.5e-4, 2e-4), "bf16-emulating": (0.03, 0.025)},
                 "bf16": {"exact": (0.025, 0.025), "bf16-emulating": (0.03, 0.025)}}


# ------------------------------------------------------------------------------------------------ CosyVoice2 flow
# The conformer encoder and the causal U-Net estimator of oracle/flow.py (flow/flow.py:235-281 of the reference) restated on the
# packed time-major rows the kernels use, in fp64, one unit at a time: the encoder's input embedding with the PreLookahead layer
# (enc_embed), one conformer layer (enc_layer), the x2 up-sampling with up_embed (enc_upsample) and after_norm; the estimator's time
# embedding with every per-stage projection (est_time), one stage resnet (est_resnet), one transformer block (est_tblock) and the
# tail (est_tail).  rounding=True emulates the bf16 path: the values it stores as bf16 (or rounds to bf16 on chip) and reads again
# are rounded at the same points (FLOW_ROUNDING), and the tensor-core weights are taken as bf16.  `mutate` applies one of
# FLOW_MUTATIONS, the defects the sensitivity test of test_kernel_refs_cpu.py injects.
from oracle import flow as oflow  # noqa: E402

FLOW_D, FLOW_C = oflow.D_ENC, oflow.C_EST
FLOW_ROUNDING = {
    # encoder: token rows written as the embed Linear's operand, embed output as the PreLookahead operand, its leaky-ReLU output,
    # LN1 / LN2 outputs, the qkv projection, the position table and its projection, q + pos_bias_u / v, the attention output, the
    # SiLU hidden, the residual stream as the up-sampler's operand and the up-sampler's output
    "enc": ("emb", "h0a", "c1", "xn", "qkv", "pe", "pos", "quv", "att", "ff", "xa", "up"),
    # estimator: the packed [x | mu | spks | cond] input, LN-Mish + temb of each resnet's first block, LN1 / LN3 outputs, qkv, the
    # attention output, the GELU hidden (on chip in the fused feed-forward), the bf16 copy of every stage output that the next stage
    # and the skip read, the down_blocks.0.2 output, and the tail's up_blocks.0.2 output and LN-Mish
    "est": ("in", "h1", "xn", "qkv", "att", "ff", "act", "xa", "tail"),
}
FLOW_MUTATIONS = {
    "est": ("chunk48", "chunk_edge", "temb_neighbour", "temb_before_mish", "skip_swap", "centred_pad", "silu_for_mish", "gelu_tanh",
            "time_div", "ln_eps"),
    "enc": ("pos_bias_swap", "rel_shift", "chunk24", "lookahead2", "up_pad3", "no_sqrt", "ln_eps"),
}


def flow_weights(sd, cfg):
    """the flow's weights in fp64 (oracle.flow.param_shapes names, without the "flow." prefix), with the config"""
    W = {k: v.double() for k, v in sd.items()}
    W["cfg"] = cfg
    return W


def _rdw(rounding):
    return bf16 if rounding else (lambda t: t)


def _ln(x, g, b, eps):
    return _layer_norm(x, eps) * g + b


def _seq_conv(x, w, b, lens, shift0):
    """a conv-GEMM on packed rows, sequence by sequence (rows outside a sequence read as zero): x [sum T, K], w [N, K, taps]"""
    outs, o = [], 0
    for L in lens:
        outs.append(conv_rows(x[o:o + L], w, 1, shift0) + b)
        o += L
    return torch.cat(outs, 0)


def _enc_in(W, p, x, rounding, mutate):
    """LinearNoSubsampling + scaled positional input (subsampling.py:92-113, embedding.py:270-272): Linear -> LN(1e-5) -> x sqrt(512)"""
    y = x @ _rdw(rounding)(W[p + ".out.0.weight"]).t() + W[p + ".out.0.bias"]
    y = _ln(y, W[p + ".out.1.weight"], W[p + ".out.1.bias"], 1e-5)
    return y if mutate == "no_sqrt" else y * math.sqrt(FLOW_D)


def enc_embed(W, tokens, lens, context_len=0, rounding=False, mutate=None):
    """token embedding -> embed -> PreLookaheadLayer (upsample_encoder.py:82-103: k4 convolution over the next 3 rows, which are
    the context rows or zeros, leaky ReLU 0.01, causal k3 convolution, + input).  tokens [sum T] (context included); returns dict
    h0 (embed output, every row) and x [sum (T - context_len), 512], the stream entering the first conformer layer."""
    rd = bf16 if rounding else (lambda t: t)
    p = "encoder.pre_lookahead_layer."
    emb = rd(W["input_embedding.weight"][tokens.long().clamp(min=0)])
    h0 = _enc_in(W, "encoder.embed", emb, rounding, mutate)
    w1, w2 = _rdw(rounding)(W[p + "conv1.weight"]), _rdw(rounding)(W[p + "conv2.weight"])
    xs, o = [], 0
    for L in lens:
        Lo = L - context_len
        a = rd(h0[o:o + L])
        c1 = rd(act("lrelu", conv_rows(a, w1, 1, -1 if mutate == "lookahead2" else 0)[:Lo] + W[p + "conv1.bias"], 0.01))
        xs.append(conv_rows(c1, w2, 1, -2) + W[p + "conv2.bias"] + h0[o:o + Lo])
        o += L
    return dict(h0=h0, x=torch.cat(xs, 0))


def rel_pos_table(T, extra=0):
    """the ESPnet relative position table (embedding.py:224-254) in fp64: rows m = 0 .. 2(T + extra) - 2 hold relative position
    r = T + extra - 1 - m: pe[2i] = sin(r w_i), pe[2i+1] = cos(r w_i), w_i = 10000^(-2i/512)"""
    n = T + extra
    r = torch.arange(n - 1, -n, -1, dtype=torch.float64)[:, None]
    w = torch.exp(torch.arange(0, FLOW_D, 2, dtype=torch.float64) * -(math.log(10000.0) / FLOW_D))
    pe = torch.zeros(2 * n - 1, FLOW_D, dtype=torch.float64)
    pe[:, 0::2], pe[:, 1::2] = torch.sin(r * w), torch.cos(r * w)
    return pe


def enc_layer(W, p, x, lens, chunk, rounding=False, mutate=None):
    """ConformerEncoderLayer (encoder_layer.py:160-236: LN 1e-12, relative-position MHA with pos_bias_u / v, SiLU feed-forward) on
    packed rows x [sum T, 512]; p the layer's prefix ("encoder.encoders.i" / "encoder.up_encoders.i"); chunk 0 or the block-causal
    chunk (25 tokens, 50 after the up-sampler).  The position table is sized by the longest sequence, as the kernels size it."""
    rd = bf16 if rounding else (lambda t: t)
    wt = _rdw(rounding)
    a = p + ".self_attn."
    eps = 1e-5 if mutate == "ln_eps" else 1e-12
    x = x.double()
    xn = rd(_ln(x, W[p + ".norm_mha.weight"], W[p + ".norm_mha.bias"], eps))
    wqkv = torch.cat([W[a + f"linear_{n}.weight"] for n in "qkv"])
    bqkv = torch.cat([W[a + f"linear_{n}.bias"] for n in "qkv"])
    qkv = rd(xn @ wt(wqkv).t() + bqkv)
    T = max(lens)
    pe = rd(rel_pos_table(T, 1 if mutate == "rel_shift" else 0))      # rel_shift: every relative position read one too far
    pos = rd(pe @ wt(W[a + "linear_pos.weight"]).t())
    bu, bv = W[a + "pos_bias_u"].reshape(-1), W[a + "pos_bias_v"].reshape(-1)
    if mutate == "pos_bias_swap":
        bu, bv = bv, bu
    q, k, v = qkv.split(FLOW_D, -1)
    if rounding:       # the wgmma kernel reads q + u and q + v as bf16
        qu, qv = bf16(q + bu), bf16(q + bv)
        att64 = _relpos_att_split(qu, qv, k, v, pos, T - 1, lens, 24 if mutate == "chunk24" else chunk)
    else:
        att64 = relpos_attention(q, k, v, pos, T - 1, bu, bv, lens, 8, 24 if mutate == "chunk24" else chunk, 0.125)
    att = rd(att64)
    x_mid = x + att @ wt(W[a + "linear_out.weight"]).t() + W[a + "linear_out.bias"]
    xn2 = rd(_ln(x_mid, W[p + ".norm_ff.weight"], W[p + ".norm_ff.bias"], eps))
    ff = rd(act("silu", xn2 @ wt(W[p + ".feed_forward.w_1.weight"]).t() + W[p + ".feed_forward.w_1.bias"]))
    x_out = x_mid + ff @ wt(W[p + ".feed_forward.w_2.weight"]).t() + W[p + ".feed_forward.w_2.bias"]
    return dict(x=x, xn=xn, qkv=qkv, pos=pos, att=att, x_mid=x_mid, xn2=xn2, ff=ff, x_out=x_out)


def _relpos_att_split(qu, qv, k, v, pos, center, lens, chunk):
    """relpos_attention with q + u and q + v given separately (already rounded as the bf16 path stores them)"""
    ac_att = []
    o = 0
    for L in lens:
        qq, qqv, kk, vv = (t[o:o + L].view(L, 8, HD).transpose(0, 1) for t in (qu, qv, k, v))
        pp = pos[center - (L - 1):center + L].view(2 * L - 1, 8, HD).transpose(0, 1)
        s = (qq @ kk.transpose(1, 2) + rel_shift(qqv @ pp.transpose(1, 2))) * 0.125
        s = s.masked_fill(~visible(L, L, 0, chunk)[None], float("-inf"))
        ac_att.append((torch.softmax(s, -1) @ vv).transpose(0, 1).reshape(L, FLOW_D))
        o += L
    return torch.cat(ac_att, 0)


def enc_upsample(W, x, lens, rounding=False, mutate=None):
    """Upsample1D (upsample_encoder.py:59-63: nearest x2, left pad 4, k5 convolution) and up_embed on packed token rows
    x [sum T, 512] -> [sum 2T, 512].  The kernels fold the x2 repeat into a 3-tap polyphase convolution on the token rows whose
    weights are sums of taps (flow.cu upsample_poly_kernel); the bf16 path holds those sums as bf16, so they are rounded here."""
    rd = bf16 if rounding else (lambda t: t)
    w, b = W["encoder.up_layer.conv.weight"], W["encoder.up_layer.conv.bias"]
    xa = rd(x.double())
    outs, o = [], 0
    for L in lens:
        if mutate == "up_pad3":
            u = xa[o:o + L].repeat_interleave(2, 0)
            outs.append(conv_rows(u, w, 1, -3) + b)
        else:
            wp0 = torch.stack([w[..., 0] + w[..., 1], w[..., 2] + w[..., 3], w[..., 4]], -1)
            wp1 = torch.stack([w[..., 0], w[..., 1] + w[..., 2], w[..., 3] + w[..., 4]], -1)
            y = torch.stack([conv_rows(xa[o:o + L], _rdw(rounding)(wp), 1, -2) for wp in (wp0, wp1)], 1)   # [L, 2, 512]
            outs.append(y.reshape(2 * L, FLOW_D) + b)
        o += L
    up = rd(torch.cat(outs, 0))
    return dict(up=up, y=_enc_in(W, "encoder.up_embed", up, rounding, mutate))


def enc_after_norm(W, y):
    return _ln(y.double(), W["encoder.after_norm.weight"], W["encoder.after_norm.bias"], 1e-5)


def flow_encoder(W, tokens, lens, streaming, context_len=0, rounding=False, n_layers=None, mutate=None):
    """the composed encoder: returns (the residual stream after n_layers units (all by default; cvk_flow_encoder_hidden's units),
    the encoder output (None when n_layers stops short))"""
    cfg = W["cfg"]
    n = cfg.enc_blocks + 1 + cfg.enc_up_blocks if n_layers is None else n_layers
    lo = [L - context_len for L in lens]
    h = enc_embed(W, tokens, lens, context_len, rounding, mutate)["x"]
    for i in range(min(n, cfg.enc_blocks)):
        h = enc_layer(W, f"encoder.encoders.{i}", h, lo, 25 if streaming else 0, rounding, mutate)["x_out"]
    if n > cfg.enc_blocks:
        h = enc_upsample(W, h, lo, rounding, mutate)["y"]
        lo2 = [2 * L for L in lo]
        for i in range(n - cfg.enc_blocks - 1):
            h = enc_layer(W, f"encoder.up_encoders.{i}", h, lo2, 50 if streaming else 0, rounding, mutate)["x_out"]
    full = n_layers is None or n_layers == cfg.enc_blocks + 1 + cfg.enc_up_blocks
    return h, (enc_after_norm(W, h) if full else None)


def est_stage_names(cfg):
    e = "decoder.estimator."
    return [e + "down_blocks.0"] + [e + f"mid_blocks.{i}" for i in range(cfg.num_mid_blocks)] + [e + "up_blocks.0"]


def est_time(W, t, mutate=None):
    """SinusoidalPosEmb(320) with scale 1000 (frequencies 10000^(-i/159)), TimestepEmbedding (Linear, SiLU, Linear), then every
    stage resnet's mlp (Mish, Linear) in fp64: t [B] -> dict(a (the angles), sc, te, temb [B, n_stages, 256]).  The kernels keep
    all of it in fp32 (fp32 weights, no bf16 rounding point)."""
    e = "decoder.estimator."
    half = 160
    div = half if mutate == "time_div" else half - 1
    fr = torch.exp(torch.arange(half, dtype=torch.float64) * -(math.log(10000.0) / div))
    a = 1000.0 * t.double()[:, None] * fr[None]
    sc = torch.cat([a.sin(), a.cos()], -1)
    te = act("silu", sc @ W[e + "time_mlp.linear_1.weight"].t() + W[e + "time_mlp.linear_1.bias"])
    te = te @ W[e + "time_mlp.linear_2.weight"].t() + W[e + "time_mlp.linear_2.bias"]
    m = _mish(te)
    temb = torch.stack([m @ W[s + ".0.mlp.1.weight"].t() + W[s + ".0.mlp.1.bias"] for s in est_stage_names(W["cfg"])], 1)
    return dict(a=a, sc=sc, te=te, temb=temb)


def est_resnet(W, k, xin, temb, lens, rounding=False, mutate=None):
    """ResnetBlock1D of stage k (Matcha decoder.py:55-61 with CausalBlock1D, decoder.py:65-78): causal k3 convolution (2 zero rows in
    front of every sequence), LN 1e-5, Mish, + the stage's time projection, the same again without it, + a 1x1 residual convolution
    of the input.  xin [sum T, Cin] is the stage input as the kernels read it (the act operand); temb = est_time(...)["temb"]."""
    rd = bf16 if rounding else (lambda t: t)
    wt = _rdw(rounding)
    nst = temb.shape[1]
    p = est_stage_names(W["cfg"])[k] + ".0."
    eps = 1e-6 if mutate == "ln_eps" else 1e-5
    sh = -1 if mutate == "centred_pad" else -2
    mish = (lambda v: act("silu", v)) if mutate == "silu_for_mish" else _mish
    tv = temb[:, (k + 1) % nst if mutate == "temb_neighbour" else k][_seq_ids(lens)]
    xin = xin.double()
    c = _seq_conv(xin, wt(W[p + "block1.block.0.weight"]), W[p + "block1.block.0.bias"], lens, sh)
    n1 = _ln(c, W[p + "block1.block.2.weight"], W[p + "block1.block.2.bias"], eps)
    h1 = rd(mish(n1 + tv) if mutate == "temb_before_mish" else mish(n1) + tv)
    c2 = _seq_conv(h1, wt(W[p + "block2.block.0.weight"]), W[p + "block2.block.0.bias"], lens, sh)
    h2 = mish(_ln(c2, W[p + "block2.block.2.weight"], W[p + "block2.block.2.bias"], eps))
    x_out = xin @ wt(W[p + "res_conv.weight"][..., 0]).t() + W[p + "res_conv.bias"] + h2
    return dict(c=c, h1=h1, h2=h2, x_out=x_out)


def est_tblock(W, k, j, x, lens, chunk, rounding=False, mutate=None):
    """BasicTransformerBlock j of stage k (Matcha transformer.py:243-316 with diffusers Attention and GELU): LN 1e-5, q / k / v without
    bias, 8 heads, scale 1/8, full or block-causal (chunk 50) attention, out projection + residual, LN 1e-5, Linear, exact-erf GELU,
    Linear + residual.  x [sum T, 256] the residual stream."""
    rd = bf16 if rounding else (lambda t: t)
    wt = _rdw(rounding)
    p = est_stage_names(W["cfg"])[k] + f".1.{j}."
    eps = 1e-6 if mutate == "ln_eps" else 1e-5
    x = x.double()
    xn = rd(_ln(x, W[p + "norm1.weight"], W[p + "norm1.bias"], eps))
    qkv = rd(xn @ wt(torch.cat([W[p + f"attn1.to_{n}.weight"] for n in "qkv"])).t())
    ch = 48 if (mutate == "chunk48" and chunk) else chunk
    outs, o = [], 0
    for L in lens:
        q, kk, v = (qkv[o:o + L, n * 512:(n + 1) * 512].reshape(L, 8, HD).transpose(0, 1) for n in range(3))
        s = (q @ kk.transpose(1, 2)) * 0.125
        s = s.masked_fill(~_dit_visible(L, ch, 1 if (mutate == "chunk_edge" and chunk) else 0)[None], float("-inf"))
        outs.append((torch.softmax(s, -1) @ v).transpose(0, 1).reshape(L, 512))
        o += L
    att = rd(torch.cat(outs, 0))
    x_mid = x + att @ wt(W[p + "attn1.to_out.0.weight"]).t() + W[p + "attn1.to_out.0.bias"]
    xn3 = rd(_ln(x_mid, W[p + "norm3.weight"], W[p + "norm3.bias"], eps))
    ff = rd(act("gelu_tanh" if mutate == "gelu_tanh" else "gelu", xn3 @ wt(W[p + "ff.net.0.proj.weight"]).t() + W[p + "ff.net.0.proj.bias"]))
    x_out = x_mid + ff @ wt(W[p + "ff.net.2.weight"]).t() + W[p + "ff.net.2.bias"]
    return dict(x=x, xn=xn, qkv=qkv, att=att, x_mid=x_mid, xn3=xn3, ff=ff, x_out=x_out)


def est_down_conv(W, skip_act, lens, rounding=False, mutate=None):
    """down_blocks.0.2: the causal k3 convolution from the down stage's output (its act copy) to the first mid stage's input"""
    e = "decoder.estimator.down_blocks.0.2."
    return (bf16 if rounding else (lambda t: t))(
        _seq_conv(skip_act.double(), _rdw(rounding)(W[e + "weight"]), W[e + "bias"], lens, -1 if mutate == "centred_pad" else -2))


def est_tail(W, up_act, lens, rounding=False, mutate=None):
    """up_blocks.0.2 (causal k3), final_block (causal k3, LN 1e-5, Mish) and final_proj on the up stage's output (its act copy)"""
    rd = bf16 if rounding else (lambda t: t)
    wt = _rdw(rounding)
    e = "decoder.estimator."
    sh = -1 if mutate == "centred_pad" else -2
    h1 = rd(_seq_conv(up_act.double(), wt(W[e + "up_blocks.0.2.weight"]), W[e + "up_blocks.0.2.bias"], lens, sh))
    c = _seq_conv(h1, wt(W[e + "final_block.block.0.weight"]), W[e + "final_block.block.0.bias"], lens, sh)
    mish = (lambda v: act("silu", v)) if mutate == "silu_for_mish" else _mish
    xa = rd(mish(_ln(c, W[e + "final_block.block.2.weight"], W[e + "final_block.block.2.bias"], 1e-6 if mutate == "ln_eps" else 1e-5)))
    return xa @ wt(W[e + "final_proj.weight"][..., 0]).t() + W[e + "final_proj.bias"]


def est_pack(x, mu, cond, spks, lens, rounding=False):
    """the estimator's packed input [x | mu | spks | cond] (decoder.py:431-434), as the bf16 path stores it"""
    inp = torch.cat([x.double(), mu.double(), spks.double()[_seq_ids(lens)], cond.double()], -1)
    return bf16(inp) if rounding else inp


def est_stage_input(W, k, acts, lens, rounding=False, mutate=None):
    """the act operand stage k reads, from the act copies acts[i] of the earlier stages' outputs: the packed input for the down
    stage (acts[-1] holds it), down_blocks.0.2 of the down stage's output for the first mid stage, the previous stage's output for
    the other mid stages, and [last mid output | down output] (the U-Net skip) for the up stage"""
    nst = len(est_stage_names(W["cfg"]))
    if k == 0:
        return acts[-1]
    down = est_down_conv(W, acts[0], lens, rounding, mutate) if (k == 1 or nst == 2) else None
    if k < nst - 1:
        return down if k == 1 else acts[k - 1]
    mid = acts[k - 1] if nst > 2 else down
    return torch.cat([acts[0], mid] if mutate == "skip_swap" else [mid, acts[0]], -1)


def flow_estimator(W, x, mu, cond, spks, t, lens, streaming, rounding=False, n_units=None, mutate=None):
    """the composed estimator on packed rows: returns (the residual stream after n_units units (all by default; the units of
    cvk_cfm_estimator_hidden), the output [sum T, 80] (None when n_units stops short))"""
    cfg = W["cfg"]
    nst, per = cfg.num_mid_blocks + 2, 1 + cfg.n_blocks
    n = nst * per if n_units is None else n_units
    rd = bf16 if rounding else (lambda v: v)
    temb = est_time(W, t, mutate)["temb"]
    acts = {-1: est_pack(x, mu, cond, spks, lens, rounding)}
    chunk = 50 if streaming else 0
    done = 0
    h = None
    for k in range(nst):
        h = est_resnet(W, k, est_stage_input(W, k, acts, lens, rounding, mutate), temb, lens, rounding, mutate)["x_out"]
        done += 1
        for j in range(cfg.n_blocks):
            if done == n:
                return h, None
            h = est_tblock(W, k, j, h, lens, chunk, rounding, mutate)["x_out"]
            done += 1
        if done == n and k < nst - 1:
            return h, None
        acts[k] = rd(h)
    return h, est_tail(W, acts[nst - 1], lens, rounding, mutate)


def flow_test_state_dict(cfg, seed):
    """CosyVoice2 flow weights for the block checks (oracle.flow.param_shapes names): fan-in-scaled matrices, so every resnet,
    transformer block and conformer layer changes the residual stream by O(1); pos_bias_u / v of O(1) (the synthetic default,
    0.1, leaves them under the noise of the content term); and every matrix the bf16 path streams as bf16 bf16-representable, so
    both references see the kernels' weights.  The time MLP, the per-stage time projections and the speaker projection stay fp32,
    as the kernels hold them."""
    from oracle import weights as oweights
    sd = oweights.synth_state_dict(oflow.param_shapes(cfg), seed, oflow.SYNTH_GAINS)
    g = torch.Generator().manual_seed(seed)
    for k in sd:
        if "pos_bias_" in k:
            sd[k] = torch.randn(sd[k].shape, generator=g)
        elif sd[k].dim() >= 2 and "time_mlp" not in k and ".mlp.1." not in k and "spk_embed" not in k and k != "input_embedding.weight":
            sd[k] = bf16(sd[k])
    return sd


# bounds of test_flow_blocks_gpu.py: largest |kernel - reference| of a unit over the rms of that row's contribution (encoder embedding,
# up-sampler, estimator resnet: the unit's output; conformer layer, transformer block: x_out - x; after_norm and the estimator tail:
# the output row).  Largest ratios measured on an H100 80GB HBM3 (700 W) over every layout, both masks and both contexts, in one run:
#   fp32: embedding 6.9e-6, conformer layer 1.6e-5, up-sampler 6.1e-6, after_norm 1.1e-6, resnet 2.0e-5, block 5.9e-6, tail 4.9e-6.
#     The fp32 sinusoids set that floor: the angles 1000 t 10000^(-i/159) (up to 950 rad) rounded to fp32 move the time projections
#     by 1e-5 and the resnet by 1.6e-5 of its rms on their own (four fifths of the measured 2.0e-5, at 1500 frames); the position
#     table's fp32 angles r 10000^(-2i/512) (r up to 749) move an up layer by 3.8e-6 on their own (a quarter of the layer's 1.6e-5).
#   bf16 (against the bf16-emulating reference): embedding 2.4e-3, conformer layer 9.5e-3, up-sampler 3.8e-3, after_norm 9.9e-7 (an
#     fp32 LayerNorm of the fp32 stream), resnet 4.3e-3, block 1.2e-2, tail 6.1e-3.
# Each bound is about twice that.
FLOW_TOL = {"fp32": dict(enc_embed=1.5e-5, enc_layer=3.5e-5, enc_up=1.2e-5, enc_out=2.5e-6, est_resnet=4e-5, est_block=1.2e-5,
                         est_out=1e-5),
            "bf16": dict(enc_embed=5e-3, enc_layer=0.02, enc_up=7.5e-3, enc_out=2.5e-6, est_resnet=9e-3, est_block=0.025,
                         est_out=0.0125)}
# full config (6, 4, 12, 4): largest error over the mean row rms of the reference, (encoder hidden, encoder output, estimator hidden
# after 70 units, estimator output), per reference, offline and streaming.  Measured, same run: fp32 vs exact 6.8e-6 / 7.1e-6 /
# 1.2e-5 / 1.3e-5, fp32 vs bf16-emulating 1.9e-2 / 2.2e-2 / 2.9e-2 / 3.6e-2, bf16 vs exact 2.0e-2 / 2.1e-2 / 3.1e-2 / 4.0e-2, bf16
# vs bf16-emulating 1.2e-2 / 1.2e-2 / 3.9e-2 / 4.7e-2 (over 70 units the two bf16 trajectories drift apart as far as each drifts
# from the exact one).  Bounds about twice that.
FLOW_STACK_TOL = {"fp32": {"exact": (1.5e-5, 1.5e-5, 2.5e-5, 2.5e-5), "bf16-emulating": (0.04, 0.045, 0.06, 0.075)},
                  "bf16": {"exact": (0.04, 0.04, 0.06, 0.08), "bf16-emulating": (0.025, 0.025, 0.08, 0.095)}}


# ------------------------------------------------------------------------------------------------ HiFT vocoders
# The CosyVoice2 vocoder (oracle/hift.py, generator.py:507-569 of the reference) and the CosyVoice3 causal one (oracle/hift_causal.py,
# generator.py:572-726) restated per sequence on time-major rows [rows, channels], in fp64, one read-out of cvk_hift_hidden at a
# time: the f0 predictor (hift_f0), the harmonic source (hift_phase, hift_source), the source STFT (hift_stft, read-out 0), conv_pre
# (1), per level i the up-sampling (hift_ups, 2 + 6i), the source branch (hift_source_branch, 3 + 6i), the three resblocks
# (hift_resblock, 4 + 6i .. 6 + 6i), the level output (hift_level_out, 7 + 6i), conv_post (hift_conv_post, 20) and the ISTFT
# (hift_istft).  Every convolution pads with zeros at the ends of the rows it is given, so a unit fed a window of a sequence's rows
# is exact on the window's inner rows.  `causal` selects the CosyVoice3 form: left-padded convolutions, conv_pre looking 4 frames to
# the right, nearest up-sampling + causal convolution, left-only source_downs padding, nearest phase up-sampling, stored noise
# indexed from the utterance's start.  `rounding` ("fp16" for IEEE half, "bf16" for hift_f16 = 0, None for exact) rounds where the
# 16-bit path stores a 16-bit value that the next kernel reads: the source STFT, the packed mel, xin, the Snake-activated operands a
# and ya of every resblock convolution and the level outputs; xu, xs, the resblock stream and si stay fp32 in the kernels and
# exact here.  `mutate` applies one of HIFT_MUTATIONS, the defects the sensitivity test of test_kernel_refs_cpu.py injects.
from oracle import hift as ohift  # noqa: E402
import numpy as np  # noqa: E402

HIFT_CH = (512, 256, 128, 64)
HIFT_RATE = (8, 40, 120)                 # level rows per mel frame (level 2 has one more row, the reflect pad, in front)
HIFT_MUTATIONS = ("lrelu_post", "no_reflect", "reflect_back", "down_pad", "poly_phase", "snake_swap", "dil1", "no_div3", "hann_sym",
                  "no_env", "phase_x", "clip_first", "uv_ge", "pre_left", "f0_look2")


def hift_weights(sd, causal):
    """the vocoder's weights in fp64 with every weight norm folded in float64 (the reference's CosyVoice3 f0 predictor runs as a
    float64 module, generator.py:716-717, so its parametrization computes g v / ||v|| in double; the fp32 folds of the other
    convolutions are within an fp32 ulp of it).  Keys: the state-dict names, "<conv>.weight" for the weight-normed ones."""
    W = {"causal": causal}
    for k, v in sd.items():
        if k.endswith(".parametrizations.weight.original0"):
            p = k[:-len(".parametrizations.weight.original0")]
            g, vv = v.double(), sd[p + ".parametrizations.weight.original1"].double()
            W[p + ".weight"] = g * vv / vv.flatten(1).norm(dim=1).view(g.shape)
        elif not k.endswith(".parametrizations.weight.original1"):
            W[k] = v.double()
    return W


def hift_test_state_dict(seed, causal, clip=False):
    """synthetic vocoder weights (oracle SYNTH_GAINS); clip=True shifts the bias of conv_post's magnitude channels so that some
    frames exceed ln 100 (the ISTFT's magnitude clip) and some samples exceed +-0.99 (the output clamp)"""
    from oracle import hift_causal as ohc, weights as oweights
    sd = oweights.synth_state_dict((ohc if causal else ohift).param_shapes(), seed, ohift.SYNTH_GAINS)
    if clip:
        b = sd["conv_post.bias"].clone()
        b[:9] += 2.5
        sd["conv_post.bias"] = b
    return sd


def _hrd(rounding):
    return (lambda t: t) if rounding is None else (lambda t: round_to(t, rounding))


def _conv(x, w, b, shift0, dil=1):
    return conv_rows(x, w, dil, shift0) + b.double()


def _elu(x):
    return torch.where(x > 0, x, torch.expm1(x))


def hift_f0(W, mel, mutate=None):
    """f0 predictor (f0_predictor.py:56-59; causal: :60-103, conv 0 reading 3 frames ahead, the others causal) on one sequence's
    mel rows [T, 80] -> f0 [T].  A streaming CosyVoice3 call's f0 (T - 3 frames) is the first T - 3 rows: its look-ahead frames are
    the next rows of the same mel."""
    x = mel.double()
    for i in range(5):
        p = f"f0_predictor.condnet.{2 * i}"
        if W["causal"]:
            sh = (-1 if mutate == "f0_look2" else 0) if i == 0 else -2
        else:
            sh = -1
        x = _elu(_conv(x, W[p + ".weight"], W[p + ".bias"], sh))
    return (x @ W["f0_predictor.classifier.weight"].t() + W["f0_predictor.classifier.bias"]).abs()[:, 0]


def hift_phase(f0, emulate=False):
    """SineGen2's per-frame phase (generator.py:255-257; the 1/480 linear down-sampling reads samples 480 d + 239 and 480 d + 240,
    both of frame d, so it is the frame's own value): (cumsum over frames of (f0 h / 24000 mod 1)) 2 pi 480 for harmonics h = 1..9,
    f0 [T] -> [T, 9].  emulate=True: the fp32 arithmetic of phase_kernel - fmodf(f0 h / 24000, 1) in fp32, a running sum in double
    rounded to float, ((c 2) pi_f) 480 in fp32 - returned as float32 values in fp64."""
    h = torch.arange(1, 10, dtype=torch.float64)
    if not emulate:
        rad = torch.remainder(f0.double()[:, None] * h / ohift.SR, 1.0)
        return torch.cumsum(rad, 0) * 2 * math.pi * ohift.UPSCALE
    f = f0.float().numpy().astype(np.float32)
    fn = f[:, None] * np.arange(1, 10, dtype=np.float32)[None]
    rad = np.fmod(fn / np.float32(24000.0), np.float32(1.0))
    c = np.cumsum(rad.astype(np.float64), 0).astype(np.float32)
    ph = ((c * np.float32(2.0)) * np.float32(math.pi)) * np.float32(480.0)
    return torch.from_numpy(ph.astype(np.float64))


def _interp_index(L, T):
    """F.interpolate(scale_factor=480, mode='linear', align_corners=False) as source_kernel computes it in fp32: srcf =
    fma(1/480, l + 0.5, -0.5) clamped at 0, i0 = trunc, i1 = min(i0 + 1, T - 1), l1 = srcf - i0, l0 = 1 - l1"""
    l = np.arange(L, dtype=np.float32)
    srcf = ((l + np.float32(0.5)).astype(np.float64) * np.float64(np.float32(1.0 / 480.0)) - 0.5).astype(np.float32)
    srcf = np.maximum(srcf, np.float32(0.0))
    i0 = srcf.astype(np.int64)
    i1 = np.minimum(i0 + 1, T - 1)
    l1 = (srcf - i0.astype(np.float32)).astype(np.float32)
    return i0, i1, (np.float32(1.0) - l1).astype(np.float32), l1


def hift_sample_phase(phase, causal, emulate=False):
    """the phase at every sample [480 T, 9] from the per-frame phase [T, 9]: linear x480 up-sampling (align_corners False) or,
    causal, nearest.  emulate=True: source_kernel's fp32 interpolation, fma(l0, p0, l1 * p1) with one rounding of the fused sum"""
    T = phase.shape[0]
    L = T * ohift.UPSCALE
    if causal:
        return phase.repeat_interleave(ohift.UPSCALE, 0)
    i0, i1, l0, l1 = _interp_index(L, T)
    if not emulate:
        p = phase.double()
        return torch.from_numpy(l0.astype(np.float64))[:, None] * p[i0] + torch.from_numpy(l1.astype(np.float64))[:, None] * p[i1]
    p = phase.numpy().astype(np.float32)
    t = (l1[:, None] * p[i1]).astype(np.float32)
    ph = (l0.astype(np.longdouble)[:, None] * p[i0].astype(np.longdouble) + t.astype(np.longdouble)).astype(np.float32)
    return torch.from_numpy(ph.astype(np.float64))


def hift_source(W, f0, noise, emulate=False, mutate=None):
    """the harmonic source of one sequence (SourceModuleHnNSF + SineGen2, generator.py:289-317, 358-375): f0 [T], noise [480 T, 9]
    (the CosyVoice2 Gaussian draws, or the CosyVoice3 stored noise from the utterance's start) -> s [480 T].  emulate=False: exact
    fp64 phase; emulate=True: the kernel's fp32 phase (hift_phase, hift_sample_phase), the rest in fp64."""
    causal = W["causal"]
    ph = hift_sample_phase(hift_phase(f0, emulate), causal, emulate)
    f0u = f0.double().repeat_interleave(ohift.UPSCALE)[:, None]
    uv = ((f0u >= ohift.VOICED_THR) if mutate == "uv_ge" else (f0u > ohift.VOICED_THR)).double()
    sines = (ph if mutate == "phase_x" else torch.sin(ph)) * ohift.SINE_AMP
    amp = uv * ohift.NOISE_STD + (1 - uv) * ohift.SINE_AMP / 3
    sw = sines * uv + amp * noise.double()[:f0u.shape[0]]
    return torch.tanh(sw @ W["m_source.l_linear.weight"].t() + W["m_source.l_linear.bias"])[:, 0]


def _hann(mutate):
    n = torch.arange(ohift.N_FFT, dtype=torch.float64)
    return 0.5 - 0.5 * torch.cos(2 * math.pi * n / (ohift.N_FFT - 1 if mutate == "hann_sym" else ohift.N_FFT))


def hift_stft(s, rounding=None, mutate=None):
    """torch.stft(n_fft 16, hop 4, periodic Hann, center, reflect) of one source s [L] -> [L / 4 + 1, 18] (re 0..8, im 9..17)"""
    x = torch.nn.functional.pad(s.double()[None, None], (8, 8), mode="reflect")[0, 0]
    fr = x.unfold(0, ohift.N_FFT, ohift.HOP) * _hann(mutate)
    n = torch.arange(ohift.N_FFT, dtype=torch.float64)
    ang = 2 * math.pi * torch.arange(9, dtype=torch.float64)[:, None] * n[None] / ohift.N_FFT
    return _hrd(rounding)(torch.cat([fr @ torch.cos(ang).t(), -(fr @ torch.sin(ang).t())], -1))


def hift_conv_pre(W, mel, rows=None, rounding=None, mutate=None):
    """conv_pre + leaky ReLU 0.1 (the first up-sampler's activation, stored as xin) on mel rows [T, 80] -> [rows (T), 512].  Causal:
    k5 reading 4 frames to the right; a streaming call's body covers rows = T - 7 frames of the mel it is given"""
    rd = _hrd(rounding)
    sh = (-4 if mutate == "pre_left" else 0) if W["causal"] else -3
    y = _conv(rd(mel.double()), W["conv_pre.weight"], W["conv_pre.bias"], sh)
    return rd(act("lrelu", y, 0.1))[:rows]


def hift_ups(W, i, x, head=True, mutate=None):
    """ups[i] on the level input x [R, C_i] (xin or the previous level output) -> xu [u R (+1 at i = 2 when head), C_(i+1)].
    CosyVoice2: ConvTranspose1d(stride u, padding (k - u) / 2); CosyVoice3: nearest x u then a causal k convolution.  At the last
    level the reflect pad (1, 0) puts a copy of row 1 in front when the rows start the sequence (head)."""
    u, k = ohift.UPS_RATES[i], ohift.UPS_KERNELS[i]
    w, b = W[f"ups.{i}.weight"], W[f"ups.{i}.bias"]
    R = x.shape[0]
    shift = 1 if mutate == "poly_phase" else 0
    if W["causal"]:
        y = _conv(x.double().repeat_interleave(u, 0), w, b, -(k - 1) + shift)
    else:
        full = torch.nn.functional.conv_transpose1d(x.double().t()[None], w, None, stride=u)[0].t()     # [(R - 1) u + k, C]
        full = torch.cat([full, full.new_zeros(1, full.shape[1])], 0)
        p = (k - u) // 2 + shift
        y = full[p:p + u * R] + b
    if i == 2 and head:
        if mutate == "no_reflect":
            y = torch.cat([torch.zeros_like(y[:1]), y], 0)
        elif mutate == "reflect_back":
            y = torch.cat([y, y[-2:-1]], 0)
        else:
            y = torch.cat([y[1:2], y], 0)
    return y


def _snake(x, alpha):
    return act("snake", x, alpha=alpha.double())


def hift_resblock(W, p, x, k, rounding=None, mutate=None):
    """ResBlock (generator.py:110-117; causal: left-padded convolutions) on x [R, C] (fp32 in the kernels): three dilation steps
    x += conv2(snake2(conv1(snake1(x), dilation d))), d = 1, 3, 5; the Snake outputs a and ya are the 16-bit operands.  Returns x."""
    rd = _hrd(rounding)
    x = x.double()
    for n, d in enumerate(ohift.RB_DILS):
        d = 1 if mutate == "dil1" else d
        a1, a2 = W[f"{p}.activations1.{n}.alpha"], W[f"{p}.activations2.{n}.alpha"]
        if mutate == "snake_swap":
            a1, a2 = a2, a1
        s1, s2 = (-(k - 1) * d, -(k - 1)) if W["causal"] else (-((k - 1) * d) // 2, -(k - 1) // 2)
        ya = rd(_snake(_conv(rd(_snake(x, a1)), W[f"{p}.convs1.{n}.weight"], W[f"{p}.convs1.{n}.bias"], s1, d), a2))
        x = x + _conv(ya, W[f"{p}.convs2.{n}.weight"], W[f"{p}.convs2.{n}.bias"], s2)
    return x


def hift_source_downs(W, i, stft, rounding=None, mutate=None):
    """source_downs[i] on the source STFT rows [F, 18] (the 16-bit operand) -> si [F / s rows at the level's rate, C].  CosyVoice2:
    Conv1d(k 2s, stride s, padding s / 2) (k 1 at the last level); CosyVoice3: left padding s - 1 only.  The STFT rows given start
    at frame 120 f of the level's first mel frame f (or at the front pad row at the last level's head)."""
    s = (15, 3, 1)[i]
    w, b = W[f"source_downs.{i}.weight"], W[f"source_downs.{i}.bias"]
    x = stft.double()
    if s == 1:
        return x @ w[:, :, 0].t() + b
    F = x.shape[0]
    left = (s - 1) if W["causal"] else (7, 1)[i]
    left += 1 if mutate == "down_pad" else 0
    xp = torch.nn.functional.pad(x.t()[None], (left, 2 * s))
    y = torch.nn.functional.conv1d(xp, w, b, stride=s)[0].t()
    return y[:F // s]


def hift_source_branch(W, i, stft, xu, rounding=None, mutate=None):
    """read-out 3 + 6i: xu + source_resblocks[i](source_downs[i](stft)); stft rows as hift_source_downs takes them, xu the level's
    rows (the same rows of the sequence)"""
    si = hift_source_downs(W, i, stft, rounding, mutate)[:xu.shape[0]]
    return xu.double() + hift_resblock(W, f"source_resblocks.{i}", si, ohift.SRC_RB_KERNELS[i], rounding, mutate)


def hift_level_out(i, xs, rounding=None, mutate=None):
    """read-out 7 + 6i: leaky ReLU(xs / 3), slope 0.1 before the next up-sampler and the default 0.01 before conv_post
    (generator.py:513, 532), stored as the next convolution's operand"""
    slope = 0.1 if (i < 2 or mutate == "lrelu_post") else 0.01
    return _hrd(rounding)(act("lrelu", xs.double() if mutate == "no_div3" else xs.double() / 3, slope))


def hift_conv_post(W, x):
    """read-out 20: conv_post (k7, centred or causal) on the last level output [R, 64] -> [R, 18]"""
    return _conv(x.double(), W["conv_post.weight"], W["conv_post.bias"], -6 if W["causal"] else -3)


def hift_istft(xp, drop=0, mutate=None):
    """magnitude min(exp(x[:9]), 100), phase sin(x[9:]), inverse real DFT, periodic-Hann overlap-add over the window envelope, trim
    8, clamp +-0.99 (generator.py:533-538): conv_post rows [F, 18] -> wav [4 (F - 1) - drop]"""
    x = xp.double()
    mag = torch.exp(x[:, :9].clamp(max=100.0)) if mutate == "clip_first" else torch.exp(x[:, :9]).clamp(max=100.0)
    ph = torch.sin(x[:, 9:])
    re, im = mag * torch.cos(ph), mag * torch.sin(ph)
    Fr = x.shape[0]
    w = _hann(mutate)
    n = torch.arange(16, dtype=torch.float64)
    ang = 2 * math.pi * torch.arange(9, dtype=torch.float64)[:, None] * n[None] / 16
    coef = torch.full((9, 1), 2.0, dtype=torch.float64)
    coef[0] = coef[-1] = 1.0
    ci = -coef * torch.sin(ang) / 16
    ci[0] = ci[-1] = 0
    frames = (re @ (coef * torch.cos(ang) / 16) + im @ ci) * w
    total = 4 * (Fr - 1) + 16
    y = torch.zeros(total, dtype=torch.float64)
    env = torch.zeros(total, dtype=torch.float64)
    idx = (torch.arange(Fr)[:, None] * 4 + torch.arange(16)[None]).reshape(-1)
    y.index_add_(0, idx, frames.reshape(-1))
    env.index_add_(0, idx, (w * w).repeat(Fr))
    y = y[8:total - 8]
    if mutate != "no_env":
        y = y / env[8:total - 8]
    return y[:y.shape[0] - drop].clamp(-ohift.AUDIO_LIMIT, ohift.AUDIO_LIMIT)


def hift_body(W, mel, s, body_frames=None, rounding=None, mutate=None):
    """the composed body of one sequence, every read-out of cvk_hift_hidden: mel [T, 80], source s [480 T_src] -> list of 21
    read-outs (fp64).  body_frames: Tb (T by default; a streaming CosyVoice3 call's T - 7, with its STFT cut to 120 Tb + 1 frames)"""
    Tb = mel.shape[0] if body_frames is None else body_frames
    stft = hift_stft(s, rounding, mutate)[:120 * Tb + 1]
    outs = [stft, hift_conv_pre(W, mel, Tb, rounding, mutate)]
    x = outs[1]
    for i in range(3):
        xu = hift_ups(W, i, x, True, mutate)
        outs.append(xu)
        xu = hift_source_branch(W, i, stft, xu, rounding, mutate)
        outs.append(xu)
        xs = 0
        for j, k in enumerate(ohift.RB_KERNELS):
            xs = xs + hift_resblock(W, f"resblocks.{3 * i + j}", xu, k, rounding, mutate)
            outs.append(xs)
        x = hift_level_out(i, xs, rounding, mutate)
        outs.append(x)
    outs.append(hift_conv_post(W, x))
    return outs


def hift_decode(W, mel, s, finalize=True, rounding=None, mutate=None):
    """decode of one sequence: (read-outs, wav).  CosyVoice3 streaming (finalize False): mel [T, 80] with T - 3 source frames; the
    body covers T - 7 frames, the last 480 samples are dropped"""
    T = mel.shape[0]
    Tb = T if finalize else T - 7
    outs = hift_body(W, mel, s, Tb, rounding, mutate)
    return outs, hift_istft(outs[20], 0 if finalize else ohift.UPSCALE, mutate)


# frames of halo a window of a level's rows needs on each side, so that the rows a unit computes from zero padding at the window's
# cut edges stay outside the frames that are compared: the receptive field of the unit at that rate (an 11-tap resblock with
# dilations 1, 3, 5 reaches 60 rows each way, twice that to the left when causal; conv_pre 4 frames) rounded up to whole frames
_HALO = {False: (8, 2, 1), True: (16, 4, 2)}


def hift_level_rows(i, f0, f1):
    """rows of mel frames [f0, f1) at level i (0, 1, 2; -1 the mel rate): the last level's row 0 is the reflect pad, in front of
    frame 0"""
    if i < 0:
        return f0, f1
    if i < 2:
        return HIFT_RATE[i] * f0, HIFT_RATE[i] * f1
    return (0 if f0 == 0 else 120 * f0 + 1), 120 * f1 + 1


def _unit_level(u):
    return -1 if u == 1 else (2 if u in (0, 20) else (u - 2) // 6)


def hift_unit_refs(W, K, mel, Tb, windows, rounding=None):
    """fp64 references of read-outs 1 .. 20 of one sequence, each unit fed the kernel's own read-outs K[u] (fp64, the sequence's
    rows) of the units before it: per window [fa, fb) of body frames, {u: (reference rows, kernel rows)} of the frames [fa, fb) at
    the unit's rate, each computed from the window widened by the unit's halo.  mel [T, 80] (T >= Tb: a streaming call's conv_pre
    reads look-ahead rows past Tb)."""
    halo = _HALO[W["causal"]]
    T = mel.shape[0]
    res = []
    for fa, fb in windows:
        out = {}

        def grab(u, g0, g1):
            lo, hi = hift_level_rows(_unit_level(u), g0, g1)
            return K[u][lo:hi]

        def keep(u, ref, g0):
            i = _unit_level(u)
            base = hift_level_rows(i, g0, g0 + 1)[0]
            lo, hi = hift_level_rows(i, fa, fb)
            out[u] = (ref[lo - base:hi - base], K[u][lo:hi])

        g0, g1 = max(0, fa - 5), min(Tb, fb + 5)
        keep(1, hift_conv_pre(W, mel[g0:min(T, g1 + 5)], g1 - g0, rounding), g0)
        for i in range(3):
            h = halo[i]
            g0, g1 = max(0, fa - h), min(Tb, fb + h)
            prev = 1 if i == 0 else 7 + 6 * (i - 1)
            keep(2 + 6 * i, hift_ups(W, i, grab(prev, g0, g1), g0 == 0), g0)
            if i < 2:
                stft = K[0][120 * g0:120 * g1 + 1]
            else:
                lo, hi = hift_level_rows(2, g0, g1)
                stft = K[0][lo:hi]
            keep(3 + 6 * i, hift_source_branch(W, i, stft, grab(2 + 6 * i, g0, g1), rounding), g0)
            xu = grab(3 + 6 * i, g0, g1)
            for j, k in enumerate(ohift.RB_KERNELS):
                xs = grab(3 + 6 * i + j, g0, g1) if j > 0 else 0
                keep(4 + 6 * i + j, xs + hift_resblock(W, f"resblocks.{3 * i + j}", xu, k, rounding), g0)
            keep(7 + 6 * i, hift_level_out(i, grab(6 + 6 * i, g0, g1), rounding), g0)
        g0, g1 = max(0, fa - 1), min(Tb, fb + 1)
        keep(20, hift_conv_post(W, grab(19, g0, g1)), g0)
        res.append(out)
    return res


def hift_windows(Tb, seams=(), width=6):
    """the body frames checked on a long sequence: the head, the tail and `width` frames around every seam frame; the whole
    sequence when it is short"""
    if Tb <= 3 * width + 4:
        return [(0, Tb)]
    w = [(0, width), (Tb - width, Tb)]
    for s in seams:
        if width < s < Tb - width:
            w.append((s - width // 2, s + width - width // 2))
    return w


def hift_ratio(ref, got):
    """largest |got - ref| over the rms of its reference row, the row rms floored at a tenth of the mean row rms (a row of a
    leaky-ReLU output can be nearly zero)"""
    rms = ref.pow(2).mean(-1, keepdim=True).sqrt()
    rms = rms.clamp_min(0.1 * rms.mean().item() + 1e-30)
    r = ((got.double() - ref) / rms).abs().max().item()
    assert r == r, "NaN"
    return r


HIFT_UNIT_GROUP = {1: "conv_pre", 20: "conv_post", **{2 + 6 * i: "ups" for i in range(3)}, **{3 + 6 * i: "source_branch" for i in range(3)},
                   **{4 + 6 * i + j: "resblock" for i in range(3) for j in range(3)}, **{7 + 6 * i: "level_out" for i in range(3)}}


def hift_source_ulp_bound(W, f0):
    """what one fp32 ulp of the phase can move the source by: the phase is held in fp32 (the reference's own arithmetic), and one
    ulp of phase harmonic h (up to 2 rad at 2.7e7 rad) moves sin by up to min(2, ulp), the sine by 0.1 times that and the tanh of the
    merged source by at most sum_h 0.1 |l_linear_h| min(2, 2 ulp_h) - the rounding of c, of (c 2) pi 480 and of the interpolation
    each contribute half an ulp.  Plus 1e-5 for the rest of the fp32 arithmetic."""
    ph = hift_phase(f0).abs().max(0).values.float()
    ulp = (torch.nextafter(ph, torch.full_like(ph, float("inf"))) - ph).double()
    return (0.1 * W["m_source.l_linear.weight"][0].abs() * (2 * ulp).clamp(max=2.0)).sum().item() + 1e-5


# bounds of test_hift_blocks_gpu.py and test_zz_hift3_blocks_gpu.py: largest |kernel - reference| of a unit over the rms of its
# reference row (kernel_refs.hift_ratio), fp32 against the exact reference, f16 (hift_f16 = 1, IEEE-half operands) and bf16
# (hift_f16 = 0) against the reference rounding where the 16-bit path stores; istft: largest |wav - fp64 ISTFT of the kernel's
# conv_post|; f0: largest error over the utterance's f0 rms (the CosyVoice2 predictor runs fp32 in every mode).  Largest values
# measured on an H100 80GB HBM3 (700 W) in one run over every length, layout, final and streaming call of both vocoders:
#   fp32: stft 1.1e-6, conv_pre 4.2e-6, ups 9.5e-6, source_branch 1.0e-5, resblock 8.0e-6, level_out 4.4e-7, conv_post 2.5e-6,
#     istft 4.5e-6, f0 2.6e-6;
#   f16: stft 3.4e-3, conv_pre 4.4e-3, ups 1.2e-3, source_branch 4.5e-3, resblock 4.6e-3, level_out 2.5e-3, conv_post 7.1e-4,
#     istft 4.5e-6;
#   bf16: stft 2.9e-2, conv_pre 3.5e-2, ups 9.7e-3, source_branch 3.6e-2, resblock 4.0e-2, level_out 1.2e-2, conv_post 6.8e-3,
#     istft 4.4e-6.
# (A 16-bit STFT element that the kernel's fp32 sum and the fp64 sum round to neighbouring 16-bit values is one 16-bit ulp apart;
# over the rms of an 18-column row that is up to the stft ratios above.)  Each bound is about twice the measurement.  source: the
# largest |source - fp32-emulating source|, measured 4.5e-8; held at 1e-5, far under the 1e-2 .. 1e-1 that one ulp of a long
# utterance's phase moves the source by.  The CosyVoice3 f0 is held to one fp32 ulp of the fp64-fold predictor (measured 0.5 ulp:
# correctly rounded).
HIFT_TOL = {
    "fp32": dict(stft=2.5e-6, conv_pre=1e-5, ups=2e-5, source_branch=2e-5, resblock=1.6e-5, level_out=1e-6, conv_post=5e-6, istft=1e-5,
                 f0=5e-6),
    "f16": dict(stft=7e-3, conv_pre=9e-3, ups=2.5e-3, source_branch=9e-3, resblock=1e-2, level_out=5e-3, conv_post=1.5e-3, istft=1e-5,
                f0=5e-6),
    "bf16": dict(stft=6e-2, conv_pre=7e-2, ups=2e-2, source_branch=7e-2, resblock=8e-2, level_out=2.5e-2, conv_post=1.4e-2, istft=1e-5,
                 f0=5e-6),
    "source": 1e-5,
}
