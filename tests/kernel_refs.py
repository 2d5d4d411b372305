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
    # where a decode path stores a bf16 value that the next stage reads: the fused chain and the persistent kernel keep the qkv and
    # gate/up projections in fp32 (split-K partial sums reduced by the attention unit, SwiGLU in the GEMM epilogue); the per-op chain
    # stores both as bf16 first
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
