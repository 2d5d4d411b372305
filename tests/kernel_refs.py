"""Plain fp64 CPU references of the kernels checked by test_kernel_edges_gpu.py.  test_kernel_refs_cpu.py checks them against
torch's scaled_dot_product_attention and the oracle LM, so that the yardsticks are trusted before they judge a kernel."""
import torch

from oracle import lm as olm

HD = 64
NH, NKV = olm.N_HEAD, olm.N_KV              # 14 query heads, 2 kv heads
QKV_N = (NH + 2 * NKV) * HD                 # 1152


def bf16(x):
    """round to bf16 (nearest even), returned in x's dtype"""
    return x.to(torch.bfloat16).to(x.dtype)


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
