"""Kernel time of the tensor-core attention (`attn_wg_kernel`, bf16) at the shapes the pipeline runs it at, through
`cvk_op_attention_ex` with the library's per-family profiler: only the attention launch is timed, not the fp32 -> bf16 operand
packing around it.

Shapes (lengths from the batch-32 Z10 workload, synth.batch32_zero_shot: 150 prompt mel frames + 2 x 5 x (40..60) text ids):
  flow      64 sequences (32 utterances x 2 CFG branches), 8 heads, full attention (chunk 0, the offline flow)
  flow-c50  the same with block-causal chunks of 50 frames (streaming flow)
  dit       the same 64 sequences, 16 heads (CosyVoice3 DiT)
  lm        LM prefill, 14 query / 2 key-value heads, causal, 32 rows of 12 + (40..60) + 75 + 2 positions

Each shape is warmed up, then launched until more than a second of kernel time has been recorded.  TFLOP/s counts the visible
(query, key) pairs only: 4 x 64 x heads FLOP per pair (QK^T and PV).  Writes <out>/attn_shapes.json and prints a table with the
card's name and power limit.

  python tools/attn_shapes_prof.py --out /tmp/attn
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from cosyvoice_b200 import cvk  # noqa: E402

FAM_ATTN = 2
MIN_MS = 1000.0

ap = argparse.ArgumentParser()
ap.add_argument("--out", required=True, help="directory for attn_shapes.json")
a = ap.parse_args()
os.makedirs(a.out, exist_ok=True)

n_text = [40 + (i * 7) % 21 for i in range(32)]           # synth.batch32_zero_shot(32)
flow_lens = [150 + 10 * n for n in n_text] * 2              # mel frames = 2 x (75 prompt + 5 n_text) tokens; both CFG branches
lm_lens = [12 + n + 75 + 2 for n in n_text]
SHAPES = [("flow", flow_lens, 8, 8, 0), ("flow-c50", flow_lens, 8, 8, 50), ("dit", flow_lens, 16, 16, 0), ("lm", lm_lens, 14, 2, 1)]


def visible_pairs(lens, chunk):
    """(query, key) pairs inside the mask: all keys, or keys up to the end of the query's chunk"""
    tot = 0
    for L in lens:
        if chunk == 0:
            tot += L * L
        else:
            tot += sum(min(L, (i // chunk + 1) * chunk) for i in range(L))
    return tot


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info = r.stdout.strip() or "not reported"
    except (OSError, subprocess.SubprocessError):
        info = "not reported"
    return name, info


ctx = cvk.Context(0, "bf16", workspace_gb=4.0)
g = torch.Generator().manual_seed(0)
rows = []
for name, lens, H, kvh, chunk in SHAPES:
    R = sum(lens)
    q = torch.randn(R, H * 64, generator=g).cuda()
    k = torch.randn(R, kvh * 64, generator=g).cuda()
    v = torch.randn(R, kvh * 64, generator=g).cuda()
    off = [0] * len(lens)

    def run(n):
        ctx.profile(1)
        for _ in range(n):
            ctx.attention_ex(q, k, v, lens, lens, off, H, kvh, chunk=chunk)
        r = ctx.profile_read(FAM_ATTN)
        ctx.profile(0)
        assert r["launches"] == n, r
        return r["ms"]

    run(5)                                                   # module load, tensor-map encoder, arena
    per = run(5) / 5
    n = max(20, int(MIN_MS / max(per, 1e-3)) + 1)
    ms = run(n)
    while ms < MIN_MS:                                       # the estimate above came from a short window
        n *= 2
        ms = run(n)
    pairs = visible_pairs(lens, chunk)
    flop = 4.0 * 64 * H * pairs
    row = dict(shape=name, seqs=len(lens), len_min=min(lens), len_max=max(lens), heads=H, kv_heads=kvh, chunk=chunk, launches=n,
               ms_total=ms, ms_per_launch=ms / n, gflop_per_launch=flop / 1e9, tflops=flop / (ms / n) / 1e9)
    rows.append(row)
    print(f"{name:9s} {len(lens)} seqs of {min(lens)}-{max(lens)}, H {H}/{kvh}, chunk {chunk}: {ms / n:.4f} ms/launch "
          f"({n} launches, {ms:.0f} ms), {row['tflops']:.1f} TFLOP/s", flush=True)
    del q, k, v

name, info = card()
print(f"card: {name}; power.limit, clocks.max.sm: {info}")
json.dump(dict(card=name, power_limit_max_sm_clock=info, shapes=rows), open(os.path.join(a.out, "attn_shapes.json"), "w"), indent=1)
