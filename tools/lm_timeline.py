"""Per-kernel timeline of ONE LM decode step inside the replayed CUDA graph (debug option chain_timeline: %globaltimer stamps
written by the kernels themselves - entry of CTA 0, CTA 0 past griddepcontrol.wait, last CTA end).  Not a bench."""
import argparse, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from cosyvoice_b200 import synth
from cosyvoice_b200.model import B200CosyVoice2Model

ap = argparse.ArgumentParser()
ap.add_argument("--pdl", type=int, default=1)
ap.add_argument("--steps", type=int, default=96)
ap.add_argument("--layers", type=int, default=24)
a = ap.parse_args()
dev = torch.device("cuda", 0)
sds = synth.cosyvoice2_state_dicts(dev, 1986, a.layers, (2, 1, 2, 2))
m = B200CosyVoice2Model(precision="bf16", device=0, workspace_gb=8.0)
m.load_state_dicts(*sds)
m.ctx.set_option("pdl", a.pdl)
m.ctx.set_option("chain_timeline", 1)
m.min_token_text_ratio = m.max_token_text_ratio = a.steps / 50.0
inputs = synth.batch32_zero_shot(32)
ids = m.lm_generate([i["text"] for i in inputs], [i["prompt_text"] for i in inputs], [i["llm_prompt_speech_token"] for i in inputs])
torch.cuda.synchronize()
tl = m.ctx.debug_read(4096)
names = ["head", "head_finish", "sampler"]
for l in range(a.layers):
    names += [f"L{l}.qkv", f"L{l}.attn", f"L{l}.o", f"L{l}.fin1", f"L{l}.gate_up", f"L{l}.down", f"L{l}.fin2"]
rows = [(names[i] if i < len(names) else f"k{i}", tl[4 * i], tl[4 * i + 1], tl[4 * i + 2]) for i in range(len(tl) // 4) if tl[4 * i]]
t0 = rows[0][1]
print(f"pdl={a.pdl} kernels={len(rows)} tokens/row={len(ids[0])}")
print(f"{'kernel':14s} {'entry':>8s} {'waited':>8s} {'end':>8s} | {'body':>6s} {'to next waited':>8s}   (us, relative to first entry)")
agg = {}
for i, (n, e, w, d) in enumerate(rows):
    nxt = rows[i + 1][2] if i + 1 < len(rows) else d
    body = (d - w) / 1e3 if d else float("nan")
    period = (nxt - w) / 1e3
    k = n.split(".")[-1]
    agg.setdefault(k, []).append((body, period, (w - e) / 1e3))
    if i < 3 + 14 or i >= len(rows) - 7:
        print(f"{n:14s} {(e - t0) / 1e3:8.2f} {(w - t0) / 1e3:8.2f} {(d - t0) / 1e3 if d else float('nan'):8.2f} | {body:6.2f} {period:8.2f}")
print("\nper kernel kind: mean body (waited->last CTA end), mean period (waited->next kernel waited), mean early start (entry->waited)")
for k, v in agg.items():
    n = len(v)
    print(f"  {k:12s} n={n:3d} body {sum(x[0] for x in v) / n:6.2f}  period {sum(x[1] for x in v) / n:6.2f}  early {sum(x[2] for x in v) / n:6.2f}")
print(f"step total (first waited -> last end): {(rows[-1][3] - rows[0][2]) / 1e3:.1f} us")
