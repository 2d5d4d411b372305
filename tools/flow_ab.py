"""A/B timing of the flow stage (batch-32 Z10 shapes, 10 Euler steps, bf16) under two values of one library option.  Not a bench."""
import argparse, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from cosyvoice_b200 import synth
from cosyvoice_b200.model import B200CosyVoice2Model, cfm_rand_noise

ap = argparse.ArgumentParser()
ap.add_argument("--opt", default="enc_tc_attn")
ap.add_argument("--values", default="0,1")
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--batch", type=int, default=32)
a = ap.parse_args()
dev = torch.device("cuda", 0)
llm, flow, hift = synth.cosyvoice2_state_dicts(dev)
m = B200CosyVoice2Model(precision="bf16", device=0, workspace_gb=40.0)
m.ctx.load_state_dict("flow", flow, [6, 4, 12, 4])
m.ctx.set_cfm_noise(cfm_rand_noise())
del llm, flow, hift
inputs = synth.batch32_zero_shot(a.batch)
g = torch.Generator().manual_seed(0)
toks = [torch.randint(0, 6561, (1, 5 * i["text"].shape[1]), generator=g, dtype=torch.int32) for i in inputs]
args = (toks, [i["flow_prompt_speech_token"] for i in inputs], [i["prompt_speech_feat"] for i in inputs], [i["flow_embedding"] for i in inputs])
outs = {}
for v in [int(x) for x in a.values.split(",")]:
    m.ctx.set_option(a.opt, v)
    ms = []
    for r in range(a.reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(m.stream):
            e0.record()
        mel, lens = m.flow_batch(*args)
        with torch.cuda.stream(m.stream):
            e1.record()
        e1.synchronize()
        if r:
            ms.append(e0.elapsed_time(e1))
    outs[v] = mel.clone()
    m.ctx.profile(1)
    m.flow_batch(*args)
    torch.cuda.synchronize()
    fam = {n: m.ctx.profile_read(i) for i, n in enumerate(("gemm_tc", "gemm_simt", "attention"))}
    m.ctx.profile(0)
    print(f"{a.opt}={v}: flow {sum(ms) / len(ms):.1f} ms (runs {[round(x, 1) for x in ms]}); instrumented families (ms, launches):",
          {k: (round(x["ms"], 1), x["launches"]) for k, x in fam.items()})
vs = list(outs)
if len(vs) == 2:
    d = (outs[vs[0]] - outs[vs[1]]).abs()
    print(f"mel: max |{vs[0]} - {vs[1]}| = {d.max().item():.4g}, mean {d.mean().item():.4g}, |mel| max {outs[vs[0]].abs().max().item():.3g}")
