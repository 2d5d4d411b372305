"""Kernel table of one batch-32 flow stage (flow_batch, Z10 shapes, 10 Euler steps, bf16) under torch.profiler with CUDA activities.

Writes <out>/flow_kernels_<opt><value>.md: per kernel name the time and launch count of one flow_batch, then the
time of the estimator's transformer-block launches by role.  Roles come from the launch order inside a block: the attention kernel
is preceded by the qkv GEMM (the generic kernel or the row-panel one; and, for the first block of a stage, LN1) and followed either by
the fused feed-forward kernel, which also does the out projection, or by the out GEMM, LN3, the ff1 and the ff2 GEMMs (and the next
block's LN1).  Not a bench: the profiler slows the host.

  python tools/flow_tblock_prof.py --opt flow_fused_ff --values 0,1 --out /tmp/flow_prof
"""
import argparse
import collections
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from cosyvoice_b200 import synth  # noqa: E402
from cosyvoice_b200.model import B200CosyVoice2Model, cfm_rand_noise  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--opt", default="flow_fused_ff")
ap.add_argument("--values", default="0,1")
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--out", required=True, help="directory for the kernel tables")
a = ap.parse_args()
os.makedirs(a.out, exist_ok=True)

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


def short(name):
    """demangled kernel name without the parameter list"""
    return name.replace("(anonymous namespace)::", "").split("(")[0]


def is_ln(n):
    return "layernorm256_kernel" in n


def roles(kern):
    """(role, name, us) of the estimator transformer-block launches, found by their order around each attention launch"""
    out = []
    names = [short(k["name"]) for k in kern]
    for i, n in enumerate(names):
        if "attn_wg_kernel" not in n or i < 1 or i + 1 >= len(names):
            continue
        if not ("conv_gemm_wg_kernel" in names[i - 1] or "qkv_panel_kernel" in names[i - 1]):
            continue
        fused = "ffn_fused_kernel" in names[i + 1]
        if not fused and not ("conv_gemm_wg_kernel" in names[i + 1] and i + 2 < len(names) and is_ln(names[i + 2])):
            continue      # the conformer encoder's layers continue otherwise
        seq = [("qkv", i - 1), ("attention", i)]
        if i >= 2 and is_ln(names[i - 2]):
            seq.insert(0, ("ln1 (stage's first block)", i - 2))
        if fused:
            seq.append(("out + ffn (out projection + LN3 + ff1 + ff2 + LN1)", i + 1))
        else:
            seq += [("out", i + 1), ("ln3", i + 2), ("ff1", i + 3), ("ff2", i + 4)]
            if i + 5 < len(names) and is_ln(names[i + 5]):
                seq.append(("ln1 (next block)", i + 5))
        out += [(r, names[j], kern[j]["dur"]) for r, j in seq]
    return out


for v in [int(x) for x in a.values.split(",")]:
    m.ctx.set_option(a.opt, v)
    m.flow_batch(*args)                      # warm-up: module loads, workspace
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        m.flow_batch(*args)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        trace = os.path.join(td, "trace.json")
        prof.export_chrome_trace(trace)
        ev = json.load(open(trace))["traceEvents"]
    kern = sorted((e for e in ev if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    total = sum(k["dur"] for k in kern)
    span = (kern[-1]["ts"] + kern[-1]["dur"] - kern[0]["ts"]) if kern else 0
    by = collections.defaultdict(lambda: [0.0, 0])
    for k in kern:
        b = by[short(k["name"])]
        b[0] += k["dur"]
        b[1] += 1
    lines = [f"# flow_batch, batch {a.batch}, {a.opt}={v}, {torch.cuda.get_device_name(0)}", "",
             f"kernel time {total / 1e3:.1f} ms in {len(kern)} launches; first kernel start to last kernel end {span / 1e3:.1f} ms", "",
             "| kernel | ms | launches | share |", "|---|---:|---:|---:|"]
    for n, (us, c) in sorted(by.items(), key=lambda t: -t[1][0]):
        lines.append(f"| `{n[:110]}` | {us / 1e3:.2f} | {c} | {100 * us / max(total, 1):.1f}% |")
    rs = collections.defaultdict(lambda: [0.0, 0])
    for r, n, us in roles(kern):
        b = rs[(r, n)]
        b[0] += us
        b[1] += 1
    lines += ["", "## estimator transformer blocks by role", "", "| role | kernel | ms | launches | share of all kernel time |", "|---|---|---:|---:|---:|"]
    for (r, n), (us, c) in sorted(rs.items(), key=lambda t: -t[1][0]):
        lines.append(f"| {r} | `{n[:80]}` | {us / 1e3:.2f} | {c} | {100 * us / max(total, 1):.1f}% |")
    ffn = sum(us for (r, _), (us, _) in rs.items() if r.startswith(("out", "ln3", "ff1", "ff2", "ln1 (next")))
    nff = sum(c for (r, _), (_, c) in rs.items() if r.startswith(("out + ffn", "ff2")))
    lines += ["", f"out projection + LN3 + ff1 + ff2 + next LN1 (or the fused kernel): {ffn / 1e3:.1f} ms, {100 * ffn / max(total, 1):.1f}% of the "
              f"flow's kernel time; {ffn / max(nff, 1):.1f} us per block ({nff} blocks)"]
    txt = "\n".join(lines) + "\n"
    open(os.path.join(a.out, f"flow_kernels_{a.opt}{v}.md"), "w").write(txt)
    print(txt)
