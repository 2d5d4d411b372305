"""A/B of the conv-GEMM epilogue on the accumulator fragments (option "tc_epi_frag" = 1) against the epilogue that first transposes the
fragments to rows (= 0), in one call.  Not a bench.

Writes <out>/epi_ab.md (and prints it), with the card's name, power limit and maximum SM clock read in the same call:
  probe   one cvk_op_conv_gemm launch per shape below, the option values alternating, `reps` timings per value of `iters` back-to-back
          launches each; the time is the GEMM kernel's own device time from a torch.profiler trace (the call also converts its operands)
  flow    tools/flow_ab.py --opt tc_epi_frag --values 0,1 (flow stage ms, equality of the mels)
  bench   bench.py --steps 3 --warmup 3 with --opt tc_epi_frag=0 and without, alternating, the dumped waveforms compared value for value

  python tools/epi_ab.py --out /tmp/epi_ab [--only probe,flow,bench] [--reps 5] [--iters 50] [--bench-runs 3] [--values 0,1]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ap = argparse.ArgumentParser()
ap.add_argument("--out", required=True)
ap.add_argument("--only", default="probe,flow,bench")
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--iters", type=int, default=50)
ap.add_argument("--bench-runs", type=int, default=3)
ap.add_argument("--values", default="0,1")
a = ap.parse_args()
only = a.only.split(",")
values = [int(v) for v in a.values.split(",")]
os.makedirs(a.out, exist_ok=True)
lines = []

# name: rows, K, N, taps, shift0, operand / output dtype, epilogue keywords of Context.conv_gemm, kernel
PROBES = {
    "flow qkv projection (row-panel kernel)": (40064, 256, 1536, 1, 0, "bf16", dict(), "qkv_panel_kernel"),
    "flow resnet k3 conv": (40064, 256, 256, 3, -1, "bf16", dict(bias=True), "conv_gemm_wg_kernel"),
    "flow attention out projection, fp32 residual": (40064, 512, 256, 1, 0, "fp32", dict(bias=True, resid=True), "conv_gemm_wg_kernel"),
    "flow out projection, accumulated (direct stores)": (40064, 512, 256, 1, 0, "fp32", dict(bias=True, accumulate=True), "conv_gemm_wg_kernel"),
    "DiT linear 1024 -> 1024": (16384, 1024, 1024, 1, 0, "bf16", dict(bias=True), "conv_gemm_wg_kernel"),
    "HiFT resblock conv 128 ch, k11, Snake": (131072, 128, 128, 11, -5, "fp16", dict(bias=True, act1="snake", alpha1=True), "conv_gemm_wg_kernel"),
}


def say(s=""):
    print(s, flush=True)
    lines.append(s)
    open(os.path.join(a.out, "epi_ab.md"), "w").write("\n".join(lines) + "\n")


def run(cmd):
    p = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if p.returncode != 0:
        say(f"FAILED ({p.returncode}): {' '.join(cmd)}\n{p.stdout[-3000:]}")
        sys.exit(1)
    return p.stdout


say("# tc_epi_frag A/B")
say("card: " + run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"]).strip())

if "probe" in only:
    import torch
    from torch.profiler import ProfilerActivity, profile
    from cosyvoice_b200 import cvk
    c = cvk.Context(0, "bf16", 12.0)
    g = torch.Generator().manual_seed(0)
    say(f"\n## probe: one conv-GEMM launch, {a.iters} launches per timing, {a.reps} timings per value, alternating; kernel device time\n")
    say("| shape | rows x K -> N, taps | tc_epi_frag | µs per launch (median) | min-max | TFLOP/s | TB/s over algorithmic bytes |")
    say("|---|---|---:|---:|---:|---:|---:|")
    for name, (rows, K, N, taps, shift0, dt, kw, kernel) in PROBES.items():
        x = torch.randn(rows, K, generator=g).cuda()
        w = (torch.randn(N, K, taps, generator=g) * (K * taps) ** -0.5).cuda()
        args = dict(operand="bf16" if dt == "fp32" else dt, out=torch.randn(rows, N).cuda(), out_dtype=dt, shift0=shift0)
        if kw.get("bias"):
            args["bias"] = (0.1 * torch.randn(N, generator=g)).cuda()
        if kw.get("resid"):
            args["resid"] = torch.randn(rows, N, generator=g).cuda()
        if kw.get("accumulate"):
            args["accumulate"] = True
        if kw.get("act1"):
            args["act1"] = kw["act1"]
        if kw.get("alpha1"):
            args["alpha1"] = (torch.rand(N, generator=g) * 2.7 + 0.3).cuda()
        us = {v: [] for v in values}
        for rep in range(a.reps + 1):
            for v in values:
                c.set_option("tc_epi_frag", v)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(a.iters):
                        c.conv_gemm(x, [0], [rows], w, **args)
                    torch.cuda.synchronize()
                ev = [e for e in prof.key_averages() if kernel in e.key]
                assert len(ev) == 1 and ev[0].count == a.iters, [(e.key, e.count) for e in prof.key_averages()]
                if rep:
                    us[v].append(ev[0].device_time_total / ev[0].count)
        c.set_option("tc_epi_frag", 1)
        esz = 4 if dt == "fp32" else 2
        flop = 2.0 * rows * K * N * taps
        byt = rows * K * 2 + N * K * taps * 2 + rows * N * esz * (2 if (kw.get("resid") or kw.get("accumulate")) else 1)
        for v in values:
            med = statistics.median(us[v])
            say(f"| {name} | {rows} x {K} -> {N}, {taps} | {v} | {med:.1f} | {min(us[v]):.1f}-{max(us[v]):.1f} | {flop / med / 1e6:.0f} | "
                f"{byt / med / 1e6:.2f} |")
    del c

if "flow" in only:
    say(f"\n## flow stage (tools/flow_ab.py --opt tc_epi_frag --values 0,1 --reps {a.reps})\n")
    say("```\n" + run([sys.executable, "tools/flow_ab.py", "--opt", "tc_epi_frag", "--values", "0,1", "--reps", str(a.reps)]).strip() + "\n```")

if "bench" in only:
    import numpy as np
    say(f"\n## bench.py --steps 3 --warmup 3, {a.bench_runs} runs per value, alternating\n")
    with tempfile.TemporaryDirectory() as td:
        res = {0: [], 1: []}
        for i in range(a.bench_runs):
            for o in (0, 1):
                d = os.path.join(td, f"o{o}_{i}")
                cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", "3", "--warmup", "3", "--no-cpu-baseline", "--dump-outputs", d]
                if o == 0:
                    cmd += ["--opt", "tc_epi_frag=0"]
                out = run(cmd)
                js = [json.loads(l) for l in out.splitlines() if l.startswith("{")]
                res[o].append(js[-1])
                say(f"- tc_epi_frag={o} run {i}: value {js[-1].get('value')} {js[-1].get('unit', '')}")
        ref = np.load(os.path.join(td, "o0_0", "wav.npy"))
        same = all(np.array_equal(ref, np.load(os.path.join(td, f"o{o}_{i}", "wav.npy"))) and
                   np.array_equal(np.load(os.path.join(td, "o0_0", "wav_lens.npy")), np.load(os.path.join(td, f"o{o}_{i}", "wav_lens.npy")))
                   for o in (0, 1) for i in range(a.bench_runs))
        say(f"\nwaveforms of all {2 * a.bench_runs} runs identical value for value ({ref.size} values): {same}")
        for o in (0, 1):
            v = [r["value"] for r in res[o]]
            say(f"tc_epi_frag={o}: value median {statistics.median(v):.1f}, min-max {min(v):.1f}-{max(v):.1f}")
        json.dump(res, open(os.path.join(a.out, "bench_lines.json"), "w"), indent=1)
        if not same:
            sys.exit(1)
