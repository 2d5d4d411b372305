"""A/B of the row-panel GEMM (qkv_panel_kernel, option "flow_qkv_panel") against the generic conv-GEMM, in one call.  Not a bench.

Writes <out>/gemm_panel_ab.md (and prints it), with the card's name, power limit and maximum SM clock read in the same call:
  probe   the estimator's qkv shape (40064 x 256 -> 1536, bf16 out): option 0 / 1 alternating, CUDA events around `op_iters` back-to-back
          launches inside cvk_op_conv1d; then option 0 / 2 over smaller row counts (where the row threshold of option 1 sits)
  flow    tools/flow_ab.py --opt flow_qkv_panel --values 0,1 (flow stage ms, equality of the mels)
  bench   bench.py --steps 3 --warmup 3 with --opt flow_qkv_panel=0 and without, alternating, the dumped waveforms compared value for value
  prof    tools/flow_tblock_prof.py --opt flow_qkv_panel --values 0,1 (torch.profiler run: the qkv role's total)

  python tools/gemm_panel_ab.py --out /tmp/panel_ab [--only probe,flow,bench,prof] [--reps 5] [--bench-runs 3]
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
ap.add_argument("--only", default="probe,flow,bench,prof")
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--iters", type=int, default=50)
ap.add_argument("--bench-runs", type=int, default=3)
a = ap.parse_args()
only = a.only.split(",")
os.makedirs(a.out, exist_ok=True)
lines = []


def say(s=""):
    print(s, flush=True)
    lines.append(s)
    open(os.path.join(a.out, "gemm_panel_ab.md"), "w").write("\n".join(lines) + "\n")


def run(cmd):
    p = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if p.returncode != 0:
        say(f"FAILED ({p.returncode}): {' '.join(cmd)}\n{p.stdout[-3000:]}")
        sys.exit(1)
    return p.stdout


say("# flow_qkv_panel A/B")
say("card: " + run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"]).strip())

if "probe" in only:
    import torch
    from cosyvoice_b200 import cvk
    c = cvk.Context(0, "bf16", 12.0)
    c.set_option("op_iters", a.iters)
    c.set_option("op_out_bf16", 1)
    K, N = 256, 1536
    g = torch.Generator().manual_seed(0)
    w = torch.randn(N, K, 1, generator=g) / K ** 0.5

    def time_rows(rows, opts):
        """µs per launch for each option value, alternating, a.reps repetitions each after one untimed round"""
        x = torch.randn(rows, K, generator=g)
        us = {o: [] for o in opts}
        for rep in range(a.reps + 1):
            for o in opts:
                c.set_option("flow_qkv_panel", o)
                st = torch.cuda.Stream()
                with torch.cuda.stream(st):
                    c.conv1d(x, [rows], w, None)
                if rep:
                    us[o].append(c.last_op_ms() * 1e3)
        c.set_option("flow_qkv_panel", 1)
        return us

    def row(rows, o, v):
        med = statistics.median(v)
        flop = 2.0 * rows * K * N
        byt = rows * K * 2 + N * K * 2 + rows * N * 2          # A read, W read, qkv written: the algorithmic HBM traffic
        return (f"| {rows} | {o} | {med:.1f} | {min(v):.1f}-{max(v):.1f} | {flop / med / 1e6:.0f} | {byt / med / 1e6:.2f} | "
                f"{byt / 1e6:.0f} |")

    say(f"\n## probe: rows x 256 -> 1536, bf16 out, {a.iters} launches per timing, {a.reps} timings per arm, alternating\n")
    say("| rows | flow_qkv_panel | µs per launch (median) | min-max | TFLOP/s | TB/s over algorithmic bytes | MB |")
    say("|---:|---:|---:|---:|---:|---:|---:|")
    for o, v in time_rows(40064, (0, 1)).items():
        say(row(40064, o, v))
    say("\nsmaller row counts, generic (0) against forced panel kernel (2):\n")
    say("| rows | flow_qkv_panel | µs per launch (median) | min-max | TFLOP/s | TB/s over algorithmic bytes | MB |")
    say("|---:|---:|---:|---:|---:|---:|---:|")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for rows in (3200, 64 * sms, 128 * sms, 192 * sms):
        for o, v in time_rows(rows, (0, 2)).items():
            say(row(rows, o, v))
    del c

if "flow" in only:
    say(f"\n## flow stage (tools/flow_ab.py --opt flow_qkv_panel --values 0,1 --reps {a.reps})\n")
    say("```\n" + run([sys.executable, "tools/flow_ab.py", "--opt", "flow_qkv_panel", "--values", "0,1", "--reps", str(a.reps)]).strip() + "\n```")

if "bench" in only:
    import numpy as np
    say(f"\n## bench.py --steps 3 --warmup 3, {a.bench_runs} runs per arm, alternating\n")
    with tempfile.TemporaryDirectory() as td:
        res = {0: [], 1: []}
        for i in range(a.bench_runs):
            for o in (0, 1):
                d = os.path.join(td, f"o{o}_{i}")
                cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", "3", "--warmup", "3", "--no-cpu-baseline", "--dump-outputs", d]
                if o == 0:
                    cmd += ["--opt", "flow_qkv_panel=0"]
                out = run(cmd)
                js = [json.loads(l) for l in out.splitlines() if l.startswith("{")]
                res[o].append(js[-1])
                say(f"- flow_qkv_panel={o} run {i}: value {js[-1].get('value')} {js[-1].get('unit', '')}")
        ref = np.load(os.path.join(td, "o0_0", "wav.npy"))
        same = all(np.array_equal(ref, np.load(os.path.join(td, f"o{o}_{i}", "wav.npy"))) and
                   np.array_equal(np.load(os.path.join(td, "o0_0", "wav_lens.npy")), np.load(os.path.join(td, f"o{o}_{i}", "wav_lens.npy")))
                   for o in (0, 1) for i in range(a.bench_runs))
        say(f"\nwaveforms of all {2 * a.bench_runs} runs identical value for value ({ref.size} values): {same}")
        for o in (0, 1):
            v = [r["value"] for r in res[o]]
            say(f"flow_qkv_panel={o}: value median {statistics.median(v):.1f}, min-max {min(v):.1f}-{max(v):.1f}")
        json.dump(res, open(os.path.join(a.out, "bench_lines.json"), "w"), indent=1)
        if not same:
            sys.exit(1)

if "prof" in only:
    say("\n## estimator blocks by role (tools/flow_tblock_prof.py, torch.profiler run)\n")
    run([sys.executable, "tools/flow_tblock_prof.py", "--opt", "flow_qkv_panel", "--values", "0,1", "--out", a.out])
    for v in (0, 1):
        txt = open(os.path.join(a.out, f"flow_kernels_flow_qkv_panel{v}.md")).read()
        say(f"flow_qkv_panel={v}:\n")
        say("\n".join(l for l in txt.splitlines() if l.startswith(("| qkv", "| role", "|---|---|", "kernel time"))))
        say()
