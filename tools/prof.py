#!/usr/bin/env python
"""Single-stage runner for profiler captures.  Runs one stage of the batch-32 Z10 workload with
eager launches (no CUDA graph) so that every kernel shows up as its own launch.

  ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file gpurun_out/lm.csv python tools/prof.py --stage lm --steps 4
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cosyvoice_b200 import synth  # noqa: E402
from cosyvoice_b200.model import B200CosyVoice2Model  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--stage", default="lm", choices=["lm", "flow", "hift", "all"])
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--steps", type=int, default=4, help="lm: decode steps; flow: Euler steps")
ap.add_argument("--precision", default="bf16")
ap.add_argument("--graph", type=int, default=0)
args = ap.parse_args()

dev = torch.device("cuda", 0)
llm, flow, hift = synth.cosyvoice2_state_dicts(dev)
m = B200CosyVoice2Model(precision=args.precision, device=0, workspace_gb=40.0)
if args.stage in ("lm", "all"):
    m.ctx.load_state_dict("llm", llm, [24])
if args.stage in ("flow", "all"):
    m.ctx.load_state_dict("flow", flow, [6, 4, 12, 4])
    from cosyvoice_b200.model import cfm_rand_noise
    m.ctx.set_cfm_noise(cfm_rand_noise())
if args.stage in ("hift", "all"):
    m.ctx.load_state_dict("hift", hift)
del llm, flow, hift
m.ctx.set_option("use_graph", args.graph)
m.min_token_text_ratio = m.max_token_text_ratio = 5.0
inputs = synth.batch32_zero_shot(args.batch)
torch.cuda.synchronize()
torch.cuda.profiler.start()
if args.stage in ("lm", "all"):
    m.max_token_text_ratio = m.min_token_text_ratio = args.steps / 40.0 if args.stage == "lm" else 5.0
    ids = m.lm_generate([i["text"] for i in inputs], [i["prompt_text"] for i in inputs], [i["llm_prompt_speech_token"] for i in inputs],
                        steps_per_sync=args.steps)
    print("lm tokens", [len(x) for x in ids][:4])
g = torch.Generator().manual_seed(0)
toks = [torch.randint(0, 6561, (1, 5 * i["text"].shape[1]), generator=g, dtype=torch.int32) for i in inputs]
if args.stage in ("flow", "all"):
    m.n_timesteps = args.steps if args.stage == "flow" else 10
    mel, lens = m.flow_batch(toks, [i["flow_prompt_speech_token"] for i in inputs], [i["prompt_speech_feat"] for i in inputs],
                             [i["flow_embedding"] for i in inputs])
    print("mel", mel.shape)
if args.stage in ("hift", "all"):
    lens = [2 * t.shape[1] for t in toks]
    mel = torch.randn(sum(lens), 80, device=dev) * 2 - 5
    wav, _ = m.hift_batch(mel, lens)
    print("wav", wav.shape)
torch.cuda.synchronize()
torch.cuda.profiler.stop()
