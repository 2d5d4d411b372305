"""CosyVoice3 batched offline synthesis, full-size Fun-CosyVoice3-0.5B shape (synthetic weights), bf16.

Two measurements in one process, after the card's name, power limit and max SM clock:
  f0:      one batch-32 hift3_inference (the mel lengths of the 32 requests below) under torch.profiler: device time of the f0
           predictor's convolution kernels, of the rest of the call's kernels, and the f0 convolutions' FLOP rate.
  feature: two arms alternated after a warm-up of each - (a) one tts_batch of the 32 requests, (b) 32 threads each calling tts()
           offline - with audio-s/s, the per-stage ms of tts_batch (return_stats), libcvk launches per arm and the maximum waveform
           difference between the arms (both arms draw the same uniforms per request).
`--f0-only` runs the first part alone (it only needs cvk hift3_inference, so it also runs on builds without tts_batch for
CosyVoice3).  min_token_text_ratio = max_token_text_ratio = 5: the synthetic LM never emits eos.  Needs an H100; there is no CPU path.

    python tools/cv3_batch_bench.py [--rounds 2] [--f0-only] [--small]
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def f0_profile(model, lens):
    import torch
    from torch.profiler import ProfilerActivity, profile
    g = torch.Generator(device="cpu").manual_seed(7)
    mel = (torch.randn(sum(lens), 80, generator=g) * 2 - 5).to(model.device)
    with torch.cuda.stream(model.stream):
        model.ctx.hift3_inference(mel, lens, finalize=True)                  # warm-up
    model.stream.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        with torch.cuda.stream(model.stream):
            model.ctx.hift3_inference(mel, lens, finalize=True)
        model.stream.synchronize()
    f0_us, rest_us, names = 0.0, 0.0, {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        t = t if t is not None else getattr(e, "cuda_time_total", 0.0)
        if t <= 0 or e.key.startswith("cuda") or "Memcpy" in e.key or "Memset" in e.key:
            continue
        if "f0_conv_dmma_kernel" in e.key or "conv_f64_kernel" in e.key:
            f0_us += t
            names[e.key[:60]] = round(t / 1e3, 3)
        else:
            rest_us += t
    rows = sum(lens)
    flop = 2.0 * rows * 512 * (4 * 80 + 4 * 3 * 512)                     # layer 0 (80 -> 512, k4) + four 512 -> 512 k3 layers
    return {"batch": len(lens), "mel_frames": rows, "f0_conv_ms": round(f0_us / 1e3, 3), "rest_of_call_ms": round(rest_us / 1e3, 3),
            "f0_conv_tflops": round(flop / (f0_us * 1e-6) / 1e12, 2) if f0_us else None, "f0_kernels": names}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2, help="timed runs of each arm (alternating)")
    ap.add_argument("--f0-only", action="store_true")
    ap.add_argument("--small", action="store_true", help="debug: 2-layer LM / 2-block DiT (NOT the measured configuration)")
    args = ap.parse_args()
    import torch
    from cosyvoice_b200 import synth
    from cosyvoice_b200.model3 import B200CosyVoice3Model
    assert torch.cuda.is_available(), "needs a CUDA device (H100); there is no CPU path"
    dev = torch.device("cuda", 0)
    nl, depth = (2, 2) if args.small else (24, 22)
    model = B200CosyVoice3Model(precision="bf16", device=0, workspace_gb=40.0)
    model.load_state_dicts(*synth.cosyvoice3_state_dicts(dev, 1986, nl, depth))
    torch.cuda.empty_cache()
    model.min_token_text_ratio = model.max_token_text_ratio = 5.0
    reqs = synth.batch32_zero_shot()
    for r in reqs:
        r["prompt_text"][0, 5] = 151646                                   # <|endofprompt|> closes the CosyVoice3 prompt text (llm.py:585)
    lens = [2 * 5 * int(r["text"].shape[1]) for r in reqs]                 # mel frames the flow makes of 5 ids per text id
    print(json.dumps({"card (name, power limit, max SM clock)": card(), "model": "small debug" if args.small else
                      "Fun-CosyVoice3-0.5B shape, synthetic weights", "precision": "bf16"}), flush=True)
    print(json.dumps({"f0": f0_profile(model, lens)}), flush=True)
    if args.f0_only:
        return

    U = torch.rand(5 * max(int(r["text"].shape[1]) for r in reqs) + 8, 1, 2, generator=torch.Generator().manual_seed(11))
    Ub = U.expand(-1, len(reqs), -1).contiguous()
    model.uniforms_override = U                                          # the threads' tts(): every request draws U

    def batch_arm():
        t0 = time.perf_counter()
        wavs, stats = model.tts_batch(reqs, uniforms=Ub, return_stats=True)
        return time.perf_counter() - t0, wavs, stats

    def thread_arm():
        out = [None] * len(reqs)

        def one(i):
            kw = {k: v for k, v in reqs[i].items()}
            out[i] = torch.cat([o["tts_speech"] for o in model.tts(**kw, stream=False)], 1)
        t0 = time.perf_counter()
        th = [threading.Thread(target=one, args=(i,)) for i in range(len(reqs))]
        for t in th:
            t.start()
        for t in th:
            t.join()
        return time.perf_counter() - t0, out, None

    arms = {"tts_batch": batch_arm, "threads_tts": thread_arm}
    for name, fn in arms.items():                                         # warm-up: every shape of the timed runs
        fn()
    torch.cuda.synchronize()
    res = {k: [] for k in arms}
    last = {}
    for r in range(args.rounds):
        for name, fn in arms.items():
            l0 = model.ctx.launch_count()
            dt, wavs, stats = fn()
            launches = model.ctx.launch_count() - l0
            audio = sum(w.shape[1] for w in wavs) / 24000.0
            row = {"round": r, "s": round(dt, 3), "audio_s": round(audio, 2), "audio_s_per_s": round(audio / dt, 1), "launches": launches}
            if stats:
                row.update({k: round(stats[k], 1) for k in ("lm_ms", "flow_ms", "hift_ms")})
            res[name].append(row)
            last[name] = wavs
            print(json.dumps({name: row}), flush=True)
    a, b = last["tts_batch"], last["threads_tts"]
    same = [x.shape == y.shape for x, y in zip(a, b)]
    d = max(((x - y).abs().max().item() for x, y, s in zip(a, b, same) if s), default=None)
    print(json.dumps({"summary": {k: {"audio_s_per_s_mean": round(sum(x["audio_s_per_s"] for x in v) / len(v), 1)} for k, v in res.items()},
                      "same_lengths": f"{sum(same)}/{len(same)}", "max_abs_wav_diff_between_arms": d}), flush=True)


if __name__ == "__main__":
    main()
