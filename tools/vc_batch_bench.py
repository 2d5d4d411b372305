"""Batched voice conversion: 32 VC requests (inference_vc inputs: 250 source speech tokens, a 75-token / 150-frame prompt and a
speaker embedding, the Z10 shape) with synthetic full-size weights in bf16, CosyVoice2 or (--cv3) CosyVoice3.

After the card's name, power limit and max SM clock (one nvidia-smi query), two arms alternate after a warm-up of each:
  (a) one tts_batch of the 32 requests (no LM call: every row is a VC row),
  (b) 32 threads each calling tts(source_speech_token=...) offline,
with audio-s/s, the per-stage ms of tts_batch (return_stats), libcvk launches per arm and the maximum waveform difference between
the arms (CosyVoice2 draws its vocoder noise from the model's generator in both arms, so only the lengths compare there).
`--resample` instead times one batch-32 cvk_mel_resample at speed 0.8 (500 -> 625 frames per request) with CUDA events over
many launches.  Needs an H100; there is no CPU path.

    python tools/vc_batch_bench.py [--cv3] [--rounds 2] [--resample]
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


def vc_requests(n=32, n_source=250):
    import torch
    from cosyvoice_b200 import synth
    out = []
    for i in range(n):
        u = synth.z10_utterance(i)
        g = torch.Generator().manual_seed(5000 + i)
        out.append(dict(source_speech_token=torch.randint(0, 6561, (1, n_source), generator=g, dtype=torch.int32),
                        flow_prompt_speech_token=u["flow_prompt_speech_token"], prompt_speech_feat=u["prompt_speech_feat"],
                        flow_embedding=u["flow_embedding"]))
    return out


def resample_timing(iters=500, batch=32, T=500, speed=0.8):
    import torch
    from cosyvoice_b200 import cvk
    c = cvk.Context(0, "bf16", workspace_gb=0.25)
    Tn = int(T / speed)
    mel = torch.randn(batch * T, 80, device="cuda")
    for _ in range(10):
        c.mel_resample(mel, [T] * batch, [Tn] * batch)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        c.mel_resample(mel, [T] * batch, [Tn] * batch)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / iters
    moved = 4 * 80 * batch * (T + Tn)                                    # each input row read once (L2 serves the re-reads), each output row written
    c.close()
    return {"batch": batch, "frames_in": T, "frames_out": Tn, "speed": speed, "us_per_call": round(us, 2),
            "effective_GB_s": round(moved / (us * 1e-6) / 1e9, 1), "launches_timed": iters}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cv3", action="store_true", help="CosyVoice3 (DiT flow, causal vocoder) instead of CosyVoice2")
    ap.add_argument("--rounds", type=int, default=2, help="timed runs of each arm (alternating)")
    ap.add_argument("--resample", action="store_true", help="time one batch-32 cvk_mel_resample at speed 0.8 instead")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a CUDA device (H100); there is no CPU path"
    head = {"card (name, power limit, max SM clock)": card()}
    if args.resample:
        print(json.dumps(head), flush=True)
        print(json.dumps({"mel_resample": resample_timing()}), flush=True)
        return
    from cosyvoice_b200 import synth
    dev = torch.device("cuda", 0)
    if args.cv3:
        from cosyvoice_b200.model3 import B200CosyVoice3Model
        model = B200CosyVoice3Model(precision="bf16", device=0, workspace_gb=40.0)
        model.load_state_dicts(*synth.cosyvoice3_state_dicts(dev))
    else:
        from cosyvoice_b200.model import B200CosyVoice2Model
        model = B200CosyVoice2Model(precision="bf16", device=0, workspace_gb=24.0)
        model.load_state_dicts(*synth.cosyvoice2_state_dicts(dev))
    torch.cuda.empty_cache()
    reqs = vc_requests()
    head.update({"model": ("Fun-CosyVoice3-0.5B" if args.cv3 else "CosyVoice2-0.5B") + " shape, synthetic weights", "precision": "bf16",
                 "requests": f"{len(reqs)} VC: 250 source tokens, 75 prompt tokens, 150 prompt frames"})
    print(json.dumps(head), flush=True)

    def batch_arm():
        t0 = time.perf_counter()
        wavs, stats = model.tts_batch(reqs, return_stats=True)
        return time.perf_counter() - t0, wavs, stats

    def thread_arm():
        out = [None] * len(reqs)

        def one(i):
            out[i] = torch.cat([o["tts_speech"] for o in model.tts(**reqs[i], stream=False)], 1)
        t0 = time.perf_counter()
        th = [threading.Thread(target=one, args=(i,)) for i in range(len(reqs))]
        for t in th:
            t.start()
        for t in th:
            t.join()
        return time.perf_counter() - t0, out, None

    arms = {"tts_batch": batch_arm, "threads_tts": thread_arm}
    for fn in arms.values():                                              # warm-up: every shape of the timed runs
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
    d = max(((x - y).abs().max().item() for x, y, s in zip(a, b, same) if s), default=None) if args.cv3 else None
    print(json.dumps({"summary": {k: {"audio_s_per_s_mean": round(sum(x["audio_s_per_s"] for x in v) / len(v), 1)} for k, v in res.items()},
                      "same_lengths": f"{sum(same)}/{len(same)}", "max_abs_wav_diff_between_arms": d}), flush=True)


if __name__ == "__main__":
    main()
