"""Batched streaming synthesis vs one thread per stream, full-size CosyVoice2 (synthetic weights), bf16.

B concurrent streaming Z10 requests (75 prompt tokens, 50 text ids -> 250 speech ids, hop 25 -> 50 -> 100) in two arms, alternated
in one process after warm-up:
  (a) B threads, each calling tts(stream=True) on the shared model (how bench.py --workload cv3-bistream drives its model);
  (b) one tts_stream_batch over the B requests (multi-slot flow session, one launch sequence per stage per poll round).
Prints audio-s/s, first-chunk latency, libcvk launches per arm, the slot-pool size, the card's name and power limit, and whether
both arms produced the same chunk lengths.  They do not: the threads of arm (a) share the model's token_hop_len, which every tts()
call doubles after each chunk (the reference's behaviour, cli/model.py:359-360), so arm (a) runs fewer, longer chunks than a
request served alone - less work per audio second than arm (b), whose requests each keep the single-request schedule.  Both arms
produce the same number of samples per request.  Needs an H100; there is no CPU path.

    python tools/stream_batch_bench.py [--batches 8 16] [--rounds 2] [--small]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[8, 16])
    ap.add_argument("--rounds", type=int, default=2, help="timed runs of each arm per batch size (alternating)")
    ap.add_argument("--small", action="store_true", help="debug: 2-layer LM / reduced flow (NOT the measured configuration)")
    args = ap.parse_args()
    import torch
    from cosyvoice_b200 import synth
    from cosyvoice_b200.model import B200CosyVoice2Model
    assert torch.cuda.is_available(), "needs a CUDA device (H100); there is no CPU path"
    dev = torch.device("cuda", 0)
    nl, fcfg = (2, (2, 1, 2, 2)) if args.small else (24, (6, 4, 12, 4))
    model = B200CosyVoice2Model(precision="bf16", device=0, workspace_gb=10.0)
    model.load_state_dicts(*synth.cosyvoice2_state_dicts(dev, 1986, nl, fcfg))
    torch.cuda.empty_cache()
    model.min_token_text_ratio = model.max_token_text_ratio = 5.0       # exactly 250 speech ids per request (bench.py TOKEN_RATIO)
    model.stream_cache_frames = 768                                     # 75 prompt + 250 speech tokens = 650 mel frames
    model.stream_batch_slots = max(args.batches)
    info = {"card": card(), "model": "small debug" if args.small else "CosyVoice2-0.5B shape, synthetic weights", "precision": "bf16"}
    print(json.dumps(info), flush=True)

    def threaded(reqs):
        out = [None] * len(reqs)

        def one(i):
            t0, first, lens = time.perf_counter(), None, []
            for o in model.tts(**reqs[i], stream=True):
                first = first if first is not None else time.perf_counter() - t0
                lens.append(o["tts_speech"].shape[1])
            out[i] = (first, lens)
        model.token_hop_len = 25
        ts = [threading.Thread(target=one, args=(i,)) for i in range(len(reqs))]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        return out

    def batched(reqs):
        t0 = time.perf_counter()
        first, lens = [None] * len(reqs), [[] for _ in reqs]
        for i, o in model.tts_stream_batch(reqs):
            first[i] = first[i] if first[i] is not None else time.perf_counter() - t0
            lens[i].append(o["tts_speech"].shape[1])
        return list(zip(first, lens))

    for B in args.batches:
        reqs = [synth.z10_utterance(i, 50) for i in range(B)]
        arms = {"threads": threaded, "batched": batched}
        for f in arms.values():                     # warm-up: every shape, sessions, slot pool
            f(reqs)
        res = {k: {"audio_s": 0.0, "wall_s": 0.0, "first": [], "launches": 0, "lens": None} for k in arms}
        for _ in range(args.rounds):
            for name, f in arms.items():
                torch.cuda.synchronize()
                l0 = model.ctx.launch_count()
                t0 = time.perf_counter()
                out = f(reqs)
                torch.cuda.synchronize()
                r = res[name]
                r["wall_s"] += time.perf_counter() - t0
                r["launches"] += model.ctx.launch_count() - l0
                r["audio_s"] += sum(sum(lens) for _, lens in out) / 24000.0
                r["first"] += [f0 for f0, _ in out]
                r["lens"] = [lens for _, lens in out]
        line = {"batch": B, "card": info["card"], "slots": model.stream_slots,
                "slot_pool_bytes": model.ctx.flow_stream_bytes(model._slot_pool) if model._slot_pool else 0,
                "same_chunk_lengths": res["threads"]["lens"] == res["batched"]["lens"],
                "same_samples_per_request": [sum(x) for x in res["threads"]["lens"]] == [sum(x) for x in res["batched"]["lens"]]}
        for name, r in res.items():
            fs = sorted(r["first"])
            line[name] = {"audio_s_per_s": r["audio_s"] / r["wall_s"], "first_chunk_s": {"median": fs[len(fs) // 2], "max": fs[-1]},
                          "launches_per_run": r["launches"] // args.rounds}
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
