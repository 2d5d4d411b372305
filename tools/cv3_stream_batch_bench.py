"""Batched CosyVoice3 streaming vs one thread per stream, full-size Fun-CosyVoice3-0.5B shape (synthetic weights), bf16.

B concurrent config #4 requests (synth.cv3_bistream_request: 75 prompt tokens / 150 prompt mel frames, 48 text ids in 4 chunks ->
240 speech ids, hop 25 -> 50 -> 100 with 3 look-ahead tokens), `bistream_max_tokens` and `silent_tokens = []` as bench.py sets
them, in three arms alternated in one process after warm-up:
  (a) one tts_bistream_batch over the B text generators;
  (b) B threads, each calling tts(text=<generator>, stream=True) on the shared model (bench.py --workload cv3-bistream's arm);
  (c) one tts_stream_batch over the same requests with the text as one token tensor (min = max token ratio 5: 240 ids).
Prints audio-s/s, first-chunk latency (median, max), libcvk launches per run, the slot-pool size and its bytes, the card's name,
power limit and max SM clock, and whether the arms produced the same chunk lengths.  The threaded arm's do not match: its threads
share the model's token_hop_len, which every tts() call doubles after each chunk (the reference's behaviour, cli/model.py:359-360),
so it runs fewer, longer chunks than a request served alone - less vocoder and flow work per audio second than the batched arms.
The text-streaming arms (a) and (b) yield 237 ids per request where arm (c) yields 240: the text-streaming decode's cap of 240
counts the 3 forced fill tokens it does not yield.

Then it times one mixed vocoder round (B/2 streaming histories + B/2 final utterances in one hift3_inference_rows call) against the
two homogeneous hift3_inference calls it replaces, with CUDA events around the calls only.  Needs an H100; there is no CPU path.

    python tools/cv3_stream_batch_bench.py [--batches 8 16] [--rounds 2] [--small]
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
    ap.add_argument("--small", action="store_true", help="debug: 2-layer LM / depth-2 DiT (NOT the measured configuration)")
    args = ap.parse_args()
    import torch
    from cosyvoice_b200 import synth
    from cosyvoice_b200.model3 import B200CosyVoice3Model
    assert torch.cuda.is_available(), "needs a CUDA device (H100); there is no CPU path"
    dev = torch.device("cuda", 0)
    nl, depth = (2, 2) if args.small else (24, 22)
    model = B200CosyVoice3Model(precision="bf16", device=0, workspace_gb=10.0)
    model.load_state_dicts(*synth.cosyvoice3_state_dicts(dev, 1986, nl, depth))
    torch.cuda.empty_cache()
    model.silent_tokens = []                                            # uniform synthetic ids: count every id (bench.py)
    n_text = 48
    model.bistream_max_tokens = int(n_text * 5.0)                       # bench.py: the decode is capped at 240 ids
    model.min_token_text_ratio = model.max_token_text_ratio = 5.0       # arm (c): exactly 240 ids per request
    model.stream_cache_frames = 768                                     # 150 prompt + 480 generated mel frames
    model.stream_batch_slots = max(args.batches)
    info = {"card": card(), "model": "small debug" if args.small else "Fun-CosyVoice3-0.5B shape, synthetic weights", "precision": "bf16"}
    print(json.dumps(info), flush=True)

    def kwargs(r, text):
        return dict(text=text, flow_embedding=r["flow_embedding"], llm_embedding=r["llm_embedding"], prompt_text=r["prompt_text"],
                    llm_prompt_speech_token=r["llm_prompt_speech_token"], flow_prompt_speech_token=r["flow_prompt_speech_token"],
                    prompt_speech_feat=r["prompt_speech_feat"])

    def threaded(reqs):
        out = [None] * len(reqs)

        def one(i):
            t0, first, lens = time.perf_counter(), None, []
            for o in model.tts(**kwargs(reqs[i], iter(reqs[i]["text_chunks"])), stream=True):
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

    def batched(gen_fn, reqs):
        model.token_hop_len = 25                    # the threaded arm leaves it at 100; the batched arms never change it
        t0 = time.perf_counter()
        first, lens = [None] * len(reqs), [[] for _ in reqs]
        for i, o in gen_fn(reqs):
            first[i] = first[i] if first[i] is not None else time.perf_counter() - t0
            lens[i].append(o["tts_speech"].shape[1])
        return list(zip(first, lens))

    arms = {
        "bistream_batch": lambda reqs: batched(lambda rs: model.tts_bistream_batch([kwargs(r, iter(r["text_chunks"])) for r in rs]), reqs),
        "threads": threaded,
        "stream_batch": lambda reqs: batched(lambda rs: model.tts_stream_batch([kwargs(r, r["text"]) for r in rs]), reqs),
    }
    for B in args.batches:
        reqs = [synth.cv3_bistream_request(i, n_text) for i in range(B)]
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
        line = {"batch": B, "card": card(), "slots": model.stream_slots,
                "slot_pool_bytes": model.ctx.flow_stream_bytes(model._slot_pool) if model._slot_pool else 0,
                "same_chunk_lengths_threads_vs_bistream_batch": res["threads"]["lens"] == res["bistream_batch"]["lens"],
                "same_samples_per_request_threads_vs_bistream_batch":
                    [sum(x) for x in res["threads"]["lens"]] == [sum(x) for x in res["bistream_batch"]["lens"]],
                "request0_chunk_lengths": {k: r["lens"][0] for k, r in res.items()},
                "request0_ids": {k: sum(r["lens"][0]) // 960 for k, r in res.items()}}
        for name, r in res.items():
            fs = sorted(r["first"])
            line[name] = {"audio_s_per_s": r["audio_s"] / r["wall_s"], "first_chunk_s": {"median": fs[len(fs) // 2], "max": fs[-1]},
                          "launches_per_run": r["launches"] // args.rounds}
        print(json.dumps(line), flush=True)

    # one mixed vocoder round against the two homogeneous calls it replaces: half the requests stream a chunk over 420 mel frames
    # of history, half finish over all 480
    B = max(args.batches)
    g = torch.Generator(device=dev).manual_seed(3)
    hist = [420] * (B // 2) + [480] * (B - B // 2)
    fin = [False] * (B // 2) + [True] * (B - B // 2)
    mel = torch.randn(sum(hist), 80, device=dev, generator=g) * 2 - 5
    n_st = sum(hist[:B // 2])

    def mixed():
        model.ctx.hift3_inference_rows(mel, hist, fin)

    def split():
        model.ctx.hift3_inference(mel[:n_st], hist[:B // 2], finalize=False)
        model.ctx.hift3_inference(mel[n_st:], hist[B // 2:], finalize=True)

    def timed(fn, reps=10):
        with torch.cuda.stream(model.stream):
            for _ in range(2):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                fn()
            e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / reps

    t = {"mixed": [], "split": []}
    for _ in range(3):
        t["mixed"].append(timed(mixed))
        t["split"].append(timed(split))
    print(json.dumps({"vocoder_round": {"card": card(), "utterances": B, "frames": hist, "finalize": fin,
                                        "mixed_call_ms": sorted(t["mixed"]), "two_calls_ms": sorted(t["split"])}}), flush=True)


if __name__ == "__main__":
    main()
