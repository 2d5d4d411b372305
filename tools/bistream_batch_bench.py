"""Batched text-streaming synthesis vs one thread per request, full-size models (synthetic weights), bf16.

B concurrent text-streaming requests (the tts text arrives as a generator of 4 chunks; 12 prompt-text ids, 48 text ids, 75 prompt
speech tokens; the decode is capped at 5 speech ids per text id because synthetic weights never draw eos) in two arms, alternated in
one process after warm-up:
  (a) B threads, each calling tts(text=<generator>, stream=True) on the shared CosyVoice2 model;
  (b) one tts_bistream_batch over the B requests (one ragged LM session, multi-slot flow session).
Prints audio-s/s, first-chunk latency (median, max) and libcvk launches per arm.  Then the LM stage of config #4 alone, for the
CosyVoice3 LM at B = 8: B threads of lm_generate_bistream against one lm_generate_bistream_batch over the same chunks (ids/s and
time to first id).  The card's name, power limit and maximum SM clock are printed first.  Needs an H100; there is no CPU path.

    python tools/bistream_batch_bench.py [--batches 8 16] [--rounds 2] [--small]
"""
import argparse
import json
import os
import sys
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.stream_batch_bench import card  # noqa: E402


def alternate(arms, reqs, rounds, torch, ctx):
    """warm-up once per arm, then `rounds` timed runs of each arm alternated; each arm returns [(first_s, amount)] per request"""
    for f in arms.values():
        f(reqs)
    res = {k: {"amount": 0.0, "wall_s": 0.0, "first": [], "launches": 0} for k in arms}
    for _ in range(rounds):
        for name, f in arms.items():
            torch.cuda.synchronize()
            l0 = ctx.launch_count()
            t0 = time.perf_counter()
            out = f(reqs)
            torch.cuda.synchronize()
            r = res[name]
            r["wall_s"] += time.perf_counter() - t0
            r["launches"] += ctx.launch_count() - l0
            r["amount"] += sum(a for _, a in out)
            r["first"] += [f0 for f0, _ in out]
    return res


def summary(res, rounds, unit):
    line = {}
    for name, r in res.items():
        fs = sorted(r["first"])
        line[name] = {unit: r["amount"] / r["wall_s"], "first_s": {"median": fs[len(fs) // 2], "max": fs[-1]},
                      "launches_per_run": r["launches"] // rounds}
    return line


def threads(fn, n):
    out = [None] * n
    ts = [threading.Thread(target=lambda i=i: out.__setitem__(i, fn(i))) for i in range(n)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[8, 16])
    ap.add_argument("--rounds", type=int, default=2, help="timed runs of each arm (alternating)")
    ap.add_argument("--small", action="store_true", help="debug: 2-layer LM / reduced flow (NOT the measured configuration)")
    args = ap.parse_args()
    import torch
    from cosyvoice_b200 import synth
    from cosyvoice_b200.model import B200CosyVoice2Model
    from cosyvoice_b200.model3 import B200CosyVoice3Model
    assert torch.cuda.is_available(), "needs a CUDA device (H100); there is no CPU path"
    dev = torch.device("cuda", 0)
    print(json.dumps({"card": card(), "model": "small debug" if args.small else "full-size shapes, synthetic weights", "precision": "bf16"}),
          flush=True)
    n_text = 48

    def request(i):
        r = synth.cv3_bistream_request(i, n_text)
        r["prompt_text"][0, 5] = 0                  # CosyVoice2 prompt (no <|endofprompt|>)
        return r

    # ---- (a) / (b): synthesis, CosyVoice2
    nl, fcfg = (2, (2, 1, 2, 2)) if args.small else (24, (6, 4, 12, 4))
    model = B200CosyVoice2Model(precision="bf16", device=0, workspace_gb=10.0)
    model.load_state_dicts(*synth.cosyvoice2_state_dicts(dev, 1986, nl, fcfg))
    torch.cuda.empty_cache()
    model.bistream_max_tokens = 5 * n_text
    model.stream_cache_frames = 768
    model.stream_batch_slots = max(args.batches)
    keys = ("flow_embedding", "llm_embedding", "prompt_text", "llm_prompt_speech_token", "flow_prompt_speech_token", "prompt_speech_feat")

    def kwargs(r):
        return dict({k: r[k] for k in keys}, text=iter(r["text_chunks"]))

    def threaded(reqs):
        def one(i):
            t0, first, n = time.perf_counter(), None, 0
            for o in model.tts(**kwargs(reqs[i]), stream=True):
                first = first if first is not None else time.perf_counter() - t0
                n += o["tts_speech"].shape[1]
            model.token_hop_len = 25
            return first, n / 24000.0
        return threads(one, len(reqs))

    def batched(reqs):
        t0 = time.perf_counter()
        first, n = [None] * len(reqs), [0] * len(reqs)
        for i, o in model.tts_bistream_batch([kwargs(r) for r in reqs]):
            first[i] = first[i] if first[i] is not None else time.perf_counter() - t0
            n[i] += o["tts_speech"].shape[1]
        return [(f, k / 24000.0) for f, k in zip(first, n)]

    for B in args.batches:
        reqs = [request(i) for i in range(B)]
        res = alternate({"threads": threaded, "batched": batched}, reqs, args.rounds, torch, model.ctx)
        print(json.dumps(dict(batch=B, stage="tts_bistream", **summary(res, args.rounds, "audio_s_per_s"))), flush=True)
    del model
    torch.cuda.empty_cache()

    # ---- LM stage of config #4: CosyVoice3 LM, B = 8
    m3 = B200CosyVoice3Model(precision="bf16", device=0, workspace_gb=2.0)
    llm_sd, _, _ = synth.cosyvoice3_state_dicts(dev, 1986, 2 if args.small else 24, 2)
    m3.ctx.load_state_dict("llm", llm_sd, [2 if args.small else 24])
    del llm_sd
    torch.cuda.empty_cache()
    m3.bistream_max_tokens = 5 * n_text
    reqs = [synth.cv3_bistream_request(i, n_text) for i in range(8)]

    def lm_threads(reqs):
        def one(i):
            r = reqs[i]
            t0, first, n = time.perf_counter(), None, 0
            with m3._lm_stream() as st:
                for _ in m3.lm_generate_bistream(iter(r["text_chunks"]), r["prompt_text"], r["llm_prompt_speech_token"], stream=st):
                    first = first if first is not None else time.perf_counter() - t0
                    n += 1
            return first, n
        return threads(one, len(reqs))

    def lm_batched(reqs):
        t0 = time.perf_counter()
        first, n = [None] * len(reqs), [0] * len(reqs)
        with m3._lm_stream() as st:
            for i, _ in m3.lm_generate_bistream_batch([iter(r["text_chunks"]) for r in reqs], [r["prompt_text"] for r in reqs],
                                                      [r["llm_prompt_speech_token"] for r in reqs], stream=st):
                first[i] = first[i] if first[i] is not None else time.perf_counter() - t0
                n[i] += 1
        return list(zip(first, n))

    res = alternate({"threads": lm_threads, "batched": lm_batched}, reqs, args.rounds, torch, m3.ctx)
    print(json.dumps(dict(batch=8, stage="cosyvoice3_lm_bistream", **summary(res, args.rounds, "ids_per_s"))), flush=True)


if __name__ == "__main__":
    main()
