"""Continuous batching in front of ``tts_batch`` + the reference servers' wire format (SURVEY.md §8(f) rank 3).

The reference serves one request per thread: every FastAPI / gRPC handler calls ``cosyvoice.inference_*`` itself and streams
``(tts_speech.numpy() * 2**15).astype(np.int16).tobytes()`` back (runtime/python/fastapi/server.py:40-43,
runtime/python/grpc/server.py:62-64).  On a GPU of this class a single utterance leaves the GPU launch-bound, while the batched pipeline
(``B200CosyVoice2Model.tts_batch``) is what the headline metric measures - so the step after the hot path is a queue that turns
concurrent requests into ragged batches.  This module is that queue and nothing else: no HTTP / gRPC layer, no text
normalisation, no tokenizer (those stay with the reference's frontend and server code, which call ``submit`` instead of
``model.tts``).

Admission policy: a batch is closed when ``max_batch`` requests are waiting or ``max_wait_ms`` have passed since the first one
arrived.  Requests that were queued while the previous batch ran (a backlog) have already waited through that batch: the next batch
takes them at once, up to ``max_batch``, instead of holding a partial remainder for the wait budget.  Requests are never reordered
inside a batch (the model's RNG streams are consumed in input order, so a fixed arrival order gives fixed results).  One worker thread owns the model; ``tts_batch`` itself is ragged, so no padding or bucketing is
needed here.

Streaming requests (``submit_stream`` / ``submit_stream_pcm``) are served by ``tts_stream_batch``, which hands out every request's
chunks as they become ready.  A batch is either all streaming or all offline: it is the run of requests of the same kind at the
head of the queue, so it also closes early when a request of the other kind is waiting behind it, and no request is ever moved
ahead of an earlier one of the other kind.
"""
import queue
import threading
import time
from concurrent.futures import Future

import numpy as np


def pcm16(wave):
    """float waveform tensor / array in [-1, 1) -> little-endian int16 PCM bytes, the reference servers' wire format
    (runtime/python/fastapi/server.py:42: ``(i['tts_speech'].numpy() * (2 ** 15)).astype(np.int16).tobytes()``, same expression in
    grpc/server.py:64).  Like the reference there is no clipping: callers own the [-1, 1) range (the vocoder clamps to 0.99,
    hifigan/generator.py:566)."""
    a = wave.detach().cpu().numpy() if hasattr(wave, "detach") else np.asarray(wave)
    return (a * (2 ** 15)).astype(np.int16).tobytes()


def pcm16_decode(buf):
    """int16 PCM bytes -> float32 [1, N] in [-1, 1): how the gRPC server reads a prompt waveform from the request
    (runtime/python/grpc/server.py:45-46: ``np.frombuffer(..., dtype=np.int16)`` then ``.float() / (2 ** 15)``)."""
    import torch
    return torch.from_numpy(np.array(np.frombuffer(buf, dtype=np.int16))).unsqueeze(0).float() / (2 ** 15)


_END = object()


class _Failed:
    def __init__(self, exc):
        self.exc = exc


class ChunkStream:
    """Iterator over one streaming request's chunks, filled by the batcher's worker: yields each chunk as soon as it is produced,
    ends after the request's batch has produced its last chunk, and re-raises the batch's exception if the batch fails."""

    def __init__(self):
        self._q = queue.Queue()

    def __iter__(self):
        return self

    def __next__(self):
        item = self._q.get()
        if item is _END or isinstance(item, _Failed):
            self._q.put(item)                    # every later next() ends the same way
            if item is _END:
                raise StopIteration
            raise item.exc
        return item


class TtsBatcher:
    """``submit(**tts_kwargs)`` -> Future of the waveform ([1, N] float32 CPU tensor, what ``tts`` yields for stream=False);
    ``submit_pcm`` -> Future of the int16 PCM bytes.  ``submit_stream`` / ``submit_stream_pcm`` -> iterator over the request's
    chunks (what ``tts`` yields for stream=True: float [1, n] tensors, or their int16 PCM bytes).  ``tts_kwargs`` are the keyword
    arguments of ``CosyVoice2Model.tts`` that the batched pipeline consumes: text, prompt_text, llm_prompt_speech_token,
    flow_prompt_speech_token, prompt_speech_feat, flow_embedding."""

    def __init__(self, model, max_batch=32, max_wait_ms=10.0):
        assert max_batch >= 1
        self.model = model
        self.max_batch = int(max_batch)
        self.max_wait = float(max_wait_ms) / 1e3
        self._q = []                       # (request dict, Future, wants_pcm)
        self._cv = threading.Condition()
        self._closed = False
        self.batches = []                  # sizes of the batches run so far (observability / tests)
        self._worker = threading.Thread(target=self._run, name="cvk-batcher", daemon=True)
        self._worker.start()

    # ------------------------------------------------------------------ client side
    def submit(self, **request):
        return self._enqueue(request, False)

    def submit_pcm(self, **request):
        return self._enqueue(request, True)

    def submit_stream(self, **request):
        return self._enqueue(request, False, ChunkStream())

    def submit_stream_pcm(self, **request):
        return self._enqueue(request, True, ChunkStream())

    def _enqueue(self, request, pcm, stream=None):
        sink = stream if stream is not None else Future()
        with self._cv:
            if self._closed:
                raise RuntimeError("TtsBatcher is closed")
            self._q.append((request, sink, pcm, time.monotonic()))
            self._cv.notify_all()
        return sink

    def close(self, wait=True):
        """Stop admitting; requests already queued are still served."""
        with self._cv:
            self._closed = True
            self._cv.notify_all()
        if wait:
            self._worker.join()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # ------------------------------------------------------------------ worker
    def _take_batch(self):
        free_at = time.monotonic()         # the previous batch (if any) has just finished
        with self._cv:
            while not self._q and not self._closed:
                self._cv.wait()
            if not self._q:
                return None
            # a head queued while the previous batch ran is a backlog: no further wait for company
            deadline = self._q[0][3] + self.max_wait if self._q[0][3] >= free_at else free_at
            while self._run_length() < self.max_batch and self._run_length() == len(self._q) and not self._closed:
                left = deadline - time.monotonic()
                if left <= 0:
                    break
                self._cv.wait(left)
            n = min(self._run_length(), self.max_batch)
            batch, self._q = self._q[:n], self._q[n:]
            return batch

    def _run_length(self):
        """requests of the head's kind (streaming or offline) at the head of the queue"""
        kind = isinstance(self._q[0][1], ChunkStream)
        n = 1
        while n < len(self._q) and isinstance(self._q[n][1], ChunkStream) == kind:
            n += 1
        return n

    def _run(self):
        while True:
            batch = self._take_batch()
            if batch is None:
                return
            if isinstance(batch[0][1], ChunkStream):
                self.batches.append(len(batch))
                self._run_stream(batch)
                continue
            live = [b for b in batch if b[1].set_running_or_notify_cancel()]
            if not live:
                continue
            self.batches.append(len(live))
            try:
                waves = self.model.tts_batch([b[0] for b in live])
            except BaseException as e:          # the whole batch shares the failure (one launch sequence)
                for _, fut, _, _ in live:
                    fut.set_exception(e)
                continue
            for (_, fut, pcm, _), w in zip(live, waves):
                try:
                    fut.set_result(pcm16(w) if pcm else w)
                except BaseException as e:
                    fut.set_exception(e)

    def _run_stream(self, batch):
        try:
            for i, out in self.model.tts_stream_batch([b[0] for b in batch]):
                _, sink, pcm, _ = batch[i]
                w = out["tts_speech"]
                sink._q.put(pcm16(w) if pcm else w)
        except BaseException as e:              # the whole batch shares the failure (one launch sequence per stage)
            for _, sink, _, _ in batch:
                sink._q.put(_Failed(e))
            return
        for _, sink, _, _ in batch:
            sink._q.put(_END)
