"""ctypes binding of libcvk.so (include/cvk.h).  PyTorch is used only as the allocator / stream provider:
tensors are passed as raw device pointers + explicit shapes, nothing here computes.

There is no CPU or eager fallback: if the shared library or a CUDA device is missing every entry point raises.
"""
import ctypes
import os
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "lib", "libcvk.so")

PREC_FP32, PREC_BF16 = 0, 1
ACT = dict(none=0, gelu=1, silu=2, mish=3, elu=4, lrelu=5, snake=6, tanh=7, abs=8, gelu_tanh=9)
DTYPE = dict(fp32=0, bf16=1, fp16=2)       # CVK_DT_*

_lib = None
_lib_lock = threading.Lock()

_c_int_p = ctypes.POINTER(ctypes.c_int)
_vp = ctypes.c_void_p

# name -> (restype, argtypes); mirrors include/cvk.h one to one (tests/test_abi.py checks every symbol resolves)
SIGNATURES = {
    "cvk_create": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.POINTER(_vp)]),
    "cvk_destroy": (None, [_vp]),
    "cvk_last_error": (ctypes.c_char_p, [_vp]),
    "cvk_version": (ctypes.c_char_p, []),
    "cvk_launch_count": (ctypes.c_int64, [_vp]),
    "cvk_stream_create": (ctypes.c_int, [_vp, ctypes.POINTER(_vp)]),
    "cvk_stream_destroy": (None, [_vp, _vp]),
    "cvk_last_op_ms": (ctypes.c_double, [_vp]),
    "cvk_debug_read": (ctypes.c_int, [_vp, ctypes.POINTER(ctypes.c_longlong), ctypes.c_int]),
    "cvk_set_option": (ctypes.c_int, [_vp, ctypes.c_char_p, ctypes.c_int]),
    "cvk_profile": (ctypes.c_int, [_vp, ctypes.c_int]),
    "cvk_profile_read": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double),
                                        ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_int64)]),
    "cvk_set_tensor": (ctypes.c_int, [_vp, ctypes.c_char_p, _vp, ctypes.c_int, ctypes.POINTER(ctypes.c_int64), ctypes.c_int]),
    "cvk_finalize": (ctypes.c_int, [_vp, ctypes.c_char_p, _c_int_p, ctypes.c_int]),
    "cvk_op_conv1d": (ctypes.c_int, [_vp, _vp, _c_int_p, ctypes.c_int, ctypes.c_int, _vp, _vp, ctypes.c_int, ctypes.c_int,
                                     ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp, _vp]),
    "cvk_op_linear_small": (ctypes.c_int, [_vp, _vp, ctypes.c_int, ctypes.c_int, _vp, _vp, ctypes.c_int, _vp, ctypes.c_int,
                                           ctypes.POINTER(ctypes.c_float), _vp]),
    "cvk_op_attention": (ctypes.c_int, [_vp, _vp, _vp, _vp, _c_int_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, _vp, _vp]),
    "cvk_op_attention_ex": (ctypes.c_int, [_vp, _vp, _vp, _vp, _c_int_p, _c_int_p, _c_int_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_int, ctypes.c_float, _vp, _vp]),
    "cvk_op_decode_attention": (ctypes.c_int, [_vp, _vp, ctypes.c_int, ctypes.c_int, _vp, _vp, _vp, _c_int_p, ctypes.c_int, _vp, _vp]),
    "cvk_op_ragged_attention": (ctypes.c_int, [_vp, _vp, _vp, _vp, ctypes.c_int, ctypes.c_int, _c_int_p, ctypes.c_int, _vp, _vp]),
    "cvk_op_lm_decode_layers": (ctypes.c_int, [_vp, ctypes.c_int, _c_int_p, ctypes.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "cvk_op_conv_gemm": (ctypes.c_int, [_vp, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_int_p, _c_int_p, ctypes.c_int,
                                        _vp, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, _vp,
                                        _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                        ctypes.c_float, _vp, _vp, ctypes.c_int, ctypes.c_int, _vp]),
    "cvk_op_flow_ff": (ctypes.c_int, [_vp, _vp, ctypes.c_int, _c_int_p, _c_int_p, ctypes.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                      _vp, _vp, _vp, _vp, _vp]),
    "cvk_op_relpos_attention": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, ctypes.c_int, _vp, _vp, _c_int_p, ctypes.c_int, ctypes.c_int,
                                               ctypes.c_int, ctypes.c_float, _vp, _vp]),
    "cvk_hift_f0": (ctypes.c_int, [_vp, _vp, _c_int_p, ctypes.c_int, _vp, _vp]),
    "cvk_hift_source": (ctypes.c_int, [_vp, _vp, _c_int_p, ctypes.c_int, _vp, _vp, _vp]),
    "cvk_hift_decode": (ctypes.c_int, [_vp, _vp, _c_int_p, ctypes.c_int, _vp, _vp, _vp]),
    "cvk_hift_inference": (ctypes.c_int, [_vp, _vp, _c_int_p, ctypes.c_int, _vp, _vp, _c_int_p, _vp, _vp, _vp]),
    "cvk_flow_encoder": (ctypes.c_int, [_vp, _vp, _c_int_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp, _vp]),
    "cvk_cfm_estimator": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _c_int_p, ctypes.c_int, ctypes.c_int, _vp, _vp]),
    "cvk_flow_encoder_hidden": (ctypes.c_int, [_vp, _vp, _c_int_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp, _vp]),
    "cvk_cfm_estimator_hidden": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _c_int_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp, _vp]),
    "cvk_cfm_estimator_inplace": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _c_int_p, ctypes.c_int, ctypes.c_int, _vp]),
    "cvk_workspace_bytes": (ctypes.c_int, [_vp, ctypes.POINTER(ctypes.c_size_t), ctypes.POINTER(ctypes.c_size_t)]),
    "cvk_cfm_solve": (ctypes.c_int, [_vp, _vp, _vp, _vp, _c_int_p, ctypes.c_int, _vp, ctypes.c_int, ctypes.c_float, ctypes.c_int, _vp, _vp]),
    "cvk_flow_inference": (ctypes.c_int, [_vp, _vp, _c_int_p, _vp, _c_int_p, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp, _vp]),
    "cvk_flow_stream_create": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.POINTER(_vp)]),
    "cvk_flow3_stream_create": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.POINTER(_vp)]),
    "cvk_flow_stream_destroy": (None, [_vp, _vp]),
    "cvk_flow_stream_bytes": (ctypes.c_longlong, [_vp]),
    "cvk_flow_stream_begin": (ctypes.c_int, [_vp, _vp, _vp, ctypes.c_int, _vp, _vp]),
    "cvk_flow_stream_chunk": (ctypes.c_int, [_vp, _vp, _vp, ctypes.c_int, _vp, ctypes.c_int, _c_int_p, _vp]),
    "cvk_flow_stream_create_slots": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(_vp)]),
    "cvk_flow_stream_begin_slot": (ctypes.c_int, [_vp, _vp, ctypes.c_int, _vp, ctypes.c_int, _vp, _vp]),
    "cvk_flow_stream_chunk_batch": (ctypes.c_int, [_vp, _vp, ctypes.c_int, _c_int_p, _vp, _c_int_p, _vp, ctypes.c_int, _c_int_p, _vp]),
    "cvk_cfm_set_noise": (ctypes.c_int, [_vp, _vp, ctypes.c_int, ctypes.c_int]),
    "cvk_hift3_set_noise": (ctypes.c_int, [_vp, _vp, _vp, ctypes.c_longlong, ctypes.c_int]),
    "cvk_hift3_inference": (ctypes.c_int, [_vp, _vp, _c_int_p, ctypes.c_int, ctypes.c_int, _vp, _vp, _vp, _vp]),
    "cvk_hift3_inference_rows": (ctypes.c_int, [_vp, _vp, _c_int_p, _c_int_p, ctypes.c_int, _vp, _vp, _vp, _vp]),
    "cvk_dit_estimator": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _c_int_p, ctypes.c_int, ctypes.c_int, _vp, _vp]),
    "cvk_hift_hidden": (ctypes.c_int, [_vp, ctypes.c_int, _vp, _c_int_p, _c_int_p, ctypes.c_int, _vp, ctypes.c_int, _vp, _vp]),
    "cvk_dit_hidden": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _c_int_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp, _vp]),
    "cvk_flow3_inference": (ctypes.c_int, [_vp, _vp, _c_int_p, _vp, _c_int_p, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp, _vp]),
    "cvk_lm_session_create": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.POINTER(_vp)]),
    "cvk_lm_session_destroy": (None, [_vp, _vp]),
    "cvk_lm_prefill": (ctypes.c_int, [_vp, _vp, _vp, _c_int_p, _vp, _c_int_p, ctypes.c_int, _vp]),
    "cvk_lm_decode": (ctypes.c_int, [_vp, _vp, ctypes.c_int, _vp, _vp, _vp, _vp, ctypes.c_int, _vp, _vp, _c_int_p, _vp]),
    "cvk_lm_forward_logp": (ctypes.c_int, [_vp, _vp, _c_int_p, ctypes.c_int, _vp, _vp]),
    "cvk_lm_last_logits": (ctypes.c_int, [_vp, _vp, _vp, _vp]),
    "cvk_lm_vocab": (ctypes.c_int, [_vp]),
    "cvk_lm_begin": (ctypes.c_int, [_vp, _vp, ctypes.c_int, _vp]),
    "cvk_lm_feed": (ctypes.c_int, [_vp, _vp, _c_int_p, _c_int_p, ctypes.c_int, _vp]),
    "cvk_lm_next_logp": (ctypes.c_int, [_vp, _vp, _vp, _vp]),
    "cvk_lm_feed_rows": (ctypes.c_int, [_vp, _vp, ctypes.c_int, _c_int_p, _c_int_p, _c_int_p, _c_int_p, _vp]),
    "cvk_lm_next_logp_rows": (ctypes.c_int, [_vp, _vp, ctypes.c_int, _c_int_p, _vp, _vp]),
    "cvk_ras_sample": (ctypes.c_int, [_vp, _vp, ctypes.c_int, ctypes.c_int, _vp, ctypes.c_int, _vp, _vp, _vp, _vp, _vp]),
    "cvk_op_sample_step": (ctypes.c_int, [_vp, _vp, ctypes.c_int, ctypes.c_int, _vp, ctypes.c_int, _vp, _vp, _vp, ctypes.c_int, _vp, _vp,
                                          _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "cvk_op_log_softmax": (ctypes.c_int, [_vp, _vp, ctypes.c_int, ctypes.c_int, _vp]),
    "cvk_mel_spectrogram": (ctypes.c_int, [_vp, _vp, _c_int_p, ctypes.c_int, _vp, _vp]),
    "cvk_mel_spectrogram_ex": (ctypes.c_int, [_vp, _vp, _c_int_p, ctypes.c_int, ctypes.c_int, _vp, _vp]),
    "cvk_mel_resample": (ctypes.c_int, [_vp, _vp, _c_int_p, _c_int_p, ctypes.c_int, _vp, _vp]),
    "cvk_whisper_log_mel": (ctypes.c_int, [_vp, _vp, _c_int_p, ctypes.c_int, _vp, _vp]),
    "cvk_kaldi_fbank": (ctypes.c_int, [_vp, _vp, _c_int_p, ctypes.c_int, ctypes.c_int, _vp, _vp]),
}


def lib_path():
    return _LIB_PATH


def load_library():
    """dlopen libcvk.so and bind every symbol of include/cvk.h.  Raises if the library has not been built."""
    global _lib
    with _lib_lock:
        if _lib is None:
            if not os.path.exists(_LIB_PATH):
                raise RuntimeError(f"{_LIB_PATH} not found - run `python -m cosyvoice_b200.build` (needs nvcc); "
                                   "there is no CPU fallback")
            lib = ctypes.CDLL(_LIB_PATH)
            for name, (res, args) in SIGNATURES.items():
                fn = getattr(lib, name)
                fn.restype = res
                fn.argtypes = args
            _lib = lib
    return _lib


def _ints(v):
    v = [int(x) for x in v]
    return (ctypes.c_int * len(v))(*v)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _f32(t, device):
    return t.to(device=device, dtype=torch.float32).contiguous()


class CvkError(RuntimeError):
    pass


class Context:
    """One cvk_ctx per (process, GPU)."""

    def __init__(self, device=0, precision="bf16", workspace_gb=4.0):
        if not torch.cuda.is_available():
            raise RuntimeError("cosyvoice_b200 requires a CUDA device (sm_90a); there is no CPU fallback")
        self.lib = load_library()
        self.device = torch.device("cuda", device)
        self.precision = PREC_BF16 if precision in ("bf16", PREC_BF16) else PREC_FP32
        h = ctypes.c_void_p()
        torch.cuda.set_device(self.device)
        torch.zeros(1, device=self.device)           # make sure the primary context exists
        rc = self.lib.cvk_create(device, self.precision, int(workspace_gb * (1 << 30)), ctypes.byref(h))
        if rc != 0:
            raise CvkError(f"cvk_create failed with status {rc} (needs an sm_90 GPU: H100)")
        self.h = h
        self.lock = threading.Lock()

    def close(self):
        if getattr(self, "h", None):
            self.lib.cvk_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            msg = self.lib.cvk_last_error(self.h)
            raise CvkError(f"libcvk status {rc}: {msg.decode() if msg else ''}")

    # ------------------------------------------------------------------ weights
    def load_state_dict(self, stage, state_dict, cfg=()):
        """Hand a reference state_dict (fp32) to the library and finalise the stage."""
        torch.cuda.synchronize(self.device)
        for k, v in state_dict.items():
            if not torch.is_tensor(v) or not v.dtype.is_floating_point:
                continue
            if stage == "llm" and k == "llm.model.lm_head.weight":
                continue      # tied alias of embed_tokens, never used at inference (llm/llm.py:542 uses llm_decoder)
            t = v.detach().to(dtype=torch.float32).contiguous()
            on_dev = 1 if t.is_cuda else 0
            shape = (ctypes.c_int64 * max(t.dim(), 1))(*(list(t.shape) or [1]))
            self._check(self.lib.cvk_set_tensor(self.h, f"{stage}.{k}".encode(), _ptr(t), on_dev, shape, max(t.dim(), 1)))
        self.finalize(stage, cfg)

    def finalize(self, stage, cfg=()):
        cfg = list(cfg)
        self._check(self.lib.cvk_finalize(self.h, stage.encode(), _ints(cfg) if cfg else None, len(cfg)))

    def set_option(self, key, value):
        self._check(self.lib.cvk_set_option(self.h, key.encode(), int(value)))

    def profile(self, enable):
        self._check(self.lib.cvk_profile(self.h, int(enable)))

    def profile_read(self, family):
        ms, fl, by, n = ctypes.c_double(), ctypes.c_double(), ctypes.c_double(), ctypes.c_int64()
        self._check(self.lib.cvk_profile_read(self.h, family, ctypes.byref(ms), ctypes.byref(fl), ctypes.byref(by), ctypes.byref(n)))
        return dict(ms=ms.value, flops=fl.value, bytes=by.value, launches=n.value)

    def debug_read(self, n=4096):
        buf = (ctypes.c_longlong * n)()
        self._check(self.lib.cvk_debug_read(self.h, buf, n))
        return list(buf)

    def last_op_ms(self):
        return float(self.lib.cvk_last_op_ms(self.h))

    def stream_create(self):
        """a non-blocking CUDA stream owned by the caller (cvk_stream_create), as a torch ExternalStream; give it back with
        stream_destroy"""
        s = ctypes.c_void_p()
        self._check(self.lib.cvk_stream_create(self.h, ctypes.byref(s)))
        return torch.cuda.ExternalStream(s.value, device=self.device)

    def stream_destroy(self, stream):
        self.lib.cvk_stream_destroy(self.h, ctypes.c_void_p(stream.cuda_stream))

    def launch_count(self):
        return int(self.lib.cvk_launch_count(self.h))

    # ------------------------------------------------------------------ generic ops (tests)
    def conv1d(self, x, lens, w, bias, dil=1, shift0=0, act="none"):
        """x [sum(lens), K] time-major; w torch Conv1d weight [N,K,taps]."""
        x = _f32(x, self.device)
        w = _f32(w, self.device)
        b = _f32(bias, self.device) if bias is not None else None
        N, K, taps = w.shape
        out = torch.empty(x.shape[0], N, device=self.device)
        self._check(self.lib.cvk_op_conv1d(self.h, _ptr(x), _ints(lens), len(lens), K, _ptr(w), _ptr(b), N, taps, dil, shift0,
                                           ACT[act], _ptr(out), _stream()))
        return out

    def linear_small(self, x, w, bias=None, iters=0):
        x, w = _f32(x, self.device), _f32(w, self.device)
        b = _f32(bias, self.device) if bias is not None else None
        out = torch.empty(x.shape[0], w.shape[0], device=self.device)
        ms = ctypes.c_float(0)
        self._check(self.lib.cvk_op_linear_small(self.h, _ptr(x), x.shape[0], x.shape[1], _ptr(w), _ptr(b), w.shape[0], _ptr(out), iters,
                                                 ctypes.byref(ms), _stream()))
        return out, ms.value

    def attention(self, q, k, v, lens, heads, chunk=0, scale=0.125):
        q, k, v = (_f32(t, self.device) for t in (q, k, v))
        out = torch.empty_like(q)
        self._check(self.lib.cvk_op_attention(self.h, _ptr(q), _ptr(k), _ptr(v), _ints(lens), len(lens), heads, chunk, scale,
                                              _ptr(out), _stream()))
        return out

    def attention_ex(self, q, k, v, q_lens, k_lens, q_offset, heads, kv_heads, chunk=0, scale=0.125):
        """q [sum q_lens, heads*64], k / v [sum k_lens, kv_heads*64]; query i of sequence b at position q_offset[b] + i"""
        q, k, v = (_f32(t, self.device) for t in (q, k, v))
        out = torch.empty_like(q)
        self._check(self.lib.cvk_op_attention_ex(self.h, _ptr(q), _ptr(k), _ptr(v), _ints(q_lens), _ints(k_lens), _ints(q_offset),
                                                 len(q_lens), heads, kv_heads, chunk, scale, _ptr(out), _stream()))
        return out

    def decode_attention(self, partial, bias, k_cache, v_cache, ctx_len):
        """one LM decode-attention step: partial [splits, rows, 1152], bias [1152], caches [rows, 2, max_ctx, 64] (copies are
        returned with the new row appended), ctx_len [rows] (python ints).  Returns (out [rows, 896], k_cache, v_cache)."""
        partial, bias = _f32(partial, self.device), _f32(bias, self.device)
        k_cache, v_cache = _f32(k_cache, self.device).clone(), _f32(v_cache, self.device).clone()
        splits, rows = partial.shape[0], partial.shape[1]
        out = torch.empty(rows, 896, device=self.device)
        self._check(self.lib.cvk_op_decode_attention(self.h, _ptr(partial), splits, rows, _ptr(bias), _ptr(k_cache), _ptr(v_cache),
                                                     _ints(ctx_len), k_cache.shape[2], _ptr(out), _stream()))
        return out, k_cache, v_cache

    def lm_decode_layers(self, x, k_cache, v_cache, ctx_len):
        """every layer of the loaded LM for one decode step (cvk_op_lm_decode_layers): x [B, 896] residual stream, caches
        [layers, B, 2, max_ctx, 64], ctx_len [B] (python ints, the new row's position).  Returns copies (x, k_cache, v_cache) updated
        by the step and (xn [B, 896], att [B, 896], ffa [B, 4864]): the final-normed row and the last layer's o_proj / down_proj
        operands."""
        x = _f32(x, self.device).clone()
        k_cache, v_cache = _f32(k_cache, self.device).clone(), _f32(v_cache, self.device).clone()
        B = x.shape[0]
        xn = torch.empty(B, 896, device=self.device)
        att = torch.empty(B, 896, device=self.device)
        ffa = torch.empty(B, 4864, device=self.device)
        self._check(self.lib.cvk_op_lm_decode_layers(self.h, B, _ints(ctx_len), k_cache.shape[3], _ptr(x), _ptr(k_cache), _ptr(v_cache),
                                                     _ptr(xn), _ptr(att), _ptr(ffa), _stream()))
        return x, k_cache, v_cache, (xn, att, ffa)

    def ragged_attention(self, q, k_cache, v_cache, rowpos):
        """the feed attention of cvk_lm_feed_rows (cvk_op_ragged_attention): q [M, 896], caches [rows, 2, max_ctx, 64], rowpos: M python
        (cache row, position) pairs.  Returns out [M, 896]."""
        q, k_cache, v_cache = _f32(q, self.device), _f32(k_cache, self.device), _f32(v_cache, self.device)
        assert len(rowpos) == q.shape[0] and k_cache.shape == v_cache.shape
        out = torch.empty(q.shape[0], 896, device=self.device)
        self._check(self.lib.cvk_op_ragged_attention(self.h, _ptr(q), _ptr(k_cache), _ptr(v_cache), k_cache.shape[0], k_cache.shape[2],
                                                     _ints([v for rp in rowpos for v in rp]), len(rowpos), _ptr(out), _stream()))
        return out

    def conv_gemm(self, x, seq_start, seq_len, w, bias=None, dil=1, shift0=0, operand="fp32", act1="none", act1_param=0.0, alpha1=None,
                  resid=None, resid_is_out=False, accumulate=False, out=None, out_dtype="fp32", act2="none", act2_param=0.0, alpha2=None,
                  out2=None, out2_dtype="fp32"):
        """One conv-GEMM launch with the stage epilogue on packed matrices (cvk_op_conv_gemm): x [rows, x_ld] (columns >= K =
        w.shape[1] are never read), w a torch Conv1d weight [N,K,taps], sequences b at rows [seq_start[b], + seq_len[b]).  out / out2:
        fp32 [rows, ld] initial contents (out required, out2 None for no second output); returns the updated (out, out2) copies."""
        x, w = _f32(x, self.device), _f32(w, self.device)
        b, a1, a2, r = (_f32(t, self.device) if t is not None else None for t in (bias, alpha1, alpha2, resid))
        out = _f32(out, self.device).clone()
        out2 = _f32(out2, self.device).clone() if out2 is not None else None
        N, K, taps = w.shape
        self._check(self.lib.cvk_op_conv_gemm(
            self.h, _ptr(x), x.shape[0], K, x.shape[1], DTYPE[operand], _ints(seq_start), _ints(seq_len), len(seq_len), _ptr(w), _ptr(b),
            N, taps, dil, shift0, ACT[act1], act1_param, _ptr(a1), _ptr(r), r.shape[1] if r is not None else 0, int(resid_is_out),
            int(accumulate), _ptr(out), DTYPE[out_dtype], out.shape[1], ACT[act2], act2_param, _ptr(a2), _ptr(out2), DTYPE[out2_dtype],
            out2.shape[1] if out2 is not None else 0, _stream()))
        return out, out2

    def flow_ff(self, x, seq_start, seq_len, ln3_g, ln3_b, w1, b1, w2, b2, ln_g=None, ln_b=None, att=None, wo=None, bo=None):
        """the feed-forward half of a flow-estimator transformer block (cvk_op_flow_ff): x [rows, 256]; w1 [1024, 256], w2 [256, 1024]
        torch Linear weights; with att [rows, 512], wo [256, 512] and bo [256] the block's attention output projection and its residual
        come first.  Returns (new x, out): out = the next block's LN1 (ln_g, ln_b) of the new x, or the new x itself, both as rounded to
        the activation dtype."""
        x = _f32(x, self.device).clone()
        t = [_f32(v, self.device) if v is not None else None for v in (ln3_g, ln3_b, w1, b1, w2, b2, ln_g, ln_b, att, wo, bo)]
        out = torch.empty_like(x)
        self._check(self.lib.cvk_op_flow_ff(self.h, _ptr(x), x.shape[0], _ints(seq_start), _ints(seq_len), len(seq_len), *(_ptr(v) for v in t),
                                            _ptr(out), _stream()))
        return x, out

    def relpos_attention(self, q, k, v, pos, center, bias_u, bias_v, lens, heads, chunk=0, scale=0.125):
        """conformer relative-position attention (cvk_op_relpos_attention): q, k, v [sum lens, heads*64], pos [2*center+1, heads*64]
        (row t: relative position center - t), bias_u / bias_v [heads*64]"""
        q, k, v, pos, bu, bv = (_f32(t, self.device) for t in (q, k, v, pos, bias_u, bias_v))
        out = torch.empty_like(q)
        self._check(self.lib.cvk_op_relpos_attention(self.h, _ptr(q), _ptr(k), _ptr(v), _ptr(pos), int(center), _ptr(bu), _ptr(bv),
                                                     _ints(lens), len(lens), heads, chunk, scale, _ptr(out), _stream()))
        return out

    # ------------------------------------------------------------------ HiFT
    def hift_f0(self, mel, lens):
        mel = _f32(mel, self.device)
        f0 = torch.empty(mel.shape[0], device=self.device)
        self._check(self.lib.cvk_hift_f0(self.h, _ptr(mel), _ints(lens), len(lens), _ptr(f0), _stream()))
        return f0

    def hift_source(self, f0, lens, noise):
        f0, noise = _f32(f0, self.device), _f32(noise, self.device)
        src = torch.empty(f0.shape[0] * 480, device=self.device)
        self._check(self.lib.cvk_hift_source(self.h, _ptr(f0), _ints(lens), len(lens), _ptr(noise), _ptr(src), _stream()))
        return src

    def hift_decode(self, mel, lens, source):
        mel, source = _f32(mel, self.device), _f32(source, self.device)
        wav = torch.empty(mel.shape[0] * 480, device=self.device)
        self._check(self.lib.cvk_hift_decode(self.h, _ptr(mel), _ints(lens), len(lens), _ptr(source), _ptr(wav), _stream()))
        return wav

    def hift_inference(self, mel, lens, noise, cache_source=None, cache_lens=None):
        mel, noise = _f32(mel, self.device), _f32(noise, self.device)
        wav = torch.empty(mel.shape[0] * 480, device=self.device)
        src = torch.empty(mel.shape[0] * 480, device=self.device)
        cs = _f32(cache_source, self.device) if cache_source is not None else None
        cl = _ints(cache_lens) if cache_lens is not None else None
        self._check(self.lib.cvk_hift_inference(self.h, _ptr(mel), _ints(lens), len(lens), _ptr(noise), _ptr(cs), cl, _ptr(wav),
                                                _ptr(src), _stream()))
        return wav, src

    def hift_hidden(self, mel, lens, unit, source=None, causal=False, finalize=None):
        """parity tests: read-out `unit` (0 .. 20) of the vocoder body, sequence rows only, as fp32.  causal=False: stage "hift" on the
        given source [sum 480 T] (as hift_decode); causal=True: stage "hift3" on its own f0 and source (as hift3_inference_rows, every
        utterance final when finalize is None).  With Tb the body frames (T, or T - 7 for a streaming utterance): unit 0 the source
        STFT [sum 120 Tb + 1, 18], 1 conv_pre [sum Tb, 512], 2 + 6i .. 7 + 6i level i (up-sampled, + source branch, after each of the
        three resblocks, level output) with [8 Tb, 40 Tb, 120 Tb + 1][i] rows and [256, 128, 64][i] channels, 20 conv_post
        [sum 120 Tb + 1, 18]"""
        mel = _f32(mel, self.device)
        fin = [True] * len(lens) if finalize is None else [bool(f) for f in finalize]
        tb = [int(l) - (0 if f or not causal else 7) for l, f in zip(lens, fin)]
        if unit == 1:
            rows, cols = sum(tb), 512
        elif 2 <= unit <= 19:
            i = (unit - 2) // 6
            rows, cols = sum([8 * t, 40 * t, 120 * t + 1][i] for t in tb), [256, 128, 64][i]
        else:
            rows, cols = sum(120 * t + 1 for t in tb), 18
        out = torch.empty(max(rows, 1), cols, device=self.device)
        src = _f32(source, self.device) if source is not None else None
        fl = _ints([int(f) for f in fin]) if finalize is not None else None
        self._check(self.lib.cvk_hift_hidden(self.h, int(causal), _ptr(mel), _ints(lens), fl, len(lens), _ptr(src), int(unit), _ptr(out),
                                             _stream()))
        return out[:rows]

    # ------------------------------------------------------------------ flow
    def set_cfm_noise(self, noise_tm):
        noise_tm = _f32(noise_tm, self.device)
        self._check(self.lib.cvk_cfm_set_noise(self.h, _ptr(noise_tm), noise_tm.shape[0], 1))

    def flow_encoder(self, tokens, lens, streaming=False, context_len=0):
        tokens = tokens.to(device=self.device, dtype=torch.int32).contiguous()
        rows = sum(2 * (int(l) - context_len) for l in lens)
        h = torch.empty(rows, 512, device=self.device)
        self._check(self.lib.cvk_flow_encoder(self.h, _ptr(tokens), _ints(lens), len(lens), int(streaming), context_len, _ptr(h), _stream()))
        return h

    def flow_encoder_hidden(self, tokens, lens, n_layers, enc_blocks, streaming=False, context_len=0):
        """parity tests: the encoder's fp32 residual stream after n_layers units (0: embedding + PreLookahead, then one per
        conformer layer, enc_blocks + 1: up_layer + up_embed, then one per up layer); [sum T - context_len, 512] up to enc_blocks
        (the loaded model's), [sum 2 (T - context_len), 512] after; same inputs as flow_encoder"""
        tokens = tokens.to(device=self.device, dtype=torch.int32).contiguous()
        rate = 1 if n_layers <= enc_blocks else 2
        h = torch.empty(max(1, sum(rate * (int(l) - context_len) for l in lens)), 512, device=self.device)
        self._check(self.lib.cvk_flow_encoder_hidden(self.h, _ptr(tokens), _ints(lens), len(lens), int(streaming), context_len,
                                                     int(n_layers), _ptr(h), _stream()))
        return h

    def cfm_estimator_hidden(self, x, mu, t, spks, cond, lens, n_units, streaming=False):
        """parity tests: the estimator's fp32 residual stream [sum T, 256] after n_units units (a stage's resnet or one of its
        transformer blocks, in execution order; 1 <= n_units <= n_stages * (1 + n_blocks)); same inputs as cfm_estimator"""
        x, mu, t, spks, cond = (_f32(a, self.device) for a in (x, mu, t, spks, cond))
        out = torch.empty(x.shape[0], 256, device=self.device)
        self._check(self.lib.cvk_cfm_estimator_hidden(self.h, _ptr(x), _ptr(mu), _ptr(t), _ptr(spks), _ptr(cond), _ints(lens),
                                                      len(lens), int(streaming), int(n_units), _ptr(out), _stream()))
        return out

    def cfm_estimator(self, x, mu, t, spks, cond, lens, streaming=False):
        x, mu, t, spks, cond = (_f32(a, self.device) for a in (x, mu, t, spks, cond))
        out = torch.empty_like(x)
        self._check(self.lib.cvk_cfm_estimator(self.h, _ptr(x), _ptr(mu), _ptr(t), _ptr(spks), _ptr(cond), _ints(lens), len(lens),
                                               int(streaming), _ptr(out), _stream()))
        return out

    def cfm_estimator_inplace(self, x, mu, t, spks, cond, lens, streaming=False):
        """the TensorRT engine contract (flow_matching.py:140-148): x [sum T, 80] float32 on the device is overwritten"""
        assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()
        mu, t, spks, cond = (_f32(a, self.device) for a in (mu, t, spks, cond))
        self._check(self.lib.cvk_cfm_estimator_inplace(self.h, _ptr(x), _ptr(mu), _ptr(t), _ptr(spks), _ptr(cond), _ints(lens), len(lens),
                                                       int(streaming), _stream()))
        return x

    def workspace_bytes(self):
        cap, high = ctypes.c_size_t(), ctypes.c_size_t()
        self._check(self.lib.cvk_workspace_bytes(self.h, ctypes.byref(cap), ctypes.byref(high)))
        return cap.value, high.value

    def hift3_set_noise(self, rand_ini, sine_noise):
        """CosyVoice3 vocoder: SineGen2.rand_ini [9] and SineGen2.sine_waves [n,9] (module attributes of the reference)"""
        rand_ini = _f32(rand_ini.reshape(-1), self.device)
        sine_noise = _f32(sine_noise.reshape(-1, 9), self.device)
        self._check(self.lib.cvk_hift3_set_noise(self.h, _ptr(rand_ini), _ptr(sine_noise), sine_noise.shape[0], 1))

    def hift3_inference(self, mel, lens, finalize=True):
        """CausalHiFTGenerator.inference: mel [sum T, 80] -> (wav [sum 480 T], f0 [sum T], source [sum 480 T]); with finalize=False
        (streaming call) wav [sum 480 (T-8)], f0 [sum T-3], source [sum 480 (T-3)]"""
        mel = _f32(mel, self.device)
        # streaming call (finalize=False): 3 frames of f0 look-ahead, 4 of conv_pre look-ahead, the last frame's samples dropped
        n_src = sum(int(l) - (0 if finalize else 3) for l in lens)
        n_out = sum(int(l) - (0 if finalize else 8) for l in lens)
        wav = torch.empty(n_out * 480, device=self.device)
        f0 = torch.empty(n_src, device=self.device)
        src = torch.empty(n_src * 480, device=self.device)
        self._check(self.lib.cvk_hift3_inference(self.h, _ptr(mel), _ints(lens), len(lens), int(finalize), _ptr(wav), _ptr(f0), _ptr(src),
                                                 _stream()))
        return wav, f0, src

    def hift3_inference_rows(self, mel, lens, finalize):
        """hift3_inference with a finalize flag per utterance: mel [sum T, 80] -> (wav, f0, src), utterance b's parts back to back,
        480 T / T / 480 T samples when finalize[b] and 480 (T-8) / T-3 / 480 (T-3) when not (streaming, T >= 9).  Each utterance
        gets exactly what hift3_inference gives it alone with its own flag; one launch sequence serves the whole call."""
        if len(finalize) != len(lens):
            raise ValueError("hift3_inference_rows: one finalize flag per utterance")
        mel = _f32(mel, self.device)
        fin = [bool(f) for f in finalize]
        n_src = sum(int(l) - (0 if f else 3) for l, f in zip(lens, fin))
        n_out = sum(int(l) - (0 if f else 8) for l, f in zip(lens, fin))
        wav = torch.empty(max(n_out, 0) * 480, device=self.device)
        f0 = torch.empty(max(n_src, 0), device=self.device)
        src = torch.empty(max(n_src, 0) * 480, device=self.device)
        self._check(self.lib.cvk_hift3_inference_rows(self.h, _ptr(mel), _ints(lens), _ints([int(f) for f in fin]), len(lens), _ptr(wav),
                                                      _ptr(f0), _ptr(src), _stream()))
        return wav, f0, src

    def dit_estimator(self, x, mu, t, spks, cond, lens, streaming=False):
        """CosyVoice3 DiT estimator (stage "flow3"); same layout as cfm_estimator."""
        x, mu, t, spks, cond = (_f32(a, self.device) for a in (x, mu, t, spks, cond))
        out = torch.empty_like(x)
        self._check(self.lib.cvk_dit_estimator(self.h, _ptr(x), _ptr(mu), _ptr(t), _ptr(spks), _ptr(cond), _ints(lens), len(lens),
                                               int(streaming), _ptr(out), _stream()))
        return out

    def dit_hidden(self, x, mu, t, spks, cond, lens, n_blocks, streaming=False):
        """parity tests: the DiT residual stream [sum T, 1024] after the input embedding and the first n_blocks blocks (0 <= n_blocks
        <= depth); same inputs as dit_estimator"""
        x, mu, t, spks, cond = (_f32(a, self.device) for a in (x, mu, t, spks, cond))
        out = torch.empty(x.shape[0], 1024, device=self.device)
        self._check(self.lib.cvk_dit_hidden(self.h, _ptr(x), _ptr(mu), _ptr(t), _ptr(spks), _ptr(cond), _ints(lens), len(lens),
                                            int(streaming), int(n_blocks), _ptr(out), _stream()))
        return out

    def flow3_inference(self, tokens, token_lens, prompt_feat, prompt_feat_lens, embedding, n_timesteps=10, streaming=False,
                        finalize=True):
        """CosyVoice3 flow (CausalMaskedDiffWithDiT.inference); same layout as flow_inference."""
        tokens = tokens.to(device=self.device, dtype=torch.int32).contiguous()
        prompt_feat = _f32(prompt_feat, self.device) if prompt_feat is not None and prompt_feat.numel() else None
        embedding = _f32(embedding, self.device)
        ctxl = 0 if finalize else 3
        out_lens = [2 * (int(n) - ctxl) - int(p) for n, p in zip(token_lens, prompt_feat_lens)]
        mel = torch.empty(sum(out_lens), 80, device=self.device)
        self._check(self.lib.cvk_flow3_inference(self.h, _ptr(tokens), _ints(token_lens), _ptr(prompt_feat), _ints(prompt_feat_lens),
                                                 _ptr(embedding), len(token_lens), n_timesteps, int(streaming), int(finalize),
                                                 _ptr(mel), _stream()))
        return mel, out_lens

    def cfm_solve(self, mu, spks, cond, lens, z=None, n_timesteps=10, cfg_rate=0.7, streaming=False):
        mu, spks, cond = (_f32(a, self.device) for a in (mu, spks, cond))
        z = _f32(z, self.device) if z is not None else None
        out = torch.empty_like(mu)
        self._check(self.lib.cvk_cfm_solve(self.h, _ptr(mu), _ptr(spks), _ptr(cond), _ints(lens), len(lens), _ptr(z), n_timesteps,
                                           cfg_rate, int(streaming), _ptr(out), _stream()))
        return out

    def flow_inference(self, tokens, token_lens, prompt_feat, prompt_feat_lens, embedding, n_timesteps=10, streaming=False,
                       finalize=True):
        tokens = tokens.to(device=self.device, dtype=torch.int32).contiguous()
        prompt_feat = _f32(prompt_feat, self.device) if prompt_feat is not None and prompt_feat.numel() else None
        embedding = _f32(embedding, self.device)
        ctxl = 0 if finalize else 3
        out_lens = [2 * (int(n) - ctxl) - int(p) for n, p in zip(token_lens, prompt_feat_lens)]
        mel = torch.empty(sum(out_lens), 80, device=self.device)
        self._check(self.lib.cvk_flow_inference(self.h, _ptr(tokens), _ints(token_lens), _ptr(prompt_feat), _ints(prompt_feat_lens),
                                                _ptr(embedding), len(token_lens), n_timesteps, int(streaming), int(finalize),
                                                _ptr(mel), _stream()))
        return mel, out_lens

    # ------------------------------------------------------------------ incremental streaming flow (cvk.h: cvk_flow_stream_*)
    def flow_stream(self, max_frames, n_timesteps=10, dit=False, slots=1):
        """dit=False: CosyVoice2 U-Net estimator (stage "flow"); dit=True: CosyVoice3 DiT (stage "flow3").  slots > 1: one session
        holding `slots` independent utterances (cvk_flow_stream_create_slots), driven by flow_stream_begin_slot /
        flow_stream_chunk_batch."""
        s = ctypes.c_void_p()
        if slots == 1:
            fn = self.lib.cvk_flow3_stream_create if dit else self.lib.cvk_flow_stream_create
            self._check(fn(self.h, int(max_frames), int(n_timesteps), ctypes.byref(s)))
        else:
            self._check(self.lib.cvk_flow_stream_create_slots(self.h, int(bool(dit)), int(slots), int(max_frames), int(n_timesteps),
                                                              ctypes.byref(s)))
        return s

    def flow_stream_destroy(self, fs):
        self.lib.cvk_flow_stream_destroy(self.h, fs)

    def flow_stream_bytes(self, fs):
        return int(self.lib.cvk_flow_stream_bytes(fs))

    def flow_stream_begin(self, fs, prompt_feat, embedding):
        """prompt_feat [Tp,80] (may be empty), embedding [192] or [1,192]"""
        pf = _f32(prompt_feat, self.device) if prompt_feat is not None and prompt_feat.numel() else None
        emb = _f32(embedding, self.device)
        self._check(self.lib.cvk_flow_stream_begin(self.h, fs, _ptr(pf), 0 if pf is None else int(pf.shape[0]), _ptr(emb), _stream()))

    def flow_stream_chunk(self, fs, tokens):
        """tokens: 1-D int32 = prompt tokens + speech tokens so far + 3 look-ahead tokens.  Returns the new mel frames [n,80]."""
        tokens = tokens.to(device=self.device, dtype=torch.int32).contiguous().reshape(-1)
        cap = 2 * int(tokens.numel())
        mel = torch.empty(cap, 80, device=self.device)
        n = ctypes.c_int(0)
        self._check(self.lib.cvk_flow_stream_chunk(self.h, fs, _ptr(tokens), int(tokens.numel()), _ptr(mel), cap, ctypes.byref(n), _stream()))
        return mel[:n.value]

    def flow_stream_begin_slot(self, fs, slot, prompt_feat, embedding):
        """new utterance in `slot` of a multi-slot session; prompt_feat [Tp,80] (may be empty), embedding [192] or [1,192]"""
        pf = _f32(prompt_feat, self.device) if prompt_feat is not None and prompt_feat.numel() else None
        emb = _f32(embedding, self.device)
        self._check(self.lib.cvk_flow_stream_begin_slot(self.h, fs, int(slot), _ptr(pf), 0 if pf is None else int(pf.shape[0]), _ptr(emb),
                                                        _stream()))

    def flow_stream_chunk_batch(self, fs, slots, token_list):
        """One chunk for each slot in `slots`; token_list[b]: 1-D int tokens of slots[b] (as for flow_stream_chunk).  Returns
        (mel [sum n_b, 80], [n_b]): the new frames of every slot back to back."""
        toks = torch.cat([t.reshape(-1).to(device=self.device, dtype=torch.int32) for t in token_list]).contiguous()
        lens = [int(t.numel()) for t in token_list]
        cap = 2 * sum(lens)
        mel = torch.empty(cap, 80, device=self.device)
        n = (ctypes.c_int * len(lens))()
        self._check(self.lib.cvk_flow_stream_chunk_batch(self.h, fs, len(lens), _ints(slots), _ptr(toks), _ints(lens), _ptr(mel), cap, n,
                                                         _stream()))
        out = [int(v) for v in n]
        return mel[:sum(out)], out

    # ------------------------------------------------------------------ LM
    def lm_session(self, max_batch, max_context):
        s = ctypes.c_void_p()
        self._check(self.lib.cvk_lm_session_create(self.h, max_batch, max_context, ctypes.byref(s)))
        return s

    def lm_session_destroy(self, s):
        self.lib.cvk_lm_session_destroy(self.h, s)

    def lm_prefill(self, sess, text, text_lens, speech, speech_lens):
        text = text.to(device=self.device, dtype=torch.int32).contiguous()
        speech = speech.to(device=self.device, dtype=torch.int32).contiguous()
        self._check(self.lib.cvk_lm_prefill(self.h, sess, _ptr(text), _ints(text_lens), _ptr(speech), _ints(speech_lens),
                                            len(text_lens), _stream()))

    def lm_decode(self, sess, n_steps, uniforms, min_len, max_len, out_ids, out_count, done, want_live=True):
        live = ctypes.c_int(0)
        self._check(self.lib.cvk_lm_decode(self.h, sess, n_steps, _ptr(uniforms), _ptr(min_len), _ptr(max_len), _ptr(out_ids),
                                           out_ids.shape[1], _ptr(out_count), _ptr(done),
                                           ctypes.byref(live) if want_live else None, _stream()))
        return live.value

    def lm_forward_logp(self, embeds, lens):
        embeds = _f32(embeds, self.device)
        out = torch.empty(embeds.shape[0], self.lm_vocab(), device=self.device)
        self._check(self.lib.cvk_lm_forward_logp(self.h, _ptr(embeds), _ints(lens), len(lens), _ptr(out), _stream()))
        return out

    def lm_vocab(self):
        """width of the LM's log-prob rows: 6564 (Qwen2LM) or 6764 (CosyVoice3LM, 3 impossible pad ids)"""
        return int(self.lib.cvk_lm_vocab(self.h))

    def lm_begin(self, sess, B=1):
        self._check(self.lib.cvk_lm_begin(self.h, sess, B, _stream()))

    def lm_feed(self, sess, ids, kinds):
        """ids / kinds: python int lists (kind 0 text id, 1 speech id, 2 llm_embedding row)"""
        self._check(self.lib.cvk_lm_feed(self.h, sess, _ints(ids), _ints(kinds), len(ids), _stream()))

    def lm_next_logp(self, sess, B=1):
        out = torch.empty(B, self.lm_vocab(), device=self.device)
        self._check(self.lib.cvk_lm_next_logp(self.h, sess, _ptr(out), _stream()))
        return out

    def lm_feed_rows(self, sess, rows, counts, ids, kinds):
        """rows: distinct session rows; row rows[r] receives counts[r] positions; ids / kinds: python int lists of all positions,
        concatenated in row order (kinds as in lm_feed).  One forward for every row and position (cvk_lm_feed_rows)."""
        if len(counts) != len(rows) or len(ids) != len(kinds) or len(ids) != sum(int(c) for c in counts):
            raise ValueError("lm_feed_rows: need len(counts) == len(rows) and len(ids) == len(kinds) == sum(counts)")
        self._check(self.lib.cvk_lm_feed_rows(self.h, sess, len(rows), _ints(rows), _ints(counts), _ints(ids), _ints(kinds), _stream()))

    def lm_next_logp_rows(self, sess, rows):
        """log-probs [len(rows), V] of the next id of each listed row (cvk_lm_next_logp_rows)"""
        out = torch.empty(len(rows), self.lm_vocab(), device=self.device)
        self._check(self.lib.cvk_lm_next_logp_rows(self.h, sess, len(rows), _ints(rows), _ptr(out), _stream()))
        return out

    def lm_last_logits(self, sess, B):
        """the row the last decode step sampled from: log-probs with the sampler's -inf marks (masked eos, repeated id of a
        fallback draw); rows done before that step hold the raw head logits"""
        out = torch.empty(B, self.lm_vocab(), device=self.device)
        self._check(self.lib.cvk_lm_last_logits(self.h, sess, _ptr(out), _stream()))
        return out

    def ras_sample(self, logp, history, hist_count, uniforms, ignore_eos):
        logp = _f32(logp, self.device).clone()
        history = history.to(device=self.device, dtype=torch.int32).contiguous()
        hist_count = hist_count.to(device=self.device, dtype=torch.int32).contiguous()
        uniforms = _f32(uniforms, self.device)
        ignore_eos = ignore_eos.to(device=self.device, dtype=torch.int32).contiguous()
        out = torch.empty(logp.shape[0], dtype=torch.int32, device=self.device)
        self._check(self.lib.cvk_ras_sample(self.h, _ptr(logp), logp.shape[0], logp.shape[1], _ptr(history), history.shape[1],
                                            _ptr(hist_count), _ptr(uniforms), _ptr(ignore_eos), _ptr(out), _stream()))
        return out

    def sample_step(self, logits, uniforms, min_len, max_len, out_ids, out_count, done, ctx_len, base_len, live, speech_emb, next_x,
                    gamma=None, xn=None):
        """one decode-graph sampler step (cvk_op_sample_step) on device tensors, updated in place: logits [B,V] fp32, uniforms
        [steps,B,2] fp32, min_len / max_len / out_count / done / ctx_len / base_len [B] int32, out_ids [B,out_ld] int32, live [1] int32,
        speech_emb [V,896], next_x [B,896] fp32; gamma [896] and xn [B,896] fp32 both or neither (fused layer-0 RMSNorm)."""
        B, V = logits.shape
        self._check(self.lib.cvk_op_sample_step(
            self.h, _ptr(logits), B, V, _ptr(uniforms), uniforms.shape[0], _ptr(min_len), _ptr(max_len), _ptr(out_ids), out_ids.shape[1],
            _ptr(out_count), _ptr(done), _ptr(ctx_len), _ptr(base_len), _ptr(live), _ptr(speech_emb), _ptr(next_x), _ptr(gamma), _ptr(xn),
            _stream()))

    def log_softmax(self, x):
        """log_softmax of every row of x [rows, V] with the LM's log-prob kernel (cvk_op_log_softmax); returns a new tensor"""
        x = _f32(x, self.device).clone()
        self._check(self.lib.cvk_op_log_softmax(self.h, _ptr(x), x.shape[0], x.shape[1], _stream()))
        return x

    # ------------------------------------------------------------------ mel
    def whisper_log_mel(self, wav, lens):
        """wav [sum N_b] at 16 kHz -> [sum N_b // 160, 128] (whisper.log_mel_spectrogram(n_mels=128), time-major)"""
        wav = _f32(wav, self.device)
        out = torch.empty(sum(int(l) // 160 for l in lens), 128, device=self.device)
        self._check(self.lib.cvk_whisper_log_mel(self.h, _ptr(wav), _ints(lens), len(lens), _ptr(out), _stream()))
        return out

    def kaldi_fbank(self, wav, lens, subtract_mean=True):
        """wav [sum N_b] at 16 kHz -> [sum 1 + (N_b - 400) // 160, 80] (kaldi.fbank(num_mel_bins=80, dither=0) [- mean over frames])"""
        wav = _f32(wav, self.device)
        out = torch.empty(sum(1 + (int(l) - 400) // 160 for l in lens), 80, device=self.device)
        self._check(self.lib.cvk_kaldi_fbank(self.h, _ptr(wav), _ints(lens), len(lens), int(bool(subtract_mean)), _ptr(out), _stream()))
        return out

    def mel_spectrogram(self, wav, lens, fmax=8000):
        """wav [sum N_b] -> mel [sum N_b // 480, 80]; fmax 8000 (CosyVoice2) or None / 12000 (CosyVoice3)"""
        wav = _f32(wav, self.device)
        mel = torch.empty(sum(int(l) // 480 for l in lens), 80, device=self.device)
        self._check(self.lib.cvk_mel_spectrogram_ex(self.h, _ptr(wav), _ints(lens), len(lens), int(fmax or 0), _ptr(mel), _stream()))
        return mel

    def mel_resample(self, mel, lens, out_lens):
        """the `speed` time-stretch (cvk_mel_resample): mel [sum lens, 80] time-major -> [sum out_lens, 80], utterance b linearly
        interpolated from lens[b] to out_lens[b] frames exactly as F.interpolate(mode="linear") on the device.  A length of 0 is a
        ValueError (F.interpolate refuses it too)."""
        lens, out_lens = [int(v) for v in lens], [int(v) for v in out_lens]
        if len(lens) != len(out_lens) or not lens or min(lens + out_lens) < 1:
            raise ValueError(f"mel_resample: one input and one output length >= 1 per utterance, got {lens} -> {out_lens}")
        mel = _f32(mel, self.device)
        if mel.shape != (sum(lens), 80):
            raise ValueError(f"mel_resample: mel must be [sum lens, 80] = [{sum(lens)}, 80], got {list(mel.shape)}")
        out = torch.empty(sum(out_lens), 80, device=self.device)
        self._check(self.lib.cvk_mel_resample(self.h, _ptr(mel), _ints(lens), _ints(out_lens), len(lens), _ptr(out), _stream()))
        return out
