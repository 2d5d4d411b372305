"""Import shims for running the UNMODIFIED reference (a CosyVoice checkout, located by $COSYVOICE_REF_ROOT) on CPU.

Used only by ``oracle/make_golden.py`` to regenerate ``tests/golden/``; no test imports the reference.

The reference imports, at module import time, packages that are absent from this
image (SURVEY.md §8c): onnxruntime, omegaconf, conformer, diffusers, and
matcha.utils drags in hydra/lightning.  None of them is on the arithmetic path
except diffusers' ``Attention``/``GELU`` (restated below from diffusers 0.29.0
``models/attention_processor.py`` / ``models/activations.py`` semantics; parity
for those two classes is therefore unpinned, see oracle/__init__.py).
"""
import importlib
import importlib.machinery
import os
import sys
import types

import torch
import torch.nn as nn
import torch.nn.functional as F

REF_ROOT = os.environ.get("COSYVOICE_REF_ROOT", "/root/reference")
MATCHA_ROOT = os.path.join(REF_ROOT, "third_party", "Matcha-TTS")


def available() -> bool:
    return os.path.isdir(os.path.join(REF_ROOT, "cosyvoice"))


# --------------------------------------------------------------------------- diffusers restatement
class _Attention(nn.Module):
    """diffusers 0.29.0 ``Attention`` as used by Matcha ``BasicTransformerBlock``:
    to_q/to_k/to_v without bias, to_out[0] with bias, scale = dim_head**-0.5,
    SDPA with the additive mask broadcast over heads (AttnProcessor2_0)."""

    def __init__(self, query_dim, heads=8, dim_head=64, dropout=0.0, bias=False,
                 cross_attention_dim=None, upcast_attention=False, **kw):
        super().__init__()
        inner = heads * dim_head
        self.heads = heads
        self.dim_head = dim_head
        self.scale = dim_head ** -0.5
        self.to_q = nn.Linear(query_dim, inner, bias=bias)
        self.to_k = nn.Linear(cross_attention_dim or query_dim, inner, bias=bias)
        self.to_v = nn.Linear(cross_attention_dim or query_dim, inner, bias=bias)
        self.to_out = nn.ModuleList([nn.Linear(inner, query_dim, bias=True), nn.Dropout(dropout)])

    def forward(self, hidden_states, encoder_hidden_states=None, attention_mask=None, **kw):
        b, t, _ = hidden_states.shape
        ctx = hidden_states if encoder_hidden_states is None else encoder_hidden_states
        q = self.to_q(hidden_states).view(b, t, self.heads, self.dim_head).transpose(1, 2)
        k = self.to_k(ctx).view(b, -1, self.heads, self.dim_head).transpose(1, 2)
        v = self.to_v(ctx).view(b, -1, self.heads, self.dim_head).transpose(1, 2)
        if attention_mask is not None:
            # prepare_attention_mask: [B, T, S] -> repeat per head -> [B, H, T, S]
            attention_mask = attention_mask.unsqueeze(1)
        o = F.scaled_dot_product_attention(q, k, v, attn_mask=attention_mask, dropout_p=0.0, is_causal=False)
        o = o.transpose(1, 2).reshape(b, t, self.heads * self.dim_head)
        o = self.to_out[0](o)
        return self.to_out[1](o)


class _GELU(nn.Module):
    """diffusers 0.29.0 ``GELU``: Linear + F.gelu(approximate=...)"""

    def __init__(self, dim_in, dim_out, approximate="none", bias=True):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out, bias=bias)
        self.approximate = approximate

    def forward(self, x):
        return F.gelu(self.proj(x), approximate=self.approximate)


# --------------------------------------------------------------------------- x_transformers restatement (CosyVoice3 DiT)
class _RotaryEmbedding(nn.Module):
    """x_transformers==2.11.24 ``RotaryEmbedding`` (requirements.txt:39) as used by cosyvoice/flow/DiT/dit.py:128,159:
    ``inv_freq = base**-(arange(0, dim, 2)/dim)``; ``forward_from_seq_len(n)`` -> ``forward(arange(n))`` -> freqs [1, n, dim] with
    every frequency duplicated in ADJACENT positions (``stack((f, f), -1)`` flattened), scale 1.0 (no xpos).  Restated from the
    published source: the package is not installed offline, so parity of this class and of ``apply_rotary_pos_emb`` is unpinned."""

    def __init__(self, dim, base=10000, interpolation_factor=1.0, **kw):
        super().__init__()
        self.register_buffer("inv_freq", 1.0 / (base ** (torch.arange(0, dim, 2).float() / dim)), persistent=False)
        self.interpolation_factor = interpolation_factor

    def forward_from_seq_len(self, seq_len):
        return self.forward(torch.arange(seq_len, device=self.inv_freq.device))

    def forward(self, t):
        if t.ndim == 1:
            t = t[None, :]
        freqs = torch.einsum("b i , j -> b i j", t.type_as(self.inv_freq), self.inv_freq) / self.interpolation_factor
        freqs = torch.stack((freqs, freqs), dim=-1).flatten(-2)
        return freqs, 1.0


def _rotate_half(x):
    x = x.reshape(*x.shape[:-1], -1, 2)
    x1, x2 = x.unbind(dim=-1)
    return torch.stack((-x2, x1), dim=-1).flatten(-2)


def _apply_rotary_pos_emb(t, freqs, scale=1):
    """x_transformers==2.11.24 ``apply_rotary_pos_emb``: partial rotary over the first ``freqs.shape[-1]`` channels of the LAST
    dimension (the DiT applies it to the un-split [b, n, heads*dim_head] projections, so only the first head's 64 channels rotate,
    cosyvoice/flow/DiT/modules.py:368-373), interleaved pairs (GPT-J style)."""
    rot_dim, seq_len, orig_dtype = freqs.shape[-1], t.shape[-2], t.dtype
    freqs = freqs[:, -seq_len:, :]
    if t.ndim == 4 and freqs.ndim == 3:
        freqs = freqs[:, None]
    t, t_unrotated = t[..., :rot_dim], t[..., rot_dim:]
    t = (t * freqs.cos() * scale) + (_rotate_half(t) * freqs.sin() * scale)
    return torch.cat((t, t_unrotated), dim=-1).type(orig_dtype)


class _Unused(nn.Module):
    def __init__(self, *a, **k):
        super().__init__()
        raise NotImplementedError("shim class not on the CosyVoice2 inference path")


def _get_activation(name):
    return {"silu": nn.SiLU(), "swish": nn.SiLU(), "mish": nn.Mish(), "gelu": nn.GELU(), "relu": nn.ReLU()}[name]


class _DictConfig(dict):
    def __init__(self, content=None, **kw):
        super().__init__(content or {}, **kw)

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e


def _mod(name, **attrs):
    m = types.ModuleType(name)
    m.__spec__ = importlib.machinery.ModuleSpec(name, None)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


_installed = False


def install():
    """Put the reference on sys.path and register the stub modules (idempotent)."""
    global _installed
    if _installed:
        return
    if not available():
        raise RuntimeError(f"reference tree not found at {REF_ROOT}")
    for p in (REF_ROOT, MATCHA_ROOT):
        if p not in sys.path:
            sys.path.insert(0, p)
    # resolve transformers' lazy optional-dependency probes BEFORE any stub module is registered
    from transformers import Qwen2Config, Qwen2ForCausalLM  # noqa: F401
    if "onnxruntime" not in sys.modules:
        try:
            importlib.import_module("onnxruntime")
        except Exception:
            _mod("onnxruntime", InferenceSession=_Unused, SessionOptions=_Unused,
                 GraphOptimizationLevel=types.SimpleNamespace(ORT_ENABLE_ALL=0))
    try:
        importlib.import_module("omegaconf")
    except Exception:
        _mod("omegaconf", DictConfig=_DictConfig)
    try:
        importlib.import_module("conformer")
    except Exception:
        _mod("conformer", ConformerBlock=_Unused)
    try:
        importlib.import_module("diffusers")
    except Exception:
        _mod("diffusers")
        _mod("diffusers.models")
        _mod("diffusers.models.activations", get_activation=_get_activation, GELU=_GELU)
        _mod("diffusers.models.attention", GEGLU=_Unused, GELU=_GELU, AdaLayerNorm=_Unused,
             AdaLayerNormZero=_Unused, ApproximateGELU=_Unused)
        _mod("diffusers.models.attention_processor", Attention=_Attention)
        _mod("diffusers.models.lora", LoRACompatibleLinear=nn.Linear)
        _mod("diffusers.utils")
        _mod("diffusers.utils.torch_utils", maybe_allow_in_graph=lambda c: c)
    try:
        importlib.import_module("x_transformers.x_transformers")
    except Exception:
        _mod("x_transformers")
        _mod("x_transformers.x_transformers", RotaryEmbedding=_RotaryEmbedding, apply_rotary_pos_emb=_apply_rotary_pos_emb)
    # matcha/utils/__init__.py imports hydra/lightning/rich; only audio.py is needed
    import logging
    mu = _mod("matcha.utils")
    mu.__path__ = [os.path.join(MATCHA_ROOT, "matcha", "utils")]
    _mod("matcha.utils.pylogger", get_pylogger=lambda name=__name__: logging.getLogger(name))
    try:
        importlib.import_module("librosa")
    except Exception:
        from . import mel as _mel
        _mod("librosa")
        _mod("librosa.filters", mel=_mel.librosa_mel_filterbank)
    _installed = True


QWEN_CFG = dict(vocab_size=151936, hidden_size=896, intermediate_size=4864, num_hidden_layers=24,
                num_attention_heads=14, num_key_value_heads=2, rope_theta=1000000.0, rms_norm_eps=1e-6,
                max_position_embeddings=32768, tie_word_embeddings=True, hidden_act="silu",
                attention_dropout=0.0, use_sliding_window=False)


def build_hift():
    """Reference HiFTGenerator with the cosyvoice2.yaml:89-111 hyper-parameters."""
    install()
    from cosyvoice.hifigan.generator import HiFTGenerator
    from cosyvoice.hifigan.f0_predictor import ConvRNNF0Predictor
    m = HiFTGenerator(in_channels=80, base_channels=512, nb_harmonics=8, sampling_rate=24000,
                      nsf_alpha=0.1, nsf_sigma=0.003, nsf_voiced_threshold=10,
                      upsample_rates=[8, 5, 3], upsample_kernel_sizes=[16, 11, 7],
                      istft_params={"n_fft": 16, "hop_len": 4},
                      resblock_kernel_sizes=[3, 7, 11], resblock_dilation_sizes=[[1, 3, 5]] * 3,
                      source_resblock_kernel_sizes=[7, 7, 11], source_resblock_dilation_sizes=[[1, 3, 5]] * 3,
                      lrelu_slope=0.1, audio_limit=0.99,
                      f0_predictor=ConvRNNF0Predictor(num_class=1, in_channels=80, cond_channels=512))
    return m.eval()


def build_flow(num_mid_blocks=12, n_blocks=4, enc_blocks=6, enc_up_blocks=4):
    """Reference CausalMaskedDiffWithXvec with cosyvoice2.yaml:38-87 hyper-parameters.
    Layer counts can be reduced for fast tests (the reference constructors take them)."""
    install()
    from cosyvoice.flow.flow import CausalMaskedDiffWithXvec
    from cosyvoice.flow.flow_matching import CausalConditionalCFM
    from cosyvoice.flow.decoder import CausalConditionalDecoder
    from cosyvoice.transformer.upsample_encoder import UpsampleConformerEncoder
    enc = UpsampleConformerEncoder(output_size=512, attention_heads=8, linear_units=2048, num_blocks=enc_blocks,
                                   dropout_rate=0.1, positional_dropout_rate=0.1, attention_dropout_rate=0.1,
                                   normalize_before=True, input_layer="linear", pos_enc_layer_type="rel_pos_espnet",
                                   selfattention_layer_type="rel_selfattn", input_size=512, use_cnn_module=False,
                                   macaron_style=False, static_chunk_size=25)
    if enc_up_blocks != 4:
        enc.up_encoders = enc.up_encoders[:enc_up_blocks]
    est = CausalConditionalDecoder(in_channels=320, out_channels=80, channels=[256], dropout=0.0,
                                   attention_head_dim=64, n_blocks=n_blocks, num_mid_blocks=num_mid_blocks,
                                   num_heads=8, act_fn="gelu", static_chunk_size=50, num_decoding_left_chunks=-1)
    cfm = CausalConditionalCFM(in_channels=240, n_spks=1, spk_emb_dim=80,
                               cfm_params=_DictConfig(dict(sigma_min=1e-6, solver="euler", t_scheduler="cosine",
                                                           training_cfg_rate=0.2, inference_cfg_rate=0.7,
                                                           reg_loss_type="l1")),
                               estimator=est)
    flow = CausalMaskedDiffWithXvec(input_size=512, output_size=80, spk_embed_dim=192, output_type="mel",
                                    vocab_size=6561, input_frame_rate=25, only_mask_loss=True, token_mel_ratio=2,
                                    pre_lookahead_len=3, encoder=enc, decoder=cfm)
    return flow.eval()


def build_llm(num_layers=24, tmpdir=None):
    """Reference Qwen2LM over a random-init HF Qwen2ForCausalLM of Qwen2.5-0.5B shape
    (cosyvoice2.yaml:23-36; config per SURVEY.md §8c)."""
    install()
    import tempfile
    from transformers import Qwen2Config, Qwen2ForCausalLM
    from cosyvoice.llm.llm import Qwen2LM, Qwen2Encoder
    from cosyvoice.utils.common import ras_sampling
    from functools import partial
    cfg = dict(QWEN_CFG)
    cfg["num_hidden_layers"] = num_layers
    d = tmpdir or tempfile.mkdtemp(prefix="qwen_blank_")
    with torch.device("cpu"):
        Qwen2ForCausalLM(Qwen2Config(**cfg)).save_pretrained(d)
    enc = Qwen2Encoder(d)
    lm = Qwen2LM(llm_input_size=896, llm_output_size=896, speech_token_size=6561, llm=enc,
                 sampling=partial(ras_sampling, top_p=0.8, top_k=25, win_size=10, tau_r=0.1),
                 length_normalized_loss=True, lsm_weight=0, mix_ratio=[5, 15])
    _pin_forward_one_step(enc)
    return lm.eval()


def _pin_forward_one_step(enc):
    """transformers-version shim, NOT a change of reference semantics.

    ``Qwen2Encoder.forward_one_step`` (llm/llm.py:242-254) hands HF a 2-D attention mask whose length is the
    number of NEW positions only (``masks[:, -1, :]`` of a [1,q,q] tril, llm.py:540).  Under the pinned
    transformers==4.51.3 an all-ones 2-D mask is dropped on the SDPA path, i.e. the step is plain causal
    KV-cache decoding.  transformers 5.5.0 (the only version installed offline) instead applies the too-short
    mask to the cached keys and the step output no longer equals the teacher-forced forward (measured:
    max|diff| 4.5 vs 2e-6).  The oracle follows the pinned behaviour, so the golden generator passes
    ``attention_mask=None`` (equivalent to an all-ones mask) to the unmodified HF model."""
    import types

    class _CacheView:
        """inference_bistream reads the cached length as ``cache[0][0].size(2)`` (llm.py:621): the tuple-style indexing that
        the pinned transformers' DynamicCache still offers and 5.5's does not.  Index access only; HF gets the real object."""
        def __init__(self, dc):
            self.dc = dc

        def __getitem__(self, i):
            if hasattr(self.dc, "layers"):
                return self.dc.layers[i].keys, self.dc.layers[i].values
            return self.dc.key_cache[i], self.dc.value_cache[i]

    def forward_one_step(self, xs, masks, cache=None):
        outs = self.model(inputs_embeds=xs, attention_mask=None, output_hidden_states=True, return_dict=True,
                          use_cache=True, past_key_values=cache.dc if isinstance(cache, _CacheView) else cache)
        return outs.hidden_states[-1], _CacheView(outs.past_key_values)
    enc.forward_one_step = types.MethodType(forward_one_step, enc)


def build_dit(depth=22):
    """Reference DiT estimator with the cosyvoice3.yaml hyper-parameters (depth reducible for fast tests)."""
    install()
    from cosyvoice.flow.DiT.dit import DiT
    return DiT(dim=1024, depth=depth, heads=16, dim_head=64, ff_mult=2, mel_dim=80, mu_dim=80, spk_dim=80, out_channels=80,
               static_chunk_size=50, num_decoding_left_chunks=-1).eval()


def build_flow3(depth=22):
    """Reference CausalMaskedDiffWithDiT (CosyVoice3 flow) with the cosyvoice3.yaml hyper-parameters."""
    install()
    from cosyvoice.flow.flow import CausalMaskedDiffWithDiT
    from cosyvoice.flow.flow_matching import CausalConditionalCFM
    from cosyvoice.transformer.upsample_encoder import PreLookaheadLayer
    cfm = CausalConditionalCFM(in_channels=240, n_spks=1, spk_emb_dim=80,
                               cfm_params=_DictConfig(dict(sigma_min=1e-6, solver="euler", t_scheduler="cosine",
                                                           training_cfg_rate=0.2, inference_cfg_rate=0.7,
                                                           reg_loss_type="l1")),
                               estimator=build_dit(depth))
    flow = CausalMaskedDiffWithDiT(input_size=80, output_size=80, spk_embed_dim=192, output_type="mel", vocab_size=6561,
                                   input_frame_rate=25, only_mask_loss=True, token_mel_ratio=2, pre_lookahead_len=3,
                                   pre_lookahead_layer=PreLookaheadLayer(in_channels=80, channels=1024, pre_lookahead_len=3),
                                   decoder=cfm)
    return flow.eval()


def build_hift_causal():
    """Reference CausalHiFTGenerator with the cosyvoice3.yaml hyper-parameters.  (The constructor draws ~260 MB of 'stored
    noise' from the global RNG; the golden generator overwrites it with explicit tensors.)"""
    install()
    from cosyvoice.hifigan.generator import CausalHiFTGenerator
    from cosyvoice.hifigan.f0_predictor import CausalConvRNNF0Predictor
    m = CausalHiFTGenerator(in_channels=80, base_channels=512, nb_harmonics=8, sampling_rate=24000,
                            nsf_alpha=0.1, nsf_sigma=0.003, nsf_voiced_threshold=10,
                            upsample_rates=[8, 5, 3], upsample_kernel_sizes=[16, 11, 7],
                            istft_params={"n_fft": 16, "hop_len": 4},
                            resblock_kernel_sizes=[3, 7, 11], resblock_dilation_sizes=[[1, 3, 5]] * 3,
                            source_resblock_kernel_sizes=[7, 7, 11], source_resblock_dilation_sizes=[[1, 3, 5]] * 3,
                            lrelu_slope=0.1, audio_limit=0.99, conv_pre_look_right=4,
                            f0_predictor=CausalConvRNNF0Predictor(num_class=1, in_channels=80, cond_channels=512))
    return m.eval()


def build_llm3(num_layers=24, tmpdir=None):
    """Reference CosyVoice3LM (cosyvoice3.yaml) over a random-init HF Qwen2ForCausalLM of Qwen2.5-0.5B shape."""
    install()
    import tempfile
    from functools import partial
    from transformers import Qwen2Config, Qwen2ForCausalLM
    from cosyvoice.llm.llm import CosyVoice3LM, Qwen2Encoder
    from cosyvoice.utils.common import ras_sampling
    cfg = dict(QWEN_CFG)
    cfg["num_hidden_layers"] = num_layers
    d = tmpdir or tempfile.mkdtemp(prefix="qwen_blank_")
    with torch.device("cpu"):
        Qwen2ForCausalLM(Qwen2Config(**cfg)).save_pretrained(d)
    enc = Qwen2Encoder(d)
    lm = CosyVoice3LM(llm_input_size=896, llm_output_size=896, speech_token_size=6561, llm=enc,
                      sampling=partial(ras_sampling, top_p=0.8, top_k=25, win_size=10, tau_r=0.1),
                      length_normalized_loss=True, lsm_weight=0, mix_ratio=[5, 15])
    _pin_forward_one_step(enc)
    return lm.eval()
