"""Geometry of the Qwen3-ASR audio tower as the causal streaming encoder runs it
(reference third_party/qwen3-asr-causal/src/qwen3_asr_causal/causal.py:60-140, config.py:17-45)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict

import numpy as np


@dataclass(frozen=True)
class QwenTowerDims:
    n_mels: int = 128
    conv_channels: int = 480          # conv2d1/2/3 output channels (3x3, stride 2, pad 1; 8 mel frames -> 1 step)
    d_model: int = 896
    n_head: int = 14                  # head_dim must be 64
    n_layer: int = 18
    ffn_dim: int = 3584
    out_dim: int = 1024               # proj2 output (the LLM's embedding width)
    max_positions: int = 1500         # rows of the sinusoid table; beyond it the formula is evaluated (causal.py:204-228)
    chunk_frames: int = 8             # one decoder step = 80 ms = 8 mel frames (config.py:87-89)
    block_frames: int = 192           # fixed attention block (config.py:31-36); 0 = consume per chunk
    left_context_steps: int = 150     # 12 s of left context in steps (causal.py:103-106)
    block_bidirectional: bool = True
    conv_out_bias: bool = True
    mutable_tail_steps: int = 0       # bounded mutable tail (causal.py:101-113, 548-640): the last steps are re-encoded by
                                      # every call until they leave the tail; 0 = strict append-only; exclusive with blocks

    @property
    def freq_out(self) -> int:
        return self.n_mels // 8

    @property
    def conv_features(self) -> int:
        return self.conv_channels * self.freq_out

    def as_tuple(self):
        return (self.n_mels, self.conv_channels, self.d_model, self.n_head, self.n_layer, self.ffn_dim, self.out_dim,
                self.max_positions, self.chunk_frames, self.block_frames, self.left_context_steps,
                int(self.block_bidirectional), int(self.conv_out_bias), self.mutable_tail_steps)


QWEN_DIMS: Dict[str, QwenTowerDims] = {
    # test geometries (head_dim 64 like the real tower)
    "qnano": QwenTowerDims(conv_channels=8, d_model=128, n_head=2, n_layer=2, ffn_dim=256, out_dim=96, max_positions=40,
                           left_context_steps=30),
    "qnano-chunk": QwenTowerDims(conv_channels=8, d_model=128, n_head=2, n_layer=2, ffn_dim=256, out_dim=96,
                                 max_positions=4096, block_frames=0, left_context_steps=25, block_bidirectional=False),
    # bounded mutable tail: the last 6 steps (0.48 s) stay re-computable; causal, and bidirectional within a call
    "qnano-tail": QwenTowerDims(conv_channels=8, d_model=128, n_head=2, n_layer=2, ffn_dim=256, out_dim=96,
                                max_positions=4096, block_frames=0, left_context_steps=25, block_bidirectional=False,
                                mutable_tail_steps=6),
    "qnano-tail-bidir": QwenTowerDims(conv_channels=8, d_model=128, n_head=2, n_layer=2, ffn_dim=256, out_dim=96,
                                      max_positions=4096, block_frames=0, left_context_steps=25, block_bidirectional=True,
                                      mutable_tail_steps=6),
    # Qwen3-ASR-0.6B audio tower (public HF audio_config: d_model 896, 18 layers, 14 heads, ffn 3584,
    # downsample_hidden_size 480, output_dim 1024); to be confirmed against the checkpoint when it is mounted
    "qwen3-asr-0.6b": QwenTowerDims(),
}


def sinusoid_table(max_positions: int, d_model: int) -> np.ndarray:
    """The tower's fixed positional table: [sin | cos] of pos * exp(-ln(1e4)/(half-1) * i)."""
    half = d_model // 2
    inv = np.exp(-np.log(10000.0) / float(max(1, half - 1)) * np.arange(half, dtype=np.float32)).astype(np.float32)
    pos = np.arange(max_positions, dtype=np.float32)
    scaled = pos[:, None] * inv[None, :]
    return np.concatenate([np.sin(scaled), np.cos(scaled)], axis=1).astype(np.float32)


def synthetic_tower_state_dict(dims: QwenTowerDims, seed: int = 0) -> Dict[str, np.ndarray]:
    """Seeded weights with the tower's own parameter names, scaled for unit-variance activations."""
    rng = np.random.default_rng(seed)
    C, d, F = dims.conv_channels, dims.d_model, dims.ffn_dim

    def w(*shape, fan_in):
        return (rng.standard_normal(shape) / np.sqrt(fan_in)).astype(np.float32)

    def b(n, s=0.02):
        return (rng.standard_normal(n) * s).astype(np.float32)

    sd = {
        "conv2d1.weight": w(C, 1, 3, 3, fan_in=9) * 1.5, "conv2d1.bias": b(C),
        "conv2d2.weight": w(C, C, 3, 3, fan_in=9 * C) * 1.5, "conv2d2.bias": b(C),
        "conv2d3.weight": w(C, C, 3, 3, fan_in=9 * C) * 1.5, "conv2d3.bias": b(C),
        "conv_out.weight": w(d, dims.conv_features, fan_in=dims.conv_features) * 2.0,
        "positional_embedding.positional_embedding": sinusoid_table(dims.max_positions, d),
        "ln_post.weight": (1.0 + 0.1 * rng.standard_normal(d)).astype(np.float32), "ln_post.bias": b(d),
        "proj1.weight": w(d, d, fan_in=d), "proj1.bias": b(d),
        "proj2.weight": w(dims.out_dim, d, fan_in=d), "proj2.bias": b(dims.out_dim),
    }
    if dims.conv_out_bias:
        sd["conv_out.bias"] = b(d)
    for i in range(dims.n_layer):
        p = f"layers.{i}."
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            sd[p + f"self_attn.{n}.weight"] = w(d, d, fan_in=d) * (1.6 if n in ("q_proj", "k_proj") else 1.0)
            sd[p + f"self_attn.{n}.bias"] = b(d)
        for n in ("self_attn_layer_norm", "final_layer_norm"):
            sd[p + n + ".weight"] = (1.0 + 0.1 * rng.standard_normal(d)).astype(np.float32)
            sd[p + n + ".bias"] = b(d)
        sd[p + "fc1.weight"] = w(F, d, fan_in=d); sd[p + "fc1.bias"] = b(F)
        sd[p + "fc2.weight"] = w(d, F, fan_in=F); sd[p + "fc2.bias"] = b(d)
    return sd


@dataclass(frozen=True)
class QwenTextDims:
    """Geometry of the Qwen3 text decoder behind Qwen3-ASR (HF ``Qwen3Model`` + ``lm_head``; reference
    third_party/qwen3-asr-causal/src/qwen3_asr_causal/model.py:1498-1507).

    Qwen3-ASR's thinker uses MRoPE; with audio rows and text only, its three position streams are equal, so it reduces
    to plain 1D rotate-half RoPE over ``head_dim`` with ``inv_freq = rope_theta ** (-2i / head_dim)`` (``rope_inv_freq``,
    in HF's fp32 arithmetic).  The engine assumes exactly that."""
    vocab: int = 151936
    d_model: int = 1024
    n_layer: int = 28
    n_head: int = 16
    n_kv_head: int = 8
    head_dim: int = 128               # the kernels specialise on 128
    ffn_dim: int = 3072
    rope_theta: float = 1e6
    rms_eps: float = 1e-6
    tied: bool = True                 # lm_head shares embed_tokens
    max_ctx: int = 1024               # positions per session

    def as_tuple(self):
        return (self.vocab, self.d_model, self.n_layer, self.n_head, self.n_kv_head, self.head_dim, self.ffn_dim,
                int(self.tied), self.max_ctx, float(self.rope_theta), float(self.rms_eps))


QWEN_TEXT_DIMS: Dict[str, QwenTextDims] = {
    "tnano": QwenTextDims(vocab=2048, d_model=256, n_layer=2, n_head=4, n_kv_head=2, ffn_dim=512, rope_theta=1e6,
                          tied=False, max_ctx=1024),
    # Qwen3-ASR-0.6B text model (public Qwen3-0.6B numbers: d 1024, 28 layers, 16 / 8 heads of 128, ffn 3072,
    # vocab 151936, theta 1e6, tied embeddings); to be confirmed against the checkpoint's thinker_config.text_config
    "qwen3-asr-0.6b": QwenTextDims(),
}


def rope_inv_freq(rope_theta: float, head_dim: int = 128) -> np.ndarray:
    """RoPE frequencies [head_dim / 2] exactly as HF's default rope init computes them (transformers'
    ``Qwen3RotaryEmbedding``, and the reference's ``_qwen3_asr_default_rope_init``): fp32 torch arithmetic,
    ``1 / base ** (arange(0, dim, 2).float() / dim)``.  Rounded once from a double-precision pow, or by a C ``powf``, some
    entries land one ulp away, and the angle error grows with the position."""
    import torch
    base = float(rope_theta)
    inv = 1.0 / (base ** (torch.arange(0, head_dim, 2, dtype=torch.int64).to(dtype=torch.float) / head_dim))
    return inv.numpy().astype(np.float32)


def synthetic_text_state_dict(dims: QwenTextDims, seed: int = 0) -> Dict[str, np.ndarray]:
    """Seeded weights with HF ``Qwen3Model`` parameter names (plus ``lm_head.weight`` when untied).  Embedding rows
    have unit variance (the residual stream's scale); the head is scaled so that logits have sigma ~3.  With tied
    embeddings the embedding table carries that head scale instead."""
    rng = np.random.default_rng(seed)
    d, F, hd = dims.d_model, dims.ffn_dim, dims.head_dim
    qd, kvd = dims.n_head * hd, dims.n_kv_head * hd

    def w(*shape, fan_in, s=1.0):
        return (rng.standard_normal(shape) * (s / np.sqrt(fan_in))).astype(np.float32)

    def g(n):
        return (1.0 + 0.1 * rng.standard_normal(n)).astype(np.float32)

    emb = w(dims.vocab, d, fan_in=d, s=3.0) if dims.tied else rng.standard_normal((dims.vocab, d)).astype(np.float32)
    sd = {"embed_tokens.weight": emb}
    for i in range(dims.n_layer):
        p = f"layers.{i}."
        sd[p + "self_attn.q_proj.weight"] = w(qd, d, fan_in=d)
        sd[p + "self_attn.k_proj.weight"] = w(kvd, d, fan_in=d)
        sd[p + "self_attn.v_proj.weight"] = w(kvd, d, fan_in=d)
        sd[p + "self_attn.o_proj.weight"] = w(d, qd, fan_in=qd, s=0.5)
        sd[p + "self_attn.q_norm.weight"] = g(hd)
        sd[p + "self_attn.k_norm.weight"] = g(hd)
        sd[p + "mlp.gate_proj.weight"] = w(F, d, fan_in=d)
        sd[p + "mlp.up_proj.weight"] = w(F, d, fan_in=d)
        sd[p + "mlp.down_proj.weight"] = w(d, F, fan_in=F, s=0.5)
        sd[p + "input_layernorm.weight"] = g(d)
        sd[p + "post_attention_layernorm.weight"] = g(d)
    sd["norm.weight"] = g(d)
    if not dims.tied:
        sd["lm_head.weight"] = w(dims.vocab, d, fan_in=d, s=3.0)
    return sd


def synthetic_adapter_state_dict(in_dim: int, d_model: int, hidden: int = 0, layers: int = 0, residual_scale: float = 0.1,
                                 seed: int = 0) -> Dict[str, np.ndarray]:
    """Seeded frame-adapter weights (QwenAudioSurgeryFrameAdapter) under the text engine's "adapter.*" names.  proj is
    not the identity (trained checkpoints move it away from the reference's init): a near-orthogonal [d_model][in_dim]
    matrix plus noise, so rows keep their scale."""
    rng = np.random.default_rng(seed)
    proj = rng.standard_normal((d_model, in_dim)) / np.sqrt(in_dim)
    if in_dim == d_model:
        proj = np.eye(d_model) + 0.5 * proj
    sd = {"adapter.proj.weight": proj.astype(np.float32)}
    for i in range(layers):
        p = f"adapter.blocks.{i}."
        sd[p + "norm.weight"] = (1.0 + 0.1 * rng.standard_normal(d_model)).astype(np.float32)
        sd[p + "mlp.gate.weight"] = (rng.standard_normal((hidden, d_model)) / np.sqrt(d_model)).astype(np.float32)
        sd[p + "mlp.up.weight"] = (rng.standard_normal((hidden, d_model)) / np.sqrt(d_model)).astype(np.float32)
        sd[p + "mlp.down.weight"] = (rng.standard_normal((d_model, hidden)) / np.sqrt(hidden)).astype(np.float32)
    if layers:
        sd["adapter.residual_scale"] = np.asarray([residual_scale], np.float32)
    return sd
