#!/usr/bin/env python
"""Build container only: golden fixtures for the Qwen3-ASR causal audio tower, produced by the REFERENCE itself.

The reference's QwenAudioCausalKVEncoder (third_party/qwen3-asr-causal/src/qwen3_asr_causal/causal.py) duck-types the
audio tower (conv2d1-3, conv_out, positional_embedding, layers[i].{self_attn, *_layer_norm, fc1, fc2}, ln_post, proj1,
act, proj2).  Here a tower module of the requested geometry is filled with the seeded weights of
whisperlivekit_b200.qwen_dims.synthetic_tower_state_dict and driven, unchanged, through forward_chunk with a ragged
chunk schedule; sampled outputs and the complete state trace go to tests/golden/qwen_<name>.npz.

    python oracle/make_golden_qwen.py            # writes tests/golden/qwen_qnano.npz, qwen_qnano-chunk.npz
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))   # the staged reference holds qwen3_asr_causal

from whisperlivekit_b200.qwen_dims import QWEN_DIMS, synthetic_tower_state_dict  # noqa: E402


class _Attn(torch.nn.Module):
    def __init__(self, d, h):
        super().__init__()
        self.num_heads, self.head_dim = h, d // h
        self.scaling = self.head_dim ** -0.5
        self.attention_dropout = 0.0
        self.q_proj, self.k_proj = torch.nn.Linear(d, d), torch.nn.Linear(d, d)
        self.v_proj, self.out_proj = torch.nn.Linear(d, d), torch.nn.Linear(d, d)


class _Layer(torch.nn.Module):
    def __init__(self, d, h, f):
        super().__init__()
        self.self_attn = _Attn(d, h)
        self.self_attn_layer_norm, self.final_layer_norm = torch.nn.LayerNorm(d), torch.nn.LayerNorm(d)
        self.fc1, self.fc2 = torch.nn.Linear(d, f), torch.nn.Linear(f, d)
        self.activation_fn = torch.nn.GELU()
        self.dropout = self.activation_dropout = 0.0


class _Pos(torch.nn.Module):
    def __init__(self, table):
        super().__init__()
        self.register_buffer("positional_embedding", table)


class GeometryTower(torch.nn.Module):
    """A tower with the attribute names the reference encoder reads, at arbitrary dims."""

    def __init__(self, dims, sd):
        super().__init__()
        C = dims.conv_channels
        self.conv2d1 = torch.nn.Conv2d(1, C, 3, stride=2, padding=1)
        self.conv2d2 = torch.nn.Conv2d(C, C, 3, stride=2, padding=1)
        self.conv2d3 = torch.nn.Conv2d(C, C, 3, stride=2, padding=1)
        self.conv_out = torch.nn.Linear(dims.conv_features, dims.d_model, bias=dims.conv_out_bias)
        self.positional_embedding = _Pos(torch.from_numpy(sd["positional_embedding.positional_embedding"]))
        self.layers = torch.nn.ModuleList([_Layer(dims.d_model, dims.n_head, dims.ffn_dim) for _ in range(dims.n_layer)])
        self.ln_post = torch.nn.LayerNorm(dims.d_model)
        self.proj1 = torch.nn.Linear(dims.d_model, dims.d_model)
        self.act = torch.nn.GELU()
        self.proj2 = torch.nn.Linear(dims.d_model, dims.out_dim)
        missing, unexpected = self.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=False)
        assert not unexpected and not missing, (missing, unexpected)

    def _get_feat_extract_output_lengths(self, lengths):
        return lengths // 8


def reference_encoder(dims, sd):
    from qwen3_asr_causal.causal import QwenAudioCausalKVEncoder
    from qwen3_asr_causal.config import RealtimeAudioConfig
    cfg = RealtimeAudioConfig(d_model=dims.out_dim, qwen_audio_block_bidirectional=dims.block_bidirectional,
                              qwen_audio_block_frames=dims.block_frames,
                              qwen_audio_left_context_sec=dims.left_context_steps * 0.08,
                              qwen_audio_mutable_tail_sec=dims.mutable_tail_steps * 0.08)
    enc = QwenAudioCausalKVEncoder(GeometryTower(dims, sd).eval(), cfg).eval()
    assert enc.left_context_steps == dims.left_context_steps, (enc.left_context_steps, dims.left_context_steps)
    assert enc.mutable_tail_steps == dims.mutable_tail_steps, (enc.mutable_tail_steps, dims.mutable_tail_steps)
    return enc


def mel_stream(n_frames, n_mels=128, seed=0):
    """Log-mel-like values in the range Whisper features live in ([-1, 1.5], smooth along time)."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n_frames + 8, n_mels)).astype(np.float32)
    x = np.stack([x[i: i + n_frames] for i in range(8)]).mean(0) * 1.4          # temporal smoothing
    return np.clip(0.3 + x, -1.0, 1.5).astype(np.float32)


# frames per append: sub-chunk, exact blocks, several blocks at once, empty
SCHEDULE = [25, 25, 7, 135, 0, 192, 400, 1, 183, 96, 600, 25]


TAIL_SCHEDULE = [25, 25, 7, 135, 0, 192, 400, 1, 183, 96, 25, 3, 64, 25]


def main():
    out_dir = os.path.join(ROOT, "tests", "golden")
    for name in ("qnano", "qnano-chunk", "qnano-tail", "qnano-tail-bidir"):
        dims = QWEN_DIMS[name]
        sd = synthetic_tower_state_dict(dims, seed=11)
        enc = reference_encoder(dims, sd)
        # a mutable tail re-encodes tail + new steps in ONE piece: appends stay below the engine's 128 steps per call
        schedule = SCHEDULE if dims.mutable_tail_steps == 0 else TAIL_SCHEDULE
        mels = mel_stream(sum(schedule), dims.n_mels, seed=3)
        state = enc.init_state()
        rec = dict(schedule=np.asarray(schedule, np.int64))
        a = 0
        with torch.no_grad():
            for i, n in enumerate(schedule):
                hidden, state = enc.forward_chunk(torch.from_numpy(mels[a: a + n])[None], state)
                a += n
                h = hidden[0].numpy()
                rec[f"steps{i}"] = np.asarray(h.shape[0], np.int64)
                rec[f"emitted{i}"] = np.asarray(state.emitted_steps, np.int64)
                rec[f"pending{i}"] = np.asarray(state.pending_frames, np.int64)
                rec[f"mutable{i}"] = np.asarray(state.mutable_steps, np.int64)
                rec[f"cache_len{i}"] = np.asarray(0 if state.layer_caches[0].key is None else state.layer_caches[0].key.shape[-2], np.int64)
                if h.size:
                    flat = h.reshape(-1)
                    idx = np.arange(0, flat.shape[0], max(1, flat.shape[0] // 509), dtype=np.int64)
                    rec[f"idx{i}"], rec[f"val{i}"] = idx, flat[idx].astype(np.float32)
                    rec[f"rowsum{i}"] = h.astype(np.float64).sum(axis=1).astype(np.float32)
            hidden, state = enc.flush_pending(state)                      # end of stream (causal.py:687-711)
            h = hidden[0].numpy()
            rec["flush_steps"] = np.asarray(h.shape[0], np.int64)
            rec["flush_emitted"] = np.asarray(state.emitted_steps, np.int64)
            if h.size:
                rec["flush_rowsum"] = h.astype(np.float64).sum(axis=1).astype(np.float32)
                rec["flush_first_row"] = h[0].astype(np.float32)
        np.savez_compressed(os.path.join(out_dir, f"qwen_{name}.npz"), **rec)
        print(name, "emitted", state.emitted_steps, "pending", state.pending_frames, "std", float(np.std(h)))


if __name__ == "__main__":
    main()
