"""Drop-in for the reference's ``QwenAudioCausalKVEncoder`` (third_party/qwen3-asr-causal/src/qwen3_asr_causal/
causal.py:60-782) over the H100 tower engine.

The realtime model owns one encoder object and threads a per-stream state through it
(``audio_hidden, state.audio = self.audio_encoder.forward_chunk(mels, state.audio)``, causal.py:841;
``flush_pending`` :881; ``init_state`` model.py:804).  Here the state object is a handle on a device session:
mel buffering, per-layer K/V and positions live in the engine.  Integration is one assignment on the loaded model::

    model.audio_encoder = B200QwenAudioCausalKVEncoder.from_reference(model.audio_encoder, precision="bf16")

Needs torch only for the tensors that cross the seam (mels in, hidden out), as the reference does."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Optional

import numpy as np

from .qwen_dims import QwenTowerDims


@dataclass
class B200QwenAudioState:
    """Field-compatible with QwenAudioCausalKVState (causal.py:44-57) where callers read it."""
    sid: int
    engine: object = field(repr=False, default=None)
    frames_seen: int = 0
    emitted_steps: int = 0
    last_input_frames: int = 0
    last_recomputed_frames: int = 0
    last_recomputed_context_frames: int = 0
    pending_frames: int = 0
    mutable_steps: int = 0

    def close(self):
        if self.engine is not None:
            self.engine.close_session(self.sid)
            self.engine = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class B200QwenAudioCausalKVEncoder:
    def __init__(self, engine, dims: QwenTowerDims):
        self.engine, self.dims = engine, dims
        self.chunk_frames = dims.chunk_frames
        self.block_frames = dims.block_frames
        self.left_context_steps = dims.left_context_steps
        self.block_bidirectional = dims.block_bidirectional
        self.mutable_tail_steps = dims.mutable_tail_steps

    # -- construction from the reference object ----------------------------------------------------------
    @staticmethod
    def dims_of(ref_encoder) -> QwenTowerDims:
        t = ref_encoder.audio_tower
        layer = t.layers[0]
        return QwenTowerDims(
            n_mels=int(ref_encoder.config.n_mels), conv_channels=int(t.conv2d1.out_channels),
            d_model=int(t.conv_out.out_features), n_head=int(layer.self_attn.num_heads), n_layer=len(t.layers),
            ffn_dim=int(layer.fc1.out_features), out_dim=int(t.proj2.out_features),
            max_positions=int(t.positional_embedding.positional_embedding.shape[0]),
            chunk_frames=int(ref_encoder.chunk_frames), block_frames=int(ref_encoder.block_frames),
            left_context_steps=int(ref_encoder.left_context_steps), block_bidirectional=bool(ref_encoder.block_bidirectional),
            conv_out_bias=t.conv_out.bias is not None, mutable_tail_steps=int(getattr(ref_encoder, "mutable_tail_steps", 0)))

    @classmethod
    def from_reference(cls, ref_encoder, engine_factory=None, **engine_kw):
        """Pack the reference encoder's tower weights (its own state_dict names) into an engine."""
        dims = cls.dims_of(ref_encoder)
        sd = {k: v.detach().float().cpu().numpy() for k, v in ref_encoder.audio_tower.state_dict().items()}
        if engine_factory is None:
            from .qwen_engine import QwenTowerEngine
            engine_factory = QwenTowerEngine
        return cls(engine_factory(dims, sd, **engine_kw), dims)

    # -- the reference's surface ----------------------------------------------------------------------------
    @property
    def right_context_frames(self) -> int:
        return 0                                                           # causal.py:133-135

    def output_steps_for_mel_frames(self, mel_frames: int) -> int:
        return max(0, int(mel_frames)) // 8                                # causal.py:143-154 over lengths // 8

    def init_state(self) -> B200QwenAudioState:
        return B200QwenAudioState(sid=self.engine.open_session(), engine=self.engine)

    def _sync(self, state):
        state.emitted_steps = self.engine.emitted_steps(state.sid)
        state.pending_frames = self.engine.pending_frames(state.sid)
        state.mutable_steps = self.engine.mutable_steps(state.sid) if self.mutable_tail_steps else 0

    def forward_chunk(self, mels, state: Optional[B200QwenAudioState] = None):
        import torch
        if state is None:
            state = self.init_state()
        if mels.ndim != 3:
            raise ValueError("mels must have shape [batch, frames, n_mels]")
        if mels.shape[-1] != self.dims.n_mels:
            raise ValueError(f"expected {self.dims.n_mels} mel bins, got {mels.shape[-1]}")
        if mels.shape[0] != 1:
            raise ValueError("one stream per state: batch sessions through engine.forward_chunk")
        n = int(mels.shape[1])
        state.last_input_frames = n
        state.frames_seen += n
        before = self.engine.pending_frames(state.sid)
        tail_frames = state.mutable_steps * self.chunk_frames if n else 0     # causal.py:753-760: tail mels run again
        h = self.engine.forward_chunk([state.sid], [mels[0].detach().float().cpu().numpy()])[0]
        self._sync(state)
        state.last_recomputed_frames = tail_frames + before + n - state.pending_frames if n else 0
        state.last_recomputed_context_frames = tail_frames
        return torch.from_numpy(np.ascontiguousarray(h))[None].to(mels.device), state

    def flush_pending(self, state: B200QwenAudioState):
        import torch
        before = self.engine.pending_frames(state.sid)
        h = self.engine.flush_pending([state.sid])[0]
        self._sync(state)
        state.last_recomputed_frames = before // self.chunk_frames * self.chunk_frames
        state.last_recomputed_context_frames = 0
        return torch.from_numpy(np.ascontiguousarray(h))[None], state

    def forward_full(self, mels):
        state = self.init_state()
        try:
            consume = self.block_frames if self.block_frames > 0 else self.chunk_frames
            if int(mels.shape[1]) % consume:
                raise ValueError("forward_full expects whole blocks")
            return self.forward_chunk(mels, state)[0]
        finally:
            state.close()


class B200StreamingMelExtractor:
    """Drop-in for the reference's ``StreamingMelExtractor`` (features.py:32-112) bound to one engine session: the
    sample window and the featurization live on the device (``wlk_qwen_append_audio``).  On the reference's host path
    one ``append`` costs 170-350 ms of numpy per 0.25 s chunk (measured in the build container), which caps a CPU core
    below two real-time streams; here it is one small launch pair per batch of streams."""

    def __init__(self, engine, sid: int, sample_rate: int = 16_000):
        self.engine, self.sid, self.sample_rate = engine, sid, sample_rate
        self._emitted = 0

    @property
    def emitted_frames(self) -> int:
        return self._emitted

    def _wrap(self, m):
        import torch
        self._emitted += int(m.shape[0])
        return None if m.shape[0] == 0 else torch.from_numpy(m)[None]          # [1, frames, n_mels] like the reference

    def append(self, audio):
        return self._wrap(self.engine.mel_append([self.sid], [np.asarray(audio, np.float32)])[0])

    def flush(self):
        return self._wrap(self.engine.mel_flush([self.sid])[0])

    def reset(self) -> None:
        self.engine.reset_session(self.sid)
        self._emitted = 0
