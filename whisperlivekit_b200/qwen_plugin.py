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

from ._lib import pack
from .qwen_dims import QwenTowerDims


class _SessionHandle:
    """An engine session (``sid`` on ``engine``) that closes once, on close() or when the object is collected."""

    def close(self):
        if self.engine is not None:
            self.engine.close_session(self.sid)
            self.engine = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _check_mels(mels, n_mels: int):
    if mels.ndim != 3:
        raise ValueError("mels must have shape [batch, frames, n_mels]")
    if mels.shape[-1] != n_mels:
        raise ValueError(f"expected {n_mels} mel bins, got {mels.shape[-1]}")
    if mels.shape[0] != 1:
        raise ValueError("one stream per state: batch sessions through encode_rows")


def _host_rows(hs, out_dim: int):
    """Per-stream host rows -> (CPU tensor [total, out_dim], row offsets [N + 1])."""
    import torch
    flat, offs = pack(hs, np.float32, (out_dim,), np.int64)
    return torch.from_numpy(flat[:offs[-1]]), offs


@dataclass
class B200QwenAudioState(_SessionHandle):
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

    @property
    def mel_buffer(self):
        """The session's pending mel frames [1, frames, n_mels] (None when there are none).  Assigning loads frames into
        the session, which is how the reference's segment rollover carries them into a fresh encoder state."""
        if self.engine is None:
            return None
        m = self.engine.get_pending(self.sid)
        if m.shape[0] == 0:
            return None
        import torch
        return torch.from_numpy(np.ascontiguousarray(m))[None]

    @mel_buffer.setter
    def mel_buffer(self, value):
        if value is None:
            m = np.zeros((0, 1), np.float32)
        else:
            if value.ndim != 3 or value.shape[0] != 1:
                raise ValueError("mel_buffer must have shape [1, frames, n_mels]")
            m = value[0].detach().float().cpu().numpy() if hasattr(value, "detach") else np.asarray(value[0], np.float32)
        self.engine.set_pending(self.sid, m)      # like the reference, pending_frames follows at the next forward_chunk


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

    def encode_rows(self, states, mels=None, flush: bool = False, device_rows: bool = True):
        """forward_chunk (flush=False, mels [1, frames, n_mels] per state) or flush_pending (flush=True) for N states in
        one engine call, with each state's fields updated as those two methods do.  Returns (rows [total, out_dim],
        row offsets [N + 1]): a CUDA tensor when the engine runs on the device and device_rows is set, else a CPU
        tensor."""
        if flush:
            before = [self.engine.pending_frames(s.sid) for s in states]
            sids = [s.sid for s in states]
            dev = device_rows and hasattr(self.engine, "flush_pending_device")
            if dev:
                rows, offs = self.engine.flush_pending_device(sids)
            else:
                hs = self.engine.flush_pending(sids)
        else:
            for m in mels:
                _check_mels(m, self.dims.n_mels)
            ns = [int(m.shape[1]) for m in mels]
            for st, n in zip(states, ns):
                st.last_input_frames = n
                st.frames_seen += n
            before = [self.engine.pending_frames(s.sid) for s in states]
            tails = [st.mutable_steps * self.chunk_frames if n else 0 for st, n in zip(states, ns)]  # causal.py:753-760
            sids = [s.sid for s in states]
            host = [m[0].detach().float().cpu().numpy() for m in mels]
            dev = device_rows and hasattr(self.engine, "forward_chunk_device")
            if dev:
                rows, offs = self.engine.forward_chunk_device(sids, host)
            else:
                hs = self.engine.forward_chunk(sids, host)
        if not dev:
            rows, offs = _host_rows(hs, self.dims.out_dim)
        for i, st in enumerate(states):
            self._sync(st)
            if flush:
                st.last_recomputed_frames = before[i] // self.chunk_frames * self.chunk_frames
                st.last_recomputed_context_frames = 0
            else:
                n = ns[i]
                st.last_recomputed_frames = tails[i] + before[i] + n - st.pending_frames if n else 0
                st.last_recomputed_context_frames = tails[i]
        return rows, [int(o) for o in offs]

    def forward_chunk(self, mels, state: Optional[B200QwenAudioState] = None):
        if state is None:
            state = self.init_state()
        rows, _ = self.encode_rows([state], [mels], device_rows=False)
        return rows[None].to(mels.device), state

    def flush_pending(self, state: B200QwenAudioState):
        rows, _ = self.encode_rows([state], flush=True, device_rows=False)
        return rows[None], state

    def forward_full(self, mels):
        state = self.init_state()
        try:
            consume = self.block_frames if self.block_frames > 0 else self.chunk_frames
            if int(mels.shape[1]) % consume:
                raise ValueError("forward_full expects whole blocks")
            return self.forward_chunk(mels, state)[0]
        finally:
            state.close()


@dataclass
class B200QwenWindowState(_SessionHandle):
    """Field-compatible with QwenAudioSurgeryState (reference model.py:36-43) where callers read it; the mel window
    itself lives on the device."""
    sid: int
    engine: object = field(repr=False, default=None)
    frames_seen: int = 0
    window_start_frame: int = 0
    emitted_steps: int = 0
    last_input_frames: int = 0
    last_recomputed_frames: int = 0
    last_recomputed_context_frames: int = 0


class B200QwenAudioSurgeryEncoder:
    """Drop-in for the reference's windowed ``QwenAudioSurgeryEncoder`` (model.py:441-608) over the windowed tower
    engine.  Nothing is ever re-computable after it is emitted, so ``mutable_tail_steps`` is 0 and ``encode_rows`` has
    the causal drop-in's contract.  The windowed model has no flush: end of stream is right_context_frames of zeros
    through forward_chunk, as the reference streamer does it."""

    mutable_tail_steps = 0

    def __init__(self, engine, dims):
        self.engine, self.dims = engine, dims
        self.left_context_frames = dims.left_context_frames
        self.right_context_frames = dims.right_context_frames

    @property
    def max_recompute_frames(self) -> int:
        return self.left_context_frames + self.right_context_frames

    @staticmethod
    def tower_uses_attention_blocks(tower) -> bool:
        """Whether the stock tower's n_window_infer blocks take effect.  The tower hands its layers only cu_seqlens
        (transformers 5.5 modeling_qwen3_omni_moe.py:753-762), and only flash-attention implementations read them:
        eager and SDPA attend over the whole window.  Decided as transformers decides it for the same tower
        (``is_flash_attention_requested(config)``, which it uses in ``_prepare_attention_mask``).  A custom
        registered varlen implementation cannot be recognised from its name: pass ``attention_blocks=True``."""
        cfg = getattr(tower, "config", None)
        if cfg is None:
            return False
        try:
            from transformers.utils.generic import is_flash_attention_requested
        except ImportError:
            return "flash" in str(getattr(cfg, "_attn_implementation", "") or "")
        return bool(is_flash_attention_requested(cfg))

    @classmethod
    def dims_of(cls, ref_encoder, attention_blocks: Optional[bool] = None):
        """The window geometry of an installed reference encoder.  attention_blocks None: decided from the tower's
        attention implementation (tower_uses_attention_blocks); False keeps one block over the window (n_window_infer
        0); True keeps the tower's n_window_infer."""
        from .qwen_dims import QwenWindowDims
        t = ref_encoder.audio_tower
        layer = t.layers[0]
        cfg = getattr(t, "config", None)
        if attention_blocks is None:
            attention_blocks = cls.tower_uses_attention_blocks(t)
        n_window = int(getattr(t, "n_window", getattr(cfg, "n_window", 50)))
        infer = int(getattr(t, "n_window_infer", getattr(cfg, "n_window_infer", 0)) or 0)
        return QwenWindowDims(
            n_mels=int(ref_encoder.config.n_mels), conv_channels=int(t.conv2d1.out_channels),
            d_model=int(t.conv_out.out_features), n_head=int(layer.self_attn.num_heads), n_layer=len(t.layers),
            ffn_dim=int(layer.fc1.out_features), out_dim=int(t.proj2.out_features),
            max_positions=int(t.positional_embedding.positional_embedding.shape[0]),
            conv_out_bias=t.conv_out.bias is not None, n_window=n_window,
            n_window_infer=infer if attention_blocks else 0,
            left_context_frames=int(ref_encoder.left_context_frames), right_context_frames=int(ref_encoder.right_context_frames))

    @classmethod
    def from_reference(cls, ref_encoder, engine_factory=None, attention_blocks: Optional[bool] = None, **engine_kw):
        """Pack the reference tower's weights.  The positional table is a non-persistent buffer, absent from
        state_dict(): the live buffer is packed.  attention_blocks as dims_of."""
        dims = cls.dims_of(ref_encoder, attention_blocks)
        t = ref_encoder.audio_tower
        sd = {k: v.detach().float().cpu().numpy() for k, v in t.state_dict().items()}
        sd["positional_embedding.positional_embedding"] = t.positional_embedding.positional_embedding.detach().float().cpu().numpy()
        if engine_factory is None:
            from .qwen_engine import QwenWindowEngine
            engine_factory = QwenWindowEngine
        return cls(engine_factory(dims, sd, **engine_kw), dims)

    def output_steps_for_mel_frames(self, mel_frames: int) -> int:
        from .qwen_dims import window_output_steps
        return window_output_steps(int(mel_frames))                       # model.py:514-524, the mod-100 rule

    def init_state(self) -> B200QwenWindowState:
        return B200QwenWindowState(sid=self.engine.open_session(), engine=self.engine)

    def encode_rows(self, states, mels, flush: bool = False, device_rows: bool = True):
        """forward_chunk for N states in one engine call, each state's fields updated as forward_chunk does.  Returns
        (rows [total, out_dim], row offsets [N + 1]): a CUDA tensor when the engine runs on the device and device_rows
        is set, else a CPU tensor."""
        if flush:
            raise ValueError("the windowed encoder has no flush: feed right_context_frames of zeros")
        for m in mels:
            _check_mels(m, self.dims.n_mels)
        sids = [s.sid for s in states]
        host = [m[0].detach().float().cpu().numpy() for m in mels]
        if device_rows and hasattr(self.engine, "forward_chunk_device"):
            rows, offs = self.engine.forward_chunk_device(sids, host)
        else:
            rows, offs = _host_rows(self.engine.forward_chunk(sids, host), self.dims.out_dim)
        for st in states:
            f = self.engine.state(st.sid)
            for k in ("frames_seen", "window_start_frame", "emitted_steps", "last_input_frames", "last_recomputed_frames",
                      "last_recomputed_context_frames"):
                setattr(st, k, f[k])
        return rows, [int(o) for o in offs]

    def forward_chunk(self, mels, state: Optional[B200QwenWindowState] = None):
        if state is None:
            state = self.init_state()
        _check_mels(mels, self.dims.n_mels)
        if mels.shape[1] == 0:                                             # model.py:568-570
            return mels.new_zeros(mels.shape[0], 0, self.dims.out_dim), state
        rows, _ = self.encode_rows([state], [mels], device_rows=False)
        return rows[None].to(mels.device), state

    def forward_full(self, mels):
        """The tower over each window of mels [batch, frames, n_mels] (model.py:526-557), zero-padded to the longest.
        Unlike the reference, a window may hold at most max_recompute_frames (left + right) frames: the engine's
        workspace and its attention blocks are sized for the streaming window."""
        import torch
        if mels.ndim != 3 or mels.shape[-1] != self.dims.n_mels:
            raise ValueError("mels must have shape [batch, frames, n_mels]")
        if mels.shape[1] > self.max_recompute_frames:
            raise ValueError(f"forward_full takes at most {self.max_recompute_frames} frames per window "
                             f"(left + right context), got {mels.shape[1]}")
        hs = self.engine.encode([m.detach().float().cpu().numpy() for m in mels])
        steps = max((h.shape[0] for h in hs), default=0)
        out = torch.zeros(len(hs), steps, self.dims.out_dim)
        for i, h in enumerate(hs):
            out[i, :h.shape[0]] = torch.from_numpy(h)
        return out.to(mels.device)


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


class B200DecoderRollingState(_SessionHandle):
    """Stands in for the reference's DecoderRollingState (model.py:53-68) in ``state.decoder``: the KV of
    [head + audio_steps] lives in an engine session, ``cache`` is that session's handle.  The session closes when the
    object is collected (segment rollover builds fresh decode states)."""

    disabled = False

    def __init__(self, engine, sid: int):
        self.engine, self.sid = engine, sid
        self.head_token_ids: tuple = ()
        self.head_len = 0
        self.audio_steps = 0

    @property
    def cache(self):
        return self if self.engine is not None else None

    def get_seq_length(self) -> int:
        return self.engine.session_len(self.sid)


class B200QwenTextDecoder:
    """Drop-in for the text half of the reference's realtime model: ``generate_full_hypothesis_rolling`` (model.py:
    991-1250) and ``generate_full_hypothesis_from_cached_audio`` (:839-989) rebound on one model instance over the text
    engine (``wlk_qtext_*``), the rolling prefix KV in a device session per stream::

        B200QwenTextDecoder.install(model, precision="bf16")

    Frame rows cross the seam as the host tensor the reference hands over; only the rows the session has not seen are
    uploaded.  ``use_decoder_kv_cache=False`` takes the same cached path (the reference documents the two as
    greedy-equal).  The non-rolling generate runs on scratch sessions the decoder keeps open between calls (``close``
    releases them)."""

    def __init__(self, model, engine, dims):
        self.model, self.engine, self.dims = model, engine, dims
        self._scratch: list = []

    @staticmethod
    def dims_of(model, max_ctx: int = 1024):
        from .qwen_dims import QwenTextDims
        c = model.text_model.config
        rope = getattr(c, "rope_parameters", None) or {}
        theta = rope.get("rope_theta", getattr(c, "rope_theta", 10000.0))
        tied = model.lm_head.weight.data_ptr() == model.text_model.embed_tokens.weight.data_ptr()
        return QwenTextDims(vocab=int(model.lm_head.weight.shape[0]), d_model=int(c.hidden_size),
                            n_layer=int(c.num_hidden_layers), n_head=int(c.num_attention_heads),
                            n_kv_head=int(c.num_key_value_heads),
                            head_dim=int(getattr(c, "head_dim", c.hidden_size // c.num_attention_heads)),
                            ffn_dim=int(c.intermediate_size), rope_theta=float(theta), rms_eps=float(c.rms_norm_eps),
                            tied=bool(tied), max_ctx=int(max_ctx))

    @classmethod
    def install(cls, model, engine_factory=None, precision: str = "bf16", max_ctx: int = 1024, max_sessions: int = 8,
                extra_tensors=None, **engine_kw):
        """extra_tensors: more named tensors for the engine, e.g. the frame adapter's (adapter_tensors)."""
        dims = cls.dims_of(model, max_ctx)
        sd = {k: v.detach().float().cpu().numpy() for k, v in model.text_model.state_dict().items()}
        sd.update(extra_tensors or {})
        rotary = getattr(model.text_model, "rotary_emb", None)
        if rotary is not None and getattr(rotary, "inv_freq", None) is not None:
            # the live buffer the model rotates with (non-persistent, so not in state_dict())
            sd["rotary_emb.inv_freq"] = rotary.inv_freq.detach().float().cpu().numpy()
        if not dims.tied:
            sd["lm_head.weight"] = model.lm_head.weight.detach().float().cpu().numpy()
        if engine_factory is None:
            from .qwen_text_engine import QwenTextEngine
            engine = QwenTextEngine(dims, sd, precision=precision, max_sessions=max_sessions, **engine_kw)
        else:
            engine = engine_factory(dims, sd)
        dec = cls(model, engine, dims)
        model.generate_full_hypothesis_rolling = dec.generate_full_hypothesis_rolling
        model.generate_full_hypothesis_from_cached_audio = dec.generate_full_hypothesis_from_cached_audio
        model.b200_text_decoder = dec
        return dec

    def _controls(self, eos_token_id, stop_token_ids, suppress_token_ids, repetition_penalty, no_repeat_ngram_size,
                  max_consecutive_text_tokens):
        return dict(eos_token_id=eos_token_id, stop_token_ids=stop_token_ids, suppress_token_ids=suppress_token_ids,
                    repetition_penalty=repetition_penalty, no_repeat_ngram_size=no_repeat_ngram_size,
                    max_consecutive_text_tokens=max_consecutive_text_tokens, wait_token_id=self.model.wait_token_id)

    def generate_full_hypothesis_from_cached_audio(self, frame_hidden, *, prefix_token_ids=None,
                                                   audio_placeholder_token_id=None, prompt_token_ids=None,
                                                   max_new_tokens: int = 128, eos_token_id=None, stop_token_ids=None,
                                                   suppress_token_ids=None, repetition_penalty: float = 1.0,
                                                   no_repeat_ngram_size: int = 0, max_consecutive_text_tokens: int = 0,
                                                   use_decoder_kv_cache: bool = True):
        import torch
        if frame_hidden.ndim != 3:
            raise ValueError("frame_hidden must have shape [batch, steps, hidden]")
        if max_new_tokens < 0:
            raise ValueError("max_new_tokens must be >= 0")
        batch = int(frame_hidden.shape[0])
        device = frame_hidden.device
        if max_new_tokens == 0:
            return torch.empty(batch, 0, dtype=torch.long, device=device)
        kw = self._controls(eos_token_id, stop_token_ids, suppress_token_ids, repetition_penalty, no_repeat_ngram_size,
                            max_consecutive_text_tokens)
        ctl = self.engine.make_controls(**kw)
        outs = self.full_tokens([frame_hidden[b] for b in range(batch)], token_rows(prefix_token_ids, batch),
                                token_rows(prompt_token_ids, batch), audio_placeholder_token_id, max_new_tokens, ctl)
        return padded_tokens(outs, ctl, device)

    def full_tokens(self, frame_rows, prefix_rows, prompt_rows, audio_placeholder_token_id, max_new_tokens: int, ctl):
        """The cached path's tokens per stream: frame_rows[b] [steps, d], prefix_rows[b] / prompt_rows[b] token lists or
        None.  Streams with an empty prefix get no tokens; the others run in one generate_full_batch (waves of
        max_batch)."""
        prefixes = [self.engine.full_prefix(self._rows(f), prefix_token_ids=p,
                                            audio_placeholder_token_id=audio_placeholder_token_id,
                                            prompt_token_ids=q, bos_token_id=self.model.bos_token_id)
                    for f, p, q in zip(frame_rows, prefix_rows, prompt_rows)]
        live = [b for b in range(len(prefixes)) if prefixes[b][0].shape[0]]
        outs = [[] for _ in prefixes]
        for b, toks in zip(live, self._generate_full([prefixes[b][1] for b in live], [prefixes[b][0] for b in live],
                                                     max_new_tokens, ctl)):
            outs[b] = toks
        return outs

    def _generate_full(self, frame_rows, srcs, max_new_tokens: int, ctl):
        """engine.generate_full_batch over the scratch sessions, in waves of the engine's max_batch."""
        n = len(srcs)
        if n == 0:
            return []
        wave = int(getattr(self.engine, "max_batch", 0) or n)
        while len(self._scratch) < min(n, wave):
            self._scratch.append(self.engine.open_session())
        out = []
        for a in range(0, n, wave):
            k = min(wave, n - a)
            out += self.engine.generate_full_batch(self._scratch[:k], frame_rows[a: a + k], srcs[a: a + k],
                                                   max_new_tokens=max_new_tokens, controls=ctl)
        return out

    def generate_full_batch(self, frame_rows, prefix_token_ids, *, audio_placeholder_token_id, max_new_tokens: int = 128,
                            **controls):
        """generate_full_hypothesis_from_cached_audio for N streams in one lockstep pass (the windowed tick):
        frame_rows[i] [steps_i, d] (a CUDA tensor stays on the device), prefix_token_ids[i] the stream's prompt with one
        audio placeholder per frame row.  controls: the generate method's decode controls plus wait_token_id.  N above
        the engine's max_batch runs in waves.  Returns the tokens per stream."""
        if max_new_tokens < 0:
            raise ValueError("max_new_tokens must be >= 0")
        controls.setdefault("wait_token_id", self.model.wait_token_id)
        ctl = self.engine.make_controls(**controls)
        prefixes = [self.engine.full_prefix(self._rows(f), prefix_token_ids=p,
                                            audio_placeholder_token_id=audio_placeholder_token_id)
                    for f, p in zip(frame_rows, prefix_token_ids)]
        if max_new_tokens == 0:
            return [[] for _ in prefixes]
        return self._generate_full([fh for _, fh in prefixes], [src for src, _ in prefixes], max_new_tokens, ctl)

    def close(self) -> None:
        """Close the scratch sessions of the non-rolling generate."""
        while self._scratch:
            self.engine.close_session(self._scratch.pop())

    def _rows(self, frame_hidden):
        """CUDA frame rows stay on the device when the engine reads device rows; otherwise they go to the host."""
        fh = frame_hidden.detach().float()
        return fh if fh.is_cuda and getattr(self.engine, "device_rows", False) else fh.cpu().numpy()

    def generate_full_hypothesis_rolling(self, frame_hidden, *, state, template_token_ids, audio_placeholder_token_id,
                                         draft_token_ids=None, max_new_tokens: int = 128, eos_token_id=None,
                                         stop_token_ids=None, suppress_token_ids=None, repetition_penalty: float = 1.0,
                                         no_repeat_ngram_size: int = 0, max_consecutive_text_tokens: int = 0):
        import torch
        from .qwen_text_engine import split_template
        if frame_hidden.ndim != 3:
            raise ValueError("frame_hidden must have shape [batch, steps, hidden]")
        head, tail = split_template(template_token_ids, audio_placeholder_token_id)
        kw = self._controls(eos_token_id, stop_token_ids, suppress_token_ids, repetition_penalty, no_repeat_ngram_size,
                            max_consecutive_text_tokens)
        audio_steps = int(frame_hidden.shape[1])
        if int(frame_hidden.shape[0]) != 1 or max_new_tokens <= 0 or audio_steps == 0:
            expanded = head + [int(audio_placeholder_token_id)] * audio_steps + tail
            toks = self.generate_full_hypothesis_from_cached_audio(
                frame_hidden, prefix_token_ids=expanded, audio_placeholder_token_id=audio_placeholder_token_id,
                max_new_tokens=max_new_tokens, **{k: v for k, v in kw.items() if k != "wait_token_id"})
            return toks, {"decoder_path": "full"}
        toks, stats = self.generate_rolling_batch(
            [frame_hidden[0]], [state], [draft_token_ids], template_token_ids=template_token_ids,
            audio_placeholder_token_id=audio_placeholder_token_id, max_new_tokens=max_new_tokens, **kw)
        return torch.tensor([toks[0]], dtype=torch.long, device=frame_hidden.device), stats[0]

    def generate_rolling_batch(self, frame_rows, states, drafts, *, template_token_ids, audio_placeholder_token_id,
                               max_new_tokens: int = 128, **controls):
        """generate_full_hypothesis_rolling for N streams in one lockstep pass: frame_rows[i] [steps_i, d] (the
        stream's whole frame_hidden; only the rows its decoder session has not seen are forwarded), states[i] the
        stream's CachedAudioDecodeState (its ``decoder`` is read and set), drafts[i] a token list or None.  controls:
        the generate method's decode controls plus wait_token_id.  Returns (tokens per stream, stats per stream)."""
        from .qwen_text_engine import RollingState
        decs, prevs = [], []
        for state in states:
            dec = getattr(state, "decoder", None)
            if not isinstance(dec, B200DecoderRollingState) or dec.engine is not self.engine:
                dec = B200DecoderRollingState(self.engine, self.engine.open_session())
                prevs.append(None)
            else:
                prevs.append(RollingState(dec.head_token_ids, dec.head_len, dec.audio_steps))
            decs.append(dec)
        controls.setdefault("wait_token_id", self.model.wait_token_id)
        toks, stats, new = self.engine.generate_rolling_batch(
            [d.sid for d in decs], [self._rows(f) for f in frame_rows], prevs, template_token_ids,
            audio_placeholder_token_id, [None if d is None else [int(t) for t in d] for d in drafts],
            max_new_tokens=max_new_tokens, bos_token_id=self.model.bos_token_id, scratch=self._scratch, **controls)
        for dec, state, st, s in zip(decs, states, new, stats):
            if s.get("decoder_path") != "full":
                dec.head_token_ids, dec.head_len, dec.audio_steps = st.head_token_ids, st.head_len, st.audio_steps
                state.decoder = dec
        return toks, stats


def token_rows(ids, batch: int):
    """A generate method's prefix_token_ids / prompt_token_ids ([steps] shared, or [batch, steps]) as one list per row."""
    if ids is None:
        return [None] * batch
    import torch
    t = torch.as_tensor(ids).long()
    return [(t if t.ndim == 1 else t[b]).tolist() for b in range(batch)]


def padded_tokens(outs, ctl, device):
    """Tokens per row -> the reference's [batch, width] long tensor: rows that stopped early are filled with the
    stop-fill id while the others decode (model.py:419-436)."""
    import torch
    width = max(len(o) for o in outs)
    if ctl.stop_ids:
        fill = ctl.eos_token_id if ctl.eos_token_id is not None else min(ctl.stop_ids)
        outs = [o + [fill] * (width - len(o)) for o in outs]
    return torch.tensor(outs, dtype=torch.long, device=device).reshape(len(outs), width)


def adapter_tensors(adapter) -> dict:
    """The reference frame adapter (QwenAudioSurgeryFrameAdapter, model.py:631-691) as the text engine's "adapter.*"
    tensors.  residual_scale is a plain float on each block, the same for all of them; dropout is off in eval."""
    sd = {"adapter.proj.weight": adapter.proj.weight.detach().float().cpu().numpy()}
    scales = {float(b.residual_scale) for b in adapter.blocks}
    if len(scales) > 1:
        raise ValueError("the adapter's blocks have different residual scales")
    for i, b in enumerate(adapter.blocks):
        p = f"adapter.blocks.{i}."
        sd[p + "norm.weight"] = b.norm.weight.detach().float().cpu().numpy()
        for n in ("gate", "up", "down"):
            sd[p + f"mlp.{n}.weight"] = getattr(b.mlp, n).weight.detach().float().cpu().numpy()
    if scales:
        sd["adapter.residual_scale"] = np.asarray([scales.pop()], np.float32)
    return sd


def _is_window_encoder(encoder) -> bool:
    """Whether a reference audio encoder is the windowed QwenAudioSurgeryEncoder (model.py:441-608)."""
    return any(c.__name__ == "QwenAudioSurgeryEncoder" for c in type(encoder).__mro__)


class B200QwenRealtimeModel:
    """The whole realtime model on the engines, installed on one instance::

        B200QwenRealtimeModel.install(model, precision="bf16")

    Either backend of the reference: the causal ``Qwen3ASRRealtimeQwenAudioCausalModel`` or the windowed
    ``Qwen3ASRRealtimeQwenAudioSurgeryModel`` (model.py:1421-1509), told apart by ``model.audio_encoder``.  Install
    replaces ``model.audio_encoder`` with the matching tower drop-in, installs the text decoder drop-in with the frame
    adapter packed into its engine, and rebinds ``append_audio_to_cache`` onto ``qwen_realtime.RealtimeFrames``
    (N = 1), plus ``flush_audio_to_cache`` for the causal model only: the windowed model has none, so the streamer's
    ``flush_pending_audio`` returns None as in the reference.  With CUDA engines ``state.frame_hidden`` is a device
    tensor and the generate methods read it in place: no frame row reaches the host.  The reference streamers
    (``SegmentedCachedFullHypothesisStreamer``) run over the installed model unchanged.

    ``batching=True`` serves many sessions, each driven from its own thread, in shared engine calls: the four seam
    methods submit to a ``batching.BatchingEngine`` whose dispatcher thread merges concurrent calls of one kind and equal
    static arguments (template, placeholder id, max_new_tokens, decode controls) into one call of
    ``RealtimeFrames.append`` (appends and flushes apart), ``generate_rolling_batch`` or the cached path's batch.  While
    it is on, the dispatcher thread is the only caller of the engines' compute; callers only open, close and read their
    sessions.  Bracket each caller's iteration (one ``process_iter``) with ``batcher.begin_iter()`` /
    ``batcher.end_iter()`` (``plugin.install_qwen_cohorts`` does it for ``Qwen3StreamingOnlineProcessor``) so that a
    cohort's appends and generates land in the same merged calls.  A merged call that fails is replayed one caller at
    a time, so an error reaches only the caller whose session caused it.  ``close()`` stops the dispatcher."""

    def __init__(self, model, encoder, decoder):
        from .qwen_realtime import RealtimeFrames
        self.model, self.encoder, self.decoder = model, encoder, decoder
        self.frames = RealtimeFrames(encoder, decoder.engine, decoder.dims.d_model)
        self.batcher = None

    @classmethod
    def install(cls, model, precision: str = "bf16", max_ctx: int = 1024, max_sessions: int = 8, tower_factory=None,
                text_factory=None, attention_blocks: Optional[bool] = None, batching: bool = False,
                max_batch: Optional[int] = None, max_wait_s: float = 0.002):
        """tower_factory(dims, state_dict) / text_factory(dims, state_dict): engines to use instead of the CUDA ones
        (the CPU oracles in tests).  attention_blocks: the windowed tower's, as B200QwenAudioSurgeryEncoder.dims_of.
        max_batch: sessions per call of both CUDA engines (their default, 8, when None).  batching: coalesce
        concurrent seam calls (see the class docstring), at most as many sessions per merged call as the smaller of the
        two engines' max_batch, so that no merged call exceeds what the engines take.  Size max_sessions for every
        stream's tower and decoder session plus max_batch scratch sessions of the non-rolling generate."""
        engine_kw = {} if max_batch is None else dict(max_batch=int(max_batch))
        tower_kw = {} if tower_factory else dict(precision=precision, max_sessions=max_sessions, **engine_kw)
        windowed = _is_window_encoder(model.audio_encoder)
        if windowed:
            encoder = B200QwenAudioSurgeryEncoder.from_reference(model.audio_encoder, engine_factory=tower_factory,
                                                                 attention_blocks=attention_blocks, **tower_kw)
        else:
            encoder = B200QwenAudioCausalKVEncoder.from_reference(model.audio_encoder, engine_factory=tower_factory,
                                                                  **tower_kw)
        if encoder.dims.out_dim != model.adapter.proj.weight.shape[1]:
            raise ValueError(f"tower rows are {encoder.dims.out_dim} wide, the adapter takes "
                             f"{model.adapter.proj.weight.shape[1]}")
        decoder = B200QwenTextDecoder.install(model, engine_factory=text_factory, precision=precision, max_ctx=max_ctx,
                                              max_sessions=max_sessions, extra_tensors=adapter_tensors(model.adapter),
                                              **engine_kw)
        rt = cls(model, encoder, decoder)
        if "audio_encoder" in getattr(model, "_modules", {}):
            del model._modules["audio_encoder"]        # an nn.Module takes only modules as child attributes
        model.audio_encoder = encoder
        model.append_audio_to_cache = rt.append_audio_to_cache
        if not windowed:
            model.flush_audio_to_cache = rt.flush_audio_to_cache
        if batching:
            from .batching import BatchingEngine
            caps = [int(e.max_batch) for e in (encoder.engine, decoder.engine) if getattr(e, "max_batch", None)]
            cap = min(caps) if caps else (max_batch or 64)        # the CPU oracles take any batch
            rt.batcher = BatchingEngine(_RealtimeOps(rt), max_batch=min(cap, max_batch or cap), max_wait_s=max_wait_s)
            model.generate_full_hypothesis_rolling = rt.generate_full_hypothesis_rolling
            model.generate_full_hypothesis_from_cached_audio = rt.generate_full_hypothesis_from_cached_audio
        model.b200_realtime = rt
        return rt

    def append_audio_to_cache(self, mels, state=None):
        if state is None:
            state = self.model.init_cached_audio_decode_state()
        if self.batcher is not None:
            (cached, delta), = self.batcher.submit("append_audio_to_cache", [state], [mels]).result()
        else:
            (cached, delta), = self.frames.append([state], [mels])
        return cached, delta, state

    def flush_audio_to_cache(self, state=None):
        if state is None:
            state = self.model.init_cached_audio_decode_state()
        if self.batcher is not None:
            (cached, delta), = self.batcher.submit("flush_audio_to_cache", [state]).result()
        else:
            (cached, delta), = self.frames.append([state], flush=True)
        return cached, delta, state

    # -- the generate methods with batching on (without it they are B200QwenTextDecoder's) -------------------------
    def _controls(self, eos_token_id, stop_token_ids, suppress_token_ids, repetition_penalty, no_repeat_ngram_size,
                  max_consecutive_text_tokens):
        """The decode controls as a merge key: hashable, equal when the decoder would build equal controls."""
        return dict(eos_token_id=None if eos_token_id is None else int(eos_token_id),
                    stop_token_ids=None if stop_token_ids is None else tuple(int(t) for t in stop_token_ids),
                    suppress_token_ids=None if suppress_token_ids is None else tuple(int(t) for t in suppress_token_ids),
                    repetition_penalty=float(repetition_penalty), no_repeat_ngram_size=int(no_repeat_ngram_size),
                    max_consecutive_text_tokens=int(max_consecutive_text_tokens))

    def generate_full_hypothesis_from_cached_audio(self, frame_hidden, *, prefix_token_ids=None,
                                                   audio_placeholder_token_id=None, prompt_token_ids=None,
                                                   max_new_tokens: int = 128, eos_token_id=None, stop_token_ids=None,
                                                   suppress_token_ids=None, repetition_penalty: float = 1.0,
                                                   no_repeat_ngram_size: int = 0, max_consecutive_text_tokens: int = 0,
                                                   use_decoder_kv_cache: bool = True):
        import torch
        if frame_hidden.ndim != 3:
            raise ValueError("frame_hidden must have shape [batch, steps, hidden]")
        if max_new_tokens < 0:
            raise ValueError("max_new_tokens must be >= 0")
        batch = int(frame_hidden.shape[0])
        if max_new_tokens == 0:
            return torch.empty(batch, 0, dtype=torch.long, device=frame_hidden.device)
        kw = self._controls(eos_token_id, stop_token_ids, suppress_token_ids, repetition_penalty, no_repeat_ngram_size,
                            max_consecutive_text_tokens)
        items = list(zip([frame_hidden[b] for b in range(batch)], token_rows(prefix_token_ids, batch),
                         token_rows(prompt_token_ids, batch)))
        outs = self.batcher.submit("generate_full_hypothesis_from_cached_audio", [object() for _ in items], items,
                                   audio_placeholder_token_id=audio_placeholder_token_id,
                                   max_new_tokens=int(max_new_tokens), **kw).result()
        return padded_tokens(outs, self.decoder.engine.make_controls(**kw), frame_hidden.device)

    def generate_full_hypothesis_rolling(self, frame_hidden, *, state, template_token_ids, audio_placeholder_token_id,
                                         draft_token_ids=None, max_new_tokens: int = 128, eos_token_id=None,
                                         stop_token_ids=None, suppress_token_ids=None, repetition_penalty: float = 1.0,
                                         no_repeat_ngram_size: int = 0, max_consecutive_text_tokens: int = 0):
        import torch
        from .qwen_text_engine import split_template
        if frame_hidden.ndim != 3:
            raise ValueError("frame_hidden must have shape [batch, steps, hidden]")
        head, tail = split_template(template_token_ids, audio_placeholder_token_id)
        kw = self._controls(eos_token_id, stop_token_ids, suppress_token_ids, repetition_penalty, no_repeat_ngram_size,
                            max_consecutive_text_tokens)
        audio_steps = int(frame_hidden.shape[1])
        if int(frame_hidden.shape[0]) != 1 or max_new_tokens <= 0 or audio_steps == 0:
            expanded = head + [int(audio_placeholder_token_id)] * audio_steps + tail
            toks = self.generate_full_hypothesis_from_cached_audio(
                frame_hidden, prefix_token_ids=expanded, audio_placeholder_token_id=audio_placeholder_token_id,
                max_new_tokens=max_new_tokens, **kw)
            return toks, {"decoder_path": "full"}
        draft = None if draft_token_ids is None else [int(t) for t in draft_token_ids]
        (toks, stats), = self.batcher.submit(
            "generate_full_hypothesis_rolling", [state], [(frame_hidden[0], draft)],
            template_token_ids=tuple(int(t) for t in template_token_ids),
            audio_placeholder_token_id=int(audio_placeholder_token_id), max_new_tokens=int(max_new_tokens), **kw).result()
        return torch.tensor([toks], dtype=torch.long, device=frame_hidden.device), stats

    def close(self) -> None:
        """Stop the dispatcher of batching=True (pending calls fail)."""
        if self.batcher is not None:
            self.batcher.close()


class _RealtimeOps:
    """The realtime model's seam calls in the batch form BatchingEngine's dispatcher makes them: the first argument is
    one key per caller row (the CachedAudioDecodeStates; placeholders for the stateless cached path)."""

    def __init__(self, rt: B200QwenRealtimeModel):
        self.rt = rt

    def _append(self, states, mels=None, flush: bool = False):
        engine = self.rt.encoder.engine
        for st in states:                          # fail before any session is touched: the batch is then replayed
            if getattr(st.audio, "engine", None) is not engine:
                raise ValueError("the stream's audio session is closed")
        saved = [(st.audio.frames_seen, st.audio.last_input_frames) for st in states]
        try:
            return self.rt.frames.append(states, mels, flush=flush)
        except BaseException:
            for st, (seen, last) in zip(states, saved):
                st.audio.frames_seen, st.audio.last_input_frames = seen, last
            raise

    def append_audio_to_cache(self, states, mels):
        return self._append(states, mels)

    def flush_audio_to_cache(self, states):
        return self._append(states, flush=True)

    def generate_full_hypothesis_rolling(self, states, items, *, template_token_ids, audio_placeholder_token_id,
                                         max_new_tokens, **controls):
        dec = self.rt.decoder
        toks, stats = dec.generate_rolling_batch([fh for fh, _ in items], states, [d for _, d in items],
                                                 template_token_ids=list(template_token_ids),
                                                 audio_placeholder_token_id=audio_placeholder_token_id,
                                                 max_new_tokens=max_new_tokens, **controls)
        return list(zip(toks, stats))

    def generate_full_hypothesis_from_cached_audio(self, keys, items, *, audio_placeholder_token_id, max_new_tokens,
                                                   **controls):
        dec = self.rt.decoder
        ctl = dec.engine.make_controls(wait_token_id=dec.model.wait_token_id, **controls)
        return dec.full_tokens([fh for fh, _, _ in items], [p for _, p, _ in items], [q for _, _, q in items],
                               audio_placeholder_token_id, max_new_tokens, ctl)

    def close(self):
        pass
