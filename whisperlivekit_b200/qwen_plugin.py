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

    def _check_mels(self, mels):
        if mels.ndim != 3:
            raise ValueError("mels must have shape [batch, frames, n_mels]")
        if mels.shape[-1] != self.dims.n_mels:
            raise ValueError(f"expected {self.dims.n_mels} mel bins, got {mels.shape[-1]}")
        if mels.shape[0] != 1:
            raise ValueError("one stream per state: batch sessions through engine.forward_chunk")

    def encode_rows(self, states, mels=None, flush: bool = False, device_rows: bool = True):
        """forward_chunk (flush=False, mels [1, frames, n_mels] per state) or flush_pending (flush=True) for N states in
        one engine call, with each state's fields updated as those two methods do.  Returns (rows [total, out_dim],
        row offsets [N + 1]): a CUDA tensor when the engine runs on the device and device_rows is set, else a CPU
        tensor."""
        import torch
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
                self._check_mels(m)
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
            offs = np.zeros(len(states) + 1, np.int64)
            offs[1:] = np.cumsum([h.shape[0] for h in hs])
            rows = torch.from_numpy(np.ascontiguousarray(np.concatenate(hs) if hs else np.zeros((0, self.dims.out_dim),
                                                                                              np.float32)))
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


class B200DecoderRollingState:
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

    def close(self):
        if self.engine is not None:
            self.engine.close_session(self.sid)
            self.engine = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class B200QwenTextDecoder:
    """Drop-in for the text half of the reference's realtime model: ``generate_full_hypothesis_rolling`` (model.py:
    991-1250) and ``generate_full_hypothesis_from_cached_audio`` (:839-989) rebound on one model instance over the text
    engine (``wlk_qtext_*``), the rolling prefix KV in a device session per stream::

        B200QwenTextDecoder.install(model, precision="bf16")

    Frame rows cross the seam as the host tensor the reference hands over; only the rows the session has not seen are
    uploaded.  ``use_decoder_kv_cache=False`` takes the same cached path (the reference documents the two as
    greedy-equal)."""

    def __init__(self, model, engine, dims):
        self.model, self.engine, self.dims = model, engine, dims

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
        fh = self._rows(frame_hidden)

        def rows(ids, b):
            if ids is None:
                return None
            t = torch.as_tensor(ids).long()
            return (t if t.ndim == 1 else t[b]).tolist()

        outs = [self.engine.generate_full(fh[b], prefix_token_ids=rows(prefix_token_ids, b),
                                          audio_placeholder_token_id=audio_placeholder_token_id,
                                          prompt_token_ids=rows(prompt_token_ids, b), max_new_tokens=max_new_tokens,
                                          controls=ctl, bos_token_id=self.model.bos_token_id) for b in range(batch)]
        # rows that stopped early are filled with the stop-fill id while the others decode (model.py:419-436)
        width = max(len(o) for o in outs)
        if ctl.stop_ids:
            fill = ctl.eos_token_id if ctl.eos_token_id is not None else min(ctl.stop_ids)
            outs = [o + [fill] * (width - len(o)) for o in outs]
        return torch.tensor(outs, dtype=torch.long, device=device).reshape(batch, width)

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
        toks, stats, new = self.engine.generate_rolling(
            [d.sid for d in decs], [self._rows(f) for f in frame_rows], prevs, template_token_ids,
            audio_placeholder_token_id, [None if d is None else [int(t) for t in d] for d in drafts],
            max_new_tokens=max_new_tokens, bos_token_id=self.model.bos_token_id, **controls)
        for dec, state, st, s in zip(decs, states, new, stats):
            if s.get("decoder_path") != "full":
                dec.head_token_ids, dec.head_len, dec.audio_steps = st.head_token_ids, st.head_len, st.audio_steps
                state.decoder = dec
        return toks, stats


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


class B200QwenRealtimeModel:
    """The whole realtime model (``Qwen3ASRRealtimeQwenAudioCausalModel``) on the engines, installed on one instance::

        B200QwenRealtimeModel.install(model, precision="bf16")

    replaces ``model.audio_encoder`` with the tower drop-in, installs the text decoder drop-in with the frame adapter
    packed into its engine, and rebinds ``append_audio_to_cache`` / ``flush_audio_to_cache`` onto
    ``qwen_realtime.RealtimeFrames`` (N = 1).  With CUDA engines ``state.frame_hidden`` is a device tensor and the
    generate methods read it in place: no frame row reaches the host.  The reference streamers
    (``SegmentedCachedFullHypothesisStreamer``) run over the installed model unchanged."""

    def __init__(self, model, encoder, decoder):
        from .qwen_realtime import RealtimeFrames
        self.model, self.encoder, self.decoder = model, encoder, decoder
        self.frames = RealtimeFrames(encoder, decoder.engine, decoder.dims.d_model)

    @classmethod
    def install(cls, model, precision: str = "bf16", max_ctx: int = 1024, max_sessions: int = 8, tower_factory=None,
                text_factory=None):
        """tower_factory(dims, state_dict) / text_factory(dims, state_dict): engines to use instead of the CUDA ones
        (the CPU oracles in tests)."""
        tower_kw = {} if tower_factory else dict(precision=precision, max_sessions=max_sessions)
        encoder = B200QwenAudioCausalKVEncoder.from_reference(model.audio_encoder, engine_factory=tower_factory, **tower_kw)
        if encoder.dims.out_dim != model.adapter.proj.weight.shape[1]:
            raise ValueError(f"tower rows are {encoder.dims.out_dim} wide, the adapter takes "
                             f"{model.adapter.proj.weight.shape[1]}")
        decoder = B200QwenTextDecoder.install(model, engine_factory=text_factory, precision=precision, max_ctx=max_ctx,
                                              max_sessions=max_sessions, extra_tensors=adapter_tensors(model.adapter))
        rt = cls(model, encoder, decoder)
        if "audio_encoder" in getattr(model, "_modules", {}):
            del model._modules["audio_encoder"]        # an nn.Module takes only modules as child attributes
        model.audio_encoder = encoder
        model.append_audio_to_cache = rt.append_audio_to_cache
        model.flush_audio_to_cache = rt.flush_audio_to_cache
        model.b200_realtime = rt
        return rt

    def append_audio_to_cache(self, mels, state=None):
        if state is None:
            state = self.model.init_cached_audio_decode_state()
        (cached, delta), = self.frames.append([state], [mels])
        return cached, delta, state

    def flush_audio_to_cache(self, state=None):
        if state is None:
            state = self.model.init_cached_audio_decode_state()
        (cached, delta), = self.frames.append([state], flush=True)
        return cached, delta, state
