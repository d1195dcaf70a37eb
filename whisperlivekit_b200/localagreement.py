"""LocalAgreement seam: a Whisper-shaped model object for the reference's ``whisper.transcribe()``.

The LocalAgreement policy (reference local_agreement/online_asr.py:219-261) calls
``asr.transcribe(audio, init_prompt)`` -> ``whisper.transcribe(model, audio, ...)``
(local_agreement/backends.py:62-77), whose host logic (30 s seek loop, temperature fallback,
timestamp rules, DecodingTask, add_word_timestamps/find_alignment, DTW) stays the reference's.  This
module supplies the *model*: every tensor operation it is asked for goes to the H100 engine through
the C ABI.  Needs WhisperLiveKit importable (it reuses the reference's decode/transcribe functions).

What the reference touches on ``model`` (whisper/decoding.py:144-160,636-704; whisper/timing.py:163-215;
whisper/transcribe.py:111-146) and what answers here:
    model.dims / device / is_multilingual / num_languages / alignment_heads     -> attributes
    model.encoder(mel)                         -> wlk_encode_mel, returns an opaque AudioFeatures handle
    model.decoder(tokens, xa, kv_cache=dict)   -> wlk_decode (+ wlk_read_logits of the rows the caller reads)
    model.logits(tokens, xa)                   -> decoder without cache
    model(mel, tokens)                         -> encoder + wlk_decode_all_logits (word-timestamp pass)
    decoder.blocks[i].cross_attn.register_forward_hook(fn)  -> fn gets log-probabilities of the alignment
                                                  heads (wlk_read_align_rows): softmax over any frame slice
                                                  of log p equals the reference's softmax of qk on that slice
    model.decode / detect_language / transcribe -> the reference's own functions bound to this object
"""
from __future__ import annotations

from typing import List, Optional

import numpy as np


class AudioFeatures:
    """Opaque stand-in for the encoder output tensor [1, 1500, d] (it never leaves the device)."""

    def __init__(self, model, sid):
        import torch
        self.model, self.sid = model, sid
        self.shape = (1, model.dims.n_audio_ctx, model.dims.n_audio_state)
        self.dtype = torch.float32
        self.device = model.device
        self.ndim = 3

    def __len__(self):
        return 1

    def __iter__(self):
        yield self

    def __getitem__(self, key):
        return self

    def repeat_interleave(self, n, dim=0):
        return self          # beam_size / best_of rows all read the one encoder output (forked sessions)

    def to(self, *a, **k):
        return self

    def half(self):
        return self


class _KvHandle:
    """Stand-in for a self-attention K/V cache tensor inside the reference's ``kv_cache`` dict.  The only thing
    the reference does with it is ``kv_cache[id] = kv_cache[id][source_indices].detach()``
    (PyTorchInference.rearrange_kv_cache, decoding.py:165-170): indexing records the permutation, which the model
    applies on the device (wlk_sessions_gather_decoder) before the next decoder call."""

    def __init__(self, model):
        self.model = model

    def __getitem__(self, source_indices):
        self.model._pending_perm = [int(i) for i in source_indices]
        return self

    def detach(self):
        return self


class _Hookable:
    def __init__(self):
        self.hooks = []

    class _Handle:
        def __init__(self, owner, fn):
            self.owner, self.fn = owner, fn

        def remove(self):
            if self.fn in self.owner.hooks:
                self.owner.hooks.remove(self.fn)

    def register_forward_hook(self, fn):
        self.hooks.append(fn)
        return self._Handle(self, fn)


class _Attn(_Hookable):
    def __init__(self, cache_id):
        super().__init__()
        self.key_cache_id = f"{cache_id}_key"
        self.value_cache_id = f"{cache_id}_value"


class _Block:
    def __init__(self, i):
        self.attn = _Attn(f"dec_layer{i}_self_attn")
        self.cross_attn = _Attn(f"dec_layer{i}_cross_attn")


class _Decoder:
    def __init__(self, model):
        self.model = model
        self.blocks = [_Block(i) for i in range(model.dims.n_text_layer)]

    def __call__(self, tokens, xa, kv_cache: Optional[dict] = None, return_cross_attn: bool = False):
        return self.model._decode(tokens, xa, kv_cache)


class B200TranscribeModel:
    """Duck-types the reference ``Whisper`` module for whisper.transcribe()/decode()/find_alignment."""

    def __init__(self, engine):
        import torch
        from whisperlivekit.whisper.decoding import decode as decode_function
        from whisperlivekit.whisper.decoding import detect_language as detect_language_function
        from whisperlivekit.whisper.transcribe import transcribe as transcribe_function
        self.engine = engine
        self.dims = engine.dims
        self.device = torch.device("cpu")          # host-side tensors (tokens, logits views) live on the CPU
        self.decoder = _Decoder(self)
        mask = torch.zeros(self.dims.n_text_layer, self.dims.n_text_head, dtype=torch.bool)
        for l, h in engine.align_heads:
            mask[l, h] = True
        self.alignment_heads = mask.to_sparse()
        self.sid = engine.open_session()
        self._last_mel = None
        self.encoder_calls = 0
        self.encoder_reuses = 0
        self._forks: List[int] = []            # beam_size / best_of rows beyond the first: sessions forked from self.sid
        self._pending_perm = None
        self.gathers = 0
        self._decode_fn, self._detect_fn, self._transcribe_fn = decode_function, detect_language_function, transcribe_function

    # -- attributes the reference reads ---------------------------------------------------
    @property
    def is_multilingual(self):
        return self.dims.is_multilingual

    @property
    def num_languages(self):
        return self.dims.num_languages

    def decode(self, mel, options=None, **kw):
        from whisperlivekit.whisper.decoding import DecodingOptions
        return self._decode_fn(self, mel, options or DecodingOptions(), **kw)

    def detect_language(self, mel, tokenizer=None):
        return self._detect_fn(self, mel, tokenizer)

    def transcribe(self, audio, **kw):
        return self._transcribe_fn(self, audio, **kw)

    # -- tensor operations -> engine -------------------------------------------------------
    def encoder(self, mel):
        m = mel.detach().cpu().float().numpy()
        if m.ndim == 3:
            if m.shape[0] != 1:
                raise NotImplementedError("H100 LocalAgreement model: one audio segment per call")
            m = m[0]
        # The word-timestamp pass (timing.py:197) asks for model(mel, tokens) on the very segment that
        # DecodingTask just encoded: the session still holds that encoder output and its cross-K/V, so a
        # bit-identical mel is not encoded twice (SURVEY.md section 8f item 2: halves the encoder work of this path).
        if self._last_mel is not None and self._last_mel.shape == m.shape and np.array_equal(self._last_mel, m):
            self.encoder_reuses += 1
        else:
            self.engine.encode_mel(self.sid, m, 1500)
            self._last_mel = m.copy()
            self.encoder_calls += 1
        return AudioFeatures(self, self.sid)

    embed_audio = encoder

    def _rows(self, n: int) -> List[int]:
        """Sessions behind the n decoder rows of a beam / best_of group (decoding.py:728): row 0 is the segment's
        session, the others are forks sharing its encoder output and cross-K/V."""
        while len(self._forks) < n - 1:
            self._forks.append(self.engine.fork_session(self.sid))
        return [self.sid] + self._forks[: n - 1]

    def _decode(self, tokens, xa, kv_cache):
        import torch
        B = int(tokens.shape[0])
        sids = self._rows(B)
        rows = [[int(t) for t in tokens[b].tolist()] for b in range(B)]
        fresh = kv_cache is None or len(kv_cache) == 0
        if fresh:
            for sid in sids:
                self.engine.reset_decoder(sid)
            self._pending_perm = None
            if kv_cache is not None:
                kv_cache["b200_session"] = self.sid
                for blk in self.decoder.blocks:                     # what rearrange_kv_cache will index
                    kv_cache[blk.attn.key_cache_id] = _KvHandle(self)
                    kv_cache[blk.attn.value_cache_id] = _KvHandle(self)
        elif self._pending_perm is not None:
            if self._pending_perm != list(range(B)):
                self.engine.gather_decoder(sids, self._pending_perm)
                self.gathers += 1
            self._pending_perm = None
        sot = self.engine.specials.sot
        sot_index = rows[0].index(sot) if (fresh and sot in rows[0]) else 0
        self.engine.decode(sids, rows, sot_index=sot_index)
        T = len(rows[0])
        logits = torch.zeros(B, T, self.dims.n_vocab)
        for b, sid in enumerate(sids):
            logits[b, -1] = torch.from_numpy(self.engine.read_logits(sid))
            if fresh and T > 1:
                logits[b, sot_index] = torch.from_numpy(self.engine.read_sot_logits(sid))
        return logits

    def logits(self, tokens, audio_features, kv_cache=None, return_cross_attn=False):
        return self._decode(tokens, audio_features, kv_cache)

    def __call__(self, mel, tokens):
        """Whisper.forward(mel, tokens) (model.py:388-391): used by find_alignment with cross-attn hooks."""
        import torch
        self.encoder(mel)
        toks = [int(t) for t in tokens[0].tolist()]
        self.engine.reset_decoder(self.sid)
        all_logits = self.engine.decode_all_logits(self.sid, toks, sot_index=0)
        hooked = [b for b in self.decoder.blocks if b.cross_attn.hooks]
        if hooked:
            rows = self.engine.read_align_rows(self.sid)                 # [n_align, T, 1500] probabilities
            with np.errstate(divide="ignore"):
                logp = np.log(rows)
            per_layer = {}
            for rank, (l, h) in enumerate(self.engine.align_heads):
                qk = per_layer.setdefault(l, torch.zeros(1, self.dims.n_text_head, len(toks), 1500))
                qk[0, h] = torch.from_numpy(logp[rank])
            for i, b in enumerate(self.decoder.blocks):
                qk = per_layer.get(i)
                if qk is None:
                    qk = torch.zeros(1, self.dims.n_text_head, len(toks), 1500)
                for fn in list(b.cross_attn.hooks):
                    fn(b.cross_attn, (), (None, qk))
        return torch.from_numpy(all_logits)[None]

    def close(self):
        for sid in reversed(self._forks):
            self.engine.close_session(sid)
        self._forks = []
        self.engine.close_session(self.sid)


def install_native_timing(engine):
    """Route the reference's word-timestamp kernels to the engine: ``whisper.timing.median_filter`` and
    ``whisper.timing.dtw`` (timing.py:19-54,141-151; their GPU versions are the Triton kernels of
    whisper/triton_ops.py) are looked up in the module at call time by ``find_alignment`` (timing.py:204-213),
    so rebinding the two names is the whole integration.  Both native kernels are bit-exact against the
    reference's CPU path (tests/test_timing.py), hence word boundaries do not move."""
    import torch
    import whisperlivekit.whisper.timing as timing

    def median_filter(x, filter_width: int):
        pad = filter_width // 2
        if x.shape[-1] <= pad:                      # same early-out as the reference (timing.py:23-26)
            return x
        return torch.from_numpy(engine.median_filter_host(x.detach().cpu().float().numpy(), filter_width))

    def dtw(x):
        text_indices, time_indices = engine.dtw_host(x.detach().cpu().float().numpy())
        return np.stack([text_indices, time_indices]).astype(np.int64)

    if not hasattr(timing, "_b200_saved"):
        timing._b200_saved = (timing.median_filter, timing.dtw)
    timing.median_filter, timing.dtw = median_filter, dtw


def uninstall_native_timing():
    import whisperlivekit.whisper.timing as timing
    if hasattr(timing, "_b200_saved"):
        timing.median_filter, timing.dtw = timing._b200_saved
        del timing._b200_saved


class B200WhisperASR:
    """Mirror of the reference's ``WhisperASR`` (local_agreement/backends.py:39-99) over B200TranscribeModel:
    same ``transcribe / ts_words / segments_end_ts / use_vad`` duck-type that ``OnlineASRProcessor`` drives."""
    sep = " "

    def __init__(self, engine, lan: str = "en", native_timing: bool = True):
        self.model = B200TranscribeModel(engine)
        if native_timing:
            install_native_timing(engine)
        self.original_language = None if lan == "auto" else lan
        self.transcribe_kargs = {}

    def transcribe(self, audio, init_prompt=""):
        options = dict(self.transcribe_kargs)
        options.pop("vad", None)
        options.pop("vad_filter", None)
        language = self.original_language if self.original_language else None
        return self.model.transcribe(audio, language=language, initial_prompt=init_prompt,
                                     condition_on_previous_text=True, word_timestamps=True, **options)

    def ts_words(self, r):
        from whisperlivekit.timed_objects import ASRToken
        return [ASRToken(w["start"], w["end"], w["word"], probability=w.get("probability"))
                for seg in r["segments"] for w in seg["words"]]

    def segments_end_ts(self, res) -> List[float]:
        return [seg["end"] for seg in res["segments"]]

    def use_vad(self):
        pass
