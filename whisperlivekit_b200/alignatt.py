"""Host side of the AlignAtt seam (the reference's primary plugin surface).

Two things live here:

* ``AlignAttHooks`` -- the ~20 tensor hooks ``AlignAttBase`` declares abstract
  (reference whisperlivekit/simul_whisper/align_att_base.py:541-649), written
  against the engine session API (``engine.WhisperEngine``).  With
  WhisperLiveKit importable, ``plugin.make_b200_alignatt_class()`` mixes these
  into the reference's own ``AlignAttBase`` so its ``infer()`` and the
  SimulStreaming processor run unchanged on the H100 engine.
* ``StreamingAlignAtt`` -- a self-contained mirror of the control flow of
  ``AlignAttBase.infer`` (align_att_base.py:174-322) and ``AlignAtt.insert_audio``
  (simul_whisper.py:219-237) on token ids only (no tokenizer/text), for hosts
  where WhisperLiveKit is not installed (the GPU test box, bench.py).  Same
  names, same stop / rewind / suppression rules, same defaults.

Neither class contains tensor math: that is all behind the engine's C-ABI.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np

from .dims import SpecialTokens

DEC_PAD = 50257                     # reference align_att_base.py:10
TOKENS_PER_SECOND = 50              # reference whisper/audio.py:22


@dataclass
class AlignAttConfig:
    """Mirror of reference simul_whisper/config.py:5-23 (hot-path fields) with the
    values core.py passes for the default SimulStreaming setup (config.py:104-108)."""
    frame_threshold: int = 25
    rewind_threshold: int = 200
    audio_max_len: float = 30.0
    audio_min_len: float = 0.0
    nonspeech_prob: float = 0.5
    beam_size: int = 1
    decoder_type: str = "greedy"
    language: str = "en"
    task: str = "transcribe"
    max_context_tokens: Optional[int] = None
    dry_penalty: bool = True


def dry_penalties(seq: Sequence[int], eot: int, max_run: int = 50) -> List[Tuple[int, float]]:
    """DRY repetition penalty, host part -- the integer rule of the reference's ``_apply_dry_penalty``
    (align_att_base.py:492-537), which must be reproduced exactly because it decides tokens: wherever the newest text
    token occurred before, the token that FOLLOWED it then is penalised by 2^(run - 2), ``run`` being how many tokens the
    two contexts share going backwards (special tokens end a run, at most ``max_run``; the longest run per follower wins;
    runs of one are free).  -> [(token, amount_to_subtract)]"""
    toks = list(seq)
    tail = len(toks) - 1
    if tail < 4 or toks[tail] >= eot:
        return []

    def shared_run(i: int) -> int:
        run = 1                                          # toks[i] == toks[tail] by construction
        for back in range(1, max_run):
            a, b = i - back, tail - back
            if a < 0 or b <= i or toks[a] != toks[b] or toks[a] >= eot:
                break
            run += 1
        return run

    longest: dict = {}
    for i in reversed(range(tail)):                      # earlier occurrences, newest first (the reference's scan order)
        if toks[i] != toks[tail] or toks[i + 1] >= eot:
            continue
        run = shared_run(i)
        if run > longest.get(toks[i + 1], 0):
            longest[toks[i + 1]] = run
    return [(tok, 2.0 ** (run - 2)) for tok, run in longest.items() if run >= 2]


def engine_select(eng, sids, suppress, first_ids, first_mask, biases, window_iters=16):
    """The "pick" half of a policy iteration.  Engines with the fused entry point (WhisperEngine.select ->
    wlk_select, BatchingEngine.select) take it in one call; a duck-typed engine that only has the elementary calls
    gets the same steps in the same order."""
    sel = getattr(eng, "select", None)
    if sel is not None:
        return sel(sids, suppress, first_ids, first_mask, biases, window_iters=window_iters)
    for i, sid in enumerate(sids):
        if first_mask[i] and len(first_ids):
            eng.suppress([sid], list(first_ids))
    if len(suppress):
        eng.suppress(list(sids), list(suppress))
    for sid, b in zip(sids, biases):
        if b:
            eng.add_logit_bias(sid, [t for t, _ in b], [v for _, v in b])
    return eng.greedy_and_align(list(sids), window_iters=window_iters)


@dataclass
class InferTrace:
    """What one ``infer`` did -- compared token-for-token with the reference in tests."""
    content_mel_len: int = 0
    prefix_len: int = 0
    no_speech: bool = False
    no_speech_prob: float = 0.0
    step_tokens: List[int] = field(default_factory=list)      # argmax token of every loop iteration
    step_frames: List[int] = field(default_factory=list)      # most attended frame of every iteration
    step_logprobs: List[float] = field(default_factory=list)
    new_tokens: List[int] = field(default_factory=list)       # hypothesis appended to state.tokens
    timestamps: List[float] = field(default_factory=list)
    stop: str = ""


class StreamingAlignAtt:
    """Per-session AlignAtt policy over an engine session (greedy, beam_size 1)."""

    def __init__(self, engine, cfg: Optional[AlignAttConfig] = None, lang_index: int = 0):
        self.engine = engine
        self.cfg = cfg or AlignAttConfig()
        if self.cfg.decoder_type != "greedy" or self.cfg.beam_size != 1:
            raise NotImplementedError("StreamingAlignAtt implements the greedy policy (reference default beams=1)")
        self.sp: SpecialTokens = engine.specials
        self.sid = engine.open_session()
        self.max_text_len = engine.dims.n_text_ctx
        self.max_context_tokens = self.cfg.max_context_tokens or self.max_text_len
        self.initial_tokens = list(self.sp.sot_sequence_including_notimestamps(lang_index, self.cfg.task))
        self.sot_index = 0                                   # tokenizer.sot_sequence.index(sot)
        self.suppress_tokens = self.sp.alignatt_suppress_tokens()
        self.segments: List[int] = []                        # sample counts of buffered chunks
        self.tokens: List[List[int]] = [list(self.initial_tokens)]
        self.context: List[int] = []                         # token ids moved out of the window
        self.last_attend_frame = -self.cfg.rewind_threshold
        self.cumulative_time_offset = 0.0
        self.first_timestamp: Optional[float] = None
        self.closed = False

    # -- audio window ------------------------------------------------------
    def segments_len(self) -> float:
        return sum(self.segments) / 16000

    def insert_audio(self, segment: Optional[np.ndarray] = None) -> float:
        """reference simul_whisper.py:219-237."""
        if segment is not None:
            seg = np.ascontiguousarray(np.asarray(segment, dtype=np.float32).reshape(-1))
            self.segments.append(int(seg.shape[0]))
            self.engine.append_audio(self.sid, seg)
        removed_len = 0.0
        segments_len = self.segments_len()
        while len(self.segments) > 1 and segments_len > self.cfg.audio_max_len:
            removed = self.segments[0]
            removed_len = removed / 16000
            segments_len -= removed_len
            self.last_attend_frame -= int(TOKENS_PER_SECOND * removed_len)
            self.cumulative_time_offset += removed_len
            self.segments = self.segments[1:]
            self.engine.drop_audio(self.sid, removed)
            if len(self.tokens) > 1:
                self.context.extend(self.tokens[1])
                self.tokens = [list(self.initial_tokens)] + self.tokens[2:]
        return removed_len

    def refresh_segment(self, complete: bool = False) -> None:
        """reference align_att_base.py:115-132 (token-id form)."""
        self.tokens = [list(self.initial_tokens)]
        self.last_attend_frame = -self.cfg.rewind_threshold
        self.cumulative_time_offset = 0.0
        self.context = []
        if not complete and len(self.segments) > 2:
            drop = sum(self.segments[:-2])
            self.segments = self.segments[-2:]
            self.engine.drop_audio(self.sid, drop)
        else:
            self.segments = []
            self.engine.clear_audio(self.sid)

    def trim_context(self) -> None:
        """reference align_att_base.py:100-113; the reference trims whole words of the
        context *text*, this id-only mirror trims one token at a time."""
        c = len(self.context)
        l = sum(len(t) for t in self.tokens) + c
        while c > self.max_context_tokens or l > self.max_text_len - 20:
            if not self.context:
                break
            self.context.pop(0)
            c -= 1
            l -= 1

    def _current_tokens(self) -> List[int]:
        """reference simul_whisper.py:239-254."""
        toks: List[int] = []
        if self.context:
            toks += [self.sp.sot_prev] + self.context
        for t in self.tokens:
            toks += t
        return toks

    # -- the template infer() ------------------------------------------------
    def infer(self, is_last: bool = False) -> InferTrace:
        begin = getattr(self.engine, "begin_iter", None)
        if begin is None:
            return self._infer(is_last)
        begin()                                   # BatchingEngine: one more session inside a policy iteration
        try:
            return self._infer(is_last)
        finally:
            self.engine.end_iter()

    def _infer(self, is_last: bool = False) -> InferTrace:
        """Run the iteration against this policy's own engine, one call per request."""
        eng, sid = self.engine, self.sid
        gen = self.infer_steps(is_last)
        try:
            req = next(gen)
            while True:
                op = req[0]
                if op == "encode":
                    res = eng.encode([sid])[0]
                elif op == "decode":
                    res = eng.decode([sid], [req[1]], sot_index=self.sot_index)
                elif op == "no_speech":
                    res = eng.no_speech_prob([sid])[0]
                else:                             # "select"
                    res = engine_select(eng, [sid], self.suppress_tokens, [self.sp.blank, self.sp.eot], [req[1]], [req[2]],
                                        window_iters=16)[0]
                req = gen.send(res)
        except StopIteration as stop:
            return stop.value

    def infer_steps(self, is_last: bool = False):
        """reference align_att_base.py:174-322 (control flow) as a generator: every engine request of the iteration is
        yielded -- ("encode",) -> content_mel_len; ("decode", tokens) -> None; ("no_speech",) -> probability;
        ("select", first_iteration, dry_bias_pairs) -> (token, logprob, frame) -- and the InferTrace is the return
        value.  ``_infer`` serves the requests one by one; ``cohort.CohortRunner`` advances many policies in lockstep
        and serves each round of requests with ONE batched engine call, without a thread per stream."""
        cfg = self.cfg
        tr = InferTrace()
        if len(self.segments) == 0:
            tr.stop = "no_segments"
            return tr
        if self.segments_len() < cfg.audio_min_len:
            tr.stop = "minseglen"
            return tr

        content_mel_len = yield ("encode",)                                  # _encode
        tr.content_mel_len = content_mel_len
        self.trim_context()
        current_tokens = self._current_tokens()
        token_len_before = len(current_tokens)
        tr.prefix_len = token_len_before

        completed = False
        new_segment = True
        l_absolute_timestamps: List[float] = []
        audio_duration_s = self.segments_len()
        max_tokens = max(50, int(audio_duration_s * 15 * 1.5))
        tokens_produced = 0

        while not completed and len(current_tokens) < self.max_text_len:
            tokens_produced += 1
            if tokens_produced > max_tokens:
                current_tokens = current_tokens[:token_len_before]
                tr.stop = "loop_detection"
                break
            feed = current_tokens if new_segment else current_tokens[-1:]
            yield ("decode", list(feed))                                     # _get_logits_and_cross_attn
            if new_segment:
                p = yield ("no_speech",)                                     # _check_no_speech
                tr.no_speech_prob = p
                if p > cfg.nonspeech_prob:
                    tr.no_speech = True
                    tr.stop = "no_speech"
                    break
            first = new_segment                                              # _suppress_blank_tokens applies
            new_segment = False
            pen = dry_penalties(current_tokens, self.sp.eot) if cfg.dry_penalty else []     # _apply_dry_penalty
            # _suppress_blank_tokens, _apply_token_suppression, _apply_dry_penalty, _update_tokens,
            # _process_cross_attention and _get_attended_frames: one engine call (wlk_select)
            tok, logprob, frame = yield ("select", first, [(t, -a) for t, a in pen])
            if current_tokens[-1] == self.sp.eot:                            # decoding.py:282
                tok = self.sp.eot
            current_tokens = current_tokens + [tok]
            completed = tok == self.sp.eot
            tr.step_tokens.append(tok)
            tr.step_frames.append(frame)
            tr.step_logprobs.append(logprob)
            l_absolute_timestamps.append(frame * 0.02 + self.cumulative_time_offset)

            if completed:
                current_tokens = current_tokens[:-1]
                tr.stop = "eot"
                break
            if (not is_last) and self.last_attend_frame - frame > cfg.rewind_threshold:
                if len(current_tokens) > 1 and current_tokens[-2] >= DEC_PAD:
                    self.last_attend_frame = frame
                else:
                    self.last_attend_frame = -cfg.rewind_threshold
                    current_tokens = [t for seg in self.tokens for t in seg]  # _rewind_tokens
                    tr.stop = "rewind"
                    break
            else:
                self.last_attend_frame = frame
            if content_mel_len - frame <= (4 if is_last else cfg.frame_threshold):
                current_tokens = current_tokens[:-1]
                tr.stop = "attention_end"
                break
        else:
            tr.stop = tr.stop or "max_text_len"

        new_hypothesis = current_tokens[token_len_before:]                   # always_fire: keep all
        n = len(new_hypothesis)
        ts = [float(x) for x in l_absolute_timestamps[:n]]
        if len(ts) < n:
            ts += [ts[-1] if ts else 0.0] * (n - len(ts))
        tr.new_tokens = list(new_hypothesis)
        tr.timestamps = ts
        self.tokens.append(list(new_hypothesis))
        if len(l_absolute_timestamps) >= 2 and self.first_timestamp is None:
            self.first_timestamp = l_absolute_timestamps[0]
        return tr

    def close(self) -> None:
        if not self.closed:
            self.engine.close_session(self.sid)
            self.closed = True


# =============================================================================================
# Drop-in hooks for the reference's own AlignAttBase.infer()
# =============================================================================================
class _EncoderFeature:
    """What AlignAttBase.infer treats opaquely: `encoder_feature[:, :content_mel_len, :]`
    (align_att_base.py:193) and pass-through to the hooks.  The tensor stays on the device."""

    def __init__(self, engine, sid, content_len=None):
        self.engine, self.sid, self.content_len = engine, sid, content_len
        self.shape = (1, 1500, engine.dims.n_audio_state)
        self.ndim = 3

    def __getitem__(self, key):
        c = self.content_len
        if isinstance(key, tuple) and len(key) >= 2 and isinstance(key[1], slice) and key[1].stop is not None:
            c = key[1].stop
        return _EncoderFeature(self.engine, self.sid, c)

    def numpy(self):
        a = self.engine.read_encoder(self.sid)[None]
        return a if self.content_len is None else a[:, : self.content_len]


class _Logits:
    """Return value of _get_logits_and_cross_attn: the base class only does `logits[:, -1, :]`."""

    def __init__(self, engine, sid):
        self.engine, self.sid = engine, sid

    def __getitem__(self, key):
        return self

    def numpy(self):
        return self.engine.read_logits(self.sid)[None]


class _BeamInference:
    """The one thing whisper.decoding.BeamSearchDecoder asks of its ``inference`` (decoding.py:361):
    re-index the self-attention K/V rows after ranking (reference simul_whisper/beam.py:15-19)."""

    def __init__(self, hooks):
        self.hooks = hooks
        self.kv_cache = {}

    def rearrange_kv_cache(self, source_indices):
        src = [int(i) for i in source_indices]
        if src != list(range(len(src))):
            self.hooks.engine.gather_decoder(self.hooks.beam_sids, src)


class AlignAttHooks:
    """Engine-backed implementation of every abstract hook of the reference's AlignAttBase
    (align_att_base.py:541-649).  Mixed in front of AlignAttBase by plugin.make_b200_alignatt_class();
    token tensors stay CPU torch.LongTensors (the base class slices them and calls .tolist()),
    everything heavy stays on the device behind one C call per hook."""

    def __init__(self, cfg, loaded_model=None, mlx_encoder=None, fw_encoder=None):
        from whisperlivekit.simul_whisper.decoder_state import DecoderState
        self.engine = loaded_model.engine
        self.device = "cpu"
        self.mlx_encoder, self.fw_encoder = None, None
        self._base_init(cfg, loaded_model)
        self.state = DecoderState()
        self.sid = self.engine.open_session()
        self._frame = 0
        self._n_audio = 0
        self._init_state(cfg)

    def close(self) -> None:
        """Release the session (and its beam forks) now: ~350 MB of device state at large-v3.  The online processor's
        teardown should call this; ``__del__`` is only a backstop (the _BeamInference <-> hooks cycle leaves collection
        to the cyclic GC, and under connection churn the engine would run out of sessions first)."""
        if getattr(self, "_closed", False):
            return
        self._closed = True
        for sid in reversed(getattr(self, "beam_sids", [self.sid])):         # forks before their parent
            try:
                self.engine.close_session(sid)
            except Exception:
                pass
        if getattr(self.state, "inference", None) is not None:
            self.state.inference.hooks = None                                # break the cycle

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def infer(self, is_last: bool = False):
        """The reference's template (align_att_base.py:174-322), bracketed so that a BatchingEngine knows how
        many sessions are inside a policy iteration and can fire a batch as soon as all of them have called."""
        begin = getattr(self.engine, "begin_iter", None)
        if begin is None:
            return super().infer(is_last=is_last)
        begin()
        try:
            return super().infer(is_last=is_last)
        finally:
            self.engine.end_iter()

    # ---- state -----------------------------------------------------------------
    def _init_state(self, cfg):
        from whisperlivekit.simul_whisper.eow_detection import load_cif
        self._init_state_common(cfg)
        self.state.CIFLinear, self.state.always_fire, self.state.never_fire = load_cif(
            cfg, n_audio_state=self.model.dims.n_audio_state, device="cpu")
        self.state.num_align_heads = len(self.engine.align_heads)
        t = self.tokenizer
        sup = [t.transcribe, t.translate, t.sot, t.sot_prev, t.sot_lm, t.no_timestamps] + list(t.all_language_tokens)
        if t.no_speech is not None:
            sup.append(t.no_speech)
        self._suppress = sorted(set(sup))                         # simul_whisper.py:161-172
        self._blank = list(t.encode(" ")) + [t.eot]
        self.init_tokens()
        self.init_context()
        self.state.decoder_type = cfg.decoder_type
        self.beam, self.beam_sids = 1, [self.sid]
        if cfg.decoder_type == "beam":
            # reference simul_whisper.py:182-192: beam_size decoder rows over ONE encoder output.  Here every beam
            # row is a session forked from the stream's session (shared encoder output / cross-K/V), ranked by the
            # reference's own BeamSearchDecoder on the host.
            from whisperlivekit.whisper.decoding import BeamSearchDecoder
            self.beam = int(cfg.beam_size)
            self.beam_sids = [self.sid] + [self.engine.fork_session(self.sid) for _ in range(self.beam - 1)]
            self.state.inference = _BeamInference(self)
            self.state.token_decoder = BeamSearchDecoder(inference=self.state.inference, eot=self.tokenizer.eot,
                                                         beam_size=self.beam)
        elif cfg.decoder_type != "greedy":
            raise NotImplementedError(f"decoder_type {cfg.decoder_type!r}")

    def init_tokens(self):
        import torch
        self.state.initial_tokens = torch.tensor(self.tokenizer.sot_sequence_including_notimestamps,
                                                 dtype=torch.long).unsqueeze(0)
        self.state.initial_token_length = self.state.initial_tokens.shape[1]
        self.state.sot_index = self.tokenizer.sot_sequence.index(self.tokenizer.sot)
        self.state.tokens = [self.state.initial_tokens]

    def init_context(self):
        from whisperlivekit.simul_whisper.token_buffer import TokenBuffer
        kw = dict(tokenizer=self.tokenizer, device="cpu", prefix_token_ids=[self.tokenizer.sot_prev])
        self.state.context = TokenBuffer.empty(**kw)
        if self.cfg.static_init_prompt is not None:
            self.state.context = TokenBuffer.from_text(self.cfg.static_init_prompt, **kw)
        if self.cfg.init_prompt is not None:
            self.state.context.text += self.cfg.init_prompt

    # ---- audio window (simul_whisper.py:219-237), mirrored into the device ring -------------
    def insert_audio(self, segment=None):
        if segment is not None:
            self.state.segments.append(segment)
            self.engine.append_audio(self.sid, np.asarray(segment, dtype=np.float32))
        removed_len = 0
        segments_len = self.segments_len()
        while len(self.state.segments) > 1 and segments_len > self.cfg.audio_max_len:
            removed_len = self.state.segments[0].shape[0] / 16000
            segments_len -= removed_len
            self.state.last_attend_frame -= int(TOKENS_PER_SECOND * removed_len)
            self.state.cumulative_time_offset += removed_len
            self.engine.drop_audio(self.sid, int(self.state.segments[0].shape[0]))
            self.state.segments = self.state.segments[1:]
            if len(self.state.tokens) > 1:
                self.state.context.append_token_ids(self.state.tokens[1][0, :].tolist())
                self.state.tokens = [self.state.initial_tokens] + self.state.tokens[2:]
        return removed_len

    def refresh_segment(self, complete=False):
        n_before = sum(int(s.shape[0]) for s in self.state.segments)
        super().refresh_segment(complete=complete)
        n_after = sum(int(s.shape[0]) for s in self.state.segments)
        if n_after == 0:
            self.engine.clear_audio(self.sid)
        elif n_after < n_before:
            self.engine.drop_audio(self.sid, n_before - n_after)

    def _concat_segments(self):
        return sum(int(s.shape[0]) for s in self.state.segments)      # the audio itself is already on the device

    def _current_tokens(self):
        import torch
        toks = self.state.tokens
        if toks[0].shape[0] == 1 and self.beam > 1:                          # simul_whisper.py:240-243
            toks[0] = toks[0].repeat_interleave(self.beam, dim=0)
        if not self.state.context.is_empty():
            toks = [self.state.context.as_tensor_beam(self.beam, device="cpu")] + toks
        return torch.cat(toks, dim=1) if len(toks) > 1 else toks[0]

    def fire_at_boundary(self, feature):
        if self.state.always_fire:
            return True
        if self.state.never_fire:
            return False
        if self.state.CIFLinear is None:
            return False
        import torch
        from whisperlivekit.simul_whisper.eow_detection import fire_at_boundary
        return fire_at_boundary(torch.from_numpy(feature.numpy()), self.state.CIFLinear)

    # ---- hot-path hooks -----------------------------------------------------------
    def _encode(self, input_segments):
        n = self.engine.audio_len(self.sid)
        if n != input_segments:
            raise RuntimeError(f"device audio ring ({n}) out of sync with state.segments ({input_segments})")
        content = self.engine.encode([self.sid])[0]
        self._iters = 0
        return _EncoderFeature(self.engine, self.sid), content

    def lang_id(self, encoder_features):
        self.engine.reset_decoder(self.sid)
        self.engine.decode([self.sid], [[self.tokenizer.sot]], sot_index=0)
        lg = self.engine.read_logits(self.sid).astype(np.float64)
        toks = list(self.tokenizer.all_language_tokens)
        sel = lg[toks]
        p = np.exp(sel - sel.max())
        p /= p.sum()
        probs = {c: float(p[j]) for j, c in enumerate(self.tokenizer.all_language_codes)}
        self._clean_cache()
        return [toks[int(np.argmax(sel))]], [probs]

    def _clean_cache(self):
        for sid in self.beam_sids:
            self.engine.reset_decoder(sid)
        if self.beam > 1:
            self.state.token_decoder.reset()                                 # decoder_state.py:55-59

    def _init_sum_logprobs(self):
        if self.beam > 1:
            import torch
            return torch.zeros(self.beam)                                    # simul_whisper.py:354-355
        return [0.0]

    def _get_logits_and_cross_attn(self, tokens, encoder_feature):
        rows = [tokens[b].tolist() for b in range(self.beam)] if self.beam > 1 else [tokens[0].tolist()]
        self.engine.decode(self.beam_sids, rows, sot_index=self.state.sot_index)
        self._iters += 1
        return _Logits(self.engine, self.sid), self._iters

    def _check_no_speech(self, logits):
        if self.tokenizer.no_speech is not None:
            return self.engine.no_speech_prob([self.sid])[0] > self.cfg.nonspeech_prob
        return False

    # The three logit edits below are recorded and applied, in this order, inside the one engine call that
    # _update_tokens makes (wlk_select): the base class only passes `logits` through between them
    # (align_att_base.py:229-237), so nothing can observe the difference, and a policy iteration costs two round
    # trips to the engine (decode, select) instead of five.
    def _suppress_blank_tokens(self, logits):
        self._pend_first = True
        return logits

    def _apply_token_suppression(self, logits):
        self._pend_suppress = True
        return logits

    def _apply_dry_penalty(self, logits, current_tokens):
        # the reference scans beam row 0 and penalises that token set on every row (align_att_base.py:501,535)
        self._pend_bias = [(t, -a) for t, a in dry_penalties(current_tokens[0].tolist(), self.tokenizer.eot)]
        return logits

    def _select(self):
        n = len(self.beam_sids)
        first, self._pend_first = getattr(self, "_pend_first", False), False
        sup, self._pend_suppress = getattr(self, "_pend_suppress", False), False
        bias, self._pend_bias = getattr(self, "_pend_bias", []), []
        return engine_select(self.engine, self.beam_sids, self._suppress if sup else [], self._blank, [first] * n,
                             [list(bias) for _ in range(n)], window_iters=16)

    def _update_tokens_beam(self, current_tokens, sum_logprobs):
        """whisper/decoding.py:317-376 (BeamSearchDecoder.update, unchanged, on the host) over the beams' fp32
        logits; its rearrange_kv_cache lands in wlk_sessions_gather_decoder.  The attended frames come from each
        row's own alignment history, which the reference does not re-index either."""
        import torch
        res = self._select()
        self._frames = [int(r[2]) for r in res]
        lg = torch.from_numpy(np.stack([self.engine.read_logits(sid) for sid in self.beam_sids]))
        return self.state.token_decoder.update(current_tokens, lg, sum_logprobs)

    def _update_tokens(self, current_tokens, logits, sum_logprobs):
        import torch
        if self.beam > 1:
            return self._update_tokens_beam(current_tokens, sum_logprobs)
        tok, lp, frame = self._select()[0]
        eot = self.tokenizer.eot
        if int(current_tokens[0, -1]) == eot:                       # decoding.py:280-282
            tok = eot
        else:
            sum_logprobs[0] += lp
        self._frame = frame
        tokens = torch.cat([current_tokens, torch.tensor([[tok]], dtype=torch.long)], dim=-1)
        return tokens, tok == eot

    def _process_cross_attention(self, accumulated_cross_attns, content_mel_len):
        return self._frames if self.beam > 1 else self._frame       # computed with the token, one D2H for both

    def _get_attended_frames(self, attn):
        if self.beam > 1:
            return list(attn), int(attn[0])                         # simul_whisper.py:435-437
        return [int(attn)], int(attn)

    def _is_special_token(self, current_tokens):
        return int(current_tokens[0, -2]) >= DEC_PAD

    def _rewind_tokens(self):
        import torch
        return torch.cat(self.state.tokens, dim=1) if len(self.state.tokens) > 0 else self.state.tokens[0]

    def _tokens_to_list(self, current_tokens, start_col):
        return current_tokens[0, start_col:].flatten().tolist()

    def _make_new_tokens_tensor(self, hypothesis):
        import torch
        t = torch.tensor([hypothesis], dtype=torch.long)
        return t.repeat_interleave(self.beam, dim=0) if self.beam > 1 else t      # simul_whisper.py:450-455

    def _evaluate(self, tensor):
        pass
