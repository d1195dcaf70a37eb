"""Host side of the Qwen3-ASR text decoder (ctypes over wlk_qtext_* in include/wlk_b200.h).

``QwenTextEngine`` owns sessions with a croppable KV cache on the device, a forward over token / embedding rows and the
greedy decode controls + argmax (``pick``).  ``TextDecodeDriver`` runs the reference's two generate methods
(third_party/qwen3-asr-causal/src/qwen3_asr_causal/model.py) on top of those four primitives, batched over sessions:

  * ``generate_rolling``  - generate_full_hypothesis_rolling (:991-1250): persistent [head + audio] prefix, the template
    tail and the previous hypothesis (draft) in one forward, verification of the draft, sequential decode from the
    first divergence, crop back to the prefix.  N sessions run in lockstep: one forward for every session's block,
    one pick over all verify rows, then one forward + pick per step over the sessions still decoding.
  * ``generate_full``     - generate_full_hypothesis_from_cached_audio (:839-989) on a scratch session.
  * ``generate_full_batch`` - the same cached path for N caller-owned sessions in lockstep: one forward of every prefix,
    then one forward + pick per step over the sessions still decoding.  ``generate_full`` is its N = 1 case.

``QwenTextEngine`` runs ``generate_full_batch`` and ``generate_rolling_batch`` (``generate_rolling`` in one call) as single
engine calls (wlk_qtext_generate_full / wlk_qtext_generate_rolling); its ``generate_full`` and ``generate_rolling`` stay
the driver loops over forward / pick, the reference the engine calls are tested against.

The CPU oracle (oracle/qwen_text_oracle.py) implements the same primitives, so both run the same driver code."""
from __future__ import annotations

import ctypes as C
import threading
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib as L
from ._lib import _ptr
from .qwen_dims import QwenTextDims, rope_inv_freq


def _frame_rows(x):
    """Frame rows as an engine takes them: a CUDA tensor stays where it is (fp32), anything else becomes fp32 numpy."""
    if getattr(x, "is_cuda", False):
        return x.float()
    return np.ascontiguousarray(x, np.float32)


@dataclass
class RollingState:
    """The part of the reference's DecoderRollingState (model.py:53-68) the engine needs: the session holds the KV of
    exactly [head + audio_steps] positions between calls."""
    head_token_ids: Tuple[int, ...] = ()
    head_len: int = 0
    audio_steps: int = 0


@dataclass
class Controls:
    stop_ids: frozenset
    suppress: np.ndarray            # int32, in-vocab
    penalty: float
    ngram: int
    max_consecutive: int
    wait_id: int                    # -1: none
    eos_token_id: Optional[int]


def split_template(template_token_ids: Sequence[int], placeholder: int) -> Tuple[List[int], List[int]]:
    """_split_prompt_template (model.py:238-251)."""
    ids = [int(t) for t in template_token_ids]
    pos = [i for i, t in enumerate(ids) if t == int(placeholder)]
    if len(pos) != 1:
        raise ValueError(f"prompt template must contain exactly one audio placeholder token, got {len(pos)}")
    return ids[:pos[0]], ids[pos[0] + 1:]


class TextDecodeDriver:
    """Generate logic over the primitives open_session / close_session / reset_session / session_len / crop /
    forward / pick of a text engine (device or oracle)."""

    vocab: int

    @property
    def phase_lock(self) -> threading.RLock:
        """Held across every forward + pick phase of the generate drivers: the engine keeps only the last forward's
        logit rows, so threads sharing one engine must not interleave their phases."""
        lk = self.__dict__.get("_phase_lock")
        if lk is None:
            lk = self.__dict__.setdefault("_phase_lock", threading.RLock())
        return lk

    def generate_rolling(self, *args, **kwargs):
        with self.phase_lock:
            return self._generate_rolling(*args, **kwargs)

    def generate_full(self, *args, **kwargs) -> List[int]:
        with self.phase_lock:
            return self._generate_full(*args, **kwargs)

    def generate_full_batch(self, *args, **kwargs) -> List[List[int]]:
        with self.phase_lock:
            return self._generate_full_batch(*args, **kwargs)

    def generate_rolling_batch(self, *args, scratch: Optional[list] = None, **kwargs):
        """generate_rolling; an engine that runs the whole call in one engine call overrides it.  scratch: sessions
        the full path may use (generate_full opens and closes its own here)."""
        return self.generate_rolling(*args, **kwargs)

    def make_controls(self, *, eos_token_id=None, stop_token_ids=None, suppress_token_ids=None, repetition_penalty=1.0,
                      no_repeat_ngram_size=0, max_consecutive_text_tokens=0, wait_token_id=None) -> Controls:
        stop = {int(t) for t in (stop_token_ids or ())}
        if eos_token_id is not None:
            stop.add(int(eos_token_id))
        sup = [int(t) for t in (suppress_token_ids or ()) if 0 <= int(t) < self.vocab]
        wait = int(wait_token_id) if wait_token_id is not None and int(wait_token_id) not in set(sup) else None
        return Controls(frozenset(stop), np.asarray(sorted(set(sup)), np.int32), float(repetition_penalty),
                        int(no_repeat_ngram_size), int(max_consecutive_text_tokens),
                        wait if wait is not None and 0 <= wait < self.vocab else -1,
                        None if eos_token_id is None else int(eos_token_id))

    def _pick_histories(self, hists: List[List[int]], ctl: Controls) -> np.ndarray:
        """pick() with one explicit history per logit row (rows of the last forward, in order)."""
        off = np.zeros(len(hists), np.int32)
        ln = np.asarray([len(h) for h in hists], np.int32)
        if len(hists) > 1:
            off[1:] = np.cumsum(ln[:-1])
        flat = np.asarray([t for h in hists for t in h], np.int32)
        return self.pick(flat, off, ln, ctl)

    def _step(self, sids: List[int], toks: List[int]) -> None:
        self.forward(sids, [(np.asarray([t], np.int32), None) for t in toks], [1] * len(sids))

    # -- generate_full_hypothesis_rolling (model.py:991-1250), N sessions in lockstep ------------------------------
    def _generate_rolling(self, sids: Sequence[int], frame_hidden: Sequence[np.ndarray], states: Sequence[Optional[RollingState]],
                         template_token_ids: Sequence[int], audio_placeholder_token_id: int,
                         drafts: Optional[Sequence[Optional[Sequence[int]]]] = None, *, max_new_tokens: int = 128,
                         eos_token_id=None, stop_token_ids=None, suppress_token_ids=None, repetition_penalty=1.0,
                         no_repeat_ngram_size=0, max_consecutive_text_tokens=0, wait_token_id=None, bos_token_id=None):
        """Returns (tokens per session, stats per session, new RollingState per session)."""
        head, tail = split_template(template_token_ids, audio_placeholder_token_id)
        ctl = self.make_controls(eos_token_id=eos_token_id, stop_token_ids=stop_token_ids,
                                 suppress_token_ids=suppress_token_ids, repetition_penalty=repetition_penalty,
                                 no_repeat_ngram_size=no_repeat_ngram_size,
                                 max_consecutive_text_tokens=max_consecutive_text_tokens, wait_token_id=wait_token_id)
        n = len(sids)
        out_tokens: List[Optional[List[int]]] = [None] * n
        out_stats: List[Optional[Dict]] = [None] * n
        new_states = list(states)
        full, live = self._rolling_plan(sids, frame_hidden, states, head, tail, drafts, max_new_tokens, ctl)
        for i, fh in full:
            expanded = head + [int(audio_placeholder_token_id)] * fh.shape[0] + tail
            out_tokens[i] = self.generate_full(fh, prefix_token_ids=expanded,
                                               audio_placeholder_token_id=audio_placeholder_token_id,
                                               max_new_tokens=max_new_tokens, controls=ctl, bos_token_id=bos_token_id)
            out_stats[i] = {"decoder_path": "full"}
        if not live:
            return out_tokens, out_stats, new_states

        self.forward([sids[i] for i, *_ in live], [blk for _, blk, _, _ in live], [len(d) + 1 for _, _, d, _ in live])
        picks = self._pick_histories([d[:j] for _, _, d, _ in live for j in range(len(d) + 1)], ctl)

        seq = []                        # sessions decoding sequentially: [i, gen, budget, steps, pending token]
        base = 0
        for i, (src, _), draft, stats in live:
            dl = len(draft)
            row = picks[base: base + dl + 1]
            base += dl + 1
            fh_steps = stats["audio_steps"]
            prefix_len = len(head) + fh_steps + len(tail)
            accepted, corrected = dl, None
            for j in range(dl):
                if int(row[j]) != draft[j]:
                    accepted, corrected = j, int(row[j])
                    break
            gen = draft[:accepted]
            stats["draft_accepted"] = accepted
            stats["draft_all_accepted"] = bool(dl) and accepted == dl
            stats["_corrected"] = corrected is not None
            if corrected is not None:
                self.crop(sids[i], prefix_len + accepted)
                gen = gen + [corrected]
                if corrected not in ctl.stop_ids and len(gen) < max_new_tokens:
                    seq.append([i, gen, int(max_new_tokens) - len(gen), 0, corrected])
            elif dl < max_new_tokens:
                budget = int(max_new_tokens) - dl
                tok = int(row[dl])                     # the verify row after the draft is the tail's first pick
                gen = gen + [tok]
                if tok in ctl.stop_ids or budget == 1:
                    seq.append([i, gen, budget, 1, None])
                else:
                    seq.append([i, gen, budget, 1, tok])
            out_tokens[i] = gen
        while True:
            active = [e for e in seq if e[4] is not None]
            if not active:
                break
            self._step([sids[e[0]] for e in active], [e[4] for e in active])
            p = self._pick_histories([e[1] for e in active], ctl)
            for e, tok in zip(active, p):
                tok = int(tok)
                e[1].append(tok)
                e[3] += 1
                e[4] = None if (tok in ctl.stop_ids or e[3] == e[2]) else tok
        steps = {e[0]: e[3] for e in seq}
        for e in seq:
            out_tokens[e[0]] = e[1]
        for i, _, _, stats in live:
            corrected = stats.pop("_corrected")
            self.crop(sids[i], len(head) + stats["audio_steps"])
            new_states[i] = RollingState(tuple(head), len(head), stats["audio_steps"])
            stats["decode_steps"] = steps.get(i, 0) + (1 if corrected else 0)
            out_stats[i] = self._rolling_stats(stats)
        return out_tokens, out_stats, new_states

    _ROLLING_STATS = ("decoder_path", "decoder_rebuilt", "draft_tokens", "draft_accepted", "draft_all_accepted",
                      "decode_steps", "prefill_positions", "audio_steps", "audio_delta_steps", "reused_audio_steps",
                      "prompt_head_tokens", "template_tail_tokens")

    @classmethod
    def _rolling_stats(cls, stats: Dict) -> Dict:
        return {k: stats[k] for k in cls._ROLLING_STATS}

    def _rolling_plan(self, sids, frame_hidden, states, head: List[int], tail: List[int], drafts, max_new_tokens: int,
                      ctl: Controls):
        """generate_rolling's per-session decisions before any forward.  Returns (full, live): the sessions that take
        the full path as (i, frame rows), the others as (i, (row sources, delta frame rows), draft, stats skeleton).
        A session whose state does not validate is reset here, so its block rebuilds [head + audio] from scratch."""
        n = len(sids)
        drafts = list(drafts) if drafts is not None else [None] * n
        full, live = [], []
        for i in range(n):
            fh = _frame_rows(frame_hidden[i])
            audio_steps = int(fh.shape[0])
            if max_new_tokens <= 0 or audio_steps == 0:
                full.append((i, fh))
                continue
            draft = [int(t) for t in (drafts[i] or [])]
            for k, t in enumerate(draft):
                if t in ctl.stop_ids:
                    draft = draft[:k]
                    break
            draft = draft[:int(max_new_tokens)]
            st = states[i]
            valid = (st is not None and st.head_token_ids == tuple(head) and 0 <= st.audio_steps <= audio_steps
                     and self.session_len(sids[i]) == st.head_len + st.audio_steps)
            if valid:
                reused = int(st.audio_steps)
                audio_rows = fh[reused:]
                lead: List[int] = []
            else:
                reused = 0
                audio_rows = fh
                lead = list(head)
            if len(lead) + audio_rows.shape[0] + len(tail) + len(draft) == 0:
                full.append((i, fh))
                continue
            src = np.concatenate([np.asarray(lead, np.int32), -1 - np.arange(audio_rows.shape[0], dtype=np.int32),
                                  np.asarray(tail + draft, np.int32)])
            if not valid:
                self.reset_session(sids[i])
            live.append((i, (src, audio_rows), draft, {
                "decoder_path": "rolling+draft" if draft else "rolling",
                "decoder_rebuilt": not valid,
                "draft_tokens": len(draft),
                "prefill_positions": int(src.shape[0]),
                "audio_steps": audio_steps,
                "audio_delta_steps": int(audio_rows.shape[0]),
                "reused_audio_steps": reused,
                "prompt_head_tokens": len(head),
                "template_tail_tokens": len(tail),
            }))
        return full, live

    # -- generate_full_hypothesis_from_cached_audio (model.py:839-989), cached path -----------------------------------
    def full_prefix(self, frame_hidden, *, prefix_token_ids: Optional[Sequence[int]] = None,
                    audio_placeholder_token_id: Optional[int] = None, prompt_token_ids: Optional[Sequence[int]] = None,
                    bos_token_id=None) -> Tuple[np.ndarray, object]:
        """The cached path's input rows: (row sources int32 — a token id, or -1 - j for frame row j —, the frame rows)."""
        fh = _frame_rows(frame_hidden).reshape(-1, self.dims.d_model)
        if prefix_token_ids is not None:
            if audio_placeholder_token_id is None:
                raise ValueError("audio_placeholder_token_id is required when prefix_token_ids is set")
            prefix = np.asarray([int(t) for t in prefix_token_ids], np.int32)
            mask = prefix == int(audio_placeholder_token_id)
            if int(mask.sum()) != fh.shape[0]:
                raise ValueError("prefix_token_ids must contain exactly one audio placeholder per cached audio step; got "
                                 f"{[int(mask.sum())]} placeholders for {fh.shape[0]} cached steps")
            src = prefix.copy()
            src[mask] = -1 - np.arange(fh.shape[0], dtype=np.int32)     # masked_scatter, in order (model.py:129-153)
        else:
            src = -1 - np.arange(fh.shape[0], dtype=np.int32)
        if prompt_token_ids is None:
            prompt = [] if prefix_token_ids is not None else [int(bos_token_id)]
        else:
            prompt = [int(t) for t in prompt_token_ids]
        return np.concatenate([src, np.asarray(prompt, np.int32)]), fh

    def _generate_full(self, frame_hidden: np.ndarray, *, prefix_token_ids: Optional[Sequence[int]] = None,
                      audio_placeholder_token_id: Optional[int] = None, prompt_token_ids: Optional[Sequence[int]] = None,
                      max_new_tokens: int = 128, controls: Optional[Controls] = None, bos_token_id=None,
                      **control_kwargs) -> List[int]:
        """One stream on a scratch session: generate_full_batch with N = 1."""
        if max_new_tokens < 0:
            raise ValueError("max_new_tokens must be >= 0")
        if max_new_tokens == 0:
            return []
        src, fh = self.full_prefix(frame_hidden, prefix_token_ids=prefix_token_ids,
                                   audio_placeholder_token_id=audio_placeholder_token_id,
                                   prompt_token_ids=prompt_token_ids, bos_token_id=bos_token_id)
        if src.shape[0] == 0:
            return []
        sid = self.open_session()
        try:
            return self._generate_full_batch([sid], [fh], [src], max_new_tokens=max_new_tokens, controls=controls,
                                             **control_kwargs)[0]
        finally:
            self.close_session(sid)

    def _generate_full_batch(self, sids: Sequence[int], frame_rows: Sequence, prefixes: Sequence[Sequence[int]], *,
                             max_new_tokens: int = 128, controls: Optional[Controls] = None,
                             **control_kwargs) -> List[List[int]]:
        """The cached path for N caller-owned sessions in lockstep.  Session i is reset and forwards prefixes[i] (row
        sources: a token id, or -1 - j for row j of frame_rows[i]) with one logit row; each step then forwards one row
        per session still decoding, in session order, and picks over that session's generated tokens.  A session stops
        on a stop id or after max_new_tokens picks.  Returns the tokens per session; every session is reset on return."""
        if max_new_tokens < 0:
            raise ValueError("max_new_tokens must be >= 0")
        ctl = controls if controls is not None else self.make_controls(**control_kwargs)
        n = len(sids)
        blocks = []
        for fr, p in zip(frame_rows, prefixes):
            src = np.asarray(p, np.int32).reshape(-1)
            if src.shape[0] == 0:
                raise ValueError("every session needs a non-empty prefix")
            blocks.append((src, None if fr is None else _frame_rows(fr).reshape(-1, self.dims.d_model)))
        if len(blocks) != n:
            raise ValueError("sids, frame_rows and prefixes must have the same length")
        for sid in sids:
            self.reset_session(sid)
        try:
            gens: List[List[int]] = [[] for _ in range(n)]
            if max_new_tokens == 0 or n == 0:
                return gens
            self.forward(list(sids), blocks, [1] * n)
            live = list(range(n))
            while live:
                picks = self._pick_histories([gens[i] for i in live], ctl)
                nxt = []
                for i, tok in zip(live, picks):
                    gens[i].append(int(tok))
                    if int(tok) not in ctl.stop_ids and len(gens[i]) < max_new_tokens:
                        nxt.append(i)
                live = nxt
                if live:
                    self._step([sids[i] for i in live], [gens[i][-1] for i in live])
            return gens
        finally:
            for sid in sids:
                self.reset_session(sid)


class QwenTextEngine(TextDecodeDriver, L.Engine):
    """The text decoder on the H100.  No CPU fallback: construction fails without the CUDA library or a device.
    Embedding rows may be host arrays or fp32 CUDA tensors; the latter are read in place by the forward."""

    device_rows = True
    CREATE, DESTROY = "wlk_qtext_create", "wlk_qtext_destroy"
    LOAD_TENSOR, FINALIZE, MEMORY = "wlk_qtext_load_tensor", "wlk_qtext_finalize_weights", "wlk_qtext_memory"
    SESSION_OPEN, SESSION_CLOSE, SESSION_RESET = "wlk_qtext_session_open", "wlk_qtext_session_close", "wlk_qtext_session_reset"

    def __init__(self, dims: QwenTextDims, state_dict: Optional[Dict[str, np.ndarray]] = None, *, precision: str = "bf16",
                 device: int = 0, max_sessions: int = 8, max_batch: int = 8):
        self.dims = dims
        self.vocab = dims.vocab
        self._create(L.wlk_qtext_dims(*dims.as_tuple()), precision=precision, device=device, max_sessions=max_sessions,
                     max_batch=max_batch)
        self._n_logit = 0
        self._dev_rows = None                    # device rows the last forward reads: alive until its pick synchronizes
        # HF's fp32 RoPE frequencies; a state dict that carries the model's own buffer overrides them
        self.load_tensor("rotary_emb.inv_freq", rope_inv_freq(dims.rope_theta, dims.head_dim))
        if state_dict is not None:
            self.load_state_dict(state_dict)

    def session_len(self, sid: int) -> int:
        n = C.c_int32()
        L.check(self.lib.wlk_qtext_session_len(self.h, int(sid), C.byref(n)))
        return n.value

    def crop(self, sid: int, length: int) -> None:
        L.check(self.lib.wlk_qtext_crop(self.h, int(sid), int(length)))

    def _pack(self, blocks):
        """blocks as forward takes them -> (flat row sources, row offsets, embedding rows, their count, row pitch).
        Pitch 0: host fp32 rows.  Otherwise one fp32 CUDA tensor the engine reads in place, complete on return."""
        if any(getattr(e, "is_cuda", False) and len(e) for _, e in blocks):
            return self._pack_device(blocks)
        srcs, embs, offs, base = [], [], [0], 0
        for src, emb in blocks:
            src = np.asarray(src, np.int32).copy()
            if emb is not None and len(emb):
                src[src < 0] -= base
                e = _frame_rows(emb).reshape(-1, self.dims.d_model)
                embs.append(e)
                base += e.shape[0]
            srcs.append(src)
            offs.append(offs[-1] + src.shape[0])
        emb = np.concatenate(embs) if embs else np.zeros((1, self.dims.d_model), np.float32)
        return np.concatenate(srcs).astype(np.int32), np.asarray(offs, np.int32), emb, base, 0

    def _pack_device(self, blocks):
        import torch
        d = self.dims.d_model
        srcs, parts, offs, base = [], [], [0], 0
        for src, emb in blocks:
            src = np.asarray(src, np.int32).copy()
            if emb is not None and len(emb):
                if not getattr(emb, "is_cuda", False):
                    raise ValueError("a forward takes its embedding rows either all from the host or all from the device")
                e = emb.reshape(-1, d)
                src[src < 0] -= base
                parts.append(e)
                base += e.shape[0]
            srcs.append(src)
            offs.append(offs[-1] + src.shape[0])
        rows = parts[0] if len(parts) == 1 else torch.cat(parts)       # one session: its rows in place
        if rows.dtype != torch.float32 or rows.stride(-1) != 1 or (rows.shape[0] > 1 and rows.stride(0) < d):
            rows = rows.float().contiguous()
        ld = rows.stride(0) if rows.shape[0] > 1 else d
        torch.cuda.current_stream(rows.device).synchronize()         # the rows are complete before the engine reads them
        return np.concatenate(srcs).astype(np.int32), np.asarray(offs, np.int32), rows, base, int(ld)

    @staticmethod
    def _rows_ptr(rows, ld):
        return C.c_void_p(rows.data_ptr()) if ld else _ptr(rows)

    def forward(self, sids: Sequence[int], blocks, logit_rows: Sequence[int]) -> None:
        """blocks[i] = (row_src int32 [r], embeds [k][d] or None): row_src >= 0 is a token id, -1 - j is embeds row j.
        Embeddings that are CUDA tensors go through wlk_qtext_forward_device without leaving the GPU."""
        flat, off, rows, n_rows, ld = self._pack(blocks)
        ids = np.asarray(list(sids), np.int32)
        lr = np.asarray(list(logit_rows), np.int32)
        if ld:
            self._dev_rows = rows                    # alive until the pick that follows synchronizes
            L.check(self.lib.wlk_qtext_forward_device(self.h, _ptr(ids), len(ids), _ptr(flat), _ptr(off),
                                                      self._rows_ptr(rows, ld), ld, n_rows, _ptr(lr)))
        else:
            L.check(self.lib.wlk_qtext_forward(self.h, _ptr(ids), len(ids), _ptr(flat), _ptr(off), _ptr(rows), n_rows,
                                               _ptr(lr)))
        self._n_logit = int(lr.sum())

    def generate_full_batch(self, sids: Sequence[int], frame_rows: Sequence, prefixes: Sequence[Sequence[int]], *,
                            max_new_tokens: int = 128, controls: Optional[Controls] = None,
                            **control_kwargs) -> List[List[int]]:
        """TextDecodeDriver.generate_full_batch in one engine call (wlk_qtext_generate_full): the decode loop runs in
        the engine and the generated histories stay on the device.  Same rounds, same tokens.  Invalid input raises
        WlkError (the engine checks it) and leaves every named session reset."""
        ctl = controls if controls is not None else self.make_controls(**control_kwargs)
        n = len(sids)
        if len(frame_rows) != n or len(prefixes) != n:
            raise ValueError("sids, frame_rows and prefixes must have the same length")
        blocks = [(np.asarray(p, np.int32).reshape(-1), fr) for fr, p in zip(frame_rows, prefixes)]
        for i, (src, fr) in enumerate(blocks):          # the engine sees the rows packed: check each stream's own bound
            if src.size and int(-1 - src.min()) >= (0 if fr is None else len(fr)):
                raise ValueError(f"session {i}: frame row {int(-1 - src.min())} past its {0 if fr is None else len(fr)} rows")
        flat, off, rows, n_rows, ld = (self._pack(blocks) if blocks else       # the engine rejects n = 0
                                       (np.zeros(1, np.int32), np.zeros(1, np.int32), np.zeros((1, 1), np.float32), 0, 0))
        ids = np.asarray(list(sids), np.int32)
        stop = np.asarray(sorted(ctl.stop_ids), np.int32) if ctl.stop_ids else np.zeros(1, np.int32)
        sup = ctl.suppress if len(ctl.suppress) else np.zeros(1, np.int32)
        toks = np.zeros((max(n, 1), max(int(max_new_tokens), 1)), np.int32)
        counts = np.zeros(max(n, 1), np.int32)
        with self.phase_lock:
            L.check(self.lib.wlk_qtext_generate_full(
                self.h, _ptr(ids), n, _ptr(flat), _ptr(off), self._rows_ptr(rows, ld), ld, n_rows, int(max_new_tokens),
                _ptr(stop), len(ctl.stop_ids), _ptr(sup), len(ctl.suppress), float(ctl.penalty), ctl.ngram,
                ctl.max_consecutive, ctl.wait_id, _ptr(toks), _ptr(counts)))
            self._n_logit = 0
        return [toks[i, :counts[i]].tolist() for i in range(n)]

    def generate_rolling_batch(self, sids: Sequence[int], frame_hidden: Sequence, states: Sequence[Optional[RollingState]],
                               template_token_ids: Sequence[int], audio_placeholder_token_id: int,
                               drafts: Optional[Sequence[Optional[Sequence[int]]]] = None, *, max_new_tokens: int = 128,
                               bos_token_id=None, scratch: Optional[list] = None, **control_kwargs):
        """TextDecodeDriver.generate_rolling with its verify pass and decode loop in one engine call
        (wlk_qtext_generate_rolling): the picks, the draft check and the generated histories stay on the device.  Same
        rounds, tokens, stats and states.

        Sessions take the full path when they have no audio steps, when max_new_tokens <= 0 or when their block would
        be empty; those go through one generate_full_batch on scratch sessions: the open sessions of the caller's
        `scratch` list (B200QwenTextDecoder passes the ones it keeps for the non-rolling generate), and for the rest
        sessions opened for the call and closed after it, which need free slots within max_sessions while it runs.

        Sessions whose rolling state does not validate are reset before the engine call, as the driver resets them.
        Input the engine rejects raises WlkError before any work and changes no session beyond that reset; a failure
        after the work started resets every named session.  Either way the states the caller keeps no longer validate
        for the reset sessions, and the next call rebuilds them."""
        head, tail = split_template(template_token_ids, audio_placeholder_token_id)
        ctl = self.make_controls(**control_kwargs)
        n = len(sids)
        if n and max_new_tokens < 0:
            raise ValueError("max_new_tokens must be >= 0")
        out_tokens: List[Optional[List[int]]] = [None] * n
        out_stats: List[Optional[Dict]] = [None] * n
        new_states = list(states)
        with self.phase_lock:
            full, live = self._rolling_plan(sids, frame_hidden, states, head, tail, drafts, max_new_tokens, ctl)
            if full:
                self._generate_full_scratch(full, head, tail, audio_placeholder_token_id, max_new_tokens, ctl,
                                            out_tokens, out_stats, scratch)
            if not live:
                return out_tokens, out_stats, new_states
            m = len(live)
            flat, off, rows, n_rows, ld = self._pack([blk for _, blk, _, _ in live])
            ids = np.asarray([sids[i] for i, *_ in live], np.int32)
            dl = np.asarray([len(d) for _, _, d, _ in live], np.int32)
            prefix = np.asarray([len(head) + st["audio_steps"] + len(tail) for *_, st in live], np.int32)
            stop = np.asarray(sorted(ctl.stop_ids), np.int32) if ctl.stop_ids else np.zeros(1, np.int32)
            sup = ctl.suppress if len(ctl.suppress) else np.zeros(1, np.int32)
            toks = np.zeros((m, int(max_new_tokens)), np.int32)
            counts = np.zeros(m, np.int32)
            res = np.zeros((m, 4), np.int32)
            try:
                L.check(self.lib.wlk_qtext_generate_rolling(
                    self.h, _ptr(ids), m, _ptr(flat), _ptr(off), self._rows_ptr(rows, ld), ld, n_rows, _ptr(dl),
                    _ptr(prefix), len(tail), int(max_new_tokens), _ptr(stop), len(ctl.stop_ids), _ptr(sup),
                    len(ctl.suppress), float(ctl.penalty), ctl.ngram, ctl.max_consecutive, ctl.wait_id, _ptr(toks),
                    _ptr(counts), _ptr(res)))
            finally:
                self._n_logit = 0
        for k, (i, _, _, stats) in enumerate(live):
            accepted, decode_steps, all_accepted, _ = (int(v) for v in res[k])
            out_tokens[i] = toks[k, :counts[k]].tolist()
            stats.update(draft_accepted=accepted, draft_all_accepted=bool(all_accepted), decode_steps=decode_steps)
            out_stats[i] = self._rolling_stats(stats)
            new_states[i] = RollingState(tuple(head), len(head), stats["audio_steps"])
        return out_tokens, out_stats, new_states

    def _generate_full_scratch(self, full, head, tail, placeholder, max_new_tokens, ctl, out_tokens, out_stats,
                               keep: Optional[list] = None):
        """generate_rolling_batch's full-path sessions [(i, frame rows)]: generate_full_batch in waves of max_batch
        over the open sessions of `keep`, plus sessions opened for the call and closed after it for the rest."""
        srcs = []
        for i, fh in full:
            expanded = head + [int(placeholder)] * fh.shape[0] + tail
            srcs.append(self.full_prefix(fh, prefix_token_ids=expanded, audio_placeholder_token_id=placeholder)[0])
            out_tokens[i] = []
            out_stats[i] = {"decoder_path": "full"}
        todo = [k for k, s in enumerate(srcs) if s.shape[0]] if max_new_tokens > 0 else []
        need = min(len(todo), self.max_batch)
        scratch = list(keep or [])[:need]
        temp = []
        try:
            while len(scratch) < need:
                temp.append(self.open_session())
                scratch.append(temp[-1])
            for a in range(0, len(todo), self.max_batch):
                wave = todo[a: a + self.max_batch]
                got = self.generate_full_batch(scratch[:len(wave)], [full[k][1] for k in wave], [srcs[k] for k in wave],
                                               max_new_tokens=max_new_tokens, controls=ctl)
                for k, g in zip(wave, got):
                    out_tokens[full[k][0]] = g
        finally:
            for sid in temp:
                self.close_session(sid)

    def adapter_dims(self) -> Tuple[int, int, int]:
        """(in_dim, blocks, hidden width) of the loaded frame adapter; in_dim 0 without one."""
        a, b, c = C.c_int32(), C.c_int32(), C.c_int32()
        L.check(self.lib.wlk_qtext_adapter_dims(self.h, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, c.value

    def adapt(self, x, out=None):
        """The frame adapter (wlk_qtext_adapt) over fp32 CUDA rows x [rows, in_dim] (any row pitch): a new fp32 CUDA tensor
        [rows, d_model], or `out` (a [rows, >= d_model] row-major view) filled in place."""
        import torch
        if x.dim() != 2 or x.dtype != torch.float32 or not x.is_cuda or (x.shape[0] and x.stride(1) != 1):
            raise ValueError("adapt takes fp32 CUDA rows [rows, in_dim] with unit column stride")
        rows = int(x.shape[0])
        if out is None:
            out = torch.empty(rows, self.dims.d_model, dtype=torch.float32, device=x.device)
        torch.cuda.current_stream(x.device).synchronize()
        L.check(self.lib.wlk_qtext_adapt(self.h, C.c_void_p(x.data_ptr()), rows, int(x.stride(0)),
                                         C.c_void_p(out.data_ptr()), int(out.stride(0))))
        return out

    def pick(self, hist: np.ndarray, hist_off: np.ndarray, hist_len: np.ndarray, ctl: Controls,
             return_values: bool = False):
        n_hist = len(hist)
        hist = np.ascontiguousarray(hist, np.int32) if n_hist else np.zeros(1, np.int32)
        off = np.ascontiguousarray(hist_off, np.int32)
        ln = np.ascontiguousarray(hist_len, np.int32)
        picks = np.zeros(max(self._n_logit, 1), np.int32)
        vals = np.zeros(max(self._n_logit, 1), np.float32)
        sup = ctl.suppress if len(ctl.suppress) else np.zeros(1, np.int32)
        L.check(self.lib.wlk_qtext_pick(self.h, _ptr(hist), n_hist, _ptr(off), _ptr(ln), _ptr(sup),
                                        len(ctl.suppress), float(ctl.penalty), ctl.ngram, ctl.max_consecutive, ctl.wait_id,
                                        _ptr(picks), _ptr(vals)))
        picks, vals = picks[:self._n_logit], vals[:self._n_logit]
        return (picks, vals) if return_values else picks

    def logits(self, row0: int = 0, n_rows: Optional[int] = None) -> np.ndarray:
        n_rows = self._n_logit - row0 if n_rows is None else n_rows
        out = np.zeros((max(n_rows, 1), self.vocab), np.float32)
        L.check(self.lib.wlk_qtext_logits(self.h, int(row0), int(n_rows), _ptr(out)))
        return out[:n_rows]

    # -- op-level (device pointers, e.g. torch tensors' data_ptr(); activations are fp32 or bf16 as the precision) ----
    def op_rmsnorm(self, x_ptr, w_ptr, out_ptr, rows: int, out_row: Optional[Sequence[int]] = None) -> None:
        orow = None if out_row is None else np.ascontiguousarray(out_row, np.int32)
        L.check(self.lib.wlk_qtext_op_rmsnorm(self.h, x_ptr, w_ptr, out_ptr, int(rows), None if orow is None else _ptr(orow)))

    @staticmethod
    def _rows(row_pos, row_slot, kv_ptrs):
        pos = np.ascontiguousarray(row_pos, np.int32)
        slot = np.ascontiguousarray(row_slot, np.int32)
        kv = (C.c_void_p * len(kv_ptrs))(*[int(p) for p in kv_ptrs])
        return pos, slot, kv

    def op_qk_rope(self, qkv_ptr, q_norm_ptr, k_norm_ptr, row_pos, row_slot, kv_ptrs: Sequence[int], layer: int,
                   q_out_ptr) -> None:
        pos, slot, kv = self._rows(row_pos, row_slot, kv_ptrs)
        L.check(self.lib.wlk_qtext_op_qk_rope(self.h, qkv_ptr, q_norm_ptr, k_norm_ptr, _ptr(pos), _ptr(slot), len(pos), kv,
                                              len(kv_ptrs), int(layer), q_out_ptr))

    def op_attention(self, q_ptr, row_pos, row_slot, kv_ptrs: Sequence[int], layer: int, out_ptr) -> None:
        pos, slot, kv = self._rows(row_pos, row_slot, kv_ptrs)
        L.check(self.lib.wlk_qtext_op_attention(self.h, q_ptr, _ptr(pos), _ptr(slot), len(pos), kv, len(kv_ptrs), int(layer),
                                                out_ptr))

    def op_swiglu(self, gu_ptr, hid_ptr, rows: int) -> None:
        L.check(self.lib.wlk_qtext_op_swiglu(self.h, gu_ptr, hid_ptr, int(rows)))
