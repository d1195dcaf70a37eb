"""Batching-aware caller shim (SURVEY.md section 8f item 1).

WhisperLiveKit drives every session from its own worker thread (reference audio_processor.py:543-551:
``await asyncio.to_thread(self.transcription.process_iter)``) and each thread issues single-session model
calls (``_encode``, ``_get_logits_and_cross_attn``, ... -- simul_whisper/align_att_base.py:174-322).  On the
H100 engine the unit of efficiency is a *batched* call: one ``wlk_encode`` over 96 sessions costs about as
much GPU time as 96 back-to-back single-session calls cost in launch latency alone.

``BatchingEngine`` keeps the per-session call surface (it duck-types ``WhisperEngine``) and coalesces
concurrent calls of the same kind into one C-ABI call:

    caller threads                      dispatcher thread
    --------------                      -----------------
    eng.encode([sid])   --submit-->     gather requests with the same (op, static args)
    (blocks on a Future)                until every caller of the running cohort has submitted, or `max_wait_s` passed
                         <--result--    engine.encode([sid_a, sid_b, ...]) ; split the results

Cohorts.  A policy iteration (``infer()``: encode, prefill, then a data-dependent number of token steps, each a
host sync) is bracketed by ``begin_iter()`` / ``end_iter()``.  Callers are admitted in COHORTS: while one cohort is
inside its iteration, newly arriving callers wait at ``begin_iter()``; when the last member leaves, everybody waiting
is admitted at once.  The members of a cohort advance in lockstep, so every engine call serves the whole cohort --
without admission control, streams arriving at their own phases interleave their encodes with other streams' token
steps and every call degenerates to a dozen sessions while costing the same fixed step latency.  The cohort size
regulates itself: the longer a cohort takes, the more callers arrive meanwhile (n = arrival_rate x T(n)); an idle
engine admits a lone caller immediately.

Semantics are unchanged: one call in flight per session (as the reference guarantees), results are what the
single-session call would have returned (the batched kernels are batch-invariant: tests/test_gpu_parity.py
``test_batched_equals_single``); when a merged call fails its requests are replayed one by one, so an error reaches
only the caller whose session caused it.
``submit()`` returns a ``concurrent.futures.Future`` so an asyncio caller can ``await asyncio.wrap_future(f)``
instead of parking an OS thread per stream.
"""
from __future__ import annotations

import threading
import time
from concurrent.futures import Future
from typing import Any, Dict, List, Sequence

# op name -> (takes one payload item per session, takes one payload shared by the batch).  Single-session requests of
# one op (and equal static arguments) are merged into one engine call over the concatenated sessions.
_OPS = {
    # WhisperEngine (AlignAtt hooks)
    "encode": (False, False), "decode": (True, False), "no_speech_prob": (False, False), "suppress": (False, True),
    "greedy_and_align": (False, False), "select": (True, True),
    # QwenTowerEngine (QwenAudioCausalKVEncoder.forward_chunk / StreamingMelExtractor.append per stream: mel_append)
    "forward_chunk": (True, False), "mel_append": (True, False), "mel_flush": (False, False),
    "flush_pending": (False, False),
}
_BATCHED = tuple(_OPS)


class _Request:
    __slots__ = ("op", "key", "sids", "payload", "future", "t_submit")

    def __init__(self, op, key, sids, payload):
        self.op, self.key, self.sids, self.payload = op, key, list(sids), payload
        self.future: Future = Future()
        self.t_submit = time.perf_counter()


class BatchingEngine:
    """Duck-types ``WhisperEngine``; see the module docstring.

    max_batch    upper bound on sessions per engine call (the engine's own ``max_batch``)
    max_wait_s   how long the dispatcher holds the first request of a batch for companions
    """

    def __init__(self, engine, max_batch: int = 64, max_wait_s: float = 0.002, cohort_wait_s: float = 0.05):
        self.engine = engine
        self.max_batch = int(max_batch)
        self.max_wait_s = float(max_wait_s)
        self.cohort_wait_s = float(cohort_wait_s)
        self._lock = threading.RLock()              # serialises every call into the wrapped engine
        self._cv = threading.Condition()
        self._pending: List[_Request] = []
        self._cohort = set()                        # thread ids admitted to the running policy iteration
        self._waiting = set()                       # thread ids parked in begin_iter() until the cohort drains
        self._stop = False
        self.stats: Dict[str, Any] = dict(calls=0, requests=0, sessions=0, max_sessions_in_call=0,
                                          cohorts=0, cohort_sessions=0, max_cohort=0,
                                          by_op={op: dict(calls=0, sessions=0) for op in _BATCHED})
        self._thread = threading.Thread(target=self._run, name="wlk-b200-batcher", daemon=True)
        self._thread.start()

    # -- static attributes of the wrapped engine -------------------------------------------------------
    def __getattr__(self, name):
        # anything not batched (attributes such as dims/specials/align_heads, and debug taps) goes straight through
        attr = getattr(self.engine, name)
        if callable(attr):
            def locked(*a, **k):
                with self._lock:
                    return attr(*a, **k)
            return locked
        return attr

    # -- bracket a caller's policy iteration: lets the dispatcher fire as soon as everybody has arrived --
    def _admit(self) -> None:
        """Condition held, cohort empty: everybody waiting becomes the next cohort."""
        if self._waiting:
            self._cohort, self._waiting = self._waiting, set()
            st = self.stats
            st["cohorts"] += 1
            st["cohort_sessions"] += len(self._cohort)
            st["max_cohort"] = max(st["max_cohort"], len(self._cohort))
            self._cv.notify_all()

    def begin_iter(self) -> None:
        me = threading.get_ident()
        with self._cv:
            self._waiting.add(me)
            while not self._stop:
                if not self._cohort:
                    self._admit()
                if me in self._cohort:
                    return
                self._cv.wait()
            self._waiting.discard(me)
            raise RuntimeError("BatchingEngine is closed")

    def end_iter(self) -> None:
        me = threading.get_ident()
        with self._cv:
            self._cohort.discard(me)
            self._waiting.discard(me)
            if not self._cohort:
                self._admit()
            self._cv.notify_all()

    # -- submission ---------------------------------------------------------------------------------------
    def submit(self, op: str, sids: Sequence[int], *payload, **static) -> Future:
        """Queue one request; the Future resolves to what ``engine.<op>(sids, ...)`` returns."""
        if op not in _BATCHED:
            raise ValueError(f"{op} is not a batched operation")
        key = (op,) + tuple(sorted((k, _freeze(v)) for k, v in static.items()))
        if op == "suppress":
            key += (_freeze(payload[0]),)
        elif op == "select":
            key += (_freeze(payload[1]),)
        req = _Request(op, key, sids, (payload, static))
        with self._cv:
            if self._stop:
                raise RuntimeError("BatchingEngine is closed")
            self._pending.append(req)
            self._cv.notify_all()
        return req.future

    def encode(self, sids):
        return self.submit("encode", sids).result()

    def decode(self, sids, tokens, sot_index: int = 0):
        return self.submit("decode", sids, [list(t) for t in tokens], sot_index=int(sot_index)).result()

    def no_speech_prob(self, sids):
        return self.submit("no_speech_prob", sids).result()

    def suppress(self, sids, token_ids):
        return self.submit("suppress", sids, tuple(int(t) for t in token_ids)).result()

    def greedy_and_align(self, sids, window_iters: int = 16):
        return self.submit("greedy_and_align", sids, window_iters=int(window_iters)).result()

    def select(self, sids, suppress, first_ids=(), first_mask=None, biases=None, window_iters: int = 16):
        """The fused pick (WhisperEngine.select); per session: (first-iteration flag, DRY bias pairs)."""
        n = len(sids)
        fm = list(first_mask) if first_mask is not None else [False] * n
        bs = [list(b) for b in biases] if biases is not None else [[] for _ in range(n)]
        items = [(bool(fm[i]), bs[i]) for i in range(n)]
        shared = (tuple(int(t) for t in suppress), tuple(int(t) for t in first_ids))
        return self.submit("select", sids, items, shared, window_iters=int(window_iters)).result()

    # Qwen3 tower engine
    def forward_chunk(self, sids, mels):
        return self.submit("forward_chunk", sids, list(mels)).result()

    def mel_append(self, sids, audios):
        return self.submit("mel_append", sids, list(audios)).result()

    def mel_flush(self, sids):
        return self.submit("mel_flush", sids).result()

    def flush_pending(self, sids):
        return self.submit("flush_pending", sids).result()

    # -- dispatcher -----------------------------------------------------------------------------------------
    def _take_batch(self) -> List[_Request]:
        """Called with the condition held and at least one request pending: wait for companions of the oldest
        request, then remove and return every pending request with its key (up to max_batch sessions)."""
        first = self._pending[0]
        # inside a cohort every member is about to submit (it is between two engine calls of its policy iteration, a few
        # hundred microseconds of Python each, serialised by the GIL): wait for all of them, the short window is for
        # callers outside any iteration
        deadline = first.t_submit + (max(self.max_wait_s, self.cohort_wait_s) if self._cohort else self.max_wait_s)
        while not self._stop:
            same = [r for r in self._pending if r.key == first.key]
            n_sess = sum(len(r.sids) for r in same)
            waiting = len(self._pending)
            everyone_here = len(self._cohort) > 0 and waiting >= len(self._cohort)
            if n_sess >= self.max_batch or everyone_here:
                break
            left = deadline - time.perf_counter()
            if left <= 0:
                break
            self._cv.wait(left)
        batch, n = [], 0
        for r in list(self._pending):
            if r.key != first.key:
                continue
            if batch and n + len(r.sids) > self.max_batch:
                break
            batch.append(r)
            n += len(r.sids)
            self._pending.remove(r)
        return batch

    def _run(self) -> None:
        while True:
            with self._cv:
                while not self._pending and not self._stop:
                    self._cv.wait()
                if self._stop and not self._pending:
                    return
                batch = self._take_batch()
            if batch:
                self._execute(batch)

    def _call(self, batch: List[_Request]):
        op = batch[0].op
        sids = [s for r in batch for s in r.sids]
        payload, static = batch[0].payload
        per_session, shared = _OPS[op]
        if op == "select":
            items = [item for r in batch for item in r.payload[0][0]]
            suppress, first_ids = payload[1]
            from .alignatt import engine_select          # one fused call, or the elementary ones on a duck-typed engine
            with self._lock:
                return sids, engine_select(self.engine, sids, list(suppress), list(first_ids), [m for m, _ in items],
                                           [b for _, b in items], **static)
        args = [sids]
        if per_session:
            args.append([item for r in batch for item in r.payload[0][0]])
        if shared:
            args.append(list(payload[0]))
        with self._lock:
            return sids, getattr(self.engine, op)(*args, **static)

    def _execute(self, batch: List[_Request]) -> None:
        op = batch[0].op
        try:
            sids, out = self._call(batch)
        except BaseException as e:                      # noqa: BLE001
            if len(batch) == 1:
                batch[0].future.set_exception(e)
                return
            # One stream's error (n_text_ctx overflow, closed session, decode before encode ...) must not abort the
            # other callers of the merged call: the engine validates a batch before it touches any session, so the
            # requests are replayed one by one and only the offending caller sees its exception.
            for r in batch:
                self._execute([r])
            return
        st = self.stats
        st["calls"] += 1
        st["requests"] += len(batch)
        st["sessions"] += len(sids)
        st["max_sessions_in_call"] = max(st["max_sessions_in_call"], len(sids))
        st["by_op"][op]["calls"] += 1
        st["by_op"][op]["sessions"] += len(sids)
        pos = 0
        for r in batch:
            n = len(r.sids)
            r.future.set_result(None if out is None else list(out[pos: pos + n]))
            pos += n

    # -- lifetime ---------------------------------------------------------------------------------------------
    def close(self, close_engine: bool = False) -> None:
        with self._cv:
            self._stop = True
            self._cv.notify_all()
        self._thread.join(timeout=5)
        for r in self._pending:
            r.future.set_exception(RuntimeError("BatchingEngine closed"))
        self._pending.clear()
        if close_engine:
            self.engine.close()


def _freeze(v):
    if isinstance(v, (list, tuple)):
        return tuple(_freeze(x) for x in v)
    return v
