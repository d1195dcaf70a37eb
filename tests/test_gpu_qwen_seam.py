"""The rolling generate in one engine call (wlk_qtext_generate_rolling, QwenTextEngine.generate_rolling_batch) on the H100 against the Python driver loop over the
same engine, its error contract and its host traffic per step; and the coalesced realtime seam over the CUDA engines
against the causal fixtures."""
import dataclasses

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
TEMPLATE = [10, 11, 7, 12, 13]
GEN = dict(eos_token_id=5, suppress_token_ids=[7, 10, 11, 12, 13])
CONTROLS_ON = dict(repetition_penalty=1.15, no_repeat_ngram_size=3, max_consecutive_text_tokens=5, wait_token_id=3)


def _text(precision, max_batch=8, max_ctx=256, max_sessions=32):
    from whisperlivekit_b200.qwen_dims import QWEN_TEXT_DIMS, synthetic_text_state_dict
    from whisperlivekit_b200.qwen_text_engine import QwenTextEngine
    dims = dataclasses.replace(QWEN_TEXT_DIMS["tnano"], max_ctx=max_ctx)
    return QwenTextEngine(dims, synthetic_text_state_dict(dims, 5), precision=precision, max_sessions=max_sessions,
                          max_batch=max_batch)


def _rows(eng, n, seed, device_rows):
    """Ragged frame rows per stream; the last stream has none (the full path)."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        steps = 0 if i == n - 1 else int(rng.integers(3, 30))
        x = rng.standard_normal((steps, eng.dims.d_model)).astype(np.float32)
        out.append(torch.from_numpy(x).cuda() if device_rows else x)
    return out


def _grow(rows, k, seed):
    rng = np.random.default_rng(seed)
    out = []
    for r in rows:
        extra = rng.standard_normal((k, r.shape[1])).astype(np.float32)
        out.append(torch.cat([r, torch.from_numpy(extra).cuda()]) if torch.is_tensor(r) else np.concatenate([r, extra]))
    return out


def _drafts(hyps, max_new, vocab):
    """none, fully accepted, rejected at 0, rejected mid-way, with a stop id, longer than max_new_tokens, ..."""
    h = [list(t) or [20] for t in hyps]
    return [None,
            h[1][:max(1, min(len(h[1]), max_new) - 1)],
            [(h[2][0] + 1) % vocab] + h[2][1:],
            h[3][:2] + [(h[3][2 % len(h[3])] + 7) % vocab, 30, 31],
            h[4][:1] + [GEN["eos_token_id"], 40, 41],
            (h[5] * (max_new + 6))[: max_new + 5],
            [50, 51, 52],
            [60, 61]]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("controls", ["off", "on"])
@pytest.mark.parametrize("device_rows", [True, False])
def test_engine_call_equals_driver_loop(precision, controls, device_rows):
    from whisperlivekit_b200.qwen_text_engine import TextDecodeDriver
    eng = _text(precision)
    n = 8
    kw = dict(GEN, **(CONTROLS_ON if controls == "on" else {}))
    for max_new in (1, 9):
        rows = _rows(eng, n, seed=3 + max_new, device_rows=device_rows)
        probe = [eng.open_session() for _ in range(n)]
        hyps, _, _ = eng.generate_rolling_batch(probe, rows, [None] * n, TEMPLATE, 7, None, max_new_tokens=max_new, **kw)
        for s in probe:
            eng.close_session(s)
        a = [eng.open_session() for _ in range(n)]           # the driver loop's sessions
        b = [eng.open_session() for _ in range(n)]           # the engine call's
        sa = sb = [None] * n
        drafts = _drafts(hyps, max_new, eng.vocab)
        for rnd in range(3):
            loop = TextDecodeDriver.generate_rolling(eng, a, rows, sa, TEMPLATE, 7, drafts, max_new_tokens=max_new, **kw)
            call = eng.generate_rolling_batch(b, rows, sb, TEMPLATE, 7, drafts, max_new_tokens=max_new, **kw)
            assert call[0] == loop[0], (rnd, max_new, call[0], loop[0])
            assert call[1] == loop[1], (rnd, max_new, call[1], loop[1])
            assert call[2] == loop[2]
            for i in range(n):
                want = 0 if loop[1][i]["decoder_path"] == "full" else 2 + len(rows[i])     # head + audio_steps
                assert eng.session_len(a[i]) == eng.session_len(b[i]) == want, (rnd, i)
            paths = [s["decoder_path"] for s in call[1]]
            assert paths[0] == "rolling" and "rolling+draft" in paths and (paths[-1] == "full") == (rnd == 0)
            rebuilt = [s["decoder_rebuilt"] for s in call[1][:-1]]
            assert rebuilt == [rnd == 0 or (rnd == 2 and i == 2) for i in range(n - 1)], (rnd, rebuilt)
            assert call[1][-1]["decoder_rebuilt"] == (rnd == 1) if rnd else call[1][-1] == {"decoder_path": "full"}
            sa, sb = loop[2], call[2]
            if rnd == 1:                                   # a state that no longer validates: rebuilt
                sa, sb = list(sa), list(sb)
                eng.reset_session(a[2])
                eng.reset_session(b[2])
            drafts = [None] + [t for t in call[0][1:]]
            rows = _grow(rows, 1 + rnd, seed=rnd)
        if max_new == 9:
            st = {k: sum(int(s.get(k, 0)) for s in call[1]) for k in ("draft_accepted", "decode_steps")}
            assert st["decode_steps"] > 0 and st["draft_accepted"] > 0, st
        for s in a + b:
            eng.close_session(s)
    eng.close()


def _raw_call(eng, sids, srcs, dl, prefix, tail, max_new, rows=None):
    import ctypes as C
    from whisperlivekit_b200._lib import _ptr
    ids = np.asarray(sids, np.int32)
    flat = np.concatenate(srcs).astype(np.int32) if srcs else np.zeros(1, np.int32)
    off = np.zeros(len(srcs) + 1, np.int32)
    off[1:] = np.cumsum([len(s) for s in srcs])
    emb = rows if rows is not None else np.zeros((1, eng.dims.d_model), np.float32)
    n_emb = 0 if rows is None else rows.shape[0]
    d, p = np.asarray(dl, np.int32), np.asarray(prefix, np.int32)
    m = max(len(sids), 1)
    toks, cnt, st = np.zeros((m, max(max_new, 1)), np.int32), np.zeros(m, np.int32), np.zeros((m, 4), np.int32)
    from whisperlivekit_b200 import _lib as L
    L.check(eng.lib.wlk_qtext_generate_rolling(eng.h, _ptr(ids), len(sids), _ptr(flat), _ptr(off), _ptr(emb), 0, n_emb,
                                               _ptr(d), _ptr(p), tail, max_new, _ptr(np.asarray([5], np.int32)), 1,
                                               _ptr(np.zeros(1, np.int32)), 0, C.c_float(1.0), 0, 0, -1, _ptr(toks),
                                               _ptr(cnt), _ptr(st)))
    return toks, cnt, st


def test_rolling_error_contract():
    from whisperlivekit_b200._lib import WlkError
    eng = _text("fp32", max_batch=4, max_ctx=64)
    sids = [eng.open_session() for _ in range(5)]
    closed = sids.pop()
    eng.close_session(closed)
    rows = np.random.default_rng(0).standard_normal((6, eng.dims.d_model)).astype(np.float32)
    # a valid rolling state: 2 head tokens + 6 audio rows held
    for s in sids:
        eng.forward([s], [(np.concatenate([[10, 11], -1 - np.arange(6)]).astype(np.int32), rows)], [0])
    held = [eng.session_len(s) for s in sids]
    blk = np.asarray([12, 13, 20, 21], np.int32)          # tail + a 2-token draft
    ok = dict(srcs=[blk, blk], dl=[2, 2], prefix=[10, 10], tail=2, max_new=4)
    toks, cnt, st = _raw_call(eng, sids[:2], **ok)        # the valid call works, and leaves [head + audio]
    assert [eng.session_len(s) for s in sids[:2]] == [8, 8] and all(1 <= c <= 4 for c in cnt)
    cases = {
        "batch 0": dict(ok, sids=[], srcs=[], dl=[], prefix=[]),
        "batch 5": dict(ok, sids=sids + [sids[0]], srcs=[blk] * 5, dl=[2] * 5, prefix=[10] * 5),
        "repeated": dict(ok, sids=[sids[0], sids[0]]),
        "closed": dict(ok, sids=[sids[0], closed]),
        "max_new 0": dict(ok, sids=sids[:2], max_new=0),
        "draft past rows": dict(ok, sids=sids[:2], dl=[2, 4]),
        "draft past max_new": dict(ok, sids=sids[:2], dl=[2, 2], max_new=1),
        "draft not a token": dict(ok, sids=sids[:2], srcs=[blk, np.asarray([12, 13, 20, -1], np.int32)]),
        "prefix mismatch": dict(ok, sids=sids[:2], prefix=[10, 11]),
        "token id": dict(ok, sids=sids[:2], srcs=[blk, np.asarray([12, eng.dims.vocab, 20, 21], np.int32)]),
        "max_ctx": dict(ok, sids=sids[:2], max_new=64 - 12 + 1),
    }
    for what, c in cases.items():
        for s, h in zip(sids, held):                      # every session back at 8 positions
            if eng.session_len(s) != h:
                eng.reset_session(s)
                eng.forward([s], [(np.concatenate([[10, 11], -1 - np.arange(6)]).astype(np.int32), rows)], [0])
        before = [eng.session_len(s) for s in sids]
        with pytest.raises(WlkError):
            _raw_call(eng, c["sids"], c["srcs"], c["dl"], c["prefix"], c["tail"], c["max_new"])
        assert [eng.session_len(s) for s in sids] == before, what
    # the largest budget that fits
    _raw_call(eng, sids[:2], **dict(ok, max_new=64 - 12))
    eng.close()


def test_d2h_bytes_per_continuation_step_are_4_per_live_stream():
    from test_gpu_qwen_window_realtime import _d2h_bytes
    eng = _text("fp32")
    n = 8
    rows = [r for r in _rows(eng, n + 1, seed=9, device_rows=False)[:n]]
    kw = dict(suppress_token_ids=GEN["suppress_token_ids"])         # no stop id: every stream takes its whole budget
    got = {}
    for max_new in (8, 24):
        sids = [eng.open_session() for _ in range(n)]
        out = []
        got[max_new] = _d2h_bytes(lambda: out.append(eng.generate_rolling_batch(sids, rows, [None] * n, TEMPLATE, 7, None,
                                                                          max_new_tokens=max_new, **kw)))
        assert all(len(t) == max_new for t in out[0][0])
        for s in sids:
            eng.close_session(s)
    print("D2H bytes of a rolling call by max_new_tokens", got)
    assert got[24] - got[8] == 4 * n * 16
    assert got[8] <= 8 * n + 4 * n * 7 + 1024
    eng.close()


def _seam(name, threads, **install_kw):
    """`threads` streams of the causal fixture through the coalesced seam over the CUDA engines in fp32, each chunk one
    cohort iteration.  Returns (realtime model, the fixture's events, events per stream, sessions per merged call by op)."""
    import json
    import os
    import threading
    pytest.importorskip("transformers")
    from oracle import stage_reference
    stage_reference.import_staged_reference()
    from oracle.make_golden_qwen import mel_stream
    from oracle.make_golden_qwen_realtime import CHUNK, MEL_SEED, N_FRAMES, build_model, build_streamer, event_record
    from whisperlivekit_b200.qwen_plugin import B200QwenRealtimeModel
    z = np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                             f"qwen_realtime_{name}.npz"))
    want = json.loads(bytes(z["events"]).decode())
    model = build_model(name)
    rt = B200QwenRealtimeModel.install(model, precision="fp32", max_ctx=256, batching=True, **install_kw)
    sizes = {}
    ops = rt.batcher.engine
    for op in ("append_audio_to_cache", "flush_audio_to_cache", "generate_full_hypothesis_rolling",
               "generate_full_hypothesis_from_cached_audio"):
        def logged(keys, *a, _f=getattr(ops, op), _op=op, **k):
            out = _f(keys, *a, **k)
            sizes.setdefault(_op, []).append(len(keys))          # calls that succeeded, merged or replayed
            return out
        setattr(ops, op, logged)
    mels = mel_stream(N_FRAMES, 128, seed=MEL_SEED)
    streamers = [build_streamer(model) for _ in range(threads)]
    got, err = [None] * threads, [None] * threads

    def one(fn):
        rt.batcher.begin_iter()
        try:
            return fn()
        finally:
            rt.batcher.end_iter()

    def run(i):
        try:
            s, ev = streamers[i], []
            with torch.no_grad():
                for a in range(0, mels.shape[0], CHUNK):
                    ev.append(event_record(one(lambda: s.append_mel_chunk(torch.from_numpy(mels[a: a + CHUNK])[None])), s))
                e = one(s.flush_pending_audio)
                if e is not None:
                    ev.append(event_record(e, s))
            got[i] = ev
        except BaseException as e:              # noqa: BLE001
            err[i] = e

    ts = [threading.Thread(target=run, args=(i,)) for i in range(threads)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=900)
    assert err == [None] * threads, err
    for i, g in enumerate(got):
        assert len(g) == len(want)
        for k, (a, b) in enumerate(zip(g, want)):
            assert a == b, (i, k, {x: (a.get(x), b.get(x)) for x in set(a) | set(b) if a.get(x) != b.get(x)})
    del streamers
    return rt, sizes


def _close(rt):
    import gc
    rt.close()
    rt.decoder.close()
    gc.collect()


@pytest.mark.parametrize("name", ["qnano", "qnano-tail"])
def test_fp32_coalesced_seam_reproduces_causal_fixture(name):
    rt, sizes = _seam(name, 8, max_sessions=40)
    st = rt.batcher.stats
    print(f"SEAM {name}: {st['requests']} caller calls in {st['calls']} engine calls, mean cohort "
          f"{st['sessions'] / st['calls']:.2f}")
    assert st["calls"] < st["requests"]
    assert rt.batcher.max_batch == 8 == rt.encoder.engine.max_batch == rt.decoder.engine.max_batch
    _close(rt)


def test_cohort_above_the_default_batch_merges_into_one_call_per_op():
    """install(max_batch=16) builds both engines for 16 sessions per call, so merged calls of more than the engines'
    default 8 sessions run as one engine call each (the events still equal the fixture's)."""
    rt, sizes = _seam("qnano", 12, max_sessions=64, max_batch=16)
    assert rt.batcher.max_batch == 16 == rt.encoder.engine.max_batch == rt.decoder.engine.max_batch
    print("SEAM 12 streams, sessions per merged call:", {op: (max(v), round(float(np.mean(v)), 2)) for op, v in sizes.items()})
    for op in ("append_audio_to_cache", "generate_full_hypothesis_rolling"):
        assert max(sizes[op]) > 8, (op, sizes[op])
    _close(rt)
