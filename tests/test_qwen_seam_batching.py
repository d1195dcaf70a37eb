"""The coalescing seam of the Qwen3 realtime model (B200QwenRealtimeModel.install(batching=True)) with the CPU oracles
behind the engine API: eight threads drive the reference's segmented streamer over one installed model, each iteration
bracketed as a cohort, and every stream's events equal the fixture and an untouched twin's, while the dispatcher merges
the appends, flushes and generates of concurrent streams into shared engine calls.  A stream whose session breaks gets
the error; the others finish unharmed.  After close no engine session is left open."""
import gc
import json
import os
import threading

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.reference
pytest.importorskip("transformers")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
THREADS = 8


def _events(path):
    z = np.load(os.path.join(ROOT, "tests", "golden", path))
    return json.loads(bytes(z["events"]).decode())


def _oracles(kind="causal"):
    from oracle import stage_reference
    stage_reference.import_staged_reference()
    if kind == "causal":
        from test_oracle_qwen_realtime import oracle_factories
    else:
        from test_oracle_qwen_window_realtime import oracle_factories
    return oracle_factories()


def _causal_chunks():
    from oracle.make_golden_qwen import mel_stream
    from oracle.make_golden_qwen_realtime import CHUNK, MEL_SEED, N_FRAMES
    m = mel_stream(N_FRAMES, 128, seed=MEL_SEED)
    return [(m[a: a + CHUNK], False) for a in range(0, m.shape[0], CHUNK)], True


def _window_chunks():
    from oracle.make_golden_qwen_window_realtime import SCHEDULE, TOWER, mels
    from whisperlivekit_b200.qwen_dims import QWEN_WINDOW_DIMS
    m, out, a = mels(), [], 0
    sizes = SCHEDULE + [QWEN_WINDOW_DIMS[TOWER].right_context_frames]
    for k, n in enumerate(sizes):
        out.append((m[a: a + n], k == len(sizes) - 1))
        a += n
    return out, False


def _drive(streamer, chunks, flush, record, batcher=None, on_chunk=None):
    """The streamer over chunks, one cohort iteration per chunk (and one for the flush); returns the event records."""
    def one(fn):
        if batcher is not None:
            batcher.begin_iter()
        try:
            return fn()
        finally:
            if batcher is not None:
                batcher.end_iter()

    events = []
    with torch.no_grad():
        for k, (m, is_flush) in enumerate(chunks):
            ev = one(lambda: streamer.append_mel_chunk(torch.from_numpy(m)[None], is_flush=is_flush))
            events.append(record(ev, streamer))
            if on_chunk is not None:
                on_chunk(k, streamer)
        if flush:
            ev = one(streamer.flush_pending_audio)
            if ev is not None:
                events.append(record(ev, streamer))
    return events


def _threads(n, target):
    """target(i) in n threads; returns (results, exceptions) per thread."""
    res, err = [None] * n, [None] * n

    def run(i):
        try:
            res[i] = target(i)
        except BaseException as e:              # noqa: BLE001
            err[i] = e

    ts = [threading.Thread(target=run, args=(i,)) for i in range(n)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    assert not any(t.is_alive() for t in ts)
    return res, err


def _setup(kind, param):
    from whisperlivekit_b200.qwen_plugin import B200QwenRealtimeModel
    tower, text, made = _oracles(kind)
    if kind == "causal":
        from oracle.make_golden_qwen_realtime import build_model, build_streamer, event_record
        mine, twin = build_model(param), build_model(param)
        rt = B200QwenRealtimeModel.install(mine, tower_factory=tower, text_factory=text, batching=True, max_batch=THREADS)
        chunks, flush = _causal_chunks()
        want = _events(f"qwen_realtime_{param}.npz")
        streamer = build_streamer
    else:
        from oracle.make_golden_qwen_window_realtime import FIXTURES, build_model, build_streamer, event_record
        mine, twin = build_model(), build_model()
        rt = B200QwenRealtimeModel.install(mine, tower_factory=tower, text_factory=text, attention_blocks=True,
                                           batching=True, max_batch=THREADS)
        chunks, flush = _window_chunks()
        want = _events(f"qwen_window_realtime_{param}.npz")

        def streamer(model, keep=FIXTURES[param]):
            return build_streamer(model, keep)
    return rt, mine, twin, streamer, chunks, flush, want, event_record, made


def _sessions_left(made):
    tower = made["tower"][0]
    open_tower = tower._s if hasattr(tower, "_s") else tower.open
    return len(open_tower), len(made["text"][0].sessions)


@pytest.mark.parametrize("kind,param", [("causal", "qnano"), ("causal", "qnano-tail"), ("window", "w0"), ("window", "wtail")])
def test_eight_threads_reproduce_fixture_and_twin_in_merged_calls(kind, param):
    rt, mine, twin, make_streamer, chunks, flush, want, record, made = _setup(kind, param)
    twin_events = _drive(make_streamer(twin), chunks, flush, record)
    assert twin_events == want
    streamers = [make_streamer(mine) for _ in range(THREADS)]
    got, err = _threads(THREADS, lambda i: _drive(streamers[i], chunks, flush, record, rt.batcher))
    assert err == [None] * THREADS, err
    for i, g in enumerate(got):
        assert len(g) == len(want)
        for k, (a, b) in enumerate(zip(g, want)):
            assert a == b, (i, k, {x: (a.get(x), b.get(x)) for x in set(a) | set(b) if a.get(x) != b.get(x)})
    st = rt.batcher.stats
    print(f"{kind}/{param}: {st['requests']} caller calls in {st['calls']} engine calls, mean cohort "
          f"{st['sessions'] / st['calls']:.2f}, by op {st['by_op']}")
    assert st["calls"] < st["requests"] and st["sessions"] / st["calls"] > 1
    gen_op = "generate_full_hypothesis_rolling" if kind == "causal" else "generate_full_hypothesis_from_cached_audio"
    for op in ("append_audio_to_cache", gen_op):
        assert 0 < st["by_op"][op]["calls"] < st["by_op"][op]["sessions"], (op, st["by_op"][op])
    rt.close()
    rt.decoder.close()
    del streamers, got
    gc.collect()
    assert _sessions_left(made) == (0, 0)


def test_broken_session_fails_only_its_caller():
    rt, mine, twin, make_streamer, chunks, flush, want, record, made = _setup("causal", "qnano")
    streamers = [make_streamer(mine) for _ in range(4)]

    def breaker(k, s):
        if k == 2:
            s.state.audio.close()                   # the stream's tower session is closed underneath it

    got, err = _threads(4, lambda i: _drive(streamers[i], chunks, flush, record, rt.batcher,
                                            on_chunk=breaker if i == 1 else None))
    assert isinstance(err[1], ValueError) and "closed" in str(err[1])
    for i in (0, 2, 3):
        assert err[i] is None and got[i] == want, i
    rt.close()
    rt.decoder.close()
    del streamers, got, err                         # the error's traceback holds the broken stream's states
    gc.collect()
    assert _sessions_left(made) == (0, 0)


def test_batching_off_keeps_the_decoder_methods():
    from whisperlivekit_b200.qwen_plugin import B200QwenRealtimeModel
    from oracle.make_golden_qwen_realtime import build_model
    tower, text, _ = _oracles()
    model = build_model("qnano")
    rt = B200QwenRealtimeModel.install(model, tower_factory=tower, text_factory=text)
    assert rt.batcher is None
    assert model.generate_full_hypothesis_rolling == rt.decoder.generate_full_hypothesis_rolling
    assert model.generate_full_hypothesis_from_cached_audio == rt.decoder.generate_full_hypothesis_from_cached_audio


def test_cohort_installer_brackets_process_iter():
    from whisperlivekit_b200.plugin import install_qwen_cohorts, uninstall_qwen_cohorts
    calls = []

    class Batcher:
        def begin_iter(self):
            calls.append("begin")

        def end_iter(self):
            calls.append("end")

    class RT:
        batcher = Batcher()

    class Processor:
        def process_iter(self, is_last=False):
            calls.append(("iter", is_last))
            return [], 1.0

    install_qwen_cohorts(RT(), Processor)
    install_qwen_cohorts(RT(), Processor)           # idempotent: one bracket
    assert Processor().process_iter(is_last=True) == ([], 1.0)
    assert calls == ["begin", ("iter", True), "end"]
    uninstall_qwen_cohorts(Processor)
    calls.clear()
    Processor().process_iter()
    assert calls == [("iter", False)]
