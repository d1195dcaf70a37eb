"""The windowed realtime model on the H100: the reference streamer over the model installed on the CUDA engines against
the reference's fixtures (fp32 exact, bf16 reported), the engine's one-call non-rolling generate (wlk_qtext_generate_full)
against the driver loop over the same engine, an N-stream windowed tick against N single-stream ones, the host traffic
of a tick, and the generate's error contract."""
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["w0", "wtail"]
GEN = dict(audio_placeholder_token_id=7, eos_token_id=5, suppress_token_ids=[7, 10, 11, 12, 13])
CONTROLS_ON = dict(repetition_penalty=1.15, no_repeat_ngram_size=3, max_consecutive_text_tokens=5, wait_token_id=3)


def _fixture(name):
    z = np.load(os.path.join(ROOT, "tests", "golden", f"qwen_window_realtime_{name}.npz"))
    return json.loads(bytes(z["events"]).decode())


def _stream(name, precision):
    pytest.importorskip("transformers")
    from oracle import stage_reference
    stage_reference.import_staged_reference()
    from oracle.make_golden_qwen_window_realtime import FIXTURES, build_model, build_streamer, drive, mels
    from whisperlivekit_b200.qwen_plugin import B200QwenAudioSurgeryEncoder, B200QwenRealtimeModel
    model = build_model()
    rt = B200QwenRealtimeModel.install(model, precision=precision, max_ctx=256, max_sessions=4, attention_blocks=True)
    assert isinstance(model.audio_encoder, B200QwenAudioSurgeryEncoder) and not hasattr(model, "flush_audio_to_cache")
    streamer = build_streamer(model, FIXTURES[name])
    on_device = []
    got = drive(streamer, mels(), on_chunk=lambda s: on_device.append(s.state.frame_hidden.is_cuda))
    rt.decoder.close()
    return got, on_device


@pytest.mark.parametrize("name", NAMES)
def test_fp32_streamer_over_installed_windowed_model_equals_fixture(name):
    want = _fixture(name)
    got, on_device = _stream(name, "fp32")
    assert all(on_device)
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, (i, {k: (g.get(k), w.get(k)) for k in set(g) | set(w) if g.get(k) != w.get(k)})


@pytest.mark.parametrize("name", NAMES)
def test_bf16_streamer_over_installed_windowed_model_completes(name):
    want = _fixture(name)
    got, _ = _stream(name, "bf16")
    assert len(got) == len(want)
    same = sum(g == w for g, w in zip(got, want))
    tokens = sum(g["hypothesis_tokens"] == w["hypothesis_tokens"] for g, w in zip(got, want))
    print(f"BF16_WINDOW_REALTIME {name}: {same}/{len(want)} events equal, {tokens}/{len(want)} hypotheses equal")


def _text(precision, max_batch=8, max_ctx=256, adapter_sd=None):
    import dataclasses
    from whisperlivekit_b200.qwen_dims import QWEN_TEXT_DIMS, synthetic_text_state_dict
    from whisperlivekit_b200.qwen_text_engine import QwenTextEngine
    dims = dataclasses.replace(QWEN_TEXT_DIMS["tnano"], max_ctx=max_ctx)
    sd = dict(synthetic_text_state_dict(dims, 5), **(adapter_sd or {}))
    return QwenTextEngine(dims, sd, precision=precision, max_sessions=max_batch + 2, max_batch=max_batch)


def _ragged(dims, n=8, seed=4, device_rows=True):
    rng = np.random.default_rng(seed)
    rows, prefixes = [], []
    for i in range(n):
        steps = int(rng.integers(1, 40))
        fh = torch.from_numpy(rng.standard_normal((steps, dims.d_model)).astype(np.float32))
        rows.append(fh.cuda() if device_rows else fh.numpy())
        prefixes.append(np.concatenate([np.asarray([10, 11][: 1 + i % 2], np.int32),
                                        -1 - np.arange(steps, dtype=np.int32), np.asarray([12, 13], np.int32)]))
    return rows, prefixes


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("controls", ["off", "on"])
@pytest.mark.parametrize("device_rows", [True, False])
def test_engine_call_equals_driver_loop(precision, controls, device_rows):
    from whisperlivekit_b200.qwen_text_engine import TextDecodeDriver
    eng = _text(precision)
    rows, prefixes = _ragged(eng.dims, device_rows=device_rows)
    ctl_kw = dict(GEN, **(CONTROLS_ON if controls == "on" else {}))
    ctl_kw.pop("audio_placeholder_token_id")
    sids = [eng.open_session() for _ in rows]
    for max_new in (0, 1, 24):
        loop = TextDecodeDriver.generate_full_batch(eng, sids, rows, prefixes, max_new_tokens=max_new, **ctl_kw)
        # stop ids that the loop hits at different steps in a second pass
        stops = sorted({t[k] for t, k in zip(loop, (2, 5, 9)) if len(t) > k})
        loop2 = TextDecodeDriver.generate_full_batch(eng, sids, rows, prefixes, max_new_tokens=max_new,
                                                     stop_token_ids=stops, **ctl_kw)
        call = eng.generate_full_batch(sids, rows, prefixes, max_new_tokens=max_new, **ctl_kw)
        call2 = eng.generate_full_batch(sids, rows, prefixes, max_new_tokens=max_new, stop_token_ids=stops, **ctl_kw)
        assert call == loop, (max_new, call, loop)
        assert call2 == loop2, (max_new, call2, loop2)
        assert all(1 <= len(t) <= max_new for t in call) if max_new else call == [[]] * len(rows)
        assert all(eng.session_len(s) == 0 for s in sids)


def _window(precision, n):
    import dataclasses
    from whisperlivekit_b200.qwen_dims import QWEN_TEXT_DIMS, QWEN_WINDOW_DIMS, synthetic_adapter_state_dict, synthetic_tower_state_dict
    from whisperlivekit_b200.qwen_engine import QwenWindowEngine
    from whisperlivekit_b200.qwen_plugin import B200QwenAudioSurgeryEncoder, B200QwenTextDecoder
    from whisperlivekit_b200.qwen_realtime import RealtimeFrames
    wd = QWEN_WINDOW_DIMS["wnano"]
    tower = QwenWindowEngine(wd, synthetic_tower_state_dict(wd, 11), precision=precision, max_sessions=2 * n, max_batch=n)
    text = _text(precision, max_batch=n, max_ctx=512, adapter_sd=synthetic_adapter_state_dict(96, 256, 128, 2, 0.1, seed=4))
    enc = B200QwenAudioSurgeryEncoder(tower, wd)
    dec = B200QwenTextDecoder(SimpleNamespace(wait_token_id=3, bos_token_id=1), text, QWEN_TEXT_DIMS["tnano"])
    return enc, dec, RealtimeFrames(enc, text, 256)


def _state(enc):
    return SimpleNamespace(audio=enc.init_state(), adapter=SimpleNamespace(audio_frames_seen=0, decoder_steps_seen=0),
                           frame_hidden=None, decoder=None)


def _prefix(st):
    return [10, 11] + [7] * int(st.frame_hidden.shape[1]) + [12, 13]


def _generate(dec, states, max_new):
    live = [s for s in states if s.frame_hidden is not None and s.frame_hidden.shape[1]]
    toks = dec.generate_full_batch([s.frame_hidden[0] for s in live], [_prefix(s) for s in live],
                                   max_new_tokens=max_new, **{k: v for k, v in GEN.items()})
    got = dict(zip(map(id, live), toks))
    return [got.get(id(s), []) for s in states]


def test_batched_windowed_tick_equals_streams_one_at_a_time():
    from oracle.make_golden_qwen import mel_stream
    n = 8
    enc, dec, frames = _window("fp32", n)
    batch, single = [_state(enc) for _ in range(n)], [_state(enc) for _ in range(n)]
    mels = [mel_stream(12 * 140, 128, seed=30 + i) for i in range(n)]
    for k in range(10):
        sizes = [(k * 37 + i * 23) % 140 for i in range(n)]              # ragged, some chunks empty
        chunk = [torch.from_numpy(mels[i][k * 140: k * 140 + sizes[i]])[None] for i in range(n)]
        frames.append(batch, chunk)
        tb = _generate(dec, batch, 10)
        for i in range(n):
            frames.append([single[i]], [chunk[i]])
            ts = _generate(dec, [single[i]], 10)
            assert ts[0] == tb[i], (k, i, ts[0], tb[i])
            if single[i].frame_hidden is not None:
                err = float((single[i].frame_hidden - batch[i].frame_hidden).abs().max()) if single[i].frame_hidden.numel() else 0.0
                assert single[i].frame_hidden.shape == batch[i].frame_hidden.shape and err <= 1e-5, (k, i, err)
        if k == 6:                                                     # a rollover with a kept tail, then one without
            for s in batch + single:
                s.frame_hidden = s.frame_hidden[:, -5:]
        if k == 8:
            for s in batch + single:
                s.frame_hidden = s.frame_hidden[:, 0:0]
    dec.close()


def _d2h_bytes(fn):
    import tempfile
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        ev = json.load(open(path)).get("traceEvents", [])
    return sum(int(e.get("args", {}).get("bytes", 0)) for e in ev
               if e.get("cat") == "gpu_memcpy" and "DtoH" in e.get("name", "") + str(e.get("args", {})))


def test_d2h_bytes_per_tick_are_the_picks_only():
    from oracle.make_golden_qwen import mel_stream
    n, max_new = 8, 16
    enc, dec, frames = _window("fp32", n)
    states = [_state(enc) for _ in range(n)]
    mels = [mel_stream(30 * 100, 128, seed=50 + i) for i in range(n)]
    per_tick = []
    for k in range(30):
        def tick():
            frames.append(states, [torch.from_numpy(mels[i][k * 100: (k + 1) * 100])[None] for i in range(n)])
            _generate(dec, states, max_new)
        if k in (3, 4, 26, 27):
            per_tick.append((int(states[0].frame_hidden.shape[1]), _d2h_bytes(tick)))
        else:
            tick()
    print("D2H per tick (cached steps, bytes)", per_tick)
    assert per_tick[2][0] > 5 * per_tick[0][0]
    bound = 4 * n * (max_new + 1) + 4096
    assert all(b <= bound for _, b in per_tick), (per_tick, bound)
    assert max(b for _, b in per_tick[2:]) <= max(b for _, b in per_tick[:2])
    dec.close()


def test_generate_full_error_contract():
    from whisperlivekit_b200._lib import WlkError
    eng = _text("fp32", max_batch=4, max_ctx=64)
    rows = [torch.randn(6, eng.dims.d_model, device="cuda") for _ in range(5)]
    prefixes = [np.concatenate([[10], -1 - np.arange(6, dtype=np.int32), [12]]).astype(np.int32) for _ in rows]
    sids = [eng.open_session() for _ in range(4)]

    def dirty():
        for x in sids:
            eng.reset_session(x)
        eng.forward(sids, [(np.asarray([1, 2, 3], np.int32), None)] * 4, [1] * 4)
        eng.pick(np.zeros(1, np.int32), np.zeros(4, np.int32), np.zeros(4, np.int32), eng.make_controls())
        assert all(eng.session_len(s) == 3 for s in sids)

    bad_src = [p.copy() for p in prefixes[:2]]
    bad_src[1][0] = eng.dims.vocab
    cases = {
        "batch 0": ([], [], [], 4),
        "batch 5": (sids + [sids[0]], rows, prefixes, 4),
        "repeated": ([sids[0], sids[0]], rows[:2], prefixes[:2], 4),
        "token id": (sids[:2], rows[:2], bad_src, 4),
        "max_new < 0": (sids[:2], rows[:2], prefixes[:2], -1),
        "max_ctx": (sids[:2], rows[:2], prefixes[:2], 64 - 8 + 1),
    }
    for what, (s, r, p, mx) in cases.items():
        dirty()
        with pytest.raises(WlkError):
            eng.generate_full_batch(s, r, p, max_new_tokens=mx, **{k: v for k, v in GEN.items() if k != "audio_placeholder_token_id"})
        assert all(eng.session_len(x) == 0 for x in s if x in sids), what
    # frame row 6 of a 6-row stream is caught on the host: the engine sees the streams' rows packed
    far2 = [prefixes[0].copy(), prefixes[1]]
    far2[0][1] = -1 - 6
    with pytest.raises(ValueError, match="past its 6 rows"):
        eng.generate_full_batch(sids[:2], rows[:2], far2, max_new_tokens=4)
    # the largest budget that fits
    out = eng.generate_full_batch(sids[:2], rows[:2], prefixes[:2], max_new_tokens=64 - 8,
                                  **{k: v for k, v in GEN.items() if k not in ("audio_placeholder_token_id", "eos_token_id")})
    assert [len(t) for t in out] == [56, 56]
