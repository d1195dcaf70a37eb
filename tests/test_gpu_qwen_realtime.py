"""The realtime model's device seam on the H100: the frame adapter kernel against a float64 reference, device rows into the
text forward and out of the tower bit for bit equal to the host entries, the reference streamer over the installed model
(fp32) against the reference's fixtures, frame-row copies to the host that do not grow with the segment, an N-stream tick
equal to N single-stream ticks, and the error contract."""
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BOUND = {"fp32": 2e-6, "bf16": 1e-2}          # fraction of max|ref| over the output


def text_engine(precision, adapter_sd=None, max_sessions=4, max_ctx=1024):
    import dataclasses
    from whisperlivekit_b200.qwen_dims import QWEN_TEXT_DIMS, synthetic_text_state_dict
    from whisperlivekit_b200.qwen_text_engine import QwenTextEngine
    dims = dataclasses.replace(QWEN_TEXT_DIMS["tnano"], max_ctx=max_ctx)
    sd = dict(synthetic_text_state_dict(dims, 5), **(adapter_sd or {}))
    return QwenTextEngine(dims, sd, precision=precision, max_sessions=max_sessions, max_batch=max_sessions)


_ENGINES = {}


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("in_dim,blocks", [(96, 0), (96, 2), (256, 0), (256, 2)])
@pytest.mark.parametrize("rows", [1, 24, 1100])
@pytest.mark.parametrize("scale", [1e3, 1e-5])
def test_adapt_matches_float64(precision, in_dim, blocks, rows, scale):
    from oracle.qwen_realtime_oracle import adapter_f64
    from whisperlivekit_b200.qwen_dims import synthetic_adapter_state_dict
    key = (precision, in_dim, blocks)
    sd = synthetic_adapter_state_dict(in_dim, 256, 128 if blocks else 0, blocks, 0.1, seed=in_dim + blocks)
    if key not in _ENGINES:
        _ENGINES[key] = text_engine(precision, sd)
    eng = _ENGINES[key]
    assert eng.adapter_dims() == (in_dim, blocks, 128 if blocks else 0)
    x = np.random.default_rng(rows).standard_normal((rows, in_dim)).astype(np.float32) * np.float32(scale)
    wide = torch.zeros(rows, in_dim + 8, device="cuda")                  # row pitch > in_dim
    wide[:, :in_dim] = torch.from_numpy(x)
    y = eng.adapt(wide[:, :in_dim]).cpu().numpy()
    ref = adapter_f64(x, sd)
    err = float(np.abs(y - ref).max() / np.abs(ref).max())
    print(f"ADAPT_ERR precision={precision} in={in_dim} blocks={blocks} rows={rows} scale={scale:g} err={err:.3e}")
    assert err <= BOUND[precision], err


def test_adapt_errors():
    from whisperlivekit_b200._lib import WlkError
    from whisperlivekit_b200.qwen_dims import synthetic_adapter_state_dict
    eng = text_engine("fp32")
    x = torch.zeros(3, 256, device="cuda")
    with pytest.raises(WlkError, match="no adapter loaded"):
        eng.adapt(x)
    eng = text_engine("fp32", synthetic_adapter_state_dict(96, 256, seed=1))
    y = torch.zeros(3, 256, device="cuda")
    for in_ld, out_ld, what in ((96, 255, "out_ld"), (95, 256, "in_ld")):       # row pitches below the row widths
        assert eng.lib.wlk_qtext_adapt(eng.h, x.data_ptr(), 3, in_ld, y.data_ptr(), out_ld) != 0
        assert what in eng.lib.wlk_last_error().decode()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_forward_device_bit_identical_to_host(precision):
    from whisperlivekit_b200._lib import WlkError
    eng = text_engine(precision, max_ctx=64)
    rows = np.random.default_rng(3).standard_normal((20, 256)).astype(np.float32)
    src = np.concatenate([[10, 11], -1 - np.arange(20), [12, 13]]).astype(np.int32)
    a, b = eng.open_session(), eng.open_session()
    eng.forward([a], [(src, rows)], [len(src)])
    la = eng.logits()
    wide = torch.zeros(20, 256 + 40, device="cuda")
    wide[:, 8:264] = torch.from_numpy(rows)
    eng.forward([b], [(src, wide[:, 8:264])], [len(src)])                 # ld = 296 > d_model
    lb = eng.logits()
    assert np.array_equal(la, lb)
    # two sessions in one device forward (their rows concatenated on the device) equal the host forward
    c, d = eng.open_session(), eng.open_session()
    dev = torch.from_numpy(rows).cuda()
    eng.crop(a, 0)
    eng.forward([a, c], [(src, rows), (src[:5], rows[:3])], [2, 1])
    lh = eng.logits()
    eng.crop(a, 0)
    eng.forward([a, d], [(src, dev), (src[:5], dev[:3])], [2, 1])
    assert np.array_equal(lh, eng.logits())
    # a forward past max_ctx fails and leaves the session unchanged
    n0 = eng.session_len(b)
    long_src = -1 - np.arange(50, dtype=np.int32)
    with pytest.raises(WlkError, match="context full"):
        eng.forward([b], [(long_src, torch.zeros(50, 256, device="cuda"))], [1])
    assert eng.session_len(b) == n0


def test_forward_device_rejects_narrow_pitch():
    import ctypes as C
    eng = text_engine("fp32")
    s = eng.open_session()
    x = torch.zeros(4, 256, device="cuda")
    ids, src = np.asarray([s], np.int32), -1 - np.arange(4, dtype=np.int32)
    off, lr = np.asarray([0, 4], np.int32), np.asarray([1], np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)                            # noqa: E731
    rc = eng.lib.wlk_qtext_forward_device(eng.h, p(ids), 1, p(src), p(off), C.c_void_p(x.data_ptr()), 255, 4, p(lr))
    assert rc != 0 and "embeds_ld" in eng.lib.wlk_last_error().decode()
    assert eng.session_len(s) == 0


@pytest.mark.parametrize("name", ["qnano", "qnano-tail"])
def test_tower_device_entries_bit_identical(name):
    from oracle.make_golden_qwen import SCHEDULE, TAIL_SCHEDULE, mel_stream
    from whisperlivekit_b200.qwen_dims import QWEN_DIMS, synthetic_tower_state_dict
    from whisperlivekit_b200.qwen_engine import QwenTowerEngine
    dims = QWEN_DIMS[name]
    sched = TAIL_SCHEDULE if dims.mutable_tail_steps else SCHEDULE
    eng = QwenTowerEngine(dims, synthetic_tower_state_dict(dims, 11), precision="fp32", max_sessions=2, max_batch=2)
    a, b = eng.open_session(), eng.open_session()
    mels = mel_stream(sum(sched), dims.n_mels, seed=2)
    o = 0
    for n in sched:
        h = eng.forward_chunk([a], [mels[o: o + n]])[0]
        d, offs = eng.forward_chunk_device([b], [mels[o: o + n]])
        o += n
        assert np.array_equal(h, d.cpu().numpy()) and offs[-1] == h.shape[0]
    assert np.array_equal(eng.get_pending(a), eng.get_pending(b))
    h = eng.flush_pending([a])[0]
    d, _ = eng.flush_pending_device([b])
    assert np.array_equal(h, d.cpu().numpy())


def _fixture(name):
    z = np.load(os.path.join(ROOT, "tests", "golden", f"qwen_realtime_{name}.npz"))
    return json.loads(bytes(z["events"]).decode())


@pytest.mark.reference
@pytest.mark.parametrize("name", ["qnano", "qnano-tail"])
def test_fp32_streamer_over_installed_model_equals_fixture(name):
    pytest.importorskip("transformers")
    from oracle import stage_reference
    stage_reference.import_staged_reference()
    from oracle.make_golden_qwen import mel_stream
    from oracle.make_golden_qwen_realtime import CHUNK, MEL_SEED, N_FRAMES, build_model, build_streamer, event_record
    from whisperlivekit_b200.qwen_plugin import B200QwenRealtimeModel
    want = _fixture(name)
    model = build_model(name)
    B200QwenRealtimeModel.install(model, precision="fp32", max_ctx=256, max_sessions=4)
    streamer = build_streamer(model)
    mels = mel_stream(N_FRAMES, 128, seed=MEL_SEED)
    got, d2h = [], []
    with torch.no_grad():
        for a in range(0, N_FRAMES, CHUNK):
            got.append(event_record(streamer.append_mel_chunk(torch.from_numpy(mels[a: a + CHUNK])[None]), streamer))
            assert streamer.state.frame_hidden is None or streamer.state.frame_hidden.is_cuda
        ev = streamer.flush_pending_audio()
        if ev is not None:
            got.append(event_record(ev, streamer))
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, (i, {k: (g.get(k), w.get(k)) for k in set(g) | set(w) if g.get(k) != w.get(k)})


def _d2h_bytes(fn):
    """Device-to-host bytes of the frame seam while fn runs, from a torch.profiler trace (CUDA activities)."""
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


def _realtime(max_sessions=16, precision="fp32"):
    import dataclasses
    from whisperlivekit_b200.qwen_dims import QWEN_DIMS, QWEN_TEXT_DIMS, synthetic_adapter_state_dict, synthetic_tower_state_dict
    from whisperlivekit_b200.qwen_engine import QwenTowerEngine
    from whisperlivekit_b200.qwen_plugin import B200QwenAudioCausalKVEncoder, B200QwenTextDecoder
    from whisperlivekit_b200.qwen_realtime import RealtimeFrames
    td = dataclasses.replace(QWEN_DIMS["qnano-chunk"], out_dim=256)
    tower = QwenTowerEngine(td, synthetic_tower_state_dict(td, 11), precision=precision, max_sessions=max_sessions,
                            max_batch=max_sessions)
    text = text_engine(precision, synthetic_adapter_state_dict(256, 256, 128, 2, 0.1, seed=4), max_sessions=max_sessions)
    enc = B200QwenAudioCausalKVEncoder(tower, td)
    dec = B200QwenTextDecoder(SimpleNamespace(wait_token_id=3, bos_token_id=1), text, QWEN_TEXT_DIMS["tnano"])
    return enc, dec, RealtimeFrames(enc, text, 256)


def _state(enc):
    return SimpleNamespace(audio=enc.init_state(), adapter=SimpleNamespace(audio_frames_seen=0, decoder_steps_seen=0),
                           frame_hidden=None, decoder=None)


GEN = dict(template_token_ids=[10, 11, 7, 12, 13], audio_placeholder_token_id=7, max_new_tokens=8, eos_token_id=5,
           suppress_token_ids=[7, 10, 11, 12, 13], repetition_penalty=1.15, no_repeat_ngram_size=3)


def test_d2h_bytes_per_chunk_do_not_grow_with_cached_steps():
    from oracle.make_golden_qwen import mel_stream
    enc, dec, frames = _realtime(max_sessions=2)
    st = _state(enc)
    mels = mel_stream(40 * 25, 128, seed=1)
    hyp, per_chunk = [], []
    for k in range(40):
        def chunk():
            nonlocal hyp
            frames.append([st], [torch.from_numpy(mels[k * 25: (k + 1) * 25])[None]])
            toks, _ = dec.generate_rolling_batch([st.frame_hidden[0]], [st], [hyp], **GEN)
            hyp = toks[0]
        if k in (2, 3, 36, 37):
            per_chunk.append((int(st.frame_hidden.shape[1]) if st.frame_hidden is not None else 0, _d2h_bytes(chunk)))
        else:
            chunk()
    print("D2H", per_chunk)
    short = max(b for _, b in per_chunk[:2])
    assert per_chunk[2][0] > 8 * max(1, per_chunk[0][0])               # a much longer segment
    assert short > 0
    assert max(b for _, b in per_chunk[2:]) <= short


def test_batched_tick_equals_streams_one_at_a_time():
    from oracle.make_golden_qwen import mel_stream
    enc, dec, frames = _realtime(max_sessions=16)
    n = 8
    batch, single = [_state(enc) for _ in range(n)], [_state(enc) for _ in range(n)]
    mels = [mel_stream(12 * 27, 128, seed=10 + i) for i in range(n)]
    hb, hs = [[] for _ in range(n)], [[] for _ in range(n)]
    for k in range(12):
        sizes = [(k * 7 + i * 5) % 40 for i in range(n)]               # ragged, some chunks empty
        chunk = [torch.from_numpy(mels[i][k * 27: k * 27 + sizes[i]])[None] for i in range(n)]
        frames.append(batch, chunk)
        tb, sb = dec.generate_rolling_batch([s.frame_hidden[0] for s in batch], batch, hb, **GEN)
        for i in range(n):
            frames.append([single[i]], [chunk[i]])
            ts, ss = dec.generate_rolling_batch([single[i].frame_hidden[0]], [single[i]], [hs[i]], **GEN)
            assert ts[0] == tb[i] and ss[0] == sb[i], (k, i, ts[0], tb[i], ss[0], sb[i])
            assert torch.equal(single[i].frame_hidden, batch[i].frame_hidden)
            hs[i] = ts[0]
        hb = tb
