"""The windowed realtime model (Qwen3ASRRealtimeQwenAudioSurgeryModel) installed on the engines, with the CPU oracles
behind the engine API, against fixtures recorded from the reference (oracle/make_golden_qwen_window_realtime.py); and the
text driver's batched non-rolling generate against N single ones."""
import gc
import json
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["w0", "wtail"]


def fixture(name):
    z = np.load(os.path.join(ROOT, "tests", "golden", f"qwen_window_realtime_{name}.npz"))
    return z, json.loads(bytes(z["events"]).decode())


def oracle_factories():
    from oracle.qwen_realtime_oracle import QwenRealtimeTextOracle
    from test_plugin_qwen_window import OracleWindowEngine
    made = {"tower": [], "text": []}

    def tower(d, sd):
        made["tower"].append(OracleWindowEngine(d, sd))
        return made["tower"][-1]

    def text(d, sd):
        made["text"].append(QwenRealtimeTextOracle(d, sd))
        return made["text"][-1]
    return tower, text, made


def _reference():
    pytest.importorskip("transformers")
    from oracle import stage_reference
    stage_reference.import_staged_reference()


def test_fixtures_cover_the_windowed_schedule():
    from oracle.make_golden_qwen_window_realtime import FIXTURES, SCHEDULE
    for name in NAMES:
        _, ev = fixture(name)
        assert len(ev) == len(SCHEDULE) + 1
        assert sum(1 for e in ev if e.get("segment_rollover")) >= 3
        assert ev[-1]["is_flush"] and ev[-1]["input_mel_frames"] == 64
        assert all(e["encoder_pending_frames"] == 0 for e in ev)
        assert any(0 < n < 100 for n in SCHEDULE)
    # the keep-tail fixture starts a segment on a trimmed [:, -k:] copy of the previous one
    _, w0 = fixture("w0")
    _, wt = fixture("wtail")
    assert FIXTURES["wtail"] > 0 and [e["cached_steps"] for e in w0] != [e["cached_steps"] for e in wt]


@pytest.mark.reference
@pytest.mark.parametrize("name", NAMES)
def test_installed_windowed_model_with_oracles_reproduces_every_event(name):
    _reference()
    from oracle.make_golden_qwen_window_realtime import FIXTURES, build_model, build_streamer, drive, mels
    from whisperlivekit_b200.qwen_plugin import B200QwenAudioSurgeryEncoder, B200QwenRealtimeModel
    _, want = fixture(name)
    model = build_model()
    tower, text, made = oracle_factories()
    # the fixture tower's varlen attention applies its blocks, which no attention name tells apart
    rt = B200QwenRealtimeModel.install(model, tower_factory=tower, text_factory=text, attention_blocks=True)
    assert isinstance(model.audio_encoder, B200QwenAudioSurgeryEncoder)
    assert not hasattr(model, "flush_audio_to_cache")
    streamer = build_streamer(model, FIXTURES[name])
    got = drive(streamer, mels())
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, (i, {k: (g.get(k), w.get(k)) for k in set(g) | set(w) if g.get(k) != w.get(k)})
    rt.decoder.close()
    assert made["text"][0].sessions == {}
    del streamer
    gc.collect()
    assert made["tower"][0].open == set()


@pytest.mark.reference
@pytest.mark.parametrize("name", NAMES)
def test_reference_streamer_drives_installed_model_and_untouched_twin_alike(name):
    _reference()
    from oracle.make_golden_qwen_window_realtime import FIXTURES, build_model, build_streamer, drive, mels
    from whisperlivekit_b200.qwen_plugin import B200QwenRealtimeModel
    twin, model = build_model(), build_model()
    tower, text, _ = oracle_factories()
    B200QwenRealtimeModel.install(model, tower_factory=tower, text_factory=text, attention_blocks=True)
    ref_streamer, dev_streamer = build_streamer(twin, FIXTURES[name]), build_streamer(model, FIXTURES[name])
    per_chunk = []
    drive(ref_streamer, mels(), on_chunk=lambda s: per_chunk.append(s.last_hypothesis_tokens[:]))
    k = 0

    def check(s):
        nonlocal k
        assert s.last_hypothesis_tokens == per_chunk[k], k
        k += 1
    drive(dev_streamer, mels(), on_chunk=check)
    assert k == len(per_chunk)


@pytest.mark.reference
def test_install_rejects_tower_wider_than_the_adapter():
    _reference()
    import dataclasses
    from oracle.make_golden_qwen_window_realtime import build_model
    from whisperlivekit_b200.qwen_plugin import B200QwenAudioSurgeryEncoder, B200QwenRealtimeModel
    model = build_model()
    tower, text, _ = oracle_factories()
    real = B200QwenAudioSurgeryEncoder.dims_of

    def wider(ref, attention_blocks=None):
        return dataclasses.replace(real(ref, attention_blocks), out_dim=128)
    B200QwenAudioSurgeryEncoder.dims_of = staticmethod(wider)
    try:
        with pytest.raises(ValueError, match="adapter takes"):
            B200QwenRealtimeModel.install(model, tower_factory=tower, text_factory=text)
    finally:
        B200QwenAudioSurgeryEncoder.dims_of = real


def _text_oracle():
    from oracle.qwen_text_oracle import QwenTextOracle
    from whisperlivekit_b200.qwen_dims import QWEN_TEXT_DIMS, synthetic_text_state_dict
    dims = QWEN_TEXT_DIMS["tnano"]
    return QwenTextOracle(dims, synthetic_text_state_dict(dims, 5)), dims


def ragged_case(dims, n=5, seed=3):
    """Ragged prefixes (tokens around frame rows) with frame rows of their own per session."""
    rng = np.random.default_rng(seed)
    rows, prefixes = [], []
    for i in range(n):
        steps = int(rng.integers(1, 9))
        fh = rng.standard_normal((steps, dims.d_model)).astype(np.float32)
        head = [10, 11] if i % 2 else [10]
        src = np.concatenate([np.asarray(head, np.int32), -1 - np.arange(steps, dtype=np.int32),
                              np.asarray([12, 13][: 1 + i % 2], np.int32)])
        rows.append(fh)
        prefixes.append(src)
    return rows, prefixes


@pytest.mark.parametrize("controls", [
    dict(suppress_token_ids=[7, 10, 11, 12, 13]),
    dict(suppress_token_ids=[7, 10, 11, 12, 13], repetition_penalty=1.15, no_repeat_ngram_size=3,
         max_consecutive_text_tokens=4, wait_token_id=3),
])
@pytest.mark.parametrize("max_new", [0, 1, 9])
def test_batched_oracle_equals_single_generates(controls, max_new):
    orc, dims = _text_oracle()
    rows, prefixes = ragged_case(dims)
    def singles(**kw):
        return [orc.generate_full(fh, prefix_token_ids=[int(t) if t >= 0 else 7 for t in src], audio_placeholder_token_id=7,
                                  max_new_tokens=max_new, **controls, **kw) for fh, src in zip(rows, prefixes)]
    free = singles()
    # stop ids that the single runs hit at different steps
    stops = sorted({s[k] for s, k in zip(free, (1, 3, 5)) if len(s) > k})
    want = singles(stop_token_ids=stops)
    assert len({len(s) for s in want}) > 1 or max_new <= 1
    assert orc.sessions == {}
    sids = [orc.open_session() for _ in rows]
    got = orc.generate_full_batch(sids, rows, prefixes, max_new_tokens=max_new, stop_token_ids=stops, **controls)
    assert got == want
    assert all(len(g) == max_new for g in got) if max_new == 0 else all(1 <= len(g) <= max_new for g in got)
    assert all(orc.session_len(s) == 0 for s in sids)


def test_generate_full_is_the_batch_of_one():
    orc, dims = _text_oracle()
    rows, prefixes = ragged_case(dims, n=1, seed=9)
    ctl = orc.make_controls(suppress_token_ids=[7], repetition_penalty=1.15, no_repeat_ngram_size=3)
    # the same tokens as the prefix written with placeholders through generate_full
    prefix = [int(t) if t >= 0 else 7 for t in prefixes[0]]
    a = orc.generate_full(rows[0], prefix_token_ids=prefix, audio_placeholder_token_id=7, max_new_tokens=10, controls=ctl)
    sid = orc.open_session()
    b = orc.generate_full_batch([sid], rows, prefixes, max_new_tokens=10, controls=ctl)[0]
    assert a == b and len(a) == 10
    with pytest.raises(ValueError):
        orc.generate_full_batch([sid], rows, prefixes, max_new_tokens=-1)
    with pytest.raises(ValueError):
        orc.generate_full_batch([sid], rows, [np.zeros(0, np.int32)], max_new_tokens=2)
