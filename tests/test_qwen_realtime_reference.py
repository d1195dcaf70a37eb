"""The whole realtime model installed on a reference Qwen3ASRRealtimeQwenAudioCausalModel (needs the staged reference,
oracle/_ref, and transformers; the CPU oracles stand behind the engine API): the reference's segmented streamer drives the
installed model and an untouched twin side by side, and the events must be equal on every chunk.  When the streamer and
the model are gone, no engine session is left open."""
import gc

import pytest
import torch

pytestmark = pytest.mark.reference
pytest.importorskip("transformers")


@pytest.mark.parametrize("name", ["qnano", "qnano-tail"])
def test_installed_model_equals_reference_side_by_side(name):
    from oracle import stage_reference
    stage_reference.import_staged_reference()
    from oracle.make_golden_qwen import mel_stream
    from oracle.make_golden_qwen_realtime import CHUNK, build_model, build_streamer, event_record
    from test_oracle_qwen_realtime import oracle_factories
    from whisperlivekit_b200.qwen_plugin import B200QwenAudioState, B200QwenRealtimeModel
    ref, mine = build_model(name), build_model(name)
    tower, text, made = oracle_factories()
    B200QwenRealtimeModel.install(mine, tower_factory=tower, text_factory=text)
    sr, sm = build_streamer(ref), build_streamer(mine)
    mels = mel_stream(1400, 128, seed=9)
    rollovers = 0
    with torch.no_grad():
        for a in range(0, mels.shape[0], CHUNK):
            chunk = torch.from_numpy(mels[a: a + CHUNK])[None]
            er = event_record(sr.append_mel_chunk(chunk), sr)
            em = event_record(sm.append_mel_chunk(chunk), sm)
            assert em == er, (a, {k: (em.get(k), er.get(k)) for k in set(em) | set(er) if em.get(k) != er.get(k)})
            assert isinstance(sm.state.audio, B200QwenAudioState)
            rollovers += int(bool(er.get("segment_rollover") or er.get("segment_rolled_before_generate")))
        er, em = sr.flush_pending_audio(), sm.flush_pending_audio()
        assert (em is None) == (er is None)
        assert er is None or event_record(em, sm) == event_record(er, sr)
    assert rollovers >= 3
    del sm, mine
    gc.collect()
    assert not made["tower"][0]._s, "tower sessions left open"
    assert not made["text"][0].sessions, "text sessions left open"
