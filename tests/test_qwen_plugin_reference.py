"""The Qwen3 seam (needs the staged reference, oracle/_ref).  The reference's QwenAudioCausalKVEncoder and the drop-in built FROM it
(weights taken from its tower's state_dict, geometry read off its modules) are driven with the same ragged chunk
schedule; hidden states and the state fields callers read must agree.  The CPU oracle stands behind the engine API."""
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.reference


@pytest.mark.parametrize("name", ["qnano", "qnano-chunk", "qnano-tail", "qnano-tail-bidir"])
def test_drop_in_encoder_equals_reference(name):
    from oracle import stage_reference
    stage_reference.import_staged_reference()              # oracle/_ref also holds qwen3_asr_causal
    from oracle.make_golden_qwen import SCHEDULE, TAIL_SCHEDULE, mel_stream, reference_encoder
    from oracle.qwen_oracle import QwenTowerOracle
    from whisperlivekit_b200.qwen_dims import QWEN_DIMS, synthetic_tower_state_dict
    from whisperlivekit_b200.qwen_plugin import B200QwenAudioCausalKVEncoder

    dims = QWEN_DIMS[name]
    if dims.mutable_tail_steps:
        SCHEDULE = TAIL_SCHEDULE                                          # tail + new steps stay below 128 per call
    ref = reference_encoder(dims, synthetic_tower_state_dict(dims, seed=23))
    mine = B200QwenAudioCausalKVEncoder.from_reference(ref, engine_factory=lambda d, sd: QwenTowerOracle(d, sd))
    assert mine.dims == dims                                              # geometry recovered from the modules
    mels = torch.from_numpy(mel_stream(sum(SCHEDULE), dims.n_mels, seed=4))
    sr, sm = ref.init_state(), mine.init_state()
    a = 0
    with torch.no_grad():
        for n in SCHEDULE:
            hr, sr = ref.forward_chunk(mels[None, a: a + n], sr)
            hm, sm = mine.forward_chunk(mels[None, a: a + n], sm)
            a += n
            assert hm.shape == hr.shape
            if hr.numel():
                assert float((hm - hr).abs().max()) < 2e-5
            for f in ("frames_seen", "emitted_steps", "pending_frames", "last_input_frames", "last_recomputed_frames",
                      "last_recomputed_context_frames", "mutable_steps"):
                assert getattr(sm, f) == getattr(sr, f), f
        hr, sr = ref.flush_pending(sr)
        hm, sm = mine.flush_pending(sm)
        assert hm.shape == hr.shape and (not hr.numel() or float((hm - hr).abs().max()) < 2e-5)
        assert sm.emitted_steps == sr.emitted_steps and sm.pending_frames == 0
    assert mine.right_context_frames == ref.right_context_frames
    assert mine.output_steps_for_mel_frames(195) == ref.output_steps_for_mel_frames(195)


def test_drop_in_mel_extractor_equals_reference():
    """StreamingMelExtractor (reference, over the real Hugging Face featurizer) vs the drop-in over the engine API
    (CPU oracle behind it): same frames per append / flush, same values."""
    from oracle import stage_reference
    stage_reference.import_staged_reference()              # oracle/_ref also holds qwen3_asr_causal
    from transformers import WhisperFeatureExtractor
    from qwen3_asr_causal.features import StreamingMelExtractor
    from oracle.make_golden_qwen_mel import speechlike
    from oracle.qwen_oracle import QwenTowerOracle
    from whisperlivekit_b200.qwen_dims import QWEN_DIMS, synthetic_tower_state_dict
    from whisperlivekit_b200.qwen_plugin import B200StreamingMelExtractor

    dims = QWEN_DIMS["qnano"]
    eng = QwenTowerOracle(dims, synthetic_tower_state_dict(dims, seed=1))
    eng.load_mel_filters()
    ref = StreamingMelExtractor(WhisperFeatureExtractor(feature_size=128))
    mine = B200StreamingMelExtractor(eng, eng.open_session())
    audio = speechlike(16000 * 4, seed=77)
    a = 0
    for n in (100, 150, 4000, 333, 4000, 0, 12000, 4001):
        r, m = ref.append(audio[a: a + n]), mine.append(audio[a: a + n])
        a += n
        assert (r is None) == (m is None)
        if r is not None:
            assert tuple(r.shape) == tuple(m.shape) and float((r - m).abs().max()) < 5e-5
        assert ref.emitted_frames == mine.emitted_frames
    r, m = ref.flush(), mine.flush()
    assert (r is None) == (m is None) and (r is None or float((r - m).abs().max()) < 5e-5)
    assert ref.emitted_frames == mine.emitted_frames == a // 160
