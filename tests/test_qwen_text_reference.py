"""The Qwen3 text-decoder seam (needs the staged reference, oracle/_ref, and transformers).  A reference realtime model
with the drop-in installed (B200QwenTextDecoder, the CPU oracle behind the engine API) and an untouched twin with the
same seeded Qwen3Model are driven side by side: tokens and stats must be equal on every call, including rebuilds,
draft accept / reject and the fallback paths; a segment rollover leaves no open sessions behind."""
import gc

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.reference
pytest.importorskip("transformers")


def _models():
    from oracle import stage_reference
    stage_reference.import_staged_reference()              # oracle/_ref also holds qwen3_asr_causal
    from oracle.make_golden_qwen_text import build_reference
    from oracle.qwen_text_oracle import QwenTextOracle
    from whisperlivekit_b200.qwen_dims import QWEN_TEXT_DIMS, synthetic_text_state_dict
    from whisperlivekit_b200.qwen_plugin import B200QwenTextDecoder
    dims = QWEN_TEXT_DIMS["tnano"]
    sd = synthetic_text_state_dict(dims, 9)
    ref, mine = build_reference(dims, sd), build_reference(dims, sd)
    oracles = []

    def factory(d, s):
        oracles.append(QwenTextOracle(d, s))
        return oracles[-1]

    dec = B200QwenTextDecoder.install(mine, engine_factory=factory)
    assert dec.dims == dims                                  # geometry recovered from the HF config
    # the engine gets the model's live RoPE buffer (non-persistent: not in state_dict())
    assert torch.equal(oracles[0].inv_freq, mine.text_model.rotary_emb.inv_freq)
    return ref, mine, oracles[0]


def test_drop_in_equals_reference_side_by_side():
    from oracle.make_golden_qwen_text import CONTROLS_OFF, CONTROLS_ON, EOS, PLACEHOLDER, TEMPLATE_A, TEMPLATE_B
    from qwen3_asr_causal.model import CachedAudioDecodeState
    ref, mine, orc = _models()
    frames = torch.as_tensor(np.random.default_rng(5).standard_normal((1, 40, 256)).astype(np.float32))
    sr, sm = CachedAudioDecodeState(audio=None, adapter=None), CachedAudioDecodeState(audio=None, adapter=None)
    prev = None
    plan = [(5, TEMPLATE_A, "prev", CONTROLS_ON), (9, TEMPLATE_A, "prev", CONTROLS_ON), (9, TEMPLATE_A, "prev", CONTROLS_ON),
            (14, TEMPLATE_A, "bad", CONTROLS_ON), (20, TEMPLATE_B, "prev", CONTROLS_OFF), (26, TEMPLATE_B, "eos", CONTROLS_ON),
            (30, TEMPLATE_B, "long", CONTROLS_ON)]
    with torch.no_grad():
        for steps, tpl, rule, ctl in plan:
            draft = None
            if prev:
                draft = {"prev": prev, "bad": prev[:2] + [77] + prev[3:], "eos": prev[:3] + [EOS] + prev[3:],
                         "long": prev * 2}[rule]
            kw = dict(template_token_ids=tpl, audio_placeholder_token_id=PLACEHOLDER, draft_token_ids=draft,
                      max_new_tokens=10, eos_token_id=EOS, **ctl)
            tr, str_ = ref.generate_full_hypothesis_rolling(frames[:, :steps], state=sr, **kw)
            tm, stm = mine.generate_full_hypothesis_rolling(frames[:, :steps], state=sm, **kw)
            assert tm.tolist() == tr.tolist(), (steps, tm, tr)
            assert stm == str_, (stm, str_)
            prev = tr[0].tolist()
        # fallbacks: batch 2, max_new_tokens 0, no audio; the non-rolling method with and without the decoder cache
        for fh, mnt in ((frames[:, :6].repeat(2, 1, 1), 6), (frames[:, :6], 0), (frames[:, :0], 6)):
            kw = dict(template_token_ids=TEMPLATE_A, audio_placeholder_token_id=PLACEHOLDER, max_new_tokens=mnt,
                      eos_token_id=EOS, **CONTROLS_ON)
            tr, str_ = ref.generate_full_hypothesis_rolling(fh, state=sr, **kw)
            tm, stm = mine.generate_full_hypothesis_rolling(fh, state=sm, **kw)
            assert tm.tolist() == tr.tolist() and stm == str_
        for cache in (True, False):
            kw = dict(prefix_token_ids=[10, 11] + [PLACEHOLDER] * 8 + [12, 13], audio_placeholder_token_id=PLACEHOLDER,
                      max_new_tokens=9, eos_token_id=EOS, use_decoder_kv_cache=cache, **CONTROLS_ON)
            assert (mine.generate_full_hypothesis_from_cached_audio(frames[:, :8], **kw).tolist()
                    == ref.generate_full_hypothesis_from_cached_audio(frames[:, :8], **kw).tolist())
            kw = dict(max_new_tokens=9, eos_token_id=EOS, use_decoder_kv_cache=cache)
            assert (mine.generate_full_hypothesis_from_cached_audio(frames[:, :7], **kw).tolist()
                    == ref.generate_full_hypothesis_from_cached_audio(frames[:, :7], **kw).tolist())


def test_segment_rollover_leaves_no_open_sessions():
    from oracle.make_golden_qwen_text import CONTROLS_ON, EOS, PLACEHOLDER, TEMPLATE_A
    from qwen3_asr_causal.model import CachedAudioDecodeState
    _, mine, orc = _models()
    frames = torch.as_tensor(np.random.default_rng(6).standard_normal((1, 12, 256)).astype(np.float32))
    kw = dict(template_token_ids=TEMPLATE_A, audio_placeholder_token_id=PLACEHOLDER, max_new_tokens=4, eos_token_id=EOS,
              **CONTROLS_ON)
    with torch.no_grad():
        for segment in range(3):                            # each segment starts from a fresh decode state
            st = CachedAudioDecodeState(audio=None, adapter=None)
            for steps in (4, 8, 12):
                mine.generate_full_hypothesis_rolling(frames[:, :steps], state=st, **kw)
            assert len(orc.sessions) == 1
            del st
            gc.collect()
    assert len(orc.sessions) == 0
