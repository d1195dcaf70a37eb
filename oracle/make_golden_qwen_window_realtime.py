#!/usr/bin/env python
"""Build container only: golden fixtures for the windowed Qwen3-ASR realtime model, produced by the REFERENCE itself.

The reference's SegmentedCachedFullHypothesisStreamer (third_party/qwen3-asr-causal/src/qwen3_asr_causal/streamer.py) runs,
unchanged, with the windowed backend's settings (asr.py:151-158: no rolling decoder KV, no speculative draft, penalty
1.0, n-gram 0, stable_iterations 2, no punctuation rollover, no roll before generate, no encoder reset) over a
Qwen3ASRRealtimeQwenAudioSurgeryModel (model.py:1421-1509) built from the "wnano" stock tower of
make_golden_qwen_window (varlen attention blocks, out_dim 96), the tnano Qwen3Model of make_golden_qwen_text and a
2-block frame adapter with a non-square 96 -> 256 projection.  1400 mel frames go in ragged chunks around the 2 s
cadence, chunks under 100 frames included.  There is no empty chunk: the reference encoder answers one with a
[1, 0, d_model] tensor (model.py:568-570), which the adapter's 96-wide projection rejects.  A small
segment_max_cached_steps makes the segment roll over at least three times; right_context_frames of zeros with
is_flush=True end the stream (online.py:230-237).
Two fixtures: segment_keep_tail_steps 0 and KEEP_TAIL (the streamer's [:, -k:] trim).  Per event: the event record of
make_golden_qwen_realtime; plus the adapter's first inputs / outputs and strided samples of every lm_head output.

    python oracle/make_golden_qwen_window_realtime.py   # writes tests/golden/qwen_window_realtime_{w0,wtail}.npz
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))

from oracle.make_golden_qwen_realtime import (ADAPTER_HIDDEN, ADAPTER_LAYERS, ADAPTER_RECORD_CALLS,  # noqa: E402
                                              BOS, EOS, PLACEHOLDER, RESIDUAL_SCALE, SAMPLE_STRIDE, SUPPRESS, TEMPLATE,
                                              WAIT, WORD_START, StubTokenizer, event_record, load_adapter)
from whisperlivekit_b200.qwen_dims import (QWEN_TEXT_DIMS, QWEN_WINDOW_DIMS, synthetic_adapter_state_dict,  # noqa: E402
                                           synthetic_text_state_dict, synthetic_tower_state_dict)

TOWER = "wnano"
SCHEDULE = [150, 230, 60, 210, 190, 45, 250, 180, 85]           # 1400 mel frames
MAX_NEW, SEGMENT_MAX_STEPS, KEEP_TAIL = 12, 40, 9
MEL_SEED = 8
FIXTURES = {"w0": 0, "wtail": KEEP_TAIL}                         # name -> segment_keep_tail_steps


def adapter_sd(seed=5):
    return synthetic_adapter_state_dict(QWEN_WINDOW_DIMS[TOWER].out_dim, QWEN_TEXT_DIMS["tnano"].d_model, ADAPTER_HIDDEN,
                                        ADAPTER_LAYERS, RESIDUAL_SCALE, seed=seed + 1)


def build_model(seed=5):
    from qwen3_asr_causal.config import RealtimeAudioConfig
    from qwen3_asr_causal.model import Qwen3ASRRealtimeQwenAudioSurgeryModel
    from oracle.make_golden_qwen_text import build_reference
    from oracle.make_golden_qwen_window import stock_tower
    wd, xd = QWEN_WINDOW_DIMS[TOWER], QWEN_TEXT_DIMS["tnano"]
    text = build_reference(xd, synthetic_text_state_dict(xd, seed))
    cfg = RealtimeAudioConfig(d_model=xd.d_model, n_mels=wd.n_mels,
                              qwen_audio_left_context_sec=wd.left_context_frames / 100.0,
                              qwen_audio_right_context_ms=wd.right_context_frames * 10,
                              qwen_audio_adapter_hidden_dim=ADAPTER_HIDDEN, qwen_audio_adapter_layers=ADAPTER_LAYERS,
                              qwen_audio_adapter_residual_scale=RESIDUAL_SCALE)
    model = Qwen3ASRRealtimeQwenAudioSurgeryModel(
        cfg, qwen_model_id="seeded", audio_tower=stock_tower(wd, synthetic_tower_state_dict(wd, seed=11), "wlk_varlen"),
        text_model=text.text_model, lm_head=text.lm_head, bos_token_id=BOS, wait_token_id=WAIT,
        audio_output_dim=wd.out_dim).eval()
    assert model.audio_encoder.left_context_frames == wd.left_context_frames
    assert model.audio_encoder.right_context_frames == wd.right_context_frames
    load_adapter(model.adapter, adapter_sd(seed))
    return model


def build_streamer(model, keep_tail: int):
    from qwen3_asr_causal.streamer import CachedFullHypothesisConfig, SegmentedCachedFullHypothesisStreamer
    config = CachedFullHypothesisConfig(
        wait_token_id=WAIT, word_start_token_id=WORD_START, eos_token_id=EOS, max_new_tokens=MAX_NEW, hold_back_words=2,
        stable_iterations=2, commit_mode="word", suppress_token_ids=SUPPRESS, repetition_penalty=1.0,
        no_repeat_ngram_size=0, prompt_prefix_template=TEMPLATE, audio_placeholder_token_id=PLACEHOLDER,
        decoder_rolling_kv=False, speculative_draft=False)
    return SegmentedCachedFullHypothesisStreamer(
        model, StubTokenizer(), config, segment_max_cached_steps=SEGMENT_MAX_STEPS, segment_keep_tail_steps=keep_tail,
        segment_finalize_mode="latest", segment_punct_rollover=False, segment_roll_before_generate=False,
        reset_encoder_on_rollover=False)


def mels():
    """The stream's mel frames followed by the right-context drain of zeros."""
    from oracle.make_golden_qwen import mel_stream
    wd = QWEN_WINDOW_DIMS[TOWER]
    m = mel_stream(sum(SCHEDULE), wd.n_mels, seed=MEL_SEED)
    return np.concatenate([m, np.zeros((wd.right_context_frames, wd.n_mels), np.float32)])


def drive(streamer, m, on_chunk=None):
    """The streamer over SCHEDULE, then the drain with is_flush=True.  on_chunk(streamer) runs after every event."""
    events, a = [], 0
    chunks = SCHEDULE + [QWEN_WINDOW_DIMS[TOWER].right_context_frames]
    with torch.no_grad():
        for k, n in enumerate(chunks):
            ev = streamer.append_mel_chunk(torch.from_numpy(m[a: a + n])[None], is_flush=k == len(chunks) - 1)
            a += n
            events.append(event_record(ev, streamer))
            if on_chunk is not None:
                on_chunk(streamer)
        assert streamer.flush_pending_audio() is None          # the windowed model has no flush_audio_to_cache
    return events


def main():
    import json
    for name, keep in FIXTURES.items():
        model = build_model()
        ad_in, ad_out, samples = [], [], []
        model.adapter.proj.register_forward_hook(
            lambda m, i, o: ad_in.append(i[0].detach().reshape(-1, i[0].shape[-1]).numpy().copy())
            if len(ad_in) < ADAPTER_RECORD_CALLS and i[0].shape[1] else None)
        orig = model.adapter._project

        def project(x, orig=orig):
            y = orig(x)
            if x.shape[1] and len(ad_out) < ADAPTER_RECORD_CALLS:
                ad_out.append(y.detach().reshape(-1, y.shape[-1]).numpy().copy())
            return y
        model.adapter._project = project
        model.lm_head.register_forward_hook(
            lambda m, i, o: samples.append(o.detach().reshape(-1, o.shape[-1])[:, ::SAMPLE_STRIDE].numpy().copy()))
        events = drive(build_streamer(model, keep), mels())
        rolls = sum(1 for e in events if e.get("segment_rollover"))
        print(name, len(events), "events,", rolls, "rollovers, cached steps", [e["cached_steps"] for e in events])
        assert rolls >= 3
        out = os.path.join(ROOT, "tests", "golden", f"qwen_window_realtime_{name}.npz")
        np.savez_compressed(
            out, events=np.frombuffer(json.dumps(events).encode(), np.uint8),
            adapter_in=np.concatenate(ad_in), adapter_out=np.concatenate(ad_out),
            adapter_rows=np.asarray([a.shape[0] for a in ad_in], np.int32),
            samples=np.concatenate([s.reshape(-1) for s in samples]).astype(np.float32),
            sample_rows=np.asarray([s.shape[0] for s in samples], np.int32), sample_stride=np.int32(SAMPLE_STRIDE))
        print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
