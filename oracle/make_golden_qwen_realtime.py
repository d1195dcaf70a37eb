#!/usr/bin/env python
"""Build container only: golden fixtures for the whole Qwen3-ASR realtime model, produced by the REFERENCE itself.

The reference's SegmentedCachedFullHypothesisStreamer (third_party/qwen3-asr-causal/src/qwen3_asr_causal/streamer.py) runs,
unchanged, with the causal backend's settings (asr.py:159-187: rolling decoder KV, speculative draft, penalty 1.15,
n-gram 3, punctuation rollover, roll before generate, reset_encoder_on_rollover) over a Qwen3ASRRealtimeQwenAudioCausalModel
built from the seeded tower of make_golden_qwen (out_dim 256 = the text width), the tnano Qwen3Model of
make_golden_qwen_text and a 2-block frame adapter (hidden 128, residual_scale 0.1, seeded non-identity proj).  A stub
tokenizer ends some ids with "." so that punctuation rollover fires.  1200 mel frames (make_golden_qwen.mel_stream, seed MEL_SEED) go in 25-frame chunks, then
flush_pending_audio.  Per event: the event dict (hypothesis text, cached_steps, new_cached_steps, rollover fields, the
decoder stats) and the encoder's pending frames; plus the adapter's full inputs and outputs of its first calls and
strided samples of every lm_head output.

    python oracle/make_golden_qwen_realtime.py    # writes tests/golden/qwen_realtime_qnano.npz, qwen_realtime_qnano-tail.npz
"""
import dataclasses
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))

from whisperlivekit_b200.qwen_dims import (QWEN_DIMS, QWEN_TEXT_DIMS, synthetic_adapter_state_dict,  # noqa: E402
                                           synthetic_text_state_dict, synthetic_tower_state_dict)

PLACEHOLDER, BOS, EOS, WAIT, WORD_START = 7, 1, 5, 3, 4
TEMPLATE = [10, 11, PLACEHOLDER, 12, 13]
SUPPRESS = (PLACEHOLDER, 10, 11, 12, 13)
CHUNK, N_FRAMES, MAX_NEW = 25, 1200, 12
ADAPTER_HIDDEN, ADAPTER_LAYERS, RESIDUAL_SCALE = 128, 2, 0.1
SEGMENT_MAX_STEPS, PUNCT_MIN_STEPS = 40, 12
ADAPTER_RECORD_CALLS, SAMPLE_STRIDE = 6, 31
MEL_SEED = 6
GEOMETRIES = ("qnano", "qnano-tail")


class StubTokenizer:
    """Ids become words; every id divisible by 11 ends a sentence."""

    def decode(self, ids, skip_special_tokens=True):
        return " ".join(f"w{int(t)}" + ("." if int(t) % 11 == 0 else "") for t in ids)

    def encode(self, text, add_special_tokens=False):
        return list(TEMPLATE)


def tower_dims(name):
    return dataclasses.replace(QWEN_DIMS[name], out_dim=QWEN_TEXT_DIMS["tnano"].d_model)


def load_adapter(adapter, sd):
    """Seeded weights (qwen_dims.synthetic_adapter_state_dict) into the reference's QwenAudioSurgeryFrameAdapter."""
    with torch.no_grad():
        adapter.proj.weight.copy_(torch.from_numpy(sd["adapter.proj.weight"]))
        for i, b in enumerate(adapter.blocks):
            p = f"adapter.blocks.{i}."
            b.norm.weight.copy_(torch.from_numpy(sd[p + "norm.weight"]))
            for n in ("gate", "up", "down"):
                getattr(b.mlp, n).weight.copy_(torch.from_numpy(sd[p + f"mlp.{n}.weight"]))


def adapter_sd(name, seed=5):
    return synthetic_adapter_state_dict(tower_dims(name).out_dim, QWEN_TEXT_DIMS["tnano"].d_model, ADAPTER_HIDDEN,
                                        ADAPTER_LAYERS, RESIDUAL_SCALE, seed=seed + 1)


def build_model(name, seed=5):
    from qwen3_asr_causal.config import RealtimeAudioConfig
    from qwen3_asr_causal.causal import Qwen3ASRRealtimeQwenAudioCausalModel
    from oracle.make_golden_qwen import GeometryTower
    from oracle.make_golden_qwen_text import build_reference
    tdims, xdims = tower_dims(name), QWEN_TEXT_DIMS["tnano"]
    text = build_reference(xdims, synthetic_text_state_dict(xdims, seed))
    cfg = RealtimeAudioConfig(d_model=xdims.d_model, qwen_audio_block_bidirectional=tdims.block_bidirectional,
                              qwen_audio_block_frames=tdims.block_frames,
                              qwen_audio_left_context_sec=tdims.left_context_steps * 0.08,
                              qwen_audio_mutable_tail_sec=tdims.mutable_tail_steps * 0.08,
                              qwen_audio_adapter_hidden_dim=ADAPTER_HIDDEN, qwen_audio_adapter_layers=ADAPTER_LAYERS,
                              qwen_audio_adapter_residual_scale=RESIDUAL_SCALE)
    model = Qwen3ASRRealtimeQwenAudioCausalModel(
        cfg, qwen_model_id="seeded", audio_tower=GeometryTower(tdims, synthetic_tower_state_dict(tdims, seed=11)).eval(),
        text_model=text.text_model, lm_head=text.lm_head, bos_token_id=BOS, wait_token_id=WAIT,
        audio_output_dim=tdims.out_dim).eval()
    load_adapter(model.adapter, adapter_sd(name, seed))
    return model


def build_streamer(model):
    from qwen3_asr_causal.streamer import CachedFullHypothesisConfig, SegmentedCachedFullHypothesisStreamer
    config = CachedFullHypothesisConfig(
        wait_token_id=WAIT, word_start_token_id=WORD_START, eos_token_id=EOS, max_new_tokens=MAX_NEW, hold_back_words=2,
        stable_iterations=1, commit_mode="word", suppress_token_ids=SUPPRESS, repetition_penalty=1.15,
        no_repeat_ngram_size=3, prompt_prefix_template=TEMPLATE, audio_placeholder_token_id=PLACEHOLDER,
        decoder_rolling_kv=True, speculative_draft=True)
    return SegmentedCachedFullHypothesisStreamer(
        model, StubTokenizer(), config, segment_max_cached_steps=SEGMENT_MAX_STEPS, segment_keep_tail_steps=0,
        segment_finalize_mode="latest", segment_punct_rollover=True, segment_punct_min_steps=PUNCT_MIN_STEPS,
        segment_roll_before_generate=True, reset_encoder_on_rollover=True)


def event_record(event, streamer):
    """The deterministic part of an event (no timings) plus the encoder's pending frames."""
    rec = {k: v for k, v in event.items() if k != "generate_ms"}
    rec["encoder_pending_frames"] = int(getattr(streamer.state.audio, "pending_frames", 0))
    rec["hypothesis_tokens"] = [int(t) for t in streamer.last_hypothesis_tokens]
    return json.loads(json.dumps(rec))


def drive(streamer, mels):
    """The streamer over mels [frames, n_mels] in CHUNK-frame chunks, then flush_pending_audio."""
    events = []
    with torch.no_grad():
        for a in range(0, mels.shape[0], CHUNK):
            ev = streamer.append_mel_chunk(torch.from_numpy(mels[a: a + CHUNK])[None])
            events.append(event_record(ev, streamer))
        ev = streamer.flush_pending_audio()
        if ev is not None:
            events.append(event_record(ev, streamer))
    return events


def main():
    from oracle.make_golden_qwen import mel_stream
    for name in GEOMETRIES:
        model = build_model(name)
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
        streamer = build_streamer(model)
        mels = mel_stream(N_FRAMES, 128, seed=MEL_SEED)
        events = drive(streamer, mels)
        rolls = sum(1 for e in events if e.get("segment_rollover") or e.get("segment_rolled_before_generate"))
        carried = [e["encoder_pending_frames"] for e in events]
        print(name, len(events), "events,", rolls, "rollovers, pending after events", carried)
        out = os.path.join(ROOT, "tests", "golden", f"qwen_realtime_{name}.npz")
        np.savez_compressed(
            out, events=np.frombuffer(json.dumps(events).encode(), np.uint8),
            adapter_in=np.concatenate(ad_in), adapter_out=np.concatenate(ad_out),
            adapter_rows=np.asarray([a.shape[0] for a in ad_in], np.int32),
            samples=np.concatenate([s.reshape(-1) for s in samples]).astype(np.float32),
            sample_rows=np.asarray([s.shape[0] for s in samples], np.int32), sample_stride=np.int32(SAMPLE_STRIDE))
        print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
