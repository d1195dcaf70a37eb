#!/usr/bin/env python
"""Build container only: fixtures for the incremental log-mel front end, produced by the REFERENCE's
StreamingMelExtractor (features.py) over the real Hugging Face WhisperFeatureExtractor(feature_size=128).
    python oracle/make_golden_qwen_mel.py     # -> tests/golden/qwen_mel.npz"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))   # the staged reference holds qwen3_asr_causal

# samples per append: sub-window, sub-frame, typical 0.25 s, long, empty
MEL_SCHEDULE = [150, 60, 4000, 4000, 100, 150, 37, 8000, 0, 4000, 16000, 4001, 399]


def speechlike(n, seed=0):
    from whisperlivekit_b200.weights import synthetic_audio
    return synthetic_audio(n / 16000.0 + 0.01, seed=seed)[:n]


def main():
    from transformers import WhisperFeatureExtractor
    from qwen3_asr_causal.features import StreamingMelExtractor
    sx = StreamingMelExtractor(WhisperFeatureExtractor(feature_size=128))
    audio = speechlike(sum(MEL_SCHEDULE), seed=17)
    rec = dict(schedule=np.asarray(MEL_SCHEDULE, np.int64))
    a = 0
    for i, n in enumerate(MEL_SCHEDULE + [-1]):
        out = sx.flush() if n < 0 else sx.append(audio[a: a + n])
        a += max(n, 0)
        m = np.zeros((0, 128), np.float32) if out is None else out[0].numpy()
        rec[f"frames{i}"] = np.asarray(m.shape[0], np.int64)
        rec[f"emitted{i}"] = np.asarray(sx.emitted_frames, np.int64)
        if m.size:
            flat = m.reshape(-1)
            idx = np.arange(0, flat.shape[0], max(1, flat.shape[0] // 389), dtype=np.int64)
            rec[f"idx{i}"], rec[f"val{i}"] = idx, flat[idx]
            rec[f"rowsum{i}"] = m.astype(np.float64).sum(axis=1).astype(np.float32)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "qwen_mel.npz"), **rec)
    print("emitted", sx.emitted_frames, "of", sum(MEL_SCHEDULE) // 160)


if __name__ == "__main__":
    main()
