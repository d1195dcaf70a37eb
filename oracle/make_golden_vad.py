#!/usr/bin/env python
"""Build container only: Silero VAD fixtures from the REFERENCE's scripted model (silero_vad.jit, loaded the way
silero_vad_iterator.py:20-29 does) with its weights replaced by seeded ones of the same shapes (the trained weights
are a reference asset and stay there); a second record uses the trained weights and keeps only the probabilities.
    python oracle/make_golden_vad.py     # -> tests/golden/vad.npz"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
JIT = os.path.join(ROOT, "oracle", "_ref", "whisperlivekit", "silero_vad_models", "silero_vad.jit")


def main():
    from oracle.vad_oracle import synthetic_vad_state_dict
    from whisperlivekit_b200.weights import synthetic_audio
    audio = np.concatenate([synthetic_audio(2.0, seed=31), np.zeros(8000, np.float32), 0.3 * synthetic_audio(1.5, seed=32)])
    n = len(audio) // 512
    rec = dict(n_windows=np.asarray(n, np.int64))
    for tag in ("seeded", "trained"):
        m = torch.jit.load(JIT, map_location="cpu").eval()
        if tag == "seeded":
            sd = m.state_dict()
            for k, v in synthetic_vad_state_dict(seed=9).items():
                sd[k] = torch.from_numpy(v)
            m.load_state_dict(sd)
        m.reset_states()
        with torch.no_grad():
            probs = [float(m(torch.from_numpy(audio[i * 512:(i + 1) * 512])[None], 16000)[0, 0]) for i in range(n)]
        rec[f"probs_{tag}"] = np.asarray(probs, np.float32)
        print(tag, "min/max", min(probs), max(probs))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "vad.npz"), **rec)


if __name__ == "__main__":
    main()
