#!/usr/bin/env python
"""The FP8 serving mode (WLK_PREC_FP8) against the bf16 one on the encode tick, in one process.

    python tools/bench_fp8.py [--streams 48] [--rounds 3] [--steps 16]

Builds a bf16 and an fp8 large-v3 engine on the same seeded weights, then alternates them over the same encode tick
(--streams streams of full 30 s windows) for --rounds rounds: per round and mode the tick time (CUDA events around the
encode call) and the per-class milliseconds of the profile (gemm_enc, gemm_xkv, attn_enc, layernorm; a separate
profiled encode, so the tick time is taken with the profile off).  Then the fp8-vs-bf16 agreement on a teacher-forced
prefix: greedy tokens of --steps steps fed the bf16 engine's choice, and the max |delta logit|.  The card's name, power
limit and maximum SM clock are printed beside the figures (nvidia-smi, read-only query)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

from whisperlivekit_b200.dims import ALIGNMENT_HEADS, DIMS  # noqa: E402
from whisperlivekit_b200.engine import WhisperEngine  # noqa: E402
from whisperlivekit_b200.weights import synthetic_audio, synthetic_state_dict  # noqa: E402

CLASSES = ("gemm_enc", "gemm_xkv", "attn_enc", "layernorm")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=48)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=16)
    a = ap.parse_args()
    dims = DIMS["large-v3"]
    sd = synthetic_state_dict(dims, seed=0)
    engs = {p: WhisperEngine(dims, sd, ALIGNMENT_HEADS["large-v3"], precision=p, max_sessions=a.streams,
                             max_batch=a.streams) for p in ("bf16", "fp8")}
    del sd
    audio = [synthetic_audio(30.0, seed=k) for k in range(a.streams)]
    sids = {}
    for p, e in engs.items():
        sids[p] = [e.open_session() for _ in range(a.streams)]
        for s, au in zip(sids[p], audio):
            e.append_audio(s, au)
        e.encode(sids[p])                                   # warm-up: every shape of the tick
        e.sync()
    rounds = []
    for r in range(a.rounds):
        row = {}
        for p, e in engs.items():
            e.timer_record(0)
            e.encode(sids[p])
            e.timer_record(1)
            tick = e.timer_elapsed_ms(0, 1)
            e.profile_reset()
            e.profile_enable(True)
            e.encode(sids[p])
            prof = e.profile_read()
            e.profile_enable(False)
            e.profile_reset()
            row[p] = dict(tick_ms=round(tick, 2), **{c: round(prof[c]["ms"], 2) for c in CLASSES})
        rounds.append(row)
        print(json.dumps(dict(round=r, **row)), flush=True)

    # agreement on a teacher-forced prefix of the first stream (bf16's greedy choice fed to both)
    e16, e8 = engs["bf16"], engs["fp8"]
    s16, s8 = sids["bf16"][0], sids["fp8"][0]
    e16.encode([s16]); e8.encode([s8])
    feed = list(e16.specials.sot_sequence_including_notimestamps())
    same, dmax = 0, 0.0
    for _ in range(a.steps):
        e16.decode([s16], [feed]); e8.decode([s8], [feed])
        l16, l8 = e16.read_logits(s16), e8.read_logits(s8)
        t16, t8 = int(np.argmax(l16)), int(np.argmax(l8))
        same += t16 == t8
        dmax = max(dmax, float(np.abs(l16 - l8).max()))
        feed = [t16]
    med = {p: {k: float(np.median([r[p][k] for r in rounds])) for k in rounds[0][p]} for p in engs}
    print(json.dumps(dict(card=card(), streams=a.streams, median=med, tokens_agree=same, steps=a.steps,
                          max_abs_dlogit=round(dmax, 4))))
    for e in engs.values():
        e.close()


if __name__ == "__main__":
    main()
