#!/usr/bin/env python
"""Cost of the Qwen3-ASR text decoder (csrc/qwen_text.cu) at the causal backend's operating point: S streams per GPU,
0.25 s chunks (3 new audio steps of 80 ms per tick), the previous hypothesis as the draft, repetition_penalty 1.15,
no_repeat_ngram_size 3.  Prints one JSON line.

Seeded weights never emit EOS and make drafts churn, so the cost of a tick is bracketed instead of simulated:
  accepted   every draft verifies: one forward of [audio delta + template tail + draft] per stream and one pick over
             all verify rows (the whole tick)
  rejected   every draft is rejected at its first token: the same verify, then `hyp` sequential steps (one-row forward
             + pick over all streams) to rebuild a hypothesis of the same length
Neither bracket is a prediction of real speech.  Per-step bytes come from shapes: the bf16 weights the step streams plus
K/V bytes of every cached position of every stream; the ratio to 3.35 TB/s is the step's share of H100 SXM HBM
bandwidth.

    python tools/bench_qwen_text.py [--streams 128] [--prefix 160] [--hyp 32] [--iters 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from whisperlivekit_b200.qwen_dims import QWEN_TEXT_DIMS, synthetic_text_state_dict  # noqa: E402
from whisperlivekit_b200.qwen_text_engine import QwenTextEngine  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:                                   # noqa: BLE001
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dims", default="qwen3-asr-0.6b")
    ap.add_argument("--streams", type=int, default=128)
    ap.add_argument("--prefix", type=int, default=160, help="positions cached per stream (head + audio) at the tick")
    ap.add_argument("--delta", type=int, default=3, help="new audio steps per tick (0.25 s of 80 ms steps)")
    ap.add_argument("--tail", type=int, default=5, help="template tail tokens")
    ap.add_argument("--hyp", type=int, default=32, help="hypothesis (draft) length")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--precision", default="bf16")
    a = ap.parse_args()
    D = QWEN_TEXT_DIMS[a.dims]
    S = a.streams
    name, power = gpu_info()
    t0 = time.perf_counter()
    eng = QwenTextEngine(D, synthetic_text_state_dict(D, 0), precision=a.precision, max_sessions=S, max_batch=S)
    load_s = time.perf_counter() - t0
    rng = np.random.default_rng(1)
    sids = [eng.open_session() for _ in range(S)]
    # cached prefix of every stream
    eng.forward(sids, [(-1 - np.arange(a.prefix, dtype=np.int32), rng.standard_normal((a.prefix, D.d_model)).astype(np.float32))
                       for _ in sids], [1] * S)
    ctl = eng.make_controls(eos_token_id=151645, repetition_penalty=1.15, no_repeat_ngram_size=3,
                            suppress_token_ids=[151669, 151670, 151669 + 7, 151669 + 8, 151669 + 9, 151644])
    delta = rng.standard_normal((a.delta, D.d_model)).astype(np.float32)
    draft = rng.integers(100, 150000, a.hyp).astype(np.int32)
    tail = np.arange(1000, 1000 + a.tail, dtype=np.int32)
    block = (np.concatenate([-1 - np.arange(a.delta, dtype=np.int32), tail, draft]), delta)
    hist = np.tile(draft, S)
    v_off = np.concatenate([np.full(a.hyp + 1, i * a.hyp, np.int32) for i in range(S)])
    v_len = np.tile(np.arange(a.hyp + 1, dtype=np.int32), S)
    base = a.prefix

    def verify():
        eng.forward(sids, [block] * S, [a.hyp + 1] * S)
        return eng.pick(hist, v_off, v_len, ctl)

    def step(k):
        eng.forward(sids, [(np.asarray([int(draft[k % a.hyp])], np.int32), None)] * S, [1] * S)
        return eng.pick(hist, np.arange(S, dtype=np.int32) * a.hyp, np.full(S, min(k + 1, a.hyp), np.int32), ctl)

    def crop(n):
        for s in sids:
            eng.crop(s, n)

    verify(); crop(base); step(0); crop(base)                  # warm-up
    tv, ts = [], []
    for _ in range(a.iters):
        t = time.perf_counter(); verify(); tv.append(time.perf_counter() - t)
        crop(base + a.delta + a.tail + 1)                      # rejected at the first draft token
        for k in range(a.hyp):
            t = time.perf_counter(); step(k); ts.append(time.perf_counter() - t)
        crop(base)
    t_verify = float(np.median(tv))
    t_step = float(np.median(ts))
    es = 2 if a.precision == "bf16" else 4
    L, d, F, H, KV, hd = D.n_layer, D.d_model, D.ffn_dim, D.n_head, D.n_kv_head, D.head_dim
    w_bytes = es * (L * (d * (H + 2 * KV) * hd + H * hd * d + 3 * d * F) + D.vocab * d)
    kv_per_pos = es * L * 2 * KV * hd
    ctx_mean = base + a.delta + a.tail + a.hyp // 2
    step_bytes = w_bytes + S * ctx_mean * kv_per_pos
    res = {
        "bench": "qwen_text", "gpu": name, "power_limit": power, "dims": a.dims, "precision": a.precision, "streams": S,
        "prefix_positions": base, "delta_steps": a.delta, "tail_tokens": a.tail, "hyp_tokens": a.hyp,
        "verify_ms": round(t_verify * 1e3, 3), "step_ms": round(t_step * 1e3, 3),
        "tick_ms_all_accepted": round(t_verify * 1e3, 3),
        "tick_ms_all_rejected": round((t_verify + a.hyp * t_step) * 1e3, 3),
        "step_weight_bytes": w_bytes, "kv_bytes_per_position_per_stream": kv_per_pos,
        "step_bytes": step_bytes, "step_bytes_per_s": round(step_bytes / t_step, 1),
        "step_hbm_fraction_of_3.35TBps": round(step_bytes / t_step / 3.35e12, 4),
        "load_s": round(load_s, 1), "memory": eng.memory(),
    }
    for s in sids:
        eng.close_session(s)
    eng.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
