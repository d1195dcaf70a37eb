#!/usr/bin/env python
"""Config 5 as one tick: the whole Qwen3-ASR realtime model (device mel -> causal audio tower -> frame adapter -> rolling
text decoder) for S streams per GPU at the 0.6B geometries with seeded weights.  Prints one JSON line.

Per tick every stream brings 0.25 s of PCM: the device mel (mel_append), the tower for all streams in one call with block
phases staggered so that a 192-frame block fires for about 1/8 of the streams per tick (24 steps each), one adapter call
over all new rows (adapter_layers 0, the production default, with a seeded non-identity 1024 -> 1024 proj), and a rolling
generate for every stream with its previous hypothesis as the draft (the streamer generates on every chunk, even when the
delta is zero).  Seeded weights make drafts churn; two text regimes are timed:
  prev_draft  the previous hypothesis as the draft, as the streamer passes it (with seeded weights most drafts fail early)
  rejected    every draft fails at its first token (a suppressed id): verify, then max_new_tokens sequential steps, the
              upper bracket (seeded weights never emit EOS)
The all-accepted bracket (verify only) is tools/bench_qwen_text.py's tick_ms_all_accepted.
Frame-row bytes between host and device per tick are computed from shapes for the previous seam (tower rows to the host
and back, the whole cached frame_hidden to the host at every generate, the delta rows up again) and for this one (none).

    python tools/bench_qwen_realtime.py [--streams 128] [--ticks 24] [--warmup-ticks 40]

--audio-backend windowed times the windowed model instead (the reference's default backend): the 0.6B window tower
(left 1200, right 64 frames) and the 0.6B text decoder in bf16 with seeded weights.  Each tick, S streams each bring
2.0 s of PCM through the device mel (a tower engine used for its mel front end only); then one windowed tower call,
one adapter call (adapter_layers 0, a seeded out_dim -> d_model proj) and one generate_full_batch with the 9-token
template for every stream with cached steps (no rolling KV, no draft, penalty 1.0, n-gram 0).  Segment phases are
staggered so that cached steps spread over 0-200, with a rollover (trim to 0) past 200 as the reference's default
segment_max_steps.  Seeded weights never emit EOS, so each --max-new-tokens bracket (default 32 and 256) decodes
exactly that many steps.  In the same process, alternating with the engine call, the same generate also runs through
the Python driver loop (TextDecodeDriver.generate_full_batch over the engine's forward / pick), the loop that
wlk_qtext_generate_full moves into the engine; python_loop_streams_equal is the share of streams whose tokens the two
agree on, and python_loop_self_streams_equal the same share between two runs of the driver loop.  At these shapes the
bf16 GEMMs split K and the last split to arrive adds the others' partials to its own, so two runs of the same forward
can differ in the last bits and flip near-tied picks of the seeded weights (tests/test_gpu_qwen_window_realtime.py
checks exact equality of the two loops at test sizes).

    python tools/bench_qwen_realtime.py --audio-backend windowed [--streams 128] [--ticks 6] [--warmup-ticks 8]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from whisperlivekit_b200.qwen_dims import (QWEN_DIMS, QWEN_TEXT_DIMS, synthetic_adapter_state_dict,  # noqa: E402
                                           synthetic_text_state_dict, synthetic_tower_state_dict)
from whisperlivekit_b200.qwen_engine import QwenTowerEngine  # noqa: E402
from whisperlivekit_b200.qwen_plugin import B200QwenAudioCausalKVEncoder, B200QwenTextDecoder  # noqa: E402
from whisperlivekit_b200.qwen_realtime import RealtimeFrames  # noqa: E402
from whisperlivekit_b200.qwen_text_engine import QwenTextEngine  # noqa: E402

PLACEHOLDER, BOS, EOS = 151676, 151643, 151645
TEMPLATE = [151644, 872, 198, PLACEHOLDER, 151645, 198, 151644, 77091, 198]
SUPPRESS = [151669, 151670, PLACEHOLDER]
CHUNK_SAMPLES, CHUNK_SEC = 4000, 0.25


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:                                   # noqa: BLE001
        return f"unknown ({e})", "unknown"


def pct(xs, q):
    return round(float(np.percentile(np.asarray(xs) * 1e3, q)), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--audio-backend", default="causal", choices=["causal", "windowed"])
    ap.add_argument("--streams", type=int, default=128)
    ap.add_argument("--ticks", type=int, default=None, help="timed ticks (causal 24, windowed 6 per bracket)")
    ap.add_argument("--warmup-ticks", type=int, default=None,
                    help="ticks before timing: the cached segment grows (causal 40, windowed 8)")
    ap.add_argument("--max-new-tokens", type=int, nargs="+", default=None, help="causal 32; windowed brackets 32 256")
    ap.add_argument("--precision", default="bf16")
    a = ap.parse_args()
    if a.audio_backend == "windowed":
        return windowed(a)
    a.ticks = 24 if a.ticks is None else a.ticks
    a.warmup_ticks = 40 if a.warmup_ticks is None else a.warmup_ticks
    a.max_new_tokens = 32 if a.max_new_tokens is None else a.max_new_tokens[0]
    import torch
    S = a.streams
    name, power = gpu_info()
    td, xd = QWEN_DIMS["qwen3-asr-0.6b"], QWEN_TEXT_DIMS["qwen3-asr-0.6b"]
    tower = QwenTowerEngine(td, synthetic_tower_state_dict(td, 1), precision=a.precision, max_sessions=S, max_batch=S)
    tower.load_mel_filters()
    sd = dict(synthetic_text_state_dict(xd, 2), **synthetic_adapter_state_dict(td.out_dim, xd.d_model, seed=3))
    text = QwenTextEngine(xd, sd, precision=a.precision, max_sessions=S + 1, max_batch=S)   # + the full path's scratch
    encoder = B200QwenAudioCausalKVEncoder(tower, td)
    decoder = B200QwenTextDecoder(SimpleNamespace(wait_token_id=None, bos_token_id=BOS), text, xd)
    frames = RealtimeFrames(encoder, text, xd.d_model)
    adapt_t = []
    _adapt = text.adapt

    def timed_adapt(x, out=None):
        t = time.perf_counter()
        y = _adapt(x, out)
        adapt_t.append(time.perf_counter() - t)
        return y
    text.adapt = timed_adapt
    rng = np.random.default_rng(7)
    states = []
    for i in range(S):
        st = SimpleNamespace(audio=encoder.init_state(), adapter=SimpleNamespace(audio_frames_seen=0, decoder_steps_seen=0),
                             frame_hidden=None, decoder=None)
        tower.set_pending(st.audio.sid, rng.standard_normal(((i % 8) * 24, td.n_mels)).astype(np.float32) * 0.3)
        states.append(st)
    sids = [s.audio.sid for s in states]
    hyps = [[] for _ in range(S)]
    gen_kw = dict(template_token_ids=TEMPLATE, audio_placeholder_token_id=PLACEHOLDER, max_new_tokens=a.max_new_tokens,
                  eos_token_id=EOS, suppress_token_ids=SUPPRESS, repetition_penalty=1.15, no_repeat_ngram_size=3)
    byte_log = {"old": [], "new": []}

    def tick(timed, rejected):
        pcm = [rng.standard_normal(CHUNK_SAMPLES).astype(np.float32) * 0.1 for _ in range(S)]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        mels = tower.mel_append(sids, pcm)
        n_adapt = len(adapt_t)
        before = [0 if s.frame_hidden is None else int(s.frame_hidden.shape[1]) for s in states]
        out = frames.append(states, [torch.from_numpy(m)[None] for m in mels])
        t1 = time.perf_counter()
        t_adapt = sum(adapt_t[n_adapt:])
        drafts = [([SUPPRESS[0]] + h[1:]) if rejected and h else h for h in hyps]
        frame_rows = [s.frame_hidden[0] for s in states]
        toks, stats = decoder.generate_rolling_batch(frame_rows, states, drafts, **gen_kw)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        for i, t in enumerate(toks):
            hyps[i] = list(t)
        new_rows = [int(d.shape[1]) for _, d in out]
        cached = [int(s.frame_hidden.shape[1]) for s in states]
        old = sum(4 * (2 * n * td.out_dim + c * xd.d_model + n * xd.d_model) for n, c in zip(new_rows, cached))
        if timed:
            byte_log["old"].append(old)
            byte_log["new"].append(0)
        return t1 - t0 - t_adapt, t_adapt, t2 - t1, sum(new_rows), float(np.mean(before))

    for _ in range(a.warmup_ticks):
        tick(False, True)
    res_br = {}
    for br in ("prev_draft", "rejected"):
        rows = [tick(True, br == "rejected") for _ in range(a.ticks)]
        tw, ta, tt = [r[0] for r in rows], [r[1] for r in rows], [r[2] for r in rows]
        tot = [x + y + z for x, y, z in zip(tw, ta, tt)]
        res_br[br] = {"tick_ms_p50": pct(tot, 50), "tick_ms_p95": pct(tot, 95),
                      "tower_ms_p50": pct(tw, 50), "tower_ms_p95": pct(tw, 95),
                      "adapter_ms_p50": pct(ta, 50), "adapter_ms_p95": pct(ta, 95),
                      "text_ms_p50": pct(tt, 50), "text_ms_p95": pct(tt, 95),
                      "new_rows_per_tick_mean": round(float(np.mean([r[3] for r in rows])), 1),
                      "cached_steps_mean": round(float(np.mean([r[4] for r in rows])), 1),
                      "streams_per_gpu_rtf1": int(S * CHUNK_SEC * 1e3 / max(pct(tot, 50), 1e-9))}
    res = {"bench": "qwen_realtime", "gpu": name, "power_limit": power, "precision": a.precision, "streams": S,
           "chunk_sec": CHUNK_SEC, "max_new_tokens": a.max_new_tokens, "ticks": a.ticks, "warmup_ticks": a.warmup_ticks,
           "prev_draft": res_br["prev_draft"], "all_rejected": res_br["rejected"],
           "frame_row_bytes_per_tick_old_seam": int(np.mean(byte_log["old"])),
           "frame_row_bytes_per_tick_new_seam": int(np.mean(byte_log["new"])),
           "memory_text": text.memory(), "memory_tower": tower.memory()}
    print(json.dumps(res))


WINDOW_TICK_SEC, SEGMENT_MAX_STEPS = 2.0, 200                # asr.py:106, :110


def windowed(a):
    import torch
    from whisperlivekit_b200.qwen_dims import QWEN_WINDOW_DIMS, window_output_steps
    from whisperlivekit_b200.qwen_engine import QwenWindowEngine
    from whisperlivekit_b200.qwen_plugin import B200QwenAudioSurgeryEncoder
    from whisperlivekit_b200.qwen_text_engine import TextDecodeDriver
    ticks = 6 if a.ticks is None else a.ticks
    warm = 8 if a.warmup_ticks is None else a.warmup_ticks
    brackets = a.max_new_tokens or [32, 256]
    S = a.streams
    name, power = gpu_info()
    wd, xd = QWEN_WINDOW_DIMS["qwen3-asr-0.6b"], QWEN_TEXT_DIMS["qwen3-asr-0.6b"]
    mel = QwenTowerEngine(QWEN_DIMS["qwen3-asr-0.6b"], None, precision=a.precision, max_sessions=S, max_batch=S)
    mel.load_mel_filters()
    tower = QwenWindowEngine(wd, synthetic_tower_state_dict(wd, 1), precision=a.precision, max_sessions=S, max_batch=S)
    sd = dict(synthetic_text_state_dict(xd, 2), **synthetic_adapter_state_dict(wd.out_dim, xd.d_model, seed=3))
    text = QwenTextEngine(xd, sd, precision=a.precision, max_sessions=S, max_batch=S)
    encoder = B200QwenAudioSurgeryEncoder(tower, wd)
    decoder = B200QwenTextDecoder(SimpleNamespace(wait_token_id=None, bos_token_id=BOS), text, xd)
    frames = RealtimeFrames(encoder, text, xd.d_model)
    adapt_t = []
    _adapt = text.adapt

    def timed_adapt(x, out=None):
        t = time.perf_counter()
        y = _adapt(x, out)
        adapt_t.append(time.perf_counter() - t)
        return y
    text.adapt = timed_adapt
    rng = np.random.default_rng(7)
    head, tail = TEMPLATE[:TEMPLATE.index(PLACEHOLDER)], TEMPLATE[TEMPLATE.index(PLACEHOLDER) + 1:]
    states, mel_sids = [], []
    for i in range(S):
        st = SimpleNamespace(audio=encoder.init_state(), adapter=SimpleNamespace(audio_frames_seen=0, decoder_steps_seen=0),
                             frame_hidden=None, decoder=None)
        phase = (i * SEGMENT_MAX_STEPS) // S                         # staggered segments: cached steps spread over 0-200
        st.frame_hidden = torch.randn(1, phase, xd.d_model, device="cuda") * 0.3
        states.append(st)
        mel_sids.append(mel.open_session())
    samples = int(WINDOW_TICK_SEC * 16000)
    ctl_kw = dict(eos_token_id=EOS, suppress_token_ids=SUPPRESS, wait_token_id=None)

    def tick(max_new, timed):
        pcm = [rng.standard_normal(samples).astype(np.float32) * 0.1 for _ in range(S)]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        mels = mel.mel_append(mel_sids, pcm)
        n_adapt = len(adapt_t)
        frames.append(states, [torch.from_numpy(m)[None] for m in mels])
        t1 = time.perf_counter()
        t_adapt = sum(adapt_t[n_adapt:])
        live = [s for s in states if s.frame_hidden.shape[1]]
        rows = [s.frame_hidden[0] for s in live]
        prefixes = [head + [PLACEHOLDER] * int(r.shape[0]) + tail for r in rows]
        toks = decoder.generate_full_batch(rows, prefixes, audio_placeholder_token_id=PLACEHOLDER,
                                           max_new_tokens=max_new, **ctl_kw)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        cached = float(np.mean([int(s.frame_hidden.shape[1]) for s in states]))
        py, same, self_same = 0.0, 0.0, 0.0
        if timed:                                                    # the same generate through the Python driver loop
            srcs = [text.full_prefix(r, prefix_token_ids=p, audio_placeholder_token_id=PLACEHOLDER)[0]
                    for r, p in zip(rows, prefixes)]
            t3 = time.perf_counter()
            ref = TextDecodeDriver.generate_full_batch(text, decoder._scratch[:len(rows)], rows, srcs,
                                                       max_new_tokens=max_new, **ctl_kw)
            torch.cuda.synchronize()
            py = time.perf_counter() - t3
            same = sum(x == y for x, y in zip(ref, toks)) / max(len(toks), 1)
            ref2 = TextDecodeDriver.generate_full_batch(text, decoder._scratch[:len(rows)], rows, srcs,
                                                        max_new_tokens=max_new, **ctl_kw)
            self_same = sum(x == y for x, y in zip(ref, ref2)) / max(len(toks), 1)
        for s in states:                                             # the reference's rollover: a new segment
            if s.frame_hidden.shape[1] > SEGMENT_MAX_STEPS:
                s.frame_hidden = s.frame_hidden[:, 0:0]
        return t1 - t0 - t_adapt, t_adapt, t2 - t1, py, same, cached, [len(t) for t in toks], len(live), self_same

    for _ in range(warm):
        tick(brackets[0], False)
    res_br = {}
    for mx in brackets:
        tick(mx, False)                                              # the bracket's decode length warmed up
        rows = [tick(mx, True) for _ in range(ticks)]
        tw, ta, tt, tp = ([r[k] for r in rows] for k in range(4))
        tot = [x + y + z for x, y, z in zip(tw, ta, tt)]
        res_br[f"max_new_tokens_{mx}"] = {
            "tick_ms_p50": pct(tot, 50), "tick_ms_p95": pct(tot, 95),
            "tower_ms_p50": pct(tw, 50), "adapter_ms_p50": pct(ta, 50), "text_ms_p50": pct(tt, 50),
            "text_ms_p95": pct(tt, 95), "text_python_loop_ms_p50": pct(tp, 50), "text_python_loop_ms_p95": pct(tp, 95),
            "python_loop_streams_equal": round(float(np.mean([r[4] for r in rows])), 3),
            "python_loop_self_streams_equal": round(float(np.mean([r[8] for r in rows])), 3),
            "decode_steps": max(max(r[6]) for r in rows), "generating_streams_min": min(r[7] for r in rows),
            "cached_steps_mean": round(float(np.mean([r[5] for r in rows])), 1),
            "streams_per_gpu_rtf1": int(S * WINDOW_TICK_SEC * 1e3 / max(pct(tot, 50), 1e-9))}
    res = {"bench": "qwen_realtime_windowed", "gpu": name, "power_limit": power, "precision": a.precision,
           "streams": S, "tick_sec": WINDOW_TICK_SEC,
           "new_rows_per_stream_tick": window_output_steps(int(WINDOW_TICK_SEC * 100)),
           "window_frames": wd.window_frames, "ticks": ticks, "warmup_ticks": warm, **res_br,
           "memory_text": text.memory(), "memory_tower": tower.memory()}
    print(json.dumps(res))
    decoder.close()


if __name__ == "__main__":
    main()
