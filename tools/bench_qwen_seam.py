#!/usr/bin/env python
"""The qwen3-streaming seam under K concurrent sessions: K threads each drive the reference's
SegmentedCachedFullHypothesisStreamer over one installed B200QwenRealtimeModel at real-time pacing, for the causal and the
windowed backend, with the coalescing seam off and on.  Prints one JSON line (and each backend's part to stderr as it
completes).

Models: the reference's realtime models built at the 0.6B geometries with seeded weights, as tools/bench_qwen_realtime.py
seeds them (tower seed 1, text seed 2, adapter seed 3 with adapter_layers 0), on the CUDA engines in --precision.  The
streamer uses the fixture generators' settings (oracle/make_golden_qwen_realtime.py and _window_realtime.py: template,
suppress ids, segment sizes) with --max-new-tokens.  Each stream gets its own seeded mel frames; a chunk is 0.25 s
(25 frames) for the causal backend and 2.0 s (200 frames) for the windowed one, as in bench_qwen_realtime.py.  Stream i
starts i/K of a chunk late, and chunk k is handed to the streamer at start + k x chunk (or later, when the previous
call has not returned: the stream falls behind).

  batching off  the model as installed by default; the streamer calls run one at a time under one lock, since without
                the dispatcher the engines' shared output buffers admit one caller at a time
  batching on   install(batching=True, max_batch=K); every streamer call is one cohort iteration
                (begin_iter / end_iter, what plugin.install_qwen_cohorts does around process_iter)

Reported per backend and mode:
  tick_ms_p50 / p95       wall time of one append_mel_chunk (append + generate) as its caller sees it
  mean_cohort             sessions per engine call of the dispatcher (1.0 with batching off)
  rtf_p50 / rtf_max       per stream: busy time / audio time, where busy is the sum of its call times
  lag_s_max               how far the last chunk of a stream was handed over behind its real-time arrival
  streams_rtf_lt_1        streams with rtf < 1 and lag below one chunk
With --direct, tools/bench_qwen_realtime.py runs in a subprocess at the same stream count and its direct N-stream tick
figure (streams_per_gpu_rtf1) is printed beside the seam's.

    python tools/bench_qwen_seam.py [--threads 64] [--seconds 12] [--backend causal] [--direct]
"""
import argparse
import dataclasses
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CHUNK_SEC = {"causal": 0.25, "windowed": 2.0}


def build(backend, geometry):
    """(reference model, streamer factory): at the 0.6B geometries with seeded weights, or the fixture geometries."""
    import torch
    from oracle import stage_reference
    stage_reference.import_staged_reference()
    from whisperlivekit_b200.qwen_dims import (QWEN_DIMS, QWEN_TEXT_DIMS, QWEN_WINDOW_DIMS, synthetic_adapter_state_dict,
                                               synthetic_text_state_dict, synthetic_tower_state_dict)
    if backend == "causal":
        from oracle import make_golden_qwen_realtime as G
    else:
        from oracle import make_golden_qwen_window_realtime as G

    def streamer(model):
        s = G.build_streamer(model) if backend == "causal" else G.build_streamer(model, 0)
        return s
    if geometry == "fixture":
        return (G.build_model("qnano") if backend == "causal" else G.build_model()), streamer
    from qwen3_asr_causal.config import RealtimeAudioConfig
    from oracle.make_golden_qwen_realtime import BOS, WAIT, load_adapter
    from oracle.make_golden_qwen_text import build_reference
    xd = QWEN_TEXT_DIMS["qwen3-asr-0.6b"]
    text = build_reference(xd, synthetic_text_state_dict(xd, 2))
    if backend == "causal":
        from oracle.make_golden_qwen import GeometryTower
        from qwen3_asr_causal.causal import Qwen3ASRRealtimeQwenAudioCausalModel
        td = QWEN_DIMS["qwen3-asr-0.6b"]
        cfg = RealtimeAudioConfig(d_model=xd.d_model, qwen_audio_block_bidirectional=td.block_bidirectional,
                                  qwen_audio_block_frames=td.block_frames,
                                  qwen_audio_left_context_sec=td.left_context_steps * 0.08,
                                  qwen_audio_mutable_tail_sec=td.mutable_tail_steps * 0.08, qwen_audio_adapter_layers=0)
        model = Qwen3ASRRealtimeQwenAudioCausalModel(
            cfg, qwen_model_id="seeded", audio_tower=GeometryTower(td, synthetic_tower_state_dict(td, 1)).eval(),
            text_model=text.text_model, lm_head=text.lm_head, bos_token_id=BOS, wait_token_id=WAIT,
            audio_output_dim=td.out_dim).eval()
        out_dim = td.out_dim
    else:
        from oracle.make_golden_qwen_window import stock_tower
        from qwen3_asr_causal.model import Qwen3ASRRealtimeQwenAudioSurgeryModel
        wd = QWEN_WINDOW_DIMS["qwen3-asr-0.6b"]
        cfg = RealtimeAudioConfig(d_model=xd.d_model, n_mels=wd.n_mels,
                                  qwen_audio_left_context_sec=wd.left_context_frames / 100.0,
                                  qwen_audio_right_context_ms=wd.right_context_frames * 10, qwen_audio_adapter_layers=0)
        model = Qwen3ASRRealtimeQwenAudioSurgeryModel(
            cfg, qwen_model_id="seeded", audio_tower=stock_tower(wd, synthetic_tower_state_dict(wd, 1), "wlk_varlen"),
            text_model=text.text_model, lm_head=text.lm_head, bos_token_id=BOS, wait_token_id=WAIT,
            audio_output_dim=wd.out_dim).eval()
        out_dim = wd.out_dim
    with torch.no_grad():
        load_adapter(model.adapter, synthetic_adapter_state_dict(out_dim, xd.d_model, seed=3))
    return model, streamer


def run(backend, batching, a):
    import torch
    from oracle.make_golden_qwen import mel_stream
    from whisperlivekit_b200.qwen_plugin import B200QwenRealtimeModel
    K, chunk_sec = a.threads, CHUNK_SEC[backend]
    model, make_streamer = build(backend, a.geometry)
    kw = dict(precision=a.precision, max_ctx=a.max_ctx, max_sessions=3 * K + 8, max_batch=K)
    if a.cpu_oracles:                              # the plumbing on the CPU oracles (no timing meaning)
        from test_oracle_qwen_realtime import oracle_factories as causal_factories
        from test_oracle_qwen_window_realtime import oracle_factories as window_factories
        tower, text, _ = (causal_factories if backend == "causal" else window_factories)()
        kw = dict(tower_factory=tower, text_factory=text)
    rt = B200QwenRealtimeModel.install(model, batching=batching, attention_blocks=True if backend == "windowed" else None,
                                       **kw)
    streamers = []
    for _ in range(K):
        s = make_streamer(model)
        s.config = dataclasses.replace(s.config, max_new_tokens=a.max_new_tokens)
        streamers.append(s)
    frames = int(round(chunk_sec * 100))
    n_chunks = max(1, int(a.seconds / chunk_sec))
    mels = [mel_stream(n_chunks * frames, 128, seed=100 + i) for i in range(K)]
    lock = threading.Lock()
    calls, lag, err = [[] for _ in range(K)], [0.0] * K, [None] * K

    def one(fn):
        if batching:
            rt.batcher.begin_iter()
            try:
                return fn()
            finally:
                rt.batcher.end_iter()
        with lock:
            return fn()

    t0 = time.perf_counter() + 0.5

    def stream(i):
        try:
            s = streamers[i]
            with torch.no_grad():
                for k in range(n_chunks):
                    due = t0 + (i / K + k + 1) * chunk_sec            # the chunk's audio has arrived
                    now = time.perf_counter()
                    if now < due:
                        time.sleep(due - now)
                    start = time.perf_counter()
                    lag[i] = start - due
                    m = torch.from_numpy(mels[i][k * frames: (k + 1) * frames])[None]
                    one(lambda: s.append_mel_chunk(m))
                    calls[i].append(time.perf_counter() - start)
        except BaseException as e:                                   # noqa: BLE001
            err[i] = repr(e)

    ts = [threading.Thread(target=stream, args=(i,)) for i in range(K)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if any(err):
        raise RuntimeError(f"{sum(e is not None for e in err)} streams failed, first: {next(e for e in err if e)}")
    flat = np.asarray([c for cs in calls for c in cs]) * 1e3
    rtf = np.asarray([sum(cs) / (n_chunks * chunk_sec) for cs in calls])
    st = rt.batcher.stats if batching else None
    res = {"tick_ms_p50": round(float(np.percentile(flat, 50)), 2), "tick_ms_p95": round(float(np.percentile(flat, 95)), 2),
           "mean_cohort": round(st["sessions"] / max(st["calls"], 1), 2) if st else 1.0,
           "engine_calls": st["calls"] if st else None, "caller_calls": st["requests"] if st else None,
           "rtf_p50": round(float(np.median(rtf)), 3), "rtf_max": round(float(rtf.max()), 3),
           "lag_s_max": round(max(lag), 3),
           "streams_rtf_lt_1": int(sum(r < 1 and g < chunk_sec for r, g in zip(rtf, lag)))}
    rt.close()
    rt.decoder.close()
    return res


def direct(backend, a):
    """tools/bench_qwen_realtime.py's direct N-stream tick at the same stream count."""
    cmd = [sys.executable, os.path.join(ROOT, "tools", "bench_qwen_realtime.py"), "--streams", str(a.threads),
           "--precision", a.precision, "--max-new-tokens", str(a.max_new_tokens), "--ticks", "4", "--warmup-ticks", "4"]
    if backend == "windowed":
        cmd += ["--audio-backend", "windowed"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=3600)
    try:
        r = json.loads(out.stdout.strip().splitlines()[-1])
    except Exception:                                                # noqa: BLE001
        return {"error": (out.stderr or out.stdout)[-400:]}
    br = r.get("prev_draft") or r.get(f"max_new_tokens_{a.max_new_tokens}") or {}
    return {"tick_ms_p50": br.get("tick_ms_p50"), "streams_per_gpu_rtf1": br.get("streams_per_gpu_rtf1")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--threads", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=12.0, help="audio per stream")
    ap.add_argument("--backend", nargs="+", default=["causal"], choices=["causal", "windowed"],
                    help="windowed at --geometry 0.6b stops in the fixture helper's positional-table check of the stock "
                         "tower (oracle/make_golden_qwen_window.py); it runs at --geometry fixture")
    ap.add_argument("--batching", nargs="+", default=["off", "on"], choices=["off", "on"])
    ap.add_argument("--precision", default="bf16")
    ap.add_argument("--max-new-tokens", type=int, default=32)
    ap.add_argument("--max-ctx", type=int, default=1024)
    ap.add_argument("--geometry", default="0.6b", choices=["0.6b", "fixture"])
    ap.add_argument("--cpu-oracles", action="store_true", help="run the plumbing on the CPU oracles (no timing meaning)")
    ap.add_argument("--direct", action="store_true", help="also run bench_qwen_realtime.py at the same stream count")
    a = ap.parse_args()
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from bench_qwen_realtime import gpu_info  # noqa: E402
    name, power = gpu_info() if not a.cpu_oracles else ("cpu oracles", "n/a")
    res = {"bench": "qwen_seam", "gpu": name, "power_limit": power, "precision": a.precision, "threads": a.threads,
           "seconds": a.seconds, "max_new_tokens": a.max_new_tokens, "geometry": a.geometry}
    for be in a.backend:
        r = {"chunk_sec": CHUNK_SEC[be]}
        for mode in a.batching:
            r[f"batching_{mode}"] = run(be, mode == "on", a)
        if a.direct and not a.cpu_oracles:
            r["direct_tick"] = direct(be, a)
        res[be] = r
        print(json.dumps({be: r}), file=sys.stderr, flush=True)         # progress: one backend at a time
    print(json.dumps(res))


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    main()
