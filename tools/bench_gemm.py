#!/usr/bin/env python
"""Per-shape rates of the wgmma GEMM next to cuBLAS (torch.matmul, bf16 out), in one process.

    python tools/bench_gemm.py [--streams 48] [--shapes qkv,fc1,...] [--backend tcgen05|tcgen05_pair|tcgen05_1cta]
    python tools/bench_gemm.py --mnk M N K           (one custom shape, plain bf16 out)

Default shapes: the large-v3 encoder GEMMs of one tick at --streams streams (M = streams x 1500 rows, or x 3000 for
conv1), each with the epilogue the engine uses where `op_gemm` exposes it.  The cross-K/V GEMM runs with a plain bf16
output here (its head-major scatter is an engine-internal mode); the attention-out GEMM is timed as FC2's epilogue
twin (fp32 residual accumulated in place).  cuBLAS computes the same product without the epilogue.  TFLOP/s come from
the shapes (2 M N K per call) and CUDA events around many calls.  The card's name, power limit and maximum SM clock
are printed beside the figures (nvidia-smi, read-only query)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from whisperlivekit_b200.dims import DIMS  # noqa: E402
from whisperlivekit_b200.engine import WhisperEngine  # noqa: E402

D, NMEL = 1280, 128          # large-v3 width and mel bins
# name: (rows per stream, N, K, lda or None (dense), epilogue: "bias" | "gelu" | "residual" | "plain", layers per tick)
SHAPES = {
    "qkv": (1500, 3 * D, D, None, "bias", 32),
    "attn_out": (1500, D, D, None, "residual", 32),
    "fc1": (1500, 4 * D, D, None, "gelu", 32),
    "fc2": (1500, D, 4 * D, None, "residual", 32),
    "cross_kv": (1500, 32 * 2 * D, D, None, "plain", 1),
    "conv1": (3000, D, 3 * NMEL, NMEL, "gelu", 1),       # overlapping rows: row t reads mel frames t-1..t+1
    "conv2": (1500, D, 3 * D, 2 * D, "gelu", 1),         # stride 2 over conv1's rows
}
GELU_BITS = {"plain": 0, "bias": 0, "gelu": 1, "residual": 2}


def card_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.TimeoutExpired):
        out = []
    return {"gpu": out[0] if out else "unknown", "torch_name": torch.cuda.get_device_name(0)}


def operand_a(M, K, lda, g):
    """A as the engine sees it: dense [M, K], or an overlapping-row view of pitch lda over one buffer."""
    if lda is None:
        return torch.randn(M, K, device="cuda", generator=g).bfloat16(), K
    n = (M - 1) * lda + K
    buf = torch.randn(n, device="cuda", generator=g).bfloat16()
    return buf.as_strided((M, K), (lda, 1)), lda


def time_ms(fn, record, elapsed, iters, warmup=3):
    for _ in range(warmup):
        fn()
    record(0)
    for _ in range(iters):
        fn()
    record(1)
    return elapsed() / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=48)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--backend", default="tcgen05", choices=["tcgen05", "tcgen05_pair", "tcgen05_1cta"])
    ap.add_argument("--mnk", type=int, nargs=3, default=None)
    ap.add_argument("--window-ms", type=float, default=300.0, help="timed work per shape and side")
    ap.add_argument("--no-cublas", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_gemm.py measures on a GPU"

    eng = WhisperEngine(DIMS["micro"], None, [(0, 0)], precision="bf16", max_sessions=1, max_batch=1)
    g = torch.Generator(device="cuda").manual_seed(0)
    todo = {"custom": (args.mnk[0], args.mnk[1], args.mnk[2], None, "plain", 1)} if args.mnk else \
        {k: SHAPES[k] for k in args.shapes.split(",")}
    print(json.dumps({"card": card_info(), "backend": args.backend, "streams": args.streams}), flush=True)
    total = {"engine_ms": 0.0, "cublas_ms": 0.0, "tflop": 0.0}
    for name, (rows, N, K, lda, epi, layers) in todo.items():
        M = rows if name == "custom" else rows * args.streams
        A, lda_el = operand_a(M, K, lda, g)
        W = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
        b = torch.randn(N, device="cuda", generator=g) if epi != "plain" else None
        C = torch.zeros(M, N, device="cuda", dtype=torch.float32 if epi == "residual" else torch.bfloat16)
        c_code = 0 if epi == "residual" else 1
        flop = 2.0 * M * N * K

        def eng_call():
            eng.op_gemm(args.backend, A.data_ptr(), 1, lda_el, W.data_ptr(), 1, K, b.data_ptr() if b is not None else None,
                        C.data_ptr(), c_code, N, M, N, K, GELU_BITS[epi])

        # rough rate first, then a window of about --window-ms
        probe = time_ms(eng_call, eng.timer_record, lambda: eng.timer_elapsed_ms(0, 1), 2, warmup=1)
        iters = max(3, int(args.window_ms / max(probe, 1e-3)))
        ms = time_ms(eng_call, eng.timer_record, lambda: eng.timer_elapsed_ms(0, 1), iters)
        line = {"shape": name, "M": M, "N": N, "K": K, "lda": lda_el, "epilogue": epi, "iters": iters,
                "engine_ms": round(ms, 4), "engine_tflops": round(flop / ms / 1e9, 1)}
        if not args.no_cublas:
            eng.sync()
            Cb = C if C.dtype == torch.bfloat16 else None
            if Cb is None:
                del C
                torch.cuda.empty_cache()
                Cb = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
            Wt = W.t()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ms_cb = time_ms(lambda: torch.matmul(A, Wt, out=Cb), lambda i: ev[i].record(),
                            lambda: (torch.cuda.synchronize(), ev[0].elapsed_time(ev[1]))[1], iters)
            line.update(cublas_ms=round(ms_cb, 4), cublas_tflops=round(flop / ms_cb / 1e9, 1),
                        engine_over_cublas=round(ms_cb / ms, 3))
            total["cublas_ms"] += layers * ms_cb
            del Cb
        total["engine_ms"] += layers * ms
        total["tflop"] += layers * flop / 1e12
        print(json.dumps(line), flush=True)
        del A, W, b
        C = None
        torch.cuda.empty_cache()
    if len(todo) > 1:
        total = {k: round(v, 2) for k, v in total.items()}
        total["engine_tflops"] = round(total["tflop"] / total["engine_ms"] * 1e3, 1)
        print(json.dumps({"per_tick_layers_weighted": total}), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
