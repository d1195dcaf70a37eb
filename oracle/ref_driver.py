"""Drive the STAGED, unmodified reference (oracle/_ref, see oracle/stage_reference.py) through the same per-chunk
workload bench.py times on the H100 engine, on the host cores: the reference arm (`bench.py --impl reference`)
and the `cpu_baseline` leg.  Benchmark infrastructure only -- nothing in whisperlivekit_b200/ imports this.

What is timed is the reference's own code: ``AlignAtt.insert_audio`` (rolling 30 s window, simul_whisper.py:219-237),
``AlignAtt._encode`` (log_mel_spectrogram + vendored torch ``AudioEncoder``, :299-352),
``_get_logits_and_cross_attn`` (``TextDecoder`` with its dict KV cache, :357-368), ``_check_no_speech``,
``_suppress_blank_tokens`` / ``_apply_token_suppression``, ``_update_tokens`` (GreedyDecoder), ``_process_cross_attention``
and ``_get_attended_frames`` -- called in the order ``AlignAttBase.infer`` calls them (align_att_base.py:174-322), with
the step count scripted (PREFIX-token prefill + STEPS single-token iterations) so that both arms do identical work:
on seeded random weights the policy's own stop rules would end most iterations after one or two tokens.
"""
from __future__ import annotations

import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

CHUNK = 8000


def host_cores() -> int:
    try:
        return len(os.sched_getaffinity(0))
    except Exception:
        return os.cpu_count() or 1


def default_threads() -> int:
    """The intra-op thread count torch picks on this box when nothing overrides it (OMP_NUM_THREADS unset) -- what the
    reference runs with by default; torchrun exports OMP_NUM_THREADS=1, which this ignores on purpose.  Bounded by the
    cgroup CPU quota when there is one."""
    import subprocess
    env = {k: v for k, v in os.environ.items() if k not in ("OMP_NUM_THREADS", "MKL_NUM_THREADS")}
    n = host_cores()
    try:
        out = subprocess.run([sys.executable, "-c", "import torch; print(torch.get_num_threads())"], env=env,
                             capture_output=True, text=True, timeout=120).stdout.strip().splitlines()
        n = int(out[-1])
    except Exception:
        pass
    q = cpu_quota()
    if q:
        n = max(1, min(n, int(q)))
    return n


def cpu_quota():
    """cgroup v2 cpu.max as a number of CPUs, or None when unlimited / unreadable."""
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()
        return None if quota == "max" else float(quota) / float(period)
    except Exception:
        return None


def cpu_model() -> str:
    try:
        for line in open("/proc/cpuinfo"):
            if line.startswith("model name"):
                return line.split(":", 1)[1].strip()
    except Exception:
        pass
    return "unknown"


def build_model(dims, sd, heads):
    """Seeded weights -> the reference's own ``Whisper`` module (fp32, CPU)."""
    import torch
    from oracle.stage_reference import import_staged_reference
    import_staged_reference()
    from whisperlivekit.whisper.model import ModelDimensions as RefDims, Whisper
    # The random initialisation of 1.5 G parameters (a minute of single-thread work at large-v3) would be overwritten by
    # load_state_dict anyway: torch.nn.init's samplers are no-ops while the module is constructed.
    import torch.nn.init as init
    saved = {k: getattr(init, k) for k in ("kaiming_uniform_", "uniform_", "normal_", "trunc_normal_")}
    try:
        for k in saved:
            setattr(init, k, lambda t, *a, **kw: t)
        m = Whisper(RefDims(*dims.as_tuple())).eval()
    finally:
        for k, f in saved.items():
            setattr(init, k, f)
    tsd = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sd.items()}
    missing, unexpected = m.load_state_dict(tsd, strict=False)
    assert not unexpected, unexpected
    assert all("mask" in k or "alignment_heads" in k for k in missing), missing
    mask = torch.zeros(dims.n_text_layer, dims.n_text_head, dtype=torch.bool)
    for l, h in heads:
        mask[l, h] = True
    m.register_buffer("alignment_heads", mask.to_sparse(), persistent=False)
    return m


class RefStream:
    """One stream of the reference's AlignAtt over a full 30 s window."""

    def __init__(self, model, dims, prefix_len: int, steps: int, seed: int = 1):
        import logging
        import torch
        from whisperlivekit.simul_whisper.config import AlignAttConfig
        from whisperlivekit.simul_whisper.simul_whisper import AlignAtt
        from whisperlivekit_b200.weights import synthetic_audio
        logging.getLogger("whisperlivekit").setLevel(logging.ERROR)
        cfg = AlignAttConfig(tokenizer_is_multilingual=dims.is_multilingual, language="en", audio_min_len=0.0,
                             audio_max_len=30.0, decoder_type="greedy", beam_size=1, segment_length=0.5,
                             frame_threshold=25)
        self.torch = torch
        self.a = AlignAtt(cfg=cfg, loaded_model=model)
        self.a.device = "cpu"             # AlignAtt picks 'cuda' whenever a GPU is visible (simul_whisper.py:134); this arm
        self.steps = steps                # times the reference's CPU backend: the model and every tensor stay on the host
        audio = synthetic_audio(30.0, seed=seed)
        for c in range(0, len(audio), CHUNK):                       # 60 segments of 0.5 s: the window is full
            self.a.insert_audio(torch.from_numpy(audio[c:c + CHUNK]))
        init = self.a.state.initial_tokens[0].tolist()
        self.prefix = torch.tensor([init + list(range(1000, 1000 + prefix_len - len(init)))], dtype=torch.long)
        self.rng = np.random.default_rng(100 + seed)

    @property
    def n_window(self) -> int:
        return int(sum(s.shape[0] for s in self.a.state.segments))

    def chunk(self):
        """One 0.5 s tick of this stream.  -> (last token, last attended frame)"""
        torch, a = self.torch, self.a
        with torch.no_grad():
            a.insert_audio(torch.from_numpy((0.05 * self.rng.standard_normal(CHUNK)).astype(np.float32)))
            enc, content = a._encode(a._concat_segments())
            tokens = self.prefix
            accumulated = []
            sum_logprobs = a._init_sum_logprobs()
            new_segment = True
            frame = -1
            for it in range(self.steps + 1):                        # prefill iteration + `steps` single-token ones
                feed = tokens if new_segment else tokens[:, -1:]
                logits, cross = a._get_logits_and_cross_attn(feed, enc)
                accumulated.append(cross)
                accumulated = accumulated[-16:]
                if new_segment:
                    a._check_no_speech(logits)                       # computed; the scripted workload does not stop on it
                if it == self.steps:
                    break                                            # the H100 arm's last call is a decode as well
                logits = logits[:, -1, :]
                if new_segment:
                    logits = a._suppress_blank_tokens(logits)
                new_segment = False
                logits = a._apply_token_suppression(logits)
                tokens, _ = a._update_tokens(tokens, logits, sum_logprobs)
                attn = a._process_cross_attention(accumulated, content)
                _, frame = a._get_attended_frames(attn)
            a._clean_cache()
        return int(tokens[0, -1]), int(frame)


def time_single_stream(model, dims, prefix_len, steps, n_chunks, threads, warmup=0):
    """Seconds per stream-chunk with one stream using `threads` host threads."""
    import torch
    torch.set_num_threads(int(threads))                              # also overrides torchrun's OMP_NUM_THREADS=1
    st = RefStream(model, dims, prefix_len, steps, seed=1)
    assert st.n_window == 480000, st.n_window
    for _ in range(warmup):
        st.chunk()
    per = []
    for _ in range(n_chunks):
        t0 = time.perf_counter()
        st.chunk()
        per.append(time.perf_counter() - t0)
    return per, torch.get_num_threads()


def time_parallel_single_thread(model, dims, prefix_len, steps, procs, timeout_s=300.0):
    """`procs` single-thread streams in parallel (BASELINE.md section 3, figure ii): fork one process per stream (the
    model's weights are shared copy-on-write), each runs ONE stream-chunk; returns (wall seconds, finished).
    Must be called before this process has run any multi-threaded torch op (OpenMP pools do not survive fork)."""
    import select
    import torch
    torch.set_num_threads(1)
    r, w = os.pipe()              # children -> parent: b"r" ready, b"1" chunk done, b"0" failed
    gr, gw = os.pipe()            # parent -> children: the start signal (one byte each)
    pids = []
    for i in range(procs):
        pid = os.fork()
        if pid == 0:
            ok = b"0"
            try:
                os.close(r); os.close(gw)
                torch.set_num_threads(1)
                st = RefStream(model, dims, prefix_len, steps, seed=10 + i)
                os.write(w, b"r")
                os.read(gr, 1)
                st.chunk()
                ok = b"1"
            finally:
                try:
                    os.write(w, ok)
                finally:
                    os._exit(0)
        pids.append(pid)
    os.close(w); os.close(gr)

    def collect(token, deadline):
        n = 0
        while n < procs:
            left = deadline - time.perf_counter()
            if left <= 0:
                break
            rl, _, _ = select.select([r], [], [], left)
            if not rl:
                break
            data = os.read(r, 4096)
            if not data:
                break
            n += data.count(token)
            if token == b"r" and data.count(b"0"):
                break
        return n

    ready = collect(b"r", time.perf_counter() + 120.0)
    done, wall = 0, 0.0
    if ready == procs:
        t0 = time.perf_counter()
        os.write(gw, b"g" * procs)
        done = collect(b"1", t0 + timeout_s)
        wall = time.perf_counter() - t0
    for pid in pids:
        if done < procs:
            try:
                os.kill(pid, 9)
            except ProcessLookupError:
                pass
        try:
            os.waitpid(pid, 0)
        except ChildProcessError:
            pass
    os.close(r); os.close(gw)
    return wall, done
