#!/usr/bin/env python
"""Generate tests/golden/*.npz by running the REAL reference on CPU.

Needs the staged reference (oracle/_ref, see oracle/stage_reference.py):

    python oracle/make_golden.py

For each case it (1) builds seeded weights (whisperlivekit_b200.weights), loads
them into the reference's own ``whisperlivekit.whisper.model.Whisper``, (2) runs
the reference's ``log_mel_spectrogram`` / encoder / decoder / ``AlignAtt.infer``
on seeded audio, and (3) stores compact fixtures: strided samples of the float
tensors (full tensors would be MBs) and the complete integer traces
(tokens, attended frames).  Nothing from the reference is copied; only its
outputs are recorded.  The fixtures pin oracle/whisper_oracle.py (CPU tests) and
the CUDA engine (GPU tests).
"""
from __future__ import annotations

import hashlib
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")   # the staged reference (oracle/stage_reference.py)


def import_reference():
    if "soundfile" not in sys.modules:                      # only OpenaiApiASR needs it
        m = types.ModuleType("soundfile")
        m.__spec__ = __import__("importlib.machinery").machinery.ModuleSpec("soundfile", loader=None)   # find_spec() must not choke on the stub
        m.read = m.write = m.info = lambda *a, **k: (_ for _ in ()).throw(RuntimeError("stub"))
        sys.modules["soundfile"] = m
    if REF not in sys.path:
        sys.path.insert(0, REF)
    import whisperlivekit  # noqa: F401
    return whisperlivekit


def build_reference_model(dims, sd, align_heads):
    from whisperlivekit.whisper.model import ModelDimensions as RefDims, Whisper
    m = Whisper(RefDims(*dims.as_tuple())).eval()
    tsd = {k: torch.from_numpy(v) for k, v in sd.items()}
    missing, unexpected = m.load_state_dict(tsd, strict=False)
    assert not unexpected, unexpected
    assert all("mask" in k or "alignment_heads" in k for k in missing), missing
    mask = torch.zeros(dims.n_text_layer, dims.n_text_head, dtype=torch.bool)
    for l, h in align_heads:
        mask[l, h] = True
    m.register_buffer("alignment_heads", mask.to_sparse(), persistent=False)
    return m


def sample_idx(n, k=257):
    """Deterministic strided sample of a flattened tensor."""
    step = max(1, n // k)
    return np.arange(0, n, step, dtype=np.int64)


def pack(name, t, out):
    a = t.detach().cpu().float().numpy() if isinstance(t, torch.Tensor) else np.asarray(t, np.float32)
    flat = a.reshape(-1)
    idx = sample_idx(flat.shape[0])
    out[name + "__shape"] = np.asarray(a.shape, np.int64)
    out[name + "__idx"] = idx
    out[name + "__val"] = flat[idx].astype(np.float32)
    out[name + "__absmax"] = np.float32(np.abs(flat).max())
    out[name + "__sum"] = np.float64(flat.astype(np.float64).sum())


CASES = {
    # name: (dims key, weight seed, audio seconds, audio seed, align heads)
    "micro":   ("micro", 11, 7.3, 21, [(0, 1), (1, 0), (1, 1)]),
    "microml": ("micro-ml", 12, 4.1, 22, [(1, 0), (1, 1)]),
    "tiny":    ("tiny", 13, 9.0, 23, None),
}

FORCED_TOKENS = [1169, 2068, 7586, 21831, 18045, 625, 262, 16931, 3290, 13, 314, 1101]


def run_case(name, spec, wlk):
    from whisperlivekit.whisper.audio import log_mel_spectrogram, pad_or_trim, N_FRAMES, N_SAMPLES
    from whisperlivekit.simul_whisper.config import AlignAttConfig as RefCfg
    from whisperlivekit.simul_whisper.simul_whisper import AlignAtt
    from whisperlivekit_b200.dims import DIMS, ALIGNMENT_HEADS, SpecialTokens
    from whisperlivekit_b200.weights import synthetic_state_dict, synthetic_audio

    dkey, wseed, secs, aseed, heads = spec
    dims = DIMS[dkey]
    heads = heads or ALIGNMENT_HEADS[dkey]
    sd = synthetic_state_dict(dims, seed=wseed)
    model = build_reference_model(dims, sd, heads)
    audio = synthetic_audio(secs, seed=aseed)
    sp = SpecialTokens.for_dims(dims)
    out = {"dims": np.asarray(dims.as_tuple(), np.int64), "weight_seed": np.int64(wseed),
           "audio_seconds": np.float64(secs), "audio_seed": np.int64(aseed),
           "align_heads": np.asarray(heads, np.int64),
           "audio_sha256": np.frombuffer(hashlib.sha256(audio.tobytes()).digest(), np.uint8)}

    with torch.no_grad():
        # ---- a1 mel + a2 encoder (reference simul_whisper.py:345-351)
        mel_padded = log_mel_spectrogram(torch.from_numpy(audio), n_mels=dims.n_mels,
                                         padding=N_SAMPLES, device="cpu").unsqueeze(0)
        mel = pad_or_trim(mel_padded, N_FRAMES)
        content = int((mel_padded.shape[2] - mel.shape[2]) / 2)
        out["content_mel_len"] = np.int64(content)
        pack("mel", mel[0], out)
        enc = model.encoder(mel)
        pack("enc", enc[0], out)

        # ---- a4 decoder: prefill + forced single-token steps with the dict KV cache
        prefix = list(sp.sot_sequence_including_notimestamps()) + FORCED_TOKENS[:5]
        kv = {}
        logits, cross = model.decoder(torch.tensor([prefix]), enc, kv_cache=kv, return_cross_attn=True)
        pack("logits_prefill_last", logits[0, -1], out)
        pack("logits_prefill_sot", logits[0, 0], out)
        out["argmax_prefill"] = np.asarray(logits[0].argmax(-1).numpy(), np.int64)
        accumulated = [cross]
        step_argmax = []
        for i, tkn in enumerate(FORCED_TOKENS[5:10]):
            logits, cross = model.decoder(torch.tensor([[tkn]]), enc, kv_cache=kv, return_cross_attn=True)
            accumulated.append(cross)
            step_argmax.append(int(logits[0, -1].argmax()))
            if i in (0, 4):
                pack(f"logits_step{i}", logits[0, -1], out)
        out["argmax_steps"] = np.asarray(step_argmax, np.int64)
        out["forced_prefix"] = np.asarray(prefix, np.int64)
        out["forced_steps"] = np.asarray(FORCED_TOKENS[5:10], np.int64)

        # ---- a7 alignment post-processing through the reference's own hook
        cfg = RefCfg(tokenizer_is_multilingual=dims.is_multilingual, language="en", audio_min_len=0.0,
                     audio_max_len=30.0, decoder_type="greedy", beam_size=1, segment_length=0.5,
                     frame_threshold=25)
        a = AlignAtt(cfg=cfg, loaded_model=model)
        attn = a._process_cross_attention(accumulated, content)
        pack("align_attn", attn[0], out)
        out["align_argmax_rows"] = attn[0].argmax(-1).numpy().astype(np.int64)
        out["blank_token"] = np.asarray(a.tokenizer.encode(" "), np.int64)
        out["suppress_tokens"] = np.asarray(sorted(set(
            [a.tokenizer.transcribe, a.tokenizer.translate, a.tokenizer.sot, a.tokenizer.sot_prev,
             a.tokenizer.sot_lm, a.tokenizer.no_timestamps, a.tokenizer.no_speech]
            + list(a.tokenizer.all_language_tokens))), np.int64)
        out["initial_tokens"] = a.state.initial_tokens[0].numpy().astype(np.int64)

        # ---- streaming policy: the reference's AlignAtt.infer over 0.5 s chunks.
        # nonspeech_prob=1.01 keeps the no-speech exit from hiding the decode loop on
        # random weights (SURVEY.md §8c); a second run keeps the default 0.5.
        for tag, nsp in (("pol", 1.01), ("poldef", 0.5)):
            cfg = RefCfg(tokenizer_is_multilingual=dims.is_multilingual, language="en", audio_min_len=0.0,
                         audio_max_len=30.0, decoder_type="greedy", beam_size=1, segment_length=0.5,
                         frame_threshold=25, nonspeech_prob=nsp)
            a = AlignAtt(cfg=cfg, loaded_model=model)
            frames_log, toks_log = [], []
            orig_frames = a._get_attended_frames
            orig_update = a._update_tokens

            def spy_frames(attn, _o=orig_frames, _l=frames_log):
                r = _o(attn); _l.append(r[1]); return r

            def spy_update(ct, lg, sl, _o=orig_update, _l=toks_log):
                r = _o(ct, lg, sl); _l.append(int(r[0][0, -1])); return r

            a._get_attended_frames = spy_frames
            a._update_tokens = spy_update
            new_tokens, step_tokens, step_frames, offs_t, offs_s = [], [], [], [0], [0]
            n_chunks = int(np.ceil(len(audio) / 8000))
            for c in range(n_chunks):
                a.insert_audio(torch.from_numpy(audio[c * 8000:(c + 1) * 8000]))
                frames_log.clear(); toks_log.clear()
                n_before = len(a.state.tokens)
                a.infer(is_last=(c == n_chunks - 1))
                hyp = a.state.tokens[-1][0].tolist() if len(a.state.tokens) > n_before else []
                new_tokens += hyp; offs_t.append(len(new_tokens))
                step_tokens += list(toks_log); step_frames += list(frames_log); offs_s.append(len(step_tokens))
            out[f"{tag}_new_tokens"] = np.asarray(new_tokens, np.int64)
            out[f"{tag}_new_tokens_offsets"] = np.asarray(offs_t, np.int64)
            out[f"{tag}_step_tokens"] = np.asarray(step_tokens, np.int64)
            out[f"{tag}_step_frames"] = np.asarray(step_frames, np.int64)
            out[f"{tag}_step_offsets"] = np.asarray(offs_s, np.int64)
            print(f"  [{name}/{tag}] chunks={n_chunks} steps={len(step_tokens)} kept_tokens={len(new_tokens)}")
    return out


def filters_fixture():
    """Pin the recomputed mel filterbank against the reference asset."""
    from whisperlivekit.whisper.audio import mel_filters
    from whisperlivekit_b200.weights import mel_filterbank
    out = {}
    for n in (80, 128):
        ref = mel_filters("cpu", n).numpy()
        mine = mel_filterbank(n)
        d = float(np.abs(ref - mine).max())
        print(f"  mel_filterbank({n}): max|ref-mine| = {d:.3e}, nonzero mismatch = "
              f"{int(((ref != 0) != (mine != 0)).sum())}")
        out[f"max_abs_diff_{n}"] = np.float64(d)
        out[f"ref_sha256_{n}"] = np.frombuffer(hashlib.sha256(ref.tobytes()).digest(), np.uint8)
        idx = sample_idx(ref.size, 1024)
        out[f"idx_{n}"] = idx
        out[f"val_{n}"] = ref.reshape(-1)[idx]
        out[f"rowsum_{n}"] = ref.sum(1)
    return out


def timing_fixture():
    """Reference median_filter (torch CPU path) and dtw_cpu (numba) on seeded attention-like matrices."""
    from whisperlivekit.whisper.timing import dtw_cpu, median_filter
    rng = np.random.default_rng(7)
    out = {}
    for idx, (n, m) in enumerate([(5, 40), (23, 310), (61, 750), (1, 12), (9, 9)]):
        a = rng.random((n, m)).astype(np.float32)
        a = a / a.sum(-1, keepdims=True)
        a[np.arange(n), np.minimum(m - 1, (np.arange(n) * m) // max(n, 1))] += 0.5      # a noisy diagonal ridge
        z = (a - a.mean(0, keepdims=True)) / (a.std(0, keepdims=True) + 1e-8)
        med = median_filter(torch.from_numpy(z), 7).numpy()
        ti, fi = dtw_cpu((-med).astype(np.float64))
        out[f"x{idx}"] = z.astype(np.float32)
        out[f"med{idx}"] = med.astype(np.float32)
        out[f"text{idx}"] = np.asarray(ti, np.int64)
        out[f"time{idx}"] = np.asarray(fi, np.int64)
    # ties: quantised costs make equal-cost moves frequent, pinning the move preference
    q = np.round(rng.random((17, 90)) * 4).astype(np.float32) / 4
    ti, fi = dtw_cpu(q.astype(np.float64))
    out["xq"], out["textq"], out["timeq"] = q, np.asarray(ti, np.int64), np.asarray(fi, np.int64)
    out["n_cases"] = np.int64(5)
    return out


def main():
    torch.manual_seed(0)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    wlk = import_reference()
    gdir = os.path.join(ROOT, "tests", "golden")
    os.makedirs(gdir, exist_ok=True)
    np.savez_compressed(os.path.join(gdir, "mel_filters.npz"), **filters_fixture())
    np.savez_compressed(os.path.join(gdir, "timing.npz"), **timing_fixture())
    only = sys.argv[1:]
    for name, spec in CASES.items():
        if only and name not in only:
            continue
        print(f"case {name}")
        out = run_case(name, spec, wlk)
        path = os.path.join(gdir, f"{name}.npz")
        np.savez_compressed(path, **out)
        print(f"  wrote {path} ({os.path.getsize(path) / 1024:.1f} KiB)")


if __name__ == "__main__":
    main()
