#!/usr/bin/env python
"""Generate tests/golden/large_v3_forced.npz by running the REAL reference on CPU at the true large-v3
geometry (the geometry bench.py times).  Needs the staged reference (oracle/_ref):

    python oracle/make_golden_large.py

Two streams (different audio), a 20-token prefill and 64 greedy steps each, driven the way
``AlignAttBase.infer`` drives its hooks (align_att_base.py:174-322): decoder with dict KV cache and
``return_cross_attn=True``, blank/EOT suppression on the first step, the AlignAtt suppression set on
every step, the DRY repetition penalty (``_apply_dry_penalty``, the reference's own method), argmax,
``_process_cross_attention`` over the last 16 iterations, most attended frame.
Stored per step: the token, the attended frame, the reference's top-2 logit gap (so a test can say where
token identity is *required* of a reduced-precision mode), the top-8 ids/values and a strided sample of
the logits.  Nothing from the reference is copied; only its outputs are recorded.
"""
from __future__ import annotations

import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.make_golden import build_reference_model, import_reference, pack   # noqa: E402

MODEL = "large-v3"
WEIGHT_SEED = 3
STREAMS = [(6.0, 31), (11.5, 32)]           # (audio seconds, audio seed)
N_STEPS = 64
PREFIX_EXTRA = [1169, 2068, 7586, 21831, 18045, 625, 262, 16931, 3290, 13, 314, 1101, 257, 1310, 517, 621]


def main():
    torch.manual_seed(0)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    import_reference()
    from whisperlivekit.simul_whisper.config import AlignAttConfig as RefCfg
    from whisperlivekit.simul_whisper.simul_whisper import AlignAtt
    from whisperlivekit.whisper.audio import N_FRAMES, N_SAMPLES, log_mel_spectrogram, pad_or_trim
    from whisperlivekit_b200.dims import ALIGNMENT_HEADS, DIMS, SpecialTokens
    from whisperlivekit_b200.weights import synthetic_audio, synthetic_state_dict

    dims = DIMS[MODEL]
    heads = ALIGNMENT_HEADS[MODEL]
    t0 = time.time()
    sd = synthetic_state_dict(dims, seed=WEIGHT_SEED)
    model = build_reference_model(dims, sd, heads)
    print(f"reference model built in {time.time() - t0:.1f}s")
    sp = SpecialTokens.for_dims(dims)
    cfg = RefCfg(tokenizer_is_multilingual=dims.is_multilingual, language="en", audio_min_len=0.0, audio_max_len=30.0,
                 decoder_type="greedy", beam_size=1, segment_length=0.5, frame_threshold=25)
    a = AlignAtt(cfg=cfg, loaded_model=model)
    suppress = sorted(set([a.tokenizer.transcribe, a.tokenizer.translate, a.tokenizer.sot, a.tokenizer.sot_prev,
                           a.tokenizer.sot_lm, a.tokenizer.no_timestamps, a.tokenizer.no_speech]
                          + list(a.tokenizer.all_language_tokens)))
    blank = list(a.tokenizer.encode(" ")) + [a.tokenizer.eot]
    prefix = list(sp.sot_sequence_including_notimestamps()) + PREFIX_EXTRA
    out = {"dims": np.asarray(dims.as_tuple(), np.int64), "weight_seed": np.int64(WEIGHT_SEED),
           "align_heads": np.asarray(heads, np.int64), "prefix": np.asarray(prefix, np.int64),
           "suppress_tokens": np.asarray(suppress, np.int64), "blank_tokens": np.asarray(blank, np.int64),
           "n_streams": np.int64(len(STREAMS)), "n_steps": np.int64(N_STEPS),
           "audio_seconds": np.asarray([s for s, _ in STREAMS], np.float64),
           "audio_seeds": np.asarray([s for _, s in STREAMS], np.int64)}

    with torch.no_grad():
        for si, (secs, aseed) in enumerate(STREAMS):
            audio = synthetic_audio(secs, seed=aseed)
            mel_padded = log_mel_spectrogram(torch.from_numpy(audio), n_mels=dims.n_mels, padding=N_SAMPLES,
                                             device="cpu").unsqueeze(0)
            mel = pad_or_trim(mel_padded, N_FRAMES)
            content = int((mel_padded.shape[2] - mel.shape[2]) / 2)
            t0 = time.time()
            enc = model.encoder(mel)
            print(f"stream {si}: encoder {time.time() - t0:.1f}s, content={content}")
            out[f"s{si}_content"] = np.int64(content)
            pack(f"s{si}_enc", enc[0], out)
            kv = {}
            tokens, frames, gaps, logprobs = [], [], [], []
            top_ids = np.zeros((N_STEPS, 8), np.int64)
            top_vals = np.zeros((N_STEPS, 8), np.float32)
            accumulated = []
            feed = torch.tensor([prefix])
            current = torch.tensor([prefix])
            for it in range(N_STEPS):
                logits, cross = model.decoder(feed, enc, kv_cache=kv, return_cross_attn=True)
                accumulated.append(cross)
                accumulated = accumulated[-16:]                      # align_att_base.py:222-224
                lg = logits[0, -1].float().clone()
                if it == 0:
                    pack(f"s{si}_logits_sot", logits[0, 0], out)
                    lg[blank] = -float("inf")                        # simul_whisper.py:379-381
                lg[suppress] = -float("inf")                         # simul_whisper.py:383-385
                lg = a._apply_dry_penalty(lg[None], current)[0]      # align_att_base.py:235 / :492-537
                if it in (0, 1, 31, N_STEPS - 1):
                    pack(f"s{si}_logits_step{it}", lg, out)
                v, ix = torch.topk(lg, 8)
                top_ids[it], top_vals[it] = ix.numpy(), v.numpy()
                tok = int(ix[0])
                gaps.append(float(v[0] - v[1]))
                logprobs.append(float(torch.log_softmax(lg, -1)[tok]))
                attn = a._process_cross_attention(accumulated, content)
                frames.append(int(attn[0, -1].argmax()))
                tokens.append(tok)
                feed = torch.tensor([[tok]])
                current = torch.cat([current, feed], dim=1)
            out[f"s{si}_tokens"] = np.asarray(tokens, np.int64)
            out[f"s{si}_frames"] = np.asarray(frames, np.int64)
            out[f"s{si}_gaps"] = np.asarray(gaps, np.float32)
            out[f"s{si}_logprobs"] = np.asarray(logprobs, np.float32)
            out[f"s{si}_top_ids"] = top_ids
            out[f"s{si}_top_vals"] = top_vals
            print(f"  distinct tokens={len(set(tokens))} tokens[:12]={tokens[:12]} frames[:8]={frames[:8]} min gap={min(gaps):.4f} "
                  f"median gap={float(np.median(gaps)):.3f}")
    path = os.path.join(ROOT, "tests", "golden", "large_v3_forced.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path) / 1024:.1f} KiB)")


if __name__ == "__main__":
    main()
