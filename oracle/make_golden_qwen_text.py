#!/usr/bin/env python
"""Build container only: golden fixtures for the Qwen3-ASR text decoder, produced by the REFERENCE itself.

The reference's Qwen3ASRRealtimeQwenDecoderModel (third_party/qwen3-asr-causal/src/qwen3_asr_causal/model.py; the
causal model inherits both generate methods from it) is given a transformers ``Qwen3Model`` and an ``lm_head`` filled with
whisperlivekit_b200.qwen_dims.synthetic_text_state_dict and driven, unchanged, through generate_full_hypothesis_rolling
over a chunk schedule (rebuild, growing audio, a zero-delta chunk, a template change, the previous hypothesis as the
draft, a corrupted draft, a draft ending in EOS, a draft longer than max_new_tokens, controls on and off, the
max-consecutive rule) and through generate_full_hypothesis_from_cached_audio.  Tokens, stats and strided samples of
every lm_head output (a forward hook) go to tests/golden/qwen_text_tnano.npz and, for the true
0.6B geometry (three 24-step deltas, max_new_tokens 16), tests/golden/qwen_text_0.6b.npz.

    python oracle/make_golden_qwen_text.py         # needs transformers and the staged reference (oracle/_ref)
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))

from whisperlivekit_b200.qwen_dims import QWEN_TEXT_DIMS, synthetic_text_state_dict  # noqa: E402

SAMPLE_STRIDE = 7
PLACEHOLDER, BOS, EOS, WAIT = 7, 1, 5, 3
TEMPLATE_A = [10, 11, PLACEHOLDER, 12, 13]
TEMPLATE_B = [10, 14, PLACEHOLDER, 12, 13]
CONTROLS_ON = dict(repetition_penalty=1.15, no_repeat_ngram_size=3, suppress_token_ids=[PLACEHOLDER, 10, 11, 12, 13, 14])
CONTROLS_OFF = dict(repetition_penalty=1.0, no_repeat_ngram_size=0, suppress_token_ids=[])


def schedule():
    """(audio steps, template, draft rule, controls, extra) per rolling call; the draft rule transforms the previous
    hypothesis the way the streamer (prev), a bad guess (corrupt), an ended hypothesis (eos) or a stale long one (long)
    would."""
    return [
        (6, "A", "none", "on", {}),
        (10, "A", "prev", "on", {}),
        (10, "A", "prev", "on", {}),                      # zero audio delta
        (15, "A", "corrupt", "on", {}),                   # mid-draft correction
        (18, "A", "eos", "on", {}),                       # draft trimmed at EOS
        (22, "A", "long", "on", {}),                      # draft longer than max_new_tokens
        (24, "B", "prev", "on", {}),                      # template change: rebuild
        (28, "B", "prev", "off", {}),
        (30, "B", "prev", "on", {"max_consecutive_text_tokens": 4}),
        (32, "B", "corrupt", "off", {}),
    ]


def make_draft(rule, prev):
    if rule == "none" or not prev:
        return None
    if rule == "prev":
        return list(prev)
    if rule == "corrupt":
        d = list(prev)
        d[min(3, len(d) - 1)] = (d[min(3, len(d) - 1)] + 17) % 2000 + 20
        return d
    if rule == "eos":
        return list(prev[:4]) + [EOS] + list(prev[4:])
    if rule == "long":
        return list(prev) + list(prev) + [21, 22, 23]
    raise ValueError(rule)


def build_reference(dims, sd):
    from transformers import Qwen3Config, Qwen3Model
    from qwen3_asr_causal.model import Qwen3ASRRealtimeQwenDecoderModel
    cfg = Qwen3Config(vocab_size=dims.vocab, hidden_size=dims.d_model, intermediate_size=dims.ffn_dim,
                      num_hidden_layers=dims.n_layer, num_attention_heads=dims.n_head, num_key_value_heads=dims.n_kv_head,
                      head_dim=dims.head_dim, rms_norm_eps=dims.rms_eps, tie_word_embeddings=dims.tied,
                      rope_parameters={"rope_type": "default", "rope_theta": dims.rope_theta},
                      max_position_embeddings=max(dims.max_ctx, 2048), attn_implementation="eager")
    tm = Qwen3Model(cfg).eval()
    tm.load_state_dict({k: torch.as_tensor(v) for k, v in sd.items() if k != "lm_head.weight"}, strict=True)
    lm = torch.nn.Linear(dims.d_model, dims.vocab, bias=False)
    lm.weight.data.copy_(torch.as_tensor(sd["lm_head.weight"] if not dims.tied else sd["embed_tokens.weight"]))
    return Qwen3ASRRealtimeQwenDecoderModel(None, qwen_model_id="seeded", text_model=tm, lm_head=lm, bos_token_id=BOS,
                                            wait_token_id=WAIT, audio_encoder=torch.nn.Identity(),
                                            adapter=torch.nn.Identity(), audio_backend="seeded").eval()


def schedule_06b():
    """The true geometry: three 24-step audio deltas (1.92 s each) with the previous hypothesis as the draft."""
    return [
        (24, "A", "none", "on", {}),
        (48, "A", "prev", "on", {}),
        (72, "A", "corrupt", "on", {}),
    ]


def run(name, seed=3, max_new_tokens=12, sched=None, stride=SAMPLE_STRIDE):
    from qwen3_asr_causal.model import CachedAudioDecodeState
    dims = QWEN_TEXT_DIMS[name]
    sd = synthetic_text_state_dict(dims, seed)
    model = build_reference(dims, sd)
    sched = sched or schedule()
    steps_max = max(s for s, *_ in sched)
    frames = np.random.default_rng(seed + 100).standard_normal((steps_max, dims.d_model)).astype(np.float32)
    log = []
    model.lm_head.register_forward_hook(lambda m, i, o: log.append(o.detach().reshape(-1, o.shape[-1])[:, ::stride].numpy().copy()))
    state = CachedAudioDecodeState(audio=None, adapter=None)
    calls, prev = [], []
    for steps, tpl, rule, ctl, extra in sched:
        draft = make_draft(rule, prev)
        kw = dict(CONTROLS_ON if ctl == "on" else CONTROLS_OFF, **extra)
        n0 = len(log)
        with torch.no_grad():
            toks, stats = model.generate_full_hypothesis_rolling(
                torch.as_tensor(frames[None, :steps]), state=state,
                template_token_ids=TEMPLATE_A if tpl == "A" else TEMPLATE_B, audio_placeholder_token_id=PLACEHOLDER,
                draft_token_ids=draft, max_new_tokens=max_new_tokens, eos_token_id=EOS, **kw)
        toks = [int(t) for t in toks[0].tolist()]
        calls.append(dict(kind="rolling", steps=steps, template=tpl, draft=draft, controls=kw, tokens=toks,
                          stats=stats, n_logit_calls=len(log) - n0))
        prev = toks
        print(name, steps, tpl, rule, ctl, toks, stats["decoder_path"], stats["draft_accepted"], stats["decode_steps"])
    for steps, prefix in ((12, True), (9, False)):
        n0 = len(log)
        kw = dict(CONTROLS_ON)
        with torch.no_grad():
            toks = model.generate_full_hypothesis_from_cached_audio(
                torch.as_tensor(frames[None, :steps]),
                prefix_token_ids=([10, 11] + [PLACEHOLDER] * steps + [12, 13]) if prefix else None,
                audio_placeholder_token_id=PLACEHOLDER if prefix else None, max_new_tokens=max_new_tokens,
                eos_token_id=EOS, **kw)
        toks = [int(t) for t in toks[0].tolist()]
        calls.append(dict(kind="full", steps=steps, prefix=prefix, controls=kw, tokens=toks, n_logit_calls=len(log) - n0))
        print(name, "full", steps, prefix, toks)
    samples = np.concatenate([a.reshape(-1) for a in log]).astype(np.float32)
    rows = np.asarray([a.shape[0] for a in log], np.int32)
    out = os.path.join(ROOT, "tests", "golden", f"qwen_text_{'0.6b' if name == 'qwen3-asr-0.6b' else name}.npz")
    np.savez_compressed(out, seed=np.int32(seed), max_new_tokens=np.int32(max_new_tokens), frames=frames,
                        calls=np.frombuffer(json.dumps(calls).encode(), np.uint8), samples=samples, sample_rows=rows,
                        sample_stride=np.int32(stride),
                        consts=np.asarray([PLACEHOLDER, BOS, EOS, WAIT], np.int32))
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    torch.manual_seed(0)
    run("tnano")
    run("qwen3-asr-0.6b", seed=4, max_new_tokens=16, sched=schedule_06b(), stride=97)
