"""Replays a recorded Qwen3 text-decoder fixture (oracle/make_golden_qwen_text.py) through a text engine (the device
engine or the CPU oracle) with the shared generate driver, capturing the raw lm_head rows of every forward."""
from __future__ import annotations

import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_fixture(name: str) -> dict:
    z = np.load(os.path.join(GOLDEN, f"qwen_text_{name}.npz"))
    fx = {k: z[k] for k in z.files}
    fx["calls"] = json.loads(bytes(fx["calls"]).decode())
    placeholder, bos, eos, wait = (int(v) for v in fx["consts"])
    fx.update(placeholder=placeholder, bos=bos, eos=eos, wait=wait)
    rows, stride = fx["sample_rows"], int(fx["sample_stride"])
    width = fx["samples"].shape[0] // int(rows.sum())
    fx["sample_blocks"] = np.split(fx["samples"].reshape(-1, width), np.cumsum(rows)[:-1])
    fx["stride"] = stride
    return fx


def capture_logits(engine, stride: int) -> list:
    """Wrap engine.forward so that every forward's lm_head rows (strided columns) are recorded."""
    log = []
    inner = engine.forward

    def forward(sids, blocks, logit_rows):
        inner(sids, blocks, logit_rows)
        log.append(engine.logits()[:, ::stride].copy())

    engine.forward = forward
    return log


TEMPLATES = {"A": [10, 11, 7, 12, 13], "B": [10, 14, 7, 12, 13]}


def replay(engine, fx, drafts=None):
    """Drive every recorded call; drafts[k] overrides the draft of rolling call k.  Returns [(tokens, stats)]."""
    frames, max_new = fx["frames"], int(fx["max_new_tokens"])
    sid = engine.open_session()
    state, out = None, []
    try:
        for k, c in enumerate(fx["calls"]):
            ctl = dict(c["controls"])
            if c["kind"] == "rolling":
                draft = c["draft"] if drafts is None else drafts[k]
                toks, stats, states = engine.generate_rolling(
                    [sid], [frames[:c["steps"]]], [state], TEMPLATES[c["template"]], fx["placeholder"], [draft],
                    max_new_tokens=max_new, eos_token_id=fx["eos"], wait_token_id=fx["wait"], bos_token_id=fx["bos"],
                    **ctl)
                state = states[0]
                out.append((toks[0], stats[0]))
            else:
                steps = c["steps"]
                prefix = ([10, 11] + [fx["placeholder"]] * steps + [12, 13]) if c["prefix"] else None
                toks = engine.generate_full(frames[:steps], prefix_token_ids=prefix,
                                            audio_placeholder_token_id=fx["placeholder"] if c["prefix"] else None,
                                            max_new_tokens=max_new, bos_token_id=fx["bos"], eos_token_id=fx["eos"],
                                            wait_token_id=fx["wait"], **ctl)
                out.append((toks, None))
    finally:
        engine.close_session(sid)
    return out
