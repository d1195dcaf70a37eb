"""CPU restatement (torch, fp32) of the Qwen3-ASR text decoder with the device engine's primitives, the way
QwenTowerOracle stands behind the audio tower.

  forward            HF Qwen3Model over a croppable KV cache (transformers' Qwen3DecoderLayer: RMSNorm -> q/k/v ->
                     q_norm / k_norm -> rotate-half RoPE -> causal SDPA (scale head_dim^-0.5) -> o_proj; RMSNorm ->
                     down(silu(gate) * up)); final norm + lm_head on the last logit_rows rows of each session
  pick               _GreedyControlSession.controlled_logits + argmax (reference model.py:335-418)
  generate_rolling   model.py:991-1250 and generate_full model.py:839-989, by the shared driver
                     (whisperlivekit_b200.qwen_text_engine.TextDecodeDriver)

``logit_log`` keeps every forward's raw lm_head rows, for parity checks against recorded reference outputs."""
from __future__ import annotations

from typing import Dict, List

import numpy as np
import torch

from whisperlivekit_b200.qwen_dims import QwenTextDims
from whisperlivekit_b200.qwen_text_engine import Controls, TextDecodeDriver


def banned_ngram_tokens(history: List[int], n: int) -> set:
    """_banned_ngram_tokens (model.py:176-187)."""
    if n <= 0 or len(history) < n - 1:
        return set()
    if n == 1:
        return set(history)
    prefix = tuple(history[-(n - 1):])
    return {history[s + n - 1] for s in range(0, len(history) - n + 1) if tuple(history[s:s + n - 1]) == prefix}


def controlled_logits(logits: torch.Tensor, history: List[int], ctl: Controls, vocab: int) -> torch.Tensor:
    """One row of _GreedyControlSession.controlled_logits (model.py:335-398)."""
    x = logits.clone()
    if len(ctl.suppress):
        x[torch.as_tensor(ctl.suppress, dtype=torch.long)] = -torch.inf
    penalize = ctl.penalty != 1.0 and ctl.penalty > 0.0
    fmin = torch.finfo(x.dtype).min
    if penalize:
        seen = sorted({t for t in history if 0 <= t < vocab})
        if seen:
            idx = torch.tensor(seen, dtype=torch.long)
            v = x[idx]
            x[idx] = torch.where(v < 0, v * ctl.penalty, v / ctl.penalty)
    banned = [t for t in banned_ngram_tokens(history, ctl.ngram) if 0 <= t < vocab]
    if banned:
        x[torch.tensor(banned, dtype=torch.long)] = fmin
    if ctl.max_consecutive > 0 and ctl.wait_id >= 0 and len(history) >= ctl.max_consecutive:
        w = x[ctl.wait_id].clone()
        x[:] = fmin
        x[ctl.wait_id] = w
    return x


class QwenTextOracle(TextDecodeDriver):
    def __init__(self, dims: QwenTextDims, sd: Dict[str, np.ndarray]):
        self.dims = dims
        self.vocab = dims.vocab
        self.w = {k: torch.as_tensor(np.asarray(v, np.float32)) for k, v in sd.items()}
        if dims.tied:
            self.w["lm_head.weight"] = self.w["embed_tokens.weight"]
        hd = dims.head_dim
        if "rotary_emb.inv_freq" in self.w:                 # the model's own buffer, when the host passes it
            self.inv_freq = self.w["rotary_emb.inv_freq"].clone()
        else:
            self.inv_freq = 1.0 / (dims.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.int64).float() / hd))
        self.sessions: Dict[int, list] = {}
        self._next = 0
        self._last = torch.zeros(0, dims.vocab)
        self.logit_log: List[np.ndarray] = []

    # -- sessions --------------------------------------------------------------------------------------------------
    def open_session(self) -> int:
        sid = self._next
        self._next += 1
        self.sessions[sid] = [None] * self.dims.n_layer
        return sid

    def close_session(self, sid: int) -> None:
        del self.sessions[sid]

    def reset_session(self, sid: int) -> None:
        self.sessions[sid] = [None] * self.dims.n_layer

    def session_len(self, sid: int) -> int:
        kv = self.sessions[sid][0]
        return 0 if kv is None else int(kv[0].shape[1])

    def crop(self, sid: int, length: int) -> None:
        if not 0 <= length <= self.session_len(sid):
            raise ValueError(f"crop to {length} outside [0, {self.session_len(sid)}]")
        self.sessions[sid] = [None if kv is None else (kv[0][:, :length], kv[1][:, :length]) for kv in self.sessions[sid]]

    # -- model -----------------------------------------------------------------------------------------------------
    def _rms(self, x, w):
        v = x.pow(2).mean(-1, keepdim=True)
        return w * (x * torch.rsqrt(v + self.dims.rms_eps))

    @staticmethod
    def _rot(x):
        h = x.shape[-1] // 2
        return torch.cat((-x[..., h:], x[..., :h]), dim=-1)

    def _session_forward(self, sid: int, x: torch.Tensor) -> torch.Tensor:
        D = self.dims
        H, KV, hd = D.n_head, D.n_kv_head, D.head_dim
        past = self.session_len(sid)
        r = x.shape[0]
        pos = torch.arange(past, past + r, dtype=torch.float32)
        freqs = pos[:, None] * self.inv_freq[None, :]
        emb = torch.cat((freqs, freqs), dim=-1)
        cos, sin = emb.cos(), emb.sin()
        cache = self.sessions[sid]
        for li in range(D.n_layer):
            p = f"layers.{li}."
            h = self._rms(x, self.w[p + "input_layernorm.weight"])
            q = (h @ self.w[p + "self_attn.q_proj.weight"].T).view(r, H, hd).transpose(0, 1)
            k = (h @ self.w[p + "self_attn.k_proj.weight"].T).view(r, KV, hd).transpose(0, 1)
            v = (h @ self.w[p + "self_attn.v_proj.weight"].T).view(r, KV, hd).transpose(0, 1)
            q = self._rms(q, self.w[p + "self_attn.q_norm.weight"])
            k = self._rms(k, self.w[p + "self_attn.k_norm.weight"])
            q = q * cos + self._rot(q) * sin
            k = k * cos + self._rot(k) * sin
            if cache[li] is not None:
                k = torch.cat([cache[li][0], k], dim=1)
                v = torch.cat([cache[li][1], v], dim=1)
            cache[li] = (k, v)
            kk = k.repeat_interleave(H // KV, dim=0)
            vv = v.repeat_interleave(H // KV, dim=0)
            s = (q @ kk.transpose(1, 2)) * hd ** -0.5
            mask = torch.arange(past + r)[None, :] > (past + torch.arange(r))[:, None]
            s = s.masked_fill(mask, -torch.inf)
            a = torch.softmax(s, dim=-1) @ vv
            x = x + a.transpose(0, 1).reshape(r, H * hd) @ self.w[p + "self_attn.o_proj.weight"].T
            h = self._rms(x, self.w[p + "post_attention_layernorm.weight"])
            g = h @ self.w[p + "mlp.gate_proj.weight"].T
            u = h @ self.w[p + "mlp.up_proj.weight"].T
            x = x + (torch.nn.functional.silu(g) * u) @ self.w[p + "mlp.down_proj.weight"].T
        return x

    @torch.no_grad()
    def forward(self, sids, blocks, logit_rows) -> None:
        D = self.dims
        for sid, (src, _), lr in zip(sids, blocks, logit_rows):
            if self.session_len(sid) + len(src) > D.max_ctx:
                raise ValueError(f"context full: session {sid}")
        outs = []
        for sid, (src, emb), lr in zip(sids, blocks, logit_rows):
            src = np.asarray(src, np.int64)
            emb_t = None if emb is None else torch.as_tensor(np.asarray(emb, np.float32)).reshape(-1, D.d_model)
            rows = [self.w["embed_tokens.weight"][int(s)] if s >= 0 else emb_t[-1 - int(s)] for s in src]
            x = self._session_forward(sid, torch.stack(rows))
            if lr:
                h = self._rms(x[-lr:], self.w["norm.weight"])
                outs.append(h @ self.w["lm_head.weight"].T)
        self._last = torch.cat(outs) if outs else torch.zeros(0, D.vocab)
        self.logit_log.append(self._last.numpy().copy())

    def pick(self, hist, hist_off, hist_len, ctl: Controls, return_values: bool = False):
        picks, vals = [], []
        for j in range(self._last.shape[0]):
            h = [int(t) for t in hist[int(hist_off[j]): int(hist_off[j]) + int(hist_len[j])]]
            x = controlled_logits(self._last[j], h, ctl, self.vocab)
            k = int(torch.argmax(x))
            picks.append(k)
            vals.append(float(x[k]))
        picks = np.asarray(picks, np.int32)
        return (picks, np.asarray(vals, np.float32)) if return_values else picks

    def controlled_gap(self, hist: List[int], ctl: Controls, row: int) -> float:
        """Top-1 minus top-2 of the controlled logits of one row of the last forward."""
        x = controlled_logits(self._last[row], hist, ctl, self.vocab)
        top = torch.topk(x, 2).values
        return float(top[0] - top[1])

    def logits(self, row0: int = 0, n_rows=None) -> np.ndarray:
        n_rows = self._last.shape[0] - row0 if n_rows is None else n_rows
        return self._last[row0: row0 + n_rows].numpy().copy()
