"""CPU stand-ins for the realtime model's engines, behind the same API as the CUDA ones (qwen_engine.QwenTowerEngine,
qwen_text_engine.QwenTextEngine):

  QwenRealtimeTowerOracle   QwenTowerOracle plus the session's pending mel frames (get_pending / set_pending)
  QwenRealtimeTextOracle    QwenTextOracle plus the frame adapter (``adapt``), in fp32 torch with the reference module's
                            own operations (QwenAudioSurgeryFrameAdapter, model.py:631-691)
  adapter_f64               the same adapter restated in float64, the yardstick for the device kernel"""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch
import torch.nn.functional as F

from oracle.qwen_oracle import QwenTowerOracle
from oracle.qwen_text_oracle import QwenTextOracle

ADAPTER_EPS = 1e-6


class QwenRealtimeTowerOracle(QwenTowerOracle):
    def get_pending(self, sid: int) -> np.ndarray:
        return self._s[sid]["buf"].numpy().copy()

    def set_pending(self, sid: int, mels: np.ndarray) -> None:
        self._s[sid]["buf"] = torch.as_tensor(np.asarray(mels, np.float32).reshape(-1, self.dims.n_mels)).clone()


def _blocks(sd: Dict) -> int:
    n = 0
    while f"adapter.blocks.{n}.norm.weight" in sd:
        n += 1
    return n


class QwenRealtimeTextOracle(QwenTextOracle):
    @torch.no_grad()
    def adapt(self, x: torch.Tensor) -> torch.Tensor:
        if "adapter.proj.weight" not in self.w:
            raise ValueError("no adapter loaded")
        y = F.linear(x.float(), self.w["adapter.proj.weight"])
        for i in range(_blocks(self.w)):
            p = f"adapter.blocks.{i}."
            n = y * torch.rsqrt(y.pow(2).mean(dim=-1, keepdim=True) + ADAPTER_EPS) * self.w[p + "norm.weight"]
            u = F.linear(F.silu(F.linear(n, self.w[p + "mlp.gate.weight"])) * F.linear(n, self.w[p + "mlp.up.weight"]),
                         self.w[p + "mlp.down.weight"])
            y = y + u * float(self.w["adapter.residual_scale"][0])
        return y


def adapter_f64(x, sd: Dict) -> np.ndarray:
    """The adapter over rows x [rows, in_dim] in float64 (numpy)."""
    w = {k: np.asarray(v, np.float64) for k, v in sd.items() if k.startswith("adapter.")}
    y = np.asarray(x, np.float64) @ w["adapter.proj.weight"].T
    for i in range(_blocks(w)):
        p = f"adapter.blocks.{i}."
        n = y / np.sqrt((y * y).mean(-1, keepdims=True) + ADAPTER_EPS) * w[p + "norm.weight"]
        g, u = n @ w[p + "mlp.gate.weight"].T, n @ w[p + "mlp.up.weight"].T
        y = y + (g / (1.0 + np.exp(-g)) * u) @ w[p + "mlp.down.weight"].T * float(w["adapter.residual_scale"][0])
    return y
