"""Host side of the Silero VAD ingest step (SURVEY.md section 8f item 3) over the C ABI (``wlk_vad_*``).

* ``VadEngine`` -- batched: many streams, each with its own model state (64-sample context + LSTM h, c) on the device;
  ``forward(sids, audios)`` consumes every complete 512-sample window of every stream in one kernel launch.
* ``B200VadModel`` -- duck-types the scripted model the reference hands to ``VADIterator`` / ``FixedVADIterator``
  (whisperlivekit/silero_vad_iterator.py:20-29, 181-331): ``model(x, 16000) -> tensor [[p]]`` and ``reset_states()``,
  so the reference's iterator (thresholds, min-silence / padding logic, event list) runs unchanged on top.
The weights are the scripted model's own ``state_dict()`` (names kept).  No CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Sequence

import numpy as np

from . import _lib as L

WINDOW = 512


class VadEngine:
    def __init__(self, state_dict: Dict[str, np.ndarray], device: int = 0, max_sessions: int = 64):
        self.lib = L.load()
        h = C.c_void_p()
        L.check(self.lib.wlk_vad_create(int(device), int(max_sessions), C.byref(h)))
        self.h = h
        self._closed = False
        for k, v in state_dict.items():
            name = k[7:] if k.startswith("_model.") else k
            if name.startswith("_model_8k") or k.startswith("_model_8k"):
                continue                                              # the 8 kHz branch of the scripted model is not used at 16 kHz
            a = np.ascontiguousarray(np.asarray(v, np.float32))
            L.check(self.lib.wlk_vad_load_tensor(self.h, name.encode(), a.ctypes.data_as(C.c_void_p), a.size))

    def open_session(self) -> int:
        sid = C.c_int32()
        L.check(self.lib.wlk_vad_session_open(self.h, C.byref(sid)))
        return int(sid.value)

    def reset_session(self, sid: int) -> None:
        L.check(self.lib.wlk_vad_session_reset(self.h, int(sid)))

    def close_session(self, sid: int) -> None:
        L.check(self.lib.wlk_vad_session_close(self.h, int(sid)))

    def forward(self, sids: Sequence[int], audios: Sequence[np.ndarray]) -> List[np.ndarray]:
        """audios[i]: fp32 samples of stream i, a whole number of 512-sample windows -> probabilities per window."""
        s = np.ascontiguousarray(sids, np.int32)
        wins = []
        offs = np.zeros(len(s) + 1, np.int32)
        for i, a in enumerate(audios):
            a = np.ascontiguousarray(np.asarray(a, np.float32).reshape(-1))
            if a.shape[0] % WINDOW:
                raise ValueError("VAD input must be whole 512-sample windows (FixedVADIterator buffers the remainder)")
            wins.append(a)
            offs[i + 1] = offs[i] + a.shape[0] // WINDOW
        pcm = np.concatenate(wins) if wins else np.zeros(0, np.float32)
        probs = np.zeros(int(offs[-1]), np.float32)
        L.check(self.lib.wlk_vad_forward(self.h, s.ctypes.data_as(C.c_void_p), len(s), pcm.ctypes.data_as(C.c_void_p),
                                         offs.ctypes.data_as(C.c_void_p), probs.ctypes.data_as(C.c_void_p)))
        return [probs[offs[i]: offs[i + 1]].copy() for i in range(len(s))]

    def close(self) -> None:
        if not self._closed:
            self._closed = True
            L.check(self.lib.wlk_vad_destroy(self.h))

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class B200VadModel:
    """One stream's view of a ``VadEngine`` with the call surface of the scripted Silero model."""

    def __init__(self, engine: VadEngine):
        self.engine = engine
        self.sid = engine.open_session()

    def reset_states(self, batch_size: int = 1) -> None:
        self.engine.reset_session(self.sid)

    def __call__(self, x, sr: int = 16000):
        import torch
        if sr != 16000:
            raise ValueError("the H100 VAD engine implements the 16 kHz branch")
        a = x.detach().cpu().float().numpy() if hasattr(x, "detach") else np.asarray(x, np.float32)
        a = a.reshape(-1)
        if a.shape[0] != WINDOW:
            raise ValueError(f"Provided number of samples is {a.shape[0]} (supported: 512 for 16000 sampling rate)")
        p = self.engine.forward([self.sid], [a])[0]
        return torch.from_numpy(p.reshape(1, 1))

    def close(self) -> None:
        self.engine.close_session(self.sid)
