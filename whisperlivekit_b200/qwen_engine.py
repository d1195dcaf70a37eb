"""Host wrapper of the Qwen3-ASR causal audio tower engine (ctypes over wlk_qwen_* in include/wlk_b200.h).

Mirrors how the reference drives QwenAudioCausalKVEncoder (third_party/qwen3-asr-causal/src/qwen3_asr_causal/
causal.py:713-782): ``forward_chunk(mels, state) -> (hidden, state)`` becomes ``forward_chunk(sids, mels)`` over
device-resident per-session state, batched over sessions.  No CPU fallback: construction fails without the CUDA
library or a H100."""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import _lib as L
from .qwen_dims import QwenTowerDims


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


class QwenTowerEngine:
    def __init__(self, dims: QwenTowerDims, state_dict: Optional[Dict[str, np.ndarray]] = None, *, precision: str = "bf16",
                 device: int = 0, max_sessions: int = 8, max_batch: int = 8, gemm_backend: str = "auto"):
        self.lib = L.load()
        self.dims = dims
        self.precision = precision
        self.device = int(device)
        be = {"auto": L.BACKEND_AUTO, "simt": L.BACKEND_SIMT, "tcgen05": L.BACKEND_TCGEN05}
        cdims = L.wlk_qwen_dims(*dims.as_tuple())
        cfg = L.wlk_config(device=device, precision={"fp32": L.PREC_FP32, "bf16": L.PREC_BF16}[precision],
                           max_sessions=max_sessions, max_batch=max_batch, gemm_backend=be[gemm_backend],
                           attn_backend=L.BACKEND_SIMT, max_align_heads=0, reserved=0)
        h = C.c_void_p()
        L.check(self.lib.wlk_qwen_create(C.byref(cdims), C.byref(cfg), C.byref(h)))
        self.h = h
        self._closed = False
        if state_dict is not None:
            self.load_state_dict(state_dict)

    def load_state_dict(self, sd: Dict[str, np.ndarray]) -> None:
        for name, arr in sd.items():
            a = np.ascontiguousarray(arr, np.float32)
            shape = (C.c_int64 * a.ndim)(*a.shape)
            L.check(self.lib.wlk_qwen_load_tensor(self.h, name.encode(), _ptr(a), shape, a.ndim))
        L.check(self.lib.wlk_qwen_finalize_weights(self.h))

    def memory(self) -> Dict[str, int]:
        w, s, k = C.c_size_t(), C.c_size_t(), C.c_size_t()
        L.check(self.lib.wlk_qwen_memory(self.h, C.byref(w), C.byref(s), C.byref(k)))
        return dict(weights=w.value, sessions=s.value, workspace=k.value)

    # -- sessions (QwenAudioCausalKVState, causal.py:44-57) ------------------------------------
    def open_session(self) -> int:
        sid = C.c_int32()
        L.check(self.lib.wlk_qwen_session_open(self.h, C.byref(sid)))
        return sid.value

    def close_session(self, sid: int) -> None:
        L.check(self.lib.wlk_qwen_session_close(self.h, sid))

    def reset_session(self, sid: int) -> None:
        L.check(self.lib.wlk_qwen_session_reset(self.h, sid))

    def _state(self, sid: int):
        p, e = C.c_int32(), C.c_int64()
        L.check(self.lib.wlk_qwen_session_state(self.h, sid, C.byref(p), C.byref(e)))
        return p.value, e.value

    def pending_frames(self, sid: int) -> int:
        return self._state(sid)[0]

    def emitted_steps(self, sid: int) -> int:
        return self._state(sid)[1]

    def mutable_steps(self, sid: int) -> int:
        """steps of the bounded mutable tail (QwenAudioCausalKVState.mutable_steps); emitted_steps counts frozen steps"""
        m = C.c_int32()
        L.check(self.lib.wlk_qwen_session_mutable_steps(self.h, sid, C.byref(m)))
        return m.value

    def get_pending(self, sid: int) -> np.ndarray:
        """QwenAudioCausalKVState.mel_buffer: the session's pending mel frames [frames, n_mels]."""
        out = np.zeros((max(self.pending_frames(sid), 1), self.dims.n_mels), np.float32)
        n = C.c_int32()
        L.check(self.lib.wlk_qwen_session_get_pending(self.h, sid, _ptr(out), out.shape[0], C.byref(n)))
        return out[:n.value]

    def set_pending(self, sid: int, mels: np.ndarray) -> None:
        m = np.ascontiguousarray(mels, np.float32).reshape(-1, self.dims.n_mels)
        L.check(self.lib.wlk_qwen_session_set_pending(self.h, sid, _ptr(m if m.shape[0] else np.zeros(1, np.float32)),
                                                      m.shape[0]))

    # -- forward_chunk (causal.py:713-782), batched over sessions -----------------------------
    def _chunk_args(self, sids, mels):
        n = len(sids)
        if n != len(mels):
            raise ValueError("sids and mels differ in length")
        D = self.dims
        parts = [np.ascontiguousarray(m, np.float32).reshape(-1, D.n_mels) for m in mels]
        offs = np.zeros(n + 1, np.int32)
        offs[1:] = np.cumsum([p.shape[0] for p in parts])
        flat = np.concatenate(parts, axis=0) if offs[-1] else np.zeros((1, D.n_mels), np.float32)
        consume = D.block_frames if D.block_frames > 0 else D.chunk_frames
        cap = int(sum((self.pending_frames(s) + p.shape[0]) // consume * consume // D.chunk_frames for s, p in zip(sids, parts)))
        cap += D.mutable_tail_steps * n                      # a mutable tail re-emits its steps with every call
        return np.asarray(list(sids), np.int32), flat, offs, cap

    def forward_chunk(self, sids: Sequence[int], mels: Sequence[np.ndarray]) -> List[np.ndarray]:
        ids, flat, offs, cap = self._chunk_args(sids, mels)
        out = np.zeros((max(cap, 1), self.dims.out_dim), np.float32)
        rows = np.zeros(len(ids) + 1, np.int32)
        L.check(self.lib.wlk_qwen_forward_chunk(self.h, _ptr(ids), len(ids), _ptr(flat), _ptr(offs), _ptr(out), cap, _ptr(rows)))
        return [out[rows[i]: rows[i + 1]].copy() for i in range(len(ids))]

    def _device_out(self, cap: int):
        import torch
        out = torch.empty(max(cap, 1), self.dims.out_dim, dtype=torch.float32, device=f"cuda:{self.device}")
        torch.cuda.current_stream(out.device).synchronize()   # the engine's stream does not order itself after torch's
        return out

    def forward_chunk_device(self, sids: Sequence[int], mels: Sequence[np.ndarray]):
        """forward_chunk with the rows left on the device: (fp32 CUDA tensor [rows, out_dim], row offsets [n + 1])."""
        ids, flat, offs, cap = self._chunk_args(sids, mels)
        out = self._device_out(cap)
        rows = np.zeros(len(ids) + 1, np.int32)
        L.check(self.lib.wlk_qwen_forward_chunk_device(self.h, _ptr(ids), len(ids), _ptr(flat), _ptr(offs),
                                                       C.c_void_p(out.data_ptr()), cap, _ptr(rows)))
        return out[:int(rows[-1])], rows

    # -- incremental log-mel front end (StreamingMelExtractor, features.py:32-112) on the device -------------
    def load_mel_filters(self, filters: Optional[np.ndarray] = None) -> None:
        from .weights import mel_filterbank
        a = np.ascontiguousarray(mel_filterbank(self.dims.n_mels) if filters is None else filters, np.float32)
        shape = (C.c_int64 * 2)(*a.shape)
        L.check(self.lib.wlk_qwen_load_tensor(self.h, b"mel_filters", _ptr(a), shape, 2))

    def _mel_call(self, sids, audios, flush: bool) -> List[np.ndarray]:
        n = len(sids)
        D = self.dims
        parts = [np.ascontiguousarray(a, np.float32).reshape(-1) for a in audios] if not flush else [np.zeros(0, np.float32)] * n
        offs = np.zeros(n + 1, np.int64)
        offs[1:] = np.cumsum([p.shape[0] for p in parts])
        flat = np.concatenate(parts) if offs[-1] else np.zeros(1, np.float32)
        cap = int(offs[-1] // 160 + 4 * n + 8) if not flush else 4 * n + 8
        out = np.zeros((cap, D.n_mels), np.float32)
        rows = np.zeros(n + 1, np.int32)
        ids = np.asarray(list(sids), np.int32)
        L.check(self.lib.wlk_qwen_append_audio(self.h, _ptr(ids), n, _ptr(flat), _ptr(offs), _ptr(out), cap, _ptr(rows), int(flush)))
        return [out[rows[i]: rows[i + 1]].copy() for i in range(n)]

    def mel_append(self, sids: Sequence[int], audios: Sequence[np.ndarray]) -> List[np.ndarray]:
        """StreamingMelExtractor.append per session: raw samples in, newly determined mel frames [frames, n_mels] out."""
        return self._mel_call(sids, audios, False)

    def mel_flush(self, sids: Sequence[int]) -> List[np.ndarray]:
        """StreamingMelExtractor.flush per session."""
        return self._mel_call(sids, None, True)

    def flush_pending(self, sids: Sequence[int]) -> List[np.ndarray]:
        """End of stream (causal.py:687-711): encode the buffered whole chunks, drop the sub-chunk remainder."""
        n = len(sids)
        D = self.dims
        cap = int(sum(self.pending_frames(s) // D.chunk_frames for s in sids))
        out = np.zeros((max(cap, 1), D.out_dim), np.float32)
        rows = np.zeros(n + 1, np.int32)
        ids = np.asarray(list(sids), np.int32)
        L.check(self.lib.wlk_qwen_flush_pending(self.h, _ptr(ids), n, _ptr(out), cap, _ptr(rows)))
        return [out[rows[i]: rows[i + 1]].copy() for i in range(n)]

    def flush_pending_device(self, sids: Sequence[int]):
        """flush_pending with the rows left on the device, as forward_chunk_device returns them."""
        cap = int(sum(self.pending_frames(s) // self.dims.chunk_frames for s in sids))
        out = self._device_out(cap)
        rows = np.zeros(len(sids) + 1, np.int32)
        ids = np.asarray(list(sids), np.int32)
        L.check(self.lib.wlk_qwen_flush_pending_device(self.h, _ptr(ids), len(ids), C.c_void_p(out.data_ptr()), cap, _ptr(rows)))
        return out[:int(rows[-1])], rows

    def close(self) -> None:
        if not self._closed:
            self._closed = True
            L.check(self.lib.wlk_qwen_destroy(self.h))

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
