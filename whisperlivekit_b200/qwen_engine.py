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
from ._lib import _ptr, pack, split
from .qwen_dims import sinusoid_inv_freq


class _QwenEngineBase(L.Engine):
    """What both tower engines share: one ``wlk_qwen`` handle, its weights, sessions and memory."""

    DESTROY = "wlk_qwen_destroy"
    LOAD_TENSOR, FINALIZE, MEMORY = "wlk_qwen_load_tensor", "wlk_qwen_finalize_weights", "wlk_qwen_memory"
    SESSION_OPEN, SESSION_CLOSE, SESSION_RESET = "wlk_qwen_session_open", "wlk_qwen_session_close", "wlk_qwen_session_reset"

    def __init__(self, dims, state_dict: Optional[Dict[str, np.ndarray]] = None, *, precision: str = "bf16",
                 device: int = 0, max_sessions: int = 8, max_batch: int = 8, gemm_backend: str = "auto"):
        self.dims = dims
        self._create(self._DIMS(*dims.as_tuple()), precision=precision, device=device, max_sessions=max_sessions,
                     max_batch=max_batch, gemm_backend=gemm_backend)
        # the reference's fp32 frequencies of the positional rows past the table, evaluated on this device like the
        # reference evaluates them on its own
        self.load_tensor("positional_embedding.inv_freq", sinusoid_inv_freq(dims.d_model, f"cuda:{self.device}"))
        if state_dict is not None:
            self.load_state_dict(state_dict)

    def _pack(self, sids, mels):
        """(session ids, the mels [frames, n_mels] of every session back to back, frame offsets [n + 1])"""
        n = len(sids)
        if n != len(mels):
            raise ValueError("sids and mels differ in length")
        flat, offs = pack(mels, np.float32, (self.dims.n_mels,))
        return np.asarray(list(sids), np.int32), flat, offs

    def _device_out(self, cap: int):
        import torch
        out = torch.empty(max(cap, 1), self.dims.out_dim, dtype=torch.float32, device=f"cuda:{self.device}")
        torch.cuda.current_stream(out.device).synchronize()   # the engine's stream does not order itself after torch's
        return out

    # -- op-level (device pointers, e.g. torch tensors' data_ptr(); "act" is fp32 or bf16 as the precision) ------------
    def op_positions(self, positions: Sequence[int], out_ptr) -> None:
        """The positional rows fp32 [rows][d_model] of absolute positions: table rows, the closed form past the table."""
        pos = np.ascontiguousarray(positions, np.int32)
        L.check(self.lib.wlk_qwen_op_positions(self.h, _ptr(pos), len(pos), out_ptr))

    def op_conv_stem(self, mel_ptr, avail: Sequence[int], p0: Sequence[int], a1_ptr, a2_ptr, a3_ptr) -> None:
        """The mode's conv stem over chunks fp32 [n][T0][n_mels] (T0 = 8 causal, 100 windowed) -> the three activations
        in act: a1 [n][n_mels/2][T1][C], a2 [n][n_mels/4][T2][C], a3 [n][T3][n_mels/8][C]."""
        av = np.ascontiguousarray(avail, np.int32)
        pz = np.ascontiguousarray(p0, np.int32)
        if len(av) != len(pz):
            raise ValueError("avail and p0 differ in length")
        L.check(self.lib.wlk_qwen_op_conv_stem(self.h, mel_ptr, _ptr(av), _ptr(pz), len(av), a1_ptr, a2_ptr, a3_ptr))

    def op_qkv(self, layer: int, xn_ptr, row_slot: Sequence[int], row_pos: Sequence[int], kv_ptrs: Sequence[int],
               q_out_ptr) -> None:
        """Causal engine: the QKV projection of xn act [rows][d_model] with the round's epilogue (bias, head_dim^-0.5 on
        q) -> q act [rows][d_model], k / v into ring kv_ptrs[row_slot[r]] at slot row_pos[r] % ring of layer."""
        slot = np.ascontiguousarray(row_slot, np.int32)
        pos = np.ascontiguousarray(row_pos, np.int32)
        if len(slot) != len(pos):
            raise ValueError("row_slot and row_pos differ in length")
        kv = (C.c_void_p * len(kv_ptrs))(*[int(p) for p in kv_ptrs])
        L.check(self.lib.wlk_qwen_op_qkv(self.h, int(layer), xn_ptr, _ptr(slot), _ptr(pos), len(pos), kv, len(kv_ptrs),
                                         q_out_ptr))

    def op_attention(self, layer: int, q_ptr, starts: Sequence[int], n_steps: Sequence[int], kv_ptrs: Sequence[int],
                     out_ptr) -> None:
        """Causal engine: one round's attention.  Job j owns the next n_steps[j] rows of q / out (act [rows][d_model]) at
        positions starts[j] ..; its keys are in ring kv_ptrs[j]."""
        st = np.ascontiguousarray(starts, np.int32)
        ns = np.ascontiguousarray(n_steps, np.int32)
        if not (len(st) == len(ns) == len(kv_ptrs)):
            raise ValueError("starts, n_steps and kv_ptrs differ in length")
        kv = (C.c_void_p * max(len(kv_ptrs), 1))(*[int(p) for p in kv_ptrs])
        L.check(self.lib.wlk_qwen_op_attention(self.h, int(layer), q_ptr, _ptr(st), _ptr(ns), len(st), kv, out_ptr))


class QwenTowerEngine(_QwenEngineBase):
    """The causal tower (wlk_qwen_create) over a QwenTowerDims geometry."""

    _DIMS, CREATE = L.wlk_qwen_dims, "wlk_qwen_create"

    # -- sessions (QwenAudioCausalKVState, causal.py:44-57) ------------------------------------
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
        ids, flat, offs = self._pack(sids, mels)
        D = self.dims
        consume = D.block_frames if D.block_frames > 0 else D.chunk_frames
        cap = int(sum((self.pending_frames(s) + int(offs[i + 1] - offs[i])) // consume * consume // D.chunk_frames
                      for i, s in enumerate(sids)))
        cap += D.mutable_tail_steps * len(ids)               # a mutable tail re-emits its steps with every call
        return ids, flat, offs, cap

    def forward_chunk(self, sids: Sequence[int], mels: Sequence[np.ndarray]) -> List[np.ndarray]:
        ids, flat, offs, cap = self._chunk_args(sids, mels)
        out = np.zeros((max(cap, 1), self.dims.out_dim), np.float32)
        rows = np.zeros(len(ids) + 1, np.int32)
        L.check(self.lib.wlk_qwen_forward_chunk(self.h, _ptr(ids), len(ids), _ptr(flat), _ptr(offs), _ptr(out), cap, _ptr(rows)))
        return split(out, rows)

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
        self.load_tensor("mel_filters", mel_filterbank(self.dims.n_mels) if filters is None else filters)

    def _mel_call(self, sids, audios, flush: bool) -> List[np.ndarray]:
        n = len(sids)
        flat, offs = pack([()] * n if flush else audios, np.float32, offs_dtype=np.int64)
        cap = int(offs[-1] // 160 + 4 * n + 8)
        out = np.zeros((cap, self.dims.n_mels), np.float32)
        rows = np.zeros(n + 1, np.int32)
        ids = np.asarray(list(sids), np.int32)
        L.check(self.lib.wlk_qwen_append_audio(self.h, _ptr(ids), n, _ptr(flat), _ptr(offs), _ptr(out), cap, _ptr(rows), int(flush)))
        return split(out, rows)

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
        return split(out, rows)

    def flush_pending_device(self, sids: Sequence[int]):
        """flush_pending with the rows left on the device, as forward_chunk_device returns them."""
        cap = int(sum(self.pending_frames(s) // self.dims.chunk_frames for s in sids))
        out = self._device_out(cap)
        rows = np.zeros(len(sids) + 1, np.int32)
        ids = np.asarray(list(sids), np.int32)
        L.check(self.lib.wlk_qwen_flush_pending_device(self.h, _ptr(ids), len(ids), C.c_void_p(out.data_ptr()), cap, _ptr(rows)))
        return out[:int(rows[-1])], rows


class QwenWindowEngine(_QwenEngineBase):
    """Host wrapper of the windowed Qwen3-ASR audio tower (wlk_qwen_window_* in include/wlk_b200.h).

    Mirrors QwenAudioSurgeryEncoder (third_party/qwen3-asr-causal/src/qwen3_asr_causal/model.py:441-608):
    ``forward_chunk(mels, state)`` becomes ``forward_chunk(sids, mels)`` over per-session device windows, batched over
    sessions; ``forward_full`` becomes ``encode``.  No CPU fallback."""

    _DIMS, CREATE = L.wlk_qwen_window_dims, "wlk_qwen_window_create"
    STATE_FIELDS = ("frames_seen", "window_start_frame", "emitted_steps", "last_input_frames", "last_recomputed_frames",
                    "last_recomputed_context_frames", "window_frames")

    def state(self, sid: int) -> Dict[str, int]:
        """QwenAudioSurgeryState's counters (model.py:36-43) plus the frames the device window holds."""
        f = np.zeros(7, np.int64)
        L.check(self.lib.wlk_qwen_window_state(self.h, sid, _ptr(f)))
        return dict(zip(self.STATE_FIELDS, (int(v) for v in f)))

    def _cap(self, n: int) -> int:
        from .qwen_dims import window_output_steps
        return n * window_output_steps(self.dims.window_frames)

    def forward_chunk(self, sids: Sequence[int], mels: Sequence[np.ndarray]) -> List[np.ndarray]:
        """forward_chunk per session: new mel frames [frames, n_mels] in, the newly emitted rows [steps, out_dim] out."""
        ids, flat, offs = self._pack(sids, mels)
        cap = self._cap(len(ids))
        out = np.zeros((max(cap, 1), self.dims.out_dim), np.float32)
        rows = np.zeros(len(ids) + 1, np.int32)
        L.check(self.lib.wlk_qwen_window_forward(self.h, _ptr(ids), len(ids), _ptr(flat), _ptr(offs), _ptr(out), cap,
                                                 _ptr(rows), 0))
        return split(out, rows)

    def forward_chunk_device(self, sids: Sequence[int], mels: Sequence[np.ndarray]):
        """forward_chunk with the rows left on the device: (fp32 CUDA tensor [rows, out_dim], row offsets [n + 1])."""
        ids, flat, offs = self._pack(sids, mels)
        cap = self._cap(len(ids))
        out = self._device_out(cap)
        rows = np.zeros(len(ids) + 1, np.int32)
        L.check(self.lib.wlk_qwen_window_forward(self.h, _ptr(ids), len(ids), _ptr(flat), _ptr(offs),
                                                 C.c_void_p(out.data_ptr()), cap, _ptr(rows), 1))
        return out[:int(rows[-1])], rows

    def encode(self, mels: Sequence[np.ndarray]) -> List[np.ndarray]:
        """forward_full: every row of each stateless window (at most left + right frames each)."""
        n = len(mels)
        _, flat, offs = self._pack(list(range(n)), mels)
        cap = self._cap(n)
        out = np.zeros((max(cap, 1), self.dims.out_dim), np.float32)
        rows = np.zeros(n + 1, np.int32)
        L.check(self.lib.wlk_qwen_window_encode(self.h, n, _ptr(flat), _ptr(offs), _ptr(out), cap, _ptr(rows)))
        return split(out, rows)


def window_attention(qkv, stream_rows: Sequence[int], block_rows: int, device: int = 0, out=None):
    """The windowed tower's block-diagonal attention kernel on a CUDA tensor qkv [rows, 3 * d_model] (fp32 runs the SIMT
    parity kernel, bf16 the tensor-core one; q pre-scaled) -> [rows, d_model] of the same dtype (written into ``out``
    when given: rows past the streams are left as they are).  Kernel tests only."""
    import torch
    lib = L.load()
    d = qkv.shape[1] // 3
    qkv = qkv.contiguous()
    if out is None:
        out = torch.empty(qkv.shape[0], d, dtype=qkv.dtype, device=qkv.device)
    torch.cuda.synchronize(qkv.device)
    rows = np.asarray(list(stream_rows), np.int32)
    prec = L.PREC_FP32 if qkv.dtype == torch.float32 else L.PREC_BF16
    L.check(lib.wlk_qwen_window_attention(device, prec, C.c_void_p(qkv.data_ptr()), C.c_void_p(out.data_ptr()), d,
                                          _ptr(rows), len(rows), int(block_rows)))
    return out
