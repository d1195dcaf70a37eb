"""Host wrapper of the streaming Sortformer engine (ctypes over wlk_sf_* in include/wlk_b200.h) and the drop-in objects
for the reference's diarization seam (SURVEY.md section 8b item 3).

Reference: whisperlivekit/diarization/sortformer_backend.py --
  ``SortformerDiarization`` (:55-128, the shared model)          -> ``B200SortformerDiarization``
  ``SortformerDiarizationOnline`` (:151-373, one per connection) -> ``B200SortformerDiarizationOnline``: the pipeline only
  calls ``insert_audio_chunk(np)``, ``await diarize() -> List[SpeakerSegment]``, ``insert_silence(sec)``, ``close()`` and
  tests ``hasattr(.., 'buffer_audio')`` (audio_processor.py:848-885, 1080-1081).
The forward (mel front end, FastConformer, Transformer, sigmoid head, speaker-cache update) runs on the device for all
streams of a call; ``_process_predictions`` is the device run-length kernel of ``diarization.py`` over the stream's
device-resident total_preds, so only segments are copied back.  No CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import threading
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import _lib as L
from ._lib import _ptr, pack, split
from .diarization import DiarizationSegmenter, SpeakerSegment, resolve_max_speakers
from .sortformer_dims import SortformerDims
from .weights import mel_filterbank


_INT_FIELDS = ("n_mels", "n_fft", "win_length", "hop", "conv_channels", "d_model", "n_head", "n_layer", "ff_mult", "conv_kernel",
               "tf_d_model", "tf_n_head", "tf_n_layer", "tf_inner", "n_spk", "spkcache_len", "fifo_len", "spkcache_update_period",
               "chunk_len", "subsampling_factor", "encoder_subsampling", "spkcache_sil_frames_per_spk")
_FLOAT_FIELDS = ("pred_score_threshold", "scores_boost_latest", "sil_threshold", "strong_boost_rate", "weak_boost_rate",
                 "min_pos_scores_rate")


class SortformerEngine(L.Engine):
    CREATE, DESTROY = "wlk_sf_create", "wlk_sf_destroy"
    LOAD_TENSOR, FINALIZE, MEMORY = "wlk_sf_load_tensor", "wlk_sf_finalize_weights", "wlk_sf_memory"
    SESSION_OPEN, SESSION_CLOSE, SESSION_RESET = "wlk_sf_session_open", "wlk_sf_session_close", "wlk_sf_session_reset"

    def __init__(self, dims: SortformerDims, state_dict: Optional[Dict[str, np.ndarray]] = None, *, precision: str = "bf16",
                 device: int = 0, max_sessions: int = 8, max_batch: int = 8, gemm_backend: str = "auto"):
        self.dims = dims
        cd = L.wlk_sf_dims(**{k: int(getattr(dims, k)) for k in _INT_FIELDS}, **{k: float(getattr(dims, k)) for k in _FLOAT_FIELDS})
        self._create(cd, precision=precision, device=device, max_sessions=max_sessions, max_batch=max_batch,
                     gemm_backend=gemm_backend)
        self.chunk_samples = dims.chunk_len * dims.subsampling_factor * dims.hop
        self.chunk_duration_seconds = self.chunk_samples / 16000.0           # sortformer_backend.py:190-194
        if state_dict is not None:
            self.load_state_dict(state_dict)

    def load_state_dict(self, sd: Dict[str, np.ndarray]) -> None:
        full = dict(sd)
        full.setdefault("mel_filters", mel_filterbank(self.dims.n_mels, 16000, self.dims.n_fft))
        super().load_state_dict(full)

    @staticmethod
    def _skip(name: str, arr) -> bool:
        # a NeMo checkpoint also carries buffers of modules this path replaces or never calls: the preprocessor's window /
        # filterbank (the front end is rebuilt from the geometry), BatchNorm's counter, the unused hidden_to_spks layer
        return (np.ndim(arr) == 0 or name.startswith(("preprocessor.", "sortformer_modules.hidden_to_spks."))
                or name.endswith("num_batches_tracked"))

    def step_audio(self, sids: Sequence[int], chunks: Sequence[np.ndarray], want_preds: bool = True) -> List[np.ndarray]:
        """diarize()'s device part for n streams: one ``chunk_samples`` chunk each -> chunk_preds [rows, n_spk] each."""
        n = len(sids)
        flat, offs = pack(chunks, np.float32, offs_dtype=np.int64)
        ids = np.asarray(list(sids), np.int32)
        rows = np.zeros(n + 1, np.int32)
        out = np.zeros((n * 32, self.dims.n_spk), np.float32)
        L.check(self.lib.wlk_sf_step_audio(self.h, _ptr(ids), n, _ptr(flat), _ptr(offs), _ptr(out) if want_preds else None, _ptr(rows)))
        return split(out, rows) if want_preds else [rows[i + 1] - rows[i] for i in range(n)]

    def step_features(self, sids: Sequence[int], feats: Sequence[np.ndarray], left_offset: int, right_offset: int) -> List[np.ndarray]:
        """forward_streaming_step for n streams: time-major features [frames, n_mels] each."""
        n = len(sids)
        flat, offs = pack(feats, np.float32, (self.dims.n_mels,))
        ids = np.asarray(list(sids), np.int32)
        rows = np.zeros(n + 1, np.int32)
        out = np.zeros((n * 32, self.dims.n_spk), np.float32)
        L.check(self.lib.wlk_sf_step_features(self.h, _ptr(ids), n, _ptr(flat), _ptr(offs), int(left_offset), int(right_offset),
                                              _ptr(out), _ptr(rows)))
        return split(out, rows)

    def total_preds(self, sid: int):
        """(device address of the stream's total_preds [rows, n_spk], rows)"""
        p, r = C.c_void_p(), C.c_int32()
        L.check(self.lib.wlk_sf_total_preds(self.h, sid, C.byref(p), C.byref(r)))
        return p.value, r.value

    def read_state(self, sid: int) -> dict:
        d = self.dims
        lengths = np.zeros(4, np.int32)
        cache = np.zeros((d.spkcache_len, d.d_model), np.float32)
        cpreds = np.zeros((d.spkcache_len, d.n_spk), np.float32)
        fifo = np.zeros((d.fifo_len, d.d_model), np.float32)
        msil = np.zeros(d.d_model, np.float32)
        L.check(self.lib.wlk_sf_read_state(self.h, sid, _ptr(lengths), _ptr(cache), _ptr(cpreds), _ptr(fifo), _ptr(msil)))
        return dict(spkcache_len=int(lengths[0]), fifo_len=int(lengths[1]), n_sil=int(lengths[2]), chunk_index=int(lengths[3]),
                    spkcache=cache, spkcache_preds=cpreds, fifo=fifo, mean_sil_emb=msil)


# ---------------------------------------------------------------------------------------------------------------
# the diarization seam
# ---------------------------------------------------------------------------------------------------------------
class B200SortformerDiarization:
    """Shared model object (``SortformerDiarization``, sortformer_backend.py:55-128): one engine per process / GPU."""

    def __init__(self, dims: SortformerDims, state_dict: Dict[str, np.ndarray], *, precision: str = "bf16", device: int = 0,
                 max_sessions: int = 64, max_batch: int = 64):
        self.engine = SortformerEngine(dims, state_dict, precision=precision, device=device, max_sessions=max_sessions,
                                       max_batch=max_batch)
        self.dims = dims

    def close(self):
        self.engine.close()


class B200SortformerDiarizationOnline:
    """Per-connection object with the surface ``audio_processor.py`` uses (sortformer_backend.py:151-373)."""

    def __init__(self, shared_model: B200SortformerDiarization, sample_rate: int = 16000, max_speakers: Optional[int] = None):
        self.sample_rate = sample_rate
        self.engine = shared_model.engine
        d = shared_model.dims
        self.max_speakers = resolve_max_speakers(max_speakers, int(d.n_spk))
        self.buffer_audio = np.array([], dtype=np.float32)
        self.segment_lock = threading.Lock()
        self.debug = False
        self.audio_buffer: List[np.ndarray] = []
        self.chunk_duration_seconds = self.engine.chunk_duration_seconds
        self.sid = self.engine.open_session()
        self._seg = DiarizationSegmenter(d.n_spk, self.chunk_duration_seconds, self.max_speakers, device=self.engine.device)
        self.diarization_segments: List[SpeakerSegment] = []

    @property
    def global_time_offset(self) -> float:
        return self._seg.global_time_offset

    @property
    def _chunk_index(self) -> int:
        return self._seg._chunk_index

    def insert_silence(self, silence_duration: Optional[float]):
        with self.segment_lock:
            self._seg.insert_silence(silence_duration)

    def insert_audio_chunk(self, pcm_array: np.ndarray):
        if self.debug:
            self.audio_buffer.append(pcm_array.copy())
        self.buffer_audio = np.concatenate([self.buffer_audio, np.asarray(pcm_array, np.float32)])

    def _take_chunk(self) -> Optional[np.ndarray]:
        threshold = int(self.chunk_duration_seconds * self.sample_rate)                    # :261
        if len(self.buffer_audio) < threshold:
            return None
        audio = self.buffer_audio[:threshold]
        self.buffer_audio = self.buffer_audio[threshold:]
        return audio

    async def diarize(self) -> List[SpeakerSegment]:
        audio = self._take_chunk()
        if audio is None:
            return []
        return diarize_batch([self], [audio])[0]

    def get_segments(self) -> List[SpeakerSegment]:
        with self.segment_lock:
            return self.diarization_segments.copy()

    def close(self):
        if self.sid is not None:
            try:
                self.engine.close_session(self.sid)
            finally:
                self.sid = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def diarize_batch(onlines: Sequence[B200SortformerDiarizationOnline], chunks: Sequence[np.ndarray]) -> List[List[SpeakerSegment]]:
    """One device step for many connections of the same engine (what a batching host calls instead of n ``diarize()``s):
    forward + cache update, then the run-length kernel over each stream's device-resident total_preds."""
    eng = onlines[0].engine
    sids = [o.sid for o in onlines]
    eng.step_audio(sids, chunks, want_preds=False)
    ptrs, rows = zip(*[eng.total_preds(s) for s in sids])
    for o in onlines:
        o.segment_lock.acquire()
    try:
        return DiarizationSegmenter.process_batch([o._seg for o in onlines], list(ptrs), list(rows))
    finally:
        for o in onlines:
            o.segment_lock.release()
