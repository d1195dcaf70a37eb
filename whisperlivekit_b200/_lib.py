"""ctypes binding of include/wlk_b200.h (the C-ABI boundary).

There is no CPU fallback: if the in-tree library is missing this raises, and
``wlk_engine_create`` itself fails when no sm_90 device is present.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "csrc", "libwlk_b200.so")


class wlk_dims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "n_mels", "n_audio_ctx", "n_audio_state", "n_audio_head", "n_audio_layer",
        "n_vocab", "n_text_ctx", "n_text_state", "n_text_head", "n_text_layer")]


class wlk_qwen_dims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "n_mels", "conv_channels", "d_model", "n_head", "n_layer", "ffn_dim", "out_dim", "max_positions",
        "chunk_frames", "block_frames", "left_context_steps", "block_bidirectional", "conv_out_bias", "mutable_tail_steps")]


class wlk_qwen_window_dims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "n_mels", "conv_channels", "d_model", "n_head", "n_layer", "ffn_dim", "out_dim", "max_positions", "conv_out_bias",
        "n_window", "n_window_infer", "left_context_frames", "right_context_frames")]


class wlk_qtext_dims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "vocab", "d_model", "n_layer", "n_head", "n_kv_head", "head_dim", "ffn_dim", "tied", "max_ctx")] + [
        (n, C.c_float) for n in ("rope_theta", "rms_eps")]


class wlk_sf_dims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "n_mels", "n_fft", "win_length", "hop", "conv_channels", "d_model", "n_head", "n_layer", "ff_mult", "conv_kernel",
        "tf_d_model", "tf_n_head", "tf_n_layer", "tf_inner", "n_spk", "spkcache_len", "fifo_len", "spkcache_update_period",
        "chunk_len", "subsampling_factor", "encoder_subsampling", "spkcache_sil_frames_per_spk")] + [(n, C.c_float) for n in (
        "pred_score_threshold", "scores_boost_latest", "sil_threshold", "strong_boost_rate", "weak_boost_rate",
        "min_pos_scores_rate")]


class wlk_config(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "device", "precision", "max_sessions", "max_batch", "gemm_backend", "attn_backend",
        "max_align_heads", "reserved")]


PREC_FP32, PREC_BF16, PREC_BF16X3, PREC_FP8 = 0, 1, 2, 3
BACKEND_AUTO, BACKEND_SIMT, BACKEND_TCGEN05 = 0, 1, 2
PRECISIONS = {"fp32": PREC_FP32, "bf16": PREC_BF16, "bf16x3": PREC_BF16X3, "fp8": PREC_FP8}
BACKENDS = {"auto": BACKEND_AUTO, "simt": BACKEND_SIMT, "tcgen05": BACKEND_TCGEN05}
KERNEL_CLASSES = ["mel", "gemm_enc", "attn_enc", "layernorm", "gemm_xkv", "gemm_dec",
                  "attn_dec_self", "attn_dec_cross", "logits", "align", "misc"]

_i32p = C.POINTER(C.c_int32)
_f32p = C.POINTER(C.c_float)
_i64p = C.POINTER(C.c_int64)
_vp = C.c_void_p

# name -> (restype, argtypes); every symbol declared in include/wlk_b200.h
SIGNATURES = {
    "wlk_last_error": (C.c_char_p, []),
    "wlk_abi_version": (C.c_int, []),
    "wlk_engine_create": (C.c_int, [C.POINTER(wlk_dims), C.POINTER(wlk_config), C.POINTER(_vp)]),
    "wlk_engine_destroy": (C.c_int, [_vp]),
    "wlk_engine_load_tensor": (C.c_int, [_vp, C.c_char_p, _vp, _i64p, C.c_int]),
    "wlk_engine_finalize_weights": (C.c_int, [_vp]),
    "wlk_engine_weight_blob": (C.c_int, [_vp, C.POINTER(_vp), C.POINTER(C.c_size_t)]),
    "wlk_engine_adopt_weights": (C.c_int, [_vp]),
    "wlk_engine_set_alignment_heads": (C.c_int, [_vp, _i32p, C.c_int]),
    "wlk_engine_stream": (C.c_int, [_vp, C.POINTER(_vp)]),
    "wlk_engine_sync": (C.c_int, [_vp]),
    "wlk_engine_memory": (C.c_int, [_vp, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    "wlk_session_open": (C.c_int, [_vp, _i32p]),
    "wlk_session_close": (C.c_int, [_vp, C.c_int32]),
    "wlk_session_append_audio": (C.c_int, [_vp, C.c_int32, _vp, C.c_int64]),
    "wlk_session_drop_audio": (C.c_int, [_vp, C.c_int32, C.c_int64]),
    "wlk_session_clear_audio": (C.c_int, [_vp, C.c_int32]),
    "wlk_session_audio_len": (C.c_int, [_vp, C.c_int32, _i64p]),
    "wlk_session_reset_decoder": (C.c_int, [_vp, C.c_int32]),
    "wlk_qwen_create": (C.c_int, [_vp, _vp, _vp]),
    "wlk_qwen_destroy": (C.c_int, [_vp]),
    "wlk_qwen_load_tensor": (C.c_int, [_vp, C.c_char_p, _vp, _vp, C.c_int]),
    "wlk_qwen_finalize_weights": (C.c_int, [_vp]),
    "wlk_qwen_memory": (C.c_int, [_vp, _vp, _vp, _vp]),
    "wlk_qwen_session_open": (C.c_int, [_vp, _vp]),
    "wlk_qwen_session_close": (C.c_int, [_vp, C.c_int32]),
    "wlk_qwen_session_reset": (C.c_int, [_vp, C.c_int32]),
    "wlk_qwen_session_state": (C.c_int, [_vp, C.c_int32, _vp, _vp]),
    "wlk_qwen_session_mutable_steps": (C.c_int, [_vp, C.c_int32, _vp]),
    "wlk_qwen_forward_chunk": (C.c_int, [_vp, _vp, C.c_int, _vp, _vp, _vp, C.c_int64, _vp]),
    "wlk_qwen_append_audio": (C.c_int, [_vp, _vp, C.c_int, _vp, _vp, _vp, C.c_int64, _vp, C.c_int32]),
    "wlk_qwen_flush_pending": (C.c_int, [_vp, _vp, C.c_int, _vp, C.c_int64, _vp]),
    "wlk_qwen_forward_chunk_device": (C.c_int, [_vp, _vp, C.c_int, _vp, _vp, _vp, C.c_int64, _vp]),
    "wlk_qwen_flush_pending_device": (C.c_int, [_vp, _vp, C.c_int, _vp, C.c_int64, _vp]),
    "wlk_qwen_session_get_pending": (C.c_int, [_vp, C.c_int32, _vp, C.c_int64, _vp]),
    "wlk_qwen_session_set_pending": (C.c_int, [_vp, C.c_int32, _vp, C.c_int32]),
    "wlk_qwen_window_create": (C.c_int, [_vp, _vp, _vp]),
    "wlk_qwen_window_forward": (C.c_int, [_vp, _vp, C.c_int, _vp, _vp, _vp, C.c_int64, _vp, C.c_int32]),
    "wlk_qwen_window_encode": (C.c_int, [_vp, C.c_int, _vp, _vp, _vp, C.c_int64, _vp]),
    "wlk_qwen_window_state": (C.c_int, [_vp, C.c_int32, _vp]),
    "wlk_qwen_window_attention": (C.c_int, [C.c_int, C.c_int, _vp, _vp, C.c_int, _vp, C.c_int, C.c_int]),
    "wlk_qwen_op_positions": (C.c_int, [_vp, _vp, C.c_int32, _vp]),
    "wlk_qwen_op_conv_stem": (C.c_int, [_vp, _vp, _vp, _vp, C.c_int32, _vp, _vp, _vp]),
    "wlk_qwen_op_qkv": (C.c_int, [_vp, C.c_int32, _vp, _vp, _vp, C.c_int32, _vp, C.c_int32, _vp]),
    "wlk_qwen_op_attention": (C.c_int, [_vp, C.c_int32, _vp, _vp, _vp, C.c_int32, _vp, _vp]),
    "wlk_qtext_create": (C.c_int, [_vp, _vp, _vp]),
    "wlk_qtext_destroy": (C.c_int, [_vp]),
    "wlk_qtext_load_tensor": (C.c_int, [_vp, C.c_char_p, _vp, _vp, C.c_int]),
    "wlk_qtext_finalize_weights": (C.c_int, [_vp]),
    "wlk_qtext_memory": (C.c_int, [_vp, _vp, _vp, _vp]),
    "wlk_qtext_session_open": (C.c_int, [_vp, _vp]),
    "wlk_qtext_session_close": (C.c_int, [_vp, C.c_int32]),
    "wlk_qtext_session_reset": (C.c_int, [_vp, C.c_int32]),
    "wlk_qtext_session_len": (C.c_int, [_vp, C.c_int32, _vp]),
    "wlk_qtext_crop": (C.c_int, [_vp, C.c_int32, C.c_int32]),
    "wlk_qtext_forward": (C.c_int, [_vp, _vp, C.c_int, _vp, _vp, _vp, C.c_int32, _vp]),
    "wlk_qtext_forward_device": (C.c_int, [_vp, _vp, C.c_int, _vp, _vp, _vp, C.c_int64, C.c_int32, _vp]),
    "wlk_qtext_adapt": (C.c_int, [_vp, _vp, C.c_int32, C.c_int64, _vp, C.c_int64]),
    "wlk_qtext_adapter_dims": (C.c_int, [_vp, _vp, _vp, _vp]),
    "wlk_qtext_pick": (C.c_int, [_vp, _vp, C.c_int32, _vp, _vp, _vp, C.c_int32, C.c_float, C.c_int32, C.c_int32,
                                 C.c_int32, _vp, _vp]),
    "wlk_qtext_generate_full": (C.c_int, [_vp, _vp, C.c_int32, _vp, _vp, _vp, C.c_int64, C.c_int32, C.c_int32, _vp,
                                          C.c_int32, _vp, C.c_int32, C.c_float, C.c_int32, C.c_int32, C.c_int32, _vp, _vp]),
    "wlk_qtext_generate_rolling": (C.c_int, [_vp, _vp, C.c_int32, _vp, _vp, _vp, C.c_int64, C.c_int32, _vp, _vp, C.c_int32,
                                             C.c_int32, _vp, C.c_int32, _vp, C.c_int32, C.c_float, C.c_int32, C.c_int32,
                                             C.c_int32, _vp, _vp, _vp]),
    "wlk_qtext_logits": (C.c_int, [_vp, C.c_int32, C.c_int32, _vp]),
    "wlk_qtext_op_rmsnorm": (C.c_int, [_vp, _vp, _vp, _vp, C.c_int32, _vp]),
    "wlk_qtext_op_qk_rope": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, C.c_int32, _vp, C.c_int32, C.c_int32, _vp]),
    "wlk_qtext_op_attention": (C.c_int, [_vp, _vp, _vp, _vp, C.c_int32, _vp, C.c_int32, C.c_int32, _vp]),
    "wlk_qtext_op_swiglu": (C.c_int, [_vp, _vp, _vp, C.c_int32]),
    "wlk_select": (C.c_int, [_vp, _vp, C.c_int, _vp, C.c_int, _vp, C.c_int, _vp, _vp, _vp, _vp, C.c_int32, _vp, _vp, _vp]),
    "wlk_vad_create": (C.c_int, [C.c_int, C.c_int, _vp]),
    "wlk_vad_destroy": (C.c_int, [_vp]),
    "wlk_vad_load_tensor": (C.c_int, [_vp, C.c_char_p, _vp, C.c_int64]),
    "wlk_vad_session_open": (C.c_int, [_vp, _vp]),
    "wlk_vad_session_reset": (C.c_int, [_vp, C.c_int32]),
    "wlk_vad_session_close": (C.c_int, [_vp, C.c_int32]),
    "wlk_vad_forward": (C.c_int, [_vp, _vp, C.c_int, _vp, _vp, _vp]),
    "wlk_sf_create": (C.c_int, [_vp, _vp, _vp]),
    "wlk_sf_destroy": (C.c_int, [_vp]),
    "wlk_sf_load_tensor": (C.c_int, [_vp, C.c_char_p, _vp, _vp, C.c_int]),
    "wlk_sf_finalize_weights": (C.c_int, [_vp]),
    "wlk_sf_session_open": (C.c_int, [_vp, _vp]),
    "wlk_sf_session_close": (C.c_int, [_vp, C.c_int32]),
    "wlk_sf_session_reset": (C.c_int, [_vp, C.c_int32]),
    "wlk_sf_step_audio": (C.c_int, [_vp, _vp, C.c_int, _vp, _vp, _vp, _vp]),
    "wlk_sf_step_features": (C.c_int, [_vp, _vp, C.c_int, _vp, _vp, C.c_int32, C.c_int32, _vp, _vp]),
    "wlk_sf_total_preds": (C.c_int, [_vp, C.c_int32, _vp, _vp]),
    "wlk_sf_read_state": (C.c_int, [_vp, C.c_int32, _vp, _vp, _vp, _vp, _vp]),
    "wlk_sf_memory": (C.c_int, [_vp, _vp, _vp, _vp]),
    "wlk_diar_segments": (C.c_int, [C.c_int, _vp, _vp, _vp, C.c_int, C.c_int, C.c_int, _vp, _vp, C.c_int]),
    "wlk_session_append_pcm16": (C.c_int, [_vp, C.c_int32, _vp, C.c_int64]),
    "wlk_session_fork": (C.c_int, [_vp, C.c_int32, _vp]),
    "wlk_sessions_gather_decoder": (C.c_int, [_vp, _vp, _vp, C.c_int]),
    "wlk_encode": (C.c_int, [_vp, _vp, C.c_int, _vp]),
    "wlk_encode_incremental": (C.c_int, [_vp, _vp, C.c_int, _vp, _vp]),
    "wlk_session_reset_incremental": (C.c_int, [_vp, C.c_int32]),
    "wlk_decode": (C.c_int, [_vp, _vp, C.c_int, _vp, _vp, C.c_int32]),
    "wlk_encode_mel": (C.c_int, [_vp, C.c_int32, _vp, C.c_int32]),
    "wlk_decode_all_logits": (C.c_int, [_vp, C.c_int32, _vp, C.c_int, C.c_int32, _vp]),
    "wlk_read_align_rows": (C.c_int, [_vp, C.c_int32, _vp, C.c_int64, _i32p, _i32p]),
    "wlk_no_speech_prob": (C.c_int, [_vp, _vp, C.c_int, _vp]),
    "wlk_suppress": (C.c_int, [_vp, _vp, C.c_int, _vp, C.c_int]),
    "wlk_add_logit_bias": (C.c_int, [_vp, C.c_int32, _vp, _vp, C.c_int]),
    "wlk_greedy_and_align": (C.c_int, [_vp, _vp, C.c_int, C.c_int32, _vp, _vp, _vp]),
    "wlk_read_mel": (C.c_int, [_vp, C.c_int32, _vp]),
    "wlk_read_encoder": (C.c_int, [_vp, C.c_int32, _vp]),
    "wlk_read_logits": (C.c_int, [_vp, C.c_int32, C.c_int32, _vp]),
    "wlk_read_align_attn": (C.c_int, [_vp, C.c_int32, _vp, C.c_int64, _i32p, _i32p]),
    "wlk_op_gemm": (C.c_int, [_vp, C.c_int, _vp, C.c_int, C.c_int64, _vp, C.c_int, C.c_int64, _vp,
                              _vp, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int]),
    "wlk_op_encoder_attention": (C.c_int, [_vp, C.c_int, _vp, C.c_int, C.c_int, _vp]),
    "wlk_op_gemm_fp8": (C.c_int, [_vp, C.c_int, _vp, _vp, C.c_int64, _vp, _vp, C.c_int64, _vp, C.c_float, C.c_int,
                                  _vp, C.c_int, _vp, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int]),
    "wlk_op_quantize_rows": (C.c_int, [_vp, _vp, C.c_int, C.c_int64, C.c_int, C.c_int, _vp, C.c_int64, _vp]),
    "wlk_op_layernorm_fp8": (C.c_int, [_vp, _vp, C.c_int64, _vp, _vp, C.c_int, C.c_int, _vp, C.c_int64, _vp, _vp,
                                       C.c_float, C.c_float]),
    "wlk_op_median_filter": (C.c_int, [_vp, _vp, _vp, C.c_int, C.c_int, C.c_int]),
    "wlk_op_dtw": (C.c_int, [_vp, _vp, C.c_int, C.c_int, _vp, _vp, _i32p]),
    "wlk_timer_record": (C.c_int, [_vp, C.c_int]),
    "wlk_timer_elapsed_ms": (C.c_int, [_vp, C.c_int, C.c_int, _f32p]),
    "wlk_profile_enable": (C.c_int, [_vp, C.c_int]),
    "wlk_profile_reset": (C.c_int, [_vp]),
    "wlk_profile_read": (C.c_int, [_vp, C.c_int, C.POINTER(C.c_double), _i64p, C.POINTER(C.c_double),
                                   C.POINTER(C.c_double)]),
    "wlk_profile_class_name": (C.c_int, [C.c_int, C.POINTER(C.c_char_p)]),
}

_lib = None


class WlkError(RuntimeError):
    pass


def load():
    """Load csrc/libwlk_b200.so (built by whisperlivekit_b200.build / __graft_entry__.build)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise WlkError(
            f"{LIB_PATH} is missing: build it with `python -m whisperlivekit_b200.build` "
            "(nvcc, sm_90a). The H100 engine has no CPU or PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if lib.wlk_abi_version() != 1:
        raise WlkError("ABI version mismatch")
    _lib = lib
    return lib


def check(rc: int):
    if rc != 0:
        raise WlkError(load().wlk_last_error().decode("utf-8", "replace"))


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def pack(parts, dtype, shape=(), offs_dtype=np.int32):
    """Per-stream arrays -> (their rows [*shape] of ``dtype`` back to back, offsets [n + 1] of ``offs_dtype``): stream i
    is flat[offs[i]: offs[i + 1]].  Without any row, flat is one zero row, so the engine is never handed a null pointer."""
    parts = [np.ascontiguousarray(p, dtype).reshape(-1, *shape) for p in parts]
    offs = np.zeros(len(parts) + 1, offs_dtype)
    offs[1:] = np.cumsum([p.shape[0] for p in parts])
    flat = np.concatenate(parts) if offs[-1] else np.zeros((1, *shape), dtype)
    return flat, offs


def split(out: np.ndarray, offs):
    """Per-stream copies of the rows of ``out``: stream i owns rows offs[i] .. offs[i + 1]."""
    return [out[offs[i]: offs[i + 1]].copy() for i in range(len(offs) - 1)]


class Engine:
    """One engine handle of the library: create, weights, memory, sessions and one destroy.

    A subclass names its entry points as the class data below, each ``wlk_*`` name in full; where the library has no
    such entry point, the subclass sets the method that would call it to None.  ``close`` destroys the
    handle once and sets ``h`` to None: a later call reaches the library as a null handle, which every entry point
    refuses ("null engine"), instead of a pointer into the freed engine."""

    CREATE = DESTROY = LOAD_TENSOR = FINALIZE = MEMORY = SESSION_OPEN = SESSION_CLOSE = SESSION_RESET = None
    precisions = ("fp32", "bf16")                         # the precision names the engine takes
    h = None

    def _create_handle(self, device: int, *args) -> None:
        """h = CREATE(*args, &h) for an engine on ``device``."""
        self.lib = load()
        self.device = int(device)
        h = C.c_void_p()
        check(getattr(self.lib, self.CREATE)(*args, C.byref(h)))
        self.h = h

    def _create(self, cdims, *, precision: str, device: int, max_sessions: int, max_batch: int, gemm_backend: str = "auto",
                attn_backend: str = "simt", max_align_heads: int = 0) -> None:
        """CREATE(&cdims, &config) with the config built from the precision and backend names."""
        if precision not in self.precisions:
            raise KeyError(precision)
        cfg = wlk_config(device=device, precision=PRECISIONS[precision], max_sessions=max_sessions, max_batch=max_batch,
                         gemm_backend=BACKENDS[gemm_backend], attn_backend=BACKENDS[attn_backend],
                         max_align_heads=max_align_heads, reserved=0)
        self.precision = precision
        self.max_batch = int(max_batch)
        self._create_handle(device, C.byref(cdims), C.byref(cfg))

    def close(self) -> None:
        h, self.h = self.h, None
        if h is not None:
            check(getattr(self.lib, self.DESTROY)(h))

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- weights ------------------------------------------------------------------------------------------------------
    def load_tensor(self, name: str, arr) -> None:
        a = np.ascontiguousarray(arr, np.float32)
        shape = (C.c_int64 * a.ndim)(*a.shape)
        check(getattr(self.lib, self.LOAD_TENSOR)(self.h, name.encode(), _ptr(a), shape, a.ndim))

    def finalize(self) -> None:
        check(getattr(self.lib, self.FINALIZE)(self.h))

    @staticmethod
    def _skip(name: str, arr) -> bool:
        """Whether load_state_dict leaves this checkpoint entry out."""
        return False

    def load_state_dict(self, sd) -> None:
        for name, arr in sd.items():
            if not self._skip(name, arr):
                self.load_tensor(name, arr)
        self.finalize()

    def memory(self) -> dict:
        w, s, k = C.c_size_t(), C.c_size_t(), C.c_size_t()
        check(getattr(self.lib, self.MEMORY)(self.h, C.byref(w), C.byref(s), C.byref(k)))
        return dict(weights=w.value, sessions=s.value, workspace=k.value)

    # -- sessions -----------------------------------------------------------------------------------------------------
    def open_session(self) -> int:
        sid = C.c_int32()
        check(getattr(self.lib, self.SESSION_OPEN)(self.h, C.byref(sid)))
        return sid.value

    def close_session(self, sid: int) -> None:
        if self.h is None:          # destroyed first (a session handle collected in the same garbage cycle): its
            return                  # sessions went with it
        check(getattr(self.lib, self.SESSION_CLOSE)(self.h, int(sid)))

    def reset_session(self, sid: int) -> None:
        check(getattr(self.lib, self.SESSION_RESET)(self.h, int(sid)))
