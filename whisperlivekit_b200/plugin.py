"""Registration of the H100 engine behind WhisperLiveKit's SimulStreaming/AlignAtt seam.

Needs WhisperLiveKit importable (it is not a dependency of the engine itself).  Nothing in
WhisperLiveKit is modified on disk: ``install()`` swaps the ``AlignAtt`` symbol that
``SimulStreamingOnlineProcessor._create_alignatt`` instantiates
(reference simul_whisper/backend.py:61-71) and wraps ``SimulStreamingASR.load_model``
(backend.py:530-553) so the weights it loads are packed into a ``WhisperEngine``.
``core.py``, the AlignAtt policy (``AlignAttBase.infer``), ``SimulStreamingOnlineProcessor`` and
``tokens_alignment.py`` run unchanged.  See INTEGRATION.md.
"""
from __future__ import annotations


from .dims import ModelDimensions
from .weights import state_dict_from_torch


class B200WhisperModel:
    """What AlignAttBase / SimulStreamingASR read from ``shared_model``:
    ``dims``, ``len(decoder.blocks)``, ``num_languages``, ``is_multilingual``, ``device``."""

    class _Decoder:
        def __init__(self, n):
            self.blocks = [None] * n

    def __init__(self, engine):
        self.engine = engine
        self.dims = engine.dims
        self.decoder = self._Decoder(engine.dims.n_text_layer)
        self.device = "cpu"                      # host-side token tensors live on the CPU

    @property
    def is_multilingual(self):
        return self.dims.is_multilingual

    @property
    def num_languages(self):
        return self.dims.num_languages


def engine_from_torch_whisper(model, *, precision="bf16", device=0, max_sessions=64, max_batch=64, **kw):
    """Pack a loaded reference ``Whisper`` module (whisper/model.py:335) into a WhisperEngine."""
    from .engine import WhisperEngine
    d = model.dims
    dims = ModelDimensions(d.n_mels, d.n_audio_ctx, d.n_audio_state, d.n_audio_head, d.n_audio_layer,
                           d.n_vocab, d.n_text_ctx, d.n_text_state, d.n_text_head, d.n_text_layer)
    heads = [(int(l), int(h)) for l, h in model.alignment_heads.indices().T]      # simul_whisper.py:151-159
    return WhisperEngine(dims, state_dict_from_torch(model.state_dict()), heads, precision=precision,
                         device=device, max_sessions=max_sessions, max_batch=max_batch, **kw)


def make_b200_alignatt_class():
    """class B200AlignAtt(AlignAttHooks, AlignAttBase): the reference's template infer() over our hooks."""
    from whisperlivekit.simul_whisper.align_att_base import AlignAttBase
    from .alignatt import AlignAttHooks

    class B200AlignAtt(AlignAttHooks, AlignAttBase):
        pass

    return B200AlignAtt


def install(precision: str = "bf16", device: int = 0, max_sessions: int = 64, max_batch: int = 64,
            batching: bool = True, max_wait_s: float = 0.002, engine_factory=None, incremental_encoder: bool = False):
    """Route WhisperLiveKit's SimulStreaming backend through the H100 engine (call once, before
    TranscriptionEngine is constructed).  With ``batching`` the per-session calls of the worker threads
    (audio_processor.py:543-551) are coalesced into batched C-ABI calls by batching.BatchingEngine.

    ``engine_factory(torch_whisper) -> engine`` replaces the construction of the CUDA engine; the CPU tests pass the
    oracle engine through it so that the registration itself (the symbols swapped below) is exercised without a GPU.
    Returns the B200AlignAtt class; ``uninstall()`` restores the reference's symbols."""
    import whisperlivekit.simul_whisper.backend as be
    cls = make_b200_alignatt_class()
    if not hasattr(be, "_b200_saved"):
        be._b200_saved = (be.AlignAtt, be.SimulStreamingASR.load_model, be.SimulStreamingOnlineProcessor.__del__)
    be.AlignAtt = cls                                   # what _create_alignatt instantiates (backend.py:61-71)
    orig_load = be._b200_saved[1]

    def load_model(self, *a, **k):                      # backend.py:530-553
        torch_model = orig_load(self, *a, **k)
        if engine_factory is not None:
            eng = engine_factory(torch_model)
        else:
            eng = engine_from_torch_whisper(torch_model, precision=precision, device=device,
                                            max_sessions=max_sessions, max_batch=max_batch)
            # the labelled approximate mode (engine.encode docstring): retained encoder K/V, ~29 positions per chunk
            eng.incremental_encoder = bool(incremental_encoder)
        if batching:
            from .batching import BatchingEngine
            eng = BatchingEngine(eng, max_batch=max_batch, max_wait_s=max_wait_s)
        return B200WhisperModel(eng)

    orig_del = be._b200_saved[2]

    def processor_del(self):                            # backend.py:284-290: the session's device state dies with it
        try:
            model = getattr(self, "model", None)
            if model is not None and hasattr(model, "close"):
                model.close()
        finally:
            orig_del(self)

    be.SimulStreamingASR.load_model = load_model
    be.SimulStreamingOnlineProcessor.__del__ = processor_del
    return cls


def uninstall():
    import whisperlivekit.simul_whisper.backend as be
    if hasattr(be, "_b200_saved"):
        be.AlignAtt, be.SimulStreamingASR.load_model, be.SimulStreamingOnlineProcessor.__del__ = be._b200_saved
        del be._b200_saved


# ---------------------------------------------------------------------------------------------------------------
# diarization seam (SURVEY.md section 8b item 3)
# ---------------------------------------------------------------------------------------------------------------
def sortformer_state_dict_from_nemo(path: str):
    """Weights of a ``.nemo`` checkpoint (a tar archive holding ``model_weights.ckpt``, a plain torch state_dict under
    NeMo's parameter names) as numpy arrays -- read without NeMo."""
    import io
    import tarfile

    import torch
    with tarfile.open(path, "r:*") as tar:
        member = next(m for m in tar.getmembers() if m.name.endswith("model_weights.ckpt"))
        blob = tar.extractfile(member).read()
    sd = torch.load(io.BytesIO(blob), map_location="cpu", weights_only=True)
    return {k: v.detach().float().cpu().numpy() for k, v in sd.items()}


def install_sortformer(state_dict=None, dims=None, precision: str = "bf16", device: int = 0, max_sessions: int = 64,
                       max_batch: int = 64):
    """Route ``--diarization-backend sortformer`` through the H100 engine without editing WhisperLiveKit: core.py imports
    ``SortformerDiarization`` / ``SortformerDiarizationOnline`` from ``whisperlivekit.diarization.sortformer_backend``
    (core.py:297-299, 472-477), a module that exits at import when NeMo is missing (sortformer_backend.py:14-22).  This
    puts a module of that name in ``sys.modules`` whose two classes are the H100 drop-ins, with the reference's constructor
    signatures (``SortformerDiarization(model_name=..., model_path=...)``, ``SortformerDiarizationOnline(shared_model,
    sample_rate, max_speakers)``).  Weights: ``state_dict`` (NeMo names), else ``model_path`` must point at a ``.nemo``."""
    import sys
    import types

    from .sortformer_dims import SORTFORMER_DIMS
    from .sortformer_engine import B200SortformerDiarization, B200SortformerDiarizationOnline
    d = dims or SORTFORMER_DIMS["diar_streaming_sortformer_4spk-v2"]

    class SortformerDiarization(B200SortformerDiarization):
        def __init__(self, model_name: str = "nvidia/diar_streaming_sortformer_4spk-v2", model_path=None):
            sd = state_dict
            if sd is None:
                if not model_path:
                    raise FileNotFoundError("no network on this host: pass --sortformer-model-path <file.nemo> "
                                            f"(cannot download {model_name})")
                sd = sortformer_state_dict_from_nemo(model_path)
            super().__init__(d, sd, precision=precision, device=device, max_sessions=max_sessions, max_batch=max_batch)

    mod = types.ModuleType("whisperlivekit.diarization.sortformer_backend")
    mod.SortformerDiarization = SortformerDiarization
    mod.SortformerDiarizationOnline = B200SortformerDiarizationOnline
    mod.__b200__ = True
    sys.modules["whisperlivekit.diarization.sortformer_backend"] = mod
    return mod


def uninstall_sortformer():
    import sys
    m = sys.modules.get("whisperlivekit.diarization.sortformer_backend")
    if m is not None and getattr(m, "__b200__", False):
        del sys.modules["whisperlivekit.diarization.sortformer_backend"]
