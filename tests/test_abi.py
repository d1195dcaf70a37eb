"""CPU: the C-ABI library builds/loads and exports every symbol include/wlk_b200.h declares;
the product path fails loudly without a GPU (no CPU fallback)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "wlk_b200.h")).read()
    return sorted(set(re.findall(r"\b(wlk_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from whisperlivekit_b200.build import build
    build()
    from whisperlivekit_b200 import _lib
    lib = _lib.load()
    syms = header_symbols()
    assert len(syms) >= 35
    for s in syms:
        assert hasattr(lib, s), s
        assert s in _lib.SIGNATURES, f"{s} has no ctypes signature"
    assert lib.wlk_abi_version() == 1


def test_engine_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from whisperlivekit_b200 import _lib
    from whisperlivekit_b200.dims import DIMS
    from whisperlivekit_b200.engine import WhisperEngine
    with pytest.raises(_lib.WlkError, match="no CPU fallback"):
        WhisperEngine(DIMS["micro"], None, [(0, 0)])


BAD_DEVICE = 99


def _qwen():
    from whisperlivekit_b200.qwen_dims import QWEN_DIMS
    from whisperlivekit_b200.qwen_engine import QwenTowerEngine
    QwenTowerEngine(QWEN_DIMS["qnano"], device=BAD_DEVICE)


def _qtext():
    from whisperlivekit_b200.qwen_dims import QWEN_TEXT_DIMS
    from whisperlivekit_b200.qwen_text_engine import QwenTextEngine
    QwenTextEngine(QWEN_TEXT_DIMS["tnano"], device=BAD_DEVICE)


def _sortformer():
    from whisperlivekit_b200.sortformer_dims import SORTFORMER_DIMS
    from whisperlivekit_b200.sortformer_engine import SortformerEngine
    SortformerEngine(SORTFORMER_DIMS["micro"], device=BAD_DEVICE)


def _vad():
    from whisperlivekit_b200.vad import VadEngine
    VadEngine({}, device=BAD_DEVICE)


def _diar():
    from whisperlivekit_b200.diarization import diar_segments
    diar_segments([0], [0], [0], n_spk=1, max_speakers=1, device=BAD_DEVICE)


@pytest.mark.parametrize("entry", [_qwen, _qtext, _sortformer, _vad, _diar], ids=["qwen", "qtext", "sortformer", "vad", "diar"])
def test_entry_point_rejects_unusable_device(entry):
    """Every C-ABI unit opens its device through the same checks and reports the failure through the same guard:
    without a GPU there is no CPU fallback, and with one a device index past the last is refused."""
    import torch
    from whisperlivekit_b200 import _lib
    want = f"device {BAD_DEVICE} out of range" if torch.cuda.is_available() else "no CPU fallback"
    with pytest.raises(_lib.WlkError, match=want):
        entry()


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "whisperlivekit_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            src = open(os.path.join(pkg, fn)).read()
            assert "import oracle" not in src and "from oracle" not in src, fn
