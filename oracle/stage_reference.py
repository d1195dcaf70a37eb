#!/usr/bin/env python
"""Stage the UNMODIFIED reference (QuentinFuxa/WhisperLiveKit, pure Python) under oracle/_ref/ so that its own
CPU backend -- the vendored torch Whisper behind ``AlignAtt`` (``--backend whisper``) -- can be timed on the host
cores next to the GPU engine (``bench.py --impl reference`` and the ``cpu_baseline`` leg), and so that the tests
marked ``reference`` can drive the original code from inside the repository tree.

    python oracle/stage_reference.py          # needs a checkout of the reference: $WLK_REFERENCE_SRC

Recipe: a plain copy of the two pure-Python packages the tests and the benchmark import -- ``whisperlivekit`` (with
its packaged Silero VAD model) and ``third_party/qwen3-asr-causal/src/qwen3_asr_causal``.  Their heavy optional
dependencies (faster-whisper, torchaudio, librosa) are not needed: the exercised path (whisper/model.py,
whisper/audio.py, simul_whisper/*, the Qwen3 causal tower) needs only torch, numpy and tiktoken.
oracle/_ref/ is git-ignored: no reference source enters the history.
Test / benchmark infrastructure only: nothing under whisperlivekit_b200/ imports it.
"""
from __future__ import annotations

import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SRC = os.environ.get("WLK_REFERENCE_SRC", "/root/reference")
TARGET = os.path.join(ROOT, "oracle", "_ref")
STAMP = os.path.join(TARGET, ".staged_from")
PACKAGES = (("whisperlivekit", "whisperlivekit"),
            (os.path.join("third_party", "qwen3-asr-causal", "src", "qwen3_asr_causal"), "qwen3_asr_causal"))


def source_available() -> bool:
    return os.path.isdir(os.path.join(REF_SRC, "whisperlivekit", "whisper"))


def staged() -> bool:
    return os.path.isfile(STAMP) and all(os.path.isdir(os.path.join(TARGET, dst)) for _, dst in PACKAGES)


def stage(force: bool = False) -> str:
    if staged() and not force:
        return TARGET
    if not source_available():
        raise RuntimeError(f"{REF_SRC} holds no WhisperLiveKit checkout: set WLK_REFERENCE_SRC")
    if os.path.isdir(TARGET):
        shutil.rmtree(TARGET)
    os.makedirs(TARGET)
    for src, dst in PACKAGES:
        shutil.copytree(os.path.join(REF_SRC, src), os.path.join(TARGET, dst), ignore=shutil.ignore_patterns("__pycache__"))
    with open(STAMP, "w") as f:                      # written last: a partial copy never counts as staged
        f.write("plain copy of " + ", ".join(dst for _, dst in PACKAGES) + "\n")
    return TARGET


def import_staged_reference():
    """Put oracle/_ref first on sys.path (with a stub ``soundfile``, which one backend file imports at module scope and
    the exercised path never calls) and import the reference package."""
    import importlib.machinery
    import types
    if not staged():
        raise RuntimeError("oracle/_ref is empty: run `python oracle/stage_reference.py` where the reference is available")
    if "soundfile" not in sys.modules:
        try:
            import soundfile  # noqa: F401
        except Exception:
            m = types.ModuleType("soundfile")
            m.__spec__ = importlib.machinery.ModuleSpec("soundfile", loader=None)   # find_spec() must not choke on the stub
            m.read = m.write = m.info = lambda *a, **k: (_ for _ in ()).throw(RuntimeError("soundfile stub"))
            sys.modules["soundfile"] = m
    if TARGET not in sys.path:
        sys.path.insert(0, TARGET)
    import whisperlivekit
    assert os.path.abspath(whisperlivekit.__file__).startswith(TARGET), whisperlivekit.__file__
    return whisperlivekit


if __name__ == "__main__":
    print(stage(force="--force" in sys.argv))
    print(open(STAMP).read().strip())
