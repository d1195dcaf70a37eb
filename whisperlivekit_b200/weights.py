"""Weight containers for the H100 streaming-Whisper engine.

* ``synthetic_state_dict`` – seeded "trained-like" random weights with the
  reference's parameter names (reference whisperlivekit/whisper/model.py:224-332;
  key names as produced by ``Whisper(dims).state_dict()``).  There are no
  released checkpoints in the build container (SURVEY.md §8c), so parity and
  benchmarks run on these; a real ``.pt`` state_dict with the same names loads
  through the same path.
* ``mel_filterbank`` – the Slaney-normalised librosa filterbank the reference
  ships as an asset (whisper/audio.py:91-107); recomputed here so no data file
  is copied.  oracle/make_golden.py pins it against the asset.
* ``sinusoids`` – encoder positional table (whisper/model.py:62-68).
"""
from __future__ import annotations

import math
from typing import Dict

import numpy as np

from .dims import ModelDimensions, N_FFT, SAMPLE_RATE


# ----------------------------------------------------------------------------
# mel filterbank (librosa.filters.mel(sr=16000, n_fft=400, n_mels=n), slaney)
# ----------------------------------------------------------------------------
def _hz_to_mel(f):
    f = np.asanyarray(f, dtype=np.float64)
    f_sp = 200.0 / 3
    mels = f / f_sp
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    out = np.where(f >= min_log_hz,
                   min_log_mel + np.log(np.maximum(f, 1e-30) / min_log_hz) / logstep, mels)
    return out


def _mel_to_hz(m):
    m = np.asanyarray(m, dtype=np.float64)
    f_sp = 200.0 / 3
    freqs = f_sp * m
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), freqs)


def mel_filterbank(n_mels: int, sr: int = SAMPLE_RATE, n_fft: int = N_FFT) -> np.ndarray:
    """[n_mels, n_fft//2+1] float32 Slaney mel filterbank."""
    fmax = sr / 2.0
    n_freq = 1 + n_fft // 2
    fftfreqs = np.linspace(0.0, fmax, n_freq, dtype=np.float64)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(0.0), _hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    weights = np.zeros((n_mels, n_freq), dtype=np.float32)
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        weights[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels])
    weights *= enorm[:, np.newaxis].astype(np.float32)
    return weights


def sinusoids(length: int, channels: int, max_timescale: float = 10000.0) -> np.ndarray:
    """reference whisper/model.py:62-68, evaluated in float32 like torch does."""
    import torch
    assert channels % 2 == 0
    inc = np.log(max_timescale) / (channels // 2 - 1)
    inv = torch.exp(-inc * torch.arange(channels // 2))
    st = torch.arange(length)[:, None] * inv[None, :]
    return torch.cat([torch.sin(st), torch.cos(st)], dim=1).numpy().astype(np.float32)


def hann_window(n: int = N_FFT) -> np.ndarray:
    """torch.hann_window(n) (periodic) in float32 (reference whisper/audio.py:147)."""
    import torch
    return torch.hann_window(n).numpy()


# ----------------------------------------------------------------------------
# synthetic weights
# ----------------------------------------------------------------------------
def synthetic_state_dict(dims: ModelDimensions, seed: int = 0,
                         logit_std: float = 3.0) -> Dict[str, np.ndarray]:
    """Seeded float32 weights with trained-like scales.

    Linear/conv weights ~ N(0, 1/fan_in) so activations keep unit scale through
    depth, LayerNorm gains ~ 1 +- 0.1, and the tied token embedding is scaled so
    logits have standard deviation ``logit_std`` (released checkpoints sit at a
    few units).  Values depend only on (dims, seed, numpy's PCG64 stream).
    """
    rng = np.random.default_rng(seed)

    def normal(shape, std):
        return (rng.standard_normal(shape, dtype=np.float32) * np.float32(std))

    sd: Dict[str, np.ndarray] = {}

    def linear(prefix, n_out, n_in, bias=True, gain=1.0):
        sd[prefix + ".weight"] = normal((n_out, n_in), gain / math.sqrt(n_in))
        if bias:
            sd[prefix + ".bias"] = normal((n_out,), 0.02)

    def lnorm(prefix, n):
        sd[prefix + ".weight"] = (1.0 + normal((n,), 0.1)).astype(np.float32)
        sd[prefix + ".bias"] = normal((n,), 0.1)

    def block(prefix, n, cross):
        for att in (["attn", "cross_attn"] if cross else ["attn"]):
            linear(f"{prefix}.{att}.query", n, n)
            linear(f"{prefix}.{att}.key", n, n, bias=False)
            linear(f"{prefix}.{att}.value", n, n)
            linear(f"{prefix}.{att}.out", n, n, gain=0.5)
            lnorm(f"{prefix}.{att}_ln", n)
        linear(f"{prefix}.mlp.0", 4 * n, n)
        linear(f"{prefix}.mlp.2", n, 4 * n, gain=0.5)
        lnorm(f"{prefix}.mlp_ln", n)

    d = dims.n_audio_state
    sd["encoder.conv1.weight"] = normal((d, dims.n_mels, 3), 1.0 / math.sqrt(3 * dims.n_mels))
    sd["encoder.conv1.bias"] = normal((d,), 0.02)
    sd["encoder.conv2.weight"] = normal((d, d, 3), 1.0 / math.sqrt(3 * d))
    sd["encoder.conv2.bias"] = normal((d,), 0.02)
    sd["encoder.positional_embedding"] = sinusoids(dims.n_audio_ctx, d)
    for i in range(dims.n_audio_layer):
        block(f"encoder.blocks.{i}", d, cross=False)
    lnorm("encoder.ln_post", d)

    t = dims.n_text_state
    sd["decoder.token_embedding.weight"] = normal((dims.n_vocab, t), logit_std / math.sqrt(t))
    sd["decoder.positional_embedding"] = normal((dims.n_text_ctx, t), 0.02)
    for i in range(dims.n_text_layer):
        block(f"decoder.blocks.{i}", t, cross=True)
    lnorm("decoder.ln", t)
    return sd


def state_dict_from_torch(module_state_dict) -> Dict[str, np.ndarray]:
    """Convert a torch ``Whisper.state_dict()`` (or a loaded ``.pt``'s
    ``model_state_dict``) into the float32 numpy form the engine ingests."""
    out = {}
    for k, v in module_state_dict.items():
        out[k] = v.detach().to("cpu").float().contiguous().numpy()
    return out


def synthetic_audio(seconds: float, seed: int = 1234, sr: int = SAMPLE_RATE) -> np.ndarray:
    """Deterministic speech-like test signal in [-1, 1]: a few drifting
    harmonics under a 3 Hz syllabic envelope plus a little noise."""
    n = int(round(seconds * sr))
    rng = np.random.default_rng(seed)
    t = np.arange(n, dtype=np.float64) / sr
    f0 = 120.0 + 40.0 * np.sin(2 * np.pi * 0.31 * t + rng.uniform(0, 6.28))
    phase = 2 * np.pi * np.cumsum(f0) / sr
    sig = np.zeros(n)
    for h, a in enumerate([1.0, 0.6, 0.4, 0.25, 0.15, 0.1], start=1):
        sig += a * np.sin(h * phase + rng.uniform(0, 6.28))
    env = 0.55 + 0.45 * np.sin(2 * np.pi * 3.0 * t + rng.uniform(0, 6.28))
    gate = (np.sin(2 * np.pi * 0.23 * t + rng.uniform(0, 6.28)) > -0.6).astype(np.float64)
    sig = 0.18 * sig * env * gate + 0.004 * rng.standard_normal(n)
    return np.clip(sig, -1.0, 1.0).astype(np.float32)
