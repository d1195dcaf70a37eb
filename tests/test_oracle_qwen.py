"""CPU: the Qwen3-ASR causal-tower oracle against fixtures recorded from the reference's own
QwenAudioCausalKVEncoder (oracle/make_golden_qwen.py): same ragged append schedule, same seeded tower."""
import os

import numpy as np
import pytest

from whisperlivekit_b200.qwen_dims import QWEN_DIMS, synthetic_tower_state_dict

HERE = os.path.dirname(os.path.abspath(__file__))


def qwen_case(name):
    import sys
    sys.path.insert(0, os.path.dirname(HERE))
    from oracle.make_golden_qwen import mel_stream
    g = dict(np.load(os.path.join(HERE, "golden", f"qwen_{name}.npz")))
    dims = QWEN_DIMS[name]
    sd = synthetic_tower_state_dict(dims, seed=11)
    sched = [int(x) for x in g["schedule"]]
    return g, dims, sd, mel_stream(sum(sched), dims.n_mels, seed=3), sched


def check_stream(engine, g, mels, sched, tol):
    """Drive `engine.forward_chunk` with the fixture's schedule and compare every call with the reference."""
    sid = engine.open_session()
    a, worst = 0, 0.0
    for i, n in enumerate(sched):
        h = engine.forward_chunk([sid], [mels[a: a + n]])[0]
        a += n
        assert h.shape[0] == int(g[f"steps{i}"]), f"call {i}: emitted rows"
        assert engine.emitted_steps(sid) == int(g[f"emitted{i}"])
        assert engine.pending_frames(sid) == int(g[f"pending{i}"])
        if f"mutable{i}" in g:
            assert engine.mutable_steps(sid) == int(g[f"mutable{i}"]), f"call {i}: mutable tail"
        if h.size:
            flat = h.reshape(-1)
            worst = max(worst, float(np.abs(flat[g[f"idx{i}"]] - g[f"val{i}"]).max()))
            worst = max(worst, float(np.abs(h.astype(np.float64).sum(axis=1) - g[f"rowsum{i}"]).max()) / h.shape[1] ** 0.5)
    h = engine.flush_pending([sid])[0]                                   # end of stream
    assert h.shape[0] == int(g["flush_steps"]) and engine.emitted_steps(sid) == int(g["flush_emitted"])
    assert engine.pending_frames(sid) == 0
    if h.size:
        worst = max(worst, float(np.abs(h[0] - g["flush_first_row"]).max()))
        worst = max(worst, float(np.abs(h.astype(np.float64).sum(axis=1) - g["flush_rowsum"]).max()) / h.shape[1] ** 0.5)
    engine.close_session(sid)
    assert worst < tol, worst
    return worst


@pytest.mark.parametrize("name", ["qnano", "qnano-chunk", "qnano-tail", "qnano-tail-bidir"])
def test_oracle_matches_reference_fixtures(name):
    from oracle.qwen_oracle import QwenTowerOracle
    g, dims, sd, mels, sched = qwen_case(name)
    worst = check_stream(QwenTowerOracle(dims, sd), g, mels, sched, 2e-5)
    assert sum(int(g[f"steps{i}"]) for i in range(len(sched))) > 100


def test_sessions_are_independent_and_resettable():
    from oracle.qwen_oracle import QwenTowerOracle
    g, dims, sd, mels, sched = qwen_case("qnano")
    orc = QwenTowerOracle(dims, sd)
    a, b = orc.open_session(), orc.open_session()
    ha = orc.forward_chunk([a, b], [mels[:400], mels[100:300]])
    hb = orc.forward_chunk([b], [mels[300:500]])[0]
    orc.reset_session(b)
    hb2 = orc.forward_chunk([b], [mels[:400]])[0]
    assert ha[0].shape[0] == 48 and ha[1].shape[0] == 24 and hb.shape[0] == 24
    np.testing.assert_allclose(hb2, ha[0], atol=1e-6)


@pytest.mark.parametrize("d", [128, 896, 1024, 1280])
def test_sinusoid_inv_freq_is_the_oracles_closed_form(d):
    """The frequencies the engine loads for the positional rows past the table reproduce the oracle's closed form
    (causal.py _position_embedding) bit for bit on the CPU, at the 0.6B width (896) and around it.  At 896 the scale
    evaluated as an fp32 quotient of fp32 operands is one ulp away from the reference's double rounded once."""
    import math

    import torch
    from oracle.qwen_oracle import QwenTowerOracle
    from whisperlivekit_b200.qwen_dims import QwenTowerDims, sinusoid_inv_freq, sinusoid_table
    T = 40
    dims = QwenTowerDims(d_model=d, n_head=d // 64, max_positions=T)
    orc = QwenTowerOracle(dims, {"positional_embedding.positional_embedding": sinusoid_table(T, d)})
    inv = torch.from_numpy(sinusoid_inv_freq(d))
    assert inv.dtype == torch.float32 and inv.shape == (d // 2,)
    for offset, length in ((T, 24), (4095, 8), (45000, 24), (2 ** 20, 1)):
        pos = torch.arange(offset, offset + length, dtype=torch.float32)
        scaled = pos[:, None] * inv[None, :]
        mine = torch.cat([scaled.sin(), scaled.cos()], dim=1)
        assert torch.equal(mine, orc._pos(offset, length)), (d, offset)
    half = d // 2
    ref_scale = np.float32(-math.log(10000.0) / float(half - 1))
    f32_scale = np.float32(-np.log(np.float32(10000.0))) / np.float32(half - 1)
    assert (ref_scale != f32_scale) == (d == 896), (d, ref_scale, f32_scale)
