"""GPU: the FP8 serving mode (WLK_PREC_FP8: e4m3 QKV, FC1 and FC2 in every encoder layer, bf16 elsewhere) end to end at
large-v3 against tests/golden/large_v3_forced.npz (the harness of test_gpu_large_v3.py), and the properties the mode
keeps: batch invariance, the incremental encoder's first block against the parity encode, the e4m3 weights travelling
in the weight blob, and its interface."""
import json

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from test_gpu_large_v3 import FRAME_TOL, fixture, run_mode, summarise
from whisperlivekit_b200.dims import ALIGNMENT_HEADS, DIMS
from whisperlivekit_b200.weights import synthetic_audio, synthetic_state_dict

FP8_LOGIT_TOL = 1.0         # e4m3 operands in 22 of the 24 T d^2 units of each of the 32 encoder layers
EPS_GAP_FP8 = 2.0           # reference top-2 gap above which the fp8 mode must pick the same token (>= 4 x measured)


def test_large_v3_fp8_mode_tokens_match_reference():
    res = run_mode("fp8")
    rep = summarise("fp8", res)
    g = fixture()[0]
    for i, (r, s) in enumerate(zip(res, rep["streams"])):
        assert np.isfinite(s["max_abs_dlogits_top8"]) and np.isfinite(s["enc_err"]), s
        assert s["max_abs_dlogits_top8"] <= FP8_LOGIT_TOL, s
        assert EPS_GAP_FP8 >= 4.0 * s["max_abs_dlogits_top8"], ("EPS_GAP_FP8 no longer covers the measured error", s)
        gaps, ref_t = g[f"s{i}_gaps"], g[f"s{i}_tokens"]
        for it in range(len(ref_t)):
            if gaps[it] > EPS_GAP_FP8:
                assert r["tokens"][it] == int(ref_t[it]), (i, it, float(gaps[it]), r["tokens"][it], int(ref_t[it]))
        # attended frames: reported only (argmaxes of nearly flat rows on random alignment heads, DESIGN.md section 1)
        print(json.dumps(dict(stream=i, frames_within_tol=s["frames_within_tol"], frame_tol=FRAME_TOL, steps=s["steps"])))


_ENG = {}


def _engine(max_batch=4):
    from whisperlivekit_b200.engine import WhisperEngine
    if "sd" not in _ENG:
        _ENG["sd"] = synthetic_state_dict(DIMS["large-v3"], seed=0)
    return WhisperEngine(DIMS["large-v3"], _ENG["sd"], ALIGNMENT_HEADS["large-v3"], precision="fp8",
                         max_sessions=max_batch, max_batch=max_batch)


def test_fp8_batch_invariance_incremental_anchor_and_weight_blob():
    import torch
    eng = _engine()
    audios = [synthetic_audio(s, seed=k) for k, s in enumerate((30.0, 11.0, 23.0, 7.0))]
    sids = [eng.open_session() for _ in range(4)]
    for s, a in zip(sids, audios):
        eng.append_audio(s, a)
    prefix = list(eng.specials.sot_sequence_including_notimestamps()) + [1169, 2068]
    eng.encode(sids)
    eng.decode(sids, [prefix] * 4)
    batch = {s: (eng.read_encoder(s), eng.read_logits(s)) for s in sids}
    eng.encode([sids[1]])                                   # the same stream alone
    eng.decode([sids[1]], [prefix])
    assert np.array_equal(eng.read_encoder(sids[1]), batch[sids[1]][0])
    # the decoder's split-K partials fold in arrival order: the logits agree to rounding, not bitwise
    assert np.abs(eng.read_logits(sids[1]) - batch[sids[1]][1]).max() < 1e-1
    assert np.isfinite(batch[sids[0]][0]).all() and np.isfinite(batch[sids[0]][1]).all()

    # the incremental encoder's first block is the whole window: the parity computation through the incremental path's
    # kernel pairing (cross-attention kernel, scatter epilogues), which the bf16 anchor also bounds rather than equates
    eng.close_session(sids[3])
    s_inc = eng.open_session()
    eng.append_audio(s_inc, audios[0])
    eng.encode([s_inc], incremental=True)
    assert np.abs(eng.read_encoder(s_inc) - batch[sids[0]][0]).max() < 0.25

    # a second fp8 engine adopting this one's weight blob encodes the same bits
    ptr, nbytes = eng.weight_blob()
    from whisperlivekit_b200.engine import WhisperEngine
    other = WhisperEngine(DIMS["large-v3"], None, ALIGNMENT_HEADS["large-v3"], precision="fp8", max_sessions=1, max_batch=1)
    optr, onbytes = other.weight_blob()
    assert onbytes == nbytes

    def view(p):                                            # the blob as a torch tensor (as bench.py broadcasts it)
        class _Blob:
            __cuda_array_interface__ = dict(shape=(nbytes,), typestr="|u1", data=(p, False), version=2)
        return torch.as_tensor(_Blob(), device="cuda")
    torch.cuda.synchronize()
    view(optr).copy_(view(ptr))
    torch.cuda.synchronize()
    other.adopt_weights()
    s2 = other.open_session()
    other.append_audio(s2, audios[0])
    other.encode([s2])
    assert np.array_equal(other.read_encoder(s2), batch[sids[0]][0])
    other.close()
    eng.close()


def test_fp8_interface():
    from whisperlivekit_b200._lib import WlkError
    from whisperlivekit_b200.engine import WhisperEngine
    dims = DIMS["large-v3"]
    mem = {}
    for p in ("bf16", "fp8"):
        e = WhisperEngine(dims, None, ALIGNMENT_HEADS["large-v3"], precision=p, max_sessions=1, max_batch=1)
        mem[p] = e.memory()
        e.close()
    d, L = dims.n_audio_state, dims.n_audio_layer
    # Wqkv, W1, W2 of each encoder layer: 11 d^2 elements, once, in e4m3 (bf16: 2 bytes) + fp32 row scales (3d + 4d + d)
    # + the 2-float FC1 bound, each buffer at a 256-byte boundary
    saved = L * (11 * d * d - 8 * d * 4 - 8)
    assert abs((mem["bf16"]["weights"] - mem["fp8"]["weights"]) - saved) <= L * 8 * 256, mem
    # the e4m3 LayerNorm output and its two row-scale vectors (the e4m3 hidden shares the bf16 one's buffer)
    assert mem["fp8"]["workspace"] - mem["bf16"]["workspace"] == 1500 * d + 2 * 1500 * 4, mem
    with pytest.raises(WlkError):
        WhisperEngine(dims, None, [(0, 0)], precision="fp8", gemm_backend="simt", max_sessions=1, max_batch=1)
    with pytest.raises(KeyError):
        WhisperEngine(dims, None, [(0, 0)], precision="fp4", max_sessions=1, max_batch=1)
