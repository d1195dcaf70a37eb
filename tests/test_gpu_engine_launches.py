"""GPU: what the Whisper engine's profile records per call (wlk_profile_read), pinned against counts derived from the
dims.  bench.py's per-class lines read these numbers, and a layer's launches changing by accident (a step dropped from
one copy of the block, an epilogue split off into its own kernel) shows up here as a launch or flop count that moved."""
import pytest

pytestmark = pytest.mark.gpu

N_CTX, MEL_ROWS = 1500, 3002
ES = {"fp32": 4, "bf16": 2, "bf16x3": 4}            # bytes per activation element


def _engine(precision, n=2):
    from whisperlivekit_b200.dims import ALIGNMENT_HEADS, DIMS
    from whisperlivekit_b200.engine import WhisperEngine
    from whisperlivekit_b200.weights import synthetic_state_dict
    dims = DIMS["tiny"]
    eng = WhisperEngine(dims, synthetic_state_dict(dims, seed=3), ALIGNMENT_HEADS["tiny"], precision=precision,
                        max_sessions=n, max_batch=n)
    eng.profile_enable(True)
    return dims, eng


def _profile(eng, call):
    eng.profile_reset()
    call()
    return {k: v for k, v in eng.profile_read().items() if v["launches"]}


def _check(got, want):
    assert set(got) == set(want), (sorted(got), sorted(want))
    for cls, w in want.items():
        for field, v in w.items():
            assert got[cls][field] == pytest.approx(v, rel=1e-12, abs=0), (cls, field, got[cls][field], v)


def _encoder(dims, es, n, R, conv_rows, attn_flops, attn_bytes):
    """the log-mel of n streams, the conv stem (conv1 and conv2 over conv_rows), L encoder blocks over R rows, ln_post
    and the cross-K/V GEMM"""
    d, dt, nm, L = dims.n_audio_state, dims.n_text_state, dims.n_mels, dims.n_audio_layer
    return {
        "mel": dict(launches=1, flops=0, bytes=n * (480000.0 * 4 + 3000.0 * nm * es)),
        "gemm_enc": dict(launches=2 + 4 * L, flops=2.0 * conv_rows[0] * d * 3 * nm + 2.0 * conv_rows[1] * d * 3 * d
                         + L * 24.0 * R * d * d),
        "layernorm": dict(launches=2 * L + 1, flops=0, bytes=(2 * L + 1) * float(R) * d * (4 + es)),
        "attn_enc": dict(launches=L, flops=L * attn_flops, bytes=L * attn_bytes),
        "gemm_xkv": dict(launches=1, flops=2.0 * R * dims.n_text_layer * 2 * dt * d),
    }


def _decoder(dims, es, n, R, n_sel):
    """one decoder call over R packed rows of n sessions, logits of n_sel rows: 11 launches per layer plus 3"""
    dt, L = dims.n_text_state, dims.n_text_layer
    return {
        "misc": dict(launches=1, flops=0, bytes=0),
        "layernorm": dict(launches=3 * L + 1, flops=0, bytes=0),
        "gemm_dec": dict(launches=6 * L, flops=L * 28.0 * R * dt * dt),
        "attn_dec_self": dict(launches=L, flops=0, bytes=0),
        "attn_dec_cross": dict(launches=L, flops=0, bytes=L * float(n) * 2 * dims.n_text_head * N_CTX * 64 * es),
        "logits": dict(launches=1, flops=2.0 * n_sel * dims.n_vocab * dt),
    }


@pytest.mark.parametrize("precision", ["fp32", "bf16", "bf16x3"])
def test_parity_encode_prefill_and_token_step(precision):
    from whisperlivekit_b200.weights import synthetic_audio
    dims, eng = _engine(precision)
    es, n, d = ES[precision], 2, dims.n_audio_state
    sids = [eng.open_session() for _ in range(n)]
    for k, s in enumerate(sids):
        eng.append_audio(s, synthetic_audio(4.0 + 3 * k, seed=5 + k))
    R = n * N_CTX
    # conv1 over the n * MEL_ROWS - 2 overlapping rows of the padded mel, conv2 over n * (N_CTX + 1) - 1
    _check(_profile(eng, lambda: eng.encode(sids)),
           _encoder(dims, es, n, R, (n * MEL_ROWS - 2, n * (N_CTX + 1) - 1),
                    4.0 * n * dims.n_audio_head * N_CTX * N_CTX * 64, R * 4.0 * d * es))
    prefix = list(eng.specials.sot_sequence_including_notimestamps())
    prefix += list(range(1000, 1000 + 20 - len(prefix)))
    assert len(prefix) == 20
    _check(_profile(eng, lambda: eng.decode(sids, [prefix] * n)), _decoder(dims, es, n, 20 * n, 2 * n))
    _check(_profile(eng, lambda: eng.decode(sids, [[7586]] * n)), _decoder(dims, es, n, n, n))
    eng.close()


def test_incremental_encode_first_call_and_grown_chunk():
    from whisperlivekit_b200.weights import synthetic_audio
    dims, eng = _engine("bf16", n=1)
    es, d, H = 2, dims.n_audio_state, dims.n_audio_head
    audio = synthetic_audio(8.0, seed=7)
    s = eng.open_session()
    eng.append_audio(s, audio[: 7 * 16000])
    for rows_expected in (N_CTX, None):                         # the whole window first, then the appended block
        got = _profile(eng, lambda: eng.encode([s], incremental=True))
        (R,) = eng.last_block_rows
        if rows_expected:
            assert R == rows_expected
        else:
            assert 0 < R < N_CTX
        want = _encoder(dims, es, 1, R, (2 * R + 1, R), 4.0 * H * R * N_CTX * 64, 2.0 * d * N_CTX * es)
        want["misc"] = dict(launches=3, flops=0, bytes=0)     # gather conv1 rows, gather conv2 rows, scatter into xa
        _check(got, want)
        eng.append_audio(s, audio[7 * 16000: 7 * 16000 + 8000])
    eng.close()
