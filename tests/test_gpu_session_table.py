"""GPU: the session table every engine shares -- a full table refuses another session, a batch that names a session
twice or a closed session is refused, and every refusal leaves the open sessions working.  Each engine at its smallest
geometry with max_sessions=2, through the batch entry point it exposes (a Whisper session gets its audio on open).
And the handle every wrapper shares: once the engine is closed, no call reaches the destroyed engine."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _whisper():
    from golden_util import case_setup
    from whisperlivekit_b200.engine import WhisperEngine
    from whisperlivekit_b200.weights import synthetic_audio
    _, dims, sd, audio, heads = case_setup("micro")
    eng = WhisperEngine(dims, sd, heads, precision="fp32", max_sessions=2, max_batch=2)
    return eng, eng.encode, lambda sid: eng.append_audio(sid, synthetic_audio(1.0, seed=sid + 1))


def _tower():
    from whisperlivekit_b200.qwen_dims import QWEN_DIMS, synthetic_tower_state_dict
    from whisperlivekit_b200.qwen_engine import QwenTowerEngine
    dims = QWEN_DIMS["qnano"]
    eng = QwenTowerEngine(dims, synthetic_tower_state_dict(dims, 3), precision="fp32", max_sessions=2, max_batch=2)
    mel = np.random.default_rng(0).standard_normal((16, dims.n_mels)).astype(np.float32)
    return eng, lambda sids: eng.forward_chunk(sids, [mel] * len(sids)), None


def _text():
    from whisperlivekit_b200.qwen_dims import QWEN_TEXT_DIMS, synthetic_text_state_dict
    from whisperlivekit_b200.qwen_text_engine import QwenTextEngine
    dims = QWEN_TEXT_DIMS["tnano"]
    eng = QwenTextEngine(dims, synthetic_text_state_dict(dims, 3), precision="fp32", max_sessions=2, max_batch=2)
    return eng, lambda sids: eng.forward(sids, [(np.arange(4, dtype=np.int32), None)] * len(sids), [1] * len(sids)), None


def _sortformer():
    from whisperlivekit_b200.sortformer_dims import SORTFORMER_DIMS, synthetic_sortformer_state_dict
    from whisperlivekit_b200.sortformer_engine import SortformerEngine
    d = SORTFORMER_DIMS["micro"]
    eng = SortformerEngine(d, synthetic_sortformer_state_dict(d, 1), precision="fp32", max_sessions=2, max_batch=2)
    return eng, lambda sids: eng.step_audio(sids, [np.zeros(16000, np.float32)] * len(sids)), None


def _vad():
    from oracle.vad_oracle import synthetic_vad_state_dict
    from whisperlivekit_b200.vad import VadEngine
    eng = VadEngine(synthetic_vad_state_dict(seed=9), max_sessions=2)
    return eng, lambda sids: eng.forward(sids, [np.zeros(512, np.float32)] * len(sids)), None


@pytest.mark.parametrize("make", [_whisper, _tower, _text, _sortformer], ids=["whisper", "tower", "text", "sortformer"])
def test_session_table_refusals(make):
    from whisperlivekit_b200._lib import WlkError
    eng, call, prepare = make()

    def open_session():
        sid = eng.open_session()
        if prepare:
            prepare(sid)
        return sid
    try:
        a, b = open_session(), open_session()
        call([a, b])
        with pytest.raises(WlkError, match="sessions in use"):
            eng.open_session()
        call([a, b])
        with pytest.raises(WlkError, match="twice"):
            call([a, a])
        call([a, b])
        eng.close_session(b)
        with pytest.raises(WlkError, match="invalid session"):
            call([a, b])
        call([a])
        b = open_session()                              # the freed slot is reused
        call([b, a])
    finally:
        eng.close()


@pytest.mark.parametrize("make", [_whisper, _tower, _text, _sortformer, _vad],
                         ids=["whisper", "tower", "text", "sortformer", "vad"])
def test_closed_engine(make):
    """A session handle may be collected after its engine (in the same garbage cycle): closing the session then does
    nothing, a second close() does nothing, and any other call is refused as a null handle instead of reaching the
    destroyed engine."""
    from whisperlivekit_b200._lib import WlkError
    eng, call, prepare = make()
    sid = eng.open_session()
    if prepare:
        prepare(sid)
    call([sid])
    eng.close()
    assert eng.h is None
    eng.close_session(sid)
    eng.close()
    with pytest.raises(WlkError, match="null engine"):
        call([sid])
