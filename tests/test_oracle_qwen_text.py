"""The CPU oracle of the Qwen3 text decoder, run by the shared generate driver, reproduces the reference's own outputs
(tests/golden/qwen_text_tnano.npz, and qwen_text_0.6b.npz at the true geometry): tokens and stats of every rolling / full
call, and the lm_head rows."""
import numpy as np
import pytest

from oracle.qwen_text_oracle import QwenTextOracle, banned_ngram_tokens
from whisperlivekit_b200.qwen_dims import QWEN_TEXT_DIMS, rope_inv_freq, synthetic_text_state_dict
from qwen_text_replay import capture_logits, load_fixture, replay


DIMS = {"tnano": "tnano", "0.6b": "qwen3-asr-0.6b"}
LOGIT_BOUND = {"tnano": 2e-5, "0.6b": 1e-4}       # 0.6b: 28 layers of fp32 reduction-order differences vs transformers


@pytest.fixture(scope="module", params=["tnano", "0.6b"])
def tnano(request):
    fx = load_fixture(request.param)
    fx["name"] = request.param
    dims = QWEN_TEXT_DIMS[DIMS[request.param]]
    orc = QwenTextOracle(dims, synthetic_text_state_dict(dims, int(fx["seed"])))
    log = capture_logits(orc, fx["stride"])
    return fx, replay(orc, fx), log


def test_tokens_and_stats(tnano):
    fx, got, _ = tnano
    for c, (toks, stats) in zip(fx["calls"], got):
        assert toks == c["tokens"], c
        if c["kind"] == "rolling":
            assert stats == c["stats"], (stats, c["stats"])


def test_logit_samples(tnano):
    fx, _, log = tnano
    assert len(log) == len(fx["sample_blocks"])
    worst = max(float(np.abs(a - b).max()) for a, b in zip(log, fx["sample_blocks"]))
    print(f"{fx['name']}: oracle max|dlogits| = {worst:.3e}")
    assert worst < LOGIT_BOUND[fx["name"]], worst


def test_schedule_covers_the_paths():
    fx = load_fixture("tnano")
    st = [c["stats"] for c in fx["calls"] if c["kind"] == "rolling"]
    assert any(s["decoder_rebuilt"] for s in st[1:])                       # template change
    assert any(s["audio_delta_steps"] == 0 for s in st)
    assert any(s["draft_all_accepted"] for s in st)
    assert any(s["draft_tokens"] and not s["draft_all_accepted"] for s in st)
    assert any(c.get("draft") and len(c["draft"]) > int(fx["max_new_tokens"]) for c in fx["calls"])


@pytest.mark.parametrize("theta", [1e4, 1e6])
def test_rope_inv_freq_is_transformers_bit_for_bit(theta):
    """The RoPE frequencies every QwenTextEngine loads are transformers' own buffer, bit for bit.  Rounding a
    double-precision pow once instead puts 19 (1e4) and 24 (1e6) of the 64 entries one ulp away: 2e-3 rad of angle at
    position 32767."""
    pytest.importorskip("transformers")
    from transformers import Qwen3Config
    from transformers.models.qwen3.modeling_qwen3 import Qwen3RotaryEmbedding
    cfg = Qwen3Config(hidden_size=256, num_attention_heads=2, num_key_value_heads=1, head_dim=128,
                      rope_parameters={"rope_type": "default", "rope_theta": theta})
    want = Qwen3RotaryEmbedding(cfg).inv_freq.numpy()
    got = rope_inv_freq(theta, 128)
    assert got.dtype == np.float32 and got.shape == (64,)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.flatnonzero(got != want)
    rounded_once = np.asarray([1.0 / theta ** (2 * i / 128) for i in range(64)], np.float64).astype(np.float32)
    assert (rounded_once != want).sum() >= 19                # what the helper exists to avoid


def test_banned_ngrams_match_the_reference_rule():
    assert banned_ngram_tokens([1, 2, 3, 1, 2], 3) == {3}
    assert banned_ngram_tokens([4, 4, 4], 1) == {4}
    assert banned_ngram_tokens([1], 3) == set()
