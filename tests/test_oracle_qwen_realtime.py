"""The realtime model's frame adapter and the whole-model install against fixtures recorded from the reference
(oracle/make_golden_qwen_realtime.py): the float64 and fp32 oracle adapters reproduce the reference adapter's outputs, and
the reference's segmented streamer over the installed model, with the CPU oracles behind the engine API, reproduces every
event, including the segment rollovers and the pending mel frames carried across them."""
import json
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GEOMETRIES = ["qnano", "qnano-tail"]


def fixture(name):
    z = np.load(os.path.join(ROOT, "tests", "golden", f"qwen_realtime_{name}.npz"))
    return z, json.loads(bytes(z["events"]).decode())


@pytest.mark.parametrize("name", GEOMETRIES)
def test_adapter_oracles_match_reference_outputs(name):
    from oracle.make_golden_qwen_realtime import adapter_sd
    from oracle.qwen_realtime_oracle import QwenRealtimeTextOracle, adapter_f64
    from whisperlivekit_b200.qwen_dims import QWEN_TEXT_DIMS, synthetic_text_state_dict
    z, _ = fixture(name)
    x, ref = z["adapter_in"], z["adapter_out"]
    assert x.shape[0] == ref.shape[0] >= 24 and int(z["adapter_rows"].sum()) == x.shape[0]
    sd = adapter_sd(name)
    y64 = adapter_f64(x, sd)
    assert np.abs(y64 - ref).max() <= 1e-5 * np.abs(ref).max()
    dims = QWEN_TEXT_DIMS["tnano"]
    orc = QwenRealtimeTextOracle(dims, dict(synthetic_text_state_dict(dims, 5), **sd))
    y32 = orc.adapt(torch.from_numpy(x)).numpy()
    assert np.abs(y32 - ref).max() <= 1e-6 * np.abs(ref).max()
    assert np.abs(y64 - np.asarray(x, np.float64) @ sd["adapter.proj.weight"].T.astype(np.float64)).max() > 1e-3  # blocks act


def oracle_factories():
    from oracle.qwen_realtime_oracle import QwenRealtimeTextOracle, QwenRealtimeTowerOracle
    made = {"tower": [], "text": []}

    def tower(d, sd):
        made["tower"].append(QwenRealtimeTowerOracle(d, sd))
        return made["tower"][-1]

    def text(d, sd):
        made["text"].append(QwenRealtimeTextOracle(d, sd))
        return made["text"][-1]
    return tower, text, made


@pytest.mark.reference
@pytest.mark.parametrize("name", GEOMETRIES)
def test_installed_model_with_oracles_reproduces_every_event(name):
    pytest.importorskip("transformers")
    from oracle import stage_reference
    stage_reference.import_staged_reference()
    from oracle.make_golden_qwen import mel_stream
    from oracle.make_golden_qwen_realtime import MEL_SEED, N_FRAMES, build_model, build_streamer, drive
    from whisperlivekit_b200.qwen_plugin import B200QwenRealtimeModel
    _, want = fixture(name)
    model = build_model(name)
    tower, text, _ = oracle_factories()
    B200QwenRealtimeModel.install(model, tower_factory=tower, text_factory=text)
    got = drive(build_streamer(model), mel_stream(N_FRAMES, 128, seed=MEL_SEED))
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, (i, {k: (g.get(k), w.get(k)) for k in set(g) | set(w) if g.get(k) != w.get(k)})
    assert sum(1 for e in want if e.get("segment_rollover") or e.get("segment_rolled_before_generate")) >= 2
    if name == "qnano":             # pending frames carried into the fresh encoder state at a rollover, then consumed
        rolled = [i for i, e in enumerate(want) if e.get("segment_rollover")]
        assert any(want[i + 1]["encoder_pending_frames"] > 25 for i in rolled if i + 1 < len(want))
