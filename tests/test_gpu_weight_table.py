"""GPU: the weight table every CUDA engine declares its checkpoint tensors in.  Each engine at its smallest geometry,
built empty and loaded tensor by tensor from its synthetic state dict: a missing tensor is named by finalize, a name
that is not declared (unknown, a layer index out of range or malformed, a tensor this geometry does not have) is
refused, a wrong shape is refused by the engine's own shape rule, and the optional tensors load."""
import dataclasses
import re

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _whisper():
    from golden_util import case_setup
    from whisperlivekit_b200.engine import WhisperEngine
    _, dims, sd, _, _ = case_setup("micro")
    return dict(
        make=lambda: WhisperEngine(dims, None, precision="fp32", max_sessions=1, max_batch=1),
        sd={k: v for k, v in sd.items() if not WhisperEngine._skip(k, v)},
        layer="decoder.blocks.1.cross_attn.value.weight",
        undeclared=[f"encoder.blocks.{dims.n_audio_layer}.mlp_ln.weight", "encoder.blocks.x.mlp_ln.weight",
                    "decoder.blocks.1x.mlp_ln.weight", "decoder.blocks.0.cross_attn.key.bias"],
        like="decoder.blocks.0.mlp_ln.weight",
        # element count only: the transpose loads, one element more does not
        accepted={"encoder.blocks.0.mlp.0.weight": sd["encoder.blocks.0.mlp.0.weight"].T},
        wrong=("encoder.conv1.bias", np.zeros(dims.n_audio_state + 1, np.float32),
               f"has {dims.n_audio_state + 1} elements, expected {dims.n_audio_state}"),
        optional={})


def _tower(window=False):
    from whisperlivekit_b200.qwen_dims import QWEN_DIMS, QWEN_WINDOW_DIMS, synthetic_tower_state_dict
    from whisperlivekit_b200.qwen_engine import QwenTowerEngine, QwenWindowEngine
    from whisperlivekit_b200.weights import mel_filterbank
    dims = QWEN_WINDOW_DIMS["wnano"] if window else QWEN_DIMS["qnano"]
    cls = QwenWindowEngine if window else QwenTowerEngine
    sd = synthetic_tower_state_dict(dims, 3)
    d = dims.d_model
    undeclared = [f"layers.{dims.n_layer}.fc1.weight", "layers.1x.fc1.weight", "layers.x.fc1.weight"]
    if not dims.conv_out_bias:
        undeclared.append("conv_out.bias")
    return dict(
        make=lambda: cls(dims, None, precision="fp32", max_sessions=1, max_batch=1),
        sd=sd, layer="layers.1.self_attn.k_proj.bias", undeclared=undeclared, like="layers.0.fc1.weight",
        accepted={},
        wrong=("layers.0.fc1.weight", sd["layers.0.fc1.weight"].T.copy(), "wrong shape"),
        optional={"mel_filters": mel_filterbank(dims.n_mels),
                  "positional_embedding.inv_freq": np.ones(d // 2, np.float32)})


def _text(tied=False):
    from whisperlivekit_b200.qwen_dims import QWEN_TEXT_DIMS, synthetic_text_state_dict
    from whisperlivekit_b200.qwen_text_engine import QwenTextEngine
    dims = dataclasses.replace(QWEN_TEXT_DIMS["tnano"], tied=tied)
    sd = synthetic_text_state_dict(dims, 3)
    undeclared = [f"layers.{dims.n_layer}.mlp.up_proj.weight", "layers.1x.mlp.up_proj.weight"]
    if tied:
        undeclared.append("lm_head.weight")
    return dict(
        make=lambda: QwenTextEngine(dims, None, precision="fp32", max_sessions=1, max_batch=1),
        sd=sd, layer="layers.1.mlp.up_proj.weight", undeclared=undeclared, like="layers.0.mlp.up_proj.weight",
        accepted={},
        wrong=("layers.0.mlp.down_proj.weight", sd["layers.0.mlp.down_proj.weight"].T.copy(), "wrong shape"),
        optional={"rotary_emb.inv_freq": np.ones(dims.head_dim // 2, np.float32)})


def _sortformer():
    from whisperlivekit_b200.sortformer_dims import SORTFORMER_DIMS, synthetic_sortformer_state_dict
    from whisperlivekit_b200.sortformer_engine import SortformerEngine
    from whisperlivekit_b200.weights import mel_filterbank
    dims = SORTFORMER_DIMS["micro"]
    sd = {k: v for k, v in synthetic_sortformer_state_dict(dims, 1).items() if not SortformerEngine._skip(k, v)}
    sd["mel_filters"] = mel_filterbank(dims.n_mels, 16000, dims.n_fft)
    conv = "encoder.pre_encode.conv.0.weight"
    return dict(
        make=lambda: SortformerEngine(dims, None, precision="fp32", max_sessions=1, max_batch=1),
        sd=sd, layer="transformer_encoder.layers.1.first_sub_layer.key_net.bias",
        undeclared=[f"encoder.layers.{dims.n_layer}.norm_out.weight", "encoder.layers.1x.norm_out.weight",
                    f"transformer_encoder.layers.{dims.tf_n_layer}.layer_norm_1.weight"],
        like="encoder.layers.0.norm_out.weight",
        # element count and leading axis: a Conv kernel may carry trailing singleton axes
        accepted={conv: sd[conv].reshape(sd[conv].shape[0], 1, 3, 3)},
        wrong=("encoder.layers.0.feed_forward1.linear1.weight",
               sd["encoder.layers.0.feed_forward1.linear1.weight"].T.copy(), "wrong shape"),
        optional={"encoder.layers.0.conv.batch_norm.num_batches_tracked": np.zeros(1, np.float32)})


ENGINES = {"whisper": _whisper, "tower": _tower, "window": lambda: _tower(window=True), "text": _text,
           "text-tied": lambda: _text(tied=True), "sortformer": _sortformer}


@pytest.fixture(params=list(ENGINES))
def case(request):
    return ENGINES[request.param]()


def _load_all(eng, sd, skip=None):
    for name, arr in sd.items():
        if name != skip:
            eng.load_tensor(name, arr)


@pytest.mark.parametrize("which", ["first", "layer", "last"])
def test_missing_tensor_is_named(case, which):
    from whisperlivekit_b200._lib import WlkError
    names = list(case["sd"])
    drop = {"first": names[0], "layer": case["layer"], "last": names[-1]}[which]
    assert drop in case["sd"]
    eng = case["make"]()
    try:
        _load_all(eng, case["sd"], skip=drop)
        with pytest.raises(WlkError, match=r"1 tensors missing, e\.g\. " + re.escape(drop) + " "):
            eng.finalize()
    finally:
        eng.close()


def test_undeclared_and_misshapen_tensors_are_refused(case):
    from whisperlivekit_b200._lib import WlkError
    eng = case["make"]()
    try:
        like = case["sd"][case["like"]]
        for name in ["no_such.weight"] + case["undeclared"]:
            with pytest.raises(WlkError, match="unknown tensor " + re.escape(name)):
                eng.load_tensor(name, like)
        name, arr, msg = case["wrong"]
        with pytest.raises(WlkError, match=msg):
            eng.load_tensor(name, arr)
        for name, arr in case["accepted"].items():
            eng.load_tensor(name, arr)
        _load_all(eng, case["sd"])                      # the refusals changed nothing: the full set still finalizes
        eng.finalize()
    finally:
        eng.close()


def test_optional_tensors_load(case):
    eng = case["make"]()
    try:
        _load_all(eng, case["sd"])
        for name, arr in case["optional"].items():
            eng.load_tensor(name, arr)
        eng.finalize()
    finally:
        eng.close()
