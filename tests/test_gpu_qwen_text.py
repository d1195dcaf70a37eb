"""The Qwen3 text decoder on the H100 (csrc/qwen_text.cu) against the reference's own outputs
(tests/golden/qwen_text_tnano.npz, and qwen_text_0.6b.npz at the true geometry with tied embeddings and the 151936-id
vocabulary) and the CPU oracle.

fp32 (SIMT GEMMs) is the parity mode: tokens and stats identical, lm_head rows within 1e-3.  bf16 (wgmma GEMMs, fp32
residual / statistics / softmax / logits) is teacher-forced through the verify path with the reference's tokens as the
draft: its verify picks must equal the reference wherever the oracle's controlled top-2 gap exceeds BF16_PICK_EPS.
The bf16 attention runs on tensor cores (mma.sync), the fp32 attention on SIMT."""
import dataclasses

import numpy as np
import pytest
import torch

from oracle.qwen_text_oracle import QwenTextOracle, controlled_logits
from whisperlivekit_b200._lib import WlkError
from whisperlivekit_b200.qwen_dims import QWEN_TEXT_DIMS, synthetic_text_state_dict
from whisperlivekit_b200.qwen_text_engine import QwenTextEngine
from qwen_text_replay import TEMPLATES, capture_logits, load_fixture, replay

pytestmark = pytest.mark.gpu

# ~2x the max |bf16 - fp32| over the verify rows measured on H100 SXM (700 W), per fixture: tnano 4.2e-2, 0.6b 2.85e-1
# and 2.97e-1 in two runs (split-K accumulation order varies).  A pick cannot flip where the top-2 gap exceeds twice the
# bound.  MIN_CHECKED is the share of verify rows whose gap clears that bar: with seeded weights the 151936-id vocabulary
# has close runners-up, so at 0.6b only 5 of 48 rows are decidable against 28 layers of bf16 error; tnano decides 90 of 120
BF16_LOGIT_BOUND = {"tnano": 0.08, "0.6b": 0.57}
MIN_CHECKED = {"tnano": 0.6, "0.6b": 0.08}
DIMS = {"tnano": "tnano", "0.6b": "qwen3-asr-0.6b"}


@pytest.fixture(scope="module", params=["tnano", "0.6b"])
def case(request):
    fx = load_fixture(request.param)
    fx["name"] = request.param
    dims = QWEN_TEXT_DIMS[DIMS[request.param]]
    return fx, dims, synthetic_text_state_dict(dims, int(fx["seed"]))


@pytest.fixture(scope="module")
def fx():
    return load_fixture("tnano")


@pytest.fixture(scope="module")
def sd(fx):
    return synthetic_text_state_dict(QWEN_TEXT_DIMS["tnano"], int(fx["seed"]))


def test_fp32_reproduces_the_reference(case):
    fx, dims, sd = case
    eng = QwenTextEngine(dims, sd, precision="fp32", max_sessions=4, max_batch=4)
    log = capture_logits(eng, fx["stride"])
    got = replay(eng, fx)
    for c, (toks, stats) in zip(fx["calls"], got):
        assert toks == c["tokens"], (c, toks)
        if c["kind"] == "rolling":
            assert stats == c["stats"], (stats, c["stats"])
    assert len(log) == len(fx["sample_blocks"])
    worst = max(float(np.abs(a - b).max()) for a, b in zip(log, fx["sample_blocks"]))
    print(f"{fx['name']} fp32 max|dlogits| = {worst:.3e}")
    assert worst < 1e-3, worst
    eng.close()


def test_bf16_teacher_forced(case):
    fx, dims, sd = case
    bound = BF16_LOGIT_BOUND[fx["name"]]
    eps = 2 * bound
    rolling = [k for k, c in enumerate(fx["calls"]) if c["kind"] == "rolling"]
    forced = {k: fx["calls"][k]["tokens"] for k in rolling}
    sub = dict(fx, calls=[fx["calls"][k] for k in rolling])
    drafts = [forced[k] for k in rolling]
    # controlled gaps of every verify row, from the oracle on the same teacher-forced schedule
    orc = QwenTextOracle(dims, sd)
    gaps = []
    inner = orc.pick

    def pick(hist, off, ln, ctl, return_values=False):
        gaps.append([orc.controlled_gap([int(t) for t in hist[off[j]: off[j] + ln[j]]], ctl, j) for j in range(len(off))])
        return inner(hist, off, ln, ctl, return_values)

    orc.pick = pick
    ref = replay(orc, sub, drafts)
    assert [t for t, _ in ref] == drafts                    # the oracle accepts the reference's tokens whole
    eng = QwenTextEngine(dims, sd, precision="bf16", max_sessions=2, max_batch=2)
    log = capture_logits(eng, fx["stride"])
    verify_picks = []
    eng_pick = eng.pick

    def record(hist, off, ln, ctl, return_values=False):
        out = eng_pick(hist, off, ln, ctl, return_values)
        if len(off) > 1:                                    # the verify pick of a call (steps pick one row)
            verify_picks.append(np.asarray(out[0] if return_values else out))
        return out

    eng.pick = record
    replay(eng, sub, drafts)
    assert len(gaps) == len(rolling) == len(verify_picks)
    mismatched = []
    checked = total = 0
    for k, p, g in zip(rolling, verify_picks, gaps):
        want = forced[k]
        for j in range(len(want)):                          # row j's history is the reference's want[:j]
            total += 1
            if g[j] > eps:
                checked += 1
                if int(p[j]) != want[j]:
                    mismatched.append((k, j, int(p[j]), want[j], g[j]))
    # logit error of every verify row against the oracle's fp32 rows of the same teacher-forced forwards (the oracle
    # reproduces the reference's lm_head rows within 2e-5: tests/test_oracle_qwen_text.py)
    # (a near-tie the bf16 picks resolve differently adds single-row step forwards after that call's verify forward)
    verify = [a for a in log if a.shape[0] > 1]
    assert len(verify) == len(orc.logit_log)
    worst = max(float(np.abs(a - b[:, ::fx["stride"]]).max()) for a, b in zip(verify, orc.logit_log))
    print(f"{fx['name']} bf16 max|dlogits| = {worst:.3e} over {len(verify)} verify blocks; "
          f"{checked} of {total} verify picks above the gap bar")
    assert worst < bound, worst
    assert not mismatched, mismatched
    assert checked >= MIN_CHECKED[fx["name"]] * total, (checked, total)
    eng.close()


def test_ragged_batch_matches_the_oracle_per_session(fx, sd):
    dims = QWEN_TEXT_DIMS["tnano"]
    frames = fx["frames"]
    eng = QwenTextEngine(dims, sd, precision="fp32", max_sessions=4, max_batch=4)
    orc = QwenTextOracle(dims, sd)
    ctl = dict(repetition_penalty=1.15, no_repeat_ngram_size=3, suppress_token_ids=[7, 10, 11, 12, 13, 14])
    kw = dict(max_new_tokens=10, eos_token_id=fx["eos"], wait_token_id=fx["wait"], bos_token_id=fx["bos"], **ctl)
    n = 4
    es = [eng.open_session() for _ in range(n)]
    os_ = [orc.open_session() for _ in range(n)]
    e_state, o_state, prev = [None] * n, [None] * n, [None] * n
    schedule = [[3, 5, 8, 2], [7, 5, 12, 9], [7, 11, 20, 9], [10, 13, 21, 14]]
    for r, steps in enumerate(schedule):
        if r == 2:                                          # session 3 restarts (segment rollover)
            e_state[3] = o_state[3] = None
            prev[3] = None
            eng.reset_session(es[3]); orc.reset_session(os_[3])
        drafts = [None if p is None else (p[:2] + [99] + p[3:] if i == 1 else p) for i, p in enumerate(prev)]
        tpl = TEMPLATES["A" if r < 3 else "B"]
        fh = [frames[:s] for s in steps]
        toks, stats, e_state = eng.generate_rolling(es, fh, e_state, tpl, fx["placeholder"], drafts, **kw)
        for i in range(n):
            t, s, st = orc.generate_rolling([os_[i]], [fh[i]], [o_state[i]], tpl, fx["placeholder"], [drafts[i]], **kw)
            o_state[i] = st[0]
            assert toks[i] == t[0], (r, i, toks[i], t[0])
            assert stats[i] == s[0], (r, i, stats[i], s[0])
        prev = toks
    for s in es:
        eng.close_session(s)
    eng.close()


def _tie_weights(dims, seed):
    """lm_head rows repeat in groups of four: every logit ties with three neighbours."""
    sd = synthetic_text_state_dict(dims, seed)
    head = sd["lm_head.weight"]
    sd["lm_head.weight"] = np.repeat(head[::4], 4, axis=0)[:dims.vocab].copy()
    return sd


def _long_histories(logits, vocab, rng):
    """Histories of 600 .. 2000 tokens, longer than the pick kernel's 512-thread CTA, so its strided penalty and n-gram
    loops run several times: the rows' own best ids repeated across thread strides (the first occurrence must claim the
    penalty, whichever thread meets it), n-gram matches at both ends, ids outside the vocabulary, and a period-512
    history that puts every repeat on the same thread."""
    top = [[int(t) for t in torch.topk(logits[j], 6).indices] for j in range(logits.shape[0])]
    a, b = vocab - 7, vocab - 6                              # the n-gram prefix: nowhere else in these histories
    h8 = rng.integers(0, 64, 600)
    for k, i in enumerate([3, 515, 300, 599, 4, 516]):     # same thread (3 / 515, 4 / 516) and other threads
        h8[i] = top[8][k % 3]
    n = 1100
    h9 = rng.integers(100, 1000, n)
    h9[:3] = [a, b, top[9][0]]                               # matches at the first window ...
    h9[n - 5:n - 2] = [a, b, top[9][1]]                      # ... and the last windows
    h9[n - 2:] = [a, b]
    h10 = rng.integers(-3, vocab + 3, 2000)                  # a few ids outside [0, vocab): skipped by every control
    h10[0] = h10[1999] = top[10][0]
    h10[1024] = top[10][1]
    h11 = np.tile(rng.integers(0, vocab, 512), 4)[:1537]
    h11[[7, 519, 1031, 1536]] = top[11][0]
    return [[int(t) for t in h] for h in (h8, h9, h10, h11)]


def test_pick_kernel_adversarial_rows():
    """The pick kernel against the oracle's controls, at the tnano vocabulary and at Qwen3's 151936 ids (a 19 KB
    seen-bitmap), on short adversarial rows and on histories up to 4x the 512-thread CTA."""
    for vocab in (2048, 151936):
        _pick_adversarial_rows(vocab)


def _pick_adversarial_rows(vocab):
    dims = dataclasses.replace(QWEN_TEXT_DIMS["tnano"], vocab=vocab, max_ctx=64)
    eng = QwenTextEngine(dims, _tie_weights(dims, 5), precision="fp32", max_sessions=1, max_batch=1)
    sid = eng.open_session()
    n_rows = 12
    eng.forward([sid], [(np.arange(20, 20 + n_rows, dtype=np.int32), None)], [n_rows])
    logits = torch.as_tensor(eng.logits())
    top = [int(torch.argmax(logits[j])) for j in range(n_rows)]
    hists = [[], [top[1]], [top[2], top[2] + 1, 5, 6, 5], [5, 6, 7, 5, 6], [3] * 6, [1, 2, 1, 2, 1], list(range(40)),
             [top[7]] * 3] + _long_histories(logits, dims.vocab, np.random.default_rng(vocab))
    assert len(hists) == n_rows and min(len(h) for h in hists[8:]) >= 600
    everything = list(range(dims.vocab))
    cases = [
        eng.make_controls(),
        eng.make_controls(repetition_penalty=1.15, no_repeat_ngram_size=3, suppress_token_ids=[7, 10, 11]),
        eng.make_controls(suppress_token_ids=everything),                                   # all -inf
        eng.make_controls(suppress_token_ids=everything[2:], no_repeat_ngram_size=1),       # finfo.min next to -inf
        eng.make_controls(repetition_penalty=1.15, max_consecutive_text_tokens=3, wait_token_id=3),
        eng.make_controls(no_repeat_ngram_size=1, max_consecutive_text_tokens=2, wait_token_id=6),
        eng.make_controls(repetition_penalty=0.5, no_repeat_ngram_size=2, suppress_token_ids=top[:4]),
    ]
    off = np.zeros(n_rows, np.int32)
    ln = np.asarray([len(h) for h in hists], np.int32)
    off[1:] = np.cumsum(ln[:-1])
    flat = np.asarray([t for h in hists for t in h], np.int32)
    for ci, ctl in enumerate(cases):
        picks, vals = eng.pick(flat, off, ln, ctl, return_values=True)
        for j in range(n_rows):
            x = controlled_logits(logits[j], hists[j], ctl, dims.vocab)
            want = int(torch.argmax(x))
            assert int(picks[j]) == want, (vocab, ci, j, int(picks[j]), want)
            assert vals[j] == pytest.approx(float(x[want]), rel=1e-6), (vocab, ci, j, vals[j], float(x[want]))
    eng.close()


def test_error_contract(sd):
    dims = dataclasses.replace(QWEN_TEXT_DIMS["tnano"], max_ctx=16)
    eng = QwenTextEngine(dims, None, precision="fp32", max_sessions=2, max_batch=2)
    sid = eng.open_session()
    with pytest.raises(WlkError, match="not finalized"):
        eng.forward([sid], [(np.asarray([1, 2], np.int32), None)], [1])
    with pytest.raises(WlkError, match="wrong shape"):
        eng.load_tensor("norm.weight", np.ones(dims.d_model + 1, np.float32))
    with pytest.raises(WlkError, match="unknown tensor"):
        eng.load_tensor("layers.0.mlp.fc1.weight", np.ones((4, 4), np.float32))
    for name, arr in sd.items():
        if name != "layers.1.mlp.down_proj.weight":
            eng.load_tensor(name, arr)
    with pytest.raises(WlkError, match="missing"):
        eng.finalize()
    eng.load_tensor("layers.1.mlp.down_proj.weight", sd["layers.1.mlp.down_proj.weight"])
    eng.finalize()
    with pytest.raises(WlkError, match="invalid session"):
        eng.forward([sid + 1], [(np.asarray([1], np.int32), None)], [1])
    eng.forward([sid], [(np.arange(10, dtype=np.int32), None)], [1])
    with pytest.raises(WlkError, match="context full"):
        eng.forward([sid], [(np.arange(7, dtype=np.int32), None)], [1])
    assert eng.session_len(sid) == 10                       # the failed forward changed nothing
    eng.forward([sid], [(np.arange(6, dtype=np.int32), None)], [1])
    assert eng.session_len(sid) == 16
    eng.crop(sid, 4)
    assert eng.session_len(sid) == 4
    with pytest.raises(WlkError, match="crop"):
        eng.crop(sid, 5)
    eng.close_session(sid)
    eng.close()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_long_forward_and_many_logit_rows(precision):
    """One forward of 1100 rows (two rounds of the 1024-row workspace) with 1060 logit rows (three lm_head + pick groups
    at the 151936-id vocabulary), tied head, against the oracle: picks where the oracle's gap clears the bar, and the raw
    lm_head rows at the group seams."""
    dims = dataclasses.replace(QWEN_TEXT_DIMS["qwen3-asr-0.6b"], n_layer=2, max_ctx=2048)
    sd = synthetic_text_state_dict(dims, 12)
    eng = QwenTextEngine(dims, sd, precision=precision, max_sessions=2, max_batch=4)
    orc = QwenTextOracle(dims, sd)
    rng = np.random.default_rng(3)
    n_rows, n_logit = 1100, 1060
    emb = rng.standard_normal((300, dims.d_model)).astype(np.float32)
    src = np.concatenate([rng.integers(0, dims.vocab, 400), -1 - np.arange(300), rng.integers(0, dims.vocab, 400)]).astype(np.int32)
    hist = rng.integers(0, 5000, 64).astype(np.int32)
    ctl = eng.make_controls(repetition_penalty=1.15, no_repeat_ngram_size=3, suppress_token_ids=[1, 2, 3])
    off = np.zeros(n_logit, np.int32)
    ln = (np.arange(n_logit) % 65).astype(np.int32)
    results = {}
    for name, e in (("eng", eng), ("orc", orc)):
        sid = e.open_session()
        e.forward([sid], [(src, emb)], [n_logit])
        assert e.session_len(sid) == n_rows
        results[name] = (e.pick(hist, off, ln, ctl), e.logits(0, n_logit) if name == "orc" else None)
    picks, _ = results["eng"]
    want, orc_logits = results["orc"]
    seams = [0, 1, 439, 440, 441, 442, 880, 881, 882, 883, 1058, 1059]
    got_rows = np.concatenate([eng.logits(r, 1) for r in seams])
    err = float(np.abs(got_rows - orc_logits[seams]).max())
    tol = 1e-3 if precision == "fp32" else 0.28             # bf16: 2x the 1.38e-1 measured on H100 SXM (700 W)
    bar = 1e-2 if precision == "fp32" else 2 * tol
    checked = 0
    for j in range(n_logit):
        x = controlled_logits(torch.as_tensor(orc_logits[j]), [int(t) for t in hist[:ln[j]]], ctl, dims.vocab)
        top = torch.topk(x, 2).values
        if float(top[0] - top[1]) > bar:
            checked += 1
            assert int(picks[j]) == int(want[j]), (j, int(picks[j]), int(want[j]))
    print(f"long forward [{precision}]: max|dlogits| at the seams = {err:.3e}, {checked} of {n_logit} picks checked")
    assert err < tol, err
    assert checked >= 0.6 * n_logit
    eng.close()
