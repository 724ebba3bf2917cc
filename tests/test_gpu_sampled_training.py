"""Sampled-softmax training with negatives drawn on the GPU (c2v_sample_log_uniform, Trainer.step_sampled,
C2V_NUM_SAMPLED; DESIGN.md §6j).

  * The sampler against its statement (tests/sampler_model.py): the ids and num_tries exactly, the log expected counts bit
    for bit -- a float32 that differs must come from a float64 value within a few double ulps of a float32 rounding
    boundary (CUDA's double log / expm1 / log1p are not correctly rounded) -- for S in {1, 25, 1023, 1024},
    Y in {small, 1025, 261,246}, B in {1, 37, 1024} and several (seed, step).  The same (seed, step) gives the same bits,
    the next step other ids; the call's refusals.
  * One Trainer.step_sampled against reference64.train_step64 on the ids it drew, within the sampled case's bounds.
  * Deterministic runs: two fresh runs give the same bits, and 2 steps + save + load + 2 steps equal 4 steps.
  * Code2VecModel with C2V_NUM_SAMPLED: learns the toy rule; the batch ring, the device reader and the synchronous path
    give the same losses and checkpoints; a mid-training evaluate() equals evaluate() on the checkpoint saved there; the
    command line trains, evaluates, exports and logs the loss line."""
import ctypes
import os

import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests import sampler_model as SM
from tests.util import dev_batch, make_engine

pytestmark = pytest.mark.gpu

SEEDS = [(0, 1), (7, 2), (0x5EED, 123456), (2 ** 40 + 3, 2 ** 33 + 1)]


def _sampler_engine(Y, max_batch=1024):
    from code2vec_b200.engine import EngineDims, PathAttentionEngine
    return PathAttentionEngine(EngineDims(8, 8, Y, 4, 4, 1, max_batch, 1), device=0, training=False)


def _check_logq(got, c, Y, S, tries, label):
    """got == the statement's float32, or the float64 value lies within 8 double ulps (of max(|x|, 1)) of the midpoint
    between the two float32s: a rounding boundary, where a last-bit difference of the double chain flips the float."""
    want = SM.logq(c, Y, S, tries)
    bad = got.view(np.uint32) != want.view(np.uint32)
    if bad.any():
        x = np.log(SM.expected_count64(np.asarray(c)[bad], Y, S, tries))
        g, w = got[bad].astype(np.float64), want[bad].astype(np.float64)
        adjacent = np.abs(np.nextafter(got[bad], want[bad]).astype(np.float64) - w) == 0
        mid = (g + w) / 2
        near = np.abs(x - mid) <= 8 * np.spacing(np.maximum(np.abs(x), 1.0))
        assert adjacent.all() and near.all(), (label, np.asarray(c)[bad][:5], g[:5], w[:5], x[:5])
    return int(bad.sum())


@pytest.mark.parametrize("Y", [64, 1025, 261246])
def test_sampler_equals_the_statement(Y):
    import torch
    eng = _sampler_engine(Y)
    rng = np.random.default_rng(Y)
    flips = 0
    for S in (1, 25, 1023, 1024):
        if S > Y // 2:
            continue
        for B in (1, 37, 1024):
            target = rng.integers(0, Y, size=B).astype(np.int32)
            target[0] = Y - 1
            tdev = eng.to_device(target, torch.int32)
            for seed, step in SEEDS:
                sampled, lq_t, lq_s, tries = eng.sample_log_uniform(tdev, S, seed, step)
                want, want_tries = SM.sample(S, Y, seed, step)
                label = "Y=%d S=%d B=%d seed=%d step=%d" % (Y, S, B, seed, step)
                assert int(tries.cpu()[0]) == want_tries, label
                assert np.array_equal(sampled.cpu().numpy(), want), label
                flips += _check_logq(lq_s.cpu().numpy(), want, Y, S, want_tries, label + " sampled")
                flips += _check_logq(lq_t.cpu().numpy(), target, Y, S, want_tries, label + " true")
    print("SAMPLER", Y, "logq values off by the rounding boundary:", flips)
    assert eng.get_option("sampler_cap_hits") == 0
    eng.close()


def test_sampler_replays_and_moves_on():
    import torch
    Y = 261246
    eng = _sampler_engine(Y)
    target = eng.to_device(np.arange(0, 1024 * 200, 200, dtype=np.int32), torch.int32)
    runs = []
    for step in (5, 5, 6):
        out = eng.sample_log_uniform(target, 1024, 3, step)
        runs.append([t.clone() for t in out])
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a, b)
    assert not torch.equal(runs[0][0], runs[2][0])
    other_seed = eng.sample_log_uniform(target, 1024, 4, 5)[0].clone()
    assert not torch.equal(runs[0][0], other_seed)
    eng.close()


def test_sampler_refusals():
    import torch
    from code2vec_b200.engine import EngineError, c2v_table_shards
    eng = _sampler_engine(100, max_batch=8)
    target = eng.to_device(np.zeros(8, dtype=np.int32), torch.int32)
    for S, B in ((0, 8), (51, 8), (1025, 8), (-1, 8)):
        with pytest.raises(EngineError) as ei:
            eng.sample_log_uniform(target[:B], S, 0, 1)
        assert ei.value.code == -1
    big = eng.to_device(np.zeros(9, dtype=np.int32), torch.int32)
    with pytest.raises(EngineError) as ei:
        eng.sample_log_uniform(big, 5, 0, 1)
    assert ei.value.code == -1
    eng.sample_log_uniform(target, 50, 0, 1)                  # S = Y / 2 is accepted
    st = c2v_table_shards()
    st.world, st.rank = 2, 0
    for r in range(2):
        st.tok[r], st.path[r] = eng.params["tok"].data_ptr(), eng.params["path"].data_ptr()
    assert eng.lib.c2v_bind_table_shards(eng.h, ctypes.byref(st), None, 0.5) == 0
    with pytest.raises(EngineError) as ei:
        eng.sample_log_uniform(target, 5, 0, 1)
    assert ei.value.code == -4 and "single-GPU" in str(ei.value)
    eng.close()


# ---- one step against float64 --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("math", [0, 1, 2])
def test_step_sampled_against_float64(math):
    import torch
    from code2vec_b200.trainer import Trainer
    from tests import reference64 as R
    from tests.test_gpu_reference64 import KEEP, LOSS_TOL, SAMP, SEED, check_adam_slots, report
    B, S = 200, 64
    params = O.init_params(SAMP, seed=4321)
    batch = O.synthetic_batch(SAMP, B, seed=77)
    eng, _ = make_engine(SAMP, max_batch=B, params=params)
    eng.set_option("math_mode", math)
    tr = Trainer(eng, keep_prob=KEEP, seed=SEED)
    d = dev_batch(eng, *batch)
    sampled, tries = SM.sample(S, SAMP.target_vocab, SEED, 1)
    lq_t = SM.logq(batch[4], SAMP.target_vocab, S, tries)
    lq_s = SM.logq(sampled, SAMP.target_vocab, S, tries)
    dm = O.dropout_keep_mask(SEED, 1, B * SAMP.max_contexts, SAMP.ctx_dim, KEEP)
    ref = R.train_step64(params, *batch, keep=KEEP, dropout_mask=dm, sampled=sampled, logq_true=lq_t, logq_sampled=lq_s)
    loss = float(tr.step_sampled(*d, S).cpu()[0])
    got = eng._sampler_out
    assert np.array_equal(got[0][:S].cpu().numpy(), sampled) and int(got[3].cpu()[0]) == tries
    assert abs(loss - ref.loss) < LOSS_TOL
    eng.sync_tables()
    label = "step_sampled math=%d" % math
    worst = check_adam_slots(eng, ref, math, O.PARAM_NAMES, label)
    worst["loss"] = abs(loss - ref.loss)
    report(label, worst)
    eng.close()


# ---- determinism and resume --------------------------------------------------------------------------------------------
DET = O.Dims(token_vocab=3001, path_vocab=2003, target_vocab=4001, embed_dim=32, code_dim=96, max_contexts=20)
DET_B, DET_S = 96, 100


def _state(eng):
    eng.sync_tables()
    out = {}
    for group, d in (("theta", eng.params), ("m", eng.adam_m), ("v", eng.adam_v)):
        for k in O.PARAM_NAMES:
            out[group + "/" + k] = d[k].detach().cpu().numpy().copy()
    return out


def _run(steps, state=None, adam_t=0, first=0):
    import torch
    from code2vec_b200.trainer import Trainer
    eng, _ = make_engine(DET, max_batch=DET_B, params=None if state is None else {k: state["theta/" + k] for k in O.PARAM_NAMES})
    eng.set_option("math_mode", 1)
    if state is not None:
        for k in O.PARAM_NAMES:
            eng.adam_m[k].copy_(torch.from_numpy(state["m/" + k]))
            eng.adam_v[k].copy_(torch.from_numpy(state["v/" + k]))
        eng.adam_t = adam_t
        eng.set_option("adam_step_count", adam_t)
    tr = Trainer(eng, keep_prob=0.75, seed=99, deterministic=True)
    losses = []
    for i in range(first, first + steps):
        batch = O.synthetic_batch(DET, DET_B, seed=1000 + i)
        losses.append(float(tr.step_sampled(*dev_batch(eng, *batch), DET_S).cpu()[0]))
    st, t = _state(eng), eng.adam_t
    eng.close()
    return losses, st, t


def test_deterministic_runs_and_resume():
    l1, s1, t1 = _run(4)
    l2, s2, _ = _run(4)
    assert l1 == l2 and all(np.array_equal(s1[k].view(np.uint32), s2[k].view(np.uint32)) for k in s1)
    la, sa, ta = _run(2)
    lb, sb, tb = _run(2, state=sa, adam_t=ta, first=2)
    assert tb == t1 == 4
    assert la + lb == l1
    for k in s1:
        assert np.array_equal(sb[k].view(np.uint32), s1[k].view(np.uint32)), k


# ---- the model ---------------------------------------------------------------------------------------------------------
def _losses_of(monkeypatch):
    """Every step_sampled's loss, kept on the device until the end (no sync added)."""
    from code2vec_b200.trainer import Trainer
    seen = []
    orig = Trainer.step_sampled

    def step(self, *a, **k):
        loss = orig(self, *a, **k)
        seen.append(loss.clone())
        return loss
    monkeypatch.setattr(Trainer, "step_sampled", step)
    return seen


def test_model_learns_the_toy_rule(tmp_path, monkeypatch):
    from code2vec_b200.b200_model import Code2VecModel
    from tests.test_gpu_model import _config, _make_dataset
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv("C2V_NUM_SAMPLED", "4")
    prefix, _ = _make_dataset(tmp_path)
    cfg = _config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, MODEL_SAVE_PATH=str(tmp_path / "m" / "saved"),
                  TEST_DATA_PATH=prefix + ".test.c2v", DROPOUT_KEEP_RATE=1.0)
    model = Code2VecModel(cfg)
    seen = _losses_of(monkeypatch)
    model.train()
    assert len(seen) == 150 * 3
    res = model.evaluate()
    assert res.topk_acc[0] > 0.6, res
    assert model.engine.get_option("sampler_cap_hits") == 0
    model.close_session()


def test_routes_agree(tmp_path, monkeypatch):
    """C2V_DETERMINISTIC=1: the batch ring, the device reader and the synchronous path give the same per-step losses and
    the same checkpoint bytes."""
    from code2vec_b200.b200_model import Code2VecModel
    from tests.test_gpu_model import _config, _make_dataset
    monkeypatch.chdir(tmp_path)
    prefix, _ = _make_dataset(tmp_path, n_train=101)
    out = {}
    for route, env in (("ring", {}), ("device_reader", {"C2V_DEVICE_READER": "1"}),
                       ("synchronous", {"C2V_BATCH_RING": "0", "C2V_HINT_NEXT": "1"})):
        with monkeypatch.context() as m:
            for k, v in dict({"C2V_DETERMINISTIC": "1", "C2V_SEED": "7", "C2V_NUM_SAMPLED": "3"}, **env).items():
                m.setenv(k, v)
            save = str(tmp_path / route / "saved")
            cfg = _config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, MODEL_SAVE_PATH=save, NUM_TRAIN_EPOCHS=5,
                          NUM_BATCHES_TO_LOG_PROGRESS=3, SHUFFLE_BUFFER_SIZE=40, DROPOUT_KEEP_RATE=0.75)
            model = Code2VecModel(cfg)
            lines = []
            model.log = lines.append
            seen = _losses_of(m)
            model.train()
            model.close_session()
            assert any(line.startswith("Average loss at batch 3: ") for line in lines), route
            with open(save + ".c2v_b200", "rb") as f:
                out[route] = ([float(x.cpu()[0]) for x in seen], f.read())
    (l0, c0) = out["ring"]
    assert len(l0) == -(-101 * 5 // 32)                     # the reader batches the 5 epochs as one stream
    for route, (losses, ckpt) in out.items():
        assert losses == l0 and ckpt == c0, route


def test_mid_training_evaluate_equals_the_saved_checkpoint(tmp_path, monkeypatch):
    """Evaluation mid-training reads the whole target table: its lazily updated rows must be current by then."""
    from code2vec_b200.b200_model import Code2VecModel
    from tests.test_gpu_model import _config, _make_dataset
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv("C2V_NUM_SAMPLED", "4")
    prefix, _ = _make_dataset(tmp_path)
    save = str(tmp_path / "m" / "saved")
    cfg = _config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, MODEL_SAVE_PATH=save, TEST_DATA_PATH=prefix + ".test.c2v",
                  NUM_TRAIN_EPOCHS=4, SAVE_EVERY_EPOCHS=2)
    model = Code2VecModel(cfg)
    results = []
    orig = Code2VecModel.evaluate

    def evaluate(self):
        r = orig(self)
        results.append(r)
        return r
    monkeypatch.setattr(Code2VecModel, "evaluate", evaluate)
    model.train()
    model.close_session()
    assert len(results) == 2
    for epoch, r in zip((2, 4), results):
        cfg2 = _config(prefix, tmp_path, MODEL_LOAD_PATH=save + "_iter%d" % epoch, TEST_DATA_PATH=prefix + ".test.c2v")
        m2 = Code2VecModel(cfg2)
        r2 = orig(m2)
        m2.close_session()
        assert np.array_equal(r.topk_acc, r2.topk_acc) and r.subtoken_f1 == r2.subtoken_f1, (epoch, r, r2)


def test_command_line(tmp_path, monkeypatch):
    from code2vec_b200.__main__ import main
    from code2vec_b200.b200_model import Code2VecModel
    from tests.test_gpu_model import _make_dataset
    import tests.test_gpu_model as toy
    monkeypatch.setattr(toy, "C", 200)
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv("C2V_NUM_SAMPLED", "4")
    lines = []
    monkeypatch.setattr(Code2VecModel, "log", lambda self, msg: lines.append(msg))
    prefix, _ = _make_dataset(tmp_path)
    save = str(tmp_path / "cli" / "saved")
    assert main(["--data", prefix, "--test", prefix + ".test.c2v", "--save", save, "--framework", "b200",
                 "--save_t2v", str(tmp_path / "tgt.w2v")]) == 0
    assert ("b200 backend training loss: sampled softmax, 4 unique log-uniform negatives of the 9 target words drawn on "
            "the GPU each step (C2V_NUM_SAMPLED=4)") in lines
    assert any(line.startswith("After 1 epochs -- top10_acc: [") for line in lines)
    assert os.path.exists(save + ".c2v_b200") and os.path.exists(save + "_iter1.c2v_b200")
    assert open(str(tmp_path / "tgt.w2v")).readline().split() == ["9", "384"]
    del lines[:]
    assert main(["--load", save, "--test", prefix + ".test.c2v", "--framework", "b200"]) == 0
    assert "C2V_NUM_SAMPLED=4 has no effect: this run does not train (no --data)" in lines
    assert not any("training loss" in line for line in lines)
