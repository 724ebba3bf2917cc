"""The sampled-softmax step on a row-sharded target table, without a GPU.

  * tests/sharded_sampled_model.py (pack, head, partials, fold) on W in {1, 2, 4, 8} ranks equals, in float64, the
    sampled softmax of oracle.path_attention_oracle on the global batch: loss, dv and the target-table gradient --
    with a rank that owns no negative, a rank that owns none of its own examples' targets, accidental hits, ids at a
    block's first row and the row before it, Y not divisible by W, targets shared across ranks and short batches.
  * The model's block split is the trainer's.
  * C2V_SHARDED_SAMPLED parses as 0 / 1; it needs C2V_NUM_SAMPLED; without it several ranks keep their refusal, with it
    they pass it; on one GPU it is accepted and logged as having no effect.
"""
import os

import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests import sharded_sampled_model as M


def _case(Y, D, world, Bl, rng, sampled=None, target=None):
    Bt = world * Bl
    Yt = rng.standard_normal((Y, D)) * 0.5
    v = rng.standard_normal((Bt, D)) * 0.5
    if target is None:
        target = rng.integers(0, Y, Bt)
    if sampled is None:
        sampled = rng.choice(Y, size=min(25, Y // 2), replace=False)
    target, sampled = np.asarray(target, np.int64), np.asarray(sampled, np.int64)
    lq_t = rng.standard_normal(Bt) - 3.0
    lq_s = rng.standard_normal(len(sampled)) - 3.0
    return Yt, v, target, sampled, lq_t, lq_s


def _check(Yt, v, target, sampled, lq_t, lq_s, world):
    loss, dv, g, parts = M.step(Yt, v, target, sampled, lq_t, lq_s, world)
    ref_loss, ref_dv, ref_g, _ = O.sampled_softmax_loss_and_grads({"tgt": Yt}, v, target, sampled, lq_t, lq_s,
                                                                  dtype=np.float64)
    assert len(parts) == world
    np.testing.assert_allclose(loss, ref_loss, rtol=1e-12, atol=0)
    np.testing.assert_allclose(dv, ref_dv, rtol=1e-10, atol=1e-15)
    np.testing.assert_allclose(g, ref_g, rtol=1e-10, atol=1e-15)
    touched = np.zeros(len(Yt), bool)
    touched[target] = touched[sampled] = True
    assert not g[~touched].any()                 # rows nobody references are exactly zero
    return g


@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_random_batches_against_the_oracle(world):
    rng = np.random.default_rng(world)
    for Y, Bl in ((1001, 6), (97, 3), (4096, 70)):      # 1001 and 97 are not multiples of any W > 1; 70 > one chunk
        _check(*_case(Y, 8, world, Bl, rng), world)


@pytest.mark.parametrize("world", [2, 4, 8])
def test_edge_cases(world):
    rng = np.random.default_rng(100 + world)
    Y, D, Bl = 1001, 12, 5
    blocks = [M.target_row_block(Y, r, world) for r in range(world)]
    last0, last1 = blocks[-1]
    # every negative in rank 0's block: the other ranks own none
    _check(*_case(Y, D, world, Bl, rng, sampled=rng.choice(blocks[0][1], 20, replace=False)), world)
    # rank 0's examples all target the last rank's rows, and the other ranks' examples rank 0's rows
    tgt = np.concatenate([rng.integers(last0, last1, Bl), rng.integers(0, blocks[0][1], (world - 1) * Bl)])
    _check(*_case(Y, D, world, Bl, rng, target=tgt), world)
    # accidental hits: every example's target is among the negatives, on every rank
    samp = rng.choice(Y, 30, replace=False)
    _check(*_case(Y, D, world, Bl, rng, sampled=samp, target=rng.choice(samp, world * Bl)), world)
    # ids at each block's first row and the row before it, as negatives and as targets; the same target on every rank
    edges = sorted({r0 for r0, _ in blocks[1:]} | {r0 - 1 for r0, _ in blocks[1:]} | {0, Y - 1})
    tgt = np.resize(np.array(edges), world * Bl)
    tgt[::Bl] = edges[1]
    g = _check(*_case(Y, D, world, Bl, rng, sampled=np.array(edges), target=tgt), world)
    assert g[edges].any(axis=1).all()
    # short batch: one example per rank
    _check(*_case(Y, D, world, 1, rng), world)


def test_block_split_is_the_trainers():
    from code2vec_b200.trainer import target_row_block
    for Y in (9, 1001, 261246):
        for W in (1, 2, 4, 8):
            for r in range(W):
                assert M.target_row_block(Y, r, W) == target_row_block(Y, r, W)


def test_float32_statement_is_close_to_float64():
    rng = np.random.default_rng(7)
    Yt, v, target, sampled, lq_t, lq_s = _case(2000, 16, 4, 40, rng)
    l64, dv64, g64, _ = M.step(Yt, v, target, sampled, lq_t, lq_s, 4)
    l32, dv32, g32, _ = M.step(Yt.astype(np.float32), v.astype(np.float32), target, sampled, lq_t.astype(np.float32),
                               lq_s.astype(np.float32), 4)
    assert abs(float(l32) - l64) < 1e-5 * abs(l64)
    assert np.abs(g32 - g64).max() < 1e-5 * np.abs(g64).max()


# ---- the switch ---------------------------------------------------------------------------------------------------------
def test_sharded_sampled_flag():
    from code2vec_b200.b200_model import sharded_sampled_flag
    assert sharded_sampled_flag({}) is False
    assert sharded_sampled_flag({"C2V_SHARDED_SAMPLED": ""}) is False
    assert sharded_sampled_flag({"C2V_SHARDED_SAMPLED": "0"}) is False
    assert sharded_sampled_flag({"C2V_SHARDED_SAMPLED": "1"}) is True
    for bad in ("2", "yes", " 1", "true", "-1"):
        with pytest.raises(ValueError, match="C2V_SHARDED_SAMPLED must be 0 or 1"):
            sharded_sampled_flag({"C2V_SHARDED_SAMPLED": bad})


def _cfg(**kw):
    from code2vec_b200.config import Config
    cfg = Config(set_defaults=True)
    cfg.VERBOSE_MODE = 0
    cfg.DL_FRAMEWORK = "b200"
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


class _Joined(Exception):
    pass


def test_switch_refusals_and_acceptance_on_several_ranks(monkeypatch):
    import code2vec_b200.b200_model as bm
    from code2vec_b200 import load_model_dynamically
    monkeypatch.setenv("WORLD_SIZE", "2")

    def joined(self):
        raise _Joined()
    monkeypatch.setattr(bm.Code2VecModel, "_join_group", joined)
    monkeypatch.setenv("C2V_SHARDED_SAMPLED", "1")
    monkeypatch.delenv("C2V_NUM_SAMPLED", raising=False)
    with pytest.raises(ValueError, match="C2V_SHARDED_SAMPLED=1 .* needs C2V_NUM_SAMPLED"):
        load_model_dynamically(_cfg(TRAIN_BATCH_SIZE=1024))
    monkeypatch.setenv("C2V_SHARDED_SAMPLED", "2")
    monkeypatch.setenv("C2V_NUM_SAMPLED", "25")
    with pytest.raises(ValueError, match="C2V_SHARDED_SAMPLED must be 0 or 1"):
        load_model_dynamically(_cfg(TRAIN_BATCH_SIZE=1024))
    # without the switch the one-GPU refusal stands; with it the constructor goes on to join the process group
    monkeypatch.setenv("C2V_SHARDED_SAMPLED", "0")
    with pytest.raises(ValueError, match="C2V_NUM_SAMPLED=25: the sampled softmax trains on one GPU"):
        load_model_dynamically(_cfg(TRAIN_BATCH_SIZE=1024))
    monkeypatch.setenv("C2V_SHARDED_SAMPLED", "1")
    with pytest.raises(_Joined):
        load_model_dynamically(_cfg(TRAIN_BATCH_SIZE=1024))
    # the Keras backend stays refused
    with pytest.raises(ValueError, match="runs on one GPU"):
        load_model_dynamically(_cfg(DL_FRAMEWORK="b200-keras", TRAIN_BATCH_SIZE=1024))


def test_keras_backend_refuses_the_switch(monkeypatch):
    from code2vec_b200.b200_keras_model import Code2VecModel
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    monkeypatch.setenv("C2V_NUM_SAMPLED", "25")
    monkeypatch.setenv("C2V_SHARDED_SAMPLED", "1")
    with pytest.raises(ValueError, match="not available with --framework b200-keras"):
        Code2VecModel(_cfg(DL_FRAMEWORK="b200-keras"))


def test_one_gpu_accepts_and_logs_no_effect(tmp_path, monkeypatch):
    from tests.test_sampler_model import _model_until_engine, _NoEngine, _toy
    prefix, make = _toy(tmp_path)
    lines, exc = _model_until_engine(monkeypatch, make(TRAIN_DATA_PATH_PREFIX=prefix),
                                     {"C2V_NUM_SAMPLED": "4", "C2V_SHARDED_SAMPLED": "1"})
    assert isinstance(exc, _NoEngine)
    assert "C2V_SHARDED_SAMPLED=1 has no effect on one GPU: the sampled softmax runs its one-GPU step" in lines
    lines, exc = _model_until_engine(monkeypatch, make(TRAIN_DATA_PATH_PREFIX=prefix), {"C2V_NUM_SAMPLED": "4",
                                                                                         "C2V_SHARDED_SAMPLED": "0"})
    assert isinstance(exc, _NoEngine)
    assert not any("C2V_SHARDED_SAMPLED" in line for line in lines)
    assert os.environ.get("C2V_SHARDED_SAMPLED") == "0"
