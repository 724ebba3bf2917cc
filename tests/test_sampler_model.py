"""The unique log-uniform sampler's statement (tests/sampler_model.py) and the C2V_NUM_SAMPLED switch, without a GPU.

  * The statement equals a plain transcription of TF's unique loop (RangeSampler::SampleBatchGetExpectedCountAvoid with
    unique=True: draw until S values are in the set, counting tries) on the same draws, over many (S, Y, seed, step) --
    S = 1, S = floor(Y / 2) at Y = 2, 3 and 1025, and steps whose first S draws are already distinct.
  * p sums to 1 over [0, Y) and single draws pass a chi-square test against it.
  * C2V_NUM_SAMPLED parses as a non-negative integer; several ranks, --framework b200-keras and values outside
    [1, min(1024, floor(Y / 2))] are refused before any engine exists; a run that does not train says the switch does
    nothing."""
import math
import os

import numpy as np
import pytest

from tests import sampler_model as SM


def tf_unique_loop(S, Y, seed, step):
    """TF's loop, transcribed: one uniform at a time, `static_cast<int64>(exp(x * log_range)) - 1` then `% range`."""
    log_range = math.log1p(Y)
    used, out, tries, i = set(), [], 0, 0
    while len(out) < S:
        x = float(SM.uniforms(seed, step, i, 1)[0])
        i += 1
        tries += 1
        value = (int(math.exp(x * log_range)) - 1) % Y
        if value not in used:
            used.add(value)
            out.append(value)
    return out, tries


CASES = [(1, 2), (1, 3), (1, 1025), (1, 261246), (512, 1025), (7, 15), (25, 100), (25, 261246), (100, 5003),
         (256, 261246), (1024, 261246), (1024, 2048)]


@pytest.mark.parametrize("S,Y", CASES)
def test_statement_equals_tf_loop(S, Y):
    for seed, step in ((0, 1), (7, 2), (0x5EED, 123456), (2 ** 40 + 3, 2 ** 33 + 1)):
        got, tries = SM.sample(S, Y, seed, step)
        want, want_tries = tf_unique_loop(S, Y, seed, step)
        assert got.tolist() == want and tries == want_tries, (S, Y, seed, step)
        assert len(set(got.tolist())) == S and got.min() >= 0 and got.max() < Y


def test_half_vocabulary_edges():
    """S = floor(Y / 2) at Y = 2 and 3 (one value from a set of two or three) over many steps."""
    for Y in (2, 3):
        seen = set()
        for step in range(1, 200):
            got, tries = SM.sample(Y // 2, Y, 11, step)
            assert ([int(got[0])], tries) == (tf_unique_loop(Y // 2, Y, 11, step)[0], tries) and tries == 1
            seen.add(int(got[0]))
        assert seen == set(range(Y))


def test_all_distinct_first_draws():
    """Steps whose first S draws are distinct: num_tries == S, and the counts are then S p(c)."""
    found = 0
    for step in range(1, 400):
        got, tries = SM.sample(3, 261246, 5, step)
        assert tries == tf_unique_loop(3, 261246, 5, step)[1]
        if tries == 3:
            found += 1
            c = got.astype(np.int64)
            assert np.array_equal(SM.logq(c, 261246, 3, tries), np.log(3 * SM.prob(c, 261246)).astype(np.float32))
    assert found > 0


def test_expected_counts_follow_tf():
    got, tries = SM.sample(200, 1000, 3, 9)
    assert tries > 200
    p = SM.prob(got, 1000)
    assert np.array_equal(SM.logq(got, 1000, 200, tries), np.log(-np.expm1(tries * np.log1p(-p))).astype(np.float32))


def test_probabilities_sum_to_one():
    for Y in (2, 3, 1025, 261246):
        assert abs(math.fsum(SM.prob(np.arange(Y), Y).tolist()) - 1.0) < 1e-12


def test_single_draws_follow_p():
    from scipy import stats
    Y, n = 40, 400000
    vals = SM.draws(1234, 1, Y, 0, n)
    obs = np.bincount(vals, minlength=Y)
    exp = n * SM.prob(np.arange(Y), Y)
    assert stats.chisquare(obs, exp).pvalue > 1e-3


def test_stream_differs_from_dropout_key():
    k = SM.key(0)
    assert k != (0, 0) and SM.key(2 ** 32 + 5) != (5, 1)
    a = SM.draws(1, 1, 1000, 0, 64)
    assert not np.array_equal(a, SM.draws(1, 2, 1000, 0, 64)) and not np.array_equal(a, SM.draws(2, 1, 1000, 0, 64))


def test_statement_refuses_out_of_range():
    for S, Y in ((0, 10), (6, 10), (1025, 4000), (1, 1)):
        with pytest.raises(ValueError):
            SM.sample(S, Y, 0, 1)


# ---- the switch ---------------------------------------------------------------------------------------------------------
def test_num_sampled_flag():
    from code2vec_b200.b200_model import check_num_sampled, num_sampled_flag
    assert num_sampled_flag({}) == 0
    assert num_sampled_flag({"C2V_NUM_SAMPLED": ""}) == 0
    assert num_sampled_flag({"C2V_NUM_SAMPLED": "0"}) == 0
    assert num_sampled_flag({"C2V_NUM_SAMPLED": "25"}) == 25
    for bad in ("-1", "2.5", "x", " 5", "5 ", "1e3"):
        with pytest.raises(ValueError, match="C2V_NUM_SAMPLED must be a non-negative integer"):
            num_sampled_flag({"C2V_NUM_SAMPLED": bad})
    check_num_sampled(1, 2)
    check_num_sampled(1024, 261246)
    check_num_sampled(512, 1025)
    for S, Y in ((0, 100), (513, 1025), (1025, 261246), (1, 1), (2, 3)):
        with pytest.raises(ValueError, match="C2V_NUM_SAMPLED=%d is outside" % S):
            check_num_sampled(S, Y)


def _cfg(**kw):
    from code2vec_b200.config import Config
    cfg = Config(set_defaults=True)
    cfg.VERBOSE_MODE = 0
    cfg.DL_FRAMEWORK = "b200"
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


@pytest.mark.parametrize("framework", ["b200", "b200-keras"])
def test_several_ranks_refuse_before_any_engine(monkeypatch, framework):
    from code2vec_b200 import load_model_dynamically
    monkeypatch.setenv("WORLD_SIZE", "2")
    monkeypatch.setenv("C2V_NUM_SAMPLED", "25")
    err = "C2V_NUM_SAMPLED=25: the sampled softmax trains on one GPU" if framework == "b200" else "runs on one GPU"
    with pytest.raises(ValueError, match=err):
        load_model_dynamically(_cfg(DL_FRAMEWORK=framework, TRAIN_BATCH_SIZE=1024))


def test_keras_backend_refuses(monkeypatch):
    from code2vec_b200.b200_keras_model import Code2VecModel
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    monkeypatch.setenv("C2V_NUM_SAMPLED", "25")
    with pytest.raises(ValueError, match="C2V_NUM_SAMPLED is not available with --framework b200-keras.*--framework b200"):
        Code2VecModel(_cfg(DL_FRAMEWORK="b200-keras"))
    monkeypatch.setenv("C2V_NUM_SAMPLED", "0")          # the default is accepted (the constructor then goes on)
    from code2vec_b200.b200_model import num_sampled_flag
    assert num_sampled_flag(os.environ) == 0


class _NoEngine(Exception):
    pass


def _model_until_engine(monkeypatch, cfg, env):
    """Code2VecModel(cfg) up to the point where it makes its engine: (log lines, exception raised)."""
    import code2vec_b200.b200_model as bm
    lines = []
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)

    def no_engine(*a, **k):
        raise _NoEngine()
    monkeypatch.setattr(bm, "PathAttentionEngine", no_engine)
    monkeypatch.setattr(bm.Code2VecModel, "log", lambda self, msg: lines.append(msg))
    try:
        bm.Code2VecModel(cfg)
    except Exception as exc:                  # noqa: BLE001 -- the test looks at which one
        return lines, exc
    return lines, None


def _toy(tmp_path):
    from tests.test_gpu_model import _config, _make_dataset
    prefix, _ = _make_dataset(tmp_path)
    return prefix, lambda **kw: _config(prefix, tmp_path, **kw)


def test_half_vocabulary_bound_and_loss_line(tmp_path, monkeypatch):
    prefix, make = _toy(tmp_path)
    Y = 9                                      # the toy's 8 method names and the special word
    lines, exc = _model_until_engine(monkeypatch, make(TRAIN_DATA_PATH_PREFIX=prefix), {"C2V_NUM_SAMPLED": str(Y // 2 + 1)})
    assert isinstance(exc, ValueError) and "C2V_NUM_SAMPLED=%d is outside [1, %d]" % (Y // 2 + 1, Y // 2) in str(exc)
    lines, exc = _model_until_engine(monkeypatch, make(TRAIN_DATA_PATH_PREFIX=prefix), {"C2V_NUM_SAMPLED": str(Y // 2)})
    assert isinstance(exc, _NoEngine)
    assert ("b200 backend training loss: sampled softmax, %d unique log-uniform negatives of the %d target words drawn on "
            "the GPU each step (C2V_NUM_SAMPLED=%d)" % (Y // 2, Y, Y // 2)) in lines
    lines, exc = _model_until_engine(monkeypatch, make(TRAIN_DATA_PATH_PREFIX=prefix), {"C2V_NUM_SAMPLED": "0"})
    assert isinstance(exc, _NoEngine)
    assert "b200 backend training loss: full softmax over the %d target words (C2V_NUM_SAMPLED=0)" % Y in lines
    assert not any("has no effect" in line for line in lines)


def test_no_effect_without_training(tmp_path, monkeypatch):
    from code2vec_b200.vocabularies import Code2VecVocabs
    prefix, make = _toy(tmp_path)
    save = str(tmp_path / "model" / "saved")
    os.makedirs(os.path.dirname(save))
    train_cfg = make(TRAIN_DATA_PATH_PREFIX=prefix)
    Code2VecVocabs(train_cfg).save(train_cfg.get_vocabularies_path_from_model_path(save))
    cfg = make(MODEL_LOAD_PATH=save, TEST_DATA_PATH=prefix + ".test.c2v")
    lines, exc = _model_until_engine(monkeypatch, cfg, {"C2V_NUM_SAMPLED": "3"})
    assert isinstance(exc, _NoEngine)
    assert "C2V_NUM_SAMPLED=3 has no effect: this run does not train (no --data)" in lines
    assert not any("training loss" in line for line in lines)
