"""evaluate() on the GPU (C2V_DEVICE_EVAL=1: device_reader.py evaluate mode, csrc/reader.cu eval kernels) against the host
evaluation it replaces: equal ModelEvaluationResults (== on every float), byte-identical log.txt and .vectors, the same
top-k ids per batch, the same errors, the same per-epoch lines in train(), and the same outputs on 2 and 4 emulated ranks.
The toy dataset is tests/test_gpu_model's, with extra target words and hand-written adversarial names."""
import os
import pickle

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

EXTRA_TARGETS = ["|", "a||b", "get|x", "get|get|x", "getx", "get_x2", "x1", "name|copy|copy"]
ADVERSARIAL = ["", "<OOV>", "a,b", "get2x", "_", "123", "|", "||", "|get", "get|", "get|get|x", "getX", "get|x", "GETX",
               "get_x", "a||b", "ü", "K", "KelvinK", "name|ü", "copy|copy|name", "read|name,x"]


@pytest.fixture
def _ten_target_rows(monkeypatch):
    """A ninth method name in the toy data, so that 4 ranks all hold target rows (as tests/test_gpu_multi_rank_model)."""
    import tests.test_gpu_model as toy
    monkeypatch.setattr(toy, "TARGETS", toy.TARGETS + ["make|copy"])


def _dataset(tmp_path, n_test=150, adversarial=True, seed=0):
    """The toy dataset with EXTRA_TARGETS in the target vocabulary and, appended to the test file, one line per
    adversarial name (the contexts of a synthetic test line), plus a blank line and a line with no valid context."""
    from tests.test_gpu_model import _make_dataset
    prefix, test = _make_dataset(tmp_path, n_test=n_test, seed=seed)
    with open(prefix + ".dict.c2v", "rb") as f:
        dicts = [pickle.load(f) for _ in range(3)] + [pickle.load(f)]
    for w in EXTRA_TARGETS:
        dicts[2][w] = 1
    with open(prefix + ".dict.c2v", "wb") as f:
        for d in dicts:
            pickle.dump(d, f)
    if adversarial:
        ctx = [t.split(" ", 1)[1] for t in test]
        C = len(test[0].split(" ")) - 1
        lines = ["%s %s" % (name, ctx[i % len(ctx)]) for i, name in enumerate(ADVERSARIAL)]
        lines.insert(3, "")
        lines.insert(7, "dropped " + " " * (C - 1))
        with open(prefix + ".test.c2v", "a", encoding="utf-8") as f:
            f.write("\n".join(lines) + "\n")
    return prefix


def _train(prefix, tmp_path, epochs=3):
    from code2vec_b200.b200_model import Code2VecModel
    from tests.test_gpu_model import _config
    save = str(tmp_path / "model" / "saved")
    m = Code2VecModel(_config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, MODEL_SAVE_PATH=save,
                              NUM_TRAIN_EPOCHS=epochs))
    try:
        m.train()
    finally:
        m.close_session()
    return save


def _evaluate(monkeypatch, prefix, tmp_path, save, flag, **kw):
    """(results, log.txt bytes, .vectors bytes) of evaluate() on a model loaded from `save`, C2V_DEVICE_EVAL=flag."""
    from code2vec_b200.b200_model import Code2VecModel
    from tests.test_gpu_model import _config
    monkeypatch.setenv("C2V_DEVICE_EVAL", flag)
    vectors = prefix + ".test.c2v.vectors"
    if os.path.exists(vectors):
        os.remove(vectors)
    m = Code2VecModel(_config(prefix, tmp_path, MODEL_LOAD_PATH=save, TEST_DATA_PATH=prefix + ".test.c2v",
                              EXPORT_CODE_VECTORS=True, **kw))
    try:
        res = m.evaluate()
        assert (m._dev_eval_reader is not None) == (flag == "1")      # the route the switch names was taken
    finally:
        m.close_session()
    return res, open("log.txt", "rb").read(), open(vectors, "rb").read()


def _assert_same(a, b):
    (ra, la, va), (rb, lb, vb) = a, b
    assert np.array_equal(ra.topk_acc, rb.topk_acc) and ra.topk_acc.dtype == rb.topk_acc.dtype
    assert (ra.subtoken_precision, ra.subtoken_recall, ra.subtoken_f1) == (
        rb.subtoken_precision, rb.subtoken_recall, rb.subtoken_f1)
    assert str(ra) == str(rb)
    assert la == lb, "log.txt differs"
    assert va == vb, ".vectors differs"


@pytest.mark.parametrize("batch,chunk", [(32, None), (1, None), (7, 600), (1024, None), (7, None), (1024, 900)])
def test_device_evaluation_equals_the_host(tmp_path, monkeypatch, batch, chunk):
    from tests.test_gpu_device_reader import _small_chunks
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    prefix = _dataset(tmp_path)
    save = _train(prefix, tmp_path)
    if chunk:
        _small_chunks(monkeypatch, chunk)            # batches cross chunk boundaries
    host = _evaluate(monkeypatch, prefix, tmp_path, save, "0", TEST_BATCH_SIZE=batch)
    dev = _evaluate(monkeypatch, prefix, tmp_path, save, "1", TEST_BATCH_SIZE=batch)
    _assert_same(dev, host)
    log = host[1].decode("utf-8")
    assert "No results for predicting: " in log and "predicted 1st" in log
    assert host[1].count(b"\n") >= 10


def test_ids_equal_predict_batch_host(tmp_path, monkeypatch):
    """Per batch, forward + topk on the device batch gives predict_batch_host's ids bit for bit in the evaluation math."""
    import torch
    from code2vec_b200.b200_model import Code2VecModel
    from tests.test_gpu_model import _config
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    prefix = _dataset(tmp_path)
    save = _train(prefix, tmp_path)
    monkeypatch.setenv("C2V_DEVICE_EVAL", "1")
    m = Code2VecModel(_config(prefix, tmp_path, MODEL_LOAD_PATH=save, TEST_DATA_PATH=prefix + ".test.c2v",
                              TEST_BATCH_SIZE=13))
    try:
        e = m.engine
        e.set_option("math_mode", m._math_eval)
        reader = m._device_eval_reader()
        n_batches = 0
        for batch in reader:
            batch.wait()
            code, _ = e.forward(*batch.tensors[:4], want_attention=False)
            ids, _ = e.topk(code, normalize=False)
            host = [t.cpu().numpy() for t in batch.tensors[:4]]
            torch.cuda.synchronize()
            want, _, _, _ = e.predict_batch_host(*host, normalize=False, want_code=False, want_attention=False)
            assert np.array_equal(ids.cpu().numpy(), want)
            batch.release()
            n_batches += 1
        assert n_batches >= 10
        held = reader.device_bytes()
        assert held > 0
    finally:
        m.close_session()
    assert m._dev_eval_reader is None and m._device_vocabs is None


def test_errors_match_the_host(tmp_path, monkeypatch):
    from code2vec_b200.b200_model import Code2VecModel
    from tests.test_gpu_model import _config
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    prefix = _dataset(tmp_path, adversarial=False)
    save = _train(prefix, tmp_path, epochs=1)
    good = open(prefix + ".test.c2v", "rb").read().splitlines()

    def run(flag, text):
        with open(prefix + ".test.c2v", "wb") as f:
            f.write(text)
        monkeypatch.setenv("C2V_DEVICE_EVAL", flag)
        m = Code2VecModel(_config(prefix, tmp_path, MODEL_LOAD_PATH=save, TEST_DATA_PATH=prefix + ".test.c2v",
                                  TEST_BATCH_SIZE=7))
        try:
            m.evaluate()
        finally:
            m.close_session()

    malformed = b"\n".join(good[:20] + [good[20] + b" extra"] + good[21:]) + b"\n"
    invalid_utf8 = b"\n".join(good[:5] + [b"\xff\xfe" + good[5][good[5].index(b" "):]] + good[6:]) + b"\n"
    for text, exc in ((malformed, ValueError), (invalid_utf8, UnicodeDecodeError)):
        with pytest.raises(exc) as host:
            run("0", text)
        with pytest.raises(exc) as dev:
            run("1", text)
        if exc is ValueError:
            assert str(dev.value) == str(host.value)


def test_no_legal_word_raises_index_error_in_both_routes(tmp_path, monkeypatch):
    """A target vocabulary without a legal word (every name has a digit): SubtokensEvaluationMetric raises IndexError."""
    import tests.test_gpu_model as toy
    from code2vec_b200.b200_model import Code2VecModel
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    monkeypatch.setattr(toy, "TARGETS", ["x%d" % i for i in range(len(toy.TARGETS))])
    prefix = _dataset(tmp_path, adversarial=False)
    with open(prefix + ".dict.c2v", "rb") as f:
        dicts = [pickle.load(f) for _ in range(4)]
    dicts[2] = {w: n for w, n in dicts[2].items() if w not in EXTRA_TARGETS}
    with open(prefix + ".dict.c2v", "wb") as f:
        for d in dicts:
            pickle.dump(d, f)
    save = _train(prefix, tmp_path, epochs=1)
    for flag in ("0", "1"):
        monkeypatch.setenv("C2V_DEVICE_EVAL", flag)
        m = Code2VecModel(toy._config(prefix, tmp_path, MODEL_LOAD_PATH=save, TEST_DATA_PATH=prefix + ".test.c2v"))
        try:
            with pytest.raises(IndexError):
                m.evaluate()
        finally:
            m.close_session()


def test_per_epoch_evaluation_in_train(tmp_path, monkeypatch):
    from code2vec_b200.b200_model import Code2VecModel
    from tests.test_gpu_model import _config
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    prefix = _dataset(tmp_path)
    lines = {}
    orig = Code2VecModel.log
    for flag in ("0", "1"):
        got = lines[flag] = []

        def log(self, msg, got=got):
            if str(msg).startswith("After "):
                got.append(msg)
            return orig(self, msg)
        with monkeypatch.context() as m:
            m.setattr(Code2VecModel, "log", log)
            for k, v in {"C2V_DETERMINISTIC": "1", "C2V_SEED": "7", "C2V_DEVICE_READER": "1",
                         "C2V_DEVICE_EVAL": flag}.items():
                m.setenv(k, v)
            model = Code2VecModel(_config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, TEST_DATA_PATH=prefix + ".test.c2v",
                                          NUM_TRAIN_EPOCHS=3, SAVE_EVERY_EPOCHS=1, TEST_BATCH_SIZE=7))
            try:
                model.train()
            finally:
                model.close_session()
    assert len(lines["0"]) == 3 and lines["1"] == lines["0"]


@pytest.mark.parametrize("world", [2, 4])
def test_ranks_equal_one_gpu_host_evaluation(tmp_path, monkeypatch, _ten_target_rows, world):
    from tests.test_gpu_model import _config
    from tests.test_gpu_multi_rank_model import _models
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    prefix = _dataset(tmp_path, n_test=60)
    save = _train(prefix, tmp_path, epochs=5)
    host = _evaluate(monkeypatch, prefix, tmp_path, save, "0", TEST_BATCH_SIZE=50)
    os.remove(prefix + ".test.c2v.vectors")
    make = lambda: _config(prefix, tmp_path, MODEL_LOAD_PATH=save, TEST_DATA_PATH=prefix + ".test.c2v",
                           EXPORT_CODE_VECTORS=True, TEST_BATCH_SIZE=50)
    got = _models(monkeypatch, world, make, lambda model, r: model.evaluate(), {"C2V_DEVICE_EVAL": "1"})
    for r in range(world):
        _assert_same((got[r], open("log.txt", "rb").read(), open(prefix + ".test.c2v.vectors", "rb").read()), host)
