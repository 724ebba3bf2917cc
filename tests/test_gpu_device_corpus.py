"""`--score_names` and `--nearest` on the GPU (C2V_DEVICE_EVAL=1, DESIGN.md §6o) against the host route they replace, on
the same loaded model in one process: byte-identical `.name_scores` and `.nearest` files, equal returned arrays (NaNs in
the same places), the same summary and log lines, and the same exceptions with no file left for a corpus the reader
rejects.  The toy dataset is tests/test_gpu_device_eval's: extra target words, names outside the vocabulary, empty
names, names with commas and non-ASCII names, a filtered line; plus a token only one example uses, whose row is NaN."""
import logging
import os
import pickle

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

B = 7                       # TEST_BATCH_SIZE of these models
NAN_TOKEN = "nan|token"


@pytest.fixture(scope="module")
def trained(tmp_path_factory):
    """(prefix, save, the test file's lines): the device-eval toy dataset with one example that alone uses NAN_TOKEN."""
    from tests.test_gpu_device_eval import _dataset, _train
    tmp = tmp_path_factory.mktemp("corpus")
    with pytest.MonkeyPatch.context() as mp:
        mp.chdir(tmp)
        mp.delenv("WORLD_SIZE", raising=False)
        mp.delenv("C2V_DEVICE_EVAL", raising=False)
        prefix = _dataset(tmp)
        with open(prefix + ".dict.c2v", "rb") as f:
            dicts = [pickle.load(f) for _ in range(4)]
        dicts[0][NAN_TOKEN] = 1
        with open(prefix + ".dict.c2v", "wb") as f:
            for d in dicts:
                pickle.dump(d, f)
        lines = open(prefix + ".test.c2v", "rb").read().splitlines()
        ctx = lines[0].split(b" ")
        ctx[1] = b"%s,%s" % (NAN_TOKEN.encode(), ctx[1].split(b",", 1)[1])
        lines.insert(10, b" ".join(ctx))
        with open(prefix + ".test.c2v", "wb") as f:
            f.write(b"\n".join(lines) + b"\n")
        save = _train(prefix, tmp, epochs=3)
    return prefix, save, lines


def _model(monkeypatch, tmp_path, trained, math=None):
    """The trained model loaded with C2V_DEVICE_EVAL=1 (the routes are switched on the same object), NAN_TOKEN's row NaN."""
    from code2vec_b200.b200_model import Code2VecModel
    from tests.test_gpu_model import _config
    prefix, save, _ = trained
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    monkeypatch.setenv("C2V_DEVICE_EVAL", "1")
    if math:
        monkeypatch.setenv("C2V_MATH", math)
    else:
        monkeypatch.delenv("C2V_MATH", raising=False)
    m = Code2VecModel(_config(prefix, tmp_path, MODEL_LOAD_PATH=save, TEST_BATCH_SIZE=B))
    m.engine.params["tok"][m.vocabs.token_vocab.word_to_index[NAN_TOKEN]] = float("nan")
    return m


class _Log(logging.Handler):
    def __init__(self):
        super().__init__()
        self.lines = []

    def emit(self, record):
        self.lines.append(record.getMessage())


def _run(m, route: str, path: str, topn: int):
    """Both commands and both API calls on one route: (file bytes, API results, log lines) per command."""
    from code2vec_b200.__main__ import write_name_scores, write_nearest
    m._device_eval = route == "device"
    log = _Log()
    logger = m.config.get_logger()
    logger.addHandler(log)
    try:
        out = {}
        for cmd, write, suffix, api in (
                ("scores", lambda: write_name_scores(m, path), ".name_scores", lambda: m.score_names(path)),
                ("nearest", lambda: write_nearest(m, path, topn), ".nearest", lambda: m.nearest_code_vectors(path, topn))):
            if os.path.exists(path + suffix):
                os.remove(path + suffix)
            log.lines = []
            assert write() == path + suffix
            lines = [l for l in log.lines if not l.startswith("b200 backend")]
            out[cmd] = (open(path + suffix, "rb").read(), api(), lines)
        return out
    finally:
        logger.removeHandler(log)
        m._device_eval = True


def _assert_equal_arrays(a, b):
    assert len(a) == len(b)
    assert a[0] == b[0]                                   # names
    for x, y in zip(a[1:], b[1:]):
        assert x.dtype == y.dtype and x.shape == y.shape
        assert np.array_equal(x, y, equal_nan=x.dtype.kind == "f")


def _check_routes(m, path, topn):
    host = _run(m, "host", path, topn)
    dev = _run(m, "device", path, topn)
    for cmd in ("scores", "nearest"):
        assert dev[cmd][0] == host[cmd][0], "%s file differs" % cmd
        _assert_equal_arrays(dev[cmd][1], host[cmd][1])
        assert dev[cmd][2] == host[cmd][2], "%s log lines differ" % cmd
    assert m._dev_corpus_reader is not None              # the device route read the corpus
    return host


def _corpus(tmp_path, lines, n, name):
    path = str(tmp_path / name)
    with open(path, "wb") as f:
        f.write(b"".join(l + b"\n" for l in lines[:n]))
    return path


@pytest.mark.parametrize("math", [None, "fp32"])
def test_routes_equal_on_every_corpus_size(tmp_path, monkeypatch, trained, math):
    from tests.test_gpu_device_reader import _small_chunks
    _, _, lines = trained
    kept = [l for l in lines if l.strip() and not l.startswith(b"dropped ")]
    m = _model(monkeypatch, tmp_path, trained, math)
    try:
        for n, topn in ((0, 10), (1, 10), (B - 1, 10), (B, 63), (B + 1, 3)):
            _check_routes(m, _corpus(tmp_path, kept, n, "c%d.c2v" % n), topn)
        full = str(tmp_path / "full.c2v")
        with open(full, "wb") as f:
            f.write(b"\n".join(lines) + b"\n")
        host = _check_routes(m, full, 10)
        text = host["scores"][0].decode("utf-8")
        assert "\tnan\t" in text and "ü" in text and "a,b\t" in text and "<OOV>\t-\t-\t" in text
        assert host["nearest"][0].count(b"\n") == len(host["scores"][1][0]) > 3 * B
        _small_chunks(monkeypatch, 600)                  # batches cross reader chunks
        _check_routes(m, full, 63)
        m.close_session()
        assert m._dev_corpus_reader is None and m._device_vocabs is None
    finally:
        m.close_session()


def test_clones_and_a_dominant_logit(tmp_path, monkeypatch, trained):
    """Identical examples are each other's nearest at similarity 1; a target table scaled until one logit dominates makes
    the top-1 log-probability -log 1 = -0.0, printed -0.000000."""
    _, _, lines = trained
    kept = [l for l in lines if l.strip() and not l.startswith(b"dropped ")]
    m = _model(monkeypatch, tmp_path, trained)
    try:
        path = _corpus(tmp_path, kept[:5] + kept[:5] + kept[20:24], 14, "clones.c2v")
        host = _check_routes(m, path, 5)
        _names, _vec, idx, val = host["nearest"][1]
        assert idx[0, 0] == 5 and idx[5, 0] == 0 and abs(float(val[0, 0]) - 1.0) < 1e-5
        m.engine.params["tgt"].mul_(1e4)
        host = _check_routes(m, path, 5)
        assert b"\t-0.000000\n" in host["scores"][0]
    finally:
        m.close_session()


def test_rejected_corpus_raises_the_host_exception_and_leaves_no_file(tmp_path, monkeypatch, trained):
    from code2vec_b200.__main__ import write_name_scores, write_nearest
    _, _, lines = trained
    good = [l for l in lines if l.strip() and not l.startswith(b"dropped ")]
    malformed = good[:12] + [good[12] + b" extra"] + good[13:]
    invalid_utf8 = good[:9] + [b"na\xc3me\xed\xa0\x80" + good[9][good[9].index(b" "):]] + good[10:]
    m = _model(monkeypatch, tmp_path, trained)
    try:
        for bad, exc in ((malformed, ValueError), (invalid_utf8, UnicodeDecodeError)):
            path = _corpus(tmp_path, bad, len(bad), "bad.c2v")
            for write, suffix in ((lambda: write_name_scores(m, path), ".name_scores"),
                                  (lambda: write_nearest(m, path, 10), ".nearest")):
                msgs = []
                for route in ("host", "device"):
                    m._device_eval = route == "device"
                    with pytest.raises(exc) as e:
                        write()
                    msgs.append(str(e.value))
                    assert not os.path.exists(path + suffix)
                    assert not [f for f in os.listdir(tmp_path) if f.endswith(".tmp")]
                assert msgs[0] == msgs[1]
            m._device_eval = True
        assert m._dev_corpus_reader is None              # a failed pass drops its reader
        path = _corpus(tmp_path, good, len(good), "good.c2v")
        msgs = []
        for route in ("host", "device"):                 # --topn keeps its bound
            m._device_eval = route == "device"
            with pytest.raises(ValueError) as e:
                write_nearest(m, path, 64)
            msgs.append(str(e.value))
            assert not os.path.exists(path + ".nearest")
        assert msgs[0] == msgs[1]
        m._device_eval = True
        _check_routes(m, _corpus(tmp_path, good, len(good), "good.c2v"), 10)
    finally:
        m.close_session()


def test_command_line(tmp_path, monkeypatch):
    """python -m code2vec_b200 --load M --score_names F --nearest F writes the same files with C2V_DEVICE_EVAL=0 and 1, on a
    model the command line trained (its default dims)."""
    import tests.test_gpu_model as G
    from code2vec_b200.__main__ import main
    monkeypatch.setattr(G, "C", 200)                 # the default MAX_CONTEXTS
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    monkeypatch.delenv("C2V_MATH", raising=False)
    monkeypatch.delenv("C2V_DEVICE_EVAL", raising=False)
    prefix, test_lines = G._make_dataset(tmp_path)
    save = str(tmp_path / "m" / "saved")
    assert main(["--data", prefix, "--save", save, "--framework", "b200"]) == 0
    path = prefix + ".test.c2v"
    with open(path, "a", encoding="utf-8") as f:      # names outside the vocabulary, one with a comma, one not ASCII
        for i, name in enumerate(["no|such|name", "a,b", "n\u00e4me", ""]):
            f.write("%s %s\n" % (name, test_lines[i].split(" ", 1)[1]))
    out = {}
    for flag in ("0", "1"):
        monkeypatch.setenv("C2V_DEVICE_EVAL", flag)
        assert main(["--load", save, "--score_names", path, "--nearest", path, "--topn", "4", "--framework", "b200"]) == 0
        out[flag] = (open(path + ".name_scores", "rb").read(), open(path + ".nearest", "rb").read())
    assert out["0"] == out["1"]
    assert out["1"][0].count(b"\n") == len(test_lines) + 4
