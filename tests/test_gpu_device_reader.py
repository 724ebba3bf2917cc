"""The device reader (code2vec_b200/device_reader.py, csrc/reader.cu) against the host reader it replaces: the same batches,
compared on their bit patterns, for the same config and shuffle seed; the same ValueErrors for malformed files; each
rank's slice of every batch; and Code2VecModel.train() with C2V_DEVICE_READER=1 saving the checkpoint the host path saves."""
import os
import pickle

import numpy as np
import pytest

from code2vec_b200 import vocabularies as V
from code2vec_b200.config import Config
from code2vec_b200.path_context_reader import EstimatorAction, PathContextReader, _Chunk
from tests.test_reader_native import _random_lines

pytestmark = pytest.mark.gpu

NAMES = ("path_source_token_indices", "path_indices", "path_target_token_indices", "context_valid_mask", "target_index")


class _Former:
    def to_model_input_form(self, t):
        return t

    def from_model_input_form(self, row):
        return row


def _write(tmp_path, text: bytes, C, batch, epochs=1, shuffle=8, separate=False, n_tok=36, n_path=25, n_tgt=12):
    rng = np.random.default_rng(0)
    prefix = str(tmp_path / "ds")
    tok = {"t%d" % i: int(rng.integers(1, 50)) for i in range(n_tok)}
    tok.update({"ü" * 3: 5, "x" * 301: 4, "名前": 3, "": 2})
    pth = {str(100 + i): int(rng.integers(1, 50)) for i in range(n_path)}
    tgt = {"name|%d" % i: int(rng.integers(1, 50)) for i in range(n_tgt)}
    with open(prefix + ".dict.c2v", "wb") as f:
        for d in (tok, pth, tgt):
            pickle.dump(d, f)
        pickle.dump(1000, f)
    with open(prefix + ".train.c2v", "wb") as f:
        f.write(text)
    cfg = Config(set_defaults=True)
    cfg.VERBOSE_MODE = 0
    cfg.TRAIN_DATA_PATH_PREFIX = prefix
    cfg.MAX_CONTEXTS = C
    cfg.TRAIN_BATCH_SIZE = batch
    cfg.NUM_TRAIN_EPOCHS = epochs
    cfg.SHUFFLE_BUFFER_SIZE = shuffle
    cfg.SEPARATE_OOV_AND_PAD = separate
    cfg.READER_NUM_PARALLEL_BATCHES = 3
    cfg.MAX_TOKEN_VOCAB_SIZE, cfg.MAX_PATH_VOCAB_SIZE, cfg.MAX_TARGET_VOCAB_SIZE = 10 ** 7, 10 ** 7, 10 ** 7
    return cfg, V.Code2VecVocabs(cfg)


def _small_chunks(monkeypatch, size):
    """Both readers read the file in chunks of at most `size` bytes of complete lines (a longer line is a chunk of its
    own, as the chunker's retry makes it)."""
    orig = PathContextReader._native_chunks

    def chunks(self):
        for ch in orig(self):
            data = bytes(ch.buf[:ch.n])
            start = 0
            while start < len(data):
                end = data.rfind(b"\n", start, start + size)
                if end < 0:
                    end = data.find(b"\n", start + size)
                end = len(data) if end < 0 else end + 1
                yield _Chunk(data[start:end], end - start)
                start = end
    monkeypatch.setattr(PathContextReader, "_native_chunks", chunks)


def _host_batches(cfg, vs, seed):
    r = PathContextReader(vs, cfg, _Former(), EstimatorAction.Train, use_native=True, shuffle_seed=seed)
    return [tuple(np.array(getattr(b, n)) for n in NAMES) for b in r.get_dataset()]


def _device_batches(cfg, vs, seed, world=1, rank=0):
    import torch
    from code2vec_b200.device_reader import DeviceBatchReader
    r = PathContextReader(vs, cfg, _Former(), EstimatorAction.Train, shuffle_seed=seed)
    dr = DeviceBatchReader(r, torch.device("cuda", 0), world=world, rank=rank)
    out = []
    try:
        for b in dr:
            b.wait()
            out.append((b.rows, b.lo, b.hi, tuple(t.cpu().numpy() for t in b.tensors)))
            b.release()
    finally:
        dr.close()
    return out


def _bits(a):
    return a.view(np.int32) if a.dtype == np.float32 else a


def _assert_same(host, dev, world=1, rank=0):
    assert len(host) == len(dev) > 0
    for k, (h, (rows, lo, hi, d)) in enumerate(zip(host, dev)):
        assert rows == len(h[4]), k
        b = rows // world
        assert (lo, hi) == ((rank * b, (rank + 1) * b) if world > 1 else (0, rows)), k
        for name, x, y in zip(NAMES, h, d):
            assert x.dtype == y.dtype and np.array_equal(_bits(x[lo:hi]), _bits(y)), (k, name)


def _text(lines, crlf=False, blanks=False, last_newline=True):
    out = []
    for i, l in enumerate(lines):
        out.append(l + ("\r\n" if crlf and i % 2 else "\n"))
        if blanks and i % 5 == 1:
            out.append("\n" if i % 2 else "\n\n")          # ("\r\n" alone is a record: a line with one field)
    s = "".join(out)
    if not last_newline:
        s = s.rstrip("\n")
    return s.encode("utf-8")


def _odd_lines(C):
    """Lines with every field shape the parse rules name: empty targets and contexts, 1-, 2- and 3-part contexts, empty
    parts, multi-byte and 301-byte words, OOV words, rows dropped for an OOV target or for having no valid context."""
    pad = [""] * C
    return [" ".join((["name|1", "t1", "t2,101", "t3,102,t4", ",,", "t5,,t6", "üüü,100,名前", "x" * 301 + ",103,x" * 1] + pad)[:C + 1]),
            " ".join(([""] + ["t1,100,t2"] + pad)[:C + 1]),                  # empty target: OOV, dropped
            " ".join((["name|2"] + pad)[:C + 1]),                            # no context: dropped
            " ".join((["unknown", "t1,100,t2"] + pad)[:C + 1]),              # OOV target: dropped
            " ".join((["name|3", "zz,999,yy"] + pad)[:C + 1]),               # OOV words only: kept (OOV != PAD)
            " ".join((["name,|4", "a,b"] + pad)[:C + 1])]                    # a comma inside the target


@pytest.mark.parametrize("C", [13, 200])
@pytest.mark.parametrize("case", ["plain", "small_chunks", "epochs3_big_shuffle", "separate", "crlf_blank_no_eol"])
def test_batches_equal_the_host_reader(tmp_path, monkeypatch, C, case):
    n = 300 if C == 13 else 60
    lines = _random_lines(n, C, seed=C) + _odd_lines(C) * 3
    np.random.default_rng(1).shuffle(lines)
    kw = dict(C=C, batch=17)
    text = _text(lines)
    if case == "small_chunks":
        _small_chunks(monkeypatch, 700)                         # many chunks, and lines longer than a chunk (C = 200)
    if case == "epochs3_big_shuffle":
        kw.update(epochs=3, shuffle=10 ** 6)                    # the pool holds the whole file: every batch is a drain
    if case == "separate":
        kw.update(separate=True)
    if case == "crlf_blank_no_eol":
        text = _text(lines, crlf=True, blanks=True, last_newline=False)
        _small_chunks(monkeypatch, 2000)
    cfg, vs = _write(tmp_path, text, **kw)
    host = _host_batches(cfg, vs, seed=3)
    assert len(host[-1][4]) < 17 or case == "epochs3_big_shuffle"        # a short last batch
    _assert_same(host, _device_batches(cfg, vs, seed=3))


@pytest.mark.parametrize("world", [2, 4, 8])
def test_each_rank_gets_its_slice(tmp_path, monkeypatch, world):
    C = 13
    lines = _random_lines(250, C, seed=9) + _odd_lines(C)
    _small_chunks(monkeypatch, 1500)
    cfg, vs = _write(tmp_path, _text(lines), C=C, batch=32, shuffle=40)
    host = _host_batches(cfg, vs, seed=5)
    for rank in range(world):
        _assert_same(host, _device_batches(cfg, vs, seed=5, world=world, rank=rank), world=world, rank=rank)


def test_java14m_sized_vocabularies(tmp_path):
    """A 1024-line batch against vocabularies of 1.3 M / 911 K / 261 K words (the tables the host probes)."""
    C, n_lines = 200, 2300
    rng = np.random.default_rng(0)
    n_tok, n_path, n_tgt = 1_300_000, 911_000, 261_000
    lines = []
    for _ in range(n_lines):
        k = int(rng.integers(60, C + 1))
        s = rng.integers(0, n_tok + 1000, size=(k, 2))
        p = rng.integers(0, n_path + 1000, size=k)
        lines.append(" ".join(["name|%d" % int(rng.integers(0, n_tgt + 100))] +
                              ["t%d,%d,t%d" % (a, 100 + b, c) for (a, c), b in zip(s, p)] + [""] * (C - k)))
    cfg, vs = _write(tmp_path, _text(lines), C=C, batch=1024, shuffle=500, n_tok=n_tok, n_path=n_path, n_tgt=n_tgt)
    host = _host_batches(cfg, vs, seed=11)
    assert len(host[0][4]) == 1024
    _assert_same(host, _device_batches(cfg, vs, seed=11))


@pytest.mark.parametrize("bad", ["fields", "parts", "parts_and_fields", "short_lines", "after_blanks", "last_no_eol"])
def test_malformed_lines_raise_the_host_error(tmp_path, bad):
    C = 6
    good = _random_lines(40, C, seed=2)
    lines = list(good)
    if bad == "fields":
        lines[17] = " ".join(lines[17].split(" ")[:-1])
        lines[30] = lines[30] + " "
    elif bad == "parts":
        lines[21] = " ".join(["name|1", "a,b,c,d"] + [""] * (C - 1))
    elif bad == "parts_and_fields":
        lines[9] = " ".join(["name|1", "a,b,c,d"] + [""] * C)
    elif bad == "short_lines":
        lines = lines[:2] + ["x"] * 400
    elif bad == "after_blanks":
        lines[25] = lines[25] + " extra"
    text = _text(lines, blanks=bad == "after_blanks", last_newline=bad != "last_no_eol")
    if bad == "last_no_eol":
        text += b" " + b"t1,100,t2"                   # the unterminated last line gains a field
    cfg, vs = _write(tmp_path, text, C=C, batch=4)
    cfg.READER_NUM_PARALLEL_BATCHES = 1               # the host then reports the lowest malformed line, as the device does
    with pytest.raises(ValueError) as host:
        _host_batches(cfg, vs, seed=1)
    with pytest.raises(ValueError) as dev:
        _device_batches(cfg, vs, seed=1)
    assert str(dev.value) == str(host.value)


# ---- Code2VecModel.train() with C2V_DEVICE_READER=1 ------------------------------------------------------------------
@pytest.fixture
def _ten_target_rows(monkeypatch):
    """The toy dataset with a ninth method name, so that 4 ranks all hold target rows (as tests/test_gpu_multi_rank_model)."""
    import tests.test_gpu_model as toy
    monkeypatch.setattr(toy, "TARGETS", toy.TARGETS + ["make|copy"])


def _train_logged(monkeypatch, make_cfg, env, world):
    """The checkpoint bytes and the (batch, summed loss) of every progress line of train() on `world` ranks."""
    from code2vec_b200.b200_model import Code2VecModel
    logged = []
    orig = Code2VecModel._trace_training

    def trace(self, sum_loss, batch_num, t0):
        if self.rank == 0:
            logged.append((batch_num, sum_loss))
        return orig(self, sum_loss, batch_num, t0)
    env = dict({"C2V_DETERMINISTIC": "1", "C2V_SEED": "7"}, **env)
    with monkeypatch.context() as m:
        m.setattr(Code2VecModel, "_trace_training", trace)
        if world == 1:
            for k, v in env.items():
                m.setenv(k, v)
            cfg = make_cfg()
            model = Code2VecModel(cfg)
            try:
                model.train()
            finally:
                model.close_session()
        else:
            from tests.test_gpu_multi_rank_model import _models
            cfg = make_cfg()
            _models(m, world, make_cfg, lambda model, r: model.train(), env)
    with open(cfg.MODEL_SAVE_PATH + ".c2v_b200", "rb") as f:
        return f.read(), logged


@pytest.mark.parametrize("world,hint", [(1, "0"), (1, "1"), (2, "0"), (4, "0")])
def test_train_saves_the_host_paths_checkpoint(tmp_path, monkeypatch, _ten_target_rows, world, hint):
    from tests.test_gpu_model import _config, _make_dataset
    monkeypatch.chdir(tmp_path)
    prefix, _ = _make_dataset(tmp_path, n_train=101)
    out = {}
    for flag in ("0", "1"):
        save = str(tmp_path / ("reader" + flag) / "saved")
        make = lambda: _config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, MODEL_SAVE_PATH=save, NUM_TRAIN_EPOCHS=5,
                               NUM_BATCHES_TO_LOG_PROGRESS=3, SHUFFLE_BUFFER_SIZE=40, DROPOUT_KEEP_RATE=0.75)
        out[flag] = _train_logged(monkeypatch, make, {"C2V_DEVICE_READER": flag, "C2V_HINT_NEXT": hint}, world)
    (ckpt0, log0), (ckpt1, log1) = out["0"], out["1"]
    assert len(log0) >= 4 and log1 == log0
    assert ckpt1 == ckpt0
