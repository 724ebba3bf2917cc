"""C2V_DEVICE_PREPROCESS=1 (code2vec_b200/device_preprocess.py) against the host route: the golden fixture made by the
reference preprocess.py, edge files, and a corpus large enough that the histogram table rehashes.  Every output file is
compared byte for byte and the rng must end in the host route's state."""
import os
import random
import shutil

import pytest

from code2vec_b200 import device_preprocess as D
from code2vec_b200 import preprocess as P

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "preprocess")
ARGS = ["--train_data", "raw.train.txt", "--test_data", "raw.test.txt", "--val_data", "raw.val.txt", "--max_contexts", "8",
        "--word_vocab_size", "40", "--path_vocab_size", "25", "--target_vocab_size", "12"]
HISTOS = ["--word_histogram", "histo.ori.c2v", "--path_histogram", "histo.path.c2v", "--target_histogram", "histo.tgt.c2v"]
OUTPUTS = ["test.c2v", "val.c2v", "train.c2v", "dict.c2v"]
COUNTED = ["histo.ori.c2v", "histo.path.c2v", "histo.tgt.c2v"]


def read(path):
    with open(path, "rb") as f:
        return f.read()


def run_both(argv, window=D.WINDOW_BYTES, seed=20240921):
    """(host logs, device logs, host rng, device rng) of both routes on argv, outputs `host.*` and `dev.*`."""
    host_rng, dev_rng = random.Random(seed), random.Random(seed)
    host_log, dev_log = [], []
    P.main(argv + ["--output_name", "host"], rng=host_rng, log=host_log.append)
    D.main(argv + ["--output_name", "dev"], rng=dev_rng, log=dev_log.append, window=window)
    return host_log, dev_log, host_rng, dev_rng


def assert_same(host_log, dev_log, host_rng, dev_rng, counted):
    for name in OUTPUTS + (COUNTED if counted else []):
        assert read("dev." + name) == read("host." + name), name
    assert dev_rng.getstate() == host_rng.getstate()
    assert [s for s in dev_log if not s.startswith(("Dictionaries saved", "Preprocessing on", "Device preprocessing"))] == \
        [s for s in host_log if not s.startswith("Dictionaries saved")]


@pytest.fixture()
def golddir(tmp_path, monkeypatch):
    for name in os.listdir(GOLD):
        if not name.startswith("expected."):
            shutil.copy(os.path.join(GOLD, name), tmp_path / name)
    monkeypatch.chdir(tmp_path)
    return tmp_path


@pytest.mark.parametrize("histos", [True, False], ids=["histogram_files", "counted"])
@pytest.mark.parametrize("window", [D.WINDOW_BYTES, 97], ids=["one_chunk", "small_window"])
def test_golden_fixture(golddir, histos, window):
    argv = ARGS + (HISTOS if histos else [])
    host_log, dev_log, host_rng, dev_rng = run_both(argv, window)
    for role in ("train", "val", "test", "dict"):
        assert read("dev.%s.c2v" % role) == read(os.path.join(GOLD, "expected.%s.c2v" % role)), role
    assert_same(host_log, dev_log, host_rng, dev_rng, not histos)
    if not histos:                                  # the counted histograms are the files count_histograms makes
        for counter, name in zip(P.count_histograms("raw.train.txt"), COUNTED):
            P.write_histogram(counter, "want." + name)
            assert read("dev." + name) == read("want." + name), name


def test_switch_routes_main(golddir, monkeypatch):
    monkeypatch.setenv("C2V_DEVICE_PREPROCESS", "1")
    logged = []
    n = P.main(ARGS + HISTOS + ["--output_name", "out"], rng=random.Random(20240921), log=logged.append)
    assert n == 61 and any(s.startswith("Preprocessing on the GPU") for s in logged)
    assert read("out.train.c2v") == read(os.path.join(GOLD, "expected.train.c2v"))


def _edge_corpus(rng, eol=b"\n", n_lines=300, C=6):
    toks = ["a", "b", "c", "d", "é", "名前", "x,y", ""]
    paths = ["1", "2", "3", "(λ)", ""]
    lines = []
    for i in range(n_lines):
        kind = i % 9
        tgt = rng.choice(["f", "g|h", "get", "ünï", "", "t,u"])
        if kind == 0:
            lines.append(b"")                                   # blank line
            continue
        if kind == 1:
            lines.append(tgt.encode())                          # a name with no context
            continue
        n = rng.choice([0, 1, C - 1, C, C, C + 1, C + 1, 2 * C, 5 * C, 40])
        ctxs = ["%s,%s,%s" % (rng.choice(toks), rng.choice(paths), rng.choice(toks)) for _ in range(n)]
        if kind == 2 and n:
            ctxs[0] = "z%d,q%d,z%d" % (i, i, i)                  # all-unknown parts
        if kind == 3 and n <= C:
            ctxs += ["a", "a,1", "", "a,1,b,c,d"][:max(0, C - n)]   # 1, 2, 0 and 5 parts in a short line
        if kind == 4 and n <= C:
            ctxs += ["a,1,b,extra"]
        line = tgt + " " + " ".join(ctxs)
        if kind == 5 and n < C:
            line = line.replace(" ", "  ", 1)                   # a double space: an empty context
        if kind == 6 and n < C:
            line += " "                                         # a trailing space: an empty context
        lines.append(line.encode())
    return eol.join(lines)


def _rate_tool():
    import importlib.util
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "preprocess_rate.py")
    spec = importlib.util.spec_from_file_location("preprocess_rate", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _write(path, data):
    with open(path, "wb") as f:
        f.write(data)


@pytest.mark.parametrize("eol,final", [(b"\n", True), (b"\r\n", True), (b"\r", True), (b"\n", False), (b"\r\n", False),
                                       (b"\r", False)], ids=["lf", "crlf", "cr", "lf_unterminated", "crlf_unterminated",
                                                             "cr_unterminated"])
@pytest.mark.parametrize("window", [D.WINDOW_BYTES, 64], ids=["one_chunk", "hundreds_of_chunks"])
def test_edge_files(tmp_path, monkeypatch, eol, final, window):
    monkeypatch.chdir(tmp_path)
    rng = random.Random(7)
    for role in ("train", "test", "val"):
        data = _edge_corpus(rng, eol)
        _write("raw.%s.txt" % role, data + (eol if final else b""))
    # the long lines of this corpus hold only contexts of 3+ parts: the 1- and 2-part ones are in short lines
    argv = ["--train_data", "raw.train.txt", "--test_data", "raw.test.txt", "--val_data", "raw.val.txt",
            "--max_contexts", "6", "--word_vocab_size", "5", "--path_vocab_size", "3", "--target_vocab_size", "4"]
    host_log, dev_log, host_rng, dev_rng = run_both(argv, window)
    assert_same(host_log, dev_log, host_rng, dev_rng, True)
    if window == 64:
        assert os.path.getsize("raw.train.txt") > 100 * 64


def test_mixed_line_ends_and_exact_limits(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    C = 4
    full = ["a,1,b"] * 3 + ["b,1,a", "a,2,a"]
    lines = [
        "m " + " ".join(full[:C]),                       # exactly max_contexts
        "m " + " ".join(full[:C + 1]),                   # max_contexts + 1, all full: sampled
        "n " + " ".join(["q,9,q"] * (C + 3)),            # all unknown: dropped, an empty example
        "p " + " ".join(["a,9,q", "q,1,q", "a,1,b"] * 2),    # full + sampled partial
        "r " + " ".join(["a,1,b", "q,9,q", "a,9,q"] * 2),    # full + all partial, no draw
    ]
    data = b"\r\n".join(l.encode() for l in lines[:2]) + b"\r" + b"\n".join(l.encode() for l in lines[2:]) + b"\r\n"
    for role in ("train", "test", "val"):
        _write("raw.%s.txt" % role, data)
    argv = ["--train_data", "raw.train.txt", "--test_data", "raw.test.txt", "--val_data", "raw.val.txt",
            "--max_contexts", str(C), "--word_vocab_size", "2", "--path_vocab_size", "1", "--target_vocab_size", "4"]
    for window in (D.WINDOW_BYTES, 8, 1):
        host_log, dev_log, host_rng, dev_rng = run_both(argv, window, seed=window)
        assert_same(host_log, dev_log, host_rng, dev_rng, True)


def test_invalid_utf8_raises_unicode_decode_error(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    good = b"f a,1,b c,2,d\n"
    for bad in (b"\xff", b"\xc0\xaf", b"\xed\xa0\x80", b"\xe2\x82", b"\xf4\x90\x80\x80", b"\x80"):
        _write("raw.train.txt", good * 3 + b"g a,1," + bad + b" x,1,y\n" + good)
        _write("raw.test.txt", good)
        _write("raw.val.txt", good)
        argv = ["--train_data", "raw.train.txt", "--test_data", "raw.test.txt", "--val_data", "raw.val.txt",
                "--max_contexts", "4"]
        with pytest.raises(UnicodeDecodeError):
            P.main(argv + ["--output_name", "host"], rng=random.Random(1), log=lambda s: None)
        with pytest.raises(UnicodeDecodeError) as e:
            D.main(argv + ["--output_name", "dev"], rng=random.Random(1), log=lambda s: None)
        assert "raw.train.txt" in str(e.value)
        # in a file that is only down-sampled: the test file, after the histograms were counted from the train file
        _write("raw.train.txt", good)
        _write("raw.test.txt", good + b"g a,1," + bad + b"\n")
        with pytest.raises(UnicodeDecodeError):
            P.main(argv + ["--output_name", "host"], rng=random.Random(1), log=lambda s: None)
        with pytest.raises(UnicodeDecodeError) as e:
            D.main(argv + ["--output_name", "dev"], rng=random.Random(1), log=lambda s: None)
        assert "raw.test.txt" in str(e.value)


def test_short_context_in_a_long_line_raises_index_error(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    ok = "f " + " ".join(["a,1,b"] * 6)
    bad = "g " + " ".join(["a,1,b"] * 5 + ["a,1"])
    _write("raw.train.txt", ("\n".join([ok] * 5 + [bad] + [ok] * 3) + "\n").encode())
    _write("raw.test.txt", (ok + "\n").encode())
    _write("raw.val.txt", (ok + "\n").encode())
    argv = ["--train_data", "raw.train.txt", "--test_data", "raw.test.txt", "--val_data", "raw.val.txt",
            "--max_contexts", "4"]
    host_rng, dev_rng = random.Random(3), random.Random(3)
    with pytest.raises(IndexError):
        P.main(argv + ["--output_name", "host"], rng=host_rng, log=lambda s: None)
    with pytest.raises(IndexError) as e:
        D.main(argv + ["--output_name", "dev"], rng=dev_rng, log=lambda s: None, window=40)
    assert "line 6 of raw.train.txt" in str(e.value)
    assert dev_rng.getstate() == host_rng.getstate()


def test_nothing_written_raises_zero_division(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    for role in ("train", "test", "val"):
        _write("raw.%s.txt" % role, b"name\n\n")
    argv = ["--train_data", "raw.train.txt", "--test_data", "raw.test.txt", "--val_data", "raw.val.txt"]
    with pytest.raises(ZeroDivisionError):
        P.main(argv + ["--output_name", "host"], rng=random.Random(1), log=lambda s: None)
    with pytest.raises(ZeroDivisionError):
        D.main(argv + ["--output_name", "dev"], rng=random.Random(1), log=lambda s: None)
    for name in COUNTED:
        assert read("dev." + name) == read("host." + name)


def test_large_corpus_rehashes_the_histogram_table(tmp_path, monkeypatch):
    R = _rate_tool()
    monkeypatch.chdir(tmp_path)
    stats = R.write_corpus(str(tmp_path), methods=30000, seed=11)
    assert stats["contexts"] >= 2_000_000
    argv = R.arguments(str(tmp_path))
    host_log, dev_log, host_rng, dev_rng = run_both(argv, window=4 << 20)
    assert_same(host_log, dev_log, host_rng, dev_rng, True)
    prep = D.DevicePreprocessor(0, 4 << 20)
    try:
        keys, slots, rehashes = prep.count_histograms(os.path.join(str(tmp_path), "raw.train.txt"))
    finally:
        prep.close()
    assert rehashes >= 1 and keys * 2 <= slots
