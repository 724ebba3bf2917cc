"""`--predict` on the GPU (C2V_DEVICE_PREDICT=1, DESIGN.md §6i) against the host route, byte for byte.

First the fact the route rests on: a row's prediction does not depend on the batch it is in.  Then the command line's
stdout with the flag at 0 and at 1, for both frameworks, with and without --export_code_vectors, in all three math
modes, on the golden extractor output, a seeded synthetic input of more than 20,000 methods, batch edges, empty input,
non-ASCII input, a numeric path the device cannot key, and "\\r" line ends through both sources."""
import io
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.predict_inputs import synthetic_lines

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MATHS = ["fp32", "tf32", "3xtf32"]


@pytest.fixture(scope="module")
def saved_model(tmp_path_factory):
    """A model trained from the command line with the reference's defaults (d = 128, 200 contexts, batches of 1024)."""
    import tests.test_gpu_model as toy
    from code2vec_b200.__main__ import main
    tmp = tmp_path_factory.mktemp("predict")
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(toy, "C", 200)
        mp.chdir(tmp)
        mp.delenv("WORLD_SIZE", raising=False)
        prefix, _ = toy._make_dataset(tmp)
        save = str(tmp / "model" / "saved")
        assert main(["--data", prefix, "--save", save, "--framework", "b200"]) == 0
    return save


@pytest.fixture(scope="module")
def golden_model(tmp_path_factory):
    """A model trained from the command line on the golden extractor output itself (its lines prepared as
    print_predictions prepares them, 64 copies), so its tokens, hashed paths and names are in the vocabularies."""
    import pickle
    from code2vec_b200.__main__ import main, prepare_extracted_lines
    tmp = tmp_path_factory.mktemp("golden")
    lines, _ = prepare_extracted_lines(_golden_input().decode("utf-8").splitlines(), 200)
    prefix = str(tmp / "golden")
    with open(prefix + ".train.c2v", "w") as f:
        f.write("\n".join(lines * 64) + "\n")
    tok, pth, tgt = {}, {}, {}
    for line in lines:
        parts = line.split(" ")
        tgt[parts[0]] = tgt.get(parts[0], 0) + 1
        for c in parts[1:]:
            if c:
                a, b, d = c.split(",")
                tok[a] = tok.get(a, 0) + 1
                tok[d] = tok.get(d, 0) + 1
                pth[b] = pth.get(b, 0) + 1
    with open(prefix + ".dict.c2v", "wb") as f:
        for d in (tok, pth, tgt):
            pickle.dump(d, f)
        pickle.dump(64 * len(lines), f)
    with pytest.MonkeyPatch.context() as mp:
        mp.chdir(tmp)
        mp.delenv("WORLD_SIZE", raising=False)
        save = str(tmp / "model" / "saved")
        assert main(["--data", prefix, "--save", save, "--framework", "b200"]) == 0
    return save


def _vocab_words():
    import tests.test_gpu_model as toy
    return toy.TOKENS, toy.TARGETS, toy.PATHS


# ---- batch invariance ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("math", MATHS)
def test_a_row_predicts_the_same_bits_alone_and_anywhere_in_a_full_batch(saved_model, monkeypatch, math):
    import torch
    from code2vec_b200.b200_model import Code2VecModel
    from code2vec_b200.config import Config
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    cfg = Config(set_defaults=True)
    cfg.MODEL_LOAD_PATH = saved_model
    cfg.DL_FRAMEWORK = "b200"
    cfg.VERBOSE_MODE = 0
    cfg.PREDICT = True
    m = Code2VecModel(cfg)
    try:
        e = m.engine
        e.set_option("math_mode", {"fp32": 0, "tf32": 1, "3xtf32": 2}[math])
        B, C = cfg.TEST_BATCH_SIZE, cfg.MAX_CONTEXTS
        rng = np.random.default_rng(3)
        dims = e.dims

        def rows(n):
            src = rng.integers(0, dims.token_vocab, size=(n, C), dtype=np.int32)
            pth = rng.integers(0, dims.path_vocab, size=(n, C), dtype=np.int32)
            tgt = rng.integers(0, dims.token_vocab, size=(n, C), dtype=np.int32)
            mask = (rng.random((n, C)) < 0.6).astype(np.float32)
            return src, pth, tgt, mask

        batch = rows(B)
        probe = rows(4)
        probe[3][3] = 0.0                                            # an all-masked row: NaN everywhere
        for normalize in (1, 2):
            for p in range(4):
                alone = e.predict_batch_host(*(a[p:p + 1] for a in probe), normalize=normalize)
                for pos in (0, 127, 128, B - 1):
                    full = [a.copy() for a in batch]
                    for a, b in zip(full, probe):
                        a[pos] = b[p]
                    got = e.predict_batch_host(*full, normalize=normalize)
                    for name, x, y in zip(("idx", "val", "code", "attn"), alone, got):
                        assert np.array_equal(x[0].view(np.uint32), y[pos].view(np.uint32)), (math, normalize, p, pos, name)
        torch.cuda.synchronize()
    finally:
        m.close_session()


# ---- the command line, byte for byte ------------------------------------------------------------------------------------
def _run(monkeypatch, save, data: bytes, flag: str, framework="b200", math=None, export=False, stdin=False, tmp=None,
         batch=None):
    """stdout bytes of `python -m code2vec_b200 --load save --predict ...` run in this process on `data`."""
    from code2vec_b200.__main__ import main
    monkeypatch.setenv("C2V_DEVICE_PREDICT", flag)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    if math:
        monkeypatch.setenv("C2V_MATH", math)
    else:
        monkeypatch.delenv("C2V_MATH", raising=False)
    out = io.BytesIO()
    wrapper = io.TextIOWrapper(out, encoding="utf-8", newline="\n", write_through=True)
    monkeypatch.setattr(sys, "stdout", wrapper)
    argv = ["--load", save, "--predict", "--framework", framework, "-v", "0"] + (["--export_code_vectors"] if export else [])
    if batch:
        from code2vec_b200 import config as cfgmod
        orig = cfgmod.Config.load_from_args

        def load_from_args(self, a):
            orig(self, a)
            self.TEST_BATCH_SIZE = batch
        monkeypatch.setattr(cfgmod.Config, "load_from_args", load_from_args)
    if stdin:
        monkeypatch.setattr(sys, "stdin", io.TextIOWrapper(io.BytesIO(data), encoding="utf-8", newline="\n"))
    else:
        path = tmp / "input.txt"
        path.write_bytes(data)
        argv += ["--predict_input", str(path)]
    try:
        assert main(argv) == 0
        wrapper.flush()
        return out.getvalue()
    finally:
        monkeypatch.setattr(sys, "stdout", sys.__stdout__)


def _both(monkeypatch, save, data, tmp, on_device=True, chunk_bytes=None, **kw):
    """(host route's stdout, device route's stdout); on_device: whether the device route must have taken the input
    itself (True) or handed it to the host route (False)."""
    from code2vec_b200 import device_predict as DP
    host = _run(monkeypatch, save, data, "0", tmp=tmp, **kw)
    ran = []
    orig = DP.DevicePredictor.run

    def run(self, *a, **k):
        if chunk_bytes is not None:
            k["chunk_bytes"] = chunk_bytes
        ok = orig(self, *a, **k)
        ran.append(ok)
        return ok
    monkeypatch.setattr(DP.DevicePredictor, "run", run)
    dev = _run(monkeypatch, save, data, "1", tmp=tmp, **kw)
    monkeypatch.setattr(DP.DevicePredictor, "run", orig)
    assert ran == [on_device]
    return host, dev


def _golden_input() -> bytes:
    g = json.load(open(os.path.join(ROOT, "tests", "golden", "host_golden2.json")))
    return g["extractor"]["jar_output"].encode("utf-8")


def _synthetic(n, seed=11, **kw) -> bytes:
    tokens, targets, paths = _vocab_words()
    return ("\n".join(synthetic_lines(n, seed, tokens, targets, numeric_paths=paths, **kw)) + "\n").encode("ascii")


@pytest.mark.parametrize("framework", ["b200", "b200-keras"])
@pytest.mark.parametrize("export", [False, True])
@pytest.mark.parametrize("math", MATHS)
def test_golden_and_small_inputs_are_byte_identical(saved_model, golden_model, monkeypatch, tmp_path, framework, export,
                                                    math):
    for model, data in ((golden_model, _golden_input()), (saved_model, _golden_input()), (saved_model, _synthetic(300, seed=5))):
        host, dev = _both(monkeypatch, model, data, tmp_path, framework=framework, export=export, math=math)
        assert host.count(b"Original name:\t") > 0
        assert dev == host
    # the golden model knows the golden words: its predictions name them and its attention lines print paths
    host, _ = _both(monkeypatch, golden_model, _golden_input(), tmp_path, framework=framework, export=export, math=math)
    assert b"predicted: ['get', 'name']" in host and b"context: a,(A)^(B),b" in host


@pytest.mark.parametrize("chunk_bytes", [1, 97, 1000, 4096])
def test_small_chunks_are_byte_identical(saved_model, monkeypatch, tmp_path, chunk_bytes):
    """Chunks far smaller than the input: methods, "\r\n" line ends and colliding keys ("Aa" / "BB" / "2112" early and
    late) fall on every side of chunk edges, and a method prints the path of a context in another chunk."""
    body = _synthetic(400, seed=13).split(b"\n")
    data = b"early x,Aa,y\r\n" + b"".join(line + (b"\r\n" if i % 2 else b"\n") for i, line in enumerate(body))
    data += b"late p,BB,q r,2112,s\r\n" + b"m1 u,Aa,v\n" * 3
    for stdin in (False, True):
        host, dev = _both(monkeypatch, saved_model, data, tmp_path, export=True, stdin=stdin, chunk_bytes=chunk_bytes)
        assert host.count(b"Original name:\t") > 400
        assert dev == host


@pytest.mark.parametrize("framework,math,export", [("b200", "fp32", True), ("b200", "tf32", False),
                                                   ("b200", None, True), ("b200-keras", None, False)])
def test_twenty_thousand_methods_are_byte_identical(saved_model, monkeypatch, tmp_path, framework, math, export):
    data = _synthetic(20500, seed=7)
    host, dev = _both(monkeypatch, saved_model, data, tmp_path, framework=framework, export=export, math=math)
    assert host.count(b"Original name:\t") >= 20000
    assert dev == host


@pytest.mark.parametrize("n", [1, 63, 64, 65, 200])
def test_batch_edges_are_byte_identical(saved_model, monkeypatch, tmp_path, n):
    data = _synthetic(n, seed=n, specials=False)
    host, dev = _both(monkeypatch, saved_model, data, tmp_path, export=True, batch=64)
    assert host.count(b"Original name:\t") == n
    assert dev == host


def test_empty_non_ascii_and_unkeyable_inputs(saved_model, monkeypatch, tmp_path):
    for data, on_device in ((b"", True), (b"\n\n  \n", True),
                            ("café a,b,c x,Aa,y\n".encode("utf-8") + _synthetic(20, seed=2), False),
                            (_synthetic(20, seed=3) + b"m a,007,b c,Aa,d\n", False)):
        host, dev = _both(monkeypatch, saved_model, data, tmp_path, on_device=on_device, export=True)
        assert dev == host
    assert _both(monkeypatch, saved_model, b"", tmp_path)[1] == b""


def test_a_malformed_context_raises_before_any_output(saved_model, monkeypatch, tmp_path):
    data = _synthetic(50, seed=4) + b"bad a,b c,d,e\n" + _synthetic(5, seed=6)
    for flag in ("0", "1"):
        with pytest.raises(ValueError):
            _run(monkeypatch, saved_model, data, flag, tmp=tmp_path)


def test_carriage_returns_follow_each_source(saved_model, monkeypatch, tmp_path):
    body = _synthetic(40, seed=9, specials=False).split(b"\n")
    data = b"".join(line + (b"\r\n" if i % 3 == 0 else b"\r" if i % 3 == 1 else b"\n") for i, line in enumerate(body))
    data += b"tail a,x,b\rc d,BB,e\r\n"         # two methods in a file, one (with "b\rc" a token) on standard input
    f_host, f_dev = _both(monkeypatch, saved_model, data, tmp_path, export=True)
    s_host, s_dev = _both(monkeypatch, saved_model, data, tmp_path, export=True, stdin=True)
    assert f_dev == f_host
    assert s_dev == s_host
    assert f_host != s_host


def test_standard_input_of_a_real_process(saved_model, tmp_path):
    """sys.stdin as Python sets it up for a pipe, not a stand-in: '\\r' stays in the line."""
    data = b"a\rb x,Aa,y\r\nc p,BB,q\rr s,2112,t\n"
    outs = []
    for flag in ("0", "1"):
        env = dict(os.environ, C2V_DEVICE_PREDICT=flag, PYTHONPATH=ROOT)
        env.pop("WORLD_SIZE", None)
        r = subprocess.run([sys.executable, "-m", "code2vec_b200", "--load", saved_model, "--predict", "-v", "0"],
                           input=data,
                           capture_output=True, cwd=str(tmp_path), env=env, timeout=600)
        assert r.returncode == 0, r.stderr.decode()[-2000:]
        outs.append(r.stdout)
    assert outs[0].count(b"Original name:\t") == 2
    assert outs[1] == outs[0]
