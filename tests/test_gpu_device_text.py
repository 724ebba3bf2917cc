"""`.vectors` and word2vec files formatted on the GPU (C2V_DEVICE_TEXT=1: csrc/text.cu, text_export.py) against the host
writers they replace: the kernel on the value sets of tests/test_device_text_model against numpy, rows across warp
widths and chunk boundaries, a buffer too small for every row, and byte-identical files from evaluate() (host and
device routes, 1, 2 and 4 ranks) and save_word2vec_format (b200 and b200-keras), the java14m-sized target table too."""
import io

import numpy as np
import pytest

from tests.test_device_text_model import _bits, _neighbours

pytestmark = pytest.mark.gpu


def _host_lines(x, words=None) -> bytes:
    from code2vec_b200.common import common
    from code2vec_b200.model_base import Code2VecModelBase
    f = io.StringIO()
    if words is None:
        Code2VecModelBase._write_code_vectors(None, f, x)
    else:
        common.save_word2vec_file(f, words, x)
    return f.getvalue().encode("utf-8")


def _device_lines(x, chunk_bytes=None, words=None) -> bytes:
    import torch
    from code2vec_b200 import text_export as T
    f = io.BytesIO()
    t = torch.as_tensor(x).cuda() if not isinstance(x, torch.Tensor) else x
    if words is None:
        T.write_lines(f, t, chunk_bytes or T.CHUNK_BYTES)
        return f.getvalue()
    w = io.TextIOWrapper(f, encoding="utf-8", write_through=True)
    T.save_word2vec_file(w, words, t, chunk_bytes or T.CHUNK_BYTES)
    return f.getvalue()


def _edge_values():
    rng = np.random.default_rng(5)
    twos = np.ldexp(np.float32(1), np.arange(-149, 128)).astype(np.float32)
    tens = np.float32([10.0 ** k for k in range(-45, 39)])
    tens = tens[(tens != 0) & np.isfinite(tens)]
    nan = _bits([0x7FC00000, 0x7F800001, 0x7FFFFFFF, 0xFFC00000, 0xFFA5A5A5])
    special = np.float32([0.0, -0.0, np.inf, -np.inf])
    sub = _bits([1 << i for i in range(23)] + [0x007FFFFF])
    return np.concatenate([special, nan, _neighbours(twos), _neighbours(tens), _neighbours(sub),
                           _neighbours(np.float32([1e-4, 1e6]), k=8), _bits([0x00800000, 0x7F7FFFFF]),
                           _bits(rng.integers(0, 1 << 32, size=1 << 20, dtype=np.uint64))])


def test_kernel_equals_numpy_on_the_edge_values():
    x = _edge_values()
    D = 384
    x = np.concatenate([x, np.zeros((-x.size) % D, np.float32)]).reshape(-1, D)
    got = _device_lines(x).split(b"\n")[:-1]
    want = [" ".join(str(v) for v in row).encode() for row in x]
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert len(got) == len(want) and not bad, bad[:5]


@pytest.mark.parametrize("D", [1, 2, 31, 32, 33, 63, 64, 65, 96, 127, 384, 1000])
def test_rows_across_warp_widths_and_chunks(D):
    """Rows of every width around multiples of 32; a chunk of a few rows, so a pass takes many chunks and ends mid-row
    count; the same with a word prefix per row."""
    rng = np.random.default_rng(D)
    n = 203
    x = (rng.standard_normal((n, D)) * 10.0 ** rng.integers(-6, 8, size=(n, D))).astype(np.float32)
    x[rng.random((n, D)) < 0.01] = np.nan
    want = _host_lines(x)
    assert _device_lines(x) == want
    small = 7 * D * 16 + 5            # 7 rows' bound a chunk: 29 chunks, the last of 0 < rows < 7
    assert _device_lines(x, small) == want
    words = {i: ("w%d" % i) * (1 + i % 5) + ("ü" if i % 7 == 0 else "") for i in range(n)}
    assert _device_lines(x, small, words) == _host_lines(x, words)
    assert _device_lines(x, None, words) == _host_lines(x, words)


def test_strided_rows_and_a_buffer_too_small():
    """c2v_text_format_rows directly: rows of a strided view (ld > cols), and an output buffer that holds only some of
    the rows: those are written, the call reports them, and the next call writes the rest."""
    import torch
    from code2vec_b200 import engine as E
    lib = E.load_library()
    rng = np.random.default_rng(1)
    full = torch.as_tensor(rng.standard_normal((50, 80)).astype(np.float32)).cuda()
    x = full[:, 3:40]                                      # cols 37, ld 80
    rows, cols = x.shape
    want = _host_lines(x.cpu().numpy())
    stage = torch.empty(rows * cols * 16, dtype=torch.uint8, device="cuda")
    out = torch.empty(rows * cols * 16, dtype=torch.uint8, device="cuda")
    ends = torch.empty(rows + 1, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    text, r0 = b"", 0
    cap = len(want) // 3
    calls = 0
    while r0 < rows:
        rc = lib.c2v_text_format_rows(x[r0].data_ptr(), rows - r0, cols, x.stride(0), None, None, stage.data_ptr(),
                                      stage.numel(), out.data_ptr(), cap, ends[1:].data_ptr(), ends.data_ptr(), s)
        assert rc == 0
        done = int(ends[0])
        assert 0 < done < rows - r0 or r0 + done == rows
        n = int(ends[done])
        assert n <= cap and (r0 + done == rows or int(ends[done + 1]) > cap)
        text += bytes(out[:n].cpu().numpy())
        r0 += done
        calls += 1
    assert calls >= 3 and text == want
    # arguments it refuses
    assert lib.c2v_text_format_rows(x.data_ptr(), rows, cols, cols - 1, None, None, stage.data_ptr(), stage.numel(),
                                    out.data_ptr(), cap, ends[1:].data_ptr(), ends.data_ptr(), s) < 0
    assert lib.c2v_text_format_rows(x.data_ptr(), rows, cols, 80, None, None, stage.data_ptr(), 16, out.data_ptr(), cap,
                                    ends[1:].data_ptr(), ends.data_ptr(), s) < 0
    assert b"stage_bytes" in lib.c2v_last_error(None)


class _SampleSink(io.RawIOBase):
    """A binary file that keeps only the lines whose numbers are in `keep` (the text of the others is dropped)."""

    def __init__(self, keep):
        self.keep, self.lines, self.n, self.part = set(keep), {}, 0, b""

    def writable(self):
        return True

    def write(self, b):
        data = self.part + bytes(b)
        nl = np.flatnonzero(np.frombuffer(data, dtype=np.uint8) == 10)
        start = 0
        for p in nl:
            if self.n in self.keep:
                self.lines[self.n] = data[start:p + 1]
            self.n += 1
            start = int(p) + 1
        self.part = data[start:]
        return len(b)


def test_java14m_sized_target_table():
    """261,246 x 384 (1.1 GB of text, 17 chunks of 64 MB): a seeded sample of rows, the first and the last row."""
    import torch
    from code2vec_b200 import text_export as T
    from code2vec_b200.common import common
    n, D = 261246, 384
    g = torch.Generator(device="cuda")
    g.manual_seed(14)
    table = torch.empty((n, D), dtype=torch.float32, device="cuda").uniform_(-0.1, 0.1, generator=g)
    words = {i: "word%d" % i for i in range(n)}
    rows = sorted(set(np.random.default_rng(2).choice(n, 300, replace=False).tolist()) | {0, n - 1})
    sink = _SampleSink([0] + [r + 1 for r in rows])
    out = io.TextIOWrapper(io.BufferedWriter(sink), encoding="utf-8")
    writer = T.save_word2vec_file(out, words, table)
    assert sink.n == n + 1 and sink.part == b""
    assert writer.bytes_written > 8 * T.CHUNK_BYTES
    assert writer.peak_host_bytes <= 2 * T.CHUNK_BYTES + 64
    assert sink.lines[0] == b"%d %d\n" % (n, D)
    sample = table[torch.tensor(rows, device="cuda")].cpu().numpy()
    f = io.StringIO()
    common.save_word2vec_file(f, {j: words[r] for j, r in enumerate(rows)}, sample)
    want = f.getvalue().encode().split(b"\n")[1:-1]
    for j, r in enumerate(rows):
        assert sink.lines[r + 1] == want[j] + b"\n", r


# ---- the model ------------------------------------------------------------------------------------------------------------
@pytest.fixture
def _count_device_writes(monkeypatch):
    from code2vec_b200.text_export import DeviceTextWriter
    calls = []
    orig = DeviceTextWriter.write_rows

    def write_rows(self, x, prefixes=None):
        calls.append(tuple(x.shape))
        return orig(self, x, prefixes)
    monkeypatch.setattr(DeviceTextWriter, "write_rows", write_rows)
    return calls


@pytest.mark.parametrize("device_eval,batch", [("0", 32), ("1", 32), ("0", 7), ("1", 1024)])
def test_vectors_files_are_byte_identical(tmp_path, monkeypatch, _count_device_writes, device_eval, batch):
    from tests.test_gpu_device_eval import _dataset, _evaluate, _train
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    prefix = _dataset(tmp_path)
    save = _train(prefix, tmp_path)
    monkeypatch.setenv("C2V_DEVICE_TEXT", "0")
    host = _evaluate(monkeypatch, prefix, tmp_path, save, device_eval, TEST_BATCH_SIZE=batch)
    assert not _count_device_writes
    monkeypatch.setenv("C2V_DEVICE_TEXT", "1")
    dev = _evaluate(monkeypatch, prefix, tmp_path, save, device_eval, TEST_BATCH_SIZE=batch)
    assert _count_device_writes and sum(s[0] for s in _count_device_writes) == host[2].count(b"\n")
    assert dev[1] == host[1] and str(dev[0]) == str(host[0])
    assert dev[2] == host[2], ".vectors differs"
    assert host[2].count(b"\n") > 150


@pytest.mark.parametrize("framework", ["b200", "b200-keras"])
def test_word2vec_files_are_byte_identical(tmp_path, monkeypatch, _count_device_writes, framework):
    from code2vec_b200 import load_model_dynamically
    from code2vec_b200.common import common
    from code2vec_b200.vocabularies import VocabType
    from tests.test_gpu_model import _config, _make_dataset
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    prefix, _ = _make_dataset(tmp_path)
    monkeypatch.setenv("C2V_DETERMINISTIC", "1")           # both trainings end on the same tables
    monkeypatch.setenv("C2V_SEED", "7")
    files = {}
    for flag in ("0", "1"):
        monkeypatch.setenv("C2V_DEVICE_TEXT", flag)
        m = load_model_dynamically(_config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, DL_FRAMEWORK=framework,
                                           NUM_TRAIN_EPOCHS=2, SAVE_EVERY_EPOCHS=2))
        try:
            m.train()
            for vt in (VocabType.Token, VocabType.Target, VocabType.Path):
                path = str(tmp_path / ("%s.%s.w2v" % (flag, vt.name)))
                m.save_word2vec_format(path, vt)
                files[flag, vt] = open(path, "rb").read()
                f = io.StringIO()
                common.save_word2vec_file(f, m.vocabs.get(vt).index_to_word, m._get_vocab_embedding_as_np_array(vt))
                assert files[flag, vt] == f.getvalue().encode(), (flag, vt)
        finally:
            m.close_session()
    assert len(_count_device_writes) == 3
    for vt in (VocabType.Token, VocabType.Target, VocabType.Path):
        assert files["0", vt] == files["1", vt], vt


@pytest.fixture
def _ten_target_rows(monkeypatch):
    import tests.test_gpu_model as toy
    monkeypatch.setattr(toy, "TARGETS", toy.TARGETS + ["make|copy"])


@pytest.mark.parametrize("world", [2, 4])
def test_files_on_emulated_ranks_are_byte_identical(tmp_path, monkeypatch, _ten_target_rows, world):
    """evaluate() on the host and device routes and the three word2vec files on W emulated ranks, C2V_DEVICE_TEXT=1,
    against C2V_DEVICE_TEXT=0 on the same ranks and against one GPU."""
    from code2vec_b200.b200_model import Code2VecModel
    from code2vec_b200.vocabularies import VocabType
    from tests.test_gpu_model import _config, _make_dataset
    from tests.test_gpu_multi_rank_model import _models
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    monkeypatch.delenv("C2V_DEVICE_TEXT", raising=False)
    prefix, _ = _make_dataset(tmp_path, n_test=45)
    save = str(tmp_path / "model" / "saved")
    m = Code2VecModel(_config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, MODEL_SAVE_PATH=save, NUM_TRAIN_EPOCHS=10))
    try:
        m.train()
    finally:
        m.close_session()
    make = lambda: _config(prefix, tmp_path, MODEL_LOAD_PATH=save, TEST_DATA_PATH=prefix + ".test.c2v",
                           EXPORT_CODE_VECTORS=True, TEST_BATCH_SIZE=64)
    outputs = {}

    def run(model, r, tag):
        model.evaluate()
        if r == 0:
            outputs[tag] = dict(vectors=open(prefix + ".test.c2v.vectors", "rb").read())
        for vt in (VocabType.Token, VocabType.Target, VocabType.Path):
            model.save_word2vec_format(str(tmp_path / ("%s.%s.w2v" % (tag, vt.name))), vt)
        if r == 0:
            outputs[tag].update({vt: open(str(tmp_path / ("%s.%s.w2v" % (tag, vt.name))), "rb").read()
                                 for vt in (VocabType.Token, VocabType.Target, VocabType.Path)})

    one = Code2VecModel(make())
    try:
        run(one, 0, "one")
    finally:
        one.close_session()
    for device_eval in ("0", "1"):
        for text in ("0", "1"):
            tag = "w%s-e%s-t%s" % (world, device_eval, text)
            _models(monkeypatch, world, make, lambda model, r: run(model, r, tag),
                    env={"C2V_DEVICE_EVAL": device_eval, "C2V_DEVICE_TEXT": text})
            assert outputs[tag] == outputs["one"], tag
    assert outputs["one"]["vectors"].count(b"\n") == 45


def test_a_bad_switch_is_refused(tmp_path, monkeypatch):
    from code2vec_b200.b200_model import Code2VecModel
    from tests.test_gpu_model import _config, _make_dataset
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    prefix, _ = _make_dataset(tmp_path)
    monkeypatch.setenv("C2V_DEVICE_TEXT", "2")
    with pytest.raises(ValueError, match="C2V_DEVICE_TEXT must be 0 or 1"):
        Code2VecModel(_config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix))
