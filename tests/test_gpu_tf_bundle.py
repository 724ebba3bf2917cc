"""TensorFlow V2 checkpoints on the GPU: c2v_crc32c_rows / c2v_crc32c_combine against the plain CRC-32C model, and
Code2VecModel loading and saving bundles on one GPU and on 2, 4 and 8 emulated ranks (tests/emulated_ranks.py) against
the same weights in a .c2v_b200 checkpoint.  The toy dataset is tests/test_gpu_model's, with 16 target rows so that
each of 8 ranks holds some."""
import os
import shutil

import numpy as np
import pytest

from code2vec_b200 import tf_bundle as T
from tests import crc32c_model as M
from tests.test_gpu_model import _config, _make_dataset
from tests.test_gpu_multi_rank_model import TABLES, _models, _read_whole, _state

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _sixteen_target_rows(monkeypatch):
    import tests.test_gpu_model as toy
    monkeypatch.setattr(toy, "TARGETS", toy.TARGETS + ["make|copy", "do|it", "read|all", "write|all", "open", "flush",
                                                       "hash|code"])
    monkeypatch.setattr(toy, "TOKENS", ["tok%d" % i for i in range(64)])          # 4 source tokens per target


def _dev_bytes(data: bytes, offset: int):
    """data on the device at `offset` bytes past a 256-byte-aligned allocation."""
    import torch
    buf = torch.zeros(len(data) + offset + 16, dtype=torch.uint8, device="cuda")
    if data:
        buf[offset:offset + len(data)].copy_(torch.frombuffer(bytearray(data), dtype=torch.uint8))
    return buf, buf.data_ptr() + offset


def _rows(ptr, rows, row_bytes, stride):
    import torch
    from code2vec_b200.engine import load_library
    lib = load_library()
    out = torch.full((max(rows, 1),), -1, dtype=torch.int32, device="cuda")
    assert lib.c2v_crc32c_rows(ptr, rows, row_bytes, stride, out.data_ptr(), None) == 0
    torch.cuda.synchronize()
    return out[:rows].cpu().numpy().view(np.uint32)


def _combine(crcs, n, seg):
    import torch
    from code2vec_b200.engine import crc32c_combine
    out = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    crc32c_combine(crcs, n, seg, out)
    return int(out.cpu().numpy().view(np.uint32)[0])


@pytest.mark.parametrize("row_bytes", [0, 1, 3, 4, 15, 16, 17, 511, 512, 513, 1536])
def test_crc32c_rows_against_the_model(row_bytes):
    rng = np.random.default_rng(row_bytes)
    for rows in (1, 31, 32, 33):
        stride = row_bytes + (rows % 3)
        data = rng.integers(0, 256, rows * stride + 8, dtype=np.uint8).tobytes()
        want = [M.crc32c(data[r * stride:r * stride + row_bytes]) for r in range(rows)]
        for offset in range(16):
            if rows != 33 and offset not in (0, 5, 15):
                continue
            buf, ptr = _dev_bytes(data, offset)
            got = _rows(ptr, rows, row_bytes, stride)
            assert list(got) == want, (rows, offset)


def test_crc32c_rows_empty_and_refusals():
    from code2vec_b200.engine import load_library
    lib = load_library()
    assert lib.c2v_crc32c_rows(None, 0, 512, 512, None, None) == 0
    assert lib.c2v_crc32c_rows(None, 2, 16, 8, None, None) < 0
    assert b"row_stride" in lib.c2v_last_error(None)


def test_crc32c_java14m_token_table_and_combine():
    """1,301,136 rows of 512 B (the java14m token table), built from 8 random 4 KB chunks repeated: every row against
    the model, and the whole table's CRC by combining the device row CRCs against combining host CRCs of 4 KB chunks."""
    import torch
    rows, row_bytes = 1301136, 512
    rng = np.random.default_rng(7)
    chunks = rng.integers(0, 256, (8, 4096), dtype=np.uint8)
    n_chunks = rows * row_bytes // 4096
    order = np.arange(n_chunks) % 8
    dev = torch.from_numpy(chunks).cuda()[torch.from_numpy(order).cuda()].reshape(-1)
    got = _rows(dev.data_ptr(), rows, row_bytes, row_bytes)
    row_crc = np.array([[M.crc32c(chunks[c, 512 * j:512 * (j + 1)].tobytes()) for j in range(8)] for c in range(8)],
                       dtype=np.uint32)
    assert np.array_equal(got, row_crc[order.repeat(8), np.tile(np.arange(8), n_chunks)])
    chunk_crc = [M.crc32c(c.tobytes()) for c in chunks]
    k = M._xpow8(4096)
    acc = 0
    for i in range(n_chunks):
        acc = M._mulmodp(k, acc) ^ chunk_crc[order[i]]
    dev_crcs = torch.from_numpy(got.view(np.int32)).cuda()
    assert _combine(dev_crcs, rows, row_bytes) == acc
    for n in (1, 2, 3):
        assert _combine(dev_crcs, n, row_bytes) == M.combine_many(got[:n], row_bytes)
    assert _combine(dev_crcs, 0, row_bytes) == 0


# ---- the model --------------------------------------------------------------------------------------------------------
def _train_toy(tmp_path, monkeypatch, epochs=20):
    from code2vec_b200.b200_model import Code2VecModel
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    monkeypatch.setenv("C2V_DETERMINISTIC", "1")
    monkeypatch.setenv("C2V_SEED", "5")
    prefix, _ = _make_dataset(tmp_path, n_test=45)
    save = str(tmp_path / "model" / "saved")
    m = Code2VecModel(_config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, MODEL_SAVE_PATH=save,
                              NUM_TRAIN_EPOCHS=epochs))
    try:
        m.train()
    finally:
        m.close_session()
    return prefix, save


def _to_bundle(save, dest, optimizer=True):
    """The .c2v_b200 checkpoint `save` rewritten by the host writer as the bundle `dest`, dictionaries.bin beside it."""
    full = _read_whole(save + ".c2v_b200")
    arrays = {k: v for k, v in full.items() if k != "adam_t" and (optimizer or k.startswith("theta/"))}
    os.makedirs(os.path.dirname(dest), exist_ok=True)
    T.write_bundle_host(dest, arrays, adam_t=full["adam_t"] if optimizer else None)
    shutil.copy(os.path.join(os.path.dirname(save), "dictionaries.bin"), os.path.join(os.path.dirname(dest),
                                                                                      "dictionaries.bin"))
    return full


def _one_gpu_state(e):
    import torch
    torch.cuda.synchronize()
    s = {"adam_t": e.adam_t}
    for g, src in (("theta", e.params), ("adam_m", e.adam_m), ("adam_v", e.adam_v)):
        if src is not None:
            s.update({g + "/" + n: src[n].cpu().numpy().copy() for n in TABLES})
    return s


def _load(prefix, tmp_path, path, training=True, **kw):
    from code2vec_b200.b200_model import Code2VecModel
    extra = dict(TRAIN_DATA_PATH_PREFIX=prefix, NUM_TRAIN_EPOCHS=0) if training else {}
    return Code2VecModel(_config(prefix, tmp_path, MODEL_LOAD_PATH=path, **extra, **kw))


def test_import_bit_equal_and_outputs_byte_equal(tmp_path, monkeypatch):
    from code2vec_b200.vocabularies import VocabType
    prefix, save = _train_toy(tmp_path, monkeypatch)
    tf = str(tmp_path / "tf" / "saved")
    full = _to_bundle(save, tf)
    assert full["adam_t"] > 0
    m = _load(prefix, tmp_path, tf)
    try:
        got = _one_gpu_state(m.engine)
    finally:
        m.close_session()
    assert got["adam_t"] == full["adam_t"]
    for k, v in full.items():
        if k != "adam_t":
            assert got[k].tobytes() == v.tobytes(), k
    # --test (host and device evaluation), --predict, word2vec files and code vectors: byte-equal
    outputs = {}
    pred_lines = open(prefix + ".test.c2v").read().splitlines()[:6]
    for dev_eval in ("0", "1"):
        monkeypatch.setenv("C2V_DEVICE_EVAL", dev_eval)
        for tag, path in (("c2v", save), ("tf", tf)):
            m = _load(prefix, tmp_path, path, training=False, TEST_DATA_PATH=prefix + ".test.c2v",
                      EXPORT_CODE_VECTORS=True)
            try:
                res = m.evaluate()
                out = dict(res=str(res), log=open("log.txt").read(), vectors=open(prefix + ".test.c2v.vectors").read())
                for vt, n in ((VocabType.Token, "tok"), (VocabType.Target, "tgt"), (VocabType.Path, "path")):
                    m.save_word2vec_format(str(tmp_path / ("%s.%s.w2v" % (tag, n))), vt)
                    out[n] = open(str(tmp_path / ("%s.%s.w2v" % (tag, n))), "rb").read()
                out["predict"] = repr([(p.original_name, p.topk_predicted_words.tolist(),
                                        np.asarray(p.topk_predicted_words_scores).tobytes(),
                                        sorted(p.attention_per_context.items()), np.asarray(p.code_vector).tobytes())
                                       for p in m.predict(pred_lines)])
            finally:
                m.close_session()
            outputs[dev_eval + tag] = out
        assert outputs[dev_eval + "tf"] == outputs[dev_eval + "c2v"], dev_eval


@pytest.mark.parametrize("world", [2, 4, 8])
def test_import_on_emulated_ranks(tmp_path, monkeypatch, world):
    prefix, save = _train_toy(tmp_path, monkeypatch)
    tf = str(tmp_path / "tf" / "saved")
    _to_bundle(save, tf)
    make = lambda path: (lambda: _config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, NUM_TRAIN_EPOCHS=0,
                                         MODEL_LOAD_PATH=path))
    want = _models(monkeypatch, world, make(save), lambda model, r: _state(model.engine))
    got = _models(monkeypatch, world, make(tf), lambda model, r: _state(model.engine))
    for r in range(world):
        assert got[r]["adam_t"] == want[r]["adam_t"]
        for k in want[r]:
            if k != "adam_t":
                assert np.array_equal(got[r][k], want[r][k]), (r, k)
    # one flipped byte in the data file: the CRC error on every rank
    bad = str(tmp_path / "bad" / "saved")
    os.makedirs(os.path.dirname(bad))
    for f in os.listdir(os.path.dirname(tf)):
        shutil.copy(os.path.join(os.path.dirname(tf), f), os.path.join(os.path.dirname(bad), f))
    _, index = T.read_index(bad)
    at = index["model/PATHS_VOCAB"]["offset"] + 4 * 16 * 3 + 2                # row 3 of the path table: one rank's
    with open(T.data_file(bad), "r+b") as f:
        f.seek(at)
        b = f.read(1)
        f.seek(at)
        f.write(bytes([b[0] ^ 0x10]))
    errors = []

    def load_bad(r):
        from code2vec_b200.b200_model import Code2VecModel
        try:
            Code2VecModel(make(bad)()).close_session()
        except Exception as exc:                                              # noqa: BLE001
            errors.append((r, type(exc).__name__, str(exc)))
    from tests.test_gpu_multi_rank_model import _on_ranks
    _on_ranks(monkeypatch, world, load_bad, {"C2V_DETERMINISTIC": "1", "C2V_SEED": "5"})
    assert len(errors) == world, errors
    for r, kind, msg in errors:
        assert "model/PATHS_VOCAB fails its CRC-32C" in msg, (r, kind, msg)


def test_one_gpu_flipped_byte_raises(tmp_path, monkeypatch):
    prefix, save = _train_toy(tmp_path, monkeypatch, epochs=2)
    tf = str(tmp_path / "tf" / "saved")
    _to_bundle(save, tf)
    _, index = T.read_index(tf)
    at = index["model/TRANSFORM"]["offset"] + 1000
    with open(T.data_file(tf), "r+b") as f:
        f.seek(at)
        b = f.read(1)
        f.seek(at)
        f.write(bytes([b[0] ^ 0x01]))
    with pytest.raises(ValueError, match=r"checkpoint tensor model/TRANSFORM fails its CRC-32C: stored 0x[0-9a-f]{8}, "
                                         r"computed 0x[0-9a-f]{8}"):
        _load(prefix, tmp_path, tf)


def test_export_round_trip_resume_and_release(tmp_path, monkeypatch):
    from code2vec_b200.b200_model import Code2VecModel
    prefix, save = _train_toy(tmp_path, monkeypatch)
    full = _read_whole(save + ".c2v_b200")
    tf = str(tmp_path / "tf" / "saved")
    m = _load(prefix, tmp_path, save)
    try:
        monkeypatch.setattr(m, "_save_format", "tf")
        m.save(tf)
        m._save_inner_model(tf + ".release", release=True)
    finally:
        m.close_session()
    # the device-computed entry CRCs are the model's over the data file's bytes
    data = open(T.data_file(tf), "rb").read()
    _, index = T.read_index(tf)
    assert len(index) == 17 and T.adam_step_from_powers(
        *[np.frombuffer(data[index[k]["offset"]:index[k]["offset"] + 4], "<f4")[0] for k in T.BETA_KEYS],
        0.9, 0.999) == full["adam_t"]
    for k, e in index.items():
        assert T.unmask_crc(e["crc32c"]) == M.crc32c(data[e["offset"]:e["offset"] + e["size"]]), k
    _, rel = T.read_index(tf + ".release")
    assert sorted(rel) == sorted(T.tf_key("theta", n) for n in TABLES)
    # loads back bit-equal, Adam state included
    m = _load(prefix, tmp_path, tf)
    try:
        got = _one_gpu_state(m.engine)
    finally:
        m.close_session()
    assert got["adam_t"] == full["adam_t"]
    for k, v in full.items():
        if k != "adam_t":
            assert got[k].tobytes() == v.tobytes(), k
    # resuming two more epochs: from the bundle as from the .c2v_b200 checkpoint
    finals = {}
    for tag, path in (("c2v", save), ("tf", tf)):
        out = str(tmp_path / ("resumed_" + tag))
        m = Code2VecModel(_config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, NUM_TRAIN_EPOCHS=2,
                                  MODEL_LOAD_PATH=path, MODEL_SAVE_PATH=out))
        try:
            m.train()
        finally:
            m.close_session()
        finals[tag] = _read_whole(out + ".c2v_b200")
    for k in finals["c2v"]:
        assert np.array_equal(finals["tf"][k], finals["c2v"][k]), k
    # a release bundle loads for prediction with the same weights
    m = _load(prefix, tmp_path, tf + ".release", training=False)
    try:
        rel_state = _one_gpu_state(m.engine)
    finally:
        m.close_session()
    for n in TABLES:
        assert rel_state["theta/" + n].tobytes() == full["theta/" + n].tobytes(), n
