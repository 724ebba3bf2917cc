"""TensorFlow V2 checkpoints on the host (code2vec_b200/tf_bundle.py): CRC-32C against its published check values, the
index bytes assembled field by field, reading other writers' layouts, every refusal, the Adam step <-> beta powers
mapping, and which checkpoint --load reads."""
import os
import struct

import numpy as np
import pytest

from code2vec_b200 import tf_bundle as T
from tests import crc32c_model as M


# ---- CRC-32C ----------------------------------------------------------------------------------------------------------
CHECK_VALUES = [(b"123456789", 0xE3069283), (bytes(32), 0x8A9136AA), (b"\xff" * 32, 0x62A8AB43),
                (bytes(range(32)), 0x46DD794E), (bytes(range(31, -1, -1)), 0x113FDB5C)]


@pytest.mark.parametrize("data,want", CHECK_VALUES)
def test_crc32c_check_values(data, want):
    assert M.crc32c(data) == want
    assert T.crc32c(data) == want


def test_masks():
    assert M.mask(0xE3069283) == 0xC78AB0E5 and M.mask(0) == 0xA282EAD8
    assert T.mask_crc(0xE3069283) == 0xC78AB0E5 and T.mask_crc(0) == 0xA282EAD8
    for c in (0, 1, 0xE3069283, 0xFFFFFFFF, 0x12345678):
        assert T.unmask_crc(T.mask_crc(c)) == c


def test_combine_model():
    rng = np.random.default_rng(1)
    data = rng.integers(0, 256, 3 * 37, dtype=np.uint8).tobytes()
    assert M.combine(M.crc32c(data[:50]), M.crc32c(data[50:]), len(data) - 50) == M.crc32c(data)
    assert M.combine_many([M.crc32c(data[i:i + 37]) for i in range(0, len(data), 37)], 37) == M.crc32c(data)
    assert M.combine_many([], 37) == 0 and M.crc32c(b"") == 0


# ---- index bytes ------------------------------------------------------------------------------------------------------
def _v(n):
    out = b""
    while n >= 0x80:
        out += bytes([(n & 0x7F) | 0x80])
        n >>= 7
    return out + bytes([n])


def _trailer(block):
    return b"\x00" + struct.pack("<I", M.mask(M.crc32c(block + b"\x00")))


def test_writer_index_bytes_field_by_field(tmp_path):
    prefix = str(tmp_path / "m")
    crc_a, crc_w = 0x01020304, 0xA0B0C0D0
    T.write_index(prefix, [("model/TRANSFORM", (6, 4), 16, 96, crc_w), ("model/ATTENTION", (4, 1), 0, 16, crc_a)])
    header = b"\x08\x01" + b"\x1a\x02" + b"\x08\x01"                    # num_shards 1, version {producer 1}
    ent_a = (b"\x08\x01" + b"\x12\x08" + b"\x12\x02\x08\x04" + b"\x12\x02\x08\x01" + b"\x28\x10" +
             b"\x35" + struct.pack("<I", M.mask(crc_a)))                 # dtype, shape [4, 1], size 16, crc32c
    ent_w = (b"\x08\x01" + b"\x12\x08" + b"\x12\x02\x08\x06" + b"\x12\x02\x08\x04" + b"\x20\x10" + b"\x28\x60" +
             b"\x35" + struct.pack("<I", M.mask(crc_w)))                 # ... offset 16, size 96
    data = (_v(0) + _v(0) + _v(len(header)) + header +
            _v(0) + _v(15) + _v(len(ent_a)) + b"model/ATTENTION" + ent_a +
            _v(6) + _v(9) + _v(len(ent_w)) + b"TRANSFORM" + ent_w +      # "model/" shared with the previous key
            struct.pack("<I", 0) + struct.pack("<I", 1))
    meta = struct.pack("<I", 0) + struct.pack("<I", 1)
    meta_off = len(data) + 5
    handle = _v(0) + _v(len(data))
    index = _v(0) + _v(15) + _v(len(handle)) + b"model/TRANSFORM" + handle + struct.pack("<I", 0) + struct.pack("<I", 1)
    index_off = meta_off + len(meta) + 5
    footer = _v(meta_off) + _v(len(meta)) + _v(index_off) + _v(len(index))
    want = (data + _trailer(data) + meta + _trailer(meta) + index + _trailer(index) +
            footer + bytes(40 - len(footer)) + struct.pack("<Q", 0xdb4775248b80fb57))
    got = open(prefix + ".index", "rb").read()
    assert got == want
    open(prefix + ".data-00000-of-00001", "wb").write(bytes(112))
    header_d, entries = T.read_index(prefix)
    assert header_d["num_shards"] == 1 and header_d["producer"] == 1 and header_d["min_consumer"] == 0
    assert entries["model/ATTENTION"]["shape"] == [4, 1] and T.unmask_crc(entries["model/ATTENTION"]["crc32c"]) == crc_a
    assert entries["model/TRANSFORM"]["offset"] == 16 and entries["model/TRANSFORM"]["size"] == 96


def _handle(off, size):
    return T.put_varint(off) + T.put_varint(size)


def _table(blocks_items, restart_interval, compress_type=0, index_interval=16):
    """A table of several data blocks (each a list of sorted items) at the given restart interval."""
    out, index_items = bytearray(), []
    for items in blocks_items:
        c = T.build_block(items, restart_interval)
        index_items.append((items[-1][0], _handle(len(out), len(c))))
        out += c + T.block_trailer(c, compress_type)
    meta = T.build_block([])
    meta_h = _handle(len(out), len(meta))
    out += meta + T.block_trailer(meta)
    idx = T.build_block(index_items, index_interval)
    idx_h = _handle(len(out), len(idx))
    out += idx + T.block_trailer(idx)
    footer = meta_h + idx_h
    return bytes(out + footer + bytes(40 - len(footer)) + struct.pack("<Q", T.TABLE_MAGIC))


def _bundle_items(n, seed=0):
    rng = np.random.default_rng(seed)
    items = [(b"", T.encode_header(1))]
    for i in range(n):
        items.append((("model/T%03d/x" % i).encode(), T.encode_entry((2, 3), 24 * i, 24, int(rng.integers(0, 2 ** 32)))))
    return items


@pytest.mark.parametrize("restart_interval", [1, 3, 16, 1000])
def test_reader_parses_many_blocks_and_restart_intervals(tmp_path, restart_interval):
    items = _bundle_items(40)
    blocks = [items[:7], items[7:8], items[8:30], items[30:]]
    prefix = str(tmp_path / "m")
    open(prefix + ".index", "wb").write(_table(blocks, restart_interval, index_interval=2))
    open(prefix + ".data-00000-of-00001", "wb").write(bytes(24 * 40))
    assert T.parse_table(open(prefix + ".index", "rb").read()) == items
    _, entries = T.read_index(prefix)
    assert sorted(entries) == sorted(k.decode() for k, _ in items[1:])
    assert entries["model/T017/x"]["offset"] == 24 * 17


# ---- refusals ---------------------------------------------------------------------------------------------------------
DIMS = dict(token_vocab=7, path_vocab=5, target_vocab=6, embed_dim=4, code_dim=8, max_contexts=3, max_batch=2, top_k=2)


def _arrays(seed=0, dims=DIMS, optimizer=True):
    from code2vec_b200.engine import EngineDims
    rng = np.random.default_rng(seed)
    shapes = EngineDims(**dims).shapes()
    groups = ("theta", "adam_m", "adam_v") if optimizer else ("theta",)
    return {g + "/" + k: rng.standard_normal(s).astype(np.float32) for g in groups for k, s in shapes.items()}


def _write(tmp_path, adam_t=7, **kw):
    prefix = str(tmp_path / "m")
    T.write_bundle_host(prefix, _arrays(**kw), adam_t=adam_t)
    return prefix


def _rewrite_index(prefix, edit):
    """Re-encode the index after edit(header dict-of-bytes items) changes its items."""
    items = T.parse_table(open(prefix + ".index", "rb").read())
    items = edit(items)
    open(prefix + ".index", "wb").write(T.build_table(items))


def _entries(prefix, optimizer=True):
    return T.bundle_entries(prefix, DIMS, optimizer, 0.9, 0.999)


def test_host_bundle_round_trip(tmp_path):
    prefix = _write(tmp_path)
    arrays = _arrays()
    entries, adam_t = _entries(prefix)
    assert adam_t == 7 and len(entries) == 15
    for ent in entries:
        raw = open(ent["file"], "rb").read()[ent["offset"]:ent["offset"] + ent["nbytes"]]
        assert np.array_equal(np.frombuffer(raw, "<f4").reshape(ent["shape"]), arrays[ent["name"]])
        assert M.crc32c(raw) == ent["crc"]
    # data in key order, back to back
    keys = sorted(T.read_index(prefix)[1].items(), key=lambda kv: kv[0].encode())
    assert [e["offset"] for _, e in keys] == list(np.cumsum([0] + [e["size"] for _, e in keys])[:-1])
    # a release: weights only, adam_t 0, also when the model wants its slots
    rel = str(tmp_path / "r")
    T.write_bundle_host(rel, _arrays(optimizer=False))
    entries, adam_t = _entries(rel)
    assert adam_t == 0 and [e["name"].split("/")[0] for e in entries] == ["theta"] * 5


def test_refuses_bad_magic(tmp_path):
    prefix = _write(tmp_path)
    buf = bytearray(open(prefix + ".index", "rb").read())
    buf[-1] ^= 0xFF
    open(prefix + ".index", "wb").write(bytes(buf))
    with pytest.raises(ValueError, match="bad table magic"):
        _entries(prefix)


def test_refuses_block_trailer_crc(tmp_path):
    prefix = _write(tmp_path)
    buf = bytearray(open(prefix + ".index", "rb").read())
    buf[3] ^= 0x01                                          # inside the data block
    open(prefix + ".index", "wb").write(bytes(buf))
    with pytest.raises(ValueError, match="fails its trailer CRC-32C"):
        _entries(prefix)


def test_refuses_compressed_block(tmp_path):
    prefix = str(tmp_path / "m")
    open(prefix + ".index", "wb").write(_table([_bundle_items(3)], 16, compress_type=1))
    with pytest.raises(ValueError, match="is compressed"):
        T.read_index(prefix)


def _edit_entry(prefix, key, **fields):
    def edit(items):
        out = []
        for k, v in items:
            if k == key.encode():
                e = T.decode_entry(v)
                e.update(fields)
                v = (T._pb_varint(1, e["dtype"]) + T._pb_bytes(2, b"".join(T._pb_bytes(2, T._pb_varint(1, s))
                                                                          for s in e["shape"])) +
                     T._pb_varint(4, e["offset"]) + T._pb_varint(5, e["size"]) + T._field(6, 5) +
                     struct.pack("<I", e["crc32c"]) + (T._pb_bytes(7, b"\x0a\x00") if e["slices"] else b""))
            out.append((k, v))
        return out
    _rewrite_index(prefix, edit)


def test_refuses_non_float_dtype(tmp_path):
    prefix = _write(tmp_path)
    _edit_entry(prefix, "model/TRANSFORM", dtype=19)        # DT_HALF
    with pytest.raises(ValueError, match="model/TRANSFORM has dtype 19; only DT_FLOAT"):
        _entries(prefix)


def test_refuses_slices(tmp_path):
    prefix = _write(tmp_path)
    _edit_entry(prefix, "model/TRANSFORM", slices=1)
    with pytest.raises(ValueError, match="model/TRANSFORM is partitioned"):
        _entries(prefix)


def _edit_header(prefix, payload):
    _rewrite_index(prefix, lambda items: [(k, payload if k == b"" else v) for k, v in items])


def test_refuses_big_endian_and_newer_consumers(tmp_path):
    prefix = _write(tmp_path)
    _edit_header(prefix, T._pb_varint(1, 1) + T._pb_varint(2, 1) + T._pb_bytes(3, T._pb_varint(1, 1)))
    with pytest.raises(ValueError, match="big-endian"):
        _entries(prefix)
    _edit_header(prefix, T._pb_varint(1, 1) + T._pb_bytes(3, T._pb_varint(1, 3) + T._pb_varint(2, 2)))
    with pytest.raises(ValueError, match="version >= 2"):
        _entries(prefix)
    _edit_header(prefix, T._pb_varint(1, 1) + T._pb_bytes(3, T._pb_varint(1, 3) + T._pb_varint(2, 1)))
    assert _entries(prefix)[1] == 7                         # min_consumer 1 is read


def test_refuses_missing_shard(tmp_path):
    prefix = _write(tmp_path)
    _edit_header(prefix, T._pb_varint(1, 2) + T._pb_bytes(3, T._pb_varint(1, 1)))
    os.rename(prefix + ".data-00000-of-00001", prefix + ".data-00000-of-00002")
    with pytest.raises(ValueError, match=r"missing its data shard `.*\.data-00001-of-00002`"):
        _entries(prefix)


def test_refuses_missing_key(tmp_path):
    prefix = _write(tmp_path)
    _rewrite_index(prefix, lambda items: [(k, v) for k, v in items if k != b"model/PATHS_VOCAB/Adam_1"])
    with pytest.raises(ValueError, match="has no tensor model/PATHS_VOCAB/Adam_1"):
        _entries(prefix)
    _entries(prefix, optimizer=False)                       # the weights alone are all there


def test_refuses_wrong_shape(tmp_path):
    prefix = _write(tmp_path)
    dims = dict(DIMS, token_vocab=8)
    with pytest.raises(ValueError, match=r"model/WORDS_VOCAB has shape \[7, 4\]; the model needs \[8, 4\]"):
        T.bundle_entries(prefix, dims, True, 0.9, 0.999)


def test_refuses_truncated_data_file(tmp_path):
    prefix = _write(tmp_path)
    with open(prefix + ".data-00000-of-00001", "r+b") as f:
        f.truncate(100)
    with pytest.raises(ValueError, match="lie past the end"):
        _entries(prefix)


def test_unscoped_beta_powers_are_read(tmp_path):
    prefix = _write(tmp_path, adam_t=3)
    _rewrite_index(prefix, lambda items: sorted((k.replace(b"model/beta", b"beta"), v) for k, v in items))
    assert _entries(prefix)[1] == 3


# ---- Adam step <-> beta powers ----------------------------------------------------------------------------------------
def _tf1_powers(t, b1=0.9, b2=0.999):
    out = []
    for beta in (b1, b2):
        p = np.float32(beta)
        for _ in range(t):
            p = np.float32(p * np.float32(beta))
        out.append(p)
    return out


@pytest.mark.parametrize("t", [0, 1, 2, 1000, 50000])
def test_adam_t_round_trip(t):
    p1, p2 = T.beta_powers(t, 0.9, 0.999)
    want = _tf1_powers(t)
    assert p1.tobytes() == want[0].tobytes() and p2.tobytes() == want[1].tobytes()
    assert T.adam_step_from_powers(p1, p2, 0.9, 0.999) == t


def test_adam_t_past_the_denormal_plateau():
    p1, p2 = T.beta_powers(10 ** 6, 0.9, 0.999)
    assert 0 < p2 < np.finfo(np.float32).tiny and 0 < p1 < np.finfo(np.float32).tiny      # both denormal, not 0
    t0 = T.adam_step_from_powers(p1, p2, 0.9, 0.999)
    assert t0 < 10 ** 6
    q1, q2 = T.beta_powers(t0, 0.9, 0.999)
    assert (q1.tobytes(), q2.tobytes()) == (p1.tobytes(), p2.tobytes())
    r1, r2 = T.beta_powers(t0 - 1, 0.9, 0.999)
    assert (r1.tobytes(), r2.tobytes()) != (p1.tobytes(), p2.tobytes())                   # the smallest such t


def test_adam_t_refuses_powers_no_step_gives():
    with pytest.raises(ValueError, match="beta powers of no step count"):
        T.adam_step_from_powers(np.float32(0.5), np.float32(0.5), 0.9, 0.999)
    p1, _ = T.beta_powers(5, 0.9, 0.999)
    _, p2 = T.beta_powers(6, 0.9, 0.999)
    with pytest.raises(ValueError, match="beta powers of no step count"):
        T.adam_step_from_powers(p1, p2, 0.9, 0.999)


# ---- format selection -------------------------------------------------------------------------------------------------
class _Cfg:
    def __init__(self, path):
        self.MODEL_LOAD_PATH = path


def _load_calls(monkeypatch, path):
    from code2vec_b200.b200_model import Code2VecModel
    calls = []
    m = Code2VecModel.__new__(Code2VecModel)
    m.config, m.world, m.rank = _Cfg(path), 1, 0
    monkeypatch.setattr(m, "_make_engine", lambda: None, raising=False)
    monkeypatch.setattr(m, "log", lambda msg: calls.append(("log", msg)), raising=False)
    monkeypatch.setattr(m, "_read_checkpoint", lambda p: calls.append(("c2v_b200", p)), raising=False)
    monkeypatch.setattr(m, "_read_bundle", lambda p: calls.append(("tf", p)), raising=False)
    m._load_inner_model()
    return [c for c in calls if c[0] != "log"], [c[1] for c in calls if c[0] == "log"]


def test_load_prefers_c2v_b200(tmp_path, monkeypatch):
    x = str(tmp_path / "saved_model_iter8.release")
    open(x + ".index", "wb").write(b"")
    got, logs = _load_calls(monkeypatch, x)
    assert got == [("tf", x)] and any("TensorFlow checkpoint" in l for l in logs)
    open(x + ".c2v_b200", "wb").write(b"")
    assert _load_calls(monkeypatch, x)[0] == [("c2v_b200", x + ".c2v_b200")]
    os.remove(x + ".index")
    os.remove(x + ".c2v_b200")
    assert _load_calls(monkeypatch, x)[0] == [("c2v_b200", x + ".c2v_b200")]   # which raises "There is no model"


def test_save_format_flag_and_multi_rank_refusal():
    from code2vec_b200.multi_rank import check_multi_rank_run
    assert T.save_format_flag({}) == "c2v_b200" and T.save_format_flag({"C2V_SAVE_FORMAT": "tf"}) == "tf"
    with pytest.raises(ValueError, match="C2V_SAVE_FORMAT must be"):
        T.save_format_flag({"C2V_SAVE_FORMAT": "TF"})

    class Cfg:
        TRAIN_BATCH_SIZE, PREDICT, RELEASE, DL_FRAMEWORK = 8, False, False, "b200"
    for w in (2, 4, 8):
        with pytest.raises(ValueError, match="C2V_SAVE_FORMAT=tf"):
            check_multi_rank_run(Cfg, w, "tf")
        check_multi_rank_run(Cfg, w)
    check_multi_rank_run(Cfg, 1, "tf")


def test_model_refuses_tf_save_on_ranks_before_any_engine(monkeypatch):
    from code2vec_b200 import b200_model as bm
    monkeypatch.setenv("WORLD_SIZE", "2")
    monkeypatch.setenv("C2V_SAVE_FORMAT", "tf")
    monkeypatch.setattr(bm.Code2VecModel, "_join_group", lambda self: pytest.fail("joined a process group"))

    class Cfg:
        TRAIN_BATCH_SIZE, PREDICT, RELEASE, DL_FRAMEWORK = 8, False, False, "b200"
    with pytest.raises(ValueError, match="C2V_SAVE_FORMAT=tf"):
        bm.Code2VecModel(Cfg())
