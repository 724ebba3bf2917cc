"""TensorFlow's V2 checkpoint format (the tensor bundle) without TensorFlow or protobuf (DESIGN.md §6k).

A checkpoint `<prefix>` is `<prefix>.index` plus data shards `<prefix>.data-%05d-of-%05d`:
  * the index is a LevelDB-format table: data blocks of prefix-compressed entries (varint shared / non-shared / value
    lengths, the key's new bytes, the value), a uint32 restart array and its count, each block followed by a 5-byte
    trailer (type byte 0 = uncompressed, then the masked CRC-32C of the contents and the type byte); a metaindex block;
    an index block whose entries map a key >= a data block's last key to that block's handle (varint offset, varint
    size); a 48-byte footer (the metaindex and index handles padded to 40 bytes, then 0xdb4775248b80fb57 little-endian);
  * the table maps "" to a BundleHeaderProto (num_shards 1, endianness 2 (LITTLE = 0), version 3 = VersionDef
    (producer 1, min_consumer 2)) and every tensor name to a BundleEntryProto (dtype 1, shape 2 (TensorShapeProto.dim 2,
    Dim.size 1), shard_id 3, offset 4, size 5, crc32c 6 (fixed32, masked), slices 7);
  * a data shard is the raw little-endian bytes of its tensors.
The reference's variables are the engine's tensors in the same layout (model/TRANSFORM is W [3d, D], model/ATTENTION is
a [D, 1]), so a bundle maps onto multi_rank's checkpoint entries {"name", "shape", "offset", "nbytes"} with a file per
entry; the CRC-32C of every tensor is computed on the GPU (c2v_crc32c_rows / c2v_crc32c_combine).  The host CRC here is
for the index's blocks and the two scalars only."""
from __future__ import annotations

import os
import struct
from typing import Dict, List, Optional, Tuple

import numpy as np

from .engine import PARAM_NAMES, EngineDims
from .multi_rank import _TF_NAMES

INDEX_SUFFIX = ".index"
TABLE_MAGIC = 0xdb4775248b80fb57
FOOTER_BYTES = 48
RESTART_INTERVAL = 16
DT_FLOAT = 1
BIG_ENDIAN = 1
MAX_ADAM_T = 10 ** 7
SAVE_FORMATS = ("c2v_b200", "tf", "keras")

_GROUP_SUFFIX = {"theta": "", "adam_m": "/Adam", "adam_v": "/Adam_1"}
BETA_KEYS = ("model/beta1_power", "model/beta2_power")


def save_format_flag(environ) -> str:
    """C2V_SAVE_FORMAT: "c2v_b200" (the default), "tf" (a TensorFlow V2 checkpoint: <path>.index + data) or "keras" (the
    reference Keras backend's <path>__entire-model/ckpt-N or <path>__only-weights, keras_ckpt.py)."""
    flag = environ.get("C2V_SAVE_FORMAT", "c2v_b200") or "c2v_b200"
    if flag not in SAVE_FORMATS:
        raise ValueError("C2V_SAVE_FORMAT must be c2v_b200, tf or keras, got %r" % flag)
    return flag


def data_file(prefix: str, shard: int = 0, num_shards: int = 1) -> str:
    return "%s.data-%05d-of-%05d" % (prefix, shard, num_shards)


def tf_key(group: str, name: str) -> str:
    """The TF variable of checkpoint tensor group/name ("theta/W" -> "model/TRANSFORM", "adam_v/tok" ->
    "model/WORDS_VOCAB/Adam_1")."""
    return _TF_NAMES[name] + _GROUP_SUFFIX[group]


def tf_shape(name: str, shape) -> Tuple[int, ...]:
    """The TF shape of an engine tensor: ATTENTION is [D, 1] where the engine holds a [D]."""
    return (int(shape[0]), 1) if name == "a" else tuple(int(s) for s in shape)


# ---- CRC-32C (host) -------------------------------------------------------------------------------------------------
def _crc_table():
    t = []
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ 0x82F63B78 if c & 1 else c >> 1
        t.append(c)
    return t


_CRC_TABLE = _crc_table()


def crc32c(data: bytes) -> int:
    c = 0xFFFFFFFF
    t = _CRC_TABLE
    for b in bytes(data):
        c = t[(c ^ b) & 0xFF] ^ (c >> 8)
    return c ^ 0xFFFFFFFF


def mask_crc(c: int) -> int:
    return ((((c >> 15) | (c << 17)) & 0xFFFFFFFF) + 0xA282EAD8) & 0xFFFFFFFF


def unmask_crc(m: int) -> int:
    r = (m - 0xA282EAD8) & 0xFFFFFFFF
    return ((r >> 17) | (r << 15)) & 0xFFFFFFFF


# ---- varints and protobuf fields ------------------------------------------------------------------------------------
def put_varint(v: int) -> bytes:
    v &= (1 << 64) - 1                             # negative int32 / int64 fields are ten-byte varints
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def get_varint(buf: bytes, pos: int) -> Tuple[int, int]:
    v = shift = 0
    while True:
        if pos >= len(buf) or shift > 63:
            raise ValueError("truncated or overlong varint in the checkpoint index")
        b = buf[pos]
        pos += 1
        v |= (b & 0x7F) << shift
        shift += 7
        if not b & 0x80:
            return v, pos


def _field(num: int, wire: int) -> bytes:
    return put_varint(num << 3 | wire)


def _pb_varint(num: int, v: int) -> bytes:
    return _field(num, 0) + put_varint(v) if v else b""


def _pb_bytes(num: int, payload: bytes) -> bytes:
    return _field(num, 2) + put_varint(len(payload)) + payload


def parse_fields(buf: bytes) -> List[Tuple[int, int, object]]:
    """[(field number, wire type, value)]: ints for varint / fixed fields, bytes for length-delimited ones."""
    out, pos = [], 0
    while pos < len(buf):
        key, pos = get_varint(buf, pos)
        num, wire = key >> 3, key & 7
        if wire == 0:
            v, pos = get_varint(buf, pos)
        elif wire == 1:
            if pos + 8 > len(buf):
                raise ValueError("truncated fixed64 field in the checkpoint index")
            (v,), pos = struct.unpack_from("<Q", buf, pos), pos + 8
        elif wire == 2:
            n, pos = get_varint(buf, pos)
            if pos + n > len(buf):
                raise ValueError("truncated length-delimited field in the checkpoint index")
            v, pos = bytes(buf[pos:pos + n]), pos + n
        elif wire == 5:
            if pos + 4 > len(buf):
                raise ValueError("truncated fixed32 field in the checkpoint index")
            (v,), pos = struct.unpack_from("<I", buf, pos), pos + 4
        else:
            raise ValueError("unsupported protobuf wire type %d in the checkpoint index" % wire)
        out.append((num, wire, v))
    return out


def _signed(v: int, bits: int = 64) -> int:
    v &= (1 << bits) - 1
    return v - (1 << bits) if v >> (bits - 1) else v


def encode_header(num_shards: int = 1) -> bytes:
    """BundleHeaderProto: num_shards, endianness LITTLE (0, omitted), version {producer 1, min_consumer 0}."""
    return _pb_varint(1, num_shards) + _pb_bytes(3, _pb_varint(1, 1))


def decode_header(buf: bytes) -> dict:
    h = {"num_shards": 0, "endianness": 0, "producer": 0, "min_consumer": 0}
    for num, wire, v in parse_fields(buf):
        if num == 1 and wire == 0:
            h["num_shards"] = _signed(v, 32)
        elif num == 2 and wire == 0:
            h["endianness"] = v
        elif num == 3 and wire == 2:
            for n2, w2, v2 in parse_fields(v):
                if n2 == 1 and w2 == 0:
                    h["producer"] = _signed(v2, 32)
                elif n2 == 2 and w2 == 0:
                    h["min_consumer"] = _signed(v2, 32)
    return h


def encode_entry(shape, offset: int, size: int, crc: int, shard_id: int = 0, dtype: int = DT_FLOAT) -> bytes:
    """BundleEntryProto of an unpartitioned tensor; `crc` is the plain CRC-32C (stored masked)."""
    dims = b"".join(_pb_bytes(2, _pb_varint(1, int(s))) for s in shape)
    return (_pb_varint(1, dtype) + _pb_bytes(2, dims) + _pb_varint(3, shard_id) + _pb_varint(4, offset) +
            _pb_varint(5, size) + _field(6, 5) + struct.pack("<I", mask_crc(crc)))


def decode_entry(buf: bytes) -> dict:
    e = {"dtype": 0, "shape": [], "shard_id": 0, "offset": 0, "size": 0, "crc32c": 0, "slices": 0}
    for num, wire, v in parse_fields(buf):
        if num == 1 and wire == 0:
            e["dtype"] = v
        elif num == 2 and wire == 2:
            for n2, w2, v2 in parse_fields(v):
                if n2 == 2 and w2 == 2:
                    size = 0
                    for n3, w3, v3 in parse_fields(v2):
                        if n3 == 1 and w3 == 0:
                            size = _signed(v3)
                    e["shape"].append(size)
        elif num == 3 and wire == 0:
            e["shard_id"] = _signed(v, 32)
        elif num == 4 and wire == 0:
            e["offset"] = _signed(v)
        elif num == 5 and wire == 0:
            e["size"] = _signed(v)
        elif num == 6 and wire == 5:
            e["crc32c"] = v
        elif num == 7:
            e["slices"] += 1
    return e


# ---- LevelDB table --------------------------------------------------------------------------------------------------
def build_block(items: List[Tuple[bytes, bytes]], restart_interval: int = RESTART_INTERVAL) -> bytes:
    """A block of sorted (key, value) items: prefix-compressed entries, restarts every `restart_interval` entries."""
    out, restarts, last = bytearray(), [0], b""
    for i, (k, v) in enumerate(items):
        shared = 0
        if i % restart_interval == 0:
            if i:
                restarts.append(len(out))
        else:
            n = min(len(last), len(k))
            while shared < n and last[shared] == k[shared]:
                shared += 1
        out += put_varint(shared) + put_varint(len(k) - shared) + put_varint(len(v)) + k[shared:] + v
        last = k
    for r in restarts:
        out += struct.pack("<I", r)
    out += struct.pack("<I", len(restarts))
    return bytes(out)


def block_trailer(contents: bytes, block_type: int = 0) -> bytes:
    return bytes([block_type]) + struct.pack("<I", mask_crc(crc32c(contents + bytes([block_type]))))


def _handle(offset: int, size: int) -> bytes:
    return put_varint(offset) + put_varint(size)


def build_table(items: List[Tuple[bytes, bytes]]) -> bytes:
    """The whole table of sorted items: one data block, an empty metaindex block, the index block (one entry keyed by
    the last key), the footer."""
    out = bytearray()

    def put(contents):
        off = len(out)
        out.extend(contents + block_trailer(contents))
        return _handle(off, len(contents))
    data = put(build_block(items))
    meta = put(build_block([]))
    index = put(build_block([(items[-1][0], data)] if items else []))
    footer = meta + index
    return bytes(out + footer + b"\0" * (40 - len(footer)) + struct.pack("<Q", TABLE_MAGIC))


def _read_block(buf: bytes, handle: bytes, what: str) -> bytes:
    off, pos = get_varint(handle, 0)
    size, _ = get_varint(handle, pos)
    if off + size + 5 > len(buf):
        raise ValueError("checkpoint index: the %s block [%d, %d) lies past the end of the file" % (what, off, off + size))
    contents, btype = buf[off:off + size], buf[off + size]
    (stored,) = struct.unpack_from("<I", buf, off + size + 1)
    if unmask_crc(stored) != crc32c(contents + bytes([btype])):
        raise ValueError("checkpoint index: the %s block at offset %d fails its trailer CRC-32C" % (what, off))
    if btype != 0:
        raise ValueError("checkpoint index: the %s block at offset %d is compressed (type %d); TensorFlow writes bundle "
                         "indexes uncompressed and only those are read" % (what, off, btype))
    return contents


def parse_block(contents: bytes) -> List[Tuple[bytes, bytes]]:
    """The (key, value) items of a block, whatever its restart interval."""
    if len(contents) < 4:
        raise ValueError("checkpoint index: a block of %d bytes has no restart count" % len(contents))
    (n_restarts,) = struct.unpack_from("<I", contents, len(contents) - 4)
    limit = len(contents) - 4 - 4 * n_restarts
    if n_restarts < 1 or limit < 0:
        raise ValueError("checkpoint index: a block has a bad restart count (%d)" % n_restarts)
    restarts = set(struct.unpack_from("<%dI" % n_restarts, contents, limit))
    items, pos, last = [], 0, b""
    while pos < limit:
        at = pos
        shared, pos = get_varint(contents, pos)
        non_shared, pos = get_varint(contents, pos)
        vlen, pos = get_varint(contents, pos)
        if shared > len(last) or (at in restarts and shared) or pos + non_shared + vlen > limit:
            raise ValueError("checkpoint index: a corrupt block entry at offset %d" % at)
        key = last[:shared] + contents[pos:pos + non_shared]
        pos += non_shared
        items.append((bytes(key), bytes(contents[pos:pos + vlen])))
        pos += vlen
        last = key
    return items


def parse_table(buf: bytes) -> List[Tuple[bytes, bytes]]:
    """Every item of every data block, in order."""
    if len(buf) < FOOTER_BYTES:
        raise ValueError("checkpoint index: %d bytes is shorter than a table footer" % len(buf))
    footer = buf[len(buf) - FOOTER_BYTES:]
    (magic,) = struct.unpack_from("<Q", footer, 40)
    if magic != TABLE_MAGIC:
        raise ValueError("checkpoint index: bad table magic 0x%016x (want 0x%016x)" % (magic, TABLE_MAGIC))
    pos = 0
    for _ in range(2):                                # the metaindex handle, not needed
        _, pos = get_varint(footer, pos)
    start = pos
    for _ in range(2):
        _, pos = get_varint(footer, pos)
    items = []
    for _, handle in parse_block(_read_block(buf, footer[start:pos], "index")):
        items += parse_block(_read_block(buf, handle, "data"))
    return items


# ---- Adam step <-> beta powers --------------------------------------------------------------------------------------
def beta_powers(t: int, beta1: float, beta2: float) -> Tuple[np.float32, np.float32]:
    """What TF1's AdamOptimizer holds after t steps: p_(t+1), where p_1 = fl(beta), p_k = fl(p_(k-1) * fl(beta))."""
    out = []
    for beta in (beta1, beta2):
        b = np.float32(beta)
        p = b
        for _ in range(int(t)):
            np_p = np.float32(p * b)
            if np_p == p:                             # the denormal fixed point: no later step changes it
                break
            p = np_p
        out.append(p)
    return out[0], out[1]


def adam_step_from_powers(p1, p2, beta1: float, beta2: float, max_t: int = MAX_ADAM_T) -> int:
    """The smallest t <= max_t whose beta powers are (p1, p2) bit for bit; ValueError if there is none."""
    want = (np.float32(p1), np.float32(p2))
    b = (np.float32(beta1), np.float32(beta2))
    p = list(b)
    for t in range(max_t + 1):
        if p[0] == want[0] and p[1] == want[1]:
            return t
        nxt = [np.float32(p[i] * b[i]) for i in range(2)]
        if nxt == p:                                  # both at their fixed points: no larger t matches either
            break
        p = nxt
    raise ValueError("model/beta1_power = %r and model/beta2_power = %r are the Adam beta powers of no step count up to "
                     "%d (beta1 = %r, beta2 = %r)" % (float(want[0]), float(want[1]), max_t, beta1, beta2))


# ---- bundles --------------------------------------------------------------------------------------------------------
def read_index(prefix: str, other_dtypes: Optional[Dict[str, int]] = None) -> Tuple[dict, Dict[str, dict]]:
    """(header, {tensor key: entry}) of the bundle `prefix`, with the refusals of the format's limits.  Every tensor is
    DT_FLOAT except the keys of `other_dtypes`, which must have the dtype it gives them (keras_ckpt.py)."""
    path = prefix + INDEX_SUFFIX
    with open(path, "rb") as f:
        buf = f.read()
    items = parse_table(buf)
    entries, header = {}, None
    for k, v in items:
        if k == b"":
            header = decode_header(v)
        else:
            entries[k.decode("utf-8")] = decode_entry(v)
    if header is None:
        raise ValueError("`%s` has no bundle header (the entry under the empty key)" % path)
    if header["endianness"] == BIG_ENDIAN:
        raise ValueError("`%s` is a big-endian bundle; only little-endian bundles are read" % path)
    if header["min_consumer"] > 1:
        raise ValueError("`%s` needs a bundle reader of version >= %d (this one is version 1)" % (path, header["min_consumer"]))
    if header["num_shards"] < 1:
        raise ValueError("`%s` has num_shards = %d" % (path, header["num_shards"]))
    for k, e in entries.items():
        if e["slices"]:
            raise ValueError("`%s`: tensor %s is partitioned (slices); only whole tensors are read" % (path, k))
        if other_dtypes and k in other_dtypes:
            if e["dtype"] != other_dtypes[k]:
                raise ValueError("`%s`: tensor %s has dtype %d; it must be %d" % (path, k, e["dtype"], other_dtypes[k]))
        elif e["dtype"] != DT_FLOAT:
            raise ValueError("`%s`: tensor %s has dtype %d; only DT_FLOAT (1) is read" % (path, k, e["dtype"]))
        if not 0 <= e["shard_id"] < header["num_shards"]:
            raise ValueError("`%s`: tensor %s is in shard %d of %d" % (path, k, e["shard_id"], header["num_shards"]))
        e["file"] = data_file(prefix, e["shard_id"], header["num_shards"])
    for s in range(header["num_shards"]):
        if not os.path.isfile(data_file(prefix, s, header["num_shards"])):
            raise ValueError("bundle `%s` is missing its data shard `%s`" % (prefix, data_file(prefix, s, header["num_shards"])))
    return header, entries


def _check_entry(key: str, e: dict, want_shape) -> None:
    if tuple(e["shape"]) != tuple(want_shape):
        raise ValueError("checkpoint tensor %s has shape %s; the model needs %s (dictionaries.bin and the config)" % (
            key, list(e["shape"]), list(want_shape)))
    n = 4 * int(np.prod(want_shape, dtype=np.int64))
    if e["size"] != n:
        raise ValueError("checkpoint tensor %s: its entry says %d bytes, its shape %d" % (key, e["size"], n))
    size = os.path.getsize(e["file"])
    if e["offset"] < 0 or e["offset"] + n > size:
        raise ValueError("checkpoint tensor %s: bytes [%d, %d) lie past the end of `%s` (%d bytes)" % (
            key, e["offset"], e["offset"] + n, e["file"], size))


def bundle_entries(prefix: str, dims: dict, with_optimizer: bool, beta1: float, beta2: float):
    """(entries, adam_t): this model's tensors in the bundle `prefix` as multi_rank's checkpoint entries {"name", "shape",
    "offset", "nbytes"} plus "file" (the data shard) and "crc" (the plain CRC-32C the bundle stores) and "key", in PARAM_NAMES
    order per group ("theta", and "adam_m" / "adam_v" with `with_optimizer` when the bundle has Adam slots), and the
    Adam step the beta powers give (0 without them).  ValueError if a tensor is missing or has another shape than `dims` (vars(EngineDims)) give."""
    _, index = read_index(prefix)
    shapes = EngineDims(**dims).shapes()
    with_optimizer = with_optimizer and tf_key("adam_m", "tok") in index     # a release: weights only, adam_t = 0
    out = []
    for g in ("theta", "adam_m", "adam_v") if with_optimizer else ("theta",):
        for name in PARAM_NAMES:
            key = tf_key(g, name)
            if key not in index:
                raise ValueError("bundle `%s` has no tensor %s" % (prefix, key))
            e = index[key]
            _check_entry(key, e, tf_shape(name, shapes[name]))
            out.append({"name": g + "/" + name, "shape": list(shapes[name]), "offset": e["offset"], "nbytes": e["size"],
                        "file": e["file"], "crc": unmask_crc(e["crc32c"]), "key": key})
    adam_t = 0
    if with_optimizer:
        powers = []
        for key in BETA_KEYS:
            e = index.get(key, index.get(key.split("/", 1)[1]))
            if e is None:
                raise ValueError("bundle `%s` has no tensor %s" % (prefix, key))
            _check_entry(key, e, ())
            with open(e["file"], "rb") as f:
                f.seek(e["offset"])
                raw = f.read(4)
            if crc32c(raw) != unmask_crc(e["crc32c"]):
                raise ValueError("checkpoint tensor %s fails its CRC-32C: stored 0x%08x, computed 0x%08x" % (
                    key, unmask_crc(e["crc32c"]), crc32c(raw)))
            powers.append(np.frombuffer(raw, dtype="<f4")[0])
        adam_t = adam_step_from_powers(powers[0], powers[1], beta1, beta2)
    return out, adam_t


def crc_view(name: str, shape) -> Tuple[int, int]:
    """(rows, row_bytes) the CRC kernels see a tensor as: its rows, or one row for the [D] attention vector."""
    shape = tuple(int(s) for s in shape)
    return (shape[0], 4 * int(np.prod(shape[1:], dtype=np.int64))) if len(shape) == 2 else (1, 4 * int(np.prod(shape)))


def bundle_layout(dims: dict, with_optimizer: bool, adam_t: int, beta1: float, beta2: float):
    """(tensors, scalars) of a bundle written from a model with `dims`: tensors = [(key, "group/name", TF shape, offset,
    nbytes)] and scalars = [(key, float32 value, offset)] in key order, back to back in one data shard."""
    shapes = EngineDims(**dims).shapes()
    items = []
    for g in ("theta", "adam_m", "adam_v") if with_optimizer else ("theta",):
        for name in PARAM_NAMES:
            items.append((tf_key(g, name), g + "/" + name, tf_shape(name, shapes[name])))
    powers = dict(zip(BETA_KEYS, beta_powers(adam_t, beta1, beta2))) if with_optimizer else {}
    items += [(k, None, ()) for k in powers]
    items.sort(key=lambda it: it[0].encode())
    tensors, scalars, off = [], [], 0
    for key, name, shape in items:
        n = 4 * int(np.prod(shape, dtype=np.int64))
        if name is None:
            scalars.append((key, powers[key], off))
        else:
            tensors.append((key, name, shape, off, n))
        off += n
    return tensors, scalars


def write_index(prefix: str, entries: List[Tuple[str, Tuple[int, ...], int, int, int]]) -> None:
    """<prefix>.index for one data shard: entries = [(key, TF shape, offset, size, plain CRC-32C)]."""
    items = [(b"", encode_header(1))]
    items += sorted((k.encode(), encode_entry(shape, off, size, crc)) for k, shape, off, size, crc in entries)
    with open(prefix + INDEX_SUFFIX, "wb") as f:
        f.write(build_table(items))


def write_bundle_host(prefix: str, arrays: Dict[str, np.ndarray], adam_t: Optional[int] = None,
                      beta1: float = 0.9, beta2: float = 0.999) -> None:
    """A bundle from host arrays {"theta/tok": ..., "adam_m/W": ...} (the engine's shapes), CRCs on the host: for
    tests and tools.  With adam_t, the beta powers of that step are written too."""
    items = [(tf_key(*n.split("/")), n) for n in arrays]
    if adam_t is not None:
        items += [(k, k) for k in BETA_KEYS]
    items.sort(key=lambda it: it[0].encode())
    powers = dict(zip(BETA_KEYS, beta_powers(adam_t, beta1, beta2))) if adam_t is not None else {}
    entries, off = [], 0
    with open(data_file(prefix), "wb") as f:
        for key, n in items:
            if n in powers:
                raw, shape = np.asarray(powers[n], dtype="<f4").tobytes(), ()
            else:
                a = np.ascontiguousarray(arrays[n], dtype="<f4")
                raw, shape = a.tobytes(), tf_shape(n.split("/")[1], a.shape)
            f.write(raw)
            entries.append((key, shape, off, len(raw), crc32c(raw)))
            off += len(raw)
    write_index(prefix, entries)
