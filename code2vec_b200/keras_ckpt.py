"""The reference Keras backend's checkpoints (keras_model.py:230-296) without TensorFlow (DESIGN.md §6l).

They are tensor bundles (tf_bundle.py) with object-based keys:
  * `X__entire-model/ckpt-N` is what tf.train.CheckpointManager(tf.train.Checkpoint(optimizer=..., model=...)) writes:
    the layers under `model/`, the optimizer under `optimizer/`, `save_counter`, and beside them the state file
    `X__entire-model/checkpoint` that names the kept checkpoints;
  * `X__only-weights` is what `save_weights` writes: the model is the root, so the layers have no `model/` prefix.
A variable's key is its path of child names from the root plus `/.ATTRIBUTES/VARIABLE_VALUE`; an Adam slot's is its
variable's path plus `/.OPTIMIZER_SLOT/optimizer/<m|v>/.ATTRIBUTES/VARIABLE_VALUE`.  The entry
`_CHECKPOINTABLE_OBJECT_GRAPH` (a DT_STRING scalar) holds the serialized TrackableObjectGraph that names them, and the
reader finds every variable through it, by its path under a `layer_with_weights-N` node and its shape:
    embeddings [T, d] -> tok, embeddings [P, d] -> path (T = P: the lower N is path_embedding, created first),
    layer/kernel [3d, D] -> W, attention_param [D, 1] -> a, kernel [D, Y] -> tgt transposed (the engine holds [Y, D]).
`optimizer/iter` (DT_INT64) is the Adam step; `beta_1`, `beta_2`, `decay` and `learning_rate` are float32 scalars that
must be the loading framework's Adam.  The writer numbers the layers in keras_model.py's creation order."""
from __future__ import annotations

import glob
import os
import re
import struct
from typing import Dict, List, Optional, Tuple

import numpy as np

from .engine import PARAM_NAMES, EngineDims
from .tf_bundle import (DT_FLOAT, INDEX_SUFFIX, _check_entry, _pb_bytes, _pb_varint, build_table, crc32c, encode_entry,
                        encode_header, get_varint, mask_crc, parse_fields, put_varint, read_index, unmask_crc)

DT_STRING = 7
DT_INT64 = 9
OBJECT_GRAPH_KEY = "_CHECKPOINTABLE_OBJECT_GRAPH"
VALUE = "/.ATTRIBUTES/VARIABLE_VALUE"
ITER_KEY = "optimizer/iter" + VALUE
SAVE_COUNTER_KEY = "save_counter" + VALUE
STATE_FILE = "checkpoint"
# engine tensor -> (layer name, attribute path under its layer_with_weights-N node), in keras_model.py:46-70's order
LAYERS = (("path", "path_embedding", "embeddings"), ("tok", "token_embedding", "embeddings"),
          ("W", "time_distributed", "layer/kernel"), ("a", "attention", "attention_param"),
          ("tgt", "target_index", "kernel"))
HYPERS = ("beta_1", "beta_2", "decay", "iter", "learning_rate")          # the optimizer's variables, sorted
SLOTS = (("adam_m", "m"), ("adam_v", "v"))


def keras_shape(name: str, dims: EngineDims) -> Tuple[int, ...]:
    """The Keras shape of engine tensor `name`: a is [D, 1], tgt is [D, Y]."""
    shape = tuple(dims.shapes()[name])
    if name == "a":
        return shape + (1,)
    return shape[::-1] if name == "tgt" else shape


# ---- TrackableObjectGraph ---------------------------------------------------------------------------------------------
def new_node() -> dict:
    """A TrackableObject: children [(node_id, local_name)], attributes [(name, full_name, checkpoint_key,
    optional_restore)], slot_variables [(original_variable_node_id, slot_name, slot_variable_node_id)]."""
    return {"children": [], "attributes": [], "slot_variables": []}


def _pb_str(num: int, s: str) -> bytes:
    return _pb_bytes(num, s.encode()) if s else b""                     # proto3: an empty string is not written


def encode_object_graph(nodes: List[dict]) -> bytes:
    out = bytearray()
    for n in nodes:
        body = b"".join(_pb_bytes(1, _pb_varint(1, nid) + _pb_str(2, name)) for nid, name in n["children"])
        body += b"".join(_pb_bytes(2, _pb_str(1, a) + _pb_str(2, f) + _pb_str(3, k) + _pb_varint(4, int(o)))
                         for a, f, k, o in n["attributes"])
        body += b"".join(_pb_bytes(3, _pb_varint(1, o) + _pb_str(2, s) + _pb_varint(3, v))
                         for o, s, v in n["slot_variables"])
        out += _pb_bytes(1, body)
    return bytes(out)


def decode_object_graph(buf: bytes) -> List[dict]:
    def msg(b, fields):
        out = dict.fromkeys(fields.values())
        for num, wire, v in parse_fields(b):
            if num in fields:
                out[fields[num]] = v.decode() if wire == 2 else v
        return out
    nodes = []
    for num, wire, v in parse_fields(buf):
        if num != 1 or wire != 2:
            continue
        n = new_node()
        for n2, w2, v2 in parse_fields(v):
            if w2 != 2:
                continue
            if n2 == 1:
                r = msg(v2, {1: "id", 2: "name"})
                n["children"].append((r["id"] or 0, r["name"] or ""))
            elif n2 == 2:
                r = msg(v2, {1: "name", 2: "full", 3: "key", 4: "opt"})
                n["attributes"].append((r["name"] or "", r["full"] or "", r["key"] or "", bool(r["opt"])))
            elif n2 == 3:
                r = msg(v2, {1: "orig", 2: "slot", 3: "var"})
                n["slot_variables"].append((r["orig"] or 0, r["slot"] or "", r["var"] or 0))
        nodes.append(n)
    return nodes


# ---- DT_STRING tensors (tensor_bundle.cc's layout) ----------------------------------------------------------------------
def encode_strings(elements: List[bytes]) -> Tuple[bytes, int]:
    """(stored bytes, entry CRC-32C) of a DT_STRING tensor: the varint64 lengths, the masked CRC-32C of the lengths taken
    as raw little-endian uint64s, then the bytes.  The entry CRC runs over the raw uint64 lengths, the 4 checksum bytes
    and the element bytes, so it is not the CRC of the stored bytes."""
    raw_lens = b"".join(struct.pack("<Q", len(e)) for e in elements)
    check = struct.pack("<I", mask_crc(crc32c(raw_lens)))
    body = b"".join(elements)
    return b"".join(put_varint(len(e)) for e in elements) + check + body, crc32c(raw_lens + check + body)


def decode_strings(key: str, buf: bytes, n: int, entry_crc: int) -> List[bytes]:
    """The n elements of the stored DT_STRING tensor `buf`; ValueError if a checksum fails."""
    lens, pos = [], 0
    for _ in range(n):
        v, pos = get_varint(buf, pos)
        lens.append(v)
    raw_lens = b"".join(struct.pack("<Q", v) for v in lens)
    check = buf[pos:pos + 4]
    if len(check) < 4 or struct.unpack("<I", check)[0] != mask_crc(crc32c(raw_lens)):
        raise ValueError("checkpoint tensor %s: the CRC-32C of its string lengths does not match" % key)
    body = buf[pos + 4:]
    if len(body) != sum(lens):
        raise ValueError("checkpoint tensor %s holds %d string bytes; its lengths say %d" % (key, len(body), sum(lens)))
    got = crc32c(raw_lens + check + body)
    if got != entry_crc:
        raise ValueError("checkpoint tensor %s fails its CRC-32C: stored 0x%08x, computed 0x%08x" % (key, entry_crc, got))
    out, p = [], 0
    for v in lens:
        out.append(body[p:p + v])
        p += v
    return out


# ---- reading ----------------------------------------------------------------------------------------------------------
def _read_raw(e: dict) -> bytes:
    with open(e["file"], "rb") as f:
        f.seek(e["offset"])
        return f.read(e["size"])


def _scalar(prefix: str, index: dict, key: str, dtype: int):
    """The host value of the scalar `key` (float32 or int64), its CRC-32C checked."""
    if key not in index:
        raise ValueError("Keras checkpoint `%s` has no tensor %s" % (prefix, key))
    e = index[key]
    if e["dtype"] != dtype:
        raise ValueError("`%s`: tensor %s has dtype %d; it must be %d" % (prefix, key, e["dtype"], dtype))
    n = 8 if dtype == DT_INT64 else 4
    if tuple(e["shape"]) != () or e["size"] != n or e["offset"] + n > os.path.getsize(e["file"]):
        raise ValueError("checkpoint tensor %s: a scalar of %d bytes is expected, the entry has shape %s and %d bytes" % (
            key, n, list(e["shape"]), e["size"]))
    raw = _read_raw(e)
    if crc32c(raw) != unmask_crc(e["crc32c"]):
        raise ValueError("checkpoint tensor %s fails its CRC-32C: stored 0x%08x, computed 0x%08x" % (
            key, unmask_crc(e["crc32c"]), crc32c(raw)))
    return struct.unpack("<q" if dtype == DT_INT64 else "<f", raw)[0]


def _child(nodes: List[dict], nid: int, name: str) -> Optional[int]:
    for c, n in nodes[nid]["children"]:
        if n == name:
            return c
    return None


def _value_key(nodes: List[dict], nid: int) -> Optional[str]:
    for a, _, key, _ in nodes[nid]["attributes"]:
        if a == "VARIABLE_VALUE":
            return key
    return None


def _variables(nodes: List[dict], nid: int, path: str = ""):
    """(attribute path, node id, checkpoint key) of every variable below node nid."""
    seen, stack = set(), [(nid, path)]
    while stack:
        n, p = stack.pop()
        if n in seen or not 0 <= n < len(nodes):
            continue
        seen.add(n)
        key = _value_key(nodes, n)
        if key is not None and p:
            yield p, n, key
        for c, name in reversed(nodes[n]["children"]):
            stack.append((c, p + "/" + name if p else name))


def read_object_graph(prefix: str, index: dict) -> List[dict]:
    if OBJECT_GRAPH_KEY not in index:
        raise ValueError("Keras checkpoint `%s` has no tensor %s" % (prefix, OBJECT_GRAPH_KEY))
    e = index[OBJECT_GRAPH_KEY]
    if tuple(e["shape"]) != ():
        raise ValueError("checkpoint tensor %s has shape %s; a scalar is expected" % (OBJECT_GRAPH_KEY, list(e["shape"])))
    nodes = decode_object_graph(decode_strings(OBJECT_GRAPH_KEY, _read_raw(e), 1, unmask_crc(e["crc32c"]))[0])
    if not nodes:
        raise ValueError("Keras checkpoint `%s`: its object graph has no root" % prefix)
    return nodes


def keras_entries(prefix: str, dims: dict, with_optimizer: bool, adam: dict):
    """(entries, adam_t, save_counter) of the Keras checkpoint `prefix`, entries as tf_bundle.bundle_entries gives them
    ("name", "shape" (the engine's), "offset", "nbytes", "file", "crc", "key") plus "transposed" (tgt: the file holds
    [D, Y]).  The Adam slots come with `with_optimizer` when the checkpoint has an optimizer, and `adam` (lr, beta1,
    beta2) must then be its hyper-parameters with decay 0.  ValueError naming the key for anything missing, of another
    shape or dtype, or failing its CRC."""
    d = EngineDims(**dims)
    _, index = read_index(prefix, {OBJECT_GRAPH_KEY: DT_STRING, ITER_KEY: DT_INT64, SAVE_COUNTER_KEY: DT_INT64})
    nodes = read_object_graph(prefix, index)
    model = _child(nodes, 0, "model")
    model = 0 if model is None else model
    found = {}                                                        # engine name -> (node id, key)
    embeddings = []
    layer_ids = sorted((int(m.group(1)), c) for c, n in nodes[model]["children"]
                       for m in [re.fullmatch(r"layer_with_weights-(\d+)", n)] if m)
    for _, layer in layer_ids:
        for path, nid, key in _variables(nodes, layer):
            if key not in index:
                raise ValueError("the object graph of Keras checkpoint `%s` names tensor %s, which it does not hold" % (
                    prefix, key))
            for name, _, want_path in LAYERS:
                if path == want_path and name not in ("tok", "path"):
                    found.setdefault(name, (nid, key))
            if path == "embeddings":
                embeddings.append((nid, key))
    T, P = d.token_vocab, d.path_vocab
    if T == P:
        for name, item in zip(("path", "tok"), embeddings):
            found[name] = item
    else:
        for nid, key in embeddings:
            rows = index[key]["shape"][0] if index[key]["shape"] else None
            name = {T: "tok", P: "path"}.get(rows)
            if name is None:
                _check_entry(key, index[key], (T, d.embed_dim))               # raises: the shape fits neither table
            found.setdefault(name, (nid, key))
    for name, layer, path in LAYERS:
        if name not in found:
            raise ValueError("Keras checkpoint `%s` has no variable for %s (`%s` of shape %s under a layer_with_weights-N "
                             "node, the %s layer)" % (prefix, name, path, list(keras_shape(name, d)), layer))
    opt = _child(nodes, 0, "optimizer")
    if opt is None:
        opt = _child(nodes, model, "optimizer")
    slots = {}
    if opt is not None:
        for orig, slot, var in nodes[opt]["slot_variables"]:
            if 0 <= var < len(nodes):
                slots[(orig, slot)] = _value_key(nodes, var)
    with_optimizer = with_optimizer and opt is not None and bool(slots)
    out = []
    for group, slot in (("theta", None),) + (SLOTS if with_optimizer else ()):
        for name in PARAM_NAMES:
            nid, key = found[name]
            if slot is not None:
                key = slots.get((nid, slot))
                if key is None:
                    raise ValueError("Keras checkpoint `%s` has no Adam slot %s of %s" % (prefix, slot, found[name][1]))
            if key not in index:
                raise ValueError("Keras checkpoint `%s` has no tensor %s" % (prefix, key))
            e = index[key]
            _check_entry(key, e, keras_shape(name, d))
            out.append({"name": group + "/" + name, "shape": list(d.shapes()[name]), "offset": e["offset"],
                        "nbytes": e["size"], "file": e["file"], "crc": unmask_crc(e["crc32c"]), "key": key,
                        "transposed": name == "tgt"})
    adam_t = 0
    if with_optimizer:
        hyper = {}
        for h in HYPERS:
            c = _child(nodes, opt, h)
            key = _value_key(nodes, c) if c is not None else None
            if key is None:
                raise ValueError("Keras checkpoint `%s` has no optimizer variable %s" % (prefix, h))
            hyper[h] = _scalar(prefix, index, key, DT_INT64 if h == "iter" else DT_FLOAT), key
        for h, want in (("learning_rate", adam["lr"]), ("beta_1", adam["beta1"]), ("beta_2", adam["beta2"]),
                        ("decay", 0.0)):
            v, key = hyper[h]
            if np.float32(v) != np.float32(want):
                raise ValueError("Keras checkpoint `%s`: optimizer variable %s = %r, but this framework's Adam has %s = %r"
                                 % (prefix, key, v, h, float(np.float32(want))))
        adam_t, key = hyper["iter"]
        if adam_t < 0:
            raise ValueError("Keras checkpoint `%s`: optimizer variable %s = %d is negative" % (prefix, key, adam_t))
    c = _child(nodes, 0, "save_counter")
    key = _value_key(nodes, c) if c is not None else None
    save_counter = _scalar(prefix, index, key, DT_INT64) if key is not None else 0
    return out, int(adam_t), int(save_counter)


# ---- writing ----------------------------------------------------------------------------------------------------------
def keras_layout(dims: dict, entire: bool, with_optimizer: bool, adam_t: int, save_counter: int, adam: dict):
    """(tensors, scalars) of a Keras checkpoint written from a model with `dims`, back to back in key order in one data
    shard: tensors = [(key, "group/name", Keras shape, offset, nbytes)], scalars = [(key, dtype, shape, stored bytes,
    offset, entry CRC-32C)] (the object graph, the optimizer's variables, save_counter).  `entire`: the manager's
    checkpoint (root children model, optimizer, save_counter); else a save_weights file (the model is the root)."""
    d = EngineDims(**dims)
    nodes = [new_node()]

    def add(parent: Optional[int], name: str) -> int:
        nodes.append(new_node())
        if parent is not None:
            nodes[parent]["children"].append((len(nodes) - 1, name))
        return len(nodes) - 1
    model = add(0, "model") if entire else 0
    opt = add(0, "optimizer") if with_optimizer else None
    counter = add(0, "save_counter") if entire else None
    lead = "model/" if entire else ""
    tensors, scalars = [], []
    variables = []
    for i, (name, layer, path) in enumerate(LAYERS):
        nid = add(model, "layer_with_weights-%d" % i)
        for part in path.split("/"):
            nid = add(nid, part)
        key = "%slayer_with_weights-%d/%s" % (lead, i, path)
        full = "%s/%s" % (layer, path.split("/")[-1])
        nodes[nid]["attributes"].append(("VARIABLE_VALUE", full, key + VALUE, False))
        tensors.append((key + VALUE, "theta/" + name, keras_shape(name, d)))
        variables.append((name, nid, key, full))
    if with_optimizer:
        values = {"beta_1": adam["beta1"], "beta_2": adam["beta2"], "decay": 0.0, "learning_rate": adam["lr"]}
        for h in HYPERS:
            nid = add(opt, h)
            nodes[nid]["attributes"].append(("VARIABLE_VALUE", "Adam/" + h, "optimizer/%s%s" % (h, VALUE), False))
            raw = struct.pack("<q", int(adam_t)) if h == "iter" else np.float32(values[h]).tobytes()
            scalars.append(("optimizer/%s%s" % (h, VALUE), DT_INT64 if h == "iter" else DT_FLOAT, (), raw))
        for name, var, key, full in variables:
            for group, slot in SLOTS:
                sid = add(None, "")
                skey = "%s/.OPTIMIZER_SLOT/optimizer/%s%s" % (key, slot, VALUE)
                nodes[sid]["attributes"].append(("VARIABLE_VALUE", "Adam/%s/%s" % (full, slot), skey, False))
                nodes[opt]["slot_variables"].append((var, slot, sid))
                tensors.append((skey, group + "/" + name, keras_shape(name, d)))
    if entire:
        nodes[counter]["attributes"].append(("VARIABLE_VALUE", "save_counter", SAVE_COUNTER_KEY, False))
        scalars.append((SAVE_COUNTER_KEY, DT_INT64, (), struct.pack("<q", int(save_counter))))
    graph, graph_crc = encode_strings([encode_object_graph(nodes)])
    scalars = [(k, t, s, raw, crc32c(raw)) for k, t, s, raw in scalars] + [(OBJECT_GRAPH_KEY, DT_STRING, (), graph, graph_crc)]
    items = [(k, n, s) for k, n, s in tensors] + list(scalars)
    items.sort(key=lambda it: it[0].encode())
    out_t, out_s, off = [], [], 0
    for it in items:
        if len(it) == 3:
            n = 4 * int(np.prod(it[2], dtype=np.int64))
            out_t.append((it[0], it[1], it[2], off, n))
        else:
            n = len(it[3])
            out_s.append((it[0], it[1], it[2], it[3], off, it[4]))
        off += n
    return out_t, out_s


def write_keras_index(prefix: str, tensors, scalars, tensor_crcs) -> None:
    """<prefix>.index of keras_layout's (tensors, scalars), the tensors' plain CRC-32Cs in `tensor_crcs`."""
    items = [(k.encode(), encode_entry(shape, off, n, int(c))) for (k, _, shape, off, n), c in zip(tensors, tensor_crcs)]
    items += [(k.encode(), encode_entry(shape, off, len(raw), crc, dtype=dtype)) for k, dtype, shape, raw, off, crc in scalars]
    with open(prefix + INDEX_SUFFIX, "wb") as f:
        f.write(build_table([(b"", encode_header(1))] + sorted(items)))


# ---- the CheckpointManager's state file -------------------------------------------------------------------------------
_STATE_LINE = re.compile(r'^\s*(\w+)\s*:\s*(?:"((?:[^"\\]|\\.)*)"|([-+0-9.eE]+|inf|nan))\s*$')


def read_state(directory: str) -> dict:
    """The fields of `directory`/checkpoint (a CheckpointState text proto): model_checkpoint_path and
    all_model_checkpoint_paths joined to `directory` when relative, with all_model_checkpoint_timestamps and
    last_preserved_timestamp; {} when there is no state file."""
    path = os.path.join(directory, STATE_FILE)
    if not os.path.isfile(path):
        return {}
    state = {"all_model_checkpoint_paths": [], "all_model_checkpoint_timestamps": []}
    with open(path, encoding="utf-8") as f:
        for line in f:
            m = _STATE_LINE.match(line)
            if not m:
                continue
            field, text, number = m.groups()
            if text is not None:
                value = re.sub(r"\\(.)", r"\1", text)
                value = value if os.path.isabs(value) else os.path.join(directory, value)
            else:
                value = float(number)
            if field in ("all_model_checkpoint_paths", "all_model_checkpoint_timestamps"):
                state[field].append(value)
            else:
                state[field] = value
    return state


def latest_checkpoint(directory: str) -> Optional[str]:
    """tf.train.latest_checkpoint: the state file's model_checkpoint_path (a relative one joined to `directory`), or None
    when there is no state file, it names no checkpoint, or the checkpoint's .index is missing."""
    path = read_state(directory).get("model_checkpoint_path")
    if not path or not os.path.isfile(path + INDEX_SUFFIX):
        return None
    return path


def _quote(s: str) -> str:
    return '"%s"' % s.replace("\\", "\\\\").replace('"', '\\"')


def record_checkpoint(directory: str, prefix: str, max_to_keep: Optional[int], now: float) -> List[str]:
    """What CheckpointManager.save does after writing `prefix`: it becomes the latest checkpoint, the oldest kept ones
    beyond max_to_keep (None or 0: keep all) are deleted, and the state file lists the rest with relative paths.
    Returns the deleted prefixes."""
    state = read_state(directory)
    paths = list(state.get("all_model_checkpoint_paths", []))
    stamps = list(state.get("all_model_checkpoint_timestamps", []))
    stamps = (stamps + [now] * len(paths))[:len(paths)]
    kept = [(p, t) for p, t in zip(paths, stamps) if os.path.normpath(p) != os.path.normpath(prefix)] + [(prefix, now)]
    deleted = []
    while max_to_keep and len(kept) > max_to_keep:
        old, _ = kept.pop(0)
        for f in [old + INDEX_SUFFIX] + glob.glob(glob.escape(old) + ".data-?????-of-?????"):
            if os.path.isfile(f):
                os.remove(f)
        deleted.append(old)
    rel = lambda p: os.path.relpath(p, directory)
    lines = ["model_checkpoint_path: " + _quote(rel(prefix))]
    lines += ["all_model_checkpoint_paths: " + _quote(rel(p)) for p, _ in kept]
    lines += ["all_model_checkpoint_timestamps: " + repr(float(t)) for _, t in kept]
    lines.append("last_preserved_timestamp: " + repr(float(state.get("last_preserved_timestamp", kept[0][1]))))
    tmp = os.path.join(directory, STATE_FILE + ".tmp")
    with open(tmp, "w", encoding="utf-8") as f:
        f.write("\n".join(lines) + "\n")
    os.replace(tmp, os.path.join(directory, STATE_FILE))
    return deleted
