"""A plain statement of the reference Keras backend's checkpoint files (code2vec_b200/keras_ckpt.py, DESIGN.md §6l),
written byte by byte from the definitions with numpy and crc32c_model: the TrackableObjectGraph proto, tensor_bundle.cc's
DT_STRING layout, BundleHeaderProto / BundleEntryProto, and a LevelDB table of one data block (restart interval 16), an
empty metaindex block, an index block keyed by the last key, and the 48-byte footer.

Object graph node numbering (the writer's): 0 the root; in a manager checkpoint 1 `model`, then `optimizer` (with Adam),
then `save_counter`; then per layer in creation order (path_embedding, token_embedding, time_distributed, attention,
target_index) its `layer_with_weights-i` node and the nodes of its attribute path; then the optimizer's variables in
name order; then each variable's m and v slot nodes."""
import struct

import numpy as np

from tests import crc32c_model as M

VALUE = "/.ATTRIBUTES/VARIABLE_VALUE"
LAYERS = [("path", "path_embedding", ["embeddings"]), ("tok", "token_embedding", ["embeddings"]),
          ("W", "time_distributed", ["layer", "kernel"]), ("a", "attention", ["attention_param"]),
          ("tgt", "target_index", ["kernel"])]
DT_FLOAT, DT_STRING, DT_INT64 = 1, 7, 9


def varint(n: int) -> bytes:
    out = b""
    while n >= 0x80:
        out += bytes([(n & 0x7F) | 0x80])
        n >>= 7
    return out + bytes([n])


def pb_int(num, v):
    return varint(num << 3) + varint(v) if v else b""


def pb_len(num, payload):
    return varint(num << 3 | 2) + varint(len(payload)) + payload


def pb_str(num, s):
    return pb_len(num, s.encode()) if s else b""


def graph_nodes(entire: bool, optimizer: bool):
    """[(children, attributes, slot_variables)] in the numbering above, and {key: engine group/name}."""
    nodes = [[[], [], []]]

    def add(parent, name):
        nodes.append([[], [], []])
        if parent is not None:
            nodes[parent][0].append((len(nodes) - 1, name))
        return len(nodes) - 1
    model = add(0, "model") if entire else 0
    opt = add(0, "optimizer") if optimizer else None
    counter = add(0, "save_counter") if entire else None
    lead = "model/" if entire else ""
    keys, variables = {}, []
    for i, (name, layer, path) in enumerate(LAYERS):
        nid = add(model, "layer_with_weights-%d" % i)
        for part in path:
            nid = add(nid, part)
        key = "%slayer_with_weights-%d/%s" % (lead, i, "/".join(path))
        full = layer + "/" + path[-1]
        nodes[nid][1].append(("VARIABLE_VALUE", full, key + VALUE, False))
        keys[key + VALUE] = "theta/" + name
        variables.append((name, nid, key, full))
    if optimizer:
        for h in ("beta_1", "beta_2", "decay", "iter", "learning_rate"):
            nid = add(opt, h)
            nodes[nid][1].append(("VARIABLE_VALUE", "Adam/" + h, "optimizer/" + h + VALUE, False))
        for name, nid, key, full in variables:
            for group, slot in (("adam_m", "m"), ("adam_v", "v")):
                sid = add(None, "")
                skey = key + "/.OPTIMIZER_SLOT/optimizer/" + slot + VALUE
                nodes[sid][1].append(("VARIABLE_VALUE", "Adam/%s/%s" % (full, slot), skey, False))
                nodes[opt][2].append((nid, slot, sid))
                keys[skey] = group + "/" + name
    if entire:
        nodes[counter][1].append(("VARIABLE_VALUE", "save_counter", "save_counter" + VALUE, False))
    return nodes, keys


def encode_graph(nodes) -> bytes:
    out = b""
    for children, attrs, slots in nodes:
        body = b"".join(pb_len(1, pb_int(1, c) + pb_str(2, n)) for c, n in children)
        body += b"".join(pb_len(2, pb_str(1, a) + pb_str(2, f) + pb_str(3, k) + pb_int(4, int(o))) for a, f, k, o in attrs)
        body += b"".join(pb_len(3, pb_int(1, o) + pb_str(2, s) + pb_int(3, v)) for o, s, v in slots)
        out += pb_len(1, body)
    return out


def string_scalar(payload: bytes):
    """(stored bytes, entry CRC) of a one-element DT_STRING tensor."""
    raw_len = struct.pack("<Q", len(payload))
    check = struct.pack("<I", M.mask(M.crc32c(raw_len)))
    return varint(len(payload)) + check + payload, M.crc32c(raw_len + check + payload)


def entry(dtype, shape, offset, size, crc) -> bytes:
    dims = b"".join(pb_len(2, pb_int(1, s)) for s in shape)
    return pb_int(1, dtype) + pb_len(2, dims) + pb_int(4, offset) + pb_int(5, size) + b"\x35" + struct.pack("<I", M.mask(crc))


def block(items) -> bytes:
    out, restarts, last = b"", [0], b""
    for i, (k, v) in enumerate(items):
        shared = 0
        if i % 16 == 0:
            if i:
                restarts.append(len(out))
        else:
            while shared < min(len(k), len(last)) and k[shared] == last[shared]:
                shared += 1
        out += varint(shared) + varint(len(k) - shared) + varint(len(v)) + k[shared:] + v
        last = k
    return out + b"".join(struct.pack("<I", r) for r in restarts) + struct.pack("<I", len(restarts))


def table(items) -> bytes:
    out = b""
    handles = []
    for contents in (block(items), block([])):
        handles.append(varint(len(out)) + varint(len(contents)))
        out += contents + b"\x00" + struct.pack("<I", M.mask(M.crc32c(contents + b"\x00")))
    index = block([(items[-1][0], handles[0])])
    handles.append(varint(len(out)) + varint(len(index)))
    out += index + b"\x00" + struct.pack("<I", M.mask(M.crc32c(index + b"\x00")))
    footer = handles[1] + handles[2]
    return out + footer + bytes(40 - len(footer)) + struct.pack("<Q", 0xdb4775248b80fb57)


def keras_array(name: str, a: np.ndarray) -> np.ndarray:
    """An engine tensor in its Keras layout: a as [D, 1], tgt transposed to [D, Y]."""
    a = np.asarray(a, dtype="<f4")
    return a.reshape(-1, 1) if name == "a" else (np.ascontiguousarray(a.T) if name == "tgt" else a)


def write_checkpoint(prefix: str, arrays: dict, entire: bool, adam_t=None, save_counter: int = 1,
                     hypers=None, rename=None) -> None:
    """<prefix>.index and <prefix>.data-00000-of-00001 from host arrays in the engine's layout ({"theta/tok": ...,
    "adam_m/tgt": ...}).  adam_t: with the optimizer (its slots from arrays) at that step.  hypers overrides the
    optimizer's float variables (lr 1e-3, betas 0.9 / 0.999, decay 0); rename maps keys the object graph names to other
    keys (the data keeps the true ones)."""
    nodes, keys = graph_nodes(entire, adam_t is not None)
    graph_nodes_out = [[c, [(a, f, (rename or {}).get(k, k), o) for a, f, k, o in at], s] for c, at, s in nodes]
    tensors = {k: (DT_FLOAT, keras_array(n.split("/")[1], arrays[n])) for k, n in keys.items()}
    scalars = {}
    if adam_t is not None:
        h = dict(dict(beta_1=0.9, beta_2=0.999, decay=0.0, learning_rate=1e-3), **(hypers or {}))
        for name, v in h.items():
            raw = np.float32(v).tobytes()
            scalars["optimizer/" + name + VALUE] = (DT_FLOAT, raw, M.crc32c(raw))
        raw = struct.pack("<q", adam_t)
        scalars["optimizer/iter" + VALUE] = (DT_INT64, raw, M.crc32c(raw))
    if entire:
        raw = struct.pack("<q", save_counter)
        scalars["save_counter" + VALUE] = (DT_INT64, raw, M.crc32c(raw))
    raw, crc = string_scalar(encode_graph(graph_nodes_out))
    scalars["_CHECKPOINTABLE_OBJECT_GRAPH"] = (DT_STRING, raw, crc)
    data, items = b"", [(b"", pb_int(1, 1) + pb_len(3, pb_int(1, 1)))]
    for key in sorted(list(tensors) + list(scalars), key=str.encode):
        if key in tensors:
            dtype, a = tensors[key]
            raw, shape = a.tobytes(), a.shape
            crc = M.crc32c(raw)
        else:
            dtype, raw, crc = scalars[key]
            shape = ()
        items.append((key.encode(), entry(dtype, shape, len(data), len(raw), crc)))
        data += raw
    with open(prefix + ".data-00000-of-00001", "wb") as f:
        f.write(data)
    with open(prefix + ".index", "wb") as f:
        f.write(table(items))
