"""The reference Keras backend's checkpoints on the host (code2vec_b200/keras_ckpt.py): the object-graph codec, the
DT_STRING entry and its CRC, the reader on files tests/keras_ckpt_model.py writes byte by byte, the writer's layout and
index against those bytes, every refusal, which file --load reads, the state file and MAX_TO_KEEP rotation."""
import os

import numpy as np
import pytest

from code2vec_b200 import keras_ckpt as K
from code2vec_b200 import tf_bundle as T
from tests import crc32c_model as M
from tests import keras_ckpt_model as KM

DIMS = dict(token_vocab=7, path_vocab=5, target_vocab=6, embed_dim=4, code_dim=8, max_contexts=3, max_batch=2, top_k=2)
SAME = dict(DIMS, path_vocab=7)                                       # T = P: the two tables have the same shape
ADAM = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-7)
OPT = "model/layer_with_weights-%d/%s/.OPTIMIZER_SLOT/optimizer/%s/.ATTRIBUTES/VARIABLE_VALUE"


def _arrays(dims=DIMS, seed=0, optimizer=True):
    from code2vec_b200.engine import EngineDims
    rng = np.random.default_rng(seed)
    groups = ("theta", "adam_m", "adam_v") if optimizer else ("theta",)
    return {g + "/" + k: rng.standard_normal(s).astype(np.float32) for g in groups
            for k, s in EngineDims(**dims).shapes().items()}


def _write(tmp_path, dims=DIMS, entire=True, adam_t=11, name="ckpt-3", **kw):
    prefix = str(tmp_path / name)
    KM.write_checkpoint(prefix, _arrays(dims, optimizer=adam_t is not None), entire, adam_t=adam_t, save_counter=4, **kw)
    return prefix


# ---- object graph and DT_STRING ---------------------------------------------------------------------------------------
def test_object_graph_round_trip():
    nodes = [K.new_node() for _ in range(4)]
    nodes[0]["children"] = [(1, "model"), (0, "self"), (3, "")]
    nodes[1]["attributes"] = [("VARIABLE_VALUE", "x/y", "model/x/.ATTRIBUTES/VARIABLE_VALUE", True), ("a", "", "", False)]
    nodes[2]["slot_variables"] = [(1, "m", 3), (0, "v", 0)]
    assert K.decode_object_graph(K.encode_object_graph(nodes)) == nodes
    for entire, optimizer in ((True, True), (True, False), (False, False)):
        want, _ = KM.graph_nodes(entire, optimizer)
        got = K.decode_object_graph(KM.encode_graph(want))
        assert [(n["children"], n["attributes"], n["slot_variables"]) for n in got] == [tuple(n) for n in want]
        assert K.encode_object_graph(got) == KM.encode_graph(want)


def test_string_entry_crc_is_not_the_crc_of_the_stored_bytes():
    payload = bytes(range(256)) * 3
    stored, crc = K.encode_strings([payload])
    assert (stored, crc) == KM.string_scalar(payload)
    assert stored[:2] == b"\x80\x06" and stored[6:] == payload                       # varint(768), 4 check bytes
    assert crc != M.crc32c(stored)
    assert K.decode_strings("k", stored, 1, crc) == [payload]
    assert K.decode_strings("k", *K.encode_strings([b"ab", b"", b"cde"])[:1], 3,
                            K.encode_strings([b"ab", b"", b"cde"])[1]) == [b"ab", b"", b"cde"]
    with pytest.raises(ValueError, match="k fails its CRC-32C"):
        K.decode_strings("k", stored, 1, M.crc32c(stored))
    bad = bytearray(stored)
    bad[3] ^= 1
    with pytest.raises(ValueError, match="string lengths"):
        K.decode_strings("k", bytes(bad), 1, crc)


# ---- the reader -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dims", [DIMS, SAME], ids=["T!=P", "T=P"])
@pytest.mark.parametrize("entire", [True, False], ids=["entire", "weights"])
def test_reader_maps_every_variable_and_slot(tmp_path, dims, entire):
    prefix = _write(tmp_path, dims, entire=entire)
    arrays = _arrays(dims)
    entries, adam_t, counter = K.keras_entries(prefix, dims, True, ADAM)
    assert (adam_t, counter) == (11, 4 if entire else 0)
    assert [e["name"] for e in entries] == [g + "/" + n for g in ("theta", "adam_m", "adam_v")
                                            for n in ("tok", "path", "tgt", "W", "a")]
    lead = "model/" if entire else ""
    for e in entries:
        g, n = e["name"].split("/")
        raw = open(e["file"], "rb").read()[e["offset"]:e["offset"] + e["nbytes"]]
        assert raw == KM.keras_array(n, arrays[e["name"]]).tobytes(), e["name"]
        assert M.crc32c(raw) == e["crc"] and e["transposed"] == (n == "tgt")
        assert e["shape"] == list(arrays[e["name"]].shape)
        assert e["key"].startswith(lead + "layer_with_weights-%d/" % [l[0] for l in KM.LAYERS].index(n))
    assert entries[5]["key"] == lead + "layer_with_weights-1/embeddings/.OPTIMIZER_SLOT/optimizer/m/.ATTRIBUTES/VARIABLE_VALUE"
    theta, t0, _ = K.keras_entries(prefix, dims, False, ADAM)            # an inference engine: the weights alone
    assert len(theta) == 5 and t0 == 0


def test_weights_without_optimizer_load_with_zero_step(tmp_path):
    prefix = _write(tmp_path, entire=False, adam_t=None, name="X__only-weights")
    entries, adam_t, counter = K.keras_entries(prefix, DIMS, True, ADAM)
    assert len(entries) == 5 and adam_t == 0 and counter == 0


# ---- the writer -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("entire,optimizer", [(True, True), (True, False), (False, False)])
def test_writer_layout_and_index_equal_the_statement(tmp_path, entire, optimizer):
    arrays = _arrays(optimizer=optimizer)
    want = str(tmp_path / "want")
    KM.write_checkpoint(want, arrays, entire, adam_t=9 if optimizer else None, save_counter=2)
    got = str(tmp_path / "got")
    tensors, scalars = K.keras_layout(DIMS, entire, optimizer, 9, 2, ADAM)
    pieces = [(off, KM.keras_array(n.split("/")[1], arrays[n]).tobytes()) for _, n, _, off, _ in tensors]
    pieces += [(off, raw) for _, _, _, raw, off, _ in scalars]
    data = b"".join(p for _, p in sorted(pieces))
    open(T.data_file(got), "wb").write(data)
    crcs = [M.crc32c(KM.keras_array(n.split("/")[1], arrays[n]).tobytes()) for _, n, _, _, _ in tensors]
    K.write_keras_index(got, tensors, scalars, crcs)
    assert open(T.data_file(got), "rb").read() == open(T.data_file(want), "rb").read()
    assert open(got + ".index", "rb").read() == open(want + ".index", "rb").read()


# ---- refusals ---------------------------------------------------------------------------------------------------------
def _rewrite_index(prefix, edit):
    items = T.parse_table(open(prefix + ".index", "rb").read())
    open(prefix + ".index", "wb").write(T.build_table(edit(items)))


def test_refuses_missing_key(tmp_path):
    prefix = _write(tmp_path)
    key = OPT % (2, "layer/kernel", "v")
    _rewrite_index(prefix, lambda items: [(k, v) for k, v in items if k != key.encode()])
    with pytest.raises(ValueError, match="has no tensor %s" % key.replace(".", r"\.")):
        K.keras_entries(prefix, DIMS, True, ADAM)
    prefix = _write(tmp_path, name="b")
    key = "optimizer/iter/.ATTRIBUTES/VARIABLE_VALUE"
    _rewrite_index(prefix, lambda items: [(k, v) for k, v in items if k != key.encode()])
    with pytest.raises(ValueError, match="has no tensor optimizer/iter/"):
        K.keras_entries(prefix, DIMS, True, ADAM)
    K.keras_entries(prefix, DIMS, False, ADAM)                           # the weights alone are all there


def test_refuses_wrong_shape(tmp_path):
    prefix = _write(tmp_path)
    with pytest.raises(ValueError, match=r"model/layer_with_weights-4/kernel/\.ATTRIBUTES/VARIABLE_VALUE has shape "
                                         r"\[8, 6\]; the model needs \[9, 6\]"):
        K.keras_entries(prefix, dict(DIMS, code_dim=9), True, ADAM)
    with pytest.raises(ValueError, match=r"layer_with_weights-\d/embeddings/\.ATTRIBUTES/VARIABLE_VALUE has shape \[\d, 4\]; "
                                         r"the model needs \[8, 4\]"):
        K.keras_entries(prefix, dict(DIMS, token_vocab=8), True, ADAM)


def test_refuses_wrong_dtype(tmp_path):
    prefix = _write(tmp_path)
    key = b"model/layer_with_weights-4/kernel/.ATTRIBUTES/VARIABLE_VALUE"

    def edit(items):
        out = []
        for k, v in items:
            if k == key:
                e = T.decode_entry(v)
                v = T.encode_entry(e["shape"], e["offset"], e["size"], T.unmask_crc(e["crc32c"]), dtype=19)
            out.append((k, v))
        return out
    _rewrite_index(prefix, edit)
    with pytest.raises(ValueError, match="layer_with_weights-4/kernel/.ATTRIBUTES/VARIABLE_VALUE has dtype 19"):
        K.keras_entries(prefix, DIMS, True, ADAM)
    prefix = _write(tmp_path, name="b")
    key = b"optimizer/iter/.ATTRIBUTES/VARIABLE_VALUE"
    _rewrite_index(prefix, edit)
    with pytest.raises(ValueError, match="optimizer/iter/.ATTRIBUTES/VARIABLE_VALUE has dtype 19; it must be 9"):
        K.keras_entries(prefix, DIMS, True, ADAM)


@pytest.mark.parametrize("hyper,value", [("beta_1", 0.8), ("decay", 1e-4), ("learning_rate", 0.01), ("beta_2", 0.99)])
def test_refuses_other_adam_hyper_parameters(tmp_path, hyper, value):
    prefix = _write(tmp_path, hypers={hyper: value})
    with pytest.raises(ValueError, match="optimizer variable optimizer/%s/.ATTRIBUTES/VARIABLE_VALUE = %s" % (
            hyper, repr(float(np.float32(value)))[:6])):
        K.keras_entries(prefix, DIMS, True, ADAM)
    K.keras_entries(prefix, DIMS, False, ADAM)                           # not read without the optimizer


def test_refuses_graph_pointing_at_absent_key(tmp_path):
    key = "model/layer_with_weights-3/attention_param/.ATTRIBUTES/VARIABLE_VALUE"
    prefix = _write(tmp_path, rename={key: key.replace("attention_param", "attention_weight")})
    with pytest.raises(ValueError, match="names tensor model/layer_with_weights-3/attention_weight/"):
        K.keras_entries(prefix, DIMS, True, ADAM)


def test_refuses_corrupt_object_graph(tmp_path):
    prefix = _write(tmp_path)
    _, index = T.read_index(prefix, {K.OBJECT_GRAPH_KEY: K.DT_STRING, K.ITER_KEY: K.DT_INT64,
                                     K.SAVE_COUNTER_KEY: K.DT_INT64})
    at = index[K.OBJECT_GRAPH_KEY]["offset"] + 40
    with open(T.data_file(prefix), "r+b") as f:
        f.seek(at)
        b = f.read(1)
        f.seek(at)
        f.write(bytes([b[0] ^ 4]))
    with pytest.raises(ValueError, match="_CHECKPOINTABLE_OBJECT_GRAPH fails its CRC-32C"):
        K.keras_entries(prefix, DIMS, True, ADAM)


# ---- which file --load reads ------------------------------------------------------------------------------------------
class _Cfg:
    def __init__(self, path, training):
        self.MODEL_LOAD_PATH = path
        self.is_training = training


def _load(monkeypatch, path, training, world=1):
    from code2vec_b200.b200_keras_model import Code2VecModel
    calls = []
    m = Code2VecModel.__new__(Code2VecModel)
    m.config, m.world, m.rank, m.nr_epochs_trained = _Cfg(path, training), world, 0, 0
    monkeypatch.setattr(m, "_make_engine", lambda: None, raising=False)
    monkeypatch.setattr(m, "log", lambda msg: None, raising=False)
    monkeypatch.setattr(m, "_read_checkpoint", lambda p: calls.append(("c2v_b200", p)), raising=False)
    monkeypatch.setattr(m, "_read_bundle", lambda p: calls.append(("tf", p)), raising=False)
    monkeypatch.setattr(m, "_read_keras", lambda p: calls.append(("keras", p)), raising=False)
    try:
        m._load_inner_model()
    except ValueError as exc:
        return str(exc)
    return calls, m.nr_epochs_trained


MUST_ENTIRE = ("There is no model at path `{x}__entire-model`. When loading the model for further training, we must use "
               "an entire saved model file (not just weights).")
NO_LATEST = "Failed to load model: Model latest checkpoint is not found."


@pytest.mark.parametrize("c2v,index,weights,entire", [(a, b, c, d) for a in (0, 1) for b in (0, 1) for c in (0, 1)
                                                       for d in (0, 1, 2)])
@pytest.mark.parametrize("training", [False, True])
def test_selection_matrix(tmp_path, monkeypatch, c2v, index, weights, entire, training):
    """entire: 0 no directory, 1 a directory without a checkpoint, 2 a directory whose state file names ckpt-7."""
    x = str(tmp_path / "saved")
    if c2v:
        open(x + ".c2v_b200", "wb").close()
    if index:
        open(x + ".index", "wb").close()
    if weights:
        open(x + "__only-weights.index", "wb").close()
    if entire:
        os.makedirs(x + "__entire-model")
    if entire == 2:
        open(x + "__entire-model/ckpt-7.index", "wb").close()
        open(x + "__entire-model/checkpoint", "w").write('model_checkpoint_path: "ckpt-7"\n')
    got = _load(monkeypatch, x, training)
    if c2v:
        want = ([("c2v_b200", x + ".c2v_b200")], 0)
    elif index:
        want = ([("tf", x)], 0)
    elif not weights and not entire:
        want = ([("c2v_b200", x + ".c2v_b200")], 0)                     # which raises "There is no model"
    elif training and not entire:
        want = MUST_ENTIRE.format(x=x)
    elif weights and not training:
        want = ([("keras", x + "__only-weights")], 0)
    elif entire == 1:
        want = NO_LATEST
    else:
        want = ([("keras", x + "__entire-model/ckpt-7")], 7)
    assert got == want


def test_neither_keras_file_message(tmp_path, monkeypatch):
    from code2vec_b200.b200_model import Code2VecModel
    x = str(tmp_path / "saved")
    m = Code2VecModel.__new__(Code2VecModel)
    m.config, m.world = _Cfg(x, False), 1
    with pytest.raises(ValueError) as ei:
        m._load_keras(x)
    assert str(ei.value) == ("There is no entire model to load at path `{x}__entire-model`, and there is no model weights "
                             "file to load at path `{x}__only-weights`.".format(x=x))


@pytest.mark.parametrize("world", [2, 4, 8])
def test_keras_load_refused_on_ranks(tmp_path, monkeypatch, world):
    x = str(tmp_path / "saved")
    open(x + "__only-weights.index", "wb").close()
    msg = _load(monkeypatch, x, False, world=world)
    assert "Keras checkpoints are read by one GPU; convert it once in a single process" in msg


# ---- the state file and rotation --------------------------------------------------------------------------------------
def test_latest_checkpoint(tmp_path):
    d = str(tmp_path / "m__entire-model")
    os.makedirs(d)
    assert K.latest_checkpoint(d) is None                                # no state file
    open(os.path.join(d, "ckpt-2.index"), "wb").close()
    open(os.path.join(d, "checkpoint"), "w").write('model_checkpoint_path: "ckpt-2"\nall_model_checkpoint_paths: "ckpt-2"\n')
    assert K.latest_checkpoint(d) == os.path.join(d, "ckpt-2")
    other = str(tmp_path / "elsewhere")
    open(other + ".index", "wb").close()
    open(os.path.join(d, "checkpoint"), "w").write('model_checkpoint_path: "%s"\n' % other)
    assert K.latest_checkpoint(d) == other                               # an absolute path is taken as it is
    open(os.path.join(d, "checkpoint"), "w").write('model_checkpoint_path: "ckpt-5"\n')
    assert K.latest_checkpoint(d) is None                                # its .index is missing
    open(os.path.join(d, "checkpoint"), "w").write('all_model_checkpoint_paths: "ckpt-2"\n')
    assert K.latest_checkpoint(d) is None                                # no model_checkpoint_path


def test_rotation_keeps_the_last_two(tmp_path):
    d = str(tmp_path / "m__entire-model")
    os.makedirs(d)
    for n in range(1, 5):
        prefix = os.path.join(d, "ckpt-%d" % n)
        open(prefix + ".index", "wb").close()
        open(T.data_file(prefix), "wb").close()
        K.record_checkpoint(d, prefix, 2, 1000.0 + n)
    assert sorted(os.listdir(d)) == ["checkpoint", "ckpt-3.data-00000-of-00001", "ckpt-3.index",
                                     "ckpt-4.data-00000-of-00001", "ckpt-4.index"]
    lines = open(os.path.join(d, "checkpoint")).read().splitlines()
    assert lines[:3] == ['model_checkpoint_path: "ckpt-4"', 'all_model_checkpoint_paths: "ckpt-3"',
                         'all_model_checkpoint_paths: "ckpt-4"']
    assert lines[3:5] == ["all_model_checkpoint_timestamps: 1003.0", "all_model_checkpoint_timestamps: 1004.0"]
    assert K.latest_checkpoint(d) == os.path.join(d, "ckpt-4")
    K.record_checkpoint(d, os.path.join(d, "ckpt-3"), 2, 1005.0)         # saved again: it becomes the newest
    assert K.read_state(d)["all_model_checkpoint_paths"] == [os.path.join(d, "ckpt-4"), os.path.join(d, "ckpt-3")]


# ---- C2V_SAVE_FORMAT=keras --------------------------------------------------------------------------------------------
def test_save_format_flag():
    assert T.save_format_flag({"C2V_SAVE_FORMAT": "keras"}) == "keras"
    for bad in ("TF", "Keras", "h5"):
        with pytest.raises(ValueError, match="C2V_SAVE_FORMAT must be"):
            T.save_format_flag({"C2V_SAVE_FORMAT": bad})


@pytest.mark.parametrize("world", [2, 4, 8])
def test_keras_save_refused_on_ranks_before_any_engine(monkeypatch, world):
    from code2vec_b200 import b200_model as bm
    from code2vec_b200.multi_rank import check_multi_rank_run

    class Cfg:
        TRAIN_BATCH_SIZE, PREDICT, RELEASE, DL_FRAMEWORK = 8, False, False, "b200"
    with pytest.raises(ValueError, match="C2V_SAVE_FORMAT=keras: .* with C2V_SAVE_FORMAT=keras"):
        check_multi_rank_run(Cfg, world, "keras")
    monkeypatch.setenv("WORLD_SIZE", str(world))
    monkeypatch.setenv("C2V_SAVE_FORMAT", "keras")
    monkeypatch.setattr(bm.Code2VecModel, "_join_group", lambda self: pytest.fail("joined a process group"))
    with pytest.raises(ValueError, match="C2V_SAVE_FORMAT=keras"):
        bm.Code2VecModel(Cfg())
