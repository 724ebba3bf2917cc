"""The reference Keras backend's checkpoints on the GPU: c2v_rows_to_cols / c2v_cols_to_rows against numpy bit for bit,
the streamed output-kernel CRC at java14m shape, and Code2VecModel saving and loading `__entire-model/ckpt-N` and
`__only-weights` against the host statement in tests/keras_ckpt_model.py.  The toy dataset is tests/test_gpu_model's."""
import glob
import os

import numpy as np
import pytest

from code2vec_b200 import keras_ckpt as K
from code2vec_b200 import tf_bundle as T
from tests import crc32c_model as M
from tests import keras_ckpt_model as KM
from tests.test_gpu_model import _config, _make_dataset

pytestmark = pytest.mark.gpu
TABLES = ("tok", "path", "tgt", "W", "a")


def _bits(shape, seed):
    """Random float32 bit patterns (NaNs with payloads among them), with -0.0, +inf and two NaN payloads planted."""
    rng = np.random.default_rng(seed)
    u = rng.integers(0, 2 ** 32, int(np.prod(shape)), dtype=np.uint64).astype(np.uint32)
    u[:: 7] = 0x80000000
    u[3:: 11] = 0x7FC00001
    u[5:: 13] = 0xFFBADBAD
    u[1:: 17] = 0x7F800000
    return u.reshape(shape).view(np.float32)


@pytest.mark.parametrize("k,Y,D,col0", [(1, 1, 4, 0), (7, 1025, 96, 89), (33, 100, 40, 5), (32, 31, 64, 32),
                                        (61, 261246, 384, 323)])
def test_transpose_kernels_bit_for_bit(k, Y, D, col0):
    import torch
    from code2vec_b200.engine import cols_to_rows, rows_to_cols
    rows = _bits((k, Y), 1)
    table = _bits((Y, D), 2)
    dev_rows = torch.from_numpy(rows.view(np.int32).copy()).cuda().view(torch.float32)
    dev_table = torch.from_numpy(table.view(np.int32).copy()).cuda().view(torch.float32)
    rows_to_cols(dev_rows, k, Y, dev_table, col0)
    want = table.view(np.uint32).copy()
    want[:, col0:col0 + k] = rows.view(np.uint32).T
    assert np.array_equal(dev_table.view(torch.int32).cpu().numpy().view(np.uint32), want)
    out = torch.from_numpy(np.full(k * Y + 5, -7, dtype=np.int32)).cuda()
    cols_to_rows(dev_table, col0, k, Y, out.view(torch.float32))
    got = out.cpu().numpy().view(np.uint32)
    assert np.array_equal(got[:k * Y], rows.view(np.uint32).reshape(-1)) and np.all(got[k * Y:] == 0xFFFFFFF9)


def test_transpose_refusals():
    from code2vec_b200.engine import load_library
    lib = load_library()
    assert lib.c2v_rows_to_cols(None, 0, 10, None, 4, 0, None) == 0
    assert lib.c2v_rows_to_cols(None, 3, 10, None, 4, 2, None) < 0
    assert b"ld >= col0 + k" in lib.c2v_last_error(None)
    assert lib.c2v_cols_to_rows(2, 4, 0, 1, 1, 8, None) < 0
    assert b"4-byte aligned" in lib.c2v_last_error(None)


# ---- the output kernel at java14m shape -------------------------------------------------------------------------------
JAVA_KERNEL = dict(token_vocab=1000, path_vocab=900, target_vocab=261246, embed_dim=128, code_dim=384, max_contexts=200,
                   max_batch=64, top_k=10)


def _model(engine, save_format, release=True):
    """A Code2VecModel around `engine` with only what its checkpoint methods use."""
    from code2vec_b200.b200_model import Code2VecModel

    class Cfg:
        RELEASE, MAX_TO_KEEP = release, 10
    m = Code2VecModel.__new__(Code2VecModel)
    m.engine, m.world, m.rank, m._save_format, m.config = engine, 1, 0, save_format, Cfg()
    return m


def test_java14m_target_kernel(tmp_path):
    """A [261,246, 384] target table built from four distinct Keras rows: the saved kernel's CRC is the host CRC-32C of
    the whole [384, 261,246] tensor, its load equals the .c2v_b200 load bit for bit, and one flipped byte is caught."""
    import torch
    from code2vec_b200.engine import EngineDims, PathAttentionEngine
    Y, D = 261246, 384
    rng = np.random.default_rng(3)
    pattern = _bits((4, Y), 4)
    order = rng.integers(0, 4, D)
    e = PathAttentionEngine(EngineDims(**JAVA_KERNEL), device=0, training=False)
    try:
        e.init_params()
        kernel = torch.from_numpy(pattern.view(np.int32)[order].copy()).cuda().view(torch.float32)     # [D, Y]
        e.params["tgt"].copy_(kernel.t())
        x = str(tmp_path / "m")
        _model(e, "keras")._save_inner_model(x)
        _model(e, "c2v_b200")._save_inner_model(x)
        want = [e.params[n].cpu().numpy().copy() for n in TABLES]
    finally:
        e.close()
    row_crc = [T.crc32c(p.tobytes()) for p in pattern]
    whole = M.combine_many([row_crc[o] for o in order], 4 * Y)
    _, index = T.read_index(x + "__only-weights", {K.OBJECT_GRAPH_KEY: K.DT_STRING})
    key = "layer_with_weights-4/kernel/.ATTRIBUTES/VARIABLE_VALUE"
    assert T.unmask_crc(index[key]["crc32c"]) == whole
    got = {}
    for tag, load in (("keras", lambda m: m._read_keras(x + "__only-weights")),
                      ("c2v", lambda m: m._read_checkpoint(x + ".c2v_b200"))):
        e = PathAttentionEngine(EngineDims(**JAVA_KERNEL), device=0, training=False)
        try:
            load(_model(e, "c2v_b200"))
            got[tag] = [e.params[n].cpu().numpy() for n in TABLES]
        finally:
            e.close()
    for n, a, b, w in zip(TABLES, got["keras"], got["c2v"], want):
        assert a.tobytes() == b.tobytes() == w.tobytes(), n
    at = index[key]["offset"] + 4 * Y * 200 + 12345
    with open(T.data_file(x + "__only-weights"), "r+b") as f:
        f.seek(at)
        b = f.read(1)
        f.seek(at)
        f.write(bytes([b[0] ^ 0x40]))
    e = PathAttentionEngine(EngineDims(**JAVA_KERNEL), device=0, training=False)
    try:
        with pytest.raises(ValueError, match=r"checkpoint tensor layer_with_weights-4/kernel/\.ATTRIBUTES/VARIABLE_VALUE "
                                             r"fails its CRC-32C: stored 0x%08x, computed 0x[0-9a-f]{8}" % whole):
            _model(e, "c2v_b200")._read_keras(x + "__only-weights")
    finally:
        e.close()


# ---- the model --------------------------------------------------------------------------------------------------------
def _keras_cfg(prefix, tmp_path, **kw):
    kw.setdefault("DL_FRAMEWORK", "b200-keras")
    return _config(prefix, tmp_path, **kw)


def _run(cfg, train=True):
    from code2vec_b200 import load_model_dynamically
    m = load_model_dynamically(cfg)
    lines = []
    m.log = lambda msg: lines.append(str(msg))
    try:
        if train:
            m.train()
        return m, lines
    except BaseException:
        m.close_session()
        raise


def _state(e):
    import torch
    torch.cuda.synchronize()
    s = {"adam_t": e.adam_t}
    for g, src in (("theta", e.params), ("adam_m", e.adam_m), ("adam_v", e.adam_v)):
        if src is not None:
            s.update({g + "/" + n: src[n].cpu().numpy().copy() for n in TABLES})
    return s


def _env(monkeypatch, tmp_path):
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    monkeypatch.setenv("C2V_SAVE_FORMAT", "keras")
    monkeypatch.setenv("C2V_DETERMINISTIC", "1")
    monkeypatch.setenv("C2V_SEED", "5")


def test_save_byte_identical_reload_and_rotation(tmp_path, monkeypatch):
    """train() saving every epoch with MAX_TO_KEEP = 2 keeps the last two checkpoints; the last one's bytes are the host
    statement's for the engine's state, and it loads back bit for bit with adam_t and the epochs trained."""
    _env(monkeypatch, tmp_path)
    prefix, _ = _make_dataset(tmp_path)
    x = str(tmp_path / "model" / "saved")
    m, _ = _run(_keras_cfg(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, MODEL_SAVE_PATH=x, NUM_TRAIN_EPOCHS=4,
                           SAVE_EVERY_EPOCHS=1, MAX_TO_KEEP=2))
    try:
        state = _state(m.engine)
    finally:
        m.close_session()
    d = x + "__entire-model"
    assert sorted(os.listdir(d)) == ["checkpoint", "ckpt-3.data-00000-of-00001", "ckpt-3.index",
                                     "ckpt-4.data-00000-of-00001", "ckpt-4.index"]
    assert open(os.path.join(d, "checkpoint")).read().splitlines()[:3] == [
        'model_checkpoint_path: "ckpt-4"', 'all_model_checkpoint_paths: "ckpt-3"', 'all_model_checkpoint_paths: "ckpt-4"']
    want = str(tmp_path / "want")
    KM.write_checkpoint(want, {k: v for k, v in state.items() if k != "adam_t"}, True, adam_t=state["adam_t"],
                        save_counter=4)
    for suffix in (".index", ".data-00000-of-00001"):
        assert open(os.path.join(d, "ckpt-4") + suffix, "rb").read() == open(want + suffix, "rb").read(), suffix
    m, _ = _run(_keras_cfg(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, MODEL_LOAD_PATH=x, NUM_TRAIN_EPOCHS=4),
                train=False)
    try:
        got = _state(m.engine)
        assert m.nr_epochs_trained == 4 and m._keras_save_counter == 4
    finally:
        m.close_session()
    assert got["adam_t"] == state["adam_t"] > 0
    for k, v in state.items():
        if k != "adam_t":
            assert got[k].tobytes() == v.tobytes(), k


def test_resume_equals_uninterrupted(tmp_path, monkeypatch):
    """2 epochs, a Keras checkpoint, 2 more epochs from it == 4 epochs in one run: losses, parameters and Adam slots.  The
    reader draws each batch at random from its pool and a resumed run starts a new reader, so the training file here
    repeats one example: every draw is the same batch, and the comparison sees only what the checkpoint carries.  Dropout
    is drawn from (seed, step), so it continues across the checkpoint."""
    _env(monkeypatch, tmp_path)
    prefix, _ = _make_dataset(tmp_path)
    first_line = open(prefix + ".train.c2v").readline()
    open(prefix + ".train.c2v", "w").write(first_line * 96)
    common = dict(TRAIN_DATA_PATH_PREFIX=prefix, DROPOUT_KEEP_RATE=0.75, SAVE_EVERY_EPOCHS=2)
    losses = lambda lines: [l for l in lines if l.startswith("Completed epoch")]
    whole, lw = _run(_keras_cfg(prefix, tmp_path, NUM_TRAIN_EPOCHS=4, **common))
    try:
        want = _state(whole.engine)
    finally:
        whole.close_session()
    x = str(tmp_path / "half" / "saved")
    first, l1 = _run(_keras_cfg(prefix, tmp_path, NUM_TRAIN_EPOCHS=2, MODEL_SAVE_PATH=x, **common))
    first.close_session()
    second, l2 = _run(_keras_cfg(prefix, tmp_path, NUM_TRAIN_EPOCHS=4, MODEL_LOAD_PATH=x, **common))
    try:
        got = _state(second.engine)
    finally:
        second.close_session()
    assert losses(l1) + losses(l2) == losses(lw) and len(losses(lw)) == 4
    assert got["adam_t"] == want["adam_t"]
    for k in want:
        if k != "adam_t":
            assert got[k].tobytes() == want[k].tobytes(), k


def test_release_evaluates_alike_and_refuses_training(tmp_path, monkeypatch):
    _env(monkeypatch, tmp_path)
    prefix, _ = _make_dataset(tmp_path)
    x = str(tmp_path / "model" / "saved")
    m, _ = _run(_keras_cfg(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, MODEL_SAVE_PATH=x, NUM_TRAIN_EPOCHS=3,
                           SAVE_EVERY_EPOCHS=3, TEST_DATA_PATH=prefix + ".test.c2v"))
    try:
        want = m.evaluate()
        m.config.RELEASE = True
        m._save_inner_model(x)
    finally:
        m.close_session()
    assert os.path.isfile(x + "__only-weights.index")
    _, index = T.read_index(x + "__only-weights", {K.OBJECT_GRAPH_KEY: K.DT_STRING})
    assert sorted(index) == sorted([K.OBJECT_GRAPH_KEY] + ["layer_with_weights-%d/%s/.ATTRIBUTES/VARIABLE_VALUE" % (
        i, "/".join(p)) for i, (_, _, p) in enumerate(KM.LAYERS)])
    import shutil
    shutil.rmtree(x + "__entire-model")
    m, _ = _run(_keras_cfg(prefix, tmp_path, MODEL_LOAD_PATH=x, TEST_DATA_PATH=prefix + ".test.c2v"), train=False)
    try:
        got = m.evaluate()
    finally:
        m.close_session()
    assert got == want
    with pytest.raises(ValueError) as ei:
        _run(_keras_cfg(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, MODEL_LOAD_PATH=x), train=False)
    assert str(ei.value) == ("There is no model at path `%s__entire-model`. When loading the model for further training, "
                             "we must use an entire saved model file (not just weights)." % x)


def test_command_line_evaluates_a_keras_model(tmp_path, monkeypatch):
    """Train and save in Keras format from the command line, then `--load X --test F` evaluates from the latest
    checkpoint: no .c2v_b200 file exists, so any other route would raise "There is no model"."""
    import tests.test_gpu_model as toy
    from code2vec_b200.__main__ import main
    monkeypatch.setattr(toy, "C", 200)                    # the default MAX_CONTEXTS: lines carry 200 context fields
    monkeypatch.setattr(toy, "TARGETS", toy.TARGETS + ["make|copy", "do|it", "read|all", "write|all", "open", "flush",
                                                       "hash|code"])           # more target words than the default top 10
    monkeypatch.setattr(toy, "TOKENS", ["tok%d" % i for i in range(64)])
    _env(monkeypatch, tmp_path)
    prefix, _ = _make_dataset(tmp_path)
    x = str(tmp_path / "cli" / "saved")
    assert main(["--data", prefix, "--save", x, "--framework", "b200-keras"]) == 0
    assert os.path.isfile(K.latest_checkpoint(x + "__entire-model") + ".index") and not glob.glob(x + "*.c2v_b200")
    monkeypatch.delenv("C2V_SAVE_FORMAT")
    assert main(["--framework", "b200-keras", "--load", x, "--test", prefix + ".test.c2v"]) == 0
