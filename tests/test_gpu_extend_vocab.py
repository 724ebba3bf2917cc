"""C2V_EXTEND_VOCAB=1 on the GPU (DESIGN.md §6m): a model loaded from each checkpoint format and grown to the merged
vocabularies of a new dataset holds the checkpoint in its leading rows and a fresh model's initialisation in the new
ones; with nothing new it trains exactly as without the switch; it learns names the loaded vocabulary lacks; its first
step equals dense Adam; on 2 and 4 emulated ranks it loads and steps as one GPU; and what it saves loads back without
the switch.  The toy datasets are tests/test_gpu_model's: A, and B, which keeps four of A's method names and replaces
the other four, and the source tokens that decide them, by new ones."""
import os

import numpy as np
import pytest

from code2vec_b200 import tf_bundle as T
from tests import keras_ckpt_model as KM
from tests.test_gpu_model import _config, _make_dataset

pytestmark = pytest.mark.gpu
TABLES = ("tok", "path", "tgt", "W", "a")
NEW_TARGETS = ["fetch|data", "store|data", "parse|line", "emit|event"]
SCHEME = {"b200": "tensorflow", "b200-keras": "keras"}


def _datasets(tmp_path, monkeypatch, n_train_b=96):
    """(prefix of A, prefix of B, B's test lines)."""
    import tests.test_gpu_model as toy
    for d in ("a", "b"):
        (tmp_path / d).mkdir(exist_ok=True)
    a, _ = _make_dataset(tmp_path / "a")
    with monkeypatch.context() as m:
        m.setattr(toy, "TARGETS", toy.TARGETS[:4] + NEW_TARGETS)
        m.setattr(toy, "TOKENS", toy.TOKENS[:16] + ["new%d" % i for i in range(16)] + toy.TOKENS[32:])
        b, test_b = _make_dataset(tmp_path / "b", n_train=n_train_b, n_test=40, seed=1)
    return a, b, test_b


def _env(monkeypatch, tmp_path, **extra):
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    monkeypatch.setenv("C2V_DETERMINISTIC", "1")
    monkeypatch.setenv("C2V_SEED", "5")
    for k, v in extra.items():
        monkeypatch.setenv(k, v)


def _model(cfg):
    from code2vec_b200 import load_model_dynamically
    return load_model_dynamically(cfg)


def _state(e):
    import torch
    torch.cuda.synchronize()
    if e.adam_m is not None:
        e.sync_tables()
    s = {"adam_t": e.adam_t}
    for g, src in (("theta", e.params), ("adam_m", e.adam_m), ("adam_v", e.adam_v)):
        if src is not None:
            s.update({g + "/" + n: src[n].cpu().numpy().copy() for n in TABLES})
    return s


def _old_dims(tmp_path, a):
    """Writes A's vocabularies as old/dictionaries.bin; the EngineDims of a model with them."""
    from code2vec_b200.engine import EngineDims
    from code2vec_b200.vocabularies import Code2VecVocabs
    (tmp_path / "old").mkdir(exist_ok=True)
    cfg = _config(a, tmp_path, TRAIN_DATA_PATH_PREFIX=a)
    v = Code2VecVocabs(cfg)
    v.save(str(tmp_path / "old" / "dictionaries.bin"))
    return EngineDims(token_vocab=v.token_vocab.size, path_vocab=v.path_vocab.size, target_vocab=v.target_vocab.size,
                      embed_dim=cfg.TOKEN_EMBEDDINGS_SIZE, code_dim=cfg.CODE_VECTOR_SIZE, max_contexts=cfg.MAX_CONTEXTS,
                      max_batch=cfg.TRAIN_BATCH_SIZE, top_k=cfg.TOP_K_WORDS_CONSIDERED_DURING_PREDICTION)


def _arrays(dims, seed, optimizer=True):
    rng = np.random.default_rng(seed)
    out = {}
    for g in ("theta", "adam_m", "adam_v") if optimizer else ("theta",):
        for k, s in dims.shapes().items():
            a = (0.1 * rng.standard_normal(s)).astype(np.float32)
            out[g + "/" + k] = np.abs(a) * 1e-3 if g == "adam_v" else a
    return out


ADAM_T = 7


def _write_old(tmp_path, dims, fmt):
    """The old model at old/saved in format `fmt`: (load path, its arrays, whether they carry the optimizer)."""
    from code2vec_b200.keras_ckpt import record_checkpoint
    from code2vec_b200.multi_rank import checkpoint_header, write_checkpoint
    x = str(tmp_path / "old" / "saved")
    optimizer = fmt not in ("c2v_release", "keras_weights")
    arrays = _arrays(dims, 11, optimizer)
    if fmt in ("c2v", "c2v_release"):
        load = x + (".release" if fmt == "c2v_release" else "")
        prefix, entries, _ = checkpoint_header(vars(dims), ADAM_T, 0, optimizer)
        write_checkpoint(load + ".c2v_b200", prefix, [arrays[e["name"]] for e in entries])
        return load, arrays, optimizer
    if fmt == "tf":
        T.write_bundle_host(x, arrays, adam_t=ADAM_T)
        return x, arrays, optimizer
    # Keras: a training run reads the entire model; `keras_weights` is read into the grown engine by _read_keras itself
    directory = x + "__entire-model"
    os.makedirs(directory)
    entire = arrays if optimizer else _arrays(dims, 12)
    KM.write_checkpoint(os.path.join(directory, "ckpt-3"), entire, True, adam_t=ADAM_T, save_counter=3)
    record_checkpoint(directory, os.path.join(directory, "ckpt-3"), 10, 0.0)
    if fmt == "keras_weights":
        KM.write_checkpoint(x + "__only-weights", arrays, False)
    return x, arrays, optimizer


def _check_grown(m, arrays, optimizer, framework):
    """Old rows bit for bit the checkpoint's, new rows a fresh merged-size model's, new Adam rows zero, adam_t kept."""
    from code2vec_b200.engine import PathAttentionEngine
    from code2vec_b200.vocabularies import VocabType
    e = m.engine
    got = _state(e)
    old = m.vocabs.loaded_sizes
    assert old is not None
    grown = {"tok": e.dims.token_vocab, "path": e.dims.path_vocab, "tgt": e.dims.target_vocab}
    n_old = {"tok": old[VocabType.Token], "path": old[VocabType.Path], "tgt": old[VocabType.Target]}
    assert grown["tok"] > n_old["tok"] and grown["tgt"] == n_old["tgt"] + len(NEW_TARGETS)
    fresh = PathAttentionEngine(e.dims, device=0, training=False)
    try:
        fresh.init_params(scheme=SCHEME[framework])
        init = {n: fresh.params[n].cpu().numpy().copy() for n in TABLES}
    finally:
        fresh.close()
    assert got["adam_t"] == (ADAM_T if optimizer else 0)
    for n in TABLES:
        k = n_old.get(n, got["theta/" + n].shape[0])
        bits = lambda a: a.view(np.int32)
        assert np.array_equal(bits(got["theta/" + n][:k]), bits(arrays["theta/" + n])), n
        assert np.array_equal(bits(got["theta/" + n][k:]), bits(init[n][k:])), n
        for g in ("adam_m", "adam_v"):
            want = arrays[g + "/" + n] if optimizer else np.zeros_like(arrays["theta/" + n])
            assert np.array_equal(bits(got[g + "/" + n][:k]), bits(want)), (g, n)
            assert not got[g + "/" + n][k:].any(), (g, n)


@pytest.mark.parametrize("fmt, framework", [("c2v", "b200"), ("c2v", "b200-keras"), ("c2v_release", "b200"),
                                            ("tf", "b200"), ("tf", "b200-keras"), ("keras", "b200"),
                                            ("keras", "b200-keras"), ("keras_weights", "b200-keras")])
def test_each_load_format(tmp_path, monkeypatch, fmt, framework):
    _env(monkeypatch, tmp_path, C2V_EXTEND_VOCAB="1")
    a, b, _ = _datasets(tmp_path, monkeypatch)
    load, arrays, optimizer = _write_old(tmp_path, _old_dims(tmp_path, a), fmt)
    m = _model(_config(b, tmp_path, DL_FRAMEWORK=framework, MODEL_LOAD_PATH=load, TRAIN_DATA_PATH_PREFIX=b))
    try:
        if fmt == "keras_weights":                   # the same grown engine, re-initialised, reads the weights file
            m.engine.init_params(scheme=SCHEME[framework])
            for d in (m.engine.adam_m, m.engine.adam_v):
                for t in d.values():
                    t.zero_()
            m._read_keras(load + "__only-weights")
        _check_grown(m, arrays, optimizer, framework)
    finally:
        m.close_session()


def _train_logged(cfg):
    """train() of a new model for `cfg`: (losses of every step, final state)."""
    m = _model(cfg)
    losses, step = [], m.trainer.step_host

    def recording(*a, **k):
        losses.append(step(*a, **k))
        return losses[-1]
    m.trainer.step_host = recording
    try:
        m.train()
        return losses, _state(m.engine), m
    finally:
        m.close_session()


def test_nothing_new_equals_switch_off(tmp_path, monkeypatch):
    """Fine-tuning on the dataset the model was trained on: no word is new, and the run with the switch equals the run
    without it in every loss, parameter and Adam slot, and in the bytes it saves."""
    _env(monkeypatch, tmp_path, C2V_BATCH_RING="0")
    a, _, _ = _datasets(tmp_path, monkeypatch)
    old = str(tmp_path / "old" / "saved")
    _train_logged(_config(a, tmp_path, TRAIN_DATA_PATH_PREFIX=a, MODEL_SAVE_PATH=old, NUM_TRAIN_EPOCHS=4))
    out = {}
    for flag in ("0", "1"):
        monkeypatch.setenv("C2V_EXTEND_VOCAB", flag)
        save = str(tmp_path / ("ft" + flag) / "saved")
        losses, state, m = _train_logged(_config(a, tmp_path, TRAIN_DATA_PATH_PREFIX=a, MODEL_LOAD_PATH=old,
                                                 MODEL_SAVE_PATH=save, NUM_TRAIN_EPOCHS=3, DROPOUT_KEEP_RATE=0.75))
        assert (m.vocabs.loaded_sizes is not None) == (flag == "1")
        files = {f: open(os.path.join(os.path.dirname(save), f), "rb").read() for f in ("saved.c2v_b200", "dictionaries.bin")}
        out[flag] = (losses, state, files)
    (l0, s0, f0), (l1, s1, f1) = out["0"], out["1"]
    assert len(l0) == 9 and l1 == l0
    assert s1["adam_t"] == s0["adam_t"] == 12 + 9
    for k in s0:
        if k != "adam_t":
            assert s1[k].tobytes() == s0[k].tobytes(), k
    assert f1 == f0


def _count_rows(model, prefix):
    """Rows of one epoch of `prefix`.train.c2v that the training reader yields with the model's vocabularies."""
    import copy
    from code2vec_b200.b200_model import _TrainInputFormer
    from code2vec_b200.path_context_reader import EstimatorAction, PathContextReader
    cfg = copy.copy(model.config)
    cfg.NUM_TRAIN_EPOCHS = 1
    f = _TrainInputFormer()
    rd = PathContextReader(vocabs=model.vocabs, model_input_tensors_former=f, config=cfg,
                           estimator_action=EstimatorAction.Train, shuffle_seed=1)
    return sum(int(f.from_model_input_form(t).target_index.shape[0]) for t in rd.get_dataset())


def test_learns_new_names_and_round_trips(tmp_path, monkeypatch):
    """A model trained on A, fine-tuned on B: with the switch it trains on B's rows whose names A lacks and predicts
    those names on B's test file; without it those rows are dropped and those names cannot be predicted.  The
    fine-tuned model, saved and loaded back without the switch, has the merged vocabularies and evaluates alike."""
    _env(monkeypatch, tmp_path)
    a, b, test_b = _datasets(tmp_path, monkeypatch)
    old = str(tmp_path / "old" / "saved")
    _train_logged(_config(a, tmp_path, TRAIN_DATA_PATH_PREFIX=a, MODEL_SAVE_PATH=old, DROPOUT_KEEP_RATE=1.0))
    new_train = sum(1 for line in open(b + ".train.c2v") if line.split(" ")[0] in NEW_TARGETS)
    new_test = [line for line in test_b if line.split(" ")[0] in NEW_TARGETS]
    assert new_train > 20 and len(new_test) > 5
    results = {}
    for flag in ("0", "1"):
        monkeypatch.setenv("C2V_EXTEND_VOCAB", flag)
        save = str(tmp_path / ("ft" + flag) / "saved")
        m = _model(_config(b, tmp_path, TRAIN_DATA_PATH_PREFIX=b, MODEL_LOAD_PATH=old, MODEL_SAVE_PATH=save,
                           TEST_DATA_PATH=b + ".test.c2v", DROPOUT_KEEP_RATE=1.0))
        try:
            rows = _count_rows(m, b)
            m.train()
            res = m.evaluate()
            preds = m.predict(new_test)
            vocabs = m.vocabs
        finally:
            m.close_session()
        hits = sum(p.topk_predicted_words[0] == p.original_name for p in preds)
        results[flag] = (rows, res, hits, vocabs, save)
    (rows0, _, hits0, voc0, _), (rows1, res1, hits1, voc1, save1) = results["0"], results["1"]
    assert rows1 == 96 and rows0 == 96 - new_train                   # the switch-off run drops every new-name row
    assert not any(n in voc0.target_vocab.word_to_index for n in NEW_TARGETS) and hits0 == 0
    assert all(n in voc1.target_vocab.word_to_index for n in NEW_TARGETS)
    assert hits1 >= 0.6 * len(new_test), (hits1, len(new_test))
    # the round trip: dictionaries.bin holds the merged vocabularies, and evaluation is the fine-tuned model's
    monkeypatch.setenv("C2V_EXTEND_VOCAB", "0")
    m = _model(_config(b, tmp_path, MODEL_LOAD_PATH=save1, TEST_DATA_PATH=b + ".test.c2v"))
    try:
        for attr in ("token_vocab", "path_vocab", "target_vocab"):
            x, y = getattr(m.vocabs, attr), getattr(voc1, attr)
            assert (x.size, x.word_to_index, x.index_to_word) == (y.size, y.word_to_index, y.index_to_word), attr
        assert str(m.evaluate()) == str(res1)
    finally:
        m.close_session()


@pytest.mark.parametrize("math", [1, 2])
def test_first_step_after_growth_matches_dense(tmp_path, monkeypatch, math):
    """The grown model's first step, Trainer("single") with lazy embedding Adam, on a batch of B that touches new rows,
    equals the same step run densely (c2v_train_step + c2v_adam_step over every row) on a copy of the grown state."""
    import torch
    from code2vec_b200.b200_model import _TrainInputFormer
    from code2vec_b200.engine import PathAttentionEngine
    from code2vec_b200.path_context_reader import EstimatorAction, PathContextReader
    from code2vec_b200.vocabularies import VocabType
    _env(monkeypatch, tmp_path, C2V_EXTEND_VOCAB="1")
    monkeypatch.delenv("C2V_DETERMINISTIC")              # both engines with the default reduction order
    a, b, _ = _datasets(tmp_path, monkeypatch)
    load, _, _ = _write_old(tmp_path, _old_dims(tmp_path, a), "c2v")
    m = _model(_config(b, tmp_path, MODEL_LOAD_PATH=load, TRAIN_DATA_PATH_PREFIX=b, DROPOUT_KEEP_RATE=0.75))
    dense = None
    try:
        fast, tr = m.engine, m.trainer
        start = _state(fast)
        dense = PathAttentionEngine(fast.dims, device=0, training=True)
        for g, dst in (("theta", dense.params), ("adam_m", dense.adam_m), ("adam_v", dense.adam_v)):
            for n in TABLES:
                dst[n].copy_(torch.from_numpy(start[g + "/" + n]))
        dense.adam_t = fast.adam_t
        dense.set_option("adam_step_count", dense.adam_t)
        for e in (fast, dense):
            e.set_option("math_mode", math)
        f = _TrainInputFormer()
        rd = PathContextReader(vocabs=m.vocabs, model_input_tensors_former=f, config=m.config,
                               estimator_action=EstimatorAction.Train, shuffle_seed=3)
        t = f.from_model_input_form(next(iter(rd.get_dataset())))
        batch = (t.path_source_token_indices, t.path_indices, t.path_target_token_indices, t.context_valid_mask,
                 t.target_index)
        assert (np.asarray(t.target_index) >= m.vocabs.loaded_sizes[VocabType.Target]).any()
        assert (np.asarray(t.path_source_token_indices) >= m.vocabs.loaded_sizes[VocabType.Token]).any()
        dev = lambda e: [e.to_device(x, torch.float32 if i == 3 else torch.int32) for i, x in enumerate(batch)]
        step = fast.adam_t + 1
        la = float(tr.step_device(*dev(fast)).cpu()[0])
        lb = float(dense.train_step(*dev(dense), keep=tr.keep, seed=tr.seed, step=step).cpu()[0])
        dense.adam_step(t=step, **tr.adam)
        assert abs(la - lb) < 1e-5, (la, lb)
        got, want = _state(fast), _state(dense)
        assert got["adam_t"] == want["adam_t"] == ADAM_T + 1
        assert np.array_equal(got["theta/tgt"], want["theta/tgt"])
        for k in want:
            if k != "adam_t":
                assert np.abs(got[k] - want[k]).max() < 2e-6, k
    finally:
        if dense is not None:
            dense.close()
        m.close_session()


def test_device_reader_trains_the_grown_model_as_the_host_reader(tmp_path, monkeypatch):
    """train() of the grown model with C2V_DEVICE_READER=1 (the device vocabulary tables built from the merged
    vocabularies) logs the losses and saves the checkpoint of the host reader's run."""
    from tests.test_gpu_device_reader import _train_logged as train_logged
    _env(monkeypatch, tmp_path, C2V_EXTEND_VOCAB="1")
    a, b, _ = _datasets(tmp_path, monkeypatch, n_train_b=101)
    load, _, _ = _write_old(tmp_path, _old_dims(tmp_path, a), "c2v")
    out = {}
    for flag in ("0", "1"):
        save = str(tmp_path / ("reader" + flag) / "saved")
        make = lambda: _config(b, tmp_path, TRAIN_DATA_PATH_PREFIX=b, MODEL_LOAD_PATH=load, MODEL_SAVE_PATH=save,
                               NUM_TRAIN_EPOCHS=3, NUM_BATCHES_TO_LOG_PROGRESS=2, SHUFFLE_BUFFER_SIZE=40,
                               DROPOUT_KEEP_RATE=0.75)
        out[flag] = train_logged(monkeypatch, make, {"C2V_DEVICE_READER": flag, "C2V_EXTEND_VOCAB": "1"}, 1)
    (ckpt0, log0), (ckpt1, log1) = out["0"], out["1"]
    assert len(log0) >= 4 and log1 == log0
    assert ckpt1 == ckpt0


@pytest.mark.parametrize("world", [2, 4])
def test_emulated_ranks_load_and_step_as_one_gpu(tmp_path, monkeypatch, world):
    """On `world` emulated ranks the grown model's shards and target blocks are the one-GPU grown tensors' rows, and
    train()'s two steps equal the fully sharded Trainer stepping the reader's batches from the one-GPU grown state."""
    from tests.test_gpu_multi_rank_model import _drive, _models, _state as rank_state, _train_and_record
    from code2vec_b200.trainer import target_row_block
    _env(monkeypatch, tmp_path, C2V_EXTEND_VOCAB="1")
    a, b, _ = _datasets(tmp_path, monkeypatch, n_train_b=64)
    load, _, _ = _write_old(tmp_path, _old_dims(tmp_path, a), "c2v")
    make = lambda: _config(b, tmp_path, TRAIN_DATA_PATH_PREFIX=b, MODEL_LOAD_PATH=load, NUM_TRAIN_EPOCHS=1,
                           DROPOUT_KEEP_RATE=0.75)
    m = _model(make())
    try:
        one = _state(m.engine)
        Y = m.engine.dims.target_vocab
    finally:
        m.close_session()

    def action(model, r):
        loaded = rank_state(model.engine)
        return dict(_train_and_record(model, r), loaded=loaded)
    got = _models(monkeypatch, world, make, action, {"C2V_EXTEND_VOCAB": "1"})
    for r in range(world):
        y0, y1 = target_row_block(Y, r, world)
        for k, v in got[r]["loaded"].items():
            if k == "adam_t":
                assert v == one[k] == ADAM_T
                continue
            n = k.split("/")[1]
            want = one[k][r::world] if n in ("tok", "path") else one[k][y0:y1] if n == "tgt" else one[k]
            assert np.array_equal(v[:want.shape[0]].view(np.int32), want.view(np.int32)), (r, k)
    batches = got[0]["batches"]
    assert [len(x[4]) for x in batches] == [32, 32]
    losses, states = _drive(monkeypatch, world, got[0]["dims"], 32 // world, batches, keep=0.75, start=one)
    for r in range(world):
        assert got[r]["losses"] == losses[r] == losses[0], r
        for k, v in states[r].items():
            if k == "adam_t":
                assert got[r]["state"][k] == v == ADAM_T + 2
                continue
            n = k.split("/")[1]
            rows = {"tok": one["theta/tok"].shape[0], "path": one["theta/path"].shape[0]}.get(n)
            real = -(-(rows - r) // world) if rows else v.shape[0]      # the shard's rows below the table's end
            assert np.array_equal(got[r]["state"][k][:real].view(np.int32), v[:real].view(np.int32)), (r, k)
