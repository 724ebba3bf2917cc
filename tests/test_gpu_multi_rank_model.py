"""Code2VecModel on 2 and 4 ranks emulated on one GPU (tests/emulated_ranks.py): train(), save / load, evaluate() and the
embedding exports through the fully sharded schedule, against a fully sharded Trainer driven by hand on the same global
batches and against the one-GPU model.  Each rank is a thread with its own Code2VecModel; make_fully_sharded_engine is
wrapped so that every rank's engine library shares one IpcProxy handle table.  The toy dataset is tests/test_gpu_model's."""
import os

import numpy as np
import pytest

from tests.emulated_ranks import EmulatedGroup, IpcProxy, emulate_ipc, run_ranks
from tests.test_gpu_model import _config, _make_dataset

pytestmark = pytest.mark.gpu

SEED = "5"
TABLES = ("tok", "path", "tgt", "W", "a")


@pytest.fixture(autouse=True)
def _ten_target_rows(monkeypatch):
    """The toy dataset with a ninth method name: 10 target rows (OOV included), in blocks of 5 on 2 ranks and 3, 3, 3, 1
    on 4.  With 9 rows the fourth rank would hold none, which make_fully_sharded_engine refuses."""
    import tests.test_gpu_model as toy
    monkeypatch.setattr(toy, "TARGETS", toy.TARGETS + ["make|copy"])


def _on_ranks(monkeypatch, world, fn, env=None):
    """[fn(rank) for every rank] on `world` emulated ranks, with WORLD_SIZE=world and the other variables of `env`."""
    import torch
    import code2vec_b200.b200_model as bm
    from code2vec_b200.trainer import make_fully_sharded_engine
    out = [None] * world
    table = {}

    def make(*a, **k):
        e = make_fully_sharded_engine(*a, **k)
        e.lib = IpcProxy(e.lib, table)
        return e

    with monkeypatch.context() as m:
        group = EmulatedGroup(world).install(m)
        m.setattr(bm, "make_fully_sharded_engine", make)
        m.setenv("WORLD_SIZE", str(world))
        for k, v in (env or {}).items():
            m.setenv(k, v)

        def body(r):
            torch.cuda.set_device(0)
            out[r] = fn(r)
        run_ranks(world, body, group)
    return out


def _models(monkeypatch, world, make_cfg, action, env=None):
    """action(model, rank) on a Code2VecModel per emulated rank (closed afterwards)."""
    from code2vec_b200.b200_model import Code2VecModel

    def fn(r):
        model = Code2VecModel(make_cfg())
        try:
            return action(model, r)
        finally:
            model.close_session()
    return _on_ranks(monkeypatch, world, fn, dict({"C2V_DETERMINISTIC": "1", "C2V_SEED": SEED}, **(env or {})))


def _state(e):
    """Every tensor a fully sharded rank holds: shards, target block, W, a and their Adam slots, and the step."""
    import torch
    torch.cuda.synchronize()
    s = {"adam_t": e.adam_t}
    for g, shard, rest in (("theta", e.shard_params, e.params), ("adam_m", e.shard_m, e.adam_m),
                           ("adam_v", e.shard_v, e.adam_v)):
        for n in TABLES:
            s[g + "/" + n] = (shard if n in ("tok", "path") else rest)[n].cpu().numpy().copy()
    return s


def _load_state(e, full, r, world):
    """Put a whole model (the arrays of a checkpoint) into rank r's tensors."""
    import torch
    y0, y1 = e.target_row0, e.target_row0 + e.dims.target_vocab
    for g, shard, rest in (("theta", e.shard_params, e.params), ("adam_m", e.shard_m, e.adam_m),
                           ("adam_v", e.shard_v, e.adam_v)):
        for n in TABLES:
            a = full[g + "/" + n]
            a = a[r::world] if n in ("tok", "path") else a[y0:y1] if n == "tgt" else a
            dst = shard[n] if n in ("tok", "path") else rest[n]
            dst[:a.shape[0]].copy_(torch.from_numpy(np.ascontiguousarray(a)))
    e.adam_t = int(full["adam_t"])
    e.set_option("adam_step_count", e.adam_t)


def _read_whole(path):
    from code2vec_b200.multi_rank import read_checkpoint_header
    meta, base = read_checkpoint_header(path)
    full = {"adam_t": meta["adam_t"]}
    for ent in meta["tensors"]:
        full[ent["name"]] = np.fromfile(path, dtype="<f4", count=ent["nbytes"] // 4,
                                        offset=base + ent["offset"]).reshape(ent["shape"])
    return full


def _reader_batches(model):
    """The global batches train() draws: the training reader with the run's shuffle seed."""
    from code2vec_b200.b200_model import _TrainInputFormer
    from code2vec_b200.path_context_reader import EstimatorAction, PathContextReader
    f = _TrainInputFormer()
    rd = PathContextReader(vocabs=model.vocabs, model_input_tensors_former=f, config=model.config,
                           estimator_action=EstimatorAction.Train, shuffle_seed=model._seed)
    return [tuple(np.array(a) for a in (t.path_source_token_indices, t.path_indices, t.path_target_token_indices,
                                         t.context_valid_mask, t.target_index))
            for t in map(f.from_model_input_form, rd.get_dataset())]


def _drive(monkeypatch, world, dims, local_batch, batches, keep, start=None):
    """A fully sharded Trainer per emulated rank stepping on `batches` split by hand (rank r: rows [r*b, (r+1)*b) with
    b = rows // world), from the model's initialisation or from the whole model `start`.  ([losses], [states])."""
    import torch
    import torch.distributed as dist
    from code2vec_b200.engine import EngineDims
    from code2vec_b200.trainer import Trainer, make_fully_sharded_engine
    losses, states, engines = [[] for _ in range(world)], [None] * world, []
    with monkeypatch.context() as m:
        group = EmulatedGroup(world).install(m)
        try:
            for r in range(world):
                with group.as_rank(r):
                    e = make_fully_sharded_engine(EngineDims(**dims), local_batch, device=0)
                if start is None:
                    e.init_params(whole_target_table=True)
                engines.append(e)
            emulate_ipc(engines)

            def body(r):
                torch.cuda.set_device(0)
                e = engines[r]
                tr = Trainer(e, keep_prob=keep, seed=int(SEED), schedule="fully_sharded", deterministic=True,
                             ordered_exchange=True)
                if start is not None:
                    _load_state(e, start, r, world)
                    # the first step gathers embedding rows from the peers' shards: every rank's load must have landed
                    torch.cuda.synchronize()
                    dist.barrier()
                e.set_option("math_mode", 1)
                for batch in batches:
                    b = len(batch[4]) // world           # the split stated independently of multi_rank.batch_split
                    if b:
                        losses[r].append(tr.step_host(*(a[r * b:(r + 1) * b] for a in batch)))
                states[r] = _state(e)
            run_ranks(world, body, group)
        finally:
            torch.cuda.synchronize()
            for e in engines:
                e.close()
    return losses, states


def _assert_states_equal(got, want, label):
    for r, (g, w) in enumerate(zip(got, want)):
        assert g["adam_t"] == w["adam_t"], (label, r)
        for k in w:
            if k != "adam_t":
                assert np.array_equal(g[k].view(np.int32), w[k].view(np.int32)), (label, r, k)


def _train_and_record(model, r):
    """train() on one rank; the losses its steps returned, its state, its dims, and (rank 0) the reader's batches."""
    batches = _reader_batches(model) if r == 0 else None
    losses, step = [], model.trainer.step_host

    def recording(*a, **k):
        losses.append(step(*a, **k))
        return losses[-1]
    model.trainer.step_host = recording
    model.train()
    return dict(losses=losses, state=_state(model.engine), dims=vars(model._engine_dims()), batches=batches)


# ---- 1. training learns, and repeats byte for byte ------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 4])
def test_train_learns_and_repeats(tmp_path, monkeypatch, world):
    monkeypatch.chdir(tmp_path)
    prefix, _ = _make_dataset(tmp_path)
    saves = [str(tmp_path / ("run%d" % i) / "saved") for i in range(2)]
    results = []
    for save in saves:
        def action(model, r):
            model.train()
            return model.evaluate()
        make = lambda: _config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, MODEL_SAVE_PATH=save,
                               TEST_DATA_PATH=prefix + ".test.c2v", DROPOUT_KEEP_RATE=1.0)
        results.append(_models(monkeypatch, world, make, action))
    res = results[0][0]
    assert res.topk_acc[0] > 0.6 and res.topk_acc[-1] >= res.topk_acc[0]      # the toy rule is learnt
    assert all(str(x) == str(res) for run in results for x in run)          # every rank returns rank 0's results
    a, b = (open(s + ".c2v_b200", "rb").read() for s in saves)
    assert a == b
    assert os.path.exists(str(tmp_path / "run0" / "dictionaries.bin"))
    assert not [f for f in os.listdir(str(tmp_path / "run0")) if f.endswith(".tmp")]


# ---- 2, 3. the model feeds exactly the hand-split global batches, short last batch included --------------------------
@pytest.mark.parametrize("n_train", [32, 39])            # one full batch; a full batch and a short one of 7 rows
@pytest.mark.parametrize("world", [2, 4])
def test_steps_match_trainer_on_hand_split_batches(tmp_path, monkeypatch, world, n_train):
    monkeypatch.chdir(tmp_path)
    prefix, _ = _make_dataset(tmp_path, n_train=n_train)
    make = lambda: _config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, NUM_TRAIN_EPOCHS=1, DROPOUT_KEEP_RATE=0.75)
    got = _models(monkeypatch, world, make, _train_and_record)
    batches = got[0]["batches"]
    assert [len(b[4]) for b in batches] == ([32] if n_train == 32 else [32, 7])
    losses, states = _drive(monkeypatch, world, got[0]["dims"], 32 // world, batches, keep=0.75)
    assert len(got[0]["losses"]) == len(batches)
    for r in range(world):
        assert got[r]["losses"] == losses[r] == losses[0], r          # the global mean, bit for bit, on every rank
    _assert_states_equal([g["state"] for g in got], states, "world=%d n_train=%d" % (world, n_train))


# ---- 4. resume: two steps, save, load, two more == four steps ----------------------------------------------------------
@pytest.mark.parametrize("world", [2, 4])
def test_resume_continues_exactly(tmp_path, monkeypatch, world):
    monkeypatch.chdir(tmp_path)
    prefix, _ = _make_dataset(tmp_path, n_train=64)
    first, second = str(tmp_path / "a" / "saved"), str(tmp_path / "b" / "saved")
    make1 = lambda: _config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, NUM_TRAIN_EPOCHS=1, MODEL_SAVE_PATH=first)
    got1 = _models(monkeypatch, world, make1, _train_and_record)
    make2 = lambda: _config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, NUM_TRAIN_EPOCHS=1, MODEL_LOAD_PATH=first,
                            MODEL_SAVE_PATH=second)
    got2 = _models(monkeypatch, world, make2, _train_and_record)
    batches = got1[0]["batches"]
    assert len(batches) == 2          # the resumed run reads the same two batches again (same file, same shuffle seed)
    assert all(np.array_equal(a, b) for x, y in zip(batches, got2[0]["batches"]) for a, b in zip(x, y))
    _, four = _drive(monkeypatch, world, got1[0]["dims"], 32 // world, batches + batches, keep=0.75)
    _assert_states_equal([g["state"] for g in got2], four, "resumed world=%d" % world)
    assert all(g["state"]["adam_t"] == 4 for g in got2)

    # the checkpoint saved on several ranks loads in a one-GPU model: the same whole tensors
    from code2vec_b200.b200_model import Code2VecModel
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    whole = _read_whole(second + ".c2v_b200")
    one = Code2VecModel(_config(prefix, tmp_path, MODEL_LOAD_PATH=second))
    try:
        for k, v in one.engine.export_params().items():
            assert np.array_equal(v, whole["theta/" + k]), k
    finally:
        one.close_session()
    for r, g in enumerate(got2):                        # and the file holds exactly what the ranks held
        for k in ("theta/tok", "adam_m/path", "adam_v/tok"):
            mine = whole[k][r::world]
            assert np.array_equal(mine, g["state"][k][:mine.shape[0]]), (r, k)


def test_resume_across_world_sizes(tmp_path, monkeypatch):
    """Saved on 4 ranks, loaded on 2: saving again gives the same bytes, and two more steps equal a 2-rank Trainer that
    starts from the file's tensors."""
    monkeypatch.chdir(tmp_path)
    prefix, _ = _make_dataset(tmp_path, n_train=64)
    f4, f2, f2b = (str(tmp_path / d / "saved") for d in ("w4", "w2", "w2b"))
    make4 = lambda: _config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, NUM_TRAIN_EPOCHS=1, MODEL_SAVE_PATH=f4)
    got4 = _models(monkeypatch, 4, make4, _train_and_record)
    make2 = lambda: _config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, NUM_TRAIN_EPOCHS=1, MODEL_LOAD_PATH=f4,
                            MODEL_SAVE_PATH=f2b)

    def save_then_train(model, r):
        model.save(f2)
        return _train_and_record(model, r)
    got2 = _models(monkeypatch, 2, make2, save_then_train)
    assert open(f4 + ".c2v_b200", "rb").read() == open(f2 + ".c2v_b200", "rb").read()
    _, want = _drive(monkeypatch, 2, got4[0]["dims"], 16, got4[0]["batches"], keep=0.75,
                     start=_read_whole(f4 + ".c2v_b200"))
    _assert_states_equal([g["state"] for g in got2], want, "4 -> 2 ranks")


# ---- 5, 6. evaluate() and the exports on W ranks == one GPU ----------------------------------------------------------
@pytest.mark.parametrize("world", [2, 4])
def test_evaluate_and_exports_match_one_gpu(tmp_path, monkeypatch, world):
    """45 test rows in one reader batch of up to 64: global batches of 32 and 13 rows, the last padded (13 is no multiple
    of 2 or 4); every example is scored once."""
    from code2vec_b200.b200_model import Code2VecModel
    from code2vec_b200.vocabularies import VocabType
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    prefix, _ = _make_dataset(tmp_path, n_test=45)
    save = str(tmp_path / "model" / "saved")
    m = Code2VecModel(_config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, MODEL_SAVE_PATH=save, NUM_TRAIN_EPOCHS=20))
    try:
        m.train()
    finally:
        m.close_session()
    make = lambda: _config(prefix, tmp_path, MODEL_LOAD_PATH=save, TEST_DATA_PATH=prefix + ".test.c2v",
                           EXPORT_CODE_VECTORS=True, TEST_BATCH_SIZE=64)
    outputs = {}

    def run(model, r, tag):
        res = model.evaluate()
        if r == 0:
            outputs[tag] = dict(log=open("log.txt").read(), vectors=open(prefix + ".test.c2v.vectors").read())
        for vt, name in ((VocabType.Token, "tok"), (VocabType.Target, "tgt"), (VocabType.Path, "path")):
            model.save_word2vec_format(str(tmp_path / ("%s.%s.w2v" % (tag, name))), vt)
        if r == 0:
            outputs[tag].update({n: open(str(tmp_path / ("%s.%s.w2v" % (tag, n))), "rb").read()
                                 for n in ("tok", "tgt", "path")})
        return res

    one = Code2VecModel(make())
    try:
        want = run(one, 0, "one")
    finally:
        one.close_session()
    got = _models(monkeypatch, world, make, lambda model, r: run(model, r, "multi"))
    lines = outputs["one"]["vectors"].splitlines()
    assert len(lines) == 45 and len(outputs["multi"]["vectors"].splitlines()) == 45
    bad = [i for i, (a, b) in enumerate(zip(lines, outputs["multi"]["vectors"].splitlines())) if a != b]
    assert not bad, ("code vectors differ in rows", bad[:10])
    assert outputs["multi"]["log"] == outputs["one"]["log"], "log.txt differs (a top-k near-tie would show here)"
    for r in range(world):
        assert np.array_equal(got[r].topk_acc, want.topk_acc) and str(got[r]) == str(want), r
    for n in ("tok", "tgt", "path"):
        assert outputs["multi"][n] == outputs["one"][n], n
