"""Host side of Code2VecModel on 2, 4 and 8 GPUs (code2vec_b200/multi_rank.py), without a GPU: the split of a global
batch over the ranks, the checkpoint written and read by several ranks (byte-identical to the one-GPU file, readable on
any world size), and the runs that are refused before any engine exists."""
import json
import struct

import numpy as np
import pytest

from code2vec_b200.engine import PARAM_NAMES, EngineDims
from code2vec_b200.multi_rank import (CKPT_MAGIC, batch_split, check_multi_rank_run, checkpoint_header,
                                      create_checkpoint_file, read_checkpoint_part, write_checkpoint,
                                      write_checkpoint_part)
from code2vec_b200.trainer import target_row_block

PAD = np.float32(-7.5e30)          # what padding rows hold before and after a read


# ---- the batch split -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("rows", [1, 3, 7, 8, 9, 63, 64, 65, 127, 128, 1024])
def test_batch_split(world, rows):
    parts = [batch_split(rows, world, r) for r in range(world)]
    b = rows // world
    assert all(hi - lo == b for lo, hi, _ in parts)
    assert all(d == rows - world * b and 0 <= d < world for _, _, d in parts)
    covered = [i for lo, hi, _ in parts for i in range(lo, hi)]
    assert covered == list(range(world * b))          # disjoint, contiguous, in rank order, from row 0
    if rows < world:
        assert covered == [] and parts[0][2] == rows   # the batch is skipped and every row counted as left out


# ---- the checkpoint --------------------------------------------------------------------------------------------------
DIMS = dict(vars(EngineDims(token_vocab=1001, path_vocab=517, target_vocab=203, embed_dim=4, code_dim=6, max_contexts=9,
                            max_batch=64, top_k=5)))


def _model(seed, with_optimizer=True):
    rng = np.random.default_rng(seed)
    shapes = EngineDims(**DIMS).shapes()
    groups = ("theta", "adam_m", "adam_v") if with_optimizer else ("theta",)
    return {g + "/" + k: rng.standard_normal(shapes[k]).astype(np.float32) for g in groups for k in PARAM_NAMES}


def _legacy_bytes(model, adam_t, epochs, with_optimizer):
    """The file the one-GPU model wrote before the format moved into multi_rank: json header of the same fields."""
    names = [g + "/" + k for g in (("theta", "adam_m", "adam_v") if with_optimizer else ("theta",)) for k in PARAM_NAMES]
    meta = {"format": 1, "dims": DIMS, "adam_t": adam_t if with_optimizer else 0, "epochs_trained": epochs,
            "tf_names": {"tok": "model/WORDS_VOCAB", "path": "model/PATHS_VOCAB", "tgt": "model/TARGET_WORDS_VOCAB",
                         "W": "model/TRANSFORM", "a": "model/ATTENTION"}, "tensors": []}
    off = 0
    for n in names:
        meta["tensors"].append({"name": n, "shape": list(model[n].shape), "offset": off, "nbytes": model[n].size * 4})
        off += model[n].size * 4
    header = json.dumps(meta).encode()
    return CKPT_MAGIC + struct.pack("<Q", len(header)) + header + b"".join(model[n].astype("<f4").tobytes() for n in names)


def _rank_tensors(model, rank, world):
    """What rank `rank` of `world` holds: embedding shards of ceil(T / world) rows (padding rows = PAD), its target block,
    W and a."""
    out = {}
    y0, y1 = target_row_block(DIMS["target_vocab"], rank, world)
    for name, t in model.items():
        k = name.split("/")[1]
        if k in ("tok", "path"):
            shard = np.full(((t.shape[0] + world - 1) // world, t.shape[1]), PAD, dtype=np.float32)
            mine = t[rank::world]
            shard[:mine.shape[0]] = mine
            out[name] = shard
        elif k == "tgt":
            out[name] = t[y0:y1].copy()
        else:
            out[name] = t.copy()
    return out


def _write_on(path, world, held, adam_t=17, epochs=3, with_optimizer=True):
    prefix, entries, total = checkpoint_header(DIMS, adam_t, epochs, with_optimizer)
    create_checkpoint_file(path, prefix, total)
    for r in reversed(range(world)):         # any order: the ranks write disjoint bytes
        write_checkpoint_part(path, len(prefix), entries, r, world, target_row_block(DIMS["target_vocab"], r, world),
                              held[r])


def _read_on(path, world, names):
    held = []
    for r in range(world):
        shapes = {n: s.shape for n, s in _rank_tensors({n: np.zeros(EngineDims(**DIMS).shapes()[n.split("/")[1]],
                                                                      dtype=np.float32) for n in names}, r, world).items()}
        out = {n: np.full(s, PAD, dtype=np.float32) for n, s in shapes.items()}
        read_checkpoint_part(path, r, world, target_row_block(DIMS["target_vocab"], r, world), out)
        held.append(out)
    return held


@pytest.mark.parametrize("with_optimizer", [True, False])
def test_one_gpu_writer_keeps_its_bytes(tmp_path, with_optimizer):
    model = _model(1, with_optimizer)
    prefix, _, total = checkpoint_header(DIMS, 17, 3, with_optimizer)
    path = str(tmp_path / "one.c2v_b200")
    write_checkpoint(path, prefix, list(model.values()))
    data = open(path, "rb").read()
    assert data == _legacy_bytes(model, 17, 3, with_optimizer) and len(data) == total


@pytest.mark.parametrize("with_optimizer", [True, False])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_sharded_write_equals_one_gpu_file(tmp_path, world, with_optimizer):
    model = _model(world, with_optimizer)
    path = str(tmp_path / "w.c2v_b200")
    _write_on(path, world, [_rank_tensors(model, r, world) for r in range(world)], with_optimizer=with_optimizer)
    assert open(path, "rb").read() == _legacy_bytes(model, 17, 3, with_optimizer)


@pytest.mark.parametrize("world_written", [1, 8])
@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_read_on_any_world_size(tmp_path, world_written, world):
    model = _model(5)
    path = str(tmp_path / "w.c2v_b200")
    _write_on(path, world_written, [_rank_tensors(model, r, world_written) for r in range(world_written)])
    held = _read_on(path, world, list(model))
    for r in range(world):
        want = _rank_tensors(model, r, world)
        for n in model:
            # exactly the rank's rows; padding rows past the table's end still hold what they held before the read
            assert np.array_equal(held[r][n], want[n]), (r, n)


def test_read_leaves_missing_tensors_alone(tmp_path):
    """A checkpoint without Adam slots (--release) read into a training rank: the slots are left as they are."""
    model = _model(6, with_optimizer=False)
    path = str(tmp_path / "w.c2v_b200")
    _write_on(path, 2, [_rank_tensors(model, r, 2) for r in range(2)], with_optimizer=False)
    held = _read_on(path, 2, list(_model(6)))
    assert all((held[r]["adam_m/tok"] == PAD).all() and (held[r]["adam_v/W"] == PAD).all() for r in range(2))
    assert np.array_equal(held[1]["theta/W"], model["theta/W"])


def test_written_on_4_read_on_2_written_again(tmp_path):
    model = _model(7)
    first, second = str(tmp_path / "a.c2v_b200"), str(tmp_path / "b.c2v_b200")
    _write_on(first, 4, [_rank_tensors(model, r, 4) for r in range(4)])
    _write_on(second, 2, _read_on(first, 2, list(model)))
    assert open(first, "rb").read() == open(second, "rb").read()


# ---- what is refused --------------------------------------------------------------------------------------------------
def _config(**kw):
    from code2vec_b200.config import Config
    cfg = Config(set_defaults=True)
    cfg.DL_FRAMEWORK = "b200"
    cfg.TRAIN_BATCH_SIZE = 1024
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


@pytest.mark.parametrize("world, kw, words", [
    (3, {}, ["WORLD_SIZE=3", "1, 2, 4 or 8", "--nproc-per-node"]),
    (16, {}, ["WORLD_SIZE=16", "1, 2, 4 or 8"]),
    (8, {"TRAIN_BATCH_SIZE": 100}, ["TRAIN_BATCH_SIZE=100", "multiple of the 8 ranks", "divisible by 8"]),
    (2, {"PREDICT": True}, ["--predict runs on one GPU", "single process"]),
    (4, {"RELEASE": True}, ["--release runs on one GPU", "single process"]),
    (2, {"DL_FRAMEWORK": "b200-keras"}, ["b200-keras runs on one GPU", "--framework b200"]),
])
def test_refusals(world, kw, words):
    with pytest.raises(ValueError) as err:
        check_multi_rank_run(_config(**kw), world)
    for w in words:
        assert w in str(err.value), (w, str(err.value))


@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_accepted(world):
    check_multi_rank_run(_config(), world)
    if world == 1:         # one GPU keeps every option
        check_multi_rank_run(_config(PREDICT=True, RELEASE=True, DL_FRAMEWORK="b200-keras", TRAIN_BATCH_SIZE=7), 1)


@pytest.mark.parametrize("framework", ["b200", "b200-keras"])
def test_model_refuses_before_any_engine(monkeypatch, framework):
    """Code2VecModel checks the launch first: these raise without a GPU, a process group or a dataset."""
    from code2vec_b200 import load_model_dynamically
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(ValueError, match="runs on one GPU"):
        load_model_dynamically(_config(DL_FRAMEWORK=framework, PREDICT=framework == "b200"))
    monkeypatch.setenv("WORLD_SIZE", "6")
    with pytest.raises(ValueError, match="WORLD_SIZE=6"):
        load_model_dynamically(_config(DL_FRAMEWORK=framework))


# ---- a failure on one rank reaches every rank --------------------------------------------------------------------------
@pytest.mark.parametrize("failing", [0, 1])
def test_all_ok_reports_a_failure_to_every_rank(monkeypatch, failing):
    """The rank-0 work of a multi-GPU run (side-car counts, the checkpoint's header and rename) and every rank's share of a
    save end in one all-gather that carries each rank's error, so the other ranks raise at once instead of waiting in the
    next collective for a rank that has gone."""
    from code2vec_b200.b200_model import Code2VecModel
    from tests.emulated_ranks import EmulatedGroup, run_ranks
    group = EmulatedGroup(2).install(monkeypatch)
    raised = [None, None]

    def work():
        if group.rank == failing:
            raise OSError("disk full")

    def rank(r):
        model = Code2VecModel.__new__(Code2VecModel)
        model.world, model.rank = 2, r
        try:
            model._all_ok(work, ranks=(failing,) if failing == 0 else None)
        except Exception as exc:
            raised[r] = exc
        model._all_ok(lambda: None)              # the group is still in step afterwards
    run_ranks(2, rank, group)
    assert isinstance(raised[failing], OSError)
    assert isinstance(raised[1 - failing], RuntimeError) and "rank %d failed: OSError: disk full" % failing in str(raised[1 - failing])
