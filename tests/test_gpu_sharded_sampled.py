"""The sampled softmax on the fully sharded schedule (DESIGN.md section 6j, "Several GPUs"), with 2, 4 and 8 ranks emulated
on one GPU (tests/emulated_ranks.py).

  * c2v_sample_log_uniform_vocab on a row-sharded engine draws what c2v_sample_log_uniform draws on an engine holding the
    whole table: ids, num_tries and every log count, bit for bit; the plain call keeps its refusal there.
  * The first Trainer.step_sampled on W ranks, in fp32, tf32 and 3xTF32, against reference64.train_step64(sampled=...) on
    the global batch through the Adam slots (as test_gpu_emulated_ranks), at a toy shape and at the benchmark shape
    (Bt = 1024, D = 384, Y = 261,246, S in {25, 1024}).  The same checks fail with logq_sampled + 1e-3 and with the
    all-gather of the negatives' partial gradients off by 1 %.
  * Deterministic runs on 4 ranks repeat bit for bit, a short batch included.
  * Code2VecModel.train() on 2 and 4 ranks with C2V_NUM_SAMPLED and C2V_SHARDED_SAMPLED: the toy rule is learnt, the host,
    device-reader and sharded-reader routes give the same per-step losses and checkpoint bytes, and the checkpoint
    evaluates as a one-GPU model does."""
import gc
import threading

import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests import reference64 as R
from tests import sampler_model as SM
from tests.emulated_ranks import EmulatedGroup, emulate_ipc, run_ranks
from tests.test_gpu_emulated_ranks import KEEP, MID, SEED, check_loss, check_slots, rank_dropout, run_schedule
from tests.test_gpu_reference64 import PROD, PROD_B, report

pytestmark = pytest.mark.gpu

_cache = {}


@pytest.fixture(scope="module", autouse=True)
def _release_references():
    yield
    _cache.clear()


# ---- the vocabulary-explicit sampler -------------------------------------------------------------------------------------
def _sharded_engines(world, Y, group, monkeypatch, Bl=64):
    """`world` fully sharded engines (small tables, Y target rows in blocks) whose Trainers have sharded the tables."""
    import torch
    from code2vec_b200.engine import EngineDims
    from code2vec_b200.trainer import Trainer, make_fully_sharded_engine
    group.install(monkeypatch)
    dims = EngineDims(1001, 501, Y, 32, 96, 8, Bl, 10)
    engines = []
    for r in range(world):
        with group.as_rank(r):
            e = make_fully_sharded_engine(dims, Bl, device=0)
        e.init_params(whole_target_table=True)
        engines.append(e)
    emulate_ipc(engines)

    def body(r):
        torch.cuda.set_device(0)
        Trainer(engines[r], seed=SEED, schedule="fully_sharded")
    run_ranks(world, body, group)
    return engines


@pytest.mark.parametrize("Y", [1025, 261246])
def test_vocab_sampler_equals_the_whole_table_sampler(monkeypatch, Y):
    import torch
    from tests.test_gpu_sampled_training import SEEDS, _sampler_engine
    world = 2
    group = EmulatedGroup(world)
    engines = _sharded_engines(world, Y, group, monkeypatch)
    whole = _sampler_engine(Y)
    try:
        rng = np.random.default_rng(Y)
        for e in engines:
            assert e.table_world == world and e.dims.target_vocab < Y
            tgt = e.to_device(np.zeros(4, np.int32), torch.int32)
            with pytest.raises(RuntimeError, match="single-GPU"):
                e.sample_log_uniform(tgt, 1, 0, 1)
        for S in (1, 25, 1024):
            S = min(S, Y // 2)
            for seed, step in SEEDS:
                target = rng.integers(0, Y, 64).astype(np.int32)
                want = [t.cpu().numpy().copy() for t in whole.sample_log_uniform(whole.to_device(target, torch.int32), S,
                                                                                 seed, step)]
                for r, e in enumerate(engines):
                    lo = r * 32
                    got = [t.cpu().numpy().copy() for t in e.sample_log_uniform_vocab(
                        e.to_device(target[lo:lo + 32], torch.int32), S, Y, seed, step)]
                    label = (Y, S, seed, step, r)
                    assert np.array_equal(got[0], want[0]), label
                    assert got[3][0] == want[3][0], label
                    assert np.array_equal(got[1].view(np.int32), want[1][lo:lo + 32].view(np.int32)), label
                    assert np.array_equal(got[2].view(np.int32), want[2].view(np.int32)), label
        for e in engines:
            assert e.get_option("sampler_cap_hits") == 0
    finally:
        torch.cuda.synchronize()
        whole.close()
        for e in engines:
            e.close()


# ---- the first step against float64 --------------------------------------------------------------------------------------
def _sampled_reference(key, dims, params, batch, world, S):
    """The global batch's float64 step with the negatives every rank draws for (SEED, t = 1)."""
    if key not in _cache:
        _cache.clear()
        sampled, tries, lq_t, lq_s = SM.sample_with_logq(S, dims.target_vocab, batch[4], SEED, 1)
        dm = rank_dropout(dims, world, batch[0].shape[0] // world, 1)
        ref = R.train_step64(params, *batch, keep=KEEP, dropout_mask=dm, sampled=sampled, logq_true=lq_t,
                             logq_sampled=lq_s)
        ref.extra["sampled"] = sampled
        _cache[key] = ref
    return _cache[key]


def _toy_case(S):
    """MID with targets that hit the sampled ids and repeat across ranks."""
    params = O.init_params(MID, seed=4321)
    batch = list(O.synthetic_batch(MID, 512, seed=2024))
    sampled, _ = SM.sample(S, MID.target_vocab, SEED, 1)
    tgt = batch[4].copy()
    tgt[3], tgt[300], tgt[511] = sampled[0], sampled[S - 1], sampled[5]     # accidental hits on three ranks
    tgt[64 + 1] = tgt[1]                                                    # the same target on ranks 0 and 1 (W >= 4)
    tgt[256 + 7] = tgt[7]
    batch[4] = tgt
    return params, tuple(batch)


def run_sampled_schedule(monkeypatch, dims, params, batch, world, math, S, setup=None, group=None, steps=1):
    def sampled_setup(r, e, tr):
        tr.step_device = lambda *d: tr.step_sampled(*d, S)
        if setup:
            setup(r, e, tr)
    return run_schedule(monkeypatch, dims, params, batch, world, "fully_sharded", math, steps=steps, setup=sampled_setup,
                        group=group)


def check_sampled(monkeypatch, dims, params, batch, world, math, S, key, label, setup=None, group=None):
    # a Trainer whose step_device is replaced holds itself in a cycle: free the last run's engines before the next
    gc.collect()
    ref = _sampled_reference(key, dims, params, batch, world, S)
    out, engines = run_sampled_schedule(monkeypatch, dims, params, batch, world, math, S, setup=setup, group=group)
    worst = check_slots(out, engines, dims, "fully_sharded", world, ref, math, label)
    worst["loss"] = check_loss(out, "fully_sharded", ref, label)
    for o in out:
        ph = o["step1"]["phases"]
        assert ph.get("sampler", 0) == 1 and ph.get("sampled_softmax", 0) == 3, (label, ph)
        assert ph.get("logits", 0) == 0, (label, ph)            # no full-softmax phase ran
    report(label, worst)
    return worst


@pytest.mark.parametrize("math", [0, 1, 2])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_first_step_against_float64(monkeypatch, world, math):
    S = 64
    params, batch = _toy_case(S)
    check_sampled(monkeypatch, MID, params, batch, world, math, S, ("toy", world, S),
                  "sharded-sampled toy world=%d math=%d" % (world, math))


# S = 1024 first: each reference is built once and dropped when the next one is built
@pytest.mark.parametrize("math", [0, 1, 2])
@pytest.mark.parametrize("S", [1024, 25])
def test_first_step_at_the_benchmark_shape(monkeypatch, S, math):
    world = 8
    params = O.init_params(PROD, seed=4321)
    batch = O.synthetic_batch(PROD, PROD_B, seed=4242)
    check_sampled(monkeypatch, PROD, params, batch, world, math, S, ("prod", world, S),
                  "sharded-sampled prod world=%d S=%d math=%d" % (world, S, math))


def test_negative_controls(monkeypatch):
    """3xTF32 on 4 ranks: the checks the true step passes fail with logq_sampled + 1e-3 on every rank, and with the
    all-gather of the negatives' partial target gradients (the second all-gather of the step) scaled by 1.01."""
    world, math, S = 4, 2, 64
    params, batch = _toy_case(S)
    key = ("toy", world, S)

    def shifted(r, e, tr):
        draw = e.sample_log_uniform_vocab

        def draw_shifted(*a, **k):
            sampled, lq_t, lq_s, tries = draw(*a, **k)
            lq_s.add_(1e-3)
            return sampled, lq_t, lq_s, tries
        e.sample_log_uniform_vocab = draw_shifted
    with pytest.raises(AssertionError):
        check_sampled(monkeypatch, MID, params, batch, world, math, S, key, "control logq + 1e-3", setup=shifted)
    group = EmulatedGroup(world)
    group.fault("all_gather_into_tensor", 2, 1.01)
    with pytest.raises(AssertionError):
        check_sampled(monkeypatch, MID, params, batch, world, math, S, key, "control G_r all-gather x 1.01", group=group)


# ---- determinism ---------------------------------------------------------------------------------------------------------
def _deterministic_run(monkeypatch, world, S, batches, seed_of_rank=lambda r: SEED):
    """Every batch of `batches` (global, split by rank) as a sampled step on `world` ranks with deterministic +
    ordered_exchange: (losses, final parameters and Adam slots of the shards, blocks, W and a)."""
    import torch
    from code2vec_b200.engine import EngineDims
    from code2vec_b200.trainer import Trainer, make_fully_sharded_engine
    from tests.util import dev_batch
    group = EmulatedGroup(world).install(monkeypatch)
    Bl = batches[0][0].shape[0] // world
    dims = EngineDims(MID.token_vocab, MID.path_vocab, MID.target_vocab, MID.embed_dim, MID.code_dim, MID.max_contexts,
                      Bl, 10)
    params = O.init_params(MID, seed=99)
    engines, out = [], [None] * world
    from code2vec_b200.trainer import target_row_block
    try:
        for r in range(world):
            with group.as_rank(r):
                e = make_fully_sharded_engine(dims, Bl, device=0)
            r0, r1 = target_row_block(MID.target_vocab, r, world)
            e.load_params(dict(params, tgt=params["tgt"][r0:r1]))
            e.set_option("math_mode", 1)
            engines.append(e)
        emulate_ipc(engines)

        def body(r):
            torch.cuda.set_device(0)
            e = engines[r]
            tr = Trainer(e, keep_prob=KEEP, seed=seed_of_rank(r), schedule="fully_sharded", deterministic=True,
                         ordered_exchange=True)
            losses = []
            for batch in batches:
                b = batch[0].shape[0] // world
                d = dev_batch(e, *(a[r * b:(r + 1) * b] for a in batch))
                losses.append(float(tr.step_sampled(*d, S).cpu()[0]))
            torch.cuda.synchronize()
            out[r] = dict(losses=losses, p=e.flat_params.cpu().numpy().copy(), m=e.flat_m.cpu().numpy().copy(),
                          v=e.flat_v.cpu().numpy().copy(),
                          shards={"%s/%s" % (g, n): d[n].cpu().numpy().copy() for n in ("tok", "path")
                                  for g, d in (("p", e.shard_params), ("m", e.shard_m), ("v", e.shard_v))})
        run_ranks(world, body, group)
        return out
    finally:
        torch.cuda.synchronize()
        for e in engines:
            e.close()


def test_deterministic_runs_repeat(monkeypatch):
    world, S = 4, 100
    full = O.synthetic_batch(MID, 256, seed=11)
    short = tuple(a[:4 * 37] for a in O.synthetic_batch(MID, 256, seed=12))       # 37 rows per rank
    batches = [full, short, O.synthetic_batch(MID, 256, seed=13)]
    a = _deterministic_run(monkeypatch, world, S, batches)
    b = _deterministic_run(monkeypatch, world, S, batches)
    for r in range(world):
        assert a[r]["losses"] == b[r]["losses"] == a[0]["losses"], r
        for k in ("p", "m", "v"):
            assert np.array_equal(a[r][k].view(np.int32), b[r][k].view(np.int32)), (r, k)
        assert sorted(a[r]["shards"]) == ["m/path", "m/tok", "p/path", "p/tok", "v/path", "v/tok"]
        for n in a[r]["shards"]:
            assert np.array_equal(a[r]["shards"][n].view(np.int32), b[r]["shards"][n].view(np.int32)), (r, n)
    assert all(np.isfinite(a[0]["losses"]))


def test_ranks_with_different_seeds_refuse(monkeypatch):
    """Every rank must draw the same negatives: Trainers whose seeds differ raise on every rank at the first sampled
    step instead of summing rows of different ids."""
    with pytest.raises(ValueError, match="same Trainer seed on every rank"):
        _deterministic_run(monkeypatch, 2, 16, [O.synthetic_batch(MID, 64, seed=11)], seed_of_rank=lambda r: SEED + r)


# ---- Code2VecModel.train() -----------------------------------------------------------------------------------------------
@pytest.fixture
def _ten_target_rows(monkeypatch):
    """The toy dataset with a ninth method name, so that 4 ranks all hold target rows (as tests/test_gpu_multi_rank_model)."""
    import tests.test_gpu_model as toy
    monkeypatch.setattr(toy, "TARGETS", toy.TARGETS + ["make|copy"])


SAMPLED_ENV = {"C2V_NUM_SAMPLED": "4", "C2V_SHARDED_SAMPLED": "1"}


def _per_rank_losses(monkeypatch):
    """Every rank's step_sampled losses, kept on the device until read."""
    from code2vec_b200.trainer import Trainer
    seen, lock = {}, threading.Lock()
    orig = Trainer.step_sampled

    def step(self, *a, **k):
        loss = orig(self, *a, **k)
        with lock:
            seen.setdefault(self.rank, []).append(loss.clone())
        return loss
    monkeypatch.setattr(Trainer, "step_sampled", step)
    return seen


@pytest.mark.parametrize("world", [2, 4])
def test_model_learns_and_evaluates_as_one_gpu(tmp_path, monkeypatch, _ten_target_rows, world):
    from code2vec_b200.b200_model import Code2VecModel
    from tests.test_gpu_model import _config, _make_dataset
    from tests.test_gpu_multi_rank_model import _models
    monkeypatch.chdir(tmp_path)
    prefix, _ = _make_dataset(tmp_path)
    save = str(tmp_path / "m" / "saved")
    seen = _per_rank_losses(monkeypatch)

    def action(model, r):
        assert model.trainer.schedule == "fully_sharded"
        model.train()
        assert model.engine.get_option("sampler_cap_hits") == 0
        return model.evaluate()
    make = lambda: _config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, MODEL_SAVE_PATH=save,
                           TEST_DATA_PATH=prefix + ".test.c2v", DROPOUT_KEEP_RATE=1.0)
    res = _models(monkeypatch, world, make, action, SAMPLED_ENV)
    assert sorted(seen) == list(range(world)) and len(seen[0]) > 0
    losses = [[float(x.cpu()[0]) for x in seen[r]] for r in range(world)]
    assert all(l == losses[0] for l in losses)                   # the global loss, the same bits on every rank
    assert res[0].topk_acc[0] > 0.6, res[0]                      # the toy rule is learnt
    assert all(str(x) == str(res[0]) for x in res)
    # the checkpoint evaluates on one GPU as on the ranks
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    one = Code2VecModel(_config(prefix, tmp_path, MODEL_LOAD_PATH=save, TEST_DATA_PATH=prefix + ".test.c2v"))
    try:
        assert str(one.evaluate()) == str(res[0])
    finally:
        one.close_session()


@pytest.mark.parametrize("world", [2, 4])
def test_routes_agree(tmp_path, monkeypatch, _ten_target_rows, world):
    """The host route, the device reader and the sharded device reader give the same per-step losses and checkpoint
    bytes."""
    import code2vec_b200.device_reader as DR
    from tests.test_gpu_model import _config, _make_dataset
    from tests.test_gpu_multi_rank_model import _models
    from tests.test_gpu_sharded_reader import _Hub, _ThreadTransport
    monkeypatch.chdir(tmp_path)
    prefix, _ = _make_dataset(tmp_path, n_train=101)
    hubs, lock = {}, threading.Lock()

    def make(device):
        import torch.distributed as dist
        with lock:
            hub = hubs.setdefault("hub", _Hub(dist.get_world_size()))
        return _ThreadTransport(hub, dist.get_rank())
    monkeypatch.setattr(DR, "make_share_transport", make)
    out = {}
    for route, env in (("host", {}), ("device_reader", {"C2V_DEVICE_READER": "1"}),
                       ("sharded_reader", {"C2V_DEVICE_READER": "1", "C2V_SHARDED_READER": "1"})):
        hubs.clear()
        save = str(tmp_path / route / "saved")
        with monkeypatch.context() as m:
            seen = _per_rank_losses(m)
            make_cfg = lambda: _config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, MODEL_SAVE_PATH=save,
                                       NUM_TRAIN_EPOCHS=5, NUM_BATCHES_TO_LOG_PROGRESS=3, SHUFFLE_BUFFER_SIZE=40,
                                       DROPOUT_KEEP_RATE=0.75)
            _models(m, world, make_cfg, lambda model, r: model.train(),
                    dict({"C2V_DETERMINISTIC": "1", "C2V_SEED": "7"}, **SAMPLED_ENV, **env))
            losses = [[float(x.cpu()[0]) for x in seen[r]] for r in range(world)]
        with open(save + ".c2v_b200", "rb") as f:
            out[route] = (losses, f.read())
    l0, c0 = out["host"]
    assert len(l0[0]) == -(-101 * 5 // 32)
    for route, (losses, ckpt) in out.items():
        assert losses == l0 and ckpt == c0, route


# ---- resume: two steps, save, load, two more == four steps; saved on 4 ranks, loaded on 2 -------------------------------
def _record_sampled(model, r):
    """train() on one rank through the host route: the losses and negatives (ids, num_tries) of its sampled steps, its
    state, its dims and (rank 0) the reader's batches."""
    from tests.test_gpu_multi_rank_model import _reader_batches, _state
    batches = _reader_batches(model) if r == 0 else None
    tr = model.trainer
    losses, draws, step = [], [], tr.step_host_sampled

    def recording(*a, **k):
        losses.append(step(*a, **k))
        out = tr.e._sampler_out
        draws.append((int(tr.e.adam_t), out[0][:int(a[-1])].cpu().numpy().copy(), int(out[3].cpu()[0])))   # t of the step
        return losses[-1]
    tr.step_host_sampled = recording
    model.train()
    return dict(losses=losses, draws=draws, state=_state(model.engine), dims=vars(model._engine_dims()), batches=batches)


def _drive_sampled(monkeypatch, world, dims, local_batch, batches, start=None):
    """tests/test_gpu_multi_rank_model._drive with every step a sampled one (Trainer.step_host_sampled, S = 4)."""
    from code2vec_b200.trainer import Trainer
    from tests.test_gpu_multi_rank_model import _drive
    S = int(SAMPLED_ENV["C2V_NUM_SAMPLED"])
    with monkeypatch.context() as m:
        m.setattr(Trainer, "step_host", lambda self, *a, **k: Trainer.step_host_sampled(self, *a, S))
        return _drive(m, world, dims, local_batch, batches, keep=0.75, start=start)


def _check_draws(got, Y):
    """Every recorded step drew what the one-GPU sampler statement draws for (C2V_SEED, t) over the whole vocabulary."""
    from tests.test_gpu_multi_rank_model import SEED as RUN_SEED
    S = int(SAMPLED_ENV["C2V_NUM_SAMPLED"])
    for g in got:
        assert g["draws"]
        for t, ids, tries in g["draws"]:
            want, want_tries = SM.sample(S, Y, int(RUN_SEED), t)
            assert np.array_equal(ids, want) and tries == want_tries, (t, ids, want)


@pytest.mark.parametrize("world", [2, 4])
def test_resume_continues_exactly(tmp_path, monkeypatch, _ten_target_rows, world):
    """C2V_DETERMINISTIC=1, C2V_SEED fixed: 2 sampled steps, save, load and 2 more equal 4 uninterrupted steps in every
    loss, parameter and Adam slot (shards, target blocks, W, a) and in the step count."""
    from tests.test_gpu_model import _config, _make_dataset
    from tests.test_gpu_multi_rank_model import _assert_states_equal, _models
    monkeypatch.chdir(tmp_path)
    prefix, _ = _make_dataset(tmp_path, n_train=64)
    first, second = str(tmp_path / "a" / "saved"), str(tmp_path / "b" / "saved")
    make1 = lambda: _config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, NUM_TRAIN_EPOCHS=1, MODEL_SAVE_PATH=first)
    got1 = _models(monkeypatch, world, make1, _record_sampled, SAMPLED_ENV)
    make2 = lambda: _config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, NUM_TRAIN_EPOCHS=1, MODEL_LOAD_PATH=first,
                            MODEL_SAVE_PATH=second)
    got2 = _models(monkeypatch, world, make2, _record_sampled, SAMPLED_ENV)
    batches = got1[0]["batches"]
    assert len(batches) == 2
    assert all(np.array_equal(a, b) for x, y in zip(batches, got2[0]["batches"]) for a, b in zip(x, y))
    losses, four = _drive_sampled(monkeypatch, world, got1[0]["dims"], 32 // world, batches + batches)
    _assert_states_equal([g["state"] for g in got2], four, "resumed sampled world=%d" % world)
    assert all(g["state"]["adam_t"] == 4 for g in got2)
    for r in range(world):
        assert got1[r]["losses"] + got2[r]["losses"] == losses[r] == losses[0], r
    assert [t for t, _, _ in got1[0]["draws"]] == [1, 2] and [t for t, _, _ in got2[0]["draws"]] == [3, 4]
    _check_draws(got1 + got2, got1[0]["dims"]["target_vocab"])


def test_resume_across_world_sizes(tmp_path, monkeypatch, _ten_target_rows):
    """Saved on 4 ranks, loaded on 2: the 2-rank run continues with the negatives of the step count it resumed at (the
    ones a one-GPU run draws), and equals a 2-rank Trainer that starts from the file's tensors."""
    from tests.test_gpu_model import _config, _make_dataset
    from tests.test_gpu_multi_rank_model import _assert_states_equal, _models, _read_whole
    monkeypatch.chdir(tmp_path)
    prefix, _ = _make_dataset(tmp_path, n_train=64)
    f4, f2 = str(tmp_path / "w4" / "saved"), str(tmp_path / "w2" / "saved")
    make4 = lambda: _config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, NUM_TRAIN_EPOCHS=1, MODEL_SAVE_PATH=f4)
    got4 = _models(monkeypatch, 4, make4, _record_sampled, SAMPLED_ENV)
    make2 = lambda: _config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, NUM_TRAIN_EPOCHS=1, MODEL_LOAD_PATH=f4,
                            MODEL_SAVE_PATH=f2)
    got2 = _models(monkeypatch, 2, make2, _record_sampled, SAMPLED_ENV)
    assert [t for t, _, _ in got2[0]["draws"]] == [3, 4]
    _check_draws(got4 + got2, got4[0]["dims"]["target_vocab"])
    losses, want = _drive_sampled(monkeypatch, 2, got4[0]["dims"], 16, got4[0]["batches"], start=_read_whole(f4 + ".c2v_b200"))
    _assert_states_equal([g["state"] for g in got2], want, "sampled 4 -> 2 ranks")
    for r in range(2):
        assert got2[r]["losses"] == losses[r], r
    assert all(g["state"]["adam_t"] == 4 for g in got2)
