"""The in-process rank emulator (tests/emulated_ranks.py) on CPU tensors: every collective at world 2, 4 and 8 against
numpy, the object all-gather, the fault hook, failure propagation through the barrier, and the monkeypatch's undo."""
import threading
import time

import numpy as np
import pytest
import torch
import torch.distributed as dist

from tests.emulated_ranks import EmulatedGroup, run_ranks

WORLDS = [2, 4, 8]


def inputs(world, n, seed):
    rng = np.random.default_rng(seed)
    return [rng.standard_normal(n).astype(np.float32) for _ in range(world)]


def rank_order_sum(parts):
    acc = parts[0].copy()
    for p in parts[1:]:
        acc += p                  # float32, in rank order: what every rank computes
    return acc


@pytest.mark.parametrize("op", ["sum", "avg"])
@pytest.mark.parametrize("world", WORLDS)
def test_all_reduce(monkeypatch, world, op):
    g = EmulatedGroup(world).install(monkeypatch)
    xs = inputs(world, 1000, world)
    want = rank_order_sum(xs)
    if op == "avg":
        want = want / np.float32(world)
    out = [None] * world

    def fn(r):
        t = torch.from_numpy(xs[r].copy())
        w = dist.all_reduce(t, op=dist.ReduceOp.SUM if op == "sum" else dist.ReduceOp.AVG, async_op=True)
        w.wait()
        out[r] = t.numpy()

    run_ranks(world, fn, g)
    for r in range(world):
        assert np.array_equal(out[r], want), r          # the same bits on every rank
    np.testing.assert_allclose(want, np.sum(np.stack(xs).astype(np.float64), axis=0) / (world if op == "avg" else 1),
                               rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("world", WORLDS)
def test_reduce_scatter_tensor(monkeypatch, world):
    g = EmulatedGroup(world).install(monkeypatch)
    n = 37
    xs = inputs(world, n * world, 10 + world)
    total = rank_order_sum(xs)
    out = [None] * world

    def fn(r):
        o = torch.empty(n)
        dist.reduce_scatter_tensor(o, torch.from_numpy(xs[r]).view(world, n), op=dist.ReduceOp.AVG)
        out[r] = o.numpy()

    run_ranks(world, fn, g)
    for r in range(world):
        assert np.array_equal(out[r], total[r * n:(r + 1) * n] / np.float32(world)), r


@pytest.mark.parametrize("world", WORLDS)
def test_all_gather_into_tensor(monkeypatch, world):
    g = EmulatedGroup(world).install(monkeypatch)
    xs = [np.arange(5, dtype=np.int32) + 100 * r for r in range(world)]
    out = [None] * world

    def fn(r):
        o = torch.empty(5 * world, dtype=torch.int32)
        dist.all_gather_into_tensor(o, torch.from_numpy(xs[r]))
        out[r] = o.numpy()

    run_ranks(world, fn, g)
    for r in range(world):
        assert np.array_equal(out[r], np.concatenate(xs)), r


@pytest.mark.parametrize("world", WORLDS)
def test_all_gather_object_and_rank_queries(monkeypatch, world):
    g = EmulatedGroup(world).install(monkeypatch)
    out = [None] * world

    def fn(r):
        assert dist.is_available() and dist.is_initialized()
        assert dist.get_world_size() == world and dist.get_rank() == r and dist.get_backend() == "nccl"
        got = [None] * world
        dist.all_gather_object(got, {"rank": r, "h": b"x" * r})
        dist.barrier()
        out[r] = got

    run_ranks(world, fn, g)
    for r in range(world):
        assert out[r] == [{"rank": s, "h": b"x" * s} for s in range(world)]


def test_fault_hook_scales_the_nth_call(monkeypatch):
    world = 4
    g = EmulatedGroup(world).install(monkeypatch)
    g.fault("reduce_scatter_tensor", 2, 1.01)
    out = [None] * world

    def fn(r):
        o = torch.empty(3)
        res = []
        for _ in range(3):
            dist.reduce_scatter_tensor(o, torch.ones(3 * world), op=dist.ReduceOp.SUM)
            res.append(o.clone().numpy())
        out[r] = res

    run_ranks(world, fn, g)
    for r in range(world):
        assert np.array_equal(out[r][0], np.full(3, 4.0, np.float32))
        assert np.array_equal(out[r][1], np.full(3, 4.0, np.float32) * np.float32(1.01))
        assert np.array_equal(out[r][2], np.full(3, 4.0, np.float32))


def test_a_failing_rank_aborts_the_others(monkeypatch):
    world = 4
    g = EmulatedGroup(world, timeout=30.0).install(monkeypatch)
    t0 = time.monotonic()

    def fn(r):
        if r == 2:
            raise ValueError("rank 2 fails before the collective")
        dist.all_reduce(torch.ones(4))

    with pytest.raises(ValueError, match="rank 2 fails"):
        run_ranks(world, fn, g)
    assert time.monotonic() - t0 < 10.0          # aborted, not timed out
    assert not [t for t in threading.enumerate() if t.name.startswith("rank")]


def test_a_missing_rank_times_out(monkeypatch):
    world = 2
    g = EmulatedGroup(world, timeout=0.5).install(monkeypatch)

    def fn(r):
        if r == 0:
            dist.all_reduce(torch.ones(4))        # rank 1 never joins

    with pytest.raises(threading.BrokenBarrierError):
        run_ranks(world, fn, g)


def test_monkeypatch_is_undone():
    before = {k: getattr(dist, k, None) for k in ("all_reduce", "get_rank", "get_world_size", "is_initialized", "barrier")}
    with pytest.MonkeyPatch.context() as mp:
        EmulatedGroup(2).install(mp)
        assert dist.get_world_size() == 2 and dist.is_initialized()
    for k, v in before.items():
        assert getattr(dist, k, None) is v, k
    assert not dist.is_initialized()


@pytest.mark.parametrize("Y,world", [(9, 8), (9, 4), (3, 4)])
def test_fully_sharded_refuses_ranks_without_target_rows(monkeypatch, Y, world):
    """Blocks of ceil(Y / world) rows leave the last ranks empty here (Y = 9 on 8 ranks: blocks of 2 for ranks 0..4).  An
    engine needs at least one target row, and that row's logit would enter every example's normaliser, so every rank
    refuses the split before any engine is made."""
    from code2vec_b200.engine import EngineDims
    from code2vec_b200.trainer import make_fully_sharded_engine, target_row_block
    g = EmulatedGroup(world).install(monkeypatch)
    assert target_row_block(Y, world - 1, world)[0] == Y
    dims = EngineDims(101, 51, Y, 8, 24, 5, 4, 10)
    for r in range(world):
        with g.as_rank(r):
            with pytest.raises(ValueError, match="without a row"):
                make_fully_sharded_engine(dims, 4, device=0)
