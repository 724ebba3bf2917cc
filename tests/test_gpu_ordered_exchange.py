"""Option "ordered_exchange" (include/c2v_b200.h, DESIGN.md section 5.1) on 2, 4 and 8 ranks emulated on one GPU
(tests/emulated_ranks.py): deterministic training on row-sharded embedding tables.

The exchange is pinned bit for bit to the numpy statement of its order (tests/ordered_exchange.py); whole Trainer steps of
the two row-sharded schedules repeat bit for bit, still pass the float64 per-element bounds of the multi-rank suite, and
agree with the plain push where no order can matter."""
import ctypes
import zlib

import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests import ordered_exchange as OX
from tests.emulated_ranks import EmulatedGroup, emulate_ipc, run_ranks
from tests.test_gpu_emulated_ranks import (KEEP, MID, SEED, _np, _snapshot, assemble, check_loss, check_slots,
                                           reference)
from tests.util import dev_batch, make_engine

pytestmark = pytest.mark.gpu

SENTINEL = np.float32(-7.25)


def _bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


# ---- 1. the order, bit for bit -------------------------------------------------------------------------------------------
T, P = 1003, 509          # neither a multiple of 2, 4 or 8: the last local row exists on some ranks only
CAP_B, CAP_C = 32, 50     # a sender may push 3 * 32 * 50 = 4800 entries


def _vals(rng, n, d):
    v = (rng.standard_normal((n, d)) * 2.0 ** rng.uniform(-20, 20, (n, 1))).astype(np.float32)
    v[rng.random(v.shape) < 0.05] = -0.0
    return v


def _order_case(case, world, d, rng):
    """Per table ("tok", "path"): per sender (global rows, values), in entry order."""
    W = world
    quiet = {2: 0, 4: 2, 8: 5}[W] if case == "quiet" else None       # a sender with nothing at all
    out = {}
    for name, V in (("tok", T), ("path", P)):
        lists = [[] for _ in range(W)]

        def add(s, row, n=1, vals=None):
            lists[s].append((np.full(n, row), _vals(rng, n, d) if vals is None else vals))

        free = iter(rng.permutation(np.arange(8, V)))
        for _ in range(40):                              # listed by every sender, a few entries each
            r = next(free)
            for s in range(W):
                add(s, r, int(rng.integers(1, 4)))
        for _ in range(60):                              # by a random subset
            r = next(free)
            for s in np.flatnonzero(rng.random(W) < 0.5):
                add(s, r, int(rng.integers(1, 3)))
        for _ in range(20):                              # by the highest rank only
            add(W - 1, next(free))
        for n in (1, 32, 33, 1100):                      # chunk boundaries on one sender; others list the row as well
            r = next(free)
            add(W - 1, r, n)
            if n in (32, 33):
                add(0, r, 2)
        # cancellation across senders: 2^20, -2^20, 2^-20 on the first two and the last sender (the last two at world 2)
        r = next(free)
        for s, x in zip(sorted({0, 1, W - 1}) if W > 2 else (0, 0, 1), (2.0 ** 20, -2.0 ** 20, 2.0 ** -20)):
            add(s, r, 1, np.full((1, d), x, dtype=np.float32))
        r = next(free)                                   # nothing but negative zeros, from every sender
        for s in range(W):
            add(s, r, 2, np.full((2, d), -0.0, dtype=np.float32))
        senders = []
        for s in range(W):
            rows = np.concatenate([a for a, _ in lists[s]])
            vals = np.concatenate([b for _, b in lists[s]])
            order = rng.permutation(len(rows))           # interleave the rows; the stable sort keeps each row's order
            rows, vals = rows[order], vals[order]
            keep = np.ones(len(rows), dtype=bool)
            if s == 0:
                keep = rows % W != 1                     # sender 0 has nothing for owner 1
            if s == quiet:
                keep[:] = False
            senders.append((rows[keep].astype(np.int32), vals[keep]))
        out[name] = senders
    return out


@pytest.mark.parametrize("d", [32, 128, 256])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_exchange_order_matches_the_numpy_model_bit_for_bit(monkeypatch, world, d):
    import torch
    import torch.distributed as dist
    dims = O.Dims(token_vocab=T, path_vocab=P, target_vocab=64, embed_dim=d, code_dim=64, max_contexts=CAP_C)
    group = EmulatedGroup(world).install(monkeypatch)
    engines = [make_engine(dims, max_batch=CAP_B)[0] for _ in range(world)]
    emulate_ipc(engines)
    cases = {c: _order_case(c, world, d, np.random.default_rng(zlib.crc32(b"%s/%d/%d" % (c.encode(), world, d))))
             for c in ("mixed", "quiet")}
    got = {c: [None] * world for c in cases}
    try:
        def rank(r):
            torch.cuda.set_device(0)
            e = engines[r]
            e.enable_table_sharding(None, ordered_exchange=True)
            assert e.get_option("ordered_exchange") == 1 and e.get_option("ordered_exchange_rows") == 0
            for c, lists in cases.items():
                for n in ("tok", "path"):
                    e.shard_grads[n].fill_(float(SENTINEL))
                torch.cuda.synchronize()
                dist.barrier()
                e.selftest_exchange_push(*lists["tok"][r], *lists["path"][r])
                dist.barrier()
                e.apply_scatter_inbox()
                torch.cuda.synchronize()
                got[c][r] = ({n: _np(e.shard_grads[n]) for n in ("tok", "path")}, e.get_option("ordered_exchange_rows"))
                dist.barrier()

        run_ranks(world, rank, group)
    finally:
        torch.cuda.synchronize()
        for e in engines:
            e.close()
    for c, lists in cases.items():
        differs = False
        for n, V in (("tok", T), ("path", P)):
            G, ref = OX.fold(lists[n], V)
            Gr, _ = OX.fold(lists[n], V, sender_order=range(world - 1, -1, -1))
            differs |= not np.array_equal(_bits(G[ref]), _bits(Gr[ref]))
            assert not ref.all() and not (np.signbit(G) & (G == 0)).any()      # no row everybody lists, no -0.0
            for o in range(world):
                want = np.full(got[c][o][0][n].shape, SENTINEL)
                mine = OX.shard(np.where(ref[:, None], G, SENTINEL), o, world)
                want[:len(mine)] = mine
                assert np.array_equal(_bits(got[c][o][0][n]), _bits(want)), (c, n, o)
        # the comparison tells the rank order from its reverse (two senders commute: only from three on)
        assert differs == (world > 2), (c, world)
        for s in range(world):
            distinct = sum(len(np.unique(lists[n][s][0])) for n in ("tok", "path"))
            assert got[c][s][1] == distinct, (c, s)
            assert distinct < sum(len(lists[n][s][0]) for n in ("tok", "path")) or distinct == 0


# ---- 2, 3. whole steps: reproducible, and still the right gradient ----------------------------------------------------------
B_GLOBAL = 512


def dup_batch(seed=31):
    """Ragged bags at the mid shape in which 60 % of the indices come from a few dozen hot rows."""
    src, pth, tgt, mask, target = O.synthetic_batch(MID, B_GLOBAL, seed=seed)
    rng = np.random.default_rng(seed)
    hot_tok = np.r_[0, rng.choice(np.arange(1, MID.token_vocab), 40)]
    hot_path = np.r_[0, rng.choice(np.arange(1, MID.path_vocab), 25)]
    for a, hot in ((src, hot_tok), (tgt, hot_tok), (pth, hot_path)):
        pick = rng.random(a.shape) < 0.6
        a[pick] = hot[rng.integers(0, len(hot), a.shape)][pick]
    lengths = rng.integers(1, MID.max_contexts + 1, B_GLOBAL)
    mask[...] = (np.arange(MID.max_contexts)[None, :] < lengths[:, None]).astype(np.float32)
    for a in (src, pth, tgt):
        a[mask == 0] = 0
    return src, pth, tgt, mask, target


def run_schedule(monkeypatch, dims, params, batch, world, schedule, math, steps=3, snap_steps=(1,), **trainer_args):
    """tests/test_gpu_emulated_ranks.run_schedule with the Trainer arguments of this option: `steps` steps of `schedule` on
    `world` emulated ranks, each on its 1/world of `batch`; snapshots (with parameters) after snap_steps, and the records
    every rank pushed in step 1."""
    import torch
    from code2vec_b200.engine import EngineDims, PathAttentionEngine
    from code2vec_b200.trainer import Trainer, make_fully_sharded_engine, target_row_block
    group = EmulatedGroup(world).install(monkeypatch)
    Bl = batch[0].shape[0] // world
    gd = EngineDims(dims.token_vocab, dims.path_vocab, dims.target_vocab, dims.embed_dim, dims.code_dim,
                    dims.max_contexts, Bl, 10)
    engines = []
    try:
        for r in range(world):
            with group.as_rank(r):
                if schedule == "fully_sharded":
                    e = make_fully_sharded_engine(gd, Bl, device=0)
                    r0, r1 = target_row_block(dims.target_vocab, r, world)
                    e.load_params(dict(params, tgt=params["tgt"][r0:r1]))
                else:
                    e = PathAttentionEngine(gd, device=0, training=True)
                    e.load_params(params)
            e.set_option("math_mode", math)
            e.set_option("profile", 1)
            engines.append(e)
        emulate_ipc(engines)
        out = [{"loss": []} for _ in engines]

        def rank(r):
            torch.cuda.set_device(0)
            e = engines[r]
            tr = Trainer(e, keep_prob=KEEP, seed=SEED, schedule=schedule, **trainer_args)
            assert tr.schedule == schedule and e.push_grads
            d = dev_batch(e, *(a[r * Bl:(r + 1) * Bl] for a in batch))
            for s in range(1, steps + 1):
                out[r]["loss"].append(float(tr.step_device(*d).cpu()[0]))
                torch.cuda.synchronize()
                if s == 1:
                    out[r]["records"] = e.get_option("ordered_exchange_rows")
                if s in snap_steps:
                    out[r]["step%d" % s] = _snapshot(e, tr, True)

        run_ranks(world, rank, group)
        return out, engines
    finally:
        torch.cuda.synchronize()
        for e in engines:
            e.close()


def _assert_same_bits(a, b, label):
    assert a.keys() == b.keys(), label
    for k in a:
        if isinstance(a[k], dict):
            _assert_same_bits(a[k], b[k], label + "/" + k)
        elif isinstance(a[k], np.ndarray):
            assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), label + "/" + k


@pytest.mark.parametrize("math", [0, 1, 2])
@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("schedule", ["table_sharded", "fully_sharded"])
def test_deterministic_steps_repeat_bit_for_bit_and_pass_the_float64_bounds(monkeypatch, schedule, world, math):
    params = O.init_params(MID, seed=4321)
    batch = dup_batch()
    label = "%s world=%d math=%d ordered" % (schedule, world, math)
    runs = [run_schedule(monkeypatch, MID, params, batch, world, schedule, math, steps=3, snap_steps=(1, 3),
                         deterministic=True, ordered_exchange=True) for _ in range(2)]
    (out, engines), (out2, _) = runs
    Bl = B_GLOBAL // world
    for r in range(world):
        assert out[r]["loss"] == out2[r]["loss"], (label, r)
        for s in (1, 3):
            a, b = (o[r]["step%d" % s] for o in (out, out2))
            _assert_same_bits({k: a[k] for k in a if k not in ("phases", "fallbacks")},
                              {k: b[k] for k in b if k not in ("phases", "fallbacks")}, "%s rank %d step %d" % (label, r, s))
        ph = out[r]["step1"]["phases"]
        assert ph.get("inbox_apply", 0) > 0 and ph.get("dx_scatter", 0) > 0 and not ph.get("peer_sort", 0), (label, ph)
        mine = [a[r * Bl:(r + 1) * Bl] for a in batch[:4]]
        assert out[r]["records"] == out2[r]["records"] == OX.pushed_records(*mine), (label, r)
        assert out[r]["records"] < 3 * int(mine[3].sum()) // 2, (label, r)      # far fewer records than live entries
    # step 1 is still the right gradient: the float64 per-element bounds of the plain push
    ref = reference(("ordered-dup", world), MID, params, batch, world)
    check_slots(out, engines, MID, schedule, world, ref, math, label)
    check_loss(out, schedule, ref, label)


# ---- 4. agreement with the plain push where order cannot matter --------------------------------------------------------
@pytest.mark.parametrize("math", [0, 1])
def test_ordered_route_equals_the_plain_push_when_no_row_repeats(monkeypatch, math):
    world, schedule, Bg = 2, "table_sharded", 128
    params = O.init_params(MID, seed=4321)
    src, pth, tgt, mask, target = O.synthetic_batch(MID, Bg, seed=9)
    rng = np.random.default_rng(9)
    n = Bg * MID.max_contexts
    tok = rng.permutation(MID.token_vocab)[:2 * n]
    src[...] = tok[:n].reshape(src.shape)
    tgt[...] = tok[n:].reshape(tgt.shape)
    pth[...] = rng.permutation(MID.path_vocab)[:n].reshape(pth.shape)
    batch = (src, pth, tgt, mask, target)
    ordered, _ = run_schedule(monkeypatch, MID, params, batch, world, schedule, math, steps=1, ordered_exchange=True)
    plain, _ = run_schedule(monkeypatch, MID, params, batch, world, schedule, math, steps=1, push_grads=True)
    for r in range(world):
        assert ordered[r]["records"] == 3 * int(mask[r * Bg // 2:(r + 1) * Bg // 2].sum()) and plain[r]["records"] == 0
        assert ordered[r]["loss"] == plain[r]["loss"]
        a, b = ordered[r]["step1"], plain[r]["step1"]
        _assert_same_bits({k: a[k] for k in ("shard_p", "shard_m", "shard_v")},
                          {k: b[k] for k in ("shard_p", "shard_m", "shard_v")}, "rank %d" % r)
        assert np.abs(a["shard_m"]["tok"]).max() > 0


# ---- 5. the options -------------------------------------------------------------------------------------------------------
DIMS = O.Dims(token_vocab=1001, path_vocab=501, target_vocab=1001, embed_dim=32, code_dim=96, max_contexts=20)


def _two_rank_shards(eng):
    """Both "ranks" of a two-rank sharding mapped onto this engine's own tables (enough to bind, and to run a forward)."""
    from code2vec_b200.engine import c2v_table_shards
    sp, sg = c2v_table_shards(), c2v_table_shards()
    for st, src in ((sp, eng.params), (sg, eng.grads)):
        st.world, st.rank = 2, 0
        for r in range(2):
            st.tok[r], st.path[r] = src["tok"].data_ptr(), src["path"].data_ptr()
    return sp, sg


def test_option_semantics():
    from code2vec_b200.engine import EngineError
    eng, _ = make_engine(DIMS, max_batch=64)
    assert eng.get_option("ordered_exchange") == 0 and eng.get_option("ordered_exchange_rows") == 0
    sp, sg = _two_rank_shards(eng)
    bind = lambda: eng.lib.c2v_bind_table_shards(eng.h, ctypes.byref(sp), ctypes.byref(sg), 0.5)
    with pytest.raises(EngineError) as ei:
        eng.set_option("ordered_exchange", 2)
    assert ei.value.code == -1
    # without the option both refusals of "deterministic" stand
    eng.set_option("deterministic", 1)
    assert bind() == -4
    eng.set_option("deterministic", 0)
    # with it, shards may be bound while deterministic is set ...
    eng.set_option("ordered_exchange", 1)
    eng.set_option("deterministic", 1)
    assert bind() == 0
    # ... and deterministic may be set while they are bound
    eng.set_option("deterministic", 0)
    eng.set_option("deterministic", 1)
    assert eng.get_option("deterministic") == 1
    with pytest.raises(EngineError) as ei:
        eng.set_option("ordered_exchange", 0)
    assert ei.value.code == -4 and "deterministic" in str(ei.value)
    assert eng.get_option("ordered_exchange") == 1
    # no inbox: the backward pass has nowhere to push
    batch = dev_batch(eng, *O.synthetic_batch(DIMS, 64, seed=3))
    for math in (0, 1):
        eng.set_option("math_mode", math)
        with pytest.raises(EngineError) as ei:
            eng.train_step(*batch, keep=1.0, seed=1, step=1)
        assert ei.value.code == -3 and "c2v_bind_scatter_inbox" in str(ei.value)
    eng.set_option("deterministic", 0)
    eng.set_option("ordered_exchange", 0)
    eng.close()


def test_trainer_still_refuses_deterministic_without_ordered_exchange(monkeypatch):
    from code2vec_b200.engine import EngineDims
    from code2vec_b200.trainer import Trainer, make_fully_sharded_engine
    group = EmulatedGroup(2).install(monkeypatch)
    gd = EngineDims(DIMS.token_vocab, DIMS.path_vocab, DIMS.target_vocab, DIMS.embed_dim, DIMS.code_dim, DIMS.max_contexts, 32, 10)
    with group.as_rank(0):
        e = make_fully_sharded_engine(gd, 32, device=0)
        try:
            for push in (False, True):
                with pytest.raises(ValueError, match="pass ordered_exchange=True"):
                    Trainer(e, schedule="fully_sharded", deterministic=True, push_grads=push)
        finally:
            e.close()
