"""Prediction against a row-sharded target table (c2v_topk_partial + c2v_topk_merge, Trainer.predict) against c2v_topk of
one engine that holds the whole table.

Each rank's engine holds one contiguous block of target rows (trainer.target_row_block).  idx must equal the whole-table
engine's bit for bit, and so must val for normalize 0 and 1 (NaN by bit pattern); for normalize 2 the normaliser is summed
in another order, so val agrees to 2e-6 relative.  The edges: a partial last column tile (Y = 1537), blocks smaller than k
(Y = 37 on 8 ranks, the last block has 2 rows), k = 20 (the logits-slab route), exact ties placed inside one partial slot,
across the two slots of a tile, across tiles and across a rank boundary, an all-masked bag (NaN code vector), and the
production width (Y = 261,246 on 8 ranks).  Trainer.predict runs on 1 (allow_single_rank), 2, 4 and 8 ranks emulated on
one GPU (tests/emulated_ranks.py), on training=False engines and after two training steps."""
import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests.emulated_ranks import EmulatedGroup, emulate_ipc, run_ranks
from tests.util import dev_batch

pytestmark = pytest.mark.gpu

SMALL = O.Dims(token_vocab=2003, path_vocab=1009, target_vocab=1537, embed_dim=64, code_dim=128, max_contexts=20)
B_GLOBAL = 320
NORM2_RTOL = 2e-6


def _engine_dims(dims, Y, max_batch, top_k):
    from code2vec_b200.engine import EngineDims
    return EngineDims(dims.token_vocab, dims.path_vocab, Y, dims.embed_dim, dims.code_dim, dims.max_contexts, max_batch,
                      top_k)


def whole_engine(dims, params, Bt, math, top_k=10):
    from code2vec_b200.engine import PathAttentionEngine
    e = PathAttentionEngine(_engine_dims(dims, dims.target_vocab, Bt, top_k), device=0, training=False)
    e.load_params(params)
    e.set_option("math_mode", math)
    return e


def assert_same(idx, val, ref_idx, ref_val, normalize, label):
    import torch
    assert torch.equal(idx, ref_idx), (label, (idx != ref_idx).nonzero()[:5].tolist())
    if normalize < 2:
        same = val.view(torch.int32) == ref_val.view(torch.int32)
        assert bool(same.all()), (label, val[~same][:5].tolist(), ref_val[~same][:5].tolist())
    else:
        np.testing.assert_allclose(val.cpu().numpy(), ref_val.cpu().numpy(), rtol=NORM2_RTOL, atol=0, equal_nan=True,
                                   err_msg=label)


# ---- the two entry points, ranks run one after another on one stream ------------------------------------------------

class RankBlocks:
    """`world` engines, rank r holding target rows target_row_block(Y, r, world) of `tgt`."""

    def __init__(self, dims, params, world, Bt, math, top_k):
        from code2vec_b200.engine import PathAttentionEngine
        from code2vec_b200.trainer import target_row_block
        self.world, self.Bt = world, Bt
        self.k = min(top_k, dims.target_vocab)
        self.engines, self.row0 = [], []
        for r in range(world):
            r0, r1 = target_row_block(dims.target_vocab, r, world)
            e = PathAttentionEngine(_engine_dims(dims, r1 - r0, Bt, top_k), device=0, training=False)
            e.load_params(dict(params, tgt=params["tgt"][r0:r1]))
            e.set_option("math_mode", math)
            self.engines.append(e)
            self.row0.append(r0)

    def topk(self, code_all, normalize):
        import torch
        from code2vec_b200.trainer import shard_bounds
        W, Bt, k, dev = self.world, self.Bt, self.k, code_all.device
        idx = torch.empty((W, Bt, k), dtype=torch.int32, device=dev)
        val = torch.empty((W, Bt, k), dtype=torch.float32, device=dev)
        full = normalize == 2
        maxes = torch.empty((W, Bt), dtype=torch.float32, device=dev) if full else None
        sums = torch.empty((W, Bt), dtype=torch.float32, device=dev) if full else None
        for r, e in enumerate(self.engines):
            e.topk_partial(code_all, self.row0[r], k, idx[r], val[r], maxes[r] if full else None, sums[r] if full else None)
        out_i = torch.empty((Bt, k), dtype=torch.int32, device=dev)
        out_v = torch.empty((Bt, k), dtype=torch.float32, device=dev)
        for r, e in enumerate(self.engines):      # each rank merges its own examples
            lo, hi = shard_bounds(Bt, r, W)
            e.topk_merge(idx, val, maxes, sums, lo, hi - lo, normalize, out_i[lo:hi], out_v[lo:hi])
        return out_i, out_v

    def close(self):
        for e in self.engines:
            e.close()


def code_vectors(D, Bt, seed, nan_rows=(5,), direction=None):
    """Code vectors [Bt, D] on the device: normal, row(s) `nan_rows` all NaN (a bag with no valid context)."""
    import torch
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((Bt, D)).astype(np.float32)
    if direction is not None:
        v = (direction[None, :] + 0.3 * v).astype(np.float32)
    v[list(nan_rows)] = np.nan
    return torch.from_numpy(v).cuda()


def run_blocks(dims, params, world, math, normalizes, Bt=B_GLOBAL, top_k=10, code=None, label=""):
    import torch
    code = code_vectors(dims.code_dim, Bt, seed=11) if code is None else code
    ref = whole_engine(dims, params, Bt, math, top_k)
    blocks = RankBlocks(dims, params, world, Bt, math, top_k)
    try:
        out = {}
        for n in normalizes:
            want = ref.topk(code, n)
            got = blocks.topk(code, n)
            torch.cuda.synchronize()
            assert_same(*got, *want, n, "%s world=%d math=%d normalize=%d" % (label, world, math, n))
            out[n] = want
        return out
    finally:
        torch.cuda.synchronize()
        blocks.close()
        ref.close()


@pytest.mark.parametrize("math", [0, 1, 2])
@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_partial_last_tile(world, math):
    params = O.init_params(SMALL, seed=4321)
    out = run_blocks(SMALL, params, world, math, (0, 1, 2), label="Y=1537")
    idx0 = out[0][0].cpu().numpy()
    assert (idx0[5] == 2 ** 31 - 1).all() and (idx0[:5] < SMALL.target_vocab).all()      # the NaN row pads, the others do not


@pytest.mark.parametrize("math", [0, 1, 2])
def test_blocks_smaller_than_k(math):
    from code2vec_b200.trainer import target_row_block
    dims = O.Dims(token_vocab=2003, path_vocab=1009, target_vocab=37, embed_dim=64, code_dim=128, max_contexts=20)
    assert target_row_block(37, 7, 8) == (35, 37)
    run_blocks(dims, O.init_params(dims, seed=99), 8, math, (0, 1, 2), label="Y=37")


@pytest.mark.parametrize("math", [0, 1, 2])
@pytest.mark.parametrize("world", [2, 8])
def test_k20_slab_route(world, math):
    run_blocks(SMALL, O.init_params(SMALL, seed=4321), world, math, (0, 1, 2), top_k=20, label="k=20")


@pytest.mark.parametrize("normalize", [0, 1, 2])
@pytest.mark.parametrize("math", [0, 1, 2])
def test_exact_ties(math, normalize):
    """Target rows 3, 40, 70, 300, 768 and 769 are one vector that dominates every logit row: columns 3 and 70 share a
    partial slot (quarters 0 and 2 of tile 0), 3 and 40 are the two slots of one tile, 300 is in another tile, and 768 |
    769 straddle the boundary of the two ranks' blocks.  The six equal logits must come out in id order."""
    params = O.init_params(SMALL, seed=4321)
    rng = np.random.default_rng(5)
    w = rng.standard_normal(SMALL.code_dim).astype(np.float32)
    dup = [3, 40, 70, 300, 768, 769]
    params["tgt"][dup] = (w / np.linalg.norm(w)).astype(np.float32)
    code = code_vectors(SMALL.code_dim, B_GLOBAL, seed=6, direction=w)
    out = run_blocks(SMALL, params, 2, math, (normalize,), code=code, label="ties")
    idx, val = (t.cpu().numpy() for t in out[normalize])
    ok = np.ones(B_GLOBAL, dtype=bool)
    ok[5] = False
    assert (idx[ok, :6] == dup).mean() > 0.95, idx[:3]
    assert (val[ok, 0] == val[ok, 5]).mean() > 0.95


@pytest.mark.parametrize("math", [1, 2])
def test_production_width_world8(math):
    """Y = 261,246 on 8 ranks (blocks of 32,656 rows), the global batch of 8 x 128 examples, D = 384."""
    dims = O.Dims(token_vocab=101, path_vocab=101, target_vocab=261246, embed_dim=128, code_dim=384, max_contexts=8)
    rng = np.random.default_rng(4321)
    lim = np.float32((3.0 / dims.code_dim) ** 0.5)
    params = {"tok": np.zeros((dims.token_vocab, dims.embed_dim), np.float32),
              "path": np.zeros((dims.path_vocab, dims.embed_dim), np.float32),
              "tgt": rng.uniform(-lim, lim, (dims.target_vocab, dims.code_dim)).astype(np.float32),
              "W": np.zeros((3 * dims.embed_dim, dims.code_dim), np.float32),
              "a": np.zeros(dims.code_dim, np.float32)}
    run_blocks(dims, params, 8, math, (0, 1, 2), Bt=1024, code=code_vectors(dims.code_dim, 1024, seed=8),
               label="Y=261246")


# ---- Trainer.predict on emulated ranks --------------------------------------------------------------------------------

def _interleave(shards, n_rows, world):
    """Global table rows from row-interleaved shards: row r lives on rank r % world at local row r // world."""
    full = np.zeros((n_rows, shards[0].shape[1]), dtype=shards[0].dtype)
    for r in range(world):
        full[r::world] = shards[r][:len(range(r, n_rows, world))]
    return full


def predict_on_ranks(monkeypatch, dims, params, batch, world, math, normalizes, training=False, steps=0):
    """Fully sharded engines for `world` emulated ranks loaded with `params`; `steps` training steps (training=True), then
    Trainer.predict of each rank's 1/world of `batch` for every normalize.  Returns ({normalize: (idx, val, code)} with the
    ranks' rows concatenated, the global parameters the engines hold at predict time)."""
    import torch
    from code2vec_b200.engine import EngineDims
    from code2vec_b200.trainer import Trainer, make_fully_sharded_engine, target_row_block
    group = EmulatedGroup(world).install(monkeypatch)
    Bl = B_GLOBAL // world
    gd = EngineDims(dims.token_vocab, dims.path_vocab, dims.target_vocab, dims.embed_dim, dims.code_dim,
                    dims.max_contexts, Bl, 10)
    engines = []
    try:
        for r in range(world):
            with group.as_rank(r):
                e = make_fully_sharded_engine(gd, Bl, device=0, training=training)
                r0, r1 = target_row_block(dims.target_vocab, r, world)
                e.load_params(dict(params, tgt=params["tgt"][r0:r1]))
            e.set_option("math_mode", math)
            engines.append(e)
        emulate_ipc(engines)
        res = [dict() for _ in range(world)]

        def rank(r):
            torch.cuda.set_device(0)
            e = engines[r]
            tr = Trainer(e, keep_prob=0.75, seed=7, schedule="fully_sharded", allow_single_rank=(world == 1))
            assert tr.schedule == "fully_sharded"
            d = dev_batch(e, *(a[r * Bl:(r + 1) * Bl] for a in batch))
            for _ in range(steps):
                tr.step_device(*d)
            for n in normalizes:
                idx, val, code = tr.predict(*d[:4], normalize=n)
                torch.cuda.synchronize()
                res[r][n] = tuple(t.clone() for t in (idx, val, code))
            res[r]["tgt"] = e.params["tgt"].cpu().numpy().copy()
            res[r]["shards"] = {n: e.shard_params[n].cpu().numpy().copy() for n in ("tok", "path")}
            res[r]["Wa"] = {n: e.params[n].cpu().numpy().copy() for n in ("W", "a")}

        run_ranks(world, rank, group)
        torch.cuda.synchronize()
        out = {n: tuple(torch.cat([res[r][n][i] for r in range(world)]) for i in range(3)) for n in normalizes}
        held = {"tgt": np.concatenate([res[r]["tgt"] for r in range(world)]), **res[0]["Wa"]}
        for n, V in (("tok", dims.token_vocab), ("path", dims.path_vocab)):
            held[n] = _interleave([res[r]["shards"][n] for r in range(world)], V, world)
        return out, held
    finally:
        torch.cuda.synchronize()
        for e in engines:
            e.close()


def check_against_whole(out, params, batch, math, label):
    """Every rank's (idx, val, code) against forward + topk of one whole-model engine on the global batch, and the top-k
    against that engine's c2v_topk on the gathered code vectors."""
    import torch
    ref = whole_engine(SMALL, params, B_GLOBAL, math)
    try:
        d = dev_batch(ref, *batch)
        code, _ = ref.forward(*d[:4], want_attention=False)
        for n, (idx, val, got_code) in out.items():
            lab = "%s normalize=%d" % (label, n)
            assert torch.equal(got_code.view(torch.int32), code.view(torch.int32)), lab
            assert_same(idx, val, *ref.topk(got_code, n), n, lab + " (gathered code vectors)")
            assert_same(idx, val, *ref.topk(code, n), n, lab)
        torch.cuda.synchronize()
    finally:
        ref.close()


def small_batch():
    src, pth, tgt, mask, target = O.synthetic_batch(SMALL, B_GLOBAL, seed=2024)
    mask[7] = 0          # an all-masked bag: NaN code vector, padded predictions
    return src, pth, tgt, mask, target


@pytest.mark.parametrize("math", [0, 1, 2])
@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_trainer_predict(monkeypatch, world, math):
    params = O.init_params(SMALL, seed=4321)
    batch = small_batch()
    out, _ = predict_on_ranks(monkeypatch, SMALL, params, batch, world, math, (0, 1, 2))
    assert (out[0][0][7].cpu().numpy() == 2 ** 31 - 1).all()
    check_against_whole(out, params, batch, math, "predict world=%d math=%d" % (world, math))


@pytest.mark.parametrize("math", [1, 2])
def test_trainer_predict_after_training(monkeypatch, math):
    """Two fully sharded training steps, predict on the trained engines; then fresh training=False engines loaded with
    the parameters the trained ones hold must predict the same."""
    world = 2
    params = O.init_params(SMALL, seed=4321)
    batch = small_batch()
    out, held = predict_on_ranks(monkeypatch, SMALL, params, batch, world, math, (0, 2), training=True, steps=2)
    assert not np.array_equal(held["tgt"], params["tgt"])            # the steps moved the target table
    check_against_whole(out, held, batch, math, "trained world=%d math=%d" % (world, math))
    out2, _ = predict_on_ranks(monkeypatch, SMALL, held, batch, world, math, (0, 2))
    for n in (0, 2):
        for a, b in zip(out[n], out2[n]):
            assert np.array_equal(a.cpu().numpy().view(np.int32), b.cpu().numpy().view(np.int32)), n
