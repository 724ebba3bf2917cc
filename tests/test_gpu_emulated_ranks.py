"""The multi-rank training schedules against the float64 reference, with 2, 4 and 8 ranks emulated on one GPU.

`world` engines live on one device in one process, one thread per rank (tests/emulated_ranks.py): the collectives are
done in software and CUDA IPC is replaced by the owners' own pointers, so every kernel is the one a multi-GPU run
launches -- the row interleave of the sharded tables and its 1/world scatter scale, the row-offset head of the fully
sharded schedule with classes on other ranks and a short last target block, the push-based gradient inbox and the
page-sorted peer accesses.

The multi-rank schedules run dense Adam from zero slots and the fully sharded one never writes the target gradient, so
the gradients of step 1 are read through the Adam slots (m / (1 - beta1) and v, test_gpu_reference64.check_adam_slots)
against reference64.train_step64 on the global batch, whose dropout mask is the row-wise concatenation of the ranks' own
masks (seed + rank, local rows).  A first-step Adam update is about lr * sign(g), so comparing parameters is blunt to a
gradient's scale; the negative controls at the end show that these checks see a wrong scale, a 1 % error in the dv
reduce-scatter and a skipped inbox fold."""
import types

import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests import reference64 as R
from tests.emulated_ranks import EmulatedGroup, emulate_ipc, run_ranks
from tests.test_gpu_reference64 import LOSS_TOL, PROD, SLICE, TAU, check_adam_slots, report
from tests.util import dev_batch

pytestmark = pytest.mark.gpu

MID = O.Dims(token_vocab=20011, path_vocab=10007, target_vocab=5003, embed_dim=128, code_dim=384, max_contexts=50)
B_GLOBAL = 512
KEEP = 0.75
SEED = 0x5EED
BETA1 = 0.9
C1 = float(np.float32(1.0) - np.float32(BETA1))

_cache = {}


@pytest.fixture(scope="module", autouse=True)
def _release_references():
    yield
    _cache.clear()


def rank_dropout(dims, world, b_local, step, keep=KEEP):
    """The dropout mask of the global batch: rank r draws rows of its local batch with seed SEED + r."""
    if keep >= 1.0:
        return None
    return np.concatenate([O.dropout_keep_mask(SEED + r, step, b_local * dims.max_contexts, dims.ctx_dim, keep)
                           for r in range(world)])


def mid_batch(seed=2024):
    return O.synthetic_batch(MID, B_GLOBAL, seed=seed)      # ragged bags


def reference(key, dims, params, batch, world, step=1, keep=KEEP):
    if key not in _cache:
        dm = rank_dropout(dims, world, batch[0].shape[0] // world, step, keep)
        _cache[key] = R.train_step64(params, *batch, keep=keep, dropout_mask=dm)
        _cache[key].extra["dropout_mask"] = dm
    return _cache[key]


# ---- running a schedule on emulated ranks ------------------------------------------------------------------------

def _np(t):
    return t.detach().cpu().numpy().copy()


def _snapshot(e, tr, params):
    s = {"flat_m": _np(e.flat_m), "flat_v": _np(e.flat_v)}
    if getattr(e, "table_world", 1) > 1:
        s["shard_m"] = {n: _np(e.shard_m[n]) for n in ("tok", "path")}
        s["shard_v"] = {n: _np(e.shard_v[n]) for n in ("tok", "path")}
    if params:
        s["flat_p"] = _np(e.flat_params)
        if getattr(e, "table_world", 1) > 1:
            s["shard_p"] = {n: _np(e.shard_params[n]) for n in ("tok", "path")}
    if tr.schedule == "fully_sharded":
        s["fs"] = {k: _np(tr._fs[k]) for k in ("v_all", "lse", "dv_part")}
    s["fallbacks"] = e.get_option("exp_slab_fallbacks")
    s["phases"] = {k: n for k, (_, n) in e.phase_stats(reset=True).items()}
    return s


def run_schedule(monkeypatch, dims, params, batch, world, schedule, math, steps=3, push=False, sort=None, keep=KEEP,
                 setup=None, before_step=None, snap_steps=(1,), params_at=(), group=None):
    """`steps` Trainer steps of `schedule` on `world` emulated ranks, each on its 1/world of `batch` (the same batch every
    step).  Returns (per-rank dicts: "loss" list, "step<s>" snapshots, "final" parameters, engines' workspace bytes)."""
    import torch
    from code2vec_b200.engine import EngineDims, PathAttentionEngine
    from code2vec_b200.trainer import Trainer, make_fully_sharded_engine, target_row_block
    group = group or EmulatedGroup(world)
    group.install(monkeypatch)
    B = batch[0].shape[0]
    Bl = B // world
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
            if sort is not None:
                e.set_option("sort_peer_access", sort)
            engines.append(e)
        emulate_ipc(engines)
        out = [{"loss": [], "workspace": int(e.workspace.numel())} for e in engines]

        def rank(r):
            torch.cuda.set_device(0)
            e = engines[r]
            tr = Trainer(e, keep_prob=keep, seed=SEED, schedule=schedule, push_grads=push)
            assert tr.schedule == schedule
            assert bool(getattr(e, "push_grads", False)) == push
            if setup:
                setup(r, e, tr)
            lo, hi = r * Bl, (r + 1) * Bl
            d = dev_batch(e, *(a[lo:hi] for a in batch))
            for s in range(1, steps + 1):
                if before_step:
                    before_step(s, r, e, tr)
                out[r]["loss"].append(float(tr.step_device(*d).cpu()[0]))
                torch.cuda.synchronize()
                if s in snap_steps:
                    out[r]["step%d" % s] = _snapshot(e, tr, s in params_at)
            out[r]["final"] = {"flat_p": _np(e.flat_params)}
            if getattr(e, "table_world", 1) > 1:
                out[r]["final"]["shard_p"] = {n: _np(e.shard_params[n]) for n in ("tok", "path")}

        run_ranks(world, rank, group)
        return out, engines
    finally:
        torch.cuda.synchronize()
        for e in engines:
            e.close()


def _interleave(shards, n_rows, world):
    """Global table rows from row-interleaved shards: row r lives on rank r % world at local row r // world."""
    full = np.zeros((n_rows, shards[0].shape[1]), dtype=shards[0].dtype)
    for r in range(world):
        full[r::world] = shards[r][:len(range(r, n_rows, world))]
    return full


def assemble(out, engines, dims, schedule, world, step, key):
    """Global tensors {tok, path, tgt, W, a} of snapshot `key` ("m", "v" or "p") after `step`."""
    from code2vec_b200.trainer import target_row_block
    snaps = [o["step%d" % step] if step else o["final"] for o in out]
    flats = [s["flat_" + key] for s in snaps]
    e0 = engines[0]
    layout, total = e0.flat_layout()
    shapes = e0.dims.shapes()
    g = flats[0].copy()
    if schedule in ("sharded", "table_sharded") and key != "p":      # sliced Adam: rank r owns 1/world of each bucket
        buckets = e0.bucket_bounds() if schedule == "sharded" else e0.bucket_bounds()[:1]
        for lo, hi in buckets:
            n = (hi - lo) // world
            for r in range(world):
                g[lo + r * n:lo + (r + 1) * n] = flats[r][lo + r * n:lo + (r + 1) * n]
    res = {k: g[off:off + n].reshape(shapes[k]) for k, off, n in layout}
    if schedule in ("table_sharded", "fully_sharded"):
        sk = "shard_" + key
        for name, V in (("tok", dims.token_vocab), ("path", dims.path_vocab)):
            res[name] = _interleave([s[sk][name] for s in snaps], V, world)
    if schedule == "fully_sharded":
        blocks = []
        for r in range(world):
            r0, r1 = target_row_block(dims.target_vocab, r, world)
            off, n = [(o, n) for k, o, n in engines[r].flat_layout()[0] if k == "tgt"][0]
            blocks.append(flats[r][off:off + n].reshape(r1 - r0, dims.code_dim))
        res["tgt"] = np.concatenate(blocks)
    return res


def check_slots(out, engines, dims, schedule, world, ref, math, label, step=1):
    """Step-1 gradients through the Adam slots, element by element and by slices."""
    import torch
    m, v = (assemble(out, engines, dims, schedule, world, step, k) for k in ("m", "v"))
    slots = types.SimpleNamespace(adam_m={k: torch.from_numpy(np.ascontiguousarray(m[k])) for k in O.PARAM_NAMES},
                                  adam_v={k: torch.from_numpy(np.ascontiguousarray(v[k])) for k in O.PARAM_NAMES})
    worst = check_adam_slots(slots, ref, math, O.PARAM_NAMES, label)
    got = {k: m[k].astype(np.float64) / C1 for k in O.PARAM_NAMES}
    worst.update({"slice:" + k: e for k, e in R.check_slices(got, ref, SLICE[math]).items()})
    return worst


def check_loss(out, schedule, ref, label, target=None):
    target = ref.loss if target is None else target
    losses = np.array([o["loss"][0] for o in out])
    if schedule == "fully_sharded":          # the global loss, the same bits on every rank
        assert np.all(losses == losses[0]), (label, losses)
        got = float(losses[0])
    else:                                    # each rank's local mean
        got = float(losses.astype(np.float64).mean())
    assert abs(got - target) < LOSS_TOL, (label, got, target, ref.loss)
    return abs(got - target)


def check_fs_phases(out, ref, params, math, label):
    """The fully sharded step's intermediates: gathered code vectors, the combined log-sum-exp, the summed dv partials."""
    fs = [o["step1"]["fs"] for o in out]
    tau = TAU[math]
    worst = {"fs:v_all": R.check_elementwise(label + " v_all", fs[0]["v_all"], ref.vals["v"], ref.mags["v"], tau)}
    Y = np.asarray(params["tgt"], dtype=np.float64)
    lse = ref.extra["lse"]
    M_lse = ref.mags["v"] @ np.abs(Y).max(axis=0) + np.abs(lse) + 1.0     # bounds max_y M(s) and the exp / log rounding
    worst["fs:lse"] = R.check_elementwise(label + " lse", fs[0]["lse"], lse, M_lse, tau)
    for o in fs[1:]:
        assert np.array_equal(o["v_all"], fs[0]["v_all"]) and np.array_equal(o["lse"], fs[0]["lse"]), label
    dv = np.sum([o["dv_part"].astype(np.float64) for o in fs], axis=0)
    worst["fs:dv"] = R.check_elementwise(label + " dv", dv, ref.vals["dv"], ref.mags["dv"], tau)
    worst["slice:dv"] = R.normwise(dv, ref.vals["dv"])
    assert worst["slice:dv"] <= SLICE[math], (label, worst["slice:dv"])
    return worst


def check_replicas(out, engines, schedule, world, label):
    """After the last step: W and a bit-identical on every rank, and the target table wherever it is replicated."""
    names = ("W", "a") if schedule == "fully_sharded" else ("W", "a", "tgt")
    if schedule in ("allreduce", "sharded"):
        names = O.PARAM_NAMES

    def views(r):          # per rank: the fully sharded engines' flat layouts differ with their target blocks
        flat = out[r]["final"]["flat_p"]
        return {k: flat[off:off + n] for k, off, n in engines[r].flat_layout()[0] if k in names}
    first = views(0)
    for r in range(1, world):
        for k, x in views(r).items():
            assert np.array_equal(first[k], x), "%s: rank %d diverged on %s" % (label, r, k)


def assert_paths(out, math, sort_expected, push_expected, label):
    for r, o in enumerate(out):
        ph = o["step1"]["phases"]
        assert (ph.get("peer_sort", 0) > 0) == sort_expected, (label, r, ph)
        assert (ph.get("inbox_apply", 0) > 0) == push_expected, (label, r, ph)


def run_and_check(monkeypatch, schedule, world, math, push=False, sort=None, batch=None, params=None, key=None,
                  label=None, fallbacks="none"):
    params = O.init_params(MID, seed=4321) if params is None else params
    batch = mid_batch() if batch is None else batch
    key = key or ("mid", world)
    ref = reference(key, MID, params, batch, world)
    label = label or "%s world=%d math=%d%s%s" % (schedule, world, math, " push" if push else "",
                                                   "" if sort is None else " sort=%d" % sort)
    out, engines = run_schedule(monkeypatch, MID, params, batch, world, schedule, math, push=push, sort=sort)
    worst = check_slots(out, engines, MID, schedule, world, ref, math, label)
    tf32_loss = None
    if fallbacks == "some" and math == 1:
        tf32_loss = R.tf32_model_loss(params, *batch, keep=KEEP, dropout_mask=ref.extra["dropout_mask"])
    worst["loss"] = check_loss(out, schedule, ref, label, tf32_loss)
    if schedule == "fully_sharded":
        worst.update(check_fs_phases(out, ref, params, math, label))
        fb = [o["step1"]["fallbacks"] for o in out]
        if fallbacks == "none" or math == 0:
            assert fb == [0] * world, (label, fb)
        else:
            assert any(fb) and not all(fb), (label, fb)
    tc = math != 0 and schedule in ("table_sharded", "fully_sharded")
    assert_paths(out, math, sort_expected=tc and (push or sort == 2), push_expected=tc and push, label=label)
    check_replicas(out, engines, schedule, world, label)
    report(label, worst)
    return worst


# ---- 1. every schedule at the mid shape ------------------------------------------------------------------------------

@pytest.mark.parametrize("math", [0, 1, 2])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_fully_sharded(monkeypatch, world, math):
    run_and_check(monkeypatch, "fully_sharded", world, math)


@pytest.mark.parametrize("math", [0, 2])
@pytest.mark.parametrize("world", [2, 8])
def test_table_sharded(monkeypatch, world, math):
    run_and_check(monkeypatch, "table_sharded", world, math)


@pytest.mark.parametrize("math", [0, 2])
@pytest.mark.parametrize("schedule", ["sharded", "allreduce"])
def test_replicated_tables(monkeypatch, schedule, math):
    run_and_check(monkeypatch, schedule, 2, math)


@pytest.mark.parametrize("world", [2, 8])
@pytest.mark.parametrize("schedule", ["table_sharded", "fully_sharded"])
def test_push_grads(monkeypatch, schedule, world):
    run_and_check(monkeypatch, schedule, world, 2, push=True)


@pytest.mark.parametrize("schedule,math", [("fully_sharded", 1), ("fully_sharded", 2), ("table_sharded", 2)])
def test_sorted_peer_access(monkeypatch, schedule, math):
    run_and_check(monkeypatch, schedule, 4, math, sort=2)


# ---- 2. edges of the fully sharded head --------------------------------------------------------------------------

def _blocks(world):
    from code2vec_b200.trainer import target_row_block
    return [target_row_block(MID.target_vocab, r, world) for r in range(world)]


@pytest.mark.parametrize("math", [1, 2])
@pytest.mark.parametrize("case", ["last_block", "block_edges", "one_block_out_of_window"])
def test_fully_sharded_edges(monkeypatch, case, math):
    world = 4
    blocks = _blocks(world)
    assert blocks[-1][1] - blocks[-1][0] < blocks[0][1] - blocks[0][0]          # a short last block
    src, pth, tgt, mask, target = mid_batch(seed=77)
    params = O.init_params(MID, seed=4321)
    fallbacks = "none"
    if case == "last_block":           # every class on rank 3: c_b = 0 for every example on ranks 0..2
        target = np.random.default_rng(5).integers(blocks[-1][0], blocks[-1][1], size=B_GLOBAL).astype(np.int32)
    elif case == "block_edges":        # r0 - 1, r0 and r1 - 1 of every block
        edges = sorted({x for r0, r1 in blocks for x in (r0 - 1, r0, r1 - 1) if x >= 0})
        target = np.resize(np.array(edges, dtype=np.int32), B_GLOBAL)
    else:
        # rank 1's block scaled until its largest logit is 74.5: there exp(s - c_b) with c_b = 0 exceeds 1e30 and rank 1
        # falls back, while on the other ranks exp(s) stays in the window and c_b - lse stays above -80, so they do not
        r0, r1 = blocks[1]
        dm = rank_dropout(MID, world, B_GLOBAL // world, 1)
        v = R.train_step64(params, src, pth, tgt, mask, target, keep=KEEP, dropout_mask=dm).vals["v"]
        f = np.float32(74.5 / (v @ params["tgt"][r0:r1].astype(np.float64).T).max())
        params["tgt"][r0:r1] = (params["tgt"][r0:r1] * f).astype(np.float32)
        fallbacks = "some"
    batch = (src, pth, tgt, mask, target)
    run_and_check(monkeypatch, "fully_sharded", world, math, batch=batch, params=params, key=("edge", case, world),
                  label="fully_sharded edge=%s world=%d math=%d" % (case, world, math), fallbacks=fallbacks)


def test_push_grads_survive_a_math_mode_change(monkeypatch):
    """push_grads, step 1 in 3xTF32 (rows pushed into the inbox and folded), step 2 in fp32 (the SIMT scatter red.adds
    straight into the shards and pushes nothing).  Step 2's fold must add nothing: its gradients, m2 - beta1 m1 over
    1 - beta1, against a float64 step from the parameters step 1 left."""
    world, schedule = 2, "table_sharded"
    params = O.init_params(MID, seed=4321)
    batch = mid_batch()
    ref1 = reference(("mid", world), MID, params, batch, world)

    def before_step(s, r, e, tr):
        if s == 2:
            e.set_option("math_mode", 0)

    out, engines = run_schedule(monkeypatch, MID, params, batch, world, schedule, 2, steps=2, push=True,
                                before_step=before_step, snap_steps=(1, 2), params_at=(1,))
    label = "push math 2 -> 0"
    worst = check_slots(out, engines, MID, schedule, world, ref1, 2, label + " step 1")
    p1 = {k: np.ascontiguousarray(x, dtype=np.float32) for k, x in assemble(out, engines, MID, schedule, world, 1, "p").items()}
    ref2 = R.train_step64(p1, *batch, keep=KEEP, dropout_mask=rank_dropout(MID, world, B_GLOBAL // world, 2))
    m1, m2 = (assemble(out, engines, MID, schedule, world, s, "m") for s in (1, 2))
    b1 = float(np.float32(BETA1))
    for k in O.PARAM_NAMES:
        a1, a2 = m1[k].astype(np.float64), m2[k].astype(np.float64)
        g2 = (a2 - b1 * a1) / C1
        # m2 = fl(beta1 m1 + (1 - beta1) g2): its rounding, seen through the division by 1 - beta1
        M = ref2.mags[k] + 2.0 ** -22 * (b1 * np.abs(a1) + np.abs(a2)) / C1 / TAU[0]
        worst["g2:" + k] = R.check_elementwise(label + " step 2 " + k, g2, ref2.vals[k], M, TAU[0])
    assert out[0]["step2"]["phases"].get("inbox_apply", 0) > 0       # the fold ran after the fp32 step as well
    report(label, worst)


# ---- 3. production width ---------------------------------------------------------------------------------------------

PROD_B = 1024
# the large model's widths (d = 256, D = 768, Y = 261,246; bench.py --workload large) with token / path tables reduced
# 10x, so that eight engines share one GPU
LARGE_RED = O.Dims(token_vocab=300001, path_vocab=200001, target_vocab=261246, embed_dim=256, code_dim=768,
                   max_contexts=200)
WIDTHS = {"java14m": (PROD, PROD_B), "large": (LARGE_RED, 512)}


@pytest.mark.parametrize("math", [1, 2])
@pytest.mark.parametrize("shape", ["java14m", "large"])
def test_production_width_fully_sharded_world8(monkeypatch, shape, math):
    world = 8
    dims, B = WIDTHS[shape]
    key = ("prod", shape)
    if key not in _cache:            # one shape's reference at a time (about 2 GB for java14m, 5 GB for large)
        for k in [k for k in _cache if k[0] in ("prod", "prod-inputs")]:
            del _cache[k]
        _cache[("prod-inputs", shape)] = (O.init_params(dims, seed=4321), O.synthetic_batch(dims, B, seed=1234))
    params, batch = _cache[("prod-inputs", shape)]
    ref = reference(key, dims, params, batch, world)
    label = "%s fully_sharded world=8 math=%d" % (shape, math)
    out, engines = run_schedule(monkeypatch, dims, params, batch, world, "fully_sharded", math, steps=1)
    print("workspace bytes, 8 engines: %d (%.2f GB)" % (sum(o["workspace"] for o in out),
                                                          sum(o["workspace"] for o in out) / 1e9))
    worst = check_slots(out, engines, dims, "fully_sharded", world, ref, math, label)
    worst["loss"] = check_loss(out, "fully_sharded", ref, label)
    worst.update(check_fs_phases(out, ref, params, math, label))
    assert [o["step1"]["fallbacks"] for o in out] == [0] * world
    report(label, worst)


# ---- 4. negative controls --------------------------------------------------------------------------------------------

def _worst_slot_ratio(out, engines, schedule, world, ref, names):
    m = assemble(out, engines, MID, schedule, world, 1, "m")
    return max(R.err_ratio(m[k].astype(np.float64) / C1, ref.vals[k], ref.mags[k])[0] for k in names)


def test_control_one_rank_with_the_scatter_scale_applied_twice(monkeypatch):
    """table_sharded, world 2: rank 1 scatters with 1/4 instead of the 1/2 the Trainer binds (1/world applied twice)."""
    world, schedule, math = 2, "table_sharded", 2
    params, batch = O.init_params(MID, seed=4321), mid_batch()
    ref = reference(("mid", world), MID, params, batch, world)

    def setup(r, e, tr):
        if r == 1:
            e.set_option("grad_scale_inverse", 4)

    out, engines = run_schedule(monkeypatch, MID, params, batch, world, schedule, math, steps=1, setup=setup)
    with pytest.raises(AssertionError, match="m:tok|m:path"):
        check_slots(out, engines, MID, schedule, world, ref, math, "control scale")
    worst = _worst_slot_ratio(out, engines, schedule, world, ref, ("tok", "path"))
    print("control scale: slot err/M %.3g" % worst)
    assert worst >= 4 * TAU[math], worst


def test_control_dv_reduce_scatter_off_by_one_percent(monkeypatch):
    """fully_sharded, world 2: the dv reduce-scatter's result scaled by 1.01.  Every context gradient is then 1 % off, which
    the element-wise bound (M sums magnitudes) barely sees; the normwise slices fail by 100 times their tolerance."""
    world, schedule, math = 2, "fully_sharded", 2
    params, batch = O.init_params(MID, seed=4321), mid_batch()
    ref = reference(("mid", world), MID, params, batch, world)
    group = EmulatedGroup(world)
    group.fault("reduce_scatter_tensor", 1, 1.01)
    out, engines = run_schedule(monkeypatch, MID, params, batch, world, schedule, math, steps=1, group=group)
    with pytest.raises(AssertionError):
        check_slots(out, engines, MID, schedule, world, ref, math, "control dv")
    m = assemble(out, engines, MID, schedule, world, 1, "m")
    errs = R.slice_errors({k: m[k].astype(np.float64) / C1 for k in ("tok", "path", "W", "a")}, ref)
    print("control dv x 1.01: slot err/M %.3g, slices %s" % (
        _worst_slot_ratio(out, engines, schedule, world, ref, ("tok", "path", "W", "a")), errs))
    assert min(errs.values()) >= 4 * SLICE[math], errs


def test_control_one_rank_skips_its_inbox_fold(monkeypatch):
    """table_sharded with push_grads, world 2: rank 1 never folds its inbox, so its shards miss every pushed row."""
    world, schedule, math = 2, "table_sharded", 2
    params, batch = O.init_params(MID, seed=4321), mid_batch()
    ref = reference(("mid", world), MID, params, batch, world)

    def setup(r, e, tr):
        if r == 1:
            e.apply_scatter_inbox = lambda: None

    out, engines = run_schedule(monkeypatch, MID, params, batch, world, schedule, math, steps=1, push=True, setup=setup)
    with pytest.raises(AssertionError, match="m:tok|m:path"):
        check_slots(out, engines, MID, schedule, world, ref, math, "control inbox")
    worst = _worst_slot_ratio(out, engines, schedule, world, ref, ("tok", "path"))
    print("control skipped fold: slot err/M %.3g" % worst)
    assert worst >= 4 * TAU[math], worst
