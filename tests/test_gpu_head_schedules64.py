"""Every schedule of the softmax head, and the exp_slab schedule's device-side fallback, against the float64 reference.

tests/test_gpu_reference64.py checks the default schedules (fp32 SIMT, exp_slab in tf32 and 3xTF32).  This module
checks the others, and the fallback the exp_slab schedule takes when a row leaves its fp32 window, with the same
element-wise bounds (|got - ref| <= tau M + 1e-30) and normwise slices:

  a. the production shape (B = 1024, C = 200, Y = 261,246, keep 0.75, uniform and contended indices) in every
     schedule: two-pass (exp_slab = 0), the softmax gradient in the GEMMs' loaders (fuse_softmax_grad, tf32 only) and
     recomputed logits (recompute_logits), in tf32 and 3xTF32;
  b. the batch tile edges, and the three places dY can run (dy_late), in every schedule;
  c. trained-scale logits in every schedule;
  d. one row of the production batch leaving the window (its largest U = exp(s - s_true) about e^75, in the last and in
     the first column of the logits GEMM): the step, the ordinary step after it, and the shipped Trainer("single")
     step, whose target-table Adam runs in the dY epilogue on the rebuilt slab;
  e. the deferred path just inside the window: a few dozen rows whose largest U is about 5e29 over every column (their
     normaliser Z approaches Y 5e29, so the row factor r = 1 / (B Z) approaches FLT_MIN and dY's operand r v_b would be
     subnormal: the combine's operand guard sends that step to the fallback), and one row at 5e29 on one column (stays
     deferred);
  f. c2v_loss, on the tensor cores and on the SIMT path (code vectors offset by one float), at the production vocabulary;
  g. negative controls: a softmax normaliser off by 3e-2 (tf32) or 1e-3 (3xTF32) must fail, in every schedule and at
     production for case d.

Each step also asserts which schedule ran: the exp_slab fallback counter, and a launch count equal to that of an engine
with only the winning options and different from the other schedules'.  At most two production references are alive at
a time (about 3 GB each): the ordinary uniform one, from whose code vectors cases d and e are crafted, and one other."""
import json

import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests import reference64 as R
from tests.test_gpu_reference64 import (EDGE, KEEP, LOSS_TOL, PROD, PROD_B, SEED, SLICE, TAU, check_adam_slots,
                                        check_forward, hot_batch, report)
from tests.util import dev_batch, make_engine

pytestmark = pytest.mark.gpu

# name -> (options, math modes, options of the engine that runs only the winning choice)
SCHEDULES = {
    "two_pass": (dict(exp_slab=0), (1, 2), dict(exp_slab=0, recompute_logits=0, fuse_softmax_grad=0)),
    "loaders": (dict(fuse_softmax_grad=1), (1,), dict(fuse_softmax_grad=1, exp_slab=0, recompute_logits=0)),
    "recompute": (dict(recompute_logits=1), (1, 2), dict(recompute_logits=1, exp_slab=0, fuse_softmax_grad=0)),
}
MATRIX = [(name, math) for name, (_, modes, _) in SCHEDULES.items() for math in modes]
IDS = ["%s-math%d" % c for c in MATRIX]
CONTROL = {1: 1 + 3e-2, 2: 1 + 1e-3}       # softmax normaliser factor each mode's check must see
LOG_U_OUT = 75.0                            # e^75 > 1e30: the row leaves the exp_slab window

_prod = {}
_edge = {}
_launches = {}


@pytest.fixture(scope="module", autouse=True)
def _release_references():
    yield
    _prod.clear()
    _edge.clear()


# ---- references ------------------------------------------------------------------------------------------------------

def _ordinary(name):
    batch = O.synthetic_batch(PROD, PROD_B, seed=1234) if name == "uniform" else hot_batch(PROD, PROD_B, seed=1234)
    params = O.init_params(PROD, seed=4321)
    dm = O.dropout_keep_mask(SEED, 1, PROD_B * PROD.max_contexts, PROD.ctx_dim, KEEP)
    ref = R.train_step64(params, *batch, keep=KEEP, dropout_mask=dm)
    ref.extra["dropout_mask"] = dm
    v, Mv, al, Mal = R.forward64(params, *batch[:4])
    fwd = R.Ref64(float("nan"), dict(v=v, alpha=al), dict(v=Mv, alpha=Mal), ref.targets)
    return dict(params=params, batch=batch, ref=ref, fwd=fwd)


def _crafted(name):
    """Production parameters crafted from the ordinary step's own code vectors (after dropout); same batch and mask."""
    base = prod("uniform")
    batch, ref0 = base["batch"], base["ref"]
    v, target = ref0.vals["v"], batch[4]
    kind = name.split(":")
    control = 1.0
    if kind[0] == "out":                           # d: one row leaves the window, at column Y - 1 or 0
        b = R.quiet_row(v)
        col = PROD.target_vocab - 1 if kind[1] == "last" else 0
        params = R.raise_column(base["params"], v, target, b, col, LOG_U_OUT)
        rows, log_u = np.array([b]), LOG_U_OUT
        if len(kind) > 2:
            control = CONTROL[2]
    elif kind[0] == "column":                      # e: one row at U = 5e29 on one column
        b = R.quiet_row(v)
        col = PROD.target_vocab - 1
        params = R.raise_column(base["params"], v, target, b, col, R.LOG_U_EDGE)
        rows, log_u = np.array([b]), R.LOG_U_EDGE
    else:                                          # e: a few dozen rows at U = 5e29 over every column
        rows = R.rows_to_lower(v, target, 32)
        col = None
        params = R.lower_true_rows(base["params"], v, target, rows, R.LOG_U_EDGE)
        log_u = R.LOG_U_EDGE
    dm = ref0.extra["dropout_mask"]
    ref = R.train_step64(params, *batch, keep=KEEP, dropout_mask=dm, soft_factor=control)
    ref.extra["dropout_mask"] = dm
    return dict(params=params, batch=batch, ref=ref, rows=rows, col=col, log_u=log_u)


def prod(name):
    """Cached production case: "uniform", "hot" (ordinary), or crafted ("out:last", "out:first", "out:last:control",
    "lowered", "column").  Keeps the uniform case and at most one other."""
    if name in _prod:
        return _prod[name]
    for k in [k for k in _prod if k not in ("uniform", name)]:
        del _prod[k]
    _prod[name] = _ordinary(name) if name in ("uniform", "hot") else _crafted(name)
    return _prod[name]


def assert_window(case, inside):
    """What a crafted case claims, from float64: its rows' largest U, where it sits, and every other row far inside."""
    ex = case["ref"].extra
    log_u, col, rows = ex["log_umax"], ex["umax_col"], case["rows"]
    others = np.setdiff1d(np.arange(len(log_u)), rows)
    assert np.all(np.abs(log_u[rows] - case["log_u"]) < 0.05), (log_u[rows].min(), log_u[rows].max())
    if case["col"] is not None:
        assert np.all(col[rows] == case["col"])
    assert log_u[others].max() < 20.0, log_u[others].max()
    hi = np.log(1e30)
    assert np.all(log_u[rows] < hi - 0.5) if inside else np.all(log_u[rows] > hi + 5.0)


def edge_case(B):
    if B not in _edge:
        params = O.init_params(EDGE, seed=4321)
        batch = O.synthetic_batch(EDGE, B, seed=500 + B)
        dm = O.dropout_keep_mask(SEED, 3, B * EDGE.max_contexts, EDGE.ctx_dim, KEEP)
        ref = R.train_step64(params, *batch, keep=KEEP, dropout_mask=dm)
        v, Mv, al, Mal = R.forward64(params, *batch[:4])
        fwd = R.Ref64(float("nan"), dict(v=v, alpha=al), dict(v=Mv, alpha=Mal), ref.targets)
        _edge[B] = dict(params=params, batch=batch, ref=ref, fwd=fwd, dm=dm)
    return _edge[B]


# ---- running a step --------------------------------------------------------------------------------------------------

def engine(dims, B, params, math, opts):
    eng, _ = make_engine(dims, max_batch=B, params=params)
    eng.set_option("math_mode", math)
    for k, val in opts.items():
        eng.set_option(k, val)
    return eng


def step(eng, batch, keep, step_no):
    """One train_step: (loss, gradients, kernel launches)."""
    n0 = eng.launch_count
    loss = float(eng.train_step(*dev_batch(eng, *batch), keep=keep, seed=SEED, step=step_no).cpu()[0])
    return loss, eng.export_grads(), eng.launch_count - n0


def schedule_launches(key, dims, B, params, batch, math, keep, step_no):
    """Launches of one step of an engine with only the winning options of each schedule of `math`, and of the default
    (exp_slab) engine, on this batch."""
    if (key, math) not in _launches:
        out = {}
        for name, (_, modes, winner) in list(SCHEDULES.items()) + [("exp_slab", ({}, (1, 2), {}))]:
            if math in modes:
                eng = engine(dims, B, params, math, winner)
                out[name] = step(eng, batch, keep, step_no)[2]
                eng.close()
        _launches[(key, math)] = out
    return _launches[(key, math)]


def assert_schedule(eng, name, launches, counts):
    assert eng.get_option("exp_slab_fallbacks") == 0
    assert launches == counts[name], (name, launches, counts)
    assert all(n != launches for k, n in counts.items() if k != name), (name, counts)


def check_grads(g, math, ref, label):
    return R.check_step({k: g[k] for k in O.PARAM_NAMES}, ref, TAU[math], SLICE[math], label=label + " ")


def loss_tol(math, ref):
    """The loss bound of the crafted cases, whose logits are in the hundreds: tau M_loss + 1e-4."""
    return TAU[math] * ref.extra["loss_mag"] + LOSS_TOL


def run_schedule(key, dims, case, name, math, label, keep, step_no, tf32_loss=None, fwd=True):
    opts = SCHEDULES[name][0]
    B = case["batch"][0].shape[0]
    counts = schedule_launches(key, dims, B, case["params"], case["batch"], math, keep, step_no)
    eng = engine(dims, B, case["params"], math, opts)
    worst = check_forward(eng, math, case["batch"], case["fwd"], label) if fwd else {}
    loss, g, n = step(eng, case["batch"], keep, step_no)
    target = tf32_loss if (tf32_loss is not None and math == 1) else case["ref"].loss
    assert abs(loss - target) < LOSS_TOL, (label, loss, target, case["ref"].loss)
    assert_schedule(eng, name, n, counts)
    worst.update(check_grads(g, math, case["ref"], label))
    worst["loss"] = abs(loss - target)
    eng.close()
    return worst, g


# ---- a. the production shape -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("name,math", MATRIX, ids=IDS)
@pytest.mark.parametrize("dist", ["hot", "uniform"])
def test_production_shape(dist, name, math):
    case = prod(dist)
    label = "prod-%s %s math=%d" % (dist, name, math)
    worst, _ = run_schedule("prod-" + dist, PROD, case, name, math, label, KEEP, 1)
    report(label, worst)


# ---- b. batch tile edges ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name,math", MATRIX, ids=IDS)
@pytest.mark.parametrize("B", [1, 63, 65, 129, 257, 1000])
def test_batch_tile_edges(B, name, math):
    label = "edge B=%d %s math=%d" % (B, name, math)
    worst, _ = run_schedule(("edge", B), EDGE, edge_case(B), name, math, label, KEEP, 3)
    report(label, worst)


@pytest.mark.parametrize("name,math", MATRIX, ids=IDS)
@pytest.mark.parametrize("dy_late", [0, 1, 2])
def test_dy_placement(dy_late, name, math):
    """dY after dv (0), inside context_backward (1: the loaders still read lse and the targets through PendingDy), and on
    the second side stream (2)."""
    case = edge_case(257)
    eng = engine(EDGE, 257, case["params"], math, dict(SCHEDULES[name][0], dy_late=dy_late))
    loss, g, _ = step(eng, case["batch"], KEEP, 3)
    assert abs(loss - case["ref"].loss) < LOSS_TOL
    assert eng.get_option("exp_slab_fallbacks") == 0
    label = "edge B=257 dy_late=%d %s math=%d" % (dy_late, name, math)
    worst = check_grads(g, math, case["ref"], label)
    worst["loss"] = abs(loss - case["ref"].loss)
    report(label, worst)
    eng.close()


# ---- c. trained-scale logits -----------------------------------------------------------------------------------------

def trained_params(dims):
    params = O.init_params(dims, seed=4321)
    params["tgt"] = (params["tgt"] * np.float32(80.0)).astype(np.float32)
    params["a"] = (params["a"] * np.float32(4.0)).astype(np.float32)
    return params


@pytest.mark.parametrize("name,math", MATRIX, ids=IDS)
def test_trained_scale_logits(name, math):
    """Peaked logits (smallest probability below 1e-20).  In tf32 the loss is held to the truncation model: two-pass and
    loaders read the true-class logit from the tensor-core slab, recompute computes it in fp32."""
    key = "trained"
    if key not in _edge:
        params = trained_params(EDGE)
        batch = O.synthetic_batch(EDGE, 256, seed=90)
        ref = R.train_step64(params, *batch)
        v, Mv, al, Mal = R.forward64(params, *batch[:4])
        fwd = R.Ref64(float("nan"), dict(v=v, alpha=al), dict(v=Mv, alpha=Mal), ref.targets)
        _edge[key] = dict(params=params, batch=batch, ref=ref, fwd=fwd,
                          model={t: R.tf32_model_loss(params, *batch, true_logit=t) for t in ("fp32", "tf32")})
    case = _edge[key]
    assert case["ref"].extra["pmin"] < 1e-20
    model = case["model"]["fp32" if name == "recompute" else "tf32"]
    label = "trained-scale %s math=%d" % (name, math)
    worst, _ = run_schedule(key, EDGE, case, name, math, label, 1.0, 0, tf32_loss=model)
    report(label, worst)


# ---- d. the fallback at the production vocabulary --------------------------------------------------------------------

@pytest.mark.parametrize("math", [1, 2])
@pytest.mark.parametrize("where", ["first", "last"])
def test_fallback_step_then_deferred_step(where, math):
    """d1: exactly one row of the 1024 leaves the window (its U is e^75 in column Y - 1, the partial last N tile of the
    logits GEMM, or in column 0); the step falls back and meets the bounds.  d2: the next step, on ordinary parameters,
    runs the deferred schedule again (the counter stays at 1) and meets the bounds."""
    case = prod("out:" + where)
    assert_window(case, inside=False)
    ref = case["ref"]
    eng = engine(PROD, PROD_B, case["params"], math, {})
    assert eng.get_option("exp_slab") == 1
    loss, g, _ = step(eng, case["batch"], KEEP, 1)
    assert eng.get_option("exp_slab_fallbacks") == 1
    assert abs(loss - ref.loss) <= loss_tol(math, ref), (loss, ref.loss, loss_tol(math, ref))
    label = "fallback %s math=%d" % (where, math)
    worst = check_grads(g, math, ref, label)
    worst["loss"] = abs(loss - ref.loss)
    report(label, worst)
    base = prod("uniform")
    eng.load_params(base["params"])
    loss, g, _ = step(eng, base["batch"], KEEP, 1)
    assert eng.get_option("exp_slab_fallbacks") == 1
    assert abs(loss - base["ref"].loss) < LOSS_TOL
    label = "after fallback %s math=%d" % (where, math)
    worst = check_grads(g, math, base["ref"], label)
    worst["loss"] = abs(loss - base["ref"].loss)
    report(label, worst)
    eng.close()


def trainer_step(case, math, dy_late, prefetch):
    from code2vec_b200.trainer import Trainer
    eng = engine(PROD, PROD_B, case["params"], math, {})
    tr = Trainer(eng, keep_prob=KEEP, seed=SEED)
    assert tr.schedule == "single" and tr.fuse_tgt
    eng.set_option("dy_late", dy_late)
    eng.set_option("adam_epilogue_prefetch", prefetch)
    assert eng.get_option("lazy_adam") == 1 and eng.get_option("adam_epilogue_prefetch") == prefetch
    loss = float(tr.step_device(*dev_batch(eng, *case["batch"])).cpu()[0])
    assert eng.get_option("exp_slab_fallbacks") == 1
    eng.sync_tables()
    return eng, loss


@pytest.mark.parametrize("math", [1, 2])
def test_fallback_trainer_step(math):
    """d3: the shipped Trainer("single") step on the d1 batch (lazy Adam, the target table's Adam in the dY epilogue,
    which then reads the rebuilt slab with the row factors reset to 1) for every dy_late, through the Adam slots; and
    once with adam_epilogue_prefetch, whose target table and slots must equal the prefetch-free run bit for bit."""
    case = prod("out:last")
    ref = case["ref"]
    kept = None
    for dy_late in (0, 1, 2):
        eng, loss = trainer_step(case, math, dy_late, 0)
        assert abs(loss - ref.loss) <= loss_tol(math, ref), (loss, ref.loss)
        label = "fallback trainer math=%d dy_late=%d" % (math, dy_late)
        worst = check_adam_slots(eng, ref, math, O.PARAM_NAMES, label)
        c1 = float(np.float32(1.0) - np.float32(0.9))
        got = {k: eng.adam_m[k].cpu().numpy().astype(np.float64) / c1 for k in O.PARAM_NAMES}
        worst.update({"slice:" + k: e for k, e in R.check_slices(got, ref, SLICE[math]).items()})
        worst["loss"] = abs(loss - ref.loss)
        report(label, worst)
        if dy_late == 0:
            kept = [t["tgt"].cpu().numpy() for t in (eng.params, eng.adam_m, eng.adam_v)]
        eng.close()
    eng, loss = trainer_step(case, math, 0, 1)
    for a, t in zip(kept, (eng.params, eng.adam_m, eng.adam_v)):
        assert np.array_equal(a, t["tgt"].cpu().numpy())
    eng.close()


def test_fallback_negative_control():
    """g at production: the d1 step in 3xTF32 against a reference whose softmax normaliser is off by 1e-3 must fail."""
    case = prod("out:last:control")
    eng = engine(PROD, PROD_B, case["params"], 2, {})
    _, g, _ = step(eng, case["batch"], KEEP, 1)
    assert eng.get_option("exp_slab_fallbacks") == 1
    eng.close()
    with pytest.raises(AssertionError) as ei:
        check_grads(g, 2, case["ref"], "control fallback math=2")
    print("R64-CONTROL fallback math=2: %s" % str(ei.value)[:400])


# ---- e. the deferred path at its window edge -------------------------------------------------------------------------

@pytest.mark.parametrize("math", [1, 2])
@pytest.mark.parametrize("kind", ["lowered", "column"])
def test_window_edge(kind, math):
    """Rows whose largest U is about 5e29, inside the U window, must meet the bounds.  "lowered": 32 rows whose
    true-class logit sits about 68 below every other class, so Z approaches Y 5e29 and the row factor r = 1 / (B Z)
    approaches FLT_MIN; r v_b, dY's operand, would be subnormal, and the combine's operand guard sends the step to the
    fallback.  "column": one row at 5e29 on one column only; Z stays near 5e29 and the step stays deferred."""
    case = prod(kind)
    assert_window(case, inside=True)
    ref = case["ref"]
    if kind == "lowered":
        assert len(case["rows"]) == 32
    # the combine's guard on dY's operand r v_b, r = 1 / (B Z): a step falls back when some row's r max|v_b| is below
    # 2^-112 (kExpSlabMinOperand); no row may sit within a factor 2 of that limit
    log2_op = (-np.log(PROD_B) - (ref.extra["lse"] - np.einsum("bd,bd->b", ref.vals["v"], case["params"]["tgt"][
        case["batch"][4]].astype(np.float64))) + np.log(np.abs(ref.vals["v"]).max(axis=1))) / np.log(2.0)
    assert np.abs(log2_op + 112.0).min() > 1.0, log2_op.min()
    expect = int((log2_op < -112.0).any())
    eng = engine(PROD, PROD_B, case["params"], math, {})
    loss, g, _ = step(eng, case["batch"], KEEP, 1)
    fallbacks = eng.get_option("exp_slab_fallbacks")
    eng.close()
    label = "window-edge %s math=%d" % (kind, math)
    print("R64-EDGE %s: fallbacks=%d, expected %d; smallest log2(r max|v_b|) %.1f over its rows" % (
        label, fallbacks, expect, log2_op[case["rows"]].min()))
    assert abs(loss - ref.loss) <= loss_tol(math, ref), (loss, ref.loss)
    worst = check_grads(g, math, ref, label)
    worst["loss"] = abs(loss - ref.loss)
    worst["fallbacks"] = fallbacks
    report(label, worst)
    assert fallbacks == expect


# ---- f. c2v_loss -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("math", [0, 1, 2])
@pytest.mark.parametrize("scale", ["init", "trained"])
def test_loss_entry_point(scale, math):
    """c2v_loss (what Keras evaluate calls) at the production vocabulary, from the engine's own code vectors: aligned
    (tensor-core logits with log-sum-exp partials and xent_combine_kernel in tf32 / 3xTF32) and offset by one float (the
    SIMT logits and xent_kernel), each against the float64 loss of those code vectors, within tau M_loss + 1e-4 (the
    SIMT path at the fp32 tau in every mode)."""
    import torch
    B = 256
    key = ("loss", scale)
    params = trained_params(PROD) if scale == "trained" else O.init_params(PROD, seed=4321)
    batch = O.synthetic_batch(PROD, B, seed=1235)
    eng, _ = make_engine(PROD, max_batch=B, training=False, params=params)
    eng.set_option("math_mode", math)
    d = dev_batch(eng, *batch)
    code, _ = eng.forward(*d[:4], want_attention=False)
    v = code.cpu().numpy()
    if (key, math) not in _edge:
        _edge[(key, math)] = R.head_loss64(params, v, batch[4])
    want, ex = _edge[(key, math)]
    flat = torch.empty(B * PROD.code_dim + 1, dtype=torch.float32, device=eng.dev)
    off = flat[1:].view(B, PROD.code_dim)
    off.copy_(code)
    assert off.data_ptr() % 16 == 4
    got = {"aligned": float(eng.loss(code, d[4]).cpu()[0]), "offset": float(eng.loss(off, d[4]).cpu()[0])}
    eng.close()
    tol = {"aligned": TAU[math] * ex["loss_mag"] + LOSS_TOL, "offset": R.TAU_FP32 * ex["loss_mag"] + LOSS_TOL}
    for k in got:
        assert abs(got[k] - want) <= tol[k], (k, got[k], want, tol[k])
    print("R64 " + json.dumps({"case": "loss %s math=%d" % (scale, math), "aligned": float("%.3g" % abs(got["aligned"] - want)),
                               "offset": float("%.3g" % abs(got["offset"] - want)), "loss_mag": float("%.3g" % ex["loss_mag"])}))


# ---- g. negative controls --------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name,math", MATRIX, ids=IDS)
def test_negative_control(name, math):
    """Every schedule's gradients at B = 257 must fail against a reference with the softmax normaliser off by 3e-2
    (tf32) or 1e-3 (3xTF32): the checks above can see a wrong normaliser in each schedule."""
    case = edge_case(257)
    key = ("control", math)
    if key not in _edge:
        _edge[key] = R.train_step64(case["params"], *case["batch"], keep=KEEP, dropout_mask=case["dm"],
                                    soft_factor=CONTROL[math])
    eng = engine(EDGE, 257, case["params"], math, SCHEDULES[name][0])
    _, g, _ = step(eng, case["batch"], KEEP, 3)
    eng.close()
    check_grads(g, math, case["ref"], "edge B=257 %s math=%d" % (name, math))      # the true reference passes
    with pytest.raises(AssertionError) as ei:
        check_grads(g, math, _edge[key], "control %s math=%d" % (name, math))
    print("R64-CONTROL %s math=%d: %s" % (name, math, str(ei.value)[:400]))
