"""The float64 reference with per-element error magnitudes (tests/reference64.py) has teeth.

The float32 numpy oracle must pass the fp32-class check, and each fault below, applied to the oracle's outputs, must
fail it by at least 4x tau:
  * the softmax part of dL/dlogits scaled by 1.01 (a wrong 1 / sum normaliser, the one-hot part intact);
  * the non-target rows of dY scaled by 1.01, or set to 0;
  * one (context, segment) contribution dropped from a token row;
  * a masked context's dx added into its row;
  * one 32 x 32 block of dW transposed;
  * one example's attention weights rotated by one context.
At the java14m target vocabulary the first three leave `rel_err` of dY below the 5e-5 fp32-class tolerance of the
older parity tests, which is the gap this check closes.  The normwise slice checks must catch factors of 1.001 at the
fp32-class tolerance and 1.05 at the tf32 one.  The model of tf32's truncated operands must reproduce the loss offsets
the H100 shows where tf32 cannot meet 1e-4 of the float64 loss.  CPU only."""
import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests import reference64 as R
from tests.util import rel_err

SHAPES = {
    "small": (O.Dims(1001, 501, 1001, 32, 96, 20), 64, 0.75),
    "mid": (O.Dims(3001, 2003, 32771, 128, 384, 200), 256, 1.0),
    "java14m_y": (O.Dims(3001, 2003, 261246, 128, 384, 200), 64, 1.0),
}

_cache = {}


def case(name):
    """(params, batch, keep, dropout mask, float64 reference, float32 oracle outputs, hole), built once per shape.
    Example `hole[0]` has a masked slot `hole[1]` in the middle of its bag with a nonzero source token, one that no
    valid context uses where the vocabulary has such a row."""
    if name in _cache:
        return _cache[name]
    dims, B, keep = SHAPES[name]
    params = O.init_params(dims, seed=4321)
    src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=21)
    n = np.where(mask.sum(axis=1) >= 3, mask.sum(axis=1), np.inf)
    b = int(np.argmin(n))                                    # the shortest bag with a middle slot
    mask[b, 1] = 0.0
    used = np.zeros(dims.token_vocab, bool)
    used[src[mask > 0]] = used[tgt[mask > 0]] = True
    if (~used[1:]).any():
        src[b, 1] = int(np.flatnonzero(~used[1:])[0]) + 1
    batch = (src, pth, tgt, mask, target)
    dm = O.dropout_keep_mask(5, 3, B * dims.max_contexts, dims.ctx_dim, keep) if keep < 1.0 else None
    ref = R.train_step64(params, *batch, keep=keep, dropout_mask=dm)
    loss, g, o = O.train_loss_and_grads(params, *batch, keep=keep, dropout_mask=dm)
    got = dict(g, v=o["v"], alpha=o["alpha"], dv=o["dv"])
    _cache[name] = (params, batch, keep, dm, ref, loss, got, (b, 1))
    return _cache[name]


def softmax_scaled(name, factor):
    """The oracle's outputs with the softmax part of dL/dlogits scaled by `factor`: every output that depends on it
    moves by exactly what the float64 step moves by."""
    params, batch, keep, dm, ref, _, got, _ = case(name)
    bad_ref = R.train_step64(params, *batch, keep=keep, dropout_mask=dm, soft_factor=factor)
    return {k: (got[k] + (bad_ref.vals[k] - ref.vals[k])).astype(np.float32) for k in ("tgt", "dv", "tok", "path", "W", "a")}


def nontarget_scaled(name, factor):
    _, _, _, _, ref, _, got, _ = case(name)
    g = got["tgt"].copy()
    other = np.ones(g.shape[0], bool)
    other[ref.targets] = False
    g[other] *= np.float32(factor)
    return {"tgt": g}


def mutation(name, kind):
    """{tensor name: faulty float32 values} for one fault."""
    params, (src, pth, tgt, mask, target), keep, dm, ref, _, got, (hb, hc) = case(name)
    d = params["tok"].shape[1]
    if kind == "softmax_x1.01":
        return softmax_scaled(name, 1.01)
    if kind == "nontarget_dY_x1.01":
        return nontarget_scaled(name, 1.01)
    if kind == "nontarget_dY_zero":
        return nontarget_scaled(name, 0.0)
    if kind == "dropped_contribution":
        # the source-token segment of the context with the largest attention weight
        b, c = np.unravel_index(int(np.argmax(ref.vals["alpha"])), mask.shape)
        dx = R.example_dx64(params, src, pth, tgt, mask, ref.vals["dv"], b, keep=keep, dropout_mask=dm)
        g = got["tok"].copy()
        g[src[b, c]] -= dx[c, :d].astype(np.float32)
        return {"tok": g}
    if kind == "masked_context_added":
        assert mask[hb, hc] == 0 and src[hb, hc] != 0
        # the masked slot's dx as if it were valid
        m2 = mask.copy()
        m2[hb, hc] = 1.0
        dx = R.example_dx64(params, src, pth, tgt, m2, ref.vals["dv"], hb, keep=keep, dropout_mask=dm)
        g = got["tok"].copy()
        g[src[hb, hc]] += dx[hc, :d].astype(np.float32)
        return {"tok": g}
    if kind == "dW_block_transposed":
        g = got["W"].copy()
        g[32:64, 32:64] = g[32:64, 32:64].T.copy()
        return {"W": g}
    if kind == "alpha_rotated":
        a = got["alpha"].copy()
        b = int(np.flatnonzero(mask.sum(axis=1) >= 2)[0])
        a[b] = np.roll(a[b], 1)
        return {"alpha": a}
    raise ValueError(kind)


GLOBAL = ["softmax_x1.01", "nontarget_dY_x1.01", "nontarget_dY_zero"]
LOCAL = ["dropped_contribution", "masked_context_added", "dW_block_transposed", "alpha_rotated"]


@pytest.mark.parametrize("name", ["small", "mid"])
def test_float32_oracle_passes(name):
    _, _, _, _, ref, loss, got, _ = case(name)
    assert abs(loss - ref.loss) < 1e-6
    worst = R.check_step(got, ref, R.TAU_FP32)
    print(name, {k: "%.1e" % r for k, r in worst.items()})
    # far inside the bound: tau leaves room for other summation orders and the tensor cores' 3xTF32 split
    assert max(worst.values()) < R.TAU_FP32 / 10
    errs = R.check_slices(got, ref, R.SLICE_TOL_FP32)
    print(name, "slices", {k: "%.1e" % e for k, e in errs.items()})
    assert max(errs.values()) < 1e-5, errs


@pytest.mark.parametrize("kind", GLOBAL + LOCAL)
@pytest.mark.parametrize("name", ["small", "mid"])
def test_mutation_fails_elementwise_check(name, kind):
    _, _, _, _, ref, _, _, _ = case(name)
    bad = mutation(name, kind)
    worst = max(R.err_ratio(a, ref.vals[k], ref.mags[k])[0] for k, a in bad.items())
    print(name, kind, "max err/M %.2e" % worst)
    with pytest.raises(AssertionError):
        R.check_step(bad, ref, R.TAU_FP32)
    assert worst >= 4 * R.TAU_FP32, worst
    if kind in LOCAL:
        # local faults stay visible in tf32: through the element-wise bound or a normwise slice
        tf32_elem = worst >= 4 * R.TAU_TF32
        tf32_slice = max(R.slice_errors(bad, ref).values()) >= 4 * R.SLICE_TOL_TF32
        assert tf32_elem or tf32_slice


@pytest.mark.parametrize("kind", GLOBAL)
def test_mutation_fails_at_java14m_vocabulary_but_passes_rel_err(kind):
    """At Y = 261,246 these faults pass the old parity tests' `rel_err` bound on dY and fail the new check."""
    _, _, _, _, ref, _, got, _ = case("java14m_y")
    bad = mutation("java14m_y", kind)
    assert rel_err(bad["tgt"], ref.vals["tgt"]) < 5e-5
    assert rel_err(got["tgt"], ref.vals["tgt"]) < 1e-6
    worst = R.err_ratio(bad["tgt"], ref.vals["tgt"], ref.mags["tgt"])[0]
    print(kind, "rel_err %.2e, max err/M %.2e" % (rel_err(bad["tgt"], ref.vals["tgt"]), worst))
    assert worst >= 4 * R.TAU_FP32, worst
    with pytest.raises(AssertionError):
        R.check_step(bad, ref, R.TAU_FP32)


def slice_probe(name, kind, factor, tol):
    _, _, _, _, ref, _, _, _ = case(name)
    bad = softmax_scaled(name, factor) if kind.startswith("softmax") else nontarget_scaled(name, factor)
    errs = R.slice_errors(bad, ref)
    print(name, kind, {k: "%.2e" % e for k, e in errs.items()})
    assert max(errs.values()) >= 4 * tol, errs
    with pytest.raises(AssertionError):
        R.check_slices(bad, ref, tol)


@pytest.mark.parametrize("kind", ["softmax_x1.05", "nontarget_dY_x1.05"])
@pytest.mark.parametrize("name", ["small", "mid"])
def test_tf32_slice_check_catches_systematic_error(name, kind):
    slice_probe(name, kind, 1.05, R.SLICE_TOL_TF32)


@pytest.mark.parametrize("kind", ["softmax_x1.001", "nontarget_dY_x1.001"])
@pytest.mark.parametrize("name", ["small", "mid"])
def test_fp32_slice_check_catches_systematic_error(name, kind):
    """0.1 % systematic errors, which the element-wise fp32-class bound lets through on the non-target dY rows."""
    slice_probe(name, kind, 1.001, R.SLICE_TOL_FP32)


# (name, dims, B, batch seed, parameter scale of tgt and a, keep, dropout (seed, step), loss offset measured on an H100
# in tf32): the two cases where tf32 misses the float64 loss by more than 1e-4, and one at the initialisation scale
TF32_LOSS_CASES = [
    ("d4", O.Dims(777, 333, 1537, 4, 4, 2), 37, 6, (1.0, 1.0), 0.75, (0x5EED, 5), -2.4095e-4),
    ("trained_scale", O.Dims(20011, 10007, 5003, 128, 384, 50), 256, 90, (80.0, 4.0), 1.0, None, -6.4896e-3),
    ("init_scale", O.Dims(777, 333, 1537, 28, 128, 33), 64, 161, (1.0, 1.0), 0.75, (0x5EED, 5), None),
]


@pytest.mark.parametrize("case_", TF32_LOSS_CASES, ids=[c[0] for c in TF32_LOSS_CASES])
def test_tf32_truncation_model_reproduces_the_loss_offset(case_):
    """tf32 reads the top 10 mantissa bits of each fp32 operand, a bias toward zero that the batch does not average
    away.  Where that moves the loss by more than 1e-4, the GPU tests hold tf32 to 1e-4 of reference64.tf32_model_loss
    instead of the float64 loss; this checks that the model accounts for the whole offset measured on the H100."""
    name, dims, B, seed, (ys, as_), keep, drop, measured = case_
    params = O.init_params(dims, seed=4321)
    params["tgt"] = (params["tgt"] * np.float32(ys)).astype(np.float32)
    params["a"] = (params["a"] * np.float32(as_)).astype(np.float32)
    batch = O.synthetic_batch(dims, B, seed=seed)
    dm = O.dropout_keep_mask(drop[0], drop[1], B * dims.max_contexts, dims.ctx_dim, keep) if drop else None
    ref = R.train_step64(params, *batch, keep=keep, dropout_mask=dm)
    offset = R.tf32_model_loss(params, *batch, keep=keep, dropout_mask=dm) - ref.loss
    print(name, "model offset %.4e, measured %s" % (offset, measured))
    if measured is None:
        assert abs(offset) < 2e-5
    else:
        assert abs(offset) > 1e-4
        assert abs(offset - measured) < 2e-5


def test_sampled_head_matches_oracle_and_float32_passes():
    dims, B, _ = SHAPES["small"]
    params = O.init_params(dims, seed=4321)
    src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=22)
    rng = np.random.default_rng(4)
    S = 25
    sampled = O.log_uniform_sample(rng, S, dims.target_vocab)
    sampled[0] = target[3]
    sampled[1] = sampled[2]
    lq_t = O.log_uniform_logq(target, S, dims.target_vocab)
    lq_s = O.log_uniform_logq(sampled, S, dims.target_vocab)
    ref = R.train_step64(params, src, pth, tgt, mask, target, sampled=sampled, logq_true=lq_t, logq_sampled=lq_s)
    v, _, _ = O.forward(params, src, pth, tgt, mask)
    loss, dv, g_tgt, _ = O.sampled_softmax_loss_and_grads(params, v, target, sampled, lq_t, lq_s)
    assert abs(loss - ref.loss) < 1e-6
    R.check_step({"v": v, "dv": dv, "tgt": g_tgt}, ref, R.TAU_FP32)
    bad = g_tgt.copy()
    bad[sampled[5]] *= np.float32(1.01)
    with pytest.raises(AssertionError):
        R.check_step({"tgt": bad}, ref, R.TAU_FP32)


# ---- the loss bound of logits in the hundreds, the truncation model's true-class logit, the window-edge recipes ----------

ODD = O.Dims(777, 333, 1537, 20, 52, 13)


def wide_logits_case(name):
    """(params, batch): trained-scale logits (target table x 80, attention vector x 4), or logits up to +-400."""
    if name == "trained":
        dims = O.Dims(20011, 10007, 5003, 128, 384, 50)
        params = O.init_params(dims, seed=4321)
        params["tgt"] = (params["tgt"] * np.float32(80.0)).astype(np.float32)
        params["a"] = (params["a"] * np.float32(4.0)).astype(np.float32)
        return params, O.synthetic_batch(dims, 64, seed=90)
    batch = O.synthetic_batch(ODD, 37, seed=81)
    params = O.init_params(ODD, seed=9)
    v, _, _ = O.forward(params, *batch[:4])
    params["tgt"] = (params["tgt"] * np.float32(400.0 / np.abs(O.logits_of(params, v)).max())).astype(np.float32)
    return params, batch


@pytest.mark.parametrize("name", ["trained", "logits_400"])
def test_float32_oracle_meets_the_loss_bound(name):
    """The float32 oracle's loss is within TAU_FP32 M_loss of the float64 one, with no absolute floor."""
    params, batch = wide_logits_case(name)
    ref = R.train_step64(params, *batch)
    loss, _, _ = O.train_loss_and_grads(params, *batch)
    if name == "logits_400":
        assert np.abs(ref.extra["log_umax"]).max() > 100
    err, bound = abs(loss - ref.loss), R.TAU_FP32 * ref.extra["loss_mag"]
    print(name, "loss %.6g err %.2e bound %.2e" % (ref.loss, err, bound))
    assert err <= bound


def tf32_emulated_loss(params, src, pth, tgt, mask, target, true_logit):
    """tf32_model_loss's model in float32 numpy: truncated operands, float32 arithmetic everywhere else."""
    f32 = lambda a: np.asarray(a, dtype=np.float32)
    tr = lambda a: f32(R.tf32_truncate(a))
    B, C = src.shape
    x = np.concatenate([params["tok"][src], params["path"][pth], params["tok"][tgt]], axis=-1).reshape(B * C, -1)
    h = np.tanh(tr(x) @ tr(params["W"]))
    z = np.where(mask > 0, (h @ params["a"]).reshape(B, C), np.float32(-np.inf))
    al = np.exp(z - z.max(axis=1, keepdims=True))
    al /= al.sum(axis=1, keepdims=True)
    v = np.einsum("bc,bcd->bd", al, h.reshape(B, C, -1))
    s = tr(v) @ tr(params["tgt"]).T
    m = s.max(axis=1)
    lse = m + np.log(np.exp(s - m[:, None]).sum(axis=1))
    st = s[np.arange(B), target] if true_logit == "tf32" else np.einsum("bd,bd->b", v, params["tgt"][target])
    return float(np.mean(lse - st))


@pytest.mark.parametrize("true_logit", ["fp32", "tf32"])
def test_tf32_model_true_logit_variants_match_a_float32_emulation(true_logit):
    params, batch = wide_logits_case("trained")
    model = R.tf32_model_loss(params, *batch, true_logit=true_logit)
    emulated = tf32_emulated_loss(params, *batch, true_logit)
    other = R.tf32_model_loss(params, *batch, true_logit="tf32" if true_logit == "fp32" else "fp32")
    print(true_logit, "model %.7g emulated %.7g other variant %.7g" % (model, emulated, other))
    assert abs(model - emulated) < 1e-5
    assert abs(model - other) > 1e-4                  # the choice matters at trained scale


RECIPE = O.Dims(1001, 501, 5003, 128, 384, 20)


@pytest.mark.parametrize("recipe", ["column_last", "column_first", "lowered"])
def test_window_edge_recipes_put_the_largest_u_where_they_claim(recipe):
    params = O.init_params(RECIPE, seed=4321)
    src, pth, tgt, mask, target = O.synthetic_batch(RECIPE, 256, seed=7)
    target = np.where(np.isin(target, [0, RECIPE.target_vocab - 1]), 1, target).astype(target.dtype)
    v, Mv, _, _ = R.forward64(params, src, pth, tgt, mask)
    if recipe == "lowered":
        rows = R.rows_to_lower(v, target, 24)
        crafted = R.lower_true_rows(params, v, target, rows, R.LOG_U_EDGE)
        col = None
    else:
        rows = np.array([R.quiet_row(v)])
        col = RECIPE.target_vocab - 1 if recipe == "column_last" else 0
        crafted = R.raise_column(params, v, target, rows[0], col, R.LOG_U_EDGE)
    _, ex = R.head_loss64(crafted, v, target, Mv=Mv)
    log_u = ex["log_umax"]
    others = np.setdiff1d(np.arange(len(target)), rows)
    print(recipe, "rows %.4f..%.4f, others below %.2f" % (log_u[rows].min(), log_u[rows].max(), log_u[others].max()))
    assert np.all(np.abs(log_u[rows] - R.LOG_U_EDGE) < 0.05)
    assert np.all(log_u[rows] < np.log(1e30))
    assert log_u[others].max() < 20.0
    if col is not None:
        assert ex["umax_col"][rows[0]] == col
    else:
        # the rows' true-class logits sit below every other class: U = exp(s - s_true) is large in every column
        Yt = crafted["tgt"].astype(np.float64)
        s = v[rows] @ Yt.T
        s[np.arange(len(rows)), target[rows]] = np.inf
        assert (s.min(axis=1) - np.einsum("bd,bd->b", v[rows], Yt[target[rows]])).min() > R.LOG_U_EDGE - 5.0
