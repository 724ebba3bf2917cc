"""The engine against the float64 reference with per-element error magnitudes (tests/reference64.py).

Every case checks the loss (|delta| < 1e-4), and the five gradients element by element, |got - ref| <= tau M + 1e-30,
with tau = 2e-6 in the fp32-class modes (fp32 FFMA, 3xTF32) and 4e-3 in tf32.  The normwise relative errors over named
slices (dY target rows, dY non-target rows, tok, path, W, a) must also stay below 1e-4 in the fp32-class modes and 1e-2
in tf32: M bounds signed sums by sums of magnitudes, so on its own it would let a small systematic error through.  Code
vectors and attention weights are checked the same way through the evaluation forward.  Elements with M = 0 -- rows
that only masked contexts reference, masked attention weights -- must be exactly 0.

Shapes: the production batch (B = 1024, C = 200, d = 128, D = 384, Y = 261,246 with reduced token / path tables) with
uniform and contended (one row holding a third of the entries) indices; the batch sizes around the 64- and 128-row tiles;
the attention kernels' ceil(D / 128) dispatch and the fused gather's d % 32 condition; masks with holes, one-context
bags and src == tgt; trained-scale logits; the sampled softmax across its 64-example chunks; and one shipped
`Trainer("single")` step, whose fused target-table Adam never writes dY, through the Adam slots it leaves behind; and
top-k evaluation at the production batch and with fewer target rows than k."""
import json

import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests import reference64 as R
from tests.util import dev_batch, make_engine

pytestmark = pytest.mark.gpu

TAU = {0: R.TAU_FP32, 1: R.TAU_TF32, 2: R.TAU_FP32}
SLICE = R.SLICE_TOL
MODES = [0, 1, 2]
LOSS_TOL = 1e-4
KEEP = 0.75
SEED = 0x5EED

PROD = O.Dims(token_vocab=100003, path_vocab=50021, target_vocab=261246, embed_dim=128, code_dim=384, max_contexts=200)
PROD_B = 1024

_cache = {}


@pytest.fixture(scope="module", autouse=True)
def _release_references():
    yield
    _cache.clear()


def report(label, worst):
    print("R64 " + json.dumps({"case": label, **{k: float("%.3g" % v) for k, v in worst.items()}}))


def hot_batch(dims, B, seed, frac=0.32, hot=7):
    """Zipf(1.3) indices with one row of each table holding `frac` of the valid entries (atomic contention)."""
    src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=seed)
    rng = np.random.default_rng(seed + 1)
    valid = mask > 0
    for a, V in ((src, dims.token_vocab), (pth, dims.path_vocab), (tgt, dims.token_vocab)):
        z = 1 + (rng.zipf(1.3, size=a.shape) - 1) % (V - 1)
        a[valid] = z[valid]
        a[valid & (rng.random(a.shape) < frac)] = hot
    return src, pth, tgt, mask, target


def reference(key, dims, batch, keep=1.0, seed=0, step=0, params=None, **kw):
    """(params, batch, train-step reference, evaluation-forward reference), cached by `key`."""
    if key in _cache:
        return _cache[key]
    if params is None:
        params = O.init_params(dims, seed=4321)
    B = batch[0].shape[0]
    dm = O.dropout_keep_mask(seed, step, B * dims.max_contexts, dims.ctx_dim, keep) if keep < 1.0 else None
    ref = R.train_step64(params, *batch, keep=keep, dropout_mask=dm, **kw)
    ref.extra["dropout_mask"] = dm
    v, Mv, al, Mal = R.forward64(params, *batch[:4])
    fwd = R.Ref64(float("nan"), dict(v=v, alpha=al), dict(v=Mv, alpha=Mal), ref.targets)
    _cache[key] = (params, batch, ref, fwd)
    return _cache[key]


def check_forward(eng, math, batch, fwd, label):
    code, attn = eng.forward(*dev_batch(eng, *batch[:4]))
    got = {"v": code.cpu().numpy(), "alpha": attn.cpu().numpy()}
    return R.check_step(got, fwd, TAU[math], SLICE[math], label=label + " ")


def check_train(eng, math, batch, ref, label, keep=1.0, seed=0, step=0, want=("tok", "path", "tgt", "W", "a"),
                tf32_loss=None):
    """One train step against `ref`.  tf32_loss: in tf32 the loss is held to 1e-4 of this value instead, the loss of
    reference64.tf32_model_loss.  The tensor cores read only the top 10 mantissa bits of each fp32 operand (truncation,
    biased toward zero), and with trained-scale logits or 4-term logits (D = 4) that bias moves the loss by far more than
    1e-4 (6.5e-3 and 2.4e-4); the model of truncated operands reproduces both offsets, see
    tests/test_reference64.py::test_tf32_truncation_model_reproduces_the_loss_offset."""
    loss = float(eng.train_step(*dev_batch(eng, *batch), keep=keep, seed=seed, step=step).cpu()[0])
    target = tf32_loss if (tf32_loss is not None and math == 1) else ref.loss
    assert abs(loss - target) < LOSS_TOL, (label, loss, target, ref.loss)
    g = eng.export_grads()
    worst = R.check_step({k: g[k] for k in want}, ref, TAU[math], SLICE[math], label=label + " ")
    worst["loss"] = abs(loss - target)
    return worst


def check_adam_slots(eng, ref, math, names, label, beta1=0.9, beta2=0.999):
    """After Adam step 1 (from zero slots): m = (1 - beta1) g and v = (1 - beta2) g^2, with the engine's float32 betas."""
    c1 = float(np.float32(1.0) - np.float32(beta1))
    c2 = float(np.float32(1.0) - np.float32(beta2))
    tau = TAU[math]
    out = {}
    for k in names:
        g, M = ref.vals[k], ref.mags[k]
        m = eng.adam_m[k].cpu().numpy().astype(np.float64)
        v = eng.adam_v[k].cpu().numpy().astype(np.float64)
        em = tau * M
        out["m:" + k] = R.check_elementwise(label + " m:" + k, m / c1, g, M, tau)
        bound = c2 * (2.0 * np.abs(g) * em + em * em) + 1e-30
        err = np.abs(v - c2 * g * g)
        bad = ~(err <= bound)
        assert not bad.any(), "%s v:%s: %d elements off, worst row %d" % (
            label, k, int(bad.sum()), int(np.unravel_index(int(np.argmax(err - bound)), err.shape)[0]))
        with np.errstate(divide="ignore", invalid="ignore"):
            out["v:%s/bound" % k] = float(np.nanmax(np.where(err == 0, 0.0, err / bound)))     # fraction of the bound used
    return out


# ---- 1. the production shape ---------------------------------------------------------------------------------------

def prod_case(dist):
    """One production reference is kept at a time (about 2 GB): the contended one's tests run first, then every test of
    the uniform one."""
    key = "prod-" + dist
    for k in [k for k in _cache if isinstance(k, str) and k.startswith("prod-") and k != key]:
        del _cache[k]
    batch = O.synthetic_batch(PROD, PROD_B, seed=1234) if dist == "uniform" else hot_batch(PROD, PROD_B, seed=1234)
    return reference(key, PROD, batch, keep=KEEP, seed=SEED, step=1)


@pytest.mark.parametrize("math", MODES)
@pytest.mark.parametrize("dist", ["hot", "uniform"])
def test_production_shape(dist, math):
    params, batch, ref, fwd = prod_case(dist)
    if dist == "hot":
        src, _, _, mask, _ = batch
        assert (src[mask > 0] == 7).mean() >= 0.30
    eng, _ = make_engine(PROD, max_batch=PROD_B, params=params)
    eng.set_option("math_mode", math)
    label = "prod-%s math=%d" % (dist, math)
    worst = check_forward(eng, math, batch, fwd, label)
    worst.update(check_train(eng, math, batch, ref, label, keep=KEEP, seed=SEED, step=1))
    if math != 0:
        assert eng.get_option("exp_slab") == 1
        assert eng.get_option("exp_slab_fallbacks") == 0
    report(label, worst)
    eng.close()


# ---- 2. the training schedule as shipped ---------------------------------------------------------------------------

@pytest.mark.parametrize("dy_late", [0, 1, 2])
@pytest.mark.parametrize("math", [1, 2])
def test_trainer_step_adam_slots(math, dy_late):
    """One Trainer("single") step (lazy Adam, target-table Adam fused into the dY epilogue): the fused path never writes
    dY, so the Adam slots are the only place its target gradient can be seen."""
    from code2vec_b200.trainer import Trainer
    params, batch, ref, _ = prod_case("uniform")
    eng, _ = make_engine(PROD, max_batch=PROD_B, params=params)
    eng.set_option("math_mode", math)
    tr = Trainer(eng, keep_prob=KEEP, seed=SEED)
    assert tr.schedule == "single" and tr.fuse_tgt
    eng.set_option("dy_late", dy_late)
    assert eng.get_option("lazy_adam") == 1
    loss = float(tr.step_device(*dev_batch(eng, *batch)).cpu()[0])
    assert abs(loss - ref.loss) < LOSS_TOL
    eng.sync_tables()
    label = "trainer math=%d dy_late=%d" % (math, dy_late)
    worst = check_adam_slots(eng, ref, math, O.PARAM_NAMES, label)
    c1 = float(np.float32(1.0) - np.float32(0.9))
    got = {k: eng.adam_m[k].cpu().numpy().astype(np.float64) / c1 for k in O.PARAM_NAMES}
    worst.update({"slice:" + k: e for k, e in R.check_slices(got, ref, SLICE[math]).items()})
    report(label, worst)
    eng.close()


# ---- 3. batch tile edges -------------------------------------------------------------------------------------------

EDGE = O.Dims(token_vocab=20011, path_vocab=10007, target_vocab=5003, embed_dim=128, code_dim=384, max_contexts=50)


@pytest.mark.parametrize("math", MODES)
@pytest.mark.parametrize("B", [1, 2, 63, 65, 127, 129, 255, 257, 1000])
def test_batch_tile_edges(B, math):
    params, batch, ref, fwd = reference(("edge", B), EDGE, O.synthetic_batch(EDGE, B, seed=500 + B), keep=KEEP,
                                        seed=SEED, step=3)
    eng, _ = make_engine(EDGE, max_batch=B, params=params)
    eng.set_option("math_mode", math)
    label = "edge B=%d math=%d" % (B, math)
    worst = check_forward(eng, math, batch, fwd, label)
    worst.update(check_train(eng, math, batch, ref, label, keep=KEEP, seed=SEED, step=3))
    report(label, worst)
    eng.close()


# ---- 4. dispatch edges ---------------------------------------------------------------------------------------------

# (d, D, C, B): every attention instantiation NV = ceil(D / 128) in {1, 2, 3, 4, 5 -> 6, 7 -> 8, 8}, D = 4 and the
# D = 1024 limit, d on both sides of the fused gather's d % 32 == 0, and B * C on both sides of % 4 == 0.  The fused
# gather (d % 32 == 0 and B * C % 4 == 0) runs at D = 384, and with a partial last N tile at D = 516 and 772.
DISPATCH = [(4, 4, 2, 37), (28, 128, 33, 64), (32, 132, 1, 37), (36, 500, 257, 12), (32, 516, 33, 37),
            (4, 772, 2, 64), (128, 1024, 33, 37), (32, 384, 257, 16), (32, 516, 4, 37), (64, 772, 4, 16)]
VARIANTS = [(0, 0), (1, 0), (1, 1), (2, 0)]          # (math mode, fuse_gather)


@pytest.mark.parametrize("math,fuse", VARIANTS)
@pytest.mark.parametrize("d,D,C,B", DISPATCH)
def test_dispatch_edges(d, D, C, B, math, fuse):
    dims = O.Dims(token_vocab=777, path_vocab=333, target_vocab=1537, embed_dim=d, code_dim=D, max_contexts=C)
    params, batch, ref, fwd = reference(("dispatch", d, D, C, B), dims, O.synthetic_batch(dims, B, seed=D + C),
                                        keep=KEEP, seed=SEED, step=5)
    eng, _ = make_engine(dims, max_batch=B, params=params)
    eng.set_option("math_mode", math)
    eng.set_option("fuse_gather", fuse)
    label = "dispatch d=%d D=%d C=%d B=%d math=%d fuse_gather=%d" % (d, D, C, B, math, fuse)
    worst = check_forward(eng, math, batch, fwd, label)
    model = R.tf32_model_loss(params, *batch, keep=KEEP, dropout_mask=ref.extra["dropout_mask"]) if D == 4 else None
    worst.update(check_train(eng, math, batch, ref, label, keep=KEEP, seed=SEED, step=5, tf32_loss=model))
    report(label, worst)
    eng.close()


# ---- 5. input edges ------------------------------------------------------------------------------------------------

MIDE = O.Dims(token_vocab=5003, path_vocab=3001, target_vocab=4099, embed_dim=128, code_dim=384, max_contexts=200)


def edge_inputs(B=129):
    """Holes in the middle of bags with nonzero indices in masked slots (some rows only masked slots reference),
    one-context bags, and src == tgt inside a context."""
    dims = MIDE
    src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=77, full_bags=True)
    rng = np.random.default_rng(78)
    mask = (rng.random(mask.shape) < 0.6).astype(np.float32)
    mask[:, 0] = 1.0                                         # no empty bag
    mask[3:9] = 0.0
    mask[3:9, [0, 5, 7, 11, 42, 150]] = np.eye(6, dtype=np.float32)   # one valid context, anywhere in the bag
    src[10, :50] = tgt[10, :50]                              # src == tgt
    src[11] = tgt[11] = src[11, 0]                           # one token in every slot of a bag
    # rows 1..20 of both tables only appear in masked slots
    holes = np.argwhere(mask == 0)
    pick = holes[rng.choice(len(holes), 60, replace=False)]
    for i, (b, c) in enumerate(pick):
        src[b, c] = 1 + i % 20
        pth[b, c] = 1 + i % 20
    live = mask > 0
    for a in (src, pth, tgt):
        a[live & (a <= 20)] += 21
    assert not np.isin(np.r_[src[live], tgt[live], pth[live]], np.arange(1, 21)).any()
    return dims, (src, pth, tgt, mask, target)


@pytest.mark.parametrize("math", MODES)
def test_input_edges(math):
    dims, batch = edge_inputs()
    params, batch, ref, fwd = reference("inputs", dims, batch, keep=KEEP, seed=SEED, step=2)
    B = batch[0].shape[0]
    eng, _ = make_engine(dims, max_batch=B, params=params)
    eng.set_option("math_mode", math)
    label = "inputs math=%d" % math
    worst = check_forward(eng, math, batch, fwd, label)
    worst.update(check_train(eng, math, batch, ref, label, keep=KEEP, seed=SEED, step=2))
    g = eng.export_grads()
    assert np.all(g["tok"][1:21] == 0.0) and np.all(g["path"][1:21] == 0.0)
    report(label, worst)
    eng.close()


@pytest.mark.parametrize("math", MODES)
def test_trained_scale_logits(math):
    """Peaked logits: the smallest softmax probabilities reach 1e-20 and below, inside the exp_slab window."""
    dims = EDGE
    params = O.init_params(dims, seed=4321)
    params["tgt"] = (params["tgt"] * np.float32(80.0)).astype(np.float32)
    params["a"] = (params["a"] * np.float32(4.0)).astype(np.float32)
    params, batch, ref, fwd = reference("trained", dims, O.synthetic_batch(dims, 256, seed=90), params=params)
    assert ref.extra["pmin"] < 1e-20, ref.extra["pmin"]
    eng, _ = make_engine(dims, max_batch=256, params=params)
    eng.set_option("math_mode", math)
    label = "trained-scale math=%d" % math
    worst = check_forward(eng, math, batch, fwd, label)
    worst.update(check_train(eng, math, batch, ref, label, tf32_loss=R.tf32_model_loss(params, *batch)))
    if math != 0:
        assert eng.get_option("exp_slab_fallbacks") == 0
    report(label, worst)
    eng.close()


# ---- 6. sampled softmax --------------------------------------------------------------------------------------------

SAMP = O.Dims(token_vocab=5003, path_vocab=3001, target_vocab=5003, embed_dim=32, code_dim=96, max_contexts=20)


def sampled_case(B, S):
    key = ("sampled", B, S)
    if key in _cache:
        return _cache[key]
    dims = SAMP
    batch = O.synthetic_batch(dims, B, seed=B * 7 + S)
    target = batch[4]
    rng = np.random.default_rng(B + S)
    sampled = O.log_uniform_sample(rng, S, dims.target_vocab)
    if S >= 3:
        sampled[0] = target[3]                               # an accidental hit
        sampled[1] = sampled[2]                              # a duplicate sampled class
    if S >= 65:
        sampled[64] = target[B - 1]                          # a hit in the second 64-sample group
    lq_t = O.log_uniform_logq(target, S, dims.target_vocab)
    lq_s = O.log_uniform_logq(sampled, S, dims.target_vocab)
    out = reference(key, dims, batch, keep=KEEP, seed=SEED, step=1, sampled=sampled, logq_true=lq_t, logq_sampled=lq_s)
    _cache[key] = out + ((sampled, lq_t, lq_s),)
    return _cache[key]


@pytest.mark.parametrize("det", [0, 1])
@pytest.mark.parametrize("math", MODES)
@pytest.mark.parametrize("S", [1, 25, 64, 65, 1024])
@pytest.mark.parametrize("B", [65, 200, 1024])
def test_sampled_softmax(B, S, math, det):
    import torch
    params, batch, ref, _, (sampled, lq_t, lq_s) = sampled_case(B, S)
    eng, _ = make_engine(SAMP, max_batch=B, params=params)
    eng.set_option("math_mode", math)
    eng.set_option("deterministic", det)
    d = dev_batch(eng, *batch)
    loss = float(eng.sampled_train_step(*d, eng.to_device(sampled, torch.int32), eng.to_device(lq_t, torch.float32),
                                        eng.to_device(lq_s, torch.float32), keep=KEEP, seed=SEED, step=1).cpu()[0])
    assert abs(loss - ref.loss) < LOSS_TOL
    g = eng.export_grads()
    label = "sampled B=%d S=%d math=%d det=%d" % (B, S, math, det)
    worst = R.check_step(g, ref, TAU[math], SLICE[math], label=label + " ")
    worst["loss"] = abs(loss - ref.loss)
    report(label, worst)
    eng.close()


@pytest.mark.parametrize("math", MODES)
def test_sampled_trainer_lazy_target(math):
    """Trainer.step_device_sampled with lazy Adam: the target table's rows are updated lazily too."""
    import torch
    from code2vec_b200.trainer import Trainer
    params, batch, ref, _, (sampled, lq_t, lq_s) = sampled_case(200, 64)
    eng, _ = make_engine(SAMP, max_batch=200, params=params)
    eng.set_option("math_mode", math)
    tr = Trainer(eng, keep_prob=KEEP, seed=SEED)
    assert eng.get_option("lazy_adam") == 1
    loss = float(tr.step_device_sampled(*dev_batch(eng, *batch), eng.to_device(sampled, torch.int32),
                                        eng.to_device(lq_t, torch.float32), eng.to_device(lq_s, torch.float32)).cpu()[0])
    assert abs(loss - ref.loss) < LOSS_TOL
    eng.sync_tables()
    label = "sampled-trainer math=%d" % math
    worst = check_adam_slots(eng, ref, math, O.PARAM_NAMES, label)
    worst["loss"] = abs(loss - ref.loss)
    report(label, worst)
    eng.close()


# ---- 7. evaluation -------------------------------------------------------------------------------------------------

def check_topk(eng, math, batch, fwd, k, normalize, params, label, min_frac=0.95):
    """Top-k indices through check_topk_rows; values (raw scores, or full-softmax probabilities for normalize = 2)
    element by element against M on the rows whose indices are compared."""
    from tests.test_gpu_parity import check_topk_rows
    top = R.topk64(params, fwd.vals["v"], fwd.mags["v"], k)
    code, _ = eng.forward(*dev_batch(eng, *batch[:4]), want_attention=False)
    idx, val = eng.topk(code, normalize=normalize)
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    kk = min(k, params["tgt"].shape[0])
    assert idx.shape == val.shape == (batch[0].shape[0], kk)
    ok, _ = check_topk_rows(idx, top["idx"][:, :kk], top["s"], kk, min_frac=min_frac)
    ref, M = (top["p"], top["Mp"]) if normalize == 2 else (top["s"], top["Ms"])
    worst = {"values": R.check_elementwise(label + " values", val[ok], ref[ok, :kk], M[ok, :kk], TAU[math]),
             "rows compared": float(ok.mean())}
    return worst, idx


@pytest.mark.parametrize("k,normalize", [(10, 0), (64, 0), (10, 2)])
def test_production_evaluation(k, normalize):
    """3xTF32 top-k at B = 1024 and Y = 261,246: several M tiles of the logits GEMM and both ends of the k range."""
    params, batch, _, fwd = prod_case("uniform")
    eng, _ = make_engine(PROD, max_batch=PROD_B, top_k=k, training=False, params=params)
    eng.set_option("math_mode", 2)
    label = "eval k=%d normalize=%d" % (k, normalize)
    # among the top 65 of 261,246 scores the median neighbour gap is 8e-7, below check_topk_rows' 1e-6: 44 % of the rows
    # (448) qualify at k = 64, 96 % at k = 10
    worst, _ = check_topk(eng, 2, batch, fwd, k, normalize, params, label, min_frac=0.95 if k <= 10 else 0.4)
    report(label, worst)
    eng.close()


@pytest.mark.parametrize("normalize", [0, 2])
@pytest.mark.parametrize("math", [0, 2])
def test_fewer_targets_than_k(math, normalize):
    """Y = 50 < top_k = 64: every row returns all min(k, Y) = 50 target rows, ranked."""
    dims = O.Dims(token_vocab=777, path_vocab=333, target_vocab=50, embed_dim=32, code_dim=96, max_contexts=20)
    params, batch, _, fwd = reference("small-y", dims, O.synthetic_batch(dims, 65, seed=50))
    eng, _ = make_engine(dims, max_batch=65, top_k=64, training=False, params=params)
    eng.set_option("math_mode", math)
    label = "eval Y=50 k=64 math=%d normalize=%d" % (math, normalize)
    worst, idx = check_topk(eng, math, batch, fwd, 64, normalize, params, label, min_frac=0.9)
    assert np.array_equal(np.sort(idx, axis=1), np.broadcast_to(np.arange(50), idx.shape))
    report(label, worst)
    eng.close()
