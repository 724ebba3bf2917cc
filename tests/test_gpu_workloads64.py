"""Two of bench.py's training workloads against the float64 reference (tests/reference64.py), per element, at the shapes
they are timed at: the sampled-softmax step (`--mode sampled`) and the large model (`--workload large`).

Sampled softmax, java14m shape (B = 1024, C = 200, d = 128, D = 384, Y = 261,246; reduced token / path tables),
S in {25, 1024}: the ids are the device sampler's for (SEED, step 1), with one overwritten by a batch target (an accidental
hit) and one by a copy of another id (bench's host sampler draws duplicates).  At D = 384 the head kernels' loops over D
run three passes (one at the D = 96 of test_gpu_reference64's sampled cases).  Loss and the five gradients in fp32, tf32
and 3xTF32, the deterministic target-gradient kernel, and one lazy-Adam Trainer step through its Adam slots.

Large model, one GPU, real table sizes (T = 3,000,001, P = 2,000,001, d = 256, D = 768, C = 200, Y = 261,246; B = 512):
the token table alone is 3.07 GB, so any 32-bit byte offset into it would show here and nowhere else; the context GEMMs
run K = 768 and the row kernels take two 128-column passes.  The engine holds the real tables; the float64 reference
holds only the rows the batch touches (its tables are those rows, read from the engine after init_params, and its
indices remapped into them).  Every touched engine row is compared with its compacted reference row, and every other
gradient row, and after a Trainer step every other Adam-slot row, must be exactly zero (counted on the device).

Negative controls show each family can fail: the engine is fed a perturbation that a reference built from the perturbed
input would also carry -- logq_sampled shifted by 1e-3, and W's last 128 rows (the K range 640..767, which the java14m
shape never reaches) scaled by 1 + 1e-3 -- and checked against the true reference.  Perturbing the engine's input
rather than the reference's keeps one reference per family alive (about 4 GB and 8 GB of host memory).

Each reference is cached at module scope, built by the first test that needs it, and its build time is printed."""
import resource
import time
import types

import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests import reference64 as R
from tests.test_gpu_reference64 import (KEEP, LOSS_TOL, PROD, PROD_B, SEED, SLICE, TAU, check_adam_slots, check_forward,
                                        check_topk, report)
from tests.util import dev_batch, make_engine

pytestmark = pytest.mark.gpu

_cache = {}


@pytest.fixture(scope="module", autouse=True)
def _release_references():
    yield
    _cache.clear()


def cached(key, build):
    """One reference alive at a time: building `key` drops every other."""
    if key not in _cache:
        _cache.clear()
        t0, c0 = time.perf_counter(), time.process_time()
        _cache[key] = build()
        print("REF %s: %.1f s wall, %.1f s CPU, process peak RSS %.2f GB" % (
            key, time.perf_counter() - t0, time.process_time() - c0,
            resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1e6))
    return _cache[key]


# ---- 1. sampled softmax at the benchmark shape -----------------------------------------------------------------------

def sampled_case(S):
    """(params, batch, reference, (sampled, logq_true, logq_sampled)) of the java14m-shaped sampled step."""
    def build():
        import torch
        from tests.test_gpu_sampled_training import _sampler_engine
        params = O.init_params(PROD, seed=4321)
        batch = O.synthetic_batch(PROD, PROD_B, seed=4242)
        target = batch[4]
        eng = _sampler_engine(PROD.target_vocab)
        out = eng.sample_log_uniform(eng.to_device(target, torch.int32), S, SEED, 1)
        sampled, lq_t, lq_s = (t.cpu().numpy().copy() for t in out[:3])
        eng.close()
        assert len(np.unique(sampled)) == S
        sampled[0], lq_s[0] = target[3], lq_t[3]                    # an accidental hit
        sampled[1], lq_s[1] = sampled[2], lq_s[2]                   # a duplicate
        sampled[S - 1], lq_s[S - 1] = target[PROD_B - 1], lq_t[PROD_B - 1]     # a hit in the last 64-sample group
        dm = O.dropout_keep_mask(SEED, 1, PROD_B * PROD.max_contexts, PROD.ctx_dim, KEEP)
        ref = R.train_step64(params, *batch, keep=KEEP, dropout_mask=dm, sampled=sampled, logq_true=lq_t,
                             logq_sampled=lq_s)
        return params, batch, ref, (sampled, lq_t, lq_s)
    return cached(("sampled", S), build)


def run_sampled(eng, batch, ids, shift=0.0):
    """One sampled_train_step with logq_sampled + shift: (loss, gradients)."""
    import torch
    sampled, lq_t, lq_s = ids
    loss = eng.sampled_train_step(*dev_batch(eng, *batch), eng.to_device(sampled, torch.int32),
                                  eng.to_device(lq_t, torch.float32),
                                  eng.to_device(lq_s + np.float32(shift), torch.float32), keep=KEEP, seed=SEED, step=1)
    return float(loss.cpu()[0]), eng.export_grads()


# S = 1024 first, so the S = 25 reference built next serves the Trainer step and the control after it
@pytest.mark.parametrize("math,det", [(0, 0), (1, 0), (2, 0), (1, 1)])
@pytest.mark.parametrize("S", [1024, 25])
def test_sampled_production_shape(S, math, det):
    params, batch, ref, ids = sampled_case(S)
    eng, _ = make_engine(PROD, max_batch=PROD_B, params=params)
    eng.set_option("math_mode", math)
    eng.set_option("deterministic", det)
    label = "sampled-prod S=%d math=%d det=%d" % (S, math, det)
    loss, g = run_sampled(eng, batch, ids)
    assert abs(loss - ref.loss) < LOSS_TOL, (label, loss, ref.loss)
    worst = R.check_step(g, ref, TAU[math], SLICE[math], label=label + " ")
    worst["loss"] = abs(loss - ref.loss)
    report(label, worst)
    eng.close()


@pytest.mark.parametrize("math", [1, 2])
def test_sampled_production_trainer(math):
    """Trainer.step_device_sampled -- the step Trainer.step_sampled runs after its draw -- with lazy Adam on the target
    table as well, through the Adam slots."""
    import torch
    from code2vec_b200.trainer import Trainer
    params, batch, ref, (sampled, lq_t, lq_s) = sampled_case(25)
    eng, _ = make_engine(PROD, max_batch=PROD_B, params=params)
    eng.set_option("math_mode", math)
    tr = Trainer(eng, keep_prob=KEEP, seed=SEED)
    assert eng.get_option("lazy_adam") == 1
    loss = float(tr.step_device_sampled(*dev_batch(eng, *batch), eng.to_device(sampled, torch.int32),
                                        eng.to_device(lq_t, torch.float32), eng.to_device(lq_s, torch.float32)).cpu()[0])
    assert abs(loss - ref.loss) < LOSS_TOL, (loss, ref.loss)
    eng.sync_tables()
    label = "sampled-prod-trainer S=25 math=%d" % math
    worst = check_adam_slots(eng, ref, math, O.PARAM_NAMES, label)
    worst["loss"] = abs(loss - ref.loss)
    report(label, worst)
    eng.close()


def test_sampled_production_negative_control():
    """3xTF32, S = 25: the engine's logq_sampled shifted by 1e-3 (as a reference whose logq_sampled is shifted by -1e-3)
    fails the check that the true logq passes."""
    params, batch, ref, ids = sampled_case(25)
    eng, _ = make_engine(PROD, max_batch=PROD_B, params=params)
    eng.set_option("math_mode", 2)
    _, g = run_sampled(eng, batch, ids)
    R.check_step(g, ref, TAU[2], SLICE[2], label="control true logq ")
    _, g = run_sampled(eng, batch, ids, shift=1e-3)
    with pytest.raises(AssertionError):
        R.check_step(g, ref, TAU[2], SLICE[2], label="control shifted logq ")
    print("control logq + 1e-3: dY err/M %.3g" % R.err_ratio(g["tgt"], ref.vals["tgt"], ref.mags["tgt"])[0])
    eng.close()


# ---- 2. the large model on one GPU at its real table sizes -----------------------------------------------------------

LARGE = O.Dims(token_vocab=3000001, path_vocab=2000001, target_vocab=261246, embed_dim=256, code_dim=768, max_contexts=200)
LARGE_B = 512
HOT_TOK, HOT_PATH = 2999000, 1999000          # contended rows beyond 2 GiB and 1 GiB into their tables


def large_batch():
    """Uniform indices; a third of the valid entries of each table on one row (atomic contention); rows 0, T - 1 and
    P - 1 in valid slots (slot 0 of every bag is valid), and the last target class."""
    src, pth, tgt, mask, target = O.synthetic_batch(LARGE, LARGE_B, seed=2561)
    rng = np.random.default_rng(2562)
    valid = mask > 0
    for a, hot in ((src, HOT_TOK), (pth, HOT_PATH), (tgt, HOT_TOK)):
        a[valid & (rng.random(a.shape) < 0.32)] = hot
    src[0, 0], tgt[0, 0], pth[0, 0] = 0, LARGE.token_vocab - 1, LARGE.path_vocab - 1
    src[1, 0], tgt[1, 0], pth[1, 0] = LARGE.token_vocab - 1, 0, 0
    target[0] = LARGE.target_vocab - 1
    return src, pth, tgt, mask, target


def large_engine(math):
    from code2vec_b200.engine import EngineDims, PathAttentionEngine
    d = LARGE
    eng = PathAttentionEngine(EngineDims(d.token_vocab, d.path_vocab, d.target_vocab, d.embed_dim, d.code_dim,
                                         d.max_contexts, LARGE_B, 10), device=0, training=True)
    eng.init_params(seed=4321)
    eng.set_option("math_mode", math)
    return eng


def _rows(eng, t, rows):
    import torch
    return t[torch.from_numpy(rows.astype(np.int64)).to(eng.dev)].cpu().numpy()


def large_case(eng):
    """(compacted params, batch, compacted batch, token rows, path rows, train-step reference, forward reference).  The
    reference's tables are the rows the batch touches, masked slots included (their gradient must be exactly 0)."""
    def build():
        batch = large_batch()
        src, pth, tgt, mask, target = batch
        tok_rows, path_rows = np.unique(np.r_[src.ravel(), tgt.ravel()]), np.unique(pth.ravel())
        params = {"tok": _rows(eng, eng.params["tok"], tok_rows), "path": _rows(eng, eng.params["path"], path_rows),
                  **{k: eng.params[k].cpu().numpy() for k in ("tgt", "W", "a")}}
        cbatch = (np.searchsorted(tok_rows, src).astype(np.int32), np.searchsorted(path_rows, pth).astype(np.int32),
                  np.searchsorted(tok_rows, tgt).astype(np.int32), mask, target)
        dm = O.dropout_keep_mask(SEED, 1, LARGE_B * LARGE.max_contexts, LARGE.ctx_dim, KEEP)
        ref = R.train_step64(params, *cbatch, keep=KEEP, dropout_mask=dm)
        v, Mv, al, Mal = R.forward64(params, *cbatch[:4])
        fwd = R.Ref64(float("nan"), dict(v=v, alpha=al), dict(v=Mv, alpha=Mal), ref.targets)
        print("large case: %d token rows, %d path rows touched" % (len(tok_rows), len(path_rows)))
        return params, batch, cbatch, tok_rows, path_rows, ref, fwd
    case = cached("large", build)
    params, _, _, tok_rows, path_rows, _, _ = case
    # every engine starts from init_params(4321): the same values the reference was built from
    for k in ("W", "a"):
        assert np.array_equal(eng.params[k].cpu().numpy(), params[k]), k
    assert np.array_equal(_rows(eng, eng.params["tok"], tok_rows), params["tok"])
    assert np.array_equal(_rows(eng, eng.params["path"], path_rows), params["path"])
    return case


def stray_rows(eng, t, rows):
    """Rows of table tensor t outside `rows` holding any nonzero element, counted on the device."""
    import torch
    nz = torch.count_nonzero(t, dim=1)
    nz[torch.from_numpy(rows.astype(np.int64)).to(eng.dev)] = 0
    return int(torch.count_nonzero(nz).cpu())


def compacted(eng, tensors, tok_rows, path_rows):
    """{tok, path, tgt, W, a} of the engine's `tensors` with the tables restricted to the touched rows."""
    return {"tok": _rows(eng, tensors["tok"], tok_rows), "path": _rows(eng, tensors["path"], path_rows),
            **{k: tensors[k].cpu().numpy() for k in ("tgt", "W", "a")}}


@pytest.mark.parametrize("math", [0, 1, 2])
def test_large_model(math):
    eng = large_engine(math)
    params, batch, _, tok_rows, path_rows, ref, fwd = large_case(eng)
    label = "large math=%d" % math
    worst = check_forward(eng, math, batch, fwd, label)
    loss = float(eng.train_step(*dev_batch(eng, *batch), keep=KEEP, seed=SEED, step=1).cpu()[0])
    assert abs(loss - ref.loss) < LOSS_TOL, (label, loss, ref.loss)
    worst.update(R.check_step(compacted(eng, eng.grads, tok_rows, path_rows), ref, TAU[math], SLICE[math],
                              label=label + " "))
    worst["loss"] = abs(loss - ref.loss)
    for k, rows in (("tok", tok_rows), ("path", path_rows)):
        assert stray_rows(eng, eng.grads[k], rows) == 0, (label, k)
    report(label, worst)
    eng.close()


@pytest.mark.parametrize("math", [1, 2])
def test_large_model_trainer_adam_slots(math):
    """One Trainer("single") step (lazy Adam, target-table Adam fused into the dY epilogue) through its Adam slots;
    untouched rows of m and v exactly 0 after sync_tables."""
    from code2vec_b200.trainer import Trainer
    eng = large_engine(math)
    _, batch, _, tok_rows, path_rows, ref, _ = large_case(eng)
    tr = Trainer(eng, keep_prob=KEEP, seed=SEED)
    assert tr.schedule == "single" and eng.get_option("lazy_adam") == 1
    loss = float(tr.step_device(*dev_batch(eng, *batch)).cpu()[0])
    assert abs(loss - ref.loss) < LOSS_TOL, (loss, ref.loss)
    eng.sync_tables()
    import torch
    slots = types.SimpleNamespace(
        **{name: {k: torch.from_numpy(x) for k, x in compacted(eng, t, tok_rows, path_rows).items()}
           for name, t in (("adam_m", eng.adam_m), ("adam_v", eng.adam_v))})
    label = "large-trainer math=%d" % math
    worst = check_adam_slots(slots, ref, math, O.PARAM_NAMES, label)
    c1 = float(np.float32(1.0) - np.float32(0.9))
    got = {k: slots.adam_m[k].numpy().astype(np.float64) / c1 for k in O.PARAM_NAMES}
    worst.update({"slice:" + k: e for k, e in R.check_slices(got, ref, SLICE[math]).items()})
    worst["loss"] = abs(loss - ref.loss)
    for k, rows in (("tok", tok_rows), ("path", path_rows)):
        for slot in (eng.adam_m, eng.adam_v):
            assert stray_rows(eng, slot[k], rows) == 0, (label, k)
    report(label, worst)
    eng.close()


def test_large_model_evaluation():
    """3xTF32 top-10 at B = 512 and Y = 261,246 with D = 768."""
    eng = large_engine(2)
    params, batch, _, _, _, _, fwd = large_case(eng)
    label = "large eval k=10"
    worst, _ = check_topk(eng, 2, batch, fwd, 10, 0, params, label)
    report(label, worst)
    eng.close()


def test_large_model_negative_control():
    """3xTF32: the engine's W with its last 128 rows scaled by 1 + 1e-3 (as a reference whose W is scaled there) fails
    the check of the train step that test_large_model[2] passes with the true W."""
    eng = large_engine(2)
    _, batch, _, tok_rows, path_rows, ref, _ = large_case(eng)
    eng.params["W"][-128:] *= 1.0 + 1e-3
    eng.train_step(*dev_batch(eng, *batch), keep=KEEP, seed=SEED, step=1)
    got = compacted(eng, eng.grads, tok_rows, path_rows)
    with pytest.raises(AssertionError):
        R.check_step(got, ref, TAU[2], SLICE[2], label="control W ")
    print("control W[-128:] x (1 + 1e-3): err/M " + ", ".join(
        "%s %.3g" % (k, R.err_ratio(got[k], ref.vals[k], ref.mags[k])[0]) for k in O.PARAM_NAMES))
    eng.close()
