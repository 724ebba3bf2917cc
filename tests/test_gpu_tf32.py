"""The tensor-core path (math_mode = tf32: wgmma tf32, fp32 accumulate) against the fp32
oracle.  tf32 operands keep 10 mantissa bits, so outputs are compared at tf32-level tolerances
(stated per assertion); the loss bound of BASELINE.json (1e-4) still holds."""
import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests.util import dev_batch, make_engine, rel_err

pytestmark = pytest.mark.gpu

TINY = O.Dims(token_vocab=1001, path_vocab=501, target_vocab=1001, embed_dim=32, code_dim=96, max_contexts=20)
ODD = O.Dims(token_vocab=777, path_vocab=333, target_vocab=1537, embed_dim=20, code_dim=52, max_contexts=13)
MID = O.Dims(token_vocab=5003, path_vocab=3001, target_vocab=4099, embed_dim=128, code_dim=384, max_contexts=200)
# BASELINE config 5's model shape (d=256, D=768, 200 contexts) at a vocabulary the oracle finishes in seconds
LARGE = O.Dims(token_vocab=3001, path_vocab=2003, target_vocab=2600, embed_dim=256, code_dim=768, max_contexts=200)


@pytest.mark.parametrize("dims,B", [(TINY, 64), (ODD, 37), (MID, 48), (LARGE, 12)])
def test_tf32_forward_and_topk(dims, B):
    eng, params = make_engine(dims, max_batch=B)
    eng.set_option("math_mode", 1)
    assert eng.get_option("math_mode") == 1
    src, pth, tgt, mask, _ = O.synthetic_batch(dims, B, seed=11)
    idx_ref, val_ref, v_ref, alpha_ref, scores = O.evaluate_topk(params, src, pth, tgt, mask, k=10)
    code, attn = eng.forward(*dev_batch(eng, src, pth, tgt, mask))
    assert rel_err(code.cpu().numpy(), v_ref) < 3e-3
    assert np.abs(attn.cpu().numpy() - alpha_ref).max() < 2e-3
    idx, val = eng.topk(code)
    assert np.abs(val.cpu().numpy() - val_ref).max() < 3e-3 * max(1.0, np.abs(val_ref).max())
    # top-1 agrees wherever the fp32 margin exceeds the tf32 error bound
    srt = -np.sort(-scores, axis=1)
    clear = (srt[:, 0] - srt[:, 1]) > 2e-3
    assert np.array_equal(idx.cpu().numpy()[clear, 0], idx_ref[clear, 0])


@pytest.mark.parametrize("cta_pair", [0, 1, 2])
@pytest.mark.parametrize("dims,B", [(TINY, 64), (ODD, 37), (MID, 48), (LARGE, 12)])
def test_tf32_train_step(dims, B, cta_pair):
    eng, params = make_engine(dims, max_batch=B)
    eng.set_option("math_mode", 1)
    eng.set_option("cta_pair", cta_pair)
    src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=21)
    src[0, 0] = tgt[0, 0] = src[1, 0] = 3
    dm = O.dropout_keep_mask(seed=5, step=2, n_rows=B * dims.max_contexts, ctx_dim=dims.ctx_dim, keep=0.75)
    loss_ref, g_ref, _ = O.train_loss_and_grads(params, src, pth, tgt, mask, target, keep=0.75, dropout_mask=dm)
    d = dev_batch(eng, src, pth, tgt, mask, target)
    loss = float(eng.train_step(*d, keep=0.75, seed=5, step=2).cpu()[0])
    assert abs(loss - loss_ref) < 1e-4                      # BASELINE.json's loss bound
    g = eng.export_grads()
    for k in O.PARAM_NAMES:
        assert rel_err(g[k], g_ref[k]) < 1e-2, k            # tf32 operands: ~1e-3 relative per product
    touched = np.zeros(dims.token_vocab, bool)
    touched[src[mask > 0]] = True
    touched[tgt[mask > 0]] = True
    assert np.all(g["tok"][~touched] == 0.0)
    # three optimizer steps stay close to the fp32 oracle trajectory
    params = {k: v.copy() for k, v in params.items()}
    eng.load_params(params)
    m = {k: np.zeros_like(p) for k, p in params.items()}
    v = {k: np.zeros_like(p) for k, p in params.items()}
    for t in (1, 2, 3):
        lr, gr, _ = O.train_loss_and_grads(params, src, pth, tgt, mask, target)
        O.adam_step(params, gr, m, v, t)
        l = float(eng.train_step(*d).cpu()[0])
        eng.adam_step()
        # same parameters (t = 1): BASELINE.json's 1e-4.  Later steps compare two TRAJECTORIES: Adam's first
        # updates are +-lr whatever the gradient's size, so a tf32-level difference in a near-zero gradient
        # element moves that parameter by a full step; at D = 768 the loss drifts by ~1e-4 after two of them.
        assert abs(l - lr) < (1e-4 if t == 1 or dims.code_dim <= 384 else 3e-4), (t, l, lr)


@pytest.mark.parametrize("dims,B,keep", [(TINY, 64, 1.0), (TINY, 64, 0.75), (MID, 48, 0.75), (LARGE, 12, 0.75), (MID, 3, 1.0)])
def test_fused_gather_projection_is_bit_identical_to_the_unfused_path(dims, B, keep):
    """umma::launch_ctx_fused (gather -> dropout -> wgmma projection -> tanh in one kernel) feeds the tensor core the same
    operand image TMA would have loaded from a materialised X', so everything downstream of it must carry the same
    bits as with option fuse_gather = 0: code vectors, attention, loss, and the gradients that do not go through
    float atomics (dW reads the X' the fused kernel wrote out)."""
    import torch
    src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=41)
    out = {}
    for fuse in (1, 0):
        eng, _ = make_engine(dims, max_batch=B)
        eng.set_option("math_mode", 1)
        eng.set_option("fuse_gather", fuse)
        assert eng.get_option("fuse_gather") == fuse
        d = dev_batch(eng, src, pth, tgt, mask, target)
        code, attn = eng.forward(*d[:4])
        loss = eng.train_step(*d, keep=keep, seed=11, step=3)
        torch.cuda.synchronize()
        out[fuse] = (code.cpu().numpy(), attn.cpu().numpy(), float(loss.cpu()[0]), eng.export_grads())
        eng.close()
    assert np.array_equal(out[1][0], out[0][0]) and np.array_equal(out[1][1], out[0][1])
    assert out[1][2] == out[0][2]
    for k in ("W", "a", "tgt"):
        assert np.array_equal(out[1][3][k], out[0][3][k]), k
    for k in ("tok", "path"):
        assert rel_err(out[1][3][k], out[0][3][k]) < 1e-5, k


@pytest.mark.parametrize("dims,B", [(TINY, 64), (ODD, 37), (MID, 48), (LARGE, 12)])
def test_softmax_gradient_computed_inside_the_gradient_gemms(dims, B):
    """Option fuse_softmax_grad (off by default): the dv = P.Ytab and dY = P^T.v GEMMs read the LOGITS slab and turn each A tile
    into (softmax - onehot)/B in shared memory (umma_gemm.cuh, AXSoftmaxGrad<true> / AXSoftmaxGrad<false>, in the GEMM's loaders) instead of reading a slab
    that a separate pass rewrote.  Same gradients as with the separate pass, to the rounding of one exp (ex2.approx vs expf
    on values that are then cut to tf32 anyway), and as the oracle's at the tf32 tolerance."""
    src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=51)
    out = {}
    for fuse in (1, 0):
        eng, params = make_engine(dims, max_batch=B)
        eng.set_option("math_mode", 1)
        eng.set_option("exp_slab", 0)                # compare against the two-pass schedule that stores logits
        eng.set_option("fuse_softmax_grad", fuse)
        assert eng.get_option("fuse_softmax_grad") == fuse
        loss = float(eng.train_step(*dev_batch(eng, src, pth, tgt, mask, target), keep=1.0).cpu()[0])
        out[fuse] = (loss, eng.export_grads())
        eng.close()
    assert out[1][0] == out[0][0]                       # the loss does not depend on it
    _, g_ref, _ = O.train_loss_and_grads(params, src, pth, tgt, mask, target)
    for k in O.PARAM_NAMES:
        assert rel_err(out[1][1][k], out[0][1][k]) < 2e-3, k
        assert rel_err(out[1][1][k], g_ref[k]) < 1e-2, k


@pytest.mark.parametrize("math", [1, 2])
@pytest.mark.parametrize("dims,B", [(TINY, 64), (ODD, 37), (MID, 48)])
def test_recomputed_logits_schedule_matches_the_stored_one(dims, B, math):
    """Option recompute_logits (off by default): the logits GEMM runs twice -- once leaving only the
    log-sum-exp partials, once writing (softmax - onehot)/B from its epilogue -- so the [B, Y] slab is written once and never
    rewritten.  The gradients must be those of the schedule that stores logits and rewrites them (same products, same exp),
    the loss may differ by the fp32-vs-tensor-core rounding of the one true-class logit per example."""
    src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=61)
    out = {}
    for rec in (1, 0):
        eng, params = make_engine(dims, max_batch=B)
        eng.set_option("math_mode", math)
        eng.set_option("exp_slab", 0)                # "the stored one" = the two-pass schedule
        eng.set_option("recompute_logits", rec)
        assert eng.get_option("recompute_logits") == rec
        loss = float(eng.train_step(*dev_batch(eng, src, pth, tgt, mask, target), keep=1.0).cpu()[0])
        out[rec] = (loss, eng.export_grads())
        eng.close()
    assert abs(out[1][0] - out[0][0]) < (2e-4 if math == 1 else 2e-6)
    loss_ref, g_ref, _ = O.train_loss_and_grads(params, src, pth, tgt, mask, target)
    assert abs(out[1][0] - loss_ref) < 1e-4
    for k in O.PARAM_NAMES:
        assert rel_err(out[1][1][k], out[0][1][k]) < (1e-4 if math == 1 else 2e-6), k
        assert rel_err(out[1][1][k], g_ref[k]) < (1e-2 if math == 1 else 5e-5), k


@pytest.mark.parametrize("math", [1, 2])
@pytest.mark.parametrize("dims,B", [(TINY, 64), (ODD, 37), (MID, 48), (LARGE, 12)])
def test_deferred_softmax_normalisation_matches_the_two_pass_schedule(dims, B, math):
    """Option exp_slab (default on in the tensor-core modes): the logits epilogue writes U = exp(s - true logit), the combine
    kernel patches one element per row and leaves a per-row factor 1/(B sum U) that the dv reduction and dY's small operand
    apply -- no pass rewrites the slab.  Same gradients as the two-pass schedule (logits stored, then rewritten to
    (softmax - onehot)/B) up to the rounding of one multiply per element; the loss uses the fp32 true-class logit instead of
    the tensor-core one, as recompute_logits does.  No step may have needed the device-side fallback."""
    src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=71)
    out = {}
    for slab in (1, 0):
        eng, params = make_engine(dims, max_batch=B)
        eng.set_option("math_mode", math)
        eng.set_option("exp_slab", slab)
        assert eng.get_option("exp_slab") == slab
        loss = float(eng.train_step(*dev_batch(eng, src, pth, tgt, mask, target), keep=1.0).cpu()[0])
        out[slab] = (loss, eng.export_grads())
        assert eng.get_option("exp_slab_fallbacks") == 0
        eng.close()
    assert abs(out[1][0] - out[0][0]) < (2e-4 if math == 1 else 2e-6)
    loss_ref, g_ref, _ = O.train_loss_and_grads(params, src, pth, tgt, mask, target)
    assert abs(out[1][0] - loss_ref) < (1e-4 if math == 1 else 5e-6)
    for k in O.PARAM_NAMES:
        assert rel_err(out[1][1][k], out[0][1][k]) < (2e-3 if math == 1 else 2e-5), k
        assert rel_err(out[1][1][k], g_ref[k]) < (1e-2 if math == 1 else 5e-5), k


@pytest.mark.parametrize("math", [1, 2])
def test_exp_slab_falls_back_on_the_device_when_a_row_leaves_the_fp32_window(math):
    """Logits hundreds of units apart: exp(s - true logit) overflows fp32 for some rows, the combine kernel raises the range
    flag and the gated kernels behind it redo the step's softmax as the two-pass schedule -- so the step's loss and
    gradients are exactly those of an engine with exp_slab off.  The flag is per step: the next step, on ordinary
    parameters, runs the deferred schedule again (the fallback counter stays at 1)."""
    dims, B = ODD, 37
    src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=81)
    wild = O.init_params(dims, seed=9)
    v, _, _ = O.forward(wild, src, pth, tgt, mask)
    spread = np.abs(O.logits_of(wild, v)).max()
    wild["tgt"] = (wild["tgt"] * np.float32(400.0 / spread)).astype(np.float32)       # logits up to +-400
    lg = O.logits_of(wild, v)
    assert (lg.max(axis=1) - lg[np.arange(B), target]).max() > 100
    calm = O.init_params(dims, seed=10)
    out = {}
    for slab in (1, 0):
        eng, _ = make_engine(dims, max_batch=B, params=wild)
        eng.set_option("math_mode", math)
        eng.set_option("exp_slab", slab)
        batch = dev_batch(eng, src, pth, tgt, mask, target)
        loss = float(eng.train_step(*batch, keep=1.0).cpu()[0])
        g = eng.export_grads()
        assert eng.get_option("exp_slab_fallbacks") == slab
        eng.load_params(calm)
        loss2 = float(eng.train_step(*batch, keep=1.0).cpu()[0])
        g2 = eng.export_grads()
        assert eng.get_option("exp_slab_fallbacks") == slab
        out[slab] = (loss, g, loss2, g2)
        eng.close()
    assert np.isfinite(out[1][0]) and out[1][0] == out[0][0]
    for k in ("tgt", "W", "a"):
        assert np.array_equal(out[1][1][k], out[0][1][k]), k
    for k in ("tok", "path"):                    # float atomics: the same addends in whatever order
        assert rel_err(out[1][1][k], out[0][1][k]) < 1e-5, k
    assert abs(out[1][2] - out[0][2]) < (2e-4 if math == 1 else 2e-6)
    for k in O.PARAM_NAMES:
        assert rel_err(out[1][3][k], out[0][3][k]) < (2e-3 if math == 1 else 2e-5), k
