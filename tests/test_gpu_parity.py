"""GPU parity: the CUDA path, called through the C ABI, against the CPU oracle on identical
seeded inputs.  Tolerances: integer outputs (top-k indices) bit-exact on batches whose top-(k+1)
logit gaps exceed GAP_EPS; fp32 outputs to the relative tolerances stated per test (the two
sides differ only in fp32 summation order); loss within 1e-4 absolute (BASELINE.json)."""
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

GAP_EPS = 1e-6
LOSS_TOL = 1e-4
# the two fp32-class arithmetic modes: 0 = fp32 FFMA on the SIMT pipe, 2 = 3xTF32 on the tensor cores (wgmma)
FP32_MODES = [0, 2]


def check_topk_rows(idx, idx_ref, scores, k, min_frac=0.95, gap_eps=GAP_EPS):
    """Top-k indices must be IDENTICAL on every row whose top-(k+1) neighbouring logit gaps all exceed gap_eps
    (fp32 summation order makes a smaller gap a coin flip for any implementation, TensorFlow included); at least
    min_frac of the rows must be in that set.  Returns the gap statistics for the test log."""
    srt = -np.sort(-scores, axis=1)[:, :min(k + 1, scores.shape[1])]
    gaps = (srt[:, :-1] - srt[:, 1:]).min(axis=1)
    ok = gaps > gap_eps
    stats = "rows %d, compared %d (%.1f %%), min/median top-(k+1) gap %.3g / %.3g" % (
        len(gaps), int(ok.sum()), 100.0 * ok.mean(), gaps.min(), np.median(gaps))
    print("top-k parity:", stats)
    assert ok.mean() >= min_frac, "parity batch has too many near-ties: " + stats
    assert np.array_equal(idx[ok], idx_ref[ok]), stats
    return ok, gaps


@pytest.mark.parametrize("math", FP32_MODES)
@pytest.mark.parametrize("dims,B", [(TINY, 64), (ODD, 37), (MID, 48), (LARGE, 12)])
def test_forward_matches_oracle(dims, B, math):
    eng, params = make_engine(dims, max_batch=B)
    eng.set_option("math_mode", math)
    src, pth, tgt, mask, _ = O.synthetic_batch(dims, B, seed=11)
    v_ref, alpha_ref, _ = O.forward(params, src, pth, tgt, mask)
    d = dev_batch(eng, src, pth, tgt, mask)
    code, attn = eng.forward(*d)
    code, attn = code.cpu().numpy(), attn.cpu().numpy()
    assert rel_err(code, v_ref) < 2e-5
    assert np.abs(attn - alpha_ref).max() < 2e-6
    assert np.all(attn[mask == 0] == 0.0)          # log(0) = -inf -> exact zeros
    np.testing.assert_allclose(attn.sum(axis=1), 1.0, atol=1e-5)


def test_all_masked_bag_is_nan():
    eng, params = make_engine(TINY, max_batch=8)
    src, pth, tgt, mask, _ = O.synthetic_batch(TINY, 8, seed=3)
    mask[5, :] = 0
    src[5], pth[5], tgt[5] = 0, 0, 0
    code, attn = eng.forward(*dev_batch(eng, src, pth, tgt, mask))
    code, attn = code.cpu().numpy(), attn.cpu().numpy()
    assert np.all(np.isnan(code[5])) and np.all(np.isnan(attn[5]))
    assert np.all(np.isfinite(np.delete(code, 5, axis=0)))


@pytest.mark.parametrize("math", FP32_MODES)
@pytest.mark.parametrize("dims,B,k", [(TINY, 64, 10), (ODD, 37, 10), (MID, 48, 10), (TINY, 16, 33), (LARGE, 12, 10)])
def test_topk_bit_exact(dims, B, k, math):
    eng, params = make_engine(dims, max_batch=B, top_k=k)
    eng.set_option("math_mode", math)
    src, pth, tgt, mask, _ = O.synthetic_batch(dims, B, seed=5)
    idx_ref, val_ref, v_ref, _, scores = O.evaluate_topk(params, src, pth, tgt, mask, k=k)
    code, _ = eng.forward(*dev_batch(eng, src, pth, tgt, mask))
    idx, val = eng.topk(code)
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    # rows whose top-(k+1) neighbouring gaps are all above GAP_EPS must match exactly, and >= 95 % of the rows are such
    check_topk_rows(idx, idx_ref, scores, k)
    assert np.abs(val - val_ref).max() < 1e-5
    # predict: softmax over the k values
    idx2, val2 = eng.topk(code, normalize=True)
    np.testing.assert_allclose(val2.cpu().numpy(), O.softmax_over_k(val_ref), atol=1e-6)


@pytest.mark.parametrize("math", FP32_MODES)
@pytest.mark.parametrize("dims,B,scale,seed", [(TINY, 64, 12.0, 70), (MID, 48, 60.0, 71)])
def test_topk_identical_on_trained_scale_parameters(dims, B, scale, seed, math):
    """north_star: "bit-exact top-k predictions".  A trained model's logit margins are far above fp32 rounding
    (its target rows and code vectors have grown away from the initialiser's +-0.09): with parameters of that
    scale EVERY row of the batch must give exactly the oracle's top-10, no row excluded."""
    params = {k: v.copy() for k, v in O.init_params(dims, seed=99).items()}
    params["tgt"] *= scale                                  # logits of magnitude 10 - 40 instead of < 1
    params["tok"] *= 3.0
    params["path"] *= 3.0
    eng, _ = make_engine(dims, max_batch=B, params=params)
    eng.set_option("math_mode", math)
    src, pth, tgt, mask, _ = O.synthetic_batch(dims, B, seed=seed)
    idx_ref, val_ref, _, _, scores = O.evaluate_topk(params, src, pth, tgt, mask, k=10)
    code, _ = eng.forward(*dev_batch(eng, src, pth, tgt, mask))
    idx, val = eng.topk(code)
    ok, gaps = check_topk_rows(idx.cpu().numpy(), idx_ref, scores, 10, min_frac=1.0, gap_eps=2e-4)
    assert ok.all() and gaps.min() > 2e-4                   # every margin is >= 20x the fp32 rounding of a logit
    assert np.array_equal(idx.cpu().numpy(), idx_ref)       # 100 % of the rows, all ten positions


def test_topk_ties_prefer_lower_index():
    eng, params = make_engine(TINY, max_batch=4)
    params = {k: v.copy() for k, v in params.items()}
    params["tgt"][7] = params["tgt"][3]            # identical rows -> identical scores
    params["tgt"][900] = params["tgt"][3]
    eng.load_params(params)
    import torch
    code = torch.from_numpy(np.tile(params["tgt"][3] * 50.0, (4, 1)).astype(np.float32)).cuda()
    idx, val = eng.topk(code)
    idx = idx.cpu().numpy()
    assert idx[:, :3].tolist() == [[3, 7, 900]] * 4


@pytest.mark.parametrize("math", FP32_MODES)
@pytest.mark.parametrize("dims,B", [(TINY, 64), (ODD, 37), (MID, 48), (LARGE, 12)])
def test_train_step_grads_match_oracle(dims, B, math):
    eng, params = make_engine(dims, max_batch=B)
    eng.set_option("math_mode", math)
    src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=21)
    src[0, 0] = tgt[0, 0] = src[1, 0] = 3          # duplicates across src/tgt and examples
    loss_ref, g_ref, aux = O.train_loss_and_grads(params, src, pth, tgt, mask, target)
    d = dev_batch(eng, src, pth, tgt, mask, target)
    loss = float(eng.train_step(*d).cpu()[0])
    assert abs(loss - loss_ref) < LOSS_TOL
    g = eng.export_grads()
    for k in O.PARAM_NAMES:
        assert rel_err(g[k], g_ref[k]) < 5e-5, k
    # rows never touched by a valid context are exactly zero
    touched = np.zeros(dims.token_vocab, bool)
    touched[src[mask > 0]] = True
    touched[tgt[mask > 0]] = True
    assert np.all(g["tok"][~touched] == 0.0)
    # a second step overwrites (does not accumulate into) the gradients
    loss2 = float(eng.train_step(*d).cpu()[0])
    g2 = eng.export_grads()
    assert abs(loss2 - loss) < 1e-6
    assert rel_err(g2["tok"], g_ref["tok"]) < 5e-5


@pytest.mark.parametrize("math", FP32_MODES)
def test_train_step_with_injected_and_philox_dropout(math):
    dims, B = TINY, 32
    eng, params = make_engine(dims, max_batch=B)
    eng.set_option("math_mode", math)
    src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=8)
    d = dev_batch(eng, src, pth, tgt, mask, target)
    import torch
    # (a) Philox mask regenerated by the oracle bit for bit
    dm = O.dropout_keep_mask(seed=0xC0FFEE1234, step=7, n_rows=B * dims.max_contexts, ctx_dim=dims.ctx_dim, keep=0.75)
    loss_ref, g_ref, _ = O.train_loss_and_grads(params, src, pth, tgt, mask, target, keep=0.75, dropout_mask=dm)
    loss = float(eng.train_step(*d, keep=0.75, seed=0xC0FFEE1234, step=7).cpu()[0])
    assert abs(loss - loss_ref) < LOSS_TOL
    g = eng.export_grads()
    for k in O.PARAM_NAMES:
        assert rel_err(g[k], g_ref[k]) < 5e-5, k
    # (b) caller-supplied mask
    rng = np.random.default_rng(0)
    dm2 = (rng.random((B * dims.max_contexts, dims.ctx_dim)) < 0.75).astype(np.float32)
    loss_ref2, g_ref2, _ = O.train_loss_and_grads(params, src, pth, tgt, mask, target, keep=0.75, dropout_mask=dm2)
    loss2 = float(eng.train_step(*d, keep=0.75, dropout_mask=torch.from_numpy(dm2).cuda()).cpu()[0])
    assert abs(loss2 - loss_ref2) < LOSS_TOL
    g2 = eng.export_grads()
    for k in O.PARAM_NAMES:
        assert rel_err(g2[k], g_ref2[k]) < 5e-5, k


@pytest.mark.parametrize("math", FP32_MODES)
def test_adam_three_steps_match_oracle(math):
    dims, B = TINY, 32
    eng, params = make_engine(dims, max_batch=B)
    eng.set_option("math_mode", math)
    params = {k: v.copy() for k, v in params.items()}
    src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=13)
    d = dev_batch(eng, src, pth, tgt, mask, target)
    m = {k: np.zeros_like(p) for k, p in params.items()}
    v = {k: np.zeros_like(p) for k, p in params.items()}
    for t in (1, 2, 3):
        loss_ref, g_ref, _ = O.train_loss_and_grads(params, src, pth, tgt, mask, target)
        O.adam_step(params, g_ref, m, v, t)
        loss = float(eng.train_step(*d).cpu()[0])
        eng.adam_step()
        assert abs(loss - loss_ref) < LOSS_TOL
    got = eng.export_params()
    for k in O.PARAM_NAMES:
        # after 3 steps of size ~1e-3 the parameters agree to a small fraction of one step
        assert np.abs(got[k] - params[k]).max() < 5e-5, k
    # untouched embedding rows did not move and their gradient buffers were cleared
    assert eng.grads["tok"].abs().max().item() == 0.0


@pytest.mark.parametrize("math", FP32_MODES)
def test_host_entry_points_match_device_entry_points(math):
    dims, B = TINY, 64
    eng, params = make_engine(dims, max_batch=B)
    eng.set_option("math_mode", math)
    src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=17)
    idx_ref, val_ref, v_ref, alpha_ref, _ = O.evaluate_topk(params, src, pth, tgt, mask, k=10, normalize=True)
    idx, val, code, attn = eng.predict_batch_host(src, pth, tgt, mask, normalize=True)
    assert rel_err(code, v_ref) < 2e-5
    assert np.abs(attn - alpha_ref).max() < 2e-6
    np.testing.assert_allclose(val, val_ref, atol=1e-6)
    n0 = eng.launch_count
    loss_ref, _, _ = O.train_loss_and_grads(params, src, pth, tgt, mask, target)
    loss = eng.train_batch_host(src, pth, tgt, mask, target, keep=1.0)
    assert abs(loss - loss_ref) < LOSS_TOL
    assert eng.launch_count - n0 >= 10            # the step really ran kernels of this library


def test_loss_entry_point():
    dims, B = ODD, 37
    eng, params = make_engine(dims, max_batch=B)
    src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=2)
    v_ref, _, _ = O.forward(params, src, pth, tgt, mask)
    loss_ref, _, _ = O.softmax_xent(O.logits_of(params, v_ref), target)
    d = dev_batch(eng, src, pth, tgt, mask, target)
    code, _ = eng.forward(*d[:4])
    assert abs(float(eng.loss(code, d[4]).cpu()[0]) - loss_ref) < LOSS_TOL


def test_error_behaviour():
    from code2vec_b200.engine import EngineDims, EngineError, PathAttentionEngine
    with pytest.raises(EngineError):
        PathAttentionEngine(EngineDims(10, 10, 10, 30, 96, 5, 4))       # embed_dim % 4 != 0
    eng, _ = make_engine(TINY, max_batch=4)
    src, pth, tgt, mask, target = O.synthetic_batch(TINY, 8, seed=1)
    with pytest.raises(EngineError):
        eng.forward(*dev_batch(eng, src, pth, tgt, mask))                # B > max_batch


@pytest.mark.parametrize("math", FP32_MODES)
@pytest.mark.parametrize("dims,B,S", [(TINY, 64, 25), (ODD, 37, 7), (MID, 48, 25)])
def test_sampled_softmax_train_step(dims, B, S, math):
    """BASELINE config 3.  Not in the reference (tensorflow_model.py:226-230 trains with the full
    softmax), so this pins the CUDA path to the oracle's stated definition only."""
    import torch
    eng, params = make_engine(dims, max_batch=B)
    eng.set_option("math_mode", math)
    src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=31)
    rng = np.random.default_rng(4)
    sampled = O.log_uniform_sample(rng, S, dims.target_vocab)
    sampled[0] = target[3]                           # an accidental hit
    sampled[1] = sampled[2]                          # a duplicate sampled class
    lq_t = O.log_uniform_logq(target, S, dims.target_vocab)
    lq_s = O.log_uniform_logq(sampled, S, dims.target_vocab)
    v_ref, alpha_ref, cache = O.forward(params, src, pth, tgt, mask)
    loss_ref, dv_ref, g_tgt_ref, _ = O.sampled_softmax_loss_and_grads(params, v_ref, target, sampled, lq_t, lq_s)
    # context gradients of the oracle given dv (reuse the full-softmax backward with dl replaced): recompute by hand
    d = dev_batch(eng, src, pth, tgt, mask, target)
    loss = float(eng.sampled_train_step(*d, eng.to_device(sampled, torch.int32), eng.to_device(lq_t, torch.float32),
                                        eng.to_device(lq_s, torch.float32)).cpu()[0])
    assert abs(loss - loss_ref) < LOSS_TOL
    g = eng.export_grads()
    assert rel_err(g["tgt"], g_tgt_ref) < 5e-5
    # chain dv through the oracle's context backward (same code path as the full softmax)
    hB, C_ = src.shape
    h = cache.h.reshape(hB, C_, -1)
    a = params["a"]
    dalpha = np.einsum("bcd,bd->bc", h, dv_ref)
    t = (alpha_ref * dalpha).sum(axis=1, keepdims=True)
    dz = alpha_ref * (dalpha - t)
    dh = alpha_ref[:, :, None] * dv_ref[:, None, :] + dz[:, :, None] * a[None, None, :]
    du = (dh * (1.0 - h * h)).reshape(hB * C_, -1).astype(np.float32)
    assert rel_err(g["a"], np.einsum("bc,bcd->d", dz, h)) < 5e-5
    assert rel_err(g["W"], cache.x.T @ du) < 5e-5
    dx = du @ params["W"].T
    g_tok = np.zeros_like(params["tok"]); g_path = np.zeros_like(params["path"])
    dd = dims.embed_dim
    np.add.at(g_tok, src.reshape(-1), dx[:, :dd]); np.add.at(g_path, pth.reshape(-1), dx[:, dd:2 * dd])
    np.add.at(g_tok, tgt.reshape(-1), dx[:, 2 * dd:])
    assert rel_err(g["tok"], g_tok) < 5e-5 and rel_err(g["path"], g_path) < 5e-5


def test_async_pinned_entry_point_matches_the_synchronous_one():
    """c2v_train_batch_async (uploads on the engine's copy stream, double-buffered staging, nothing waited for) against
    c2v_train_batch_host step by step: same losses, same model, and the upload-done events release the pinned buffers."""
    import torch
    dims, B = TINY, 64
    a, params = make_engine(dims, max_batch=B)
    b, _ = make_engine(dims, max_batch=B, params=params)
    steps = 6
    batches = [O.synthetic_batch(dims, B, seed=300 + s) for s in range(steps)]
    pinned = [[torch.from_numpy(np.ascontiguousarray(x)).pin_memory() for x in bt] for bt in batches]
    losses = torch.zeros(steps, dtype=torch.float32).pin_memory()
    events = []
    for s in range(steps):
        ev = torch.cuda.Event()
        a.train_batch_async(*pinned[s], rows=B, loss_out=losses[s:s + 1], upload_done=ev, keep=0.75, seed=7)
        events.append(ev)
    for ev in events:
        ev.synchronize()
    torch.cuda.synchronize()
    ref = [b.train_batch_host(*batches[s], keep=0.75, seed=7) for s in range(steps)]
    assert np.allclose(losses.numpy(), np.array(ref, dtype=np.float32), rtol=0, atol=1e-6)
    pa, pb = a.export_params(), b.export_params()
    for k in O.PARAM_NAMES:
        assert np.abs(pa[k] - pb[k]).max() < 2e-6, k
