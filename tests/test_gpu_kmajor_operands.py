"""K-major copies of the operands the engine stores MN-major (W^T for ctx_fwd, v^T for dY, Ytab^T for dv; DESIGN.md
section 4.2).  Each copy is made from the current parameters inside the step that reads it: a table or TRANSFORM written
between steps through the parameter tensors, as a checkpoint restore does, must give exactly the step a fresh engine
initialised to those values gives.  The shape has B, Y, d and D off every tile and alignment size, so v^T's pitch is
padded (61 -> 64) and the tails of all three copies are read through TMA's zero fill."""
import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests.util import dev_batch, make_engine, rel_err

pytestmark = pytest.mark.gpu

DIMS = O.Dims(token_vocab=1001, path_vocab=501, target_vocab=1001, embed_dim=36, code_dim=100, max_contexts=20)
B, KEEP, SEED = 61, 0.75, 0x7A11
TOL = {1: 1e-2, 2: 5e-5}          # gradients, rel_err against the oracle
LOSS_TOL = {1: 2e-4, 2: 1e-5}


def _bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


def _engine(math, params):
    eng, _ = make_engine(DIMS, max_batch=B, params=params)
    eng.set_option("math_mode", math)
    eng.set_option("deterministic", 1)
    return eng


def _step(eng, api, batch, step):
    """One train step (keep 0.75) through the fused entry point or the phase-split one on a world of one; returns the loss."""
    import torch
    s, p, t, m, tg = batch
    if api == "fused":
        return float(eng.train_step(s, p, t, m, tg, keep=KEEP, seed=SEED, step=step).cpu()[0])
    f32 = dict(dtype=torch.float32, device=eng.dev)
    v, dv = torch.empty((B, DIMS.code_dim), **f32), torch.empty((B, DIMS.code_dim), **f32)
    rmax, rsum, tlogit, lse, loss = (torch.empty(n, **f32) for n in (B, B, B, B, 1))
    eng.context_forward(s, p, t, m, v, keep=KEEP, seed=SEED, step=step)
    eng.target_forward(v, tg, 0, rmax, rsum, tlogit)
    eng.lse_combine(rmax.view(1, B), rsum.view(1, B), tlogit, lse, loss)
    eng.target_backward(v, lse, tg, 0, dv)
    eng.context_backward(s, p, t, m, dv, keep=KEEP, seed=SEED, step=step)
    return float(loss.cpu()[0])


@pytest.mark.parametrize("rows,cols,ld_t", [(1001, 100, 1024), (61, 100, 64), (108, 100, 108), (33, 12, 36)])
def test_transposed_copy_is_the_transpose_bit_for_bit(rows, cols, ld_t):
    import torch
    eng, _ = make_engine(DIMS, max_batch=B, training=False)
    x = torch.from_numpy(np.random.default_rng(rows).standard_normal((rows, cols)).astype(np.float32)).cuda()
    xT = eng.selftest_transpose(x, ld_t)
    assert torch.equal(xT[:, :rows], x.t())
    hT, lT = eng.selftest_transpose(x, ld_t, split=True)
    h, lo = eng.selftest_split(x)
    assert torch.equal(hT[:, :rows], h.t()) and torch.equal(lT[:, :rows], lo.t())
    eng.close()


@pytest.mark.parametrize("api", ["fused", "phase_split"])
@pytest.mark.parametrize("math", [1, 2])
def test_parameters_written_between_steps_reach_the_transposed_operands(math, api):
    import torch
    rng = np.random.default_rng(17 + math)
    batches = [O.synthetic_batch(DIMS, B, seed=s) for s in (31, 32, 33)]
    eng = _engine(math, O.init_params(DIMS, seed=4321))
    # step 1 updates the target table in dY's epilogue and TRANSFORM in adam_step; step 2 has no Adam step, so the copies
    # it made describe the current parameters until the writes below
    eng.arm_target_adam(1)
    _step(eng, api, dev_batch(eng, *batches[0]), step=1)
    eng.adam_step(t=1)
    _step(eng, api, dev_batch(eng, *batches[1]), step=2)
    restored = {"tgt": rng.uniform(-0.2, 0.2, (DIMS.target_vocab, DIMS.code_dim)).astype(np.float32),
                "W": rng.uniform(-0.2, 0.2, (DIMS.ctx_dim, DIMS.code_dim)).astype(np.float32)}
    for k, x in restored.items():
        eng.params[k].copy_(torch.from_numpy(x))
    params = eng.export_params()
    for k, x in restored.items():
        assert np.array_equal(params[k], x), k
    loss = _step(eng, api, dev_batch(eng, *batches[2]), step=3)
    g = eng.export_grads()
    eng.close()

    fresh = _engine(math, params)
    loss_f = _step(fresh, api, dev_batch(fresh, *batches[2]), step=3)
    g_f = fresh.export_grads()
    fresh.close()
    assert loss == loss_f
    for k in O.PARAM_NAMES:
        assert np.array_equal(_bits(g[k]), _bits(g_f[k])), k

    dm = O.dropout_keep_mask(seed=SEED, step=3, n_rows=B * DIMS.max_contexts, ctx_dim=DIMS.ctx_dim, keep=KEEP)
    loss_ref, g_ref, _ = O.train_loss_and_grads(params, *batches[2], keep=KEEP, dropout_mask=dm)
    assert abs(loss - loss_ref) < LOSS_TOL[math]
    for k in O.PARAM_NAMES:
        assert rel_err(g[k], g_ref[k]) < TOL[math], k
