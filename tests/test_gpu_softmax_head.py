"""Schedule choice of the softmax head (logits, cross-entropy, dL/dlogits, dv and dY).

The fused step picks one schedule from the math mode and the options, with a fixed precedence: recompute_logits
wins over exp_slab, fuse_softmax_grad switches both off, and in fp32 none of them applies.  An engine with a
combination of options must therefore compute exactly what the engine with only the winning option computes, with
the same kernel launches.  The phase-split entry points of the fully sharded schedule run the same head on one
engine (row offset 0, a world of one), and must agree with the fused step on the same batch."""
import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests.util import dev_batch, make_engine, rel_err

pytestmark = pytest.mark.gpu

ODD = O.Dims(token_vocab=777, path_vocab=333, target_vocab=1537, embed_dim=20, code_dim=52, max_contexts=13)
MID = O.Dims(token_vocab=5003, path_vocab=3001, target_vocab=4099, embed_dim=128, code_dim=384, max_contexts=200)
SHAPES = [(ODD, 37), (MID, 48)]


def _fused_step(dims, B, math, opts, seed):
    """One train_step with keep = 1.0: (loss, gradients, kernel launches of the step)."""
    src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=seed)
    eng, _ = make_engine(dims, max_batch=B)
    eng.set_option("math_mode", math)
    for k, val in opts.items():
        eng.set_option(k, val)
    batch = dev_batch(eng, src, pth, tgt, mask, target)
    n0 = eng.launch_count
    loss = float(eng.train_step(*batch, keep=1.0).cpu()[0])
    out = (loss, eng.export_grads(), eng.launch_count - n0)
    eng.close()
    return out


def _assert_same_step(a, b):
    assert a[0] == b[0]
    for k in ("tgt", "W", "a"):
        assert np.array_equal(a[1][k], b[1][k]), k
    for k in ("tok", "path"):                    # float atomics: the same addends in whatever order
        assert rel_err(a[1][k], b[1][k]) < 1e-5, k
    assert a[2] == b[2]


PRECEDENCE = [
    (1, dict(recompute_logits=1, exp_slab=1), dict(recompute_logits=1, exp_slab=0)),
    (2, dict(recompute_logits=1, exp_slab=1), dict(recompute_logits=1, exp_slab=0)),
    (1, dict(fuse_softmax_grad=1, exp_slab=1), dict(fuse_softmax_grad=1, exp_slab=0)),
    (2, dict(fuse_softmax_grad=1, exp_slab=1), dict(fuse_softmax_grad=1, exp_slab=0)),
    (1, dict(fuse_softmax_grad=1, recompute_logits=1, exp_slab=0), dict(fuse_softmax_grad=1, exp_slab=0)),
    (2, dict(fuse_softmax_grad=1, recompute_logits=1, exp_slab=0), dict(fuse_softmax_grad=1, exp_slab=0)),
    (2, dict(fuse_softmax_grad=1), dict(exp_slab=0)),                  # 3xTF32 has no loader form of the gradient
    (0, dict(recompute_logits=1), {}),                                 # fp32: no option changes the head
    (0, dict(exp_slab=0, fuse_softmax_grad=1), {}),
    (0, dict(recompute_logits=1, exp_slab=0, fuse_softmax_grad=1), {}),
]


@pytest.mark.parametrize("math,opts,winner", PRECEDENCE)
@pytest.mark.parametrize("dims,B", SHAPES)
def test_option_combination_runs_the_winning_schedule(dims, B, math, opts, winner):
    _assert_same_step(_fused_step(dims, B, math, opts, seed=91), _fused_step(dims, B, math, winner, seed=91))


@pytest.mark.parametrize("math,opts", [(0, {}), (1, {}), (1, dict(exp_slab=0)), (1, dict(exp_slab=0, fuse_softmax_grad=1)),
                                       (2, {}), (2, dict(exp_slab=0))])
@pytest.mark.parametrize("dims,B", SHAPES)
def test_phase_split_head_on_one_engine_matches_the_fused_step(dims, B, math, opts):
    """context_forward -> target_forward -> lse_combine -> target_backward -> context_backward on one engine with the
    whole target table (row offset 0, world 1) and no process group, against train_step on the same batch."""
    import torch
    loss_ref, g_ref, _ = _fused_step(dims, B, math, opts, seed=93)
    src, pth, tgt, mask, target = O.synthetic_batch(dims, B, seed=93)
    eng, _ = make_engine(dims, max_batch=B)
    eng.set_option("math_mode", math)
    for k, val in opts.items():
        eng.set_option(k, val)
    s, p, t, m, tg = dev_batch(eng, src, pth, tgt, mask, target)
    f32 = dict(dtype=torch.float32, device=eng.dev)
    v = torch.empty((B, dims.code_dim), **f32)
    rmax, rsum, tlogit = torch.empty(B, **f32), torch.empty(B, **f32), torch.empty(B, **f32)
    lse, loss = torch.empty(B, **f32), torch.empty(1, **f32)
    dv = torch.empty((B, dims.code_dim), **f32)
    eng.context_forward(s, p, t, m, v)
    eng.target_forward(v, tg, 0, rmax, rsum, tlogit)
    eng.lse_combine(rmax.view(1, B), rsum.view(1, B), tlogit, lse, loss)
    eng.target_backward(v, lse, tg, 0, dv)
    eng.context_backward(s, p, t, m, dv)
    got_loss = float(loss.cpu()[0])
    g = eng.export_grads()
    assert eng.get_option("exp_slab_fallbacks") == 0
    eng.close()
    assert abs(got_loss - loss_ref) < {0: 1e-5, 1: 2e-4, 2: 2e-6}[math]
    tol = {0: 5e-5, 1: 2e-3, 2: 2e-5}[math]
    for k in O.PARAM_NAMES:
        assert rel_err(g[k], g_ref[k]) < tol, k
