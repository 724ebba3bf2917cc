"""Ytab^T, the K-major copy of the target table that dv reads, is written by the logits GEMM of the training step from the
Ytab tiles it streams (DESIGN.md section 4.2).  After a step it must hold exactly what the standalone transpose makes of the
table the step read -- tf32: the table, 3xTF32: its transposed split -- with the pitch padding columns untouched.  Shapes:
the java14m target table at B = 1024, and small tables whose last tile holds 1, 64 or 127 classes at batches under one
tile, with code_dim off the 32-wide K block.  A phase-split dv that no logits pass preceded makes the copy itself.  The
kernel option alone (c2v_selftest_gemm_bt): the product is the plain GEMM's, bit for bit, and B^T is B transposed."""
import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests.util import dev_batch, make_engine

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FBADBAD          # a NaN payload neither the copy nor a transpose can produce

# (name, dims, B); token / path tables are small: only the target table's shape matters here
SHAPES = {
    "java14m": (O.Dims(token_vocab=1001, path_vocab=501, target_vocab=261246, embed_dim=128, code_dim=384, max_contexts=8), 1024),
    "y_tail1": (O.Dims(token_vocab=1001, path_vocab=501, target_vocab=1025, embed_dim=36, code_dim=100, max_contexts=8), 61),
    "y_tail64": (O.Dims(token_vocab=1001, path_vocab=501, target_vocab=1088, embed_dim=32, code_dim=96, max_contexts=8), 100),
    "y_tail127": (O.Dims(token_vocab=1001, path_vocab=501, target_vocab=1151, embed_dim=36, code_dim=100, max_contexts=8), 127),
}
# the logits pass of each head schedule that writes the copy: U = exp(s - c) (exp_slab), logits + partials (two-pass),
# partials only (recompute)
SCHEDULES = {"exp_slab": {}, "two_pass": {"exp_slab": 0}, "recompute": {"recompute_logits": 1}}
CASES = [(s, m, h) for s in SHAPES for m in (1, 2) for h in SCHEDULES if s != "java14m" or h == "exp_slab"]


def _engine(shape, math, options=None):
    dims, B = SHAPES[shape]
    eng, _ = make_engine(dims, max_batch=B, params=O.init_params(dims, seed=77))
    eng.set_option("math_mode", math)
    for k, v in (options or {}).items():
        eng.set_option(k, v)
    return eng, dims, B


def _fill_sentinel(eng, math):
    import torch
    for lo in ([False, True] if math == 2 else [False]):
        eng.selftest_target_t(lo).view(torch.int32).fill_(SENTINEL)


def _check_copy(eng, math, table):
    """The workspace copy equals the standalone transpose of `table`; the padding still holds the sentinel."""
    import torch
    Y = table.shape[0]
    hi = eng.selftest_target_t()
    ld = hi.shape[1]
    if math == 2:
        want = eng.selftest_transpose(table, ld, split=True)
        got = (hi, eng.selftest_target_t(lo=True))
    else:
        want, got = (eng.selftest_transpose(table, ld),), (hi,)
    for g, w in zip(got, want):
        assert torch.equal(g[:, :Y].view(torch.int32), w[:, :Y].view(torch.int32))
        assert bool((g[:, Y:].view(torch.int32) == SENTINEL).all())


@pytest.mark.parametrize("M,N,K", [(61, 1025, 100), (128, 1088, 96), (200, 1151, 36), (1, 129, 4), (300, 4000, 384)])
def test_gemm_writes_b_transposed(M, N, K):
    import torch
    eng, _ = make_engine(SHAPES["y_tail1"][0], max_batch=8)
    g = torch.Generator(device="cuda").manual_seed(M * N + K)
    A = torch.randn((M, K), device="cuda", generator=g)
    Bm = torch.randn((N, K), device="cuda", generator=g)
    ld = (N + 63) // 64 * 64
    bt = torch.full((K, ld), 0.0, device="cuda")
    bt.view(torch.int32).fill_(SENTINEL)
    C = eng.selftest_gemm_bt(A, Bm, M, N, K, bt)
    if N % 4 == 0:              # selftest_gemm stores C at pitch N, which its float4 stores need 16-byte aligned
        assert torch.equal(C.view(torch.int32), eng.selftest_gemm(A, Bm, False, False, M, N, K).view(torch.int32))
    assert float((C - A @ Bm.t()).abs().max()) < 1e-2 * float((A @ Bm.t()).abs().max())
    assert torch.equal(bt[:, :N].view(torch.int32), Bm.t().contiguous().view(torch.int32))
    assert bool((bt[:, N:].view(torch.int32) == SENTINEL).all())
    eng.close()


@pytest.mark.parametrize("shape,math,schedule", CASES)
def test_logits_pass_writes_the_transposed_table(shape, math, schedule):
    eng, dims, B = _engine(shape, math, SCHEDULES[schedule])
    src, pth, tgt, mask, target = dev_batch(eng, *O.synthetic_batch(dims, B, seed=5))
    table = eng.params["tgt"].clone()           # no Adam step is armed: the step leaves the table as it is
    _fill_sentinel(eng, math)
    loss = eng.train_step(src, pth, tgt, mask, target, keep=0.75, seed=3, step=1)
    assert np.isfinite(float(loss.cpu()[0]))
    _check_copy(eng, math, table)
    eng.close()


@pytest.mark.parametrize("math", [1, 2])
def test_phase_split_dv_without_a_logits_pass_makes_the_copy(math):
    """target_backward after an Adam step, with no target_forward in between: the copy the last logits pass wrote describes
    the old table, so dv must transpose the current one itself."""
    import torch
    eng, dims, B = _engine("y_tail64", math)
    src, pth, tgt, mask, target = dev_batch(eng, *O.synthetic_batch(dims, B, seed=6))
    f32 = dict(dtype=torch.float32, device=eng.dev)
    v, dv = torch.empty((B, dims.code_dim), **f32), torch.empty((B, dims.code_dim), **f32)
    rmax, rsum, tlogit, lse, loss = (torch.empty(n, **f32) for n in (B, B, B, B, 1))
    eng.context_forward(src, pth, tgt, mask, v)
    eng.target_forward(v, target, 0, rmax, rsum, tlogit)
    eng.lse_combine(rmax.view(1, B), rsum.view(1, B), tlogit, lse, loss)
    eng.target_backward(v, lse, target, 0, dv)
    eng.context_backward(src, pth, tgt, mask, dv)
    before = eng.params["tgt"].clone()
    eng.adam_step(t=1)
    table = eng.params["tgt"].clone()
    assert not torch.equal(table, before)
    _fill_sentinel(eng, math)
    eng.target_backward(v, lse, target, 0, dv)
    torch.cuda.synchronize()
    _check_copy(eng, math, table)
    eng.close()
