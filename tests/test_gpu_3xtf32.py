"""C2V_MATH_3XTF32: the wgmma GEMM issued as a_lo.b_hi + a_hi.b_lo + a_hi.b_hi on tf32 (hi, lo) operand
splits, fp32 accumulation in registers -- fp32-equivalent results on the tensor cores.  The building block is
checked against a float64 product at an fp32-class bound (about 2000x tighter than the plain tf32 bound of
tests/test_gpu_umma.py) for every operand layout; the whole path in this mode runs the fp32 parity tests of
tests/test_gpu_parity.py (math = 2) at their fp32 tolerances."""
import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests.util import make_engine

pytestmark = pytest.mark.gpu

TINY = O.Dims(token_vocab=101, path_vocab=51, target_vocab=101, embed_dim=32, code_dim=96, max_contexts=20)


def test_split_is_exact_to_2_pow_minus_22():
    import torch
    eng, _ = make_engine(TINY, max_batch=8)
    rng = np.random.default_rng(0)
    x = (rng.standard_normal(1 << 16) * np.exp(rng.uniform(-20, 20, 1 << 16))).astype(np.float32)
    hi, lo = eng.selftest_split(torch.from_numpy(x).cuda())
    hi, lo = hi.cpu().numpy(), lo.cpu().numpy()
    # both parts are tf32 numbers (low 13 mantissa bits clear) and together reproduce x to 2^-22 relative
    assert np.all(hi.view(np.uint32) & 0x1FFF == 0) and np.all(lo.view(np.uint32) & 0x1FFF == 0)
    err = np.abs(hi.astype(np.float64) + lo.astype(np.float64) - x.astype(np.float64))
    assert np.all(err <= np.abs(x).astype(np.float64) * 2.0 ** -22)
    assert np.all(np.abs(lo) <= np.abs(x) * 2.0 ** -11 * 1.001)


@pytest.mark.parametrize("cta_pair", [0, 1])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,K,bn,splits", [(256, 384, 384, 192, 1), (300, 200, 100, 192, 1), (1024, 1000, 384, 256, 1),
                                              (130, 384, 4100, 192, 7)])
def test_3xtf32_gemm_matches_float64(a_mn, b_mn, M, N, K, bn, splits, cta_pair):
    import torch
    eng, _ = make_engine(TINY, max_batch=8)
    eng.set_option("cta_pair", cta_pair)
    rng = np.random.default_rng(M * 7 + N * 3 + K)
    A = rng.standard_normal((M, K)).astype(np.float32)
    B = rng.standard_normal((K, N)).astype(np.float32)

    def dev(mat):
        r, c = mat.shape
        ld = (c + 3) // 4 * 4
        buf = torch.zeros((r, ld), dtype=torch.float32, device="cuda")
        buf[:, :c] = torch.from_numpy(mat).cuda()
        return buf
    dA = dev(A.T.copy()) if a_mn else dev(A)
    dB = dev(B) if b_mn else dev(B.T.copy())
    C = eng.selftest_gemm(dA, dB, a_mn, b_mn, M, N, K, bn=bn, splits=splits, three=True).cpu().numpy()
    ref = A.astype(np.float64) @ B.astype(np.float64)
    absprod = np.abs(A).astype(np.float64) @ np.abs(B).astype(np.float64)
    err = np.abs(C - ref)
    # fp32-class: a sequential fp32 dot product of length K is bounded by K * 2^-24 * sum|a||b|; the split's own
    # error is ~3 * 2^-22 per product.  2e-6 * sum|a||b| covers both; plain tf32 needs 4e-3 (test_gpu_umma.py).
    assert np.all(err <= 2e-6 * absprod + 1e-7), "max err %g at %s (sum|a||b| %g)" % (
        err.max(), np.unravel_index(err.argmax(), err.shape), absprod.flat[err.argmax()])
    # and on average it is as good as numpy's own fp32 product
    err32 = np.abs((A @ B).astype(np.float64) - ref)
    assert err.mean() <= 4.0 * err32.mean() + 1e-9
