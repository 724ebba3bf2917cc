"""The wgmma (tf32) GEMM building block against a float64 product, for every operand
layout combination the engine uses, with M/N/K tails (zero fill) and split-K.
Tolerance: tf32 operands carry 10 mantissa bits -> relative error per product <= 2^-10; with
random data the result error is far below 4e-3 * sum_k |a||b|, while a wrong shared-memory
descriptor / swizzle gives O(1) errors."""
import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests.util import make_engine

pytestmark = pytest.mark.gpu

TINY = O.Dims(token_vocab=101, path_vocab=51, target_vocab=101, embed_dim=32, code_dim=96, max_contexts=20)


@pytest.mark.parametrize("cta_pair", [0, 1])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,K,bn,splits", [(128, 192, 32, 192, 1), (256, 384, 384, 192, 1), (300, 200, 100, 192, 1),
                                              (1024, 1000, 384, 256, 1), (130, 384, 4100, 192, 7), (384, 384, 2000, 192, 48)])
def test_umma_gemm_matches_float64(a_mn, b_mn, M, N, K, bn, splits, cta_pair):
    """cta_pair is accepted and ignored on sm_90a: both settings must give the same correct product."""
    import torch
    eng, _ = make_engine(TINY, max_batch=8)
    eng.set_option("cta_pair", cta_pair)
    rng = np.random.default_rng(M * 7 + N * 3 + K)
    A = rng.standard_normal((M, K)).astype(np.float32)
    B = rng.standard_normal((K, N)).astype(np.float32)
    # pitches padded to a multiple of 4 floats (TMA: 16-byte row pitch)
    def dev(mat):
        r, c = mat.shape
        ld = (c + 3) // 4 * 4
        buf = torch.zeros((r, ld), dtype=torch.float32, device="cuda")
        buf[:, :c] = torch.from_numpy(mat).cuda()
        return buf
    dA = dev(A.T.copy()) if a_mn else dev(A)             # [K, M] or [M, K]
    dB = dev(B) if b_mn else dev(B.T.copy())             # [K, N] or [N, K]
    C = eng.selftest_gemm(dA, dB, a_mn, b_mn, M, N, K, bn=bn, splits=splits).cpu().numpy()
    ref = A.astype(np.float64) @ B.astype(np.float64)
    bound = 4e-3 * (np.abs(A).astype(np.float64) @ np.abs(B).astype(np.float64))
    err = np.abs(C - ref)
    assert np.all(err <= bound + 1e-6), "max err %g (bound %g) at %s" % (err.max(), bound.flat[err.argmax()], np.unravel_index(err.argmax(), err.shape))
    # and it is not accidentally exact-zero output
    assert np.abs(C).max() > 1.0
