"""The wgmma GEMM in every operand layout is bit for bit the all-K-major product of the same matrices.

An MN-major operand reaches shared memory in 32 x 32 TMA boxes that the producer transposes in place into the
tile wgmma reads; the K-major tile comes from TMA as is.  Both must be the same bytes at the same swizzled
addresses (zero fill of M / N / K tails included), and the MMA issue order does not depend on the layout, so any
difference at all -- even one within the tf32 tolerance of tests/test_gpu_umma.py, such as two transposed elements
or a wrong lane in a tail box -- is a loader bug."""
import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests.util import make_engine

pytestmark = pytest.mark.gpu

TINY = O.Dims(token_vocab=101, path_vocab=51, target_vocab=101, embed_dim=32, code_dim=96, max_contexts=20)


@pytest.mark.parametrize("three", [False, True])
@pytest.mark.parametrize("a_mn,b_mn", [(False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,K,bn,splits", [(128, 192, 32, 192, 1), (256, 384, 384, 192, 1), (300, 200, 100, 192, 1),
                                              (1024, 1000, 384, 256, 1), (130, 384, 4100, 192, 7), (384, 384, 2000, 192, 48)])
def test_mn_major_layouts_are_bit_identical(a_mn, b_mn, M, N, K, bn, splits, three):
    import torch
    eng, _ = make_engine(TINY, max_batch=8)
    rng = np.random.default_rng(M * 7 + N * 3 + K)
    A = rng.standard_normal((M, K)).astype(np.float32)
    B = rng.standard_normal((K, N)).astype(np.float32)

    def dev(mat):          # row pitch padded to a multiple of 4 floats (TMA: 16-byte row pitch)
        r, c = mat.shape
        ld = (c + 3) // 4 * 4
        buf = torch.zeros((r, ld), dtype=torch.float32, device="cuda")
        buf[:, :c] = torch.from_numpy(np.ascontiguousarray(mat)).cuda()
        return buf
    ref = eng.selftest_gemm(dev(A), dev(B.T), False, False, M, N, K, bn=bn, splits=splits, three=three)
    C = eng.selftest_gemm(dev(A.T) if a_mn else dev(A), dev(B) if b_mn else dev(B.T), a_mn, b_mn, M, N, K, bn=bn,
                          splits=splits, three=three)
    torch.cuda.synchronize()
    diff = (C.view(torch.int32) != ref.view(torch.int32)).nonzero()
    assert diff.numel() == 0, "%d elements differ, first at %s" % (diff.shape[0], diff[0].tolist())
    assert C.abs().max().item() > 1.0
