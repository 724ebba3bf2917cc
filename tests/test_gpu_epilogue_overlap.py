"""The GEMM's epilogue warpgroup drains a tile from the shared-memory staging blocks while the consumer warpgroups run
the MMAs of the CTA's next tile.  The shapes here give every CTA several work items, an uneven count per CTA (the last
wave is partial) and a last n-tile whose third 32-column quarter holds only 8 columns, so the hand-over of the staging
blocks runs many times in each CTA, including the drain of a quarter that is mostly padding and of one that is empty:

  * (M, N, K) = (33000, 200, 64): 258 m-tiles x 2 n-tiles = 516 work items, 3.9 per CTA on 132 SMs;
  * a target vocabulary of 40000 and code_dim 96: 313 dY tiles through the Adam epilogue, 2.4 per CTA.

Each case runs an existing check at the new shape: the product against float64 in every operand layout, every MN-major
layout bit for bit against the all-K-major product (tf32 and 3xTF32), and the Adam epilogue bit for bit against the
separate Adam pass."""
import pytest

from oracle import path_attention_oracle as O
from tests import test_gpu_fused_adam as fused_adam
from tests import test_gpu_umma as umma
from tests import test_gpu_umma_layouts as layouts

pytestmark = pytest.mark.gpu

MANY_ITEMS = (33000, 200, 64, 192, 1)       # M, N, K, bn, splits


@pytest.mark.parametrize("cta_pair", [0, 1])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
def test_gemm_matches_float64_with_several_tiles_per_cta(a_mn, b_mn, cta_pair):
    M, N, K, bn, splits = MANY_ITEMS
    umma.test_umma_gemm_matches_float64(a_mn, b_mn, M, N, K, bn, splits, cta_pair)


@pytest.mark.parametrize("three", [False, True])
@pytest.mark.parametrize("a_mn,b_mn", [(False, True), (True, False), (True, True)])
def test_mn_major_layouts_bit_identical_with_several_tiles_per_cta(a_mn, b_mn, three):
    M, N, K, bn, splits = MANY_ITEMS
    layouts.test_mn_major_layouts_are_bit_identical(a_mn, b_mn, M, N, K, bn, splits, three)


@pytest.mark.parametrize("cta_pair", [0, 1])
def test_fused_target_adam_bit_identical_with_several_tiles_per_cta(cta_pair):
    dims = O.Dims(token_vocab=5000, path_vocab=3000, target_vocab=40000, embed_dim=32, code_dim=96, max_contexts=16)
    fused_adam.test_fused_target_adam_is_bit_identical(dims, 64, cta_pair)
