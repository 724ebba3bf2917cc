"""Times the tensor-core (wgmma) GEMM kernels alone (c2v_selftest_gemm) at the shapes of the train step."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from code2vec_b200.engine import EngineDims, PathAttentionEngine  # noqa: E402

eng = PathAttentionEngine(EngineDims(101, 51, 101, 32, 96, 20, 8, 10), device=0, training=True)   # any engine: the GEMM self-test only needs a handle
eng.init_params()
def bench(M, N, K, a_mn, b_mn, bn, splits, pair, reps=10):
    eng.set_option("cta_pair", pair)
    A = torch.randn((K, M) if a_mn else (M, (K + 63)//64*64), device="cuda")
    B = torch.randn((K, N) if b_mn else (N, K), device="cuda")
    for _ in range(2): eng.selftest_gemm(A, B, a_mn, b_mn, M, N, K, bn=bn, splits=splits)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): eng.selftest_gemm(A, B, a_mn, b_mn, M, N, K, bn=bn, splits=splits)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    print("M=%d N=%d K=%d a_mn=%d b_mn=%d bn=%d splits=%d pair=%d : %.3f ms  %.0f TFLOP/s (incl. slice sum)" % (M, N, K, a_mn, b_mn, bn, splits, pair, ms, 2.0*M*N*K/ms/1e9))
for pair in (0, 1):
    print("--- logits-like"); bench(1024, 261248, 384, False, False, 256, 1, pair)
    print("--- dv-like N=1"); [bench(1024, 384, 261246, False, True, 192, s, pair) for s in (18,)]
    print("--- dv-like N=8 shard"); [bench(8192, 384, 32656, False, True, 192, s, pair) for s in (1, 3, 6, 18)]
    print("--- dY-like"); bench(261248, 384, 1024, True, True, 192, 1, pair)
    print("--- ctx-like"); bench(204800, 384, 384, False, True, 192, 1, pair)
    print("--- dW-like"); bench(384, 384, 204800, True, True, 192, 48, pair)
