"""Times the tensor-core (wgmma) GEMM kernel alone (c2v_selftest_gemm, plain store epilogue) at the shapes of the
java14m train step (B = 1024, C = 200), each product in the operand layout the engine uses and, on transposed
copies made by torch, in the all-K-major layout.  The all-K-major time is the ceiling to compare against: there
both operands go from TMA straight to wgmma, with no transpose in shared memory.

    python tools/gemm_micro.py [--reps 20]
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from code2vec_b200.engine import EngineDims, PathAttentionEngine  # noqa: E402

B, CTX, d, D, Y = 1024, 200, 128, 384, 261246
N_CTX = B * CTX
# name, M, N, K, (A MN-major, B MN-major) as the engine issues it, split-K slices (dW: engine.cu's kSplitDw; dv: what
# run_dv picks on 132 SMs, two waves of 128 x 128 tiles)
SHAPES = [
    ("ctx_fwd  X'.W", N_CTX, D, 3 * d, (False, True), 1),
    ("logits   v.Ytab^T", B, Y, D, (False, False), 1),
    ("dx_gemm  dU.W^T", N_CTX, 3 * d, D, (False, False), 1),
    ("dW       X'^T.dU", 3 * d, D, N_CTX, (True, True), 48),
    ("dv       P.Ytab", B, D, Y, (False, True), 11),
    ("dY       P^T.v", Y, D, B, (True, True), 1),
]


def padded(rows, cols):
    """[rows, cols] fp32 with the row pitch rounded up to 4 floats (TMA: 16-byte row pitch)"""
    return torch.empty((rows, (cols + 3) // 4 * 4), device="cuda").normal_()[:, :cols]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    eng = PathAttentionEngine(EngineDims(101, 51, 101, 32, 96, 20, 8, 10), device=0, training=True)  # a handle for the self-test
    print(torch.cuda.get_device_name(0))

    def time_gemm(A, Bm, a_mn, b_mn, M, N, K, splits, out):
        def run():
            rc = eng.lib.c2v_selftest_gemm(eng.h, int(a_mn), int(b_mn), 192, M, N, K, splits, A.data_ptr(), A.stride(0),
                                           Bm.data_ptr(), Bm.stride(0), out.data_ptr(), out.stride(1), eng._stream())
            if rc < 0:
                eng._check(rc)
        for _ in range(2):
            run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            run()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.reps

    for name, M, N, K, (a_mn, b_mn), splits in SHAPES:
        A = padded(K, M) if a_mn else padded(M, K)
        Bm = padded(K, N) if b_mn else padded(N, K)
        out = torch.empty((splits, M, (N + 3) // 4 * 4), device="cuda")     # the epilogue stores float4s: 16-byte row pitch
        flop = 2.0 * M * N * K
        ms = time_gemm(A, Bm, a_mn, b_mn, M, N, K, splits, out)
        line = "%-20s M=%-6d N=%-6d K=%-6d splits=%-2d  engine layout (a_mn=%d b_mn=%d): %7.3f ms %6.1f TFLOP/s" % (
            name, M, N, K, splits, a_mn, b_mn, ms, flop / ms / 1e9)
        if a_mn or b_mn:
            Ak = padded(M, K) if a_mn else A
            Bk = padded(N, K) if b_mn else Bm
            if a_mn:
                Ak.copy_(A.t())
            if b_mn:
                Bk.copy_(Bm.t())
            del A, Bm
            ms_k = time_gemm(Ak, Bk, False, False, M, N, K, splits, out)
            line += "   all-K-major: %7.3f ms %6.1f TFLOP/s" % (ms_k, flop / ms_k / 1e9)
        print(line, flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
