"""Times the tensor-core (wgmma) GEMM kernel alone (c2v_selftest_gemm, plain store epilogue) at the shapes of the
java14m train step (B = 1024, C = 200), each product in the operand layout the engine uses and, on transposed
copies made by torch, in the all-K-major layout.  The all-K-major time is the ceiling to compare against: there
both operands go from TMA straight to wgmma, with no transpose in shared memory.  Where the engine now feeds a
K-major copy of an operand it stores MN-major (W^T, v^T, Ytab^T), the layout it used before is timed as well, and
so are the copies themselves (c2v_selftest_transpose; plain, and as the 3xTF32 split).  The logits GEMM is also timed
writing Ytab^T from its B tiles, as the train step runs it (c2v_selftest_gemm_bt), alternating with the plain product.

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
# name, M, N, K, (A MN-major, B MN-major) as the engine issues it, the layout it issued before it made K-major copies
# (None: unchanged), split-K slices (dW: engine.cu's kSplitDw; dv: what run_dv picks on 132 SMs, two waves of 128 x 128
# tiles)
SHAPES = [
    ("ctx_fwd  X'.W", N_CTX, D, 3 * d, (False, False), (False, True), 1),
    ("logits   v.Ytab^T", B, Y, D, (False, False), None, 1),
    ("dx_gemm  dU.W^T", N_CTX, 3 * d, D, (False, False), None, 1),
    ("dW       X'^T.dU", 3 * d, D, N_CTX, (True, True), None, 48),
    ("dv       P.Ytab", B, D, Y, (False, False), (False, True), 11),
    ("dY       P^T.v", Y, D, B, (True, False), (True, True), 1),
]
# the K-major copies the engine makes per step: name, rows, cols of the row-major operand, pitch of the copy
COPIES = [
    ("W^T", 3 * d, D, 3 * d),
    ("v^T", B, D, (B + 3) // 4 * 4),
    ("Ytab^T", Y, D, (Y + 63) // 64 * 64),
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
        return time_fn(run)

    def time_fn(run):
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

    for name, M, N, K, layout, before, splits in SHAPES:
        out = torch.empty((splits, M, (N + 3) // 4 * 4), device="cuda")     # the epilogue stores float4s: 16-byte row pitch
        flop = 2.0 * M * N * K
        line = "%-20s M=%-6d N=%-6d K=%-6d splits=%-2d" % (name, M, N, K, splits)
        runs = [("engine layout", layout)] + ([("before", before)] if before else [])
        if layout != (False, False):                                       # else the engine layout is the ceiling
            runs.append(("all-K-major", (False, False)))
        for label, (a_mn, b_mn) in runs:
            A = padded(K, M) if a_mn else padded(M, K)
            Bm = padded(K, N) if b_mn else padded(N, K)
            ms = time_gemm(A, Bm, a_mn, b_mn, M, N, K, splits, out)
            line += "   %s (a_mn=%d b_mn=%d): %7.3f ms %6.1f TFLOP/s" % (label, a_mn, b_mn, ms, flop / ms / 1e9)
            del A, Bm
            torch.cuda.empty_cache()
        print(line, flush=True)
        del out
        torch.cuda.empty_cache()

    # the logits GEMM with and without the Ytab^T write, alternated so that clock drift falls on both arms alike
    A, Bm = padded(B, D), padded(Y, D)
    out = torch.empty((B, (Y + 3) // 4 * 4), device="cuda")
    bt = torch.empty((D, (Y + 63) // 64 * 64), device="cuda")
    plain, write = [], []
    for _ in range(5):
        plain.append(time_gemm(A, Bm, False, False, B, Y, D, 1, out[None]))
        write.append(time_fn(lambda: eng.selftest_gemm_bt(A, Bm, B, Y, D, bt, out)))
    med = lambda xs: sorted(xs)[len(xs) // 2]
    print("%-20s plain: %s ms   + Ytab^T write: %s ms   median %.3f -> %.3f ms (+%.3f)" % (
        "logits   v.Ytab^T", " ".join("%.3f" % x for x in plain), " ".join("%.3f" % x for x in write), med(plain), med(write),
        med(write) - med(plain)), flush=True)
    del A, Bm, out, bt
    torch.cuda.empty_cache()

    for name, rows, cols, ld_t in COPIES:
        x = torch.empty((rows, cols), device="cuda").normal_()
        hi, lo = (torch.empty((cols, ld_t), device="cuda") for _ in range(2))
        line = "%-20s [%d, %d] -> [%d, %d]" % ("copy " + name, rows, cols, cols, ld_t)
        for label, split in [("tf32", False), ("3xTF32 split", True)]:
            def run():
                eng._check(eng.lib.c2v_selftest_transpose(eng.h, x.data_ptr(), rows, cols, hi.data_ptr(),
                                                          lo.data_ptr() if split else None, ld_t, eng._stream()))
            ms = time_fn(run)
            moved = 4.0 * rows * cols * (3 if split else 2)                 # read x, write the copy (split: two copies)
            line += "   %s: %7.4f ms %6.0f GB/s" % (label, ms, moved / ms / 1e6)
        print(line, flush=True)
        del x, hi, lo
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
