"""Compare the float32 formatter of csrc/text.cu with numpy on all 2^32 bit patterns (DESIGN.md §6f).

The formatter runs on the CPU through c2v_selftest_format_floats, the same __host__ __device__ function the device
kernel runs.  numpy's side is `x.astype("S16")`, numpy's own cast of a float32 array to bytes, which writes each value
as str(np.float32(x)) does (tests/test_device_text_model.py checks that the two agree) and is the fast way to ask
numpy for 2^32 strings.  Blocks of 2^22 patterns are spread over worker processes.

    python tools/float_text_sweep.py [--procs N] [--first BLOCK --last BLOCK]

Prints one JSON line: the patterns compared, the mismatch count (with up to 20 examples) and the longest text.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from multiprocessing import Pool

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BLOCK = 1 << 22
BLOCKS = (1 << 32) // BLOCK


def format_floats(lib, x: np.ndarray):
    """(text as an 'S16' array, lengths) of the float32 array x, by c2v_selftest_format_floats."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    out = np.zeros(x.size * 16, dtype=np.uint8)
    lens = np.zeros(x.size, dtype=np.int32)
    rc = lib.c2v_selftest_format_floats(x.ctypes.data, x.size, out.ctypes.data, lens.ctypes.data)
    if rc != 0:
        raise RuntimeError("c2v_selftest_format_floats failed: %d" % rc)
    return out.view("S16"), lens


def _block(i: int):
    from code2vec_b200 import engine
    lib = engine.load_library()
    bits = np.arange(i * BLOCK, (i + 1) * BLOCK, dtype=np.uint64).astype(np.uint32)
    x = bits.view(np.float32)
    ours, lens = format_floats(lib, x)
    ref = x.astype("S16")
    bad = np.nonzero(ours != ref)[0]
    j = int(np.argmax(lens))
    return (i, int(bad.size), [(hex(int(bits[k])), ours[k].decode(), ref[k].decode()) for k in bad[:20]],
            int(lens[j]), ours[j].decode())


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--procs", type=int, default=os.cpu_count())
    ap.add_argument("--first", type=int, default=0)
    ap.add_argument("--last", type=int, default=BLOCKS - 1)
    a = ap.parse_args(argv)
    from code2vec_b200 import engine
    engine.load_library()                       # builds the library once, before the workers load it
    t0 = time.time()
    mismatches, examples, longest, longest_text, done = 0, [], 0, "", 0
    with Pool(a.procs) as pool:
        for i, n_bad, ex, n_long, text in pool.imap_unordered(_block, range(a.first, a.last + 1)):
            mismatches += n_bad
            examples = (examples + ex)[:20]
            if n_long > longest:
                longest, longest_text = n_long, text
            done += 1
            if done % 64 == 0:
                print("%d / %d blocks, %d mismatches, %.0f s" % (done, a.last - a.first + 1, mismatches,
                                                                 time.time() - t0), file=sys.stderr, flush=True)
    print(json.dumps({"patterns": (a.last - a.first + 1) * BLOCK, "mismatches": mismatches, "examples": examples,
                      "longest": longest, "longest_text": longest_text, "seconds": round(time.time() - t0, 1),
                      "numpy": np.__version__}))
    return 0 if mismatches == 0 else 1


if __name__ == "__main__":
    sys.exit(main())
