"""Compare the '%f' formatter of csrc/float_text.cuh (format_fixed6, what the device predict route prints scores and
attention with) with C's printf("%f", (double)x) on all 2^32 float32 bit patterns (DESIGN.md §6i).

Python's '%f' % float(x) and glibc's printf("%f") both print the exact binary value rounded to six decimals, ties to
even; the tool first checks that the two agree on a seeded sample of 10^6 patterns (specials, ties and extremes
included), so the sweep's reference is Python's.  Every NaN prints "nan" in Python whatever its sign, so the sweep maps
printf's "-nan" to "nan".  The sweep itself is a small C++ program, compiled by nvcc from this file's source into a
temporary directory, that runs the same __host__ __device__ function the kernels run, on all cores.

    python tools/fixed_text_sweep.py [--threads N]

Prints one JSON line: the patterns compared, the mismatch count (with up to 10 examples) and the seconds taken.
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SWEEP = r'''
#include <stdio.h>
#include <string.h>
#include <atomic>
#include <thread>
#include <vector>
#include "float_text.cuh"

int main(int argc, char** argv) {
  const int threads = argc > 1 ? atoi(argv[1]) : 8;
  std::atomic<unsigned long long> bad{0};
  std::atomic<int> shown{0};
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; ++t) {
    pool.emplace_back([t, threads, &bad, &shown] {
      char ours[kFixedBytes + 1], ref[128];
      for (unsigned long long b = t; b < (1ull << 32); b += threads) {
        const unsigned int bits = (unsigned int)b;
        float x;
        memcpy(&x, &bits, 4);
        const int n = format_fixed6(x, ours);
        ours[n] = 0;
        if (x != x) strcpy(ref, "nan");
        else snprintf(ref, sizeof ref, "%f", (double)x);
        if (strcmp(ours, ref)) {
          ++bad;
          if (shown++ < 10) printf("MISMATCH %08x %s %s\n", bits, ours, ref);
        }
      }
    });
  }
  for (auto& th : pool) th.join();
  printf("BAD %llu\n", (unsigned long long)bad);
  return 0;
}
'''

PRINTF = r'''
#include <stdio.h>
#include <string.h>
int main() {
  unsigned int bits;
  while (fread(&bits, 4, 1, stdin) == 1) {
    float x;
    memcpy(&x, &bits, 4);
    if (x != x) printf("nan\n"); else printf("%f\n", (double)x);
  }
  return 0;
}
'''


def _sample(n: int) -> np.ndarray:
    rng = np.random.default_rng(32)
    special = np.array([0, 1 << 31, 1, 0x80000001, 0x007fffff, 0x00800000, 0x7f7fffff, 0xff7fffff, 0x7f800000, 0xff800000],
                       dtype=np.uint32)
    ties = np.float32([0.5e-6, 1.5e-6, 2.5e-6, 0.0078125, 1.0000005, 2.5]).view(np.uint32)
    return np.concatenate([special, ties, rng.integers(0, 1 << 32, size=n, dtype=np.uint64).astype(np.uint32)])


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--threads", type=int, default=os.cpu_count())
    a = ap.parse_args(argv)
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    tmp = tempfile.mkdtemp(prefix="c2v_fixed_sweep_")
    try:
        for name, src in (("sweep", SWEEP), ("printf", PRINTF)):
            with open(os.path.join(tmp, name + ".cu"), "w") as f:
                f.write(src)
            subprocess.run([nvcc, "-O2", "-std=c++17", "-I", os.path.join(ROOT, "code2vec_b200", "csrc"),
                            os.path.join(tmp, name + ".cu"), "-o", os.path.join(tmp, name)], check=True)
        # printf against Python on a sample: the sweep's reference is Python's '%f'
        bits = _sample(1000000)
        got = subprocess.run([os.path.join(tmp, "printf")], input=bits.tobytes(), capture_output=True,
                             check=True).stdout.decode().split("\n")[:-1]
        py = ["%f" % float(v) for v in bits.view(np.float32)]
        sample_bad = sum(1 for g, p in zip(got, py) if g != p)
        t0 = time.time()
        out = subprocess.run([os.path.join(tmp, "sweep"), str(a.threads)], capture_output=True, check=True,
                             text=True).stdout.splitlines()
        bad = int(out[-1].split()[1])
        print(json.dumps({"patterns": 1 << 32, "mismatches": bad, "examples": [l for l in out if l.startswith("MISMATCH")],
                          "printf_vs_python_sample": len(py), "printf_vs_python_mismatches": sample_bad,
                          "seconds": round(time.time() - t0, 1)}))
        return 0 if bad == 0 and sample_bad == 0 else 1
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    sys.exit(main())
