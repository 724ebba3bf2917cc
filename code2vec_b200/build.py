"""Builds libc2v_b200.so (the C-ABI shared library) in-tree with nvcc for sm_90a (H100).

The library is the product's only compute path; there is no CPU fallback.  `python -m
code2vec_b200.build` (or __graft_entry__.build()) cross-compiles without a GPU.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.path.join(PKG_DIR, "libc2v_b200.so")
OBJ_DIR = os.path.join(PKG_DIR, "csrc", "_obj")

SOURCES = ["engine.cu", "reader.cu", "text.cu", "preprocess.cu", "knn.cu", "predict.cu", "sampler.cu", "crc32c.cu",
           "corpus_text.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found: cannot build libc2v_b200.so")
    return exe


def _newest_source_mtime() -> float:
    m = 0.0
    for root in (CSRC, os.path.join(os.path.dirname(PKG_DIR), "include")):
        for dp, _, files in os.walk(root):
            if "_obj" in dp:
                continue
            for f in files:
                if f.endswith((".cu", ".cuh", ".h")):
                    m = max(m, os.path.getmtime(os.path.join(dp, f)))
    return m


def needs_build() -> bool:
    # this file counts as a source: it holds NVCC_FLAGS (the target architecture among them)
    newest = max(_newest_source_mtime(), os.path.getmtime(os.path.abspath(__file__)))
    return (not os.path.exists(LIB_PATH)) or os.path.getmtime(LIB_PATH) < newest


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB_PATH
    os.makedirs(OBJ_DIR, exist_ok=True)
    nvcc = _nvcc()

    def compile_one(src):
        obj = os.path.join(OBJ_DIR, os.path.splitext(src)[0] + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    tmp = LIB_PATH + ".tmp"
    r = subprocess.run([nvcc, "-shared", "-o", tmp, *objs, "-lcudart"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    os.replace(tmp, LIB_PATH)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
