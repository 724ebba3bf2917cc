"""Builds libc2v_batcher.so (host-side native tensoriser) in-tree with g++."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "batcher.cpp")
LIB = os.path.join(HERE, "libc2v_batcher.so")


def needs_build() -> bool:
    # this file counts as a source: it holds the compiler flags
    newest = max(os.path.getmtime(SRC), os.path.getmtime(os.path.abspath(__file__)))
    return (not os.path.exists(LIB)) or os.path.getmtime(LIB) < newest


def build(force: bool = False) -> str:
    if force or needs_build():
        tmp = LIB + ".tmp"
        subprocess.check_call(["g++", "-O3", "-std=c++17", "-shared", "-fPIC", "-pthread", SRC, "-o", tmp])
        os.replace(tmp, LIB)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
