"""The unique log-uniform sampler of c2v_sample_log_uniform (include/c2v_b200.h, DESIGN.md §6j), stated in numpy.

Draw i of (seed, step) is Philox4x32-10 (oracle.philox4x32_10) at counter (i, 0, step_lo, step_hi) with the key
(seed_lo ^ 0x6C6F6775, seed_hi ^ 0x73616D70); u = ((x >> 5) 2^26 + (y >> 6)) 2^-53 and the class is
((int64)floor(exp(u log1p(Y))) - 1) mod Y.  The sample is the first S distinct classes in draw order and num_tries the
1-based index of the draw that supplied the S-th; the log expected counts follow TF's ExpectedCountHelper in double and are
rounded to float32 once."""
import numpy as np

from oracle import path_attention_oracle as O

KEY_XOR = (0x6C6F6775, 0x73616D70)
MAX_DRAWS = 1 << 31


def key(seed: int):
    return (seed & 0xFFFFFFFF) ^ KEY_XOR[0], ((seed >> 32) & 0xFFFFFFFF) ^ KEY_XOR[1]


def uniforms(seed: int, step: int, i0: int, n: int) -> np.ndarray:
    """u of draws i0 .. i0 + n - 1 (float64)."""
    k0, k1 = key(seed)
    i = np.arange(i0, i0 + n, dtype=np.uint64).astype(np.uint32)
    x, y, _, _ = O.philox4x32_10(i, np.uint32(0), np.uint32(step & 0xFFFFFFFF), np.uint32((step >> 32) & 0xFFFFFFFF), k0, k1)
    return ((x >> np.uint32(5)).astype(np.float64) * 67108864.0 + (y >> np.uint32(6)).astype(np.float64)) * 2.0 ** -53


def draws(seed: int, step: int, Y: int, i0: int, n: int) -> np.ndarray:
    """The classes of draws i0 .. i0 + n - 1 (int64)."""
    u = uniforms(seed, step, i0, n)
    return (np.floor(np.exp(u * np.log1p(float(Y)))).astype(np.int64) - 1) % Y


def prob(c, Y: int) -> np.ndarray:
    c = np.asarray(c, dtype=np.float64)
    return np.log((c + 2.0) / (c + 1.0)) / np.log1p(float(Y))


def expected_count64(c, Y: int, S: int, tries: int) -> np.ndarray:
    """The expected counts in float64, before the log."""
    p = prob(c, Y)
    if tries == S:
        return S * p
    return -np.expm1(float(tries) * np.log1p(-p))


def logq(c, Y: int, S: int, tries: int) -> np.ndarray:
    return np.log(expected_count64(c, Y, S, tries)).astype(np.float32)


def sample(S: int, Y: int, seed: int, step: int, block: int = 4096):
    """(sampled int32 [S], num_tries) of the statement, drawing `block` values at a time."""
    if not 1 <= S <= min(1024, Y // 2):
        raise ValueError("S out of range")
    seen = {}
    out = []
    i0 = 0
    while i0 < MAX_DRAWS:
        vals = draws(seed, step, Y, i0, block)
        for j, v in enumerate(vals.tolist()):
            if v not in seen:
                seen[v] = True
                out.append(v)
                if len(out) == S:
                    return np.array(out, dtype=np.int32), i0 + j + 1
        i0 += block
    raise RuntimeError("draw cap reached")


def sample_with_logq(S: int, Y: int, target, seed: int, step: int):
    """(sampled, num_tries, logq_true [B] float32, logq_sampled [S] float32)."""
    sampled, tries = sample(S, Y, seed, step)
    return sampled, tries, logq(np.asarray(target), Y, S, tries), logq(sampled, Y, S, tries)
