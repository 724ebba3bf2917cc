"""The float32 statement of one Adam step that every Adam path of the engine must reproduce bit for bit: adam_kernel,
the dY epilogue's update (umma::EpiAdam) and the lazy row replay (replay_row) all apply these correctly rounded
float32 operations in this order, with lr_t from oracle.adam_lr_t:

    m     <- fl(fl(m b1) + fl((1 - b1) g))
    v     <- fl(fl(v b2) + fl((1 - b2) fl(g g)))
    theta <- fl(theta - fl(fl(lr_t m) / fl(fl(sqrt(v)) + eps)))

numpy evaluates each float32 operation with IEEE round-to-nearest and keeps subnormals, as the kernels do (they are
built without -ftz / --use_fast_math).  NaN payloads are not part of the statement: compare NaN as NaN."""
import numpy as np

from oracle.path_attention_oracle import adam_lr_t

F = np.float32


def step(p, m, v, g, lr_t, b1, b2, eps):
    """One step in place on float32 arrays p, m, v with gradient g; lr_t, b1, b2, eps are rounded to float32."""
    lr_t, b1, b2, eps = F(lr_t), F(b1), F(b2), F(eps)
    with np.errstate(all="ignore"):
        m[...] = m * b1 + (F(1) - b1) * g
        v[...] = v * b2 + (F(1) - b2) * (g * g)
        p[...] = p - (lr_t * m) / (np.sqrt(v) + eps)


def step_t(p, m, v, g, t, lr=1e-3, b1=0.9, b2=0.999, eps=1e-8):
    """step() with the step size of Adam step t."""
    step(p, m, v, g, adam_lr_t(t, lr, b1, b2), b1, b2, eps)


def same_bits(a, b):
    """Element mask: identical float32 bit patterns, or both NaN."""
    a, b = np.asarray(a, dtype=F), np.asarray(b, dtype=F)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))
