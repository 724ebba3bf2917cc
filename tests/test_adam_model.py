"""The float32 Adam step every engine path reproduces (tests/adam_model.py) and its step size (oracle.adam_lr_t),
checked on the CPU: adam_lr_t against the host formula that engine.cu evaluates at each of its four sites, and the
float32 step against a float64 Adam driven by the same gradients, per element, within a rounding-error bound that is
accumulated operation by operation."""
import math
import os
import re

import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests import adam_model

F = np.float32
ENGINE_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "code2vec_b200", "csrc", "engine.cu")
HP = [(1e-3, 0.9, 0.999), (3e-2, 0.0, 0.9999), (2.5e-4, 0.95, 0.99), (1e-1, 0.5, 0.9)]


def _host_lr_t_sites():
    """(lr, beta2, t, beta1, t) variable names of every `lr * sqrt(1 - b2^t) / (1 - b1^t)` in engine.cu."""
    src = re.sub(r"\s+", " ", open(ENGINE_CU).read())
    pat = (r"\(double\)([\w>.-]+) \* sqrt\(1\.0 - pow\(\(double\)([\w>.-]+), \(double\)([\w>.-]+)\)\) / "
           r"\(1\.0 - pow\(\(double\)([\w>.-]+), \(double\)([\w>.-]+)\)\)")
    return re.findall(pat, src), src.count("sqrt(1.0 - pow(")


def _host_lr_t(t, lr, b1, b2):
    """engine.cu's formula in Python: double arithmetic on the float32 arguments, libm pow / sqrt, one cast to float."""
    lr, b1, b2 = float(F(lr)), float(F(b1)), float(F(b2))
    return F(lr * math.sqrt(1.0 - b2 ** float(t)) / (1.0 - b1 ** float(t)))


def test_every_host_site_evaluates_the_same_lr_t_formula():
    """c2v_adam_step, the armed dY epilogue, early_catchup and c2v_adam_step_range each compute lr_t on the host; the
    lazy replay reads the value c2v_adam_step (or early_catchup) stored, so all four must be the same expression."""
    sites, total = _host_lr_t_sites()
    assert total == 4 and len(sites) == 4, sites
    for lr, b2, t2, b1, t1 in sites:
        assert t1 == t2
        assert {lr, b1, b2} in ({"lr", "b1", "b2"}, {"lr", "beta1", "beta2"},
                                {"e->tgt_lr", "e->tgt_b1", "e->tgt_b2"}), (lr, b1, b2)


@pytest.mark.parametrize("lr,b1,b2", HP[:2])
def test_adam_lr_t_is_the_host_formula_for_a_million_steps(lr, b1, b2):
    for t in range(1, 10 ** 6 + 1):
        a, h = O.adam_lr_t(t, lr, b1, b2), _host_lr_t(t, lr, b1, b2)
        if a.view(np.uint32) != h.view(np.uint32):
            pytest.fail("t = %d: adam_lr_t %r, host %r" % (t, a, h))


def test_oracle_adam_step_uses_adam_lr_t():
    """The oracle's lr_t was once evaluated on the Python doubles 0.9 / 0.999, 72 float32 ulps away at t = 1."""
    p = {k: np.ones(4, F) for k in O.PARAM_NAMES}
    z = {k: np.zeros(4, F) for k in O.PARAM_NAMES}
    for t in (1, 2, 100, 1000, 65536):
        lr_t = O.adam_step(p, z, dict(z), dict(z), t)
        assert lr_t.view(np.uint32) == O.adam_lr_t(t).view(np.uint32)
    doubles = F(1e-3 * math.sqrt(1.0 - 0.999) / (1.0 - 0.9))
    assert int(doubles.view(np.int32)) - int(O.adam_lr_t(1).view(np.int32)) == 72


def _gradients(T, per_class, rng):
    """[T, n] float32 gradients, `per_class` columns of each kind: zero; subnormal; g^2 underflowing; sign alternating;
    scaled by 1e-6 and by 1e6; ordinary; sparse bursts; magnitudes spread over 10^-6 .. 10^6."""
    t = np.arange(1, T + 1)[:, None]
    shape = (T, per_class)
    sign = rng.choice([-1.0, 1.0], size=shape)
    cols = [
        np.zeros(shape),
        sign * rng.uniform(0.5, 1.0, shape) * 1e-40,
        sign * rng.uniform(0.5, 1.0, shape) * 1e-25,
        (-1.0) ** t * np.abs(rng.standard_normal(shape)) * 1e-2,
        (-1.0) ** t * np.ones(shape),
        rng.standard_normal(shape) * 1e-6,
        rng.standard_normal(shape) * 1e6,
        rng.standard_normal(shape) * 1e-2,
        np.where(rng.random(shape) < 0.05, rng.standard_normal(shape), 0.0),
        rng.standard_normal(shape) * 10.0 ** rng.uniform(-6, 6, shape),
    ]
    return np.concatenate(cols, axis=1).astype(F)


@pytest.mark.parametrize("lr,b1,b2,eps", [(1e-3, 0.9, 0.999, 1e-8), (3e-2, 0.0, 0.9999, 1e-3), (1e-1, 0.5, 0.9, 1e-8)])
def test_float32_step_follows_float64_adam_within_its_rounding_bound(lr, b1, b2, eps):
    """10^4 steps.  Every float32 operation rounds with a relative error of at most u = 2^-24, plus an absolute 2^-150
    where its result is subnormal; a bound on |x32 - x64| is carried for m, v and theta through the same operations
    (first order, each operand's error propagated with its derivative) and the float32 values must stay inside it.
    A bound that grew with no relation to the work done would prove nothing, so it must also stay far below the
    distance theta travels."""
    T = 10 ** 4
    rng = np.random.default_rng(7)
    G = _gradients(T, 6, rng)
    n = G.shape[1]
    p32 = rng.standard_normal(n).astype(F)
    p32[::5] = 0.0
    m32, v32 = np.zeros(n, F), np.zeros(n, F)
    lr, b1, b2, eps = (float(F(x)) for x in (lr, b1, b2, eps))       # both sides run on the same hyper-parameters
    omb1, omb2 = 1.0 - b1, 1.0 - b2                                   # exact in float32 too (b = 0 or 0.5 <= b <= 1)
    p, m, v = p32.astype(np.float64), np.zeros(n), np.zeros(n)
    Ep, Em, Ev = np.zeros(n), np.zeros(n), np.zeros(n)
    travel = np.abs(p.copy())
    u, eta = 2.0 ** -24, 2.0 ** -150
    with np.errstate(all="ignore"):
        for t in range(1, T + 1):
            g32 = G[t - 1]
            g = g32.astype(np.float64)
            m_prev, v_prev = m32.astype(np.float64), v32.astype(np.float64)
            lr_t = lr * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)
            m = b1 * m + omb1 * g
            v = b2 * v + omb2 * (g * g)
            q = lr_t * m / (np.sqrt(v) + eps)
            p = p - q
            travel += np.abs(q)
            adam_model.step_t(p32, m32, v32, g32, t, lr, b1, b2, eps)
            mh, vh, ph = m32.astype(np.float64), v32.astype(np.float64), p32.astype(np.float64)
            # m: fl(fl(m b1) + fl(omb1 g));  v: fl(fl(v b2) + fl(omb2 fl(g g)))
            Em = b1 * Em + u * (b1 * np.abs(m_prev) + omb1 * np.abs(g) + np.abs(mh)) + 2 * eta
            Ev = b2 * Ev + u * (b2 * v_prev + 2 * omb2 * g * g + vh) + (2 + omb2) * eta
            # den = fl(fl(sqrt v) + eps), num = fl(lr_t32 m), q = fl(num / den)
            sh = np.sqrt(vh)
            Es = u * sh + np.minimum(np.sqrt(Ev), Ev / np.maximum(np.maximum(sh, np.sqrt(v)), 1e-300))
            dh = sh + eps
            Ed = Es + u * dh
            qh = np.abs(lr_t * mh) / dh
            Enum = lr_t * Em + 2 * u * lr_t * np.abs(mh) + eta
            assert np.all(Ed < 0.5 * dh), t
            Eq = (Enum + qh * Ed) / (dh - Ed) + u * qh + eta
            Ep = Ep + Eq + u * np.abs(ph)
            for name, got, ref, bound in (("m", mh, m, Em), ("v", vh, v, Ev), ("theta", ph, p, Ep)):
                bad = np.abs(got - ref) > 2 * bound
                if bad.any():
                    j = int(np.flatnonzero(bad)[0])
                    pytest.fail("%s, step %d, element %d: float32 %r, float64 %r, bound %r"
                                % (name, t, j, got[j], ref[j], 2 * bound[j]))
    assert np.all(2 * Ep <= 1e-2 * travel + 1e-30), (2 * Ep / travel).max()
    assert np.abs(p32 - p).max() > 0                  # the two sides did round differently somewhere
