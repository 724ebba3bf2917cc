"""The deferred-update scheme of `lazy_adam` (DESIGN.md section 4.4) as a numpy model, against the dense TF1 Adam of
the oracle (SURVEY A.3), in float32 with the same operation order as adam_kernel / replay_row (tests/adam_model.py).
This pins the ALGORITHM on the CPU (tests/test_gpu_adam_model.py pins the CUDA kernels to the same float32 step):
  * a row that is only brought up to date when a batch references it again, when the periodic sweep reaches it or at
    a flush -- one step with the gradient that was left in its gradient row, then zero-gradient steps -- ends with
    the same bits as a row updated densely;
  * the "theta rests" exit of the replay is exact: once a zero-gradient step changes no element of the row, no later
    one does, so only m and v keep decaying (no division, no square root);
  * with a sweep of period R no row is ever more than R steps behind.
"""
import numpy as np

from oracle.path_attention_oracle import adam_lr_t
from tests import adam_model

F = np.float32


def lr_at(t, lr=1e-3, b1=0.9, b2=0.999):
    return adam_lr_t(t, lr, b1, b2)


def dense_step(p, m, v, g, t, b1, b2, eps, lr=1e-3):
    """adam_kernel: every element, every step (correctly rounded fp32 operations in this order)."""
    adam_model.step(p, m, v, g, lr_at(t, lr, b1, b2), b1, b2, eps)


class LazyTable:
    """Rows + slots + the bookkeeping of the engine: `last[r]` = step the row is current for, `g[r]` = the
    scatter-add of the step that last touched it (zeros otherwise).  `rest`: replay_row's exit; `sweep`: period R."""

    def __init__(self, p, b1, b2, eps, lr=1e-3, rest=False, sweep=0):
        self.p, self.m, self.v = p.copy(), np.zeros_like(p), np.zeros_like(p)
        self.g = np.zeros_like(p)
        self.last = np.zeros(p.shape[0], dtype=np.int64)
        self.t_done, self.hp, self.lr, self.rest, self.sweep = 0, (b1, b2, eps), lr, rest, sweep
        self.expensive_steps = 0
        self.max_lag = 0

    def catch_up(self, rows):
        b1, b2, eps = self.hp
        for r in rows:
            if self.last[r] >= self.t_done:
                continue
            self.max_lag = max(self.max_lag, self.t_done - self.last[r])
            p, m, v = self.p[r:r + 1], self.m[r:r + 1], self.v[r:r + 1]
            s = self.last[r] + 1
            dense_step(p, m, v, self.g[r:r + 1], s, b1, b2, eps, self.lr)               # the deferred gradient step
            self.expensive_steps += 1
            self.g[r] = 0
            zero = np.zeros_like(p)
            s += 1
            while s <= self.t_done:
                before = p.copy()
                dense_step(p, m, v, zero, s, b1, b2, eps, self.lr)
                self.expensive_steps += 1
                s += 1
                if self.rest and np.array_equal(before.view(np.uint32), p.view(np.uint32)):   # no element moved: theta rests
                    break
            while s <= self.t_done:                                                     # only the slots still decay
                m[:] = m * F(b1) + (F(1) - F(b1)) * zero
                v[:] = v * F(b2) + (F(1) - F(b2)) * zero
                s += 1
            self.last[r] = self.t_done

    def train_step(self, rows, grads):
        self.catch_up(rows)                       # before the forward pass reads the rows
        np.add.at(self.g, rows, grads)            # backward: scatter-add
        self.t_done += 1                          # c2v_adam_step records the step ...
        if self.sweep:                            # ... and sweeps a 1/R slice of the table
            n, ph = self.p.shape[0], self.t_done % self.sweep
            self.catch_up(range(n * ph // self.sweep, n * (ph + 1) // self.sweep))

    def flush(self):
        self.catch_up(range(self.p.shape[0]))


def _run(n_rows, d, steps, touch_prob, hp, seed, lr=1e-3, scale=1.0, **kw):
    rng = np.random.default_rng(seed)
    p0 = (rng.standard_normal((n_rows, d)) * scale).astype(F)
    dense_p, dense_m, dense_v = p0.copy(), np.zeros_like(p0), np.zeros_like(p0)
    lazy = LazyTable(p0, *hp, lr=lr, **kw)
    for t in range(1, steps + 1):
        rows = np.flatnonzero(rng.random(n_rows) < touch_prob)
        grads = (rng.standard_normal((rows.size, d)) * 1e-2).astype(F)
        lazy.train_step(rows, grads)
        g = np.zeros_like(p0)
        g[rows] = grads
        dense_step(dense_p, dense_m, dense_v, g, t, *hp, lr=lr)
    lazy.flush()
    return lazy, dense_p, dense_m, dense_v


def _same_bits(lazy, p, m, v):
    for a, b in ((lazy.p, p), (lazy.m, m), (lazy.v, v)):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))     # bit for bit, signs of zeros included


def test_deferred_updates_are_bit_identical_to_dense_adam():
    lazy, p, m, v = _run(n_rows=40, d=8, steps=60, touch_prob=0.25, hp=(0.9, 0.999, 1e-8), seed=0)
    _same_bits(lazy, p, m, v)
    assert not lazy.g.any()                       # every gradient row was consumed and cleared


def test_sweep_bounds_the_lag_and_changes_nothing():
    lazy, p, m, v = _run(n_rows=64, d=4, steps=200, touch_prob=0.02, hp=(0.9, 0.999, 1e-8), seed=1, sweep=8)
    _same_bits(lazy, p, m, v)
    assert lazy.max_lag <= 8
    free, *_ = _run(n_rows=64, d=4, steps=200, touch_prob=0.02, hp=(0.9, 0.999, 1e-8), seed=1)
    assert free.max_lag > 50                      # without the sweep rows fall far behind


def test_theta_rests_exit_is_exact_and_bounds_the_work():
    """TF1's defaults and the edges of the range the engine enables the exit for (0 < b1 <= 0.95, 0.99 <= b2 < 1),
    parameters of ordinary size, tiny ones (where a vanishing update still moves them) and exact zeros."""
    with np.errstate(under="ignore"):
        for hp, lr, scale, seed in (((0.9, 0.999, 1e-8), 1e-3, 1.0, 3), ((0.95, 0.99, 1e-8), 1e-3, 1.0, 4),
                                    ((0.9, 0.999, 1e-7), 1e-2, 1e-3, 5), ((0.5, 0.995, 1e-8), 1e-3, 1e-30, 6),
                                    ((0.9, 0.999, 1e-8), 1e-3, 0.0, 7)):
            plain, p, m, v = _run(n_rows=10, d=4, steps=1500, touch_prob=0.004, hp=hp, seed=seed, lr=lr, scale=scale)
            quick, *_ = _run(n_rows=10, d=4, steps=1500, touch_prob=0.004, hp=hp, seed=seed, lr=lr, scale=scale, rest=True)
            _same_bits(plain, p, m, v)
            _same_bits(quick, p, m, v)
            if scale >= 1e-3 and hp[0] <= 0.9:    # ordinary parameters, TF1's betas: they rest after ~150 idle steps
                assert quick.expensive_steps < 0.5 * plain.expensive_steps, (hp, quick.expensive_steps, plain.expensive_steps)


def test_rest_exit_with_the_sweep_on_a_busy_table():
    lazy, p, m, v = _run(n_rows=48, d=4, steps=400, touch_prob=0.05, hp=(0.9, 0.999, 1e-8), seed=9, rest=True, sweep=16)
    _same_bits(lazy, p, m, v)
