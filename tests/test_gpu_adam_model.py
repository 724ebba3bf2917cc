"""Every Adam path of the engine against the float32 statement of the step (tests/adam_model.py), bit for bit.

(B) adam_kernel itself, through c2v_adam_step_range on caller-filled (theta, g, m, v): lengths around the float4
    vectorisation and past one grid-stride wave, slices inside sentinel-filled buffers, zero_grad 0 / 1, step counts
    up to 10^6, default and unusual hyper-parameters (b1 = 0, b2 = 0.9999, eps = 1e-3, eps = 0) and special values
    (signed zeros, subnormals, g^2 underflowing and overflowing, infinities, NaN, v = 0).
(C) The engine's own paths after real train steps: before each adam_step the step's gradients are read with
    export_grads and fed to the model, so the scatter's atomic order does not matter; after the flush every element
    of the five tensors and of their m and v must equal the model.  A lazily updated row's gradient for step s is its
    exported row if batch s references it (mask > 0), zero otherwise -- an unreferenced gradient row may still hold
    an earlier step's deferred gradient.  NaN is compared as NaN (the GPU's canonical NaN is not x86's)."""
import time

import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests import adam_model as AM
from tests.util import dev_batch, make_engine

pytestmark = pytest.mark.gpu

F = np.float32
DEFAULT = (1e-3, 0.9, 0.999, 1e-8)
HPS = [DEFAULT, (3e-2, 0.0, 0.9999, 1e-3), (1e-3, 0.9, 0.999, 0.0)]
TS = [1, 2, 10, 1000, 65535, 65536, 10 ** 6]
SENTINEL = np.uint32(0xA5A5A5A5)


def _assert_same(got, want, what):
    got, want = np.asarray(got, F).ravel(), np.asarray(want, F).ravel()
    ok = AM.same_bits(got, want)
    if not ok.all():
        j = int(np.flatnonzero(~ok)[0])
        pytest.fail("%s: %d of %d elements differ; first at %d: got %r (0x%08x), model %r (0x%08x)"
                    % (what, int((~ok).sum()), ok.size, j, got[j], got[j:j + 1].view(np.uint32)[0], want[j],
                       want[j:j + 1].view(np.uint32)[0]))


# ---------------------------------------------------------------------------------------------------------------------
# (B) adam_kernel through c2v_adam_step_range
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def tiny_engine():
    dims = O.Dims(token_vocab=16, path_vocab=16, target_vocab=16, embed_dim=4, code_dim=4, max_contexts=2)
    eng, _ = make_engine(dims, max_batch=2)
    return eng


def _operands(n, rng):
    """theta, g, m, v with ordinary values and, in about a third of the places, special ones."""
    def pick(ordinary, specials):
        x = ordinary.astype(F)
        sel = rng.random(n) < 0.35
        x[sel] = rng.choice(np.array(specials, dtype=F), size=int(sel.sum()))
        return x
    sub = [1e-40, -1e-40, 1.4e-45, -3e-39]
    theta = pick(rng.standard_normal(n), [0.0, -0.0, np.inf, -np.inf, np.nan, 3e38] + sub)
    g = pick(rng.standard_normal(n) * 10.0 ** rng.integers(-6, 7, n),
             [0.0, -0.0, 1e-25, -3e-23, 2e19, -3e19, 1.9e19, np.inf, -np.inf, np.nan] + sub)      # 1e-25^2 underflows, 2e19^2 overflows
    m = pick(rng.standard_normal(n) * 1e-2, [0.0, -0.0, np.inf, -np.inf, np.nan, 1e30] + sub)
    v = pick(rng.random(n) * 1e-3, [0.0, 0.0, np.inf, np.nan, 1e38, 1e-40, 1.4e-45])
    return theta, g, m, v


def _kernel_case(eng, count, t, hp, zero_grad, rng, pad=4):
    """One c2v_adam_step_range call on a slice [pad, pad + count) of four sentinel-filled buffers."""
    import torch
    lr, b1, b2, eps = hp
    host = _operands(count, rng)
    bufs = []
    for x in host:
        full = np.full(count + 2 * pad, SENTINEL, dtype=np.uint32).view(F)
        full[pad:pad + count] = x
        bufs.append(torch.from_numpy(full).to(eng.dev))
    th, g, m, v = (b[pad:pad + count] for b in bufs)
    eng.adam_step_range(th, g, m, v, t, lr=lr, beta1=b1, beta2=b2, eps=eps, zero_grad=zero_grad)
    got = [b.cpu().numpy() for b in bufs]
    p_ref, g_ref, m_ref, v_ref = (x.copy() for x in host)
    AM.step(p_ref, m_ref, v_ref, g_ref, O.adam_lr_t(t, lr, b1, b2), b1, b2, eps)
    what = "count %d, t %d, hp %s, zero_grad %d" % (count, t, hp, zero_grad)
    for name, full in zip("theta g m v".split(), got):
        assert np.all(full[:pad].view(np.uint32) == SENTINEL) and np.all(full[pad + count:].view(np.uint32) == SENTINEL), \
            "%s: %s written outside the slice" % (what, name)
    _assert_same(got[0][pad:pad + count], p_ref, what + ", theta")
    _assert_same(got[2][pad:pad + count], m_ref, what + ", m")
    _assert_same(got[3][pad:pad + count], v_ref, what + ", v")
    g_want = np.zeros(count, F) if zero_grad else host[1]
    assert np.array_equal(got[1][pad:pad + count].view(np.uint32), g_want.view(np.uint32)), what + ", g"


@pytest.mark.parametrize("zero_grad", [0, 1])
@pytest.mark.parametrize("count", [4, 8, 1020, 4 * 12345 + 4, "past_one_wave"])
def test_adam_kernel_is_the_float32_step(tiny_engine, count, zero_grad):
    import torch
    eng = tiny_engine
    if count == "past_one_wave":        # the grid is capped at num_sms * 16 blocks of 256 float4s: loop around it
        count = torch.cuda.get_device_properties(eng.dev).multi_processor_count * 16 * 256 * 4 + 4 * 257
    rng = np.random.default_rng(count + zero_grad)
    for hp in HPS:
        for t in TS:
            _kernel_case(eng, count, t, hp, zero_grad, rng)


def test_adam_step_range_refusals(tiny_engine):
    import torch
    from code2vec_b200.engine import EngineError
    eng = tiny_engine
    x = [torch.ones(64, dtype=torch.float32, device=eng.dev) for _ in range(4)]
    before = [a.clone() for a in x]
    with pytest.raises(EngineError):
        eng.adam_step_range(*(a[:6] for a in x), t=1)                         # not a multiple of 4 floats
    for i in range(4):                                                        # each pointer off 16-byte alignment in turn
        with pytest.raises(EngineError):
            eng.adam_step_range(*((a[1:9] if j == i else a[:8]) for j, a in enumerate(x)), t=1)
    for t in (0, -1):
        with pytest.raises(EngineError):
            eng.adam_step_range(*(a[:8] for a in x), t=t)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(x, before))                  # nothing was launched


# ---------------------------------------------------------------------------------------------------------------------
# (C) the engine's paths after train steps
# ---------------------------------------------------------------------------------------------------------------------

DIMS = O.Dims(token_vocab=2001, path_vocab=1003, target_vocab=301, embed_dim=20, code_dim=52, max_contexts=10)
B = 8
FAST_B1 = (1e-3, 0.5, 0.995, 1e-8)           # m halves every idle step: replayed rows reach the "theta rests" exit
SLOW_BIAS = (1e-3, 0.9999, 0.99999, 1e-8)    # lr_t still changes by ~90 ulps per step around t = 65536


class Model:
    """The five tensors and their slots in one flat float32 buffer each (one numpy pass per step)."""

    def __init__(self, params0):
        self.shapes = [(k, params0[k].shape) for k in O.PARAM_NAMES]
        self.p = np.concatenate([params0[k].ravel() for k in O.PARAM_NAMES]).astype(F)
        self.m, self.v = np.zeros_like(self.p), np.zeros_like(self.p)

    def flat(self, d):
        return np.concatenate([np.asarray(d[k], F).ravel() for k in O.PARAM_NAMES])

    def step(self, grads, t, hp):
        lr, b1, b2, eps = hp
        AM.step(self.p, self.m, self.v, self.flat(grads), O.adam_lr_t(t, lr, b1, b2), b1, b2, eps)

    def assert_engine(self, eng, what):
        got = eng.export_params()                        # replays every deferred update first
        slots = [{k: s[k].cpu().numpy() for k in O.PARAM_NAMES} for s in (eng.adam_m, eng.adam_v)]
        for name, mine, theirs in (("theta", self.p, self.flat(got)), ("m", self.m, self.flat(slots[0])),
                                   ("v", self.v, self.flat(slots[1]))):
            off = 0
            for k, shp in self.shapes:
                n = int(np.prod(shp))
                _assert_same(theirs[off:off + n], mine[off:off + n], "%s: %s %s" % (what, name, k))
                off += n


def _referenced(n_rows, *index_arrays):
    hit = np.zeros(n_rows, dtype=bool)
    for a in index_arrays:
        hit[a] = True
    return hit[:, None]


def _step_grads(eng, batch, sampled=None):
    """The gradients adam_step is about to apply, as the model must see them."""
    g = eng.export_grads()
    if eng.get_option("lazy_adam"):
        src, pth, tgt, mask = batch[:4]
        live = mask > 0
        g["tok"] = np.where(_referenced(DIMS.token_vocab, src[live], tgt[live]), g["tok"], F(0))
        g["path"] = np.where(_referenced(DIMS.path_vocab, pth[live]), g["path"], F(0))
        if sampled is not None:                          # the target table is lazily updated on sampled steps
            g["tgt"] = np.where(_referenced(DIMS.target_vocab, batch[4], sampled), g["tgt"], F(0))
    return g


def _train(eng, model, steps, hp=DEFAULT, keep=0.75, seed0=0, zipf=True, t0=1, between=None):
    for i in range(steps):
        t = t0 + i
        batch = O.synthetic_batch(DIMS, B, seed=seed0 + i, zipf=zipf)
        h = hp(t) if callable(hp) else hp
        eng.train_step(*dev_batch(eng, *batch), keep=keep, seed=11, step=t)
        g = _step_grads(eng, batch)
        eng.adam_step(*h, t=t)
        model.step(g, t, h)
        if between:
            between(t)


@pytest.mark.parametrize("math_mode", [0, 1, 2])
def test_dense_adam_is_the_model(math_mode):
    eng, params0 = make_engine(DIMS, max_batch=B)
    eng.set_option("math_mode", math_mode)
    model = Model(params0)
    _train(eng, model, 5, zipf=False)
    model.assert_engine(eng, "dense, math_mode %d" % math_mode)


@pytest.mark.parametrize("rest", [0, 1])
@pytest.mark.parametrize("period", [0, 1, 3, 32])
def test_lazy_adam_is_the_model(period, rest):
    """40 Zipfian batches: most rows are referenced rarely, so replays span many steps; with b1 = 0.5 idle rows come to
    rest within ~20 steps, so the rest exit of replay_row is taken wherever it is enabled."""
    eng, params0 = make_engine(DIMS, max_batch=B)
    eng.set_option("lazy_adam", 1)
    eng.set_option("adam_sweep_period", period)
    eng.set_option("adam_rest_shortcut", rest)
    model = Model(params0)
    _train(eng, model, 40, hp=FAST_B1 if rest else DEFAULT)
    model.assert_engine(eng, "lazy, period %d, rest %d" % (period, rest))


def test_trainer_single_fused_target_adam_and_early_catchup_are_the_model():
    """Trainer("single"): lazy Adam, the target table's Adam in the dY epilogue and the next-batch hint, whose early
    catch-up replays the next batch's rows inside the train step (and clears their gradient rows there).  So the
    step's gradients come from a twin engine without any of that: the fused target update never writes dY, and the
    option "deterministic" on both makes the twin's embedding gradients the trainer's own bits."""
    from code2vec_b200.trainer import Trainer
    steps = 6
    fast, params0 = make_engine(DIMS, max_batch=B)
    twin, _ = make_engine(DIMS, max_batch=B, params=params0)
    for eng in (fast, twin):
        eng.set_option("math_mode", 1)
    twin.set_option("deterministic", 1)
    tr = Trainer(fast, keep_prob=0.75, seed=3, deterministic=True)
    assert tr.schedule == "single" and tr.fuse_tgt and fast.get_option("lazy_adam") == 1
    batches = [O.synthetic_batch(DIMS, B, seed=40 + s, zipf=True) for s in range(steps)]
    model = Model(params0)
    for s, batch in enumerate(batches):
        t = s + 1
        nxt = dev_batch(fast, *batches[s + 1][:4])[:3] if s + 1 < steps else None
        tr.step_device(*dev_batch(fast, *batch), next_batch=nxt)
        twin.train_step(*dev_batch(twin, *batch), keep=0.75, seed=3, step=t)
        g = _step_grads(twin, batch)
        twin.adam_step(*DEFAULT, t=t)
        model.step(g, t, DEFAULT)
    assert fast.get_option("early_catchup_count") == steps - 2
    model.assert_engine(twin, "twin")
    model.assert_engine(fast, "Trainer(single)")


def test_sampled_softmax_lazy_target_rows_then_full_softmax_are_the_model():
    import torch
    S = 7
    eng, params0 = make_engine(DIMS, max_batch=B)
    eng.set_option("lazy_adam", 1)
    eng.set_option("adam_sweep_period", 4)
    model = Model(params0)
    rng = np.random.default_rng(9)
    for s in range(6):
        t = s + 1
        batch = O.synthetic_batch(DIMS, B, seed=700 + s)
        d = dev_batch(eng, *batch)
        sampled = None
        if s < 5:
            sampled = O.log_uniform_sample(rng, S, DIMS.target_vocab)
            lq_t, lq_s = O.log_uniform_logq(batch[4], S, DIMS.target_vocab), O.log_uniform_logq(sampled, S, DIMS.target_vocab)
            eng.sampled_train_step(*d, eng.to_device(sampled, torch.int32), eng.to_device(lq_t, torch.float32),
                                   eng.to_device(lq_s, torch.float32))
        else:
            eng.train_step(*d, keep=1.0)
        g = _step_grads(eng, batch, sampled)
        eng.adam_step(*DEFAULT, t=t)
        model.step(g, t, DEFAULT)
    model.assert_engine(eng, "sampled softmax")


def test_hyper_parameter_change_flushes_with_the_old_values():
    eng, params0 = make_engine(DIMS, max_batch=B)
    eng.set_option("lazy_adam", 1)
    model = Model(params0)
    _train(eng, model, 8, hp=lambda t: DEFAULT if t <= 4 else (2e-3, 0.8, 0.99, 1e-7))
    model.assert_engine(eng, "hyper-parameter change")


def test_lazy_adam_off_and_on_again():
    eng, params0 = make_engine(DIMS, max_batch=B)
    eng.set_option("lazy_adam", 1)
    model = Model(params0)
    switch = {3: 0, 5: 1}
    _train(eng, model, 8, between=lambda t: eng.set_option("lazy_adam", switch[t]) if t in switch else None)
    assert eng.get_option("lazy_adam") == 1
    model.assert_engine(eng, "lazy off and on")


def test_restored_step_count():
    eng, params0 = make_engine(DIMS, max_batch=B)
    eng.set_option("lazy_adam", 1)
    model = Model(params0)
    _train(eng, model, 3)
    eng.set_option("adam_step_count", 50)
    _train(eng, model, 5, seed0=3, t0=51)
    model.assert_engine(eng, "restored step count")


def test_learning_rate_ring_wraps():
    """The lazy replay reads each pending step's lr_t from a ring of 65536 entries: restore the step count to 65530 and
    run 26 steps across the wrap, rows replayed over it.  The hyper-parameters keep lr_t changing from step to step
    there, so an entry read for the wrong step shows."""
    eng, params0 = make_engine(DIMS, max_batch=B)
    eng.set_option("lazy_adam", 1)
    eng.set_option("adam_sweep_period", 0)
    eng.set_option("adam_step_count", 65530)
    assert O.adam_lr_t(65535, *SLOW_BIAS[:3]) != O.adam_lr_t(65536, *SLOW_BIAS[:3])
    model = Model(params0)
    _train(eng, model, 26, hp=SLOW_BIAS, t0=65531)
    model.assert_engine(eng, "ring wrap")


def test_forced_flush_before_a_row_falls_a_ring_behind():
    """Sweep off and rows left idle from step 1 to step 65541: the engine must bring every row up to date before the
    ring entry of its first pending step is overwritten.  Tiny dims and adam_step calls without train steps; the
    target table, W and a keep applying the gradient of the one train step."""
    dims = O.Dims(token_vocab=13, path_vocab=11, target_vocab=9, embed_dim=4, code_dim=8, max_contexts=3)
    eng, params0 = make_engine(dims, max_batch=2)
    eng.set_option("lazy_adam", 1)
    eng.set_option("adam_sweep_period", 0)
    model = Model(params0)
    batch = O.synthetic_batch(dims, 2, seed=5)
    eng.train_step(*dev_batch(eng, *batch), keep=1.0)
    g = eng.export_grads()
    src, pth, tgt, mask = batch[:4]
    live = mask > 0
    g["tok"] = np.where(_referenced(dims.token_vocab, src[live], tgt[live]), g["tok"], F(0))
    g["path"] = np.where(_referenced(dims.path_vocab, pth[live]), g["path"], F(0))
    later = dict(g, tok=np.zeros_like(g["tok"]), path=np.zeros_like(g["path"]))
    t0 = time.perf_counter()
    T = 65541
    for t in range(1, T + 1):
        eng.adam_step(*DEFAULT, t=t)
        model.step(g if t == 1 else later, t, DEFAULT)
    model.assert_engine(eng, "forced flush")
    print("forced flush: %d adam steps in %.1f s" % (T, time.perf_counter() - t0))


def test_eps_zero_lazy_equals_dense_equals_model():
    """eps = 0: an element with m = v = 0 divides 0 / 0.  The dense kernel writes NaN there; the lazy replay must
    too, not keep theta by its zero-numerator exit."""
    engines = {}
    for lazy in (0, 1):
        eng, params0 = make_engine(DIMS, max_batch=B)
        eng.set_option("deterministic", 1)
        eng.set_option("lazy_adam", lazy)
        engines[lazy] = eng
    hp = (1e-3, 0.9, 0.999, 0.0)
    batch = O.synthetic_batch(DIMS, B, seed=77)
    thetas = []
    for lazy, eng in engines.items():
        model = Model(params0)
        eng.train_step(*dev_batch(eng, *batch), keep=0.75, seed=1, step=1)
        g = _step_grads(eng, batch)
        for t in (1, 2, 3):             # steps 2 and 3 without a train step: only the dense tensors keep a gradient
            eng.adam_step(*hp, t=t)
            model.step(g, t, hp)
            g = dict(g, tok=np.zeros_like(g["tok"]), path=np.zeros_like(g["path"]))
        model.assert_engine(eng, "eps = 0, lazy %d" % lazy)
        assert np.isnan(model.p).any() and not np.isnan(model.p).all()
        thetas.append(model.flat(eng.export_params()))
    _assert_same(thetas[1], thetas[0], "eps = 0: lazy against dense")
