"""Option "deterministic" (include/c2v_b200.h, DESIGN.md section 5.1): a train step's results depend only on its inputs,
seeds and options.  The sort + chunked reduce is pinned bit for bit to the numpy order model (tests/deterministic_order.py);
whole steps are bit-identical across engines and schedules and stay at the oracle's parity tolerances."""
import glob
import os
import pickle
import re
import zlib

import numpy as np
import pytest

from oracle import path_attention_oracle as O
from tests import deterministic_order as DO
from tests.util import dev_batch, make_engine, rel_err

pytestmark = pytest.mark.gpu

K = DO.K


def _bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


# ---- 1. the order, bit for bit -------------------------------------------------------------------------------------------
ROW_DIMS = {d: O.Dims(token_vocab=60013, path_vocab=40009, target_vocab=64, embed_dim=d, code_dim=64, max_contexts=200)
            for d in (32, 128, 256)}
_row_engines = {}


def _row_engine(d):
    if d not in _row_engines:
        _row_engines[d] = make_engine(ROW_DIMS[d], max_batch=1024, training=False)[0]
    return _row_engines[d]


def _row_case(name, n_rows, d, rng):
    if name == "unique":
        rows = rng.permutation(n_rows)[:30000]
    elif name == "hot":
        n = 600_000
        rows = rng.integers(0, n_rows, n)
        rows[rng.random(n) < 0.6] = 7
    elif name == "zipf":
        rows = np.minimum(rng.zipf(1.2, 200_000) - 1, n_rows - 1)
    elif name == "boundaries":
        lengths = [K - 1, K, K + 1, 2 * K + 1] * 50
        rows = np.concatenate([np.full(n, 11 * i + 3) for i, n in enumerate(lengths)])
        rng.shuffle(rows)
    else:                                           # "signs": negative zeros and cancelling mixed signs
        rows = np.repeat(rng.integers(0, 50, 10000), 2)
    vals = (rng.standard_normal((len(rows), d)) * 10.0 ** rng.uniform(-4, 4, (len(rows), 1))).astype(np.float32)
    if name == "signs":
        vals[rng.random(vals.shape) < 0.3] = -0.0
        vals[1::2] = -vals[0::2][:len(vals[1::2])]
    return rows.astype(np.int32), vals


@pytest.mark.parametrize("d", [32, 128, 256])
@pytest.mark.parametrize("case", ["unique", "hot", "zipf", "boundaries", "signs"])
def test_row_sum_order_matches_the_numpy_model_bit_for_bit(d, case):
    import torch
    eng = _row_engine(d)
    table = 1 if case in ("zipf", "signs") else 0
    n_rows = ROW_DIMS[d].path_vocab if table else ROW_DIMS[d].token_vocab
    rows, vals = _row_case(case, n_rows, d, np.random.default_rng(zlib.crc32(b"%s/%d" % (case.encode(), d))))
    got = eng.selftest_row_sum(table, torch.from_numpy(rows), torch.from_numpy(vals)).cpu().numpy()
    ref = DO.row_sums(rows, vals, n_rows)
    assert np.array_equal(_bits(got), _bits(ref))
    exact = np.zeros((n_rows, d))
    np.add.at(exact, rows, vals.astype(np.float64))
    assert np.all(np.abs(got - exact) <= DO.reorder_bound(rows, vals, n_rows) + 1e-37)
    again = eng.selftest_row_sum(table, torch.from_numpy(rows), torch.from_numpy(vals)).cpu().numpy()
    assert np.array_equal(_bits(again), _bits(got))


# ---- 2. train steps on a duplicate-heavy batch ------------------------------------------------------------------------
DIMS = O.Dims(token_vocab=1001, path_vocab=501, target_vocab=1001, embed_dim=32, code_dim=96, max_contexts=20)
B, KEEP, SEED, STEP = 64, 0.75, 0xD5EED, 3
TOL = {0: 5e-5, 1: 1e-2, 2: 5e-5}


def _dup_batch(seed=5):
    """Indices from a few dozen rows plus row 0 (PAD / OOV), ragged bags."""
    src, pth, tgt, mask, target = O.synthetic_batch(DIMS, B, seed=seed)
    rng = np.random.default_rng(seed)
    hot_tok, hot_path = np.r_[0, rng.choice(np.arange(1, DIMS.token_vocab), 30)], np.r_[0, rng.choice(np.arange(1, 501), 20)]
    for a, hot in ((src, hot_tok), (tgt, hot_tok), (pth, hot_path)):
        a[...] = hot[rng.integers(0, len(hot), a.shape)]
    lengths = rng.integers(1, DIMS.max_contexts + 1, B)
    mask[...] = (np.arange(DIMS.max_contexts)[None, :] < lengths[:, None]).astype(np.float32)
    for a in (src, pth, tgt):
        a[mask == 0] = 0
    target[...] = rng.integers(0, 12, B)
    return src, pth, tgt, mask, target


def _step_grads(math, params, batch, **opts):
    eng, _ = make_engine(DIMS, max_batch=B, params=params)
    eng.set_option("math_mode", math)
    eng.set_option("deterministic", opts.pop("deterministic", 1))
    for k, v in opts.items():
        eng.set_option(k, v)
    loss = float(eng.train_step(*dev_batch(eng, *batch), keep=KEEP, seed=SEED, step=STEP).cpu()[0])
    g = eng.export_grads()
    eng.close()
    return loss, g


@pytest.mark.parametrize("math", [0, 1, 2])
def test_train_step_is_bit_identical_and_matches_the_oracle(math):
    params = O.init_params(DIMS, seed=4321)
    batch = _dup_batch()
    dm = O.dropout_keep_mask(seed=SEED, step=STEP, n_rows=B * DIMS.max_contexts, ctx_dim=DIMS.ctx_dim, keep=KEEP)
    loss_ref, g_ref, _ = O.train_loss_and_grads(params, *batch, keep=KEEP, dropout_mask=dm)
    loss, g = _step_grads(math, params, batch)
    assert abs(loss - loss_ref) < 1e-4
    for k in O.PARAM_NAMES:
        assert rel_err(g[k], g_ref[k]) < TOL[math], k
    variants = [{}, {"dy_late": 0}, {"dy_late": 2}]
    if math == 1:
        variants.append({"fuse_gather": 1})
    for opts in variants:
        loss2, g2 = _step_grads(math, params, batch, **opts)
        assert loss2 == loss, opts
        for k in O.PARAM_NAMES:
            assert np.array_equal(_bits(g2[k]), _bits(g[k])), (opts, k)
    # the atomic scatter sums the same addends in another order: reordering noise only
    _, ga = _step_grads(math, params, batch, deterministic=0)
    for k in ("tok", "path"):
        assert rel_err(g[k], ga[k]) < 1e-5, k
    for k in ("tgt", "W", "a"):
        assert np.array_equal(_bits(ga[k]), _bits(g[k])), k
    assert np.abs(g["tok"][0]).max() > 0                    # row 0 took part (masked contexts did not make it huge)


def _trainer_run(math, params, batches, lazy, hint):
    from code2vec_b200.trainer import Trainer
    eng, _ = make_engine(DIMS, max_batch=B, params=params)
    eng.set_option("math_mode", math)
    tr = Trainer(eng, keep_prob=KEEP, seed=SEED, lazy_adam=lazy, deterministic=True)
    dev = [dev_batch(eng, *b) for b in batches]
    for i, d in enumerate(dev):
        nxt = dev[i + 1][:3] if (hint and i + 1 < len(dev)) else None
        tr.step_device(*d, next_batch=nxt)
    eng.sync_tables()
    out = {}
    for role, tens in (("theta", eng.params), ("m", eng.adam_m), ("v", eng.adam_v)):
        for k in O.PARAM_NAMES:
            out[role + "/" + k] = tens[k].detach().cpu().numpy()
    eng.close()
    return out


@pytest.mark.parametrize("math", [0, 1, 2])
def test_lazy_adam_trainer_matches_dense_bit_for_bit(math):
    params = O.init_params(DIMS, seed=99)
    batches = [_dup_batch(seed=s) for s in (1, 2, 3)]
    lazy = _trainer_run(math, params, batches, lazy=True, hint=False)
    for other in (_trainer_run(math, params, batches, lazy=True, hint=True),
                  _trainer_run(math, params, batches, lazy=False, hint=False)):
        for k in lazy:
            assert np.array_equal(_bits(other[k]), _bits(lazy[k])), k


# ---- 3. sampled softmax ----------------------------------------------------------------------------------------------------
def test_sampled_softmax_is_bit_identical_and_matches_the_oracle():
    import torch
    from code2vec_b200.trainer import Trainer
    params = O.init_params(DIMS, seed=4321)
    src, pth, tgt, mask, target = _dup_batch(seed=9)
    S = 64
    rng = np.random.default_rng(4)
    sampled = O.log_uniform_sample(rng, S, DIMS.target_vocab)
    sampled[:4] = target[:4]                              # sampled classes that are some rows' targets
    sampled[5] = sampled[6]                               # a duplicate sampled class
    lq_t = O.log_uniform_logq(target, S, DIMS.target_vocab)
    lq_s = O.log_uniform_logq(sampled, S, DIMS.target_vocab)
    v_ref, _, _ = O.forward(params, src, pth, tgt, mask)
    loss_ref, _, g_tgt_ref, _ = O.sampled_softmax_loss_and_grads(params, v_ref, target, sampled, lq_t, lq_s)
    eng, _ = make_engine(DIMS, max_batch=B, params=params)
    eng.set_option("deterministic", 1)
    d = dev_batch(eng, src, pth, tgt, mask, target)
    extra = (eng.to_device(sampled, torch.int32), eng.to_device(lq_t, torch.float32), eng.to_device(lq_s, torch.float32))
    loss = float(eng.sampled_train_step(*d, *extra).cpu()[0])
    g1 = eng.export_grads()
    assert abs(loss - loss_ref) < 1e-4
    assert rel_err(g1["tgt"], g_tgt_ref) < 5e-5
    eng.sampled_train_step(*d, *extra)
    g2 = eng.export_grads()
    for k in O.PARAM_NAMES:
        assert np.array_equal(_bits(g2[k]), _bits(g1[k])), k
    eng.close()
    # the lazy target-row path (Trainer, lazy Adam): two fresh runs of 3 steps agree bit for bit
    runs = []
    for _ in range(2):
        eng, _ = make_engine(DIMS, max_batch=B, params=params)
        tr = Trainer(eng, keep_prob=KEEP, seed=SEED, deterministic=True)
        d = dev_batch(eng, src, pth, tgt, mask, target)
        extra = (eng.to_device(sampled, torch.int32), eng.to_device(lq_t, torch.float32), eng.to_device(lq_s, torch.float32))
        for _ in range(3):
            tr.step_device_sampled(*d, *extra)
        runs.append(eng.export_params())
        eng.close()
    for k in O.PARAM_NAMES:
        assert np.array_equal(_bits(runs[0][k]), _bits(runs[1][k])), k


# ---- 4. real size ----------------------------------------------------------------------------------------------------------
JAVA14M = O.Dims(token_vocab=1301137, path_vocab=911418, target_vocab=261246, embed_dim=128, code_dim=384, max_contexts=200)


def _java14m_run(zipf):
    import torch
    from code2vec_b200.engine import EngineDims, PathAttentionEngine
    from code2vec_b200.trainer import Trainer
    Bj, C = 256, JAVA14M.max_contexts
    eng = PathAttentionEngine(EngineDims(JAVA14M.token_vocab, JAVA14M.path_vocab, JAVA14M.target_vocab, 128, 384, C, Bj))
    eng.init_params(seed=11)
    eng.set_option("math_mode", 1)
    tr = Trainer(eng, keep_prob=KEEP, seed=SEED, deterministic=True)
    rng = np.random.default_rng(3)
    for _ in range(3):
        def idx(n):
            return (np.minimum(rng.zipf(1.3, (Bj, C)) - 1, n - 1) if zipf else rng.integers(0, n, (Bj, C))).astype(np.int32)
        lengths = rng.integers(1, C + 1, Bj)
        mask = (np.arange(C)[None, :] < lengths[:, None]).astype(np.float32)
        batch = (idx(JAVA14M.token_vocab), idx(JAVA14M.path_vocab), idx(JAVA14M.token_vocab), mask,
                 rng.integers(0, JAVA14M.target_vocab, Bj).astype(np.int32))
        tr.step_device(*dev_batch(eng, *batch))
    eng.sync_tables()
    h = {role: [t.reshape(-1).view(torch.int32).sum().item() for t in tens.values()]      # checksums of the bits
         for role, tens in (("theta", eng.params), ("m", eng.adam_m), ("v", eng.adam_v))}
    sample = {k: eng.params[k][:4096].cpu().numpy() for k in ("tok", "path")}
    eng.close()
    return h, sample


@pytest.mark.parametrize("zipf", [False, True])
def test_java14m_runs_are_bit_identical(zipf):
    h1, s1 = _java14m_run(zipf)
    h2, s2 = _java14m_run(zipf)
    assert h1 == h2
    for k in s1:
        assert np.array_equal(_bits(s1[k]), _bits(s2[k])), k


# ---- 5. end to end through Code2VecModel ----------------------------------------------------------------------------------
C = 8
TOKENS = ["tok%d" % i for i in range(40)]
PATHS = [str(1000 + 7 * i) for i in range(25)]
TARGETS = ["get|name", "set|name", "run", "to|string", "main", "close", "is|empty", "add|item"]


def _make_dataset(tmp_path, n_train=96, seed=0):
    """The toy dataset of tests/test_gpu_model.py: the target follows from the group of the source tokens."""
    rng = np.random.default_rng(seed)
    prefix = str(tmp_path / "ds")

    def example():
        t = int(rng.integers(0, len(TARGETS)))
        n = int(rng.integers(2, C + 1))
        ctxs = []
        for i in range(n):
            s = TOKENS[t * 4 + int(rng.integers(0, 4))]
            ctxs.append("%s,%s,%s" % (s, PATHS[int(rng.integers(0, 25))], TOKENS[32 + int(rng.integers(0, 8))]))
        return " ".join([TARGETS[t]] + ctxs + [""] * (C - n))

    train = [example() for _ in range(n_train)]
    with open(prefix + ".train.c2v", "w") as f:
        f.write("\n".join(train) + "\n")
    tok, pth, tgt = {}, {}, {}
    for line in train:
        parts = line.split(" ")
        tgt[parts[0]] = tgt.get(parts[0], 0) + 1
        for c in parts[1:]:
            if c:
                s, p, t = c.split(",")
                tok[s] = tok.get(s, 0) + 1
                tok[t] = tok.get(t, 0) + 1
                pth[p] = pth.get(p, 0) + 1
    with open(prefix + ".dict.c2v", "wb") as f:
        for d in (tok, pth, tgt):
            pickle.dump(d, f)
        pickle.dump(n_train, f)
    return prefix


def _train_once(tmp_path, framework, run, seed, monkeypatch):
    from code2vec_b200.config import Config
    if framework == "b200":
        from code2vec_b200.b200_model import Code2VecModel
    else:
        from code2vec_b200.b200_keras_model import Code2VecModel
    monkeypatch.setenv("C2V_DETERMINISTIC", "1")
    monkeypatch.setenv("C2V_SEED", str(seed))
    prefix = _make_dataset(tmp_path)
    out = tmp_path / ("%s_%s" % (framework, run))
    cfg = Config(set_defaults=True)
    cfg.VERBOSE_MODE = 0
    cfg.DL_FRAMEWORK = framework
    cfg.MAX_CONTEXTS = C
    cfg.DEFAULT_EMBEDDINGS_SIZE = cfg.TOKEN_EMBEDDINGS_SIZE = cfg.PATH_EMBEDDINGS_SIZE = 16
    cfg.CODE_VECTOR_SIZE = cfg.TARGET_EMBEDDINGS_SIZE = 48
    cfg.TRAIN_BATCH_SIZE = cfg.TEST_BATCH_SIZE = 32
    cfg.NUM_TRAIN_EPOCHS = 6
    cfg.SAVE_EVERY_EPOCHS = 3 if framework == "b200-keras" else 1000      # the Keras schedule only saves at epoch marks
    cfg.NUM_BATCHES_TO_LOG_PROGRESS = 3
    cfg.SHUFFLE_BUFFER_SIZE = 64
    cfg.DROPOUT_KEEP_RATE = 0.75
    cfg.TOP_K_WORDS_CONSIDERED_DURING_PREDICTION = 5
    cfg.TRAIN_DATA_PATH_PREFIX = prefix
    cfg.MODEL_SAVE_PATH = str(out / "saved")
    model = Code2VecModel(cfg)
    lines = []
    model.log = lines.append
    model.train()
    model.close_session()
    losses = [float(x) for line in lines for x in re.findall(r"(?:loss at batch \d+: |'loss': )([-0-9.e]+)", line)]
    blobs = {os.path.basename(p): open(p, "rb").read() for p in sorted(glob.glob(str(out / "*.c2v_b200")))}
    return losses, blobs


@pytest.mark.parametrize("framework", ["b200", "b200-keras"])
def test_end_to_end_runs_replay_bit_for_bit(tmp_path, monkeypatch, framework):
    monkeypatch.chdir(tmp_path)
    l1, c1 = _train_once(tmp_path, framework, "a", 7, monkeypatch)
    l2, c2 = _train_once(tmp_path, framework, "b", 7, monkeypatch)
    assert c1 and l1
    assert l1 == l2
    assert c1.keys() == c2.keys() and all(c1[k] == c2[k] for k in c1)
    _, c3 = _train_once(tmp_path, framework, "c", 8, monkeypatch)
    assert any(c3[k] != c1[k] for k in c1)


# ---- 6. the option itself ----------------------------------------------------------------------------------------------------
def test_option_round_trip_and_refusals():
    import ctypes
    from code2vec_b200.engine import EngineError, c2v_table_shards
    eng, _ = make_engine(DIMS, max_batch=B)
    assert eng.get_option("deterministic") == 0
    eng.set_option("deterministic", 1)
    assert eng.get_option("deterministic") == 1
    with pytest.raises(EngineError) as ei:
        eng.set_option("deterministic", 2)
    assert ei.value.code == -1

    def shards(world):
        st = c2v_table_shards()
        st.world, st.rank = world, 0
        for r in range(world):
            st.tok[r], st.path[r] = eng.params["tok"].data_ptr(), eng.params["path"].data_ptr()
        return st

    sp = shards(2)
    rc = eng.lib.c2v_bind_table_shards(eng.h, ctypes.byref(sp), ctypes.byref(sp), 0.5)      # refused: nothing is bound
    assert rc == -4 and b"deterministic" in eng.lib.c2v_last_error(eng.h)
    one = shards(1)
    assert eng.lib.c2v_bind_table_shards(eng.h, ctypes.byref(one), ctypes.byref(one), 1.0) == 0     # world 1 is local
    eng.set_option("deterministic", 0)
    assert eng.lib.c2v_bind_table_shards(eng.h, ctypes.byref(sp), ctypes.byref(sp), 0.5) == 0
    with pytest.raises(EngineError) as ei:
        eng.set_option("deterministic", 1)
    assert ei.value.code == -4 and "row-sharded" in str(ei.value)
    eng.close()
