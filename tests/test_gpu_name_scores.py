"""c2v_name_scores (csrc/name_rank.cuh, DESIGN.md §6n) on the H100: against the float64 statement of
tests/name_scores_model.py in fp32, tf32 and 3xTF32; bit for bit against c2v_topk on the same slab; against c2v_loss; and
`--score_names` end to end on a small trained model, for both frameworks.

Error bound (derived before any run, not fitted).  Let u = 2^-24 and vb = tests/similarity_model.value_bound(mode, D) =
2 eps_mode + (2 D + 5) u, the relative error of one float32 dot product on the mode's operands.  The stored logit S_b[j]
then lies within delta_j = vb |v_b| |Y_j| of its float64 value (v_b, Y_j the float32 inputs), and:
  * t_b moves by at most delta_y, m_b by at most dmax = max_j delta_j, and lse_b, whose gradient is the softmax (weights
    summing to 1), by at most dmax.  So the data error of logp is delta_y + dmax, that of top1_logp = m - lse 2 dmax.
  * The kernel's own rounding.  sum_j exp(S_j - m) is a sum of positive terms; each term's relative error is the sum of
    the errors of the operations on its path: its exp (2 ulp = 4 u) and the rounding of its argument x - m (u |x - m|),
    at most 3 adds inside its float4 and 1 into the thread's sum, then per later float4 of the thread (n_t =
    ceil(floor(Y / 4) / 512) of them) one rescale (exp 4 u, product u, argument u |dm|) and one add, one tail element (6 u),
    and at most 5 warp-shuffle and 15 shared-memory folds (6 u each).  The |dm| along a path add up to at most the row's
    range R, so the sum is within u (6 n_t + 134 + 2 R) relative (x 1.01 for second-order terms), R = the float64 range
    of the row + 2 dmax.  logf adds 1 ulp (2 u log Y), t - m u R, the final subtraction u (|result| + 1).
  * rank equals the float64 rank unless some j != y_b has |S64_j - t64| <= delta_j + delta_y (twice the bound when the
    norms are equal): only those comparisons can flip, so the rank then lies within their count of the float64 rank.
  * top1 is the float64 argmax or a column within dmax + delta_top1 of the float64 max.
c2v_loss reads the same slab: per row its lse and this kernel's both lie within their own rounding of the exact lse of the
stored logits (the loss path's: its epilogue partials of 64 columns, ex2.approx with a 2^-22 relative error and an
argument of error u (|x| + |max|) log2 e, combined over ceil(Y / 128) * 2 slots), so |-mean(logp) - loss| <= the mean of
both rounding bounds + 2 (B + 1) u mean|logp| (two float32 B-term means)."""
import math

import numpy as np
import pytest

from code2vec_b200.name_scores import format_line
from tests import similarity_model as SM
from tests.name_scores_model import name_scores64

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
D, THREADS = 384, 512
MODES = [0, 1, 2]
YS = [1, 2, 127, 128, 129, 257, 261245]
BS = [1, 37, 1024]

_eng = {}
_ref = {}


@pytest.fixture(scope="module", autouse=True)
def _release():
    yield
    for e in _eng.values():
        e.close()
    _eng.clear()
    _ref.clear()


def _engine(Y):
    """One engine at a time: java14m code width, Y target rows, max batch 1024, seeded parameters."""
    from code2vec_b200.engine import EngineDims, PathAttentionEngine
    if Y not in _eng:
        for e in _eng.values():
            e.close()
        _eng.clear()
        eng = PathAttentionEngine(EngineDims(101, 101, Y, 128, D, 8, 1024, 10), device=0, training=False)
        eng.init_params(seed=7 + Y)
        _eng[Y] = eng
    return _eng[Y]


def _inputs(eng, Y, B, seed):
    import torch
    g = torch.Generator(device=eng.dev).manual_seed(seed)
    v = 3.0 * torch.randn((B, D), generator=g, device=eng.dev)          # logits of standard deviation about 3
    y = torch.randint(0, Y, (B,), generator=g, device=eng.dev, dtype=torch.int32)
    return v, y


def _chain(Y):
    return 6 * math.ceil((Y // 4) / THREADS) + 134


def _round(Y, R, mag, chain):
    return U * (1.01 * (chain + 2 * R) + 2 * math.log(max(Y, 2)) + R + mag + 1)


def _loss_chain(Y):
    return 6 * (math.ceil(2 * math.ceil(Y / 128) / 256) + 64 + 20) + 134


def _reference(Y, B):
    """Per row: the float64 statement's results, and per mode the bounds, the close-logit counts and the near-max columns."""
    import torch
    key = (Y, B)
    if key in _ref:
        return _ref[key]
    eng = _engine(Y)
    v, y = _inputs(eng, Y, B, seed=Y * 31 + B)
    T64 = eng.params["tgt"].double()
    tn = torch.linalg.vector_norm(T64, dim=1)
    v64 = v.double()
    vn = torch.linalg.vector_norm(v64, dim=1)
    cols = torch.arange(Y, device=eng.dev)
    out = dict(rank=[], logp=[], top1=[], top1_logp=[], R=[], A=[], close={m: [] for m in MODES}, dmax={m: [] for m in MODES},
               dy={m: [] for m in MODES}, near={m: [] for m in MODES})
    for r0 in range(0, B, 64):
        r1 = min(B, r0 + 64)
        S = v64[r0:r1] @ T64.T
        yy = y[r0:r1].long()
        res = name_scores64(S.cpu().numpy(), yy.cpu().numpy())
        for k, a in zip(("rank", "logp", "top1", "top1_logp"), res):
            out[k].append(a)
        t = S.gather(1, yy[:, None])
        m = S.max(dim=1, keepdim=True).values
        for mode in MODES:
            vb = SM.value_bound(mode, D)
            delta = vb * vn[r0:r1, None] * tn[None, :]
            dmax = delta.max(dim=1).values
            dy = delta.gather(1, yy[:, None])
            close = ((S - t).abs() <= delta + dy) & (cols[None, :] != yy[:, None])
            out["close"][mode].append(close.sum(dim=1).cpu().numpy())
            out["dmax"][mode].append(dmax.cpu().numpy())
            out["dy"][mode].append(dy[:, 0].cpu().numpy())
            near = S >= m - (dmax[:, None] + delta)
            out["near"][mode].extend([set(torch.nonzero(near[i]).flatten().tolist()) for i in range(r1 - r0)])
        out["R"].append((m[:, 0] - S.min(dim=1).values).cpu().numpy())
        out["A"].append(S.abs().max(dim=1).values.cpu().numpy())
        del S
    ref = {k: (np.concatenate(a) if isinstance(a, list) else a) for k, a in out.items()}
    for k in ("close", "dmax", "dy"):
        ref[k] = {mode: np.concatenate(a) for mode, a in out[k].items()}
    ref["v"], ref["y"] = v, y
    _ref[key] = ref
    return ref


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B", BS)
@pytest.mark.parametrize("Y", YS)
def test_against_float64(Y, B, mode):
    import torch
    ref = _reference(Y, B)
    eng = _engine(Y)
    eng.set_option("math_mode", mode)
    rank, logp, top1, top1_logp = (x.cpu().numpy() for x in eng.name_scores(ref["v"], ref["y"]))
    loss = float(eng.loss(ref["v"], ref["y"]).cpu()[0])
    torch.cuda.synchronize()
    dmax, dy, close = ref["dmax"][mode], ref["dy"][mode], ref["close"][mode]
    R = ref["R"] + 2 * dmax
    worst = 0.0
    for b in range(B):
        lb = dy[b] + dmax[b] + _round(Y, R[b], abs(ref["logp"][b]), _chain(Y))
        tb = 2 * dmax[b] + _round(Y, R[b], abs(ref["top1_logp"][b]), _chain(Y))
        assert abs(logp[b] - ref["logp"][b]) <= lb, (b, logp[b], ref["logp"][b], lb)
        assert abs(top1_logp[b] - ref["top1_logp"][b]) <= tb, (b, top1_logp[b], ref["top1_logp"][b], tb)
        worst = max(worst, abs(logp[b] - ref["logp"][b]) / lb)
        if close[b] == 0:
            assert rank[b] == ref["rank"][b], (b, rank[b], ref["rank"][b])
        else:
            assert abs(int(rank[b]) - int(ref["rank"][b])) <= close[b], (b, rank[b], ref["rank"][b], close[b])
        assert top1[b] == ref["top1"][b] or int(top1[b]) in ref["near"][mode][b], (b, top1[b], ref["top1"][b])
    assert np.all(rank >= 1) and np.all(rank <= Y)
    mean_logp = float(np.mean(np.abs(ref["logp"])))
    lb = np.mean([_round(Y, R[b], abs(ref["logp"][b]), _chain(Y)) +
                  _round(Y, R[b] + 3 * (ref["A"][b] + 2 * dmax[b]), abs(ref["logp"][b]), max(_chain(Y), _loss_chain(Y))) for b in range(B)])
    lb += 2 * (B + 1) * U * mean_logp
    assert abs(-float(np.mean(logp.astype(np.float64))) - loss) <= lb, (-np.mean(logp), loss, lb)
    print("NAME-SCORES Y=%d B=%d mode=%d worst logp error / bound = %.3g" % (Y, B, mode, worst))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("Y", [129, 261245])
def test_bit_exact_against_topk(Y, mode):
    """A table with duplicated rows (exact ties at tile edges) and code vectors pointing at them: top1 is c2v_topk's first
    id; a target taken from position j of the top-k list has rank j + 1; a rank r <= k sits at position r - 1, and a
    rank beyond k is not in the list."""
    import torch
    from code2vec_b200.engine import EngineDims, PathAttentionEngine
    eng = PathAttentionEngine(EngineDims(101, 101, Y, 128, D, 8, 1024, 10), device=0, training=False)
    try:
        eng.init_params(seed=99)
        tgt = eng.params["tgt"]
        c = 100
        dups = sorted({d for d in (0, 63, 64, 127, 128, Y - 1) if d != c and d < Y})
        tgt[dups] = tgt[c].clone()
        B = 1024
        g = torch.Generator(device=eng.dev).manual_seed(5)
        v = 0.5 * torch.randn((B, D), generator=g, device=eng.dev)
        v[::2] += 30.0 * tgt[c]                          # even rows: c and its duplicates lead, tied
        eng.set_option("math_mode", mode)
        ids, _ = eng.topk(v, normalize=False)
        k = ids.shape[1]
        ids_h = ids.cpu().numpy()
        y = torch.randint(0, Y, (B,), generator=g, device=eng.dev, dtype=torch.int32)
        pos = np.arange(B) % k
        take = np.arange(B) % 3 == 0                     # a third of the rows: the target is a top-k entry
        y_h = y.cpu().numpy()
        y_h[take] = ids_h[take, pos[take]]
        y_h[1::6] = np.array(dups + [c])[np.arange(len(y_h[1::6])) % (len(dups) + 1)]
        y = torch.from_numpy(y_h).to(eng.dev)
        rank, _, top1, _ = (x.cpu().numpy() for x in eng.name_scores(v, y))
        ids2, _ = eng.topk(v, normalize=False)
        assert torch.equal(ids, ids2)                    # the slab is rebuilt the same way every call
        assert np.array_equal(top1, ids_h[:, 0])
        assert np.array_equal(rank[take], pos[take] + 1)
        for b in range(B):
            if rank[b] <= k:
                assert ids_h[b, rank[b] - 1] == y_h[b], b
            else:
                assert y_h[b] not in ids_h[b], b
        assert ids_h[0, :len(dups) + 1].tolist() == sorted(dups + [c])
    finally:
        eng.close()


# ---- the command line ---------------------------------------------------------------------------------------------------
def _lines(prefix):
    return [l for l in open(prefix + ".test.c2v").read().splitlines() if l.strip()]


def test_score_names_end_to_end(tmp_path, monkeypatch):
    """Train a small model from the command line, then `--score_names` for both frameworks on the same checkpoint."""
    import tests.test_gpu_model as G
    from code2vec_b200 import load_model_dynamically
    from code2vec_b200.__main__ import main
    from code2vec_b200.b200_model import _EvaluateInputFormer
    from code2vec_b200.config import Config
    from code2vec_b200.path_context_reader import EstimatorAction, PathContextReader
    monkeypatch.setattr(G, "C", 200)                 # the default MAX_CONTEXTS
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    prefix, test_lines = G._make_dataset(tmp_path)
    save = str(tmp_path / "m" / "saved")
    assert main(["--data", prefix, "--save", save, "--framework", "b200"]) == 0
    data = prefix + ".test.c2v"
    with open(data, "a") as f:                       # names outside the target vocabulary
        for i, line in enumerate(test_lines[:3]):
            f.write("no|such|name%d %s\n" % (i, line.split(" ", 1)[1]))
    assert main(["--load", save, "--test", data, "--export_code_vectors", "--framework", "b200"]) == 0
    n_vectors = len(open(data + ".vectors").read().splitlines())
    out = {}
    for fw in ("b200", "b200-keras"):
        assert main(["--load", save, "--score_names", data, "--framework", fw]) == 0
        out[fw] = open(data + ".name_scores", "rb").read()
    assert out["b200"] == out["b200-keras"]
    rows = [l.split("\t") for l in out["b200"].decode().splitlines()]
    names = [l.split(" ")[0] for l in _lines(prefix)]
    assert len(rows) == n_vectors == len(names)
    assert [r[0] for r in rows] == names
    assert all(len(r) == 5 for r in rows)
    oov = [r for r in rows if r[0].startswith("no|such|name")]
    assert len(oov) == 3 and all(r[1] == "-" and r[2] == "-" and r[4] != "nan" for r in oov)
    assert all(r[1] != "-" for r in rows if not r[0].startswith("no|such|name"))

    config = Config(set_defaults=True)
    config.load_from_args(["--load", save])
    config.verify()
    model = load_model_dynamically(config)
    try:
        names2, ids, rank, logp, top1, top1_logp = model.score_names(data)
        assert names2 == names
        cfg = config
        cfg.TEST_DATA_PATH = data
        reader = PathContextReader(vocabs=model.vocabs, model_input_tensors_former=_EvaluateInputFormer(), config=cfg,
                                   estimator_action=EstimatorAction.Evaluate)
        model.engine.set_option("math_mode", model._math_eval)
        pred = []
        for batch in reader.get_dataset():
            t = _EvaluateInputFormer().from_model_input_form(batch)
            idx, _, _, _ = model.engine.predict_batch_host(t.path_source_token_indices, t.path_indices,
                                                           t.path_target_token_indices, t.context_valid_mask,
                                                           normalize=False, want_code=False, want_attention=False)
            pred.append(idx)
        pred = np.concatenate(pred)
        k = pred.shape[1]
        assert np.array_equal(top1, pred[:, 0])
        ranked = 0
        for r in range(len(names)):
            if rank[r] <= k:
                assert pred[r, rank[r] - 1] == ids[r], r
                ranked += 1
            else:
                assert ids[r] not in pred[r], r
        assert ranked > len(names) // 2                 # the toy rule is learnable: most names rank in the top k
        vocab = model.vocabs.target_vocab
        for r, row in enumerate(rows):
            in_vocab = ids[r] != vocab.word_to_index[vocab.special_words.OOV]
            assert "\t".join(row) + "\n" == format_line(names[r], bool(in_vocab), int(rank[r]), float(logp[r]),
                                                       vocab.lookup_word(int(top1[r])), float(top1_logp[r]))
    finally:
        model.close_session()
