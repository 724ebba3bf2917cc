"""What the evaluation kernels of csrc/reader.cu compute (C2V_DEVICE_EVAL=1, DESIGN.md §6e), stated in pure Python / numpy
and checked without a GPU against the host code they replace:
  * scoring: eval_score_kernel's rank, first legal word, subtoken counts and host-row flags, on the byte tables
    device_reader.eval_tables builds, against common.get_first_match_word_from_top_predictions,
    SubtokensEvaluationMetric and TopKAccuracyEvaluationMetric;
  * batching: the stable append of every chunk's kept rows and the cut into TEST_BATCH_SIZE batches, against
    PathContextReader._iterate_batches_native in evaluate mode;
  * the switch, the Keras refusal, and the new C ABI in the cross-compiled library."""
import random
from collections import Counter
from functools import partial

import numpy as np
import pytest

from code2vec_b200.common import common
from code2vec_b200.vocabularies import _SpecialVocabWords_JoinedOovPad as _JOIN, _SpecialVocabWords_OnlyOov as _SEP


# ---- scoring -----------------------------------------------------------------------------------------------------------
class _Vocab:
    def __init__(self, words, special):
        self.special_words = special
        self.index_to_word = dict(enumerate(words))
        self.size = len(words)


def _letter(c: int) -> bool:
    return 0x41 <= c <= 0x5A or 0x61 <= c <= 0x7A


def _norm_equal(name: bytes, nw: bytes) -> bool:
    letters = bytes(c | 0x20 for c in name if _letter(c))
    return (letters if letters else name) == nw


def score_row(name: bytes, ids, tables):
    """eval_score_kernel for one row: (rank, first, flags, (tp, fp, fn) or None)."""
    w, w_off, n, n_off, legal = tables
    Y = legal.size
    if any(c >= 0x80 for c in name):
        return -1, -1, 1, None
    word = lambda i: bytes(w[w_off[i]:w_off[i + 1]])
    norm = lambda i: bytes(n[n_off[i]:n_off[i + 1]])
    rank, first, before = -1, -1, 0
    for i in ids:
        lg = 0 <= i < Y and legal[i]
        if not lg:
            continue
        if first < 0:
            first = int(i)
        if rank < 0 and _norm_equal(name, norm(i)):
            rank = before
        before += 1
    if first < 0:
        return -1, -1, 2, None
    truth, guess = name.split(b"|"), word(first).split(b"|")
    tp = sum(1 for g in guess if g in truth)
    fn = sum(1 for t in truth if t not in guess)
    return rank, first, 0, (tp, len(guess) - tp, fn)


def _host(name: str, ids, vocab):
    """The host metrics on one row: (found, (tp, fp, fn)) or the exception they raise."""
    from code2vec_b200.b200_model import SubtokensEvaluationMetric
    special = vocab.special_words
    top = [vocab.index_to_word.get(int(i), special.OOV) for i in ids]
    found = common.get_first_match_word_from_top_predictions(special, name, top)
    m = SubtokensEvaluationMetric(partial(common.filter_impossible_names, special))
    try:
        m.update_batch([(name, top)])
    except IndexError:
        return found, "IndexError"
    return found, (m.nr_true_positives, m.nr_false_positives, m.nr_false_negatives)


NAMES = ["", "<OOV>", "<PAD_OR_OOV>", "a,b", "get2x", "_", "123", "|", "||", "|get", "get|", "get|get|x", "getX",
         "get|x", "GETX", "get_x", "a||b", "x", "copy|name", "name|copy|copy", "get,x|y"]
NON_ASCII = ["ü", "\u212a", "Kelvin\u212a", "name|ü", "名前"]
WORDS = ["|", "a||b", "get|x", "getx", "GetX", "get|get|x", "x", "get_x2", "x1", "", "name|copy", "copy|name", "get",
         "name|copy|copy", "ü", "a|b|", "|a"]


@pytest.fixture(params=["separate", "joined"])
def vocab(request):
    from code2vec_b200.device_reader import eval_tables
    special = _SEP if request.param == "separate" else _JOIN
    specials = [special.OOV]
    v = _Vocab(specials + WORDS, special)
    return v, eval_tables(v)


def _check(name: str, ids, v, tables):
    data = (v.special_words.OOV if name == "" else name).encode("utf-8")     # an empty name field is the OOV word
    rank, first, flags, counts = score_row(data, ids, tables)
    if flags == 1:
        return "host"
    found, host = _host(data.decode("utf-8"), ids, v)
    if flags == 2:
        assert host == "IndexError" and found is None
        return "no legal"
    assert (found is None) == (rank < 0) and (found is None or found[0] == rank), (name, ids)
    if rank == 0:                                        # log.txt's "predicted 1st" word is the first legal one
        assert found[1] == v.index_to_word[first]
    assert host == counts, (name, ids, host, counts)
    return "device"


def test_adversarial_names_score_like_the_host(vocab):
    v, tables = vocab
    Y = v.size
    kinds = Counter()
    for name in NAMES:
        for ids in (list(range(Y))[:10], list(range(Y))[::-1][:10], list(range(Y))[3:8], [Y - 1, 0, 1],
                    [i for i in range(Y) if i not in (2, 3, 4)][:10]):
            kinds[_check(name, ids, v, tables)] += 1
    for name in NON_ASCII:
        assert score_row(name.encode("utf-8"), [0, 1], tables)[2] == 1          # flagged: the host scores it
        assert score_row(b"\xff\xfe", [0, 1], tables)[2] == 1
    assert kinds["device"] > 50


def test_normalized_matches_and_ranks_within_the_legal_list(vocab):
    v, tables = vocab
    idx = {w: i for i, w in v.index_to_word.items()}
    ids = [idx["get_x2"], idx["x1"], idx["GetX"], idx["get|x"], idx["x"]]        # two illegal words first
    assert score_row(b"getX", ids, tables)[:2] == (0, idx["GetX"])
    assert score_row(b"get|x", ids, tables)[:2] == (0, idx["GetX"])
    assert score_row(b"x", ids, tables)[:2] == (2, idx["GetX"])
    assert score_row(b"|", [idx["|"], idx["x"]], tables)[:2] == (0, idx["|"])
    assert score_row(b"123", [idx["x"]], tables)[0] == -1
    for name in ("getX", "get|x", "x", "|", "123", "||"):
        _check(name, ids, v, tables)


def test_all_illegal_top_k_and_y_below_k(vocab):
    v, tables = vocab
    idx = {w: i for i, w in v.index_to_word.items()}
    illegal = [idx["get_x2"], idx["x1"], idx[v.special_words.OOV]]
    assert score_row(b"getx", illegal, tables)[2] == 2
    assert _check("getx", illegal, v, tables) == "no legal"
    small = _Vocab([v.special_words.OOV, "get", "x"], v.special_words)
    from code2vec_b200.device_reader import eval_tables
    t = eval_tables(small)
    for name in NAMES:
        _check(name, [2, 0, 1], small, t)                                       # k = Y = 3 < TOP_K


def test_random_sweep(vocab):
    v, tables = vocab
    rng = random.Random(5)
    alphabet = ["get", "x", "X", "|", "", "a", "B", "1", "_", ",", "name", "copy"]
    for _ in range(3000):
        name = "".join(rng.choice(alphabet) for _ in range(rng.randint(0, 5)))
        ids = rng.sample(range(v.size), min(v.size, rng.randint(1, 10)))
        _check(name, ids, v, tables)


def test_accumulators_give_the_host_metrics_floats(vocab):
    """Integer sums of the device rows, added to the metric objects, give the same floats as update_batch row by row."""
    from code2vec_b200.b200_model import SubtokensEvaluationMetric, TopKAccuracyEvaluationMetric
    v, tables = vocab
    special = v.special_words
    rng = random.Random(9)
    K = 10
    rows = []
    for _ in range(400):
        name = rng.choice(NAMES[3:] + [w for w in WORDS if w])
        ids = rng.sample(range(v.size), min(v.size, K))
        if score_row(name.encode(), ids, tables)[2] == 0:
            rows.append((name, ids))
    top = lambda ids: [v.index_to_word[i] for i in ids]
    want_s = SubtokensEvaluationMetric(partial(common.filter_impossible_names, special))
    want_t = TopKAccuracyEvaluationMetric(K, partial(common.get_first_match_word_from_top_predictions, special))
    pairs = [(n, top(i)) for n, i in rows]
    want_t.update_batch(pairs)
    want_s.update_batch(pairs)
    got_s = SubtokensEvaluationMetric(partial(common.filter_impossible_names, special))
    got_t = TopKAccuracyEvaluationMetric(K, partial(common.get_first_match_word_from_top_predictions, special))
    hist, acc = np.zeros(K, dtype=np.int64), np.zeros(4, dtype=np.int64)
    for n, ids in reversed(rows):                                            # the order does not matter
        rank, _, _, (tp, fp, fn) = score_row(n.encode(), ids, tables)
        if rank >= 0:
            hist[rank] += 1
        acc += (1, tp, fp, fn)
    got_t.nr_correct_predictions = got_t.nr_correct_predictions + np.cumsum(hist).astype(np.float64)
    got_t.nr_predictions += int(acc[0])
    got_s.nr_predictions += int(acc[0])
    got_s.nr_true_positives += int(acc[1])
    got_s.nr_false_positives += int(acc[2])
    got_s.nr_false_negatives += int(acc[3])
    assert np.array_equal(got_t.topk_correct_predictions, want_t.topk_correct_predictions)
    assert (got_s.precision, got_s.recall, got_s.f1) == (want_s.precision, want_s.recall, want_s.f1)


# ---- batching ----------------------------------------------------------------------------------------------------------
def _eval_reader(tmp_path, lines, batch, chunk_bytes, C=4):
    import pickle
    from code2vec_b200 import vocabularies as V
    from code2vec_b200.config import Config
    from code2vec_b200.path_context_reader import EstimatorAction, PathContextReader
    prefix = str(tmp_path / "ds")
    with open(prefix + ".dict.c2v", "wb") as f:
        for d in ({"t%d" % i: 3 for i in range(6)}, {"1%d" % i: 3 for i in range(4)}, {"n%d" % i: 3 for i in range(3)}):
            pickle.dump(d, f)
        pickle.dump(10, f)
    with open(prefix + ".test.c2v", "w") as f:
        f.write("".join(lines))
    cfg = Config(set_defaults=True)
    cfg.VERBOSE_MODE = 0
    cfg.TRAIN_DATA_PATH_PREFIX = prefix
    cfg.TEST_DATA_PATH = prefix + ".test.c2v"
    cfg.MAX_CONTEXTS = C
    cfg.TEST_BATCH_SIZE = batch
    cfg.MAX_TOKEN_VOCAB_SIZE = cfg.MAX_PATH_VOCAB_SIZE = cfg.MAX_TARGET_VOCAB_SIZE = 10 ** 6

    class F:
        def to_model_input_form(self, t):
            return t

        def from_model_input_form(self, r):
            return r
    r = PathContextReader(V.Code2VecVocabs(cfg), cfg, F(), EstimatorAction.Evaluate, use_native=True)
    r.chunk_bytes = chunk_bytes
    r._native_ready()
    return r


def device_batches(reader):
    """The evaluation queue: each chunk's records parsed, the kept ones (a valid context, any target) appended in file
    order with their names (the OOV word for an empty field 0), and a batch cut whenever B rows are queued; the last
    batch is what remains."""
    B = reader.config.TEST_BATCH_SIZE
    queue, out = [], []
    for chunk in reader._native_chunks():
        arrs, names = reader._native_parse(chunk)     # the kept records of the chunk and their names, in file order
        rows = list(zip(*(a.tolist() for a in arrs)))
        queue += list(zip(rows, names))
        while len(queue) >= B:
            out.append(queue[:B])
            queue = queue[B:]
    if queue:
        out.append(queue)
    return out


def _lines(rng, n, C=4):
    lines = []
    for i in range(n):
        kind = rng.integers(0, 10)
        if kind == 0:
            lines.append("\n")                                   # blank: skipped
            continue
        name = ["n0", "n1", "", "zz", "a,b", "n2|x"][int(rng.integers(0, 6))]
        if kind == 1:
            ctx = [""] * C                                       # no valid context: dropped
        else:
            ctx = ["t%d,1%d,t%d" % (rng.integers(0, 8), rng.integers(0, 5), rng.integers(0, 8)) if rng.random() < 0.7
                   else "" for _ in range(C)]
        lines.append(" ".join([name] + ctx) + "\n")
    return lines


@pytest.mark.parametrize("batch", [1, 7, 500])
@pytest.mark.parametrize("chunk_bytes", [64, 300, 16 << 20])
def test_stable_append_and_batch_cut_equal_the_host_reader(tmp_path, batch, chunk_bytes):
    from code2vec_b200.path_context_reader import load_native_tensoriser
    if load_native_tensoriser() is None:
        pytest.skip("libc2v_batcher.so cannot be built here")
    rng = np.random.default_rng(batch * 7 + chunk_bytes)
    reader = _eval_reader(tmp_path, _lines(rng, 120), batch, chunk_bytes)
    want = [b for b in reader._iterate_batches_native()]
    got = device_batches(reader)
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert [n for _, n in g] == list(w.target_string)
        cols = list(zip(*[r for r, _ in g]))
        for c, name in zip(cols, ("path_source_token_indices", "path_indices", "path_target_token_indices",
                                  "context_valid_mask", "target_index")):
            assert np.array_equal(np.array(c), getattr(w, name)), name
    assert sum(len(b) for b in got) < 120


# ---- switch and ABI ----------------------------------------------------------------------------------------------------
def test_device_eval_flag():
    from code2vec_b200.device_reader import device_eval_flag
    assert device_eval_flag({}) is False
    assert device_eval_flag({"C2V_DEVICE_EVAL": "0"}) is False
    assert device_eval_flag({"C2V_DEVICE_EVAL": ""}) is False
    assert device_eval_flag({"C2V_DEVICE_EVAL": "1"}) is True
    for bad in ("2", "yes", "true", " 1"):
        with pytest.raises(ValueError, match="C2V_DEVICE_EVAL must be 0 or 1"):
            device_eval_flag({"C2V_DEVICE_EVAL": bad})


def test_keras_backend_refuses_device_evaluation(monkeypatch):
    from code2vec_b200.b200_keras_model import Code2VecModel
    from code2vec_b200.config import Config
    cfg = Config(set_defaults=True)
    cfg.DL_FRAMEWORK = "b200-keras"
    cfg.VERBOSE_MODE = 0
    monkeypatch.delenv("C2V_DEVICE_READER", raising=False)
    monkeypatch.setenv("C2V_DEVICE_EVAL", "1")
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    with pytest.raises(ValueError, match="C2V_DEVICE_EVAL=1 is not available with --framework b200-keras"):
        Code2VecModel(cfg)
    monkeypatch.setenv("C2V_DEVICE_EVAL", "on")
    with pytest.raises(ValueError, match="C2V_DEVICE_EVAL must be 0 or 1"):
        Code2VecModel(cfg)


def test_the_evaluation_reader_refuses_predict_mode_and_missing_tables(tmp_path):
    from code2vec_b200.device_reader import DeviceBatchReader
    from code2vec_b200.path_context_reader import EstimatorAction
    reader = _eval_reader(tmp_path, ["n0 t0,10,t1    \n"], 4, 1 << 20)
    with pytest.raises(ValueError, match="target-word tables"):
        DeviceBatchReader(reader, "cuda:0")
    reader.estimator_action = EstimatorAction.Predict
    with pytest.raises(ValueError, match="training and evaluation files only"):
        DeviceBatchReader(reader, "cuda:0")


def test_eval_abi_is_declared_and_exported():
    import ctypes
    import re
    from code2vec_b200 import engine as E
    from code2vec_b200.build import LIB_PATH
    header = open(E._build.PKG_DIR + "/../include/c2v_b200.h").read()
    names = ("c2v_reader_eval_tables", "c2v_reader_eval_append", "c2v_reader_eval_take", "c2v_reader_eval_queued",
             "c2v_reader_eval_score")
    E.load_library()
    lib = ctypes.CDLL(LIB_PATH)
    for n in names:
        assert re.search(r"\b%s\(" % n, header), n
        assert n in E._SIGNATURES
        assert hasattr(lib, n), n
