"""Nearest-neighbour search on the GPU (csrc/knn.cu, similarity.py, DESIGN.md §6h) against the float64 statement of
tests/similarity_model.py, in fp32, tf32 and 3xTF32: tables of 1 to 261,246 rows at d = 128 and 384, k on the epilogue
route (1, 10, 16) and the slab route (40, and 16 with exclusions past 16), one and several query blocks, exact ties at
slot, tile and block edges, zero and NaN rows; then most_similar and --nearest on a small trained model."""
import numpy as np
import pytest

from tests import similarity_model as M

pytestmark = pytest.mark.gpu

MODES = [0, 1, 2]


def _nn():
    from code2vec_b200.similarity import NearestNeighbours
    return NearestNeighbours("cuda:0")


def _table(N, d, seed):
    import torch
    g = torch.Generator(device="cuda:0").manual_seed(seed)
    t = torch.randn((N, d), generator=g, device="cuda:0", dtype=torch.float32)
    if N > 40:
        t[5] = 0.0                      # zero row
        t[17, 3] = float("nan")         # NaN row
        t[33] = t[20]                   # an exact duplicate
    return t


def _oracle(t64, q64, k, exclude):
    """Per query: (oracle ids, float64 scores of every row) -- scores in float64 on the device, the ranking on the host."""
    import torch
    s = (t64 @ q64.T) / torch.linalg.vector_norm(t64, dim=1, keepdim=True)        # [N, nq]
    s = torch.nan_to_num(s, nan=-np.inf).T.contiguous()
    out = []
    take = min(int(s.shape[1]), k + 64)
    for r in range(s.shape[0]):
        v, i = torch.topk(s[r], take)
        v, i = v.cpu().numpy(), i.cpu().numpy()
        row = np.full(int(s.shape[1]), np.nan)
        row[i] = v
        row[row == -np.inf] = np.nan
        out.append(M.search64(row, k, exclude[r]))
    return out, s


def _check(idx, val, oracle, s64, bound):
    """values within `bound` of float64; ids the oracle's except where two candidates are within 2 bound."""
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    for r, want in enumerate(oracle):
        got = [int(i) for i in idx[r] if i != M.PAD]
        assert len(got) == len(want), (r, got, want)
        assert np.all(idx[r, len(got):] == M.PAD) and np.all(val[r, len(got):] == -np.inf)
        exact = s64[r, got].cpu().numpy()
        assert np.all(np.isfinite(exact)), "a NaN or zero row was returned"
        assert np.all(np.abs(val[r, :len(got)] - exact) <= bound), (r, np.abs(val[r, :len(got)] - exact).max(), bound)
        for j, (g, w) in enumerate(zip(got, want)):
            if g != w:
                assert abs(float(s64[r, g]) - float(s64[r, w])) <= 2 * bound, (r, j, g, w)
        assert got == sorted(got, key=lambda i: (-val[r, got.index(i)], i))


def _word_queries(nn, N, nq, seed):
    rng = np.random.default_rng(seed)
    lists, weights = [], []
    for _ in range(nq):
        a = int(rng.integers(1, 4))
        lists.append([int(x) for x in rng.integers(0, N, size=a)])
        weights.append([1.0] * (a - 1 if a > 1 else 1) + [-1.0] * (1 if a > 1 else 0))
    off = np.zeros(nq + 1, dtype=np.int64)
    np.cumsum([len(x) for x in lists], out=off[1:])
    q = nn.queries(np.concatenate(lists), np.concatenate(weights), off)
    return q, lists, weights


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("d", [128, 384])
@pytest.mark.parametrize("N", [1, 37, 127, 128, 129, 1537])
@pytest.mark.parametrize("k,excl", [(1, 0), (10, 2), (16, 0), (16, 3), (40, 1)])
def test_search_matches_float64(mode, d, N, k, excl):
    import torch
    nq = 129
    nn = _nn()
    try:
        t = _table(N, d, seed=N + d)
        nn.bind(t, mode)
        q, lists, _ = _word_queries(nn, N, nq, seed=N * 7 + k)
        exclude = [lst[:excl] for lst in lists]
        idx, val = nn.search(q, k, exclude=exclude)
        torch.cuda.synchronize()
        oracle, s64 = _oracle(t.double(), q.double(), k, exclude)
        _check(idx, val, oracle, s64, M.value_bound(mode, d))
    finally:
        nn.close()


@pytest.mark.parametrize("mode", MODES)
def test_query_vectors_are_gensims(mode):
    import torch
    nn = _nn()
    try:
        t = _table(300, 128, seed=3)
        nn.bind(t, mode)
        q = nn.queries(np.array([4, 9, 4, 7, 7]), np.array([1, 1, -1, 1, -1], np.float32), np.array([0, 2, 3, 5]))
        t64 = t.double().cpu().numpy()
        want = [M.query64(t64, [4, 9], [1, 1]), M.query64(t64, [4], [-1]), np.zeros(128)]
        assert np.abs(q.cpu().numpy() - np.array(want)).max() <= 2 ** -24
        assert not q[2].any()                       # p = n: a zero query; every finite row then scores 0
        idx, val = nn.search(q[2:3], 5, exclude=[[7, 7]])
        assert idx[0].tolist() == [0, 1, 2, 3, 4] and not val.any()
        torch.cuda.synchronize()
    finally:
        nn.close()


@pytest.mark.parametrize("mode", MODES)
def test_java14m_sized_table_over_several_query_blocks(mode):
    """N = 261,246 target rows; 1,600 queries span more than one block on every route; duplicated rows sit at slot, tile
    and block edges and come back in ascending id order with the same bits; queries equal across a block boundary get
    equal results."""
    import torch
    N, d, k, nq = 261246, 128, 10, 1600
    nn = _nn()
    try:
        t = _table(N, d, seed=11)
        dups = [63, 64, 127, 128, 129, 260095, 261245]
        t[dups] = t[1000].clone()
        t[2000:2010] = 0.0
        nn.bind(t, mode)
        rows = np.random.default_rng(5).integers(0, N, size=nq)
        rows[1407:1409] = 1000               # a tensor-core block holds 1408 queries here, a slab block 512
        rows[511:513] = 1000
        q = nn.queries(rows, np.ones(nq, np.float32), np.arange(nq + 1))
        exclude = [[int(r)] for r in rows]
        idx, val = nn.search(q, k, exclude=exclude)
        torch.cuda.synchronize()
        for r in (511, 512, 1407, 1408):
            assert idx[r].tolist()[:7] == sorted(dups), idx[r].tolist()
            assert torch.equal(val[r, :7], val[r, :1].expand(7))
            assert torch.equal(idx[r], idx[511]) and torch.equal(val[r], val[511])
        pick = list(range(0, nq, 97)) + [511, 512, 1407, 1408]
        oracle, s64 = _oracle(t.double(), q[pick].double(), k, [exclude[r] for r in pick])
        _check(idx[pick], val[pick], oracle, s64, M.value_bound(mode, d))
        assert not set(range(2000, 2010)) & set(idx.flatten().tolist())
        assert nn.device_bytes() < (3 << 30)
    finally:
        nn.close()


@pytest.mark.parametrize("mode", MODES)
def test_single_query_at_d384(mode):
    import torch
    N, d = 261246, 384
    nn = _nn()
    try:
        t = _table(N, d, seed=12)
        nn.bind(t, mode)
        q, lists, _ = _word_queries(nn, N, 1, seed=1)
        for k in (1, 10, 16, 40):
            idx, val = nn.search(q, k, exclude=[lists[0]])
            torch.cuda.synchronize()
            oracle, s64 = _oracle(t.double(), q.double(), k, [lists[0]])
            _check(idx, val, oracle, s64, M.value_bound(mode, d))
    finally:
        nn.close()


# ---- the model ------------------------------------------------------------------------------------------------------------
def _read_w2v(path):
    with open(path) as f:
        n, dim = (int(x) for x in f.readline().split())
        words, rows = [], []
        for line in f:
            parts = line.rstrip("\n").split(" ")
            words.append(parts[0])
            rows.append(np.array(parts[1:], dtype=np.float32))
    assert len(words) == n and all(r.size == dim for r in rows)
    return words, np.stack(rows)


@pytest.mark.parametrize("math", ["fp32", "tf32", "3xtf32"])
def test_most_similar_on_a_trained_model(tmp_path, monkeypatch, math):
    from code2vec_b200.b200_model import Code2VecModel
    from code2vec_b200.vocabularies import VocabType
    from tests.test_gpu_device_eval import _dataset, _train
    from tests.test_gpu_model import _config
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    prefix = _dataset(tmp_path, adversarial=False)
    save = _train(prefix, tmp_path, epochs=1)
    monkeypatch.setenv("C2V_MATH", math)
    m = Code2VecModel(_config(prefix, tmp_path, MODEL_LOAD_PATH=save))
    try:
        for vt in (VocabType.Target, VocabType.Token):
            path = str(tmp_path / ("%s.w2v" % vt.name))
            m.save_word2vec_format(path, vt)            # what --save_t2v / --save_w2v write
            words, table = _read_w2v(path)
            w2i = {w: i for i, w in enumerate(words)}
            mode = {"fp32": 0, "tf32": 1, "3xtf32": 2}[math]
            for pos, neg in ((words[3:5], []), (words[6:8], words[9:10]), (words[2:3] * 2, [])):
                got = m.most_similar(pos, neg, topn=7, vocab_type=vt)
                want, s64 = M.most_similar64(table, w2i, pos, neg, topn=7)
                bound = M.value_bound(mode, table.shape[1])
                assert len(got) == len(want)
                for (gw, gv), (wi, wv) in zip(got, want):
                    assert abs(gv - s64[w2i[gw]]) <= bound
                    assert gw == words[wi] or abs(s64[w2i[gw]] - wv) <= 2 * bound
                assert not set(pos + neg) & {w for w, _ in got}
        assert m.most_similar(words[:1], topn=0, vocab_type=VocabType.Token) == []
        with pytest.raises(KeyError, match="not present in vocabulary"):
            m.most_similar(["no|such|word"])
    finally:
        m.close_session()


def test_nearest_code_vectors(tmp_path, monkeypatch):
    from code2vec_b200.__main__ import write_nearest
    from code2vec_b200.b200_model import Code2VecModel
    from tests.test_gpu_device_eval import _dataset, _evaluate, _train
    from tests.test_gpu_model import _config
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    prefix = _dataset(tmp_path)
    save = _train(prefix, tmp_path, epochs=1)
    _, _, vectors_text = _evaluate(monkeypatch, prefix, tmp_path, save, "0", TEST_BATCH_SIZE=32)
    exported = np.array([np.array(l.split(" "), dtype=np.float32) for l in vectors_text.decode().splitlines()])
    m = Code2VecModel(_config(prefix, tmp_path, MODEL_LOAD_PATH=save, TEST_BATCH_SIZE=32))
    try:
        names, vectors, idx, val = m.nearest_code_vectors(prefix + ".test.c2v", 5)
        assert np.array_equal(vectors, exported)                   # the .vectors file's code vectors, bit for bit
        n = vectors.shape[0]
        t64 = vectors.astype(np.float64)
        bound = M.value_bound(m._math_eval, vectors.shape[1])
        for r in range(n):
            s = M.scores64(t64, M.query64(t64, [r], [1.0]))
            want = M.search64(s, 5, [r])
            got = [int(i) for i in idx[r] if i != M.PAD]
            assert len(got) == len(want) and r not in got
            assert np.all(np.abs(val[r, :len(got)] - s[got]) <= bound)
            assert all(g == w or abs(s[g] - s[w]) <= 2 * bound for g, w in zip(got, want))
        out = write_nearest(m, prefix + ".test.c2v", 5)
        lines = open(out).read().splitlines()
        assert len(lines) == n
        first = lines[0].split("\t")
        assert first[0] == names[0] and first[1].split(",")[0] == str(int(idx[0, 0]))
    finally:
        m.close_session()
