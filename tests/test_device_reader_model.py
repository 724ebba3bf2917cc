"""Host-side statements of the device reader (code2vec_b200/device_reader.py, csrc/reader.cu), checked without a GPU:
  * the vocabulary tables c2v_vocab_export hands to the device, probed in numpy as the parse kernel probes them, give
    c2v_vocab_lookup's index for every word;
  * the index arithmetic of the pool kernels -- commit (holes from the dropped rows' ranks, movers from the kept rows'
    prefix counts) and draw (holes ranked by value among the picks, movers from the unpicked tail) -- stated in numpy,
    reproduces _RowPool's row order on id-tagged rows;
  * C2V_DEVICE_READER is 0 or 1, and --framework b200-keras refuses it."""
import numpy as np
import pytest

from code2vec_b200.path_context_reader import _RowPool, load_native_tensoriser


def _fnv1a(b: bytes) -> int:
    h = 1469598103934665603
    for c in b:
        h = ((h ^ c) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h or 1


def _probe(slots, words, mask, oov, word: bytes) -> int:
    """parse_kernel's lookup(): linear probing from h & mask over the exported slots."""
    h = _fnv1a(word)
    i = h & mask
    while True:
        s_h, s_off, s_len, s_idx = slots[i]
        if s_h == 0:
            return oov
        if s_h == h and s_len == len(word) and words[s_off:s_off + s_len].tobytes() == word:
            return int(s_idx)
        i = (i + 1) & mask


def _native_vocab(lib, words, indices, oov, pad):
    from code2vec_b200.path_context_reader import _NativeVocab

    class _V:
        pass
    v = _V()
    v.word_to_index = dict(zip(words, indices))         # a dict keeps the last index of a repeated word
    v.special_words = type("S", (), {"OOV": words[oov], "PAD": words[pad]})
    return _NativeVocab(lib, v)


needs_native = pytest.mark.skipif(load_native_tensoriser() is None, reason="g++ build of the native tensoriser failed")


@needs_native
@pytest.mark.parametrize("n_words", [5, 40, 3000])
def test_exported_tables_probe_like_the_host_lookup(n_words):
    from code2vec_b200.device_reader import export_vocab
    lib = load_native_tensoriser()
    rng = np.random.default_rng(n_words)
    words = ["<OOV>", "<PAD>", "", "a", "é", "名前|変数", "x" * 301, "dup"]
    words += ["w%d_%s" % (i, "ü" * int(rng.integers(0, 4))) for i in range(n_words)]
    indices = list(range(len(words)))
    # a repeated word: c2v_vocab_create sees it twice and the last index wins, as in the dict the reader builds
    nv = _native_vocab(lib, words + ["dup"], indices + [len(words) + 7], 0, 1)
    slots_raw, byte_arr, mask, oov, pad = export_vocab(lib, nv.h)
    assert (oov, pad) == (0, 1)
    assert slots_raw.shape == (mask + 1, 24) and mask + 1 >= 2 * len(words)
    slots = slots_raw.copy().view(np.dtype([("h", "<u8"), ("off", "<i8"), ("len", "<i4"), ("idx", "<i4")])).ravel()
    slots = [(int(s["h"]), int(s["off"]), int(s["len"]), int(s["idx"])) for s in slots]
    queries = words + ["", "not a word", "x" * 300, "x" * 302, "名前", "w0_", "dupe", "b"]
    chains = 0
    for w in queries:
        b = w.encode("utf-8")
        want = lib.c2v_vocab_lookup(nv.h, b, len(b))
        assert _probe(slots, byte_arr, mask, oov, b) == want, w
        chains += slots[_fnv1a(b) & mask][0] not in (0, _fnv1a(b))
    assert lib.c2v_vocab_lookup(nv.h, b"dup", 3) == len(words) + 7
    if n_words == 3000:
        assert chains > 0                                  # some probe walks past another word's slot


# ---- the pool kernels' index arithmetic --------------------------------------------------------------------------------
def _commit_moves(keep):
    """commit_index_kernel: K(i) = kept rows before i; the dropped row i < kept is hole i - K(i), the kept row i >= kept is
    mover K(i) - K(kept)."""
    keep = np.asarray(keep, dtype=np.int64)
    K = np.concatenate([[0], np.cumsum(keep)])
    kept = int(K[-1])
    m = kept - int(K[kept])
    holes, movers = np.full(m, -1), np.full(m, -1)
    for i in range(len(keep)):
        if i < kept and not keep[i]:
            holes[i - K[i]] = i
        if i >= kept and keep[i]:
            movers[K[i] - K[kept]] = i
    return kept, holes, movers


def _draw_moves(pick, n):
    """draw_index_kernel: a pick below new_n is hole number (how many picks are smaller); the unpicked tail rows are the
    movers in ascending order (an exclusive scan of the tail's flags)."""
    pick = np.asarray(pick)
    b = len(pick)
    new_n = n - b
    tail = np.zeros(b, dtype=bool)
    tail[pick[pick >= new_n] - new_n] = True
    holes = np.full(int((pick < new_n).sum()), -1)
    for v in pick[pick < new_n]:
        holes[int((pick < v).sum())] = v
    movers = new_n + np.flatnonzero(~tail)
    return holes, movers


class _IdPool:
    """The device pool stated with the two index models above, on rows that are their own ids."""

    def __init__(self):
        self.rows = np.zeros(0, dtype=np.int64)

    def commit(self, ids, keep):
        kept, holes, movers = _commit_moves(keep)
        new = np.asarray(ids).copy()
        new[holes] = new[movers]
        self.rows = np.concatenate([self.rows, new[:kept]])

    def take(self, pick, lo, hi):
        out = self.rows[np.asarray(pick)[lo:hi]].copy()
        holes, movers = _draw_moves(pick, len(self.rows))
        assert len(holes) == len(movers)
        self.rows[holes] = self.rows[movers]
        self.rows = self.rows[:len(self.rows) - len(pick)]
        return out


@pytest.mark.parametrize("seed", range(6))
def test_pool_index_model_gives_the_host_pool_order(seed):
    """Chunks of id-tagged rows with random keep masks, then draws as _iterate_batches_native schedules them (while
    n >= S + B, then the drain): every batch and every pool state equal _RowPool's."""
    rng = np.random.default_rng(seed)
    B, S = int(rng.integers(1, 40)), int(rng.integers(1, 120))
    host, dev = _RowPool(), _IdPool()
    r_host, r_dev = np.random.default_rng(seed + 100), np.random.default_rng(seed + 100)
    next_id = 0
    batches = 0

    def draw(b):
        n = host.n
        got = host.take(b, r_host)[0]                     # the id column of the src matrix
        pick = r_dev.choice(n, size=b, replace=False) if b < n else r_dev.permutation(n)
        assert np.array_equal(dev.take(pick, 0, b), got[:, 0])
        assert np.array_equal(dev.rows, host.arrays[0][:host.n, 0])
    for _ in range(int(rng.integers(3, 9))):
        k = int(rng.integers(0, 200))
        ids = np.arange(next_id, next_id + k)
        next_id += k
        keep = rng.random(k) < rng.choice([0.0, 0.3, 0.8, 1.0])
        host.reserve(k, 1)
        host.arrays[0][host.n:host.n + k, 0] = ids
        host.commit(k, keep.astype(np.uint8))
        dev.commit(ids, keep)
        assert np.array_equal(dev.rows, host.arrays[0][:host.n, 0])
        while host.n >= S + B:
            draw(B)
            batches += 1
    while host.n > 0:
        draw(min(B, host.n))
        batches += 1
    assert len(dev.rows) == 0


def test_commit_model_is_not_a_stable_compaction():
    """Hole j takes mover j: with keep = [0, 1, 0, 1, 1] the kept rows end up in the order 3, 1, 4 (a stable compaction
    would give 1, 3, 4)."""
    kept, holes, movers = _commit_moves([0, 1, 0, 1, 1])
    rows = np.arange(5)
    rows[holes] = rows[movers]
    assert kept == 3 and list(rows[:kept]) == [3, 1, 4]


# ---- the switch --------------------------------------------------------------------------------------------------------
def test_device_reader_flag():
    from code2vec_b200.device_reader import device_reader_flag
    assert device_reader_flag({}) is False
    assert device_reader_flag({"C2V_DEVICE_READER": "0"}) is False
    assert device_reader_flag({"C2V_DEVICE_READER": ""}) is False
    assert device_reader_flag({"C2V_DEVICE_READER": "1"}) is True
    for bad in ("2", "yes", "true", " 1"):
        with pytest.raises(ValueError, match="C2V_DEVICE_READER"):
            device_reader_flag({"C2V_DEVICE_READER": bad})


def test_keras_backend_refuses_the_device_reader(monkeypatch):
    from code2vec_b200.b200_keras_model import Code2VecModel
    from code2vec_b200.config import Config
    cfg = Config(set_defaults=True)
    cfg.DL_FRAMEWORK = "b200-keras"
    cfg.VERBOSE_MODE = 0
    monkeypatch.setenv("C2V_DEVICE_READER", "1")
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    with pytest.raises(ValueError, match="C2V_DEVICE_READER"):
        Code2VecModel(cfg)
    monkeypatch.setenv("C2V_DEVICE_READER", "3")
    with pytest.raises(ValueError, match="C2V_DEVICE_READER must be 0 or 1"):
        Code2VecModel(cfg)
