"""The device reader's kernels (csrc/reader.cu) called through their C ABI on one reader handle, against the host
statements they reproduce, bit for bit, on inputs built to reach their warp, tile and block edges
(tests/test_reader_edges_model.py shows the inputs reach them):
  a. parse + commit (c2v_reader_parse_chunk) against c2v_parse_chunk's rows committed by _commit_moves, and its error
     against the host parser's lowest (line, kind);
  b. the sharded path (c2v_reader_parse_share, c2v_reader_commit_shares) on shares cut by share_range, against the same
     pool, and chunk_error against the host parser's verdict;
  c. draws (c2v_reader_draw) of 1 to 4097 rows from pools of 3,000-20,000 rows against _IdPool;
  d. the evaluation queue (c2v_reader_eval_append / _eval_take) against c2v_parse_chunk in evaluate mode, in file order;
  e. the metric kernel (c2v_reader_eval_score) against score_row and the host metrics, for k up to 100."""
import ctypes

import numpy as np
import pytest

from code2vec_b200.path_context_reader import share_range
from tests.test_device_eval_model import _host, score_row
from tests.test_device_reader_model import _commit_moves, _IdPool
from tests.test_reader_edges_model import (TILE, EdgeText, HostTables, _target_word, edge_chunk, host_parse,
                                           malformed_chunk, metric_rows, metric_vocab, parse_chunks)

pytestmark = pytest.mark.gpu

INT64_MIN = np.iinfo(np.int64).min


class _Handle:
    """A reader handle on cuda:0 over HostTables' vocabularies (uploaded as DeviceVocabs), called on torch buffers."""

    def __init__(self, H, C):
        import torch
        from code2vec_b200.device_reader import DeviceVocabs
        from code2vec_b200.engine import load_library

        class _Native:                                  # what DeviceVocabs reads from a reader
            _native = (H.lib, *H.native)
        self.torch, self.H, self.C = torch, H, C
        self.lib = load_library()
        self.vocabs = DeviceVocabs(_Native(), torch.device("cuda", 0))
        s = self.vocabs.structs
        h = ctypes.c_void_p()
        self._ok(self.lib.c2v_reader_create(C, ctypes.byref(s[0]), ctypes.byref(s[1]), ctypes.byref(s[2]), 0,
                                            ctypes.byref(h)))
        self.h = h
        self.stream = torch.cuda.Stream()

    def _ok(self, rc):
        assert rc == 0, self.lib.c2v_last_error(None).decode()

    def close(self):
        self.torch.cuda.synchronize()
        self.lib.c2v_reader_destroy(self.h)

    def sync(self):
        self.stream.synchronize()

    def dev(self, arr):
        t = self.torch.from_numpy(np.ascontiguousarray(arr)).cuda()
        self.torch.cuda.synchronize()
        return t

    def text(self, text: bytes):
        return self.dev(np.frombuffer(text, dtype=np.uint8).copy()) if text else None

    def parse_chunk(self, text: bytes):
        """(rc, kept, bad_line, bad_kind)."""
        t = self.text(text)
        kept, line, kind = ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int32()
        rc = self.lib.c2v_reader_parse_chunk(self.h, t.data_ptr(), len(text), ctypes.byref(kept), ctypes.byref(line),
                                             ctypes.byref(kind), self.stream.cuda_stream)
        self.sync()
        return rc, kept.value, line.value, kind.value

    def live(self) -> int:
        return int(self.lib.c2v_reader_live_rows(self.h))

    def rows(self, n):
        torch = self.torch
        n = max(n, 1)
        return (torch.full((n, self.C), -7, dtype=torch.int32, device="cuda"),
                torch.full((n, self.C), -7, dtype=torch.int32, device="cuda"),
                torch.full((n, self.C), -7, dtype=torch.int32, device="cuda"),
                torch.full((n, self.C), -7.0, dtype=torch.float32, device="cuda"),
                torch.full((n,), -7, dtype=torch.int32, device="cuda"))

    def draw(self, pick, lo, hi):
        """c2v_reader_draw of `pick`: the gathered rows [lo, hi) as numpy arrays."""
        pick = np.ascontiguousarray(pick, dtype=np.int64)
        out = self.rows(hi - lo)
        self.torch.cuda.synchronize()
        self._ok(self.lib.c2v_reader_draw(self.h, pick.ctypes.data, len(pick), lo, hi, *(t.data_ptr() for t in out),
                                          self.stream.cuda_stream))
        self.sync()
        return tuple(t[:hi - lo].cpu().numpy() for t in out)

    def drain(self):
        """The whole pool, read out by drawing pick = arange(live)."""
        n = self.live()
        return self.draw(np.arange(n), 0, n) if n else None


def _bits(a):
    return a.view(np.int32) if a.dtype == np.float32 else a


def _assert_rows(got, want, what=""):
    for name, g, w in zip(("src", "path", "dst", "mask", "target"), got, want):
        assert g.shape == w.shape, (what, name, g.shape, w.shape)
        bad = np.flatnonzero((_bits(g) != _bits(w)).reshape(len(g), -1).any(axis=1)) if len(g) else []
        assert len(bad) == 0, (what, name, "rows", list(bad[:10]))


def _committed(rows, keep):
    """The pool rows one chunk adds: _RowPool.commit's order, stated by _commit_moves."""
    kept, holes, movers = _commit_moves(keep)
    new = tuple(a.copy() for a in rows)
    for a in new:
        a[holes] = a[movers]
    return tuple(a[:kept] for a in new)


def _cat(parts):
    return tuple(np.concatenate(c) for c in zip(*parts))


def _verdict(H, text, C):
    """The host parser's verdict on a chunk: None, (None, 3), or (line, kind) of its lowest malformed line."""
    n, err, *_ = host_parse(H, text, C)
    if n >= 0:
        return None
    return (None, 3) if n == INT64_MIN else (-n - 1, err)


_TABLES = {}


def _tables(separate):
    if separate not in _TABLES:
        _TABLES[separate] = HostTables(separate)
    return _TABLES[separate]


# ---- a. parse and commit -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("separate", [False, True])
@pytest.mark.parametrize("C", [1, 13, 31, 32, 33, 200])
def test_parse_and_commit_equal_the_host(C, separate):
    H = _tables(separate)
    r = _Handle(H, C)
    try:
        want = []
        for text, _ in parse_chunks(C, H.vocabs):       # test_reader_edges_model shows what these chunks hold
            n, err, rows, keep, _, _ = host_parse(H, text, C)
            assert n > 0, (n, err)
            rc, kept, line, kind = r.parse_chunk(text)
            assert (rc, kept, line, kind) == (0, int(keep.sum()), -1, 0)
            want.append(_committed(rows, keep))
        want = _cat(want)
        assert r.live() == len(want[4])
        _assert_rows(r.drain(), want)
    finally:
        r.close()


@pytest.mark.parametrize("C", [1, 13, 33, 200])
@pytest.mark.parametrize("case", ["lane0_ctx", "lane31_ctx", "lane0_beyond", "lane31_beyond", "fields", "kind3"])
def test_malformed_chunk_reports_the_hosts_lowest_line(C, case):
    if C == 1 and case == "kind3":
        pytest.skip("with one context no chunk has more records than well-formed lines")
    H = _tables(False)
    text, _ = malformed_chunk(C, H.vocabs, 7, case)
    want = _verdict(H, text, C)
    r = _Handle(H, C)
    try:
        rc, kept, line, kind = r.parse_chunk(text)
        assert rc != 0 and kept == 0 and r.live() == 0
        assert (kind, line if kind != 3 else None) == (want[1], want[0])
    finally:
        r.close()


def test_third_comma_beyond_the_contexts_is_a_field_count_error():
    """A 4-part field after the C contexts: the host counts it as a field (kind 1), not a context (kind 2)."""
    H = _tables(False)
    for lane in (0, 31):
        t = EdgeText(13, H.vocabs, lane)
        t.record()
        t.bad_record(lane, beyond=True)
        r = _Handle(H, 13)
        try:
            assert r.parse_chunk(t.text())[2:] == (1, 1) == _verdict(H, t.text(), 13)
        finally:
            r.close()


# ---- b. the sharded path -----------------------------------------------------------------------------------------------
def _share_text(C, H, case):
    t = EdgeText(C, H.vocabs, 3)
    if case == "edges":
        return edge_chunk(C, H.vocabs, 5, edge=0)[0]
    if case == "tile_cut":                              # W = 2 cuts at byte 8192, a record start
        t.pad_to(2 * TILE)
        for _ in range(20):
            t.record()
        t.pad_to(4 * TILE)
    elif case == "blank_cut":                           # W = 2 cuts just after a blank line
        t.pad_to(2 * TILE - 1)
        t.buf += b"\n"
        for _ in range(20):
            t.record()
        t.pad_to(4 * TILE)
    elif case == "one_record":                          # one record a share
        for _ in range(8):
            t.filler(C + 300)
    elif case == "long_record":                         # a 5000-byte record swallows the shares around it
        t.record()
        t.long_record()
        t.record()
    elif case in ("lane0_ctx", "lane31_beyond", "kind3"):
        return malformed_chunk(C, H.vocabs, 11, case)[0]
    return t.text()


@pytest.mark.parametrize("world", [2, 3, 8])
@pytest.mark.parametrize("case", ["edges", "tile_cut", "blank_cut", "one_record", "long_record", "lane0_ctx",
                                  "lane31_beyond", "kind3"])
def test_shares_commit_the_whole_chunks_pool(tmp_path, world, case):
    from code2vec_b200.device_reader import chunk_error
    from code2vec_b200.engine import c2v_reader_share_status
    C = 13
    H = _tables(True)
    text = _share_text(C, H, case)
    path = tmp_path / "chunk.c2v"
    path.write_bytes(text)
    with open(path, "rb") as f:
        cuts = [share_range(f.fileno(), 0, len(text), world, r) for r in range(world)]
    if case == "tile_cut" and world == 2:
        assert cuts[0][1] == 2 * TILE
    if case == "blank_cut" and world == 2:
        assert cuts[0][1] == 2 * TILE and text[2 * TILE - 2:2 * TILE] == b"\n\n"
    if case == "one_record" and world == 8:
        assert all(text[s0:s1].count(b"\n") == 1 for s0, s1 in cuts)
    if case == "long_record" and world == 8:
        assert sum(s0 == s1 for s0, s1 in cuts) > 0
    r = _Handle(H, C)
    try:
        stages, statuses = [], []
        for s0, s1 in cuts:
            part = r.text(text[s0:s1])
            rows = (s1 - s0) // (C + 1) + 1
            stage = r.torch.zeros(int(r.lib.c2v_reader_stage_bytes(C, rows)), dtype=r.torch.uint8, device="cuda")
            r.torch.cuda.synchronize()
            st = c2v_reader_share_status()
            r._ok(r.lib.c2v_reader_parse_share(r.h, part.data_ptr() if part is not None else None, s1 - s0, len(text),
                                               stage.data_ptr(), rows, ctypes.byref(st), r.stream.cuda_stream))
            stages.append(stage)
            statuses.append(st)
        assert chunk_error(statuses, len(text), C) == _verdict(H, text, C)
        if _verdict(H, text, C) is not None:
            return
        n, err, host_rows, keep, _, _ = host_parse(H, text, C)
        ptrs = (ctypes.c_void_p * world)(*[s.data_ptr() for s in stages])
        recs = (ctypes.c_int64 * world)(*[s.records for s in statuses])
        kept = ctypes.c_int64()
        r._ok(r.lib.c2v_reader_commit_shares(r.h, ptrs, recs, world, ctypes.byref(kept), r.stream.cuda_stream))
        r.sync()
        assert sum(s.records for s in statuses) == n and kept.value == int(keep.sum())
        assert kept.value > 0
        _assert_rows(r.drain(), _committed(host_rows, keep))
    finally:
        r.close()


# ---- c. draws ----------------------------------------------------------------------------------------------------------
def _keep_chunk(H, C, rng, kept, records):
    """A chunk of `records` records of which exactly `kept` pass the training filter: dropped records (an OOV target)
    below the kept count and kept ones beyond it, spread over every 1024-row tile."""
    moves = min(kept, records - kept, 300)
    keep = np.zeros(records, dtype=bool)
    keep[:kept] = True
    keep[rng.choice(kept, moves, replace=False)] = False
    keep[kept + rng.choice(records - kept, moves, replace=False)] = True
    tok = H.vocabs[0].words[2:]
    lines = []
    for k in keep:
        ctx = ["%s,1,%s" % (tok[int(rng.integers(len(tok)))], tok[int(rng.integers(len(tok)))]) for _ in range(C)]
        lines.append(" ".join([_target_word(int(rng.integers(1, 96))) if k else "unknown"] + ctx))
    text = ("\n".join(lines) + "\n").encode()
    assert np.array_equal(host_parse(H, text, C)[3].astype(bool), keep)
    return text


@pytest.mark.parametrize("seed", [0, 1])
def test_draws_equal_the_id_pool(seed):
    C = 3
    H = _tables(True)
    rng = np.random.default_rng(seed)
    r = _Handle(H, C)
    try:
        pool = _IdPool()
        host_rows = []
        next_id = 0

        def add(kept, records):
            nonlocal next_id
            text = _keep_chunk(H, C, rng, kept, records)
            n, err, rows, keep, _, _ = host_parse(H, text, C)
            assert n == records
            rc, got_kept, _, _ = r.parse_chunk(text)
            assert rc == 0 and got_kept == int(keep.sum())
            host_rows.append(rows)
            pool.commit(np.arange(next_id, next_id + n), keep.astype(bool))
            next_id += n
            return int(keep.sum())

        sizes = [1, 31, 1023, 1024, 1025, 2048, 4097]
        slices = [lambda b: (0, b), lambda b: (0, 0), lambda b: (b // 3, b - b // 4), lambda b: (b, b)]
        step = [0]

        def draw():
            all_rows = _cat(host_rows)
            n = r.live()
            assert n == len(pool.rows)
            i = step[0]
            step[0] += 1
            b = min(sizes[i % len(sizes)], n)
            mode = i % 3
            if mode == 0:                                   # every pick in the tail [n - b, n)
                pick = n - b + rng.permutation(b)
            elif mode == 1 and 2 * b <= n:                  # none in the tail
                pick = rng.choice(n - b, b, replace=False)
            else:
                pick = rng.choice(n, b, replace=False)
            lo, hi = slices[i % len(slices)](b)
            got = r.draw(pick, lo, hi)
            ids = pool.take(pick, lo, hi)
            _assert_rows(got, tuple(a[ids] for a in all_rows), ("draw", i, b, mode, lo, hi))

        kept = [add(k, rec) for k, rec in [(2047, 2600), (2048, 3100), (2049, 2500)]]
        assert sum(kept) == 6144
        for _ in range(5):
            draw()
        for k, rec in [(3072, 4000), (1023, 2000), (4097, 4600), (1025, 1400)]:
            add(k, rec)
        assert r.live() > 10000
        while r.live() > 0:
            draw()
        assert step[0] >= 2 * len(sizes) and len(pool.rows) == 0
    finally:
        r.close()


# ---- d. the evaluation queue -------------------------------------------------------------------------------------------
def _eval_chunk(rng, C, tok, j):
    """Chunk j of a test file: names of 0-400 bytes (0: the OOV word), rows without a valid context, blank lines.
    Chunk 0 is the largest, so the reader's per-chunk scratch reaches its size there."""
    lines = []
    for i in range(100 if j == 0 else int(rng.integers(5, 40))):
        L = 400 if j == 0 else [0, 1, 31, 32, 33, 64, 400, int(rng.integers(1, 401))][int(rng.integers(0, 8))]
        name = ("Nm|%d_" % (j + i) + "getValue|" * 50)[:L]
        ctx = ["%s,1,%s" % (tok[int(rng.integers(len(tok)))], tok[int(rng.integers(len(tok)))])
               if rng.random() < 0.6 else "" for _ in range(C)]
        if rng.random() < 0.1:
            ctx = [""] * C                              # no valid context: not queued
        lines.append(" ".join([name] + ctx))
        if rng.random() < 0.05:
            lines.append("")
    return ("\n".join(lines) + "\n").encode()


@pytest.mark.parametrize("schedule", ["keep_up", "lag"])
def test_evaluation_queue_equals_the_hosts_batches(schedule):
    from code2vec_b200.device_reader import eval_tables
    from tests.test_device_eval_model import _Vocab
    C = 5
    H = _tables(True)
    tv = H.vocabs[2]
    w, w_off, nm, n_off, legal = eval_tables(_Vocab(tv.words, tv.special))
    oov_word = tv.words[0].encode()
    r = _Handle(H, C)
    r._ok(r.lib.c2v_reader_eval_tables(r.h, int(legal.size), w.ctypes.data, w_off.ctypes.data, nm.ctypes.data,
                                       n_off.ctypes.data, legal.ctypes.data, r.stream.cuda_stream))
    rng = np.random.default_rng(3)
    tok = [x for x in H.vocabs[0].words[2:] if len(x.encode()) <= 8]
    queue = []                                          # (row arrays, name) in file order, from the host parser
    name_cap = [0]
    # keeping up, the queue holds fewer rows than one take; lagging, takes of up to 1024 rows cross many appends
    sizes, k = ([1, 7, 33] if schedule == "keep_up" else [1, 7, 33, 1024]), [0]
    grew_with_rows = []
    mem = []
    # the queue as c2v_reader_eval_append sees it: the name lengths of the rows from its front, and how many were taken;
    # an append compacts when the rows left are fewer than the rows taken and their names fit in the taken ones' bytes
    front = {"names": [], "taken": 0, "compactions": 0}

    def append(j):
        text = _eval_chunk(rng, C, tok, j)
        n, err, rows, keep, toff, tlen = host_parse(H, text, C, mode=1)
        assert n > 0
        for i in np.flatnonzero(keep):
            queue.append((tuple(a[i] for a in rows), text[toff[i]:toff[i] + tlen[i]] if tlen[i] else oov_word))
        left, taken = len(front["names"]) - front["taken"], front["taken"]
        if left == 0:
            front["names"], front["taken"] = [], 0
        elif 0 < taken and left < taken and sum(front["names"][taken:]) <= sum(front["names"][:taken]):
            front["names"], front["taken"] = front["names"][taken:], 0
            front["compactions"] += 1
        front["names"] += [len(q[1]) for q in queue[len(queue) - int(keep.sum()):]]
        before = int(r.lib.c2v_reader_device_bytes(r.h))
        queued = int(r.lib.c2v_reader_eval_queued(r.h))
        t = r.text(text)
        app, nb, line, kind = ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int32()
        r._ok(r.lib.c2v_reader_eval_append(r.h, t.data_ptr(), len(text), ctypes.byref(app), ctypes.byref(nb),
                                           ctypes.byref(line), ctypes.byref(kind), r.stream.cuda_stream))
        r.sync()
        assert app.value == int(keep.sum()) and r.lib.c2v_reader_eval_queued(r.h) == len(queue)
        name_cap[0] = nb.value
        after = int(r.lib.c2v_reader_device_bytes(r.h))
        if after > before and queued > 0:
            grew_with_rows.append(j)
        mem.append(after)

    def take(b):
        torch = r.torch
        out = r.rows(b)
        off = torch.full((b + 1,), -1, dtype=torch.int64, device="cuda")
        names = torch.zeros(max(name_cap[0], 1), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        r._ok(r.lib.c2v_reader_eval_take(r.h, b, *(x.data_ptr() for x in out), off.data_ptr(), names.data_ptr(),
                                         names.numel(), r.stream.cuda_stream))
        r.sync()
        want = queue[:b]
        del queue[:b]
        front["taken"] += b
        _assert_rows(tuple(x.cpu().numpy() for x in out), tuple(np.stack(c) for c in zip(*[w for w, _ in want])),
                     ("take", b))
        lens = [len(n) for _, n in want]
        o = off.cpu().numpy()
        assert list(o) == [0] + list(np.cumsum(lens)), ("name_off", b)
        assert names[:o[-1]].cpu().numpy().tobytes() == b"".join(n for _, n in want)

    try:
        for j in range(200):
            append(j)
            if schedule == "lag" and j % 25 != 24:
                continue
            while len(queue) >= sizes[k[0] % len(sizes)]:
                take(sizes[k[0] % len(sizes)])
                k[0] += 1
        while queue:
            take(min(sizes[k[0] % len(sizes)], len(queue)))
            k[0] += 1
        assert k[0] > (200 if schedule == "keep_up" else 12)
        if schedule == "keep_up":
            assert front["compactions"] > 20            # eval_compact_kernel ran, and its moves were read back
            assert mem[5] == mem[-1]                    # bounded: the taken rows are compacted away
        else:
            assert grew_with_rows                       # the queue grew with rows in it
    finally:
        r.close()


# ---- e. the metric kernel ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 2, 10, 31, 32, 33, 63, 64, 100])
@pytest.mark.parametrize("n", [1, 7, 8, 9, "two_passes"])
def test_metric_kernel_equals_score_row_and_the_host(k, n):
    import torch
    from code2vec_b200.device_reader import eval_tables
    if n == "two_passes":                               # row_grid: at most num_sms * 8 blocks of 8 rows, one warp a row
        n = torch.cuda.get_device_properties(0).multi_processor_count * 64 + 9
    v = metric_vocab()
    tables = eval_tables(v)
    H = _tables(True)
    r = _Handle(H, 4)
    try:
        w, w_off, nm, n_off, legal = tables
        r._ok(r.lib.c2v_reader_eval_tables(r.h, int(legal.size), w.ctypes.data, w_off.ctypes.data, nm.ctypes.data,
                                           n_off.ctypes.data, legal.ctypes.data, r.stream.cuda_stream))
        rows = metric_rows(v, k, n, seed=k * 1000 + n)
        ids = np.array([i for _, i in rows], dtype=np.int32).reshape(n, k)
        names = [name for name, _ in rows]
        off = np.zeros(n + 1, dtype=np.int64)
        off[1:] = np.cumsum([len(x) for x in names])
        blob = np.frombuffer(b"".join(names) or b"\0", dtype=np.uint8).copy()
        d_ids, d_off, d_names = r.dev(ids), r.dev(off), r.dev(blob)
        torch = r.torch
        res = torch.full((3, n), -9, dtype=torch.int32, device="cuda")
        acc = torch.full((k + 4,), -9, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        r._ok(r.lib.c2v_reader_eval_score(r.h, d_ids.data_ptr(), n, k, d_off.data_ptr(), d_names.data_ptr(),
                                          res[0].data_ptr(), res[1].data_ptr(), res[2].data_ptr(), acc.data_ptr(),
                                          r.stream.cuda_stream))
        r.sync()
        rank, first, flags = res.cpu().numpy()
        acc = acc.cpu().numpy()
        hist, sums = np.zeros(k, dtype=np.int64), np.zeros(4, dtype=np.int64)
        for i, (name, row) in enumerate(rows):
            want = score_row(name, row, tables)
            assert (rank[i], first[i], flags[i]) == want[:3], (i, name, row)
            if want[2]:
                continue
            if want[0] >= 0:
                hist[want[0]] += 1
            sums += (1,) + want[3]
            if i < 1500:
                found, counts = _host(name.decode(), row, v)
                assert (found is None) == (want[0] < 0) and (found is None or found[0] == want[0])
                assert counts == want[3]
        assert np.array_equal(acc, np.concatenate([hist, sums])), (acc, hist, sums)
        if n > 9:
            assert sums[0] > 0 and (flags == 1).any() and (flags == 2).any()
    finally:
        r.close()
