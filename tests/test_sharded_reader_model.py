"""Host-side statements of the sharded device reader (C2V_SHARDED_READER=1, code2vec_b200/device_reader.py), checked
without a GPU:
  * chunk_ranges cuts a file exactly where the chunker it replaced did (a verbatim copy of it is kept below);
  * share_range cuts a chunk into whole-line shares, in rank order, that cover it;
  * "every stage in rank order behind the live end, then the commit of the whole chunk" builds _RowPool's pool;
  * the chunk error decided from the share statuses is the host parser's (line, kind) for the whole chunk;
  * C2V_SHARDED_READER is 0 or 1 and needs C2V_DEVICE_READER=1."""
import ctypes as C
import os

import numpy as np
import pytest

from code2vec_b200.path_context_reader import (PathContextReader, _Chunk, _RowPool, chunk_ranges, load_native_tensoriser,
                                               share_range)
from tests.test_device_reader_model import _IdPool


def _reference_chunks(path, chunk_bytes):
    """The chunker the native path used before chunk_ranges (one pass), verbatim but for yielding (start, end)."""
    with open(path, "rb") as f:
        size = chunk_bytes
        while True:
            start = f.tell()
            buf = f.read(size)
            if not buf:
                break
            at_eof = len(buf) < size
            cut = buf.rfind(b"\n")
            if cut < 0:
                if at_eof:
                    if buf.strip(b"\r\n"):
                        yield start, start + len(buf)
                    break
                f.seek(start)                # a line longer than the chunk: retry with a bigger one
                size *= 2
                continue
            if at_eof:
                yield start, start + len(buf)  # includes a last line without a trailing newline
                break
            f.seek(start + cut + 1)          # re-read the partial last line with the next chunk
            yield start, start + cut + 1


def _ranges(path, chunk_bytes):
    with open(path, "rb") as f:
        return list(chunk_ranges(f.fileno(), chunk_bytes))


def _random_text(rng, n_lines, max_len, crlf=False, blanks=False):
    out = []
    for _ in range(n_lines):
        n = int(rng.integers(0, max_len))
        out.append(bytes(rng.choice(np.frombuffer(b"abc ,xyz|", dtype=np.uint8), size=n)))
        out.append(b"\r\n" if crlf and rng.random() < 0.5 else b"\n")
        if blanks and rng.random() < 0.2:
            out.append(b"\n" * int(rng.integers(1, 4)))
    return b"".join(out)


SPECIAL = {
    "long_lines": b"short\n" + b"y" * 5000 + b"\n" + b"z" * 300 + b"\nq\n" + b"w" * 9000,
    "exact_chunks": b"abcdefg\n" * 64,                      # 512 bytes: exactly 8 chunks of 64, and 2 of 256
    "no_trailing_newline": b"one line\nanother one\nlast without newline",
    "crlf": b"a b c\r\nd e f\r\n\r\ng h\r\n",
    "blank_lines": b"\n\n\nline one\n\n\n\nline two\n\n",
    "cr_tail": b"line one\nline two\n\r\r\r",
    "cr_only": b"\r\r\r\r",
    "newline_tail": b"line\n\n\n",
    "empty": b"",
    "one_newline": b"\n",
}


@pytest.mark.parametrize("case", sorted(SPECIAL))
@pytest.mark.parametrize("chunk", [1, 3, 64, 256, 4096])
def test_chunk_ranges_cut_where_the_old_chunker_cut_special_files(tmp_path, case, chunk):
    path = str(tmp_path / "f.c2v")
    with open(path, "wb") as f:
        f.write(SPECIAL[case])
    assert _ranges(path, chunk) == list(_reference_chunks(path, chunk))


@pytest.mark.parametrize("seed", range(12))
def test_chunk_ranges_cut_where_the_old_chunker_cut_random_files(tmp_path, seed):
    rng = np.random.default_rng(seed)
    path = str(tmp_path / "f.c2v")
    text = _random_text(rng, int(rng.integers(1, 400)), int(rng.choice([20, 300, 3000])), crlf=seed % 2 == 1,
                        blanks=seed % 3 == 0)
    if seed % 4 == 2:
        text = text.rstrip(b"\n")
    if seed % 4 == 3:
        text += b"\r" * int(rng.integers(1, 5))
    with open(path, "wb") as f:
        f.write(text)
    for chunk in (64, 100, 1000, 4096, 65536, int(rng.integers(64, 65536))):
        assert _ranges(path, chunk) == list(_reference_chunks(path, chunk)), chunk


def test_native_chunks_read_the_ranges(tmp_path):
    path = str(tmp_path / "f.c2v")
    text = _random_text(np.random.default_rng(3), 300, 200)
    with open(path, "wb") as f:
        f.write(text)

    class _Reader:
        def _native_chunk_ranges(self):
            with open(path, "rb") as f:
                for a, b in chunk_ranges(f.fileno(), 512):
                    yield f.fileno(), a, b
    got = list(PathContextReader._native_chunks(_Reader()))
    assert all(isinstance(c, _Chunk) and c.n == len(c.buf) for c in got)
    assert [bytes(c.buf) for c in got] == [text[a:b] for a, b in _reference_chunks(path, 512)]
    assert b"".join(bytes(c.buf) for c in got) == text


# ---- shares ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("seed", range(4))
def test_shares_are_whole_lines_in_order_covering_the_chunk(tmp_path, world, seed):
    rng = np.random.default_rng(seed)
    path = str(tmp_path / "f.c2v")
    text = _random_text(rng, 200, [30, 400, 3000, 12000][seed], crlf=True, blanks=True)
    with open(path, "wb") as f:
        f.write(text)
    empty = 0
    with open(path, "rb") as f:
        fd = f.fileno()
        for a, b in chunk_ranges(fd, 2048):
            shares = [share_range(fd, a, b, world, r) for r in range(world)]
            assert shares[0][0] == a and shares[-1][1] == b
            for (s0, s1), (t0, _) in zip(shares, shares[1:]):
                assert s1 == t0
            for r, (s0, s1) in enumerate(shares):
                assert a <= s0 <= s1 <= b
                assert s0 == a or text[s0 - 1:s0] == b"\n"                 # a share starts at a line start
                t = a + r * (b - a) // world
                assert s0 >= t
                if t > a:
                    assert b"\n" not in text[t - 1:s0 - 1]                  # the first line start at or after t
                empty += s0 == s1
    if world > 1 and seed >= 2:
        assert empty > 0                           # lines longer than a share leave shares empty


def test_a_line_longer_than_a_share_empties_the_shares_it_spans(tmp_path):
    path = str(tmp_path / "f.c2v")
    text = b"a\n" + b"x" * 1000 + b"\nb\n"
    with open(path, "wb") as f:
        f.write(text)
    with open(path, "rb") as f:
        shares = [share_range(f.fileno(), 0, len(text), 8, r) for r in range(8)]
    # the split points of ranks 1..7 (125, 251, ..., 880) all fall inside the long line: rank 0 holds "a\n" and the
    # long line, ranks 1..6 nothing, rank 7 "b\n"
    assert shares == [(0, 1003)] + [(1003, 1003)] * 6 + [(1003, len(text))]


# ---- assembly ----------------------------------------------------------------------------------------------------------
def _assemble(pool, stages, records):
    """assemble_shares_kernel then the commit: stages[r] (a dict by rank, as the exchange delivers them) holds a stage
    of `rows` rows, of which records[r] are share r's; share r lands at row0 = the records of the ranks below r, and
    only its records are copied (the rows beyond them are stale, here -1)."""
    total = int(sum(records))
    ids, keep = np.full(total, -2, dtype=np.int64), np.zeros(total, dtype=bool)
    row0 = np.concatenate([[0], np.cumsum(records)])
    for r in range(len(records)):
        st_ids, st_keep = stages[r]
        n = int(records[r])
        ids[row0[r]:row0[r] + n] = st_ids[:n]
        keep[row0[r]:row0[r] + n] = st_keep[:n]
    assert (ids >= 0).all()                          # every row of the chunk was written once
    pool.commit(ids, keep)


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("seed", range(4))
def test_assembled_stages_commit_to_the_host_pool(world, seed):
    rng = np.random.default_rng(seed)
    host, dev = _RowPool(), _IdPool()
    next_id = 0
    for _ in range(6):
        k = int(rng.integers(0, 300))
        ids = np.arange(next_id, next_id + k)
        next_id += k
        keep = rng.random(k) < rng.choice([0.0, 0.4, 0.9, 1.0])
        cuts = np.sort(rng.integers(0, k + 1, size=world - 1))        # shares of any size, empty ones included
        bounds = [0] + list(cuts) + [k]
        records = [hi - lo for lo, hi in zip(bounds, bounds[1:])]
        stages = {}
        for r in rng.permutation(world):                              # stages arrive in any order, with stale rows
            lo, hi = bounds[r], bounds[r + 1]
            rows = hi - lo + int(rng.integers(1, 20))
            st_ids, st_keep = np.full(rows, -1, dtype=np.int64), rng.random(rows) < 0.5
            st_ids[:hi - lo], st_keep[:hi - lo] = ids[lo:hi], keep[lo:hi]
            stages[int(r)] = (st_ids, st_keep)
        host.reserve(k, 1)
        host.arrays[0][host.n:host.n + k, 0] = ids
        host.commit(k, keep.astype(np.uint8))
        _assemble(dev, stages, records)
        assert np.array_equal(dev.rows, host.arrays[0][:host.n, 0])
        if host.n > 40:                                                   # a draw between chunks
            pick = np.random.default_rng(seed).choice(host.n, size=17, replace=False)
            host.take(17, np.random.default_rng(seed))
            dev.take(pick, 0, 17)
            assert np.array_equal(dev.rows, host.arrays[0][:host.n, 0])


# ---- the chunk's error from the share statuses ---------------------------------------------------------------------------
needs_native = pytest.mark.skipif(load_native_tensoriser() is None, reason="g++ build of the native tensoriser failed")


class _Status:
    def __init__(self, records, newlines, bad_line, bad_kind, overflow):
        self.records, self.newlines, self.bad_line, self.bad_kind, self.overflow = records, newlines, bad_line, bad_kind, overflow


def _host_parse(reader, data: bytes, cap: int):
    """(line, kind) of the lowest malformed line of `data` by the host parser with room for `cap` records (one thread),
    (None, 3) when it has more records than that, None when it is clean."""
    lib, tok, pth, tgt = reader._native
    Cn = reader.config.MAX_CONTEXTS
    cap = max(cap, 1)
    bufs = [np.empty((cap, Cn), dtype=np.int32) for _ in range(3)] + [np.empty((cap, Cn), dtype=np.float32)]
    target, keep = np.empty(cap, dtype=np.int32), np.zeros(cap, dtype=np.uint8)
    toff, tlen = np.empty(cap, dtype=np.int64), np.empty(cap, dtype=np.int32)
    err = C.c_int32(0)
    n = lib.c2v_parse_chunk(data, len(data), Cn, tok.h, pth.h, tgt.h, 0, 1, cap, *(b.ctypes.data for b in bufs),
                            target.ctypes.data, keep.ctypes.data, toff.ctypes.data, tlen.ctypes.data, C.byref(err))
    if n >= 0:
        return None
    if n == -(1 << 63):
        return None, 3
    return -n - 1, err.value


def _records(data: bytes) -> int:
    return sum(1 for p in range(len(data)) if (p == 0 or data[p - 1] == 10) and data[p] != 10)


def _share_status(reader, share: bytes, chunk_bytes: int):
    """What c2v_reader_parse_share reports for a share, stated with the host parser: its records and newlines, and its
    lowest malformed line, found with room for every record when the share overflows its stage."""
    Cn = reader.config.MAX_CONTEXTS
    recs = _records(share)
    rows = len(share) // (Cn + 1) + 1
    overflow = recs > rows
    line, kind = None, 0
    if not overflow or recs <= chunk_bytes // (Cn + 1) + 1:
        got = _host_parse(reader, share, max(rows, recs))
        if got is not None:
            line, kind = got
    return _Status(recs, share.count(b"\n"), -1 if line is None else line, kind, int(overflow))


def _bad_lines(C, kind, seed):
    from tests.test_reader_native import _random_lines
    lines = _random_lines(60, C, seed=seed)
    rng = np.random.default_rng(seed)
    if kind in ("fields", "mixed"):
        for i in rng.choice(60, size=3, replace=False):
            lines[i] = lines[i] + " extra"
    if kind in ("parts", "mixed"):
        for i in rng.choice(60, size=2, replace=False):
            lines[i] = " ".join(["name|1", "a,b,c,d"] + [""] * (C - 1))
    if kind == "short":
        at = int(rng.integers(0, 60))
        lines = lines[:at] + ["x"] * 120 + lines[at:]             # a run of short lines: some share overflows
    if kind == "very_short":
        lines = lines[:2] + ["x"] * 400                            # more records than the chunk holds: kind 3
    return lines


@needs_native
@pytest.mark.parametrize("kind", ["clean", "fields", "parts", "mixed", "short", "very_short"])
@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("seed", range(3))
def test_chunk_error_from_share_statuses_is_the_host_error(tmp_path, kind, world, seed):
    from code2vec_b200.device_reader import chunk_error
    from code2vec_b200.path_context_reader import EstimatorAction
    from tests.test_reader_native import _Former, _setup
    C = 6
    cfg, vs = _setup(tmp_path, ["x"], C=C)
    reader = PathContextReader(vs, cfg, _Former(), EstimatorAction.Train, use_native=True)
    assert reader._native_ready()
    text = ("".join(l + ("\r\n" if i % 3 == 0 else "\n") + ("\n" if i % 7 == 0 else "")
                    for i, l in enumerate(_bad_lines(C, kind, seed)))).encode()
    path = str(tmp_path / "chunk.c2v")
    with open(path, "wb") as f:
        f.write(text)
    with open(path, "rb") as f:
        fd = f.fileno()
        shares = [share_range(fd, 0, len(text), world, r) for r in range(world)]
    statuses = [_share_status(reader, text[s0:s1], len(text)) for s0, s1 in shares]
    want = _host_parse(reader, text, len(text) // (C + 1) + 1)
    if kind == "clean":
        assert want is None
    if kind == "very_short":
        assert want == (None, 3)
    if kind == "short" and seed == 0 and world == 8:
        assert any(s.overflow for s in statuses)
    assert chunk_error(statuses, len(text), C) == want


def test_chunk_error_rule_on_constructed_statuses():
    from code2vec_b200.device_reader import chunk_error
    S = _Status
    # lower shares' newlines offset a share's local line; the lowest share with an error decides
    assert chunk_error([S(3, 4, -1, 0, 0), S(2, 2, 1, 2, 0), S(5, 5, 0, 1, 0)], 1000, 6) == (5, 2)
    assert chunk_error([S(3, 4, -1, 0, 0), S(2, 2, -1, 0, 0), S(5, 5, 0, 1, 0)], 1000, 6) == (6, 1)
    assert chunk_error([S(3, 4, -1, 0, 0), S(0, 0, -1, 0, 0), S(2, 2, -1, 0, 0)], 1000, 6) is None
    # more records than the chunk holds: kind 3 whatever the shares say
    assert chunk_error([S(100, 100, 0, 1, 1), S(100, 100, -1, 0, 1)], 1000, 6) == (None, 3)
    assert chunk_error([S(143, 143, 3, 1, 1)], 1000, 6) == (3, 1)             # cap = 1000 // 7 + 1 = 143
    assert chunk_error([S(144, 144, 3, 1, 1)], 1000, 6) == (None, 3)
    with pytest.raises(RuntimeError):
        chunk_error([S(10, 10, -1, 0, 1)], 1000, 6)                          # an overflow is always a malformed line


# ---- the switch ----------------------------------------------------------------------------------------------------------
def test_sharded_reader_flag():
    from code2vec_b200.device_reader import sharded_reader_flag
    assert sharded_reader_flag({}) is False
    assert sharded_reader_flag({"C2V_SHARDED_READER": "0"}) is False
    assert sharded_reader_flag({"C2V_SHARDED_READER": ""}) is False
    assert sharded_reader_flag({"C2V_SHARDED_READER": "1"}) is True
    for bad in ("2", "yes", "true", " 1", "on"):
        with pytest.raises(ValueError, match="C2V_SHARDED_READER"):
            sharded_reader_flag({"C2V_SHARDED_READER": bad})


@pytest.mark.parametrize("framework", ["b200", "b200-keras"])
def test_model_refuses_a_bad_switch_before_any_engine(monkeypatch, framework):
    from code2vec_b200 import b200_model
    from code2vec_b200.b200_keras_model import Code2VecModel as KerasModel
    from code2vec_b200.config import Config
    model_cls = b200_model.Code2VecModel if framework == "b200" else KerasModel
    cfg = Config(set_defaults=True)
    cfg.DL_FRAMEWORK = framework
    cfg.VERBOSE_MODE = 0
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    monkeypatch.setattr(b200_model.Code2VecModel, "_make_engine", None)     # no engine may be made: the refusal comes first
    monkeypatch.setenv("C2V_SHARDED_READER", "1")
    monkeypatch.delenv("C2V_DEVICE_READER", raising=False)
    with pytest.raises(ValueError, match="C2V_SHARDED_READER=1 .*C2V_DEVICE_READER=1"):
        model_cls(cfg)
    monkeypatch.setenv("C2V_DEVICE_READER", "0")
    with pytest.raises(ValueError, match="C2V_SHARDED_READER"):
        model_cls(cfg)
    monkeypatch.setenv("C2V_SHARDED_READER", "maybe")
    monkeypatch.setenv("C2V_DEVICE_READER", "1")
    with pytest.raises(ValueError, match="C2V_SHARDED_READER must be 0 or 1"):
        model_cls(cfg)
    if framework == "b200-keras":                  # the device reader's own refusal stands
        monkeypatch.setenv("C2V_SHARDED_READER", "1")
        with pytest.raises(ValueError, match="C2V_DEVICE_READER=1 is not available with --framework b200-keras"):
            model_cls(cfg)


def test_stage_bytes_cover_rows_keep_flags_and_status():
    from code2vec_b200.engine import c2v_reader_share_status, load_library
    lib = load_library()
    assert C.sizeof(c2v_reader_share_status) == 48
    for Cn, rows in ((13, 1), (200, 10434), (200, 83469)):
        n = lib.c2v_reader_stage_bytes(Cn, rows)
        assert n >= 256 + rows * ((4 * Cn + 1) * 4 + 1) and n % 256 == 0
    assert lib.c2v_reader_stage_bytes(0, 5) == 0 and lib.c2v_reader_stage_bytes(5, 0) == 0
