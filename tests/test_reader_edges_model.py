"""Inputs built to reach the warp, tile and block edges of the device reader's kernels (csrc/reader.cu), and checks, without
a GPU, that they do reach them.  tests/test_gpu_reader_kernels.py runs the kernels on these inputs against the host
statements; this file shows what those inputs hold:
  * parse texts: a separator at every offset 0-95 of a record, fields of 0-65 bytes around the 32-byte ballot windows,
    runs of spaces, commas in targets, every part shape, '\\r' inside fields and '\\r\\r\\n' endings, records and blank
    lines starting exactly at a 4096-byte line-index tile, records longer than a tile, chunks of 4096 j - 1, 4096 j and
    4096 j + 1 bytes, and a last line without a newline;
  * malformed records whose third comma sits at lane 0 or lane 31 of a window, inside the first C contexts (kind 2) or in
    a field beyond them (kind 1), and chunks with more records than they hold well-formed lines (kind 3), with the host
    parser's verdict on each;
  * vocabularies of 64-256 slots whose probe chains wrap from the last slot to slot 0, with absent words that hash into
    a wrapped chain;
  * metric inputs: top-k lists of up to 64 ids whose first legal match is in the second or third 32-id window, and names
    and words with more than 32 subtokens."""
import ctypes

import numpy as np
import pytest

from code2vec_b200.path_context_reader import load_native_tensoriser
from code2vec_b200.vocabularies import _SpecialVocabWords_JoinedOovPad as _JOIN
from code2vec_b200.vocabularies import _SpecialVocabWords_OnlyOov as _ONLY_OOV
from code2vec_b200.vocabularies import _SpecialVocabWords_SeparateOovPad as _SEP
from tests.test_device_eval_model import _Vocab, score_row
from tests.test_device_reader_model import _fnv1a, _native_vocab

TILE = 4096


# ---- vocabularies ------------------------------------------------------------------------------------------------------
def _slots(n: int) -> int:
    """The slot count c2v_vocab_create gives a table of n words."""
    cap = 16
    while cap < 2 * n + 2:
        cap <<= 1
    return cap


def _homed(prefix: str, mask: int, homes, count: int, skip=()):
    """`count` words prefix%d whose FNV-1a 64 & mask is one of `homes` (brute force)."""
    out, i = [], 0
    while len(out) < count:
        w = "%s%d" % (prefix, i)
        if (_fnv1a(w.encode()) & mask) in homes and w not in skip:
            out.append(w)
        i += 1
    return out


class EdgeVocab:
    """Words of one table, in index order: index 0 is OOV, index 1 PAD (token and path tables with separate OOV and PAD;
    the target table and joined tables have one special word).  `n` words make a table of _slots(n) slots; `wrap` words
    hash into its last three slots, so their chain runs past the last slot to slot 0; `absent` words are not in the table
    and hash into that chain (a lookup walks it, wraps, and ends at an empty slot: OOV)."""

    def __init__(self, special, words, n, prefix, n_wrap=6):
        specials = [special.OOV] if special.OOV == getattr(special, "PAD", special.OOV) else [special.OOV, special.PAD]
        self.special = special
        mask = _slots(n) - 1
        last = {mask - 2, mask - 1, mask}
        self.wrap = _homed(prefix + "w", mask, last, n_wrap)
        self.absent = _homed(prefix + "a", mask, last | {0}, 4)
        fill = ["%s%d" % (prefix, i) for i in range(n)]
        self.words = (specials + self.wrap + list(words) + fill)[:n]
        assert len(set(self.words)) == n == len(self.words)
        self.mask = mask
        self.oov = 0
        self.pad = len(specials) - 1

    def native(self, lib):
        return _native_vocab(lib, self.words, list(range(len(self.words))), self.oov, self.pad)


TOKEN_WORDS = ["", "a", "b", "ab", "a\rb", "x" * 31, "x" * 32, "x" * 33, "y" * 63, "y" * 64, "y" * 65,
               "p" * 31 + "A", "p" * 31 + "B", "q" * 32 + "A", "q" * 32 + "B", "lastA", "lastB", "üüü", "名前", "名前x",
               "é" * 16, "z" * 301]
PATH_WORDS = ["", "1", "12", "9" * 31, "9" * 32, "9" * 33, "7" * 64, "55A", "55B"]


def _target_word(L: int) -> str:
    """A target word of L bytes with '|' subtokens and commas (field 0 is split on spaces only)."""
    return ("ab,c|Def|" * 12)[:L]


def edge_vocabs(separate: bool):
    """(token, path, target) EdgeVocab: 80 + 40 + 120 words, tables of 256, 128 and 256 slots.  The target table holds a
    word of every length 1-95, so a kept record's first space can be at any offset 0-95."""
    tp = _SEP if separate else _JOIN
    tok = EdgeVocab(tp, TOKEN_WORDS, 80, "tok")
    pth = EdgeVocab(tp, PATH_WORDS, 40, "pth")
    tgt = EdgeVocab(_ONLY_OOV if separate else _JOIN, [_target_word(L) for L in range(1, 96)], 120, "tgt")
    return tok, pth, tgt


# ---- parse texts -------------------------------------------------------------------------------------------------------
class EdgeText:
    """A seeded writer of one chunk of `.c2v` text for MAX_CONTEXTS = C over edge_vocabs: well-formed records of every
    field and part shape, with helpers that place a record, a blank line or a malformed record at chosen byte offsets."""

    def __init__(self, C, vocabs, seed):
        self.C, self.rng = C, np.random.default_rng(seed)
        self.tok, self.pth, self.tgt = vocabs
        self.buf = bytearray()
        self.bad = []                                   # (line number, kind) of every malformed record written
        self.n_targets = int(seed)                      # target lengths cycle through 1-95

    # words and fields
    def _pick(self, words):
        return words[int(self.rng.integers(0, len(words)))]

    def _tok(self):
        r = self.rng.random()
        if r < 0.1:
            return "oov%d" % int(self.rng.integers(0, 1000))
        if r < 0.2:
            return self._pick(self.tok.absent)
        if r < 0.3:
            return self._pick(self.tok.wrap)
        return self._pick(self.tok.words[2:])

    def _pth(self):
        r = self.rng.random()
        if r < 0.1:
            return self._pick(self.pth.absent)
        return self._pick(self.pth.words[2:])

    def _context(self):
        k = int(self.rng.integers(0, 12))
        s, p, t = self._tok(), self._pth(), self._tok()
        return ["", s, "%s,%s" % (s, p), "%s,%s,%s" % (s, p, t), ",", ",,", "%s,," % s, ",%s" % p, "%s,,%s" % (s, t),
                "%s,%s," % (s, p), "%s,%s,%s" % (s, p, t), "%s,%s,%s" % (s, p, t)][k]

    def _target(self):
        r = self.rng.random()
        if r < 0.08:
            return ""                                   # a leading space: OOV target
        if r < 0.16:
            return "unknown,%d" % int(self.rng.integers(0, 99))        # OOV target: dropped in training
        if r < 0.22:
            return self._pick(self.tgt.wrap)
        self.n_targets += 1
        return _target_word(1 + self.n_targets % 95)

    def _contexts(self):
        C = self.C
        ctx = [self._context() for _ in range(C)]
        if C > 3 and self.rng.random() < 0.4:           # a run of 2-70 spaces: empty contexts in a row
            run = int(self.rng.integers(1, min(C, 70)))
            at = int(self.rng.integers(0, C - run + 1))
            ctx[at:at + run] = [""] * run
        if self.rng.random() < 0.2:                     # trailing spaces
            n = min(C, int(self.rng.integers(1, 6)))
            ctx[-n:] = [""] * n
        return ctx

    def _end(self):
        return ["\n", "\n", "\n", "\r\n", "\r\r\n"][int(self.rng.integers(0, 5))]

    # writing
    @property
    def line(self) -> int:
        return self.buf.count(b"\n")

    def record(self):
        self.buf += (" ".join([self._target()] + self._contexts()) + self._end()).encode("utf-8")

    def filler(self, length: int):
        """A kept record of exactly `length` bytes (newline included; an OOV token and a known path); length >= C + 4."""
        C = self.C
        assert length >= C + 4
        tgt = self._pick([w for w in self.tgt.words[1:] if len(w.encode()) <= length - C - 4])
        m = length - len(tgt.encode()) - C - 3
        self.buf += (tgt + " " + "f" * m + ",1" + " " * (C - 1) + "\n").encode()

    def pad_to(self, pos: int):
        """Fill the chunk up to byte `pos` (or the next tile after it, if the gap is too short for a record)."""
        while pos - len(self.buf) < self.C + 4:
            pos += TILE
        gap = pos - len(self.buf)
        while gap > 2000 + self.C:                      # several records, then one of the exact length left
            self.filler(1000 + self.C)
            gap -= 1000 + self.C
        self.filler(gap)
        return pos

    def long_record(self, nbytes=5000):
        """A record longer than a line-index tile (an OOV token of nbytes bytes)."""
        ctx = self._contexts()
        ctx[int(self.rng.integers(0, self.C))] = "L" * nbytes + "," + self._pth()
        self.buf += (" ".join([self._target()] + ctx) + "\n").encode()

    def bad_record(self, lane: int, beyond: bool):
        """A record whose third comma of one field is at `lane` (mod 32) of its window: in a context among the first C
        (kind 2), or, with beyond=True, in an extra field after them (kind 1, the field count)."""
        C = self.C
        ctx = self._contexts()
        head = (" ".join([self._target()] + (ctx if beyond else ctx[:C - 1])) + " ").encode()
        pos = len(head)                                 # the bad field starts here, within the record
        m = (lane - (pos + 4)) % 32                     # 'q' * m + ",1,a," puts the third comma at pos + m + 4
        bad = ("q" * m + ",1,a,b").encode()
        assert (pos + len(bad) - 2) % 32 == lane
        self.bad.append((self.line, 1 if beyond else 2))
        self.buf += head + bad + b"\n"

    def short_field_count(self):
        self.bad.append((self.line, 1))
        self.buf += (" ".join([self._target()] + self._contexts()[:-1]) + "\n").encode()

    def text(self) -> bytes:
        return bytes(self.buf)


def edge_chunk(C, vocabs, seed, edge=None, records=100, eol=True):
    """One well-formed chunk: records of every shape, a record and a blank line at tile starts, a record longer than a
    tile, and, when `edge` is -1, 0 or 1, the chunk filled to 4096 j + edge bytes exactly; eol=False drops the last
    newline.  Returns the text and the offset of the blank line."""
    t = EdgeText(C, vocabs, seed)
    for _ in range(records):
        t.record()
    t.pad_to(TILE)
    t.record()                                          # a record starting at byte 4096
    t.long_record()                                     # spans tiles
    for _ in range(records // 4):
        t.record()
    blank = t.pad_to((len(t.buf) // TILE + 1) * TILE)
    t.buf += b"\n"                                      # a blank line at byte 4096 j
    t.record()
    if edge is not None:
        t.pad_to((len(t.buf) // TILE + 1) * TILE + edge)
    text = t.text()
    return (text if eol else text[:-1]), blank


SIZE_EDGES = (-1, 0, 1)


def parse_chunks(C, vocabs):
    """The chunks the device parse is checked on for MAX_CONTEXTS = C, in order, as (text, offset of its blank line):
    one of a free size, one each of 4096 j - 1, 4096 j and 4096 j + 1 bytes (all ending in a newline), and one whose
    last line has no newline."""
    sizes = (None,) + SIZE_EDGES + (None,)
    return [edge_chunk(C, vocabs, 10 * C + i, edge=edge, eol=i < len(sizes) - 1) for i, edge in enumerate(sizes)]


def malformed_chunk(C, vocabs, seed, case):
    """A chunk with malformed records and the host's expected verdict (line, kind) of its lowest one."""
    t = EdgeText(C, vocabs, seed)
    for _ in range(12):
        t.record()
    if case == "kind3":
        t.buf += b"x\n" * (2 * len(t.buf) // (C + 1) + 8)
        return t.text(), None
    lane, beyond = {"lane0_ctx": (0, False), "lane31_ctx": (31, False), "lane0_beyond": (0, True),
                    "lane31_beyond": (31, True)}.get(case, (None, None))
    if lane is not None:
        t.bad_record(lane, beyond)
    else:
        t.short_field_count()
    for _ in range(6):
        t.record()
    t.bad_record(31 - (lane or 0), not beyond if lane is not None else True)          # a second, higher bad line
    for _ in range(4):
        t.record()
    return t.text(), t.bad[0]


# ---- the host parser ---------------------------------------------------------------------------------------------------
class HostTables:
    """The native tensoriser's tables of edge_vocabs (what the device reader is given, through c2v_vocab_export)."""

    def __init__(self, separate):
        self.lib = load_native_tensoriser()
        self.vocabs = edge_vocabs(separate)
        self.native = [v.native(self.lib) for v in self.vocabs]


def host_parse(H, text: bytes, C: int, mode: int = 0):
    """c2v_parse_chunk on one thread: (n, err_kind, rows (src, path, dst, mask, target), keep, tgt_off, tgt_len);
    n < 0 is -(line + 1) of the lowest malformed line, INT64_MIN a chunk with too many records."""
    cap = len(text) // (C + 1) + 1
    src, path, dst = (np.zeros((cap, C), dtype=np.int32) for _ in range(3))
    mask = np.zeros((cap, C), dtype=np.float32)
    target = np.zeros(cap, dtype=np.int32)
    keep = np.zeros(cap, dtype=np.uint8)
    toff, tlen = np.zeros(cap, dtype=np.int64), np.zeros(cap, dtype=np.int32)
    err = ctypes.c_int32(0)
    tok, pth, tgt = H.native
    n = H.lib.c2v_parse_chunk(text, len(text), C, tok.h, pth.h, tgt.h, mode, 1, cap, src.ctypes.data, path.ctypes.data,
                              dst.ctypes.data, mask.ctypes.data, target.ctypes.data, keep.ctypes.data, toff.ctypes.data,
                              tlen.ctypes.data, ctypes.byref(err))
    m = max(int(n), 0)
    return int(n), err.value, (src[:m], path[:m], dst[:m], mask[:m], target[:m]), keep[:m], toff[:m], tlen[:m]


def record_starts(text: bytes):
    """Byte offsets of the records (non-blank lines) of a chunk."""
    starts, pos = [], 0
    while pos < len(text):
        nl = text.find(b"\n", pos)
        nxt = len(text) if nl < 0 else nl + 1
        if nl != pos:
            starts.append(pos)
        pos = nxt
    return starts


def separator_offsets(text: bytes):
    """Offsets from their record's start of the spaces and of the commas after the first space."""
    sp, cm = set(), set()
    for s in record_starts(text):
        e = text.find(b"\n", s)
        line = text[s:len(text) if e < 0 else e]
        first = line.find(b" ")
        for i, c in enumerate(line):
            if c == 0x20:
                sp.add(i)
            elif c == 0x2C and 0 <= first < i:
                cm.add(i)
    return sp, cm


# ---- metric inputs -----------------------------------------------------------------------------------------------------
def metric_words():
    """Target words of the metric tests, index order (index 0 the OOV word): long words with more than 32 subtokens,
    empty and repeated subtokens, illegal words (digits, '_'), and short legal ones."""
    long1 = "|".join(["get", "", "Name", "get"] * 10)                          # 40 subtokens, 2 empty, repeats
    long2 = "|".join("abcdefghijklmnopqrstuvwxyzABCDEFGHIJ")                  # 36 one-letter subtokens
    long3 = "X" * 40
    words = [long1, long2, long3, "get|name", "getName", "name", "get", "x|y", "|", "a||b", "set|value|value",
             "n" * 33, "abc|abc|abc"]
    illegal = ["get2", "x_y", "9", "get|1", "a b"[0:1] + "1"]
    return words, illegal


def metric_names():
    """Names (bytes) of the metric tests: over 32 bytes and 32 subtokens, mixed case and digits, no letters, bytes >= 0x80,
    and each target word itself."""
    words, _ = metric_words()
    names = [w.encode() for w in words]
    names += [b"GET|NAME", b"get_name_2", b"12345", b"||||", b"|" * 40, b"a" * 70, b"A1b2|C3d4" * 6,
              ("|".join(["sub%d" % i for i in range(45)])).encode(), b"\xc3\xbc|get", b"get|name\xff", b"<OOV>", b"Get|Name|" * 8, b"n" * 33]
    return names


def metric_vocab(separate=True):
    words, illegal = metric_words()
    special = _ONLY_OOV if separate else _JOIN
    return _Vocab([special.OOV] + words + illegal, special)


def metric_rows(vocab, k, n, seed):
    """n rows of (name, top-k ids): ids mixing illegal words, OOV, repeated ids, INT_MAX padding (Y < k), and rows whose
    first legal match is placed in the second or third 32-id window, or that hold no legal word at all."""
    from code2vec_b200.common import common
    rng = np.random.default_rng(seed)
    Y = vocab.size
    legal = [i for i in range(Y) if common.legal_method_names_checker(vocab.special_words, vocab.index_to_word[i])]
    illegal = [i for i in range(Y) if i not in legal]
    names = metric_names()
    rows = []
    for r in range(n):
        name = names[int(rng.integers(0, len(names)))]
        kind = r % 6
        if kind == 0:                                   # uniform ids, repeats allowed
            ids = rng.integers(0, Y, size=k)
        elif kind == 1:                                 # no legal word
            ids = rng.choice(illegal, size=k)
        elif kind == 2:                                 # Y < k: INT_MAX padding after the real ids
            ids = np.full(k, np.iinfo(np.int32).max)
            m = int(rng.integers(0, k + 1))
            ids[:m] = rng.integers(0, Y, size=m)
        else:                                           # illegal ids first, the name's own word at position pos
            ids = rng.choice(illegal, size=k)
            pos = int(rng.integers(min(32, k - 1) if kind == 3 else 0, k))
            if kind == 5 and k > 32:                    # the second window, or the third when there is one
                pos = int(rng.integers(64 if k > 64 else 32, k))
            word = name.decode("utf-8", "replace")
            match = [i for i in legal if vocab.index_to_word[i] == word]
            ids[pos] = match[0] if match else int(rng.choice(legal))
            if kind == 4:                               # some legal non-matching words before it, in earlier windows
                for q in rng.integers(0, pos + 1, size=min(pos, 5)):
                    if q != pos:
                        ids[q] = int(rng.choice(legal))
        rows.append((name, [int(i) for i in ids]))
    return rows


# ---- the checks --------------------------------------------------------------------------------------------------------
needs_native = pytest.mark.skipif(load_native_tensoriser() is None, reason="g++ build of the native tensoriser failed")


@needs_native
@pytest.mark.parametrize("separate", [False, True])
def test_tables_have_chains_that_wrap(separate):
    from code2vec_b200.device_reader import export_vocab
    from tests.test_device_reader_model import _probe
    H = HostTables(separate)
    for v, nv in zip(H.vocabs, H.native):
        slots_raw, byte_arr, mask, oov, pad = export_vocab(H.lib, nv.h)
        assert mask == v.mask and 64 <= mask + 1 <= 256
        slots = slots_raw.copy().view(np.dtype([("h", "<u8"), ("off", "<i8"), ("len", "<i4"), ("idx", "<i4")])).ravel()
        home = [int(s["h"]) & mask if s["h"] else -1 for s in slots]
        wrapped = [i for i in range(mask + 1) if home[i] > i]          # placed past the last slot, at or after slot 0
        assert wrapped, "no chain wraps"
        # an absent word walks a wrapped chain and ends at an empty slot: OOV
        assert any(home[_fnv1a(w.encode()) & mask] >= 0 for w in v.absent)
        tup = [(int(s["h"]), int(s["off"]), int(s["len"]), int(s["idx"])) for s in slots]
        for w in v.words + v.absent:
            b = w.encode()
            assert _probe(tup, byte_arr, mask, oov, b) == H.lib.c2v_vocab_lookup(nv.h, b, len(b))
        for w in v.absent:
            assert H.lib.c2v_vocab_lookup(nv.h, w.encode(), len(w.encode())) == oov


@needs_native
@pytest.mark.parametrize("separate", [False, True])
@pytest.mark.parametrize("C", [1, 13, 31, 32, 33, 200])
def test_edge_chunks_reach_the_window_and_tile_edges(C, separate):
    H = HostTables(separate)
    sp, cm, starts_at_tile, spans = set(), set(), 0, 0
    chunks = parse_chunks(C, H.vocabs)
    # the three size edges, every one ending in a newline (so a chunk of 4096 j + 1 bytes ends with a tile holding only
    # the last '\n'), and a last chunk whose last line has no newline
    assert [len(text) % TILE for text, _ in chunks[1:4]] == [e % TILE for e in SIZE_EDGES]
    assert all(text.endswith(b"\n") for text, _ in chunks[:-1]) and not chunks[-1][0].endswith(b"\n")
    for text, blank_at in chunks:
        assert text[blank_at:blank_at + 1] == b"\n" and text[blank_at - 1:blank_at] == b"\n"
        starts = record_starts(text)
        starts_at_tile += sum(1 for s in starts if s > 0 and s % TILE == 0)
        ends = starts[1:] + [len(text)]
        spans += sum(1 for s, e in zip(starts, ends) if e - s > TILE)
        a, b = separator_offsets(text)
        sp |= a
        cm |= b
        n, err, rows, keep, _, _ = host_parse(H, text, C)
        assert n == len(starts), (n, err)                              # well-formed: every record parses
        assert 0 < keep.sum() < n
    assert set(range(96)) <= sp                                        # a space at every offset 0-95
    assert {o % 32 for o in cm} == set(range(32))
    assert {o % 32 for o in sp} == set(range(32))
    assert starts_at_tile >= 5 and spans >= 5


@needs_native
@pytest.mark.parametrize("C", [1, 13, 33, 200])
@pytest.mark.parametrize("case", ["lane0_ctx", "lane31_ctx", "lane0_beyond", "lane31_beyond", "fields", "kind3"])
def test_malformed_chunks_have_the_host_verdict(C, case):
    H = HostTables(False)
    if C == 1 and case == "kind3":
        pytest.skip("with one context a record of 2 bytes is as short as a well-formed one: no chunk has too many")
    text, want = malformed_chunk(C, H.vocabs, 7, case)
    n, err, *_ = host_parse(H, text, C)
    if want is None:
        assert n == np.iinfo(np.int64).min
    else:
        assert (-n - 1, err) == want


def test_metric_inputs_reach_the_second_and_third_windows():
    v = metric_vocab()
    from code2vec_b200.device_reader import eval_tables
    tables = eval_tables(v)
    ranks, positions, subtokens, flags = [], [], [], set()
    for k in (33, 63, 64, 100):
        for name, ids in metric_rows(v, k, 300, seed=k):
            rank, first, flag, counts = score_row(name, ids, tables)
            flags.add(flag)
            if rank >= 0:
                ranks.append(rank)
                pos = next(i for i, x in enumerate(ids) if 0 <= x < v.size and tables[4][x] and
                           score_row(name, [x], tables)[0] == 0)
                positions.append(pos)
            if counts is not None:
                subtokens.append(max(name.count(b"|"), v.index_to_word[first].count("|")) + 1)
    assert max(positions) >= 64 and sum(32 <= p < 64 for p in positions) > 10
    assert max(ranks) >= 1
    assert flags == {0, 1, 2}
    assert max(subtokens) > 32
