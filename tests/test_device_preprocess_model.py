"""The host-side statements of the device preprocessing route (code2vec_b200/device_preprocess.py), without a GPU: the
chunk cutter and the line index under universal newlines against open(..., "r"), the first-occurrence order the
histograms are written in, the sampler identity the route rests on, and the switch."""
import random
from collections import Counter

import pytest

from code2vec_b200 import device_preprocess as D
from code2vec_b200 import preprocess as P


def lines_by_chunks(data: bytes, window: int):
    """Every line's text as the device route sees it: chunks of whole lines, each indexed on its own."""
    read = lambda off, n: data[off:off + n]
    out, end = [], 0
    for a, b in D.chunk_ranges(read, len(data), window):
        assert a == end and b > a
        end = b
        chunk = data[a:b]
        out += [chunk[s:e].decode() for s, e in D.line_spans(chunk)]
    assert end == len(data)
    return out


def host_lines(tmp_path, data: bytes):
    path = tmp_path / "f.txt"
    path.write_bytes(data)
    with open(path, "r") as f:
        return [line.rstrip("\n") for line in f]


@pytest.mark.parametrize("eol", [b"\n", b"\r\n", b"\r"], ids=["lf", "crlf", "cr"])
def test_line_ends_at_every_chunk_edge(tmp_path, eol):
    words = [b"ab", b"", b"c d", b"", b"", b"efg h,i", b"j"]
    for final in (True, False):
        data = eol.join(words) + (eol if final else b"")
        want = host_lines(tmp_path, data)
        for window in range(1, len(data) + 2):
            assert lines_by_chunks(data, window) == want, (eol, final, window)


def test_mixed_line_ends_at_every_chunk_edge(tmp_path):
    data = b"a\r\nb\rc\n\r\n\rd\r\r\ne f\n\n\r"
    want = host_lines(tmp_path, data)
    assert want == ["a", "b", "c", "", "", "d", "", "e f", "", ""]
    for window in range(1, len(data) + 2):
        assert lines_by_chunks(data, window) == want, window
    # a chunk never ends between the '\r' and the '\n' of "\r\n"
    read = lambda off, n: data[off:off + n]
    for window in range(1, len(data) + 2):
        for a, b in D.chunk_ranges(read, len(data), window):
            assert not (b < len(data) and data[b - 1] == 0x0D and data[b] == 0x0A)


def test_a_line_longer_than_the_window(tmp_path):
    data = b"x" * 1000 + b"\r\n" + b"short\n" + b"y" * 300 + b"\rz"
    want = host_lines(tmp_path, data)
    for window in (1, 7, 64, 999, 1000, 1001, 1002):
        assert lines_by_chunks(data, window) == want
    # the doubled window stays: the short line after the long one rides in the same chunk
    read = lambda off, n: data[off:off + n]
    chunks = list(D.chunk_ranges(read, len(data), 64))
    assert chunks == [(0, 1008), (1008, len(data))]


def test_histograms_in_order_of_first_byte_offset(tmp_path):
    """count_histograms' Counters are in insertion order, which is the order of each key's first byte offset -- the
    sort key the device uses."""
    rng = random.Random(5)
    lines = []
    for _ in range(200):
        ctxs = []
        for _ in range(rng.randrange(0, 6)):
            parts = [rng.choice(["a", "b", "c", "", "d"]) for _ in range(rng.choice([1, 2, 3, 3, 4]))]
            ctxs.append(",".join(parts))
        lines.append(" ".join([rng.choice(["t", "u", ""])] + ctxs))
    data = "\n".join(lines) + "\n"
    path = tmp_path / "raw.txt"
    path.write_text(data)
    tokens, paths, targets = P.count_histograms(str(path))
    first = {0: {}, 1: {}, 2: {}}                     # kind -> key -> first offset, from the bytes
    count = {0: Counter(), 1: Counter(), 2: Counter()}
    raw = data.encode()
    for s, e in D.line_spans(raw):
        line, f0 = raw[s:e].decode(), s
        fields = line.split(" ")
        occ = [(2, fields[0], s)]
        pos = s + len(fields[0]) + 1
        for ctx in fields[1:]:
            parts, p = ctx.split(","), pos
            starts = []
            for part in parts:
                starts.append(p)
                p += len(part) + 1
            if len(parts) >= 3:
                occ += [(0, parts[0], starts[0]), (1, parts[1], starts[1]), (0, parts[2], starts[2])]
            else:
                occ.append((0, parts[0], starts[0]))
                if len(parts) > 1:
                    occ.append((1, parts[1], starts[1]))
            pos += len(ctx) + 1
        for kind, key, off in occ:
            first[kind].setdefault(key, off)
            count[kind][key] += 1
    for kind, counter in ((0, tokens), (1, paths), (2, targets)):
        assert list(counter.items()) == sorted(count[kind].items(), key=lambda kv: first[kind][kv[0]])


@pytest.mark.parametrize("n,k", [(5, 2), (20, 20), (300, 200), (1000, 200), (2000, 5), (21, 1), (7, 0)])
def test_sampling_indices_is_sampling_the_list(n, k):
    """rng.sample(range(n), k) returns the indices of rng.sample(list_of_n, k) and leaves the same state -- in both of
    random.sample's branches (a pool for small populations, a set of picks for large ones)."""
    population = ["ctx%d" % i for i in range(n)]
    for seed in range(3):
        a, b = random.Random(seed), random.Random(seed)
        picked = a.sample(population, k)
        idx = b.sample(range(n), k)
        assert picked == [population[i] for i in idx]
        assert a.getstate() == b.getstate()


def test_switch_values():
    assert D.device_preprocess_flag({}) is False
    assert D.device_preprocess_flag({"C2V_DEVICE_PREPROCESS": ""}) is False
    assert D.device_preprocess_flag({"C2V_DEVICE_PREPROCESS": "0"}) is False
    assert D.device_preprocess_flag({"C2V_DEVICE_PREPROCESS": "1"}) is True
    for bad in ("2", "yes", "true", " 1"):
        with pytest.raises(ValueError):
            D.device_preprocess_flag({"C2V_DEVICE_PREPROCESS": bad})


def test_main_rejects_a_bad_switch_before_reading(monkeypatch, tmp_path):
    monkeypatch.setenv("C2V_DEVICE_PREPROCESS", "on")
    with pytest.raises(ValueError):
        P.main(["-trd", str(tmp_path / "missing"), "-ted", "x", "-vd", "y", "-o", str(tmp_path / "o")])
