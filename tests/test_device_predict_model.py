"""CPU checks of the device predict route (DESIGN.md §6i): the '%f' formatter against Python, the switch, the two sources'
line rules, and a Python statement of the device's line scan, key rule, last-writer table and attention ranking
against __main__.print_predictions driven by a scripted model."""
import io
import struct

import numpy as np
import pytest

from code2vec_b200 import device_predict as DP
from code2vec_b200.__main__ import SHOW_TOP_CONTEXTS, java_string_hashcode, print_predictions
from code2vec_b200.model_base import Code2VecModelBase, ModelPredictionResults
from tests.predict_inputs import synthetic_lines


# ---- '%f' ------------------------------------------------------------------------------------------------------------
def _fixed(x: np.ndarray):
    from code2vec_b200 import engine as E
    lib = E.load_library()
    x = np.ascontiguousarray(x, dtype=np.float32)
    out = np.zeros(x.size * 48, dtype=np.uint8)
    ln = np.zeros(x.size, dtype=np.int32)
    assert lib.c2v_selftest_format_fixed(x.ctypes.data, x.size, out.ctypes.data, ln.ctypes.data) == 0
    return [out[i * 48:i * 48 + ln[i]].tobytes().decode() for i in range(x.size)]


def test_fixed_format_equals_python_on_a_seeded_sample():
    rng = np.random.default_rng(20)
    bits = [rng.integers(0, 2 ** 32, size=50000, dtype=np.uint64).astype(np.uint32)]
    bits.append(np.array([0, 1 << 31, 0x7f800000, 0xff800000, 0x7fc00000, 0xffc00000, 0x7f800001, 0xffffffff, 0x7f7fffff,
                          0xff7fffff, 1, 0x80000001, 0x007fffff, 0x00800000], dtype=np.uint32))     # specials, extremes
    ties = np.array([0.5e-6, 1.5e-6, 2.5e-6, 0.0078125, 0.0000005, 1.0000005, 2.5, 1e-6, 3.0517578125e-05],
                    dtype=np.float32)     # exact or nearest halves of the sixth decimal
    bits.append(ties.view(np.uint32))
    bits.append(rng.integers(0, 0x00800000, size=2000, dtype=np.uint64).astype(np.uint32))      # subnormals
    bits.append((rng.integers(0x34000000, 0x4b000000, size=20000, dtype=np.uint64)).astype(np.uint32))
    x = np.concatenate(bits).view(np.float32)
    got = _fixed(x)
    for v, g in zip(x, got):
        assert g == "%f" % float(v), (struct.pack("<f", v).hex(), g)


def test_the_switch():
    assert DP.device_predict_flag({}) is False
    assert DP.device_predict_flag({"C2V_DEVICE_PREDICT": ""}) is False
    assert DP.device_predict_flag({"C2V_DEVICE_PREDICT": "1"}) is True
    for bad in ("2", "yes", "true", " 1"):
        with pytest.raises(ValueError):
            DP.device_predict_flag({"C2V_DEVICE_PREDICT": bad})


# ---- a Python statement of the device route ----------------------------------------------------------------------------
_SPACE = b" \t\n\x0b\x0c\r\x1c\x1d\x1e\x1f"


def device_lines(data: bytes, universal: bool):
    """c2v_pred_chunk's lines: ends at '\\n' and (universal) a '\\r' not followed by '\\n'; each rstripped."""
    ends = [p for p in range(len(data)) if data[p] == 10 or (universal and data[p] == 13 and data[p + 1:p + 2] != b"\n")]
    starts = [0] + [e + 1 for e in ends]
    stops = ends + ([len(data)] if not ends or ends[-1] != len(data) - 1 else [])
    return [data[s:e].rstrip(_SPACE) for s, e in zip(starts, stops) if s < len(data) or e > s]


def key_of(path: bytes):
    """(key text, True), or (None, False) for a numeric path that is not an int32's canonical decimal."""
    body = path[1:] if path[:1] == b"-" else path
    if body and body.isdigit():
        v = int(path)
        return (path, True) if str(v).encode() == path and -2 ** 31 <= v < 2 ** 31 else (None, False)
    return str(java_string_hashcode(path.decode())).encode(), True


def device_text(data: bytes, universal: bool, C: int, results, oov: str, export: bool):
    """The device route's text for `data`, given the model's results per method (idx words, scores, attention per
    slot, code vector).  None where the route hands the input to the host."""
    methods, last = [], {}
    offset = 0
    for line in device_lines(data, universal):
        fields = line.split(b" ")
        if not fields[0]:
            continue
        ctx = [f for f in fields[1:] if f][:C]
        slots = []
        for c in ctx:
            parts = c.split(b",")
            if len(parts) != 3:
                raise ValueError("malformed")
            key, ok = key_of(parts[1])
            if not ok:
                return None
            offset += 1
            last[key] = max(last.get(key, (-1, b"")), (offset, parts[1]))
            slots.append((parts[0], key, parts[2]))
        methods.append((fields[0], slots))
    out = []
    for (name, slots), (words, scores, attn, vec) in zip(methods, results):
        out.append(b"Original name:\t" + name + b"\n")
        for w, s in zip(words, scores):
            if w != oov:
                out.append(b"\t(%s) predicted: %s\n" % (("%f" % float(s)).encode(), str(w.split("|")).encode()))
        out.append(b"Attention:\n")
        triples = slots + [None] * (C - len(slots))              # None: the padding triple
        first = [c for c in range(C) if triples[c] not in triples[:c]]
        val = {c: attn[max(d for d in range(C) if triples[d] == triples[c])] for c in first}
        nan = [np.isnan(val[c]) for c in first]
        if any(nan) and not all(nan):
            raise RuntimeError("partly NaN")
        rank = {c: sum(1 for d in first if d != c and (d < c if all(nan) else (val[d] > val[c] or (val[d] == val[c] and d < c))))
                for c in first}
        for c in sorted((c for c in first if rank[c] < SHOW_TOP_CONTEXTS), key=rank.get):
            if triples[c] is None:
                continue
            t1, key, t2 = triples[c]
            out.append(b"%s\tcontext: %s,%s,%s\n" % (("%f" % float(val[c])).encode(), t1, last[key][1], t2))
        if export:
            out.append(b"Code vector:\n" + " ".join(map(str, vec)).encode() + b"\n")
    return b"".join(out)


class _Special:
    OOV = "<OOV>"
    PAD = "<PAD>"


class _Scripted:
    """A model whose predictions are fixed per method: what print_predictions sees from Code2VecModel.predict."""

    def __init__(self, C, results):
        self.C, self.results, self.calls = C, results, 0

        class V:
            pass
        self.vocabs = V()
        self.vocabs.target_vocab = V()
        self.vocabs.target_vocab.special_words = _Special

    def predict(self, lines):
        out = []
        for line in lines:
            words, scores, attn, vec = self.results[self.calls]
            self.calls += 1
            fields = line.split(" ")
            trip = [f.split(",") if f else [_Special.PAD] * 3 for f in fields[1:self.C + 1]]
            att = Code2VecModelBase._get_attention_weight_per_context(
                None, [t[0] for t in trip], [t[1] for t in trip], [t[2] for t in trip], attn)
            out.append(ModelPredictionResults(fields[0], np.array(words), np.float32(scores), att, np.float32(vec)))
        return out


class _Cfg:
    def __init__(self, C, export):
        self.MAX_CONTEXTS, self.EXPORT_CODE_VECTORS = C, export


def _results(n, C, seed, nan_rows=()):
    rng = np.random.default_rng(seed)
    words = ["get|name", "set", "<OOV>", "run|it|now", "x"]
    res = []
    for m in range(n):
        w = [words[i] for i in rng.permutation(len(words))[:4]]
        attn = rng.choice(np.float32([0.125, 0.25, 0.5, 0.0625]), size=C).astype(np.float32)   # many ties
        if m in nan_rows:
            attn[:] = np.nan
        res.append((w, rng.random(4).astype(np.float32), attn, rng.standard_normal(3).astype(np.float32)))
    return res


def _host(data: bytes, universal: bool, C: int, results, export: bool) -> bytes:
    out = io.StringIO()
    print_predictions(_Cfg(C, export), _Scripted(C, results), DP.split_source_lines(data, universal), out=out)
    return out.getvalue().encode()


@pytest.mark.parametrize("universal", [True, False])
@pytest.mark.parametrize("C", [4, 12])
def test_the_device_statement_prints_what_print_predictions_prints(universal, C):
    tokens = ["a", "b", "c", "dd"]
    lines = synthetic_lines(300, 3, tokens, ["m|x", "n"], max_bag=C + 5, n_paths=6, numeric_paths=["12", "-5"])
    tail = ["h1 a,Aa,b c,BB,d a,Aa,b", "h2 a,2112,b", "h3 x,,y -,-,- p,a,,q".replace("p,a,,q", "p,a|b,q"), "empty",
            "ws a,b,c \x0b\x0c\x1c", "  lead a,b,c"]
    text = "\n".join(lines + tail)
    text = text.replace("\nh1", "\r\nh1").replace("\nh2", "\rh2")
    data = text.encode()
    n = sum(1 for _ in device_lines(data, universal))
    results = _results(n, C, seed=C, nan_rows={5, 77})
    host = _host(data, universal, C, results, export=True)
    dev = device_text(data, universal, C, results, "<OOV>", export=True)
    assert dev == host
    assert host.count(b"Original name:\t") > 300


def test_the_sources_split_carriage_returns_differently():
    data = b"a\rb x,Aa,y\r\nc p,BB,q\n"
    assert list(DP.split_source_lines(data, False)) == ["a\rb x,Aa,y\r\n", "c p,BB,q\n"]
    assert list(DP.split_source_lines(data, True)) == ["a\n", "b x,Aa,y\n", "c p,BB,q\n"]
    assert [bytes(x) for x in device_lines(data, False)] == [b"a\rb x,Aa,y", b"c p,BB,q"]
    assert [bytes(x) for x in device_lines(data, True)] == [b"a", b"b x,Aa,y", b"c p,BB,q"]


def test_keys_collide_and_odd_numeric_paths_leave_the_device():
    assert key_of(b"Aa") == key_of(b"BB") == (b"2112", True)
    assert key_of(b"2112") == (b"2112", True)
    assert key_of(b"-2147483648") == (b"-2147483648", True)
    assert key_of(b"") == (b"0", True) and key_of(b"-")[1]
    for odd in (b"007", b"-0", b"2147483648", b"-2147483649", b"00"):
        assert key_of(odd) == (None, False)


def test_a_partly_nan_row_raises_and_malformed_contexts_raise_before_output():
    C = 4
    results = _results(2, C, seed=1)
    results[1][2][1] = np.nan
    with pytest.raises(RuntimeError):
        device_text(b"m a,b,c d,e,f\nn a,b,c x,y,z\n", True, C, results, "<OOV>", False)
    for bad in (b"m a,b\n", b"m a,b,c,d\n"):
        with pytest.raises(ValueError):
            _host(bad, True, C, results, False)
        with pytest.raises(ValueError):
            device_text(bad, True, C, results, "<OOV>", False)


@pytest.mark.parametrize("chunk_bytes", [1, 2, 3, 7, 64, 1 << 20])
def test_chunks_are_whole_lines_under_both_rules(chunk_bytes):
    data = b"ab\r\ncd\ref\n\ngh x,y,z\r\n" * 5 + b"tail\r"
    ranges = DP.chunk_ranges(data, chunk_bytes)
    assert ranges[0][0] == 0 and ranges[-1][1] == len(data)
    assert all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
    for lo, hi in ranges:
        assert hi == len(data) or data[hi - 1:hi] == b"\n"          # never inside a line, never between "\r" and "\n"
        assert hi - lo <= chunk_bytes or data.count(b"\n", lo, hi - 1) == 0
    for universal in (True, False):
        whole = [bytes(x) for x in device_lines(data, universal)]
        pieces = [bytes(x) for lo, hi in ranges for x in device_lines(data[lo:hi], universal)]
        assert pieces == whole
    assert DP.chunk_ranges(b"", 8) == []
