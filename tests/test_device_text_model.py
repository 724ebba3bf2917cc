"""The float32 text of csrc/text.cu (C2V_DEVICE_TEXT=1, DESIGN.md §6f) against numpy, without a GPU.

c2v_selftest_format_floats runs on the CPU the __host__ __device__ formatter the device kernel runs; every value must
be written as str(np.float32(x)) writes it.  The line layout the kernel builds from those values (single spaces, '\\n',
word prefixes) is checked against model_base._write_code_vectors and common.save_word2vec_file."""
import io

import numpy as np
import pytest

from tools.float_text_sweep import format_floats

F32_MIN_BITS, F32_MAX_BITS = 0x00800000, 0x7F7FFFFF


@pytest.fixture(scope="module")
def lib():
    from code2vec_b200 import engine as E
    return E.load_library()


def _texts(lib, x):
    """Our text of every value of x, as str."""
    ours, lens = format_floats(lib, np.asarray(x, dtype=np.float32))
    assert lens.max(initial=0) <= 15
    return [t.decode() for t in ours]


def _bits(b):
    return np.asarray(b, dtype=np.uint64).astype(np.uint32).view(np.float32)


def _assert_numpy(lib, x):
    x = np.asarray(x, dtype=np.float32)
    got = _texts(lib, x)
    want = [str(v) for v in x]
    bad = [(hex(int(v.view(np.uint32))), g, w) for v, g, w in zip(x, got, want) if g != w]
    assert not bad, bad[:10]
    # the exhaustive sweep (tools/float_text_sweep.py) asks numpy through astype("S16"): the same text as str()
    assert [t.decode() for t in x.astype("S16")] == want


def _neighbours(x, k=3):
    """x and its k nearest float32 neighbours on each side, both signs, finite ones only."""
    b = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.int64)
    out = (b[:, None] + np.arange(-k, k + 1)[None, :]).ravel()
    out = out[(out >= 0) & (out <= F32_MAX_BITS)]
    out = np.unique(out).astype(np.uint32)
    return np.concatenate([out, out | 0x80000000]).view(np.float32)


# ---- the rules, pinned against numpy ------------------------------------------------------------------------------------
RULES = [
    (0.0, "0.0"), (-0.0, "-0.0"), (np.inf, "inf"), (-np.inf, "-inf"), (0.5, "0.5"), (-3.0, "-3.0"),
    (1234.5, "1234.5"), (999999.0, "999999.0"), (1e6, "1e+06"), (9999999.0, "9.999999e+06"), (1e7, "1e+07"),
    (1.5e8, "1.5e+08"), (1e-5, "1e-05"), (1e-4, "1e-04"), (float(np.float32(1.1754944e-38)), "1.1754944e-38"),
    (float(np.float32(3.4028235e38)), "3.4028235e+38"), (float(np.float32(1e-45)), "1e-45"),
]


@pytest.mark.parametrize("value,text", RULES)
def test_rules_hold_for_numpy_and_for_the_formatter(lib, value, text):
    assert str(np.float32(value)) == text
    assert _texts(lib, [value]) == [text]


def test_the_boundaries_lie_between_float32_values(lib):
    below = np.float32(1e-4)                       # 9.9999997e-05: the nearest float32 is below 1e-4
    above = np.nextafter(below, np.float32(1))
    assert float(below) < 1e-4 < float(above)
    assert _texts(lib, [below, above, -below, -above]) == ["1e-04", "0.000100000005", "-1e-04", "-0.000100000005"]
    top = np.nextafter(np.float32(1e6), np.float32(0))
    assert _texts(lib, [top, np.float32(1e6)]) == [str(top), "1e+06"] and "e" not in str(top)


def test_nan_is_nan_whatever_its_sign_and_payload(lib):
    payloads = [0x7FC00000, 0x7F800001, 0x7FBFFFFF, 0x7FFFFFFF, 0x7FC00001, 0x7FA5A5A5]
    x = _bits(payloads + [p | 0x80000000 for p in payloads])
    assert np.isnan(x).all()
    assert _texts(lib, x) == ["nan"] * len(x)
    _assert_numpy(lib, x)


def test_specials_and_subnormals(lib):
    subnormal_powers = _bits([1 << i for i in range(23)])                 # 2^-149 .. 2^-127
    largest_subnormal = _bits([0x007FFFFF])
    x = np.concatenate([np.float32([0.0, -0.0, np.inf, -np.inf]), subnormal_powers, largest_subnormal,
                        _bits([F32_MIN_BITS, F32_MAX_BITS])])
    _assert_numpy(lib, np.concatenate([x, -x]))
    _assert_numpy(lib, _neighbours(np.concatenate([subnormal_powers, largest_subnormal])))


def test_powers_of_two_and_ten_with_neighbours(lib):
    twos = np.ldexp(np.float32(1), np.arange(-149, 128)).astype(np.float32)
    tens = np.float32([10.0 ** k for k in range(-45, 39)])
    tens = tens[(tens != 0) & np.isfinite(tens)]
    _assert_numpy(lib, _neighbours(twos))
    _assert_numpy(lib, _neighbours(tens))


def test_both_sides_of_the_positional_range(lib):
    edges = np.float32([1e-4, 1e6])
    _assert_numpy(lib, _neighbours(edges, k=8))


def test_nine_digit_values(lib):
    rng = np.random.default_rng(9)
    x = _bits(rng.integers(0, 1 << 32, size=1 << 16, dtype=np.uint64))
    x = x[np.isfinite(x)]
    texts = [str(v) for v in x]
    digits = [len(t.split("e")[0].lstrip("-").replace(".", "").lstrip("0")) for t in texts]
    nine = x[np.array(digits) == 9]
    assert nine.size > 500
    _assert_numpy(lib, nine)


def test_seeded_random_bit_patterns(lib):
    """2^22 patterns against str() itself; the exhaustive sweep covers all 2^32."""
    rng = np.random.default_rng(20261017)
    x = _bits(rng.integers(0, 1 << 32, size=1 << 22, dtype=np.uint64))
    got, lens = format_floats(lib, x)
    want = np.array([str(v).encode() for v in x], dtype="S16")
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, [(hex(int(x[i].view(np.uint32))), got[i], want[i]) for i in bad[:10]]
    assert lens.max() <= 15


def test_selftest_refuses_bad_arguments(lib):
    assert lib.c2v_selftest_format_floats(None, -1, None, None) < 0
    assert b"c2v_selftest_format_floats" in lib.c2v_last_error(None)
    assert lib.c2v_selftest_format_floats(None, 0, None, None) == 0


# ---- lines ----------------------------------------------------------------------------------------------------------------
def _lines(lib, x, words=None):
    """The text the device writer produces, composed from the formatter's values as the kernel lays them out."""
    out = []
    for r, row in enumerate(np.asarray(x, dtype=np.float32)):
        out.append(("" if words is None else words[r] + " ") + " ".join(_texts(lib, row)) + "\n")
    return "".join(out)


def _matrices():
    rng = np.random.default_rng(3)
    for D in (1, 31, 32, 33, 384):
        yield "normal-%d" % D, rng.standard_normal((5, D)).astype(np.float32)
        sci = (rng.standard_normal((3, D)) * 10.0 ** rng.integers(-40, 38, size=(3, D))).astype(np.float32)
        sci[np.abs(sci) < 1e-38] = np.float32(1e-30)
        sci[(np.abs(sci) >= 1e-4) & (np.abs(sci) < 1e6)] = np.float32(-2.5e7)
        yield "scientific-%d" % D, sci
        nan = rng.standard_normal((3, D)).astype(np.float32)
        nan[0, 0] = np.nan
        nan[1, -1] = -np.nan
        nan[2, D // 2] = np.inf
        yield "nan-%d" % D, nan


@pytest.mark.parametrize("name,x", list(_matrices()), ids=[n for n, _ in _matrices()])
def test_line_layout_equals_the_host_writers(lib, name, x):
    from code2vec_b200.common import common
    from code2vec_b200.model_base import Code2VecModelBase
    if name.startswith("scientific"):
        assert all("e" in t for t in _texts(lib, x.ravel()))
    f = io.StringIO()
    Code2VecModelBase._write_code_vectors(None, f, x)
    assert _lines(lib, x) == f.getvalue()
    words = {i: w for i, w in enumerate(["<PAD>", "<OOV>", "get|x", "ü", "a,b", "x"][:x.shape[0]])}
    f = io.StringIO()
    common.save_word2vec_file(f, words, x)
    assert f.getvalue() == "%d %d\n" % x.shape + _lines(lib, x, words)


def test_word_prefixes_encode_and_assert_as_the_host_writer():
    from code2vec_b200.text_export import word_prefixes
    blob, off = word_prefixes({0: "a", 1: "ü", 2: ""}, 3, "utf-8")
    assert blob == "a ü  ".encode("utf-8") and off.tolist() == [0, 2, 5, 6]
    with pytest.raises(AssertionError):
        word_prefixes({0: "a", 2: "b"}, 3, "utf-8")


def test_device_text_flag():
    from code2vec_b200.text_export import device_text_flag
    assert device_text_flag({}) is False
    assert device_text_flag({"C2V_DEVICE_TEXT": "0"}) is False
    assert device_text_flag({"C2V_DEVICE_TEXT": ""}) is False
    assert device_text_flag({"C2V_DEVICE_TEXT": "1"}) is True
    for bad in ("2", "yes", "true", " 1"):
        with pytest.raises(ValueError, match="C2V_DEVICE_TEXT must be 0 or 1"):
            device_text_flag({"C2V_DEVICE_TEXT": bad})


def test_models_refuse_a_bad_switch(monkeypatch):
    from code2vec_b200.b200_keras_model import Code2VecModel as KerasModel
    from code2vec_b200.b200_model import Code2VecModel
    from code2vec_b200.config import Config
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    for cls, fw in ((Code2VecModel, "b200"), (KerasModel, "b200-keras")):
        cfg = Config(set_defaults=True)
        cfg.DL_FRAMEWORK = fw
        cfg.VERBOSE_MODE = 0
        monkeypatch.setenv("C2V_DEVICE_TEXT", "on")
        with pytest.raises(ValueError, match="C2V_DEVICE_TEXT must be 0 or 1"):
            cls(cfg)


def test_text_abi_is_declared_and_exported(lib):
    import ctypes
    import re
    from code2vec_b200 import engine as E
    from code2vec_b200.build import LIB_PATH
    header = open(E._build.PKG_DIR + "/../include/c2v_b200.h").read()
    so = ctypes.CDLL(LIB_PATH)
    for n in ("c2v_text_format_rows", "c2v_selftest_format_floats"):
        assert re.search(r"\b%s\(" % n, header), n
        assert n in E._SIGNATURES
        assert hasattr(so, n), n
    assert "#define C2V_TEXT_VALUE_BYTES 16" in header
