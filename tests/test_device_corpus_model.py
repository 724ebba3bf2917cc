"""The host side of `--score_names` and `--nearest` on the GPU (DESIGN.md §6o) that needs no GPU: the output file that
appears only once it is complete, the evaluation route's start-up line, and the command line's choice of route."""
import os

import pytest

from code2vec_b200 import __main__ as cli
from code2vec_b200.corpus_text import atomic_output
from code2vec_b200.device_reader import evaluation_route_line


def test_atomic_output_renames_a_complete_file(tmp_path):
    path = str(tmp_path / "x.name_scores")
    with atomic_output(path) as f:
        f.write(b"a\tb\n")
        assert not os.path.exists(path)
    assert open(path, "rb").read() == b"a\tb\n"
    assert os.listdir(tmp_path) == ["x.name_scores"]


def test_atomic_output_leaves_no_file_when_the_block_raises(tmp_path):
    path = str(tmp_path / "x.nearest")
    with pytest.raises(UnicodeDecodeError):
        with atomic_output(path) as f:
            f.write(b"partial\n")
            b"\xff".decode("utf-8")
    assert os.listdir(tmp_path) == []
    with open(path, "wb") as f:                        # an earlier file stays as it was
        f.write(b"old\n")
    with pytest.raises(ValueError):
        with atomic_output(path) as f:
            f.write(b"new\n")
            raise ValueError("malformed line")
    assert open(path, "rb").read() == b"old\n"
    assert os.listdir(tmp_path) == ["x.nearest"]


def test_atomic_output_of_nothing_is_an_empty_file(tmp_path):
    path = str(tmp_path / "empty.name_scores")
    with atomic_output(path):
        pass
    assert open(path, "rb").read() == b""


def test_evaluation_route_line_names_both_commands():
    on, off = evaluation_route_line(True), evaluation_route_line(False)
    assert on.startswith("b200 backend evaluation: ") and on.endswith("(C2V_DEVICE_EVAL=1)")
    assert off.endswith("(C2V_DEVICE_EVAL=0)")
    for line in (on, off):
        assert "--score_names" in line and "--nearest" in line and "evaluate()" in line
    assert "GPU" in on and "GPU" not in off


class _DeviceModel:
    device_eval = True

    def __init__(self):
        self.calls = []

    def write_name_scores_device(self, path):
        self.calls.append(("scores", path))
        return path + ".name_scores"

    def write_nearest_device(self, path, topn):
        self.calls.append(("nearest", path, topn))
        return path + ".nearest"

    def score_names(self, path):
        raise AssertionError("the device route formats on the GPU")

    nearest_code_vectors = score_names


def test_command_line_takes_the_device_route_when_the_model_has_it():
    m = _DeviceModel()
    assert cli.write_name_scores(m, "F.c2v") == "F.c2v.name_scores"
    assert cli.write_nearest(m, "F.c2v", 7) == "F.c2v.nearest"
    assert m.calls == [("scores", "F.c2v"), ("nearest", "F.c2v", 7)]
