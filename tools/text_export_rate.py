#!/usr/bin/env python
"""The host writers of `.vectors` and word2vec files against the device ones (C2V_DEVICE_TEXT=0 vs 1, DESIGN.md §6f),
in one process, alternating, with the bytes of every pair of files checked equal:
  vectors  : rows/s of `.vectors` text at D = 384 (model_base._write_code_vectors vs DeviceTextWriter), seeded rows;
  evaluate : the whole Code2VecModel.evaluate() with EXPORT_CODE_VECTORS on tools/eval_rate.py's synthetic java14m-shaped
             test file at java14m model dims, both evaluation routes (C2V_DEVICE_EVAL=0 and 1), each with the switch at
             0 and at 1;
  word2vec : --save_w2v (1,301,139 x 128) and --save_t2v (261,247 x 384) tables on the device; the device writer writes
             the whole table, the host writer (common.save_word2vec_file) the first --w2v_host_rows rows of each, so its
             time for the whole table is extrapolated from its rate (reported as such).
Prints one JSON line with the card's name and power limit and the host's core count.  Writes only to a temporary
directory."""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from eval_rate import JAVA14M, _card, _dataset  # noqa: E402


def _timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def _vectors(tmp, rows, passes):
    import torch
    from code2vec_b200.model_base import Code2VecModelBase
    from code2vec_b200.text_export import write_lines
    g = torch.Generator(device="cuda")
    g.manual_seed(3)
    code = torch.tanh(torch.randn((rows, 384), device="cuda", generator=g))     # code vectors are tanh outputs
    host_path, dev_path = os.path.join(tmp, "host.vectors"), os.path.join(tmp, "dev.vectors")

    def host():
        with open(host_path, "w") as f:
            Code2VecModelBase._write_code_vectors(None, f, code.cpu().numpy())

    def dev():
        with open(dev_path, "wb") as f:
            return write_lines(f, code)

    host_s, dev_s = [], []
    dev()                                                    # warm-up: module load, buffers
    for _ in range(passes):
        host_s.append(_timed(host)[1])
        w, s = _timed(dev)
        dev_s.append(s)
        assert open(host_path, "rb").read() == open(dev_path, "rb").read(), ".vectors differ"
    return {"rows": rows, "D": 384, "text_mb": round(os.path.getsize(dev_path) / 1e6, 1),
            "host_s": [round(s, 3) for s in host_s], "device_s": [round(s, 4) for s in dev_s],
            "host_rows_per_s": round(rows / min(host_s)), "device_rows_per_s": round(rows / min(dev_s)),
            "device_writer": w.report(), "bytes_identical": True}


def _evaluate(tmp, lines):
    from code2vec_b200.b200_model import Code2VecModel
    from code2vec_b200.config import Config
    T, P, Y = JAVA14M
    prefix = _dataset(tmp, lines, 200, T - 2, P - 2, Y - 1)
    cfg = Config(set_defaults=True)
    cfg.VERBOSE_MODE = 0
    cfg.DL_FRAMEWORK = "b200"
    cfg.TRAIN_DATA_PATH_PREFIX = prefix
    cfg.TEST_DATA_PATH = prefix + ".test.c2v"
    cfg.EXPORT_CODE_VECTORS = True
    cfg.MAX_TOKEN_VOCAB_SIZE, cfg.MAX_PATH_VOCAB_SIZE, cfg.MAX_TARGET_VOCAB_SIZE = T, P, Y
    os.environ.setdefault("C2V_SEED", "7")
    os.environ["C2V_DEVICE_EVAL"] = os.environ["C2V_DEVICE_TEXT"] = "0"
    model = Code2VecModel(cfg)
    out = {}
    try:
        def run(device_eval, device_text):
            model._device_eval, model._device_text = device_eval, device_text
            res, s = _timed(model.evaluate)
            return res, s, open(cfg.TEST_DATA_PATH + ".vectors", "rb").read()

        run(True, True)                                     # warm-up: page cache, tables, reader and text buffers
        for device_eval in (False, True):
            (r0, s0, v0), (r1, s1, v1) = run(device_eval, False), run(device_eval, True)
            assert str(r0) == str(r1) and v0 == v1, ".vectors differ"
            out["device_eval_%d" % device_eval] = {"text_0_s": round(s0, 3), "text_1_s": round(s1, 3),
                                                    "vectors_mb": round(len(v0) / 1e6, 1), "bytes_identical": True}
        out["lines"] = lines
    finally:
        model.close_session()
    return out


def _word2vec(tmp, host_rows):
    import torch
    from code2vec_b200 import text_export
    from code2vec_b200.common import common
    T, _, Y = JAVA14M
    out = {}
    for name, n, D in (("save_w2v", T + 2, 128), ("save_t2v", Y + 1, 384)):
        g = torch.Generator(device="cuda")
        g.manual_seed(n)
        table = torch.empty((n, D), device="cuda").uniform_(-0.1, 0.1, generator=g)
        words = {i: "w%d" % i for i in range(n)}
        dev_path, host_path = os.path.join(tmp, name + ".dev"), os.path.join(tmp, name + ".host")

        def dev():
            with open(dev_path, "w") as f:
                return text_export.save_word2vec_file(f, words, table)

        def host():
            with open(host_path, "w") as f:
                common.save_word2vec_file(f, words, table[:host_rows].cpu().numpy())

        w, dev_s = _timed(dev)
        _, host_s = _timed(host)
        with open(dev_path, "rb") as f:
            f.readline()
            head = b"".join(f.readline() for _ in range(host_rows))
        with open(host_path, "rb") as f:
            f.readline()
            assert f.read() == head, "%s rows differ" % name
        out[name] = {"rows": n, "D": D, "device_s": round(dev_s, 3), "device_writer": w.report(),
                     "host_rows_timed": host_rows, "host_s_for_those": round(host_s, 3),
                     "host_s_whole_table_extrapolated": round(host_s * n / host_rows, 1), "bytes_identical_rows": host_rows}
        del table
        os.remove(dev_path)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=16384)
    ap.add_argument("--passes", type=int, default=2)
    ap.add_argument("--lines", type=int, default=65536)
    ap.add_argument("--w2v_host_rows", type=int, default=32768)
    ap.add_argument("--skip", default="", help="comma-separated parts to skip: vectors, evaluate, word2vec")
    a = ap.parse_args()
    skip = set(filter(None, a.skip.split(",")))
    tmp = tempfile.mkdtemp(prefix="c2v_text_rate_")
    cwd = os.getcwd()
    out = {"what": "host (C2V_DEVICE_TEXT=0) vs device (=1) text writers, one process, alternating",
           "card_and_power_limit": _card(), "host_cores": os.cpu_count()}
    try:
        os.chdir(tmp)                                       # evaluate() writes log.txt in the working directory
        if "vectors" not in skip:
            out["vectors"] = _vectors(tmp, a.rows, a.passes)
        if "evaluate" not in skip:
            out["evaluate"] = _evaluate(tmp, a.lines)
        if "word2vec" not in skip:
            out["word2vec"] = _word2vec(tmp, a.w2v_host_rows)
    finally:
        os.chdir(cwd)
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
