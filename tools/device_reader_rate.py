#!/usr/bin/env python
"""The training reader alone, on the GPU and on the host: lines/s of DeviceBatchReader (file -> device batches, the
device synchronised at the end) and of PathContextReader's native path (file -> host batches), over the synthetic
java14m-shaped `.c2v` file of tools/reader_rate.py, with that tool's vocabulary sizes and with java14m's (1.3 M tokens,
911 K paths, 261 K targets).  Also reports the device memory the reader holds, the card's name and power limit and the
host's core count.  `--profile` runs one more device pass under torch.profiler and reports the reader's kernel time per
batch.  Prints one JSON line per vocabulary size.  Writes only to a temporary directory."""
import json
import os
import pickle
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def _dataset(tmp, n_lines, C, n_tok, n_path, n_tgt):
    prefix = os.path.join(tmp, "syn%d" % n_tok)
    rng = np.random.default_rng(0)
    toks = ["tok%d" % i for i in range(n_tok)]
    paths = [str(1000003 * i % 2147483647 - 1073741823) for i in range(n_path)]
    tgts = ["do|thing%d" % i for i in range(n_tgt)]
    with open(prefix + ".train.c2v", "w") as f:
        for _ in range(n_lines):
            k = int(rng.integers(60, C + 1))
            s = rng.integers(0, n_tok, size=(k, 2))
            p = rng.integers(0, n_path, size=k)
            f.write(" ".join([tgts[int(rng.integers(0, n_tgt))]] + ["%s,%s,%s" % (toks[a], paths[b], toks[c])
                                                                     for (a, c), b in zip(s, p)] + [""] * (C - k)) + "\n")
    with open(prefix + ".dict.c2v", "wb") as f:
        for words in (toks, paths, tgts):
            pickle.dump({w: 2 for w in words}, f)
        pickle.dump(n_lines, f)
    return prefix


def run(tmp, n_tok, n_path, n_tgt, n_lines=65536, C=200, threads=16, batch=1024, profile=False):
    import torch
    from code2vec_b200.b200_model import _TrainInputFormer
    from code2vec_b200.config import Config
    from code2vec_b200.device_reader import DeviceBatchReader
    from code2vec_b200.path_context_reader import EstimatorAction, PathContextReader
    from code2vec_b200.vocabularies import Code2VecVocabs
    prefix = _dataset(tmp, n_lines, C, n_tok, n_path, n_tgt)
    cfg = Config(set_defaults=True)
    cfg.VERBOSE_MODE = 0
    cfg.DL_FRAMEWORK = "b200"
    cfg.TRAIN_DATA_PATH_PREFIX = prefix
    cfg.NUM_TRAIN_EPOCHS = 1
    cfg.TRAIN_BATCH_SIZE = batch
    cfg.READER_NUM_PARALLEL_BATCHES = threads
    cfg.MAX_TOKEN_VOCAB_SIZE, cfg.MAX_PATH_VOCAB_SIZE, cfg.MAX_TARGET_VOCAB_SIZE = n_tok, n_path, n_tgt
    vocabs = Code2VecVocabs(cfg)
    dev = torch.device("cuda", 0)
    reader = lambda: PathContextReader(vocabs=vocabs, model_input_tensors_former=_TrainInputFormer(), config=cfg,
                                       estimator_action=EstimatorAction.Train, shuffle_seed=1)
    device_rates, host_rates, held, setup_s, batches = [], [], 0, [], 0
    for _ in range(3):                                   # alternating; the first pass also warms the page cache
        t0 = time.time()
        rows = sum(int(b[0].shape[0]) for b in reader().get_dataset())
        host_rates.append(rows / (time.time() - t0))
        t0 = time.time()
        dr = DeviceBatchReader(reader(), dev)
        torch.cuda.synchronize()
        setup_s.append(time.time() - t0)                 # vocabulary upload and handle creation
        t0 = time.time()
        rows = batches = 0
        for b in dr:
            b.wait()
            rows += b.rows
            batches += 1
            b.release()
        torch.cuda.synchronize()
        device_rates.append(rows / (time.time() - t0))
        held = dr.device_bytes()
        dr.close()
    out = {"what": "training reader alone: DeviceBatchReader (file -> device batches) vs PathContextReader (file -> host "
                   "batches)", "card_and_power_limit": _card(), "host_cores": os.cpu_count(), "lines": n_lines,
           "contexts_per_line": C, "batch": batch, "host_reader_threads": threads,
           "vocab_words": [n_tok, n_path, n_tgt], "device_lines_per_s": [round(r) for r in device_rates],
           "host_lines_per_s": [round(r) for r in host_rates], "best_device_lines_per_s": round(max(device_rates)),
           "best_host_lines_per_s": round(max(host_rates)), "device_reader_setup_s": [round(s, 2) for s in setup_s],
           "device_bytes_held": held, "batches": batches}
    if profile:
        from torch.profiler import ProfilerActivity, profile as prof
        dr = DeviceBatchReader(reader(), dev)
        with prof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
            for b in dr:
                b.wait()
                b.release()
            torch.cuda.synchronize()
        dr.close()
        kernels = {}
        for e in p.key_averages():
            if e.device_type.name == "CUDA" or getattr(e, "self_device_time_total", 0) > 0:
                us = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)
                if us > 0:
                    kernels[e.key[:60]] = round(us / max(batches, 1), 1)
        out["profile_us_per_batch"] = dict(sorted(kernels.items(), key=lambda kv: -kv[1])[:14])
    return out


class _SoloTransport:
    """Rank 0 of a sharded reader of `world` ranks in one process: the exchange parses the other ranks' shares of the
    chunk itself, with a second reader handle into stages of this device, and hands their statuses back as the peers
    would.  The time it spends on that is kept apart (peer_s), so that rank 0's own path can be timed."""

    def __init__(self, lib, world, C, make_handle):
        import torch
        self.lib, self.world, self.C, self.h = lib, world, C, make_handle()
        self.stream = torch.cuda.Stream()
        self.table, self.stages, self.chunk, self.peer_s = {}, {}, None, 0.0

    def alloc(self, nbytes):
        import ctypes as C
        ptr, hbuf = C.c_void_p(), C.create_string_buffer(64)
        assert self.lib.c2v_ipc_alloc(0, nbytes, C.byref(ptr), hbuf) == 0
        self.table[hbuf.raw] = ptr.value
        return ptr.value, hbuf.raw

    def free(self, ptr):
        assert self.lib.c2v_ipc_free(0, ptr) == 0

    def open(self, handle):
        return self.table[handle]

    def close(self, ptr):
        pass

    def gather(self, obj):
        if obj is None or self.chunk is None:
            return [obj] + [None] * (self.world - 1)
        import ctypes as C
        import torch
        from code2vec_b200.engine import c2v_reader_share_status
        from code2vec_b200.path_context_reader import pread_into, share_range
        t0 = time.perf_counter()
        fd, a, b, k = self.chunk
        out = [obj]
        for r in range(1, self.world):
            s0, s1 = share_range(fd, a, b, self.world, r)
            n = s1 - s0
            rows, handle = n // (self.C + 1) + 1, None
            st = self.stages.get((r, k % 2))
            if st is None or st[1] < rows:
                if st is not None:
                    self.free(st[0])
                ptr, handle = self.alloc(int(self.lib.c2v_reader_stage_bytes(self.C, rows)))
                self.stages[(r, k % 2)] = st = (ptr, rows)
            text = torch.empty(max(n, 1), dtype=torch.uint8)
            pread_into(fd, text.numpy()[:n], s0)
            dev = text.cuda()
            status = c2v_reader_share_status()
            assert self.lib.c2v_reader_parse_share(self.h, dev.data_ptr(), n, b - a, st[0], st[1], C.byref(status),
                                                   self.stream.cuda_stream) == 0
            out.append((tuple(getattr(status, f) for f, _ in status._fields_), handle, None))
        torch.cuda.synchronize()
        self.peer_s += time.perf_counter() - t0
        return out

    def destroy(self):
        for ptr, _ in self.stages.values():
            self.free(ptr)
        self.lib.c2v_reader_destroy(self.h)


def run_world(tmp, world, n_tok=1300000, n_path=911000, n_tgt=261000, n_lines=65536, C=200, batch=1024):
    """Rank 0 of a sharded device reader of `world` ranks (world 1: the unsharded reader), timed per phase of its own
    path: share read, upload, share parse, exchange (local here), assembly + commit, draws."""
    import ctypes as C_
    import torch
    import code2vec_b200.device_reader as DR
    from code2vec_b200.b200_model import _TrainInputFormer
    from code2vec_b200.config import Config
    from code2vec_b200.path_context_reader import EstimatorAction, PathContextReader
    from code2vec_b200.vocabularies import Code2VecVocabs
    prefix = _dataset(tmp, n_lines, C, n_tok, n_path, n_tgt)
    cfg = Config(set_defaults=True)
    cfg.VERBOSE_MODE = 0
    cfg.DL_FRAMEWORK = "b200"
    cfg.TRAIN_DATA_PATH_PREFIX = prefix
    cfg.NUM_TRAIN_EPOCHS = 1
    cfg.TRAIN_BATCH_SIZE = batch
    cfg.MAX_TOKEN_VOCAB_SIZE, cfg.MAX_PATH_VOCAB_SIZE, cfg.MAX_TARGET_VOCAB_SIZE = n_tok, n_path, n_tgt
    vocabs = Code2VecVocabs(cfg)
    dev = torch.device("cuda", 0)
    reader = lambda: PathContextReader(vocabs=vocabs, model_input_tensors_former=_TrainInputFormer(), config=cfg,
                                       estimator_action=EstimatorAction.Train, shuffle_seed=1)
    file_bytes = os.path.getsize(prefix + ".train.c2v")

    def one_pass(timed):
        phases = {"read": 0.0, "upload": 0.0, "parse": 0.0, "exchange": 0.0, "assemble_commit": 0.0, "draws": 0.0}
        dr = DR.DeviceBatchReader(reader(), dev, world=world, rank=0)
        solo = None
        if world > 1:
            def make_handle():
                h = C_.c_void_p()
                assert dr.lib.c2v_reader_create(dr.C, *[C_.byref(s) for s in dr._structs], 0, C_.byref(h)) == 0
                return h
            solo = _SoloTransport(dr.lib, world, dr.C, make_handle)
            dr.transport = solo
        lib = dr.lib

        def clock(name, fn, sync=None):
            def wrapped(*a):
                t0 = time.perf_counter()
                r = fn(*a)
                if sync is not None:
                    sync()
                phases[name] += time.perf_counter() - t0
                return r
            return wrapped
        if timed:
            read, parse_sharded, exchange, draw = DR.pread_into, dr._parse_sharded, dr._exchange, dr._draw
            DR.pread_into = clock("read", read)

            def parse_share(*a):
                t0 = time.perf_counter()
                dr.copy_stream.synchronize()
                phases["upload"] += time.perf_counter() - t0
                return clock("parse", lib.c2v_reader_parse_share)(*a)

            class _Lib:
                def __getattr__(self, name):
                    return getattr(lib, name)
            dr.lib = _Lib()
            dr.lib.c2v_reader_parse_share = parse_share
            dr.lib.c2v_reader_commit_shares = clock("assemble_commit", lib.c2v_reader_commit_shares)
            dr._exchange = clock("exchange", exchange)
            dr._draw = clock("draws", draw, sync=dr.stream.synchronize)
        if solo is not None:
            inner = dr._parse_sharded

            def parse_sharded(fd, a, b, k):
                solo.chunk = (fd, a, b, k)
                return inner(fd, a, b, k)
            dr._parse_sharded = parse_sharded
        t0 = time.perf_counter()
        rows = chunks = 0
        try:
            for bt in dr:
                bt.wait()
                rows += bt.rows
                bt.release()
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            held = dr.device_bytes()
            text = dr.h2d_bytes
        finally:
            if timed:
                DR.pread_into = read
            dr.close()
            if solo is not None:
                solo.destroy()
        peer_s = solo.peer_s if solo is not None else 0.0
        if timed:
            phases["exchange"] -= peer_s
        return rows, wall - peer_s, phases, held, text

    one_pass(False)                                     # warms the page cache and the library
    rows, wall, _, held, text = one_pass(False)
    _, _, phases, _, _ = one_pass(True)
    chunks = max(1, -(-file_bytes // (16 << 20)))
    return {"what": "sharded device reader, rank 0 of %d timed alone (peers' stages are parsed by the same process, "
                    "untimed, and read from local memory, not over NVLink): a per-rank estimate" % world,
            "card_and_power_limit": _card(), "world": world, "lines": n_lines, "contexts_per_line": C, "batch": batch,
            "vocab_words": [n_tok, n_path, n_tgt], "file_bytes": file_bytes, "chunks": chunks,
            "rank0_lines_per_s": round(rows / wall), "rank0_text_and_index_bytes_uploaded": text,
            "device_bytes_held": held,
            # the unsharded reader (world 1) is timed for its draws only: its read, upload and parse are not instrumented
            "rank0_ms_per_chunk": {k: round(1e3 * v / chunks, 2) for k, v in phases.items()
                                   if world > 1 or k == "draws"},
            "not_timed": [] if world > 1 else ["read", "upload", "parse"],
            # no collective runs here: the exchange is a local call that parses the peers' shares (subtracted)
            "exchange_is_local": world > 1}


def main():
    tmp = tempfile.mkdtemp()
    try:
        if "--world" in sys.argv:
            worlds = [int(w) for w in sys.argv[sys.argv.index("--world") + 1].split(",")]
            for w in worlds:
                if w not in (1, 2, 4, 8):
                    raise SystemExit("--world takes 1, 2, 4 or 8 (comma-separated)")
                print(json.dumps(run_world(tmp, w)), flush=True)
            return
        prof = "--profile" in sys.argv
        print(json.dumps(run(tmp, 200000, 150000, 30000, profile=prof)), flush=True)         # tools/reader_rate.py's sizes
        print(json.dumps(run(tmp, 1300000, 911000, 261000, profile=prof)), flush=True)       # java14m's
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
