"""The sharded device reader (C2V_SHARDED_READER=1: device_reader.DeviceBatchReader with a ShareTransport) against the host
reader: every rank's batches are its slice of the host reader's batches, bit for bit; malformed files raise the host's
ValueError on every rank; the ranks upload the file's bytes once between them; and Code2VecModel.train() saves the host
path's checkpoint.  W = 2, 4 and 8 ranks run as threads on one GPU with a transport that shares raw device pointers
(CUDA IPC cannot open a handle in the process that made it); two processes on one or two GPUs use the real transport, a
gloo group and CUDA IPC."""
import os
import socket
import threading
import traceback

import numpy as np
import pytest

from code2vec_b200.path_context_reader import EstimatorAction, PathContextReader, chunk_ranges, share_range
from tests.test_gpu_device_reader import _Former, _assert_same, _odd_lines, _text, _write
from tests.test_reader_native import _random_lines

pytestmark = pytest.mark.gpu

JOIN_TIMEOUT_S = 300.0


class _Hub:
    """What the threads of one emulated group share: a barrier for the exchange and a handle -> pointer table."""

    def __init__(self, world, timeout=120.0):
        self.world = world
        self.barrier = threading.Barrier(world, timeout=timeout)
        self.slots = [None] * world
        self.table = {}
        self.lock = threading.Lock()


class _ThreadTransport:
    """device_reader.ShareTransport for ranks that are threads of one process: the exchange meets at the hub's barrier,
    and a stage's handle opens to its owner's own pointer."""

    def __init__(self, hub, rank):
        from code2vec_b200.engine import load_library
        self.hub, self.rank, self.world, self.lib = hub, rank, hub.world, load_library()
        self.allocs = 0

    def alloc(self, nbytes):
        import ctypes as C
        self.allocs += 1
        ptr, hbuf = C.c_void_p(), C.create_string_buffer(64)
        assert self.lib.c2v_ipc_alloc(0, nbytes, C.byref(ptr), hbuf) == 0
        with self.hub.lock:
            assert hbuf.raw not in self.hub.table
            self.hub.table[hbuf.raw] = ptr.value
        return ptr.value, hbuf.raw

    def free(self, ptr):
        with self.hub.lock:
            for k in [k for k, p in self.hub.table.items() if p == ptr]:
                del self.hub.table[k]
        assert self.lib.c2v_ipc_free(0, ptr) == 0

    def open(self, handle):
        with self.hub.lock:
            return self.hub.table[handle]

    def close(self, ptr):
        pass

    def gather(self, obj):
        self.hub.slots[self.rank] = obj
        self.hub.barrier.wait()
        out = list(self.hub.slots)
        self.hub.barrier.wait()
        return out

    def destroy(self):
        pass


def _reader(cfg, vs, seed, chunk):
    r = PathContextReader(vs, cfg, _Former(), EstimatorAction.Train, shuffle_seed=seed)
    if chunk:
        r.chunk_bytes = chunk
    return r


def _host_batches(cfg, vs, seed, chunk=None):
    r = PathContextReader(vs, cfg, _Former(), EstimatorAction.Train, use_native=True, shuffle_seed=seed)
    if chunk:
        r.chunk_bytes = chunk
    names = ("path_source_token_indices", "path_indices", "path_target_token_indices", "context_valid_mask", "target_index")
    return [tuple(np.array(getattr(b, n)) for n in names) for b in r.get_dataset()]


def _sharded_batches(cfg, vs, seed, world, chunk=None):
    """(per rank: batches as test_gpu_device_reader._device_batches gives them or None, per rank: the exception or None,
    per rank: bytes uploaded) of `world` ranks reading together as threads."""
    import torch
    from code2vec_b200.device_reader import DeviceBatchReader
    hub = _Hub(world)
    out, errs, up = [None] * world, [None] * world, [0] * world

    def body(r):
        try:
            torch.cuda.set_device(0)
            dr = DeviceBatchReader(_reader(cfg, vs, seed, chunk), torch.device("cuda", 0), world=world, rank=r,
                                   transport=_ThreadTransport(hub, r))
            got = []
            try:
                for b in dr:
                    b.wait()
                    got.append((b.rows, b.lo, b.hi, tuple(t.cpu().numpy() for t in b.tensors)))
                    b.release()
                up[r] = dr.h2d_bytes
            finally:
                dr.close()
            out[r] = got
        except BaseException as exc:           # noqa: B902 -- reported to the caller
            errs[r] = exc
            hub.barrier.abort()

    threads = [threading.Thread(target=body, args=(r,), daemon=True) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(JOIN_TIMEOUT_S)
    assert not any(t.is_alive() for t in threads), "a rank is still waiting"
    return out, errs, up


def _empty_shares(path, chunk, world):
    with open(path, "rb") as f:
        fd = f.fileno()
        return sum(s0 == s1 for a, b in chunk_ranges(fd, chunk) for s0, s1 in
                   (share_range(fd, a, b, world, r) for r in range(world)))


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("C", [13, 200])
@pytest.mark.parametrize("case", ["plain", "small_chunks", "epochs3_big_shuffle", "separate", "crlf_blank_no_eol"])
def test_every_rank_gets_its_slice_of_the_host_batches(tmp_path, world, C, case):
    n = 300 if C == 13 else 60
    lines = _random_lines(n, C, seed=C) + _odd_lines(C) * 3
    np.random.default_rng(1).shuffle(lines)
    kw = dict(C=C, batch=17)
    text = _text(lines)
    chunk = None
    if case == "small_chunks":
        chunk = 700                                             # many chunks, and lines longer than a chunk (C = 200)
    if case == "epochs3_big_shuffle":
        kw.update(epochs=3, shuffle=10 ** 6)                    # the pool holds the whole file: every batch is a drain
    if case == "separate":
        kw.update(separate=True)
    if case == "crlf_blank_no_eol":
        text = _text(lines, crlf=True, blanks=True, last_newline=False)
        chunk = 2000
    cfg, vs = _write(tmp_path, text, **kw)
    host = _host_batches(cfg, vs, seed=3, chunk=chunk)
    assert len(host[-1][4]) < kw["batch"] or case == "epochs3_big_shuffle"        # a short last batch
    out, errs, up = _sharded_batches(cfg, vs, seed=3, world=world, chunk=chunk)
    assert errs == [None] * world, errs
    for r in range(world):
        _assert_same(host, out[r], world=world, rank=r)
    # between them the ranks upload the file once per epoch, besides every rank's draw indices (8 bytes a row)
    drawn = 8 * sum(len(h[4]) for h in host)
    assert sum(u - drawn for u in up) == len(text) * kw.get("epochs", 1)
    if case == "small_chunks" and C == 200:
        assert _empty_shares(cfg.TRAIN_DATA_PATH_PREFIX + ".train.c2v", chunk, world) > 0


def test_java14m_sized_vocabularies_on_8_ranks(tmp_path):
    """A 1024-line batch against vocabularies of 1.3 M / 911 K / 261 K words, read by 8 ranks."""
    C, n_lines = 200, 2300
    rng = np.random.default_rng(0)
    n_tok, n_path, n_tgt = 1_300_000, 911_000, 261_000
    lines = []
    for _ in range(n_lines):
        k = int(rng.integers(60, C + 1))
        s = rng.integers(0, n_tok + 1000, size=(k, 2))
        p = rng.integers(0, n_path + 1000, size=k)
        lines.append(" ".join(["name|%d" % int(rng.integers(0, n_tgt + 100))] +
                              ["t%d,%d,t%d" % (a, 100 + b, c) for (a, c), b in zip(s, p)] + [""] * (C - k)))
    cfg, vs = _write(tmp_path, _text(lines), C=C, batch=1024, shuffle=500, n_tok=n_tok, n_path=n_path, n_tgt=n_tgt)
    host = _host_batches(cfg, vs, seed=11, chunk=1 << 20)
    assert len(host[0][4]) == 1024
    out, errs, _ = _sharded_batches(cfg, vs, seed=11, world=8, chunk=1 << 20)
    assert errs == [None] * 8, errs
    for r in range(8):
        _assert_same(host, out[r], world=8, rank=r)


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("bad", ["fields", "parts", "parts_and_fields", "short_lines", "after_blanks", "last_no_eol"])
def test_malformed_lines_raise_the_host_error_on_every_rank(tmp_path, world, bad):
    C = 6
    good = _random_lines(40, C, seed=2)
    lines = list(good)
    if bad == "fields":
        lines[17] = " ".join(lines[17].split(" ")[:-1])
        lines[30] = lines[30] + " "
    elif bad == "parts":
        lines[21] = " ".join(["name|1", "a,b,c,d"] + [""] * (C - 1))
    elif bad == "parts_and_fields":
        lines[9] = " ".join(["name|1", "a,b,c,d"] + [""] * C)
    elif bad == "short_lines":
        lines = lines[:2] + ["x"] * 400
    elif bad == "after_blanks":
        lines[25] = lines[25] + " extra"
    text = _text(lines, blanks=bad == "after_blanks", last_newline=bad != "last_no_eol")
    if bad == "last_no_eol":
        text += b" " + b"t1,100,t2"                   # the unterminated last line gains a field
    cfg, vs = _write(tmp_path, text, C=C, batch=4)
    cfg.READER_NUM_PARALLEL_BATCHES = 1               # the host then reports the lowest malformed line, as the device does
    with pytest.raises(ValueError) as host:
        _host_batches(cfg, vs, seed=1)
    _, errs, _ = _sharded_batches(cfg, vs, seed=1, world=world)
    for r in range(world):
        assert isinstance(errs[r], ValueError), (r, errs[r])
        assert str(errs[r]) == str(host.value)


class _OpenFails(_ThreadTransport):
    """A transport whose first open of a peer's stage fails: the rank fails after the exchange of chunk 0."""

    def open(self, handle):
        raise RuntimeError("opening a peer's stage failed")


@pytest.mark.parametrize("how", ["consumer_stops", "open_fails"])
def test_a_rank_that_leaves_after_an_exchange_stops_its_peers(tmp_path, how):
    """Rank 1 stops after an exchange: its consumer leaves after the first batch, or it fails to open a peer's stage.
    The other ranks learn it in their next exchange and raise, instead of waiting there for it."""
    import torch
    from code2vec_b200.device_reader import DeviceBatchReader
    world, C = 4, 13
    cfg, vs = _write(tmp_path, _text(_random_lines(400, C, seed=4)), C=C, batch=8, shuffle=8)
    hub = _Hub(world)
    errs, counts = [None] * world, [0] * world

    def body(r):
        try:
            torch.cuda.set_device(0)
            tr = _OpenFails(hub, r) if (how == "open_fails" and r == 1) else _ThreadTransport(hub, r)
            dr = DeviceBatchReader(_reader(cfg, vs, 1, 700), torch.device("cuda", 0), world=world, rank=r, transport=tr)
            try:
                for b in dr:
                    b.wait()
                    b.release()
                    counts[r] += 1
                    if how == "consumer_stops" and r == 1:
                        break
            finally:
                dr.close()
        except BaseException as exc:           # noqa: B902 -- reported to the test
            errs[r] = exc

    threads = [threading.Thread(target=body, args=(r,), daemon=True) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(JOIN_TIMEOUT_S)
    assert not any(t.is_alive() for t in threads), "a rank is still waiting"
    if how == "consumer_stops":
        assert errs[1] is None and counts[1] == 1
    else:
        assert isinstance(errs[1], RuntimeError) and "opening a peer's stage failed" in str(errs[1])
    for r in (0, 2, 3):
        assert isinstance(errs[r], RuntimeError) and "rank 1" in str(errs[r]), (r, errs[r])


def test_stages_grown_while_the_default_stream_is_busy(tmp_path):
    """Stages are grown mid-pass while every rank's consumer keeps the default stream busy, as training steps do: the zero
    fill of a new stage must land before the parse writes it.  A 10 KB line half-way through the file doubles the chunk
    window twice (it stays doubled), so the shares after it need four times the rows."""
    import torch
    from code2vec_b200.device_reader import DeviceBatchReader
    world, C = 4, 13
    lines = _random_lines(900, C, seed=6)
    lines.insert(500, " ".join(["name|1"] + ["t%s,100,t%s" % ("0" * 400, "0" * 400)] * C))
    cfg, vs = _write(tmp_path, _text(lines), C=C, batch=16, shuffle=32)
    chunk = 4096
    host = _host_batches(cfg, vs, seed=2, chunk=chunk)
    hub = _Hub(world)
    out, errs, transports = [None] * world, [None] * world, [_ThreadTransport(hub, r) for r in range(world)]

    def body(r):
        try:
            torch.cuda.set_device(0)
            a = torch.randn(2048, 2048, device="cuda")
            dr = DeviceBatchReader(_reader(cfg, vs, 2, chunk), torch.device("cuda", 0), world=world, rank=r,
                                   transport=transports[r])
            got = []
            try:
                for b in dr:
                    for _ in range(4):               # work queued on the default stream, not waited for
                        a = torch.tanh(a @ a * 1e-3)
                    b.wait()
                    got.append((b.rows, b.lo, b.hi, tuple(t.cpu().numpy() for t in b.tensors)))
                    b.release()
            finally:
                dr.close()
            out[r] = got
        except BaseException as exc:           # noqa: B902 -- reported to the test
            errs[r] = exc
            hub.barrier.abort()

    threads = [threading.Thread(target=body, args=(r,), daemon=True) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(JOIN_TIMEOUT_S)
    assert not any(t.is_alive() for t in threads), "a rank is still waiting"
    assert errs == [None] * world, errs
    assert all(t.allocs > 2 for t in transports), [t.allocs for t in transports]      # stages grew after the first two
    for r in range(world):
        _assert_same(host, out[r], world=world, rank=r)


# ---- Code2VecModel.train() with C2V_SHARDED_READER=1 ------------------------------------------------------------------------
@pytest.fixture
def _ten_target_rows(monkeypatch):
    """The toy dataset with a ninth method name, so that 4 ranks all hold target rows (as tests/test_gpu_multi_rank_model)."""
    import tests.test_gpu_model as toy
    monkeypatch.setattr(toy, "TARGETS", toy.TARGETS + ["make|copy"])


@pytest.mark.parametrize("world", [2, 4])
def test_train_saves_the_host_paths_checkpoint(tmp_path, monkeypatch, _ten_target_rows, world):
    import code2vec_b200.device_reader as DR
    from tests.test_gpu_device_reader import _train_logged
    from tests.test_gpu_model import _config, _make_dataset
    monkeypatch.chdir(tmp_path)
    prefix, _ = _make_dataset(tmp_path, n_train=101)
    hubs, made, lock = {}, [], threading.Lock()

    def make(device):
        import torch.distributed as dist
        with lock:
            hub = hubs.setdefault("hub", _Hub(dist.get_world_size()))
        t = _ThreadTransport(hub, dist.get_rank())
        made.append(t)
        return t
    monkeypatch.setattr(DR, "make_share_transport", make)
    out = {}
    for flag in ("0", "1"):
        save = str(tmp_path / ("reader" + flag) / "saved")
        make_cfg = lambda: _config(prefix, tmp_path, TRAIN_DATA_PATH_PREFIX=prefix, MODEL_SAVE_PATH=save, NUM_TRAIN_EPOCHS=5,
                                   NUM_BATCHES_TO_LOG_PROGRESS=3, SHUFFLE_BUFFER_SIZE=40, DROPOUT_KEEP_RATE=0.75)
        env = {"C2V_DEVICE_READER": flag, "C2V_SHARDED_READER": flag}
        out[flag] = _train_logged(monkeypatch, make_cfg, env, world)
    assert len(made) == world                         # the sharded run read through the transport on every rank
    (ckpt0, log0), (ckpt1, log1) = out["0"], out["1"]
    assert len(log0) >= 4 and log1 == log0
    assert ckpt1 == ckpt0


# ---- two processes, the real transport -----------------------------------------------------------------------------------
def _cfg(prefix, C, batch, shuffle):
    """test_gpu_device_reader._write's config for files it wrote already."""
    from code2vec_b200.config import Config
    cfg = Config(set_defaults=True)
    cfg.VERBOSE_MODE = 0
    cfg.TRAIN_DATA_PATH_PREFIX = prefix
    cfg.MAX_CONTEXTS = C
    cfg.TRAIN_BATCH_SIZE = batch
    cfg.NUM_TRAIN_EPOCHS = 1
    cfg.SHUFFLE_BUFFER_SIZE = shuffle
    cfg.SEPARATE_OOV_AND_PAD = False
    cfg.READER_NUM_PARALLEL_BATCHES = 3
    cfg.MAX_TOKEN_VOCAB_SIZE, cfg.MAX_PATH_VOCAB_SIZE, cfg.MAX_TARGET_VOCAB_SIZE = 10 ** 7, 10 ** 7, 10 ** 7
    return cfg


def _process_rank(rank, world, port, device, prefix, C, chunk, result):
    """One rank of a two-process run: the sharded reader through make_share_transport against the host reader."""
    try:
        import torch
        import torch.distributed as dist
        from code2vec_b200 import vocabularies as V
        from code2vec_b200.device_reader import DeviceBatchReader, make_share_transport
        torch.cuda.set_device(device)
        dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, world_size=world, rank=rank)
        try:
            cfg = _cfg(prefix, C, batch=32, shuffle=40)
            vs = V.Code2VecVocabs(cfg)
            host = _host_batches(cfg, vs, seed=5, chunk=chunk)
            transport = make_share_transport(device)
            dr = DeviceBatchReader(_reader(cfg, vs, 5, chunk), torch.device("cuda", device), world=world, rank=rank,
                                   transport=transport)
            got = []
            try:
                for b in dr:
                    b.wait()
                    got.append((b.rows, b.lo, b.hi, tuple(t.cpu().numpy() for t in b.tensors)))
                    b.release()
                peer = dr.peer_bytes
            finally:
                dr.close()
                transport.destroy()
            _assert_same(host, got, world=world, rank=rank)
            assert peer > 0
        finally:
            dist.destroy_process_group()
        with open(result, "w") as f:
            f.write("ok")
    except BaseException:                      # noqa: B902 -- reported through the result file
        with open(result, "w") as f:
            f.write(traceback.format_exc())


@pytest.mark.parametrize("gpus", [1, 2])
def test_two_processes_over_cuda_ipc(tmp_path, gpus):
    import multiprocessing as mp
    import torch
    if gpus > torch.cuda.device_count():
        pytest.skip("needs %d GPUs" % gpus)
    C = 13
    lines = _random_lines(400, C, seed=9) + _odd_lines(C) * 2
    cfg, _ = _write(tmp_path, _text(lines), C=C, batch=32, shuffle=40)
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    results = [str(tmp_path / ("rank%d.txt" % r)) for r in range(2)]
    procs = [ctx.Process(target=_process_rank, args=(r, 2, port, r % gpus, cfg.TRAIN_DATA_PATH_PREFIX, C, 1500, results[r]))
             for r in range(2)]
    for p in procs:
        p.start()
    try:
        for p in procs:
            p.join(JOIN_TIMEOUT_S)
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(30)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    for r in results:
        with open(r) as f:
            assert f.read() == "ok"
