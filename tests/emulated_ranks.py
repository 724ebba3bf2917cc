"""Several ranks of a data-parallel run emulated on one device, in one process.

`run_ranks(world, fn)` runs fn(rank) on `world` threads.  `EmulatedGroup.install(monkeypatch)` replaces the part of
torch.distributed that code2vec_b200/trainer.py and PathAttentionEngine.enable_table_sharding call with collectives
done in software over the threads' tensors, and `IpcProxy` stands in for CUDA IPC, which cannot open a handle made in
the same process.  The row-sharded tables, their peer pointers and every kernel are then exactly what a multi-GPU run
launches; only the transport differs.

The fake collectives are more strongly ordered than NCCL's: each one synchronises the device on entry, exchanges the
inputs behind a barrier, computes the same fp32 result on every rank in rank order, and waits on a second barrier before
any rank writes its output (so an in-place all-reduce never overwrites an input a peer still reads).  Every kernel of
every rank issued before a collective has therefore finished when it returns.  Races that only NCCL's weaker ordering
could expose are not covered here.  Test infrastructure only.
"""
from __future__ import annotations

import contextlib
import threading

BARRIER_TIMEOUT_S = 120.0


class ReduceOp:
    SUM = "sum"
    AVG = "avg"


class _Done:
    """What an async_op=True collective returns: the work is complete already."""

    def wait(self):
        return True


def run_ranks(world, fn, group=None):
    """fn(rank) on `world` threads (rank set in `group`'s thread-local state); re-raises the first exception in the
    caller.  A rank that raises aborts `group`'s barrier, so ranks waiting in a collective fail instead of hanging."""
    errors = []
    lock = threading.Lock()

    def body(r):
        try:
            if group is not None:
                group._local.rank = r
            fn(r)
        except BaseException as exc:          # noqa: B902 -- re-raised in the caller
            with lock:
                errors.append((r, exc))
            if group is not None:
                group.barrier.abort()

    threads = [threading.Thread(target=body, args=(r,), name="rank%d" % r, daemon=True) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errors:
        # the first failure is the cause; the BrokenBarrierErrors of the other ranks follow from it
        primary = [e for e in errors if not isinstance(e[1], threading.BrokenBarrierError)] or errors
        raise primary[0][1]


class EmulatedGroup:
    """One process group of `world` emulated ranks (see the module docstring)."""

    def __init__(self, world, timeout=BARRIER_TIMEOUT_S):
        self.world = int(world)
        self.barrier = threading.Barrier(self.world, timeout=timeout)
        self._local = threading.local()
        self._slots = [None] * self.world
        self._calls = [dict() for _ in range(self.world)]      # per rank: collective name -> calls so far
        self._faults = {}                                      # (name, n) -> factor

    # ---- rank bookkeeping ------------------------------------------------------------------------------------------
    @property
    def rank(self):
        r = getattr(self._local, "rank", None)
        if r is None:
            raise RuntimeError("not inside an emulated rank (run_ranks or as_rank)")
        return r

    @contextlib.contextmanager
    def as_rank(self, r):
        """The calling thread acts as rank `r` (for set-up that needs get_rank but no collective)."""
        old = getattr(self._local, "rank", None)
        self._local.rank = r
        try:
            yield
        finally:
            self._local.rank = old

    def fault(self, name, n, factor):
        """Scale the result of the n-th (1-based) call of collective `name` by `factor`, on every rank."""
        self._faults[(name, int(n))] = float(factor)

    # ---- the collectives -------------------------------------------------------------------------------------------
    def _sync(self, *tensors):
        for t in tensors:
            if getattr(t, "is_cuda", False):
                import torch
                torch.cuda.synchronize(t.device)
                return

    def _wait(self):
        self.barrier.wait()

    def _collective(self, name, inp, combine, write, out):
        """Exchange `inp`, compute combine([inputs in rank order]) on every rank, then write(result) into `out`."""
        r = self.rank
        calls = self._calls[r]
        calls[name] = n = calls.get(name, 0) + 1
        self._sync(inp, out)
        self._slots[r] = inp
        self._wait()
        res = combine(list(self._slots))
        factor = self._faults.get((name, n))
        if factor is not None:
            res = res * factor
        self._sync(res)
        self._wait()                      # nobody writes an output before every rank has read every input
        write(res)
        self._sync(out)
        self._wait()                      # the slots are reused by the next collective
        self._slots[r] = None
        return _Done()

    @staticmethod
    def _sum(parts, op):
        acc = parts[0].float().clone()
        for p in parts[1:]:
            acc += p.float()
        if op == ReduceOp.AVG:
            acc /= len(parts)
        elif op != ReduceOp.SUM:
            raise NotImplementedError("reduce op %r" % (op,))
        return acc

    def all_reduce(self, tensor, op=ReduceOp.SUM, group=None, async_op=False):
        return self._collective("all_reduce", tensor, lambda ps: self._sum(ps, op), tensor.copy_, tensor)

    def reduce_scatter_tensor(self, output, input, op=ReduceOp.SUM, group=None, async_op=False):
        n, r = output.numel(), self.rank
        assert input.numel() == n * self.world, (input.shape, output.shape)
        return self._collective("reduce_scatter_tensor", input,
                                lambda ps: self._sum([p.reshape(-1)[r * n:(r + 1) * n] for p in ps], op),
                                lambda res: output.copy_(res.view(output.shape)), output)

    def all_gather_into_tensor(self, output_tensor, input_tensor, group=None, async_op=False):
        assert output_tensor.numel() == input_tensor.numel() * self.world
        import torch
        return self._collective("all_gather_into_tensor", input_tensor,
                                lambda ps: torch.cat([p.reshape(-1) for p in ps]),
                                lambda res: output_tensor.copy_(res.view(output_tensor.shape).to(output_tensor.dtype)),
                                output_tensor)

    def all_gather_object(self, object_list, obj, group=None):
        r = self.rank
        self._slots[r] = obj
        self._wait()
        object_list[:] = list(self._slots)
        self._wait()
        self._slots[r] = None

    def barrier_(self, group=None, async_op=False, device_ids=None):
        import torch
        if torch.cuda.is_available() and torch.cuda.is_initialized():
            torch.cuda.synchronize()
        self._wait()
        return _Done() if async_op else None

    # ---- installation ----------------------------------------------------------------------------------------------
    def install(self, monkeypatch):
        """Replace torch.distributed's entry points with this group's (undone with `monkeypatch`)."""
        import torch.distributed as dist
        world = self.world
        fakes = dict(is_available=lambda: True, is_initialized=lambda: True,
                     get_world_size=lambda group=None: world, get_rank=lambda group=None: self.rank,
                     get_backend=lambda group=None: "nccl", ReduceOp=ReduceOp,
                     all_reduce=self.all_reduce, reduce_scatter_tensor=self.reduce_scatter_tensor,
                     all_gather_into_tensor=self.all_gather_into_tensor, all_gather_object=self.all_gather_object,
                     barrier=self.barrier_)
        for name, fn in fakes.items():
            monkeypatch.setattr(dist, name, fn, raising=False)
        return self


class IpcProxy:
    """The engine library with CUDA IPC replaced by a handle -> pointer table shared by the emulated ranks: a handle
    opens to the owner's own pointer, closing it is a no-op, and the owner's c2v_ipc_free releases the memory.  Close
    the engines only once every rank is done with them."""

    def __init__(self, lib, table):
        self._lib = lib
        self._table = table

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def c2v_ipc_alloc(self, device, nbytes, ptr_ref, handle_buf):
        rc = self._lib.c2v_ipc_alloc(device, nbytes, ptr_ref, handle_buf)
        if rc == 0:
            key = bytes(handle_buf.raw)
            assert key not in self._table, "two live allocations share an IPC handle"
            self._table[key] = ptr_ref._obj.value
        return rc

    def c2v_ipc_open(self, device, handle, ptr_ref):
        ptr_ref._obj.value = self._table[bytes(handle)]
        return 0

    def c2v_ipc_close(self, device, ptr):
        return 0

    def c2v_ipc_free(self, device, ptr):
        for k in [k for k, p in self._table.items() if p == ptr]:
            del self._table[k]
        return self._lib.c2v_ipc_free(device, ptr)


def emulate_ipc(engines):
    """Give every engine of one emulated group an IpcProxy over a shared handle table (before its Trainer is built)."""
    table = {}
    for e in engines:
        e.lib = IpcProxy(e.lib, table)
    return table
