"""Python face of the device Communicator (csrc/src/device/communicator.cpp).

One :class:`Communicator` per MPI rank / GPU.  Two ways to get one:

* :func:`init_from_env` — one process per GPU (torchrun): rank, world size and
  local rank come from RANK / WORLD_SIZE / LOCAL_RANK; peer memory is wired
  through the native Unix-socket bootstrap (VMM fds or CUDA IPC handles).
* :class:`LocalGroup` — all ranks inside this process (the reference's
  rank-thread model); several ranks may share one GPU, which is how the
  single-GPU test-suite exercises the cross-rank flag protocol.

All collectives are stream-ordered kernel launches (no host sync) and fuse the
reduce op; see csrc/kernels.  Tensors allocated with :meth:`Communicator.empty`
live in the symmetric heap and take the zero-copy paths.
"""

from __future__ import annotations

import ctypes as C
import os
from typing import Callable, Optional, Sequence

import torch

from .. import _lib
from .._lib import FbConfig

# FbDtype
_DTYPES = {
    torch.int8: 0,
    torch.uint8: 1,
    torch.int16: 2,
    torch.int32: 4,
    torch.int64: 6,
    torch.float32: 8,
    torch.float64: 9,
    torch.float16: 10,
    torch.bfloat16: 11,
    torch.bool: 1,
}
for _name, _code in (("uint16", 3), ("uint32", 5), ("uint64", 7)):
    if hasattr(torch, _name):
        _DTYPES[getattr(torch, _name)] = _code

# Every FbDtype by name, with its element size in bytes (fbDtypeSize).  The
# `dtype=` argument of the reductions takes one of these names: the tensor is
# then read as raw bytes of that type, which reaches the unsigned integers on
# any torch version and the MAXLOC/MINLOC {value, int32} pairs (the 16-byte
# pairs include 4 bytes of padding).
FB_DTYPES = {
    "i8": (0, 1),
    "u8": (1, 1),
    "i16": (2, 2),
    "u16": (3, 2),
    "i32": (4, 4),
    "u32": (5, 4),
    "i64": (6, 8),
    "u64": (7, 8),
    "f32": (8, 4),
    "f64": (9, 8),
    "f16": (10, 2),
    "bf16": (11, 2),
    "f64_i32": (12, 16),
    "f32_i32": (13, 8),
    "i32_i32": (14, 8),
    "i64_i32": (15, 16),
}

OPS = {
    "max": 0,
    "min": 1,
    "sum": 2,
    "prod": 3,
    "land": 4,
    "lor": 5,
    "band": 6,
    "bor": 7,
    "maxloc": 8,
    "minloc": 9,
    "lxor": 10,
    "bxor": 11,
    # one-sided accumulate only (FB_OP_REPLACE, FB_OP_NO_OP); every collective
    # rejects them
    "replace": 32,
    "no_op": 33,
}
ALGOS = {"auto": 0, "oneshot": 1, "twoshot": 2, "nvls": 3, "ll": 4}
ALGO_NAMES = {v: k for k, v in ALGOS.items()}
FLAG_SYMMETRIC = 1
FLAG_NOSYNC = 2


class CommError(RuntimeError):
    pass


class _CudaBuf:
    """Minimal __cuda_array_interface__ carrier for heap memory."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {
            "shape": (nbytes,),
            "typestr": "|u1",
            "data": (ptr, False),
            "version": 3,
        }


def make_config(**kw) -> FbConfig:
    lib = _lib.load()
    cfg = FbConfig()
    lib.fb_default_config(C.byref(cfg))
    for k, v in kw.items():
        if not hasattr(cfg, k):
            raise KeyError(k)
        setattr(cfg, k, int(v))
    return cfg


class Communicator:
    def __init__(self, handle: int, owner=None):
        self._lib = _lib.load()
        self._h = C.c_void_p(handle)
        self._owner = owner  # keeps a LocalGroup alive
        self.rank = self._lib.fb_comm_rank(self._h)
        self.size = self._lib.fb_comm_size(self._h)
        self.device = self._lib.fb_comm_device(self._h)
        self.backing = self._lib.fb_comm_backing(self._h).decode()
        self.has_multicast = bool(self._lib.fb_comm_has_multicast(self._h))
        # cross-rank synchronisation through stream memory operations instead
        # of in-kernel spins (ranks sharing a GPU): not CUDA-graph capturable
        self.stream_sync = bool(self._lib.fb_comm_stream_sync(self._h))
        self.stream_wait_supported = bool(self._lib.fb_comm_stream_wait_supported(self._h))
        self.is_subset = bool(self._lib.fb_comm_is_subset(self._h))
        self._allocs: dict[int, int] = {}

    # ------------------------------------------------------------ lifecycle
    def close(self):
        if self._h:
            self._lib.fb_comm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------- helpers
    def _stream(self, stream) -> C.c_void_p:
        if stream is None:
            stream = torch.cuda.current_stream(self.device)
        return C.c_void_p(stream.cuda_stream)

    def _check(self, rc: int, what: str):
        if rc != 0:
            raise CommError(
                f"{what} failed: {self._lib.fb_error_string(rc).decode()} "
                f"[{_lib.last_error()}]"
            )

    def _sym(self, *tensors) -> int:
        for t in tensors:
            if t is None:
                continue
            if not self._lib.fb_comm_in_heap(
                self._h, C.c_void_p(t.data_ptr()), max(t.numel() * t.element_size(), 1)
            ):
                return 0
        return FLAG_SYMMETRIC

    @staticmethod
    def _dtype(t: torch.Tensor) -> int:
        try:
            return _DTYPES[t.dtype]
        except KeyError:
            raise CommError(f"unsupported dtype {t.dtype}")

    @classmethod
    def _typed(cls, t: torch.Tensor, dtype: Optional[str]) -> tuple[int, int]:
        """(element count, FbDtype code) of ``t``, read as ``dtype`` when given
        (an FbDtype name, see FB_DTYPES) or as its own torch dtype otherwise."""
        if dtype is None:
            return t.numel(), cls._dtype(t)
        try:
            code, esize = FB_DTYPES[dtype]
        except KeyError:
            raise CommError(f"unknown dtype {dtype!r}; one of {', '.join(FB_DTYPES)}")
        nbytes = t.numel() * t.element_size()
        if nbytes % esize != 0:
            raise CommError(f"{nbytes} bytes is not a whole number of {dtype} elements ({esize} bytes)")
        return nbytes // esize, code

    # ------------------------------------------------------ sub-communicators
    def subset(self, members: Sequence[int], slot: int) -> "Communicator":
        """A communicator over ``members`` (ranks of this one, in the order that
        becomes the child's rank order; this rank must be one of them).  Every
        member passes the same list and slot, a slot free on every member (see
        :meth:`free_subset_slots`).  No communication and no allocation: the
        child runs the same fused kernels over the members' heaps, so tensors
        from :meth:`empty` on the parent are symmetric on the child too.
        Closing the child zeroes this rank's slot pad and frees the slot: close
        it only after its last collective has completed (synchronise the
        streams it ran on; :meth:`LocalGroup.subset` groups do that)."""
        members = [int(m) for m in members]
        arr = (C.c_int * max(len(members), 1))(*members)
        h = self._lib.fb_comm_subset(self._h, arr, len(members), int(slot))
        if not h:
            raise CommError(f"subset {members} on slot {slot} failed [{_lib.last_error()}]")
        return Communicator(h, owner=self)

    def free_subset_slots(self) -> int:
        """Bit s set: sub-communicator slot s is free on this rank."""
        return int(self._lib.fb_comm_free_subset_slots(self._h))

    def _parent_only(self, what: str):
        if self.is_subset:
            raise CommError(f"{what} on a sub-communicator: use the parent communicator")

    # ------------------------------------------------------------ heap
    def empty(self, shape, dtype=torch.float32) -> torch.Tensor:
        """Allocate a tensor in the symmetric heap.  Call collectively (same
        order and sizes on every rank) so offsets match across ranks."""
        self._parent_only("empty")
        if isinstance(shape, int):
            shape = (shape,)
        numel = 1
        for s in shape:
            numel *= int(s)
        esize = torch.empty((), dtype=dtype).element_size()
        nbytes = max(numel * esize, 16)
        off = self._lib.fb_comm_alloc(self._h, nbytes)
        if off < 0:
            raise CommError(f"symmetric heap exhausted ({nbytes} bytes)")
        ptr = self._lib.fb_comm_heap_ptr(self._h, off, -1)
        with torch.cuda.device(self.device):
            flat = torch.as_tensor(_CudaBuf(ptr, nbytes), device=f"cuda:{self.device}")
        t = flat[: numel * esize].view(dtype).view(*shape)
        self._allocs[t.data_ptr()] = off
        return t

    def zeros(self, shape, dtype=torch.float32) -> torch.Tensor:
        t = self.empty(shape, dtype)
        t.zero_()
        return t

    def free(self, t: torch.Tensor):
        self._parent_only("free")
        off = self._allocs.pop(t.data_ptr(), None)
        if off is not None:
            self._lib.fb_comm_free(self._h, off)

    def heap_offset(self, t: torch.Tensor) -> int:
        base = self._lib.fb_comm_heap_ptr(self._h, 0, -1)
        return t.data_ptr() - base

    def set_allreduce_table(self, table):
        """table: [(max_bytes, algo_name), ...] measured by the autotuner."""
        n = len(table)
        mb = (C.c_uint64 * n)(*[int(t[0]) for t in table])
        al = (C.c_int * n)(*[ALGOS[t[1]] for t in table])
        self._check(self._lib.fb_comm_set_allreduce_table(self._h, n, mb, al), "set table")

    def load_tuning(self, path):
        """Apply a tuning file (see ``faabric_b200.parallel.autotune``)."""
        self._check(self._lib.fb_comm_load_tuning(self._h, str(path).encode()), f"load tuning {path}")

    def configure(self, **kw):
        keys = {
            "llMaxBytes": 0,
            "oneShotMaxBytes": 1,
            "nvlsMinBytes": 2,
            "bcast2StepMinBytes": 3,
            "maxBlocks": 4,
            "threads": 5,
            "tmaMinBytes": 6,
            "nvlsScalarMinBytes": 7,
            "groupBlocks": 8,
        }
        for k, v in kw.items():
            self._check(self._lib.fb_comm_configure(self._h, keys[k], int(v)), k)

    def stats(self, reset: bool = False) -> dict:
        out = (C.c_uint64 * 16)()
        self._lib.fb_comm_stats(self._h, out, 1 if reset else 0)
        d = {"launches": out[0], "bytes": out[1], "staged_copies": out[2], "tma_launches": out[15]}
        for code, name in ALGO_NAMES.items():
            d[f"algo_{name}"] = out[3 + code]
        return d

    @property
    def last_algo(self) -> str:
        return ALGO_NAMES.get(self._lib.fb_comm_last_algo(self._h), "?")

    def check_error(self, stream=None) -> int:
        return int(self._lib.fb_comm_check_error(self._h, self._stream(stream)))

    def host_barrier(self):
        self._parent_only("host_barrier")
        self._lib.fb_comm_host_barrier(self._h)

    # ------------------------------------------------------------ collectives
    def all_reduce(self, send, recv=None, op="sum", algo="auto", stream=None, flags=None, channel=0, dtype=None):
        recv = send if recv is None else recv
        count, dt = self._typed(send, dtype)
        # only the source needs to be symmetric; the native side stages the
        # destination when a push algorithm needs it
        f = self._sym(send) if flags is None else flags
        f |= (channel & 0xF) << 8
        rc = self._lib.fb_allreduce(
            self._h,
            C.c_void_p(send.data_ptr()),
            C.c_void_p(recv.data_ptr()),
            count,
            dt,
            OPS[op],
            ALGOS[algo],
            f,
            self._stream(stream),
        )
        self._check(rc, "all_reduce")
        return recv

    def reduce(self, send, recv, root=0, op="sum", stream=None, flags=None, dtype=None):
        f = self._sym(send) if flags is None else flags
        count, dt = self._typed(send, dtype)
        rp = recv.data_ptr() if recv is not None else 0
        rc = self._lib.fb_reduce(
            self._h,
            C.c_void_p(send.data_ptr()),
            C.c_void_p(rp),
            count,
            dt,
            OPS[op],
            root,
            f,
            self._stream(stream),
        )
        self._check(rc, "reduce")
        return recv

    def reduce_scatter(self, send, recv, op="sum", stream=None, flags=None, dtype=None):
        f = self._sym(send) if flags is None else flags
        count, _ = self._typed(recv, dtype)
        _, dt = self._typed(send, dtype)
        rc = self._lib.fb_reduce_scatter(
            self._h,
            C.c_void_p(send.data_ptr()),
            C.c_void_p(recv.data_ptr()),
            count,
            dt,
            OPS[op],
            f,
            self._stream(stream),
        )
        self._check(rc, "reduce_scatter")
        return recv

    def scan(self, send, recv, op="sum", stream=None, flags=None, dtype=None):
        f = self._sym(send) if flags is None else flags
        count, dt = self._typed(send, dtype)
        rc = self._lib.fb_scan(
            self._h,
            C.c_void_p(send.data_ptr()),
            C.c_void_p(recv.data_ptr()),
            count,
            dt,
            OPS[op],
            f,
            self._stream(stream),
        )
        self._check(rc, "scan")
        return recv

    def broadcast(self, buf, root=0, stream=None, flags=None):
        f = self._sym(buf) if flags is None else flags
        rc = self._lib.fb_broadcast(
            self._h,
            C.c_void_p(buf.data_ptr()),
            buf.numel() * buf.element_size(),
            root,
            f,
            self._stream(stream),
        )
        self._check(rc, "broadcast")
        return buf

    def all_gather(self, send, recv, stream=None, flags=None):
        # pull only needs the source symmetric; the native side additionally
        # checks the destination before taking the NVLS path
        f = self._sym(send) if flags is None else flags
        rc = self._lib.fb_allgather(
            self._h,
            C.c_void_p(send.data_ptr()),
            C.c_void_p(recv.data_ptr()),
            send.numel() * send.element_size(),
            f,
            self._stream(stream),
        )
        self._check(rc, "all_gather")
        return recv

    def gather(self, send, recv, root=0, stream=None, flags=None):
        f = self._sym(send) if flags is None else flags
        rp = recv.data_ptr() if recv is not None else 0
        rc = self._lib.fb_gather(
            self._h,
            C.c_void_p(send.data_ptr()),
            C.c_void_p(rp),
            send.numel() * send.element_size(),
            root,
            f,
            self._stream(stream),
        )
        self._check(rc, "gather")
        return recv

    def scatter(self, send, recv, root=0, stream=None, flags=None):
        # `send` is only significant on the root.  The zero-copy path is taken
        # when EVERY rank passes a symmetric `send` (SPMD style); otherwise the
        # root stages through the fixed staging area.
        f = flags
        if f is None:
            f = self._sym(send) if send is not None else 0
        sp = send.data_ptr() if send is not None else 0
        rc = self._lib.fb_scatter(
            self._h,
            C.c_void_p(sp),
            C.c_void_p(recv.data_ptr()),
            recv.numel() * recv.element_size(),
            root,
            f,
            self._stream(stream),
        )
        self._check(rc, "scatter")
        return recv

    def all_to_all(self, send, recv, stream=None, flags=None):
        f = self._sym(send) if flags is None else flags
        rc = self._lib.fb_alltoall(
            self._h,
            C.c_void_p(send.data_ptr()),
            C.c_void_p(recv.data_ptr()),
            send.numel() * send.element_size() // self.size,
            f,
            self._stream(stream),
        )
        self._check(rc, "all_to_all")
        return recv

    # ------------------------------------------------- grouped all-reduce
    def _group_arrays(self, sends, recvs, dtype):
        n = len(sends)
        sp = (C.c_void_p * n)(*[t.data_ptr() for t in sends])
        rp = (C.c_void_p * n)(*[t.data_ptr() for t in recvs])
        typed = [self._typed(t, dtype) for t in sends]
        if len({dt for _, dt in typed}) != 1:
            raise CommError("grouped all-reduce: every tensor must have the same dtype")
        cnt = (C.c_uint64 * n)(*[c for c, _ in typed])
        return n, sp, rp, cnt, typed[0][1]

    def prepare_group(self, sends, recvs=None, dtype=None) -> "GroupPlan":
        """Plan ONE launch that all-reduces every tensor of ``sends`` (each with
        per-tensor semantics).  Tensors must live in the symmetric heap at
        16-byte aligned addresses; call collectively with the same list."""
        recvs = sends if recvs is None else recvs
        if len(sends) != len(recvs) or not sends:
            raise CommError("prepare_group: need equally long, non-empty lists")
        n, sp, rp, cnt, dt = self._group_arrays(sends, recvs, dtype)
        h = self._lib.fb_group_prepare(self._h, n, sp, rp, cnt, dt)
        if not h:
            raise CommError(f"prepare_group failed [{_lib.last_error()}]")
        return GroupPlan(self, h, n, sum(t.numel() * t.element_size() for t in sends))

    def all_reduce_group(self, plan: "GroupPlan", op="sum", stream=None, channel=0, flags=FLAG_SYMMETRIC):
        rc = self._lib.fb_group_allreduce(
            self._h, plan._h, OPS[op], flags | ((channel & 0xF) << 8), self._stream(stream)
        )
        self._check(rc, "all_reduce_group")

    def all_reduce_many(self, sends, recvs=None, op="sum", stream=None, channel=0, dtype=None):
        """Transient variant of :meth:`prepare_group` + :meth:`all_reduce_group`
        (the table is rebuilt and uploaded in stream order on every call)."""
        recvs = sends if recvs is None else recvs
        if not sends:
            raise CommError("all_reduce_many: need a non-empty list")
        n, sp, rp, cnt, dt = self._group_arrays(sends, recvs, dtype)
        f = self._sym(*sends) | ((channel & 0xF) << 8)
        rc = self._lib.fb_allreduce_many(self._h, n, sp, rp, cnt, dt, OPS[op], f, self._stream(stream))
        self._check(rc, "all_reduce_many")

    # ------------------------------ grouped reduce-scatter and all-gather
    def _shard_arrays(self, what, sends, recvs, dtype, gather):
        """(n, send ptrs, recv ptrs, per-rank counts, FbDtype) of a shard group;
        raises before any native call when a shape does not fit: reduce-scatter
        needs send.numel() == size * recv.numel(), all-gather the reverse."""
        if len(sends) != len(recvs) or not sends:
            raise CommError(f"{what}: need equally long, non-empty lists")
        for i, (s, r) in enumerate(zip(sends, recvs)):
            small, big = (s, r) if gather else (r, s)
            if big.numel() != self.size * small.numel():
                raise CommError(
                    f"{what}: item {i} has {s.numel()} send and {r.numel()} recv elements; "
                    f"{'recv' if gather else 'send'} must hold {self.size} x {'send' if gather else 'recv'}"
                )
        n = len(sends)
        sp = (C.c_void_p * n)(*[t.data_ptr() for t in sends])
        rp = (C.c_void_p * n)(*[t.data_ptr() for t in recvs])
        typed = [self._typed(s if gather else r, dtype) for s, r in zip(sends, recvs)]
        if len({dt for _, dt in typed}) != 1:
            raise CommError(f"{what}: every tensor must have the same dtype")
        cnt = (C.c_uint64 * n)(*[c for c, _ in typed])
        return n, sp, rp, cnt, typed[0][1]

    def prepare_reduce_scatter_group(self, sends, recvs, dtype=None) -> "GroupPlan":
        """Plan ONE launch that reduce-scatters every pair of the lists
        (MPI_Reduce_scatter_block per pair: ``recvs[i]`` gets this rank's
        shard of the reduction of ``sends[i]`` over the ranks).  Tensors live in
        the symmetric heap at 16-byte aligned addresses, shards are multiples
        of 16 bytes, and no output overlaps an input; call collectively with
        the same lists."""
        n, sp, rp, cnt, dt = self._shard_arrays("prepare_reduce_scatter_group", sends, recvs, dtype, False)
        h = self._lib.fb_group_prepare_reduce_scatter(self._h, n, sp, rp, cnt, dt)
        if not h:
            raise CommError(f"prepare_reduce_scatter_group failed [{_lib.last_error()}]")
        return GroupPlan(self, h, n, sum(t.numel() * t.element_size() for t in sends))

    def prepare_all_gather_group(self, sends, recvs, dtype=None) -> "GroupPlan":
        """Plan ONE launch that all-gathers every pair of the lists
        (MPI_Allgather per pair: block p of ``recvs[i]`` gets ``sends[i]`` of
        rank p).  Same conditions as :meth:`prepare_reduce_scatter_group`; in
        place (``sends[i]`` is block ``rank`` of ``recvs[i]``) is allowed."""
        n, sp, rp, cnt, dt = self._shard_arrays("prepare_all_gather_group", sends, recvs, dtype, True)
        h = self._lib.fb_group_prepare_all_gather(self._h, n, sp, rp, cnt, dt)
        if not h:
            raise CommError(f"prepare_all_gather_group failed [{_lib.last_error()}]")
        return GroupPlan(self, h, n, sum(t.numel() * t.element_size() for t in recvs))

    def reduce_scatter_group(self, plan: "GroupPlan", op="sum", stream=None, channel=0, flags=FLAG_SYMMETRIC):
        rc = self._lib.fb_group_reduce_scatter(
            self._h, plan._h, OPS[op], flags | ((channel & 0xF) << 8), self._stream(stream)
        )
        self._check(rc, "reduce_scatter_group")

    def all_gather_group(self, plan: "GroupPlan", stream=None, channel=0, flags=FLAG_SYMMETRIC):
        rc = self._lib.fb_group_all_gather(self._h, plan._h, flags | ((channel & 0xF) << 8), self._stream(stream))
        self._check(rc, "all_gather_group")

    def reduce_scatter_many(self, sends, recvs, op="sum", stream=None, channel=0, dtype=None):
        """Transient variant of :meth:`prepare_reduce_scatter_group` +
        :meth:`reduce_scatter_group`; lists that cannot be grouped run one
        :meth:`reduce_scatter` per pair."""
        n, sp, rp, cnt, dt = self._shard_arrays("reduce_scatter_many", sends, recvs, dtype, False)
        f = self._sym(*sends) | ((channel & 0xF) << 8)
        rc = self._lib.fb_reduce_scatter_many(self._h, n, sp, rp, cnt, dt, OPS[op], f, self._stream(stream))
        self._check(rc, "reduce_scatter_many")

    def all_gather_many(self, sends, recvs, stream=None, channel=0, dtype=None):
        """Transient variant of :meth:`prepare_all_gather_group` +
        :meth:`all_gather_group`; lists that cannot be grouped run one
        :meth:`all_gather` per pair."""
        n, sp, rp, cnt, dt = self._shard_arrays("all_gather_many", sends, recvs, dtype, True)
        f = self._sym(*sends) | ((channel & 0xF) << 8)
        rc = self._lib.fb_all_gather_many(self._h, n, sp, rp, cnt, dt, f, self._stream(stream))
        self._check(rc, "all_gather_many")

    def send_recv(self, send_buf, dst, recv_buf, src, stream=None):
        rc = self._lib.fb_sendrecv(
            self._h,
            C.c_void_p(send_buf.data_ptr()),
            send_buf.numel() * send_buf.element_size(),
            dst,
            C.c_void_p(recv_buf.data_ptr()),
            recv_buf.numel() * recv_buf.element_size(),
            src,
            self._stream(stream),
        )
        self._check(rc, "send_recv")

    def synchronize(self, stream=None, timeout_ms: int = 30000) -> bool:
        """Bounded wait for ``stream``; False if it had to be aborted."""
        return bool(self._lib.fb_comm_sync_bounded(self._h, self._stream(stream), int(timeout_ms)))

    def barrier(self, stream=None):
        self._check(self._lib.fb_barrier(self._h, self._stream(stream)), "barrier")

    def send(self, buf, peer, stream=None):
        rc = self._lib.fb_send(
            self._h,
            C.c_void_p(buf.data_ptr()),
            buf.numel() * buf.element_size(),
            peer,
            self._stream(stream),
        )
        self._check(rc, "send")

    def recv(self, buf, peer, stream=None):
        rc = self._lib.fb_recv(
            self._h,
            C.c_void_p(buf.data_ptr()),
            buf.numel() * buf.element_size(),
            peer,
            self._stream(stream),
        )
        self._check(rc, "recv")

    def put_signal(self, local, dst_sym, peer, signal=0, blocks=8, stream=None):
        """Copy `local` into the peer's copy of symmetric tensor `dst_sym` and
        bump its user signal `signal` (once per CTA)."""
        rc = self._lib.fb_put_signal(
            self._h,
            C.c_void_p(local.data_ptr()),
            self.heap_offset(dst_sym),
            local.numel() * local.element_size(),
            peer,
            signal,
            blocks,
            self._stream(stream),
        )
        self._check(rc, "put_signal")

    def wait_signal(self, signal=0, count=8, stream=None):
        self._check(
            self._lib.fb_wait_signal(self._h, signal, count, self._stream(stream)),
            "wait_signal",
        )

    # ------------------------------------------------------ one-sided atomics
    def _rma_ptr(self, t, what) -> int:
        if t is None:
            return 0
        if not t.is_cuda or not t.is_contiguous():
            raise CommError(f"{what} must be a contiguous CUDA tensor")
        return t.data_ptr()

    def _rma_offset(self, dst_sym, nbytes) -> int:
        if not dst_sym.is_contiguous() or dst_sym.numel() * dst_sym.element_size() < nbytes:
            raise CommError(f"dst_sym must be a contiguous symmetric tensor of at least {nbytes} bytes")
        if not self._lib.fb_comm_in_heap(self._h, C.c_void_p(dst_sym.data_ptr()), max(nbytes, 1)):
            raise CommError("dst_sym is not in the symmetric heap")
        return self.heap_offset(dst_sym)

    def _put_get_many(self, what, locals_, syms, peers, get, stream):
        """One batched copy between ``locals_[i]`` and ``peers[i]``'s copy of the
        symmetric tensor ``syms[i]``; every item is checked before the native
        call."""
        self._parent_only(what)
        n = len(locals_)
        if len(syms) != n or len(peers) != n:
            raise CommError(f"{what}: {n} local tensors, {len(syms)} symmetric tensors and {len(peers)} peers")
        ptrs, offs, nbytes, prs = [], [], [], []
        for i, (loc, sym, peer) in enumerate(zip(locals_, syms, peers)):
            if not loc.is_cuda or not loc.is_contiguous() or not sym.is_contiguous():
                raise CommError(f"{what}: item {i} must be contiguous CUDA tensors")
            if loc.device.index != self.device:
                raise CommError(f"{what}: item {i} local tensor is on {loc.device}, not on cuda:{self.device}")
            nb = loc.numel() * loc.element_size()
            if sym.numel() * sym.element_size() != nb:
                raise CommError(
                    f"{what}: item {i} has {nb} local bytes and {sym.numel() * sym.element_size()} symmetric bytes"
                )
            # (an empty item is skipped: only its peer is checked)
            if nb > 0 and not self._lib.fb_comm_in_heap(self._h, C.c_void_p(sym.data_ptr()), nb):
                raise CommError(f"{what}: item {i} symmetric tensor is not in the symmetric heap")
            peer = int(peer)
            if peer < 0 or peer >= self.size:
                raise CommError(f"{what}: item {i} peer {peer} outside a communicator of {self.size}")
            ptrs.append(loc.data_ptr())
            offs.append(self.heap_offset(sym) if nb > 0 else 0)
            nbytes.append(nb)
            prs.append(peer)
        if n == 0:
            return
        rc = self._lib.fb_put_get_many(
            self._h,
            n,
            (C.c_void_p * n)(*ptrs),
            (C.c_uint64 * n)(*offs),
            (C.c_uint64 * n)(*nbytes),
            (C.c_int32 * n)(*prs),
            (C.c_int32 * n)(*([1 if get else 0] * n)),
            self._stream(stream),
        )
        self._check(rc, what)

    def put_many(self, srcs, dsts_sym, peers, stream=None):
        """Copy every ``srcs[i]`` into ``peers[i]``'s copy of the symmetric
        tensor ``dsts_sym[i]`` (byte sizes must match), as one batched launch
        per 1024 items (MPI_Rput).  Any alignment and length; ``peers[i]`` may
        be this rank.  Stream-ordered: complete when ``stream`` passes it.
        Destinations that overlap within one list get unspecified bytes."""
        self._put_get_many("put_many", srcs, dsts_sym, peers, False, stream)

    def get_many(self, dsts, srcs_sym, peers, stream=None):
        """Copy ``peers[i]``'s copy of the symmetric tensor ``srcs_sym[i]`` into
        every ``dsts[i]`` (MPI_Rget); the same rules as :meth:`put_many`."""
        self._put_get_many("get_many", dsts, srcs_sym, peers, True, stream)

    def accumulate(self, src, dst_sym, peer, op="sum", dtype=None, fetch=None, stream=None):
        """Atomically combine ``src`` into ``peer``'s copy of the symmetric tensor
        ``dst_sym``, element by element: ``dst[i] = op(dst[i], src[i])``
        (MPI_Accumulate).  With ``fetch``, every element's previous value is
        written there first (MPI_Get_accumulate).  ``op`` is any reduction op
        of :meth:`all_reduce` for the dtype, ``"replace"``, or ``"no_op"``,
        an atomic read into ``fetch`` for which ``src`` may be None.  The
        target elements must be aligned to their size; ``src`` and ``fetch``
        need no alignment.  Concurrent accumulates from any rank to the same
        element compose atomically.  Stream-ordered; returns ``fetch``."""
        if op not in OPS:
            raise CommError(f"unknown op {op!r}")
        ref = src if src is not None else fetch
        if ref is None:
            raise CommError("accumulate needs src (or fetch for no_op)")
        count, dt = self._typed(ref, dtype)
        nbytes = ref.numel() * ref.element_size()
        if fetch is not None and fetch.numel() * fetch.element_size() != nbytes:
            raise CommError(f"fetch must hold {nbytes} bytes like src")
        rc = self._lib.fb_accumulate(
            self._h,
            C.c_void_p(self._rma_ptr(src, "src")),
            self._rma_offset(dst_sym, nbytes),
            count,
            dt,
            OPS[op],
            peer,
            C.c_void_p(self._rma_ptr(fetch, "fetch")),
            self._stream(stream),
        )
        self._check(rc, "accumulate")
        return fetch

    def fetch_and_op(self, src, dst_sym, peer, result, op="sum", dtype=None, stream=None):
        """MPI_Fetch_and_op: :meth:`accumulate` of ONE element with fetch into
        ``result`` (``src`` may be None for ``"no_op"``)."""
        for t, what in ((src, "src"), (result, "result")):
            if t is not None and self._typed(t, dtype)[0] != 1:
                raise CommError(f"fetch_and_op: {what} must be exactly one element")
        return self.accumulate(src, dst_sym, peer, op=op, dtype=dtype, fetch=result, stream=stream)

    def compare_and_swap(self, compare, swap, dst_sym, peer, result, dtype=None, stream=None):
        """MPI_Compare_and_swap on one integer element of ``peer``'s copy of
        ``dst_sym``: ``result = old; if old == compare: target = swap``."""
        dts = set()
        for t, what in ((compare, "compare"), (swap, "swap"), (result, "result")):
            count, dt = self._typed(t, dtype)
            if count != 1:
                raise CommError(f"compare_and_swap: {what} must be exactly one element")
            dts.add(dt)
        if len(dts) != 1:
            raise CommError("compare_and_swap: compare, swap and result must have one dtype")
        rc = self._lib.fb_compare_and_swap(
            self._h,
            C.c_void_p(self._rma_ptr(compare, "compare")),
            C.c_void_p(self._rma_ptr(swap, "swap")),
            C.c_void_p(self._rma_ptr(result, "result")),
            self._rma_offset(dst_sym, result.numel() * result.element_size()),
            dts.pop(),
            peer,
            self._stream(stream),
        )
        self._check(rc, "compare_and_swap")
        return result


class GroupPlan:
    """Device-resident segment tables of a grouped all-reduce, reduce-scatter
    or all-gather."""

    def __init__(self, comm: Communicator, handle, n_tensors: int, nbytes: int):
        self._comm = comm
        self._h = C.c_void_p(handle)
        self.n_tensors = n_tensors
        self.nbytes = nbytes
        self.launches = int(comm._lib.fb_group_plan_launches(self._h))

    def close(self):
        if self._h:
            self._comm._lib.fb_group_plan_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class LocalGroup:
    """N ranks inside this process.  ``devices[i]`` is rank i's GPU; repeating a
    device id puts several ranks on one GPU (each rank then needs its own
    stream so the per-rank kernels are co-resident)."""

    def __init__(self, nranks: int, devices: Optional[Sequence[int]] = None, **cfg):
        lib = _lib.load()
        ndev = lib.fb_cuda_device_count()
        if ndev <= 0:
            raise CommError("no CUDA device")
        if devices is None:
            devices = [i % ndev for i in range(nranks)]
        self.devices = list(devices)
        arr = (C.c_int * nranks)(*self.devices)
        c = make_config(**cfg)
        h = lib.fb_group_create_local(nranks, arr, C.byref(c))
        if not h:
            raise CommError(f"group creation failed: {_lib.last_error()}")
        self._lib = lib
        self._h = C.c_void_p(h)
        self.comms = [
            Communicator(lib.fb_group_comm(self._h, r), owner=self)
            for r in range(nranks)
        ]
        self.streams = []
        for d in self.devices:
            with torch.cuda.device(d):
                self.streams.append(torch.cuda.Stream(device=d))
        self.size = nranks

    def run(self, fn: Callable[[Communicator, int, "torch.cuda.Stream"], object]):
        """Issue ``fn(comm, rank, stream)`` for every rank, each on its own
        stream, without synchronising in between (launches are asynchronous, so
        the per-rank kernels overlap on the device(s))."""
        out = []
        for r, c in enumerate(self.comms):
            with torch.cuda.device(c.device):
                # Rank streams are non-blocking: order them after whatever the
                # caller has queued on the device's current stream (e.g. the
                # copies that filled the input buffers)
                self.streams[r].wait_stream(torch.cuda.current_stream(c.device))
                with torch.cuda.stream(self.streams[r]):
                    out.append(fn(c, r, self.streams[r]))
        return out

    def synchronize(self):
        for s in self.streams:
            s.synchronize()

    def check_errors(self):
        return [c.check_error(self.streams[r]) for r, c in enumerate(self.comms)]

    @property
    def shares_devices(self) -> bool:
        return len(set(self.devices)) < len(self.devices)

    def coresident(self) -> bool:
        """Probe for groups that synchronise INSIDE kernels while several ranks
        share a GPU: one barrier kernel per rank must meet on the device.  False
        (and a poisoned group: close it) when the ranks' kernels do not overlap,
        e.g. their streams alias one hardware queue or a tool serialises them."""
        self.run(lambda c, r, st: c.barrier())
        return self.check_errors() == [0] * self.size

    def subset(self, members: Sequence[int]) -> "SubGroup":
        """The ranks ``members`` of this group as a group of their own (child
        rank i is rank ``members[i]`` here), on the lowest sub-communicator
        slot free on every member.  Its collectives run the same fused
        kernels; close it to free the slot."""
        members = [int(m) for m in members]
        if not members or any(m < 0 or m >= self.size for m in members):
            raise CommError(f"subset: members {members} outside a group of {self.size}")
        free = ~0
        for m in members:
            free &= self.comms[m].free_subset_slots()
        if free == 0:
            raise CommError(f"subset: no sub-communicator slot is free on every member of {members}")
        slot = (free & -free).bit_length() - 1
        return SubGroup(self, members, slot)

    def close(self):
        for c in self.comms:
            c.close()
        self.comms = []
        if self._h:
            self._lib.fb_group_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class SubGroup(LocalGroup):
    """Members of a :class:`LocalGroup` as a group of their own (made by
    :meth:`LocalGroup.subset`).  ``comms[i]`` is the child communicator of
    parent rank ``members[i]`` and ``streams[i]`` that rank's parent stream, so
    calls on the child and on the parent issued through ``run`` stay ordered."""

    def __init__(self, parent: LocalGroup, members: Sequence[int], slot: int):
        self._lib = parent._lib
        self._h = None
        self.parent = parent
        self.members = list(members)
        self.slot = slot
        self.devices = [parent.devices[m] for m in self.members]
        self.streams = [parent.streams[m] for m in self.members]
        self.comms = []
        try:
            for m in self.members:
                self.comms.append(parent.comms[m].subset(self.members, slot))
        except Exception:
            self.close()
            raise
        self.size = len(self.members)

    def close(self):
        # a child frees its slot by zeroing its pad: its kernels must be done
        if self.comms:
            self.synchronize()
        for c in self.comms:
            c.close()
        self.comms = []


def init_from_env(**cfg) -> Communicator:
    """One-process-per-GPU initialisation (torchrun environment)."""
    lib = _lib.load()
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    job = os.environ.get("FAABRIC_JOB_ID") or (
        os.environ.get("MASTER_PORT", "0") + "-" + os.environ.get("TORCHELASTIC_RUN_ID", "x")
    )
    torch.cuda.set_device(local)
    c = make_config(**cfg)
    h = lib.fb_comm_create_ipc(rank, world, local, job.encode(), C.byref(c))
    if not h:
        raise CommError(f"ipc communicator creation failed: {_lib.last_error()}")
    return Communicator(h)
