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
# Communicator::GroupKind
GROUP_KINDS = {
    "all_reduce": 0,
    "reduce_scatter": 1,
    "all_gather": 2,
    "broadcast": 3,
    "all_to_all": 4,
    "gather": 5,
    "scatter": 6,
    "reduce": 7,
    "scan": 8,
    "exscan": 9,
    "neighbor_all_gather": 10,
    "neighbor_all_to_all": 11,
    "neighbor_all_gather_v": 12,
    "neighbor_all_to_all_v": 13,
}
ALGOS = {"auto": 0, "oneshot": 1, "twoshot": 2, "nvls": 3, "ll": 4}
ALGO_NAMES = {v: k for k, v in ALGOS.items()}
FLAG_SYMMETRIC = 1
FLAG_NOSYNC = 2


class CommError(RuntimeError):
    pass


def neighbor_in_edges(sources_per_rank, destinations_per_rank):
    """Every rank's in-edges of a distributed graph given by its adjacency
    lists (MPI_Dist_graph_create_adjacent's ``sources`` and ``destinations``
    of every rank): ``out[d][j]`` is ``(s, idx)`` for the j-th source s of
    rank d, where idx is the position of the matching edge in s's
    destinations.  The k-th occurrence of s in d's sources pairs with the
    k-th occurrence of d in s's destinations (MPI-3.1 section 7.6), so
    self-edges and multi-edges are allowed.  Raises CommError for lists of
    different lengths, a rank outside the graph, or an edge s -> d whose
    multiplicity in s's destinations differs from that of s in d's sources."""
    src = [[int(x) for x in v] for v in sources_per_rank]
    dst = [[int(x) for x in v] for v in destinations_per_rank]
    n = len(src)
    if len(dst) != n:
        raise CommError(f"neighbor_in_edges: {n} source lists and {len(dst)} destination lists")
    for what, lists in (("source", src), ("destination", dst)):
        for r, v in enumerate(lists):
            for x in v:
                if not 0 <= x < n:
                    raise CommError(f"neighbor_in_edges: rank {r} names {what} {x} outside a graph of {n}")
    # positions of d in s's destinations, in order
    out_pos = [{} for _ in range(n)]
    for s, v in enumerate(dst):
        for i, d in enumerate(v):
            out_pos[s].setdefault(d, []).append(i)
    in_count = [{} for _ in range(n)]
    for d, v in enumerate(src):
        for s in v:
            in_count[d][s] = in_count[d].get(s, 0) + 1
    for s in range(n):
        for d in range(n):
            a = len(out_pos[s].get(d, ()))
            b = in_count[d].get(s, 0)
            if a != b:
                raise CommError(
                    f"neighbor_in_edges: edge {s} -> {d} is {a} times in {s}'s destinations "
                    f"and {b} times in {d}'s sources"
                )
    edges = []
    for d, v in enumerate(src):
        seen = {}
        mine = []
        for s in v:
            k = seen.get(s, 0)
            seen[s] = k + 1
            mine.append((s, out_pos[s][d][k]))
        edges.append(mine)
    return edges


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
        # (in-degree, out-degree) once set_neighbors has run
        self._neighbors: Optional[tuple[int, int]] = None

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
        """All-reduce ``send`` into ``recv`` (in place when ``recv`` is None).
        Heap tensors take the symmetric path at any heap offset, the same on
        every rank; offsets not a multiple of 16 are staged.  So do
        :meth:`reduce`, :meth:`reduce_scatter` and :meth:`scan`."""
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

    # ------------------------------------------------- grouped collectives
    def _group_items(self, what, kind, sends, recvs, dtype, root=0):
        """(n, send ptrs, recv ptrs, counts, FbDtype) of a grouped list of
        ``kind`` (a GROUP_KINDS name); raises before any native call for empty
        or unequally long lists and for shapes that do not fit the kind:
        reduce-scatter needs send.numel() == size * recv.numel(), all-gather
        the reverse; all-to-all needs equal send and recv numel and element
        size, numel divisible by ``size`` (in ``dtype`` elements too), and
        counts per block; a broadcast (each buffer as send and recv) needs
        contiguous tensors and a root in the communicator, and counts bytes.
        Gather follows the all-gather rule and scatter the reduce-scatter
        rule, with a root in the communicator and contiguous tensors on this
        communicator's GPU; the root's side (gather recvs, scatter sends) may
        be None off the root, or a list of None.  Reduce needs the rooted
        rules with equal send and recv numel and element size (recvs as for
        gather); scan and exscan the same, with a send and a recv on every
        rank and no root."""
        if kind in ("gather", "scatter", "reduce"):
            if not 0 <= int(root) < self.size:
                raise CommError(f"{what}: root {root} outside a communicator of {self.size}")
            if kind != "scatter" and recvs is None:
                recvs = [None] * len(sends or [])
            if kind == "scatter" and sends is None:
                sends = [None] * len(recvs or [])
        if kind in ("scan", "exscan") and (sends is None or recvs is None):
            raise CommError(f"{what}: need equally long, non-empty lists")
        if len(sends) != len(recvs) or not sends:
            raise CommError(f"{what}: need equally long, non-empty lists")
        per = 1
        if kind in ("reduce", "scan", "exscan"):
            rooted = kind != "reduce" or self.rank == int(root)
            for i, (s, r) in enumerate(zip(sends, recvs)):
                for t in (s, r):
                    if t is not None and (not t.is_cuda or t.device.index != self.device or not t.is_contiguous()):
                        raise CommError(
                            f"{what}: item {i} must be contiguous tensors on cuda:{self.device}, not {t.device}"
                            f"{'' if t.is_contiguous() else ' (non-contiguous)'}"
                        )
                if s is None or (r is None and rooted):
                    raise CommError(
                        f"{what}: item {i} needs a send on every rank and a recv on "
                        f"{'the root' if kind == 'reduce' else 'every rank'}"
                    )
                if r is not None and (r.numel() != s.numel() or r.element_size() != s.element_size()):
                    raise CommError(
                        f"{what}: item {i} has {s.numel()} send and {r.numel()} recv elements of "
                        f"{s.element_size()} and {r.element_size()} bytes; both must be equal"
                    )
                if r is not None and dtype is None and r.dtype != s.dtype:
                    raise CommError(f"{what}: item {i} has a {s.dtype} send and a {r.dtype} recv")
            typed = [self._typed(s, dtype) for s in sends]
        elif kind in ("gather", "scatter"):
            gather = kind == "gather"
            rooted = self.rank == int(root)
            for i, (s, r) in enumerate(zip(sends, recvs)):
                small, big = (s, r) if gather else (r, s)
                # (the kernels load and store these addresses as they are)
                for t in (s, r):
                    if t is not None and (not t.is_cuda or t.device.index != self.device or not t.is_contiguous()):
                        raise CommError(
                            f"{what}: item {i} must be contiguous tensors on cuda:{self.device}, not {t.device}"
                            f"{'' if t.is_contiguous() else ' (non-contiguous)'}"
                        )
                if small is None or (big is None and rooted):
                    raise CommError(f"{what}: item {i} needs a {'send' if gather else 'recv'} on every rank "
                                    f"and a {'recv' if gather else 'send'} on the root")
                if big is not None and big.numel() != self.size * small.numel():
                    raise CommError(
                        f"{what}: item {i} has {s.numel()} send and {r.numel()} recv elements; "
                        f"{'recv' if gather else 'send'} must hold {self.size} x {'send' if gather else 'recv'}"
                    )
                if big is not None and big.element_size() != small.element_size():
                    raise CommError(f"{what}: item {i} has send and recv elements of different sizes")
            typed = [self._typed(s if gather else r, dtype) for s, r in zip(sends, recvs)]
        elif kind == "broadcast":
            if not 0 <= int(root) < self.size:
                raise CommError(f"{what}: root {root} outside a communicator of {self.size}")
            for i, t in enumerate(sends):
                if not t.is_contiguous():
                    raise CommError(f"{what}: item {i} must be contiguous")
            typed = [(t.numel() * t.element_size(), FB_DTYPES["u8"][0]) for t in sends]
        elif kind == "all_to_all":
            for i, (s, r) in enumerate(zip(sends, recvs)):
                if s.numel() != r.numel() or s.numel() % self.size != 0:
                    raise CommError(
                        f"{what}: item {i} has {s.numel()} send and {r.numel()} recv elements; "
                        f"both must be equal and divisible by {self.size}"
                    )
                if s.element_size() != r.element_size():
                    # (the native side sizes recv from the send's elements)
                    raise CommError(
                        f"{what}: item {i} has {s.element_size()}-byte send and {r.element_size()}-byte recv elements"
                    )
            typed = [self._typed(s, dtype) for s in sends]
            per = self.size
        elif kind == "all_reduce":
            typed = [self._typed(t, dtype) for t in sends]
        else:
            gather = kind == "all_gather"
            for i, (s, r) in enumerate(zip(sends, recvs)):
                small, big = (s, r) if gather else (r, s)
                if big.numel() != self.size * small.numel():
                    raise CommError(
                        f"{what}: item {i} has {s.numel()} send and {r.numel()} recv elements; "
                        f"{'recv' if gather else 'send'} must hold {self.size} x {'send' if gather else 'recv'}"
                    )
            typed = [self._typed(s if gather else r, dtype) for s, r in zip(sends, recvs)]
        if len({dt for _, dt in typed}) != 1:
            raise CommError(f"{what}: every tensor must have the same dtype")
        for i, (c, _) in enumerate(typed):
            if c % per != 0:
                raise CommError(f"{what}: item {i} has {c} {dtype} elements, not divisible by {self.size}")
        n = len(sends)
        sp = (C.c_void_p * n)(*[t.data_ptr() if t is not None else None for t in sends])
        rp = (C.c_void_p * n)(*[t.data_ptr() if t is not None else None for t in recvs])
        cnt = (C.c_uint64 * n)(*[c // per for c, _ in typed])
        return n, sp, rp, cnt, typed[0][1]

    def _prepare(self, what, kind, sends, recvs, dtype, sized, root=0):
        """A GroupPlan of ``kind``; ``sized`` is the list whose bytes it moves."""
        n, sp, rp, cnt, dt = self._group_items(what, kind, sends, recvs, dtype, root)
        h = self._lib.fb_group_prepare(self._h, GROUP_KINDS[kind], n, sp, rp, cnt, dt)
        if not h:
            raise CommError(f"{what} failed [{_lib.last_error()}]")
        plan = GroupPlan(self, h, n, sum(t.numel() * t.element_size() for t in sized if t is not None))
        plan.root = int(root)
        plan.kind = kind
        return plan

    def _launch(self, what, kind, plan, op, root, stream, channel, flags):
        if kind in ("gather", "scatter", "reduce") and int(root) != plan.root:
            # (the root's side was checked, and on other ranks may be missing,
            # for the root the plan was prepared for)
            raise CommError(f"{what}: plan prepared for root {plan.root}, launched with root {root}")
        rc = self._lib.fb_group_launch(
            self._h, GROUP_KINDS[kind], plan._h, op, root, flags | ((channel & 0xF) << 8), self._stream(stream)
        )
        self._check(rc, what)

    def _many(self, what, kind, sends, recvs, dtype, op, root, stream, channel):
        n, sp, rp, cnt, dt = self._group_items(what, kind, sends, recvs, dtype, root)
        staged = kind in ("gather", "scatter", "reduce", "scan", "exscan")
        f = (0 if staged else self._sym(*sends)) | ((channel & 0xF) << 8)
        fop = OPS[op] if op is not None else 0
        rc = self._lib.fb_group_many(
            self._h, GROUP_KINDS[kind], n, sp, rp, cnt, dt, fop, int(root), f, self._stream(stream)
        )
        self._check(rc, what)

    def prepare_group(self, sends, recvs=None, dtype=None) -> "GroupPlan":
        """Plan ONE launch that all-reduces every tensor of ``sends`` (each with
        per-tensor semantics).  Tensors must live in the symmetric heap at
        16-byte aligned addresses; call collectively with the same list."""
        recvs = sends if recvs is None else recvs
        return self._prepare("prepare_group", "all_reduce", sends, recvs, dtype, sends)

    def all_reduce_group(self, plan: "GroupPlan", op="sum", stream=None, channel=0, flags=FLAG_SYMMETRIC):
        self._launch("all_reduce_group", "all_reduce", plan, OPS[op], 0, stream, channel, flags)

    def all_reduce_many(self, sends, recvs=None, op="sum", stream=None, channel=0, dtype=None):
        """Transient variant of :meth:`prepare_group` + :meth:`all_reduce_group`
        (the table is rebuilt and uploaded in stream order on every call)."""
        recvs = sends if recvs is None else recvs
        self._many("all_reduce_many", "all_reduce", sends, recvs, dtype, op, 0, stream, channel)

    def prepare_reduce_scatter_group(self, sends, recvs, dtype=None) -> "GroupPlan":
        """Plan ONE launch that reduce-scatters every pair of the lists
        (MPI_Reduce_scatter_block per pair: ``recvs[i]`` gets this rank's
        shard of the reduction of ``sends[i]`` over the ranks).  Tensors live in
        the symmetric heap at 16-byte aligned addresses, shards are multiples
        of 16 bytes, and no output overlaps an input; call collectively with
        the same lists."""
        return self._prepare("prepare_reduce_scatter_group", "reduce_scatter", sends, recvs, dtype, sends)

    def prepare_all_gather_group(self, sends, recvs, dtype=None) -> "GroupPlan":
        """Plan ONE launch that all-gathers every pair of the lists
        (MPI_Allgather per pair: block p of ``recvs[i]`` gets ``sends[i]`` of
        rank p).  Same conditions as :meth:`prepare_reduce_scatter_group`; in
        place (``sends[i]`` is block ``rank`` of ``recvs[i]``) is allowed."""
        return self._prepare("prepare_all_gather_group", "all_gather", sends, recvs, dtype, recvs)

    def reduce_scatter_group(self, plan: "GroupPlan", op="sum", stream=None, channel=0, flags=FLAG_SYMMETRIC):
        self._launch("reduce_scatter_group", "reduce_scatter", plan, OPS[op], 0, stream, channel, flags)

    def all_gather_group(self, plan: "GroupPlan", stream=None, channel=0, flags=FLAG_SYMMETRIC):
        self._launch("all_gather_group", "all_gather", plan, 0, 0, stream, channel, flags)

    def reduce_scatter_many(self, sends, recvs, op="sum", stream=None, channel=0, dtype=None):
        """Transient variant of :meth:`prepare_reduce_scatter_group` +
        :meth:`reduce_scatter_group`; lists that cannot be grouped run one
        :meth:`reduce_scatter` per pair."""
        self._many("reduce_scatter_many", "reduce_scatter", sends, recvs, dtype, op, 0, stream, channel)

    def all_gather_many(self, sends, recvs, stream=None, channel=0, dtype=None):
        """Transient variant of :meth:`prepare_all_gather_group` +
        :meth:`all_gather_group`; lists that cannot be grouped run one
        :meth:`all_gather` per pair."""
        self._many("all_gather_many", "all_gather", sends, recvs, dtype, None, 0, stream, channel)

    def prepare_broadcast_group(self, bufs) -> "GroupPlan":
        """Plan ONE launch that broadcasts every tensor of ``bufs`` (MPI_Bcast
        per tensor, any dtype and length) from the root given to
        :meth:`broadcast_group`.  Tensors live in the symmetric heap at 16-byte
        aligned addresses; call collectively with the same list."""
        return self._prepare("prepare_broadcast_group", "broadcast", bufs, bufs, None, bufs)

    def broadcast_group(self, plan: "GroupPlan", root=0, stream=None, channel=0, flags=FLAG_SYMMETRIC):
        self._launch("broadcast_group", "broadcast", plan, 0, int(root), stream, channel, flags)

    def broadcast_many(self, bufs, root=0, stream=None, channel=0):
        """Transient variant of :meth:`prepare_broadcast_group` +
        :meth:`broadcast_group`; lists that cannot be grouped run one
        :meth:`broadcast` per tensor."""
        self._many("broadcast_many", "broadcast", bufs, bufs, None, None, root, stream, channel)

    def prepare_all_to_all_group(self, sends, recvs, dtype=None) -> "GroupPlan":
        """Plan ONE launch that exchanges every pair of the lists (MPI_Alltoall
        per pair: block r of ``recvs[i]`` on rank p gets block p of
        ``sends[i]`` on rank r, with ``size`` equal blocks per tensor).
        Tensors live in the symmetric heap at 16-byte aligned addresses, blocks
        are multiples of 16 bytes, and no output overlaps an input; call
        collectively with the same lists."""
        return self._prepare("prepare_all_to_all_group", "all_to_all", sends, recvs, dtype, sends)

    def all_to_all_group(self, plan: "GroupPlan", stream=None, channel=0, flags=FLAG_SYMMETRIC):
        self._launch("all_to_all_group", "all_to_all", plan, 0, 0, stream, channel, flags)

    def all_to_all_many(self, sends, recvs, stream=None, channel=0, dtype=None):
        """Transient variant of :meth:`prepare_all_to_all_group` +
        :meth:`all_to_all_group`; lists that cannot be grouped run one
        :meth:`all_to_all` per pair."""
        self._many("all_to_all_many", "all_to_all", sends, recvs, dtype, None, 0, stream, channel)

    def prepare_gather_group(self, sends, recvs=None, root=0, dtype=None) -> "GroupPlan":
        """Plan the launches that gather every pair of the lists to the root
        given to :meth:`gather_group` (MPI_Gather per pair: block p of
        ``recvs[i]`` on the root gets ``sends[i]`` of rank p).  Tensors are
        any device memory at any alignment; ``recvs`` is only read on the
        root (None elsewhere).  In place (``sends[i]`` is block ``root`` of
        ``recvs[i]``) is allowed.  The plan launches with this ``root`` only;
        call collectively with the same counts."""
        return self._prepare("prepare_gather_group", "gather", sends, recvs, dtype, sends, root)

    def gather_group(self, plan: "GroupPlan", root=0, stream=None, channel=0, flags=0):
        self._launch("gather_group", "gather", plan, 0, int(root), stream, channel, flags)

    def gather_many(self, sends, recvs=None, root=0, stream=None, channel=0, dtype=None):
        """Transient variant of :meth:`prepare_gather_group` +
        :meth:`gather_group`."""
        self._many("gather_many", "gather", sends, recvs, dtype, None, root, stream, channel)

    def prepare_scatter_group(self, sends, recvs, root=0, dtype=None) -> "GroupPlan":
        """Plan the launches that scatter every pair of the lists from the
        root given to :meth:`scatter_group` (MPI_Scatter per pair: ``recvs[i]``
        of rank p gets block p of ``sends[i]`` on the root).  Tensors are any
        device memory at any alignment; ``sends`` is only read on the root
        (None elsewhere).  In place (``recvs[i]`` is block ``root`` of
        ``sends[i]``) is allowed.  The plan launches with this ``root`` only;
        call collectively with the same counts."""
        return self._prepare("prepare_scatter_group", "scatter", sends, recvs, dtype, recvs, root)

    def scatter_group(self, plan: "GroupPlan", root=0, stream=None, channel=0, flags=0):
        self._launch("scatter_group", "scatter", plan, 0, int(root), stream, channel, flags)

    def scatter_many(self, sends, recvs, root=0, stream=None, channel=0, dtype=None):
        """Transient variant of :meth:`prepare_scatter_group` +
        :meth:`scatter_group`."""
        self._many("scatter_many", "scatter", sends, recvs, dtype, None, root, stream, channel)

    def prepare_reduce_group(self, sends, recvs=None, root=0, dtype=None) -> "GroupPlan":
        """Plan the launches that reduce every pair of the lists to the root
        given to :meth:`reduce_group` (MPI_Reduce per pair: ``recvs[i]`` on the
        root gets the op over ``sends[i]`` of every rank, folded in rank
        order).  Tensors are any device memory at any alignment; ``recvs`` is
        only read on the root (None elsewhere) and no other rank's recv is
        written.  In place (``recvs[i]`` is ``sends[i]``) is allowed.  The
        dtype is fixed here, the op is given at launch; the plan launches with
        this ``root`` only.  Call collectively with the same counts."""
        return self._prepare("prepare_reduce_group", "reduce", sends, recvs, dtype, sends, root)

    def reduce_group(self, plan: "GroupPlan", op="sum", root=0, stream=None, channel=0, flags=0):
        self._launch("reduce_group", "reduce", plan, OPS[op], int(root), stream, channel, flags)

    def reduce_many(self, sends, recvs=None, op="sum", root=0, stream=None, channel=0, dtype=None):
        """Transient variant of :meth:`prepare_reduce_group` +
        :meth:`reduce_group`."""
        self._many("reduce_many", "reduce", sends, recvs, dtype, op, root, stream, channel)

    def prepare_scan_group(self, sends, recvs, exclusive=False, dtype=None) -> "GroupPlan":
        """Plan the launches of a prefix reduction of every pair of the lists
        given to :meth:`scan_group`: MPI_Scan per pair (``recvs[i]`` on rank r
        gets the op over ``sends[i]`` of ranks 0..r, folded in rank order), or
        with ``exclusive`` MPI_Exscan (ranks 0..r-1; rank 0's recvs are not
        written).  Tensors are any device memory at any alignment, and every
        rank passes both lists; in place (``recvs[i]`` is ``sends[i]``) is
        allowed on any rank.  The dtype is fixed here, the op is given at
        launch.  Call collectively with the same counts."""
        kind = "exscan" if exclusive else "scan"
        return self._prepare("prepare_scan_group", kind, sends, recvs, dtype, sends)

    def scan_group(self, plan: "GroupPlan", op="sum", stream=None, channel=0, flags=0):
        if plan.kind not in ("scan", "exscan"):
            raise CommError(f"scan_group: a {plan.kind} plan")
        self._launch("scan_group", plan.kind, plan, OPS[op], 0, stream, channel, flags)

    def scan_many(self, sends, recvs, op="sum", exclusive=False, stream=None, channel=0, dtype=None):
        """Transient variant of :meth:`prepare_scan_group` +
        :meth:`scan_group`."""
        self._many("scan_many", "exscan" if exclusive else "scan", sends, recvs, dtype, op, 0, stream, channel)

    # -------------------------------------------- neighbourhood collectives
    def set_neighbors(self, in_edges, out_degree: int, max_out_degree: int, max_in_degree: int):
        """Set this rank's neighbourhood topology, once, before the first
        neighbour call: its in-edges in recv-block order, each ``(source rank,
        index of the edge among the source's out-edges)`` (see
        :func:`neighbor_in_edges`), its out-degree, and the largest out- and
        in-degree over every member, which every member passes alike.
        :meth:`LocalGroup.set_neighbors` does this for a whole group."""
        in_edges = [(int(s), int(i)) for s, i in in_edges]
        n = len(in_edges)
        srcs = (C.c_int * max(n, 1))(*[s for s, _ in in_edges])
        idxs = (C.c_int * max(n, 1))(*[i for _, i in in_edges])
        rc = self._lib.fb_comm_set_neighbors(
            self._h, n, srcs, idxs, int(out_degree), int(max_out_degree), int(max_in_degree)
        )
        self._check(rc, "set_neighbors")
        self._neighbors = (n, int(out_degree))

    def _neighbor_items(self, what, kind, sends, recvs, counts, dtype):
        """(n, send ptrs, recv ptrs, counts, FbDtype) of a neighbour list;
        raises before any native call.  Item i moves blocks of ``counts[i]``
        elements (in ``dtype``): the all-gather's send holds one block, the
        all-to-all's one per out-edge, and every recv one per in-edge, all
        contiguous tensors on this communicator's GPU.  ``counts`` may be
        left out where the tensors tell the count: always for the
        all-gather, and for the all-to-all on a rank with an edge."""
        if self._neighbors is None:
            raise CommError(f"{what}: no neighbourhood topology; call set_neighbors first")
        indeg, outdeg = self._neighbors
        if sends is None or recvs is None or len(sends) != len(recvs) or not sends:
            raise CommError(f"{what}: need equally long, non-empty lists")
        if counts is not None and len(counts) != len(sends):
            raise CommError(f"{what}: {len(counts)} counts for {len(sends)} items")
        a2a = kind == "neighbor_all_to_all"
        typed = []
        for i, (s, r) in enumerate(zip(sends, recvs)):
            for t in (s, r):
                if not t.is_cuda or t.device.index != self.device or not t.is_contiguous():
                    raise CommError(
                        f"{what}: item {i} must be contiguous tensors on cuda:{self.device}, not {t.device}"
                        f"{'' if t.is_contiguous() else ' (non-contiguous)'}"
                    )
            if dtype is None and r.dtype != s.dtype:
                raise CommError(f"{what}: item {i} has a {s.dtype} send and a {r.dtype} recv")
            ns, code = self._typed(s, dtype)
            nr, _ = self._typed(r, dtype)
            if counts is not None:
                c = int(counts[i])
            elif not a2a:
                c = ns
            elif outdeg or indeg:
                c = ns // outdeg if outdeg else nr // indeg
            else:
                raise CommError(f"{what}: item {i}: this rank has no edge, so pass counts")
            blocks = outdeg if a2a else 1
            if c < 0 or ns != c * blocks or nr != c * indeg:
                raise CommError(
                    f"{what}: item {i} has {ns} send and {nr} recv elements; with blocks of {c}, "
                    f"send must hold {blocks} and recv {indeg} blocks"
                )
            typed.append((c, code))
        if len({dt for _, dt in typed}) != 1:
            raise CommError(f"{what}: every tensor must have the same dtype")
        n = len(sends)
        sp = (C.c_void_p * n)(*[t.data_ptr() or None for t in sends])
        rp = (C.c_void_p * n)(*[t.data_ptr() or None for t in recvs])
        cnt = (C.c_uint64 * n)(*[c for c, _ in typed])
        return n, sp, rp, cnt, typed[0][1]

    def _prepare_neighbor(self, what, kind, sends, recvs, counts, dtype) -> "GroupPlan":
        n, sp, rp, cnt, dt = self._neighbor_items(what, kind, sends, recvs, counts, dtype)
        h = self._lib.fb_group_prepare(self._h, GROUP_KINDS[kind], n, sp, rp, cnt, dt)
        if not h:
            raise CommError(f"{what} failed [{_lib.last_error()}]")
        plan = GroupPlan(self, h, n, sum(t.numel() * t.element_size() for t in recvs))
        plan.kind = kind
        return plan

    def _neighbor_many(self, what, kind, sends, recvs, counts, dtype, stream):
        n, sp, rp, cnt, dt = self._neighbor_items(what, kind, sends, recvs, counts, dtype)
        rc = self._lib.fb_group_many(self._h, GROUP_KINDS[kind], n, sp, rp, cnt, dt, 0, 0, 0, self._stream(stream))
        self._check(rc, what)

    def prepare_neighbor_all_gather_group(self, sends, recvs, counts=None, dtype=None) -> "GroupPlan":
        """Plan the launches of MPI_Neighbor_allgather per pair of the lists
        over this communicator's topology (:meth:`set_neighbors`): block j of
        ``recvs[i]`` gets ``sends[i]`` of in-edge j's source.  Tensors are any
        device memory at any alignment.  Call collectively with the same
        counts; every member takes part, edges or not."""
        return self._prepare_neighbor(
            "prepare_neighbor_all_gather_group", "neighbor_all_gather", sends, recvs, counts, dtype
        )

    def neighbor_all_gather_group(self, plan: "GroupPlan", stream=None, flags=0):
        self._launch("neighbor_all_gather_group", "neighbor_all_gather", plan, 0, 0, stream, 0, flags)

    def neighbor_all_gather_many(self, sends, recvs, counts=None, stream=None, dtype=None):
        """Transient variant of :meth:`prepare_neighbor_all_gather_group` +
        :meth:`neighbor_all_gather_group`."""
        self._neighbor_many("neighbor_all_gather_many", "neighbor_all_gather", sends, recvs, counts, dtype, stream)

    def prepare_neighbor_all_to_all_group(self, sends, recvs, counts=None, dtype=None) -> "GroupPlan":
        """Plan the launches of MPI_Neighbor_alltoall per pair of the lists
        over this communicator's topology: block j of ``recvs[i]`` gets block
        idx of ``sends[i]`` on the source of in-edge j = (source, idx).
        Otherwise as :meth:`prepare_neighbor_all_gather_group`."""
        return self._prepare_neighbor(
            "prepare_neighbor_all_to_all_group", "neighbor_all_to_all", sends, recvs, counts, dtype
        )

    def neighbor_all_to_all_group(self, plan: "GroupPlan", stream=None, flags=0):
        self._launch("neighbor_all_to_all_group", "neighbor_all_to_all", plan, 0, 0, stream, 0, flags)

    def neighbor_all_to_all_many(self, sends, recvs, counts=None, stream=None, dtype=None):
        """Transient variant of :meth:`prepare_neighbor_all_to_all_group` +
        :meth:`neighbor_all_to_all_group`."""
        self._neighbor_many("neighbor_all_to_all_many", "neighbor_all_to_all", sends, recvs, counts, dtype, stream)

    # ------------------------------- neighbourhood v-collectives (per-edge sizes)
    def _neighbor_v_items(self, what, kind, sends, recvs, sendcounts, sdispls, recvcounts, rdispls, dtype):
        """The C arguments of a neighbour v list; raises before any native
        call.  Counts and displacements are in elements of ``dtype`` (or of
        the tensors' own dtype).  Item i: the all-gather's send holds
        ``sendcounts[i]`` elements (default: all of it), the all-to-all's send
        block k is ``sendcounts[i][k]`` elements at ``sdispls[i][k]``, one per
        out-edge; recv block j is ``recvcounts[i][j]`` elements at
        ``rdispls[i][j]``, one per in-edge.  A tensor may be None where all its
        counts are 0."""
        if self._neighbors is None:
            raise CommError(f"{what}: no neighbourhood topology; call set_neighbors first")
        indeg, outdeg = self._neighbors
        a2a = kind == "neighbor_all_to_all_v"
        n = len(sends) if sends is not None else 0
        if n == 0 or recvs is None or len(recvs) != n:
            raise CommError(f"{what}: need equally long, non-empty lists")
        for name, v in (("recvcounts", recvcounts), ("rdispls", rdispls)) + (
            (("sendcounts", sendcounts), ("sdispls", sdispls)) if a2a else ()
        ):
            if v is None or len(v) != n:
                raise CommError(f"{what}: {name} needs one entry per item")
        codes = set()
        sw = outdeg if a2a else 1
        sc, sd, rc, rd = [], [], [], []

        def side(i, t, counts, displs, width, label):
            counts = [int(x) for x in counts]
            displs = [int(x) for x in displs]
            if len(counts) != width or len(displs) != width:
                raise CommError(f"{what}: item {i} needs {width} {label} counts and displacements")
            if any(x < 0 for x in counts + displs):
                raise CommError(f"{what}: item {i} has a negative {label} count or displacement")
            if t is None:
                if any(counts):
                    raise CommError(f"{what}: item {i} has {label} counts but no {label} tensor")
                return counts, displs
            if not t.is_cuda or t.device.index != self.device or not t.is_contiguous():
                raise CommError(f"{what}: item {i}: {label} must be a contiguous tensor on cuda:{self.device}")
            numel, code = self._typed(t, dtype)
            codes.add(code)
            for c, d in zip(counts, displs):
                if c and c + d > numel:
                    raise CommError(f"{what}: item {i}: a {label} block of {c} at {d} overruns {numel} elements")
            return counts, displs

        for i in range(n):
            s, r = sends[i], recvs[i]
            if a2a:
                c, d = side(i, s, sendcounts[i], sdispls[i], outdeg, "send")
            else:
                cnt = sendcounts[i] if sendcounts is not None else (self._typed(s, dtype)[0] if s is not None else 0)
                c, d = side(i, s, [cnt], [0], 1, "send")
            sc += c
            sd += d
            c, d = side(i, r, recvcounts[i], rdispls[i], indeg, "recv")
            rc += c
            rd += d
        if len(codes) > 1:
            raise CommError(f"{what}: every tensor must have the same dtype")
        code = codes.pop() if codes else FB_DTYPES[dtype or "u8"][0]
        u64 = lambda v: (C.c_uint64 * max(len(v), 1))(*v)  # noqa: E731
        sp = (C.c_void_p * n)(*[(t.data_ptr() or None) if t is not None else None for t in sends])
        rp = (C.c_void_p * n)(*[(t.data_ptr() or None) if t is not None else None for t in recvs])
        return (self._h, GROUP_KINDS[kind], n, sp, rp, u64(sc), u64(sd), sw, u64(rc), u64(rd), indeg, code)

    def _neighbor_v_streams(self, what, kind, args):
        cap = len(args[3]) + 1
        out = (C.c_uint64 * cap)()
        w = self._lib.fb_neighbor_v_streams(*args, out, cap)
        self._check(min(w, 0), what)
        return [int(out[i]) for i in range(w)]

    @staticmethod
    def _agreed(agreed):
        v = [int(x) for x in agreed]
        return (C.c_uint64 * max(len(v), 1))(*v), len(v)

    def _prepare_neighbor_v(self, what, kind, args, agreed, nbytes) -> "GroupPlan":
        a, na = self._agreed(agreed)
        h = self._lib.fb_group_prepare_v(*args, a, na)
        if not h:
            raise CommError(f"{what} failed [{_lib.last_error()}]")
        plan = GroupPlan(self, h, args[2], nbytes)
        plan.kind = kind
        return plan

    def _neighbor_v_many(self, what, args, agreed, stream):
        a, na = self._agreed(agreed)
        self._check(self._lib.fb_group_many_v(*args, a, na, 0, self._stream(stream)), what)

    def neighbor_all_gather_v_streams(self, sends, recvs, recvcounts, rdispls, sendcounts=None, dtype=None):
        """This rank's longest stream of every launch window of a neighbour
        all-gatherv list, in bytes (see :meth:`prepare_neighbor_all_gather_v_group`).
        Every member's lists are combined by an elementwise maximum, the
        agreement (:meth:`LocalGroup.agree_neighbor_v` for a local group)."""
        kind = "neighbor_all_gather_v"
        args = self._neighbor_v_items(
            "neighbor_all_gather_v_streams", kind, sends, recvs, sendcounts, None, recvcounts, rdispls, dtype
        )
        return self._neighbor_v_streams("neighbor_all_gather_v_streams", kind, args)

    def prepare_neighbor_all_gather_v_group(
        self, sends, recvs, recvcounts, rdispls, agreed, sendcounts=None, dtype=None
    ) -> "GroupPlan":
        """Plan MPI_Neighbor_allgatherv per item over this communicator's
        topology: block j of ``recvs[i]`` (``recvcounts[i][j]`` elements at
        ``rdispls[i][j]``) gets the send of in-edge j's source.  ``agreed`` is
        the elementwise maximum over every member of their
        :meth:`neighbor_all_gather_v_streams`; each launch window then takes
        ``ceil(agreed[w] / W)`` launches, W the room of a staging slot.
        Tensors are any device memory at any alignment; call collectively,
        every member takes part, edges or not."""
        what = "prepare_neighbor_all_gather_v_group"
        kind = "neighbor_all_gather_v"
        args = self._neighbor_v_items(what, kind, sends, recvs, sendcounts, None, recvcounts, rdispls, dtype)
        nbytes = sum(t.numel() * t.element_size() for t in recvs if t is not None)
        return self._prepare_neighbor_v(what, kind, args, agreed, nbytes)

    def neighbor_all_gather_v_group(self, plan: "GroupPlan", stream=None, flags=0):
        self._launch("neighbor_all_gather_v_group", "neighbor_all_gather_v", plan, 0, 0, stream, 0, flags)

    def neighbor_all_gather_v_many(
        self, sends, recvs, recvcounts, rdispls, agreed, sendcounts=None, stream=None, dtype=None
    ):
        """Transient variant of :meth:`prepare_neighbor_all_gather_v_group` +
        :meth:`neighbor_all_gather_v_group`."""
        what = "neighbor_all_gather_v_many"
        args = self._neighbor_v_items(
            what, "neighbor_all_gather_v", sends, recvs, sendcounts, None, recvcounts, rdispls, dtype
        )
        self._neighbor_v_many(what, args, agreed, stream)

    def neighbor_all_to_all_v_streams(self, sends, recvs, sendcounts, sdispls, recvcounts, rdispls, dtype=None):
        """As :meth:`neighbor_all_gather_v_streams`, for a neighbour
        all-to-allv list."""
        kind = "neighbor_all_to_all_v"
        args = self._neighbor_v_items(
            "neighbor_all_to_all_v_streams", kind, sends, recvs, sendcounts, sdispls, recvcounts, rdispls, dtype
        )
        return self._neighbor_v_streams("neighbor_all_to_all_v_streams", kind, args)

    def prepare_neighbor_all_to_all_v_group(
        self, sends, recvs, sendcounts, sdispls, recvcounts, rdispls, agreed, dtype=None
    ) -> "GroupPlan":
        """Plan MPI_Neighbor_alltoallv per item: send block k of ``sends[i]``
        (``sendcounts[i][k]`` elements at ``sdispls[i][k]``) goes to out-edge
        k, and recv block j gets the block of in-edge j = (source, idx), the
        source's send block idx.  Otherwise as
        :meth:`prepare_neighbor_all_gather_v_group`."""
        what = "prepare_neighbor_all_to_all_v_group"
        kind = "neighbor_all_to_all_v"
        args = self._neighbor_v_items(what, kind, sends, recvs, sendcounts, sdispls, recvcounts, rdispls, dtype)
        nbytes = sum(t.numel() * t.element_size() for t in recvs if t is not None)
        return self._prepare_neighbor_v(what, kind, args, agreed, nbytes)

    def neighbor_all_to_all_v_group(self, plan: "GroupPlan", stream=None, flags=0):
        self._launch("neighbor_all_to_all_v_group", "neighbor_all_to_all_v", plan, 0, 0, stream, 0, flags)

    def neighbor_all_to_all_v_many(
        self, sends, recvs, sendcounts, sdispls, recvcounts, rdispls, agreed, stream=None, dtype=None
    ):
        """Transient variant of :meth:`prepare_neighbor_all_to_all_v_group` +
        :meth:`neighbor_all_to_all_v_group`."""
        what = "neighbor_all_to_all_v_many"
        args = self._neighbor_v_items(
            what, "neighbor_all_to_all_v", sends, recvs, sendcounts, sdispls, recvcounts, rdispls, dtype
        )
        self._neighbor_v_many(what, args, agreed, stream)

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

    def accumulate_many(self, srcs, dsts_sym, peers, op="sum", dtype=None, fetches=None, stream=None):
        """:meth:`accumulate` of every ``srcs[i]`` into ``peers[i]``'s copy of
        the symmetric tensor ``dsts_sym[i]``, with one ``op`` and dtype for
        the whole list (MPI_Raccumulate / MPI_Rget_accumulate bursts).
        ``fetches`` (None, or one tensor or None per item) receive the
        previous values; ``srcs[i]`` may be None for ``"no_op"``, which needs
        a fetch on every item.  Items whose targets intersect apply in list
        order, also in what they fetch.  Typically one launch for up to 1024
        items; the exact rule is Communicator::accumulateMany's.
        Stream-ordered; returns ``fetches``."""
        self._parent_only("accumulate_many")
        if op not in OPS:
            raise CommError(f"unknown op {op!r}")
        n = len(dsts_sym)
        fl = [None] * n if fetches is None else list(fetches)
        if len(srcs) != n or len(peers) != n or len(fl) != n:
            raise CommError(
                f"accumulate_many: {len(srcs)} sources, {n} symmetric tensors, {len(peers)} peers and {len(fl)} fetches"
            )
        ptrs, fptrs, offs, counts, prs, dts = [], [], [], [], [], set()
        for i, (src, sym, peer, fetch) in enumerate(zip(srcs, dsts_sym, peers, fl)):
            ref = src if src is not None else fetch
            if ref is None:
                raise CommError(f"accumulate_many: item {i} needs src (or fetch for no_op)")
            if src is None and op != "no_op":
                raise CommError(f"accumulate_many: item {i} has no src for {op!r}")
            for t, what in ((src, "src"), (fetch, "fetch")):
                if t is None:
                    continue
                if not t.is_cuda or not t.is_contiguous():
                    raise CommError(f"accumulate_many: item {i} {what} must be a contiguous CUDA tensor")
                if t.device.index != self.device:
                    raise CommError(f"accumulate_many: item {i} {what} is on {t.device}, not on cuda:{self.device}")
            count, dt = self._typed(ref, dtype)
            dts.add(dt)
            nb = ref.numel() * ref.element_size()
            for t, what in ((fetch, "fetch"), (sym, "symmetric tensor")):
                if t is not None and t.numel() * t.element_size() != nb:
                    raise CommError(f"accumulate_many: item {i} {what} holds {t.numel() * t.element_size()} bytes, not {nb}")
            if not sym.is_contiguous():
                raise CommError(f"accumulate_many: item {i} symmetric tensor must be contiguous")
            # (an empty item is skipped: only its peer is checked)
            if nb > 0 and not self._lib.fb_comm_in_heap(self._h, C.c_void_p(sym.data_ptr()), nb):
                raise CommError(f"accumulate_many: item {i} symmetric tensor is not in the symmetric heap")
            peer = int(peer)
            if peer < 0 or peer >= self.size:
                raise CommError(f"accumulate_many: item {i} peer {peer} outside a communicator of {self.size}")
            ptrs.append(src.data_ptr() if src is not None else None)
            fptrs.append(fetch.data_ptr() if fetch is not None else None)
            offs.append(self.heap_offset(sym) if nb > 0 else 0)
            counts.append(count)
            prs.append(peer)
        if len(dts) > 1:
            raise CommError("accumulate_many: every item must have one dtype")
        if n == 0:
            return fetches
        rc = self._lib.fb_accumulate_many(
            self._h,
            n,
            (C.c_void_p * n)(*ptrs),
            (C.c_void_p * n)(*fptrs),
            (C.c_uint64 * n)(*offs),
            (C.c_uint64 * n)(*counts),
            (C.c_int32 * n)(*prs),
            dts.pop(),
            OPS[op],
            self._stream(stream),
        )
        self._check(rc, "accumulate_many")
        return fetches

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
    """Device-resident segment tables of a grouped all-reduce, reduce-scatter,
    all-gather, broadcast, all-to-all, gather, scatter, reduce, scan, exscan,
    or neighbourhood all-gather and all-to-all (equal blocks or v)."""

    def __init__(self, comm: Communicator, handle, n_tensors: int, nbytes: int):
        self._comm = comm
        self._h = C.c_void_p(handle)
        self.n_tensors = n_tensors
        self.nbytes = nbytes
        self.launches = int(comm._lib.fb_group_plan_launches(self._h))
        # gather and scatter: the root the plan was prepared for
        self.root = 0
        # the GROUP_KINDS name it was prepared as
        self.kind = None

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

    def set_neighbors(self, sources_per_rank, destinations_per_rank):
        """Give every rank the neighbourhood topology of the graph with these
        adjacency lists (see :func:`neighbor_in_edges`, which checks it)."""
        edges = neighbor_in_edges(sources_per_rank, destinations_per_rank)
        if len(edges) != self.size:
            raise CommError(f"set_neighbors: a graph of {len(edges)} ranks for a group of {self.size}")
        max_out = max(len(v) for v in destinations_per_rank)
        max_in = max(len(v) for v in edges)
        for r, c in enumerate(self.comms):
            c.set_neighbors(edges[r], len(destinations_per_rank[r]), max_out, max_in)

    @staticmethod
    def agree_neighbor_v(streams_per_rank):
        """The agreement of a neighbour v list over the whole group: the
        elementwise maximum of every rank's ``neighbor_*_v_streams``, which
        every rank then passes as ``agreed``.  (An MPI program gets the same
        from one host reduction over the members.)"""
        lists = [[int(x) for x in v] for v in streams_per_rank]
        if len({len(v) for v in lists}) > 1:
            raise CommError(f"agree_neighbor_v: ranks have different window counts {[len(v) for v in lists]}")
        return [max(col) for col in zip(*lists)] if lists else []

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
