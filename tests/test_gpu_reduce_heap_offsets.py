"""Device reductions on symmetric-heap buffers at every heap offset, bit for bit.

tests/test_gpu_reduce_matrix.py allocates its symmetric buffers with
``Communicator.empty``, so their heap offsets are multiples of 16.  A tensor
view such as ``bucket[3:]`` of a flat gradient bucket is in the heap too, at an
offset that is not: the reduction kernels load and store 16-byte vectors at
``heap[p] + offset``, so such a buffer must go through the staging copy rather
than the symmetric (zero-copy) path.  Every rank uses the same offset, as the
symmetric contract asks.

Each case checks the result against the rank-order fold of reduce_oracle.py,
that the inputs and 16 guard bytes on each side of every buffer are
unchanged, and the staging count: above zero for a shifted call (LL excepted:
it moves unaligned bytes itself and never stages), exactly zero for an
aligned one, which shows the aligned fast path is untouched."""

import numpy as np
import pytest
import torch

from reduce_oracle import (
    DTYPES,
    FLOAT_DTYPES,
    FLOAT_OPS,
    INT_DTYPES,
    INT_OPS,
    NP_DTYPES,
    PAIR_DTYPES,
    PAIR_OPS,
    SUPPORTED,
    assert_same,
    fold,
    itemsize,
)
from test_gpu_reduce_matrix import make_inputs

pytestmark = pytest.mark.gpu

from faabric_b200.parallel import LocalGroup  # noqa: E402

# launch_api.h: FB_LL_BLOCKS (8) x FB_LL_THREADS (512) vectors of 16 bytes
FB_LL_MAX_BYTES = 8 * 512 * 16
GUARD = 16

# a staging piece of 128 KiB: the largest messages below take three pieces
CFG = dict(heapBytes=64 << 20, stageBytes=128 << 10, maxBlocks=4, threads=512, oneShotMaxBytes=64 << 10, timeoutMs=8000)
OPS_FOR = {**{d: INT_OPS for d in INT_DTYPES}, **{d: FLOAT_OPS for d in FLOAT_DTYPES}, **{d: PAIR_OPS for d in PAIR_DTYPES}}

GROUPS = {}


def group(n, spin=False):
    """Stream-ordered synchronisation, or (spin) the in-kernel protocol, which
    LL needs; None where the ranks' kernels are not co-resident."""
    key = (n, spin)
    if key not in GROUPS:
        g = LocalGroup(n, **(dict(CFG, streamSync=0, timeoutMs=2000) if spin else CFG))
        if spin and g.shares_devices and not g.coresident():
            g.close()
            g = None
        GROUPS[key] = g
    return GROUPS[key]


@pytest.fixture(scope="module", autouse=True)
def _cleanup():
    yield
    for g in GROUPS.values():
        if g is not None:
            g.close()
    GROUPS.clear()


def shifts_of(dtype):
    """Every element-aligned heap offset in 1..15 (the 16-byte pairs: 8)."""
    e = itemsize(dtype)
    return [8] if e == 16 else list(range(e, 16, e))


# ----------------------------------------------------------------- buffers ----
class Sym:
    """``nbytes`` at heap offset ``16 + shift`` of a fresh heap allocation on
    every rank, with GUARD bytes of a seeded pattern on each side."""

    def __init__(self, g, nbytes, shift, rng, fill=None):
        self.g, self.nbytes, self.shift = g, nbytes, shift
        total = GUARD + 16 + nbytes + GUARD
        self.raw = [c.empty(total, torch.uint8) for c in g.comms]
        self.before = []
        for r, t in enumerate(self.raw):
            img = np.frombuffer(rng.bytes(total), dtype=np.uint8).copy()
            if fill is not None:
                img[self.lo : self.lo + nbytes] = np.ascontiguousarray(fill[r]).view(np.uint8)
            t.copy_(torch.from_numpy(img))
            self.before.append(img)
        self.views = [t[self.lo : self.lo + nbytes] for t in self.raw]

    @property
    def lo(self):
        return 16 + self.shift

    def image(self, r):
        return self.raw[r].cpu().numpy()

    def data(self, r, dtype):
        return self.image(r)[self.lo : self.lo + self.nbytes].view(NP_DTYPES[dtype])

    def assert_untouched(self, what, ranks=None, keep=None):
        """Every byte unchanged, except `keep` bytes from the data start."""
        for r in range(self.g.size) if ranks is None else ranks:
            got, want = self.image(r), self.before[r]
            if keep is not None:
                got, want = got.copy(), want.copy()
                got[self.lo : self.lo + keep] = want[self.lo : self.lo + keep]
            assert np.array_equal(got, want), f"{what}: rank {r} bytes outside the result changed"

    def free(self):
        for c, t in zip(self.g.comms, self.raw):
            c.free(t)


def run(g, fn):
    for c in g.comms:
        c.stats(reset=True)
    torch.cuda.synchronize()
    g.run(fn)
    g.synchronize()
    assert g.check_errors() == [0] * g.size
    return [c.stats()["staged_copies"] for c in g.comms]


def check_staged(staged, shifted, what):
    if shifted:
        assert all(s > 0 for s in staged), f"{what}: a shifted call was not staged ({staged})"
    else:
        assert staged == [0] * len(staged), f"{what}: the aligned call staged ({staged})"


# -------------------------------------------------------------- all-reduce ----
def allreduce_sizes(dtype, algo):
    e = itemsize(dtype)
    sizes = [16 - e, 16 + e] if e < 16 else [16, 32]  # one vector, one element less or more
    if algo != "ll":
        sizes.append(FB_LL_MAX_BYTES + 16 + e)  # above llMaxBytes
    if algo == "twoshot":
        sizes.append(2 * CFG["stageBytes"] + 48 + e)  # three staging pieces
    return [b // e for b in sizes]


def allreduce_case(g, rng, dtype, op, algo, count, send_shift, recv_shift, in_place):
    n = g.size
    ins = make_inputs(rng, dtype, op, n, count)
    exp = fold(ins, dtype, op)
    nb = exp.nbytes
    what = f"all_reduce n={n} {dtype} {op} {algo} count={count} shifts=({send_shift},{recv_shift}) in_place={in_place}"
    send = Sym(g, nb, send_shift, rng, fill=ins)
    recv = send if in_place else Sym(g, nb, recv_shift, rng)
    try:
        staged = run(g, lambda c, r, st: c.all_reduce(send.views[r], recv.views[r], op=op, algo=algo, dtype=dtype))
        assert [c.last_algo for c in g.comms] == [algo] * n, what
        for r in range(n):
            assert_same(recv.data(r, dtype), exp, dtype, f"{what} rank {r}")
        if not in_place:
            send.assert_untouched(what + " (send)")
        recv.assert_untouched(what, keep=nb)
        check_staged(staged, algo != "ll" and (send_shift or recv_shift), what)
    finally:
        send.free()
        if not in_place:
            recv.free()


@pytest.mark.parametrize("n", [2, 4])
@pytest.mark.parametrize("dtype", ["i8", "i32", "f32", "bf16", "f64_i32"])
def test_allreduce_every_op_at_every_heap_offset(n, dtype):
    rng = np.random.default_rng([700 + n, DTYPES.index(dtype)])
    for algo in ("ll", "oneshot", "twoshot"):
        g = group(n, spin=algo == "ll")
        if g is None:
            continue
        for op in OPS_FOR[dtype]:
            for shift in [0] + shifts_of(dtype):
                for count in allreduce_sizes(dtype, algo):
                    allreduce_case(g, rng, dtype, op, algo, count, shift, shift, False)
                    # in place on symmetric buffers takes the two-shot path
                    if algo != "oneshot":
                        allreduce_case(g, rng, dtype, op, algo, count, shift, shift, True)
        # send and recv at different offsets
        op = OPS_FOR[dtype][0]
        s = shifts_of(dtype)[0]
        for count in allreduce_sizes(dtype, algo):
            allreduce_case(g, rng, dtype, op, algo, count, s, 0, False)
            allreduce_case(g, rng, dtype, op, algo, count, 0, s, False)


@pytest.mark.parametrize("algo", ["oneshot", "twoshot"])
def test_allreduce_every_supported_pair_at_one_shifted_offset(algo):
    n = 3
    g = group(n)
    rng = np.random.default_rng([800, len(algo)])
    for dtype, op in SUPPORTED:
        e = itemsize(dtype)
        count = (16 * 3 * n + e) // e
        allreduce_case(g, rng, dtype, op, algo, count, shifts_of(dtype)[0], shifts_of(dtype)[0], False)


# ---------------------------------------------------- reduce / scan / reduce_scatter ----
@pytest.mark.parametrize("n", [2, 3, 4, 8])
@pytest.mark.parametrize("spin", [False, True], ids=["stream-ordered", "spin"])
@pytest.mark.parametrize("dtype,op", [("i32", "sum"), ("bf16", "max"), ("i64_i32", "minloc")])
def test_reduce_scan_reduce_scatter_at_heap_offsets(n, spin, dtype, op):
    g = group(n, spin)
    if g is None:
        pytest.skip("kernels of different ranks are not co-resident on this GPU")
    e = itemsize(dtype)
    rng = np.random.default_rng([900 + n, int(spin), DTYPES.index(dtype)])
    for shift in (0, shifts_of(dtype)[0]):
        # reduce: one-shot, and two-shot above 2 x oneShotMaxBytes
        for nbytes in (16 * n + e, 2 * CFG["oneShotMaxBytes"] + 16 * n + e):
            count = nbytes // e
            ins = make_inputs(rng, dtype, op, n, count)
            exp = fold(ins, dtype, op)
            algo = "twoshot" if exp.nbytes > 2 * CFG["oneShotMaxBytes"] else "oneshot"
            for root in range(n):
                what = f"reduce n={n} spin={spin} {dtype} {op} count={count} shift={shift} root={root}"
                send = Sym(g, exp.nbytes, shift, rng, fill=ins)
                recv = Sym(g, exp.nbytes, shift, rng)
                try:
                    staged = run(g, lambda c, r, st: c.reduce(send.views[r], recv.views[r], root=root, op=op, dtype=dtype))
                    assert g.comms[0].last_algo == algo, what
                    assert_same(recv.data(root, dtype), exp, dtype, what)
                    send.assert_untouched(what + " (send)")
                    recv.assert_untouched(what, ranks=[root], keep=exp.nbytes)
                    recv.assert_untouched(what + " (non-root output)", ranks=[r for r in range(n) if r != root])
                    # two-shot reduce pushes into the root's staging area whatever the offset
                    root_only = [1 if (algo == "twoshot" and r == root) else 0 for r in range(n)]
                    if shift == 0:
                        assert [min(s, 1) for s in staged] == root_only, f"{what}: staged {staged}"
                    else:
                        check_staged(staged, True, what)
                finally:
                    send.free()
                    recv.free()
            # scan
            what = f"scan n={n} spin={spin} {dtype} {op} count={count} shift={shift}"
            send = Sym(g, exp.nbytes, shift, rng, fill=ins)
            recv = Sym(g, exp.nbytes, shift, rng)
            try:
                staged = run(g, lambda c, r, st: c.scan(send.views[r], recv.views[r], op=op, dtype=dtype))
                for r in range(n):
                    assert_same(recv.data(r, dtype), fold(ins[: r + 1], dtype, op), dtype, f"{what} rank {r}")
                send.assert_untouched(what + " (send)")
                recv.assert_untouched(what, keep=exp.nbytes)
                check_staged(staged, shift != 0, what)
            finally:
                send.free()
                recv.free()
        # reduce-scatter: whole-vector slices; the shifted input is staged whole
        for slice_bytes in (16, 16 * 7):
            per = slice_bytes // e
            ins = make_inputs(rng, dtype, op, n, per * n)
            exp = fold(ins, dtype, op)
            what = f"reduce_scatter n={n} spin={spin} {dtype} {op} slice={slice_bytes} shift={shift}"
            send = Sym(g, exp.nbytes, shift, rng, fill=ins)
            recv = Sym(g, slice_bytes, shift, rng)
            try:
                staged = run(g, lambda c, r, st: c.reduce_scatter(send.views[r], recv.views[r], op=op, dtype=dtype))
                for r in range(n):
                    assert_same(recv.data(r, dtype), exp[r * per : (r + 1) * per], dtype, f"{what} rank {r}")
                send.assert_untouched(what + " (send)")
                recv.assert_untouched(what, keep=slice_bytes)
                check_staged(staged, shift != 0, what)
            finally:
                send.free()
                recv.free()


# ------------------------------------------------------- sub-communicator ----
def test_subset_all_reduce_and_scan_at_heap_offset_4():
    parent = group(4)
    sub = parent.subset([3, 1, 0])
    rng = np.random.default_rng(1000)
    try:
        n = sub.size
        count = (FB_LL_MAX_BYTES + 16 + 4) // 4
        ins = make_inputs(rng, "i32", "sum", n, count)
        exp = fold(ins, "i32", "sum")
        # heap tensors come from the parent; the child sees them at the same offsets
        send = Sym(parent, exp.nbytes, 4, rng)
        recv = Sym(parent, exp.nbytes, 4, rng)
        try:
            for i, m in enumerate(sub.members):
                send.views[m].copy_(torch.from_numpy(np.ascontiguousarray(ins[i]).view(np.uint8)))
                send.before[m][send.lo : send.lo + exp.nbytes] = np.ascontiguousarray(ins[i]).view(np.uint8)
            staged = run(sub, lambda c, i, st: c.all_reduce(send.views[sub.members[i]], recv.views[sub.members[i]], op="sum", dtype="i32"))
            for i, m in enumerate(sub.members):
                assert_same(recv.data(m, "i32"), exp, "i32", f"subset all_reduce member {i}")
            check_staged(staged, True, "subset all_reduce")
            staged = run(sub, lambda c, i, st: c.scan(send.views[sub.members[i]], recv.views[sub.members[i]], op="sum", dtype="i32"))
            for i, m in enumerate(sub.members):
                assert_same(recv.data(m, "i32"), fold(ins[: i + 1], "i32", "sum"), "i32", f"subset scan member {i}")
            check_staged(staged, True, "subset scan")
            send.assert_untouched("subset (send)")
            recv.assert_untouched("subset", ranks=sub.members, keep=exp.nbytes)
            recv.assert_untouched("subset (non-member)", ranks=[2])
        finally:
            send.free()
            recv.free()
    finally:
        sub.close()
