"""Grouped scan and exscan (one launch per staging buffer of a list of
MPI_Scan or MPI_Exscan items) against ``reduce_oracle.fold`` over each rank's
prefix, bit for bit.

N ranks share one GPU inside this process, on the default group (ranks
sharing a GPU synchronise in stream order: the LOCAL, MOVE and UNSTAGE steps
are three launches) and on a spin group whose kernels meet at in-kernel
barriers (skipped where the ranks' kernels are not co-resident).  Every
rank's items sit in one byte buffer (symmetric heap or cudaMalloc) at offsets
that may be unaligned, with random guard bytes around every item: every byte
the oracle does not write must come back unchanged (an exscan's rank 0 recv
included), and the communicator's stats must show one launch per plan
launch.
"""

import numpy as np
import pytest
import torch

import reduce_oracle as ro

pytestmark = pytest.mark.gpu

from faabric_b200.models.resnet50_grads import resnet50_grad_sizes  # noqa: E402
from faabric_b200.parallel import LocalGroup  # noqa: E402
from faabric_b200.parallel.comm import CommError  # noqa: E402

NS = [2, 4, 8]
KINDS = ["stream", "spin"]
GUARD = 32
STAGE = 1 << 20
MAX_ITEMS = 1016  # FB_GROUP_MAX_SEGS - 8 pieces per launch
# f32 elements per rank: one, zero, odd lengths, ragged chunk ends (the chunk
# is 1 KiB at 8 ranks, 2 KiB otherwise), whole chunks, and more than the
# 1 MiB staging buffer
COUNTS = [1, 0, 5, 12, 513, 129 * 4, 65 * 4 + 3, 75000, 3 * STAGE // 4 + 5]

_GROUPS = {}


def group(n, kind, stage=STAGE):
    if (n, kind, stage) not in _GROUPS:
        cfg = dict(heapBytes=160 << 20, stageBytes=stage, maxBlocks=8, timeoutMs=8000)
        if kind == "spin":
            cfg.update(maxBlocks=4, groupBlocks=8, timeoutMs=4000, streamSync=0)
        g = LocalGroup(n, **cfg)
        if kind == "spin" and g.shares_devices and not g.coresident():
            g.close()
            g = None
        _GROUPS[(n, kind, stage)] = g
    g = _GROUPS[(n, kind, stage)]
    if g is None:
        pytest.skip(f"kernels of {n} ranks are not co-resident on this GPU")
    return g


@pytest.fixture(scope="module", autouse=True)
def _cleanup():
    yield
    for g in _GROUPS.values():
        if g is not None:
            g.close()
    _GROUPS.clear()


def inputs(rng, dtype, n, count):
    """Per-rank inputs of ``count`` elements; floats carry NaN and +-0 on the
    first and last rank, pairs few values (many ties)."""
    npd = ro.NP_DTYPES[dtype]
    out = []
    for r in range(n):
        if dtype in ro.INT_DTYPES:
            a = rng.integers(0, 256, count * npd.itemsize, dtype=np.uint8).view(npd)
        elif dtype in ro.PAIR_DTYPES:
            a = np.zeros(count, dtype=npd)
            a["v"] = rng.integers(-2, 3, count)
            a["i"] = rng.integers(-1000, 1000, count)
        else:
            x = (rng.standard_normal(count) * 8).astype(np.float32)
            if r in (0, n - 1) and count:
                k = rng.integers(0, count, max(1, count // 8))
                x[k[0::3]] = np.nan
                x[k[1::3]] = 0.0
                x[k[2::3]] = -0.0
            a = ro.f32_to_bf16(x) if dtype == "bf16" else x.astype(npd)
        out.append(np.ascontiguousarray(a))
    return out


class Bufs:
    """One byte buffer per rank with every item's send and recv (a guard
    before each, ``shift`` bytes off 16-byte alignment), random and different
    on every rank.  Ranks in ``in_place`` pass each send as its recv."""

    def __init__(self, g, dtype, counts, exclusive, rng, shift=0, heap=True, in_place=()):
        n = g.size
        self.g, self.dtype, self.counts, self.exclusive = g, dtype, counts, exclusive
        es = ro.itemsize(dtype)
        self.send_offs, self.recv_offs, self.nbytes = [], [], 0
        for r in range(n):
            so, ro_ = [], []
            pos = GUARD + shift
            for c in counts:
                b = c * es
                so.append(pos)
                ro_.append(pos if r in in_place else (pos + b + 15) // 16 * 16 + GUARD + shift)
                pos = (ro_[-1] + b + 15) // 16 * 16 + GUARD + shift
            self.send_offs.append(so)
            self.recv_offs.append(ro_)
            self.nbytes = max(self.nbytes, pos + GUARD)
        self.init = [rng.integers(0, 256, self.nbytes, dtype=np.uint8) for _ in range(n)]
        self.ins = [inputs(rng, dtype, n, c) for c in counts]
        for i, c in enumerate(counts):
            for r in range(n):
                o = self.send_offs[r][i]
                self.init[r][o : o + c * es] = self.ins[i][r].view(np.uint8)
        if heap:
            self.t = [c.empty(self.nbytes, torch.uint8) for c in g.comms]
        else:
            dev = torch.device("cuda", g.devices[0])
            self.t = [torch.empty(self.nbytes, dtype=torch.uint8, device=dev) for _ in range(n)]
        self.heap = heap
        for t, a in zip(self.t, self.init):
            t.copy_(torch.from_numpy(a))
        torch.cuda.synchronize()

    def lists(self, r):
        """(sends, recvs) of rank r"""
        es = ro.itemsize(self.dtype)
        sends = [self.t[r][o : o + c * es] for o, c in zip(self.send_offs[r], self.counts)]
        return sends, [self.t[r][o : o + c * es] for o, c in zip(self.recv_offs[r], self.counts)]

    def expected(self, i, r, op):
        """rank r's result of item i; None where nothing is written"""
        k = r if self.exclusive else r + 1
        return ro.fold(self.ins[i][:k], self.dtype, op) if k > 0 and self.counts[i] else None

    def check(self, what, op):
        es = ro.itemsize(self.dtype)
        for r in range(self.g.size):
            got = self.t[r].cpu().numpy()
            want = self.init[r].copy()
            for i, c in enumerate(self.counts):
                exp = self.expected(i, r, op)
                if exp is None:
                    continue
                o = self.recv_offs[r][i]
                ro.assert_same(got[o : o + c * es].copy(), exp, self.dtype, f"{what}: rank {r} item {i}")
                # (bits compared above, NaN payloads and pair padding aside)
                want[o : o + c * es] = got[o : o + c * es]
            bad = np.nonzero(got != want)[0]
            assert bad.size == 0, f"{what}: rank {r} byte {bad[0]} changed outside its results"

    def free(self):
        if self.heap:
            for c, t in zip(self.g.comms, self.t):
                c.free(t)


def _run(g, fn):
    torch.cuda.synchronize()
    before = [c.stats()["launches"] for c in g.comms]
    g.run(fn)
    g.synchronize()
    assert g.check_errors() == [0] * g.size
    return [c.stats()["launches"] - b for c, b in zip(g.comms, before)]


def _case(g, dtype, op, counts, exclusive, rng, many, shift=0, heap=True, in_place=()):
    """One list through a plan or scan_many; returns the launches per rank."""
    bufs = Bufs(g, dtype, counts, exclusive, rng, shift, heap, in_place)
    plans = [None] * g.size
    try:
        for r, c in enumerate(g.comms):
            s, rv = bufs.lists(r)
            plans[r] = c.prepare_scan_group(s, rv, exclusive=exclusive, dtype=dtype)
        expect = plans[0].launches
        assert all(p.launches == expect for p in plans)

        def fn(c, r, st):
            if many:
                s, rv = bufs.lists(r)
                c.scan_many(s, rv, op=op, exclusive=exclusive, dtype=dtype)
            else:
                c.scan_group(plans[r], op=op)

        got = _run(g, fn)
        what = "exscan" if exclusive else "scan"
        bufs.check(f"{what} {dtype} {op} n={g.size} many={many} shift={shift} heap={heap} in_place={in_place}", op)
        if exclusive and g.size == 1:
            expect = 0  # nothing to write
        assert got == [expect] * g.size, (got, expect)
        return expect
    finally:
        for p in plans:
            if p is not None:
                p.close()
        bufs.free()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", NS)
def test_every_dtype_and_op(n, kind):
    g = group(n, kind)
    rng = np.random.default_rng([n, KINDS.index(kind)])
    for i, (dtype, op) in enumerate(ro.SUPPORTED):
        # a ragged length: whole chunks, a partial vector and a < 16-byte tail
        count = (5 * 2048 + 40) // ro.itemsize(dtype) + 1
        in_place = {r for r in range(n) if (r + i) % 3 == 0}
        _case(g, dtype, op, [count, 3], i % 2 == 1, rng, many=i // 2 % 2 == 1, shift=i % 3, in_place=in_place)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", NS)
def test_every_length(n, kind):
    g = group(n, kind)
    rng = np.random.default_rng([n, 5, KINDS.index(kind)])
    for exclusive in (False, True):
        # 3 MiB + 20 bytes per rank through a 1 MiB staging buffer: 4+ launches
        launches = _case(g, "f32", "sum", COUNTS, exclusive, rng, many=exclusive, shift=1 + exclusive)
        assert launches >= 4


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", [2, 4])
def test_cudamalloc_unaligned_and_in_place(n, kind):
    g = group(n, kind)
    rng = np.random.default_rng([n, 7, KINDS.index(kind)])
    counts = [4, 5, 1024, 1027, 17500]
    for heap in (False, True):
        for shift in (0, 1, 4):
            for exclusive in (False, True):
                # in place on rank 0 only, on every rank but 0, or nowhere
                in_place = [{0}, set(range(1, n)), set()][(shift + exclusive) % 3]
                dtype, op = ("bf16", "sum") if shift == 1 else ("i64", "max")
                _case(g, dtype, op, counts, exclusive, rng, many=exclusive, shift=shift, heap=heap, in_place=in_place)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", NS)
def test_resnet50_gradients_and_launch_boundaries(n, kind):
    rng = np.random.default_rng([n, 3, KINDS.index(kind)])
    # the 214 ResNet-50 fp32 gradient tensors; cudaMalloc buffers: 200 MiB
    # per rank.  Through 32 MiB staging buffers (the default): all ranks are
    # issued from this one thread, and a rank's stream must not hold more
    # work than the driver queues before its peers are issued.
    stage = 32 << 20
    sizes = resnet50_grad_sizes()
    cb = 1024 if n == 8 else 2048
    chunks = sum(-(-e * 4 // cb) for e in sizes)
    launches = _case(group(n, kind, stage), "f32", "sum", sizes, False, rng, many=False, heap=False)
    assert launches == -(-chunks // (stage // cb)) and launches >= 4
    g = group(n, kind)
    # every small item takes a whole chunk: a launch takes MAX_ITEMS of them
    # or as many as fit the staging buffer (MoE offsets: i64 exclusive sums)
    per = min(MAX_ITEMS, STAGE // cb)
    for k in (MAX_ITEMS, MAX_ITEMS + 1):
        assert _case(g, "i64", "sum", [1] * k, True, rng, many=k == MAX_ITEMS) == -(-k // per)


def test_one_rank():
    g = group(1, "stream")
    rng = np.random.default_rng([1, 13])
    counts = [3, 0, 1027, 17500]
    for exclusive in (False, True):
        for in_place in (set(), {0}):
            for many in (False, True):
                # a scan copies send to recv, an exscan writes nothing
                _case(g, "f32", "sum", counts, exclusive, rng, many=many, shift=1, in_place=in_place)


@pytest.mark.parametrize("kind", KINDS)
def test_sub_communicator_children(kind):
    g = group(8, kind)
    rng = np.random.default_rng([11, KINDS.index(kind)])
    for members in ([0, 2, 4, 6], [7, 6, 5, 4, 3, 2, 1, 0], [5, 2]):
        sub = g.subset(members)
        try:
            for exclusive in (False, True):
                # (cudaMalloc buffers: the heap is allocated on the whole parent)
                _case(sub, "f16", "max", [1, 2049, 150000, 5], exclusive, rng, many=exclusive, shift=1, heap=False,
                      in_place={1})
        finally:
            sub.close()


@pytest.mark.parametrize("n", NS)
def test_inclusive_matches_blocking_scan(n):
    g = group(n, "stream")
    rng = np.random.default_rng([n, 17])
    counts = [1, 7, 4099, 70001]
    for dtype, op in (("f32", "sum"), ("bf16", "sum"), ("f64", "prod"), ("i32", "max"), ("f32_i32", "minloc")):
        es = ro.itemsize(dtype)
        ins = [inputs(rng, dtype, n, c) for c in counts]
        t = {}
        for name in ("send", "grouped", "blocking"):
            t[name] = [[c.empty(k * es, torch.uint8) for k in counts] for c in g.comms]
        for r in range(n):
            for i in range(len(counts)):
                t["send"][r][i].copy_(torch.from_numpy(ins[i][r].view(np.uint8)))
        torch.cuda.synchronize()

        def fn(c, r, st):
            c.scan_many(t["send"][r], t["grouped"][r], op=op, dtype=dtype)
            for s, rv in zip(t["send"][r], t["blocking"][r]):
                c.scan(s, rv, op=op, dtype=dtype)

        _run(g, fn)
        for r in range(n):
            for i in range(len(counts)):
                a = t["grouped"][r][i].cpu().numpy()
                b = t["blocking"][r][i].cpu().numpy()
                assert np.array_equal(a, b), f"{dtype} {op} n={n}: rank {r} item {i} differs from the blocking scan"
        for name in t:
            for r, c in enumerate(g.comms):
                for x in t[name][r]:
                    c.free(x)


class _NoNative:
    def __getattr__(self, name):
        raise AssertionError(f"native call {name} made")


def test_refusals():
    g = group(2, "stream")
    c = g.comms[0]
    dev = torch.device("cuda", g.devices[0])
    send = torch.zeros(8, dtype=torch.float32, device=dev)
    recv = torch.zeros(8, dtype=torch.float32, device=dev)
    before = c.stats()["launches"]
    # bad lists, shapes, dtypes and tensors raise before any native call
    lib = c._lib
    c._lib = _NoNative()
    try:
        for exclusive in (False, True):
            for sends, recvs in (
                ([send], [recv, recv]),
                ([], []),
                ([send], None),
                (None, [recv]),
                ([send], [None]),
                ([None], [recv]),
                ([send], [torch.zeros(9, device=dev)]),
                ([send], [torch.zeros(8, dtype=torch.float64, device=dev)]),
                ([send], [torch.zeros(8, dtype=torch.int32, device=dev)]),
                ([send, send.to(torch.int32)], [recv, recv.to(torch.int32)]),
            ):
                with pytest.raises(CommError):
                    c.scan_many(sends, recvs, exclusive=exclusive)
            # host memory, another device's tensor or a strided view would be
            # loaded and stored as raw addresses: refused
            for bad in (send.cpu(), torch.zeros(8, 2, device=dev).t()[0], torch.zeros(16, device=dev)[::2]):
                with pytest.raises(CommError):
                    c.scan_many([bad], [recv], exclusive=exclusive)
                with pytest.raises(CommError):
                    c.scan_many([send], [bad], exclusive=exclusive)
    finally:
        c._lib = lib
    for exclusive in (False, True):
        with pytest.raises(CommError):
            c.scan_many([send], [recv], op="band", exclusive=exclusive)  # FB_E_UNSUPPORTED
    plan = c.prepare_scan_group([send], [recv])
    explan = c.prepare_scan_group([send], [recv], exclusive=True)
    reduce = c.prepare_reduce_group([send], [recv], root=0)
    try:
        with pytest.raises(CommError):
            c.reduce_group(plan, root=0)  # a plan of another kind
        with pytest.raises(CommError):
            c.scan_group(reduce)
        for p in (plan, explan):
            with pytest.raises(CommError):
                c.scan_group(p, op="bxor")  # no such reduction on f32
            with pytest.raises(CommError):
                c.scan_group(p, channel=1)  # one staging buffer per rank
    finally:
        plan.close()
        explan.close()
        reduce.close()
    # nothing was launched, so no peer is left waiting
    g.synchronize()
    assert g.check_errors() == [0] * g.size
    assert c.stats()["launches"] == before
