"""Grouped gather and scatter (one launch per staging buffer of a list)
against ``move_oracle.gather`` / ``move_oracle.scatter``, byte for byte.

N ranks share one GPU inside this process, on the default group (ranks
sharing a GPU synchronise in stream order: the LOCAL and MOVE steps are two
launches) and on a spin group whose kernels meet at in-kernel barriers
(skipped where the ranks' kernels are not co-resident).  Every rank's items
sit in one byte buffer (symmetric heap or cudaMalloc) at offsets that may be
unaligned, with random guard bytes around every item: every byte the oracle
does not write must come back unchanged, and the communicator's stats must
show one launch per plan launch.
"""

import numpy as np
import pytest
import torch

import move_oracle as mo

pytestmark = pytest.mark.gpu

from faabric_b200.models.resnet50_grads import resnet50_grad_sizes  # noqa: E402
from faabric_b200.parallel import LocalGroup  # noqa: E402
from faabric_b200.parallel.comm import CommError  # noqa: E402

NS = [2, 4, 8]
KINDS = ["stream", "spin"]
OPS = ["gather", "scatter"]
GUARD = 32
STAGE = 1 << 20
MAX_ITEMS = 1016  # FB_GROUP_MAX_SEGS - 8 pieces per launch
# bytes per rank: one byte, zero, odd lengths, ragged chunk ends (the chunk
# is 1 KiB at 8 ranks, 2 KiB otherwise), whole chunks, and more than the
# 1 MiB staging buffer
BYTES = [1, 0, 5, 48, 2049, 129 * 16, 65 * 16 + 3, 300000, 3 * STAGE + 17]

_GROUPS = {}


def group(n, kind):
    if (n, kind) not in _GROUPS:
        cfg = dict(heapBytes=160 << 20, stageBytes=STAGE, maxBlocks=8, timeoutMs=8000)
        if kind == "spin":
            cfg.update(maxBlocks=4, groupBlocks=8, timeoutMs=4000, streamSync=0)
        g = LocalGroup(n, **cfg)
        if kind == "spin" and g.shares_devices and not g.coresident():
            g.close()
            g = None
        _GROUPS[(n, kind)] = g
    g = _GROUPS[(n, kind)]
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


class Bufs:
    """One byte buffer per rank with every item's send and recv (a guard
    before each, `shift` bytes off 16-byte alignment), random and different
    on every rank.  ``in_place``: the root's send (gather) or recv (scatter)
    is its own block of the other buffer."""

    def __init__(self, g, op, sizes, root, rng, shift=0, heap=True, in_place=False):
        self.g, self.op, self.sizes, self.root = g, op, sizes, root
        n = g.size
        self.in_place = in_place
        self.send_offs = [[] for _ in range(n)]
        self.recv_offs = [[] for _ in range(n)]
        pos = GUARD + shift
        for b in sizes:
            big = b * n
            small_first, big_off = pos, (pos + b + 15) // 16 * 16 + GUARD + shift
            pos = (big_off + big + 15) // 16 * 16 + GUARD + shift
            for r in range(n):
                if op == "gather":
                    own = in_place and r == root
                    self.send_offs[r].append(big_off + root * b if own else small_first)
                    self.recv_offs[r].append(big_off)
                else:
                    own = in_place and r == root
                    self.send_offs[r].append(big_off)
                    self.recv_offs[r].append(big_off + root * b if own else small_first)
        self.nbytes = pos + GUARD
        self.init = [rng.integers(0, 256, self.nbytes, dtype=np.uint8) for _ in range(n)]
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
        """(sends, recvs) of rank r: the root-only side is None elsewhere."""
        n = self.g.size
        small, big = (1, n) if self.op == "gather" else (n, 1)
        sends = [self.t[r][o : o + b * small] for o, b in zip(self.send_offs[r], self.sizes)]
        recvs = [self.t[r][o : o + b * big] for o, b in zip(self.recv_offs[r], self.sizes)]
        if r != self.root:
            if self.op == "gather":
                recvs = None
            else:
                sends = None
        return sends, recvs

    def free(self):
        if self.heap:
            for c, t in zip(self.g.comms, self.t):
                c.free(t)

    def check(self, what):
        n = self.g.size
        want = [b.copy() for b in self.init]
        fn = mo.gather if self.op == "gather" else mo.scatter
        for i, b in enumerate(self.sizes):
            if b:
                # (the oracle on the item's extent of every buffer: it copies
                # whole buffers)
                so = [self.send_offs[r][i] for r in range(n)]
                ro = [self.recv_offs[r][i] for r in range(n)]
                lo, hi = min(so + ro), max(so + ro) + b * n
                got = fn([w[lo:hi] for w in want], [o - lo for o in so], [w[lo:hi] for w in want], [o - lo for o in ro], b, self.root)
                for w, g in zip(want, got):
                    w[lo:hi] = g
        for r in range(n):
            got = self.t[r].cpu().numpy()
            assert np.array_equal(got, want[r]), f"{what}: rank {r} first difference {mo.first_difference(got, want[r])}"


def _run(g, fn):
    torch.cuda.synchronize()
    before = [c.stats()["launches"] for c in g.comms]
    g.run(fn)
    g.synchronize()
    assert g.check_errors() == [0] * g.size
    return [c.stats()["launches"] - b for c, b in zip(g.comms, before)]


def _case(g, op, sizes, root, rng, many, shift=0, heap=True, in_place=False, dtype=None):
    """One list through a plan or *_many; returns the launches per rank."""
    bufs = Bufs(g, op, sizes, root, rng, shift, heap, in_place)
    plans = [None] * g.size
    try:
        for r, c in enumerate(g.comms):
            s, rv = bufs.lists(r)
            prep = c.prepare_gather_group if op == "gather" else c.prepare_scatter_group
            plans[r] = prep(s, rv, root=root, dtype=dtype)
        expect = plans[0].launches
        assert all(p.launches == expect for p in plans)

        def fn(c, r, st):
            if many:
                s, rv = bufs.lists(r)
                (c.gather_many if op == "gather" else c.scatter_many)(s, rv, root=root, dtype=dtype)
            else:
                (c.gather_group if op == "gather" else c.scatter_group)(plans[r], root=root)

        got = _run(g, fn)
        bufs.check(f"{op} n={g.size} root={root} many={many} shift={shift} heap={heap} in_place={in_place}")
        assert got == [expect] * g.size, (got, expect)
        return expect
    finally:
        for p in plans:
            if p is not None:
                p.close()
        bufs.free()


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", NS)
def test_every_root_and_length(n, kind, op):
    g = group(n, kind)
    rng = np.random.default_rng([n, KINDS.index(kind), OPS.index(op)])
    for root in range(n):
        # 3 MiB + 17 bytes per rank through a 1 MiB staging buffer: 4+ launches
        launches = _case(g, op, BYTES, root, rng, many=root % 2 == 1, shift=root % 3)
        assert launches >= 4


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", [2, 4])
def test_cudamalloc_unaligned_and_in_place(n, kind, op):
    g = group(n, kind)
    rng = np.random.default_rng([n, 7, KINDS.index(kind), OPS.index(op)])
    sizes = [16, 5, 4096, 4099, 70000]
    for heap in (False, True):
        for shift in (0, 1, 4):
            for in_place in (False, True):
                root = (shift + in_place) % n
                _case(g, op, sizes, root, rng, many=in_place, shift=shift, heap=heap, in_place=in_place)


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", NS)
def test_resnet50_shards_and_launch_boundaries(n, kind, op):
    g = group(n, kind)
    rng = np.random.default_rng([n, 3, KINDS.index(kind), OPS.index(op)])
    # each rank's 1/n shard of every ResNet-50 tensor (fp32), as in a
    # full-state-dict save or load
    shards = [(e + n - 1) // n * 4 for e in resnet50_grad_sizes()]
    # pieces fill each launch's staging chunks: 1 KiB at 8 ranks, 2 KiB else
    cb = 1024 if n == 8 else 2048
    chunks = sum(-(-b // cb) for b in shards)
    assert _case(g, op, shards, 0, rng, many=False) == -(-chunks // (STAGE // cb))
    # every small item takes a whole chunk: a launch takes MAX_ITEMS of them
    # or as many as fit the staging buffer
    per = min(MAX_ITEMS, STAGE // cb)
    for k in (MAX_ITEMS, MAX_ITEMS + 1):
        assert _case(g, op, [4] * k, n - 1, rng, many=k == MAX_ITEMS) == -(-k // per)


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("kind", KINDS)
def test_sub_communicator_children(kind, op):
    g = group(8, kind)
    rng = np.random.default_rng([11, KINDS.index(kind), OPS.index(op)])
    for members in ([0, 2, 4, 6], [7, 6, 5, 4, 3, 2, 1, 0], [5, 2]):
        sub = g.subset(members)
        try:
            for root in (0, len(members) - 1):
                # (cudaMalloc buffers: the heap is allocated on the whole parent)
                _case(sub, op, [1, 2049, 300000, 5], root, rng, many=root == 0, shift=1, heap=False)
        finally:
            sub.close()


class _NoNative:
    def __getattr__(self, name):
        raise AssertionError(f"native call {name} made")


@pytest.mark.parametrize("op", OPS)
def test_refusals(op):
    g = group(2, "stream")
    c = g.comms[0]
    dev = torch.device("cuda", g.devices[0])
    small = torch.zeros(8, dtype=torch.float32, device=dev)
    big = torch.zeros(16, dtype=torch.float32, device=dev)
    sends, recvs = ([small], [big]) if op == "gather" else ([big], [small])
    many = c.gather_many if op == "gather" else c.scatter_many
    prep = c.prepare_gather_group if op == "gather" else c.prepare_scatter_group
    launch = c.gather_group if op == "gather" else c.scatter_group
    other = c.scatter_group if op == "gather" else c.gather_group
    # bad shapes and roots raise before any native call
    lib = c._lib
    c._lib = _NoNative()
    try:
        with pytest.raises(CommError):
            many(sends, recvs, root=2)
        with pytest.raises(CommError):
            many(sends, recvs, root=-1)
        bad = [torch.zeros(3, device=dev)]
        with pytest.raises(CommError):
            many(sends, bad, root=0) if op == "gather" else many(bad, recvs, root=0)
        with pytest.raises(CommError):
            # the root's side is required on the root
            many(sends, None, root=0) if op == "gather" else many(None, recvs, root=0)
        with pytest.raises(CommError):
            many([], [], root=0)
        # host memory, another device's tensor or a strided view would be
        # loaded and stored as raw addresses: refused
        for bad in (small.cpu(), torch.zeros(16, 2, device=dev).t()[0], torch.zeros(32, device=dev)[::2]):
            one = bad[: small.numel()] if bad.numel() >= small.numel() else bad
            with pytest.raises(CommError):
                many([one], recvs, root=0) if op == "gather" else many(sends, [one], root=0)
    finally:
        c._lib = lib
    plan = prep(sends, recvs, root=0)
    try:
        with pytest.raises(CommError):
            other(plan, root=0)  # a plan of the other kind
        with pytest.raises(CommError):
            launch(plan, root=1)  # the plan was prepared for root 0
        plan.root = 5
        with pytest.raises(CommError):
            launch(plan, root=5)  # the native root check
        plan.root = 0
        with pytest.raises(CommError):
            launch(plan, root=0, channel=1)  # one staging buffer per rank
    finally:
        plan.close()
    # nothing was launched, so no peer is left waiting
    g.synchronize()
    assert g.check_errors() == [0] * g.size
