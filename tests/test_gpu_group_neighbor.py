"""Grouped neighbourhood all-gather and all-to-all (neighbor_all_gather_many,
neighbor_all_to_all_many and their plans) against
``neighbor_oracle.neighbor_exchange``, byte for byte.

N ranks share one GPU inside this process, on the default group (ranks
sharing a GPU synchronise in stream order: the LOCAL and MOVE steps are two
launches) and on a spin group whose kernels meet at in-kernel barriers
(skipped where the ranks' kernels are not co-resident).  A topology is set
once per communicator, so every graph runs on a fresh subset of all the
ranks.  The graphs are seeded random ones with self-edges, multi-edges and
ranks of degree 0.  Every rank's items sit in one byte buffer (symmetric
heap or cudaMalloc) at offsets that may be unaligned, with random guard
bytes around every item: every byte the oracle does not write must come back
unchanged, and the communicator's stats must show one launch per plan
launch.
"""

import numpy as np
import pytest
import torch

import neighbor_oracle as no

pytestmark = pytest.mark.gpu

from faabric_b200.parallel import LocalGroup  # noqa: E402
from faabric_b200.parallel.comm import CommError, neighbor_in_edges  # noqa: E402

NS = [2, 3, 4, 5, 8]
KINDS = ["stream", "spin"]
OPS = list(no.KINDS)
GUARD = 32
STAGE = 1 << 20
# bytes per block: one byte, zero, odd lengths, ragged chunk ends (2 KiB
# chunks), and more than a launch's staging room
BYTES = [1, 0, 5, 2049, 70001, STAGE + 17]

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


def random_graph(n, rng, max_deg=3):
    """(sources, destinations) per rank: about a third of the ranks send
    nothing, the others 1..max_deg edges to random ranks (self and repeated
    targets included)."""
    dst = [[] for _ in range(n)]
    src = [[] for _ in range(n)]
    start = int(rng.integers(3))
    for r in range(n):
        deg = 0 if (r + start) % 3 == 0 else 1 + int(rng.integers(max_deg))
        for _ in range(deg):
            t = int(rng.integers(n))
            dst[r].append(t)
            src[t].append(r)
    for v in src:
        rng.shuffle(v)
    return src, dst


class Bufs:
    """One byte buffer per rank with every item's send and recv (a guard
    before each, ``shift`` bytes off 16-byte alignment), random and different
    on every rank."""

    def __init__(self, sub, op, src, dst, sizes, rng, shift=0, heap=True):
        self.sub, self.op, self.sizes = sub, op, sizes
        self.edges = neighbor_in_edges(src, dst)
        n = sub.size
        a2a = op == "neighbor_all_to_all"
        self.sblocks = [len(dst[r]) if a2a else 1 for r in range(n)]
        self.indeg = [len(e) for e in self.edges]
        self.send_offs = [[] for _ in range(n)]
        self.recv_offs = [[] for _ in range(n)]
        ends = []
        for r in range(n):
            pos = GUARD + shift
            for b in sizes:
                self.send_offs[r].append(pos)
                pos = (pos + b * self.sblocks[r] + 15) // 16 * 16 + GUARD + shift
                self.recv_offs[r].append(pos)
                pos = (pos + b * self.indeg[r] + 15) // 16 * 16 + GUARD + shift
            ends.append(pos + GUARD)
        # (heap allocations are collective: the same size everywhere)
        self.nbytes = max(ends)
        self.heap = heap
        parent = sub.parent
        if heap:
            self.t = [parent.comms[m].empty(self.nbytes, torch.uint8) for m in sub.members]
        else:
            dev = torch.device("cuda", sub.devices[0])
            self.t = [torch.empty(self.nbytes, dtype=torch.uint8, device=dev) for _ in range(n)]
        self.fill(rng)

    def fill(self, rng):
        self.init = [rng.integers(0, 256, self.nbytes, dtype=np.uint8) for _ in self.t]
        for t, a in zip(self.t, self.init):
            t.copy_(torch.from_numpy(a))
        torch.cuda.synchronize()

    def lists(self, r):
        sends = [self.t[r][o : o + b * self.sblocks[r]] for o, b in zip(self.send_offs[r], self.sizes)]
        recvs = [self.t[r][o : o + b * self.indeg[r]] for o, b in zip(self.recv_offs[r], self.sizes)]
        return sends, recvs

    def want(self):
        """Every rank's whole buffer after the exchange, item by item."""
        out = [a.copy() for a in self.init]
        for i, b in enumerate(self.sizes):
            sends = [a[o[i] : o[i] + b * s] for a, o, s in zip(self.init, self.send_offs, self.sblocks)]
            out = no.neighbor_exchange(self.op, sends, out, self.edges, b, offset=[o[i] for o in self.recv_offs])
        return out

    def check(self):
        torch.cuda.synchronize()
        want = self.want()
        for r, t in enumerate(self.t):
            got = t.cpu().numpy()
            bad = np.nonzero(got != want[r])[0]
            assert bad.size == 0, f"{self.op}: rank {r} differs at {bad[:8]} of {self.nbytes} bytes"

    def close(self):
        if self.heap:
            for m, t in zip(self.sub.members, self.t):
                self.sub.parent.comms[m].free(t)
        self.t = []


def expected_launches(op, sizes, dst):
    """Launches of a list: 2 KiB chunks per block, and a launch's staging
    room shared by the largest out-degree's slots (all-to-all)"""
    chunks = sum((b + 2047) // 2048 for b in sizes)
    slots = max(max(len(d) for d in dst), 1) if op == "neighbor_all_to_all" else 1
    room = STAGE // 2048 // slots
    return (chunks + room - 1) // room


def fresh(g, src, dst):
    sub = g.subset(list(range(g.size)))
    sub.set_neighbors(src, dst)
    return sub


def launches(sub):
    return [c.stats()["launches"] for c in sub.comms]


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", NS)
def test_random_graphs_byte_for_byte(n, kind, op):
    g = group(n, kind)
    rng = np.random.default_rng(1000 * n + 10 * KINDS.index(kind) + OPS.index(op))
    for graph in range(2):
        src, dst = random_graph(n, rng)
        sub = fresh(g, src, dst)
        try:
            for heap, shift, many in ((True, 0, False), (False, 3, True), (True, 5, True)):
                b = Bufs(sub, op, src, dst, BYTES, rng, shift=shift, heap=heap)
                plans = [None] * n
                if not many:
                    plans = sub.run(lambda c, r, st: getattr(c, f"prepare_{op}_group")(*b.lists(r), counts=b.sizes))
                before = launches(sub)
                if many:
                    sub.run(lambda c, r, st: getattr(c, f"{op}_many")(*b.lists(r), counts=b.sizes, stream=st))
                else:
                    sub.run(lambda c, r, st: getattr(c, f"{op}_group")(plans[r], stream=st))
                sub.synchronize()
                assert sub.check_errors() == [0] * n
                b.check()
                # every rank makes the launches the counts and the staging
                # room give, none when no rank has an edge
                after = launches(sub)
                want = 0 if not any(dst) else expected_launches(op, BYTES, dst)
                if plans[0] is not None:
                    assert plans[0].launches == expected_launches(op, BYTES, dst)
                assert [a - bf for a, bf in zip(after, before)] == [want] * n
                for p in plans:
                    if p is not None:
                        p.close()
                b.close()
        finally:
            sub.close()


@pytest.mark.parametrize("kind", KINDS)
def test_halo_plan_reused_40_rounds(kind):
    """The 2 x 2 periodic halo (left, right, down, up) of five fields: one
    plan, 40 launches with rewritten inputs, each checked."""
    g = group(4, kind)
    rng = np.random.default_rng(40)
    px, py = 2, 2
    nbrs = []
    for r in range(4):
        x, y = r % px, r // px
        nbrs.append([((x - 1) % px) + y * px, ((x + 1) % px) + y * px, x + ((y - 1) % py) * px, x + ((y + 1) % py) * px])
    sub = fresh(g, nbrs, nbrs)
    try:
        b = Bufs(sub, "neighbor_all_to_all", nbrs, nbrs, [4096 * 4] * 5, rng, shift=0, heap=True)
        plans = sub.run(lambda c, r, st: c.prepare_neighbor_all_to_all_group(*b.lists(r)))
        assert plans[0].launches == 1
        for _ in range(40):
            b.fill(rng)
            before = launches(sub)
            sub.run(lambda c, r, st: c.neighbor_all_to_all_group(plans[r], stream=st))
            sub.synchronize()
            assert [a - bf for a, bf in zip(launches(sub), before)] == [1] * 4
            b.check()
        for p in plans:
            p.close()
        b.close()
    finally:
        sub.close()


def test_refusals_raise_before_any_launch():
    g = group(2, "stream")
    c = g.comms[0]
    t = torch.zeros(64, dtype=torch.uint8, device=f"cuda:{c.device}")
    sub = g.subset([0, 1])
    try:
        with pytest.raises(CommError, match="no neighbourhood topology"):
            sub.comms[0].neighbor_all_gather_many([t], [t])
        sub.set_neighbors([[1], [0]], [[1], [0]])
        with pytest.raises(CommError, match="set_neighbors"):
            sub.comms[0].set_neighbors([(1, 0)], 1, 1, 1)
        before = launches(sub)
        # recv must hold one block per in-edge
        with pytest.raises(CommError, match="blocks"):
            sub.comms[0].neighbor_all_to_all_many([t[:16]], [t[:32]])
        with pytest.raises(CommError, match="non-empty"):
            sub.comms[0].neighbor_all_gather_many([], [])
        with pytest.raises(CommError):
            sub.set_neighbors([[1], []], [[1], [0]])
        assert launches(sub) == before
    finally:
        sub.close()
