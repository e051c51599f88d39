"""Grouped neighbourhood v-collectives (neighbor_all_gather_v_many,
neighbor_all_to_all_v_many and their plans) against
``neighbor_v_oracle.neighbor_exchange_v``, byte for byte.

N ranks share one GPU inside this process, on the default group (ranks
sharing a GPU synchronise in stream order: LOCAL and MOVE are two launches)
and on a spin group whose kernels meet at in-kernel barriers (skipped where
the ranks' kernels are not co-resident).  A topology is set once per
communicator, so every graph runs on a fresh subset of all the ranks.  The
graphs are seeded random ones with self-edges, multi-edges and ranks of
degree 0; the counts are random per edge and item, with zero-count edges,
ranks whose counts are all zero, and blocks larger than a staging slot.  Every
rank's items sit in one byte buffer at odd offsets with random guard bytes
around them: every byte the oracle does not write must come back unchanged.
The agreement is the group's elementwise maximum of every rank's streams
(LocalGroup.agree_neighbor_v), and every rank must make the launches it
gives.
"""

import numpy as np
import pytest
import torch

import neighbor_v_oracle as nv

pytestmark = pytest.mark.gpu

from faabric_b200.parallel import LocalGroup  # noqa: E402
from faabric_b200.parallel.comm import CommError, neighbor_in_edges  # noqa: E402

NS = [2, 4, 8]
KINDS = ["stream", "spin"]
OPS = list(nv.KINDS)
GUARD = 8
# a small staging buffer, so that large blocks take several rounds
STAGE = 1 << 16

_GROUPS = {}


def group(n, kind):
    if (n, kind) not in _GROUPS:
        cfg = dict(heapBytes=96 << 20, stageBytes=STAGE, maxBlocks=8, timeoutMs=8000)
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


def random_count(rng):
    """Zero, a few bytes, ragged chunk ends, or more than a staging slot"""
    return int(rng.choice([0, 0, 1, 7, 2047, 2049, 9001, STAGE + 5, 3 * STAGE + 1]))


class Case:
    """Counts, displacements and one byte buffer per rank for a list of
    ``items`` calls of ``op`` over a graph.  ``count(i, s, k)`` is the byte
    count of item i on out-edge k of rank s (all-gather: k = 0, per rank)."""

    def __init__(self, sub, op, src, dst, items, rng, count, heap):
        self.sub, self.op, self.items = sub, op, items
        self.edges = neighbor_in_edges(src, dst)
        self.dst = dst
        n = sub.size
        a2a = op == "neighbor_all_to_all_v"
        self.nsend = [len(dst[r]) if a2a else min(len(dst[r]), 1) for r in range(n)]
        c = [[[count(i, s, k) for k in range(max(len(dst[s]), 1) if a2a else 1)] for s in range(n)] for i in range(items)]
        self.sc = [[c[i][s][: self.nsend[s]] if a2a else [c[i][s][0]] for i in range(items)] for s in range(n)]
        self.rc = [[[c[i][s][idx if a2a else 0] for s, idx in self.edges[d]] for i in range(items)] for d in range(n)]
        self.sd, self.rd, self.so, self.ro, self.sl, self.rl = ([[] for _ in range(n)] for _ in range(6))
        ends = []
        for r in range(n):
            pos = GUARD + 1 + int(rng.integers(5))
            for i in range(items):
                for counts, displs, offs, lens in ((self.sc[r][i], self.sd, self.so, self.sl),
                                                   (self.rc[r][i], self.rd, self.ro, self.rl)):
                    # blocks in a shuffled order with gaps, at odd offsets
                    at = [0] * len(counts)
                    p = 0
                    for k in rng.permutation(len(counts)):
                        p += int(rng.integers(3))
                        at[k] = p
                        p += counts[k]
                    displs[r].append(at)
                    offs[r].append(pos)
                    lens[r].append(p)
                    pos += p + GUARD + int(rng.integers(3))
            ends.append(pos + GUARD)
        self.nbytes = max(ends)
        self.heap = heap
        if heap:
            self.t = [sub.parent.comms[m].empty(self.nbytes, torch.uint8) for m in sub.members]
        else:
            dev = torch.device("cuda", sub.devices[0])
            self.t = [torch.empty(self.nbytes, dtype=torch.uint8, device=dev) for _ in range(n)]
        self.fill(rng)

    def fill(self, rng):
        self.init = [rng.integers(0, 256, self.nbytes, dtype=np.uint8) for _ in self.t]
        for t, a in zip(self.t, self.init):
            t.copy_(torch.from_numpy(a))
        torch.cuda.synchronize()

    def args(self, r):
        t = self.t[r]
        sends = [t[o : o + ln] for o, ln in zip(self.so[r], self.sl[r])]
        recvs = [t[o : o + ln] for o, ln in zip(self.ro[r], self.rl[r])]
        if self.op == "neighbor_all_to_all_v":
            return dict(sends=sends, recvs=recvs, sendcounts=self.sc[r], sdispls=self.sd[r],
                        recvcounts=self.rc[r], rdispls=self.rd[r])
        # (the all-gather's send is its one block, at displacement 0)
        sends = [t[o + d[0] : o + d[0] + c[0]] for o, d, c in zip(self.so[r], self.sd[r], self.sc[r])]
        return dict(sends=sends, recvs=recvs, sendcounts=[c[0] for c in self.sc[r]],
                    recvcounts=self.rc[r], rdispls=self.rd[r])

    def want(self):
        out = [a.copy() for a in self.init]
        n = len(out)
        a2a = self.op == "neighbor_all_to_all_v"
        for i in range(self.items):
            if a2a:
                sends = [self.init[r][self.so[r][i] :] for r in range(n)]
                sc = [self.sc[r][i] for r in range(n)]
                sd = [self.sd[r][i] for r in range(n)]
            else:
                sends = [self.init[r][self.so[r][i] + self.sd[r][i][0] :] for r in range(n)]
                sc = sd = None
            recvs = [out[r][self.ro[r][i] :] for r in range(n)]
            got = nv.neighbor_exchange_v(self.op, sends, recvs, self.edges,
                                         [self.rc[r][i] for r in range(n)], [self.rd[r][i] for r in range(n)],
                                         sendcounts=sc, sdispls=sd)
            for r in range(n):
                out[r][self.ro[r][i] :] = got[r]
        return out

    def agreed(self):
        """The oracle's agreement: per launch window, the longest stream of
        any rank"""
        n = len(self.t)
        w = nv.window_items(self.op, max(len(d) for d in self.dst), max(len(e) for e in self.edges))
        out = []
        for b in range(0, self.items, w):
            out.append(max(max(nv.stream_lengths(self.op, len(self.dst[r]), len(self.edges[r]),
                                                 self.sc[r][b : b + w], self.rc[r][b : b + w], 1), default=0)
                           for r in range(n)))
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


def fresh(g, src, dst):
    sub = g.subset(list(range(g.size)))
    sub.set_neighbors(src, dst)
    return sub


def launches(sub):
    return [c.stats()["launches"] for c in sub.comms]


def streams(sub, case):
    op = case.op
    return sub.run(lambda c, r, st: getattr(c, f"{op}_streams")(**case.args(r)))


def run_case(sub, case, many):
    """One exchange of the case (plans or *_many); returns (agreed, launches
    per rank)"""
    n = sub.size
    op = case.op
    mine = streams(sub, case)
    agreed = LocalGroup.agree_neighbor_v(mine)
    assert agreed == case.agreed()
    plans = [None] * n
    if not many:
        plans = sub.run(lambda c, r, st: getattr(c, f"prepare_{op}_group")(agreed=agreed, **case.args(r)))
    before = launches(sub)
    if many:
        sub.run(lambda c, r, st: getattr(c, f"{op}_many")(agreed=agreed, stream=st, **case.args(r)))
    else:
        sub.run(lambda c, r, st: getattr(c, f"{op}_group")(plans[r], stream=st))
    sub.synchronize()
    assert sub.check_errors() == [0] * n
    case.check()
    made = [a - b for a, b in zip(launches(sub), before)]
    want = nv.launches(agreed, STAGE, max(len(d) for d in case.dst), op)
    assert made == [want] * n, (made, want, agreed)
    for p in plans:
        if p is not None:
            assert p.launches == want
            p.close()
    return mine, agreed, want


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
            # every count of this rank is 0 (all-to-all: its recv counts too)
            quiet = int(rng.integers(n))
            a2a = op == "neighbor_all_to_all_v"
            count = lambda i, s, k: (  # noqa: E731
                0 if s == quiet or (a2a and k < len(dst[s]) and dst[s][k] == quiet) else random_count(rng)
            )
            for heap, many in ((True, False), (False, True)):
                case = Case(sub, op, src, dst, 5, rng, count, heap)
                run_case(sub, case, many)
                case.close()
        finally:
            sub.close()


@pytest.mark.parametrize("op", OPS)
def test_many_items_take_several_windows(op):
    """1100 small items over a degree-3 graph: more items than one launch's
    table holds, so the list runs as several windows, each agreed alone"""
    g = group(4, "stream")
    rng = np.random.default_rng(77)
    dst = [[1, 2, 3], [2, 3, 0], [3, 0, 1], [0, 1, 2]]
    src = [[d for d in range(4) for x in dst[d] if x == r] for r in range(4)]
    sub = fresh(g, src, dst)
    try:
        case = Case(sub, op, src, dst, 1100, rng, lambda i, s, k: int(rng.integers(0, 40)), True)
        assert len(case.agreed()) >= 2
        for many in (False, True):
            case.fill(rng)
            run_case(sub, case, many)
        case.close()
    finally:
        sub.close()


@pytest.mark.parametrize("kind", KINDS)
def test_one_large_edge_sets_every_ranks_rounds(kind):
    """One edge, 0 -> 1, carries more than the staging slot; every other edge
    a few bytes.  The ranks' own streams then need different round counts
    (ranks 2 and 3 alone would launch once), but the agreement gives every
    rank the same launches, and the exchange completes and matches."""
    g = group(4, kind)
    rng = np.random.default_rng(5)
    dst = [[1, 2], [0, 3], [3, 1], [2, 0]]
    src = [[d for d in range(4) for x in dst[d] if x == r] for r in range(4)]
    sub = fresh(g, src, dst)
    try:
        for op in OPS:
            big = lambda i, s, k: 5 * STAGE + 3 if (s == 0 and k == 0 and i == 1) else 11  # noqa: E731
            case = Case(sub, op, src, dst, 3, rng, big, True)
            mine, agreed, want = run_case(sub, case, True)
            local = [nv.launches(m, STAGE, 2, op) for m in mine]
            assert len(set(local)) > 1 and want == max(local) > 1, (local, want)
            case.close()
    finally:
        sub.close()


def test_equal_counts_match_the_equal_block_kind():
    """A v list whose counts are all equal moves what the equal-block
    neighbour all-to-all moves, bit for bit"""
    g = group(4, "stream")
    rng = np.random.default_rng(9)
    src, dst = random_graph(4, rng)
    while not any(dst):
        src, dst = random_graph(4, rng)
    sub = fresh(g, src, dst)
    try:
        block = 3001
        edges = neighbor_in_edges(src, dst)
        dev = torch.device("cuda", sub.devices[0])
        sends = [torch.from_numpy(rng.integers(0, 256, block * len(dst[r]), dtype=np.uint8)).to(dev) for r in range(4)]
        ra = [torch.zeros(block * len(edges[r]), dtype=torch.uint8, device=dev) for r in range(4)]
        rb = [torch.ones(block * len(edges[r]), dtype=torch.uint8, device=dev) for r in range(4)]
        sub.run(lambda c, r, st: c.neighbor_all_to_all_many([sends[r]], [ra[r]], counts=[block], stream=st))
        sub.synchronize()
        args = lambda r: dict(  # noqa: E731
            sends=[sends[r]], recvs=[rb[r]], sendcounts=[[block] * len(dst[r])],
            sdispls=[[k * block for k in range(len(dst[r]))]], recvcounts=[[block] * len(edges[r])],
            rdispls=[[j * block for j in range(len(edges[r]))]])
        agreed = LocalGroup.agree_neighbor_v(sub.run(lambda c, r, st: c.neighbor_all_to_all_v_streams(**args(r))))
        sub.run(lambda c, r, st: c.neighbor_all_to_all_v_many(agreed=agreed, stream=st, **args(r)))
        sub.synchronize()
        assert sub.check_errors() == [0] * 4
        for a, b in zip(ra, rb):
            assert torch.equal(a, b)
    finally:
        sub.close()


def test_refusals_raise_before_any_launch():
    g = group(2, "stream")
    c = g.comms[0]
    t = torch.zeros(64, dtype=torch.uint8, device=f"cuda:{c.device}")
    sub = g.subset([0, 1])
    try:
        with pytest.raises(CommError, match="no neighbourhood topology"):
            sub.comms[0].neighbor_all_gather_v_many([t], [t], [[1]], [[0]], agreed=[1])
        sub.set_neighbors([[1], [0]], [[1], [0]])
        c0 = sub.comms[0]
        before = launches(sub)
        with pytest.raises(CommError, match="negative"):
            c0.neighbor_all_to_all_v_many([t], [t], [[-1]], [[0]], [[1]], [[0]], agreed=[1])
        with pytest.raises(CommError, match="overruns"):
            c0.neighbor_all_to_all_v_many([t], [t], [[60]], [[10]], [[1]], [[0]], agreed=[60])
        with pytest.raises(CommError, match="counts and displacements"):
            c0.neighbor_all_to_all_v_many([t], [t], [[1, 1]], [[0, 1]], [[1]], [[0]], agreed=[2])
        # an agreement below this rank's own stream, or of the wrong length
        with pytest.raises(CommError):
            c0.neighbor_all_to_all_v_many([t], [t], [[8]], [[0]], [[8]], [[0]], agreed=[7])
        with pytest.raises(CommError):
            c0.neighbor_all_to_all_v_many([t], [t], [[8]], [[0]], [[8]], [[0]], agreed=[8, 8])
        with pytest.raises(CommError):
            c0.prepare_neighbor_all_gather_v_group([t], [t], [[8]], [[0]], agreed=[], sendcounts=[8])
        assert launches(sub) == before
    finally:
        sub.close()
