"""Sub-communicators of a LocalGroup on the GPU: every fused collective over
member subsets in child order, on heap and local buffers, with the default
stream-ordered wiring and with in-kernel barriers (spin).  Results are exact
(int32) closed forms over the members; the child's statistics never count LL
or NVLS and the parent's launch count does not move during child calls."""

import pytest
import torch

pytestmark = pytest.mark.gpu

from faabric_b200.parallel import LocalGroup  # noqa: E402
from faabric_b200.parallel.comm import CommError  # noqa: E402

N = 4100  # int32 per rank and chunk: reduce-scatter slices are 16-byte multiples
MEMBER_SETS = [
    [0, 1, 2, 3],
    [4, 5, 6, 7],
    [0, 2, 4, 6],
    [1, 3, 5, 7],
    [5, 2, 7, 0],
    [3, 6],
    [4],
    [7, 6, 5, 4, 3, 2, 1, 0],
]
_GROUPS = {}


def group(kind):
    if kind not in _GROUPS:
        cfg = dict(heapBytes=64 << 20, stageBytes=8 << 20, maxBlocks=8, timeoutMs=8000)
        if kind == "spin":
            cfg.update(maxBlocks=4, timeoutMs=4000, streamSync=0)
        g = LocalGroup(8, **cfg)
        if kind == "spin" and g.shares_devices and not g.coresident():
            g.close()
            g = None
        else:
            # heap tensors at the same offsets on every rank
            g.heap = [(c.empty(8 * N, torch.int32), c.empty(8 * N, torch.int32)) for c in g.comms]
        _GROUPS[kind] = g
    g = _GROUPS[kind]
    if g is None:
        pytest.skip("kernels of 8 ranks are not co-resident on this GPU")
    return g


@pytest.fixture(scope="module", autouse=True)
def _cleanup():
    yield
    for g in _GROUPS.values():
        if g is not None:
            g.close()
    _GROUPS.clear()


def vals(w, dev, scale=1):
    return (torch.arange(N, dtype=torch.int32, device=dev) % 97 + 1000 * w) * scale


def run_all(g, sub, members, heap):
    """Every collective on `sub`; returns {name: [per child rank result]}."""
    n = len(members)
    out = {}

    def bufs(i):
        c = g.comms[members[i]]
        dev = f"cuda:{c.device}"
        if heap:
            a, b = g.heap[members[i]]
            return a, b
        return torch.empty(8 * N, dtype=torch.int32, device=dev), torch.empty(8 * N, dtype=torch.int32, device=dev)

    ab = [bufs(i) for i in range(n)]

    def step(name, fn):
        res = sub.run(lambda c, i, st: fn(c, i, st, *ab[i]))
        sub.synchronize()
        assert sub.check_errors() == [0] * n, name
        out[name] = [r.cpu() if r is not None else None for r in res]

    def fill(a, i, scale=1):
        a[:N].copy_(vals(members[i], a.device, scale))

    def allreduce(algo):
        def f(c, i, st, a, b):
            fill(a, i)
            c.all_reduce(a[:N], b[:N], algo=algo, stream=st)
            return b[:N].clone()

        return f

    for algo in ("auto", "oneshot", "twoshot"):
        step(f"allreduce-{algo}", allreduce(algo))

    def reduce(c, i, st, a, b):
        fill(a, i)
        b[:N].fill_(-1)
        c.reduce(a[:N], b[:N], root=n - 1, op="max", stream=st)
        return b[:N].clone()

    step("reduce", reduce)

    def reduce_scatter(c, i, st, a, b):
        for j in range(n):
            a[j * N : (j + 1) * N].copy_(vals(members[i], a.device) + j)
        c.reduce_scatter(a[: n * N], b[:N], stream=st)
        return b[:N].clone()

    step("reduce_scatter", reduce_scatter)

    def scan(c, i, st, a, b):
        fill(a, i)
        c.scan(a[:N], b[:N], stream=st)
        return b[:N].clone()

    step("scan", scan)

    root = 1 if n > 1 else 0

    def bcast(c, i, st, a, b):
        if i == root:
            fill(b, i, 3)
        else:
            b[:N].fill_(-1)
        c.broadcast(b[:N], root=root, stream=st)
        return b[:N].clone()

    step("bcast", bcast)

    def allgather(c, i, st, a, b):
        fill(a, i)
        c.all_gather(a[:N], b[: n * N], stream=st)
        return b[: n * N].clone()

    step("allgather", allgather)

    def gather(c, i, st, a, b):
        fill(a, i)
        c.gather(a[:N], b[: n * N], root=0, stream=st)
        return b[: n * N].clone() if i == 0 else None

    step("gather", gather)

    def scatter(c, i, st, a, b):
        for j in range(n):
            a[j * N : (j + 1) * N].copy_(vals(members[i], a.device) * 2 + j)
        c.scatter(a[: n * N], b[:N], root=n - 1, stream=st)
        return b[:N].clone()

    step("scatter", scatter)

    def alltoall(c, i, st, a, b):
        for j in range(n):
            a[j * N : (j + 1) * N].copy_(vals(members[i], a.device) + 7 * j)
        c.all_to_all(a[: n * N], b[: n * N], stream=st)
        return b[: n * N].clone()

    step("alltoall", alltoall)
    step("barrier", lambda c, i, st, a, b: c.barrier(stream=st))
    return out


def check(out, members):
    n = len(members)
    v = [vals(w, "cpu") for w in members]
    total = sum(v)
    for algo in ("auto", "oneshot", "twoshot"):
        for i in range(n):
            assert torch.equal(out[f"allreduce-{algo}"][i], total), (algo, i)
    top = max(members)
    assert torch.equal(out["reduce"][n - 1], vals(top, "cpu"))
    for i in range(n):
        assert torch.equal(out["reduce_scatter"][i], total + n * i), i
        assert torch.equal(out["scan"][i], sum(v[: i + 1])), i
        assert torch.equal(out["bcast"][i], v[1 if n > 1 else 0] * 3), i
        assert torch.equal(out["allgather"][i], torch.cat(v)), i
        assert torch.equal(out["scatter"][i], v[n - 1] * 2 + i), i
        assert torch.equal(out["alltoall"][i], torch.cat([v[j] + 7 * i for j in range(n)])), i
    assert torch.equal(out["gather"][0], torch.cat(v))


@pytest.mark.parametrize("kind", ["stream", "spin"])
@pytest.mark.parametrize("members", MEMBER_SETS, ids=lambda m: "-".join(map(str, m)))
def test_subset_collectives(kind, members):
    g = group(kind)
    g.synchronize()
    parent_launches = [c.stats()["launches"] for c in g.comms]
    sub = g.subset(members)
    try:
        assert [c.rank for c in sub.comms] == list(range(len(members)))
        assert all(c.size == len(members) and c.is_subset for c in sub.comms)
        for heap in (True, False):
            check(run_all(g, sub, members, heap), members)
        for c in sub.comms:
            st = c.stats()
            assert st["launches"] > 0 and st["algo_ll"] == 0 and st["algo_nvls"] == 0
        assert [c.stats()["launches"] for c in g.comms] == parent_launches
        with pytest.raises(CommError):
            sub.comms[0].empty(16)
        with pytest.raises(CommError):
            sub.comms[0].all_reduce(g.heap[members[0]][0][:4], algo="ll")
    finally:
        sub.close()
    assert all(g.comms[m].free_subset_slots() == (1 << 15) - 1 for m in members)


@pytest.mark.parametrize("kind", ["stream", "spin"])
def test_disjoint_children_at_the_same_time(kind):
    g = group(kind)
    lo, hi = g.subset([0, 1, 2, 3]), g.subset([7, 6, 5, 4])
    try:
        assert lo.slot == hi.slot == 0  # disjoint members: the same slot
        # one pass over all eight ranks: both children issue before either waits
        subs = [(lo, i) for i in range(4)] + [(hi, i) for i in range(4)]
        outs = []
        for s, i in subs:
            c = s.comms[i]
            a, _ = g.heap[s.members[i]]
            with torch.cuda.device(c.device):
                st = s.streams[i]
                st.wait_stream(torch.cuda.current_stream(c.device))
                with torch.cuda.stream(st):
                    a[:N].copy_(vals(s.members[i], a.device))
                    r = torch.empty(N, dtype=torch.int32, device=a.device)
                    c.all_reduce(a[:N], r, stream=st)
                    outs.append(r)
        lo.synchronize()
        hi.synchronize()
        for k, (s, i) in enumerate(subs):
            assert torch.equal(outs[k].cpu(), sum(vals(w, "cpu") for w in s.members)), (s.members, i)
    finally:
        lo.close()
        hi.close()


@pytest.mark.parametrize("kind", ["stream", "spin"])
def test_child_and_parent_alternate(kind):
    g = group(kind)
    members = [6, 1, 3]
    sub = g.subset(members)
    try:
        for rnd in range(50):
            if rnd % 2 == 0:

                def f(c, i, st):
                    a, b = g.heap[members[i]]
                    a[:N].copy_(vals(members[i], a.device, rnd + 1))
                    c.all_reduce(a[:N], b[:N], stream=st)
                    return b[:N]

                res = sub.run(f)
                want = sum(vals(w, "cpu", rnd + 1) for w in members)
            else:

                def f(c, r, st):
                    a, b = g.heap[r]
                    a[:N].copy_(vals(r, a.device, rnd + 1))
                    c.all_reduce(a[:N], b[:N], stream=st)
                    return b[:N]

                res = g.run(f)
                want = sum(vals(w, "cpu", rnd + 1) for w in range(8))
            g.synchronize()
            for r in res:
                assert torch.equal(r.cpu(), want), rnd
        assert g.check_errors() == [0] * 8
    finally:
        sub.close()


def test_slot_released_and_retaken_by_other_members():
    g = group("stream")
    first = g.subset([0, 1, 2, 3])
    held = g.subset([0, 4])  # slot 1 on ranks 0 and 4
    assert (first.slot, held.slot) == (0, 1)
    check(run_all(g, first, [0, 1, 2, 3], True), [0, 1, 2, 3])
    first.close()
    assert g.comms[1].free_subset_slots() & 1
    # another member set takes slot 0 again, across the released pads
    again = g.subset([3, 1, 5, 2])
    try:
        assert again.slot == 0
        check(run_all(g, again, [3, 1, 5, 2], True), [3, 1, 5, 2])
        check(run_all(g, held, [0, 4], False), [0, 4])
    finally:
        again.close()
        held.close()
    assert all(c.free_subset_slots() == (1 << 15) - 1 for c in g.comms)
