"""Launch, staging-copy, byte and algorithm counts of every grouped kind.

Each of the 14 kinds runs one small fixed list through its plan and through
``*_many``, on a one-rank group (no barriers: every phase in one launch) and on
two ranks sharing cuda:0 (stream-ordered barriers: one kernel run per phase,
the runs beyond the first counted as staged copies).  The rooted and
neighbour lists have an item larger than the staging buffer, so they take
several launches; the v lists have more items than one launch window holds
and a first window longer than a staging slot, so they take several windows
and rounds.  Every rank's deltas of ``launches``, ``staged_copies``, ``bytes``
and ``algo_twoshot``, and the plan's launches, are checked against constants.
"""

import pytest
import torch

pytestmark = pytest.mark.gpu

from faabric_b200.parallel import LocalGroup  # noqa: E402

STAGE = 1 << 16
# (sources, destinations) per rank: a self-edge on one rank; on two, rank 0
# sends to both ranks and rank 1 to rank 0
GRAPHS = {1: ([[0]], [[0]]), 2: ([[1, 0], [0]], [[1, 0], [0]])}

# float32 elements per item: whole 16-byte vectors for the two-shot kinds,
# one item larger than the staging buffer for the rooted and neighbour kinds
TWO_SHOT = [1024, 256, 4096]
ROOTED = [1000, 40000, 16]
NEIGHBOR = [1000, 20000, 16]
# v lists: bytes per edge of each item
V_ITEMS = 1100
V_BIG = 100000

# kind -> n -> (launches, staged copies, bytes per rank, two-shot launches,
# plan launches), for one call
EXPECT = {
    "all_reduce": {1: (1, 0, (21504,), 1, 1), 2: (1, 0, (21504, 21504), 1, 1)},
    "reduce_scatter": {1: (1, 0, (21504,), 0, 1), 2: (1, 0, (43008, 43008), 0, 1)},
    "all_gather": {1: (1, 0, (21504,), 0, 1), 2: (1, 0, (43008, 43008), 0, 1)},
    # (one member: the root's buffers already hold the result)
    "broadcast": {1: (0, 0, (0,), 0, 1), 2: (1, 0, (21504, 21504), 0, 1)},
    "all_to_all": {1: (1, 0, (21504,), 0, 1), 2: (1, 0, (43008, 43008), 0, 1)},
    "gather": {1: (3, 0, (164064,), 0, 3), 2: (3, 3, (328128, 328128), 0, 3)},
    "scatter": {1: (3, 0, (164064,), 0, 3), 2: (3, 3, (328128, 328128), 0, 3)},
    "reduce": {1: (3, 0, (164064,), 0, 3), 2: (3, 6, (328128, 328128), 0, 3)},
    "scan": {1: (3, 0, (164064,), 0, 3), 2: (3, 6, (328128, 328128), 0, 3)},
    # (one member: an exscan writes nothing)
    "exscan": {1: (0, 0, (0,), 0, 3), 2: (3, 6, (328128, 328128), 0, 3)},
    "neighbor_all_gather": {1: (2, 0, (84064,), 0, 2), 2: (2, 2, (168128, 84064), 0, 2)},
    "neighbor_all_to_all": {1: (2, 0, (84064,), 0, 2), 2: (3, 3, (168128, 84064), 0, 3)},
    "neighbor_all_gather_v": {1: (3, 0, (101099,), 0, 3), 2: (3, 3, (202198, 101099), 0, 3)},
    "neighbor_all_to_all_v": {1: (3, 0, (101099,), 0, 3), 2: (6, 6, (202198, 101099), 0, 6)},
}

_GROUPS = {}


def group(n):
    if n not in _GROUPS:
        g = LocalGroup(n, devices=[0] * n, heapBytes=64 << 20, stageBytes=STAGE, maxBlocks=8, timeoutMs=8000)
        g.set_neighbors(*GRAPHS[n])
        _GROUPS[n] = g
    return _GROUPS[n]


@pytest.fixture(scope="module", autouse=True)
def _cleanup():
    yield
    for g in _GROUPS.values():
        g.close()
    _GROUPS.clear()


def dev_zeros(numel, dtype=torch.float32):
    return torch.zeros(numel, dtype=dtype, device="cuda:0")


def lists(kind, g, r):
    """Rank r's arguments of the prepare call (the *_many call takes the same)"""
    n, c = g.size, g.comms[r]
    root = n - 1
    if kind == "all_reduce":
        return dict(sends=[c.zeros(k) for k in TWO_SHOT])
    if kind == "broadcast":
        return dict(bufs=[c.zeros(k) for k in TWO_SHOT])
    if kind == "reduce_scatter":
        return dict(sends=[c.zeros(n * k) for k in TWO_SHOT], recvs=[c.zeros(k) for k in TWO_SHOT])
    if kind == "all_gather":
        return dict(sends=[c.zeros(k) for k in TWO_SHOT], recvs=[c.zeros(n * k) for k in TWO_SHOT])
    if kind == "all_to_all":
        return dict(sends=[c.zeros(n * k) for k in TWO_SHOT], recvs=[c.zeros(n * k) for k in TWO_SHOT])
    if kind == "gather":
        return dict(sends=[dev_zeros(k) for k in ROOTED],
                    recvs=[dev_zeros(n * k) if r == root else None for k in ROOTED], root=root)
    if kind == "scatter":
        return dict(sends=[dev_zeros(n * k) if r == root else None for k in ROOTED],
                    recvs=[dev_zeros(k) for k in ROOTED], root=root)
    if kind == "reduce":
        return dict(sends=[dev_zeros(k) for k in ROOTED],
                    recvs=[dev_zeros(k) if r == root else None for k in ROOTED], root=root)
    if kind in ("scan", "exscan"):
        return dict(sends=[dev_zeros(k) for k in ROOTED], recvs=[dev_zeros(k) for k in ROOTED])
    src, dst = GRAPHS[n]
    outdeg, indeg = len(dst[r]), len(src[r])
    if kind in ("neighbor_all_gather", "neighbor_all_to_all"):
        blocks = outdeg if kind == "neighbor_all_to_all" else 1
        return dict(sends=[dev_zeros(blocks * k) for k in NEIGHBOR],
                    recvs=[dev_zeros(indeg * k) for k in NEIGHBOR], counts=NEIGHBOR)
    # v lists of bytes: every edge of item i carries the same count
    counts = [V_BIG] + [1] * (V_ITEMS - 1)
    a2a = kind == "neighbor_all_to_all_v"
    blocks = outdeg if a2a else 1
    sbuf = dev_zeros(blocks * sum(counts), torch.uint8)
    rbuf = dev_zeros(indeg * sum(counts), torch.uint8)
    sends, recvs, so, ro = [], [], 0, 0
    for k in counts:
        sends.append(sbuf[so : so + blocks * k])
        recvs.append(rbuf[ro : ro + indeg * k])
        so += blocks * k
        ro += indeg * k
    args = dict(sends=sends, recvs=recvs, recvcounts=[[k] * indeg for k in counts],
                rdispls=[[j * k for j in range(indeg)] for k in counts])
    if a2a:
        args.update(sendcounts=[[k] * outdeg for k in counts], sdispls=[[j * k for j in range(outdeg)] for k in counts])
    else:
        args.update(sendcounts=counts)
    return args


PREPARE = {"all_reduce": "prepare_group", "exscan": "prepare_scan_group"}
LAUNCH = {"exscan": "scan_group"}
MANY = {"exscan": "scan_many"}


def call(kind, c, st, args, plan):
    """One call of ``kind`` on communicator c: the plan's launch, or the
    transient *_many call when plan is None"""
    extra = dict(exclusive=True) if kind == "exscan" else {}
    if plan is not None:
        kw = {"root": args["root"]} if "root" in args else {}
        if kind == "broadcast":
            kw["root"] = c.size - 1
        getattr(c, LAUNCH.get(kind, f"{kind}_group"))(plan, stream=st, **kw)
    elif kind == "broadcast":
        c.broadcast_many(args["bufs"], root=c.size - 1, stream=st)
    else:
        getattr(c, MANY.get(kind, f"{kind}_many"))(stream=st, **args, **extra)


def snapshot(g):
    return [c.stats() for c in g.comms]


@pytest.mark.parametrize("many", [False, True], ids=["plan", "many"])
@pytest.mark.parametrize("kind", list(EXPECT))
@pytest.mark.parametrize("n", [1, 2])
def test_counts(n, kind, many):
    g = group(n)
    args = [lists(kind, g, r) for r in range(n)]
    if kind.endswith("_v"):
        name = kind[: -len("_v")] + "_v_streams"
        mine = g.run(lambda c, r, st: getattr(c, name)(**args[r]))
        agreed = LocalGroup.agree_neighbor_v(mine)
        for a in args:
            a["agreed"] = agreed
    plans = [None] * n
    if not many:
        extra = dict(exclusive=True) if kind == "exscan" else {}
        plans = g.run(lambda c, r, st: getattr(c, PREPARE.get(kind, f"prepare_{kind}_group"))(**args[r], **extra))
    g.synchronize()
    before = snapshot(g)
    g.run(lambda c, r, st: call(kind, c, st, args[r], plans[r]))
    g.synchronize()
    assert g.check_errors() == [0] * n
    after = snapshot(g)
    launches, staged, nbytes, twoshot, plan_launches = EXPECT[kind][n]
    for r in range(n):
        got = {k: after[r][k] - before[r][k] for k in ("launches", "staged_copies", "bytes", "algo_twoshot")}
        want = dict(launches=launches, staged_copies=staged, bytes=nbytes[r], algo_twoshot=twoshot)
        assert got == want, f"{kind}, rank {r} of {n}"
    for p in plans:
        if p is not None:
            assert p.launches == plan_launches
            p.close()
    # (free() leaves tensors outside the heap alone)
    for r, a in enumerate(args):
        for key in ("sends", "recvs", "bufs"):
            for t in a.get(key, []):
                if t is not None:
                    g.comms[r].free(t)
