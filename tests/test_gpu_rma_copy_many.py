"""Batched one-sided copies (Communicator.put_many / get_many, the
rmaCopyManyKernel behind MPI_Rput / MPI_Rget), byte for byte against NumPy.

All ranks share cuda:0, so "peer" memory is the same GPU's HBM reached through
the peer mapping the kernel uses for any peer.  The kernel never waits on a
peer, so no co-residency is needed.

* Every length of {1, 3, 15, 16, 17, 31, 4103, 1 MiB + 5} crossed with source
  and destination offsets mod 16 in {0, 1, 4, 8, 15}, in one list per rank:
  item k of rank r goes to (or comes from) rank (r + k) % n, so every list
  mixes this rank and other peers, and every destination slot has exactly one
  writer.  Every byte of every window and local buffer is compared with a
  NumPy model that starts from random bytes, so the guard bytes around each
  copy are checked too, and sources are checked unchanged.
* Lists of 1, 1000 and two launches' capacity + 3 items take exactly the
  launches they need (one per 1024 items).
* Refusals (outside the heap, a bad peer, a child communicator) raise before
  any launch."""

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from faabric_b200.parallel import LocalGroup  # noqa: E402
from faabric_b200.parallel.comm import CommError  # noqa: E402

DEV = "cuda:0"
LENGTHS = [1, 3, 15, 16, 17, 31, 4103, (1 << 20) + 5]
SHIFTS = [0, 1, 4, 8, 15]
PAIRS = [(s, d) for s in SHIFTS for d in SHIFTS]
CAPACITY = 1024  # items per launch (FB_RMA_COPY_MAX_ITEMS)
FB_E_INVALID = -2
FB_E_UNSUPPORTED = -1
MAX_SLOT = ((1 << 20) + 5 + 48 + 15) // 16 * 16
WIN = len(PAIRS) * MAX_SLOT
CFG = dict(heapBytes=WIN + (8 << 20), stageBytes=1 << 20, maxBlocks=4, timeoutMs=8000)

GROUPS = {}


def group(n):
    if n not in GROUPS:
        g = LocalGroup(n, devices=[0] * n, **CFG)
        g.wins = [c.empty(WIN, torch.uint8) for c in g.comms]
        g.locs = [torch.empty(WIN, dtype=torch.uint8, device=DEV) for _ in range(n)]
        GROUPS[n] = g
    return GROUPS[n]


@pytest.fixture(scope="module", autouse=True)
def _cleanup():
    yield
    for g in GROUPS.values():
        g.close()
    GROUPS.clear()


def _randomise(rng, tensors):
    """Fills every tensor with random bytes; returns the NumPy models."""
    models = []
    for t in tensors:
        a = rng.integers(0, 256, t.numel(), dtype=np.uint8)
        t.copy_(torch.from_numpy(a))
        models.append(a)
    torch.cuda.synchronize()
    return models


def _launches(g):
    return [c.stats()["launches"] for c in g.comms]


def _assert_bytes(got, want, what):
    got = got.cpu().numpy()
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{what}: {bad.size} bytes differ, first at {bad[0]} (got {got[bad[0]]}, want {want[bad[0]]})"


@pytest.mark.parametrize("n", [2, 4, 8])
@pytest.mark.parametrize("length", LENGTHS)
@pytest.mark.parametrize("direction", ["put", "get"])
def test_every_length_and_alignment(n, length, direction):
    g = group(n)
    slot = (length + 48 + 15) // 16 * 16
    rng = np.random.default_rng(length * 31 + n * 7 + (direction == "get"))
    wins = _randomise(rng, g.wins)
    locs = _randomise(rng, g.locs)
    lists = []
    for r in range(n):
        items = []
        for k, (so, do) in enumerate(PAIRS):
            peer = (r + k) % n
            base = k * slot + 16
            if direction == "put":
                # local source at shift so, remote destination at shift do
                items.append((g.locs[r][base + so : base + so + length], g.wins[r][base + do : base + do + length], peer))
                wins[peer][base + do : base + do + length] = locs[r][base + so : base + so + length]
            else:
                items.append((g.locs[r][base + do : base + do + length], g.wins[r][base + so : base + so + length], peer))
                locs[r][base + do : base + do + length] = wins[peer][base + so : base + so + length]
        lists.append(items)
    before = _launches(g)

    def issue(c, r, st):
        loc, sym, peers = zip(*lists[r])
        if direction == "put":
            c.put_many(list(loc), list(sym), list(peers), stream=st)
        else:
            c.get_many(list(loc), list(sym), list(peers), stream=st)

    g.run(issue)
    g.synchronize()
    assert g.check_errors() == [0] * n
    assert _launches(g) == [b + 1 for b in before]
    for r in range(n):
        _assert_bytes(g.wins[r], wins[r], f"{direction} n={n} len={length}: window of rank {r}")
        _assert_bytes(g.locs[r], locs[r], f"{direction} n={n} len={length}: local buffer of rank {r}")


@pytest.mark.parametrize("n", [2, 4, 8])
@pytest.mark.parametrize("count", [1, 1000, 2 * CAPACITY + 3])
def test_list_lengths_take_the_launches_they_need(n, count):
    """Many small records at odd displacements (zero-byte items mixed into the
    list of 1000): one launch per CAPACITY non-empty items, every record
    exact, sources unchanged."""
    g = group(n)
    rng = np.random.default_rng(count + 100 * n)
    wins = _randomise(rng, g.wins)
    locs = _randomise(rng, g.locs)
    stride = 48
    lens = rng.integers(1, 41, count)
    if count == 1000:
        lens[::97] = 0  # skipped: they take no room in a launch
    lists = []
    for r in range(n):
        items = []
        for k in range(count):
            peer = int(rng.integers(0, n))
            ln = int(lens[k])
            soff = k * stride + 1 + (k % 7)
            doff = (r * count + k) * stride + 3 + (k % 5)
            # (the symmetric side is this rank's view of the window: its
            # heap offset names the same bytes in the peer's heap)
            items.append((g.locs[r][soff : soff + ln], g.wins[r][doff : doff + ln], peer))
            wins[peer][doff : doff + ln] = locs[r][soff : soff + ln]
        lists.append(items)
    before = _launches(g)
    src_before = [t.clone() for t in g.locs]

    def issue(c, r, st):
        loc, sym, peers = zip(*lists[r])
        c.put_many(list(loc), list(sym), list(peers), stream=st)

    g.run(issue)
    g.synchronize()
    assert g.check_errors() == [0] * n
    need = -(-int((lens > 0).sum()) // CAPACITY)
    assert need == (3 if count > 2 * CAPACITY else 1)
    assert _launches(g) == [b + need for b in before]
    for r in range(n):
        _assert_bytes(g.wins[r], wins[r], f"{count} records, window of rank {r}")
        assert torch.equal(g.locs[r], src_before[r])


def test_get_many_reads_what_put_many_wrote():
    g = group(4)
    n = g.size
    rng = np.random.default_rng(5)
    _randomise(rng, g.wins)
    recs = [torch.from_numpy(rng.integers(0, 256, 24 * 256, dtype=np.uint8)).to(DEV) for _ in range(n)]
    back = [torch.zeros(24 * 256 * n, dtype=torch.uint8, device=DEV) for _ in range(n)]
    torch.cuda.synchronize()

    def put(c, r, st):
        srcs, dsts, peers = [], [], []
        for t in range(n):
            for i in range(256):
                off = 1 + (r * 256 + i) * 25
                srcs.append(recs[r][24 * i : 24 * i + 24])
                dsts.append(g.wins[r][off : off + 24])
                peers.append(t)
        c.put_many(srcs, dsts, peers, stream=st)

    g.run(put)
    g.synchronize()

    def get(c, r, st):
        dsts, srcs, peers = [], [], []
        for o in range(n):
            for i in range(256):
                off = 1 + (o * 256 + i) * 25
                dsts.append(back[r][(o * 256 + i) * 24 :][:24])
                srcs.append(g.wins[r][off : off + 24])
                peers.append((r + o) % n)
        c.get_many(dsts, srcs, peers, stream=st)

    g.run(get)
    g.synchronize()
    assert g.check_errors() == [0] * n
    for r in range(n):
        assert torch.equal(back[r], torch.cat(recs))


def test_refusals_raise_before_any_launch():
    g = group(2)
    c = g.comms[0]
    w = g.wins[0]
    src = torch.ones(64, dtype=torch.uint8, device=DEV)
    before = _launches(g)
    with pytest.raises(CommError):  # symmetric side not in the heap
        c.put_many([src], [torch.zeros(64, dtype=torch.uint8, device=DEV)], [1])
    with pytest.raises(CommError):  # byte sizes differ
        c.put_many([src], [w[:63]], [1])
    with pytest.raises(CommError):  # peer outside the group
        c.put_many([src, src], [w[:64], w[64:128]], [1, 2])
    with pytest.raises(CommError):
        c.get_many([src], [w[:64]], [-1])
    with pytest.raises(CommError):  # list lengths differ
        c.get_many([src, src], [w[:64]], [1])
    with pytest.raises(CommError):  # local side not on the device
        c.put_many([torch.ones(64, dtype=torch.uint8)], [w[:64]], [1])
    # the native checks: every item before anything is launched; the last
    # item here is past the end of the heap, wraps around, sits below the
    # user heap, or names a bad peer
    st = torch.cuda.current_stream().cuda_stream
    lib = c._lib
    import ctypes as C

    good = c.heap_offset(w)
    for off, peer in ((1 << 40, 1), ((1 << 64) - 16, 1), (0, 1), (good, 2)):
        n = 3
        rc = lib.fb_put_get_many(
            c._h,
            n,
            (C.c_void_p * n)(*([src.data_ptr()] * n)),
            (C.c_uint64 * n)(good, good + 64, off),
            (C.c_uint64 * n)(64, 64, 64),
            (C.c_int32 * n)(1, 0, peer),
            (C.c_int32 * n)(0, 1, 0),
            st,
        )
        assert rc == FB_E_INVALID, (off, peer, rc)
    sub = g.subset([0, 1])
    try:
        with pytest.raises(CommError):
            sub.comms[0].put_many([src], [w[:64]], [1])
        rc = lib.fb_put_get_many(
            sub.comms[0]._h, 1, (C.c_void_p * 1)(src.data_ptr()), (C.c_uint64 * 1)(good), (C.c_uint64 * 1)(64), (C.c_int32 * 1)(1), (C.c_int32 * 1)(0), st
        )
        assert rc == FB_E_UNSUPPORTED
    finally:
        sub.close()
    torch.cuda.synchronize()
    assert _launches(g) == before
    assert g.check_errors() == [0, 0]
