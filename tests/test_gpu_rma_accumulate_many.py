"""Batched one-sided atomics (Communicator.accumulate_many, the
rmaAccumulateManyKernel behind MPI_Raccumulate / MPI_Rget_accumulate bursts),
byte for byte against a NumPy model that applies every list in order.

All ranks share cuda:0, so "peer" memory is the same GPU's HBM reached through
the peer mapping the kernel uses for any peer.  The kernel never waits on a
peer, so no co-residency is needed.

* Every (dtype, op) of tests/rma_oracle.py's fetch set (REPLACE, NO_OP with
  fetch, the 16-byte pairs with their padding), fetching and plain items mixed
  in one list, to this rank and to others, with items that repeat an earlier
  target so that chains run for every pair.
* Lengths from one element to 1 MiB + 1 element; lists of 1, 1000 and 2051
  items.
* Order: an f32 sum whose result depends on it, REPLACE where the last item
  wins, 1024 fetching increments of one counter that fetch 0 .. 1023 in list
  order in one launch.
* The launch count of every list is the documented rule's
  (Communicator::accumulateMany), modelled in ``launches_of``.
* All ranks updating the same integer counters at once end exact.
* Refusals raise before any launch and leave the targets unchanged.

Every target and fetch buffer sits among random guard bytes that must stay as
they were, and origins must be unchanged."""

import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import rma_oracle as rm
from reduce_oracle import NP_DTYPES, itemsize
from test_gpu_reduce_matrix import make_inputs

pytestmark = pytest.mark.gpu

from faabric_b200.parallel import LocalGroup  # noqa: E402
from faabric_b200.parallel.comm import CommError  # noqa: E402

DEV = "cuda:0"
WIN = 10 << 20  # eight writers' regions of a little over 1 MiB each
CFG = dict(heapBytes=WIN + (8 << 20), stageBytes=1 << 20, maxBlocks=4, timeoutMs=8000)
CAPACITY = 1024  # descriptors per launch (FB_RMA_ACC_MAX_ITEMS)
CHAIN_BYTES = 16384  # FB_RMA_ACC_CHAIN_BYTES
FB_E_INVALID = -2
FB_E_UNSUPPORTED = -1

GROUPS = {}


def group(n):
    if n not in GROUPS:
        g = LocalGroup(n, devices=[0] * n, **CFG)
        g.wins = [c.empty(WIN, torch.uint8) for c in g.comms]
        g.orgs = [torch.empty(WIN, dtype=torch.uint8, device=DEV) for _ in range(n)]
        g.fets = [torch.empty(WIN, dtype=torch.uint8, device=DEV) for _ in range(n)]
        GROUPS[n] = g
    return GROUPS[n]


@pytest.fixture(scope="module", autouse=True)
def _cleanup():
    yield
    for g in GROUPS.values():
        g.close()
    GROUPS.clear()


def launches_of(items):
    """Launches the documented rule takes for a list of (peer, offset, bytes):
    a launch takes the next non-empty item unless it would be the 1025th, would
    intersect two chains, or would bring its chain above CHAIN_BYTES."""
    count = 0
    spans = None  # [peer, lo, hi, bytes] per chain of the current launch
    taken = 0
    for peer, off, nb in items:
        if nb == 0:
            continue
        for _ in range(2):
            if spans is not None:
                hits = [s for s in spans if s[0] == peer and s[1] < off + nb and off < s[2]]
                if taken < CAPACITY and len(hits) <= 1 and (not hits or hits[0][3] + nb <= CHAIN_BYTES):
                    if hits:
                        h = hits[0]
                        h[1], h[2], h[3] = min(h[1], off), max(h[2], off + nb), h[3] + nb
                    else:
                        spans.append([peer, off, off + nb, nb])
                    taken += 1
                    break
            spans, taken = [], 0
            count += 1
    return count


def _stats(g):
    return [c.stats()["launches"] for c in g.comms]


def _np(t):
    return t.cpu().numpy()


class Lists:
    """Per-rank item lists with their NumPy models: windows, origin and fetch
    buffers start as random bytes; every target range is set to values of the
    (dtype, op) once, before the first item that touches it."""

    def __init__(self, g, dtype, op, seed):
        self.g, self.dtype, self.op = g, dtype, op
        self.e = itemsize(dtype)
        self.rng = np.random.default_rng(seed)
        self.wins = [self.rng.integers(0, 256, WIN, dtype=np.uint8) for _ in range(g.size)]
        self.orgs = [self.rng.integers(0, 256, WIN, dtype=np.uint8) for _ in range(g.size)]
        self.fets = [self.rng.integers(0, 256, WIN, dtype=np.uint8) for _ in range(g.size)]
        self.ocur = [0] * g.size
        self.fcur = [0] * g.size
        self.items = [[] for _ in range(g.size)]
        self.targets = set()

    def _take(self, cur, r, nbytes, shift):
        base = (cur[r] + 15) // 16 * 16 + 16 + shift
        cur[r] = base + nbytes
        assert cur[r] + 16 <= WIN
        return base

    def add(self, r, peer, toff, count, fetch, oshift=3, fshift=5):
        """Item of rank r: `count` elements at window offset `toff` of `peer`."""
        e, nb = self.e, count * self.e
        if (peer, toff, count) not in self.targets:
            self.targets.add((peer, toff, count))
            tgt, _ = make_inputs(self.rng, self.dtype, self.op, 2, count)
            tgt = np.ascontiguousarray(tgt).view(np.uint8).copy()
            if self.dtype in rm.PADDED_PAIRS:
                tgt.reshape(-1, 16)[:, 12:] = self.rng.integers(1, 255, (count, 4), dtype=np.uint8)
            self.wins[peer][toff : toff + nb] = tgt
        o = None
        if self.op != "no_op":
            o = self._take(self.ocur, r, nb, oshift)
            org = make_inputs(self.rng, self.dtype, self.op, 2, count)[1]
            self.orgs[r][o : o + nb] = np.ascontiguousarray(org).view(np.uint8)
        f = self._take(self.fcur, r, nb, fshift) if fetch else None
        self.items[r].append((o, f, peer, toff, count))

    def run(self):
        g, e = self.g, self.e
        for r in range(g.size):
            g.wins[r].copy_(torch.from_numpy(self.wins[r]))
            g.orgs[r].copy_(torch.from_numpy(self.orgs[r]))
            g.fets[r].copy_(torch.from_numpy(self.fets[r]))
        torch.cuda.synchronize()
        before = _stats(g)

        def issue(c, r, st):
            srcs, dsts, peers, fetches = [], [], [], []
            for o, f, peer, toff, count in self.items[r]:
                nb = count * e
                srcs.append(None if o is None else g.orgs[r][o : o + nb])
                dsts.append(g.wins[r][toff : toff + nb])
                peers.append(peer)
                fetches.append(None if f is None else g.fets[r][f : f + nb])
            c.accumulate_many(srcs, dsts, peers, op=self.op, dtype=self.dtype, fetches=fetches, stream=st)

        g.run(issue)
        g.synchronize()
        assert g.check_errors() == [0] * g.size
        # the model: rank after rank (their targets are disjoint), list order
        mask = [np.zeros(WIN, dtype=bool) for _ in range(g.size)]
        fmask = [np.zeros(WIN, dtype=bool) for _ in range(g.size)]
        for r in range(g.size):
            for o, f, peer, toff, count in self.items[r]:
                nb = count * e
                old = self.wins[peer][toff : toff + nb].view(NP_DTYPES[self.dtype])
                org = None if o is None else self.orgs[r][o : o + nb].view(NP_DTYPES[self.dtype])
                new, fetched = rm.accumulate(old, org, self.dtype, self.op)
                self.wins[peer][toff : toff + nb] = new.view(np.uint8)
                mask[peer][toff : toff + nb] = True
                if f is not None:
                    self.fets[r][f : f + nb] = fetched.view(np.uint8)
                    fmask[r][f : f + nb] = True
        what = f"{self.dtype} {self.op}"
        for r in range(g.size):
            for got, want, m, name in ((_np(g.wins[r]), self.wins[r], mask[r], "window"), (_np(g.fets[r]), self.fets[r], fmask[r], "fetch buffer")):
                bad = np.flatnonzero((got != want) & ~m)
                assert bad.size == 0, f"{what}: {bad.size} guard bytes of rank {r}'s {name} changed, first at {bad[0]}"
                for lo, hi in _runs(m):
                    rm.assert_same(got[lo:hi].view(NP_DTYPES[self.dtype]), want[lo:hi].view(NP_DTYPES[self.dtype]), self.dtype, f"{what}: rank {r}'s {name} [{lo}, {hi})")
            assert np.array_equal(_np(g.orgs[r]), self.orgs[r]), f"{what}: rank {r}'s origins changed"
        got = [a - b for a, b in zip(_stats(g), before)]
        want = [launches_of([(peer, toff, count * e) for _, _, peer, toff, count in self.items[r]]) for r in range(g.size)]
        assert got == want, f"{what}: launches {got}, the rule gives {want}"
        return got


def _runs(mask):
    """[lo, hi) of every run of True in a boolean array."""
    d = np.diff(np.concatenate(([0], mask.astype(np.int8), [0])))
    return zip(np.flatnonzero(d == 1), np.flatnonzero(d == -1))


@pytest.mark.parametrize("dtype,op", rm.FETCH, ids=[f"{d}-{o}" for d, o in rm.FETCH])
def test_every_pair_with_mixed_fetch_and_chains(dtype, op):
    """Writer 0 sends one list to itself and rank 1: lengths 1, 3, 17 and 4099
    elements, every other item fetching (every item for NO_OP), then two items
    that repeat the targets of the first two (chains)."""
    g = group(2)
    L = Lists(g, dtype, op, seed=zlib.crc32(f"{dtype}-{op}".encode()))
    e = L.e
    toff = 4096
    for k, count in enumerate([1, 3, 17, 4099, 2, 64]):
        L.add(0, k % 2, toff, count, fetch=op == "no_op" or k % 2 == 0, oshift=k % 16, fshift=(5 * k) % 16)
        toff += (count * e + 64) // 16 * 16 + 16
    first = L.items[0][0]
    second = L.items[0][1]
    L.add(0, first[2], first[3], first[4], fetch=True)
    L.add(0, second[2], second[3], second[4], fetch=op == "no_op")
    assert L.run() == [1, 0]


@pytest.mark.parametrize("n", [2, 4, 8])
@pytest.mark.parametrize("dtype,op", [("i32", "sum"), ("f64", "sum"), ("u8", "bxor"), ("f16", "max")])
def test_lengths_up_to_one_mib_and_one_element(n, dtype, op):
    g = group(n)
    L = Lists(g, dtype, op, seed=n * 1000 + len(dtype))
    e = L.e
    for r in range(n):
        toff = r * (WIN // n) + 64
        for k, count in enumerate([1, 2, 31, 33, 1000, (1 << 20) // e + 1]):
            L.add(r, (r + k) % n, toff, count, fetch=k % 2 == 1, oshift=(k * 3) % 16, fshift=k % 16)
            toff += (count * e + 32) // 16 * 16 + 16
    assert L.run() == [1] * n


@pytest.mark.parametrize("n", [2, 4, 8])
@pytest.mark.parametrize("size", [1, 1000, 2 * CAPACITY + 3])
def test_list_lengths_take_the_launches_they_need(n, size):
    """Small disjoint items to every rank, some repeating an earlier target:
    one launch per CAPACITY descriptors, the repeats applied in list order."""
    g = group(n)
    L = Lists(g, "i64", "sum", seed=size * 10 + n)
    rng = np.random.default_rng(size + n)
    span = WIN // n
    for r in range(n):
        placed = []
        for k in range(size):
            if placed and k % 5 == 4:
                peer, toff, count = placed[int(rng.integers(0, len(placed)))]
            else:
                peer, toff, count = (r + k) % n, r * span + 64 + 48 * k, int(rng.integers(1, 5))
                placed.append((peer, toff, count))
            L.add(r, peer, toff, count, fetch=k % 3 == 0)
    assert L.run() == [-(-size // CAPACITY)] * n


def test_order_dependent_float_sum_and_replace():
    g = group(2)
    c = g.comms[0]
    w = g.wins[0]
    g.wins[1][:64].zero_()
    vals = torch.tensor([1e8, 1.0, -1e8], dtype=torch.float32, device=DEV)
    tgt = w[:4].view(torch.float32)
    before = _stats(g)
    c.accumulate_many([vals[0:1], vals[1:2], vals[2:3]], [tgt] * 3, [1, 1, 1])
    # REPLACE on overlapping ranges: the last item wins where it covers
    a = torch.full((4,), 1, dtype=torch.int32, device=DEV)
    b = torch.full((2,), 2, dtype=torch.int32, device=DEV)
    d = torch.full((1,), 3, dtype=torch.int32, device=DEV)
    iw = w[16:32].view(torch.int32)
    prev = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    c.accumulate_many([a, b, d], [iw, iw[1:3], iw[2:3]], [1, 1, 1], op="replace", fetches=[None, None, prev])
    torch.cuda.synchronize()
    assert _stats(g)[0] == before[0] + 2
    # (1e8, -1e8, 1 would give 1: 1 is below half an ulp of 1e8)
    assert float(g.wins[1][:4].view(torch.float32)[0]) == 0.0
    assert g.wins[1][16:32].view(torch.int32).tolist() == [1, 2, 3, 1]
    assert int(prev[0]) == 2


@pytest.mark.parametrize("n", [2, 4, 8])
def test_fetching_increments_of_one_counter_are_one_launch_in_list_order(n):
    """Every rank takes 1024 tickets from a counter of its right neighbour in
    one list: one launch each; each rank's tickets ascend in list order and
    all tickets of one counter are 0 .. 1023 (only its owner's left neighbour
    takes them)."""
    g = group(n)
    k = 1024
    for w in g.wins:
        w[:64].zero_()
    one = torch.ones(1, dtype=torch.int64, device=DEV)
    tickets = [torch.full((k,), -1, dtype=torch.int64, device=DEV) for _ in range(n)]
    torch.cuda.synchronize()
    before = _stats(g)

    def issue(c, r, st):
        ctr = g.wins[r][8:16].view(torch.int64)
        c.accumulate_many([one] * k, [ctr] * k, [(r + 1) % n] * k, fetches=list(tickets[r].split(1)), stream=st)

    g.run(issue)
    g.synchronize()
    assert g.check_errors() == [0] * n
    assert [a - b for a, b in zip(_stats(g), before)] == [1] * n
    for r in range(n):
        assert tickets[r].tolist() == list(range(k)), r
        assert int(g.wins[r][8:16].view(torch.int64)[0]) == k


@pytest.mark.parametrize("n", [2, 4, 8])
@pytest.mark.parametrize("dtype", ["i64", "i32", "i16", "u8"])
def test_all_ranks_updating_the_same_counters_end_exact(n, dtype):
    """Every rank sends 600 increments (with and without fetch) over 8
    counters of every rank at once: each counter ends at its exact total and
    the fetched values of one counter are distinct."""
    g = group(n)
    e = itemsize(dtype)
    tdt = {"i64": torch.int64, "i32": torch.int32, "i16": torch.int16, "u8": torch.uint8}[dtype]
    k = 600
    for w in g.wins:
        w[:64].zero_()
    one = torch.ones(1, dtype=tdt, device=DEV)
    fet = [torch.zeros(k, dtype=tdt, device=DEV) for _ in range(n)]
    torch.cuda.synchronize()

    def issue(c, r, st):
        dsts = [g.wins[r][e * (i % 8) : e * (i % 8 + 1)].view(tdt) for i in range(k)]
        peers = [(i // 8 + r) % n for i in range(k)]
        fetches = [fet[r][i : i + 1] if i % 2 else None for i in range(k)]
        c.accumulate_many([one] * k, dsts, peers, fetches=fetches, stream=st)

    g.run(issue)
    g.synchronize()
    assert g.check_errors() == [0] * n
    per = {}
    for r in range(n):
        for i in range(k):
            key = ((i // 8 + r) % n, i % 8)
            per[key] = per.get(key, 0) + 1
    fetched = {}
    for r in range(n):
        f = fet[r].cpu().numpy().astype(np.int64)
        for i in range(1, k, 2):
            fetched.setdefault(((i // 8 + r) % n, i % 8), []).append(int(f[i]))
    for t in range(n):
        got = g.wins[t][: 8 * e].view(tdt).cpu().numpy().astype(np.int64)
        for j in range(8):
            total = per.get((t, j), 0)
            assert got[j] == total % (1 << (8 * e)), (t, j, got[j], total)
            vals = fetched.get((t, j), [])
            if total < (1 << (8 * e - 1)):
                assert len(set(vals)) == len(vals), (t, j)


def test_refusals_raise_before_any_launch():
    g = group(2)
    c = g.comms[0]
    w = g.wins[0]
    w.zero_()
    g.wins[1].zero_()
    src = torch.ones(8, dtype=torch.int64, device=DEV)
    good = w[:64].view(torch.int64)
    torch.cuda.synchronize()
    before = _stats(g)
    with pytest.raises(CommError):  # not in the heap
        c.accumulate_many([src], [torch.zeros(8, dtype=torch.int64, device=DEV)], [1])
    with pytest.raises(CommError):  # byte sizes differ
        c.accumulate_many([src], [good[:7]], [1])
    with pytest.raises(CommError):  # peer outside the group
        c.accumulate_many([src, src], [good, good], [1, 2])
    with pytest.raises(CommError):  # list lengths differ
        c.accumulate_many([src, src], [good], [1])
    with pytest.raises(CommError):  # origin not on the device
        c.accumulate_many([torch.ones(8, dtype=torch.int64)], [good], [1])
    with pytest.raises(CommError):  # no src for sum
        c.accumulate_many([None], [good], [1], fetches=[src])
    with pytest.raises(CommError):  # no_op without fetch
        c.accumulate_many([src], [good], [1], op="no_op")
    with pytest.raises(CommError):  # unsupported pair
        c.accumulate_many([src.view(torch.float64)], [good.view(torch.float64)], [1], op="band")
    with pytest.raises(CommError):
        c.accumulate_many([src], [good], [1], op="maxloc")
    with pytest.raises(CommError):  # misaligned target
        c.accumulate_many([src[:1]], [w[4:12]], [1], dtype="i64")
    with pytest.raises(CommError):  # dtypes differ
        c.accumulate_many([src, src.view(torch.float64)], [good, good.view(torch.float64)], [1, 1])
    with pytest.raises(CommError):
        c.accumulate_many([src], [good], [1], op="nope")
    # the native checks: every item before anything is launched; the last
    # item here is past the end of the heap, below the user heap, misaligned
    # or names a bad peer
    st = torch.cuda.current_stream().cuda_stream
    goff = c.heap_offset(good)
    for off, peer in ((1 << 40, 1), ((1 << 64) - 16, 1), (0, 1), (goff + 4, 1), (goff, 2)):
        n = 3
        rc = c._lib.fb_accumulate_many(
            c._h,
            n,
            (C.c_void_p * n)(*([src.data_ptr()] * n)),
            None,
            (C.c_uint64 * n)(goff, goff + 8, off),
            (C.c_uint64 * n)(1, 1, 1),
            (C.c_int32 * n)(1, 0, peer),
            6,  # FB_I64
            2,  # FB_OP_SUM
            st,
        )
        assert rc == FB_E_INVALID, (off, peer, rc)
    sub = g.subset([0, 1])
    try:
        with pytest.raises(CommError):
            sub.comms[0].accumulate_many([src], [good], [1])
    finally:
        sub.close()
    torch.cuda.synchronize()
    assert _stats(g) == before
    assert g.check_errors() == [0, 0]
    assert int(g.wins[1].count_nonzero()) == 0 and int(w.count_nonzero()) == 0


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_tickets_in_list_order_over_another_gpus_mapping():
    """The chain order across the peer mapping of another GPU: each rank takes
    1024 tickets from a counter on the other GPU in one launch."""
    k = 1024
    g = LocalGroup(2, devices=[0, 1], **CFG)
    try:
        wins = [c.empty(64, torch.int64) for c in g.comms]
        for w in wins:
            w.zero_()
        tickets = [torch.full((k,), -1, dtype=torch.int64, device=f"cuda:{r}") for r in range(2)]
        ones = [torch.ones(1, dtype=torch.int64, device=f"cuda:{r}") for r in range(2)]
        for r in range(2):
            torch.cuda.synchronize(r)
        before = _stats(g)

        def issue(c, r, st):
            c.accumulate_many([ones[r]] * k, [wins[r][:1]] * k, [1 - r] * k, fetches=list(tickets[r].split(1)), stream=st)

        g.run(issue)
        g.synchronize()
        assert g.check_errors() == [0, 0]
        assert [a - b for a, b in zip(_stats(g), before)] == [1, 1]
        for r in range(2):
            assert tickets[r].tolist() == list(range(k)), r
            assert int(wins[r][0]) == k
    finally:
        g.close()
