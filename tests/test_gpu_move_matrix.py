"""Data-movement collectives and point-to-point calls, byte for byte against
tests/move_oracle.py.

N ranks share one GPU inside this process.  Two wirings run every case: the
default group, where ranks sharing a GPU synchronise in stream order, and a
spin group whose kernels synchronise inside the kernel with per-CTA flag
barriers, as ranks on distinct GPUs do (skipped where the ranks' kernels are
not co-resident).  Payloads are random bytes: movement ignores dtypes, and
random bytes show every misplaced or reordered word.  Every destination has
random guard bytes on both sides, and every source is checked unchanged.

* sources in the symmetric heap at offsets of 0, 1, 4 and 8 bytes (the same
  on every rank), or in local memory (staged through the heap);
* destinations in local memory at a different alignment on every rank
  (0, 4, 1, 12, 8 bytes past a 16-byte boundary);
* sizes around the copy widths (1, 3, 15, 16, 17, 4095, 4100 bytes), one TMA
  tile + 16 and the TMA threshold +- 16, and small sizes with the TMA
  threshold lowered to 16 bytes (partial tiles, CTAs without a tile);
* the two-step broadcast with empty and uneven slices, staged calls of many
  pieces whose length is not a multiple of 32 bytes, and point-to-point at
  every local alignment around the bounce-slot size.
"""

import zlib

import numpy as np
import pytest
import torch

import move_oracle as mo

pytestmark = pytest.mark.gpu

from faabric_b200.parallel import LocalGroup  # noqa: E402

NS = [2, 3, 4, 5, 8]
SYM_OFFSETS = [0, 1, 4, 8]
DST_MISALIGN = [0, 4, 1, 12, 8]  # rank r's destination: DST_MISALIGN[r % 5]
LEAD = 16  # guard bytes before the 16-byte boundary a payload is offset from
TAIL = 32  # guard bytes after a payload
TILE = 32 << 10  # bytes per TMA tile
TMA_MIN = 256 << 10  # CommConfig::tmaMinBytes
BCAST_2STEP_MIN = 1 << 20  # CommConfig::bcast2StepMinBytes
BOUNCE = 256 << 10  # p2p ring per peer: messages split into BOUNCE / 2 chunks
# (bytes per rank or rank pair, tmaMinBytes)
SIZES = [(b, TMA_MIN) for b in (1, 3, 15, 16, 17, 4095, 4096 + 4, TILE + 16, TMA_MIN - 16, TMA_MIN + 16)] + [
    (b, 16) for b in (16, 48, 4096, TILE + 16)
]
MAX_PER = max(b for b, _ in SIZES)

_GROUPS = {}


def group(n, kind):
    """One group per (n, kind), kept for the module.  ``stream``: default
    wiring; ``spin``: in-kernel barriers (``None`` when not co-resident);
    ``-64k`` suffix: 64 KiB staging area, so staged calls take many pieces."""
    if (n, kind) not in _GROUPS:
        cfg = dict(heapBytes=64 << 20, stageBytes=8 << 20, maxBlocks=8, timeoutMs=8000, p2pBounceBytes=BOUNCE)
        if kind.endswith("-64k"):
            cfg["stageBytes"] = 64 << 10
        if kind.startswith("spin"):
            cfg.update(maxBlocks=4, timeoutMs=4000, streamSync=0)
        g = LocalGroup(n, **cfg)
        if kind.startswith("spin") and g.shares_devices and not g.coresident():
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


def rng_for(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


def configure(g, **kw):
    for c in g.comms:
        c.configure(**kw)


class Arenas:
    """Per-rank byte arenas a case reuses: sources in the heap and in local
    memory, destinations in local memory.  The heap arena is allocated
    collectively, so it sits at one offset on every rank."""

    def __init__(self, g, src_bytes, dst_bytes):
        self.g = g
        pad = LEAD + 16 + TAIL
        self.heap = [c.empty(src_bytes + pad, torch.uint8) for c in g.comms]
        self.local = [torch.empty(src_bytes + pad, dtype=torch.uint8, device=f"cuda:{c.device}") for c in g.comms]
        self.dst = [torch.empty(dst_bytes + pad, dtype=torch.uint8, device=f"cuda:{c.device}") for c in g.comms]

    def close(self):
        for c, t in zip(self.g.comms, self.heap):
            c.free(t)


class Regions:
    """A payload at ``LEAD + misalign`` of each rank's arena, with the guard
    bytes around it filled with random bytes."""

    def __init__(self, arenas, nbytes, misaligns, rng):
        self.views, self.regions, self.initial, self.offs = [], [], [], []
        for arena, m in zip(arenas, misaligns):
            off = LEAD + m
            region = arena[: off + nbytes + TAIL]
            data = rng.integers(0, 256, region.numel(), dtype=np.uint8)
            region.copy_(torch.from_numpy(data))
            self.views.append(arena[off : off + nbytes])
            self.regions.append(region)
            self.initial.append(data)
            self.offs.append(off)

    def now(self):
        return [r.cpu().numpy() for r in self.regions]


def assert_bytes(got, want, what):
    for r, (a, b) in enumerate(zip(got, want)):
        if b is None:
            continue
        i = mo.first_difference(a, b)
        assert i is None, f"{what}: rank {r} differs at byte {i} of its region (got {a[i] if i < a.size else None}, want {b[i] if i < b.size else None})"


def run_collective(g, arenas, kind, per, symmetric, sym_off, root, rng, what):
    n = g.size
    src_rows = n if kind in ("scatter", "all_to_all") else 1
    dst_bytes = per if kind in ("scatter", "broadcast") else per * n
    dst_mis = [DST_MISALIGN[r % 5] for r in range(n)]
    if kind == "broadcast":
        # in place: a symmetric buffer sits at one heap offset on every rank
        bufs = Regions(arenas.heap, per, [sym_off] * n, rng) if symmetric else Regions(arenas.dst, per, dst_mis, rng)
        srcs, dsts = None, bufs
    else:
        srcs = Regions(arenas.heap if symmetric else arenas.local, per * src_rows, [sym_off] * n, rng)
        dsts = Regions(arenas.dst, dst_bytes, dst_mis, rng)

    def issue(c, r, st):
        if kind == "all_gather":
            c.all_gather(srcs.views[r], dsts.views[r])
        elif kind == "gather":
            c.gather(srcs.views[r], dsts.views[r], root=root)
        elif kind == "scatter":
            c.scatter(srcs.views[r], dsts.views[r], root=root)
        elif kind == "all_to_all":
            c.all_to_all(srcs.views[r], dsts.views[r])
        else:
            c.broadcast(dsts.views[r], root=root)

    g.run(issue)
    g.synchronize()
    assert g.check_errors() == [0] * n, what
    if srcs is None:
        want = mo.broadcast(dsts.initial, dsts.offs, per, root)
    else:
        want = mo.collective(kind, srcs.initial, srcs.offs, dsts.initial, dsts.offs, per, root)
        assert_bytes(srcs.now(), mo.untouched(srcs.initial), what + " (source)")
    assert_bytes(dsts.now(), want, what)


def roots_for(kind, n, per, i):
    """Every root for small messages, one root (cycling) for large ones."""
    if kind not in mo.ROOTED:
        return [0]
    return range(n) if per < TILE else [i % n]


@pytest.mark.parametrize("symmetric", [True, False], ids=["symmetric", "staged"])
@pytest.mark.parametrize("wiring", ["stream", "spin"])
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("kind", mo.COLLECTIVES)
def test_collective_matrix(kind, n, wiring, symmetric):
    g = group(n, wiring)
    src_rows = n if kind in ("scatter", "all_to_all") else 1
    arenas = Arenas(g, MAX_PER * src_rows, MAX_PER * n)
    for c in g.comms:
        c.stats(reset=True)
    try:
        i = 0
        for per, tma in SIZES:
            configure(g, tmaMinBytes=tma)
            for sym_off in SYM_OFFSETS:
                for root in roots_for(kind, n, per, i):
                    what = f"{kind} n={n} {wiring} {'symmetric' if symmetric else 'staged'} offset={sym_off} bytes={per} tmaMinBytes={tma} root={root}"
                    run_collective(g, arenas, kind, per, symmetric, sym_off, root, rng_for(what), what)
                i += 1
    finally:
        configure(g, tmaMinBytes=TMA_MIN)
        arenas.close()
    stats = [c.stats() for c in g.comms]
    # the TMA kernel ran (ranks with 16-byte aligned destinations at offset 0)
    assert sum(s["tma_launches"] for s in stats) > 0, stats
    if not symmetric:
        assert sum(s["staged_copies"] for s in stats) > 0, stats


@pytest.mark.parametrize("wiring", ["stream", "spin"])
@pytest.mark.parametrize("n", [2, 3, 5, 8])
def test_staged_calls_of_many_pieces(n, wiring):
    """64 KiB of staging: a call runs in pieces of 65536 / rows bytes rounded
    down to 16 (21840 at three ranks: not a multiple of 32), plus a tail."""
    g = group(n, wiring + "-64k")
    sizes = (65536 + 4, 100003, 131072 + 48)
    arenas = Arenas(g, max(sizes) * n, max(sizes) * n)
    for c in g.comms:
        c.stats(reset=True)
    calls = 0
    try:
        for i, per in enumerate(sizes):
            for kind in mo.COLLECTIVES:
                root = (i + n - 1) % n
                what = f"{kind} n={n} {wiring} 64 KiB staging bytes={per} root={root}"
                run_collective(g, arenas, kind, per, False, DST_MISALIGN[i], root, rng_for(what), what)
                calls += 1
    finally:
        arenas.close()
    stats = [c.stats() for c in g.comms]
    # more staged copies than calls: the calls were split into pieces
    assert max(s["staged_copies"] for s in stats) > calls, stats


@pytest.mark.parametrize("n", [3, 5, 8])
def test_two_step_broadcast_slices(n):
    """Symmetric broadcast through the two-step kernel (in-kernel barrier
    between its steps, so spin group only).  With bcast2StepMinBytes = 16,
    totals of 16 and 48 bytes leave some ranks an empty slice and 1 MiB + 16k
    gives uneven ones; from a heap offset that is not 16-byte aligned the
    call takes the one-step path."""
    g = group(n, "spin")
    totals = [16, 48, 4096 + 16] + [BCAST_2STEP_MIN + 16 * k for k in (1, n, 7)]
    arenas = Arenas(g, max(totals), 16)
    for c in g.comms:
        c.stats(reset=True)
    configure(g, bcast2StepMinBytes=16)
    try:
        for i, total in enumerate(totals):
            for sym_off in (0, 4, 8):
                for root in range(n) if total < TILE else [i % n]:
                    what = f"two-step broadcast n={n} bytes={total} offset={sym_off} root={root}"
                    run_collective(g, arenas, "broadcast", total, True, sym_off, root, rng_for(what), what)
                    algo = g.comms[0].last_algo
                    assert (algo == "twoshot") == (sym_off == 0), f"{what}: {algo}"
    finally:
        configure(g, bcast2StepMinBytes=BCAST_2STEP_MIN)
        arenas.close()
    assert all(c.stats()["algo_twoshot"] > 0 for c in g.comms)


# ---------------------------------------------------------------------------
# point to point
# ---------------------------------------------------------------------------
P2P_OFFSETS = [0, 1, 4, 12]
P2P_SIZES = [0, 1, 15, 16, 17, BOUNCE // 2 - 1, BOUNCE // 2, BOUNCE // 2 + 1]


@pytest.mark.parametrize("n", [2, 3])
def test_send_recv_every_alignment(n):
    """Ring r -> r + 1 with send / recv, then with send_recv; messages of one
    bounce slot + 1 byte split into a full chunk and a 1-byte tail."""
    g = group(n, "stream")
    arenas = Arenas(g, MAX_PER, MAX_PER)
    nxt = lambda r: (r + 1) % n  # noqa: E731
    prv = lambda r: (r - 1) % n  # noqa: E731
    try:
        for nbytes in P2P_SIZES:
            for i, off in enumerate(P2P_OFFSETS):
                what = f"p2p n={n} bytes={nbytes} send offset={off}"
                rng = rng_for(what)
                recv_mis = [P2P_OFFSETS[(i + r + 1) % 4] for r in range(n)]
                for call in ("send/recv", "send_recv"):
                    srcs = Regions(arenas.local, nbytes, [off] * n, rng)
                    dsts = Regions(arenas.dst, nbytes, recv_mis, rng)

                    def issue(c, r, st):
                        if call == "send/recv":
                            c.send(srcs.views[r], nxt(r))
                            c.recv(dsts.views[r], prv(r))
                        else:
                            c.send_recv(srcs.views[r], nxt(r), dsts.views[r], prv(r))

                    g.run(issue)
                    g.synchronize()
                    assert g.check_errors() == [0] * n, what
                    assert_bytes(srcs.now(), mo.untouched(srcs.initial), f"{what} {call} (source)")
                    assert_bytes(dsts.now(), mo.send_recv(srcs.initial, srcs.offs, dsts.initial, dsts.offs, nbytes, prv), f"{what} {call}")
    finally:
        arenas.close()


@pytest.mark.parametrize("n", [2, 3])
def test_put_signal_into_unaligned_symmetric_destinations(n):
    g = group(n, "stream")
    sizes = [1, 15, 16, 17, 4096 + 4, BOUNCE // 2 + 1]
    arenas = Arenas(g, max(sizes), max(sizes))
    prv = lambda r: (r - 1) % n  # noqa: E731
    try:
        for nbytes in sizes:
            for i, off in enumerate(P2P_OFFSETS):
                what = f"put_signal n={n} bytes={nbytes} destination offset={off}"
                rng = rng_for(what)
                srcs = Regions(arenas.local, nbytes, [P2P_OFFSETS[(i + r + 1) % 4] for r in range(n)], rng)
                dsts = Regions(arenas.heap, nbytes, [off] * n, rng)

                def issue(c, r, st):
                    c.put_signal(srcs.views[r], dsts.views[r], peer=(r + 1) % n, signal=2, blocks=3)
                    c.wait_signal(signal=2, count=3)

                g.run(issue)
                g.synchronize()
                assert g.check_errors() == [0] * n, what
                assert_bytes(srcs.now(), mo.untouched(srcs.initial), what + " (source)")
                assert_bytes(dsts.now(), mo.send_recv(srcs.initial, srcs.offs, dsts.initial, dsts.offs, nbytes, prv), what)
    finally:
        arenas.close()
