"""Grouped broadcast (one launch per list of up to 1016 tensors) against
``move_oracle.broadcast``, byte for byte.

N ranks share one GPU inside this process.  Every case runs on the default
group, where ranks sharing a GPU synchronise in stream order, and on a spin
group whose kernels meet at in-kernel barriers (skipped where the ranks'
kernels are not co-resident).  All tensors of a list sit in one symmetric
buffer per rank with random guard bytes around every payload; the root's
buffer must come back unchanged, and the communicator's stats must show one
launch per plan launch.
"""

import numpy as np
import pytest
import torch

import move_oracle as mo

pytestmark = pytest.mark.gpu

from faabric_b200.models.resnet50_grads import resnet50_grad_sizes  # noqa: E402
from faabric_b200.parallel import LocalGroup  # noqa: E402
from faabric_b200.parallel.comm import CommError  # noqa: E402

NS = [2, 3, 4, 5, 8]
KINDS = ["stream", "spin"]
GUARD = 32
MAX_ITEMS = 1016  # FB_GROUP_MAX_SEGS - 8 items per launch
# 1 byte, 15 bytes, one vector + tail, several chunks (+ tail)
LENGTHS = [1, 15, 17, 16, 4096 * 16 + 3, 1000, 130 * 16]

_GROUPS = {}


def group(n, kind):
    if (n, kind) not in _GROUPS:
        cfg = dict(heapBytes=160 << 20, stageBytes=1 << 20, maxBlocks=8, timeoutMs=8000)
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


def _layout(sizes):
    offs, pos = [], GUARD
    for b in sizes:
        offs.append(pos)
        pos = (pos + b + GUARD + 15) // 16 * 16 + GUARD
    return offs, pos + GUARD


class Bufs:
    """One symmetric byte buffer per rank holding a list's payloads, every
    byte random (payloads and guards differ on every rank)."""

    def __init__(self, g, sizes, rng, shift=0):
        self.g = g
        self.offs, self.nbytes = _layout(sizes)
        self.offs = [o + shift for o in self.offs]
        self.nbytes += shift
        self.sizes = sizes
        self.init = [rng.integers(0, 256, self.nbytes, dtype=np.uint8) for _ in range(g.size)]
        self.t = [c.empty(self.nbytes, torch.uint8) for c in g.comms]
        for t, a in zip(self.t, self.init):
            t.copy_(torch.from_numpy(a))
        torch.cuda.synchronize()

    def views(self, r):
        return [self.t[r][o : o + b] for o, b in zip(self.offs, self.sizes)]

    def free(self):
        for c, t in zip(self.g.comms, self.t):
            c.free(t)

    def check(self, root, what):
        """Every rank's buffer equals the oracle's: each payload the root's,
        every guard byte (and the root's whole buffer) unchanged."""
        want = [b.copy() for b in self.init]
        for o, s in zip(self.offs, self.sizes):
            want = mo.broadcast(want, [o] * len(want), s, root)
        for r in range(self.g.size):
            got = self.t[r].cpu().numpy()
            assert np.array_equal(got, want[r]), f"{what}: rank {r} first difference {mo.first_difference(got, want[r])}"
        assert np.array_equal(self.t[root].cpu().numpy(), self.init[root]), f"{what}: root modified"


def _run(g, fn):
    torch.cuda.synchronize()
    before = [c.stats()["launches"] for c in g.comms]
    g.run(fn)
    g.synchronize()
    assert g.check_errors() == [0] * g.size
    return [c.stats()["launches"] - b for c, b in zip(g.comms, before)]


def _case(g, rng, sizes, root, many, shift=0, channel=0):
    n = g.size
    b = Bufs(g, sizes, rng, shift)
    want = (len(sizes) + MAX_ITEMS - 1) // MAX_ITEMS
    if many:
        launches = _run(g, lambda c, r, st: c.broadcast_many(b.views(r), root=root, channel=channel))
    else:
        plans = [c.prepare_broadcast_group(b.views(r)) for r, c in enumerate(g.comms)]
        assert [p.launches for p in plans] == [want] * n
        launches = _run(g, lambda c, r, st: c.broadcast_group(plans[r], root=root, channel=channel))
    b.check(root, f"n={n} root={root} items={len(sizes)} many={many}")
    b.free()
    return launches, want


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", NS)
def test_every_root_every_length(n, kind):
    g = group(n, kind)
    rng = np.random.default_rng([n, KINDS.index(kind)])
    for root in range(n):
        for many in (False, True):
            launches, want = _case(g, rng, LENGTHS, root, many, channel=root % 2)
            assert launches == [want] * n
        # each length alone
        for s in LENGTHS[:4]:
            launches, _ = _case(g, rng, [s], root, True)
            assert launches == [1] * n


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", NS)
def test_resnet50_list_and_launch_boundaries(n, kind):
    g = group(n, kind)
    rng = np.random.default_rng([100 + n, KINDS.index(kind)])
    # the 214 ResNet-50 tensors, f32 bytes scaled down 16x (lengths stay
    # arbitrary: not all multiples of 16)
    sizes = [max(1, s // 16) * 4 + (i % 3) for i, s in enumerate(resnet50_grad_sizes())]
    assert len(sizes) == 214
    launches, _ = _case(g, rng, sizes, n - 1, False)
    assert launches == [1] * n
    for count, want in ((1, 1), (MAX_ITEMS, 1), (MAX_ITEMS + 1, 2)):
        launches, _ = _case(g, rng, [1 + i % 40 for i in range(count)], count % n, True)
        assert launches == [want] * n


@pytest.mark.parametrize("n", [2, 5])
def test_unaligned_list_falls_back_to_per_item_broadcast(n):
    g = group(n, "stream")
    rng = np.random.default_rng([200 + n])
    launches, _ = _case(g, rng, [33, 70, 5], 1, True, shift=3)
    # one broadcast call per item, each at least one launch
    assert all(x >= 3 for x in launches)


def test_refusals():
    g = group(3, "stream")
    c = g.comms[0]
    a = c.empty(64, torch.uint8)
    before = c.stats()["launches"]
    with pytest.raises(CommError):
        c.broadcast_many([a], root=3)
    with pytest.raises(CommError):
        c.broadcast_many([], root=0)
    with pytest.raises(CommError):
        c.prepare_broadcast_group([a[1:17]])  # not 16-byte aligned
    plan = c.prepare_broadcast_group([a])
    with pytest.raises(CommError):
        c.broadcast_group(plan, root=-1)
    with pytest.raises(CommError):
        c.all_reduce_group(plan)  # a plan of another kind
    other = c.prepare_group([a[:16].view(torch.float32)])
    with pytest.raises(CommError):
        c.broadcast_group(other, root=0)
    assert c.stats()["launches"] == before
    plan.close()
    other.close()
    c.free(a)
