"""Grouped all-to-all (one launch per list of up to 1016 tensors) against
``move_oracle.all_to_all``, byte for byte.

N ranks share one GPU inside this process.  Every case runs on the default
group, where ranks sharing a GPU synchronise in stream order, and on a spin
group whose kernels meet at in-kernel barriers (skipped where the ranks'
kernels are not co-resident).  All sends and recvs of a list sit in one
symmetric buffer per rank with random guard bytes around every buffer; every
byte outside the recv payloads must come back unchanged, and the
communicator's stats must show one launch per plan launch.
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
# bytes per block: one vector, zero, a few vectors, ragged chunk ends (the
# chunk is 64 vectors at 8 ranks, 128 otherwise) and many whole chunks
BLOCKS = [16, 0, 48, 129 * 16, 4096 * 16, 1000 * 16, 65 * 16]
DTYPES = [torch.uint8, torch.float32, torch.bfloat16, torch.int64]

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


class Bufs:
    """One symmetric byte buffer per rank holding a list's sends and recvs
    (n blocks each, send i then recv i, a guard before each), every byte
    random and different on every rank."""

    def __init__(self, g, blocks, rng, shift=0):
        self.g = g
        self.blocks = blocks
        n = g.size
        self.send_offs, self.recv_offs, pos = [], [], GUARD + shift
        for b in blocks:
            self.send_offs.append(pos)
            pos = (pos + b * n + 15) // 16 * 16 + GUARD + shift
            self.recv_offs.append(pos)
            pos = (pos + b * n + 15) // 16 * 16 + GUARD + shift
        self.nbytes = pos + GUARD
        self.init = [rng.integers(0, 256, self.nbytes, dtype=np.uint8) for _ in range(n)]
        self.t = [c.empty(self.nbytes, torch.uint8) for c in g.comms]
        for t, a in zip(self.t, self.init):
            t.copy_(torch.from_numpy(a))
        torch.cuda.synchronize()

    def views(self, r, offs, dtype):
        return [self.t[r][o : o + b * self.g.size].view(dtype) for o, b in zip(offs, self.blocks)]

    def sends(self, r, dtype=torch.uint8):
        return self.views(r, self.send_offs, dtype)

    def recvs(self, r, dtype=torch.uint8):
        return self.views(r, self.recv_offs, dtype)

    def free(self):
        for c, t in zip(self.g.comms, self.t):
            c.free(t)

    def check(self, what):
        """Every rank's buffer equals the oracle's: each recv the exchange of
        the sends, every other byte unchanged."""
        n = self.g.size
        want = [b.copy() for b in self.init]
        for so, ro, b in zip(self.send_offs, self.recv_offs, self.blocks):
            if b:
                # (the oracle on each item's extents: it copies whole buffers)
                got = mo.all_to_all([w[so : so + b * n] for w in want], [0] * n, [w[ro : ro + b * n] for w in want], [0] * n, b)
                for w, g in zip(want, got):
                    w[ro : ro + b * n] = g
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


def _case(g, rng, blocks, many, dtype=torch.uint8, shift=0, channel=0):
    n = g.size
    b = Bufs(g, blocks, rng, shift)
    want = (len(blocks) + MAX_ITEMS - 1) // MAX_ITEMS
    if many:
        launches = _run(g, lambda c, r, st: c.all_to_all_many(b.sends(r, dtype), b.recvs(r, dtype), channel=channel))
    else:
        plans = [c.prepare_all_to_all_group(b.sends(r, dtype), b.recvs(r, dtype)) for r, c in enumerate(g.comms)]
        assert [p.launches for p in plans] == [want] * n
        launches = _run(g, lambda c, r, st: c.all_to_all_group(plans[r], channel=channel))
        for p in plans:
            p.close()
    b.check(f"n={n} items={len(blocks)} many={many} dtype={dtype}")
    b.free()
    return launches, want


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", NS)
def test_every_block_length_and_dtype(n, kind):
    g = group(n, kind)
    rng = np.random.default_rng([n, KINDS.index(kind)])
    for i, dtype in enumerate(DTYPES):
        for many in (False, True):
            launches, want = _case(g, rng, BLOCKS, many, dtype, channel=i % 2)
            assert launches == [want] * n
    # each block length alone
    for blk in BLOCKS[:4]:
        launches, _ = _case(g, rng, [blk], True)
        assert launches == [1] * n


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", NS)
def test_resnet50_list_and_launch_boundaries(n, kind):
    g = group(n, kind)
    rng = np.random.default_rng([100 + n, KINDS.index(kind)])
    # the 214 ResNet-50 tensors, f32 bytes scaled down 16x, each padded to a
    # multiple of 16 * n bytes: blocks of one vector up to thousands
    blocks = [(s * 4 // 16 + 16 * n - 1) // (16 * n) * 16 for s in resnet50_grad_sizes()]
    assert len(blocks) == 214
    launches, _ = _case(g, rng, blocks, False, torch.float32)
    assert launches == [1] * n
    for count, want in ((1, 1), (MAX_ITEMS, 1), (MAX_ITEMS + 1, 2)):
        launches, _ = _case(g, rng, [16 * (1 + i % 3) for i in range(count)], True)
        assert launches == [want] * n


@pytest.mark.parametrize("n", [2, 5])
def test_unaligned_list_falls_back_to_per_item_all_to_all(n):
    g = group(n, "stream")
    rng = np.random.default_rng([200 + n])
    launches, _ = _case(g, rng, [32, 64, 16], True, torch.float32, shift=4)
    # one all_to_all call per item, each at least one launch
    assert all(x >= 3 for x in launches)


def test_refusals():
    g = group(3, "stream")
    c = g.comms[0]
    a = c.empty(96, torch.float32)
    b = c.empty(96, torch.float32)
    before = c.stats()["launches"]
    with pytest.raises(CommError):
        c.all_to_all_many([a], [b[:93]])  # unequal numel
    with pytest.raises(CommError):
        c.all_to_all_many([a[:94]], [b[:94]])  # not divisible by size
    with pytest.raises(CommError):
        c.all_to_all_many([a[:48]], [b.view(torch.uint8)[:48]])  # equal numel, 4x fewer recv bytes
    with pytest.raises(CommError):
        c.prepare_all_to_all_group([a[:48]], [b.view(torch.int16)[:48]])
    with pytest.raises(CommError):
        c.prepare_all_to_all_group([a], [b[:90]])
    with pytest.raises(CommError):
        c.all_to_all_many([], [])
    with pytest.raises(CommError):
        c.all_to_all_many([a[:48], a[48:]], [b[:48]])
    with pytest.raises(CommError):
        c.prepare_all_to_all_group([a[1:13]], [b[:12]])  # not 16-byte aligned
    with pytest.raises(CommError):
        c.prepare_all_to_all_group([a[:48]], [a[24:72]])  # recv overlaps send
    plan = c.prepare_all_to_all_group([a[:48]], [b[:48]])
    with pytest.raises(CommError):
        c.all_gather_group(plan)  # a plan of another kind
    other = c.prepare_all_gather_group([a[:4]], [b[:12]])
    with pytest.raises(CommError):
        c.all_to_all_group(other)
    assert c.stats()["launches"] == before
    plan.close()
    other.close()
    c.free(a)
    c.free(b)
