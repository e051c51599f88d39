"""Grouped reduce-scatter and all-gather (one launch per list) against the
NumPy oracles: reduce-scatter bit for bit against ``reduce_oracle.fold`` for
every (dtype, op) pair ``reduce_oracle.supported`` allows, all-gather byte for
byte against ``move_oracle.all_gather``.

N ranks share one GPU inside this process.  Every case runs on the default
group, where ranks sharing a GPU synchronise in stream order, and on a spin
group whose kernels meet at in-kernel barriers (skipped where the ranks'
kernels are not co-resident).  All tensors of a list sit in one symmetric
buffer per rank with random guard bytes around every output; every send
buffer is checked unchanged, and the communicator's stats must show one
launch per plan launch.
"""

import numpy as np
import pytest
import torch

import move_oracle as mo
import reduce_oracle as ro

pytestmark = pytest.mark.gpu

from faabric_b200.models.resnet50_grads import resnet50_grad_sizes  # noqa: E402
from faabric_b200.parallel import LocalGroup  # noqa: E402
from faabric_b200.parallel.comm import CommError  # noqa: E402

NS = [2, 3, 4, 5, 8]
KINDS = ["stream", "spin"]
GUARD = 32  # random bytes before and after every output
# shard sizes in 16-byte vectors: one vector, a partial chunk, several chunks
SHARD_VECS = [1, 3, 130, 1100]
MAX_SEGS = 1024  # FB_GROUP_MAX_SEGS; a launch takes MAX_SEGS - 8 items

_GROUPS = {}


def group(n, kind):
    if (n, kind) not in _GROUPS:
        cfg = dict(heapBytes=160 << 20, stageBytes=1 << 20, maxBlocks=8, timeoutMs=8000)
        if kind == "spin":
            # in-kernel barriers need every rank's grid resident at once on
            # the shared GPU: 8 ranks x 8 CTAs of 512 threads fit
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
    """Byte offsets of payloads of ``sizes`` bytes in one buffer, each 16-byte
    aligned with GUARD bytes on both sides; and the buffer's length."""
    offs, pos = [], GUARD
    for b in sizes:
        offs.append(pos)
        pos = (pos + b + GUARD + 15) // 16 * 16 + GUARD
    return offs, pos + GUARD


class Bufs:
    """One symmetric byte buffer per rank holding a list's payloads."""

    def __init__(self, g, sizes, rng):
        self.g = g
        self.offs, self.nbytes = _layout(sizes)
        self.sizes = sizes
        self.init = [rng.integers(0, 256, self.nbytes, dtype=np.uint8) for _ in range(g.size)]
        self.t = [c.empty(self.nbytes, torch.uint8) for c in g.comms]
        self.upload()

    def upload(self):
        for t, a in zip(self.t, self.init):
            t.copy_(torch.from_numpy(a))
        torch.cuda.synchronize()

    def set(self, r, i, data):
        data = np.ascontiguousarray(data).view(np.uint8)
        self.init[r][self.offs[i] : self.offs[i] + data.size] = data

    def outside(self, got, r):
        """``got`` with everything but the payloads replaced by the initial
        bytes: equal to ``got`` iff nothing outside the payloads changed."""
        want = self.init[r].copy()
        for o, b in zip(self.offs, self.sizes):
            want[o : o + b] = got[o : o + b]
        return want

    def views(self, r):
        return [self.t[r][o : o + b] for o, b in zip(self.offs, self.sizes)]

    def host(self, r):
        return self.t[r].cpu().numpy()

    def free(self):
        for c, t in zip(self.g.comms, self.t):
            c.free(t)


def _run(g, fn):
    torch.cuda.synchronize()
    before = [c.stats()["launches"] for c in g.comms]
    g.run(fn)
    g.synchronize()
    assert g.check_errors() == [0] * g.size
    return [c.stats()["launches"] - b for c, b in zip(g.comms, before)]


def _inputs(rng, dtype, op, count):
    dt = ro.NP_DTYPES[dtype]
    if dtype in ro.PAIR_DTYPES:
        p = np.zeros(count, dtype=dt)
        p["v"] = rng.integers(-2, 3, count)  # few values: many ties
        p["i"] = rng.integers(-1000, 1000, count)
        return p
    if dtype in ro.FLOAT_DTYPES:
        x = rng.uniform(1.0, 2.0, count) * rng.choice([-1.0, 1.0], count) * np.exp2(rng.integers(-4, 5, count))
        x[rng.random(count) < 0.02] = np.inf
        if dtype == "bf16":
            return ro.f32_to_bf16(x.astype(np.float32))
        return x.astype(dt)
    x = np.frombuffer(rng.bytes(count * dt.itemsize), dtype=dt).copy()
    if op in ("land", "lor", "lxor"):
        x[rng.random(count) < 0.5] = 0
    return x


def _check_reduce_scatter(sends, recvs, ins, dtype, op, n, what):
    """recvs' payloads equal the fold of shard r, guards and sends unchanged."""
    e = ro.itemsize(dtype)
    for r in range(n):
        got = recvs.host(r)
        for i, shard in enumerate(recvs.sizes):
            c = shard // e
            exp = ro.fold([ins[p][i][r * c : (r + 1) * c] for p in range(n)], dtype, op)
            ro.assert_same(mo.payload(got, recvs.offs[i], shard).view(ro.NP_DTYPES[dtype]), exp, dtype, f"{what} rank {r} item {i}")
        assert np.array_equal(got, recvs.outside(got, r)), f"{what}: rank {r} wrote outside its outputs"
        assert np.array_equal(sends.host(r), sends.init[r]), f"{what}: rank {r} send modified"


def _rs_case(g, rng, dtype, op, shard_vecs, channel=0, many=False):
    n = g.size
    e = ro.itemsize(dtype)
    shards = [v * 16 for v in shard_vecs]
    sends = Bufs(g, [s * n for s in shards], rng)
    recvs = Bufs(g, shards, rng)
    ins = [[_inputs(rng, dtype, op, s * n // e) for s in shards] for _ in range(n)]
    for r in range(n):
        for i in range(len(shards)):
            sends.set(r, i, ins[r][i])
    sends.upload()
    if many:
        launches = _run(
            g, lambda c, r, st: c.reduce_scatter_many(sends.views(r), recvs.views(r), op=op, channel=channel, dtype=dtype)
        )
        plans = None
    else:
        plans = [c.prepare_reduce_scatter_group(sends.views(r), recvs.views(r), dtype=dtype) for r, c in enumerate(g.comms)]
        launches = _run(g, lambda c, r, st: c.reduce_scatter_group(plans[r], op=op, channel=channel))
    want = (len(shards) + MAX_SEGS - 9) // (MAX_SEGS - 8)
    assert launches == [want] * n
    if plans:
        assert [p.launches for p in plans] == [want] * n
    _check_reduce_scatter(sends, recvs, ins, dtype, op, n, f"{dtype} {op} n={n}")
    sends.free()
    recvs.free()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", NS)
def test_reduce_scatter_every_supported_pair(n, kind):
    g = group(n, kind)
    rng = np.random.default_rng([n, KINDS.index(kind)])
    for k, (dtype, op) in enumerate(ro.SUPPORTED):
        e = ro.itemsize(dtype)
        assert all(v * 16 % e == 0 for v in SHARD_VECS)
        # plans and transient tables, on channels 0 and 1
        _rs_case(g, rng, dtype, op, SHARD_VECS, channel=k % 2, many=bool(k % 3 == 0))


def _ag_case(g, rng, shard_bytes, channel=0, many=False, in_place=False, steps=1):
    n = g.size
    sends = Bufs(g, shard_bytes, rng)
    recvs = Bufs(g, [s * n for s in shard_bytes], rng)
    if in_place:
        # send i is block `rank` of output i
        for r in range(n):
            for i, s in enumerate(shard_bytes):
                recvs.set(r, i, mo.place(mo.payload(recvs.init[r], recvs.offs[i], s * n), r * s, mo.payload(sends.init[r], sends.offs[i], s)))
        recvs.upload()
        send_views = [[v[r * s : (r + 1) * s] for v, s in zip(recvs.views(r), shard_bytes)] for r in range(n)]
    else:
        send_views = [sends.views(r) for r in range(n)]
    plans = None
    if not many:
        plans = [c.prepare_all_gather_group(send_views[r], recvs.views(r)) for r, c in enumerate(g.comms)]
    for step in range(steps):
        if step > 0:
            # new data into the same buffers, same plan
            for r in range(n):
                sends.init[r] = rng.integers(0, 256, sends.nbytes, dtype=np.uint8)
            sends.upload()
        if many:
            launches = _run(g, lambda c, r, st: c.all_gather_many(send_views[r], recvs.views(r), channel=channel))
        else:
            launches = _run(g, lambda c, r, st: c.all_gather_group(plans[r], channel=channel))
        want = (len(shard_bytes) + MAX_SEGS - 9) // (MAX_SEGS - 8)
        assert launches == [want] * n
        got = [recvs.host(r) for r in range(n)]
        for i, s in enumerate(shard_bytes):
            if in_place:
                src = [mo.payload(sends.init[r], sends.offs[i], s) for r in range(n)]
            else:
                src = [mo.payload(sends.host(r), sends.offs[i], s) for r in range(n)]
            exp = mo.all_gather(src, [0] * n, [np.zeros(s * n, np.uint8)] * n, [0] * n, s)
            for r in range(n):
                assert np.array_equal(
                    mo.payload(got[r], recvs.offs[i], s * n), exp[r]
                ), f"all-gather item {i} ({s} B) rank {r} step {step}"
        for r in range(n):
            assert np.array_equal(got[r], recvs.outside(got[r], r)), f"rank {r} wrote outside its outputs"
            if not in_place:
                assert np.array_equal(sends.host(r), sends.init[r]), f"rank {r} send modified"
    sends.free()
    recvs.free()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", NS)
def test_all_gather_plans_transient_in_place_and_channels(n, kind):
    g = group(n, kind)
    rng = np.random.default_rng([200 + n, KINDS.index(kind)])
    sizes = [v * 16 for v in SHARD_VECS]
    _ag_case(g, rng, sizes, channel=0, steps=3)
    _ag_case(g, rng, sizes, channel=1, many=True)
    _ag_case(g, rng, sizes[::-1], channel=1, in_place=True)
    _ag_case(g, rng, sizes, channel=0, many=True, in_place=True)


def _resnet_shards(n, esize, scale):
    """Per-rank element counts of the 214 ResNet-50 gradients (scaled down by
    ``scale``), each shard padded to a multiple of 16 bytes."""
    per_vec = 16 // esize
    return [max(1, -(-max(1, s // scale) // n)) for s in resnet50_grad_sizes()], per_vec


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", NS)
def test_resnet50_shaped_list_and_two_launch_list(n, kind):
    g = group(n, kind)
    rng = np.random.default_rng([300 + n, KINDS.index(kind)])
    for dtype, scale in (("f32", 16), ("bf16", 16)):
        e = ro.itemsize(dtype)
        counts, per_vec = _resnet_shards(n, e, scale)
        vecs = [-(-c // per_vec) for c in counts]
        assert len(vecs) == 214
        _rs_case(g, rng, dtype, "sum", vecs)
        _ag_case(g, rng, [v * 16 for v in vecs], channel=1)
    # a list longer than one segment table: two launches per call
    long_vecs = [1 + i % 3 for i in range(MAX_SEGS + 100)]
    _rs_case(g, rng, "i32", "sum", long_vecs, many=True)
    _ag_case(g, rng, [v * 16 for v in long_vecs])


def test_python_shape_checks_raise_before_any_native_call():
    g = group(2, "stream")
    c = g.comms[0]
    a = c.empty(64, torch.float32)
    b = c.empty(16, torch.float32)
    with pytest.raises(CommError):
        c.prepare_reduce_scatter_group([a], [a[:20]])
    with pytest.raises(CommError):
        c.prepare_all_gather_group([b], [a[:40]])
    with pytest.raises(CommError):
        c.reduce_scatter_many([a], [b, b])
    with pytest.raises(CommError):
        c.all_gather_many([], [])
    # the native checks: an output over its own input cannot be grouped
    with pytest.raises(CommError):
        c.prepare_reduce_scatter_group([a[:32]], [a[:16]])
    c.free(a)
    c.free(b)
