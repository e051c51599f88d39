"""The grouped kinds (all-reduce, reduce-scatter, all-gather, broadcast) on
``LocalGroup.subset`` children, 8 ranks on one GPU: parity splits of 4 and 8,
a reversed-order child, two disjoint children back to back, and a child and
its parent alternating, each bit-exact against ``reduce_oracle.fold`` /
``move_oracle``; and 40 rounds of slot reuse with grouped launches between
them.  One launch per list on the child; the parent's count does not move."""

import numpy as np
import pytest
import torch

import move_oracle as mo
import reduce_oracle as ro

pytestmark = pytest.mark.gpu

from faabric_b200.parallel import LocalGroup  # noqa: E402

KINDS = ["stream", "spin"]
SIZES = [16 * 3, 16 * 130 + 16, 16 * 1100]  # bytes per tensor (per shard for the shard kinds)
_GROUPS = {}


def group(kind):
    if kind not in _GROUPS:
        cfg = dict(heapBytes=96 << 20, stageBytes=1 << 20, maxBlocks=8, timeoutMs=8000)
        if kind == "spin":
            cfg.update(maxBlocks=4, groupBlocks=8, timeoutMs=4000, streamSync=0)
        g = LocalGroup(8, **cfg)
        if kind == "spin" and g.shares_devices and not g.coresident():
            g.close()
            g = None
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


def _launches(comms):
    return [c.stats()["launches"] for c in comms]


def _lists(g, rng, members, nbytes_each):
    """Per parent rank: a list of int32 heap tensors (allocated on every
    parent rank: allocation is collective) with random contents."""
    out = []
    for c in g.comms:
        out.append([c.empty(b // 4, torch.int32) for b in nbytes_each])
    host = [[rng.integers(-(2**31), 2**31, b // 4, dtype=np.int64).astype(np.int32) for b in nbytes_each] for _ in g.comms]
    for r in range(g.size):
        for t, h in zip(out[r], host[r]):
            t.copy_(torch.from_numpy(h))
    torch.cuda.synchronize()
    return out, host


def _free(g, lists):
    for c, ts in zip(g.comms, lists):
        for t in ts:
            c.free(t)


def _all_kinds_on(g, sub, rng, root):
    """Runs one list of each grouped kind on ``sub`` and checks it."""
    members = sub.members
    m = len(members)
    parent_before = _launches(g.comms)
    # all-reduce, in place
    ar, ar_in = _lists(g, rng, members, SIZES)
    before = _launches(sub.comms)
    sub.run(lambda c, i, st: c.all_reduce_many([ar[members[i]][k] for k in range(len(SIZES))], op="sum"))
    sub.synchronize()
    assert sub.check_errors() == [0] * m
    assert [a - b for a, b in zip(_launches(sub.comms), before)] == [1] * m
    for k in range(len(SIZES)):
        want = ro.fold([ar_in[p][k] for p in members], "i32", "sum")
        for p in members:
            ro.assert_same(ar[p][k].cpu().numpy(), want, "i32", f"all-reduce {members} item {k} rank {p}")
    _free(g, ar)
    # reduce-scatter: send m shards, recv one
    rs_send, rs_in = _lists(g, rng, members, [s * m for s in SIZES])
    rs_recv, _ = _lists(g, rng, members, SIZES)
    sub.run(
        lambda c, i, st: c.reduce_scatter_many(
            [rs_send[members[i]][k] for k in range(len(SIZES))], [rs_recv[members[i]][k] for k in range(len(SIZES))]
        )
    )
    sub.synchronize()
    assert sub.check_errors() == [0] * m
    for k, s in enumerate(SIZES):
        c = s // 4
        for i, p in enumerate(members):
            want = ro.fold([rs_in[q][k][i * c : (i + 1) * c] for q in members], "i32", "sum")
            ro.assert_same(rs_recv[p][k].cpu().numpy(), want, "i32", f"reduce-scatter {members} item {k} rank {p}")
            assert np.array_equal(rs_send[p][k].cpu().numpy(), rs_in[p][k]), "send modified"
    _free(g, rs_send)
    _free(g, rs_recv)
    # all-gather
    ag_send, ag_in = _lists(g, rng, members, SIZES)
    ag_recv, _ = _lists(g, rng, members, [s * m for s in SIZES])
    sub.run(
        lambda c, i, st: c.all_gather_many(
            [ag_send[members[i]][k] for k in range(len(SIZES))], [ag_recv[members[i]][k] for k in range(len(SIZES))]
        )
    )
    sub.synchronize()
    assert sub.check_errors() == [0] * m
    for k, s in enumerate(SIZES):
        srcs = [ag_in[p][k].view(np.uint8) for p in members]
        exp = mo.all_gather(srcs, [0] * m, [np.zeros(s * m, np.uint8)] * m, [0] * m, s)
        for i, p in enumerate(members):
            assert np.array_equal(ag_recv[p][k].cpu().numpy().view(np.uint8), exp[i]), f"all-gather {members} item {k}"
    _free(g, ag_send)
    _free(g, ag_recv)
    # broadcast from child rank `root`, with a plan
    bc, bc_in = _lists(g, rng, members, SIZES)
    plans = [sub.comms[i].prepare_broadcast_group([t.view(torch.uint8)[:-3] for t in bc[p]]) for i, p in enumerate(members)]
    sub.run(lambda c, i, st: c.broadcast_group(plans[i], root=root))
    sub.synchronize()
    assert sub.check_errors() == [0] * m
    for k, s in enumerate(SIZES):
        bufs = [bc_in[p][k].view(np.uint8) for p in members]
        exp = mo.broadcast(bufs, [0] * m, s - 3, root)
        for i, p in enumerate(members):
            assert np.array_equal(bc[p][k].cpu().numpy().view(np.uint8), exp[i]), f"broadcast {members} item {k} rank {p}"
    for pl in plans:
        pl.close()
    _free(g, bc)
    assert _launches(g.comms) == parent_before


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("members", [[0, 2, 4, 6], [1, 3, 5, 7], [7, 6, 5, 4, 3, 2, 1, 0], [5, 2, 7, 0], [3, 6]],
                         ids=lambda m: "-".join(map(str, m)))
def test_grouped_kinds_on_a_child(kind, members):
    g = group(kind)
    rng = np.random.default_rng([len(members), members[0], KINDS.index(kind)])
    sub = g.subset(members)
    try:
        for root in (0, len(members) - 1):
            _all_kinds_on(g, sub, rng, root)
    finally:
        sub.close()
    assert all(c.free_subset_slots() == (1 << 15) - 1 for c in g.comms)


@pytest.mark.parametrize("kind", KINDS)
def test_disjoint_children_back_to_back_and_parent_alternating(kind):
    g = group(kind)
    rng = np.random.default_rng([77, KINDS.index(kind)])
    lo, hi = g.subset([0, 1, 2, 3]), g.subset([7, 6, 5, 4])
    try:
        for rnd in range(2):
            _all_kinds_on(g, lo, rng, rnd % 4)
            _all_kinds_on(g, hi, rng, (rnd + 1) % 4)
            # the parent: a grouped all-reduce over all 8
            ts, ins = _lists(g, rng, list(range(8)), [16 * 50])
            g.run(lambda c, r, st: c.all_reduce_many(ts[r]))
            g.synchronize()
            assert g.check_errors() == [0] * 8
            want = ro.fold([ins[p][0] for p in range(8)], "i32", "sum")
            for r in range(8):
                ro.assert_same(ts[r][0].cpu().numpy(), want, "i32", f"parent round {rnd}")
            _free(g, ts)
    finally:
        lo.close()
        hi.close()


@pytest.mark.parametrize("kind", KINDS)
def test_slot_reuse_40_rounds(kind):
    g = group(kind)
    rng = np.random.default_rng([99, KINDS.index(kind)])
    ts, ins = _lists(g, rng, list(range(8)), [16 * 8 + 4, 1000])
    for rnd in range(40):
        members = [0, 2, 4, 6] if rnd % 2 == 0 else [7, 5, 3, 1]
        sub = g.subset(members)
        root = rnd % 4
        try:
            before = _launches(sub.comms)
            sub.run(lambda c, i, st: c.broadcast_many([t.view(torch.uint8) for t in ts[members[i]]], root=root))
            sub.run(lambda c, i, st: c.all_reduce_many(ts[members[i]]))
            sub.synchronize()
            assert sub.check_errors() == [0] * 4
            assert [a - b for a, b in zip(_launches(sub.comms), before)] == [2] * 4
        finally:
            sub.close()
        # expected: every member holds 4 x the root's values
        for k in range(2):
            want = ro.fold([ins[members[root]][k]] * 4, "i32", "sum")
            for p in members:
                ro.assert_same(ts[p][k].cpu().numpy(), want, "i32", f"round {rnd} item {k}")
                ins[p][k] = want.copy()
        # a grouped launch on the parent between the rounds
        g.run(lambda c, r, st: c.broadcast_many([t.view(torch.uint8) for t in ts[r]], root=rnd % 8))
        g.synchronize()
        assert g.check_errors() == [0] * 8
        for p in range(8):
            for k in range(2):
                ins[p][k] = ins[rnd % 8][k].copy()
    _free(g, ts)
    assert all(c.free_subset_slots() == (1 << 15) - 1 for c in g.comms)
