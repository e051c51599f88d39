"""GPU numerics tests of the peer-memory collectives against plain PyTorch
references.  Runs N ranks inside one process; with a single GPU all ranks share
it (each on its own stream), which exercises the same flag/barrier protocol as
a real multi-GPU run.  Mirrors the reference's collective tests
(tests/test/mpi/test_mpi_world.cpp: "Test collective messaging locally",
"Test reduce", "Test operator reduce", "Test gather and allgather",
"Test scan", "Test all-to-all")."""

import numpy as np
import pytest
import torch
from reduce_oracle import assert_same, fold

pytestmark = pytest.mark.gpu

from faabric_b200.parallel import LocalGroup  # noqa: E402

GROUPS = {}
SPIN_GROUPS = {}


def group(n):
    """Default wiring.  Ranks that share a GPU synchronise with stream memory
    operations (no kernel ever waits for another rank's kernel), ranks on
    distinct GPUs with the in-kernel flag barriers."""
    if n not in GROUPS:
        GROUPS[n] = LocalGroup(
            n,
            heapBytes=96 << 20,
            stageBytes=8 << 20,
            maxBlocks=8,
            timeoutMs=8000,
        )
    return GROUPS[n]


def spin_group(n):
    """In-kernel barriers (the multi-GPU product path: LL slots, two-step
    broadcast, CUDA-graph replay) even when the ranks share one GPU.  That
    needs the ranks' kernels to be co-resident, which is ASSERTED first: the
    test is skipped, not failed, where the device does not overlap them."""
    if n not in SPIN_GROUPS:
        g = LocalGroup(
            n,
            heapBytes=64 << 20,
            stageBytes=4 << 20,
            maxBlocks=4,
            timeoutMs=2000,
            streamSync=0,
        )
        if g.shares_devices and not g.coresident():
            g.close()
            SPIN_GROUPS[n] = None
        else:
            SPIN_GROUPS[n] = g
    if SPIN_GROUPS[n] is None:
        pytest.skip("kernels of different ranks are not co-resident on this GPU")
    return SPIN_GROUPS[n]


@pytest.fixture(scope="module", autouse=True)
def _cleanup():
    yield
    for g in list(GROUPS.values()) + list(SPIN_GROUPS.values()):
        if g is not None:
            g.close()
    GROUPS.clear()
    SPIN_GROUPS.clear()


def make_inputs(n, numel, dtype, dev, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    out = []
    for r in range(n):
        if dtype.is_floating_point:
            t = (torch.rand(numel, generator=g) * 2 - 1).to(dtype)
        elif dtype == torch.bool:
            t = torch.randint(0, 2, (numel,), generator=g).to(dtype)
        else:
            t = torch.randint(-50, 50, (numel,), generator=g).to(dtype)
        out.append(t.to(dev))
    return out


_FB_NAMES = {
    torch.int8: "i8",
    torch.uint8: "u8",
    torch.int16: "i16",
    torch.int32: "i32",
    torch.int64: "i64",
    torch.float32: "f32",
    torch.float64: "f64",
    torch.float16: "f16",
    torch.bfloat16: "bf16",
}


def to_numpy(t):
    t = t.cpu()
    if t.dtype == torch.bfloat16:
        return t.view(torch.int16).numpy().view(np.uint16)
    return t.numpy()


def check(out, inputs, op):
    """`out` must be the rank-order fold of `inputs`, bit for bit (see
    tests/reduce_oracle.py)."""
    name = _FB_NAMES[out.dtype]
    assert_same(to_numpy(out), fold([to_numpy(t) for t in inputs], name, op), name, op)


def no_errors(g):
    assert g.check_errors() == [0] * g.size


@pytest.mark.parametrize("n", [2, 4, 8, 3])
@pytest.mark.parametrize("algo", ["ll", "oneshot", "twoshot"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.int32, torch.bfloat16])
@pytest.mark.parametrize("symmetric", [True, False])
def test_allreduce_sum(n, algo, dtype, symmetric):
    g = group(n)
    for numel in (1, 7, 1000, 4099, 65536 + 5):
        if algo == "ll" and numel * 4 > 65536:
            continue
        ins = make_inputs(n, numel, dtype, f"cuda:{g.devices[0]}", seed=numel)
        sends, recvs = [], []
        for r, c in enumerate(g.comms):
            if symmetric:
                s = c.empty(numel, dtype)
                s.copy_(ins[r].to(s.device))
                o = c.empty(numel, dtype)
            else:
                s = ins[r].to(f"cuda:{c.device}").clone()
                o = torch.empty_like(s)
            sends.append(s)
            recvs.append(o)
        torch.cuda.synchronize()
        g.run(lambda c, r, st: c.all_reduce(sends[r], recvs[r], op="sum", algo=algo))
        g.synchronize()
        no_errors(g)
        for r in range(n):
            check(recvs[r], ins, "sum")
            # inputs must be untouched
            assert torch.equal(sends[r].cpu(), ins[r].cpu())
        # identical bits on every rank
        for r in range(1, n):
            assert torch.equal(recvs[r].cpu().view(torch.uint8), recvs[0].cpu().view(torch.uint8))
        if symmetric:
            for c, s, o in zip(g.comms, sends, recvs):
                c.free(s)
                c.free(o)


@pytest.mark.parametrize("n", [2, 8])
def test_allreduce_inplace_and_auto(n):
    g = group(n)
    for numel in (33, 50000, 600000):
        ins = make_inputs(n, numel, torch.float32, "cuda:0", seed=numel + 1)
        bufs = []
        for r, c in enumerate(g.comms):
            b = c.empty(numel, torch.float32)
            b.copy_(ins[r].to(b.device))
            bufs.append(b)
        torch.cuda.synchronize()
        g.run(lambda c, r, st: c.all_reduce(bufs[r]))
        g.synchronize()
        no_errors(g)
        for r in range(n):
            check(bufs[r], ins, "sum")
        for c, b in zip(g.comms, bufs):
            c.free(b)


def test_unsupported_combo_rejected():
    g = group(2)
    from faabric_b200.parallel import CommError

    t = torch.zeros(8, device="cuda:0")
    with pytest.raises(CommError):
        g.comms[0].all_reduce(t, t.clone(), op="band")


@pytest.mark.parametrize("n", [2, 4, 5])
def test_reduce_scan_reducescatter(n):
    g = group(n)
    dtype = torch.float32
    for numel in (5, 4096, 70001):
        ins = make_inputs(n, numel, dtype, "cuda:0", seed=numel)
        sends = []
        for r, c in enumerate(g.comms):
            s = c.empty(numel, dtype)
            s.copy_(ins[r].to(s.device))
            sends.append(s)
        torch.cuda.synchronize()
        # reduce to root 1
        root = 1
        outs = [torch.full((numel,), -7.0, device=f"cuda:{c.device}") for c in g.comms]
        g.run(lambda c, r, st: c.reduce(sends[r], outs[r], root=root))
        g.synchronize()
        no_errors(g)
        check(outs[root], ins, "sum")
        for r in range(n):
            if r != root:
                assert torch.all(outs[r] == -7.0)
        # scan
        outs = [torch.empty(numel, device=f"cuda:{c.device}") for c in g.comms]
        g.run(lambda c, r, st: c.scan(sends[r], outs[r]))
        g.synchronize()
        no_errors(g)
        for r in range(n):
            check(outs[r], ins[: r + 1], "sum")
        for c, s in zip(g.comms, sends):
            c.free(s)
    # reduce-scatter: per-rank slice must be a multiple of 16 bytes
    per = 1024
    ins = make_inputs(n, per * n, dtype, "cuda:0", seed=3)
    sends = []
    for r, c in enumerate(g.comms):
        s = c.empty(per * n, dtype)
        s.copy_(ins[r].to(s.device))
        sends.append(s)
    outs = [torch.empty(per, device=f"cuda:{c.device}") for c in g.comms]
    torch.cuda.synchronize()
    g.run(lambda c, r, st: c.reduce_scatter(sends[r], outs[r]))
    g.synchronize()
    no_errors(g)
    for r in range(n):
        check(outs[r], [t[r * per : (r + 1) * per] for t in ins], "sum")
    for c, s in zip(g.comms, sends):
        c.free(s)


@pytest.mark.parametrize("n", [2, 4, 8, 3])
@pytest.mark.parametrize("symmetric", [True, False])
def test_move_collectives(n, symmetric):
    g = group(n)
    for numel in (1, 13, 1024, 40001):
        dtype = torch.int32

        def alloc(c, count):
            if symmetric:
                return c.empty(count, dtype)
            return torch.empty(count, dtype=dtype, device=f"cuda:{c.device}")

        # ---- allgather
        sends = [alloc(c, numel) for c in g.comms]
        for r, s in enumerate(sends):
            s.copy_(torch.arange(numel, dtype=dtype) + 1000 * r)
        recvs = [torch.zeros(numel * n, dtype=dtype, device=f"cuda:{c.device}") for c in g.comms]
        torch.cuda.synchronize()
        g.run(lambda c, r, st: c.all_gather(sends[r], recvs[r]))
        g.synchronize()
        no_errors(g)
        ref = torch.cat([torch.arange(numel, dtype=dtype) + 1000 * r for r in range(n)])
        for r in range(n):
            assert torch.equal(recvs[r].cpu(), ref)
        # ---- gather to root n-1
        root = n - 1
        recvs = [torch.zeros(numel * n, dtype=dtype, device=f"cuda:{c.device}") for c in g.comms]
        g.run(lambda c, r, st: c.gather(sends[r], recvs[r], root=root))
        g.synchronize()
        no_errors(g)
        assert torch.equal(recvs[root].cpu(), ref)
        # ---- broadcast from root 0
        bufs = [alloc(c, numel) for c in g.comms]
        for r, b in enumerate(bufs):
            b.fill_(r + 1)
        bufs[0].copy_(torch.arange(numel, dtype=dtype) * 3)
        torch.cuda.synchronize()
        g.run(lambda c, r, st: c.broadcast(bufs[r], root=0))
        g.synchronize()
        no_errors(g)
        for r in range(n):
            assert torch.equal(bufs[r].cpu(), torch.arange(numel, dtype=dtype) * 3)
        # ---- alltoall / scatter
        a2a_send = [alloc(c, numel * n) for c in g.comms]
        for r, s in enumerate(a2a_send):
            s.copy_(torch.arange(numel * n, dtype=dtype) + 100000 * r)
        a2a_recv = [torch.zeros(numel * n, dtype=dtype, device=f"cuda:{c.device}") for c in g.comms]
        torch.cuda.synchronize()
        g.run(lambda c, r, st: c.all_to_all(a2a_send[r], a2a_recv[r]))
        g.synchronize()
        no_errors(g)
        for r in range(n):
            exp = torch.cat(
                [torch.arange(r * numel, (r + 1) * numel, dtype=dtype) + 100000 * p for p in range(n)]
            )
            assert torch.equal(a2a_recv[r].cpu(), exp)
        sc_recv = [torch.zeros(numel, dtype=dtype, device=f"cuda:{c.device}") for c in g.comms]
        g.run(lambda c, r, st: c.scatter(a2a_send[r], sc_recv[r], root=1))
        g.synchronize()
        no_errors(g)
        for r in range(n):
            exp = torch.arange(r * numel, (r + 1) * numel, dtype=dtype) + 100000
            assert torch.equal(sc_recv[r].cpu(), exp)
        if symmetric:
            for c, a, b, d in zip(g.comms, sends, bufs, a2a_send):
                c.free(a)
                c.free(b)
                c.free(d)


def test_large_symmetric_broadcast_two_step():
    n = 4
    g = group(n)
    numel = (3 << 20) // 4 + 4  # > bcast2StepMinBytes, multiple of 16 bytes
    bufs = [c.empty(numel, torch.int32) for c in g.comms]
    for r, b in enumerate(bufs):
        b.fill_(r)
    bufs[2].copy_(torch.arange(numel, dtype=torch.int32))
    torch.cuda.synchronize()
    g.run(lambda c, r, st: c.broadcast(bufs[r], root=2))
    g.synchronize()
    no_errors(g)
    if not g.comms[0].stream_sync:
        assert g.comms[0].last_algo == "twoshot"
    for r in range(n):
        assert torch.equal(bufs[r].cpu(), torch.arange(numel, dtype=torch.int32))
    for c, b in zip(g.comms, bufs):
        c.free(b)


def _ring_payload(g, nbytes):
    srcs = [
        (torch.arange(nbytes, dtype=torch.int64) * (r + 3) % 251).to(torch.uint8).to(f"cuda:{c.device}")
        for r, c in enumerate(g.comms)
    ]
    dsts = [torch.zeros(nbytes, dtype=torch.uint8, device=f"cuda:{c.device}") for c in g.comms]
    return srcs, dsts


@pytest.mark.parametrize("nbytes", [0, 1, 15, 4096, 300001, 3 << 20])
def test_send_recv_ring(nbytes):
    """Ring r -> r+1 with a plain send followed by a recv on the SAME stream:
    sends are eager (payload parked in the sender's heap, descriptor posted), no
    kernel waits for a peer, so the ring cannot deadlock whatever the device
    does with the four ranks' kernels (reference: MpiWorld::send never blocks,
    src/mpi/MpiWorld.cpp:590-649)."""
    n = 4
    g = group(n)
    srcs, dsts = _ring_payload(g, nbytes)
    torch.cuda.synchronize()

    def step(c, r, st):
        c.send(srcs[r], (r + 1) % n)
        c.recv(dsts[r], (r - 1) % n)

    for _ in range(3):  # sequence numbers / slot reuse across messages
        g.run(step)
    g.synchronize()
    no_errors(g)
    for r in range(n):
        assert torch.equal(dsts[r].cpu(), srcs[(r - 1) % n].cpu())


@pytest.mark.parametrize("nbytes", [64, 300001, 20 << 20])
def test_sendrecv_exchange_larger_than_the_bounce_ring(nbytes):
    """MPI_Sendrecv-shaped exchange: chunks of both directions are interleaved,
    so messages far beyond the eager capacity (8 MiB per peer) still flow."""
    n = 4
    g = group(n)
    srcs, dsts = _ring_payload(g, nbytes)
    torch.cuda.synchronize()
    g.run(lambda c, r, st: c.send_recv(srcs[r], (r + 1) % n, dsts[r], (r - 1) % n))
    g.synchronize()
    no_errors(g)
    for r in range(n):
        assert torch.equal(dsts[r].cpu(), srcs[(r - 1) % n].cpu())


def test_send_to_self():
    g = group(2)
    c = g.comms[0]
    src = torch.arange(70000, dtype=torch.int32, device=f"cuda:{c.device}")
    dst = torch.zeros_like(src)
    c.send(src, 0, stream=g.streams[0])
    c.recv(dst, 0, stream=g.streams[0])
    g.synchronize()
    no_errors(g)
    assert torch.equal(src, dst)


def test_recv_without_sender_is_aborted_not_hung():
    """Stream-level waits have no timeout of their own: the bounded host wait
    releases them and reports the failure (SURVEY 5.3 failure detection)."""
    g = LocalGroup(2, heapBytes=1 << 20, stageBytes=1 << 20, maxBlocks=2, timeoutMs=200)
    try:
        dst = torch.zeros(1024, dtype=torch.uint8, device=f"cuda:{g.comms[0].device}")
        g.comms[0].recv(dst, 1, stream=g.streams[0])
        assert g.comms[0].check_error(g.streams[0]) != 0
    finally:
        g.close()


def test_send_recv_fifo_order():
    g = group(2)
    a, b = g.comms
    msgs = [torch.full((1000 + i,), i, dtype=torch.int32, device=f"cuda:{a.device}") for i in range(6)]
    outs = [torch.zeros(1000 + i, dtype=torch.int32, device=f"cuda:{b.device}") for i in range(6)]
    for m in msgs:
        a.send(m, 1, stream=g.streams[0])
    for o in outs:
        b.recv(o, 0, stream=g.streams[1])
    g.synchronize()
    no_errors(g)
    for m, o in zip(msgs, outs):
        assert torch.equal(m.cpu(), o.cpu())


def test_put_signal_and_barrier():
    g = group(2)
    a, b = g.comms
    dst = [c.zeros(5000, torch.float32) for c in g.comms]
    src = torch.arange(5000, dtype=torch.float32, device=f"cuda:{a.device}")
    torch.cuda.synchronize()
    a.put_signal(src, dst[0], peer=1, signal=3, blocks=4, stream=g.streams[0])
    b.wait_signal(signal=3, count=4, stream=g.streams[1])
    g.run(lambda c, r, st: c.barrier())
    g.synchronize()
    no_errors(g)
    assert torch.equal(dst[1].cpu(), src.cpu())
    for c, d in zip(g.comms, dst):
        c.free(d)


def test_channels_run_concurrently():
    """Independent all-reduces on different channels/streams use disjoint flag
    slots, so they may overlap and complete in any order."""
    n = 4
    g = group(n)
    sizes = [100, 5000, 70000, 300000, 9, 2048, 40000, 1]
    nch = 4
    lanes = [[torch.cuda.Stream(device=c.device) for _ in range(nch)] for c in g.comms]
    sends = [[c.empty(s, torch.int32) for s in sizes] for c in g.comms]
    recvs = [[c.empty(s, torch.int32) for s in sizes] for c in g.comms]
    for r in range(n):
        for t in sends[r]:
            t.fill_(r + 1)
    torch.cuda.synchronize()
    for rep in range(3):
        for r, c in enumerate(g.comms):
            for i in range(len(sizes)):
                ch = i % nch
                c.all_reduce(sends[r][i], recvs[r][i], stream=lanes[r][ch], channel=ch)
    torch.cuda.synchronize()
    no_errors(g)
    for r in range(n):
        for t in recvs[r]:
            assert bool((t == n * (n + 1) // 2).all())
    for r, c in enumerate(g.comms):
        for t in sends[r] + recvs[r]:
            c.free(t)


def test_graph_capture_replay():
    """Collectives keep their epochs in device memory so a captured graph can be
    replayed (launch-bound loops are captured once, replayed many times)."""
    n = 2
    g = spin_group(n)
    numel = 2048
    bufs = [c.empty(numel, torch.float32) for c in g.comms]
    outs = [c.empty(numel, torch.float32) for c in g.comms]
    for r, b in enumerate(bufs):
        b.fill_(float(r + 1))
    torch.cuda.synchronize()
    graphs = []
    for r, c in enumerate(g.comms):
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=g.streams[r]):
            c.all_reduce(bufs[r], outs[r], algo="oneshot", stream=g.streams[r])
            c.all_reduce(bufs[r], outs[r], algo="ll", stream=g.streams[r])
        graphs.append(gr)
    for it in range(3):
        for r, b in enumerate(bufs):
            b.fill_(float(r + 1 + it))
        torch.cuda.synchronize()
        for r in range(n):
            with torch.cuda.stream(g.streams[r]):
                graphs[r].replay()
        g.synchronize()
        torch.cuda.synchronize()
        no_errors(g)
        for r in range(n):
            assert torch.all(outs[r] == float(3 + 2 * it))
    for c, a, b in zip(g.comms, bufs, outs):
        c.free(a)
        c.free(b)


def test_watchdog_reports_missing_peer():
    """A rank that never shows up must not hang the GPU: the bounded spin sets
    the error word and the kernel retires (failure-detection, SURVEY 5.3)."""
    g = LocalGroup(2, heapBytes=1 << 20, stageBytes=1 << 20, maxBlocks=2, timeoutMs=300, streamSync=0)
    try:
        t = torch.ones(1 << 16, device="cuda:0")
        o = torch.empty_like(t)
        g.comms[0].all_reduce(t, o, algo="oneshot", stream=g.streams[0])
        g.streams[0].synchronize()
        assert g.comms[0].check_error(g.streams[0]) != 0
    finally:
        g.close()


def test_stress_random_skew_and_sizes():
    """Flag-ordering stress: back-to-back collectives of random kinds, sizes
    and algorithms while every rank starts each one at a random time offset
    (device-side sleep), without host synchronisation inside a batch."""
    import random

    n = 4
    g = group(n)
    rng = random.Random(1234)
    dev = [c.device for c in g.comms]
    max_elems = 1 << 18
    sends = [c.empty(max_elems, torch.int32) for c in g.comms]
    recvs = [[c.empty(max_elems, torch.int32) for _ in range(6)] for c in g.comms]
    gathers = [c.empty(max_elems, torch.int32) for c in g.comms]
    try:
        for it in range(30):
            base = [torch.randint(-1000, 1000, (max_elems,), dtype=torch.int32) for _ in range(n)]
            for r in range(n):
                sends[r].copy_(base[r].to(f"cuda:{dev[r]}"))
            g.synchronize()
            torch.cuda.synchronize()
            plan = []
            for k in range(6):
                kind = rng.choice(["allreduce", "allreduce", "allreduce", "allgather", "bcast"])
                numel = rng.choice([1, 7, 256, 1000, 4096, 33333, 1 << 16, 1 << 18])
                algo = rng.choice(["auto", "ll", "oneshot", "twoshot"])
                if algo == "ll" and numel * 4 > 32 * 1024:
                    algo = "auto"
                plan.append((kind, numel, algo, rng.randrange(n)))
            for k, (kind, numel, algo, root) in enumerate(plan):
                skew = [rng.randrange(0, 400_000) for _ in range(n)]

                def issue(c, r, st, kind=kind, numel=numel, algo=algo, root=root, k=k, skew=skew):
                    torch.cuda._sleep(skew[r])
                    if kind == "allreduce":
                        c.all_reduce(sends[r][:numel], recvs[r][k][:numel], op="sum", algo=algo)
                    elif kind == "allgather":
                        per = max(1, numel // n)
                        c.all_gather(sends[r][:per], gathers[r][: per * n])
                        recvs[r][k][: per * n].copy_(gathers[r][: per * n])
                    else:
                        recvs[r][k][:numel].copy_(sends[r][:numel])
                        c.broadcast(recvs[r][k][:numel], root=root)

                g.run(issue)
            g.synchronize()
            assert g.check_errors() == [0] * n
            for k, (kind, numel, algo, root) in enumerate(plan):
                if kind == "allreduce":
                    exp = sum(b[:numel].to(torch.int64) for b in base).to(torch.int32)
                elif kind == "allgather":
                    per = max(1, numel // n)
                    exp = torch.cat([b[:per] for b in base])
                else:
                    exp = base[root][:numel]
                for r in range(n):
                    got = recvs[r][k][: exp.numel()].cpu()
                    assert torch.equal(got, exp), f"iteration {it} op {k} {kind} numel {numel} algo {algo} rank {r}"
    finally:
        for r, c in enumerate(g.comms):
            c.free(sends[r])
            c.free(gathers[r])
            for t in recvs[r]:
                c.free(t)


@pytest.mark.parametrize("n", [2, 4])
@pytest.mark.parametrize("symmetric", [True, False])
def test_large_pull_collectives_use_the_bulk_copy_engine(n, symmetric):
    """Chunks >= 256 KiB go through the TMA kernel (cp.async.bulk through
    shared memory); results must match the LDG/STG path bit for bit, including
    a chunk size that is not a multiple of the 32 KiB tile."""
    g = group(n)
    per = (384 << 10) // 4 + 36  # 384 KiB + 144 B per rank (int32), 16-byte multiple
    base = [torch.randint(-(2**31), 2**31 - 1, (per * n,), dtype=torch.int32) for _ in range(n)]

    def alloc(c, numel):
        return c.empty(numel, torch.int32) if symmetric else torch.empty(numel, dtype=torch.int32, device=f"cuda:{c.device}")

    sends = [alloc(c, per * n) for c in g.comms]
    outs = [alloc(c, per * n) for c in g.comms]
    for r, c in enumerate(g.comms):
        sends[r].copy_(base[r].to(f"cuda:{c.device}"))
    for c in g.comms:
        c.stats(reset=True)

    # all-gather of the first `per` elements
    g.run(lambda c, r, st: c.all_gather(sends[r][:per], outs[r]))
    g.synchronize()
    no_errors(g)
    exp = torch.cat([b[:per] for b in base])
    for r in range(n):
        assert torch.equal(outs[r].cpu(), exp)
    # all-to-all
    g.run(lambda c, r, st: c.all_to_all(sends[r], outs[r]))
    g.synchronize()
    no_errors(g)
    for r in range(n):
        exp = torch.cat([base[p][r * per : (r + 1) * per] for p in range(n)])
        assert torch.equal(outs[r].cpu(), exp)
    # scatter from rank 1, gather to rank 0, broadcast (below the 2-step size)
    small = [alloc(c, per) for c in g.comms]
    g.run(lambda c, r, st: c.scatter(sends[r], small[r], root=1))
    g.synchronize()
    for r in range(n):
        assert torch.equal(small[r].cpu(), base[1][r * per : (r + 1) * per])
    g.run(lambda c, r, st: c.gather(small[r], outs[r], root=0))
    g.synchronize()
    assert torch.equal(outs[0].cpu(), base[1])
    bc = [alloc(c, per) for c in g.comms]
    for r, c in enumerate(g.comms):
        bc[r].copy_(base[r][:per].to(f"cuda:{c.device}"))
    g.run(lambda c, r, st: c.broadcast(bc[r], root=n - 1))
    g.synchronize()
    no_errors(g)
    for r in range(n):
        assert torch.equal(bc[r].cpu(), base[n - 1][:per])
    # ...and it really was the copy engine
    # (some modes take other routes for symmetric buffers; most go through it)
    assert all(c.stats()["tma_launches"] >= 3 for c in g.comms), [c.stats() for c in g.comms]
    # same results with the engine switched off
    for c in g.comms:
        c.configure(tmaMinBytes=0)
        c.stats(reset=True)
    g.run(lambda c, r, st: c.all_to_all(sends[r], outs[r]))
    g.synchronize()
    for r in range(n):
        exp = torch.cat([base[p][r * per : (r + 1) * per] for p in range(n)])
        assert torch.equal(outs[r].cpu(), exp)
    assert all(c.stats()["tma_launches"] == 0 for c in g.comms)
    for c in g.comms:
        c.configure(tmaMinBytes=256 << 10)
    if symmetric:
        for r, c in enumerate(g.comms):
            for t in (sends[r], outs[r], small[r], bc[r]):
                c.free(t)


# ---------------------------------------------------------------------------
# grouped all-reduce: many tensors, one launch
# ---------------------------------------------------------------------------
GROUP_SIZES = [1, 3, 4, 7, 64, 1000, 4099, 65536 + 5, 9408, 300000, 2, 33]


@pytest.mark.parametrize("n", [1, 2, 4, 8, 3])
@pytest.mark.parametrize("dtype,op", [(torch.int32, "sum"), (torch.float32, "sum"), (torch.bfloat16, "max"), (torch.int64, "min"), (torch.uint8, "bor")])
def test_grouped_allreduce_matches_per_tensor_reference(n, dtype, op):
    """One launch over a mixed list of tensors (odd sizes: < 16-byte tails,
    tensors smaller than one vector, tensors spanning several ranks' ownership
    ranges) equals an independent all-reduce of every tensor."""
    g = group(n)
    esize = torch.empty((), dtype=dtype).element_size()
    sends = [[c.empty(s, dtype) for s in GROUP_SIZES] for c in g.comms]
    recvs = [[c.empty(s, dtype) for s in GROUP_SIZES] for c in g.comms]
    ins = [make_inputs(n, s, dtype, "cpu", seed=s) for s in GROUP_SIZES]
    for r in range(n):
        for i, t in enumerate(sends[r]):
            t.copy_(ins[i][r])
            recvs[r][i].fill_(0)
    torch.cuda.synchronize()
    plans = [c.prepare_group(sends[r], recvs[r]) for r, c in enumerate(g.comms)]
    assert plans[0].launches == 1
    for _ in range(2):
        g.run(lambda c, r, st: c.all_reduce_group(plans[r], op=op))
    g.synchronize()
    no_errors(g)
    for i, s in enumerate(GROUP_SIZES):
        for r in range(n):
            check(recvs[r][i], ins[i], op)
    # in place + transient table
    g.run(lambda c, r, st: c.all_reduce_many(sends[r], op=op))
    g.synchronize()
    no_errors(g)
    for i, s in enumerate(GROUP_SIZES):
        for r in range(n):
            check(sends[r][i], ins[i], op)
    for p in plans:
        p.close()
    for r, c in enumerate(g.comms):
        for t in sends[r] + recvs[r]:
            c.free(t)
    assert esize > 0


def test_grouped_allreduce_many_tensors_split_into_launches():
    n = 2
    g = group(n)
    k = 1500  # > FB_GROUP_MAX_SEGS: two launches
    flat = [c.empty(k * 64, torch.int32) for c in g.comms]
    for r, f in enumerate(flat):
        f.copy_(torch.arange(k * 64, dtype=torch.int32) + r)
    torch.cuda.synchronize()
    views = [[f[i * 64 : i * 64 + 1 + (i % 60)] for i in range(k)] for f in flat]
    plans = [c.prepare_group(views[r]) for r, c in enumerate(g.comms)]
    assert plans[0].launches == 2
    g.run(lambda c, r, st: c.all_reduce_group(plans[r]))
    g.synchronize()
    no_errors(g)
    base = torch.arange(k * 64, dtype=torch.int32)
    touched = torch.zeros(k * 64, dtype=torch.bool)
    for i in range(k):
        touched[i * 64 : i * 64 + 1 + (i % 60)] = True
    for r in range(n):
        # reduced positions hold the sum over ranks, the padding between the
        # views keeps this rank's own values
        exp = torch.where(touched, n * base + n * (n - 1) // 2, base + r)
        assert torch.equal(flat[r].cpu(), exp)
    for p in plans:
        p.close()
    for c, f in zip(g.comms, flat):
        c.free(f)


def test_grouped_rejects_non_symmetric_tensors():
    g = group(2)
    c = g.comms[0]
    t = torch.zeros(64, dtype=torch.int32, device=f"cuda:{c.device}")
    from faabric_b200.parallel.comm import CommError

    with pytest.raises(CommError):
        c.prepare_group([t])


@pytest.mark.parametrize("n", [2, 4])
def test_in_kernel_barrier_path_ll_oneshot_twoshot(n):
    """The product path on one GPU: LL slots, in-kernel flag barriers, grouped
    kernel with its two barriers (co-residency asserted by spin_group)."""
    g = spin_group(n)
    assert not g.comms[0].stream_sync
    for algo, numel in (("ll", 1000), ("oneshot", 5000), ("twoshot", 70001)):
        sends = [c.empty(numel, torch.int32) for c in g.comms]
        recvs = [c.empty(numel, torch.int32) for c in g.comms]
        for r, t in enumerate(sends):
            t.copy_(torch.arange(numel, dtype=torch.int32) * (r + 1))
        torch.cuda.synchronize()
        g.run(lambda c, r, st: c.all_reduce(sends[r], recvs[r], algo=algo))
        g.synchronize()
        no_errors(g)
        assert g.comms[0].last_algo == algo
        exp = torch.arange(numel, dtype=torch.int32) * (n * (n + 1) // 2)
        for r in range(n):
            assert torch.equal(recvs[r].cpu(), exp)
        plans = [c.prepare_group([sends[r]], [recvs[r]]) for r, c in enumerate(g.comms)]
        for t in recvs:
            t.zero_()
        torch.cuda.synchronize()
        g.run(lambda c, r, st: c.all_reduce_group(plans[r]))
        g.synchronize()
        no_errors(g)
        for r in range(n):
            assert torch.equal(recvs[r].cpu(), exp)
        for p in plans:
            p.close()
        for c, a, b in zip(g.comms, sends, recvs):
            c.free(a)
            c.free(b)
