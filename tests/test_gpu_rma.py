"""One-sided atomics on the device (accumulate, fetch, compare-and-swap), bit
for bit against tests/rma_oracle.py.

All ranks share cuda:0, so "peer" memory is the same GPU's HBM reached through
the peer mapping the kernels use for any peer.  The kernels never wait on a
peer, so no co-residency is needed.

* One writer per element: every supported (dtype, op), with and without
  fetch, at one element, one vector plus a scalar tail, a range across a page
  boundary and several MiB, at natural-alignment offsets inside 16-byte
  blocks, from unaligned origins into unaligned fetch buffers; the bytes
  around the target stay untouched.
* Contention: every rank accumulates K times into the same elements; ops that
  are exact in any order must match the oracle fold, and a random float sum
  stays inside the math.fsum bound.
* Atomicity of fetch and compare-and-swap: counters end exact and the fetched
  tickets are exactly 0 .. N*K-1, also for 1- and 2-byte counters whose
  neighbouring bytes other ranks update at the same time.
* Rejections happen before any launch, and every collective rejects the
  one-sided ops."""

import math
import threading
import zlib

import numpy as np
import pytest
import torch

import rma_oracle as rm
from reduce_oracle import FLOAT_DTYPES, INT_DTYPES, INT_OPS, NP_DTYPES, PAIR_DTYPES, f32_to_bf16, itemsize
from test_gpu_reduce_matrix import float_values, make_inputs

pytestmark = pytest.mark.gpu

from faabric_b200.parallel import LocalGroup  # noqa: E402
from faabric_b200.parallel.comm import CommError  # noqa: E402

CFG = dict(heapBytes=24 << 20, stageBytes=1 << 20, maxBlocks=4, timeoutMs=8000)
WIN = (4 << 20) + (32 << 10)
SENTINEL = 0xA5
DEV = "cuda:0"

GROUPS = {}


def group(n):
    if n not in GROUPS:
        g = LocalGroup(n, devices=[0] * n, **CFG)
        g.wins = [c.empty(WIN, torch.uint8) for c in g.comms]
        GROUPS[n] = g
    return GROUPS[n]


@pytest.fixture(scope="module", autouse=True)
def _cleanup():
    yield
    for g in GROUPS.values():
        g.close()
    GROUPS.clear()


def raw(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).to(DEV)


def host(t, dtype):
    return t.cpu().numpy().view(NP_DTYPES[dtype])


def shifted(nbytes, shift):
    """A device byte buffer that starts `shift` bytes past a 16-byte boundary."""
    return torch.empty(nbytes + 16, dtype=torch.uint8, device=DEV)[shift : shift + nbytes]


def no_errors(g):
    assert g.check_errors() == [0] * g.size


def target_values(rng, dtype, op, count):
    tgt, org = make_inputs(rng, dtype, op, 2, count)
    if dtype in rm.PADDED_PAIRS:
        # non-zero padding, which every op must keep
        tgt.view(np.uint8).reshape(-1, 16)[:, 12:] = rng.integers(1, 255, (count, 4), dtype=np.uint8)
    return tgt, org


# ---------------------------------------------------------- one writer ----
def cases(e):
    """(target offset in the window, element count, origin shift, writer == peer)"""
    last_slot = 16 - e if e < 16 else 0
    return [
        (64 + last_slot, 1, 1, False),  # one element in the last slot of a 16-byte block
        (128 + (e if e < 16 else 0), 16 // e + 3, 3, True),  # a vector and a scalar tail, to self
        (8192 - 5 * e, 64 // e * 4 + 5, 5, False),  # across a page boundary
        (16384, (3 << 20) // e + 1, 0, False),  # several MiB, 16-byte aligned origin
    ]


def accumulate_case(g, dtype, op, fetch, toff, count, oshift, self_target, rng):
    e = itemsize(dtype)
    nbytes = count * e
    writer, peer = 0, (0 if self_target else 1)
    c = g.comms[writer]
    tgt, org = target_values(rng, dtype, op, count)
    win = g.wins[peer]
    win.fill_(SENTINEL)
    win[toff : toff + nbytes].copy_(raw(tgt))
    src = None
    if op != "no_op":
        src = shifted(nbytes, oshift)
        src.copy_(raw(org))
    res = None
    if fetch:
        res = shifted(nbytes, 7)
        res.fill_(0x5A)
    torch.cuda.synchronize()
    launches = c.stats()["launches"]
    with torch.cuda.stream(g.streams[writer]):
        c.accumulate(src, g.wins[writer][toff : toff + nbytes], peer, op=op, dtype=dtype, fetch=res)
    g.synchronize()
    assert c.stats()["launches"] == launches + 1
    exp_t, exp_f = rm.accumulate(tgt, org, dtype, op)
    what = f"{dtype} {op} fetch={fetch} count={count} offset={toff}"
    rm.assert_same(host(win[toff : toff + nbytes], dtype), exp_t, dtype, what + " target")
    if fetch:
        rm.assert_same(host(res, dtype), exp_f, dtype, what + " fetched")
    assert bool((win[:toff] == SENTINEL).all()) and bool((win[toff + nbytes :] == SENTINEL).all()), what + ": bytes around the target changed"
    if src is not None:
        assert np.array_equal(src.cpu().numpy(), np.ascontiguousarray(org).view(np.uint8)), what + ": origin modified"


@pytest.mark.parametrize("dtype,op", rm.ACCUMULATE, ids=[f"{d}-{o}" for d, o in rm.ACCUMULATE])
def test_accumulate_one_writer(dtype, op):
    g = group(2)
    rng = np.random.default_rng(zlib.crc32(f"{dtype}-{op}".encode()))
    for toff, count, oshift, self_target in cases(itemsize(dtype)):
        accumulate_case(g, dtype, op, False, toff, count, oshift, self_target, rng)
    no_errors(g)


@pytest.mark.parametrize("dtype,op", rm.FETCH, ids=[f"{d}-{o}" for d, o in rm.FETCH])
def test_get_accumulate_one_writer(dtype, op):
    g = group(2)
    rng = np.random.default_rng((zlib.crc32(f"{dtype}-{op}".encode())) + 1)
    for toff, count, oshift, self_target in cases(itemsize(dtype)):
        accumulate_case(g, dtype, op, True, toff, count, oshift, self_target, rng)
    no_errors(g)


# ---------------------------------------------------------- contention ----
K = 12
EXACT_ANY_ORDER = (
    [(d, o) for d in INT_DTYPES for o in INT_OPS]
    + [(d, o) for d in FLOAT_DTYPES for o in ("max", "min", "sum")]
    + [(d, o) for d in PAIR_DTYPES for o in ("maxloc", "minloc")]
)


def contention_inputs(rng, dtype, op, n, count):
    if dtype in FLOAT_DTYPES and op == "sum":
        # small integers: every partial sum is exact, so every order agrees
        vals = [rng.integers(-1, 2, count).astype(np.float64) for _ in range(n * K + 1)]
        if dtype == "bf16":
            return [f32_to_bf16(v.astype(np.float32)) for v in vals]
        return [v.astype(NP_DTYPES[dtype]) for v in vals]
    return make_inputs(rng, dtype, op, n * K + 1, count)


@pytest.mark.parametrize("n", [2, 8])
@pytest.mark.parametrize("dtype,op", EXACT_ANY_ORDER, ids=[f"{d}-{o}" for d, o in EXACT_ANY_ORDER])
def test_concurrent_accumulates_are_exact(n, dtype, op):
    g = group(n)
    rng = np.random.default_rng(n * 1000 + zlib.crc32(f"{dtype}-{op}".encode()))
    count = 257
    e = itemsize(dtype)
    nbytes = count * e
    toff = 4096
    vals = contention_inputs(rng, dtype, op, n, count)
    init, origins = vals[0], vals[1:]
    if dtype in rm.PADDED_PAIRS:
        init.view(np.uint8).reshape(-1, 16)[:, 12:] = 0x3C
    srcs = [[shifted(nbytes, 1 + (r + k) % 5) for k in range(K)] for r in range(n)]
    for r in range(n):
        for k in range(K):
            srcs[r][k].copy_(raw(origins[r * K + k]))
    g.wins[0].fill_(SENTINEL)
    g.wins[0][toff : toff + nbytes].copy_(raw(init))
    torch.cuda.synchronize()

    def issue(c, r, st):
        for k in range(K):
            c.accumulate(srcs[r][k], g.wins[r][toff : toff + nbytes], 0, op=op, dtype=dtype)

    g.run(issue)
    g.synchronize()
    no_errors(g)
    exp = rm.fold(init, origins, dtype, op)
    rm.assert_same(host(g.wins[0][toff : toff + nbytes], dtype), exp, dtype, f"{n} ranks x {K} {dtype} {op}")
    assert bool((g.wins[0][:toff] == SENTINEL).all()) and bool((g.wins[0][toff + nbytes :] == SENTINEL).all())


@pytest.mark.parametrize("n", [2, 8])
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_packed_and_cas_half_sums_mix_on_the_same_words(n, dtype):
    """Even ranks send 16-byte aligned origins (packed red.add.noftz, eight
    elements per instruction), odd ranks unaligned ones (CAS on the enclosing
    word, element by element), into the same elements at once."""
    g = group(n)
    rng = np.random.default_rng(n * 31 + len(dtype))
    count = 8 * 40 + 3
    nbytes = count * 2
    toff = 4096
    vals = contention_inputs(rng, dtype, "sum", n, count)
    init, origins = vals[0], vals[1:]
    srcs = [[shifted(nbytes, 0 if r % 2 == 0 else 2 + 2 * (k % 7)) for k in range(K)] for r in range(n)]
    for r in range(n):
        for k in range(K):
            srcs[r][k].copy_(raw(origins[r * K + k]))
    assert all((srcs[r][k].data_ptr() % 16 == 0) == (r % 2 == 0) for r in range(n) for k in range(K))
    g.wins[0].fill_(SENTINEL)
    g.wins[0][toff : toff + nbytes].copy_(raw(init))
    torch.cuda.synchronize()
    g.run(lambda c, r, st: [c.accumulate(srcs[r][k], g.wins[r][toff : toff + nbytes], 0, dtype=dtype) for k in range(K)])
    g.synchronize()
    no_errors(g)
    rm.assert_same(host(g.wins[0][toff : toff + nbytes], dtype), rm.fold(init, origins, dtype, "sum"), dtype, f"{n} ranks {dtype} packed + CAS")
    assert bool((g.wins[0][:toff] == SENTINEL).all()) and bool((g.wins[0][toff + nbytes :] == SENTINEL).all())


@pytest.mark.parametrize("fetch", [False, True])
@pytest.mark.parametrize("op", ["maxloc", "minloc"])
@pytest.mark.parametrize("dtype", PAIR_DTYPES)
def test_concurrent_pair_ties_end_at_the_lowest_index(dtype, op, fetch):
    """Every writer offers the same value with its own index, so every update
    is decided by the index alone (the case a torn read of a pair would get
    wrong); the padding of the 16-byte pairs must survive."""
    n = 8
    g = group(n)
    count = 4
    e = itemsize(dtype)
    nbytes = count * e
    toff = 12288
    init = np.zeros(count, NP_DTYPES[dtype])
    init["v"] = 1
    init["i"] = 1 << 30
    if dtype in rm.PADDED_PAIRS:
        init.view(np.uint8).reshape(-1, 16)[:, 12:] = 0x5C
    origins = []
    for r in range(n):
        for k in range(K):
            o = np.zeros(count, NP_DTYPES[dtype])
            o["v"] = 1
            o["i"] = 1000 - (k * n + r) * 7 + np.arange(count)
            origins.append(o)
    srcs = [raw(o) for o in origins]
    res = [torch.empty(nbytes, dtype=torch.uint8, device=DEV) for _ in origins] if fetch else [None] * len(origins)
    g.wins[0][toff : toff + nbytes].copy_(raw(init))
    torch.cuda.synchronize()
    g.run(lambda c, r, st: [c.accumulate(srcs[r * K + k], g.wins[r][toff : toff + nbytes], 0, op=op, dtype=dtype, fetch=res[r * K + k]) for k in range(K)])
    g.synchronize()
    no_errors(g)
    rm.assert_same(host(g.wins[0][toff : toff + nbytes], dtype), rm.fold(init, origins, dtype, op), dtype, f"{dtype} {op} ties")
    if fetch:
        # every fetched pair is a state the element really held: the initial
        # pair or one of the offered ones, never a mix of two
        offered = {(1, int(o["i"][j]), j) for o in origins for j in range(count)} | {(1, 1 << 30, j) for j in range(count)}
        for t in res:
            got = host(t, dtype)
            assert all((int(got["v"][j]), int(got["i"][j]), j) in offered for j in range(count))


UNIT_ROUNDOFF = {"f32": 2.0**-24, "f64": 2.0**-53}


@pytest.mark.parametrize("dtype", ["f32", "f64"])
def test_concurrent_random_float_sums_stay_in_the_fsum_bound(dtype):
    n = 8
    g = group(n)
    rng = np.random.default_rng(77)
    count = 1000
    nbytes = count * itemsize(dtype)
    vals = [float_values(rng, dtype, count, narrow_only=True) for _ in range(n * K + 1)]
    srcs = [raw(v) for v in vals[1:]]
    g.wins[0][:nbytes].copy_(raw(vals[0]))
    torch.cuda.synchronize()
    g.run(lambda c, r, st: [c.accumulate(srcs[r * K + k], g.wins[r][:nbytes], 0, dtype=dtype) for k in range(K)])
    g.synchronize()
    no_errors(g)
    got = host(g.wins[0][:nbytes], dtype).astype(np.float64)
    xs = np.stack([v.astype(np.float64) for v in vals])
    exact = np.array([math.fsum(col) for col in xs.T])
    bound = (len(vals) - 1) * UNIT_ROUNDOFF[dtype] * np.sum(np.abs(xs), axis=0)
    err = np.abs(got - exact)
    assert np.all(err <= bound), f"worst excess {np.max(err - bound)}"


# ------------------------------------------------- fetch and CAS atomicity ----
@pytest.mark.parametrize("n", [2, 4, 8])
@pytest.mark.parametrize("dtype", ["i64", "i16", "i8"])
def test_fetch_and_op_tickets_are_unique(n, dtype):
    """N ranks x K fetch_and_op(sum, 1) on one counter: it ends at N*K and the
    fetched tickets are 0 .. N*K-1.  For the sub-word counters, the other
    bytes of the 16-byte block are counters other ranks bump at the same time."""
    g = group(n)
    e = itemsize(dtype)
    slots = 16 // e
    mine = 1  # the ticket counter's slot; every other slot is a neighbour counter
    base = 8192
    g.wins[0][base : base + 16].zero_()
    one = raw(np.array([1], NP_DTYPES[dtype]))
    tickets = torch.full((n, K, 16), 0x77, dtype=torch.uint8, device=DEV)
    torch.cuda.synchronize()

    def issue(c, r, st):
        for k in range(K):
            c.fetch_and_op(one, g.wins[r][base + mine * e : base + (mine + 1) * e], 0, tickets[r, k, 3 : 3 + e], dtype=dtype)
            nb = [s for s in range(slots) if s != mine][(r + k) % (slots - 1)] if slots > 1 else mine
            if nb != mine:
                c.accumulate(one, g.wins[r][base + nb * e : base + (nb + 1) * e], 0, dtype=dtype)

    g.run(issue)
    g.synchronize()
    no_errors(g)
    counters = host(g.wins[0][base : base + 16], dtype)
    assert int(counters[mine]) == n * K
    got = sorted(int(np.frombuffer(tickets[r, k, 3 : 3 + e].cpu().numpy().tobytes(), NP_DTYPES[dtype])[0]) for r in range(n) for k in range(K))
    assert got == list(range(n * K))
    if slots > 1:
        expect = np.zeros(slots, np.int64)
        for r in range(n):
            for k in range(K):
                expect[[s for s in range(slots) if s != mine][(r + k) % (slots - 1)]] += 1
        expect[mine] = n * K
        assert counters.astype(np.int64).tolist() == expect.tolist()


@pytest.mark.parametrize("dtype", INT_DTYPES)
def test_compare_and_swap_retry_loops_count_exactly(dtype):
    """Every rank thread increments one counter K times with a host-driven
    compare-and-swap retry loop; the byte after the counter is a neighbour
    that must stay as it was."""
    n = 4
    g = group(n)
    e = itemsize(dtype)
    np_dt = NP_DTYPES[dtype]
    off = 12288 + (16 - e if e < 8 else 8)
    g.wins[0][off - 8 : off + 16].fill_(0xEE)
    g.wins[0][off : off + e].zero_()
    torch.cuda.synchronize()
    errors = []

    def worker(r):
        try:
            c, st = g.comms[r], g.streams[r]
            with torch.cuda.device(0), torch.cuda.stream(st):
                cmp = torch.zeros(e, dtype=torch.uint8, device=DEV)
                swp = torch.zeros(e, dtype=torch.uint8, device=DEV)
                res = torch.zeros(e, dtype=torch.uint8, device=DEV)
                guess = 0
                done = 0
                tries = 0
                while done < K:
                    tries += 1
                    assert tries < 100000, "no progress"
                    cmp.copy_(raw(np.array([guess], np_dt)))
                    swp.copy_(raw(np.array([guess + 1], np_dt)))
                    c.compare_and_swap(cmp, swp, g.wins[r][off : off + e], 0, res, dtype=dtype)
                    old = int(np.frombuffer(res.cpu().numpy().tobytes(), np_dt)[0])
                    if old == guess:
                        done += 1
                        guess += 1
                    else:
                        guess = old
        except Exception as ex:  # reported by the main thread
            errors.append(ex)

    ts = [threading.Thread(target=worker, args=(r,)) for r in range(n)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=300)
    assert not errors, errors
    g.synchronize()
    no_errors(g)
    assert int(host(g.wins[0][off : off + e], dtype)[0]) == n * K
    around = g.wins[0][off - 8 : off + 16].cpu().numpy()
    assert (around[:8] == 0xEE).all() and (around[8 + e :] == 0xEE).all()


# ------------------------------------------------------------ rejections ----
def _launches(g):
    return [c.stats()["launches"] for c in g.comms]


@pytest.mark.parametrize("dtype,op", rm.UNSUPPORTED, ids=[f"{d}-{o}" for d, o in rm.UNSUPPORTED])
def test_unsupported_pairs_are_rejected_before_any_launch(dtype, op):
    g = group(2)
    c = g.comms[0]
    e = itemsize(dtype)
    src = torch.zeros(4 * e, dtype=torch.uint8, device=DEV)
    res = torch.zeros(4 * e, dtype=torch.uint8, device=DEV)
    before = _launches(g)
    with pytest.raises(CommError):
        c.accumulate(src, g.wins[0][: 4 * e], 1, op=op, dtype=dtype)
    with pytest.raises(CommError):
        c.accumulate(src, g.wins[0][: 4 * e], 1, op=op, dtype=dtype, fetch=res)
    assert _launches(g) == before


def test_bad_arguments_are_rejected_before_any_launch():
    g = group(2)
    c = g.comms[0]
    w = g.wins[0]
    src = torch.ones(4, dtype=torch.int32, device=DEV)
    before = _launches(g)
    with pytest.raises(CommError):  # NO_OP needs a fetch buffer
        c.accumulate(src, w[:16].view(torch.int32), 1, op="no_op")
    for dtype in ("i16", "f32", "i64", "f32_i32", "f64_i32"):
        e = itemsize(dtype)
        with pytest.raises(CommError):  # misaligned target
            c.accumulate(torch.zeros(e, dtype=torch.uint8, device=DEV), w[e // 2 : e // 2 + e], 1, dtype=dtype, op="replace")
    with pytest.raises(CommError):  # not in the heap
        c.accumulate(src, torch.zeros(4, dtype=torch.int32, device=DEV), 1)
    with pytest.raises(CommError):  # longer than the symmetric tensor
        c.accumulate(torch.ones(8, dtype=torch.int32, device=DEV), w[WIN - 16 :].view(torch.int32), 1)
    # the native range check: past the end of the heap, and inside the
    # communicator's own area below the user heap (FB_E_INVALID)
    st = torch.cuda.current_stream().cuda_stream
    for off in (1 << 40, CFG["heapBytes"] * 2 - 8, 0):
        rc = c._lib.fb_accumulate(c._h, src.data_ptr(), off, 4, 4, 2, 1, None, st)
        assert rc == -2, (off, rc)
    with pytest.raises(CommError):  # peer outside the group
        c.accumulate(src, w[:16].view(torch.int32), 2)
    with pytest.raises(CommError):  # compare-and-swap is integer only
        one = torch.ones(1, dtype=torch.float32, device=DEV)
        c.compare_and_swap(one, one, w[:4].view(torch.float32), 1, one.clone())
    with pytest.raises(CommError):  # fetch_and_op takes one element
        c.fetch_and_op(src, w[:16].view(torch.int32), 1, src.clone())
    assert _launches(g) == before
    no_errors(g)


@pytest.mark.parametrize("op", ["replace", "no_op"])
def test_collectives_reject_one_sided_ops(op):
    g = group(2)
    c = g.comms[0]
    a = c.empty(64, torch.float32)
    b = c.empty(64, torch.float32)
    before = _launches(g)
    for call in (
        lambda: c.all_reduce(a, b, op=op),
        lambda: c.reduce(a, b, root=0, op=op),
        lambda: c.scan(a, b, op=op),
        lambda: c.reduce_scatter(a, b[:32], op=op),
        lambda: c.all_reduce_many([a], [b], op=op),
    ):
        with pytest.raises(CommError):
            call()
    assert _launches(g) == before
    c.free(a)
    c.free(b)
