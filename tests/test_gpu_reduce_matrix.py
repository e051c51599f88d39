"""Every device reduction instance, bit for bit against the NumPy oracle.

The reduce kernels exist once per supported (dtype, op) pair and, inside each,
once per unrolled rank count (NR = 2, 4, 8 and a generic loop), plus the LL
and grouped kernels, so a defect can live in a single (type, NR) instance.
Every single-GPU path folds the ranks in rank order, so the exact result is
known (tests/reduce_oracle.py) and compared bit for bit; a NaN matches any
NaN.  Inputs reach the edges: full-range integers (SUM/PROD wrap, top bits set
for MAX/MIN signedness), zeros and low-byte-zero values for the logical ops,
signed zeros, infinities, subnormals, wide exponents and cancelling sums for
the floats, value ties for MAXLOC/MINLOC.

All ranks share cuda:0.  One-shot, two-shot, reduce, scan, reduce-scatter and
the grouped kernel run on a group with stream-ordered synchronisation; LL needs
the in-kernel protocol (its slots are its synchronisation), so it runs on a
group whose ranks' kernels are co-resident.  Multimem (NVLS) reductions need a
multicast-capable multi-GPU machine and are not covered here."""

import math

import numpy as np
import pytest
import torch

from reduce_oracle import (
    DTYPES,
    FLOAT_DTYPES,
    FLOAT_OPS,
    INT_DTYPES,
    INT_OPS,
    NP_DTYPES,
    PAIR_DTYPES,
    PAIR_OPS,
    SUPPORTED,
    UNSUPPORTED,
    assert_same,
    f32_to_bf16,
    fold,
    itemsize,
)

pytestmark = pytest.mark.gpu

from faabric_b200.parallel import LocalGroup  # noqa: E402
from faabric_b200.parallel.comm import CommError  # noqa: E402

# launch_api.h: FB_LL_BLOCKS (8) x FB_LL_THREADS (512) vectors of 16 bytes
FB_LL_MAX_BYTES = 8 * 512 * 16

CFG = dict(
    heapBytes=128 << 20,
    stageBytes=1 << 20,
    maxBlocks=4,
    threads=512,
    oneShotMaxBytes=64 << 10,
    timeoutMs=8000,
)
ALGOS = ["ll", "oneshot", "twoshot"]
OPS_FOR = {**{d: INT_OPS for d in INT_DTYPES}, **{d: FLOAT_OPS for d in FLOAT_DTYPES}, **{d: PAIR_OPS for d in PAIR_DTYPES}}
SENTINEL = 0xA5

GROUPS = {}
LL_GROUPS = {}


def group(n):
    if n not in GROUPS:
        GROUPS[n] = LocalGroup(n, **CFG)
    return GROUPS[n]


def ll_group(n):
    """In-kernel synchronisation (streamSync=0), which LL needs; None where
    the ranks' kernels are not co-resident on the shared GPU."""
    if n not in LL_GROUPS:
        g = LocalGroup(n, **{**CFG, "timeoutMs": 2000, "streamSync": 0})
        if g.shares_devices and not g.coresident():
            g.close()
            g = None
        LL_GROUPS[n] = g
    return LL_GROUPS[n]


@pytest.fixture(scope="module", autouse=True)
def _cleanup():
    yield
    for g in list(GROUPS.values()) + list(LL_GROUPS.values()):
        if g is not None:
            g.close()
    GROUPS.clear()
    LL_GROUPS.clear()


def pass_bytes(n):
    """Bytes one grid-wide pass of reduceKernel covers: maxBlocks CTAs x
    threads x UNROLL vectors (UNROLL is 2 for the 8-rank variant, else 4)."""
    return CFG["maxBlocks"] * CFG["threads"] * (2 if n == 8 else 4) * 16


def counts(dtype, byte_sizes):
    e = itemsize(dtype)
    return sorted({b // e for b in byte_sizes if b >= e})


def allreduce_counts(dtype, n, ll):
    e = itemsize(dtype)
    sizes = [
        e,  # one element
        15 // e * e,  # the largest count below one vector
        16,  # exactly one vector
        16 * (n - 1) + e,  # fewer full vectors than ranks: the two-shot tail owner owns none
        FB_LL_MAX_BYTES - e,
        FB_LL_MAX_BYTES,
    ]
    if not ll:
        # every rank's two-shot slice is longer than one pass of the grid
        sizes.append(n * pass_bytes(n) + pass_bytes(n) // 2 + e)
    return counts(dtype, sizes)


# ------------------------------------------------------------------ inputs ----
def rand_bits(rng, dt, count):
    return np.frombuffer(rng.bytes(count * dt.itemsize), dtype=dt).copy()


def _unsigned(dt):
    return np.dtype(f"<u{dt.itemsize}")


def int_inputs(rng, dtype, op, n, count):
    dt = NP_DTYPES[dtype]
    xs = [rand_bits(rng, dt, count) for _ in range(n)]
    if op in ("land", "lor", "lxor"):
        for x in xs:
            u = x.view(_unsigned(dt))
            if dt.itemsize > 1:
                # non-zero values whose low byte is 0
                low0 = rng.random(count) < 0.3
                u[low0] &= ~np.array(0xFF, dtype=u.dtype)
                u[low0 & (u == 0)] = 0x100
            u[rng.random(count) < 0.5] = 0
    return xs


# (smallest subnormal exponent, smallest normal exponent, largest exponent)
EXP_RANGE = {"f16": (-24, -14, 15), "bf16": (-133, -126, 127), "f32": (-149, -126, 127), "f64": (-1074, -1022, 1023)}
SIGN_BIT = {"f16": 0x8000, "bf16": 0x8000, "f32": 0x80000000, "f64": 0x8000000000000000}


def to_float_dtype(x64, dtype):
    with np.errstate(all="ignore"):
        if dtype == "bf16":
            return f32_to_bf16(x64.astype(np.float32))
        return x64.astype(NP_DTYPES[dtype])


def float_values(rng, dtype, count, narrow_only=False):
    lo_sub, lo_norm, hi = EXP_RANGE[dtype]
    mant = rng.uniform(1.0, 2.0, count) * rng.choice([-1.0, 1.0], count)
    x = mant * np.exp2(rng.integers(-4, 5, count)).astype(np.float64)
    if not narrow_only:
        kind = rng.integers(0, 10, count)
        wide = kind == 0
        x[wide] = np.ldexp(mant[wide], rng.integers(lo_norm, hi + 1, int(wide.sum())))
        sub = kind == 1
        x[sub] = np.ldexp(mant[sub], rng.integers(lo_sub, lo_norm, int(sub.sum())))
        special = kind == 2
        x[special] = rng.choice([0.0, -0.0, np.inf, -np.inf], int(special.sum()))
    return to_float_dtype(x, dtype)


def float_inputs(rng, dtype, n, count, narrow_only=False):
    xs = [float_values(rng, dtype, count, narrow_only) for _ in range(n)]
    if n > 1 and not narrow_only:
        # cancelling sums: rank 1 holds -x of rank 0 at about a tenth of the positions
        cancel = rng.random(count) < 0.1
        u0 = xs[0].view(_unsigned(xs[0].dtype))
        u1 = xs[1].view(_unsigned(xs[1].dtype))
        u1[cancel] = u0[cancel] ^ np.array(SIGN_BIT[dtype], dtype=u0.dtype)
    return xs


def pair_inputs(rng, dtype, n, count):
    out = []
    for _ in range(n):
        p = np.zeros(count, dtype=NP_DTYPES[dtype])
        p["v"] = rng.integers(-2, 3, count)  # few values: many ties
        p["i"] = rng.integers(-1000, 1000, count)
        out.append(p)
    return out


def make_inputs(rng, dtype, op, n, count):
    if dtype in INT_DTYPES:
        return int_inputs(rng, dtype, op, n, count)
    if dtype in FLOAT_DTYPES:
        return float_inputs(rng, dtype, n, count)
    return pair_inputs(rng, dtype, n, count)


# ----------------------------------------------------------------- buffers ----
def _raw(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy())


def device_bufs(g, nbytes, symmetric, shifts=None, fill=None):
    """One byte buffer per rank: in the symmetric heap, or ordinary device
    memory starting `shifts[r]` bytes past a 16-byte boundary."""
    bufs = []
    for r, c in enumerate(g.comms):
        if symmetric:
            t = c.empty(nbytes, torch.uint8)
        else:
            s = 0 if shifts is None else shifts[r]
            t = torch.empty(nbytes + s, dtype=torch.uint8, device=f"cuda:{c.device}")[s:]
        if fill is not None:
            t.copy_(_raw(fill[r]))
        else:
            t.fill_(SENTINEL)
        bufs.append(t)
    return bufs


def host(t, dtype):
    return t.cpu().numpy().view(NP_DTYPES[dtype])


def release(g, *buf_lists):
    for bufs in buf_lists:
        for c, t in zip(g.comms, bufs):
            c.free(t)


def no_errors(g):
    assert g.check_errors() == [0] * g.size


def run(g, fn):
    torch.cuda.synchronize()
    g.run(fn)
    g.synchronize()
    no_errors(g)


def untouched(t):
    return bool((t == SENTINEL).all())


def allreduce(g, ins, dtype, op, algo, symmetric, shifts=None):
    nbytes = ins[0].nbytes
    sends = device_bufs(g, nbytes, symmetric, shifts, fill=ins)
    recvs = device_bufs(g, nbytes, symmetric, shifts)
    run(g, lambda c, r, st: c.all_reduce(sends[r], recvs[r], op=op, algo=algo, dtype=dtype))
    assert [c.last_algo for c in g.comms] == [algo] * g.size
    outs = [host(t, dtype) for t in recvs]
    for r, t in enumerate(sends):
        assert np.array_equal(host(t, dtype).view(np.uint8), ins[r].view(np.uint8)), "input modified"
    release(g, sends, recvs)
    return outs


def same_bytes(a, b, dtype):
    if dtype in PAIR_DTYPES:  # padding is unspecified
        assert_same(a, b, dtype, "across ranks / algorithms")
    else:
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), "results differ across ranks / algorithms"


# --------------------------------------------------------------- all_reduce ----
@pytest.mark.parametrize("n", [2, 3, 4, 8])
@pytest.mark.parametrize("dtype", DTYPES)
def test_allreduce_every_op_algorithm_and_size(n, dtype):
    g = group(n)
    gl = ll_group(n)
    rng = np.random.default_rng([n, DTYPES.index(dtype)])
    for op in OPS_FOR[dtype]:
        for count in allreduce_counts(dtype, n, ll=False):
            ins = make_inputs(rng, dtype, op, n, count)
            exp = fold(ins, dtype, op)
            first = None
            for algo in ALGOS:
                grp = gl if algo == "ll" else g
                if grp is None or (algo == "ll" and exp.nbytes > FB_LL_MAX_BYTES):
                    continue
                for symmetric in (True, False):
                    outs = allreduce(grp, ins, dtype, op, algo, symmetric)
                    what = f"n={n} {dtype} {op} {algo} count={count} symmetric={symmetric}"
                    for r in range(n):
                        assert_same(outs[r], exp, dtype, f"{what} rank {r}")
                        first = outs[r] if first is None else first
                        same_bytes(outs[r], first, dtype)


@pytest.mark.parametrize("n", [2, 3, 4, 8])
def test_ll_runs_in_kernel_on_this_device(n):
    """The LL cases above need co-resident rank kernels; say so if they were
    skipped rather than pass silently."""
    if ll_group(n) is None:
        pytest.skip("kernels of different ranks are not co-resident on this GPU: LL not covered")


@pytest.mark.parametrize("dtype,op", UNSUPPORTED)
def test_unsupported_pairs_raise_on_every_path(dtype, op):
    g = group(2)
    nb = 64  # a whole number of elements of every dtype

    def rejected(fn):
        out = []

        def call(c, r, st):
            try:
                fn(c, r)
                out.append(False)
            except CommError:
                out.append(True)

        g.run(call)
        g.synchronize()
        return out == [True] * g.size

    sends = [c.empty(nb * g.size, torch.uint8) for c in g.comms]
    recvs = [c.empty(nb * g.size, torch.uint8) for c in g.comms]
    try:
        for algo in ["auto"] + ALGOS:
            assert rejected(lambda c, r: c.all_reduce(sends[r][:nb], recvs[r][:nb], op=op, algo=algo, dtype=dtype)), algo
        assert rejected(lambda c, r: c.reduce(sends[r][:nb], recvs[r][:nb], root=1, op=op, dtype=dtype))
        assert rejected(lambda c, r: c.scan(sends[r][:nb], recvs[r][:nb], op=op, dtype=dtype))
        assert rejected(lambda c, r: c.reduce_scatter(sends[r], recvs[r][:nb], op=op, dtype=dtype))
        plans = [c.prepare_group([sends[r][:nb], sends[r][nb:]], [recvs[r][:nb], recvs[r][nb:]], dtype=dtype) for r, c in enumerate(g.comms)]
        assert rejected(lambda c, r: c.all_reduce_group(plans[r], op=op))
        assert rejected(lambda c, r: c.all_reduce_many([sends[r][:nb], sends[r][nb:]], [recvs[r][:nb], recvs[r][nb:]], op=op, dtype=dtype))
        for p in plans:
            p.close()
        no_errors(g)
    finally:
        release(g, sends, recvs)


def test_dtype_override_needs_whole_elements():
    g = group(2)
    t = torch.zeros(24, dtype=torch.uint8, device=f"cuda:{g.comms[0].device}")
    with pytest.raises(CommError):
        g.comms[0].all_reduce(t, t.clone(), op="maxloc", dtype="f64_i32")  # 24 bytes: 1.5 pairs
    with pytest.raises(CommError):
        g.comms[0].all_reduce(t, t.clone(), dtype="u128")


# ---------------------------------------------------- reduce / scan / reduce_scatter ----
@pytest.mark.parametrize("n", [3, 4])
@pytest.mark.parametrize("dtype", DTYPES)
def test_reduce_scan_reduce_scatter_every_op(n, dtype):
    g = group(n)
    e = itemsize(dtype)
    rng = np.random.default_rng([100 + n, DTYPES.index(dtype)])
    two_shot_bytes = 2 * CFG["oneShotMaxBytes"] + 16 * n + e  # reduce takes two-shot above 2 x oneShotMaxBytes
    sizes = counts(dtype, [e, 16, 16 * (n - 1) + e, FB_LL_MAX_BYTES + e, two_shot_bytes])
    multicast = g.comms[0].has_multicast
    for op in OPS_FOR[dtype]:
        for count in sizes:
            ins = make_inputs(rng, dtype, op, n, count)
            exp = fold(ins, dtype, op)
            for symmetric in (True, False):
                what = f"n={n} {dtype} {op} count={count} symmetric={symmetric}"
                sends = device_bufs(g, exp.nbytes, symmetric, fill=ins)
                for root in range(n):
                    outs = device_bufs(g, exp.nbytes, False)
                    run(g, lambda c, r, st: c.reduce(sends[r], outs[r], root=root, op=op, dtype=dtype))
                    if not multicast:
                        want = "twoshot" if exp.nbytes > 2 * CFG["oneShotMaxBytes"] else "oneshot"
                        assert g.comms[0].last_algo == want
                    assert_same(host(outs[root], dtype), exp, dtype, f"reduce root {root} {what}")
                    assert all(untouched(outs[r]) for r in range(n) if r != root), f"reduce wrote a non-root output {what}"
                outs = device_bufs(g, exp.nbytes, symmetric)
                run(g, lambda c, r, st: c.scan(sends[r], outs[r], op=op, dtype=dtype))
                for r in range(n):
                    assert_same(host(outs[r], dtype), fold(ins[: r + 1], dtype, op), dtype, f"scan rank {r} {what}")
                release(g, sends, outs)
    # reduce-scatter: every rank's slice is a whole number of 16-byte vectors
    for op in OPS_FOR[dtype]:
        for slice_bytes in (16, 16 * 7, pass_bytes(n) + 16):
            per = slice_bytes // e
            ins = make_inputs(rng, dtype, op, n, per * n)
            exp = fold(ins, dtype, op)
            for symmetric in (True, False):
                sends = device_bufs(g, exp.nbytes, symmetric, fill=ins)
                outs = device_bufs(g, slice_bytes, symmetric)
                run(g, lambda c, r, st: c.reduce_scatter(sends[r], outs[r], op=op, dtype=dtype))
                for r in range(n):
                    assert_same(host(outs[r], dtype), exp[r * per : (r + 1) * per], dtype, f"reduce_scatter n={n} {dtype} {op} rank {r} slice={slice_bytes}")
                release(g, sends, outs)


# ----------------------------------------------------------------- grouped ----
def group_sizes(dtype, n):
    """Mixed tensor sizes for one grouped launch: tails under 16 bytes,
    tensors smaller than one vector, ragged last chunks, tensors spanning
    several ranks' ownership ranges."""
    e = itemsize(dtype)
    chunk = 32 * (2 if n == 8 else 8 if n == 1 else 4) * 16  # fbGroupChunkVecs (launch_api.h), bytes
    sizes = [e, 15 // e * e, 16, 16 + e, 16 * (n - 1) + e, chunk - 16 + e, chunk + 48 + e, 3 * n * chunk + e, 5 * e]
    return [b // e for b in sizes if b >= e]


def grouped(g, ins_per_tensor, dtype, op, transient):
    sends = [[c.empty(x[r].nbytes, torch.uint8) for x in ins_per_tensor] for r, c in enumerate(g.comms)]
    recvs = [[c.empty(x[r].nbytes, torch.uint8) for x in ins_per_tensor] for r, c in enumerate(g.comms)]
    for r in range(g.size):
        for i, x in enumerate(ins_per_tensor):
            sends[r][i].copy_(_raw(x[r]))
            recvs[r][i].fill_(SENTINEL)
    if transient:
        run(g, lambda c, r, st: c.all_reduce_many(sends[r], recvs[r], op=op, dtype=dtype))
    else:
        plans = [c.prepare_group(sends[r], recvs[r], dtype=dtype) for r, c in enumerate(g.comms)]
        run(g, lambda c, r, st: c.all_reduce_group(plans[r], op=op))
        for p in plans:
            p.close()
    outs = [[host(t, dtype) for t in recvs[r]] for r in range(g.size)]
    for r, c in enumerate(g.comms):
        for t in sends[r] + recvs[r]:
            c.free(t)
    return outs


@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_grouped_every_op(n):
    g = group(n)
    rng = np.random.default_rng([200 + n])
    for dtype, op in SUPPORTED:
        ins = [make_inputs(rng, dtype, op, n, k) for k in group_sizes(dtype, n)]
        exps = [fold(x, dtype, op) for x in ins]
        for transient in (False, True):
            outs = grouped(g, ins, dtype, op, transient)
            for r in range(n):
                for i, exp in enumerate(exps):
                    assert_same(outs[r][i], exp, dtype, f"grouped n={n} {dtype} {op} tensor {i} ({exp.size}) rank {r} transient={transient}")


# ------------------------------------------------------- staging, alignment ----
@pytest.mark.parametrize("n", [2, 3, 4])
@pytest.mark.parametrize("dtype,op", [("i32", "sum"), ("f32", "sum"), ("bf16", "max")])
def test_messages_larger_than_the_staging_buffer(n, dtype, op):
    """Non-symmetric buffers go through the staging area in pieces of
    stageBytes: three pieces here, the last one with a tail."""
    g = group(n)
    e = itemsize(dtype)
    count = (2 * CFG["stageBytes"] + 48 + e) // e
    rng = np.random.default_rng([300 + n, len(dtype)])
    ins = make_inputs(rng, dtype, op, n, count)
    exp = fold(ins, dtype, op)
    sends = device_bufs(g, exp.nbytes, False, fill=ins)
    calls = [
        ("all_reduce oneshot", lambda c, r, o: c.all_reduce(sends[r], o, op=op, algo="oneshot", dtype=dtype)),
        ("all_reduce twoshot", lambda c, r, o: c.all_reduce(sends[r], o, op=op, algo="twoshot", dtype=dtype)),
        ("reduce", lambda c, r, o: c.reduce(sends[r], o, root=n - 1, op=op, dtype=dtype)),
        ("scan", lambda c, r, o: c.scan(sends[r], o, op=op, dtype=dtype)),
    ]
    for name, fn in calls:
        outs = device_bufs(g, exp.nbytes, False)
        for c in g.comms:
            c.stats(reset=True)
        run(g, lambda c, r, st: fn(c, r, outs[r]))
        assert all(c.stats()["launches"] == 3 for c in g.comms), name
        for r in range(n):
            if name == "scan":
                assert_same(host(outs[r], dtype), fold(ins[: r + 1], dtype, op), dtype, f"{name} rank {r}")
            elif name != "reduce" or r == n - 1:
                assert_same(host(outs[r], dtype), exp, dtype, f"{name} rank {r}")


@pytest.mark.parametrize("n", [2, 3, 4])
@pytest.mark.parametrize("dtype", ["i8", "u16", "f16", "bf16", "i32", "f32", "f64", "u64", "f32_i32", "i32_i32"])
def test_ranks_with_buffers_one_element_off_alignment(n, dtype):
    """Odd ranks pass local buffers that start one element past a 16-byte
    boundary (LL moves their bytes one by one, one-shot stages the output);
    even ranks pass aligned ones.  Results must not depend on it."""
    e = itemsize(dtype)
    shifts = [e if r % 2 else 0 for r in range(n)]
    rng = np.random.default_rng([400 + n, DTYPES.index(dtype)])
    op = OPS_FOR[dtype][2 if dtype not in PAIR_DTYPES else 0]  # sum, or maxloc
    for algo in ("ll", "oneshot"):
        g = ll_group(n) if algo == "ll" else group(n)
        if g is None:
            continue
        for count in counts(dtype, [e, 16 + e, 16 * 33 + e, FB_LL_MAX_BYTES - e]):
            ins = make_inputs(rng, dtype, op, n, count)
            exp = fold(ins, dtype, op)
            outs = allreduce(g, ins, dtype, op, algo, False, shifts)
            for r in range(n):
                assert_same(outs[r], exp, dtype, f"{algo} n={n} {dtype} count={count} rank {r} shift={shifts[r]}")


# ---------------------------------------------------- exhaustive 16-bit floats ----
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_every_16bit_pattern(dtype):
    """Rank 0 holds all 65,536 bit patterns, rank 1 a seeded permutation of them."""
    n = 2
    g = group(n)
    gl = ll_group(n)
    bits = np.arange(1 << 16, dtype=np.uint16)
    ins = [bits.view(NP_DTYPES[dtype]), np.random.default_rng(16).permutation(bits).view(NP_DTYPES[dtype])]
    piece = FB_LL_MAX_BYTES // 2
    for op in FLOAT_OPS:
        exp = fold(ins, dtype, op)
        for algo in ("oneshot", "twoshot"):
            for symmetric in (True, False):
                outs = allreduce(g, ins, dtype, op, algo, symmetric)
                for r in range(n):
                    assert_same(outs[r], exp, dtype, f"{dtype} {op} {algo} symmetric={symmetric} rank {r}")
        if gl is not None:
            for k in range(0, 1 << 16, piece):
                part = [x[k : k + piece] for x in ins]
                outs = allreduce(gl, part, dtype, op, "ll", False)
                for r in range(n):
                    assert_same(outs[r], exp[k : k + piece], dtype, f"{dtype} {op} ll piece {k} rank {r}")


# ------------------------------------------------------ high-precision check ----
# unit roundoff u = ulp(1) / 2: the error bound of round-to-nearest
UNIT_ROUNDOFF = {"f16": 2.0**-11, "bf16": 2.0**-8, "f32": 2.0**-24, "f64": 2.0**-53}


def as_f64(x, dtype):
    if dtype == "bf16":
        return (x.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    return x.astype(np.float64)


@pytest.mark.parametrize("n", [2, 3, 4, 8])
@pytest.mark.parametrize("dtype", FLOAT_DTYPES)
def test_float_sum_is_within_the_rounding_bound_of_the_exact_sum(n, dtype):
    """Keeps the oracle honest: a rank-order fold of n finite values whose
    partial sums stay normal is within (n-1) u sum|x| of the exact sum, with u
    the unit roundoff of round-to-nearest (a fold that rounds toward zero can
    miss by up to twice that)."""
    g = group(n)
    rng = np.random.default_rng([500 + n, FLOAT_DTYPES.index(dtype)])
    count = 4099
    ins = float_inputs(rng, dtype, n, count, narrow_only=True)
    outs = allreduce(g, ins, dtype, "sum", "oneshot", True)
    assert_same(outs[0], fold(ins, dtype, "sum"), dtype, "oneshot sum")
    xs = [as_f64(x, dtype) for x in ins]
    exact = np.array([math.fsum(col) for col in zip(*xs)])
    bound = (n - 1) * UNIT_ROUNDOFF[dtype] * np.sum(np.abs(np.stack(xs)), axis=0)
    err = np.abs(as_f64(outs[0], dtype) - exact)
    assert np.all(err <= bound), f"worst excess {np.max(err - bound)}"


# ------------------------------------------------------------ NaN placement ----
def nan_of(dtype, negative=False):
    if dtype == "bf16":
        return np.uint16(0xFFC0 if negative else 0x7FC0)
    v = NP_DTYPES[dtype].type(np.nan)
    return -v if negative else v


@pytest.mark.parametrize("n", [2, 3, 4, 8])
@pytest.mark.parametrize("dtype", FLOAT_DTYPES)
def test_nan_on_one_rank_or_on_every_rank_max_min(n, dtype):
    """MPI MAX/MIN are commutative: where a NaN sits must not change the
    result.  Position p holds a NaN on rank (p + shift) % (n + 1), or on every
    rank where that is n.  The message has full vectors and a < 16-byte tail,
    and the pattern is rotated through every shift, so the vector path and the
    scalar tail (whose last element gets every placement) both see each one."""
    g = group(n)
    gl = ll_group(n)
    rng = np.random.default_rng([600 + n, FLOAT_DTYPES.index(dtype)])
    e = itemsize(dtype)
    count = (n + 1) * 7
    if (count * e) % 16 == 0:
        count += 1
    for shift in range(n + 1):
        check_nan_placement(g, gl, rng, n, dtype, count, shift)


def check_nan_placement(g, gl, rng, n, dtype, count, shift):
    ins = float_inputs(rng, dtype, n, count, narrow_only=True)
    where = (np.arange(count) + shift) % (n + 1)
    for r in range(n):
        hit = (where == r) | (where == n)
        ins[r][hit] = nan_of(dtype, negative=bool(r % 2))
    all_nan = where == n
    for op in ("max", "min"):
        exp = fold(ins, dtype, op)
        nan_exp = (exp & 0x7FFF) > 0x7F80 if dtype == "bf16" else np.isnan(exp)
        assert np.array_equal(nan_exp, all_nan)
        results = []
        for algo in ALGOS:
            grp = gl if algo == "ll" else g
            if grp is None:
                continue
            for symmetric in (True, False):
                outs = allreduce(grp, ins, dtype, op, algo, symmetric)
                results += [(f"{algo} symmetric={symmetric} rank {r}", o) for r, o in enumerate(outs)]
        for transient in (False, True):
            outs = grouped(g, [ins], dtype, op, transient)
            results += [(f"grouped transient={transient} rank {r}", o[0]) for r, o in enumerate(outs)]
        for what, got in results:
            assert_same(got, exp, dtype, f"n={n} {dtype} {op} shift={shift} {what}")
