"""Device snapshot kernels against ``snapshot_oracle`` bit for bit: every
(data type x merge op) at every scalar placement, with dirty hints, both fill
modes, base updates, concurrent writers, diff application, dirty scans and
chunk runs, and the checks the wrappers make before any launch."""

import numpy as np
import pytest
import torch

import snapshot_oracle as so
from faabric_b200.ops import snapshot as snap

pytestmark = pytest.mark.gpu

PAGE = so.PAGE
TYPES = [so.INT, so.LONG, so.FLOAT, so.DOUBLE]
OPS = [so.SUM, so.SUBTRACT, so.PRODUCT, so.MAX, so.MIN]
TYPE_NAMES = {so.INT: "int", so.LONG: "long", so.FLOAT: "float", so.DOUBLE: "double"}
OP_NAMES = {so.SUM: "sum", so.SUBTRACT: "sub", so.PRODUCT: "prod", so.MAX: "max", so.MIN: "min"}

F32_BITS = [0x7FC00000, 0x7FC00001, 0xFFC12345, 0x7F800001,  # NaNs (quiet, payload, negative, signalling)
            0x00000000, 0x80000000, 0x7F800000, 0xFF800000,  # ±0, ±inf
            0x00000001, 0x80000001, 0x007FFFFF, 0x00800000,  # subnormals, smallest normal
            0x7F7FFFFF, 0xFF7FFFFF, 0x3F800000, 0x3F800001,  # largest finite, 1, 1 + ulp
            0x33800000, 0x40400000, 0xBF800000, 0x3DCCCCCD]  # 2^-24 (rounds against 1), 3, -1, 0.1
F64_BITS = [0x7FF8000000000000, 0x7FF8000000000001, 0xFFF8DEADBEEF0000, 0x7FF0000000000001,
            0x0000000000000000, 0x8000000000000000, 0x7FF0000000000000, 0xFFF0000000000000,
            0x0000000000000001, 0x8000000000000001, 0x000FFFFFFFFFFFFF, 0x0010000000000000,
            0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF, 0x3FF0000000000000, 0x3FF0000000000001,
            0x3CA0000000000000, 0x4008000000000000, 0xBFF0000000000000, 0x3FB999999999999A]


def pool(dt):
    if dt == so.INT:
        return np.array([-(2**31), 2**31 - 1, -1, 0, 1, 2, -2, 7, -(2**30), 123456], np.int32).view(np.uint8).reshape(-1, 4)
    if dt == so.LONG:
        return np.array([-(2**63), 2**63 - 1, -1, 0, 1, 2, -2, 7, 2**40, -(2**62)], np.int64).view(np.uint8).reshape(-1, 8)
    if dt == so.FLOAT:
        return np.array(F32_BITS, np.uint32).view(np.uint8).reshape(-1, 4)
    return np.array(F64_BITS, np.uint64).view(np.uint8).reshape(-1, 8)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


def put(buf, off, raw):
    buf[off : off + len(raw)] = raw


def build_case(dt, op, size, rng):
    """Images and regions with scalars of type dt at every placement, an
    array, an Ignore region and byte edits next to the scalars."""
    sz = 4 if dt in (so.INT, so.FLOAT) else 8
    orig = rng.integers(0, 256, size, dtype=np.uint8)
    mem = orig.copy()
    main = orig.copy()
    vals = pool(dt)
    regions = []

    def scalar(off, n=1, length=None):
        regions.append(so.Region(off, n * sz if length is None else length, dt, op))
        for k in range(n):
            o = off + k * sz
            if o + sz > size:
                # the part of a scalar that does not fit still changes
                mem[o:size] ^= 0xA5
                continue
            a, b, c = (vals[i] for i in rng.integers(0, len(vals), 3))
            if rng.random() < 0.2:
                b = a  # unchanged
            put(orig, o, a), put(mem, o, b), put(main, o, c)

    # byte edits all over, including the first and last byte; the typed
    # scalars below overwrite whatever lands on them
    idx = rng.integers(0, size, 300)
    mem[idx] ^= rng.integers(1, 256, len(idx), dtype=np.uint8)
    mem[0] ^= 1
    mem[-1] ^= 2
    placements = [
        64,                          # naturally aligned
        256 + (3 if sz == 4 else 5),  # unaligned inside a 16-byte block
        512 + 14,                    # across a 16-byte boundary
        2 * PAGE - 2,                # across a page
        PAGE + 1024 + 7,             # odd offset, shares its block with byte edits
    ]
    for off in placements:
        scalar(off)
    blk = PAGE + 1024
    mem[blk + 1] ^= 0x11  # bytewise edits in the same 16-byte vector as a scalar
    mem[blk + 7 + sz] ^= 0x22
    scalar(3 * PAGE - 5 * sz, n=11, length=11 * sz + 3)  # an array across a page, with trailing bytes
    regions.append(so.Region(5 * PAGE + 100, 300, so.RAW, so.IGNORE))
    mem[5 * PAGE + 100 : 5 * PAGE + 400] ^= 0x3C
    # at the image end: the last whole scalar, or one that does not fit
    if size % 16 == 0:
        scalar(size - sz)
    else:
        scalar(size - sz - 3, length=sz + 3)  # one whole scalar, 3 bytes left over
    return orig, mem, main, regions


def dirty_modes(size, rng):
    n = (size + PAGE - 1) // PAGE
    rand = (rng.random(n) < 0.5).astype(np.uint8)
    first = np.zeros(n, np.uint8)  # only the first page of the straddling scalar at 2 * PAGE - 2
    first[1] = 1
    second = np.zeros(n, np.uint8)
    second[2] = 1
    return [("all", None), ("none", np.zeros(n, np.uint8)), ("random", rand), ("first", first), ("second", second)]


def check(res, d_main, d_orig, page_flags, chunk_flags, stats, update_base, orig):
    got = host(d_main)
    bad = so.mismatches(got, res.main, res.nan_spans)
    assert len(bad) == 0, f"main differs at {bad[:10].tolist()}: {got[bad[:10]].tolist()} want {res.main[bad[:10]].tolist()}"
    want_base = res.base if update_base else orig
    assert np.array_equal(host(d_orig), want_base), np.nonzero(host(d_orig) != want_base)[0][:10]
    assert np.array_equal(host(page_flags).astype(bool), res.page_flags)
    assert set(np.nonzero(host(chunk_flags))[0].tolist()) == res.chunks
    assert host(stats).tolist() == [res.diff_bytes, res.pages_with_diffs]


@pytest.mark.parametrize("size", [33 * PAGE + 777, 8 * PAGE], ids=["ragged", "pages"])
@pytest.mark.parametrize("fill", [so.BYTEWISE, so.XOR], ids=["bytewise", "xor"])
@pytest.mark.parametrize("op", OPS, ids=lambda o: OP_NAMES[o])
@pytest.mark.parametrize("dt", TYPES, ids=lambda t: TYPE_NAMES[t])
def test_diff_push_matrix(dt, op, fill, size):
    rng = np.random.default_rng([dt, op, fill, size])
    orig, mem, main, regions = build_case(dt, op, size, rng)
    regs = snap.prepare_regions([snap.MergeRegion(r.offset, r.length, r.data_type, r.op) for r in regions], size, "cuda", fill_op=fill)
    filled = so.fill_gaps(regions, size, fill)
    assert [(r.offset, r.length, r.data_type, r.op) for r in regs.host] == [(r.offset, r.length, r.data_type, r.op) for r in filled]
    n_pages = (size + PAGE - 1) // PAGE
    d_mem = dev(mem)
    for i, (name, dirty) in enumerate(dirty_modes(size, rng)):
        update_base = i % 2 == 0
        res = so.merge(orig, mem, main, filled, dirty, update_base)
        outs = []
        for blocks in (0, 1):  # the default grid, and one CTA walking every grid-stride loop
            d_orig, d_main = dev(orig), dev(main)
            page_flags = torch.zeros(n_pages, dtype=torch.uint8, device="cuda")
            chunk_flags = torch.zeros((size + 127) // 128, dtype=torch.uint8, device="cuda")
            stats = snap.diff_push(d_mem, d_orig, d_main, regs, dirty_pages=None if dirty is None else dev(dirty),
                                   update_base=update_base, page_flags_out=page_flags, chunk_flags=chunk_flags, blocks=blocks)
            torch.cuda.synchronize()
            check(res, d_main, d_orig, page_flags, chunk_flags, stats, update_base, orig)
            outs.append(host(d_main))
        assert np.array_equal(outs[0], outs[1]), name
        if update_base and dirty is None:
            # the base now holds the memory outside Ignore regions: a second
            # pass only finds the NaN scalars again (NaN != NaN)
            again = so.merge(res.base, mem, res.main, filled)
            stats = snap.diff_push(d_mem, d_orig, d_main, regs)
            torch.cuda.synchronize()
            assert int(stats[0]) == again.diff_bytes


@pytest.mark.parametrize("size", [1, 4095, PAGE, 33 * PAGE + 777, 16 * 2**20 + 5])
@pytest.mark.parametrize("fill", [so.BYTEWISE, so.XOR], ids=["bytewise", "xor"])
def test_diff_push_sizes(size, fill):
    """Byte regions at ragged sizes, with a typed array over the whole tail."""
    rng = np.random.default_rng([size, fill])
    orig = rng.integers(0, 256, size, dtype=np.uint8)
    mem = orig.copy()
    k = max(1, size // 997)
    idx = rng.integers(0, size, k)
    mem[idx] ^= 0x5A
    mem[-1] ^= 0x80
    if size >= PAGE * 4:
        mem[PAGE * 2 : PAGE * 3] = rng.integers(0, 256, PAGE, dtype=np.uint8)
    regions = []
    if size > 64:
        tail = size - (size // 3)
        regions = [so.Region(tail, 0, so.FLOAT, so.SUM)]
        t = np.arange(tail, size - 3, 4)
        vals = rng.integers(-1000, 1000, len(t)).astype(np.float32) / 8
        for o, v in zip(t[::7], vals[::7]):
            mem[o : o + 4] = np.array([v], np.float32).view(np.uint8)
    main = orig.copy()
    main[rng.integers(0, size, k)] ^= 0xFF  # another writer already changed main
    regs = snap.prepare_regions([snap.MergeRegion(r.offset, r.length, r.data_type, r.op) for r in regions], size, "cuda", fill_op=fill)
    filled = so.fill_gaps(regions, size, fill)
    res = so.merge(orig, mem, main, filled)
    d_orig, d_main = dev(orig), dev(main)
    n_pages = (size + PAGE - 1) // PAGE
    page_flags = torch.zeros(n_pages, dtype=torch.uint8, device="cuda")
    chunk_flags = torch.zeros((size + 127) // 128, dtype=torch.uint8, device="cuda")
    stats = snap.diff_push(dev(mem), d_orig, d_main, regs, page_flags_out=page_flags, chunk_flags=chunk_flags)
    torch.cuda.synchronize()
    check(res, d_main, d_orig, page_flags, chunk_flags, stats, False, orig)
    # the runs derived from the chunk flags cover every diffed byte
    covered = np.zeros(size, dtype=bool)
    for off, ln in snap.chunk_runs(chunk_flags, size):
        covered[off : off + ln] = True
    assert all(covered[c * 128 : min(size, c * 128 + 128)].all() for c in res.chunks)


def test_dirty_page_hint_skips_clean_pages():
    size = PAGE * 16
    rng = np.random.default_rng(1)
    orig = rng.integers(0, 256, size, dtype=np.uint8)
    mem = orig.copy()
    mem[PAGE * 3 + 5] ^= 1
    mem[PAGE * 9 + 100] ^= 1  # changed but not flagged dirty: ignored
    dirty = np.zeros(16, dtype=np.uint8)
    dirty[3] = 1
    regs = snap.prepare_regions([], size, "cuda")
    d_main = dev(orig)
    stats = snap.diff_push(dev(mem), dev(orig), d_main, regs, dirty_pages=dev(dirty))
    torch.cuda.synchronize()
    res = so.merge(orig, mem, orig, so.fill_gaps([], size), dirty)
    assert np.array_equal(host(d_main), res.main)
    assert int(stats[0]) == res.diff_bytes == 1


# ---------------------------------------------------------- concurrency ----
def _concurrent(dt, op, values, n_main):
    """len(values) - 1 writers push into one main image at once; values[0] is
    the base.  Returns the merged scalars (one per 16-byte block slot)."""
    sz = 4 if dt in (so.INT, so.FLOAT) else 8
    t = so.NP_TYPES[dt]
    size = PAGE * 2
    offs = [64 + 3, 512 + 8, 1024 + 16 - sz]  # unaligned, aligned, block end: each inside one 16-byte block
    orig = np.zeros(size, np.uint8)
    for o in offs:
        orig[o : o + sz] = np.array([values[0]], t).view(np.uint8)
    main = orig.copy()
    for o in offs:
        main[o : o + sz] = np.array([n_main], t).view(np.uint8)
    regs = snap.prepare_regions([snap.MergeRegion(o, sz, dt, op) for o in offs], size, "cuda")
    filled = so.fill_gaps([so.Region(o, sz, dt, op) for o in offs], size)
    mems = []
    for v in values[1:]:
        m = orig.copy()
        for o in offs:
            m[o : o + sz] = np.array([v], t).view(np.uint8)
        mems.append(m)
    exp = main
    nan_spans = []
    for m in mems:  # any order gives the same bits for these operations
        r = so.merge(orig, m, exp, filled)
        exp, nan_spans = r.main, r.nan_spans
    d_mems = [dev(m) for m in mems]
    d_orig = dev(orig)
    streams = [torch.cuda.Stream() for _ in mems]
    for rep in range(3):
        d_main = dev(main)
        torch.cuda.synchronize()
        order = range(len(mems)) if rep % 2 == 0 else reversed(range(len(mems)))
        for w in order:
            with torch.cuda.stream(streams[w]):
                snap.diff_push(d_mems[w], d_orig, d_main, regs)
        torch.cuda.synchronize()
        bad = so.mismatches(host(d_main), exp, nan_spans)
        assert len(bad) == 0, (rep, bad[:8].tolist())


@pytest.mark.parametrize("aligned", [True, False], ids=["aligned", "unaligned"])
@pytest.mark.parametrize("dt", [so.FLOAT, so.DOUBLE], ids=["float", "double"])
def test_subnormal_sums_are_kept(dt, aligned):
    """Float sums keep subnormal operands and results on every path, the
    aligned double one (a hardware red.add.f64) included."""
    t = so.NP_TYPES[dt]
    sz = np.dtype(t).itemsize
    tiny = np.array([1], np.uint32 if sz == 4 else np.uint64).view(t)[0]
    size = PAGE
    rows = [(0.0, tiny, tiny), (0.0, tiny, -tiny * 3), (tiny * 5, tiny, tiny * 2), (1.0, 1.0 + tiny, 0.0)]
    regions, orig, mem, main = [], np.zeros(size, np.uint8), np.zeros(size, np.uint8), np.zeros(size, np.uint8)
    for i, (o, m, c) in enumerate(rows):
        for j, op in enumerate((so.SUM, so.SUBTRACT)):
            off = 64 * (2 * i + j) + (0 if aligned else 3)
            regions.append(so.Region(off, sz, dt, op))
            for buf, v in ((orig, o), (mem, m), (main, c)):
                buf[off : off + sz] = np.array([v], t).view(np.uint8)
    regs = snap.prepare_regions([snap.MergeRegion(r.offset, r.length, r.data_type, r.op) for r in regions], size, "cuda")
    res = so.merge(orig, mem, main, so.fill_gaps(regions, size))
    d_main = dev(main)
    snap.diff_push(dev(mem), dev(orig), d_main, regs)
    torch.cuda.synchronize()
    got = host(d_main)
    assert np.array_equal(got, res.main)
    first = 0 if aligned else 3
    assert got[first : first + sz].view(t)[0] == 2 * tiny  # tiny + (tiny - 0), not flushed to 0


@pytest.mark.parametrize("dt", [so.INT, so.LONG], ids=["int", "long"])
@pytest.mark.parametrize("op", OPS, ids=lambda o: OP_NAMES[o])
def test_concurrent_integer_writers(dt, op):
    big = 2**31 - 7 if dt == so.INT else 2**63 - 7
    if op == so.PRODUCT:
        values = [3, 6, -9, 3 * big // 3, 12, 0]  # quotients 2, -3, big // 3, 4, 0
    else:
        values = [5, big, -big, 6, -1, 1 << 20, 0]
    _concurrent(dt, op, values, n_main=big - 3)


@pytest.mark.parametrize("dt", [so.FLOAT, so.DOUBLE], ids=["float", "double"])
@pytest.mark.parametrize("op", [so.MAX, so.MIN], ids=["max", "min"])
@pytest.mark.parametrize("main_val", [0.0, -0.0, float("nan"), 1.0])
def test_concurrent_float_max_min_nan_and_signed_zero(dt, op, main_val):
    _concurrent(dt, op, [2.0, float("nan"), -0.0, 0.0, float("nan"), -0.0, 0.0], n_main=main_val)


@pytest.mark.parametrize("dt", [so.FLOAT, so.DOUBLE], ids=["float", "double"])
@pytest.mark.parametrize("op", [so.SUM, so.SUBTRACT])
def test_concurrent_float_sums_that_are_exact(dt, op):
    _concurrent(dt, op, [1.0, 1.5, 0.25, 3.0, -2.0, 1.125, 8.0], n_main=100.0)


def test_concurrent_xor_and_disjoint_bytewise_writers():
    size = PAGE * 64
    rng = np.random.default_rng(11)
    orig = rng.integers(0, 256, size, dtype=np.uint8)
    for fill in (so.BYTEWISE, so.XOR):
        mems = [orig.copy() for _ in range(4)]
        for w in range(4):
            if fill == so.BYTEWISE:  # interleaved single bytes inside the same 16-byte vectors
                mems[w][1000 + w : size - 16 : 37] ^= 0x0F << (w % 2 * 4)
            else:  # xor writers may hit the same bytes
                mems[w][rng.integers(0, size, 5000)] ^= rng.integers(1, 256, 5000, dtype=np.uint8)
        regs = snap.prepare_regions([], size, "cuda", fill_op=fill)
        filled = so.fill_gaps([], size, fill)
        exp = orig
        for m in mems:
            exp = so.merge(orig, m, exp, filled).main
        d_main, d_orig = dev(orig), dev(orig)
        d_mems = [dev(m) for m in mems]
        streams = [torch.cuda.Stream() for _ in mems]
        torch.cuda.synchronize()
        for w in range(4):
            with torch.cuda.stream(streams[w]):
                snap.diff_push(d_mems[w], d_orig, d_main, regs)
        torch.cuda.synchronize()
        assert np.array_equal(host(d_main), exp)


def test_concurrent_writers_merge_unaligned_typed_regions():
    """Typed regions at odd offsets of their 16-byte blocks: eight writers
    add into the same scalars at once; the 128-bit CAS keeps every one."""
    size = PAGE * 4
    orig = np.zeros(size, dtype=np.uint8)
    offs = {"int": 64 + 6, "long": 256 + 3, "double": 1024 + 5}
    orig[offs["int"] : offs["int"] + 4] = np.array([1000], dtype=np.int32).view(np.uint8)
    orig[offs["long"] : offs["long"] + 8] = np.array([1 << 40], dtype=np.int64).view(np.uint8)
    orig[offs["double"] : offs["double"] + 8] = np.array([2.5], dtype=np.float64).view(np.uint8)
    regs = snap.prepare_regions(
        [snap.MergeRegion(offs["int"], 4, snap.INT, snap.SUM), snap.MergeRegion(offs["long"], 8, snap.LONG, snap.SUM),
         snap.MergeRegion(offs["double"], 8, snap.DOUBLE, snap.SUM)], size, "cuda")
    n_writers = 8
    d_orig = dev(orig)
    d_mems = []
    for w in range(n_writers):
        m = orig.copy()
        m[offs["int"] : offs["int"] + 4] = np.array([1000 + (w + 1)], dtype=np.int32).view(np.uint8)
        m[offs["long"] : offs["long"] + 8] = np.array([(1 << 40) + 10 * (w + 1)], dtype=np.int64).view(np.uint8)
        m[offs["double"] : offs["double"] + 8] = np.array([2.5 + 0.25 * (w + 1)], dtype=np.float64).view(np.uint8)
        d_mems.append(dev(m))
    streams = [torch.cuda.Stream() for _ in range(n_writers)]
    for rep in range(3):
        d_main = dev(orig)
        torch.cuda.synchronize()
        for w in range(n_writers):
            with torch.cuda.stream(streams[w]):
                snap.diff_push(d_mems[w], d_orig, d_main, regs)
        torch.cuda.synchronize()
        got = host(d_main)
        tot = n_writers * (n_writers + 1) // 2
        assert int(got[offs["int"] : offs["int"] + 4].view(np.int32)[0]) == 1000 + tot
        assert int(got[offs["long"] : offs["long"] + 8].view(np.int64)[0]) == (1 << 40) + 10 * tot
        assert float(got[offs["double"] : offs["double"] + 8].view(np.float64)[0]) == 2.5 + 0.25 * tot
        untouched = np.ones(size, dtype=bool)
        for k, ln in (("int", 4), ("long", 8), ("double", 8)):
            untouched[offs[k] : offs[k] + ln] = False
        assert not got[untouched].any()


# -------------------------------------------------------------- apply ----
@pytest.mark.parametrize("op", OPS, ids=lambda o: OP_NAMES[o])
@pytest.mark.parametrize("dt", TYPES, ids=lambda t: TYPE_NAMES[t])
def test_apply_diffs_matrix(dt, op):
    rng = np.random.default_rng([dt, op, 7])
    sz = 4 if dt in (so.INT, so.FLOAT) else 8
    size = 3 * PAGE + 5
    vals = pool(dt)
    img = rng.integers(0, 256, size, dtype=np.uint8)
    diffs = []
    for off in (64, 256 + 3, 512 + 14, PAGE - 2):
        put(img, off, vals[rng.integers(len(vals))])
        diffs.append((off, dt, op, vals[rng.integers(len(vals))].tobytes()))
    # every pool value against every other as an array diff, with 3 trailing bytes
    n = len(vals)
    arr_off = PAGE + 100
    cur = np.repeat(np.arange(n), n)
    val = np.tile(np.arange(n), n)
    img[arr_off : arr_off + n * n * sz] = vals[cur].reshape(-1)
    diffs.append((arr_off, dt, op, vals[val].tobytes() + b"\x01\x02\x03"))
    # a diff that passes the image end: only its whole scalars inside are applied
    diffs.append((size - sz - 1, dt, op, vals[:2].tobytes()))
    diffs += [(10, so.RAW, so.BYTEWISE, bytes([1, 2, 3])), (50, so.RAW, so.XOR, bytes([0xFF, 0x0F])),
              (40, so.RAW, so.IGNORE, bytes([9, 9]))]
    exp, nan_spans = so.apply(img, diffs)
    d_img = dev(img)
    snap.apply_diffs(d_img, diffs)
    torch.cuda.synchronize()
    bad = so.mismatches(host(d_img), exp, nan_spans)
    assert len(bad) == 0, bad[:10].tolist()


# ------------------------------------------------- dirty scan and runs ----
@pytest.mark.parametrize("size", [1, 15, 4095, PAGE, PAGE + 1, 40 * PAGE + 100])
@pytest.mark.parametrize("where", ["first", "last", "tail_page", "none"])
def test_dirty_scan_ragged(size, where):
    rng = np.random.default_rng(size)
    base = rng.integers(0, 256, size, dtype=np.uint8)
    mem = base.copy()
    pos = {"first": 0, "last": size - 1, "tail_page": (size - 1) // PAGE * PAGE + (size % PAGE) // 2, "none": None}[where]
    if pos is not None:
        mem[pos] ^= 1
    flags, count = snap.dirty_scan(dev(mem), dev(base))
    torch.cuda.synchronize()
    n_pages = (size + PAGE - 1) // PAGE
    exp = np.zeros(n_pages, np.uint8)
    if pos is not None:
        exp[pos // PAGE] = 1
    assert host(flags).tolist() == exp.tolist()
    assert int(count) == int(exp.sum())
    other = torch.zeros_like(flags)
    other[-1] = 1
    snap.flags_or(flags, other)
    torch.cuda.synchronize()
    exp[-1] = 1
    assert host(flags).tolist() == exp.tolist()


def test_chunk_runs_at_maximum_fragmentation():
    n = 10_001
    flags = torch.zeros(n, dtype=torch.uint8, device="cuda")
    flags[::2] = 1
    total = n * 128 - 50  # the last run is cut at the end
    runs = snap.chunk_runs(flags, total)
    assert len(runs) == (n + 1) // 2
    assert runs[:2] == [(0, 128), (256, 128)]
    assert runs[-1] == ((n - 1) * 128, 78)
    assert all(off == 256 * i for i, (off, _) in enumerate(runs))
    with pytest.raises(RuntimeError):
        snap.chunk_runs(flags, total, max_out=len(runs) - 1)
    assert snap.chunk_runs(flags, total, max_out=len(runs)) == runs


# ------------------------------------------------ checks before launch ----
def test_wrappers_reject_misaligned_and_short_tensors():
    size = PAGE * 4
    buf = torch.zeros(size + 64, dtype=torch.uint8, device="cuda")
    mem, orig, dst = buf[16 : 16 + size], torch.zeros(size, dtype=torch.uint8, device="cuda"), torch.zeros(size, dtype=torch.uint8, device="cuda")
    regs = snap.prepare_regions([], size, "cuda")
    mis = buf[1 : 1 + size]
    launches = torch.zeros(2, dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError):
        snap.diff_push(mis, orig, dst, regs, stats=launches)
    with pytest.raises(ValueError):
        snap.diff_push(mem, mis, dst, regs, stats=launches)
    with pytest.raises(ValueError):
        snap.diff_push(mem, orig, mis, regs, stats=launches)
    with pytest.raises(ValueError):
        snap.diff_push(mem, orig, dst.data_ptr() + 4, regs, stats=launches)
    with pytest.raises(ValueError):
        snap.diff_push(mem, orig, dst[: size - 1], regs, stats=launches)
    short = torch.zeros(3, dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError):
        snap.diff_push(mem, orig, dst, regs, dirty_pages=short, stats=launches)
    with pytest.raises(ValueError):
        snap.diff_push(mem, orig, dst, regs, page_flags_out=short, stats=launches)
    with pytest.raises(ValueError):
        snap.diff_push(mem, orig, dst, regs, chunk_flags=torch.zeros(size // 128 - 1, dtype=torch.uint8, device="cuda"), stats=launches)
    with pytest.raises(ValueError):
        snap.dirty_scan(mis, orig)
    with pytest.raises(ValueError):
        snap.dirty_scan(mem, mis)
    torch.cuda.synchronize()
    assert host(launches).tolist() == [0, 0]
    # the aligned call goes through
    mem.fill_(3)
    stats = snap.diff_push(mem, orig, dst, regs, stats=launches)
    torch.cuda.synchronize()
    assert host(stats).tolist() == [size, 4]


def test_prepare_regions_rejects_overlap():
    with pytest.raises(ValueError):
        snap.prepare_regions([snap.MergeRegion(0, 8, snap.LONG, snap.SUM), snap.MergeRegion(4, 4, snap.INT, snap.SUM)], 100, "cuda")
    with pytest.raises(ValueError):
        snap.prepare_regions([snap.MergeRegion(8, 0, snap.RAW, snap.IGNORE), snap.MergeRegion(64, 4, snap.INT, snap.SUM)], 100, "cuda")
