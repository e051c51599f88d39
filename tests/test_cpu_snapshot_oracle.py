"""The snapshot merge oracle against hand-computed cases (no GPU)."""

import struct

import numpy as np
import pytest

import snapshot_oracle as so

I32_MIN, I32_MAX = -(2**31), 2**31 - 1
I64_MIN, I64_MAX = -(2**63), 2**63 - 1
FMT = {so.INT: "<i", so.LONG: "<q", so.FLOAT: "<f", so.DOUBLE: "<d"}


def one(dt, op, old, new, cur, off=64, size=4096):
    """Merge one scalar that went old -> new into a main image holding cur;
    returns the merged value and the oracle result."""
    fmt = FMT[dt]
    sz = struct.calcsize(fmt)
    orig = np.zeros(size, np.uint8)
    mem = orig.copy()
    main = orig.copy()
    orig[off : off + sz] = np.frombuffer(struct.pack(fmt, old), np.uint8)
    mem[off : off + sz] = np.frombuffer(struct.pack(fmt, new), np.uint8)
    main[off : off + sz] = np.frombuffer(struct.pack(fmt, cur), np.uint8)
    regions = so.fill_gaps([so.Region(off, sz, dt, op)], size)
    res = so.merge(orig, mem, main, regions, update_base=True)
    return struct.unpack(fmt, res.main[off : off + sz].tobytes())[0], res


def bits(x, fmt):
    return struct.pack(fmt, x)


@pytest.mark.parametrize(
    "dt,op,old,new,cur,want",
    [
        # int32 wrap: delta new - old overflows, the sum wraps
        (so.INT, so.SUM, I32_MIN, I32_MAX, 5, 5 + (2**32 - 1) - 2**32),
        (so.INT, so.SUM, 0, 1, I32_MAX, I32_MIN),
        (so.INT, so.SUBTRACT, 1, 0, I32_MIN, I32_MAX),  # main -= old - new
        (so.INT, so.SUBTRACT, I32_MAX, I32_MIN, 0, 1),  # old - new wraps to -1
        (so.INT, so.PRODUCT, 1, 2, 2**30, I32_MIN),
        (so.INT, so.PRODUCT, 1, 3, I32_MAX, 2147483645),
        # int64 wrap
        (so.LONG, so.SUM, 0, 1, I64_MAX, I64_MIN),
        (so.LONG, so.SUBTRACT, 1, 0, I64_MIN, I64_MAX),
        (so.LONG, so.PRODUCT, 1, 2, 2**62, I64_MIN),
        # product quotient: old == 0 gives 0, MIN / -1 wraps, truncation toward 0
        (so.INT, so.PRODUCT, 0, 7, 9, 0),
        (so.LONG, so.PRODUCT, 0, -7, 9, 0),
        (so.INT, so.PRODUCT, -1, I32_MIN, 3, I32_MIN),  # q = MIN / -1 = MIN
        (so.LONG, so.PRODUCT, -1, I64_MIN, 1, I64_MIN),
        (so.INT, so.PRODUCT, 2, -7, 10, -30),  # -7 / 2 = -3
        (so.INT, so.PRODUCT, -2, 7, 10, -30),
        # integer max / min
        (so.INT, so.MAX, 0, -1, I32_MIN, -1),
        (so.LONG, so.MIN, 0, I64_MAX, 5, 5),
    ],
)
def test_integer_rules(dt, op, old, new, cur, want):
    got, res = one(dt, op, old, new, cur)
    assert got == want
    assert res.diff_bytes == struct.calcsize(FMT[dt])


@pytest.mark.parametrize("dt", [so.FLOAT, so.DOUBLE])
def test_float_product_with_zero_original(dt):
    fmt = FMT[dt]
    got, _ = one(dt, so.PRODUCT, 0.0, 3.0, 2.0)
    assert got == float("inf")
    got, _ = one(dt, so.PRODUCT, 0.0, -3.0, 2.0)
    assert got == float("-inf")
    got, _ = one(dt, so.PRODUCT, -0.0, 3.0, 2.0)
    assert got == float("-inf")
    # 0 * inf is NaN
    got, res = one(dt, so.PRODUCT, 0.0, 3.0, 0.0)
    assert got != got and len(res.nan_spans) == 1
    # from 0 to -0 is no change
    got, res = one(dt, so.PRODUCT, 0.0, -0.0, 2.0)
    assert bits(got, fmt) == bits(2.0, fmt) and res.diff_bytes == 0


@pytest.mark.parametrize("dt", [so.FLOAT, so.DOUBLE])
@pytest.mark.parametrize("op", [so.MAX, so.MIN])
def test_nan_and_signed_zero_in_both_orders(dt, op):
    fmt = FMT[dt]
    nan = float("nan")
    # a NaN in the new value is a change, and is ignored by the merge
    got, res = one(dt, op, 1.0, nan, 2.0)
    assert res.diff_bytes == struct.calcsize(fmt) and got == 2.0
    # a NaN already in main is replaced
    got, _ = one(dt, op, 1.0, 3.0, nan)
    assert got == 3.0
    # NaN in both stays NaN
    got, res = one(dt, op, 1.0, nan, nan)
    assert got != got and res.nan_spans
    # a NaN in the original: NaN != x, so x is merged
    got, res = one(dt, op, nan, 5.0, 4.0)
    assert res.diff_bytes > 0 and got == (5.0 if op == so.MAX else 4.0)
    # NaN -> NaN (same payload) still counts as a change
    _, res = one(dt, op, nan, nan, 4.0)
    assert res.diff_bytes > 0
    # ±0: max gives +0 and min gives -0 whichever side holds which
    want = 0.0 if op == so.MAX else -0.0
    got, _ = one(dt, op, 1.0, 0.0, -0.0)
    assert bits(got, fmt) == bits(want, fmt)
    got, _ = one(dt, op, 1.0, -0.0, 0.0)
    assert bits(got, fmt) == bits(want, fmt)
    # +0 -> -0 is no change
    got, res = one(dt, op, 0.0, -0.0, 7.0)
    assert res.diff_bytes == 0 and got == 7.0
    # a signalling NaN is ignored like a quiet one, new or in main
    snan = struct.unpack(fmt, struct.pack("<I", 0x7F800001) if dt == so.FLOAT else struct.pack("<Q", 0x7FF0000000000001))[0]
    got, res = one(dt, op, 1.0, snan, 2.0)
    assert got == 2.0 and not res.nan_spans


def test_f32_subnormal_deltas():
    tiny = np.float32(1.4e-45)  # smallest subnormal
    got, _ = one(so.FLOAT, so.SUM, 0.0, float(tiny), float(tiny))
    assert np.float32(got) == np.float32(2 * tiny)
    got, _ = one(so.FLOAT, so.SUBTRACT, float(3 * tiny), float(tiny), float(5 * tiny))
    assert np.float32(got) == np.float32(3 * tiny)
    # a rounding sum: 1 + 2^-24 rounds to 1 (ties to even)
    got, _ = one(so.FLOAT, so.SUM, 0.0, 2.0**-24, 1.0)
    assert got == 1.0


def test_array_region_with_some_scalars_unchanged():
    size = 4096
    orig = np.zeros(size, np.uint8)
    vals = np.array([1, 2, 3, 4, 5], np.int32)
    orig[100:120] = vals.view(np.uint8)
    mem = orig.copy()
    mem[100:120] = np.array([1, 12, 3, 14, 5], np.int32).view(np.uint8)
    main = orig.copy()
    main[100:120] = np.array([100, 100, 100, 100, 100], np.int32).view(np.uint8)
    # 22 bytes: five scalars and two trailing bytes that are not a scalar
    mem[120:122] = 0xFF
    regions = so.fill_gaps([so.Region(100, 22, so.INT, so.SUM)], size)
    res = so.merge(orig, mem, main, regions)
    assert res.main[100:120].view(np.int32).tolist() == [100, 110, 100, 110, 100]
    assert res.diff_bytes == 8
    assert res.main[120:122].tolist() == [0, 0]
    assert res.chunks == {0}


def test_scalar_that_does_not_fit_at_the_image_end():
    size = 4095
    orig = np.zeros(size, np.uint8)
    mem = orig.copy()
    mem[-3:] = 9  # a Long at size - 3 would pass the end
    mem[size - 11 : size - 3] = np.array([7], np.int64).view(np.uint8)
    regions = so.fill_gaps(
        [so.Region(size - 11, 8, so.LONG, so.SUM), so.Region(size - 3, 8, so.LONG, so.SUM)], size
    )
    res = so.merge(orig, mem, orig.copy(), regions)
    assert res.main[size - 11 : size - 3].view(np.int64)[0] == 7
    assert res.main[-3:].tolist() == [0, 0, 0]
    assert res.diff_bytes == 8


def test_dirty_hint_on_either_page_of_a_straddling_scalar():
    size = 3 * 4096
    off = 4096 - 4
    orig = np.zeros(size, np.uint8)
    mem = orig.copy()
    mem[off : off + 8] = np.array([1.5], np.float64).view(np.uint8)
    regions = so.fill_gaps([so.Region(off, 8, so.DOUBLE, so.SUM)], size)
    for dirty, merged in (([1, 0, 0], True), ([0, 1, 0], True), ([0, 0, 1], False)):
        res = so.merge(orig, mem, orig.copy(), regions, dirty=np.array(dirty))
        assert (res.diff_bytes == 8) == merged
        # the page of the first byte is flagged, the chunks of both halves
        assert res.page_flags.tolist() == ([True, False, False] if merged else [False] * 3)
        assert res.chunks == ({31, 32} if merged else set())


def test_fill_gaps_rejects_overlap_and_regions_after_a_to_end_region():
    with pytest.raises(ValueError):
        so.fill_gaps([so.Region(0, 8, so.LONG, so.SUM), so.Region(4, 4, so.INT, so.SUM)], 100)
    with pytest.raises(ValueError):
        so.fill_gaps([so.Region(10, 0, so.RAW, so.IGNORE), so.Region(50, 4, so.INT, so.SUM)], 100)
    got = so.fill_gaps([so.Region(4, 4, so.INT, so.SUM), so.Region(8, 4, so.INT, so.MAX)], 100, so.XOR)
    assert [(r.offset, r.length, r.op) for r in got] == [(0, 4, so.XOR), (4, 4, so.SUM), (8, 4, so.MAX), (12, 0, so.XOR)]


def test_apply_typed_array_diff():
    img = np.zeros(64, np.uint8)
    img[8:20] = np.array([1, 2, 3], np.int32).view(np.uint8)
    diff = np.array([10, 20, 30], np.int32).tobytes() + b"\x01\x02"  # 14 bytes: 3 scalars
    got, _ = so.apply(img, [(8, so.INT, so.SUM, diff)])
    assert got[8:20].view(np.int32).tolist() == [11, 22, 33]
    assert got[20:22].tolist() == [0, 0]
    # cut at the image end: only whole scalars inside the image
    got, _ = so.apply(img, [(56, so.LONG, so.SUM, np.array([5, 6], np.int64).tobytes())])
    assert got[56:64].view(np.int64)[0] == 5
