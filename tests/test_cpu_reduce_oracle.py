"""The reduction oracle (tests/reduce_oracle.py) against hand-computed cases:
the GPU reduction matrix trusts it bit for bit, so it is checked here first."""

import numpy as np
import pytest

from reduce_oracle import (
    NP_DTYPES,
    SUPPORTED,
    UNSUPPORTED,
    assert_same,
    bf16_to_f32,
    f32_to_bf16,
    fold,
    mismatches,
)


def arr(dtype, values):
    return np.array(values, dtype=NP_DTYPES[dtype])


def test_support_table_has_every_device_instance():
    # 8 integer types x 10 ops, 4 float types x 4 ops, 4 pair types x 2 ops
    assert len(SUPPORTED) == 80 + 16 + 8 == 104
    assert len(SUPPORTED) + len(UNSUPPORTED) == 16 * 12


def test_bf16_sum_ties_round_to_even():
    # ulp(1.0) = 2^-7 in bf16; adding 2^-8 lands exactly halfway
    one, one_ulp, half_ulp = 0x3F80, 0x3F81, 0x3B80
    assert bf16_to_f32(np.uint16(half_ulp)) == 2.0**-8
    got = fold([arr("bf16", [one, one_ulp]), arr("bf16", [half_ulp, half_ulp])], "bf16", "sum")
    assert got.tolist() == [0x3F80, 0x3F82]  # both ties go to the even neighbour
    # just above the tie rounds up
    got = fold([arr("bf16", [one]), arr("bf16", [0x3B81])], "bf16", "sum")
    assert got.tolist() == [0x3F81]


def test_bf16_rounding_of_specials():
    f = np.array([np.inf, -np.inf, np.nan, 3.3895314e38, -0.0], dtype=np.float32)
    b = f32_to_bf16(f)
    assert b[0] == 0x7F80 and b[1] == 0xFF80
    assert (b[2] & 0x7FFF) > 0x7F80  # NaN stays NaN (not -0.0)
    assert f32_to_bf16(np.array([np.float32(3.4028235e38)]))[0] == 0x7F80  # rounds up to inf
    assert b[4] == 0x8000
    # a NaN whose payload would carry into the sign bit under plain rounding
    nan_all_ones = np.array([0x7FFFFFFF], dtype=np.uint32).view(np.float32)
    assert (f32_to_bf16(nan_all_ones)[0] & 0x7FFF) > 0x7F80


def test_f16_sum_ties_round_to_even():
    # ulp(1.0) = 2^-10 in f16; 2^-11 is half an ulp
    a = np.array([1.0, 1.0 + 2.0**-10], dtype=np.float16)
    b = np.array([2.0**-11, 2.0**-11], dtype=np.float16)
    got = fold([a, b], "f16", "sum")
    assert got.view(np.uint16).tolist() == [0x3C00, 0x3C02]


def test_f16_subnormal_sums_and_overflow_to_inf():
    u = lambda *v: np.array(v, dtype=np.uint16).view(np.float16)  # noqa: E731
    got = fold([u(0x0001, 0x03FF, 0x8001), u(0x0001, 0x0001, 0x0001)], "f16", "sum")
    # 2 x smallest subnormal; largest subnormal + smallest = smallest normal;
    # -tiny + tiny = +0 (no flush to zero anywhere)
    assert got.view(np.uint16).tolist() == [0x0002, 0x0400, 0x0000]
    # 65504 + 65504 overflows; 65504 + 16 is the tie between 65504 (odd
    # mantissa) and 65536 (= inf in f16): it rounds to even, i.e. to inf
    got = fold([u(0x7BFF, 0x7BFF, 0x7BFF), u(0x7BFF, 0x4C00, 0x4800)], "f16", "sum")
    assert got.view(np.uint16).tolist() == [0x7C00, 0x7C00, 0x7BFF]
    # subnormal products are computed in f32 and only rounded once
    got = fold([u(0x0200), u(0x3800)], "f16", "prod")  # 2^-15 * 0.5
    assert got.view(np.uint16).tolist() == [0x0100]


def test_int8_wraps():
    got = fold([arr("i8", [127, -128, 100]), arr("i8", [1, -1, 3])], "i8", "sum")
    assert got.tolist() == [-128, 127, 103]
    got = fold([arr("i8", [127, -128, 100]), arr("i8", [1, -1, 3])], "i8", "prod")
    assert got.tolist() == [127, -128, 44]  # 300 mod 256 = 44
    got = fold([arr("u8", [255]), arr("u8", [2]), arr("u8", [3])], "u8", "sum")
    assert got.tolist() == [4]


def test_unsigned_max_min_see_the_top_bit():
    a, b = arr("u32", [0x80000000]), arr("u32", [1])
    assert fold([a, b], "u32", "max").tolist() == [0x80000000]
    assert fold([a, b], "u32", "min").tolist() == [1]
    # the same bits as signed: the top bit makes it negative
    assert fold([a.view(np.int32), b.view(np.int32)], "i32", "max").tolist() == [1]
    assert fold([arr("u64", [1 << 63]), arr("u64", [7])], "u64", "max").tolist() == [1 << 63]
    assert fold([arr("u16", [0x8000]), arr("u16", [0x7FFF])], "u16", "min").tolist() == [0x7FFF]


def test_int16_logical_ops_look_at_the_whole_value():
    # 0x0100 is non-zero although its low byte is 0
    a = arr("i16", [0x0100, 0x0100, 0, 0x0100])
    b = arr("i16", [1, 0, 0, 0x0200])
    assert fold([a, b], "i16", "land").tolist() == [1, 0, 0, 1]
    assert fold([a, b], "i16", "lor").tolist() == [1, 1, 0, 1]
    assert fold([a, b], "i16", "lxor").tolist() == [0, 1, 0, 0]
    assert fold([a, b], "i16", "bxor").tolist() == [0x0101, 0x0100, 0, 0x0300]
    # lxor over three ranks: parity of the non-zero count
    c = arr("i16", [-1, 5, 0, 0])
    assert fold([a, b, c], "i16", "lxor").tolist() == [1, 0, 0, 0]


@pytest.mark.parametrize("dtype", ["f64_i32", "f32_i32", "i32_i32", "i64_i32"])
def test_maxloc_minloc_ties_go_to_the_lower_index(dtype):
    def pairs(*vi):
        out = np.zeros(len(vi), dtype=NP_DTYPES[dtype])
        for k, (v, i) in enumerate(vi):
            out[k] = (v, i)
        return out

    ranks = [pairs((3, 5), (1, 9), (2, 4)), pairs((3, 2), (0, 1), (2, 8)), pairs((3, 7), (1, 0), (-1, 3))]
    mx = fold(ranks, dtype, "maxloc")
    assert mx["v"].tolist() == [3, 1, 2] and mx["i"].tolist() == [2, 0, 4]
    mn = fold(ranks, dtype, "minloc")
    assert mn["v"].tolist() == [3, 0, -1] and mn["i"].tolist() == [2, 1, 3]
    assert NP_DTYPES[dtype].itemsize == (16 if dtype in ("f64_i32", "i64_i32") else 8)


@pytest.mark.parametrize("dtype", ["f32", "f64", "f16"])
def test_float_max_min_ignore_a_nan_wherever_it_sits(dtype):
    nan = np.nan
    ranks = [arr(dtype, [nan, 1, nan, 1]), arr(dtype, [2, 2, nan, 3]), arr(dtype, [1, nan, nan, 2])]
    mx = fold(ranks, dtype, "max")
    mn = fold(ranks, dtype, "min")
    assert mx[[0, 1, 3]].tolist() == [2, 2, 3] and np.isnan(mx[2])
    assert mn[[0, 1, 3]].tolist() == [1, 1, 1] and np.isnan(mn[2])


def test_bf16_max_min_ignore_nan_and_order_signed_zeros():
    nan, one, two = 0x7FC0, 0x3F80, 0x4000
    ranks = [arr("bf16", [nan, one, 0x8000]), arr("bf16", [two, nan, 0x0000])]
    assert fold(ranks, "bf16", "max").tolist() == [two, one, 0x0000]
    assert fold(ranks, "bf16", "min").tolist() == [two, one, 0x8000]


def test_mismatches_is_bit_exact_but_any_nan_matches():
    a = np.array([0.0, np.nan, 1.0], dtype=np.float32)
    b = np.array([-0.0, -np.nan, 1.0], dtype=np.float32)
    assert mismatches(a, b, "f32").tolist() == [0]
    with pytest.raises(AssertionError):
        assert_same(a, b, "f32")
    p = np.zeros(2, dtype=NP_DTYPES["f64_i32"])
    q = p.copy()
    q.view(np.uint8)[12] = 0xFF  # padding
    assert mismatches(p, q, "f64_i32").size == 0
    q["i"][1] = 1
    assert mismatches(p, q, "f64_i32").tolist() == [1]
