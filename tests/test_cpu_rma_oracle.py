"""The one-sided atomics oracle (tests/rma_oracle.py) against hand-computed
cases, so that the GPU tests compare the kernels with something known right."""

import numpy as np
import pytest

import rma_oracle as rm
from reduce_oracle import NP_DTYPES


def test_supported_sets():
    # every reduction pair, REPLACE everywhere, NO_OP only when fetching
    assert ("i32", "sum") in rm.ACCUMULATE and ("f32", "replace") in rm.ACCUMULATE
    assert ("f64_i32", "replace") in rm.ACCUMULATE and ("bf16", "no_op") not in rm.ACCUMULATE
    assert ("bf16", "no_op") in rm.FETCH and ("i64_i32", "no_op") in rm.FETCH
    assert len(rm.ACCUMULATE) == 104 + 16 and len(rm.FETCH) == 104 + 32
    assert ("f32", "band") in rm.UNSUPPORTED and ("i8", "maxloc") in rm.UNSUPPORTED
    assert not any(o in ("replace", "no_op") for _, o in rm.UNSUPPORTED)


def test_integer_sum_and_prod_wrap():
    t, f = rm.accumulate(np.array([127, -128, 5], np.int8), np.array([1, -1, 3], np.int8), "i8", "sum")
    assert t.tolist() == [-128, 127, 8] and f.tolist() == [127, -128, 5]
    t, _ = rm.accumulate(np.array([0xFFFF], np.uint16), np.array([2], np.uint16), "u16", "prod")
    assert t.tolist() == [0xFFFE]
    t, _ = rm.accumulate(np.array([2**62], np.int64), np.array([4], np.int64), "i64", "prod")
    assert t.tolist() == [0]
    t, _ = rm.accumulate(np.array([2**31 - 1], np.int32), np.array([1], np.int32), "i32", "sum")
    assert t.tolist() == [-(2**31)]


def test_float_max_min_ignore_nan_and_order_signed_zeros():
    nan = np.float32("nan")
    t, _ = rm.accumulate(np.array([nan, 1.0, 0.0, -0.0], np.float32), np.array([2.0, nan, -0.0, 0.0], np.float32), "f32", "max")
    assert t[0] == 2.0 and t[1] == 1.0
    assert t[2] == 0 and not np.signbit(t[2]) and not np.signbit(t[3])
    t, _ = rm.accumulate(np.array([0.0, -0.0, nan], np.float64), np.array([-0.0, 0.0, nan], np.float64), "f64", "min")
    assert np.signbit(t[0]) and np.signbit(t[1]) and np.isnan(t[2])


def test_maxloc_ties_pick_the_lower_index():
    dt = NP_DTYPES["f32_i32"]
    tgt = np.array([(1.0, 7), (3.0, 2), (1.0, 1)], dtype=dt)
    org = np.array([(1.0, 3), (2.0, 0), (1.0, 4)], dtype=dt)
    t, f = rm.accumulate(tgt, org, "f32_i32", "maxloc")
    assert t["i"].tolist() == [3, 2, 1] and t["v"].tolist() == [1.0, 3.0, 1.0]
    t, _ = rm.accumulate(tgt, org, "f32_i32", "minloc")
    assert t["i"].tolist() == [3, 0, 1]
    assert f["i"].tolist() == [7, 2, 1]


@pytest.mark.parametrize("op", ["maxloc", "minloc", "replace", "no_op"])
@pytest.mark.parametrize("dtype", ["f64_i32", "i64_i32"])
def test_pair_padding_is_preserved(dtype, op):
    raw_t = np.arange(32, dtype=np.uint8)
    raw_o = np.arange(100, 132, dtype=np.uint8)
    raw_t[0:8] = np.frombuffer(np.array([5], NP_DTYPES[dtype]["v"]).tobytes(), np.uint8)
    raw_o[0:8] = np.frombuffer(np.array([9], NP_DTYPES[dtype]["v"]).tobytes(), np.uint8)
    t, f = rm.accumulate(raw_t.view(NP_DTYPES[dtype]), raw_o.view(NP_DTYPES[dtype]), dtype, op)
    tb = t.view(np.uint8).reshape(2, 16)
    assert (tb[:, 12:] == raw_t.reshape(2, 16)[:, 12:]).all()
    assert (f.view(np.uint8) == raw_t).all()
    if op in ("maxloc", "replace"):
        assert (tb[0, :12] == raw_o[:12]).all()  # 9 > 5: the origin's value and index
    else:
        assert (tb[0, :12] == raw_t[:12]).all()
    # the comparison counts padding bytes
    other = t.view(np.uint8).copy().view(t.dtype)
    other.view(np.uint8)[15] ^= 1
    assert rm.mismatches(other, t, dtype).tolist() == [0]


def test_replace_and_no_op():
    t, f = rm.accumulate(np.array([1, 2], np.uint16), np.array([7, 8], np.uint16), "bf16", "replace")
    assert t.tolist() == [7, 8] and f.tolist() == [1, 2]
    t, f = rm.accumulate(np.array([3.5], np.float16), None, "f16", "no_op")
    assert t.tolist() == [3.5] and f.tolist() == [3.5]
    with pytest.raises(ValueError):
        rm.accumulate(np.array([1], np.float32), np.array([1], np.float32), "f32", "band")


def test_sub_word_accumulate_leaves_neighbours_alone():
    buf = np.arange(16, dtype=np.uint8)
    view = buf[4:6].view(np.int16)
    new, _ = rm.accumulate(view, np.array([1], np.int16), "i16", "sum")
    buf[4:6] = new.view(np.uint8)
    expect = np.arange(16, dtype=np.uint8)
    expect[4:6] = (np.array([0x0504 + 1], np.int16)).view(np.uint8)
    assert buf.tolist() == expect.tolist()


def test_half_sum_rounds_like_the_reductions():
    # f16: 2048 + 1 is a tie and rounds to even; 1 + 2^-24 (subnormal) is kept
    t, _ = rm.accumulate(np.array([2048, 2**-24], np.float16), np.array([1, 2**-24], np.float16), "f16", "sum")
    assert t.tolist() == [2048.0, 2**-23]
    # bf16 bits: 1.0 + 2^-8 is a tie, rounds to even (1.0)
    t, _ = rm.accumulate(np.array([0x3F80], np.uint16), np.array([0x3B80], np.uint16), "bf16", "sum")
    assert t.tolist() == [0x3F80]


def test_fold_applies_in_order():
    assert rm.fold(np.array([0], np.int32), [np.array([i], np.int32) for i in range(1, 5)], "i32", "sum").tolist() == [10]
    assert rm.fold(np.array([0], np.int32), [np.array([i], np.int32) for i in range(1, 5)], "i32", "replace").tolist() == [4]


def test_compare_and_swap():
    t, f = rm.compare_and_swap(np.array([5], np.int8), np.array([5], np.int8), np.array([-1], np.int8), "i8")
    assert t.tolist() == [-1] and f.tolist() == [5]
    t, f = rm.compare_and_swap(np.array([2**64 - 1], np.uint64), np.array([0], np.uint64), np.array([3], np.uint64), "u64")
    assert t.tolist() == [2**64 - 1] and f.tolist() == [2**64 - 1]
    with pytest.raises(ValueError):
        rm.compare_and_swap(np.array([1.0], np.float32), np.array([1.0], np.float32), np.array([2.0], np.float32), "f32")
