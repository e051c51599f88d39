"""Exact reference for the device reductions (NumPy only).

Every single-GPU reduction path folds the ranks' inputs in rank order,
``acc = x[0]; acc = op(acc, x[p])`` for p = 1..n-1, so the expected result is
fully determined and a kernel must match it bit for bit:

* integers: arithmetic in the dtype itself, wrapping; MAX/MIN are signed or
  unsigned as the dtype is; land/lor/lxor give 0 or 1;
* f32/f64: a left fold in that dtype;
* f16/bf16: both operands are widened to f32, the op is applied in f32 and the
  result is rounded to the dtype (round to nearest even) after every step;
* float MAX/MIN are fmax/fmin: a NaN operand is ignored, the result is NaN only
  where both operands are; between +0 and -0, MAX gives +0 and MIN gives -0;
* MAXLOC/MINLOC on {value, int32 index} pairs laid out like ``PairVI<T>``
  (the 16-byte pairs carry 4 bytes of padding, whose contents are
  unspecified); value ties go to the lower index.

bf16 values are carried as their uint16 bit patterns (NumPy has no bf16).
"""

from __future__ import annotations

import numpy as np

INT_DTYPES = ["i8", "u8", "i16", "u16", "i32", "u32", "i64", "u64"]
FLOAT_DTYPES = ["f32", "f64", "f16", "bf16"]
PAIR_DTYPES = ["f64_i32", "f32_i32", "i32_i32", "i64_i32"]
DTYPES = INT_DTYPES + FLOAT_DTYPES + PAIR_DTYPES

INT_OPS = ["max", "min", "sum", "prod", "land", "lor", "lxor", "band", "bor", "bxor"]
FLOAT_OPS = ["max", "min", "sum", "prod"]
PAIR_OPS = ["maxloc", "minloc"]
ALL_OPS = sorted(set(INT_OPS + PAIR_OPS))


def _pair(vfmt: str, itemsize: int) -> np.dtype:
    # PairVI<T> {T v; int32_t i;}: i follows v, the struct is aligned like T
    return np.dtype({"names": ["v", "i"], "formats": [vfmt, "<i4"], "offsets": [0, np.dtype(vfmt).itemsize], "itemsize": itemsize})


# storage dtype of every FbDtype (bf16: raw bits)
NP_DTYPES = {
    "i8": np.dtype(np.int8),
    "u8": np.dtype(np.uint8),
    "i16": np.dtype("<i2"),
    "u16": np.dtype("<u2"),
    "i32": np.dtype("<i4"),
    "u32": np.dtype("<u4"),
    "i64": np.dtype("<i8"),
    "u64": np.dtype("<u8"),
    "f32": np.dtype("<f4"),
    "f64": np.dtype("<f8"),
    "f16": np.dtype("<f2"),
    "bf16": np.dtype("<u2"),
    "f64_i32": _pair("<f8", 16),
    "f32_i32": _pair("<f4", 8),
    "i32_i32": _pair("<i4", 8),
    "i64_i32": _pair("<i8", 16),
}


def supported(dtype: str, op: str) -> bool:
    if dtype in INT_DTYPES:
        return op in INT_OPS
    if dtype in FLOAT_DTYPES:
        return op in FLOAT_OPS
    return op in PAIR_OPS


SUPPORTED = [(d, o) for d in DTYPES for o in ALL_OPS if supported(d, o)]
UNSUPPORTED = [(d, o) for d in DTYPES for o in ALL_OPS if not supported(d, o)]


def itemsize(dtype: str) -> int:
    return NP_DTYPES[dtype].itemsize


# ------------------------------------------------------------------ bf16 ----
def bf16_to_f32(bits: np.ndarray) -> np.ndarray:
    return (np.asarray(bits, dtype=np.uint32) << 16).view(np.float32)


def f32_to_bf16(x: np.ndarray) -> np.ndarray:
    """Round f32 to bf16 bits, to nearest even; a NaN stays a quiet NaN."""
    u = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    rounded = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) & 0xFFFF
    nan = (u & 0x7FFFFFFF) > 0x7F800000
    return np.where(nan, (u >> 16) | 0x40, rounded).astype(np.uint16)


# ----------------------------------------------------------------- float ----
def _fmaxmin(a: np.ndarray, b: np.ndarray, op: str) -> np.ndarray:
    r = np.fmax(a, b) if op == "max" else np.fmin(a, b)
    # +0 and -0 compare equal: MAX prefers +0, MIN prefers -0
    zero = (a == 0) & (b == 0)
    if zero.any():
        neg = np.signbit(a) & np.signbit(b) if op == "max" else np.signbit(a) | np.signbit(b)
        r = np.where(zero, np.where(neg, -np.zeros_like(r), np.zeros_like(r)), r)
    return r


def _float_op(a: np.ndarray, b: np.ndarray, op: str) -> np.ndarray:
    with np.errstate(all="ignore"):
        if op == "sum":
            return a + b
        if op == "prod":
            return a * b
    return _fmaxmin(a, b, op)


# -------------------------------------------------------------------- int ----
def _int_op(a: np.ndarray, b: np.ndarray, op: str) -> np.ndarray:
    dt = a.dtype
    if op == "max":
        return np.maximum(a, b)
    if op == "min":
        return np.minimum(a, b)
    if op == "sum":
        return np.add(a, b, dtype=dt)
    if op == "prod":
        return np.multiply(a, b, dtype=dt)
    if op == "land":
        return ((a != 0) & (b != 0)).astype(dt)
    if op == "lor":
        return ((a != 0) | (b != 0)).astype(dt)
    if op == "lxor":
        return ((a != 0) != (b != 0)).astype(dt)
    if op == "band":
        return a & b
    if op == "bor":
        return a | b
    if op == "bxor":
        return a ^ b
    raise ValueError(op)


def _pair_op(a: np.ndarray, b: np.ndarray, op: str) -> np.ndarray:
    better = b["v"] > a["v"] if op == "maxloc" else b["v"] < a["v"]
    take = better | ((b["v"] == a["v"]) & (b["i"] < a["i"]))
    out = a.copy()
    out[take] = b[take]
    return out


def combine(a: np.ndarray, b: np.ndarray, dtype: str, op: str) -> np.ndarray:
    """One step of the fold: op(a, b) with a the accumulator."""
    if not supported(dtype, op):
        raise ValueError(f"{dtype} {op} is not a device reduction")
    if dtype in PAIR_DTYPES:
        return _pair_op(a, b, op)
    if dtype in INT_DTYPES:
        return _int_op(a, b, op)
    if dtype == "bf16":
        return f32_to_bf16(_float_op(bf16_to_f32(a), bf16_to_f32(b), op))
    if dtype == "f16":
        r = _float_op(a.astype(np.float32), b.astype(np.float32), op)
        with np.errstate(all="ignore"):
            return r.astype(np.float16)  # NumPy rounds to nearest even
    return _float_op(a, b, op)


def fold(inputs, dtype: str, op: str) -> np.ndarray:
    """What every kernel must produce from the per-rank ``inputs`` (rank order,
    arrays of ``NP_DTYPES[dtype]``)."""
    acc = np.array(inputs[0], dtype=NP_DTYPES[dtype], copy=True)
    for x in inputs[1:]:
        acc = combine(acc, np.asarray(x, dtype=NP_DTYPES[dtype]), dtype, op)
    return acc


# ------------------------------------------------------------- comparing ----
def _is_nan(x: np.ndarray, dtype: str) -> np.ndarray:
    if dtype == "bf16":
        return (x & 0x7FFF) > 0x7F80
    return np.isnan(x)


def _bits(x: np.ndarray) -> np.ndarray:
    return x.view(np.dtype(f"<u{x.dtype.itemsize}"))


def mismatches(got: np.ndarray, exp: np.ndarray, dtype: str) -> np.ndarray:
    """Indices where ``got`` differs from ``exp``: bit for bit, except that
    any NaN matches any NaN and pair padding is ignored."""
    got = np.asarray(got).view(NP_DTYPES[dtype])
    exp = np.asarray(exp).view(NP_DTYPES[dtype])
    assert got.shape == exp.shape, (got.shape, exp.shape)
    if dtype in PAIR_DTYPES:
        v_got, v_exp = np.ascontiguousarray(got["v"]), np.ascontiguousarray(exp["v"])
        bad = _bits(v_got) != _bits(v_exp)
        if dtype in ("f64_i32", "f32_i32"):
            bad &= ~(np.isnan(v_got) & np.isnan(v_exp))
        return np.nonzero(bad | (got["i"] != exp["i"]))[0]
    bad = _bits(got) != _bits(exp)
    if dtype in FLOAT_DTYPES:
        bad &= ~(_is_nan(got, dtype) & _is_nan(exp, dtype))
    return np.nonzero(bad)[0]


def assert_same(got: np.ndarray, exp: np.ndarray, dtype: str, what: str = ""):
    bad = mismatches(got, exp, dtype)
    if bad.size:
        i = bad[:8]
        g = np.asarray(got).view(NP_DTYPES[dtype])
        e = np.asarray(exp).view(NP_DTYPES[dtype])
        raise AssertionError(
            f"{what}: {bad.size} of {e.size} {dtype} elements differ; first at {i.tolist()}: "
            f"got {g[i].tolist()} expected {e[i].tolist()}"
        )
