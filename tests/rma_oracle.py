"""Exact reference for the one-sided atomics (NumPy only).

Builds on ``reduce_oracle``: an accumulate sets every target element to
``combine(target, origin)``, the same step the reduce kernels fold with, so
``target`` is the accumulator and the origin element the new operand.  Added
here:

* ``replace`` stores the origin element, ``no_op`` keeps the target (an atomic
  read, only with a fetch);
* the fetch variants return every element's previous value;
* the 16-byte MAXLOC/MINLOC pairs (``f64_i32``, ``i64_i32``) keep the
  target's 4 padding bytes, whatever the op;
* compare-and-swap on one integer element.

Each element is updated atomically, so accumulates of one (dtype, op) from
several origins give the fold of their operands in SOME order; ops that are
commutative and associative on the values used (integers, MAX/MIN, small
integers in floats) give one exact answer.
"""

from __future__ import annotations

import numpy as np

import reduce_oracle as ro
from reduce_oracle import ALL_OPS, DTYPES, INT_DTYPES, NP_DTYPES, PAIR_DTYPES

RMA_OPS = ALL_OPS + ["replace", "no_op"]
PADDED_PAIRS = ("f64_i32", "i64_i32")


def supported(dtype: str, op: str, fetch: bool) -> bool:
    if dtype not in DTYPES:
        return False
    if op == "replace":
        return True
    if op == "no_op":
        return fetch
    return op in ALL_OPS and ro.supported(dtype, op)


ACCUMULATE = [(d, o) for d in DTYPES for o in RMA_OPS if supported(d, o, False)]
FETCH = [(d, o) for d in DTYPES for o in RMA_OPS if supported(d, o, True)]
UNSUPPORTED = [(d, o) for d in DTYPES for o in ALL_OPS if not supported(d, o, True)]
CAS_DTYPES = INT_DTYPES


def _as(x, dtype: str) -> np.ndarray:
    """A 1-D copy of every byte (NumPy's own copies of structured arrays may
    drop padding bytes)."""
    a = np.asarray(x)
    if a.dtype != NP_DTYPES[dtype]:
        a = np.array(x, dtype=NP_DTYPES[dtype])
    return np.ascontiguousarray(a).reshape(-1).view(np.uint8).copy().view(NP_DTYPES[dtype])


def _keep_padding(new: np.ndarray, old: np.ndarray, dtype: str) -> np.ndarray:
    if dtype in PADDED_PAIRS and new.size:
        nb = new.view(np.uint8).reshape(-1, 16)
        nb[:, 12:] = old.view(np.uint8).reshape(-1, 16)[:, 12:]
    return new


def accumulate(target, origin, dtype: str, op: str):
    """(new target, fetched previous values) of one accumulate."""
    old = _as(target, dtype)
    if op == "no_op":
        return _as(old, dtype), old
    if not supported(dtype, op, False):
        raise ValueError(f"{dtype} {op} is not a one-sided accumulate")
    o = _as(origin, dtype)
    new = o if op == "replace" else _as(ro.combine(_as(old, dtype), o, dtype, op), dtype)
    return _keep_padding(new, old, dtype), old


def fold(target, origins, dtype: str, op: str) -> np.ndarray:
    """Target after the accumulates of ``origins``, applied in list order."""
    t = _as(target, dtype)
    for o in origins:
        t, _ = accumulate(t, o, dtype, op)
    return t


def compare_and_swap(target, compare, swap, dtype: str):
    """(new target, fetched previous value) of one element."""
    if dtype not in CAS_DTYPES:
        raise ValueError(f"compare-and-swap takes an integer dtype, not {dtype}")
    old = _as(target, dtype)
    new = _as(swap, dtype) if old[0] == _as(compare, dtype)[0] else _as(old, dtype)
    return new, old


def mismatches(got, exp, dtype: str) -> np.ndarray:
    """As ``reduce_oracle.mismatches``; padding of the 16-byte pairs counts."""
    bad = ro.mismatches(got, exp, dtype)
    if dtype in PADDED_PAIRS:
        g = np.asarray(got).view(np.uint8).reshape(-1, 16)[:, 12:]
        e = np.asarray(exp).view(np.uint8).reshape(-1, 16)[:, 12:]
        bad = np.union1d(bad, np.nonzero((g != e).any(axis=1))[0])
    return bad


def assert_same(got, exp, dtype: str, what: str = ""):
    bad = mismatches(got, exp, dtype)
    if bad.size:
        i = bad[:8]
        g = np.asarray(got).view(NP_DTYPES[dtype])
        e = np.asarray(exp).view(NP_DTYPES[dtype])
        raise AssertionError(
            f"{what}: {bad.size} of {e.size} {dtype} elements differ; first at {i.tolist()}: "
            f"got {g[i].tolist()} expected {e[i].tolist()}"
        )


__all__ = [
    "ACCUMULATE",
    "CAS_DTYPES",
    "FETCH",
    "PAIR_DTYPES",
    "RMA_OPS",
    "UNSUPPORTED",
    "accumulate",
    "assert_same",
    "compare_and_swap",
    "fold",
    "mismatches",
    "supported",
]
