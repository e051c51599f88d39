"""NumPy model of a snapshot merge: what ``SnapshotData::diffWithDirtyRegions``
followed by ``applyDiffs`` (csrc/src/util/snapshot.cpp), and the fused device
diff-push, do to a main image.

Rules (the host is the specification, see faabric/util/reduce_ops.h):

* Bytewise copies each byte that differs, XOR applies ``old ^ new``; both only
  on dirty pages.  Ignore does nothing;
* a typed region is an array of ``length // size`` scalars, cut at the image
  end.  A scalar is merged when its first or its last page is dirty and
  ``new != old`` as values (NaN always differs, +0 == -0);
* Sum adds ``new - old``, Subtract subtracts ``old - new``, Product multiplies
  by ``new / old``: integers wrap; the integer quotient is 0 for ``old == 0``,
  a wrapping negation for ``old == -1`` and truncated otherwise; floats use
  IEEE division;
* float Max / Min ignore a NaN operand, quiet or signalling, and order -0
  below +0.

``merge`` also returns what the device reports: page flags and
``pages_with_diffs`` for the pages where a diff starts, the set of 128-byte
chunks that hold a diffed byte, and ``diff_bytes``.
"""

from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

PAGE = 4096
CHUNK = 128

RAW, BOOL, INT, LONG, FLOAT, DOUBLE = range(6)
BYTEWISE, SUM, PRODUCT, SUBTRACT, MAX, MIN, IGNORE, XOR = range(8)

NP_TYPES = {INT: np.int32, LONG: np.int64, FLOAT: np.float32, DOUBLE: np.float64}
TYPED_OPS = (SUM, PRODUCT, SUBTRACT, MAX, MIN)


@dataclass
class Region:
    offset: int
    length: int  # 0: to the end of the image
    data_type: int = RAW
    op: int = BYTEWISE


@dataclass
class Result:
    main: np.ndarray
    base: np.ndarray
    page_flags: np.ndarray  # bool per page: a diff starts there
    chunks: set  # 128-byte chunks holding a diffed byte
    diff_bytes: int
    pages_with_diffs: int
    nan_spans: list = field(default_factory=list)  # (offset, size) of NaN results


# ------------------------------------------------------------------ rules ----
def quotient(n: np.ndarray, o: np.ndarray) -> np.ndarray:
    """Product factor for values that went from ``o`` to ``n``."""
    if n.dtype.kind == "f":
        with np.errstate(all="ignore"):
            return n / o
    safe = np.where((o == 0) | (o == -1), 1, o)
    q = n // safe
    q = q + ((n % safe != 0) & ((n < 0) != (safe < 0)))  # floor -> truncation
    with np.errstate(all="ignore"):
        neg = np.zeros_like(n) - n  # wraps for MIN / -1
    return np.where(o == 0, 0, np.where(o == -1, neg, q)).astype(n.dtype)


def _ignore_nan(a: np.ndarray, b: np.ndarray, r: np.ndarray) -> np.ndarray:
    # a NaN operand, quiet or signalling, is ignored (np.fmax would quiet a
    # signalling one into the result)
    return np.where(np.isnan(a), b, np.where(np.isnan(b), a, r))


def fmax0(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    if a.dtype.kind != "f":
        return np.maximum(a, b)
    with np.errstate(invalid="ignore"):
        return _ignore_nan(a, b, np.where(a == b, np.where(np.signbit(a), b, a), np.where(a > b, a, b)))


def fmin0(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    if a.dtype.kind != "f":
        return np.minimum(a, b)
    with np.errstate(invalid="ignore"):
        return _ignore_nan(a, b, np.where(a == b, np.where(np.signbit(a), a, b), np.where(a < b, a, b)))


def diff_value(op: int, o: np.ndarray, n: np.ndarray) -> np.ndarray:
    """What a typed diff carries."""
    with np.errstate(all="ignore"):
        if op == SUM:
            return n - o
        if op == SUBTRACT:
            return o - n
        if op == PRODUCT:
            return quotient(n, o)
    return n.copy()  # Max / Min


def apply_value(op: int, c: np.ndarray, v: np.ndarray) -> np.ndarray:
    """Merges a received typed value into the current one."""
    with np.errstate(all="ignore"):
        if op == SUM:
            return c + v
        if op == SUBTRACT:
            return c - v
        if op == PRODUCT:
            return c * v
        if op == MAX:
            return fmax0(c, v)
        if op == MIN:
            return fmin0(c, v)
    raise ValueError(f"not a typed op: {op}")


# ---------------------------------------------------------------- regions ----
def fill_gaps(regions, size: int, fill_op: int = BYTEWISE) -> list:
    """``fillGapsWithBytewiseRegions``: sorted, gaps filled with ``fill_op``.
    Raises ValueError for overlapping regions or any region after one that
    runs to the end."""
    out = []
    cursor = 0
    to_end = False
    for r in sorted(regions, key=lambda r: r.offset):
        if to_end or r.offset < cursor:
            raise ValueError("overlapping merge regions")
        if r.offset > cursor:
            out.append(Region(cursor, r.offset - cursor, RAW, fill_op))
        out.append(Region(r.offset, r.length, r.data_type, r.op))
        if r.length == 0:
            to_end = True
        else:
            cursor = r.offset + r.length
    if not to_end and cursor < size:
        out.append(Region(cursor, 0, RAW, fill_op))
    return out


def _view(buf: np.ndarray, off: int, count: int, sz: int, t) -> np.ndarray:
    """``count`` scalars of type ``t`` every ``sz`` bytes from ``off`` (any alignment)."""
    idx = off + np.arange(count)[:, None] * sz + np.arange(sz)[None, :]
    return buf[idx].copy().view(t).reshape(count)


def _store(buf: np.ndarray, off: int, vals: np.ndarray, sz: int) -> None:
    idx = off + np.arange(len(vals))[:, None] * sz + np.arange(sz)[None, :]
    buf[idx] = vals.view(np.uint8).reshape(len(vals), sz)


# ------------------------------------------------------------------ merge ----
def merge(orig, mem, main, regions, dirty=None, update_base=False) -> Result:
    """One writer: diff ``mem`` against ``orig`` under the (gap-filled)
    ``regions`` and merge into ``main``."""
    orig = np.asarray(orig, dtype=np.uint8)
    mem = np.asarray(mem, dtype=np.uint8)
    size = min(len(orig), len(mem))
    main = np.array(main, dtype=np.uint8, copy=True)
    base = orig.copy()
    n_pages = (size + PAGE - 1) // PAGE
    dirty_p = np.ones(n_pages, dtype=bool) if dirty is None else np.asarray(dirty[:n_pages]).astype(bool)
    page_flags = np.zeros(n_pages, dtype=bool)
    chunks: set = set()
    diff_bytes = 0
    nan_spans = []
    for r in regions:
        beg = r.offset
        end = size if r.length == 0 else min(size, r.offset + r.length)
        if beg >= end or r.op == IGNORE:
            continue
        if r.op in (BYTEWISE, XOR):
            for p in range(beg // PAGE, (end - 1) // PAGE + 1):
                if not dirty_p[p]:
                    continue
                b, e = max(beg, p * PAGE), min(end, (p + 1) * PAGE)
                o, m = orig[b:e], mem[b:e]
                d = o != m
                if not d.any():
                    continue
                pos = np.nonzero(d)[0] + b
                diff_bytes += len(pos)
                page_flags[p] = True
                chunks.update((pos // CHUNK).tolist())
                if r.op == BYTEWISE:
                    main[pos] = mem[pos]
                else:
                    main[pos] ^= orig[pos] ^ mem[pos]
                if update_base:
                    base[pos] = mem[pos]
            continue
        t = NP_TYPES.get(r.data_type)
        if t is None or r.op not in TYPED_OPS:
            raise ValueError(f"unsupported region {r}")
        sz = np.dtype(t).itemsize
        count = (end - beg) // sz
        if count == 0:
            continue
        offs = beg + np.arange(count) * sz
        first, last = offs // PAGE, (offs + sz - 1) // PAGE
        o = _view(orig, beg, count, sz, t)
        m = _view(mem, beg, count, sz, t)
        with np.errstate(invalid="ignore"):
            sel = (dirty_p[first] | dirty_p[last]) & (o != m)
        if not sel.any():
            continue
        ks = np.nonzero(sel)[0]
        c = _view(main, beg, count, sz, t)
        v = diff_value(r.op, o[ks], m[ks])
        res = apply_value(r.op, c[ks], v).astype(t)
        for k, val in zip(ks.tolist(), res):
            off = beg + k * sz
            main[off : off + sz] = np.array([val], dtype=t).view(np.uint8)
            if update_base:
                base[off : off + sz] = mem[off : off + sz]
            page_flags[off // PAGE] = True
            chunks.update(range(off // CHUNK, (off + sz - 1) // CHUNK + 1))
            if t in (np.float32, np.float64) and np.isnan(val):
                nan_spans.append((off, sz))
        diff_bytes += sz * len(ks)
    return Result(main, base, page_flags, chunks, diff_bytes, int(page_flags.sum()), nan_spans)


def apply(image, diffs) -> tuple:
    """``SnapshotData::applyDiffs`` for [(offset, data_type, op, bytes)] in
    order.  Returns the new image and the (offset, size) spans holding a NaN."""
    img = np.array(image, dtype=np.uint8, copy=True)
    nan_spans = []
    for off, dt, op, data in diffs:
        data = np.frombuffer(bytes(data), dtype=np.uint8)
        if op == IGNORE or off >= len(img):
            continue
        n = min(len(data), len(img) - off)
        if op == BYTEWISE:
            img[off : off + n] = data[:n]
        elif op == XOR:
            img[off : off + n] ^= data[:n]
        else:
            t = NP_TYPES[dt]
            sz = np.dtype(t).itemsize
            cnt = n // sz
            if cnt == 0:
                continue
            c = _view(img, off, cnt, sz, t)
            v = _view(data, 0, cnt, sz, t)
            res = apply_value(op, c, v).astype(t)
            _store(img, off, res, sz)
            if t in (np.float32, np.float64):
                nan_spans += [(off + k * sz, sz) for k in np.nonzero(np.isnan(res))[0].tolist()]
    return img, nan_spans


def mismatches(got, exp, nan_spans=()) -> np.ndarray:
    """Byte positions where ``got`` differs from ``exp``: bit for bit, except
    that a scalar the oracle computed as NaN matches any NaN of its type."""
    got = np.asarray(got, dtype=np.uint8)
    exp = np.asarray(exp, dtype=np.uint8)
    bad = got != exp
    for off, sz in nan_spans:
        t = np.float32 if sz == 4 else np.float64
        if np.isnan(got[off : off + sz].copy().view(t)[0]):
            bad[off : off + sz] = False
    return np.nonzero(bad)[0]
