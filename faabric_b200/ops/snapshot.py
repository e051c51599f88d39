"""Device snapshot ops: fused diff + merge-op + push, dirty-page detection,
chunk-run extraction and diff application (csrc/kernels/snapshot_kernels.cu).

Semantics follow SnapshotData / SnapshotMergeRegion (csrc/src/util/snapshot.cpp),
the host implementation; enum values are ABI-identical.  Typed merges use the
rules of faabric/util/reduce_ops.h on both sides:

* a typed region is an array of ``length // size`` scalars; trailing bytes and
  a scalar that would pass the image end produce nothing.  A scalar is merged
  when its first or its last 4 KiB page is dirty;
* a scalar is unchanged when ``new == old`` as values: a NaN always counts as
  a change, +0 and -0 never do;
* integer Sum / Subtract / Product wrap (two's complement);
* the Product factor is ``new / old``: IEEE for floats (±inf or NaN when old
  is 0); for integers 0 when old is 0, a wrapping negation when old is -1,
  otherwise truncated;
* float Max / Min ignore a NaN operand and order -0 below +0, so the merged
  value does not depend on which writer lands first;
* regions may not overlap, and no region may follow one that runs to the end
  (length 0): ``prepare_regions`` raises ``ValueError``;
* ``pages_with_diffs`` (``stats[1]``) and ``page_flags_out`` count the pages
  in which a diff starts: a changed Bytewise / XOR byte, or the first byte of
  a typed scalar that produced a diff.

Concurrent writers into one image agree bit for bit for order-independent
operations.  A scalar that straddles a 16-byte boundary is merged by a plain
load / modify / store, so there the last writer wins.

Every launch checks its tensors first: ``diff_push`` and ``dirty_scan`` need
16-byte aligned, contiguous images, and every flag, page or destination
buffer must cover the image.
"""

from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional, Sequence

import torch

from .. import _lib
from .._lib import FbDiffDesc, FbMergeRegion

PAGE = 4096
CHUNK = 128

# SnapshotDataType
RAW, BOOL, INT, LONG, FLOAT, DOUBLE = range(6)
# SnapshotMergeOperation
BYTEWISE, SUM, PRODUCT, SUBTRACT, MAX, MIN, IGNORE, XOR = range(8)


@dataclass
class MergeRegion:
    offset: int
    length: int  # 0 => to the end of the image
    data_type: int = RAW
    op: int = BYTEWISE


@dataclass
class PreparedRegions:
    regions: torch.Tensor  # uint8 view of FbMergeRegionDev[n] on device
    n: int
    typed: torch.Tensor  # int32 indices on device
    n_typed: int
    host: list


def _nbytes(t: torch.Tensor) -> int:
    return t.numel() * t.element_size()


def _check_image(name: str, t: torch.Tensor) -> None:
    # the kernels use 16-byte vector loads / stores and 32-bit atomics on
    # offsets relative to the image start
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")
    if t.data_ptr() % 16 != 0:
        raise ValueError(f"{name} must be 16-byte aligned (address {t.data_ptr():#x})")


def _check_covers(name: str, t: Optional[torch.Tensor], nbytes: int) -> None:
    if t is None:
        return
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")
    if _nbytes(t) < nbytes:
        raise ValueError(f"{name} has {_nbytes(t)} bytes, needs {nbytes}")


def _stream(device, stream):
    if stream is None:
        stream = torch.cuda.current_stream(device)
    return C.c_void_p(stream.cuda_stream)


def prepare_regions(
    regions: Sequence[MergeRegion], size: int, device, fill_op: int = BYTEWISE
) -> PreparedRegions:
    """Sort, fill gaps with `fill_op` regions (reference
    fillGapsWithBytewiseRegions) and upload."""
    lib = _lib.load()
    n_in = len(regions)
    arr = (FbMergeRegion * max(n_in, 1))()
    for i, r in enumerate(regions):
        arr[i] = FbMergeRegion(r.offset, r.length, r.data_type, r.op)
    cap = 2 * n_in + 2
    out = (FbMergeRegion * cap)()
    typed = (C.c_int32 * cap)()
    n_typed = C.c_int(0)
    n = lib.fb_snapshot_prepare_regions(
        arr, n_in, fill_op, size, out, cap, typed, C.byref(n_typed)
    )
    if n == -2:  # FB_E_INVALID
        raise ValueError("overlapping merge regions, or a region after one that runs to the end")
    if n < 0:
        raise RuntimeError("too many merge regions")
    raw = bytes(out)[: n * C.sizeof(FbMergeRegion)]
    reg_dev = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(device)
    typed_host = torch.tensor(list(typed)[: n_typed.value] or [0], dtype=torch.int32)
    host = [MergeRegion(out[i].offset, out[i].length, out[i].dataType, out[i].op) for i in range(n)]
    return PreparedRegions(reg_dev, n, typed_host.to(device), n_typed.value, host)


def diff_push(
    mem: torch.Tensor,
    orig: torch.Tensor,
    dst: torch.Tensor | int,
    regions: Optional[PreparedRegions] = None,
    dirty_pages: Optional[torch.Tensor] = None,
    update_base: bool = False,
    page_flags_out: Optional[torch.Tensor] = None,
    chunk_flags: Optional[torch.Tensor] = None,
    stats: Optional[torch.Tensor] = None,
    blocks: int = 0,
    stream=None,
) -> torch.Tensor:
    """Fused scan + diff + merge + push.  `dst` is the main image: a tensor or
    a raw (peer-mapped) device pointer.  Returns the stats tensor
    ``[diff_bytes, pages_with_diffs]`` (uint64 as int64, on device; accumulates)."""
    lib = _lib.load()
    dev = mem.device
    size = min(_nbytes(mem), _nbytes(orig))
    n_pages = (size + PAGE - 1) // PAGE
    _check_image("mem", mem)
    _check_image("orig", orig)
    if isinstance(dst, int):
        if dst % 16 != 0:
            raise ValueError(f"dst must be 16-byte aligned (address {dst:#x})")
        dst_ptr = dst
    else:
        _check_image("dst", dst)
        _check_covers("dst", dst, size)
        dst_ptr = dst.data_ptr()
    _check_covers("dirty_pages", dirty_pages, n_pages)
    _check_covers("page_flags_out", page_flags_out, n_pages)
    _check_covers("chunk_flags", chunk_flags, (size + CHUNK - 1) // CHUNK)
    _check_covers("stats", stats, 16)
    if regions is None:
        regions = prepare_regions([], size, dev)
    if stats is None:
        stats = torch.zeros(2, dtype=torch.int64, device=dev)
    rc = lib.fb_snapshot_diff_push(
        C.c_void_p(mem.data_ptr()),
        C.c_void_p(orig.data_ptr()),
        C.c_void_p(dst_ptr),
        size,
        C.c_void_p(regions.regions.data_ptr()),
        regions.n,
        C.c_void_p(regions.typed.data_ptr()),
        regions.n_typed,
        C.c_void_p(dirty_pages.data_ptr() if dirty_pages is not None else 0),
        C.c_void_p(page_flags_out.data_ptr() if page_flags_out is not None else 0),
        C.c_void_p(chunk_flags.data_ptr() if chunk_flags is not None else 0),
        C.c_void_p(stats.data_ptr()),
        1 if update_base else 0,
        blocks,
        _stream(dev, stream),
    )
    if rc != 0:
        raise RuntimeError(f"fb_snapshot_diff_push failed ({rc})")
    return stats


def dirty_scan(mem: torch.Tensor, base: torch.Tensor, stream=None):
    """Compare-with-base dirty page detection: returns (flags uint8[nPages],
    count int64[1])."""
    lib = _lib.load()
    dev = mem.device
    _check_image("mem", mem)
    _check_image("base", base)
    size = min(_nbytes(mem), _nbytes(base))
    n_pages = (size + PAGE - 1) // PAGE
    flags = torch.empty(n_pages, dtype=torch.uint8, device=dev)
    count = torch.zeros(1, dtype=torch.int64, device=dev)
    rc = lib.fb_dirty_scan(
        C.c_void_p(mem.data_ptr()),
        C.c_void_p(base.data_ptr()),
        size,
        C.c_void_p(flags.data_ptr()),
        C.c_void_p(count.data_ptr()),
        0,
        _stream(dev, stream),
    )
    if rc != 0:
        raise RuntimeError("fb_dirty_scan failed")
    return flags, count


def flags_or(dst: torch.Tensor, src: torch.Tensor, stream=None):
    lib = _lib.load()
    rc = lib.fb_flags_or(
        C.c_void_p(dst.data_ptr()),
        C.c_void_p(src.data_ptr()),
        min(dst.numel(), src.numel()),
        _stream(dst.device, stream),
    )
    if rc != 0:
        raise RuntimeError("fb_flags_or failed")
    return dst


def chunk_runs(chunk_flags: torch.Tensor, total_bytes: int, chunk_bytes: int = CHUNK, max_out: int = 1 << 20, stream=None):
    """Chunk flags -> sorted list of (offset, length) runs.  Raises
    ``RuntimeError`` when there are more than ``max_out`` runs."""
    lib = _lib.load()
    dev = chunk_flags.device
    _check_covers("chunk_flags", chunk_flags, 0)
    out = torch.empty(max_out * C.sizeof(FbDiffDesc), dtype=torch.uint8, device=dev)
    count = torch.zeros(1, dtype=torch.int32, device=dev)
    rc = lib.fb_chunk_runs(
        C.c_void_p(chunk_flags.data_ptr()),
        chunk_flags.numel(),
        chunk_bytes,
        total_bytes,
        C.c_void_p(out.data_ptr()),
        max_out,
        C.c_void_p(count.data_ptr()),
        _stream(dev, stream),
    )
    if rc != 0:
        raise RuntimeError("fb_chunk_runs failed")
    n = int(count.item())
    if n > max_out:
        raise RuntimeError(f"{n} chunk runs do not fit max_out={max_out}")
    raw = out[: n * C.sizeof(FbDiffDesc)].cpu().numpy().tobytes()
    descs = (FbDiffDesc * n).from_buffer_copy(raw) if n else []
    return sorted((d.offset, d.length) for d in descs)


def apply_diffs(image: torch.Tensor, diffs: Sequence[tuple], stream=None):
    """Apply [(offset, data_type, op, bytes-like / uint8 tensor)] to a device
    image (SnapshotData::applyDiffs).  A typed diff of L bytes holds L // size
    scalars."""
    lib = _lib.load()
    dev = image.device
    _check_covers("image", image, 0)
    n = len(diffs)
    if n == 0:
        return image
    descs = (FbDiffDesc * n)()
    offs = []
    blobs = []
    cur = 0
    for i, (offset, data_type, op, data) in enumerate(diffs):
        if isinstance(data, torch.Tensor):
            b = data.detach().contiguous().view(torch.uint8).cpu().numpy().tobytes()
        else:
            b = bytes(data)
        descs[i] = FbDiffDesc(offset, len(b), data_type, op)
        offs.append(cur)
        blobs.append(b)
        cur += (len(b) + 15) // 16 * 16
        blobs.append(b"\0" * (cur - offs[-1] - len(b)))
    blob = torch.frombuffer(bytearray(b"".join(blobs) or b"\0"), dtype=torch.uint8).to(dev)
    d_dev = torch.frombuffer(bytearray(bytes(descs)), dtype=torch.uint8).to(dev)
    o_dev = torch.tensor(offs, dtype=torch.int64, device=dev)
    rc = lib.fb_snapshot_apply(
        C.c_void_p(image.data_ptr()),
        image.numel() * image.element_size(),
        C.c_void_p(d_dev.data_ptr()),
        C.c_void_p(o_dev.data_ptr()),
        C.c_void_p(blob.data_ptr()),
        n,
        _stream(dev, stream),
    )
    if rc != 0:
        raise RuntimeError("fb_snapshot_apply failed")
    return image
