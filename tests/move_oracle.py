"""Exact reference for the data-movement collectives and point-to-point calls
(NumPy only).

Movement ignores dtypes, so everything here is bytes.  Every buffer a call
may touch is given as a whole ``uint8`` array: the payload sits at ``offset``
inside it and the bytes around it are guards.  Each function returns what
every such array must hold afterwards, including what must stay untouched:

* the guard bytes around every output;
* the receive buffers of gather on ranks other than the root;
* the root's buffer in a broadcast;
* every send buffer (returned by :func:`untouched`).

``per`` is the payload per rank (all-gather, gather), per rank pair
(all-to-all, scatter: the send buffers hold ``n * per`` bytes) or the whole
message (broadcast, point-to-point).
"""

from __future__ import annotations

import numpy as np

COLLECTIVES = ("all_gather", "gather", "scatter", "all_to_all", "broadcast")
ROOTED = ("gather", "scatter", "broadcast")


def _bytes(a) -> np.ndarray:
    a = np.asarray(a)
    if a.dtype != np.uint8 or a.ndim != 1:
        raise TypeError("buffers are 1-D uint8 arrays")
    return a


def payload(buf, offset: int, nbytes: int) -> np.ndarray:
    """The ``nbytes`` payload bytes of ``buf`` at ``offset`` (a copy)."""
    buf = _bytes(buf)
    if offset < 0 or offset + nbytes > buf.size:
        raise ValueError(f"payload [{offset}, {offset + nbytes}) outside a {buf.size}-byte buffer")
    return buf[offset : offset + nbytes].copy()


def place(buf, offset: int, data) -> np.ndarray:
    """A copy of ``buf`` with ``data`` written at ``offset``; nothing else changes."""
    out = _bytes(buf).copy()
    data = _bytes(data)
    if offset < 0 or offset + data.size > out.size:
        raise ValueError(f"payload [{offset}, {offset + data.size}) outside a {out.size}-byte buffer")
    out[offset : offset + data.size] = data
    return out


def untouched(bufs) -> list:
    """Send buffers (and their guards) after any call: unchanged copies."""
    return [_bytes(b).copy() for b in bufs]


def all_gather(sends, send_offs, recvs, recv_offs, per: int) -> list:
    """Every rank's output is the concatenation of all ranks' payloads, in
    rank order."""
    cat = np.concatenate([payload(s, o, per) for s, o in zip(sends, send_offs)])
    return [place(r, o, cat) for r, o in zip(recvs, recv_offs)]


def gather(sends, send_offs, recvs, recv_offs, per: int, root: int) -> list:
    """The root's output is the rank-ordered concatenation; every other
    rank's receive buffer stays as it was (``None`` stays ``None``)."""
    cat = np.concatenate([payload(s, o, per) for s, o in zip(sends, send_offs)])
    out = []
    for r, (buf, o) in enumerate(zip(recvs, recv_offs)):
        if r == root:
            out.append(place(buf, o, cat))
        else:
            out.append(None if buf is None else _bytes(buf).copy())
    return out


def scatter(sends, send_offs, recvs, recv_offs, per: int, root: int) -> list:
    """Rank r receives bytes ``[r * per, (r + 1) * per)`` of the root's send
    payload; only the root's send buffer is read."""
    src = payload(sends[root], send_offs[root], per * len(recvs))
    return [place(buf, o, src[r * per : (r + 1) * per]) for r, (buf, o) in enumerate(zip(recvs, recv_offs))]


def all_to_all(sends, send_offs, recvs, recv_offs, per: int) -> list:
    """Block p of rank r's output is block r of rank p's send payload."""
    n = len(sends)
    srcs = [payload(s, o, per * n) for s, o in zip(sends, send_offs)]
    out = []
    for r, (buf, o) in enumerate(zip(recvs, recv_offs)):
        out.append(place(buf, o, np.concatenate([srcs[p][r * per : (r + 1) * per] for p in range(n)])))
    return out


def broadcast(bufs, offs, nbytes: int, root: int) -> list:
    """In place: every rank's payload becomes the root's; the root's buffer
    stays as it was."""
    src = payload(bufs[root], offs[root], nbytes)
    return [(_bytes(b).copy() if r == root else place(b, o, src)) for r, (b, o) in enumerate(zip(bufs, offs))]


def collective(kind: str, sends, send_offs, recvs, recv_offs, per: int, root: int = 0) -> list:
    """Expected receive buffers of collective ``kind`` (one of
    :data:`COLLECTIVES`); for ``broadcast`` the send arguments are ignored and
    ``recvs`` are the in-place buffers."""
    if kind == "all_gather":
        return all_gather(sends, send_offs, recvs, recv_offs, per)
    if kind == "gather":
        return gather(sends, send_offs, recvs, recv_offs, per, root)
    if kind == "scatter":
        return scatter(sends, send_offs, recvs, recv_offs, per, root)
    if kind == "all_to_all":
        return all_to_all(sends, send_offs, recvs, recv_offs, per)
    if kind == "broadcast":
        return broadcast(recvs, recv_offs, per, root)
    raise ValueError(f"unknown collective {kind!r}")


def send_recv(sends, send_offs, recvs, recv_offs, nbytes: int, src_of) -> list:
    """Point-to-point: rank r receives the ``nbytes`` payload of rank
    ``src_of(r)`` (send / recv, send_recv and put_signal alike)."""
    return [place(buf, o, payload(sends[src_of(r)], send_offs[src_of(r)], nbytes)) for r, (buf, o) in enumerate(zip(recvs, recv_offs))]


def first_difference(got, want):
    """Index of the first differing byte, or None when equal."""
    got, want = _bytes(got), _bytes(want)
    if got.size != want.size:
        return min(got.size, want.size)
    diff = np.flatnonzero(got != want)
    return int(diff[0]) if diff.size else None
