"""NumPy model of the neighbourhood v-collectives (MPI_Neighbor_allgatherv
and MPI_Neighbor_alltoallv, and the grouped neighbour v kinds behind them):
every rank's whole recv buffer after the call, from the buffers before it
and the graph's in-edges (see faabric_b200.parallel.comm.neighbor_in_edges),
and the launch count the device path takes.  Counts and displacements are in
elements of the arrays' dtype."""

import numpy as np

KINDS = ("neighbor_all_gather_v", "neighbor_all_to_all_v")
CHUNK = 2048  # FB_NEIGHBOR_CHUNK


def neighbor_exchange_v(kind, sends, recvs, in_edges, recvcounts, rdispls, sendcounts=None, sdispls=None):
    """Every rank's recv after one call.  Rank d's recv block j
    (``recvcounts[d][j]`` elements at ``rdispls[d][j]``) gets, for in-edge j
    = (s, idx), the send of s (all-gather: its first ``recvcounts[d][j]``
    elements) or s's send block idx (all-to-all: ``sendcounts[s][idx]``
    elements at ``sdispls[s][idx]``).  Every other element is unchanged.  A
    recv count must equal its sender's count for the edge; the results are new
    arrays."""
    if kind not in KINDS:
        raise ValueError(f"unknown kind {kind!r}")
    out = [np.array(r, copy=True) for r in recvs]
    for d, edges in enumerate(in_edges):
        for j, (s, idx) in enumerate(edges):
            c = int(recvcounts[d][j])
            if kind == "neighbor_all_to_all_v":
                if int(sendcounts[s][idx]) != c:
                    raise ValueError(f"edge {s} -> {d}: send count {sendcounts[s][idx]}, recv count {c}")
                at = int(sdispls[s][idx])
            else:
                at = 0
            src = np.asarray(sends[s])[at : at + c]
            if src.size != c:
                raise ValueError(f"rank {s}'s send has no {c} elements at {at}")
            out[d][int(rdispls[d][j]) : int(rdispls[d][j]) + c] = src
    return out


def stream_lengths(kind, out_degree, in_degree, sendcounts, recvcounts, esize):
    """One rank's stream lengths in bytes over a list of items: a send stream
    per out-edge (all-gather: one, when the rank has an out-edge) and a recv
    stream per in-edge, each the sum of its edge's block over the items.
    ``sendcounts[i]`` is a list per item (all-gather: one count)."""
    sends = out_degree if kind == "neighbor_all_to_all_v" else min(out_degree, 1)
    streams = [sum(int(sc[k]) for sc in sendcounts) * esize for k in range(sends)]
    streams += [sum(int(rc[j]) for rc in recvcounts) * esize for j in range(in_degree)]
    return streams


def launches(agreed, stage_bytes, max_out_degree, kind):
    """Kernel launches of a v list whose launch windows have the agreed
    longest streams ``agreed``: a slot holds stage_bytes (over the largest
    out-degree for the all-to-all) in whole chunks, at most the window's
    stream rounded up to a chunk, and a window takes one launch per slot
    width of its longest stream."""
    slots = max(max_out_degree, 1) if kind == "neighbor_all_to_all_v" else 1
    room = min(stage_bytes, 1 << 31) // CHUNK // slots * CHUNK
    total = 0
    for m in agreed:
        if m:
            width = min(room, -(-m // CHUNK) * CHUNK)
            total += -(-m // width)
    return total


def window_items(kind, max_out_degree, max_in_degree):
    """Items per launch window: every stream of the largest degrees, one
    16-byte entry per item and one more, and the in-edges (8 bytes each) fill
    at most the 1024 32-byte slots of a launch's table."""
    sends = max_out_degree if kind == "neighbor_all_to_all_v" else min(max_out_degree, 1)
    entries = (1024 * 32 - max_in_degree * 8) // 16
    return min(entries // (sends + max_in_degree) - 1, 1024 - 8)
