"""NumPy model of the neighbourhood collectives (MPI_Neighbor_allgather and
MPI_Neighbor_alltoall, and the grouped neighbour kinds behind them): every
rank's whole recv buffer after the call, guard bytes included, from the
buffers before it and the graph's in-edges (see
faabric_b200.parallel.comm.neighbor_in_edges).  Byte copies: any dtype is
its bytes."""

import numpy as np

KINDS = ("neighbor_all_gather", "neighbor_all_to_all")


def neighbor_exchange(kind, sends, recvs, in_edges, block, offset=0):
    """Rank d's recv after the call: block j (``block`` bytes at ``offset +
    j * block`` of ``recvs[d]``; ``offset`` is one int, or one per rank) gets
    the send of in-edge j's source s, or, for the all-to-all, block idx of it
    for the in-edge (s, idx).  Every other byte of ``recvs[d]`` is unchanged.
    ``sends[r]`` and ``recvs[r]`` are uint8 arrays; the results are new
    arrays."""
    if kind not in KINDS:
        raise ValueError(f"unknown kind {kind!r}")
    out = [np.array(r, dtype=np.uint8, copy=True) for r in recvs]
    offsets = [offset] * len(recvs) if isinstance(offset, int) else list(offset)
    for d, edges in enumerate(in_edges):
        offset = offsets[d]
        for j, (s, idx) in enumerate(edges):
            k = idx if kind == "neighbor_all_to_all" else 0
            src = np.asarray(sends[s], dtype=np.uint8)[k * block : (k + 1) * block]
            if src.size != block:
                raise ValueError(f"rank {s}'s send has no block {k} of {block} bytes")
            out[d][offset + j * block : offset + (j + 1) * block] = src
    return out


def staged_bytes(kind, out_degrees, in_degrees, block):
    """Bytes the staged device path moves for one item over every rank: each
    rank writes its staged blocks (reading its send) and each in-edge's block
    is read from staging and written to recv."""
    staged = sum((d if kind == "neighbor_all_to_all" else min(d, 1)) for d in out_degrees) * block
    pulled = sum(in_degrees) * block
    return 2 * staged + 2 * pulled
