"""The neighbourhood oracle (tests/neighbor_oracle.py) and
faabric_b200.parallel.comm.neighbor_in_edges against hand-worked graphs:
self-edges, multi-edges, asymmetric and empty neighbourhoods, and the graphs
MPI_Dist_graph_create_adjacent refuses.  No GPU needed."""

import numpy as np
import pytest

import neighbor_oracle as no
from faabric_b200.parallel.comm import CommError, neighbor_in_edges


def u8(*v):
    return np.array(v, dtype=np.uint8)


def test_directed_ring():
    # 0 -> 1 -> 2 -> 0: one in-edge each, from the previous rank
    assert neighbor_in_edges([[2], [0], [1]], [[1], [2], [0]]) == [[(2, 0)], [(0, 0)], [(1, 0)]]


def test_periodic_2x1_halo_has_multi_and_self_edges():
    # neighbours left, right, down, up of a 2 x 1 periodic grid: left and
    # right are the other rank, down and up the rank itself
    nbrs = [[1, 1, 0, 0], [0, 0, 1, 1]]
    edges = neighbor_in_edges(nbrs, nbrs)
    # the k-th 1 in rank 0's sources pairs with the k-th 0 in rank 1's
    # destinations (MPI-3.1 7.6)
    assert edges == [[(1, 0), (1, 1), (0, 2), (0, 3)], [(0, 0), (0, 1), (1, 2), (1, 3)]]


def test_source_order_is_recv_order_and_multi_edges_pair_in_order():
    # rank 2 lists its sources as 1, 0, 0; rank 0 sends to 2 twice (positions
    # 1 and 2 of its destinations)
    dst = [[1, 2, 2], [2], []]
    src = [[], [0], [1, 0, 0]]
    assert neighbor_in_edges(src, dst) == [[], [(0, 0)], [(1, 0), (0, 1), (0, 2)]]


def test_asymmetric_and_empty_neighbourhoods():
    # rank 1 only sends, rank 2 only receives, rank 3 has no edge at all
    dst = [[2], [0, 2], [], []]
    src = [[1], [], [0, 1], []]
    assert neighbor_in_edges(src, dst) == [[(1, 0)], [], [(0, 0), (1, 1)], []]
    assert neighbor_in_edges([[]], [[]]) == [[]]


@pytest.mark.parametrize(
    "src,dst,what",
    [
        # an edge 0 -> 1 that rank 1 does not list
        ([[], []], [[1], []], "times"),
        # listed twice on one side, once on the other
        ([[], [0, 0]], [[1], []], "times"),
        # a rank outside the graph
        ([[], [5]], [[1], []], "outside"),
        ([[], [0]], [[-1], []], "outside"),
        # lists of different lengths
        ([[], []], [[]], "lists"),
    ],
)
def test_invalid_graphs_are_refused(src, dst, what):
    with pytest.raises(CommError, match=what):
        neighbor_in_edges(src, dst)


def test_oracle_all_gather_and_all_to_all_keep_the_guards():
    edges = [[(1, 0), (0, 1)], [(0, 0)]]
    # rank 0 sends to 1 then to itself; rank 1 sends to 0
    sends = [u8(1, 2, 3, 4), u8(5, 6)]
    recvs = [u8(0, 0, 0, 0, 0, 0), u8(9, 9, 9, 9)]
    ag = no.neighbor_exchange("neighbor_all_gather", sends, recvs, edges, 2, offset=1)
    assert ag[0].tolist() == [0, 5, 6, 1, 2, 0]
    assert ag[1].tolist() == [9, 1, 2, 9]
    a2a = no.neighbor_exchange("neighbor_all_to_all", sends, recvs, edges, 2, offset=1)
    # rank 0's in-edge (0, 1) takes block 1 of its own send
    assert a2a[0].tolist() == [0, 5, 6, 3, 4, 0]
    assert a2a[1].tolist() == [9, 1, 2, 9]
    # the inputs are not changed
    assert recvs[0].tolist() == [0] * 6


def test_oracle_refuses_a_missing_block_and_counts_staged_bytes():
    with pytest.raises(ValueError):
        no.neighbor_exchange("neighbor_all_to_all", [u8(1, 2)], [u8(0, 0)], [[(0, 1)]], 2)
    # a ring of 3 with 8-byte blocks: 3 staged blocks and 3 pulled, each read
    # and written once
    assert no.staged_bytes("neighbor_all_to_all", [1, 1, 1], [1, 1, 1], 8) == 96
    # the all-gather stages one block per rank with an out-edge
    assert no.staged_bytes("neighbor_all_gather", [2, 0], [1, 1], 8) == 2 * 8 + 2 * 16
