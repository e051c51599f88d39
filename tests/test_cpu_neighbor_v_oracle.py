"""The neighbourhood v oracle (neighbor_v_oracle) on graphs worked by hand,
with no GPU: self-edges, multi-edges, zero counts, a member of degree 0, and
the launch counts of the device path."""

import numpy as np
import pytest

import neighbor_v_oracle as nv

from faabric_b200.parallel.comm import neighbor_in_edges


def test_allgatherv_by_hand():
    # 0 -> 1, 0 -> 2, 1 -> 0, 1 -> 1 (self); rank 2 sends nothing
    src = [[1], [0, 1], [0]]
    dst = [[1, 2], [0, 1], []]
    edges = neighbor_in_edges(src, dst)
    sends = [np.array([10, 11, 12]), np.array([20, 21]), np.array([], dtype=np.int64)]
    recvs = [np.full(4, -1), np.full(6, -1), np.full(3, -1)]
    out = nv.neighbor_exchange_v(
        "neighbor_all_gather_v", sends, recvs, edges, recvcounts=[[2], [3, 2], [3]], rdispls=[[1], [0, 4], [0]]
    )
    assert out[0].tolist() == [-1, 20, 21, -1]
    assert out[1].tolist() == [10, 11, 12, -1, 20, 21]
    assert out[2].tolist() == [10, 11, 12]


def test_alltoallv_by_hand_with_multi_edges_and_zero_counts():
    # 0 sends twice to 1 (a multi-edge) and once to itself; 1 sends to 0
    src = [[0, 1], [0, 0], []]
    dst = [[1, 0, 1], [0], []]
    edges = neighbor_in_edges(src, dst)
    assert edges == [[(0, 1), (1, 0)], [(0, 0), (0, 2)], []]
    sends = [np.array([1, 2, 3, 4, 5]), np.array([7, 8]), np.array([], dtype=np.int64)]
    sendcounts = [[2, 1, 0], [2], []]
    sdispls = [[0, 4, 2], [0], []]
    recvs = [np.zeros(4, dtype=np.int64), np.zeros(3, dtype=np.int64), np.zeros(1, dtype=np.int64)]
    out = nv.neighbor_exchange_v(
        "neighbor_all_to_all_v",
        sends,
        recvs,
        edges,
        recvcounts=[[1, 2], [2, 0], []],
        rdispls=[[3, 0], [1, 0], []],
        sendcounts=sendcounts,
        sdispls=sdispls,
    )
    assert out[0].tolist() == [7, 8, 0, 5]
    assert out[1].tolist() == [0, 1, 2]
    assert out[2].tolist() == [0]


def test_mismatched_counts_are_refused():
    edges = neighbor_in_edges([[1], [0]], [[1], [0]])
    with pytest.raises(ValueError):
        nv.neighbor_exchange_v(
            "neighbor_all_to_all_v",
            [np.zeros(2), np.zeros(2)],
            [np.zeros(2), np.zeros(2)],
            edges,
            recvcounts=[[2], [1]],
            rdispls=[[0], [0]],
            sendcounts=[[2], [2]],
            sdispls=[[0], [0]],
        )


def test_stream_lengths_and_launches():
    # two items; out-edges 0, 1 and one in-edge, 4-byte elements
    lens = nv.stream_lengths("neighbor_all_to_all_v", 2, 1, [[3, 0], [5, 1]], [[2], [7]], 4)
    assert lens == [32, 4, 36]
    assert nv.stream_lengths("neighbor_all_gather_v", 2, 0, [[3], [5]], [], 4) == [32]
    assert nv.stream_lengths("neighbor_all_gather_v", 0, 1, [[0], [0]], [[1], [2]], 1) == [3]
    # a window of 0 bytes launches nothing; one within a chunk once
    assert nv.launches([0, 1, 2048], 1 << 20, 3, "neighbor_all_to_all_v") == 2
    # 64 KiB staging over 4 slots: 16 KiB per slot, so 40000 bytes take 3
    assert nv.launches([40000], 1 << 16, 4, "neighbor_all_to_all_v") == 3
    assert nv.launches([40000], 1 << 16, 4, "neighbor_all_gather_v") == 1
