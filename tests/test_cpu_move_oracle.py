"""The data-movement oracle (tests/move_oracle.py) against hand-worked cases,
so that the GPU tests compare the kernels with something known right."""

import numpy as np
import pytest

import move_oracle as mo


def u8(*v):
    return np.array(v, dtype=np.uint8)


def test_place_and_payload_touch_only_the_payload():
    buf = u8(9, 9, 9, 9, 9)
    out = mo.place(buf, 1, u8(1, 2))
    assert out.tolist() == [9, 1, 2, 9, 9]
    assert buf.tolist() == [9, 9, 9, 9, 9]  # the input is not modified
    assert mo.payload(out, 1, 3).tolist() == [1, 2, 9]
    with pytest.raises(ValueError):
        mo.place(buf, 4, u8(1, 2))
    with pytest.raises(TypeError):
        mo.place(np.zeros(4, np.int32), 0, u8(1))


def test_all_gather_concatenates_in_rank_order_at_each_ranks_offset():
    # rank 0 sends [1, 2] at offset 1, rank 1 sends [3, 4] at offset 0
    sends = [u8(0, 1, 2), u8(3, 4, 0)]
    recvs = [u8(7, 7, 7, 7, 7, 7), u8(8, 8, 8, 8, 8, 8)]
    out = mo.all_gather(sends, [1, 0], recvs, [0, 2], 2)
    assert out[0].tolist() == [1, 2, 3, 4, 7, 7]
    assert out[1].tolist() == [8, 8, 1, 2, 3, 4]


def test_gather_writes_the_root_only():
    sends = [u8(1), u8(2), u8(3)]
    recvs = [u8(0, 0, 0, 0), u8(5, 5, 5, 5), None]
    out = mo.gather(sends, [0, 0, 0], recvs, [1, 0, 0], 1, root=0)
    assert out[0].tolist() == [0, 1, 2, 3]
    assert out[1].tolist() == [5, 5, 5, 5]
    assert out[2] is None
    out = mo.gather(sends, [0, 0, 0], recvs, [0, 1, 0], 1, root=1)
    assert out[0].tolist() == [0, 0, 0, 0] and out[1].tolist() == [5, 1, 2, 3]


def test_scatter_reads_the_roots_send_buffer_only():
    # per = 2, n = 2: the root (rank 1) holds [10, 11 | 12, 13] at offset 1
    sends = [u8(99, 99, 99, 99, 99), u8(0, 10, 11, 12, 13)]
    recvs = [u8(6, 6, 6), u8(6, 6, 6)]
    out = mo.scatter(sends, [0, 1], recvs, [0, 1], 2, root=1)
    assert out[0].tolist() == [10, 11, 6]
    assert out[1].tolist() == [6, 12, 13]


def test_all_to_all_transposes_blocks():
    # n = 3, per = 1: rank p sends [10p, 10p + 1, 10p + 2]
    sends = [u8(0, 1, 2), u8(10, 11, 12), u8(20, 21, 22)]
    recvs = [u8(0, 0, 0, 0) for _ in range(3)]
    out = mo.all_to_all(sends, [0, 0, 0], recvs, [0, 1, 0], 1)
    assert out[0].tolist() == [0, 10, 20, 0]
    assert out[1].tolist() == [0, 1, 11, 21]
    assert out[2].tolist() == [2, 12, 22, 0]


def test_broadcast_copies_the_roots_payload_and_leaves_the_root_alone():
    bufs = [u8(1, 2, 3, 4), u8(5, 6, 7, 8), u8(9, 9, 9, 9)]
    # the root's payload is [6, 7], at offset 1
    out = mo.broadcast(bufs, [0, 1, 2], 2, root=1)
    assert out[0].tolist() == [6, 7, 3, 4]
    assert out[1].tolist() == [5, 6, 7, 8]
    assert out[2].tolist() == [9, 9, 6, 7]


def test_collective_dispatch_and_zero_bytes():
    sends = [u8(1, 2), u8(3, 4)]
    recvs = [u8(0, 0, 0, 0), u8(0, 0, 0, 0)]
    assert [b.tolist() for b in mo.collective("all_gather", sends, [0, 0], recvs, [0, 0], 2)] == [[1, 2, 3, 4]] * 2
    assert [b.tolist() for b in mo.collective("broadcast", None, None, recvs, [0, 0], 0, root=1)] == [[0, 0, 0, 0]] * 2
    with pytest.raises(ValueError):
        mo.collective("reduce", sends, [0, 0], recvs, [0, 0], 2)


def test_send_recv_ring_and_untouched_sends():
    sends = [u8(1, 2, 3), u8(4, 5, 6), u8(7, 8, 9)]
    recvs = [u8(0, 0, 0), u8(0, 0, 0), u8(0, 0, 0)]
    # rank r receives from r - 1, payload of 2 bytes at send offset 1
    out = mo.send_recv(sends, [1, 1, 1], recvs, [0, 1, 0], 2, lambda r: (r - 1) % 3)
    assert out[0].tolist() == [8, 9, 0]
    assert out[1].tolist() == [0, 2, 3]
    assert out[2].tolist() == [5, 6, 0]
    kept = mo.untouched(sends)
    assert [k.tolist() for k in kept] == [s.tolist() for s in sends] and kept[0] is not sends[0]


def test_first_difference():
    assert mo.first_difference(u8(1, 2, 3), u8(1, 2, 3)) is None
    assert mo.first_difference(u8(1, 2, 3), u8(1, 0, 3)) == 1
    assert mo.first_difference(u8(1, 2), u8(1, 2, 3)) == 2
