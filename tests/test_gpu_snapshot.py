"""Device snapshot kernels on hand-picked values with closed-form results.
The bit-exact matrix against ``snapshot_oracle`` is test_gpu_snapshot_matrix.py."""

import numpy as np
import pytest
import torch

import snapshot_oracle as so
from faabric_b200.ops import snapshot as snap

pytestmark = pytest.mark.gpu

PAGE = 4096


def dev(a):
    return torch.from_numpy(a.copy()).cuda()


def test_typed_regions_and_update_base():
    size = PAGE * 4
    rng = np.random.default_rng(7)
    orig = rng.integers(0, 256, size, dtype=np.uint8)
    mem = orig.copy()
    main = orig.copy()

    def put(arr, off, val, t):
        arr[off : off + np.dtype(t).itemsize] = np.array([val], dtype=t).view(np.uint8)

    R = snap.MergeRegion
    regions = [
        R(64, 4, snap.INT, snap.SUM),
        R(128, 8, snap.LONG, snap.MAX),
        R(256, 4, snap.FLOAT, snap.MIN),
        R(512, 8, snap.DOUBLE, snap.SUM),
        R(1024, 4, snap.INT, snap.SUBTRACT),
        R(2048, 16, snap.INT, snap.SUM),  # array of 4 ints
        R(3000, 100, snap.RAW, snap.IGNORE),
        R(PAGE + 3, 8, snap.DOUBLE, snap.PRODUCT),  # unaligned scalar
        R(PAGE * 2, 4, snap.FLOAT, snap.PRODUCT),
    ]
    put(orig, 64, 10, np.int32), put(mem, 64, 17, np.int32), put(main, 64, 100, np.int32)
    put(orig, 128, 5, np.int64), put(mem, 128, 99, np.int64), put(main, 128, 50, np.int64)
    put(orig, 256, 2.0, np.float32), put(mem, 256, -3.5, np.float32), put(main, 256, 1.0, np.float32)
    put(orig, 512, 1.5, np.float64), put(mem, 512, 4.0, np.float64), put(main, 512, 10.0, np.float64)
    put(orig, 1024, 30, np.int32), put(mem, 1024, 20, np.int32), put(main, 1024, 7, np.int32)
    for k in range(4):
        put(orig, 2048 + 4 * k, k, np.int32), put(mem, 2048 + 4 * k, k * 3, np.int32), put(main, 2048 + 4 * k, 1000, np.int32)
    mem[3000:3100] ^= 0xFF  # ignored
    put(orig, PAGE + 3, 2.0, np.float64), put(mem, PAGE + 3, 6.0, np.float64), put(main, PAGE + 3, 5.0, np.float64)
    put(orig, PAGE * 2, 4.0, np.float32), put(mem, PAGE * 2, 2.0, np.float32), put(main, PAGE * 2, 8.0, np.float32)
    mem[PAGE * 3 + 10] ^= 0x11  # bytewise gap

    regs = snap.prepare_regions(regions, size, "cuda")
    d_mem, d_orig, d_main = dev(mem), dev(orig), dev(main)
    snap.diff_push(d_mem, d_orig, d_main, regs, update_base=True)
    torch.cuda.synchronize()
    res = so.merge(orig, mem, main, [so.Region(r.offset, r.length, r.data_type, r.op) for r in regs.host])
    got = d_main.cpu().numpy()
    assert np.array_equal(got, res.main)
    assert got[64:68].view(np.int32)[0] == 107
    assert got[128:136].view(np.int64)[0] == 99
    assert got[512:520].view(np.float64)[0] == 12.5
    assert got[1024:1028].view(np.int32)[0] == -3
    assert got[2048:2064].view(np.int32).tolist() == [1000, 1002, 1004, 1006]  # every scalar of the array
    assert got[PAGE + 3 : PAGE + 11].view(np.float64)[0] == 15.0
    assert got[PAGE * 2 : PAGE * 2 + 4].view(np.float32)[0] == 4.0
    # update_base folded the changes into the base everywhere except Ignore
    base = d_orig.cpu().numpy()
    keep = np.ones(size, dtype=bool)
    keep[3000:3100] = False
    assert np.array_equal(base[keep], mem[keep])
    assert np.array_equal(base[3000:3100], orig[3000:3100])
    # second pass: nothing left to push
    stats = snap.diff_push(d_mem, d_orig, d_main, regs)
    torch.cuda.synchronize()
    assert int(stats[0].item()) == 0


def test_apply_diffs():
    size = 10000
    img = np.zeros(size, dtype=np.uint8)
    img[100:104] = np.array([10], dtype=np.int32).view(np.uint8)
    img[200:208] = np.array([2.5], dtype=np.float64).view(np.uint8)
    d_img = dev(img)
    diffs = [
        (10, snap.RAW, snap.BYTEWISE, bytes([1, 2, 3])),
        (50, snap.RAW, snap.XOR, bytes([0xFF, 0x0F])),
        (100, snap.INT, snap.SUM, np.array([5], dtype=np.int32).tobytes()),
        (200, snap.DOUBLE, snap.PRODUCT, np.array([4.0], dtype=np.float64).tobytes()),
        (300, snap.INT, snap.MAX, np.array([-3], dtype=np.int32).tobytes()),
        (400, snap.RAW, snap.IGNORE, bytes([9, 9])),
    ]
    snap.apply_diffs(d_img, diffs)
    torch.cuda.synchronize()
    got = d_img.cpu().numpy()
    assert got[10:13].tolist() == [1, 2, 3]
    assert got[50:52].tolist() == [0xFF, 0x0F]
    assert got[100:104].view(np.int32)[0] == 15
    assert got[200:208].view(np.float64)[0] == 10.0
    assert got[300:304].view(np.int32)[0] == 0
    assert got[400:402].tolist() == [0, 0]
