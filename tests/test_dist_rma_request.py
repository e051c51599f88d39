"""Request-based one-sided operations across worker PROCESSES: the
`rma-request` function of faabric_worker (csrc/tests/mpi_rma_request_body.h).
MPI_Rput, MPI_Rget, MPI_Raccumulate and MPI_Rget_accumulate to a rank in
another process are queued like MPI_Put and shipped at the flush or unlock of
the target, or at the wait of the request; a wait after the unlock, and a
request freed before the unlock, complete without shipping anything twice."""

import pytest

from faabric_b200 import build as fb_build
from faabric_b200.runtime import LocalCluster


@pytest.fixture(scope="module", autouse=True)
def _built():
    fb_build.build(verbose=False)


def _run(c, world_size, payload, n_hosts):
    st = c.client.invoke("mpi", "rma-request", mpi_world_size=world_size, input_data=payload, timeout=300)
    res = sorted(st.get("messageResults", []), key=lambda m: m.get("mpiRank", 0))
    assert len(res) == world_size, res
    assert all(m.get("returnValue", 0) == 0 for m in res), [m.get("output_data") for m in res]
    assert len({m["executedHost"] for m in res}) == n_hosts, res


@pytest.mark.parametrize("n_workers", [2, 3])
def test_request_based_operations_on_host_windows_across_workers(tmp_path, n_workers):
    with LocalCluster(n_workers=n_workers, slots_per_worker=2, log_dir=tmp_path) as c:
        _run(c, 2 * n_workers, "host", n_workers)
        # a second world in the same workers: nothing of the first one's
        # windows or request sequences answers for it
        _run(c, 2 * n_workers, "host", n_workers)


@pytest.mark.gpu
def test_request_based_operations_on_device_windows_across_workers(tmp_path):
    # cudaMalloc windows, 2 processes x 2 ranks sharing the GPU
    with LocalCluster(n_workers=2, slots_per_worker=2, log_dir=tmp_path / "cuda") as c:
        _run(c, 4, "cuda,device", 2)
        _run(c, 4, "cuda", 2)
    # symmetric-heap windows, 2 processes x 1 rank (a heap spans the ranks of
    # one process): the target in this process (the rank itself) takes the
    # batched copies, the one in the other process is shipped
    with LocalCluster(n_workers=2, slots_per_worker=1, log_dir=tmp_path / "heap") as c:
        _run(c, 2, "heap,device", 2)
        _run(c, 2, "heap,heapbuf", 2)
        _run(c, 2, "heap", 2)
