"""MPI passive-target synchronisation across worker PROCESSES: the
`rma-passive` function of faabric_worker (csrc/tests/mpi_rma_passive_body.h).
Locks of a target live in its process; lock, flush and unlock requests of
origins in other processes go to that process's point-to-point server, which
applies shipped operations without a fence."""

import pytest

from faabric_b200 import build as fb_build
from faabric_b200.runtime import LocalCluster


@pytest.fixture(scope="module", autouse=True)
def _built():
    fb_build.build(verbose=False)


def _run(c, world_size, payload, n_hosts):
    st = c.client.invoke("mpi", "rma-passive", mpi_world_size=world_size, input_data=payload, timeout=300)
    res = sorted(st.get("messageResults", []), key=lambda m: m.get("mpiRank", 0))
    assert len(res) == world_size, res
    assert all(m.get("returnValue", 0) == 0 for m in res), [m.get("output_data") for m in res]
    assert len({m["executedHost"] for m in res}) == n_hosts, res


@pytest.mark.parametrize("n_workers", [2, 3])
def test_passive_target_on_host_windows_across_workers(tmp_path, n_workers):
    with LocalCluster(n_workers=n_workers, slots_per_worker=2, log_dir=tmp_path) as c:
        _run(c, 2 * n_workers, "host", n_workers)
        # a second world in the same workers: the first one's windows and
        # locks are gone, nothing of it answers for the new one
        _run(c, 2 * n_workers, "host", n_workers)


@pytest.mark.gpu
def test_passive_target_on_device_windows_across_workers(tmp_path):
    # cudaMalloc windows, 2 processes x 2 ranks sharing the GPU: the pointer
    # kernel serves every segment, shipped operations included
    with LocalCluster(n_workers=2, slots_per_worker=2, log_dir=tmp_path / "cuda") as c:
        _run(c, 4, "cuda,device", 2)
        _run(c, 4, "cuda", 2)
    # symmetric-heap windows, 2 processes x 1 rank: each target applies what
    # it is shipped through its own communicator, on the server's stream
    with LocalCluster(n_workers=2, slots_per_worker=1, log_dir=tmp_path / "heap") as c:
        _run(c, 2, "heap,device", 2)
        _run(c, 2, "heap", 2)
