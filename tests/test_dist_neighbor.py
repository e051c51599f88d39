"""The distributed-graph topology and the neighbourhood collectives on the
world and on a split whose members live in different worker PROCESSES: the
`neighbor-coll` function of faabric_worker (csrc/tests/mpi_neighbor_body.h) on
4 workers with one rank each.  The children's heaps and signal pads are peer
mappings into other processes, and the graph gathering and slot agreement
travel over TCP."""

import pytest

from faabric_b200 import build as fb_build
from faabric_b200.runtime import LocalCluster

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _built():
    fb_build.build(verbose=False)


def test_neighbor_collectives_across_processes(tmp_path):
    # The processes share one GPU on a single-GPU machine: cross-rank
    # synchronisation through stream memory operations
    with LocalCluster(
        n_workers=4, slots_per_worker=1, log_dir=tmp_path, extra_env={"FAABRIC_STREAM_SYNC": "1"}
    ) as c:
        st = c.client.invoke("mpi", "neighbor-coll", mpi_world_size=4, timeout=300)
        res = sorted(st.get("messageResults", []), key=lambda m: m.get("mpiRank", 0))
        assert len(res) == 4, res
        assert all(m.get("returnValue", 0) == 0 for m in res), [m.get("output_data") for m in res]
        assert len({m["executedHost"] for m in res}) == 4, res
