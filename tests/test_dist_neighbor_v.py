"""The neighbourhood v-collectives on the world and on a split whose members
live in different worker PROCESSES: the `neighbor-v-coll` function of
faabric_worker (csrc/tests/mpi_neighbor_v_body.h) on 4 workers with one rank
each.  The children's heaps and signal pads are peer mappings into other
processes, and the agreement on every launch's rounds travels over TCP."""

import pytest

from faabric_b200 import build as fb_build
from faabric_b200.runtime import LocalCluster

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _built():
    fb_build.build(verbose=False)


def _logs(tmp_path):
    """The end of every process log of the cluster, for a failure message"""
    out = []
    for f in sorted(tmp_path.glob("*.log")):
        out.append(f"---- {f.name}\n" + "\n".join(f.read_text(errors="replace").splitlines()[-15:]))
    return "\n".join(out)


def test_neighbor_v_collectives_across_processes(tmp_path):
    # The processes share one GPU on a single-GPU machine: cross-rank
    # synchronisation through stream memory operations
    c = LocalCluster(n_workers=4, slots_per_worker=1, log_dir=tmp_path, extra_env={"FAABRIC_STREAM_SYNC": "1"})
    try:
        try:
            c.start()
        except RuntimeError as e:
            raise AssertionError(f"{e}\n{_logs(tmp_path)}") from e
        st = c.client.invoke("mpi", "neighbor-v-coll", mpi_world_size=4, timeout=300)
        res = sorted(st.get("messageResults", []), key=lambda m: m.get("mpiRank", 0))
        assert len(res) == 4, res
        assert all(m.get("returnValue", 0) == 0 for m in res), [m.get("output_data") for m in res]
        assert len({m["executedHost"] for m in res}) == 4, res
    finally:
        c.stop()
