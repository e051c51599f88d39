"""Fused device collectives on sub-communicators whose members live in
different worker PROCESSES: the `subcomm-device` function of faabric_worker
(csrc/tests/mpi_subcomm_device_body.h) on 3 workers with one rank each, so the
world's device communicator is wired over IPC, every child's heap and signal
slot pointers are peer mappings into other processes, and the slot agreement
travels over TCP."""

import pytest

from faabric_b200 import build as fb_build
from faabric_b200.runtime import LocalCluster

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _built():
    fb_build.build(verbose=False)


@pytest.mark.parametrize("memory", ["heap", "cuda"])
def test_subcomm_device_across_processes(tmp_path, memory):
    # The three processes share one GPU on a single-GPU machine: cross-rank
    # synchronisation through stream memory operations, as for ranks of one
    # process that share a device
    with LocalCluster(
        n_workers=3, slots_per_worker=1, log_dir=tmp_path, extra_env={"FAABRIC_STREAM_SYNC": "1"}
    ) as c:
        st = c.client.invoke("mpi", "subcomm-device", mpi_world_size=3, input_data=memory, timeout=300)
        res = sorted(st.get("messageResults", []), key=lambda m: m.get("mpiRank", 0))
        assert len(res) == 3, res
        assert all(m.get("returnValue", 0) == 0 for m in res), [m.get("output_data") for m in res]
        assert len({m["executedHost"] for m in res}) == 3, res
