// The neighbourhood v-collectives' MPI program (mpi_neighbor_v_body.h) on GPU
// memory, ranks sharing the GPU: 2, 4 and 8 ranks, then 4 with grouping off
#include "fixtures.h"
#include "mpi_neighbor_v_run.h"

namespace {
// Up to 8 ranks share the GPU here and meet at stream-ordered barriers: with
// the default 8 hardware queues, two ranks' streams can land on one queue,
// and a rank's wait then blocks the peer signal queued behind it.  Set before
// the first CUDA call (an explicit setting in the environment wins).
const bool kConnections = setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32", 0) == 0;
}

TEST_CASE("mpi neighbourhood v-collectives on the world and on a split on the GPU", "[gpu][mpi]")
{
    if (!faabric::device::cudaAvailable()) {
        SKIP_TEST("no CUDA device");
    }
    for (int n : { 2, 4, 8 }) {
        runNeighborVMpi("neighbor-v-gpu-" + std::to_string(n), n, true);
    }
    runNeighborVMpi("neighbor-v-gpu-4-ungrouped", 4, false);
}
