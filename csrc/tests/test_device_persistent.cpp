// Persistent collectives (MPI_*_init, MPI_Start, MPI_Startall) on GPU memory,
// on the world and on sub-communicators: the program of mpi_persistent_body.h
// on 2, 4 and 8 ranks that share the GPU, then 4 ranks with grouping off
// (FAABRIC_MPI_GROUP_IALLREDUCE=0).
#include "fixtures.h"
#include "mpi_persistent_run.h"

namespace {
// Up to 8 ranks share the GPU here and meet at stream-ordered barriers: with
// the default 8 hardware queues, two ranks' streams can land on one queue,
// and a rank's wait then blocks the peer signal queued behind it.  Set before
// the first CUDA call (an explicit setting in the environment wins).
const bool kConnections = setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32", 0) == 0;
}

TEST_CASE("mpi persistent collectives on the world and on sub-communicators on the GPU", "[gpu][mpi]")
{
    if (!faabric::device::cudaAvailable()) {
        SKIP_TEST("no CUDA device");
    }
    for (int worldSize : { 2, 4, 8 }) {
        runPersistentMpi("persistent-gpu-" + std::to_string(worldSize), worldSize, true, true);
    }
    runPersistentMpi("persistent-gpu-4-ungrouped", 4, false, true);
}
