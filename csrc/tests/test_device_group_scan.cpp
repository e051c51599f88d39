// MPI_Iscan and MPI_Iexscan bursts and MPI_Exscan on GPU memory, on the world
// and on sub-communicators: the program of mpi_group_scan_body.h on ranks that
// share the GPU, checked against host-computed results, one grouped launch
// per burst; and once more with grouping off (FAABRIC_MPI_GROUP_IALLREDUCE=0).
#include "fixtures.h"
#include "mpi_group_scan_run.h"

namespace {
// Up to 8 ranks share the GPU here and meet at stream-ordered barriers: with
// the default 8 hardware queues, two ranks' streams can land on one queue,
// and a rank's wait then blocks the peer signal queued behind it.  Set before
// the first CUDA call (an explicit setting in the environment wins).
const bool kConnections = setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32", 0) == 0;
}

TEST_CASE("mpi group scan bursts on the world and on sub-communicators on the GPU", "[gpu][mpi]")
{
    if (!faabric::device::cudaAvailable()) {
        SKIP_TEST("no CUDA device");
    }
    runMpiGroupScanBody(false);
}
