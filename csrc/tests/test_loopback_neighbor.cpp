// The neighbourhood collectives' MPI program (mpi_neighbor_body.h) on the
// loopback backend at 2 and 4 ranks, grouped and with grouping off at 4
#include "fixtures.h"
#include "mpi_neighbor_run.h"

TEST_CASE("loopback MPI neighbourhood collectives on the world and on a split", "[loopback][mpi]")
{
    tests::LoopbackBackend loopback;
    runNeighborMpi("neighbor-loopback-2", 2, true);
    runNeighborMpi("neighbor-loopback-4", 4, true);
    runNeighborMpi("neighbor-loopback-4-ungrouped", 4, false);
}
