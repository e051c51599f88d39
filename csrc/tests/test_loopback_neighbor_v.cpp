// The neighbourhood v-collectives' MPI program (mpi_neighbor_v_body.h) on the
// loopback backend at 2 and 4 ranks, grouped and with grouping off at 4
#include "fixtures.h"
#include "mpi_neighbor_v_run.h"

TEST_CASE("loopback MPI neighbourhood v-collectives on the world and on a split", "[loopback][mpi]")
{
    tests::LoopbackBackend loopback;
    runNeighborVMpi("neighbor-v-loopback-2", 2, true);
    runNeighborVMpi("neighbor-v-loopback-4", 4, true);
    runNeighborVMpi("neighbor-v-loopback-4-ungrouped", 4, false);
}
