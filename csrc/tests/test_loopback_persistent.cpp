// Persistent collectives (MPI_*_init, MPI_Start, MPI_Startall) on the loopback
// backend (no GPU): the program of mpi_persistent_body.h at 2 and 4 ranks,
// then 4 ranks with grouping off (FAABRIC_MPI_GROUP_IALLREDUCE=0).
#include "fixtures.h"
#include "mpi_persistent_run.h"

TEST_CASE("loopback persistent collectives on the world and on sub-communicators", "[loopback][mpi]")
{
    tests::LoopbackBackend loopback;
    runPersistentMpi("persistent-loopback-2", 2, true, false);
    runPersistentMpi("persistent-loopback-4", 4, true, false);
    runPersistentMpi("persistent-loopback-4-ungrouped", 4, false, false);
}
