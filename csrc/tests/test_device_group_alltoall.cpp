// MPI_Ialltoall bursts on GPU memory, on the world and on sub-communicators:
// the program of mpi_group_alltoall_body.h on ranks that share the GPU,
// checked against host-computed results, one grouped launch per burst; and
// once more with grouping off (FAABRIC_MPI_GROUP_IALLREDUCE=0).
#include "fixtures.h"
#include "mpi_group_alltoall_body.h"

#include <faabric/executor/ExecutorContext.h>

using namespace tests;

namespace {
// Up to 8 ranks share the GPU here and meet at stream-ordered barriers: with
// the default 8 hardware queues, two ranks' streams can land on one queue,
// and a rank's wait then blocks the peer signal queued behind it.  Set before
// the first CUDA call, as the Python package does for its processes (an
// explicit setting in the environment wins).
const bool kConnections = setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32", 0) == 0;
}

TEST_CASE("mpi group alltoall bursts on the world and on sub-communicators on the GPU", "[gpu][mpi]")
{
    if (!faabric::device::cudaAvailable()) {
        SKIP_TEST("no CUDA device");
    }
    for (int run = 0; run < 4; run++) {
        // world sizes 2, 4 and 8, then 4 with grouping off
        const int worldSize = run < 3 ? 2 << run : 4;
        const bool grouped = run < 3;
        const std::string name = "group-alltoall-gpu-" + std::to_string(worldSize) + (grouped ? "" : "-ungrouped");
        if (!grouped) {
            setenv("FAABRIC_MPI_GROUP_IALLREDUCE", "0", 1);
        }
        ClusterFixture f(worldSize);
        registerTestFunction("mpi", name, [&](auto*, int, int, auto) {
            MPI_Init(nullptr, nullptr);
            int rank = -1, size = -1;
            MPI_Comm_rank(MPI_COMM_WORLD, &rank);
            MPI_Comm_size(MPI_COMM_WORLD, &size);
            std::string why;
            faabric::Message& msg = faabric::executor::ExecutorContext::get()->getMsg();
            int rc = group_alltoall::body(rank, size, msg.mpiworldid(), grouped, &why);
            if (rc != 0) {
                printf("         %s\n", why.c_str());
                msg.set_outputdata(why);
            }
            MPI_Finalize();
            return rc;
        });
        auto req = faabric::util::batchExecFactory("mpi", name, 1);
        req->mutable_messages(0)->set_ismpi(true);
        req->mutable_messages(0)->set_mpiworldsize(worldSize);
        f.plannerCli.callFunctions(req);
        auto status = f.awaitBatch(req, 120000);
        unsetenv("FAABRIC_MPI_GROUP_IALLREDUCE");
        REQUIRE_EQ(status->messageresults_size(), worldSize);
        for (auto& m : status->messageresults()) {
            if (m.returnvalue() != 0) {
                fbtest::fail(__FILE__, __LINE__, name + ": rank " + std::to_string(m.mpirank()) + " failed: " + m.outputdata());
            }
        }
        faabric::mpi::getMpiWorldRegistry().clear();
    }
}
