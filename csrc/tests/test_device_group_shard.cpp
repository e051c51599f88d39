// MPI_Ireduce_scatter_block and MPI_Iallgather bursts on GPU memory: the
// program of mpi_group_shard_body.h on ranks that share the GPU, checked
// against host-computed results, one grouped launch per burst.
#include "fixtures.h"
#include "mpi_group_shard_body.h"

#include <faabric/executor/ExecutorContext.h>

using namespace tests;

TEST_CASE("mpi grouped reduce-scatter and all-gather bursts on the GPU", "[gpu][mpi]")
{
    if (!faabric::device::cudaAvailable()) {
        SKIP_TEST("no CUDA device");
    }
    for (int worldSize : { 2, 4 }) {
        const std::string name = "group-shard-gpu-" + std::to_string(worldSize);
        ClusterFixture f(worldSize);
        registerTestFunction("mpi", name, [&](auto*, int, int, auto) {
            MPI_Init(nullptr, nullptr);
            int rank = -1, size = -1;
            MPI_Comm_rank(MPI_COMM_WORLD, &rank);
            MPI_Comm_size(MPI_COMM_WORLD, &size);
            std::string why;
            faabric::Message& msg = faabric::executor::ExecutorContext::get()->getMsg();
            int rc = group_shard::body(rank, size, msg.mpiworldid(), &why);
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
        REQUIRE_EQ(status->messageresults_size(), worldSize);
        for (auto& m : status->messageresults()) {
            if (m.returnvalue() != 0) {
                fbtest::fail(__FILE__, __LINE__, name + ": rank " + std::to_string(m.mpirank()) + " failed: " + m.outputdata());
            }
        }
        faabric::mpi::getMpiWorldRegistry().clear();
    }
}
