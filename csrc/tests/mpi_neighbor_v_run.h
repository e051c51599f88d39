// Runs the MPI program of mpi_neighbor_v_body.h on a local cluster (the loopback
// and GPU tests of the neighbourhood v-collectives)
#pragma once

#include "fixtures.h"
#include "mpi_neighbor_v_body.h"

#include <faabric/executor/ExecutorContext.h>

// The program on `worldSize` ranks of a local cluster (grouped, or with
// FAABRIC_MPI_GROUP_IALLREDUCE=0); every rank must return 0
inline void runNeighborVMpi(const std::string& name, int worldSize, bool grouped)
{
    using namespace tests;
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
        int rc = neighbor_v_coll::body(rank, size, msg.mpiworldid(), grouped, &why);
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
