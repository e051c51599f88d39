// MPI_Raccumulate / MPI_Rget_accumulate deferred into the request batch of a
// symmetric-heap window (Communicator::accumulateMany); the program is in
// mpi_rma_accumulate_batch_body.h.
#include "fixtures.h"
#include "mpi_rma_accumulate_batch_body.h"

#include <faabric/executor/ExecutorContext.h>

using namespace tests;
using rma_request::Origin;

namespace {

void runBatch(const std::string& name, int worldSize, Origin origin)
{
    ClusterFixture f(worldSize);
    registerTestFunction("mpi", name, [&](auto*, int, int, auto) {
        MPI_Init(nullptr, nullptr);
        int rank = -1, size = -1;
        MPI_Comm_rank(MPI_COMM_WORLD, &rank);
        MPI_Comm_size(MPI_COMM_WORLD, &size);
        std::string why;
        faabric::Message& msg = faabric::executor::ExecutorContext::get()->getMsg();
        int rc = rma_acc_batch::body(rank, size, msg.mpiworldid(), origin, &why);
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
    auto status = f.awaitBatch(req, 180000);
    REQUIRE_EQ(status->messageresults_size(), worldSize);
    for (auto& m : status->messageresults()) {
        if (m.returnvalue() != 0) {
            fbtest::fail(__FILE__, __LINE__, name + ": rank " + std::to_string(m.mpirank()) + " failed: " + m.outputdata());
        }
    }
    faabric::mpi::getMpiWorldRegistry().clear();
}
}

TEST_CASE("mpi rma accumulate batch: symmetric-heap windows (loopback)", "[mpi][rma][loopback]")
{
    LoopbackBackend loopback;
    runBatch("rma-acc-batch-loopback-2", 2, Origin::Heap);
    runBatch("rma-acc-batch-loopback-4", 4, Origin::Heap);
}

TEST_CASE("mpi rma accumulate batch on the GPU: symmetric-heap windows", "[gpu][mpi][rma]")
{
    if (!faabric::device::cudaAvailable()) {
        SKIP_TEST("no CUDA device");
    }
    for (int n : { 2, 4, 8 }) {
        const std::string sz = std::to_string(n);
        runBatch("rma-acc-batch-dev-" + sz, n, Origin::Device);
        runBatch("rma-acc-batch-heap-" + sz, n, Origin::Heap);
    }
}
