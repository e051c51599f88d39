// Request-based one-sided operations (MPI_Rput, MPI_Rget, MPI_Raccumulate,
// MPI_Rget_accumulate) on every kind of window segment of an in-process
// world, with host, device and heap origin buffers; the program is in
// mpi_rma_request_body.h.
#include "fixtures.h"
#include "mpi_rma_request_body.h"

#include <faabric/executor/ExecutorContext.h>

using namespace tests;
using rma_request::Origin;
using rma_request::Setup;
using rma_request::WindowMemory;

namespace {

#define NEED_GPU()                                                             \
    do {                                                                       \
        if (!faabric::device::cudaAvailable()) {                               \
            SKIP_TEST("no CUDA device");                                       \
        }                                                                      \
    } while (0)

void runRequest(const std::string& name, int worldSize, const Setup& s)
{
    ClusterFixture f(worldSize);
    registerTestFunction("mpi", name, [&](auto*, int, int, auto) {
        MPI_Init(nullptr, nullptr);
        int rank = -1, size = -1;
        MPI_Comm_rank(MPI_COMM_WORLD, &rank);
        MPI_Comm_size(MPI_COMM_WORLD, &size);
        std::string why;
        faabric::Message& msg = faabric::executor::ExecutorContext::get()->getMsg();
        int rc = rma_request::body(rank, size, msg.mpiworldid(), s, &why);
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

TEST_CASE("mpi rma request: host windows", "[mpi][rma]")
{
    runRequest("rma-request-host-2", 2, Setup{ WindowMemory::Host, Origin::Host });
    runRequest("rma-request-host-3", 3, Setup{ WindowMemory::Host, Origin::Host });
}

TEST_CASE("mpi rma request: symmetric-heap windows (loopback), batched and host origins", "[mpi][rma][loopback]")
{
    LoopbackBackend loopback;
    runRequest("rma-request-heap-loopback-batched", 4, Setup{ WindowMemory::Heap, Origin::Heap, true });
    runRequest("rma-request-heap-loopback-batched-3", 3, Setup{ WindowMemory::Heap, Origin::Heap, true });
    runRequest("rma-request-heap-loopback-host", 2, Setup{ WindowMemory::Heap, Origin::Host });
}

TEST_CASE("mpi rma request on the GPU: symmetric-heap windows", "[gpu][mpi][rma]")
{
    NEED_GPU();
    for (int n : { 2, 4, 8 }) {
        const std::string sz = std::to_string(n);
        runRequest("rma-request-heap-dev-" + sz, n, Setup{ WindowMemory::Heap, Origin::Device, true });
        runRequest("rma-request-heap-heap-" + sz, n, Setup{ WindowMemory::Heap, Origin::Heap, true });
        runRequest("rma-request-heap-host-" + sz, n, Setup{ WindowMemory::Heap, Origin::Host });
    }
}

TEST_CASE("mpi rma request on the GPU: cudaMalloc and host windows", "[gpu][mpi][rma]")
{
    NEED_GPU();
    for (int n : { 2, 4, 8 }) {
        const std::string sz = std::to_string(n);
        runRequest("rma-request-cuda-dev-" + sz, n, Setup{ WindowMemory::CudaMalloc, Origin::Device });
        runRequest("rma-request-cuda-host-" + sz, n, Setup{ WindowMemory::CudaMalloc, Origin::Host });
        runRequest("rma-request-hostwin-dev-" + sz, n, Setup{ WindowMemory::Host, Origin::Device });
    }
}
