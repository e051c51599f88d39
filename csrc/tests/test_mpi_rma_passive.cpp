// Passive-target synchronisation (MPI_Win_lock, MPI_Win_flush and friends) on
// every kind of window segment of an in-process world; the program is in
// mpi_rma_passive_body.h.
#include "fixtures.h"
#include "mpi_rma_passive_body.h"

#include <faabric/executor/ExecutorContext.h>

using namespace tests;
using rma_passive::Setup;
using rma_passive::WindowMemory;

namespace {

#define NEED_GPU()                                                             \
    do {                                                                       \
        if (!faabric::device::cudaAvailable()) {                               \
            SKIP_TEST("no CUDA device");                                       \
        }                                                                      \
    } while (0)

void runPassive(const std::string& name, int worldSize, const Setup& s)
{
    ClusterFixture f(worldSize);
    registerTestFunction("mpi", name, [&](auto*, int, int, auto) {
        MPI_Init(nullptr, nullptr);
        int rank = -1, size = -1;
        MPI_Comm_rank(MPI_COMM_WORLD, &rank);
        MPI_Comm_size(MPI_COMM_WORLD, &size);
        std::string why;
        faabric::Message& msg = faabric::executor::ExecutorContext::get()->getMsg();
        int rc = rma_passive::body(rank, size, msg.mpiworldid(), s, &why);
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

// 2 and 4 ranks sharing the GPU, and one rank per GPU when there are several
std::vector<int> gpuWorldSizes()
{
    std::vector<int> sizes{ 2, 4 };
    const int gpus = faabric::device::cudaDeviceCountSafe();
    if (gpus > 1) {
        sizes.push_back(gpus);
    }
    return sizes;
}
}

TEST_CASE("mpi rma passive: host windows, exclusion, tickets, flush visibility, shared locks, errors", "[mpi][rma]")
{
    runPassive("rma-passive-host-2", 2, Setup{ WindowMemory::Host, false, false });
    runPassive("rma-passive-host-4", 4, Setup{ WindowMemory::Host, false, false });
}

TEST_CASE("mpi rma passive: symmetric-heap windows (loopback)", "[mpi][rma][loopback]")
{
    LoopbackBackend loopback;
    runPassive("rma-passive-heap-loopback", 4, Setup{ WindowMemory::Heap, false, false });
}

TEST_CASE("mpi rma passive on the GPU: symmetric-heap windows", "[gpu][mpi][rma]")
{
    NEED_GPU();
    for (int n : gpuWorldSizes()) {
        runPassive("rma-passive-heap-" + std::to_string(n), n, Setup{ WindowMemory::Heap, true, false });
        runPassive("rma-passive-heap-hostbuf-" + std::to_string(n), n, Setup{ WindowMemory::Heap, false, false });
    }
}

TEST_CASE("mpi rma passive on the GPU: cudaMalloc windows", "[gpu][mpi][rma]")
{
    NEED_GPU();
    for (int n : gpuWorldSizes()) {
        runPassive("rma-passive-cuda-" + std::to_string(n), n, Setup{ WindowMemory::CudaMalloc, true, false });
        runPassive("rma-passive-cuda-hostbuf-" + std::to_string(n), n, Setup{ WindowMemory::CudaMalloc, false, false });
    }
}

TEST_CASE("mpi rma passive on the GPU: host windows with device buffers", "[gpu][mpi][rma]")
{
    NEED_GPU();
    for (int n : gpuWorldSizes()) {
        runPassive("rma-passive-hostwin-" + std::to_string(n), n, Setup{ WindowMemory::Host, true, false });
    }
}
