// MPI_Accumulate, MPI_Get_accumulate, MPI_Fetch_and_op and MPI_Compare_and_swap
// on every kind of window segment of an in-process world (the body is in
// mpi_rma_atomics_body.h), and the collectives' refusal of MPI_REPLACE and
// MPI_NO_OP.
#include "fixtures.h"
#include "mpi_rma_atomics_body.h"

#include <faabric/executor/ExecutorContext.h>

using namespace tests;
using rma_atomics::Setup;
using rma_atomics::WindowMemory;

namespace {

#define NEED_GPU()                                                             \
    do {                                                                       \
        if (!faabric::device::cudaAvailable()) {                               \
            SKIP_TEST("no CUDA device");                                       \
        }                                                                      \
    } while (0)

void runWorld(const std::string& name, int worldSize, const std::function<int(int, int, int, std::string*)>& body)
{
    ClusterFixture f(worldSize);
    registerTestFunction("mpi", name, [&](auto*, int, int, auto) {
        MPI_Init(nullptr, nullptr);
        int rank = -1, size = -1;
        MPI_Comm_rank(MPI_COMM_WORLD, &rank);
        MPI_Comm_size(MPI_COMM_WORLD, &size);
        std::string why;
        faabric::Message& msg = faabric::executor::ExecutorContext::get()->getMsg();
        int rc = body(rank, size, msg.mpiworldid(), &why);
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

void runAtomics(const std::string& name, int worldSize, const Setup& s)
{
    runWorld(name, worldSize, [&](int rank, int size, int worldId, std::string* why) {
        return rma_atomics::body(rank, size, worldId, s, why);
    });
}

// Every reduction call refuses the two accumulate-only ops before any rank
// sends, waits or launches: a later collective still lines up
int refusedByCollectives(int rank, int size, bool deviceBuffers, std::string* why)
{
    const int n = 64 * size;
    uint8_t* send = nullptr;
    uint8_t* recv = nullptr;
    std::vector<int> hostSend(n, 1), hostRecv(n, 0);
    if (!deviceBuffers) {
        send = (uint8_t*)hostSend.data();
        recv = (uint8_t*)hostRecv.data();
    } else if (faabric::device::cudaAvailable()) {
        RMA_CHECK(cudaMalloc((void**)&send, n * sizeof(int)) == cudaSuccess);
        RMA_CHECK(cudaMalloc((void**)&recv, n * sizeof(int)) == cudaSuccess);
    } else {
        RMA_CHECK(MPI_Alloc_mem(n * sizeof(int), MPI_INFO_FAABRIC_DEVICE, &send) == MPI_SUCCESS);
        RMA_CHECK(MPI_Alloc_mem(n * sizeof(int), MPI_INFO_FAABRIC_DEVICE, &recv) == MPI_SUCCESS);
    }
    std::vector<int> counts(size, 64);
    for (MPI_Op op : { MPI_REPLACE, MPI_NO_OP }) {
        RMA_CHECK(MPI_Reduce(send, recv, n, MPI_INT, op, 0, MPI_COMM_WORLD) == MPI_ERR_OP);
        RMA_CHECK(MPI_Allreduce(send, recv, n, MPI_INT, op, MPI_COMM_WORLD) == MPI_ERR_OP);
        RMA_CHECK(MPI_Allreduce(MPI_IN_PLACE, recv, n, MPI_INT, op, MPI_COMM_WORLD) == MPI_ERR_OP);
        MPI_Request req = nullptr;
        RMA_CHECK(MPI_Iallreduce(send, recv, n, MPI_INT, op, MPI_COMM_WORLD, &req) == MPI_ERR_OP);
        RMA_CHECK(req == nullptr);
        RMA_CHECK(MPI_Reduce_scatter(send, recv, counts.data(), MPI_INT, op, MPI_COMM_WORLD) == MPI_ERR_OP);
        RMA_CHECK(MPI_Scan(send, recv, n, MPI_INT, op, MPI_COMM_WORLD) == MPI_ERR_OP);
    }
    int one = 1, total = 0;
    RMA_CHECK(MPI_Allreduce(&one, &total, 1, MPI_INT, MPI_SUM, MPI_COMM_WORLD) == MPI_SUCCESS);
    RMA_CHECK(total == size);
    if (deviceBuffers && faabric::device::cudaAvailable()) {
        cudaFree(send);
        cudaFree(recv);
    } else if (deviceBuffers) {
        MPI_Free_mem(send);
        MPI_Free_mem(recv);
    }
    return 0;
}
}

TEST_CASE("mpi rma atomics: host windows, exact results, tickets, compare-and-swap, order, rejections", "[mpi][rma]")
{
    runAtomics("rma-atomics-host", 4, Setup{ WindowMemory::Host, false, false });
}

TEST_CASE("mpi rma atomics: symmetric-heap windows go through Communicator::accumulate (loopback)", "[mpi][rma][loopback]")
{
    LoopbackBackend loopback;
    runAtomics("rma-atomics-heap-loopback", 4, Setup{ WindowMemory::Heap, false, true });
}

TEST_CASE("mpi rma atomics: reductions refuse MPI_REPLACE and MPI_NO_OP", "[mpi][rma]")
{
    runWorld("rma-refuse-host", 4, [](int rank, int size, int, std::string* why) {
        return refusedByCollectives(rank, size, false, why);
    });
    LoopbackBackend loopback;
    runWorld("rma-refuse-heap", 4, [](int rank, int size, int, std::string* why) {
        return refusedByCollectives(rank, size, true, why);
    });
}

namespace {
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

TEST_CASE("mpi rma atomics on the GPU: symmetric-heap windows", "[gpu][mpi][rma]")
{
    NEED_GPU();
    for (int n : gpuWorldSizes()) {
        runAtomics("rma-atomics-heap-" + std::to_string(n), n, Setup{ WindowMemory::Heap, true, false });
        runAtomics("rma-atomics-heap-hostbuf-" + std::to_string(n), n, Setup{ WindowMemory::Heap, false, false });
    }
}

TEST_CASE("mpi rma atomics on the GPU: cudaMalloc windows", "[gpu][mpi][rma]")
{
    NEED_GPU();
    for (int n : gpuWorldSizes()) {
        runAtomics("rma-atomics-cuda-" + std::to_string(n), n, Setup{ WindowMemory::CudaMalloc, true, false });
        runAtomics("rma-atomics-cuda-hostbuf-" + std::to_string(n), n, Setup{ WindowMemory::CudaMalloc, false, false });
    }
}

TEST_CASE("mpi rma atomics on the GPU: host windows with device buffers", "[gpu][mpi][rma]")
{
    NEED_GPU();
    for (int n : gpuWorldSizes()) {
        runAtomics("rma-atomics-hostwin-" + std::to_string(n), n, Setup{ WindowMemory::Host, true, false });
    }
}

TEST_CASE("mpi rma atomics on the GPU: reductions refuse MPI_REPLACE and MPI_NO_OP on device buffers", "[gpu][mpi][rma]")
{
    NEED_GPU();
    runWorld("rma-refuse-gpu", 2, [](int rank, int size, int, std::string* why) {
        return refusedByCollectives(rank, size, true, why);
    });
}
