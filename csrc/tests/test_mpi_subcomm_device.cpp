// The fused device path of sub-communicators (MPI_Comm_split and friends) in
// an in-process world; the program is in mpi_subcomm_device_body.h.
#include "fixtures.h"
#include "mpi_subcomm_device_body.h"

#include <faabric/executor/ExecutorContext.h>

using namespace tests;
using subcomm_device::BufferMemory;
using subcomm_device::Setup;

namespace {

#define NEED_GPU()                                                             \
    do {                                                                       \
        if (!faabric::device::cudaAvailable()) {                               \
            SKIP_TEST("no CUDA device");                                       \
        }                                                                      \
    } while (0)

void runSubcommDevice(const std::string& name, int worldSize, const Setup& s)
{
    ClusterFixture f(worldSize);
    registerTestFunction("mpi", name, [&](auto*, int, int, auto) {
        MPI_Init(nullptr, nullptr);
        int rank = -1, size = -1;
        MPI_Comm_rank(MPI_COMM_WORLD, &rank);
        MPI_Comm_size(MPI_COMM_WORLD, &size);
        std::string why;
        faabric::Message& msg = faabric::executor::ExecutorContext::get()->getMsg();
        int rc = subcomm_device::body(rank, size, msg.mpiworldid(), s, &why);
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
    auto status = f.awaitBatch(req, 240000);
    REQUIRE_EQ(status->messageresults_size(), worldSize);
    for (auto& m : status->messageresults()) {
        if (m.returnvalue() != 0) {
            fbtest::fail(__FILE__, __LINE__, name + ": rank " + std::to_string(m.mpirank()) + " failed: " + m.outputdata());
        }
    }
    faabric::mpi::getMpiWorldRegistry().clear();
}
}

TEST_CASE("mpi sub-communicators: fused collectives on heap buffers (loopback)", "[mpi][loopback]")
{
    LoopbackBackend loopback;
    runSubcommDevice("subcomm-device-loopback-4", 4, Setup{ BufferMemory::Heap });
    runSubcommDevice("subcomm-device-loopback-8", 8, Setup{ BufferMemory::Heap });
}

TEST_CASE("mpi sub-communicators on the GPU: fused collectives on heap and cudaMalloc buffers", "[gpu][mpi]")
{
    NEED_GPU();
    // 4 ranks sharing the GPU, and one rank per GPU when there are several
    std::vector<int> sizes{ 4 };
    const int gpus = faabric::device::cudaDeviceCountSafe();
    if (gpus > 1) {
        sizes.push_back(gpus);
    }
    for (int n : sizes) {
        runSubcommDevice("subcomm-device-heap-" + std::to_string(n), n, Setup{ BufferMemory::Heap });
        runSubcommDevice("subcomm-device-cuda-" + std::to_string(n), n, Setup{ BufferMemory::CudaMalloc });
    }
}
