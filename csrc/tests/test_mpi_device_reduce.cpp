// Every MPI reduction call, on every datatype and built-in op, on heap, shifted
// heap, cudaMalloc and host buffers, bit for bit against a host fold (the
// program is in mpi_device_reduce_body.h).
#include "fixtures.h"
#include "mpi_device_reduce_body.h"

#include <faabric/executor/ExecutorContext.h>

using namespace tests;

namespace {

#define NEED_GPU()                                                             \
    do {                                                                       \
        if (!faabric::device::cudaAvailable()) {                               \
            SKIP_TEST("no CUDA device");                                       \
        }                                                                      \
    } while (0)

// A staging piece of 64 KiB: above llMaxBytes and below oneShotMaxBytes, so
// the program's sizes cross every algorithm and staging boundary while its
// messages stay small
struct SmallStaging
{
    SmallStaging() { setenv("FAABRIC_STAGE_BYTES", "65536", 1); }
    ~SmallStaging() { unsetenv("FAABRIC_STAGE_BYTES"); }
};

void runReduce(const std::string& name, int worldSize, const mpi_device_reduce::Options& o)
{
    SmallStaging staging;
    ClusterFixture f(worldSize);
    registerTestFunction("mpi", name, [&](auto*, int, int, auto) {
        MPI_Init(nullptr, nullptr);
        int rank = -1, size = -1;
        MPI_Comm_rank(MPI_COMM_WORLD, &rank);
        MPI_Comm_size(MPI_COMM_WORLD, &size);
        std::string why;
        faabric::Message& msg = faabric::executor::ExecutorContext::get()->getMsg();
        int rc = mpi_device_reduce::body(rank, size, msg.mpiworldid(), o, &why);
        if (rc != 0) {
            printf("%s", why.c_str());
            msg.set_outputdata(why);
        }
        MPI_Finalize();
        return rc;
    });
    auto req = faabric::util::batchExecFactory("mpi", name, 1);
    req->mutable_messages(0)->set_ismpi(true);
    req->mutable_messages(0)->set_mpiworldsize(worldSize);
    f.plannerCli.callFunctions(req);
    auto status = f.awaitBatch(req, 900000);
    REQUIRE_EQ(status->messageresults_size(), worldSize);
    for (auto& m : status->messageresults()) {
        if (m.returnvalue() != 0) {
            fbtest::fail(__FILE__, __LINE__, name + ": rank " + std::to_string(m.mpirank()) + " failed: " + m.outputdata());
        }
    }
    faabric::mpi::getMpiWorldRegistry().clear();
}
}

TEST_CASE("mpi device reduce: every datatype, op, call and placement on 2 ranks (loopback)", "[mpi][loopback]")
{
    LoopbackBackend loopback;
    runReduce("device-reduce-loopback-2", 2, {});
}

TEST_CASE("mpi device reduce: every datatype, op, call and placement on 4 ranks (loopback)", "[mpi][loopback]")
{
    LoopbackBackend loopback;
    runReduce("device-reduce-loopback-4", 4, {});
}

TEST_CASE("mpi device reduce on the GPU: every datatype, op, call and placement", "[gpu][mpi]")
{
    NEED_GPU();
    std::vector<int> sizes{ 2, 4 };
    const int gpus = faabric::device::cudaDeviceCountSafe();
    if (gpus > 1) {
        sizes.push_back(gpus);
    }
    for (int n : sizes) {
        runReduce("device-reduce-gpu-" + std::to_string(n), n, { true });
    }
}
