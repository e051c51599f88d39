// The non-blocking and persistent reductions (MPI_Ireduce, MPI_Iscan,
// MPI_Iexscan, MPI_Exscan, MPI_Ireduce_scatter_block and the five persistent
// inits) on every datatype and built-in op, on heap, shifted heap, cudaMalloc
// and host buffers, on the world and on sub-communicators, bit for bit against
// a host fold (the program is in mpi_nb_reduce_types_body.h).
#include "fixtures.h"
#include "mpi_nb_reduce_types_body.h"

#include <faabric/executor/ExecutorContext.h>

using namespace tests;

namespace {

#define NEED_GPU()                                                             \
    do {                                                                       \
        if (!faabric::device::cudaAvailable()) {                               \
            SKIP_TEST("no CUDA device");                                       \
        }                                                                      \
    } while (0)

// A staging piece of 64 KiB, as in test_mpi_device_reduce.cpp: the sized
// counts cross the LL limit and make several staging pieces while the
// messages stay small
struct SmallStaging
{
    SmallStaging() { setenv("FAABRIC_STAGE_BYTES", "65536", 1); }
    ~SmallStaging() { unsetenv("FAABRIC_STAGE_BYTES"); }
};

using nb_reduce_types::Part;

void runNbTypes(const std::string& name, int worldSize, const nb_reduce_types::Options& o)
{
    SmallStaging staging;
    if (!o.grouped) {
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
        int rc = nb_reduce_types::body(rank, size, msg.mpiworldid(), o, &why);
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
    unsetenv("FAABRIC_MPI_GROUP_IALLREDUCE");
    REQUIRE_EQ(status->messageresults_size(), worldSize);
    for (auto& m : status->messageresults()) {
        if (m.returnvalue() != 0) {
            fbtest::fail(__FILE__, __LINE__, name + ": rank " + std::to_string(m.mpirank()) + " failed: " + m.outputdata());
        }
    }
    faabric::mpi::getMpiWorldRegistry().clear();
}

const char* partName(Part p)
{
    switch (p) {
        case Part::Bursts:
            return "bursts";
        case Part::Persistent:
            return "persistent";
        case Part::CrossKey:
            return "cross-key";
        default:
            return "subcomms";
    }
}

void loopback(int worldSize, Part part, bool grouped = true)
{
    LoopbackBackend lb;
    nb_reduce_types::Options o;
    o.part = part;
    o.grouped = grouped;
    runNbTypes(std::string("nb-reduce-types-loopback-") + partName(part) + "-" + std::to_string(worldSize) +
                 (grouped ? "" : "-ungrouped"),
               worldSize, o);
}

// `n` ranks sharing the GPU, with cudaMalloc buffers added; the 4-rank case
// adds one rank per GPU when there are several.  The matrix leaves out
// undefined pairs and host buffers (the loopback cases check them) and runs
// its sized counts at one root; it runs count 1 at 2 ranks and count 7
// beyond, so the GPU sees both.
void gpu(Part part, int n)
{
    nb_reduce_types::Options o;
    o.part = part;
    o.cudaMalloc = true;
    o.deviceOnly = true;
    o.count = n == 2 ? 1 : 7;
    runNbTypes(std::string("nb-reduce-types-gpu-") + partName(part) + "-" + std::to_string(n), n, o);
    const int gpus = faabric::device::cudaDeviceCountSafe();
    if (n == 4 && gpus > 1) {
        runNbTypes(std::string("nb-reduce-types-gpu-") + partName(part) + "-per-gpu-" + std::to_string(gpus), gpus, o);
    }
}
}

TEST_CASE("mpi nb reduce types: bursts of every datatype, op and placement on 2 ranks (loopback)", "[mpi][loopback]")
{
    loopback(2, Part::Bursts);
}

TEST_CASE("mpi nb reduce types: bursts of every datatype, op and placement on 4 ranks (loopback)", "[mpi][loopback]")
{
    loopback(4, Part::Bursts);
}

TEST_CASE("mpi nb reduce types: persistent inits of every datatype, op and placement on 2 ranks (loopback)",
          "[mpi][loopback]")
{
    loopback(2, Part::Persistent);
}

TEST_CASE("mpi nb reduce types: persistent inits of every datatype, op and placement on 4 ranks (loopback)",
          "[mpi][loopback]")
{
    loopback(4, Part::Persistent);
}

TEST_CASE("mpi nb reduce types: burst keys and the plan cache on 2 ranks (loopback)", "[mpi][loopback]")
{
    loopback(2, Part::CrossKey);
}

TEST_CASE("mpi nb reduce types: burst keys and the plan cache on 4 ranks (loopback)", "[mpi][loopback]")
{
    loopback(4, Part::CrossKey);
}

TEST_CASE("mpi nb reduce types: sub-communicators on 2 ranks (loopback)", "[mpi][loopback]")
{
    loopback(2, Part::SubComms);
}

TEST_CASE("mpi nb reduce types: sub-communicators on 4 ranks (loopback)", "[mpi][loopback]")
{
    loopback(4, Part::SubComms);
}

TEST_CASE("mpi nb reduce types: bursts and burst keys on 4 ranks, grouping off (loopback)", "[mpi][loopback]")
{
    loopback(4, Part::Bursts, false);
    loopback(4, Part::CrossKey, false);
}

TEST_CASE("mpi nb reduce types on the GPU: bursts on 2 ranks", "[gpu][mpi]")
{
    NEED_GPU();
    gpu(Part::Bursts, 2);
}

TEST_CASE("mpi nb reduce types on the GPU: bursts on 4 ranks (and one rank per GPU)", "[gpu][mpi]")
{
    NEED_GPU();
    gpu(Part::Bursts, 4);
}

TEST_CASE("mpi nb reduce types on the GPU: persistent inits on 2 ranks", "[gpu][mpi]")
{
    NEED_GPU();
    gpu(Part::Persistent, 2);
}

TEST_CASE("mpi nb reduce types on the GPU: persistent inits on 4 ranks (and one rank per GPU)", "[gpu][mpi]")
{
    NEED_GPU();
    gpu(Part::Persistent, 4);
}

TEST_CASE("mpi nb reduce types on the GPU: burst keys and the plan cache on 2 ranks", "[gpu][mpi]")
{
    NEED_GPU();
    gpu(Part::CrossKey, 2);
}

TEST_CASE("mpi nb reduce types on the GPU: burst keys and the plan cache on 4 ranks (and one rank per GPU)", "[gpu][mpi]")
{
    NEED_GPU();
    gpu(Part::CrossKey, 4);
}

TEST_CASE("mpi nb reduce types on the GPU: sub-communicators on 2 ranks", "[gpu][mpi]")
{
    NEED_GPU();
    gpu(Part::SubComms, 2);
}

TEST_CASE("mpi nb reduce types on the GPU: sub-communicators on 4 ranks (and one rank per GPU)", "[gpu][mpi]")
{
    NEED_GPU();
    gpu(Part::SubComms, 4);
}
