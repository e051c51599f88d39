// Device-path tests written WITHOUT access to a GPU (the round's GPU budget was
// spent): tag [unverified] keeps them out of `--tag gpu`, which is what the
// pytest GPU suite runs.  First thing to do with a GPU: run
//   build/bin/faabric_tests --tag unverified
// fix what they find, then retag them [gpu].  They skip without a device.
#include "fixtures.h"

#include <faabric/device/communicator.h>
#include <faabric/device/cuda_driver.h>
#include <faabric/mpi/MpiWorld.h>
#include <faabric/mpi/MpiWorldRegistry.h>
#include <faabric/mpi/mpi.h>
#include <faabric/snapshot/DeviceSnapshot.h>
#include <faabric/snapshot/SnapshotRegistry.h>
#include <faabric/state/State.h>
#include <faabric/util/snapshot.h>

#include <cuda_runtime.h>

#include <barrier>
#include <filesystem>
#include <unistd.h>

using namespace tests;

#define NEED_GPU()                                                             \
    do {                                                                       \
        if (!faabric::device::cudaAvailable()) {                               \
            SKIP_TEST("no CUDA device");                                       \
        }                                                                      \
    } while (0)

#define CHECK_RANK(cond)                                                       \
    do {                                                                       \
        if (!(cond)) {                                                         \
            printf("         rank %d: check failed at line %d: %s\n", rank, __LINE__, #cond); \
            return 1;                                                          \
        }                                                                      \
    } while (0)

namespace {
void runMpiOnGpus(const std::string& name, int worldSize, const std::function<int(int, int)>& body)
{
    ClusterFixture f(worldSize);
    registerTestFunction("mpi", name, [&](auto*, int, int, auto) {
        MPI_Init(nullptr, nullptr);
        int rank = -1, size = -1;
        MPI_Comm_rank(MPI_COMM_WORLD, &rank);
        MPI_Comm_size(MPI_COMM_WORLD, &size);
        int rc = body(rank, size);
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
            fbtest::fail(__FILE__, __LINE__, "rank " + std::to_string(m.mpirank()) + " failed: " + m.outputdata());
        }
    }
    faabric::mpi::getMpiWorldRegistry().clear();
}

// Windows in the symmetric heap: puts and gets are peer copies
int deviceRmaBody(int rank, int size)
{
    const int n = 4096;
    long* window = nullptr;
    CHECK_RANK(MPI_Alloc_mem(n * sizeof(long), MPI_INFO_FAABRIC_DEVICE, &window) == MPI_SUCCESS);
    std::vector<long> init(n, -1);
    cudaMemcpy(window, init.data(), n * sizeof(long), cudaMemcpyHostToDevice);
    MPI_Win win = nullptr;
    MPI_Win_create(window, n * sizeof(long), sizeof(long), MPI_INFO_NULL, MPI_COMM_WORLD, &win);
    MPI_Win_fence(0, win);
    // host origin -> device window of every rank
    long mine = 100 + rank;
    for (int t = 0; t < size; t++) {
        MPI_Put(&mine, 1, MPI_LONG, t, rank, 1, MPI_LONG, win);
    }
    MPI_Win_fence(0, win);
    std::vector<long> seen(n);
    cudaMemcpy(seen.data(), window, n * sizeof(long), cudaMemcpyDeviceToHost);
    for (int r = 0; r < size; r++) {
        CHECK_RANK(seen[r] == 100 + r);
    }
    CHECK_RANK(seen[size] == -1);
    // device origin <- device window of the right neighbour
    long* strip = nullptr;
    cudaMalloc(&strip, 8 * sizeof(long));
    MPI_Get(strip, 8, MPI_LONG, (rank + 1) % size, 0, 8, MPI_LONG, win);
    MPI_Win_fence(0, win);
    std::vector<long> got(8);
    cudaMemcpy(got.data(), strip, 8 * sizeof(long), cudaMemcpyDeviceToHost);
    CHECK_RANK(got[0] == 100);
    cudaFree(strip);
    MPI_Win_free(&win);
    MPI_Free_mem(window);
    return 0;
}

// Sub-communicator collectives on device buffers go through the p2p layer
int deviceSubCommBody(int rank, int size)
{
    MPI_Comm half = nullptr;
    MPI_Comm_split(MPI_COMM_WORLD, rank % 2, rank, &half);
    int hSize = -1;
    MPI_Comm_size(half, &hSize);
    const int n = 10000;
    int *send = nullptr, *recv = nullptr;
    cudaMalloc(&send, n * sizeof(int));
    cudaMalloc(&recv, n * sizeof(int));
    std::vector<int> host(n, rank + 1);
    cudaMemcpy(send, host.data(), n * sizeof(int), cudaMemcpyHostToDevice);
    MPI_Allreduce(send, recv, n, MPI_INT, MPI_SUM, half);
    cudaMemcpy(host.data(), recv, n * sizeof(int), cudaMemcpyDeviceToHost);
    int expected = 0;
    for (int r = rank % 2; r < size; r += 2) {
        expected += r + 1;
    }
    CHECK_RANK(host[0] == expected && host[n - 1] == expected);
    MPI_Bcast(recv, n, MPI_INT, 0, half);
    cudaFree(send);
    cudaFree(recv);
    MPI_Comm_free(&half);
    return 0;
}
}

TEST_CASE("next: one-sided windows in device memory", "[unverified][mpi]")
{
    NEED_GPU();
    runMpiOnGpus("device-rma", std::max(2, faabric::device::cudaDeviceCountSafe()), deviceRmaBody);
}

TEST_CASE("next: sub-communicator collectives on device buffers", "[unverified][mpi]")
{
    NEED_GPU();
    runMpiOnGpus("device-subcomm", 4, deviceSubCommBody);
}

TEST_CASE("next: device snapshots spill to host, files and back", "[unverified][snapshot]")
{
    NEED_GPU();
    using namespace faabric::util;
    const size_t size = 3 * HOST_PAGE_SIZE + 77;
    std::vector<uint8_t> bytes(size);
    for (size_t i = 0; i < size; i++) {
        bytes[i] = (uint8_t)(i * 13);
    }
    faabric::snapshot::DeviceSnapshot dev(size, 0);
    dev.copyInData(bytes);
    dev.addMergeRegion(128, 8, SnapshotDataType::Long, SnapshotMergeOperation::Sum);
    auto host = dev.spillToHost();
    REQUIRE(host->getDataCopy() == bytes);
    REQUIRE_EQ(host->getMergeRegions().size(), (size_t)1);
    auto back = faabric::snapshot::DeviceSnapshot::fromHost(*host, 0);
    REQUIRE(back->getDataCopy() == bytes);
    REQUIRE_EQ(back->getMergeRegions().size(), (size_t)1);
    const std::string dir = "/tmp/fb_dev_ckpt_" + std::to_string(getpid());
    std::filesystem::create_directories(dir);
    dev.writeToFile(dir + "/d.snap");
    auto fromFile = faabric::snapshot::DeviceSnapshot::readFromFile(dir + "/d.snap", 0);
    REQUIRE(fromFile->getDataCopy() == bytes);
    // registry: device images return to the device
    auto& reg = faabric::snapshot::getSnapshotRegistry();
    reg.clear();
    reg.registerDeviceSnapshot("dev/key", back);
    REQUIRE_EQ(reg.checkpointToDir(dir + "/reg"), (size_t)1);
    reg.clear();
    REQUIRE_EQ(reg.restoreFromDir(dir + "/reg", 0), (size_t)1);
    REQUIRE(reg.deviceSnapshotExists("dev/key"));
    REQUIRE(reg.getDeviceSnapshot("dev/key")->getDataCopy() == bytes);
    reg.clear();
    std::filesystem::remove_all(dir);
}

TEST_CASE("next: a tuning file steers the all-reduce algorithm", "[unverified][device]")
{
    NEED_GPU();
    using namespace faabric::device;
    const std::string path = "/tmp/fb_tuning_gpu_" + std::to_string(getpid()) + ".txt";
    CommTuning t = CommTuning::parse("allreduce 1048576 twoshot\nallreduce 18446744073709551615 oneshot\n");
    faabric::util::writeBytesToFile(path, faabric::util::stringToBytes(t.serialise()));
    setenv("FAABRIC_TUNING_FILE", path.c_str(), 1);
    int nDev = cudaDeviceCountSafe();
    int n = std::max(2, std::min(nDev, 4));
    std::vector<int> devices(n);
    for (int i = 0; i < n; i++) {
        devices[i] = i % nDev;
    }
    CommConfig cfg;
    cfg.heapBytes = 64 << 20;
    auto comms = Communicator::createLocal(n, devices, cfg);
    unsetenv("FAABRIC_TUNING_FILE");
    ::unlink(path.c_str());
    // 4 KiB would be LL by the built-in thresholds; the file says two-shot
    REQUIRE_EQ(comms[0]->pickAllReduceAlgo(4096, false), (int)FB_ALGO_TWOSHOT);
    REQUIRE_EQ(comms[0]->pickAllReduceAlgo(8 << 20, false), (int)FB_ALGO_ONESHOT);
}

// ---------------------------------------------------------------------------
// device-resident state values
// ---------------------------------------------------------------------------
TEST_CASE("device state: main copy in HBM, replicas pull chunks and push dirty blocks with one kernel", "[gpu][state]")
{
    NEED_GPU();
    int nDev = 0;
    cudaGetDeviceCount(&nDev);
    const int devMain = 0;
    const int devReplica = nDev > 1 ? 1 : 0; // on one GPU the "peer" is the same device
    faabric::state::State state("test-host");
    const size_t size = (3 << 20) + 777; // not a multiple of anything interesting
    auto mainKv = state.getDeviceKV("demo", "weights", size, devMain);
    REQUIRE(mainKv->isMain());
    // a second object for the same device is the same object
    REQUIRE(state.getDeviceKV("demo", "weights", size, devMain) == mainKv);

    std::vector<uint8_t> init(size);
    for (size_t i = 0; i < size; i++) {
        init[i] = (uint8_t)(i * 7 + 3);
    }
    mainKv->set(init.data());

    // replica (size taken from the main copy)
    std::shared_ptr<faabric::state::DeviceStateKeyValue> rep;
    if (devReplica != devMain) {
        rep = state.getDeviceKV("demo", "weights", 0, devReplica);
    } else {
        rep = std::make_shared<faabric::state::DeviceStateKeyValue>("demo", "weights", size, devReplica, mainKv);
    }
    REQUIRE(!rep->isMain());
    REQUIRE_EQ(rep->size(), size);

    // lazy chunk pull: only the 64 KiB chunks that cover the request move
    REQUIRE(!rep->isChunkPulled(100000, 10));
    std::vector<uint8_t> got(5000);
    rep->getChunk(100000, got.data(), got.size());
    REQUIRE(memcmp(got.data(), init.data() + 100000, got.size()) == 0);
    REQUIRE(rep->isChunkPulled(100000, 5000));
    REQUIRE(!rep->isChunkPulled(1 << 20, 10));
    REQUIRE_EQ(rep->getBytesPulled(), (uint64_t)STATE_STREAMING_CHUNK_SIZE); // bytes 100000..104999 sit in chunk 1
    rep->pull();
    std::vector<uint8_t> whole(size);
    rep->get(whole.data());
    REQUIRE(whole == init);

    // modify scattered ranges ON THE DEVICE, flag them, push partially
    struct Edit
    {
        long off;
        long len;
        uint8_t val;
    };
    std::vector<Edit> edits = { { 5, 3, 0xa1 }, { 4096 * 9 + 100, 1000, 0xb2 }, { 1 << 20, 128, 0xc3 }, { (long)size - 50, 50, 0xd4 } };
    cudaSetDevice(devReplica);
    for (auto& e : edits) {
        cudaMemset(rep->getDevicePtr() + e.off, e.val, e.len);
        rep->flagChunkDirty(e.off, e.len);
        memset(init.data() + e.off, e.val, e.len);
    }
    cudaDeviceSynchronize();
    // the device scan reports exactly the flagged blocks, as runs
    auto runs = rep->getDirtyChunks();
    REQUIRE_EQ(runs.size(), 4u);
    REQUIRE_EQ(runs[0].offset, 0u);
    REQUIRE_EQ(runs[0].length, 128u);
    REQUIRE_EQ(runs[1].offset, (uint64_t)(4096 * 9));      // 36864 = 288 * 128
    REQUIRE_EQ(runs[1].length, (uint64_t)(9 * 128));        // 36964..37964 touches blocks 288..296
    REQUIRE_EQ(runs[3].offset + runs[3].length, (uint64_t)size);
    uint64_t pushed = rep->pushPartial();
    REQUIRE_EQ(rep->getPushKernelLaunches(), 1u);
    REQUIRE(pushed >= 3 + 1000 + 128 + 50);
    REQUIRE(pushed <= (uint64_t)(1 + 9 + 1 + 2) * 128);
    // the main copy now has the edits and nothing else changed
    mainKv->get(whole.data());
    REQUIRE(whole == init);
    // the mask was cleared by the kernel: a second push moves nothing
    REQUIRE_EQ(rep->pushPartial(), 0u);
    REQUIRE(rep->getDirtyChunks().empty());
    // host mirror
    uint8_t* mirror = mainKv->syncHostMirror();
    REQUIRE(memcmp(mirror, init.data(), size) == 0);
    state.deleteDeviceKV("demo", "weights");
    REQUIRE_EQ(state.getDeviceKVCount(), 0u);
}

// ---------------------------------------------------------------------------
// point-to-point groups on the device
// ---------------------------------------------------------------------------
namespace {
faabric::batch_scheduler::SchedulingDecision gpuDecision(int appId, int groupId, int n)
{
    faabric::batch_scheduler::SchedulingDecision d(appId, groupId);
    for (int i = 0; i < n; i++) {
        faabric::Message m;
        m.set_appid(appId);
        m.set_groupid(groupId);
        m.set_groupidx(i);
        m.set_appidx(i);
        m.set_id(1000 + i);
        d.addMessage("gpu" + std::to_string(i), m);
    }
    return d;
}
}

TEST_CASE("ptp on device buffers: many in-order messages between group members", "[gpu][ptp]")
{
    NEED_GPU();
    ClusterFixture f(0, 4, 1);
    auto& broker = faabric::transport::getPointToPointBroker();
    const int groupId = 7701;
    const int n = 4;
    broker.setUpLocalMappingsFromSchedulingDecision(gpuDecision(77, groupId, n));
    broker.createLocalDeviceGroup(groupId);
    REQUIRE(broker.isDeviceGroup(groupId));
    // (reference test: "Test many in-order messages",
    //  tests/dist/transport/functions.cpp - here the payloads never leave HBM)
    const int nMsgs = 60;
    std::vector<std::thread> members;
    std::atomic<int> failures{ 0 };
    std::barrier allDrained(n);
    for (int idx = 0; idx < n; idx++) {
        members.emplace_back([&, idx] {
            auto comm = broker.getDeviceCommunicator(groupId, idx);
            cudaSetDevice(comm->device());
            cudaStream_t s;
            cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
            const int next = (idx + 1) % n;
            const int prev = (idx + n - 1) % n;
            std::vector<int*> outs(nMsgs), ins(nMsgs);
            for (int k = 0; k < nMsgs; k++) {
                size_t count = 1 + (size_t)k * 37; // growing sizes, odd byte counts
                cudaMalloc(&outs[k], count * 4);
                cudaMalloc(&ins[k], count * 4);
                std::vector<int> h(count, idx * 100000 + k);
                cudaMemcpy(outs[k], h.data(), count * 4, cudaMemcpyHostToDevice);
                cudaMemset(ins[k], 0, count * 4);
            }
            // (allocation may synchronise with the device too: see below)
            allDrained.arrive_and_wait();
            // all sends first (eager), then all receives: order must hold
            for (int k = 0; k < nMsgs; k++) {
                broker.sendDeviceMessage(groupId, idx, next, outs[k], (1 + (size_t)k * 37) * 4, s);
            }
            for (int k = 0; k < nMsgs; k++) {
                broker.recvDeviceMessage(groupId, prev, idx, ins[k], (1 + (size_t)k * 37) * 4, s);
            }
            if (!comm->syncStreamBounded(s, 20000) || comm->peekError() != 0) {
                failures++;
            }
            // cudaFree (below) waits for the WHOLE device to go idle while it
            // holds the context: a member that frees early would stall the
            // members that have not issued their sends yet, whose messages the
            // device is waiting for.  Free only once every stream has drained.
            allDrained.arrive_and_wait();
            for (int k = 0; k < nMsgs; k++) {
                size_t count = 1 + (size_t)k * 37;
                std::vector<int> h(count);
                cudaMemcpy(h.data(), ins[k], count * 4, cudaMemcpyDeviceToHost);
                for (size_t i = 0; i < count; i++) {
                    if (h[i] != prev * 100000 + k) {
                        failures++;
                        break;
                    }
                }
                cudaFree(outs[k]);
                cudaFree(ins[k]);
            }
            cudaStreamDestroy(s);
        });
    }
    for (auto& t : members) {
        t.join();
    }
    REQUIRE_EQ(failures.load(), 0);
    broker.clearGroup(groupId);
    REQUIRE(!broker.isDeviceGroup(groupId));
}

TEST_CASE("ptp group barrier on the device", "[gpu][ptp]")
{
    NEED_GPU();
    ClusterFixture f(0, 4, 1);
    auto& broker = faabric::transport::getPointToPointBroker();
    const int groupId = 7702;
    const int n = 4;
    broker.setUpLocalMappingsFromSchedulingDecision(gpuDecision(78, groupId, n));
    faabric::transport::PointToPointGroup::addGroupIfNotExists(78, groupId, n);
    broker.createLocalDeviceGroup(groupId);
    auto group = faabric::transport::PointToPointGroup::getGroup(groupId);
    // (reference test: "Test distributed barrier", tests/dist/transport/functions.cpp:
    //  nobody may enter round r+1 before everybody finished round r)
    const int rounds = 25;
    std::atomic<int> arrived{ 0 };
    std::atomic<int> violations{ 0 };
    std::vector<std::thread> members;
    for (int idx = 0; idx < n; idx++) {
        members.emplace_back([&, idx] {
            auto comm = broker.getDeviceCommunicator(groupId, idx);
            cudaSetDevice(comm->device());
            for (int r = 0; r < rounds; r++) {
                if (idx == r % n) {
                    std::this_thread::sleep_for(std::chrono::milliseconds(3)); // a straggler per round
                }
                arrived++;
                group->barrier(idx);
                if (arrived.load() < (r + 1) * n) {
                    violations++;
                }
                group->barrier(idx);
            }
        });
    }
    for (auto& t : members) {
        t.join();
    }
    REQUIRE_EQ(violations.load(), 0);
    REQUIRE_EQ(arrived.load(), rounds * n);
    broker.clearGroup(groupId);
}

TEST_CASE("device snapshot: overlapping diffs are applied in order, like the host image", "[gpu][snapshot]")
{
    NEED_GPU();
    using namespace faabric::util;
    const size_t size = 4 * HOST_PAGE_SIZE;
    std::vector<uint8_t> base(size, 0);
    int start = 10;
    memcpy(base.data() + 128, &start, 4);
    auto host = std::make_shared<SnapshotData>(std::span<const uint8_t>(base.data(), base.size()));
    faabric::snapshot::DeviceSnapshot dsnap(size, 0);
    dsnap.copyInData(base);
    // five Sum diffs onto ONE int (what five threads reducing into a shared
    // variable produce), a Bytewise diff overwritten by a later one, and an
    // XOR on top of a Bytewise diff
    std::vector<std::vector<uint8_t>> payloads;
    std::vector<SnapshotDiff> diffs;
    auto add = [&](SnapshotDataType t, SnapshotMergeOperation op, uint32_t off, std::vector<uint8_t> bytes) {
        payloads.push_back(std::move(bytes));
        diffs.emplace_back(t, op, off, payloads.back());
    };
    payloads.reserve(16);
    for (int k = 1; k <= 5; k++) {
        std::vector<uint8_t> b(4);
        memcpy(b.data(), &k, 4);
        add(SnapshotDataType::Int, SnapshotMergeOperation::Sum, 128, b);
    }
    add(SnapshotDataType::Raw, SnapshotMergeOperation::Bytewise, 1000, std::vector<uint8_t>(64, 0x11));
    add(SnapshotDataType::Raw, SnapshotMergeOperation::Bytewise, 1032, std::vector<uint8_t>(64, 0x22));
    add(SnapshotDataType::Raw, SnapshotMergeOperation::XOR, 1000, std::vector<uint8_t>(8, 0xff));
    host->applyDiffs(diffs);
    dsnap.applyDiffs(diffs);
    auto got = dsnap.getDataCopy();
    REQUIRE(memcmp(got.data(), host->getDataPtr(), size) == 0);
    int sum = 0;
    memcpy(&sum, got.data() + 128, 4);
    REQUIRE_EQ(sum, 10 + 15);
    REQUIRE_EQ((int)got[1000], 0xee);
    REQUIRE_EQ((int)got[1040], 0x22);
}

TEST_CASE("device snapshot: delta encoding on the GPU is byte-identical to the host codec and applies in place", "[gpu][snapshot][delta]")
{
    if (!faabric::device::cudaAvailable()) {
        SKIP_TEST("no CUDA device");
    }
    const size_t size = 64 * 4096 + 100; // a ragged last page
    std::vector<uint8_t> oldHost(size), newHost;
    for (size_t i = 0; i < size; i++) {
        oldHost[i] = (uint8_t)(i * 7 + 3);
    }
    newHost = oldHost;
    // a lone page, a run of three pages, single bytes at page edges, the ragged tail
    for (size_t i = 5 * 4096 + 10; i < 5 * 4096 + 900; i++) {
        newHost[i] ^= 0x5a;
    }
    for (size_t i = 20 * 4096; i < 23 * 4096; i++) {
        newHost[i] = (uint8_t)(i % 251);
    }
    newHost[30 * 4096] ^= 1;
    newHost[31 * 4096 - 1] ^= 2;
    newHost[size - 1] ^= 0x80;

    faabric::snapshot::DeviceSnapshot image(size, 0);
    image.copyInData(oldHost, 0);
    uint8_t* mem = nullptr;
    cudaSetDevice(0);
    REQUIRE(cudaMalloc(&mem, size) == cudaSuccess);
    cudaMemcpy(mem, newHost.data(), size, cudaMemcpyHostToDevice);

    for (const char* def : { "pages=4096;xor;", "pages=4096;", "pages=4096;xor;zstd=1;", "xor;" }) {
        faabric::util::DeltaSettings cfg(def);
        if (cfg.useZstd && !faabric::util::deltaZstdAvailable()) {
            continue;
        }
        std::vector<uint8_t> onDevice = image.serializeDelta(cfg, mem, size);
        std::vector<uint8_t> onHost = faabric::util::serializeDelta(cfg, oldHost.data(), size, newHost.data(), size);
        REQUIRE(onDevice == onHost);
        if (cfg.usePages && !cfg.useZstd) {
            // only the changed pages travel: 1 + 3 + 2 + 1 pages and a few headers
            REQUIRE(onDevice.size() < 8 * 4096);
        }
        // applying it to another copy of the old image gives the new bytes
        faabric::snapshot::DeviceSnapshot other(size, 0);
        other.copyInData(oldHost, 0);
        other.applyDelta(onDevice);
        REQUIRE(other.getDataCopy() == newHost);
    }
    // an unchanged image encodes to just the header and the end marker
    faabric::util::DeltaSettings plain("pages=4096;xor;");
    cudaMemcpy(mem, oldHost.data(), size, cudaMemcpyHostToDevice);
    REQUIRE_EQ(image.serializeDelta(plain, mem, size).size(), 6u);
    // a shorter new buffer is a valid target, a longer one is not
    REQUIRE(image.serializeDelta(plain, mem, size - 4096) ==
            faabric::util::serializeDelta(plain, oldHost.data(), size, oldHost.data(), size - 4096));
    REQUIRE_THROWS(image.serializeDelta(plain, mem, size + 1));
    cudaFree(mem);
}
