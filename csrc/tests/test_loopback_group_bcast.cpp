// Grouped broadcast (Communicator::runGroup / groupMany, GROUP_BROADCAST) and the
// grouped calls on sub-communicator children, on the loopback backend (no
// GPU): results against a closed form at 1-8 ranks, launch counts, refusals
// and fall-backs, and the MPI program of mpi_group_subcomm_body.h.
#include "fixtures.h"
#include "mpi_group_subcomm_body.h"

#include <faabric/device/communicator.h>
#include <faabric/executor/ExecutorContext.h>

#include "launch_api.h"

#include <atomic>
#include <cstring>
#include <functional>
#include <random>
#include <thread>

using faabric::device::CommConfig;
using faabric::device::Communicator;

namespace {
std::vector<std::shared_ptr<Communicator>> loopGroup(int n)
{
    CommConfig cfg;
    cfg.loopback = true;
    cfg.heapBytes = (size_t)16 << 20;
    cfg.stageBytes = (size_t)1 << 20;
    cfg.p2pBounceBytes = (size_t)1 << 20;
    cfg.channels = 2;
    cfg.maxBlocks = 4;
    cfg.timeoutMs = 5000;
    return Communicator::createLocal(n, std::vector<int>(n, 0), cfg);
}

// fn(i) on one thread per index; returns the number of failures
int runThreads(int n, const std::function<bool(int)>& fn)
{
    std::atomic<int> failures{ 0 };
    std::vector<std::thread> ts;
    for (int i = 0; i < n; i++) {
        ts.emplace_back([&, i] {
            try {
                if (!fn(i)) {
                    printf("         thread %d failed\n", i);
                    failures++;
                }
            } catch (const std::exception& e) {
                printf("         thread %d threw: %s\n", i, e.what());
                failures++;
            }
        });
    }
    for (auto& t : ts) {
        t.join();
    }
    return failures.load();
}

// Byte j of item i as rank r wrote it before the broadcast
uint8_t pattern(int r, int i, size_t j)
{
    return (uint8_t)(r * 61 + i * 17 + j * 7 + 3);
}

// Lengths: 1 byte, 15 bytes, one vector + tail, several chunks (the chunk of
// 8 ranks is 64 vectors), and some in between
const std::vector<size_t> LENGTHS = { 1, 15, 16, 17, 31, 250, 1024 + 9, 16 * 300 + 5, 16 * 2000, 7 };

size_t slotOf(size_t len)
{
    return (len + 64 + 255) / 256 * 256; // 16-byte aligned items, guard gaps
}

// Every rank fills its items (and the gaps) with its own pattern, broadcasts
// from `root` with `call`, and checks that items hold the root's bytes and
// gaps its own
bool broadcastCase(Communicator& c, uint8_t* base, int root, const std::function<int(std::vector<Communicator::GroupItem>&)>& call)
{
    const int r = c.rank();
    std::vector<Communicator::GroupItem> items;
    size_t pos = 0;
    for (size_t i = 0; i < LENGTHS.size(); i++) {
        for (size_t j = 0; j < slotOf(LENGTHS[i]); j++) {
            base[pos + j] = pattern(r, (int)i, j);
        }
        items.push_back({ base + pos, base + pos, LENGTHS[i] });
        pos += slotOf(LENGTHS[i]);
    }
    if (call(items) != FB_OK) {
        return false;
    }
    pos = 0;
    for (size_t i = 0; i < LENGTHS.size(); i++) {
        for (size_t j = 0; j < slotOf(LENGTHS[i]); j++) {
            const uint8_t want = j < LENGTHS[i] ? pattern(root, (int)i, j) : pattern(r, (int)i, j);
            if (base[pos + j] != want) {
                printf("         rank %d item %zu byte %zu: %u, want %u\n", r, i, j, base[pos + j], want);
                return false;
            }
        }
        pos += slotOf(LENGTHS[i]);
    }
    return true;
}

size_t totalBytes()
{
    size_t t = 0;
    for (size_t l : LENGTHS) {
        t += slotOf(l);
    }
    return t;
}
}

TEST_CASE("loopback group broadcast: plans and transient lists from every root at 1-8 ranks", "[loopback]")
{
    for (int n = 1; n <= 8; n++) {
        auto comms = loopGroup(n);
        const uint64_t off = comms[0]->alloc(totalBytes());
        for (int r = 1; r < n; r++) {
            REQUIRE_EQ(comms[r]->alloc(totalBytes()), off);
        }
        int fails = runThreads(n, [&](int r) {
            Communicator& c = *comms[r];
            uint8_t* base = c.heapPtr(off);
            bool ok = true;
            for (int root = 0; root < n && ok; root++) {
                const uint64_t l0 = c.stats().launches;
                ok = ok && broadcastCase(c, base, root, [&](auto& items) {
                    return c.groupMany(Communicator::GROUP_BROADCAST, items.data(), items.size(), FB_U8, 0, root, FB_FLAG_SYMMETRIC, nullptr);
                });
                ok = ok && c.stats().launches == l0 + (n > 1 ? 1 : 0);
                std::shared_ptr<Communicator::GroupPlan> plan;
                ok = ok && broadcastCase(c, base, root, [&](auto& items) {
                    int rc = FB_OK;
                    plan = c.prepareGroup(items.data(), items.size(), FB_U8, &rc, Communicator::GROUP_BROADCAST);
                    return plan == nullptr ? rc : c.runGroup(Communicator::GROUP_BROADCAST, *plan, 0, root, FB_FLAG_SYMMETRIC, nullptr);
                });
                ok = ok && plan && Communicator::groupPlanLaunches(*plan) == 1;
                ok = ok && c.stats().launches == l0 + (n > 1 ? 2 : 0);
            }
            return ok && c.checkError(nullptr) == 0;
        });
        REQUIRE_EQ(fails, 0);
    }
}

TEST_CASE("loopback group broadcast: 1017 items take two launches, 1016 one", "[loopback]")
{
    const int n = 3;
    auto comms = loopGroup(n);
    const size_t items = 1017;
    const uint64_t off = comms[0]->alloc(items * 32);
    for (int r = 1; r < n; r++) {
        REQUIRE_EQ(comms[r]->alloc(items * 32), off);
    }
    int fails = runThreads(n, [&](int r) {
        Communicator& c = *comms[r];
        uint8_t* base = c.heapPtr(off);
        bool ok = true;
        for (size_t cnt : { (size_t)1016, items }) {
            std::vector<Communicator::GroupItem> list;
            for (size_t i = 0; i < cnt; i++) {
                for (size_t j = 0; j < 32; j++) {
                    base[i * 32 + j] = pattern(r, (int)i, j);
                }
                list.push_back({ base + i * 32, base + i * 32, 1 + i % 20 });
            }
            const uint64_t l0 = c.stats().launches;
            ok = ok && c.groupMany(Communicator::GROUP_BROADCAST, list.data(), list.size(), FB_U8, 0, 1, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            ok = ok && c.stats().launches == l0 + (cnt == items ? 2 : 1);
            for (size_t i = 0; i < cnt && ok; i++) {
                for (size_t j = 0; j < 32; j++) {
                    ok = ok && base[i * 32 + j] == (j < 1 + i % 20 ? pattern(1, (int)i, j) : pattern(r, (int)i, j));
                }
            }
        }
        return ok;
    });
    REQUIRE_EQ(fails, 0);
}

TEST_CASE("loopback group broadcast: refusals, and unaligned lists fall back to broadcast", "[loopback]")
{
    const int n = 4;
    auto comms = loopGroup(n);
    const uint64_t off = comms[0]->alloc(4096);
    for (int r = 1; r < n; r++) {
        REQUIRE_EQ(comms[r]->alloc(4096), off);
    }
    int fails = runThreads(n, [&](int r) {
        Communicator& c = *comms[r];
        uint8_t* base = c.heapPtr(off);
        Communicator::GroupItem aligned{ base, base, 64 };
        Communicator::GroupItem shifted{ base + 1, base + 1, 64 };
        int rc = FB_OK;
        bool ok = true;
        // an unaligned item cannot be planned
        ok = ok && c.prepareGroup(&shifted, 1, FB_U8, &rc, Communicator::GROUP_BROADCAST) == nullptr && rc == FB_E_INVALID;
        // root out of range, or a plan of another kind: nothing launched
        auto plan = c.prepareGroup(&aligned, 1, FB_U8, &rc, Communicator::GROUP_BROADCAST);
        auto arPlan = c.prepareGroup(&aligned, 1, FB_U8, &rc);
        ok = ok && plan && arPlan;
        const uint64_t l0 = c.stats().launches;
        ok = ok && c.runGroup(Communicator::GROUP_BROADCAST, *plan, 0, n, FB_FLAG_SYMMETRIC, nullptr) == FB_E_INVALID;
        ok = ok && c.runGroup(Communicator::GROUP_BROADCAST, *plan, 0, -1, FB_FLAG_SYMMETRIC, nullptr) == FB_E_INVALID;
        ok = ok && c.runGroup(Communicator::GROUP_BROADCAST, *arPlan, 0, 0, FB_FLAG_SYMMETRIC, nullptr) == FB_E_INVALID;
        ok = ok && c.groupMany(Communicator::GROUP_BROADCAST, &aligned, 1, FB_U8, 0, n, FB_FLAG_SYMMETRIC, nullptr) == FB_E_INVALID;
        ok = ok && c.stats().launches == l0;
        // the unaligned list runs one broadcast per item, with the same bytes
        for (int j = 0; j < 200; j++) {
            base[j] = pattern(r, 0, j);
        }
        Communicator::GroupItem two[2] = { shifted, { base + 100, base + 100, 37 } };
        ok = ok && c.groupMany(Communicator::GROUP_BROADCAST, two, 2, FB_U8, 0, 2, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
        for (int j = 0; j < 200 && ok; j++) {
            const bool in = (j >= 1 && j < 65) || (j >= 100 && j < 137);
            ok = base[j] == (in ? pattern(2, 0, j) : pattern(r, 0, j));
        }
        return ok && c.checkError(nullptr) == 0;
    });
    REQUIRE_EQ(fails, 0);
}

TEST_CASE("loopback subset group: every grouped kind runs on children of a parity split", "[loopback]")
{
    const int n = 8;
    auto comms = loopGroup(n);
    const uint64_t off = comms[0]->alloc(1 << 16);
    for (int r = 1; r < n; r++) {
        REQUIRE_EQ(comms[r]->alloc(1 << 16), off);
    }
    int fails = runThreads(n, [&](int r) {
        Communicator& c = *comms[r];
        std::vector<int> members;
        for (int p = r % 2; p < n; p += 2) {
            members.push_back(p);
        }
        // reversed order on the odd child: child rank 0 is parent rank 7
        if (r % 2) {
            std::reverse(members.begin(), members.end());
        }
        bool ok = true;
        for (int round = 0; round < 40 && ok; round++) {
            auto child = c.subset(members, round % 3);
            if (child == nullptr) {
                return false;
            }
            const int m = child->size();
            const int cr = child->rank();
            int32_t* buf = (int32_t*)c.heapPtr(off);
            // all-reduce of 2 tensors, in place
            for (int i = 0; i < 64; i++) {
                buf[i] = r + i + round;
            }
            Communicator::GroupItem ar[2] = { { buf, buf, 40 }, { buf + 48, buf + 48, 16 } };
            const uint64_t l0 = child->stats().launches;
            ok = ok && child->groupMany(Communicator::GROUP_ALLREDUCE, ar, 2, FB_I32, FB_OP_SUM, 0, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            int sum = 0;
            for (int p : members) {
                sum += p;
            }
            for (int i = 0; i < 40 && ok; i++) {
                ok = buf[i] == sum + m * (i + round);
            }
            // reduce-scatter: 4 int32 per member
            int32_t* rs = buf + 1024;
            int32_t* rsOut = buf + 2048;
            for (int i = 0; i < 4 * m; i++) {
                rs[i] = r * 3 + i;
            }
            Communicator::GroupItem rsIt{ rs, rsOut, 4 };
            ok = ok && child->groupMany(Communicator::GROUP_REDUCE_SCATTER, &rsIt, 1, FB_I32, FB_OP_SUM, 0, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            for (int j = 0; j < 4 && ok; j++) {
                ok = rsOut[j] == 3 * sum + m * (cr * 4 + j);
            }
            // all-gather: block q gets member q's 4 int32
            int32_t* ag = buf + 3072;
            int32_t* agOut = buf + 4096;
            for (int j = 0; j < 4; j++) {
                ag[j] = r * 10 + j;
            }
            Communicator::GroupItem agIt{ ag, agOut, 4 };
            ok = ok && child->groupMany(Communicator::GROUP_ALLGATHER, &agIt, 1, FB_I32, 0, 0, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            for (int q = 0; q < m && ok; q++) {
                for (int j = 0; j < 4 && ok; j++) {
                    ok = agOut[q * 4 + j] == members[q] * 10 + j;
                }
            }
            // broadcast from child rank round % m, 21 bytes
            uint8_t* bc = (uint8_t*)(buf + 5120);
            for (int j = 0; j < 32; j++) {
                bc[j] = pattern(r, round, j);
            }
            Communicator::GroupItem bcIt{ bc, bc, 21 };
            const int root = round % m;
            ok = ok && child->groupMany(Communicator::GROUP_BROADCAST, &bcIt, 1, FB_U8, 0, root, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            for (int j = 0; j < 32 && ok; j++) {
                ok = bc[j] == (j < 21 ? pattern(members[root], round, j) : pattern(r, round, j));
            }
            ok = ok && child->stats().launches == l0 + 4;
            // the parent in between: a grouped all-reduce over all 8 ranks
            child.reset();
            for (int i = 0; i < 8; i++) {
                buf[6144 + i] = r;
            }
            Communicator::GroupItem whole{ buf + 6144, buf + 6144, 8 };
            ok = ok && c.groupMany(Communicator::GROUP_ALLREDUCE, &whole, 1, FB_I32, FB_OP_SUM, 0, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            ok = ok && buf[6144] == n * (n - 1) / 2;
        }
        return ok && c.checkError(nullptr) == 0 && c.freeSubsetSlots() == (1u << FB_SUB_SLOTS) - 1;
    });
    REQUIRE_EQ(fails, 0);
}

TEST_CASE("loopback subset: child ranks, heap addressing, refused calls and grouped plans", "[loopback]")
{
    auto comms = loopGroup(4);
    const uint64_t off = comms[0]->alloc(4096);
    for (int r = 1; r < 4; r++) {
        REQUIRE_EQ(comms[r]->alloc(4096), off);
    }
    const std::vector<int> members{ 3, 0, 2 };
    auto child = comms[2]->subset(members, 5);
    REQUIRE(child != nullptr);
    REQUIRE(child->isSubset() && !comms[2]->isSubset());
    REQUIRE_EQ(child->rank(), 2);
    REQUIRE_EQ(child->size(), 3);
    REQUIRE(!child->hasMulticast());
    for (int i = 0; i < 3; i++) {
        REQUIRE(child->heapPtr(off, i) == comms[2]->heapPtr(off, members[i]));
    }
    REQUIRE(child->heapPtr(off) == comms[2]->heapPtr(off));
    REQUIRE(child->inHeap(comms[2]->heapPtr(off), 4096));
    REQUIRE_EQ(child->offsetOf(comms[2]->heapPtr(off)), off);
    // slot 5 of member i is the child's pad of child rank i
    const auto& d = child->devStruct();
    for (int i = 0; i < 3; i++) {
        REQUIRE(d.sig[i] == comms[members[i]]->devStruct().sig[members[i]] + 6 * FB_SIG_TOTAL_WORDS);
    }
    uint8_t* buf = comms[2]->heapPtr(off);
    uint32_t word = 0;
    REQUIRE_EQ(child->send(buf, 16, 0, nullptr), FB_E_UNSUPPORTED);
    REQUIRE_EQ(child->recv(buf, 16, 0, nullptr), FB_E_UNSUPPORTED);
    REQUIRE_EQ(child->sendRecv(buf, 16, 0, buf, 16, 0, nullptr), FB_E_UNSUPPORTED);
    REQUIRE_EQ(child->putSignal(buf, off, 16, 0, 0, 1, nullptr), FB_E_UNSUPPORTED);
    REQUIRE_EQ(child->waitSignal(0, 1, nullptr), FB_E_UNSUPPORTED);
    REQUIRE_EQ(child->accumulate(buf, off, 1, FB_I32, FB_OP_SUM, 0, nullptr, nullptr), FB_E_UNSUPPORTED);
    REQUIRE_EQ(child->compareAndSwap(&word, &word, &word, off, FB_I32, 0, nullptr), FB_E_UNSUPPORTED);
    // grouped plans are built on a child as on its parent (a local call);
    // a plan of another kind or a root outside the child is refused
    Communicator::GroupItem item{ buf, buf, 4 };
    int rc = FB_OK;
    auto plan = child->prepareGroup(&item, 1, FB_I32, &rc);
    REQUIRE(plan != nullptr);
    REQUIRE_EQ(rc, FB_OK);
    auto bplan = child->prepareGroup(&item, 1, FB_U8, &rc, Communicator::GROUP_BROADCAST);
    REQUIRE(bplan != nullptr);
    REQUIRE_EQ(child->runGroup(Communicator::GROUP_BROADCAST, *plan, 0, 0, FB_FLAG_SYMMETRIC, nullptr), FB_E_INVALID);
    REQUIRE_EQ(child->runGroup(Communicator::GROUP_BROADCAST, *bplan, 0, 3, FB_FLAG_SYMMETRIC, nullptr), FB_E_INVALID);
    REQUIRE_EQ(child->runGroup(Communicator::GROUP_BROADCAST, *bplan, 0, -1, FB_FLAG_SYMMETRIC, nullptr), FB_E_INVALID);
    REQUIRE_EQ(child->runGroup(Communicator::GROUP_ALLREDUCE, *bplan, FB_OP_SUM, 0, FB_FLAG_SYMMETRIC, nullptr), FB_E_INVALID);
    REQUIRE_EQ(child->groupMany(Communicator::GROUP_BROADCAST, &item, 1, FB_U8, 0, 3, FB_FLAG_SYMMETRIC, nullptr), FB_E_INVALID);
    REQUIRE_EQ(child->hostBarrier(), FB_E_UNSUPPORTED);
    REQUIRE_EQ(child->allReduce(buf, buf, 4, FB_I32, FB_OP_SUM, FB_ALGO_LL, FB_FLAG_SYMMETRIC, nullptr), FB_E_UNSUPPORTED);
    REQUIRE_EQ(child->allReduce(buf, buf, 4, FB_I32, FB_OP_SUM, FB_ALGO_NVLS, FB_FLAG_SYMMETRIC, nullptr), FB_E_UNSUPPORTED);
    bool threw = false;
    try {
        child->alloc(256);
    } catch (const std::logic_error&) {
        threw = true;
    }
    REQUIRE(threw);
    threw = false;
    try {
        child->free(off);
    } catch (const std::logic_error&) {
        threw = true;
    }
    REQUIRE(threw);
    // nothing was launched by the refused calls or the plans
    REQUIRE_EQ(child->stats().launches, 0u);
}


namespace {
void runGroupSubcommMpi(const std::string& name, int worldSize)
{
    using namespace tests;
    ClusterFixture f(worldSize);
    registerTestFunction("mpi", name, [&](auto*, int, int, auto) {
        MPI_Init(nullptr, nullptr);
        int rank = -1, size = -1;
        MPI_Comm_rank(MPI_COMM_WORLD, &rank);
        MPI_Comm_size(MPI_COMM_WORLD, &size);
        std::string why;
        faabric::Message& msg = faabric::executor::ExecutorContext::get()->getMsg();
        int rc = group_subcomm::body(rank, size, msg.mpiworldid(), &why);
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

TEST_CASE("loopback group broadcast: MPI_Ibcast bursts and grouped bursts on sub-communicators", "[loopback][mpi]")
{
    tests::LoopbackBackend loopback;
    runGroupSubcommMpi("group-subcomm-loopback-2", 2);
    runGroupSubcommMpi("group-subcomm-loopback-4", 4);
}
