// Grouped all-to-all (Communicator::runGroup / groupMany, GROUP_ALLTOALL) on the
// loopback backend (no GPU): every byte of the buffers, random guard bytes
// between blocks included, against an exchange computed on the host at 1-8
// ranks; launch counts; refusals and fall-backs; a plan on a sub-communicator
// child; and the MPI program of mpi_group_alltoall_body.h.
#include "fixtures.h"
#include "mpi_group_alltoall_body.h"

#include <faabric/device/communicator.h>
#include <faabric/executor/ExecutorContext.h>

#include "launch_api.h"

#include <atomic>
#include <cstdlib>
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

// One item at byte offsets of the heap region: `block` bytes per block
struct Item
{
    size_t send;
    size_t recv;
    size_t block;
};

// A region of `bytes` at the same heap offset on every rank, filled with
// random bytes per rank; expect() computes what a list of items leaves there
struct Region
{
    std::vector<std::shared_ptr<Communicator>> comms;
    uint64_t off = 0;
    size_t bytes = 0;
    std::vector<std::vector<uint8_t>> before;

    Region(std::vector<std::shared_ptr<Communicator>> cs, size_t b)
      : comms(std::move(cs))
      , bytes(b)
    {
        off = comms[0]->alloc(bytes);
        for (size_t r = 1; r < comms.size(); r++) {
            REQUIRE_EQ(comms[r]->alloc(bytes), off);
        }
    }

    uint8_t* at(int r) { return comms[r]->heapPtr(off); }

    void randomise(uint32_t seed)
    {
        before.assign(comms.size(), std::vector<uint8_t>(bytes));
        for (size_t r = 0; r < comms.size(); r++) {
            std::mt19937 rng(seed * 131 + (uint32_t)r);
            for (auto& v : before[r]) {
                v = (uint8_t)rng();
            }
            memcpy(at((int)r), before[r].data(), bytes);
        }
    }

    // The items run one after another (MPI_Alltoall per item, in list order):
    // block q of item i's recv on rank p is block p of its send on rank q
    std::vector<std::vector<uint8_t>> expect(const std::vector<Item>& items) const
    {
        const size_t n = comms.size();
        auto cur = before;
        for (const Item& it : items) {
            auto next = cur;
            for (size_t p = 0; p < n; p++) {
                for (size_t q = 0; q < n; q++) {
                    memcpy(next[p].data() + it.recv + q * it.block, cur[q].data() + it.send + p * it.block, it.block);
                }
            }
            cur = std::move(next);
        }
        return cur;
    }

    bool matches(const std::vector<std::vector<uint8_t>>& want)
    {
        for (size_t r = 0; r < comms.size(); r++) {
            const uint8_t* got = at((int)r);
            for (size_t j = 0; j < bytes; j++) {
                if (got[j] != want[r][j]) {
                    printf("         rank %zu byte %zu: %u, want %u\n", r, j, got[j], want[r][j]);
                    return false;
                }
            }
        }
        return true;
    }
};

// Blocks of 16 bytes, a count of 0, ragged chunk ends (the chunk is 64
// vectors at 8 ranks, 128 at 2-5, 256 at 1) and several whole chunks
const std::vector<size_t> BLOCKS = { 16, 0, 48, 4096 + 48, 2048, 16 * 300, 16 * 1111, 16 * 65 };

// Sends then recvs, each n blocks long, with a random gap of 16-64 bytes
// before every buffer (so every block has guard bytes around it)
std::vector<Item> layout(int n, size_t& end, std::mt19937& rng)
{
    std::vector<Item> items;
    size_t pos = 0;
    for (size_t b : BLOCKS) {
        Item it;
        pos += 16 * (1 + rng() % 4);
        it.send = pos;
        pos += b * n;
        pos += 16 * (1 + rng() % 4);
        it.recv = pos;
        pos += b * n;
        it.block = b;
        items.push_back(it);
    }
    end = pos + 64;
    return items;
}

std::vector<Communicator::GroupItem> groupItems(Communicator& c, uint8_t* base, const std::vector<Item>& items, size_t esize)
{
    std::vector<Communicator::GroupItem> g;
    for (const Item& it : items) {
        g.push_back({ base + it.send, base + it.recv, it.block / esize });
    }
    return g;
}
}

TEST_CASE("loopback group alltoall: plans and transient lists byte-exact at 1-8 ranks", "[loopback]")
{
    for (int n : { 1, 2, 3, 4, 5, 8 }) {
        std::mt19937 rng(n);
        size_t bytes = 0;
        const auto items = layout(n, bytes, rng);
        Region reg(loopGroup(n), bytes);
        // (the dtype only sets the unit of count: a byte copy)
        for (int dtype : { FB_U8, FB_I32, FB_F64, FB_BF16 }) {
            const size_t es = fbDtypeSize(dtype);
            for (int usePlan = 0; usePlan < 2; usePlan++) {
                reg.randomise((uint32_t)(n * 100 + dtype * 2 + usePlan));
                const auto want = reg.expect(items);
                int fails = runThreads(n, [&](int r) {
                    Communicator& c = *reg.comms[r];
                    auto list = groupItems(c, reg.at(r), items, es);
                    const uint64_t l0 = c.stats().launches;
                    const uint64_t b0 = c.stats().bytes;
                    if (usePlan) {
                        int rc = FB_OK;
                        auto plan = c.prepareGroup(list.data(), list.size(), dtype, &rc, Communicator::GROUP_ALLTOALL);
                        if (plan == nullptr || Communicator::groupPlanLaunches(*plan) != 1 ||
                            c.runGroup(Communicator::GROUP_ALLTOALL, *plan, 0, 0, FB_FLAG_SYMMETRIC, nullptr) != FB_OK) {
                            return false;
                        }
                    } else if (c.groupMany(Communicator::GROUP_ALLTOALL, list.data(), list.size(), dtype, 0, 0, FB_FLAG_SYMMETRIC, nullptr) != FB_OK) {
                        return false;
                    }
                    size_t total = 0;
                    for (const Item& it : items) {
                        total += it.block * n;
                    }
                    // one launch, also on one rank (a local copy)
                    return c.stats().launches == l0 + 1 && c.stats().bytes == b0 + total && c.checkError(nullptr) == 0;
                });
                REQUIRE_EQ(fails, 0);
                REQUIRE(reg.matches(want));
            }
        }
    }
}

TEST_CASE("loopback group alltoall: 1017 items take two launches, 1016 one", "[loopback]")
{
    const int n = 3;
    const size_t items = 1017;
    Region reg(loopGroup(n), items * 2 * 16 * n + 4096);
    for (size_t cnt : { (size_t)1016, items }) {
        std::vector<Item> list;
        for (size_t i = 0; i < cnt; i++) {
            // one 16-byte block per rank; zero-count items in between
            list.push_back({ i * 2 * 16 * n, i * 2 * 16 * n + 16 * n, i % 7 == 3 ? (size_t)0 : (size_t)16 });
        }
        reg.randomise((uint32_t)cnt);
        const auto want = reg.expect(list);
        int fails = runThreads(n, [&](int r) {
            Communicator& c = *reg.comms[r];
            auto g = groupItems(c, reg.at(r), list, 4);
            const uint64_t l0 = c.stats().launches;
            if (c.groupMany(Communicator::GROUP_ALLTOALL, g.data(), g.size(), FB_F32, 0, 0, FB_FLAG_SYMMETRIC, nullptr) != FB_OK) {
                return false;
            }
            int rc = FB_OK;
            auto plan = c.prepareGroup(g.data(), g.size(), FB_F32, &rc, Communicator::GROUP_ALLTOALL);
            const size_t per = cnt == items ? 2 : 1;
            return c.stats().launches == l0 + per && plan != nullptr && Communicator::groupPlanLaunches(*plan) == per;
        });
        REQUIRE_EQ(fails, 0);
        REQUIRE(reg.matches(want));
    }
}

TEST_CASE("loopback group alltoall: unaligned, off-heap and overlapping lists are refused and fall back", "[loopback]")
{
    const int n = 4;
    const size_t B = 64;
    Region reg(loopGroup(n), 8192);
    std::vector<std::vector<uint8_t>> offHeap(n, std::vector<uint8_t>(B * n + 64));
    // recv of item 1 is the send of item 0: in list order, item 0 reads it
    // before item 1 overwrites it
    const std::vector<Item> overlap = { { 0, 1024, B }, { 2048, 0, B } };
    const std::vector<Item> shifted = { { 4, 1024 + 4, B }, { 2048, 3072, B } };
    const std::vector<Item> aligned = { { 0, 1024, B } };
    for (int which = 0; which < 3; which++) {
        const std::vector<Item>& list = which == 0 ? overlap : which == 1 ? shifted : aligned;
        reg.randomise((uint32_t)(which + 7));
        for (auto& h : offHeap) {
            std::fill(h.begin(), h.end(), 0xEE);
        }
        auto want = reg.expect(list);
        int fails = runThreads(n, [&](int r) {
            Communicator& c = *reg.comms[r];
            auto g = groupItems(c, reg.at(r), list, 1);
            if (which == 2) {
                g[0].recv = offHeap[r].data() + 16; // outside the heap
            }
            int rc = FB_OK;
            bool ok = c.prepareGroup(g.data(), g.size(), FB_U8, &rc, Communicator::GROUP_ALLTOALL) == nullptr &&
                      rc == FB_E_INVALID;
            const uint64_t l0 = c.stats().launches;
            ok = ok && c.groupMany(Communicator::GROUP_ALLTOALL, g.data(), g.size(), FB_U8, 0, 0, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            // one per-item allToAll per item
            return ok && c.stats().launches == l0 + g.size() && c.checkError(nullptr) == 0;
        });
        REQUIRE_EQ(fails, 0);
        if (which == 2) {
            // the heap keeps its bytes; block q of the off-heap recv on rank p
            // is block p of the send on rank q
            want = reg.expect({});
            for (int p = 0; p < n; p++) {
                for (int q = 0; q < n; q++) {
                    REQUIRE(memcmp(offHeap[p].data() + 16 + q * B, reg.before[q].data() + p * B, B) == 0);
                }
                REQUIRE(offHeap[p][15] == 0xEE);
                REQUIRE(offHeap[p][16 + n * B] == 0xEE);
            }
        }
        REQUIRE(reg.matches(want));
    }
    // a plan of another kind, and an all-to-all plan given to another call
    int fails = runThreads(n, [&](int r) {
        Communicator& c = *reg.comms[r];
        auto g = groupItems(c, reg.at(r), aligned, 1);
        int rc = FB_OK;
        auto a2a = c.prepareGroup(g.data(), g.size(), FB_U8, &rc, Communicator::GROUP_ALLTOALL);
        auto ag = c.prepareGroup(g.data(), g.size(), FB_U8, &rc, Communicator::GROUP_ALLGATHER);
        const uint64_t l0 = c.stats().launches;
        bool ok = a2a && ag;
        ok = ok && c.runGroup(Communicator::GROUP_ALLTOALL, *ag, 0, 0, FB_FLAG_SYMMETRIC, nullptr) == FB_E_INVALID;
        ok = ok && c.runGroup(Communicator::GROUP_ALLGATHER, *a2a, 0, 0, FB_FLAG_SYMMETRIC, nullptr) == FB_E_INVALID;
        ok = ok && c.runGroup(Communicator::GROUP_BROADCAST, *a2a, 0, 0, FB_FLAG_SYMMETRIC, nullptr) == FB_E_INVALID;
        return ok && c.stats().launches == l0;
    });
    REQUIRE_EQ(fails, 0);
}

TEST_CASE("loopback group alltoall: a plan on a subset child exchanges among its members", "[loopback]")
{
    const int n = 8;
    const size_t B = 48;
    Region reg(loopGroup(n), 4096);
    reg.randomise(99);
    // reversed odd members: child rank 0 is parent rank 7
    auto membersOf = [](int r) {
        std::vector<int> m;
        for (int p = r % 2; p < 8; p += 2) {
            m.push_back(p);
        }
        if (r % 2) {
            std::reverse(m.begin(), m.end());
        }
        return m;
    };
    const Item it{ 32, 1024, B };
    int fails = runThreads(n, [&](int r) {
        Communicator& c = *reg.comms[r];
        auto child = c.subset(membersOf(r), 2);
        if (child == nullptr) {
            return false;
        }
        Communicator::GroupItem g{ reg.at(r) + it.send, reg.at(r) + it.recv, B / 16 };
        int rc = FB_OK;
        // (16-byte elements: one per block)
        auto plan = child->prepareGroup(&g, 1, FB_F64_I32, &rc, Communicator::GROUP_ALLTOALL);
        const uint64_t l0 = child->stats().launches;
        const bool ok = plan != nullptr && child->runGroup(Communicator::GROUP_ALLTOALL, *plan, 0, 0, FB_FLAG_SYMMETRIC, nullptr) == FB_OK &&
                        child->stats().launches == l0 + 1;
        plan.reset();
        child.reset();
        return ok && c.checkError(nullptr) == 0;
    });
    REQUIRE_EQ(fails, 0);
    // expected: the exchange among each parity's members, in child rank order
    auto want = reg.before;
    for (int r = 0; r < n; r++) {
        const auto m = membersOf(r);
        const int cr = (int)(std::find(m.begin(), m.end(), r) - m.begin());
        for (size_t q = 0; q < m.size(); q++) {
            memcpy(want[r].data() + it.recv + q * B, reg.before[m[q]].data() + it.send + cr * B, B);
        }
    }
    REQUIRE(reg.matches(want));
}

namespace {
void runGroupAllToAllMpi(const std::string& name, int worldSize, bool grouped)
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
        int rc = group_alltoall::body(rank, size, msg.mpiworldid(), grouped, &why);
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
}

TEST_CASE("loopback group alltoall: MPI_Ialltoall bursts on the world and on sub-communicators", "[loopback][mpi]")
{
    tests::LoopbackBackend loopback;
    runGroupAllToAllMpi("group-alltoall-loopback-2", 2, true);
    runGroupAllToAllMpi("group-alltoall-loopback-4", 4, true);
    runGroupAllToAllMpi("group-alltoall-loopback-ungrouped-4", 4, false);
}
