// Grouped gather and scatter (Communicator::runGroup / groupMany,
// GROUP_GATHER and GROUP_SCATTER) on the loopback backend (no GPU): every
// byte of every rank's buffers, guard bytes included, against a gather or
// scatter computed on the host at 1-8 ranks, every root, in place and not,
// items larger than the staging buffer; launch counts; the refusals; and the
// MPI program of mpi_group_rooted_body.h.
#include "fixtures.h"
#include "mpi_group_rooted_run.h"

#include <faabric/device/communicator.h>

#include <atomic>
#include <cstring>
#include <functional>
#include <random>
#include <thread>

using faabric::device::CommConfig;
using faabric::device::Communicator;

namespace {
const size_t STAGE = (size_t)1 << 20;

std::vector<std::shared_ptr<Communicator>> rootedGroup(int n, size_t stage = STAGE)
{
    CommConfig cfg;
    cfg.loopback = true;
    cfg.heapBytes = (size_t)4 << 20;
    cfg.stageBytes = stage;
    cfg.p2pBounceBytes = (size_t)1 << 20;
    cfg.channels = 2;
    cfg.maxBlocks = 4;
    cfg.timeoutMs = 5000;
    return Communicator::createLocal(n, std::vector<int>(n, 0), cfg);
}

int runRanks(int n, const std::function<bool(int)>& fn)
{
    std::atomic<int> failures{ 0 };
    std::vector<std::thread> ts;
    for (int i = 0; i < n; i++) {
        ts.emplace_back([&, i] {
            if (!fn(i)) {
                failures++;
            }
        });
    }
    for (auto& t : ts) {
        t.join();
    }
    return failures.load();
}

// Every rank's items in one host buffer (plain memory: the user side of the
// rooted kinds is any memory), a guard before each, offsets off 16-byte
// alignment by `shift`
struct RootedCase
{
    bool gather;
    int n;
    int root;
    bool inPlace;
    std::vector<size_t> sizes;
    std::vector<std::vector<uint8_t>> buf, want;
    std::vector<std::vector<size_t>> sendOff, recvOff;

    RootedCase(bool g, int nranks, int r, bool ip, std::vector<size_t> sz, size_t shift, std::mt19937& rng)
      : gather(g)
      , n(nranks)
      , root(r)
      , inPlace(ip)
      , sizes(std::move(sz))
      , buf(nranks)
      , sendOff(nranks)
      , recvOff(nranks)
    {
        size_t pos = 32 + shift;
        for (size_t b : sizes) {
            const size_t single = pos;
            const size_t blocks = (pos + b + 15) / 16 * 16 + 32 + shift;
            pos = (blocks + b * n + 15) / 16 * 16 + 32 + shift;
            for (int p = 0; p < n; p++) {
                const size_t own = inPlace && p == root ? blocks + root * b : single;
                sendOff[p].push_back(gather ? own : blocks);
                recvOff[p].push_back(gather ? blocks : own);
            }
        }
        for (auto& v : buf) {
            v.resize(pos + 32);
            for (auto& x : v) {
                x = (uint8_t)rng();
            }
        }
        want = buf;
        for (size_t i = 0; i < sizes.size(); i++) {
            const size_t b = sizes[i];
            for (int p = 0; p < n; p++) {
                if (gather) {
                    memmove(&want[root][recvOff[root][i] + p * b], &buf[p][sendOff[p][i]], b);
                } else {
                    memmove(&want[p][recvOff[p][i]], &buf[root][sendOff[root][i] + p * b], b);
                }
            }
        }
    }

    // rank p's items: the root-only side is null elsewhere
    std::vector<Communicator::GroupItem> items(int p)
    {
        std::vector<Communicator::GroupItem> out;
        for (size_t i = 0; i < sizes.size(); i++) {
            const bool rootSide = p == root;
            Communicator::GroupItem it;
            it.send = gather || rootSide ? &buf[p][sendOff[p][i]] : nullptr;
            it.recv = !gather || rootSide ? &buf[p][recvOff[p][i]] : nullptr;
            it.count = sizes[i];
            out.push_back(it);
        }
        return out;
    }
};

uint64_t chunkBytes(int n)
{
    return n == 8 ? 1024 : (n == 1 ? 4096 : 2048);
}
}

TEST_CASE("loopback group rooted: every byte at 1-8 ranks, every root, in place, pieces", "[loopback]")
{
    std::mt19937 rng(42);
    for (int n = 1; n <= 8; n++) {
        auto comms = rootedGroup(n);
        for (int gather = 0; gather < 2; gather++) {
            const auto kind = gather ? Communicator::GROUP_GATHER : Communicator::GROUP_SCATTER;
            for (int root = 0; root < n; root++) {
                const bool inPlace = root % 2 == 1;
                const bool many = (root + n) % 2 == 0;
                // one byte, zero, odd, ragged chunk ends, and more than the
                // staging buffer (cut into pieces over several launches)
                RootedCase c(gather, n, root, inPlace, { 1, 0, 5, 2049, 300000, 3 * STAGE + 17 }, root % 3, rng);
                uint64_t chunks = 0;
                for (size_t b : c.sizes) {
                    chunks += (b + chunkBytes(n) - 1) / chunkBytes(n);
                }
                const uint64_t room = STAGE / chunkBytes(n);
                const uint64_t launches = (chunks + room - 1) / room;
                std::vector<uint64_t> got(n);
                const int fails = runRanks(n, [&](int p) {
                    auto& comm = *comms[p];
                    auto items = c.items(p);
                    int rc = FB_OK;
                    auto plan = comm.prepareGroup(items.data(), items.size(), FB_U8, &rc, kind);
                    if (!plan || Communicator::groupPlanLaunches(*plan) != launches) {
                        return false;
                    }
                    const uint64_t before = comm.stats().launches;
                    rc = many ? comm.groupMany(kind, items.data(), items.size(), FB_U8, 0, root, 0, nullptr)
                              : comm.runGroup(kind, *plan, 0, root, 0, nullptr);
                    got[p] = comm.stats().launches - before;
                    return rc == FB_OK && comm.peekError() == 0;
                });
                REQUIRE(fails == 0);
                for (int p = 0; p < n; p++) {
                    REQUIRE(got[p] == launches);
                    REQUIRE(c.buf[p] == c.want[p]);
                }
            }
        }
    }
}

TEST_CASE("loopback group rooted: 1016 items take one launch, 1017 two", "[loopback]")
{
    std::mt19937 rng(7);
    // (every item takes a whole 2 KiB chunk of staging: 1016 of them fit 4 MiB)
    auto comms = rootedGroup(3, (size_t)4 << 20);
    for (size_t k : { (size_t)1016, (size_t)1017 }) {
        RootedCase c(true, 3, 2, false, std::vector<size_t>(k, 4), 1, rng);
        const int fails = runRanks(3, [&](int p) {
            auto items = c.items(p);
            const uint64_t before = comms[p]->stats().launches;
            const int rc = comms[p]->groupMany(Communicator::GROUP_GATHER, items.data(), k, FB_U8, 0, 2, 0, nullptr);
            return rc == FB_OK && comms[p]->stats().launches - before == (k == 1016 ? 1u : 2u);
        });
        REQUIRE(fails == 0);
        for (int p = 0; p < 3; p++) {
            REQUIRE(c.buf[p] == c.want[p]);
        }
    }
}

TEST_CASE("loopback group rooted: refusals", "[loopback]")
{
    std::mt19937 rng(9);
    auto comms = rootedGroup(2);
    RootedCase c(false, 2, 0, false, { 64, 100 }, 0, rng);
    auto items = c.items(0);
    int rc = FB_OK;
    auto plan = comms[0]->prepareGroup(items.data(), items.size(), FB_U8, &rc, Communicator::GROUP_SCATTER);
    REQUIRE(plan != nullptr);
    const uint64_t before = comms[0]->stats().launches;
    // nothing is launched: no peer is left at a barrier
    REQUIRE(comms[0]->runGroup(Communicator::GROUP_GATHER, *plan, 0, 0, 0, nullptr) == FB_E_INVALID);
    REQUIRE(comms[0]->runGroup(Communicator::GROUP_SCATTER, *plan, 0, 2, 0, nullptr) == FB_E_INVALID);
    REQUIRE(comms[0]->runGroup(Communicator::GROUP_SCATTER, *plan, 0, -1, 0, nullptr) == FB_E_INVALID);
    REQUIRE(comms[0]->runGroup(Communicator::GROUP_SCATTER, *plan, 0, 0, FB_FLAG_CHANNEL(1), nullptr) ==
          FB_E_INVALID);
    REQUIRE(comms[0]->groupMany(Communicator::GROUP_GATHER, items.data(), items.size(), FB_U8, 0, 5, 0, nullptr) ==
          FB_E_INVALID);
    REQUIRE(comms[0]->groupMany(Communicator::GROUP_SCATTER, items.data(), items.size(), FB_U8, 0, 0,
                              FB_FLAG_CHANNEL(2), nullptr) == FB_E_INVALID);
    // the root needs both sides: rank 0 of a scatter rooted at 0 without recv
    items[1].recv = nullptr;
    REQUIRE(comms[0]->groupMany(Communicator::GROUP_SCATTER, items.data(), items.size(), FB_U8, 0, 0, 0, nullptr) ==
          FB_E_INVALID);
    REQUIRE(comms[0]->stats().launches == before);
    REQUIRE(std::string(Communicator::groupKindName(Communicator::GROUP_GATHER)) == "gather");
    REQUIRE(std::string(Communicator::groupKindName(Communicator::GROUP_SCATTER)) == "scatter");
}

TEST_CASE("loopback group rooted: one member copies, or does nothing in place", "[loopback]")
{
    std::mt19937 rng(3);
    auto comms = rootedGroup(1);
    for (int gather = 0; gather < 2; gather++) {
        for (bool inPlace : { false, true }) {
            RootedCase c(gather, 1, 0, inPlace, { 3, 4096, 70001 }, 5, rng);
            auto items = c.items(0);
            const auto kind = gather ? Communicator::GROUP_GATHER : Communicator::GROUP_SCATTER;
            REQUIRE(comms[0]->groupMany(kind, items.data(), items.size(), FB_U8, 0, 0, 0, nullptr) == FB_OK);
            REQUIRE(c.buf[0] == c.want[0]);
        }
    }
}

TEST_CASE("loopback group rooted: MPI_Igather and MPI_Iscatter bursts on the world and on sub-communicators",
          "[loopback][mpi]")
{
    tests::LoopbackBackend loopback;
    runMpiGroupRootedBody(true);
}
