// Grouped neighbourhood all-gather and all-to-all (Communicator::runGroup /
// groupMany, GROUP_NEIGHBOR_ALLGATHER and GROUP_NEIGHBOR_ALLTOALL) on the
// loopback backend (no GPU): every byte of every rank's buffers, guard bytes
// included, against an exchange computed on the host over seeded random
// graphs with self-edges, multi-edges and ranks of degree 0, at 1-8 ranks;
// heap and plain buffers off 16-byte alignment; bursts cut into several
// launches; a plan on a subset child; and the refusals.
#include "harness.h"

#include <faabric/device/communicator.h>

#include <algorithm>
#include <atomic>
#include <cstring>
#include <functional>
#include <random>
#include <thread>

using faabric::device::CommConfig;
using faabric::device::Communicator;

namespace {
const size_t STAGE = (size_t)256 << 10;
const uint64_t CB = 2048; // FB_NEIGHBOR_CHUNK

std::vector<std::shared_ptr<Communicator>> neighborGroup(int n, size_t stage = STAGE)
{
    CommConfig cfg;
    cfg.loopback = true;
    cfg.heapBytes = (size_t)8 << 20;
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

// A graph by its adjacency lists, and every rank's in-edges: source j of
// rank d is the k-th occurrence of that source in d's list, so it pairs with
// the k-th occurrence of d in the source's destinations (MPI-3.1 7.6)
struct Graph
{
    int n = 0;
    std::vector<std::vector<int>> dst, src;
    std::vector<std::vector<std::pair<int, int>>> in;
    int maxOut = 0, maxIn = 0;

    Graph(std::vector<std::vector<int>> d, std::vector<std::vector<int>> s)
      : n((int)d.size())
      , dst(std::move(d))
      , src(std::move(s))
      , in(n)
    {
        for (int r = 0; r < n; r++) {
            std::vector<int> seen(n, 0);
            for (int s : src[r]) {
                int k = seen[s]++;
                int idx = -1;
                for (size_t i = 0; i < dst[s].size() && idx < 0; i++) {
                    if (dst[s][i] == r && k-- == 0) {
                        idx = (int)i;
                    }
                }
                in[r].push_back({ s, idx });
            }
            maxOut = std::max(maxOut, (int)dst[r].size());
            maxIn = std::max(maxIn, (int)src[r].size());
        }
    }

    static Graph random(int n, int maxDeg, std::mt19937& rng)
    {
        std::vector<std::vector<int>> d(n), s(n);
        for (int r = 0; r < n; r++) {
            // every third rank (from a seeded start) sends nothing
            const int deg = (r + (int)(rng() % 3)) % 3 == 0 ? 0 : 1 + (int)(rng() % maxDeg);
            for (int k = 0; k < deg; k++) {
                const int t = (int)(rng() % n);
                d[r].push_back(t);
                s[t].push_back(r);
            }
        }
        for (auto& v : s) {
            std::shuffle(v.begin(), v.end(), rng);
        }
        return Graph(d, s);
    }

    void set(Communicator& c, int r) const
    {
        REQUIRE(c.setNeighbors(in[r], (int)dst[r].size(), maxOut, maxIn) == FB_OK);
    }
};

// Every rank's items in one buffer (plain memory or its heap), a guard before
// each, offsets off 16-byte alignment by `shift`
struct NeighborCase
{
    const Graph& g;
    bool a2a;
    std::vector<size_t> sizes;
    std::vector<uint8_t*> base;
    std::vector<std::vector<uint8_t>> host, want;
    std::vector<std::vector<size_t>> sendOff, recvOff;

    NeighborCase(const Graph& graph, bool allToAll, std::vector<size_t> sz, size_t shift, std::mt19937& rng,
                 std::vector<std::shared_ptr<Communicator>>* heapOf = nullptr)
      : g(graph)
      , a2a(allToAll)
      , sizes(std::move(sz))
      , base(g.n)
      , host(g.n)
      , sendOff(g.n)
      , recvOff(g.n)
    {
        size_t len = 0;
        for (int p = 0; p < g.n; p++) {
            size_t pos = 32 + shift;
            for (size_t b : sizes) {
                sendOff[p].push_back(pos);
                pos = (pos + b * (a2a ? g.dst[p].size() : 1) + 15) / 16 * 16 + 32 + shift;
                recvOff[p].push_back(pos);
                pos = (pos + b * g.src[p].size() + 15) / 16 * 16 + 32 + shift;
            }
            host[p].resize(pos + 32);
            for (auto& x : host[p]) {
                x = (uint8_t)rng();
            }
            len = std::max(len, pos + 32);
        }
        for (int p = 0; p < g.n; p++) {
            if (heapOf != nullptr) {
                // (the heap allocator is collective: the same size on every rank)
                base[p] = (*heapOf)[p]->heapPtr((*heapOf)[p]->alloc(len));
                memcpy(base[p], host[p].data(), host[p].size());
            } else {
                base[p] = host[p].data();
            }
        }
        want = host;
        for (size_t i = 0; i < sizes.size(); i++) {
            const size_t b = sizes[i];
            for (int d = 0; d < g.n; d++) {
                for (size_t j = 0; j < g.in[d].size(); j++) {
                    const auto [s, idx] = g.in[d][j];
                    memcpy(&want[d][recvOff[d][i] + j * b], &host[s][sendOff[s][i] + (a2a ? idx * b : 0)], b);
                }
            }
        }
    }

    Communicator::GroupKind kind() const
    {
        return a2a ? Communicator::GROUP_NEIGHBOR_ALLTOALL : Communicator::GROUP_NEIGHBOR_ALLGATHER;
    }

    std::vector<Communicator::GroupItem> items(int p) const
    {
        std::vector<Communicator::GroupItem> out;
        for (size_t i = 0; i < sizes.size(); i++) {
            out.push_back({ base[p] + sendOff[p][i], base[p] + recvOff[p][i], sizes[i] });
        }
        return out;
    }

    bool matches(int p) const { return memcmp(base[p], want[p].data(), want[p].size()) == 0; }

    // launches of the list: the staging room per launch is shared by the
    // largest out-degree's slots (all-to-all)
    uint64_t launches(size_t stage) const
    {
        uint64_t chunks = 0;
        for (size_t b : sizes) {
            chunks += (b + CB - 1) / CB;
        }
        const uint64_t room = stage / CB / (a2a ? std::max(g.maxOut, 1) : 1);
        return (chunks + room - 1) / room;
    }
};
}

TEST_CASE("loopback group neighbor: every byte over random graphs at 1-8 ranks, plans and many, heap and plain",
          "[loopback]")
{
    std::mt19937 rng(1234);
    for (int n : { 1, 2, 3, 4, 5, 8 }) {
        for (int round = 0; round < 2; round++) {
            auto comms = neighborGroup(n);
            const Graph g = Graph::random(n, 3, rng);
            for (int p = 0; p < n; p++) {
                g.set(*comms[p], p);
            }
            for (int a2a = 0; a2a < 2; a2a++) {
                for (int heap = 0; heap < 2; heap++) {
                    const bool many = (round + a2a + heap) % 2 == 1;
                    // one byte, zero, odd, ragged chunk ends, and more than a
                    // launch's staging room (cut into pieces)
                    std::vector<size_t> sizes = { 1, 0, 5, 2049, 70001 };
                    if (!heap) {
                        sizes.push_back(STAGE + 17);
                    }
                    NeighborCase c(g, a2a, sizes, (size_t)(n + round + heap) % 5, rng, heap ? &comms : nullptr);
                    const uint64_t launches = c.launches(STAGE);
                    std::vector<uint64_t> got(n), tables(n);
                    const int fails = runRanks(n, [&](int p) {
                        auto& comm = *comms[p];
                        auto items = c.items(p);
                        int rc = FB_OK;
                        auto plan = comm.prepareGroup(items.data(), items.size(), FB_U8, &rc, c.kind());
                        if (!plan || Communicator::groupPlanLaunches(*plan) != launches) {
                            return false;
                        }
                        const uint64_t before = comm.stats().launches;
                        const uint64_t t0 = comm.stats().segTables;
                        rc = many ? comm.groupMany(c.kind(), items.data(), items.size(), FB_U8, 0, 0, 0, nullptr)
                                  : comm.runGroup(c.kind(), *plan, 0, 0, 0, nullptr);
                        got[p] = comm.stats().launches - before;
                        tables[p] = comm.stats().segTables - t0;
                        return rc == FB_OK && comm.peekError() == 0;
                    });
                    REQUIRE(fails == 0);
                    for (int p = 0; p < n; p++) {
                        // (a graph with no edge launches nothing)
                        REQUIRE(got[p] == (g.maxIn == 0 ? 0 : launches));
                        REQUIRE(tables[p] == (many && g.maxIn > 0 ? launches : 0));
                        REQUIRE(c.matches(p));
                    }
                }
            }
        }
    }
}

TEST_CASE("loopback group neighbor: a 2x1 periodic halo has multi-edges, a one-member ring only self-edges",
          "[loopback]")
{
    std::mt19937 rng(5);
    // 2 x 1 periodic grid, 4 neighbours (left, right, down, up): left and
    // right are the other rank, down and up the rank itself
    {
        const Graph g({ { 1, 1, 0, 0 }, { 0, 0, 1, 1 } }, { { 1, 1, 0, 0 }, { 0, 0, 1, 1 } });
        REQUIRE((g.in[0] == std::vector<std::pair<int, int>>{ { 1, 0 }, { 1, 1 }, { 0, 2 }, { 0, 3 } }));
        auto comms = neighborGroup(2);
        for (int p = 0; p < 2; p++) {
            g.set(*comms[p], p);
        }
        NeighborCase c(g, true, { 4096, 100, 7 }, 3, rng);
        REQUIRE(runRanks(2, [&](int p) {
                    auto items = c.items(p);
                    return comms[p]->groupMany(c.kind(), items.data(), items.size(), FB_U8, 0, 0, 0, nullptr) ==
                           FB_OK;
                }) == 0);
        REQUIRE(c.matches(0));
        REQUIRE(c.matches(1));
    }
    // one member: self-edges are a local copy; no edge, no launch
    for (int edges : { 2, 0 }) {
        const Graph g({ std::vector<int>(edges, 0) }, { std::vector<int>(edges, 0) });
        auto comms = neighborGroup(1);
        g.set(*comms[0], 0);
        for (bool a2a : { false, true }) {
            NeighborCase c(g, a2a, { 3, 4096, 70001 }, 5, rng);
            auto items = c.items(0);
            const uint64_t before = comms[0]->stats().launches;
            REQUIRE(comms[0]->groupMany(c.kind(), items.data(), items.size(), FB_U8, 0, 0, 0, nullptr) == FB_OK);
            REQUIRE(comms[0]->stats().launches - before == (edges ? 1u : 0u));
            REQUIRE(c.matches(0));
        }
    }
}

TEST_CASE("loopback group neighbor: 1016 items take one launch, 1017 two; a small staging buffer cuts a burst",
          "[loopback]")
{
    std::mt19937 rng(7);
    const Graph g({ { 1, 2 }, { 2 }, { 0, 0, 1 } }, { { 2, 2 }, { 0, 2 }, { 1, 0 } });
    // (every item takes a whole 2 KiB chunk of staging per slot: 1016 of them
    // fit 3 slots of 6 MiB)
    auto comms = neighborGroup(3, (size_t)6 << 20);
    for (int p = 0; p < 3; p++) {
        g.set(*comms[p], p);
    }
    for (size_t k : { (size_t)1016, (size_t)1017 }) {
        NeighborCase c(g, true, std::vector<size_t>(k, 4), 1, rng);
        REQUIRE(runRanks(3, [&](int p) {
                    auto items = c.items(p);
                    const uint64_t before = comms[p]->stats().launches;
                    const int rc = comms[p]->groupMany(c.kind(), items.data(), k, FB_U8, 0, 0, 0, nullptr);
                    return rc == FB_OK && comms[p]->stats().launches - before == (k == 1016 ? 1u : 2u);
                }) == 0);
        for (int p = 0; p < 3; p++) {
            REQUIRE(c.matches(p));
        }
    }
    // 64 KiB of staging: 32 chunks, 10 per launch for 3 slots, so 12
    // blocks of 5000 bytes (3 chunks each) take 4 launches
    auto small = neighborGroup(3, (size_t)64 << 10);
    for (int p = 0; p < 3; p++) {
        g.set(*small[p], p);
    }
    for (bool a2a : { true, false }) {
        NeighborCase c(g, a2a, std::vector<size_t>(12, 5000), 2, rng);
        REQUIRE(c.launches((size_t)64 << 10) == (a2a ? 4u : 2u));
        REQUIRE(runRanks(3, [&](int p) {
                    auto items = c.items(p);
                    const uint64_t before = small[p]->stats().launches;
                    const int rc = small[p]->groupMany(c.kind(), items.data(), items.size(), FB_U8, 0, 0, 0, nullptr);
                    return rc == FB_OK && small[p]->stats().launches - before == c.launches((size_t)64 << 10);
                }) == 0);
        for (int p = 0; p < 3; p++) {
            REQUIRE(c.matches(p));
        }
    }
}

TEST_CASE("loopback group neighbor: a plan on a subset child", "[loopback]")
{
    std::mt19937 rng(11);
    const int n = 5;
    auto comms = neighborGroup(n);
    // members 4, 1, 3 of the parent: a directed ring in child ranks
    const std::vector<int> members = { 4, 1, 3 };
    const Graph g({ { 1 }, { 2 }, { 0 } }, { { 2 }, { 0 }, { 1 } });
    NeighborCase c(g, false, { 3000, 9 }, 7, rng);
    const int fails = runRanks(n, [&](int r) {
        auto it = std::find(members.begin(), members.end(), r);
        if (it == members.end()) {
            return true;
        }
        const int cr = (int)(it - members.begin());
        auto child = comms[r]->subset(members, 3);
        if (child == nullptr || child->setNeighbors(g.in[cr], 1, 1, 1) != FB_OK) {
            return false;
        }
        auto items = c.items(cr);
        int rc = FB_OK;
        auto plan = child->prepareGroup(items.data(), items.size(), FB_U8, &rc, c.kind());
        const bool ok = plan != nullptr && child->runGroup(c.kind(), *plan, 0, 0, 0, nullptr) == FB_OK &&
                        child->stats().launches == 1;
        plan.reset();
        child.reset();
        return ok && comms[r]->peekError() == 0 && !comms[r]->hasNeighbors();
    });
    REQUIRE(fails == 0);
    for (int p = 0; p < 3; p++) {
        REQUIRE(c.matches(p));
    }
}

TEST_CASE("loopback group neighbor: refusals", "[loopback]")
{
    std::mt19937 rng(9);
    auto comms = neighborGroup(2);
    const Graph g({ { 1 }, { 0, 1 } }, { { 1 }, { 0, 1 } });
    NeighborCase c(g, true, { 64, 100 }, 0, rng);
    auto items = c.items(0);
    const auto A2A = Communicator::GROUP_NEIGHBOR_ALLTOALL;
    const auto AG = Communicator::GROUP_NEIGHBOR_ALLGATHER;
    // no topology yet
    int rc = FB_OK;
    REQUIRE(comms[0]->prepareGroup(items.data(), items.size(), FB_U8, &rc, A2A) == nullptr);
    REQUIRE(rc == FB_E_INVALID);
    REQUIRE(comms[0]->groupMany(AG, items.data(), items.size(), FB_U8, 0, 0, 0, nullptr) == FB_E_INVALID);
    // bad topologies, then a good one, then a second one
    REQUIRE(comms[0]->setNeighbors({ { 2, 0 } }, 1, 2, 2) == FB_E_INVALID);  // source outside
    REQUIRE(comms[0]->setNeighbors({ { 1, 2 } }, 1, 2, 2) == FB_E_INVALID);  // index outside
    REQUIRE(comms[0]->setNeighbors({ { 1, 0 } }, 3, 2, 2) == FB_E_INVALID);  // out-degree above its maximum
    REQUIRE(comms[0]->setNeighbors({ { 1, 0 } }, 1, 2, 0) == FB_E_INVALID);  // in-degree above its maximum
    REQUIRE(!comms[0]->hasNeighbors());
    g.set(*comms[0], 0);
    REQUIRE(comms[0]->setNeighbors(g.in[0], 1, 2, 2) == FB_E_INVALID);
    auto plan = comms[0]->prepareGroup(items.data(), items.size(), FB_U8, &rc, A2A);
    REQUIRE(plan != nullptr);
    const uint64_t before = comms[0]->stats().launches;
    // nothing is launched: no peer is left at a barrier
    REQUIRE(comms[0]->runGroup(AG, *plan, 0, 0, 0, nullptr) == FB_E_INVALID);
    REQUIRE(comms[0]->runGroup(Communicator::GROUP_ALLTOALL, *plan, 0, 0, 0, nullptr) == FB_E_INVALID);
    REQUIRE(comms[0]->runGroup(A2A, *plan, 0, 0, FB_FLAG_CHANNEL(1), nullptr) == FB_E_INVALID);
    REQUIRE(comms[0]->groupMany(A2A, items.data(), items.size(), 99, 0, 0, 0, nullptr) == FB_E_INVALID);
    // rank 0 has an out-edge and an in-edge: it needs both buffers
    items[1].send = nullptr;
    REQUIRE(comms[0]->groupMany(A2A, items.data(), items.size(), FB_U8, 0, 0, 0, nullptr) == FB_E_INVALID);
    items = c.items(0);
    items[0].recv = nullptr;
    REQUIRE(comms[0]->groupMany(AG, items.data(), items.size(), FB_U8, 0, 0, 0, nullptr) == FB_E_INVALID);
    REQUIRE(comms[0]->stats().launches == before);
    // staging (64 KiB at least: 32 chunks) smaller than one chunk per slot
    // of the all-to-all: 40 edges from rank 0 to rank 1
    const Graph wide({ std::vector<int>(40, 1), {} }, { {}, std::vector<int>(40, 0) });
    auto tiny = neighborGroup(2, (size_t)64 << 10);
    wide.set(*tiny[0], 0);
    NeighborCase w(wide, true, { 8 }, 0, rng);
    auto witems = w.items(0);
    REQUIRE(tiny[0]->groupMany(A2A, witems.data(), 1, FB_U8, 0, 0, 0, nullptr) == FB_E_TOO_LARGE);
    REQUIRE(tiny[0]->stats().launches == 0);
    REQUIRE(std::string(Communicator::groupKindName(AG)) == "neighbor-allgather");
    REQUIRE(std::string(Communicator::groupKindName(A2A)) == "neighbor-alltoall");
}
