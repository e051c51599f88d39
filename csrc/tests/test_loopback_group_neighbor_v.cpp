// Grouped neighbourhood v-collectives (Communicator::groupMany / prepareGroup
// with NeighborVItem, GROUP_NEIGHBOR_ALLGATHERV and GROUP_NEIGHBOR_ALLTOALLV)
// on the loopback backend (no GPU): every byte of every rank's buffers, guard
// bytes included, against an exchange computed on the host over seeded
// random graphs with self-edges, multi-edges and ranks of degree 0, random
// per-edge counts (zero included) and displacements at any byte offset, at
// 1-8 ranks; a small staging buffer, so large edges take several rounds, with
// the launches the agreement gives on every rank; and the refusals.
#include "harness.h"

#include <faabric/device/communicator.h>

#include <algorithm>
#include <atomic>
#include <functional>
#include <random>
#include <thread>

using faabric::device::CommConfig;
using faabric::device::Communicator;

namespace {
const size_t VSTAGE = (size_t)64 << 10; // the smallest staging buffer
const uint64_t VCB = 2048; // FB_NEIGHBOR_CHUNK
const size_t VGUARD = 8;

std::vector<std::shared_ptr<Communicator>> vGroup(int n)
{
    CommConfig cfg;
    cfg.loopback = true;
    cfg.heapBytes = (size_t)4 << 20;
    cfg.stageBytes = VSTAGE;
    cfg.p2pBounceBytes = (size_t)1 << 20;
    cfg.channels = 2;
    cfg.maxBlocks = 4;
    cfg.timeoutMs = 5000;
    return Communicator::createLocal(n, std::vector<int>(n, 0), cfg);
}

int vRunRanks(int n, const std::function<bool(int)>& fn)
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

// A random graph: every third rank sends nothing; in-edge j of rank d is the
// k-th occurrence of its source, paired with the k-th occurrence of d in the
// source's destinations
struct VGraph
{
    int n = 0;
    std::vector<std::vector<int>> dst;
    std::vector<std::vector<std::pair<int, int>>> in;
    int maxOut = 0, maxIn = 0;

    VGraph(int nIn, std::mt19937& rng)
      : n(nIn)
      , dst(nIn)
      , in(nIn)
    {
        std::vector<std::vector<int>> src(n);
        for (int r = 0; r < n; r++) {
            const int deg = (r + (int)(rng() % 3)) % 3 == 0 ? 0 : 1 + (int)(rng() % 3);
            for (int k = 0; k < deg; k++) {
                const int t = (int)(rng() % n);
                dst[r].push_back(t);
                src[t].push_back(r);
            }
        }
        for (int r = 0; r < n; r++) {
            std::shuffle(src[r].begin(), src[r].end(), rng);
            std::vector<int> seen(n, 0);
            for (int s : src[r]) {
                int k = seen[s]++;
                for (size_t i = 0; i < dst[s].size(); i++) {
                    if (dst[s][i] == r && k-- == 0) {
                        in[r].push_back({ s, (int)i });
                        break;
                    }
                }
            }
            maxOut = std::max(maxOut, (int)dst[r].size());
            maxIn = std::max(maxIn, (int)in[r].size());
        }
    }
};

// One list of `items` calls: per rank a byte buffer with every item's send
// and recv region (guards around, blocks in shuffled order with gaps)
struct VCase
{
    const VGraph& g;
    bool a2a;
    int items;
    // count[i][s][k]: bytes of item i on out-edge k of rank s (all-gather: k = 0)
    std::vector<std::vector<std::vector<size_t>>> count;
    std::vector<std::vector<uint8_t>> buf, want;
    std::vector<std::vector<size_t>> sendOff, recvOff;
    std::vector<std::vector<std::vector<size_t>>> sc, sd, rc, rd;

    VCase(const VGraph& gIn, bool a2aIn, int itemsIn, std::mt19937& rng, const std::function<size_t(int, int, int)>& cnt)
      : g(gIn)
      , a2a(a2aIn)
      , items(itemsIn)
    {
        const int n = g.n;
        count.assign(items, std::vector<std::vector<size_t>>(n));
        for (int i = 0; i < items; i++) {
            for (int s = 0; s < n; s++) {
                const int blocks = a2a ? (int)g.dst[s].size() : 1;
                for (int k = 0; k < blocks; k++) {
                    count[i][s].push_back(cnt(i, s, k));
                }
            }
        }
        buf.resize(n);
        sendOff.resize(n);
        recvOff.resize(n);
        sc.resize(n);
        sd.resize(n);
        rc.resize(n);
        rd.resize(n);
        for (int r = 0; r < n; r++) {
            size_t pos = VGUARD + rng() % 5;
            auto lay = [&](const std::vector<size_t>& counts, std::vector<size_t>& displs) {
                displs.assign(counts.size(), 0);
                std::vector<size_t> order(counts.size());
                for (size_t k = 0; k < order.size(); k++) {
                    order[k] = k;
                }
                std::shuffle(order.begin(), order.end(), rng);
                size_t p = 0;
                for (size_t k : order) {
                    p += rng() % 3;
                    displs[k] = p;
                    p += counts[k];
                }
                return p;
            };
            for (int i = 0; i < items; i++) {
                sc[r].push_back(count[i][r]);
                sd[r].emplace_back();
                sendOff[r].push_back(pos);
                pos += lay(sc[r][i], sd[r][i]) + VGUARD;
                rc[r].emplace_back();
                for (auto [s, idx] : g.in[r]) {
                    rc[r][i].push_back(count[i][s][a2a ? idx : 0]);
                }
                rd[r].emplace_back();
                recvOff[r].push_back(pos);
                pos += lay(rc[r][i], rd[r][i]) + VGUARD;
            }
            buf[r].resize(pos + VGUARD);
            for (auto& b : buf[r]) {
                b = (uint8_t)rng();
            }
        }
        want = buf;
        for (int d = 0; d < n; d++) {
            for (int i = 0; i < items; i++) {
                for (size_t j = 0; j < g.in[d].size(); j++) {
                    const auto [s, idx] = g.in[d][j];
                    const size_t k = a2a ? (size_t)idx : 0;
                    const uint8_t* from = buf[s].data() + sendOff[s][i] + sd[s][i][k];
                    std::copy(from, from + rc[d][i][j], want[d].begin() + recvOff[d][i] + rd[d][i][j]);
                }
            }
        }
    }

    Communicator::GroupKind kind() const
    {
        return a2a ? Communicator::GROUP_NEIGHBOR_ALLTOALLV : Communicator::GROUP_NEIGHBOR_ALLGATHERV;
    }

    std::vector<Communicator::NeighborVItem> list(int r)
    {
        std::vector<Communicator::NeighborVItem> out;
        for (int i = 0; i < items; i++) {
            uint8_t* base = buf[r].data();
            // (the all-gather's send is its one block)
            out.push_back({ base + sendOff[r][i] + (a2a ? 0 : sd[r][i][0]), base + recvOff[r][i], sc[r][i].data(),
                            sd[r][i].data(), rc[r][i].data(), rd[r][i].data() });
        }
        return out;
    }

    // Launches of the agreed windows: a slot of VSTAGE (over the largest
    // out-degree) in whole chunks, at most a window's stream rounded up
    uint64_t launches(const std::vector<uint64_t>& agreed) const
    {
        const uint64_t slots = a2a ? std::max(g.maxOut, 1) : 1;
        const uint64_t room = VSTAGE / VCB / slots * VCB;
        uint64_t total = 0;
        for (uint64_t m : agreed) {
            if (m > 0) {
                const uint64_t w = std::min(room, (m + VCB - 1) / VCB * VCB);
                total += (m + w - 1) / w;
            }
        }
        return total;
    }
};

// Agree (elementwise maximum over the ranks), then run the list on every
// rank (`many`, or a plan): true if every byte and every launch count match
bool runV(std::vector<std::shared_ptr<Communicator>>& comms, VCase& c, bool many, std::vector<uint64_t>* mineOut)
{
    const int n = c.g.n;
    std::vector<std::vector<Communicator::NeighborVItem>> lists(n);
    std::vector<uint64_t> agreed;
    for (int r = 0; r < n; r++) {
        lists[r] = c.list(r);
        std::vector<uint64_t> mine;
        REQUIRE(comms[r]->neighborVStreams(c.kind(), lists[r].data(), lists[r].size(), FB_U8, mine) == FB_OK);
        if (r == 0) {
            agreed = mine;
        }
        REQUIRE(mine.size() == agreed.size());
        for (size_t w = 0; w < mine.size(); w++) {
            agreed[w] = std::max(agreed[w], mine[w]);
        }
        if (mineOut != nullptr) {
            mineOut->push_back(mine.empty() ? 0 : *std::max_element(mine.begin(), mine.end()));
        }
    }
    const uint64_t want = c.launches(agreed);
    std::vector<uint64_t> got(n, 0);
    const int failures = vRunRanks(n, [&](int r) {
        Communicator& comm = *comms[r];
        const uint64_t before = comm.stats().launches;
        int rc = FB_OK;
        if (many) {
            rc = comm.groupMany(c.kind(), lists[r].data(), lists[r].size(), FB_U8, agreed, 0, nullptr);
        } else {
            auto plan = comm.prepareGroup(lists[r].data(), lists[r].size(), FB_U8, agreed, &rc, c.kind());
            if (plan == nullptr || Communicator::groupPlanLaunches(*plan) != want) {
                return false;
            }
            rc = comm.runGroup(c.kind(), *plan, 0, 0, 0, nullptr);
        }
        got[r] = comm.stats().launches - before;
        return rc == FB_OK;
    });
    REQUIRE(failures == 0);
    for (int r = 0; r < n; r++) {
        REQUIRE(got[r] == want);
        REQUIRE(c.buf[r] == c.want[r]);
    }
    return true;
}
} // namespace

TEST_CASE("loopback group neighbor v: every byte over random graphs at 1-8 ranks, plans and many", "[loopback]")
{
    for (int n : { 1, 2, 3, 4, 8 }) {
        for (bool a2a : { false, true }) {
            std::mt19937 rng(100 * n + (a2a ? 1 : 0));
            for (int graph = 0; graph < 2; graph++) {
                auto comms = vGroup(n);
                VGraph g(n, rng);
                for (int r = 0; r < n; r++) {
                    REQUIRE(comms[r]->setNeighbors(g.in[r], (int)g.dst[r].size(), g.maxOut, g.maxIn) == FB_OK);
                }
                const size_t sizes[] = { 0, 0, 1, 7, 2047, 2049, 9001, VSTAGE + 5 };
                const int quiet = (int)(rng() % n); // sends nothing
                for (bool many : { false, true }) {
                    VCase c(g, a2a, 4, rng, [&](int, int s, int) { return s == quiet ? 0 : sizes[rng() % 8]; });
                    REQUIRE(runV(comms, c, many, nullptr));
                }
            }
        }
    }
}

TEST_CASE("loopback group neighbor v: one large edge sets every rank's rounds; many items take several windows",
          "[loopback]")
{
    std::mt19937 rng(7);
    for (bool a2a : { false, true }) {
        auto comms = vGroup(4);
        VGraph g(4, rng);
        while (g.maxIn == 0) {
            g = VGraph(4, rng);
        }
        for (int r = 0; r < 4; r++) {
            REQUIRE(comms[r]->setNeighbors(g.in[r], (int)g.dst[r].size(), g.maxOut, g.maxIn) == FB_OK);
        }
        int big = 0;
        while (g.dst[big].empty()) {
            big++;
        }
        VCase c(g, a2a, 3, rng, [&](int i, int s, int k) { return s == big && k == 0 && i == 1 ? 5 * VSTAGE + 3 : 11; });
        std::vector<uint64_t> mine;
        REQUIRE(runV(comms, c, true, &mine));
        // the ranks' own streams differ: some would launch once alone
        REQUIRE(*std::min_element(mine.begin(), mine.end()) < *std::max_element(mine.begin(), mine.end()));
        VCase many(g, a2a, 700, rng, [&](int, int, int) { return (size_t)(rng() % 30); });
        REQUIRE(runV(comms, many, false, nullptr));
        REQUIRE(runV(comms, many, true, nullptr));
    }
}

TEST_CASE("loopback group neighbor v: refusals before any launch", "[loopback]")
{
    auto comms = vGroup(2);
    uint8_t a[64] = {}, b[64] = {};
    size_t eight = 8, zero = 0;
    Communicator::NeighborVItem it{ a, b, &eight, &zero, &eight, &zero };
    std::vector<uint64_t> out;
    const auto A2AV = Communicator::GROUP_NEIGHBOR_ALLTOALLV;
    // no topology
    REQUIRE(comms[0]->neighborVStreams(A2AV, &it, 1, FB_U8, out) == FB_E_INVALID);
    REQUIRE(comms[0]->setNeighbors({ { 1, 0 } }, 1, 1, 1) == FB_OK);
    REQUIRE(comms[0]->neighborVStreams(A2AV, &it, 1, FB_U8, out) == FB_OK);
    REQUIRE(out == std::vector<uint64_t>{ 8 });
    const uint64_t before = comms[0]->stats().launches;
    // an agreement below this rank's own stream, or of the wrong length
    REQUIRE(comms[0]->groupMany(A2AV, &it, 1, FB_U8, { 7 }, 0, nullptr) == FB_E_INVALID);
    REQUIRE(comms[0]->groupMany(A2AV, &it, 1, FB_U8, { 8, 8 }, 0, nullptr) == FB_E_INVALID);
    int rc = FB_OK;
    REQUIRE(comms[0]->prepareGroup(&it, 1, FB_U8, { 7 }, &rc, A2AV) == nullptr);
    REQUIRE(rc == FB_E_INVALID);
    // a missing buffer with a count, missing counts, a GroupItem kind
    Communicator::NeighborVItem noSend{ nullptr, b, &eight, &zero, &eight, &zero };
    REQUIRE(comms[0]->groupMany(A2AV, &noSend, 1, FB_U8, { 8 }, 0, nullptr) == FB_E_INVALID);
    Communicator::NeighborVItem noCounts{ a, b, nullptr, nullptr, &eight, &zero };
    REQUIRE(comms[0]->groupMany(A2AV, &noCounts, 1, FB_U8, { 8 }, 0, nullptr) == FB_E_INVALID);
    REQUIRE(comms[0]->groupMany(Communicator::GROUP_NEIGHBOR_ALLTOALL, &it, 1, FB_U8, { 8 }, 0, nullptr) ==
            FB_E_INVALID);
    // a channel other than 0
    REQUIRE(comms[0]->groupMany(A2AV, &it, 1, FB_U8, { 8 }, FB_FLAG_CHANNEL(1), nullptr) == FB_E_INVALID);
    REQUIRE(comms[0]->stats().launches == before);
    // degrees above FB_NEIGHBOR_V_MAX_DEGREE
    REQUIRE(comms[1]->setNeighbors({ { 0, 0 } }, 1, 200, 100) == FB_OK);
    REQUIRE(comms[1]->neighborVStreams(A2AV, &it, 1, FB_U8, out) == FB_E_TOO_LARGE);
}
