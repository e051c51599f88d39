// Batched one-sided atomics (Communicator::accumulateMany) on the loopback
// backend: the argument checks of the GPU path, the launch-count rule, and
// list order for items whose targets intersect.  The host twin applies the
// table in table order, so chains and launches decide the results here as on
// the GPU.
#include "harness.h"

#include <faabric/device/communicator.h>

#include <atomic>
#include <cstring>
#include <functional>
#include <thread>
#include <vector>

#include "launch_api.h"

using faabric::device::CommConfig;
using faabric::device::Communicator;
using Item = Communicator::RmaAccumulate;

namespace {
struct AccGroup
{
    std::vector<std::shared_ptr<Communicator>> comms;
    std::vector<uint64_t> win; // symmetric offset, one per rank (all equal)

    explicit AccGroup(int n)
    {
        CommConfig cfg;
        cfg.loopback = true;
        cfg.heapBytes = (size_t)8 << 20;
        cfg.stageBytes = (size_t)1 << 20;
        cfg.p2pBounceBytes = (size_t)1 << 20;
        cfg.timeoutMs = 5000;
        comms = Communicator::createLocal(n, std::vector<int>(n, 0), cfg);
        for (auto& c : comms) {
            win.push_back(c->alloc(1 << 20));
            memset(c->heapPtr(win.back()), 0, 1 << 20);
        }
    }

    uint8_t* at(int rank, size_t byteOff) { return comms[rank]->heapPtr(win[rank] + byteOff); }
    uint64_t launches(int rank) { return comms[rank]->stats().launches; }

    int run(const std::function<bool(int, Communicator&)>& fn)
    {
        std::atomic<int> failures{ 0 };
        std::vector<std::thread> ts;
        for (int r = 0; r < (int)comms.size(); r++) {
            ts.emplace_back([&, r] {
                if (!fn(r, *comms[r])) {
                    failures++;
                }
            });
        }
        for (auto& t : ts) {
            t.join();
        }
        return failures.load();
    }
};

template<typename T>
T load(const uint8_t* p)
{
    T v;
    memcpy(&v, p, sizeof(T));
    return v;
}
}

TEST_CASE("rma many: 1024 fetching increments of one counter are one launch, tickets in list order", "[loopback][rma]")
{
    AccGroup g(2);
    Communicator& c = *g.comms[0];
    const int k = 1024;
    const int64_t one = 1;
    std::vector<int64_t> tickets(k, -1);
    std::vector<Item> items;
    for (int i = 0; i < k; i++) {
        items.push_back(Item{ &one, &tickets[i], g.win[0] + 64, 1, 1 });
    }
    const uint64_t before = g.launches(0);
    REQUIRE_EQ(c.accumulateMany(items.data(), items.size(), FB_I64, FB_OP_SUM, nullptr), FB_OK);
    REQUIRE_EQ(g.launches(0), before + 1);
    REQUIRE_EQ(load<int64_t>(g.at(1, 64)), (int64_t)k);
    for (int i = 0; i < k; i++) {
        REQUIRE_EQ(tickets[i], (int64_t)i);
    }
}

TEST_CASE("rma many: overlapping items apply in list order", "[loopback][rma]")
{
    AccGroup g(2);
    Communicator& c = *g.comms[0];
    // f32: 0 + 1e8 + 1 - 1e8 is 0 in this order (1 is below half an ulp of
    // 1e8) and 1 if the last two swap
    const float f[3] = { 1e8f, 1.0f, -1e8f };
    std::vector<Item> items;
    for (int i = 0; i < 3; i++) {
        items.push_back(Item{ &f[i], nullptr, g.win[0], 1, 1 });
    }
    REQUIRE_EQ(c.accumulateMany(items.data(), items.size(), FB_F32, FB_OP_SUM, nullptr), FB_OK);
    REQUIRE_EQ(load<float>(g.at(1, 0)), 0.0f);
    // REPLACE: the last of three overlapping ranges wins where it covers
    const int32_t a[4] = { 1, 1, 1, 1 };
    const int32_t b[2] = { 2, 2 };
    const int32_t d[1] = { 3 };
    int32_t prev[4] = { -1, -1, -1, -1 };
    items = { Item{ a, nullptr, g.win[0] + 16, 4, 1 }, Item{ b, nullptr, g.win[0] + 20, 2, 1 },
              Item{ d, prev, g.win[0] + 24, 1, 1 } };
    const uint64_t before = g.launches(0);
    REQUIRE_EQ(c.accumulateMany(items.data(), items.size(), FB_I32, FB_OP_REPLACE, nullptr), FB_OK);
    REQUIRE_EQ(g.launches(0), before + 1);
    const int32_t want[4] = { 1, 2, 3, 1 };
    REQUIRE(memcmp(g.at(1, 16), want, 16) == 0);
    REQUIRE_EQ(prev[0], 2); // fetched after the second item
}

TEST_CASE("rma many: the launch count follows the documented rule", "[loopback][rma]")
{
    AccGroup g(2);
    Communicator& c = *g.comms[0];
    std::vector<int64_t> ones(4096, 1);
    auto launchesFor = [&](const std::vector<Item>& items) {
        const uint64_t before = g.launches(0);
        REQUIRE_EQ(c.accumulateMany(items.data(), items.size(), FB_I64, FB_OP_SUM, nullptr), FB_OK);
        return g.launches(0) - before;
    };
    // disjoint items: one launch per 1024 descriptors; zero-count items take no room
    std::vector<Item> items;
    for (int i = 0; i < 2051; i++) {
        items.push_back(Item{ ones.data(), nullptr, g.win[0] + 8 * (uint64_t)i, (size_t)(i == 7 ? 0 : 1), i % 2 });
    }
    REQUIRE_EQ(launchesFor(items), 3u); // 2050 non-empty items
    // the same offset on two peers does not overlap
    items = { Item{ ones.data(), nullptr, g.win[0], 1, 0 }, Item{ ones.data(), nullptr, g.win[0], 1, 1 } };
    REQUIRE_EQ(launchesFor(items), 1u);
    // a chain reaches FB_RMA_ACC_CHAIN_BYTES (two 8 KiB items), a third
    // overlapping 8 KiB item starts the next launch
    const size_t half = FB_RMA_ACC_CHAIN_BYTES / 16;
    items.assign(3, Item{ ones.data(), nullptr, g.win[0] + 65536, half, 1 });
    REQUIRE_EQ(launchesFor(items), 2u);
    // an item that overlaps two chains starts the next launch
    items = { Item{ ones.data(), nullptr, g.win[0] + 131072, 1, 1 }, Item{ ones.data(), nullptr, g.win[0] + 131088, 1, 1 },
              Item{ ones.data(), nullptr, g.win[0] + 131072, 3, 1 } };
    REQUIRE_EQ(launchesFor(items), 2u);
    // a large single item is no chain: any length in one launch
    items = { Item{ ones.data(), nullptr, g.win[0] + 262144, 4096, 1 }, Item{ ones.data(), nullptr, g.win[0], 1, 1 } };
    REQUIRE_EQ(launchesFor(items), 1u);
    REQUIRE_EQ(launchesFor({}), 0u);
    const int64_t* t = (const int64_t*)g.at(1, 0);
    REQUIRE_EQ(t[0], 2); // the second list and the last one (item 0 of the first goes to peer 0)
    REQUIRE_EQ(t[65536 / 8], 3);
    REQUIRE_EQ(t[65536 / 8 + half - 1], 3);
    REQUIRE_EQ(t[131072 / 8], 2);
    REQUIRE_EQ(t[131072 / 8 + 1], 1);
    REQUIRE_EQ(t[131072 / 8 + 2], 2);
    REQUIRE_EQ(t[262144 / 8 + 4095], 1);
}

TEST_CASE("rma many: concurrent lists of every rank give exact counters", "[loopback][rma]")
{
    const int n = 4;
    AccGroup g(n);
    const int k = 300;
    int fails = g.run([&](int rank, Communicator& c) {
        std::vector<int32_t> add(k);
        std::vector<Item> items;
        for (int i = 0; i < k; i++) {
            add[i] = rank + 1;
            // eight int32 counters on every rank
            items.push_back(Item{ &add[i], nullptr, g.win[rank] + 4 * (uint64_t)(i % 8), 1, i % n });
        }
        return c.accumulateMany(items.data(), items.size(), FB_I32, FB_OP_SUM, nullptr) == FB_OK;
    });
    REQUIRE_EQ(fails, 0);
    for (int t = 0; t < n; t++) {
        for (int j = 0; j < 8; j++) {
            int64_t want = 0;
            for (int r = 0; r < n; r++) {
                for (int i = 0; i < k; i++) {
                    want += (i % n == t && i % 8 == j) ? r + 1 : 0;
                }
            }
            REQUIRE_EQ((int64_t)load<int32_t>(g.at(t, 4 * j)), want);
        }
    }
}

TEST_CASE("rma many: refusals come before any launch and leave the targets unchanged", "[loopback][rma]")
{
    AccGroup g(2);
    Communicator& c = *g.comms[0];
    int64_t buf[4] = { 1, 2, 3, 4 };
    int64_t out[4] = { 0 };
    const uint64_t w = g.win[0];
    const Item good{ buf, nullptr, w, 2, 1 };
    auto refuse = [&](Item bad, int dtype, int op) {
        const Item items[3] = { good, good, bad };
        return c.accumulateMany(items, 3, dtype, op, nullptr);
    };
    const uint64_t before = g.launches(0);
    REQUIRE_EQ(refuse(Item{ buf, nullptr, w, 1, 2 }, FB_I64, FB_OP_SUM), FB_E_INVALID);  // peer
    REQUIRE_EQ(refuse(Item{ buf, nullptr, w, 0, -1 }, FB_I64, FB_OP_SUM), FB_E_INVALID); // peer of an empty item
    REQUIRE_EQ(refuse(Item{ buf, nullptr, 0, 1, 1 }, FB_I64, FB_OP_SUM), FB_E_INVALID);  // below the user heap
    REQUIRE_EQ(refuse(Item{ buf, nullptr, (uint64_t)1 << 40, 1, 1 }, FB_I64, FB_OP_SUM), FB_E_INVALID);
    REQUIRE_EQ(refuse(Item{ buf, nullptr, w, (size_t)1 << 40, 1 }, FB_I64, FB_OP_SUM), FB_E_INVALID);
    REQUIRE_EQ(refuse(Item{ buf, nullptr, w + 4, 1, 1 }, FB_I64, FB_OP_SUM), FB_E_INVALID);   // misaligned
    REQUIRE_EQ(refuse(Item{ nullptr, nullptr, w, 1, 1 }, FB_I64, FB_OP_SUM), FB_E_INVALID); // null origin
    REQUIRE_EQ(refuse(Item{ buf, out, w, 1, 1 }, FB_I64, FB_OP_NO_OP), FB_E_INVALID);       // good items lack fetch
    REQUIRE_EQ(refuse(good, FB_F64, FB_OP_BAND), FB_E_UNSUPPORTED);
    REQUIRE_EQ(refuse(good, FB_I64, FB_OP_MAXLOC), FB_E_UNSUPPORTED);
    REQUIRE_EQ(refuse(good, FB_DTYPE_COUNT, FB_OP_SUM), FB_E_INVALID);
    REQUIRE_EQ(c.accumulateMany(nullptr, 1, FB_I64, FB_OP_SUM, nullptr), FB_E_INVALID);
    REQUIRE_EQ(g.launches(0), before);
    for (int i = 0; i < 4; i++) {
        REQUIRE_EQ(load<int64_t>(g.at(1, 8 * i)), (int64_t)0);
    }
    // NO_OP with a fetch on every item, and empty items, are fine
    const Item reads[2] = { Item{ nullptr, out, w, 2, 1 }, Item{ nullptr, nullptr, w, 0, 1 } };
    REQUIRE_EQ(c.accumulateMany(reads, 2, FB_I64, FB_OP_NO_OP, nullptr), FB_OK);
    REQUIRE_EQ(g.launches(0), before + 1);
    auto sub = c.subset({ 0, 1 }, 0);
    REQUIRE(sub != nullptr);
    REQUIRE_EQ(sub->accumulateMany(&good, 1, FB_I64, FB_OP_SUM, nullptr), FB_E_UNSUPPORTED);
    REQUIRE_EQ(g.launches(0), before + 1);
}
