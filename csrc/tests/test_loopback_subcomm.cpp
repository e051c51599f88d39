// Communicator::subset on the loopback backend (no GPU): validation, the calls
// a child refuses, slot masks before and after release, child ranks and heap
// addressing, and the fused collectives over member subsets in child order.
#include "harness.h"

#include <faabric/device/communicator.h>

#include <atomic>
#include <cstring>
#include <functional>
#include <stdexcept>
#include <thread>

using faabric::device::CommConfig;
using faabric::device::Communicator;

namespace {
std::vector<std::shared_ptr<Communicator>> loopGroup(int n)
{
    CommConfig cfg;
    cfg.loopback = true;
    cfg.heapBytes = (size_t)8 << 20;
    cfg.stageBytes = (size_t)1 << 20;
    cfg.p2pBounceBytes = (size_t)1 << 20;
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

constexpr uint32_t ALL_SLOTS = (1u << FB_SUB_SLOTS) - 1;
}

TEST_CASE("loopback subset: validation errors", "[loopback]")
{
    auto comms = loopGroup(4);
    Communicator& c = *comms[1];
    int rc = FB_OK;
    REQUIRE(c.subset({}, 0, &rc) == nullptr);
    REQUIRE_EQ(rc, FB_E_INVALID);
    REQUIRE(c.subset({ 1, 4 }, 0, &rc) == nullptr); // out of range
    REQUIRE_EQ(rc, FB_E_INVALID);
    REQUIRE(c.subset({ -1, 1 }, 0, &rc) == nullptr);
    REQUIRE_EQ(rc, FB_E_INVALID);
    REQUIRE(c.subset({ 1, 2, 1 }, 0, &rc) == nullptr); // duplicated
    REQUIRE_EQ(rc, FB_E_INVALID);
    REQUIRE(c.subset({ 0, 2 }, 0, &rc) == nullptr); // this rank not a member
    REQUIRE_EQ(rc, FB_E_INVALID);
    REQUIRE(c.subset({ 0, 1 }, -1, &rc) == nullptr);
    REQUIRE_EQ(rc, FB_E_INVALID);
    REQUIRE(c.subset({ 0, 1 }, FB_SUB_SLOTS, &rc) == nullptr);
    REQUIRE_EQ(rc, FB_E_INVALID);
    // no failed call took a slot
    REQUIRE_EQ(c.freeSubsetSlots(), ALL_SLOTS);
    auto child = c.subset({ 0, 1 }, 3, &rc);
    REQUIRE(child != nullptr);
    REQUIRE_EQ(rc, FB_OK);
    REQUIRE(c.subset({ 1, 3 }, 3, &rc) == nullptr); // slot in use on this rank
    REQUIRE_EQ(rc, FB_E_INVALID);
    // a child cannot be split further
    REQUIRE(child->subset({ 0 }, 4, &rc) == nullptr);
    REQUIRE_EQ(rc, FB_E_UNSUPPORTED);
    REQUIRE_EQ(child->freeSubsetSlots(), 0u);
}

TEST_CASE("loopback subset: slot masks before and after release", "[loopback]")
{
    auto comms = loopGroup(3);
    REQUIRE_EQ(comms[0]->freeSubsetSlots(), ALL_SLOTS);
    std::vector<std::shared_ptr<Communicator>> held;
    for (int s = 0; s < FB_SUB_SLOTS; s++) {
        held.push_back(comms[0]->subset({ 0, 2 }, s));
        REQUIRE(held.back() != nullptr);
        REQUIRE_EQ(comms[0]->freeSubsetSlots(), ALL_SLOTS & ~((2u << s) - 1));
    }
    REQUIRE_EQ(comms[0]->freeSubsetSlots(), 0u);
    // other ranks are untouched: slots are per rank
    REQUIRE_EQ(comms[2]->freeSubsetSlots(), ALL_SLOTS);
    held[6].reset();
    REQUIRE_EQ(comms[0]->freeSubsetSlots(), 1u << 6);
    held.clear();
    REQUIRE_EQ(comms[0]->freeSubsetSlots(), ALL_SLOTS);
}

TEST_CASE("loopback subset: child ranks, sizes, heap addressing and refused calls", "[loopback]")
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
    Communicator::GroupItem item{ buf, buf, 4 };
    int rc = FB_OK;
    REQUIRE(child->prepareGroup(&item, 1, FB_I32, &rc) == nullptr);
    REQUIRE_EQ(rc, FB_E_UNSUPPORTED);
    REQUIRE_EQ(child->allReduceMany(&item, 1, FB_I32, FB_OP_SUM, FB_FLAG_SYMMETRIC, nullptr), FB_E_UNSUPPORTED);
    auto plan = comms[2]->prepareGroup(&item, 1, FB_I32, &rc);
    REQUIRE(plan != nullptr);
    REQUIRE_EQ(child->allReduceGroup(*plan, FB_OP_SUM, FB_FLAG_SYMMETRIC, nullptr), FB_E_UNSUPPORTED);
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
    // nothing was launched by the refused calls
    REQUIRE_EQ(child->stats().launches, 0u);
}

TEST_CASE("loopback subset: fused collectives over members in child order", "[loopback]")
{
    auto comms = loopGroup(8);
    const size_t N = 3000; // not a vector multiple
    const uint64_t inOff = comms[0]->alloc(N * 4 * 8);
    const uint64_t outOff = comms[0]->alloc(N * 4 * 8);
    for (int r = 1; r < 8; r++) {
        comms[r]->alloc(N * 4 * 8);
        comms[r]->alloc(N * 4 * 8);
    }
    for (const std::vector<int>& members : std::vector<std::vector<int>>{ { 5, 2, 7, 0 }, { 1, 3, 5, 7 }, { 6 }, { 7, 6, 5, 4, 3, 2, 1, 0 } }) {
        const int n = (int)members.size();
        std::vector<std::shared_ptr<Communicator>> kids(n);
        for (int i = 0; i < n; i++) {
            kids[i] = comms[members[i]]->subset(members, 2);
            REQUIRE(kids[i] != nullptr);
        }
        const uint64_t parentLaunches = comms[members[0]]->stats().launches;
        int fails = runThreads(n, [&](int i) {
            Communicator& c = *kids[i];
            const int w = members[i];
            int32_t* in = (int32_t*)c.heapPtr(inOff);
            int32_t* out = (int32_t*)c.heapPtr(outOff);
            std::vector<int32_t> local(N * n, -1);
            bool ok = true;
            for (size_t k = 0; k < N; k++) {
                in[k] = (int32_t)(k % 97) + 1000 * w;
            }
            ok = c.barrier(nullptr) == FB_OK;
            // all-reduce (one-shot and two-shot), symmetric and staged output
            for (int algo : { FB_ALGO_AUTO, FB_ALGO_ONESHOT, FB_ALGO_TWOSHOT }) {
                ok = ok && c.allReduce(in, local.data(), N, FB_I32, FB_OP_SUM, algo, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
                int32_t sumW = 0;
                for (int m : members) {
                    sumW += 1000 * m;
                }
                for (size_t k = 0; k < N && ok; k++) {
                    ok = local[k] == (int32_t)(k % 97) * n + sumW;
                }
            }
            // scan: prefixes in child order
            ok = ok && c.scan(in, out, N, FB_I32, FB_OP_SUM, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            int32_t pre = 0;
            for (int j = 0; j <= i; j++) {
                pre += 1000 * members[j];
            }
            for (size_t k = 0; k < N && ok; k++) {
                ok = out[k] == (int32_t)(k % 97) * (i + 1) + pre;
            }
            // reduce to child rank n-1
            ok = ok && c.reduce(in, local.data(), N, FB_I32, FB_OP_MAX, n - 1, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            if (i == n - 1) {
                int maxW = 0;
                for (int m : members) {
                    maxW = std::max(maxW, m);
                }
                for (size_t k = 0; k < N && ok; k++) {
                    ok = local[k] == (int32_t)(k % 97) + 1000 * maxW;
                }
            }
            // all-gather from a local source: chunks in child order
            std::vector<int32_t> mine(N, 7 * w + 1);
            ok = ok && c.allGather(mine.data(), local.data(), N * 4, 0, nullptr) == FB_OK;
            for (int j = 0; j < n && ok; j++) {
                ok = local[(size_t)j * N] == 7 * members[j] + 1 && local[(size_t)j * N + N - 1] == 7 * members[j] + 1;
            }
            // broadcast from child rank 0 (symmetric)
            if (i == 0) {
                for (size_t k = 0; k < N; k++) {
                    out[k] = (int32_t)k * 3 + w;
                }
            }
            ok = ok && c.barrier(nullptr) == FB_OK;
            ok = ok && c.broadcast(out, N * 4, 0, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            for (size_t k = 0; k < N && ok; k++) {
                ok = out[k] == (int32_t)k * 3 + members[0];
            }
            ok = ok && c.barrier(nullptr) == FB_OK && c.checkError(nullptr) == 0;
            return ok;
        });
        if (fails != 0) {
            fbtest::fail(__FILE__, __LINE__, "members of size " + std::to_string(n) + ": " + std::to_string(fails) + " ranks failed");
        }
        // the child counts its own launches, never LL or NVLS; the parent's do not move
        REQUIRE(kids[0]->stats().launches > 0);
        REQUIRE_EQ(kids[0]->stats().algoCount[FB_ALGO_LL], 0u);
        REQUIRE_EQ(kids[0]->stats().algoCount[FB_ALGO_NVLS], 0u);
        REQUIRE_EQ(comms[members[0]]->stats().launches, parentLaunches);
        kids.clear();
        for (int m : members) {
            REQUIRE_EQ(comms[m]->freeSubsetSlots(), ALL_SLOTS);
            // released pads are zero again
            const uint32_t* pad = comms[m]->devStruct().sig[m] + 3 * FB_SIG_TOTAL_WORDS;
            bool zero = true;
            for (int k = 0; k < FB_SIG_TOTAL_WORDS; k++) {
                zero = zero && pad[k] == 0;
            }
            REQUIRE(zero);
        }
    }
}
