// One-sided atomics (Communicator::accumulate / compareAndSwap) on the
// loopback backend: the same argument checks as on the GPU, and host twins of
// the kernels that are atomic across rank threads.  Several threads updating
// one location must end exact, like several GPUs do.
#include "harness.h"

#include <faabric/device/communicator.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <functional>
#include <thread>
#include <vector>

using faabric::device::CommConfig;
using faabric::device::Communicator;

namespace {
struct RmaGroup
{
    std::vector<std::shared_ptr<Communicator>> comms;
    std::vector<uint64_t> win; // symmetric offset, one per rank (all equal)

    explicit RmaGroup(int n)
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
}

TEST_CASE("rma: fetch-and-add tickets are unique and sub-word neighbours stay exact", "[loopback][rma]")
{
    const int n = 4;
    const int k = 25;
    RmaGroup g(n);
    // byte 0..7: i64 ticket counter; bytes 8..11: four i8 counters in one word,
    // byte 9 a ticket counter, the others bumped by the other ranks
    std::vector<std::vector<int64_t>> tickets(n);
    std::vector<std::vector<int8_t>> tickets8(n);
    int fails = g.run([&](int rank, Communicator& c) {
        bool ok = true;
        const int64_t one = 1;
        const int8_t one8 = 1;
        for (int i = 0; i < k && ok; i++) {
            int64_t t = -1;
            int8_t t8 = -1;
            ok = c.accumulate(&one, g.win[rank], 1, FB_I64, FB_OP_SUM, 0, &t, nullptr) == FB_OK;
            ok = ok && c.accumulate(&one8, g.win[rank] + 9, 1, FB_I8, FB_OP_SUM, 0, &t8, nullptr) == FB_OK;
            const uint64_t nb = g.win[rank] + 8 + (rank % 2 == 0 ? 0 : 2) + (i % 2 == 0 ? 0 : 1) * (rank % 2 == 0 ? 3 : 1);
            ok = ok && c.accumulate(&one8, nb, 1, FB_I8, FB_OP_SUM, 0, nullptr, nullptr) == FB_OK;
            tickets[rank].push_back(t);
            tickets8[rank].push_back(t8);
        }
        return ok;
    });
    REQUIRE_EQ(fails, 0);
    int64_t counter;
    memcpy(&counter, g.at(0, 0), 8);
    REQUIRE_EQ(counter, (int64_t)n * k);
    std::vector<int64_t> all;
    std::vector<int64_t> all8;
    for (int r = 0; r < n; r++) {
        all.insert(all.end(), tickets[r].begin(), tickets[r].end());
        all8.insert(all8.end(), tickets8[r].begin(), tickets8[r].end());
    }
    std::sort(all.begin(), all.end());
    std::sort(all8.begin(), all8.end());
    for (int i = 0; i < n * k; i++) {
        REQUIRE_EQ(all[i], (int64_t)i);
        REQUIRE_EQ(all8[i], (int64_t)i);
    }
    const int8_t* b = (const int8_t*)g.at(0, 8);
    // ranks 0 and 2 alternate bytes 8 and 11, ranks 1 and 3 bytes 10 and 11
    REQUIRE_EQ((int)b[1], n * k);
    REQUIRE_EQ((int)b[0], 2 * ((k + 1) / 2));
    REQUIRE_EQ((int)b[2], 2 * ((k + 1) / 2));
    REQUIRE_EQ((int)b[3], 4 * (k / 2));
}

TEST_CASE("rma: accumulate, replace, no-op and pair padding", "[loopback][rma]")
{
    const int n = 3;
    RmaGroup g(n);
    int fails = g.run([&](int rank, Communicator& c) {
        // every rank adds rank+1 to 1000 i32 elements of rank 1 and takes the
        // running max of f64 values on rank 2
        std::vector<int32_t> add(1000, rank + 1);
        std::vector<double> mx(10, (double)rank - 0.5);
        bool ok = c.accumulate(add.data(), g.win[rank] + 64, add.size(), FB_I32, FB_OP_SUM, 1, nullptr, nullptr) == FB_OK;
        ok = ok && c.accumulate(mx.data(), g.win[rank] + 8192, mx.size(), FB_F64, FB_OP_MAX, 2, nullptr, nullptr) == FB_OK;
        return ok;
    });
    REQUIRE_EQ(fails, 0);
    const int32_t* s = (const int32_t*)g.at(1, 64);
    REQUIRE_EQ(s[0], 6);
    REQUIRE_EQ(s[999], 6);
    REQUIRE_EQ(((const int32_t*)g.at(1, 60))[0], 0);
    REQUIRE_EQ(((const int32_t*)g.at(1, 64 + 4000))[0], 0);
    REQUIRE(((const double*)g.at(2, 8192))[9] == 1.5);

    Communicator& c = *g.comms[0];
    // MAXLOC on a 16-byte pair keeps the target's padding
    uint8_t tgt[16];
    memset(tgt, 0xCD, 16);
    const double v0 = 1.0;
    const int32_t i0 = 4;
    memcpy(tgt, &v0, 8);
    memcpy(tgt + 8, &i0, 4);
    memcpy(g.at(1, 16384), tgt, 16);
    uint8_t org[16];
    memset(org, 0x11, 16);
    const double v1 = 2.0;
    const int32_t i1 = 9;
    memcpy(org, &v1, 8);
    memcpy(org + 8, &i1, 4);
    uint8_t prev[16];
    REQUIRE_EQ(c.accumulate(org, g.win[0] + 16384, 1, FB_F64_I32, FB_OP_MAXLOC, 1, prev, nullptr), FB_OK);
    REQUIRE(memcmp(prev, tgt, 16) == 0);
    REQUIRE(memcmp(g.at(1, 16384), org, 12) == 0);
    REQUIRE(memcmp(g.at(1, 16384 + 12), tgt + 12, 4) == 0);
    // REPLACE and an atomic read (NO_OP)
    const uint8_t b7 = 0x7f;
    const uint16_t h = 0x3c00;
    uint16_t old = 0;
    REQUIRE_EQ(c.accumulate(&b7, g.win[0] + 3, 1, FB_I8, FB_OP_REPLACE, 2, nullptr, nullptr), FB_OK);
    REQUIRE_EQ(c.accumulate(&h, g.win[0] + 6, 1, FB_F16, FB_OP_REPLACE, 2, &old, nullptr), FB_OK);
    REQUIRE_EQ(old, 0);
    uint16_t read = 0;
    REQUIRE_EQ(c.accumulate(nullptr, g.win[0] + 6, 1, FB_BF16, FB_OP_NO_OP, 2, &read, nullptr), FB_OK);
    REQUIRE_EQ(read, 0x3c00);
    REQUIRE_EQ((int)g.at(2, 0)[3], 0x7f);
    REQUIRE_EQ((int)g.at(2, 0)[2], 0);
    REQUIRE_EQ((int)g.at(2, 0)[4], 0);
    REQUIRE(c.stats().launches >= 4);
}

TEST_CASE("rma: compare-and-swap retry loops count exactly", "[loopback][rma]")
{
    const int n = 4;
    const int k = 40;
    RmaGroup g(n);
    int fails = g.run([&](int rank, Communicator& c) {
        bool ok = true;
        for (int dt : { FB_U8, FB_I16, FB_I32, FB_U64 }) {
            const size_t e = fbDtypeSize(dt);
            const uint64_t off = g.win[rank] + 256 + 16 * dt + (16 - e) % 8;
            uint64_t guess = 0;
            for (int done = 0; done < k && ok;) {
                uint64_t next = guess + 1;
                uint64_t got = 0;
                ok = c.compareAndSwap(&guess, &next, &got, off, dt, 0, nullptr) == FB_OK;
                if (got == guess) {
                    done++;
                    guess = next;
                } else {
                    guess = got;
                }
            }
        }
        return ok;
    });
    REQUIRE_EQ(fails, 0);
    for (int dt : { FB_U8, FB_I16, FB_I32, FB_U64 }) {
        const size_t e = fbDtypeSize(dt);
        uint64_t v = 0;
        memcpy(&v, g.at(0, 256 + 16 * dt + (16 - e) % 8), e);
        REQUIRE_EQ(v, (uint64_t)n * k);
    }
}

TEST_CASE("rma: argument checks", "[loopback][rma]")
{
    RmaGroup g(2);
    Communicator& c = *g.comms[0];
    const uint64_t w = g.win[0];
    uint8_t buf[64] = { 0 };
    uint8_t out[64] = { 0 };
    const uint64_t launches = c.stats().launches;
    // unsupported pairs, whatever the fetch
    REQUIRE_EQ(c.accumulate(buf, w, 1, FB_F32, FB_OP_BAND, 1, nullptr, nullptr), FB_E_UNSUPPORTED);
    REQUIRE_EQ(c.accumulate(buf, w, 1, FB_I32, FB_OP_MAXLOC, 1, out, nullptr), FB_E_UNSUPPORTED);
    REQUIRE_EQ(c.accumulate(buf, w, 1, FB_F64_I32, FB_OP_SUM, 1, nullptr, nullptr), FB_E_UNSUPPORTED);
    REQUIRE_EQ(c.accumulate(buf, w, 1, FB_I32, FB_OP_COUNT, 1, nullptr, nullptr), FB_E_UNSUPPORTED);
    // NO_OP needs a fetch buffer
    REQUIRE_EQ(c.accumulate(buf, w, 1, FB_I32, FB_OP_NO_OP, 1, nullptr, nullptr), FB_E_INVALID);
    // misaligned targets, a range outside the user heap, a bad peer or dtype
    REQUIRE_EQ(c.accumulate(buf, w + 2, 1, FB_I32, FB_OP_SUM, 1, nullptr, nullptr), FB_E_INVALID);
    REQUIRE_EQ(c.accumulate(buf, w + 8, 1, FB_F64_I32, FB_OP_MAXLOC, 1, nullptr, nullptr), FB_E_INVALID);
    REQUIRE_EQ(c.accumulate(buf, w + 1, 1, FB_I16, FB_OP_REPLACE, 1, nullptr, nullptr), FB_E_INVALID);
    REQUIRE_EQ(c.accumulate(buf, 0, 1, FB_I32, FB_OP_SUM, 1, nullptr, nullptr), FB_E_INVALID);
    REQUIRE_EQ(c.accumulate(buf, (uint64_t)1 << 40, 1, FB_I32, FB_OP_SUM, 1, nullptr, nullptr), FB_E_INVALID);
    REQUIRE_EQ(c.accumulate(buf, w, (size_t)1 << 40, FB_I32, FB_OP_SUM, 1, nullptr, nullptr), FB_E_INVALID);
    REQUIRE_EQ(c.accumulate(buf, w, 1, FB_I32, FB_OP_SUM, 2, nullptr, nullptr), FB_E_INVALID);
    REQUIRE_EQ(c.accumulate(buf, w, 1, FB_DTYPE_COUNT, FB_OP_SUM, 1, nullptr, nullptr), FB_E_INVALID);
    // compare-and-swap: integers only, aligned, all three buffers
    REQUIRE_EQ(c.compareAndSwap(buf, buf, out, w, FB_F32, 1, nullptr), FB_E_UNSUPPORTED);
    REQUIRE_EQ(c.compareAndSwap(buf, buf, out, w + 4, FB_I64, 1, nullptr), FB_E_INVALID);
    REQUIRE_EQ(c.compareAndSwap(buf, buf, nullptr, w, FB_I64, 1, nullptr), FB_E_INVALID);
    REQUIRE_EQ(c.stats().launches, launches);
    // the collectives reject the one-sided ops
    int32_t* a = (int32_t*)g.at(0, 0);
    REQUIRE_EQ(c.allReduce(a, a, 4, FB_I32, FB_OP_REPLACE, FB_ALGO_AUTO, FB_FLAG_SYMMETRIC, nullptr), FB_E_UNSUPPORTED);
    REQUIRE_EQ(c.allReduce(a, a, 4, FB_I32, FB_OP_NO_OP, FB_ALGO_AUTO, FB_FLAG_SYMMETRIC, nullptr), FB_E_UNSUPPORTED);
    REQUIRE_EQ(c.stats().launches, launches);
    // count 0 is a valid no-op
    REQUIRE_EQ(c.accumulate(nullptr, w, 0, FB_I32, FB_OP_SUM, 1, nullptr, nullptr), FB_OK);
}
