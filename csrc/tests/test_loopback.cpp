// The communicator's host-side logic on the loopback backend (no GPU): one
// thread per rank, heaps and signal pads in host memory, host twins of the
// kernels speaking the same flag protocol.  What is tested here is everything
// the CPU decides: algorithm choice, staging of non-symmetric buffers,
// chunking, channels, grouped segment tables, p2p sequence numbers / bounce
// rings, and that those decisions agree across ranks.
// (Reference collective tests: tests/test/mpi/test_mpi_world.cpp.)
#include "harness.h"

#include <faabric/device/communicator.h>

#include "launch_api.h"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <functional>
#include <limits>
#include <numeric>
#include <random>
#include <set>
#include <thread>

using faabric::device::CommConfig;
using faabric::device::Communicator;

namespace {
struct LoopGroup
{
    std::vector<std::shared_ptr<Communicator>> comms;

    explicit LoopGroup(int n, int channels = 4, size_t stageBytes = (size_t)1 << 20, uint64_t timeoutMs = 5000)
    {
        CommConfig cfg;
        cfg.loopback = true;
        cfg.heapBytes = (size_t)32 << 20;
        cfg.stageBytes = stageBytes;
        cfg.p2pBounceBytes = (size_t)1 << 20;
        cfg.channels = channels;
        cfg.timeoutMs = timeoutMs;
        cfg.maxBlocks = 4;
        std::vector<int> devices(n, 0);
        comms = Communicator::createLocal(n, devices, cfg);
    }

    // fn(rank, comm) on one thread per rank; returns the number of failures
    int run(const std::function<bool(int, Communicator&)>& fn)
    {
        std::atomic<int> failures{ 0 };
        std::vector<std::thread> ts;
        for (int r = 0; r < (int)comms.size(); r++) {
            ts.emplace_back([&, r] {
                try {
                    if (!fn(r, *comms[r])) {
                        failures++;
                    }
                } catch (const std::exception& e) {
                    printf("         rank %d threw: %s\n", r, e.what());
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
T* heapArray(Communicator& c, size_t n)
{
    return reinterpret_cast<T*>(c.heapPtr(c.alloc(std::max<size_t>(n * sizeof(T), 16))));
}
}

TEST_CASE("loopback: backend needs no GPU and reports itself", "[loopback]")
{
    LoopGroup g(2);
    REQUIRE(g.comms[0]->isLoopback());
    REQUIRE_EQ(g.comms[0]->backing(), std::string("loopback"));
    REQUIRE(!g.comms[0]->hasMulticast());
    REQUIRE(!g.comms[0]->streamSync());
    REQUIRE_EQ(g.comms[1]->rank(), 1);
    // symmetric allocations land at the same offset on every rank
    uint64_t a = g.comms[0]->alloc(1000);
    uint64_t b = g.comms[1]->alloc(1000);
    REQUIRE_EQ(a, b);
    REQUIRE(g.comms[0]->heapPtr(a, 1) == g.comms[1]->heapPtr(b));
}

TEST_CASE("loopback: all-reduce, every algorithm, symmetric and staged, odd sizes", "[loopback]")
{
    for (int n : { 2, 3, 4, 8 }) {
        LoopGroup g(n);
        for (int algo : { FB_ALGO_LL, FB_ALGO_ONESHOT, FB_ALGO_TWOSHOT, FB_ALGO_AUTO }) {
            for (size_t count : { (size_t)1, (size_t)7, (size_t)1000, (size_t)4099, (size_t)70001 }) {
                if (algo == FB_ALGO_LL && count * 4 > FB_LL_MAX_BYTES) {
                    continue;
                }
                for (bool symmetric : { true, false }) {
                    int fails = g.run([&](int rank, Communicator& c) {
                        std::vector<int32_t> plain(count), plainOut(count, -1);
                        int32_t* send = symmetric ? heapArray<int32_t>(c, count) : plain.data();
                        int32_t* recv = symmetric ? heapArray<int32_t>(c, count) : plainOut.data();
                        for (size_t i = 0; i < count; i++) {
                            send[i] = (int32_t)(i % 1000) * (rank + 1);
                        }
                        c.hostBarrier();
                        int rc = c.allReduce(send, recv, count, FB_I32, FB_OP_SUM, algo, symmetric ? FB_FLAG_SYMMETRIC : 0, nullptr);
                        if (rc != FB_OK) {
                            return false;
                        }
                        bool ok = c.checkError(nullptr) == 0;
                        for (size_t i = 0; i < count && ok; i++) {
                            ok = recv[i] == (int32_t)(i % 1000) * (n * (n + 1) / 2);
                        }
                        c.hostBarrier();
                        if (symmetric) {
                            c.free(c.offsetOf(recv));
                            c.free(c.offsetOf(send));
                        }
                        return ok;
                    });
                    if (fails != 0) {
                        fbtest::fail(__FILE__, __LINE__, "n=" + std::to_string(n) + " algo=" + std::to_string(algo) + " count=" + std::to_string(count) + " sym=" + std::to_string(symmetric));
                    }
                }
            }
        }
    }
}

TEST_CASE("loopback: reductions over dtypes and ops, pairs included", "[loopback]")
{
    LoopGroup g(4);
    int fails = g.run([&](int rank, Communicator& c) {
        const int n = c.size();
        bool ok = true;
        // float max
        float* f = heapArray<float>(c, 333);
        for (int i = 0; i < 333; i++) {
            f[i] = (float)((i * 7 + rank * 13) % 31) - 15.0f;
        }
        c.hostBarrier();
        ok = ok && c.allReduce(f, f, 333, FB_F32, FB_OP_MAX, FB_ALGO_TWOSHOT, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
        for (int i = 0; i < 333 && ok; i++) {
            float m = -1e9f;
            for (int r = 0; r < n; r++) {
                m = std::max(m, (float)((i * 7 + r * 13) % 31) - 15.0f);
            }
            ok = f[i] == m;
        }
        // double product, bitwise or, logical and
        double* d = heapArray<double>(c, 50);
        uint8_t* b = heapArray<uint8_t>(c, 100);
        int64_t* l = heapArray<int64_t>(c, 17);
        for (int i = 0; i < 50; i++) {
            d[i] = 1.0 + 0.5 * rank;
        }
        for (int i = 0; i < 100; i++) {
            b[i] = (uint8_t)(1u << rank);
        }
        for (int i = 0; i < 17; i++) {
            l[i] = (i % (rank + 2)) != 0;
        }
        c.hostBarrier();
        ok = ok && c.allReduce(d, d, 50, FB_F64, FB_OP_PROD, FB_ALGO_AUTO, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
        ok = ok && c.allReduce(b, b, 100, FB_U8, FB_OP_BOR, FB_ALGO_AUTO, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
        ok = ok && c.allReduce(l, l, 17, FB_I64, FB_OP_LAND, FB_ALGO_AUTO, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
        double prod = 1.0;
        for (int r = 0; r < n; r++) {
            prod *= 1.0 + 0.5 * r;
        }
        ok = ok && d[49] == prod && b[99] == 0x0f;
        for (int i = 0; i < 17 && ok; i++) {
            bool all = true;
            for (int r = 0; r < n; r++) {
                all = all && (i % (r + 2)) != 0;
            }
            ok = l[i] == (int64_t)all;
        }
        // MAXLOC on {double, int}: ties pick the lower index
        struct DI
        {
            double v;
            int32_t i;
            int32_t pad;
        };
        DI* p = heapArray<DI>(c, 9);
        for (int i = 0; i < 9; i++) {
            p[i] = { (double)((i + rank) % 3), rank, 0 };
        }
        c.hostBarrier();
        ok = ok && c.allReduce(p, p, 9, FB_F64_I32, FB_OP_MAXLOC, FB_ALGO_ONESHOT, 0, nullptr) == FB_OK;
        for (int i = 0; i < 9 && ok; i++) {
            double best = -1;
            int who = -1;
            for (int r = 0; r < n; r++) {
                double v = (double)((i + r) % 3);
                if (v > best) {
                    best = v;
                    who = r;
                }
            }
            ok = p[i].v == best && p[i].i == who;
        }
        // bitwise ops on floats are rejected, identically on every rank
        ok = ok && c.allReduce(f, f, 4, FB_F32, FB_OP_BAND, FB_ALGO_AUTO, FB_FLAG_SYMMETRIC, nullptr) == FB_E_UNSUPPORTED;
        return ok && c.checkError(nullptr) == 0;
    });
    REQUIRE_EQ(fails, 0);
}

namespace {
// Full-range integer SUM/PROD: the inputs have the top bit set, so both wrap.
// Expected values are computed in uint64_t (wrapping by definition) and then
// truncated to the width of T.
template<typename T>
bool wrapSumProd(int rank, int n, Communicator& c, int dtype)
{
    const size_t count = 37; // two full vectors and a tail for every width
    auto input = [](int r, size_t i) {
        return (uint64_t)0x9e3779b97f4a7c15ull * (uint64_t)(r + 1) + (uint64_t)0xf00d * i | ((uint64_t)1 << 63) |
               ((uint64_t)1 << (8 * sizeof(T) - 1));
    };
    T* s = heapArray<T>(c, count);
    T* sum = heapArray<T>(c, count);
    T* prod = heapArray<T>(c, count);
    for (size_t i = 0; i < count; i++) {
        s[i] = (T)input(rank, i);
    }
    c.hostBarrier();
    bool ok = c.allReduce(s, sum, count, dtype, FB_OP_SUM, FB_ALGO_ONESHOT, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
    ok = ok && c.allReduce(s, prod, count, dtype, FB_OP_PROD, FB_ALGO_LL, 0, nullptr) == FB_OK;
    for (size_t i = 0; i < count && ok; i++) {
        uint64_t es = 0;
        uint64_t ep = 1;
        for (int r = 0; r < n; r++) {
            es += input(r, i);
            ep *= input(r, i);
        }
        ok = sum[i] == (T)es && prod[i] == (T)ep;
    }
    c.hostBarrier();
    c.free(c.offsetOf(prod));
    c.free(c.offsetOf(sum));
    c.free(c.offsetOf(s));
    return ok;
}

uint16_t bf16Bits(float f)
{
    uint32_t u;
    memcpy(&u, &f, 4);
    return (uint16_t)(u >> 16); // exact for the small integers used below
}

float bf16Value(uint16_t h)
{
    uint32_t u = (uint32_t)h << 16;
    float f;
    memcpy(&f, &u, 4);
    return f;
}
}

TEST_CASE("loopback: integer SUM/PROD wrap and float MAX/MIN ignore where a NaN or -0 sits", "[loopback]")
{
    LoopGroup g(4);
    int fails = g.run([&](int rank, Communicator& c) {
        const int n = c.size();
        bool ok = wrapSumProd<int8_t>(rank, n, c, FB_I8);
        ok = wrapSumProd<uint8_t>(rank, n, c, FB_U8) && ok;
        ok = wrapSumProd<int16_t>(rank, n, c, FB_I16) && ok;
        ok = wrapSumProd<uint16_t>(rank, n, c, FB_U16) && ok;
        ok = wrapSumProd<int32_t>(rank, n, c, FB_I32) && ok;
        ok = wrapSumProd<uint32_t>(rank, n, c, FB_U32) && ok;
        ok = wrapSumProd<int64_t>(rank, n, c, FB_I64) && ok;
        ok = wrapSumProd<uint64_t>(rank, n, c, FB_U64) && ok;

        // rank r holds r + 1; element 0 has a NaN on rank 0, element 1 on rank
        // n - 1, element 2 on every rank.  MAX/MIN skip a NaN operand, so only
        // element 2 is NaN: max = {n, n - 1, NaN, n}, min = {2, 1, NaN, 1}.
        // Elements 4 and 5 are zeros, -0 on rank 0 or on rank n - 1 and +0
        // elsewhere: -0 orders below +0 wherever it sits, so MAX is +0 and MIN -0
        const float nan = std::numeric_limits<float>::quiet_NaN();
        const int count = 6;
        auto input = [&](int r, int i) {
            if (i >= 4) {
                return (i == 4 && r == 0) || (i == 5 && r == n - 1) ? -0.0f : 0.0f;
            }
            bool isNan = (i == 0 && r == 0) || (i == 1 && r == n - 1) || i == 2;
            return isNan ? nan : (float)(r + 1);
        };
        const float expMax[count] = { (float)n, (float)(n - 1), nan, (float)n, 0.0f, 0.0f };
        const float expMin[count] = { 2.0f, 1.0f, nan, 1.0f, -0.0f, -0.0f };
        auto same = [](float got, float exp) {
            return std::isnan(exp) ? std::isnan(got) : got == exp && std::signbit(got) == std::signbit(exp);
        };
        float* f = heapArray<float>(c, count);
        float* fMax = heapArray<float>(c, count);
        float* fMin = heapArray<float>(c, count);
        uint16_t* h = heapArray<uint16_t>(c, count);
        uint16_t* hMax = heapArray<uint16_t>(c, count);
        uint16_t* hMin = heapArray<uint16_t>(c, count);
        for (int i = 0; i < count; i++) {
            f[i] = input(rank, i);
            h[i] = std::isnan(f[i]) ? (uint16_t)0x7fc0 : bf16Bits(f[i]);
        }
        c.hostBarrier();
        for (int algo : { FB_ALGO_LL, FB_ALGO_ONESHOT, FB_ALGO_TWOSHOT }) {
            ok = ok && c.allReduce(f, fMax, count, FB_F32, FB_OP_MAX, algo, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            ok = ok && c.allReduce(f, fMin, count, FB_F32, FB_OP_MIN, algo, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            ok = ok && c.allReduce(h, hMax, count, FB_BF16, FB_OP_MAX, algo, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            ok = ok && c.allReduce(h, hMin, count, FB_BF16, FB_OP_MIN, algo, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            for (int i = 0; i < count && ok; i++) {
                ok = same(fMax[i], expMax[i]) && same(fMin[i], expMin[i]) && same(bf16Value(hMax[i]), expMax[i]) &&
                     same(bf16Value(hMin[i]), expMin[i]);
            }
            if (!ok) {
                printf("         rank %d algo %d: float MAX/MIN depends on where a NaN or -0 sits\n", rank, algo);
            }
        }
        return ok && c.checkError(nullptr) == 0;
    });
    REQUIRE_EQ(fails, 0);
}

TEST_CASE("loopback: a rank with unaligned local buffers stays in step with its peers", "[loopback]")
{
    // advisor finding: the algorithm / number of launches must not depend on
    // rank-local pointer alignment
    LoopGroup g(4);
    int fails = g.run([&](int rank, Communicator& c) {
        std::vector<int32_t> sendStore(2000 + 4), recvStore(2000 + 4);
        // rank 1 and 3 get buffers that are only 4-byte aligned
        int32_t* send = sendStore.data() + (rank % 2);
        int32_t* recv = recvStore.data() + (rank % 2);
        bool ok = true;
        for (int round = 0; round < 3 && ok; round++) {
            for (int i = 0; i < 2000; i++) {
                send[i] = i + rank + round;
            }
            c.hostBarrier();
            ok = c.allReduce(send, recv, 2000, FB_I32, FB_OP_SUM, FB_ALGO_LL, 0, nullptr) == FB_OK;
            ok = ok && c.lastAlgo() == FB_ALGO_LL;
            for (int i = 0; i < 2000 && ok; i++) {
                ok = recv[i] == 4 * (i + round) + 6;
            }
        }
        return ok && c.checkError(nullptr) == 0;
    });
    REQUIRE_EQ(fails, 0);
}

TEST_CASE("loopback: reduce, scan and reduce-scatter, in place on symmetric buffers too", "[loopback]")
{
    for (int n : { 2, 5 }) {
        LoopGroup g(n);
        int fails = g.run([&](int rank, Communicator& c) {
            const int n = c.size();
            bool ok = true;
            const size_t count = 1234;
            int32_t* s = heapArray<int32_t>(c, count);
            int32_t* o = heapArray<int32_t>(c, count);
            for (size_t i = 0; i < count; i++) {
                s[i] = (int32_t)i + rank;
            }
            c.hostBarrier();
            // rooted reduce
            ok = ok && c.reduce(s, o, count, FB_I32, FB_OP_SUM, n - 1, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            if (rank == n - 1) {
                for (size_t i = 0; i < count && ok; i++) {
                    ok = o[i] == (int32_t)i * n + n * (n - 1) / 2;
                }
            }
            // scan IN PLACE on symmetric memory (input overlaps output: staged)
            c.hostBarrier();
            ok = ok && c.scan(s, s, count, FB_I32, FB_OP_SUM, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            for (size_t i = 0; i < count && ok; i++) {
                ok = s[i] == (int32_t)i * (rank + 1) + rank * (rank + 1) / 2;
            }
            // reduce-scatter, output aliasing the head of the input
            const size_t per = 64;
            int32_t* rs = heapArray<int32_t>(c, per * n);
            for (size_t i = 0; i < per * n; i++) {
                rs[i] = (int32_t)(i * 3) + rank;
            }
            c.hostBarrier();
            ok = ok && c.reduceScatter(rs, rs, per, FB_I32, FB_OP_SUM, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            for (size_t i = 0; i < per && ok; i++) {
                size_t gi = (size_t)rank * per + i;
                ok = rs[i] == (int32_t)(gi * 3) * n + n * (n - 1) / 2;
            }
            return ok && c.checkError(nullptr) == 0;
        });
        REQUIRE_EQ(fails, 0);
    }
}

TEST_CASE("loopback: data movement collectives, staged pieces and the two-step broadcast", "[loopback]")
{
    for (int n : { 2, 4, 3 }) {
        // a small staging area forces the non-symmetric paths into several pieces
        LoopGroup g(n, 2, (size_t)64 << 10);
        int fails = g.run([&](int rank, Communicator& c) {
            const int n = c.size();
            bool ok = true;
            const size_t per = 50000; // bytes per pair: > stage / n  => pieces
            std::vector<uint8_t> send(per * n), gathered(per * n, 0), a2a(per * n, 0), got(per, 0);
            for (size_t i = 0; i < send.size(); i++) {
                send[i] = (uint8_t)((i * 31 + rank * 7) % 251);
            }
            c.hostBarrier();
            ok = ok && c.allGather(send.data(), gathered.data(), per, 0, nullptr) == FB_OK;
            for (int r = 0; r < n && ok; r++) {
                for (size_t i = 0; i < per && ok; i += 997) {
                    ok = gathered[(size_t)r * per + i] == (uint8_t)((i * 31 + r * 7) % 251);
                }
            }
            ok = ok && c.allToAll(send.data(), a2a.data(), per, 0, nullptr) == FB_OK;
            for (int r = 0; r < n && ok; r++) {
                for (size_t i = 0; i < per && ok; i += 991) {
                    size_t srcIdx = (size_t)rank * per + i; // what rank r had for me
                    ok = a2a[(size_t)r * per + i] == (uint8_t)((srcIdx * 31 + r * 7) % 251);
                }
            }
            ok = ok && c.scatter(send.data(), got.data(), per, 1 % n, 0, nullptr) == FB_OK;
            for (size_t i = 0; i < per && ok; i += 983) {
                size_t srcIdx = (size_t)rank * per + i;
                ok = got[i] == (uint8_t)((srcIdx * 31 + (1 % n) * 7) % 251);
            }
            std::vector<uint8_t> rootBuf(per * n, 0);
            ok = ok && c.gather(send.data(), rank == 0 ? rootBuf.data() : nullptr, per, 0, 0, nullptr) == FB_OK;
            if (rank == 0) {
                for (int r = 0; r < n && ok; r++) {
                    ok = rootBuf[(size_t)r * per + 5] == (uint8_t)((5 * 31 + r * 7) % 251);
                }
            }
            // symmetric broadcast large enough for scatter + all-gather
            const size_t big = (size_t)3 << 20;
            uint8_t* sym = heapArray<uint8_t>(c, big);
            memset(sym, rank == n - 1 ? 0x5c : 0, big);
            c.hostBarrier();
            ok = ok && c.broadcast(sym, big, n - 1, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            ok = ok && c.lastAlgo() == FB_ALGO_TWOSHOT && sym[0] == 0x5c && sym[big - 1] == 0x5c && sym[big / 2 + 7] == 0x5c;
            ok = ok && c.barrier(nullptr) == FB_OK;
            return ok && c.checkError(nullptr) == 0;
        });
        REQUIRE_EQ(fails, 0);
    }
}

// ---------------------------------------------------------------------------
// Pull collectives whose ranks' destinations differ in alignment.  BlockBarrier
// pairs CTA i of every rank, so every rank must launch the same number of CTAs
// (and kernels) whatever its own pointer; a rank that launches more waits for
// CTAs that never come.  The host twins check the copy width they are given,
// so a width the CUDA kernel could not use fails here too.
// ---------------------------------------------------------------------------
namespace {
// bytes past a 16-byte boundary of rank r's destination: MISALIGN[r % 5]
const size_t MISALIGN[] = { 0, 4, 1, 12, 8 };

uint8_t movePat(int rank, size_t i)
{
    return (uint8_t)(((uint32_t)i * 2654435761u + (uint32_t)rank * 40503u + 17u) >> 13);
}

// `bytes` at `misalign` bytes past a 16-byte boundary, between sentinel bytes
struct Guarded
{
    std::vector<uint8_t> store;
    uint8_t* p;
    size_t bytes;

    Guarded(size_t bytes, size_t misalign)
      : store(bytes + 64, 0xa5)
      , bytes(bytes)
    {
        p = reinterpret_cast<uint8_t*>(((uintptr_t)store.data() + 31) & ~(uintptr_t)15) + misalign;
    }

    bool guardsIntact() const
    {
        for (const uint8_t* q = store.data(); q < store.data() + store.size(); q++) {
            if ((q < p || q >= p + bytes) && *q != 0xa5) {
                return false;
            }
        }
        return true;
    }
};

enum MoveKind
{
    MK_ALLGATHER,
    MK_ALLTOALL,
    MK_GATHER,
    MK_SCATTER,
    MK_BCAST,
};
const char* const MOVE_NAMES[] = { "allGather", "allToAll", "gather", "scatter", "broadcast" };

// One pull collective of `per` bytes per rank (pair), sources in the heap
// (`symmetric`) or in local memory (staged), every destination at its rank's
// MISALIGN; gather passes a destination on the root only.  Checks the return
// code, the error word, every destination byte and the sentinels around it.
// Every rank makes every call, failed or not, so a failure cannot leave the
// other ranks waiting in hostBarrier.
bool divergentMove(int rank, Communicator& c, MoveKind kind, size_t per, bool symmetric, int root)
{
    const int n = c.size();
    const size_t srcRows = (kind == MK_ALLTOALL || kind == MK_SCATTER) ? n : 1;
    const size_t dstBytes = (kind == MK_SCATTER || kind == MK_BCAST) ? per : per * n;
    const int flags = symmetric ? FB_FLAG_SYMMETRIC : 0;
    Guarded dst(dstBytes, MISALIGN[rank % 5]);
    Guarded localSrc(per * srcRows, 0);
    uint64_t symOff = 0;
    uint8_t* src = localSrc.p;
    if (symmetric) {
        symOff = c.alloc(per * srcRows);
        src = c.heapPtr(symOff);
    }
    for (size_t i = 0; i < per * srcRows; i++) {
        src[i] = movePat(rank, i);
    }
    if (kind == MK_BCAST && rank == root) {
        memcpy(dst.p, src, per);
    }
    c.hostBarrier();
    int rc = FB_E_INVALID;
    switch (kind) {
        case MK_ALLGATHER:
            rc = c.allGather(src, dst.p, per, flags, nullptr);
            break;
        case MK_ALLTOALL:
            rc = c.allToAll(src, dst.p, per, flags, nullptr);
            break;
        case MK_GATHER:
            rc = c.gather(src, rank == root ? dst.p : nullptr, per, root, flags, nullptr);
            break;
        case MK_SCATTER:
            rc = c.scatter(src, dst.p, per, root, flags, nullptr);
            break;
        case MK_BCAST:
            rc = c.broadcast(dst.p, per, root, 0, nullptr);
            break;
    }
    const uint32_t err = c.checkError(nullptr);
    bool ok = rc == FB_OK && err == 0 && dst.guardsIntact();
    for (size_t i = 0; i < dstBytes && ok; i++) {
        const size_t p = i / per;
        const size_t k = i % per;
        uint8_t want = dst.p[i];
        switch (kind) {
            case MK_ALLGATHER:
                want = movePat((int)p, k);
                break;
            case MK_ALLTOALL:
                want = movePat((int)p, (size_t)rank * per + k);
                break;
            case MK_GATHER:
                want = rank == root ? movePat((int)p, k) : 0xa5;
                break;
            case MK_SCATTER:
                want = movePat(root, (size_t)rank * per + i);
                break;
            case MK_BCAST:
                want = movePat(root, i);
                break;
        }
        ok = dst.p[i] == want;
    }
    if (!ok) {
        printf("         rank %d %s of %zu bytes (%s, root %d): rc %d, error word %u\n", rank, MOVE_NAMES[kind], per,
               symmetric ? "symmetric" : "staged", root, rc, err);
    }
    c.hostBarrier();
    if (symmetric) {
        c.free(symOff);
    }
    return ok;
}
}

TEST_CASE("loopback: pull collectives launch one grid when ranks' destinations differ in alignment", "[loopback]")
{
    // 8 KiB takes one CTA with 16-byte words and two or more with narrower
    // ones; with tmaMinBytes = 4 KiB, aligned ranks take the TMA kernel and
    // the others cannot (its grid is sized from tiles)
    for (int n : { 2, 3, 4 }) {
        for (size_t tmaMin : { (size_t)256 << 10, (size_t)4096 }) {
            LoopGroup g(n);
            int fails = g.run([&](int rank, Communicator& c) {
                c.config().maxBlocks = 16;
                c.config().tmaMinBytes = tmaMin;
                const uint64_t tmaBefore = c.stats().tmaLaunches;
                bool ok = true;
                for (size_t per : { (size_t)8192, (size_t)40016 }) {
                    for (bool symmetric : { false, true }) {
                        for (int k = MK_ALLGATHER; k <= MK_BCAST; k++) {
                            if (symmetric && k == MK_BCAST) {
                                continue; // a symmetric buffer sits at one offset on every rank
                            }
                            ok = divergentMove(rank, c, (MoveKind)k, per, symmetric, n - 1) && ok;
                        }
                    }
                }
                // rank 0's destinations are aligned: it really ran the TMA twin
                if (ok && rank == 0 && tmaMin == 4096) {
                    ok = c.stats().tmaLaunches > tmaBefore;
                }
                return ok;
            });
            if (fails != 0) {
                printf("         n %d, tmaMinBytes %zu\n", n, tmaMin);
            }
            REQUIRE_EQ(fails, 0);
        }
    }
}

TEST_CASE("loopback: staged pieces stay in step when ranks' destinations differ in alignment", "[loopback]")
{
    // 64 KiB of staging: 100000 and 100004 bytes per rank pair take several
    // pieces; with 100004 the last one is not a multiple of 16 bytes
    for (int n : { 2, 3, 4 }) {
        LoopGroup g(n, 4, (size_t)64 << 10);
        int fails = g.run([&](int rank, Communicator& c) {
            c.config().maxBlocks = 16;
            const uint64_t stagedBefore = c.stats().stagedCopies;
            bool ok = true;
            for (size_t per : { (size_t)100000, (size_t)100004 }) {
                for (int k = MK_ALLGATHER; k <= MK_BCAST; k++) {
                    ok = divergentMove(rank, c, (MoveKind)k, per, false, (int)(per % 3) % n) && ok;
                }
            }
            return ok && c.stats().stagedCopies > stagedBefore;
        });
        if (fails != 0) {
            printf("         n %d\n", n);
        }
        REQUIRE_EQ(fails, 0);
    }
}

TEST_CASE("loopback: the two-step broadcast only runs on 16-byte aligned heap offsets", "[loopback]")
{
    // (total, heap offset mod 16, bcast2StepMinBytes): 16 and 48 bytes give
    // empty and uneven slices; the two-step kernel moves 16-byte words
    struct Case
    {
        size_t total;
        size_t misalign;
        size_t minBytes;
    };
    const Case cases[] = {
        { ((size_t)1 << 20) + 16, 4, (size_t)1 << 20 },  { ((size_t)1 << 20) + 16, 0, (size_t)1 << 20 },
        { ((size_t)1 << 20) + 48, 8, (size_t)1 << 20 },   { 16, 0, 16 },
        { 48, 0, 16 },                                    { 4096 + 16, 0, 16 },
        { 4096 + 16, 12, 16 },                            { ((size_t)1 << 20) + 16 * 5, 0, 16 },
    };
    for (int n : { 4, 3, 5 }) {
        LoopGroup g(n);
        int fails = g.run([&](int rank, Communicator& c) {
            bool ok = true;
            for (const Case& cs : cases) {
                c.config().bcast2StepMinBytes = cs.minBytes;
                const int root = (int)(cs.total / 16) % c.size();
                const uint64_t off = c.alloc(cs.total + 64);
                uint8_t* base = c.heapPtr(off);
                uint8_t* buf = base + 16 + cs.misalign;
                memset(base, 0xa5, cs.total + 64);
                if (rank == root) {
                    for (size_t i = 0; i < cs.total; i++) {
                        buf[i] = movePat(root, i);
                    }
                }
                c.hostBarrier();
                const int rc = c.broadcast(buf, cs.total, root, FB_FLAG_SYMMETRIC, nullptr);
                const bool twoStep = c.lastAlgo() == FB_ALGO_TWOSHOT;
                bool good = rc == FB_OK && c.checkError(nullptr) == 0 && twoStep == (cs.misalign == 0);
                for (size_t i = 0; i < cs.total + 64 && good; i++) {
                    const uint8_t* q = base + i;
                    good = *q == ((q >= buf && q < buf + cs.total) ? movePat(root, (size_t)(q - buf)) : 0xa5);
                }
                if (!good) {
                    printf("         rank %d broadcast of %zu bytes at heap offset +%zu: rc %d, two-step %d\n", rank,
                           cs.total, cs.misalign, rc, (int)twoStep);
                }
                ok = ok && good;
                c.hostBarrier();
                c.free(off);
            }
            return ok;
        });
        if (fails != 0) {
            printf("         n %d\n", n);
        }
        REQUIRE_EQ(fails, 0);
    }
}

TEST_CASE("loopback: point-to-point and put-with-signal at every local alignment", "[loopback]")
{
    LoopGroup g(3);
    int fails = g.run([&](int rank, Communicator& c) {
        const int n = c.size();
        const int next = (rank + 1) % n;
        const int prev = (rank + n - 1) % n;
        // the bounce slot (largest eager chunk) is half the 1 MiB ring
        const size_t slot = (size_t)512 << 10;
        bool ok = true;
        for (size_t misalign : { 0, 1, 4, 12 }) {
            for (size_t bytes : { (size_t)0, (size_t)1, (size_t)15, (size_t)16, (size_t)17, slot - 1, slot, slot + 1 }) {
                Guarded out(bytes, misalign);
                Guarded in(bytes, (misalign * 3) % 16);
                Guarded in2(bytes, (misalign + 1) % 16);
                for (size_t i = 0; i < bytes; i++) {
                    out.p[i] = movePat(rank, i + bytes);
                }
                int rc = c.send(out.p, bytes, next, nullptr);
                rc = rc == FB_OK ? c.recv(in.p, bytes, prev, nullptr) : rc;
                rc = rc == FB_OK ? c.sendRecv(out.p, bytes, next, in2.p, bytes, prev, nullptr) : rc;
                bool good = rc == FB_OK && c.checkError(nullptr) == 0 && in.guardsIntact() && in2.guardsIntact();
                for (size_t i = 0; i < bytes && good; i++) {
                    good = in.p[i] == movePat(prev, i + bytes) && in2.p[i] == movePat(prev, i + bytes);
                }
                if (!good) {
                    printf("         rank %d p2p of %zu bytes at +%zu: rc %d\n", rank, bytes, misalign, rc);
                }
                ok = ok && good;
            }
        }
        // put-with-signal into a symmetric destination at an odd heap offset
        for (size_t misalign : { 0, 1, 4, 12 }) {
            for (size_t bytes : { (size_t)1, (size_t)17, (size_t)4099 }) {
                const uint64_t off = c.alloc(bytes + 64);
                uint8_t* base = c.heapPtr(off);
                memset(base, 0xa5, bytes + 64);
                Guarded out(bytes, (misalign + 4) % 16);
                for (size_t i = 0; i < bytes; i++) {
                    out.p[i] = movePat(rank, i);
                }
                c.hostBarrier();
                int rc = c.putSignal(out.p, off + 16 + misalign, bytes, next, 7, 2, nullptr);
                rc = rc == FB_OK ? c.waitSignal(7, 2, nullptr) : rc;
                bool good = rc == FB_OK && c.checkError(nullptr) == 0;
                for (size_t i = 0; i < bytes + 64 && good; i++) {
                    const bool inside = i >= 16 + misalign && i < 16 + misalign + bytes;
                    good = base[i] == (inside ? movePat(prev, i - 16 - misalign) : 0xa5);
                }
                if (!good) {
                    printf("         rank %d put of %zu bytes at heap +%zu: rc %d\n", rank, bytes, misalign, rc);
                }
                ok = ok && good;
                c.hostBarrier();
                c.free(off);
            }
        }
        return ok;
    });
    REQUIRE_EQ(fails, 0);
}

TEST_CASE("loopback: grouped all-reduce equals per-tensor all-reduces", "[loopback]")
{
    const std::vector<size_t> sizes = { 1, 3, 4, 7, 64, 1000, 4099, 65541, 9408, 2, 33, 300000 };
    for (int n : { 1, 2, 4, 8, 3 }) {
        LoopGroup g(n, 1);
        int fails = g.run([&](int rank, Communicator& c) {
            const int n = c.size();
            std::vector<Communicator::GroupItem> items;
            std::vector<int16_t*> sends, recvs;
            for (size_t sz : sizes) {
                int16_t* s = heapArray<int16_t>(c, sz);
                int16_t* r = heapArray<int16_t>(c, sz);
                for (size_t i = 0; i < sz; i++) {
                    s[i] = (int16_t)((i % 97) + rank);
                    r[i] = -1;
                }
                sends.push_back(s);
                recvs.push_back(r);
                items.push_back({ s, r, sz });
            }
            c.hostBarrier();
            int rc = FB_OK;
            auto plan = c.prepareGroup(items.data(), items.size(), FB_I16, &rc);
            bool ok = plan != nullptr && rc == FB_OK && Communicator::groupPlanLaunches(*plan) == 1;
            ok = ok && c.allReduceGroup(*plan, FB_OP_SUM, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            for (size_t t = 0; t < sizes.size() && ok; t++) {
                for (size_t i = 0; i < sizes[t] && ok; i++) {
                    ok = recvs[t][i] == (int16_t)((i % 97) * n + n * (n - 1) / 2);
                }
            }
            // transient table, in place, MAX
            c.hostBarrier();
            for (auto& it : items) {
                it.recv = const_cast<void*>(it.send);
            }
            ok = ok && c.allReduceMany(items.data(), items.size(), FB_I16, FB_OP_MAX, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            for (size_t t = 0; t < sizes.size() && ok; t++) {
                for (size_t i = 0; i < sizes[t] && ok; i++) {
                    ok = sends[t][i] == (int16_t)((i % 97) + n - 1);
                }
            }
            // a tensor outside the heap cannot be grouped
            std::vector<int16_t> outside(8);
            Communicator::GroupItem bad{ outside.data(), outside.data(), 8 };
            ok = ok && c.prepareGroup(&bad, 1, FB_I16, &rc) == nullptr && rc == FB_E_INVALID;
            return ok && c.checkError(nullptr) == 0;
        });
        REQUIRE_EQ(fails, 0);
    }
}

TEST_CASE("loopback: a group larger than one segment table is split into launches", "[loopback]")
{
    LoopGroup g(2, 1);
    int fails = g.run([&](int rank, Communicator& c) {
        const size_t k = 2500;
        int32_t* flat = heapArray<int32_t>(c, k * 16);
        std::vector<Communicator::GroupItem> items;
        for (size_t i = 0; i < k; i++) {
            for (size_t j = 0; j < 16; j++) {
                flat[i * 16 + j] = (int32_t)(i + j) + rank;
            }
            items.push_back({ flat + i * 16, flat + i * 16, 1 + i % 13 });
        }
        c.hostBarrier();
        int rc = FB_OK;
        auto plan = c.prepareGroup(items.data(), items.size(), FB_I32, &rc);
        bool ok = plan != nullptr && Communicator::groupPlanLaunches(*plan) == 3;
        ok = ok && c.allReduceGroup(*plan, FB_OP_SUM, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
        for (size_t i = 0; i < k && ok; i++) {
            for (size_t j = 0; j < 16 && ok; j++) {
                int32_t own = (int32_t)(i + j) + rank;
                int32_t red = 2 * (int32_t)(i + j) + 1;
                ok = flat[i * 16 + j] == (j < 1 + i % 13 ? red : own);
            }
        }
        return ok && c.checkError(nullptr) == 0;
    });
    REQUIRE_EQ(fails, 0);
}

TEST_CASE("loopback: point-to-point FIFO, deep eager buffering, big exchanges, self messages", "[loopback]")
{
    LoopGroup g(4);
    int fails = g.run([&](int rank, Communicator& c) {
        const int n = c.size();
        const int next = (rank + 1) % n;
        const int prev = (rank + n - 1) % n;
        bool ok = true;
        // 40 sends before the first receive: eager (bounce ring + descriptors)
        const int nMsgs = 40;
        std::vector<std::vector<int32_t>> outs(nMsgs), ins(nMsgs);
        for (int k = 0; k < nMsgs; k++) {
            outs[k].assign(1 + (size_t)k * 53, rank * 1000 + k);
            ins[k].assign(outs[k].size(), -1);
        }
        for (int k = 0; k < nMsgs && ok; k++) {
            ok = c.send(outs[k].data(), outs[k].size() * 4, next, nullptr) == FB_OK;
        }
        for (int k = 0; k < nMsgs && ok; k++) {
            ok = c.recv(ins[k].data(), ins[k].size() * 4, prev, nullptr) == FB_OK;
            ok = ok && ins[k].front() == prev * 1000 + k && ins[k].back() == prev * 1000 + k;
        }
        // exchange far larger than the bounce ring (1 MiB): chunks interleave
        std::vector<uint8_t> bigOut((size_t)5 << 20, (uint8_t)(rank + 1)), bigIn(bigOut.size(), 0);
        ok = ok && c.sendRecv(bigOut.data(), bigOut.size(), next, bigIn.data(), bigIn.size(), prev, nullptr) == FB_OK;
        ok = ok && bigIn.front() == (uint8_t)(prev + 1) && bigIn.back() == (uint8_t)(prev + 1);
        // zero-byte message still synchronises; message to self
        ok = ok && c.send(nullptr, 0, next, nullptr) == FB_OK && c.recv(nullptr, 0, prev, nullptr) == FB_OK;
        int32_t selfOut = 77 + rank;
        int32_t selfIn = 0;
        ok = ok && c.send(&selfOut, 4, rank, nullptr) == FB_OK && c.recv(&selfIn, 4, rank, nullptr) == FB_OK;
        ok = ok && selfIn == 77 + rank;
        // one-sided put + signal
        int32_t* window = heapArray<int32_t>(c, 256);
        memset(window, 0, 1024);
        c.hostBarrier();
        std::vector<int32_t> payload(256, rank + 500);
        ok = ok && c.putSignal(payload.data(), c.offsetOf(window), 1024, next, 5, 3, nullptr) == FB_OK;
        ok = ok && c.waitSignal(5, 3, nullptr) == FB_OK;
        ok = ok && window[0] == prev + 500 && window[255] == prev + 500;
        return ok && c.checkError(nullptr) == 0;
    });
    REQUIRE_EQ(fails, 0);
}

TEST_CASE("loopback: channels keep independent collectives apart", "[loopback]")
{
    LoopGroup g(2, 4);
    int fails = g.run([&](int rank, Communicator& c) {
        bool ok = true;
        int32_t* bufs[4];
        for (int ch = 0; ch < 4; ch++) {
            bufs[ch] = heapArray<int32_t>(c, 5000);
            for (int i = 0; i < 5000; i++) {
                bufs[ch][i] = ch * 10 + rank;
            }
        }
        c.hostBarrier();
        for (int round = 0; round < 3; round++) {
            for (int ch = 3; ch >= 0 && ok; ch--) {
                ok = c.allReduce(bufs[ch], bufs[ch], 5000, FB_I32, FB_OP_MAX, FB_ALGO_TWOSHOT,
                                 FB_FLAG_SYMMETRIC | FB_FLAG_CHANNEL(ch), nullptr) == FB_OK;
            }
        }
        for (int ch = 0; ch < 4 && ok; ch++) {
            ok = bufs[ch][4999] == ch * 10 + 1;
        }
        // staged (non-symmetric) buffers only exist on channel 0
        std::vector<int32_t> plain(10, 1);
        ok = ok && c.allReduce(plain.data(), plain.data(), 10, FB_I32, FB_OP_SUM, FB_ALGO_ONESHOT, FB_FLAG_CHANNEL(2), nullptr) == FB_E_INVALID;
        return ok && c.checkError(nullptr) == 0;
    });
    REQUIRE_EQ(fails, 0);
}

TEST_CASE("loopback: a missing peer trips the watchdog instead of hanging", "[loopback]")
{
    LoopGroup g(2, 1, (size_t)1 << 20, 200);
    std::vector<int32_t> a(100, 1), b(100, 0);
    // only rank 0 shows up
    int rc = g.comms[0]->allReduce(a.data(), b.data(), 100, FB_I32, FB_OP_SUM, FB_ALGO_ONESHOT, 0, nullptr);
    REQUIRE_EQ(rc, FB_OK);
    REQUIRE(g.comms[0]->checkError(nullptr) != 0);
}

// ---------------------------------------------------------------------------
// The MPI C API over the loopback backend: device dispatch, symmetric
// MPI_Alloc_mem memory, MPI_Iallreduce bursts coalesced into grouped launches,
// MPI_IN_PLACE at the root - all without a GPU.
// ---------------------------------------------------------------------------
#include "fixtures.h"

#include <faabric/mpi/MpiWorld.h>
#include <faabric/mpi/MpiWorldRegistry.h>
#include <faabric/mpi/mpi.h>

#define CHECK_RANK_LB(cond)                                                    \
    do {                                                                       \
        if (!(cond)) {                                                         \
            printf("         rank %d: check failed at line %d: %s\n", rank, __LINE__, #cond); \
            return 1;                                                          \
        }                                                                      \
    } while (0)

namespace {
std::atomic<uint64_t> loopbackDeviceCollectives{ 0 };
std::atomic<uint64_t> loopbackGroupLaunches{ 0 };

int loopbackMpiBody(int rank, int size)
{
    auto& world =
      faabric::mpi::getMpiWorldRegistry().getWorld(faabric::executor::ExecutorContext::get()->getMsg().mpiworldid());
    auto comm = world.getDeviceComm(rank);
    CHECK_RANK_LB(comm != nullptr);
    CHECK_RANK_LB(comm->isLoopback());
    const int nTensors = 30;
    const size_t per = 777; // odd: tails in the grouped kernel
    int *send = nullptr, *recv = nullptr;
    CHECK_RANK_LB(MPI_Alloc_mem(nTensors * 1024 * sizeof(int), MPI_INFO_FAABRIC_DEVICE, &send) == MPI_SUCCESS);
    CHECK_RANK_LB(MPI_Alloc_mem(nTensors * 1024 * sizeof(int), MPI_INFO_FAABRIC_DEVICE, &recv) == MPI_SUCCESS);
    CHECK_RANK_LB(comm->inHeap(send, 16) && faabric::mpi::MpiWorld::isDevicePointer(send));
    for (int t = 0; t < nTensors; t++) {
        for (size_t i = 0; i < per; i++) {
            send[t * 1024 + i] = t + rank;
        }
    }
    // burst of non-blocking all-reduces -> ONE grouped launch at the wait
    const uint64_t launchesBefore = comm->stats().launches;
    std::vector<MPI_Request> reqs(nTensors);
    for (int t = 0; t < nTensors; t++) {
        MPI_Iallreduce(send + t * 1024, recv + t * 1024, (int)per, MPI_INT, MPI_SUM, MPI_COMM_WORLD, &reqs[t]);
    }
    MPI_Waitall(nTensors, reqs.data(), MPI_STATUSES_IGNORE);
    const uint64_t launchesAfter = comm->stats().launches;
    for (int t = 0; t < nTensors; t++) {
        int expected = t * size + size * (size - 1) / 2;
        CHECK_RANK_LB(recv[t * 1024] == expected && recv[t * 1024 + per - 1] == expected);
    }
    if (rank == 0) {
        loopbackGroupLaunches = launchesAfter - launchesBefore;
    }
    // blocking collectives on the same memory
    MPI_Allreduce(MPI_IN_PLACE, recv, (int)per, MPI_INT, MPI_MAX, MPI_COMM_WORLD);
    CHECK_RANK_LB(recv[0] == 0 * size + size * (size - 1) / 2);
    // MPI_IN_PLACE at the root only: every rank must take the same path
    for (size_t i = 0; i < per; i++) {
        send[i] = rank + 1;
    }
    if (rank == 1) {
        MPI_Reduce(MPI_IN_PLACE, send, (int)per, MPI_INT, MPI_SUM, 1, MPI_COMM_WORLD);
        CHECK_RANK_LB(send[0] == size * (size + 1) / 2 && send[per - 1] == send[0]);
    } else {
        MPI_Reduce(send, nullptr, (int)per, MPI_INT, MPI_SUM, 1, MPI_COMM_WORLD);
    }
    for (int i = 0; i < 16; i++) {
        send[2048 + i] = rank * 10 + i;
    }
    if (rank == 0) {
        for (int i = 0; i < 16 * size; i++) {
            recv[i] = -1;
        }
        for (int i = 0; i < 16; i++) {
            recv[i] = i; // own chunk already in place
        }
        MPI_Gather(MPI_IN_PLACE, 0, MPI_DATATYPE_NULL, recv, 16, MPI_INT, 0, MPI_COMM_WORLD);
        for (int r = 0; r < size; r++) {
            CHECK_RANK_LB(recv[r * 16 + 3] == r * 10 + 3);
        }
    } else {
        MPI_Gather(send + 2048, 16, MPI_INT, nullptr, 0, MPI_INT, 0, MPI_COMM_WORLD);
    }
    // broadcast / all-gather / scan on heap memory
    if (rank == 2 % size) {
        for (int i = 0; i < 100; i++) {
            send[i] = 4242 + i;
        }
    }
    MPI_Bcast(send, 100, MPI_INT, 2 % size, MPI_COMM_WORLD);
    CHECK_RANK_LB(send[99] == 4242 + 99);
    for (int i = 0; i < 8; i++) {
        send[4096 + i] = rank;
    }
    MPI_Allgather(send + 4096, 8, MPI_INT, recv, 8, MPI_INT, MPI_COMM_WORLD);
    for (int r = 0; r < size; r++) {
        CHECK_RANK_LB(recv[r * 8 + 7] == r);
    }
    MPI_Barrier(MPI_COMM_WORLD);
    if (rank == 0) {
        loopbackDeviceCollectives = world.getDeviceCollectiveCount();
    }
    MPI_Free_mem(send);
    MPI_Free_mem(recv);
    return 0;
}
}

TEST_CASE("loopback: the MPI C API dispatches to the device communicator without a GPU", "[loopback][mpi]")
{
    using namespace tests;
    LoopbackBackend loopback;
    const int worldSize = 4;
    {
        ClusterFixture f(worldSize);
        REQUIRE_EQ(f.conf.deviceBackend, std::string("loopback"));
        registerTestFunction("mpi", "loopback-device", [&](auto*, int, int, auto) {
            MPI_Init(nullptr, nullptr);
            int rank = -1, size = -1;
            MPI_Comm_rank(MPI_COMM_WORLD, &rank);
            MPI_Comm_size(MPI_COMM_WORLD, &size);
            int rc = loopbackMpiBody(rank, size);
            MPI_Finalize();
            return rc;
        });
        auto req = faabric::util::batchExecFactory("mpi", "loopback-device", 1);
        req->mutable_messages(0)->set_ismpi(true);
        req->mutable_messages(0)->set_mpiworldsize(worldSize);
        loopbackDeviceCollectives = 0;
        loopbackGroupLaunches = 99;
        f.plannerCli.callFunctions(req);
        auto status = f.awaitBatch(req, 60000);
        REQUIRE_EQ(status->messageresults_size(), worldSize);
        for (auto& m : status->messageresults()) {
            if (m.returnvalue() != 0) {
                fbtest::fail(__FILE__, __LINE__, "rank " + std::to_string(m.mpirank()) + " failed: " + m.outputdata());
            }
        }
        // the 30 non-blocking all-reduces were ONE grouped launch
        REQUIRE_EQ(loopbackGroupLaunches.load(), 1u);
        REQUIRE(loopbackDeviceCollectives.load() >= 30u + 5u);
        faabric::mpi::getMpiWorldRegistry().clear();
    }
}

namespace {
// Commutative and associative: a op b = a + b + 1, so a missing or stale
// contribution shows in every element
void plusOneFn(void* in, void* inout, int* len, MPI_Datatype*)
{
    auto* a = (const int*)in;
    auto* b = (int*)inout;
    for (int i = 0; i < *len; i++) {
        b[i] = a[i] + b[i] + 1;
    }
}

// Host fallbacks of the MPI C API on MPI_Alloc_mem(MPI_INFO_FAABRIC_DEVICE)
// memory, which the loopback backend keeps in host memory: a user-defined
// operation, the own blocks of the v-collectives and uneven reduce-scatter
// blocks.  Every rank runs every call whatever it finds, so a wrong result
// cannot leave a peer waiting.
int loopbackHostFallbackBody(int rank, int size)
{
    std::set<int> failedLines;
    auto check = [&](bool ok, int line) {
        if (!ok && failedLines.insert(line).second) {
            printf("         rank %d: check failed at line %d\n", rank, line);
        }
    };
    MPI_Op plusOne = nullptr;
    check(MPI_Op_create(plusOneFn, 1, &plusOne) == MPI_SUCCESS, __LINE__);
    const int n = 300;
    int *a = nullptr, *b = nullptr;
    check(MPI_Alloc_mem(n * sizeof(int), MPI_INFO_FAABRIC_DEVICE, &a) == MPI_SUCCESS, __LINE__);
    check(MPI_Alloc_mem(n * sizeof(int), MPI_INFO_FAABRIC_DEVICE, &b) == MPI_SUCCESS, __LINE__);
    check(faabric::mpi::MpiWorld::isDevicePointer(a) && faabric::mpi::MpiWorld::isDevicePointer(b), __LINE__);
    auto value = [](int r, int i) { return r * 1000 + i; };
    // op over ranks [0, last]
    auto folded = [&](int last, int i) {
        int v = 0;
        for (int r = 0; r <= last; r++) {
            v += value(r, i);
        }
        return v + last;
    };
    auto fill = [&](int* p, int v) { std::fill(p, p + n, v); };
    auto load = [&]() {
        for (int i = 0; i < n; i++) {
            a[i] = value(rank, i);
        }
    };

    load();
    fill(b, -1);
    MPI_Allreduce(a, b, n, MPI_INT, plusOne, MPI_COMM_WORLD);
    for (int i = 0; i < n; i++) {
        check(b[i] == folded(size - 1, i) && a[i] == value(rank, i), __LINE__);
    }
    MPI_Allreduce(MPI_IN_PLACE, a, n, MPI_INT, plusOne, MPI_COMM_WORLD);
    for (int i = 0; i < n; i++) {
        check(a[i] == folded(size - 1, i), __LINE__);
    }

    const int root = 2;
    load();
    fill(b, -1);
    MPI_Reduce(a, rank == root ? b : nullptr, n, MPI_INT, plusOne, root, MPI_COMM_WORLD);
    for (int i = 0; rank == root && i < n; i++) {
        check(b[i] == folded(size - 1, i), __LINE__);
    }

    load();
    fill(b, -1);
    MPI_Scan(a, b, n, MPI_INT, plusOne, MPI_COMM_WORLD);
    for (int i = 0; i < n; i++) {
        check(b[i] == folded(rank, i), __LINE__);
    }

    // Gatherv to rank 1: rank r sends r + 1 ints, blocks two apart
    const int gatherRoot = 1;
    std::vector<int> counts(size), displs(size);
    for (int r = 0, off = 0; r < size; r++) {
        counts[r] = r + 1;
        displs[r] = off;
        off += counts[r] + 2;
    }
    load();
    fill(b, -1);
    MPI_Gatherv(a, rank + 1, MPI_INT, b, counts.data(), displs.data(), MPI_INT, gatherRoot, MPI_COMM_WORLD);
    for (int r = 0; rank == gatherRoot && r < size; r++) {
        for (int j = 0; j < counts[r]; j++) {
            check(b[displs[r] + j] == value(r, j), __LINE__);
        }
        check(b[displs[r] + counts[r]] == -1, __LINE__);
    }

    // Alltoallv: rank s sends (s + d) % 3 + 1 ints to rank d
    auto pairCount = [](int s, int d) { return (s + d) % 3 + 1; };
    std::vector<int> sendCounts(size), sendDispls(size), recvCounts(size), recvDispls(size);
    for (int r = 0, so = 0, ro = 0; r < size; r++) {
        sendCounts[r] = pairCount(rank, r);
        recvCounts[r] = pairCount(r, rank);
        sendDispls[r] = so;
        recvDispls[r] = ro;
        so += sendCounts[r];
        ro += recvCounts[r];
    }
    for (int r = 0; r < size; r++) {
        for (int j = 0; j < sendCounts[r]; j++) {
            a[sendDispls[r] + j] = value(rank, r * 10 + j);
        }
    }
    fill(b, -1);
    MPI_Alltoallv(a, sendCounts.data(), sendDispls.data(), MPI_INT, b, recvCounts.data(), recvDispls.data(), MPI_INT,
                  MPI_COMM_WORLD);
    for (int r = 0; r < size; r++) {
        for (int j = 0; j < recvCounts[r]; j++) {
            check(b[recvDispls[r] + j] == value(r, rank * 10 + j), __LINE__);
        }
    }

    // Reduce_scatter with uneven blocks: rank r keeps r + 1 elements
    load();
    fill(b, -1);
    MPI_Reduce_scatter(a, b, counts.data(), MPI_INT, MPI_SUM, MPI_COMM_WORLD);
    const int first = rank * (rank + 1) / 2;
    for (int j = 0; j < counts[rank]; j++) {
        check(b[j] == folded(size - 1, first + j) - (size - 1), __LINE__);
    }
    check(b[counts[rank]] == -1, __LINE__);

    check(MPI_Op_free(&plusOne) == MPI_SUCCESS, __LINE__);
    MPI_Free_mem(a);
    MPI_Free_mem(b);
    return (int)failedLines.size();
}
}

TEST_CASE("loopback: host fallbacks of the MPI C API on device-role memory without a GPU", "[loopback][mpi]")
{
    using namespace tests;
    LoopbackBackend loopback;
    const int worldSize = 4;
    ClusterFixture f(worldSize);
    REQUIRE_EQ(f.conf.deviceBackend, std::string("loopback"));
    registerTestFunction("mpi", "loopback-host-fallback", [&](auto*, int, int, auto) {
        MPI_Init(nullptr, nullptr);
        int rank = -1, size = -1;
        MPI_Comm_rank(MPI_COMM_WORLD, &rank);
        MPI_Comm_size(MPI_COMM_WORLD, &size);
        int rc = loopbackHostFallbackBody(rank, size);
        MPI_Finalize();
        return rc;
    });
    auto req = faabric::util::batchExecFactory("mpi", "loopback-host-fallback", 1);
    req->mutable_messages(0)->set_ismpi(true);
    req->mutable_messages(0)->set_mpiworldsize(worldSize);
    f.plannerCli.callFunctions(req);
    auto status = f.awaitBatch(req, 60000);
    REQUIRE_EQ(status->messageresults_size(), worldSize);
    for (auto& m : status->messageresults()) {
        if (m.returnvalue() != 0) {
            fbtest::fail(__FILE__, __LINE__, "rank " + std::to_string(m.mpirank()) + " failed");
        }
    }
    faabric::mpi::getMpiWorldRegistry().clear();
}
