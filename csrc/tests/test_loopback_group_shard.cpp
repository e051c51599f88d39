// Grouped reduce-scatter and all-gather on the loopback backend (no GPU): the
// segment tables, the grouping conditions and fall-backs, the launch and
// stats accounting, and the MPI_Ireduce_scatter_block / MPI_Iallgather
// bursts.  Reduce-scatter results are compared byte for byte with per-item
// reduceScatter calls (a different host twin with the same fold order);
// all-gather results with a closed form.
#include "fixtures.h"
#include "mpi_group_shard_body.h"

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
struct ShardGroup
{
    std::vector<std::shared_ptr<Communicator>> comms;

    explicit ShardGroup(int n)
    {
        CommConfig cfg;
        cfg.loopback = true;
        cfg.heapBytes = (size_t)32 << 20;
        cfg.stageBytes = (size_t)1 << 20;
        cfg.p2pBounceBytes = (size_t)1 << 20;
        cfg.channels = 2;
        cfg.timeoutMs = 5000;
        cfg.maxBlocks = 4;
        comms = Communicator::createLocal(n, std::vector<int>(n, 0), cfg);
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
                        printf("         rank %d failed\n", r);
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

uint8_t* heapBytes(Communicator& c, size_t n)
{
    return c.heapPtr(c.alloc(std::max<size_t>(n, 16)));
}

void randomBytes(uint8_t* p, size_t n, uint32_t seed)
{
    std::mt19937 g(seed);
    for (size_t i = 0; i < n; i++) {
        p[i] = (uint8_t)g();
    }
}

// Fills `n` elements of `dtype` with values every op is defined on (floats
// are finite, pair indices small)
void randomElems(uint8_t* p, size_t n, int dtype, uint32_t seed)
{
    std::mt19937 g(seed);
    std::uniform_real_distribution<float> u(-4.f, 4.f);
    const size_t es = fbDtypeSize(dtype);
    for (size_t i = 0; i < n; i++) {
        uint8_t* e = p + i * es;
        randomBytes(e, es, seed * 7919u + (uint32_t)i);
        if (dtype == FB_F32) {
            float f = u(g);
            memcpy(e, &f, 4);
        } else if (dtype == FB_BF16) {
            float f = u(g);
            uint32_t b;
            memcpy(&b, &f, 4);
            uint16_t h = (uint16_t)(b >> 16);
            memcpy(e, &h, 2);
        } else if (dtype == FB_F64_I32) {
            double d = (double)(int)(u(g) * 2); // ties on purpose
            int32_t idx = (int32_t)(g() % 1000);
            memcpy(e, &d, 8);
            memcpy(e + 8, &idx, 4);
        } else if (dtype == FB_I32_I32) {
            int32_t v = (int32_t)(g() % 5);
            int32_t idx = (int32_t)(g() % 1000);
            memcpy(e, &v, 4);
            memcpy(e + 4, &idx, 4);
        }
    }
}
}

TEST_CASE("loopback group shard: reduce-scatter equals per-item reduce-scatters, every dtype kind", "[loopback]")
{
    struct Case
    {
        int dtype;
        int op;
    };
    const std::vector<Case> cases = {
        { FB_I32, FB_OP_SUM }, { FB_I32, FB_OP_BXOR }, { FB_U8, FB_OP_MAX },       { FB_I64, FB_OP_PROD },
        { FB_F32, FB_OP_SUM }, { FB_F32, FB_OP_MIN },  { FB_BF16, FB_OP_SUM },     { FB_F64, FB_OP_MAX },
        { FB_F64_I32, FB_OP_MAXLOC },                  { FB_I32_I32, FB_OP_MINLOC },
    };
    // shards in 16-byte vectors: one vector up to several chunks
    const std::vector<size_t> shardVecs = { 1, 3, 64, 129, 700 };
    for (int n : { 1, 2, 3, 4, 5, 8 }) {
        ShardGroup g(n);
        int fails = g.run([&](int rank, Communicator& c) {
            bool ok = true;
            for (const Case& k : cases) {
                const size_t es = fbDtypeSize(k.dtype);
                std::vector<Communicator::GroupItem> items;
                std::vector<uint8_t*> refs;
                for (size_t t = 0; t < shardVecs.size(); t++) {
                    const size_t count = shardVecs[t] * 16 / es;
                    uint8_t* s = heapBytes(c, count * es * n);
                    uint8_t* r = heapBytes(c, count * es);
                    uint8_t* ref = heapBytes(c, count * es);
                    randomElems(s, count * n, k.dtype, 1000u * rank + (uint32_t)t + 17u * k.dtype);
                    memset(r, 0xAB, count * es);
                    items.push_back({ s, r, count });
                    refs.push_back(ref);
                }
                c.hostBarrier();
                const uint64_t l0 = c.stats().launches;
                int rc = FB_OK;
                auto plan = c.prepareGroup(items.data(), items.size(), k.dtype, &rc, Communicator::GROUP_REDUCE_SCATTER);
                ok = ok && plan != nullptr && Communicator::groupPlanLaunches(*plan) == 1;
                ok = ok && c.reduceScatterGroup(*plan, k.op, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
                ok = ok && c.stats().launches == l0 + 1;
                for (size_t t = 0; t < items.size() && ok; t++) {
                    ok = c.reduceScatter(items[t].send, refs[t], items[t].count, k.dtype, k.op, FB_FLAG_SYMMETRIC, nullptr) ==
                           FB_OK &&
                         memcmp(items[t].recv, refs[t], items[t].count * es) == 0;
                }
                // transient table, on channel 1
                c.hostBarrier();
                for (auto& it : items) {
                    memset(it.recv, 0xCD, it.count * es);
                }
                ok = ok && c.reduceScatterMany(items.data(), items.size(), k.dtype, k.op,
                                               FB_FLAG_SYMMETRIC | FB_FLAG_CHANNEL(1), nullptr) == FB_OK;
                for (size_t t = 0; t < items.size() && ok; t++) {
                    ok = memcmp(items[t].recv, refs[t], items[t].count * es) == 0;
                }
                c.hostBarrier();
                if (!ok) {
                    printf("         dtype %d op %d, %d ranks\n", k.dtype, k.op, n);
                    return false;
                }
            }
            return c.checkError(nullptr) == 0;
        });
        REQUIRE_EQ(fails, 0);
    }
}

TEST_CASE("loopback group shard: all-gather with empty items, in place, plan reuse", "[loopback]")
{
    for (int n : { 1, 2, 3, 4, 5, 8 }) {
        ShardGroup g(n);
        int fails = g.run([&](int rank, Communicator& c) {
            // int16 counts: 0 (skipped), one vector, several chunks
            const std::vector<size_t> counts = { 8, 0, 1048, 0, 16, 4096 };
            std::vector<Communicator::GroupItem> items;
            for (size_t cnt : counts) {
                uint8_t* s = heapBytes(c, cnt * 2);
                uint8_t* r = heapBytes(c, cnt * 2 * n + 32);
                items.push_back({ s, r, cnt });
            }
            auto fill = [&](int step) {
                for (size_t t = 0; t < items.size(); t++) {
                    int16_t* s = (int16_t*)items[t].send;
                    for (size_t j = 0; j < items[t].count; j++) {
                        s[j] = (int16_t)(rank * 1000 + t * 100 + j + step * 7);
                    }
                    memset(items[t].recv, 0xEE, items[t].count * 2 * n + 32);
                }
            };
            auto check = [&](int step) {
                for (size_t t = 0; t < items.size(); t++) {
                    const int16_t* r = (const int16_t*)items[t].recv;
                    const size_t cnt = items[t].count;
                    for (size_t i = 0; i < cnt * n; i++) {
                        if (r[i] != (int16_t)((i / cnt) * 1000 + t * 100 + i % cnt + step * 7)) {
                            return false;
                        }
                    }
                    // nothing written past the output
                    const uint8_t* tail = (const uint8_t*)items[t].recv + cnt * 2 * n;
                    for (int b = 0; b < 32; b++) {
                        if (tail[b] != 0xEE) {
                            return false;
                        }
                    }
                }
                return true;
            };
            int rc = FB_OK;
            auto plan = c.prepareGroup(items.data(), items.size(), FB_I16, &rc, Communicator::GROUP_ALLGATHER);
            bool ok = plan != nullptr && Communicator::groupPlanLaunches(*plan) == 1;
            for (int step = 0; step < 3 && ok; step++) {
                fill(step);
                c.hostBarrier();
                const uint64_t l0 = c.stats().launches;
                ok = c.allGatherGroup(*plan, FB_FLAG_SYMMETRIC, nullptr) == FB_OK && c.stats().launches == l0 + 1;
                c.hostBarrier();
                ok = ok && check(step);
            }
            // in place: each send is block `rank` of its own output
            c.hostBarrier();
            std::vector<Communicator::GroupItem> inPlace;
            for (size_t t = 0; t < items.size(); t++) {
                uint8_t* r = (uint8_t*)items[t].recv;
                memset(r, 0xEE, items[t].count * 2 * n + 32);
                int16_t* own = (int16_t*)(r + items[t].count * 2 * rank);
                for (size_t j = 0; j < items[t].count; j++) {
                    own[j] = (int16_t)(rank * 1000 + t * 100 + j + 9 * 7);
                }
                inPlace.push_back({ own, r, items[t].count });
            }
            c.hostBarrier();
            auto ipPlan = c.prepareGroup(inPlace.data(), inPlace.size(), FB_I16, &rc, Communicator::GROUP_ALLGATHER);
            ok = ok && ipPlan != nullptr && c.allGatherGroup(*ipPlan, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            c.hostBarrier();
            ok = ok && check(9);
            // and transient
            c.hostBarrier();
            fill(4);
            c.hostBarrier();
            ok = ok && c.allGatherMany(items.data(), items.size(), FB_I16, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            c.hostBarrier();
            ok = ok && check(4);
            return ok && c.checkError(nullptr) == 0;
        });
        REQUIRE_EQ(fails, 0);
    }
}

TEST_CASE("loopback group shard: more items than one segment table take two launches", "[loopback]")
{
    const int n = 3;
    ShardGroup g(n);
    int fails = g.run([&](int rank, Communicator& c) {
        const size_t k = FB_GROUP_MAX_SEGS - 8 + 100;
        const size_t shard = 4; // int32: one vector
        int32_t* rsIn = (int32_t*)heapBytes(c, k * shard * n * 4);
        int32_t* rsOutBuf = (int32_t*)heapBytes(c, k * shard * 4);
        int32_t* agOut = (int32_t*)heapBytes(c, k * shard * n * 4);
        std::vector<Communicator::GroupItem> rs, ag;
        for (size_t i = 0; i < k; i++) {
            for (size_t j = 0; j < shard * n; j++) {
                rsIn[i * shard * n + j] = (int32_t)(i * 10 + j + rank);
            }
            rs.push_back({ rsIn + i * shard * n, rsOutBuf + i * shard, shard });
            ag.push_back({ rsOutBuf + i * shard, agOut + i * shard * n, shard });
        }
        c.hostBarrier();
        int rc = FB_OK;
        auto rsPlan = c.prepareGroup(rs.data(), rs.size(), FB_I32, &rc, Communicator::GROUP_REDUCE_SCATTER);
        auto agPlan = c.prepareGroup(ag.data(), ag.size(), FB_I32, &rc, Communicator::GROUP_ALLGATHER);
        bool ok = rsPlan != nullptr && agPlan != nullptr && Communicator::groupPlanLaunches(*rsPlan) == 2 &&
                  Communicator::groupPlanLaunches(*agPlan) == 2;
        c.resetStats();
        ok = ok && c.reduceScatterGroup(*rsPlan, FB_OP_SUM, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
        ok = ok && c.stats().launches == 2 && c.stats().bytes == k * shard * n * 4;
        c.hostBarrier();
        ok = ok && c.allGatherGroup(*agPlan, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
        ok = ok && c.stats().launches == 4 && c.stats().bytes == 2 * k * shard * n * 4;
        c.hostBarrier();
        // all-gather of the reduce-scatter: the all-reduce of the inputs
        for (size_t i = 0; i < k && ok; i++) {
            for (size_t j = 0; j < shard * n && ok; j++) {
                ok = agOut[i * shard * n + j] == (int32_t)(n * (i * 10 + j) + n * (n - 1) / 2);
            }
        }
        // the transient calls split the same way
        c.hostBarrier();
        c.resetStats();
        ok = ok && c.reduceScatterMany(rs.data(), rs.size(), FB_I32, FB_OP_SUM, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
        ok = ok && c.allGatherMany(ag.data(), ag.size(), FB_I32, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
        ok = ok && c.stats().launches == 4;
        return ok && c.checkError(nullptr) == 0;
    });
    REQUIRE_EQ(fails, 0);
}

TEST_CASE("loopback group shard: lists that cannot be grouped are refused, *Many falls back", "[loopback]")
{
    for (int n : { 2, 4 }) {
        ShardGroup g(n);
        int fails = g.run([&](int rank, Communicator& c) {
            const int RS = Communicator::GROUP_REDUCE_SCATTER;
            const int AG = Communicator::GROUP_ALLGATHER;
            auto prep = [&](const Communicator::GroupItem& it, int kind) {
                int rc = FB_OK;
                auto p = c.prepareGroup(&it, 1, FB_I32, &rc, (Communicator::GroupKind)kind);
                return p == nullptr ? rc : FB_OK;
            };
            int32_t* a = (int32_t*)heapBytes(c, 64 * n * 4 + 64);
            int32_t* b = (int32_t*)heapBytes(c, 64 * n * 4 + 64);
            std::vector<int32_t> host(64 * n);
            bool ok = true;
            // outside the heap
            ok = ok && prep({ host.data(), b, 16 }, RS) == FB_E_INVALID;
            ok = ok && prep({ a, host.data(), 16 }, AG) == FB_E_INVALID;
            // not 16-byte aligned
            ok = ok && prep({ a + 1, b, 16 }, RS) == FB_E_INVALID;
            ok = ok && prep({ a, b + 2, 16 }, AG) == FB_E_INVALID;
            // a shard that is not a whole number of vectors
            ok = ok && prep({ a, b, 6 }, RS) == FB_E_INVALID;
            ok = ok && prep({ a, b, 6 }, AG) == FB_E_INVALID;
            // an output over an input the peers (or the kernel) read
            ok = ok && prep({ a, a, 16 }, RS) == FB_E_INVALID;
            ok = ok && prep({ a + 16 * ((rank + 1) % n), a, 16 }, AG) == FB_E_INVALID;
            {
                Communicator::GroupItem two[2] = { { a, b, 16 }, { b + 16 * n, a + 16, 16 } };
                int rc = FB_OK;
                ok = ok && c.prepareGroup(two, 2, FB_I32, &rc, Communicator::GROUP_REDUCE_SCATTER) == nullptr &&
                     rc == FB_E_INVALID;
            }
            // ... but in place is an all-gather's own business
            ok = ok && prep({ a + 16 * rank, a, 16 }, AG) == FB_OK;
            // the wrong plan kind, and a pair without a kernel
            int rc = FB_OK;
            Communicator::GroupItem good{ a, b + 64 * n, 16 };
            Communicator::GroupItem goodAg{ a, b, 16 };
            auto rsPlan = c.prepareGroup(&good, 1, FB_I32, &rc, Communicator::GROUP_REDUCE_SCATTER);
            auto agPlan = c.prepareGroup(&goodAg, 1, FB_I32, &rc, Communicator::GROUP_ALLGATHER);
            auto arPlan = c.prepareGroup(&goodAg, 1, FB_I32, &rc);
            ok = ok && rsPlan && agPlan && arPlan;
            ok = ok && c.allReduceGroup(*rsPlan, FB_OP_SUM, FB_FLAG_SYMMETRIC, nullptr) == FB_E_INVALID;
            ok = ok && c.reduceScatterGroup(*agPlan, FB_OP_SUM, FB_FLAG_SYMMETRIC, nullptr) == FB_E_INVALID;
            ok = ok && c.reduceScatterGroup(*arPlan, FB_OP_SUM, FB_FLAG_SYMMETRIC, nullptr) == FB_E_INVALID;
            ok = ok && c.allGatherGroup(*rsPlan, FB_FLAG_SYMMETRIC, nullptr) == FB_E_INVALID;
            ok = ok && c.allGatherGroup(*arPlan, FB_FLAG_SYMMETRIC, nullptr) == FB_E_INVALID;
            {
                auto fPlan = c.prepareGroup(&good, 1, FB_F32, &rc, Communicator::GROUP_REDUCE_SCATTER);
                ok = ok && fPlan && c.reduceScatterGroup(*fPlan, FB_OP_BAND, FB_FLAG_SYMMETRIC, nullptr) == FB_E_UNSUPPORTED;
                ok = ok && c.reduceScatterMany(&good, 1, FB_F32, FB_OP_BAND, FB_FLAG_SYMMETRIC, nullptr) == FB_E_UNSUPPORTED;
            }
            // *Many runs what cannot be grouped as per-item calls, with their
            // results: an output over its own input (reduce-scatter) ...
            c.hostBarrier();
            const size_t cnt = 8;
            for (size_t i = 0; i < cnt * n; i++) {
                a[i] = (int32_t)(i * 3 + rank);
            }
            c.hostBarrier();
            Communicator::GroupItem rsOver{ a, a, cnt };
            ok = ok && c.reduceScatterMany(&rsOver, 1, FB_I32, FB_OP_SUM, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            c.hostBarrier();
            for (size_t j = 0; j < cnt && ok; j++) {
                ok = a[j] == (int32_t)(n * (rank * cnt + j) * 3 + n * (n - 1) / 2);
            }
            // ... host memory (reduce-scatter) ...
            std::vector<int32_t> hs(cnt * n), hr(cnt);
            for (size_t i = 0; i < cnt * n; i++) {
                hs[i] = (int32_t)(i + rank);
            }
            Communicator::GroupItem hostItem{ hs.data(), hr.data(), cnt };
            c.hostBarrier();
            ok = ok && c.reduceScatterMany(&hostItem, 1, FB_I32, FB_OP_SUM, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            for (size_t j = 0; j < cnt && ok; j++) {
                ok = hr[j] == (int32_t)(n * (rank * cnt + j) + n * (n - 1) / 2);
            }
            // ... and shards of 24 bytes (all-gather).  A reduce-scatter of
            // such shards is refused like the per-item call refuses it.
            const size_t odd = 6;
            int32_t* gIn = (int32_t*)heapBytes(c, odd * 4);
            int32_t* gOut = (int32_t*)heapBytes(c, odd * n * 4);
            for (size_t j = 0; j < odd; j++) {
                gIn[j] = (int32_t)(rank * 100 + j);
            }
            Communicator::GroupItem agOdd{ gIn, gOut, odd };
            c.hostBarrier();
            ok = ok && c.allGatherMany(&agOdd, 1, FB_I32, FB_FLAG_SYMMETRIC, nullptr) == FB_OK;
            c.hostBarrier();
            for (size_t i = 0; i < odd * n && ok; i++) {
                ok = gOut[i] == (int32_t)((i / odd) * 100 + i % odd);
            }
            Communicator::GroupItem rsOdd{ b, b + 64 * n, odd };
            ok = ok && c.reduceScatterMany(&rsOdd, 1, FB_I32, FB_OP_SUM, FB_FLAG_SYMMETRIC, nullptr) == FB_E_UNSUPPORTED &&
                 c.reduceScatter(b, b + 64 * n, odd, FB_I32, FB_OP_SUM, FB_FLAG_SYMMETRIC, nullptr) == FB_E_UNSUPPORTED;
            return ok && c.checkError(nullptr) == 0;
        });
        REQUIRE_EQ(fails, 0);
    }
}

TEST_CASE("loopback group shard: every grouped shard call is refused on a sub-communicator", "[loopback]")
{
    ShardGroup g(4);
    int fails = g.run([&](int rank, Communicator& c) {
        int32_t* a = (int32_t*)heapBytes(c, 1024);
        int32_t* b = (int32_t*)heapBytes(c, 1024);
        c.hostBarrier();
        auto child = c.subset({ 0, 1, 2, 3 }, 0);
        bool ok = child != nullptr;
        Communicator::GroupItem it{ a, b, 16 };
        int rc = FB_OK;
        ok = ok && child->prepareGroup(&it, 1, FB_I32, &rc, Communicator::GROUP_REDUCE_SCATTER) == nullptr &&
             rc == FB_E_UNSUPPORTED;
        ok = ok && child->prepareGroup(&it, 1, FB_I32, &rc, Communicator::GROUP_ALLGATHER) == nullptr &&
             rc == FB_E_UNSUPPORTED;
        auto rsPlan = c.prepareGroup(&it, 1, FB_I32, &rc, Communicator::GROUP_REDUCE_SCATTER);
        Communicator::GroupItem agIt{ a, b, 4 };
        auto agPlan = c.prepareGroup(&agIt, 1, FB_I32, &rc, Communicator::GROUP_ALLGATHER);
        ok = ok && rsPlan && agPlan;
        ok = ok && child->reduceScatterGroup(*rsPlan, FB_OP_SUM, FB_FLAG_SYMMETRIC, nullptr) == FB_E_UNSUPPORTED;
        ok = ok && child->allGatherGroup(*agPlan, FB_FLAG_SYMMETRIC, nullptr) == FB_E_UNSUPPORTED;
        ok = ok && child->reduceScatterMany(&it, 1, FB_I32, FB_OP_SUM, FB_FLAG_SYMMETRIC, nullptr) == FB_E_UNSUPPORTED;
        ok = ok && child->allGatherMany(&agIt, 1, FB_I32, FB_FLAG_SYMMETRIC, nullptr) == FB_E_UNSUPPORTED;
        child.reset();
        return ok;
    });
    REQUIRE_EQ(fails, 0);
}

namespace {
void runGroupShardMpi(const std::string& name, int worldSize)
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
        int rc = group_shard::body(rank, size, msg.mpiworldid(), &why);
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

TEST_CASE("loopback group shard: MPI_Ireduce_scatter_block and MPI_Iallgather bursts", "[loopback][mpi]")
{
    tests::LoopbackBackend loopback;
    runGroupShardMpi("group-shard-loopback-4", 4);
    runGroupShardMpi("group-shard-loopback-3", 3);
}
