// Grouped reduce (Communicator::runGroup / groupMany, GROUP_REDUCE) on the
// loopback backend (no GPU): every byte of every rank's buffers, guard bytes
// included, against a fold in rank order computed on the host at 1-8 ranks,
// every root, in place and not, items larger than the staging buffer; launch
// counts; the one-member copy; the refusals; and the MPI program of
// mpi_group_reduce_body.h.
#include "fixtures.h"
#include "mpi_group_reduce_run.h"

#include <faabric/device/communicator.h>

#include <atomic>
#include <cstring>
#include <functional>
#include <random>
#include <thread>
#include <type_traits>

using faabric::device::CommConfig;
using faabric::device::Communicator;

namespace {
const size_t STAGE = (size_t)1 << 20;

std::vector<std::shared_ptr<Communicator>> reduceGroup(int n, size_t stage = STAGE)
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

// The (dtype, op) pairs checked here, each with its own host fold
enum class Fold
{
    I32Sum,
    F32Max,
    U8Bxor,
    F64Sum
};

int dtypeOf(Fold f)
{
    return f == Fold::I32Sum ? FB_I32 : f == Fold::F32Max ? FB_F32 : f == Fold::U8Bxor ? FB_U8 : FB_F64;
}

int opOf(Fold f)
{
    return f == Fold::F32Max ? FB_OP_MAX : f == Fold::U8Bxor ? FB_OP_BXOR : FB_OP_SUM;
}

template<typename E>
void foldInto(uint8_t* acc, const uint8_t* in, size_t count, Fold f)
{
    for (size_t e = 0; e < count; e++) {
        E a, b;
        memcpy(&a, acc + e * sizeof(E), sizeof(E));
        memcpy(&b, in + e * sizeof(E), sizeof(E));
        if constexpr (std::is_same_v<E, uint8_t>) {
            a = (E)(a ^ b);
        } else if constexpr (std::is_same_v<E, int32_t>) {
            a = (E)((uint32_t)a + (uint32_t)b);
        } else if (f == Fold::F32Max) {
            a = b > a ? b : a;
        } else {
            a = a + b;
        }
        memcpy(acc + e * sizeof(E), &a, sizeof(E));
    }
}

void fold(uint8_t* acc, const uint8_t* in, size_t count, Fold f)
{
    switch (f) {
        case Fold::I32Sum:
            foldInto<int32_t>(acc, in, count, f);
            break;
        case Fold::F32Max:
            foldInto<float>(acc, in, count, f);
            break;
        case Fold::U8Bxor:
            foldInto<uint8_t>(acc, in, count, f);
            break;
        case Fold::F64Sum:
            foldInto<double>(acc, in, count, f);
            break;
    }
}

// Every rank's items in one host buffer (plain memory: the user side of the
// rooted kinds is any memory), a guard before each, offsets off 16-byte
// alignment by `shift`.  Floats are small integers (no NaN, exact sums).
struct ReduceCase
{
    Fold f;
    size_t esize;
    int n;
    int root;
    bool inPlace;
    std::vector<size_t> counts;
    std::vector<std::vector<uint8_t>> buf, want;
    std::vector<size_t> sendOff, recvOff;

    ReduceCase(Fold fo, int nranks, int r, bool ip, std::vector<size_t> cnt, size_t shift, std::mt19937& rng)
      : f(fo)
      , esize(fbDtypeSize(dtypeOf(fo)))
      , n(nranks)
      , root(r)
      , inPlace(ip)
      , counts(std::move(cnt))
      , buf(nranks)
    {
        size_t pos = 32 + shift;
        for (size_t c : counts) {
            const size_t b = c * esize;
            sendOff.push_back(pos);
            recvOff.push_back(inPlace ? pos : (pos + b + 15) / 16 * 16 + 32 + shift);
            pos = (recvOff.back() + b + 15) / 16 * 16 + 32 + shift;
        }
        for (auto& v : buf) {
            v.resize(pos + 32);
            for (auto& x : v) {
                x = (uint8_t)rng();
            }
            for (size_t i = 0; i < counts.size(); i++) {
                for (size_t e = 0; e < counts[i]; e++) {
                    uint8_t* p = &v[sendOff[i] + e * esize];
                    if (f == Fold::F32Max) {
                        const float x = (float)(rng() % 2001) - 1000.0f;
                        memcpy(p, &x, 4);
                    } else if (f == Fold::F64Sum) {
                        const double x = (double)(rng() % 2001) - 1000.0;
                        memcpy(p, &x, 8);
                    }
                }
            }
        }
        want = buf;
        for (size_t i = 0; i < counts.size(); i++) {
            const size_t b = counts[i] * esize;
            std::vector<uint8_t> acc(buf[0].begin() + sendOff[i], buf[0].begin() + sendOff[i] + b);
            for (int p = 1; p < n; p++) {
                fold(acc.data(), &buf[p][sendOff[i]], counts[i], f);
            }
            if (b > 0) {
                memcpy(&want[root][recvOff[i]], acc.data(), b);
            }
        }
    }

    // rank p's items: recv is null off the root
    std::vector<Communicator::GroupItem> items(int p)
    {
        std::vector<Communicator::GroupItem> out;
        for (size_t i = 0; i < counts.size(); i++) {
            Communicator::GroupItem it;
            it.send = &buf[p][sendOff[i]];
            it.recv = p == root ? &buf[p][recvOff[i]] : nullptr;
            it.count = counts[i];
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

TEST_CASE("loopback group reduce: every byte at 1-8 ranks, every root, in place, pieces", "[loopback]")
{
    std::mt19937 rng(42);
    const Fold folds[] = { Fold::I32Sum, Fold::F32Max, Fold::U8Bxor, Fold::F64Sum };
    for (int n = 1; n <= 8; n++) {
        auto comms = reduceGroup(n);
        for (int root = 0; root < n; root++) {
            const Fold f = folds[(root + n) % 4];
            const bool inPlace = root % 2 == 1;
            const bool many = (root + n) % 2 == 0;
            // one element, zero, odd, ragged chunk ends, and more than the
            // staging buffer (cut into pieces over several launches)
            const size_t es = fbDtypeSize(dtypeOf(f));
            ReduceCase c(f, n, root, inPlace, { 1, 0, 5, 2049 / es + 1, 300000 / es, (3 * STAGE + 17) / es }, root % 3,
                         rng);
            uint64_t chunks = 0;
            for (size_t k : c.counts) {
                chunks += (k * es + chunkBytes(n) - 1) / chunkBytes(n);
            }
            const uint64_t room = STAGE / chunkBytes(n);
            const uint64_t launches = (chunks + room - 1) / room;
            std::vector<uint64_t> got(n);
            const int fails = runRanks(n, [&](int p) {
                auto& comm = *comms[p];
                auto items = c.items(p);
                int rc = FB_OK;
                auto plan = comm.prepareGroup(items.data(), items.size(), dtypeOf(f), &rc, Communicator::GROUP_REDUCE);
                if (!plan || Communicator::groupPlanLaunches(*plan) != launches) {
                    return false;
                }
                const uint64_t before = comm.stats().launches;
                rc = many ? comm.groupMany(
                              Communicator::GROUP_REDUCE, items.data(), items.size(), dtypeOf(f), opOf(f), root, 0, nullptr)
                          : comm.runGroup(Communicator::GROUP_REDUCE, *plan, opOf(f), root, 0, nullptr);
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

TEST_CASE("loopback group reduce: 1016 items take one launch, 1017 two", "[loopback]")
{
    std::mt19937 rng(7);
    // (every item takes a whole 2 KiB chunk of staging: 1016 of them fit 4 MiB)
    auto comms = reduceGroup(3, (size_t)4 << 20);
    for (size_t k : { (size_t)1016, (size_t)1017 }) {
        ReduceCase c(Fold::I32Sum, 3, 2, false, std::vector<size_t>(k, 3), 1, rng);
        const int fails = runRanks(3, [&](int p) {
            auto items = c.items(p);
            const uint64_t before = comms[p]->stats().launches;
            const int rc =
              comms[p]->groupMany(Communicator::GROUP_REDUCE, items.data(), k, FB_I32, FB_OP_SUM, 2, 0, nullptr);
            return rc == FB_OK && comms[p]->stats().launches - before == (k == 1016 ? 1u : 2u);
        });
        REQUIRE(fails == 0);
        for (int p = 0; p < 3; p++) {
            REQUIRE(c.buf[p] == c.want[p]);
        }
    }
}

TEST_CASE("loopback group reduce: refusals", "[loopback]")
{
    std::mt19937 rng(9);
    auto comms = reduceGroup(2);
    ReduceCase c(Fold::F32Max, 2, 0, false, { 16, 25 }, 0, rng);
    auto items = c.items(0);
    int rc = FB_OK;
    auto plan = comms[0]->prepareGroup(items.data(), items.size(), FB_F32, &rc, Communicator::GROUP_REDUCE);
    REQUIRE(plan != nullptr);
    auto gather = comms[0]->prepareGroup(items.data(), items.size(), FB_U8, &rc, Communicator::GROUP_GATHER);
    REQUIRE(gather != nullptr);
    const uint64_t before = comms[0]->stats().launches;
    const uint64_t before1 = comms[1]->stats().launches;
    // nothing is launched: no peer is left at a barrier
    REQUIRE(comms[0]->runGroup(Communicator::GROUP_REDUCE, *gather, FB_OP_SUM, 0, 0, nullptr) == FB_E_INVALID);
    REQUIRE(comms[0]->runGroup(Communicator::GROUP_GATHER, *plan, 0, 0, 0, nullptr) == FB_E_INVALID);
    REQUIRE(comms[0]->runGroup(Communicator::GROUP_REDUCE, *plan, FB_OP_BAND, 0, 0, nullptr) == FB_E_UNSUPPORTED);
    REQUIRE(comms[0]->runGroup(Communicator::GROUP_REDUCE, *plan, FB_OP_SUM, 2, 0, nullptr) == FB_E_INVALID);
    REQUIRE(comms[0]->runGroup(Communicator::GROUP_REDUCE, *plan, FB_OP_SUM, -1, 0, nullptr) == FB_E_INVALID);
    REQUIRE(comms[0]->runGroup(Communicator::GROUP_REDUCE, *plan, FB_OP_SUM, 0, FB_FLAG_CHANNEL(1), nullptr) ==
            FB_E_INVALID);
    REQUIRE(comms[0]->groupMany(Communicator::GROUP_REDUCE, items.data(), items.size(), FB_F32, FB_OP_BXOR, 0, 0,
                                nullptr) == FB_E_UNSUPPORTED);
    REQUIRE(comms[0]->groupMany(Communicator::GROUP_REDUCE, items.data(), items.size(), FB_F32, FB_OP_SUM, 5, 0,
                                nullptr) == FB_E_INVALID);
    REQUIRE(comms[0]->groupMany(Communicator::GROUP_REDUCE, items.data(), items.size(), FB_F32, FB_OP_SUM, 0,
                                FB_FLAG_CHANNEL(2), nullptr) == FB_E_INVALID);
    // the root needs both sides, every rank its send
    items[1].recv = nullptr;
    REQUIRE(comms[0]->groupMany(Communicator::GROUP_REDUCE, items.data(), items.size(), FB_F32, FB_OP_SUM, 0, 0,
                                nullptr) == FB_E_INVALID);
    auto other = c.items(1);
    other[0].send = nullptr;
    REQUIRE(comms[1]->groupMany(Communicator::GROUP_REDUCE, other.data(), other.size(), FB_F32, FB_OP_SUM, 0, 0,
                                nullptr) == FB_E_INVALID);
    auto missing = comms[0]->prepareGroup(items.data(), items.size(), FB_F32, &rc, Communicator::GROUP_REDUCE);
    REQUIRE(missing != nullptr);
    REQUIRE(comms[0]->runGroup(Communicator::GROUP_REDUCE, *missing, FB_OP_SUM, 0, 0, nullptr) == FB_E_INVALID);
    REQUIRE(comms[0]->stats().launches == before);
    REQUIRE(comms[1]->stats().launches == before1);
    REQUIRE(std::string(Communicator::groupKindName(Communicator::GROUP_REDUCE)) == "reduce");
}

TEST_CASE("loopback group reduce: one member copies, or does nothing in place", "[loopback]")
{
    std::mt19937 rng(3);
    auto comms = reduceGroup(1);
    for (bool inPlace : { false, true }) {
        ReduceCase c(Fold::F64Sum, 1, 0, inPlace, { 3, 512, 70001 }, 5, rng);
        auto items = c.items(0);
        const uint64_t before = comms[0]->stats().launches;
        REQUIRE(comms[0]->groupMany(Communicator::GROUP_REDUCE, items.data(), items.size(), FB_F64, FB_OP_SUM, 0, 0,
                                    nullptr) == FB_OK);
        REQUIRE(comms[0]->stats().launches == before + 1);
        REQUIRE(c.buf[0] == c.want[0]);
    }
}

TEST_CASE("loopback group reduce: MPI_Ireduce bursts on the world and on sub-communicators", "[loopback][mpi]")
{
    tests::LoopbackBackend loopback;
    runMpiGroupReduceBody(true);
}
