// Grouped scan and exscan (Communicator::runGroup / groupMany, GROUP_SCAN and
// GROUP_EXSCAN) on the loopback backend (no GPU): every byte of every rank's
// buffers, guard bytes included, against closed forms at 1-8 ranks (3, 5, 6
// and 7 take the kernel's generic NR = 0 path), in place on some ranks and
// not, items larger than the staging buffer; launch counts; one member; the
// refusals; and the MPI program of mpi_group_scan_body.h.
#include "fixtures.h"
#include "mpi_group_scan_run.h"

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

std::vector<std::shared_ptr<Communicator>> scanGroup(int n, size_t stage = STAGE)
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

// Element e of item i on rank p: small integers, so every prefix sum is exact
// in float and double and has a closed form
int64_t value(int p, size_t i, size_t e)
{
    return (int64_t)((p * 7 + i * 3 + e) % 101) - 50;
}

// The ops checked here: sum (closed form below) and max over i32, f32 and
// f64
enum class Fold
{
    I32Sum,
    F32Max,
    F64Sum
};

int dtypeOf(Fold f)
{
    return f == Fold::I32Sum ? FB_I32 : f == Fold::F32Max ? FB_F32 : FB_F64;
}

int opOf(Fold f)
{
    return f == Fold::F32Max ? FB_OP_MAX : FB_OP_SUM;
}

// The fold of element e of item i over ranks [0, k)
double prefix(Fold f, int k, size_t i, size_t e)
{
    double acc = (double)value(0, i, e);
    for (int p = 1; p < k; p++) {
        const double v = (double)value(p, i, e);
        acc = f == Fold::F32Max ? std::max(acc, v) : acc + v;
    }
    return acc;
}

void store(uint8_t* at, Fold f, double v)
{
    if (f == Fold::I32Sum) {
        const int32_t x = (int32_t)v;
        memcpy(at, &x, 4);
    } else if (f == Fold::F32Max) {
        const float x = (float)v;
        memcpy(at, &x, 4);
    } else {
        memcpy(at, &v, 8);
    }
}

// Every rank's items in one host buffer (plain memory: the user side of the
// rooted kinds is any memory), a guard before each, offsets off 16-byte
// alignment by `shift`.  Ranks with bit p of `inPlace` pass each send as its
// recv.
struct ScanCase
{
    Fold f;
    size_t esize;
    int n;
    bool ex;
    std::vector<size_t> counts;
    std::vector<std::vector<uint8_t>> buf, want;
    std::vector<std::vector<size_t>> sendOff, recvOff;

    ScanCase(Fold fo, int nranks, bool exclusive, unsigned inPlace, std::vector<size_t> cnt, size_t shift,
             std::mt19937& rng)
      : f(fo)
      , esize(fbDtypeSize(dtypeOf(fo)))
      , n(nranks)
      , ex(exclusive)
      , counts(std::move(cnt))
      , buf(nranks)
      , sendOff(nranks)
      , recvOff(nranks)
    {
        for (int p = 0; p < n; p++) {
            const bool own = (inPlace >> p) & 1u;
            size_t pos = 32 + shift;
            for (size_t c : counts) {
                const size_t b = c * esize;
                sendOff[p].push_back(pos);
                recvOff[p].push_back(own ? pos : (pos + b + 15) / 16 * 16 + 32 + shift);
                pos = (recvOff[p].back() + b + 15) / 16 * 16 + 32 + shift;
            }
            buf[p].resize(pos + 32);
            for (auto& x : buf[p]) {
                x = (uint8_t)rng();
            }
            for (size_t i = 0; i < counts.size(); i++) {
                for (size_t e = 0; e < counts[i]; e++) {
                    store(&buf[p][sendOff[p][i] + e * esize], f, (double)value(p, i, e));
                }
            }
        }
        want = buf;
        for (int p = 0; p < n; p++) {
            const int k = ex ? p : p + 1;
            for (size_t i = 0; k > 0 && i < counts.size(); i++) {
                for (size_t e = 0; e < counts[i]; e++) {
                    store(&want[p][recvOff[p][i] + e * esize], f, prefix(f, k, i, e));
                }
            }
        }
    }

    std::vector<Communicator::GroupItem> items(int p)
    {
        std::vector<Communicator::GroupItem> out;
        for (size_t i = 0; i < counts.size(); i++) {
            out.push_back({ &buf[p][sendOff[p][i]], &buf[p][recvOff[p][i]], counts[i] });
        }
        return out;
    }
};

uint64_t chunkBytes(int n)
{
    return n == 8 ? 1024 : (n == 1 ? 4096 : 2048);
}

Communicator::GroupKind kindOf(bool ex)
{
    return ex ? Communicator::GROUP_EXSCAN : Communicator::GROUP_SCAN;
}
}

TEST_CASE("loopback group scan: every byte at 1-8 ranks, both kinds, in place on some ranks, pieces", "[loopback]")
{
    std::mt19937 rng(42);
    const Fold folds[] = { Fold::I32Sum, Fold::F32Max, Fold::F64Sum };
    for (int n = 1; n <= 8; n++) {
        auto comms = scanGroup(n);
        for (int round = 0; round < 4; round++) {
            const bool ex = round % 2 == 1;
            const Fold f = folds[(round + n) % 3];
            // in place nowhere, on the odd ranks, on rank 0 only, everywhere
            const unsigned inPlace = std::vector<unsigned>{ 0u, 0xAAu, 1u, 0xFFu }[round];
            const bool many = (round + n) % 2 == 0;
            // one element, zero, odd, ragged chunk ends, and more than the
            // staging buffer (cut into pieces over several launches)
            const size_t es = fbDtypeSize(dtypeOf(f));
            ScanCase c(f, n, ex, inPlace, { 1, 0, 5, 2049 / es + 1, 300000 / es, (3 * STAGE + 17) / es }, round % 3,
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
                auto plan = comm.prepareGroup(items.data(), items.size(), dtypeOf(f), &rc, kindOf(ex));
                if (!plan || Communicator::groupPlanLaunches(*plan) != launches) {
                    return false;
                }
                const uint64_t before = comm.stats().launches;
                // (`root` is ignored: any value)
                rc = many ? comm.groupMany(kindOf(ex), items.data(), items.size(), dtypeOf(f), opOf(f), 99, 0, nullptr)
                          : comm.runGroup(kindOf(ex), *plan, opOf(f), -3, 0, nullptr);
                got[p] = comm.stats().launches - before;
                return rc == FB_OK && comm.peekError() == 0;
            });
            REQUIRE(fails == 0);
            for (int p = 0; p < n; p++) {
                // (a one-member exscan writes nothing and launches nothing)
                REQUIRE(got[p] == (ex && n == 1 ? 0 : launches));
                REQUIRE(c.buf[p] == c.want[p]);
            }
        }
    }
}

TEST_CASE("loopback group scan: 1016 items take one launch, 1017 two", "[loopback]")
{
    std::mt19937 rng(7);
    // (every item takes a whole 2 KiB chunk of staging: 1016 of them fit 4 MiB)
    auto comms = scanGroup(5, (size_t)4 << 20);
    for (size_t k : { (size_t)1016, (size_t)1017 }) {
        ScanCase c(Fold::I32Sum, 5, k == 1017, 0x6u, std::vector<size_t>(k, 3), 1, rng);
        const int fails = runRanks(5, [&](int p) {
            auto items = c.items(p);
            const uint64_t before = comms[p]->stats().launches;
            const int rc = comms[p]->groupMany(kindOf(c.ex), items.data(), k, FB_I32, FB_OP_SUM, 0, 0, nullptr);
            return rc == FB_OK && comms[p]->stats().launches - before == (k == 1016 ? 1u : 2u);
        });
        REQUIRE(fails == 0);
        for (int p = 0; p < 5; p++) {
            REQUIRE(c.buf[p] == c.want[p]);
        }
    }
}

TEST_CASE("loopback group scan: refusals", "[loopback]")
{
    std::mt19937 rng(9);
    auto comms = scanGroup(2);
    for (bool ex : { false, true }) {
        ScanCase c(Fold::F32Max, 2, ex, 0, { 16, 25 }, 0, rng);
        auto items = c.items(0);
        int rc = FB_OK;
        auto plan = comms[0]->prepareGroup(items.data(), items.size(), FB_F32, &rc, kindOf(ex));
        REQUIRE(plan != nullptr);
        auto reduce = comms[0]->prepareGroup(items.data(), items.size(), FB_F32, &rc, Communicator::GROUP_REDUCE);
        REQUIRE(reduce != nullptr);
        const uint64_t before = comms[0]->stats().launches;
        const uint64_t before1 = comms[1]->stats().launches;
        // nothing is launched: no peer is left at a barrier
        REQUIRE(comms[0]->runGroup(kindOf(ex), *reduce, FB_OP_SUM, 0, 0, nullptr) == FB_E_INVALID);
        REQUIRE(comms[0]->runGroup(kindOf(!ex), *plan, FB_OP_SUM, 0, 0, nullptr) == FB_E_INVALID);
        REQUIRE(comms[0]->runGroup(kindOf(ex), *plan, FB_OP_BAND, 0, 0, nullptr) == FB_E_UNSUPPORTED);
        REQUIRE(comms[0]->runGroup(kindOf(ex), *plan, FB_OP_SUM, 0, FB_FLAG_CHANNEL(1), nullptr) == FB_E_INVALID);
        REQUIRE(comms[0]->groupMany(kindOf(ex), items.data(), items.size(), FB_F32, FB_OP_BXOR, 0, 0, nullptr) ==
                FB_E_UNSUPPORTED);
        REQUIRE(comms[0]->groupMany(kindOf(ex), items.data(), items.size(), FB_F32, FB_OP_SUM, 0, FB_FLAG_CHANNEL(2),
                                    nullptr) == FB_E_INVALID);
        // every rank needs both sides
        for (int side = 0; side < 2; side++) {
            auto missing = c.items(side);
            if (side == 0) {
                missing[1].recv = nullptr;
            } else {
                missing[0].send = nullptr;
            }
            REQUIRE(comms[side]->groupMany(kindOf(ex), missing.data(), missing.size(), FB_F32, FB_OP_SUM, 0, 0,
                                           nullptr) == FB_E_INVALID);
            auto mplan = comms[side]->prepareGroup(missing.data(), missing.size(), FB_F32, &rc, kindOf(ex));
            REQUIRE(mplan != nullptr);
            REQUIRE(comms[side]->runGroup(kindOf(ex), *mplan, FB_OP_SUM, 0, 0, nullptr) == FB_E_INVALID);
        }
        REQUIRE(comms[0]->stats().launches == before);
        REQUIRE(comms[1]->stats().launches == before1);
    }
    REQUIRE(std::string(Communicator::groupKindName(Communicator::GROUP_SCAN)) == "scan");
    REQUIRE(std::string(Communicator::groupKindName(Communicator::GROUP_EXSCAN)) == "exscan");
}

TEST_CASE("loopback group scan: MPI_Iscan and MPI_Iexscan bursts on the world and on sub-communicators",
          "[loopback][mpi]")
{
    tests::LoopbackBackend loopback;
    runMpiGroupScanBody(true);
}
