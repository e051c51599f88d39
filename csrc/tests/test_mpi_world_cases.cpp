// MpiWorld driven directly (no planner-scheduled functions): one case per case
// of the reference's world tests, all ranks on this host
// (reference: tests/test/mpi/test_mpi_world.cpp:30-1500, test_mpi_message.cpp,
// test_mpi_context.cpp, test_multiple_mpi_worlds.cpp)
#include "fixtures.h"

#include <faabric/batch-scheduler/SchedulingDecision.h>
#include <faabric/mpi/MpiContext.h>
#include <faabric/mpi/MpiMessage.h>
#include <faabric/mpi/MpiWorld.h>
#include <faabric/mpi/MpiWorldRegistry.h>
#include <faabric/mpi/mpi.h>
#include <faabric/transport/PointToPointBroker.h>
#include <faabric/util/gids.h>

#include <cmath>
#include <cstring>
#include <limits>
#include <numeric>
#include <thread>

using namespace tests;
using namespace faabric::mpi;

namespace {
// A world of `size` ranks, all on this host, set up the way the planner would
struct LocalWorld
{
    int worldId;
    int size;
    faabric::Message msg = faabric::util::messageFactory("mpi", "hellompi");
    MpiWorld world;

    explicit LocalWorld(int sizeIn = 5, int worldIdIn = 123)
      : worldId(worldIdIn)
      , size(sizeIn)
    {
        faabric::util::setMockMode(false);
        msg.set_ismpi(true);
        msg.set_mpiworldid(worldId);
        msg.set_mpiworldsize(size);
        msg.set_groupid(faabric::util::generateGid() % 100000 + 1000);
        faabric::batch_scheduler::SchedulingDecision decision(msg.appid(), msg.groupid());
        std::string thisHost = faabric::util::getSystemConfig().endpointHost;
        for (int r = 0; r < size; r++) {
            decision.addMessage(thisHost, msg.id() + r, r, r);
        }
        faabric::transport::getPointToPointBroker().setUpLocalMappingsFromSchedulingDecision(decision);
        world.initialiseFromMsg(msg);
    }

    ~LocalWorld()
    {
        world.destroy();
        faabric::transport::getPointToPointBroker().clear();
    }
};

template<typename T>
std::vector<T> recvVec(MpiWorld& w, int from, int to, faabric_datatype_t* type, int count, MPI_Status* status = nullptr)
{
    std::vector<T> out((size_t)std::max(count, 0), T{});
    w.recv(from, to, BYTES(out.data()), type, count, status);
    return out;
}
}

TEST_CASE("mpi world case: creation sets id, size, user and function", "[mpi][world][cases]")
{
    LocalWorld f(10);
    REQUIRE_EQ(f.world.getSize(), 10);
    REQUIRE_EQ(f.world.getId(), 123);
    REQUIRE_EQ(f.world.getUser(), std::string("mpi"));
    REQUIRE_EQ(f.world.getFunction(), std::string("hellompi"));
    std::string thisHost = faabric::util::getSystemConfig().endpointHost;
    for (int r = 0; r < 10; r++) {
        REQUIRE_EQ(f.world.getHostForRank(r), thisHost);
    }
    REQUIRE_THROWS(f.world.getHostForRank(10));
}

TEST_CASE("mpi world case: a world of one rank", "[mpi][world][cases]")
{
    LocalWorld f(1);
    REQUIRE_EQ(f.world.getSize(), 1);
    // collectives degenerate to copies
    std::vector<int> v = { 4, 5, 6 }, out(3, 0);
    f.world.allReduce(0, BYTES(v.data()), BYTES(out.data()), MPI_INT, 3, MPI_SUM);
    REQUIRE(out == v);
    f.world.barrier(0);
}

TEST_CASE("mpi world case: send and recv between two ranks of one host, with and without data", "[mpi][world][cases]")
{
    LocalWorld f;
    for (std::vector<int> data : { std::vector<int>{ 0, 1, 2 }, std::vector<int>{} }) {
        f.world.send(0, 1, BYTES(data.data()), MPI_INT, (int)data.size());
        MPI_Status status{};
        auto got = recvVec<int>(f.world, 0, 1, MPI_INT, (int)data.size(), &status);
        REQUIRE(got == data);
        REQUIRE_EQ(status.MPI_ERROR, MPI_SUCCESS);
        REQUIRE_EQ(status.MPI_SOURCE, 0);
        REQUIRE_EQ(status.bytesSize, (int)(data.size() * sizeof(int)));
    }
}

TEST_CASE("mpi world case: sendrecv between two ranks", "[mpi][world][cases]")
{
    LocalWorld f;
    std::vector<int> a = { 0, 1, 2 }, b = { 3, 2, 1, 0 };
    std::vector<int> gotByA(b.size()), gotByB(a.size());
    MPI_Status sa{}, sb{};
    std::thread other([&] {
        f.world.sendRecv(BYTES(b.data()), (int)b.size(), MPI_INT, 1, BYTES(gotByB.data()), (int)a.size(), MPI_INT, 1, 2, &sb);
    });
    f.world.sendRecv(BYTES(a.data()), (int)a.size(), MPI_INT, 2, BYTES(gotByA.data()), (int)b.size(), MPI_INT, 2, 1, &sa);
    other.join();
    REQUIRE(gotByA == b);
    REQUIRE(gotByB == a);
    REQUIRE_EQ(sa.MPI_SOURCE, 2);
    REQUIRE_EQ(sb.MPI_SOURCE, 1);
}

TEST_CASE("mpi world case: a ring of sendrecvs", "[mpi][world][cases]")
{
    LocalWorld f(5);
    std::vector<int> fromLeft(5, -1);
    std::vector<std::thread> ranks;
    for (int r = 0; r < 5; r++) {
        ranks.emplace_back([&, r] {
            int right = (r + 1) % 5, left = (r + 4) % 5;
            int mine = r;
            f.world.sendRecv(BYTES(&mine), 1, MPI_INT, right, BYTES(&fromLeft[r]), 1, MPI_INT, left, r, nullptr);
        });
    }
    for (auto& t : ranks) {
        t.join();
    }
    for (int r = 0; r < 5; r++) {
        REQUIRE_EQ(fromLeft[r], (r + 4) % 5);
    }
}

TEST_CASE("mpi world case: asynchronous sends and receives complete in any await order", "[mpi][world][cases]")
{
    LocalWorld f;
    std::vector<int> a = { 0, 1, 2 }, b = { 3, 4, 5, 6 };
    int sendA = f.world.isend(0, 1, BYTES(a.data()), MPI_INT, 3);
    int sendB = f.world.isend(2, 1, BYTES(b.data()), MPI_INT, 4);
    std::vector<int> gotA(3), gotB(4);
    int recvB = f.world.irecv(2, 1, BYTES(gotB.data()), MPI_INT, 4);
    int recvA = f.world.irecv(0, 1, BYTES(gotA.data()), MPI_INT, 3);
    // out of order on purpose
    f.world.awaitAsyncRequest(recvA);
    f.world.awaitAsyncRequest(sendB);
    f.world.awaitAsyncRequest(recvB);
    f.world.awaitAsyncRequest(sendA);
    REQUIRE(gotA == a);
    REQUIRE(gotB == b);
}

TEST_CASE("mpi world case: a message with no data still carries its metadata", "[mpi][world][cases]")
{
    LocalWorld f;
    f.world.send(1, 2, nullptr, MPI_INT, 0);
    MPI_Status status{};
    f.world.recv(1, 2, nullptr, MPI_INT, 0, &status);
    REQUIRE_EQ(status.MPI_SOURCE, 1);
    REQUIRE_EQ(status.MPI_ERROR, MPI_SUCCESS);
    REQUIRE_EQ(status.bytesSize, 0);
}

TEST_CASE("mpi world case: receiving into a bigger buffer reports the size that arrived", "[mpi][world][cases]")
{
    LocalWorld f;
    std::vector<int> data = { 7, 8, 9 };
    f.world.send(1, 2, BYTES(data.data()), MPI_INT, 3);
    std::vector<int> buf(10, -1);
    MPI_Status status{};
    f.world.recv(1, 2, BYTES(buf.data()), MPI_INT, 10, &status);
    REQUIRE(buf[0] == 7 && buf[1] == 8 && buf[2] == 9 && buf[3] == -1);
    REQUIRE_EQ(status.bytesSize, (int)(3 * sizeof(int)));
    int count = -1;
    MPI_Get_count(&status, MPI_INT, &count);
    REQUIRE_EQ(count, 3);
}

TEST_CASE("mpi world case: probe reports the next message without consuming it", "[mpi][world][cases]")
{
    LocalWorld f;
    std::vector<int> first = { 1, 2, 3, 4 }, second = { 5, 6 };
    f.world.send(1, 2, BYTES(first.data()), MPI_INT, 4);
    f.world.send(1, 2, BYTES(second.data()), MPI_INT, 2);
    MPI_Status p{};
    f.world.probe(1, 2, &p);
    REQUIRE_EQ(p.bytesSize, (int)(4 * sizeof(int)));
    REQUIRE_EQ(p.MPI_SOURCE, 1);
    // probing again sees the same message
    f.world.probe(1, 2, &p);
    REQUIRE_EQ(p.bytesSize, (int)(4 * sizeof(int)));
    REQUIRE(recvVec<int>(f.world, 1, 2, MPI_INT, 4) == first);
    f.world.probe(1, 2, &p);
    REQUIRE_EQ(p.bytesSize, (int)(2 * sizeof(int)));
    REQUIRE(recvVec<int>(f.world, 1, 2, MPI_INT, 2) == second);
}

TEST_CASE("mpi world case: ranks outside the world are refused", "[mpi][world][cases]")
{
    LocalWorld f(3);
    int v = 1;
    REQUIRE_THROWS(f.world.send(0, 3, BYTES(&v), MPI_INT, 1));
    REQUIRE_THROWS(f.world.send(-1, 1, BYTES(&v), MPI_INT, 1));
    REQUIRE_THROWS(f.world.recv(0, 5, BYTES(&v), MPI_INT, 1, nullptr));
    REQUIRE_THROWS(f.world.isend(7, 0, BYTES(&v), MPI_INT, 1));
}

TEST_CASE("mpi world case: a world can be destroyed with requests outstanding", "[mpi][world][cases]")
{
    LocalWorld f(2);
    int v = 3, sink = 0;
    f.world.isend(0, 1, BYTES(&v), MPI_INT, 1);
    f.world.irecv(1, 0, BYTES(&sink), MPI_INT, 1); // never satisfied
    // the fixture's destructor destroys the world: nothing must hang or throw
}

namespace {
// Runs `body(rank)` on one thread per rank of the world
void onEveryRank(LocalWorld& f, const std::function<void(int)>& body)
{
    std::vector<std::thread> ranks;
    std::atomic<int> failures{ 0 };
    for (int r = 0; r < f.size; r++) {
        ranks.emplace_back([&, r] {
            try {
                body(r);
            } catch (const std::exception& e) {
                printf("         rank %d threw: %s\n", r, e.what());
                failures++;
            }
        });
    }
    for (auto& t : ranks) {
        t.join();
    }
    REQUIRE_EQ(failures.load(), 0);
}
}

TEST_CASE("mpi world case: a local barrier holds every rank until the last one arrives", "[mpi][world][cases]")
{
    LocalWorld f(4);
    std::atomic<int> arrived{ 0 };
    std::atomic<bool> early{ false };
    onEveryRank(f, [&](int r) {
        if (r == 3) {
            std::this_thread::sleep_for(std::chrono::milliseconds(50));
        }
        arrived++;
        f.world.barrier(r);
        if (arrived.load() != 4) {
            early = true;
        }
    });
    REQUIRE(!early.load());
}

TEST_CASE("mpi world case: broadcast from every possible root", "[mpi][world][cases]")
{
    LocalWorld f(5);
    for (int root = 0; root < 5; root++) {
        std::vector<std::vector<int>> bufs(5, std::vector<int>(3, -1));
        bufs[root] = { root, 10 + root, 20 + root };
        onEveryRank(f, [&](int r) { f.world.broadcast(root, r, BYTES(bufs[r].data()), MPI_INT, 3); });
        for (int r = 0; r < 5; r++) {
            REQUIRE(bufs[r] == (std::vector<int>{ root, 10 + root, 20 + root }));
        }
    }
}

TEST_CASE("mpi world case: scatter, gather and allgather", "[mpi][world][cases]")
{
    LocalWorld f(4);
    const int per = 3, root = 2;
    std::vector<int> all(4 * per);
    std::iota(all.begin(), all.end(), 100);
    std::vector<std::vector<int>> mine(4, std::vector<int>(per, -1));
    onEveryRank(f, [&](int r) {
        f.world.scatter(root, r, BYTES(all.data()), MPI_INT, per, BYTES(mine[r].data()), MPI_INT, per);
    });
    for (int r = 0; r < 4; r++) {
        REQUIRE(mine[r] == std::vector<int>(all.begin() + r * per, all.begin() + (r + 1) * per));
    }
    // gather puts them back together on the root
    std::vector<int> gathered(4 * per, -1);
    onEveryRank(f, [&](int r) {
        f.world.gather(r, root, BYTES(mine[r].data()), MPI_INT, per, r == root ? BYTES(gathered.data()) : nullptr, MPI_INT, per);
    });
    REQUIRE(gathered == all);
    // allgather gives everyone the whole thing
    std::vector<std::vector<int>> everyone(4, std::vector<int>(4 * per, -1));
    onEveryRank(f, [&](int r) {
        f.world.allGather(r, BYTES(mine[r].data()), MPI_INT, per, BYTES(everyone[r].data()), MPI_INT, per);
    });
    for (int r = 0; r < 4; r++) {
        REQUIRE(everyone[r] == all);
    }
}

TEST_CASE("mpi world case: reduce to a root and all-reduce, sums of ints", "[mpi][world][cases]")
{
    LocalWorld f(5);
    const int root = 3, n = 4;
    std::vector<std::vector<int>> in(5, std::vector<int>(n));
    std::vector<int> expected(n, 0);
    for (int r = 0; r < 5; r++) {
        for (int i = 0; i < n; i++) {
            in[r][i] = r * 10 + i;
            expected[i] += in[r][i];
        }
    }
    std::vector<int> atRoot(n, -1);
    onEveryRank(f, [&](int r) {
        f.world.reduce(r, root, BYTES(in[r].data()), r == root ? BYTES(atRoot.data()) : nullptr, MPI_INT, n, MPI_SUM);
    });
    REQUIRE(atRoot == expected);
    // the inputs are untouched
    REQUIRE_EQ(in[0][1], 1);
    std::vector<std::vector<int>> out(5, std::vector<int>(n, -1));
    onEveryRank(f, [&](int r) { f.world.allReduce(r, BYTES(in[r].data()), BYTES(out[r].data()), MPI_INT, n, MPI_SUM); });
    for (int r = 0; r < 5; r++) {
        REQUIRE(out[r] == expected);
    }
    // in place on every rank
    auto copy = in;
    onEveryRank(f, [&](int r) { f.world.allReduce(r, BYTES(copy[r].data()), BYTES(copy[r].data()), MPI_INT, n, MPI_SUM); });
    for (int r = 0; r < 5; r++) {
        REQUIRE(copy[r] == expected);
    }
}

TEST_CASE("mpi world case: the reduce operators on ints, doubles and long longs", "[mpi][world][cases]")
{
    LocalWorld f(2);
    auto& w = f.world;
    {
        std::vector<int> in = { 1, 7, -3 }, acc = { 4, 2, -5 };
        std::vector<int> a = acc;
        w.op_reduce(MPI_MAX, MPI_INT, 3, BYTES(in.data()), BYTES(a.data()));
        REQUIRE(a == (std::vector<int>{ 4, 7, -3 }));
        a = acc;
        w.op_reduce(MPI_MIN, MPI_INT, 3, BYTES(in.data()), BYTES(a.data()));
        REQUIRE(a == (std::vector<int>{ 1, 2, -5 }));
        a = acc;
        w.op_reduce(MPI_SUM, MPI_INT, 3, BYTES(in.data()), BYTES(a.data()));
        REQUIRE(a == (std::vector<int>{ 5, 9, -8 }));
        a = acc;
        w.op_reduce(MPI_PROD, MPI_INT, 3, BYTES(in.data()), BYTES(a.data()));
        REQUIRE(a == (std::vector<int>{ 4, 14, 15 }));
    }
    {
        std::vector<double> in = { 1.5, -2.25 }, a = { 0.5, 4.0 };
        w.op_reduce(MPI_SUM, MPI_DOUBLE, 2, BYTES(in.data()), BYTES(a.data()));
        REQUIRE(a == (std::vector<double>{ 2.0, 1.75 }));
        a = { 0.5, 4.0 };
        w.op_reduce(MPI_MAX, MPI_DOUBLE, 2, BYTES(in.data()), BYTES(a.data()));
        REQUIRE(a == (std::vector<double>{ 1.5, 4.0 }));
        a = { 0.5, 4.0 };
        w.op_reduce(MPI_MIN, MPI_DOUBLE, 2, BYTES(in.data()), BYTES(a.data()));
        REQUIRE(a == (std::vector<double>{ 0.5, -2.25 }));
    }
    {
        std::vector<long long> in = { 1LL << 40, -7 }, a = { 1LL << 41, 9 };
        w.op_reduce(MPI_SUM, MPI_LONG_LONG, 2, BYTES(in.data()), BYTES(a.data()));
        REQUIRE(a == (std::vector<long long>{ 3LL << 40, 2 }));
        a = { 1LL << 41, 9 };
        w.op_reduce(MPI_MAX, MPI_LONG_LONG, 2, BYTES(in.data()), BYTES(a.data()));
        REQUIRE(a == (std::vector<long long>{ 1LL << 41, 9 }));
        a = { 1LL << 41, 9 };
        w.op_reduce(MPI_MIN, MPI_LONG_LONG, 2, BYTES(in.data()), BYTES(a.data()));
        REQUIRE(a == (std::vector<long long>{ 1LL << 40, -7 }));
    }
}

namespace {
// Position i % 6 of rank r: 0 a NaN on rank 0, 1 a NaN on the last rank, 2 a
// NaN on every rank, 3 -0 on rank 0 (+0 elsewhere), 4 -0 on the last rank,
// 5 no special value; the other entries hold r + 1
template<typename T>
T placed(int r, int n, size_t i)
{
    const T nan = std::numeric_limits<T>::quiet_NaN();
    switch (i % 6) {
        case 0:
            return r == 0 ? nan : (T)(r + 1);
        case 1:
            return r == n - 1 ? nan : (T)(r + 1);
        case 2:
            return nan;
        case 3:
            return r == 0 ? (T)-0.0 : (T)0.0;
        case 4:
            return r == n - 1 ? (T)-0.0 : (T)0.0;
        default:
            return (T)(r + 1);
    }
}

// Closed forms: MAX ignores the NaNs and orders -0 below +0
template<typename T>
bool placedMaxMinOk(const std::vector<T>& got, int n, bool isMax)
{
    for (size_t i = 0; i < got.size(); i++) {
        T g = got[i];
        bool ok;
        switch (i % 6) {
            case 0:
                ok = g == (isMax ? (T)n : (T)2);
                break;
            case 1:
                ok = g == (isMax ? (T)(n - 1) : (T)1);
                break;
            case 2:
                ok = std::isnan(g);
                break;
            case 3:
            case 4:
                ok = g == 0 && std::signbit(g) == !isMax;
                break;
            default:
                ok = g == (isMax ? (T)n : (T)1);
        }
        if (!ok) {
            printf("         %s element %zu: got %g\n", isMax ? "MAX" : "MIN", i, (double)g);
            return false;
        }
    }
    return true;
}

uint16_t toBf16(float f)
{
    uint32_t u;
    memcpy(&u, &f, 4);
    return std::isnan(f) ? (uint16_t)0x7fc0 : (uint16_t)(u >> 16); // exact for the values used here
}

float fromBf16(uint16_t h)
{
    uint32_t u = (uint32_t)h << 16;
    float f;
    memcpy(&f, &u, 4);
    return f;
}

// Full-range int32: every input has its top bit set, so SUM and PROD wrap
uint32_t wideInput(int r, size_t i)
{
    return (0x9e3779b9u * (uint32_t)(r + 1) + 0x7f4a7c15u * (uint32_t)i) | 0x80000000u;
}
}

TEST_CASE("mpi world case: host reductions ignore where a NaN or -0 sits and wrap integers, small and shared-memory sizes", "[mpi][world][cases]")
{
    // 5 elements take the message path (op_reduce); 64 Ki + 5 (> 256 KiB)
    // take the shared-memory fused reduction in a world whose ranks all live
    // here.  reduce() to the last rank folds the root's own input first, so a
    // NaN or -0 on the last rank is the accumulator there.
    const int n = 4;
    LocalWorld f(n);
    for (size_t count : { (size_t)5, (size_t)(64 * 1024 + 5) }) {
        std::vector<std::vector<float>> fin(n, std::vector<float>(count));
        std::vector<std::vector<double>> din(n, std::vector<double>(count));
        std::vector<std::vector<uint16_t>> hin(n, std::vector<uint16_t>(count));
        std::vector<std::vector<int32_t>> iin(n, std::vector<int32_t>(count));
        for (int r = 0; r < n; r++) {
            for (size_t i = 0; i < count; i++) {
                fin[r][i] = placed<float>(r, n, i);
                din[r][i] = placed<double>(r, n, i);
                hin[r][i] = toBf16(fin[r][i]);
                iin[r][i] = (int32_t)wideInput(r, i);
            }
        }
        for (bool isMax : { true, false }) {
            faabric_op_t* op = isMax ? MPI_MAX : MPI_MIN;
            std::vector<std::vector<float>> fout(n, std::vector<float>(count));
            std::vector<std::vector<double>> dout(n, std::vector<double>(count));
            std::vector<std::vector<uint16_t>> hout(n, std::vector<uint16_t>(count));
            onEveryRank(f, [&](int r) {
                f.world.allReduce(r, BYTES(fin[r].data()), BYTES(fout[r].data()), MPI_FLOAT, (int)count, op);
                f.world.allReduce(r, BYTES(din[r].data()), BYTES(dout[r].data()), MPI_DOUBLE, (int)count, op);
                f.world.allReduce(r, BYTES(hin[r].data()), BYTES(hout[r].data()), MPI_BFLOAT16, (int)count, op);
            });
            for (int r = 0; r < n; r++) {
                REQUIRE(placedMaxMinOk(fout[r], n, isMax));
                REQUIRE(placedMaxMinOk(dout[r], n, isMax));
                std::vector<float> widened(count);
                for (size_t i = 0; i < count; i++) {
                    widened[i] = fromBf16(hout[r][i]);
                }
                REQUIRE(placedMaxMinOk(widened, n, isMax));
            }
            std::vector<float> atRoot(count);
            std::vector<double> dAtRoot(count);
            onEveryRank(f, [&](int r) {
                f.world.reduce(r, n - 1, BYTES(fin[r].data()), r == n - 1 ? BYTES(atRoot.data()) : nullptr, MPI_FLOAT, (int)count, op);
                f.world.reduce(r, n - 1, BYTES(din[r].data()), r == n - 1 ? BYTES(dAtRoot.data()) : nullptr, MPI_DOUBLE, (int)count, op);
            });
            REQUIRE(placedMaxMinOk(atRoot, n, isMax));
            REQUIRE(placedMaxMinOk(dAtRoot, n, isMax));
        }
        for (faabric_op_t* op : { MPI_SUM, MPI_PROD }) {
            std::vector<std::vector<int32_t>> out(n, std::vector<int32_t>(count));
            onEveryRank(f, [&](int r) { f.world.allReduce(r, BYTES(iin[r].data()), BYTES(out[r].data()), MPI_INT, (int)count, op); });
            std::vector<int32_t> atRoot(count);
            onEveryRank(f, [&](int r) {
                f.world.reduce(r, n - 1, BYTES(iin[r].data()), r == n - 1 ? BYTES(atRoot.data()) : nullptr, MPI_INT, (int)count, op);
            });
            for (size_t i = 0; i < count; i++) {
                uint32_t e = op == MPI_SUM ? 0u : 1u;
                for (int r = 0; r < n; r++) {
                    e = op == MPI_SUM ? e + wideInput(r, i) : e * wideInput(r, i);
                }
                REQUIRE_EQ(atRoot[i], (int32_t)e);
                for (int r = 0; r < n; r++) {
                    REQUIRE_EQ(out[r][i], (int32_t)e);
                }
            }
        }
    }
}

TEST_CASE("mpi world case: scan gives every rank the reduction of the ranks up to itself", "[mpi][world][cases]")
{
    LocalWorld f(5);
    const int n = 3;
    std::vector<std::vector<int>> in(5, std::vector<int>(n)), out(5, std::vector<int>(n, -1));
    for (int r = 0; r < 5; r++) {
        for (int i = 0; i < n; i++) {
            in[r][i] = r * 10 + i;
        }
    }
    onEveryRank(f, [&](int r) { f.world.scan(r, BYTES(in[r].data()), BYTES(out[r].data()), MPI_INT, n, MPI_SUM); });
    std::vector<int> running(n, 0);
    for (int r = 0; r < 5; r++) {
        for (int i = 0; i < n; i++) {
            running[i] += in[r][i];
        }
        REQUIRE(out[r] == running);
    }
}

TEST_CASE("mpi world case: all-to-all", "[mpi][world][cases]")
{
    LocalWorld f(4);
    const int per = 2;
    std::vector<std::vector<int>> in(4, std::vector<int>(4 * per)), out(4, std::vector<int>(4 * per, -1));
    for (int r = 0; r < 4; r++) {
        for (int i = 0; i < 4 * per; i++) {
            in[r][i] = r * 100 + i;
        }
    }
    onEveryRank(f, [&](int r) {
        f.world.allToAll(r, BYTES(in[r].data()), MPI_INT, per, BYTES(out[r].data()), MPI_INT, per);
    });
    for (int r = 0; r < 4; r++) {
        for (int from = 0; from < 4; from++) {
            for (int k = 0; k < per; k++) {
                REQUIRE_EQ(out[r][from * per + k], from * 100 + r * per + k);
            }
        }
    }
}

TEST_CASE("mpi world case: the cartesian communicator of a 5 x 1 grid", "[mpi][world][cases]")
{
    LocalWorld f(5);
    int dims[2] = { 5, 1 };
    int periods[2] = { 0, 0 };
    for (int r = 0; r < 5; r++) {
        int coords[2] = { -1, -1 };
        f.world.getCartesianRank(r, 2, dims, periods, coords);
        REQUIRE(coords[0] == r && coords[1] == 0);
        REQUIRE(periods[0] == 1 && periods[1] == 1);
        int back = -1;
        f.world.getRankFromCoords(&back, coords);
        REQUIRE_EQ(back, r);
        // neighbours along the first dimension wrap around, the second has none but itself
        int src = -1, dst = -1;
        f.world.shiftCartesianCoords(r, 0, 1, &src, &dst);
        REQUIRE_EQ(src, (r + 4) % 5);
        REQUIRE_EQ(dst, (r + 1) % 5);
        f.world.shiftCartesianCoords(r, 1, 1, &src, &dst);
        REQUIRE_EQ(src, r);
        REQUIRE_EQ(dst, r);
    }
    // a grid that does not match the world size is refused
    int bad[2] = { 3, 3 };
    int c[2];
    REQUIRE_THROWS(f.world.getCartesianRank(0, 2, bad, periods, c));
}

TEST_CASE("mpi message case: sizes with and without a payload", "[mpi][message][cases]")
{
    MpiMessage msg{};
    msg.typeSize = sizeof(int);
    msg.count = 0;
    msg.buffer = nullptr;
    REQUIRE_EQ(payloadSize(msg), 0u);
    REQUIRE_EQ(msgSize(msg), sizeof(MpiMessage));
    std::vector<int> payload = { 1, 2, 3 };
    msg.count = 3;
    msg.buffer = payload.data();
    REQUIRE_EQ(payloadSize(msg), 3 * sizeof(int));
    REQUIRE_EQ(msgSize(msg), sizeof(MpiMessage) + 3 * sizeof(int));
}

TEST_CASE("mpi message case: serialise and parse, with and without a payload", "[mpi][message][cases]")
{
    for (bool withData : { false, true }) {
        std::vector<int> payload = { 4, 5, 6, 7 };
        MpiMessage msg{};
        msg.id = 11;
        msg.worldId = 22;
        msg.sendRank = 3;
        msg.recvRank = 4;
        msg.typeSize = sizeof(int);
        msg.count = withData ? 4 : 0;
        msg.requestId = 99;
        msg.messageType = MpiMessageType::BROADCAST;
        msg.buffer = withData ? (void*)payload.data() : nullptr;
        std::vector<uint8_t> wire;
        serializeMpiMsg(wire, msg);
        REQUIRE_EQ(wire.size(), msgSize(msg));
        MpiMessage parsed{};
        parseMpiMsg(wire, &parsed);
        REQUIRE_EQ(parsed.id, 11);
        REQUIRE_EQ(parsed.worldId, 22);
        REQUIRE_EQ(parsed.sendRank, 3);
        REQUIRE_EQ(parsed.recvRank, 4);
        REQUIRE_EQ(parsed.typeSize, (int)sizeof(int));
        REQUIRE_EQ(parsed.count, withData ? 4 : 0);
        REQUIRE_EQ(parsed.requestId, 99);
        REQUIRE(parsed.messageType == MpiMessageType::BROADCAST);
        if (withData) {
            REQUIRE(parsed.buffer != nullptr);
            REQUIRE(memcmp(parsed.buffer, payload.data(), 4 * sizeof(int)) == 0);
            free(parsed.buffer);
        } else {
            REQUIRE(parsed.buffer == nullptr);
        }
    }
}

TEST_CASE("mpi world case: two worlds side by side keep their messages apart", "[mpi][world][cases]")
{
    LocalWorld a(3, 123);
    LocalWorld b(4, 245);
    REQUIRE_EQ(a.world.getSize(), 3);
    REQUIRE_EQ(b.world.getSize(), 4);
    REQUIRE_EQ(a.world.getId(), 123);
    REQUIRE_EQ(b.world.getId(), 245);
    std::vector<int> forA = { 1, 2, 3 }, forB = { 9, 8 };
    a.world.send(0, 1, BYTES(forA.data()), MPI_INT, 3);
    b.world.send(0, 1, BYTES(forB.data()), MPI_INT, 2);
    // the same rank pair in the other world sees only its own traffic
    REQUIRE(recvVec<int>(b.world, 0, 1, MPI_INT, 2) == forB);
    REQUIRE(recvVec<int>(a.world, 0, 1, MPI_INT, 3) == forA);
    // rank 3 exists in one of them only
    int v = 0;
    REQUIRE_THROWS(a.world.send(0, 3, BYTES(&v), MPI_INT, 1));
    b.world.send(0, 3, BYTES(&v), MPI_INT, 1);
    recvVec<int>(b.world, 0, 3, MPI_INT, 1);
}

TEST_CASE("mpi context case: a fresh context is not part of any world", "[mpi][context][cases]")
{
    MpiContext c;
    REQUIRE(!c.getIsMpi());
    REQUIRE_EQ(c.getWorldId(), -1);
    REQUIRE_EQ(c.getRank(), -1);
}

TEST_CASE("mpi context case: only rank zero may create a world", "[mpi][context][cases]")
{
    ClusterFixture f(8);
    auto req = faabric::util::batchExecFactory("mpi", "hellompi", 1);
    auto& msg = *req->mutable_messages(0);
    msg.set_mpiworldsize(4);
    msg.set_mpirank(2);
    MpiContext c;
    REQUIRE_THROWS(c.createWorld(msg));
    REQUIRE(!c.getIsMpi());
}

TEST_CASE("mpi context case: creating a world names it and sizes it; other ranks join by message", "[mpi][context][cases]")
{
    ClusterFixture f(8);
    std::atomic<int> joined{ 0 };
    std::atomic<int> bad{ 0 };
    std::atomic<int> worldIdSeen{ 0 };
    registerTestFunction("mpi", "ctxcase", [&](auto*, int, int idx, auto req) {
        auto& m = *req->mutable_messages(idx);
        MpiContext c;
        if (m.mpirank() == 0) {
            int id = c.createWorld(m);
            if (id <= 0 || !c.getIsMpi() || c.getRank() != 0 || c.getWorldId() != id) {
                bad++;
            }
            worldIdSeen = id;
            m.set_mpiworldid(id);
            MpiWorld& w = getMpiWorldRegistry().getOrInitialiseWorld(m);
            if (w.getId() != id || w.getSize() != 3 || w.getUser() != "mpi" || w.getFunction() != "ctxcase") {
                bad++;
            }
            w.barrier(0);
            w.destroy();
        } else {
            c.joinWorld(m);
            if (!c.getIsMpi() || c.getRank() != m.mpirank() || c.getWorldId() != m.mpiworldid()) {
                bad++;
            }
            MpiWorld& w = getMpiWorldRegistry().getOrInitialiseWorld(m);
            if (w.getHostForRank(m.mpirank()) != faabric::util::getSystemConfig().endpointHost) {
                bad++;
            }
            joined++;
            w.barrier(m.mpirank());
            w.destroy();
        }
        return 0;
    });
    auto req = faabric::util::batchExecFactory("mpi", "ctxcase", 1);
    req->mutable_messages(0)->set_ismpi(true);
    req->mutable_messages(0)->set_mpiworldsize(3);
    f.plannerCli.callFunctions(req);
    auto res = f.awaitResult(req->messages(0), 20000);
    REQUIRE_EQ(res.returnvalue(), 0);
    for (int i = 0; i < 400 && joined.load() < 2; i++) {
        std::this_thread::sleep_for(std::chrono::milliseconds(5));
    }
    REQUIRE_EQ(joined.load(), 2);
    REQUIRE_EQ(bad.load(), 0);
    REQUIRE(worldIdSeen.load() > 0);
    f.awaitBatch(req);
    getMpiWorldRegistry().clear();
}

TEST_CASE("mpi context case: the configured default size applies when the message names none", "[mpi][context][cases]")
{
    ClusterFixture f(8);
    f.conf.defaultMpiWorldSize = 3;
    std::atomic<int> sizeSeen{ 0 };
    registerTestFunction("mpi", "defsize", [&](auto*, int, int idx, auto req) {
        auto& m = *req->mutable_messages(idx);
        MpiContext c;
        if (m.mpirank() == 0) {
            // (the planner reserved room for the size the request named; the
            // function itself then asks for "whatever the default is")
            m.set_mpiworldsize(0);
            int id = c.createWorld(m);
            m.set_mpiworldid(id);
            MpiWorld& w = getMpiWorldRegistry().getOrInitialiseWorld(m);
            sizeSeen = w.getSize();
            w.barrier(0);
            w.destroy();
        } else {
            c.joinWorld(m);
            MpiWorld& w = getMpiWorldRegistry().getOrInitialiseWorld(m);
            w.barrier(m.mpirank());
            w.destroy();
        }
        return 0;
    });
    auto req = faabric::util::batchExecFactory("mpi", "defsize", 1);
    req->mutable_messages(0)->set_ismpi(true);
    req->mutable_messages(0)->set_mpiworldsize(5);
    f.plannerCli.callFunctions(req);
    REQUIRE_EQ(f.awaitResult(req->messages(0), 20000).returnvalue(), 0);
    REQUIRE_EQ(sizeSeen.load(), 3);
    f.awaitBatch(req);
    f.conf.reset();
    getMpiWorldRegistry().clear();
}
