// General purpose worker: embeds the runtime with a table of built-in
// functions (a demo set plus the MPI example programs used by the
// distributed tests and the CPU baseline benchmarks).
//
// Plays the role of the reference's tests/dist/server.cpp + DistTestExecutor,
// and of the tests/dist/mpi/examples/*.cpp programs.
#include <faabric/endpoint/FaabricEndpoint.h>
#include <faabric/endpoint/FaabricEndpointHandler.h>
#include <faabric/executor/ExecutorFactory.h>
#include <faabric/mpi/MpiWorld.h>
#include <faabric/mpi/MpiWorldRegistry.h>
#include <faabric/executor/ExecutorContext.h>
#include <faabric/mpi/migration.h>
#include <faabric/mpi/mpi.h>
#include <faabric/planner/PlannerClient.h>
#include <faabric/runner/FaabricMain.h>
#include <faabric/scheduler/Scheduler.h>
#include <faabric/state/State.h>
#include <faabric/transport/PointToPointBroker.h>
#include <faabric/util/batch.h>
#include <faabric/util/config.h>
#include <faabric/util/logging.h>
#include <faabric/util/memory.h>
#include <faabric/util/snapshot.h>

#include "../tests/mpi_rma_atomics_body.h"
#include "../tests/mpi_rma_passive_body.h"
#include "../tests/mpi_rma_request_body.h"
#include "../tests/mpi_subcomm_device_body.h"

#include <cuda_runtime.h>

#include <chrono>
#include <cmath>
#include <functional>
#include <map>
#include <numeric>
#include <thread>
#include <unistd.h>

using namespace faabric::executor;

typedef std::function<int(faabric::Message&)> WorkerFunction;

static std::map<std::string, WorkerFunction>& functions()
{
    static std::map<std::string, WorkerFunction> t;
    return t;
}

#define EXPECT(cond)                                                           \
    do {                                                                       \
        if (!(cond)) {                                                         \
            SPDLOG_ERROR("rank {}: check failed at line {}: {}", rank, __LINE__, #cond); \
            return 1;                                                          \
        }                                                                      \
    } while (0)

// Wraps an MPI program body with Init / Finalize
static void mpiFunction(const std::string& name, std::function<int(int, int, faabric::Message&)> body)
{
    functions()["mpi/" + name] = [body](faabric::Message& msg) {
        MPI_Init(nullptr, nullptr);
        int rank = 0, size = 0;
        MPI_Comm_rank(MPI_COMM_WORLD, &rank);
        MPI_Comm_size(MPI_COMM_WORLD, &size);
        int rc = body(rank, size, msg);
        MPI_Finalize();
        return rc;
    };
}

static void registerFunctions()
{
    functions()["demo/echo"] = [](faabric::Message& msg) {
        msg.set_outputdata(msg.inputdata());
        return 0;
    };
    functions()["demo/hello"] = [](faabric::Message& msg) {
        msg.set_outputdata("hello from " + faabric::scheduler::getScheduler().getThisHost());
        return 0;
    };
    functions()["demo/sleep"] = [](faabric::Message& msg) {
        int ms = msg.inputdata().empty() ? 100 : std::stoi(msg.inputdata());
        std::this_thread::sleep_for(std::chrono::milliseconds(ms));
        return 0;
    };
    functions()["demo/error"] = [](faabric::Message& msg) {
        msg.set_outputdata("deliberate failure");
        return 1;
    };
    functions()["demo/noop"] = [](faabric::Message&) { return 0; };

    // Distributed coordination: the functions of one batch (spread over the
    // workers) increment a shared counter held in distributed state under the
    // group's lock, then meet at the group barrier; idx 0 reports the total.
    functions()["ptp/counter"] = [](faabric::Message& msg) {
        const int rounds = msg.inputdata().empty() ? 5 : std::stoi(msg.inputdata());
        auto group = faabric::transport::PointToPointGroup::getOrAwaitGroup(msg.groupid());
        const int idx = msg.groupidx();
        auto& state = faabric::state::getGlobalState();
        const std::string key = "counter-" + std::to_string(msg.appid());
        auto kv = state.getKV("ptp", key, sizeof(int));
        for (int i = 0; i < rounds; i++) {
            group->lock(idx, false);
            kv->pull();
            int v = 0;
            kv->get((uint8_t*)&v);
            v++;
            kv->set((const uint8_t*)&v);
            kv->pushFull();
            group->unlock(idx, false);
        }
        group->barrier(idx);
        kv->pull();
        int total = 0;
        kv->get((uint8_t*)&total);
        msg.set_outputdata(std::to_string(total) + " on " + faabric::scheduler::getScheduler().getThisHost());
        group->barrier(idx);
        if (idx == 0) {
            state.deleteKV("ptp", key);
        }
        return 0;
    };

    // Ordered point-to-point streams between every pair of group members
    // (reference dist test "many in-order messages", tests/dist/transport)
    functions()["ptp/stream"] = [](faabric::Message& msg) {
        const int n = msg.inputdata().empty() ? 500 : std::stoi(msg.inputdata());
        auto& broker = faabric::transport::getPointToPointBroker();
        auto group = faabric::transport::PointToPointGroup::getOrAwaitGroup(msg.groupid());
        const int idx = msg.groupidx();
        const int size = msg.groupsize() > 0 ? msg.groupsize() : (int)broker.getIdxsRegisteredForGroup(msg.groupid()).size();
        // everybody streams n numbered messages to everybody else...
        for (int i = 0; i < n; i++) {
            for (int peer = 0; peer < size; peer++) {
                if (peer != idx) {
                    int payload[2] = { idx, i };
                    broker.sendMessage(msg.groupid(), idx, peer, (const uint8_t*)payload, sizeof(payload), true);
                }
            }
        }
        // ...and must see each stream in order
        int bad = 0;
        for (int peer = 0; peer < size; peer++) {
            if (peer == idx) {
                continue;
            }
            for (int i = 0; i < n; i++) {
                auto bytes = broker.recvMessage(msg.groupid(), peer, idx, true);
                const int* payload = (const int*)bytes.data();
                if (bytes.size() != 2 * sizeof(int) || payload[0] != peer || payload[1] != i) {
                    bad++;
                }
            }
        }
        group->barrier(idx);
        msg.set_outputdata(std::to_string(bad) + " out of order on " + faabric::scheduler::getScheduler().getThisHost());
        broker.resetThreadLocalCache();
        return bad == 0 ? 0 : 1;
    };

    // Fork-join over THREADS: the main function spawns N threads that may land
    // on other workers; they start from its snapshot, write their own slot and
    // add into a Sum-merged word; the diffs are merged back into main memory.
    functions()["demo/threads"] = [](faabric::Message& msg) {
        auto ctx = ExecutorContext::get();
        auto* exec = ctx->getExecutor();
        auto mem = exec->getMemoryView();
        int* sumCell = (int*)(mem.data() + 64);
        if (ctx->getBatchRequest()->type() == faabric::BatchExecuteRequest::THREADS) {
            int t = msg.appidx();
            mem[8192 + t] = (uint8_t)(10 + t);
            __atomic_fetch_add(sumCell, t + 1, __ATOMIC_RELAXED);
            msg.set_outputdata("thread " + std::to_string(t) + " on " + faabric::scheduler::getScheduler().getThisHost());
            return t;
        }
        int nThreads = msg.inputdata().empty() ? 4 : std::stoi(msg.inputdata());
        *sumCell = 100;
        auto threads = faabric::util::batchExecFactory(msg.user(), msg.function(), nThreads);
        faabric::util::updateBatchExecAppId(threads, msg.appid());
        for (int i = 0; i < nThreads; i++) {
            threads->mutable_messages(i)->set_appidx(i + 1);
            threads->mutable_messages(i)->set_groupidx(i + 1);
        }
        std::vector<faabric::util::SnapshotMergeRegion> regions = {
            { 64, sizeof(int), faabric::util::SnapshotDataType::Int, faabric::util::SnapshotMergeOperation::Sum }
        };
        auto results = exec->executeThreads(threads, regions);
        int expectedSum = 100;
        std::string hosts;
        for (int i = 0; i < nThreads; i++) {
            expectedSum += i + 2;
            if (results.at(i).second != i + 1) {
                msg.set_outputdata("thread " + std::to_string(i + 1) + " returned " + std::to_string(results.at(i).second));
                return 1;
            }
            if (mem[8192 + i + 1] != 10 + i + 1) {
                msg.set_outputdata("slot of thread " + std::to_string(i + 1) + " not merged");
                return 1;
            }
        }
        if (*sumCell != expectedSum) {
            msg.set_outputdata("sum is " + std::to_string(*sumCell) + ", expected " + std::to_string(expectedSum));
            return 1;
        }
        msg.set_outputdata("merged sum " + std::to_string(*sumCell));
        return 0;
    };

    // Repeated fork-join with two Sum reductions (one sharing a page with a
    // per-thread array) across whatever hosts the threads land on; checks that
    // snapshots stay in step over many rounds
    // (reference dist test "Check repeated reduction",
    // tests/dist/scheduler/functions.cpp:201-360)
    functions()["demo/reduction"] = [](faabric::Message& msg) {
        auto ctx = ExecutorContext::get();
        auto* exec = ctx->getExecutor();
        auto mem = exec->getMemoryView();
        const size_t page = faabric::util::HOST_PAGE_SIZE;
        int32_t* reductionA = (int32_t*)(mem.data() + page);
        int32_t* reductionB = (int32_t*)(mem.data() + 2 * page);
        int32_t* array = (int32_t*)(mem.data() + page + 10 * sizeof(int32_t));
        const int nThreads = 4;
        if (ctx->getBatchRequest()->type() == faabric::BatchExecuteRequest::THREADS) {
            int idx = msg.appidx();
            // threads sharing an executor's memory take turns
            auto group = faabric::transport::PointToPointGroup::getGroup(msg.groupid());
            group->localLock();
            *reductionA += 10;
            *reductionB += 20;
            array[idx] = idx * 30;
            group->localUnlock();
            msg.set_outputdata("thread " + std::to_string(idx) + " on " + faabric::scheduler::getScheduler().getThisHost());
            return 0;
        }
        const int nRepeats = msg.inputdata().empty() ? 20 : std::stoi(msg.inputdata());
        for (int r = 0; r < nRepeats; r++) {
            auto threads = faabric::util::batchExecFactory(msg.user(), msg.function(), nThreads);
            faabric::util::updateBatchExecAppId(threads, msg.appid());
            for (int i = 0; i < nThreads; i++) {
                threads->mutable_messages(i)->set_appidx(i);
                threads->mutable_messages(i)->set_groupidx(i);
            }
            std::vector<faabric::util::SnapshotMergeRegion> regions = {
                { (uint32_t)page, sizeof(int32_t), faabric::util::SnapshotDataType::Int, faabric::util::SnapshotMergeOperation::Sum },
                { (uint32_t)(2 * page), sizeof(int32_t), faabric::util::SnapshotDataType::Int, faabric::util::SnapshotMergeOperation::Sum }
            };
            auto results = exec->executeThreads(threads, regions);
            for (auto& [id, rv] : results) {
                if (rv != 0) {
                    msg.set_outputdata("round " + std::to_string(r) + ": thread " + std::to_string(id) + " returned " + std::to_string(rv));
                    return 1;
                }
            }
            int expectedA = (r + 1) * nThreads * 10, expectedB = (r + 1) * nThreads * 20;
            if (*reductionA != expectedA || *reductionB != expectedB) {
                msg.set_outputdata("round " + std::to_string(r) + ": reductions " + std::to_string(*reductionA) + " / " +
                                   std::to_string(*reductionB) + ", expected " + std::to_string(expectedA) + " / " +
                                   std::to_string(expectedB));
                return 1;
            }
            for (int i = 0; i < nThreads; i++) {
                if (array[i] != i * 30) {
                    msg.set_outputdata("round " + std::to_string(r) + ": array[" + std::to_string(i) + "] = " + std::to_string(array[i]));
                    return 1;
                }
            }
        }
        msg.set_outputdata("reduced " + std::to_string(nRepeats) + " rounds to " + std::to_string(*reductionA) + " / " +
                           std::to_string(*reductionB));
        return 0;
    };

    mpiFunction("helloworld", [](int rank, int size, faabric::Message& msg) {
        char name[MPI_MAX_PROCESSOR_NAME];
        int len = 0;
        MPI_Get_processor_name(name, &len);
        msg.set_outputdata("rank " + std::to_string(rank) + "/" + std::to_string(size) + " on " + name);
        return 0;
    });

    mpiFunction("allreduce", [](int rank, int size, faabric::Message&) {
        std::vector<int> v(1000, rank + 1), out(1000, 0);
        MPI_Allreduce(v.data(), out.data(), 1000, MPI_INT, MPI_SUM, MPI_COMM_WORLD);
        EXPECT(out[0] == size * (size + 1) / 2 && out[999] == out[0]);
        std::vector<double> d(17, rank), dout(17, 0);
        MPI_Allreduce(d.data(), dout.data(), 17, MPI_DOUBLE, MPI_MAX, MPI_COMM_WORLD);
        EXPECT(dout[5] == size - 1);
        MPI_Allreduce(MPI_IN_PLACE, v.data(), 1000, MPI_INT, MPI_MIN, MPI_COMM_WORLD);
        EXPECT(v[0] == 1);
        return 0;
    });

    mpiFunction("allgather", [](int rank, int size, faabric::Message&) {
        std::vector<int> mine = { rank, rank * 2 }, all(2 * size, -1);
        MPI_Allgather(mine.data(), 2, MPI_INT, all.data(), 2, MPI_INT, MPI_COMM_WORLD);
        for (int r = 0; r < size; r++) {
            EXPECT(all[2 * r] == r && all[2 * r + 1] == 2 * r);
        }
        return 0;
    });

    mpiFunction("alltoall", [](int rank, int size, faabric::Message&) {
        std::vector<int> s(size), r(size, -1);
        for (int i = 0; i < size; i++) {
            s[i] = rank * 100 + i;
        }
        MPI_Alltoall(s.data(), 1, MPI_INT, r.data(), 1, MPI_INT, MPI_COMM_WORLD);
        for (int i = 0; i < size; i++) {
            EXPECT(r[i] == i * 100 + rank);
        }
        return 0;
    });

    mpiFunction("bcast", [](int rank, int size, faabric::Message&) {
        int root = size > 2 ? 2 : 0;
        std::vector<long> v(500, rank == root ? 42 : -1);
        MPI_Bcast(v.data(), 500, MPI_LONG, root, MPI_COMM_WORLD);
        EXPECT(v[0] == 42 && v[499] == 42);
        return 0;
    });

    mpiFunction("barrier", [](int rank, int size, faabric::Message&) {
        for (int i = 0; i < 20; i++) {
            MPI_Barrier(MPI_COMM_WORLD);
        }
        return 0;
    });

    mpiFunction("gather-scatter", [](int rank, int size, faabric::Message&) {
        const int per = 3;
        std::vector<int> all(per * size), mine(per, -1);
        if (rank == 0) {
            std::iota(all.begin(), all.end(), 0);
        }
        MPI_Scatter(all.data(), per, MPI_INT, mine.data(), per, MPI_INT, 0, MPI_COMM_WORLD);
        for (int i = 0; i < per; i++) {
            EXPECT(mine[i] == rank * per + i);
            mine[i] += 1000;
        }
        int root = size - 1;
        std::vector<int> back(per * size, -1);
        MPI_Gather(mine.data(), per, MPI_INT, back.data(), per, MPI_INT, root, MPI_COMM_WORLD);
        if (rank == root) {
            for (int i = 0; i < per * size; i++) {
                EXPECT(back[i] == 1000 + i);
            }
        }
        return 0;
    });

    mpiFunction("reduce-scan", [](int rank, int size, faabric::Message&) {
        int v = rank + 1, out = 0;
        MPI_Reduce(&v, &out, 1, MPI_INT, MPI_SUM, 0, MPI_COMM_WORLD);
        if (rank == 0) {
            EXPECT(out == size * (size + 1) / 2);
        }
        MPI_Scan(&v, &out, 1, MPI_INT, MPI_SUM, MPI_COMM_WORLD);
        EXPECT(out == (rank + 1) * (rank + 2) / 2);
        return 0;
    });

    mpiFunction("sendrecv", [](int rank, int size, faabric::Message&) {
        int right = (rank + 1) % size, left = (rank + size - 1) % size;
        std::vector<double> out(2048, rank), in(2048, -1);
        MPI_Status st{};
        MPI_Sendrecv(out.data(), 2048, MPI_DOUBLE, right, 0, in.data(), 2048, MPI_DOUBLE, left, 0, MPI_COMM_WORLD, &st);
        EXPECT(in[0] == left && in[2047] == left);
        EXPECT(st.MPI_SOURCE == left);
        return 0;
    });

    mpiFunction("isendrecv", [](int rank, int size, faabric::Message&) {
        std::vector<int> sendVals(size), recvVals(size, -1);
        std::vector<MPI_Request> reqs;
        for (int r = 0; r < size; r++) {
            if (r == rank) {
                continue;
            }
            MPI_Request rq;
            MPI_Irecv(&recvVals[r], 1, MPI_INT, r, 0, MPI_COMM_WORLD, &rq);
            reqs.push_back(rq);
        }
        for (int r = 0; r < size; r++) {
            if (r == rank) {
                continue;
            }
            sendVals[r] = rank * 1000 + r;
            MPI_Request rq;
            MPI_Isend(&sendVals[r], 1, MPI_INT, r, 0, MPI_COMM_WORLD, &rq);
            reqs.push_back(rq);
        }
        MPI_Waitall((int)reqs.size(), reqs.data(), MPI_STATUSES_IGNORE);
        for (int r = 0; r < size; r++) {
            if (r != rank) {
                EXPECT(recvVals[r] == r * 1000 + rank);
            }
        }
        return 0;
    });

    // Messages between a pair keep their order even when received out of
    // posting order
    mpiFunction("order", [](int rank, int size, faabric::Message&) {
        if (rank == 0) {
            for (int i = 0; i < 50; i++) {
                MPI_Send(&i, 1, MPI_INT, size - 1, 0, MPI_COMM_WORLD);
            }
        } else if (rank == size - 1) {
            std::vector<int> got(50, -1);
            std::vector<MPI_Request> reqs(50);
            for (int i = 0; i < 50; i++) {
                MPI_Irecv(&got[i], 1, MPI_INT, 0, 0, MPI_COMM_WORLD, &reqs[i]);
            }
            for (int i = 49; i >= 0; i--) {
                MPI_Wait(&reqs[i], MPI_STATUS_IGNORE);
            }
            for (int i = 0; i < 50; i++) {
                EXPECT(got[i] == i);
            }
        }
        MPI_Barrier(MPI_COMM_WORLD);
        return 0;
    });

    mpiFunction("status-probe", [](int rank, int size, faabric::Message&) {
        if (rank == 0) {
            std::vector<int> v(33, 7);
            MPI_Send(v.data(), 33, MPI_INT, 1, 0, MPI_COMM_WORLD);
        } else if (rank == 1) {
            MPI_Status st{};
            MPI_Probe(0, 0, MPI_COMM_WORLD, &st);
            int count = 0;
            MPI_Get_count(&st, MPI_INT, &count);
            EXPECT(count == 33);
            std::vector<int> v(64, 0);
            MPI_Recv(v.data(), 64, MPI_INT, 0, 0, MPI_COMM_WORLD, &st);
            MPI_Get_count(&st, MPI_INT, &count);
            EXPECT(count == 33 && v[32] == 7 && v[33] == 0);
        }
        return 0;
    });

    mpiFunction("cart", [](int rank, int size, faabric::Message&) {
        int side = (int)std::lround(std::sqrt((double)size));
        if (side * side != size) {
            return 0;
        }
        int dims[2] = { side, side }, periods[2] = { 1, 1 }, coords[2];
        MPI_Comm cart;
        MPI_Cart_create(MPI_COMM_WORLD, 2, dims, periods, 0, &cart);
        MPI_Cart_get(cart, 2, dims, periods, coords);
        EXPECT(coords[0] == rank / side && coords[1] == rank % side);
        int src, dst;
        MPI_Cart_shift(cart, 1, 1, &src, &dst);
        int token = rank, got = -1;
        MPI_Sendrecv(&token, 1, MPI_INT, dst, 0, &got, 1, MPI_INT, src, 0, cart, MPI_STATUS_IGNORE);
        EXPECT(got == src);
        return 0;
    });

    // Many messages / collectives back to back (reference dist tests
    // mpi_send_many, mpi_reduce_many, mpi_alltoall_many, mpi_send_sync_async,
    // mpi_typesize)
    mpiFunction("send-many", [](int rank, int size, faabric::Message&) {
        const int n = 2000;
        if (rank == 0) {
            for (int i = 0; i < n; i++) {
                for (int r = 1; r < size; r++) {
                    int v = i * size + r;
                    MPI_Send(&v, 1, MPI_INT, r, 0, MPI_COMM_WORLD);
                }
            }
        } else {
            for (int i = 0; i < n; i++) {
                int v = -1;
                MPI_Recv(&v, 1, MPI_INT, 0, 0, MPI_COMM_WORLD, MPI_STATUS_IGNORE);
                EXPECT(v == i * size + rank);
            }
        }
        return 0;
    });

    mpiFunction("reduce-many", [](int rank, int size, faabric::Message&) {
        for (int i = 0; i < 300; i++) {
            int root = i % size;
            long mine[3] = { rank + i, 2L * rank, 1 }, out[3] = { 0, 0, 0 };
            MPI_Reduce(mine, out, 3, MPI_LONG, MPI_SUM, root, MPI_COMM_WORLD);
            if (rank == root) {
                long base = (long)size * (size - 1) / 2;
                EXPECT(out[0] == base + (long)i * size && out[1] == 2 * base && out[2] == size);
            }
        }
        return 0;
    });

    mpiFunction("alltoall-many", [](int rank, int size, faabric::Message&) {
        std::vector<int> out(size * 4), in(size * 4);
        for (int i = 0; i < 200; i++) {
            for (int r = 0; r < size; r++) {
                for (int k = 0; k < 4; k++) {
                    out[r * 4 + k] = i * 1000 + rank * 10 + r;
                }
            }
            MPI_Alltoall(out.data(), 4, MPI_INT, in.data(), 4, MPI_INT, MPI_COMM_WORLD);
            for (int r = 0; r < size; r++) {
                EXPECT(in[r * 4] == i * 1000 + r * 10 + rank && in[r * 4 + 3] == in[r * 4]);
            }
        }
        return 0;
    });

    // Rank 0 hands every rank a number and waits for each to answer
    // (reference dist test "MPI checks", tests/dist/mpi/examples/mpi_checks.cpp)
    mpiFunction("checks", [](int rank, int size, faabric::Message&) {
        EXPECT(rank >= 0 && size > 1);
        if (rank == 0) {
            for (int r = 1; r < size; r++) {
                int sent = -100 - r;
                MPI_Send(&sent, 1, MPI_INT, r, 0, MPI_COMM_WORLD);
            }
            int responses = 0;
            for (int r = 1; r < size; r++) {
                int got = -1;
                MPI_Recv(&got, 1, MPI_INT, r, 0, MPI_COMM_WORLD, MPI_STATUS_IGNORE);
                EXPECT(got == r);
                responses++;
            }
            EXPECT(responses == size - 1);
        } else {
            int got = 0;
            MPI_Recv(&got, 1, MPI_INT, 0, 0, MPI_COMM_WORLD, MPI_STATUS_IGNORE);
            EXPECT(got == -100 - rank);
            MPI_Send(&rank, 1, MPI_INT, 0, 0, MPI_COMM_WORLD);
        }
        return 0;
    });

    // One plain send from rank 0 to rank 1 (reference: mpi_send.cpp)
    mpiFunction("send", [](int rank, int size, faabric::Message&) {
        if (rank == 0) {
            int v = 123;
            MPI_Send(&v, 1, MPI_INT, 1, 0, MPI_COMM_WORLD);
        } else if (rank == 1) {
            int v = 0;
            MPI_Status st{};
            MPI_Recv(&v, 1, MPI_INT, 0, 0, MPI_COMM_WORLD, &st);
            EXPECT(v == 123 && st.MPI_SOURCE == 0);
        }
        return 0;
    });

    // Barriers and all-to-alls, a long pause with nothing in flight, then the
    // same again: connections and queues must survive sitting idle
    // (reference: mpi_alltoall_sleep.cpp; the pause is 1 s here, 5 s there)
    mpiFunction("alltoall-sleep", [](int rank, int size, faabric::Message&) {
        std::vector<int> out(size), in(size);
        auto round = [&](int i) {
            MPI_Barrier(MPI_COMM_WORLD);
            for (int r = 0; r < size; r++) {
                out[r] = i * 1000 + rank * 10 + r;
            }
            MPI_Alltoall(out.data(), 1, MPI_INT, in.data(), 1, MPI_INT, MPI_COMM_WORLD);
            for (int r = 0; r < size; r++) {
                if (in[r] != i * 1000 + r * 10 + rank) {
                    return false;
                }
            }
            return true;
        };
        for (int i = 0; i < 500; i++) {
            EXPECT(round(i));
        }
        std::this_thread::sleep_for(std::chrono::milliseconds(1000));
        for (int i = 0; i < 500; i++) {
            EXPECT(round(i));
        }
        return 0;
    });

    mpiFunction("sync-async", [](int rank, int size, faabric::Message&) {
        // every rank in turn sends to all: blocking first, then non-blocking
        for (int sender = 0; sender < size; sender++) {
            if (rank == sender) {
                std::vector<MPI_Request> reqs;
                std::vector<int> vals(size);
                for (int r = 0; r < size; r++) {
                    if (r == rank) {
                        continue;
                    }
                    int v = sender * 100 + r;
                    MPI_Send(&v, 1, MPI_INT, r, 0, MPI_COMM_WORLD);
                    vals[r] = v + 1;
                    MPI_Request rq;
                    MPI_Isend(&vals[r], 1, MPI_INT, r, 0, MPI_COMM_WORLD, &rq);
                    reqs.push_back(rq);
                }
                MPI_Waitall((int)reqs.size(), reqs.data(), MPI_STATUSES_IGNORE);
            } else {
                int a = -1, b = -1;
                MPI_Request rq;
                MPI_Recv(&a, 1, MPI_INT, sender, 0, MPI_COMM_WORLD, MPI_STATUS_IGNORE);
                MPI_Irecv(&b, 1, MPI_INT, sender, 0, MPI_COMM_WORLD, &rq);
                MPI_Wait(&rq, MPI_STATUS_IGNORE);
                EXPECT(a == sender * 100 + rank && b == a + 1);
            }
        }
        return 0;
    });

    mpiFunction("typesize", [](int rank, int size, faabric::Message&) {
        struct Expect
        {
            MPI_Datatype type;
            int bytes;
        };
        const Expect table[] = {
            { MPI_INT8_T, 1 },   { MPI_INT16_T, 2 },  { MPI_INT32_T, 4 },  { MPI_INT64_T, 8 },   { MPI_UINT8_T, 1 },
            { MPI_UINT16_T, 2 }, { MPI_UINT32_T, 4 }, { MPI_UINT64_T, 8 }, { MPI_INT, 4 },       { MPI_LONG, 8 },
            { MPI_LONG_LONG, 8 }, { MPI_FLOAT, 4 },   { MPI_DOUBLE, 8 },   { MPI_DOUBLE_INT, 16 }, { MPI_CHAR, 1 },
            { MPI_BYTE, 1 },
        };
        for (const auto& e : table) {
            int got = 0;
            MPI_Type_size(e.type, &got);
            EXPECT(got == e.bytes);
        }
        return 0;
    });

    // Sub-communicators whose members sit in different worker processes
    mpiFunction("subcomm", [](int rank, int size, faabric::Message& msg) {
        MPI_Comm half = nullptr;
        MPI_Comm_split(MPI_COMM_WORLD, rank % 2, rank, &half);
        int hRank = -1, hSize = -1;
        MPI_Comm_rank(half, &hRank);
        MPI_Comm_size(half, &hSize);
        EXPECT(hRank == rank / 2);
        EXPECT(hSize == (size + (rank % 2 == 0 ? 1 : 0)) / 2);
        long mine = rank, sum = -1;
        MPI_Allreduce(&mine, &sum, 1, MPI_LONG, MPI_SUM, half);
        long expected = 0;
        for (int r = rank % 2; r < size; r += 2) {
            expected += r;
        }
        EXPECT(sum == expected);
        std::vector<double> big(50000, hRank == 0 ? 3.5 + rank : 0.0);
        MPI_Bcast(big.data(), (int)big.size(), MPI_DOUBLE, 0, half);
        EXPECT(big[0] == 3.5 + rank % 2 && big.back() == 3.5 + rank % 2);
        std::vector<int> all(hSize, -1);
        MPI_Allgather(&rank, 1, MPI_INT, all.data(), 1, MPI_INT, half);
        for (int i = 0; i < hSize; i++) {
            EXPECT(all[i] == rank % 2 + 2 * i);
        }
        MPI_Barrier(half);
        // ranks of this worker process
        MPI_Comm node = nullptr;
        MPI_Comm_split_type(MPI_COMM_WORLD, MPI_COMM_TYPE_SHARED, rank, MPI_INFO_NULL, &node);
        int nodeSize = -1, nodeSum = 0, one = 1;
        MPI_Comm_size(node, &nodeSize);
        MPI_Allreduce(&one, &nodeSum, 1, MPI_INT, MPI_SUM, node);
        EXPECT(nodeSum == nodeSize);
        msg.set_outputdata("node of " + std::to_string(nodeSize));
        MPI_Comm_free(&node);
        MPI_Comm_free(&half);
        return 0;
    });

    // One-sided communication: puts and gets to every rank of the world, in
    // this process (direct copies) or another one (shipped at the fence)
    mpiFunction("rma", [](int rank, int size, faabric::Message& msg) {
        const int n = size + 2;
        std::vector<long> window(n, -1);
        MPI_Win win = nullptr;
        MPI_Win_create(window.data(), n * sizeof(long), sizeof(long), MPI_INFO_NULL, MPI_COMM_WORLD, &win);
        MPI_Win_fence(0, win);
        long mine = 100 + rank;
        for (int t = 0; t < size; t++) {
            MPI_Put(&mine, 1, MPI_LONG, t, rank, 1, MPI_LONG, win);
        }
        MPI_Win_fence(0, win);
        for (int r = 0; r < size; r++) {
            EXPECT(window[r] == 100 + r);
        }
        // second epoch: everybody reads everybody's last-but-one slot and
        // streams a large strip into the next rank
        window[size] = 9000 + rank;
        const int big = 300000;
        std::vector<long> strip(big, rank), landing(big, -1);
        MPI_Win bigWin = nullptr;
        MPI_Win_create(landing.data(), big * sizeof(long), sizeof(long), MPI_INFO_NULL, MPI_COMM_WORLD, &bigWin);
        MPI_Win_fence(0, win);
        MPI_Win_fence(0, bigWin);
        std::vector<long> seen(size, 0);
        for (int t = 0; t < size; t++) {
            MPI_Get(&seen[t], 1, MPI_LONG, t, size, 1, MPI_LONG, win);
        }
        MPI_Put(strip.data(), big, MPI_LONG, (rank + 1) % size, 0, big, MPI_LONG, bigWin);
        MPI_Win_fence(0, bigWin);
        MPI_Win_fence(0, win);
        for (int t = 0; t < size; t++) {
            EXPECT(seen[t] == 9000 + t);
        }
        int left = (rank + size - 1) % size;
        EXPECT(landing[0] == left && landing[big - 1] == left);
        MPI_Win_free(&bigWin);
        MPI_Win_free(&win);
        // shared windows need one address space
        long* shared = nullptr;
        MPI_Win sharedWin = nullptr;
        int rc = MPI_Win_allocate_shared(64, 8, MPI_INFO_NULL, MPI_COMM_WORLD, &shared, &sharedWin);
        bool oneProcess = faabric::mpi::getMpiWorldRegistry().getWorld(msg.mpiworldid()).allRanksLocal();
        EXPECT((rc == MPI_SUCCESS) == oneProcess);
        if (rc == MPI_SUCCESS) {
            MPI_Win_free(&sharedWin);
        }
        return 0;
    });

    // One-sided atomics from every rank onto every rank's window, in this
    // process or another one (shipped and applied at the fence).  Input:
    // "host" | "cuda" | "heap" window memory, then ",device" for origin and
    // result buffers in cudaMalloc memory.
    mpiFunction("rma-atomics", [](int rank, int size, faabric::Message& msg) {
        const std::string& in = msg.inputdata();
        rma_atomics::Setup s;
        s.window = in.rfind("cuda", 0) == 0   ? rma_atomics::WindowMemory::CudaMalloc
                   : in.rfind("heap", 0) == 0 ? rma_atomics::WindowMemory::Heap
                                              : rma_atomics::WindowMemory::Host;
        s.deviceBuffers = in.find(",device") != std::string::npos;
        std::string why;
        int rc = rma_atomics::body(rank, size, msg.mpiworldid(), s, &why);
        if (rc != 0) {
            SPDLOG_ERROR("rma-atomics: {}", why);
            msg.set_outputdata(why);
        }
        return rc;
    });

    // Passive-target synchronisation (locks, flushes, lock-all) with origins
    // in the target's process and in other ones; shipped operations are
    // applied by the target's point-to-point server, no fence.  Input as for
    // rma-atomics.
    mpiFunction("rma-passive", [](int rank, int size, faabric::Message& msg) {
        const std::string& in = msg.inputdata();
        rma_passive::Setup s;
        s.window = in.rfind("cuda", 0) == 0   ? rma_passive::WindowMemory::CudaMalloc
                   : in.rfind("heap", 0) == 0 ? rma_passive::WindowMemory::Heap
                                              : rma_passive::WindowMemory::Host;
        s.deviceBuffers = in.find(",device") != std::string::npos;
        std::string why;
        int rc = rma_passive::body(rank, size, msg.mpiworldid(), s, &why);
        if (rc != 0) {
            SPDLOG_ERROR("rma-passive: {}", why);
            msg.set_outputdata(why);
        }
        return rc;
    });

    // Request-based one-sided operations (MPI_Rput, MPI_Rget, MPI_Raccumulate,
    // MPI_Rget_accumulate) with targets in this process and in other ones.
    // Input: "host" | "cuda" | "heap" window memory, then ",device" for
    // origin and result buffers in cudaMalloc memory or ",heapbuf" for
    // buffers in the origin's symmetric heap.
    mpiFunction("rma-request", [](int rank, int size, faabric::Message& msg) {
        const std::string& in = msg.inputdata();
        rma_request::Setup s;
        s.window = in.rfind("cuda", 0) == 0   ? rma_request::WindowMemory::CudaMalloc
                   : in.rfind("heap", 0) == 0 ? rma_request::WindowMemory::Heap
                                              : rma_request::WindowMemory::Host;
        s.origin = in.find(",device") != std::string::npos    ? rma_request::Origin::Device
                   : in.find(",heapbuf") != std::string::npos ? rma_request::Origin::Heap
                                                              : rma_request::Origin::Host;
        std::string why;
        int rc = rma_request::body(rank, size, msg.mpiworldid(), s, &why);
        if (rc != 0) {
            SPDLOG_ERROR("rma-request: {}", why);
            msg.set_outputdata(why);
        }
        return rc;
    });

    // Fused device collectives on sub-communicators (mpi_subcomm_device_body.h).
    // Input: "heap" (symmetric heap buffers) or "cuda" (cudaMalloc buffers).
    mpiFunction("subcomm-device", [](int rank, int size, faabric::Message& msg) {
        subcomm_device::Setup s;
        s.memory = msg.inputdata().rfind("cuda", 0) == 0 ? subcomm_device::BufferMemory::CudaMalloc
                                                          : subcomm_device::BufferMemory::Heap;
        std::string why;
        int rc = subcomm_device::body(rank, size, msg.mpiworldid(), s, &why);
        if (rc != 0) {
            SPDLOG_ERROR("subcomm-device: {}", why);
            msg.set_outputdata(why);
        }
        return rc;
    });

    // MPI_Allreduce (float32 SUM) on symmetric-heap buffers.  Input:
    // "<mode>;<bytes>;<iters>" with mode
    //   fused  on the half communicator of this rank (ranks [0, size/2) and
    //          [size/2, size)): the fused kernels on a signal slot
    //   host   the same, after FB_SUB_SLOTS world splits have taken every slot:
    //          the point-to-point host path
    //   world  on MPI_COMM_WORLD
    // Rank 0 reports {"us_per_call", "device_calls"}: the device collectives
    // of rank 0's process per timed call (one per rank of the process when the
    // call is fused, 0 on the host path).
    mpiFunction("bench-subcomm", [](int rank, int size, faabric::Message& msg) {
        std::vector<std::string> f;
        std::string cur;
        for (char c : msg.inputdata() + ";") {
            if (c == ';') {
                f.push_back(cur);
                cur.clear();
            } else {
                cur += c;
            }
        }
        EXPECT(f.size() >= 3 && size >= 2);
        const std::string mode = f[0];
        const size_t bytes = std::stoul(f[1]);
        const int iters = std::stoi(f[2]);
        const int count = (int)(bytes / 4);
        faabric::mpi::MpiWorld& world = faabric::mpi::getMpiWorldRegistry().getWorld(msg.mpiworldid());
        float* send = nullptr;
        float* recv = nullptr;
        EXPECT(MPI_Alloc_mem(bytes, MPI_INFO_FAABRIC_DEVICE, &send) == MPI_SUCCESS);
        EXPECT(MPI_Alloc_mem(bytes, MPI_INFO_FAABRIC_DEVICE, &recv) == MPI_SUCCESS);
        std::vector<float> ones(count, 1.0f);
        cudaMemcpy(send, ones.data(), bytes, cudaMemcpyHostToDevice);
        std::vector<MPI_Comm> fill;
        if (mode == "host") {
            for (int i = 0; i < FB_SUB_SLOTS; i++) {
                MPI_Comm c = MPI_COMM_NULL;
                MPI_Comm_split(MPI_COMM_WORLD, 0, rank, &c);
                // (a device call: takes a slot)
                EXPECT(MPI_Allreduce(send, recv, 4, MPI_FLOAT, MPI_SUM, c) == MPI_SUCCESS);
                fill.push_back(c);
            }
        }
        MPI_Comm comm = MPI_COMM_WORLD;
        if (mode != "world") {
            MPI_Comm_split(MPI_COMM_WORLD, rank / (size / 2), rank, &comm);
        }
        int n = 0;
        MPI_Comm_size(comm, &n);
        for (int i = 0; i < 3; i++) {
            EXPECT(MPI_Allreduce(send, recv, count, MPI_FLOAT, MPI_SUM, comm) == MPI_SUCCESS);
        }
        std::vector<float> out(count);
        cudaMemcpy(out.data(), recv, bytes, cudaMemcpyDeviceToHost);
        EXPECT(out[0] == (float)n && out[count - 1] == (float)n);
        MPI_Barrier(MPI_COMM_WORLD);
        const uint64_t before = world.getDeviceCollectiveCount();
        MPI_Barrier(MPI_COMM_WORLD);
        auto t0 = std::chrono::steady_clock::now();
        for (int i = 0; i < iters; i++) {
            EXPECT(MPI_Allreduce(send, recv, count, MPI_FLOAT, MPI_SUM, comm) == MPI_SUCCESS);
        }
        const double us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count() / iters;
        MPI_Barrier(MPI_COMM_WORLD);
        const uint64_t calls = world.getDeviceCollectiveCount() - before;
        if (rank == 0) {
            msg.set_outputdata("{\"us_per_call\": " + std::to_string(us) +
                               ", \"device_calls\": " + std::to_string((double)calls / iters) + "}");
        }
        if (comm != MPI_COMM_WORLD) {
            MPI_Comm_free(&comm);
        }
        for (MPI_Comm& c : fill) {
            MPI_Comm_free(&c);
        }
        MPI_Free_mem(send);
        MPI_Free_mem(recv);
        return 0;
    });

    // Cost of the MPI one-sided atomics, rank 0 onto rank 1's window, each
    // call followed by its closing fence.  Input:
    // "fop|acc;<i32|f32|i64>;<bytes>;<iters>;<heap|cuda>;<host|device>".
    // Rank 0 reports {"us_per_call", "gb_per_s"}.
    mpiFunction("bench-rma", [](int rank, int size, faabric::Message& msg) {
        std::vector<std::string> f;
        std::string cur;
        for (char c : msg.inputdata() + ";") {
            if (c == ';') {
                f.push_back(cur);
                cur.clear();
            } else {
                cur += c;
            }
        }
        EXPECT(f.size() >= 6 && size >= 2);
        const bool fop = f[0] == "fop";
        MPI_Datatype dt = f[1] == "f32" ? MPI_FLOAT : (f[1] == "i64" ? MPI_INT64_T : MPI_INT);
        const size_t bytes = std::stoul(f[2]);
        const int iters = std::stoi(f[3]);
        const bool heap = f[4] == "heap";
        const bool devBuf = f[5] == "device";
        const int count = (int)(bytes / dt->size);
        uint8_t* window = nullptr;
        if (heap) {
            EXPECT(MPI_Alloc_mem(bytes, MPI_INFO_FAABRIC_DEVICE, &window) == MPI_SUCCESS);
        } else {
            EXPECT(cudaMalloc((void**)&window, bytes) == cudaSuccess);
        }
        cudaMemset(window, 0, bytes);
        cudaDeviceSynchronize();
        // ones: an add that leaves the target unchanged skips its write on the
        // CAS paths and would time faster than real work
        std::vector<uint8_t> hostOrigin(bytes, 0), hostResult(bytes, 0);
        for (size_t i = 0; i + dt->size <= bytes; i += dt->size) {
            const float f = 1.0f;
            const int64_t one = 1;
            memcpy(hostOrigin.data() + i, dt == MPI_FLOAT ? (const void*)&f : (const void*)&one, dt->size);
        }
        uint8_t* origin = hostOrigin.data();
        uint8_t* result = hostResult.data();
        if (devBuf) {
            EXPECT(cudaMalloc((void**)&origin, bytes) == cudaSuccess && cudaMalloc((void**)&result, bytes) == cudaSuccess);
            cudaMemcpy(origin, hostOrigin.data(), bytes, cudaMemcpyHostToDevice);
            cudaDeviceSynchronize();
        }
        MPI_Win win = nullptr;
        MPI_Win_create(window, bytes, 1, MPI_INFO_NULL, MPI_COMM_WORLD, &win);
        MPI_Win_fence(0, win);
        auto issue = [&]() {
            if (rank != 0) {
                return MPI_SUCCESS;
            }
            return fop ? MPI_Fetch_and_op(origin, result, dt, 1, 0, MPI_SUM, win)
                       : MPI_Accumulate(origin, count, dt, 1, 0, count, dt, MPI_SUM, win);
        };
        for (int i = 0; i < 3; i++) {
            EXPECT(issue() == MPI_SUCCESS);
            MPI_Win_fence(0, win);
        }
        auto t0 = std::chrono::steady_clock::now();
        for (int i = 0; i < iters; i++) {
            EXPECT(issue() == MPI_SUCCESS);
            MPI_Win_fence(0, win);
        }
        double us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count() / iters;
        if (rank == 0) {
            msg.set_outputdata("{\"us_per_call\": " + std::to_string(us) +
                               ", \"gb_per_s\": " + std::to_string((double)bytes / (us * 1e3)) + "}");
        }
        MPI_Win_free(&win);
        if (devBuf) {
            cudaFree(origin);
            cudaFree(result);
        }
        if (heap) {
            MPI_Free_mem(window);
        } else {
            cudaFree(window);
        }
        return 0;
    });

    // Cost of passive-target synchronisation, rank 0 onto rank 1's 8-byte
    // window.  Input: "<mode>;<heap|cuda|host>;<host|device>;<iters>" with mode
    //   flush  MPI_Fetch_and_op + MPI_Win_flush inside MPI_Win_lock_all
    //   fence  MPI_Fetch_and_op + MPI_Win_fence (the same call, fence-based)
    //   lock   MPI_Win_lock(EXCLUSIVE) + MPI_Win_unlock, nothing in between
    // Rank 0 reports {"us_per_call"}.
    mpiFunction("bench-rma-passive", [](int rank, int size, faabric::Message& msg) {
        std::vector<std::string> f;
        std::string cur;
        for (char c : msg.inputdata() + ";") {
            if (c == ';') {
                f.push_back(cur);
                cur.clear();
            } else {
                cur += c;
            }
        }
        EXPECT(f.size() >= 4 && size >= 2);
        const std::string mode = f[0];
        const int iters = std::stoi(f[3]);
        const bool devBuf = f[2] == "device";
        uint8_t* window = nullptr;
        if (f[1] == "heap") {
            EXPECT(MPI_Alloc_mem(8, MPI_INFO_FAABRIC_DEVICE, &window) == MPI_SUCCESS);
            cudaMemset(window, 0, 8);
        } else if (f[1] == "cuda") {
            EXPECT(cudaMalloc((void**)&window, 8) == cudaSuccess);
            cudaMemset(window, 0, 8);
        } else {
            window = (uint8_t*)calloc(1, 8);
        }
        cudaDeviceSynchronize();
        int64_t hostBufs[2] = { 1, 0 };
        int64_t* bufs = hostBufs;
        if (devBuf) {
            EXPECT(cudaMalloc((void**)&bufs, 16) == cudaSuccess);
            cudaMemcpy(bufs, hostBufs, 16, cudaMemcpyHostToDevice);
            cudaDeviceSynchronize();
        }
        MPI_Win win = nullptr;
        MPI_Win_create(window, 8, 1, MPI_INFO_NULL, MPI_COMM_WORLD, &win);
        auto step = [&]() {
            if (mode == "fence") {
                int rc = rank == 0 ? MPI_Fetch_and_op(bufs, bufs + 1, MPI_INT64_T, 1, 0, MPI_SUM, win) : MPI_SUCCESS;
                return rc == MPI_SUCCESS ? MPI_Win_fence(0, win) : rc;
            }
            if (rank != 0) {
                return MPI_SUCCESS;
            }
            if (mode == "lock") {
                int rc = MPI_Win_lock(MPI_LOCK_EXCLUSIVE, 1, 0, win);
                return rc == MPI_SUCCESS ? MPI_Win_unlock(1, win) : rc;
            }
            int rc = MPI_Fetch_and_op(bufs, bufs + 1, MPI_INT64_T, 1, 0, MPI_SUM, win);
            return rc == MPI_SUCCESS ? MPI_Win_flush(1, win) : rc;
        };
        const bool epoch = mode == "flush" && rank == 0;
        if (epoch) {
            EXPECT(MPI_Win_lock_all(0, win) == MPI_SUCCESS);
        }
        for (int i = 0; i < 3; i++) {
            EXPECT(step() == MPI_SUCCESS);
        }
        auto t0 = std::chrono::steady_clock::now();
        for (int i = 0; i < iters; i++) {
            EXPECT(step() == MPI_SUCCESS);
        }
        double us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count() / iters;
        if (epoch) {
            EXPECT(MPI_Win_unlock_all(win) == MPI_SUCCESS);
        }
        if (rank == 0) {
            msg.set_outputdata("{\"us_per_call\": " + std::to_string(us) + "}");
        }
        MPI_Win_free(&win);
        if (devBuf) {
            cudaFree(bufs);
        }
        if (f[1] == "heap") {
            MPI_Free_mem(window);
        } else if (f[1] == "cuda") {
            cudaFree(window);
        } else {
            free(window);
        }
        return 0;
    });

    // Cost of request-based puts against plain ones: rank 0 writes K
    // operations of B bytes from device memory into rank 1's symmetric-heap
    // window inside MPI_Win_lock_all, then completes them.  Input
    // "mode;B;K;iters":
    //   rput  MPI_Rput x K + MPI_Waitall + MPI_Win_flush
    //   put   MPI_Put x K + MPI_Win_flush
    // Operation k goes to slot k of the window (slots wrap at 16 MiB).  Rank 0
    // reports {"us_per_op"}.
    mpiFunction("bench-rma-request", [](int rank, int size, faabric::Message& msg) {
        std::vector<std::string> f;
        std::string cur;
        for (char c : msg.inputdata() + ";") {
            if (c == ';') {
                f.push_back(cur);
                cur.clear();
            } else {
                cur += c;
            }
        }
        EXPECT(f.size() >= 4 && size >= 2);
        const bool rput = f[0] == "rput";
        const size_t bytes = std::stoull(f[1]);
        const int K = std::stoi(f[2]);
        const int iters = std::stoi(f[3]);
        EXPECT(bytes > 0 && bytes <= ((size_t)16 << 20) && K > 0 && iters > 0);
        const size_t slots = std::min<size_t>((size_t)K, ((size_t)16 << 20) / bytes);
        const size_t winBytes = slots * bytes;
        uint8_t* window = nullptr;
        EXPECT(MPI_Alloc_mem(winBytes, MPI_INFO_FAABRIC_DEVICE, &window) == MPI_SUCCESS);
        uint8_t* src = nullptr;
        EXPECT(cudaMalloc((void**)&src, (size_t)K * bytes) == cudaSuccess);
        cudaMemset(src, rank + 1, (size_t)K * bytes);
        cudaMemset(window, 0, winBytes);
        cudaDeviceSynchronize();
        MPI_Win win = nullptr;
        MPI_Win_create(window, winBytes, 1, MPI_INFO_NULL, MPI_COMM_WORLD, &win);
        std::vector<MPI_Request> reqs(K, nullptr);
        auto step = [&]() {
            for (int k = 0; k < K; k++) {
                const uint8_t* o = src + (size_t)k * bytes;
                const MPI_Aint disp = (MPI_Aint)((k % slots) * bytes);
                int rc = rput ? MPI_Rput(o, (int)bytes, MPI_BYTE, 1, disp, (int)bytes, MPI_BYTE, win, &reqs[k])
                              : MPI_Put(o, (int)bytes, MPI_BYTE, 1, disp, (int)bytes, MPI_BYTE, win);
                if (rc != MPI_SUCCESS) {
                    return rc;
                }
            }
            if (rput) {
                int rc = MPI_Waitall(K, reqs.data(), MPI_STATUSES_IGNORE);
                if (rc != MPI_SUCCESS) {
                    return rc;
                }
            }
            return MPI_Win_flush(1, win);
        };
        double us = 0;
        if (rank == 0) {
            EXPECT(MPI_Win_lock_all(0, win) == MPI_SUCCESS);
            for (int i = 0; i < 3; i++) {
                EXPECT(step() == MPI_SUCCESS);
            }
            auto t0 = std::chrono::steady_clock::now();
            for (int i = 0; i < iters; i++) {
                EXPECT(step() == MPI_SUCCESS);
            }
            us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count() / ((double)iters * K);
            EXPECT(MPI_Win_unlock_all(win) == MPI_SUCCESS);
            msg.set_outputdata("{\"us_per_op\": " + std::to_string(us) + "}");
        }
        MPI_Win_free(&win);
        if (rank == 1) {
            // what arrived is rank 0's bytes
            std::vector<uint8_t> got(winBytes);
            cudaMemcpy(got.data(), window, winBytes, cudaMemcpyDeviceToHost);
            EXPECT(std::all_of(got.begin(), got.end(), [](uint8_t b) { return b == 1; }));
        }
        cudaFree(src);
        MPI_Free_mem(window);
        return 0;
    });

    // Iterates with an all-reduce per loop; halfway through every rank hits a
    // migration point.  Ranks that are moved resume from the loop index they
    // carried over, with their memory restored from the snapshot.
    mpiFunction("migrate", [](int rank, int size, faabric::Message& msg) {
        const int nLoops = 6, checkAt = 3;
        int start = msg.inputdata().empty() ? 0 : std::stoi(msg.inputdata());
        auto mem = ExecutorContext::get()->getExecutor()->getMemoryView();
        int* cell = (int*)(mem.data() + 256);
        if (start == 0) {
            *cell = 4000 + rank;
        } else {
            EXPECT(*cell == 4000 + rank);
        }
        for (int i = start; i < nLoops; i++) {
            if (i == checkAt && start == 0) {
                // Give the test time to change the cluster under us: a fixed
                // pause, or (cmdline = path) until the test creates that file
                if (msg.cmdline().empty()) {
                    std::this_thread::sleep_for(std::chrono::milliseconds(300));
                } else {
                    for (int waited = 0; waited < 30000 && ::access(msg.cmdline().c_str(), F_OK) != 0; waited += 5) {
                        std::this_thread::sleep_for(std::chrono::milliseconds(5));
                    }
                }
                MPI_Barrier(MPI_COMM_WORLD);
                faabric::mpi::mpiMigrationPoint(i);
            }
            int v = rank + i, sum = 0;
            MPI_Allreduce(&v, &sum, 1, MPI_INT, MPI_SUM, MPI_COMM_WORLD);
            EXPECT(sum == size * (size - 1) / 2 + i * size);
        }
        MPI_Barrier(MPI_COMM_WORLD);
        msg.set_outputdata(start == 0 ? "stayed" : "resumed at " + std::to_string(start));
        return 0;
    });

    // ---- CPU baselines (BASELINE.md configs) ----
    // Ping-pong between ranks 0 and 1; reports the mean round-trip in us
    mpiFunction("bench-pingpong", [](int rank, int size, faabric::Message& msg) {
        int bytes = msg.inputdata().empty() ? 8 : std::stoi(msg.inputdata());
        const int iters = 2000, warmup = 200;
        std::vector<uint8_t> buf((size_t)bytes, 1);
        std::chrono::steady_clock::time_point t0;
        for (int i = 0; i < iters + warmup; i++) {
            if (i == warmup) {
                t0 = std::chrono::steady_clock::now();
            }
            if (rank == 0) {
                MPI_Send(buf.data(), bytes, MPI_BYTE, 1, 0, MPI_COMM_WORLD);
                MPI_Recv(buf.data(), bytes, MPI_BYTE, 1, 0, MPI_COMM_WORLD, MPI_STATUS_IGNORE);
            } else if (rank == 1) {
                MPI_Recv(buf.data(), bytes, MPI_BYTE, 0, 0, MPI_COMM_WORLD, MPI_STATUS_IGNORE);
                MPI_Send(buf.data(), bytes, MPI_BYTE, 0, 0, MPI_COMM_WORLD);
            }
        }
        double us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count() / iters;
        if (rank == 0) {
            msg.set_outputdata("{\"bytes\": " + std::to_string(bytes) + ", \"rtt_us\": " + std::to_string(us) + "}");
        }
        return 0;
    });

    // Headline workload through the MPI C API: one MPI_Allreduce per tensor.
    // Input: "steps;warmup;host|device;n1,n2,..." (element counts).
    //  host   = the reference's design (reduce to rank 0 + broadcast over
    //           in-memory queues, malloc+memcpy per hop)
    //  device = buffers in HBM, every call is one fused P2P/NVLS kernel
    mpiFunction("bench-allreduce-list", [](int rank, int size, faabric::Message& msg) {
        const std::string& in = msg.inputdata();
        size_t s1 = in.find(';'), s2 = in.find(';', s1 + 1), s3 = in.find(';', s2 + 1);
        int steps = std::stoi(in.substr(0, s1));
        int warmup = std::stoi(in.substr(s1 + 1, s2 - s1 - 1));
        // host | device (cudaMalloc) | symmetric (MPI_Alloc_mem in the
        // symmetric heap) | symmetric-nb (same + MPI_Iallreduce/Waitall)
        std::string memory = in.substr(s2 + 1, s3 - s2 - 1);
        bool onDevice = memory != "host";
        bool symmetric = memory.rfind("symmetric", 0) == 0;
        bool nonBlocking = memory == "symmetric-nb";
        std::vector<size_t> counts;
        size_t pos = s3 + 1;
        while (pos < in.size()) {
            size_t comma = in.find(',', pos);
            counts.push_back(std::stoul(in.substr(pos, comma - pos)));
            if (comma == std::string::npos) {
                break;
            }
            pos = comma + 1;
        }
        size_t total = std::accumulate(counts.begin(), counts.end(), (size_t)0);
        std::vector<int> hostGrads(total, rank + 1), hostOut(total, 0);
        int* grads = hostGrads.data();
        int* out = hostOut.data();
        if (onDevice) {
            auto& world = faabric::mpi::getMpiWorldRegistry().getWorld(msg.mpiworldid());
            auto comm = world.getDeviceComm(rank);
            if (comm == nullptr) {
                msg.set_outputdata("no device communicator for rank " + std::to_string(rank));
                return 1;
            }
            cudaSetDevice(comm->device());
            bool ok;
            if (symmetric) {
                ok = MPI_Alloc_mem(total * sizeof(int), MPI_INFO_FAABRIC_DEVICE, &grads) == MPI_SUCCESS &&
                     MPI_Alloc_mem(total * sizeof(int), MPI_INFO_FAABRIC_DEVICE, &out) == MPI_SUCCESS;
            } else {
                ok = cudaMalloc(&grads, total * sizeof(int)) == cudaSuccess && cudaMalloc(&out, total * sizeof(int)) == cudaSuccess;
            }
            if (!ok) {
                msg.set_outputdata("device allocation failed (FAABRIC_SYMM_HEAP_BYTES too small?)");
                return 1;
            }
            if (faabric::device::Communicator::isLoopbackHeapPointer(grads)) {
                memcpy(grads, hostGrads.data(), total * sizeof(int)); // loopback backend: the heap is host memory
            } else {
                cudaMemcpy(grads, hostGrads.data(), total * sizeof(int), cudaMemcpyHostToDevice);
            }
        }
        std::vector<MPI_Request> reqs(counts.size());
        std::chrono::steady_clock::time_point t0;
        double issueMs = 0, waitMs = 0;
        uint64_t launches0 = 0;
        std::shared_ptr<faabric::device::Communicator> devComm;
        if (onDevice) {
            devComm = faabric::mpi::getMpiWorldRegistry().getWorld(msg.mpiworldid()).getDeviceComm(rank);
        }
        for (int it = 0; it < warmup + steps; it++) {
            if (it == warmup) {
                MPI_Barrier(MPI_COMM_WORLD);
                launches0 = devComm ? devComm->stats().launches : 0;
                t0 = std::chrono::steady_clock::now();
            }
            auto a0 = std::chrono::steady_clock::now();
            size_t off = 0;
            for (size_t i = 0; i < counts.size(); i++) {
                if (nonBlocking) {
                    MPI_Iallreduce(grads + off, out + off, (int)counts[i], MPI_INT, MPI_SUM, MPI_COMM_WORLD, &reqs[i]);
                } else {
                    MPI_Allreduce(grads + off, out + off, (int)counts[i], MPI_INT, MPI_SUM, MPI_COMM_WORLD);
                }
                off += counts[i];
            }
            auto a1 = std::chrono::steady_clock::now();
            if (nonBlocking) {
                MPI_Waitall((int)reqs.size(), reqs.data(), MPI_STATUSES_IGNORE);
            }
            auto a2 = std::chrono::steady_clock::now();
            if (it >= warmup) {
                issueMs += std::chrono::duration<double, std::milli>(a1 - a0).count();
                waitMs += std::chrono::duration<double, std::milli>(a2 - a1).count();
            }
        }
        const uint64_t launches = devComm ? devComm->stats().launches - launches0 : 0;
        MPI_Barrier(MPI_COMM_WORLD);
        double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count() / steps;
        if (onDevice) {
            if (faabric::device::Communicator::isLoopbackHeapPointer(out)) {
                memcpy(hostOut.data(), out, total * sizeof(int));
            } else {
                cudaMemcpy(hostOut.data(), out, total * sizeof(int), cudaMemcpyDeviceToHost);
            }
            if (symmetric) {
                MPI_Free_mem(grads);
                MPI_Free_mem(out);
            } else {
                cudaFree(grads);
                cudaFree(out);
            }
        }
        {
            // every tensor's first and last element
            size_t off = 0;
            for (size_t c : counts) {
                EXPECT(hostOut[off] == size * (size + 1) / 2 && hostOut[off + c - 1] == hostOut[off]);
                off += c;
            }
        }
        if (rank == 0) {
            double gbps = (double)total * 4 / (ms * 1e-3) / 1e9;
            msg.set_outputdata("{\"tensors\": " + std::to_string(counts.size()) + ", \"elements\": " + std::to_string(total) +
                               ", \"memory\": \"" + memory + "\", \"ms_per_step\": " + std::to_string(ms) +
                               ", \"issue_ms_per_step\": " + std::to_string(issueMs / steps) +
                               ", \"wait_ms_per_step\": " + std::to_string(waitMs / steps) +
                               ", \"kernel_launches_per_step\": " + std::to_string((double)launches / steps) +
                               ", \"algbw_GBps\": " + std::to_string(gbps) + "}");
        }
        return 0;
    });

    // The headline: one "step" of ResNet-50 gradient sync = one int32
    // MPI_Allreduce per parameter tensor, on host memory (reference CPU path)
    // Host-buffer collectives, "bytesPerRank[,steps]": microseconds per call
    mpiFunction("bench-collectives", [](int rank, int size, faabric::Message& msg) {
        size_t bytes = 1 << 20;
        int steps = 20;
        if (!msg.inputdata().empty()) {
            auto comma = msg.inputdata().find(',');
            bytes = std::stoul(msg.inputdata().substr(0, comma));
            if (comma != std::string::npos) {
                steps = std::stoi(msg.inputdata().substr(comma + 1));
            }
        }
        const int n = (int)(bytes / sizeof(int));
        std::vector<int> mine(n, rank + 1), big((size_t)n * size, 0), other((size_t)n * size, rank);
        std::string json = "{\"bytes_per_rank\": " + std::to_string(bytes) + ", \"ranks\": " + std::to_string(size);
        auto timeIt = [&](const char* name, const std::function<void()>& call) {
            call();
            MPI_Barrier(MPI_COMM_WORLD);
            auto t0 = std::chrono::steady_clock::now();
            for (int i = 0; i < steps; i++) {
                call();
            }
            MPI_Barrier(MPI_COMM_WORLD);
            double us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count() / steps;
            json += std::string(", \"") + name + "_us\": " + std::to_string(us);
        };
        timeIt("bcast", [&] { MPI_Bcast(mine.data(), n, MPI_INT, 0, MPI_COMM_WORLD); });
        timeIt("reduce", [&] { MPI_Reduce(mine.data(), big.data(), n, MPI_INT, MPI_SUM, 0, MPI_COMM_WORLD); });
        timeIt("allreduce", [&] { MPI_Allreduce(mine.data(), big.data(), n, MPI_INT, MPI_SUM, MPI_COMM_WORLD); });
        timeIt("gather", [&] { MPI_Gather(mine.data(), n, MPI_INT, big.data(), n, MPI_INT, 0, MPI_COMM_WORLD); });
        timeIt("scatter", [&] { MPI_Scatter(other.data(), n, MPI_INT, mine.data(), n, MPI_INT, 0, MPI_COMM_WORLD); });
        timeIt("allgather", [&] { MPI_Allgather(mine.data(), n, MPI_INT, big.data(), n, MPI_INT, MPI_COMM_WORLD); });
        timeIt("alltoall", [&] { MPI_Alltoall(other.data(), n, MPI_INT, big.data(), n, MPI_INT, MPI_COMM_WORLD); });
        if (rank == 0) {
            msg.set_outputdata(json + "}");
        }
        return 0;
    });

    mpiFunction("bench-allreduce", [](int rank, int size, faabric::Message& msg) {
        // "count[,steps]" in elements; default: a 25.6M-element model in 214
        // tensors is driven from Python, this is the single-size kernel
        size_t count = 1 << 20;
        int steps = 20;
        if (!msg.inputdata().empty()) {
            auto comma = msg.inputdata().find(',');
            count = std::stoul(msg.inputdata().substr(0, comma));
            if (comma != std::string::npos) {
                steps = std::stoi(msg.inputdata().substr(comma + 1));
            }
        }
        std::vector<int> v(count, rank + 1), out(count, 0);
        MPI_Allreduce(v.data(), out.data(), (int)count, MPI_INT, MPI_SUM, MPI_COMM_WORLD);
        MPI_Barrier(MPI_COMM_WORLD);
        auto t0 = std::chrono::steady_clock::now();
        for (int i = 0; i < steps; i++) {
            MPI_Allreduce(v.data(), out.data(), (int)count, MPI_INT, MPI_SUM, MPI_COMM_WORLD);
        }
        double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count() / steps;
        EXPECT(out[count - 1] == size * (size + 1) / 2);
        if (rank == 0) {
            double gbps = (double)count * 4 / (ms * 1e-3) / 1e9;
            msg.set_outputdata("{\"count\": " + std::to_string(count) + ", \"ms\": " + std::to_string(ms) +
                               ", \"algbw_GBps\": " + std::to_string(gbps) + "}");
        }
        return 0;
    });
}

class WorkerExecutor : public Executor
{
  public:
    explicit WorkerExecutor(faabric::Message& msg)
      : Executor(msg)
    {
        // A small linear memory so functions can be snapshotted / migrated
        memory = faabric::util::allocatePrivateMemory(MEMORY_BYTES);
    }

    int32_t executeTask(int threadPoolIdx, int msgIdx, std::shared_ptr<faabric::BatchExecuteRequest> req) override
    {
        auto& msg = *req->mutable_messages(msgIdx);
        auto it = functions().find(msg.user() + "/" + msg.function());
        if (it == functions().end()) {
            msg.set_outputdata("Unknown function " + msg.user() + "/" + msg.function());
            return 1;
        }
        return it->second(msg);
    }

    std::span<uint8_t> getMemoryView() override { return { memory.get(), MEMORY_BYTES }; }

    size_t getMaxMemorySize() override { return MEMORY_BYTES; }

    void restore(const std::string& snapshotKey) override
    {
        auto snap = reg.getSnapshot(snapshotKey);
        snap->mapToMemory({ memory.get(), std::min(MEMORY_BYTES, snap->getSize()) });
    }

  private:
    static constexpr size_t MEMORY_BYTES = 64 * 4096;
    faabric::util::MemoryRegion memory;
};

class WorkerExecutorFactory : public ExecutorFactory
{
  protected:
    std::shared_ptr<Executor> createExecutor(faabric::Message& msg) override
    {
        return std::make_shared<WorkerExecutor>(msg);
    }
};

int main()
{
    faabric::util::initLogging();
    faabric::util::exitWithParentIfAsked();
    registerFunctions();
    auto& conf = faabric::util::getSystemConfig();
    SPDLOG_INFO("Starting worker {} (port offset {}), planner at {}", conf.endpointHost, conf.portOffset, conf.plannerHost);

    faabric::runner::FaabricMain m(std::make_shared<WorkerExecutorFactory>());
    m.startBackground();

    // Port 0: workers take no HTTP requests, the endpoint only gives us
    // signal-driven shutdown
    faabric::endpoint::FaabricEndpoint endpoint(0, 1, std::make_shared<faabric::endpoint::FaabricEndpointHandler>());
    endpoint.start(faabric::endpoint::EndpointMode::SIGNAL);

    SPDLOG_INFO("Shutting down worker");
    m.shutdown();
    return 0;
}
