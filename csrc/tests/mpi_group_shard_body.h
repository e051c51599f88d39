// One MPI program that checks MPI_Ireduce_scatter_block, MPI_Iallgather and
// MPI_Reduce_scatter_block on every kind of buffer.  Shared by the loopback
// test (test_loopback_group_shard.cpp) and the GPU test
// (test_device_group_shard.cpp).
//
// Bursts on MPI_Alloc_mem(MPI_INFO_FAABRIC_DEVICE) memory must go out as ONE
// grouped launch per burst (this rank's communicator counts launches), a
// burst of another kind must flush the pending one, and every result is
// compared exactly against a closed form computed on the host.
#pragma once

#include "mpi_subcomm_device_body.h"

#include <faabric/mpi/MpiWorld.h>
#include <faabric/mpi/MpiWorldRegistry.h>
#include <faabric/mpi/mpi.h>

#include <cstdint>
#include <string>
#include <vector>

namespace group_shard {

using subcomm_device::BufferMemory;
using subcomm_device::DevBuffer;

#define GS_CHECK(cond)                                                         \
    do {                                                                       \
        if (!(cond)) {                                                         \
            *why = "rank " + std::to_string(rank) + ": check failed at line " + std::to_string(__LINE__) + ": " #cond; \
            return 1;                                                          \
        }                                                                      \
    } while (0)

constexpr int T = 12;    // tensors per burst
constexpr int MAXC = 64; // int32 elements per shard at most

// Shard of tensor t: a multiple of 4 int32 (16 bytes), different per tensor
inline int shardOf(int t)
{
    return 4 * (1 + t % 16);
}

// Reduce-scatter input of rank p, tensor t, element i of its size*c elements
inline int32_t rsIn(int p, int t, int i)
{
    return p * 7 + t * 3 + i;
}

// Sum over the ranks of shard r, element j
inline int32_t rsOut(int size, int r, int t, int j)
{
    return 7 * size * (size - 1) / 2 + size * (t * 3 + r * shardOf(t) + j);
}

inline int32_t agIn(int p, int t, int j)
{
    return p * 1000 + t * 10 + j + 1;
}

inline int body(int rank, int size, int worldId, std::string* why)
{
    auto& world = faabric::mpi::getMpiWorldRegistry().getWorld(worldId);
    auto comm = world.getDeviceComm(rank);
    GS_CHECK(comm != nullptr);
    auto launches = [&] { return comm->stats().launches; };
    const size_t rsStride = (size_t)size * MAXC; // per-tensor room for N shards

    DevBuffer rsSend(T * rsStride, BufferMemory::Heap);
    DevBuffer rsRecv(T * MAXC, BufferMemory::Heap);
    DevBuffer agSend(T * MAXC, BufferMemory::Heap);
    DevBuffer agRecv(T * rsStride, BufferMemory::Heap);
    DevBuffer arBuf(T * MAXC, BufferMemory::Heap);
    GS_CHECK(rsSend.ptr && rsRecv.ptr && agSend.ptr && agRecv.ptr && arBuf.ptr);

    auto fill = [&] {
        for (int t = 0; t < T; t++) {
            for (int i = 0; i < size * shardOf(t); i++) {
                rsSend.host[t * rsStride + i] = rsIn(rank, t, i);
            }
            for (int j = 0; j < MAXC; j++) {
                agSend.host[t * MAXC + j] = agIn(rank, t, j);
                arBuf.host[t * MAXC + j] = rank + t + j;
                rsRecv.host[t * MAXC + j] = -1;
            }
            for (size_t i = 0; i < rsStride; i++) {
                agRecv.host[t * rsStride + i] = -1;
            }
        }
        rsSend.upload();
        rsRecv.upload();
        agSend.upload();
        agRecv.upload();
        arBuf.upload();
    };
    auto rsOk = [&](int t0, int t1) {
        const auto& got = rsRecv.read();
        for (int t = t0; t < t1; t++) {
            for (int j = 0; j < MAXC; j++) {
                const int32_t want = j < shardOf(t) ? rsOut(size, rank, t, j) : -1;
                if (got[t * MAXC + j] != want) {
                    return false;
                }
            }
        }
        return true;
    };
    auto agOk = [&](int t0, int t1) {
        const auto& got = agRecv.read();
        for (int t = t0; t < t1; t++) {
            const int c = shardOf(t);
            for (size_t i = 0; i < rsStride; i++) {
                const int p = (int)(i / c);
                const int32_t want = i < (size_t)size * c ? agIn(p, t, (int)(i % c)) : -1;
                if (got[t * rsStride + i] != want) {
                    return false;
                }
            }
        }
        return true;
    };
    auto arOk = [&](int t0, int t1) {
        const auto& got = arBuf.read();
        for (int t = t0; t < t1; t++) {
            for (int j = 0; j < MAXC; j++) {
                if (got[t * MAXC + j] != size * (t + j) + size * (size - 1) / 2) {
                    return false;
                }
            }
        }
        return true;
    };

    // ---- one burst of each kind: one grouped launch each
    fill();
    MPI_Barrier(MPI_COMM_WORLD);
    std::vector<MPI_Request> reqs(T);
    uint64_t l0 = launches();
    for (int t = 0; t < T; t++) {
        GS_CHECK(MPI_Ireduce_scatter_block(rsSend.ptr + t * rsStride, rsRecv.ptr + t * MAXC, shardOf(t), MPI_INT, MPI_SUM,
                                           MPI_COMM_WORLD, &reqs[t]) == MPI_SUCCESS);
    }
    GS_CHECK(launches() == l0); // deferred
    MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE);
    GS_CHECK(launches() == l0 + 1);
    GS_CHECK(rsOk(0, T));

    l0 = launches();
    for (int t = 0; t < T; t++) {
        GS_CHECK(MPI_Iallgather(agSend.ptr + t * MAXC, shardOf(t), MPI_INT, agRecv.ptr + t * rsStride, shardOf(t), MPI_INT,
                                MPI_COMM_WORLD, &reqs[t]) == MPI_SUCCESS);
    }
    MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE);
    GS_CHECK(launches() == l0 + 1);
    GS_CHECK(agOk(0, T));

    // ---- interleaved kinds: every change of kind flushes the pending burst
    fill();
    MPI_Barrier(MPI_COMM_WORLD);
    const int H = T / 2;
    std::vector<MPI_Request> mixed;
    l0 = launches();
    for (int t = 0; t < H; t++) {
        mixed.emplace_back();
        MPI_Ireduce_scatter_block(rsSend.ptr + t * rsStride, rsRecv.ptr + t * MAXC, shardOf(t), MPI_INT, MPI_SUM,
                                  MPI_COMM_WORLD, &mixed.back());
    }
    for (int t = 0; t < H; t++) {
        mixed.emplace_back();
        MPI_Iallreduce(MPI_IN_PLACE, arBuf.ptr + t * MAXC, MAXC, MPI_INT, MPI_SUM, MPI_COMM_WORLD, &mixed.back());
    }
    GS_CHECK(launches() == l0 + 1); // the reduce-scatter burst went out
    for (int t = 0; t < H; t++) {
        mixed.emplace_back();
        MPI_Iallgather(agSend.ptr + t * MAXC, shardOf(t), MPI_INT, agRecv.ptr + t * rsStride, shardOf(t), MPI_INT,
                       MPI_COMM_WORLD, &mixed.back());
    }
    GS_CHECK(launches() == l0 + 2); // ... and the all-reduce burst
    // a reduce-scatter of another op is another burst
    for (int t = H; t < T; t++) {
        mixed.emplace_back();
        MPI_Ireduce_scatter_block(rsSend.ptr + t * rsStride, rsRecv.ptr + t * MAXC, shardOf(t), MPI_INT, MPI_MAX,
                                  MPI_COMM_WORLD, &mixed.back());
    }
    GS_CHECK(launches() == l0 + 3);
    MPI_Waitall((int)mixed.size(), mixed.data(), MPI_STATUSES_IGNORE);
    GS_CHECK(launches() == l0 + 4);
    GS_CHECK(rsOk(0, H) && agOk(0, H) && arOk(0, H));
    {
        // MAX over ranks of rsIn(p, t, r*c + j) is the last rank's value
        const auto& got = rsRecv.read();
        for (int t = H; t < T; t++) {
            for (int j = 0; j < shardOf(t); j++) {
                GS_CHECK(got[t * MAXC + j] == rsIn(size - 1, t, rank * shardOf(t) + j));
            }
        }
    }

    // ---- in place: MPI_Iallgather is grouped, MPI_Ireduce_scatter_block
    // completes at issue (its output overwrites input the peers read)
    fill();
    for (int t = 0; t < T; t++) {
        for (int j = 0; j < shardOf(t); j++) {
            agRecv.host[t * rsStride + (size_t)rank * shardOf(t) + j] = agIn(rank, t, j);
        }
    }
    agRecv.upload();
    MPI_Barrier(MPI_COMM_WORLD);
    l0 = launches();
    for (int t = 0; t < T; t++) {
        MPI_Iallgather(MPI_IN_PLACE, 0, MPI_DATATYPE_NULL, agRecv.ptr + t * rsStride, shardOf(t), MPI_INT, MPI_COMM_WORLD,
                       &reqs[t]);
    }
    MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE);
    GS_CHECK(launches() == l0 + 1);
    GS_CHECK(agOk(0, T));
    MPI_Request one;
    GS_CHECK(MPI_Ireduce_scatter_block(MPI_IN_PLACE, rsSend.ptr, shardOf(0), MPI_INT, MPI_SUM, MPI_COMM_WORLD, &one) ==
             MPI_SUCCESS);
    MPI_Wait(&one, MPI_STATUS_IGNORE);
    {
        const auto& got = rsSend.read();
        for (int j = 0; j < shardOf(0); j++) {
            GS_CHECK(got[j] == rsOut(size, rank, 0, j));
        }
    }

    // ---- host buffers complete at issue
    {
        const int c = 8;
        std::vector<int32_t> hs((size_t)size * c), hr(c, -1), ga(c), gr((size_t)size * c, -1);
        for (int i = 0; i < size * c; i++) {
            hs[i] = rsIn(rank, 1, i);
        }
        for (int j = 0; j < c; j++) {
            ga[j] = agIn(rank, 1, j);
        }
        MPI_Request a, b;
        MPI_Ireduce_scatter_block(hs.data(), hr.data(), c, MPI_INT, MPI_SUM, MPI_COMM_WORLD, &a);
        MPI_Iallgather(ga.data(), c, MPI_INT, gr.data(), c, MPI_INT, MPI_COMM_WORLD, &b);
        MPI_Wait(&a, MPI_STATUS_IGNORE);
        MPI_Wait(&b, MPI_STATUS_IGNORE);
        for (int j = 0; j < c; j++) {
            GS_CHECK(hr[j] == 7 * size * (size - 1) / 2 + size * (3 + rank * c + j));
        }
        for (int i = 0; i < size * c; i++) {
            GS_CHECK(gr[i] == agIn(i / c, 1, i % c));
        }
        // MPI_Reduce_scatter_block on host and on device buffers
        std::fill(hr.begin(), hr.end(), -1);
        GS_CHECK(MPI_Reduce_scatter_block(hs.data(), hr.data(), c, MPI_INT, MPI_SUM, MPI_COMM_WORLD) == MPI_SUCCESS);
        for (int j = 0; j < c; j++) {
            GS_CHECK(hr[j] == 7 * size * (size - 1) / 2 + size * (3 + rank * c + j));
        }
    }
    fill();
    MPI_Barrier(MPI_COMM_WORLD);
    GS_CHECK(MPI_Reduce_scatter_block(rsSend.ptr + 2 * rsStride, rsRecv.ptr + 2 * MAXC, shardOf(2), MPI_INT, MPI_SUM,
                                      MPI_COMM_WORLD) == MPI_SUCCESS);
    GS_CHECK(rsOk(2, 3));
    GS_CHECK(MPI_Reduce_scatter_block(rsSend.ptr, rsRecv.ptr, 4, MPI_INT, MPI_REPLACE, MPI_COMM_WORLD) == MPI_ERR_OP);
    GS_CHECK(MPI_Ireduce_scatter_block(rsSend.ptr, rsRecv.ptr, 4, MPI_INT, MPI_NO_OP, MPI_COMM_WORLD, &one) == MPI_ERR_OP);
    MPI_Barrier(MPI_COMM_WORLD);
    GS_CHECK(comm->peekError() == 0);
    return 0;
}

#undef GS_CHECK

} // namespace group_shard
