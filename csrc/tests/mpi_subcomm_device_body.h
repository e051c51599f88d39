// One MPI program that checks the fused device path of sub-communicators:
// MPI_Bcast, MPI_Reduce, MPI_Allreduce, MPI_Scan, MPI_Gather, MPI_Scatter,
// MPI_Allgather and MPI_Alltoall on device buffers of communicators made by
// MPI_Comm_split and MPI_Comm_split_type.  Shared by the in-process tests
// (test_mpi_subcomm_device.cpp) and the `subcomm-device` function of
// faabric_worker, which runs it across worker processes
// (tests/test_dist_subcomm_device.py).
//
// Every result is compared exactly against a closed form over the members in
// child order, and the world's device-collective count must rise by exactly
// one per call and rank while a communicator has a signal slot, and not at
// all once every slot is taken (host path).
#pragma once

#include "mpi_rma_atomics_body.h"

#include <faabric/mpi/MpiWorld.h>
#include <faabric/mpi/MpiWorldRegistry.h>
#include <faabric/mpi/mpi.h>

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <string>
#include <vector>

namespace subcomm_device {

enum class BufferMemory
{
    Heap,      // MPI_Alloc_mem(MPI_INFO_FAABRIC_DEVICE): the symmetric heap
    CudaMalloc // cudaMalloc memory: staged by the communicator
};

struct Setup
{
    BufferMemory memory = BufferMemory::Heap;
};

#define SUB_CHECK(cond)                                                        \
    do {                                                                       \
        if (!(cond)) {                                                         \
            *why = "rank " + std::to_string(rank) + ": check failed at line " + std::to_string(__LINE__) + ": " #cond; \
            return 1;                                                          \
        }                                                                      \
    } while (0)

constexpr int N = 1001; // elements per rank and chunk (no vector multiple)

// A device buffer of `ints` int32 values with a host shadow
struct DevBuffer
{
    std::vector<int32_t> host;
    int32_t* ptr = nullptr;
    BufferMemory memory;

    DevBuffer(size_t ints, BufferMemory m)
      : host(ints, 0)
      , memory(m)
    {
        if (m == BufferMemory::Heap) {
            if (MPI_Alloc_mem((MPI_Aint)(ints * 4), MPI_INFO_FAABRIC_DEVICE, &ptr) != MPI_SUCCESS) {
                ptr = nullptr;
            }
        } else if (cudaMalloc((void**)&ptr, ints * 4) != cudaSuccess) {
            cudaGetLastError();
            ptr = nullptr;
        }
    }
    ~DevBuffer()
    {
        if (ptr == nullptr) {
            return;
        }
        if (memory == BufferMemory::Heap) {
            MPI_Free_mem(ptr);
        } else {
            cudaFree(ptr);
        }
    }
    DevBuffer(const DevBuffer&) = delete;
    DevBuffer& operator=(const DevBuffer&) = delete;

    void upload() { rma_atomics::copyBytes(ptr, host.data(), host.size() * 4); }
    const std::vector<int32_t>& read()
    {
        rma_atomics::copyBytes(host.data(), ptr, host.size() * 4);
        return host;
    }
};

inline int32_t val(int worldRank, int k)
{
    return worldRank * 1000 + k % 101 + 1;
}

// World ranks of `comm`, in its rank order
inline std::vector<int> membersOf(MPI_Comm comm)
{
    int n = 0;
    int me = -1;
    int worldRank = -1;
    MPI_Comm_size(comm, &n);
    MPI_Comm_rank(comm, &me);
    MPI_Comm_rank(MPI_COMM_WORLD, &worldRank);
    std::vector<int> all(n);
    MPI_Allgather(&worldRank, 1, MPI_INT, all.data(), 1, MPI_INT, comm);
    return all;
}

// The eight collectives on `comm` with device buffers `a` and `b` (N * world
// size ints each), checked against closed forms.  Adds the calls made to *calls.
inline int eightCollectives(int rank, MPI_Comm comm, DevBuffer& a, DevBuffer& b, int* calls, std::string* why)
{
    const std::vector<int> m = membersOf(comm);
    const int n = (int)m.size();
    int cr = -1;
    MPI_Comm_rank(comm, &cr);
    SUB_CHECK(cr >= 0 && m[cr] == rank);

    // all-reduce SUM
    for (int k = 0; k < N; k++) {
        a.host[k] = val(rank, k);
    }
    a.upload();
    SUB_CHECK(MPI_Allreduce(a.ptr, b.ptr, N, MPI_INT, MPI_SUM, comm) == MPI_SUCCESS);
    b.read();
    for (int k = 0; k < N; k++) {
        int32_t e = 0;
        for (int w : m) {
            e += val(w, k);
        }
        SUB_CHECK(b.host[k] == e);
    }
    // reduce MAX to the last comm rank
    SUB_CHECK(MPI_Reduce(a.ptr, b.ptr, N, MPI_INT, MPI_MAX, n - 1, comm) == MPI_SUCCESS);
    if (cr == n - 1) {
        b.read();
        const int top = *std::max_element(m.begin(), m.end());
        for (int k = 0; k < N; k++) {
            SUB_CHECK(b.host[k] == val(top, k));
        }
    }
    // scan SUM: prefixes in comm order
    SUB_CHECK(MPI_Scan(a.ptr, b.ptr, N, MPI_INT, MPI_SUM, comm) == MPI_SUCCESS);
    b.read();
    for (int k = 0; k < N; k++) {
        int32_t e = 0;
        for (int j = 0; j <= cr; j++) {
            e += val(m[j], k);
        }
        SUB_CHECK(b.host[k] == e);
    }
    // broadcast from comm rank 1 (0 on a singleton)
    const int bRoot = n > 1 ? 1 : 0;
    for (int k = 0; k < N; k++) {
        a.host[k] = cr == bRoot ? val(rank, k) * 3 : -1;
    }
    a.upload();
    SUB_CHECK(MPI_Bcast(a.ptr, N, MPI_INT, bRoot, comm) == MPI_SUCCESS);
    a.read();
    for (int k = 0; k < N; k++) {
        SUB_CHECK(a.host[k] == val(m[bRoot], k) * 3);
    }
    // gather to comm rank 0
    for (int k = 0; k < N; k++) {
        a.host[k] = val(rank, k);
    }
    a.upload();
    SUB_CHECK(MPI_Gather(a.ptr, N, MPI_INT, b.ptr, N, MPI_INT, 0, comm) == MPI_SUCCESS);
    if (cr == 0) {
        b.read();
        for (int j = 0; j < n; j++) {
            for (int k = 0; k < N; k++) {
                SUB_CHECK(b.host[(size_t)j * N + k] == val(m[j], k));
            }
        }
    }
    // scatter from the last comm rank
    const int sRoot = n - 1;
    for (int j = 0; j < n; j++) {
        for (int k = 0; k < N; k++) {
            a.host[(size_t)j * N + k] = cr == sRoot ? rank * 100 + j * 7 + k % 13 : -1;
        }
    }
    a.upload();
    SUB_CHECK(MPI_Scatter(a.ptr, N, MPI_INT, b.ptr, N, MPI_INT, sRoot, comm) == MPI_SUCCESS);
    b.read();
    for (int k = 0; k < N; k++) {
        SUB_CHECK(b.host[k] == m[sRoot] * 100 + cr * 7 + k % 13);
    }
    // all-gather
    for (int k = 0; k < N; k++) {
        a.host[k] = val(rank, k) + 5;
    }
    a.upload();
    SUB_CHECK(MPI_Allgather(a.ptr, N, MPI_INT, b.ptr, N, MPI_INT, comm) == MPI_SUCCESS);
    b.read();
    for (int j = 0; j < n; j++) {
        for (int k = 0; k < N; k++) {
            SUB_CHECK(b.host[(size_t)j * N + k] == val(m[j], k) + 5);
        }
    }
    // all-to-all: chunk j of rank w is w * 100 + j * 7 + k % 5
    for (int j = 0; j < n; j++) {
        for (int k = 0; k < N; k++) {
            a.host[(size_t)j * N + k] = rank * 100 + j * 7 + k % 5;
        }
    }
    a.upload();
    SUB_CHECK(MPI_Alltoall(a.ptr, N, MPI_INT, b.ptr, N, MPI_INT, comm) == MPI_SUCCESS);
    b.read();
    for (int j = 0; j < n; j++) {
        for (int k = 0; k < N; k++) {
            SUB_CHECK(b.host[(size_t)j * N + k] == m[j] * 100 + cr * 7 + k % 5);
        }
    }
    *calls += 8;
    return 0;
}

// One device all-reduce on `comm`, checked; adds the call to *calls
inline int oneAllReduce(int rank, MPI_Comm comm, DevBuffer& a, DevBuffer& b, int salt, int* calls, std::string* why)
{
    const std::vector<int> m = membersOf(comm);
    for (int k = 0; k < N; k++) {
        a.host[k] = val(rank, k) * salt;
    }
    a.upload();
    SUB_CHECK(MPI_Allreduce(a.ptr, b.ptr, N, MPI_INT, MPI_SUM, comm) == MPI_SUCCESS);
    b.read();
    for (int k = 0; k < N; k++) {
        int32_t e = 0;
        for (int w : m) {
            e += val(w, k) * salt;
        }
        SUB_CHECK(b.host[k] == e);
    }
    *calls += 1;
    return 0;
}

// World-wide check of the device-collective count: every rank has made
// `calls` device calls since `before`.  Each worker process keeps its own
// count (shared by its ranks): the lowest rank of each process reports its
// process's rise, read at a barrier.
inline int checkCount(int rank, faabric::mpi::MpiWorld& world, uint64_t& before, int calls, std::string* why)
{
    MPI_Barrier(MPI_COMM_WORLD);
    const uint64_t now = world.getDeviceCollectiveCount();
    MPI_Barrier(MPI_COMM_WORLD);
    int size = 0;
    MPI_Comm_size(MPI_COMM_WORLD, &size);
    const std::string myHost = world.getHostForRank(rank);
    int leader = rank;
    for (int r = 0; r < size; r++) {
        if (world.getHostForRank(r) == myHost) {
            leader = r;
            break;
        }
    }
    int mine[2] = { calls, leader == rank ? (int)(now - before) : 0 };
    int total[2] = { 0, 0 };
    MPI_Allreduce(mine, total, 2, MPI_INT, MPI_SUM, MPI_COMM_WORLD);
    if (total[1] != total[0]) {
        *why = "device-collective count rose by " + std::to_string(total[1]) + ", expected " + std::to_string(total[0]);
        return 1;
    }
    before = now;
    return 0;
}

inline int body(int rank, int size, int worldId, const Setup& s, std::string* why)
{
    faabric::mpi::MpiWorld& world = faabric::mpi::getMpiWorldRegistry().getWorld(worldId);
    DevBuffer a((size_t)N * size, s.memory);
    DevBuffer b((size_t)N * size, s.memory);
    SUB_CHECK(a.ptr != nullptr && b.ptr != nullptr);
    int calls = 0;
    int worldCalls = 0;
    uint64_t before = 0;
    MPI_Barrier(MPI_COMM_WORLD);
    before = world.getDeviceCollectiveCount();
    MPI_Barrier(MPI_COMM_WORLD);

    // ---- 1. the eight collectives on five kinds of communicator, with world
    // calls in between
    std::vector<MPI_Comm> held;
    auto split = [&](MPI_Comm parent, int color, int key) {
        MPI_Comm c = MPI_COMM_NULL;
        MPI_Comm_split(parent, color, key, &c);
        return c;
    };
    const int half = size / 2;
    // parity: strided members
    held.push_back(split(MPI_COMM_WORLD, rank % 2, rank));
    // halves with reversed keys: comm order differs from world order
    held.push_back(split(MPI_COMM_WORLD, rank / half, size - rank));
    // a nested quarter of the half
    {
        int hr = -1;
        MPI_Comm_rank(held.back(), &hr);
        held.push_back(split(held.back(), hr / std::max(1, half / 2), hr));
    }
    // the last rank stays out
    held.push_back(split(MPI_COMM_WORLD, rank == size - 1 ? MPI_UNDEFINED : 0, rank));
    if (rank == size - 1) {
        SUB_CHECK(held.back() == MPI_COMM_NULL);
    }
    // ranks sharing an address space
    {
        MPI_Comm c = MPI_COMM_NULL;
        SUB_CHECK(MPI_Comm_split_type(MPI_COMM_WORLD, MPI_COMM_TYPE_SHARED, size - rank, MPI_INFO_NULL, &c) ==
                  MPI_SUCCESS);
        held.push_back(c);
    }
    for (MPI_Comm c : held) {
        if (c != MPI_COMM_NULL) {
            if (eightCollectives(rank, c, a, b, &calls, why) != 0) {
                return 1;
            }
        }
        // interleaved world call on the same buffers
        if (oneAllReduce(rank, MPI_COMM_WORLD, a, b, 3, &worldCalls, why) != 0) {
            return 1;
        }
    }
    if (checkCount(rank, world, before, calls + worldCalls, why) != 0) {
        return 1;
    }
    for (MPI_Comm& c : held) {
        if (c != MPI_COMM_NULL) {
            MPI_Comm_free(&c);
        }
    }
    held.clear();

    // ---- 2. slot reuse: more rounds than slots, two member layouts in turn,
    // so released pads are reused by other member sets
    calls = 0;
    for (int round = 0; round < 40; round++) {
        MPI_Comm c = round % 2 == 0 ? split(MPI_COMM_WORLD, rank % 2, rank) : split(MPI_COMM_WORLD, rank / half, -rank);
        if (oneAllReduce(rank, c, a, b, round + 1, &calls, why) != 0) {
            return 1;
        }
        MPI_Comm_free(&c);
    }
    if (checkCount(rank, world, before, calls, why) != 0) {
        return 1;
    }

    // ---- 3. exhaustion: with every slot held, the next communicator is
    // correct on the host path; after one free, the next one is fused again
    calls = 0;
    for (int i = 0; i < FB_SUB_SLOTS; i++) {
        held.push_back(split(MPI_COMM_WORLD, 0, rank));
        if (oneAllReduce(rank, held.back(), a, b, i + 2, &calls, why) != 0) {
            return 1;
        }
    }
    if (checkCount(rank, world, before, calls, why) != 0) {
        return 1;
    }
    {
        MPI_Comm extra = split(MPI_COMM_WORLD, 0, -rank);
        // (device buffers: the slot agreement runs and finds no common slot)
        int hostCalls = 0;
        if (oneAllReduce(rank, extra, a, b, 7, &hostCalls, why) != 0) {
            return 1;
        }
        if (eightCollectives(rank, extra, a, b, &hostCalls, why) != 0) {
            return 1;
        }
        // none of them ran on the device
        if (checkCount(rank, world, before, 0, why) != 0) {
            return 1;
        }
        MPI_Comm_free(&extra);
    }
    MPI_Comm_free(&held.back());
    held.pop_back();
    calls = 0;
    {
        MPI_Comm again = split(MPI_COMM_WORLD, 0, size - rank);
        if (eightCollectives(rank, again, a, b, &calls, why) != 0) {
            return 1;
        }
        MPI_Comm_free(&again);
    }
    for (MPI_Comm& c : held) {
        MPI_Comm_free(&c);
    }
    if (checkCount(rank, world, before, calls, why) != 0) {
        return 1;
    }
    return 0;
}

}
