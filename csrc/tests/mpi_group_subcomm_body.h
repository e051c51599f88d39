// One MPI program for MPI_Ibcast bursts and for the grouped non-blocking
// collectives on sub-communicators.  Shared by the loopback test
// (test_loopback_group_bcast.cpp), the GPU test (test_device_group_bcast.cpp)
// and faabric_worker's `group-subcomm` program, which
// tests/test_dist_group_subcomm.py runs with one rank in each of four
// worker processes.
//
// Bursts on MPI_Alloc_mem(MPI_INFO_FAABRIC_DEVICE) memory must launch nothing
// before the first wait and exactly one grouped kernel after it (counted on
// the world's device communicator, or on the sub-communicator's child); a
// change of root flushes the pending burst; host buffers complete at issue;
// MPI_Comm_free with a pending burst completes it first; refused calls return
// their error before anything is launched.  A split of a split runs the same
// bursts on its own child, and with every signal slot taken a new split runs
// all five calls on the host path with the same results.  Every result is
// compared exactly against a closed form computed on the host.
#pragma once

#include "mpi/subcomm.h"
#include "mpi_subcomm_device_body.h"

#include <faabric/mpi/MpiWorld.h>
#include <faabric/mpi/MpiWorldRegistry.h>
#include <faabric/mpi/mpi.h>

#include <cstdint>
#include <string>
#include <vector>

namespace group_subcomm {

using subcomm_device::BufferMemory;
using subcomm_device::DevBuffer;

#define GB_CHECK(cond)                                                         \
    do {                                                                       \
        if (!(cond)) {                                                         \
            *why = "rank " + std::to_string(rank) + ": check failed at line " + std::to_string(__LINE__) + ": " #cond; \
            return 1;                                                          \
        }                                                                      \
    } while (0)

constexpr int T = 10;      // tensors per burst
constexpr int STRIDE = 64; // int32 slots per tensor (256 bytes: 16-byte aligned)

// Broadcast length of tensor t in int32 (any count, not only whole vectors)
inline int bcLen(int t)
{
    return 1 + (t * 7) % 41;
}

inline int32_t bcIn(int root, int t, int j)
{
    return root * 100000 + t * 1000 + j + 7;
}

// Reduce-scatter shard of tensor t: a multiple of 4 int32 (16 bytes)
inline int rsShard(int t)
{
    return 4 * (1 + t % 3);
}

// The child of `comm` on this rank (null: host path or no agreement yet)
inline std::shared_ptr<faabric::device::Communicator> childOf(MPI_Comm comm, int rank)
{
    auto sub = faabric::mpi::getSubCommunicator(comm->id);
    return sub == nullptr ? nullptr : sub->currentDevice(rank);
}

inline int body(int rank, int size, int worldId, std::string* why)
{
    auto& world = faabric::mpi::getMpiWorldRegistry().getWorld(worldId);
    auto comm = world.getDeviceComm(rank);
    GB_CHECK(comm != nullptr);
    const size_t big = (size_t)T * STRIDE * size;
    DevBuffer a(big, BufferMemory::Heap);
    DevBuffer b(big, BufferMemory::Heap);
    GB_CHECK(a.ptr && b.ptr);
    std::vector<MPI_Request> reqs(T);

    // ---- MPI_Ibcast on the world: one grouped launch per burst, every root
    for (int root = 0; root < size; root++) {
        for (size_t i = 0; i < big; i++) {
            a.host[i] = -1 - rank;
        }
        for (int t = 0; t < T; t++) {
            for (int j = 0; j < bcLen(t); j++) {
                if (rank == root) {
                    a.host[t * STRIDE + j] = bcIn(root, t, j);
                }
            }
        }
        a.upload();
        MPI_Barrier(MPI_COMM_WORLD);
        const uint64_t l0 = comm->stats().launches;
        for (int t = 0; t < T; t++) {
            GB_CHECK(MPI_Ibcast(a.ptr + t * STRIDE, bcLen(t), MPI_INT, root, MPI_COMM_WORLD, &reqs[t]) == MPI_SUCCESS);
        }
        GB_CHECK(comm->stats().launches == l0); // deferred
        GB_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GB_CHECK(comm->stats().launches == l0 + (size > 1 ? 1 : 0));
        const auto& got = a.read();
        for (int t = 0; t < T; t++) {
            for (int j = 0; j < STRIDE; j++) {
                GB_CHECK(got[t * STRIDE + j] == (j < bcLen(t) ? bcIn(root, t, j) : -1 - rank));
            }
        }
    }

    // ---- a change of root flushes the pending burst: two launches
    {
        for (int t = 0; t < T; t++) {
            for (int j = 0; j < STRIDE; j++) {
                a.host[t * STRIDE + j] = bcIn(rank, t, j);
            }
        }
        a.upload();
        MPI_Barrier(MPI_COMM_WORLD);
        const uint64_t l0 = comm->stats().launches;
        for (int t = 0; t < T; t++) {
            const int root = t < T / 2 ? 0 : size - 1;
            GB_CHECK(MPI_Ibcast(a.ptr + t * STRIDE, STRIDE, MPI_INT, root, MPI_COMM_WORLD, &reqs[t]) == MPI_SUCCESS);
        }
        GB_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GB_CHECK(comm->stats().launches == l0 + (size > 1 ? 2 : 0));
        const auto& got = a.read();
        for (int t = 0; t < T; t++) {
            const int root = t < T / 2 ? 0 : size - 1;
            for (int j = 0; j < STRIDE; j++) {
                GB_CHECK(got[t * STRIDE + j] == bcIn(root, t, j));
            }
        }
    }

    // ---- refusals at issue: nothing deferred, nothing launched
    {
        const uint64_t l0 = comm->stats().launches;
        MPI_Request r;
        GB_CHECK(MPI_Ibcast(a.ptr, 4, MPI_INT, size, MPI_COMM_WORLD, &r) == MPI_ERR_ARG);
        GB_CHECK(MPI_Ibcast(a.ptr, 4, MPI_INT, -1, MPI_COMM_WORLD, &r) == MPI_ERR_ARG);
        GB_CHECK(MPI_Iallreduce(MPI_IN_PLACE, a.ptr, 4, MPI_INT, MPI_REPLACE, MPI_COMM_WORLD, &r) == MPI_ERR_OP);
        GB_CHECK(comm->stats().launches == l0);
    }

    // ---- host buffers complete at issue
    {
        std::vector<int32_t> h(9, rank == 0 ? 42 : 0);
        MPI_Request r;
        GB_CHECK(MPI_Ibcast(h.data(), 9, MPI_INT, 0, MPI_COMM_WORLD, &r) == MPI_SUCCESS);
        for (int v : h) {
            GB_CHECK(v == 42);
        }
        GB_CHECK(MPI_Wait(&r, MPI_STATUS_IGNORE) == MPI_SUCCESS);
    }

    // ---- parity split: the three grouped kinds and MPI_Ibcast on the child
    MPI_Comm sub;
    GB_CHECK(MPI_Comm_split(MPI_COMM_WORLD, rank % 2, rank, &sub) == MPI_SUCCESS);
    int srank = -1, ssize = -1;
    MPI_Comm_rank(sub, &srank);
    MPI_Comm_size(sub, &ssize);
    std::vector<int> members;
    for (int p = rank % 2; p < size; p += 2) {
        members.push_back(p);
    }
    GB_CHECK(ssize == (int)members.size() && members[srank] == rank);
    int memberSum = 0;
    for (int p : members) {
        memberSum += p;
    }
    for (int round = 0; round < 3; round++) {
        // all-reduce
        for (int t = 0; t < T; t++) {
            for (int j = 0; j < STRIDE; j++) {
                a.host[t * STRIDE + j] = 3 * rank + t + j + round;
            }
        }
        a.upload();
        for (int t = 0; t < T; t++) {
            GB_CHECK(MPI_Iallreduce(MPI_IN_PLACE, a.ptr + t * STRIDE, STRIDE, MPI_INT, MPI_SUM, sub, &reqs[t]) == MPI_SUCCESS);
        }
        auto child = childOf(sub, rank);
        GB_CHECK(child != nullptr && child->size() == ssize);
        uint64_t c0 = child->stats().launches;
        GB_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GB_CHECK(child->stats().launches == c0 + 1 || ssize == 1);
        {
            const auto& got = a.read();
            for (int t = 0; t < T; t++) {
                for (int j = 0; j < STRIDE; j++) {
                    GB_CHECK(got[t * STRIDE + j] == 3 * memberSum + ssize * (t + j + round));
                }
            }
        }
        // reduce-scatter: a holds ssize shards per tensor, b gets this rank's
        const size_t rsStride = (size_t)STRIDE * ssize;
        for (int t = 0; t < T; t++) {
            for (int i = 0; i < ssize * rsShard(t); i++) {
                a.host[t * rsStride + i] = 7 * rank + 3 * t + i;
            }
        }
        a.upload();
        for (size_t i = 0; i < big; i++) {
            b.host[i] = -1;
        }
        b.upload();
        c0 = child->stats().launches;
        for (int t = 0; t < T; t++) {
            GB_CHECK(MPI_Ireduce_scatter_block(a.ptr + t * rsStride, b.ptr + t * STRIDE, rsShard(t), MPI_INT, MPI_SUM, sub,
                                               &reqs[t]) == MPI_SUCCESS);
        }
        GB_CHECK(child->stats().launches == c0);
        GB_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GB_CHECK(child->stats().launches == c0 + 1 || ssize == 1);
        {
            const auto& got = b.read();
            for (int t = 0; t < T; t++) {
                const int c = rsShard(t);
                for (int j = 0; j < STRIDE; j++) {
                    GB_CHECK(got[t * STRIDE + j] == (j < c ? 7 * memberSum + ssize * (3 * t + srank * c + j) : -1));
                }
            }
        }
        // all-gather: block q of b gets a of member q
        for (int t = 0; t < T; t++) {
            for (int j = 0; j < 4; j++) {
                a.host[t * STRIDE + j] = rank * 1000 + t * 10 + j + round;
            }
        }
        a.upload();
        c0 = child->stats().launches;
        for (int t = 0; t < T; t++) {
            GB_CHECK(MPI_Iallgather(a.ptr + t * STRIDE, 4, MPI_INT, b.ptr + t * rsStride, 4, MPI_INT, sub, &reqs[t]) ==
                     MPI_SUCCESS);
        }
        GB_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GB_CHECK(child->stats().launches == c0 + 1 || ssize == 1);
        {
            const auto& got = b.read();
            for (int t = 0; t < T; t++) {
                for (int q = 0; q < ssize; q++) {
                    for (int j = 0; j < 4; j++) {
                        GB_CHECK(got[t * rsStride + q * 4 + j] == members[q] * 1000 + t * 10 + j + round);
                    }
                }
            }
        }
        // broadcast from child rank `round % ssize`
        const int root = round % ssize;
        for (int t = 0; t < T; t++) {
            for (int j = 0; j < STRIDE; j++) {
                a.host[t * STRIDE + j] = srank == root ? bcIn(members[root], t, j) : -5;
            }
        }
        a.upload();
        c0 = child->stats().launches;
        for (int t = 0; t < T; t++) {
            GB_CHECK(MPI_Ibcast(a.ptr + t * STRIDE, bcLen(t), MPI_INT, root, sub, &reqs[t]) == MPI_SUCCESS);
        }
        GB_CHECK(child->stats().launches == c0);
        GB_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GB_CHECK(child->stats().launches == c0 + (ssize > 1 ? 1 : 0));
        {
            const auto& got = a.read();
            for (int t = 0; t < T; t++) {
                for (int j = 0; j < STRIDE; j++) {
                    const int32_t want = j < bcLen(t) || srank == root ? bcIn(members[root], t, j) : -5;
                    GB_CHECK(got[t * STRIDE + j] == want);
                }
            }
        }
        // the world's bursts in between still launch on the world
        const uint64_t w0 = comm->stats().launches;
        for (int t = 0; t < T; t++) {
            GB_CHECK(MPI_Ibcast(b.ptr + t * STRIDE, 8, MPI_INT, 0, MPI_COMM_WORLD, &reqs[t]) == MPI_SUCCESS);
        }
        GB_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GB_CHECK(comm->stats().launches == w0 + (size > 1 ? 1 : 0));
    }

    // ---- blocking MPI_Reduce_scatter_block on the child
    {
        for (int i = 0; i < 4 * ssize; i++) {
            a.host[i] = rank + i;
        }
        a.upload();
        GB_CHECK(MPI_Reduce_scatter_block(a.ptr, b.ptr, 4, MPI_INT, MPI_SUM, sub) == MPI_SUCCESS);
        const auto& got = b.read();
        for (int j = 0; j < 4; j++) {
            GB_CHECK(got[j] == memberSum + ssize * (srank * 4 + j));
        }
        // host buffers take the sub-communicator's host fold
        std::vector<int32_t> hs(4 * ssize), hr(4, -1);
        for (int i = 0; i < 4 * ssize; i++) {
            hs[i] = rank * 2 + i;
        }
        GB_CHECK(MPI_Reduce_scatter_block(hs.data(), hr.data(), 4, MPI_INT, MPI_SUM, sub) == MPI_SUCCESS);
        for (int j = 0; j < 4; j++) {
            GB_CHECK(hr[j] == 2 * memberSum + ssize * (srank * 4 + j));
        }
    }

    // ---- refusals on the child
    {
        MPI_Request r;
        GB_CHECK(MPI_Ibcast(a.ptr, 4, MPI_INT, ssize, sub, &r) == MPI_ERR_ARG);
        GB_CHECK(MPI_Iallreduce(MPI_IN_PLACE, a.ptr, 4, MPI_INT, MPI_REPLACE, sub, &r) == MPI_ERR_OP);
        GB_CHECK(MPI_Ireduce_scatter_block(a.ptr, b.ptr, 4, MPI_INT, MPI_NO_OP, sub, &r) == MPI_ERR_OP);
    }

    // ---- a split of the split: its own child, bursts of one launch
    {
        MPI_Comm nested;
        GB_CHECK(MPI_Comm_split(sub, srank % 2, srank, &nested) == MPI_SUCCESS);
        int nrank = -1, nsize = -1;
        MPI_Comm_rank(nested, &nrank);
        MPI_Comm_size(nested, &nsize);
        std::vector<int> nmembers;
        for (int q = srank % 2; q < ssize; q += 2) {
            nmembers.push_back(members[q]);
        }
        GB_CHECK(nsize == (int)nmembers.size() && nmembers[nrank] == rank);
        int nsum = 0;
        for (int p : nmembers) {
            nsum += p;
        }
        for (int t = 0; t < T; t++) {
            for (int j = 0; j < STRIDE; j++) {
                a.host[t * STRIDE + j] = 5 * rank + t + j;
                b.host[t * STRIDE + j] = nrank == nsize - 1 ? bcIn(rank, t, j) : -3;
            }
        }
        a.upload();
        b.upload();
        for (int t = 0; t < T; t++) {
            GB_CHECK(MPI_Iallreduce(MPI_IN_PLACE, a.ptr + t * STRIDE, STRIDE, MPI_INT, MPI_SUM, nested, &reqs[t]) ==
                     MPI_SUCCESS);
        }
        auto child = childOf(nested, rank);
        GB_CHECK(child != nullptr && child->size() == nsize);
        uint64_t c0 = child->stats().launches;
        GB_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GB_CHECK(child->stats().launches == c0 + 1 || nsize == 1);
        c0 = child->stats().launches;
        for (int t = 0; t < T; t++) {
            GB_CHECK(MPI_Ibcast(b.ptr + t * STRIDE, bcLen(t), MPI_INT, nsize - 1, nested, &reqs[t]) == MPI_SUCCESS);
        }
        GB_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GB_CHECK(child->stats().launches == c0 + (nsize > 1 ? 1 : 0));
        const auto& ga = a.read();
        const auto& gb = b.read();
        for (int t = 0; t < T; t++) {
            for (int j = 0; j < STRIDE; j++) {
                GB_CHECK(ga[t * STRIDE + j] == 5 * nsum + nsize * (t + j));
                const int32_t want = j < bcLen(t) || nrank == nsize - 1 ? bcIn(nmembers[nsize - 1], t, j) : -3;
                GB_CHECK(gb[t * STRIDE + j] == want);
            }
        }
        child.reset();
        GB_CHECK(MPI_Comm_free(&nested) == MPI_SUCCESS);
    }

    // ---- MPI_Comm_free with a burst pending: it is issued and completed
    {
        for (int t = 0; t < T; t++) {
            for (int j = 0; j < STRIDE; j++) {
                a.host[t * STRIDE + j] = srank == 0 ? bcIn(members[0], t, j) : -9;
            }
        }
        a.upload();
        for (int t = 0; t < T; t++) {
            GB_CHECK(MPI_Ibcast(a.ptr + t * STRIDE, STRIDE, MPI_INT, 0, sub, &reqs[t]) == MPI_SUCCESS);
        }
        GB_CHECK(MPI_Comm_free(&sub) == MPI_SUCCESS);
        GB_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        const auto& got = a.read();
        for (int t = 0; t < T; t++) {
            for (int j = 0; j < STRIDE; j++) {
                GB_CHECK(got[t * STRIDE + j] == bcIn(members[0], t, j));
            }
        }
    }
    // ---- no slot left: world splits take every slot, then a new parity
    // split runs every call on device buffers on the host path (no child)
    // with the same results
    {
        std::vector<MPI_Comm> fill;
        for (int i = 0; i < FB_SUB_SLOTS; i++) {
            MPI_Comm c = MPI_COMM_NULL;
            GB_CHECK(MPI_Comm_split(MPI_COMM_WORLD, 0, rank, &c) == MPI_SUCCESS);
            // (a device call: takes a slot)
            GB_CHECK(MPI_Allreduce(MPI_IN_PLACE, b.ptr, 4, MPI_INT, MPI_SUM, c) == MPI_SUCCESS);
            fill.push_back(c);
        }
        GB_CHECK(comm->freeSubsetSlots() == 0);
        MPI_Comm hs;
        GB_CHECK(MPI_Comm_split(MPI_COMM_WORLD, rank % 2, rank, &hs) == MPI_SUCCESS);
        // all-reduce burst
        for (int t = 0; t < T; t++) {
            for (int j = 0; j < STRIDE; j++) {
                a.host[t * STRIDE + j] = 3 * rank + t + j;
            }
        }
        a.upload();
        for (int t = 0; t < T; t++) {
            GB_CHECK(MPI_Iallreduce(MPI_IN_PLACE, a.ptr + t * STRIDE, STRIDE, MPI_INT, MPI_SUM, hs, &reqs[t]) == MPI_SUCCESS);
        }
        GB_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GB_CHECK(childOf(hs, rank) == nullptr);
        {
            const auto& got = a.read();
            for (int t = 0; t < T; t++) {
                for (int j = 0; j < STRIDE; j++) {
                    GB_CHECK(got[t * STRIDE + j] == 3 * memberSum + ssize * (t + j));
                }
            }
        }
        // reduce-scatter: the bursts, and one blocking call
        const size_t rsStride = (size_t)STRIDE * ssize;
        for (int t = 0; t < T; t++) {
            for (int i = 0; i < ssize * rsShard(t); i++) {
                a.host[t * rsStride + i] = 7 * rank + 3 * t + i;
            }
        }
        a.upload();
        for (size_t i = 0; i < big; i++) {
            b.host[i] = -1;
        }
        b.upload();
        for (int t = 0; t < T; t++) {
            GB_CHECK(MPI_Ireduce_scatter_block(a.ptr + t * rsStride, b.ptr + t * STRIDE, rsShard(t), MPI_INT, MPI_SUM, hs,
                                               &reqs[t]) == MPI_SUCCESS);
        }
        GB_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GB_CHECK(MPI_Reduce_scatter_block(a.ptr, b.ptr + (T - 1) * STRIDE + 32, rsShard(0), MPI_INT, MPI_SUM, hs) ==
                 MPI_SUCCESS);
        {
            const auto& got = b.read();
            for (int t = 0; t < T; t++) {
                const int c = rsShard(t);
                for (int j = 0; j < c; j++) {
                    GB_CHECK(got[t * STRIDE + j] == 7 * memberSum + ssize * (3 * t + srank * c + j));
                }
            }
            for (int j = 0; j < rsShard(0); j++) {
                GB_CHECK(got[(T - 1) * STRIDE + 32 + j] == 7 * memberSum + ssize * (srank * rsShard(0) + j));
            }
        }
        // all-gather: block q gets a of member q
        for (int t = 0; t < T; t++) {
            for (int j = 0; j < 4; j++) {
                a.host[t * STRIDE + j] = rank * 1000 + t * 10 + j;
            }
        }
        a.upload();
        for (int t = 0; t < T; t++) {
            GB_CHECK(MPI_Iallgather(a.ptr + t * STRIDE, 4, MPI_INT, b.ptr + t * rsStride, 4, MPI_INT, hs, &reqs[t]) ==
                     MPI_SUCCESS);
        }
        GB_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        {
            const auto& got = b.read();
            for (int t = 0; t < T; t++) {
                for (int q = 0; q < ssize; q++) {
                    for (int j = 0; j < 4; j++) {
                        GB_CHECK(got[t * rsStride + q * 4 + j] == members[q] * 1000 + t * 10 + j);
                    }
                }
            }
        }
        // broadcast from the last member
        for (int t = 0; t < T; t++) {
            for (int j = 0; j < STRIDE; j++) {
                a.host[t * STRIDE + j] = srank == ssize - 1 ? bcIn(rank, t, j) : -7;
            }
        }
        a.upload();
        for (int t = 0; t < T; t++) {
            GB_CHECK(MPI_Ibcast(a.ptr + t * STRIDE, bcLen(t), MPI_INT, ssize - 1, hs, &reqs[t]) == MPI_SUCCESS);
        }
        GB_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        {
            const auto& got = a.read();
            for (int t = 0; t < T; t++) {
                for (int j = 0; j < STRIDE; j++) {
                    const int32_t want = j < bcLen(t) || srank == ssize - 1 ? bcIn(members[ssize - 1], t, j) : -7;
                    GB_CHECK(got[t * STRIDE + j] == want);
                }
            }
        }
        // no child was made at any of these calls
        GB_CHECK(childOf(hs, rank) == nullptr);
        GB_CHECK(MPI_Comm_free(&hs) == MPI_SUCCESS);
        for (MPI_Comm& c : fill) {
            GB_CHECK(MPI_Comm_free(&c) == MPI_SUCCESS);
        }
        GB_CHECK(comm->freeSubsetSlots() == (1u << FB_SUB_SLOTS) - 1);
    }
    MPI_Barrier(MPI_COMM_WORLD);
    return 0;
}

#undef GB_CHECK

}
