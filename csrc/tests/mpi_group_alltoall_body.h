// One MPI program for MPI_Ialltoall bursts on the world, on MPI_Comm_split
// halves and on a split of a split.  Shared by the loopback test
// (test_loopback_group_alltoall.cpp), the GPU test
// (test_device_group_alltoall.cpp) and faabric_worker's `group-alltoall`
// program, which tests/test_dist_group_alltoall.py runs with one rank in each
// of four worker processes.
//
// Bursts on MPI_Alloc_mem(MPI_INFO_FAABRIC_DEVICE) memory launch nothing
// before the first wait and exactly one grouped kernel after it (counted on
// the world's device communicator, or on the sub-communicator's child).
// Another device collective, non-blocking (MPI_Iallgather) or blocking,
// flushes the pending burst first; a block that is not a multiple of 16 bytes
// runs one all-to-all at issue; host buffers complete at issue; MPI_Comm_free
// with a pending burst completes it first; MPI_IN_PLACE and mismatched byte
// counts are refused before anything is issued, with the outputs untouched.
// With grouping off (FAABRIC_MPI_GROUP_IALLREDUCE=0, body(..., false)) every
// call runs one kernel at issue.  Every result is compared exactly against a
// closed form computed on the host, guard words around every block included.
#pragma once

#include "mpi/subcomm.h"
#include "mpi_subcomm_device_body.h"

#include <faabric/mpi/MpiWorld.h>
#include <faabric/mpi/MpiWorldRegistry.h>
#include <faabric/mpi/mpi.h>

#include <cstdint>
#include <string>
#include <vector>

namespace group_alltoall {

using subcomm_device::BufferMemory;
using subcomm_device::DevBuffer;

#define GA_CHECK(cond)                                                         \
    do {                                                                       \
        if (!(cond)) {                                                         \
            *why = "rank " + std::to_string(rank) + ": check failed at line " + std::to_string(__LINE__) + ": " #cond; \
            return 1;                                                          \
        }                                                                      \
    } while (0)

constexpr int T = 8;       // tensors per burst
constexpr int STRIDE = 32; // int32 per block slot: a tensor of n blocks owns n * STRIDE int32

// Block length of tensor t in int32: 16 to 64 bytes, a multiple of 16
inline int blk(int t)
{
    return 4 * (1 + t % 4);
}

// Word j of block q of tensor t in world rank r's send, in round `salt`
inline int32_t aIn(int r, int t, int q, int j, int salt)
{
    return r * 100000 + t * 1000 + q * 40 + j + salt * 7;
}

// The child of `comm` on this rank (null: host path or no agreement yet)
inline std::shared_ptr<faabric::device::Communicator> childOf(MPI_Comm comm, int rank)
{
    auto sub = faabric::mpi::getSubCommunicator(comm->id);
    return sub == nullptr ? nullptr : sub->currentDevice(rank);
}

// a: this rank's sends for a communicator of `m` members (block q of tensor t
// at t * m * STRIDE + q * blk(t)); b: guard words only
inline void fill(DevBuffer& a, DevBuffer& b, int rank, int m, int salt)
{
    for (auto& v : a.host) {
        v = -7;
    }
    for (auto& v : b.host) {
        v = -1 - rank;
    }
    for (int t = 0; t < T; t++) {
        for (int q = 0; q < m; q++) {
            for (int j = 0; j < blk(t); j++) {
                a.host[(size_t)t * m * STRIDE + q * blk(t) + j] = aIn(rank, t, q, j, salt);
            }
        }
    }
    a.upload();
    b.upload();
}

// Tensors [t0, t1) of b hold, in block q, block `cr` of member q's send, and
// guard words after the blocks; the other tensors hold guard words only
inline bool exchanged(DevBuffer& b, int rank, const std::vector<int>& members, int cr, int salt, int t0, int t1,
                      std::string* why)
{
    const int m = (int)members.size();
    const auto& got = b.read();
    for (int t = 0; t < T; t++) {
        for (int i = 0; i < m * STRIDE; i++) {
            const bool in = t >= t0 && t < t1 && i < m * blk(t);
            const int32_t want = in ? aIn(members[i / blk(t)], t, cr, i % blk(t), salt) : -1 - rank;
            const int32_t v = got[(size_t)t * m * STRIDE + i];
            if (v != want) {
                *why = "rank " + std::to_string(rank) + " tensor " + std::to_string(t) + " word " + std::to_string(i) + ": " +
                       std::to_string(v) + ", want " + std::to_string(want);
                return false;
            }
        }
    }
    return true;
}

inline int issue(int rank, DevBuffer& a, DevBuffer& b, int m, int t, MPI_Comm comm, MPI_Request* r, std::string* why)
{
    GA_CHECK(MPI_Ialltoall(a.ptr + (size_t)t * m * STRIDE, blk(t), MPI_INT, b.ptr + (size_t)t * m * STRIDE, blk(t), MPI_INT,
                           comm, r) == MPI_SUCCESS);
    return 0;
}

// A burst of all T tensors on `comm` (members: its world ranks in comm rank
// order; world: the world's device communicator), checked: nothing launched
// before the wait, one launch after it
inline int burst(int rank,
                 DevBuffer& a,
                 DevBuffer& b,
                 MPI_Comm comm,
                 const std::vector<int>& members,
                 int salt,
                 const std::shared_ptr<faabric::device::Communicator>& world,
                 std::string* why)
{
    const int m = (int)members.size();
    int cr = -1;
    MPI_Comm_rank(comm, &cr);
    fill(a, b, rank, m, salt);
    std::vector<MPI_Request> reqs(T);
    GA_CHECK(issue(rank, a, b, m, 0, comm, &reqs[0], why) == 0);
    auto dev = comm == MPI_COMM_WORLD ? world : childOf(comm, rank);
    GA_CHECK(dev != nullptr && dev->size() == m);
    const uint64_t l0 = dev->stats().launches;
    for (int t = 1; t < T; t++) {
        GA_CHECK(issue(rank, a, b, m, t, comm, &reqs[t], why) == 0);
    }
    GA_CHECK(dev->stats().launches == l0); // deferred
    GA_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
    GA_CHECK(dev->stats().launches == l0 + 1);
    GA_CHECK(exchanged(b, rank, members, cr, salt, 0, T, why));
    return 0;
}

inline int body(int rank, int size, int worldId, bool grouped, std::string* why)
{
    auto& world = faabric::mpi::getMpiWorldRegistry().getWorld(worldId);
    auto comm = world.getDeviceComm(rank);
    GA_CHECK(comm != nullptr);
    const size_t big = (size_t)T * STRIDE * size;
    DevBuffer a(big, BufferMemory::Heap);
    DevBuffer b(big, BufferMemory::Heap);
    GA_CHECK(a.ptr && b.ptr);
    std::vector<MPI_Request> reqs(T);
    std::vector<int> all;
    for (int p = 0; p < size; p++) {
        all.push_back(p);
    }

    if (!grouped) {
        // ---- grouping off: every call is one kernel at issue
        for (int round = 0; round < 2; round++) {
            fill(a, b, rank, size, round);
            MPI_Barrier(MPI_COMM_WORLD);
            for (int t = 0; t < T; t++) {
                const uint64_t l0 = comm->stats().launches;
                GA_CHECK(issue(rank, a, b, size, t, MPI_COMM_WORLD, &reqs[t], why) == 0);
                GA_CHECK(comm->stats().launches == l0 + 1);
            }
            GA_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
            GA_CHECK(exchanged(b, rank, all, rank, round, 0, T, why));
        }
        MPI_Barrier(MPI_COMM_WORLD);
        return 0;
    }

    // ---- bursts on the world: one grouped launch each
    for (int round = 0; round < 3; round++) {
        MPI_Barrier(MPI_COMM_WORLD);
        GA_CHECK(burst(rank, a, b, MPI_COMM_WORLD, all, round, comm, why) == 0);
    }

    // ---- an MPI_Iallgather flushes the pending burst (another key): three
    // launches, the first at the all-gather's issue
    {
        fill(a, b, rank, size, 5);
        DevBuffer g(STRIDE * size, BufferMemory::Heap);
        GA_CHECK(g.ptr != nullptr);
        for (int j = 0; j < 4; j++) {
            g.host[j] = rank * 10 + j;
        }
        g.upload();
        MPI_Barrier(MPI_COMM_WORLD);
        const uint64_t l0 = comm->stats().launches;
        for (int t = 0; t < T / 2; t++) {
            GA_CHECK(issue(rank, a, b, size, t, MPI_COMM_WORLD, &reqs[t], why) == 0);
        }
        MPI_Request ag;
        GA_CHECK(MPI_Iallgather(g.ptr, 4, MPI_INT, g.ptr + STRIDE, 4, MPI_INT, MPI_COMM_WORLD, &ag) == MPI_SUCCESS);
        GA_CHECK(comm->stats().launches == l0 + 1);
        for (int t = T / 2; t < T; t++) {
            GA_CHECK(issue(rank, a, b, size, t, MPI_COMM_WORLD, &reqs[t], why) == 0);
        }
        GA_CHECK(comm->stats().launches == l0 + 2);
        GA_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GA_CHECK(MPI_Wait(&ag, MPI_STATUS_IGNORE) == MPI_SUCCESS);
        GA_CHECK(comm->stats().launches == l0 + 3);
        GA_CHECK(exchanged(b, rank, all, rank, 5, 0, T, why));
        const auto& got = g.read();
        for (int q = 0; q < size; q++) {
            for (int j = 0; j < 4; j++) {
                GA_CHECK(got[STRIDE + q * 4 + j] == q * 10 + j);
            }
        }
    }

    // ---- a blocking collective flushes the pending burst before it runs
    {
        fill(a, b, rank, size, 6);
        DevBuffer s(16, BufferMemory::Heap);
        GA_CHECK(s.ptr != nullptr);
        for (int j = 0; j < 16; j++) {
            s.host[j] = rank + j;
        }
        s.upload();
        MPI_Barrier(MPI_COMM_WORLD);
        const uint64_t l0 = comm->stats().launches;
        for (int t = 0; t < T; t++) {
            GA_CHECK(issue(rank, a, b, size, t, MPI_COMM_WORLD, &reqs[t], why) == 0);
        }
        GA_CHECK(comm->stats().launches == l0);
        GA_CHECK(MPI_Allreduce(MPI_IN_PLACE, s.ptr, 16, MPI_INT, MPI_SUM, MPI_COMM_WORLD) == MPI_SUCCESS);
        const uint64_t l1 = comm->stats().launches;
        GA_CHECK(l1 >= l0 + 2);
        GA_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GA_CHECK(comm->stats().launches == l1);
        GA_CHECK(exchanged(b, rank, all, rank, 6, 0, T, why));
        const auto& got = s.read();
        for (int j = 0; j < 16; j++) {
            GA_CHECK(got[j] == size * (size - 1) / 2 + size * j);
        }
    }

    // ---- a block that is not a multiple of 16 bytes runs at issue
    {
        fill(a, b, rank, size, 0);
        MPI_Barrier(MPI_COMM_WORLD);
        const uint64_t l0 = comm->stats().launches;
        MPI_Request r;
        GA_CHECK(MPI_Ialltoall(a.ptr, 3, MPI_INT, b.ptr, 3, MPI_INT, MPI_COMM_WORLD, &r) == MPI_SUCCESS);
        GA_CHECK(comm->stats().launches == l0 + 1);
        GA_CHECK(MPI_Wait(&r, MPI_STATUS_IGNORE) == MPI_SUCCESS);
        const auto& got = b.read();
        for (int i = 0; i < STRIDE * size; i++) {
            // block q (3 words) of b: words 3*rank .. 3*rank+2 of member q's
            // send, whose words run over tensor 0's 4-word blocks
            const int w = 3 * rank + i % 3;
            GA_CHECK(got[i] == (i < 3 * size ? aIn(i / 3, 0, w / 4, w % 4, 0) : -1 - rank));
        }
    }

    // ---- host buffers complete at issue
    {
        std::vector<int32_t> hs(3 * size), hr(3 * size, -1);
        for (int i = 0; i < 3 * size; i++) {
            hs[i] = rank * 100 + i;
        }
        MPI_Request r;
        GA_CHECK(MPI_Ialltoall(hs.data(), 3, MPI_INT, hr.data(), 3, MPI_INT, MPI_COMM_WORLD, &r) == MPI_SUCCESS);
        for (int q = 0; q < size; q++) {
            for (int j = 0; j < 3; j++) {
                GA_CHECK(hr[q * 3 + j] == q * 100 + rank * 3 + j);
            }
        }
        GA_CHECK(MPI_Wait(&r, MPI_STATUS_IGNORE) == MPI_SUCCESS);
    }

    // ---- refusals at issue: nothing deferred or launched, outputs untouched
    {
        fill(a, b, rank, size, 0);
        const uint64_t l0 = comm->stats().launches;
        MPI_Request r;
        GA_CHECK(MPI_Ialltoall(MPI_IN_PLACE, 4, MPI_INT, b.ptr, 4, MPI_INT, MPI_COMM_WORLD, &r) == MPI_ERR_ARG);
        GA_CHECK(MPI_Ialltoall(a.ptr, 4, MPI_INT, b.ptr, 3, MPI_INT, MPI_COMM_WORLD, &r) == MPI_ERR_ARG);
        GA_CHECK(MPI_Ialltoall(a.ptr, 4, MPI_INT, b.ptr, 4, MPI_DOUBLE, MPI_COMM_WORLD, &r) == MPI_ERR_ARG);
        std::vector<int32_t> hs(4 * size, 1), hr(4 * size, 9);
        GA_CHECK(MPI_Ialltoall(hs.data(), 4, MPI_INT, hr.data(), 2, MPI_INT, MPI_COMM_WORLD, &r) == MPI_ERR_ARG);
        for (int v : hr) {
            GA_CHECK(v == 9);
        }
        GA_CHECK(comm->stats().launches == l0);
        GA_CHECK(exchanged(b, rank, all, rank, 0, 0, 0, why));
        // (the same counts in other types are equal byte counts: accepted)
        GA_CHECK(MPI_Ialltoall(a.ptr, 8, MPI_INT, b.ptr, 4, MPI_DOUBLE, MPI_COMM_WORLD, &r) == MPI_SUCCESS);
        GA_CHECK(MPI_Wait(&r, MPI_STATUS_IGNORE) == MPI_SUCCESS);
        GA_CHECK(comm->stats().launches == l0 + 1);
    }

    // ---- parity split: bursts on the child
    MPI_Comm sub;
    GA_CHECK(MPI_Comm_split(MPI_COMM_WORLD, rank % 2, rank, &sub) == MPI_SUCCESS);
    int srank = -1, ssize = -1;
    MPI_Comm_rank(sub, &srank);
    MPI_Comm_size(sub, &ssize);
    std::vector<int> members;
    for (int p = rank % 2; p < size; p += 2) {
        members.push_back(p);
    }
    GA_CHECK(ssize == (int)members.size() && members[srank] == rank);
    // (the first device collective on the child agrees its slot)
    GA_CHECK(MPI_Allreduce(MPI_IN_PLACE, b.ptr, 4, MPI_INT, MPI_SUM, sub) == MPI_SUCCESS);
    for (int round = 0; round < 3; round++) {
        GA_CHECK(burst(rank, a, b, sub, members, 10 + round, comm, why) == 0);
        // the world's bursts in between still launch on the world
        GA_CHECK(burst(rank, a, b, MPI_COMM_WORLD, all, 20 + round, comm, why) == 0);
    }

    // ---- a split of the split: its own child, bursts of one launch
    {
        MPI_Comm nested;
        GA_CHECK(MPI_Comm_split(sub, srank % 2, srank, &nested) == MPI_SUCCESS);
        int nrank = -1, nsize = -1;
        MPI_Comm_rank(nested, &nrank);
        MPI_Comm_size(nested, &nsize);
        std::vector<int> nmembers;
        for (int q = srank % 2; q < ssize; q += 2) {
            nmembers.push_back(members[q]);
        }
        GA_CHECK(nsize == (int)nmembers.size() && nmembers[nrank] == rank);
        GA_CHECK(MPI_Allreduce(MPI_IN_PLACE, b.ptr, 4, MPI_INT, MPI_SUM, nested) == MPI_SUCCESS);
        for (int round = 0; round < 2; round++) {
            GA_CHECK(burst(rank, a, b, nested, nmembers, 30 + round, comm, why) == 0);
        }
        GA_CHECK(MPI_Comm_free(&nested) == MPI_SUCCESS);
    }

    // ---- MPI_Comm_free with a burst pending: it is issued and completed
    {
        fill(a, b, rank, ssize, 40);
        for (int t = 0; t < T; t++) {
            GA_CHECK(issue(rank, a, b, ssize, t, sub, &reqs[t], why) == 0);
        }
        GA_CHECK(MPI_Comm_free(&sub) == MPI_SUCCESS);
        GA_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GA_CHECK(exchanged(b, rank, members, srank, 40, 0, T, why));
    }
    MPI_Barrier(MPI_COMM_WORLD);
    return 0;
}

#undef GA_CHECK

}
