// One MPI program for MPI_Igather and MPI_Iscatter bursts on the world and on
// MPI_Comm_split halves.  Shared by the loopback test
// (test_loopback_group_rooted.cpp), the GPU test
// (test_device_group_rooted.cpp), both through mpi_group_rooted_run.h, and
// faabric_worker's `group-rooted` program, which
// tests/test_dist_group_rooted.py runs with one rank in each of four worker
// processes.
//
// Bursts on device memory (MPI_Alloc_mem(MPI_INFO_FAABRIC_DEVICE), at word
// offsets that are not 16-byte aligned, with word counts that are not a
// multiple of four) launch nothing before the first wait and one grouped
// kernel after it, with every root and with in-place roots.  A change of
// root flushes the pending burst; a blocking staged collective after a burst,
// and a scatter burst right after a gather burst, reuse the staging buffer;
// host buffers complete at issue; a root outside the communicator gives
// MPI_ERR_ARG on every rank with nothing issued; MPI_Comm_free with a pending
// burst completes it.  With grouping off (FAABRIC_MPI_GROUP_IALLREDUCE=0)
// every call runs one kernel at issue.  Every word, guard words included, is
// compared against a closed form.
#pragma once

#include "mpi/subcomm.h"
#include "mpi_subcomm_device_body.h"

#include <faabric/mpi/MpiWorld.h>
#include <faabric/mpi/MpiWorldRegistry.h>
#include <faabric/mpi/mpi.h>

#include <cstdint>
#include <string>
#include <vector>

namespace group_rooted {

using subcomm_device::BufferMemory;
using subcomm_device::DevBuffer;

#define GR_CHECK(cond)                                                         \
    do {                                                                       \
        if (!(cond)) {                                                         \
            *why = "rank " + std::to_string(rank) + ": check failed at line " + std::to_string(__LINE__) + ": " #cond; \
            return 1;                                                          \
        }                                                                      \
    } while (0)

constexpr int T = 8;       // tensors per burst
constexpr int STRIDE = 32; // int32 per block slot: tensor t of m blocks owns m * STRIDE int32

// Block length of tensor t in int32: 1, 4, 7, ... 22 (odd byte counts of 16)
inline int blk(int t)
{
    return 1 + 3 * t;
}

// Word j of block q of tensor t in world rank r's send, in round `salt`
inline int32_t aIn(int r, int t, int q, int j, int salt)
{
    return r * 100000 + t * 1000 + q * 40 + j + salt * 7;
}

inline int32_t guard(int rank)
{
    return -1 - rank;
}

inline std::shared_ptr<faabric::device::Communicator> childOf(MPI_Comm comm, int rank)
{
    auto sub = faabric::mpi::getSubCommunicator(comm->id);
    return sub == nullptr ? nullptr : sub->currentDevice(rank);
}

// Tensor t of a and b starts at word 1 + t * m * STRIDE (off 16-byte
// alignment).  a: this rank's m blocks (the gather send is block 0, the
// scatter send all of them); b: guard words, except that an in-place gather
// root holds its own contribution in its block.
struct Burst
{
    bool gather;
    MPI_Comm comm;
    std::vector<int> members; // world ranks in comm rank order
    int root;
    bool inPlace;
    int salt;
};

inline size_t at(int t, int m)
{
    return 1 + (size_t)t * m * STRIDE;
}

inline void fill(const Burst& b, DevBuffer& a, DevBuffer& r, int rank, int cr)
{
    const int m = (int)b.members.size();
    for (auto& v : a.host) {
        v = -7;
    }
    for (auto& v : r.host) {
        v = guard(rank);
    }
    for (int t = 0; t < T; t++) {
        for (int q = 0; q < m; q++) {
            for (int j = 0; j < blk(t); j++) {
                a.host[at(t, m) + q * blk(t) + j] = aIn(rank, t, q, j, b.salt);
                if (b.gather && b.inPlace && cr == b.root && q == cr) {
                    r.host[at(t, m) + q * blk(t) + j] = aIn(rank, t, 0, j, b.salt);
                }
            }
        }
    }
    a.upload();
    r.upload();
}

inline int issue(const Burst& b, DevBuffer& a, DevBuffer& r, int t, int rank, int cr, MPI_Request* req, std::string* why)
{
    const int m = (int)b.members.size();
    const bool own = b.inPlace && cr == b.root;
    if (b.gather) {
        GR_CHECK(MPI_Igather(own ? MPI_IN_PLACE : (const void*)(a.ptr + at(t, m)), blk(t), MPI_INT, r.ptr + at(t, m),
                             blk(t), MPI_INT, b.root, b.comm, req) == MPI_SUCCESS);
    } else {
        GR_CHECK(MPI_Iscatter(a.ptr + at(t, m), blk(t), MPI_INT, own ? MPI_IN_PLACE : (void*)(r.ptr + at(t, m)), blk(t),
                              MPI_INT, b.root, b.comm, req) == MPI_SUCCESS);
    }
    return 0;
}

// r after tensors [0, T) of the burst (an in-place scatter root keeps its
// guard words: its block stays in a)
inline int check(const Burst& b, DevBuffer& r, int rank, int cr, std::string* why)
{
    const int m = (int)b.members.size();
    const auto& got = r.read();
    for (size_t i = 0; i < got.size(); i++) {
        int32_t want = guard(rank);
        for (int t = 0; t < T; t++) {
            if (i < at(t, m) || i >= at(t, m) + (size_t)m * blk(t)) {
                continue;
            }
            const int k = (int)(i - at(t, m));
            if (b.gather && cr == b.root) {
                want = aIn(b.members[k / blk(t)], t, 0, k % blk(t), b.salt);
            } else if (!b.gather && k < blk(t) && !(b.inPlace && cr == b.root)) {
                want = aIn(b.members[b.root], t, cr, k, b.salt);
            }
        }
        if (got[i] != want) {
            *why = "rank " + std::to_string(rank) + " word " + std::to_string(i) + ": " + std::to_string(got[i]) +
                   ", want " + std::to_string(want) + (b.gather ? " (gather" : " (scatter") + " root " +
                   std::to_string(b.root) + ")";
            return 1;
        }
    }
    return 0;
}

// A burst of T calls: nothing launched before the wait (grouped), one launch
// after it; or one launch per call at issue (grouping off)
inline int burst(const Burst& b, DevBuffer& a, DevBuffer& r, int rank, bool grouped,
                 const std::shared_ptr<faabric::device::Communicator>& world, std::string* why)
{
    int cr = -1;
    MPI_Comm_rank(b.comm, &cr);
    fill(b, a, r, rank, cr);
    MPI_Barrier(b.comm);
    std::vector<MPI_Request> reqs(T);
    GR_CHECK(issue(b, a, r, 0, rank, cr, &reqs[0], why) == 0);
    auto dev = b.comm == MPI_COMM_WORLD ? world : childOf(b.comm, rank);
    GR_CHECK(dev != nullptr && dev->size() == (int)b.members.size());
    const uint64_t l0 = dev->stats().launches;
    for (int t = 1; t < T; t++) {
        GR_CHECK(issue(b, a, r, t, rank, cr, &reqs[t], why) == 0);
    }
    GR_CHECK(dev->stats().launches == l0 + (grouped ? 0 : T - 1));
    GR_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
    GR_CHECK(dev->stats().launches == l0 + (grouped ? 1 : T - 1));
    return check(b, r, rank, cr, why);
}

inline int body(int rank, int size, int worldId, bool grouped, std::string* why)
{
    auto& world = faabric::mpi::getMpiWorldRegistry().getWorld(worldId);
    auto comm = world.getDeviceComm(rank);
    GR_CHECK(comm != nullptr);
    const size_t words = at(T, size) + 8;
    DevBuffer a(words, BufferMemory::Heap), r(words, BufferMemory::Heap);
    DevBuffer a2(words, BufferMemory::Heap), r2(words, BufferMemory::Heap);
    GR_CHECK(a.ptr && r.ptr && a2.ptr && r2.ptr);
    std::vector<int> all;
    for (int p = 0; p < size; p++) {
        all.push_back(p);
    }

    // ---- every root, in place and not, on the world
    for (int gather = 0; gather < 2; gather++) {
        for (int root = 0; root < size; root++) {
            for (int inPlace = 0; inPlace < 2; inPlace++) {
                const Burst b{ gather == 1, MPI_COMM_WORLD, all, root, inPlace == 1, root * 2 + inPlace };
                GR_CHECK(burst(b, a, r, rank, grouped, comm, why) == 0);
            }
        }
    }
    if (!grouped) {
        MPI_Barrier(MPI_COMM_WORLD);
        return 0;
    }

    // ---- a change of root flushes: half the tensors to root 0, half to the
    // last rank, two launches
    {
        const Burst b0{ true, MPI_COMM_WORLD, all, 0, false, 3 };
        const Burst b1{ true, MPI_COMM_WORLD, all, size - 1, false, 3 };
        fill(b0, a, r, rank, rank);
        MPI_Barrier(MPI_COMM_WORLD);
        std::vector<MPI_Request> reqs(T);
        const uint64_t l0 = comm->stats().launches;
        for (int t = 0; t < T; t++) {
            GR_CHECK(issue(t < T / 2 ? b0 : b1, a, r, t, rank, rank, &reqs[t], why) == 0);
        }
        GR_CHECK(comm->stats().launches == l0 + (size > 1 ? 1 : 0));
        GR_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GR_CHECK(comm->stats().launches == l0 + (size > 1 ? 2 : 1));
        const auto& got = r.read();
        for (int t = 0; t < T; t++) {
            const int root = t < T / 2 ? 0 : size - 1;
            for (int k = 0; k < size * blk(t); k++) {
                const int32_t want = rank == root ? aIn(k / blk(t), t, 0, k % blk(t), 3) : guard(rank);
                GR_CHECK(got[at(t, size) + k] == want);
            }
        }
    }

    // ---- back-to-back bursts (a scatter right after a gather: the kind
    // change flushes the gather) and a blocking staged collective after a
    // burst: all reuse the staging buffers
    {
        const Burst g{ true, MPI_COMM_WORLD, all, size - 1, false, 8 };
        const Burst s{ false, MPI_COMM_WORLD, all, 0, false, 9 };
        fill(g, a, r, rank, rank);
        fill(s, a2, r2, rank, rank);
        MPI_Barrier(MPI_COMM_WORLD);
        std::vector<MPI_Request> reqs(2 * T);
        for (int t = 0; t < T; t++) {
            GR_CHECK(issue(g, a, r, t, rank, rank, &reqs[t], why) == 0);
        }
        for (int t = 0; t < T; t++) {
            GR_CHECK(issue(s, a2, r2, t, rank, rank, &reqs[T + t], why) == 0);
        }
        // blocking gather of 5 words of a2's tail into r2's tail (staged)
        DevBuffer bg(5 * size + 3, BufferMemory::Heap);
        GR_CHECK(bg.ptr != nullptr);
        std::vector<int32_t> mine(5);
        for (int j = 0; j < 5; j++) {
            mine[j] = rank * 10 + j;
        }
        DevBuffer bs(5, BufferMemory::Heap);
        GR_CHECK(bs.ptr != nullptr);
        bs.host = mine;
        bs.upload();
        GR_CHECK(MPI_Gather(bs.ptr, 5, MPI_INT, bg.ptr + 1, 5, MPI_INT, 0, MPI_COMM_WORLD) == MPI_SUCCESS);
        GR_CHECK(MPI_Waitall(2 * T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GR_CHECK(check(g, r, rank, rank, why) == 0);
        GR_CHECK(check(s, r2, rank, rank, why) == 0);
        if (rank == 0) {
            const auto& got = bg.read();
            for (int k = 0; k < 5 * size; k++) {
                GR_CHECK(got[1 + k] == (k / 5) * 10 + k % 5);
            }
        }
    }

    // ---- host buffers complete at issue
    {
        std::vector<int32_t> hs(3), hr(3 * size, -1);
        for (int j = 0; j < 3; j++) {
            hs[j] = rank * 100 + j;
        }
        MPI_Request q;
        GR_CHECK(MPI_Igather(hs.data(), 3, MPI_INT, hr.data(), 3, MPI_INT, 0, MPI_COMM_WORLD, &q) == MPI_SUCCESS);
        if (rank == 0) {
            for (int k = 0; k < 3 * size; k++) {
                GR_CHECK(hr[k] == (k / 3) * 100 + k % 3);
            }
        }
        GR_CHECK(MPI_Wait(&q, MPI_STATUS_IGNORE) == MPI_SUCCESS);
        std::vector<int32_t> ss(3 * size), sr(3, -1);
        for (int k = 0; k < 3 * size; k++) {
            ss[k] = k;
        }
        GR_CHECK(MPI_Iscatter(ss.data(), 3, MPI_INT, sr.data(), 3, MPI_INT, 0, MPI_COMM_WORLD, &q) == MPI_SUCCESS);
        for (int j = 0; j < 3; j++) {
            GR_CHECK(sr[j] == rank * 3 + j);
        }
        GR_CHECK(MPI_Wait(&q, MPI_STATUS_IGNORE) == MPI_SUCCESS);
    }

    // ---- a root outside the communicator: MPI_ERR_ARG, nothing issued
    {
        const Burst b{ true, MPI_COMM_WORLD, all, 0, false, 0 };
        fill(b, a, r, rank, rank);
        const uint64_t l0 = comm->stats().launches;
        MPI_Request q;
        GR_CHECK(MPI_Igather(a.ptr + 1, 4, MPI_INT, r.ptr + 1, 4, MPI_INT, size, MPI_COMM_WORLD, &q) == MPI_ERR_ARG);
        GR_CHECK(MPI_Iscatter(a.ptr + 1, 4, MPI_INT, r.ptr + 1, 4, MPI_INT, -1, MPI_COMM_WORLD, &q) == MPI_ERR_ARG);
        MPI_Barrier(MPI_COMM_WORLD);
        GR_CHECK(comm->stats().launches == l0);
        const auto& got = r.read();
        for (int32_t v : got) {
            GR_CHECK(v == guard(rank));
        }
    }

    // ---- parity split: bursts on the child, every root, world bursts between
    MPI_Comm sub;
    GR_CHECK(MPI_Comm_split(MPI_COMM_WORLD, rank % 2, rank, &sub) == MPI_SUCCESS);
    int srank = -1, ssize = -1;
    MPI_Comm_rank(sub, &srank);
    MPI_Comm_size(sub, &ssize);
    std::vector<int> members;
    for (int p = rank % 2; p < size; p += 2) {
        members.push_back(p);
    }
    GR_CHECK(ssize == (int)members.size() && members[srank] == rank);
    // (the first device collective on the child agrees its slot)
    GR_CHECK(MPI_Allreduce(MPI_IN_PLACE, r.ptr, 4, MPI_INT, MPI_SUM, sub) == MPI_SUCCESS);
    for (int gather = 0; gather < 2; gather++) {
        for (int root = 0; root < ssize; root++) {
            const Burst b{ gather == 1, sub, members, root, root == ssize - 1, 50 + root };
            GR_CHECK(burst(b, a, r, rank, true, comm, why) == 0);
            const Burst w{ gather == 0, MPI_COMM_WORLD, all, root, false, 60 + root };
            GR_CHECK(burst(w, a2, r2, rank, true, comm, why) == 0);
        }
    }

    // ---- MPI_Comm_free with a burst pending: it is issued and completed
    {
        const Burst b{ false, sub, members, 0, false, 70 };
        fill(b, a, r, rank, srank);
        MPI_Barrier(sub);
        std::vector<MPI_Request> reqs(T);
        for (int t = 0; t < T; t++) {
            GR_CHECK(issue(b, a, r, t, rank, srank, &reqs[t], why) == 0);
        }
        GR_CHECK(MPI_Comm_free(&sub) == MPI_SUCCESS);
        GR_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GR_CHECK(check(b, r, rank, srank, why) == 0);
    }
    MPI_Barrier(MPI_COMM_WORLD);
    return 0;
}

#undef GR_CHECK

}
