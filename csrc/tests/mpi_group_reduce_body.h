// One MPI program for MPI_Ireduce bursts on the world and on MPI_Comm_split
// halves.  Shared by the loopback test (test_loopback_group_reduce.cpp), the
// GPU test (test_device_group_reduce.cpp), both through
// mpi_group_reduce_run.h, and faabric_worker's `group-reduce` program, which
// tests/test_dist_group_reduce.py runs with one rank in each of four worker
// processes.
//
// Bursts on device memory (MPI_Alloc_mem(MPI_INFO_FAABRIC_DEVICE), at word
// offsets that are not 16-byte aligned, with word counts that are not a
// multiple of four) launch nothing before the first wait and one grouped
// kernel after it, with every root and with in-place roots.  A change of
// root, op or datatype flushes the pending burst; back-to-back bursts and a
// blocking MPI_Reduce after a burst reuse the staging buffers; host buffers
// complete at issue; a pair no reduction takes gives MPI_ERR_OP and a root
// outside the communicator MPI_ERR_ARG, on every rank with nothing issued;
// MPI_Comm_free with a pending burst completes it.  With grouping off
// (FAABRIC_MPI_GROUP_IALLREDUCE=0) every call runs one kernel at issue.
// Every word, guard words and every non-root's recv included, is compared
// against a closed form (integer-valued sums and maxima, exact in float).
#pragma once

#include "mpi/subcomm.h"
#include "mpi_subcomm_device_body.h"

#include <faabric/mpi/MpiWorld.h>
#include <faabric/mpi/MpiWorldRegistry.h>
#include <faabric/mpi/mpi.h>

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

namespace group_reduce {

using subcomm_device::BufferMemory;
using subcomm_device::DevBuffer;

#define GRD_CHECK(cond)                                                        \
    do {                                                                       \
        if (!(cond)) {                                                         \
            *why = "rank " + std::to_string(rank) + ": check failed at line " + std::to_string(__LINE__) + ": " #cond; \
            return 1;                                                          \
        }                                                                      \
    } while (0)

constexpr int T = 8;       // tensors per burst
constexpr int STRIDE = 32; // words per tensor slot

// Length of tensor t in words: 1, 4, 7, ... 22 (odd byte counts of 16)
inline int len(int t)
{
    return 1 + 3 * t;
}

// Tensor t starts at word 1 + t * STRIDE (off 16-byte alignment)
inline size_t at(int t)
{
    return 1 + (size_t)t * STRIDE;
}

// Word j of tensor t in world rank r's send, in round `salt`
inline int64_t value(int r, int t, int j, int salt)
{
    return r * 1000 + t * 37 + j + salt * 7;
}

inline int32_t guard(int rank)
{
    return -1 - rank;
}

// One call's reduction: MPI_SUM or MPI_MAX on MPI_INT or MPI_FLOAT
struct Call
{
    MPI_Op op;
    bool flt;
};

inline int32_t bits(bool flt, int64_t v)
{
    if (!flt) {
        return (int32_t)v;
    }
    const float f = (float)v;
    int32_t out;
    memcpy(&out, &f, 4);
    return out;
}

struct Burst
{
    MPI_Comm comm;
    std::vector<int> members; // world ranks in comm rank order
    int root;
    bool inPlace;
    int salt;
    Call calls[T]; // tensor t's op and datatype
};

inline Burst uniform(MPI_Comm comm, const std::vector<int>& members, int root, bool inPlace, int salt, Call c)
{
    Burst b{ comm, members, root, inPlace, salt, {} };
    std::fill(b.calls, b.calls + T, c);
    return b;
}

// a: this rank's sends; r: guard words, except that an in-place root holds
// its own contribution
inline void fill(const Burst& b, DevBuffer& a, DevBuffer& r, int rank, int cr)
{
    std::fill(a.host.begin(), a.host.end(), -7);
    std::fill(r.host.begin(), r.host.end(), guard(rank));
    for (int t = 0; t < T; t++) {
        for (int j = 0; j < len(t); j++) {
            a.host[at(t) + j] = bits(b.calls[t].flt, value(rank, t, j, b.salt));
            if (b.inPlace && cr == b.root) {
                r.host[at(t) + j] = a.host[at(t) + j];
            }
        }
    }
    a.upload();
    r.upload();
}

inline int issue(const Burst& b, DevBuffer& a, DevBuffer& r, int t, int rank, int cr, MPI_Request* req, std::string* why)
{
    const bool own = b.inPlace && cr == b.root;
    const Call c = b.calls[t];
    GRD_CHECK(MPI_Ireduce(own ? MPI_IN_PLACE : (const void*)(a.ptr + at(t)), r.ptr + at(t), len(t),
                          c.flt ? MPI_FLOAT : MPI_INT, c.op, b.root, b.comm, req) == MPI_SUCCESS);
    return 0;
}

// r after the burst: the fold at the root, guard words everywhere else
inline int check(const Burst& b, DevBuffer& r, int rank, int cr, std::string* why)
{
    const auto& got = r.read();
    for (size_t i = 0; i < got.size(); i++) {
        int32_t want = guard(rank);
        for (int t = 0; t < T; t++) {
            if (cr != b.root || i < at(t) || i >= at(t) + (size_t)len(t)) {
                continue;
            }
            const int j = (int)(i - at(t));
            int64_t acc = value(b.members[0], t, j, b.salt);
            for (size_t p = 1; p < b.members.size(); p++) {
                const int64_t v = value(b.members[p], t, j, b.salt);
                acc = b.calls[t].op == MPI_MAX ? std::max(acc, v) : acc + v;
            }
            want = bits(b.calls[t].flt, acc);
        }
        if (got[i] != want) {
            *why = "rank " + std::to_string(rank) + " word " + std::to_string(i) + ": " + std::to_string(got[i]) +
                   ", want " + std::to_string(want) + " (root " + std::to_string(b.root) + ")";
            return 1;
        }
    }
    return 0;
}

// A burst of T calls: nothing launched before the wait (grouped), `flushes`
// launches at issue and one more after it; or one launch per call at issue
// (grouping off)
inline int burst(const Burst& b, DevBuffer& a, DevBuffer& r, int rank, bool grouped,
                 const std::shared_ptr<faabric::device::Communicator>& world, std::string* why, int flushes = 0)
{
    int cr = -1;
    MPI_Comm_rank(b.comm, &cr);
    fill(b, a, r, rank, cr);
    MPI_Barrier(b.comm);
    std::vector<MPI_Request> reqs(T);
    GRD_CHECK(issue(b, a, r, 0, rank, cr, &reqs[0], why) == 0);
    auto sub = faabric::mpi::getSubCommunicator(b.comm->id);
    auto dev = b.comm == MPI_COMM_WORLD ? world : (sub == nullptr ? nullptr : sub->currentDevice(rank));
    GRD_CHECK(dev != nullptr && dev->size() == (int)b.members.size());
    const uint64_t l0 = dev->stats().launches;
    for (int t = 1; t < T; t++) {
        GRD_CHECK(issue(b, a, r, t, rank, cr, &reqs[t], why) == 0);
    }
    GRD_CHECK(dev->stats().launches == l0 + (grouped ? flushes : T - 1));
    GRD_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
    GRD_CHECK(dev->stats().launches == l0 + (grouped ? flushes + 1 : T - 1));
    return check(b, r, rank, cr, why);
}

inline int body(int rank, int size, int worldId, bool grouped, std::string* why)
{
    auto& world = faabric::mpi::getMpiWorldRegistry().getWorld(worldId);
    auto comm = world.getDeviceComm(rank);
    GRD_CHECK(comm != nullptr);
    const size_t words = at(T) + 8;
    DevBuffer a(words, BufferMemory::Heap), r(words, BufferMemory::Heap);
    DevBuffer a2(words, BufferMemory::Heap), r2(words, BufferMemory::Heap);
    GRD_CHECK(a.ptr && r.ptr && a2.ptr && r2.ptr);
    std::vector<int> all;
    for (int p = 0; p < size; p++) {
        all.push_back(p);
    }
    const Call isum{ MPI_SUM, false }, imax{ MPI_MAX, false }, fsum{ MPI_SUM, true };

    // ---- every root, in place and not, on the world
    for (int root = 0; root < size; root++) {
        for (int inPlace = 0; inPlace < 2; inPlace++) {
            const Burst b = uniform(MPI_COMM_WORLD, all, root, inPlace == 1, root * 2 + inPlace, inPlace ? fsum : isum);
            GRD_CHECK(burst(b, a, r, rank, grouped, comm, why) == 0);
        }
    }
    if (!grouped) {
        MPI_Barrier(MPI_COMM_WORLD);
        return 0;
    }

    // ---- a change of root, op or datatype flushes: each splits the burst
    // in two launches
    for (int change = 0; change < 3; change++) {
        Burst b = uniform(MPI_COMM_WORLD, all, 0, false, 3 + change, isum);
        for (int t = T / 2; t < T; t++) {
            b.calls[t] = change == 1 ? imax : change == 2 ? fsum : isum;
        }
        if (change == 0) {
            // (the second half to the last rank: two bursts, one Burst each)
            Burst b1 = uniform(MPI_COMM_WORLD, all, size - 1, false, 3, isum);
            fill(b, a, r, rank, rank);
            MPI_Barrier(MPI_COMM_WORLD);
            std::vector<MPI_Request> reqs(T);
            const uint64_t l0 = comm->stats().launches;
            for (int t = 0; t < T; t++) {
                GRD_CHECK(issue(t < T / 2 ? b : b1, a, r, t, rank, rank, &reqs[t], why) == 0);
            }
            GRD_CHECK(comm->stats().launches == l0 + 1);
            GRD_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
            GRD_CHECK(comm->stats().launches == l0 + 2);
            const auto& got = r.read();
            for (int t = 0; t < T; t++) {
                const int root = t < T / 2 ? 0 : size - 1;
                for (int j = 0; j < len(t); j++) {
                    int64_t sum = 0;
                    for (int p = 0; p < size; p++) {
                        sum += value(p, t, j, 3);
                    }
                    GRD_CHECK(got[at(t) + j] == (rank == root ? (int32_t)sum : guard(rank)));
                }
            }
            continue;
        }
        GRD_CHECK(burst(b, a, r, rank, true, comm, why, 1) == 0);
    }

    // ---- back-to-back bursts and a blocking MPI_Reduce after a burst: all
    // reuse the staging buffers
    {
        const Burst g = uniform(MPI_COMM_WORLD, all, size - 1, false, 8, imax);
        const Burst s = uniform(MPI_COMM_WORLD, all, 0, false, 9, isum);
        fill(g, a, r, rank, rank);
        fill(s, a2, r2, rank, rank);
        MPI_Barrier(MPI_COMM_WORLD);
        std::vector<MPI_Request> reqs(2 * T);
        for (int t = 0; t < T; t++) {
            GRD_CHECK(issue(g, a, r, t, rank, rank, &reqs[t], why) == 0);
        }
        for (int t = 0; t < T; t++) {
            GRD_CHECK(issue(s, a2, r2, t, rank, rank, &reqs[T + t], why) == 0);
        }
        // blocking reduce of 5 words (staged)
        DevBuffer bs(6, BufferMemory::Heap), br(6, BufferMemory::Heap);
        GRD_CHECK(bs.ptr != nullptr && br.ptr != nullptr);
        for (int j = 0; j < 5; j++) {
            bs.host[1 + j] = rank * 10 + j;
        }
        bs.upload();
        GRD_CHECK(MPI_Reduce(bs.ptr + 1, br.ptr + 1, 5, MPI_INT, MPI_SUM, 0, MPI_COMM_WORLD) == MPI_SUCCESS);
        GRD_CHECK(MPI_Waitall(2 * T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GRD_CHECK(check(g, r, rank, rank, why) == 0);
        GRD_CHECK(check(s, r2, rank, rank, why) == 0);
        if (rank == 0) {
            const auto& got = br.read();
            for (int j = 0; j < 5; j++) {
                GRD_CHECK(got[1 + j] == 10 * size * (size - 1) / 2 + size * j);
            }
        }
    }

    // ---- host buffers complete at issue
    {
        std::vector<int32_t> hs(3), hr(3, -1);
        for (int j = 0; j < 3; j++) {
            hs[j] = rank * 100 + j;
        }
        MPI_Request q;
        GRD_CHECK(MPI_Ireduce(hs.data(), hr.data(), 3, MPI_INT, MPI_SUM, 0, MPI_COMM_WORLD, &q) == MPI_SUCCESS);
        for (int j = 0; j < 3; j++) {
            GRD_CHECK(hr[j] == (rank == 0 ? 100 * size * (size - 1) / 2 + size * j : -1));
        }
        GRD_CHECK(MPI_Wait(&q, MPI_STATUS_IGNORE) == MPI_SUCCESS);
    }

    // ---- refusals: MPI_ERR_OP, MPI_ERR_ARG, nothing issued
    {
        const Burst b = uniform(MPI_COMM_WORLD, all, 0, false, 0, isum);
        fill(b, a, r, rank, rank);
        const uint64_t l0 = comm->stats().launches;
        MPI_Request q;
        GRD_CHECK(MPI_Ireduce(a.ptr + 1, r.ptr + 1, 4, MPI_FLOAT, MPI_BAND, 0, MPI_COMM_WORLD, &q) == MPI_ERR_OP);
        GRD_CHECK(MPI_Ireduce(a.ptr + 1, r.ptr + 1, 4, MPI_INT, MPI_REPLACE, 0, MPI_COMM_WORLD, &q) == MPI_ERR_OP);
        GRD_CHECK(MPI_Ireduce(a.ptr + 1, r.ptr + 1, 4, MPI_INT, MPI_SUM, size, MPI_COMM_WORLD, &q) == MPI_ERR_ARG);
        GRD_CHECK(MPI_Ireduce(a.ptr + 1, r.ptr + 1, 4, MPI_INT, MPI_SUM, -1, MPI_COMM_WORLD, &q) == MPI_ERR_ARG);
        MPI_Barrier(MPI_COMM_WORLD);
        GRD_CHECK(comm->stats().launches == l0);
        const auto& got = r.read();
        for (int32_t v : got) {
            GRD_CHECK(v == guard(rank));
        }
    }

    // ---- parity split: bursts on the child, every root, world bursts between
    MPI_Comm sub;
    GRD_CHECK(MPI_Comm_split(MPI_COMM_WORLD, rank % 2, rank, &sub) == MPI_SUCCESS);
    int srank = -1, ssize = -1;
    MPI_Comm_rank(sub, &srank);
    MPI_Comm_size(sub, &ssize);
    std::vector<int> members;
    for (int p = rank % 2; p < size; p += 2) {
        members.push_back(p);
    }
    GRD_CHECK(ssize == (int)members.size() && members[srank] == rank);
    // (the first device collective on the child agrees its slot)
    GRD_CHECK(MPI_Allreduce(MPI_IN_PLACE, r.ptr, 4, MPI_INT, MPI_SUM, sub) == MPI_SUCCESS);
    for (int root = 0; root < ssize; root++) {
        const Burst b = uniform(sub, members, root, root == ssize - 1, 50 + root, root % 2 ? imax : isum);
        GRD_CHECK(burst(b, a, r, rank, true, comm, why) == 0);
        const Burst w = uniform(MPI_COMM_WORLD, all, root, false, 60 + root, fsum);
        GRD_CHECK(burst(w, a2, r2, rank, true, comm, why) == 0);
    }

    // ---- MPI_Comm_free with a burst pending: it is issued and completed
    {
        const Burst b = uniform(sub, members, 0, false, 70, isum);
        fill(b, a, r, rank, srank);
        MPI_Barrier(sub);
        std::vector<MPI_Request> reqs(T);
        for (int t = 0; t < T; t++) {
            GRD_CHECK(issue(b, a, r, t, rank, srank, &reqs[t], why) == 0);
        }
        GRD_CHECK(MPI_Comm_free(&sub) == MPI_SUCCESS);
        GRD_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GRD_CHECK(check(b, r, rank, srank, why) == 0);
    }
    MPI_Barrier(MPI_COMM_WORLD);
    return 0;
}

#undef GRD_CHECK

}
