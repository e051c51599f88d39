// One MPI program for MPI_Iscan / MPI_Iexscan bursts and MPI_Exscan on the
// world and on MPI_Comm_split halves.  Shared by the loopback test
// (test_loopback_group_scan.cpp), the GPU test (test_device_group_scan.cpp),
// both through mpi_group_scan_run.h, and faabric_worker's `group-scan`
// program, which tests/test_dist_group_scan.py runs with one rank in each of
// four worker processes.
//
// Bursts on device memory (MPI_Alloc_mem(MPI_INFO_FAABRIC_DEVICE), at word
// offsets that are not 16-byte aligned, with word counts that are not a
// multiple of four) launch nothing before the first wait and one grouped
// kernel after it, with in place on some ranks only.  A change of kind, op or
// datatype flushes the pending burst; blocking MPI_Exscan runs on device and
// host buffers; host buffers, user-defined ops and zero counts complete at
// issue; a pair no reduction takes, MPI_REPLACE and MPI_NO_OP give MPI_ERR_OP
// on every rank with nothing issued; MPI_Comm_free with a pending burst
// completes it.  With grouping off (FAABRIC_MPI_GROUP_IALLREDUCE=0) every
// call runs one grouped launch at issue.  Every word, guard words and an
// exscan's untouched rank 0 included, is compared against a closed form
// (integer-valued sums and maxima, exact in float).
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

namespace group_scan {

using subcomm_device::BufferMemory;
using subcomm_device::DevBuffer;

#define GSC_CHECK(cond)                                                        \
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

// One call: MPI_Iscan or MPI_Iexscan, MPI_SUM or MPI_MAX on MPI_INT or
// MPI_FLOAT
struct Call
{
    MPI_Op op;
    bool flt;
    bool ex;
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
    unsigned inPlace;         // bit c: comm rank c passes MPI_IN_PLACE
    int salt;
    Call calls[T]; // tensor t's kind, op and datatype
};

inline Burst uniform(MPI_Comm comm, const std::vector<int>& members, unsigned inPlace, int salt, Call c)
{
    Burst b{ comm, members, inPlace, salt, {} };
    std::fill(b.calls, b.calls + T, c);
    return b;
}

inline bool ownInPlace(const Burst& b, int cr)
{
    return (b.inPlace >> cr) & 1u;
}

// a: this rank's sends; r: guard words, except that an in-place rank holds
// its own contribution
inline void fill(const Burst& b, DevBuffer& a, DevBuffer& r, int rank, int cr)
{
    std::fill(a.host.begin(), a.host.end(), -7);
    std::fill(r.host.begin(), r.host.end(), guard(rank));
    for (int t = 0; t < T; t++) {
        for (int j = 0; j < len(t); j++) {
            a.host[at(t) + j] = bits(b.calls[t].flt, value(rank, t, j, b.salt));
            if (ownInPlace(b, cr)) {
                r.host[at(t) + j] = a.host[at(t) + j];
            }
        }
    }
    a.upload();
    r.upload();
}

inline int issue(const Burst& b, DevBuffer& a, DevBuffer& r, int t, int rank, int cr, MPI_Request* req, std::string* why)
{
    const Call c = b.calls[t];
    const void* send = ownInPlace(b, cr) ? MPI_IN_PLACE : (const void*)(a.ptr + at(t));
    const MPI_Datatype dt = c.flt ? MPI_FLOAT : MPI_INT;
    GSC_CHECK((c.ex ? MPI_Iexscan(send, r.ptr + at(t), len(t), dt, c.op, b.comm, req)
                    : MPI_Iscan(send, r.ptr + at(t), len(t), dt, c.op, b.comm, req)) == MPI_SUCCESS);
    return 0;
}

// Word j of tensor t at comm rank cr: the fold over comm ranks 0..cr (scan)
// or 0..cr-1 (exscan; rank 0 keeps what it had)
inline int32_t want(const Burst& b, int t, int j, int rank, int cr)
{
    const Call c = b.calls[t];
    const int k = c.ex ? cr : cr + 1;
    if (k == 0) {
        return ownInPlace(b, cr) ? bits(c.flt, value(rank, t, j, b.salt)) : guard(rank);
    }
    int64_t acc = value(b.members[0], t, j, b.salt);
    for (int p = 1; p < k; p++) {
        const int64_t v = value(b.members[p], t, j, b.salt);
        acc = c.op == MPI_MAX ? std::max(acc, v) : acc + v;
    }
    return bits(c.flt, acc);
}

inline int check(const Burst& b, DevBuffer& r, int rank, int cr, std::string* why)
{
    const auto& got = r.read();
    for (size_t i = 0; i < got.size(); i++) {
        int32_t w = guard(rank);
        for (int t = 0; t < T; t++) {
            if (i >= at(t) && i < at(t) + (size_t)len(t)) {
                w = want(b, t, (int)(i - at(t)), rank, cr);
            }
        }
        if (got[i] != w) {
            *why = "rank " + std::to_string(rank) + " word " + std::to_string(i) + ": " + std::to_string(got[i]) +
                   ", want " + std::to_string(w);
            return 1;
        }
    }
    return 0;
}

// A burst of T calls of one kind: nothing launched before the wait
// (grouped), `flushes` launches at issue and one more after it; or one launch
// per call at issue (grouping off).  A one-member exscan launches nothing.
inline int burst(const Burst& b, DevBuffer& a, DevBuffer& r, int rank, bool grouped,
                 const std::shared_ptr<faabric::device::Communicator>& world, std::string* why, int flushes = 0)
{
    int cr = -1;
    MPI_Comm_rank(b.comm, &cr);
    fill(b, a, r, rank, cr);
    MPI_Barrier(b.comm);
    std::vector<MPI_Request> reqs(T);
    GSC_CHECK(issue(b, a, r, 0, rank, cr, &reqs[0], why) == 0);
    auto sub = faabric::mpi::getSubCommunicator(b.comm->id);
    auto dev = b.comm == MPI_COMM_WORLD ? world : (sub == nullptr ? nullptr : sub->currentDevice(rank));
    GSC_CHECK(dev != nullptr && dev->size() == (int)b.members.size());
    const uint64_t per = b.calls[0].ex && b.members.size() == 1 ? 0 : 1;
    const uint64_t l0 = dev->stats().launches;
    for (int t = 1; t < T; t++) {
        GSC_CHECK(issue(b, a, r, t, rank, cr, &reqs[t], why) == 0);
    }
    GSC_CHECK(dev->stats().launches == l0 + per * (grouped ? flushes : T - 1));
    GSC_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
    GSC_CHECK(dev->stats().launches == l0 + per * (grouped ? flushes + 1 : T - 1));
    return check(b, r, rank, cr, why);
}

inline void userSum(void* in, void* inout, int* n, MPI_Datatype*)
{
    for (int i = 0; i < *n; i++) {
        ((int32_t*)inout)[i] += ((const int32_t*)in)[i];
    }
}

inline int body(int rank, int size, int worldId, bool grouped, std::string* why)
{
    auto& world = faabric::mpi::getMpiWorldRegistry().getWorld(worldId);
    auto comm = world.getDeviceComm(rank);
    GSC_CHECK(comm != nullptr);
    const size_t words = at(T) + 8;
    DevBuffer a(words, BufferMemory::Heap), r(words, BufferMemory::Heap);
    GSC_CHECK(a.ptr && r.ptr);
    std::vector<int> all;
    for (int p = 0; p < size; p++) {
        all.push_back(p);
    }
    const unsigned odd = 0xAAAAAAAAu, even = 0x55555555u;

    // ---- both kinds, both ops and datatypes, in place on no rank, on the
    // odd ranks and on the even ones
    int salt = 0;
    for (int ex = 0; ex < 2; ex++) {
        for (unsigned inPlace : { 0u, odd, even }) {
            const Call c{ salt % 2 ? MPI_MAX : MPI_SUM, inPlace == odd, ex == 1 };
            GSC_CHECK(burst(uniform(MPI_COMM_WORLD, all, inPlace, salt, c), a, r, rank, grouped, comm, why) == 0);
            salt++;
        }
    }
    if (!grouped) {
        MPI_Barrier(MPI_COMM_WORLD);
        return 0;
    }

    // ---- a change of kind, op or datatype flushes: each splits the burst
    // in two launches
    for (int change = 0; change < 3; change++) {
        const Call isum{ MPI_SUM, false, false };
        Burst b = uniform(MPI_COMM_WORLD, all, odd, 10 + change, isum);
        for (int t = T / 2; t < T; t++) {
            b.calls[t] = { change == 1 ? MPI_MAX : MPI_SUM, change == 2, change == 0 };
        }
        GSC_CHECK(burst(b, a, r, rank, true, comm, why, 1) == 0);
    }

    // ---- blocking MPI_Exscan on device buffers (one grouped launch), in
    // place on the odd ranks, then on host buffers (the chain)
    {
        const Call c{ MPI_SUM, true, true };
        const Burst b = uniform(MPI_COMM_WORLD, all, odd, 20, c);
        fill(b, a, r, rank, rank);
        MPI_Barrier(MPI_COMM_WORLD);
        const uint64_t l0 = comm->stats().launches;
        for (int t = 0; t < T; t++) {
            const void* send = ownInPlace(b, rank) ? MPI_IN_PLACE : (const void*)(a.ptr + at(t));
            GSC_CHECK(MPI_Exscan(send, r.ptr + at(t), len(t), MPI_FLOAT, MPI_SUM, MPI_COMM_WORLD) == MPI_SUCCESS);
        }
        GSC_CHECK(comm->stats().launches == l0 + T);
        GSC_CHECK(check(b, r, rank, rank, why) == 0);

        std::vector<int32_t> hs(5), hr(5, -1);
        for (int j = 0; j < 5; j++) {
            hs[j] = rank * 100 + j;
        }
        GSC_CHECK(MPI_Exscan(hs.data(), hr.data(), 5, MPI_INT, MPI_SUM, MPI_COMM_WORLD) == MPI_SUCCESS);
        for (int j = 0; j < 5; j++) {
            GSC_CHECK(hr[j] == (rank == 0 ? -1 : 100 * rank * (rank - 1) / 2 + rank * j));
        }
        // in place on the host: every rank's send is read before its recv is
        // written
        GSC_CHECK(MPI_Exscan(MPI_IN_PLACE, hs.data(), 5, MPI_INT, MPI_MAX, MPI_COMM_WORLD) == MPI_SUCCESS);
        for (int j = 0; j < 5; j++) {
            GSC_CHECK(hs[j] == (rank == 0 ? j : (rank - 1) * 100 + j));
        }
        GSC_CHECK(comm->stats().launches == l0 + T);
    }

    // ---- host buffers, user-defined ops and zero counts complete at issue
    {
        std::vector<int32_t> hs(3), hr(3, -1);
        for (int j = 0; j < 3; j++) {
            hs[j] = rank * 100 + j;
        }
        MPI_Request q;
        GSC_CHECK(MPI_Iscan(hs.data(), hr.data(), 3, MPI_INT, MPI_SUM, MPI_COMM_WORLD, &q) == MPI_SUCCESS);
        for (int j = 0; j < 3; j++) {
            GSC_CHECK(hr[j] == 100 * rank * (rank + 1) / 2 + (rank + 1) * j);
        }
        GSC_CHECK(MPI_Wait(&q, MPI_STATUS_IGNORE) == MPI_SUCCESS);

        MPI_Op user;
        GSC_CHECK(MPI_Op_create(userSum, 1, &user) == MPI_SUCCESS);
        const Call c{ MPI_SUM, false, true };
        const Burst b = uniform(MPI_COMM_WORLD, all, 0, 30, c);
        fill(b, a, r, rank, rank);
        MPI_Barrier(MPI_COMM_WORLD);
        const uint64_t l0 = comm->stats().launches;
        std::vector<MPI_Request> reqs(T);
        for (int t = 0; t < T; t++) {
            GSC_CHECK(MPI_Iexscan(a.ptr + at(t), r.ptr + at(t), len(t), MPI_INT, user, MPI_COMM_WORLD, &reqs[t]) ==
                      MPI_SUCCESS);
        }
        GSC_CHECK(check(b, r, rank, rank, why) == 0);
        GSC_CHECK(MPI_Iscan(a.ptr + 1, r.ptr + 1, 0, MPI_INT, MPI_SUM, MPI_COMM_WORLD, &q) == MPI_SUCCESS);
        MPI_Request q2;
        GSC_CHECK(MPI_Iexscan(a.ptr + 1, r.ptr + 1, 0, MPI_INT, MPI_SUM, MPI_COMM_WORLD, &q2) == MPI_SUCCESS);
        GSC_CHECK(comm->stats().launches == l0);
        GSC_CHECK(MPI_Wait(&q, MPI_STATUS_IGNORE) == MPI_SUCCESS);
        GSC_CHECK(MPI_Wait(&q2, MPI_STATUS_IGNORE) == MPI_SUCCESS);
        GSC_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GSC_CHECK(check(b, r, rank, rank, why) == 0);
        GSC_CHECK(MPI_Op_free(&user) == MPI_SUCCESS);
    }

    // ---- refusals: MPI_ERR_OP, nothing issued
    {
        const Burst b = uniform(MPI_COMM_WORLD, all, 0, 0, { MPI_SUM, false, false });
        fill(b, a, r, rank, rank);
        const uint64_t l0 = comm->stats().launches;
        MPI_Request q;
        for (MPI_Op op : { MPI_REPLACE, MPI_NO_OP }) {
            GSC_CHECK(MPI_Iscan(a.ptr + 1, r.ptr + 1, 4, MPI_INT, op, MPI_COMM_WORLD, &q) == MPI_ERR_OP);
            GSC_CHECK(MPI_Iexscan(a.ptr + 1, r.ptr + 1, 4, MPI_INT, op, MPI_COMM_WORLD, &q) == MPI_ERR_OP);
            GSC_CHECK(MPI_Exscan(a.ptr + 1, r.ptr + 1, 4, MPI_INT, op, MPI_COMM_WORLD) == MPI_ERR_OP);
        }
        GSC_CHECK(MPI_Iscan(a.ptr + 1, r.ptr + 1, 4, MPI_FLOAT, MPI_BAND, MPI_COMM_WORLD, &q) == MPI_ERR_OP);
        GSC_CHECK(MPI_Iexscan(a.ptr + 1, r.ptr + 1, 4, MPI_FLOAT, MPI_BAND, MPI_COMM_WORLD, &q) == MPI_ERR_OP);
        GSC_CHECK(MPI_Exscan(a.ptr + 1, r.ptr + 1, 4, MPI_FLOAT, MPI_BXOR, MPI_COMM_WORLD) == MPI_ERR_OP);
        MPI_Barrier(MPI_COMM_WORLD);
        GSC_CHECK(comm->stats().launches == l0);
        const auto& got = r.read();
        for (int32_t v : got) {
            GSC_CHECK(v == guard(rank));
        }
    }

    // ---- parity split: bursts and MPI_Exscan on the child, world bursts
    // between
    MPI_Comm sub;
    GSC_CHECK(MPI_Comm_split(MPI_COMM_WORLD, rank % 2, rank, &sub) == MPI_SUCCESS);
    int srank = -1, ssize = -1;
    MPI_Comm_rank(sub, &srank);
    MPI_Comm_size(sub, &ssize);
    std::vector<int> members;
    for (int p = rank % 2; p < size; p += 2) {
        members.push_back(p);
    }
    GSC_CHECK(ssize == (int)members.size() && members[srank] == rank);
    // (the first device collective on the child agrees its slot)
    GSC_CHECK(MPI_Allreduce(MPI_IN_PLACE, r.ptr, 4, MPI_INT, MPI_SUM, sub) == MPI_SUCCESS);
    for (int ex = 0; ex < 2; ex++) {
        const Burst b = uniform(sub, members, ex ? odd : even, 50 + ex, { ex ? MPI_MAX : MPI_SUM, ex == 0, ex == 1 });
        GSC_CHECK(burst(b, a, r, rank, true, comm, why) == 0);
        const Burst w = uniform(MPI_COMM_WORLD, all, ex ? even : 0, 60 + ex, { MPI_SUM, true, ex == 0 });
        GSC_CHECK(burst(w, a, r, rank, true, comm, why) == 0);
    }
    {
        const Burst b = uniform(sub, members, odd, 65, { MPI_SUM, false, true });
        fill(b, a, r, rank, srank);
        MPI_Barrier(sub);
        for (int t = 0; t < T; t++) {
            const void* send = ownInPlace(b, srank) ? MPI_IN_PLACE : (const void*)(a.ptr + at(t));
            GSC_CHECK(MPI_Exscan(send, r.ptr + at(t), len(t), MPI_INT, MPI_SUM, sub) == MPI_SUCCESS);
        }
        GSC_CHECK(check(b, r, rank, srank, why) == 0);
    }

    // ---- MPI_Comm_free with a burst pending: it is issued and completed
    {
        const Burst b = uniform(sub, members, 0, 70, { MPI_SUM, false, true });
        fill(b, a, r, rank, srank);
        MPI_Barrier(sub);
        std::vector<MPI_Request> reqs(T);
        for (int t = 0; t < T; t++) {
            GSC_CHECK(issue(b, a, r, t, rank, srank, &reqs[t], why) == 0);
        }
        GSC_CHECK(MPI_Comm_free(&sub) == MPI_SUCCESS);
        GSC_CHECK(MPI_Waitall(T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        GSC_CHECK(check(b, r, rank, srank, why) == 0);
    }
    MPI_Barrier(MPI_COMM_WORLD);
    return 0;
}

#undef GSC_CHECK

}
