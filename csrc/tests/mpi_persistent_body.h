// One MPI program for persistent collectives (MPI_*_init, MPI_Start,
// MPI_Startall) of all ten grouped kinds, on the world, on MPI_Comm_split
// halves and on a split of a split.  Shared by the loopback test
// (test_loopback_persistent.cpp), the GPU test (test_device_persistent.cpp) and
// faabric_worker's `persistent-coll` program, which
// tests/test_dist_persistent.py runs with one rank in each of four worker
// processes.
//
// Every round rewrites the inputs, starts the requests and compares every word
// of every output, guard words included, with a closed form computed on the
// host.  On the world's symmetric lists a repeated MPI_Startall launches the
// same kernels as the first one and builds no segment table; a new order of
// the same requests, or a freed and re-initialised request, builds one.  The
// error paths change no output and launch nothing.  With grouping off
// (FAABRIC_MPI_GROUP_IALLREDUCE=0, body(..., false)) every start runs its
// device call at start.
#pragma once

#include "mpi/subcomm.h"
#include "mpi_subcomm_device_body.h"

#include <faabric/mpi/MpiWorld.h>
#include <faabric/mpi/MpiWorldRegistry.h>
#include <faabric/mpi/mpi.h>

#include <algorithm>
#include <cstdint>
#include <string>
#include <vector>

namespace persistent_coll {

using subcomm_device::BufferMemory;
using subcomm_device::DevBuffer;

#define PC_CHECK(cond)                                                         \
    do {                                                                       \
        if (!(cond)) {                                                         \
            *why = "rank " + std::to_string(rank) + ": check failed at line " + std::to_string(__LINE__) + ": " #cond; \
            return 1;                                                          \
        }                                                                      \
    } while (0)

// A nested step that reports its own failure
#define PC_TRY(call)                                                           \
    do {                                                                       \
        if ((call) != 0) {                                                     \
            return 1;                                                          \
        }                                                                      \
    } while (0)

enum Kind
{
    ALLREDUCE,
    REDUCE_SCATTER,
    ALLGATHER,
    BCAST,
    ALLTOALL,
    GATHER,
    SCATTER,
    REDUCE,
    SCAN,
    EXSCAN,
    KINDS
};

constexpr int T = 4; // requests per kind
constexpr int N = 8; // int32 per block: 32 bytes

// Word j of tensor t of `kind` in world rank r's send, in round `salt`
inline int32_t in(int r, int kind, int t, int j, int salt)
{
    return r * 1000 + kind * 100 + t * 17 + j + salt * 7;
}

inline int32_t guard(int rank)
{
    return -1 - rank;
}

// The communicator a test runs on: its members (world ranks, in comm order)
struct Comm
{
    MPI_Comm comm;
    std::vector<int> members;
    int cr;
    int m() const { return (int)members.size(); }
    int root() const { return m() - 1; }
};

inline Comm commOf(MPI_Comm comm, int rank)
{
    Comm c{ comm, subcomm_device::membersOf(comm), -1 };
    MPI_Comm_rank(comm, &c.cr);
    return c;
}

// Offset of tensor t of `kind`: m * N words in both buffers
inline size_t off(const Comm& c, int kind, int t)
{
    return ((size_t)kind * T + t) * c.m() * N;
}

inline int initOne(const Comm& c, int kind, int t, DevBuffer& a, DevBuffer& b, MPI_Request* r)
{
    int32_t* s = a.ptr + off(c, kind, t);
    int32_t* d = b.ptr + off(c, kind, t);
    switch (kind) {
        case ALLREDUCE:
            return MPI_Allreduce_init(s, d, N, MPI_INT, MPI_SUM, c.comm, MPI_INFO_NULL, r);
        case REDUCE_SCATTER:
            return MPI_Reduce_scatter_block_init(s, d, N, MPI_INT, MPI_SUM, c.comm, MPI_INFO_NULL, r);
        case ALLGATHER:
            return MPI_Allgather_init(s, N, MPI_INT, d, N, MPI_INT, c.comm, MPI_INFO_NULL, r);
        case BCAST:
            return MPI_Bcast_init(d, N, MPI_INT, c.root(), c.comm, MPI_INFO_NULL, r);
        case ALLTOALL:
            return MPI_Alltoall_init(s, N, MPI_INT, d, N, MPI_INT, c.comm, MPI_INFO_NULL, r);
        case GATHER:
            return MPI_Gather_init(s, N, MPI_INT, d, N, MPI_INT, c.root(), c.comm, MPI_INFO_NULL, r);
        case SCATTER:
            return MPI_Scatter_init(s, N, MPI_INT, d, N, MPI_INT, c.root(), c.comm, MPI_INFO_NULL, r);
        case REDUCE:
            return MPI_Reduce_init(s, d, N, MPI_INT, MPI_SUM, c.root(), c.comm, MPI_INFO_NULL, r);
        case SCAN:
            return MPI_Scan_init(s, d, N, MPI_INT, MPI_SUM, c.comm, MPI_INFO_NULL, r);
        default:
            return MPI_Exscan_init(s, d, N, MPI_INT, MPI_SUM, c.comm, MPI_INFO_NULL, r);
    }
}

// Sends of round `salt` in a, guard words in b (the broadcast root's buffer
// holds its data)
inline void fill(const Comm& c, DevBuffer& a, DevBuffer& b, int rank, int salt)
{
    std::fill(a.host.begin(), a.host.end(), -7);
    std::fill(b.host.begin(), b.host.end(), guard(rank));
    for (int k = 0; k < KINDS; k++) {
        for (int t = 0; t < T; t++) {
            for (int i = 0; i < c.m() * N; i++) {
                a.host[off(c, k, t) + i] = in(rank, k, t, i, salt);
            }
            if (k == BCAST && c.cr == c.root()) {
                for (int i = 0; i < N; i++) {
                    b.host[off(c, k, t) + i] = in(rank, k, t, i, salt);
                }
            }
        }
    }
    a.upload();
    b.upload();
}

// Word i of tensor t of `kind` in this rank's recv
inline int32_t want(const Comm& c, int rank, int k, int t, int i, int salt)
{
    const int m = c.m();
    const int cr = c.cr;
    auto sum = [&](int q0, int q1, int j) {
        int32_t s = 0;
        for (int q = q0; q < q1; q++) {
            s += in(c.members[q], k, t, j, salt);
        }
        return s;
    };
    const bool first = i < N;
    switch (k) {
        case ALLREDUCE:
            return first ? sum(0, m, i) : guard(rank);
        case REDUCE_SCATTER:
            return first ? sum(0, m, cr * N + i) : guard(rank);
        case ALLGATHER:
            return in(c.members[i / N], k, t, i % N, salt);
        case BCAST:
            return first ? in(c.members[c.root()], k, t, i, salt) : guard(rank);
        case ALLTOALL:
            return in(c.members[i / N], k, t, cr * N + i % N, salt);
        case GATHER:
            return cr == c.root() ? in(c.members[i / N], k, t, i % N, salt) : guard(rank);
        case SCATTER:
            return first ? in(c.members[c.root()], k, t, cr * N + i, salt) : guard(rank);
        case REDUCE:
            return cr == c.root() && first ? sum(0, m, i) : guard(rank);
        case SCAN:
            return first ? sum(0, cr + 1, i) : guard(rank);
        default:
            return cr > 0 && first ? sum(0, cr, i) : guard(rank);
    }
}

// Kinds [k0, k1) hold the results of round `salt`; the others guard words
inline bool check(const Comm& c, DevBuffer& b, int rank, int salt, int k0, int k1, std::string* why)
{
    const auto& got = b.read();
    for (int k = 0; k < KINDS; k++) {
        for (int t = 0; t < T; t++) {
            for (int i = 0; i < c.m() * N; i++) {
                const bool bcastRoot = k == BCAST && c.cr == c.root() && i < N;
                const int32_t w = k >= k0 && k < k1    ? want(c, rank, k, t, i, salt)
                                  : bcastRoot          ? in(rank, k, t, i, (salt))
                                                       : guard(rank);
                const int32_t v = got[off(c, k, t) + i];
                if (v != w) {
                    *why = "rank " + std::to_string(rank) + " kind " + std::to_string(k) + " tensor " + std::to_string(t) +
                           " word " + std::to_string(i) + ": " + std::to_string(v) + ", want " + std::to_string(w);
                    return false;
                }
            }
        }
    }
    return true;
}

// All ten kinds on `c`: several MPI_Startall rounds (each a burst per kind),
// then an MPI_Start loop.  `counted`: launches and tables on `world` are
// checked (the world's symmetric lists)
inline int rounds(const Comm& c,
                  int rank,
                  DevBuffer& a,
                  DevBuffer& b,
                  int salt0,
                  const std::shared_ptr<faabric::device::Communicator>& world,
                  bool grouped,
                  bool counted,
                  std::vector<MPI_Request>& reqs,
                  std::string* why)
{
    reqs.assign(KINDS * T, MPI_REQUEST_NULL);
    for (int k = 0; k < KINDS; k++) {
        for (int t = 0; t < T; t++) {
            PC_CHECK(initOne(c, k, t, a, b, &reqs[k * T + t]) == MPI_SUCCESS);
        }
    }
    // (a one-member child launches nothing for some kinds: only the world's
    // lists are counted)
    auto dev = counted ? world : nullptr;
    auto launches = [&] { return dev != nullptr ? dev->stats().launches : 0; };
    auto tables = [&] { return dev != nullptr ? dev->stats().segTables : 0; };
    for (int round = 0; round < 4; round++) {
        const int salt = salt0 + round;
        fill(c, a, b, rank, salt);
        MPI_Barrier(MPI_COMM_WORLD);
        const uint64_t l0 = launches();
        const uint64_t s0 = tables();
        if (round < 3) {
            PC_CHECK(MPI_Startall(KINDS * T, reqs.data()) == MPI_SUCCESS);
        } else {
            for (auto& r : reqs) {
                const uint64_t before = launches();
                PC_CHECK(MPI_Start(&r) == MPI_SUCCESS);
                // grouping off: the device call runs at start
                PC_CHECK(grouped || !counted || launches() > before);
            }
        }
        const uint64_t atStart = launches() - l0;
        PC_CHECK(MPI_Waitall(KINDS * T, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        for (auto& r : reqs) {
            PC_CHECK(r != MPI_REQUEST_NULL); // inactive, not freed
        }
        PC_CHECK(check(c, b, rank, salt, 0, KINDS, why));
        if (!counted) {
            continue;
        }
        if (grouped) {
            // one burst per kind, each one plan launch: a change of key issues
            // the previous kind's burst at start, the wait the last one.
            // Segment tables are built on the first round only.
            PC_CHECK(atStart == KINDS - 1);
            PC_CHECK(launches() - l0 == KINDS);
            PC_CHECK(tables() - s0 == (round == 0 ? (uint64_t)KINDS : 0));
        } else {
            // every call ran at start; the wait launches nothing
            PC_CHECK(atStart >= (uint64_t)KINDS * T);
            PC_CHECK(launches() - l0 == atStart);
        }
    }
    return 0;
}

inline int freeAll(int rank, std::vector<MPI_Request>& reqs, std::string* why)
{
    for (auto& r : reqs) {
        PC_CHECK(MPI_Request_free(&r) == MPI_SUCCESS);
        PC_CHECK(r == MPI_REQUEST_NULL);
    }
    return 0;
}

// The 214 ResNet-50 gradient tensors (generated from the architecture),
// scaled down by `scale`, in int32 elements rounded up to a multiple of `q`
inline std::vector<size_t> resnet50(size_t scale, size_t q)
{
    std::vector<size_t> fwd;
    auto vecs = [&](size_t ch) {
        fwd.insert(fwd.end(), { ch, ch, ch });
    };
    fwd.push_back(7 * 7 * 3 * 64);
    vecs(64);
    size_t cin = 64;
    const size_t widths[4] = { 64, 128, 256, 512 };
    const int blocks[4] = { 3, 4, 6, 3 };
    for (int l = 0; l < 4; l++) {
        const size_t w = widths[l];
        const size_t cout = w * 4;
        for (int b = 0; b < blocks[l]; b++) {
            fwd.push_back(cin * w);
            vecs(w);
            fwd.push_back(9 * w * w);
            vecs(w);
            fwd.push_back(w * cout);
            if (b == 0) {
                fwd.push_back(cin * cout);
                vecs(cout);
            }
            vecs(cout);
            cin = cout;
        }
    }
    fwd.push_back(2048 * 1000);
    fwd.push_back(1000);
    std::reverse(fwd.begin(), fwd.end());
    for (auto& s : fwd) {
        s = (s / scale + q - 1) / q * q;
    }
    return fwd;
}

// The ResNet-50 list as persistent all-reduces and as all-to-alls on the
// world, two rounds each
inline int resnetLists(int rank, int size, const std::shared_ptr<faabric::device::Communicator>& comm, bool grouped,
                       std::string* why)
{
    for (int kind : { ALLREDUCE, ALLTOALL }) {
        const size_t q = kind == ALLTOALL ? 4 * (size_t)size : 4;
        const std::vector<size_t> sizes = resnet50(256, q);
        PC_CHECK(sizes.size() == 214);
        std::vector<size_t> offs;
        size_t total = 0;
        for (size_t s : sizes) {
            offs.push_back(total);
            total += s;
        }
        DevBuffer a(total, BufferMemory::Heap);
        DevBuffer b(total, BufferMemory::Heap);
        PC_CHECK(a.ptr != nullptr && b.ptr != nullptr);
        std::vector<MPI_Request> reqs(sizes.size(), MPI_REQUEST_NULL);
        for (size_t i = 0; i < sizes.size(); i++) {
            if (kind == ALLREDUCE) {
                PC_CHECK(MPI_Allreduce_init(a.ptr + offs[i], b.ptr + offs[i], (int)sizes[i], MPI_INT, MPI_SUM,
                                            MPI_COMM_WORLD, MPI_INFO_NULL, &reqs[i]) == MPI_SUCCESS);
            } else {
                const int blk = (int)(sizes[i] / size);
                PC_CHECK(MPI_Alltoall_init(a.ptr + offs[i], blk, MPI_INT, b.ptr + offs[i], blk, MPI_INT, MPI_COMM_WORLD,
                                           MPI_INFO_NULL, &reqs[i]) == MPI_SUCCESS);
            }
        }
        uint64_t first = 0;
        for (int round = 0; round < 2; round++) {
            for (size_t i = 0; i < total; i++) {
                a.host[i] = (int32_t)(rank * 7919 + i * 3 + round * 101);
            }
            a.upload();
            MPI_Barrier(MPI_COMM_WORLD);
            const uint64_t l0 = comm->stats().launches;
            const uint64_t s0 = comm->stats().segTables;
            PC_CHECK(MPI_Startall((int)reqs.size(), reqs.data()) == MPI_SUCCESS);
            PC_CHECK(MPI_Waitall((int)reqs.size(), reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
            const uint64_t launches = comm->stats().launches - l0;
            if (grouped) {
                // the plan's launches each round; tables on the first only
                PC_CHECK(comm->stats().segTables - s0 == (round == 0 ? launches : 0));
            }
            if (round == 0) {
                first = launches;
            }
            PC_CHECK(launches == first);
            const auto& got = b.read();
            for (size_t t = 0; t < sizes.size(); t++) {
                for (size_t j = 0; j < sizes[t]; j++) {
                    const size_t at = offs[t] + j;
                    int64_t w = 0;
                    if (kind == ALLREDUCE) {
                        for (int p = 0; p < size; p++) {
                            w += (int32_t)(p * 7919 + at * 3 + round * 101);
                        }
                    } else {
                        const size_t blk = sizes[t] / size;
                        const int p = (int)(j / blk);
                        w = (int32_t)(p * 7919 + (offs[t] + rank * blk + j % blk) * 3 + round * 101);
                    }
                    if (got[at] != (int32_t)w) {
                        *why = "rank " + std::to_string(rank) + " resnet kind " + std::to_string(kind) + " tensor " +
                               std::to_string(t) + " word " + std::to_string(j) + ": " + std::to_string(got[at]) +
                               ", want " + std::to_string((int32_t)w);
                        return 1;
                    }
                }
            }
        }
        PC_TRY(freeAll(rank, reqs, why));
    }
    return 0;
}

inline int body(int rank, int size, int worldId, bool grouped, bool gpu, std::string* why)
{
    auto& world = faabric::mpi::getMpiWorldRegistry().getWorld(worldId);
    auto comm = world.getDeviceComm(rank);
    PC_CHECK(comm != nullptr);
    const size_t words = (size_t)KINDS * T * N * size;
    DevBuffer a(words, BufferMemory::Heap);
    DevBuffer b(words, BufferMemory::Heap);
    PC_CHECK(a.ptr && b.ptr);
    const Comm w = commOf(MPI_COMM_WORLD, rank);
    std::vector<MPI_Request> reqs;

    // ---- all ten kinds on the world
    PC_TRY(rounds(w, rank, a, b, 0, comm, grouped, true, reqs, why));

    if (!grouped) {
        PC_TRY(freeAll(rank, reqs, why));
        MPI_Barrier(MPI_COMM_WORLD);
        return 0;
    }
    std::vector<MPI_Request> ar(reqs.begin(), reqs.begin() + T); // the all-reduces

    // ---- the same requests in another order: one new plan
    {
        std::vector<MPI_Request> rev(ar.rbegin(), ar.rend());
        fill(w, a, b, rank, 10);
        MPI_Barrier(MPI_COMM_WORLD);
        const uint64_t l0 = comm->stats().launches;
        const uint64_t s0 = comm->stats().segTables;
        PC_CHECK(MPI_Startall(T, rev.data()) == MPI_SUCCESS);
        PC_CHECK(MPI_Waitall(T, rev.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        PC_CHECK(comm->stats().launches == l0 + 1);
        PC_CHECK(comm->stats().segTables == s0 + 1);
        PC_CHECK(check(w, b, rank, 10, ALLREDUCE, ALLREDUCE + 1, why));
        // and the first order still has its plan
        fill(w, a, b, rank, 11);
        MPI_Barrier(MPI_COMM_WORLD);
        PC_CHECK(MPI_Startall(T, ar.data()) == MPI_SUCCESS);
        PC_CHECK(MPI_Waitall(T, ar.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        PC_CHECK(comm->stats().segTables == s0 + 1);
        PC_CHECK(check(w, b, rank, 11, ALLREDUCE, ALLREDUCE + 1, why));
    }

    // ---- a freed and re-initialised request builds again
    {
        PC_CHECK(MPI_Request_free(&ar[1]) == MPI_SUCCESS && ar[1] == MPI_REQUEST_NULL);
        PC_CHECK(initOne(w, ALLREDUCE, 1, a, b, &ar[1]) == MPI_SUCCESS);
        reqs[1] = ar[1];
        fill(w, a, b, rank, 12);
        MPI_Barrier(MPI_COMM_WORLD);
        const uint64_t s0 = comm->stats().segTables;
        PC_CHECK(MPI_Startall(T, ar.data()) == MPI_SUCCESS);
        PC_CHECK(MPI_Waitall(T, ar.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        PC_CHECK(comm->stats().segTables == s0 + 1);
        PC_CHECK(check(w, b, rank, 12, ALLREDUCE, ALLREDUCE + 1, why));
    }

    // ---- starts interleaved with an I-call burst of the same key (today's
    // transient path) and with a blocking collective (flushes first)
    {
        DevBuffer g(16, BufferMemory::Heap);
        PC_CHECK(g.ptr != nullptr);
        for (int j = 0; j < 16; j++) {
            g.host[j] = rank + j;
        }
        g.upload();
        fill(w, a, b, rank, 13);
        MPI_Barrier(MPI_COMM_WORLD);
        const uint64_t l0 = comm->stats().launches;
        PC_CHECK(MPI_Startall(T, ar.data()) == MPI_SUCCESS);
        MPI_Request ir;
        PC_CHECK(MPI_Iallreduce(MPI_IN_PLACE, g.ptr, 8, MPI_INT, MPI_SUM, MPI_COMM_WORLD, &ir) == MPI_SUCCESS);
        PC_CHECK(comm->stats().launches == l0); // one burst, still deferred
        PC_CHECK(MPI_Wait(&ir, MPI_STATUS_IGNORE) == MPI_SUCCESS && ir == MPI_REQUEST_NULL);
        PC_CHECK(comm->stats().launches == l0 + 1);
        PC_CHECK(MPI_Waitall(T, ar.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        PC_CHECK(check(w, b, rank, 13, ALLREDUCE, ALLREDUCE + 1, why));

        fill(w, a, b, rank, 14);
        MPI_Barrier(MPI_COMM_WORLD);
        const uint64_t l1 = comm->stats().launches;
        PC_CHECK(MPI_Startall(T, ar.data()) == MPI_SUCCESS);
        PC_CHECK(MPI_Allreduce(MPI_IN_PLACE, g.ptr + 8, 8, MPI_INT, MPI_SUM, MPI_COMM_WORLD) == MPI_SUCCESS);
        PC_CHECK(comm->stats().launches >= l1 + 2);
        const uint64_t l2 = comm->stats().launches;
        PC_CHECK(MPI_Waitall(T, ar.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        PC_CHECK(comm->stats().launches == l2);
        PC_CHECK(check(w, b, rank, 14, ALLREDUCE, ALLREDUCE + 1, why));
        const auto& got = g.read();
        for (int j = 0; j < 16; j++) {
            PC_CHECK(got[j] == size * (size - 1) / 2 + size * j);
        }
    }

    // ---- error paths: nothing issued, outputs untouched
    {
        fill(w, a, b, rank, 15);
        MPI_Barrier(MPI_COMM_WORLD);
        const uint64_t l0 = comm->stats().launches;
        PC_CHECK(MPI_Startall(T, ar.data()) == MPI_SUCCESS);
        PC_CHECK(MPI_Start(&ar[0]) == MPI_ERR_REQUEST);
        PC_CHECK(MPI_Startall(T, reqs.data()) == MPI_ERR_REQUEST); // (none of them started)
        PC_CHECK(MPI_Request_free(&ar[2]) == MPI_ERR_REQUEST && ar[2] != MPI_REQUEST_NULL);
        PC_CHECK(comm->stats().launches == l0);
        PC_CHECK(MPI_Waitall(T, ar.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        PC_CHECK(comm->stats().launches == l0 + 1);
        PC_CHECK(check(w, b, rank, 15, ALLREDUCE, ALLREDUCE + 1, why));
        // a wait on an inactive request returns at once; MPI_Waitany skips it
        PC_CHECK(MPI_Wait(&ar[0], MPI_STATUS_IGNORE) == MPI_SUCCESS && ar[0] != MPI_REQUEST_NULL);
        int idx = 0;
        PC_CHECK(MPI_Waitany(T, ar.data(), &idx, MPI_STATUS_IGNORE) == MPI_SUCCESS && idx == MPI_UNDEFINED);
        PC_CHECK(comm->stats().launches == l0 + 1);
        MPI_Request nonPersistent = MPI_REQUEST_NULL;
        PC_CHECK(MPI_Start(&nonPersistent) == MPI_ERR_REQUEST);

        // bad init arguments create nothing
        MPI_Request r = MPI_REQUEST_NULL;
        PC_CHECK(MPI_Allreduce_init(a.ptr, b.ptr, N, MPI_INT, MPI_REPLACE, MPI_COMM_WORLD, MPI_INFO_NULL, &r) ==
                 MPI_ERR_OP);
        PC_CHECK(MPI_Reduce_init(a.ptr, b.ptr, N, MPI_INT, MPI_SUM, size, MPI_COMM_WORLD, MPI_INFO_NULL, &r) ==
                 MPI_ERR_ARG);
        PC_CHECK(MPI_Bcast_init(b.ptr, N, MPI_INT, -1, MPI_COMM_WORLD, MPI_INFO_NULL, &r) == MPI_ERR_ARG);
        PC_CHECK(MPI_Gather_init(a.ptr, N, MPI_INT, b.ptr, N, MPI_INT, size, MPI_COMM_WORLD, MPI_INFO_NULL, &r) ==
                 MPI_ERR_ARG);
        PC_CHECK(MPI_Alltoall_init(MPI_IN_PLACE, N, MPI_INT, b.ptr, N, MPI_INT, MPI_COMM_WORLD, MPI_INFO_NULL, &r) ==
                 MPI_ERR_ARG);
        PC_CHECK(MPI_Alltoall_init(a.ptr, N, MPI_INT, b.ptr, N - 1, MPI_INT, MPI_COMM_WORLD, MPI_INFO_NULL, &r) ==
                 MPI_ERR_ARG);
        PC_CHECK(r == MPI_REQUEST_NULL);
        PC_CHECK(comm->stats().launches == l0 + 1);
        PC_CHECK(check(w, b, rank, 15, ALLREDUCE, ALLREDUCE + 1, why));
    }
    PC_TRY(freeAll(rank, reqs, why));

    // ---- host buffers, and device buffers that are not aligned (or not in
    // the heap): one call at start
    {
        std::vector<int32_t> hs(N), hr(N, -1);
        MPI_Request r;
        PC_CHECK(MPI_Allreduce_init(hs.data(), hr.data(), N, MPI_INT, MPI_SUM, MPI_COMM_WORLD, MPI_INFO_NULL, &r) ==
                 MPI_SUCCESS);
        DevBuffer u(N + 1, BufferMemory::Heap);
        DevBuffer v(N + 1, BufferMemory::Heap);
        PC_CHECK(u.ptr != nullptr && v.ptr != nullptr);
        MPI_Request ru;
        PC_CHECK(MPI_Allreduce_init(u.ptr + 1, v.ptr + 1, N, MPI_INT, MPI_SUM, MPI_COMM_WORLD, MPI_INFO_NULL, &ru) ==
                 MPI_SUCCESS);
        std::unique_ptr<DevBuffer> x, y;
        MPI_Request rx = MPI_REQUEST_NULL;
        if (gpu) {
            x = std::make_unique<DevBuffer>(N, BufferMemory::CudaMalloc);
            y = std::make_unique<DevBuffer>(N, BufferMemory::CudaMalloc);
            PC_CHECK(x->ptr != nullptr && y->ptr != nullptr);
            PC_CHECK(MPI_Allreduce_init(x->ptr, y->ptr, N, MPI_INT, MPI_SUM, MPI_COMM_WORLD, MPI_INFO_NULL, &rx) ==
                     MPI_SUCCESS);
        }
        for (int round = 0; round < 2; round++) {
            for (int j = 0; j < N; j++) {
                hs[j] = rank * 10 + j + round;
                u.host[j + 1] = rank * 20 + j + round;
                if (gpu) {
                    x->host[j] = rank * 30 + j + round;
                }
            }
            u.upload();
            if (gpu) {
                x->upload();
            }
            MPI_Barrier(MPI_COMM_WORLD);
            PC_CHECK(MPI_Start(&r) == MPI_SUCCESS);
            for (int j = 0; j < N; j++) {
                PC_CHECK(hr[j] == size * (size - 1) * 5 + size * (j + round)); // complete at start
            }
            const uint64_t l0 = comm->stats().launches;
            PC_CHECK(MPI_Start(&ru) == MPI_SUCCESS);
            PC_CHECK(comm->stats().launches >= l0 + 1); // at start
            PC_CHECK(MPI_Wait(&r, MPI_STATUS_IGNORE) == MPI_SUCCESS);
            PC_CHECK(MPI_Wait(&ru, MPI_STATUS_IGNORE) == MPI_SUCCESS);
            const auto& got = v.read();
            for (int j = 0; j < N; j++) {
                PC_CHECK(got[j + 1] == size * (size - 1) * 10 + size * (j + round));
            }
            if (gpu) {
                PC_CHECK(MPI_Start(&rx) == MPI_SUCCESS);
                PC_CHECK(MPI_Wait(&rx, MPI_STATUS_IGNORE) == MPI_SUCCESS);
                const auto& gy = y->read();
                for (int j = 0; j < N; j++) {
                    PC_CHECK(gy[j] == size * (size - 1) * 15 + size * (j + round));
                }
            }
        }
        PC_CHECK(MPI_Request_free(&r) == MPI_SUCCESS && MPI_Request_free(&ru) == MPI_SUCCESS);
        if (gpu) {
            PC_CHECK(MPI_Request_free(&rx) == MPI_SUCCESS);
        }
    }

    // ---- the ResNet-50 list
    PC_TRY(resnetLists(rank, size, comm, grouped, why));

    // ---- parity split, and a split of the split
    MPI_Comm sub;
    PC_CHECK(MPI_Comm_split(MPI_COMM_WORLD, rank % 2, rank, &sub) == MPI_SUCCESS);
    const Comm s = commOf(sub, rank);
    // (the first device collective on the child agrees its slot)
    PC_CHECK(MPI_Allreduce(MPI_IN_PLACE, b.ptr, 4, MPI_INT, MPI_SUM, sub) == MPI_SUCCESS);
    std::vector<MPI_Request> sreqs;
    PC_TRY(rounds(s, rank, a, b, 20, comm, grouped, false, sreqs, why));
    {
        MPI_Comm nested;
        PC_CHECK(MPI_Comm_split(sub, s.cr % 2, s.cr, &nested) == MPI_SUCCESS);
        const Comm n = commOf(nested, rank);
        PC_CHECK(MPI_Allreduce(MPI_IN_PLACE, b.ptr, 4, MPI_INT, MPI_SUM, nested) == MPI_SUCCESS);
        std::vector<MPI_Request> nreqs;
        PC_TRY(rounds(n, rank, a, b, 30, comm, grouped, false, nreqs, why));
        PC_TRY(freeAll(rank, nreqs, why));
        PC_CHECK(MPI_Comm_free(&nested) == MPI_SUCCESS);
    }
    // ---- after MPI_Comm_free its requests cannot start; they can be freed
    {
        fill(s, a, b, rank, 40);
        const uint64_t l0 = comm->stats().launches;
        PC_CHECK(MPI_Comm_free(&sub) == MPI_SUCCESS);
        PC_CHECK(MPI_Start(&sreqs[0]) == MPI_ERR_COMM);
        PC_CHECK(MPI_Startall((int)sreqs.size(), sreqs.data()) == MPI_ERR_COMM);
        PC_CHECK(comm->stats().launches == l0);
        PC_CHECK(check(s, b, rank, 40, 0, 0, why));
        PC_TRY(freeAll(rank, sreqs, why));
    }
    MPI_Barrier(MPI_COMM_WORLD);
    return 0;
}

#undef PC_CHECK
#undef PC_TRY

}
