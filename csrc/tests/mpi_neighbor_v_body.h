// One MPI program for the neighbourhood v-collectives: blocking and
// non-blocking MPI_Neighbor_allgatherv / MPI_Neighbor_alltoallv on the world
// graph of mpi_neighbor_body.h (self-edges, multi-edges, and from 4 ranks a
// rank with no edge that still passes device pointers) and on a ring of a
// parity split, on host, heap, unaligned-heap and (on a GPU) cudaMalloc
// buffers, checked word for word (guard words included) against a closed
// form.  Counts differ per edge and round, zero included, and blocks sit in
// reverse order with gaps.  Launch counts: one per blocking device call and
// one per burst; bursts that mix v and equal-block calls flush at each change
// of kind; with grouping off one launch per call at issue.  A v call with
// equal counts moves what the equal-block call moves, bit for bit.  The
// refusals (MPI_ERR_ARG, MPI_ERR_TOPOLOGY) leave the outputs untouched;
// MPI_Comm_free with a v burst pending completes it.  Shared by
// test_loopback_neighbor_v.cpp and test_device_neighbor_v.cpp (through
// mpi_neighbor_v_run.h) and faabric_worker's `neighbor-v-coll`, which
// tests/test_dist_neighbor_v.py runs with one rank in each of four worker
// processes.
#pragma once

#include "mpi_neighbor_body.h"

namespace neighbor_v_coll {

using neighbor_coll::Bufs;
using neighbor_coll::childOf;
using neighbor_coll::Graph;
using neighbor_coll::launchesOf;
using neighbor_coll::makeGraph;
using neighbor_coll::SLOT;

// Words of out-edge i of comm rank s in `round` (all-gather: i = 0); 0 to 31.
// Rank 0's first block is never empty, so every call moves bytes (a call
// whose counts are 0 on every member launches nothing).
inline int count(int s, int i, int round, bool a2a)
{
    return (a2a ? (s + 2 * i + round) % 5 * 7 : (s + round) % 4 * 9) + (s == 0 && i == 0 ? 3 : 0);
}

inline int32_t word(int s, int round, int i, int w)
{
    return s * 1000000 + round * 10000 + i * 1000 + w + 1;
}

// One call's counts and displacements on comm rank cr: blocks in reverse
// order, one guard word before each
struct Layout
{
    std::vector<int> sc, sd, rc, rd;

    Layout(const Graph& g, int cr, int round, bool a2a)
    {
        const int sends = a2a ? (int)g.dst[cr].size() : 1;
        for (int i = 0; i < sends; i++) {
            sc.push_back(count(cr, i, round, a2a));
        }
        for (auto [s, idx] : g.in[cr]) {
            rc.push_back(count(s, a2a ? idx : 0, round, a2a));
        }
        sd = place(sc);
        rd = place(rc);
        if (!a2a) {
            sd.assign(1, 0);
        }
    }
    static std::vector<int> place(const std::vector<int>& c)
    {
        std::vector<int> d(c.size());
        int p = 0;
        for (int k = (int)c.size() - 1; k >= 0; k--) {
            p += 1;
            d[k] = p;
            p += c[k];
        }
        return d;
    }
};

inline void fill(Bufs& b, const Graph& g, int cr, int round, bool a2a, const Layout& l)
{
    auto& h = b.host();
    std::fill(h.begin(), h.end(), -7);
    for (size_t i = 0; i < l.sc.size(); i++) {
        for (int w = 0; w < l.sc[i]; w++) {
            h[b.off + l.sd[i] + w] = word(cr, round, (int)i, w);
        }
    }
    b.put();
}

inline std::vector<int32_t> expected(Bufs& b, const Graph& g, int cr, int round, bool a2a, const Layout& l)
{
    std::vector<int32_t> want = b.host();
    for (size_t j = 0; j < g.in[cr].size(); j++) {
        const auto [s, idx] = g.in[cr][j];
        for (int w = 0; w < l.rc[j]; w++) {
            want[SLOT + b.off + l.rd[j] + w] = word(s, round, a2a ? idx : 0, w);
        }
    }
    return want;
}

inline int call(bool a2a, Bufs& b, const Layout& l, MPI_Comm comm, MPI_Request* r)
{
    if (a2a) {
        return r ? MPI_Ineighbor_alltoallv(b.send(), l.sc.data(), l.sd.data(), MPI_INT, b.recv(), l.rc.data(),
                                           l.rd.data(), MPI_INT, comm, r)
                 : MPI_Neighbor_alltoallv(b.send(), l.sc.data(), l.sd.data(), MPI_INT, b.recv(), l.rc.data(),
                                          l.rd.data(), MPI_INT, comm);
    }
    return r ? MPI_Ineighbor_allgatherv(b.send(), l.sc[0], MPI_INT, b.recv(), l.rc.data(), l.rd.data(), MPI_INT,
                                        comm, r)
             : MPI_Neighbor_allgatherv(b.send(), l.sc[0], MPI_INT, b.recv(), l.rc.data(), l.rd.data(), MPI_INT,
                                       comm);
}

#define NV_CHECK NB_CHECK

inline int blockingV(MPI_Comm comm, const Graph& g, int memory, int off, bool device, int rank, std::string* why)
{
    int cr = -1;
    MPI_Comm_rank(comm, &cr);
    Bufs b(memory, off);
    NV_CHECK(b.ok());
    // (a peer may still be in the cudaFree of an earlier buffer, which waits
    // for the whole device: issue nothing it would have to wait for)
    MPI_Barrier(comm);
    for (int round = 0; round < 3; round++) {
        for (int a2a = 0; a2a < 2; a2a++) {
            const Layout l(g, cr, round, a2a);
            fill(b, g, cr, round, a2a, l);
            const auto want = expected(b, g, cr, round, a2a, l);
            const uint64_t l0 = launchesOf(comm, rank);
            NV_CHECK(call(a2a, b, l, comm, nullptr) == MPI_SUCCESS);
            NV_CHECK(launchesOf(comm, rank) == l0 + (device ? 1u : 0u));
            NV_CHECK(b.get() == want);
        }
    }
    return 0;
}

inline int burstV(MPI_Comm comm, const Graph& g, bool grouped, int rank, std::string* why)
{
    constexpr int K = neighbor_coll::K;
    int cr = -1;
    MPI_Comm_rank(comm, &cr);
    std::vector<std::unique_ptr<Bufs>> bs;
    std::vector<Layout> ls;
    for (int k = 0; k < K; k++) {
        bs.push_back(std::make_unique<Bufs>(1, 1 + k % 3));
        NV_CHECK(bs.back()->ok());
        ls.emplace_back(g, cr, 10 + k, true);
        fill(*bs.back(), g, cr, 10 + k, true, ls.back());
    }
    MPI_Barrier(comm);
    const uint64_t l0 = launchesOf(comm, rank);
    std::vector<MPI_Request> reqs(K);
    for (int k = 0; k < K; k++) {
        NV_CHECK(call(true, *bs[k], ls[k], comm, &reqs[k]) == MPI_SUCCESS);
    }
    NV_CHECK(launchesOf(comm, rank) == l0 + (grouped ? 0u : (uint64_t)K));
    NV_CHECK(MPI_Waitall(K, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
    NV_CHECK(launchesOf(comm, rank) == l0 + (grouped ? 1u : (uint64_t)K));
    for (int k = 0; k < K; k++) {
        NV_CHECK(bs[k]->get() == expected(*bs[k], g, cr, 10 + k, true, ls[k]));
    }
    // a burst mixing v and equal-block calls: each change of kind flushes
    if (grouped) {
        ls.clear();
        for (int k = 0; k < 4; k++) {
            ls.emplace_back(g, cr, 20 + k, k != 2);
        }
        fill(*bs[0], g, cr, 20, true, ls[0]);
        fill(*bs[2], g, cr, 22, false, ls[2]);
        fill(*bs[3], g, cr, 23, true, ls[3]);
        neighbor_coll::fill(*bs[1], g, cr, 21, true);
        const uint64_t l1 = launchesOf(comm, rank);
        MPI_Request r[4];
        NV_CHECK(call(true, *bs[0], ls[0], comm, &r[0]) == MPI_SUCCESS);
        NV_CHECK(MPI_Ineighbor_alltoall(bs[1]->send(), neighbor_coll::C, MPI_INT, bs[1]->recv(), neighbor_coll::C,
                                        MPI_INT, comm, &r[1]) == MPI_SUCCESS);
        NV_CHECK(call(false, *bs[2], ls[2], comm, &r[2]) == MPI_SUCCESS);
        NV_CHECK(call(true, *bs[3], ls[3], comm, &r[3]) == MPI_SUCCESS);
        NV_CHECK(launchesOf(comm, rank) == l1 + 3);
        NV_CHECK(MPI_Waitall(4, r, MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        NV_CHECK(launchesOf(comm, rank) == l1 + 4);
        NV_CHECK(bs[0]->get() == expected(*bs[0], g, cr, 20, true, ls[0]));
        NV_CHECK(bs[1]->get() == neighbor_coll::expected(*bs[1], g, cr, 21, true));
        NV_CHECK(bs[2]->get() == expected(*bs[2], g, cr, 22, false, ls[2]));
        NV_CHECK(bs[3]->get() == expected(*bs[3], g, cr, 23, true, ls[3]));
    }
    return 0;
}

// Equal counts: MPI_Neighbor_alltoallv and MPI_Neighbor_allgatherv against
// MPI_Neighbor_alltoall and MPI_Neighbor_allgather on the same inputs
inline int equalCountsV(MPI_Comm comm, const Graph& g, int memory, int rank, std::string* why)
{
    constexpr int C = neighbor_coll::C;
    int cr = -1;
    MPI_Comm_rank(comm, &cr);
    for (int a2a = 0; a2a < 2; a2a++) {
        Bufs a(memory, 1), b(memory, 1);
        NV_CHECK(a.ok() && b.ok());
        MPI_Barrier(comm);
        neighbor_coll::fill(a, g, cr, 40, a2a);
        neighbor_coll::fill(b, g, cr, 40, a2a);
        const int sends = a2a ? (int)g.dst[cr].size() : 1;
        std::vector<int> sc(sends, C), sd(sends), rc(g.in[cr].size(), C), rd(g.in[cr].size());
        for (int i = 0; i < sends; i++) {
            sd[i] = i * C;
        }
        for (size_t j = 0; j < rd.size(); j++) {
            rd[j] = (int)j * C;
        }
        if (a2a) {
            NV_CHECK(MPI_Neighbor_alltoall(a.send(), C, MPI_INT, a.recv(), C, MPI_INT, comm) == MPI_SUCCESS);
            NV_CHECK(MPI_Neighbor_alltoallv(b.send(), sc.data(), sd.data(), MPI_INT, b.recv(), rc.data(), rd.data(),
                                            MPI_INT, comm) == MPI_SUCCESS);
        } else {
            NV_CHECK(MPI_Neighbor_allgather(a.send(), C, MPI_INT, a.recv(), C, MPI_INT, comm) == MPI_SUCCESS);
            NV_CHECK(MPI_Neighbor_allgatherv(b.send(), C, MPI_INT, b.recv(), rc.data(), rd.data(), MPI_INT, comm) ==
                     MPI_SUCCESS);
        }
        NV_CHECK(a.get() == b.get());
        NV_CHECK(a.get() == neighbor_coll::expected(a, g, cr, 40, a2a));
    }
    return 0;
}

inline int body(int rank, int size, int worldId, bool grouped, std::string* why)
{
    (void)worldId;
    const bool gpu = faabric::device::cudaAvailable() && getenv("FAABRIC_DEVICE_BACKEND") == nullptr;
    const Graph g = neighbor_coll::worldGraph(size);
    int rc = MPI_SUCCESS;
    MPI_Comm comm = makeGraph(g, MPI_COMM_WORLD, rank, &rc);
    NV_CHECK(rc == MPI_SUCCESS && comm != MPI_COMM_NULL);

    // ---- refusals: nothing sent or launched, outputs untouched ----
    {
        Bufs b(gpu ? 2 : 1, 1);
        NV_CHECK(b.ok());
        Layout l(g, rank, 0, true);
        fill(b, g, rank, 0, true, l);
        const auto before = b.get();
        NV_CHECK(MPI_Neighbor_alltoallv(MPI_IN_PLACE, l.sc.data(), l.sd.data(), MPI_INT, b.recv(), l.rc.data(),
                                        l.rd.data(), MPI_INT, comm) == MPI_ERR_ARG);
        NV_CHECK(MPI_Neighbor_allgatherv(b.send(), -1, MPI_INT, b.recv(), l.rc.data(), l.rd.data(), MPI_INT, comm) ==
                 MPI_ERR_ARG);
        if (!l.rd.empty()) {
            Layout bad = l;
            bad.rd[0] = -1;
            NV_CHECK(call(true, b, bad, comm, nullptr) == MPI_ERR_ARG);
        }
        MPI_Request r;
        NV_CHECK(MPI_Ineighbor_alltoallv(b.send(), l.sc.data(), l.sd.data(), MPI_INT, b.recv(), l.rc.data(),
                                         l.rd.data(), MPI_INT, MPI_COMM_WORLD, &r) == MPI_ERR_TOPOLOGY);
        NV_CHECK(MPI_Neighbor_allgatherv(b.send(), 1, MPI_INT, b.recv(), l.rc.data(), l.rd.data(), MPI_INT,
                                         MPI_COMM_WORLD) == MPI_ERR_TOPOLOGY);
        NV_CHECK(b.get() == before);
        NV_CHECK(launchesOf(comm, rank) == 0);
    }

    // ---- blocking calls: host, then device buffers ----
    NV_CHECK(blockingV(comm, g, 0, 0, false, rank, why) == 0);
    NV_CHECK(blockingV(comm, g, 1, 0, true, rank, why) == 0);
    NV_CHECK(blockingV(comm, g, 1, 3, true, rank, why) == 0);
    if (gpu) {
        NV_CHECK(blockingV(comm, g, 2, 1, true, rank, why) == 0);
    }
    NV_CHECK(equalCountsV(comm, g, 1, rank, why) == 0);
    NV_CHECK(equalCountsV(comm, g, 0, rank, why) == 0);

    // ---- bursts ----
    NV_CHECK(burstV(comm, g, grouped, rank, why) == 0);

    // ---- a parity split, with a ring on each half ----
    MPI_Comm half = MPI_COMM_NULL;
    MPI_Comm_split(MPI_COMM_WORLD, rank % 2, rank, &half);
    int hr = -1, hn = 0;
    MPI_Comm_rank(half, &hr);
    MPI_Comm_size(half, &hn);
    const Graph ring = neighbor_coll::ringGraph(hn);
    MPI_Comm hg = makeGraph(ring, half, hr, &rc);
    NV_CHECK(rc == MPI_SUCCESS && hg != MPI_COMM_NULL);
    NV_CHECK(blockingV(hg, ring, 1, 2, true, rank, why) == 0);
    NV_CHECK(burstV(hg, ring, grouped, rank, why) == 0);

    // ---- MPI_Comm_free with a v burst pending completes it ----
    {
        Bufs b(1, 2);
        NV_CHECK(b.ok());
        Layout l(g, rank, 30, true);
        fill(b, g, rank, 30, true, l);
        const auto want = expected(b, g, rank, 30, true, l);
        MPI_Request r;
        NV_CHECK(call(true, b, l, comm, &r) == MPI_SUCCESS);
        NV_CHECK(MPI_Comm_free(&comm) == MPI_SUCCESS && comm == MPI_COMM_NULL);
        NV_CHECK(MPI_Wait(&r, MPI_STATUS_IGNORE) == MPI_SUCCESS);
        NV_CHECK(b.get() == want);
    }
    MPI_Comm_free(&hg);
    MPI_Comm_free(&half);
    return 0;
}

} // namespace neighbor_v_coll
