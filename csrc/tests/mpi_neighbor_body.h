// One MPI program for the distributed-graph topology and the neighbourhood
// collectives: MPI_Dist_graph_create_adjacent on the world and on a parity
// split, the queries and MPI_Topo_test, blocking and non-blocking
// MPI_Neighbor_allgather / MPI_Neighbor_alltoall with inputs rewritten every
// round on host, heap, unaligned-heap and (on a GPU) cudaMalloc buffers,
// checked word for word (guard words included) against a closed form.  The
// world graph has self-edges, multi-edges listed in a different order on the
// two sides, and (from 4 ranks) a rank with no edge that still passes device
// pointers.  Launch counts: one per blocking device call, one per burst,
// nothing before the first wait, flushes by another kind and by a blocking
// call; with grouping off one launch per call at issue.  The refusals
// (MPI_ERR_ARG, MPI_ERR_TOPOLOGY, MPI_ERR_RANK) leave the outputs untouched
// and every member agrees on an invalid graph; MPI_Comm_free with a burst
// pending completes it.  Shared by test_loopback_neighbor.cpp and
// test_device_neighbor.cpp (through mpi_neighbor_run.h) and faabric_worker's
// `neighbor-coll`, which tests/test_dist_neighbor.py runs with one rank in
// each of four worker processes.
#pragma once

#include "mpi/subcomm.h"
#include "mpi_subcomm_device_body.h"

#include <faabric/device/cuda_driver.h>
#include <faabric/mpi/MpiWorld.h>
#include <faabric/mpi/MpiWorldRegistry.h>
#include <faabric/mpi/mpi.h>

#include <cstdint>
#include <memory>
#include <string>
#include <vector>

namespace neighbor_coll {

using subcomm_device::BufferMemory;
using subcomm_device::DevBuffer;

#define NB_CHECK(cond)                                                         \
    do {                                                                       \
        if (!(cond)) {                                                         \
            *why = "rank " + std::to_string(rank) + ": check failed at line " + std::to_string(__LINE__) + ": " #cond; \
            return 1;                                                          \
        }                                                                      \
    } while (0)

constexpr int C = 37;     // words per block (148 bytes: no multiple of 16)
constexpr int SLOT = 160; // words per buffer slot: room for 4 blocks
constexpr int K = 4;      // calls per burst

// A graph in comm ranks, with every rank's in-edges (source, index of the
// edge in the source's destinations)
struct Graph
{
    std::vector<std::vector<int>> src, dst;
    std::vector<std::vector<std::pair<int, int>>> in;

    void pair()
    {
        const int n = (int)src.size();
        in.assign(n, {});
        for (int d = 0; d < n; d++) {
            std::vector<int> seen(n, 0);
            for (int s : src[d]) {
                int k = seen[s]++;
                for (size_t i = 0; i < dst[s].size(); i++) {
                    if (dst[s][i] == d && k-- == 0) {
                        in[d].push_back({ s, (int)i });
                        break;
                    }
                }
            }
        }
    }
};

// Ranks [0, a) with a = n, or n - 1 from 4 ranks (the last has no edge):
// rank r sends to its successor twice and to itself, and lists itself first
// and its predecessor twice
inline Graph worldGraph(int n)
{
    const int a = n >= 4 ? n - 1 : n;
    Graph g;
    g.src.assign(n, {});
    g.dst.assign(n, {});
    for (int r = 0; r < a; r++) {
        g.dst[r] = { (r + 1) % a, (r + 1) % a, r };
        g.src[r] = { r, (r + a - 1) % a, (r + a - 1) % a };
    }
    g.pair();
    return g;
}

inline Graph ringGraph(int n)
{
    Graph g;
    g.src.assign(n, {});
    g.dst.assign(n, {});
    for (int r = 0; r < n; r++) {
        g.dst[r] = { (r + 1) % n };
        g.src[r] = { (r + n - 1) % n };
    }
    g.pair();
    return g;
}

inline int32_t word(int commRank, int round, int block, int w)
{
    return commRank * 1000000 + round * 10000 + block * 1000 + w + 1;
}

// Buffers of one call kind: send at word `off`, recv at SLOT + off; guards
// everywhere else
struct Bufs
{
    std::vector<int32_t> hostMem;
    std::unique_ptr<DevBuffer> dev;
    int32_t* base = nullptr;
    int off = 0;

    Bufs(int memory, int offIn) // 0 host, 1 heap, 2 cudaMalloc
      : off(offIn)
    {
        if (memory == 0) {
            hostMem.assign(2 * SLOT + 8, 0);
            base = hostMem.data();
        } else {
            dev = std::make_unique<DevBuffer>(2 * SLOT + 8, memory == 1 ? BufferMemory::Heap : BufferMemory::CudaMalloc);
            base = dev->ptr;
        }
    }
    bool ok() const { return base != nullptr; }
    int32_t* send() { return base + off; }
    int32_t* recv() { return base + SLOT + off; }
    std::vector<int32_t>& host()
    {
        return dev ? dev->host : hostMem;
    }
    void put()
    {
        if (dev) {
            dev->upload();
        }
    }
    const std::vector<int32_t>& get()
    {
        return dev ? dev->read() : hostMem;
    }
};

// Guards -7, the send blocks of `round`
inline void fill(Bufs& b, const Graph& g, int cr, int round, bool a2a)
{
    auto& h = b.host();
    std::fill(h.begin(), h.end(), -7);
    const int blocks = a2a ? (int)g.dst[cr].size() : 1;
    for (int i = 0; i < blocks; i++) {
        for (int w = 0; w < C; w++) {
            h[b.off + i * C + w] = word(cr, round, i, w);
        }
    }
    b.put();
}

inline std::vector<int32_t> expected(Bufs& b, const Graph& g, int cr, int round, bool a2a)
{
    std::vector<int32_t> want = b.host();
    for (size_t j = 0; j < g.in[cr].size(); j++) {
        const auto [s, idx] = g.in[cr][j];
        for (int w = 0; w < C; w++) {
            want[SLOT + b.off + j * C + w] = word(s, round, a2a ? idx : 0, w);
        }
    }
    return want;
}

inline MPI_Comm makeGraph(const Graph& g, MPI_Comm parent, int cr, int* rc)
{
    MPI_Comm out = MPI_COMM_NULL;
    *rc = MPI_Dist_graph_create_adjacent(parent, (int)g.src[cr].size(), g.src[cr].data(), MPI_UNWEIGHTED,
                                         (int)g.dst[cr].size(), g.dst[cr].data(), MPI_UNWEIGHTED, MPI_INFO_NULL, 0,
                                         &out);
    return out;
}

inline std::shared_ptr<faabric::device::Communicator> childOf(MPI_Comm comm, int rank)
{
    auto sub = faabric::mpi::getSubCommunicator(comm->id);
    return sub == nullptr ? nullptr : sub->currentDevice(rank);
}

inline uint64_t launchesOf(MPI_Comm comm, int rank)
{
    auto c = childOf(comm, rank);
    return c == nullptr ? 0 : c->stats().launches;
}

// Blocking calls of both kinds over `rounds` rounds; `device`: each is one
// launch on the communicator's child
inline int blocking(MPI_Comm comm, const Graph& g, int memory, int off, bool device, int rank, std::string* why)
{
    int cr = -1;
    MPI_Comm_rank(comm, &cr);
    Bufs b(memory, off);
    NB_CHECK(b.ok());
    for (int round = 0; round < 3; round++) {
        for (int a2a = 0; a2a < 2; a2a++) {
            fill(b, g, cr, round, a2a);
            const auto want = expected(b, g, cr, round, a2a);
            const uint64_t l0 = launchesOf(comm, rank);
            const int rc = a2a ? MPI_Neighbor_alltoall(b.send(), C, MPI_INT, b.recv(), C, MPI_INT, comm)
                               : MPI_Neighbor_allgather(b.send(), C, MPI_INT, b.recv(), C, MPI_INT, comm);
            NB_CHECK(rc == MPI_SUCCESS);
            // (the first device call creates the child: its count starts at 0)
            NB_CHECK(launchesOf(comm, rank) == l0 + (device ? 1u : 0u));
            NB_CHECK(b.get() == want);
        }
    }
    if (device) {
        NB_CHECK(childOf(comm, rank) != nullptr && childOf(comm, rank)->hasNeighbors());
    }
    return 0;
}

// K non-blocking all-to-alls on heap buffers: nothing before the first wait
// and one launch after it (grouped), or one launch per call at issue
inline int burst(MPI_Comm comm, const Graph& g, bool grouped, int rank, std::string* why)
{
    int cr = -1;
    MPI_Comm_rank(comm, &cr);
    std::vector<std::unique_ptr<Bufs>> bs;
    for (int k = 0; k < K; k++) {
        bs.push_back(std::make_unique<Bufs>(1, 1 + k % 3));
        NB_CHECK(bs.back()->ok());
        fill(*bs.back(), g, cr, 10 + k, true);
    }
    MPI_Barrier(comm);
    const uint64_t l0 = launchesOf(comm, rank);
    std::vector<MPI_Request> reqs(K);
    for (int k = 0; k < K; k++) {
        NB_CHECK(MPI_Ineighbor_alltoall(bs[k]->send(), C, MPI_INT, bs[k]->recv(), C, MPI_INT, comm, &reqs[k]) ==
                 MPI_SUCCESS);
    }
    NB_CHECK(launchesOf(comm, rank) == l0 + (grouped ? 0u : (uint64_t)K));
    NB_CHECK(MPI_Waitall(K, reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
    NB_CHECK(launchesOf(comm, rank) == l0 + (grouped ? 1u : (uint64_t)K));
    for (int k = 0; k < K; k++) {
        const auto want = expected(*bs[k], g, cr, 10 + k, true);
        NB_CHECK(bs[k]->get() == want);
    }
    // another kind flushes the pending burst at its issue, and a blocking
    // call flushes too
    if (grouped) {
        for (int k = 0; k < 3; k++) {
            fill(*bs[k], g, cr, 20 + k, k != 1);
        }
        const uint64_t l1 = launchesOf(comm, rank);
        MPI_Request r2[2];
        NB_CHECK(MPI_Ineighbor_alltoall(bs[0]->send(), C, MPI_INT, bs[0]->recv(), C, MPI_INT, comm, &r2[0]) ==
                 MPI_SUCCESS);
        NB_CHECK(MPI_Ineighbor_allgather(bs[1]->send(), C, MPI_INT, bs[1]->recv(), C, MPI_INT, comm, &r2[1]) ==
                 MPI_SUCCESS);
        NB_CHECK(launchesOf(comm, rank) == l1 + 1);
        NB_CHECK(MPI_Neighbor_alltoall(bs[2]->send(), C, MPI_INT, bs[2]->recv(), C, MPI_INT, comm) == MPI_SUCCESS);
        NB_CHECK(launchesOf(comm, rank) == l1 + 3);
        NB_CHECK(MPI_Waitall(2, r2, MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        NB_CHECK(launchesOf(comm, rank) == l1 + 3);
        for (int k = 0; k < 3; k++) {
            const auto want = expected(*bs[k], g, cr, 20 + k, k != 1);
            NB_CHECK(bs[k]->get() == want);
        }
    }
    return 0;
}

inline int body(int rank, int size, int worldId, bool grouped, std::string* why)
{
    (void)worldId;
    // (cudaMalloc buffers only on a GPU, not on the loopback backend)
    const bool gpu = faabric::device::cudaAvailable() && getenv("FAABRIC_DEVICE_BACKEND") == nullptr;
    const Graph g = worldGraph(size);
    int rc = MPI_SUCCESS;

    // ---- refusals of the constructor: every member agrees ----
    {
        // an edge r -> r+1 that r+1 does not list
        std::vector<int> d = { (rank + 1) % size };
        MPI_Comm bad = MPI_COMM_NULL;
        rc = MPI_Dist_graph_create_adjacent(MPI_COMM_WORLD, 0, nullptr, MPI_UNWEIGHTED, 1, d.data(), MPI_UNWEIGHTED,
                                            MPI_INFO_NULL, 0, &bad);
        NB_CHECK(rc == MPI_ERR_TOPOLOGY && bad == MPI_COMM_NULL);
        // a rank outside the world, on rank 0 only
        std::vector<int> s = { rank == 0 ? size : rank };
        rc = MPI_Dist_graph_create_adjacent(MPI_COMM_WORLD, 1, s.data(), MPI_UNWEIGHTED, 1, &rank, MPI_UNWEIGHTED,
                                            MPI_INFO_NULL, 0, &bad);
        NB_CHECK(rc == MPI_ERR_RANK && bad == MPI_COMM_NULL);
        // a negative degree on the last rank only
        rc = MPI_Dist_graph_create_adjacent(MPI_COMM_WORLD, rank == size - 1 ? -1 : 0, nullptr, MPI_UNWEIGHTED, 0,
                                            nullptr, MPI_UNWEIGHTED, MPI_INFO_NULL, 0, &bad);
        NB_CHECK(rc == MPI_ERR_ARG && bad == MPI_COMM_NULL);
    }

    // ---- the world graph, its queries ----
    MPI_Comm comm = makeGraph(g, MPI_COMM_WORLD, rank, &rc);
    NB_CHECK(rc == MPI_SUCCESS && comm != MPI_COMM_NULL);
    int status = 0;
    NB_CHECK(MPI_Topo_test(comm, &status) == MPI_SUCCESS && status == MPI_DIST_GRAPH);
    NB_CHECK(MPI_Topo_test(MPI_COMM_WORLD, &status) == MPI_SUCCESS && status == MPI_UNDEFINED);
    int indeg = -1, outdeg = -1, weighted = -1;
    NB_CHECK(MPI_Dist_graph_neighbors_count(comm, &indeg, &outdeg, &weighted) == MPI_SUCCESS);
    NB_CHECK(indeg == (int)g.src[rank].size() && outdeg == (int)g.dst[rank].size() && weighted == 0);
    std::vector<int> qs(4, -1), qd(4, -1);
    NB_CHECK(MPI_Dist_graph_neighbors(comm, 4, qs.data(), MPI_UNWEIGHTED, 4, qd.data(), MPI_UNWEIGHTED) ==
             MPI_SUCCESS);
    qs.resize(indeg);
    qd.resize(outdeg);
    NB_CHECK(qs == g.src[rank] && qd == g.dst[rank]);

    // ---- refusals of the calls: nothing sent or launched, outputs untouched ----
    {
        Bufs b(gpu ? 2 : 1, 1);
        NB_CHECK(b.ok());
        fill(b, g, rank, 0, true);
        const auto before = b.get();
        NB_CHECK(MPI_Neighbor_alltoall(MPI_IN_PLACE, C, MPI_INT, b.recv(), C, MPI_INT, comm) == MPI_ERR_ARG);
        NB_CHECK(MPI_Neighbor_allgather(b.send(), C, MPI_INT, b.recv(), C + 1, MPI_INT, comm) == MPI_ERR_ARG);
        MPI_Request r;
        NB_CHECK(MPI_Ineighbor_alltoall(b.send(), C, MPI_INT, b.recv(), C, MPI_INT, MPI_COMM_WORLD, &r) ==
                 MPI_ERR_TOPOLOGY);
        NB_CHECK(MPI_Neighbor_allgather(b.send(), C, MPI_INT, b.recv(), C, MPI_INT, MPI_COMM_WORLD) ==
                 MPI_ERR_TOPOLOGY);
        NB_CHECK(b.get() == before);
        NB_CHECK(launchesOf(comm, rank) == 0);
    }

    // ---- blocking calls: host, then device buffers ----
    NB_CHECK(blocking(comm, g, 0, 0, false, rank, why) == 0);
    NB_CHECK(blocking(comm, g, 1, 0, true, rank, why) == 0);
    NB_CHECK(blocking(comm, g, 1, 3, true, rank, why) == 0);
    if (gpu) {
        NB_CHECK(blocking(comm, g, 2, 1, true, rank, why) == 0);
    }

    // ---- bursts ----
    NB_CHECK(burst(comm, g, grouped, rank, why) == 0);

    // ---- a parity split, with a ring on each half ----
    MPI_Comm half = MPI_COMM_NULL;
    MPI_Comm_split(MPI_COMM_WORLD, rank % 2, rank, &half);
    int hr = -1, hn = 0;
    MPI_Comm_rank(half, &hr);
    MPI_Comm_size(half, &hn);
    const Graph ring = ringGraph(hn);
    MPI_Comm hg = makeGraph(ring, half, hr, &rc);
    NB_CHECK(rc == MPI_SUCCESS && hg != MPI_COMM_NULL);
    NB_CHECK(blocking(hg, ring, 1, 2, true, rank, why) == 0);
    NB_CHECK(burst(hg, ring, grouped, rank, why) == 0);
    // a split of a dist-graph communicator carries no topology
    MPI_Comm nested = MPI_COMM_NULL;
    MPI_Comm_split(hg, 0, hr, &nested);
    NB_CHECK(MPI_Topo_test(nested, &status) == MPI_SUCCESS && status == MPI_UNDEFINED);
    MPI_Comm_free(&nested);

    // ---- MPI_Comm_free with a burst pending completes it ----
    {
        Bufs b(1, 2);
        NB_CHECK(b.ok());
        fill(b, g, rank, 30, true);
        const auto want = expected(b, g, rank, 30, true);
        MPI_Request r;
        NB_CHECK(MPI_Ineighbor_alltoall(b.send(), C, MPI_INT, b.recv(), C, MPI_INT, comm, &r) == MPI_SUCCESS);
        NB_CHECK(MPI_Comm_free(&comm) == MPI_SUCCESS && comm == MPI_COMM_NULL);
        NB_CHECK(MPI_Wait(&r, MPI_STATUS_IGNORE) == MPI_SUCCESS);
        NB_CHECK(b.get() == want);
    }
    MPI_Comm_free(&hg);
    MPI_Comm_free(&half);
    return 0;
}

} // namespace neighbor_coll
