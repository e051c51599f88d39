// One MPI program that checks the deferral of MPI_Raccumulate and
// MPI_Rget_accumulate into the request batch of a symmetric-heap window, with
// origin and result buffers on the origin's GPU or in its heap.  Run by
// test_mpi_rma_accumulate_batch.cpp and by faabric_worker's
// `rma-accumulate-batch` function.
//
// Checked exactly, on every rank: a burst issues nothing before its first
// wait and one launch per FB_RMA_COPY_MAX_ITEMS deferred operations after it;
// counters reach their exact totals; one origin's tickets increase in its
// issue order; MPI_Rput -> MPI_Raccumulate -> MPI_Rget to one location apply
// in that order; an MPI_Accumulate(MPI_REPLACE) after deferred sums lands
// last; every error code comes at issue with nothing queued and the window
// unchanged; a wait after the unlock and a freed request behave as for
// deferred copies.
#pragma once

#include "mpi_rma_request_body.h"

namespace rma_acc_batch {

using rma_atomics::copyBytes;
using rma_request::at64;
using rma_request::Buf;
using rma_request::Origin;
using rma_request::Win;
using rma_request::WIN_BYTES;

// (all below rma_request::COUNTER_OFF, which Win::fill leaves to guard bytes)
constexpr size_t CTR_OFF = 0;        // int64 counter on every rank
constexpr size_t TKT_OFF = 64;       // int64 ticket counter on the last rank
constexpr size_t ORD_OFF = 1024;     // one int64 per origin
constexpr size_t REP_OFF = 2048;     // one int64 per origin
constexpr size_t FREE_OFF = 3072;    // one int64 per origin
constexpr size_t ERR_OFF = 4096;     // never written
constexpr size_t ZERO_BYTES = 8192;  // zeroed before the program
constexpr int K = 300;               // burst rounds

inline int body(int rank, int size, int worldId, Origin origin, std::string* why)
{
    auto comm = faabric::mpi::getMpiWorldRegistry().getWorld(worldId).getDeviceComm(rank);
    RMA_CHECK(comm != nullptr);
    auto launches = [&]() { return comm->stats().launches; };
    Win w;
    RMA_CHECK(w.create(rma_atomics::WindowMemory::Heap));
    copyBytes(w.base, std::vector<uint8_t>(ZERO_BYTES, 0).data(), ZERO_BYTES);
    Buf io(16384, origin); // [0, 8): one int64 1; results from 64 on
    RMA_CHECK(io.p != nullptr);
    {
        std::vector<uint8_t> v(io.n, 0);
        const int64_t one = 1;
        memcpy(v.data(), &one, 8);
        io.write(v);
    }
    MPI_Barrier(MPI_COMM_WORLD);
    const int owner = size - 1;

    // ---- (a) a burst of counter updates and tickets: nothing before the
    // first wait, one launch per 1024 deferred operations after it
    {
        std::vector<MPI_Request> reqs;
        RMA_CHECK(MPI_Win_lock_all(0, w.win) == MPI_SUCCESS);
        const uint64_t before = launches();
        size_t deferred = 0;
        for (int k = 0; k < K; k++) {
            for (int t = 0; t < size; t++) {
                reqs.emplace_back(nullptr);
                RMA_CHECK(MPI_Raccumulate(io.p, 1, MPI_INT64_T, t, CTR_OFF, 1, MPI_INT64_T, MPI_SUM, w.win, &reqs.back()) ==
                          MPI_SUCCESS);
            }
            reqs.emplace_back(nullptr);
            RMA_CHECK(MPI_Rget_accumulate(io.p, 1, MPI_INT64_T, io.p + 64 + 8 * k, 1, MPI_INT64_T, owner, TKT_OFF, 1,
                                          MPI_INT64_T, MPI_SUM, w.win, &reqs.back()) == MPI_SUCCESS);
            deferred += size + 1;
            // a full batch is issued at once, anything less waits
            RMA_CHECK(launches() - before == deferred / 1024);
        }
        RMA_CHECK(MPI_Wait(&reqs.back(), MPI_STATUS_IGNORE) == MPI_SUCCESS);
        RMA_CHECK(launches() - before == (deferred + 1023) / 1024);
        RMA_CHECK(MPI_Waitall((int)reqs.size(), reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        RMA_CHECK(launches() - before == (deferred + 1023) / 1024);
        const auto mine = io.read();
        RMA_CHECK(MPI_Win_unlock_all(w.win) == MPI_SUCCESS);
        MPI_Barrier(MPI_COMM_WORLD);
        RMA_CHECK(at64(w.read(), CTR_OFF) == (int64_t)size * K);
        std::vector<int64_t> tickets(K), all((size_t)size * K);
        memcpy(tickets.data(), mine.data() + 64, 8 * K);
        for (int k = 1; k < K; k++) {
            RMA_CHECK(tickets[k] > tickets[k - 1]); // this origin's issue order
        }
        MPI_Allgather(tickets.data(), K, MPI_INT64_T, all.data(), K, MPI_INT64_T, MPI_COMM_WORLD);
        std::sort(all.begin(), all.end());
        for (int i = 0; i < size * K; i++) {
            RMA_CHECK(all[i] == i);
        }
        if (rank == owner) {
            RMA_CHECK(at64(w.read(), TKT_OFF) == (int64_t)size * K);
        }
    }

    // ---- (b) MPI_Rput -> MPI_Raccumulate -> MPI_Rget to one location, one
    // launch per run of the batch
    {
        const int t = (rank + 1) % size;
        const size_t off = ORD_OFF + 8 * (size_t)rank;
        std::vector<uint8_t> v(io.n, 0);
        const int64_t five = 5, three = 3;
        memcpy(v.data(), &five, 8);
        memcpy(v.data() + 8, &three, 8);
        io.write(v);
        MPI_Request r[3] = { nullptr, nullptr, nullptr };
        RMA_CHECK(MPI_Win_lock(MPI_LOCK_SHARED, t, 0, w.win) == MPI_SUCCESS);
        const uint64_t before = launches();
        RMA_CHECK(MPI_Rput(io.p, 8, MPI_BYTE, t, off, 8, MPI_BYTE, w.win, &r[0]) == MPI_SUCCESS);
        RMA_CHECK(MPI_Raccumulate(io.p + 8, 1, MPI_INT64_T, t, off, 1, MPI_INT64_T, MPI_SUM, w.win, &r[1]) == MPI_SUCCESS);
        RMA_CHECK(MPI_Rget(io.p + 16, 8, MPI_BYTE, t, off, 8, MPI_BYTE, w.win, &r[2]) == MPI_SUCCESS);
        RMA_CHECK(launches() == before);
        RMA_CHECK(MPI_Waitall(3, r, MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        RMA_CHECK(launches() == before + 3);
        RMA_CHECK(at64(io.read(), 16) == 8);
        RMA_CHECK(MPI_Win_unlock(t, w.win) == MPI_SUCCESS);
        MPI_Barrier(MPI_COMM_WORLD);
        RMA_CHECK(at64(w.read(), ORD_OFF + 8 * (size_t)((rank + size - 1) % size)) == 8);
    }

    // ---- (c) an MPI_Accumulate(MPI_REPLACE) after deferred sums on the same
    // element lands last
    {
        const int t = (rank + 1) % size;
        const size_t off = REP_OFF + 8 * (size_t)rank;
        std::vector<uint8_t> v(io.n, 0);
        const int64_t one = 1, hundred = 100;
        memcpy(v.data(), &one, 8);
        memcpy(v.data() + 8, &hundred, 8);
        io.write(v);
        std::vector<MPI_Request> reqs(10, nullptr);
        RMA_CHECK(MPI_Win_lock(MPI_LOCK_SHARED, t, 0, w.win) == MPI_SUCCESS);
        for (auto& r : reqs) {
            RMA_CHECK(MPI_Raccumulate(io.p, 1, MPI_INT64_T, t, off, 1, MPI_INT64_T, MPI_SUM, w.win, &r) == MPI_SUCCESS);
        }
        RMA_CHECK(MPI_Accumulate(io.p + 8, 1, MPI_INT64_T, t, off, 1, MPI_INT64_T, MPI_REPLACE, w.win) == MPI_SUCCESS);
        RMA_CHECK(MPI_Waitall((int)reqs.size(), reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        RMA_CHECK(MPI_Win_unlock(t, w.win) == MPI_SUCCESS);
        MPI_Barrier(MPI_COMM_WORLD);
        RMA_CHECK(at64(w.read(), REP_OFF + 8 * (size_t)((rank + size - 1) % size)) == 100);
    }

    // ---- (d) every error code at issue: nothing queued, window unchanged
    {
        const int t = (rank + 1) % size;
        MPI_Request r = nullptr;
        MPI_Barrier(MPI_COMM_WORLD);
        const auto before = w.read();
        const uint64_t l0 = launches();
        RMA_CHECK(MPI_Raccumulate(io.p, 1, MPI_INT64_T, t, ERR_OFF, 1, MPI_INT64_T, MPI_SUM, nullptr, &r) == MPI_ERR_WIN);
        RMA_CHECK(MPI_Raccumulate(io.p, 1, MPI_INT64_T, t, ERR_OFF, 1, MPI_INT64_T, MPI_SUM, w.win, &r) ==
                  MPI_ERR_RMA_SYNC);
        RMA_CHECK(MPI_Win_lock_all(0, w.win) == MPI_SUCCESS);
        RMA_CHECK(MPI_Raccumulate(io.p, 1, MPI_INT64_T, size, ERR_OFF, 1, MPI_INT64_T, MPI_SUM, w.win, &r) == MPI_ERR_RANK);
        RMA_CHECK(MPI_Raccumulate(io.p, 1, MPI_INT64_T, t, ERR_OFF, 1, MPI_INT64_T, MPI_NO_OP, w.win, &r) == MPI_ERR_OP);
        RMA_CHECK(MPI_Raccumulate(io.p, 1, MPI_FLOAT, t, ERR_OFF, 1, MPI_FLOAT, MPI_BAND, w.win, &r) == MPI_ERR_OP);
        RMA_CHECK(MPI_Raccumulate(io.p, 1, MPI_INT64_T, t, ERR_OFF + 4, 1, MPI_INT64_T, MPI_SUM, w.win, &r) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Raccumulate(io.p, 1, MPI_INT64_T, t, WIN_BYTES - 4, 1, MPI_INT64_T, MPI_SUM, w.win, &r) ==
                  MPI_ERR_ARG);
        RMA_CHECK(MPI_Raccumulate(nullptr, 1, MPI_INT64_T, t, ERR_OFF, 1, MPI_INT64_T, MPI_SUM, w.win, &r) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Rget_accumulate(io.p, 1, MPI_INT64_T, io.p + 64, 1, MPI_INT64_T, t, ERR_OFF, 1, MPI_INT64_T, MPI_SUM,
                                      w.win, nullptr) == MPI_ERR_ARG);
        RMA_CHECK(r == nullptr);
        RMA_CHECK(MPI_Win_unlock_all(w.win) == MPI_SUCCESS);
        RMA_CHECK(launches() == l0);
        MPI_Barrier(MPI_COMM_WORLD);
        const bool unchanged = w.read() == before;
        MPI_Barrier(MPI_COMM_WORLD); // (before (e) writes to this window)
        RMA_CHECK(unchanged);
    }

    // ---- (e) a wait after the unlock returns; a freed request completes at
    // the unlock
    {
        const int t = (rank + 1) % size;
        const size_t off = FREE_OFF + 8 * (size_t)rank;
        std::vector<uint8_t> v(io.n, 0);
        const int64_t one = 1;
        memcpy(v.data(), &one, 8);
        io.write(v);
        MPI_Request late = nullptr, freed = nullptr;
        RMA_CHECK(MPI_Win_lock(MPI_LOCK_SHARED, t, 0, w.win) == MPI_SUCCESS);
        RMA_CHECK(MPI_Raccumulate(io.p, 1, MPI_INT64_T, t, off, 1, MPI_INT64_T, MPI_SUM, w.win, &late) == MPI_SUCCESS);
        RMA_CHECK(MPI_Rget_accumulate(io.p, 1, MPI_INT64_T, io.p + 64, 1, MPI_INT64_T, t, off, 1, MPI_INT64_T, MPI_SUM,
                                      w.win, &freed) == MPI_SUCCESS);
        RMA_CHECK(MPI_Request_free(&freed) == MPI_SUCCESS && freed == nullptr);
        RMA_CHECK(MPI_Win_unlock(t, w.win) == MPI_SUCCESS);
        RMA_CHECK(MPI_Wait(&late, MPI_STATUS_IGNORE) == MPI_SUCCESS && late == nullptr);
        RMA_CHECK(at64(io.read(), 64) == 1); // the freed fetch landed at the unlock
        MPI_Barrier(MPI_COMM_WORLD);
        RMA_CHECK(at64(w.read(), FREE_OFF + 8 * (size_t)((rank + size - 1) % size)) == 2);
    }

    MPI_Barrier(MPI_COMM_WORLD);
    w.destroy();
    return 0;
}

} // namespace rma_acc_batch
