// One MPI program that checks passive-target synchronisation (MPI_Win_lock,
// MPI_Win_unlock, MPI_Win_lock_all, MPI_Win_flush*, MPI_Win_sync) on one kind
// of window.  Shared by the in-process tests (test_mpi_rma_passive.cpp) and
// the `rma-passive` function of faabric_worker, which runs it across worker
// processes.  The window, buffer and setup helpers are those of
// mpi_rma_atomics_body.h.
//
// Every check is exact: a counter incremented under an exclusive lock by a
// read-modify-write that is not atomic, unique fetch-and-op tickets, values
// a target reads from its own memory after the origin's flush, a two-word
// invariant never seen half written, and every synchronisation error.
#pragma once

#include "mpi_rma_atomics_body.h"

#include <faabric/mpi/MpiWorldRegistry.h>
#include <faabric/mpi/mpi.h>

#include <cstdint>
#include <cstring>
#include <set>
#include <string>
#include <vector>

namespace rma_passive {

using rma_atomics::Buffer;
using rma_atomics::Setup;
using rma_atomics::Window;
using rma_atomics::WindowMemory;

constexpr size_t MUTEX_OFF = 0;       // int64 counter on rank 0
constexpr size_t TICKET_OFF = 64;     // int64, int32 and int8 counters on the last rank
constexpr size_t VISIBLE_OFF = 1024;  // int64 per origin
constexpr size_t PAIR_OFF = 2048;     // two int64 words on rank 0
constexpr size_t NOCHECK_OFF = 3072;  // int64 per origin
constexpr size_t ALL_OFF = 4096;      // int64 per origin
constexpr size_t FENCE_OFF = 6144;    // int64 per origin

inline int64_t load64(Buffer& b, size_t off)
{
    int64_t v;
    memcpy(&v, b.read().data() + off, 8);
    return v;
}

inline void store64(Buffer& b, size_t off, int64_t v)
{
    memcpy(b.host.data() + off, &v, 8);
    b.upload();
}

inline int body(int rank, int size, int worldId, const Setup& s, std::string* why)
{
    Window w;
    RMA_CHECK(w.create(s.window));
    Buffer io(64, s.deviceBuffers);
    RMA_CHECK(io.ok());

    // ---- 1. mutual exclusion: get, flush, put +1 under an exclusive lock.
    // The read-modify-write is not atomic; only the lock makes it count.
    {
        const int K = 10;
        for (int k = 0; k < K; k++) {
            RMA_CHECK(MPI_Win_lock(MPI_LOCK_EXCLUSIVE, 0, 0, w.win) == MPI_SUCCESS);
            RMA_CHECK(MPI_Get(io.ptr(), 1, MPI_INT64_T, 0, MUTEX_OFF, 1, MPI_INT64_T, w.win) == MPI_SUCCESS);
            RMA_CHECK(MPI_Win_flush(0, w.win) == MPI_SUCCESS);
            store64(io, 8, load64(io, 0) + 1);
            RMA_CHECK(MPI_Put(io.ptr() + 8, 1, MPI_INT64_T, 0, MUTEX_OFF, 1, MPI_INT64_T, w.win) == MPI_SUCCESS);
            RMA_CHECK(MPI_Win_unlock(0, w.win) == MPI_SUCCESS);
        }
        MPI_Barrier(MPI_COMM_WORLD);
        if (rank == 0) {
            int64_t c;
            memcpy(&c, w.read(MUTEX_OFF, 8).data(), 8);
            RMA_CHECK(c == (int64_t)size * K);
        }
    }

    // ---- 2. tickets without a fence: MPI_Fetch_and_op + MPI_Win_flush on
    // 64-, 32- and 8-bit counters inside MPI_Win_lock_all
    {
        const int K = 20; // size * K < 128: the int8 counter does not wrap
        const int owner = size - 1;
        Buffer one(16, s.deviceBuffers), got(16, s.deviceBuffers);
        RMA_CHECK(one.ok() && got.ok());
        int64_t one64 = 1;
        int32_t one32 = 1;
        int8_t one8 = 1;
        memcpy(one.host.data(), &one64, 8);
        memcpy(one.host.data() + 8, &one32, 4);
        memcpy(one.host.data() + 12, &one8, 1);
        one.upload();
        std::vector<int64_t> local(3 * K);
        RMA_CHECK(MPI_Win_lock_all(0, w.win) == MPI_SUCCESS);
        for (int k = 0; k < K; k++) {
            RMA_CHECK(MPI_Fetch_and_op(one.ptr(), got.ptr(), MPI_INT64_T, owner, TICKET_OFF, MPI_SUM, w.win) == MPI_SUCCESS);
            RMA_CHECK(MPI_Fetch_and_op(one.ptr() + 8, got.ptr() + 8, MPI_INT32_T, owner, TICKET_OFF + 8, MPI_SUM, w.win) == MPI_SUCCESS);
            RMA_CHECK(MPI_Fetch_and_op(one.ptr() + 12, got.ptr() + 12, MPI_INT8_T, owner, TICKET_OFF + 13, MPI_SUM, w.win) == MPI_SUCCESS);
            RMA_CHECK(MPI_Win_flush(owner, w.win) == MPI_SUCCESS);
            // the tickets are usable now
            const auto& t = got.read();
            int32_t t32;
            memcpy(&local[3 * k], t.data(), 8);
            memcpy(&t32, t.data() + 8, 4);
            local[3 * k + 1] = t32;
            local[3 * k + 2] = (int8_t)t[12];
        }
        RMA_CHECK(MPI_Win_unlock_all(w.win) == MPI_SUCCESS);
        std::vector<int64_t> all(3 * K * size);
        MPI_Allgather(local.data(), 3 * K, MPI_INT64_T, all.data(), 3 * K, MPI_INT64_T, MPI_COMM_WORLD);
        for (int c = 0; c < 3; c++) {
            std::set<int64_t> seen;
            for (int r = 0; r < size; r++) {
                for (int k = 0; k < K; k++) {
                    seen.insert(all[(size_t)r * 3 * K + 3 * k + c]);
                }
            }
            RMA_CHECK((int)seen.size() == size * K && *seen.begin() == 0 && *seen.rbegin() == size * K - 1);
        }
        if (rank == owner) {
            auto c = w.read(TICKET_OFF, 16);
            int64_t c64;
            int32_t c32;
            memcpy(&c64, c.data(), 8);
            memcpy(&c32, c.data() + 8, 4);
            RMA_CHECK(c64 == size * K && c32 == size * K && (int8_t)c[13] == size * K);
            // the neighbours of the int8 counter are untouched
            RMA_CHECK(c[12] == 0 && c[14] == 0 && c[15] == 0);
        }
    }

    // ---- 3. visible at the target after the origin's flush: the target
    // reads its own memory, no fence in between
    {
        const int right = (rank + 1) % size, left = (rank + size - 1) % size;
        store64(io, 0, 1000 + rank);
        RMA_CHECK(MPI_Win_lock(MPI_LOCK_SHARED, right, 0, w.win) == MPI_SUCCESS);
        RMA_CHECK(MPI_Accumulate(io.ptr(), 1, MPI_INT64_T, right, VISIBLE_OFF + 8 * rank, 1, MPI_INT64_T, MPI_SUM, w.win) == MPI_SUCCESS);
        RMA_CHECK(MPI_Win_flush(right, w.win) == MPI_SUCCESS);
        int flushed = 1, seen = 0;
        MPI_Send(&flushed, 1, MPI_INT, right, 0, MPI_COMM_WORLD);
        MPI_Recv(&seen, 1, MPI_INT, left, 0, MPI_COMM_WORLD, MPI_STATUS_IGNORE);
        int64_t v;
        memcpy(&v, w.read(VISIBLE_OFF + 8 * left, 8).data(), 8);
        RMA_CHECK(seen == 1 && v == 1000 + left);
        RMA_CHECK(MPI_Win_unlock(right, w.win) == MPI_SUCCESS);
    }

    // ---- 4a. shared locks coexist: A holds SHARED on rank 0 while B takes
    // it too (an exclusive lock would make B fail at the timeout)
    if (size >= 2) {
        const int a = size - 1, b = size - 2;
        int go = 1, bGot = -1;
        if (rank == a) {
            RMA_CHECK(MPI_Win_lock(MPI_LOCK_SHARED, 0, 0, w.win) == MPI_SUCCESS);
            MPI_Send(&go, 1, MPI_INT, b, 1, MPI_COMM_WORLD);
            MPI_Recv(&bGot, 1, MPI_INT, b, 2, MPI_COMM_WORLD, MPI_STATUS_IGNORE);
            RMA_CHECK(MPI_Win_unlock(0, w.win) == MPI_SUCCESS);
            RMA_CHECK(bGot == MPI_SUCCESS);
        } else if (rank == b) {
            MPI_Recv(&go, 1, MPI_INT, a, 1, MPI_COMM_WORLD, MPI_STATUS_IGNORE);
            int rc = MPI_Win_lock(MPI_LOCK_SHARED, 0, 0, w.win);
            // (answer either way: A must not hang)
            MPI_Send(&rc, 1, MPI_INT, a, 2, MPI_COMM_WORLD);
            RMA_CHECK(rc == MPI_SUCCESS);
            RMA_CHECK(MPI_Win_unlock(0, w.win) == MPI_SUCCESS);
        }
        MPI_Barrier(MPI_COMM_WORLD);
    }

    // ---- 4b. exclusive writers, shared readers: the two words of the pair
    // are written by two puts with a flush between them, and a reader never
    // sees them differ
    {
        const int rounds = 12;
        Buffer pair(16, s.deviceBuffers);
        RMA_CHECK(pair.ok());
        for (int k = 0; k < rounds; k++) {
            if ((k + rank) % 2 == 0) {
                store64(io, 0, 1 + rank * 1000 + k);
                RMA_CHECK(MPI_Win_lock(MPI_LOCK_EXCLUSIVE, 0, 0, w.win) == MPI_SUCCESS);
                RMA_CHECK(MPI_Put(io.ptr(), 1, MPI_INT64_T, 0, PAIR_OFF, 1, MPI_INT64_T, w.win) == MPI_SUCCESS);
                RMA_CHECK(MPI_Win_flush(0, w.win) == MPI_SUCCESS);
                RMA_CHECK(MPI_Put(io.ptr(), 1, MPI_INT64_T, 0, PAIR_OFF + 8, 1, MPI_INT64_T, w.win) == MPI_SUCCESS);
                RMA_CHECK(MPI_Win_unlock(0, w.win) == MPI_SUCCESS);
            } else {
                RMA_CHECK(MPI_Win_lock(MPI_LOCK_SHARED, 0, 0, w.win) == MPI_SUCCESS);
                RMA_CHECK(MPI_Get(pair.ptr(), 2, MPI_INT64_T, 0, PAIR_OFF, 2, MPI_INT64_T, w.win) == MPI_SUCCESS);
                RMA_CHECK(MPI_Win_unlock(0, w.win) == MPI_SUCCESS);
                RMA_CHECK(load64(pair, 0) == load64(pair, 8));
            }
        }
        MPI_Barrier(MPI_COMM_WORLD);
    }

    // ---- 5. MPI_MODE_NOCHECK, flush_local, flush_all, flush_local_all and
    // unlock_all
    {
        const int right = (rank + 1) % size;
        Buffer val(8, s.deviceBuffers), got(8 * size, s.deviceBuffers);
        RMA_CHECK(val.ok() && got.ok());
        store64(val, 0, 5);
        RMA_CHECK(MPI_Win_lock(MPI_LOCK_SHARED, right, MPI_MODE_NOCHECK, w.win) == MPI_SUCCESS);
        RMA_CHECK(MPI_Accumulate(val.ptr(), 1, MPI_INT64_T, right, NOCHECK_OFF + 8 * rank, 1, MPI_INT64_T, MPI_SUM, w.win) == MPI_SUCCESS);
        RMA_CHECK(MPI_Win_flush_local(right, w.win) == MPI_SUCCESS);
        RMA_CHECK(MPI_Fetch_and_op(nullptr, got.ptr(), MPI_INT64_T, right, NOCHECK_OFF + 8 * rank, MPI_NO_OP, w.win) == MPI_SUCCESS);
        RMA_CHECK(MPI_Win_flush(right, w.win) == MPI_SUCCESS);
        RMA_CHECK(load64(got, 0) == 5);
        RMA_CHECK(MPI_Win_unlock(right, w.win) == MPI_SUCCESS);

        store64(val, 0, 7);
        RMA_CHECK(MPI_Win_lock_all(MPI_MODE_NOPRECEDE, w.win) == MPI_SUCCESS);
        for (int t = 0; t < size; t++) {
            RMA_CHECK(MPI_Accumulate(val.ptr(), 1, MPI_INT64_T, t, ALL_OFF + 8 * rank, 1, MPI_INT64_T, MPI_SUM, w.win) == MPI_SUCCESS);
        }
        RMA_CHECK(MPI_Win_flush_all(w.win) == MPI_SUCCESS);
        for (int t = 0; t < size; t++) {
            RMA_CHECK(MPI_Get_accumulate(nullptr, 0, MPI_INT64_T, got.ptr() + 8 * t, 1, MPI_INT64_T, t, ALL_OFF + 8 * rank, 1, MPI_INT64_T, MPI_NO_OP, w.win) == MPI_SUCCESS);
        }
        RMA_CHECK(MPI_Win_flush_local_all(w.win) == MPI_SUCCESS);
        for (int t = 0; t < size; t++) {
            RMA_CHECK(load64(got, 8 * t) == 7);
        }
        RMA_CHECK(MPI_Win_unlock_all(w.win) == MPI_SUCCESS);
        MPI_Barrier(MPI_COMM_WORLD);
        const auto mine = w.read(ALL_OFF, 8 * size);
        for (int r = 0; r < size; r++) {
            int64_t v;
            memcpy(&v, mine.data() + 8 * r, 8);
            RMA_CHECK(v == 7);
        }
        int64_t left;
        memcpy(&left, w.read(NOCHECK_OFF + 8 * ((rank + size - 1) % size), 8).data(), 8);
        RMA_CHECK(left == 5);
    }

    // ---- 5b. MPI_Win_sync orders loads and stores through the pointers of an
    // MPI_Win_allocate_shared segment (one address space only)
    {
        int64_t* mem = nullptr;
        MPI_Win shared = nullptr;
        const bool oneProcess = faabric::mpi::getMpiWorldRegistry().getWorld(worldId).allRanksLocal();
        int rc = MPI_Win_allocate_shared(8, 8, MPI_INFO_NULL, MPI_COMM_WORLD, &mem, &shared);
        RMA_CHECK((rc == MPI_SUCCESS) == oneProcess);
        if (rc == MPI_SUCCESS) {
            const int right = (rank + 1) % size;
            MPI_Aint bytes = 0;
            int unit = 0;
            int64_t* theirs = nullptr;
            RMA_CHECK(MPI_Win_shared_query(shared, right, &bytes, &unit, &theirs) == MPI_SUCCESS);
            RMA_CHECK(MPI_Win_lock_all(MPI_MODE_NOCHECK, shared) == MPI_SUCCESS);
            *(volatile int64_t*)mem = 77 + rank;
            RMA_CHECK(MPI_Win_sync(shared) == MPI_SUCCESS);
            MPI_Barrier(MPI_COMM_WORLD);
            RMA_CHECK(MPI_Win_sync(shared) == MPI_SUCCESS);
            RMA_CHECK(*(volatile int64_t*)theirs == 77 + right);
            RMA_CHECK(MPI_Win_unlock_all(shared) == MPI_SUCCESS);
            RMA_CHECK(MPI_Win_free(&shared) == MPI_SUCCESS);
        }
    }

    // ---- 6. synchronisation errors change nothing; a fence epoch still
    // works afterwards
    {
        MPI_Barrier(MPI_COMM_WORLD);
        const auto snapshot = w.read(0, rma_atomics::WINDOW_BYTES);
        MPI_Barrier(MPI_COMM_WORLD);
        const int t = (rank + 1) % size;
        // no epoch
        RMA_CHECK(MPI_Win_unlock(t, w.win) == MPI_ERR_RMA_SYNC);
        RMA_CHECK(MPI_Win_flush(t, w.win) == MPI_ERR_RMA_SYNC);
        RMA_CHECK(MPI_Win_flush_local(t, w.win) == MPI_ERR_RMA_SYNC);
        RMA_CHECK(MPI_Win_flush_all(w.win) == MPI_ERR_RMA_SYNC);
        RMA_CHECK(MPI_Win_flush_local_all(w.win) == MPI_ERR_RMA_SYNC);
        RMA_CHECK(MPI_Win_unlock_all(w.win) == MPI_ERR_RMA_SYNC);
        // arguments
        RMA_CHECK(MPI_Win_lock(MPI_LOCK_SHARED, size, 0, w.win) == MPI_ERR_RANK);
        RMA_CHECK(MPI_Win_lock(MPI_LOCK_SHARED, -1, 0, w.win) == MPI_ERR_RANK);
        RMA_CHECK(MPI_Win_unlock(size, w.win) == MPI_ERR_RANK);
        RMA_CHECK(MPI_Win_flush(size, w.win) == MPI_ERR_RANK);
        RMA_CHECK(MPI_Win_flush_local(-3, w.win) == MPI_ERR_RANK);
        RMA_CHECK(MPI_Win_lock(999, t, 0, w.win) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Win_lock(MPI_LOCK_SHARED, t, 0, nullptr) == MPI_ERR_WIN);
        // inside a lock epoch
        RMA_CHECK(MPI_Win_lock(MPI_LOCK_SHARED, t, 0, w.win) == MPI_SUCCESS);
        RMA_CHECK(MPI_Win_lock(MPI_LOCK_SHARED, t, 0, w.win) == MPI_ERR_RMA_SYNC);
        RMA_CHECK(MPI_Win_lock(MPI_LOCK_EXCLUSIVE, t, 0, w.win) == MPI_ERR_RMA_SYNC);
        RMA_CHECK(MPI_Win_lock_all(0, w.win) == MPI_ERR_RMA_SYNC);
        RMA_CHECK(MPI_Win_unlock_all(w.win) == MPI_ERR_RMA_SYNC);
        RMA_CHECK(MPI_Win_fence(0, w.win) == MPI_ERR_RMA_SYNC);
        MPI_Win keep = w.win;
        RMA_CHECK(MPI_Win_free(&w.win) == MPI_ERR_RMA_SYNC);
        RMA_CHECK(w.win == keep);
        if (size > 2) {
            RMA_CHECK(MPI_Win_unlock((t + 1) % size, w.win) == MPI_ERR_RMA_SYNC);
        }
        RMA_CHECK(MPI_Win_unlock(t, w.win) == MPI_SUCCESS);
        // inside a lock-all epoch
        RMA_CHECK(MPI_Win_lock_all(0, w.win) == MPI_SUCCESS);
        RMA_CHECK(MPI_Win_lock_all(0, w.win) == MPI_ERR_RMA_SYNC);
        RMA_CHECK(MPI_Win_lock(MPI_LOCK_SHARED, t, 0, w.win) == MPI_ERR_RMA_SYNC);
        RMA_CHECK(MPI_Win_unlock(t, w.win) == MPI_ERR_RMA_SYNC);
        RMA_CHECK(MPI_Win_fence(0, w.win) == MPI_ERR_RMA_SYNC);
        RMA_CHECK(MPI_Win_free(&w.win) == MPI_ERR_RMA_SYNC);
        RMA_CHECK(MPI_Win_unlock_all(w.win) == MPI_SUCCESS);
        MPI_Barrier(MPI_COMM_WORLD);
        RMA_CHECK(w.read(0, rma_atomics::WINDOW_BYTES) == snapshot);
        MPI_Barrier(MPI_COMM_WORLD);

        // a fence epoch after all this
        store64(io, 0, 500 + rank);
        RMA_CHECK(MPI_Win_fence(0, w.win) == MPI_SUCCESS);
        RMA_CHECK(MPI_Put(io.ptr(), 1, MPI_INT64_T, t, FENCE_OFF + 8 * rank, 1, MPI_INT64_T, w.win) == MPI_SUCCESS);
        RMA_CHECK(MPI_Win_fence(0, w.win) == MPI_SUCCESS);
        const int left = (rank + size - 1) % size;
        int64_t v;
        memcpy(&v, w.read(FENCE_OFF + 8 * left, 8).data(), 8);
        RMA_CHECK(v == 500 + left);
    }

    MPI_Barrier(MPI_COMM_WORLD);
    w.destroy();
    return 0;
}

} // namespace rma_passive
