// One MPI program that checks the request-based one-sided operations
// (MPI_Rput, MPI_Rget, MPI_Raccumulate, MPI_Rget_accumulate) on one kind of
// window and origin buffer.  Run by test_mpi_rma_request.cpp.
//
// Every check is exact: 256 distinct 24-byte records per origin and target at
// odd displacements with guard bytes between them, records read back with
// only MPI_Wait, int64 counters at their exact total, unique get-accumulate
// tickets, completion by unlock of a freed or already-waited request, and
// every error code with the window unchanged.
#pragma once

#include "mpi_rma_atomics_body.h"

#include <faabric/mpi/MpiWorldRegistry.h>
#include <faabric/mpi/mpi.h>

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

namespace rma_request {

using rma_atomics::copyBytes;
using rma_atomics::WindowMemory;

// Where the origin and result buffers live
enum class Origin
{
    Host,   // malloc
    Device, // cudaMalloc
    Heap    // MPI_Alloc_mem(MPI_INFO_FAABRIC_DEVICE): the origin's own heap
};

struct Setup
{
    WindowMemory window = WindowMemory::Host;
    Origin origin = Origin::Host;
    // every target in this process and the puts and gets batched: count the
    // origin communicator's launches (one per 1024 deferred copies)
    bool countLaunches = false;
};

constexpr int RECORDS = 256;
constexpr size_t RECORD = 24;
constexpr size_t SLOT = RECORD + 1; // one guard byte after every record
constexpr size_t COUNTER_OFF = 56 << 10; // int64 on every target
constexpr size_t TICKET_OFF = COUNTER_OFF + 64; // int64 on the last rank
constexpr size_t LATE_OFF = COUNTER_OFF + 128;  // 24 bytes per origin
constexpr size_t ERROR_OFF = COUNTER_OFF + 512; // never written
constexpr size_t WIN_BYTES = 64 << 10;
constexpr uint8_t GUARD = 0xEE;

// Origin record i of origin o for target t starts at 1 + (o * RECORDS + i) *
// SLOT: odd displacements, and every byte between records is a guard byte
inline size_t recordDisp(int o, int i)
{
    return 1 + ((size_t)o * RECORDS + i) * SLOT;
}

inline uint8_t recordByte(int o, int t, int i, size_t j)
{
    return (uint8_t)rma_atomics::seedOf(o, t, i, (int)j, 7);
}

struct Buf
{
    uint8_t* p = nullptr;
    size_t n = 0;
    Origin kind;

    Buf(size_t bytes, Origin k)
      : n(bytes)
      , kind(k)
    {
        if (k == Origin::Host) {
            p = (uint8_t*)malloc(n);
        } else if (k == Origin::Device) {
            if (cudaMalloc((void**)&p, n) != cudaSuccess) {
                cudaGetLastError();
                p = nullptr;
            }
        } else if (MPI_Alloc_mem(n, MPI_INFO_FAABRIC_DEVICE, &p) != MPI_SUCCESS) {
            p = nullptr;
        }
    }
    ~Buf()
    {
        if (p == nullptr) {
            return;
        }
        if (kind == Origin::Host) {
            free(p);
        } else if (kind == Origin::Device) {
            cudaFree(p);
        } else {
            MPI_Free_mem(p);
        }
    }
    Buf(const Buf&) = delete;
    Buf& operator=(const Buf&) = delete;

    void write(const std::vector<uint8_t>& v) { copyBytes(p, v.data(), v.size()); }
    std::vector<uint8_t> read()
    {
        std::vector<uint8_t> out(n);
        copyBytes(out.data(), p, n);
        return out;
    }
};

struct Win
{
    uint8_t* base = nullptr;
    WindowMemory kind;
    MPI_Win win = nullptr;

    bool create(WindowMemory k)
    {
        kind = k;
        if (k == WindowMemory::Host) {
            void* p = nullptr;
            if (posix_memalign(&p, 64, WIN_BYTES) != 0) {
                return false;
            }
            base = (uint8_t*)p;
        } else if (k == WindowMemory::Heap) {
            if (MPI_Alloc_mem(WIN_BYTES, MPI_INFO_FAABRIC_DEVICE, &base) != MPI_SUCCESS) {
                return false;
            }
        } else if (cudaMalloc((void**)&base, WIN_BYTES) != cudaSuccess) {
            cudaGetLastError();
            return false;
        }
        fill();
        return MPI_Win_create(base, WIN_BYTES, 1, MPI_INFO_NULL, MPI_COMM_WORLD, &win) == MPI_SUCCESS;
    }
    void fill()
    {
        std::vector<uint8_t> guard(WIN_BYTES, GUARD);
        std::fill(guard.begin() + COUNTER_OFF, guard.begin() + COUNTER_OFF + 16, 0);
        std::fill(guard.begin() + TICKET_OFF, guard.begin() + TICKET_OFF + 8, 0);
        copyBytes(base, guard.data(), WIN_BYTES);
    }
    void destroy()
    {
        MPI_Win_free(&win);
        if (kind == WindowMemory::Host) {
            free(base);
        } else if (kind == WindowMemory::Heap) {
            MPI_Free_mem(base);
        } else {
            cudaFree(base);
        }
    }
    std::vector<uint8_t> read()
    {
        std::vector<uint8_t> out(WIN_BYTES);
        copyBytes(out.data(), base, WIN_BYTES);
        return out;
    }
};

inline int64_t at64(const std::vector<uint8_t>& v, size_t off)
{
    int64_t x;
    memcpy(&x, v.data() + off, 8);
    return x;
}

inline int body(int rank, int size, int worldId, const Setup& s, std::string* why)
{
    auto comm = s.countLaunches ? faabric::mpi::getMpiWorldRegistry().getWorld(worldId).getDeviceComm(rank) : nullptr;
    RMA_CHECK(!s.countLaunches || comm != nullptr);
    auto launches = [&]() { return comm != nullptr ? comm->stats().launches : 0; };
    Win w;
    RMA_CHECK(w.create(s.window));
    const size_t recBytes = (size_t)size * RECORDS * RECORD;
    Buf recs(recBytes, s.origin);  // this origin's records, target-major
    Buf back(recBytes, s.origin);  // (b): records read back
    Buf io(4096, s.origin);        // (c), (d): values and results
    RMA_CHECK(recs.p != nullptr && back.p != nullptr && io.p != nullptr);
    {
        std::vector<uint8_t> v(recBytes);
        for (int t = 0; t < size; t++) {
            for (int i = 0; i < RECORDS; i++) {
                for (size_t j = 0; j < RECORD; j++) {
                    v[((size_t)t * RECORDS + i) * RECORD + j] = recordByte(rank, t, i, j);
                }
            }
        }
        recs.write(v);
    }
    MPI_Barrier(MPI_COMM_WORLD);

    // ---- (a) MPI_Rput of every record into every target, then MPI_Waitall
    {
        std::vector<MPI_Request> reqs((size_t)size * RECORDS, nullptr);
        RMA_CHECK(MPI_Win_lock_all(0, w.win) == MPI_SUCCESS);
        const uint64_t before = launches();
        for (int t = 0; t < size; t++) {
            for (int i = 0; i < RECORDS; i++) {
                uint8_t* src = recs.p + ((size_t)t * RECORDS + i) * RECORD;
                RMA_CHECK(MPI_Rput(src, RECORD, MPI_BYTE, t, recordDisp(rank, i), RECORD, MPI_BYTE, w.win,
                                   &reqs[(size_t)t * RECORDS + i]) == MPI_SUCCESS);
            }
        }
        RMA_CHECK(MPI_Waitall((int)reqs.size(), reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        for (MPI_Request r : reqs) {
            RMA_CHECK(r == nullptr);
        }
        // one launch per 1024 deferred copies, none for the waits
        RMA_CHECK(!s.countLaunches || launches() - before == (reqs.size() + 1023) / 1024);
        RMA_CHECK(MPI_Win_unlock_all(w.win) == MPI_SUCCESS);
        MPI_Barrier(MPI_COMM_WORLD);
        const auto got = w.read();
        std::vector<uint8_t> want(WIN_BYTES);
        copyBytes(want.data(), got.data(), WIN_BYTES);
        std::fill(want.begin(), want.begin() + COUNTER_OFF, GUARD);
        for (int o = 0; o < size; o++) {
            for (int i = 0; i < RECORDS; i++) {
                for (size_t j = 0; j < RECORD; j++) {
                    want[recordDisp(o, i) + j] = recordByte(o, rank, i, j);
                }
            }
        }
        RMA_CHECK(got == want);
    }

    // ---- (b) MPI_Rget of origin (rank+1)'s records from every target, with
    // only MPI_Wait before they are read
    {
        const int o = (rank + 1) % size;
        RMA_CHECK(MPI_Win_lock_all(0, w.win) == MPI_SUCCESS);
        for (int t = 0; t < size; t++) {
            std::vector<MPI_Request> reqs(RECORDS, nullptr);
            const uint64_t before = launches();
            for (int i = 0; i < RECORDS; i++) {
                uint8_t* dst = back.p + ((size_t)t * RECORDS + i) * RECORD;
                RMA_CHECK(MPI_Rget(dst, RECORD, MPI_BYTE, t, recordDisp(o, i), RECORD, MPI_BYTE, w.win, &reqs[i]) ==
                          MPI_SUCCESS);
            }
            // deferred: nothing is launched before the first wait, and that
            // wait completes all of them in one launch
            RMA_CHECK(!s.countLaunches || launches() == before);
            for (int i = RECORDS - 1; i >= 0; i--) {
                RMA_CHECK(MPI_Wait(&reqs[i], MPI_STATUS_IGNORE) == MPI_SUCCESS);
            }
            RMA_CHECK(!s.countLaunches || launches() == before + 1);
            const auto got = back.read();
            for (int i = 0; i < RECORDS; i++) {
                for (size_t j = 0; j < RECORD; j++) {
                    RMA_CHECK(got[((size_t)t * RECORDS + i) * RECORD + j] == recordByte(o, t, i, j));
                }
            }
        }
        RMA_CHECK(MPI_Win_unlock_all(w.win) == MPI_SUCCESS);
        MPI_Barrier(MPI_COMM_WORLD);
    }

    // ---- (c) MPI_Raccumulate counters and MPI_Rget_accumulate tickets
    {
        const int K = 16;
        const int owner = size - 1;
        std::vector<uint8_t> v(io.n, 0);
        const int64_t one = 1;
        memcpy(v.data(), &one, 8);
        io.write(v);
        std::vector<MPI_Request> reqs;
        RMA_CHECK(MPI_Win_lock_all(0, w.win) == MPI_SUCCESS);
        for (int k = 0; k < K; k++) {
            for (int t = 0; t < size; t++) {
                reqs.emplace_back(nullptr);
                RMA_CHECK(MPI_Raccumulate(io.p, 1, MPI_INT64_T, t, COUNTER_OFF, 1, MPI_INT64_T, MPI_SUM, w.win,
                                          &reqs.back()) == MPI_SUCCESS);
            }
            reqs.emplace_back(nullptr);
            RMA_CHECK(MPI_Rget_accumulate(io.p, 1, MPI_INT64_T, io.p + 64 + 8 * k, 1, MPI_INT64_T, owner, TICKET_OFF, 1,
                                          MPI_INT64_T, MPI_SUM, w.win, &reqs.back()) == MPI_SUCCESS);
        }
        RMA_CHECK(MPI_Waitall((int)reqs.size(), reqs.data(), MPI_STATUSES_IGNORE) == MPI_SUCCESS);
        const auto mine = io.read();
        RMA_CHECK(MPI_Win_unlock_all(w.win) == MPI_SUCCESS);
        MPI_Barrier(MPI_COMM_WORLD);
        RMA_CHECK(at64(w.read(), COUNTER_OFF) == (int64_t)size * K);
        std::vector<int64_t> tickets(K), all((size_t)size * K);
        memcpy(tickets.data(), mine.data() + 64, 8 * K);
        MPI_Allgather(tickets.data(), K, MPI_INT64_T, all.data(), K, MPI_INT64_T, MPI_COMM_WORLD);
        std::sort(all.begin(), all.end());
        for (int i = 0; i < size * K; i++) {
            RMA_CHECK(all[i] == i);
        }
        if (rank == owner) {
            RMA_CHECK(at64(w.read(), TICKET_OFF) == (int64_t)size * K);
        }
    }

    // ---- (d) a wait after the unlock returns; a freed request completes at
    // the unlock
    {
        const int t = (rank + 1) % size;
        const size_t off = LATE_OFF + 24 * (size_t)rank;
        MPI_Request late = nullptr, freed = nullptr;
        RMA_CHECK(MPI_Win_lock(MPI_LOCK_SHARED, t, 0, w.win) == MPI_SUCCESS);
        RMA_CHECK(MPI_Rput(recs.p, 12, MPI_BYTE, t, off, 12, MPI_BYTE, w.win, &late) == MPI_SUCCESS);
        RMA_CHECK(MPI_Rput(recs.p + 12, 12, MPI_BYTE, t, off + 12, 12, MPI_BYTE, w.win, &freed) == MPI_SUCCESS);
        RMA_CHECK(MPI_Request_free(&freed) == MPI_SUCCESS && freed == nullptr);
        RMA_CHECK(MPI_Win_unlock(t, w.win) == MPI_SUCCESS);
        RMA_CHECK(MPI_Wait(&late, MPI_STATUS_IGNORE) == MPI_SUCCESS && late == nullptr);
        MPI_Barrier(MPI_COMM_WORLD);
        const int o = (rank + size - 1) % size;
        const auto got = w.read();
        for (size_t j = 0; j < 24; j++) {
            RMA_CHECK(got[LATE_OFF + 24 * (size_t)o + j] == recordByte(o, 0, 0, j));
        }
    }

    // ---- (e) every error code, with the window unchanged
    {
        const int t = (rank + 1) % size;
        MPI_Request r = nullptr;
        const auto before = w.read();
        RMA_CHECK(MPI_Rput(recs.p, 8, MPI_BYTE, t, ERROR_OFF, 8, MPI_BYTE, nullptr, &r) == MPI_ERR_WIN);
        RMA_CHECK(MPI_Rget(back.p, 8, MPI_BYTE, t, ERROR_OFF, 8, MPI_BYTE, nullptr, &r) == MPI_ERR_WIN);
        RMA_CHECK(MPI_Raccumulate(io.p, 1, MPI_INT64_T, t, ERROR_OFF, 1, MPI_INT64_T, MPI_SUM, nullptr, &r) == MPI_ERR_WIN);
        // outside any epoch
        RMA_CHECK(MPI_Rput(recs.p, 8, MPI_BYTE, t, ERROR_OFF, 8, MPI_BYTE, w.win, &r) == MPI_ERR_RMA_SYNC);
        RMA_CHECK(MPI_Rget_accumulate(io.p, 1, MPI_INT64_T, io.p + 8, 1, MPI_INT64_T, t, ERROR_OFF, 1, MPI_INT64_T, MPI_SUM,
                                      w.win, &r) == MPI_ERR_RMA_SYNC);
        RMA_CHECK(MPI_Win_lock(MPI_LOCK_SHARED, rank, 0, w.win) == MPI_SUCCESS);
        if (size > 1) {
            // an epoch that does not cover the target
            RMA_CHECK(MPI_Rget(back.p, 8, MPI_BYTE, t, ERROR_OFF, 8, MPI_BYTE, w.win, &r) == MPI_ERR_RMA_SYNC);
            RMA_CHECK(MPI_Raccumulate(io.p, 1, MPI_INT64_T, t, ERROR_OFF, 1, MPI_INT64_T, MPI_SUM, w.win, &r) ==
                      MPI_ERR_RMA_SYNC);
        }
        RMA_CHECK(MPI_Rput(recs.p, 8, MPI_BYTE, rank, ERROR_OFF, 8, MPI_BYTE, w.win, nullptr) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Rget_accumulate(io.p, 1, MPI_INT64_T, io.p + 8, 1, MPI_INT64_T, rank, ERROR_OFF, 1, MPI_INT64_T,
                                      MPI_SUM, w.win, nullptr) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Rput(recs.p, 8, MPI_BYTE, rank, ERROR_OFF, 7, MPI_BYTE, w.win, &r) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Rget(back.p, 8, MPI_BYTE, rank, WIN_BYTES - 4, 8, MPI_BYTE, w.win, &r) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Rget(back.p, 8, MPI_BYTE, rank, -1, 8, MPI_BYTE, w.win, &r) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Rput(recs.p, 8, MPI_BYTE, size, ERROR_OFF, 8, MPI_BYTE, w.win, &r) == MPI_ERR_RANK);
        RMA_CHECK(MPI_Raccumulate(io.p, 1, MPI_INT64_T, -1, ERROR_OFF, 1, MPI_INT64_T, MPI_SUM, w.win, &r) == MPI_ERR_RANK);
        // the element rules of MPI_Accumulate
        RMA_CHECK(MPI_Raccumulate(io.p, 1, MPI_INT64_T, rank, ERROR_OFF, 1, MPI_INT64_T, MPI_NO_OP, w.win, &r) ==
                  MPI_ERR_OP);
        RMA_CHECK(MPI_Raccumulate(io.p, 1, MPI_FLOAT, rank, ERROR_OFF, 1, MPI_FLOAT, MPI_BAND, w.win, &r) == MPI_ERR_OP);
        RMA_CHECK(MPI_Raccumulate(io.p, 1, MPI_INT64_T, rank, ERROR_OFF + 4, 1, MPI_INT64_T, MPI_SUM, w.win, &r) ==
                  MPI_ERR_ARG);
        RMA_CHECK(r == nullptr);
        RMA_CHECK(MPI_Win_unlock(rank, w.win) == MPI_SUCCESS);
        MPI_Barrier(MPI_COMM_WORLD);
        RMA_CHECK(w.read() == before);
    }

    MPI_Barrier(MPI_COMM_WORLD);
    w.destroy();
    return 0;
}

} // namespace rma_request
