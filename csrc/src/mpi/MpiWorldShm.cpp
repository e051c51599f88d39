// Host collectives for worlds whose ranks all live in this process: ranks
// publish their buffer pointers, meet at a barrier and work directly on each
// other's user buffers (slice-parallel fused reductions, straight copies).
#include <faabric/mpi/MpiWorld.h>
#include <faabric/util/config.h>
#include <faabric/util/logging.h>
#include <faabric/util/reduce_ops.h>

#include <algorithm>
#include <chrono>
#include <cstring>
#include <stdexcept>
#include <thread>

#include <linux/futex.h>
#include <sys/syscall.h>
#include <unistd.h>

namespace faabric::mpi {

namespace {
long futexCall(std::atomic<uint32_t>* addr, int op, uint32_t val, const timespec* timeout)
{
    return ::syscall(SYS_futex, reinterpret_cast<uint32_t*>(addr), op, val, timeout, nullptr, 0);
}
}

// Sense-reversing barrier.  Waiters poll for a few microseconds when every rank
// can have a core of its own, then park on a futex: a spinning waiter on an
// oversubscribed machine only steals time from the rank everybody waits for.
void MpiWorld::HostCollective::barrier(int timeoutMs)
{
    const uint32_t gen = generation.load(std::memory_order_acquire);
    if (arrived.fetch_add(1, std::memory_order_acq_rel) + 1 == nRanks) {
        arrived.store(0, std::memory_order_relaxed);
        generation.fetch_add(1, std::memory_order_seq_cst);
        if (sleepers.load(std::memory_order_seq_cst) > 0) {
            futexCall(&generation, FUTEX_WAKE_PRIVATE, INT32_MAX, nullptr);
        }
        return;
    }
    auto start = std::chrono::steady_clock::now();
    // Phase 1: poll, handing the core over between bursts (`spinIterations`
    // is the polling budget in microseconds)
    while (true) {
        for (int i = 0; i < 64; i++) {
            if (generation.load(std::memory_order_acquire) != gen) {
                return;
            }
            __builtin_ia32_pause();
        }
        if (std::chrono::steady_clock::now() - start > std::chrono::microseconds(spinIterations)) {
            break;
        }
        std::this_thread::yield();
    }
    // Phase 2: park
    while (generation.load(std::memory_order_acquire) == gen) {
        sleepers.fetch_add(1, std::memory_order_seq_cst);
        // Re-checked by the kernel: returns at once if the generation moved on
        timespec slice{ 0, 50 * 1000 * 1000 };
        futexCall(&generation, FUTEX_WAIT_PRIVATE, gen, &slice);
        sleepers.fetch_sub(1, std::memory_order_seq_cst);
        if (generation.load(std::memory_order_acquire) != gen) {
            break;
        }
        if (std::chrono::steady_clock::now() - start > std::chrono::milliseconds(timeoutMs)) {
            throw std::runtime_error("Timed out in shared-memory MPI barrier (a rank is missing)");
        }
    }
}

namespace {
// One pass over up to 16 sources: every element is read once per source and
// written once (a chain of pairwise reductions would re-read and re-write the
// destination for every source)
template<typename T, typename F>
void fusedReduceLoop(const T* const* srcs, int nSrc, T* dst, size_t count, F f)
{
    // Blocked so the sources stream through cache together
    constexpr size_t BLOCK = 2048;
    for (size_t b = 0; b < count; b += BLOCK) {
        const size_t e = std::min(count, b + BLOCK);
        const T* first = srcs[0];
        if (first != dst) {
            memcpy(dst + b, first + b, (e - b) * sizeof(T));
        }
        for (int s = 1; s < nSrc; s++) {
            const T* src = srcs[s];
            // element i only depends on element i: safe to vectorise
#pragma GCC ivdep
            for (size_t i = b; i < e; i++) {
                dst[i] = f(dst[i], src[i]);
            }
        }
    }
}

template<typename T>
bool fusedReduceTyped(int opId, const uint8_t* const* srcs, int nSrc, uint8_t* dst, size_t count)
{
    const T* typed[16];
    for (int s = 0; s < nSrc; s++) {
        typed[s] = reinterpret_cast<const T*>(srcs[s]);
    }
    T* out = reinterpret_cast<T*>(dst);
    // same element semantics as op_reduce (faabric/util/reduce_ops.h)
    switch (opId) {
        case FAABRIC_OP_SUM:
            fusedReduceLoop<T>(typed, nSrc, out, count, [](T a, T b) { return faabric::util::reduceSum(a, b); });
            return true;
        case FAABRIC_OP_PROD:
            fusedReduceLoop<T>(typed, nSrc, out, count, [](T a, T b) { return faabric::util::reduceProd(a, b); });
            return true;
        case FAABRIC_OP_MAX:
            fusedReduceLoop<T>(typed, nSrc, out, count, [](T a, T b) { return faabric::util::reduceMax(a, b); });
            return true;
        case FAABRIC_OP_MIN:
            fusedReduceLoop<T>(typed, nSrc, out, count, [](T a, T b) { return faabric::util::reduceMin(a, b); });
            return true;
        default:
            return false;
    }
}

// dst may alias srcs[0] (in-place); no other aliasing
bool fusedReduce(faabric_datatype_t* dt, int opId, const uint8_t* const* srcs, int nSrc, uint8_t* dst, size_t count)
{
    if (nSrc > 16) {
        return false;
    }
    switch (dt->id) {
        case FAABRIC_INT32:
        case FAABRIC_INT:
            return fusedReduceTyped<int32_t>(opId, srcs, nSrc, dst, count);
        case FAABRIC_UINT32:
        case FAABRIC_UINT:
            return fusedReduceTyped<uint32_t>(opId, srcs, nSrc, dst, count);
        case FAABRIC_INT64:
        case FAABRIC_LONG:
        case FAABRIC_LONG_LONG:
        case FAABRIC_LONG_LONG_INT:
            return fusedReduceTyped<int64_t>(opId, srcs, nSrc, dst, count);
        case FAABRIC_UINT64:
            return fusedReduceTyped<uint64_t>(opId, srcs, nSrc, dst, count);
        case FAABRIC_FLOAT:
            return fusedReduceTyped<float>(opId, srcs, nSrc, dst, count);
        case FAABRIC_DOUBLE:
            return fusedReduceTyped<double>(opId, srcs, nSrc, dst, count);
        default:
            return false;
    }
}
}

// Shared-memory variants of the other collectives (all ranks in this process,
// host buffers, >= 32 KiB): publish pointers, barrier, copy / reduce straight
// between the user buffers, barrier.
void MpiWorld::sharedBroadcast(int root, int rank, uint8_t* buffer, size_t bytes)
{
    HostCollective* hc = hostCollective.get();
    const int timeoutMs = faabric::util::getSystemConfig().globalMessageTimeout;
    hc->sendPtrs[rank] = buffer;
    hc->barrier(timeoutMs);
    if (rank != root) {
        memcpy(buffer, hc->sendPtrs[root], bytes);
    }
    hc->barrier(timeoutMs);
}

void MpiWorld::sharedAllGather(int rank, const uint8_t* sendBuffer, uint8_t* recvBuffer, size_t sendBytes)
{
    HostCollective* hc = hostCollective.get();
    const int timeoutMs = faabric::util::getSystemConfig().globalMessageTimeout;
    const int n = hc->nRanks;
    hc->sendPtrs[rank] = sendBuffer;
    hc->barrier(timeoutMs);
    for (int q = 0; q < n; q++) {
        int p = (rank + q) % n;
        uint8_t* dst = recvBuffer + (size_t)p * sendBytes;
        if (dst != hc->sendPtrs[p]) {
            memcpy(dst, hc->sendPtrs[p], sendBytes);
        }
    }
    hc->barrier(timeoutMs);
}

void MpiWorld::sharedAllToAll(int rank, const uint8_t* sendBuffer, uint8_t* recvBuffer, size_t chunkBytes)
{
    HostCollective* hc = hostCollective.get();
    const int timeoutMs = faabric::util::getSystemConfig().globalMessageTimeout;
    const int n = hc->nRanks;
    hc->sendPtrs[rank] = sendBuffer;
    hc->barrier(timeoutMs);
    for (int q = 0; q < n; q++) {
        int p = (rank + q) % n;
        memcpy(recvBuffer + (size_t)p * chunkBytes, hc->sendPtrs[p] + (size_t)rank * chunkBytes, chunkBytes);
    }
    hc->barrier(timeoutMs);
}

void MpiWorld::sharedGather(int rank, int root, const uint8_t* sendBuffer, uint8_t* recvBuffer, size_t sendBytes, bool rootInPlace)
{
    HostCollective* hc = hostCollective.get();
    const int timeoutMs = faabric::util::getSystemConfig().globalMessageTimeout;
    hc->sendPtrs[rank] = sendBuffer;
    hc->barrier(timeoutMs);
    if (rank == root) {
        for (int p = 0; p < hc->nRanks; p++) {
            uint8_t* dst = recvBuffer + (size_t)p * sendBytes;
            // (in place: the root passes the receive buffer itself and its
            // chunk already sits in its slot)
            if (!(p == root && rootInPlace) && dst != hc->sendPtrs[p]) {
                memcpy(dst, hc->sendPtrs[p], sendBytes);
            }
        }
    }
    hc->barrier(timeoutMs);
}

void MpiWorld::sharedScatter(int rank, int root, const uint8_t* sendBuffer, uint8_t* recvBuffer, size_t chunkBytes)
{
    HostCollective* hc = hostCollective.get();
    const int timeoutMs = faabric::util::getSystemConfig().globalMessageTimeout;
    if (rank == root) {
        hc->sendPtrs[root] = sendBuffer;
    }
    hc->barrier(timeoutMs);
    const uint8_t* mine = hc->sendPtrs[root] + (size_t)rank * chunkBytes;
    if (recvBuffer != nullptr && recvBuffer != mine) {
        memcpy(recvBuffer, mine, chunkBytes);
    }
    hc->barrier(timeoutMs);
}

void MpiWorld::sharedReduce(int rank,
                            int root,
                            uint8_t* sendBuffer,
                            uint8_t* recvBuffer,
                            faabric_datatype_t* datatype,
                            int count,
                            faabric_op_t* operation)
{
    HostCollective* hc = hostCollective.get();
    const int timeoutMs = faabric::util::getSystemConfig().globalMessageTimeout;
    const int n = hc->nRanks;
    const size_t esize = (size_t)datatype->size;
    hc->sendPtrs[rank] = sendBuffer;
    hc->recvPtrs[rank] = recvBuffer;
    hc->barrier(timeoutMs);
    // Every rank folds its slice of all inputs into the ROOT's output
    const size_t per = ((size_t)count + n - 1) / n;
    const size_t beg = std::min((size_t)rank * per, (size_t)count);
    const size_t len = std::min(per, (size_t)count - beg);
    if (len > 0) {
        uint8_t* dst = hc->recvPtrs[root] + beg * esize;
        // The root's own input first: its output may alias it (MPI_IN_PLACE)
        const uint8_t* srcs[16];
        bool fused = n <= 16;
        if (fused) {
            srcs[0] = hc->sendPtrs[root] + beg * esize;
            int k = 1;
            for (int q = 0; q < n; q++) {
                if (q != root) {
                    srcs[k++] = hc->sendPtrs[q] + beg * esize;
                }
            }
            fused = fusedReduce(datatype, operation->id, srcs, n, dst, len);
        }
        if (!fused) {
            if (dst != hc->sendPtrs[root] + beg * esize) {
                memcpy(dst, hc->sendPtrs[root] + beg * esize, len * esize);
            }
            for (int q = 0; q < n; q++) {
                if (q != root) {
                    op_reduce(operation, datatype, (int)len, const_cast<uint8_t*>(hc->sendPtrs[q]) + beg * esize, dst);
                }
            }
        }
    }
    hc->barrier(timeoutMs);
}

bool MpiWorld::trySharedMemoryAllReduce(int rank,
                                        uint8_t* sendBuffer,
                                        uint8_t* recvBuffer,
                                        faabric_datatype_t* datatype,
                                        int count,
                                        faabric_op_t* operation)
{
    HostCollective* hc = hostCollective.get();
    // Small messages are latency-bound: the message path is as good
    const size_t esize = (size_t)datatype->size;
    if (hc == nullptr || (size_t)count * esize < 32 * 1024 || isOrderedUserOp(operation)) {
        return false;
    }
    const int timeoutMs = faabric::util::getSystemConfig().globalMessageTimeout;
    const int n = hc->nRanks;
    hc->sendPtrs[rank] = sendBuffer;
    hc->recvPtrs[rank] = recvBuffer;
    hc->barrier(timeoutMs);

    // Reduce-scatter: this rank owns slice `rank` and folds everybody's copy
    // of it into its own receive buffer
    const size_t per = ((size_t)count + n - 1) / n;
    auto sliceOf = [&](int r, size_t& beg, size_t& len) {
        beg = std::min((size_t)r * per, (size_t)count);
        len = std::min(per, (size_t)count - beg);
    };
    size_t beg, len;
    sliceOf(rank, beg, len);
    if (len > 0) {
        uint8_t* dst = recvBuffer + beg * esize;
        // Own copy first (the destination may alias it), then the peers
        // starting at the right-hand neighbour to spread the memory traffic
        const uint8_t* srcs[16];
        bool fused = n <= 16;
        if (fused) {
            srcs[0] = sendBuffer + beg * esize;
            for (int q = 1; q < n; q++) {
                srcs[q] = hc->sendPtrs[(rank + q) % n] + beg * esize;
            }
            fused = fusedReduce(datatype, operation->id, srcs, n, dst, len);
        }
        if (!fused) {
            if (recvBuffer != sendBuffer) {
                memcpy(dst, sendBuffer + beg * esize, len * esize);
            }
            for (int q = 1; q < n; q++) {
                int p = (rank + q) % n;
                op_reduce(operation, datatype, (int)len, const_cast<uint8_t*>(hc->sendPtrs[p]) + beg * esize, dst);
            }
        }
    }
    hc->barrier(timeoutMs);

    // All-gather: fetch the other owners' finished slices
    for (int q = 1; q < n; q++) {
        int p = (rank + q) % n;
        sliceOf(p, beg, len);
        if (len > 0) {
            memcpy(recvBuffer + beg * esize, hc->recvPtrs[p] + beg * esize, len * esize);
        }
    }
    // Nobody may reuse its buffers while others still read them
    hc->barrier(timeoutMs);
    return true;
}
}
