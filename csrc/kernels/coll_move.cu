// Type-agnostic data-movement collectives over peer-mapped memory:
// allGather / allToAll / gather / scatter / broadcast (pull: every rank loads
// its peers' symmetric send buffers straight into a local output) plus the
// two-step large-message broadcast, the cross-rank barrier, and the
// device-side point-to-point mailbox (eager slots + put-with-signal).
//
// Reference algorithms replaced: MpiWorld::{broadcast,scatter,gather,allGather,
// allToAll,barrier,send,recv} message loops (src/mpi/MpiWorld.cpp:590-1111,
// 1433-1485,1753-1775).
#include "coll_group.cuh"
#include "coll_move.cuh"

namespace fb {

// ----------------------------------------------------------------------------
// Generic copy helpers
// ----------------------------------------------------------------------------
template<int W>
struct Word;
template<>
struct Word<16>
{
    using type = Vec16;
    __device__ __forceinline__ static Vec16 ld(const uint8_t* p)
    {
        return ldVecStream(p);
    }
    __device__ __forceinline__ static void st(uint8_t* p, const Vec16& v)
    {
        stVec(p, v);
    }
};
template<>
struct Word<4>
{
    using type = uint32_t;
    __device__ __forceinline__ static uint32_t ld(const uint8_t* p)
    {
        return *reinterpret_cast<const volatile uint32_t*>(p);
    }
    __device__ __forceinline__ static void st(uint8_t* p, uint32_t v)
    {
        *reinterpret_cast<volatile uint32_t*>(p) = v;
    }
};
template<>
struct Word<1>
{
    using type = uint8_t;
    __device__ __forceinline__ static uint8_t ld(const uint8_t* p)
    {
        return *reinterpret_cast<const volatile uint8_t*>(p);
    }
    __device__ __forceinline__ static void st(uint8_t* p, uint8_t v)
    {
        *reinterpret_cast<volatile uint8_t*>(p) = v;
    }
};

// Grid-strided copy of `bytes` (multiple of W) with 4 words in flight/thread
template<int W>
__device__ __forceinline__ void gridCopy(uint8_t* dst,
                                         const uint8_t* src,
                                         uint64_t bytes,
                                         uint64_t tid,
                                         uint64_t nthreads)
{
    using WT = typename Word<W>::type;
    const uint64_t n = bytes / W;
    uint64_t i = tid;
    constexpr int U = 8;
    for (; i + (U - 1) * nthreads < n; i += U * nthreads) {
        WT v[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            v[u] = Word<W>::ld(src + (i + u * nthreads) * W);
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            Word<W>::st(dst + (i + u * nthreads) * W, v[u]);
        }
    }
    for (; i < n; i += nthreads) {
        Word<W>::st(dst + i * W, Word<W>::ld(src + i * W));
    }
}

// ----------------------------------------------------------------------------
// Pull-style collectives
// ----------------------------------------------------------------------------
template<int W, int NR>
__global__ void __launch_bounds__(512, 1) moveKernel(const MoveArgs a)
{
    using WT = typename Word<W>::type;
    BlockBarrier bar;
    bar.load(a.comm);
    bool ok = true;
    if (!a.noSync) {
        ok = bar.sync(a.comm);
    }
    const int rank = a.comm.rank;
    const int n = a.comm.nranks;
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t nthreads = (uint64_t)gridDim.x * blockDim.x;

    if (ok) {
        if (a.mode == MOVE_ALLGATHER || a.mode == MOVE_ALLTOALL ||
            (a.mode == MOVE_GATHER && rank == a.root)) {
            const uint64_t srcExtra =
              (a.mode == MOVE_ALLTOALL) ? (uint64_t)rank * a.srcStride : 0;
            const uint64_t words = a.chunkBytes / W;
            if constexpr (NR > 0) {
                // NR x U words in flight per thread (NVLink latency ~2-3 us:
                // bandwidth needs ~16 outstanding 16-byte loads per thread)
                constexpr int U = (NR <= 2) ? 8 : ((NR <= 4) ? 4 : 2);
                uint64_t i = tid;
                for (; i + (U - 1) * nthreads < words; i += U * nthreads) {
                    WT v[U][NR];
#pragma unroll
                    for (int u = 0; u < U; u++) {
#pragma unroll
                        for (int p = 0; p < NR; p++) {
                            v[u][p] =
                              Word<W>::ld(a.comm.heap[p] + a.sendOff + srcExtra +
                                          (i + u * nthreads) * W);
                        }
                    }
#pragma unroll
                    for (int u = 0; u < U; u++) {
#pragma unroll
                        for (int p = 0; p < NR; p++) {
                            Word<W>::st(a.recvLocal +
                                          (uint64_t)p * a.dstStride +
                                          (i + u * nthreads) * W,
                                        v[u][p]);
                        }
                    }
                }
                for (; i < words; i += nthreads) {
                    WT v[NR];
#pragma unroll
                    for (int p = 0; p < NR; p++) {
                        v[p] = Word<W>::ld(a.comm.heap[p] + a.sendOff +
                                           srcExtra + i * W);
                    }
#pragma unroll
                    for (int p = 0; p < NR; p++) {
                        Word<W>::st(a.recvLocal + (uint64_t)p * a.dstStride +
                                      i * W,
                                    v[p]);
                    }
                }
            } else {
                for (int q = 0; q < n; q++) {
                    // start at own rank to spread the load over the peers
                    int p = (rank + q) % n;
                    gridCopy<W>(a.recvLocal + (uint64_t)p * a.dstStride,
                                a.comm.heap[p] + a.sendOff + srcExtra,
                                a.chunkBytes,
                                tid,
                                nthreads);
                }
            }
        } else if (a.mode == MOVE_SCATTER) {
            gridCopy<W>(a.recvLocal,
                        a.comm.heap[a.root] + a.sendOff +
                          (uint64_t)rank * a.srcStride,
                        a.chunkBytes,
                        tid,
                        nthreads);
        } else if (a.mode == MOVE_BCAST) {
            if (rank != a.root) {
                gridCopy<W>(a.recvLocal,
                            a.comm.heap[a.root] + a.sendOff,
                            a.chunkBytes,
                            tid,
                            nthreads);
            }
        } else if (a.mode == MOVE_BCAST_2STEP) {
            // Step 1: rank r pulls slice r from the root into its symmetric
            // buffer (root egress = (N-1)/N * S instead of (N-1) * S)
            const uint64_t total = a.chunkBytes;
            uint64_t slice = ((total / n) + 15) & ~(uint64_t)15;
            uint64_t myBeg = min((uint64_t)rank * slice, total);
            uint64_t myEnd = (rank == n - 1) ? total
                                             : min(myBeg + slice, total);
            if (rank != a.root && myEnd > myBeg) {
                // W divides (myEnd - myBeg) for every slice but possibly the
                // last; the host guarantees total % W == 0
                gridCopy<W>(a.comm.heap[rank] + a.recvOff + myBeg,
                            a.comm.heap[a.root] + a.sendOff + myBeg,
                            myEnd - myBeg,
                            tid,
                            nthreads);
            }
            ok = a.noSync ? true : bar.sync(a.comm);
            // Step 2: pull every other slice from its owner
            if (ok && rank != a.root) {
                for (int q = 1; q < n; q++) {
                    int p = (rank + q) % n;
                    uint64_t b = min((uint64_t)p * slice, total);
                    uint64_t e =
                      (p == n - 1) ? total : min(b + slice, total);
                    if (e <= b) {
                        continue;
                    }
                    const uint8_t* src = (p == a.root)
                                           ? a.comm.heap[p] + a.sendOff + b
                                           : a.comm.heap[p] + a.recvOff + b;
                    gridCopy<W>(a.comm.heap[rank] + a.recvOff + b,
                                src,
                                e - b,
                                tid,
                                nthreads);
                }
            }
        }
    }
    if (!a.noSync) {
        bar.sync(a.comm);
    }
    bar.store(a.comm);
}

template<int W>
static cudaError_t launchMoveW(const MoveArgs& a,
                               int blocks,
                               int threads,
                               cudaStream_t s)
{
    int n = a.comm.nranks;
    if (n == 2) {
        moveKernel<W, 2><<<blocks, threads, 0, s>>>(a);
    } else if (n == 4) {
        moveKernel<W, 4><<<blocks, threads, 0, s>>>(a);
    } else if (n == 8) {
        moveKernel<W, 8><<<blocks, threads, 0, s>>>(a);
    } else {
        moveKernel<W, 0><<<blocks, threads, 0, s>>>(a);
    }
    return cudaGetLastError();
}

cudaError_t launchMove(const MoveArgs& a,
                       int width,
                       int blocks,
                       int threads,
                       cudaStream_t s)
{
    if (width == 16) {
        return launchMoveW<16>(a, blocks, threads, s);
    }
    if (width == 4) {
        return launchMoveW<4>(a, blocks, threads, s);
    }
    return launchMoveW<1>(a, blocks, threads, s);
}

// ----------------------------------------------------------------------------
// Grouped all-gather: one MPI_Allgather per tensor, all in ONE launch per rank
// (launch_api.h).  A push: each chunk loads this rank's vectors once and
// stores them into block `rank` of every peer's output.  Entry barrier: every
// peer's output may be overwritten.  Exit barrier: every push into this
// rank's output has landed.  In place (send == block `rank` of recv) is safe:
// only this rank ever writes that block.  Dtype-free: a byte copy.
// ----------------------------------------------------------------------------
template<int NR>
__global__ void __launch_bounds__(512, 1) groupAllGatherKernel(const GroupArgs a)
{
    extern __shared__ __align__(16) uint8_t sGroupRaw[];
    GroupSeg* sSegs = reinterpret_cast<GroupSeg*>(sGroupRaw);
    const FbCommDev& c = a.comm;
    const int n = (NR > 0) ? NR : c.nranks;
    BlockBarrier bar;
    const bool ok = groupEnter(a, sSegs, bar);

    if (ok && a.nSegs > 0) {
        constexpr int UNROLL = (NR == 8) ? 2 : (NR == 1 ? 8 : 4);
        constexpr uint32_t CHUNK = 32u * UNROLL;
        const uint32_t lane = threadIdx.x & 31;
        const uint32_t warpsPerCta = blockDim.x >> 5;
        const uint32_t warpStride = gridDim.x * warpsPerCta;
        const uint8_t* const in = c.heap[c.rank];
        int cur = 0;
        for (uint32_t ch = blockIdx.x * warpsPerCta + (threadIdx.x >> 5);
             ch < a.totalChunks;
             ch += warpStride) {
            cur = groupSegOf(sSegs, a.nSegs, cur, ch);
            const GroupSeg sg = sSegs[cur];
            const uint32_t v0 = (ch - sg.chunk0) * CHUNK;
            const uint8_t* const src = in + sg.sendOff + (uint64_t)v0 * 16;
            const uint64_t rOff = sg.recvOff + (uint64_t)v0 * 16;
            const uint32_t rem = sg.nVec - v0;
            if (rem >= CHUNK) {
                Vec16 v[UNROLL];
#pragma unroll
                for (int u = 0; u < UNROLL; u++) {
                    v[u] = ldVecStream(src + (uint64_t)(u * 32 + lane) * 16);
                }
                if constexpr (NR > 0) {
#pragma unroll
                    for (int p = 0; p < NR; p++) {
#pragma unroll
                        for (int u = 0; u < UNROLL; u++) {
                            stVec(c.heap[p] + rOff + (uint64_t)(u * 32 + lane) * 16, v[u]);
                        }
                    }
                } else {
                    for (int p = 0; p < n; p++) {
#pragma unroll
                        for (int u = 0; u < UNROLL; u++) {
                            stVec(c.heap[p] + rOff + (uint64_t)(u * 32 + lane) * 16, v[u]);
                        }
                    }
                }
            } else {
                // ragged end of a shard (or a whole small one)
#pragma unroll
                for (int u = 0; u < UNROLL; u++) {
                    const uint32_t i = (uint32_t)u * 32 + lane;
                    if (i < rem) {
                        const Vec16 v = ldVecStream(src + (uint64_t)i * 16);
                        for (int p = 0; p < n; p++) {
                            stVec(c.heap[p] + rOff + (uint64_t)i * 16, v);
                        }
                    }
                }
            }
        }
    }
    groupExit(a, bar);
}

cudaError_t launchGroupAllGather(const GroupArgs& a,
                                 int blocks,
                                 int threads,
                                 cudaStream_t s)
{
    const size_t smem = (size_t)a.nSegs * sizeof(GroupSeg);
    const int n = a.comm.nranks;
    if (n == 1) {
        groupAllGatherKernel<1><<<blocks, threads, smem, s>>>(a);
    } else if (n == 2) {
        groupAllGatherKernel<2><<<blocks, threads, smem, s>>>(a);
    } else if (n == 4) {
        groupAllGatherKernel<4><<<blocks, threads, smem, s>>>(a);
    } else if (n == 8) {
        groupAllGatherKernel<8><<<blocks, threads, smem, s>>>(a);
    } else {
        groupAllGatherKernel<0><<<blocks, threads, smem, s>>>(a);
    }
    return cudaGetLastError();
}

// ----------------------------------------------------------------------------
// Barrier
// ----------------------------------------------------------------------------
__global__ void barrierKernel(const FbCommDev c)
{
    BlockBarrier bar;
    bar.load(c);
    bar.sync(c);
    bar.store(c);
}

cudaError_t launchBarrier(const FbCommDev& c, cudaStream_t s)
{
    barrierKernel<<<1, 32, 0, s>>>(c);
    return cudaGetLastError();
}

// ----------------------------------------------------------------------------
// Point to point.
//
// send(buf -> dst):  ONE kernel copies the payload into the sender's bounce
// ring (its own symmetric heap, i.e. local HBM), and the last CTA to finish
// posts a descriptor {offset, length} plus a sequence number into the
// RECEIVER's signal pad.  The sender never waits for the receiver inside a
// kernel: slot reuse is guarded by a stream-level wait on the ack word.
//
// recv(buf <- src):  the stream waits (cuStreamWaitValue32, no SM is occupied)
// until the sequence number arrives, then ONE kernel pulls the payload from
// the sender's heap over NVLink straight into the user buffer and the last
// CTA acknowledges into the sender's pad.
//
// No kernel ever spins on a peer, so ranks that time-share a GPU, hardware
// queue aliasing or a profiler serialising kernels cannot deadlock it; the
// reference's per-(sender, receiver) FIFO (src/mpi/MpiWorld.cpp:590-784) falls
// out of the per-pair sequence numbers.
// ----------------------------------------------------------------------------
__device__ __forceinline__ bool lastBlockDone(uint32_t* counter)
{
    __shared__ int sLast;
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        uint32_t prev = atomicAdd(counter, 1u);
        sLast = (prev == gridDim.x - 1) ? 1 : 0;
        if (sLast) {
            *counter = 0; // next launch on this (stream-ordered) pair starts clean
            __threadfence();
        }
    }
    __syncthreads();
    return sLast != 0;
}

template<int W>
__global__ void __launch_bounds__(512, 1) p2pSendKernel(const P2PArgs a)
{
    const FbCommDev& c = a.comm;
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t nthreads = (uint64_t)gridDim.x * blockDim.x;
    if (a.stage) {
        uint8_t* dst = c.heap[c.rank] + a.srcOff;
        const uint64_t lenW = a.bytes - (a.bytes % W);
        gridCopy<W>(dst, a.local, lenW, tid, nthreads);
        if (tid == 0) {
            for (uint64_t b = lenW; b < a.bytes; b++) {
                dst[b] = a.local[b];
            }
        }
    }
    uint32_t* done = c.sig[c.rank] + FB_P2P_DONE_OFF + a.peer;
    if (lastBlockDone(done) && threadIdx.x == 0) {
        uint32_t* desc = reinterpret_cast<uint32_t*>(c.heap[a.peer] + a.descOff) +
                         ((uint32_t)c.rank * FB_P2P_RING + (a.seq % FB_P2P_RING)) * 4;
        stRelaxedSys(desc + 0, (uint32_t)(a.srcOff & 0xffffffffu));
        stRelaxedSys(desc + 1, (uint32_t)(a.srcOff >> 32));
        stRelaxedSys(desc + 2, (uint32_t)(a.bytes & 0xffffffffu));
        stRelaxedSys(desc + 3, (uint32_t)(a.bytes >> 32));
        // release: payload (local HBM) and descriptor are visible before seq
        stReleaseSys(c.sig[a.peer] + FB_P2P_READY_OFF + c.rank, a.seq);
    }
}

template<int W>
__global__ void __launch_bounds__(512, 1) p2pPullKernel(const P2PArgs a)
{
    const FbCommDev& c = a.comm;
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t nthreads = (uint64_t)gridDim.x * blockDim.x;
    // the stream-level wait already saw seq; the acquire orders the reads below
    const uint32_t seen = ldAcquireSys(c.sig[c.rank] + FB_P2P_READY_OFF + a.peer);
    const uint32_t* desc = reinterpret_cast<const uint32_t*>(c.heap[c.rank] + a.descOff) +
                           ((uint32_t)a.peer * FB_P2P_RING + (a.seq % FB_P2P_RING)) * 4;
    const uint64_t srcOff = (uint64_t)ldRelaxedSys(desc + 0) | ((uint64_t)ldRelaxedSys(desc + 1) << 32);
    uint64_t len = (uint64_t)ldRelaxedSys(desc + 2) | ((uint64_t)ldRelaxedSys(desc + 3) << 32);
    bool ok = (int32_t)(seen - a.seq) >= 0 && len <= a.bytes &&
              srcOff + len <= a.heapBytes;
    if (!ok) {
        // never posted (host abort released the wait) or a size mismatch
        if (tid == 0 && c.err != nullptr) {
            stRelaxedSys(c.err, FB_ERR_BAD_DESC);
        }
        len = 0;
    }
    const uint8_t* src = c.heap[a.peer] + srcOff;
    const uint64_t lenW = len - (len % W);
    gridCopy<W>(a.local, src, lenW, tid, nthreads);
    if (tid == 0) {
        for (uint64_t b = lenW; b < len; b++) {
            a.local[b] = src[b];
        }
    }
    uint32_t* done = c.sig[c.rank] + FB_P2P_DONE_OFF + FB_MAX_RANKS + a.peer;
    if (lastBlockDone(done) && threadIdx.x == 0) {
        // every CTA's loads have completed (they fed stores): the sender may
        // recycle the bounce slot / its own buffer
        stReleaseSys(c.sig[a.peer] + FB_P2P_ACK_OFF + c.rank, a.seq);
    }
}

// Fallback for drivers without stream memory operations: a one-thread spin
// (this one DOES depend on the peer's kernel making progress)
__global__ void waitWordKernel(const FbCommDev c, const uint32_t* word, uint32_t target)
{
    waitFlagGe(c, word, target, FB_ERR_FLAG_TIMEOUT);
}

// Stream-ordered barrier, signalling half: tell every peer "I am at epoch e"
__global__ void signalPeersKernel(const FbCommDev c, uint32_t wordOff, uint32_t value)
{
    if ((int)threadIdx.x < c.nranks && (int)threadIdx.x != c.rank) {
        stReleaseSys(c.sig[threadIdx.x] + wordOff + c.rank, value);
    }
}

cudaError_t launchP2PSend(const P2PArgs& a, int width, int blocks, cudaStream_t s)
{
    if (width == 16) {
        p2pSendKernel<16><<<blocks, 512, 0, s>>>(a);
    } else if (width == 4) {
        p2pSendKernel<4><<<blocks, 512, 0, s>>>(a);
    } else {
        p2pSendKernel<1><<<blocks, 512, 0, s>>>(a);
    }
    return cudaGetLastError();
}

cudaError_t launchP2PPull(const P2PArgs& a, int width, int blocks, cudaStream_t s)
{
    if (width == 16) {
        p2pPullKernel<16><<<blocks, 512, 0, s>>>(a);
    } else if (width == 4) {
        p2pPullKernel<4><<<blocks, 512, 0, s>>>(a);
    } else {
        p2pPullKernel<1><<<blocks, 512, 0, s>>>(a);
    }
    return cudaGetLastError();
}

cudaError_t launchWaitWord(const FbCommDev& c,
                           const uint32_t* word,
                           uint32_t target,
                           cudaStream_t s)
{
    waitWordKernel<<<1, 1, 0, s>>>(c, word, target);
    return cudaGetLastError();
}

cudaError_t launchSignalPeers(const FbCommDev& c,
                              uint32_t wordOff,
                              uint32_t value,
                              cudaStream_t s)
{
    signalPeersKernel<<<1, 32, 0, s>>>(c, wordOff, value);
    return cudaGetLastError();
}

// ----------------------------------------------------------------------------
// put-with-signal / wait-signal for symmetric destinations (zero staging):
// data lands directly in the peer's buffer, then a user signal word is bumped.
// ----------------------------------------------------------------------------
template<int W>
__global__ void __launch_bounds__(512, 1) putSignalKernel(const PutArgs a)
{
    const FbCommDev& c = a.comm;
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t nthreads = (uint64_t)gridDim.x * blockDim.x;
    uint64_t lenW = a.bytes - (a.bytes % W);
    gridCopy<W>(c.heap[a.peer] + a.dstOff, a.local, lenW, tid, nthreads);
    if (tid == 0) {
        for (uint64_t b = lenW; b < a.bytes; b++) {
            (c.heap[a.peer] + a.dstOff)[b] = a.local[b];
        }
    }
    // every CTA publishes its own completion; the waiter expects gridDim.x
    // increments (red.add is atomic at the destination L2)
    __syncthreads();
    if (threadIdx.x == 0) {
        fenceSys();
        uint32_t* sigp = c.sig[a.peer] + FB_SIG_USER_OFF + a.signalIdx;
        asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(sigp),
                     "r"(1u)
                     : "memory");
    }
}

__global__ void waitSignalKernel(const FbCommDev c,
                                 int signalIdx,
                                 uint32_t addTarget)
{
    // The expected value is (consumed so far + addTarget); the consumed count
    // lives next to the signal so the wait is replayable
    uint32_t* sigp = c.sig[c.rank] + FB_SIG_USER_OFF + signalIdx;
    uint32_t* consumed = sigp + FB_SIG_USER_WORDS;
    uint32_t target = *consumed + addTarget;
    waitFlagGe(c, sigp, target, FB_ERR_FLAG_TIMEOUT);
    *consumed = target;
}

cudaError_t launchPutSignal(const PutArgs& a,
                            int width,
                            int blocks,
                            cudaStream_t s)
{
    if (width == 16) {
        putSignalKernel<16><<<blocks, 512, 0, s>>>(a);
    } else if (width == 4) {
        putSignalKernel<4><<<blocks, 512, 0, s>>>(a);
    } else {
        putSignalKernel<1><<<blocks, 512, 0, s>>>(a);
    }
    return cudaGetLastError();
}

cudaError_t launchWaitSignal(const FbCommDev& c,
                             int signalIdx,
                             uint32_t count,
                             cudaStream_t s)
{
    waitSignalKernel<<<1, 1, 0, s>>>(c, signalIdx, count);
    return cudaGetLastError();
}

cudaError_t preloadMoveKernels()
{
    cudaFuncAttributes a;
    cudaError_t e = cudaSuccess;
#define FB_PRELOAD(k)                                                          \
    if (e == cudaSuccess) {                                                    \
        e = cudaFuncGetAttributes(&a, k);                                      \
    }
#define FB_PRELOAD_W(W)                                                        \
    FB_PRELOAD((moveKernel<W, 0>))                                             \
    FB_PRELOAD((moveKernel<W, 2>))                                             \
    FB_PRELOAD((moveKernel<W, 4>))                                             \
    FB_PRELOAD((moveKernel<W, 8>))                                             \
    FB_PRELOAD((p2pSendKernel<W>))                                             \
    FB_PRELOAD((p2pPullKernel<W>))                                             \
    FB_PRELOAD((putSignalKernel<W>))
    FB_PRELOAD_W(16)
    FB_PRELOAD_W(4)
    FB_PRELOAD_W(1)
    FB_PRELOAD((groupAllGatherKernel<0>))
    FB_PRELOAD((groupAllGatherKernel<1>))
    FB_PRELOAD((groupAllGatherKernel<2>))
    FB_PRELOAD((groupAllGatherKernel<4>))
    FB_PRELOAD((groupAllGatherKernel<8>))
    FB_PRELOAD(barrierKernel)
    FB_PRELOAD(waitSignalKernel)
    FB_PRELOAD(waitWordKernel)
    FB_PRELOAD(signalPeersKernel)
#undef FB_PRELOAD_W
#undef FB_PRELOAD
    return e;
}

} // namespace fb
