// One fused "gather-from-peers + user-op reduce + scatter-to-peers" kernel that
// implements allReduce (one-shot and two-shot), reduce, reduceScatter and scan
// as parameterisations.  Replaces the reference's reduce-to-root-then-broadcast
// message algorithms (MpiWorld::reduce/allReduce/scan,
// src/mpi/MpiWorld.cpp:1127-1264,1390-1431) with a single launch per rank that
// reads peer HBM over NVLink and applies the op in registers.
#pragma once

#include "coll_group.cuh"
#include "fb_prims.cuh"
#include "launch_api.h"

namespace fb {

template<typename VR, int NR>
__device__ __forceinline__ Vec16 gatherReduce(const ReduceArgs& a,
                                              uint64_t byteOff)
{
    if constexpr (NR > 0) {
        Vec16 v[NR];
#pragma unroll
        for (int p = 0; p < NR; p++) {
            v[p] = ldVecStream(a.comm.heap[p] + a.sendOff + byteOff);
        }
        Vec16 acc = v[0];
#pragma unroll
        for (int p = 1; p < NR; p++) {
            acc = VR::apply(acc, v[p]);
        }
        return acc;
    } else {
        Vec16 acc = ldVecStream(a.comm.heap[0] + a.sendOff + byteOff);
        for (int p = 1; p < a.readRanks; p++) {
            Vec16 v = ldVecStream(a.comm.heap[p] + a.sendOff + byteOff);
            acc = VR::apply(acc, v);
        }
        return acc;
    }
}

template<typename VR, int NR>
__device__ __forceinline__ void emit(const ReduceArgs& a,
                                     uint64_t vecIdx,
                                     const Vec16& acc)
{
    if (a.pushMask == 0) {
        stVec(a.recvLocal + (vecIdx - a.outBase) * 16, acc);
    } else {
        uint64_t off = a.recvOff + vecIdx * 16;
        if constexpr (NR > 0) {
#pragma unroll
            for (int p = 0; p < NR; p++) {
                if (a.pushMask & (1u << p)) {
                    stVec(a.comm.heap[p] + off, acc);
                }
            }
        } else {
            for (int p = 0; p < a.comm.nranks; p++) {
                if (a.pushMask & (1u << p)) {
                    stVec(a.comm.heap[p] + off, acc);
                }
            }
        }
    }
}

template<typename VR, int NR>
__global__ void __launch_bounds__(512, 1) reduceKernel(const ReduceArgs a)
{
    BlockBarrier bar;
    bar.load(a.comm);
    bool ok = true;
    // Barrier 1: every rank's input is complete and every rank's output buffer
    // may be overwritten (all ranks have entered the collective)
    if (!a.noSync) {
        ok = bar.sync(a.comm);
    }

    if (ok) {
        constexpr int UNROLL = (NR == 0) ? 4 : ((NR <= 4) ? 4 : 2);
        const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
        uint64_t i = a.vecBegin + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
        // main loop: UNROLL independent vectors per thread in flight
        for (; i + (UNROLL - 1) * stride < a.vecEnd; i += UNROLL * stride) {
            Vec16 acc[UNROLL];
            if constexpr (NR > 0) {
                Vec16 v[UNROLL][NR];
#pragma unroll
                for (int u = 0; u < UNROLL; u++) {
#pragma unroll
                    for (int p = 0; p < NR; p++) {
                        v[u][p] = ldVecStream(a.comm.heap[p] + a.sendOff +
                                              (i + u * stride) * 16);
                    }
                }
#pragma unroll
                for (int u = 0; u < UNROLL; u++) {
                    acc[u] = v[u][0];
#pragma unroll
                    for (int p = 1; p < NR; p++) {
                        acc[u] = VR::apply(acc[u], v[u][p]);
                    }
                }
            } else {
#pragma unroll
                for (int u = 0; u < UNROLL; u++) {
                    acc[u] = ldVecStream(a.comm.heap[0] + a.sendOff +
                                         (i + u * stride) * 16);
                }
                for (int p = 1; p < a.readRanks; p++) {
                    Vec16 v[UNROLL];
#pragma unroll
                    for (int u = 0; u < UNROLL; u++) {
                        v[u] = ldVecStream(a.comm.heap[p] + a.sendOff +
                                           (i + u * stride) * 16);
                    }
#pragma unroll
                    for (int u = 0; u < UNROLL; u++) {
                        acc[u] = VR::apply(acc[u], v[u]);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < UNROLL; u++) {
                emit<VR, NR>(a, i + u * stride, acc[u]);
            }
        }
        for (; i < a.vecEnd; i += stride) {
            Vec16 acc = gatherReduce<VR, NR>(a, i * 16);
            emit<VR, NR>(a, i, acc);
        }

        // < 16-byte tail, element by element
        const uint64_t tailBytes = a.bytes & 15;
        if (tailBytes != 0 && blockIdx.x == 0 && threadIdx.x == 0 &&
            (a.tailOwner == -2 || a.tailOwner == a.comm.rank)) {
            const uint64_t base = a.bytes - tailBytes;
            constexpr int EB = VR::ELEM_BYTES;
            for (uint64_t e = 0; e + EB <= tailBytes; e += EB) {
                alignas(16) uint8_t acc[16];
                alignas(16) uint8_t in[16];
                const uint8_t* s0 = a.comm.heap[0] + a.sendOff + base + e;
                for (int b = 0; b < EB; b++) {
                    acc[b] = s0[b];
                }
                for (int p = 1; p < a.readRanks; p++) {
                    const uint8_t* sp = a.comm.heap[p] + a.sendOff + base + e;
                    for (int b = 0; b < EB; b++) {
                        in[b] = sp[b];
                    }
                    VR::applyTail(acc, in);
                }
                if (a.pushMask == 0) {
                    uint8_t* d = a.recvLocal + (base - a.outBase * 16) + e;
                    for (int b = 0; b < EB; b++) {
                        d[b] = acc[b];
                    }
                } else {
                    for (int p = 0; p < a.comm.nranks; p++) {
                        if (a.pushMask & (1u << p)) {
                            uint8_t* d = a.comm.heap[p] + a.recvOff + base + e;
                            for (int b = 0; b < EB; b++) {
                                d[b] = acc[b];
                            }
                        }
                    }
                }
            }
        }
    }

    // Barrier 2: all reads of my input are done (it may be modified again) and
    // all pushes into my output have landed (release/acquire at .sys scope)
    if (!a.noSync) {
        bar.sync(a.comm);
    }
    bar.store(a.comm);
}

template<typename VR>
cudaError_t launchReduce(const ReduceArgs& a,
                         int nr,
                         int blocks,
                         int threads,
                         cudaStream_t stream)
{
    // Full-unroll variants need to read *all* ranks
    bool full = (a.readRanks == a.comm.nranks);
    if (full && nr == 2) {
        reduceKernel<VR, 2><<<blocks, threads, 0, stream>>>(a);
    } else if (full && nr == 4) {
        reduceKernel<VR, 4><<<blocks, threads, 0, stream>>>(a);
    } else if (full && nr == 8) {
        reduceKernel<VR, 8><<<blocks, threads, 0, stream>>>(a);
    } else {
        reduceKernel<VR, 0><<<blocks, threads, 0, stream>>>(a);
    }
    return cudaGetLastError();
}

// ----------------------------------------------------------------------------
// Low-latency (LL) all-reduce for small messages: no barriers at all.
// Every rank pushes its contribution into a per-source slot area on every
// peer as {data, flag} 8-byte pairs (flag = call epoch), then spins on its own
// slots until all N contributions of this epoch have arrived and reduces them
// in rank order.  Latency = one NVLink store + poll.  Two parity buffers make
// reuse safe: a rank can only be two epochs ahead of a peer after it has
// received that peer's data for the epoch in between.  Send/recv buffers are
// arbitrary local pointers (no symmetric-heap requirement, in-place is fine).
// Fixed launch geometry (FB_LL_BLOCKS x FB_LL_THREADS, one 16-byte vector per
// thread) so a slot is always produced/consumed by the same CTA index and the
// per-CTA epoch words stay in lock step across ranks.
// ----------------------------------------------------------------------------
__device__ __forceinline__ void stVolatileV4(uint8_t* p,
                                             uint32_t a,
                                             uint32_t b,
                                             uint32_t c,
                                             uint32_t d)
{
    asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p),
                 "r"(a),
                 "r"(b),
                 "r"(c),
                 "r"(d)
                 : "memory");
}

__device__ __forceinline__ void ldVolatileV4(const uint8_t* p,
                                             uint32_t& a,
                                             uint32_t& b,
                                             uint32_t& c,
                                             uint32_t& d)
{
    asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(a), "=r"(b), "=r"(c), "=r"(d)
                 : "l"(p)
                 : "memory");
}

template<typename VR, int NR>
__global__ void __launch_bounds__(FB_LL_THREADS, 1) llAllReduceKernel(
  const LLArgs a)
{
    const FbCommDev& c = a.comm;
    const int n = (NR > 0) ? NR : c.nranks;
    uint32_t* epochWord =
      c.sig[c.rank] + FB_SIG_LL_EPOCH_OFF + c.llEpochBase + blockIdx.x;
    uint32_t epoch = *epochWord + 1;
    if (epoch == 0) {
        epoch = 1; // 0 is the "empty slot" value
    }
    const uint32_t par = epoch & 1;
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t nVec = (a.bytes + 15) / 16;

    if (i < nVec) {
        const uint64_t byteOff = i * 16;
        const uint32_t valid =
          (a.bytes - byteOff) >= 16 ? 16u : (uint32_t)(a.bytes - byteOff);
        Vec16 mine;
        if (valid == 16 && !a.byteAccess) {
            mine = ldVec(a.sendLocal + byteOff);
        } else {
            mine.w[0] = mine.w[1] = mine.w[2] = mine.w[3] = 0;
            uint8_t* mb = reinterpret_cast<uint8_t*>(&mine);
            for (uint32_t b = 0; b < valid; b++) {
                mb[b] = a.sendLocal[byteOff + b];
            }
        }
        // push to every rank (including myself: uniform code path)
        const uint64_t slotOff =
          a.llOff + (((uint64_t)par * n + c.rank) * FB_LL_MAX_VECS + i) * 32;
        if constexpr (NR > 0) {
#pragma unroll
            for (int p = 0; p < NR; p++) {
                uint8_t* d = c.heap[p] + slotOff;
                stVolatileV4(d, mine.w[0], epoch, mine.w[1], epoch);
                stVolatileV4(d + 16, mine.w[2], epoch, mine.w[3], epoch);
            }
        } else {
            for (int p = 0; p < n; p++) {
                uint8_t* d = c.heap[p] + slotOff;
                stVolatileV4(d, mine.w[0], epoch, mine.w[1], epoch);
                stVolatileV4(d + 16, mine.w[2], epoch, mine.w[3], epoch);
            }
        }
        // collect: spin on my own slots
        const uint8_t* base = c.heap[c.rank] + a.llOff +
                              ((uint64_t)par * n * FB_LL_MAX_VECS + i) * 32;
        Vec16 acc;
        bool ok = true;
        uint64_t t0 = 0;
        for (int p = 0; p < n && ok; p++) {
            const uint8_t* s = base + (uint64_t)p * FB_LL_MAX_VECS * 32;
            Vec16 v;
            uint32_t f0, f1, f2, f3;
            uint32_t spins = 0;
            while (true) {
                ldVolatileV4(s, v.w[0], f0, v.w[1], f1);
                ldVolatileV4(s + 16, v.w[2], f2, v.w[3], f3);
                if (f0 == epoch && f1 == epoch && f2 == epoch && f3 == epoch) {
                    break;
                }
                if ((++spins & 0x3ff) == 0) {
                    uint64_t now = globalTimerNs();
                    if (t0 == 0) {
                        t0 = now;
                    } else if (now - t0 > c.timeoutNs) {
                        if (c.err != nullptr) {
                            stRelaxedSys(c.err, FB_ERR_FLAG_TIMEOUT);
                        }
                        ok = false;
                        break;
                    }
                }
            }
            acc = (p == 0) ? v : VR::apply(acc, v);
        }
        if (ok) {
            if (valid == 16 && !a.byteAccess) {
                stVec(a.recvLocal + byteOff, acc);
            } else {
                const uint8_t* ab = reinterpret_cast<const uint8_t*>(&acc);
                for (uint32_t b = 0; b < valid; b++) {
                    a.recvLocal[byteOff + b] = ab[b];
                }
            }
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        *epochWord = epoch;
    }
}

template<typename VR>
cudaError_t launchLL(const LLArgs& a, cudaStream_t stream)
{
    int nr = a.comm.nranks;
    if (nr == 2) {
        llAllReduceKernel<VR, 2><<<FB_LL_BLOCKS, FB_LL_THREADS, 0, stream>>>(a);
    } else if (nr == 4) {
        llAllReduceKernel<VR, 4><<<FB_LL_BLOCKS, FB_LL_THREADS, 0, stream>>>(a);
    } else if (nr == 8) {
        llAllReduceKernel<VR, 8><<<FB_LL_BLOCKS, FB_LL_THREADS, 0, stream>>>(a);
    } else {
        llAllReduceKernel<VR, 0><<<FB_LL_BLOCKS, FB_LL_THREADS, 0, stream>>>(a);
    }
    return cudaGetLastError();
}


// ----------------------------------------------------------------------------
// Grouped all-reduce: every tensor of a group (e.g. the 214 gradient tensors of
// one training step, or an MPI_Iallreduce burst) in ONE launch per rank.
// Semantics are those of independent per-tensor all-reduces; what is shared is
// the synchronisation: two cross-rank barriers per GROUP instead of per tensor
// (the per-call latency is what bounded the reference benchmark, which issues
// 214 MPI_Allreduce calls per pass: tests/dist/mpi/benchmarks/mpi_allreduce.cpp
// :24-50).  Work is cut into warp-sized chunks of the rank's segment list so
// tiny tensors cost one warp iteration, not one kernel.
// ----------------------------------------------------------------------------
// One element at an element-aligned address, moved as an integer of its size
template<typename E>
__device__ __forceinline__ E ldElemGlobal(const uint8_t* p)
{
    E out;
    if constexpr (sizeof(E) == 1) {
        uint8_t v = *reinterpret_cast<const volatile uint8_t*>(p);
        memcpy(&out, &v, 1);
    } else if constexpr (sizeof(E) == 2) {
        uint16_t v = *reinterpret_cast<const volatile uint16_t*>(p);
        memcpy(&out, &v, 2);
    } else if constexpr (sizeof(E) == 4) {
        uint32_t v = *reinterpret_cast<const volatile uint32_t*>(p);
        memcpy(&out, &v, 4);
    } else if constexpr (sizeof(E) == 8) {
        uint64_t v = *reinterpret_cast<const volatile uint64_t*>(p);
        memcpy(&out, &v, 8);
    } else {
        Vec16 v = ldVec(p);
        memcpy(&out, &v, 16);
    }
    return out;
}

template<typename E>
__device__ __forceinline__ void stElemGlobal(uint8_t* p, const E& in)
{
    if constexpr (sizeof(E) == 1) {
        uint8_t v;
        memcpy(&v, &in, 1);
        *reinterpret_cast<volatile uint8_t*>(p) = v;
    } else if constexpr (sizeof(E) == 2) {
        uint16_t v;
        memcpy(&v, &in, 2);
        *reinterpret_cast<volatile uint16_t*>(p) = v;
    } else if constexpr (sizeof(E) == 4) {
        uint32_t v;
        memcpy(&v, &in, 4);
        *reinterpret_cast<volatile uint32_t*>(p) = v;
    } else if constexpr (sizeof(E) == 8) {
        uint64_t v;
        memcpy(&v, &in, 8);
        *reinterpret_cast<volatile uint64_t*>(p) = v;
    } else {
        Vec16 v;
        memcpy(&v, &in, 16);
        stVec(p, v);
    }
}

template<typename VR>
__device__ __forceinline__ void groupTail(const FbCommDev& c,
                                          const GroupSeg& sg,
                                          int n)
{
    // Elements sit at element-aligned addresses (16-byte aligned tensor start
    // + a multiple of the element size): move them by value
    using Elem = typename VR::Elem;
    constexpr uint32_t EB = VR::ELEM_BYTES;
    const uint64_t base = (uint64_t)sg.nVec * 16;
    for (uint32_t e = 0; e + EB <= sg.tailBytes; e += EB) {
        Elem acc = ldElemGlobal<Elem>(c.heap[0] + sg.sendOff + base + e);
        for (int p = 1; p < n; p++) {
            Elem v = ldElemGlobal<Elem>(c.heap[p] + sg.sendOff + base + e);
            acc = VR::combine(acc, v);
        }
        for (int p = 0; p < n; p++) {
            stElemGlobal<Elem>(c.heap[p] + sg.recvOff + base + e, acc);
        }
    }
}

template<typename VR, int NR>
__global__ void __launch_bounds__(512, 1) groupAllReduceKernel(
  const GroupArgs a)
{
    extern __shared__ __align__(16) uint8_t sGroupRaw[];
    GroupSeg* sSegs = reinterpret_cast<GroupSeg*>(sGroupRaw);
    const FbCommDev& c = a.comm;
    const int n = (NR > 0) ? NR : c.nranks;
    // the segment table is local memory: fetch it while the peers arrive
    {
        const Vec16* src = reinterpret_cast<const Vec16*>(a.segs);
        Vec16* dst = reinterpret_cast<Vec16*>(sGroupRaw);
        for (uint32_t i = threadIdx.x; i < a.nSegs * 2; i += blockDim.x) {
            dst[i] = src[i];
        }
    }
    BlockBarrier bar;
    bar.epoch = 0;
    bool ok = true;
    if (!a.noSync) {
        bar.load(c);
        ok = bar.sync(c); // (also publishes sSegs to the CTA)
    } else {
        // no cross-rank synchronisation (single rank, or done at stream
        // level): the grid is not tied to the barrier slots either
        __syncthreads();
    }

    if (ok && a.nSegs > 0) {
        constexpr int UNROLL = (NR == 8) ? 2 : (NR == 1 ? 8 : 4);
        constexpr uint32_t CHUNK = 32u * UNROLL;
        const uint32_t lane = threadIdx.x & 31;
        const uint32_t warpsPerCta = blockDim.x >> 5;
        const uint32_t warpStride = gridDim.x * warpsPerCta;
        int cur = 0;
        for (uint32_t ch = blockIdx.x * warpsPerCta + (threadIdx.x >> 5);
             ch < a.totalChunks;
             ch += warpStride) {
            // segment owning chunk `ch`: usually the same or the next one
            if (!(sSegs[cur].chunk0 <= ch &&
                  (cur + 1 == (int)a.nSegs || ch < sSegs[cur + 1].chunk0))) {
                int lo = 0;
                int hi = (int)a.nSegs - 1;
                while (lo < hi) {
                    int mid = (lo + hi + 1) >> 1;
                    if (sSegs[mid].chunk0 <= ch) {
                        lo = mid;
                    } else {
                        hi = mid - 1;
                    }
                }
                cur = lo;
            }
            const GroupSeg sg = sSegs[cur];
            const uint32_t v0 = (ch - sg.chunk0) * CHUNK;
            const uint64_t sOff = sg.sendOff + (uint64_t)v0 * 16;
            const uint64_t rOff = sg.recvOff + (uint64_t)v0 * 16;
            const uint32_t rem = sg.nVec > v0 ? sg.nVec - v0 : 0;
            if (rem >= CHUNK) {
                Vec16 acc[UNROLL];
                if constexpr (NR > 0) {
                    Vec16 v[UNROLL][NR];
#pragma unroll
                    for (int u = 0; u < UNROLL; u++) {
#pragma unroll
                        for (int p = 0; p < NR; p++) {
                            v[u][p] = ldVecStream(c.heap[p] + sOff +
                                                  (uint64_t)(u * 32 + lane) * 16);
                        }
                    }
#pragma unroll
                    for (int u = 0; u < UNROLL; u++) {
                        acc[u] = v[u][0];
#pragma unroll
                        for (int p = 1; p < NR; p++) {
                            acc[u] = VR::apply(acc[u], v[u][p]);
                        }
                    }
#pragma unroll
                    for (int u = 0; u < UNROLL; u++) {
#pragma unroll
                        for (int p = 0; p < NR; p++) {
                            stVec(c.heap[p] + rOff + (uint64_t)(u * 32 + lane) * 16,
                                  acc[u]);
                        }
                    }
                } else {
#pragma unroll
                    for (int u = 0; u < UNROLL; u++) {
                        acc[u] = ldVecStream(c.heap[0] + sOff +
                                             (uint64_t)(u * 32 + lane) * 16);
                    }
                    for (int p = 1; p < n; p++) {
                        Vec16 v[UNROLL];
#pragma unroll
                        for (int u = 0; u < UNROLL; u++) {
                            v[u] = ldVecStream(c.heap[p] + sOff +
                                               (uint64_t)(u * 32 + lane) * 16);
                        }
#pragma unroll
                        for (int u = 0; u < UNROLL; u++) {
                            acc[u] = VR::apply(acc[u], v[u]);
                        }
                    }
                    for (int p = 0; p < n; p++) {
#pragma unroll
                        for (int u = 0; u < UNROLL; u++) {
                            stVec(c.heap[p] + rOff + (uint64_t)(u * 32 + lane) * 16,
                                  acc[u]);
                        }
                    }
                }
            } else {
                // ragged end of a segment (or a whole tiny tensor)
#pragma unroll
                for (int u = 0; u < UNROLL; u++) {
                    const uint32_t i = (uint32_t)u * 32 + lane;
                    if (i < rem) {
                        Vec16 acc = ldVecStream(c.heap[0] + sOff + (uint64_t)i * 16);
                        for (int p = 1; p < n; p++) {
                            Vec16 v = ldVecStream(c.heap[p] + sOff + (uint64_t)i * 16);
                            acc = VR::apply(acc, v);
                        }
                        for (int p = 0; p < n; p++) {
                            stVec(c.heap[p] + rOff + (uint64_t)i * 16, acc);
                        }
                    }
                }
                // the < 16-byte tail rides with the segment's last chunk
                if (sg.tailBytes != 0 && lane == 0 && v0 + CHUNK > sg.nVec) {
                    groupTail<VR>(c, sg, n);
                }
            }
        }
    }

    if (!a.noSync) {
        bar.sync(c);
        bar.store(c);
    }
}

template<typename VR>
cudaError_t launchGroup(const GroupArgs& a,
                        int blocks,
                        int threads,
                        cudaStream_t stream)
{
    const size_t smem = (size_t)a.nSegs * sizeof(GroupSeg);
    const int nr = a.comm.nranks;
    if (nr == 1) {
        groupAllReduceKernel<VR, 1><<<blocks, threads, smem, stream>>>(a);
    } else if (nr == 2) {
        groupAllReduceKernel<VR, 2><<<blocks, threads, smem, stream>>>(a);
    } else if (nr == 4) {
        groupAllReduceKernel<VR, 4><<<blocks, threads, smem, stream>>>(a);
    } else if (nr == 8) {
        groupAllReduceKernel<VR, 8><<<blocks, threads, smem, stream>>>(a);
    } else {
        groupAllReduceKernel<VR, 0><<<blocks, threads, smem, stream>>>(a);
    }
    return cudaGetLastError();
}

// ----------------------------------------------------------------------------
// Grouped reduce-scatter: one MPI_Reduce_scatter_block per tensor, all in ONE
// launch per rank.  A segment is this rank's shard of one tensor (sendOff
// points at shard `rank` of the input, recvOff at the local output), and a
// shard is a whole number of 16-byte vectors.  Each chunk gathers its vectors
// from every peer, reduces them in registers and stores to this rank's output
// only.  Entry barrier: every input is complete.  Exit barrier: the peers
// have finished reading this rank's input.
// ----------------------------------------------------------------------------
template<typename VR, int NR>
__global__ void __launch_bounds__(512, 1) groupReduceScatterKernel(
  const GroupArgs a)
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
        uint8_t* const out = c.heap[c.rank];
        int cur = 0;
        for (uint32_t ch = blockIdx.x * warpsPerCta + (threadIdx.x >> 5);
             ch < a.totalChunks;
             ch += warpStride) {
            cur = groupSegOf(sSegs, a.nSegs, cur, ch);
            const GroupSeg sg = sSegs[cur];
            const uint32_t v0 = (ch - sg.chunk0) * CHUNK;
            const uint64_t sOff = sg.sendOff + (uint64_t)v0 * 16;
            uint8_t* const dst = out + sg.recvOff + (uint64_t)v0 * 16;
            const uint32_t rem = sg.nVec - v0;
            if (rem >= CHUNK) {
                Vec16 acc[UNROLL];
                if constexpr (NR > 0) {
                    Vec16 v[UNROLL][NR];
#pragma unroll
                    for (int u = 0; u < UNROLL; u++) {
#pragma unroll
                        for (int p = 0; p < NR; p++) {
                            v[u][p] = ldVecStream(c.heap[p] + sOff +
                                                  (uint64_t)(u * 32 + lane) * 16);
                        }
                    }
#pragma unroll
                    for (int u = 0; u < UNROLL; u++) {
                        acc[u] = v[u][0];
#pragma unroll
                        for (int p = 1; p < NR; p++) {
                            acc[u] = VR::apply(acc[u], v[u][p]);
                        }
                    }
                } else {
#pragma unroll
                    for (int u = 0; u < UNROLL; u++) {
                        acc[u] = ldVecStream(c.heap[0] + sOff +
                                             (uint64_t)(u * 32 + lane) * 16);
                    }
                    for (int p = 1; p < n; p++) {
                        Vec16 v[UNROLL];
#pragma unroll
                        for (int u = 0; u < UNROLL; u++) {
                            v[u] = ldVecStream(c.heap[p] + sOff +
                                               (uint64_t)(u * 32 + lane) * 16);
                        }
#pragma unroll
                        for (int u = 0; u < UNROLL; u++) {
                            acc[u] = VR::apply(acc[u], v[u]);
                        }
                    }
                }
#pragma unroll
                for (int u = 0; u < UNROLL; u++) {
                    stVec(dst + (uint64_t)(u * 32 + lane) * 16, acc[u]);
                }
            } else {
                // ragged end of a shard (or a whole small one)
#pragma unroll
                for (int u = 0; u < UNROLL; u++) {
                    const uint32_t i = (uint32_t)u * 32 + lane;
                    if (i < rem) {
                        Vec16 acc = ldVecStream(c.heap[0] + sOff + (uint64_t)i * 16);
                        for (int p = 1; p < n; p++) {
                            Vec16 v = ldVecStream(c.heap[p] + sOff + (uint64_t)i * 16);
                            acc = VR::apply(acc, v);
                        }
                        stVec(dst + (uint64_t)i * 16, acc);
                    }
                }
            }
        }
    }
    groupExit(a, bar);
}

template<typename VR>
cudaError_t launchGroupReduceScatter(const GroupArgs& a,
                                     int blocks,
                                     int threads,
                                     cudaStream_t stream)
{
    const size_t smem = (size_t)a.nSegs * sizeof(GroupSeg);
    const int nr = a.comm.nranks;
    if (nr == 1) {
        groupReduceScatterKernel<VR, 1><<<blocks, threads, smem, stream>>>(a);
    } else if (nr == 2) {
        groupReduceScatterKernel<VR, 2><<<blocks, threads, smem, stream>>>(a);
    } else if (nr == 4) {
        groupReduceScatterKernel<VR, 4><<<blocks, threads, smem, stream>>>(a);
    } else if (nr == 8) {
        groupReduceScatterKernel<VR, 8><<<blocks, threads, smem, stream>>>(a);
    } else {
        groupReduceScatterKernel<VR, 0><<<blocks, threads, smem, stream>>>(a);
    }
    return cudaGetLastError();
}

template<typename VR>
cudaError_t preloadReduce()
{
    cudaFuncAttributes a;
    cudaError_t e = cudaSuccess;
#define FB_PRELOAD(k)                                                          \
    if (e == cudaSuccess) {                                                    \
        e = cudaFuncGetAttributes(&a, k);                                      \
    }
    FB_PRELOAD((reduceKernel<VR, 0>))
    FB_PRELOAD((reduceKernel<VR, 2>))
    FB_PRELOAD((reduceKernel<VR, 4>))
    FB_PRELOAD((reduceKernel<VR, 8>))
    FB_PRELOAD((llAllReduceKernel<VR, 0>))
    FB_PRELOAD((llAllReduceKernel<VR, 2>))
    FB_PRELOAD((llAllReduceKernel<VR, 4>))
    FB_PRELOAD((llAllReduceKernel<VR, 8>))
    FB_PRELOAD((groupAllReduceKernel<VR, 0>))
    FB_PRELOAD((groupAllReduceKernel<VR, 1>))
    FB_PRELOAD((groupAllReduceKernel<VR, 2>))
    FB_PRELOAD((groupAllReduceKernel<VR, 4>))
    FB_PRELOAD((groupAllReduceKernel<VR, 8>))
    FB_PRELOAD((groupReduceScatterKernel<VR, 0>))
    FB_PRELOAD((groupReduceScatterKernel<VR, 1>))
    FB_PRELOAD((groupReduceScatterKernel<VR, 2>))
    FB_PRELOAD((groupReduceScatterKernel<VR, 4>))
    FB_PRELOAD((groupReduceScatterKernel<VR, 8>))
#undef FB_PRELOAD
    return e;
}

template<typename VR>
const ReduceLaunchers* launchersFor()
{
    static const ReduceLaunchers l = { &launchReduce<VR>,
                                       &launchLL<VR>,
                                       &launchGroup<VR>,
                                       &launchGroupReduceScatter<VR>,
                                       &preloadReduce<VR> };
    return &l;
}

} // namespace fb
