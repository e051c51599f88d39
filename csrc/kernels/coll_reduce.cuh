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

// ----------------------------------------------------------------------------
// Grouped reduce and scan: one MPI_Reduce, MPI_Scan or MPI_Exscan per item,
// all in ONE launch per rank, through the staging buffers (RootedSeg in
// launch_api.h: the table, the chunk space and the LOCAL / MOVE / UNSTAGE
// steps).  User buffers are any memory this rank's GPU can load and store, at
// any alignment; the staged slices are 16-byte aligned, so the reduction
// itself always runs on 128-bit vectors.
// ----------------------------------------------------------------------------
// MOVE of one chunk: the slices at `slice` (len bytes) of the staging buffers
// at `stageOff` of ranks 0..nFold-1 folded in rank order,
// acc = slice_0, acc = op(acc, slice_p).  After rank p, the running value of
// every vector goes to out.vec(p, slice + off, v), and of every element of the
// < 16-byte tail (lane 0) to out.elem(p, slice + off, e); `off` is its byte
// offset in the chunk.
template<typename VR, int NR, int UNROLL, typename Out>
__device__ __forceinline__ void groupFoldChunk(const FbCommDev& c,
                                               int nFold,
                                               uint64_t stageOff,
                                               uint64_t slice,
                                               uint32_t len,
                                               uint32_t lane,
                                               const Out& out)
{
    constexpr uint32_t CHUNK = 32u * UNROLL;
    const uint64_t sOff = stageOff + slice;
    const uint32_t nVec = len / 16;
    if (nVec == CHUNK) {
        if constexpr (NR > 0) {
            Vec16 v[UNROLL][NR];
#pragma unroll
            for (int u = 0; u < UNROLL; u++) {
#pragma unroll
                for (int p = 0; p < NR; p++) {
                    if (p < nFold) {
                        v[u][p] = ldVecStream(c.heap[p] + sOff + (uint64_t)(u * 32 + lane) * 16);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < UNROLL; u++) {
                const uint64_t off = slice + (uint64_t)(u * 32 + lane) * 16;
                Vec16 acc = v[u][0];
                out.vec(0, off, acc);
#pragma unroll
                for (int p = 1; p < NR; p++) {
                    if (p < nFold) {
                        acc = VR::apply(acc, v[u][p]);
                        out.vec(p, off, acc);
                    }
                }
            }
        } else {
            Vec16 acc[UNROLL];
#pragma unroll
            for (int u = 0; u < UNROLL; u++) {
                acc[u] = ldVecStream(c.heap[0] + sOff + (uint64_t)(u * 32 + lane) * 16);
                out.vec(0, slice + (uint64_t)(u * 32 + lane) * 16, acc[u]);
            }
            for (int p = 1; p < nFold; p++) {
                Vec16 v[UNROLL];
#pragma unroll
                for (int u = 0; u < UNROLL; u++) {
                    v[u] = ldVecStream(c.heap[p] + sOff + (uint64_t)(u * 32 + lane) * 16);
                }
#pragma unroll
                for (int u = 0; u < UNROLL; u++) {
                    acc[u] = VR::apply(acc[u], v[u]);
                    out.vec(p, slice + (uint64_t)(u * 32 + lane) * 16, acc[u]);
                }
            }
        }
        return;
    }
    // the ragged end of a piece (or a whole small one)
#pragma unroll
    for (int u = 0; u < UNROLL; u++) {
        const uint32_t i = (uint32_t)u * 32 + lane;
        if (i < nVec) {
            Vec16 acc = ldVecStream(c.heap[0] + sOff + (uint64_t)i * 16);
            out.vec(0, slice + (uint64_t)i * 16, acc);
            for (int p = 1; p < nFold; p++) {
                acc = VR::apply(acc, ldVecStream(c.heap[p] + sOff + (uint64_t)i * 16));
                out.vec(p, slice + (uint64_t)i * 16, acc);
            }
        }
    }
    if (lane == 0) {
        // (pieces end at element boundaries: chunks are whole elements)
        using Elem = typename VR::Elem;
        constexpr uint32_t EB = VR::ELEM_BYTES;
        for (uint32_t e = nVec * 16; e + EB <= len; e += EB) {
            Elem acc = ldElemGlobal<Elem>(c.heap[0] + sOff + e);
            out.elem(0, slice + e, acc);
            for (int p = 1; p < nFold; p++) {
                acc = VR::combine(acc, ldElemGlobal<Elem>(c.heap[p] + sOff + e));
                out.elem(p, slice + e, acc);
            }
        }
    }
}

// The reduce's results: the fold over every rank, into the root's slices
struct ReduceOut
{
    uint8_t* dst; // the root's result staging buffer
    int last;     // n - 1
    __device__ __forceinline__ void vec(int p, uint64_t off, const Vec16& v) const
    {
        if (p == last) {
            stVec(dst + off, v);
        }
    }
    template<typename Elem>
    __device__ __forceinline__ void elem(int p, uint64_t off, Elem v) const
    {
        if (p == last) {
            stElemGlobal<Elem>(dst + off, v);
        }
    }
};

// The scan's results: the fold after rank p into rank p + shift's slices
// (shift 0: inclusive, 1: exclusive; the caller folds ranks 0..n-1-shift)
struct ScanOut
{
    const FbCommDev& c;
    uint64_t stageRecvOff;
    int shift;
    __device__ __forceinline__ void vec(int p, uint64_t off, const Vec16& v) const
    {
        stVec(c.heap[p + shift] + stageRecvOff + off, v);
    }
    template<typename Elem>
    __device__ __forceinline__ void elem(int p, uint64_t off, Elem v) const
    {
        stElemGlobal<Elem>(c.heap[p + shift] + stageRecvOff + off, v);
    }
};

// This warp's walk of the chunk space: chunk ch is staged, folded and
// unstaged by the warp at position ch % warpStride of the grid on every rank
// (the same CTA index, which is what the per-CTA barriers order)
struct GroupWalk
{
    uint32_t first;
    uint32_t stride;
    uint32_t lane;
    __device__ __forceinline__ GroupWalk()
      : first(blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5))
      , stride(gridDim.x * (blockDim.x >> 5))
      , lane(threadIdx.x & 31)
    {}
};

// LOCAL: this warp's chunks of every send into its slices of `stage`; on one
// rank (NR == 1) into the recv instead, nothing in place
template<int NR, int UNROLL>
__device__ __forceinline__ void groupStageSends(const GroupArgs& a,
                                                const RootedSeg* segs,
                                                const GroupWalk& w,
                                                int& cur,
                                                uint8_t* stage)
{
    constexpr uint32_t CB = 32u * UNROLL * 16;
    for (uint32_t ch = w.first; ch < a.totalChunks; ch += w.stride) {
        const RootedChunk k = rootedChunk<UNROLL>(segs, a.nSegs, cur, ch);
        const uint8_t* const send = reinterpret_cast<const uint8_t*>(k.sg->send) + k.off;
        if constexpr (NR == 1) {
            uint8_t* const recv = reinterpret_cast<uint8_t*>(k.sg->recv) + k.off;
            if (recv != send) {
                rootedCopy<UNROLL>(recv, send, k.len, w.lane);
            }
        } else {
            rootedCopy<UNROLL>(stage + (uint64_t)ch * CB, send, k.len, w.lane);
        }
    }
}

// MOVE: the chunks this rank owns, (ch % warpStride + ch / warpStride) % n,
// which only the chunk and the grid (the same on every rank) decide: every
// warp of every rank owns a share of its walk, also when the walk is a single
// chunk long.  Each is folded over ranks 0..nFold-1 into `out`.
template<typename VR, int NR, int UNROLL, typename Out>
__device__ __forceinline__ void groupFoldOwned(const GroupArgs& a,
                                               const RootedSeg* segs,
                                               const GroupWalk& w,
                                               int& cur,
                                               int n,
                                               int nFold,
                                               const Out& out)
{
    constexpr uint32_t CB = 32u * UNROLL * 16;
    int owner = (int)(w.first % (uint32_t)n);
    for (uint32_t ch = w.first; ch < a.totalChunks; ch += w.stride, owner = owner + 1 == n ? 0 : owner + 1) {
        if (owner != a.comm.rank) {
            continue;
        }
        const RootedChunk k = rootedChunk<UNROLL>(segs, a.nSegs, cur, ch);
        groupFoldChunk<VR, NR, UNROLL>(a.comm, nFold, a.stageOff, (uint64_t)ch * CB, k.len, w.lane, out);
    }
}

// UNSTAGE: this warp's result slices of `res` into every recv
template<int UNROLL>
__device__ __forceinline__ void groupUnstage(const GroupArgs& a,
                                             const RootedSeg* segs,
                                             const GroupWalk& w,
                                             int& cur,
                                             const uint8_t* res)
{
    constexpr uint32_t CB = 32u * UNROLL * 16;
    for (uint32_t ch = w.first; ch < a.totalChunks; ch += w.stride) {
        const RootedChunk k = rootedChunk<UNROLL>(segs, a.nSegs, cur, ch);
        rootedCopy<UNROLL>(reinterpret_cast<uint8_t*>(k.sg->recv) + k.off, res + (uint64_t)ch * CB, k.len, w.lane);
    }
}

template<typename VR, int NR>
__global__ void __launch_bounds__(512, 1) groupReduceKernel(const GroupArgs a)
{
    extern __shared__ __align__(16) uint8_t sGroupRaw[];
    constexpr int UNROLL = (NR == 8) ? 2 : (NR == 1 ? 8 : 4);
    const FbCommDev& c = a.comm;
    const int n = (NR > 0) ? NR : c.nranks;
    const RootedSeg* segs = rootedLoad(a, sGroupRaw);
    const GroupWalk w;
    int cur = 0;
    if (a.phase & GROUP_PHASE_LOCAL) {
        // (one rank: the result is the send)
        groupStageSends<NR, UNROLL>(a, segs, w, cur, c.heap[c.rank] + a.stageOff);
    }
    if constexpr (NR == 1) {
        return;
    }
    BlockBarrier bar;
    bool ok = true;
    if (!a.noSync) {
        bar.load(c);
        ok = bar.sync(c);
    }
    if (ok && (a.phase & GROUP_PHASE_MOVE)) {
        groupFoldOwned<VR, NR, UNROLL>(a, segs, w, cur, n, n, ReduceOut{ c.heap[a.root] + a.stageRecvOff, n - 1 });
    }
    if (!a.noSync) {
        ok = bar.sync(c) && ok;
    }
    if (ok && c.rank == a.root && (a.phase & GROUP_PHASE_UNSTAGE)) {
        groupUnstage<UNROLL>(a, segs, w, cur, c.heap[c.rank] + a.stageRecvOff);
    }
    if (!a.noSync) {
        bar.store(c);
    }
}

// The scan's steps (a.exclusive: 0 scan, 1 exscan): LOCAL as the reduce's,
// but an exscan's last rank stages nothing (no rank reads its send); MOVE
// folds ranks 0..n-1-exclusive and stores the value after rank p into rank
// p + exclusive's result slices; UNSTAGE on every rank but an exscan's rank
// 0, whose recv is never written.  One rank: a scan copies send to recv, an
// exscan does nothing.
template<typename VR, int NR>
__global__ void __launch_bounds__(512, 1) groupScanKernel(const GroupArgs a)
{
    extern __shared__ __align__(16) uint8_t sGroupRaw[];
    constexpr int UNROLL = (NR == 8) ? 2 : (NR == 1 ? 8 : 4);
    const FbCommDev& c = a.comm;
    const int n = (NR > 0) ? NR : c.nranks;
    const int ex = a.exclusive;
    const RootedSeg* segs = rootedLoad(a, sGroupRaw);
    const GroupWalk w;
    int cur = 0;
    if ((a.phase & GROUP_PHASE_LOCAL) && !(ex && c.rank == n - 1)) {
        groupStageSends<NR, UNROLL>(a, segs, w, cur, c.heap[c.rank] + a.stageOff);
    }
    if constexpr (NR == 1) {
        return;
    }
    BlockBarrier bar;
    bool ok = true;
    if (!a.noSync) {
        bar.load(c);
        ok = bar.sync(c);
    }
    if (ok && (a.phase & GROUP_PHASE_MOVE)) {
        groupFoldOwned<VR, NR, UNROLL>(a, segs, w, cur, n, n - ex, ScanOut{ c, a.stageRecvOff, ex });
    }
    if (!a.noSync) {
        ok = bar.sync(c) && ok;
    }
    if (ok && !(ex && c.rank == 0) && (a.phase & GROUP_PHASE_UNSTAGE)) {
        groupUnstage<UNROLL>(a, segs, w, cur, c.heap[c.rank] + a.stageRecvOff);
    }
    if (!a.noSync) {
        bar.store(c);
    }
}

template<typename VR>
cudaError_t launchGroupReduce(const GroupArgs& a, int blocks, int threads, cudaStream_t stream)
{
    const size_t smem = (size_t)a.nSegs * sizeof(RootedSeg);
    const int nr = a.comm.nranks;
    if (nr == 1) {
        groupReduceKernel<VR, 1><<<blocks, threads, smem, stream>>>(a);
    } else if (nr == 2) {
        groupReduceKernel<VR, 2><<<blocks, threads, smem, stream>>>(a);
    } else if (nr == 4) {
        groupReduceKernel<VR, 4><<<blocks, threads, smem, stream>>>(a);
    } else if (nr == 8) {
        groupReduceKernel<VR, 8><<<blocks, threads, smem, stream>>>(a);
    } else {
        groupReduceKernel<VR, 0><<<blocks, threads, smem, stream>>>(a);
    }
    return cudaGetLastError();
}

template<typename VR>
cudaError_t launchGroupScan(const GroupArgs& a, int blocks, int threads, cudaStream_t stream)
{
    const size_t smem = (size_t)a.nSegs * sizeof(RootedSeg);
    const int nr = a.comm.nranks;
    if (nr == 1) {
        groupScanKernel<VR, 1><<<blocks, threads, smem, stream>>>(a);
    } else if (nr == 2) {
        groupScanKernel<VR, 2><<<blocks, threads, smem, stream>>>(a);
    } else if (nr == 4) {
        groupScanKernel<VR, 4><<<blocks, threads, smem, stream>>>(a);
    } else if (nr == 8) {
        groupScanKernel<VR, 8><<<blocks, threads, smem, stream>>>(a);
    } else {
        groupScanKernel<VR, 0><<<blocks, threads, smem, stream>>>(a);
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
    FB_PRELOAD((groupReduceKernel<VR, 0>))
    FB_PRELOAD((groupReduceKernel<VR, 1>))
    FB_PRELOAD((groupReduceKernel<VR, 2>))
    FB_PRELOAD((groupReduceKernel<VR, 4>))
    FB_PRELOAD((groupReduceKernel<VR, 8>))
    FB_PRELOAD((groupScanKernel<VR, 0>))
    FB_PRELOAD((groupScanKernel<VR, 1>))
    FB_PRELOAD((groupScanKernel<VR, 2>))
    FB_PRELOAD((groupScanKernel<VR, 4>))
    FB_PRELOAD((groupScanKernel<VR, 8>))
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
                                       &launchGroupReduce<VR>,
                                       &launchGroupScan<VR>,
                                       &preloadReduce<VR> };
    return &l;
}

} // namespace fb
