// Grouped gather and scatter: many MPI_Gather / MPI_Scatter calls with one
// root, ONE launch per rank (see RootedSeg in launch_api.h for the table and
// the steps).  The user buffers are any memory this rank's GPU can load and
// store; only the staging slices are symmetric, and their offsets follow from
// the counts alone.  So the root never needs a peer's user address, and an
// in-place root (which its peers cannot see) changes nothing but its own
// copy.  The NVLink leg runs between the root and the peers; the extra local
// copy runs on every non-root at once.  Dtype-free: a byte copy.
#include "coll_group.cuh"

namespace fb {

// The root's MOVE step of one chunk: block p of `user` (stride apart) and
// peer p's slice, in the direction `toPeers`.  With every block and the
// user side 16-byte aligned, every peer's vectors are in flight before the
// first store (NVLink latency); otherwise one peer at a time.
template<int NR, int UNROLL, bool TO_PEERS>
__device__ __forceinline__ void rootedMove(const FbCommDev& c,
                                           uint64_t stageOff,
                                           uint32_t ch,
                                           uint8_t* user,
                                           uint64_t stride,
                                           uint8_t* own,
                                           uint32_t len,
                                           uint32_t lane)
{
    constexpr uint32_t CB = 32u * UNROLL * 16;
    const int n = (NR > 0) ? NR : c.nranks;
    const int rank = c.rank;
    const uint64_t slice = stageOff + (uint64_t)ch * CB;
    // own == null: in place, the root's block stays where it is
    if constexpr (NR > 1) {
        if (len == CB && (((uintptr_t)user | stride | (uintptr_t)own) & 15) == 0) {
            Vec16 v[NR][UNROLL];
#pragma unroll
            for (int q = 0; q < NR; q++) {
                const int p = (rank + q) & (NR - 1);
                const uint8_t* s = TO_PEERS ? user + (uint64_t)p * stride : (q == 0 ? own : c.heap[p] + slice);
                if (q != 0 || own != nullptr) {
#pragma unroll
                    for (int u = 0; u < UNROLL; u++) {
                        v[q][u] = ldVecStream(s + (uint32_t)(u * 32 + lane) * 16);
                    }
                }
            }
#pragma unroll
            for (int q = 0; q < NR; q++) {
                const int p = (rank + q) & (NR - 1);
                uint8_t* d = TO_PEERS ? (q == 0 ? own : c.heap[p] + slice) : user + (uint64_t)p * stride;
                if (q != 0 || own != nullptr) {
#pragma unroll
                    for (int u = 0; u < UNROLL; u++) {
                        stVec(d + (uint32_t)(u * 32 + lane) * 16, v[q][u]);
                    }
                }
            }
            return;
        }
    }
    for (int q = 0; q < n; q++) {
        const int p = (rank + q < n) ? rank + q : rank + q - n;
        if (q == 0 && own == nullptr) {
            continue;
        }
        uint8_t* const blk = user + (uint64_t)p * stride;
        uint8_t* const peer = q == 0 ? own : c.heap[p] + slice;
        if (TO_PEERS) {
            rootedCopy<UNROLL>(peer, blk, len, lane);
        } else {
            rootedCopy<UNROLL>(blk, peer, len, lane);
        }
    }
}

template<int NR>
__global__ void __launch_bounds__(512, 1) groupGatherKernel(const GroupArgs a)
{
    extern __shared__ __align__(16) uint8_t sGroupRaw[];
    constexpr int UNROLL = (NR == 8) ? 2 : (NR == 1 ? 8 : 4);
    const FbCommDev& c = a.comm;
    const RootedSeg* segs = rootedLoad(a, sGroupRaw);
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warpsPerCta = blockDim.x >> 5;
    const uint32_t warpStride = gridDim.x * warpsPerCta;
    const uint32_t first = blockIdx.x * warpsPerCta + (threadIdx.x >> 5);
    const bool isRoot = c.rank == a.root;
    int cur = 0;
    if (!isRoot && (a.phase & GROUP_PHASE_LOCAL)) {
        uint8_t* const stage = c.heap[c.rank] + a.stageOff;
        for (uint32_t ch = first; ch < a.totalChunks; ch += warpStride) {
            const RootedChunk k = rootedChunk<UNROLL>(segs, a.nSegs, cur, ch);
            rootedCopy<UNROLL>(stage + (uint64_t)ch * (32u * UNROLL * 16),
                               reinterpret_cast<const uint8_t*>(k.sg->send) + k.off,
                               k.len,
                               lane);
        }
    }
    BlockBarrier bar;
    bool ok = true;
    if (!a.noSync) {
        bar.load(c);
        ok = bar.sync(c);
    }
    if (ok && isRoot && (a.phase & GROUP_PHASE_MOVE)) {
        for (uint32_t ch = first; ch < a.totalChunks; ch += warpStride) {
            const RootedChunk k = rootedChunk<UNROLL>(segs, a.nSegs, cur, ch);
            uint8_t* const recv = reinterpret_cast<uint8_t*>(k.sg->recv) + k.off;
            uint8_t* const send = reinterpret_cast<uint8_t*>(k.sg->send) + k.off;
            uint8_t* const own = send == recv + (uint64_t)a.root * k.sg->stride ? nullptr : send;
            rootedMove<NR, UNROLL, false>(c, a.stageOff, ch, recv, k.sg->stride, own, k.len, lane);
        }
    }
    if (!a.noSync) {
        bar.sync(c);
        bar.store(c);
    }
}

template<int NR>
__global__ void __launch_bounds__(512, 1) groupScatterKernel(const GroupArgs a)
{
    extern __shared__ __align__(16) uint8_t sGroupRaw[];
    constexpr int UNROLL = (NR == 8) ? 2 : (NR == 1 ? 8 : 4);
    const FbCommDev& c = a.comm;
    const RootedSeg* segs = rootedLoad(a, sGroupRaw);
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warpsPerCta = blockDim.x >> 5;
    const uint32_t warpStride = gridDim.x * warpsPerCta;
    const uint32_t first = blockIdx.x * warpsPerCta + (threadIdx.x >> 5);
    const bool isRoot = c.rank == a.root;
    int cur = 0;
    BlockBarrier bar;
    bool ok = true;
    if (!a.noSync) {
        bar.load(c);
        ok = bar.sync(c);
    }
    if (ok && isRoot && (a.phase & GROUP_PHASE_MOVE)) {
        for (uint32_t ch = first; ch < a.totalChunks; ch += warpStride) {
            const RootedChunk k = rootedChunk<UNROLL>(segs, a.nSegs, cur, ch);
            uint8_t* const send = reinterpret_cast<uint8_t*>(k.sg->send) + k.off;
            uint8_t* const recv = reinterpret_cast<uint8_t*>(k.sg->recv) + k.off;
            uint8_t* const own = recv == send + (uint64_t)a.root * k.sg->stride ? nullptr : recv;
            rootedMove<NR, UNROLL, true>(c, a.stageOff, ch, send, k.sg->stride, own, k.len, lane);
        }
    }
    if (!a.noSync) {
        ok = bar.sync(c) && ok;
    }
    // (the root's CTA that pushed chunk ch has the same index as this one)
    if (ok && !isRoot && (a.phase & GROUP_PHASE_LOCAL)) {
        const uint8_t* const stage = c.heap[c.rank] + a.stageOff;
        for (uint32_t ch = first; ch < a.totalChunks; ch += warpStride) {
            const RootedChunk k = rootedChunk<UNROLL>(segs, a.nSegs, cur, ch);
            rootedCopy<UNROLL>(reinterpret_cast<uint8_t*>(k.sg->recv) + k.off,
                               stage + (uint64_t)ch * (32u * UNROLL * 16),
                               k.len,
                               lane);
        }
    }
    if (!a.noSync) {
        bar.store(c);
    }
}

#define FB_ROOTED_LAUNCHER(name, kernel)                                                                               \
    cudaError_t name(const GroupArgs& a, int blocks, int threads, cudaStream_t s)                                     \
    {                                                                                                                  \
        const size_t smem = (size_t)a.nSegs * sizeof(RootedSeg);                                                       \
        const int n = a.comm.nranks;                                                                                   \
        if (n == 1) {                                                                                                  \
            kernel<1><<<blocks, threads, smem, s>>>(a);                                                                \
        } else if (n == 2) {                                                                                           \
            kernel<2><<<blocks, threads, smem, s>>>(a);                                                                \
        } else if (n == 4) {                                                                                           \
            kernel<4><<<blocks, threads, smem, s>>>(a);                                                                \
        } else if (n == 8) {                                                                                           \
            kernel<8><<<blocks, threads, smem, s>>>(a);                                                                \
        } else {                                                                                                       \
            kernel<0><<<blocks, threads, smem, s>>>(a);                                                                \
        }                                                                                                              \
        return cudaGetLastError();                                                                                     \
    }
FB_ROOTED_LAUNCHER(launchGroupGather, groupGatherKernel)
FB_ROOTED_LAUNCHER(launchGroupScatter, groupScatterKernel)
#undef FB_ROOTED_LAUNCHER

cudaError_t preloadRootedKernels()
{
    cudaFuncAttributes attr;
    cudaError_t e = cudaSuccess;
#define FB_PRELOAD(k)                                                                                                  \
    if (e == cudaSuccess) {                                                                                            \
        e = cudaFuncGetAttributes(&attr, k);                                                                           \
    }
    FB_PRELOAD((groupGatherKernel<0>))
    FB_PRELOAD((groupGatherKernel<1>))
    FB_PRELOAD((groupGatherKernel<2>))
    FB_PRELOAD((groupGatherKernel<4>))
    FB_PRELOAD((groupGatherKernel<8>))
    FB_PRELOAD((groupScatterKernel<0>))
    FB_PRELOAD((groupScatterKernel<1>))
    FB_PRELOAD((groupScatterKernel<2>))
    FB_PRELOAD((groupScatterKernel<4>))
    FB_PRELOAD((groupScatterKernel<8>))
#undef FB_PRELOAD
    return e;
}

} // namespace fb
