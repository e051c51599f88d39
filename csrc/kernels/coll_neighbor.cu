// Grouped neighbourhood all-gather and all-to-all: many
// MPI_Neighbor_allgather / MPI_Neighbor_alltoall calls over one graph, ONE
// launch per rank (see NeighborEdge in launch_api.h for the table and the
// steps).  Every rank stages its send blocks at slots that follow from the
// counts and the graph alone, and after the entry barrier pulls each in-edge's
// block from its source's staging.  So no rank needs a peer's user address,
// and user buffers are any memory this rank's GPU can load and store.
// Dtype-free: a byte copy.
#include "coll_group.cuh"

namespace fb {

template<bool A2A>
__global__ void __launch_bounds__(512, 1) groupNeighborKernel(const GroupArgs a)
{
    extern __shared__ __align__(16) uint8_t sGroupRaw[];
    constexpr int UNROLL = FB_NEIGHBOR_CHUNK / (32 * 16);
    constexpr uint32_t CB = FB_NEIGHBOR_CHUNK;
    const FbCommDev& c = a.comm;
    // the pieces and the in-edges behind them, into shared memory
    {
        const Vec16* src = reinterpret_cast<const Vec16*>(a.segs);
        Vec16* dst = reinterpret_cast<Vec16*>(sGroupRaw);
        const uint32_t vecs = (a.nSegs + FB_NEIGHBOR_EDGE_SLOTS(a.nEdges)) * 2;
        for (uint32_t i = threadIdx.x; i < vecs; i += blockDim.x) {
            dst[i] = src[i];
        }
        __syncthreads();
    }
    const RootedSeg* segs = reinterpret_cast<const RootedSeg*>(sGroupRaw);
    const NeighborEdge* edges = reinterpret_cast<const NeighborEdge*>(segs + a.nSegs);
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warpsPerCta = blockDim.x >> 5;
    const uint64_t warpStride = (uint64_t)gridDim.x * warpsPerCta;
    const uint64_t first = (uint64_t)blockIdx.x * warpsPerCta + (threadIdx.x >> 5);
    const uint64_t T = a.totalChunks;
    // one rank pulls its self-edges straight from its send
    const bool direct = c.nranks == 1;
    int cur = 0;
    if (!direct && (a.phase & GROUP_PHASE_LOCAL)) {
        uint8_t* const stage = c.heap[c.rank] + a.stageOff;
        const uint64_t units = (uint64_t)(A2A ? a.outDeg : min(a.outDeg, 1u)) * T;
        for (uint64_t u = first; u < units; u += warpStride) {
            const uint64_t k = u / T;
            const RootedChunk ch = rootedChunk<UNROLL>(segs, a.nSegs, cur, (uint32_t)(u - k * T));
            const uint8_t* const send =
              reinterpret_cast<const uint8_t*>(ch.sg->send) + (A2A ? k * ch.sg->stride : 0) + ch.off;
            rootedCopy<UNROLL>(stage + u * CB, send, ch.len, lane);
        }
    }
    BlockBarrier bar;
    bool ok = true;
    if (!a.noSync) {
        bar.load(c);
        ok = bar.sync(c);
    }
    if (ok && (a.phase & GROUP_PHASE_MOVE)) {
        // The barrier pairs CTA b of every rank only, so a staged chunk is
        // pulled by the warp whose index staged it on the source: staging
        // unit slot * T + g belongs to warp (slot * T + g) % warpStride on
        // every rank (same grid everywhere)
        for (uint32_t j = 0; j < a.nEdges; j++) {
            const NeighborEdge e = edges[j];
            const uint64_t slot = A2A ? e.idx : 0;
            const uint64_t g0 = (first + warpStride - (slot * T) % warpStride) % warpStride;
            for (uint64_t g = g0; g < T; g += warpStride) {
                const RootedChunk ch = rootedChunk<UNROLL>(segs, a.nSegs, cur, (uint32_t)g);
                const uint8_t* const src =
                  direct ? reinterpret_cast<const uint8_t*>(ch.sg->send) + slot * ch.sg->stride + ch.off
                         : c.heap[e.src] + a.stageOff + (slot * T + g) * CB;
                rootedCopy<UNROLL>(
                  reinterpret_cast<uint8_t*>(ch.sg->recv) + (uint64_t)j * ch.sg->stride + ch.off, src, ch.len, lane);
            }
        }
    }
    if (!a.noSync) {
        bar.sync(c);
        bar.store(c);
    }
}

cudaError_t launchGroupNeighbor(const GroupArgs& a, bool allToAll, int blocks, int threads, cudaStream_t s)
{
    const size_t smem = (size_t)(a.nSegs + FB_NEIGHBOR_EDGE_SLOTS(a.nEdges)) * sizeof(GroupSeg);
    if (allToAll) {
        groupNeighborKernel<true><<<blocks, threads, smem, s>>>(a);
    } else {
        groupNeighborKernel<false><<<blocks, threads, smem, s>>>(a);
    }
    return cudaGetLastError();
}

cudaError_t preloadNeighborKernels()
{
    cudaFuncAttributes attr;
    cudaError_t e = cudaSuccess;
#define FB_PRELOAD(k)                                                                                                  \
    if (e == cudaSuccess) {                                                                                            \
        e = cudaFuncGetAttributes(&attr, k);                                                                           \
    }
    FB_PRELOAD((groupNeighborKernel<false>))
    FB_PRELOAD((groupNeighborKernel<true>))
#undef FB_PRELOAD
    return e;
}

} // namespace fb
