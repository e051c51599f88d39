// Grouped neighbourhood v-collectives: many MPI_Neighbor_allgatherv /
// MPI_Neighbor_alltoallv calls over one graph, one launch per round (see
// NeighborVSeg in launch_api.h for the table and the steps).  Every rank
// stages the round's bytes of its send streams, and after the entry barrier
// pulls the round's bytes of each in-edge's recv stream from its source's
// slot.  Dtype-free: a byte copy at any alignment and any size.
#include "coll_group.cuh"

namespace fb {

// One side of a copy: a stream of the table, or a flat range whose byte `pos`
// is at flat + (pos - base)
struct VSide
{
    const NeighborVSeg* e; // null: the flat range
    uint32_t n;            // items of the stream
    uint8_t* flat;
    uint64_t base;
};

// The item of stream `e` (n items) that holds byte pos < its length
__device__ __forceinline__ uint32_t vItemOf(const NeighborVSeg* e, uint32_t n, uint64_t pos)
{
    uint32_t lo = 0;
    uint32_t hi = n - 1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (e[mid].off <= pos) {
            lo = mid;
        } else {
            hi = mid - 1;
        }
    }
    return lo;
}

// Where byte pos of side s lives, and `stop`, the first byte after it in
// another block.  m is the item of the last call (pos only grows).
__device__ __forceinline__ uint8_t* vAt(const VSide& s, uint32_t& m, uint64_t pos, uint64_t& stop)
{
    if (s.e == nullptr) {
        stop = ~(uint64_t)0;
        return s.flat + (pos - s.base);
    }
    while (s.e[m + 1].off <= pos) {
        m++;
    }
    stop = s.e[m + 1].off;
    return reinterpret_cast<uint8_t*>(s.e[m].addr) + (pos - s.e[m].off);
}

// Stream bytes [pos, end) from s to d, end - pos <= CB, end <= the length of
// every stream side: one warp
template<int UNROLL>
__device__ __forceinline__ void vCopy(const VSide& d, const VSide& s, uint64_t pos, uint64_t end, uint32_t lane)
{
    uint32_t md = d.e != nullptr ? vItemOf(d.e, d.n, pos) : 0;
    uint32_t ms = s.e != nullptr ? vItemOf(s.e, s.n, pos) : 0;
    while (pos < end) {
        uint64_t sd, ss;
        uint8_t* dp = vAt(d, md, pos, sd);
        const uint8_t* sp = vAt(s, ms, pos, ss);
        const uint64_t stop = min(end, min(sd, ss));
        rootedCopy<UNROLL>(dp, sp, (uint32_t)(stop - pos), lane);
        pos = stop;
    }
}

template<bool A2A>
__global__ void __launch_bounds__(512, 1) groupNeighborVKernel(const GroupArgs a)
{
    extern __shared__ __align__(16) uint8_t sGroupRaw[];
    constexpr int UNROLL = FB_NEIGHBOR_CHUNK / (32 * 16);
    constexpr uint64_t CB = FB_NEIGHBOR_CHUNK;
    const FbCommDev& c = a.comm;
    const uint32_t n = a.nSegs;
    const uint32_t sends = A2A ? a.outDeg : min(a.outDeg, 1u);
    {
        const Vec16* src = reinterpret_cast<const Vec16*>(a.segs);
        Vec16* dst = reinterpret_cast<Vec16*>(sGroupRaw);
        const uint32_t vecs = FB_NEIGHBOR_V_SLOTS(sends + a.nEdges, n, a.nEdges) * 2;
        for (uint32_t i = threadIdx.x; i < vecs; i += blockDim.x) {
            dst[i] = src[i];
        }
        __syncthreads();
    }
    const NeighborVSeg* tbl = reinterpret_cast<const NeighborVSeg*>(sGroupRaw);
    const NeighborEdge* edges = reinterpret_cast<const NeighborEdge*>(tbl + (uint64_t)(sends + a.nEdges) * (n + 1));
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warpsPerCta = blockDim.x >> 5;
    const uint64_t warpStride = (uint64_t)gridDim.x * warpsPerCta;
    const uint64_t first = (uint64_t)blockIdx.x * warpsPerCta + (threadIdx.x >> 5);
    const uint64_t C = a.totalChunks;
    const uint64_t W = a.vWidth;
    const bool direct = c.nranks == 1;
    if (!direct && (a.phase & GROUP_PHASE_LOCAL)) {
        uint8_t* const stage = c.heap[c.rank] + a.stageOff;
        for (uint64_t u = first; u < (uint64_t)sends * C; u += warpStride) {
            const uint64_t k = u / C;
            const NeighborVSeg* e = tbl + k * (n + 1);
            const uint64_t pos = a.vBase + (u - k * C) * CB;
            const uint64_t end = min(pos + CB, e[n].off);
            if (pos < end) {
                vCopy<UNROLL>(VSide{ nullptr, 0, stage + k * W, a.vBase }, VSide{ e, n, nullptr, 0 }, pos, end, lane);
            }
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
        // pulled by the warp whose index staged it on the source (same grid
        // and the same C everywhere)
        for (uint32_t j = 0; j < a.nEdges; j++) {
            const NeighborEdge ed = edges[j];
            const uint64_t slot = A2A ? ed.idx : 0;
            const NeighborVSeg* re = tbl + (uint64_t)(sends + j) * (n + 1);
            const NeighborVSeg* se = tbl + slot * (n + 1);
            const uint64_t len = direct ? min(re[n].off, se[n].off) : re[n].off;
            const VSide src = direct ? VSide{ se, n, nullptr, 0 }
                                     : VSide{ nullptr, 0, c.heap[ed.src] + a.stageOff + slot * W, a.vBase };
            const uint64_t c0 = (first + warpStride - (slot * C) % warpStride) % warpStride;
            for (uint64_t ch = c0; ch < C; ch += warpStride) {
                const uint64_t pos = a.vBase + ch * CB;
                const uint64_t end = min(pos + CB, len);
                if (pos >= end) {
                    break;
                }
                vCopy<UNROLL>(VSide{ re, n, nullptr, 0 }, src, pos, end, lane);
            }
        }
    }
    if (!a.noSync) {
        bar.sync(c);
        bar.store(c);
    }
}

cudaError_t launchGroupNeighborV(const GroupArgs& a, bool allToAll, int blocks, int threads, cudaStream_t s)
{
    const uint32_t sends = allToAll ? a.outDeg : std::min(a.outDeg, 1u);
    const size_t smem = (size_t)FB_NEIGHBOR_V_SLOTS(sends + a.nEdges, a.nSegs, a.nEdges) * sizeof(GroupSeg);
    if (allToAll) {
        groupNeighborVKernel<true><<<blocks, threads, smem, s>>>(a);
    } else {
        groupNeighborVKernel<false><<<blocks, threads, smem, s>>>(a);
    }
    return cudaGetLastError();
}

cudaError_t preloadNeighborVKernels()
{
    cudaFuncAttributes attr;
    cudaError_t e = cudaFuncGetAttributes(&attr, groupNeighborVKernel<false>);
    if (e == cudaSuccess) {
        e = cudaFuncGetAttributes(&attr, groupNeighborVKernel<true>);
    }
    return e;
}

} // namespace fb
