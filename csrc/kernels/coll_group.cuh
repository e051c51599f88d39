// Segment-table walk shared by the grouped reduce-scatter and all-gather
// kernels (coll_reduce.cuh, coll_move.cu).  A launch serves a whole list of
// tensors: the table is copied to shared memory, CTA b of every rank meets at
// the entry and exit barriers, and the warps of the grid stride over the flat
// chunk space of the table (see GroupSeg in launch_api.h).
#pragma once

#include "fb_prims.cuh"
#include "launch_api.h"

namespace fb {

// Copies the table to shared memory and runs the entry barrier (or, with
// noSync, only publishes the table to the CTA).  False if a peer timed out.
__device__ __forceinline__ bool groupEnter(const GroupArgs& a,
                                           GroupSeg* sSegs,
                                           BlockBarrier& bar)
{
    const Vec16* src = reinterpret_cast<const Vec16*>(a.segs);
    Vec16* dst = reinterpret_cast<Vec16*>(sSegs);
    for (uint32_t i = threadIdx.x; i < a.nSegs * 2; i += blockDim.x) {
        dst[i] = src[i];
    }
    bar.epoch = 0;
    if (!a.noSync) {
        bar.load(a.comm);
        return bar.sync(a.comm);
    }
    __syncthreads();
    return true;
}

__device__ __forceinline__ void groupExit(const GroupArgs& a, BlockBarrier& bar)
{
    if (!a.noSync) {
        bar.sync(a.comm);
        bar.store(a.comm);
    }
}

// Index of the segment that owns chunk `ch`.  A warp's chunks ascend, so the
// answer is usually `cur` again; otherwise a binary search over chunk0.
// (Seg: GroupSeg, or RootedSeg of the grouped gather and scatter)
template<typename Seg>
__device__ __forceinline__ int groupSegOf(const Seg* s,
                                          uint32_t nSegs,
                                          int cur,
                                          uint32_t ch)
{
    if (s[cur].chunk0 <= ch && (cur + 1 == (int)nSegs || ch < s[cur + 1].chunk0)) {
        return cur;
    }
    int lo = 0;
    int hi = (int)nSegs - 1;
    while (lo < hi) {
        int mid = (lo + hi + 1) >> 1;
        if (s[mid].chunk0 <= ch) {
            lo = mid;
        } else {
            hi = mid - 1;
        }
    }
    return lo;
}

} // namespace fb
