// Segment-table walk shared by the grouped kernels (coll_reduce.cuh,
// coll_move.cu, coll_rooted.cu).  A launch serves a whole list of
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
// (Seg: GroupSeg, or RootedSeg of the rooted kinds)
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

// ---- the staged chunk walk of the rooted kinds (RootedSeg tables: grouped
// gather and scatter in coll_rooted.cu, grouped reduce in coll_reduce.cuh)

// `len` <= CB bytes, one warp: 16-byte vectors where both ends are 16-byte
// aligned, else 4-byte words where both are 4-byte aligned, else bytes
template<int UNROLL>
__device__ __forceinline__ void rootedCopy(uint8_t* d, const uint8_t* s, uint32_t len, uint32_t lane)
{
    constexpr uint32_t CB = 32u * UNROLL * 16;
    const uint32_t mis = (uint32_t)(((uintptr_t)d | (uintptr_t)s) & 15);
    if (mis == 0 && len == CB) {
        Vec16 v[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; u++) {
            v[u] = ldVecStream(s + (uint32_t)(u * 32 + lane) * 16);
        }
#pragma unroll
        for (int u = 0; u < UNROLL; u++) {
            stVec(d + (uint32_t)(u * 32 + lane) * 16, v[u]);
        }
        return;
    }
    uint32_t done = 0;
    if (mis == 0) {
        for (uint32_t i = lane; i < len / 16; i += 32) {
            stVec(d + i * 16, ldVecStream(s + i * 16));
        }
        done = len & ~15u;
    } else if ((mis & 3) == 0) {
        for (uint32_t i = lane; i < len / 4; i += 32) {
            reinterpret_cast<uint32_t*>(d)[i] = reinterpret_cast<const uint32_t*>(s)[i];
        }
        done = len & ~3u;
    }
    for (uint32_t i = done + lane; i < len; i += 32) {
        d[i] = s[i];
    }
}

// The table into shared memory (no barrier yet)
__device__ __forceinline__ const RootedSeg* rootedLoad(const GroupArgs& a, uint8_t* smem)
{
    const Vec16* src = reinterpret_cast<const Vec16*>(a.segs);
    Vec16* dst = reinterpret_cast<Vec16*>(smem);
    for (uint32_t i = threadIdx.x; i < a.nSegs * 2; i += blockDim.x) {
        dst[i] = src[i];
    }
    __syncthreads();
    return reinterpret_cast<const RootedSeg*>(smem);
}

// Chunk ch of a warp's walk: its piece and where in the piece it starts
struct RootedChunk
{
    const RootedSeg* sg;
    uint32_t off;
    uint32_t len;
};

template<int UNROLL>
__device__ __forceinline__ RootedChunk rootedChunk(const RootedSeg* segs, uint32_t nSegs, int& cur, uint32_t ch)
{
    constexpr uint32_t CB = 32u * UNROLL * 16;
    cur = groupSegOf(segs, nSegs, cur, ch);
    const RootedSeg* sg = segs + cur;
    const uint32_t off = (ch - sg->chunk0) * CB;
    return { sg, off, min(CB, sg->bytes - off) };
}

} // namespace fb
