// Device snapshot kernels (sm_90a).
//
//  * snapshotDiffPushKernel — the fused north-star path: scan (optionally only
//    the dirty 4 KiB pages), compare the executor's memory with its base image,
//    apply the region's merge operation and store the result DIRECTLY into the
//    main GPU's snapshot image (a peer-mapped pointer over NVLink, or local).
//    No diff buffer, no serialisation, no separate apply kernel.
//    Fuses the reference's SnapshotData::diffWithDirtyRegions +
//    SnapshotMergeRegion::addDiffs + diffArrayRegions + SnapshotClient push +
//    SnapshotData::applyDiff (src/util/snapshot.cpp:30-97,402-492,524-578,
//    652-824; src/snapshot/SnapshotClient.cpp:76-171).
//  * dirtyScanKernel — GPU dirty-page detection by compare-with-base (there are
//    no page-fault trackers on a GPU; replaces src/util/dirty.cpp trackers).
//  * flagsOrKernel — mergeDirtyPages (src/util/memory.cpp:15-39).
//  * chunkRunsKernel — turns 128-byte chunk flags into (offset,length) diff
//    descriptors (coarse equivalent of diffArrayRegions' run detection).
//  * snapshotApplyKernel — applies a packed diff list to a device image
//    (SnapshotData::applyDiffs for diffs that arrive as descriptors).
//
// Semantics kept from the reference: Bytewise stores exactly the bytes that
// differ (byte-exact merge safety between concurrent writers), XOR merges
// orig^updated with an atomic xor, typed regions merge arrays of scalars
// (Sum: +=new-old, Subtract: -=(old-new), Product: *=new/old, Max/Min) with
// the rules of faabric/util/reduce_ops.h (see snapAdd ... snapQuotient).
#include "snapshot_kernels.cuh"

#include "fb_atomics.cuh"

#include <type_traits>

namespace fb {

static constexpr uint32_t PAGE = 4096;

// ----------------------------------------------------------------------------
// helpers
// ----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t byteDiffMask(uint32_t a, uint32_t b)
{
    // bit k set when byte k of a and b differ
    uint32_t x = a ^ b;
    uint32_t m = 0;
    m |= (x & 0x000000ffu) ? 1u : 0u;
    m |= (x & 0x0000ff00u) ? 2u : 0u;
    m |= (x & 0x00ff0000u) ? 4u : 0u;
    m |= (x & 0xff000000u) ? 8u : 0u;
    return m;
}

// Store only the differing bytes of word `m` (mask from byteDiffMask)
__device__ __forceinline__ void storeMaskedWord(uint8_t* dst,
                                                uint32_t m,
                                                uint32_t mask)
{
    if (mask == 0xf) {
        *reinterpret_cast<uint32_t*>(dst) = m;
    } else {
#pragma unroll
        for (int b = 0; b < 4; b++) {
            if (mask & (1u << b)) {
                dst[b] = (uint8_t)(m >> (8 * b));
            }
        }
    }
}

// Binary search: first region whose end is > pos.  Regions are sorted by
// offset and non-overlapping (the host fills the gaps before the launch).
__device__ __forceinline__ int firstRegionAfter(const FbMergeRegionDev* r,
                                                int n,
                                                uint64_t pos,
                                                uint64_t size)
{
    int lo = 0, hi = n;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        uint64_t end = r[mid].length == 0 ? size : r[mid].offset + r[mid].length;
        if (end > pos) {
            hi = mid;
        } else {
            lo = mid + 1;
        }
    }
    return lo;
}

// ----------------------------------------------------------------------------
// Bytewise / XOR segment, processed by one warp
// ----------------------------------------------------------------------------
template<bool XOR>
__device__ __forceinline__ uint32_t warpSegment(const SnapDiffArgs& a,
                                                uint64_t beg,
                                                uint64_t end,
                                                int lane,
                                                uint32_t& chunkAny)
{
    uint32_t diffBytes = 0;
    // unaligned head / tail bytes: one lane per byte
    uint64_t vb = (beg + 15) & ~(uint64_t)15;
    uint64_t ve = end & ~(uint64_t)15;
    if (vb > ve) {
        vb = ve = end; // segment shorter than one aligned vector
        // all bytes handled by the "head" loop below
        for (uint64_t p = beg + lane; p < end; p += 32) {
            uint8_t o = a.orig[p], m = a.mem[p];
            if (o != m) {
                diffBytes++;
                if (XOR) {
                    // byte-granular xor through the containing aligned word
                    uint64_t w = p & ~(uint64_t)3;
                    redXorSys(reinterpret_cast<uint32_t*>(a.dst + w),
                              (uint32_t)(o ^ m) << (8 * (p & 3)));
                } else {
                    a.dst[p] = m;
                }
                if (a.updateBase) {
                    a.origW[p] = m;
                }
                if (a.chunkFlags != nullptr) {
                    a.chunkFlags[p >> 7] = 1; // benign same-value race
                }
            }
        }
        chunkAny |= diffBytes;
        return diffBytes;
    }
    for (uint64_t p = beg + lane; p < vb; p += 32) {
        uint8_t o = a.orig[p], m = a.mem[p];
        if (o != m) {
            diffBytes++;
            if (XOR) {
                uint64_t w = p & ~(uint64_t)3;
                redXorSys(reinterpret_cast<uint32_t*>(a.dst + w),
                          (uint32_t)(o ^ m) << (8 * (p & 3)));
            } else {
                a.dst[p] = m;
            }
            if (a.updateBase) {
                a.origW[p] = m;
            }
            if (a.chunkFlags != nullptr) {
                a.chunkFlags[p >> 7] = 1;
            }
        }
    }
    for (uint64_t p = ve + lane; p < end; p += 32) {
        uint8_t o = a.orig[p], m = a.mem[p];
        if (o != m) {
            diffBytes++;
            if (XOR) {
                uint64_t w = p & ~(uint64_t)3;
                redXorSys(reinterpret_cast<uint32_t*>(a.dst + w),
                          (uint32_t)(o ^ m) << (8 * (p & 3)));
            } else {
                a.dst[p] = m;
            }
            if (a.updateBase) {
                a.origW[p] = m;
            }
            if (a.chunkFlags != nullptr) {
                a.chunkFlags[p >> 7] = 1;
            }
        }
    }
    // aligned body: 2 vectors per lane in flight
    const uint64_t nVec = (ve - vb) >> 4;
    for (uint64_t i = lane; i < nVec; i += 64) {
        uint64_t p0 = vb + (i << 4);
        bool has1 = (i + 32) < nVec;
        uint64_t p1 = has1 ? p0 + 512 : p0;
        Vec16 o0 = ldVecStream(a.orig + p0);
        Vec16 m0 = ldVecStream(a.mem + p0);
        Vec16 o1 = ldVecStream(a.orig + p1);
        Vec16 m1 = ldVecStream(a.mem + p1);
#pragma unroll
        for (int h = 0; h < 2; h++) {
            if (h == 1 && !has1) {
                break;
            }
            const Vec16& o = h ? o1 : o0;
            const Vec16& m = h ? m1 : m0;
            const uint64_t p = h ? p1 : p0;
            uint32_t mk[4];
            uint32_t all = 0xf, any = 0;
#pragma unroll
            for (int w = 0; w < 4; w++) {
                mk[w] = byteDiffMask(o.w[w], m.w[w]);
                all &= mk[w];
                any |= mk[w];
            }
            if (any) {
                diffBytes += __popc(mk[0]) + __popc(mk[1]) + __popc(mk[2]) +
                             __popc(mk[3]);
                if (XOR) {
#pragma unroll
                    for (int w = 0; w < 4; w++) {
                        if (mk[w]) {
                            redXorSys(
                              reinterpret_cast<uint32_t*>(a.dst + p + 4 * w),
                              o.w[w] ^ m.w[w]);
                        }
                    }
                } else if (all == 0xf) {
                    stVec(a.dst + p, m);
                } else {
#pragma unroll
                    for (int w = 0; w < 4; w++) {
                        if (mk[w]) {
                            storeMaskedWord(a.dst + p + 4 * w, m.w[w], mk[w]);
                        }
                    }
                }
                if (a.updateBase) {
                    stVec(a.origW + p, m);
                }
                if (a.chunkFlags != nullptr) {
                    a.chunkFlags[p >> 7] = 1; // benign same-value race
                }
            }
        }
    }
    chunkAny |= diffBytes;
    return diffBytes;
}

// ----------------------------------------------------------------------------
// Typed scalar merge
// ----------------------------------------------------------------------------
template<typename T>
__device__ __forceinline__ T loadUnaligned(const uint8_t* p)
{
    T v;
    uint8_t* b = reinterpret_cast<uint8_t*>(&v);
#pragma unroll
    for (int i = 0; i < (int)sizeof(T); i++) {
        b[i] = p[i];
    }
    return v;
}

template<typename T>
__device__ __forceinline__ void storeUnaligned(uint8_t* p, T v)
{
    const uint8_t* b = reinterpret_cast<const uint8_t*>(&v);
#pragma unroll
    for (int i = 0; i < (int)sizeof(T); i++) {
        p[i] = b[i];
    }
}

// RMW of a scalar that is NOT naturally aligned (an application may declare a
// typed merge region at any byte offset), atomic with respect to the other
// GPUs merging into the same image: one 128-bit compare-and-swap on the
// enclosing 16-byte block (SASS ATOMG.E.CAS.128.STRONG.SYS) recomputes the
// scalar from the bytes it observed.  A scalar that crosses a 16-byte
// boundary has no single atomic that covers it: returns false and the caller
// falls back to load / modify / store (last writer wins for that scalar).
template<typename T, typename F>
__device__ __forceinline__ bool atomicRmwUnalignedSys(uint8_t* d, F f)
{
    const uintptr_t addr = (uintptr_t)d;
    const int shift = (int)(addr & 15);
    if (shift + (int)sizeof(T) > 16) {
        return false;
    }
    uint64_t* blk = reinterpret_cast<uint64_t*>(addr & ~(uintptr_t)15);
    uint64_t o0 = *reinterpret_cast<volatile uint64_t*>(blk);
    uint64_t o1 = *reinterpret_cast<volatile uint64_t*>(blk + 1);
    while (true) {
        uint8_t bytes[16];
        memcpy(bytes, &o0, 8);
        memcpy(bytes + 8, &o1, 8);
        T cur;
        memcpy(&cur, bytes + shift, sizeof(T));
        T nv = f(cur);
        memcpy(bytes + shift, &nv, sizeof(T));
        uint64_t n0;
        uint64_t n1;
        memcpy(&n0, bytes, 8);
        memcpy(&n1, bytes + 8, 8);
        uint64_t r0;
        uint64_t r1;
        if (cas128Sys(blk, o0, o1, n0, n1, r0, r1)) {
            return true;
        }
        o0 = r0;
        o1 = r1;
    }
}

// Typed merge rules, the device form of faabric/util/reduce_ops.h (reduceSum,
// reduceSub, reduceProd, reduceMax, reduceMin, snapshotQuotient): integers
// wrap, computed in the unsigned type of the same width; float Max/Min are
// fmax/fmin as in Reducer (fb_prims.cuh), so a NaN operand is ignored and -0
// orders below +0 whichever writer lands first.
template<typename T>
__device__ __forceinline__ T snapAdd(T a, T b)
{
    if constexpr (std::is_integral_v<T>) {
        using U = std::make_unsigned_t<T>;
        return (T)(U)((U)a + (U)b);
    } else {
        return a + b;
    }
}

template<typename T>
__device__ __forceinline__ T snapSub(T a, T b)
{
    if constexpr (std::is_integral_v<T>) {
        using U = std::make_unsigned_t<T>;
        return (T)(U)((U)a - (U)b);
    } else {
        return a - b;
    }
}

template<typename T>
__device__ __forceinline__ T snapMul(T a, T b)
{
    if constexpr (std::is_integral_v<T>) {
        using U = std::make_unsigned_t<T>;
        return (T)(U)((U)a * (U)b);
    } else {
        return a * b;
    }
}

template<typename T>
__device__ __forceinline__ T snapMax(T a, T b)
{
    if constexpr (std::is_same_v<T, float>) {
        return fmaxf(a, b);
    } else if constexpr (std::is_same_v<T, double>) {
        return fmax(a, b);
    } else {
        return a > b ? a : b;
    }
}

template<typename T>
__device__ __forceinline__ T snapMin(T a, T b)
{
    if constexpr (std::is_same_v<T, float>) {
        return fminf(a, b);
    } else if constexpr (std::is_same_v<T, double>) {
        return fmin(a, b);
    } else {
        return a < b ? a : b;
    }
}

// Product factor for a value that went from o to n: IEEE n / o for floats;
// for integers 0 when o is 0, a wrapping negation when o is -1, otherwise the
// truncated quotient
template<typename T>
__device__ __forceinline__ T snapQuotient(T n, T o)
{
    if constexpr (std::is_integral_v<T>) {
        if (o == 0) {
            return 0;
        }
        if (o == (T)-1) {
            return snapSub((T)0, n);
        }
        return n / o;
    } else {
        return n / o;
    }
}

// Merge one scalar.  Returns true if a diff was produced.
template<typename T>
__device__ __forceinline__ bool mergeScalar(const SnapDiffArgs& a,
                                            uint64_t off,
                                            int op)
{
    T o = loadUnaligned<T>(a.orig + off);
    T m = loadUnaligned<T>(a.mem + off);
    if (o == m) {
        return false;
    }
    uint8_t* d = a.dst + off;
    const bool aligned = ((uintptr_t)d % sizeof(T)) == 0;
    constexpr bool isInt = std::is_integral_v<T>;
    switch (op) {
        case FB_MERGE_SUM: {
            T delta = snapSub(m, o);
            if (aligned) {
                redAddSys(reinterpret_cast<T*>(d), delta);
            } else {
                if (!atomicRmwUnalignedSys<T>(d, [delta](T c) { return snapAdd(c, delta); })) {
                    storeUnaligned<T>(d, snapAdd(loadUnaligned<T>(d), delta));
                }
            }
            break;
        }
        case FB_MERGE_SUBTRACT: {
            T diff = snapSub(o, m); // applied as main - diff
            if (aligned) {
                T neg;
                if constexpr (isInt) {
                    neg = snapSub((T)0, diff);
                } else {
                    neg = -diff;
                }
                redAddSys(reinterpret_cast<T*>(d), neg);
            } else {
                if (!atomicRmwUnalignedSys<T>(d, [diff](T c) { return snapSub(c, diff); })) {
                    storeUnaligned<T>(d, snapSub(loadUnaligned<T>(d), diff));
                }
            }
            break;
        }
        case FB_MERGE_PRODUCT: {
            T q = snapQuotient(m, o);
            if (aligned) {
                atomicRmwSys<T>(reinterpret_cast<T*>(d),
                                [q](T c) { return snapMul(c, q); });
            } else {
                if (!atomicRmwUnalignedSys<T>(d, [q](T c) { return snapMul(c, q); })) {
                    storeUnaligned<T>(d, snapMul(loadUnaligned<T>(d), q));
                }
            }
            break;
        }
        case FB_MERGE_MAX: {
            if (aligned) {
                if constexpr (isInt) {
                    redMaxSys(reinterpret_cast<T*>(d), m);
                } else {
                    atomicRmwSys<T>(reinterpret_cast<T*>(d),
                                    [m](T c) { return snapMax(c, m); });
                }
            } else {
                if (!atomicRmwUnalignedSys<T>(d, [m](T c) { return snapMax(c, m); })) {
                    storeUnaligned<T>(d, snapMax(loadUnaligned<T>(d), m));
                }
            }
            break;
        }
        case FB_MERGE_MIN: {
            if (aligned) {
                if constexpr (isInt) {
                    redMinSys(reinterpret_cast<T*>(d), m);
                } else {
                    atomicRmwSys<T>(reinterpret_cast<T*>(d),
                                    [m](T c) { return snapMin(c, m); });
                }
            } else {
                if (!atomicRmwUnalignedSys<T>(d, [m](T c) { return snapMin(c, m); })) {
                    storeUnaligned<T>(d, snapMin(loadUnaligned<T>(d), m));
                }
            }
            break;
        }
        default:
            return false;
    }
    if (a.updateBase) {
        storeUnaligned<T>(a.origW + off, m);
    }
    if (a.chunkFlags != nullptr) {
        a.chunkFlags[off >> 7] = 1;
        a.chunkFlags[(off + sizeof(T) - 1) >> 7] = 1;
    }
    return true;
}

__device__ __forceinline__ bool pageDirty(const SnapDiffArgs& a, uint64_t page)
{
    return a.dirtyPages == nullptr || a.dirtyPages[page] != 0;
}

// Typed region: the scalars of `reg` (an array of floor(length / size) of
// them, cut at the image end) whose first byte lies in [pBeg, pEnd), one lane
// per scalar.  A scalar is merged when its first or its last page is dirty.
__device__ __forceinline__ uint32_t warpTyped(const SnapDiffArgs& a,
                                              const FbMergeRegionDev& reg,
                                              uint64_t pBeg,
                                              uint64_t pEnd,
                                              uint64_t rEnd,
                                              int lane,
                                              uint32_t& pageAny)
{
    const uint32_t sz =
      (reg.dataType == FB_SNAP_INT || reg.dataType == FB_SNAP_FLOAT) ? 4 : 8;
    const uint64_t first = pBeg > reg.offset ? (pBeg - reg.offset + sz - 1) / sz : 0;
    const uint64_t count = (rEnd - reg.offset) / sz;
    uint32_t bytes = 0;
    for (uint64_t k = first + lane; k < count; k += 32) {
        const uint64_t off = reg.offset + k * sz;
        if (off >= pEnd) {
            break;
        }
        const uint64_t lastPage = (off + sz - 1) / PAGE;
        if (!pageDirty(a, off / PAGE) && !pageDirty(a, lastPage)) {
            continue;
        }
        bool d = false;
        switch (reg.dataType) {
            case FB_SNAP_INT:
                d = mergeScalar<int32_t>(a, off, reg.op);
                break;
            case FB_SNAP_LONG:
                d = mergeScalar<int64_t>(a, off, reg.op);
                break;
            case FB_SNAP_FLOAT:
                d = mergeScalar<float>(a, off, reg.op);
                break;
            case FB_SNAP_DOUBLE:
                d = mergeScalar<double>(a, off, reg.op);
                break;
            default:
                break;
        }
        if (d) {
            bytes += sz;
            // the first page is stamped with the page's other diffs
            if (a.pageStampOut != nullptr && lastPage != off / PAGE) {
                a.pageStampOut[lastPage] = a.pageStamp;
            }
        }
    }
    pageAny |= bytes;
    return bytes;
}

// ----------------------------------------------------------------------------
// The fused kernel
// ----------------------------------------------------------------------------
__global__ void __launch_bounds__(512, 2) snapshotDiffPushKernel(
  const SnapDiffArgs a)
{
    const int lane = threadIdx.x & 31;
    const uint64_t warpId =
      ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t nWarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    const uint64_t nPages = (a.size + PAGE - 1) / PAGE;

    uint32_t diffBytes = 0;
    uint32_t dirtyPagesSeen = 0;

    // ---- page-major, one warp per page: Bytewise / XOR segments of the page
    // and the typed scalars that start in it, so every diff that starts in a
    // page is seen by one warp and the page is counted once ----
    for (uint64_t page = warpId; page < nPages; page += nWarps) {
        const bool dirty = pageDirty(a, page);
        // a scalar starting on a clean page is merged when its last page is dirty
        if (!dirty && !(a.nTyped > 0 && page + 1 < nPages && pageDirty(a, page + 1))) {
            continue;
        }
        const uint64_t pBeg = page * PAGE;
        const uint64_t pEnd = min(a.size, pBeg + PAGE);
        uint32_t pageAny = 0;
        int r = firstRegionAfter(a.regions, a.nRegions, pBeg, a.size);
        while (r < a.nRegions) {
            const FbMergeRegionDev reg = a.regions[r];
            if (reg.offset >= pEnd) {
                break;
            }
            const uint64_t rEnd =
              reg.length == 0 ? a.size : min(a.size, reg.offset + reg.length);
            const uint64_t sBeg = max(pBeg, reg.offset);
            const uint64_t sEnd = min(pEnd, rEnd);
            if (sBeg < sEnd) {
                if (reg.op == FB_MERGE_BYTEWISE) {
                    if (dirty) {
                        diffBytes +=
                          warpSegment<false>(a, sBeg, sEnd, lane, pageAny);
                    }
                } else if (reg.op == FB_MERGE_XOR) {
                    if (dirty) {
                        diffBytes +=
                          warpSegment<true>(a, sBeg, sEnd, lane, pageAny);
                    }
                } else if (reg.op != FB_MERGE_IGNORE) {
                    diffBytes += warpTyped(a, reg, pBeg, pEnd, rEnd, lane, pageAny);
                }
            }
            r++;
        }
        if (__any_sync(0xffffffffu, pageAny != 0) && lane == 0) {
            dirtyPagesSeen++;
            if (a.pageFlagsOut != nullptr) {
                a.pageFlagsOut[page] = 1;
            }
            if (a.pageStampOut != nullptr) {
                a.pageStampOut[page] = a.pageStamp; // same value from every writer
            }
        }
    }

    // ---- statistics: one atomic per warp ----
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        diffBytes += __shfl_xor_sync(0xffffffffu, diffBytes, s);
    }
    if (lane == 0 && a.stats != nullptr) {
        if (diffBytes) {
            atomicAdd(reinterpret_cast<unsigned long long*>(&a.stats[0]),
                      (unsigned long long)diffBytes);
        }
        if (dirtyPagesSeen) {
            atomicAdd(reinterpret_cast<unsigned long long*>(&a.stats[1]),
                      (unsigned long long)dirtyPagesSeen);
        }
    }
    // Make the pushed bytes visible system-wide before the kernel retires so a
    // following cross-GPU signal / barrier orders after them
    __threadfence_system();
}

cudaError_t launchSnapshotDiffPush(const SnapDiffArgs& a,
                                   int blocks,
                                   cudaStream_t s)
{
    snapshotDiffPushKernel<<<blocks, 512, 0, s>>>(a);
    return cudaGetLastError();
}

// ----------------------------------------------------------------------------
// Page-granular synchronisation of two images (incremental THREADS fork-join):
// pageSync folds an executor's memory into the main image and stamps what
// changed; pagePull brings a stale copy up to date from the stamps.  One warp
// per 4 KiB page, 16-byte vectors, 8 per lane.
// ----------------------------------------------------------------------------
__device__ __forceinline__ void copyPage(const uint8_t* src, uint8_t* dst1, uint8_t* dst2, uint64_t pBeg, uint64_t nBytes, int lane)
{
    const uint64_t nVec = nBytes >> 4;
    const uint4* s4 = reinterpret_cast<const uint4*>(src + pBeg);
    uint4* d4 = reinterpret_cast<uint4*>(dst1 + pBeg);
    uint4* e4 = dst2 != nullptr ? reinterpret_cast<uint4*>(dst2 + pBeg) : nullptr;
    for (uint64_t i = lane; i < nVec; i += 32) {
        uint4 v = s4[i];
        d4[i] = v;
        if (e4 != nullptr) {
            e4[i] = v;
        }
    }
    for (uint64_t p = (nVec << 4) + lane; p < nBytes; p += 32) {
        uint8_t b = src[pBeg + p];
        dst1[pBeg + p] = b;
        if (dst2 != nullptr) {
            dst2[pBeg + p] = b;
        }
    }
}

__global__ void __launch_bounds__(512, 2) pageSyncKernel(const uint8_t* src,
                                                         uint8_t* dst,
                                                         uint32_t* pageStamps,
                                                         uint32_t stamp,
                                                         uint64_t size,
                                                         uint64_t* stats)
{
    const int lane = threadIdx.x & 31;
    const uint64_t warpId = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t nWarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    const uint64_t nPages = (size + PAGE - 1) / PAGE;
    uint32_t copied = 0;
    for (uint64_t page = warpId; page < nPages; page += nWarps) {
        const uint64_t pBeg = page * PAGE;
        const uint64_t nBytes = min((uint64_t)PAGE, size - pBeg);
        const uint64_t nVec = nBytes >> 4;
        const uint4* s4 = reinterpret_cast<const uint4*>(src + pBeg);
        const uint4* d4 = reinterpret_cast<const uint4*>(dst + pBeg);
        bool differ = false;
        for (uint64_t i = lane; i < nVec; i += 32) {
            uint4 a = s4[i], b = d4[i];
            differ |= (a.x != b.x) | (a.y != b.y) | (a.z != b.z) | (a.w != b.w);
        }
        for (uint64_t p = (nVec << 4) + lane; p < nBytes; p += 32) {
            differ |= src[pBeg + p] != dst[pBeg + p];
        }
        if (__any_sync(0xffffffffu, differ)) {
            copyPage(src, dst, nullptr, pBeg, nBytes, lane);
            if (lane == 0) {
                if (pageStamps != nullptr) {
                    pageStamps[page] = stamp;
                }
                copied++;
            }
        }
    }
    if (lane == 0 && copied != 0 && stats != nullptr) {
        atomicAdd(reinterpret_cast<unsigned long long*>(&stats[0]), (unsigned long long)copied);
    }
}

__global__ void __launch_bounds__(512, 2) pagePullKernel(const uint8_t* src,
                                                         uint8_t* dst1,
                                                         uint8_t* dst2,
                                                         const uint32_t* pageStamps,
                                                         uint32_t since,
                                                         uint64_t size,
                                                         uint64_t* stats)
{
    const int lane = threadIdx.x & 31;
    const uint64_t warpId = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t nWarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    const uint64_t nPages = (size + PAGE - 1) / PAGE;
    uint32_t copied = 0;
    // each lane looks at one stamp of a group of 32 pages, the warp then copies
    // the flagged ones one after the other
    for (uint64_t group = warpId * 32; group < nPages; group += nWarps * 32) {
        const uint64_t mine = group + lane;
        const bool want = mine < nPages && pageStamps[mine] > since;
        uint32_t mask = __ballot_sync(0xffffffffu, want);
        while (mask != 0) {
            const int k = __ffs(mask) - 1;
            mask &= mask - 1;
            const uint64_t pBeg = (group + k) * PAGE;
            copyPage(src, dst1, dst2, pBeg, min((uint64_t)PAGE, size - pBeg), lane);
            copied++;
        }
    }
    if (lane == 0 && copied != 0 && stats != nullptr) {
        atomicAdd(reinterpret_cast<unsigned long long*>(&stats[0]), (unsigned long long)copied);
    }
}

// out[k] = page pages[k] of newMem, XORed with the same page of oldImg when
// xorMode: what the delta codec (util/delta.h) sends for a changed page
__global__ void __launch_bounds__(512, 2) pageGatherKernel(const uint8_t* oldImg,
                                                           const uint8_t* newMem,
                                                           const uint32_t* pages,
                                                           uint32_t nListed,
                                                           uint64_t size,
                                                           int xorMode,
                                                           uint8_t* out)
{
    const int lane = threadIdx.x & 31;
    const uint64_t warpId = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t nWarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t k = warpId; k < nListed; k += nWarps) {
        const uint64_t pBeg = (uint64_t)pages[k] * PAGE;
        if (pBeg >= size) {
            continue;
        }
        const uint64_t nBytes = min((uint64_t)PAGE, size - pBeg);
        const uint64_t nVec = nBytes >> 4;
        const uint4* n4 = reinterpret_cast<const uint4*>(newMem + pBeg);
        const uint4* o4 = reinterpret_cast<const uint4*>(oldImg + pBeg);
        uint4* d4 = reinterpret_cast<uint4*>(out + k * PAGE);
        for (uint64_t i = lane; i < nVec; i += 32) {
            uint4 v = n4[i];
            if (xorMode) {
                uint4 o = o4[i];
                v.x ^= o.x;
                v.y ^= o.y;
                v.z ^= o.z;
                v.w ^= o.w;
            }
            d4[i] = v;
        }
        for (uint64_t p = (nVec << 4) + lane; p < nBytes; p += 32) {
            uint8_t b = newMem[pBeg + p];
            out[k * PAGE + p] = xorMode ? (uint8_t)(b ^ oldImg[pBeg + p]) : b;
        }
    }
}

cudaError_t launchPageGather(const uint8_t* oldImg,
                             const uint8_t* newMem,
                             const uint32_t* pages,
                             uint32_t nListed,
                             uint64_t size,
                             int xorMode,
                             uint8_t* out,
                             int blocks,
                             cudaStream_t s)
{
    pageGatherKernel<<<blocks, 512, 0, s>>>(oldImg, newMem, pages, nListed, size, xorMode, out);
    return cudaGetLastError();
}

cudaError_t launchPageSync(const uint8_t* src,
                           uint8_t* dst,
                           uint32_t* pageStamps,
                           uint32_t stamp,
                           uint64_t size,
                           uint64_t* stats,
                           int blocks,
                           cudaStream_t s)
{
    pageSyncKernel<<<blocks, 512, 0, s>>>(src, dst, pageStamps, stamp, size, stats);
    return cudaGetLastError();
}

cudaError_t launchPagePull(const uint8_t* src,
                           uint8_t* dst1,
                           uint8_t* dst2,
                           const uint32_t* pageStamps,
                           uint32_t since,
                           uint64_t size,
                           uint64_t* stats,
                           int blocks,
                           cudaStream_t s)
{
    pagePullKernel<<<blocks, 512, 0, s>>>(src, dst1, dst2, pageStamps, since, size, stats);
    return cudaGetLastError();
}

// ----------------------------------------------------------------------------
// Dirty page detection by compare-with-base: one warp per 4 KiB page with an
// early exit once a difference is seen.
// ----------------------------------------------------------------------------
__global__ void __launch_bounds__(512, 2) dirtyScanKernel(const uint8_t* mem,
                                                          const uint8_t* base,
                                                          uint64_t size,
                                                          uint8_t* pageFlags,
                                                          uint64_t* nDirty)
{
    const int lane = threadIdx.x & 31;
    const uint64_t warpId =
      ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t nWarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    const uint64_t nPages = (size + PAGE - 1) / PAGE;
    uint32_t found = 0;
    for (uint64_t page = warpId; page < nPages; page += nWarps) {
        const uint64_t pBeg = page * PAGE;
        const uint64_t pEnd = min(size, pBeg + PAGE);
        const uint64_t nVec = (pEnd - pBeg) >> 4;
        bool diff = false;
        // rounds of 2 vectors per lane; stop at the first differing round
        for (uint64_t b = 0; b < nVec && !diff; b += 64) {
            uint64_t i = b + lane;
            uint32_t x = 0;
            if (i < nVec) {
                uint64_t p0 = pBeg + (i << 4);
                uint64_t p1 = (i + 32 < nVec) ? p0 + 512 : p0;
                Vec16 a0 = ldVecStream(mem + p0);
                Vec16 b0 = ldVecStream(base + p0);
                Vec16 a1 = ldVecStream(mem + p1);
                Vec16 b1 = ldVecStream(base + p1);
                x = (a0.w[0] ^ b0.w[0]) | (a0.w[1] ^ b0.w[1]) |
                    (a0.w[2] ^ b0.w[2]) | (a0.w[3] ^ b0.w[3]) |
                    (a1.w[0] ^ b1.w[0]) | (a1.w[1] ^ b1.w[1]) |
                    (a1.w[2] ^ b1.w[2]) | (a1.w[3] ^ b1.w[3]);
            }
            diff = __any_sync(0xffffffffu, x != 0);
        }
        diff = __any_sync(0xffffffffu, diff);
        if (!diff) {
            // trailing bytes of a partial last page
            for (uint64_t p = pBeg + (nVec << 4) + lane; p < pEnd; p += 32) {
                if (mem[p] != base[p]) {
                    diff = true;
                }
            }
            diff = __any_sync(0xffffffffu, diff);
        }
        if (lane == 0) {
            pageFlags[page] = diff ? 1 : 0;
            found += diff ? 1 : 0;
        }
    }
    if (lane == 0 && found && nDirty != nullptr) {
        atomicAdd(reinterpret_cast<unsigned long long*>(nDirty),
                  (unsigned long long)found);
    }
}

cudaError_t launchDirtyScan(const uint8_t* mem,
                            const uint8_t* base,
                            uint64_t size,
                            uint8_t* pageFlags,
                            uint64_t* nDirty,
                            int blocks,
                            cudaStream_t s)
{
    dirtyScanKernel<<<blocks, 512, 0, s>>>(mem, base, size, pageFlags, nDirty);
    return cudaGetLastError();
}

// dst[i] |= src[i]
__global__ void flagsOrKernel(uint8_t* dst, const uint8_t* src, uint64_t n)
{
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        dst[i] |= src[i];
    }
}

cudaError_t launchFlagsOr(uint8_t* dst,
                          const uint8_t* src,
                          uint64_t n,
                          cudaStream_t s)
{
    int blocks = (int)((n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024);
    if (blocks < 1) {
        blocks = 1;
    }
    flagsOrKernel<<<blocks, 256, 0, s>>>(dst, src, n);
    return cudaGetLastError();
}

// ----------------------------------------------------------------------------
// Chunk flags -> run descriptors.  A run starts at a set flag whose predecessor
// is clear; the thread owning the start walks to the end of the run.  Runs are
// appended with an atomic cursor (order is not significant: the host sorts).
// ----------------------------------------------------------------------------
__global__ void chunkRunsKernel(const uint8_t* flags,
                                uint64_t nChunks,
                                uint32_t chunkBytes,
                                uint64_t totalBytes,
                                FbDiffDesc* out,
                                uint32_t maxOut,
                                uint32_t* count)
{
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (; i < nChunks; i += stride) {
        if (flags[i] && (i == 0 || !flags[i - 1])) {
            uint64_t j = i + 1;
            while (j < nChunks && flags[j]) {
                j++;
            }
            uint32_t slot = atomicAdd(count, 1u);
            if (slot < maxOut) {
                FbDiffDesc d;
                d.offset = i * chunkBytes;
                uint64_t e = min(j * (uint64_t)chunkBytes, totalBytes);
                d.length = e - d.offset;
                d.dataType = FB_SNAP_RAW;
                d.op = FB_MERGE_BYTEWISE;
                out[slot] = d;
            }
        }
    }
}

cudaError_t launchChunkRuns(const uint8_t* flags,
                            uint64_t nChunks,
                            uint32_t chunkBytes,
                            uint64_t totalBytes,
                            FbDiffDesc* out,
                            uint32_t maxOut,
                            uint32_t* count,
                            cudaStream_t s)
{
    int blocks = (int)((nChunks + 255) / 256 < 2048 ? (nChunks + 255) / 256 : 2048);
    if (blocks < 1) {
        blocks = 1;
    }
    chunkRunsKernel<<<blocks, 256, 0, s>>>(
      flags, nChunks, chunkBytes, totalBytes, out, maxOut, count);
    return cudaGetLastError();
}

// ----------------------------------------------------------------------------
// Apply a packed diff list: one CTA per descriptor (grid-strided).
// data for descriptor i lives at blob + dataOff[i].
// ----------------------------------------------------------------------------
__global__ void __launch_bounds__(256) snapshotApplyKernel(
  uint8_t* image,
  uint64_t imageSize,
  const FbDiffDesc* descs,
  const uint64_t* dataOff,
  const uint8_t* blob,
  uint32_t nDescs)
{
    for (uint32_t di = blockIdx.x; di < nDescs; di += gridDim.x) {
        const FbDiffDesc d = descs[di];
        const uint8_t* src = blob + dataOff[di];
        if (d.offset >= imageSize) {
            continue;
        }
        uint64_t len = min(d.length, imageSize - d.offset);
        uint8_t* dst = image + d.offset;
        switch (d.op) {
            case FB_MERGE_IGNORE:
                break;
            case FB_MERGE_BYTEWISE:
                for (uint64_t i = threadIdx.x; i < len; i += blockDim.x) {
                    dst[i] = src[i];
                }
                break;
            case FB_MERGE_XOR:
                for (uint64_t i = threadIdx.x; i < len; i += blockDim.x) {
                    dst[i] ^= src[i];
                }
                break;
            default: {
                // typed scalar ops: thread per scalar
                uint32_t sz = (d.dataType == FB_SNAP_INT ||
                               d.dataType == FB_SNAP_FLOAT)
                                ? 4
                                : 8;
                uint64_t n = len / sz;
                for (uint64_t k = threadIdx.x; k < n; k += blockDim.x) {
                    uint8_t* p = dst + k * sz;
                    const uint8_t* q = src + k * sz;
#define APPLY_T(T)                                                             \
    {                                                                          \
        T c = loadUnaligned<T>(p);                                             \
        T v = loadUnaligned<T>(q);                                             \
        T r = c;                                                               \
        if (d.op == FB_MERGE_SUM)                                              \
            r = snapAdd(c, v);                                                 \
        else if (d.op == FB_MERGE_SUBTRACT)                                    \
            r = snapSub(c, v);                                                 \
        else if (d.op == FB_MERGE_PRODUCT)                                     \
            r = snapMul(c, v);                                                 \
        else if (d.op == FB_MERGE_MAX)                                         \
            r = snapMax(c, v);                                                 \
        else if (d.op == FB_MERGE_MIN)                                         \
            r = snapMin(c, v);                                                 \
        storeUnaligned<T>(p, r);                                               \
    }
                    if (d.dataType == FB_SNAP_INT)
                        APPLY_T(int32_t)
                    else if (d.dataType == FB_SNAP_LONG)
                        APPLY_T(int64_t)
                    else if (d.dataType == FB_SNAP_FLOAT)
                        APPLY_T(float)
                    else if (d.dataType == FB_SNAP_DOUBLE)
                        APPLY_T(double)
#undef APPLY_T
                }
                break;
            }
        }
    }
}

cudaError_t launchSnapshotApply(uint8_t* image,
                                uint64_t imageSize,
                                const FbDiffDesc* descs,
                                const uint64_t* dataOff,
                                const uint8_t* blob,
                                uint32_t nDescs,
                                cudaStream_t s)
{
    if (nDescs == 0) {
        return cudaSuccess;
    }
    int blocks = (int)(nDescs < 4096u ? nDescs : 4096u);
    snapshotApplyKernel<<<blocks, 256, 0, s>>>(
      image, imageSize, descs, dataOff, blob, nDescs);
    return cudaGetLastError();
}

cudaError_t preloadSnapshotKernels()
{
    cudaFuncAttributes a;
    cudaError_t e = cudaFuncGetAttributes(&a, snapshotDiffPushKernel);
    if (e == cudaSuccess) {
        e = cudaFuncGetAttributes(&a, dirtyScanKernel);
    }
    if (e == cudaSuccess) {
        e = cudaFuncGetAttributes(&a, flagsOrKernel);
    }
    if (e == cudaSuccess) {
        e = cudaFuncGetAttributes(&a, chunkRunsKernel);
    }
    if (e == cudaSuccess) {
        e = cudaFuncGetAttributes(&a, snapshotApplyKernel);
    }
    return e;
}

} // namespace fb
