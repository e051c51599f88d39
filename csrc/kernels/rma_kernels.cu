// One-sided atomics (sm_90a): MPI_Accumulate, MPI_Get_accumulate,
// MPI_Fetch_and_op and MPI_Compare_and_swap on any memory the launching GPU
// can address.
//
//  * rmaAccumulateKernel<DT, OP, FETCH> — grid-stride over `count` elements:
//    target[i] = combine(target[i], origin[i]), where target is a pointer (a
//    peer's symmetric heap through its NVLink mapping, a cudaMalloc window, or
//    local memory).  combine is the
//    element-wise rule of the reduce kernels (fb_prims.cuh: reduceElem,
//    reducePair), REPLACE stores the origin value and NO_OP keeps the target.
//    FETCH also writes every element's previous value to `result`.
//  * rmaCompareSwapKernel<DT> — one integer element: result = old; if (old ==
//    compare) target = swap.
//
// Each element is one atomic step at system scope (fb_atomics.cuh): a native
// red / atom where the ISA has the operation (32/64-bit integer add, max, min,
// and, or, xor, exch; f64 add; packed f16/bf16 add for 16-byte aligned
// vectors), otherwise a CAS loop on the element, on its enclosing 32-bit word
// for 1- and 2-byte elements, or 128-bit for the 16-byte pairs, whose padding
// is preserved.  Concurrent accumulates from any number of GPUs therefore
// compose element by element.  The kernels never wait on a peer.
//
//  * rmaCopyManyKernel — a table of plain copies (request-based puts and gets
//    on the symmetric heap): one launch for a whole list, any alignment.
#include "fb_atomics.cuh"
#include "fb_prims.cuh"
#include "launch_api.h"

namespace fb {

static constexpr int RMA_THREADS = 256;
static constexpr int RMA_MAX_BLOCKS = FB_NUM_SMS * 8;

template<int DT>
struct RmaType;
#define FB_RMA_TYPE(dt, T_, PAIR_)                                             \
    template<>                                                                 \
    struct RmaType<dt>                                                         \
    {                                                                          \
        using T = T_;                                                          \
        static constexpr bool PAIR = PAIR_;                                    \
    };
FB_RMA_TYPE(FB_I8, int8_t, false)
FB_RMA_TYPE(FB_U8, uint8_t, false)
FB_RMA_TYPE(FB_I16, int16_t, false)
FB_RMA_TYPE(FB_U16, uint16_t, false)
FB_RMA_TYPE(FB_I32, int32_t, false)
FB_RMA_TYPE(FB_U32, uint32_t, false)
FB_RMA_TYPE(FB_I64, int64_t, false)
FB_RMA_TYPE(FB_U64, uint64_t, false)
FB_RMA_TYPE(FB_F32, float, false)
FB_RMA_TYPE(FB_F64, double, false)
FB_RMA_TYPE(FB_F16, __half, false)
FB_RMA_TYPE(FB_BF16, __nv_bfloat16, false)
FB_RMA_TYPE(FB_F64_I32, double, true)
FB_RMA_TYPE(FB_F32_I32, float, true)
FB_RMA_TYPE(FB_I32_I32, int32_t, true)
FB_RMA_TYPE(FB_I64_I32, int64_t, true)
#undef FB_RMA_TYPE

template<int DT>
using RmaElem = typename ElemOf<typename RmaType<DT>::T, RmaType<DT>::PAIR>::type;

// The supported set: the reduce kernels' (dtype, op) pairs, plus REPLACE for
// every dtype and NO_OP for every dtype when fetching
constexpr bool rmaOk(int dt, int op, bool fetch)
{
    if (dt < 0 || dt >= FB_DTYPE_COUNT) {
        return false;
    }
    if (op == FB_OP_REPLACE) {
        return true;
    }
    if (op == FB_OP_NO_OP) {
        return fetch;
    }
    if (dt <= FB_U64) {
        return op >= 0 && op < FB_OP_COUNT && op != FB_OP_MAXLOC && op != FB_OP_MINLOC;
    }
    if (dt <= FB_BF16) {
        return op == FB_OP_MAX || op == FB_OP_MIN || op == FB_OP_SUM || op == FB_OP_PROD;
    }
    return op == FB_OP_MAXLOC || op == FB_OP_MINLOC;
}

template<typename E>
__device__ __forceinline__ E ldBytes(const uint8_t* p)
{
    E v;
    uint8_t* b = reinterpret_cast<uint8_t*>(&v);
#pragma unroll
    for (int i = 0; i < (int)sizeof(E); i++) {
        b[i] = p[i];
    }
    return v;
}

template<typename E>
__device__ __forceinline__ void stBytes(uint8_t* p, const E& v)
{
    const uint8_t* b = reinterpret_cast<const uint8_t*>(&v);
#pragma unroll
    for (int i = 0; i < (int)sizeof(E); i++) {
        p[i] = b[i];
    }
}

template<typename E>
using RmaBits = std::conditional_t<sizeof(E) == 8, uint64_t, uint32_t>;

template<typename B, typename E>
__device__ __forceinline__ B toBits(const E& v)
{
    B b;
    memcpy(&b, &v, sizeof(B));
    return b;
}

template<typename E, typename B>
__device__ __forceinline__ E fromBits(B b)
{
    E v;
    memcpy(&v, &b, sizeof(E));
    return v;
}

// combine(target, origin), the rule every path of one (dtype, op) computes
template<int DT, int OP>
__device__ __forceinline__ RmaElem<DT> rmaCombine(RmaElem<DT> cur, RmaElem<DT> v)
{
    using T = typename RmaType<DT>::T;
    if constexpr (OP == FB_OP_REPLACE) {
        return v;
    } else if constexpr (OP == FB_OP_NO_OP) {
        return cur;
    } else if constexpr (RmaType<DT>::PAIR) {
        return reducePair<T, OP>(cur, v);
    } else {
        return reduceElem<T, OP>(cur, v);
    }
}

// Type of a native add: the unsigned integer of the same width (identical
// bits, wrapping), or the float type itself
template<typename T, bool = std::is_integral_v<T>>
struct RmaAddType
{
    using type = T;
};
template<typename T>
struct RmaAddType<T, true>
{
    using type = std::make_unsigned_t<T>;
};

// Operations with a native system-scope instruction
template<int DT, int OP>
constexpr bool rmaNative()
{
    using T = typename RmaType<DT>::T;
    using E = RmaElem<DT>;
    constexpr bool word = sizeof(E) == 4 || sizeof(E) == 8;
    if constexpr (OP == FB_OP_REPLACE) {
        return word;
    } else if constexpr (std::is_integral_v<T> && !RmaType<DT>::PAIR && word) {
        return OP == FB_OP_SUM || OP == FB_OP_MAX || OP == FB_OP_MIN || OP == FB_OP_BAND ||
               OP == FB_OP_BOR || OP == FB_OP_BXOR;
    } else {
        return std::is_same_v<T, double> && !RmaType<DT>::PAIR && OP == FB_OP_SUM;
    }
}

// One element: atomic, returns the previous value (meaningful when FETCH)
template<int DT, int OP, bool FETCH>
__device__ __forceinline__ RmaElem<DT> rmaApply(uint8_t* p, RmaElem<DT> v)
{
    using T = typename RmaType<DT>::T;
    using E = RmaElem<DT>;
    if constexpr (OP == FB_OP_NO_OP) {
        if constexpr (sizeof(E) == 16) {
            // atomic 16-byte read: a CAS whose compare and swap values are
            // equal never changes the location and returns its contents
            uint64_t r[2];
            cas128Sys(p, 0, 0, 0, 0, r[0], r[1]);
            E cur;
            memcpy(&cur, r, 16);
            return cur;
        } else {
            return fromBits<E>(ldRelaxedSysBytes<(int)sizeof(E)>(p));
        }
    } else if constexpr (rmaNative<DT, OP>()) {
        using B = RmaBits<E>;
        if constexpr (OP == FB_OP_REPLACE) {
            return fromBits<E>(atomExchSys(reinterpret_cast<B*>(p), toBits<B>(v)));
        } else if constexpr (OP == FB_OP_BAND || OP == FB_OP_BOR || OP == FB_OP_BXOR) {
            B* q = reinterpret_cast<B*>(p);
            const B b = toBits<B>(v);
            if constexpr (FETCH) {
                B r = OP == FB_OP_BAND ? atomAndSys(q, b) : (OP == FB_OP_BOR ? atomOrSys(q, b) : atomXorSys(q, b));
                return fromBits<E>(r);
            } else {
                if constexpr (OP == FB_OP_BAND) {
                    redAndSys(q, b);
                } else if constexpr (OP == FB_OP_BOR) {
                    redOrSys(q, b);
                } else {
                    redXorSys(q, b);
                }
                return v;
            }
        } else if constexpr (OP == FB_OP_SUM) {
            // integers: the unsigned add of the same width (identical bits)
            using A = typename RmaAddType<T>::type;
            A* q = reinterpret_cast<A*>(p);
            const A x = fromBits<A>(toBits<B>(v));
            if constexpr (FETCH) {
                return fromBits<E>(toBits<B>(atomAddSys(q, x)));
            } else {
                redAddSys(q, x);
                return v;
            }
        } else {
            T* q = reinterpret_cast<T*>(p);
            if constexpr (FETCH) {
                return OP == FB_OP_MAX ? atomMaxSys(q, v) : atomMinSys(q, v);
            } else {
                if constexpr (OP == FB_OP_MAX) {
                    redMaxSys(q, v);
                } else {
                    redMinSys(q, v);
                }
                return v;
            }
        }
    } else {
        // a pair's value and index change, its padding is kept
        constexpr int KEEP = RmaType<DT>::PAIR ? (int)sizeof(T) + 4 : (int)sizeof(E);
        return casRmwSys<E, KEEP>(p, [v](E c) { return rmaCombine<DT, OP>(c, v); });
    }
}

template<int DT, int OP, bool FETCH>
__global__ void __launch_bounds__(RMA_THREADS) rmaAccumulateKernel(const RmaArgs a)
{
    using E = RmaElem<DT>;
    uint8_t* tgt = a.target;
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t nth = (uint64_t)gridDim.x * blockDim.x;
    uint64_t first = 0;
    if constexpr (!FETCH && OP == FB_OP_SUM && (DT == FB_F16 || DT == FB_BF16)) {
        // eight elements per packed .noftz add when both sides allow it
        if ((((uintptr_t)tgt | (uintptr_t)a.origin) & 15) == 0) {
            const uint64_t nVec = a.count / 8;
            for (uint64_t i = tid; i < nVec; i += nth) {
                const Vec16 x = ldVec(a.origin + 16 * i);
                if constexpr (DT == FB_F16) {
                    redAddF16x8Sys(tgt + 16 * i, x.w[0], x.w[1], x.w[2], x.w[3]);
                } else {
                    redAddBf16x8Sys(tgt + 16 * i, x.w[0], x.w[1], x.w[2], x.w[3]);
                }
            }
            first = nVec * 8;
        }
    }
    const bool originAligned = ((uintptr_t)a.origin % sizeof(E)) == 0;
    const bool resultAligned = ((uintptr_t)a.result % sizeof(E)) == 0;
    for (uint64_t i = first + tid; i < a.count; i += nth) {
        E v{};
        if constexpr (OP != FB_OP_NO_OP) {
            const uint8_t* o = a.origin + i * sizeof(E);
            v = originAligned ? *reinterpret_cast<const E*>(o) : ldBytes<E>(o);
        }
        E old = rmaApply<DT, OP, FETCH>(tgt + i * sizeof(E), v);
        if constexpr (FETCH) {
            uint8_t* r = a.result + i * sizeof(E);
            if (resultAligned) {
                *reinterpret_cast<E*>(r) = old;
            } else {
                stBytes<E>(r, old);
            }
        }
    }
}

template<int DT>
__global__ void rmaCompareSwapKernel(const RmaCasArgs a)
{
    using T = typename RmaType<DT>::T;
    uint8_t* tgt = a.target;
    const T cmp = ldBytes<T>(a.compare);
    const T swp = ldBytes<T>(a.swap);
    T old;
    if constexpr (sizeof(T) >= 4) {
        using B = RmaBits<T>;
        old = (T)atomCasSys(reinterpret_cast<B*>(tgt), (B)cmp, (B)swp);
    } else {
        // enclosing-word CAS: the neighbouring bytes are never written
        old = casRmwSys<T>(tgt, [cmp, swp](T c) { return c == cmp ? swp : c; });
    }
    stBytes<T>(a.result, old);
}

// ---------------------------------------------------------- batched copy ----
static constexpr int RMA_COPY_THREADS = 256;
static constexpr int RMA_COPY_UNROLL = 4;

template<int W>
struct CopyWord;
template<>
struct CopyWord<16>
{
    using T = Vec16;
    static __device__ __forceinline__ T ld(const uint8_t* p) { return ldVec(p); }
    static __device__ __forceinline__ void st(uint8_t* p, const T& v) { stVec(p, v); }
};
template<>
struct CopyWord<8>
{
    using T = uint64_t;
    static __device__ __forceinline__ T ld(const uint8_t* p)
    {
        T v;
        asm volatile("ld.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
        return v;
    }
    static __device__ __forceinline__ void st(uint8_t* p, T v)
    {
        asm volatile("st.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
    }
};
template<>
struct CopyWord<4>
{
    using T = uint32_t;
    static __device__ __forceinline__ T ld(const uint8_t* p)
    {
        T v;
        asm volatile("ld.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
        return v;
    }
    static __device__ __forceinline__ void st(uint8_t* p, T v)
    {
        asm volatile("st.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
    }
};
template<>
struct CopyWord<2>
{
    using T = uint16_t;
    static __device__ __forceinline__ T ld(const uint8_t* p)
    {
        T v;
        asm volatile("ld.global.u16 %0, [%1];" : "=h"(v) : "l"(p) : "memory");
        return v;
    }
    static __device__ __forceinline__ void st(uint8_t* p, T v)
    {
        asm volatile("st.global.u16 [%0], %1;" ::"l"(p), "h"(v) : "memory");
    }
};
template<>
struct CopyWord<1>
{
    using T = uint32_t;
    static __device__ __forceinline__ T ld(const uint8_t* p)
    {
        T v;
        asm volatile("ld.global.u8 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
        return v;
    }
    static __device__ __forceinline__ void st(uint8_t* p, T v)
    {
        asm volatile("st.global.u8 [%0], %1;" ::"l"(p), "r"(v) : "memory");
    }
};

// n words of W bytes, one warp: RMA_COPY_UNROLL loads in flight per lane
// before their stores
template<int W>
__device__ __forceinline__ void copyWords(const uint8_t* s, uint8_t* d, uint32_t n, uint32_t lane)
{
    using C = CopyWord<W>;
    for (uint32_t base = 0; base < n; base += 32 * RMA_COPY_UNROLL) {
        typename C::T v[RMA_COPY_UNROLL];
#pragma unroll
        for (int u = 0; u < RMA_COPY_UNROLL; u++) {
            const uint32_t i = base + u * 32 + lane;
            if (i < n) {
                v[u] = C::ld(s + (uint64_t)i * W);
            }
        }
#pragma unroll
        for (int u = 0; u < RMA_COPY_UNROLL; u++) {
            const uint32_t i = base + u * 32 + lane;
            if (i < n) {
                C::st(d + (uint64_t)i * W, v[u]);
            }
        }
    }
}

// Item that owns chunk `ch`: usually `cur` again (a warp's chunks ascend),
// otherwise a binary search over chunk0
__device__ __forceinline__ uint32_t copyItemOf(const RmaCopyDesc* t, uint32_t n, uint32_t cur, uint64_t ch)
{
    if (t[cur].chunk0 <= ch && (cur + 1 == n || ch < t[cur + 1].chunk0)) {
        return cur;
    }
    uint32_t lo = 0;
    uint32_t hi = n - 1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (t[mid].chunk0 <= ch) {
            lo = mid;
        } else {
            hi = mid - 1;
        }
    }
    return lo;
}

// One chunk of an item: a head of single bytes up to the widest alignment
// that src and dst share (mod 16), the middle in words of that width, a tail
// of single bytes
__global__ void __launch_bounds__(RMA_COPY_THREADS, 2) rmaCopyManyKernel(const RmaCopyArgs a)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t nWarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    uint32_t cur = 0;
    for (uint64_t ch = warp; ch < a.totalChunks; ch += nWarps) {
        cur = copyItemOf(a.items, a.nItems, cur, ch);
        const RmaCopyDesc it = a.items[cur];
        const uint64_t lo = (ch - it.chunk0) * FB_RMA_COPY_CHUNK;
        const uint64_t len = min((uint64_t)FB_RMA_COPY_CHUNK, it.bytes - lo);
        const uint8_t* s = it.src + lo;
        uint8_t* d = it.dst + lo;
        const uint32_t mis = (uint32_t)(((uintptr_t)s ^ (uintptr_t)d) & 15);
        const uint32_t w = mis == 0 ? 16 : (mis & -mis);
        const uint32_t head = (uint32_t)min((uint64_t)((w - ((uintptr_t)s & (w - 1))) & (w - 1)), len);
        if (lane < head) {
            d[lane] = s[lane];
        }
        const uint32_t n = (uint32_t)((len - head) / w);
        const uint8_t* sb = s + head;
        uint8_t* db = d + head;
        switch (w) {
            case 16:
                copyWords<16>(sb, db, n, lane);
                break;
            case 8:
                copyWords<8>(sb, db, n, lane);
                break;
            case 4:
                copyWords<4>(sb, db, n, lane);
                break;
            case 2:
                copyWords<2>(sb, db, n, lane);
                break;
            default:
                copyWords<1>(sb, db, n, lane);
                break;
        }
        const uint32_t done = head + n * w;
        if (lane < len - done) {
            d[done + lane] = s[done + lane];
        }
    }
}

cudaError_t launchRmaCopyMany(const RmaCopyArgs& a, cudaStream_t s)
{
    if (a.nItems == 0 || a.totalChunks == 0) {
        return cudaSuccess;
    }
    constexpr uint64_t warpsPerBlock = RMA_COPY_THREADS / 32;
    const uint64_t want = (a.totalChunks + warpsPerBlock - 1) / warpsPerBlock;
    const unsigned blocks = (unsigned)(want > 2 * FB_NUM_SMS ? 2 * FB_NUM_SMS : want);
    void* args[] = { const_cast<RmaCopyArgs*>(&a) };
    return cudaLaunchKernel((const void*)rmaCopyManyKernel, dim3(blocks), dim3(RMA_COPY_THREADS), args, 0, s);
}

// ------------------------------------------------------------- dispatch ----
template<int DT, int OP, bool FETCH>
static const void* kernelOrNull()
{
    if constexpr (rmaOk(DT, OP, FETCH)) {
        return (const void*)rmaAccumulateKernel<DT, OP, FETCH>;
    } else {
        return nullptr;
    }
}

template<int DT, bool FETCH>
static const void* byOp(int op)
{
    switch (op) {
        case FB_OP_MAX:
            return kernelOrNull<DT, FB_OP_MAX, FETCH>();
        case FB_OP_MIN:
            return kernelOrNull<DT, FB_OP_MIN, FETCH>();
        case FB_OP_SUM:
            return kernelOrNull<DT, FB_OP_SUM, FETCH>();
        case FB_OP_PROD:
            return kernelOrNull<DT, FB_OP_PROD, FETCH>();
        case FB_OP_LAND:
            return kernelOrNull<DT, FB_OP_LAND, FETCH>();
        case FB_OP_LOR:
            return kernelOrNull<DT, FB_OP_LOR, FETCH>();
        case FB_OP_BAND:
            return kernelOrNull<DT, FB_OP_BAND, FETCH>();
        case FB_OP_BOR:
            return kernelOrNull<DT, FB_OP_BOR, FETCH>();
        case FB_OP_MAXLOC:
            return kernelOrNull<DT, FB_OP_MAXLOC, FETCH>();
        case FB_OP_MINLOC:
            return kernelOrNull<DT, FB_OP_MINLOC, FETCH>();
        case FB_OP_LXOR:
            return kernelOrNull<DT, FB_OP_LXOR, FETCH>();
        case FB_OP_BXOR:
            return kernelOrNull<DT, FB_OP_BXOR, FETCH>();
        case FB_OP_REPLACE:
            return kernelOrNull<DT, FB_OP_REPLACE, FETCH>();
        case FB_OP_NO_OP:
            return kernelOrNull<DT, FB_OP_NO_OP, FETCH>();
        default:
            return nullptr;
    }
}

template<bool FETCH>
static const void* byDtype(int dtype, int op)
{
    switch (dtype) {
#define FB_RMA_DT(dt)                                                          \
    case dt:                                                                   \
        return byOp<dt, FETCH>(op);
        FB_RMA_DT(FB_I8)
        FB_RMA_DT(FB_U8)
        FB_RMA_DT(FB_I16)
        FB_RMA_DT(FB_U16)
        FB_RMA_DT(FB_I32)
        FB_RMA_DT(FB_U32)
        FB_RMA_DT(FB_I64)
        FB_RMA_DT(FB_U64)
        FB_RMA_DT(FB_F32)
        FB_RMA_DT(FB_F64)
        FB_RMA_DT(FB_F16)
        FB_RMA_DT(FB_BF16)
        FB_RMA_DT(FB_F64_I32)
        FB_RMA_DT(FB_F32_I32)
        FB_RMA_DT(FB_I32_I32)
        FB_RMA_DT(FB_I64_I32)
#undef FB_RMA_DT
        default:
            return nullptr;
    }
}

static const void* accumulateKernel(int dtype, int op, bool fetch)
{
    return fetch ? byDtype<true>(dtype, op) : byDtype<false>(dtype, op);
}

static const void* casKernel(int dtype)
{
    switch (dtype) {
        case FB_I8:
            return (const void*)rmaCompareSwapKernel<FB_I8>;
        case FB_U8:
            return (const void*)rmaCompareSwapKernel<FB_U8>;
        case FB_I16:
            return (const void*)rmaCompareSwapKernel<FB_I16>;
        case FB_U16:
            return (const void*)rmaCompareSwapKernel<FB_U16>;
        case FB_I32:
            return (const void*)rmaCompareSwapKernel<FB_I32>;
        case FB_U32:
            return (const void*)rmaCompareSwapKernel<FB_U32>;
        case FB_I64:
            return (const void*)rmaCompareSwapKernel<FB_I64>;
        case FB_U64:
            return (const void*)rmaCompareSwapKernel<FB_U64>;
        default:
            return nullptr;
    }
}

bool rmaSupported(int dtype, int op, bool fetch)
{
    return accumulateKernel(dtype, op, fetch) != nullptr;
}

bool rmaCasSupported(int dtype)
{
    return casKernel(dtype) != nullptr;
}

cudaError_t launchRmaAccumulate(const RmaArgs& a, int dtype, int op, cudaStream_t s)
{
    const void* k = accumulateKernel(dtype, op, a.result != nullptr);
    if (k == nullptr) {
        return cudaErrorInvalidValue;
    }
    const uint64_t want = (a.count + RMA_THREADS - 1) / RMA_THREADS;
    const unsigned blocks = (unsigned)(want < 1 ? 1 : (want > RMA_MAX_BLOCKS ? RMA_MAX_BLOCKS : want));
    void* args[] = { const_cast<RmaArgs*>(&a) };
    return cudaLaunchKernel(k, dim3(blocks), dim3(RMA_THREADS), args, 0, s);
}

cudaError_t launchRmaCompareSwap(const RmaCasArgs& a, int dtype, cudaStream_t s)
{
    const void* k = casKernel(dtype);
    if (k == nullptr) {
        return cudaErrorInvalidValue;
    }
    void* args[] = { const_cast<RmaCasArgs*>(&a) };
    return cudaLaunchKernel(k, dim3(1), dim3(1), args, 0, s);
}

cudaError_t preloadRmaKernels()
{
    cudaFuncAttributes attr;
    cudaError_t e = cudaSuccess;
    for (int dt = 0; dt < FB_DTYPE_COUNT && e == cudaSuccess; dt++) {
        for (int op = 0; op <= FB_OP_NO_OP && e == cudaSuccess; op++) {
            for (int f = 0; f < 2 && e == cudaSuccess; f++) {
                const void* k = accumulateKernel(dt, op, f != 0);
                if (k != nullptr) {
                    e = cudaFuncGetAttributes(&attr, k);
                }
            }
        }
        if (e == cudaSuccess && casKernel(dt) != nullptr) {
            e = cudaFuncGetAttributes(&attr, casKernel(dt));
        }
    }
    if (e == cudaSuccess) {
        e = cudaFuncGetAttributes(&attr, (const void*)rmaCopyManyKernel);
    }
    return e;
}

} // namespace fb
