// Device primitives for the peer-memory collectives (sm_90a).
//  * system-scope release/acquire flag ops and a bounded (watchdog) spin
//  * block-level cross-rank barrier over monotonically increasing flags
//  * 16-byte vector load/store helpers (peer-safe: no .nc, no L1 staleness)
//  * element-wise reduction functors for every (dtype, op) pair; replaces the
//    scalar CPU loop of the reference's MpiWorld::op_reduce
//    (src/mpi/MpiWorld.cpp:1266-1388) and extends it to all ops/dtypes.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include <type_traits>

#include "faabric/device/comm_abi.h"

namespace fb {

// ----------------------------------------------------------------------------
// Flags
// ----------------------------------------------------------------------------
__device__ __forceinline__ void stReleaseSys(uint32_t* p, uint32_t v)
{
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v)
                 : "memory");
}

__device__ __forceinline__ void stRelaxedSys(uint32_t* p, uint32_t v)
{
    asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v)
                 : "memory");
}

__device__ __forceinline__ uint32_t ldAcquireSys(const uint32_t* p)
{
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];"
                 : "=r"(v)
                 : "l"(p)
                 : "memory");
    return v;
}

__device__ __forceinline__ uint32_t ldRelaxedSys(const uint32_t* p)
{
    uint32_t v;
    asm volatile("ld.relaxed.sys.global.u32 %0, [%1];"
                 : "=r"(v)
                 : "l"(p)
                 : "memory");
    return v;
}

__device__ __forceinline__ void fenceSys()
{
    asm volatile("fence.acq_rel.sys;" ::: "memory");
}

__device__ __forceinline__ uint64_t globalTimerNs()
{
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// Spin until *p >= target (wrap-safe).  Bounded by c.timeoutNs: on expiry the
// error word is set and the function returns false so the kernel can finish
// instead of hanging the GPU (a hung peer must never wedge the device).
__device__ __forceinline__ bool waitFlagGe(const FbCommDev& c,
                                           const uint32_t* p,
                                           uint32_t target,
                                           uint32_t errCode)
{
    if ((int32_t)(ldAcquireSys(p) - target) >= 0) {
        return true;
    }
    uint64_t t0 = globalTimerNs();
    uint32_t spins = 0;
    while (true) {
        if ((int32_t)(ldAcquireSys(p) - target) >= 0) {
            return true;
        }
        if ((++spins & 0x3ff) == 0) {
            if (globalTimerNs() - t0 > c.timeoutNs) {
                if (c.err != nullptr) {
                    stRelaxedSys(c.err, errCode); // host-mapped word: plain store, no PCIe atomic
                }
                return false;
            }
            // a peer already reported a failure: bail out too
            if (c.err != nullptr && ldRelaxedSys(c.err) != FB_ERR_NONE) {
                return false;
            }
        }
    }
}

// ----------------------------------------------------------------------------
// Cross-rank barrier between CTA `blockIdx.x` of every rank.
//
// Each CTA keeps a private epoch (loaded from the local signal pad at kernel
// start, written back at kernel end), so launches compose under CUDA-graph
// replay without host-side counters.  Flags only ever increase -> no reset
// race.  Release/acquire at .sys scope gives: everything written by this CTA
// before the barrier (including peer stores) is visible to the peers after it.
// ----------------------------------------------------------------------------
struct BlockBarrier
{
    uint32_t epoch;

    __device__ __forceinline__ void load(const FbCommDev& c)
    {
        // Plain read: only this CTA index on this rank ever writes the word,
        // and the previous writer was an earlier kernel on the same stream.
        epoch = c.sig[c.rank][FB_SIG_EPOCH_OFF + c.blockBase + blockIdx.x];
    }

    __device__ __forceinline__ void store(const FbCommDev& c)
    {
        if (threadIdx.x == 0) {
            c.sig[c.rank][FB_SIG_EPOCH_OFF + c.blockBase + blockIdx.x] = epoch;
        }
    }

    __device__ __forceinline__ bool sync(const FbCommDev& c)
    {
        epoch += 1;
        __syncthreads();
        bool ok = true;
        if (threadIdx.x < (unsigned)c.nranks) {
            int peer = threadIdx.x;
            const size_t slot = (size_t)(c.blockBase + blockIdx.x);
            uint32_t* remote = c.sig[peer] + slot * FB_MAX_RANKS + c.rank;
            stReleaseSys(remote, epoch);
            const uint32_t* mine =
              c.sig[c.rank] + slot * FB_MAX_RANKS + peer;
            ok = waitFlagGe(c, mine, epoch, FB_ERR_BARRIER_TIMEOUT);
        }
        // __syncthreads_and also makes the acquire cumulative for the CTA
        return __syncthreads_and(ok ? 1 : 0) != 0;
    }
};

// ----------------------------------------------------------------------------
// 16-byte vector access
// ----------------------------------------------------------------------------
struct alignas(16) Vec16
{
    uint32_t w[4];
};

__device__ __forceinline__ Vec16 ldVec(const void* p)
{
    Vec16 v;
    asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3])
                 : "l"(p)
                 : "memory");
    return v;
}

// Streaming variant: do not allocate in L1 (data is touched once)
__device__ __forceinline__ Vec16 ldVecStream(const void* p)
{
    Vec16 v;
    asm volatile(
      "ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
      : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3])
      : "l"(p)
      : "memory");
    return v;
}

__device__ __forceinline__ void stVec(void* p, const Vec16& v)
{
    asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p),
                 "r"(v.w[0]),
                 "r"(v.w[1]),
                 "r"(v.w[2]),
                 "r"(v.w[3])
                 : "memory");
}

// ----------------------------------------------------------------------------
// Reduce functors
// ----------------------------------------------------------------------------
template<int OP>
struct OpTag
{
    static constexpr int value = OP;
};

template<typename T>
struct PairVI
{
    T v;
    int32_t i;
};

template<typename T, int OP>
struct Reducer
{
    __device__ __forceinline__ static T apply(T a, T b)
    {
        // Float MAX/MIN use fmax/fmin (a NaN operand is ignored; NaN only if
        // both are NaN; -0 orders below +0), so the result does not depend on
        // which rank holds a NaN or a signed zero.  A plain `a > b ? a : b`
        // keeps a NaN in `b` but drops one in `a`, and returns `b` for ±0.
        if constexpr (OP == FB_OP_MAX && std::is_same_v<T, float>) {
            return fmaxf(a, b);
        } else if constexpr (OP == FB_OP_MAX && std::is_same_v<T, double>) {
            return fmax(a, b);
        } else if constexpr (OP == FB_OP_MIN && std::is_same_v<T, float>) {
            return fminf(a, b);
        } else if constexpr (OP == FB_OP_MIN && std::is_same_v<T, double>) {
            return fmin(a, b);
        } else if constexpr (OP == FB_OP_MAX) {
            return a > b ? a : b;
        } else if constexpr (OP == FB_OP_MIN) {
            return a < b ? a : b;
        } else if constexpr (OP == FB_OP_SUM) {
            return a + b;
        } else if constexpr (OP == FB_OP_PROD) {
            return a * b;
        } else if constexpr (OP == FB_OP_LAND) {
            return (T)((a != (T)0) && (b != (T)0));
        } else if constexpr (OP == FB_OP_LOR) {
            return (T)((a != (T)0) || (b != (T)0));
        } else if constexpr (OP == FB_OP_LXOR) {
            return (T)((a != (T)0) != (b != (T)0));
        } else {
            return a;
        }
    }
};

// Bitwise ops only exist for integers: specialise through a helper
template<typename T, int OP>
__device__ __forceinline__ T bitOp(T a, T b)
{
    if constexpr (OP == FB_OP_BAND) {
        return a & b;
    } else if constexpr (OP == FB_OP_BOR) {
        return a | b;
    } else {
        return a ^ b;
    }
}

template<typename T>
struct IsFloatLike
{
    static constexpr bool value = false;
};
template<>
struct IsFloatLike<float>
{
    static constexpr bool value = true;
};
template<>
struct IsFloatLike<double>
{
    static constexpr bool value = true;
};
template<>
struct IsFloatLike<__half>
{
    static constexpr bool value = true;
};
template<>
struct IsFloatLike<__nv_bfloat16>
{
    static constexpr bool value = true;
};

template<int OP>
struct IsBitwiseOp
{
    static constexpr bool value =
      (OP == FB_OP_BAND || OP == FB_OP_BOR || OP == FB_OP_BXOR);
};

// 16-bit float types: compute in fp32 (one rounding per combine, matching a
// fp32 reference within bf16/fp16 ulp)
template<typename H, int OP>
__device__ __forceinline__ H halfLikeApply(H a, H b)
{
    float r = Reducer<float, OP>::apply((float)a, (float)b);
    return (H)r;
}

template<typename T, int OP>
__device__ __forceinline__ T reduceElem(T a, T b)
{
    if constexpr (IsBitwiseOp<OP>::value) {
        if constexpr (IsFloatLike<T>::value) {
            return a; // rejected on the host; keep the template well-formed
        } else {
            return bitOp<T, OP>(a, b);
        }
    } else if constexpr (sizeof(T) == 2 && IsFloatLike<T>::value) {
        return halfLikeApply<T, OP>(a, b);
    } else {
        return Reducer<T, OP>::apply(a, b);
    }
}

// MAXLOC / MINLOC on {value,index} pairs; ties pick the lower index (MPI spec)
template<typename T, int OP>
__device__ __forceinline__ PairVI<T> reducePair(PairVI<T> a, PairVI<T> b)
{
    if constexpr (OP == FB_OP_MAXLOC) {
        if (b.v > a.v || (b.v == a.v && b.i < a.i)) {
            return b;
        }
        return a;
    } else {
        if (b.v < a.v || (b.v == a.v && b.i < a.i)) {
            return b;
        }
        return a;
    }
}

// Combine two 16-byte vectors element-wise
template<typename T, int OP>
__device__ __forceinline__ Vec16 reduceVec(const Vec16& a, const Vec16& b)
{
    constexpr int N = 16 / sizeof(T);
    union U
    {
        Vec16 v;
        T e[N];
        __device__ U() {}
    };
    U ua, ub, ur;
    ua.v = a;
    ub.v = b;
#pragma unroll
    for (int i = 0; i < N; i++) {
        ur.e[i] = reduceElem<T, OP>(ua.e[i], ub.e[i]);
    }
    return ur.v;
}

template<typename T, int OP>
__device__ __forceinline__ Vec16 reduceVecPair(const Vec16& a, const Vec16& b)
{
    using P = PairVI<T>;
    constexpr int N = 16 / sizeof(P);
    union U
    {
        Vec16 v;
        P e[N];
        __device__ U() {}
    };
    U ua, ub, ur;
    ua.v = a;
    ub.v = b;
#pragma unroll
    for (int i = 0; i < N; i++) {
        ur.e[i] = reducePair<T, OP>(ua.e[i], ub.e[i]);
    }
    return ur.v;
}

template<typename T, bool PAIR>
struct ElemOf
{
    using type = T;
};
template<typename T>
struct ElemOf<T, true>
{
    using type = PairVI<T>;
};

// Tag type so a single kernel template handles scalar and pair element kinds
template<typename T, int OP, bool PAIR>
struct VecReduce
{
    static constexpr int ELEM_BYTES = PAIR ? sizeof(PairVI<T>) : sizeof(T);
    __device__ __forceinline__ static Vec16 apply(const Vec16& a,
                                                  const Vec16& b)
    {
        if constexpr (PAIR) {
            return reduceVecPair<T, OP>(a, b);
        } else {
            return reduceVec<T, OP>(a, b);
        }
    }
    // one element, by value (tails of grouped launches)
    using Elem = typename ElemOf<T, PAIR>::type;
    __device__ __forceinline__ static Elem combine(Elem a, Elem b)
    {
        if constexpr (PAIR) {
            return reducePair<T, OP>(a, b);
        } else {
            return reduceElem<T, OP>(a, b);
        }
    }
    // scalar tail: `acc` and `in` are byte buffers, so the element is moved
    // in and out with memcpy (reading a byte array through a T lvalue is
    // undefined behaviour and was miscompiled in fully unrolled variants)
    __device__ __forceinline__ static void applyTail(uint8_t* acc,
                                                     const uint8_t* in)
    {
        if constexpr (PAIR) {
            using P = PairVI<T>;
            P a;
            P b;
            memcpy(&a, acc, sizeof(P));
            memcpy(&b, in, sizeof(P));
            P r = reducePair<T, OP>(a, b);
            memcpy(acc, &r, sizeof(P));
        } else {
            T a;
            T b;
            memcpy(&a, acc, sizeof(T));
            memcpy(&b, in, sizeof(T));
            T r = reduceElem<T, OP>(a, b);
            memcpy(acc, &r, sizeof(T));
        }
    }
};

} // namespace fb
