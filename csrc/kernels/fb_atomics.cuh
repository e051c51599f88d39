// System-scope atomic primitives (sm_90a), shared by the snapshot merge kernels
// and the one-sided accumulate kernels.  Every operation is .sys scope, so it
// is atomic with respect to every other GPU that maps the same memory (peer
// mappings over NVLink) and to the host.
//
//  * red*Sys  — fire-and-forget reductions (SASS REDG...STRONG.SYS)
//  * atom*Sys — the fetching forms, returning the previous value
//  * atomicRmwSys / casRmwSys — compare-and-swap loops for operations the ISA
//    has no instruction for; casRmwSys also covers 1- and 2-byte scalars (a CAS
//    on the enclosing 32-bit word, so neighbouring bytes are never written)
//    and 16-byte elements (atom.cas.b128)
//
// The hardware f32 atomic add flushes subnormal inputs and results to zero,
// whereas the host merges and the reduce kernels keep them: f32 sums stay a
// CAS loop.  The f16/bf16 `.noftz` adds keep subnormals and round once to
// nearest even, which equals the widen-to-f32, add, round-back rule of the
// reduce kernels (f32 carries 24 >= 2 * 11 + 2 significand bits, so the double
// rounding is innocuous).
#pragma once

#include <stdint.h>

#include <type_traits>

namespace fb {

template<typename T>
struct AtomicWord;
template<>
struct AtomicWord<int32_t>
{
    using W = int;
};
template<>
struct AtomicWord<float>
{
    using W = int;
};
template<>
struct AtomicWord<int64_t>
{
    using W = unsigned long long;
};
template<>
struct AtomicWord<double>
{
    using W = unsigned long long;
};

// Generic CAS-based atomic RMW at system scope (works on peer memory)
template<typename T, typename F>
__device__ __forceinline__ void atomicRmwSys(T* addr, F f)
{
    using W = typename AtomicWord<T>::W;
    W* wa = reinterpret_cast<W*>(addr);
    W old = *reinterpret_cast<volatile W*>(wa);
    while (true) {
        T cur;
        memcpy(&cur, &old, sizeof(T));
        T nv = f(cur);
        W nw;
        memcpy(&nw, &nv, sizeof(T));
        W prev = atomicCAS_system(wa, old, nw);
        if (prev == old) {
            return;
        }
        old = prev;
    }
}

// Native system-scope reductions where the ISA has them (integers): one
// fire-and-forget red.* instead of a CAS round trip over NVLink
__device__ __forceinline__ void redAddSys(int32_t* p, int32_t v)
{
    asm volatile("red.relaxed.sys.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void redAddSys(int64_t* p, int64_t v)
{
    asm volatile("red.relaxed.sys.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void redMaxSys(int32_t* p, int32_t v)
{
    asm volatile("red.relaxed.sys.global.max.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void redMaxSys(int64_t* p, int64_t v)
{
    asm volatile("red.relaxed.sys.global.max.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void redMinSys(int32_t* p, int32_t v)
{
    asm volatile("red.relaxed.sys.global.min.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void redMinSys(int64_t* p, int64_t v)
{
    asm volatile("red.relaxed.sys.global.min.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// (the hardware f32 add flushes subnormals to zero; the host merge of the
// reference does not, so float sums keep the exact CAS loop)
__device__ __forceinline__ void redAddSys(float* p, float v)
{
    atomicRmwSys<float>(p, [v](float c) { return c + v; });
}
__device__ __forceinline__ void redAddSys(double* p, double v)
{
    asm volatile("red.relaxed.sys.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}

__device__ __forceinline__ bool cas128Sys(void* p,
                                          uint64_t c0,
                                          uint64_t c1,
                                          uint64_t n0,
                                          uint64_t n1,
                                          uint64_t& r0,
                                          uint64_t& r1)
{
    asm volatile("{\n\t.reg .b128 c, n, r;\n\tmov.b128 c, {%2, %3};\n\tmov.b128 n, "
                 "{%4, %5};\n\tatom.relaxed.sys.global.cas.b128 r, [%6], c, n;\n\tmov.b128 "
                 "{%0, %1}, r;\n\t}"
                 : "=l"(r0), "=l"(r1)
                 : "l"(c0), "l"(c1), "l"(n0), "l"(n1), "l"(p)
                 : "memory");
    return r0 == c0 && r1 == c1;
}

// ---- unsigned and bitwise reductions (32 and 64 bit) ----
#define FB_RED_SYS(name, T, ptx, cons)                                         \
    __device__ __forceinline__ void name(T* p, T v)                            \
    {                                                                          \
        asm volatile("red.relaxed.sys.global." ptx " [%0], %1;" ::"l"(p),      \
                     cons(v)                                                   \
                     : "memory");                                              \
    }
FB_RED_SYS(redAddSys, uint32_t, "add.u32", "r")
FB_RED_SYS(redAddSys, uint64_t, "add.u64", "l")
FB_RED_SYS(redMaxSys, uint32_t, "max.u32", "r")
FB_RED_SYS(redMaxSys, uint64_t, "max.u64", "l")
FB_RED_SYS(redMinSys, uint32_t, "min.u32", "r")
FB_RED_SYS(redMinSys, uint64_t, "min.u64", "l")
FB_RED_SYS(redAndSys, uint32_t, "and.b32", "r")
FB_RED_SYS(redAndSys, uint64_t, "and.b64", "l")
FB_RED_SYS(redOrSys, uint32_t, "or.b32", "r")
FB_RED_SYS(redOrSys, uint64_t, "or.b64", "l")
FB_RED_SYS(redXorSys, uint32_t, "xor.b32", "r")
FB_RED_SYS(redXorSys, uint64_t, "xor.b64", "l")
#undef FB_RED_SYS

// ---- fetching forms: return the value the location held before ----
#define FB_ATOM_SYS(name, T, ptx, cons)                                        \
    __device__ __forceinline__ T name(T* p, T v)                               \
    {                                                                          \
        T r;                                                                   \
        asm volatile("atom.relaxed.sys.global." ptx " %0, [%1], %2;"           \
                     : "=" cons(r)                                             \
                     : "l"(p), cons(v)                                         \
                     : "memory");                                              \
        return r;                                                              \
    }
FB_ATOM_SYS(atomAddSys, int32_t, "add.s32", "r")
FB_ATOM_SYS(atomAddSys, uint32_t, "add.u32", "r")
FB_ATOM_SYS(atomAddSys, int64_t, "add.u64", "l")
FB_ATOM_SYS(atomAddSys, uint64_t, "add.u64", "l")
FB_ATOM_SYS(atomAddSys, double, "add.f64", "d")
FB_ATOM_SYS(atomMaxSys, int32_t, "max.s32", "r")
FB_ATOM_SYS(atomMaxSys, uint32_t, "max.u32", "r")
FB_ATOM_SYS(atomMaxSys, int64_t, "max.s64", "l")
FB_ATOM_SYS(atomMaxSys, uint64_t, "max.u64", "l")
FB_ATOM_SYS(atomMinSys, int32_t, "min.s32", "r")
FB_ATOM_SYS(atomMinSys, uint32_t, "min.u32", "r")
FB_ATOM_SYS(atomMinSys, int64_t, "min.s64", "l")
FB_ATOM_SYS(atomMinSys, uint64_t, "min.u64", "l")
FB_ATOM_SYS(atomAndSys, uint32_t, "and.b32", "r")
FB_ATOM_SYS(atomAndSys, uint64_t, "and.b64", "l")
FB_ATOM_SYS(atomOrSys, uint32_t, "or.b32", "r")
FB_ATOM_SYS(atomOrSys, uint64_t, "or.b64", "l")
FB_ATOM_SYS(atomXorSys, uint32_t, "xor.b32", "r")
FB_ATOM_SYS(atomXorSys, uint64_t, "xor.b64", "l")
FB_ATOM_SYS(atomExchSys, uint32_t, "exch.b32", "r")
FB_ATOM_SYS(atomExchSys, uint64_t, "exch.b64", "l")
#undef FB_ATOM_SYS

// Compare-and-swap of a global 32/64-bit word (SASS ATOMG.E.CAS...STRONG.SYS)
__device__ __forceinline__ uint32_t atomCasSys(uint32_t* p, uint32_t c, uint32_t n)
{
    uint32_t r;
    asm volatile("atom.relaxed.sys.global.cas.b32 %0, [%1], %2, %3;" : "=r"(r) : "l"(p), "r"(c), "r"(n) : "memory");
    return r;
}
__device__ __forceinline__ uint64_t atomCasSys(uint64_t* p, uint64_t c, uint64_t n)
{
    uint64_t r;
    asm volatile("atom.relaxed.sys.global.cas.b64 %0, [%1], %2, %3;" : "=l"(r) : "l"(p), "l"(c), "l"(n) : "memory");
    return r;
}

// Packed f16 / bf16 sums of one 16-byte aligned vector (8 elements), without
// flushing subnormals (SASS REDG.E.ADD.F16x8.RN / BF16x8.RN)
__device__ __forceinline__ void redAddF16x8Sys(void* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d)
{
    asm volatile("red.relaxed.sys.global.v4.f16x2.add.noftz [%0], {%1, %2, %3, %4};" ::"l"(p),
                 "r"(a),
                 "r"(b),
                 "r"(c),
                 "r"(d)
                 : "memory");
}
__device__ __forceinline__ void redAddBf16x8Sys(void* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d)
{
    asm volatile("red.relaxed.sys.global.v4.bf16x2.add.noftz [%0], {%1, %2, %3, %4};" ::"l"(p),
                 "r"(a),
                 "r"(b),
                 "r"(c),
                 "r"(d)
                 : "memory");
}

// Single-copy atomic loads of a naturally aligned 1, 2, 4 or 8-byte location
template<int N>
__device__ __forceinline__ uint64_t ldRelaxedSysBytes(const void* p)
{
    if constexpr (N == 1) {
        uint16_t v;
        asm volatile("ld.relaxed.sys.global.u8 %0, [%1];" : "=h"(v) : "l"(p) : "memory");
        return v;
    } else if constexpr (N == 2) {
        uint16_t v;
        asm volatile("ld.relaxed.sys.global.u16 %0, [%1];" : "=h"(v) : "l"(p) : "memory");
        return v;
    } else if constexpr (N == 4) {
        uint32_t v;
        asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
        return v;
    } else {
        uint64_t v;
        asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
        return v;
    }
}

// Atomic read-modify-write of the naturally aligned element E at `p` through
// a CAS loop; returns the previous value.  `f` maps the current value to the
// new one.  1- and 2-byte elements: CAS on the enclosing 32-bit word, only the
// element's bytes change.  16-byte elements: 128-bit CAS, and only the first
// `KEEP` bytes are replaced (the rest, e.g. a pair's padding, is preserved).
// A value that does not change is not written back: the read that observed it
// (a single-copy-atomic load, or for 16 bytes a CAS) is the atomic step.
template<typename E, int KEEP = (int)sizeof(E), typename F>
__device__ __forceinline__ E casRmwSys(uint8_t* p, F f)
{
    static_assert(sizeof(E) == 1 || sizeof(E) == 2 || sizeof(E) == 4 || sizeof(E) == 8 ||
                  sizeof(E) == 16);
    if constexpr (sizeof(E) == 16) {
        uint64_t* blk = reinterpret_cast<uint64_t*>(p);
        // The first snapshot comes from a 128-bit CAS (compare == swap, so it
        // never changes the location): two 64-bit loads could pair halves of
        // two different values, and an update that finds nothing to change on
        // such a torn value would skip its write on a state that never existed
        uint64_t o0;
        uint64_t o1;
        cas128Sys(blk, 0, 0, 0, 0, o0, o1);
        while (true) {
            uint64_t ob[2] = { o0, o1 };
            E cur;
            memcpy(&cur, ob, 16);
            E nv = f(cur);
            uint64_t nb[2] = { o0, o1 };
            memcpy(nb, &nv, KEEP);
            if (nb[0] == o0 && nb[1] == o1) {
                return cur;
            }
            uint64_t r0;
            uint64_t r1;
            if (cas128Sys(blk, o0, o1, nb[0], nb[1], r0, r1)) {
                return cur;
            }
            o0 = r0;
            o1 = r1;
        }
    } else {
        using W = std::conditional_t<sizeof(E) == 8, uint64_t, uint32_t>;
        const uintptr_t addr = reinterpret_cast<uintptr_t>(p);
        W* wp = reinterpret_cast<W*>(addr & ~(uintptr_t)(sizeof(W) - 1));
        const int shift = (int)(addr & (sizeof(W) - 1)) * 8; // little endian
        W mask = ~(W)0;
        if constexpr (sizeof(E) < sizeof(W)) {
            mask = (((W)1 << (8 * sizeof(E))) - 1) << shift;
        }
        W old = *reinterpret_cast<volatile W*>(wp);
        while (true) {
            const W ow = old >> shift;
            E cur;
            memcpy(&cur, &ow, sizeof(E));
            E nv = f(cur);
            W nb = 0;
            memcpy(&nb, &nv, sizeof(E));
            const W nw = (old & ~mask) | ((nb << shift) & mask);
            if (nw == old) {
                return cur;
            }
            W prev = atomCasSys(wp, old, nw);
            if (prev == old) {
                return cur;
            }
            old = prev;
        }
    }
}

} // namespace fb
