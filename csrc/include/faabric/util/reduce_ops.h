// Element-wise semantics of the host reductions (MPI on host buffers, both the
// message and the shared-memory paths, and the loopback device backend) and of
// the typed snapshot merges.  They match the device kernels
// (csrc/kernels/fb_prims.cuh, csrc/kernels/snapshot_kernels.cu):
//  * integer SUM/PROD wrap, computed in the unsigned type of the same width
//    (types narrower than int in unsigned int), so overflow is never signed;
//  * float MAX/MIN ignore a NaN operand, quiet or signalling (NaN only if both
//    are), and order -0 below +0, so the result does not depend on the order
//    of the operands.
#pragma once

#include <cmath>
#include <type_traits>

namespace faabric::util {

template<typename T, bool = std::is_integral_v<T>>
struct ReduceWrapType
{
    using type = T;
};
template<typename T>
struct ReduceWrapType<T, true>
{
    using type = std::conditional_t<(sizeof(T) < sizeof(unsigned)), unsigned, std::make_unsigned_t<T>>;
};

template<typename T>
inline T reduceSum(T a, T b)
{
    using W = typename ReduceWrapType<T>::type;
    return (T)(W)((W)a + (W)b);
}

template<typename T>
inline T reduceProd(T a, T b)
{
    using W = typename ReduceWrapType<T>::type;
    return (T)(W)((W)a * (W)b);
}

// a - b, wrapping like reduceSum (snapshot Sum / Subtract deltas)
template<typename T>
inline T reduceSub(T a, T b)
{
    using W = typename ReduceWrapType<T>::type;
    return (T)(W)((W)a - (W)b);
}

// The factor a snapshot Product merge sends for a value that went from `o` to
// `n`.  Floats: IEEE n / o (±inf or NaN when o is 0).  Integers: 0 when o is
// 0, a wrapping negation for o == -1 (MIN / -1 does not trap), otherwise the
// truncated quotient.
template<typename T>
inline T snapshotQuotient(T n, T o)
{
    if constexpr (std::is_floating_point_v<T>) {
        return n / o;
    } else {
        using W = typename ReduceWrapType<T>::type;
        if (o == 0) {
            return 0;
        }
        if (o == (T)-1) {
            return (T)(W)((W)0 - (W)n);
        }
        return n / o;
    }
}

template<typename T>
inline T reduceMax(T a, T b)
{
    if constexpr (std::is_floating_point_v<T>) {
        // explicit rather than std::fmax, which returns NaN for a signalling
        // NaN operand (the device's fmax ignores it like a quiet one)
        if (std::isnan(a)) {
            return b;
        }
        if (std::isnan(b)) {
            return a;
        }
        if (a == b) {
            return std::signbit(a) ? b : a; // +0 over -0
        }
        return a > b ? a : b;
    } else {
        return a > b ? a : b;
    }
}

template<typename T>
inline T reduceMin(T a, T b)
{
    if constexpr (std::is_floating_point_v<T>) {
        if (std::isnan(a)) {
            return b;
        }
        if (std::isnan(b)) {
            return a;
        }
        if (a == b) {
            return std::signbit(a) ? a : b; // -0 over +0
        }
        return a < b ? a : b;
    } else {
        return a < b ? a : b;
    }
}

} // namespace faabric::util
