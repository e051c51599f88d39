// Element-wise semantics of the host reductions (MPI on host buffers, both the
// message and the shared-memory paths, and the loopback device backend).  They
// match the device kernels (csrc/kernels/fb_prims.cuh):
//  * integer SUM/PROD wrap, computed in the unsigned type of the same width
//    (types narrower than int in unsigned int), so overflow is never signed;
//  * float MAX/MIN ignore a NaN operand (NaN only if both are) and order -0
//    below +0, so the result does not depend on the order of the operands.
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

template<typename T>
inline T reduceMax(T a, T b)
{
    if constexpr (std::is_floating_point_v<T>) {
        if (a == b) {
            return std::signbit(a) ? b : a; // +0 over -0
        }
        return std::fmax(a, b);
    } else {
        return a > b ? a : b;
    }
}

template<typename T>
inline T reduceMin(T a, T b)
{
    if constexpr (std::is_floating_point_v<T>) {
        if (a == b) {
            return std::signbit(a) ? a : b; // -0 over +0
        }
        return std::fmin(a, b);
    } else {
        return a < b ? a : b;
    }
}

} // namespace faabric::util
