// MAXLOC / MINLOC instantiations on {value, int} pairs, plus the top-level
// (dtype, op) -> launcher lookup.
#include "coll_reduce.cuh"

namespace fb {

template<typename T, int OP>
static const ReduceLaunchers* LP()
{
    return launchersFor<VecReduce<T, OP, true>>();
}

template<int OP>
static const ReduceLaunchers* byPair(int dtype)
{
    switch (dtype) {
        case FB_F64_I32:
            return LP<double, OP>();
        case FB_F32_I32:
            return LP<float, OP>();
        case FB_I32_I32:
            return LP<int32_t, OP>();
        case FB_I64_I32:
            return LP<int64_t, OP>();
        default:
            return nullptr;
    }
}

const ReduceLaunchers* findReduceLaunchersPair(int dtype, int op)
{
    if (op == FB_OP_MAXLOC) {
        return byPair<FB_OP_MAXLOC>(dtype);
    }
    if (op == FB_OP_MINLOC) {
        return byPair<FB_OP_MINLOC>(dtype);
    }
    return nullptr;
}

const ReduceLaunchers* findReduceLaunchers(int dtype, int op)
{
    if (dtype >= FB_I8 && dtype <= FB_U64) {
        return findReduceLaunchersInt(dtype, op);
    }
    if (dtype >= FB_F32 && dtype <= FB_BF16) {
        return findReduceLaunchersFloat(dtype, op);
    }
    return findReduceLaunchersPair(dtype, op);
}

cudaError_t preloadAllKernels()
{
    cudaError_t e = cudaSuccess;
    for (int dt = 0; dt < FB_DTYPE_COUNT && e == cudaSuccess; dt++) {
        for (int op = 0; op < FB_OP_COUNT && e == cudaSuccess; op++) {
            const ReduceLaunchers* l = findReduceLaunchers(dt, op);
            if (l != nullptr) {
                e = l->preload();
            }
        }
    }
    if (e == cudaSuccess) {
        e = preloadMoveKernels();
    }
    if (e == cudaSuccess) {
        e = preloadRootedKernels();
    }
    if (e == cudaSuccess) {
        e = preloadNeighborKernels();
    }
    if (e == cudaSuccess) {
        e = preloadNeighborVKernels();
    }
    if (e == cudaSuccess) {
        e = preloadMoveBulkKernel();
    }
    if (e == cudaSuccess) {
        e = preloadNvlsKernels();
    }
    if (e == cudaSuccess) {
        e = preloadStateKernels();
    }
    if (e == cudaSuccess) {
        e = preloadSnapshotKernels();
    }
    if (e == cudaSuccess) {
        e = preloadRmaKernels();
    }
    return e;
}

} // namespace fb
