// One MPI program that checks every reduction call on every datatype and op,
// on every kind of buffer: the symmetric heap at offset 0, the heap at an
// offset that is not a multiple of 16, cudaMalloc memory at an odd element
// offset (with a GPU) and host memory.  Run by test_mpi_device_reduce.cpp.
//
// Inputs come from a seed every rank knows, so every rank computes every
// peer's input and the expected result: a host fold in rank order with the
// element rules of faabric/util/reduce_ops.h.  Float SUM/PROD inputs are
// small integers and powers of two, whose sums and products are exact, so the
// host plane (which folds in arrival order) must match the same fold bit for
// bit.  A NaN matches any NaN; pair padding is not compared.
//
// Every rank runs every call and collects failures instead of returning at
// the first one, so no peer is left waiting in a collective.
#pragma once

#include <faabric/device/communicator.h>
#include <faabric/device/cuda_driver.h>
#include <faabric/mpi/MpiWorldRegistry.h>
#include <faabric/mpi/mpi.h>
#include <faabric/mpi/mpi_runtime.h>
#include <faabric/util/reduce_ops.h>

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace mpi_device_reduce {

enum class Place
{
    Heap,      // MPI_Alloc_mem(MPI_INFO_FAABRIC_DEVICE), 16-byte aligned
    HeapShift, // the same memory, not 16-byte aligned
    CudaOdd,   // cudaMalloc, one element past a 16-byte boundary
    Host
};

inline const char* placeName(Place p)
{
    switch (p) {
        case Place::Heap:
            return "heap";
        case Place::HeapShift:
            return "heap+shift";
        case Place::CudaOdd:
            return "cudaMalloc+1";
        default:
            return "host";
    }
}

// How the elements of a datatype combine
enum class Kind
{
    I8, U8, I16, U16, I32, U32, I64, U64, F32, F64, F16, BF16, P_F64, P_F32, P_I32, P_I64
};

struct Type
{
    MPI_Datatype dt;
    const char* name;
    Kind kind;
    int per = 1; // base elements per element (MPI_Type_contiguous)
};

inline std::vector<Type> baseTypes()
{
    return {
        { MPI_INT8_T, "MPI_INT8_T", Kind::I8 },
        { MPI_CHAR, "MPI_CHAR", Kind::I8 },
        { MPI_UINT8_T, "MPI_UINT8_T", Kind::U8 },
        { MPI_BYTE, "MPI_BYTE", Kind::U8 },
        { MPI_C_BOOL, "MPI_C_BOOL", Kind::U8 },
        { MPI_INT16_T, "MPI_INT16_T", Kind::I16 },
        { MPI_UINT16_T, "MPI_UINT16_T", Kind::U16 },
        { MPI_INT32_T, "MPI_INT32_T", Kind::I32 },
        { MPI_INT, "MPI_INT", Kind::I32 },
        { MPI_UINT32_T, "MPI_UINT32_T", Kind::U32 },
        { MPI_UINT_T, "MPI_UINT_T", Kind::U32 },
        { MPI_INT64_T, "MPI_INT64_T", Kind::I64 },
        { MPI_LONG, "MPI_LONG", Kind::I64 },
        { MPI_LONG_LONG, "MPI_LONG_LONG", Kind::I64 },
        { MPI_LONG_LONG_INT, "MPI_LONG_LONG_INT", Kind::I64 },
        { MPI_UINT64_T, "MPI_UINT64_T", Kind::U64 },
        { MPI_FLOAT, "MPI_FLOAT", Kind::F32 },
        { MPI_DOUBLE, "MPI_DOUBLE", Kind::F64 },
        { MPI_HALF, "MPI_HALF", Kind::F16 },
        { MPI_BFLOAT16, "MPI_BFLOAT16", Kind::BF16 },
        { MPI_DOUBLE_INT, "MPI_DOUBLE_INT", Kind::P_F64 },
        { MPI_FLOAT_INT, "MPI_FLOAT_INT", Kind::P_F32 },
        { MPI_2INT, "MPI_2INT", Kind::P_I32 },
        { MPI_LONG_INT, "MPI_LONG_INT", Kind::P_I64 },
    };
}

struct Op
{
    MPI_Op op;
    const char* name;
};

inline std::vector<Op> builtinOps()
{
    return { { MPI_MAX, "MPI_MAX" },   { MPI_MIN, "MPI_MIN" },       { MPI_SUM, "MPI_SUM" },
             { MPI_PROD, "MPI_PROD" }, { MPI_LAND, "MPI_LAND" },     { MPI_LOR, "MPI_LOR" },
             { MPI_LXOR, "MPI_LXOR" }, { MPI_BAND, "MPI_BAND" },     { MPI_BOR, "MPI_BOR" },
             { MPI_BXOR, "MPI_BXOR" }, { MPI_MAXLOC, "MPI_MAXLOC" }, { MPI_MINLOC, "MPI_MINLOC" } };
}

inline bool isPair(Kind k)
{
    return k == Kind::P_F64 || k == Kind::P_F32 || k == Kind::P_I32 || k == Kind::P_I64;
}

inline bool isFloat(Kind k)
{
    return k == Kind::F32 || k == Kind::F64 || k == Kind::F16 || k == Kind::BF16;
}

inline bool isLoc(int op)
{
    return op == FAABRIC_OP_MAXLOC || op == FAABRIC_OP_MINLOC;
}

inline bool isArith(int op)
{
    return op == FAABRIC_OP_MAX || op == FAABRIC_OP_MIN || op == FAABRIC_OP_SUM || op == FAABRIC_OP_PROD;
}

inline bool isLogical(int op)
{
    return op == FAABRIC_OP_LAND || op == FAABRIC_OP_LOR || op == FAABRIC_OP_LXOR;
}

// The pairs MPI reductions define: integers take every op but the location
// ops; f32/f64 the arithmetic and logical ops; f16/bf16 the arithmetic ops;
// the {value, index} pairs only MAXLOC/MINLOC
inline bool defined(const Type& t, int op)
{
    if (isPair(t.kind)) {
        return isLoc(op);
    }
    if (t.kind == Kind::F16 || t.kind == Kind::BF16) {
        return isArith(op);
    }
    if (isFloat(t.kind)) {
        return isArith(op) || isLogical(op);
    }
    return !isLoc(op);
}

// The pairs the device kernels implement (a contiguous type never reaches them)
inline bool onDevice(const Type& t, int op)
{
    if (t.per != 1 || !defined(t, op)) {
        return false;
    }
    return !isFloat(t.kind) || isArith(op);
}

inline size_t kindSize(Kind k)
{
    switch (k) {
        case Kind::I8:
        case Kind::U8:
            return 1;
        case Kind::I16:
        case Kind::U16:
        case Kind::F16:
        case Kind::BF16:
            return 2;
        case Kind::I32:
        case Kind::U32:
        case Kind::F32:
            return 4;
        case Kind::I64:
        case Kind::U64:
        case Kind::F64:
        case Kind::P_F32:
        case Kind::P_I32:
            return 8;
        default:
            return 16;
    }
}

inline uint64_t mix(uint64_t x)
{
    x += 0x9e3779b97f4a7c15ull;
    x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
    x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
    return x ^ (x >> 31);
}

// ---------------------------------------------------------------- values ----
inline float h2f(uint16_t b, bool bf)
{
    if (bf) {
        __nv_bfloat16_raw r;
        r.x = b;
        return __bfloat162float(__nv_bfloat16(r));
    }
    __half_raw r;
    r.x = b;
    return __half2float(__half(r));
}

inline uint16_t f2h(float f, bool bf)
{
    if (bf) {
        if (std::isnan(f)) {
            return 0x7fc0;
        }
        return __nv_bfloat16_raw(__float2bfloat16_rn(f)).x;
    }
    return __half_raw(__float2half_rn(f)).x;
}

// Floats whose sums and products over up to 8 ranks are exact in every
// float type
inline double exactValue(uint64_t r)
{
    static const double v[] = { 0.5, -0.5, 1.0, -1.0, 2.0, -2.0, 3.0, 0.0, -0.0, 0.25 };
    return v[r % 10];
}

// Floats for MAX/MIN: the edges (NaN, signed zeros, infinities) and random
// bit patterns
inline double edgeValue(uint64_t r)
{
    switch (r % 8) {
        case 0:
            return NAN;
        case 1:
            return 0.0;
        case 2:
            return -0.0;
        case 3:
            return (r & 8) ? INFINITY : -INFINITY;
        default:
            return std::ldexp((double)(int64_t)(r >> 16) / (double)(1ull << 47), (int)((r >> 8) % 40) - 20);
    }
}

// Element `i` of rank `rank`'s input, written to `out` (kindSize bytes)
inline void inputElem(Kind k, int op, uint64_t seed, int rank, size_t i, uint8_t* out)
{
    const uint64_t r = mix(seed ^ mix(((uint64_t)rank << 40) ^ (uint64_t)i));
    memset(out, 0, kindSize(k));
    if (isPair(k)) {
        const int32_t idx = (int32_t)((r >> 20) % 2000) - 1000;
        const int64_t v = (int64_t)(r % 5) - 2; // few values: many ties
        switch (k) {
            case Kind::P_F64: {
                double d = (double)v;
                memcpy(out, &d, 8);
                memcpy(out + 8, &idx, 4);
                break;
            }
            case Kind::P_F32: {
                float f = (float)v;
                memcpy(out, &f, 4);
                memcpy(out + 4, &idx, 4);
                break;
            }
            case Kind::P_I32: {
                int32_t x = (int32_t)v;
                memcpy(out, &x, 4);
                memcpy(out + 4, &idx, 4);
                break;
            }
            default:
                memcpy(out, &v, 8);
                memcpy(out + 8, &idx, 4);
        }
        return;
    }
    if (isFloat(k)) {
        double d = (op == FAABRIC_OP_MAX || op == FAABRIC_OP_MIN) ? edgeValue(r) : exactValue(r);
        if (k == Kind::F32) {
            float f = (float)d;
            memcpy(out, &f, 4);
        } else if (k == Kind::F64) {
            memcpy(out, &d, 8);
        } else {
            uint16_t h = f2h((float)d, k == Kind::BF16);
            memcpy(out, &h, 2);
        }
        return;
    }
    uint64_t x = mix(r);
    if (isLogical(op)) {
        // zero, or non-zero with a zero low byte, or anything
        x = (r % 3 == 0) ? 0 : (r % 3 == 1 ? (x | 0x100) & ~(uint64_t)0xff : x);
    }
    memcpy(out, &x, kindSize(k));
}

template<typename T>
inline void combineInt(int op, uint8_t* accRaw, const uint8_t* inRaw)
{
    using faabric::util::reduceMax;
    using faabric::util::reduceMin;
    using faabric::util::reduceProd;
    using faabric::util::reduceSum;
    T a, b;
    memcpy(&a, accRaw, sizeof(T));
    memcpy(&b, inRaw, sizeof(T));
    T r = a;
    switch (op) {
        case FAABRIC_OP_MAX:
            r = reduceMax(a, b);
            break;
        case FAABRIC_OP_MIN:
            r = reduceMin(a, b);
            break;
        case FAABRIC_OP_SUM:
            r = reduceSum(a, b);
            break;
        case FAABRIC_OP_PROD:
            r = reduceProd(a, b);
            break;
        case FAABRIC_OP_LAND:
            r = (T)(a != (T)0 && b != (T)0);
            break;
        case FAABRIC_OP_LOR:
            r = (T)(a != (T)0 || b != (T)0);
            break;
        case FAABRIC_OP_LXOR:
            r = (T)((a != (T)0) != (b != (T)0));
            break;
        default:
            if constexpr (std::is_integral_v<T>) {
                r = op == FAABRIC_OP_BAND ? (T)(a & b) : op == FAABRIC_OP_BOR ? (T)(a | b) : (T)(a ^ b);
            }
    }
    memcpy(accRaw, &r, sizeof(T));
}

template<typename V>
inline void combineLoc(int op, uint8_t* acc, const uint8_t* in)
{
    V va, vb;
    int32_t ia, ib;
    memcpy(&va, acc, sizeof(V));
    memcpy(&vb, in, sizeof(V));
    memcpy(&ia, acc + sizeof(V), 4);
    memcpy(&ib, in + sizeof(V), 4);
    const bool better = op == FAABRIC_OP_MAXLOC ? vb > va : vb < va;
    if (better || (vb == va && ib < ia)) {
        memcpy(acc, &vb, sizeof(V));
        memcpy(acc + sizeof(V), &ib, 4);
    }
}

// acc = op(acc, in), one element
inline void combine(Kind k, int op, uint8_t* acc, const uint8_t* in)
{
    switch (k) {
        case Kind::I8:
            return combineInt<int8_t>(op, acc, in);
        case Kind::U8:
            return combineInt<uint8_t>(op, acc, in);
        case Kind::I16:
            return combineInt<int16_t>(op, acc, in);
        case Kind::U16:
            return combineInt<uint16_t>(op, acc, in);
        case Kind::I32:
            return combineInt<int32_t>(op, acc, in);
        case Kind::U32:
            return combineInt<uint32_t>(op, acc, in);
        case Kind::I64:
            return combineInt<int64_t>(op, acc, in);
        case Kind::U64:
            return combineInt<uint64_t>(op, acc, in);
        case Kind::F32:
            return combineInt<float>(op, acc, in);
        case Kind::F64:
            return combineInt<double>(op, acc, in);
        case Kind::F16:
        case Kind::BF16: {
            const bool bf = k == Kind::BF16;
            uint16_t a, b;
            memcpy(&a, acc, 2);
            memcpy(&b, in, 2);
            uint8_t fa[4], fb[4];
            float x = h2f(a, bf), y = h2f(b, bf);
            memcpy(fa, &x, 4);
            memcpy(fb, &y, 4);
            combineInt<float>(op, fa, fb);
            memcpy(&x, fa, 4);
            uint16_t r = f2h(x, bf);
            memcpy(acc, &r, 2);
            return;
        }
        case Kind::P_F64:
            return combineLoc<double>(op, acc, in);
        case Kind::P_F32:
            return combineLoc<float>(op, acc, in);
        case Kind::P_I32:
            return combineLoc<int32_t>(op, acc, in);
        default:
            return combineLoc<int64_t>(op, acc, in);
    }
}

// Equal bit for bit, except that a NaN matches any NaN and pair padding is
// not compared
inline bool sameElem(Kind k, const uint8_t* a, const uint8_t* b)
{
    auto nan = [&](const uint8_t* p) {
        switch (k) {
            case Kind::F32:
            case Kind::P_F32: {
                float f;
                memcpy(&f, p, 4);
                return std::isnan(f);
            }
            case Kind::F64:
            case Kind::P_F64: {
                double d;
                memcpy(&d, p, 8);
                return std::isnan(d);
            }
            case Kind::F16:
            case Kind::BF16: {
                uint16_t h;
                memcpy(&h, p, 2);
                return std::isnan(h2f(h, k == Kind::BF16));
            }
            default:
                return false;
        }
    };
    if (isPair(k)) {
        const size_t vb = (k == Kind::P_F64 || k == Kind::P_I64) ? 8 : 4;
        const bool vSame = memcmp(a, b, vb) == 0 || (nan(a) && nan(b));
        return vSame && memcmp(a + vb, b + vb, 4) == 0;
    }
    return memcmp(a, b, kindSize(k)) == 0 || (nan(a) && nan(b));
}

// ------------------------------------------------------------- buffers ----
inline bool onGpu(const void* p)
{
    if (p == nullptr || !faabric::device::cudaAvailable() || faabric::device::Communicator::isLoopbackHeapPointer(p)) {
        return false;
    }
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return attr.type == cudaMemoryTypeDevice;
}

inline void copy(void* dst, const void* src, size_t n)
{
    if (n == 0) {
        return;
    }
    if (onGpu(dst) || onGpu(src)) {
        cudaMemcpy(dst, src, n, cudaMemcpyDefault);
        cudaDeviceSynchronize();
    } else {
        memcpy(dst, src, n);
    }
}

constexpr size_t GUARD = 16;

// `bytes` of data with GUARD bytes of a known pattern on each side, at the
// offset the placement asks for
struct Buffer
{
    Place place;
    uint8_t* base = nullptr;
    uint8_t* data = nullptr;
    size_t bytes = 0;
    size_t total = 0;

    Buffer(Place p, size_t n, size_t esize)
      : place(p)
      , bytes(n)
    {
        size_t shift = 0;
        if (p == Place::HeapShift) {
            shift = esize < 16 ? esize : 8;
        } else if (p == Place::CudaOdd) {
            shift = esize;
        }
        total = GUARD + shift + n + GUARD;
        if (p == Place::Heap || p == Place::HeapShift) {
            if (MPI_Alloc_mem((MPI_Aint)total, MPI_INFO_FAABRIC_DEVICE, &base) != MPI_SUCCESS) {
                base = nullptr;
            }
        } else if (p == Place::CudaOdd) {
            if (cudaMalloc((void**)&base, total) != cudaSuccess) {
                cudaGetLastError();
                base = nullptr;
            }
        } else {
            base = (uint8_t*)malloc(total);
        }
        data = base == nullptr ? nullptr : base + GUARD + shift;
    }

    ~Buffer()
    {
        if (base == nullptr) {
            return;
        }
        if (place == Place::CudaOdd) {
            cudaFree(base);
        } else if (place == Place::Host) {
            free(base);
        } else {
            MPI_Free_mem(base);
        }
    }

    Buffer(const Buffer&) = delete;
    Buffer& operator=(const Buffer&) = delete;

    // the whole allocation: guards, data and whatever the shift skipped
    std::vector<uint8_t> image() const
    {
        std::vector<uint8_t> v(total);
        copy(v.data(), base, total);
        return v;
    }

    void setImage(const std::vector<uint8_t>& v) { copy(base, v.data(), total); }

    size_t dataOff() const { return (size_t)(data - base); }
};

// A recognisable pattern for everything a call must not write
inline std::vector<uint8_t> guardImage(size_t n, uint64_t seed)
{
    std::vector<uint8_t> v(n);
    for (size_t i = 0; i < n; i++) {
        v[i] = (uint8_t)mix(seed + i);
    }
    return v;
}

// --------------------------------------------------------------- program ----
struct Ctx
{
    int rank;
    int size;
    faabric::mpi::MpiWorld* world;
    std::vector<std::string> failures;

    void fail(const std::string& what)
    {
        if (failures.size() < 20) {
            failures.push_back("rank " + std::to_string(rank) + ": " + what);
        }
    }
};

struct Case
{
    const Type* t;
    const Op* op;
    size_t count; // elements per rank's block
    Place place;
    uint64_t seed;

    size_t esize() const { return kindSize(t->kind) * (size_t)t->per; }
    int opId() const { return op->op->id; }
    std::string name() const
    {
        return std::string(t->name) + (t->per > 1 ? " x" + std::to_string(t->per) : "") + " " + op->name +
               " count=" + std::to_string(count) + " " + placeName(place);
    }
};

// Rank `r`'s input: `n` elements of the case's type
inline std::vector<uint8_t> inputOf(const Case& c, int r, size_t n)
{
    const size_t kb = kindSize(c.t->kind);
    std::vector<uint8_t> v(n * c.esize());
    for (size_t i = 0; i < n * (size_t)c.t->per; i++) {
        inputElem(c.t->kind, c.opId(), c.seed, r, i, v.data() + i * kb);
    }
    return v;
}

// The fold of the inputs of world ranks `ranks` (a communicator's members in
// its order), in that order
inline std::vector<uint8_t> foldOver(const Case& c, const std::vector<int>& ranks, size_t n)
{
    std::vector<uint8_t> acc = inputOf(c, ranks[0], n);
    const size_t kb = kindSize(c.t->kind);
    for (size_t i = 1; i < ranks.size(); i++) {
        std::vector<uint8_t> in = inputOf(c, ranks[i], n);
        for (size_t off = 0; off < acc.size(); off += kb) {
            combine(c.t->kind, c.opId(), acc.data() + off, in.data() + off);
        }
    }
    return acc;
}

// The fold of ranks [0, upto) in rank order
inline std::vector<uint8_t> foldOf(const Case& c, int upto, size_t n)
{
    std::vector<int> ranks(std::max(upto, 1));
    for (size_t r = 0; r < ranks.size(); r++) {
        ranks[r] = (int)r;
    }
    return foldOver(c, ranks, n);
}

// A buffer image: each region's `want` at its offset (compared element by
// element as `c`'s type), every other byte as in `before`
struct Region
{
    size_t off;
    std::vector<uint8_t> want;
};

inline void checkRegions(Ctx& x,
                         const Case& c,
                         const std::string& call,
                         const std::vector<uint8_t>& got,
                         const std::vector<uint8_t>& before,
                         const std::vector<Region>& regions)
{
    std::vector<bool> result(got.size(), false);
    for (const Region& r : regions) {
        std::fill(result.begin() + (long)r.off, result.begin() + (long)(r.off + r.want.size()), true);
    }
    for (size_t i = 0; i < got.size(); i++) {
        if (!result[i] && got[i] != before[i]) {
            x.fail(c.name() + " " + call + ": byte " + std::to_string(i) + " outside the result changed");
            return;
        }
    }
    const size_t kb = kindSize(c.t->kind);
    for (const Region& r : regions) {
        for (size_t e = 0; e < r.want.size(); e += kb) {
            if (!sameElem(c.t->kind, got.data() + r.off + e, r.want.data() + e)) {
                x.fail(c.name() + " " + call + ": element " + std::to_string(e / kb) + " differs");
                return;
            }
        }
    }
}

// A buffer image: `want` at each of `offs`, every other byte as in `before`
inline void checkImage(Ctx& x,
                       const Case& c,
                       const std::string& call,
                       const std::vector<uint8_t>& got,
                       const std::vector<uint8_t>& before,
                       const std::vector<size_t>& offs,
                       const std::vector<uint8_t>* want)
{
    std::vector<Region> regions;
    for (size_t off : offs) {
        regions.push_back({ off, want != nullptr ? *want : std::vector<uint8_t>() });
    }
    checkRegions(x, c, call, got, before, regions);
}

// The world's count of device collectives, once every rank has reached this
// point: the count is the world's, so a rank reads it between barriers
inline uint64_t deviceCalls(Ctx& x)
{
    MPI_Barrier(MPI_COMM_WORLD);
    const uint64_t n = x.world->getDeviceCollectiveCount();
    MPI_Barrier(MPI_COMM_WORLD);
    return n;
}

// Runs one call on fresh buffers: `send` holds this rank's input of
// `sendCount` elements (or nothing for `inPlace`), `recv` is `recvCount`
// elements of guard pattern.  Checks the return code, the result (`want`,
// null for none), that send is unchanged and every byte around the result,
// and that the call issued `deviceDelta` device collectives on every rank.
template<class Call>
void runCall(Ctx& x,
             const Case& c,
             const std::string& callName,
             size_t sendCount,
             size_t recvCount,
             bool inPlace,
             const std::vector<uint8_t>* want,
             int deviceDelta,
             Call&& call)
{
    const size_t es = c.esize();
    const bool ok = defined(*c.t, c.opId());
    Buffer send(c.place, sendCount * es, es);
    Buffer recv(c.place, std::max(recvCount, inPlace ? sendCount : 0) * es, es);
    if (send.base == nullptr || recv.base == nullptr) {
        x.fail(c.name() + " " + callName + ": allocation failed");
        return;
    }
    const std::vector<uint8_t> in = inputOf(c, x.rank, sendCount);
    std::vector<uint8_t> sendImg = guardImage(send.total, c.seed + 1);
    std::vector<uint8_t> recvImg = guardImage(recv.total, c.seed + 2);
    if (inPlace) {
        std::copy(in.begin(), in.end(), recvImg.begin() + (long)recv.dataOff());
    } else {
        std::copy(in.begin(), in.end(), sendImg.begin() + (long)send.dataOff());
    }
    send.setImage(sendImg);
    recv.setImage(recvImg);
    const uint64_t before = deviceCalls(x);
    const int rc = call(inPlace ? (uint8_t*)MPI_IN_PLACE : send.data, recv.data);
    const uint64_t calls = deviceCalls(x) - before;
    if (rc != (ok ? MPI_SUCCESS : MPI_ERR_OP)) {
        x.fail(c.name() + " " + callName + ": returned " + std::to_string(rc));
    }
    if (!inPlace) {
        checkImage(x, c, callName + " (send)", send.image(), sendImg, {}, nullptr);
    }
    if (ok && want != nullptr) {
        checkImage(x, c, callName, recv.image(), recvImg, { recv.dataOff() }, want);
    } else {
        checkImage(x, c, callName, recv.image(), recvImg, {}, nullptr);
    }
    const bool device = c.place != Place::Host;
    const int expected = (device && onDevice(*c.t, c.opId())) ? deviceDelta * x.size : 0;
    if (calls != (uint64_t)expected) {
        x.fail(c.name() + " " + callName + ": " + std::to_string(calls) + " device collectives, expected " +
               std::to_string(expected));
    }
}

inline std::vector<uint8_t> slice(const std::vector<uint8_t>& v, size_t off, size_t n)
{
    return std::vector<uint8_t>(v.begin() + (long)off, v.begin() + (long)(off + n));
}

// Every blocking call of one case
inline void blockingCalls(Ctx& x, const Case& c, size_t stageBytes)
{
    const int n = x.size;
    const size_t es = c.esize();
    const size_t count = c.count;
    MPI_Datatype dt = c.t->dt;
    MPI_Op op = c.op->op;
    const std::vector<uint8_t> all = foldOf(c, n, count);

    for (bool inPlace : { false, true }) {
        runCall(x, c, inPlace ? "MPI_Allreduce in place" : "MPI_Allreduce", count, count, inPlace, &all, 1,
                [&](uint8_t* s, uint8_t* r) { return MPI_Allreduce(s, r, (int)count, dt, op, MPI_COMM_WORLD); });
    }
    for (int root = 0; root < n; root++) {
        const bool me = root == x.rank;
        runCall(x, c, "MPI_Reduce root " + std::to_string(root), count, me ? count : 0, me, me ? &all : nullptr, 1,
                [&](uint8_t* s, uint8_t* r) { return MPI_Reduce(s, r, (int)count, dt, op, root, MPI_COMM_WORLD); });
    }
    const std::vector<uint8_t> prefix = foldOf(c, x.rank + 1, count);
    runCall(x, c, "MPI_Scan", count, count, false, &prefix, 1,
            [&](uint8_t* s, uint8_t* r) { return MPI_Scan(s, r, (int)count, dt, op, MPI_COMM_WORLD); });

    // reduce-scatter: blocks of `count`, and uneven blocks of count + r
    const std::vector<uint8_t> full = foldOf(c, n, count * (size_t)n);
    const std::vector<uint8_t> mine = slice(full, (size_t)x.rank * count * es, count * es);
    // the device takes it when the slices are whole vectors and the message
    // fits the staging area (or needs none); otherwise the host does
    const bool staged = c.place != Place::Heap;
    const int rsDevice =
      ((count * es) % 16 == 0 && (!staged || count * es * (size_t)n <= stageBytes)) ? 1 : 0;
    runCall(x, c, "MPI_Reduce_scatter_block", count * (size_t)n, count, false, &mine, rsDevice,
            [&](uint8_t* s, uint8_t* r) { return MPI_Reduce_scatter_block(s, r, (int)count, dt, op, MPI_COMM_WORLD); });
    std::vector<int> counts(n);
    size_t total = 0, myOff = 0;
    for (int r = 0; r < n; r++) {
        counts[r] = (int)count + r;
        if (r < x.rank) {
            myOff += (size_t)counts[r];
        }
        total += (size_t)counts[r];
    }
    const std::vector<uint8_t> uneven = foldOf(c, n, total);
    const std::vector<uint8_t> myUneven = slice(uneven, myOff * es, (size_t)counts[x.rank] * es);
    runCall(x, c, "MPI_Reduce_scatter uneven", total, (size_t)counts[x.rank], false, &myUneven, 0,
            [&](uint8_t* s, uint8_t* r) { return MPI_Reduce_scatter(s, r, counts.data(), dt, op, MPI_COMM_WORLD); });
}

// A burst of `k` MPI_Iallreduce calls on one pair of buffers, waited for
// together
inline void iallreduceBurst(Ctx& x, const Case& c, int k)
{
    const size_t es = c.esize();
    const size_t count = c.count;
    const size_t stride = ((count * es + 15) / 16) * 16 + (c.place == Place::HeapShift ? 16 : 0);
    const std::vector<uint8_t> all = foldOf(c, x.size, count);
    const std::string name = "MPI_Iallreduce burst of " + std::to_string(k);
    const bool ok = defined(*c.t, c.opId());
    Buffer send(c.place, stride * (size_t)k, es);
    Buffer recv(c.place, stride * (size_t)k, es);
    if (send.base == nullptr || recv.base == nullptr) {
        x.fail(c.name() + " " + name + ": allocation failed");
        return;
    }
    const std::vector<uint8_t> in = inputOf(c, x.rank, count);
    std::vector<uint8_t> sendImg = guardImage(send.total, c.seed + 3);
    const std::vector<uint8_t> recvImg = guardImage(recv.total, c.seed + 4);
    for (int j = 0; j < k; j++) {
        std::copy(in.begin(), in.end(), sendImg.begin() + (long)(send.dataOff() + stride * (size_t)j));
    }
    send.setImage(sendImg);
    recv.setImage(recvImg);
    const uint64_t before = deviceCalls(x);
    std::vector<MPI_Request> reqs(k, nullptr);
    int bad = 0;
    for (int j = 0; j < k; j++) {
        const int rc = MPI_Iallreduce(send.data + stride * (size_t)j, recv.data + stride * (size_t)j, (int)count,
                                      c.t->dt, c.op->op, MPI_COMM_WORLD, &reqs[j]);
        if (rc != (ok ? MPI_SUCCESS : MPI_ERR_OP) || (!ok && reqs[j] != nullptr)) {
            bad++;
        }
    }
    if (ok) {
        MPI_Waitall(k, reqs.data(), MPI_STATUSES_IGNORE);
    }
    if (bad != 0) {
        x.fail(c.name() + " " + name + ": " + std::to_string(bad) + " calls returned the wrong code");
    }
    const uint64_t calls = deviceCalls(x) - before;
    const uint64_t expected = (c.place != Place::Host && onDevice(*c.t, c.opId())) ? (uint64_t)(k * x.size) : 0;
    if (calls != expected) {
        x.fail(c.name() + " " + name + ": " + std::to_string(calls) + " device collectives, expected " +
               std::to_string(expected));
    }
    checkImage(x, c, name + " (send)", send.image(), sendImg, {}, nullptr);
    std::vector<size_t> offs;
    for (int j = 0; ok && j < k; j++) {
        offs.push_back(recv.dataOff() + stride * (size_t)j);
    }
    checkImage(x, c, name, recv.image(), recvImg, offs, ok ? &all : nullptr);
}

struct Options
{
    bool cudaMalloc = false; // add the cudaMalloc placement (needs a GPU)
};

// Returns 0, or 1 with the first failures in `why`
inline int body(int rank, int size, int worldId, const Options& o, std::string* why)
{
    Ctx x{ rank, size, &faabric::mpi::getMpiWorldRegistry().getWorld(worldId), {} };
    auto comm = x.world->getDeviceComm(rank);
    if (comm == nullptr) {
        *why = "rank " + std::to_string(rank) + ": no device communicator";
        return 1;
    }
    const auto& cfg = comm->config();
    std::vector<Place> places{ Place::Heap, Place::HeapShift, Place::Host };
    if (o.cudaMalloc) {
        places.push_back(Place::CudaOdd);
    }
    std::vector<Type> types = baseTypes();
    MPI_Datatype float3 = nullptr;
    MPI_Type_contiguous(3, MPI_FLOAT, &float3);
    MPI_Type_commit(&float3);
    types.push_back({ float3, "MPI_Type_contiguous(3, MPI_FLOAT)", Kind::F32, 3 });
    const std::vector<Op> ops = builtinOps();

    uint64_t seed = 1;
    // every (datatype, op) pair, defined or not, on every placement, at
    // a count below one vector and one with a tail
    for (const Type& t : types) {
        for (const Op& op : ops) {
            for (Place p : places) {
                for (size_t count : { (size_t)1, (size_t)7 }) {
                    Case c{ &t, &op, count, p, mix(seed++) };
                    blockingCalls(x, c, cfg.stageBytes);
                    iallreduceBurst(x, c, 3);
                }
            }
        }
    }
    // the sizes that select the algorithms and the staging pieces, for a few
    // pairs of every element width
    const std::vector<std::pair<int, int>> sized{ { 1, 9 }, { 7, 2 }, { 8, 0 }, { 12, 1 },
                                                  { 16, 3 }, { 17, 0 }, { 19, 3 }, { 20, 10 } };
    for (auto [ti, oi] : sized) {
        const Type& t = types[ti];
        const Op& op = ops[oi];
        const size_t es = kindSize(t.kind);
        const std::vector<size_t> counts{ cfg.llMaxBytes / es - 1, cfg.llMaxBytes / es + 1,
                                          cfg.oneShotMaxBytes / es + 1, cfg.stageBytes / es + 3 };
        for (Place p : places) {
            for (size_t count : counts) {
                Case c{ &t, &op, count, p, mix(seed++) };
                blockingCalls(x, c, cfg.stageBytes);
                iallreduceBurst(x, c, 3);
            }
        }
    }
    MPI_Type_free(&float3);

    if (x.failures.empty()) {
        return 0;
    }
    for (const std::string& f : x.failures) {
        *why += f + "\n";
    }
    return 1;
}

}
