// One MPI program that checks MPI_Accumulate, MPI_Get_accumulate,
// MPI_Fetch_and_op and MPI_Compare_and_swap on one kind of window.  Shared by
// the in-process tests (test_mpi_rma_atomics.cpp) and the `rma-atomics`
// function of faabric_worker, which runs it across worker processes.
//
// Every check compares exact bytes against a closed form: the operations used
// give the same result in any order (integer SUM/PROD wrap, logical and
// bitwise ops, float MAX/MIN with NaN and ±0, MAXLOC/MINLOC with ties, float
// SUM/PROD of small powers and integers), so concurrent origins in this
// process and in other processes must land on exactly these values.
#pragma once

#include <faabric/device/comm_abi.h>
#include <faabric/device/communicator.h>
#include <faabric/device/cuda_driver.h>
#include <faabric/mpi/MpiWorld.h>
#include <faabric/mpi/MpiWorldRegistry.h>
#include <faabric/mpi/mpi.h>
#include <faabric/util/reduce_ops.h>

#include "launch_api.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <set>
#include <string>
#include <vector>

namespace rma_atomics {

enum class WindowMemory
{
    Host,     // MPI_Win_create over host memory
    Heap,     // MPI_Alloc_mem(MPI_INFO_FAABRIC_DEVICE): the symmetric heap
    CudaMalloc // MPI_Win_create over cudaMalloc memory
};

struct Setup
{
    WindowMemory window = WindowMemory::Host;
    // origin, compare and result buffers in cudaMalloc memory
    bool deviceBuffers = false;
    // count the communicator launches of heap-window calls
    bool countLaunches = false;
};

constexpr size_t WINDOW_BYTES = 8192;
constexpr size_t EXACT_OFF = 0;      // [0, 1024): one (datatype, op) case at a time
constexpr int EXACT_N = 37;          // elements per case (odd: no vector multiple)
constexpr size_t TICKET_OFF = 1024;  // counters and their busy neighbours
constexpr size_t CAS_OFF = 1280;
constexpr size_t GETACC_OFF = 2048;  // 64 bytes per origin
constexpr size_t ORDER_OFF = 6144;   // 16 bytes per origin

#define RMA_CHECK(cond)                                                        \
    do {                                                                       \
        if (!(cond)) {                                                         \
            *why = "rank " + std::to_string(rank) + ": check failed at line " + std::to_string(__LINE__) + ": " #cond; \
            return 1;                                                          \
        }                                                                      \
    } while (0)

inline uint64_t mix(uint64_t x)
{
    x += 0x9e3779b97f4a7c15ull;
    x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
    x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
    return x ^ (x >> 31);
}

inline uint64_t seedOf(int a, int b, int c, int d, int e)
{
    return mix(mix(mix(mix(mix((uint64_t)a) + (uint64_t)b) + (uint64_t)c) + (uint64_t)d) + (uint64_t)e);
}

// True if the pointer is CUDA device memory (the loopback heaps are not)
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
    return attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged;
}

inline void copyBytes(void* dst, const void* src, size_t n)
{
    if (n == 0) {
        return;
    }
    if (onGpu(dst) || onGpu(src)) {
        cudaMemcpy(dst, src, n, cudaMemcpyDefault);
        // (a copy from pageable memory may return before its DMA lands)
        cudaStreamSynchronize(nullptr);
    } else {
        memcpy(dst, src, n);
    }
}

// A buffer in host memory, or in cudaMalloc memory with a host shadow
struct Buffer
{
    std::vector<uint8_t> host;
    uint8_t* dev = nullptr;

    Buffer(size_t n, bool onDevice)
      : host(n, 0)
    {
        if (onDevice && cudaMalloc((void**)&dev, std::max<size_t>(n, 1)) != cudaSuccess) {
            cudaGetLastError();
            dev = nullptr;
            host.clear();
        }
    }
    ~Buffer()
    {
        if (dev != nullptr) {
            cudaFree(dev);
        }
    }
    Buffer(const Buffer&) = delete;
    Buffer& operator=(const Buffer&) = delete;

    bool ok() const { return !host.empty() || dev != nullptr; }
    uint8_t* ptr() { return dev != nullptr ? dev : host.data(); }
    void upload()
    {
        if (dev != nullptr) {
            cudaMemcpy(dev, host.data(), host.size(), cudaMemcpyHostToDevice);
            cudaStreamSynchronize(nullptr);
        }
    }
    // host shadow <- buffer
    const std::vector<uint8_t>& read()
    {
        if (dev != nullptr) {
            cudaMemcpy(host.data(), dev, host.size(), cudaMemcpyDeviceToHost);
        }
        return host;
    }
};

// ---- element rules (the closed forms) ----
inline uint16_t halfBits(float f)
{
    uint32_t u;
    memcpy(&u, &f, 4);
    const uint16_t sign = (uint16_t)((u >> 16) & 0x8000);
    if (std::isnan(f)) {
        return 0x7e00;
    }
    if (f == 0.0f) {
        return sign;
    }
    // normal values exactly representable in f16 (the tests use no others)
    const int exp = (int)((u >> 23) & 0xff) - 127 + 15;
    return (uint16_t)(sign | (exp << 10) | ((u >> 13) & 0x3ff));
}

inline float halfValue(uint16_t h)
{
    const uint32_t sign = (uint32_t)(h & 0x8000) << 16;
    const int exp = (h >> 10) & 0x1f;
    const uint32_t man = h & 0x3ff;
    uint32_t u;
    if (exp == 0x1f) {
        u = sign | 0x7fc00000u;
    } else if (exp == 0 && man == 0) {
        u = sign;
    } else {
        u = sign | ((uint32_t)(exp - 15 + 127) << 23) | (man << 13);
    }
    float f;
    memcpy(&f, &u, 4);
    return f;
}

inline uint16_t bf16Bits(float f)
{
    uint32_t u;
    memcpy(&u, &f, 4);
    return std::isnan(f) ? (uint16_t)0x7fc0 : (uint16_t)(u >> 16);
}

inline float bf16Value(uint16_t h)
{
    uint32_t u = (uint32_t)h << 16;
    float f;
    memcpy(&f, &u, 4);
    return f;
}

template<typename T>
T scalarRule(int op, T a, T b)
{
    using namespace faabric::util;
    switch (op) {
        case FB_OP_SUM:
            return reduceSum(a, b);
        case FB_OP_PROD:
            return reduceProd(a, b);
        case FB_OP_MAX:
            return reduceMax(a, b);
        case FB_OP_MIN:
            return reduceMin(a, b);
        case FB_OP_REPLACE:
            return b;
        case FB_OP_NO_OP:
            return a;
        default:
            break;
    }
    if constexpr (std::is_integral_v<T>) {
        switch (op) {
            case FB_OP_LAND:
                return (T)(a != 0 && b != 0);
            case FB_OP_LOR:
                return (T)(a != 0 || b != 0);
            case FB_OP_LXOR:
                return (T)((a != 0) != (b != 0));
            case FB_OP_BAND:
                return (T)(a & b);
            case FB_OP_BOR:
                return (T)(a | b);
            case FB_OP_BXOR:
                return (T)(a ^ b);
            default:
                break;
        }
    }
    return a;
}

template<typename T>
void scalarCombine(int op, uint8_t* acc, const uint8_t* in)
{
    T a, b;
    memcpy(&a, acc, sizeof(T));
    memcpy(&b, in, sizeof(T));
    T r = scalarRule<T>(op, a, b);
    memcpy(acc, &r, sizeof(T));
}

// value, index; 16-byte pairs keep the target's padding (bytes 12..15)
template<typename V>
void pairCombine(int op, uint8_t* acc, const uint8_t* in)
{
    V av, bv;
    int32_t ai, bi;
    memcpy(&av, acc, sizeof(V));
    memcpy(&ai, acc + sizeof(V), 4);
    memcpy(&bv, in, sizeof(V));
    memcpy(&bi, in + sizeof(V), 4);
    bool takeB = op == FB_OP_REPLACE ||
                 (op == FB_OP_MAXLOC && (bv > av || (bv == av && bi < ai))) ||
                 (op == FB_OP_MINLOC && (bv < av || (bv == av && bi < ai)));
    if (takeB) {
        memcpy(acc, in, sizeof(V) + 4);
    }
}

// acc = op(acc, in) for one element of FbDtype `dt`
inline void combine(int dt, int op, uint8_t* acc, const uint8_t* in)
{
    switch (dt) {
        case FB_I8:
            return scalarCombine<int8_t>(op, acc, in);
        case FB_U8:
            return scalarCombine<uint8_t>(op, acc, in);
        case FB_I16:
            return scalarCombine<int16_t>(op, acc, in);
        case FB_U16:
            return scalarCombine<uint16_t>(op, acc, in);
        case FB_I32:
            return scalarCombine<int32_t>(op, acc, in);
        case FB_U32:
            return scalarCombine<uint32_t>(op, acc, in);
        case FB_I64:
            return scalarCombine<int64_t>(op, acc, in);
        case FB_U64:
            return scalarCombine<uint64_t>(op, acc, in);
        case FB_F32:
            return scalarCombine<float>(op, acc, in);
        case FB_F64:
            return scalarCombine<double>(op, acc, in);
        case FB_F16:
        case FB_BF16: {
            uint16_t a, b;
            memcpy(&a, acc, 2);
            memcpy(&b, in, 2);
            const bool h = dt == FB_F16;
            float r = scalarRule<float>(op, h ? halfValue(a) : bf16Value(a), h ? halfValue(b) : bf16Value(b));
            // a NaN result keeps the operand's bits (never two NaNs: see value())
            uint16_t bits = std::isnan(r) ? (std::isnan(h ? halfValue(a) : bf16Value(a)) ? a : b)
                                          : (h ? halfBits(r) : bf16Bits(r));
            memcpy(acc, &bits, 2);
            return;
        }
        case FB_F64_I32:
            return pairCombine<double>(op, acc, in);
        case FB_F32_I32:
            return pairCombine<float>(op, acc, in);
        case FB_I32_I32:
            return pairCombine<int32_t>(op, acc, in);
        case FB_I64_I32:
            return pairCombine<int64_t>(op, acc, in);
        default:
            return;
    }
}

// A value for element i of `who` (0..size-1 an origin, -1 the initial
// target) in a case of (dt, op), written to `out`.  Floats: small integers
// (SUM), powers of two (PROD), small integers with ±0 and NaN (MAX / MIN) where
// every element has at least one operand that is not NaN.
inline void value(int dt, int op, uint64_t h, int who, int i, uint8_t* out)
{
    const size_t n = fbDtypeSize(dt);
    memset(out, 0, n);
    const bool floaty = dt == FB_F32 || dt == FB_F64 || dt == FB_F16 || dt == FB_BF16;
    if (dt <= FB_U64) {
        uint64_t bits = h;
        if (op == FB_OP_LAND || op == FB_OP_LOR || op == FB_OP_LXOR) {
            bits = (h % 3 == 0) ? 0 : (h >> 8);
        }
        memcpy(out, &bits, n);
        return;
    }
    if (floaty) {
        double v;
        if (op == FB_OP_PROD) {
            const double choices[] = { 1.0, -1.0, 2.0, 0.5, -2.0 };
            v = choices[h % 5];
        } else if (op == FB_OP_SUM) {
            v = (double)((int)(h % 17) - 8);
        } else {
            v = (double)((int)(h % 9) - 4);
            if (h % 11 == 0) {
                v = (h & 1) ? -0.0 : 0.0;
            }
            // at most one NaN per element: the initial value or origin i % 5
            const bool nan = who < 0 ? (i % 7 == 3) : ((i + who) % 5 == 0 && i % 7 != 3);
            if (nan) {
                v = std::nan("");
            }
        }
        if (dt == FB_F32) {
            float f = (float)v;
            memcpy(out, &f, 4);
        } else if (dt == FB_F64) {
            memcpy(out, &v, 8);
        } else {
            uint16_t b = dt == FB_F16 ? halfBits((float)v) : bf16Bits((float)v);
            memcpy(out, &b, 2);
        }
        return;
    }
    // pairs: ties are likely (value in [-2, 2]), index in [0, 50)
    const int32_t idx = (int32_t)((h >> 16) % 50);
    const int vi = (int)(h % 5) - 2;
    switch (dt) {
        case FB_F64_I32: {
            double v = vi;
            memcpy(out, &v, 8);
            memcpy(out + 8, &idx, 4);
            memset(out + 12, who < 0 ? 0x5c : 0xab, 4);
            break;
        }
        case FB_F32_I32: {
            float v = (float)vi;
            memcpy(out, &v, 4);
            memcpy(out + 4, &idx, 4);
            break;
        }
        case FB_I32_I32: {
            int32_t v = vi;
            memcpy(out, &v, 4);
            memcpy(out + 4, &idx, 4);
            break;
        }
        case FB_I64_I32: {
            int64_t v = vi;
            memcpy(out, &v, 8);
            memcpy(out + 8, &idx, 4);
            memset(out + 12, who < 0 ? 0x5c : 0xab, 4);
            break;
        }
        default:
            break;
    }
}

// Every predefined MPI datatype with an element type
inline std::vector<MPI_Datatype> allDatatypes()
{
    return { MPI_INT8_T, MPI_INT16_T, MPI_INT32_T, MPI_INT,    MPI_INT64_T,    MPI_UINT8_T,   MPI_UINT16_T,
             MPI_UINT32_T, MPI_UINT_T, MPI_UINT64_T, MPI_LONG,   MPI_LONG_LONG,  MPI_LONG_LONG_INT, MPI_FLOAT,
             MPI_DOUBLE, MPI_DOUBLE_INT, MPI_CHAR,   MPI_C_BOOL, MPI_BYTE,       MPI_HALF,      MPI_BFLOAT16,
             MPI_FLOAT_INT, MPI_2INT,  MPI_LONG_INT };
}

inline std::vector<std::pair<MPI_Op, int>> allOps()
{
    return { { MPI_MAX, FB_OP_MAX },     { MPI_MIN, FB_OP_MIN },       { MPI_SUM, FB_OP_SUM },
             { MPI_PROD, FB_OP_PROD },   { MPI_LAND, FB_OP_LAND },     { MPI_LOR, FB_OP_LOR },
             { MPI_BAND, FB_OP_BAND },   { MPI_BOR, FB_OP_BOR },       { MPI_MAXLOC, FB_OP_MAXLOC },
             { MPI_MINLOC, FB_OP_MINLOC }, { MPI_LXOR, FB_OP_LXOR },   { MPI_BXOR, FB_OP_BXOR } };
}

// The window memory of this rank
struct Window
{
    uint8_t* base = nullptr;
    WindowMemory kind;
    MPI_Win win = nullptr;

    bool create(WindowMemory k)
    {
        kind = k;
        if (k == WindowMemory::Host) {
            void* p = nullptr;
            if (posix_memalign(&p, 64, WINDOW_BYTES) != 0) {
                return false;
            }
            base = (uint8_t*)p;
        } else if (k == WindowMemory::Heap) {
            if (MPI_Alloc_mem(WINDOW_BYTES, MPI_INFO_FAABRIC_DEVICE, &base) != MPI_SUCCESS) {
                return false;
            }
        } else if (cudaMalloc((void**)&base, WINDOW_BYTES) != cudaSuccess) {
            cudaGetLastError();
            return false;
        }
        std::vector<uint8_t> zero(WINDOW_BYTES, 0);
        copyBytes(base, zero.data(), WINDOW_BYTES);
        return MPI_Win_create(base, WINDOW_BYTES, 1, MPI_INFO_NULL, MPI_COMM_WORLD, &win) == MPI_SUCCESS;
    }

    void destroy()
    {
        MPI_Win_free(&win);
        if (kind == WindowMemory::Host) {
            free(base);
        } else if (kind == WindowMemory::Heap) {
            MPI_Free_mem(base);
        } else {
            cudaFree(base);
        }
    }

    std::vector<uint8_t> read(size_t off, size_t n)
    {
        std::vector<uint8_t> out(n);
        copyBytes(out.data(), base + off, n);
        return out;
    }

    void write(size_t off, const void* src, size_t n) { copyBytes(base + off, src, n); }
};

inline int body(int rank, int size, int worldId, const Setup& s, std::string* why)
{
    Window w;
    RMA_CHECK(w.create(s.window));
    auto& world = faabric::mpi::getMpiWorldRegistry().getWorld(worldId);
    auto comm = s.countLaunches ? world.getDeviceComm(rank) : nullptr;
    RMA_CHECK(!s.countLaunches || comm != nullptr);

    // ---- exact results: every rank accumulates into every rank's window
    int cases = 0;
    std::vector<std::unique_ptr<Buffer>> origins, results;
    for (int t = 0; t < size; t++) {
        origins.push_back(std::make_unique<Buffer>(1024, s.deviceBuffers));
        results.push_back(std::make_unique<Buffer>(1024, s.deviceBuffers));
        RMA_CHECK(origins.back()->ok() && results.back()->ok());
    }
    for (MPI_Datatype dt : allDatatypes()) {
        const int fdt = faabric::mpi::fbDtypeFor(dt);
        const size_t esize = fbDtypeSize(fdt);
        RMA_CHECK(esize == (size_t)dt->size);
        for (auto [op, fop] : allOps()) {
            if (!fb::rmaSupported(fdt, fop, false)) {
                continue;
            }
            const bool fetch = cases % 3 == 0; // every third case as MPI_Get_accumulate
            cases++;
            const size_t bytes = EXACT_N * esize;
            std::vector<uint8_t> init(bytes), expect(bytes);
            for (int i = 0; i < EXACT_N; i++) {
                value(fdt, fop, seedOf(cases, -1, rank, i, 1), -1, i, init.data() + i * esize);
            }
            expect = init;
            for (int r = 0; r < size; r++) {
                for (int i = 0; i < EXACT_N; i++) {
                    uint8_t v[16];
                    value(fdt, fop, seedOf(cases, r, rank, i, 2), r, i, v);
                    combine(fdt, fop, expect.data() + i * esize, v);
                }
            }
            w.write(EXACT_OFF, init.data(), bytes);
            MPI_Win_fence(0, w.win);
            for (int t = 0; t < size; t++) {
                for (int i = 0; i < EXACT_N; i++) {
                    value(fdt, fop, seedOf(cases, rank, t, i, 2), rank, i, origins[t]->host.data() + i * esize);
                }
                origins[t]->upload();
            }
            // targets in a different order on every rank
            for (int k = 0; k < size; k++) {
                const int t = (rank + k) % size;
                int rc = fetch ? MPI_Get_accumulate(origins[t]->ptr(), EXACT_N, dt, results[t]->ptr(), EXACT_N, dt, t,
                                                    EXACT_OFF, EXACT_N, dt, op, w.win)
                               : MPI_Accumulate(origins[t]->ptr(), EXACT_N, dt, t, EXACT_OFF, EXACT_N, dt, op, w.win);
                RMA_CHECK(rc == MPI_SUCCESS);
            }
            MPI_Win_fence(0, w.win);
            if (w.read(EXACT_OFF, bytes) != expect) {
                *why = "rank " + std::to_string(rank) + ": wrong result for datatype " + std::to_string(dt->id) +
                       " op " + std::to_string(op->id);
                return 1;
            }
            MPI_Win_fence(0, w.win);
        }
    }
    RMA_CHECK(cases >= 150);

    // a contiguous derived type reduces as its base type
    {
        MPI_Datatype pairOfInts = nullptr;
        MPI_Type_contiguous(2, MPI_INT, &pairOfInts);
        MPI_Type_commit(&pairOfInts);
        std::vector<int32_t> zero(8, 0);
        w.write(EXACT_OFF, zero.data(), sizeof(int32_t) * 8);
        MPI_Win_fence(0, w.win);
        Buffer o(8 * sizeof(int32_t), s.deviceBuffers);
        for (int i = 0; i < 8; i++) {
            int32_t v = i + 1;
            memcpy(o.host.data() + 4 * i, &v, 4);
        }
        o.upload();
        for (int t = 0; t < size; t++) {
            RMA_CHECK(MPI_Accumulate(o.ptr(), 4, pairOfInts, t, EXACT_OFF, 8, MPI_INT, MPI_SUM, w.win) == MPI_SUCCESS);
        }
        MPI_Win_fence(0, w.win);
        auto got = w.read(EXACT_OFF, 8 * sizeof(int32_t));
        for (int i = 0; i < 8; i++) {
            int32_t v;
            memcpy(&v, got.data() + 4 * i, 4);
            RMA_CHECK(v == (i + 1) * size);
        }
        MPI_Type_free(&pairOfInts);
    }

    // ---- tickets: MPI_Fetch_and_op SUM on int64 / int16 / int8 counters of
    // the last rank, next to bytes and shorts the other ranks add to
    {
        const int K = 20; // size * K < 128: the int8 counter does not wrap
        const int owner = size - 1;
        std::vector<uint8_t> zero(256, 0);
        w.write(TICKET_OFF, zero.data(), zero.size());
        MPI_Win_fence(0, w.win);
        Buffer one(16, s.deviceBuffers), tickets(K * 16, s.deviceBuffers);
        int64_t one64 = 1;
        int16_t one16 = 1;
        int8_t one8 = 1;
        memcpy(one.host.data(), &one64, 8);
        memcpy(one.host.data() + 8, &one16, 2);
        memcpy(one.host.data() + 10, &one8, 1);
        one.upload();
        RMA_CHECK(one.ok() && tickets.ok());
        for (int k = 0; k < K; k++) {
            uint8_t* t = tickets.ptr() + 16 * k;
            RMA_CHECK(MPI_Fetch_and_op(one.ptr(), t, MPI_INT64_T, owner, TICKET_OFF, MPI_SUM, w.win) == MPI_SUCCESS);
            RMA_CHECK(MPI_Fetch_and_op(one.ptr() + 8, t + 8, MPI_INT16_T, owner, TICKET_OFF + 10, MPI_SUM, w.win) == MPI_SUCCESS);
            RMA_CHECK(MPI_Fetch_and_op(one.ptr() + 10, t + 12, MPI_INT8_T, owner, TICKET_OFF + 13, MPI_SUM, w.win) == MPI_SUCCESS);
            // neighbours: the bytes around the int8 counter, the short next to the int16 one
            RMA_CHECK(MPI_Accumulate(one.ptr() + 10, 1, MPI_INT8_T, owner, TICKET_OFF + 12, 1, MPI_INT8_T, MPI_SUM, w.win) == MPI_SUCCESS);
            RMA_CHECK(MPI_Accumulate(one.ptr() + 10, 1, MPI_INT8_T, owner, TICKET_OFF + 14, 1, MPI_INT8_T, MPI_SUM, w.win) == MPI_SUCCESS);
            RMA_CHECK(MPI_Accumulate(one.ptr() + 8, 1, MPI_INT16_T, owner, TICKET_OFF + 8, 1, MPI_INT16_T, MPI_SUM, w.win) == MPI_SUCCESS);
        }
        MPI_Win_fence(0, w.win);
        const auto& mine = tickets.read();
        std::vector<int64_t> local(3 * K);
        for (int k = 0; k < K; k++) {
            int64_t t64;
            int16_t t16;
            int8_t t8;
            memcpy(&t64, mine.data() + 16 * k, 8);
            memcpy(&t16, mine.data() + 16 * k + 8, 2);
            memcpy(&t8, mine.data() + 16 * k + 12, 1);
            local[3 * k] = t64;
            local[3 * k + 1] = t16;
            local[3 * k + 2] = t8;
        }
        std::vector<int64_t> all(3 * K * size);
        MPI_Allgather(local.data(), 3 * K, MPI_INT64_T, all.data(), 3 * K, MPI_INT64_T, MPI_COMM_WORLD);
        for (int c = 0; c < 3; c++) {
            std::set<int64_t> seen;
            for (int r = 0; r < size; r++) {
                for (int k = 0; k < K; k++) {
                    seen.insert(all[(size_t)r * 3 * K + 3 * k + c]);
                }
            }
            RMA_CHECK((int)seen.size() == size * K && *seen.begin() == 0 && *seen.rbegin() == size * K - 1);
        }
        if (rank == owner) {
            auto got = w.read(TICKET_OFF, 16);
            int64_t c64;
            int16_t c16, n16;
            memcpy(&c64, got.data(), 8);
            memcpy(&n16, got.data() + 8, 2);
            memcpy(&c16, got.data() + 10, 2);
            RMA_CHECK(c64 == size * K && c16 == size * K && n16 == size * K);
            RMA_CHECK((int8_t)got[12] == size * K && (int8_t)got[13] == size * K && (int8_t)got[14] == size * K);
            RMA_CHECK(got[15] == 0);
        }
        MPI_Win_fence(0, w.win);
    }

    // ---- compare-and-swap: a retry loop counts exactly (a fence per round:
    // fetched values are defined after it)
    {
        const int reps = 4;
        const int owner = 0;
        std::vector<uint8_t> zero(32, 0);
        w.write(CAS_OFF, zero.data(), zero.size());
        MPI_Win_fence(0, w.win);
        Buffer io(32, s.deviceBuffers);
        RMA_CHECK(io.ok());
        int64_t guess64 = 0;
        int16_t guess16 = 0;
        int done64 = 0, done16 = 0, allDone = 0;
        while (allDone < 2 * reps * size) {
            const bool try64 = done64 < reps, try16 = done16 < reps;
            int64_t next64 = guess64 + 1;
            int16_t next16 = (int16_t)(guess16 + 1);
            memcpy(io.host.data(), &next64, 8);
            memcpy(io.host.data() + 8, &guess64, 8);
            memcpy(io.host.data() + 16, &next16, 2);
            memcpy(io.host.data() + 18, &guess16, 2);
            io.upload();
            if (try64) {
                RMA_CHECK(MPI_Compare_and_swap(io.ptr(), io.ptr() + 8, io.ptr() + 24, MPI_INT64_T, owner, CAS_OFF, w.win) == MPI_SUCCESS);
            }
            if (try16) {
                RMA_CHECK(MPI_Compare_and_swap(io.ptr() + 16, io.ptr() + 18, io.ptr() + 20, MPI_INT16_T, owner, CAS_OFF + 10, w.win) == MPI_SUCCESS);
            }
            MPI_Win_fence(0, w.win);
            const auto& got = io.read();
            if (try64) {
                int64_t old;
                memcpy(&old, got.data() + 24, 8);
                done64 += old == guess64 ? 1 : 0;
                guess64 = old == guess64 ? old + 1 : old;
            }
            if (try16) {
                int16_t old;
                memcpy(&old, got.data() + 20, 2);
                done16 += old == guess16 ? 1 : 0;
                guess16 = old == guess16 ? (int16_t)(old + 1) : old;
            }
            int mine = done64 + done16;
            MPI_Allreduce(&mine, &allDone, 1, MPI_INT, MPI_SUM, MPI_COMM_WORLD);
        }
        if (rank == owner) {
            auto got = w.read(CAS_OFF, 16);
            int64_t c64;
            int16_t c16;
            memcpy(&c64, got.data(), 8);
            memcpy(&c16, got.data() + 10, 2);
            RMA_CHECK(c64 == reps * size && c16 == reps * size);
            RMA_CHECK(got[8] == 0 && got[9] == 0 && got[12] == 0);
        }
        MPI_Win_fence(0, w.win);
    }

    // ---- get-accumulate returns the previous values; NO_OP reads them
    {
        const int right = (rank + 1) % size;
        std::vector<int64_t> init(8);
        for (int r = 0; r < size; r++) {
            for (int i = 0; i < 8; i++) {
                init[i] = 1000 * rank + 10 * r + i;
            }
            w.write(GETACC_OFF + 64 * r, init.data(), 64);
        }
        MPI_Win_fence(0, w.win);
        Buffer add(64, s.deviceBuffers), prev(64, s.deviceBuffers), after(64, s.deviceBuffers);
        RMA_CHECK(add.ok() && prev.ok() && after.ok());
        for (int i = 0; i < 8; i++) {
            int64_t v = 7 + i;
            memcpy(add.host.data() + 8 * i, &v, 8);
        }
        add.upload();
        const size_t mine = GETACC_OFF + 64 * rank;
        RMA_CHECK(MPI_Get_accumulate(add.ptr(), 8, MPI_INT64_T, prev.ptr(), 8, MPI_INT64_T, right, mine, 8, MPI_INT64_T, MPI_SUM, w.win) == MPI_SUCCESS);
        MPI_Win_fence(0, w.win);
        RMA_CHECK(MPI_Get_accumulate(nullptr, 0, MPI_INT64_T, after.ptr(), 8, MPI_INT64_T, right, mine, 8, MPI_INT64_T, MPI_NO_OP, w.win) == MPI_SUCCESS);
        MPI_Win_fence(0, w.win);
        const auto& p = prev.read();
        const auto& a = after.read();
        for (int i = 0; i < 8; i++) {
            int64_t pv, av;
            memcpy(&pv, p.data() + 8 * i, 8);
            memcpy(&av, a.data() + 8 * i, 8);
            RMA_CHECK(pv == 1000 * right + 10 * rank + i);
            RMA_CHECK(av == pv + 7 + i);
        }
    }

    // ---- order from one origin: REPLACE then SUM in one epoch, then NO_OP
    {
        const int target = (rank + size - 1) % size;
        MPI_Win_fence(0, w.win);
        Buffer ab(16, s.deviceBuffers), got(16, s.deviceBuffers);
        RMA_CHECK(ab.ok() && got.ok());
        int32_t a = 400 + rank, b = 23;
        memcpy(ab.host.data(), &a, 4);
        memcpy(ab.host.data() + 4, &b, 4);
        ab.upload();
        const size_t slot = ORDER_OFF + 16 * rank;
        const uint64_t before = comm != nullptr ? comm->stats().launches : 0;
        RMA_CHECK(MPI_Accumulate(ab.ptr(), 1, MPI_INT, target, slot, 1, MPI_INT, MPI_REPLACE, w.win) == MPI_SUCCESS);
        RMA_CHECK(MPI_Accumulate(ab.ptr() + 4, 1, MPI_INT, target, slot, 1, MPI_INT, MPI_SUM, w.win) == MPI_SUCCESS);
        if (comm != nullptr) {
            // both calls went through Communicator::accumulate
            RMA_CHECK(comm->stats().launches - before == 2);
        }
        MPI_Win_fence(0, w.win);
        RMA_CHECK(MPI_Fetch_and_op(nullptr, got.ptr(), MPI_INT, target, slot, MPI_NO_OP, w.win) == MPI_SUCCESS);
        MPI_Win_fence(0, w.win);
        int32_t v;
        memcpy(&v, got.read().data(), 4);
        RMA_CHECK(v == a + b);
    }

    // ---- rejections: nothing is applied, the window is unchanged
    {
        MPI_Win_fence(0, w.win);
        const auto snapshot = w.read(0, WINDOW_BYTES);
        MPI_Win_fence(0, w.win);
        const int t = (rank + 1) % size;
        Buffer buf(64, s.deviceBuffers), res(64, s.deviceBuffers);
        RMA_CHECK(buf.ok() && res.ok());
        memset(buf.host.data(), 0x11, 64);
        buf.upload();
        uint8_t* o = buf.ptr();
        uint8_t* r = res.ptr();
        MPI_Op userOp = nullptr;
        MPI_Op_create([](void*, void*, int*, MPI_Datatype*) {}, 1, &userOp);
        // different base types, different sizes
        RMA_CHECK(MPI_Accumulate(o, 2, MPI_INT, t, 0, 2, MPI_FLOAT, MPI_SUM, w.win) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Accumulate(o, 2, MPI_INT, t, 0, 1, MPI_INT64_T, MPI_SUM, w.win) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Accumulate(o, 3, MPI_INT, t, 0, 2, MPI_INT, MPI_SUM, w.win) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Get_accumulate(o, 2, MPI_INT, r, 2, MPI_UINT32_T, t, 0, 2, MPI_INT, MPI_SUM, w.win) == MPI_ERR_ARG);
        // user-defined ops; NO_OP only fetches
        RMA_CHECK(MPI_Accumulate(o, 1, MPI_INT, t, 0, 1, MPI_INT, userOp, w.win) == MPI_ERR_OP);
        RMA_CHECK(MPI_Fetch_and_op(o, r, MPI_INT, t, 0, userOp, w.win) == MPI_ERR_OP);
        RMA_CHECK(MPI_Accumulate(o, 1, MPI_INT, t, 0, 1, MPI_INT, MPI_NO_OP, w.win) == MPI_ERR_OP);
        RMA_CHECK(MPI_Get_accumulate(o, 1, MPI_INT, nullptr, 0, MPI_INT, t, 0, 1, MPI_INT, MPI_NO_OP, w.win) == MPI_ERR_OP);
        // (datatype, op) pairs the atomics do not implement
        RMA_CHECK(MPI_Accumulate(o, 1, MPI_FLOAT, t, 0, 1, MPI_FLOAT, MPI_BAND, w.win) == MPI_ERR_OP);
        RMA_CHECK(MPI_Accumulate(o, 1, MPI_2INT, t, 0, 1, MPI_2INT, MPI_SUM, w.win) == MPI_ERR_OP);
        RMA_CHECK(MPI_Fetch_and_op(o, r, MPI_INT, t, 0, MPI_MAXLOC, w.win) == MPI_ERR_OP);
        RMA_CHECK(MPI_Accumulate(o, 1, MPI_INT, t, 0, 1, MPI_INT, MPI_OP_NULL, w.win) == MPI_ERR_OP);
        // compare-and-swap: integer types only
        RMA_CHECK(MPI_Compare_and_swap(o, o, r, MPI_FLOAT, t, 0, w.win) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Compare_and_swap(o, o, r, MPI_DOUBLE, t, 0, w.win) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Compare_and_swap(o, o, r, MPI_2INT, t, 0, w.win) == MPI_ERR_ARG);
        // misaligned target elements, ranges outside the window, bad ranks
        RMA_CHECK(MPI_Accumulate(o, 1, MPI_INT, t, 2, 1, MPI_INT, MPI_SUM, w.win) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Accumulate(o, 1, MPI_DOUBLE_INT, t, 8, 1, MPI_DOUBLE_INT, MPI_MAXLOC, w.win) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Accumulate(o, 1, MPI_LONG_INT, t, 24, 1, MPI_LONG_INT, MPI_MINLOC, w.win) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Compare_and_swap(o, o, r, MPI_INT64_T, t, 4, w.win) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Fetch_and_op(o, r, MPI_INT16_T, t, 1, MPI_SUM, w.win) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Accumulate(o, 4, MPI_INT, t, WINDOW_BYTES - 8, 4, MPI_INT, MPI_SUM, w.win) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Accumulate(o, 1, MPI_INT, t, -4, 1, MPI_INT, MPI_SUM, w.win) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Compare_and_swap(o, o, r, MPI_INT, t, WINDOW_BYTES, w.win) == MPI_ERR_ARG);
        RMA_CHECK(MPI_Accumulate(o, 1, MPI_INT, size, 0, 1, MPI_INT, MPI_SUM, w.win) == MPI_ERR_RANK);
        RMA_CHECK(MPI_Accumulate(o, 1, MPI_INT, t, 0, 1, MPI_INT, MPI_SUM, nullptr) == MPI_ERR_WIN);
        MPI_Op_free(&userOp);
        MPI_Win_fence(0, w.win);
        RMA_CHECK(w.read(0, WINDOW_BYTES) == snapshot);
    }

    MPI_Win_fence(0, w.win);
    w.destroy();
    return 0;
}

} // namespace rma_atomics
