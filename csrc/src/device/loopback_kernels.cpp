// Loopback device backend: host twins of the sm_90a kernels.
//
// FAABRIC_DEVICE_BACKEND=loopback runs the WHOLE communicator - algorithm
// choice, staging, chunking, channel slicing, grouped segment tables, p2p
// sequence numbers and bounce rings - on plain host memory, with every
// "kernel" executed synchronously on the calling rank thread by the functions
// below.  They implement the SAME flag protocol on the same signal-pad layout
// (monotonic per-CTA barrier epochs, LL {data, flag} slots, p2p ready / ack /
// descriptor words), so the host-side logic that decides what is launched, in
// which order and with which arguments is exercised by the CPU test-suite of a
// GPU-less container (SURVEY 4 / 7.1: "fake multi-GPU on host memory").
//
// One thread per rank is required (as in the MPI runtime, where a rank IS a
// thread): a call returns when the rank's part of the collective is complete.
#include "loopback_kernels.h"

#include <faabric/util/reduce_ops.h>

#include <atomic>
#include <chrono>
#include <cmath>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>

namespace fb::host {

// ---------------------------------------------------------------- flags ----
static inline std::atomic<uint32_t>* aw(uint32_t* p)
{
    return reinterpret_cast<std::atomic<uint32_t>*>(p);
}

static inline void stRelease(uint32_t* p, uint32_t v)
{
    aw(p)->store(v, std::memory_order_release);
}

static inline uint32_t ldAcquire(const uint32_t* p)
{
    return aw(const_cast<uint32_t*>(p))->load(std::memory_order_acquire);
}

static bool waitFlagGe(const FbCommDev& c, const uint32_t* p, uint32_t target, uint32_t errCode)
{
    if ((int32_t)(ldAcquire(p) - target) >= 0) {
        return true;
    }
    auto t0 = std::chrono::steady_clock::now();
    uint32_t spins = 0;
    while (true) {
        if ((int32_t)(ldAcquire(p) - target) >= 0) {
            return true;
        }
        if ((++spins & 0x3f) == 0) {
            std::this_thread::yield();
            auto ns = std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
            if ((uint64_t)ns > c.timeoutNs) {
                if (c.err != nullptr) {
                    stRelease(c.err, errCode);
                }
                return false;
            }
            if (c.err != nullptr && ldAcquire(c.err) != FB_ERR_NONE) {
                return false;
            }
        }
    }
}

// One "CTA" of the cross-rank barrier (same words as BlockBarrier on the GPU)
static bool blockBarrier(const FbCommDev& c, int block)
{
    const size_t slot = (size_t)(c.blockBase + block);
    uint32_t* epochWord = c.sig[c.rank] + FB_SIG_EPOCH_OFF + slot;
    const uint32_t epoch = *epochWord + 1;
    *epochWord = epoch;
    for (int p = 0; p < c.nranks; p++) {
        stRelease(c.sig[p] + slot * FB_MAX_RANKS + c.rank, epoch);
    }
    bool ok = true;
    for (int p = 0; p < c.nranks; p++) {
        ok = waitFlagGe(c, c.sig[c.rank] + slot * FB_MAX_RANKS + p, epoch, FB_ERR_BARRIER_TIMEOUT) && ok;
    }
    return ok;
}

static bool gridBarrier(const FbCommDev& c, int blocks)
{
    bool ok = true;
    for (int b = 0; b < blocks; b++) {
        ok = blockBarrier(c, b) && ok;
    }
    return ok;
}

// ------------------------------------------------------------- reducers ----
namespace {
float halfToFloat(uint16_t h)
{
    uint32_t sign = (uint32_t)(h >> 15) << 31;
    uint32_t exp = (h >> 10) & 0x1f;
    uint32_t man = h & 0x3ff;
    uint32_t bits;
    if (exp == 0) {
        if (man == 0) {
            bits = sign;
        } else {
            int e = -1;
            do {
                e++;
                man <<= 1;
            } while ((man & 0x400) == 0);
            bits = sign | ((uint32_t)(127 - 15 - e) << 23) | ((man & 0x3ff) << 13);
        }
    } else if (exp == 31) {
        bits = sign | 0x7f800000u | (man << 13);
    } else {
        bits = sign | ((exp + 127 - 15) << 23) | (man << 13);
    }
    float f;
    memcpy(&f, &bits, 4);
    return f;
}

uint16_t floatToHalf(float f)
{
    uint32_t x;
    memcpy(&x, &f, 4);
    uint32_t sign = (x >> 16) & 0x8000;
    int32_t exp = (int32_t)((x >> 23) & 0xff) - 127 + 15;
    uint32_t man = x & 0x7fffff;
    if (((x >> 23) & 0xff) == 0xff) {
        return (uint16_t)(sign | 0x7c00 | (man ? 0x200 : 0));
    }
    if (exp >= 31) {
        return (uint16_t)(sign | 0x7c00);
    }
    if (exp <= 0) {
        if (exp < -10) {
            return (uint16_t)sign;
        }
        man |= 0x800000;
        uint32_t shift = (uint32_t)(14 - exp);
        uint32_t r = man >> shift;
        uint32_t rem = man & ((1u << shift) - 1);
        uint32_t half = 1u << (shift - 1);
        if (rem > half || (rem == half && (r & 1))) {
            r++;
        }
        return (uint16_t)(sign | r);
    }
    uint32_t r = ((uint32_t)exp << 10) | (man >> 13);
    uint32_t rem = man & 0x1fff;
    if (rem > 0x1000 || (rem == 0x1000 && (r & 1))) {
        r++;
    }
    return (uint16_t)(sign | r);
}

float bf16ToFloat(uint16_t h)
{
    uint32_t bits = (uint32_t)h << 16;
    float f;
    memcpy(&f, &bits, 4);
    return f;
}

uint16_t floatToBf16(float f)
{
    uint32_t x;
    memcpy(&x, &f, 4);
    if ((x & 0x7fffffff) > 0x7f800000u) {
        return (uint16_t)((x >> 16) | 0x40);
    }
    uint32_t lsb = (x >> 16) & 1;
    x += 0x7fff + lsb;
    return (uint16_t)(x >> 16);
}

// MAX/MIN/SUM/PROD as the kernels define them (faabric/util/reduce_ops.h)
template<typename T>
bool arith(int op, T a, T b, T& out)
{
    switch (op) {
        case FB_OP_MAX:
            out = faabric::util::reduceMax(a, b);
            return true;
        case FB_OP_MIN:
            out = faabric::util::reduceMin(a, b);
            return true;
        case FB_OP_SUM:
            out = faabric::util::reduceSum(a, b);
            return true;
        case FB_OP_PROD:
            out = faabric::util::reduceProd(a, b);
            return true;
        case FB_OP_LAND:
            out = (T)((a != (T)0) && (b != (T)0));
            return true;
        case FB_OP_LOR:
            out = (T)((a != (T)0) || (b != (T)0));
            return true;
        case FB_OP_LXOR:
            out = (T)((a != (T)0) != (b != (T)0));
            return true;
        default:
            return false;
    }
}

template<typename T>
bool intElem(int op, T a, T b, T& out)
{
    switch (op) {
        case FB_OP_BAND:
            out = (T)(a & b);
            return true;
        case FB_OP_BOR:
            out = (T)(a | b);
            return true;
        case FB_OP_BXOR:
            out = (T)(a ^ b);
            return true;
        default:
            return arith<T>(op, a, b, out);
    }
}

template<typename T>
struct PairVI
{
    T v;
    int32_t i;
};

template<typename T>
bool pairElem(int op, PairVI<T> a, PairVI<T> b, PairVI<T>& out)
{
    if (op == FB_OP_MAXLOC) {
        out = (b.v > a.v || (b.v == a.v && b.i < a.i)) ? b : a;
        return true;
    }
    if (op == FB_OP_MINLOC) {
        out = (b.v < a.v || (b.v == a.v && b.i < a.i)) ? b : a;
        return true;
    }
    return false;
}

// acc = acc (op) in, one element, by dtype
bool combineElem(int dtype, int op, uint8_t* acc, const uint8_t* in)
{
#define FB_INT_CASE(code, T)                                                   \
    case code: {                                                               \
        T a, b, r;                                                             \
        memcpy(&a, acc, sizeof(T));                                            \
        memcpy(&b, in, sizeof(T));                                             \
        if (!intElem<T>(op, a, b, r)) {                                        \
            return false;                                                      \
        }                                                                      \
        memcpy(acc, &r, sizeof(T));                                            \
        return true;                                                           \
    }
#define FB_FLT_CASE(code, T)                                                   \
    case code: {                                                               \
        T a, b, r;                                                             \
        memcpy(&a, acc, sizeof(T));                                            \
        memcpy(&b, in, sizeof(T));                                             \
        if (!arith<T>(op, a, b, r)) {                                          \
            return false;                                                      \
        }                                                                      \
        memcpy(acc, &r, sizeof(T));                                            \
        return true;                                                           \
    }
#define FB_PAIR_CASE(code, T)                                                  \
    case code: {                                                               \
        PairVI<T> a, b, r;                                                     \
        memcpy(&a, acc, sizeof(a));                                            \
        memcpy(&b, in, sizeof(b));                                             \
        if (!pairElem<T>(op, a, b, r)) {                                       \
            return false;                                                      \
        }                                                                      \
        memcpy(acc, &r, sizeof(r));                                            \
        return true;                                                           \
    }
    switch (dtype) {
        FB_INT_CASE(FB_I8, int8_t)
        FB_INT_CASE(FB_U8, uint8_t)
        FB_INT_CASE(FB_I16, int16_t)
        FB_INT_CASE(FB_U16, uint16_t)
        FB_INT_CASE(FB_I32, int32_t)
        FB_INT_CASE(FB_U32, uint32_t)
        FB_INT_CASE(FB_I64, int64_t)
        FB_INT_CASE(FB_U64, uint64_t)
        FB_FLT_CASE(FB_F32, float)
        FB_FLT_CASE(FB_F64, double)
        FB_PAIR_CASE(FB_F64_I32, double)
        FB_PAIR_CASE(FB_F32_I32, float)
        FB_PAIR_CASE(FB_I32_I32, int32_t)
        FB_PAIR_CASE(FB_I64_I32, int64_t)
        case FB_F16:
        case FB_BF16: {
            uint16_t a, b;
            memcpy(&a, acc, 2);
            memcpy(&b, in, 2);
            float fa = dtype == FB_F16 ? halfToFloat(a) : bf16ToFloat(a);
            float fb_ = dtype == FB_F16 ? halfToFloat(b) : bf16ToFloat(b);
            float r;
            if (!arith<float>(op, fa, fb_, r)) {
                return false;
            }
            uint16_t out = dtype == FB_F16 ? floatToHalf(r) : floatToBf16(r);
            memcpy(acc, &out, 2);
            return true;
        }
        default:
            return false;
    }
#undef FB_INT_CASE
#undef FB_FLT_CASE
#undef FB_PAIR_CASE
}
}

bool reducible(int dtype, int op)
{
    uint8_t a[16] = { 0 };
    uint8_t b[16] = { 0 };
    return combineElem(dtype, op, a, b);
}

// out[0..bytes) = reduce over ranks [0, readRanks) of heap[p] + off
static void reduceRange(const FbCommDev& c,
                        int dtype,
                        int op,
                        uint64_t off,
                        uint64_t bytes,
                        int readRanks,
                        uint8_t* out)
{
    const size_t es = fbDtypeSize(dtype);
    memcpy(out, c.heap[0] + off, bytes);
    for (int p = 1; p < readRanks; p++) {
        const uint8_t* in = c.heap[p] + off;
        for (uint64_t e = 0; e + es <= bytes; e += es) {
            combineElem(dtype, op, out + e, in + e);
        }
    }
}

// --------------------------------------------------------------- reduce ----
// The CUDA kernel loads and stores its vector body [vecBegin, vecEnd) as
// 16-byte vectors: every address it touches that way must be 16-byte aligned
// and the body must lie in the whole-vector part of the message.  The
// element-wise tail has no such condition.
static bool reduceBodyOk(const ReduceArgs& a)
{
    const FbCommDev& c = a.comm;
    if (a.vecEnd <= a.vecBegin) {
        return true;
    }
    if (a.vecEnd * 16 > a.bytes - (a.bytes & 15)) {
        return false;
    }
    auto aligned = [](const void* p) { return ((uintptr_t)p & 15) == 0; };
    for (int p = 0; p < a.readRanks; p++) {
        if (!aligned(c.heap[p] + a.sendOff)) {
            return false;
        }
    }
    if (a.pushMask == 0) {
        return aligned(a.recvLocal);
    }
    for (int p = 0; p < c.nranks; p++) {
        if ((a.pushMask & (1u << p)) && !aligned(c.heap[p] + a.recvOff)) {
            return false;
        }
    }
    return true;
}

cudaError_t reduceKernel(const ReduceArgs& a, int dtype, int op, int blocks, int, cudaStream_t)
{
    if (!reduceBodyOk(a)) {
        return cudaErrorMisalignedAddress;
    }
    const FbCommDev& c = a.comm;
    bool ok = true;
    if (!a.noSync) {
        ok = gridBarrier(c, blocks);
    }
    if (ok) {
        // vector body [vecBegin, vecEnd) then the < 16-byte tail, as on the GPU
        std::vector<uint8_t> tmp;
        auto run = [&](uint64_t byteBegin, uint64_t nBytes) {
            if (nBytes == 0) {
                return;
            }
            tmp.resize(nBytes);
            reduceRange(c, dtype, op, a.sendOff + byteBegin, nBytes, a.readRanks, tmp.data());
            if (a.pushMask == 0) {
                memcpy(a.recvLocal + (byteBegin - a.outBase * 16), tmp.data(), nBytes);
            } else {
                for (int p = 0; p < c.nranks; p++) {
                    if (a.pushMask & (1u << p)) {
                        memcpy(c.heap[p] + a.recvOff + byteBegin, tmp.data(), nBytes);
                    }
                }
            }
        };
        if (a.vecEnd > a.vecBegin) {
            run(a.vecBegin * 16, (a.vecEnd - a.vecBegin) * 16);
        }
        const uint64_t tailBytes = a.bytes & 15;
        if (tailBytes != 0 && (a.tailOwner == -2 || a.tailOwner == c.rank)) {
            const size_t es = fbDtypeSize(dtype);
            run(a.bytes - tailBytes, tailBytes / es * es);
        }
    }
    if (!a.noSync) {
        gridBarrier(c, blocks);
    }
    return cudaSuccess;
}

// ------------------------------------------------------------------- LL ----
cudaError_t llAllReduce(const LLArgs& a, int dtype, int op, cudaStream_t)
{
    const FbCommDev& c = a.comm;
    const int n = c.nranks;
    const size_t es = fbDtypeSize(dtype);
    const uint64_t nVec = (a.bytes + 15) / 16;
    bool ok = true;
    // every "CTA" advances its epoch word, like the fixed launch geometry does
    uint32_t epochs[FB_LL_BLOCKS];
    for (int b = 0; b < FB_LL_BLOCKS; b++) {
        uint32_t* w = c.sig[c.rank] + FB_SIG_LL_EPOCH_OFF + c.llEpochBase + b;
        uint32_t e = *w + 1;
        if (e == 0) {
            e = 1;
        }
        epochs[b] = e;
    }
    // push my contribution to every rank
    for (uint64_t i = 0; i < nVec; i++) {
        const uint32_t epoch = epochs[i / FB_LL_THREADS];
        const uint32_t par = epoch & 1;
        uint32_t w[4] = { 0, 0, 0, 0 };
        const uint64_t off = i * 16;
        const uint64_t valid = std::min<uint64_t>(16, a.bytes - off);
        memcpy(w, a.sendLocal + off, valid);
        const uint64_t slotOff = a.llOff + (((uint64_t)par * n + c.rank) * FB_LL_MAX_VECS + i) * 32;
        for (int p = 0; p < n; p++) {
            uint32_t* d = reinterpret_cast<uint32_t*>(c.heap[p] + slotOff);
            // data words first, flags last (release): a reader that sees all
            // four flags of this epoch sees the data
            d[0] = w[0];
            d[2] = w[1];
            d[4] = w[2];
            d[6] = w[3];
            stRelease(d + 1, epoch);
            stRelease(d + 3, epoch);
            stRelease(d + 5, epoch);
            stRelease(d + 7, epoch);
        }
    }
    // collect
    for (uint64_t i = 0; i < nVec && ok; i++) {
        const uint32_t epoch = epochs[i / FB_LL_THREADS];
        const uint32_t par = epoch & 1;
        uint8_t acc[16];
        for (int p = 0; p < n && ok; p++) {
            const uint32_t* s = reinterpret_cast<const uint32_t*>(
              c.heap[c.rank] + a.llOff + (((uint64_t)par * n + p) * FB_LL_MAX_VECS + i) * 32);
            for (int f = 1; f < 8 && ok; f += 2) {
                ok = waitFlagGe(c, s + f, epoch, FB_ERR_FLAG_TIMEOUT) && ldAcquire(s + f) == epoch;
            }
            uint32_t v[4] = { s[0], s[2], s[4], s[6] };
            if (p == 0) {
                memcpy(acc, v, 16);
            } else {
                for (size_t e = 0; e + es <= 16; e += es) {
                    combineElem(dtype, op, acc + e, reinterpret_cast<uint8_t*>(v) + e);
                }
            }
        }
        if (ok) {
            const uint64_t off = i * 16;
            memcpy(a.recvLocal + off, acc, std::min<uint64_t>(16, a.bytes - off));
        }
    }
    for (int b = 0; b < FB_LL_BLOCKS; b++) {
        *(c.sig[c.rank] + FB_SIG_LL_EPOCH_OFF + c.llEpochBase + b) = epochs[b];
    }
    return cudaSuccess;
}

// ---------------------------------------------------------------- group ----
cudaError_t groupAllReduce(const GroupArgs& a, int dtype, int op, int blocks, int, cudaStream_t)
{
    const FbCommDev& c = a.comm;
    bool ok = true;
    if (!a.noSync) {
        ok = gridBarrier(c, blocks);
    }
    if (ok) {
        const size_t es = fbDtypeSize(dtype);
        std::vector<uint8_t> tmp;
        for (uint32_t si = 0; si < a.nSegs; si++) {
            const GroupSeg& sg = a.segs[si];
            const uint64_t bytes = (uint64_t)sg.nVec * 16 + sg.tailBytes / es * es;
            if (bytes == 0) {
                continue;
            }
            tmp.resize(bytes);
            reduceRange(c, dtype, op, sg.sendOff, bytes, c.nranks, tmp.data());
            for (int p = 0; p < c.nranks; p++) {
                memcpy(c.heap[p] + sg.recvOff, tmp.data(), bytes);
            }
        }
    }
    if (!a.noSync) {
        gridBarrier(c, blocks);
    }
    return cudaSuccess;
}

// Every segment of the shard kinds is whole 16-byte vectors at 16-byte
// aligned addresses, as the CUDA kernels load and store them
static bool shardSegsOk(const GroupArgs& a)
{
    const FbCommDev& c = a.comm;
    for (uint32_t si = 0; si < a.nSegs; si++) {
        const GroupSeg& sg = a.segs[si];
        if (sg.tailBytes != 0 || ((uintptr_t)(c.heap[c.rank] + sg.sendOff) & 15) ||
            ((uintptr_t)(c.heap[c.rank] + sg.recvOff) & 15)) {
            return false;
        }
    }
    return true;
}

cudaError_t groupReduceScatter(const GroupArgs& a, int dtype, int op, int blocks, int, cudaStream_t)
{
    if (!shardSegsOk(a)) {
        return cudaErrorMisalignedAddress;
    }
    const FbCommDev& c = a.comm;
    bool ok = true;
    if (!a.noSync) {
        ok = gridBarrier(c, blocks);
    }
    if (ok) {
        std::vector<uint8_t> tmp;
        for (uint32_t si = 0; si < a.nSegs; si++) {
            const GroupSeg& sg = a.segs[si];
            const uint64_t bytes = (uint64_t)sg.nVec * 16;
            tmp.resize(bytes);
            reduceRange(c, dtype, op, sg.sendOff, bytes, c.nranks, tmp.data());
            memcpy(c.heap[c.rank] + sg.recvOff, tmp.data(), bytes);
        }
    }
    if (!a.noSync) {
        gridBarrier(c, blocks);
    }
    return cudaSuccess;
}

cudaError_t groupAllGather(const GroupArgs& a, int blocks, int, cudaStream_t)
{
    if (!shardSegsOk(a)) {
        return cudaErrorMisalignedAddress;
    }
    const FbCommDev& c = a.comm;
    bool ok = true;
    if (!a.noSync) {
        ok = gridBarrier(c, blocks);
    }
    if (ok) {
        for (uint32_t si = 0; si < a.nSegs; si++) {
            const GroupSeg& sg = a.segs[si];
            const uint8_t* src = c.heap[c.rank] + sg.sendOff;
            for (int p = 0; p < c.nranks; p++) {
                uint8_t* dst = c.heap[p] + sg.recvOff;
                if (dst != src) { // in place: block `rank` is already there
                    memcpy(dst, src, (uint64_t)sg.nVec * 16);
                }
            }
        }
    }
    if (!a.noSync) {
        gridBarrier(c, blocks);
    }
    return cudaSuccess;
}

cudaError_t groupBroadcast(const GroupArgs& a, int blocks, int, cudaStream_t)
{
    const FbCommDev& c = a.comm;
    // the kernel stores whole vectors at sendOff (== recvOff) on every rank
    for (uint32_t si = 0; si < a.nSegs; si++) {
        const GroupSeg& sg = a.segs[si];
        if (sg.sendOff != sg.recvOff || (sg.nVec != 0 && ((uintptr_t)(c.heap[c.rank] + sg.sendOff) & 15))) {
            return cudaErrorMisalignedAddress;
        }
    }
    bool ok = true;
    if (!a.noSync) {
        ok = gridBarrier(c, blocks);
    }
    if (ok) {
        for (uint32_t si = 0; si < a.nSegs; si++) {
            const GroupSeg& sg = a.segs[si];
            const uint8_t* src = c.heap[a.root] + sg.sendOff;
            for (int p = 0; p < c.nranks; p++) {
                if (p != a.root) {
                    memcpy(c.heap[p] + sg.sendOff, src, (uint64_t)sg.nVec * 16 + sg.tailBytes);
                }
            }
        }
    }
    if (!a.noSync) {
        gridBarrier(c, blocks);
    }
    return cudaSuccess;
}

cudaError_t groupAllToAll(const GroupArgs& a, int blocks, int, cudaStream_t)
{
    if (!shardSegsOk(a)) {
        return cudaErrorMisalignedAddress;
    }
    const FbCommDev& c = a.comm;
    bool ok = true;
    if (!a.noSync) {
        ok = gridBarrier(c, blocks);
    }
    if (ok) {
        for (uint32_t si = 0; si < a.nSegs; si++) {
            const GroupSeg& sg = a.segs[si];
            const uint64_t block = (uint64_t)sg.nVec * 16;
            for (int p = 0; p < c.nranks; p++) {
                memcpy(c.heap[p] + sg.recvOff, c.heap[c.rank] + sg.sendOff + (uint64_t)p * block, block);
            }
        }
    }
    if (!a.noSync) {
        gridBarrier(c, blocks);
    }
    return cudaSuccess;
}

// The twins of groupGatherKernel and groupScatterKernel (RootedSeg tables):
// a piece's staging slice is its chunks, [chunk0 * CB, chunk0 * CB + bytes)
static cudaError_t groupRooted(const GroupArgs& a, int blocks, bool gather)
{
    const FbCommDev& c = a.comm;
    const RootedSeg* segs = reinterpret_cast<const RootedSeg*>(a.segs);
    const uint64_t cb = (uint64_t)fbGroupChunkVecs(c.nranks) * 16;
    const bool isRoot = c.rank == a.root;
    auto slice = [&](int p, const RootedSeg& sg) { return c.heap[p] + a.stageOff + sg.chunk0 * cb; };
    auto user = [](uint64_t addr) { return reinterpret_cast<uint8_t*>(addr); };
    if (gather && !isRoot && (a.phase & GROUP_PHASE_LOCAL)) {
        for (uint32_t si = 0; si < a.nSegs; si++) {
            memcpy(slice(c.rank, segs[si]), user(segs[si].send), segs[si].bytes);
        }
    }
    bool ok = a.noSync || gridBarrier(c, blocks);
    if (ok && isRoot && (a.phase & GROUP_PHASE_MOVE)) {
        for (uint32_t si = 0; si < a.nSegs; si++) {
            const RootedSeg& sg = segs[si];
            // block p of the root's user buffer, and the root's other buffer
            uint8_t* const blocked = user(gather ? sg.recv : sg.send);
            uint8_t* const single = user(gather ? sg.send : sg.recv);
            for (int p = 0; p < c.nranks; p++) {
                uint8_t* const blk = blocked + (uint64_t)p * sg.stride;
                uint8_t* const other = p == a.root ? single : slice(p, sg);
                if (other != blk) { // in place: the root's block stays
                    gather ? memcpy(blk, other, sg.bytes) : memcpy(other, blk, sg.bytes);
                }
            }
        }
    }
    if (!a.noSync) {
        ok = gridBarrier(c, blocks) && ok;
    }
    if (ok && !gather && !isRoot && (a.phase & GROUP_PHASE_LOCAL)) {
        for (uint32_t si = 0; si < a.nSegs; si++) {
            memcpy(user(segs[si].recv), slice(c.rank, segs[si]), segs[si].bytes);
        }
    }
    return cudaSuccess;
}

cudaError_t groupGather(const GroupArgs& a, int blocks, int, cudaStream_t)
{
    return groupRooted(a, blocks, true);
}

cudaError_t groupScatter(const GroupArgs& a, int blocks, int, cudaStream_t)
{
    return groupRooted(a, blocks, false);
}

// The twin of groupNeighborKernel: a piece of staging slot k is its chunks of
// the slot, [(k * T + chunk0) * CB, ... + bytes)
cudaError_t groupNeighbor(const GroupArgs& a, bool allToAll, int blocks, int, cudaStream_t)
{
    const FbCommDev& c = a.comm;
    if ((uintptr_t)(c.heap[c.rank] + a.stageOff) & 15) {
        return cudaErrorMisalignedAddress;
    }
    const RootedSeg* segs = reinterpret_cast<const RootedSeg*>(a.segs);
    const NeighborEdge* edges = reinterpret_cast<const NeighborEdge*>(segs + a.nSegs);
    const uint64_t T = a.totalChunks;
    const bool direct = c.nranks == 1;
    auto slot = [&](int p, uint64_t k, const RootedSeg& sg) {
        return c.heap[p] + a.stageOff + (k * T + sg.chunk0) * FB_NEIGHBOR_CHUNK;
    };
    auto user = [](uint64_t addr) { return reinterpret_cast<uint8_t*>(addr); };
    if (!direct && (a.phase & GROUP_PHASE_LOCAL)) {
        const uint32_t slots = allToAll ? a.outDeg : std::min(a.outDeg, 1u);
        for (uint32_t si = 0; si < a.nSegs; si++) {
            for (uint32_t k = 0; k < slots; k++) {
                memcpy(slot(c.rank, k, segs[si]), user(segs[si].send) + (allToAll ? k * segs[si].stride : 0),
                       segs[si].bytes);
            }
        }
    }
    bool ok = a.noSync || gridBarrier(c, blocks);
    if (ok && (a.phase & GROUP_PHASE_MOVE)) {
        for (uint32_t si = 0; si < a.nSegs; si++) {
            const RootedSeg& sg = segs[si];
            for (uint32_t j = 0; j < a.nEdges; j++) {
                const uint64_t k = allToAll ? edges[j].idx : 0;
                const uint8_t* src = direct ? user(sg.send) + k * sg.stride : slot(edges[j].src, k, sg);
                memcpy(user(sg.recv) + j * sg.stride, src, sg.bytes);
            }
        }
    }
    if (!a.noSync) {
        gridBarrier(c, blocks);
    }
    return cudaSuccess;
}

// The twin of groupNeighborVKernel: the round's bytes [vBase, vBase + vWidth)
// of every stream, between the streams' blocks and the staging slots
cudaError_t groupNeighborV(const GroupArgs& a, bool allToAll, int blocks, int, cudaStream_t)
{
    const FbCommDev& c = a.comm;
    if ((uintptr_t)(c.heap[c.rank] + a.stageOff) & 15) {
        return cudaErrorMisalignedAddress;
    }
    const uint32_t n = a.nSegs;
    const uint32_t sends = allToAll ? a.outDeg : std::min(a.outDeg, 1u);
    const NeighborVSeg* tbl = reinterpret_cast<const NeighborVSeg*>(a.segs);
    const NeighborEdge* edges = reinterpret_cast<const NeighborEdge*>(tbl + (uint64_t)(sends + a.nEdges) * (n + 1));
    const bool direct = c.nranks == 1;
    const uint64_t W = a.vWidth;
    // stream bytes [pos, end) of stream e (n + 1 entries), block by block,
    // to or from the flat range whose byte pos is at flat + pos - vBase
    auto walk = [&](const NeighborVSeg* e, uint64_t pos, uint64_t end, auto&& copy) {
        for (uint32_t m = 0; m < n && pos < end; m++) {
            const uint64_t from = std::max(pos, e[m].off);
            const uint64_t to = std::min(end, e[m + 1].off);
            if (from < to) {
                copy(reinterpret_cast<uint8_t*>(e[m].addr) + (from - e[m].off), from, to - from);
            }
        }
    };
    if (!direct && (a.phase & GROUP_PHASE_LOCAL)) {
        for (uint32_t k = 0; k < sends; k++) {
            const NeighborVSeg* e = tbl + (uint64_t)k * (n + 1);
            uint8_t* const slot = c.heap[c.rank] + a.stageOff + k * W;
            walk(e, a.vBase, std::min(a.vBase + W, e[n].off),
                 [&](uint8_t* user, uint64_t p, uint64_t len) { memcpy(slot + (p - a.vBase), user, len); });
        }
    }
    bool ok = a.noSync || gridBarrier(c, blocks);
    if (ok && (a.phase & GROUP_PHASE_MOVE)) {
        for (uint32_t j = 0; j < a.nEdges; j++) {
            const uint64_t k = allToAll ? edges[j].idx : 0;
            const NeighborVSeg* re = tbl + (uint64_t)(sends + j) * (n + 1);
            const NeighborVSeg* se = tbl + k * (n + 1);
            const uint64_t end = std::min(a.vBase + W, direct ? std::min(re[n].off, se[n].off) : re[n].off);
            walk(re, a.vBase, end, [&](uint8_t* user, uint64_t p, uint64_t len) {
                if (!direct) {
                    memcpy(user, c.heap[edges[j].src] + a.stageOff + k * W + (p - a.vBase), len);
                    return;
                }
                walk(se, p, p + len,
                     [&](uint8_t* from, uint64_t q, uint64_t l2) { memcpy(user + (q - p), from, l2); });
            });
        }
    }
    if (!a.noSync) {
        gridBarrier(c, blocks);
    }
    return cudaSuccess;
}

// The twin of groupReduceKernel: every rank stages its pieces; after the
// entry barrier this rank folds the chunks it owns (the kernel's rule, with
// the same grid) into the root's result slices; after the exit barrier the
// root unstages
cudaError_t groupReduce(const GroupArgs& a, int dtype, int op, int blocks, int threads, cudaStream_t)
{
    const FbCommDev& c = a.comm;
    const RootedSeg* segs = reinterpret_cast<const RootedSeg*>(a.segs);
    const int n = c.nranks;
    const uint64_t cb = (uint64_t)fbGroupChunkVecs(n) * 16;
    const size_t es = fbDtypeSize(dtype);
    auto user = [](uint64_t addr) { return reinterpret_cast<uint8_t*>(addr); };
    if (a.phase & GROUP_PHASE_LOCAL) {
        for (uint32_t si = 0; si < a.nSegs; si++) {
            const RootedSeg& sg = segs[si];
            if (n == 1) {
                if (sg.recv != sg.send) {
                    memcpy(user(sg.recv), user(sg.send), sg.bytes);
                }
            } else {
                memcpy(c.heap[c.rank] + a.stageOff + sg.chunk0 * cb, user(sg.send), sg.bytes);
            }
        }
    }
    if (n == 1) {
        return cudaSuccess;
    }
    bool ok = a.noSync || gridBarrier(c, blocks);
    if (ok && (a.phase & GROUP_PHASE_MOVE)) {
        const uint64_t warpStride = (uint64_t)blocks * (uint64_t)(threads / 32);
        for (uint32_t si = 0; si < a.nSegs; si++) {
            const RootedSeg& sg = segs[si];
            for (uint64_t off = 0; off < sg.bytes; off += cb) {
                const uint64_t ch = sg.chunk0 + off / cb;
                if ((int)((ch % warpStride + ch / warpStride) % (uint64_t)n) != c.rank) {
                    continue;
                }
                const uint64_t len = std::min<uint64_t>(cb, sg.bytes - off);
                const uint64_t slice = ch * cb;
                uint8_t* const out = c.heap[a.root] + a.stageRecvOff + slice;
                memcpy(out, c.heap[0] + a.stageOff + slice, len);
                for (int p = 1; p < n; p++) {
                    const uint8_t* in = c.heap[p] + a.stageOff + slice;
                    for (uint64_t e = 0; e + es <= len; e += es) {
                        combineElem(dtype, op, out + e, in + e);
                    }
                }
            }
        }
    }
    if (!a.noSync) {
        ok = gridBarrier(c, blocks) && ok;
    }
    if (ok && c.rank == a.root && (a.phase & GROUP_PHASE_UNSTAGE)) {
        for (uint32_t si = 0; si < a.nSegs; si++) {
            const RootedSeg& sg = segs[si];
            memcpy(user(sg.recv), c.heap[c.rank] + a.stageRecvOff + sg.chunk0 * cb, sg.bytes);
        }
    }
    return cudaSuccess;
}

// The twin of groupScanKernel (a.exclusive: exscan): every rank stages its
// pieces (an exscan's last rank does not); after the entry barrier this rank
// folds the chunks it owns in rank order and stores the value after rank p
// into rank p + exclusive's result slices; after the exit barrier every rank
// unstages (an exscan's rank 0 does not)
cudaError_t groupScan(const GroupArgs& a, int dtype, int op, int blocks, int threads, cudaStream_t)
{
    const FbCommDev& c = a.comm;
    const RootedSeg* segs = reinterpret_cast<const RootedSeg*>(a.segs);
    const int n = c.nranks;
    const int ex = a.exclusive;
    const uint64_t cb = (uint64_t)fbGroupChunkVecs(n) * 16;
    const size_t es = fbDtypeSize(dtype);
    auto user = [](uint64_t addr) { return reinterpret_cast<uint8_t*>(addr); };
    if ((a.phase & GROUP_PHASE_LOCAL) && !(ex && c.rank == n - 1)) {
        for (uint32_t si = 0; si < a.nSegs; si++) {
            const RootedSeg& sg = segs[si];
            if (n == 1) {
                if (sg.recv != sg.send) {
                    memcpy(user(sg.recv), user(sg.send), sg.bytes);
                }
            } else {
                memcpy(c.heap[c.rank] + a.stageOff + sg.chunk0 * cb, user(sg.send), sg.bytes);
            }
        }
    }
    if (n == 1) {
        return cudaSuccess;
    }
    bool ok = a.noSync || gridBarrier(c, blocks);
    if (ok && (a.phase & GROUP_PHASE_MOVE)) {
        const uint64_t warpStride = (uint64_t)blocks * (uint64_t)(threads / 32);
        std::vector<uint8_t> acc(cb);
        for (uint32_t si = 0; si < a.nSegs; si++) {
            const RootedSeg& sg = segs[si];
            for (uint64_t off = 0; off < sg.bytes; off += cb) {
                const uint64_t ch = sg.chunk0 + off / cb;
                if ((int)((ch % warpStride + ch / warpStride) % (uint64_t)n) != c.rank) {
                    continue;
                }
                const uint64_t len = std::min<uint64_t>(cb, sg.bytes - off);
                const uint64_t slice = ch * cb;
                memcpy(acc.data(), c.heap[0] + a.stageOff + slice, len);
                for (int p = 0; p + ex < n; p++) {
                    if (p > 0) {
                        const uint8_t* in = c.heap[p] + a.stageOff + slice;
                        for (uint64_t e = 0; e + es <= len; e += es) {
                            combineElem(dtype, op, acc.data() + e, in + e);
                        }
                    }
                    memcpy(c.heap[p + ex] + a.stageRecvOff + slice, acc.data(), len);
                }
            }
        }
    }
    if (!a.noSync) {
        ok = gridBarrier(c, blocks) && ok;
    }
    if (ok && !(ex && c.rank == 0) && (a.phase & GROUP_PHASE_UNSTAGE)) {
        for (uint32_t si = 0; si < a.nSegs; si++) {
            const RootedSeg& sg = segs[si];
            memcpy(user(sg.recv), c.heap[c.rank] + a.stageRecvOff + sg.chunk0 * cb, sg.bytes);
        }
    }
    return cudaSuccess;
}

// ----------------------------------------------------------------- move ----
// The CUDA kernels copy in W-byte words.  Every address they touch that way
// must be W-aligned (a misaligned vector access is a device fault), and every
// length they copy that way a whole number of words (the kernels drop a
// remainder).  The twins check the width they are given against the same
// addresses before they copy, so a host decision that would fault on the GPU
// fails here, with the error the CUDA launch would report.
namespace {
struct MoveCopy
{
    uint8_t* dst;
    const uint8_t* src;
    uint64_t bytes;
};

bool wordsOk(const void* p, int w)
{
    return ((uintptr_t)p % (uintptr_t)w) == 0;
}

bool copiesOk(const std::vector<MoveCopy>& cs, int w)
{
    for (const MoveCopy& m : cs) {
        if (!wordsOk(m.dst, w) || !wordsOk(m.src, w) || m.bytes % (uint64_t)w != 0) {
            return false;
        }
    }
    return true;
}

void runCopies(const std::vector<MoveCopy>& cs)
{
    for (const MoveCopy& m : cs) {
        memcpy(m.dst, m.src, m.bytes);
    }
}

// The copies this rank makes in a one-step pull (moveKernel and moveBulkKernel)
std::vector<MoveCopy> pullCopies(const MoveArgs& a)
{
    const FbCommDev& c = a.comm;
    const int rank = c.rank;
    std::vector<MoveCopy> cs;
    if (a.mode == MOVE_ALLGATHER || a.mode == MOVE_ALLTOALL || (a.mode == MOVE_GATHER && rank == a.root)) {
        const uint64_t srcExtra = (a.mode == MOVE_ALLTOALL) ? (uint64_t)rank * a.srcStride : 0;
        for (int p = 0; p < c.nranks; p++) {
            cs.push_back({ a.recvLocal + (uint64_t)p * a.dstStride, c.heap[p] + a.sendOff + srcExtra, a.chunkBytes });
        }
    } else if (a.mode == MOVE_SCATTER) {
        cs.push_back({ a.recvLocal, c.heap[a.root] + a.sendOff + (uint64_t)rank * a.srcStride, a.chunkBytes });
    } else if (a.mode == MOVE_BCAST && rank != a.root) {
        cs.push_back({ a.recvLocal, c.heap[a.root] + a.sendOff, a.chunkBytes });
    }
    return cs;
}

// The copies of step 1 (this rank's slice from the root) or step 2 (every
// other slice from its owner) of the two-step broadcast
std::vector<MoveCopy> bcast2StepCopies(const MoveArgs& a, int step)
{
    const FbCommDev& c = a.comm;
    const int rank = c.rank;
    const int n = c.nranks;
    const uint64_t total = a.chunkBytes;
    const uint64_t slice = ((total / n) + 15) & ~(uint64_t)15;
    auto bounds = [&](int p, uint64_t& b, uint64_t& e) {
        b = std::min<uint64_t>((uint64_t)p * slice, total);
        e = (p == n - 1) ? total : std::min<uint64_t>(b + slice, total);
    };
    std::vector<MoveCopy> cs;
    if (rank == a.root) {
        return cs;
    }
    uint64_t b, e;
    if (step == 1) {
        bounds(rank, b, e);
        if (e > b) {
            cs.push_back({ c.heap[rank] + a.recvOff + b, c.heap[a.root] + a.sendOff + b, e - b });
        }
        return cs;
    }
    for (int q = 1; q < n; q++) {
        int p = (rank + q) % n;
        bounds(p, b, e);
        if (e <= b) {
            continue;
        }
        const uint8_t* src = (p == a.root) ? c.heap[p] + a.sendOff + b : c.heap[p] + a.recvOff + b;
        cs.push_back({ c.heap[rank] + a.recvOff + b, src, e - b });
    }
    return cs;
}

// barrier, copies, barrier: the protocol of both one-step pull kernels
cudaError_t runPull(const MoveArgs& a, const std::vector<MoveCopy>& cs, int blocks)
{
    bool ok = true;
    if (!a.noSync) {
        ok = gridBarrier(a.comm, blocks);
    }
    if (ok) {
        runCopies(cs);
    }
    if (!a.noSync) {
        gridBarrier(a.comm, blocks);
    }
    return cudaSuccess;
}
}

cudaError_t moveKernel(const MoveArgs& a, int width, int blocks, int, cudaStream_t)
{
    if (a.mode != MOVE_BCAST_2STEP) {
        const std::vector<MoveCopy> cs = pullCopies(a);
        if (!copiesOk(cs, width)) {
            return cudaErrorMisalignedAddress;
        }
        return runPull(a, cs, blocks);
    }
    const std::vector<MoveCopy> step1 = bcast2StepCopies(a, 1);
    const std::vector<MoveCopy> step2 = bcast2StepCopies(a, 2);
    if (!copiesOk(step1, width) || !copiesOk(step2, width)) {
        return cudaErrorMisalignedAddress;
    }
    const FbCommDev& c = a.comm;
    bool ok = true;
    if (!a.noSync) {
        ok = gridBarrier(c, blocks);
    }
    if (ok) {
        runCopies(step1);
        ok = a.noSync ? true : gridBarrier(c, blocks);
        if (ok) {
            runCopies(step2);
        }
    }
    if (!a.noSync) {
        gridBarrier(c, blocks);
    }
    return cudaSuccess;
}

cudaError_t moveBulk(const MoveArgs& a, int blocks, cudaStream_t)
{
    // cp.async.bulk moves 16-byte aligned ranges of whole 16-byte units
    if (!moveBulkSupported(a)) {
        return cudaErrorMisalignedAddress;
    }
    const std::vector<MoveCopy> cs = pullCopies(a);
    if (!copiesOk(cs, 16)) {
        return cudaErrorMisalignedAddress;
    }
    return runPull(a, cs, blocks);
}

cudaError_t barrierKernel(const FbCommDev& c, cudaStream_t)
{
    return blockBarrier(c, 0) ? cudaSuccess : cudaErrorUnknown;
}

// ------------------------------------------------------------------ p2p ----
// The p2p and put kernels copy bytes - bytes % W in W-byte words, then the
// tail byte by byte: with no whole word they touch nothing as a word
static bool p2pWordsOk(const void* dst, const void* src, uint64_t bytes, int w)
{
    return bytes < (uint64_t)w || (wordsOk(dst, w) && wordsOk(src, w));
}

cudaError_t p2pSend(const P2PArgs& a, int width, int, cudaStream_t)
{
    const FbCommDev& c = a.comm;
    if (a.stage && !p2pWordsOk(c.heap[c.rank] + a.srcOff, a.local, a.bytes, width)) {
        return cudaErrorMisalignedAddress;
    }
    if (a.stage && a.bytes > 0) {
        memcpy(c.heap[c.rank] + a.srcOff, a.local, a.bytes);
    }
    uint32_t* desc =
      reinterpret_cast<uint32_t*>(c.heap[a.peer] + a.descOff) + ((uint32_t)c.rank * FB_P2P_RING + (a.seq % FB_P2P_RING)) * 4;
    desc[0] = (uint32_t)(a.srcOff & 0xffffffffu);
    desc[1] = (uint32_t)(a.srcOff >> 32);
    desc[2] = (uint32_t)(a.bytes & 0xffffffffu);
    desc[3] = (uint32_t)(a.bytes >> 32);
    stRelease(c.sig[a.peer] + FB_P2P_READY_OFF + c.rank, a.seq);
    return cudaSuccess;
}

cudaError_t p2pPull(const P2PArgs& a, int width, int, cudaStream_t)
{
    const FbCommDev& c = a.comm;
    const uint32_t seen = ldAcquire(c.sig[c.rank] + FB_P2P_READY_OFF + a.peer);
    const uint32_t* desc = reinterpret_cast<const uint32_t*>(c.heap[c.rank] + a.descOff) +
                           ((uint32_t)a.peer * FB_P2P_RING + (a.seq % FB_P2P_RING)) * 4;
    const uint64_t srcOff = (uint64_t)desc[0] | ((uint64_t)desc[1] << 32);
    uint64_t len = (uint64_t)desc[2] | ((uint64_t)desc[3] << 32);
    if (!((int32_t)(seen - a.seq) >= 0 && len <= a.bytes && srcOff + len <= a.heapBytes)) {
        if (c.err != nullptr) {
            stRelease(c.err, FB_ERR_BAD_DESC);
        }
        len = 0;
    }
    if (!p2pWordsOk(a.local, c.heap[a.peer] + srcOff, len, width)) {
        return cudaErrorMisalignedAddress;
    }
    if (len > 0) {
        memcpy(a.local, c.heap[a.peer] + srcOff, len);
    }
    stRelease(c.sig[a.peer] + FB_P2P_ACK_OFF + c.rank, a.seq);
    return cudaSuccess;
}

cudaError_t putSignal(const PutArgs& a, int width, int blocks, cudaStream_t)
{
    const FbCommDev& c = a.comm;
    if (!p2pWordsOk(c.heap[a.peer] + a.dstOff, a.local, a.bytes, width)) {
        return cudaErrorMisalignedAddress;
    }
    if (a.bytes > 0) {
        memcpy(c.heap[a.peer] + a.dstOff, a.local, a.bytes);
    }
    // one increment per "CTA", like the kernel
    aw(c.sig[a.peer] + FB_SIG_USER_OFF + a.signalIdx)->fetch_add((uint32_t)blocks, std::memory_order_release);
    return cudaSuccess;
}

cudaError_t waitSignal(const FbCommDev& c, int signalIdx, uint32_t addTarget, cudaStream_t)
{
    uint32_t* sigp = c.sig[c.rank] + FB_SIG_USER_OFF + signalIdx;
    uint32_t* consumed = sigp + FB_SIG_USER_WORDS;
    const uint32_t target = *consumed + addTarget;
    bool ok = waitFlagGe(c, sigp, target, FB_ERR_FLAG_TIMEOUT);
    *consumed = target;
    return ok ? cudaSuccess : cudaErrorUnknown;
}

cudaError_t signalPeers(const FbCommDev& c, uint32_t wordOff, uint32_t value, cudaStream_t)
{
    for (int p = 0; p < c.nranks; p++) {
        if (p != c.rank) {
            stRelease(c.sig[p] + wordOff + c.rank, value);
        }
    }
    return cudaSuccess;
}

cudaError_t waitWord(const FbCommDev& c, const uint32_t* word, uint32_t target, cudaStream_t)
{
    return waitFlagGe(c, word, target, FB_ERR_FLAG_TIMEOUT) ? cudaSuccess : cudaErrorUnknown;
}

// ------------------------------------------------------------------ rma ----
// The host twins of rma_kernels.cu, also the implementation of one-sided
// atomics on host windows.  Every element is one atomic step with respect to
// the other threads of the process: a CAS loop on the enclosing 32-bit word
// (1, 2 and 4-byte elements) or on the 64-bit element, and a striped lock for
// 16-byte elements.  The target is naturally aligned (the callers check).
namespace {

// bytes of an element that an update replaces: a 16-byte pair keeps its padding
size_t rmaKeepBytes(int dtype)
{
    return (dtype == FB_F64_I32 || dtype == FB_I64_I32) ? 12 : fbDtypeSize(dtype);
}

// out = the new value of an element whose current bytes are `cur`
void rmaCombine(int dtype, int op, const uint8_t* cur, const uint8_t* in, uint8_t* out)
{
    const size_t n = fbDtypeSize(dtype);
    memcpy(out, cur, n);
    if (op == FB_OP_NO_OP) {
        return;
    }
    uint8_t tmp[16];
    memcpy(tmp, cur, n);
    if (op == FB_OP_REPLACE) {
        memcpy(tmp, in, n);
    } else {
        combineElem(dtype, op, tmp, in);
    }
    memcpy(out, tmp, rmaKeepBytes(dtype));
}

std::mutex& rmaStripe(const void* p)
{
    static std::mutex stripes[64];
    return stripes[((uintptr_t)p >> 4) % 64];
}

// Atomically replaces the n-byte element at p by f(current); `prev` (may be
// null) receives the value it replaced
template<typename W, typename F>
void rmaCasWord(uint8_t* p, size_t n, uint8_t* prev, F f)
{
    const uintptr_t addr = (uintptr_t)p;
    W* wp = reinterpret_cast<W*>(addr & ~(uintptr_t)(sizeof(W) - 1));
    const size_t shift = addr & (sizeof(W) - 1); // little endian
    std::atomic_ref<W> ref(*wp);
    W old = ref.load();
    while (true) {
        uint8_t cur[8];
        uint8_t nv[8];
        memcpy(cur, (const uint8_t*)&old + shift, n);
        f(cur, nv);
        W nw = old;
        memcpy((uint8_t*)&nw + shift, nv, n);
        if (nw == old || ref.compare_exchange_weak(old, nw)) {
            if (prev != nullptr) {
                memcpy(prev, cur, n);
            }
            return;
        }
    }
}

template<typename F>
void rmaAtomic(uint8_t* p, size_t n, uint8_t* prev, F f)
{
    if (n == 16) {
        std::lock_guard<std::mutex> lk(rmaStripe(p));
        uint8_t nv[16];
        f(p, nv);
        if (prev != nullptr) {
            memcpy(prev, p, 16);
        }
        memcpy(p, nv, 16);
    } else if (n == 8) {
        rmaCasWord<uint64_t>(p, n, prev, f);
    } else {
        rmaCasWord<uint32_t>(p, n, prev, f);
    }
}

} // namespace

cudaError_t rmaAccumulate(const RmaArgs& a, int dtype, int op, cudaStream_t)
{
    const size_t n = fbDtypeSize(dtype);
    uint8_t* tgt = a.target;
    for (uint64_t i = 0; i < a.count; i++) {
        const uint8_t* in = op == FB_OP_NO_OP ? nullptr : a.origin + i * n;
        rmaAtomic(tgt + i * n, n, a.result != nullptr ? a.result + i * n : nullptr, [&](const uint8_t* cur, uint8_t* nv) {
            rmaCombine(dtype, op, cur, in, nv);
        });
    }
    return cudaSuccess;
}

cudaError_t rmaCompareSwap(const RmaCasArgs& a, int dtype, cudaStream_t)
{
    const size_t n = fbDtypeSize(dtype);
    rmaAtomic(a.target, n, a.result, [&](const uint8_t* cur, uint8_t* nv) {
        memcpy(nv, memcmp(cur, a.compare, n) == 0 ? a.swap : cur, n);
    });
    return cudaSuccess;
}

cudaError_t rmaCopyMany(const RmaCopyArgs& a, cudaStream_t)
{
    for (uint32_t i = 0; i < a.nItems; i++) {
        memmove(a.items[i].dst, a.items[i].src, a.items[i].bytes);
    }
    return cudaSuccess;
}

cudaError_t rmaAccumulateMany(const RmaAccManyArgs& a, int dtype, int op, cudaStream_t s)
{
    for (uint32_t i = 0; i < a.nItems; i++) {
        const RmaAccDesc& it = a.items[i];
        rmaAccumulate(RmaArgs{ it.target, it.origin, it.fetch, it.count }, dtype, op, s);
    }
    return cudaSuccess;
}

// ----------------------------------------------------------------- copy ----
cudaError_t copy(void* dst, const void* src, size_t bytes, cudaStream_t)
{
    memmove(dst, src, bytes);
    return cudaSuccess;
}

cudaError_t copy2D(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t height, cudaStream_t)
{
    for (size_t row = 0; row < height; row++) {
        memcpy((uint8_t*)dst + row * dpitch, (const uint8_t*)src + row * spitch, width);
    }
    return cudaSuccess;
}

} // namespace fb::host
