// One-sided communication for MpiWorld (MPI_Win_*, MPI_Put / MPI_Get and the
// MPI_Accumulate family).
#include <faabric/device/communicator.h>
#include <faabric/device/cuda_driver.h>
#include <faabric/mpi/MpiWorld.h>
#include <faabric/util/logging.h>
#include <faabric/util/macros.h>

#include "device/loopback_kernels.h"
#include "launch_api.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <stdexcept>

namespace faabric::mpi {

// ---------------------------------------------------------------------------
// One-sided communication
// ---------------------------------------------------------------------------
namespace {
struct RmaSegment
{
    uint64_t base;
    int64_t size;
    int32_t dispUnit;
    int32_t pad;
};

struct RmaWireOp
{
    int32_t kind;
    int32_t dtype; // atomics: FbDtype and FbOp
    uint64_t dispBytes;
    uint64_t bytes;
    int32_t op;
    int32_t pad;
};

// Where a buffer lives: a CUDA device, HOST_MEMORY (also the loopback
// backend's heaps) or ANY_DEVICE (managed memory)
constexpr int HOST_MEMORY = -1;
constexpr int ANY_DEVICE = -2;

int bufferDevice(const void* p)
{
    if (p == nullptr || faabric::device::Communicator::isLoopbackHeapPointer(p) || !faabric::device::cudaAvailable()) {
        return HOST_MEMORY;
    }
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) {
        cudaGetLastError();
        return HOST_MEMORY;
    }
    if (attr.type == cudaMemoryTypeDevice) {
        return attr.device;
    }
    return attr.type == cudaMemoryTypeManaged ? ANY_DEVICE : HOST_MEMORY;
}

bool reachable(const void* p, int device)
{
    const int where = bufferDevice(p);
    return p == nullptr || where == device || where == ANY_DEVICE;
}

void cudaCheck(cudaError_t e, const char* what)
{
    if (e != cudaSuccess) {
        cudaGetLastError();
        throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
    }
}

// Restores the calling thread's current device
struct DeviceGuard
{
    int saved = -1;
    explicit DeviceGuard(int device)
    {
        if (device >= 0) {
            cudaGetDevice(&saved);
            cudaSetDevice(device);
        }
    }
    ~DeviceGuard()
    {
        if (saved >= 0) {
            cudaSetDevice(saved);
        }
    }
};

// Origin, compare and result buffers the memory at `device` (or the host)
// can read and write.  Buffers that already qualify are used in place; the
// others are copied in before the operation and the fetched values copied
// out by finish(), which waits for the stream.  `stream` is a stream on
// `device`, or null for the host.
struct RmaStage
{
    int device;
    cudaStream_t stream;
    size_t bytes;
    size_t esize;
    uint8_t* result;
    const uint8_t* in[2];
    uint8_t* out = nullptr;
    std::vector<uint8_t> host;
    uint8_t* dev = nullptr;
    bool staged = false;

    RmaStage(int deviceIn, cudaStream_t s, size_t nbytes, size_t elemSize, const uint8_t* origin, const uint8_t* compare, uint8_t* resultIn)
      : device(deviceIn)
      , stream(s)
      , bytes(nbytes)
      , esize(elemSize)
      , result(resultIn)
      , in{ origin, compare }
      , out(resultIn)
    {
        const size_t parts[3] = { origin != nullptr ? bytes : 0, compare != nullptr ? esize : 0, result != nullptr ? bytes : 0 };
        staged = !reachable(origin, device) || !reachable(compare, device) || !reachable(result, device);
        if (!staged) {
            return;
        }
        const size_t total = parts[0] + parts[1] + parts[2];
        uint8_t* buf = nullptr;
        if (device == HOST_MEMORY) {
            host.resize(total);
            buf = host.data();
        } else {
            cudaCheck(cudaMallocAsync((void**)&dev, std::max<size_t>(total, 1), stream), "Staging a one-sided operation");
            buf = dev;
        }
        for (int i = 0; i < 2; i++) {
            if (in[i] != nullptr) {
                copyIn(buf, in[i], parts[i]);
                in[i] = buf;
                buf += parts[i];
            }
        }
        out = result != nullptr ? buf : nullptr;
    }

    void copyIn(uint8_t* dst, const uint8_t* src, size_t n)
    {
        if (device == HOST_MEMORY) {
            cudaCheck(cudaMemcpy(dst, src, n, cudaMemcpyDefault), "Staging a one-sided operation");
        } else {
            cudaCheck(cudaMemcpyAsync(dst, src, n, cudaMemcpyDefault, stream), "Staging a one-sided operation");
        }
    }

    // True if the operation completed here (staged operations always do)
    bool finish()
    {
        if (!staged) {
            return false;
        }
        if (device == HOST_MEMORY) {
            if (result != nullptr) {
                cudaCheck(cudaMemcpy(result, out, bytes, cudaMemcpyDefault), "Returning fetched values");
            }
            return true;
        }
        if (result != nullptr) {
            cudaCheck(cudaMemcpyAsync(result, out, bytes, cudaMemcpyDefault, stream), "Returning fetched values");
        }
        cudaCheck(cudaFreeAsync(dev, stream), "Staging a one-sided operation");
        cudaCheck(cudaStreamSynchronize(stream), "One-sided operation");
        return true;
    }
};

void rmaCopy(void* dst, const void* src, size_t bytes)
{
    if (bytes == 0) {
        return;
    }
    if (MpiWorld::isDevicePointer(dst) || MpiWorld::isDevicePointer(src)) {
        if (cudaMemcpy(dst, src, bytes, cudaMemcpyDefault) != cudaSuccess) {
            cudaGetLastError();
            throw std::runtime_error("Device copy for a one-sided operation failed");
        }
    } else {
        memcpy(dst, src, bytes);
    }
}
}

bool MpiWorld::allRanksLocal()
{
    for (int r = 0; r < size; r++) {
        if (!isLocalRank(r)) {
            return false;
        }
    }
    return true;
}

std::shared_ptr<MpiWorld::RmaWindow> MpiWorld::getWindow(int winId)
{
    std::lock_guard<std::mutex> lk(windowsMx);
    auto it = windows.find(winId);
    if (it == windows.end()) {
        SPDLOG_ERROR("MPI window {} does not exist in world {}", winId, id);
        throw std::runtime_error("Unknown MPI window");
    }
    return it->second;
}

int MpiWorld::winCreate(int rank, void* base, int64_t sizeBytes, int dispUnit)
{
    checkRanksRange(0, rank);
    if (sizeBytes < 0 || dispUnit <= 0) {
        throw std::invalid_argument("Bad size / displacement unit for an MPI window");
    }
    int winId = 0;
    std::shared_ptr<RmaWindow> w;
    {
        std::lock_guard<std::mutex> lk(windowsMx);
        if ((int)windowsCreated.size() < size) {
            windowsCreated.resize(size, 0);
        }
        winId = ++windowsCreated[rank];
        auto& slot = windows[winId];
        if (slot == nullptr) {
            slot = std::make_shared<RmaWindow>();
            slot->pending.resize(size);
            slot->streams.resize(size);
        }
        w = slot;
    }
    // Everybody learns everybody's segment
    RmaSegment mine{ (uint64_t)(uintptr_t)base, sizeBytes, dispUnit, 0 };
    std::vector<RmaSegment> all(size);
    faabric_datatype_t* byteType = getFaabricDatatypeFromId(FAABRIC_BYTE);
    allGather(rank, BYTES(&mine), byteType, sizeof(RmaSegment), BYTES(all.data()), byteType, sizeof(RmaSegment));
    {
        std::lock_guard<std::mutex> lk(w->mx);
        if (!w->filled) {
            w->bases.resize(size);
            w->sizes.resize(size);
            w->dispUnits.resize(size);
            for (int r = 0; r < size; r++) {
                w->bases[r] = all[r].base;
                w->sizes[r] = all[r].size;
                w->dispUnits[r] = all[r].dispUnit;
            }
            w->filled = true;
        }
    }
    // Nobody may target a segment before its owner has published it
    barrier(rank);
    return winId;
}

void MpiWorld::winFree(int rank, int winId)
{
    auto w = getWindow(winId);
    // Outstanding operations complete first
    winFence(rank, winId);
    int localRanks = 0;
    for (int r = 0; r < size; r++) {
        localRanks += isLocalRank(r) ? 1 : 0;
    }
    bool last = false;
    {
        std::lock_guard<std::mutex> lk(w->mx);
        last = ++w->freed == localRanks;
    }
    if (last) {
        std::lock_guard<std::mutex> lk(windowsMx);
        windows.erase(winId);
    }
}

bool MpiWorld::winQuery(int winId, int rank, void** base, int64_t* sizeBytes, int* dispUnit)
{
    std::shared_ptr<RmaWindow> w;
    {
        std::lock_guard<std::mutex> lk(windowsMx);
        auto it = windows.find(winId);
        if (it == windows.end()) {
            return false;
        }
        w = it->second;
    }
    if (rank < 0 || rank >= size || !w->filled) {
        return false;
    }
    *base = (void*)(uintptr_t)w->bases[rank];
    *sizeBytes = w->sizes[rank];
    *dispUnit = w->dispUnits[rank];
    return true;
}

uint8_t* MpiWorld::winTargetPtr(RmaWindow& w, int targetRank, int64_t targetDisp, size_t bytes)
{
    if (targetRank < 0 || targetRank >= size) {
        throw std::runtime_error("One-sided operation on a rank outside the world");
    }
    const int64_t off = targetDisp * (int64_t)w.dispUnits[targetRank];
    if (targetDisp < 0 || off + (int64_t)bytes > w.sizes[targetRank]) {
        SPDLOG_ERROR("One-sided access [{}, {}) outside the {}-byte window of rank {}", off, off + (int64_t)bytes, w.sizes[targetRank], targetRank);
        throw std::runtime_error("One-sided operation outside the target window");
    }
    return (uint8_t*)(uintptr_t)w.bases[targetRank] + off;
}

void MpiWorld::winPut(int rank, int winId, const uint8_t* origin, size_t bytes, int targetRank, int64_t targetDisp)
{
    auto w = getWindow(winId);
    uint8_t* dst = winTargetPtr(*w, targetRank, targetDisp, bytes);
    if (isLocalRank(targetRank)) {
        // Same address space (or peer-mapped HBM): write it now, the closing
        // fence publishes it
        rmaCopy(dst, origin, bytes);
        return;
    }
    uint64_t dispBytes = (uint64_t)(dst - (uint8_t*)(uintptr_t)w->bases[targetRank]);
    w->pending[rank].push_back(RmaOp{ RMA_PUT, targetRank, dispBytes, bytes, const_cast<uint8_t*>(origin) });
}

void MpiWorld::winGet(int rank, int winId, uint8_t* origin, size_t bytes, int targetRank, int64_t targetDisp)
{
    auto w = getWindow(winId);
    uint8_t* src = winTargetPtr(*w, targetRank, targetDisp, bytes);
    if (isLocalRank(targetRank)) {
        rmaCopy(origin, src, bytes);
        return;
    }
    uint64_t dispBytes = (uint64_t)(src - (uint8_t*)(uintptr_t)w->bases[targetRank]);
    w->pending[rank].push_back(RmaOp{ RMA_GET, targetRank, dispBytes, bytes, origin });
}

std::shared_ptr<faabric::device::Communicator> MpiWorld::wiredDeviceComm(int rank)
{
    std::lock_guard<std::mutex> lk(deviceMx);
    if (rank < 0 || rank >= (int)deviceComms.size()) {
        return nullptr;
    }
    return deviceComms[rank];
}

void* MpiWorld::rmaStream(int rank, int device)
{
    // (one stream per rank and device, whatever else is wired: the calls of
    // one origin on one segment stay in issue order)
    std::lock_guard<std::mutex> lk(deviceMx);
    void*& s = rmaStreams[{ rank, device }];
    if (s == nullptr) {
        DeviceGuard on(device);
        cudaCheck(cudaStreamCreateWithFlags((cudaStream_t*)&s, cudaStreamNonBlocking), "Creating a stream for one-sided operations");
    }
    return s;
}

void MpiWorld::rmaApplyLocal(RmaWindow& w,
                             int rank,
                             int targetRank,
                             uint8_t* target,
                             size_t count,
                             int dtype,
                             int op,
                             const uint8_t* origin,
                             const uint8_t* compare,
                             uint8_t* result)
{
    const size_t esize = fbDtypeSize(dtype);
    const size_t bytes = count * esize;
    if (count == 0) {
        return;
    }
    auto streamUsed = [&](int device, void* s) {
        auto& used = w.streams[rank];
        if (std::find(used.begin(), used.end(), std::make_pair(device, s)) == used.end()) {
            used.emplace_back(device, s);
        }
    };
    // Symmetric heap: the origin rank's communicator, through its peer mapping
    auto comm = wiredDeviceComm(rank);
    auto targetComm = wiredDeviceComm(targetRank);
    if (comm != nullptr && targetComm != nullptr && targetComm->inHeap(target, bytes)) {
        const int device = comm->isLoopback() ? HOST_MEMORY : comm->device();
        cudaStream_t s = (cudaStream_t)streamForRank(rank);
        DeviceGuard on(device);
        RmaStage st(device, s, bytes, esize, origin, compare, result);
        const uint64_t off = targetComm->offsetOf(target);
        int rc = compare != nullptr ? comm->compareAndSwap(st.in[1], st.in[0], st.out, off, dtype, targetRank, s)
                                    : comm->accumulate(st.in[0], off, count, dtype, op, targetRank, st.out, s);
        if (rc != FB_OK) {
            throw std::runtime_error(std::string("Device one-sided operation failed: ") +
                                     faabric::device::Communicator::errorString(rc));
        }
        if (!st.finish() && device != HOST_MEMORY) {
            streamUsed(device, s);
        }
        return;
    }
    const int where = bufferDevice(target);
    if (where == HOST_MEMORY) {
        // Host memory: the host atomics, on this thread
        RmaStage st(HOST_MEMORY, nullptr, bytes, esize, origin, compare, result);
        if (compare != nullptr) {
            fb::RmaCasArgs a{ target, st.in[1], st.in[0], st.out };
            fb::host::rmaCompareSwap(a, dtype, nullptr);
        } else {
            fb::RmaArgs a{ target, st.in[0], st.out, count };
            fb::host::rmaAccumulate(a, dtype, op, nullptr);
        }
        st.finish();
        return;
    }
    // Other device memory: the pointer kernel, on the origin's GPU if it can
    // address the segment, otherwise on the segment's own GPU
    int device = where;
    if (where == ANY_DEVICE) {
        cudaCheck(cudaGetDevice(&device), "One-sided operation");
    }
    if (comm != nullptr && !comm->isLoopback() && comm->device() != device) {
        int canAccess = 0;
        cudaDeviceCanAccessPeer(&canAccess, comm->device(), device);
        if (canAccess != 0) {
            DeviceGuard on(comm->device());
            cudaError_t e = cudaDeviceEnablePeerAccess(device, 0);
            if (e == cudaSuccess || e == cudaErrorPeerAccessAlreadyEnabled) {
                device = comm->device();
            }
            cudaGetLastError();
        }
    }
    cudaStream_t s = (cudaStream_t)rmaStream(rank, device);
    DeviceGuard on(device);
    RmaStage st(device, s, bytes, esize, origin, compare, result);
    cudaError_t e;
    if (compare != nullptr) {
        fb::RmaCasArgs a{ target, st.in[1], st.in[0], st.out };
        e = fb::launchRmaCompareSwap(a, dtype, s);
    } else {
        fb::RmaArgs a{ target, st.in[0], st.out, count };
        e = fb::launchRmaAccumulate(a, dtype, op, s);
    }
    cudaCheck(e, "One-sided atomic kernel launch");
    if (!st.finish()) {
        streamUsed(device, s);
    }
}

namespace {
// Checks the target of an atomic and returns its address (in the target's
// address space), or an MPI error code
int rmaAtomicTarget(const std::vector<uint64_t>& bases,
                    const std::vector<int64_t>& sizes,
                    const std::vector<int32_t>& dispUnits,
                    int targetRank,
                    int64_t targetDisp,
                    size_t bytes,
                    size_t esize,
                    uint8_t** target)
{
    if (targetRank < 0 || targetRank >= (int)bases.size()) {
        return MPI_ERR_RANK;
    }
    const int64_t off = targetDisp * (int64_t)dispUnits[targetRank];
    if (targetDisp < 0 || bytes > (uint64_t)sizes[targetRank] || off > sizes[targetRank] - (int64_t)bytes) {
        SPDLOG_ERROR("One-sided atomic on [{}, {}) outside the {}-byte window of rank {}", off, off + (int64_t)bytes, sizes[targetRank], targetRank);
        return MPI_ERR_ARG;
    }
    *target = (uint8_t*)(uintptr_t)bases[targetRank] + off;
    if ((uintptr_t)*target % esize != 0) {
        SPDLOG_ERROR("One-sided atomic on a target element not aligned to its {} bytes", esize);
        return MPI_ERR_ARG;
    }
    return MPI_SUCCESS;
}
}

int MpiWorld::winAccumulate(int rank,
                            int winId,
                            const uint8_t* origin,
                            size_t count,
                            faabric_datatype_t* datatype,
                            faabric_op_t* op,
                            uint8_t* result,
                            int targetRank,
                            int64_t targetDisp)
{
    const int dtype = datatype != nullptr ? fbDtypeFor(datatype) : -1;
    const int fop = op != nullptr ? fbOpFor(op) : -1;
    if (dtype < 0) {
        return MPI_ERR_ARG;
    }
    if (fop < 0 || !fb::rmaSupported(dtype, fop, result != nullptr)) {
        return MPI_ERR_OP;
    }
    const size_t esize = fbDtypeSize(dtype);
    if (count > (size_t)INT64_MAX / esize || (origin == nullptr && fop != FB_OP_NO_OP && count > 0)) {
        return MPI_ERR_ARG;
    }
    auto w = getWindow(winId);
    uint8_t* target = nullptr;
    const size_t bytes = count * esize;
    int rc = rmaAtomicTarget(w->bases, w->sizes, w->dispUnits, targetRank, targetDisp, bytes, esize, &target);
    if (rc != MPI_SUCCESS || count == 0) {
        return rc;
    }
    if (isLocalRank(targetRank)) {
        rmaApplyLocal(*w, rank, targetRank, target, count, dtype, fop, origin, nullptr, result);
        return MPI_SUCCESS;
    }
    if (bytes > (uint64_t)INT32_MAX) {
        return MPI_ERR_ARG;
    }
    RmaOp q{ result != nullptr ? RMA_GET_ACCUMULATE : RMA_ACCUMULATE,
             targetRank,
             (uint64_t)(target - (uint8_t*)(uintptr_t)w->bases[targetRank]),
             bytes,
             nullptr };
    q.dtype = dtype;
    q.op = fop;
    q.result = result;
    if (fop != FB_OP_NO_OP) {
        q.data.resize(bytes);
        rmaCopy(q.data.data(), origin, bytes);
    }
    w->pending[rank].push_back(std::move(q));
    return MPI_SUCCESS;
}

int MpiWorld::winCompareSwap(int rank,
                             int winId,
                             const uint8_t* origin,
                             const uint8_t* compare,
                             uint8_t* result,
                             faabric_datatype_t* datatype,
                             int targetRank,
                             int64_t targetDisp)
{
    const int dtype = datatype != nullptr ? fbDtypeFor(datatype) : -1;
    if (dtype < 0 || !fb::rmaCasSupported(dtype) || origin == nullptr || compare == nullptr || result == nullptr) {
        return MPI_ERR_ARG;
    }
    const size_t esize = fbDtypeSize(dtype);
    auto w = getWindow(winId);
    uint8_t* target = nullptr;
    int rc = rmaAtomicTarget(w->bases, w->sizes, w->dispUnits, targetRank, targetDisp, esize, esize, &target);
    if (rc != MPI_SUCCESS) {
        return rc;
    }
    if (isLocalRank(targetRank)) {
        rmaApplyLocal(*w, rank, targetRank, target, 1, dtype, -1, origin, compare, result);
        return MPI_SUCCESS;
    }
    RmaOp q{ RMA_COMPARE_SWAP, targetRank, (uint64_t)(target - (uint8_t*)(uintptr_t)w->bases[targetRank]), esize, nullptr };
    q.dtype = dtype;
    q.data.resize(2 * esize);
    rmaCopy(q.data.data(), origin, esize);
    rmaCopy(q.data.data() + esize, compare, esize);
    q.result = result;
    w->pending[rank].push_back(std::move(q));
    return MPI_SUCCESS;
}

void MpiWorld::rmaSendOps(RmaWindow& w, int rank, int peer)
{
    faabric_datatype_t* byteType = getFaabricDatatypeFromId(FAABRIC_BYTE);
    std::vector<const RmaOp*> replies;
    for (const RmaOp& op : w.pending[rank]) {
        if (op.target != peer) {
            continue;
        }
        if (op.bytes > (uint64_t)INT32_MAX) {
            throw std::runtime_error("One-sided operation larger than 2 GiB to another process");
        }
        RmaWireOp wire{ op.kind, op.dtype, op.dispBytes, op.bytes, op.op, 0 };
        send(rank, peer, BYTES(&wire), byteType, sizeof(wire), MpiMessageType::RMA_OP);
        if (op.kind == RMA_PUT) {
            send(rank, peer, op.origin, byteType, (int)op.bytes, MpiMessageType::RMA_DATA);
        } else if (op.kind != RMA_GET && !op.data.empty()) {
            send(rank, peer, op.data.data(), byteType, (int)op.data.size(), MpiMessageType::RMA_DATA);
        }
        if (op.kind == RMA_GET || op.kind == RMA_GET_ACCUMULATE || op.kind == RMA_COMPARE_SWAP) {
            replies.push_back(&op);
        }
    }
    // The target answers each get / fetch as it meets it: same order
    std::vector<uint8_t> fetched;
    for (const RmaOp* op : replies) {
        if (op->kind == RMA_GET) {
            recv(peer, rank, op->origin, byteType, (int)op->bytes, nullptr, MpiMessageType::RMA_DATA);
        } else {
            fetched.resize(op->bytes);
            recv(peer, rank, fetched.data(), byteType, (int)op->bytes, nullptr, MpiMessageType::RMA_DATA);
            rmaCopy(op->result, fetched.data(), op->bytes);
        }
    }
}

void MpiWorld::rmaRecvOps(RmaWindow& w, int rank, int peer, int nOps)
{
    faabric_datatype_t* byteType = getFaabricDatatypeFromId(FAABRIC_BYTE);
    uint8_t* base = (uint8_t*)(uintptr_t)w.bases[rank];
    std::vector<uint8_t> data, fetched;
    for (int i = 0; i < nOps; i++) {
        RmaWireOp wire{};
        recv(peer, rank, BYTES(&wire), byteType, sizeof(wire), nullptr, MpiMessageType::RMA_OP);
        if ((int64_t)(wire.dispBytes + wire.bytes) > w.sizes[rank]) {
            throw std::runtime_error("Remote one-sided operation outside this rank's window");
        }
        if (wire.kind == RMA_PUT) {
            recv(peer, rank, base + wire.dispBytes, byteType, (int)wire.bytes, nullptr, MpiMessageType::RMA_DATA);
            continue;
        }
        if (wire.kind == RMA_GET) {
            send(rank, peer, base + wire.dispBytes, byteType, (int)wire.bytes, MpiMessageType::RMA_DATA);
            continue;
        }
        // Atomics, applied in arrival order through this segment's path
        const bool cas = wire.kind == RMA_COMPARE_SWAP;
        const size_t esize = fbDtypeSize(wire.dtype);
        if (esize == 0 || wire.bytes % esize != 0 || (uintptr_t)(base + wire.dispBytes) % esize != 0 ||
            (cas ? wire.bytes != esize || !fb::rmaCasSupported(wire.dtype)
                 : !fb::rmaSupported(wire.dtype, wire.op, wire.kind == RMA_GET_ACCUMULATE))) {
            throw std::runtime_error("Malformed remote one-sided atomic");
        }
        const size_t dataBytes = cas ? 2 * esize : (wire.op == FB_OP_NO_OP ? 0 : wire.bytes);
        data.resize(dataBytes);
        if (dataBytes > 0) {
            recv(peer, rank, data.data(), byteType, (int)dataBytes, nullptr, MpiMessageType::RMA_DATA);
        }
        const bool fetch = wire.kind != RMA_ACCUMULATE;
        fetched.resize(fetch ? wire.bytes : 0);
        rmaApplyLocal(w,
                      rank,
                      rank,
                      base + wire.dispBytes,
                      wire.bytes / esize,
                      wire.dtype,
                      wire.op,
                      dataBytes > 0 ? data.data() : nullptr,
                      cas ? data.data() + esize : nullptr,
                      fetch ? fetched.data() : nullptr);
        if (fetch) {
            send(rank, peer, fetched.data(), byteType, (int)wire.bytes, MpiMessageType::RMA_DATA);
        }
    }
}

void MpiWorld::winFence(int rank, int winId)
{
    auto w = getWindow(winId);
    // Atomics this rank launched on device streams complete first
    {
        auto comm = wiredDeviceComm(rank);
        for (auto [device, s] : w->streams[rank]) {
            DeviceGuard on(device);
            if (comm != nullptr && !comm->isLoopback() && comm->device() == device) {
                if (!comm->waitStreamFast((cudaStream_t)s)) {
                    throw std::runtime_error("One-sided operation failed on the device");
                }
            } else {
                cudaCheck(cudaStreamSynchronize((cudaStream_t)s), "One-sided operation");
            }
        }
        w->streams[rank].clear();
    }
    if (!allRanksLocal()) {
        // How many operations does everybody have for everybody else?
        std::vector<int> outgoing(size, 0), incoming(size, 0);
        for (const RmaOp& op : w->pending[rank]) {
            outgoing[op.target]++;
        }
        faabric_datatype_t* intType = getFaabricDatatypeFromId(FAABRIC_INT);
        allToAll(rank, BYTES(outgoing.data()), intType, 1, BYTES(incoming.data()), intType, 1);
        // Pairwise exchanges in increasing peer order; inside a pair the lower
        // rank ships first.  Every wait is on a strictly "earlier" pair, so the
        // schedule cannot cycle.
        for (int peer = 0; peer < size; peer++) {
            if (peer == rank || isLocalRank(peer)) {
                continue;
            }
            if (rank < peer) {
                rmaSendOps(*w, rank, peer);
                rmaRecvOps(*w, rank, peer, incoming[peer]);
            } else {
                rmaRecvOps(*w, rank, peer, incoming[peer]);
                rmaSendOps(*w, rank, peer);
            }
        }
        w->pending[rank].clear();
    }
    barrier(rank);
}

}
