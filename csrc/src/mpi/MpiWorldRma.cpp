// One-sided communication for MpiWorld (MPI_Win_*, MPI_Put / MPI_Get and the
// MPI_Accumulate family).
#include <faabric/device/communicator.h>
#include <faabric/device/cuda_driver.h>
#include <faabric/mpi/MpiWorld.h>
#include <faabric/mpi/MpiWorldRegistry.h>
#include <faabric/transport/PointToPointCall.h>
#include <faabric/transport/PointToPointClient.h>
#include <faabric/util/config.h>
#include <faabric/util/logging.h>
#include <faabric/util/macros.h>

#include "buffers.h"
#include "device/loopback_kernels.h"
#include "launch_api.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstring>
#include <set>
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
        auto reachable = [&](const void* p) {
            const int where = bufferDevice(p);
            return p == nullptr || where == device || where == ANY_DEVICE;
        };
        staged = !reachable(origin) || !reachable(compare) || !reachable(result);
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

// Every request of `p` to a target that `covered` names is complete
template<class F>
void markComplete(const std::shared_ptr<MpiWorld::RmaProgress>& p, F covered)
{
    if (p == nullptr) {
        return;
    }
    for (size_t t = 0; t < p->issued.size(); t++) {
        if (covered((int)t)) {
            p->completed[t] = p->issued[t];
        }
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
            slot->epochs.resize(size);
            slot->locks.resize(size);
            slot->batches.resize(size);
            slot->progress.resize(size);
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

std::shared_ptr<MpiWorld::RmaWindow> MpiWorld::findWindow(int winId)
{
    std::lock_guard<std::mutex> lk(windowsMx);
    auto it = windows.find(winId);
    return it == windows.end() || !it->second->filled ? nullptr : it->second;
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
        // fence (or flush) publishes it
        copyBytes(dst, origin, bytes);
        if (!w->epochs[rank].locked.empty()) {
            w->epochs[rank].deviceCopies |= !hostAddressable(dst) || !hostAddressable(origin);
        }
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
        copyBytes(origin, src, bytes);
        if (!w->epochs[rank].locked.empty()) {
            w->epochs[rank].deviceCopies |= !hostAddressable(origin) || !hostAddressable(src);
        }
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
    // one origin on one segment stay in issue order.  Rank -1: the streams of
    // the passive-target server path)
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
                             uint8_t* result,
                             std::vector<std::pair<int, void*>>& used,
                             bool serverPath)
{
    const size_t esize = fbDtypeSize(dtype);
    const size_t bytes = count * esize;
    if (count == 0) {
        return;
    }
    auto streamUsed = [&](int device, void* s) {
        if (std::find(used.begin(), used.end(), std::make_pair(device, s)) == used.end()) {
            used.emplace_back(device, s);
        }
    };
    // Symmetric heap: the origin rank's communicator, through its peer mapping
    auto comm = wiredDeviceComm(rank);
    auto targetComm = wiredDeviceComm(targetRank);
    if (comm != nullptr && targetComm != nullptr && targetComm->inHeap(target, bytes)) {
        const int device = comm->isLoopback() ? HOST_MEMORY : comm->device();
        cudaStream_t s = !serverPath               ? (cudaStream_t)streamForRank(rank)
                         : device == HOST_MEMORY ? nullptr
                                                 : (cudaStream_t)rmaStream(-1, device);
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
    cudaStream_t s = (cudaStream_t)rmaStream(serverPath ? -1 : rank, device);
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
        rmaApplyLocal(*w, rank, targetRank, target, count, dtype, fop, origin, nullptr, result, w->streams[rank]);
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
        copyBytes(q.data.data(), origin, bytes);
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
        rmaApplyLocal(*w, rank, targetRank, target, 1, dtype, -1, origin, compare, result, w->streams[rank]);
        return MPI_SUCCESS;
    }
    RmaOp q{ RMA_COMPARE_SWAP, targetRank, (uint64_t)(target - (uint8_t*)(uintptr_t)w->bases[targetRank]), esize, nullptr };
    q.dtype = dtype;
    q.data.resize(2 * esize);
    copyBytes(q.data.data(), origin, esize);
    copyBytes(q.data.data() + esize, compare, esize);
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
            copyBytes(op->result, fetched.data(), op->bytes);
        }
    }
}

size_t MpiWorld::rmaAtomicPayload(int kind, int dtype, int op, uint64_t bytes, const uint8_t* target)
{
    const bool cas = kind == RMA_COMPARE_SWAP;
    const size_t esize = fbDtypeSize(dtype);
    if ((kind != RMA_ACCUMULATE && kind != RMA_GET_ACCUMULATE && !cas) || esize == 0 || bytes % esize != 0 ||
        (uintptr_t)target % esize != 0 ||
        (cas ? bytes != esize || !fb::rmaCasSupported(dtype) : !fb::rmaSupported(dtype, op, kind == RMA_GET_ACCUMULATE))) {
        throw std::runtime_error("Malformed remote one-sided atomic");
    }
    return cas ? 2 * esize : (op == FB_OP_NO_OP ? 0 : bytes);
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
        const size_t dataBytes = rmaAtomicPayload(wire.kind, wire.dtype, wire.op, wire.bytes, base + wire.dispBytes);
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
                      fetch ? fetched.data() : nullptr,
                      w.streams[rank]);
        if (fetch) {
            send(rank, peer, fetched.data(), byteType, (int)wire.bytes, MpiMessageType::RMA_DATA);
        }
    }
}

void MpiWorld::rmaWaitStreams(RmaWindow& w, int rank)
{
    auto comm = wiredDeviceComm(rank);
    for (auto [device, s] : w.streams[rank]) {
        DeviceGuard on(device);
        if (comm != nullptr && !comm->isLoopback() && comm->device() == device) {
            if (!comm->waitStreamFast((cudaStream_t)s)) {
                throw std::runtime_error("One-sided operation failed on the device");
            }
        } else {
            cudaCheck(cudaStreamSynchronize((cudaStream_t)s), "One-sided operation");
        }
    }
    w.streams[rank].clear();
}

void MpiWorld::winFence(int rank, int winId)
{
    auto w = getWindow(winId);
    // Atomics this rank launched on device streams complete first
    rmaWaitStreams(*w, rank);
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

// ---------------------------------------------------------------------------
// Passive-target synchronisation (MPI_Win_lock, MPI_Win_flush, ...)
// ---------------------------------------------------------------------------
namespace {
// A request to the process of a target rank: this header, then (flush and
// unlock) nOps times an RmaWireOp followed by its payload
struct RmaPassiveHeader
{
    int32_t worldId;
    int32_t winId;
    int32_t origin;
    int32_t target;
    int32_t exclusive;
    int32_t nOps;
    uint64_t ticket;
};

// First word of every reply.  A flush / unlock reply goes on with the bytes
// of its gets and fetches, in request order.
enum RmaReply : int32_t
{
    RMA_REPLY_OK = 0,
    // lock: queued, the grant follows as RMA_LOCK_GRANT
    RMA_REPLY_QUEUED = 1,
    // the world or the window is unknown to the target's process (or freed)
    RMA_REPLY_NO_WINDOW = 2,
    RMA_REPLY_FAILED = 3,
};

std::string replyOf(int32_t status)
{
    return std::string((const char*)&status, sizeof(status));
}

// Grants of locks that origins of this process queued for elsewhere
struct GrantTable
{
    std::mutex mx;
    std::condition_variable cv;
    std::set<uint64_t> granted;
};

GrantTable& grantTable()
{
    static GrantTable t;
    return t;
}

std::atomic<uint64_t> nextTicket{ 1 };

std::chrono::milliseconds lockTimeout()
{
    return std::chrono::milliseconds(faabric::util::getSystemConfig().globalMessageTimeout);
}

// ---- reader/writer lock of a target segment (caller holds lockMx) ----
template<class Lock>
bool lockFits(const Lock& l, bool exclusive)
{
    return exclusive ? l.exclusive == 0 && l.shared == 0 : l.exclusive == 0;
}

// Grants waiters in arrival order while they fit (a shared waiter behind an
// exclusive one waits too: no starvation); returns the grant messages to send
template<class Lock>
std::vector<std::function<void()>> grantWaiters(Lock& l)
{
    std::vector<std::function<void()>> sends;
    while (!l.waiters.empty() && lockFits(l, l.waiters.front().exclusive)) {
        auto& q = l.waiters.front();
        (q.exclusive ? l.exclusive : l.shared)++;
        *q.granted = true;
        if (q.onGrant) {
            sends.push_back(std::move(q.onGrant));
        }
        l.waiters.pop_front();
    }
    return sends;
}

template<class Lock>
std::vector<std::function<void()>> releaseLock(Lock& l, bool exclusive)
{
    int& held = exclusive ? l.exclusive : l.shared;
    if (held == 0) {
        throw std::runtime_error("Releasing a one-sided lock that is not held");
    }
    held--;
    return grantWaiters(l);
}

// Drops a waiter that gave up; false if it was granted already
template<class Lock>
bool dropWaiter(Lock& l, uint64_t ticket)
{
    auto it = std::find_if(l.waiters.begin(), l.waiters.end(), [&](const auto& q) { return q.ticket == ticket; });
    if (it == l.waiters.end()) {
        return false;
    }
    l.waiters.erase(it);
    return true;
}

// Wakes the origins of this process and sends the other grants (outside
// lockMx: a send must not hold up the lock)
template<class Window>
void announceGrants(Window& w, const std::vector<std::function<void()>>& sends)
{
    w.lockCv.notify_all();
    for (const auto& send : sends) {
        try {
            send();
        } catch (const std::exception& e) {
            SPDLOG_ERROR("Could not send a one-sided lock grant: {}", e.what());
        }
    }
}

// One request to the process of a target; the reply's status, the rest of
// the reply in `rest`
int32_t rmaCall(const std::string& host, faabric::transport::PointToPointCall call, const std::vector<uint8_t>& request, std::vector<uint8_t>* rest)
{
    std::vector<uint8_t> reply;
    try {
        reply = faabric::transport::getPointToPointClient(host)->rmaRequest(call, request);
    } catch (const std::exception& e) {
        SPDLOG_ERROR("One-sided request to {} failed: {}", host, e.what());
        return RMA_REPLY_FAILED;
    }
    int32_t status = RMA_REPLY_FAILED;
    if (reply.size() >= sizeof(status)) {
        memcpy(&status, reply.data(), sizeof(status));
        if (rest != nullptr) {
            rest->assign(reply.begin() + sizeof(status), reply.end());
        }
    }
    return status;
}

int mpiErrorOf(int32_t status)
{
    return status == RMA_REPLY_OK ? MPI_SUCCESS : status == RMA_REPLY_NO_WINDOW ? MPI_ERR_WIN : MPI_ERR_OTHER;
}

template<class V>
void append(std::vector<uint8_t>& out, const V& v)
{
    out.insert(out.end(), (const uint8_t*)&v, (const uint8_t*)&v + sizeof(v));
}
}

int MpiWorld::rmaAcquire(RmaWindow& w, int winId, int rank, int targetRank, bool exclusive)
{
    const uint64_t ticket = nextTicket++;
    if (isLocalRank(targetRank)) {
        auto granted = std::make_shared<bool>(false);
        std::unique_lock<std::mutex> lk(w.lockMx);
        RmaLock& l = w.locks[targetRank];
        l.waiters.push_back(RmaLockWaiter{ ticket, exclusive, granted, nullptr });
        grantWaiters(l);
        if (w.lockCv.wait_for(lk, lockTimeout(), [&] { return *granted; })) {
            return MPI_SUCCESS;
        }
        dropWaiter(l, ticket);
        auto sends = grantWaiters(l);
        lk.unlock();
        announceGrants(w, sends);
        SPDLOG_ERROR("Rank {} timed out waiting for the lock of rank {} on window {}", rank, targetRank, winId);
        return MPI_ERR_OTHER;
    }
    // The lock lives in the target's process: granted there at once, or
    // queued and granted by a later message
    const std::string host = getHostForRank(targetRank);
    std::vector<uint8_t> req;
    append(req, RmaPassiveHeader{ id, winId, rank, targetRank, exclusive ? 1 : 0, 0, ticket });
    const int32_t status = rmaCall(host, faabric::transport::PointToPointCall::RMA_LOCK, req, nullptr);
    if (status != RMA_REPLY_QUEUED) {
        return mpiErrorOf(status);
    }
    GrantTable& g = grantTable();
    std::unique_lock<std::mutex> lk(g.mx);
    const bool granted = g.cv.wait_for(lk, lockTimeout(), [&] { return g.granted.count(ticket) > 0; });
    g.granted.erase(ticket);
    lk.unlock();
    if (granted) {
        return MPI_SUCCESS;
    }
    // (the target drops the request, or releases the lock if it was granted
    // meanwhile)
    rmaCall(host, faabric::transport::PointToPointCall::RMA_LOCK_CANCEL, req, nullptr);
    SPDLOG_ERROR("Rank {} timed out waiting for the lock of rank {} on window {}", rank, targetRank, winId);
    return MPI_ERR_OTHER;
}

int MpiWorld::rmaComplete(RmaWindow& w, int winId, int rank, int targetRank, bool release)
{
    RmaEpoch& e = w.epochs[rank];
    const RmaEpoch::Target t = e.locked.at(targetRank);
    const bool unlock = release && !t.nocheck;
    if (isLocalRank(targetRank)) {
        // Everything of this origin in this process completes: its device
        // streams, and copies from pageable memory still in flight
        rmaIssueBatch(w, rank);
        rmaWaitStreams(w, rank);
        if (e.deviceCopies) {
            cudaCheck(cudaStreamSynchronize(cudaStreamLegacy), "One-sided copy");
            e.deviceCopies = false;
        }
        markComplete(w.progress[rank], [&](int t) { return isLocalRank(t); });
        if (unlock) {
            std::vector<std::function<void()>> sends;
            {
                std::lock_guard<std::mutex> lk(w.lockMx);
                sends = releaseLock(w.locks[targetRank], t.exclusive);
            }
            announceGrants(w, sends);
        }
        return MPI_SUCCESS;
    }
    // Ship the operations queued for the target; it applies them, waits for
    // its streams and answers with the fetched values
    std::vector<uint8_t> req;
    append(req, RmaPassiveHeader{ id, winId, rank, targetRank, t.exclusive ? 1 : 0, 0, 0 });
    std::vector<const RmaOp*> replies;
    size_t replyBytes = 0;
    int nOps = 0;
    for (const RmaOp& op : w.pending[rank]) {
        if (op.target != targetRank) {
            continue;
        }
        append(req, RmaWireOp{ op.kind, op.dtype, op.dispBytes, op.bytes, op.op, 0 });
        const uint8_t* payload = op.kind == RMA_PUT ? op.origin : op.kind == RMA_GET ? nullptr : op.data.data();
        const size_t payloadBytes = op.kind == RMA_PUT ? op.bytes : op.kind == RMA_GET ? 0 : op.data.size();
        if (payloadBytes > 0) {
            req.resize(req.size() + payloadBytes);
            copyBytes(req.data() + req.size() - payloadBytes, payload, payloadBytes);
        }
        if (op.kind == RMA_GET || op.kind == RMA_GET_ACCUMULATE || op.kind == RMA_COMPARE_SWAP) {
            replies.push_back(&op);
            replyBytes += op.bytes;
        }
        nOps++;
    }
    if (nOps == 0 && !unlock) {
        markComplete(w.progress[rank], [&](int t) { return t == targetRank; });
        return MPI_SUCCESS;
    }
    reinterpret_cast<RmaPassiveHeader*>(req.data())->nOps = nOps;
    std::vector<uint8_t> fetched;
    int32_t status = rmaCall(getHostForRank(targetRank),
                             unlock ? faabric::transport::PointToPointCall::RMA_UNLOCK
                                    : faabric::transport::PointToPointCall::RMA_FLUSH,
                             req,
                             &fetched);
    if (status == RMA_REPLY_OK && fetched.size() != replyBytes) {
        status = RMA_REPLY_FAILED;
    }
    if (status == RMA_REPLY_OK) {
        size_t off = 0;
        bool toDevice = false;
        for (const RmaOp* op : replies) {
            uint8_t* dst = op->kind == RMA_GET ? op->origin : op->result;
            copyBytes(dst, fetched.data() + off, op->bytes);
            toDevice |= !hostAddressable(dst);
            off += op->bytes;
        }
        if (toDevice) {
            // (a copy from pageable memory may return before its DMA lands)
            cudaCheck(cudaStreamSynchronize(cudaStreamLegacy), "Returning fetched values");
        }
    }
    auto& pending = w.pending[rank];
    pending.erase(std::remove_if(pending.begin(), pending.end(), [&](const RmaOp& op) { return op.target == targetRank; }),
                  pending.end());
    // The requests to the target are over: done, or failed with this call's
    // error (a later wait on one of them must not ship anything again)
    markComplete(w.progress[rank], [&](int t) { return t == targetRank; });
    return mpiErrorOf(status);
}

int MpiWorld::winLock(int rank, int winId, int lockType, int targetRank, int assert)
{
    auto w = findWindow(winId);
    if (w == nullptr) {
        return MPI_ERR_WIN;
    }
    if (targetRank < 0 || targetRank >= size) {
        return MPI_ERR_RANK;
    }
    if (lockType != MPI_LOCK_EXCLUSIVE && lockType != MPI_LOCK_SHARED) {
        return MPI_ERR_ARG;
    }
    RmaEpoch& e = w->epochs[rank];
    if (e.all || e.locked.count(targetRank) > 0) {
        return MPI_ERR_RMA_SYNC;
    }
    const bool exclusive = lockType == MPI_LOCK_EXCLUSIVE;
    const bool nocheck = (assert & MPI_MODE_NOCHECK) != 0;
    if (!nocheck) {
        int rc = rmaAcquire(*w, winId, rank, targetRank, exclusive);
        if (rc != MPI_SUCCESS) {
            return rc;
        }
    }
    e.locked[targetRank] = RmaEpoch::Target{ exclusive, nocheck };
    return MPI_SUCCESS;
}

int MpiWorld::winUnlock(int rank, int winId, int targetRank)
{
    auto w = findWindow(winId);
    if (w == nullptr) {
        return MPI_ERR_WIN;
    }
    if (targetRank < 0 || targetRank >= size) {
        return MPI_ERR_RANK;
    }
    RmaEpoch& e = w->epochs[rank];
    if (e.all || e.locked.count(targetRank) == 0) {
        return MPI_ERR_RMA_SYNC;
    }
    int rc = rmaComplete(*w, winId, rank, targetRank, true);
    e.locked.erase(targetRank);
    return rc;
}

int MpiWorld::winLockAll(int rank, int winId, int assert)
{
    auto w = findWindow(winId);
    if (w == nullptr) {
        return MPI_ERR_WIN;
    }
    RmaEpoch& e = w->epochs[rank];
    if (e.all || !e.locked.empty()) {
        return MPI_ERR_RMA_SYNC;
    }
    const bool nocheck = (assert & MPI_MODE_NOCHECK) != 0;
    // Shared locks in increasing rank order
    for (int t = 0; t < size; t++) {
        if (!nocheck) {
            int rc = rmaAcquire(*w, winId, rank, t, false);
            if (rc != MPI_SUCCESS) {
                for (int u = 0; u < t; u++) {
                    rmaComplete(*w, winId, rank, u, true);
                }
                e.locked.clear();
                return rc;
            }
        }
        e.locked[t] = RmaEpoch::Target{ false, nocheck };
    }
    e.all = true;
    return MPI_SUCCESS;
}

int MpiWorld::winUnlockAll(int rank, int winId)
{
    auto w = findWindow(winId);
    if (w == nullptr) {
        return MPI_ERR_WIN;
    }
    RmaEpoch& e = w->epochs[rank];
    if (!e.all) {
        return MPI_ERR_RMA_SYNC;
    }
    int rc = MPI_SUCCESS;
    for (int t = 0; t < size; t++) {
        int r = rmaComplete(*w, winId, rank, t, true);
        rc = rc == MPI_SUCCESS ? r : rc;
    }
    e.locked.clear();
    e.all = false;
    return rc;
}

int MpiWorld::winFlush(int rank, int winId, int targetRank)
{
    auto w = findWindow(winId);
    if (w == nullptr) {
        return MPI_ERR_WIN;
    }
    RmaEpoch& e = w->epochs[rank];
    if (targetRank >= 0 && targetRank < size) {
        return e.locked.count(targetRank) == 0 ? MPI_ERR_RMA_SYNC : rmaComplete(*w, winId, rank, targetRank, false);
    }
    if (targetRank != -1) {
        return MPI_ERR_RANK;
    }
    if (e.locked.empty()) {
        return MPI_ERR_RMA_SYNC;
    }
    int rc = MPI_SUCCESS;
    for (const auto& [t, how] : e.locked) {
        int r = rmaComplete(*w, winId, rank, t, false);
        rc = rc == MPI_SUCCESS ? r : rc;
    }
    return rc;
}

bool MpiWorld::winInPassiveEpoch(int rank, int winId)
{
    auto w = findWindow(winId);
    return w != nullptr && rank >= 0 && rank < size && !w->epochs[rank].locked.empty();
}

// ---------------------------------------------------------------------------
// Request-based operations (MPI_Rput, MPI_Rget, MPI_Raccumulate,
// MPI_Rget_accumulate)
// ---------------------------------------------------------------------------
void MpiWorld::rmaIssueBatch(RmaWindow& w, int rank)
{
    auto& batch = w.batches[rank];
    if (batch.empty()) {
        return;
    }
    auto comm = wiredDeviceComm(rank);
    const int device = comm->isLoopback() ? HOST_MEMORY : comm->device();
    cudaStream_t s = (cudaStream_t)streamForRank(rank);
    DeviceGuard on(device);
    const int rc = comm->putGetMany(batch.data(), batch.size(), s);
    batch.clear();
    if (rc != FB_OK) {
        throw std::runtime_error(std::string("Batched one-sided copy failed: ") +
                                 faabric::device::Communicator::errorString(rc));
    }
    auto& used = w.streams[rank];
    if (device != HOST_MEMORY && std::find(used.begin(), used.end(), std::make_pair(device, (void*)s)) == used.end()) {
        used.emplace_back(device, (void*)s);
    }
}

int MpiWorld::rmaRequestTarget(RmaWindow& w, int rank, int targetRank, int64_t targetDisp, size_t bytes, uint8_t** target)
{
    if (targetRank < 0 || targetRank >= size) {
        return MPI_ERR_RANK;
    }
    const int64_t off = targetDisp * (int64_t)w.dispUnits[targetRank];
    if (targetDisp < 0 || bytes > (uint64_t)w.sizes[targetRank] || off > w.sizes[targetRank] - (int64_t)bytes) {
        SPDLOG_ERROR("Request-based one-sided access [{}, {}) outside the {}-byte window of rank {}", off, off + (int64_t)bytes, w.sizes[targetRank], targetRank);
        return MPI_ERR_ARG;
    }
    // MPI-3.1 11.3.5: only inside a passive epoch that covers the target
    if (w.epochs[rank].locked.count(targetRank) == 0) {
        return MPI_ERR_RMA_SYNC;
    }
    *target = (uint8_t*)(uintptr_t)w.bases[targetRank] + off;
    if (w.progress[rank] == nullptr) {
        w.progress[rank] = std::make_shared<RmaProgress>();
        w.progress[rank]->issued.resize(size, 0);
        w.progress[rank]->completed.resize(size, 0);
    }
    return MPI_SUCCESS;
}

int MpiWorld::winRputGet(int rank, int winId, uint8_t* origin, size_t bytes, int targetRank, int64_t targetDisp, bool get, int* requestId)
{
    auto w = findWindow(winId);
    if (w == nullptr) {
        return MPI_ERR_WIN;
    }
    if (requestId == nullptr || (origin == nullptr && bytes > 0)) {
        return MPI_ERR_ARG;
    }
    uint8_t* target = nullptr;
    int rc = rmaRequestTarget(*w, rank, targetRank, targetDisp, bytes, &target);
    if (rc != MPI_SUCCESS) {
        return rc;
    }
    if (isLocalRank(targetRank) && bytes > 0) {
        // Heap to heap, origin on the origin's GPU: one launch for the batch
        // (on the loopback backend the origin is in a heap: device-role
        // memory that memcpy reaches)
        auto comm = wiredDeviceComm(rank);
        auto targetComm = wiredDeviceComm(targetRank);
        const bool originOk =
          comm != nullptr && (comm->isLoopback() ? isDevicePointer(origin) && hostAddressable(origin)
                                                 : comm->inHeap(origin, bytes) || bufferDevice(origin) == comm->device());
        if (originOk && targetComm != nullptr && targetComm->inHeap(target, bytes)) {
            auto& batch = w->batches[rank];
            batch.push_back(faabric::device::Communicator::RmaCopy{
              origin, targetComm->offsetOf(target), bytes, targetRank, get ? 1 : 0 });
            if (batch.size() >= FB_RMA_COPY_MAX_ITEMS) {
                rmaIssueBatch(*w, rank);
            }
            *requestId = addRmaRequest(rank, winId, targetRank, w->progress[rank]);
            return MPI_SUCCESS;
        }
    }
    // Today's MPI_Put / MPI_Get: a copy now (this process), or queued for
    // the flush of a target in another process
    if (get) {
        winGet(rank, winId, origin, bytes, targetRank, targetDisp);
    } else {
        winPut(rank, winId, origin, bytes, targetRank, targetDisp);
    }
    if (isLocalRank(targetRank) && (!hostAddressable(origin) || !hostAddressable(target))) {
        // complete at issue: a cudaMemcpy that involves pageable memory may
        // return before its DMA lands, and the request's wait does nothing
        cudaCheck(cudaStreamSynchronize(cudaStreamLegacy), "Request-based one-sided copy");
    }
    *requestId = addRmaRequest(rank, winId, targetRank, isLocalRank(targetRank) ? nullptr : w->progress[rank]);
    return MPI_SUCCESS;
}

int MpiWorld::winRaccumulate(int rank,
                             int winId,
                             const uint8_t* origin,
                             size_t count,
                             faabric_datatype_t* datatype,
                             faabric_op_t* op,
                             uint8_t* result,
                             int targetRank,
                             int64_t targetDisp,
                             int* requestId)
{
    auto w = findWindow(winId);
    if (w == nullptr) {
        return MPI_ERR_WIN;
    }
    const int dtype = datatype != nullptr ? fbDtypeFor(datatype) : -1;
    if (requestId == nullptr || dtype < 0 || count > (size_t)INT64_MAX / fbDtypeSize(dtype)) {
        return MPI_ERR_ARG;
    }
    uint8_t* target = nullptr;
    int rc = rmaRequestTarget(*w, rank, targetRank, targetDisp, count * fbDtypeSize(dtype), &target);
    if (rc != MPI_SUCCESS) {
        return rc;
    }
    // (every other check of MPI_Accumulate runs before it applies anything)
    rc = winAccumulate(rank, winId, origin, count, datatype, op, result, targetRank, targetDisp);
    if (rc != MPI_SUCCESS) {
        return rc;
    }
    *requestId = addRmaRequest(rank, winId, targetRank, w->progress[rank]);
    return MPI_SUCCESS;
}

void MpiWorld::rmaAwait(int rank, int winId, int targetRank)
{
    auto w = findWindow(winId);
    if (w == nullptr) {
        throw std::runtime_error("Waiting for a one-sided request on a freed window");
    }
    if (isLocalRank(targetRank)) {
        rmaIssueBatch(*w, rank);
        rmaWaitStreams(*w, rank);
        markComplete(w->progress[rank], [&](int t) { return isLocalRank(t); });
        return;
    }
    const int rc = rmaComplete(*w, winId, rank, targetRank, false);
    if (rc != MPI_SUCCESS) {
        throw std::runtime_error("One-sided request to rank " + std::to_string(targetRank) + " failed");
    }
}

std::string MpiWorld::serveRmaRequest(int call, const uint8_t* buffer, size_t bytes)
{
    RmaPassiveHeader h{};
    if (bytes < sizeof(h)) {
        return replyOf(RMA_REPLY_FAILED);
    }
    memcpy(&h, buffer, sizeof(h));
    auto world = getMpiWorldRegistry().findWorld(h.worldId);
    if (world == nullptr) {
        SPDLOG_WARN("One-sided request for world {}, which this process does not know", h.worldId);
        return replyOf(RMA_REPLY_NO_WINDOW);
    }
    try {
        return world->rmaServe(call, buffer, bytes);
    } catch (const std::exception& e) {
        SPDLOG_ERROR("One-sided request from rank {} to rank {} failed: {}", h.origin, h.target, e.what());
        return replyOf(RMA_REPLY_FAILED);
    }
}

void MpiWorld::serveRmaGrant(const uint8_t* buffer, size_t bytes)
{
    uint64_t ticket = 0;
    if (bytes != sizeof(ticket)) {
        SPDLOG_ERROR("Malformed one-sided lock grant");
        return;
    }
    memcpy(&ticket, buffer, sizeof(ticket));
    GrantTable& g = grantTable();
    {
        std::lock_guard<std::mutex> lk(g.mx);
        g.granted.insert(ticket);
    }
    g.cv.notify_all();
}

std::string MpiWorld::rmaServe(int call, const uint8_t* buffer, size_t bytes)
{
    using faabric::transport::PointToPointCall;
    RmaPassiveHeader h{};
    memcpy(&h, buffer, sizeof(h));
    auto w = findWindow(h.winId);
    if (w == nullptr || h.origin < 0 || h.origin >= size || h.target < 0 || h.target >= size || !isLocalRank(h.target)) {
        SPDLOG_WARN("One-sided request for window {} of rank {} in world {}, which this process does not hold", h.winId, h.target, id);
        return replyOf(RMA_REPLY_NO_WINDOW);
    }
    RmaLock& l = w->locks[h.target];
    const bool exclusive = h.exclusive != 0;
    if (call == PointToPointCall::RMA_LOCK) {
        // Never wait here: a queued request is answered by a grant message
        const std::string originHost = getHostForRank(h.origin);
        std::lock_guard<std::mutex> lk(w->lockMx);
        auto granted = std::make_shared<bool>(false);
        l.waiters.push_back(RmaLockWaiter{ h.ticket, exclusive, granted, nullptr });
        grantWaiters(l);
        if (*granted) {
            return replyOf(RMA_REPLY_OK);
        }
        const uint64_t ticket = h.ticket;
        l.waiters.back().onGrant = [originHost, ticket] {
            faabric::transport::getPointToPointClient(originHost)->rmaLockGrant((const uint8_t*)&ticket, sizeof(ticket));
        };
        return replyOf(RMA_REPLY_QUEUED);
    }
    if (call == PointToPointCall::RMA_LOCK_CANCEL) {
        std::vector<std::function<void()>> sends;
        {
            std::lock_guard<std::mutex> lk(w->lockMx);
            sends = dropWaiter(l, h.ticket) ? grantWaiters(l) : releaseLock(l, exclusive);
        }
        announceGrants(*w, sends);
        return replyOf(RMA_REPLY_OK);
    }
    // Flush / unlock.  An unlock releases the lock even if its operations
    // fail.
    struct ReleaseAtExit
    {
        MpiWorld::RmaWindow& w;
        RmaLock& l;
        bool exclusive;
        bool armed;
        ~ReleaseAtExit()
        {
            if (!armed) {
                return;
            }
            std::vector<std::function<void()>> sends;
            {
                std::lock_guard<std::mutex> lk(w.lockMx);
                sends = releaseLock(l, exclusive);
            }
            announceGrants(w, sends);
        }
    } release{ *w, l, exclusive, call == PointToPointCall::RMA_UNLOCK };
    // Check every operation, then apply them in order
    struct Item
    {
        RmaWireOp wire;
        const uint8_t* data;
        size_t replyOff;
    };
    uint8_t* base = (uint8_t*)(uintptr_t)w->bases[h.target];
    const uint64_t segBytes = (uint64_t)w->sizes[h.target];
    std::vector<Item> items;
    size_t off = sizeof(h), replyBytes = 0;
    for (int i = 0; i < h.nOps; i++) {
        Item it{ {}, nullptr, replyBytes };
        if (bytes - off < sizeof(it.wire)) {
            throw std::runtime_error("Truncated one-sided request");
        }
        memcpy(&it.wire, buffer + off, sizeof(it.wire));
        off += sizeof(it.wire);
        const RmaWireOp& wire = it.wire;
        if (wire.bytes > segBytes || wire.dispBytes > segBytes - wire.bytes) {
            throw std::runtime_error("Remote one-sided operation outside this rank's window");
        }
        const size_t dataBytes = wire.kind == RMA_PUT   ? wire.bytes
                                 : wire.kind == RMA_GET ? 0
                                                        : rmaAtomicPayload(wire.kind, wire.dtype, wire.op, wire.bytes, base + wire.dispBytes);
        if (bytes - off < dataBytes) {
            throw std::runtime_error("Truncated one-sided request");
        }
        it.data = buffer + off;
        off += dataBytes;
        if (wire.kind != RMA_PUT && wire.kind != RMA_ACCUMULATE) {
            replyBytes += wire.bytes;
        }
        items.push_back(it);
    }
    std::string reply = replyOf(RMA_REPLY_OK);
    reply.resize(sizeof(int32_t) + replyBytes);
    uint8_t* out = (uint8_t*)reply.data() + sizeof(int32_t);
    // Device work goes on this path's own streams, waited for before the reply
    std::vector<std::pair<int, void*>> used;
    auto copy = [&](uint8_t* dst, const uint8_t* src, size_t n) {
        int device = bufferDevice(dst);
        device = device == HOST_MEMORY ? bufferDevice(src) : device;
        if (device == HOST_MEMORY) {
            memcpy(dst, src, n);
            return;
        }
        if (device == ANY_DEVICE) {
            cudaCheck(cudaGetDevice(&device), "One-sided copy");
        }
        void* s = rmaStream(-1, device);
        DeviceGuard on(device);
        cudaCheck(cudaMemcpyAsync(dst, src, n, cudaMemcpyDefault, (cudaStream_t)s), "One-sided copy");
        if (std::find(used.begin(), used.end(), std::make_pair(device, s)) == used.end()) {
            used.emplace_back(device, s);
        }
    };
    for (const Item& it : items) {
        const RmaWireOp& wire = it.wire;
        uint8_t* target = base + wire.dispBytes;
        if (wire.kind == RMA_PUT) {
            copy(target, it.data, wire.bytes);
        } else if (wire.kind == RMA_GET) {
            copy(out + it.replyOff, target, wire.bytes);
        } else {
            const bool cas = wire.kind == RMA_COMPARE_SWAP;
            const size_t esize = fbDtypeSize(wire.dtype);
            const bool hasData = cas || wire.op != FB_OP_NO_OP;
            rmaApplyLocal(*w,
                          h.target,
                          h.target,
                          target,
                          wire.bytes / esize,
                          wire.dtype,
                          wire.op,
                          hasData ? it.data : nullptr,
                          cas ? it.data + esize : nullptr,
                          wire.kind != RMA_ACCUMULATE ? out + it.replyOff : nullptr,
                          used,
                          true);
        }
    }
    for (auto [device, s] : used) {
        DeviceGuard on(device);
        cudaCheck(cudaStreamSynchronize((cudaStream_t)s), "One-sided operation");
    }
    return reply;
}

}
