// C ABI over the device layer (Communicator + snapshot/state kernels) used by
// the Python package (ctypes) and by C callers.  Every function returns 0 / a
// negative FB_E_* code or a handle; fb_last_error() gives the message of the
// last exception caught on this thread.
#include "faabric/device/communicator.h"
#include "faabric/device/cuda_driver.h"
#include "launch_api.h"

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

using faabric::device::CommConfig;
using faabric::device::Communicator;

static thread_local std::string g_lastError;

#define FB_TRY try {
#define FB_CATCH(ret)                                                          \
    }                                                                          \
    catch (const std::exception& e)                                            \
    {                                                                          \
        g_lastError = e.what();                                                \
        return ret;                                                            \
    }

namespace {
// The kernels below run on the device that OWNS the buffers, whatever the
// calling thread's current device happens to be (other calls of this library
// and of the caller's framework move it around)
struct OwnerDeviceGuard
{
    int prev = -1;
    explicit OwnerDeviceGuard(const void* devicePtr)
    {
        cudaPointerAttributes attr;
        if (devicePtr != nullptr && cudaPointerGetAttributes(&attr, devicePtr) == cudaSuccess &&
            (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged)) {
            cudaGetDevice(&prev);
            if (prev != attr.device) {
                cudaSetDevice(attr.device);
            } else {
                prev = -1;
            }
        } else {
            cudaGetLastError();
        }
    }
    ~OwnerDeviceGuard()
    {
        if (prev >= 0) {
            cudaSetDevice(prev);
        }
    }
};
}

extern "C" {

struct FbConfigC
{
    uint64_t heapBytes;
    uint64_t stageBytes;
    uint64_t slotBytes;
    uint64_t timeoutMs;
    int32_t useVmm;
    int32_t useMulticast;
    int32_t maxBlocks;
    int32_t threads;
    int32_t channels;
    int32_t reserved;
    uint64_t llMaxBytes;
    uint64_t oneShotMaxBytes;
    uint64_t nvlsMinBytes;
    uint64_t bcast2StepMinBytes;
    uint64_t p2pBounceBytes;
    int32_t groupBlocks;
    int32_t streamSync; // -1 auto, 0 in-kernel barriers, 1 stream memory ops
};

const char* fb_last_error()
{
    return g_lastError.c_str();
}

int fb_cuda_device_count()
{
    return faabric::device::cudaDeviceCountSafe();
}

void fb_default_config(FbConfigC* out)
{
    CommConfig c = CommConfig::fromEnv();
    out->heapBytes = c.heapBytes;
    out->stageBytes = c.stageBytes;
    out->slotBytes = c.slotBytes;
    out->timeoutMs = c.timeoutMs;
    out->useVmm = c.useVmm;
    out->useMulticast = c.useMulticast;
    out->maxBlocks = c.maxBlocks;
    out->threads = c.threads;
    out->channels = c.channels;
    out->reserved = 0;
    out->llMaxBytes = c.llMaxBytes;
    out->oneShotMaxBytes = c.oneShotMaxBytes;
    out->nvlsMinBytes = c.nvlsMinBytes;
    out->bcast2StepMinBytes = c.bcast2StepMinBytes;
    out->p2pBounceBytes = c.p2pBounceBytes;
    out->groupBlocks = c.groupBlocks;
    out->streamSync = c.streamSync;
}

static CommConfig fromC(const FbConfigC* in)
{
    CommConfig c = CommConfig::fromEnv();
    if (in == nullptr) {
        return c;
    }
    c.heapBytes = in->heapBytes;
    c.stageBytes = in->stageBytes;
    c.slotBytes = in->slotBytes;
    c.timeoutMs = in->timeoutMs;
    c.useVmm = in->useVmm != 0;
    c.useMulticast = in->useMulticast != 0;
    c.maxBlocks = in->maxBlocks;
    c.threads = in->threads;
    c.channels = in->channels;
    c.llMaxBytes = in->llMaxBytes;
    c.oneShotMaxBytes = in->oneShotMaxBytes;
    c.nvlsMinBytes = in->nvlsMinBytes;
    c.bcast2StepMinBytes = in->bcast2StepMinBytes;
    c.p2pBounceBytes = in->p2pBounceBytes;
    c.groupBlocks = in->groupBlocks;
    c.streamSync = in->streamSync;
    return c;
}

struct FbGroup
{
    std::vector<std::shared_ptr<Communicator>> comms;
};

struct FbCommHandle
{
    std::shared_ptr<Communicator> comm;
};

void* fb_group_create_local(int nranks, const int* devices, const FbConfigC* cfg)
{
    FB_TRY
    std::vector<int> devs(devices, devices + nranks);
    auto* g = new FbGroup();
    g->comms = Communicator::createLocal(nranks, devs, fromC(cfg));
    return g;
    FB_CATCH(nullptr)
}

void* fb_group_comm(void* group, int rank)
{
    auto* g = (FbGroup*)group;
    if (g == nullptr || rank < 0 || rank >= (int)g->comms.size()) {
        return nullptr;
    }
    auto* h = new FbCommHandle();
    h->comm = g->comms[rank];
    return h;
}

void fb_group_destroy(void* group)
{
    delete (FbGroup*)group;
}

void* fb_comm_create_ipc(int rank,
                         int nranks,
                         int device,
                         const char* jobId,
                         const FbConfigC* cfg)
{
    FB_TRY
    auto* h = new FbCommHandle();
    h->comm = Communicator::createIpc(rank, nranks, device, jobId, fromC(cfg));
    return h;
    FB_CATCH(nullptr)
}

void fb_comm_destroy(void* h)
{
    delete (FbCommHandle*)h;
}

#define COMM(h) (((FbCommHandle*)(h))->comm)

int fb_comm_rank(void* h)
{
    return COMM(h)->rank();
}
int fb_comm_size(void* h)
{
    return COMM(h)->size();
}
int fb_comm_device(void* h)
{
    return COMM(h)->device();
}
int fb_comm_has_multicast(void* h)
{
    return COMM(h)->hasMulticast() ? 1 : 0;
}
const char* fb_comm_backing(void* h)
{
    return COMM(h)->backing().c_str();
}
int fb_comm_last_algo(void* h)
{
    return COMM(h)->lastAlgo();
}

// key: 0 llMax 1 oneShotMax 2 nvlsMin 3 bcast2StepMin 4 maxBlocks 5 threads
int fb_comm_configure(void* h, int key, uint64_t value)
{
    auto& c = COMM(h)->config();
    switch (key) {
        case 0:
            c.llMaxBytes = value;
            break;
        case 1:
            c.oneShotMaxBytes = value;
            break;
        case 2:
            c.nvlsMinBytes = value;
            break;
        case 3:
            c.bcast2StepMinBytes = value;
            break;
        case 4:
            c.maxBlocks = (int)value;
            break;
        case 5:
            c.threads = (int)value;
            break;
        case 6:
            c.tmaMinBytes = value; // 0 = never use the bulk copy engine
            break;
        case 7:
            c.nvlsScalarMinBytes = value;
            break;
        case 8:
            c.groupBlocks = (int)value;
            break;
        default:
            return FB_E_INVALID;
    }
    return FB_OK;
}

// Applies a tuning file to a live communicator: 0, FB_E_INVALID (unreadable
// or malformed; the message goes to stderr)
int fb_comm_load_tuning(void* h, const char* path)
{
    try {
        faabric::device::CommTuning t;
        if (!faabric::device::CommTuning::loadFile(path, t)) {
            return FB_E_INVALID;
        }
        COMM(h)->applyTuning(t);
        return FB_OK;
    } catch (const std::exception& e) {
        fprintf(stderr, "faabric_b200: %s\n", e.what());
        return FB_E_INVALID;
    }
}

// Parses + re-serialises tuning text without a device (format checks, tools).
// Returns the length written (excluding NUL), or -1 on a parse error with the
// message in `out`.
int fb_tuning_normalise(const char* text, char* out, int cap)
{
    std::string res;
    int rc = 0;
    try {
        res = faabric::device::CommTuning::parse(text).serialise();
        rc = (int)res.size();
    } catch (const std::exception& e) {
        res = e.what();
        rc = -1;
    }
    if (cap > 0) {
        size_t n = std::min(res.size(), (size_t)cap - 1);
        memcpy(out, res.data(), n);
        out[n] = 0;
        if (rc >= 0) {
            rc = (int)n;
        }
    }
    return rc;
}

int fb_comm_set_allreduce_table(void* h,
                                int n,
                                const uint64_t* maxBytes,
                                const int* algos)
{
    std::vector<uint64_t> mb(maxBytes, maxBytes + n);
    std::vector<int> al(algos, algos + n);
    COMM(h)->setAllReduceTable(mb, al);
    return FB_OK;
}

// out[0]=launches [1]=bytes [2]=stagedCopies [3..3+FB_ALGO_COUNT) algo counts
void fb_comm_stats(void* h, uint64_t* out, int reset)
{
    const auto& s = COMM(h)->stats();
    out[0] = s.launches;
    out[1] = s.bytes;
    out[2] = s.stagedCopies;
    for (int i = 0; i < FB_ALGO_COUNT; i++) {
        out[3 + i] = s.algoCount[i];
    }
    out[15] = s.tmaLaunches;
    if (reset) {
        COMM(h)->resetStats();
    }
}

int64_t fb_comm_alloc(void* h, uint64_t bytes)
{
    FB_TRY
    return (int64_t)COMM(h)->alloc(bytes);
    FB_CATCH(-1)
}

void fb_comm_free(void* h, uint64_t off)
{
    try {
        COMM(h)->free(off);
    } catch (const std::exception& e) {
        g_lastError = e.what();
    }
}

// A communicator over `members` (ranks of `h`, in child order) using signal
// slot `slot`; null on failure (fb_last_error).  Release with fb_comm_destroy
// once the child's last collective has completed: it zeroes the slot pad
// without waiting for the caller's streams.  The child runs every
// collective and grouped call of Communicator::subset (point to point,
// put-signal, the one-sided calls and host barriers stay on the parent).
void* fb_comm_subset(void* h, const int* members, int n, int slot)
{
    FB_TRY
    int rc = FB_OK;
    auto child = COMM(h)->subset(std::vector<int>(members, members + std::max(n, 0)), slot, &rc);
    if (child == nullptr) {
        g_lastError = std::string("subset: ") + Communicator::errorString(rc);
        return nullptr;
    }
    auto* c = new FbCommHandle();
    c->comm = std::move(child);
    return c;
    FB_CATCH(nullptr)
}

uint32_t fb_comm_free_subset_slots(void* h)
{
    return COMM(h)->freeSubsetSlots();
}

int fb_comm_is_subset(void* h)
{
    return COMM(h)->isSubset() ? 1 : 0;
}

void* fb_comm_heap_ptr(void* h, uint64_t off, int rank)
{
    return COMM(h)->heapPtr(off, rank);
}

int fb_comm_in_heap(void* h, const void* p, uint64_t bytes)
{
    return COMM(h)->inHeap(p, bytes) ? 1 : 0;
}

uint32_t fb_comm_check_error(void* h, void* stream)
{
    return COMM(h)->checkError((cudaStream_t)stream);
}

void fb_comm_host_barrier(void* h)
{
    try {
        COMM(h)->hostBarrier();
    } catch (const std::exception& e) {
        g_lastError = e.what();
    }
}

int fb_allreduce(void* h,
                 const void* send,
                 void* recv,
                 uint64_t count,
                 int dtype,
                 int op,
                 int algo,
                 int flags,
                 void* stream)
{
    return COMM(h)->allReduce(
      send, recv, count, dtype, op, algo, flags, (cudaStream_t)stream);
}

int fb_reduce(void* h,
              const void* send,
              void* recv,
              uint64_t count,
              int dtype,
              int op,
              int root,
              int flags,
              void* stream)
{
    return COMM(h)->reduce(
      send, recv, count, dtype, op, root, flags, (cudaStream_t)stream);
}

int fb_reduce_scatter(void* h,
                      const void* send,
                      void* recv,
                      uint64_t recvCount,
                      int dtype,
                      int op,
                      int flags,
                      void* stream)
{
    return COMM(h)->reduceScatter(
      send, recv, recvCount, dtype, op, flags, (cudaStream_t)stream);
}

int fb_scan(void* h,
            const void* send,
            void* recv,
            uint64_t count,
            int dtype,
            int op,
            int flags,
            void* stream)
{
    return COMM(h)->scan(
      send, recv, count, dtype, op, flags, (cudaStream_t)stream);
}

int fb_broadcast(void* h,
                 void* buf,
                 uint64_t bytes,
                 int root,
                 int flags,
                 void* stream)
{
    return COMM(h)->broadcast(buf, bytes, root, flags, (cudaStream_t)stream);
}

int fb_allgather(void* h,
                 const void* send,
                 void* recv,
                 uint64_t bytesPerRank,
                 int flags,
                 void* stream)
{
    return COMM(h)->allGather(
      send, recv, bytesPerRank, flags, (cudaStream_t)stream);
}

int fb_gather(void* h,
              const void* send,
              void* recv,
              uint64_t bytesPerRank,
              int root,
              int flags,
              void* stream)
{
    return COMM(h)->gather(
      send, recv, bytesPerRank, root, flags, (cudaStream_t)stream);
}

int fb_scatter(void* h,
               const void* send,
               void* recv,
               uint64_t bytesPerRank,
               int root,
               int flags,
               void* stream)
{
    return COMM(h)->scatter(
      send, recv, bytesPerRank, root, flags, (cudaStream_t)stream);
}

int fb_alltoall(void* h,
                const void* send,
                void* recv,
                uint64_t bytesPerRank,
                int flags,
                void* stream)
{
    return COMM(h)->allToAll(
      send, recv, bytesPerRank, flags, (cudaStream_t)stream);
}

int fb_barrier(void* h, void* stream)
{
    return COMM(h)->barrier((cudaStream_t)stream);
}

int fb_send(void* h, const void* buf, uint64_t bytes, int peer, void* stream)
{
    return COMM(h)->send(buf, bytes, peer, (cudaStream_t)stream);
}

int fb_recv(void* h, void* buf, uint64_t bytes, int peer, void* stream)
{
    return COMM(h)->recv(buf, bytes, peer, (cudaStream_t)stream);
}

int fb_sendrecv(void* h,
                const void* sendBuf,
                uint64_t sendBytes,
                int dst,
                void* recvBuf,
                uint64_t recvBytes,
                int src,
                void* stream)
{
    return COMM(h)->sendRecv(
      sendBuf, sendBytes, dst, recvBuf, recvBytes, src, (cudaStream_t)stream);
}

int fb_comm_stream_sync(void* h)
{
    return COMM(h)->streamSync() ? 1 : 0;
}

int fb_comm_stream_wait_supported(void* h)
{
    return COMM(h)->streamWaitSupported() ? 1 : 0;
}

// 1 = stream drained, 0 = timed out (pending stream waits were released and
// the error word set)
int fb_comm_sync_bounded(void* h, void* stream, uint64_t timeoutMs)
{
    return COMM(h)->syncStreamBounded((cudaStream_t)stream, timeoutMs) ? 1 : 0;
}

// ---- grouped collectives: `kind` is a Communicator::GroupKind ----
struct FbGroupPlanHandle
{
    std::shared_ptr<Communicator::GroupPlan> plan;
};

static std::vector<Communicator::GroupItem> groupItems(int n,
                                                       const void* const* send,
                                                       void* const* recv,
                                                       const uint64_t* counts)
{
    std::vector<Communicator::GroupItem> items((size_t)std::max(n, 0));
    for (int i = 0; i < n; i++) {
        items[i].send = send[i];
        items[i].recv = recv[i];
        items[i].count = (size_t)counts[i];
    }
    return items;
}

void* fb_group_prepare(void* h,
                       int kind,
                       int n,
                       const void* const* send,
                       void* const* recv,
                       const uint64_t* counts,
                       int dtype)
{
    FB_TRY
    auto items = groupItems(n, send, recv, counts);
    int rc = FB_OK;
    auto plan = COMM(h)->prepareGroup(items.data(), items.size(), dtype, &rc, (Communicator::GroupKind)kind);
    if (!plan) {
        g_lastError = std::string("prepareGroup: ") + Communicator::errorString(rc);
        return nullptr;
    }
    auto* ph = new FbGroupPlanHandle();
    ph->plan = plan;
    return ph;
    FB_CATCH(nullptr)
}

int fb_group_launch(void* h, int kind, void* plan, int op, int root, int flags, void* stream)
{
    if (plan == nullptr) {
        return FB_E_INVALID;
    }
    return COMM(h)->runGroup(
      (Communicator::GroupKind)kind, *((FbGroupPlanHandle*)plan)->plan, op, root, flags, (cudaStream_t)stream);
}

int fb_group_many(void* h,
                  int kind,
                  int n,
                  const void* const* send,
                  void* const* recv,
                  const uint64_t* counts,
                  int dtype,
                  int op,
                  int root,
                  int flags,
                  void* stream)
{
    FB_TRY
    auto items = groupItems(n, send, recv, counts);
    return COMM(h)->groupMany(
      (Communicator::GroupKind)kind, items.data(), items.size(), dtype, op, root, flags, (cudaStream_t)stream);
    FB_CATCH(FB_E_CUDA)
}

int fb_group_plan_launches(void* plan)
{
    return plan ? (int)Communicator::groupPlanLaunches(*((FbGroupPlanHandle*)plan)->plan) : 0;
}

void fb_group_plan_free(void* plan)
{
    delete (FbGroupPlanHandle*)plan;
}

// ---- grouped neighbourhood v-collectives: item i's counts and
// displacements are row i of `sendWidth` (send) and `recvWidth` (recv)
// entries; the rows must cover this rank's degrees (the all-gather reads one
// send count and no send displacement) ----
static int neighborVItems(void* h,
                          int kind,
                          int n,
                          const void* const* send,
                          void* const* recv,
                          const uint64_t* sendCounts,
                          const uint64_t* sendDispls,
                          int sendWidth,
                          const uint64_t* recvCounts,
                          const uint64_t* recvDispls,
                          int recvWidth,
                          std::vector<Communicator::NeighborVItem>& items)
{
    static_assert(sizeof(size_t) == sizeof(uint64_t), "counts are passed as size_t");
    const auto [inDeg, outDeg] = COMM(h)->neighborDegrees();
    const int sends = kind == Communicator::GROUP_NEIGHBOR_ALLTOALLV ? outDeg : std::min(outDeg, 1);
    if (n < 0 || sendWidth < sends || recvWidth < inDeg) {
        return FB_E_INVALID;
    }
    items.resize((size_t)n);
    for (int i = 0; i < n; i++) {
        const size_t so = (size_t)i * sendWidth;
        const size_t ro = (size_t)i * recvWidth;
        items[i] = { send[i],
                     recv[i],
                     sendCounts ? (const size_t*)sendCounts + so : nullptr,
                     sendDispls ? (const size_t*)sendDispls + so : nullptr,
                     recvCounts ? (const size_t*)recvCounts + ro : nullptr,
                     recvDispls ? (const size_t*)recvDispls + ro : nullptr };
    }
    return FB_OK;
}

#define FB_NEIGHBOR_V_ARGS                                                                                             \
    void *h, int kind, int n, const void *const *send, void *const *recv, const uint64_t *sendCounts,                \
      const uint64_t *sendDispls, int sendWidth, const uint64_t *recvCounts, const uint64_t *recvDispls,             \
      int recvWidth, int dtype
#define FB_NEIGHBOR_V_ITEMS(items)                                                                                     \
    neighborVItems(h, kind, n, send, recv, sendCounts, sendDispls, sendWidth, recvCounts, recvDispls, recvWidth, items)

// Communicator::neighborVStreams: the number of windows (at most `cap`
// written to `out`), or an FB_E_* code
int fb_neighbor_v_streams(FB_NEIGHBOR_V_ARGS, uint64_t* out, int cap)
{
    FB_TRY
    std::vector<Communicator::NeighborVItem> items;
    int rc = FB_NEIGHBOR_V_ITEMS(items);
    std::vector<uint64_t> streams;
    rc = rc == FB_OK ? COMM(h)->neighborVStreams((Communicator::GroupKind)kind, items.data(), items.size(), dtype,
                                                 streams)
                     : rc;
    if (rc != FB_OK) {
        return rc;
    }
    for (size_t w = 0; w < streams.size() && (int)w < cap; w++) {
        out[w] = streams[w];
    }
    return (int)streams.size();
    FB_CATCH(FB_E_INVALID)
}

void* fb_group_prepare_v(FB_NEIGHBOR_V_ARGS, const uint64_t* agreed, int nAgreed)
{
    FB_TRY
    std::vector<Communicator::NeighborVItem> items;
    int rc = FB_NEIGHBOR_V_ITEMS(items);
    std::shared_ptr<Communicator::GroupPlan> plan;
    if (rc == FB_OK) {
        plan = COMM(h)->prepareGroup(items.data(), items.size(), dtype,
                                     std::vector<uint64_t>(agreed, agreed + std::max(nAgreed, 0)), &rc,
                                     (Communicator::GroupKind)kind);
    }
    if (!plan) {
        g_lastError = std::string("prepareGroup: ") + Communicator::errorString(rc);
        return nullptr;
    }
    auto* ph = new FbGroupPlanHandle();
    ph->plan = plan;
    return ph;
    FB_CATCH(nullptr)
}

int fb_group_many_v(FB_NEIGHBOR_V_ARGS, const uint64_t* agreed, int nAgreed, int flags, void* stream)
{
    FB_TRY
    std::vector<Communicator::NeighborVItem> items;
    const int rc = FB_NEIGHBOR_V_ITEMS(items);
    if (rc != FB_OK) {
        return rc;
    }
    return COMM(h)->groupMany((Communicator::GroupKind)kind, items.data(), items.size(), dtype,
                              std::vector<uint64_t>(agreed, agreed + std::max(nAgreed, 0)), flags,
                              (cudaStream_t)stream);
    FB_CATCH(FB_E_CUDA)
}
#undef FB_NEIGHBOR_V_ARGS
#undef FB_NEIGHBOR_V_ITEMS

// Communicator::setNeighbors: in-edge j is (srcs[j], idxs[j])
int fb_comm_set_neighbors(void* h,
                          int nIn,
                          const int* srcs,
                          const int* idxs,
                          int outDegree,
                          int maxOutDegree,
                          int maxInDegree)
{
    FB_TRY
    std::vector<std::pair<int, int>> in((size_t)std::max(nIn, 0));
    for (int j = 0; j < nIn; j++) {
        in[j] = { srcs[j], idxs[j] };
    }
    return COMM(h)->setNeighbors(in, outDegree, maxOutDegree, maxInDegree);
    FB_CATCH(FB_E_INVALID)
}

int fb_put_signal(void* h,
                  const void* local,
                  uint64_t dstOffset,
                  uint64_t bytes,
                  int peer,
                  int signalIdx,
                  int blocks,
                  void* stream)
{
    return COMM(h)->putSignal(
      local, dstOffset, bytes, peer, signalIdx, blocks, (cudaStream_t)stream);
}

int fb_wait_signal(void* h, int signalIdx, uint32_t count, void* stream)
{
    return COMM(h)->waitSignal(signalIdx, count, (cudaStream_t)stream);
}

// One-sided atomics on peer's copy of the symmetric heap (Communicator::
// accumulate / compareAndSwap); `fetchOut` null means no fetch
int fb_accumulate(void* h,
                  const void* origin,
                  uint64_t dstOffset,
                  uint64_t count,
                  int dtype,
                  int op,
                  int peer,
                  void* fetchOut,
                  void* stream)
{
    return COMM(h)->accumulate(origin, dstOffset, count, dtype, op, peer, fetchOut, (cudaStream_t)stream);
}

int fb_compare_and_swap(void* h,
                        const void* compare,
                        const void* swap,
                        void* result,
                        uint64_t dstOffset,
                        int dtype,
                        int peer,
                        void* stream)
{
    return COMM(h)->compareAndSwap(compare, swap, result, dstOffset, dtype, peer, (cudaStream_t)stream);
}

// Batched one-sided copies (Communicator::putGetMany): item i copies bytes[i]
// between local[i] and peer[i]'s symmetric heap at offset[i], towards the
// heap when get[i] is 0 and out of it otherwise
int fb_put_get_many(void* h,
                    int n,
                    void* const* local,
                    const uint64_t* offset,
                    const uint64_t* bytes,
                    const int32_t* peer,
                    const int32_t* get,
                    void* stream)
{
    if (n < 0 || (n > 0 && (local == nullptr || offset == nullptr || bytes == nullptr || peer == nullptr || get == nullptr))) {
        return FB_E_INVALID;
    }
    FB_TRY
    std::vector<Communicator::RmaCopy> items(n);
    for (int i = 0; i < n; i++) {
        items[i] = Communicator::RmaCopy{ local[i], offset[i], (size_t)bytes[i], peer[i], get[i] != 0 ? 1 : 0 };
    }
    return COMM(h)->putGetMany(items.data(), items.size(), (cudaStream_t)stream);
    FB_CATCH(FB_E_CUDA)
}

// Batched one-sided atomics (Communicator::accumulateMany): item i combines
// count[i] elements of origin[i] into peer[i]'s symmetric heap at offset[i];
// fetch[i] null means no fetch; `fetch` itself may be null (no item fetches)
int fb_accumulate_many(void* h,
                       int n,
                       const void* const* origin,
                       void* const* fetch,
                       const uint64_t* offset,
                       const uint64_t* count,
                       const int32_t* peer,
                       int dtype,
                       int op,
                       void* stream)
{
    if (n < 0 || (n > 0 && (origin == nullptr || offset == nullptr || count == nullptr || peer == nullptr))) {
        return FB_E_INVALID;
    }
    FB_TRY
    std::vector<Communicator::RmaAccumulate> items(n);
    for (int i = 0; i < n; i++) {
        items[i] = Communicator::RmaAccumulate{ origin[i], fetch != nullptr ? fetch[i] : nullptr, offset[i], (size_t)count[i], peer[i] };
    }
    return COMM(h)->accumulateMany(items.data(), items.size(), dtype, op, (cudaStream_t)stream);
    FB_CATCH(FB_E_CUDA)
}

const char* fb_error_string(int code)
{
    return Communicator::errorString(code);
}

// ---------------------------------------------------------------------------
// Snapshot kernels (raw device pointers)
// ---------------------------------------------------------------------------

// Sort + gap-fill merge regions exactly like
// SnapshotData::fillGapsWithBytewiseRegions (reference
// src/util/snapshot.cpp:259-324) and split out the typed ones.  `fillOp` is
// FB_MERGE_BYTEWISE or FB_MERGE_XOR.  Returns the number of regions written to
// `out` (capacity maxOut) and the typed indices in typedOut, FB_E_INVALID for
// overlapping regions and FB_E_TOO_LARGE when `out` is too small.
int fb_snapshot_prepare_regions(const FbMergeRegionDev* in,
                                int nIn,
                                int fillOp,
                                uint64_t size,
                                FbMergeRegionDev* out,
                                int maxOut,
                                int32_t* typedOut,
                                int* nTypedOut)
{
    std::vector<FbMergeRegionDev> regs(in, in + nIn);
    std::sort(regs.begin(),
              regs.end(),
              [](const FbMergeRegionDev& a, const FbMergeRegionDev& b) {
                  return a.offset < b.offset;
              });
    std::vector<FbMergeRegionDev> filled;
    uint64_t cursor = 0;
    bool toEnd = false;
    for (const auto& r : regs) {
        // overlapping regions, or any region after a to-end one, are refused
        // (SnapshotData::fillGapsWithBytewiseRegions throws on the same input)
        if (toEnd || r.offset < cursor) {
            return FB_E_INVALID;
        }
        if (r.offset > cursor) {
            filled.push_back(
              { cursor, r.offset - cursor, FB_SNAP_RAW, fillOp });
        }
        filled.push_back(r);
        if (r.length == 0) {
            toEnd = true;
        } else {
            cursor = r.offset + r.length;
        }
    }
    if (!toEnd && cursor < size) {
        filled.push_back({ cursor, 0, FB_SNAP_RAW, fillOp });
    }
    int nTyped = 0;
    int n = 0;
    for (const auto& r : filled) {
        if (n >= maxOut) {
            return FB_E_TOO_LARGE;
        }
        out[n] = r;
        if (r.op != FB_MERGE_BYTEWISE && r.op != FB_MERGE_XOR &&
            r.op != FB_MERGE_IGNORE) {
            typedOut[nTyped++] = n;
        }
        n++;
    }
    *nTypedOut = nTyped;
    return n;
}

int fb_snapshot_diff_push(const void* mem,
                          const void* orig,
                          void* dst,
                          uint64_t size,
                          const void* regionsDev,
                          int nRegions,
                          const void* typedIdxDev,
                          int nTyped,
                          const void* dirtyPagesDev,
                          void* pageFlagsOutDev,
                          void* chunkFlagsDev,
                          void* statsDev,
                          int updateBase,
                          int blocks,
                          void* stream)
{
    OwnerDeviceGuard ownerGuard(mem);
    fb::SnapDiffArgs a;
    memset(&a, 0, sizeof(a));
    a.mem = (const uint8_t*)mem;
    a.orig = (const uint8_t*)orig;
    a.origW = updateBase ? (uint8_t*)orig : nullptr;
    a.dst = (uint8_t*)dst;
    a.size = size;
    a.regions = (const FbMergeRegionDev*)regionsDev;
    a.nRegions = nRegions;
    a.typedIdx = (const int32_t*)typedIdxDev;
    a.nTyped = nTyped;
    a.dirtyPages = (const uint8_t*)dirtyPagesDev;
    a.pageFlagsOut = (uint8_t*)pageFlagsOutDev;
    a.chunkFlags = (uint8_t*)chunkFlagsDev;
    a.stats = (uint64_t*)statsDev;
    a.updateBase = updateBase;
    if (blocks <= 0) {
        blocks = FB_NUM_SMS * 2;
    }
    return fb::launchSnapshotDiffPush(a, blocks, (cudaStream_t)stream) ==
               cudaSuccess
             ? FB_OK
             : FB_E_CUDA;
}

int fb_dirty_scan(const void* mem,
                  const void* base,
                  uint64_t size,
                  void* pageFlagsDev,
                  void* nDirtyDev,
                  int blocks,
                  void* stream)
{
    OwnerDeviceGuard ownerGuard(mem);
    if (blocks <= 0) {
        blocks = FB_NUM_SMS * 2;
    }
    return fb::launchDirtyScan((const uint8_t*)mem,
                               (const uint8_t*)base,
                               size,
                               (uint8_t*)pageFlagsDev,
                               (uint64_t*)nDirtyDev,
                               blocks,
                               (cudaStream_t)stream) == cudaSuccess
             ? FB_OK
             : FB_E_CUDA;
}

// ---- device-resident state: fused dirty scan + push + mask clear ----
int fb_state_push_dirty(void* mask,
                        const void* src,
                        void* dst,
                        uint64_t size,
                        void* statsDev,
                        int blocks,
                        void* stream)
{
    OwnerDeviceGuard ownerGuard(mask);
    return fb::launchStatePushDirty((uint8_t*)mask,
                                    (const uint8_t*)src,
                                    (uint8_t*)dst,
                                    size,
                                    (uint64_t*)statsDev,
                                    blocks,
                                    (cudaStream_t)stream) == cudaSuccess
             ? FB_OK
             : FB_E_CUDA;
}

int fb_state_flag_range(void* mask, uint64_t offset, uint64_t length, void* stream)
{
    OwnerDeviceGuard ownerGuard(mask);
    if (length == 0) {
        return FB_OK;
    }
    uint64_t b0 = offset / FB_STATE_BLOCK_BYTES;
    uint64_t b1 = (offset + length - 1) / FB_STATE_BLOCK_BYTES;
    return fb::launchStateFlagRange((uint8_t*)mask, b0, b1 - b0 + 1, (cudaStream_t)stream) == cudaSuccess
             ? FB_OK
             : FB_E_CUDA;
}

int fb_state_block_bytes()
{
    return FB_STATE_BLOCK_BYTES;
}

int fb_flags_or(void* dst, const void* src, uint64_t n, void* stream)
{
    OwnerDeviceGuard ownerGuard(dst);
    return fb::launchFlagsOr(
             (uint8_t*)dst, (const uint8_t*)src, n, (cudaStream_t)stream) ==
               cudaSuccess
             ? FB_OK
             : FB_E_CUDA;
}

int fb_chunk_runs(const void* flagsDev,
                  uint64_t nChunks,
                  uint32_t chunkBytes,
                  uint64_t totalBytes,
                  void* outDescsDev,
                  uint32_t maxOut,
                  void* countDev,
                  void* stream)
{
    OwnerDeviceGuard ownerGuard(flagsDev);
    return fb::launchChunkRuns((const uint8_t*)flagsDev,
                               nChunks,
                               chunkBytes,
                               totalBytes,
                               (FbDiffDesc*)outDescsDev,
                               maxOut,
                               (uint32_t*)countDev,
                               (cudaStream_t)stream) == cudaSuccess
             ? FB_OK
             : FB_E_CUDA;
}

int fb_snapshot_apply(void* image,
                      uint64_t imageSize,
                      const void* descsDev,
                      const void* dataOffDev,
                      const void* blobDev,
                      uint32_t nDescs,
                      void* stream)
{
    OwnerDeviceGuard ownerGuard(image);
    return fb::launchSnapshotApply((uint8_t*)image,
                                   imageSize,
                                   (const FbDiffDesc*)descsDev,
                                   (const uint64_t*)dataOffDev,
                                   (const uint8_t*)blobDev,
                                   nDescs,
                                   (cudaStream_t)stream) == cudaSuccess
             ? FB_OK
             : FB_E_CUDA;
}

} // extern "C"

// ---------------------------------------------------------------------------
// Self-test hook for the bootstrap (used by the CPU test-suite): allgather,
// barrier and fd exchange across processes.  Returns 0 on success.
// ---------------------------------------------------------------------------
#include "faabric/device/bootstrap.h"
#include <unistd.h>
extern "C" int fb_test_bootstrap(int rank, int nranks, const char* jobId)
{
    try {
        faabric::device::Bootstrap bs(rank, nranks, jobId, 20000);
        int32_t mine = 100 + rank;
        auto all = bs.allGather(&mine, sizeof(mine));
        for (int r = 0; r < nranks; r++) {
            int32_t v;
            memcpy(&v, all.data() + r * sizeof(v), sizeof(v));
            if (v != 100 + r) {
                return 1;
            }
        }
        bs.barrier();
        // every rank shares a pipe; after the exchange each rank writes its id
        // into every pipe's write end and reads its own pipe
        int pfd[2];
        if (pipe(pfd) != 0) {
            return 2;
        }
        std::vector<int> wr = bs.allGatherFds(pfd[1]);
        for (int r = 0; r < nranks; r++) {
            char c = (char)('a' + rank);
            if (write(wr[r], &c, 1) != 1) {
                return 3;
            }
        }
        bs.barrier();
        int seen = 0;
        for (int r = 0; r < nranks; r++) {
            char c = 0;
            if (read(pfd[0], &c, 1) != 1) {
                return 4;
            }
            seen |= 1 << (c - 'a');
        }
        for (int fd : wr) {
            close(fd);
        }
        int b = bs.broadcastFd(pfd[1], nranks - 1);
        close(b);
        close(pfd[0]);
        close(pfd[1]);
        return seen == (1 << nranks) - 1 ? 0 : 5;
    } catch (const std::exception& e) {
        g_lastError = e.what();
        fprintf(stderr, "bootstrap self-test: %s\n", e.what());
        return 10;
    }
}
