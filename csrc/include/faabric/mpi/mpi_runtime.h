// MPI runtime: messages, worlds, registry, per-thread context, migration.
//
// One header per module: the per-class headers of the reference's layout
// (faabric/mpi/*.h) forward here, so either include style works.
#pragma once

#include <faabric/device/communicator.h>
#include <faabric/mpi/mpi.h>
#include <faabric/proto/faabric.pb.h>
#include <faabric/transport/PointToPointBroker.h>
#include <faabric/transport/tcp/Socket.h>
#include <faabric/util/clock.h>
#include <faabric/util/concurrent_map.h>
#include <faabric/util/hwloc.h>
#include <faabric/util/queue.h>

#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <string>
#include <vector>

// ==========================================================================
// mpi/MpiMessage.h
// ==========================================================================
namespace faabric::mpi {

enum MpiMessageType : int32_t
{
    NORMAL = 0,
    BARRIER_JOIN = 1,
    BARRIER_DONE = 2,
    SCATTER = 3,
    GATHER = 4,
    ALLGATHER = 5,
    REDUCE = 6,
    SCAN = 7,
    ALLREDUCE = 8,
    ALLTOALL = 9,
    ALLTOALL_PACKED = 10,
    SENDRECV = 11,
    BROADCAST = 12,
    // Special message types for async messaging
    UNACKED_MPI_MESSAGE = 13,
    HANDSHAKE = 14,
    // One-sided operations shipped to another worker process at a fence
    RMA_OP = 15,
    RMA_DATA = 16,
};

// POD descriptor travelling through the per-pair queues / sockets (40 bytes,
// reference: include/faabric/mpi/MpiMessage.h:40-53).  `buffer` points at an
// eagerly copied payload: host memory, or device memory when bufferOnDevice.
struct MpiMessage
{
    int32_t id;
    int32_t worldId;
    int32_t sendRank;
    int32_t recvRank;
    int32_t typeSize;
    int32_t count;
    // For async messaging: id of the request this message satisfies
    int32_t requestId;
    MpiMessageType messageType;
    void* buffer;
};
static_assert(sizeof(MpiMessage) == 40, "MpiMessage must stay a 40-byte POD");

inline size_t payloadSize(const MpiMessage& msg)
{
    return (size_t)msg.typeSize * (size_t)msg.count;
}

inline size_t msgSize(const MpiMessage& msg)
{
    return sizeof(MpiMessage) + payloadSize(msg);
}

// Header followed by the payload bytes
void serializeMpiMsg(std::vector<uint8_t>& buffer, const MpiMessage& msg);

// Allocates msg.buffer with malloc (caller frees)
void parseMpiMsg(const std::vector<uint8_t>& bytes, MpiMessage* msg);

}

// ==========================================================================
// mpi/MpiWorld.h
// ==========================================================================
// MpiWorld: an MPI implementation where ranks are threads bound to GPUs.
//
// Host buffers: the reference's algorithms (two-level reduce / broadcast /
// gather through per-pair in-memory queues for local ranks and TCP for ranks
// in other worker processes; src/mpi/MpiWorld.cpp:590-1775).  This path is
// also the "refcpu" baseline of the benchmarks.
//
// Device buffers (CUDA pointers): collectives become ONE fused kernel per rank
// over NVLink peer memory (faabric::device::Communicator: LL / one-shot /
// two-shot / NVLS all-reduce with the user op fused, pull all-gather /
// all-to-all, ...); point-to-point becomes an eager device copy +
// cudaMemcpyPeerAsync on the rank's stream.



// Exec-graph detail keys (reference: include/faabric/mpi/MpiWorld.h:13-18)
// (how many counters a plain send adds to a recording message)
#define NUM_MPI_EXEC_GRAPH_DETAILS 2
#define MPI_MSG_COUNT_PREFIX "mpi-msgcount-torank"
#define MPI_MSGTYPE_COUNT_PREFIX "mpi-msgtype-torank"

#define MPI_MAIN_RANK 0

namespace faabric::mpi {

#ifdef FAABRIC_USE_SPINLOCK
typedef faabric::util::SpinLockQueue<MpiMessage> InMemoryMpiQueue;
#else
typedef faabric::util::FixedCapacityQueue<MpiMessage> InMemoryMpiQueue;
#endif

// ---- user-defined reduction operations (MPI_Op_create) ----
// The reference declares MPI_Op_create and throws; here user functions run on
// the host path (device buffers are staged).  Non-commutative operations are
// folded in rank order at the root.
constexpr int FAABRIC_OP_USER_BASE = 1000;

int registerUserOp(MPI_User_function* fn, bool commutes);

bool unregisterUserOp(int opId);

bool getUserOp(int opId, MPI_User_function** fn, bool* commutes);

// True for user operations created with commute = 0 (rank-ordered fold)
bool isOrderedUserOp(const faabric_op_t* op);

inline bool isUserOp(const faabric_op_t* op)
{
    return op != nullptr && op->id >= FAABRIC_OP_USER_BASE;
}

// ---- derived datatypes (MPI_Type_contiguous) ----
// `count` consecutive elements of a predefined type.  Data movement only needs
// the size; reductions resolve the type back to (base type, count).
constexpr int FAABRIC_DERIVED_TYPE_BASE = 1000;

int registerContiguousType(int baseTypeId, int count);

bool getContiguousType(int typeId, int* baseTypeId, int* count);

bool unregisterContiguousType(int typeId);

// Messages "sent" to remote ranks in mock mode
std::vector<MpiMessage> getMpiMockedMessages(int sendRank);

void clearMpiMockedMessages();

class MpiWorld
{
  public:
    MpiWorld();

    ~MpiWorld();

    void create(faabric::Message& call, int newId, int newSize);

    void initialiseFromMsg(faabric::Message& msg);

    void initialiseRankFromMsg(faabric::Message& msg);

    // Called by every local rank on MPI_Finalize; true when the last rank of an
    // evicted host left and the world can be dropped from the registry
    bool destroy();

    std::string getHostForRank(int rank);

    int getPortForRank(int rank);

    std::string getUser();

    std::string getFunction();

    int getId() const;

    int getSize() const;

    // ---- cartesian topology (2-D periodic) ----
    void getCartesianRank(int rank,
                          int maxDims,
                          const int* dims,
                          int* periods,
                          int* coords);

    // False if no grid has been set up yet
    bool getCartesianDims(int* dims2) const;

    void getRankFromCoords(int* rank, int* coords);

    void shiftCartesianCoords(int rank,
                              int direction,
                              int disp,
                              int* source,
                              int* destination);

    // ---- point to point ----
    void send(int sendRank,
              int recvRank,
              const uint8_t* buffer,
              faabric_datatype_t* dataType,
              int count,
              MpiMessageType messageType = MpiMessageType::NORMAL);

    int isend(int sendRank,
              int recvRank,
              const uint8_t* buffer,
              faabric_datatype_t* dataType,
              int count,
              MpiMessageType messageType = MpiMessageType::NORMAL);

    void recv(int sendRank,
              int recvRank,
              uint8_t* buffer,
              faabric_datatype_t* dataType,
              int count,
              MPI_Status* status,
              MpiMessageType messageType = MpiMessageType::NORMAL);

    int irecv(int sendRank,
              int recvRank,
              uint8_t* buffer,
              faabric_datatype_t* dataType,
              int count,
              MpiMessageType messageType = MpiMessageType::NORMAL);

    void awaitAsyncRequest(int requestId);

    // MPI_Request_free: drops a request-based one-sided operation's request
    // (the operation completes at the next flush or unlock); other kinds of
    // request are kept
    void freeAsyncRequest(int requestId);

    void sendRecv(uint8_t* sendBuffer,
                  int sendCount,
                  faabric_datatype_t* sendDataType,
                  int sendRank,
                  uint8_t* recvBuffer,
                  int recvCount,
                  faabric_datatype_t* recvDataType,
                  int recvRank,
                  int myRank,
                  MPI_Status* status);

    void probe(int sendRank, int recvRank, MPI_Status* status);

    // ---- collectives ----
    void broadcast(int rootRank,
                   int thisRank,
                   uint8_t* buffer,
                   faabric_datatype_t* dataType,
                   int count,
                   MpiMessageType messageType = MpiMessageType::NORMAL);

    void scatter(int sendRank,
                 int recvRank,
                 const uint8_t* sendBuffer,
                 faabric_datatype_t* sendType,
                 int sendCount,
                 uint8_t* recvBuffer,
                 faabric_datatype_t* recvType,
                 int recvCount);

    void gather(int sendRank,
                int recvRank,
                const uint8_t* sendBuffer,
                faabric_datatype_t* sendType,
                int sendCount,
                uint8_t* recvBuffer,
                faabric_datatype_t* recvType,
                int recvCount);

    void allGather(int rank,
                   const uint8_t* sendBuffer,
                   faabric_datatype_t* sendType,
                   int sendCount,
                   uint8_t* recvBuffer,
                   faabric_datatype_t* recvType,
                   int recvCount);

    void reduce(int sendRank,
                int recvRank,
                uint8_t* sendBuffer,
                uint8_t* recvBuffer,
                faabric_datatype_t* datatype,
                int count,
                faabric_op_t* operation);

    void allReduce(int rank,
                   uint8_t* sendBuffer,
                   uint8_t* recvBuffer,
                   faabric_datatype_t* datatype,
                   int count,
                   faabric_op_t* operation);

    // Element-wise resultBuffer = op(inBuffer, resultBuffer) on the host
    // Non-blocking all-reduce (MPI-3 MPI_Iallreduce; not in the reference).
    // On device buffers it is stream-ordered: successive calls pipeline on
    // the communicator's channels, MPI_Wait drains the stream.
    int iAllReduce(int rank,
                   uint8_t* sendBuffer,
                   uint8_t* recvBuffer,
                   faabric_datatype_t* datatype,
                   int count,
                   faabric_op_t* operation);

    // MPI_Ireduce_scatter_block and MPI_Iallgather, built like iAllReduce: a
    // burst on symmetric, 16-byte aligned device buffers whose shards are
    // multiples of 16 bytes is deferred and issued as ONE grouped launch at
    // the next wait (FAABRIC_MPI_GROUP_IALLREDUCE=0 turns that off); other
    // device buffers run one stream-ordered device call at issue; host
    // buffers, and an in-place reduce-scatter (send == recv), complete at
    // issue.
    int iReduceScatter(int rank,
                       uint8_t* sendBuffer,
                       uint8_t* recvBuffer,
                       faabric_datatype_t* datatype,
                       int recvCount,
                       faabric_op_t* operation);

    int iAllGather(int rank,
                   const uint8_t* sendBuffer,
                   faabric_datatype_t* sendType,
                   int sendCount,
                   uint8_t* recvBuffer,
                   faabric_datatype_t* recvType,
                   int recvCount);

    // Symmetric-heap allocation for MPI_Alloc_mem (collective: every rank
    // must allocate the same sizes in the same order)
    void* deviceAlloc(int rank, size_t bytes);

    bool deviceFree(int rank, void* ptr);

    void op_reduce(faabric_op_t* operation,
                   faabric_datatype_t* datatype,
                   int count,
                   uint8_t* inBuffer,
                   uint8_t* resultBuffer);

    void scan(int rank,
              uint8_t* sendBuffer,
              uint8_t* recvBuffer,
              faabric_datatype_t* datatype,
              int count,
              faabric_op_t* operation);

    void allToAll(int rank,
                  uint8_t* sendBuffer,
                  faabric_datatype_t* sendType,
                  int sendCount,
                  uint8_t* recvBuffer,
                  faabric_datatype_t* recvType,
                  int recvCount);

    // recvCount elements per rank end up on each rank (MPI_Reduce_scatter with
    // equal counts); not implemented by the reference
    void reduceScatter(int rank,
                       uint8_t* sendBuffer,
                       uint8_t* recvBuffer,
                       faabric_datatype_t* datatype,
                       int recvCount,
                       faabric_op_t* operation);

    void barrier(int thisRank);

    // ---- one-sided communication (MPI_Win_*, MPI_Put / MPI_Get) ----
    // The reference declares these and throws (mpi_native.cpp:649-683).  Here
    // a target in this process is written / read directly (host memory, or
    // device memory through peer access), a target in another worker process
    // has its operations shipped and applied at the closing fence.
    // Collective; every rank gets the same window id
    int winCreate(int rank, void* base, int64_t sizeBytes, int dispUnit);

    // Collective
    void winFree(int rank, int winId);

    // Collective: completes every operation of the epoch at origin and target
    void winFence(int rank, int winId);

    void winPut(int rank, int winId, const uint8_t* origin, size_t bytes, int targetRank, int64_t targetDisp);

    void winGet(int rank, int winId, uint8_t* origin, size_t bytes, int targetRank, int64_t targetDisp);

    // One-sided atomics (MPI_Accumulate family): `count` elements of a
    // predefined `datatype`, target[i] = op(target[i], origin[i]), each element
    // atomically.  `result` (null: no fetch) receives the previous values; it
    // is defined after the closing fence.  Every argument is checked before
    // anything is applied; returns MPI_SUCCESS or an MPI error code.
    //   host segment in this process       the host atomics, on this thread
    //   symmetric heap in this process     Communicator::accumulate, on the
    //                                      origin rank's stream
    //   other device memory in this process  the pointer kernel on a GPU that
    //                                      can address the segment
    //   rank in another worker process     shipped and applied at the fence
    int winAccumulate(int rank,
                      int winId,
                      const uint8_t* origin,
                      size_t count,
                      faabric_datatype_t* datatype,
                      faabric_op_t* op,
                      uint8_t* result,
                      int targetRank,
                      int64_t targetDisp);

    // One integer element: *result = target; if (target == *compare) target = *origin
    int winCompareSwap(int rank,
                       int winId,
                       const uint8_t* origin,
                       const uint8_t* compare,
                       uint8_t* result,
                       faabric_datatype_t* datatype,
                       int targetRank,
                       int64_t targetDisp);

    // ---- passive-target synchronisation (MPI_Win_lock and friends) ----
    // Locks are reader/writer locks per target segment, held in the target's
    // process and granted in arrival order; a wait is bounded by the world's
    // message timeout (MPI_ERR_OTHER).  Inside a lock epoch every operation
    // takes its usual path; those for a rank in another worker process are
    // shipped at the next flush / unlock of that rank instead of a fence.
    // Every call returns MPI_SUCCESS or an MPI error code; MPI_ERR_RMA_SYNC
    // calls change nothing.
    int winLock(int rank, int winId, int lockType, int targetRank, int assert);

    int winUnlock(int rank, int winId, int targetRank);

    int winLockAll(int rank, int winId, int assert);

    int winUnlockAll(int rank, int winId);

    // Completes every operation of `rank` to `targetRank` (-1: every locked
    // target) at origin and target
    int winFlush(int rank, int winId, int targetRank);

    // True while `rank` holds a lock (or lock-all) epoch on the window
    bool winInPassiveEpoch(int rank, int winId);

    // ---- request-based operations (MPI_Rput, MPI_Rget, MPI_Raccumulate,
    // MPI_Rget_accumulate).  Every check runs before anything is issued:
    // MPI_ERR_WIN (unknown window), MPI_ERR_RANK, MPI_ERR_ARG (a range
    // outside the target window, or the checks of winAccumulate) and
    // MPI_ERR_RMA_SYNC (the target is not covered by a passive epoch of
    // `rank`).  On success *requestId is a request of this rank thread,
    // completed by awaitAsyncRequest.
    //   symmetric heap in this process, origin on the origin's GPU (or in
    //   its heap): deferred into the origin's batch for the window, issued
    //   as one Communicator::putGetMany at the wait, flush or unlock (or
    //   when the batch holds a launch's worth)
    //   other segments in this process: winPut / winGet at issue
    //   rank in another worker process: queued like MPI_Put, shipped at the
    //   flush or unlock of the target, or at the wait
    int winRputGet(int rank, int winId, uint8_t* origin, size_t bytes, int targetRank, int64_t targetDisp, bool get, int* requestId);
    int winRaccumulate(int rank,
                       int winId,
                       const uint8_t* origin,
                       size_t count,
                       faabric_datatype_t* datatype,
                       faabric_op_t* op,
                       uint8_t* result,
                       int targetRank,
                       int64_t targetDisp,
                       int* requestId);

    // Completion sequences of one origin's request-based operations on one
    // window, per target: a request numbered at most completed[target] is
    // complete.  Requests hold it, so a wait after the window is freed
    // never touches the window.
    struct RmaProgress
    {
        std::vector<uint64_t> issued;
        std::vector<uint64_t> completed;
    };

    // A passive-target request from another worker process (a PointToPointCall
    // RMA_* code); returns the reply
    static std::string serveRmaRequest(int call, const uint8_t* buffer, size_t bytes);

    // The grant of a lock this process queued for in another one
    static void serveRmaGrant(const uint8_t* buffer, size_t bytes);

    // Window segment of `rank`; false if the window is unknown
    bool winQuery(int winId, int rank, void** base, int64_t* sizeBytes, int* dispUnit);

    // True if every rank of the world lives in this process
    bool allRanksLocal();

    // ---- introspection / tests ----
    std::shared_ptr<InMemoryMpiQueue> getLocalQueue(int sendRank, int recvRank);

    long getLocalQueueSize(int sendRank, int recvRank);

    void overrideHost(const std::string& newHost);

    double getWTime();

    // ---- migration ----
    void prepareMigration(int newGroupId, int thisRank, bool thisRankMustMigrate);

    // ---- device path ----
    // Communicator of a local rank (creates the per-world group on first use);
    // nullptr if the device path is not available for this world
    std::shared_ptr<faabric::device::Communicator> getDeviceComm(int rank);

    // True if the pointer is CUDA device memory
    static bool isDevicePointer(const void* p);

    // Statistics of the device path (collectives that ran as fused kernels)
    uint64_t getDeviceCollectiveCount() const { return deviceCollectives.load(); }

    // ---- device branch of each collective ----
    // One branch per collective, shared by MPI_COMM_WORLD and the
    // sub-communicators.  `comm` is this rank's device communicator (the
    // world's, or a sub-communicator child of it; null: no device path),
    // `rank` the caller's WORLD rank (it picks the stream), `root` a rank of
    // `comm`.  The caller has checked that the buffers are device memory.
    // True when the collective ran as a fused kernel; false when `comm` does
    // not support it (FB_E_UNSUPPORTED, FB_E_TOO_LARGE): take the host path.
    using DeviceComm = std::shared_ptr<faabric::device::Communicator>;
    // The (datatype, op) pair has a device reduction
    static bool deviceReducible(faabric_datatype_t* dt, faabric_op_t* op);
    bool deviceBroadcast(const DeviceComm& comm, int rank, int root, uint8_t* buffer, size_t bytes);
    bool deviceReduce(const DeviceComm& comm, int rank, int root, const uint8_t* send, uint8_t* recv,
                      faabric_datatype_t* dt, int count, faabric_op_t* op);
    bool deviceAllReduce(const DeviceComm& comm, int rank, const uint8_t* send, uint8_t* recv,
                         faabric_datatype_t* dt, int count, faabric_op_t* op);
    // false for an in-place scan (send == recv)
    bool deviceScan(const DeviceComm& comm, int rank, const uint8_t* send, uint8_t* recv,
                    faabric_datatype_t* dt, int count, faabric_op_t* op);
    // send == nullptr at the root: its chunk already sits in its slot of recv
    bool deviceGather(const DeviceComm& comm, int rank, int root, const uint8_t* send, uint8_t* recv, size_t bytes);
    // recv == nullptr at the root: its chunk stays where it is in send
    bool deviceScatter(const DeviceComm& comm, int rank, int root, const uint8_t* send, uint8_t* recv, size_t bytes);
    // false for an in-place all-gather (send is this rank's slot of recv)
    bool deviceAllGather(const DeviceComm& comm, int rank, const uint8_t* send, uint8_t* recv, size_t bytes);
    bool deviceAllToAll(const DeviceComm& comm, int rank, const uint8_t* send, uint8_t* recv, size_t chunk);

  private:
    int id = -1;
    int size = -1;
    std::string thisHost;
    std::string basePort;
    faabric::util::TimePoint creationTime;

    // Grid declared by the last MPI_Cart_create (rows, cols)
    std::atomic<int> cartDims[2]{ 0, 0 };

    std::atomic<int> activeLocalRanks = 0;
    std::atomic<bool> hasBeenMigrated = false;

    std::string user;
    std::string function;

    faabric::transport::PointToPointBroker& broker;

    // ---- rank / host layout ----
    std::mutex worldMx;
    int groupId = -1;
    std::vector<std::string> hostForRank;
    // As scheduled (may be a per-GPU alias of this host)
    std::vector<std::string> virtualHostForRank;
    std::vector<int> portForRank;
    std::map<std::string, std::set<int>> ranksForHost;
    // lowest rank on each host acts as its leader in two-level collectives
    std::map<std::string, int> leaderForHost;
    void initLocalRemoteLeaders();
    bool isLocalRank(int rank) { return hostForRank.at(rank) == thisHost; }
    int getLocalLeader() { return leaderForHost.at(thisHost); }

    // ---- one-sided windows ----
    enum RmaKind : int
    {
        RMA_PUT = 0,
        RMA_GET = 1,
        RMA_ACCUMULATE = 2,
        RMA_GET_ACCUMULATE = 3,
        RMA_COMPARE_SWAP = 4,
    };
    struct RmaOp
    {
        int kind; // RmaKind
        int target;
        uint64_t dispBytes;
        uint64_t bytes;
        uint8_t* origin; // put / get: the user's buffer
        // atomics: FbDtype / FbOp, a host copy of the origin (and compare)
        // values, and where the fetched values go (or null)
        int dtype = -1;
        int op = -1;
        std::vector<uint8_t> data;
        uint8_t* result = nullptr;
    };
    // A lock request not granted yet: an origin thread of this process waits
    // for `granted`, one in another process gets `onGrant` (a message)
    struct RmaLockWaiter
    {
        uint64_t ticket;
        bool exclusive;
        std::shared_ptr<bool> granted;
        std::function<void()> onGrant;
    };
    // Reader/writer lock of one target segment
    struct RmaLock
    {
        int exclusive = 0;
        int shared = 0;
        std::deque<RmaLockWaiter> waiters;
    };
    // Passive epoch of one origin: the targets it locked (NOCHECK: without
    // taking the lock), or all of them after MPI_Win_lock_all
    struct RmaEpoch
    {
        struct Target
        {
            bool exclusive;
            bool nocheck;
        };
        bool all = false;
        std::map<int, Target> locked;
        // puts / gets of this epoch went through cudaMemcpy
        bool deviceCopies = false;
    };
    struct RmaWindow
    {
        std::mutex mx;
        bool filled = false;
        int freed = 0;
        std::vector<uint64_t> bases;
        std::vector<int64_t> sizes;
        std::vector<int32_t> dispUnits;
        // operations queued for other processes, one list per ORIGIN rank
        // (only that rank's thread touches its list)
        std::vector<std::vector<RmaOp>> pending;
        // (device, stream) pairs each rank launched atomics on this epoch,
        // waited for by its fence (only that rank's thread touches its list)
        std::vector<std::vector<std::pair<int, void*>>> streams;
        // passive epochs, one per ORIGIN rank (only that rank's thread)
        std::vector<RmaEpoch> epochs;
        // lock of each target segment in this process, under lockMx
        std::mutex lockMx;
        std::condition_variable lockCv;
        std::vector<RmaLock> locks;
        // request-based operations, one entry per ORIGIN rank (only that
        // rank's thread): deferred heap copies, and completion sequences
        std::vector<std::vector<faabric::device::Communicator::RmaCopy>> batches;
        std::vector<std::shared_ptr<RmaProgress>> progress;
    };
    std::mutex windowsMx;
    std::map<int, std::shared_ptr<RmaWindow>> windows;
    // windows created so far by each rank (collective order => same ids)
    std::vector<int> windowsCreated;
    std::shared_ptr<RmaWindow> getWindow(int winId);
    // nullptr if the window is unknown (or freed)
    std::shared_ptr<RmaWindow> findWindow(int winId);
    uint8_t* winTargetPtr(RmaWindow& w, int targetRank, int64_t targetDisp, size_t bytes);
    void rmaSendOps(RmaWindow& w, int rank, int peer);
    void rmaRecvOps(RmaWindow& w, int rank, int peer, int nOps);
    // Payload bytes of a shipped atomic on `target`; throws if it is malformed
    static size_t rmaAtomicPayload(int kind, int dtype, int op, uint64_t bytes, const uint8_t* target);
    // One atomic operation of `rank` on a segment in this process (the paths
    // of winAccumulate); `compare` non-null means compare-and-swap.  Device
    // streams that still run it are added to `used`.  `serverPath`: applied
    // for another process outside any rank thread, on streams of its own.
    void rmaApplyLocal(RmaWindow& w,
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
                       bool serverPath = false);
    // Waits for the device streams `rank` used on the window
    void rmaWaitStreams(RmaWindow& w, int rank);
    // Takes the lock of a target segment for `rank` (waits for the grant)
    int rmaAcquire(RmaWindow& w, int winId, int rank, int targetRank, bool exclusive);
    // Completes `rank`'s operations to `targetRank`; `release` also unlocks
    int rmaComplete(RmaWindow& w, int winId, int rank, int targetRank, bool release);
    // Issues `rank`'s deferred heap copies on the window (its stream joins
    // the window's streams of `rank`)
    void rmaIssueBatch(RmaWindow& w, int rank);
    // Checks and numbering shared by the request-based calls: MPI_SUCCESS
    // and the target address, or an MPI error code
    int rmaRequestTarget(RmaWindow& w, int rank, int targetRank, int64_t targetDisp, size_t bytes, uint8_t** target);
    // A request of this rank thread for the next operation of `rank` to
    // `targetRank` (numbered in `progress`; null: it completed at issue)
    int addRmaRequest(int rank, int winId, int targetRank, std::shared_ptr<RmaProgress> progress);
    // The wait of a request-based operation whose sequence is not complete:
    // the batch and streams of `rank` (target in this process), or the flush
    // of the target (another process)
    void rmaAwait(int rank, int winId, int targetRank);
    // Handles a request of serveRmaRequest on this world
    std::string rmaServe(int call, const uint8_t* buffer, size_t bytes);
    // Communicator of a rank if one is wired already (never creates one)
    std::shared_ptr<faabric::device::Communicator> wiredDeviceComm(int rank);
    // Stream of `rank` on `device` for one-sided atomics
    void* rmaStream(int rank, int device);
    std::map<std::pair<int, int>, void*> rmaStreams;

    // ---- local queues (size x size, lazily created) ----
    std::vector<std::shared_ptr<InMemoryMpiQueue>> localQueues;
    void initLocalQueues();
    int getIndexForRanks(int sendRank, int recvRank) const;

    // ---- remote (other worker process) sockets: per-thread ----
    void initSendRecvSockets(int thisRank);
    void sendRemoteMpiMessage(const std::string& dstHost, int sendRank, int recvRank, const MpiMessage& msg);
    MpiMessage recvRemoteMpiMessage(int sendRank, int recvRank);

    // ---- async requests: per-thread ----
    MpiMessage internalRecv(int sendRank, int recvRank);
    void doRecv(MpiMessage& msg,
                uint8_t* buffer,
                faabric_datatype_t* dataType,
                int count,
                MPI_Status* status,
                MpiMessageType messageType);
    void drainPendingFor(int sendRank, int recvRank, int untilRequestId);

    void checkRanksRange(int sendRank, int recvRank);

    void recordExecGraph(int recvRank, MpiMessageType type);

    // ---- device path ----
    std::mutex deviceMx;
    bool deviceTried = false;
    std::vector<std::shared_ptr<faabric::device::Communicator>> deviceComms;
    std::vector<void*> deviceStreams; // cudaStream_t per rank
    std::atomic<uint64_t> deviceCollectives = 0;
    // Channel streams MPI_Iallreduce may rotate over (see ensureDeviceComms)
    std::atomic<int> nonBlockingChannels = 1;
    // MPI_Iallreduce (and MPI_Ireduce_scatter_block / MPI_Iallgather) bursts
    // on symmetric device buffers are coalesced into one grouped kernel at the
    // next wait (FAABRIC_MPI_GROUP_IALLREDUCE=0: one kernel per call, the
    // round-1 behaviour)
    bool groupIallreduce = true;
    // FAABRIC_ALLREDUCE_ALGO (FbAlgo; AUTO = measured table / thresholds)
    int forcedAllReduceAlgo = 0;
    void ensureDeviceComms();
    // Looks up this rank thread's communicator and first stream once
    void cacheDeviceComm(int rank);

    // Host buffers, all ranks in this process: the ranks reduce straight out
    // of each other's buffers (slice-parallel reduce-scatter + all-gather in
    // shared memory, three barriers) instead of funnelling malloc'ed copies
    // through rank 0.  FAABRIC_MPI_HOST_ALLREDUCE=reference keeps the
    // reference's reduce + broadcast (used as the `refcpu` baseline).
    struct HostCollective
    {
        int nRanks = 0;
        std::atomic<int> arrived{ 0 };
        // 32 bits: waiters park on it with futex(2)
        std::atomic<uint32_t> generation{ 0 };
        std::atomic<int> sleepers{ 0 };
        // microseconds a waiter polls before it parks
        int spinIterations = 0;
        // smallest payload worth two barriers (copy collectives; all-reduce
        // pays off from 32 KiB everywhere)
        size_t minCopyBytes = 32 * 1024;
        std::vector<const uint8_t*> sendPtrs;
        std::vector<uint8_t*> recvPtrs;

        void barrier(int timeoutMs);
    };
    std::unique_ptr<HostCollective> hostCollective;
    // Rank-ordered fold at the root for non-commutative user operations
    void orderedReduce(int sendRank, int recvRank, uint8_t* sendBuffer, uint8_t* recvBuffer, faabric_datatype_t* datatype, int count, faabric_op_t* operation);
    bool sharedMemoryEligible(size_t bytes) const { return hostCollective != nullptr && bytes >= hostCollective->minCopyBytes; }
    void sharedBroadcast(int root, int rank, uint8_t* buffer, size_t bytes);
    void sharedAllGather(int rank, const uint8_t* sendBuffer, uint8_t* recvBuffer, size_t sendBytes);
    void sharedAllToAll(int rank, const uint8_t* sendBuffer, uint8_t* recvBuffer, size_t chunkBytes);
    void sharedGather(int rank, int root, const uint8_t* sendBuffer, uint8_t* recvBuffer, size_t sendBytes, bool rootInPlace);
    void sharedScatter(int rank, int root, const uint8_t* sendBuffer, uint8_t* recvBuffer, size_t chunkBytes);
    void sharedReduce(int rank, int root, uint8_t* sendBuffer, uint8_t* recvBuffer, faabric_datatype_t* datatype, int count, faabric_op_t* operation);
    bool trySharedMemoryAllReduce(int rank,
                                  uint8_t* sendBuffer,
                                  uint8_t* recvBuffer,
                                  faabric_datatype_t* datatype,
                                  int count,
                                  faabric_op_t* operation);

    // Eager device sends park their payload in the SENDER's symmetric heap;
    // the receiver pulls it over NVLink through its mapping of that heap and
    // hands the block back.  One arena per rank, carved out at wiring time.
    struct StagingArena
    {
        std::mutex mx;
        uint64_t base = 0;
        uint64_t size = 0;
        std::map<uint64_t, uint64_t> freeBlocks; // offset -> size
        std::map<uint64_t, uint64_t> usedBlocks;
    };
    std::vector<std::unique_ptr<StagingArena>> stagingArenas;
    uint8_t* stageAlloc(int rank, size_t bytes);
    void stageFree(int ownerRank, const void* ownerPtr);
    const uint8_t* peerViewOfStaged(int ownerRank, int viewerRank, const void* ownerPtr);
    void* streamForRank(int rank, int channel = 0);
};

// FbDtype / FbOp for an MPI datatype / op (-1 if there is no device mapping)
int fbDtypeFor(faabric_datatype_t* datatype);

int fbOpFor(faabric_op_t* op);

}

// ==========================================================================
// mpi/MpiContext.h
// ==========================================================================
namespace faabric::mpi {

// Per-thread (= per-rank) MPI state used by the C shim
class MpiContext
{
  public:
    MpiContext();

    int createWorld(faabric::Message& msg);

    void joinWorld(faabric::Message& msg);

    bool getIsMpi() const;

    int getRank() const;

    int getWorldId() const;

  private:
    bool isMpi;
    int rank;
    int worldId;
};

}

// ==========================================================================
// mpi/MpiWorldRegistry.h
// ==========================================================================
namespace faabric::mpi {

class MpiWorldRegistry
{
  public:
    MpiWorldRegistry() = default;

    MpiWorld& createWorld(faabric::Message& msg, int worldId, std::string hostOverride = "");

    MpiWorld& getOrInitialiseWorld(faabric::Message& msg);

    MpiWorld& getWorld(int worldId);

    // nullptr if the world does not exist (any more); keeps it alive
    std::shared_ptr<MpiWorld> findWorld(int worldId);

    bool worldExists(int worldId);

    void clearWorld(int worldId);

    void clear();

  private:
    faabric::util::ConcurrentMap<int, std::shared_ptr<MpiWorld>> worldMap;
};

MpiWorldRegistry& getMpiWorldRegistry();

}

// ==========================================================================
// mpi/migration.h
// ==========================================================================
namespace faabric::mpi {

// Migration point for long-running (MPI or plain) functions: call it at a
// point where no messages are in flight (typically right after a barrier).
//
// Asks the planner - through group idx 0 - whether the app should be
// re-distributed.  If this function must move, its memory is snapshotted and
// pushed to the destination, a MIGRATION request is dispatched there with
// `entrypointArg` as input data (the function resumes from it) and
// FunctionMigratedException unwinds this execution.  If the policy says the
// app must be FROZEN (spot eviction without spare capacity), the snapshot goes
// to the planner and FunctionFrozenException is thrown; the app thaws when
// capacity returns.  Functions that stay put line up with the new group.
//
// (The reference keeps this logic in its distributed tests,
// tests/dist/mpi/mpi_native.cpp:783-913; Faasm has its own copy.)
void mpiMigrationPoint(int entrypointArg);

}

