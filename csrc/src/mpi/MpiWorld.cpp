#include <faabric/batch-scheduler/BatchScheduler.h>
#include <faabric/device/cuda_driver.h>
#include <faabric/mpi/MpiWorld.h>

#include <chrono>
#include <thread>
#include <faabric/planner/PlannerClient.h>
#include <faabric/transport/common.h>
#include <faabric/util/network.h>
#include <faabric/util/batch.h>
#include <faabric/util/config.h>
#include <faabric/util/environment.h>
#include <faabric/util/gids.h>
#include <faabric/util/logging.h>
#include <faabric/util/macros.h>
#include <faabric/util/reduce_ops.h>
#include <faabric/util/testing.h>
#include <faabric/util/timing.h>

#include "buffers.h"

#include <cuda_runtime.h>

#include <cstring>
#include <deque>
#include <functional>
#include <list>
#include <poll.h>
#include <unistd.h>

namespace faabric::mpi {

// ---------------------------------------------------------------------------
// Per-rank (= per-thread) state
// ---------------------------------------------------------------------------
namespace {
// Where a non-blocking collective runs: deferred into this rank thread's
// burst, one device call at issue, or the blocking host path at issue
enum class Route
{
    Grouped,
    Direct,
    Host
};

// A persistent collective (MPI_*_init): the call and its route, fixed at
// init.  `active` from MPI_Start until the wait that completes the start.
struct PersistentColl
{
    Route route;
    faabric::device::Communicator::GroupKind kind;
    std::shared_ptr<faabric::device::Communicator> comm;
    int dtype;
    int op;
    int root;
    faabric::device::Communicator::GroupItem item;
    int rank;
    int commId;
    // Direct: issues the device call and sets the stream it went out on;
    // false when the communicator declines it
    std::function<bool(void**)> direct;
    std::function<void()> host;
    bool active = false;
    bool commFreed = false;
};

// A plan of a burst made only of persistent starts, and its key
struct CachedPlan
{
    faabric::device::Communicator::GroupKind kind;
    const faabric::device::Communicator* comm;
    int dtype;
    int op;
    int root;
    std::vector<int> requests;
    std::shared_ptr<faabric::device::Communicator::GroupPlan> plan;
};

struct AsyncRequest
{
    bool isSend = false;
    int sendRank = -1;
    int recvRank = -1;
    uint8_t* buffer = nullptr;
    faabric_datatype_t* dataType = nullptr;
    int count = 0;
    MpiMessageType messageType = MpiMessageType::NORMAL;
    // Stream-ordered device collective: complete when `stream` drains
    bool isDeviceCollective = false;
    // part of a burst that has not been issued yet (grouped at the next wait)
    bool deferred = false;
    // which grouped launch of this rank thread it went out with (0 = none)
    uint64_t groupSeq = 0;
    void* stream = nullptr;
    std::shared_ptr<faabric::device::Communicator> comm;
    // Request-based one-sided operation (MPI_Rput and friends): complete once
    // rmaProgress->completed[rmaTarget] reaches rmaSeq
    bool isRma = false;
    int rmaWin = -1;
    int rmaTarget = -1;
    uint64_t rmaSeq = 0;
    std::shared_ptr<MpiWorld::RmaProgress> rmaProgress;
    // Persistent collective (started, or inactive when nothing else is set)
    std::shared_ptr<PersistentColl> persistent;
};

struct RankState
{
    int worldId = -1;
    int rank = -1;
    faabric::Message* msg = nullptr;
    std::unique_ptr<faabric::util::FaabricCpuSet> pinnedCpu;

    // Remote peers (other worker processes)
    std::unique_ptr<faabric::transport::tcp::RecvSocket> recvSocket;
    std::vector<int> recvConnForRank;
    std::vector<std::unique_ptr<faabric::transport::tcp::SendSocket>> sendSockets;

    // Async messaging
    int nextRequestId = 1;
    std::map<int, AsyncRequest> requests;
    // sendRank -> request ids of outstanding irecvs, in posting order
    std::map<int, std::deque<int>> pendingIrecvs;
    // sendRank -> messages taken off the wire by a probe, not yet received
    std::map<int, std::deque<MpiMessage>> probed;
    // Non-blocking device collectives rotate over the communicator's
    // channels (every rank issues the same sequence => same channel)
    uint64_t deviceCollectiveSeq = 0;
    // MPI_Iallreduce, MPI_Ireduce_scatter_block, MPI_Iallgather or MPI_Ibcast
    // burst on symmetric device buffers: deferred and issued as ONE grouped
    // kernel at the next wait (or any other device operation).  A burst has
    // one key: (kind, communicator, dtype, op, root); the byte-copy kinds are
    // FB_U8 with op -1, and only a broadcast has a root.  The communicator is
    // the world's or a sub-communicator's child.
    faabric::device::Communicator::GroupKind groupKind = faabric::device::Communicator::GROUP_ALLREDUCE;
    std::shared_ptr<faabric::device::Communicator> groupComm;
    int groupDtype = -1;
    int groupOp = -1;
    int groupRoot = 0;
    void* groupStream = nullptr;
    std::vector<faabric::device::Communicator::GroupItem> groupItems;
    std::vector<int> groupRequests;
    // A burst of a neighbour v kind: its calls (groupItems then holds one
    // placeholder per call) and how its members agree on the launch rounds
    std::vector<MpiWorld::NeighborVCall> groupVCalls;
    MpiWorld::NeighborVAgree groupAgree;
    // every call of the pending burst is a persistent start
    bool groupAllPersistent = false;
    // Plans of such bursts, most recently used first, and plans dropped from
    // the cache.  A dropped plan's device tables are freed with the rank
    // state, at world teardown: a cudaFree waits for the whole device, where
    // a peer sharing it may wait for this rank.
    std::list<CachedPlan> plans;
    std::vector<std::shared_ptr<faabric::device::Communicator::GroupPlan>> retiredPlans;
    // grouped launches go out on one stream, in order: once a request of
    // launch k was waited for, every request of launches <= k is complete
    uint64_t groupLaunchSeq = 0;
    uint64_t groupCompletedSeq = 0;
    void* groupCompletedStream = nullptr;
    // This rank's communicator and first stream, looked up once: the per-call
    // path of a burst must not take world-wide locks (8 rank threads issuing
    // 214 calls each would serialise on them)
    std::shared_ptr<faabric::device::Communicator> cachedComm;
    void* cachedStream0 = nullptr;
    int cachedCommRank = -1;
    bool cachedCommValid = false;
    uint64_t deferredCount = 0;
    std::atomic<uint64_t>* deferredCounter = nullptr;

    void reset()
    {
        worldId = -1;
        rank = -1;
        msg = nullptr;
        pinnedCpu.reset();
        recvSocket.reset();
        recvConnForRank.clear();
        sendSockets.clear();
        requests.clear();
        pendingIrecvs.clear();
        probed.clear();
        deviceCollectiveSeq = 0;
        groupComm = nullptr;
        groupItems.clear();
        groupRequests.clear();
        groupVCalls.clear();
        groupAgree = nullptr;
        groupAllPersistent = false;
        plans.clear();
        retiredPlans.clear();
        cachedComm = nullptr;
        cachedStream0 = nullptr;
        cachedCommRank = -1;
        cachedCommValid = false;
        deferredCount = 0;
        deferredCounter = nullptr;
        nextRequestId = 1;
    }
};

thread_local RankState tls;

std::mutex mockMx;
std::map<int, std::vector<MpiMessage>> mockedMessages;
}

std::vector<MpiMessage> getMpiMockedMessages(int sendRank)
{
    std::lock_guard<std::mutex> lk(mockMx);
    return mockedMessages[sendRank];
}

void clearMpiMockedMessages()
{
    std::lock_guard<std::mutex> lk(mockMx);
    // the captured copies own their payloads
    for (auto& [rank, msgs] : mockedMessages) {
        for (auto& m : msgs) {
            free(m.buffer);
            m.buffer = nullptr;
        }
    }
    mockedMessages.clear();
}

// ---------------------------------------------------------------------------
// Datatype / op mapping for the device path
// ---------------------------------------------------------------------------
int fbDtypeFor(faabric_datatype_t* dt)
{
    switch (dt->id) {
        case FAABRIC_INT8:
        case FAABRIC_CHAR:
            return FB_I8;
        case FAABRIC_UINT8:
        case FAABRIC_BYTE:
        case FAABRIC_C_BOOL:
            return FB_U8;
        case FAABRIC_INT16:
            return FB_I16;
        case FAABRIC_UINT16:
            return FB_U16;
        case FAABRIC_INT32:
        case FAABRIC_INT:
            return FB_I32;
        case FAABRIC_UINT32:
        case FAABRIC_UINT:
            return FB_U32;
        case FAABRIC_INT64:
        case FAABRIC_LONG:
        case FAABRIC_LONG_LONG:
        case FAABRIC_LONG_LONG_INT:
            return FB_I64;
        case FAABRIC_UINT64:
            return FB_U64;
        case FAABRIC_FLOAT:
            return FB_F32;
        case FAABRIC_DOUBLE:
            return FB_F64;
        case FAABRIC_HALF:
            return FB_F16;
        case FAABRIC_BFLOAT16:
            return FB_BF16;
        case FAABRIC_DOUBLE_INT:
            return FB_F64_I32;
        case FAABRIC_FLOAT_INT:
            return FB_F32_I32;
        case FAABRIC_2INT:
            return FB_I32_I32;
        case FAABRIC_LONG_INT:
            return FB_I64_I32;
        default:
            return -1;
    }
}

int fbOpFor(faabric_op_t* op)
{
    switch (op->id) {
        case FAABRIC_OP_MAX:
            return FB_OP_MAX;
        case FAABRIC_OP_MIN:
            return FB_OP_MIN;
        case FAABRIC_OP_SUM:
            return FB_OP_SUM;
        case FAABRIC_OP_PROD:
            return FB_OP_PROD;
        case FAABRIC_OP_LAND:
            return FB_OP_LAND;
        case FAABRIC_OP_LOR:
            return FB_OP_LOR;
        case FAABRIC_OP_BAND:
            return FB_OP_BAND;
        case FAABRIC_OP_BOR:
            return FB_OP_BOR;
        case FAABRIC_OP_MAXLOC:
            return FB_OP_MAXLOC;
        case FAABRIC_OP_MINLOC:
            return FB_OP_MINLOC;
        case FAABRIC_OP_LXOR:
            return FB_OP_LXOR;
        case FAABRIC_OP_BXOR:
            return FB_OP_BXOR;
        case FAABRIC_OP_REPLACE:
            return FB_OP_REPLACE;
        case FAABRIC_OP_NO_OP:
            return FB_OP_NO_OP;
        default:
            return -1;
    }
}

bool MpiWorld::isDevicePointer(const void* p)
{
    if (p == nullptr) {
        return false;
    }
    if (faabric::device::Communicator::isHeapPointer(p)) {
        return true; // symmetric heap of a communicator here: no driver query needed
    }
    if (faabric::device::Communicator::isLoopbackHeapPointer(p)) {
        return true; // loopback backend: heap memory plays the device's role
    }
    if (!faabric::device::cudaAvailable()) {
        return false;
    }
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged;
}

// ---------------------------------------------------------------------------
// Construction / initialisation
// ---------------------------------------------------------------------------
MpiWorld::MpiWorld()
  : thisHost(faabric::transport::getThisHostAddress())
  , creationTime(faabric::util::startTimer())
  , broker(faabric::transport::getPointToPointBroker())
{}

MpiWorld::~MpiWorld()
{
    // Messages nobody received own their payloads
    for (auto& q : localQueues) {
        if (q == nullptr) {
            continue;
        }
        while (q->size() > 0) {
            MpiMessage m{};
            m.buffer = nullptr;
            q->dequeueIfPresent(&m);
            if (m.buffer != nullptr) {
                free(m.buffer);
            }
        }
    }
    for (void* s : deviceStreams) {
        if (s != nullptr) {
            cudaStreamDestroy((cudaStream_t)s);
        }
    }
    for (auto& [key, s] : rmaStreams) {
        cudaStreamDestroy((cudaStream_t)s);
    }
    cudaGetLastError();
}

std::string MpiWorld::getUser()
{
    return user;
}

std::string MpiWorld::getFunction()
{
    return function;
}

int MpiWorld::getId() const
{
    return id;
}

int MpiWorld::getSize() const
{
    return size;
}

void MpiWorld::overrideHost(const std::string& newHost)
{
    thisHost = newHost;
}

double MpiWorld::getWTime()
{
    return faabric::util::getTimeDiffMillis(creationTime) / 1000.0;
}

void MpiWorld::create(faabric::Message& call, int newId, int newSize)
{
    id = newId;
    user = call.user();
    function = call.function();
    size = newSize;
    groupId = call.groupid();

    // Rank 0 spawns the other size-1 ranks through the planner.  The planner
    // already placed the whole world when rank 0 was scheduled (it knew the
    // size from mpiWorldSize) and preloaded that decision, so this request is
    // a scale change consuming it.
    if (size > 1) {
        auto req = faabric::util::batchExecFactory(user, function, size - 1);
        faabric::util::updateBatchExecAppId(req, call.appid());
        for (int i = 0; i < req->messages_size(); i++) {
            faabric::Message& m = *req->mutable_messages(i);
            m.set_appidx(i + 1);
            m.set_ismpi(true);
            m.set_mpiworldid(id);
            m.set_mpirank(i + 1);
            m.set_mpiworldsize(size);
            m.set_groupidx(i + 1);
            m.set_groupsize(size);
            // Children inherit what the function needs to start up
            m.set_cmdline(call.cmdline());
            m.set_inputdata(call.inputdata());
            m.set_ispython(call.ispython());
            m.set_pythonuser(call.pythonuser());
            m.set_pythonfunction(call.pythonfunction());
            m.set_recordexecgraph(call.recordexecgraph());
            if (call.recordexecgraph()) {
                call.add_chainedmsgids(m.id());
            }
        }
        auto decision = faabric::planner::getPlannerClient().callFunctions(req);
        if ((int)decision.appId == NOT_ENOUGH_SLOTS) {
            SPDLOG_ERROR("Not enough slots to create MPI world {} of size {}", id, size);
            throw std::runtime_error("Not enough slots to create MPI world");
        }
        // The group grew (and got a new id): that is the world's group now
        groupId = decision.groupId;
        call.set_groupid(groupId);
        broker.waitForMappingsOnThisHost(groupId);
    } else {
        // A world of one still needs a (trivial) group for its mappings
        faabric::batch_scheduler::SchedulingDecision decision(call.appid(), call.groupid());
        decision.addMessage(thisHost, call.id(), call.appidx(), 0);
        broker.setUpLocalMappingsFromSchedulingDecision(decision);
    }
    initLocalRemoteLeaders();
    initLocalQueues();
}

void MpiWorld::initialiseFromMsg(faabric::Message& msg)
{
    id = msg.mpiworldid();
    user = msg.user();
    function = msg.function();
    size = msg.mpiworldsize();
    groupId = msg.groupid();
    broker.waitForMappingsOnThisHost(groupId);
    initLocalRemoteLeaders();
    initLocalQueues();
}

void MpiWorld::initialiseRankFromMsg(faabric::Message& msg)
{
    int rank = msg.mpirank();
    tls.reset();
    tls.worldId = id;
    tls.rank = rank;
    tls.msg = &msg;
    activeLocalRanks.fetch_add(1);
#ifdef FAABRIC_USE_SPINLOCK
    // Busy-waiting ranks must not share cores
    tls.pinnedCpu = faabric::util::pinThreadNearGpu(pthread_self(), faabric::util::gpuForRank(rank));
#endif
    faabric::util::bindThreadToGpu(faabric::util::gpuForRank(rank));
    initSendRecvSockets(rank);
}

bool MpiWorld::destroy()
{
    SPDLOG_TRACE("Destroying MPI world {} (rank {})", id, tls.rank);
    // Anything still outstanding on this rank is dropped, a deferred burst on
    // MPI_COMM_WORLD included; only a burst on a sub-communicator's child is
    // issued and waited first (below)
    if (!tls.requests.empty()) {
        SPDLOG_WARN("Destroying world {} with {} outstanding async requests on rank {}", id, tls.requests.size(), tls.rank);
    }
    // Device-plane counters of this rank travel with the exec graph (HTTP
    // GET_EXEC_GRAPH): launches, bytes and the algorithm mix
    std::shared_ptr<faabric::device::Communicator> myComm;
    if (tls.msg != nullptr && tls.msg->recordexecgraph()) {
        // (only look, never wire the device plane up just for this)
        std::lock_guard<std::mutex> lk(deviceMx);
        if (tls.rank >= 0 && tls.rank < (int)deviceComms.size()) {
            myComm = deviceComms[tls.rank];
        }
    }
    if (myComm != nullptr) {
        const faabric::device::CommStats& st = myComm->stats();
        auto* details = tls.msg->mutable_intexecgraphdetails();
        (*details)["mpi-device-launches"] = (int)std::min<uint64_t>(st.launches, INT32_MAX);
        (*details)["mpi-device-mbytes"] = (int)std::min<uint64_t>(st.bytes >> 20, INT32_MAX);
        (*details)["mpi-device-staged-copies"] = (int)std::min<uint64_t>(st.stagedCopies, INT32_MAX);
        (*details)["mpi-device-tma-launches"] = (int)std::min<uint64_t>(st.tmaLaunches, INT32_MAX);
        for (int a = 1; a < FB_ALGO_COUNT; a++) {
            if (st.algoCount[a] > 0) {
                (*details)[std::string("mpi-device-algo-") + faabric::device::CommTuning::algoName(a)] =
                  (int)std::min<uint64_t>(st.algoCount[a], INT32_MAX);
            }
        }
    }
    // A burst still deferred on a child is issued and waited, as at
    // MPI_Comm_free: the child is released with the world's sub-communicators
    if (!tls.groupItems.empty() && tls.groupComm != nullptr && tls.groupComm->isSubset()) {
        try {
            settleDeviceBurst(tls.groupComm);
        } catch (const std::exception& e) {
            SPDLOG_ERROR("Rank {}: pending device burst at world teardown failed: {}", tls.rank, e.what());
        }
    }
    tls.reset();
    int left = activeLocalRanks.fetch_sub(1) - 1;
    // Only a host the world has migrated away from clears it eagerly; otherwise
    // the registry keeps it for late joiners of the same world
    return left == 0 && hasBeenMigrated.load();
}

void MpiWorld::initLocalRemoteLeaders()
{
    std::lock_guard<std::mutex> lk(worldMx);
    hostForRank.assign(size, "");
    virtualHostForRank.assign(size, "");
    portForRank.assign(size, 0);
    ranksForHost.clear();
    leaderForHost.clear();
    auto idxs = broker.getIdxsRegisteredForGroup(groupId);
    if ((int)idxs.size() != size) {
        SPDLOG_DEBUG("World {} group {} has {} of {} ranks registered", id, groupId, idxs.size(), size);
    }
    for (int rank : idxs) {
        if (rank < 0 || rank >= size) {
            continue;
        }
        std::string host = broker.getHostForReceiver(groupId, rank);
        // Virtual per-GPU hosts served by this very process are local ranks;
        // the virtual name still picks the rank's GPU
        virtualHostForRank[rank] = host;
        if (host != thisHost && faabric::transport::resolveHostAlias(host) == thisHost) {
            host = thisHost;
        }
        hostForRank[rank] = host;
        portForRank[rank] = broker.getMpiPortForReceiver(groupId, rank);
        ranksForHost[host].insert(rank);
    }
    for (const auto& [host, ranks] : ranksForHost) {
        leaderForHost[host] = *ranks.begin();
    }
    if (leaderForHost.find(thisHost) == leaderForHost.end()) {
        // This host currently holds no rank of the world (can happen right
        // after a migration): keep a harmless entry
        leaderForHost[thisHost] = 0;
    }
}

std::string MpiWorld::getHostForRank(int rank)
{
    std::lock_guard<std::mutex> lk(worldMx);
    if (rank < 0 || rank >= (int)hostForRank.size() || hostForRank[rank].empty()) {
        SPDLOG_ERROR("No host found for rank {} in world {}", rank, id);
        throw std::runtime_error("No host found for rank");
    }
    return hostForRank[rank];
}

int MpiWorld::getPortForRank(int rank)
{
    std::lock_guard<std::mutex> lk(worldMx);
    return portForRank.at(rank);
}

int MpiWorld::getIndexForRanks(int sendRank, int recvRank) const
{
    return sendRank * size + recvRank;
}

void MpiWorld::initLocalQueues()
{
    std::lock_guard<std::mutex> lk(worldMx);
    localQueues.resize((size_t)size * size);
    // Queues whose receiver lives here
    auto it = ranksForHost.find(thisHost);
    if (it == ranksForHost.end()) {
        return;
    }
    for (int recvRank : it->second) {
        for (int sendRank = 0; sendRank < size; sendRank++) {
            auto& q = localQueues[getIndexForRanks(sendRank, recvRank)];
            if (q == nullptr) {
                q = std::make_shared<InMemoryMpiQueue>();
            }
        }
    }
    // Every rank lives here: shared-memory collectives are possible
    hostCollective.reset();
    const char* mode = getenv("FAABRIC_MPI_HOST_ALLREDUCE");
    const bool referenceOnly = mode != nullptr && std::string(mode) == "reference";
    if (!referenceOnly && ranksForHost.size() == 1 && (int)it->second.size() == size && size > 1) {
        hostCollective = std::make_unique<HostCollective>();
        hostCollective->nRanks = size;
        // Polling budget before a waiter parks: generous when ranks (plus the
        // runtime's own threads) fit on the machine, token otherwise
        const bool roomy = (unsigned)size * 2 <= faabric::util::getUsableCores();
        hostCollective->spinIterations = roomy ? 200 : 20;
        // parked waiters make the barriers dearer: measured break-even of the
        // copy collectives moves from ~32 KiB to ~256 KiB
        hostCollective->minCopyBytes = roomy ? 32 * 1024 : 256 * 1024;
        hostCollective->sendPtrs.assign(size, nullptr);
        hostCollective->recvPtrs.assign(size, nullptr);
    }
}

std::shared_ptr<InMemoryMpiQueue> MpiWorld::getLocalQueue(int sendRank, int recvRank)
{
    checkRanksRange(sendRank, recvRank);
    auto& q = localQueues.at(getIndexForRanks(sendRank, recvRank));
    if (q == nullptr) {
        std::lock_guard<std::mutex> lk(worldMx);
        if (q == nullptr) {
            q = std::make_shared<InMemoryMpiQueue>();
        }
    }
    return q;
}

long MpiWorld::getLocalQueueSize(int sendRank, int recvRank)
{
    return getLocalQueue(sendRank, recvRank)->size();
}

void MpiWorld::checkRanksRange(int sendRank, int recvRank)
{
    if (sendRank < 0 || sendRank >= size) {
        SPDLOG_ERROR("Send rank outside range: {} not in [0, {})", sendRank, size);
        throw std::runtime_error("Send rank outside range");
    }
    if (recvRank < 0 || recvRank >= size) {
        SPDLOG_ERROR("Recv rank outside range: {} not in [0, {})", recvRank, size);
        throw std::runtime_error("Recv rank outside range");
    }
}

void MpiWorld::recordExecGraph(int recvRank, MpiMessageType type)
{
    if (tls.msg == nullptr || !tls.msg->recordexecgraph()) {
        return;
    }
    auto* details = tls.msg->mutable_intexecgraphdetails();
    (*details)[std::string(MPI_MSG_COUNT_PREFIX) + "-" + std::to_string(recvRank)] += 1;
    (*details)[std::string(MPI_MSGTYPE_COUNT_PREFIX) + "-" + std::to_string((int)type) + "-" + std::to_string(recvRank)] += 1;
}

// ---------------------------------------------------------------------------
// Remote transport (ranks in other worker processes): raw TCP, lazy all-pairs
// ---------------------------------------------------------------------------
static int tcpPortFor(const std::string& host, int mpiPort)
{
    auto a = faabric::transport::parseHostAddress(host);
    // Worker processes on one box share an IP and differ by port offset, like
    // every other service port
    return mpiPort + a.portOffset;
}

void MpiWorld::initSendRecvSockets(int thisRank)
{
    tls.sendSockets.clear();
    tls.sendSockets.resize(size);
    tls.recvConnForRank.assign(size, -1);
    bool anyRemote = false;
    {
        std::lock_guard<std::mutex> lk(worldMx);
        for (int r = 0; r < size; r++) {
            if (!hostForRank[r].empty() && hostForRank[r] != thisHost) {
                anyRemote = true;
            }
        }
    }
    if (!anyRemote || faabric::util::isMockMode()) {
        return;
    }
    int port = tcpPortFor(thisHost, getPortForRank(thisRank));
    tls.recvSocket = std::make_unique<faabric::transport::tcp::RecvSocket>(port);
    tls.recvSocket->listen();
}

void MpiWorld::sendRemoteMpiMessage(const std::string& dstHost, int sendRank, int recvRank, const MpiMessage& msg)
{
    auto& sock = tls.sendSockets.at(recvRank);
    if (sock == nullptr) {
        auto a = faabric::transport::parseHostAddress(dstHost);
        sock = std::make_unique<faabric::transport::tcp::SendSocket>(a.ip, tcpPortFor(dstHost, getPortForRank(recvRank)));
        sock->dial();
        // Tell the receiver who is on this connection
        MpiMessage hello{};
        hello.worldId = id;
        hello.sendRank = sendRank;
        hello.recvRank = recvRank;
        hello.messageType = MpiMessageType::HANDSHAKE;
        sock->sendOne(BYTES_CONST(&hello), sizeof(MpiMessage));
    }
    sock->sendOne(BYTES_CONST(&msg), sizeof(MpiMessage));
    size_t payload = payloadSize(msg);
    if (payload > 0) {
        sock->sendOne(BYTES_CONST(msg.buffer), payload);
    }
}

MpiMessage MpiWorld::recvRemoteMpiMessage(int sendRank, int recvRank)
{
    if (tls.recvSocket == nullptr) {
        throw std::runtime_error("Remote MPI receive without a listening socket");
    }
    // Accept connections until the one from sendRank has said hello
    while (tls.recvConnForRank.at(sendRank) < 0) {
        int conn = tls.recvSocket->accept(faabric::util::getSystemConfig().globalMessageTimeout);
        MpiMessage hello{};
        tls.recvSocket->recvOne(conn, BYTES(&hello), sizeof(MpiMessage));
        if (hello.messageType != MpiMessageType::HANDSHAKE || hello.sendRank < 0 || hello.sendRank >= size) {
            throw std::runtime_error("Bad MPI handshake");
        }
        tls.recvConnForRank[hello.sendRank] = conn;
    }
    int conn = tls.recvConnForRank[sendRank];
    MpiMessage msg{};
    tls.recvSocket->recvOne(conn, BYTES(&msg), sizeof(MpiMessage));
    size_t payload = payloadSize(msg);
    if (payload > 0) {
        msg.buffer = malloc(payload);
        tls.recvSocket->recvOne(conn, BYTES(msg.buffer), payload);
    } else {
        msg.buffer = nullptr;
    }
    return msg;
}

// ---------------------------------------------------------------------------
// Point to point
// ---------------------------------------------------------------------------
void MpiWorld::send(int sendRank,
                    int recvRank,
                    const uint8_t* buffer,
                    faabric_datatype_t* dataType,
                    int count,
                    MpiMessageType messageType)
{
    checkRanksRange(sendRank, recvRank);
    const std::string otherHost = getHostForRank(recvRank);
    const bool isLocal = otherHost == thisHost;
    const size_t bytes = (size_t)count * dataType->size;

    MpiMessage msg{};
    msg.id = 0;
    msg.worldId = id;
    msg.sendRank = sendRank;
    msg.recvRank = recvRank;
    msg.typeSize = dataType->size;
    msg.count = count;
    msg.requestId = 0;
    msg.messageType = messageType;
    msg.buffer = nullptr;

    const bool onDevice = bytes > 0 && !hostAddressable(buffer);
    if (isLocal && !faabric::util::isMockMode()) {
        // Eager copy so the caller may reuse its buffer as soon as we return
        if (bytes > 0 && onDevice) {
            // Stay on the device when the ranks are wired: park the payload
            // in our symmetric heap, the receiver pulls it over NVLink
            uint8_t* staged = getDeviceComm(sendRank) != nullptr ? stageAlloc(sendRank, bytes) : nullptr;
            if (staged != nullptr) {
                cudaStream_t s = (cudaStream_t)streamForRank(sendRank);
                cudaSetDevice(deviceComms[sendRank]->device());
                if (cudaMemcpyAsync(staged, buffer, bytes, cudaMemcpyDeviceToDevice, s) != cudaSuccess ||
                    cudaStreamSynchronize(s) != cudaSuccess) {
                    cudaGetLastError();
                    stageFree(sendRank, staged);
                    throw std::runtime_error("Device staging for MPI send failed");
                }
                msg.buffer = staged;
            } else {
                // Arena full or no peer wiring: bounce through host memory
                msg.buffer = malloc(bytes);
                if (cudaMemcpy(msg.buffer, buffer, bytes, cudaMemcpyDeviceToHost) != cudaSuccess) {
                    cudaGetLastError();
                    free(msg.buffer);
                    throw std::runtime_error("Device to host copy for MPI send failed");
                }
            }
        } else if (bytes > 0) {
            msg.buffer = malloc(bytes);
            memcpy(msg.buffer, buffer, bytes);
        }
        getLocalQueue(sendRank, recvRank)->enqueue(msg);
    } else {
        // Another worker process: bring device data to the host first
        std::vector<uint8_t> hostCopy;
        if (onDevice) {
            hostCopy.resize(bytes);
            copyBytes(hostCopy.data(), buffer, bytes);
            msg.buffer = hostCopy.data();
        } else {
            msg.buffer = (void*)buffer;
        }
        if (faabric::util::isMockMode()) {
            std::lock_guard<std::mutex> lk(mockMx);
            MpiMessage copy = msg;
            copy.buffer = nullptr;
            if (bytes > 0) {
                copy.buffer = malloc(bytes);
                memcpy(copy.buffer, msg.buffer, bytes);
            }
            mockedMessages[sendRank].push_back(copy);
        } else {
            sendRemoteMpiMessage(otherHost, sendRank, recvRank, msg);
        }
    }
    recordExecGraph(recvRank, messageType);
}

int MpiWorld::isend(int sendRank,
                    int recvRank,
                    const uint8_t* buffer,
                    faabric_datatype_t* dataType,
                    int count,
                    MpiMessageType messageType)
{
    // Sends are eager, so an isend is complete when it returns
    send(sendRank, recvRank, buffer, dataType, count, messageType);
    int requestId = tls.nextRequestId++;
    AsyncRequest r;
    r.isSend = true;
    r.sendRank = sendRank;
    r.recvRank = recvRank;
    tls.requests[requestId] = r;
    return requestId;
}

MpiMessage MpiWorld::internalRecv(int sendRank, int recvRank)
{
    if (auto it = tls.probed.find(sendRank); it != tls.probed.end() && !it->second.empty()) {
        MpiMessage m = it->second.front();
        it->second.pop_front();
        return m;
    }
    if (getHostForRank(sendRank) == thisHost || thisHost == getHostForRank(recvRank)) {
        if (getHostForRank(sendRank) == thisHost) {
            return getLocalQueue(sendRank, recvRank)
              ->dequeue(faabric::util::getSystemConfig().globalMessageTimeout);
        }
    }
    return recvRemoteMpiMessage(sendRank, recvRank);
}

void MpiWorld::doRecv(MpiMessage& msg,
                      uint8_t* buffer,
                      faabric_datatype_t* dataType,
                      int count,
                      MPI_Status* status,
                      MpiMessageType messageType)
{
    if (msg.messageType != messageType) {
        SPDLOG_ERROR("Message types mismatched on {}->{} (expected={}, got={})", msg.sendRank, msg.recvRank, (int)messageType, (int)msg.messageType);
        if (msg.buffer != nullptr) {
            if (isDevicePointer(msg.buffer)) {
                stageFree(msg.sendRank, msg.buffer);
            } else {
                free(msg.buffer);
            }
        }
        throw std::runtime_error("Mismatched MPI message types");
    }
    if (msg.count > count) {
        SPDLOG_ERROR("Message too long for buffer (msg={}, buffer={})", msg.count, count);
        throw std::runtime_error("Message too long");
    }
    const size_t bytes = payloadSize(msg);
    if (bytes > 0 && msg.buffer != nullptr) {
        const bool srcDev = isDevicePointer(msg.buffer);
        const bool dstDev = !hostAddressable(buffer);
        if (srcDev) {
            // Parked in the sender's heap: read it through OUR mapping
            const uint8_t* src = peerViewOfStaged(msg.sendRank, msg.recvRank, msg.buffer);
            cudaStream_t s = (cudaStream_t)streamForRank(msg.recvRank);
            cudaSetDevice(deviceComms[msg.recvRank]->device());
            cudaError_t e = cudaMemcpyAsync(buffer, src, bytes, cudaMemcpyDefault, s);
            if (e == cudaSuccess) {
                e = cudaStreamSynchronize(s);
            }
            stageFree(msg.sendRank, msg.buffer);
            if (e != cudaSuccess) {
                cudaGetLastError();
                throw std::runtime_error(std::string("Peer copy for MPI recv failed: ") + cudaGetErrorString(e));
            }
        } else if (dstDev) {
            cudaError_t e = cudaMemcpy(buffer, msg.buffer, bytes, cudaMemcpyHostToDevice);
            free(msg.buffer);
            if (e != cudaSuccess) {
                cudaGetLastError();
                throw std::runtime_error("Host to device copy for MPI recv failed");
            }
        } else {
            memcpy(buffer, msg.buffer, bytes);
            free(msg.buffer);
        }
        msg.buffer = nullptr;
    }
    if (status != nullptr) {
        status->MPI_SOURCE = msg.sendRank;
        status->MPI_ERROR = MPI_SUCCESS;
        // Tags are not supported
        status->MPI_TAG = -1;
        // The message may be shorter than the buffer
        status->bytesSize = msg.count * dataType->size;
    }
}

void MpiWorld::drainPendingFor(int sendRank, int recvRank, int untilRequestId)
{
    auto& pending = tls.pendingIrecvs[sendRank];
    while (!pending.empty()) {
        int rid = pending.front();
        pending.pop_front();
        auto it = tls.requests.find(rid);
        if (it != tls.requests.end()) {
            AsyncRequest req = it->second;
            MpiMessage m = internalRecv(req.sendRank, req.recvRank);
            doRecv(m, req.buffer, req.dataType, req.count, MPI_STATUS_IGNORE, req.messageType);
            tls.requests.erase(it);
        }
        if (rid == untilRequestId) {
            return;
        }
    }
}

void MpiWorld::recv(int sendRank,
                    int recvRank,
                    uint8_t* buffer,
                    faabric_datatype_t* dataType,
                    int count,
                    MPI_Status* status,
                    MpiMessageType messageType)
{
    checkRanksRange(sendRank, recvRank);
    // Sends are only recorded in mock mode: nothing will ever arrive
    // (reference src/mpi/MpiWorld.cpp:691-696)
    if (faabric::util::isMockMode()) {
        return;
    }
    // Messages of a pair arrive in order: earlier irecvs are satisfied first
    if (!tls.pendingIrecvs[sendRank].empty()) {
        drainPendingFor(sendRank, recvRank, -1);
    }
    MpiMessage m = internalRecv(sendRank, recvRank);
    doRecv(m, buffer, dataType, count, status, messageType);
}

int MpiWorld::irecv(int sendRank,
                    int recvRank,
                    uint8_t* buffer,
                    faabric_datatype_t* dataType,
                    int count,
                    MpiMessageType messageType)
{
    checkRanksRange(sendRank, recvRank);
    int requestId = tls.nextRequestId++;
    AsyncRequest r;
    r.isSend = false;
    r.sendRank = sendRank;
    r.recvRank = recvRank;
    r.buffer = buffer;
    r.dataType = dataType;
    r.count = count;
    r.messageType = messageType;
    tls.requests[requestId] = r;
    tls.pendingIrecvs[sendRank].push_back(requestId);
    return requestId;
}

// Sorts the return code of a device collective: true if it was issued, false
// if the communicator declines it (FB_E_UNSUPPORTED, FB_E_TOO_LARGE: the host
// path takes the call); throws on any other error
static bool deviceIssued(int rc, const char* what = "Device collective")
{
    if (rc == FB_OK) {
        return true;
    }
    if (rc == FB_E_UNSUPPORTED || rc == FB_E_TOO_LARGE) {
        return false;
    }
    throw std::runtime_error(std::string(what) + " failed: " + faabric::device::Communicator::errorString(rc));
}

// Waits for the device collectives issued on `stream`; throws if one failed
static void awaitDevice(faabric::device::Communicator& comm, void* stream)
{
    if (!comm.waitStreamFast((cudaStream_t)stream)) {
        throw std::runtime_error("Device collective failed at synchronisation");
    }
    if (comm.peekError() != 0) {
        throw std::runtime_error("Device collective watchdog fired (peer missing?)");
    }
}

static AsyncRequest collectiveRequest(int rank);

// Plans a rank thread keeps for its bursts of persistent starts
constexpr size_t kPlanCacheSize = 64;

// Moves the cached plans `drop` selects out of the cache
template <typename Drop>
static void retirePlans(Drop&& drop)
{
    for (auto it = tls.plans.begin(); it != tls.plans.end();) {
        if (drop(*it)) {
            tls.retiredPlans.push_back(std::move(it->plan));
            it = tls.plans.erase(it);
        } else {
            ++it;
        }
    }
}

// The pending burst, made only of persistent starts (requests `reqs`), as a
// plan prepared once for its key: (kind, communicator, dtype, op, root, the
// ordered requests).  The cache is this rank's alone, so one rank may hit
// where a peer misses, has evicted the plan or is refused by prepareGroup.
// The barriers still pair up: a plan depends only on its list, which the
// requests fix, and prepareGroup cuts a list into launches exactly as
// groupMany does, so a cached plan, a new one and groupMany issue the same
// launches on every rank.
static int runPersistentBurst(faabric::device::Communicator& comm,
                              const std::vector<faabric::device::Communicator::GroupItem>& items,
                              const std::vector<int>& reqs,
                              cudaStream_t s)
{
    auto it = std::find_if(tls.plans.begin(), tls.plans.end(), [&](const CachedPlan& p) {
        return p.kind == tls.groupKind && p.comm == &comm && p.dtype == tls.groupDtype && p.op == tls.groupOp &&
               p.root == tls.groupRoot && p.requests == reqs;
    });
    if (it != tls.plans.end()) {
        tls.plans.splice(tls.plans.begin(), tls.plans, it);
    } else {
        int rc = FB_OK;
        auto plan = comm.prepareGroup(items.data(), items.size(), tls.groupDtype, &rc, tls.groupKind);
        if (plan == nullptr) {
            return comm.groupMany(
              tls.groupKind, items.data(), items.size(), tls.groupDtype, tls.groupOp, tls.groupRoot, FB_FLAG_SYMMETRIC, s);
        }
        tls.plans.push_front(
          CachedPlan{ tls.groupKind, &comm, tls.groupDtype, tls.groupOp, tls.groupRoot, reqs, std::move(plan) });
        if (tls.plans.size() > kPlanCacheSize) {
            tls.retiredPlans.push_back(std::move(tls.plans.back().plan));
            tls.plans.pop_back();
        }
    }
    const int rc = comm.runGroup(tls.groupKind, *tls.plans.front().plan, tls.groupOp, tls.groupRoot, FB_FLAG_SYMMETRIC, s);
    if (rc == FB_E_UNSUPPORTED) {
        // (a pair with no grouped kernel, refused before any launch:
        // groupMany runs it as per-item calls)
        tls.retiredPlans.push_back(std::move(tls.plans.front().plan));
        tls.plans.pop_front();
        return comm.groupMany(
          tls.groupKind, items.data(), items.size(), tls.groupDtype, tls.groupOp, tls.groupRoot, FB_FLAG_SYMMETRIC, s);
    }
    return rc;
}

static bool neighborVKind(faabric::device::Communicator::GroupKind kind)
{
    return kind == faabric::device::Communicator::GROUP_NEIGHBOR_ALLGATHERV ||
           kind == faabric::device::Communicator::GROUP_NEIGHBOR_ALLTOALLV;
}

// A list of neighbour v calls on `c`: one host agreement on every launch
// window's longest stream, then its launches.  Every member runs it at the
// same program point with the same number of calls, so every member agrees
// on the same number of windows.
static int runNeighborV(faabric::device::Communicator& c,
                        faabric::device::Communicator::GroupKind kind,
                        const std::vector<MpiWorld::NeighborVCall>& calls,
                        const MpiWorld::NeighborVAgree& agree,
                        cudaStream_t s)
{
    std::vector<faabric::device::Communicator::NeighborVItem> items;
    items.reserve(calls.size());
    for (const auto& v : calls) {
        items.push_back({ v.send, v.recv, v.sendCounts.data(), v.sendDispls.data(), v.recvCounts.data(),
                          v.recvDispls.data() });
    }
    std::vector<uint64_t> mine;
    const int rc = c.neighborVStreams(kind, items.data(), items.size(), FB_U8, mine);
    if (rc != FB_OK) {
        return rc;
    }
    std::vector<uint64_t> agreed(mine.size(), 0);
    if (!mine.empty()) {
        agree(mine, agreed);
    }
    return c.groupMany(kind, items.data(), items.size(), FB_U8, agreed, 0, s);
}

// Issues the deferred burst of this rank thread as one grouped launch (every
// rank defers and flushes at the same program points)
static void flushPendingGroup()
{
    using faabric::device::Communicator;
    if (tls.groupItems.empty()) {
        return;
    }
    if (tls.deferredCounter != nullptr && tls.deferredCount > 0) {
        tls.deferredCounter->fetch_add(tls.deferredCount);
        tls.deferredCount = 0;
    }
    auto comm = tls.groupComm;
    auto items = std::move(tls.groupItems);
    auto reqs = std::move(tls.groupRequests);
    auto vCalls = std::move(tls.groupVCalls);
    auto agree = std::move(tls.groupAgree);
    tls.groupItems.clear();
    tls.groupRequests.clear();
    tls.groupVCalls.clear();
    tls.groupAgree = nullptr;
    tls.groupComm = nullptr;
    cudaSetDevice(comm->device());
    const cudaStream_t s = (cudaStream_t)tls.groupStream;
    const int rc = neighborVKind(tls.groupKind)  ? runNeighborV(*comm, tls.groupKind, vCalls, agree, s)
                   : tls.groupAllPersistent      ? runPersistentBurst(*comm, items, reqs, s)
                                                 : comm->groupMany(tls.groupKind, items.data(), items.size(),
                                                                   tls.groupDtype, tls.groupOp, tls.groupRoot,
                                                                   FB_FLAG_SYMMETRIC, s);
    if (rc != FB_OK) {
        const std::string what = std::string("Grouped device ") + Communicator::groupKindName(tls.groupKind);
        // (the burst's requests have no host path left: declining is an error too)
        if (!deviceIssued(rc, what.c_str())) {
            throw std::runtime_error(what + " declined: " + Communicator::errorString(rc));
        }
    }
    const uint64_t seq = ++tls.groupLaunchSeq;
    for (int id : reqs) {
        auto it = tls.requests.find(id);
        if (it != tls.requests.end()) {
            it->second.stream = tls.groupStream;
            it->second.deferred = false;
            it->second.groupSeq = seq;
        }
    }
}

int MpiWorld::addRmaRequest(int rank, int winId, int targetRank, std::shared_ptr<RmaProgress> progress)
{
    int requestId = tls.nextRequestId++;
    AsyncRequest r;
    r.sendRank = rank;
    r.isRma = true;
    r.rmaWin = winId;
    r.rmaTarget = targetRank;
    // (no progress: the operation completed at issue)
    if (progress != nullptr) {
        r.rmaSeq = ++progress->issued[targetRank];
        r.rmaProgress = std::move(progress);
    }
    tls.requests[requestId] = r;
    return requestId;
}

int MpiWorld::freeAsyncRequest(int requestId)
{
    // A request-based one-sided operation completes at the next flush or
    // unlock of its window anyway; the other kinds stay until they are waited
    auto it = tls.requests.find(requestId);
    if (it != tls.requests.end() && it->second.isRma) {
        tls.requests.erase(it);
    } else if (it != tls.requests.end() && it->second.persistent != nullptr) {
        if (it->second.persistent->active) {
            return MPI_ERR_REQUEST;
        }
        tls.requests.erase(it);
        retirePlans([&](const CachedPlan& p) {
            return std::find(p.requests.begin(), p.requests.end(), requestId) != p.requests.end();
        });
    }
    return MPI_SUCCESS;
}

bool MpiWorld::awaitAsyncRequest(int requestId)
{
    auto it = tls.requests.find(requestId);
    if (it == tls.requests.end() || it->second.persistent == nullptr) {
        awaitRequest(requestId);
        return false;
    }
    std::shared_ptr<PersistentColl> p = it->second.persistent;
    if (p->active) {
        // the start completes as the non-blocking call would; the request
        // stays, inactive
        awaitRequest(requestId);
        p->active = false;
        AsyncRequest idle = collectiveRequest(p->rank);
        idle.persistent = std::move(p);
        tls.requests[requestId] = std::move(idle);
    }
    return true;
}

void MpiWorld::awaitRequest(int requestId)
{
    auto it = tls.requests.find(requestId);
    if (it == tls.requests.end()) {
        // Already satisfied while draining for an earlier wait
        return;
    }
    if (it->second.isRma) {
        AsyncRequest req = it->second;
        tls.requests.erase(it);
        // (completed by an earlier wait, flush or unlock: the window may be
        // gone, so nothing else is touched)
        if (req.rmaProgress != nullptr && req.rmaSeq > req.rmaProgress->completed[req.rmaTarget]) {
            rmaAwait(req.sendRank, req.rmaWin, req.rmaTarget);
        }
        return;
    }
    if (it->second.isDeviceCollective) {
        if (it->second.deferred) {
            flushPendingGroup();
            it = tls.requests.find(requestId);
        }
        AsyncRequest req = it->second;
        tls.requests.erase(it);
        if (req.groupSeq != 0 && req.groupSeq <= tls.groupCompletedSeq && req.stream == tls.groupCompletedStream) {
            // an earlier wait already saw this launch complete
            return;
        }
        cudaSetDevice(req.comm->device());
        awaitDevice(*req.comm, req.stream);
        if (req.groupSeq != 0) {
            tls.groupCompletedSeq = req.groupSeq;
            tls.groupCompletedStream = req.stream;
        }
        return;
    }
    if (it->second.isSend) {
        tls.requests.erase(it);
        return;
    }
    drainPendingFor(it->second.sendRank, it->second.recvRank, requestId);
}

void MpiWorld::sendRecv(uint8_t* sendBuffer,
                        int sendCount,
                        faabric_datatype_t* sendDataType,
                        int sendRank,
                        uint8_t* recvBuffer,
                        int recvCount,
                        faabric_datatype_t* recvDataType,
                        int recvRank,
                        int myRank,
                        MPI_Status* status)
{
    // Post the receive first so a ring of sendRecvs cannot deadlock.
    // NB: sendRank is who we send TO, recvRank who we receive FROM
    int recvId = irecv(recvRank, myRank, recvBuffer, recvDataType, recvCount, MpiMessageType::SENDRECV);
    send(myRank, sendRank, sendBuffer, sendDataType, sendCount, MpiMessageType::SENDRECV);
    awaitAsyncRequest(recvId);
    if (status != nullptr) {
        status->MPI_SOURCE = recvRank;
        status->MPI_ERROR = MPI_SUCCESS;
        status->MPI_TAG = -1;
        status->bytesSize = recvCount * recvDataType->size;
    }
}

void MpiWorld::probe(int sendRank, int recvRank, MPI_Status* status)
{
    // (The reference leaves this unimplemented.)  The next message of the
    // pair is taken off the queue / wire and parked until the matching recv.
    checkRanksRange(sendRank, recvRank);
    if (!tls.pendingIrecvs[sendRank].empty()) {
        drainPendingFor(sendRank, recvRank, -1);
    }
    auto& parked = tls.probed[sendRank];
    if (parked.empty()) {
        MpiMessage m = internalRecv(sendRank, recvRank);
        parked.push_back(m);
    }
    const MpiMessage& next = parked.front();
    if (status != nullptr) {
        status->MPI_SOURCE = next.sendRank;
        status->MPI_ERROR = MPI_SUCCESS;
        status->MPI_TAG = -1;
        status->bytesSize = (int)payloadSize(next);
    }
}

// ---------------------------------------------------------------------------
// Device path plumbing
// ---------------------------------------------------------------------------
void* MpiWorld::streamForRank(int rank, int channel)
{
    std::lock_guard<std::mutex> lk(deviceMx);
    const int perRank = FB_MAX_CHANNELS;
    if ((int)deviceStreams.size() < size * perRank) {
        deviceStreams.resize((size_t)size * perRank, nullptr);
    }
    size_t idx = (size_t)rank * perRank + (size_t)(channel % perRank);
    if (rank < (int)deviceComms.size() && deviceComms[rank] != nullptr && deviceComms[rank]->isLoopback()) {
        return nullptr; // loopback: calls complete synchronously
    }
    if (deviceStreams[idx] == nullptr) {
        // Same GPU as the rank's communicator when there is one
        int dev = (rank < (int)deviceComms.size() && deviceComms[rank] != nullptr) ? deviceComms[rank]->device()
                                                                                   : faabric::util::gpuForRank(rank);
        if (dev >= 0) {
            cudaSetDevice(dev);
            cudaStream_t s = nullptr;
            if (cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) == cudaSuccess) {
                deviceStreams[idx] = s;
            } else {
                cudaGetLastError();
            }
        }
    }
    return deviceStreams[idx];
}

void MpiWorld::ensureDeviceComms()
{
    std::lock_guard<std::mutex> lk(deviceMx);
    if (deviceTried) {
        return;
    }
    deviceTried = true;
    const std::string& backend = faabric::util::getSystemConfig().deviceBackend;
    const bool loopback = backend == "loopback";
    if (!loopback && (!faabric::device::cudaAvailable() || backend != "cuda")) {
        return;
    }
    bool allLocal;
    bool allDistinctHosts;
    {
        std::lock_guard<std::mutex> wl(worldMx);
        allLocal = ranksForHost.size() == 1 && ranksForHost.begin()->first == thisHost;
        allDistinctHosts = (int)ranksForHost.size() == size;
    }
    auto cfg = faabric::device::CommConfig::fromEnv();
    cfg.loopback = loopback;
    cfg.heapBytes = (size_t)faabric::util::getSystemConfig().symmHeapBytes;
    if (const char* g = getenv("FAABRIC_MPI_GROUP_IALLREDUCE")) {
        groupIallreduce = g[0] != '0';
    }
    // FAABRIC_ALLREDUCE_ALGO pins the algorithm of every MPI_Allreduce on
    // device buffers (auto | ll | oneshot | twoshot | nvls); FAABRIC_COMM_STREAMS
    // caps the number of channels (streams) a non-coalesced MPI_Iallreduce
    // burst is spread over
    {
        const auto& sysConf = faabric::util::getSystemConfig();
        int forced = faabric::device::CommTuning::algoFromName(sysConf.allreduceAlgo);
        forcedAllReduceAlgo = forced > 0 ? forced : FB_ALGO_AUTO;
        if (forced < 0) {
            SPDLOG_WARN("Ignoring unknown FAABRIC_ALLREDUCE_ALGO={}", sysConf.allreduceAlgo);
        }
        if (getenv("FAABRIC_COMM_CHANNELS") == nullptr && getenv("FAABRIC_COMM_STREAMS") != nullptr) {
            cfg.channels = std::clamp(sysConf.commStreams, 1, FB_MAX_CHANNELS);
        }
    }
    if (getenv("FAABRIC_COMM_CHANNELS") == nullptr && getenv("FAABRIC_COMM_STREAMS") == nullptr) {
        // MPI_Iallreduce bursts pipeline over the channels: use them all
        cfg.channels = FB_MAX_CHANNELS;
    }
    try {
        if (allLocal) {
            std::vector<int> devices(size);
            for (int r = 0; r < size; r++) {
                int fromHost = faabric::util::gpuIndexFromHostName(virtualHostForRank[r]);
                devices[r] = fromHost >= 0 ? fromHost % std::max(1, faabric::device::cudaDeviceCountSafe())
                                           : faabric::util::gpuForRank(r);
            }
            // Ranks that share a GPU also share its hardware work queues
            // (8 by default): keep (ranks on a device) x (channel streams)
            // within that, or kernels of different ranks can queue up behind
            // each other in a cycle while each waits for its peer
            std::map<int, int> ranksOnDevice;
            int maxShare = 1;
            for (int d : devices) {
                maxShare = std::max(maxShare, ++ranksOnDevice[d]);
            }
            // (half the queues, to leave room for streams created elsewhere)
            nonBlockingChannels =
              maxShare == 1 ? std::max(1, cfg.channels) : std::clamp(4 / maxShare, 1, std::max(1, cfg.channels));
            deviceComms = faabric::device::Communicator::createLocal(size, devices, cfg);
            SPDLOG_INFO("MPI world {}: device communicators up ({} ranks, backing {})", id, size, deviceComms[0]->backing());
            // Same allocation on every rank => same offset in every heap
            size_t arenaBytes = std::min<size_t>((size_t)64 << 20, cfg.heapBytes / 4);
            stagingArenas.clear();
            for (int r = 0; r < size; r++) {
                auto arena = std::make_unique<StagingArena>();
                arena->base = deviceComms[r]->alloc(arenaBytes);
                arena->size = arenaBytes;
                arena->freeBlocks[0] = arenaBytes;
                stagingArenas.push_back(std::move(arena));
            }
        } else if (allDistinctHosts && tls.rank >= 0) {
            // One rank per worker process: wire peer memory across processes
            deviceComms.assign(size, nullptr);
            nonBlockingChannels = std::max(1, cfg.channels);
            deviceComms[tls.rank] = faabric::device::Communicator::createIpc(
              tls.rank, size, faabric::util::gpuForRank(tls.rank), "mpiworld-" + std::to_string(id), cfg);
        }
    } catch (const std::exception& e) {
        SPDLOG_WARN("MPI world {}: no device communicators ({})", id, e.what());
        deviceComms.clear();
    }
}

uint8_t* MpiWorld::stageAlloc(int rank, size_t bytes)
{
    if (rank < 0 || rank >= (int)stagingArenas.size() || rank >= (int)deviceComms.size() || deviceComms[rank] == nullptr) {
        return nullptr;
    }
    StagingArena& a = *stagingArenas[rank];
    uint64_t need = (bytes + 255) & ~(uint64_t)255;
    std::lock_guard<std::mutex> lk(a.mx);
    for (auto it = a.freeBlocks.begin(); it != a.freeBlocks.end(); ++it) {
        if (it->second < need) {
            continue;
        }
        uint64_t off = it->first;
        uint64_t rest = it->second - need;
        a.freeBlocks.erase(it);
        if (rest > 0) {
            a.freeBlocks[off + need] = rest;
        }
        a.usedBlocks[off] = need;
        return deviceComms[rank]->heapPtr(a.base + off);
    }
    return nullptr;
}

void MpiWorld::stageFree(int ownerRank, const void* ownerPtr)
{
    StagingArena& a = *stagingArenas.at(ownerRank);
    uint64_t off = deviceComms[ownerRank]->offsetOf(ownerPtr) - a.base;
    std::lock_guard<std::mutex> lk(a.mx);
    auto used = a.usedBlocks.find(off);
    if (used == a.usedBlocks.end()) {
        SPDLOG_ERROR("Freeing unknown staging block of rank {}", ownerRank);
        return;
    }
    uint64_t len = used->second;
    a.usedBlocks.erase(used);
    // Coalesce with the neighbours
    auto next = a.freeBlocks.lower_bound(off);
    if (next != a.freeBlocks.end() && off + len == next->first) {
        len += next->second;
        next = a.freeBlocks.erase(next);
    }
    if (next != a.freeBlocks.begin()) {
        auto prev = std::prev(next);
        if (prev->first + prev->second == off) {
            prev->second += len;
            return;
        }
    }
    a.freeBlocks[off] = len;
}

const uint8_t* MpiWorld::peerViewOfStaged(int ownerRank, int viewerRank, const void* ownerPtr)
{
    uint64_t off = deviceComms[ownerRank]->offsetOf(ownerPtr);
    return deviceComms[viewerRank]->heapPtr(off, ownerRank);
}

std::shared_ptr<faabric::device::Communicator> MpiWorld::getDeviceComm(int rank)
{
    ensureDeviceComms();
    std::lock_guard<std::mutex> lk(deviceMx);
    if (rank < 0 || rank >= (int)deviceComms.size()) {
        return nullptr;
    }
    return deviceComms[rank];
}

// Issues `call(comm, stream)`, a device collective, and counts it in
// `counter`: false if the communicator declines it (the host path takes it)
template<class Call>
static bool issueDevice(faabric::device::Communicator& comm, void* stream, std::atomic<uint64_t>& counter, Call&& call)
{
    // keep the issue order identical on every rank
    flushPendingGroup();
    cudaSetDevice(comm.device());
    if (!deviceIssued(call(comm, (cudaStream_t)stream))) {
        return false;
    }
    counter.fetch_add(1);
    return true;
}

// A blocking device collective: issued, then waited for.  False if there is
// no communicator or it declines the call.
template<class Call>
static bool issueAndWait(const std::shared_ptr<faabric::device::Communicator>& comm,
                         void* stream,
                         std::atomic<uint64_t>& counter,
                         Call&& call)
{
    if (comm == nullptr || !issueDevice(*comm, stream, counter, call)) {
        return false;
    }
    awaitDevice(*comm, stream);
    return true;
}

static int symFlag(faabric::device::Communicator& c, const void* a, size_t bytes)
{
    return c.inHeap(a, bytes) ? FB_FLAG_SYMMETRIC : 0;
}

bool MpiWorld::deviceReducible(faabric_datatype_t* dt, faabric_op_t* op)
{
    const int fdt = fbDtypeFor(dt);
    const int fop = fbOpFor(op);
    return fdt >= 0 && fop >= 0 && faabric::device::Communicator::reduces(fdt, fop);
}

bool MpiWorld::deviceBroadcast(const DeviceComm& comm, int rank, int root, uint8_t* buffer, size_t bytes)
{
    return issueAndWait(comm, streamForRank(rank), deviceCollectives, [&](auto& c, cudaStream_t s) {
        return c.broadcast(buffer, bytes, root, symFlag(c, buffer, bytes), s);
    });
}

bool MpiWorld::deviceReduce(const DeviceComm& comm,
                            int rank,
                            int root,
                            const uint8_t* send,
                            uint8_t* recv,
                            faabric_datatype_t* dt,
                            int count,
                            faabric_op_t* op)
{
    // Inputs are staged, so aliasing the root's input and output is safe and
    // no symmetric offsets are assumed
    const int fdt = fbDtypeFor(dt);
    const int fop = fbOpFor(op);
    if (fdt < 0 || fop < 0) {
        return false;
    }
    return issueAndWait(comm, streamForRank(rank), deviceCollectives, [&](auto& c, cudaStream_t s) {
        return c.reduce(send, recv, (size_t)count, fdt, fop, root, 0, s);
    });
}

bool MpiWorld::deviceAllReduce(const DeviceComm& comm,
                               int rank,
                               const uint8_t* send,
                               uint8_t* recv,
                               faabric_datatype_t* dt,
                               int count,
                               faabric_op_t* op)
{
    const int fdt = fbDtypeFor(dt);
    const int fop = fbOpFor(op);
    if (fdt < 0 || fop < 0) {
        return false;
    }
    // LL and NVLS need the parent's rank set: a forced choice of either means
    // AUTO on a sub-communicator
    int algo = forcedAllReduceAlgo;
    if (comm != nullptr && comm->isSubset() && (algo == FB_ALGO_LL || algo == FB_ALGO_NVLS)) {
        algo = FB_ALGO_AUTO;
    }
    return issueAndWait(comm, streamForRank(rank), deviceCollectives, [&](auto& c, cudaStream_t s) {
        return c.allReduce(send, recv, (size_t)count, fdt, fop, algo, symFlag(c, send, (size_t)count * dt->size), s);
    });
}

bool MpiWorld::deviceScan(const DeviceComm& comm,
                          int rank,
                          const uint8_t* send,
                          uint8_t* recv,
                          faabric_datatype_t* dt,
                          int count,
                          faabric_op_t* op)
{
    const int fdt = fbDtypeFor(dt);
    const int fop = fbOpFor(op);
    if (send == recv || fdt < 0 || fop < 0) {
        return false;
    }
    return issueAndWait(comm, streamForRank(rank), deviceCollectives, [&](auto& c, cudaStream_t s) {
        return c.scan(send, recv, (size_t)count, fdt, fop, symFlag(c, send, (size_t)count * dt->size), s);
    });
}

bool MpiWorld::deviceExscan(const DeviceComm& comm,
                            int rank,
                            const uint8_t* send,
                            uint8_t* recv,
                            faabric_datatype_t* dt,
                            int count,
                            faabric_op_t* op)
{
    const int fdt = fbDtypeFor(dt);
    const int fop = fbOpFor(op);
    if (fdt < 0 || fop < 0) {
        return false;
    }
    const faabric::device::Communicator::GroupItem item{ send, recv, (size_t)count };
    return issueAndWait(comm, streamForRank(rank), deviceCollectives, [&](auto& c, cudaStream_t s) {
        return c.groupMany(faabric::device::Communicator::GROUP_EXSCAN, &item, 1, fdt, fop, 0, 0, s);
    });
}

bool MpiWorld::deviceGather(const DeviceComm& comm, int rank, int root, const uint8_t* send, uint8_t* recv, size_t bytes)
{
    // The device-or-host choice must come out the same on every rank, and only
    // the root knows whether it passed MPI_IN_PLACE: so the root's in-place
    // case takes the device path too (its chunk already sits in the receive
    // buffer), and no rank relies on symmetric offsets - every contribution is
    // staged through the symmetric staging area.
    if (comm != nullptr && send == nullptr) {
        send = recv + (size_t)comm->rank() * bytes;
    }
    return issueAndWait(comm, streamForRank(rank), deviceCollectives, [&](auto& c, cudaStream_t s) {
        return c.gather(send, recv, bytes, root, 0, s);
    });
}

bool MpiWorld::deviceScatter(const DeviceComm& comm, int rank, int root, const uint8_t* send, uint8_t* recv, size_t bytes)
{
    // In place at the root: its chunk is copied onto itself (the source is
    // staged before the kernel reads it)
    if (comm != nullptr && recv == nullptr) {
        recv = const_cast<uint8_t*>(send) + (size_t)comm->rank() * bytes;
    }
    return issueAndWait(comm, streamForRank(rank), deviceCollectives, [&](auto& c, cudaStream_t s) {
        return c.scatter(send, recv, bytes, root, 0, s);
    });
}

bool MpiWorld::deviceAllGather(const DeviceComm& comm, int rank, const uint8_t* send, uint8_t* recv, size_t bytes)
{
    if (comm == nullptr || send == recv + (size_t)comm->rank() * bytes) {
        return false;
    }
    return issueAndWait(comm, streamForRank(rank), deviceCollectives, [&](auto& c, cudaStream_t s) {
        return c.allGather(send, recv, bytes, symFlag(c, send, bytes), s);
    });
}

bool MpiWorld::deviceAllToAll(const DeviceComm& comm, int rank, const uint8_t* send, uint8_t* recv, size_t chunk)
{
    return issueAndWait(comm, streamForRank(rank), deviceCollectives, [&](auto& c, cudaStream_t s) {
        return c.allToAll(send, recv, chunk, symFlag(c, send, chunk * (size_t)c.size()), s);
    });
}

bool MpiWorld::deviceReduceScatter(const DeviceComm& comm,
                                   int rank,
                                   const uint8_t* send,
                                   uint8_t* recv,
                                   faabric_datatype_t* dt,
                                   int recvCount,
                                   faabric_op_t* op)
{
    const int fdt = fbDtypeFor(dt);
    const int fop = fbOpFor(op);
    if (fdt < 0 || fop < 0) {
        return false;
    }
    return issueAndWait(comm, streamForRank(rank), deviceCollectives, [&](auto& c, cudaStream_t s) {
        const size_t shard = (size_t)recvCount * dt->size;
        return c.reduceScatter(send, recv, (size_t)recvCount, fdt, fop, symFlag(c, send, shard * (size_t)c.size()), s);
    });
}

void MpiWorld::cacheDeviceComm(int rank)
{
    if (!tls.cachedCommValid || tls.cachedCommRank != rank) {
        tls.cachedComm = getDeviceComm(rank);
        tls.cachedStream0 = tls.cachedComm != nullptr ? streamForRank(rank, 0) : nullptr;
        tls.cachedCommRank = rank;
        tls.cachedCommValid = true;
    }
}

// Records the request of a non-blocking collective issued (or, deferred, to be
// issued) on `stream` of `comm`: waiting for it drains that stream
static int recordDevice(int requestId, AsyncRequest r, const std::shared_ptr<faabric::device::Communicator>& comm, void* stream)
{
    r.isDeviceCollective = true;
    r.stream = stream;
    r.comm = comm;
    tls.requests[requestId] = std::move(r);
    return requestId;
}

// Adds one call to this rank thread's deferred burst, flushing first a burst
// of another key (or one that is full)
static void deferToGroup(faabric::device::Communicator::GroupKind kind,
                         const std::shared_ptr<faabric::device::Communicator>& comm,
                         int dtype,
                         int op,
                         int root,
                         const faabric::device::Communicator::GroupItem& item,
                         int requestId,
                         AsyncRequest r,
                         std::atomic<uint64_t>& counter)
{
    if (!tls.groupItems.empty() && (tls.groupKind != kind || tls.groupComm != comm || tls.groupDtype != dtype ||
                                    tls.groupOp != op || tls.groupRoot != root || tls.groupItems.size() >= 4096)) {
        flushPendingGroup();
    }
    tls.groupAllPersistent = (tls.groupItems.empty() || tls.groupAllPersistent) && r.persistent != nullptr;
    tls.groupKind = kind;
    tls.groupComm = comm;
    tls.groupDtype = dtype;
    tls.groupOp = op;
    tls.groupRoot = root;
    tls.groupStream = tls.cachedStream0;
    tls.groupItems.push_back(item);
    tls.groupRequests.push_back(requestId);
    tls.deferredCount++; // added to the world's counter at the flush
    tls.deferredCounter = &counter;
    r.deferred = true;
    recordDevice(requestId, std::move(r), comm, tls.groupStream);
}

// The request of a non-blocking collective, complete as it stands (the call
// ran on the host) until recordDevice() makes it a device collective
static AsyncRequest collectiveRequest(int rank)
{
    AsyncRequest r;
    r.isSend = true; // nothing to drain on wait
    r.sendRank = rank;
    r.recvRank = rank;
    return r;
}

// The buffers of a non-blocking collective on `c`: `symmetric` when both
// extents lie in its heap (no driver query), `grouped` when the call may also
// join the deferred burst: grouping on, addresses and shard 16-byte aligned (a
// shard of 0 puts no condition on the length)
struct Placement
{
    bool symmetric;
    bool grouped;
};

static Placement placeCollective(const faabric::device::Communicator& c,
                                 bool grouping,
                                 const void* send,
                                 size_t sendBytes,
                                 const void* recv,
                                 size_t recvBytes,
                                 size_t shardBytes)
{
    const bool symmetric = c.inHeap(send, sendBytes) && c.inHeap(recv, recvBytes);
    return { symmetric, symmetric && grouping && (((uintptr_t)send | (uintptr_t)recv | shardBytes) & 15) == 0 };
}

int MpiWorld::iAllReduce(int rank, uint8_t* send, uint8_t* recv, faabric_datatype_t* dt, int count, faabric_op_t* op,
                         int persistentComm)
{
    checkRanksRange(0, rank);
    cacheDeviceComm(rank);
    return nbAllReduce(tls.cachedComm, rank, send, recv, dt, count, op,
                       [=, this] { allReduce(rank, send, recv, dt, count, op); }, persistentComm);
}

// Records an inactive persistent request of this rank thread
static int addPersistent(PersistentColl p)
{
    const int requestId = tls.nextRequestId++;
    AsyncRequest r = collectiveRequest(p.rank);
    r.persistent = std::make_shared<PersistentColl>(std::move(p));
    tls.requests[requestId] = std::move(r);
    return requestId;
}

int MpiWorld::nbAllReduce(const DeviceComm& comm,
                          int rank,
                          const uint8_t* send,
                          uint8_t* recv,
                          faabric_datatype_t* dt,
                          int count,
                          faabric_op_t* op,
                          const HostPath& host,
                          int persistentComm)
{
    const size_t bytes = (size_t)count * dt->size;
    const int fdt = fbDtypeFor(dt);
    const int fop = fbOpFor(op);
    cacheDeviceComm(rank);
    Route route = Route::Host;
    bool symmetric = false;
    // (a pair the kernels lack must not join a burst: the burst has no host path)
    if (bytes > 0 && deviceReducible(dt, op) && comm != nullptr) {
        const Placement at = placeCollective(*comm, groupIallreduce, send, bytes, recv, bytes, 0);
        symmetric = at.symmetric;
        route = at.grouped ? Route::Grouped : (at.symmetric || isDevicePointer(send)) ? Route::Direct : Route::Host;
    }
    const faabric::device::Communicator::GroupItem item{ send, recv, (size_t)count };
    if (persistentComm != 0) {
        PersistentColl p{ route, faabric::device::Communicator::GROUP_ALLREDUCE, comm, fdt, fop, 0, item, rank,
                          persistentComm };
        p.direct = [=, this](void** s) { return allReduceAtIssue(comm, rank, symmetric, send, recv, count, fdt, fop, s); };
        p.host = host;
        return addPersistent(std::move(p));
    }
    const int requestId = tls.nextRequestId++;
    AsyncRequest r = collectiveRequest(rank);
    if (route == Route::Grouped) {
        // Deferred: the whole burst becomes ONE kernel at the next wait
        deferToGroup(faabric::device::Communicator::GROUP_ALLREDUCE, comm, fdt, fop, 0, item, requestId, std::move(r),
                     deviceCollectives);
        return requestId;
    }
    void* s = nullptr;
    if (route == Route::Direct && allReduceAtIssue(comm, rank, symmetric, send, recv, count, fdt, fop, &s)) {
        return recordDevice(requestId, std::move(r), comm, s);
    }
    // Host path (or unsupported on the device): complete it now
    host();
    tls.requests[requestId] = std::move(r);
    return requestId;
}

bool MpiWorld::allReduceAtIssue(const DeviceComm& comm, int rank, bool symmetric, const uint8_t* send, uint8_t* recv,
                                int count, int fdt, int fop, void** stream)
{
    // Symmetric, 16-byte aligned buffers may use any channel; others (the
    // communicator stages an unaligned heap buffer too) go through the
    // single staging area on channel 0
    const int nChannels = std::clamp(nonBlockingChannels.load(), 1, std::max(1, comm->config().channels));
    const bool anyChannel = symmetric && (((uintptr_t)send | (uintptr_t)recv) & 15) == 0;
    const int channel = anyChannel ? (int)(tls.deviceCollectiveSeq++ % (uint64_t)nChannels) : 0;
    const int flags = (symmetric ? FB_FLAG_SYMMETRIC : 0) | FB_FLAG_CHANNEL(channel);
    *stream = streamForRank(rank, channel);
    return issueDevice(*comm, *stream, deviceCollectives, [&](auto& c, cudaStream_t st) {
        return c.allReduce(send, recv, (size_t)count, fdt, fop, forcedAllReduceAlgo, flags, st);
    });
}

// One call of nbReduceScatter, nbAllGather, nbBroadcast or nbAllToAll: the
// extents of item.send and item.recv and the shard size its placement is
// judged on, its burst key, its burst item, and whether buffers that cannot
// join a burst may run the single device call at issue
struct MpiWorld::NbCall
{
    size_t sendBytes;
    size_t recvBytes;
    size_t shardBytes;
    faabric::device::Communicator::GroupKind kind;
    int dtype;
    int op;
    int root;
    faabric::device::Communicator::GroupItem item;
    bool direct = true;
    // the kind stages every buffer (gather, scatter): device buffers join
    // the burst wherever they live
    bool staged = false;
};

// Symmetric, aligned buffers of a call the device takes (`device`) join this
// rank's burst; other device buffers run `issue` on stream 0; anything else
// runs `host`, which completes the request at issue
template <typename Issue>
int MpiWorld::nbCollective(const DeviceComm& comm, int rank, bool device, const NbCall& call, Issue&& issue,
                           const HostPath& host, int persistentComm)
{
    cacheDeviceComm(rank);
    Route route = Route::Host;
    if (device && comm != nullptr) {
        const Placement at = call.staged ? Placement{ false, groupIallreduce }
                                         : placeCollective(*comm, groupIallreduce, call.item.send, call.sendBytes,
                                                           call.item.recv, call.recvBytes, call.shardBytes);
        if (at.grouped) {
            route = Route::Grouped;
        } else if (call.direct && (call.staged || at.symmetric || isDevicePointer(call.item.send))) {
            route = Route::Direct;
        }
    }
    if (persistentComm != 0) {
        PersistentColl p{ route, call.kind, comm, call.dtype, call.op, call.root, call.item, rank, persistentComm };
        p.direct = [this, comm, issue](void** s) {
            *s = tls.cachedStream0;
            return issueDevice(*comm, *s, deviceCollectives, issue);
        };
        p.host = host;
        return addPersistent(std::move(p));
    }
    const int requestId = tls.nextRequestId++;
    AsyncRequest r = collectiveRequest(rank);
    if (route == Route::Grouped) {
        deferToGroup(call.kind, comm, call.dtype, call.op, call.root, call.item, requestId, std::move(r),
                     deviceCollectives);
        return requestId;
    }
    void* s = tls.cachedStream0;
    if (route == Route::Direct && issueDevice(*comm, s, deviceCollectives, issue)) {
        return recordDevice(requestId, std::move(r), comm, s);
    }
    host();
    tls.requests[requestId] = std::move(r);
    return requestId;
}

int MpiWorld::startCheck(int requestId)
{
    auto it = tls.requests.find(requestId);
    if (it == tls.requests.end() || it->second.persistent == nullptr) {
        return MPI_ERR_REQUEST;
    }
    if (it->second.persistent->commFreed) {
        return MPI_ERR_COMM;
    }
    return it->second.persistent->active ? MPI_ERR_REQUEST : MPI_SUCCESS;
}

int MpiWorld::startPersistent(int requestId)
{
    const int rc = startCheck(requestId);
    if (rc != MPI_SUCCESS) {
        return rc;
    }
    std::shared_ptr<PersistentColl> p = tls.requests[requestId].persistent;
    cacheDeviceComm(p->rank);
    AsyncRequest r = collectiveRequest(p->rank);
    r.persistent = p;
    p->active = true;
    if (p->route == Route::Grouped) {
        deferToGroup(p->kind, p->comm, p->dtype, p->op, p->root, p->item, requestId, std::move(r), deviceCollectives);
        return MPI_SUCCESS;
    }
    void* s = nullptr;
    if (p->route == Route::Direct && p->direct(&s)) {
        recordDevice(requestId, std::move(r), p->comm, s);
        return MPI_SUCCESS;
    }
    p->host();
    tls.requests[requestId] = std::move(r);
    return MPI_SUCCESS;
}

bool MpiWorld::persistentInactive(int requestId)
{
    auto it = tls.requests.find(requestId);
    return it != tls.requests.end() && it->second.persistent != nullptr && !it->second.persistent->active;
}

void MpiWorld::persistentCommFreed(int commId, const DeviceComm& child)
{
    for (auto& [id, r] : tls.requests) {
        if (r.persistent != nullptr && r.persistent->commId == commId) {
            r.persistent->commFreed = true;
            // (what the call holds of the communicator goes with it)
            r.persistent->comm = nullptr;
            r.persistent->direct = nullptr;
            r.persistent->host = nullptr;
        }
    }
    if (child != nullptr) {
        retirePlans([&](const CachedPlan& p) { return p.comm == child.get(); });
    }
}

int MpiWorld::iReduceScatter(int rank,
                             uint8_t* send,
                             uint8_t* recv,
                             faabric_datatype_t* dt,
                             int recvCount,
                             faabric_op_t* op,
                             int persistentComm)
{
    checkRanksRange(0, rank);
    cacheDeviceComm(rank);
    return nbReduceScatter(tls.cachedComm, rank, size, send, recv, dt, recvCount, op, [=, this] {
        reduceScatter(rank, send, recv, dt, recvCount, op);
    }, persistentComm);
}

int MpiWorld::nbReduceScatter(const DeviceComm& comm,
                              int rank,
                              int members,
                              const uint8_t* send,
                              uint8_t* recv,
                              faabric_datatype_t* dt,
                              int recvCount,
                              faabric_op_t* op,
                              const HostPath& host, int persistentComm)
{
    const size_t shard = (size_t)recvCount * dt->size;
    const int fdt = fbDtypeFor(dt);
    const int fop = fbOpFor(op);
    // In place, the output overwrites input the peers are still reading: that
    // case (send == recv) runs the blocking call
    const NbCall call{ shard * members, shard, shard, faabric::device::Communicator::GROUP_REDUCE_SCATTER, fdt, fop, 0,
                       { send, recv, (size_t)recvCount } };
    const bool device = shard > 0 && deviceReducible(dt, op) && send != recv;
    return nbCollective(comm, rank, device, call, [=](auto& c, cudaStream_t st) {
        return c.reduceScatter(send, recv, (size_t)recvCount, fdt, fop, symFlag(c, send, shard * members), st);
    }, host, persistentComm);
}

int MpiWorld::iAllGather(int rank,
                         const uint8_t* send,
                         faabric_datatype_t* sendType,
                         int sendCount,
                         uint8_t* recv,
                         faabric_datatype_t* recvType,
                         int recvCount,
                         int persistentComm)
{
    checkRanksRange(0, rank);
    cacheDeviceComm(rank);
    return nbAllGather(tls.cachedComm, rank, size, send, recv, (size_t)sendCount * sendType->size, [=, this] {
        allGather(rank, send, sendType, sendCount, recv, recvType, recvCount);
    }, persistentComm);
}

int MpiWorld::nbAllGather(const DeviceComm& comm,
                          int rank,
                          int members,
                          const uint8_t* send,
                          uint8_t* recv,
                          size_t bytes,
                          const HostPath& host, int persistentComm)
{
    // a byte copy: the burst's key is the communicator alone.  In place, only
    // the burst runs it on the device.
    NbCall call{ bytes, bytes * members, bytes, faabric::device::Communicator::GROUP_ALLGATHER, FB_U8, -1, 0,
                 { send, recv, bytes } };
    call.direct = comm == nullptr || send != recv + (size_t)comm->rank() * bytes;
    return nbCollective(comm, rank, bytes > 0, call, [=](auto& c, cudaStream_t st) {
        return c.allGather(send, recv, bytes, symFlag(c, send, bytes), st);
    }, host, persistentComm);
}

int MpiWorld::iBroadcast(int rank, int root, uint8_t* buffer, faabric_datatype_t* dt, int count, int persistentComm)
{
    checkRanksRange(0, rank);
    cacheDeviceComm(rank);
    return nbBroadcast(tls.cachedComm, rank, root, buffer, (size_t)count * dt->size, [=, this] {
        broadcast(root, rank, buffer, dt, count, MpiMessageType::BROADCAST);
    }, persistentComm);
}

int MpiWorld::nbBroadcast(const DeviceComm& comm, int rank, int root, uint8_t* buffer, size_t bytes, const HostPath& host, int persistentComm)
{
    // a byte copy: the burst's key is (communicator, root)
    const NbCall call{ bytes, bytes, 0, faabric::device::Communicator::GROUP_BROADCAST, FB_U8, -1, root,
                       { buffer, buffer, bytes } };
    return nbCollective(comm, rank, bytes > 0, call, [=](auto& c, cudaStream_t st) {
        return c.broadcast(buffer, bytes, root, symFlag(c, buffer, bytes), st);
    }, host, persistentComm);
}

int MpiWorld::iAllToAll(int rank,
                        uint8_t* send,
                        faabric_datatype_t* sendType,
                        int sendCount,
                        uint8_t* recv,
                        faabric_datatype_t* recvType,
                        int recvCount,
                        int persistentComm)
{
    checkRanksRange(0, rank);
    cacheDeviceComm(rank);
    return nbAllToAll(tls.cachedComm, rank, size, send, recv, (size_t)sendCount * sendType->size, [=, this] {
        allToAll(rank, send, sendType, sendCount, recv, recvType, recvCount);
    }, persistentComm);
}

int MpiWorld::nbAllToAll(const DeviceComm& comm,
                         int rank,
                         int members,
                         const uint8_t* send,
                         uint8_t* recv,
                         size_t bytes,
                         const HostPath& host, int persistentComm)
{
    // a byte copy: the burst's key is the communicator alone
    const size_t total = bytes * (size_t)members;
    const NbCall call{ total, total, bytes, faabric::device::Communicator::GROUP_ALLTOALL, FB_U8, -1, 0,
                       { send, recv, bytes } };
    return nbCollective(comm, rank, bytes > 0, call, [=](auto& c, cudaStream_t st) {
        return c.allToAll(send, recv, bytes, symFlag(c, send, total), st);
    }, host, persistentComm);
}

int MpiWorld::nbNeighbor(const DeviceComm& comm, int rank, faabric::device::Communicator::GroupKind kind,
                         const uint8_t* send, uint8_t* recv, size_t bytes, const HostPath& host)
{
    // a byte copy through the staging buffers: the burst's key is
    // (kind, communicator)
    NbCall call{ bytes, bytes, bytes, kind, FB_U8, -1, 0, { send, recv, bytes } };
    call.staged = true;
    return nbCollective(comm, rank, bytes > 0, call, [=](auto& c, cudaStream_t st) {
        const faabric::device::Communicator::GroupItem item{ send, recv, bytes };
        return c.groupMany(kind, &item, 1, FB_U8, 0, 0, 0, st);
    }, host, 0);
}

int MpiWorld::nbNeighborV(const DeviceComm& comm, int rank, faabric::device::Communicator::GroupKind kind,
                          NeighborVCall call, const NeighborVAgree& agree, const HostPath& host)
{
    cacheDeviceComm(rank);
    const int requestId = tls.nextRequestId++;
    AsyncRequest r = collectiveRequest(rank);
    if (comm != nullptr && groupIallreduce) {
        // the burst's key is (kind, communicator); a change of key flushes
        // the pending burst before this call joins
        const faabric::device::Communicator::GroupItem placeholder{ call.send, call.recv, 0 };
        deferToGroup(kind, comm, FB_U8, -1, 0, placeholder, requestId, std::move(r), deviceCollectives);
        tls.groupVCalls.push_back(std::move(call));
        tls.groupAgree = agree;
        return requestId;
    }
    void* s = tls.cachedStream0;
    const std::vector<NeighborVCall> one{ call };
    if (comm != nullptr && issueDevice(*comm, s, deviceCollectives, [&](auto& c, cudaStream_t st) {
            return runNeighborV(c, kind, one, agree, st);
        })) {
        return recordDevice(requestId, std::move(r), comm, s);
    }
    host();
    tls.requests[requestId] = std::move(r);
    return requestId;
}

bool MpiWorld::deviceNeighborV(const DeviceComm& comm, int rank, faabric::device::Communicator::GroupKind kind,
                               const NeighborVCall& call, const NeighborVAgree& agree)
{
    const std::vector<NeighborVCall> one{ call };
    return issueAndWait(comm, streamForRank(rank), deviceCollectives, [&](auto& c, cudaStream_t s) {
        return runNeighborV(c, kind, one, agree, s);
    });
}

bool MpiWorld::deviceNeighbor(const DeviceComm& comm, int rank, faabric::device::Communicator::GroupKind kind,
                              const uint8_t* send, uint8_t* recv, size_t bytes)
{
    return issueAndWait(comm, streamForRank(rank), deviceCollectives, [&](auto& c, cudaStream_t s) {
        const faabric::device::Communicator::GroupItem item{ send, recv, bytes };
        return c.groupMany(kind, &item, 1, FB_U8, 0, 0, 0, s);
    });
}

int MpiWorld::iGather(int rank, int root, const uint8_t* send, uint8_t* recv, size_t bytes, faabric_datatype_t* sendType,
                      int sendCount, faabric_datatype_t* recvType, int recvCount, int persistentComm)
{
    checkRanksRange(rank, root);
    cacheDeviceComm(rank);
    // (the blocking call takes the root's in-place send as recv itself)
    const bool inPlace = rank == root && send == recv + (size_t)root * bytes;
    const DeviceComm dev = bytes > 0 && isDevicePointer(send) ? tls.cachedComm : nullptr;
    return nbGather(dev, rank, root, send, recv, bytes, [=, this] {
        gather(rank, root, inPlace ? recv : send, sendType, sendCount, recv, recvType, recvCount);
    }, persistentComm);
}

int MpiWorld::nbGather(const DeviceComm& comm, int rank, int root, const uint8_t* send, uint8_t* recv, size_t bytes,
                       const HostPath& host, int persistentComm)
{
    // a byte copy through the staging buffers: the burst's key is
    // (communicator, root).  The caller passes `comm` only for a device
    // send (an in-place root's send lies in its recv).
    NbCall call{ bytes, bytes, bytes, faabric::device::Communicator::GROUP_GATHER, FB_U8, -1, root,
                 { send, recv, bytes } };
    call.staged = true;
    return nbCollective(comm, rank, bytes > 0, call, [=](auto& c, cudaStream_t st) {
        return c.gather(send, recv, bytes, root, 0, st);
    }, host, persistentComm);
}

int MpiWorld::iScatter(int rank, int root, const uint8_t* send, uint8_t* recv, size_t bytes, faabric_datatype_t* sendType,
                       int sendCount, faabric_datatype_t* recvType, int recvCount, int persistentComm)
{
    checkRanksRange(root, rank);
    cacheDeviceComm(rank);
    const DeviceComm dev = bytes > 0 && isDevicePointer(recv) ? tls.cachedComm : nullptr;
    return nbScatter(dev, rank, root, send, recv, bytes, [=, this] {
        scatter(root, rank, send, sendType, sendCount, recv, recvType, recvCount);
    }, persistentComm);
}

int MpiWorld::nbScatter(const DeviceComm& comm, int rank, int root, const uint8_t* send, uint8_t* recv, size_t bytes,
                        const HostPath& host, int persistentComm)
{
    // the mirror of nbGather: `comm` only for a device recv
    NbCall call{ bytes, bytes, bytes, faabric::device::Communicator::GROUP_SCATTER, FB_U8, -1, root,
                 { send, recv, bytes } };
    call.staged = true;
    return nbCollective(comm, rank, bytes > 0, call, [=](auto& c, cudaStream_t st) {
        return c.scatter(send, recv, bytes, root, 0, st);
    }, host, persistentComm);
}

int MpiWorld::iReduce(int rank, int root, const uint8_t* send, uint8_t* recv, faabric_datatype_t* dt, int count,
                      faabric_op_t* op, int persistentComm)
{
    checkRanksRange(rank, root);
    cacheDeviceComm(rank);
    const DeviceComm dev = count > 0 && isDevicePointer(send) && deviceReducible(dt, op) ? tls.cachedComm : nullptr;
    return nbReduce(dev, rank, root, send, recv, dt, count, op, [=, this] {
        reduce(rank, root, const_cast<uint8_t*>(send), recv, dt, count, op);
    }, persistentComm);
}

int MpiWorld::nbReduce(const DeviceComm& comm, int rank, int root, const uint8_t* send, uint8_t* recv,
                       faabric_datatype_t* dt, int count, faabric_op_t* op, const HostPath& host, int persistentComm)
{
    // staged like the gather: the burst's key is (communicator, dtype, op,
    // root)
    const size_t bytes = (size_t)count * dt->size;
    const int fdt = fbDtypeFor(dt);
    const int fop = fbOpFor(op);
    NbCall call{ bytes, bytes, bytes, faabric::device::Communicator::GROUP_REDUCE, fdt, fop, root,
                 { send, recv, (size_t)count } };
    call.staged = true;
    return nbCollective(comm, rank, bytes > 0, call, [=](auto& c, cudaStream_t st) {
        return c.reduce(send, recv, (size_t)count, fdt, fop, root, 0, st);
    }, host, persistentComm);
}

int MpiWorld::iScan(int rank, bool exclusive, const uint8_t* send, uint8_t* recv, faabric_datatype_t* dt, int count,
                    faabric_op_t* op, int persistentComm)
{
    checkRanksRange(0, rank);
    cacheDeviceComm(rank);
    const DeviceComm dev = count > 0 && isDevicePointer(send) && deviceReducible(dt, op) ? tls.cachedComm : nullptr;
    return nbScan(dev, rank, exclusive, send, recv, dt, count, op, [=, this] {
        if (exclusive) {
            exscan(rank, send, recv, dt, count, op);
        } else {
            scan(rank, const_cast<uint8_t*>(send), recv, dt, count, op);
        }
    }, persistentComm);
}

int MpiWorld::nbScan(const DeviceComm& comm, int rank, bool exclusive, const uint8_t* send, uint8_t* recv,
                     faabric_datatype_t* dt, int count, faabric_op_t* op, const HostPath& host, int persistentComm)
{
    // staged like the reduce: the burst's key is (kind, communicator, dtype,
    // op), and in place is each rank's own affair.  At issue (grouping off)
    // the call is a one-item grouped launch too: the blocking device scan
    // refuses in place.
    const size_t bytes = (size_t)count * dt->size;
    const int fdt = fbDtypeFor(dt);
    const int fop = fbOpFor(op);
    const auto kind =
      exclusive ? faabric::device::Communicator::GROUP_EXSCAN : faabric::device::Communicator::GROUP_SCAN;
    NbCall call{ bytes, bytes, bytes, kind, fdt, fop, 0, { send, recv, (size_t)count } };
    call.staged = true;
    return nbCollective(comm, rank, bytes > 0, call, [=](auto& c, cudaStream_t st) {
        return c.groupMany(kind, &call.item, 1, fdt, fop, 0, 0, st);
    }, host, persistentComm);
}

void MpiWorld::settleDeviceBurst(const DeviceComm& comm)
{
    if (comm == nullptr || tls.groupItems.empty() || tls.groupComm != comm) {
        return;
    }
    void* stream = tls.groupStream;
    flushPendingGroup();
    cudaSetDevice(comm->device());
    awaitDevice(*comm, stream);
}

void* MpiWorld::deviceAlloc(int rank, size_t bytes)
{
    auto comm = getDeviceComm(rank);
    if (comm == nullptr) {
        return nullptr;
    }
    try {
        return comm->heapPtr(comm->alloc(bytes));
    } catch (const std::bad_alloc&) {
        return nullptr;
    }
}

bool MpiWorld::deviceFree(int rank, void* ptr)
{
    std::shared_ptr<faabric::device::Communicator> comm;
    {
        std::lock_guard<std::mutex> lk(deviceMx);
        if (rank < 0 || rank >= (int)deviceComms.size()) {
            return false;
        }
        comm = deviceComms[rank];
    }
    if (comm == nullptr || !comm->inHeap(ptr)) {
        return false;
    }
    comm->free(comm->offsetOf(ptr));
    return true;
}

// ---------------------------------------------------------------------------
// Collectives
// ---------------------------------------------------------------------------
void MpiWorld::broadcast(int rootRank,
                         int thisRank,
                         uint8_t* buffer,
                         faabric_datatype_t* dataType,
                         int count,
                         MpiMessageType messageType)
{
    const size_t bytes = (size_t)count * dataType->size;
    if (bytes > 0 && isDevicePointer(buffer)) {
        if (deviceBroadcast(getDeviceComm(thisRank), thisRank, rootRank, buffer, bytes)) {
            return;
        }
        HostStage st;
        uint8_t* host = st.out(buffer, bytes, thisRank == rootRank);
        broadcast(rootRank, thisRank, host, dataType, count, messageType);
        if (thisRank != rootRank) {
            st.flush();
        }
        return;
    }

    if (messageType == MpiMessageType::NORMAL && sharedMemoryEligible(bytes)) {
        sharedBroadcast(rootRank, thisRank, buffer, bytes);
        return;
    }
    // Two-level tree: the root feeds its co-located ranks and one leader per
    // other host; leaders feed their own host
    const std::string rootHost = getHostForRank(rootRank);
    if (thisRank == rootRank) {
        std::set<int> localRanks;
        std::map<std::string, int> leaders;
        {
            std::lock_guard<std::mutex> lk(worldMx);
            localRanks = ranksForHost[thisHost];
            leaders = leaderForHost;
        }
        for (int r : localRanks) {
            if (r != rootRank) {
                send(rootRank, r, buffer, dataType, count, messageType);
            }
        }
        for (const auto& [host, leader] : leaders) {
            if (host != thisHost && !getHostForRank(leader).empty()) {
                send(rootRank, leader, buffer, dataType, count, messageType);
            }
        }
        return;
    }
    const bool rootIsLocal = rootHost == thisHost;
    const int localLeader = getLocalLeader();
    if (!rootIsLocal && thisRank == localLeader) {
        recv(rootRank, thisRank, buffer, dataType, count, nullptr, messageType);
        std::set<int> localRanks;
        {
            std::lock_guard<std::mutex> lk(worldMx);
            localRanks = ranksForHost[thisHost];
        }
        for (int r : localRanks) {
            if (r != thisRank) {
                send(thisRank, r, buffer, dataType, count, messageType);
            }
        }
        return;
    }
    int from = rootIsLocal ? rootRank : localLeader;
    recv(from, thisRank, buffer, dataType, count, nullptr, messageType);
}

void MpiWorld::scatter(int sendRank,
                       int recvRank,
                       const uint8_t* sendBuffer,
                       faabric_datatype_t* sendType,
                       int sendCount,
                       uint8_t* recvBuffer,
                       faabric_datatype_t* recvType,
                       int recvCount)
{
    checkRanksRange(sendRank, recvRank);
    const size_t chunk = (size_t)sendCount * sendType->size;
    if (chunk > 0 && isDevicePointer(recvBuffer)) {
        if (deviceScatter(getDeviceComm(recvRank), recvRank, sendRank, sendBuffer, recvBuffer, chunk)) {
            return;
        }
    }
    {
        // counts on the sending side only mean something at the root
        const size_t myChunk = recvRank == sendRank ? chunk : (size_t)recvCount * recvType->size;
        if (!isDevicePointer(recvBuffer) && !(recvRank == sendRank && isDevicePointer(sendBuffer)) &&
            sharedMemoryEligible(myChunk * size)) {
            sharedScatter(recvRank, sendRank, sendBuffer, recvBuffer, myChunk);
            return;
        }
    }
    // Flat: the root sends chunk r to rank r
    if (recvRank == sendRank) {
        HostStage in;
        const uint8_t* src = in.in(sendBuffer, chunk * size);
        for (int r = 0; r < size; r++) {
            const uint8_t* c = src + (size_t)r * chunk;
            if (r == sendRank) {
                HostStage out;
                uint8_t* dst = out.out(recvBuffer, chunk);
                memcpy(dst, c, chunk);
                out.flush();
            } else {
                send(sendRank, r, c, sendType, sendCount, MpiMessageType::SCATTER);
            }
        }
    } else {
        recv(sendRank, recvRank, recvBuffer, recvType, recvCount, nullptr, MpiMessageType::SCATTER);
    }
}

void MpiWorld::gather(int sendRank,
                      int recvRank,
                      const uint8_t* sendBuffer,
                      faabric_datatype_t* sendType,
                      int sendCount,
                      uint8_t* recvBuffer,
                      faabric_datatype_t* recvType,
                      int recvCount)
{
    checkRanksRange(sendRank, recvRank);
    const size_t sendBytes = (size_t)sendCount * sendType->size;
    const size_t recvBytes = (size_t)recvCount * recvType->size;
    const bool isRoot = sendRank == recvRank;
    // In place: the root's contribution already sits in its slot
    const bool inPlace = isRoot && sendBuffer == recvBuffer;

    // (the root's in-place case takes the device path too: see deviceGather)
    const bool deviceCall = isDevicePointer(isRoot && inPlace ? recvBuffer : sendBuffer);
    if (sendBytes > 0 && deviceCall &&
        deviceGather(getDeviceComm(sendRank), sendRank, recvRank, inPlace ? nullptr : sendBuffer, recvBuffer, sendBytes)) {
        return;
    }

    if (!isDevicePointer(sendBuffer) && !(isRoot && isDevicePointer(recvBuffer)) && sharedMemoryEligible(sendBytes * size)) {
        sharedGather(sendRank, recvRank, sendBuffer, recvBuffer, sendBytes, inPlace);
        return;
    }
    const std::string rootHost = getHostForRank(recvRank);
    const bool rootIsLocal = rootHost == thisHost;
    std::set<int> localRanks;
    std::map<std::string, std::set<int>> allRanks;
    {
        std::lock_guard<std::mutex> lk(worldMx);
        localRanks = ranksForHost[thisHost];
        allRanks = ranksForHost;
    }
    if (isRoot) {
        HostStage out;
        uint8_t* dst = out.out(recvBuffer, recvBytes * size, inPlace);
        if (!inPlace) {
            HostStage in;
            memcpy(dst + (size_t)recvRank * recvBytes, in.in(sendBuffer, sendBytes), sendBytes);
        }
        // Co-located ranks send their own chunk; every other host sends one
        // packed message from its leader (chunks in ascending rank order)
        for (int r : localRanks) {
            if (r != recvRank) {
                recv(r, recvRank, dst + (size_t)r * recvBytes, recvType, recvCount, nullptr, MpiMessageType::GATHER);
            }
        }
        for (const auto& [host, ranks] : allRanks) {
            if (host == thisHost || ranks.empty()) {
                continue;
            }
            int leader = *ranks.begin();
            std::vector<uint8_t> packed(recvBytes * ranks.size());
            recv(leader, recvRank, packed.data(), recvType, recvCount * (int)ranks.size(), nullptr, MpiMessageType::GATHER);
            size_t k = 0;
            for (int r : ranks) {
                memcpy(dst + (size_t)r * recvBytes, packed.data() + k * recvBytes, recvBytes);
                k++;
            }
        }
        out.flush();
        return;
    }
    HostStage in;
    const uint8_t* mine = in.in(sendBuffer, sendBytes);
    if (rootIsLocal) {
        send(sendRank, recvRank, mine, sendType, sendCount, MpiMessageType::GATHER);
        return;
    }
    const int localLeader = getLocalLeader();
    if (sendRank == localLeader) {
        std::vector<uint8_t> packed(sendBytes * localRanks.size());
        size_t k = 0;
        for (int r : localRanks) {
            if (r == sendRank) {
                memcpy(packed.data() + k * sendBytes, mine, sendBytes);
            } else {
                recv(r, sendRank, packed.data() + k * sendBytes, sendType, sendCount, nullptr, MpiMessageType::GATHER);
            }
            k++;
        }
        send(sendRank, recvRank, packed.data(), sendType, sendCount * (int)localRanks.size(), MpiMessageType::GATHER);
    } else {
        send(sendRank, localLeader, mine, sendType, sendCount, MpiMessageType::GATHER);
    }
}

void MpiWorld::allGather(int rank,
                         const uint8_t* sendBuffer,
                         faabric_datatype_t* sendType,
                         int sendCount,
                         uint8_t* recvBuffer,
                         faabric_datatype_t* recvType,
                         int recvCount)
{
    checkRanksRange(0, rank);
    const size_t sendBytes = (size_t)sendCount * sendType->size;
    if (sendBytes > 0 && isDevicePointer(sendBuffer) && sendBuffer != recvBuffer + (size_t)rank * sendBytes &&
        deviceAllGather(getDeviceComm(rank), rank, sendBuffer, recvBuffer, sendBytes)) {
        return;
    }
    if (!isDevicePointer(sendBuffer) && !isDevicePointer(recvBuffer) && sharedMemoryEligible(sendBytes * size)) {
        sharedAllGather(rank, sendBuffer, recvBuffer, sendBytes);
        return;
    }
    // gather to rank 0, then broadcast the concatenation
    const int root = MPI_MAIN_RANK;
    const int fullCount = recvCount * size;
    gather(rank, root, sendBuffer, sendType, sendCount, recvBuffer, recvType, recvCount);
    broadcast(root, rank, recvBuffer, recvType, fullCount, MpiMessageType::ALLGATHER);
}

void MpiWorld::reduce(int sendRank,
                      int recvRank,
                      uint8_t* sendBuffer,
                      uint8_t* recvBuffer,
                      faabric_datatype_t* datatype,
                      int count,
                      faabric_op_t* operation)
{
    checkRanksRange(sendRank, recvRank);
    const size_t bytes = (size_t)count * datatype->size;
    const bool isRoot = sendRank == recvRank;
    const bool inPlace = sendBuffer == recvBuffer;

    // Same choice on every rank (only the root can see MPI_IN_PLACE): in-place
    // at the root stays on the device
    if (bytes > 0 && isDevicePointer(sendBuffer) && deviceReducible(datatype, operation) &&
        deviceReduce(getDeviceComm(sendRank), sendRank, recvRank, sendBuffer, recvBuffer, datatype, count, operation)) {
        return;
    }
    if (bytes > 0 && (isDevicePointer(sendBuffer) || (isRoot && isDevicePointer(recvBuffer)))) {
        HostStage in, out;
        uint8_t* s = in.in(sendBuffer, bytes);
        uint8_t* r = isRoot ? (inPlace ? s : out.out(recvBuffer, bytes)) : recvBuffer;
        reduce(sendRank, recvRank, s, r, datatype, count, operation);
        if (isRoot) {
            if (inPlace) {
                copyBytes(recvBuffer, s, bytes);
            } else {
                out.flush();
            }
        }
        return;
    }

    if (isOrderedUserOp(operation)) {
        orderedReduce(sendRank, recvRank, sendBuffer, recvBuffer, datatype, count, operation);
        return;
    }
    if (sharedMemoryEligible(bytes)) {
        sharedReduce(sendRank, recvRank, sendBuffer, recvBuffer, datatype, count, operation);
        return;
    }
    const std::string rootHost = getHostForRank(recvRank);
    const bool rootIsLocal = rootHost == thisHost;
    std::set<int> localRanks;
    std::map<std::string, int> leaders;
    {
        std::lock_guard<std::mutex> lk(worldMx);
        localRanks = ranksForHost[thisHost];
        leaders = leaderForHost;
    }
    if (isRoot) {
        // Own contribution first, then fold in every message as it arrives
        if (!inPlace) {
            memcpy(recvBuffer, sendBuffer, bytes);
        }
        std::vector<uint8_t> incoming(bytes);
        for (int r : localRanks) {
            if (r == recvRank) {
                continue;
            }
            recv(r, recvRank, incoming.data(), datatype, count, nullptr, MpiMessageType::REDUCE);
            op_reduce(operation, datatype, count, incoming.data(), recvBuffer);
        }
        for (const auto& [host, leader] : leaders) {
            if (host == thisHost || getHostForRank(leader) != host) {
                continue;
            }
            recv(leader, recvRank, incoming.data(), datatype, count, nullptr, MpiMessageType::REDUCE);
            op_reduce(operation, datatype, count, incoming.data(), recvBuffer);
        }
        return;
    }
    if (rootIsLocal) {
        send(sendRank, recvRank, sendBuffer, datatype, count, MpiMessageType::REDUCE);
        return;
    }
    const int localLeader = getLocalLeader();
    if (sendRank == localLeader) {
        // Reduce this host's ranks into a copy (never touch the user's send
        // buffer), then one message to the root
        std::vector<uint8_t> acc(sendBuffer, sendBuffer + bytes);
        std::vector<uint8_t> incoming(bytes);
        for (int r : localRanks) {
            if (r == sendRank) {
                continue;
            }
            recv(r, sendRank, incoming.data(), datatype, count, nullptr, MpiMessageType::REDUCE);
            op_reduce(operation, datatype, count, incoming.data(), acc.data());
        }
        send(sendRank, recvRank, acc.data(), datatype, count, MpiMessageType::REDUCE);
    } else {
        send(sendRank, localLeader, sendBuffer, datatype, count, MpiMessageType::REDUCE);
    }
}

void MpiWorld::orderedReduce(int sendRank,
                             int recvRank,
                             uint8_t* sendBuffer,
                             uint8_t* recvBuffer,
                             faabric_datatype_t* datatype,
                             int count,
                             faabric_op_t* operation)
{
    // MPI requires rank order for non-commutative operations: bring every
    // contribution to the root and fold right to left,
    //   r0 op (r1 op (... op r[n-1]))
    // which equals the left-to-right order by associativity
    const size_t bytes = (size_t)count * datatype->size;
    if (sendRank != recvRank) {
        gather(sendRank, recvRank, sendBuffer, datatype, count, nullptr, datatype, count);
        return;
    }
    // (`all` never aliases the user's buffers, in-place reduce or not)
    std::vector<uint8_t> all(bytes * (size_t)size);
    gather(sendRank, recvRank, sendBuffer, datatype, count, all.data(), datatype, count);
    memcpy(recvBuffer, all.data() + (size_t)(size - 1) * bytes, bytes);
    for (int r = size - 2; r >= 0; r--) {
        op_reduce(operation, datatype, count, all.data() + (size_t)r * bytes, recvBuffer);
    }
}

void MpiWorld::allReduce(int rank,
                         uint8_t* sendBuffer,
                         uint8_t* recvBuffer,
                         faabric_datatype_t* datatype,
                         int count,
                         faabric_op_t* operation)
{
    checkRanksRange(0, rank);
    const size_t bytes = (size_t)count * datatype->size;
    if (bytes > 0 && isDevicePointer(sendBuffer)) {
        if (deviceReducible(datatype, operation) &&
            deviceAllReduce(getDeviceComm(rank), rank, sendBuffer, recvBuffer, datatype, count, operation)) {
            return;
        }
        HostStage in, out;
        uint8_t* s = in.in(sendBuffer, bytes);
        uint8_t* r = sendBuffer == recvBuffer ? s : out.out(recvBuffer, bytes);
        allReduce(rank, s, r, datatype, count, operation);
        if (sendBuffer == recvBuffer) {
            copyBytes(recvBuffer, s, bytes);
        } else {
            out.flush();
        }
        return;
    }
    if (trySharedMemoryAllReduce(rank, sendBuffer, recvBuffer, datatype, count, operation)) {
        return;
    }
    // Otherwise the reference's algorithm: reduce to rank 0 then broadcast
    const int root = MPI_MAIN_RANK;
    reduce(rank, root, sendBuffer, recvBuffer, datatype, count, operation);
    broadcast(root, rank, recvBuffer, datatype, count, MpiMessageType::ALLREDUCE);
}

void MpiWorld::reduceScatter(int rank,
                             uint8_t* sendBuffer,
                             uint8_t* recvBuffer,
                             faabric_datatype_t* datatype,
                             int recvCount,
                             faabric_op_t* operation)
{
    const size_t sliceBytes = (size_t)recvCount * datatype->size;
    if (sliceBytes > 0 && isDevicePointer(sendBuffer)) {
        int fdt = fbDtypeFor(datatype);
        int fop = fbOpFor(operation);
        auto comm = (fdt >= 0 && fop >= 0) ? getDeviceComm(rank) : nullptr;
        if (issueAndWait(comm, streamForRank(rank), deviceCollectives, [&](auto& c, cudaStream_t s) {
                return c.reduceScatter(sendBuffer, recvBuffer, (size_t)recvCount, fdt, fop, symFlag(c, sendBuffer, sliceBytes * size), s);
            })) {
            return;
        }
    }
    // Host: all-reduce everything, keep our slice
    HostStage in;
    uint8_t* s = in.in(sendBuffer, sliceBytes * size);
    std::vector<uint8_t> full(sliceBytes * size);
    allReduce(rank, s, full.data(), datatype, recvCount * size, operation);
    HostStage out;
    uint8_t* r = out.out(recvBuffer, sliceBytes);
    memcpy(r, full.data() + (size_t)rank * sliceBytes, sliceBytes);
    out.flush();
}

// ---- host-side element-wise reduction for every (op, dtype) ----
namespace {
// MAX/MIN/SUM/PROD as the device kernels define them (reduce_ops.h): integer
// SUM/PROD wrap without signed overflow, float MAX/MIN do not depend on the
// order of the operands (NaN, signed zeros)
template<typename T>
void reduceArith(int opId, int count, const uint8_t* inRaw, uint8_t* outRaw)
{
    const T* in = reinterpret_cast<const T*>(inRaw);
    T* out = reinterpret_cast<T*>(outRaw);
    switch (opId) {
        case FAABRIC_OP_MAX:
            for (int i = 0; i < count; i++) {
                out[i] = faabric::util::reduceMax(out[i], in[i]);
            }
            break;
        case FAABRIC_OP_MIN:
            for (int i = 0; i < count; i++) {
                out[i] = faabric::util::reduceMin(out[i], in[i]);
            }
            break;
        case FAABRIC_OP_SUM:
            for (int i = 0; i < count; i++) {
                out[i] = faabric::util::reduceSum(out[i], in[i]);
            }
            break;
        case FAABRIC_OP_PROD:
            for (int i = 0; i < count; i++) {
                out[i] = faabric::util::reduceProd(out[i], in[i]);
            }
            break;
        case FAABRIC_OP_LAND:
            for (int i = 0; i < count; i++) {
                out[i] = (T)((out[i] != (T)0) && (in[i] != (T)0));
            }
            break;
        case FAABRIC_OP_LOR:
            for (int i = 0; i < count; i++) {
                out[i] = (T)((out[i] != (T)0) || (in[i] != (T)0));
            }
            break;
        case FAABRIC_OP_LXOR:
            for (int i = 0; i < count; i++) {
                out[i] = (T)((out[i] != (T)0) != (in[i] != (T)0));
            }
            break;
        default:
            throw std::runtime_error("Unsupported operation for this type");
    }
}

template<typename T>
void reduceInt(int opId, int count, const uint8_t* inRaw, uint8_t* outRaw)
{
    const T* in = reinterpret_cast<const T*>(inRaw);
    T* out = reinterpret_cast<T*>(outRaw);
    switch (opId) {
        case FAABRIC_OP_BAND:
            for (int i = 0; i < count; i++) {
                out[i] = (T)(out[i] & in[i]);
            }
            break;
        case FAABRIC_OP_BOR:
            for (int i = 0; i < count; i++) {
                out[i] = (T)(out[i] | in[i]);
            }
            break;
        case FAABRIC_OP_BXOR:
            for (int i = 0; i < count; i++) {
                out[i] = (T)(out[i] ^ in[i]);
            }
            break;
        default:
            reduceArith<T>(opId, count, inRaw, outRaw);
    }
}

template<typename V>
void reduceLoc(int opId, int count, const uint8_t* inRaw, uint8_t* outRaw)
{
    struct Pair
    {
        V v;
        int i;
    };
    const Pair* in = reinterpret_cast<const Pair*>(inRaw);
    Pair* out = reinterpret_cast<Pair*>(outRaw);
    for (int k = 0; k < count; k++) {
        bool take;
        if (opId == FAABRIC_OP_MAXLOC) {
            take = in[k].v > out[k].v || (in[k].v == out[k].v && in[k].i < out[k].i);
        } else {
            take = in[k].v < out[k].v || (in[k].v == out[k].v && in[k].i < out[k].i);
        }
        if (take) {
            out[k] = in[k];
        }
    }
}

float halfToFloat(uint16_t h, bool bf16)
{
    if (bf16) {
        uint32_t u = (uint32_t)h << 16;
        float f;
        memcpy(&f, &u, 4);
        return f;
    }
    uint32_t sign = (h >> 15) & 1, exp = (h >> 10) & 0x1f, man = h & 0x3ff;
    uint32_t u;
    if (exp == 0) {
        if (man == 0) {
            u = sign << 31;
        } else {
            exp = 127 - 15 + 1;
            while ((man & 0x400) == 0) {
                man <<= 1;
                exp--;
            }
            man &= 0x3ff;
            u = (sign << 31) | (exp << 23) | (man << 13);
        }
    } else if (exp == 31) {
        u = (sign << 31) | 0x7f800000u | (man << 13);
    } else {
        u = (sign << 31) | ((exp + 127 - 15) << 23) | (man << 13);
    }
    float f;
    memcpy(&f, &u, 4);
    return f;
}

uint16_t floatToHalf(float f, bool bf16)
{
    uint32_t u;
    memcpy(&u, &f, 4);
    if (bf16) {
        // NaN stays a (quiet) NaN: the rounding increment below could carry
        // its payload into the sign bit (0x7fffffff -> 0x8000, i.e. -0.0)
        if ((u & 0x7fffffffu) > 0x7f800000u) {
            return (uint16_t)((u >> 16) | 0x40u);
        }
        // round to nearest even
        uint32_t lsb = (u >> 16) & 1;
        u += 0x7fffu + lsb;
        return (uint16_t)(u >> 16);
    }
    uint32_t sign = (u >> 16) & 0x8000u;
    int32_t exp = (int32_t)((u >> 23) & 0xff) - 127 + 15;
    uint32_t man = u & 0x7fffffu;
    if (exp >= 31) {
        return (uint16_t)(sign | 0x7c00u | (((u >> 23) & 0xff) == 0xff && man ? 0x200u : 0));
    }
    if (exp <= 0) {
        if (exp < -10) {
            return (uint16_t)sign;
        }
        man |= 0x800000u;
        uint32_t shift = (uint32_t)(14 - exp);
        uint32_t h = man >> shift;
        uint32_t rem = man & ((1u << shift) - 1);
        uint32_t half = 1u << (shift - 1);
        if (rem > half || (rem == half && (h & 1))) {
            h++;
        }
        return (uint16_t)(sign | h);
    }
    uint32_t h = ((uint32_t)exp << 10) | (man >> 13);
    uint32_t rem = man & 0x1fffu;
    if (rem > 0x1000u || (rem == 0x1000u && (h & 1))) {
        h++;
    }
    return (uint16_t)(sign | h);
}

void reduceHalf(int opId, int count, const uint8_t* inRaw, uint8_t* outRaw, bool bf16)
{
    const uint16_t* in = reinterpret_cast<const uint16_t*>(inRaw);
    uint16_t* out = reinterpret_cast<uint16_t*>(outRaw);
    for (int i = 0; i < count; i++) {
        float a = halfToFloat(out[i], bf16);
        float b = halfToFloat(in[i], bf16);
        float r;
        switch (opId) {
            case FAABRIC_OP_MAX:
                r = faabric::util::reduceMax(a, b);
                break;
            case FAABRIC_OP_MIN:
                r = faabric::util::reduceMin(a, b);
                break;
            case FAABRIC_OP_SUM:
                r = a + b;
                break;
            case FAABRIC_OP_PROD:
                r = a * b;
                break;
            default:
                throw std::runtime_error("Unsupported operation for this type");
        }
        out[i] = floatToHalf(r, bf16);
    }
}
}

void MpiWorld::op_reduce(faabric_op_t* operation,
                         faabric_datatype_t* datatype,
                         int count,
                         uint8_t* inBuffer,
                         uint8_t* resultBuffer)
{
    if (datatype->id >= FAABRIC_DERIVED_TYPE_BASE) {
        // n elements of "k x base" are n*k elements of base; user functions see
        // the base type too
        int baseId = 0, per = 0;
        if (!getContiguousType(datatype->id, &baseId, &per)) {
            throw std::runtime_error("Reduction on an unknown derived datatype");
        }
        op_reduce(operation, getFaabricDatatypeFromId(baseId), count * per, inBuffer, resultBuffer);
        return;
    }
    const int op = operation->id;
    if (isUserOp(operation)) {
        MPI_User_function* fn = nullptr;
        bool commutes = true;
        if (!getUserOp(op, &fn, &commutes)) {
            SPDLOG_ERROR("User reduce operation {} has been freed or never existed", op);
            throw std::runtime_error("Unknown user-defined reduce operation");
        }
        // inout[i] = in[i] op inout[i]
        fn(inBuffer, resultBuffer, &count, &datatype);
        return;
    }
    if (!reducible(datatype, operation)) {
        SPDLOG_ERROR("Unsupported type/op for reduce: type {} op {}", datatype->id, op);
        throw std::runtime_error("Unsupported type for reduce");
    }
    switch (datatype->id) {
        case FAABRIC_INT8:
        case FAABRIC_CHAR:
            return reduceInt<int8_t>(op, count, inBuffer, resultBuffer);
        case FAABRIC_UINT8:
        case FAABRIC_BYTE:
        case FAABRIC_C_BOOL:
            return reduceInt<uint8_t>(op, count, inBuffer, resultBuffer);
        case FAABRIC_INT16:
            return reduceInt<int16_t>(op, count, inBuffer, resultBuffer);
        case FAABRIC_UINT16:
            return reduceInt<uint16_t>(op, count, inBuffer, resultBuffer);
        case FAABRIC_INT32:
        case FAABRIC_INT:
            return reduceInt<int32_t>(op, count, inBuffer, resultBuffer);
        case FAABRIC_UINT32:
        case FAABRIC_UINT:
            return reduceInt<uint32_t>(op, count, inBuffer, resultBuffer);
        case FAABRIC_INT64:
        case FAABRIC_LONG:
        case FAABRIC_LONG_LONG:
        case FAABRIC_LONG_LONG_INT:
            return reduceInt<int64_t>(op, count, inBuffer, resultBuffer);
        case FAABRIC_UINT64:
            return reduceInt<uint64_t>(op, count, inBuffer, resultBuffer);
        case FAABRIC_FLOAT:
            return reduceArith<float>(op, count, inBuffer, resultBuffer);
        case FAABRIC_DOUBLE:
            return reduceArith<double>(op, count, inBuffer, resultBuffer);
        case FAABRIC_HALF:
            return reduceHalf(op, count, inBuffer, resultBuffer, false);
        case FAABRIC_BFLOAT16:
            return reduceHalf(op, count, inBuffer, resultBuffer, true);
        case FAABRIC_DOUBLE_INT:
            return reduceLoc<double>(op, count, inBuffer, resultBuffer);
        case FAABRIC_FLOAT_INT:
            return reduceLoc<float>(op, count, inBuffer, resultBuffer);
        case FAABRIC_2INT:
            return reduceLoc<int32_t>(op, count, inBuffer, resultBuffer);
        default:
            return reduceLoc<int64_t>(op, count, inBuffer, resultBuffer); // FAABRIC_LONG_INT
    }
}

bool MpiWorld::reducible(faabric_datatype_t* datatype, faabric_op_t* operation)
{
    if (operation == nullptr || datatype == nullptr) {
        return false;
    }
    if (isUserOp(operation)) {
        return true;
    }
    int typeId = datatype->id;
    if (typeId >= FAABRIC_DERIVED_TYPE_BASE) {
        int per = 0;
        if (!getContiguousType(datatype->id, &typeId, &per)) {
            return false;
        }
    }
    const int op = operation->id;
    if (op < FAABRIC_OP_MAX || op > FAABRIC_OP_BXOR || op == FAABRIC_OP_NULL) {
        return false;
    }
    const bool isLoc = op == FAABRIC_OP_MAXLOC || op == FAABRIC_OP_MINLOC;
    const bool isBitwise = op == FAABRIC_OP_BAND || op == FAABRIC_OP_BOR || op == FAABRIC_OP_BXOR;
    const bool isArith = op == FAABRIC_OP_MAX || op == FAABRIC_OP_MIN || op == FAABRIC_OP_SUM || op == FAABRIC_OP_PROD;
    switch (typeId) {
        case FAABRIC_INT8:
        case FAABRIC_CHAR:
        case FAABRIC_UINT8:
        case FAABRIC_BYTE:
        case FAABRIC_C_BOOL:
        case FAABRIC_INT16:
        case FAABRIC_UINT16:
        case FAABRIC_INT32:
        case FAABRIC_INT:
        case FAABRIC_UINT32:
        case FAABRIC_UINT:
        case FAABRIC_INT64:
        case FAABRIC_LONG:
        case FAABRIC_LONG_LONG:
        case FAABRIC_LONG_LONG_INT:
        case FAABRIC_UINT64:
            return !isLoc;
        case FAABRIC_FLOAT:
        case FAABRIC_DOUBLE:
            return !isLoc && !isBitwise;
        case FAABRIC_HALF:
        case FAABRIC_BFLOAT16:
            return isArith;
        case FAABRIC_DOUBLE_INT:
        case FAABRIC_FLOAT_INT:
        case FAABRIC_2INT:
        case FAABRIC_LONG_INT:
            return isLoc;
        default:
            return false;
    }
}

void MpiWorld::scan(int rank,
                    uint8_t* sendBuffer,
                    uint8_t* recvBuffer,
                    faabric_datatype_t* datatype,
                    int count,
                    faabric_op_t* operation)
{
    checkRanksRange(0, rank);
    const size_t bytes = (size_t)count * datatype->size;
    if (bytes > 0 && isDevicePointer(sendBuffer) && sendBuffer != recvBuffer && deviceReducible(datatype, operation) &&
        deviceScan(getDeviceComm(rank), rank, sendBuffer, recvBuffer, datatype, count, operation)) {
        return;
    }
    if (bytes > 0 && (isDevicePointer(sendBuffer) || isDevicePointer(recvBuffer))) {
        HostStage in, out;
        uint8_t* s = in.in(sendBuffer, bytes);
        uint8_t* r = sendBuffer == recvBuffer ? s : out.out(recvBuffer, bytes);
        scan(rank, s, r, datatype, count, operation);
        if (sendBuffer == recvBuffer) {
            copyBytes(recvBuffer, s, bytes);
        } else {
            out.flush();
        }
        return;
    }
    // Linear chain: r-1 -> r.  (The reference forwards with MPI_INT whatever
    // the datatype - src/mpi/MpiWorld.cpp:1429 - fixed here.)
    if (sendBuffer != recvBuffer) {
        memcpy(recvBuffer, sendBuffer, bytes);
    }
    if (rank > 0) {
        std::vector<uint8_t> prev(bytes);
        recv(rank - 1, rank, prev.data(), datatype, count, nullptr, MpiMessageType::SCAN);
        op_reduce(operation, datatype, count, prev.data(), recvBuffer);
    }
    if (rank < size - 1) {
        send(rank, rank + 1, recvBuffer, datatype, count, MpiMessageType::SCAN);
    }
}

void MpiWorld::exscan(int rank,
                      const uint8_t* sendBuffer,
                      uint8_t* recvBuffer,
                      faabric_datatype_t* datatype,
                      int count,
                      faabric_op_t* operation)
{
    checkRanksRange(0, rank);
    const size_t bytes = (size_t)count * datatype->size;
    // (judged on the send alone, alike on every rank: in place is the
    // grouped kernel's local matter)
    if (bytes > 0 && isDevicePointer(sendBuffer) && deviceReducible(datatype, operation) &&
        deviceExscan(getDeviceComm(rank), rank, sendBuffer, recvBuffer, datatype, count, operation)) {
        return;
    }
    // Linear chain r-1 -> r: rank r receives prefix_{r-1} and passes on
    // op(prefix_{r-1}, send_r), computed before an in-place recv is
    // overwritten
    std::vector<uint8_t> acc(bytes);
    std::vector<uint8_t> prev(bytes);
    copyBytes(acc.data(), sendBuffer, bytes);
    if (rank > 0) {
        recv(rank - 1, rank, prev.data(), datatype, count, nullptr, MpiMessageType::SCAN);
        op_reduce(operation, datatype, count, prev.data(), acc.data());
    }
    if (rank < size - 1) {
        send(rank, rank + 1, acc.data(), datatype, count, MpiMessageType::SCAN);
    }
    if (rank > 0) {
        copyBytes(recvBuffer, prev.data(), bytes);
    }
}

void MpiWorld::allToAll(int rank,
                        uint8_t* sendBuffer,
                        faabric_datatype_t* sendType,
                        int sendCount,
                        uint8_t* recvBuffer,
                        faabric_datatype_t* recvType,
                        int recvCount)
{
    checkRanksRange(0, rank);
    const size_t chunk = (size_t)sendCount * sendType->size;
    if (chunk > 0 && isDevicePointer(sendBuffer)) {
        if (deviceAllToAll(getDeviceComm(rank), rank, sendBuffer, recvBuffer, chunk)) {
            return;
        }
        HostStage in, out;
        uint8_t* s = in.in(sendBuffer, chunk * size);
        uint8_t* r = out.out(recvBuffer, chunk * size);
        allToAll(rank, s, sendType, sendCount, r, recvType, recvCount);
        out.flush();
        return;
    }
    if (sharedMemoryEligible(chunk * size)) {
        sharedAllToAll(rank, sendBuffer, recvBuffer, chunk);
        return;
    }
    // Flat pairwise exchange: send everything, then receive in rank order
    for (int r = 0; r < size; r++) {
        uint8_t* c = sendBuffer + (size_t)r * chunk;
        if (r == rank) {
            memcpy(recvBuffer + (size_t)rank * chunk, c, chunk);
        } else {
            send(rank, r, c, sendType, sendCount, MpiMessageType::ALLTOALL);
        }
    }
    for (int r = 0; r < size; r++) {
        if (r != rank) {
            recv(r, rank, recvBuffer + (size_t)r * chunk, recvType, recvCount, nullptr, MpiMessageType::ALLTOALL);
        }
    }
}

void MpiWorld::barrier(int thisRank)
{
    // Everyone joins at rank 0, which then releases everyone
    if (thisRank == MPI_MAIN_RANK) {
        for (int r = 1; r < size; r++) {
            recv(r, 0, nullptr, MPI_INT, 0, nullptr, MpiMessageType::BARRIER_JOIN);
        }
    } else {
        send(thisRank, 0, nullptr, MPI_INT, 0, MpiMessageType::BARRIER_JOIN);
    }
    broadcast(0, thisRank, nullptr, MPI_INT, 0, MpiMessageType::BARRIER_DONE);
}

// ---------------------------------------------------------------------------
// Cartesian topology (2-D, periodic)
// ---------------------------------------------------------------------------
void MpiWorld::getCartesianRank(int rank, int maxDims, const int* dims, int* periods, int* coords)
{
    if (rank > size - 1) {
        throw std::runtime_error("Rank bigger than world size");
    }
    if (dims[0] * dims[1] != size) {
        throw std::runtime_error("Product of ranks across dimensions not equal to world size");
    }
    // Every rank records the (same) grid
    cartDims[0].store(dims[0]);
    cartDims[1].store(dims[1]);
    // Row-major placement on the grid
    coords[0] = rank / dims[1];
    coords[1] = rank % dims[1];
    periods[0] = 1;
    periods[1] = 1;
    // Only two dimensions are supported; extra ones must be trivial
    for (int i = 2; i < maxDims; i++) {
        if (dims[i] != 1) {
            throw std::runtime_error("Non-zero number of processes in dimension greater than 2");
        }
        coords[i] = 0;
        periods[i] = 1;
    }
}

bool MpiWorld::getCartesianDims(int* dims2) const
{
    if (cartDims[0] <= 0 || cartDims[1] <= 0) {
        return false;
    }
    dims2[0] = cartDims[0].load();
    dims2[1] = cartDims[1].load();
    return true;
}

void MpiWorld::getRankFromCoords(int* rank, int* coords)
{
    int cols = std::max(1, cartDims[1].load());
    *rank = coords[1] + coords[0] * cols;
}

void MpiWorld::shiftCartesianCoords(int rank, int direction, int disp, int* source, int* destination)
{
    int cols = std::max(1, cartDims[1].load());
    int rows = size / cols;
    int dims[2] = { rows, cols };
    int coords[2] = { rank / cols, rank % cols };
    if (direction < 0 || direction > 1) {
        // Shifting along a trivial dimension leaves the rank where it is
        *source = rank;
        *destination = rank;
        return;
    }
    auto wrap = [](int v, int n) { return ((v % n) + n) % n; };
    int fwd[2] = { coords[0], coords[1] };
    int bwd[2] = { coords[0], coords[1] };
    fwd[direction] = wrap(coords[direction] + disp, dims[direction]);
    bwd[direction] = wrap(coords[direction] - disp, dims[direction]);
    *destination = fwd[0] * cols + fwd[1];
    *source = bwd[0] * cols + bwd[1];
}

// ---------------------------------------------------------------------------
// Migration
// ---------------------------------------------------------------------------
void MpiWorld::prepareMigration(int newGroupId, int thisRank, bool thisRankMustMigrate)
{
    // Everything in flight must have been consumed: migration points sit
    // right after a barrier
    if (!tls.requests.empty()) {
        throw std::runtime_error("Migrating with pending async messages is not supported");
    }
    // Connections to ranks that may be moving are re-established lazily
    tls.sendSockets.clear();
    tls.sendSockets.resize(size);
    for (int& c : tls.recvConnForRank) {
        c = -1;
    }
    if (thisRankMustMigrate) {
        tls.recvSocket.reset();
    }
    // One rank per host refreshes the shared layout
    bool refresh;
    {
        std::lock_guard<std::mutex> lk(worldMx);
        refresh = groupId != newGroupId;
        groupId = newGroupId;
    }
    if (refresh) {
        hasBeenMigrated.store(true);
        broker.waitForMappingsOnThisHost(newGroupId);
        initLocalRemoteLeaders();
        initLocalQueues();
        // Device communicators are rebuilt for the new layout on demand
        std::lock_guard<std::mutex> lk(deviceMx);
        deviceComms.clear();
        deviceTried = false;
    }
}

} // namespace faabric::mpi
