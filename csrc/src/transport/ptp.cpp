#include <faabric/transport/PointToPointBroker.h>
#include <faabric/transport/PointToPointClient.h>
#include <faabric/transport/PointToPointServer.h>
#include <faabric/transport/common.h>
#include <faabric/util/config.h>
#include <faabric/util/logging.h>
#include <faabric/util/testing.h>
#include <faabric/device/communicator.h>
#include <faabric/mpi/MpiWorld.h>
#include <faabric/util/hwloc.h>

#include <cuda_runtime.h>

#include <map>

#define NO_CURRENT_GROUP_ID -1
#define MAPPING_TIMEOUT_MS 20000

namespace faabric::transport {

static std::string thisHostAddress()
{
    return getThisHostAddress();
}

static bool isThisHost(const std::string& host)
{
    if (host == thisHostAddress()) {
        return true;
    }
    HostAddress a = parseHostAddress(host);
    auto& conf = faabric::util::getSystemConfig();
    return a.ip == conf.endpointHost && a.portOffset == conf.portOffset;
}

static std::string pairKey(int groupId, int sendIdx, int recvIdx)
{
    return std::to_string(groupId) + "-" + std::to_string(sendIdx) + "-" +
           std::to_string(recvIdx);
}

static std::string idxKey(int groupId, int groupIdx)
{
    return std::to_string(groupId) + "-" + std::to_string(groupIdx);
}

static std::string mailboxLabel(int groupId, int sendIdx, int recvIdx)
{
    return "ptp-" + pairKey(groupId, sendIdx, recvIdx);
}

// ---------------------------------------------------------------------------
// Mock capture + client
// ---------------------------------------------------------------------------
static std::mutex mockMutex;
static std::vector<std::pair<std::string, faabric::PointToPointMappings>> sentMappings;
static std::vector<std::pair<std::string, faabric::PointToPointMessage>> sentMessages;
static std::vector<std::tuple<std::string, PointToPointCall, faabric::PointToPointMessage>>
  sentLockMessages;

std::vector<std::pair<std::string, faabric::PointToPointMappings>> getSentMappings()
{
    std::lock_guard<std::mutex> lk(mockMutex);
    return sentMappings;
}

std::vector<std::pair<std::string, faabric::PointToPointMessage>>
getSentPointToPointMessages()
{
    std::lock_guard<std::mutex> lk(mockMutex);
    return sentMessages;
}

std::vector<std::tuple<std::string, PointToPointCall, faabric::PointToPointMessage>>
getSentLockMessages()
{
    std::lock_guard<std::mutex> lk(mockMutex);
    return sentLockMessages;
}

void clearSentMessages()
{
    std::lock_guard<std::mutex> lk(mockMutex);
    sentMappings.clear();
    sentMessages.clear();
    sentLockMessages.clear();
}

PointToPointClient::PointToPointClient(const std::string& hostIn)
  : MessageEndpointClient(hostIn,
                          POINT_TO_POINT_ASYNC_PORT,
                          POINT_TO_POINT_SYNC_PORT)
{}

void PointToPointClient::sendMappings(faabric::PointToPointMappings& mappings)
{
    if (faabric::util::isMockMode()) {
        std::lock_guard<std::mutex> lk(mockMutex);
        sentMappings.emplace_back(host, mappings);
        return;
    }
    faabric::EmptyResponse resp;
    syncSend(PointToPointCall::MAPPING, &mappings, &resp);
}

void PointToPointClient::sendMessage(const faabric::PointToPointMessage& msg,
                                     int sequenceNum)
{
    if (faabric::util::isMockMode()) {
        std::lock_guard<std::mutex> lk(mockMutex);
        sentMessages.emplace_back(host, msg);
        return;
    }
    std::string buf = msg.SerializeAsString();
    asyncSend(PointToPointCall::MESSAGE, (const uint8_t*)buf.data(), buf.size(), sequenceNum);
}

void PointToPointClient::makeCoordinationRequest(int appId,
                                                 int groupId,
                                                 int groupIdx,
                                                 PointToPointCall call)
{
    faabric::PointToPointMessage req;
    req.set_appid(appId);
    req.set_groupid(groupId);
    req.set_sendidx(groupIdx);
    req.set_recvidx(POINT_TO_POINT_MAIN_IDX);
    if (faabric::util::isMockMode()) {
        std::lock_guard<std::mutex> lk(mockMutex);
        sentLockMessages.emplace_back(host, call, req);
        return;
    }
    std::string buf = req.SerializeAsString();
    asyncSend(call, (const uint8_t*)buf.data(), buf.size());
}

void PointToPointClient::groupLock(int appId, int groupId, int groupIdx, bool recursive)
{
    makeCoordinationRequest(appId,
                            groupId,
                            groupIdx,
                            recursive ? PointToPointCall::LOCK_GROUP_RECURSIVE
                                      : PointToPointCall::LOCK_GROUP);
}

void PointToPointClient::groupUnlock(int appId, int groupId, int groupIdx, bool recursive)
{
    makeCoordinationRequest(appId,
                            groupId,
                            groupIdx,
                            recursive ? PointToPointCall::UNLOCK_GROUP_RECURSIVE
                                      : PointToPointCall::UNLOCK_GROUP);
}

std::vector<uint8_t> PointToPointClient::rmaRequest(PointToPointCall call, const std::vector<uint8_t>& request)
{
    Message res = syncSendRaw(call, request.data(), request.size());
    return std::vector<uint8_t>(res.udata().begin(), res.udata().end());
}

void PointToPointClient::rmaLockGrant(const uint8_t* buffer, size_t bytes)
{
    asyncSend(PointToPointCall::RMA_LOCK_GRANT, buffer, bytes);
}

static thread_local std::unordered_map<std::string, std::shared_ptr<PointToPointClient>>
  tlsClients;

std::shared_ptr<PointToPointClient> getPointToPointClient(const std::string& host)
{
    auto it = tlsClients.find(host);
    if (it != tlsClients.end()) {
        return it->second;
    }
    auto c = std::make_shared<PointToPointClient>(host);
    tlsClients[host] = c;
    return c;
}

void clearPointToPointClients()
{
    tlsClients.clear();
}

// ---------------------------------------------------------------------------
// Groups
// ---------------------------------------------------------------------------
static std::shared_mutex groupsMutex;
static std::unordered_map<int, std::shared_ptr<PointToPointGroup>> groups;

std::shared_ptr<PointToPointGroup> PointToPointGroup::getGroup(int groupId)
{
    std::shared_lock<std::shared_mutex> lk(groupsMutex);
    auto it = groups.find(groupId);
    if (it == groups.end()) {
        SPDLOG_ERROR("Did not find group ID {} on this host", groupId);
        throw std::runtime_error("Group ID not found on host");
    }
    return it->second;
}

std::shared_ptr<PointToPointGroup> PointToPointGroup::getOrAwaitGroup(int groupId)
{
    getPointToPointBroker().waitForMappingsOnThisHost(groupId);
    return getGroup(groupId);
}

bool PointToPointGroup::groupExists(int groupId)
{
    std::shared_lock<std::shared_mutex> lk(groupsMutex);
    return groups.count(groupId) > 0;
}

void PointToPointGroup::addGroup(int appId, int groupId, int groupSize)
{
    std::unique_lock<std::shared_mutex> lk(groupsMutex);
    if (groups.count(groupId) == 0) {
        groups.emplace(groupId,
                       std::make_shared<PointToPointGroup>(appId, groupId, groupSize));
    }
}

void PointToPointGroup::addGroupIfNotExists(int appId, int groupId, int groupSize)
{
    if (groupExists(groupId)) {
        return;
    }
    addGroup(appId, groupId, groupSize);
}

void PointToPointGroup::clearGroup(int groupId)
{
    std::unique_lock<std::shared_mutex> lk(groupsMutex);
    groups.erase(groupId);
}

void PointToPointGroup::clear()
{
    std::unique_lock<std::shared_mutex> lk(groupsMutex);
    groups.clear();
}

PointToPointGroup::PointToPointGroup(int appIdIn, int groupIdIn, int groupSizeIn)
  : conf(faabric::util::getSystemConfig())
  , appId(appIdIn)
  , groupId(groupIdIn)
  , groupSize(groupSizeIn)
{
    // (the coordinator of a group is the host of idx 0: looked up when needed,
    // a group may be registered before - or without - that mapping)
    localBarrier = faabric::util::Barrier::create(groupSize);
}

bool PointToPointGroup::isSingleHost()
{
    auto hosts = getPointToPointBroker().getHostsRegisteredForGroup(groupId);
    return hosts.size() == 1 && isThisHost(*hosts.begin());
}

void PointToPointGroup::lock(int groupIdx, bool recursive)
{
    PointToPointBroker& broker = getPointToPointBroker();
    std::string host = broker.getHostForReceiver(groupId, POINT_TO_POINT_MAIN_IDX);
    if (isThisHost(host)) {
        masterLock(groupIdx, recursive);
    } else {
        getPointToPointClient(host)->groupLock(appId, groupId, groupIdx, recursive);
    }
    // The grant arrives as a message from the coordinator idx
    broker.recvMessage(groupId, POINT_TO_POINT_MAIN_IDX, groupIdx);
}

void PointToPointGroup::masterLock(int groupIdx, bool recursive)
{
    bool granted = false;
    {
        std::lock_guard<std::mutex> lk(mx);
        if (recursive) {
            if (recursiveLockOwners.empty() || recursiveLockOwners.top() == groupIdx) {
                recursiveLockOwners.push(groupIdx);
                granted = true;
            }
        } else if (lockOwnerIdx == NO_LOCK_OWNER_IDX) {
            lockOwnerIdx = groupIdx;
            granted = true;
        }
        if (!granted) {
            lockWaiters.push(groupIdx);
        }
    }
    if (granted) {
        notifyLocked(groupIdx);
    }
}

void PointToPointGroup::notifyLocked(int groupIdx)
{
    std::vector<uint8_t> data(1, 0);
    getPointToPointBroker().sendMessage(
      groupId, POINT_TO_POINT_MAIN_IDX, groupIdx, data.data(), data.size());
}

void PointToPointGroup::unlock(int groupIdx, bool recursive)
{
    std::string host = getPointToPointBroker().getHostForReceiver(groupId, POINT_TO_POINT_MAIN_IDX);
    if (isThisHost(host)) {
        masterUnlock(groupIdx, recursive);
    } else {
        getPointToPointClient(host)->groupUnlock(appId, groupId, groupIdx, recursive);
    }
}

void PointToPointGroup::masterUnlock(int groupIdx, bool recursive)
{
    int next = NO_LOCK_OWNER_IDX;
    {
        std::lock_guard<std::mutex> lk(mx);
        if (recursive) {
            if (!recursiveLockOwners.empty()) {
                recursiveLockOwners.pop();
            }
            if (!recursiveLockOwners.empty()) {
                return;
            }
            if (!lockWaiters.empty()) {
                next = lockWaiters.front();
                lockWaiters.pop();
                recursiveLockOwners.push(next);
            }
        } else {
            lockOwnerIdx = NO_LOCK_OWNER_IDX;
            if (!lockWaiters.empty()) {
                next = lockWaiters.front();
                lockWaiters.pop();
                lockOwnerIdx = next;
            }
        }
    }
    if (next != NO_LOCK_OWNER_IDX) {
        notifyLocked(next);
    }
}

int PointToPointGroup::getLockOwner(bool recursive)
{
    std::lock_guard<std::mutex> lk(mx);
    if (recursive) {
        return recursiveLockOwners.empty() ? NO_LOCK_OWNER_IDX : recursiveLockOwners.top();
    }
    return lockOwnerIdx;
}

void PointToPointGroup::localLock()
{
    if (!localMx.try_lock_for(std::chrono::milliseconds(timeoutMs))) {
        throw std::runtime_error("Timed out acquiring local group lock");
    }
}

void PointToPointGroup::localUnlock()
{
    localMx.unlock();
}

bool PointToPointGroup::localTryLock()
{
    return localMx.try_lock();
}

void PointToPointGroup::deviceBarrier(int groupIdx, void* stream)
{
    auto comm = getPointToPointBroker().getDeviceCommunicator(groupId, groupIdx);
    if (comm == nullptr) {
        throw std::runtime_error("Group " + std::to_string(groupId) + " idx " + std::to_string(groupIdx) +
                                 " has no device communicator");
    }
    if (comm->barrier((cudaStream_t)stream) != FB_OK) {
        throw std::runtime_error("Device barrier launch failed");
    }
}

void PointToPointGroup::barrier(int groupIdx)
{
    PointToPointBroker& devBroker = getPointToPointBroker();
    if (devBroker.isDeviceGroup(groupId)) {
        // every member sits on a GPU: meet on the device
        auto comm = devBroker.getDeviceCommunicator(groupId, groupIdx);
        cudaStream_t s = comm->internalStream();
        deviceBarrier(groupIdx, s);
        if (!comm->syncStreamBounded(s, (uint64_t)timeoutMs)) {
            throw std::runtime_error("Device barrier timed out");
        }
        return;
    }
    if (isSingleHost()) {
        localBarrier->wait();
        return;
    }
    PointToPointBroker& broker = getPointToPointBroker();
    if (groupIdx == POINT_TO_POINT_MAIN_IDX) {
        // Gather then release
        for (int i = 1; i < groupSize; i++) {
            broker.recvMessage(groupId, i, POINT_TO_POINT_MAIN_IDX);
        }
        std::vector<uint8_t> data(1, 0);
        for (int i = 1; i < groupSize; i++) {
            broker.sendMessage(groupId, POINT_TO_POINT_MAIN_IDX, i, data.data(), data.size());
        }
    } else {
        std::vector<uint8_t> data(1, 0);
        broker.sendMessage(groupId, groupIdx, POINT_TO_POINT_MAIN_IDX, data.data(), data.size());
        broker.recvMessage(groupId, POINT_TO_POINT_MAIN_IDX, groupIdx);
    }
}

void PointToPointGroup::notify(int groupIdx)
{
    PointToPointBroker& broker = getPointToPointBroker();
    if (groupIdx == POINT_TO_POINT_MAIN_IDX) {
        for (int i = 1; i < groupSize; i++) {
            broker.recvMessage(groupId, i, POINT_TO_POINT_MAIN_IDX);
        }
    } else {
        std::vector<uint8_t> data(1, 0);
        broker.sendMessage(groupId, groupIdx, POINT_TO_POINT_MAIN_IDX, data.data(), data.size());
    }
}

int PointToPointGroup::getNotifyCount()
{
    // Messages idx 0 has not consumed yet
    int n = 0;
    for (int i = 1; i < groupSize; i++) {
        n += (int)getInprocMailbox(mailboxLabel(groupId, i, POINT_TO_POINT_MAIN_IDX))->size();
    }
    return n;
}

// ---------------------------------------------------------------------------
// Broker
// ---------------------------------------------------------------------------
// Receiver-side reorder state lives with the receiving thread
struct ReorderState
{
    int expectedSeq = 0;
    std::map<int, Message> pending;
};
static thread_local std::unordered_map<std::string, ReorderState> tlsReorder;

PointToPointBroker::PointToPointBroker()
  : conf(faabric::util::getSystemConfig())
{}

PointToPointBroker& getPointToPointBroker()
{
    static PointToPointBroker broker;
    return broker;
}

std::string PointToPointBroker::getHostForReceiver(int groupId, int recvIdx)
{
    std::shared_lock<std::shared_mutex> lk(brokerMutex);
    auto it = mappings.find(idxKey(groupId, recvIdx));
    if (it == mappings.end()) {
        SPDLOG_ERROR("No point-to-point mapping for group {} idx {}", groupId, recvIdx);
        throw std::runtime_error("Receiving host not registered with broker");
    }
    return it->second;
}

int PointToPointBroker::getMpiPortForReceiver(int groupId, int recvIdx)
{
    std::shared_lock<std::shared_mutex> lk(brokerMutex);
    auto it = mpiPortMappings.find(idxKey(groupId, recvIdx));
    if (it == mpiPortMappings.end()) {
        SPDLOG_ERROR("No MPI port mapping for group {} idx {}", groupId, recvIdx);
        throw std::runtime_error("MPI port not registered with broker");
    }
    return it->second;
}

std::shared_ptr<faabric::util::FlagWaiter> PointToPointBroker::getGroupFlag(int groupId)
{
    {
        std::shared_lock<std::shared_mutex> lk(brokerMutex);
        auto it = groupFlags.find(groupId);
        if (it != groupFlags.end()) {
            return it->second;
        }
    }
    std::unique_lock<std::shared_mutex> lk(brokerMutex);
    auto& slot = groupFlags[groupId];
    if (slot == nullptr) {
        slot = std::make_shared<faabric::util::FlagWaiter>(MAPPING_TIMEOUT_MS);
    }
    return slot;
}

std::set<std::string> PointToPointBroker::setUpLocalMappingsFromSchedulingDecision(
  const faabric::batch_scheduler::SchedulingDecision& decision)
{
    int groupId = decision.groupId;
    std::set<std::string> hosts;
    {
        std::unique_lock<std::shared_mutex> lk(brokerMutex);
        for (int i = 0; i < decision.nFunctions; i++) {
            int groupIdx = decision.groupIdxs.at(i);
            const std::string& host = decision.hosts.at(i);
            groupIdIdxsMap[groupId].insert(groupIdx);
            mappings[idxKey(groupId, groupIdx)] = host;
            mpiPortMappings[idxKey(groupId, groupIdx)] = decision.mpiPorts.at(i);
            hosts.insert(host);
        }
    }
    PointToPointGroup::addGroupIfNotExists((int)decision.appId, groupId, decision.nFunctions);
    // Everything is in place: release whoever is waiting for this group
    getGroupFlag(groupId)->setFlag(true);
    return hosts;
}

void PointToPointBroker::setAndSendMappingsFromSchedulingDecision(
  const faabric::batch_scheduler::SchedulingDecision& decision)
{
    std::set<std::string> hosts = setUpLocalMappingsFromSchedulingDecision(decision);
    sendMappingsFromSchedulingDecision(decision, hosts);
}

void PointToPointBroker::sendMappingsFromSchedulingDecision(
  const faabric::batch_scheduler::SchedulingDecision& decision,
  const std::set<std::string>& hostList)
{
    faabric::PointToPointMappings msg;
    msg.set_appid((int32_t)decision.appId);
    msg.set_groupid(decision.groupId);
    for (int i = 0; i < decision.nFunctions; i++) {
        auto* m = msg.add_mappings();
        m->set_host(decision.hosts.at(i));
        m->set_messageid(decision.messageIds.at(i));
        m->set_appidx(decision.appIdxs.at(i));
        m->set_groupidx(decision.groupIdxs.at(i));
        m->set_mpiport(decision.mpiPorts.at(i));
    }
    for (const auto& host : hostList) {
        if (isThisHost(host)) {
            continue;
        }
        getPointToPointClient(host)->sendMappings(msg);
    }
}

void PointToPointBroker::waitForMappingsOnThisHost(int groupId)
{
    getGroupFlag(groupId)->waitOnFlag();
}

std::set<int> PointToPointBroker::getIdxsRegisteredForGroup(int groupId)
{
    std::shared_lock<std::shared_mutex> lk(brokerMutex);
    auto it = groupIdIdxsMap.find(groupId);
    return it == groupIdIdxsMap.end() ? std::set<int>() : it->second;
}

std::set<std::string> PointToPointBroker::getHostsRegisteredForGroup(int groupId)
{
    std::shared_lock<std::shared_mutex> lk(brokerMutex);
    std::set<std::string> hosts;
    auto it = groupIdIdxsMap.find(groupId);
    if (it == groupIdIdxsMap.end()) {
        return hosts;
    }
    for (int idx : it->second) {
        hosts.insert(mappings.at(idxKey(groupId, idx)));
    }
    return hosts;
}

void PointToPointBroker::updateHostForIdx(int groupId, int groupIdx, std::string newHost)
{
    std::unique_lock<std::shared_mutex> lk(brokerMutex);
    mappings[idxKey(groupId, groupIdx)] = std::move(newHost);
}

int PointToPointBroker::getAndIncrementSentMsgCount(int groupId, int sendIdx, int recvIdx)
{
    std::lock_guard<std::mutex> lk(seqMx);
    return sentMsgCount[pairKey(groupId, sendIdx, recvIdx)]++;
}

void PointToPointBroker::sendMessage(int groupId,
                                     int sendIdx,
                                     int recvIdx,
                                     const uint8_t* buffer,
                                     size_t bufferSize,
                                     std::string hostHint,
                                     bool mustOrderMsg)
{
    sendMessage(groupId, sendIdx, recvIdx, buffer, bufferSize, mustOrderMsg, NO_SEQUENCE_NUM, std::move(hostHint));
}

void PointToPointBroker::deliverLocally(int groupId,
                                        int sendIdx,
                                        int recvIdx,
                                        const uint8_t* buffer,
                                        size_t bufferSize,
                                        int sequenceNum)
{
    getInprocMailbox(mailboxLabel(groupId, sendIdx, recvIdx))
      ->send(Message(NO_HEADER, sequenceNum, buffer, bufferSize));
}

void PointToPointBroker::sendMessage(int groupId,
                                     int sendIdx,
                                     int recvIdx,
                                     const uint8_t* buffer,
                                     size_t bufferSize,
                                     bool mustOrderMsg,
                                     int sequenceNum,
                                     std::string hostHint)
{
    std::string host = hostHint;
    if (host.empty()) {
        waitForMappingsOnThisHost(groupId);
        host = getHostForReceiver(groupId, recvIdx);
    }
    // Stamp a sequence number at the origin if ordering was requested
    int seq = sequenceNum;
    if (mustOrderMsg && seq == NO_SEQUENCE_NUM) {
        seq = getAndIncrementSentMsgCount(groupId, sendIdx, recvIdx);
    }
    if (isThisHost(host)) {
        deliverLocally(groupId, sendIdx, recvIdx, buffer, bufferSize, seq);
        return;
    }
    faabric::PointToPointMessage msg;
    msg.set_groupid(groupId);
    msg.set_sendidx(sendIdx);
    msg.set_recvidx(recvIdx);
    msg.set_data(buffer, bufferSize);
    getPointToPointClient(host)->sendMessage(msg, seq);
}

Message PointToPointBroker::doRecvMessage(int groupId, int sendIdx, int recvIdx)
{
    return getInprocMailbox(mailboxLabel(groupId, sendIdx, recvIdx))
      ->recv(conf.globalMessageTimeout);
}

std::vector<uint8_t> PointToPointBroker::recvMessage(int groupId,
                                                     int sendIdx,
                                                     int recvIdx,
                                                     bool mustOrderMsg)
{
    if (!mustOrderMsg) {
        return doRecvMessage(groupId, sendIdx, recvIdx).dataCopy();
    }
    ReorderState& st = tlsReorder[pairKey(groupId, sendIdx, recvIdx)];
    while (true) {
        auto it = st.pending.find(st.expectedSeq);
        if (it != st.pending.end()) {
            std::vector<uint8_t> out = it->second.dataCopy();
            st.pending.erase(it);
            st.expectedSeq++;
            return out;
        }
        Message m = doRecvMessage(groupId, sendIdx, recvIdx);
        int seq = m.getSequenceNum();
        if (seq == NO_SEQUENCE_NUM || seq == st.expectedSeq) {
            if (seq != NO_SEQUENCE_NUM) {
                st.expectedSeq++;
            }
            return m.dataCopy();
        }
        st.pending.emplace(seq, std::move(m));
    }
}

// ---------------------------------------------------------------------------
// Device data plane
// ---------------------------------------------------------------------------
void PointToPointBroker::createLocalDeviceGroup(int groupId, std::vector<int> devices)
{
    std::set<int> idxs = getIdxsRegisteredForGroup(groupId);
    if (idxs.empty()) {
        throw std::runtime_error("No mappings for group " + std::to_string(groupId));
    }
    const int n = (int)idxs.size();
    if (*idxs.rbegin() != n - 1) {
        throw std::runtime_error("Device groups need dense idxs 0..n-1");
    }
    if (devices.empty()) {
        int nGpus = faabric::util::getUsableGpus();
        for (int i = 0; i < n; i++) {
            int g = faabric::util::gpuIndexFromHostName(getHostForReceiver(groupId, i));
            devices.push_back(g >= 0 && nGpus > 0 ? g % nGpus : (nGpus > 0 ? i % nGpus : 0));
        }
    }
    if ((int)devices.size() != n) {
        throw std::runtime_error("createLocalDeviceGroup: one device per group idx");
    }
    faabric::device::CommConfig cfg = faabric::device::CommConfig::fromEnv();
    cfg.heapBytes = std::min<size_t>(cfg.heapBytes, (size_t)64 << 20); // messaging only
    cfg.stageBytes = (size_t)1 << 20;
    auto comms = faabric::device::Communicator::createLocal(n, devices, cfg);
    std::unique_lock<std::shared_mutex> lk(brokerMutex);
    auto& slot = deviceComms[groupId];
    for (int i = 0; i < n; i++) {
        slot[i] = comms[i];
    }
}

void PointToPointBroker::joinDeviceGroup(int groupId, int groupIdx, int groupSize, int device)
{
    faabric::device::CommConfig cfg = faabric::device::CommConfig::fromEnv();
    cfg.heapBytes = std::min<size_t>(cfg.heapBytes, (size_t)64 << 20);
    cfg.stageBytes = (size_t)1 << 20;
    auto comm = faabric::device::Communicator::createIpc(
      groupIdx, groupSize, device, "ptp-group-" + std::to_string(groupId), cfg);
    std::unique_lock<std::shared_mutex> lk(brokerMutex);
    deviceComms[groupId][groupIdx] = comm;
}

bool PointToPointBroker::isDeviceGroup(int groupId)
{
    std::shared_lock<std::shared_mutex> lk(brokerMutex);
    return deviceComms.find(groupId) != deviceComms.end();
}

std::shared_ptr<faabric::device::Communicator> PointToPointBroker::getDeviceCommunicator(int groupId, int groupIdx)
{
    std::shared_lock<std::shared_mutex> lk(brokerMutex);
    auto it = deviceComms.find(groupId);
    if (it == deviceComms.end()) {
        return nullptr;
    }
    auto jt = it->second.find(groupIdx);
    return jt == it->second.end() ? nullptr : jt->second;
}

void PointToPointBroker::sendDeviceMessage(int groupId,
                                           int sendIdx,
                                           int recvIdx,
                                           const void* deviceBuffer,
                                           size_t bufferSize,
                                           void* stream)
{
    auto comm = getDeviceCommunicator(groupId, sendIdx);
    if (comm == nullptr) {
        throw std::runtime_error("No device communicator for group " + std::to_string(groupId) + " idx " +
                                 std::to_string(sendIdx));
    }
    int rc = comm->send(deviceBuffer, bufferSize, recvIdx, (cudaStream_t)stream);
    if (rc != FB_OK) {
        throw std::runtime_error(std::string("Device send failed: ") + faabric::device::Communicator::errorString(rc));
    }
}

void PointToPointBroker::recvDeviceMessage(int groupId,
                                           int sendIdx,
                                           int recvIdx,
                                           void* deviceBuffer,
                                           size_t bufferSize,
                                           void* stream)
{
    auto comm = getDeviceCommunicator(groupId, recvIdx);
    if (comm == nullptr) {
        throw std::runtime_error("No device communicator for group " + std::to_string(groupId) + " idx " +
                                 std::to_string(recvIdx));
    }
    int rc = comm->recv(deviceBuffer, bufferSize, sendIdx, (cudaStream_t)stream);
    if (rc != FB_OK) {
        throw std::runtime_error(std::string("Device recv failed: ") + faabric::device::Communicator::errorString(rc));
    }
}

void PointToPointBroker::clearGroup(int groupId)
{
    std::set<int> idxs;
    {
        std::unique_lock<std::shared_mutex> lk(brokerMutex);
        deviceComms.erase(groupId);
        auto it = groupIdIdxsMap.find(groupId);
        if (it != groupIdIdxsMap.end()) {
            idxs = it->second;
        }
        for (int idx : idxs) {
            mappings.erase(idxKey(groupId, idx));
            mpiPortMappings.erase(idxKey(groupId, idx));
        }
        groupIdIdxsMap.erase(groupId);
        groupFlags.erase(groupId);
    }
    {
        std::lock_guard<std::mutex> lk(seqMx);
        for (int a : idxs) {
            for (int b : idxs) {
                sentMsgCount.erase(pairKey(groupId, a, b));
            }
        }
    }
    for (int a : idxs) {
        for (int b : idxs) {
            clearInprocMailbox(mailboxLabel(groupId, a, b));
        }
    }
    PointToPointGroup::clearGroup(groupId);
}

void PointToPointBroker::clear()
{
    {
        std::unique_lock<std::shared_mutex> lk(brokerMutex);
        groupIdIdxsMap.clear();
        mappings.clear();
        mpiPortMappings.clear();
        groupFlags.clear();
        deviceComms.clear();
    }
    {
        std::lock_guard<std::mutex> lk(seqMx);
        sentMsgCount.clear();
    }
    PointToPointGroup::clear();
    clearAllInprocMailboxes();
}

void PointToPointBroker::resetThreadLocalCache()
{
    tlsReorder.clear();
    clearPointToPointClients();
}

void PointToPointBroker::postMigrationHook(int groupId, int groupIdx)
{
    // Everyone in the (new) group lines up before carrying on
    waitForMappingsOnThisHost(groupId);
    PointToPointGroup::getGroup(groupId)->barrier(groupIdx);
}

// ---------------------------------------------------------------------------
// Server
// ---------------------------------------------------------------------------
PointToPointServer::PointToPointServer()
  : MessageEndpointServer(POINT_TO_POINT_ASYNC_PORT,
                          POINT_TO_POINT_SYNC_PORT,
                          POINT_TO_POINT_INPROC_LABEL,
                          faabric::util::getSystemConfig().pointToPointServerThreads)
  , broker(getPointToPointBroker())
{}

void PointToPointServer::doAsyncRecv(transport::Message& message)
{
    uint8_t header = message.getMessageCode();
    switch (header) {
        case PointToPointCall::MESSAGE: {
            faabric::PointToPointMessage msg;
            if (!msg.ParseFromArray(message.udata().data(), (int)message.udata().size())) {
                throw std::runtime_error("Bad point-to-point message");
            }
            broker.deliverLocally(msg.groupid(),
                                  msg.sendidx(),
                                  msg.recvidx(),
                                  (const uint8_t*)msg.data().data(),
                                  msg.data().size(),
                                  message.getSequenceNum());
            break;
        }
        case PointToPointCall::LOCK_GROUP:
            recvGroupLock(message.udata(), false);
            break;
        case PointToPointCall::LOCK_GROUP_RECURSIVE:
            recvGroupLock(message.udata(), true);
            break;
        case PointToPointCall::UNLOCK_GROUP:
            recvGroupUnlock(message.udata(), false);
            break;
        case PointToPointCall::UNLOCK_GROUP_RECURSIVE:
            recvGroupUnlock(message.udata(), true);
            break;
        case PointToPointCall::RMA_LOCK_GRANT:
            faabric::mpi::MpiWorld::serveRmaGrant(message.udata().data(), message.udata().size());
            break;
        default:
            SPDLOG_ERROR("Invalid async point-to-point header: {}", (int)header);
            throw std::runtime_error("Invalid async point-to-point message");
    }
}

std::string PointToPointServer::doSyncRecv(transport::Message& message)
{
    uint8_t header = message.getMessageCode();
    if (header == PointToPointCall::MAPPING) {
        return doRecvMappings(message.udata());
    }
    if (header == PointToPointCall::RMA_LOCK || header == PointToPointCall::RMA_LOCK_CANCEL ||
        header == PointToPointCall::RMA_FLUSH || header == PointToPointCall::RMA_UNLOCK) {
        return faabric::mpi::MpiWorld::serveRmaRequest(header, message.udata().data(), message.udata().size());
    }
    SPDLOG_ERROR("Invalid sync point-to-point header: {}", (int)header);
    throw std::runtime_error("Invalid sync point-to-point message");
}

std::string PointToPointServer::doRecvMappings(std::span<const uint8_t> buffer)
{
    faabric::PointToPointMappings msg;
    if (!msg.ParseFromArray(buffer.data(), (int)buffer.size())) {
        throw std::runtime_error("Bad point-to-point mappings");
    }
    auto decision = faabric::batch_scheduler::SchedulingDecision::fromPointToPointMappings(msg);
    SPDLOG_DEBUG("Receiving {} point-to-point mappings for group {}", decision.nFunctions, decision.groupId);
    broker.setUpLocalMappingsFromSchedulingDecision(decision);
    return faabric::EmptyResponse().SerializeAsString();
}

void PointToPointServer::recvGroupLock(std::span<const uint8_t> buffer, bool recursive)
{
    faabric::PointToPointMessage msg;
    msg.ParseFromArray(buffer.data(), (int)buffer.size());
    PointToPointGroup::getOrAwaitGroup(msg.groupid())->masterLock(msg.sendidx(), recursive);
}

void PointToPointServer::recvGroupUnlock(std::span<const uint8_t> buffer, bool recursive)
{
    faabric::PointToPointMessage msg;
    msg.ParseFromArray(buffer.data(), (int)buffer.size());
    PointToPointGroup::getOrAwaitGroup(msg.groupid())->masterUnlock(msg.sendidx(), recursive);
}

void PointToPointServer::onWorkerStop()
{
    // Worker threads hold thread-local clients: drop them
    broker.resetThreadLocalCache();
}

} // namespace faabric::transport
