// PlannerClient / KeepAliveThread / PlannerServer
#include <faabric/batch-scheduler/BatchScheduler.h>
#include <faabric/planner/PlannerClient.h>
#include <faabric/planner/PlannerServer.h>
#include <faabric/snapshot/SnapshotClient.h>
#include <faabric/transport/common.h>
#include <faabric/util/string_tools.h>
#include <faabric/util/batch.h>
#include <faabric/util/config.h>
#include <faabric/util/func.h>
#include <faabric/util/logging.h>
#include <faabric/util/network.h>
#include <faabric/util/ptp.h>
#include <faabric/util/testing.h>

namespace faabric::planner {

// ---------------------------------------------------------------------------
// Keep-alive
// ---------------------------------------------------------------------------
void KeepAliveThread::doWork()
{
    std::vector<std::shared_ptr<RegisterHostRequest>> reqs;
    {
        std::shared_lock<std::shared_mutex> lock(keepAliveThreadMx);
        for (const auto& [ip, req] : hostReqs) {
            reqs.push_back(req);
        }
    }
    for (const auto& req : reqs) {
        try {
            getPlannerClient().registerHost(req);
        } catch (const std::exception& e) {
            SPDLOG_WARN("Keep-alive for {} failed: {}", req->host().ip(), e.what());
        }
    }
}

void KeepAliveThread::setRequest(std::shared_ptr<RegisterHostRequest> hostReqIn)
{
    // Keep-alives must never reset the slot accounting: send a copy without
    // the overwrite flag
    auto req = std::make_shared<RegisterHostRequest>(*hostReqIn);
    req->set_overwrite(false);
    std::unique_lock<std::shared_mutex> lock(keepAliveThreadMx);
    hostReqs[req->host().ip()] = std::move(req);
}

size_t KeepAliveThread::removeRequest(const std::string& hostIp)
{
    std::unique_lock<std::shared_mutex> lock(keepAliveThreadMx);
    hostReqs.erase(hostIp);
    return hostReqs.size();
}

// ---------------------------------------------------------------------------
// Client
// ---------------------------------------------------------------------------
static std::string resolvePlannerHost()
{
    auto& conf = faabric::util::getSystemConfig();
    // "planner" is the compose service name in the reference deployment; on a
    // single box fall back to this machine when it does not resolve
    // PLANNER_HOST may carry a port offset ("host:offset")
    std::string name = conf.plannerHost;
    std::string suffix;
    size_t colon = name.rfind(':');
    if (colon != std::string::npos && faabric::util::stringIsInt(name.substr(colon + 1))) {
        suffix = name.substr(colon);
        name = name.substr(0, colon);
    }
    std::string ip = faabric::util::getIPFromHostname(name);
    if (ip.empty()) {
        ip = conf.endpointHost;
    }
    return ip + suffix;
}

PlannerClient::PlannerClient()
  : PlannerClient(resolvePlannerHost())
{}

PlannerClient::PlannerClient(const std::string& plannerIp)
  : faabric::transport::MessageEndpointClient(plannerIp, PLANNER_ASYNC_PORT, PLANNER_SYNC_PORT)
  , snapshotRegistry(faabric::snapshot::getSnapshotRegistry())
{}

PlannerClient& getPlannerClient()
{
    // One client per thread: connections are not shared across threads
    static thread_local PlannerClient client;
    return client;
}

// The result cache must be shared by all threads of the process (results are
// delivered by FunctionCallServer threads, awaited by executor threads)
static std::mutex sharedCacheMx;
static PlannerCache sharedCache;

void PlannerClient::ping()
{
    EmptyRequest req;
    PingResponse resp;
    syncSend(PlannerCalls::Ping, &req, &resp);
    // Sanity: the planner must answer with a populated config
    if (resp.config().ip().empty() && resp.config().hosttimeout() == 0) {
        SPDLOG_WARN("Planner ping returned an empty config");
    }
}

void PlannerClient::clearCache()
{
    std::lock_guard<std::mutex> lk(sharedCacheMx);
    sharedCache.plannerResults.clear();
    sharedCache.pushedSnapshots.clear();
}

std::vector<Host> PlannerClient::getAvailableHosts()
{
    EmptyRequest req;
    AvailableHostsResponse resp;
    syncSend(PlannerCalls::GetAvailableHosts, &req, &resp);
    std::vector<Host> hosts;
    for (int i = 0; i < resp.hosts_size(); i++) {
        hosts.push_back(resp.hosts(i));
    }
    return hosts;
}

int PlannerClient::registerHost(std::shared_ptr<RegisterHostRequest> req)
{
    RegisterHostResponse resp;
    syncSend(PlannerCalls::RegisterHost, req.get(), &resp);
    if (resp.status().status() != ResponseStatus::OK) {
        throw std::runtime_error("Error registering host with planner!");
    }
    // Sanity check
    if (resp.config().hosttimeout() <= 0) {
        throw std::runtime_error("Planner returned a non-positive keep-alive timeout");
    }
    return resp.config().hosttimeout();
}

void PlannerClient::removeHost(std::shared_ptr<RemoveHostRequest> req)
{
    RemoveHostResponse resp;
    syncSend(PlannerCalls::RemoveHost, req.get(), &resp);
}

// The planner of THIS process (a worker that embeds it: LocalCluster, the
// single-box deployment)?  The hot calls of a fan-out then hand typed objects
// over directly instead of encoding / decoding every message of the batch.
static bool plannerIsInProcess(const std::string& plannerHost)
{
    if (faabric::util::isMockMode() || faabric::util::FaultInjector::get().armed()) {
        return false;
    }
    return faabric::transport::MessageEndpointServer::localServerFor(plannerHost, PLANNER_SYNC_PORT, true) != nullptr;
}

void PlannerClient::setMessageResult(std::shared_ptr<faabric::Message> msg)
{
    if (plannerIsInProcess(host)) {
        // No encode / decode, and no convoy on the planner's lock when every
        // executor thread of a 1024-way fan-in reports at once: `direct` (each
        // executor thread takes the lock), `workers` (typed task on the
        // planner's RPC workers), `combine` (default: whoever arrives first
        // records everybody's pending results in one acquisition)
        static const int mode = []() {
            const char* v = getenv("FAABRIC_PLANNER_RESULTS");
            std::string m = v == nullptr ? "combine" : v;
            return m == "direct" ? 0 : (m == "workers" ? 1 : 2);
        }();
        if (mode == 0) {
            faabric::planner::getPlanner().setMessageResult(msg); // on the executor's thread
            return;
        }
        if (mode == 2) {
            faabric::planner::getPlanner().submitMessageResult(msg);
            return;
        }
        if (auto* srv = faabric::transport::MessageEndpointServer::localServerFor(host, PLANNER_ASYNC_PORT, false)) {
            srv->getAsyncHandler()->deliverLocalTask([msg] { faabric::planner::getPlanner().setMessageResult(msg); });
            return;
        }
    }
    asyncSend(PlannerCalls::SetMessageResult, msg.get());
}

void PlannerClient::setMessageResultLocally(std::shared_ptr<faabric::Message> msg, bool onlyIfAwaited)
{
    std::lock_guard<std::mutex> lk(sharedCacheMx);
    if (onlyIfAwaited && sharedCache.plannerResults.find((uint32_t)msg->id()) == sharedCache.plannerResults.end()) {
        // The waiter the planner is answering has gone (timed out, or served
        // by a result pushed to it directly): nothing to keep
        return;
    }
    // May arrive before anyone waits: the promise holds it until then
    auto& promise = sharedCache.plannerResults[(uint32_t)msg->id()];
    try {
        promise.set_value(msg);
    } catch (const std::future_error&) {
        SPDLOG_DEBUG("Result for message {} delivered twice", msg->id());
    }
}

faabric::Message PlannerClient::getMessageResult(int appId, int msgId, int timeoutMs)
{
    auto msgPtr = std::make_shared<faabric::Message>();
    msgPtr->set_appid(appId);
    msgPtr->set_id(msgId);
    return doGetMessageResult(msgPtr, timeoutMs);
}

faabric::Message PlannerClient::getMessageResult(const faabric::Message& msg, int timeoutMs)
{
    return doGetMessageResult(std::make_shared<faabric::Message>(msg), timeoutMs);
}

faabric::Message PlannerClient::doGetMessageResult(std::shared_ptr<faabric::Message> msgPtr, int timeoutMs)
{
    int msgId = msgPtr->id();
    auto& conf = faabric::util::getSystemConfig();
    // Tell the planner where to call back
    msgPtr->set_mainhost(faabric::transport::getThisHostAddress());
    (void)conf;

    faabric::Message resp;
    // Ask once.  If the result is not there the planner registers us as a
    // waiter and pushes the result to our FunctionCallServer
    std::future<std::shared_ptr<faabric::Message>> fut;
    {
        std::lock_guard<std::mutex> lk(sharedCacheMx);
        auto it = sharedCache.plannerResults.find((uint32_t)msgId);
        if (it == sharedCache.plannerResults.end()) {
            it = sharedCache.plannerResults.emplace((uint32_t)msgId, std::promise<std::shared_ptr<faabric::Message>>()).first;
        }
        try {
            fut = it->second.get_future();
        } catch (const std::future_error&) {
            // Somebody else is already waiting on this id: poll the planner
            // instead of sharing the future
        }
    }
    if (plannerIsInProcess(host)) {
        // (no RPC to ourselves: fork-joins ask once per thread)
        auto direct = faabric::planner::getPlanner().getMessageResult(msgPtr);
        if (direct != nullptr) {
            resp = *direct;
        } else {
            resp.set_type(faabric::Message::EMPTY);
        }
    } else {
        syncSend(PlannerCalls::GetMessageResult, msgPtr.get(), &resp);
    }
    bool ready = resp.id() == msgId && (resp.type() != faabric::Message::EMPTY);
    if (ready) {
        std::lock_guard<std::mutex> lk(sharedCacheMx);
        sharedCache.plannerResults.erase((uint32_t)msgId);
        return resp;
    }
    if (timeoutMs <= 0) {
        // Non-blocking probe
        faabric::Message empty;
        empty.set_type(faabric::Message::EMPTY);
        return empty;
    }
    if (fut.valid()) {
        if (fut.wait_for(std::chrono::milliseconds(timeoutMs)) != std::future_status::ready) {
            std::lock_guard<std::mutex> lk(sharedCacheMx);
            sharedCache.plannerResults.erase((uint32_t)msgId);
            SPDLOG_WARN("Timed out waiting for message result promise {}", msgId);
            faabric::Message empty;
            empty.set_type(faabric::Message::EMPTY);
            return empty;
        }
        faabric::Message out = *fut.get();
        std::lock_guard<std::mutex> lk(sharedCacheMx);
        sharedCache.plannerResults.erase((uint32_t)msgId);
        return out;
    }
    // Fallback: poll
    auto deadline = std::chrono::steady_clock::now() + std::chrono::milliseconds(timeoutMs);
    while (std::chrono::steady_clock::now() < deadline) {
        std::this_thread::sleep_for(std::chrono::milliseconds(2));
        syncSend(PlannerCalls::GetMessageResult, msgPtr.get(), &resp);
        if (resp.id() == msgId && resp.type() != faabric::Message::EMPTY) {
            return resp;
        }
    }
    faabric::Message empty;
    empty.set_type(faabric::Message::EMPTY);
    return empty;
}

std::shared_ptr<faabric::BatchExecuteRequestStatus> PlannerClient::getBatchResults(
  std::shared_ptr<faabric::BatchExecuteRequest> req)
{
    if (plannerIsInProcess(host)) {
        auto direct = faabric::planner::getPlanner().getBatchResults(req->appid());
        if (direct == nullptr) {
            direct = faabric::util::batchExecStatusFactory(req->appid());
            direct->set_appid(0);
        }
        return direct;
    }
    auto status = std::make_shared<faabric::BatchExecuteRequestStatus>();
    syncSend(PlannerCalls::GetBatchResults, req.get(), status.get());
    return status;
}

faabric::batch_scheduler::SchedulingDecision PlannerClient::callFunctions(
  std::shared_ptr<faabric::BatchExecuteRequest> req)
{
    // THREADS requests: the planner distributes the main thread snapshot, so it
    // must have it (full image the first time, tracked changes after that)
    bool isThreads = req->type() == faabric::BatchExecuteRequest::THREADS;
    if (isThreads && req->messages_size() > 0) {
        // (an executor serving a per-GPU virtual host has already stamped its
        // own name: several "hosts" share this process)
        std::string mainHost = faabric::transport::getThisHostAddress();
        for (int i = 0; i < req->messages_size(); i++) {
            if (req->messages(i).mainhost().empty() || !faabric::transport::isHostAlias(req->messages(i).mainhost())) {
                req->mutable_messages(i)->set_mainhost(mainHost);
            }
        }
        if (!req->singlehosthint()) {
            std::string key = faabric::util::getMainThreadSnapshotKey(req->messages(0));
            if (snapshotRegistry.deviceSnapshotExists(key)) {
                // Device-resident image: the planner only needs to know where
                // it lives (control descriptor), the bytes stay in HBM
                auto dsnap = snapshotRegistry.getDeviceSnapshot(key);
                faabric::snapshot::getSnapshotClient(host)->pushDeviceSnapshot(key, dsnap->describe());
                goto snapshotDone;
            }
            auto snap = snapshotRegistry.getSnapshot(key);
            bool firstPush;
            {
                std::lock_guard<std::mutex> lk(sharedCacheMx);
                firstPush = sharedCache.pushedSnapshots.insert(key).second;
            }
            auto snapClient = faabric::snapshot::getSnapshotClient(host);
            if (firstPush) {
                snapClient->pushSnapshot(key, snap);
            } else {
                auto diffs = snap->getTrackedChanges();
                snapClient->pushSnapshotUpdate(key, snap, diffs);
            }
            // Whatever the planner now has, we no longer need to track
            snap->clearTrackedChanges();
        }
    }
snapshotDone:

    faabric::batch_scheduler::SchedulingDecision decision(NOT_ENOUGH_SLOTS, NOT_ENOUGH_SLOTS);
    if (plannerIsInProcess(host)) {
        // the planner keeps (and mutates) its own copy of the request, exactly
        // as it would after decoding one from the wire
        auto own = std::make_shared<faabric::BatchExecuteRequest>(*req);
        decision = *faabric::planner::getPlanner().callBatch(own);
    } else {
        faabric::PointToPointMappings resp;
        syncSend(PlannerCalls::CallBatch, req.get(), &resp);
        decision = faabric::batch_scheduler::SchedulingDecision::fromPointToPointMappings(resp);
    }
    // An elastically scaled-up request came back bigger than it went in: mirror
    // the extra messages so the caller waits for (and accounts) all of them
    if (req->elasticscalehint() && decision.nFunctions > req->messages_size() && req->messages_size() > 0) {
        const faabric::Message proto = req->messages(req->messages_size() - 1);
        for (int i = req->messages_size(); i < decision.nFunctions; i++) {
            faabric::Message* m = req->add_messages();
            *m = proto;
            m->set_id(decision.messageIds.at(i));
            m->set_appidx(decision.appIdxs.at(i));
            m->set_groupidx(decision.groupIdxs.at(i));
        }
    }
    // The planner assigns the group id when it commits the decision: mirror it
    // into the caller's copy of the request
    if (req->messages_size() > 0 && decision.groupId > 0 && decision.groupId != req->groupid()) {
        req->set_groupid(decision.groupId);
        for (int i = 0; i < req->messages_size(); i++) {
            req->mutable_messages(i)->set_groupid(decision.groupId);
        }
    }
    return decision;
}

faabric::batch_scheduler::SchedulingDecision PlannerClient::getSchedulingDecision(
  std::shared_ptr<faabric::BatchExecuteRequest> req)
{
    faabric::PointToPointMappings resp;
    syncSend(PlannerCalls::GetSchedulingDecision, req.get(), &resp);
    return faabric::batch_scheduler::SchedulingDecision::fromPointToPointMappings(resp);
}

int PlannerClient::getNumMigrations()
{
    EmptyRequest req;
    NumMigrationsResponse resp;
    syncSend(PlannerCalls::GetNumMigrations, &req, &resp);
    return resp.nummigrations();
}

std::string PlannerClient::stateMain(const std::string& user, const std::string& key, const std::string& hostIn, bool claim, bool drop)
{
    StateMainRequest req;
    req.set_user(user);
    req.set_key(key);
    req.set_host(hostIn);
    req.set_claim(claim);
    req.set_drop(drop);
    StateMainResponse resp;
    syncSend(PlannerCalls::StateMain, &req, &resp);
    return resp.host();
}

void PlannerClient::preloadSchedulingDecision(
  std::shared_ptr<faabric::batch_scheduler::SchedulingDecision> preloadDec)
{
    faabric::PointToPointMappings mappings = faabric::util::ptpMappingsFromSchedulingDecision(preloadDec);
    EmptyResponse resp;
    syncSend(PlannerCalls::PreloadSchedulingDecision, &mappings, &resp);
}

// ---------------------------------------------------------------------------
// Server
// ---------------------------------------------------------------------------
PlannerServer::PlannerServer()
  : faabric::transport::MessageEndpointServer(PLANNER_ASYNC_PORT,
                                              PLANNER_SYNC_PORT,
                                              PLANNER_INPROC_LABEL,
                                              getPlanner().getConfig().numthreadshttpserver())
  , planner(getPlanner())
{}

void PlannerServer::doAsyncRecv(transport::Message& message)
{
    uint8_t header = message.getMessageCode();
    if (header == PlannerCalls::SetMessageResult) {
        recvSetMessageResult(message.udata());
        return;
    }
    // Bad requests must not take the planner down: log and carry on
    SPDLOG_ERROR("Unrecognised async planner call header: {}", (int)header);
}

std::string PlannerServer::doSyncRecv(transport::Message& message)
{
    uint8_t header = message.getMessageCode();
    switch (header) {
        case PlannerCalls::Ping:
            return recvPing();
        case PlannerCalls::GetAvailableHosts:
            return recvGetAvailableHosts();
        case PlannerCalls::RegisterHost:
            return recvRegisterHost(message.udata());
        case PlannerCalls::RemoveHost:
            return recvRemoveHost(message.udata());
        case PlannerCalls::GetMessageResult:
            return recvGetMessageResult(message.udata());
        case PlannerCalls::GetBatchResults:
            return recvGetBatchResults(message.udata());
        case PlannerCalls::GetSchedulingDecision:
            return recvGetSchedulingDecision(message.udata());
        case PlannerCalls::GetNumMigrations:
            return recvGetNumMigrations(message.udata());
        case PlannerCalls::PreloadSchedulingDecision:
            return recvPreloadSchedulingDecision(message.udata());
        case PlannerCalls::CallBatch:
            return recvCallBatch(message.udata());
        case PlannerCalls::StateMain:
            return recvStateMain(message.udata());
        default:
            SPDLOG_ERROR("Unrecognised sync planner call header: {}", (int)header);
            return EmptyResponse().SerializeAsString();
    }
}

template<typename T>
static bool parseInto(std::span<const uint8_t> buffer, T& msg)
{
    return msg.ParseFromArray(buffer.data(), (int)buffer.size());
}

void PlannerServer::recvSetMessageResult(std::span<const uint8_t> buffer)
{
    auto msg = std::make_shared<faabric::Message>();
    if (!parseInto(buffer, *msg)) {
        SPDLOG_ERROR("Planner could not parse message result");
        return;
    }
    planner.setMessageResult(msg);
}

std::string PlannerServer::recvPing()
{
    PingResponse resp;
    *resp.mutable_config() = planner.getConfig();
    return resp.SerializeAsString();
}

std::string PlannerServer::recvGetAvailableHosts()
{
    AvailableHostsResponse resp;
    for (const auto& h : planner.getAvailableHosts()) {
        *resp.add_hosts() = *h;
    }
    return resp.SerializeAsString();
}

std::string PlannerServer::recvRegisterHost(std::span<const uint8_t> buffer)
{
    RegisterHostRequest req;
    RegisterHostResponse resp;
    bool ok = parseInto(buffer, req) && planner.registerHost(req.host(), req.overwrite());
    if (!ok) {
        SPDLOG_ERROR("Planner failed to register host {}", req.host().ip());
    }
    *resp.mutable_config() = planner.getConfig();
    resp.mutable_status()->set_status(ok ? ResponseStatus::OK : ResponseStatus::ERROR);
    return resp.SerializeAsString();
}

std::string PlannerServer::recvRemoveHost(std::span<const uint8_t> buffer)
{
    RemoveHostRequest req;
    if (parseInto(buffer, req)) {
        planner.removeHost(req.host());
    }
    RemoveHostResponse resp;
    resp.mutable_status()->set_status(ResponseStatus::OK);
    return resp.SerializeAsString();
}

std::string PlannerServer::recvGetMessageResult(std::span<const uint8_t> buffer)
{
    auto msg = std::make_shared<faabric::Message>();
    parseInto(buffer, *msg);
    auto result = planner.getMessageResult(msg);
    if (result == nullptr) {
        faabric::Message empty;
        empty.set_appid(msg->appid());
        empty.set_id(msg->id());
        empty.set_type(faabric::Message::EMPTY);
        return empty.SerializeAsString();
    }
    return result->SerializeAsString();
}

std::string PlannerServer::recvGetBatchResults(std::span<const uint8_t> buffer)
{
    auto req = std::make_shared<faabric::BatchExecuteRequest>();
    parseInto(buffer, *req);
    auto status = planner.getBatchResults(req->appid());
    if (status == nullptr) {
        // Unknown app: empty status, not finished
        status = faabric::util::batchExecStatusFactory(req->appid());
        status->set_appid(0);
    }
    return status->SerializeAsString();
}

std::string PlannerServer::recvGetSchedulingDecision(std::span<const uint8_t> buffer)
{
    auto req = std::make_shared<faabric::BatchExecuteRequest>();
    parseInto(buffer, *req);
    auto decision = planner.getSchedulingDecision(req);
    faabric::PointToPointMappings mappings;
    if (decision != nullptr) {
        mappings = faabric::util::ptpMappingsFromSchedulingDecision(decision);
    }
    return mappings.SerializeAsString();
}

std::string PlannerServer::recvGetNumMigrations(std::span<const uint8_t> buffer)
{
    NumMigrationsResponse resp;
    resp.set_nummigrations(planner.getNumMigrations());
    return resp.SerializeAsString();
}

std::string PlannerServer::recvPreloadSchedulingDecision(std::span<const uint8_t> buffer)
{
    faabric::PointToPointMappings mappings;
    parseInto(buffer, mappings);
    auto decision = std::make_shared<faabric::batch_scheduler::SchedulingDecision>(
      faabric::batch_scheduler::SchedulingDecision::fromPointToPointMappings(mappings));
    planner.preloadSchedulingDecision((int)decision->appId, decision);
    return EmptyResponse().SerializeAsString();
}

std::string PlannerServer::recvStateMain(std::span<const uint8_t> buffer)
{
    StateMainRequest req;
    StateMainResponse resp;
    if (parseInto(buffer, req)) {
        resp.set_host(planner.stateMain(req.user(), req.key(), req.host(), req.claim(), req.drop()));
    }
    return resp.SerializeAsString();
}

std::string PlannerServer::recvCallBatch(std::span<const uint8_t> buffer)
{
    auto req = std::make_shared<faabric::BatchExecuteRequest>();
    if (!parseInto(buffer, *req)) {
        SPDLOG_ERROR("Planner could not parse batch execute request");
        faabric::batch_scheduler::SchedulingDecision bad(NOT_ENOUGH_SLOTS_DECISION);
        auto badPtr = std::make_shared<faabric::batch_scheduler::SchedulingDecision>(bad);
        return faabric::util::ptpMappingsFromSchedulingDecision(badPtr).SerializeAsString();
    }
    auto decision = planner.callBatch(req);
    return faabric::util::ptpMappingsFromSchedulingDecision(decision).SerializeAsString();
}

} // namespace faabric::planner
