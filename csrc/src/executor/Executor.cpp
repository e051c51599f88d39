#include <faabric/batch-scheduler/BatchScheduler.h>
#include <faabric/executor/Executor.h>
#include <faabric/executor/ExecutorContext.h>
#include <faabric/executor/ExecutorFactory.h>
#include <faabric/mpi/MpiWorldRegistry.h>
#include <faabric/planner/PlannerClient.h>
#include <faabric/scheduler/Scheduler.h>
#include <faabric/snapshot/DeviceSnapshot.h>
#include <faabric/snapshot/SnapshotClient.h>
#include <faabric/transport/PointToPointBroker.h>
#include <faabric/transport/common.h>
#include <faabric/util/clock.h>
#include <faabric/util/config.h>
#include <faabric/util/environment.h>
#include <faabric/util/func.h>
#include <faabric/util/gids.h>
#include <faabric/util/logging.h>
#include <faabric/util/memory.h>
#include <faabric/util/network.h>
#include <faabric/util/timing.h>

#include <cuda_runtime.h>

namespace faabric::executor {

// ---------------------------------------------------------------------------
// Context
// ---------------------------------------------------------------------------
static thread_local std::shared_ptr<ExecutorContext> tlsContext = nullptr;

ExecutorContext::ExecutorContext(Executor* executorIn,
                                 std::shared_ptr<faabric::BatchExecuteRequest> reqIn,
                                 int msgIdxIn)
  : executor(executorIn)
  , req(std::move(reqIn))
  , msgIdx(msgIdxIn)
{}

bool ExecutorContext::isSet()
{
    return tlsContext != nullptr;
}

void ExecutorContext::set(Executor* executorIn,
                          std::shared_ptr<faabric::BatchExecuteRequest> reqIn,
                          int msgIdxIn)
{
    tlsContext = std::make_shared<ExecutorContext>(executorIn, std::move(reqIn), msgIdxIn);
}

void ExecutorContext::unset()
{
    tlsContext = nullptr;
}

std::shared_ptr<ExecutorContext> ExecutorContext::get()
{
    if (tlsContext == nullptr) {
        SPDLOG_ERROR("No executor context set");
        throw ExecutorContextException("No executor context set");
    }
    return tlsContext;
}

// ---------------------------------------------------------------------------
// Factory
// ---------------------------------------------------------------------------
static std::shared_ptr<ExecutorFactory> activeFactory;
static std::mutex factoryMx;

void ExecutorFactory::flushHost()
{
    SPDLOG_WARN("Using default flush method");
}

void setExecutorFactory(std::shared_ptr<ExecutorFactory> fac)
{
    std::lock_guard<std::mutex> lk(factoryMx);
    activeFactory = std::move(fac);
}

std::shared_ptr<ExecutorFactory> getExecutorFactory()
{
    std::lock_guard<std::mutex> lk(factoryMx);
    if (activeFactory == nullptr) {
        throw std::runtime_error("No executor factory set");
    }
    return activeFactory;
}

// ---------------------------------------------------------------------------
// Executor
// ---------------------------------------------------------------------------
static std::atomic<int> executorCounter{ 0 };

Executor::Executor(faabric::Message& msg)
  : boundMessage(msg)
  , reg(faabric::snapshot::getSnapshotRegistry())
  , tracker(faabric::util::getDirtyTracker())
  , threadPoolSize(faabric::util::getUsableCores())
  , threadPoolThreads(threadPoolSize)
  , threadTaskQueues(threadPoolSize)
{
    // FAABRIC_EXECUTOR_DEQUEUE_SPIN=0: idle pool threads sleep at once instead
    // of looking for their next task for ~20 us first
    static const bool dequeueSpin = []() {
        const char* v = getenv("FAABRIC_EXECUTOR_DEQUEUE_SPIN");
        return v == nullptr || std::string(v) != "0";
    }();
    for (auto& q : threadTaskQueues) {
        q.setSpinBeforeSleep(dequeueSpin);
    }
    faabric::util::SystemConfig& conf = faabric::util::getSystemConfig();
    // Unique id: host, function, counter
    id = conf.endpointHost + "_" + std::to_string(faabric::util::generateGid());
    touchLastExec();
    for (uint32_t i = 0; i < threadPoolSize; i++) {
        availablePoolThreads.insert((int)i);
    }
    // GPU binding: "gpuN" host aliases pin to that GPU, otherwise round-robin
    int nGpus = faabric::util::getUsableGpus();
    if (nGpus > 0) {
        int alias = faabric::util::gpuIndexFromHostName(msg.executedhost());
        gpuIdx = alias >= 0 ? alias % nGpus : faabric::util::gpuForRank(executorCounter.fetch_add(1));
        int prev = -1;
        cudaGetDevice(&prev);
        if (cudaSetDevice(gpuIdx) == cudaSuccess) {
            cudaStream_t s = nullptr;
            if (cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) == cudaSuccess) {
                computeStream = s;
            }
        }
        cudaGetLastError();
        if (prev >= 0) {
            cudaSetDevice(prev);
        }
    }
    setUpThreadPool();
}

Executor::~Executor()
{
    if (!_isShutdown) {
        SPDLOG_DEBUG("Destructing executor {} without shutting down first", id);
    }
    // (also when it was shut down before: a batch dispatched concurrently with
    // the shutdown may have started a pool thread afterwards, and a thread
    // that was never poisoned only notices its stop token after a whole
    // bound timeout)
    stopPoolThreads();
    if (computeStream != nullptr) {
        cudaStreamDestroy((cudaStream_t)computeStream);
        cudaGetLastError();
    }
}

void Executor::setUpThreadPool() {}

void Executor::shutdown()
{
    if (_isShutdown.exchange(true)) {
        return;
    }
    stopPoolThreads();
}

void Executor::stopPoolThreads()
{
    // Poison every started pool thread, then join
    std::vector<std::shared_ptr<std::jthread>> toJoin;
    {
        std::lock_guard<std::mutex> lk(threadsMutex);
        for (uint32_t i = 0; i < threadPoolThreads.size(); i++) {
            if (threadPoolThreads[i] != nullptr) {
                threadTaskQueues[i].enqueue(ExecutorTask(POOL_SHUTDOWN, nullptr));
                toJoin.push_back(threadPoolThreads[i]);
            }
        }
    }
    for (auto& t : toJoin) {
        if (t->joinable() && t->get_id() != std::this_thread::get_id()) {
            t->join();
        }
    }
    {
        std::lock_guard<std::mutex> lk(threadsMutex);
        for (auto& t : threadPoolThreads) {
            t = nullptr;
        }
    }
}

void Executor::joinThreadPool()
{
    shutdown();
}

bool Executor::tryClaim()
{
    bool expected = false;
    return claimed.compare_exchange_strong(expected, true);
}

void Executor::claim()
{
    if (!tryClaim()) {
        throw std::runtime_error("Executor already claimed");
    }
}

void Executor::releaseClaim()
{
    // (the key only depends on what the executor was bound to: built once)
    if (schedulerKey.empty()) {
        schedulerKey = faabric::scheduler::Scheduler::executorKeyFor(boundMessage);
    }
    claimed.store(false);
    // Tell the scheduler so the next claim does not have to search for us
    faabric::scheduler::getScheduler().notifyExecutorIdle(schedulerKey, weak_from_this());
}

bool Executor::isExecuting()
{
    return claimed.load();
}

static int64_t steadyNowNs()
{
    return (int64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(
             faabric::util::getGlobalClock().now().time_since_epoch())
      .count();
}

void Executor::touchLastExec()
{
    lastExecNs.store(steadyNowNs(), std::memory_order_relaxed);
}

long Executor::getMillisSinceLastExec()
{
    return (long)((steadyNowNs() - lastExecNs.load(std::memory_order_relaxed)) / 1000000);
}

namespace {
struct GpuGuard
{
    int prev = -1;
    explicit GpuGuard(int dev)
    {
        cudaGetDevice(&prev);
        if (dev >= 0) {
            cudaSetDevice(dev);
        }
    }
    ~GpuGuard()
    {
        if (prev >= 0) {
            cudaSetDevice(prev);
        }
        cudaGetLastError();
    }
};

void cudaCheck(cudaError_t e, const char* what)
{
    if (e != cudaSuccess) {
        throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
    }
}
}

// The planner host this message executes on: a per-GPU virtual host name when
// the worker serves several, else the worker's own address
static std::string servedHost(const faabric::Message& msg)
{
    return msg.executedhost().empty() ? faabric::transport::getThisHostAddress() : msg.executedhost();
}

static bool mainHostIsHere(const faabric::Message& msg)
{
    return msg.mainhost().empty() || msg.mainhost() == servedHost(msg);
}

// ---- hooks (defaults) ----
void Executor::reset(faabric::Message& msg)
{
    // (reference: src/executor/Executor.cpp reset() - the chained calls of the
    // function that just finished are forgotten)
    std::lock_guard<std::mutex> lk(chainedMx);
    chainedMessages.clear();
}

DeviceMemoryView Executor::getDeviceMemoryView()
{
    return {};
}

int32_t Executor::executeTask(int threadPoolIdx,
                              int msgIdx,
                              std::shared_ptr<faabric::BatchExecuteRequest> req)
{
    return 0;
}

std::span<uint8_t> Executor::getMemoryView()
{
    SPDLOG_WARN("Executor for {} has not implemented memory view method", faabric::util::funcToString(boundMessage, false));
    return {};
}

void Executor::setMemorySize(size_t newSize)
{
    SPDLOG_WARN("Executor has not implemented set memory size method");
}

size_t Executor::getMaxMemorySize()
{
    SPDLOG_WARN("Executor has not implemented max memory size method");
    return 0;
}

void Executor::restore(const std::string& snapshotKey)
{
    DeviceMemoryView dv = getDeviceMemoryView();
    if (!dv.empty()) {
        // Device-resident function memory: the restore is a device copy (peer
        // copy over NVLink when the image lives on another GPU), or one H2D
        // copy when only a host image exists (thaw from a checkpoint)
        GpuGuard g(dv.device);
        auto stream = (cudaStream_t)computeStream;
        if (reg.deviceSnapshotExists(snapshotKey)) {
            auto snap = reg.getDeviceSnapshot(snapshotKey);
            if (snap->getSize() > dv.size) {
                setMemorySize(snap->getSize());
                dv = getDeviceMemoryView();
            }
            snap->restoreTo(dv.ptr, std::min(dv.size, snap->getSize()), stream);
        } else {
            auto snap = reg.getSnapshot(snapshotKey);
            if (snap->getSize() > dv.size) {
                setMemorySize(snap->getSize());
                dv = getDeviceMemoryView();
            }
            cudaCheck(cudaMemcpyAsync(dv.ptr, snap->getDataPtr(), std::min(dv.size, snap->getSize()), cudaMemcpyHostToDevice, stream),
                      "restore H2D");
        }
        cudaCheck(cudaStreamSynchronize(stream), "restore sync");
        return;
    }
    std::span<uint8_t> memView = getMemoryView();
    if (memView.empty()) {
        SPDLOG_WARN("Not restoring {}: empty memory view", snapshotKey);
        return;
    }
    auto snap = reg.getSnapshot(snapshotKey);
    // Grow executor memory if the image is bigger, then CoW-map it in
    if (snap->getSize() > memView.size()) {
        setMemorySize(snap->getSize());
        memView = getMemoryView();
    }
    snap->mapToMemory({ memView.data(), snap->getSize() });
}

// ---- chained messages ----
void Executor::addChainedMessage(const faabric::Message& msg)
{
    std::lock_guard<std::mutex> lk(chainedMx);
    auto ber = std::make_shared<faabric::BatchExecuteRequest>();
    *ber->add_messages() = msg;
    chainedMessages[msg.id()] = ber;
}

const faabric::Message& Executor::getChainedMessage(int messageId)
{
    std::lock_guard<std::mutex> lk(chainedMx);
    auto it = chainedMessages.find(messageId);
    if (it == chainedMessages.end()) {
        SPDLOG_ERROR("Message {} does not have chained message {}", boundMessage.id(), messageId);
        throw ChainedCallException("Message does not have chained message " + std::to_string(messageId));
    }
    return it->second->messages(0);
}

std::set<unsigned int> Executor::getChainedMessageIds()
{
    std::lock_guard<std::mutex> lk(chainedMx);
    std::set<unsigned int> ids;
    for (const auto& [mid, ber] : chainedMessages) {
        ids.insert((unsigned int)mid);
    }
    return ids;
}

// ---- snapshots ----
std::shared_ptr<faabric::util::SnapshotData> Executor::getMainThreadSnapshot(
  faabric::Message& msg,
  bool createIfNotExists)
{
    std::string key = faabric::util::getMainThreadSnapshotKey(msg);
    bool exists = false;
    {
        std::shared_lock<std::shared_mutex> lock(threadExecutionMutex);
        exists = reg.snapshotExists(key);
    }
    if (!exists && createIfNotExists) {
        std::unique_lock<std::shared_mutex> lock(threadExecutionMutex);
        if (!reg.snapshotExists(key)) {
            SPDLOG_DEBUG("Creating main thread snapshot: {} for {}", key, faabric::util::funcToString(msg, false));
            std::span<uint8_t> mem = getMemoryView();
            auto snap = std::make_shared<faabric::util::SnapshotData>(
              std::span<const uint8_t>(mem.data(), mem.size()), getMaxMemorySize());
            reg.registerSnapshot(key, snap);
        }
    } else if (!exists) {
        SPDLOG_ERROR("No main thread snapshot {}", key);
        throw std::runtime_error("No main thread snapshot");
    }
    return reg.getSnapshot(key);
}

void Executor::deleteMainThreadSnapshot(const faabric::Message& msg)
{
    std::string key = faabric::util::getMainThreadSnapshotKey(msg);
    std::unique_lock<std::shared_mutex> lock(threadExecutionMutex);
    if (reg.snapshotExists(key)) {
        reg.deleteSnapshot(key);
    }
    if (reg.deviceSnapshotExists(key)) {
        reg.deleteDeviceSnapshot(key);
    }
}

std::shared_ptr<faabric::snapshot::DeviceSnapshot> Executor::getMainThreadDeviceSnapshot(
  faabric::Message& msg,
  bool createIfNotExists)
{
    std::string key = faabric::util::getMainThreadSnapshotKey(msg);
    std::unique_lock<std::shared_mutex> lock(threadExecutionMutex);
    if (reg.deviceSnapshotExists(key)) {
        return reg.getDeviceSnapshot(key);
    }
    if (!createIfNotExists) {
        SPDLOG_ERROR("No main thread device snapshot {}", key);
        throw std::runtime_error("No main thread device snapshot");
    }
    DeviceMemoryView dv = getDeviceMemoryView();
    if (dv.empty()) {
        throw std::runtime_error("Executor has no device memory view");
    }
    SPDLOG_DEBUG("Creating main thread device snapshot: {} ({} bytes on GPU {})", key, dv.size, dv.device);
    auto snap = std::make_shared<faabric::snapshot::DeviceSnapshot>(dv.size, dv.device);
    reg.registerDeviceSnapshot(key, snap);
    return snap;
}

// FAABRIC_THREADS_INCREMENTAL=0: every fork copies the whole image again
static bool incrementalDeviceThreads()
{
    static const bool on = []() {
        const char* v = getenv("FAABRIC_THREADS_INCREMENTAL");
        return v == nullptr || std::string(v) != "0";
    }();
    return on;
}

// Every host of a THREADS batch (the main one included) diffs against a PRIVATE
// copy of what it started from: the main image is being written by the other
// hosts' merge kernels while this host still runs.
void Executor::prepareDeviceThreads(const std::string& key, bool isMain)
{
    DeviceMemoryView dv = getDeviceMemoryView();
    auto mainSnap = reg.getDeviceSnapshot(key);
    GpuGuard g(dv.device);
    auto stream = (cudaStream_t)computeStream;
    if (!isMain && mainSnap->getSize() > dv.size) {
        setMemorySize(mainSnap->getSize());
        dv = getDeviceMemoryView();
    }
    const size_t n = std::min(dv.size, mainSnap->getSize());
    const bool baseFits = threadsBase != nullptr && threadsBase->getSize() == n && threadsBase->getDevice() == dv.device;
    // After the first fork this host's memory and base equal the image as of
    // their last synchronisation: only pages stamped since are copied
    const bool incremental = incrementalDeviceThreads() && mainSnap->pageStamps() != nullptr && baseFits &&
                             threadsSyncStamp != 0 && threadsSyncImageUid == mainSnap->uid() &&
                             threadsSyncStamp >= mainSnap->fullMutationStamp();
    const uint32_t forkStamp = mainSnap->currentForkStamp();
    if (incremental) {
        if (isMain) {
            // the main thread's memory was just folded into the image
            mainSnap->pullChangedPages(threadsBase->getDevicePtr(), nullptr, threadsSyncStamp, n, dv.device, stream);
        } else {
            mainSnap->pullChangedPages(dv.ptr, threadsBase->getDevicePtr(), threadsSyncStamp, n, dv.device, stream);
        }
    } else {
        if (!isMain) {
            mainSnap->restoreTo(dv.ptr, n, stream);
        }
        if (!baseFits) {
            threadsBase = std::make_shared<faabric::snapshot::DeviceSnapshot>(n, dv.device);
        }
        cudaCheck(cudaMemcpyAsync(threadsBase->getDevicePtr(), dv.ptr, n, cudaMemcpyDeviceToDevice, stream), "thread base copy");
    }
    threadsSyncStamp = forkStamp;
    threadsSyncImageUid = mainSnap->uid();
    threadsBase->clearMergeRegions();
    for (const auto& r : mainSnap->getMergeRegions()) {
        threadsBase->addMergeRegion(r.offset, r.length, r.dataType, r.operation);
    }
    cudaCheck(cudaStreamSynchronize(stream), "thread base sync");
    threadsMain = mainSnap;
}

uint64_t Executor::mergeDirtyRegionsOnDevice(const faabric::Message& msg)
{
    if (threadsBase == nullptr || threadsMain == nullptr) {
        throw std::runtime_error("No device thread state to merge");
    }
    DeviceMemoryView dv = getDeviceMemoryView();
    GpuGuard g(dv.device);
    auto stream = (cudaStream_t)computeStream;
    // scan + diff + typed merge + store into the (possibly remote) main image;
    // the pages changed there are stamped as "merged in this batch"
    if (incrementalDeviceThreads() && threadsMain->pageStamps() != nullptr) {
        threadsBase->setPushStamps(threadsMain->pageStamps(), threadsMain->currentForkStamp() + 1);
    } else {
        threadsBase->setPushStamps(nullptr, 0);
    }
    threadsBase->diffAndPush(dv.ptr, dv.size, threadsMain->getDevicePtr(), nullptr, false, stream);
    auto stats = threadsBase->getLastStats(stream); // synchronises: the merge has landed
    deviceMergeCount.fetch_add(1);
    lastDeviceDiffBytes.store(stats.diffBytes);
    SPDLOG_DEBUG("{} merged {} bytes ({} pages) of message {} into the main image on the device",
                 id,
                 stats.diffBytes,
                 stats.pagesWithDiffs,
                 msg.id());
    threadsMain = nullptr;
    return stats.diffBytes;
}

std::vector<faabric::util::SnapshotDiff> Executor::mergeDirtyRegions(
  const faabric::Message& msg,
  const std::vector<char>& extraDirtyPages)
{
    std::string key = faabric::util::getMainThreadSnapshotKey(msg);
    auto snap = reg.getSnapshot(key);
    std::span<uint8_t> memView = getMemoryView();
    tracker->stopTracking(memView);

    // Union of: pages dirtied by each thread, process-wide pages, caller extras
    faabric::util::mergeManyDirtyPages(dirtyRegions, threadLocalDirtyRegions);
    std::vector<char> global = tracker->getDirtyPages(memView);
    faabric::util::mergeDirtyPages(dirtyRegions, global);
    if (!extraDirtyPages.empty()) {
        faabric::util::mergeDirtyPages(dirtyRegions, extraDirtyPages);
    }
    // Whatever the app did not declare a merge op for is merged bytewise/xor
    snap->fillGapsWithBytewiseRegions();
    std::vector<faabric::util::SnapshotDiff> diffs = snap->diffWithDirtyRegions(memView, dirtyRegions);
    dirtyRegions.clear();
    threadLocalDirtyRegions.clear();
    return diffs;
}

// ---------------------------------------------------------------------------
// Running tasks
// ---------------------------------------------------------------------------
void Executor::executeTasks(std::vector<int> msgIdxs,
                            std::shared_ptr<faabric::BatchExecuteRequest> req,
                            std::function<void()> prelude)
{
    const int nMessages = (int)msgIdxs.size();
    touchLastExec();
    faabric::Message& first = *req->mutable_messages(msgIdxs.at(0));
    const bool isThreads = req->type() == faabric::BatchExecuteRequest::THREADS;
    const bool isSingleHost = req->singlehost();
    const std::string funcStr = faabric::util::funcToString(first, false);
    SPDLOG_TRACE("{} executing {}/{} tasks of {} (single-host={})", id, nMessages, req->messages_size(), funcStr, isSingleHost);

    if (isThreads && !isSingleHost) {
        // Remote threads start from the main thread's snapshot and track what
        // they change so it can be diffed and sent back
        std::string key = faabric::util::getMainThreadSnapshotKey(first);
        SPDLOG_DEBUG("Restoring {} from snapshot {} before executing {} threads", funcStr, key, nMessages);
        std::unique_lock<std::shared_mutex> lock(threadExecutionMutex);
        bool isMain = mainHostIsHere(first);
        if (!getDeviceMemoryView().empty() && reg.deviceSnapshotExists(key)) {
            // Device memory: restore is a (peer) device copy, change detection
            // is the fused compare-with-base kernel at merge time
            prepareDeviceThreads(key, isMain);
        } else {
            if (!isMain) {
                restore(key);
            }
            std::span<uint8_t> memView = getMemoryView();
            // (startTracking resets this region's record; clearAll would also
            // wipe the records of executors of other virtual hosts)
            tracker->startTracking(memView);
            threadLocalDirtyRegions.clear();
            dirtyRegions.clear();
        }
    } else if (!isThreads && !first.snapshotkey().empty()) {
        // A function resuming from a snapshot (migration / thaw)
        restore(first.snapshotkey());
    }

    currentAppId.store(first.appid());
    batchCounter.fetch_add(nMessages, std::memory_order_release);
    if (isThreads) {
        threadBatchCounter.fetch_add(nMessages, std::memory_order_release);
    }

    for (int msgIdx : msgIdxs) {
        int poolIdx = -1;
        bool ownsPoolThread = true;
        {
            // Functions and threads alike take a free pool thread (reference:
            // src/executor/Executor.cpp:182-203).  A thread must never queue
            // behind the function that forked it - that function is waiting
            // for it - so when the pool is oversubscribed (more threads than
            // cores) threads double up on pool threads that run threads only.
            std::lock_guard<std::mutex> lk(threadsMutex);
            if (!availablePoolThreads.empty()) {
                poolIdx = *availablePoolThreads.begin();
                availablePoolThreads.erase(availablePoolThreads.begin());
            } else if (isThreads) {
                ownsPoolThread = false;
                for (size_t k = 0; k < threadPoolSize; k++) {
                    int candidate = (int)((overloadCursor + k) % threadPoolSize);
                    if (functionPoolThreads.count(candidate) == 0) {
                        poolIdx = candidate;
                        overloadCursor = candidate + 1;
                        break;
                    }
                }
            }
            if (poolIdx < 0) {
                SPDLOG_ERROR("No available thread pool threads (size: {})", threadPoolSize);
                throw std::runtime_error("No available thread pool threads!");
            }
            if (!isThreads) {
                functionPoolThreads.insert(poolIdx);
            }
        }
        ExecutorTask task(msgIdx, req);
        task.ownsPoolThread = ownsPoolThread;
        if (prelude) {
            task.prelude = std::move(prelude);
            prelude = nullptr;
        }
        threadTaskQueues[poolIdx].enqueue(std::move(task));
        std::lock_guard<std::mutex> lk(threadsMutex);
        if (threadPoolThreads[poolIdx] == nullptr) {
            threadPoolThreads[poolIdx] = std::make_shared<std::jthread>(
              [this, poolIdx](std::stop_token st) { threadPoolThread(st, poolIdx); });
        }
    }
}

std::vector<std::pair<uint32_t, int32_t>> Executor::executeThreads(
  std::shared_ptr<faabric::BatchExecuteRequest> req,
  const std::vector<faabric::util::SnapshotMergeRegion>& mergeRegions)
{
    SPDLOG_DEBUG("Executor {} executing {} threads", id, req->messages_size());
    faabric::Message& msg = *req->mutable_messages(0);
    std::string key = faabric::util::getMainThreadSnapshotKey(msg);
    // The main host of the threads is the (virtual) host this executor serves
    std::string myHost = boundMessage.executedhost();
    if (ExecutorContext::isSet() && ExecutorContext::get()->getExecutor() == this) {
        myHost = ExecutorContext::get()->getMsg().executedhost();
    }
    if (faabric::transport::isHostAlias(myHost)) {
        for (int i = 0; i < req->messages_size(); i++) {
            req->mutable_messages(i)->set_mainhost(myHost);
        }
    }
    DeviceMemoryView dv = getDeviceMemoryView();
    if (!dv.empty()) {
        // ---- device-resident fork-join ----
        auto snap = getMainThreadDeviceSnapshot(msg, true);
        const size_t nImage = std::min(dv.size, snap->getSize());
        const bool incremental = incrementalDeviceThreads() && snap->pageStamps() != nullptr;
        const uint32_t forkStamp = snap->beginFork();
        {
            // The main thread is authoritative: bring the image up to date.
            // Incrementally: compare, copy the pages that differ and stamp them
            // (two reads of the image's size, writes only where needed)
            GpuGuard g(dv.device);
            auto stream = (cudaStream_t)computeStream;
            if (incremental) {
                snap->syncPagesFrom(dv.ptr, nImage, forkStamp, stream);
            } else {
                cudaCheck(cudaMemcpyAsync(snap->getDevicePtr(), dv.ptr, nImage, cudaMemcpyDeviceToDevice, stream), "main image refresh");
                snap->markRewritten();
            }
            cudaCheck(cudaStreamSynchronize(stream), "main image refresh sync");
        }
        snap->clearMergeRegions();
        for (const auto& r : mergeRegions) {
            snap->addMergeRegion(r.offset, r.length, r.dataType, r.operation);
        }
        req->set_type(faabric::BatchExecuteRequest::THREADS);
        auto decision = faabric::planner::getPlannerClient().callFunctions(req);
        if ((int)decision.appId == NOT_ENOUGH_SLOTS) {
            throw std::runtime_error("Not enough slots to execute threads");
        }
        auto results = faabric::scheduler::getScheduler().awaitThreadResults(req);
        if (!decision.isSingleHost()) {
            // every host's merge kernel has completed before its result was
            // published: the image now holds the merged state.  Hosts served by
            // another process cannot stamp the pages they merged
            bool allHere = true;
            for (const auto& h : decision.hosts) {
                allHere = allHere && faabric::transport::MessageEndpointServer::localServerFor(h, FUNCTION_CALL_ASYNC_PORT, false) != nullptr;
            }
            GpuGuard g(dv.device);
            auto stream = (cudaStream_t)computeStream;
            if (incremental && allHere) {
                snap->pullChangedPages(dv.ptr, nullptr, forkStamp, nImage, dv.device, stream);
            } else {
                if (!allHere) {
                    snap->markRewritten();
                }
                snap->restoreTo(dv.ptr, nImage, stream);
            }
            cudaCheck(cudaStreamSynchronize(stream), "merged image restore");
        }
        return results;
    }
    bool existed = reg.snapshotExists(key);
    auto snap = getMainThreadSnapshot(msg, true);
    std::span<uint8_t> memView = getMemoryView();

    if (existed) {
        // Bring the snapshot up to date with what the main thread did since
        tracker->stopTracking(memView);
        tracker->stopThreadLocalTracking(memView);
        std::vector<char> dirty = tracker->getBothDirtyPages(memView);
        snap->clearMergeRegions();
        snap->fillGapsWithBytewiseRegions();
        auto updates = snap->diffWithDirtyRegions(memView, dirty);
        if (!updates.empty()) {
            snap->applyDiffs(updates);
        }
        snap->clearMergeRegions();
    }
    for (const auto& r : mergeRegions) {
        snap->addMergeRegion(r.offset, r.length, r.dataType, r.operation);
    }

    req->set_type(faabric::BatchExecuteRequest::THREADS);
    auto decision = faabric::planner::getPlannerClient().callFunctions(req);
    if ((int)decision.appId == NOT_ENOUGH_SLOTS) {
        throw std::runtime_error("Not enough slots to execute threads");
    }
    auto results = faabric::scheduler::getScheduler().awaitThreadResults(req);

    // Fold the threads' diffs into the snapshot and refresh our memory from it
    int nWritten = snap->writeQueuedDiffs();
    SPDLOG_DEBUG("Merged {} thread diffs into {}", nWritten, key);
    if (nWritten > 0 || !decision.isSingleHost()) {
        std::span<uint8_t> view = getMemoryView();
        snap->mapToMemory({ view.data(), std::min(view.size(), snap->getSize()) });
    }
    tracker->startTracking(getMemoryView());
    tracker->startThreadLocalTracking(getMemoryView());
    return results;
}

void Executor::setThreadResult(faabric::Message& msg,
                               int32_t returnValue,
                               const std::string& key,
                               const std::vector<faabric::util::SnapshotDiff>& diffs)
{
    if (mainHostIsHere(msg)) {
        if (!diffs.empty()) {
            // (the diffs point into executor memory, which outlives the merge)
            SPDLOG_DEBUG("Queueing {} diffs for {} to snapshot {}", diffs.size(), faabric::util::funcToString(msg, false), key);
            reg.getSnapshot(key)->queueDiffs(diffs);
        }
    } else {
        // result and diffs travel to the main host together
        faabric::snapshot::getSnapshotClient(msg.mainhost())->pushThreadResult(msg.appid(), msg.id(), returnValue, key, diffs);
    }
    faabric::planner::getPlannerClient().setMessageResult(std::make_shared<faabric::Message>(msg));
}

void Executor::threadPoolThread(std::stop_token st, int threadPoolIdx)
{
    SPDLOG_DEBUG("Thread pool thread {}:{} starting up", id, threadPoolIdx);
    auto& sch = faabric::scheduler::getScheduler();
    faabric::transport::PointToPointBroker& broker = faabric::transport::getPointToPointBroker();
    // (read once: tests reset the configuration while pool threads idle)
    const int boundTimeout = faabric::util::getSystemConfig().boundTimeout;
    faabric::util::bindThreadToGpu(gpuIdx);

    while (!st.stop_requested()) {
        ExecutorTask task;
        try {
            task = threadTaskQueues[threadPoolIdx].dequeue(boundTimeout);
        } catch (const faabric::util::QueueTimeoutException&) {
            // Nothing to do for a while: keep waiting, the reaper decides
            // when the whole executor goes away
            continue;
        }
        if (task.messageIndex == POOL_SHUTDOWN) {
            SPDLOG_DEBUG("Killing thread pool thread {}:{}", id, threadPoolIdx);
            break;
        }
        if (task.prelude) {
            try {
                task.prelude();
            } catch (const std::exception& ex) {
                SPDLOG_ERROR("Launching the rest of a batch from {} failed: {}", id, ex.what());
            }
            task.prelude = nullptr;
        }
        auto req = task.req;
        faabric::Message& msg = *req->mutable_messages(task.messageIndex);
        const bool isThreads = req->type() == faabric::BatchExecuteRequest::THREADS;
        const bool isMigration = req->type() == faabric::BatchExecuteRequest::MIGRATION;
        const bool deviceThreads = isThreads && !req->singlehost() && threadsBase != nullptr && threadsMain != nullptr;
        const bool doDirtyTracking = isThreads && !req->singlehost() && !deviceThreads;
        if (doDirtyTracking) {
            tracker->startThreadLocalTracking(getMemoryView());
        }

        ExecutorContext::set(this, req, task.messageIndex);
        int32_t returnValue = 0;
        bool migrated = false;
        bool frozen = false;
        try {
            if (isMigration) {
                // Everyone in the new group lines up before the app carries on
                broker.postMigrationHook(msg.groupid(), msg.groupidx());
            }
            returnValue = executeTask(threadPoolIdx, task.messageIndex, req);
        } catch (const faabric::util::FunctionMigratedException& ex) {
            SPDLOG_DEBUG("Task {} migrated, shutting down executor {}", msg.id(), id);
            returnValue = MIGRATED_FUNCTION_RETURN_VALUE;
            migrated = true;
        } catch (const faabric::util::FunctionFrozenException& ex) {
            SPDLOG_DEBUG("Task {} frozen, shutting down executor {}", msg.id(), id);
            returnValue = FROZEN_FUNCTION_RETURN_VALUE;
            frozen = true;
        } catch (const std::exception& ex) {
            returnValue = 1;
            std::string err = "Task " + std::to_string(msg.id()) + " threw exception. What: " + ex.what();
            SPDLOG_ERROR("{}", err);
            msg.set_outputdata(err);
        }
        if ((migrated || frozen || returnValue == 1) && msg.ismpi()) {
            // The rank is gone from this host: drop our view of its world
            auto& worlds = faabric::mpi::getMpiWorldRegistry();
            if (worlds.worldExists(msg.mpiworldid())) {
                bool mustClear = worlds.getWorld(msg.mpiworldid()).destroy();
                if (mustClear) {
                    worlds.clearWorld(msg.mpiworldid());
                }
            }
        }
        ExecutorContext::unset();
        msg.set_returnvalue(returnValue);

        if (doDirtyTracking) {
            tracker->stopThreadLocalTracking(getMemoryView());
            std::vector<char> mine = tracker->getThreadLocalDirtyPages(getMemoryView());
            std::unique_lock<std::shared_mutex> lock(threadExecutionMutex);
            threadLocalDirtyRegions.push_back(std::move(mine));
        }

        // Counters decide who tidies up
        int oldThreadCount = isThreads ? threadBatchCounter.fetch_sub(1, std::memory_order_acq_rel) : 0;
        bool isLastThreadInBatch = isThreads && oldThreadCount == 1;
        int oldBatchCount = batchCounter.fetch_sub(1, std::memory_order_acq_rel);
        bool isLastInBatch = oldBatchCount == 1;

        // The last thread diffs this host's memory against the snapshot
        std::vector<faabric::util::SnapshotDiff> diffs;
        bool deviceMerged = false;
        uint64_t deviceDiffBytes = 0;
        if (isLastThreadInBatch && deviceThreads) {
            try {
                std::unique_lock<std::shared_mutex> lock(threadExecutionMutex);
                deviceDiffBytes = mergeDirtyRegionsOnDevice(msg);
                deviceMerged = true;
            } catch (const std::exception& ex) {
                SPDLOG_ERROR("Failed merging device memory for {}: {}", msg.id(), ex.what());
            }
        }
        if (isLastThreadInBatch && doDirtyTracking) {
            try {
                std::unique_lock<std::shared_mutex> lock(threadExecutionMutex);
                diffs = mergeDirtyRegions(msg);
            } catch (const std::exception& ex) {
                SPDLOG_ERROR("Failed merging dirty regions for {}: {}", msg.id(), ex.what());
            }
        }

        // Release resources BEFORE publishing the result: once the result is
        // out the caller may immediately schedule onto this executor again
        if (isLastInBatch) {
            if (!isThreads) {
                try {
                    reset(msg);
                } catch (const std::exception& ex) {
                    SPDLOG_ERROR("Error resetting executor {}: {}", id, ex.what());
                }
            }
            touchLastExec();
            currentAppId.store(0);
            releaseClaim();
        }
        if (task.ownsPoolThread) {
            std::lock_guard<std::mutex> lk(threadsMutex);
            availablePoolThreads.insert(threadPoolIdx);
            functionPoolThreads.erase(threadPoolIdx);
        }

        msg.set_finishtimestamp(faabric::util::getGlobalClock().epochMillis());
        if (isThreads && deviceMerged && !mainHostIsHere(msg)) {
            // the bytes are already in the main image: control message only
            faabric::snapshot::getSnapshotClient(msg.mainhost())
              ->pushDeviceThreadResult(msg.appid(), msg.id(), returnValue, faabric::util::getMainThreadSnapshotKey(msg), deviceDiffBytes);
            faabric::planner::getPlannerClient().setMessageResult(std::make_shared<faabric::Message>(msg));
        } else if (isThreads) {
            // only the last thread of a host's batch carries the diffs
            std::string key = (!diffs.empty() || isLastThreadInBatch) ? faabric::util::getMainThreadSnapshotKey(msg) : "";
            setThreadResult(msg, returnValue, key, diffs);
        } else {
            faabric::planner::getPlannerClient().setMessageResult(std::make_shared<faabric::Message>(msg));
        }
    }
    // Thread-local caches die with the thread
    sch.resetThreadLocalCache();
    broker.resetThreadLocalCache();
}

// ---------------------------------------------------------------------------
// DeviceExecutor
// ---------------------------------------------------------------------------
DeviceExecutor::DeviceExecutor(faabric::Message& msg, size_t initialSize, size_t maxSizeIn)
  : Executor(msg)
  , currentSize(initialSize)
  , maxSize(std::max(initialSize, maxSizeIn))
{
    if (getGpuIdx() < 0) {
        throw std::runtime_error("DeviceExecutor needs a GPU");
    }
    // Reserve the maximum up front (one device allocation, 80 GB of HBM on an H100), expose
    // `currentSize` of it, like the reference's virtual reservation + mprotect
    memory = faabric::util::allocateDeviceMemory(maxSize, getGpuIdx());
    GpuGuard g(getGpuIdx());
    cudaCheck(cudaMemset(memory.ptr, 0, maxSize), "device executor memset");
}

DeviceExecutor::~DeviceExecutor() = default;

DeviceMemoryView DeviceExecutor::getDeviceMemoryView()
{
    return { memory.ptr, currentSize, getGpuIdx() };
}

void DeviceExecutor::setMemorySize(size_t newSize)
{
    if (newSize > maxSize) {
        throw std::runtime_error("Device executor memory beyond its maximum");
    }
    currentSize = newSize;
}

} // namespace faabric::executor
