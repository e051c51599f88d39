// Executors: thread pools that run the messages of a batch.
//
// One header per module: the per-class headers of the reference's layout
// (faabric/executor/*.h) forward here, so either include style works.
#pragma once

#include <faabric/proto/faabric.pb.h>
#include <faabric/snapshot/SnapshotRegistry.h>
#include <faabric/util/clock.h>
#include <faabric/util/dirty.h>
#include <faabric/util/exception.h>
#include <faabric/util/hwloc.h>
#include <faabric/util/queue.h>
#include <faabric/util/snapshot.h>

#include <atomic>
#include <memory>
#include <mutex>
#include <set>
#include <shared_mutex>
#include <span>
#include <stdexcept>
#include <thread>
#include <vector>

// ==========================================================================
// executor/ExecutorTask.h
// ==========================================================================
namespace faabric::executor {

class ExecutorTask
{
  public:
    ExecutorTask() = default;

    ExecutorTask(int messageIndexIn,
                 std::shared_ptr<faabric::BatchExecuteRequest> reqIn)
      : req(std::move(reqIn))
      , messageIndex(messageIndexIn)
    {}

    // Shutdown sentinel for pool threads
    static const int POOL_SHUTDOWN = -1;

    std::shared_ptr<faabric::BatchExecuteRequest> req;
    int messageIndex = 0;
    // Run by the pool thread before the task itself: the scheduler uses it to
    // spread the launch of a wide batch over the threads it has already woken
    std::function<void()> prelude;
    // False for a thread that had to share an already busy pool thread
    bool ownsPoolThread = true;
};

}

// ==========================================================================
// executor/Executor.h
// ==========================================================================
// Executor: a warm container for one (user, function, app) that runs the
// messages of a batch on a pool of threads.  Users subclass it and implement
// executeTask (reference: include/faabric/executor/Executor.h:21-118,
// src/executor/Executor.cpp:38-743).  Additions for GPUs: every executor is
// bound to a GPU (device id + compute stream) and may expose a device memory
// view that is snapshot / restored / diff-pushed with the device kernels.



#define POOL_SHUTDOWN -1

namespace faabric::executor {

class ChainedCallException : public faabric::util::FaabricException
{
  public:
    explicit ChainedCallException(std::string message)
      : FaabricException(std::move(message))
    {}
};

// Function memory that lives in HBM (GPU): executors that return a non-empty
// view take the device paths of restore / THREADS fork-join, where the
// snapshot image, the per-host base image and the merge all stay on the GPUs
struct DeviceMemoryView
{
    uint8_t* ptr = nullptr;
    size_t size = 0;
    int device = -1;

    bool empty() const { return ptr == nullptr || size == 0; }
};

class Executor : public std::enable_shared_from_this<Executor>
{
  public:
    std::string id;

    explicit Executor(faabric::Message& msg);

    virtual ~Executor();

    // Must be called before the executor is destroyed
    void shutdown();

    std::vector<std::pair<uint32_t, int32_t>> executeThreads(
      std::shared_ptr<faabric::BatchExecuteRequest> req,
      const std::vector<faabric::util::SnapshotMergeRegion>& mergeRegions);

    void executeTasks(std::vector<int> msgIdxs,
                      std::shared_ptr<faabric::BatchExecuteRequest> req,
                      std::function<void()> prelude = nullptr);

    // Publishes the result of one thread of a THREADS batch: the diffs are
    // queued on the main-thread snapshot when the main host is served here,
    // pushed to it together with the result otherwise; then the message result
    // goes to the planner (reference: src/executor/Executor.cpp:271-305)
    void setThreadResult(faabric::Message& msg,
                         int32_t returnValue,
                         const std::string& key,
                         const std::vector<faabric::util::SnapshotDiff>& diffs);

    // ---- hooks for subclasses ----
    virtual void reset(faabric::Message& msg);

    virtual int32_t executeTask(
      int threadPoolIdx,
      int msgIdx,
      std::shared_ptr<faabric::BatchExecuteRequest> req);

    virtual std::span<uint8_t> getMemoryView();

    // Device-resident function memory (default: none => host paths)
    virtual DeviceMemoryView getDeviceMemoryView();

    virtual void restore(const std::string& snapshotKey);

    virtual void setMemorySize(size_t newSize);

    virtual size_t getMaxMemorySize();

    // ---- GPU binding ----
    // App this executor is currently working for (0 when idle)
    int getCurrentAppId() const { return currentAppId.load(); }

    int getGpuIdx() const { return gpuIdx; }

    // Compute stream of this executor (cudaStream_t); nullptr without a GPU
    void* getComputeStream() const { return computeStream; }

    // ---- claiming ----
    bool tryClaim();

    void claim();

    void releaseClaim();

    bool isExecuting();

    bool isShutdown() { return _isShutdown; }

    long getMillisSinceLastExec();

    std::shared_ptr<faabric::util::SnapshotData> getMainThreadSnapshot(
      faabric::Message& msg,
      bool createIfNotExists = false);

    // ---- chained calls ----
    void addChainedMessage(const faabric::Message& msg);

    const faabric::Message& getChainedMessage(int messageId);

    std::set<unsigned int> getChainedMessageIds();

    std::vector<faabric::util::SnapshotDiff> mergeDirtyRegions(
      const faabric::Message& msg,
      const std::vector<char>& extraDirtyPages = {});

    // Device flavour of mergeDirtyRegions: ONE fused kernel diffs this
    // executor's HBM memory against its private base image, applies the merge
    // regions and stores the result straight into the main image (local or a
    // peer GPU's memory).  Returns the number of bytes merged.
    uint64_t mergeDirtyRegionsOnDevice(const faabric::Message& msg);

    // Device-resident main-thread snapshot (created from the device memory
    // view on first use)
    std::shared_ptr<faabric::snapshot::DeviceSnapshot> getMainThreadDeviceSnapshot(
      faabric::Message& msg,
      bool createIfNotExists = false);

    uint64_t getDeviceMergeCount() const { return deviceMergeCount.load(); }

    // The message this executor was created for
    faabric::Message& getBoundMessage() { return boundMessage; }

    std::string schedulerKey;

    // Incremental device THREADS: the stamp of the main image this executor's
    // memory and private base were last identical to (0 = never), and which
    // image that was
    uint32_t threadsSyncStamp = 0;
    uint64_t threadsSyncImageUid = 0;

    uint64_t getLastDeviceDiffBytes() const { return lastDeviceDiffBytes.load(); }

    // Blocks until every pool thread finished (tests)
    void joinThreadPool();

  protected:
    virtual void setUpThreadPool();

    faabric::Message boundMessage;

    faabric::snapshot::SnapshotRegistry& reg;

    std::shared_ptr<faabric::util::DirtyTracker> tracker;

    uint32_t threadPoolSize = 0;

    std::map<int, std::shared_ptr<faabric::BatchExecuteRequest>> chainedMessages;

  private:
    std::atomic<bool> claimed = false;

    std::atomic<bool> _isShutdown = false;

    std::atomic<int> batchCounter = 0;
    std::atomic<int> currentAppId = 0;

    std::atomic<int> threadBatchCounter = 0;

    // (steady-clock nanoseconds; written by pool threads, read by the reaper)
    std::atomic<int64_t> lastExecNs{ 0 };
    void touchLastExec();

    // ---- Application threads ----
    std::shared_mutex threadExecutionMutex;
    std::vector<char> dirtyRegions;
    std::vector<std::vector<char>> threadLocalDirtyRegions;
    void deleteMainThreadSnapshot(const faabric::Message& msg);

    // ---- Function execution thread pool ----
    std::mutex threadsMutex;
    std::vector<std::shared_ptr<std::jthread>> threadPoolThreads;
    std::set<int> availablePoolThreads;
    // Pool threads running a function (which may block on its own threads):
    // never shared with thread tasks when the pool is oversubscribed
    std::set<int> functionPoolThreads;
    int overloadCursor = 0;

    std::vector<faabric::util::Queue<ExecutorTask>> threadTaskQueues;

    std::mutex chainedMx;

    int gpuIdx = -1;
    void* computeStream = nullptr;

    // THREADS on device memory: private base image of this host's copy and the
    // main image the merge is pushed into
    std::shared_ptr<faabric::snapshot::DeviceSnapshot> threadsBase;
    std::shared_ptr<faabric::snapshot::DeviceSnapshot> threadsMain;
    std::atomic<uint64_t> deviceMergeCount = 0;
    std::atomic<uint64_t> lastDeviceDiffBytes = 0;

    void prepareDeviceThreads(const std::string& key, bool isMain);

    void stopPoolThreads();

    void threadPoolThread(std::stop_token st, int threadPoolIdx);
};

}

namespace faabric::executor {

// Ready-made executor whose function memory is a growable HBM allocation on
// the GPU the executor is bound to (reference analogue: the memory an embedder
// such as Faasm hands out through getMemoryView, here device-resident).
// Subclasses implement executeTask and work on getDeviceMemoryView().
class DeviceExecutor : public Executor
{
  public:
    DeviceExecutor(faabric::Message& msg, size_t initialSize, size_t maxSize);

    ~DeviceExecutor() override;

    DeviceMemoryView getDeviceMemoryView() override;

    void setMemorySize(size_t newSize) override;

    size_t getMaxMemorySize() override { return maxSize; }

  private:
    faabric::util::DeviceRegion memory;
    size_t currentSize = 0;
    size_t maxSize = 0;
};

}

// ==========================================================================
// executor/ExecutorContext.h
// ==========================================================================
namespace faabric::executor {

class Executor;

class ExecutorContextException : public std::runtime_error
{
  public:
    explicit ExecutorContextException(const std::string& message)
      : std::runtime_error(message)
    {}
};

// Thread-local handle on "what am I executing": set around executeTask so
// library code (MPI shim, chaining, state) can find the current message
class ExecutorContext
{
  public:
    ExecutorContext(Executor* executorIn,
                    std::shared_ptr<faabric::BatchExecuteRequest> reqIn,
                    int msgIdx);

    static bool isSet();

    static void set(Executor* executorIn,
                    std::shared_ptr<faabric::BatchExecuteRequest> reqIn,
                    int msgIdxIn);

    static void unset();

    static std::shared_ptr<ExecutorContext> get();

    Executor* getExecutor() { return executor; }

    std::shared_ptr<faabric::BatchExecuteRequest> getBatchRequest()
    {
        return req;
    }

    faabric::Message& getMsg()
    {
        if (req == nullptr) {
            throw ExecutorContextException("Getting message when no request set in context");
        }
        return *req->mutable_messages(msgIdx);
    }

    int getMsgIdx() const { return msgIdx; }

  private:
    Executor* executor = nullptr;
    std::shared_ptr<faabric::BatchExecuteRequest> req = nullptr;
    int msgIdx = 0;
};

}

// ==========================================================================
// executor/ExecutorFactory.h
// ==========================================================================
namespace faabric::executor {

class ExecutorFactory
{
  public:
    virtual ~ExecutorFactory() = default;

    virtual std::shared_ptr<Executor> createExecutor(faabric::Message& msg) = 0;

    virtual void flushHost();
};

void setExecutorFactory(std::shared_ptr<ExecutorFactory> fac);

std::shared_ptr<ExecutorFactory> getExecutorFactory();

}

