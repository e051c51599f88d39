// Utilities.
//
// One header per module: the per-class headers of the reference's layout
// (faabric/util/*.h) forward here, so either include style works.
#pragma once

#include <faabric/proto/faabric.pb.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <deque>
#include <functional>
#include <initializer_list>
#include <map>
#include <memory>
#include <mutex>
#include <optional>
#include <pthread.h>
#include <queue>
#include <sched.h>
#include <set>
#include <shared_mutex>
#include <span>
#include <sstream>
#include <stdexcept>
#include <string>
#include <string_view>
#include <thread>
#include <unistd.h>
#include <unordered_map>
#include <utility>
#include <unordered_set>
#include <vector>

// ==========================================================================
// util/exception.h
// ==========================================================================
namespace faabric::util {

class FaabricException : public std::runtime_error
{
  public:
    explicit FaabricException(const std::string& message)
      : std::runtime_error(message)
    {}
};

// Thrown by an executing function when the planner told it to move elsewhere
// (reference: include/faabric/util/func.h + scheduler migration path)
class FunctionMigratedException : public FaabricException
{
  public:
    explicit FunctionMigratedException(const std::string& message)
      : FaabricException(message)
    {}
};

// Thrown when an app must be check-pointed and parked (spot eviction)
class FunctionFrozenException : public FaabricException
{
  public:
    explicit FunctionFrozenException(const std::string& message)
      : FaabricException(message)
    {}
};

} // namespace faabric::util

// ==========================================================================
// util/ExecGraph.h
// ==========================================================================
// Execution graph of chained function calls (reference:
// include/faabric/util/ExecGraph.h:8-60, src/util/ExecGraph.cpp).  The graph
// is rebuilt on demand from message results held by the planner.



namespace faabric::util {

class ExecGraphNodeNotFoundException : public FaabricException
{
  public:
    explicit ExecGraphNodeNotFoundException(std::string message)
      : FaabricException(std::move(message))
    {}
};

struct ExecGraphNode
{
    faabric::Message msg;
    std::vector<ExecGraphNode> children;
};

struct ExecGraph
{
    ExecGraphNode rootNode;
};

ExecGraphNode getFunctionExecGraphNode(int appId, int msgId);

ExecGraph getFunctionExecGraph(const faabric::Message& msg);

void logChainedFunction(faabric::Message& parentMessage, const faabric::Message& chainedMessage);

std::set<unsigned int> getChainedFunctions(const faabric::Message& msg);

int countExecGraphNodes(const ExecGraph& graph);

std::set<std::string> getExecGraphHosts(const ExecGraph& graph);

std::vector<std::string> getMpiRankHostsFromExecGraph(const ExecGraph& graph);

// (hosts before migration, hosts after migration), indexed by rank
std::pair<std::vector<std::string>, std::vector<std::string>> getMigratedMpiRankHostsFromExecGraph(
  const ExecGraph& graph);

std::string execNodeToJson(const ExecGraphNode& node);

std::string execGraphToJson(const ExecGraph& graph);

void addDetail(faabric::Message& msg, const std::string& key, const std::string& value);

void incrementCounter(faabric::Message& msg, const std::string& key, int valueToIncrement = 1);

}

// ==========================================================================
// util/PeriodicBackgroundThread.h
// ==========================================================================
namespace faabric::util {

// Runs doWork() every `intervalSeconds` on its own thread until stop()
#define DEFAULT_BACKGROUND_INTERVAL_SECONDS 30

class PeriodicBackgroundThread
{
  public:
    virtual ~PeriodicBackgroundThread();

    void start(int intervalSecondsIn);

    // Millisecond resolution variant (used by tests and the keep-alive)
    void startMs(int intervalMsIn);

    void stop();

    virtual void doWork() = 0;

    int getIntervalSeconds() const { return intervalMs / 1000; }

    // Hook called once on the worker thread when it exits
    virtual void tidyUp();

  private:
    std::unique_ptr<std::jthread> workThread;
    std::mutex mx;
    std::condition_variable_any timeoutCv;
    int intervalMs = 0;
};

}

// ==========================================================================
// util/barrier.h
// ==========================================================================
#define DEFAULT_BARRIER_TIMEOUT_MS 10000

namespace faabric::util {

// Reusable (cyclic) thread barrier with a completion hook and timeout
class Barrier
{
  public:
    static std::shared_ptr<Barrier> create(
      int count,
      std::function<void()> completionFunction = []() {},
      int timeoutMs = DEFAULT_BARRIER_TIMEOUT_MS);

    explicit Barrier(int countIn,
                     std::function<void()> completionFunctionIn,
                     int timeoutMsIn);

    void wait();

  private:
    int count;
    int arrived = 0;
    uint64_t generation = 0;
    std::function<void()> completionFunction;
    int timeoutMs;
    std::mutex mx;
    std::condition_variable cv;
};

}

// ==========================================================================
// util/batch.h
// ==========================================================================
namespace faabric::util {

// ----------
// Batch execute requests (BER)
// ----------
std::shared_ptr<faabric::BatchExecuteRequest> batchExecFactory();

std::shared_ptr<faabric::BatchExecuteRequest> batchExecFactory(
  const std::string& user,
  const std::string& function,
  int count = 1);

bool isBatchExecRequestValid(std::shared_ptr<faabric::BatchExecuteRequest> ber);

// Results of a status that are final (migrated messages will report again)
int getNumFinishedMessagesInBatch(std::shared_ptr<faabric::BatchExecuteRequestStatus> berStatus);

void updateBatchExecAppId(std::shared_ptr<faabric::BatchExecuteRequest> ber,
                          int newAppId);

void updateBatchExecGroupId(std::shared_ptr<faabric::BatchExecuteRequest> ber,
                            int newGroupId);

// ----------
// Batch execute request status
// ----------
std::shared_ptr<faabric::BatchExecuteRequestStatus> batchExecStatusFactory(
  int32_t appId);

std::shared_ptr<faabric::BatchExecuteRequestStatus> batchExecStatusFactory(
  std::shared_ptr<faabric::BatchExecuteRequest> ber);

}

// ==========================================================================
// util/bytes.h
// ==========================================================================
namespace faabric::util {

std::vector<uint8_t> stringToBytes(const std::string& str);

// The int stored in exactly sizeof(int) bytes
int bytesToInt(const std::vector<uint8_t>& bytes);

std::string bytesToString(const std::vector<uint8_t>& bytes);

std::string formatByteArrayToIntString(const std::vector<uint8_t>& bytes);

void trimTrailingZeros(std::vector<uint8_t>& vectorIn);

// Copy a string into a fixed byte buffer, failing if it does not fit
int safeCopyToBuffer(const std::vector<uint8_t>& dataIn,
                     uint8_t* buffer,
                     int bufferLen);

int safeCopyToBuffer(const uint8_t* dataIn,
                     int dataLen,
                     uint8_t* buffer,
                     int bufferLen);

std::string byteArrayToHexString(const uint8_t* data, int dataSize);

// Zero-padded hex of an integer, two digits per byte of T
template<typename T>
std::string intToHexString(T i)
{
    static const char* digits = "0123456789abcdef";
    std::string out(sizeof(T) * 2, '0');
    auto v = (unsigned long long)i;
    if constexpr (sizeof(T) < sizeof(unsigned long long)) {
        v &= (1ull << (8 * sizeof(T))) - 1;
    }
    for (size_t k = 0; k < sizeof(T) * 2; k++) {
        out[sizeof(T) * 2 - 1 - k] = digits[v & 0xf];
        v >>= 4;
    }
    return out;
}

// Appends the object representation of `value`
template<class T>
void appendBytesOf(std::vector<uint8_t>& container, T value)
{
    const uint8_t* start = reinterpret_cast<const uint8_t*>(&value);
    container.insert(container.end(), start, start + sizeof(T));
}

std::vector<uint8_t> hexStringToByteArray(const std::string& hexString);

template<typename T>
T unalignedRead(const uint8_t* bytes)
{
    T value;
    std::memcpy(&value, bytes, sizeof(T));
    return value;
}

template<typename T>
void unalignedWrite(const T& value, uint8_t* destination)
{
    std::memcpy(destination, &value, sizeof(T));
}

template<typename T>
std::vector<uint8_t> valueToBytes(T val)
{
    std::vector<uint8_t> out(sizeof(T));
    std::memcpy(out.data(), &val, sizeof(T));
    return out;
}

template<typename T>
size_t appendDataToBytes(std::vector<uint8_t>& bytes, const T& val)
{
    size_t before = bytes.size();
    bytes.resize(before + sizeof(T));
    std::memcpy(bytes.data() + before, &val, sizeof(T));
    return bytes.size();
}

template<typename T>
size_t readBytesOf(const std::vector<uint8_t>& container, size_t offset, T* out)
{
    if (offset + sizeof(T) > container.size()) {
        throw std::range_error("readBytesOf past end of buffer");
    }
    std::memcpy(out, container.data() + offset, sizeof(T));
    return offset + sizeof(T);
}

} // namespace faabric::util

// ==========================================================================
// util/clock.h
// ==========================================================================
namespace faabric::util {

using TimePoint = std::chrono::steady_clock::time_point;

class Clock
{
  public:
    Clock() = default;

    TimePoint now() const { return std::chrono::steady_clock::now(); }

    // Wall-clock milliseconds since the Unix epoch (message timestamps)
    long epochMillis() const
    {
        return (long)std::chrono::duration_cast<std::chrono::milliseconds>(
                 std::chrono::system_clock::now().time_since_epoch())
          .count();
    }

    long epochMicros() const
    {
        return (long)std::chrono::duration_cast<std::chrono::microseconds>(
                 std::chrono::system_clock::now().time_since_epoch())
          .count();
    }

    long timeDiff(const TimePoint& t1, const TimePoint& t2) const
    {
        return (long)std::chrono::duration_cast<std::chrono::milliseconds>(t1 -
                                                                           t2)
          .count();
    }

    long timeDiffMicro(const TimePoint& t1, const TimePoint& t2) const
    {
        return (long)std::chrono::duration_cast<std::chrono::microseconds>(t1 -
                                                                           t2)
          .count();
    }

    long timeDiffNano(const TimePoint& t1, const TimePoint& t2) const
    {
        return (long)std::chrono::duration_cast<std::chrono::nanoseconds>(t1 -
                                                                          t2)
          .count();
    }
};

Clock& getGlobalClock();

} // namespace faabric::util

// ==========================================================================
// util/compare.h
// ==========================================================================
namespace faabric::util {

// Element-wise equality of two arrays (reference: include/faabric/util/compare.h)
template<typename T>
bool compareArrays(const T* v1, const T* v2, size_t size)
{
    for (size_t i = 0; i < size; i++) {
        if (!(v1[i] == v2[i])) {
            return false;
        }
    }
    return true;
}

}

// ==========================================================================
// util/locks.h
// ==========================================================================
#define DEFAULT_FLAG_WAIT_MS 10000

namespace faabric::util {

typedef std::unique_lock<std::mutex> UniqueLock;
typedef std::unique_lock<std::shared_mutex> FullLock;
typedef std::shared_lock<std::shared_mutex> SharedLock;

// One-shot flag several threads can block on (with timeout)
class FlagWaiter : public std::enable_shared_from_this<FlagWaiter>
{
  public:
    explicit FlagWaiter(int timeoutMsIn = DEFAULT_FLAG_WAIT_MS);

    // Throws std::runtime_error on timeout
    void waitOnFlag();

    void setFlag(bool value);

  private:
    int timeoutMs;
    std::mutex flagMx;
    std::condition_variable cv;
    std::atomic<bool> flag = false;
};

}

// ==========================================================================
// util/concurrent_map.h
// ==========================================================================
// shared_mutex-protected hash map with the closure-based access API of the
// reference's ConcurrentMap (include/faabric/util/concurrent_map.h:39-304).



namespace faabric::util {

template<typename Key, typename Value>
class ConcurrentMap
{
  public:
    ConcurrentMap() = default;

    explicit ConcurrentMap(size_t initialCapacity)
    {
        map.reserve(initialCapacity);
    }

    bool isEmpty() const
    {
        SharedLock lock(mx);
        return map.empty();
    }

    size_t size() const
    {
        SharedLock lock(mx);
        return map.size();
    }

    size_t capacity() const
    {
        SharedLock lock(mx);
        return map.bucket_count();
    }

    void reserve(size_t count)
    {
        FullLock lock(mx);
        map.reserve(count);
    }

    void rehash(size_t count)
    {
        FullLock lock(mx);
        map.rehash(count);
    }

    void clear()
    {
        FullLock lock(mx);
        map.clear();
    }

    bool contains(const Key& key) const
    {
        SharedLock lock(mx);
        return map.find(key) != map.end();
    }

    // Inserts a default-constructible / argument-constructed value if absent.
    // Returns true if this call inserted it.
    template<typename... Args>
    bool tryEmplace(const Key& key, Args&&... args)
    {
        FullLock lock(mx);
        return map.try_emplace(key, std::forward<Args>(args)...).second;
    }

    // Fast path takes only the shared lock when the key already exists.
    // Returns (inserted, copy of value)
    template<typename... Args>
    std::pair<bool, Value> tryEmplaceShared(const Key& key, Args&&... args)
    {
        {
            SharedLock lock(mx);
            auto it = map.find(key);
            if (it != map.end()) {
                return { false, it->second };
            }
        }
        FullLock lock(mx);
        auto [it, inserted] = map.try_emplace(key, std::forward<Args>(args)...);
        return { inserted, it->second };
    }

    // Emplace then run `mutator(inserted, value&)` under the exclusive lock
    template<typename F, typename... Args>
    bool tryEmplaceThenMutate(const Key& key, F&& mutator, Args&&... args)
    {
        FullLock lock(mx);
        auto [it, inserted] = map.try_emplace(key, std::forward<Args>(args)...);
        mutator(inserted, it->second);
        return inserted;
    }

    // True if the key was new, false if an existing value was replaced
    template<typename V>
    bool insertOrAssign(const Key& key, V&& value)
    {
        FullLock lock(mx);
        return map.insert_or_assign(key, std::forward<V>(value)).second;
    }

    // Inserts a (key, value) pair unless the key is taken; true if inserted
    template<typename P>
    bool insert(P&& pair)
    {
        FullLock lock(mx);
        return map.insert(std::forward<P>(pair)).second;
    }

    void swap(ConcurrentMap<Key, Value>& other)
    {
        if (this == &other) {
            return;
        }
        std::scoped_lock lock(mx, other.mx);
        map.swap(other.map);
    }

    bool erase(const Key& key)
    {
        FullLock lock(mx);
        return map.erase(key) > 0;
    }

    // Remove every element for which pred(key, value) is true; returns count
    template<typename F>
    size_t eraseIf(F&& pred)
    {
        FullLock lock(mx);
        size_t n = 0;
        for (auto it = map.begin(); it != map.end();) {
            if (pred(it->first, it->second)) {
                it = map.erase(it);
                n++;
            } else {
                ++it;
            }
        }
        return n;
    }

    std::optional<Value> get(const Key& key) const
    {
        SharedLock lock(mx);
        auto it = map.find(key);
        if (it == map.end()) {
            return std::nullopt;
        }
        return it->second;
    }

    // Read access to one element; returns false if missing
    template<typename F>
    bool inspect(const Key& key, F&& inspector) const
    {
        SharedLock lock(mx);
        auto it = map.find(key);
        if (it == map.end()) {
            return false;
        }
        inspector(it->second);
        return true;
    }

    template<typename F>
    bool mutate(const Key& key, F&& mutator)
    {
        FullLock lock(mx);
        auto it = map.find(key);
        if (it == map.end()) {
            return false;
        }
        mutator(it->second);
        return true;
    }

    template<typename F>
    void inspectAll(F&& inspector) const
    {
        SharedLock lock(mx);
        for (const auto& [k, v] : map) {
            inspector(k, v);
        }
    }

    template<typename F>
    void mutateAll(F&& mutator)
    {
        FullLock lock(mx);
        for (auto& [k, v] : map) {
            mutator(k, v);
        }
    }

    std::vector<std::pair<Key, Value>> sortedKvPairs() const
    {
        std::vector<std::pair<Key, Value>> out;
        {
            SharedLock lock(mx);
            out.reserve(map.size());
            for (const auto& kv : map) {
                out.emplace_back(kv.first, kv.second);
            }
        }
        std::sort(out.begin(), out.end(), [](const auto& a, const auto& b) {
            return a.first < b.first;
        });
        return out;
    }

  private:
    mutable std::shared_mutex mx;
    std::unordered_map<Key, Value> map;
};

} // namespace faabric::util

// ==========================================================================
// util/config.h
// ==========================================================================
// Environment-driven global configuration singleton.
// Same knobs and defaults as the reference's SystemConfig
// (include/faabric/util/config.h:12-73, src/util/config.cpp:19-84) plus the
// GPU-specific settings of this implementation.


#define MPI_HOST_STATE_LEN 20
#define DEFAULT_TIMEOUT 60000
#define RESULT_KEY_EXPIRY 30000
#define STATUS_KEY_EXPIRY 300000

namespace faabric::util {

class SystemConfig
{
  public:
    // System
    std::string serialisation;
    std::string logLevel;
    std::string logFile;
    std::string stateMode;
    std::string deltaSnapshotEncoding;

    // Redis-compatible store (in-process here; host/port kept for parity)
    std::string redisStateHost;
    std::string redisQueueHost;
    std::string redisPort;

    // Scheduling
    int overrideCpuCount;
    int overrideFreeCpuStart;
    std::string batchSchedulerMode;

    // Worker-related timeouts (all in milliseconds unless stated)
    int globalMessageTimeout;
    int boundTimeout;
    int reaperIntervalSeconds;

    // MPI
    int defaultMpiWorldSize;

    // Endpoint
    std::string endpointInterface;
    std::string endpointHost;
    int endpointPort;
    int endpointNumThreads;

    // Transport
    int functionServerThreads;
    int stateServerThreads;
    int snapshotServerThreads;
    int pointToPointServerThreads;

    // Dirty tracking
    std::string dirtyTrackingMode;
    std::string diffingMode;

    // Planner
    std::string plannerHost;
    int plannerPort;

    // ---- GPU additions ----
    // Comma separated GPU ordinals this worker may use ("" = all visible)
    std::string gpus;
    // cuda | loopback  (loopback = host memory, no GPU required)
    std::string deviceBackend;
    // auto | oneshot | twoshot | nvls | ll | nccl
    std::string allreduceAlgo;
    int useNvls;
    int commStreams;
    long symmHeapBytes;
    // Execution slots exposed per GPU "host"
    int slotsPerGpu;
    // Offset added to every well-known port (several workers on one box)
    int portOffset;
    // Snapshot checkpoint directory (empty = keep snapshots in memory only)
    std::string checkpointDir;

    SystemConfig();

    void print();

    void reset();

  private:
    int getSystemConfIntParam(const char* name, const char* defaultValue);
    long getSystemConfLongParam(const char* name, const char* defaultValue);

    void initialise();
};

SystemConfig& getSystemConfig();

} // namespace faabric::util

// ==========================================================================
// util/crash.h
// ==========================================================================
namespace faabric::util {

// Installs a backtrace-printing handler for fatal signals.  SIGSEGV is left
// alone by default because the segfault dirty tracker owns it.
void setUpCrashHandler(int sig = -1);

void printStackTrace(void* contextR = nullptr);

// What the installed handler does: prints the back-trace, then (unless `sig`
// is the test signal) re-raises with the default action
void handleCrash(int sig);

}

// ==========================================================================
// util/delta.h
// ==========================================================================
// Page / XOR / zstd delta codec (reference: include/faabric/util/delta.h:10-51,
// src/util/delta.cpp:15-270).  Same command stream; zstd is loaded at runtime
// from libzstd.so.1 when present (no headers in this image), otherwise the
// commands are emitted uncompressed.


namespace faabric::util {

struct DeltaSettings
{
    // pages=SIZE;
    bool usePages = true;
    size_t pageSize = 4096;
    // xor;
    bool xorWithOld = true;
    // zstd=LEVEL;
    bool useZstd = true;
    int zstdLevel = 1;

    explicit DeltaSettings(const std::string& definition);
    std::string toString() const;
};

inline constexpr uint8_t DELTA_PROTOCOL_VERSION = 1;
inline constexpr int DELTA_ZSTD_COMPRESS_LEVEL = 1;

enum DeltaCommand : uint8_t
{
    // followed by u32(total size)
    DELTACMD_TOTAL_SIZE = 0x00,
    // followed by u64(compressed length), u64(decompressed length),
    // bytes(compressed commands)
    DELTACMD_ZSTD_COMPRESSED_COMMANDS = 0x01,
    // followed by u32(offset), u32(length), bytes(data)
    DELTACMD_DELTA_OVERWRITE = 0x02,
    // followed by u32(offset), u32(length), bytes(data)
    DELTACMD_DELTA_XOR = 0x03,
    // final command
    DELTACMD_END = 0xFE,
};

std::vector<uint8_t> serializeDelta(const DeltaSettings& cfg,
                                    const uint8_t* oldDataStart,
                                    size_t oldDataLen,
                                    const uint8_t* newDataStart,
                                    size_t newDataLen);

void applyDelta(const std::vector<uint8_t>& delta,
                std::function<void(uint32_t)> setDataSize,
                std::function<uint8_t*()> getDataPointer);

// True if libzstd could be loaded at runtime
bool deltaZstdAvailable();

// ---- building blocks (used by DeviceSnapshot::serializeDelta / applyDelta,
// where the page compare and the XOR run on the GPU) ----
// A command stream under construction: TOTAL_SIZE first, then runs, then END
void deltaBegin(std::vector<uint8_t>& cmds, uint32_t totalSize);

// One run whose payload (`length` bytes: new bytes, or new ^ old when isXor)
// has already been computed
void deltaAppendRun(std::vector<uint8_t>& cmds, bool isXor, uint32_t offset, const uint8_t* payload, uint32_t length);

// Appends END and applies the zstd wrapper the settings ask for
std::vector<uint8_t> deltaFinish(const DeltaSettings& cfg, std::vector<uint8_t>&& cmds);

// Walks a (possibly compressed) delta: onSize(total) and onRun(isXor, offset, payload, length)
void deltaForEach(const std::vector<uint8_t>& delta,
                  const std::function<void(uint32_t)>& onSize,
                  const std::function<void(bool, uint32_t, const uint8_t*, uint32_t)>& onRun);

}

// ==========================================================================
// util/dirty.h
// ==========================================================================
// Dirty-page tracking.  Host memory: four interchangeable trackers selected by
// DIRTY_TRACKING_MODE (none | segfault | softpte | uffd[-wp|-thread|-thread-wp]),
// same contract as the reference (include/faabric/util/dirty.h:24-236): every
// mode reports the same pages for the same writes.  Device memory has no page
// faults to hook, so DeviceCompareDirtyTracker diffs against the base image with
// an sm_90a kernel (csrc/kernels/snapshot_kernels.cu: dirtyScanKernel).


namespace faabric::util {

// Per-page flags are chars (0/1) like the reference, so that they can be merged
// and shipped around as plain byte vectors.
class DirtyTracker
{
  public:
    virtual ~DirtyTracker() = default;

    virtual void clearAll() = 0;

    virtual std::string getType() = 0;

    virtual void startTracking(std::span<uint8_t> region) = 0;

    virtual void stopTracking(std::span<uint8_t> region) = 0;

    virtual std::vector<char> getDirtyPages(std::span<uint8_t> region) = 0;

    virtual void startThreadLocalTracking(std::span<uint8_t> region) = 0;

    virtual void stopThreadLocalTracking(std::span<uint8_t> region) = 0;

    virtual std::vector<char> getThreadLocalDirtyPages(
      std::span<uint8_t> region) = 0;

    virtual std::vector<char> getBothDirtyPages(std::span<uint8_t> region) = 0;
};

// Marks everything dirty (cheap to "track", expensive to diff)
class NoneDirtyTracker final : public DirtyTracker
{
  public:
    void clearAll() override;
    std::string getType() override { return "none"; }
    void startTracking(std::span<uint8_t> region) override;
    void stopTracking(std::span<uint8_t> region) override;
    std::vector<char> getDirtyPages(std::span<uint8_t> region) override;
    void startThreadLocalTracking(std::span<uint8_t> region) override;
    void stopThreadLocalTracking(std::span<uint8_t> region) override;
    std::vector<char> getThreadLocalDirtyPages(
      std::span<uint8_t> region) override;
    std::vector<char> getBothDirtyPages(std::span<uint8_t> region) override;

  private:
    std::vector<char> dirtyPages;
};

// mprotect(PROT_READ) + SIGSEGV handler: first write to a page faults, the
// handler flags it and re-enables writes.
class SegfaultDirtyTracker final : public DirtyTracker
{
  public:
    SegfaultDirtyTracker();
    void clearAll() override;
    std::string getType() override { return "segfault"; }
    void startTracking(std::span<uint8_t> region) override;
    void stopTracking(std::span<uint8_t> region) override;
    std::vector<char> getDirtyPages(std::span<uint8_t> region) override;
    void startThreadLocalTracking(std::span<uint8_t> region) override;
    void stopThreadLocalTracking(std::span<uint8_t> region) override;
    std::vector<char> getThreadLocalDirtyPages(
      std::span<uint8_t> region) override;
    std::vector<char> getBothDirtyPages(std::span<uint8_t> region) override;

    // SIGSEGV handler
    static void handler(int sig, void* info, void* context) noexcept;

  private:
    void setUpSignalHandler();
};

// /proc/self/clear_refs + pagemap soft-dirty bit (bit 55)
class SoftPTEDirtyTracker final : public DirtyTracker
{
  public:
    SoftPTEDirtyTracker();
    ~SoftPTEDirtyTracker() override;
    void clearAll() override;
    std::string getType() override { return "softpte"; }
    void startTracking(std::span<uint8_t> region) override;
    void stopTracking(std::span<uint8_t> region) override;
    std::vector<char> getDirtyPages(std::span<uint8_t> region) override;
    void startThreadLocalTracking(std::span<uint8_t> region) override;
    void stopThreadLocalTracking(std::span<uint8_t> region) override;
    std::vector<char> getThreadLocalDirtyPages(
      std::span<uint8_t> region) override;
    std::vector<char> getBothDirtyPages(std::span<uint8_t> region) override;

    // True if the running kernel exposes soft-dirty bits
    static bool isSupported();

  private:
    int clearRefsFd = -1;
    int pagemapFd = -1;
};

// userfaultfd write-protect tracking, faults drained by an event thread
class UffdDirtyTracker final : public DirtyTracker
{
  public:
    explicit UffdDirtyTracker(const std::string& modeIn);
    ~UffdDirtyTracker() override;
    void clearAll() override;
    std::string getType() override { return mode; }
    void startTracking(std::span<uint8_t> region) override;
    void stopTracking(std::span<uint8_t> region) override;
    std::vector<char> getDirtyPages(std::span<uint8_t> region) override;
    void startThreadLocalTracking(std::span<uint8_t> region) override;
    void stopThreadLocalTracking(std::span<uint8_t> region) override;
    std::vector<char> getThreadLocalDirtyPages(
      std::span<uint8_t> region) override;
    std::vector<char> getBothDirtyPages(std::span<uint8_t> region) override;

    static bool isSupported();

  private:
    std::string mode;
    struct Impl;
    std::unique_ptr<Impl> impl;
};

// GPU memory: compare against a base image on the device
class DeviceCompareDirtyTracker
{
  public:
    // Returns one char per 4 KiB page of [mem, mem+size) that differs from base.
    // Both pointers are device pointers on `device`; synchronises `stream`.
    static std::vector<char> getDirtyPages(const uint8_t* mem,
                                           const uint8_t* base,
                                           size_t size,
                                           int device,
                                           void* stream = nullptr);

    // Same but leaves the flags on the device (uint8 per page); async
    static void getDirtyPagesDevice(const uint8_t* mem,
                                    const uint8_t* base,
                                    size_t size,
                                    uint8_t* pageFlagsDev,
                                    uint64_t* countDev,
                                    void* stream);
};

std::shared_ptr<DirtyTracker> getDirtyTracker();

// Re-reads the mode from the config (tests switch modes)
void resetDirtyTracker();

} // namespace faabric::util

// ==========================================================================
// util/environment.h
// ==========================================================================
namespace faabric::util {

std::string getEnvVar(const std::string& key, const std::string& deflt);

std::string setEnvVar(const std::string& varName, const std::string& value);

void unsetEnvVar(const std::string& varName);

// FAABRIC_EXIT_WITH_PARENT=1: ask the kernel to SIGTERM this process when the
// process that started it dies (test clusters must not outlive a killed
// test runner).  No-op otherwise.
void exitWithParentIfAsked();

// Hardware threads usable by this process (OVERRIDE_CPU_COUNT wins)
unsigned int getUsableCores();

// Number of visible CUDA devices (0 on a CPU-only machine)
int getUsableGpus();

}

// ==========================================================================
// util/fault.h
// ==========================================================================
// Fault injection for the control plane (the reference has none; SURVEY §5.3).
// Rules match outgoing RPCs by destination port and/or message code and drop,
// delay or fail them.  Armed from code (tests) or from the environment:
//
//   FAABRIC_FAULTS="drop:port=8005,header=1,count=2;delay:port=8011,ms=50;error:header=7"
//
// The check on the hot path is one relaxed atomic load when nothing is armed.


namespace faabric::util {

enum class FaultAction
{
    DROP,  // async: silently lost; sync: the caller sees a timeout
    DELAY, // sleep before sending
    ERROR, // the send throws
};

struct FaultRule
{
    FaultAction action = FaultAction::DROP;
    int port = -1;   // -1 = any
    int header = -1; // -1 = any
    int delayMs = 0;
    int count = -1; // how many times it fires (-1 = forever)
};

class FaultInjector
{
  public:
    static FaultInjector& get();

    void addRule(const FaultRule& rule);

    // "action:key=value,..;action:.." (see above)
    void addRulesFromString(const std::string& spec);

    void clear();

    bool armed() const { return nArmed.load(std::memory_order_relaxed) > 0; }

    // The rule that fires for this send, if any (consumes one of its counts)
    std::optional<FaultRule> match(int port, int header);

    long firedCount() const { return fired.load(); }

  private:
    FaultInjector();

    std::mutex mx;
    std::vector<FaultRule> rules;
    std::atomic<int> nArmed{ 0 };
    std::atomic<long> fired{ 0 };
};

}

// ==========================================================================
// util/files.h
// ==========================================================================
namespace faabric::util {

std::string readFileToString(const std::string& path);

std::vector<uint8_t> readFileToBytes(const std::string& path);

void writeBytesToFile(const std::string& path, const std::vector<uint8_t>& data);

bool isWasm(const std::vector<uint8_t>& bytes);

}

// ==========================================================================
// util/func.h
// ==========================================================================
#define MIGRATED_FUNCTION_RETURN_VALUE -99
#define FROZEN_FUNCTION_RETURN_VALUE -98

namespace faabric::util {

std::string funcToString(const faabric::Message& msg, bool includeId);

std::string funcToString(
  const std::shared_ptr<faabric::BatchExecuteRequest>& req);

unsigned int setMessageId(faabric::Message& msg);

std::string buildAsyncResponse(const faabric::Message& msg);

std::shared_ptr<faabric::Message> messageFactoryShared(
  const std::string& user,
  const std::string& function);

faabric::Message messageFactory(const std::string& user,
                                const std::string& function);

std::string resultKeyFromMessageId(unsigned int mid);

std::string statusKeyFromMessageId(unsigned int mid);

std::vector<uint8_t> messageToBytes(const faabric::Message& msg);

std::vector<std::string> getArgvForMessage(const faabric::Message& msg);

// Key of the main-thread snapshot for this message; identical on every host
std::string getMainThreadSnapshotKey(const faabric::Message& msg);

}

// ==========================================================================
// util/gids.h
// ==========================================================================
namespace faabric::util {

// Globally unique-ish ids: a per-process random base mixed with host identity
// plus an atomic counter (reference: src/util/gids.cpp:16-35)
unsigned int generateGid();

}

// ==========================================================================
// util/hwloc.h
// ==========================================================================
// CPU pinning for busy-waiting rank threads + rank -> GPU placement
// (reference: src/util/hwloc.cpp:15-109 pins threads only).


namespace faabric::util {

// RAII claim on one CPU of the free-CPU set; released on destruction
class FaabricCpuSet
{
  public:
    explicit FaabricCpuSet(int cpuIdxIn = -1);
    FaabricCpuSet(const FaabricCpuSet&) = delete;
    FaabricCpuSet& operator=(const FaabricCpuSet&) = delete;
    ~FaabricCpuSet();

    cpu_set_t* get() { return &cpuSet; }
    int getCpuIdx() const { return cpuIdx; }

  private:
    cpu_set_t cpuSet;
    int cpuIdx;
};

// Pins the thread to a currently unclaimed CPU (throws if none left)
std::unique_ptr<FaabricCpuSet> pinThreadToFreeCpu(pthread_t thread);

// Pin near a GPU: picks a free CPU from the NUMA node the GPU hangs off when
// that can be determined from sysfs, any free CPU otherwise
std::unique_ptr<FaabricCpuSet> pinThreadNearGpu(pthread_t thread, int gpuIdx);

// Round-robin placement of an MPI rank / executor slot onto the visible GPUs
// (-1 when there is no GPU)
int gpuForRank(int rank);

// Binds the calling thread to a GPU (cudaSetDevice); no-op without GPUs
void bindThreadToGpu(int gpuIdx);

int getNumFreeCpus();

}

// ==========================================================================
// util/json.h
// ==========================================================================
// Message <-> JSON using the schema's json names (reference: src/util/json.cpp,
// enums printed as ints, default-valued fields omitted).



namespace faabric::util {

class JsonSerialisationException : public faabric::util::FaabricException
{
  public:
    explicit JsonSerialisationException(std::string message)
      : FaabricException(std::move(message))
    {}
};

template<typename M>
std::string messageToJson(const M& msg)
{
    faabric::proto::JsonWriter w;
    msg.toJson(w);
    return w.str();
}

template<typename M>
void jsonToMessage(const std::string& jsonStr, M* msg)
{
    try {
        faabric::proto::JsonValue v = faabric::proto::JsonValue::parse(jsonStr);
        msg->Clear();
        if (!msg->fromJson(v)) {
            throw JsonSerialisationException("JSON does not match message schema");
        }
    } catch (const std::runtime_error& e) {
        throw JsonSerialisationException(std::string("Bad JSON input: ") + e.what());
    }
}

}

// ==========================================================================
// util/latch.h
// ==========================================================================
#define DEFAULT_LATCH_TIMEOUT_MS 10000

namespace faabric::util {

// Count-down latch where every participant calls wait() exactly once
class Latch
{
  public:
    static std::shared_ptr<Latch> create(
      int count,
      int timeoutMs = DEFAULT_LATCH_TIMEOUT_MS);

    explicit Latch(int countIn, int timeoutMsIn = DEFAULT_LATCH_TIMEOUT_MS);

    // Throws if more than `count` callers arrive, or on timeout
    void wait();

  private:
    int count;
    int waiters = 0;
    int timeoutMs;
    std::mutex mx;
    std::condition_variable cv;
};

}

// ==========================================================================
// util/logging.h
// ==========================================================================
// Minimal logger with the spdlog-style macro surface the reference uses
// (include/faabric/util/logging.h).  Pattern: [HH:MM:SS.mmm] [tid] [L] msg.
// Format strings use {} placeholders.


namespace faabric::util {

enum class LogLevel : int
{
    trace = 0,
    debug = 1,
    info = 2,
    warn = 3,
    err = 4,
    critical = 5,
    off = 6
};

void initLogging();

LogLevel getLogLevel();

void setLogLevel(LogLevel level);

void setLogLevel(const std::string& name);

void logLine(LogLevel level, const std::string& msg);

namespace detail {
inline void fmtInto(std::ostringstream& os, std::string_view f)
{
    os << f;
}

template<typename T, typename... Rest>
void fmtInto(std::ostringstream& os,
             std::string_view f,
             const T& v,
             const Rest&... rest)
{
    size_t pos = f.find("{}");
    if (pos == std::string_view::npos) {
        os << f;
        return;
    }
    os << f.substr(0, pos) << v;
    fmtInto(os, f.substr(pos + 2), rest...);
}
}

template<typename... Args>
std::string format(std::string_view f, const Args&... args)
{
    std::ostringstream os;
    detail::fmtInto(os, f, args...);
    return os.str();
}

template<typename... Args>
void logFmt(LogLevel level, std::string_view f, const Args&... args)
{
    if ((int)level < (int)getLogLevel()) {
        return;
    }
    logLine(level, format(f, args...));
}

} // namespace faabric::util

// Compile-time floor: trace/debug compiled out unless FAABRIC_LOG_DEBUG is set
#ifdef FAABRIC_LOG_DEBUG
#define SPDLOG_TRACE(...)                                                      \
    faabric::util::logFmt(faabric::util::LogLevel::trace, __VA_ARGS__)
#define SPDLOG_DEBUG(...)                                                      \
    faabric::util::logFmt(faabric::util::LogLevel::debug, __VA_ARGS__)
#else
#define SPDLOG_TRACE(...) (void)0
#define SPDLOG_DEBUG(...)                                                      \
    faabric::util::logFmt(faabric::util::LogLevel::debug, __VA_ARGS__)
#endif
#define SPDLOG_INFO(...)                                                       \
    faabric::util::logFmt(faabric::util::LogLevel::info, __VA_ARGS__)
#define SPDLOG_WARN(...)                                                       \
    faabric::util::logFmt(faabric::util::LogLevel::warn, __VA_ARGS__)
#define SPDLOG_ERROR(...)                                                      \
    faabric::util::logFmt(faabric::util::LogLevel::err, __VA_ARGS__)
#define SPDLOG_CRITICAL(...)                                                   \
    faabric::util::logFmt(faabric::util::LogLevel::critical, __VA_ARGS__)

// ==========================================================================
// util/macros.h
// ==========================================================================
#define BYTES(arr) reinterpret_cast<uint8_t*>(arr)
#define BYTES_CONST(arr) reinterpret_cast<const uint8_t*>(arr)
#define UNUSED(x) (void)(x)

#ifndef SLEEP_MS
#define SLEEP_MS(ms) usleep((ms) * 1000)
#endif

// Symbol visibility helper for the few things looked up by dlsym / ctypes
#define FAABRIC_EXPORT __attribute__((visibility("default")))

// ==========================================================================
// util/memory.h
// ==========================================================================
// Page-level memory helpers (reference: include/faabric/util/memory.h:16-97,
// src/util/memory.cpp:15-256) plus device-memory regions.


namespace faabric::util {

// dst[i] |= src[i]
void mergeManyDirtyPages(std::vector<char>& dest,
                         const std::vector<std::vector<char>>& source);

void mergeDirtyPages(std::vector<char>& dest, const std::vector<char>& source);

// -------------------------
// Alignment
// -------------------------
struct AlignedChunk
{
    long originalOffset = 0;
    long originalLength = 0;
    long nBytesOffset = 0;
    long nBytesLength = 0;
    long nPagesOffset = 0;
    long nPagesLength = 0;
    long offsetRemainder = 0;
};

static const long HOST_PAGE_SIZE = sysconf(_SC_PAGESIZE);

bool isPageAligned(const void* ptr);

size_t getRequiredHostPages(size_t nBytes);

size_t getRequiredHostPagesRoundDown(size_t nBytes);

size_t alignOffsetDown(size_t offset);

AlignedChunk getPageAlignedChunk(long offset, long length);

// -------------------------
// Allocation
// -------------------------
typedef std::unique_ptr<uint8_t[], std::function<void(uint8_t*)>> MemoryRegion;

MemoryRegion allocatePrivateMemory(size_t size);

MemoryRegion allocateSharedMemory(size_t size);

// PROT_NONE reservation that can later be claimed page by page
MemoryRegion allocateVirtualMemory(size_t size);

void claimVirtualMemory(std::span<uint8_t> region);

void mapMemoryPrivate(std::span<uint8_t> target, int fd);

void mapMemoryShared(std::span<uint8_t> target, int fd);

void resizeFd(int fd, size_t size);

void writeToFd(int fd, off_t offset, std::span<const uint8_t> data);

int createFd(size_t size, const std::string& fdLabel);

void appendDataToFd(int fd, std::span<uint8_t> data);

// -------------------------
// Device memory (GPU)
// -------------------------
// Owning handle of cudaMalloc'd (or pinned-host) memory; empty on CPU boxes.
struct DeviceRegion
{
    uint8_t* ptr = nullptr;
    size_t size = 0;
    int device = -1;
    bool pinnedHost = false;

    DeviceRegion() = default;
    DeviceRegion(const DeviceRegion&) = delete;
    DeviceRegion& operator=(const DeviceRegion&) = delete;
    DeviceRegion(DeviceRegion&& o) noexcept;
    DeviceRegion& operator=(DeviceRegion&& o) noexcept;
    ~DeviceRegion();

    bool valid() const { return ptr != nullptr; }
    void release();
};

// Throws std::runtime_error if no device / allocation failure
DeviceRegion allocateDeviceMemory(size_t size, int device);

DeviceRegion allocatePinnedHostMemory(size_t size);

} // namespace faabric::util

// ==========================================================================
// util/network.h
// ==========================================================================
#define LOCALHOST "127.0.0.1"

namespace faabric::util {

std::string getIPFromHostname(const std::string& hostname);

std::string getPrimaryIPForThisHost(const std::string& interface);

// "gpu3" style host alias used when GPUs are registered as planner hosts
std::string gpuHostName(int gpuIdx);

// -1 if `host` is not a gpu alias
int gpuIndexFromHostName(const std::string& host);

}

// ==========================================================================
// util/ptp.h
// ==========================================================================
namespace faabric::batch_scheduler {
class SchedulingDecision;
}

namespace faabric::util {

// Unlike the reference (src/util/ptp.cpp:4-19) the MPI port / mailbox slot of
// every mapping is carried across.
faabric::PointToPointMappings ptpMappingsFromSchedulingDecision(
  std::shared_ptr<faabric::batch_scheduler::SchedulingDecision> decision);

}

// ==========================================================================
// util/queue.h
// ==========================================================================
// Host-side queues (reference: include/faabric/util/queue.h:24-265).
//  Queue<T>              mutex + condvar, timeouts, peek, drain
//  FixedCapacityQueue<T> bounded blocking SPSC/MPMC ring (own implementation)
//  SpinLockQueue<T>      bounded lock-free ring, busy-waiting (low latency)
//  TokenPool             pool of integer tokens



#if defined(__x86_64__)
#include <immintrin.h>
#define FAABRIC_CPU_PAUSE() _mm_pause()
#else
#define FAABRIC_CPU_PAUSE() std::this_thread::yield()
#endif

#define DEFAULT_QUEUE_TIMEOUT_MS 5000
#define DEFAULT_QUEUE_SIZE 1024

namespace faabric::util {

class QueueTimeoutException : public faabric::util::FaabricException
{
  public:
    explicit QueueTimeoutException(std::string message)
      : FaabricException(std::move(message))
    {}
};

template<typename T>
class Queue
{
  public:
    // Consumers that are not in a request/response exchange (an executor's
    // pool thread waiting for its next function) go to sleep at once: with a
    // thousand of them a brief yield-spin each is a scheduling storm
    void setSpinBeforeSleep(bool v) { spinBeforeSleep = v; }

    void enqueue(T value)
    {
        {
            UniqueLock lock(mx);
            mq.emplace(std::move(value));
            approxSize.store((long)mq.size(), std::memory_order_release);
        }
        enqueueNotifier.notify_one();
    }

    void dequeueIfPresent(T* res)
    {
        UniqueLock lock(mx);
        if (!mq.empty()) {
            T value = std::move(mq.front());
            mq.pop();
            approxSize.store((long)mq.size(), std::memory_order_release);
            emptyNotifier.notify_one();
            *res = std::move(value);
        }
    }

    T dequeue(long timeoutMs = DEFAULT_QUEUE_TIMEOUT_MS)
    {
        if (timeoutMs <= 0) {
            throw std::runtime_error("Dequeue timeout must be positive");
        }
        // A consumer in the middle of a request/response exchange gets its
        // next item within microseconds: look for it briefly before paying
        // for a sleep + wake-up (the yield lets a producer that shares our
        // core run)
        if (spinBeforeSleep && approxSize.load(std::memory_order_acquire) == 0) {
            auto start = std::chrono::steady_clock::now();
            for (int i = 0; approxSize.load(std::memory_order_acquire) == 0; i++) {
                if ((i & 15) == 15) {
                    std::this_thread::yield();
                    if (std::chrono::steady_clock::now() - start > std::chrono::microseconds(20)) {
                        break;
                    }
                }
            }
        }
        UniqueLock lock(mx);
        if (!enqueueNotifier.wait_for(lock,
                                      std::chrono::milliseconds(timeoutMs),
                                      [this] { return !mq.empty(); })) {
            throw QueueTimeoutException("Timeout waiting for dequeue");
        }
        T value = std::move(mq.front());
        mq.pop();
        approxSize.store((long)mq.size(), std::memory_order_release);
        emptyNotifier.notify_one();
        return value;
    }

    T* peek(long timeoutMs = DEFAULT_QUEUE_TIMEOUT_MS)
    {
        UniqueLock lock(mx);
        if (timeoutMs <= 0) {
            throw std::runtime_error("Peek timeout must be positive");
        }
        if (!enqueueNotifier.wait_for(lock,
                                      std::chrono::milliseconds(timeoutMs),
                                      [this] { return !mq.empty(); })) {
            throw QueueTimeoutException("Timeout waiting for queue to peek");
        }
        return &mq.front();
    }

    void waitToDrain(long timeoutMs = DEFAULT_QUEUE_TIMEOUT_MS)
    {
        UniqueLock lock(mx);
        if (!emptyNotifier.wait_for(lock,
                                    std::chrono::milliseconds(timeoutMs),
                                    [this] { return mq.empty(); })) {
            throw QueueTimeoutException("Timed out waiting for queue to empty");
        }
    }

    void drain()
    {
        UniqueLock lock(mx);
        while (!mq.empty()) {
            mq.pop();
        }
        approxSize.store(0, std::memory_order_release);
        emptyNotifier.notify_all();
    }

    long size()
    {
        UniqueLock lock(mx);
        return (long)mq.size();
    }

    void reset()
    {
        UniqueLock lock(mx);
        std::queue<T> empty;
        std::swap(mq, empty);
        approxSize.store(0, std::memory_order_release);
    }

  private:
    std::queue<T> mq;
    std::atomic<long> approxSize{ 0 };
    bool spinBeforeSleep = true;
    std::condition_variable enqueueNotifier;
    std::condition_variable emptyNotifier;
    std::mutex mx;
};

// Bounded ring shared by both fixed-capacity variants.  Multi-producer /
// multi-consumer safe (sequence number per cell).
template<typename T>
class BoundedRing
{
  public:
    explicit BoundedRing(size_t capacityIn)
    {
        cap = 1;
        while (cap < capacityIn) {
            cap <<= 1;
        }
        cells = std::make_unique<Cell[]>(cap);
        for (size_t i = 0; i < cap; i++) {
            cells[i].seq.store(i, std::memory_order_relaxed);
        }
    }

    bool tryPush(T&& v)
    {
        size_t pos = head.load(std::memory_order_relaxed);
        while (true) {
            Cell& c = cells[pos & (cap - 1)];
            size_t seq = c.seq.load(std::memory_order_acquire);
            intptr_t dif = (intptr_t)seq - (intptr_t)pos;
            if (dif == 0) {
                if (head.compare_exchange_weak(
                      pos, pos + 1, std::memory_order_relaxed)) {
                    c.value = std::move(v);
                    c.seq.store(pos + 1, std::memory_order_release);
                    return true;
                }
            } else if (dif < 0) {
                return false; // full
            } else {
                pos = head.load(std::memory_order_relaxed);
            }
        }
    }

    bool tryPop(T& out)
    {
        size_t pos = tail.load(std::memory_order_relaxed);
        while (true) {
            Cell& c = cells[pos & (cap - 1)];
            size_t seq = c.seq.load(std::memory_order_acquire);
            intptr_t dif = (intptr_t)seq - (intptr_t)(pos + 1);
            if (dif == 0) {
                if (tail.compare_exchange_weak(
                      pos, pos + 1, std::memory_order_relaxed)) {
                    out = std::move(c.value);
                    c.seq.store(pos + cap, std::memory_order_release);
                    return true;
                }
            } else if (dif < 0) {
                return false; // empty
            } else {
                pos = tail.load(std::memory_order_relaxed);
            }
        }
    }

    size_t sizeApprox() const
    {
        size_t h = head.load(std::memory_order_relaxed);
        size_t t = tail.load(std::memory_order_relaxed);
        return h >= t ? h - t : 0;
    }

    size_t capacity() const { return cap; }

  private:
    struct Cell
    {
        std::atomic<size_t> seq;
        T value;
    };
    size_t cap;
    std::unique_ptr<Cell[]> cells;
    alignas(64) std::atomic<size_t> head{ 0 };
    alignas(64) std::atomic<size_t> tail{ 0 };
};

// Blocking bounded queue: spins briefly then sleeps on a condition variable
template<typename T>
class FixedCapacityQueue
{
  public:
    explicit FixedCapacityQueue(int capacity)
      : ring(capacity)
    {}

    FixedCapacityQueue()
      : ring(DEFAULT_QUEUE_SIZE)
    {}

    void enqueue(T value, long timeoutMs = DEFAULT_QUEUE_TIMEOUT_MS)
    {
        if (timeoutMs <= 0) {
            throw std::runtime_error("Enqueue timeout must be positive");
        }
        auto deadline = std::chrono::steady_clock::now() +
                        std::chrono::milliseconds(timeoutMs);
        while (!ring.tryPush(std::move(value))) {
            if (std::chrono::steady_clock::now() > deadline) {
                throw QueueTimeoutException("Timeout waiting for enqueue");
            }
            UniqueLock lock(mx);
            blockedProducers.fetch_add(1, std::memory_order_acq_rel);
            notFull.wait_for(lock, std::chrono::microseconds(200));
            blockedProducers.fetch_sub(1, std::memory_order_acq_rel);
        }
        // seq_cst pairing with the consumer: it registers as a sleeper
        // (under mx) BEFORE its final emptiness check
        std::atomic_thread_fence(std::memory_order_seq_cst);
        if (sleepers.load(std::memory_order_seq_cst) > 0) {
            UniqueLock lock(mx);
            notEmpty.notify_one();
        }
    }

    void dequeueIfPresent(T* res)
    {
        T v;
        if (ring.tryPop(v)) {
            *res = std::move(v);
            wakeProducer();
        }
    }

    T dequeue(long timeoutMs = DEFAULT_QUEUE_TIMEOUT_MS)
    {
        if (timeoutMs <= 0) {
            throw std::runtime_error("Dequeue timeout must be positive");
        }
        T v;
        // Phase 1: spin for a few tens of microseconds - a peer in the
        // middle of a ping-pong answers within that time
        auto start = std::chrono::steady_clock::now();
        for (int i = 0;; i++) {
            if (ring.tryPop(v)) {
                wakeProducer();
                return v;
            }
            FAABRIC_CPU_PAUSE();
            if ((i & 31) == 31) {
                // The producer may have been woken onto OUR core (wake-affine
                // placement): give it a chance instead of starving it
                std::this_thread::yield();
                if (std::chrono::steady_clock::now() - start > std::chrono::microseconds(SPIN_BEFORE_SLEEP_US)) {
                    break;
                }
            }
        }
        // Phase 2: sleep.  The emptiness check and the wait happen under the
        // same mutex the producer takes to notify, so no wake-up is lost
        auto deadline = start + std::chrono::milliseconds(timeoutMs);
        UniqueLock lock(mx);
        sleepers.fetch_add(1, std::memory_order_seq_cst);
        std::atomic_thread_fence(std::memory_order_seq_cst);
        while (true) {
            if (ring.tryPop(v)) {
                sleepers.fetch_sub(1, std::memory_order_acq_rel);
                lock.unlock();
                wakeProducer();
                return v;
            }
            if (std::chrono::steady_clock::now() > deadline) {
                sleepers.fetch_sub(1, std::memory_order_acq_rel);
                throw QueueTimeoutException("Timeout waiting for dequeue");
            }
            notEmpty.wait_for(lock, std::chrono::milliseconds(50));
        }
    }

    void drain()
    {
        T v;
        while (ring.tryPop(v)) {
        }
    }

    long size() { return (long)ring.sizeApprox(); }

    void reset() { drain(); }

  private:
    static constexpr int SPIN_BEFORE_SLEEP_US = 50;

    BoundedRing<T> ring;
    std::mutex mx;
    std::condition_variable notEmpty;
    std::condition_variable notFull;
    std::atomic<int> sleepers{ 0 };
    std::atomic<int> blockedProducers{ 0 };

    void wakeProducer()
    {
        if (blockedProducers.load(std::memory_order_acquire) > 0) {
            UniqueLock lock(mx);
            notFull.notify_one();
        }
    }
};

// Busy-waiting bounded queue for pinned rank threads
template<typename T>
class SpinLockQueue
{
  public:
    SpinLockQueue()
      : ring(DEFAULT_QUEUE_SIZE)
    {}

    explicit SpinLockQueue(int capacity)
      : ring(capacity)
    {}

    void enqueue(T& value, long timeoutMs = DEFAULT_QUEUE_TIMEOUT_MS)
    {
        T v = value;
        spinPush(std::move(v), timeoutMs);
    }

    void enqueue(T&& value, long timeoutMs = DEFAULT_QUEUE_TIMEOUT_MS)
    {
        spinPush(std::move(value), timeoutMs);
    }

    T dequeue(long timeoutMs = DEFAULT_QUEUE_TIMEOUT_MS)
    {
        T v;
        uint64_t spins = 0;
        auto start = std::chrono::steady_clock::now();
        while (!ring.tryPop(v)) {
            FAABRIC_CPU_PAUSE();
            if ((++spins & 0xffff) == 0 &&
                std::chrono::steady_clock::now() - start >
                  std::chrono::milliseconds(timeoutMs)) {
                throw QueueTimeoutException("Timeout spinning for dequeue");
            }
        }
        return v;
    }

    bool tryDequeue(T& out) { return ring.tryPop(out); }

    // Same name as the blocking queues' non-blocking take
    void dequeueIfPresent(T* res)
    {
        T v;
        if (ring.tryPop(v)) {
            *res = std::move(v);
        }
    }

    long size() { return (long)ring.sizeApprox(); }

    void drain()
    {
        T v;
        while (ring.tryPop(v)) {
        }
    }

    void reset() { drain(); }

  private:
    BoundedRing<T> ring;

    void spinPush(T&& v, long timeoutMs)
    {
        uint64_t spins = 0;
        auto start = std::chrono::steady_clock::now();
        while (!ring.tryPush(std::move(v))) {
            FAABRIC_CPU_PAUSE();
            if ((++spins & 0xffff) == 0 &&
                std::chrono::steady_clock::now() - start >
                  std::chrono::milliseconds(timeoutMs)) {
                throw QueueTimeoutException("Timeout spinning for enqueue");
            }
        }
    }
};

class TokenPool
{
  public:
    explicit TokenPool(int nTokens);

    int getToken();

    void releaseToken(int token);

    void reset();

    int size();

    int taken();

    int free();

  private:
    int _size;
    Queue<int> queue;
};

} // namespace faabric::util

// ==========================================================================
// util/random.h
// ==========================================================================
namespace faabric::util {

std::string randomString(int len);

std::string randomStringFromSet(int len, const std::string& charSet);

// A uniformly chosen member of the set ("" for an empty one)
std::string randomStringFromSet(const std::unordered_set<std::string>& s);

int randomInteger(int iStart, int iEnd);

}

// ==========================================================================
// util/snapshot.h
// ==========================================================================
// Host snapshots: a memfd-backed memory image with typed merge regions, diffing
// against dirty pages and diff application.  Behavioural contract follows the
// reference (include/faabric/util/snapshot.h:21-346, src/util/snapshot.cpp);
// offsets are 64-bit here (the reference's uint32 offsets cap images at 4 GiB).
// The device-resident counterpart is faabric::snapshot::DeviceSnapshot.



namespace faabric::util {

// Granularity of the array comparison inside a dirty page
#define ARRAY_COMP_CHUNK_SIZE 128

// Numeric values are part of the application ABI
enum SnapshotDataType
{
    Raw,
    Bool,
    Int,
    Long,
    Float,
    Double
};

enum SnapshotMergeOperation
{
    Bytewise,
    Sum,
    Product,
    Subtract,
    Max,
    Min,
    Ignore,
    XOR
};

std::string snapshotDataTypeStr(SnapshotDataType dt);

std::string snapshotMergeOpStr(SnapshotMergeOperation op);

// A modification to a snapshot.  Non-owning: `data` points into the memory
// the diff was computed from (or into a kept-alive transport message).
class SnapshotDiff
{
  public:
    SnapshotDiff() = default;

    SnapshotDiff(SnapshotDataType dataTypeIn,
                 SnapshotMergeOperation operationIn,
                 uint64_t offsetIn,
                 std::span<const uint8_t> dataIn);

    SnapshotDataType getDataType() const { return dataType; }

    SnapshotMergeOperation getOperation() const { return operation; }

    uint64_t getOffset() const { return offset; }

    std::span<const uint8_t> getData() const { return data; }

    std::vector<uint8_t> getDataCopy() const;

  private:
    SnapshotDataType dataType = SnapshotDataType::Raw;
    SnapshotMergeOperation operation = SnapshotMergeOperation::Bytewise;
    uint64_t offset = 0;
    std::span<const uint8_t> data;
};

class SnapshotMergeRegion
{
  public:
    uint64_t offset = 0;
    uint64_t length = 0; // 0 => until the end of the original data
    SnapshotDataType dataType = SnapshotDataType::Raw;
    SnapshotMergeOperation operation = SnapshotMergeOperation::Bytewise;

    SnapshotMergeRegion() = default;

    SnapshotMergeRegion(uint64_t offsetIn,
                        uint64_t lengthIn,
                        SnapshotDataType dataTypeIn,
                        SnapshotMergeOperation operationIn);

    // Appends the diffs this region produces.  NB: XOR and the typed operations
    // overwrite `updatedData` with the value to transmit (zero-copy diffs).
    void addDiffs(std::vector<SnapshotDiff>& diffs,
                  std::span<const uint8_t> originalData,
                  std::span<uint8_t> updatedData,
                  const std::vector<char>& dirtyRegions);

    bool operator<(const SnapshotMergeRegion& other) const
    {
        return offset < other.offset;
    }

    bool operator==(const SnapshotMergeRegion& other) const
    {
        return offset == other.offset && length == other.length &&
               dataType == other.dataType && operation == other.operation;
    }
};

// Value sent for a typed region (Sum: new-old, Subtract: old-new, Product:
// new/old, Max/Min: new).  Writes it over `updated`; false if unchanged.
template<typename T>
bool calculateDiffValue(const uint8_t* original,
                        uint8_t* updated,
                        SnapshotMergeOperation operation);

// Merges a received typed value into the main copy
template<typename T>
T applyDiffValue(const uint8_t* original,
                 const uint8_t* diff,
                 SnapshotMergeOperation operation);

// Byte-exact runs of difference between a and b over [startOffset, endOffset):
// 128-byte chunks are skipped by memcmp, inside a differing chunk a run ends at
// the first equal byte.  Appends (offset, length) pairs.
void diffArrayRegions(std::vector<std::pair<uint64_t, uint64_t>>& diffs,
                      uint64_t startOffset,
                      uint64_t endOffset,
                      std::span<const uint8_t> a,
                      std::span<const uint8_t> b);

class SnapshotData
{
  public:
    SnapshotData() = default;

    explicit SnapshotData(size_t sizeIn);

    SnapshotData(size_t sizeIn, size_t maxSizeIn);

    explicit SnapshotData(std::span<const uint8_t> dataIn);

    SnapshotData(std::span<const uint8_t> dataIn, size_t maxSizeIn);

    SnapshotData(const SnapshotData&) = delete;

    SnapshotData& operator=(const SnapshotData&) = delete;

    ~SnapshotData();

    void copyInData(std::span<const uint8_t> buffer, uint64_t offset = 0);

    const uint8_t* getDataPtr(uint64_t offset = 0);

    std::vector<uint8_t> getDataCopy();

    std::vector<uint8_t> getDataCopy(uint64_t offset, size_t dataSize);

    // Private copy-on-write mapping of the image onto page-aligned `target`
    void mapToMemory(std::span<uint8_t> target);

    void addMergeRegion(uint64_t offset,
                        size_t length,
                        SnapshotDataType dataType,
                        SnapshotMergeOperation operation);

    // Gap filler type follows the DIFFING_MODE config (bytewise | xor)
    void fillGapsWithBytewiseRegions();

    void clearMergeRegions();

    std::vector<SnapshotMergeRegion> getMergeRegions();

    size_t getQueuedDiffsCount();

    void queueDiffs(const std::vector<SnapshotDiff>& diffs);

    // Applies and clears the queue; returns how many were written
    int writeQueuedDiffs();

    void applyDiffs(const std::vector<SnapshotDiff>& diffs);

    void applyDiff(const SnapshotDiff& diff);

    size_t getSize() const { return size; }

    size_t getMaxSize() const { return maxSize; }

    // ---- checkpoint persistence (the reference keeps snapshots in memory
    // only, SURVEY §5.4; here a frozen app's image can outlive the process) ----
    // Image + merge regions, written to `path` atomically (temp file + rename)
    void writeToFile(const std::string& path);

    // Throws std::runtime_error on a missing / truncated / foreign file
    static std::shared_ptr<SnapshotData> readFromFile(const std::string& path);

    // Every write since the last clear as Raw/Bytewise diffs into the image
    std::vector<SnapshotDiff> getTrackedChanges();

    void clearTrackedChanges();

    std::vector<SnapshotDiff> diffWithDirtyRegions(
      std::span<uint8_t> updated,
      const std::vector<char>& dirtyRegions);

  private:
    size_t size = 0;
    size_t maxSize = 0;
    int fd = -1;

    std::shared_mutex snapMx;

    MemoryRegion data = nullptr;

    std::vector<SnapshotDiff> queuedDiffs;
    std::deque<std::vector<uint8_t>> queuedDiffData;

    // offset -> end (exclusive)
    std::vector<std::pair<uint64_t, uint64_t>> trackedChanges;

    std::vector<SnapshotMergeRegion> mergeRegions;

    void init(size_t initialSize, size_t maxSizeIn);

    uint8_t* validatedOffsetPtr(uint64_t offset);

    void checkWriteExtension(std::span<const uint8_t> buffer, uint64_t offset);

    void writeData(std::span<const uint8_t> buffer, uint64_t offset = 0);

    void xorData(std::span<const uint8_t> buffer, uint64_t offset = 0);

    void applyDiffLocked(const SnapshotDiff& diff);
};

} // namespace faabric::util

// ==========================================================================
// util/state.h
// ==========================================================================
// Naming of state values in the backing store and mask helpers
// (reference: include/faabric/util/state.h, src/util/state.cpp)
#define STATE_MASK_8 0b11111111
#define STATE_MASK_32 0b11111111111111111111111111111111

namespace faabric::util {

// "<user>_<key>"; throws when either part is empty
std::string keyForUser(const std::string& user, const std::string& key);

// Sets the two 32-bit words of a mask that cover double number `idx`
void maskDouble(unsigned int* maskArray, unsigned long idx);

}

// ==========================================================================
// util/string_tools.h
// ==========================================================================
namespace faabric::util {

bool isAllWhitespace(const std::string& input);

bool startsWith(const std::string& input, const std::string& subStr);

bool endsWith(const std::string& value, const std::string& ending);

bool contains(const std::string& input, const std::string& subStr);

std::string removeSubstr(const std::string& input, const std::string& toErase);

bool stringIsInt(const std::string& input);

std::vector<std::string> splitString(const std::string& input, char delim);

std::string trim(const std::string& input);

std::string toLower(const std::string& input);

// "[a, b, c]"
template<class T>
std::string vectorToString(std::vector<T> vec)
{
    std::string out = "[";
    for (size_t i = 0; i < vec.size(); i++) {
        if constexpr (std::is_arithmetic_v<T>) {
            out += std::to_string(vec[i]);
        } else {
            out += vec[i];
        }
        if (i + 1 < vec.size()) {
            out += ", ";
        }
    }
    return out + "]";
}

}

// ==========================================================================
// util/testing.h
// ==========================================================================
namespace faabric::util {

// Test mode relaxes some checks; mock mode makes every RPC client record its
// calls instead of opening sockets (reference: src/util/testing.cpp:6-26)
void setTestMode(bool val);

bool isTestMode();

void setMockMode(bool val);

bool isMockMode();

}

// ==========================================================================
// util/timing.h
// ==========================================================================
// Self-tracing macros, compiled in only with -DTRACE_ALL (reference:
// include/faabric/util/timing.h:6-17).  Adds a CUDA-event timer for device
// work timed on a stream.



#ifdef TRACE_ALL
#define PROF_BEGIN faabric::util::startGlobalTimer();
#define PROF_START(name)                                                       \
    const faabric::util::TimePoint name = faabric::util::startTimer();
#define PROF_END(name) faabric::util::logEndTimer(#name, name);
#define PROF_SUMMARY faabric::util::printTimerTotals();
#define PROF_CLEAR faabric::util::clearTimerTotals();
#else
#define PROF_BEGIN
#define PROF_START(name)
#define PROF_END(name)
#define PROF_SUMMARY
#define PROF_CLEAR
#endif

namespace faabric::util {

TimePoint startTimer();

long getTimeDiffNanos(const TimePoint& begin);

long getTimeDiffMicros(const TimePoint& begin);

double getTimeDiffMillis(const TimePoint& begin);

void logEndTimer(const std::string& label, const TimePoint& begin);

void startGlobalTimer();

void printTimerTotals();

void clearTimerTotals();

// Returns "label:totalMicros:count" lines, sorted by total descending
std::string getTimerTotalsString();

uint64_t timespecToNanos(struct timespec* nativeTimespec);

void nanosToTimespec(uint64_t nanos, struct timespec* nativeTimespec);

} // namespace faabric::util

