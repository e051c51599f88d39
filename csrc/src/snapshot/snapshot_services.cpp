// SnapshotRegistry, SnapshotClient, SnapshotServer, DeviceSnapshot
#include <filesystem>
#include <faabric/device/communicator.h>
#include <faabric/scheduler/Scheduler.h>
#include <faabric/snapshot/DeviceSnapshot.h>
#include <faabric/snapshot/SnapshotClient.h>
#include <faabric/snapshot/SnapshotRegistry.h>
#include <faabric/snapshot/SnapshotServer.h>
#include <faabric/transport/common.h>
#include <faabric/util/config.h>
#include <faabric/util/dirty.h>
#include <faabric/util/logging.h>
#include <faabric/util/testing.h>

#include "launch_api.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <deque>
#include <map>
#include <atomic>
#include <cstring>
#include <unistd.h>

namespace faabric::snapshot {

using faabric::util::SnapshotData;
using faabric::util::SnapshotDataType;
using faabric::util::SnapshotDiff;
using faabric::util::SnapshotMergeOperation;
using faabric::util::SnapshotMergeRegion;

// ---------------------------------------------------------------------------
// Registry
// ---------------------------------------------------------------------------
SnapshotRegistry& getSnapshotRegistry()
{
    static SnapshotRegistry reg;
    return reg;
}

std::shared_ptr<SnapshotData> SnapshotRegistry::getSnapshot(const std::string& key)
{
    if (key.empty()) {
        SPDLOG_ERROR("Attempting to get snapshot with empty key");
        throw std::runtime_error("Getting snapshot with empty key");
    }
    std::shared_lock<std::shared_mutex> lock(snapshotsMx);
    auto it = snapshotMap.find(key);
    if (it == snapshotMap.end()) {
        SPDLOG_ERROR("Snapshot for {} does not exist", key);
        throw std::runtime_error("Snapshot doesn't exist");
    }
    return it->second;
}

bool SnapshotRegistry::snapshotExists(const std::string& key)
{
    std::shared_lock<std::shared_mutex> lock(snapshotsMx);
    return snapshotMap.find(key) != snapshotMap.end();
}

void SnapshotRegistry::registerSnapshot(const std::string& key, std::shared_ptr<SnapshotData> data)
{
    std::unique_lock<std::shared_mutex> lock(snapshotsMx);
    SPDLOG_TRACE("Registering snapshot {} size {}", key, data->getSize());
    snapshotMap.insert_or_assign(key, std::move(data));
}

void SnapshotRegistry::deleteSnapshot(const std::string& key)
{
    std::unique_lock<std::shared_mutex> lock(snapshotsMx);
    snapshotMap.erase(key);
}

size_t SnapshotRegistry::getSnapshotCount()
{
    std::shared_lock<std::shared_mutex> lock(snapshotsMx);
    return snapshotMap.size();
}

std::shared_ptr<DeviceSnapshot> SnapshotRegistry::getDeviceSnapshot(const std::string& key)
{
    DeviceSnapshotDescriptor desc;
    {
        std::shared_lock<std::shared_mutex> lock(snapshotsMx);
        auto it = deviceMap.find(key);
        if (it != deviceMap.end()) {
            return it->second;
        }
        auto dit = descriptorMap.find(key);
        if (dit == descriptorMap.end()) {
            SPDLOG_ERROR("Device snapshot for {} does not exist", key);
            throw std::runtime_error("Device snapshot doesn't exist");
        }
        desc = dit->second;
    }
    // An image owned by another process of this box: map it once
    auto mapped = DeviceSnapshot::fromDescriptor(desc);
    std::unique_lock<std::shared_mutex> lock(snapshotsMx);
    auto [it, inserted] = deviceMap.try_emplace(key, mapped);
    return it->second;
}

bool SnapshotRegistry::deviceSnapshotExists(const std::string& key)
{
    std::shared_lock<std::shared_mutex> lock(snapshotsMx);
    if (deviceMap.find(key) != deviceMap.end()) {
        return true;
    }
    auto dit = descriptorMap.find(key);
    return dit != descriptorMap.end() && !dit->second.ipcHandle.empty() &&
           dit->second.ownerPid != (int)::getpid() && faabric::util::getUsableGpus() > 0;
}

void SnapshotRegistry::registerDeviceDescriptor(const std::string& key, const DeviceSnapshotDescriptor& desc)
{
    std::unique_lock<std::shared_mutex> lock(snapshotsMx);
    descriptorMap.insert_or_assign(key, desc);
}

bool SnapshotRegistry::deviceDescriptorExists(const std::string& key)
{
    std::shared_lock<std::shared_mutex> lock(snapshotsMx);
    return descriptorMap.find(key) != descriptorMap.end();
}

DeviceSnapshotDescriptor SnapshotRegistry::getDeviceDescriptor(const std::string& key)
{
    std::shared_lock<std::shared_mutex> lock(snapshotsMx);
    auto it = descriptorMap.find(key);
    if (it == descriptorMap.end()) {
        throw std::runtime_error("Device snapshot descriptor doesn't exist");
    }
    return it->second;
}

void SnapshotRegistry::registerDeviceSnapshot(const std::string& key, std::shared_ptr<DeviceSnapshot> data)
{
    std::unique_lock<std::shared_mutex> lock(snapshotsMx);
    deviceMap.insert_or_assign(key, std::move(data));
}

void SnapshotRegistry::deleteDeviceSnapshot(const std::string& key)
{
    std::unique_lock<std::shared_mutex> lock(snapshotsMx);
    deviceMap.erase(key);
    descriptorMap.erase(key);
}

void SnapshotRegistry::clear()
{
    std::unique_lock<std::shared_mutex> lock(snapshotsMx);
    snapshotMap.clear();
    deviceMap.clear();
    descriptorMap.clear();
}

// On-disk checkpoints: "<hex(key)>.snap" for host images, ".dsnap" for images
// that lived in device memory
namespace {
std::string hexKey(const std::string& key)
{
    static const char* digits = "0123456789abcdef";
    std::string out;
    out.reserve(key.size() * 2);
    for (unsigned char c : key) {
        out.push_back(digits[c >> 4]);
        out.push_back(digits[c & 15]);
    }
    return out;
}

bool unhexKey(const std::string& hex, std::string& key)
{
    if (hex.size() % 2 != 0) {
        return false;
    }
    key.clear();
    auto nibble = [](char c) -> int {
        if (c >= '0' && c <= '9') {
            return c - '0';
        }
        if (c >= 'a' && c <= 'f') {
            return c - 'a' + 10;
        }
        return -1;
    };
    for (size_t i = 0; i < hex.size(); i += 2) {
        int hi = nibble(hex[i]);
        int lo = nibble(hex[i + 1]);
        if (hi < 0 || lo < 0) {
            return false;
        }
        key.push_back((char)((hi << 4) | lo));
    }
    return true;
}
}

size_t SnapshotRegistry::checkpointToDir(const std::string& dir)
{
    std::filesystem::create_directories(dir);
    // Copy the maps: file IO happens outside the registry lock
    std::unordered_map<std::string, std::shared_ptr<SnapshotData>> hostSnaps;
    std::unordered_map<std::string, std::shared_ptr<DeviceSnapshot>> deviceSnaps;
    {
        std::shared_lock<std::shared_mutex> lock(snapshotsMx);
        hostSnaps = snapshotMap;
        deviceSnaps = deviceMap;
    }
    size_t written = 0;
    for (const auto& [key, snap] : hostSnaps) {
        snap->writeToFile(dir + "/" + hexKey(key) + ".snap");
        written++;
    }
    for (const auto& [key, snap] : deviceSnaps) {
        snap->writeToFile(dir + "/" + hexKey(key) + ".dsnap");
        written++;
    }
    // Files of snapshots that no longer exist would resurrect them on restore
    for (const auto& entry : std::filesystem::directory_iterator(dir)) {
        const std::filesystem::path& p = entry.path();
        const std::string ext = p.extension().string();
        std::string key;
        if ((ext == ".snap" && unhexKey(p.stem().string(), key) && !hostSnaps.contains(key)) ||
            (ext == ".dsnap" && unhexKey(p.stem().string(), key) && !deviceSnaps.contains(key))) {
            std::error_code ec;
            std::filesystem::remove(p, ec);
        }
    }
    SPDLOG_DEBUG("Checkpointed {} snapshots to {}", written, dir);
    return written;
}

size_t SnapshotRegistry::restoreFromDir(const std::string& dir, int device)
{
    size_t restored = 0;
    if (!std::filesystem::is_directory(dir)) {
        return 0;
    }
    for (const auto& entry : std::filesystem::directory_iterator(dir)) {
        const std::filesystem::path& p = entry.path();
        const std::string ext = p.extension().string();
        std::string key;
        if ((ext != ".snap" && ext != ".dsnap") || !unhexKey(p.stem().string(), key)) {
            continue;
        }
        auto host = SnapshotData::readFromFile(p.string());
        if (ext == ".dsnap" && device >= 0) {
            registerDeviceSnapshot(key, DeviceSnapshot::fromHost(*host, device));
        } else {
            registerSnapshot(key, host);
        }
        restored++;
    }
    return restored;
}

// ---------------------------------------------------------------------------
// Client (+ mock capture)
// ---------------------------------------------------------------------------
static std::mutex mockMutex;
static std::vector<std::pair<std::string, std::shared_ptr<SnapshotData>>> snapshotPushes;
static std::vector<std::pair<std::string, std::shared_ptr<MockSnapshotUpdate>>> snapshotDiffPushes;
static std::vector<std::pair<std::string, std::string>> snapshotDeletes;
static std::vector<std::pair<std::string, std::tuple<int, int, std::string, int>>> threadResults;
static std::vector<std::tuple<std::string, std::string, DeviceSnapshotDescriptor>> deviceSnapshotPushes;

std::vector<std::tuple<std::string, std::string, DeviceSnapshotDescriptor>> getDeviceSnapshotPushes()
{
    std::lock_guard<std::mutex> lk(mockMutex);
    return deviceSnapshotPushes;
}

std::vector<std::pair<std::string, std::shared_ptr<SnapshotData>>> getSnapshotPushes()
{
    std::lock_guard<std::mutex> lk(mockMutex);
    return snapshotPushes;
}

std::vector<std::pair<std::string, std::shared_ptr<MockSnapshotUpdate>>> getSnapshotDiffPushes()
{
    std::lock_guard<std::mutex> lk(mockMutex);
    return snapshotDiffPushes;
}

std::vector<std::pair<std::string, std::string>> getSnapshotDeletes()
{
    std::lock_guard<std::mutex> lk(mockMutex);
    return snapshotDeletes;
}

std::vector<std::pair<std::string, std::tuple<int, int, std::string, int>>> getThreadResults()
{
    std::lock_guard<std::mutex> lk(mockMutex);
    return threadResults;
}

void clearMockSnapshotRequests()
{
    std::lock_guard<std::mutex> lk(mockMutex);
    snapshotPushes.clear();
    snapshotDiffPushes.clear();
    snapshotDeletes.clear();
    threadResults.clear();
    deviceSnapshotPushes.clear();
}

static thread_local std::unordered_map<std::string, std::shared_ptr<SnapshotClient>> tlsSnapClients;

std::shared_ptr<SnapshotClient> getSnapshotClient(const std::string& host)
{
    auto it = tlsSnapClients.find(host);
    if (it != tlsSnapClients.end()) {
        return it->second;
    }
    auto c = std::make_shared<SnapshotClient>(host);
    tlsSnapClients[host] = c;
    return c;
}

void clearSnapshotClients()
{
    tlsSnapClients.clear();
}

SnapshotClient::SnapshotClient(const std::string& hostIn)
  : faabric::transport::MessageEndpointClient(hostIn, SNAPSHOT_ASYNC_PORT, SNAPSHOT_SYNC_PORT)
{}

static void fillRegions(faabric::proto::RepeatedField<faabric::SnapshotMergeRegionRequest>* out,
                        const std::vector<SnapshotMergeRegion>& regions)
{
    for (const auto& r : regions) {
        auto* m = out->Add();
        m->set_offset(r.offset);
        m->set_length(r.length);
        m->set_datatype((int)r.dataType);
        m->set_mergeop((int)r.operation);
    }
}

static void fillDiffs(faabric::proto::RepeatedField<faabric::SnapshotDiffRequest>* out,
                      const std::vector<SnapshotDiff>& diffs)
{
    for (const auto& d : diffs) {
        auto* m = out->Add();
        m->set_offset(d.getOffset());
        m->set_datatype((int)d.getDataType());
        m->set_mergeop((int)d.getOperation());
        m->set_data(d.getData().data(), d.getData().size());
    }
}

bool SnapshotClient::receiverSharesRegistry(const std::string& key, const std::shared_ptr<SnapshotData>& data)
{
    // served from this process? (virtual hosts of one worker, in-process planner)
    auto addr = faabric::transport::parseHostAddress(host); // resolves virtual host names
    if (!faabric::transport::isLocalAddress(addr.ip) ||
        faabric::transport::MessageEndpointServer::findLocal(SNAPSHOT_SYNC_PORT + addr.portOffset, true) == nullptr) {
        return false;
    }
    auto& reg = getSnapshotRegistry();
    return reg.snapshotExists(key) && reg.getSnapshot(key) == data;
}

void SnapshotClient::pushSnapshot(const std::string& key, std::shared_ptr<SnapshotData> data)
{
    if (data->getSize() == 0) {
        SPDLOG_ERROR("Cannot push snapshot {} with zero size to {}", key, host);
        throw std::runtime_error("Pushing snapshot with zero size");
    }
    SPDLOG_DEBUG("Pushing snapshot {} to {} ({} bytes)", key, host, data->getSize());
    if (faabric::util::isMockMode()) {
        std::lock_guard<std::mutex> lk(mockMutex);
        snapshotPushes.emplace_back(host, data);
        return;
    }
    if (receiverSharesRegistry(key, data)) {
        // The destination is another (virtual) host of THIS worker: it reads
        // the same registry, and replacing the object under the key would cut
        // the owner off from the diffs queued on it
        SPDLOG_DEBUG("Snapshot {} already visible to {} (same worker)", key, host);
        return;
    }
    faabric::SnapshotPushRequest req;
    req.set_key(key);
    req.set_maxsize(data->getMaxSize());
    req.set_contents(data->getDataPtr(), data->getSize());
    fillRegions(req.mutable_mergeregions(), data->getMergeRegions());
    faabric::EmptyResponse resp;
    syncSend(SnapshotCalls::PushSnapshot, &req, &resp);
}

void SnapshotClient::pushSnapshotUpdate(std::string snapshotKey,
                                        const std::shared_ptr<SnapshotData>& data,
                                        const std::vector<SnapshotDiff>& diffs)
{
    SPDLOG_DEBUG("Pushing update to snapshot {} to {} ({} diffs)", snapshotKey, host, diffs.size());
    if (!faabric::util::isMockMode() && receiverSharesRegistry(snapshotKey, data)) {
        return; // same object: the tracked changes are already in it
    }
    if (faabric::util::isMockMode()) {
        auto upd = std::make_shared<MockSnapshotUpdate>();
        for (const auto& d : diffs) {
            upd->diffData.push_back(d.getDataCopy());
            upd->diffs.emplace_back(d.getDataType(), d.getOperation(), d.getOffset(), upd->diffData.back());
        }
        upd->mergeRegions = data->getMergeRegions();
        std::lock_guard<std::mutex> lk(mockMutex);
        snapshotDiffPushes.emplace_back(host, upd);
        return;
    }
    faabric::SnapshotUpdateRequest req;
    req.set_key(snapshotKey);
    fillRegions(req.mutable_mergeregions(), data->getMergeRegions());
    fillDiffs(req.mutable_diffs(), diffs);
    faabric::EmptyResponse resp;
    syncSend(SnapshotCalls::PushSnapshotUpdate, &req, &resp);
}

void SnapshotClient::deleteSnapshot(const std::string& key)
{
    if (faabric::util::isMockMode()) {
        std::lock_guard<std::mutex> lk(mockMutex);
        snapshotDeletes.emplace_back(host, key);
        return;
    }
    faabric::SnapshotDeleteRequest req;
    req.set_key(key);
    asyncSend(SnapshotCalls::DeleteSnapshot, &req);
}

void SnapshotClient::pushThreadResult(uint32_t appId,
                                      uint32_t messageId,
                                      int returnValue,
                                      const std::string& key,
                                      const std::vector<SnapshotDiff>& diffs)
{
    if (faabric::util::isMockMode()) {
        std::lock_guard<std::mutex> lk(mockMutex);
        threadResults.emplace_back(host, std::make_tuple((int)messageId, returnValue, key, (int)diffs.size()));
        return;
    }
    SPDLOG_DEBUG("Sending thread result for {} to {} (plus {} snapshot diffs)", messageId, host, diffs.size());
    faabric::ThreadResultRequest req;
    req.set_appid((int32_t)appId);
    req.set_messageid((int32_t)messageId);
    req.set_returnvalue(returnValue);
    req.set_key(key);
    fillDiffs(req.mutable_diffs(), diffs);
    faabric::EmptyResponse resp;
    syncSend(SnapshotCalls::ThreadResult, &req, &resp);
}

void SnapshotClient::pushDeviceSnapshot(const std::string& key, const DeviceSnapshotDescriptor& desc)
{
    SPDLOG_DEBUG("Pushing device snapshot descriptor {} to {} ({} bytes stay on GPU {})", key, host, desc.size, desc.device);
    if (faabric::util::isMockMode()) {
        std::lock_guard<std::mutex> lk(mockMutex);
        deviceSnapshotPushes.emplace_back(host, key, desc);
        return;
    }
    faabric::SnapshotPushRequest req;
    req.set_key(key);
    req.set_deviceresident(true);
    req.set_devicesize(desc.size);
    req.set_deviceid(desc.device);
    req.set_ownerpid(desc.ownerPid);
    req.set_deviceptr(desc.devicePtr);
    req.set_ipchandle(desc.ipcHandle.data(), desc.ipcHandle.size());
    fillRegions(req.mutable_mergeregions(), desc.mergeRegions);
    faabric::EmptyResponse resp;
    syncSend(SnapshotCalls::PushSnapshot, &req, &resp);
}

void SnapshotClient::pushDeviceThreadResult(uint32_t appId,
                                            uint32_t messageId,
                                            int returnValue,
                                            const std::string& key,
                                            uint64_t diffBytes)
{
    if (faabric::util::isMockMode()) {
        std::lock_guard<std::mutex> lk(mockMutex);
        threadResults.emplace_back(host, std::make_tuple((int)messageId, returnValue, key, 0));
        return;
    }
    SPDLOG_DEBUG("Sending thread result for {} to {} ({} bytes already merged on the device)", messageId, host, diffBytes);
    faabric::ThreadResultRequest req;
    req.set_appid((int32_t)appId);
    req.set_messageid((int32_t)messageId);
    req.set_returnvalue(returnValue);
    req.set_key(key);
    req.set_devicemerged(true);
    req.set_devicediffbytes(diffBytes);
    faabric::EmptyResponse resp;
    syncSend(SnapshotCalls::ThreadResult, &req, &resp);
}

// ---------------------------------------------------------------------------
// Server
// ---------------------------------------------------------------------------
SnapshotServer::SnapshotServer()
  : faabric::transport::MessageEndpointServer(SNAPSHOT_ASYNC_PORT,
                                              SNAPSHOT_SYNC_PORT,
                                              SNAPSHOT_INPROC_LABEL,
                                              faabric::util::getSystemConfig().snapshotServerThreads)
  , reg(faabric::snapshot::getSnapshotRegistry())
{}

void SnapshotServer::doAsyncRecv(transport::Message& message)
{
    uint8_t header = message.getMessageCode();
    if (header == SnapshotCalls::DeleteSnapshot) {
        recvDeleteSnapshot(message.udata());
        return;
    }
    throw std::runtime_error("Unrecognized async call header: " + std::to_string(header));
}

std::string SnapshotServer::doSyncRecv(transport::Message& message)
{
    uint8_t header = message.getMessageCode();
    switch (header) {
        case SnapshotCalls::PushSnapshot:
            return recvPushSnapshot(message.udata());
        case SnapshotCalls::PushSnapshotUpdate:
            return recvPushSnapshotUpdate(message.udata());
        case SnapshotCalls::ThreadResult:
            return recvThreadResult(message);
        default:
            throw std::runtime_error("Unrecognized sync call header: " + std::to_string(header));
    }
}

std::string SnapshotServer::recvPushSnapshot(std::span<const uint8_t> buffer)
{
    faabric::SnapshotPushRequest r;
    if (!r.ParseFromArray(buffer.data(), (int)buffer.size())) {
        throw std::runtime_error("Could not parse snapshot push");
    }
    if (r.deviceresident()) {
        // Control descriptor only: the image stays where it is (HBM of a GPU
        // of this box); it is mapped on first use
        DeviceSnapshotDescriptor d;
        d.size = r.devicesize();
        d.device = r.deviceid();
        d.ownerPid = r.ownerpid();
        d.devicePtr = r.deviceptr();
        d.ipcHandle.assign(r.ipchandle().data(), r.ipchandle().size());
        for (const auto& mr : r.mergeregions()) {
            d.mergeRegions.emplace_back(mr.offset(), mr.length(), (SnapshotDataType)mr.datatype(), (SnapshotMergeOperation)mr.mergeop());
        }
        SPDLOG_DEBUG("Receiving device snapshot descriptor {} ({} bytes on GPU {} of pid {})", r.key(), d.size, d.device, d.ownerPid);
        reg.registerDeviceDescriptor(r.key(), d);
        return faabric::EmptyResponse().SerializeAsString();
    }
    if (r.contents().empty()) {
        SPDLOG_ERROR("Received shapshot {} with zero size", r.key());
        throw std::runtime_error("Received snapshot with zero size");
    }
    SPDLOG_DEBUG("Receiving snapshot {} (size {}, max-size {})", r.key(), r.contents().size(), r.maxsize());
    auto snap = std::make_shared<SnapshotData>(
      std::span<const uint8_t>((const uint8_t*)r.contents().data(), r.contents().size()), r.maxsize());
    for (const auto& mr : r.mergeregions()) {
        snap->addMergeRegion(mr.offset(),
                             mr.length(),
                             (SnapshotDataType)mr.datatype(),
                             (SnapshotMergeOperation)mr.mergeop());
    }
    reg.registerSnapshot(r.key(), snap);
    // The initial copy-in is not a change worth tracking
    snap->clearTrackedChanges();
    return faabric::EmptyResponse().SerializeAsString();
}

std::string SnapshotServer::recvPushSnapshotUpdate(std::span<const uint8_t> buffer)
{
    faabric::SnapshotUpdateRequest r;
    if (!r.ParseFromArray(buffer.data(), (int)buffer.size())) {
        throw std::runtime_error("Could not parse snapshot update");
    }
    SPDLOG_DEBUG("Queueing {} diffs for snapshot {}", r.diffs_size(), r.key());
    auto snap = reg.getSnapshot(r.key());
    // Merge regions are replaced wholesale
    snap->clearMergeRegions();
    for (const auto& mr : r.mergeregions()) {
        snap->addMergeRegion(mr.offset(),
                             mr.length(),
                             (SnapshotDataType)mr.datatype(),
                             (SnapshotMergeOperation)mr.mergeop());
    }
    std::vector<SnapshotDiff> diffs;
    diffs.reserve(r.diffs_size());
    for (const auto& d : r.diffs()) {
        diffs.emplace_back((SnapshotDataType)d.datatype(),
                           (SnapshotMergeOperation)d.mergeop(),
                           d.offset(),
                           std::span<const uint8_t>((const uint8_t*)d.data().data(), d.data().size()));
    }
    // Applied straight away (the payloads die with this request)
    snap->applyDiffs(diffs);
    return faabric::EmptyResponse().SerializeAsString();
}

std::string SnapshotServer::recvThreadResult(transport::Message& message)
{
    auto r = std::make_shared<faabric::ThreadResultRequest>();
    if (!r->ParseFromArray(message.udata().data(), (int)message.udata().size())) {
        throw std::runtime_error("Could not parse thread result");
    }
    if (r->diffs_size() > 0) {
        auto snap = reg.getSnapshot(r->key());
        std::vector<SnapshotDiff> diffs;
        diffs.reserve(r->diffs_size());
        for (const auto& d : r->diffs()) {
            diffs.emplace_back((SnapshotDataType)d.datatype(),
                               (SnapshotMergeOperation)d.mergeop(),
                               d.offset(),
                               std::span<const uint8_t>((const uint8_t*)d.data().data(), d.data().size()));
        }
        // Queued (merged later by the main thread); the queue copies the bytes
        snap->queueDiffs(diffs);
    }
    SPDLOG_DEBUG("Receiving thread result {} for message {} with {} diffs", r->returnvalue(), r->messageid(), r->diffs_size());
    faabric::scheduler::getScheduler().setThreadResultLocally(
      (uint32_t)r->appid(), (uint32_t)r->messageid(), r->returnvalue(), message);
    return faabric::EmptyResponse().SerializeAsString();
}

void SnapshotServer::recvDeleteSnapshot(std::span<const uint8_t> buffer)
{
    faabric::SnapshotDeleteRequest r;
    r.ParseFromArray(buffer.data(), (int)buffer.size());
    SPDLOG_DEBUG("Deleting shapshot {}", r.key());
    reg.deleteSnapshot(r.key());
}

// ---------------------------------------------------------------------------
// Device snapshot
// ---------------------------------------------------------------------------
#define DS_CUDA(expr)                                                          \
    do {                                                                       \
        cudaError_t _e = (expr);                                               \
        if (_e != cudaSuccess) {                                               \
            throw std::runtime_error(std::string(#expr) + ": " + cudaGetErrorString(_e)); \
        }                                                                      \
    } while (0)

namespace {
struct DeviceGuard
{
    int prev = -1;
    explicit DeviceGuard(int dev)
    {
        cudaGetDevice(&prev);
        cudaSetDevice(dev);
    }
    ~DeviceGuard()
    {
        if (prev >= 0) {
            cudaSetDevice(prev);
        }
    }
};
}

static std::atomic<uint64_t> nextDeviceSnapshotUid{ 1 };

DeviceSnapshot::DeviceSnapshot(size_t sizeIn, int deviceIn)
  : size(sizeIn)
  , device(deviceIn)
{
    owned = faabric::util::allocateDeviceMemory(size, device);
    image = owned.ptr;
    DeviceGuard g(device);
    DS_CUDA(cudaMemset(image, 0, size));
    statsDev = faabric::util::allocateDeviceMemory(64, device);
    // one stamp per 4 KiB page
    const size_t nPages = (size + 4095) / 4096;
    stampsDev = faabric::util::allocateDeviceMemory(std::max<size_t>(1, nPages) * sizeof(uint32_t), device);
    DS_CUDA(cudaMemset(stampsDev.ptr, 0, std::max<size_t>(1, nPages) * sizeof(uint32_t)));
    uniqueId = nextDeviceSnapshotUid.fetch_add(1);
}

DeviceSnapshot::DeviceSnapshot(uint8_t* devicePtr, size_t sizeIn, int deviceIn)
  : size(sizeIn)
  , device(deviceIn)
  , image(devicePtr)
{
    statsDev = faabric::util::allocateDeviceMemory(64, device);
    uniqueId = nextDeviceSnapshotUid.fetch_add(1);
}

uint32_t* DeviceSnapshot::pageStamps()
{
    return (uint32_t*)stampsDev.ptr;
}

uint32_t DeviceSnapshot::beginFork()
{
    return 2 * (forkCounter.fetch_add(1) + 1);
}

uint64_t* DeviceSnapshot::pageStatsOn(int onDevice)
{
    std::lock_guard<std::mutex> lk(mx);
    auto it = pageStatsDev.find(onDevice);
    if (it == pageStatsDev.end()) {
        auto region = faabric::util::allocateDeviceMemory(64, onDevice);
        DeviceGuard g(onDevice);
        DS_CUDA(cudaMemset(region.ptr, 0, 64));
        it = pageStatsDev.emplace(onDevice, std::move(region)).first;
    }
    return (uint64_t*)it->second.ptr;
}

DeviceSnapshot::~DeviceSnapshot()
{
    if (ipcMapped != nullptr) {
        cudaIpcCloseMemHandle(ipcMapped);
        cudaGetLastError();
    }
}

static std::atomic<uint64_t> globalDiffPushCount{ 0 };

uint64_t DeviceSnapshot::getGlobalDiffPushCount()
{
    return globalDiffPushCount.load();
}

DeviceSnapshotDescriptor DeviceSnapshot::describe()
{
    DeviceSnapshotDescriptor d;
    d.size = size;
    d.device = device;
    d.ownerPid = (int)::getpid();
    d.devicePtr = (uint64_t)(uintptr_t)image;
    d.mergeRegions = getMergeRegions();
    if (owned.ptr != nullptr && ipcMapped == nullptr) {
        DeviceGuard g(device);
        cudaIpcMemHandle_t h;
        if (cudaIpcGetMemHandle(&h, image) == cudaSuccess) {
            d.ipcHandle.assign((const char*)&h, sizeof(h));
        } else {
            cudaGetLastError(); // e.g. VMM-backed memory: same-process use only
        }
    }
    return d;
}

std::shared_ptr<DeviceSnapshot> DeviceSnapshot::fromDescriptor(const DeviceSnapshotDescriptor& desc)
{
    if (desc.ipcHandle.size() != sizeof(cudaIpcMemHandle_t)) {
        throw std::runtime_error("Device snapshot descriptor carries no IPC handle");
    }
    cudaIpcMemHandle_t h;
    memcpy(&h, desc.ipcHandle.data(), sizeof(h));
    void* p = nullptr;
    DS_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    int cur = 0;
    cudaGetDevice(&cur);
    auto snap = std::make_shared<DeviceSnapshot>((uint8_t*)p, (size_t)desc.size, cur);
    snap->ipcMapped = p;
    for (const auto& r : desc.mergeRegions) {
        snap->addMergeRegion(r.offset, r.length, r.dataType, r.operation);
    }
    return snap;
}

void DeviceSnapshot::copyInData(std::span<const uint8_t> hostData, uint64_t offset)
{
    if (offset + hostData.size() > size) {
        throw std::runtime_error("Copying data beyond the end of the device snapshot");
    }
    DeviceGuard g(device);
    DS_CUDA(cudaMemcpy(image + offset, hostData.data(), hostData.size(), cudaMemcpyHostToDevice));
    noteFullMutation();
}

std::vector<uint8_t> DeviceSnapshot::getDataCopy(uint64_t offset, size_t n)
{
    if (offset + n > size) {
        throw std::runtime_error("Out of bounds device snapshot access");
    }
    std::vector<uint8_t> out(n);
    DeviceGuard g(device);
    DS_CUDA(cudaMemcpy(out.data(), image + offset, n, cudaMemcpyDeviceToHost));
    return out;
}

std::shared_ptr<SnapshotData> DeviceSnapshot::spillToHost()
{
    auto host = std::make_shared<SnapshotData>(size);
    if (size > 0) {
        // D2H in bounded pieces through one pinned-size staging vector
        constexpr size_t PIECE = (size_t)64 << 20;
        for (size_t off = 0; off < size; off += PIECE) {
            size_t n = std::min(PIECE, size - off);
            std::vector<uint8_t> piece = getDataCopy(off, n);
            host->copyInData(piece, off);
        }
    }
    for (const auto& r : getMergeRegions()) {
        host->addMergeRegion(r.offset, r.length, r.dataType, r.operation);
    }
    host->clearTrackedChanges();
    return host;
}

std::shared_ptr<DeviceSnapshot> DeviceSnapshot::fromHost(SnapshotData& host, int device)
{
    auto snap = std::make_shared<DeviceSnapshot>(host.getSize(), device);
    if (host.getSize() > 0) {
        snap->copyInData({ host.getDataPtr(), host.getSize() });
    }
    for (const auto& r : host.getMergeRegions()) {
        snap->addMergeRegion(r.offset, r.length, r.dataType, r.operation);
    }
    return snap;
}

void DeviceSnapshot::restoreTo(uint8_t* deviceMem, size_t n, void* stream)
{
    if (n > size) {
        throw std::runtime_error("Target memory larger than device snapshot");
    }
    DeviceGuard g(device);
    DS_CUDA(cudaMemcpyAsync(deviceMem, image, n, cudaMemcpyDefault, (cudaStream_t)stream));
}

void DeviceSnapshot::addMergeRegion(uint64_t offset,
                                    size_t length,
                                    SnapshotDataType dataType,
                                    SnapshotMergeOperation operation)
{
    std::lock_guard<std::mutex> lk(mx);
    mergeRegions.emplace_back(offset, length, dataType, operation);
    regionsDirty = true;
}

void DeviceSnapshot::clearMergeRegions()
{
    std::lock_guard<std::mutex> lk(mx);
    mergeRegions.clear();
    regionsDirty = true;
}

std::vector<SnapshotMergeRegion> DeviceSnapshot::getMergeRegions()
{
    std::lock_guard<std::mutex> lk(mx);
    return mergeRegions;
}

extern "C" int fb_snapshot_prepare_regions(const FbMergeRegionDev* in,
                                           int nIn,
                                           int fillOp,
                                           uint64_t size,
                                           FbMergeRegionDev* out,
                                           int maxOut,
                                           int32_t* typedOut,
                                           int* nTypedOut);

void DeviceSnapshot::uploadRegions()
{
    // Caller holds mx
    std::vector<FbMergeRegionDev> in;
    for (const auto& r : mergeRegions) {
        in.push_back({ r.offset, r.length, (int32_t)r.dataType, (int32_t)r.operation });
    }
    int fillOp = faabric::util::getSystemConfig().diffingMode == "bytewise" ? FB_MERGE_BYTEWISE : FB_MERGE_XOR;
    int cap = 2 * (int)in.size() + 2;
    std::vector<FbMergeRegionDev> out(cap);
    std::vector<int32_t> typed(cap);
    int nTyped = 0;
    int n = fb_snapshot_prepare_regions(in.data(), (int)in.size(), fillOp, size, out.data(), cap, typed.data(), &nTyped);
    if (n == FB_E_INVALID) {
        throw std::runtime_error("Overlapping merge regions");
    }
    if (n < 0) {
        throw std::runtime_error("Too many merge regions");
    }
    DeviceGuard g(device);
    regionsDev = faabric::util::allocateDeviceMemory(std::max<size_t>(1, (size_t)n) * sizeof(FbMergeRegionDev), device);
    typedIdxDev = faabric::util::allocateDeviceMemory(std::max<size_t>(1, (size_t)nTyped) * sizeof(int32_t), device);
    DS_CUDA(cudaMemcpy(regionsDev.ptr, out.data(), (size_t)n * sizeof(FbMergeRegionDev), cudaMemcpyHostToDevice));
    if (nTyped > 0) {
        DS_CUDA(cudaMemcpy(typedIdxDev.ptr, typed.data(), (size_t)nTyped * sizeof(int32_t), cudaMemcpyHostToDevice));
    }
    nRegionsDev = n;
    nTypedDev = nTyped;
    regionsDirty = false;
}

// The fused kernel stores straight into `target`: when that lives on another
// GPU the launching device needs peer access to it (cudaMalloc memory is not
// peer-mapped by default, unlike the communicators' VMM heaps)
static void ensurePeerAccessTo(int fromDevice, const void* target)
{
    static std::mutex peerMx;
    static std::set<std::pair<int, int>> enabled;
    cudaPointerAttributes attr{};
    if (cudaPointerGetAttributes(&attr, target) != cudaSuccess || attr.type != cudaMemoryTypeDevice) {
        cudaGetLastError();
        return;
    }
    if (attr.device == fromDevice) {
        return;
    }
    std::lock_guard<std::mutex> lk(peerMx);
    if (!enabled.insert({ fromDevice, attr.device }).second) {
        return;
    }
    DeviceGuard g(fromDevice);
    cudaError_t e = cudaDeviceEnablePeerAccess(attr.device, 0);
    if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) {
        SPDLOG_ERROR("No peer access from GPU {} to GPU {}: {}", fromDevice, attr.device, cudaGetErrorString(e));
    }
    cudaGetLastError();
}

void DeviceSnapshot::diffAndPush(const uint8_t* mem,
                                 size_t memSize,
                                 uint8_t* mainImage,
                                 const uint8_t* dirtyPagesDev,
                                 bool updateBase,
                                 void* stream)
{
    std::lock_guard<std::mutex> lk(mx);
    if (regionsDirty) {
        uploadRegions();
    }
    DeviceGuard g(device);
    if (mainImage != nullptr) {
        ensurePeerAccessTo(device, mainImage);
    }
    DS_CUDA(cudaMemsetAsync(statsDev.ptr, 0, 16, (cudaStream_t)stream));
    fb::SnapDiffArgs a;
    memset(&a, 0, sizeof(a));
    a.mem = mem;
    a.orig = image;
    a.origW = updateBase ? image : nullptr;
    a.dst = mainImage;
    a.size = std::min(memSize, size);
    a.regions = (const FbMergeRegionDev*)regionsDev.ptr;
    a.nRegions = nRegionsDev;
    a.typedIdx = (const int32_t*)typedIdxDev.ptr;
    a.nTyped = nTypedDev;
    a.dirtyPages = dirtyPagesDev;
    a.stats = (uint64_t*)statsDev.ptr;
    a.updateBase = updateBase ? 1 : 0;
    if (pushStamps != nullptr && mainImage != nullptr) {
        ensurePeerAccessTo(device, pushStamps);
        a.pageStampOut = pushStamps;
        a.pageStamp = pushStamp;
    }
    DS_CUDA(fb::launchSnapshotDiffPush(a, FB_NUM_SMS * 2, (cudaStream_t)stream));
    diffPushCount++;
    globalDiffPushCount.fetch_add(1);
}

std::vector<uint8_t> DeviceSnapshot::serializeDelta(const faabric::util::DeltaSettings& cfg, const uint8_t* mem, size_t memSize)
{
    if (memSize > size || memSize > UINT32_MAX) {
        throw std::runtime_error("Delta of a device image: new data must fit the image (and 4 GiB)");
    }
    if (!cfg.usePages || cfg.pageSize != 4096) {
        // not the device's granularity: encode from host copies
        std::vector<uint8_t> oldHost = getDataCopy(0, memSize);
        std::vector<uint8_t> newHost(memSize);
        DeviceGuard g(device);
        DS_CUDA(cudaMemcpy(newHost.data(), mem, memSize, cudaMemcpyDeviceToHost));
        return faabric::util::serializeDelta(cfg, oldHost.data(), oldHost.size(), newHost.data(), newHost.size());
    }
    // 1. which pages changed (compare kernel, one flag per page back to the host)
    std::vector<char> dirty = getDirtyPages(mem, memSize);
    std::vector<uint32_t> pages;
    for (size_t p = 0; p < dirty.size(); p++) {
        if (dirty[p]) {
            pages.push_back((uint32_t)p);
        }
    }
    std::vector<uint8_t> cmds;
    faabric::util::deltaBegin(cmds, (uint32_t)memSize);
    if (!pages.empty()) {
        // 2. gather them (as new ^ old when the settings say so) into a compact buffer
        DeviceGuard g(device);
        auto listDev = faabric::util::allocateDeviceMemory(pages.size() * sizeof(uint32_t), device);
        auto outDev = faabric::util::allocateDeviceMemory(pages.size() * 4096, device);
        DS_CUDA(cudaMemcpy(listDev.ptr, pages.data(), pages.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
        DS_CUDA(fb::launchPageGather(
          image, mem, (const uint32_t*)listDev.ptr, (uint32_t)pages.size(), memSize, cfg.xorWithOld ? 1 : 0, outDev.ptr, FB_NUM_SMS * 2, nullptr));
        std::vector<uint8_t> compact(pages.size() * 4096);
        DS_CUDA(cudaMemcpy(compact.data(), outDev.ptr, compact.size(), cudaMemcpyDeviceToHost));
        // 3. runs of consecutive pages become one command each
        size_t k = 0;
        while (k < pages.size()) {
            size_t e = k + 1;
            while (e < pages.size() && pages[e] == pages[e - 1] + 1) {
                e++;
            }
            const uint64_t off = (uint64_t)pages[k] * 4096;
            const uint64_t len = std::min<uint64_t>((uint64_t)(e - k) * 4096, memSize - off);
            faabric::util::deltaAppendRun(cmds, cfg.xorWithOld, (uint32_t)off, compact.data() + k * 4096, (uint32_t)len);
            k = e;
        }
    }
    return faabric::util::deltaFinish(cfg, std::move(cmds));
}

void DeviceSnapshot::applyDelta(const std::vector<uint8_t>& delta, void* stream)
{
    std::vector<SnapshotDiff> diffs;
    // (payloads of a compressed delta only live inside the walk: keep copies)
    std::deque<std::vector<uint8_t>> payloads;
    faabric::util::deltaForEach(
      delta,
      [&](uint32_t total) {
          if (total > size) {
              throw std::runtime_error("Delta is larger than the device image");
          }
      },
      [&](bool isXor, uint32_t offset, const uint8_t* payload, uint32_t length) {
          if ((uint64_t)offset + length > size) {
              throw std::runtime_error("Delta run beyond the end of the device image");
          }
          payloads.emplace_back(payload, payload + length);
          diffs.emplace_back(SnapshotDataType::Raw,
                             isXor ? SnapshotMergeOperation::XOR : SnapshotMergeOperation::Bytewise,
                             offset,
                             std::span<const uint8_t>(payloads.back().data(), length));
      });
    applyDiffs(diffs, stream);
}

void DeviceSnapshot::syncPagesFrom(const uint8_t* mem, size_t n, uint32_t stamp, void* stream)
{
    if (n > size) {
        throw std::runtime_error("Source memory larger than device snapshot");
    }
    DeviceGuard g(device);
    ensurePeerAccessTo(device, mem);
    DS_CUDA(fb::launchPageSync(mem, image, pageStamps(), stamp, n, pageStatsOn(device), FB_NUM_SMS * 2, (cudaStream_t)stream));
}

void DeviceSnapshot::pullChangedPages(uint8_t* dst1, uint8_t* dst2, uint32_t since, size_t n, int onDevice, void* stream)
{
    if (n > size) {
        throw std::runtime_error("Target memory larger than device snapshot");
    }
    if (pageStamps() == nullptr) {
        throw std::runtime_error("This device snapshot keeps no page stamps");
    }
    DeviceGuard g(onDevice);
    ensurePeerAccessTo(onDevice, image);
    ensurePeerAccessTo(onDevice, pageStamps());
    DS_CUDA(fb::launchPagePull(image, dst1, dst2, pageStamps(), since, n, pageStatsOn(onDevice), FB_NUM_SMS * 2, (cudaStream_t)stream));
}

uint64_t DeviceSnapshot::takePageCopyCount(int onDevice, void* stream)
{
    uint64_t* dev = pageStatsOn(onDevice);
    uint64_t host = 0;
    DeviceGuard g(onDevice);
    DS_CUDA(cudaMemcpyAsync(&host, dev, sizeof(host), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    DS_CUDA(cudaMemsetAsync(dev, 0, sizeof(host), (cudaStream_t)stream));
    DS_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    return host;
}

DeviceDiffStats DeviceSnapshot::getLastStats(void* stream)
{
    uint64_t host[2] = { 0, 0 };
    DeviceGuard g(device);
    DS_CUDA(cudaMemcpyAsync(host, statsDev.ptr, sizeof(host), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    DS_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    return { host[0], host[1] };
}

void DeviceSnapshot::applyDiffs(const std::vector<SnapshotDiff>& diffs, void* stream)
{
    if (diffs.empty()) {
        return;
    }
    noteFullMutation();
    // The kernel applies the descriptors of one launch concurrently, the
    // reference applies a diff list in order (SnapshotData::applyDiffs).  Diffs
    // that touch the same bytes (several Sum diffs onto one scalar, a Bytewise
    // diff followed by an XOR ...) therefore go into successive "waves": a
    // diff's wave is one more than the highest wave among the earlier diffs it
    // overlaps.  Waves are launched back to back on the stream.
    std::vector<int> waveOf(diffs.size(), 0);
    int nWaves = 1;
    {
        std::map<uint64_t, std::pair<uint64_t, int>> spans; // start -> (end, wave)
        for (size_t i = 0; i < diffs.size(); i++) {
            uint64_t b = diffs[i].getOffset();
            uint64_t e = b + std::max<size_t>(diffs[i].getData().size(), 1);
            int wave = 0;
            auto it = spans.lower_bound(b);
            if (it != spans.begin()) {
                --it;
            }
            uint64_t nb = b;
            uint64_t ne = e;
            while (it != spans.end() && it->first < e) {
                if (it->second.first > b) {
                    wave = std::max(wave, it->second.second + 1);
                    nb = std::min(nb, it->first);
                    ne = std::max(ne, it->second.first);
                    it = spans.erase(it);
                } else {
                    ++it;
                }
            }
            spans[nb] = { ne, wave };
            waveOf[i] = wave;
            nWaves = std::max(nWaves, wave + 1);
        }
    }
    std::vector<FbDiffDesc> descs;
    std::vector<uint64_t> offs;
    std::vector<uint8_t> blob;
    std::vector<uint32_t> waveStart(nWaves + 1, 0);
    for (int w = 0; w < nWaves; w++) {
        waveStart[w] = (uint32_t)descs.size();
        for (size_t i = 0; i < diffs.size(); i++) {
            if (waveOf[i] != w) {
                continue;
            }
            const auto& d = diffs[i];
            descs.push_back({ d.getOffset(), d.getData().size(), (int32_t)d.getDataType(), (int32_t)d.getOperation() });
            offs.push_back(blob.size());
            blob.insert(blob.end(), d.getData().begin(), d.getData().end());
            blob.resize((blob.size() + 15) / 16 * 16);
        }
    }
    waveStart[nWaves] = (uint32_t)descs.size();
    DeviceGuard g(device);
    auto dDescs = faabric::util::allocateDeviceMemory(descs.size() * sizeof(FbDiffDesc), device);
    auto dOffs = faabric::util::allocateDeviceMemory(offs.size() * sizeof(uint64_t), device);
    auto dBlob = faabric::util::allocateDeviceMemory(std::max<size_t>(16, blob.size()), device);
    DS_CUDA(cudaMemcpy(dDescs.ptr, descs.data(), descs.size() * sizeof(FbDiffDesc), cudaMemcpyHostToDevice));
    DS_CUDA(cudaMemcpy(dOffs.ptr, offs.data(), offs.size() * sizeof(uint64_t), cudaMemcpyHostToDevice));
    if (!blob.empty()) {
        DS_CUDA(cudaMemcpy(dBlob.ptr, blob.data(), blob.size(), cudaMemcpyHostToDevice));
    }
    for (int w = 0; w < nWaves; w++) {
        uint32_t n = waveStart[w + 1] - waveStart[w];
        if (n == 0) {
            continue;
        }
        DS_CUDA(fb::launchSnapshotApply(image,
                                        size,
                                        (const FbDiffDesc*)dDescs.ptr + waveStart[w],
                                        (const uint64_t*)dOffs.ptr + waveStart[w],
                                        dBlob.ptr,
                                        n,
                                        (cudaStream_t)stream));
    }
    DS_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
}

std::vector<char> DeviceSnapshot::getDirtyPages(const uint8_t* mem, size_t memSize)
{
    return faabric::util::DeviceCompareDirtyTracker::getDirtyPages(mem, image, std::min(memSize, size), device);
}

} // namespace faabric::snapshot
