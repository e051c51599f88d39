#include "faabric/device/communicator.h"
#include "faabric/device/nvtx.h"

#include "faabric/device/bootstrap.h"
#include "faabric/device/cuda_driver.h"
#include "launch_api.h"
#include "loopback_kernels.h"

#include <algorithm>
#include <chrono>
#include <thread>
#include <cstdio>
#include <initializer_list>
#include <barrier>
#include <cstdlib>
#include <cstring>
#include <set>
#include <shared_mutex>
#include <stdexcept>
#include <unistd.h>

namespace faabric::device {

// ---------------------------------------------------------------------------
// helpers
// ---------------------------------------------------------------------------
#define CUDA_OK(expr)                                                          \
    do {                                                                       \
        cudaError_t _e = (expr);                                               \
        if (_e != cudaSuccess) {                                               \
            throw std::runtime_error(std::string(#expr) + ": " +               \
                                     cudaGetErrorString(_e));                  \
        }                                                                      \
    } while (0)

#define CU_OK(api, expr)                                                       \
    do {                                                                       \
        CUresult _r = (expr);                                                  \
        if (_r != CUDA_SUCCESS) {                                              \
            throw std::runtime_error(std::string(#expr) + ": " +               \
                                     (api).errStr(_r));                        \
        }                                                                      \
    } while (0)

static size_t roundUp(size_t v, size_t a)
{
    return (v + a - 1) / a * a;
}

static size_t envSize(const char* name, size_t def)
{
    const char* v = getenv(name);
    if (v == nullptr || *v == 0) {
        return def;
    }
    return (size_t)strtoull(v, nullptr, 10);
}

CommConfig CommConfig::fromEnv()
{
    CommConfig c;
    c.heapBytes = envSize("FAABRIC_SYMM_HEAP_BYTES", c.heapBytes);
    c.stageBytes = envSize("FAABRIC_STAGE_BYTES", c.stageBytes);
    c.slotBytes = envSize("FAABRIC_P2P_SLOT_BYTES", c.slotBytes);
    c.timeoutMs = envSize("FAABRIC_DEVICE_TIMEOUT_MS", c.timeoutMs);
    c.useVmm = envSize("FAABRIC_USE_VMM", 1) != 0;
    c.useMulticast = envSize("FAABRIC_USE_NVLS", 1) != 0;
    c.maxBlocks = (int)envSize("FAABRIC_COMM_BLOCKS", c.maxBlocks);
    c.channels = (int)envSize("FAABRIC_COMM_CHANNELS", c.channels);
    c.llMaxBytes = envSize("FAABRIC_LL_MAX_BYTES", c.llMaxBytes);
    c.oneShotMaxBytes = envSize("FAABRIC_ONESHOT_MAX_BYTES", c.oneShotMaxBytes);
    c.nvlsScalarMinBytes = envSize("FAABRIC_NVLS_SCALAR_MIN_BYTES", c.nvlsScalarMinBytes);
    c.tmaMinBytes = envSize("FAABRIC_TMA_MIN_BYTES", c.tmaMinBytes);
    c.nvlsMinBytes = envSize("FAABRIC_NVLS_MIN_BYTES", c.nvlsMinBytes);
    c.p2pBounceBytes = envSize("FAABRIC_P2P_BOUNCE_BYTES", c.p2pBounceBytes);
    c.groupBlocks = (int)envSize("FAABRIC_GROUP_BLOCKS", (size_t)c.groupBlocks);
    if (const char* be = getenv("FAABRIC_DEVICE_BACKEND")) {
        c.loopback = std::string(be) == "loopback";
    }
    if (getenv("FAABRIC_STREAM_SYNC") != nullptr) {
        c.streamSync = envSize("FAABRIC_STREAM_SYNC", 0) != 0 ? 1 : 0;
    }
    c.bcast2StepMinBytes =
      envSize("FAABRIC_BCAST_2STEP_MIN_BYTES", c.bcast2StepMinBytes);
    return c;
}

// ---------------------------------------------------------------------------
// Tuning file
// ---------------------------------------------------------------------------
namespace {
struct TuningKey
{
    const char* name;
    uint64_t (*get)(const CommConfig&);
    void (*set)(CommConfig&, uint64_t);
};
#define FB_TUNING_KEY(field, type)                                                       \
    TuningKey{ #field,                                                                   \
               [](const CommConfig& c) -> uint64_t { return (uint64_t)c.field; },        \
               [](CommConfig& c, uint64_t v) { c.field = (type)v; } }
const TuningKey TUNING_KEYS[] = {
    FB_TUNING_KEY(llMaxBytes, size_t),         FB_TUNING_KEY(oneShotMaxBytes, size_t),
    FB_TUNING_KEY(nvlsMinBytes, size_t),       FB_TUNING_KEY(nvlsScalarMinBytes, size_t),
    FB_TUNING_KEY(bcast2StepMinBytes, size_t), FB_TUNING_KEY(tmaMinBytes, size_t),
    FB_TUNING_KEY(maxBlocks, int),             FB_TUNING_KEY(threads, int),
    FB_TUNING_KEY(channels, int),              FB_TUNING_KEY(groupBlocks, int),
};
#undef FB_TUNING_KEY
const char* const ALGO_NAMES[FB_ALGO_COUNT] = { "auto", "oneshot", "twoshot", "nvls", "ll", "copy-engine" };
}

int CommTuning::algoFromName(const std::string& name)
{
    for (int i = 0; i < FB_ALGO_COUNT; i++) {
        if (name == ALGO_NAMES[i]) {
            return i;
        }
    }
    return -1;
}

const char* CommTuning::algoName(int algo)
{
    return algo >= 0 && algo < FB_ALGO_COUNT ? ALGO_NAMES[algo] : "?";
}

CommTuning CommTuning::parse(const std::string& text)
{
    // Hand-rolled tokeniser: no locale-dependent stream extraction
    CommTuning t;
    int lineNo = 0;
    auto bad = [&](const std::string& why) {
        throw std::runtime_error("tuning file line " + std::to_string(lineNo) + ": " + why);
    };
    auto number = [&](const std::string& tok) -> uint64_t {
        if (tok.empty() || tok.find_first_not_of("0123456789") != std::string::npos) {
            bad("'" + tok + "' is not a non-negative integer");
        }
        return strtoull(tok.c_str(), nullptr, 10);
    };
    size_t pos = 0;
    while (pos < text.size()) {
        size_t eol = text.find('\n', pos);
        if (eol == std::string::npos) {
            eol = text.size();
        }
        std::string line = text.substr(pos, eol - pos);
        pos = eol + 1;
        lineNo++;
        size_t hash = line.find('#');
        if (hash != std::string::npos) {
            line.resize(hash);
        }
        std::vector<std::string> tok;
        size_t i = 0;
        while (i < line.size()) {
            while (i < line.size() && isspace((unsigned char)line[i])) {
                i++;
            }
            size_t j = i;
            while (j < line.size() && !isspace((unsigned char)line[j])) {
                j++;
            }
            if (j > i) {
                tok.push_back(line.substr(i, j - i));
            }
            i = j;
        }
        if (tok.empty()) {
            continue;
        }
        if (tok[0] == "allreduce") {
            if (tok.size() != 3) {
                bad("expected 'allreduce <maxBytes> <algo>'");
            }
            int a = algoFromName(tok[2]);
            if (a <= FB_ALGO_AUTO || a == FB_ALGO_COPY_ENGINE) {
                bad("unknown all-reduce algorithm '" + tok[2] + "'");
            }
            t.allReduceTable.emplace_back(number(tok[1]), a);
        } else if (tok[0] == "set") {
            if (tok.size() != 3) {
                bad("expected 'set <key> <value>'");
            }
            bool known = false;
            for (const auto& k : TUNING_KEYS) {
                known = known || tok[1] == k.name;
            }
            if (!known) {
                bad("unknown key '" + tok[1] + "'");
            }
            t.settings.emplace_back(tok[1], number(tok[2]));
        } else {
            bad("unknown directive '" + tok[0] + "'");
        }
    }
    std::sort(t.allReduceTable.begin(), t.allReduceTable.end());
    return t;
}

bool CommTuning::loadFile(const std::string& path, CommTuning& out)
{
    FILE* f = fopen(path.c_str(), "rb");
    if (f == nullptr) {
        return false;
    }
    std::string text;
    char buf[4096];
    size_t n = 0;
    while ((n = fread(buf, 1, sizeof(buf), f)) > 0) {
        text.append(buf, n);
    }
    fclose(f);
    out = parse(text);
    return true;
}

std::string CommTuning::serialise() const
{
    std::string os = "# faabric_b200 communicator tuning\n";
    for (const auto& [key, value] : settings) {
        os += "set " + key + " " + std::to_string(value) + "\n";
    }
    for (const auto& [maxBytes, algo] : allReduceTable) {
        os += "allreduce " + std::to_string(maxBytes) + " " + algoName(algo) + "\n";
    }
    return os;
}

void CommTuning::applyTo(CommConfig& cfg) const
{
    for (const auto& [key, value] : settings) {
        for (const auto& k : TUNING_KEYS) {
            if (key == k.name) {
                k.set(cfg, value);
            }
        }
    }
    cfg.channels = std::clamp(cfg.channels, 1, FB_MAX_CHANNELS);
}

void Communicator::applyTuning(const CommTuning& tuning)
{
    // the lane count is fixed once the heap is laid out
    const int channels = cfg_.channels;
    tuning.applyTo(cfg_);
    cfg_.channels = channels;
    if (!tuning.allReduceTable.empty()) {
        allReduceTable_ = tuning.allReduceTable;
    }
}

void Communicator::applyTuningFromEnv()
{
    const char* path = getenv("FAABRIC_TUNING_FILE");
    if (path == nullptr || *path == 0) {
        return;
    }
    try {
        CommTuning t;
        if (CommTuning::loadFile(path, t)) {
            applyTuning(t);
        } else {
            fprintf(stderr, "faabric_b200: tuning file %s not readable, using built-in thresholds\n", path);
        }
    } catch (const std::exception& e) {
        fprintf(stderr, "faabric_b200: ignoring tuning file %s: %s\n", path, e.what());
    }
}

const char* Communicator::errorString(int code)
{
    switch (code) {
        case FB_OK:
            return "ok";
        case FB_E_UNSUPPORTED:
            return "unsupported (dtype, op) or layout";
        case FB_E_INVALID:
            return "invalid argument";
        case FB_E_CUDA:
            return "CUDA error";
        case FB_E_TOO_LARGE:
            return "message larger than staging area";
        case FB_E_NO_DEVICE:
            return "no CUDA device";
        default:
            return "unknown";
    }
}

namespace {
std::mutex loopRangesMx;
std::vector<std::pair<const uint8_t*, size_t>> loopRanges;
}

// Symmetric heaps of the communicators alive in this process: lets hot paths
// (every MPI call classifies its buffers) recognise heap memory with a range
// check instead of a driver query
namespace {
std::shared_mutex heapRangesMx;
std::vector<std::pair<const uint8_t*, size_t>> heapRanges;
std::atomic<int> nHeapRanges{ 0 };
std::atomic<int> nLoopRanges{ 0 };
}

bool Communicator::isHeapPointer(const void* p)
{
    if (nHeapRanges.load(std::memory_order_acquire) == 0) {
        return false;
    }
    std::shared_lock<std::shared_mutex> lk(heapRangesMx);
    for (const auto& [base, n] : heapRanges) {
        if ((const uint8_t*)p >= base && (const uint8_t*)p < base + n) {
            return true;
        }
    }
    return false;
}

bool Communicator::isLoopbackHeapPointer(const void* p)
{
    if (nLoopRanges.load(std::memory_order_acquire) == 0) {
        return false;
    }
    std::lock_guard<std::mutex> lk(loopRangesMx);
    for (const auto& [base, n] : loopRanges) {
        if ((const uint8_t*)p >= base && (const uint8_t*)p < base + n) {
            return true;
        }
    }
    return false;
}

// ---------------------------------------------------------------------------
// Backing memory
// ---------------------------------------------------------------------------
struct Communicator::Backing
{
    bool vmm = false;
    size_t mapSize = 0;
    // per rank (local mode: all ranks; ipc mode: index = rank)
    std::vector<CUmemGenericAllocationHandle> handles;
    std::vector<CUdeviceptr> vas;
    std::vector<void*> mallocPtrs;  // owned cudaMalloc allocations
    std::vector<int> mallocDevices;
    std::vector<void*> ipcOpened;   // cudaIpcOpenMemHandle results
    CUmemGenericAllocationHandle mcHandle = 0;
    std::vector<CUdeviceptr> mcVas;
    bool hasMc = false;
    std::vector<uint32_t*> errWords;
    std::vector<int> errDevices;
    std::vector<void*> hostAllocs; // loopback backend

    // Binds handles[firstRank + i] (on devices[i]) to the multicast object,
    // then maps the multicast range for the `access` devices
    uint8_t* bindMulticast(const DriverApi& api,
                           int firstRank,
                           const std::vector<int>& devices,
                           size_t gran,
                           const std::vector<int>& access);
    // Zeroes the signal pad and control areas at `base` and allocates the
    // rank's error word
    uint32_t* initDeviceRank(uint8_t* base, size_t controlBytes, int device);

    ~Backing()
    {
        if (!hostAllocs.empty()) {
            {
                std::lock_guard<std::mutex> lk(loopRangesMx);
                for (void* p : hostAllocs) {
                    size_t gone = std::erase_if(loopRanges, [p](const auto& r) { return r.first == (const uint8_t*)p; });
                    nLoopRanges.fetch_sub((int)gone, std::memory_order_release);
                }
            }
            for (void* p : hostAllocs) {
                ::free(p);
            }
            return;
        }
        const DriverApi& api = getDriverApi();
        for (void* p : ipcOpened) {
            cudaIpcCloseMemHandle(p);
        }
        for (size_t i = 0; i < mcVas.size(); i++) {
            if (mcVas[i] != 0) {
                api.cuMemUnmap(mcVas[i], mapSize);
                api.cuMemAddressFree(mcVas[i], mapSize);
            }
        }
        for (size_t i = 0; i < vas.size(); i++) {
            if (vas[i] != 0) {
                api.cuMemUnmap(vas[i], mapSize);
                api.cuMemAddressFree(vas[i], mapSize);
            }
        }
        for (auto h : handles) {
            if (h != 0) {
                api.cuMemRelease(h);
            }
        }
        if (hasMc && mcHandle != 0) {
            api.cuMemRelease(mcHandle);
        }
        for (size_t i = 0; i < mallocPtrs.size(); i++) {
            cudaSetDevice(mallocDevices[i]);
            cudaFree(mallocPtrs[i]);
        }
        for (size_t i = 0; i < errWords.size(); i++) {
            cudaSetDevice(errDevices[i]);
            cudaFreeHost(errWords[i]);
        }
        cudaGetLastError();
    }
};

struct Communicator::LocalGroup
{
    std::barrier<> bar;
    explicit LocalGroup(int n)
      : bar(n)
    {}
};

// this rank's signal pad, then the pads of the sub-communicator slots
static const size_t SIG_REGION = (size_t)(1 + FB_SUB_SLOTS) * FB_SIG_BYTES;
static_assert(FB_SIG_SBAR_OFF + FB_SIG_SBAR_WORDS <= FB_SIG_TOTAL_WORDS, "signal pad overflows its slot");
static_assert(FB_SUB_SLOTS <= 32, "slot masks are 32-bit");

void Communicator::computeLayout()
{
    int n = dev_.nranks;
    cfg_.stageBytes = roundUp(std::max<size_t>(cfg_.stageBytes, 1 << 16), 4096);
    cfg_.slotBytes = roundUp(std::max<size_t>(cfg_.slotBytes, 4096), 4096);
    cfg_.channels = std::clamp(cfg_.channels, 1, FB_MAX_CHANNELS);
    llOff_ = 0;
    p2pDescOff_ = roundUp(
      llOff_ + (uint64_t)cfg_.channels * FB_LL_AREA_BYTES(n), 4096);
    mboxOff_ = roundUp(p2pDescOff_ + FB_P2P_DESC_BYTES, 4096);
    cfg_.p2pBounceBytes =
      roundUp(std::max<size_t>(cfg_.p2pBounceBytes, 64 << 10), 8192);
    bounceSlotBytes_ = cfg_.p2pBounceBytes / 2;
    stageSendOff_ =
      roundUp(mboxOff_ + (uint64_t)n * cfg_.p2pBounceBytes, 4096);
    stageRecvOff_ = stageSendOff_ + cfg_.stageBytes;
    userOff_ = stageRecvOff_ + cfg_.stageBytes;
    heapTotal_ = userOff_ + roundUp(cfg_.heapBytes, 4096);
}

void Communicator::initAllocator()
{
    freeList_.clear();
    allocated_.clear();
    freeList_[userOff_] = heapTotal_ - userOff_;
}

static bool multicastSupported(const DriverApi& api, int device)
{
    if (api.cuMulticastCreate == nullptr) {
        return false;
    }
    CUdevice d;
    if (api.cuDeviceGet(&d, device) != CUDA_SUCCESS) {
        return false;
    }
    int v = 0;
    if (api.cuDeviceGetAttribute(
          &v, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, d) != CUDA_SUCCESS) {
        return false;
    }
    return v != 0;
}

static CUmemAllocationProp vmmProp(int device, CUmemAllocationHandleType handleType)
{
    CUmemAllocationProp prop;
    memset(&prop, 0, sizeof(prop));
    prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    prop.location.id = device;
    prop.requestedHandleTypes = handleType;
    return prop;
}

static CUmulticastObjectProp multicastProp(int nranks, size_t size, CUmemAllocationHandleType handleType)
{
    CUmulticastObjectProp mp;
    memset(&mp, 0, sizeof(mp));
    mp.numDevices = nranks;
    mp.size = size;
    mp.handleTypes = handleType;
    return mp;
}

// VMM allocation granularity of a heap of `bytes`.  `mc` is set when every
// device of `mcDevices` (none: multicast not wanted) supports multicast and
// the driver reports a multicast granularity; the result then covers both.
static size_t heapGranularity(const DriverApi& api,
                              int device,
                              CUmemAllocationHandleType handleType,
                              size_t bytes,
                              int nranks,
                              const std::vector<int>& mcDevices,
                              bool& mc)
{
    size_t gran = 0;
    CUmemAllocationProp prop = vmmProp(device, handleType);
    CU_OK(api, api.cuMemGetAllocationGranularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
    mc = !mcDevices.empty();
    for (int d : mcDevices) {
        mc = mc && multicastSupported(api, d);
    }
    if (mc) {
        CUmulticastObjectProp mp = multicastProp(nranks, bytes, handleType);
        size_t mcGran = 0;
        if (api.cuMulticastGetGranularity(&mcGran, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED) == CUDA_SUCCESS) {
            gran = std::max(gran, mcGran);
        } else {
            mc = false;
        }
    }
    return gran;
}

static void setAccess(const DriverApi& api,
                      CUdeviceptr va,
                      size_t size,
                      const std::vector<int>& devices)
{
    std::vector<CUmemAccessDesc> descs;
    for (int d : devices) {
        CUmemAccessDesc a;
        memset(&a, 0, sizeof(a));
        a.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
        a.location.id = d;
        a.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
        descs.push_back(a);
    }
    CU_OK(api, api.cuMemSetAccess(va, size, descs.data(), descs.size()));
}

// Reserves an address range into `va`, maps `h` there and opens it to `devices`
static uint8_t* mapHandle(const DriverApi& api,
                          CUdeviceptr& va,
                          CUmemGenericAllocationHandle h,
                          size_t size,
                          size_t gran,
                          const std::vector<int>& devices)
{
    CU_OK(api, api.cuMemAddressReserve(&va, size, gran, 0, 0));
    CU_OK(api, api.cuMemMap(va, size, 0, h, 0));
    setAccess(api, va, size, devices);
    return reinterpret_cast<uint8_t*>(va);
}

uint8_t* Communicator::Backing::bindMulticast(const DriverApi& api,
                                              int firstRank,
                                              const std::vector<int>& devices,
                                              size_t gran,
                                              const std::vector<int>& access)
{
    for (size_t i = 0; i < devices.size(); i++) {
        CUDA_OK(cudaSetDevice(devices[i]));
        CU_OK(api, api.cuMulticastBindMem(mcHandle, 0, handles[firstRank + i], 0, mapSize, 0));
    }
    mcVas.assign(1, 0);
    return mapHandle(api, mcVas[0], mcHandle, mapSize, gran, access);
}

uint32_t* Communicator::Backing::initDeviceRank(uint8_t* base, size_t controlBytes, int device)
{
    CUDA_OK(cudaSetDevice(device));
    CUDA_OK(cudaMemset(base, 0, controlBytes));
    // Watchdog error word: pinned host memory the kernels can write, so
    // the host reads it after a stream sync without a device round trip
    uint32_t* err = nullptr;
    CUDA_OK(cudaHostAlloc((void**)&err, 256, cudaHostAllocMapped | cudaHostAllocPortable));
    memset(err, 0, 256);
    errWords.push_back(err);
    errDevices.push_back(device);
    CUDA_OK(cudaDeviceSynchronize());
    return err;
}

// Per-rank set-up shared by both wiring modes: configuration, heap layout,
// allocator
std::shared_ptr<Communicator> Communicator::makeRank(const CommConfig& cfg, int rank, int nranks, int device)
{
    auto c = std::shared_ptr<Communicator>(new Communicator());
    c->cfg_ = cfg;
    c->applyTuningFromEnv();
    c->dev_.rank = rank;
    c->dev_.nranks = nranks;
    c->device_ = device;
    c->computeLayout();
    c->initAllocator();
    return c;
}

// Wiring tail shared by every backing: `bases[p]` is rank p's signal pad,
// followed by its heap
void Communicator::attach(const std::vector<uint8_t*>& bases,
                          uint8_t* mcBase,
                          uint32_t* err,
                          std::shared_ptr<Backing> backing,
                          const std::string& kind)
{
    for (int p = 0; p < dev_.nranks; p++) {
        dev_.sig[p] = reinterpret_cast<uint32_t*>(bases[p]);
        dev_.heap[p] = bases[p] + SIG_REGION;
    }
    dev_.mcHeap = mcBase ? mcBase + SIG_REGION : nullptr;
    dev_.err = err;
    dev_.timeoutNs = cfg_.timeoutMs * 1000000ull;
    backingState_ = std::move(backing);
    backing_ = kind;
    finishSetup();
}

// ---------------------------------------------------------------------------
// Local (single-process) creation
// ---------------------------------------------------------------------------
std::vector<std::shared_ptr<Communicator>> Communicator::createLocal(
  int nranks,
  const std::vector<int>& devices,
  const CommConfig& cfgIn)
{
    if (nranks < 1 || nranks > FB_MAX_RANKS || (int)devices.size() != nranks) {
        throw std::invalid_argument("createLocal: bad rank/device list");
    }
    if (!cfgIn.loopback && !cudaAvailable()) {
        throw std::runtime_error("createLocal: no CUDA device");
    }
    std::vector<std::shared_ptr<Communicator>> comms;
    for (int r = 0; r < nranks; r++) {
        comms.push_back(makeRank(cfgIn, r, nranks, devices[r]));
    }
    const size_t total = SIG_REGION + comms[0]->heapTotal_;
    auto backing = std::make_shared<Backing>();
    auto group = std::make_shared<LocalGroup>(nranks);
    std::vector<uint8_t*> bases(nranks, nullptr);
    if (cfgIn.loopback) {
        // ---- loopback: host memory, host twins of the kernels ----
        for (int r = 0; r < nranks; r++) {
            void* p = nullptr;
            if (posix_memalign(&p, 4096, total) != 0) {
                throw std::bad_alloc();
            }
            // only the control areas need zeroing (the user heap may be GiBs)
            memset(p, 0, SIG_REGION + comms[r]->userOff_);
            backing->hostAllocs.push_back(p);
            bases[r] = (uint8_t*)p;
            std::lock_guard<std::mutex> lk(loopRangesMx);
            loopRanges.emplace_back((const uint8_t*)p, total);
            nLoopRanges.fetch_add(1, std::memory_order_release);
        }
        for (int r = 0; r < nranks; r++) {
            void* e = nullptr;
            if (posix_memalign(&e, 256, 256) != 0) {
                throw std::bad_alloc();
            }
            memset(e, 0, 256);
            backing->hostAllocs.push_back(e);
            comms[r]->loop_ = true;
            comms[r]->localGroup_ = group;
            comms[r]->attach(bases, nullptr, (uint32_t*)e, backing, "loopback");
        }
        return comms;
    }
    std::set<int> distinct(devices.begin(), devices.end());
    std::vector<int> distinctDevs(distinct.begin(), distinct.end());
    const bool allDistinct = (int)distinct.size() == nranks;

    uint8_t* mcBase = nullptr;
    std::string kind = "cudaMalloc+peer";

    const DriverApi& api = getDriverApi();
    bool vmmDone = false;
    if (cfgIn.useVmm && api.loaded) {
        try {
            bool wantMc = false;
            const bool mcAllowed = cfgIn.useMulticast && allDistinct && nranks >= 2;
            const size_t gran = heapGranularity(
              api, devices[0], CU_MEM_HANDLE_TYPE_NONE, total, nranks, mcAllowed ? distinctDevs : std::vector<int>(), wantMc);
            backing->mapSize = roundUp(total, gran);
            backing->vmm = true;
            backing->handles.assign(nranks, 0);
            backing->vas.assign(nranks, 0);
            for (int r = 0; r < nranks; r++) {
                CUDA_OK(cudaSetDevice(devices[r]));
                CUDA_OK(cudaFree(0));
                CUmemAllocationProp prop = vmmProp(devices[r], CU_MEM_HANDLE_TYPE_NONE);
                CU_OK(api, api.cuMemCreate(&backing->handles[r], backing->mapSize, &prop, 0));
                bases[r] = mapHandle(api, backing->vas[r], backing->handles[r], backing->mapSize, gran, distinctDevs);
            }
            vmmDone = true;
            kind = "vmm";
            if (wantMc) {
                try {
                    CUmulticastObjectProp mcProp = multicastProp(nranks, backing->mapSize, CU_MEM_HANDLE_TYPE_NONE);
                    CU_OK(api, api.cuMulticastCreate(&backing->mcHandle, &mcProp));
                    backing->hasMc = true;
                    for (int r = 0; r < nranks; r++) {
                        CUdevice cd;
                        CU_OK(api, api.cuDeviceGet(&cd, devices[r]));
                        CU_OK(api, api.cuMulticastAddDevice(backing->mcHandle, cd));
                    }
                    mcBase = backing->bindMulticast(api, 0, devices, gran, distinctDevs);
                    kind = "vmm+multicast";
                } catch (const std::exception& e) {
                    fprintf(stderr,
                            "[faabric-b200] multicast unavailable: %s\n",
                            e.what());
                }
            }
        } catch (const std::exception& e) {
            if (vmmDone) {
                throw;
            }
            fprintf(stderr,
                    "[faabric-b200] VMM unavailable (%s), using cudaMalloc\n",
                    e.what());
            backing = std::make_shared<Backing>();
        }
    }
    if (!vmmDone) {
        for (int r = 0; r < nranks; r++) {
            CUDA_OK(cudaSetDevice(devices[r]));
            for (int d : distinctDevs) {
                if (d != devices[r]) {
                    cudaError_t e = cudaDeviceEnablePeerAccess(d, 0);
                    if (e != cudaSuccess &&
                        e != cudaErrorPeerAccessAlreadyEnabled) {
                        throw std::runtime_error(
                          std::string("cudaDeviceEnablePeerAccess: ") +
                          cudaGetErrorString(e));
                    }
                    cudaGetLastError();
                }
            }
            void* p = nullptr;
            CUDA_OK(cudaMalloc(&p, total));
            backing->mallocPtrs.push_back(p);
            backing->mallocDevices.push_back(devices[r]);
            bases[r] = (uint8_t*)p;
        }
    }

    // Load every kernel now: with lazy module loading the first launch of a
    // kernel may synchronise the context, which deadlocks against a rank
    // whose kernel is already spinning on this rank's flags
    for (int d : distinctDevs) {
        CUDA_OK(cudaSetDevice(d));
        CUDA_OK(fb::preloadAllKernels());
    }
    for (int r = 0; r < nranks; r++) {
        auto& c = comms[r];
        uint32_t* err = backing->initDeviceRank(bases[r], SIG_REGION + c->userOff_, devices[r]);
        c->localGroup_ = group;
        if (c->cfg_.streamSync < 0) {
            c->cfg_.streamSync = allDistinct ? 0 : 1;
        }
        c->attach(bases, mcBase, err, backing, kind);
    }
    return comms;
}

// ---------------------------------------------------------------------------
// Multi-process creation
// ---------------------------------------------------------------------------
std::shared_ptr<Communicator> Communicator::createIpc(int rank,
                                                      int nranks,
                                                      int device,
                                                      const std::string& jobId,
                                                      const CommConfig& cfgIn)
{
    if (nranks < 1 || nranks > FB_MAX_RANKS || rank < 0 || rank >= nranks) {
        throw std::invalid_argument("createIpc: bad rank");
    }
    if (!cudaAvailable()) {
        throw std::runtime_error("createIpc: no CUDA device");
    }
    auto c = makeRank(cfgIn, rank, nranks, device);
    c->bootstrap_ = std::make_shared<Bootstrap>(rank, nranks, jobId);
    Bootstrap& bs = *c->bootstrap_;

    CUDA_OK(cudaSetDevice(device));
    CUDA_OK(cudaFree(0));
    const size_t total = SIG_REGION + c->heapTotal_;
    auto backing = std::make_shared<Backing>();
    std::vector<uint8_t*> bases(nranks, nullptr);
    uint8_t* mcBase = nullptr;
    std::string kind;

    const DriverApi& api = getDriverApi();
    const CUmemAllocationHandleType fdType = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    // ---- stage 1: try VMM with POSIX fd export; all ranks must agree ----
    uint8_t vmmOk = 0;
    int myFd = -1;
    size_t gran = 0;
    size_t mapSize = 0;
    uint8_t mcWanted = 0;
    if (cfgIn.useVmm && api.loaded) {
        try {
            bool mc = false;
            const bool mcAllowed = cfgIn.useMulticast && nranks >= 2;
            gran = heapGranularity(
              api, device, fdType, total, nranks, mcAllowed ? std::vector<int>{ device } : std::vector<int>(), mc);
            mcWanted = mc ? 1 : 0;
            mapSize = roundUp(total, gran);
            backing->handles.assign(nranks, 0);
            backing->vas.assign(nranks, 0);
            CUmemAllocationProp prop = vmmProp(device, fdType);
            CU_OK(api, api.cuMemCreate(&backing->handles[rank], mapSize, &prop, 0));
            CU_OK(api, api.cuMemExportToShareableHandle(&myFd, backing->handles[rank], fdType, 0));
            vmmOk = 1;
        } catch (const std::exception& e) {
            fprintf(stderr,
                    "[faabric-b200] rank %d: VMM export failed: %s\n",
                    rank,
                    e.what());
            vmmOk = 0;
        }
    }
    {
        uint8_t st[2] = { vmmOk, mcWanted };
        auto all = bs.allGather(st, 2);
        for (int r = 0; r < nranks; r++) {
            vmmOk = vmmOk && all[2 * r];
            mcWanted = mcWanted && all[2 * r + 1];
        }
    }
    if (vmmOk) {
        backing->vmm = true;
        backing->mapSize = mapSize;
        std::vector<int> fds = bs.allGatherFds(myFd);
        ::close(myFd);
        for (int p = 0; p < nranks; p++) {
            if (p != rank) {
                CU_OK(api,
                      api.cuMemImportFromShareableHandle(
                        &backing->handles[p], (void*)(uintptr_t)fds[p], fdType));
            }
            ::close(fds[p]);
            bases[p] = mapHandle(api, backing->vas[p], backing->handles[p], mapSize, gran, { device });
        }
        kind = "vmm-ipc";
        // ---- multicast ----
        if (mcWanted) {
            uint8_t ok = 1;
            int mcFd = -1;
            try {
                if (rank == 0) {
                    CUmulticastObjectProp mp = multicastProp(nranks, mapSize, fdType);
                    CU_OK(api, api.cuMulticastCreate(&backing->mcHandle, &mp));
                    backing->hasMc = true;
                    CU_OK(api, api.cuMemExportToShareableHandle(&mcFd, backing->mcHandle, fdType, 0));
                }
            } catch (const std::exception& e) {
                fprintf(stderr,
                        "[faabric-b200] multicast create failed: %s\n",
                        e.what());
                ok = 0;
            }
            // rank 0 tells everybody whether an fd follows
            {
                auto all = bs.allGather(&ok, 1);
                ok = all[0];
            }
            if (ok) {
                int got = bs.broadcastFd(mcFd, 0);
                if (mcFd >= 0) {
                    ::close(mcFd);
                }
                uint8_t step = 1;
                try {
                    if (rank != 0) {
                        CU_OK(api,
                              api.cuMemImportFromShareableHandle(
                                &backing->mcHandle, (void*)(uintptr_t)got, fdType));
                        backing->hasMc = true;
                    }
                    CUdevice cd;
                    CU_OK(api, api.cuDeviceGet(&cd, device));
                    CU_OK(api, api.cuMulticastAddDevice(backing->mcHandle, cd));
                } catch (const std::exception& e) {
                    fprintf(stderr,
                            "[faabric-b200] rank %d multicast add failed: %s\n",
                            rank,
                            e.what());
                    step = 0;
                }
                ::close(got);
                {
                    auto all = bs.allGather(&step, 1);
                    for (int r = 0; r < nranks; r++) {
                        step = step && all[r];
                    }
                }
                if (step) {
                    uint8_t* mapped = nullptr;
                    try {
                        mapped = backing->bindMulticast(api, rank, { device }, gran, { device });
                    } catch (const std::exception& e) {
                        fprintf(stderr,
                                "[faabric-b200] rank %d multicast bind/map "
                                "failed: %s\n",
                                rank,
                                e.what());
                        step = 0;
                    }
                    auto all = bs.allGather(&step, 1);
                    for (int r = 0; r < nranks; r++) {
                        step = step && all[r];
                    }
                    if (step) {
                        mcBase = mapped;
                        kind = "vmm-ipc+multicast";
                    }
                }
            }
        }
    } else {
        // ---- legacy CUDA IPC ----
        if (myFd >= 0) {
            ::close(myFd);
        }
        backing = std::make_shared<Backing>();
        void* p = nullptr;
        CUDA_OK(cudaMalloc(&p, total));
        backing->mallocPtrs.push_back(p);
        backing->mallocDevices.push_back(device);
        cudaIpcMemHandle_t h;
        CUDA_OK(cudaIpcGetMemHandle(&h, p));
        auto all = bs.allGather(&h, sizeof(h));
        for (int q = 0; q < nranks; q++) {
            if (q == rank) {
                bases[q] = (uint8_t*)p;
                continue;
            }
            cudaIpcMemHandle_t ph;
            memcpy(&ph, all.data() + (size_t)q * sizeof(h), sizeof(h));
            void* mapped = nullptr;
            CUDA_OK(cudaIpcOpenMemHandle(
              &mapped, ph, cudaIpcMemLazyEnablePeerAccess));
            backing->ipcOpened.push_back(mapped);
            bases[q] = (uint8_t*)mapped;
        }
        kind = "cuda-ipc";
    }

    CUDA_OK(fb::preloadAllKernels());
    uint32_t* err = backing->initDeviceRank(bases[rank], SIG_REGION + c->userOff_, device);
    if (c->cfg_.streamSync < 0) {
        c->cfg_.streamSync = 0;
    }
    c->attach(bases, mcBase, err, backing, kind);
    // nobody may touch a peer's pad before it has been zeroed
    bs.barrier();
    return c;
}

void Communicator::bindDevice() const
{
    if (!loop_) {
        cudaSetDevice(device_);
    }
}

cudaStream_t Communicator::internalStream()
{
    if (loop_) {
        return nullptr;
    }
    if (internalStream_ == nullptr) {
        bindDevice();
        if (cudaStreamCreateWithFlags(&internalStream_, cudaStreamNonBlocking) != cudaSuccess) {
            cudaGetLastError();
            internalStream_ = nullptr;
        }
    }
    return internalStream_;
}

Communicator::~Communicator()
{
    if (parent_ != nullptr) {
        // Zero-on-release (comm_abi.h): every collective of this child has
        // completed on this rank, so no peer write to the pad is pending
        uint32_t* pad = dev_.sig[dev_.rank];
        bool zeroed = true;
        if (loop_) {
            memset(pad, 0, FB_SIG_BYTES);
        } else {
            // a stream of our own: a device-wide synchronise could wait for a
            // peer's kernel that waits for this rank
            bindDevice();
            cudaStream_t t = internalStream();
            zeroed = t != nullptr && cudaMemsetAsync(pad, 0, FB_SIG_BYTES, t) == cudaSuccess &&
                     cudaStreamSynchronize(t) == cudaSuccess;
            if (!zeroed) {
                // a slot whose pad may hold stale flags is never handed out again
                fprintf(stderr, "[faabric-b200] rank %d: zeroing sub-communicator slot %d failed\n", dev_.rank, slot_);
                cudaGetLastError();
            }
        }
        if (zeroed) {
            parent_->usedSlots_.fetch_and(~(1u << slot_));
        }
    }
    if (heapRegistered_) {
        std::unique_lock<std::shared_mutex> lk(heapRangesMx);
        const uint8_t* base = dev_.heap[dev_.rank];
        auto it = std::find_if(heapRanges.begin(), heapRanges.end(), [base](const auto& r) { return r.first == base; });
        if (it != heapRanges.end()) {
            heapRanges.erase(it);
            nHeapRanges.fetch_sub(1, std::memory_order_release);
        }
    }
    if (internalStream_ != nullptr) {
        bindDevice();
        cudaStreamDestroy(internalStream_);
        cudaGetLastError();
    }
    // Backing is shared: freed when the last rank's communicator dies
}

int Communicator::hostBarrier()
{
    if (parent_ != nullptr) {
        return FB_E_UNSUPPORTED;
    }
    if (bootstrap_) {
        bootstrap_->barrier();
    } else if (localGroup_) {
        localGroup_->bar.arrive_and_wait();
    }
    return FB_OK;
}

// ---------------------------------------------------------------------------
// Sub-communicators
// ---------------------------------------------------------------------------
std::shared_ptr<Communicator> Communicator::subset(const std::vector<int>& members, int slot, int* rcOut)
{
    int rcLocal = FB_OK;
    int& rc = rcOut ? *rcOut : rcLocal;
    rc = FB_OK;
    if (parent_ != nullptr) {
        rc = FB_E_UNSUPPORTED;
        return nullptr;
    }
    const int n = dev_.nranks;
    int self = -1;
    uint32_t seen = 0;
    for (size_t i = 0; i < members.size(); i++) {
        const int m = members[i];
        if (m < 0 || m >= n || (seen >> m) & 1u) {
            rc = FB_E_INVALID;
            return nullptr;
        }
        seen |= 1u << m;
        if (m == dev_.rank) {
            self = (int)i;
        }
    }
    if (self < 0 || slot < 0 || slot >= FB_SUB_SLOTS) {
        rc = FB_E_INVALID;
        return nullptr;
    }
    const uint32_t bit = 1u << slot;
    if (usedSlots_.fetch_or(bit) & bit) {
        rc = FB_E_INVALID;
        return nullptr;
    }
    auto c = std::shared_ptr<Communicator>(new Communicator());
    c->parent_ = shared_from_this();
    c->slot_ = slot;
    c->cfg_ = cfg_;
    c->allReduceTable_ = allReduceTable_;
    c->device_ = device_;
    c->backing_ = backing_;
    c->llOff_ = llOff_;
    c->mboxOff_ = mboxOff_;
    c->p2pDescOff_ = p2pDescOff_;
    c->bounceSlotBytes_ = bounceSlotBytes_;
    c->stageSendOff_ = stageSendOff_;
    c->stageRecvOff_ = stageRecvOff_;
    c->userOff_ = userOff_;
    c->heapTotal_ = heapTotal_;
    c->loop_ = loop_;
    c->k_ = k_;
    c->streamSync_ = streamSync_;
    c->streamWaitOk_ = streamWaitOk_;
    c->streamWriteOk_ = streamWriteOk_;
    c->dev_.rank = self;
    c->dev_.nranks = (int32_t)members.size();
    for (size_t i = 0; i < members.size(); i++) {
        c->dev_.heap[i] = dev_.heap[members[i]];
        c->dev_.sig[i] = dev_.sig[members[i]] + (size_t)(slot + 1) * FB_SIG_TOTAL_WORDS;
    }
    c->dev_.mcHeap = nullptr;
    c->dev_.err = dev_.err;
    c->dev_.timeoutNs = dev_.timeoutNs;
    return c;
}

uint32_t Communicator::freeSubsetSlots() const
{
    // a child cannot be split further
    return parent_ != nullptr ? 0u : ~usedSlots_.load() & ((1u << FB_SUB_SLOTS) - 1);
}

// ---------------------------------------------------------------------------
// Heap allocator (first fit, deterministic => symmetric across ranks)
// ---------------------------------------------------------------------------
uint64_t Communicator::alloc(size_t bytes, size_t align)
{
    if (parent_ != nullptr) {
        throw std::logic_error("alloc on a sub-communicator: allocate collectively on the parent");
    }
    std::lock_guard<std::mutex> lk(allocMx_);
    if (align < 256) {
        align = 256;
    }
    bytes = roundUp(std::max<size_t>(bytes, 1), 256);
    for (auto it = freeList_.begin(); it != freeList_.end(); ++it) {
        uint64_t start = roundUp(it->first, align);
        uint64_t pad = start - it->first;
        if (it->second >= pad + bytes) {
            uint64_t blockOff = it->first;
            uint64_t blockSize = it->second;
            freeList_.erase(it);
            if (pad > 0) {
                freeList_[blockOff] = pad;
            }
            uint64_t rest = blockSize - pad - bytes;
            if (rest > 0) {
                freeList_[start + bytes] = rest;
            }
            allocated_[start] = bytes;
            return start;
        }
    }
    throw std::bad_alloc();
}

void Communicator::free(uint64_t offset)
{
    if (parent_ != nullptr) {
        throw std::logic_error("free on a sub-communicator: free collectively on the parent");
    }
    std::lock_guard<std::mutex> lk(allocMx_);
    auto it = allocated_.find(offset);
    if (it == allocated_.end()) {
        return;
    }
    uint64_t size = it->second;
    allocated_.erase(it);
    auto ins = freeList_.emplace(offset, size).first;
    // coalesce with the next block
    auto next = std::next(ins);
    if (next != freeList_.end() && ins->first + ins->second == next->first) {
        ins->second += next->second;
        freeList_.erase(next);
    }
    if (ins != freeList_.begin()) {
        auto prev = std::prev(ins);
        if (prev->first + prev->second == ins->first) {
            prev->second += ins->second;
            freeList_.erase(ins);
        }
    }
}

uint8_t* Communicator::heapPtr(uint64_t offset, int rank) const
{
    if (rank < 0) {
        rank = dev_.rank;
    }
    return dev_.heap[rank] + offset;
}

bool Communicator::inHeap(const void* p, size_t bytes) const
{
    const uint8_t* b = dev_.heap[dev_.rank];
    const uint8_t* q = (const uint8_t*)p;
    return q >= b && q + bytes <= b + heapTotal_;
}

uint64_t Communicator::offsetOf(const void* p) const
{
    return (uint64_t)((const uint8_t*)p - dev_.heap[dev_.rank]);
}

// ---------------------------------------------------------------------------
// Kernel tables
// ---------------------------------------------------------------------------
namespace {
cudaError_t cudaReduce(const fb::ReduceArgs& a, int dtype, int op, int blocks, int threads, cudaStream_t s)
{
    return fb::findReduceLaunchers(dtype, op)->reduce(a, a.comm.nranks, blocks, threads, s);
}

cudaError_t cudaLL(const fb::LLArgs& a, int dtype, int op, cudaStream_t s)
{
    return fb::findReduceLaunchers(dtype, op)->ll(a, s);
}

cudaError_t cudaGroup(const fb::GroupArgs& a, int dtype, int op, int blocks, int threads, cudaStream_t s)
{
    return fb::findReduceLaunchers(dtype, op)->group(a, blocks, threads, s);
}

cudaError_t cudaGroupReduceScatter(const fb::GroupArgs& a, int dtype, int op, int blocks, int threads, cudaStream_t s)
{
    return fb::findReduceLaunchers(dtype, op)->groupRs(a, blocks, threads, s);
}

cudaError_t cudaCopy(void* dst, const void* src, size_t bytes, cudaStream_t s)
{
    return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, s);
}

cudaError_t cudaCopy2D(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t height, cudaStream_t s)
{
    return cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, height, cudaMemcpyDeviceToDevice, s);
}

const fb::KernelTable CUDA_KERNELS = {
    .reduce = cudaReduce,
    .ll = cudaLL,
    .group = cudaGroup,
    .groupReduceScatter = cudaGroupReduceScatter,
    .groupAllGather = fb::launchGroupAllGather,
    .move = fb::launchMove,
    .moveBulk = fb::launchMoveBulk,
    .barrier = fb::launchBarrier,
    .p2pSend = fb::launchP2PSend,
    .p2pPull = fb::launchP2PPull,
    .putSignal = fb::launchPutSignal,
    .waitSignal = fb::launchWaitSignal,
    .waitWord = fb::launchWaitWord,
    .signalPeers = fb::launchSignalPeers,
    .rmaAccumulate = fb::launchRmaAccumulate,
    .rmaCompareSwap = fb::launchRmaCompareSwap,
    .rmaCopyMany = fb::launchRmaCopyMany,
    .copy = cudaCopy,
    .copy2D = cudaCopy2D,
};

const fb::KernelTable HOST_KERNELS = {
    .reduce = fb::host::reduceKernel,
    .ll = fb::host::llAllReduce,
    .group = fb::host::groupAllReduce,
    .groupReduceScatter = fb::host::groupReduceScatter,
    .groupAllGather = fb::host::groupAllGather,
    .move = fb::host::moveKernel,
    .moveBulk = fb::host::moveBulk,
    .barrier = fb::host::barrierKernel,
    .p2pSend = fb::host::p2pSend,
    .p2pPull = fb::host::p2pPull,
    .putSignal = fb::host::putSignal,
    .waitSignal = fb::host::waitSignal,
    .waitWord = fb::host::waitWord,
    .signalPeers = fb::host::signalPeers,
    .rmaAccumulate = fb::host::rmaAccumulate,
    .rmaCompareSwap = fb::host::rmaCompareSwap,
    .rmaCopyMany = fb::host::rmaCopyMany,
    .copy = fb::host::copy,
    .copy2D = fb::host::copy2D,
};
}

// ---------------------------------------------------------------------------
// launch helpers
// ---------------------------------------------------------------------------
int Communicator::blocksFor(uint64_t vecs, int perThread) const
{
    uint64_t perBlock = (uint64_t)cfg_.threads * perThread;
    uint64_t b = (vecs + perBlock - 1) / perBlock;
    int maxB = std::min(cfg_.maxBlocks, FB_MAX_BLOCKS / cfg_.channels);
    if (b < 1) {
        b = 1;
    }
    if (b > (uint64_t)maxB) {
        b = maxB;
    }
    return (int)b;
}

static int alignWidth(uint64_t v)
{
    if ((v & 15) == 0) {
        return 16;
    }
    if ((v & 3) == 0) {
        return 4;
    }
    return 1;
}

FbCommDev Communicator::devFor(int flags) const
{
    FbCommDev d = dev_;
    int ch = FB_FLAG_GET_CHANNEL(flags);
    if (ch >= cfg_.channels) {
        ch = ch % cfg_.channels;
    }
    d.blockBase = ch * (FB_MAX_BLOCKS / cfg_.channels);
    d.llEpochBase = ch * FB_LL_BLOCKS;
    return d;
}

void Communicator::setAllReduceTable(const std::vector<uint64_t>& maxBytes,
                                     const std::vector<int>& algos)
{
    allReduceTable_.clear();
    for (size_t i = 0; i < maxBytes.size() && i < algos.size(); i++) {
        allReduceTable_.emplace_back(maxBytes[i], algos[i]);
    }
    std::sort(allReduceTable_.begin(), allReduceTable_.end());
}

int Communicator::pickAllReduceAlgo(uint64_t bytes, bool nvlsOk) const
{
    if (!allReduceTable_.empty()) {
        int algo = allReduceTable_.back().second;
        for (const auto& [maxB, a] : allReduceTable_) {
            if (bytes <= maxB) {
                algo = a;
                break;
            }
        }
        if (algo == FB_ALGO_NVLS && !nvlsOk) {
            algo = bytes <= cfg_.oneShotMaxBytes ? FB_ALGO_ONESHOT
                                                 : FB_ALGO_TWOSHOT;
        }
        return algo;
    }
    if (bytes <= cfg_.llMaxBytes && bytes <= FB_LL_MAX_BYTES) {
        return FB_ALGO_LL;
    }
    // in-switch reduction only pays off beyond a pair of GPUs
    if (nvlsOk && dev_.nranks >= 4 && bytes >= cfg_.nvlsMinBytes) {
        return FB_ALGO_NVLS;
    }
    if (bytes <= cfg_.oneShotMaxBytes) {
        return FB_ALGO_ONESHOT;
    }
    return FB_ALGO_TWOSHOT;
}

uint32_t Communicator::checkError(cudaStream_t s)
{
    bindDevice();
    // bounded: a stream-level wait whose peer died would block forever
    if (!syncStreamBounded(s, cfg_.timeoutMs * 3)) {
        uint32_t e = peekError();
        return e != FB_ERR_NONE ? e : 0xffffffffu;
    }
    return peekError();
}

uint32_t Communicator::peekError() const
{
    // The word lives in mapped host memory: a plain (volatile) load
    return *reinterpret_cast<volatile uint32_t*>(dev_.err);
}

// ---------------------------------------------------------------------------
// Reductions
// ---------------------------------------------------------------------------
enum ReduceKind
{
    K_ALLREDUCE = 0,
    K_REDUCE = 1,
    K_REDUCE_SCATTER = 2,
    K_SCAN = 3
};

int Communicator::reduceLike(int kind,
                             const void* send,
                             void* recv,
                             size_t count,
                             int dtype,
                             int op,
                             int root,
                             int algo,
                             int flags,
                             cudaStream_t s)
{
    const int n = dev_.nranks;
    const int rank = dev_.rank;
    const size_t esize = fbDtypeSize(dtype);
    if (esize == 0) {
        return FB_E_INVALID;
    }
    if (fb::findReduceLaunchers(dtype, op) == nullptr) {
        return FB_E_UNSUPPORTED;
    }
    bindDevice();
    bool symmetric = (flags & FB_FLAG_SYMMETRIC) != 0;
    // stream-ordered synchronisation replaces the in-kernel barriers
    const bool ss = streamSync_ && !(flags & FB_FLAG_NOSYNC) && n > 1;
    const int noSync = ((flags & FB_FLAG_NOSYNC) || ss) ? 1 : 0;
    const bool isRootOrAll = (kind != K_REDUCE) || (rank == root);

    // message bytes each rank contributes
    uint64_t bytes = (uint64_t)count * esize;
    if (kind == K_REDUCE_SCATTER) {
        bytes = (uint64_t)count * esize * n; // count = per-rank output
    }
    if (bytes == 0) {
        return barrier(s);
    }
    if (symmetric && (!inHeap(send, bytes))) {
        return FB_E_INVALID;
    }
    if (symmetric && (kind == K_SCAN || kind == K_REDUCE_SCATTER)) {
        // These read the peers' inputs while every rank writes its output with
        // no barrier in between: an output that overlaps the (symmetric) input
        // range would be clobbered under a peer's loads.  Heap offsets are the
        // same on every rank, so every rank takes the same decision: go
        // through the staging copy of the input.
        const uint8_t* s0 = (const uint8_t*)send;
        const uint8_t* r0 = (const uint8_t*)recv;
        const uint64_t outBytes = (kind == K_REDUCE_SCATTER) ? (uint64_t)count * esize : bytes;
        if (r0 < s0 + bytes && s0 < r0 + outBytes) {
            symmetric = false;
            flags &= ~FB_FLAG_SYMMETRIC;
        }
    }

    const int nvVariant = fb::nvlsVariant(dtype, op);

    // ---- algorithm choice ----
    if (kind == K_ALLREDUCE && parent_ != nullptr) {
        // The LL area and the multicast object belong to the parent's rank set
        if (algo == FB_ALGO_LL || algo == FB_ALGO_NVLS) {
            return FB_E_UNSUPPORTED;
        }
        if (algo == FB_ALGO_AUTO) {
            algo = pickAllReduceAlgo(bytes, false);
            if (algo == FB_ALGO_LL) {
                algo = bytes <= cfg_.oneShotMaxBytes ? FB_ALGO_ONESHOT : FB_ALGO_TWOSHOT;
            }
        }
        if (algo == FB_ALGO_ONESHOT && symmetric && send == recv) {
            algo = FB_ALGO_TWOSHOT;
        }
    } else if (kind == K_ALLREDUCE) {
        if (algo == FB_ALGO_AUTO) {
            // Element-wise multimem variants (integers, f64) are request-rate
            // bound: AUTO leaves them to the P2P kernels unless the message is
            // very large (measured: int32 two-shot beats NVLS 2x at 0.1-9 MB)
            const bool nvlsWorthIt =
              fb::nvlsVectorised(nvVariant) || bytes >= cfg_.nvlsScalarMinBytes;
            algo = pickAllReduceAlgo(
              bytes, hasMulticast() && nvVariant >= 0 && (bytes % 16) == 0 && nvlsWorthIt);
        }
        // (the LL kernel synchronises through its data slots: no stream mode)
        // (decided from quantities every rank shares; a rank whose local
        // pointers are not 16-byte aligned stays in LL and moves its bytes
        // element-wise inside the kernel)
        if (algo == FB_ALGO_LL && (ss || bytes > FB_LL_MAX_BYTES)) {
            algo = FB_ALGO_ONESHOT;
        }
        if (algo == FB_ALGO_NVLS &&
            (!hasMulticast() || nvVariant < 0 || (bytes % 16) != 0)) {
            algo = FB_ALGO_TWOSHOT;
        }
        // one-shot reads the peers' inputs while writing the output: in-place
        // on symmetric buffers must go through the two-shot (owner-only) path
        if (algo == FB_ALGO_ONESHOT && symmetric && send == recv) {
            algo = FB_ALGO_TWOSHOT;
        }
    } else if (kind == K_REDUCE) {
        if (algo == FB_ALGO_AUTO) {
            if (hasMulticast() && nvVariant >= 0 && bytes >= cfg_.nvlsMinBytes &&
                (bytes % 16) == 0) {
                algo = FB_ALGO_NVLS;
            } else if (bytes <= cfg_.oneShotMaxBytes * 2) {
                algo = FB_ALGO_ONESHOT;
            } else {
                algo = FB_ALGO_TWOSHOT;
            }
        }
        if (algo == FB_ALGO_NVLS &&
            (!hasMulticast() || nvVariant < 0 || (bytes % 16) != 0)) {
            algo = FB_ALGO_ONESHOT;
        }
        if (algo == FB_ALGO_LL) {
            algo = FB_ALGO_ONESHOT;
        }
    } else if (kind == K_REDUCE_SCATTER) {
        uint64_t slice = (uint64_t)count * esize;
        if ((slice % 16) != 0) {
            return FB_E_UNSUPPORTED;
        }
        if (algo == FB_ALGO_AUTO || algo == FB_ALGO_NVLS) {
            algo = (hasMulticast() && nvVariant >= 0 &&
                    slice >= cfg_.nvlsMinBytes / 2)
                     ? FB_ALGO_NVLS
                     : FB_ALGO_ONESHOT;
        } else {
            algo = FB_ALGO_ONESHOT;
        }
    } else {
        algo = FB_ALGO_ONESHOT; // scan
    }
    lastAlgo_ = algo;
    stats_.algoCount[algo]++;

    // ---- LL: no staging, no symmetric requirement ----
    if (algo == FB_ALGO_LL) {
        fb::LLArgs a;
        a.comm = devFor(flags);
        a.sendLocal = (const uint8_t*)send;
        a.recvLocal = (uint8_t*)recv;
        a.bytes = bytes;
        a.byteAccess = ((((uintptr_t)send) | ((uintptr_t)recv)) & 15) ? 1 : 0;
        a.llOff = llOff_ + (uint64_t)(a.comm.llEpochBase / FB_LL_BLOCKS) *
                             FB_LL_AREA_BYTES(n);
        stats_.launches++;
        stats_.bytes += bytes;
        return k_->ll(a, dtype, op, s) == cudaSuccess ? FB_OK : FB_E_CUDA;
    }

    // ---- staged / symmetric chunk loop ----
    const bool stageSend = !symmetric;
    const FbCommDev chanDev = devFor(flags);
    // which algorithms write through the symmetric recv offset
    const bool pushes = (algo == FB_ALGO_TWOSHOT) ||
                        (algo == FB_ALGO_NVLS && kind == K_ALLREDUCE);
    bool stageRecv = false;
    if (pushes) {
        if (kind == K_REDUCE) {
            stageRecv = true; // only the root has a recv buffer
        } else {
            stageRecv = !symmetric || !inHeap(recv, bytes);
        }
    } else if (isRootOrAll && (((uintptr_t)recv) & 15)) {
        stageRecv = true; // vector stores need 16-byte alignment
    }
    // slices are addressed inside the whole message: no piecewise launches
    if (kind == K_REDUCE_SCATTER && (stageSend || stageRecv) && bytes > cfg_.stageBytes) {
        return FB_E_TOO_LARGE;
    }
    if ((stageSend || stageRecv) && chanDev.blockBase != 0) {
        return FB_E_INVALID; // staging buffers exist once, on channel 0 only
    }
    // The number of launches must be the same on every rank (the per-CTA
    // barrier epochs advance with it), so it only depends on `symmetric`,
    // `algo`, `kind` and `bytes`; a rank-LOCAL need for output staging (an
    // unaligned destination) must fit one piece
    // (whether the output lives in the symmetric heap is part of the call's
    // contract: all ranks pass the same kind of buffer)
    const bool stageRecvGlobal = pushes && (kind == K_REDUCE || !symmetric || !inHeap(recv, bytes));
    const uint64_t chunkMax =
      (stageSend || stageRecvGlobal) ? (uint64_t)cfg_.stageBytes : bytes;
    if (stageRecv && !stageRecvGlobal && !stageSend && bytes > cfg_.stageBytes) {
        return FB_E_TOO_LARGE;
    }

    for (uint64_t done = 0; done < bytes; done += chunkMax) {
        const uint64_t len = std::min<uint64_t>(chunkMax, bytes - done);
        uint64_t sendOff;
        if (stageSend) {
            if (k_->copy(heapPtr(stageSendOff_), (const uint8_t*)send + done, len, s) != cudaSuccess) {
                return FB_E_CUDA;
            }
            stats_.stagedCopies++;
            sendOff = stageSendOff_;
        } else {
            sendOff = offsetOf(send) + done;
        }
        uint8_t* recvLocal = (uint8_t*)recv + done;
        uint64_t recvOff = 0;
        if (stageRecv) {
            recvLocal = heapPtr(stageRecvOff_);
            recvOff = stageRecvOff_;
        } else if (pushes) {
            recvOff = offsetOf(recv) + done;
        }

        const uint64_t nVec = len / 16;
        uint64_t per = (nVec + n - 1) / n; // slice size in vectors
        cudaError_t ce = cudaSuccess;
        if (ss && streamBarrier(flags, s) != FB_OK) {
            return FB_E_CUDA;
        }

        if (algo == FB_ALGO_NVLS) {
            fb::NvlsArgs a;
            memset(&a, 0, sizeof(a));
            a.comm = chanDev;
            a.sendOff = sendOff;
            a.recvOff = recvOff;
            a.recvLocal = recvLocal;
            a.noSync = noSync;
            uint64_t work = 0;
            if (kind == K_ALLREDUCE) {
                a.mode = fb::NVLS_ALLREDUCE;
                a.vecBegin = std::min<uint64_t>((uint64_t)rank * per, nVec);
                a.vecEnd = std::min<uint64_t>(a.vecBegin + per, nVec);
                a.outBase = 0;
                work = per;
            } else if (kind == K_REDUCE) {
                a.mode = fb::NVLS_REDUCE_LOCAL;
                a.vecBegin = 0;
                a.vecEnd = (rank == root) ? nVec : 0;
                a.outBase = 0;
                work = nVec;
            } else { // reduce scatter
                a.mode = fb::NVLS_REDUCE_LOCAL;
                uint64_t sliceVec = (uint64_t)count * esize / 16;
                a.vecBegin = (uint64_t)rank * sliceVec;
                a.vecEnd = a.vecBegin + sliceVec;
                a.outBase = a.vecBegin;
                work = sliceVec;
            }
            ce = fb::launchNvls(
              a, nvVariant, blocksFor(work, 4), cfg_.threads, s);
        } else {
            fb::ReduceArgs a;
            memset(&a, 0, sizeof(a));
            a.comm = chanDev;
            a.sendOff = sendOff;
            a.recvOff = recvOff;
            a.recvLocal = recvLocal;
            a.bytes = len;
            a.readRanks = n;
            a.noSync = noSync;
            uint64_t work = nVec;
            if (kind == K_ALLREDUCE && algo == FB_ALGO_ONESHOT) {
                a.vecBegin = 0;
                a.vecEnd = nVec;
                a.pushMask = 0;
                a.tailOwner = -2;
            } else if (kind == K_ALLREDUCE) { // two-shot
                a.vecBegin = std::min<uint64_t>((uint64_t)rank * per, nVec);
                a.vecEnd = std::min<uint64_t>(a.vecBegin + per, nVec);
                a.pushMask = (n >= 32) ? 0xffffffffu : ((1u << n) - 1);
                a.tailOwner = n - 1;
                work = per;
            } else if (kind == K_REDUCE && algo == FB_ALGO_ONESHOT) {
                a.vecBegin = 0;
                a.vecEnd = (rank == root) ? nVec : 0;
                a.pushMask = 0;
                a.tailOwner = root;
            } else if (kind == K_REDUCE) { // two-shot, push slices to root
                a.vecBegin = std::min<uint64_t>((uint64_t)rank * per, nVec);
                a.vecEnd = std::min<uint64_t>(a.vecBegin + per, nVec);
                a.pushMask = 1u << root;
                a.tailOwner = n - 1;
                work = per;
            } else if (kind == K_REDUCE_SCATTER) {
                uint64_t sliceVec = (uint64_t)count * esize / 16;
                a.vecBegin = (uint64_t)rank * sliceVec;
                a.vecEnd = a.vecBegin + sliceVec;
                a.outBase = a.vecBegin;
                a.pushMask = 0;
                a.tailOwner = -1;
                a.bytes = len - (len & 15); // slices are vector multiples
                work = sliceVec;
            } else { // scan
                a.vecBegin = 0;
                a.vecEnd = nVec;
                a.readRanks = rank + 1;
                a.pushMask = 0;
                a.tailOwner = -2;
            }
            int perThread = (n == 8) ? 2 : 4;
            ce = k_->reduce(a, dtype, op, blocksFor(work, perThread), cfg_.threads, s);
        }
        if (ce != cudaSuccess) {
            return FB_E_CUDA;
        }
        if (ss && streamBarrier(flags, s) != FB_OK) {
            return FB_E_CUDA;
        }
        stats_.launches++;
        stats_.bytes += len;
        if (stageRecv && isRootOrAll) {
            uint64_t outLen = (kind == K_REDUCE_SCATTER) ? count * esize : len;
            if (k_->copy((uint8_t*)recv + done, heapPtr(stageRecvOff_), outLen, s) != cudaSuccess) {
                return FB_E_CUDA;
            }
            stats_.stagedCopies++;
        }
    }
    return FB_OK;
}

int Communicator::allReduce(const void* send,
                            void* recv,
                            size_t count,
                            int dtype,
                            int op,
                            int algo,
                            int flags,
                            cudaStream_t s)
{
    NvtxRange nvtxRange("fb::allReduce");
    return reduceLike(
      K_ALLREDUCE, send, recv, count, dtype, op, 0, algo, flags, s);
}

int Communicator::reduce(const void* send,
                         void* recv,
                         size_t count,
                         int dtype,
                         int op,
                         int root,
                         int flags,
                         cudaStream_t s)
{
    NvtxRange nvtxRange("fb::reduce");
    if (root < 0 || root >= dev_.nranks) {
        return FB_E_INVALID;
    }
    return reduceLike(
      K_REDUCE, send, recv, count, dtype, op, root, FB_ALGO_AUTO, flags, s);
}

int Communicator::reduceScatter(const void* send,
                                void* recv,
                                size_t recvCount,
                                int dtype,
                                int op,
                                int flags,
                                cudaStream_t s)
{
    NvtxRange nvtxRange("fb::reduceScatter");
    return reduceLike(K_REDUCE_SCATTER,
                      send,
                      recv,
                      recvCount,
                      dtype,
                      op,
                      0,
                      FB_ALGO_AUTO,
                      flags,
                      s);
}

int Communicator::scan(const void* send,
                       void* recv,
                       size_t count,
                       int dtype,
                       int op,
                       int flags,
                       cudaStream_t s)
{
    NvtxRange nvtxRange("fb::scan");
    return reduceLike(
      K_SCAN, send, recv, count, dtype, op, 0, FB_ALGO_AUTO, flags, s);
}

// ---------------------------------------------------------------------------
// Grouped all-reduce
// ---------------------------------------------------------------------------
// One launch of the grouped kernel: this rank's segment table
struct Communicator::GroupLaunch
{
    fb::GroupSeg* dSegs = nullptr; // host memory on the loopback backend
    uint32_t nSegs = 0;
    uint32_t totalChunks = 0;
    uint64_t vecsPerRank = 0; // same on every rank: sizes the grid
    uint64_t bytes = 0;
};

struct Communicator::GroupPlan
{
    std::vector<GroupLaunch> launches;
    GroupKind kind = GROUP_ALLREDUCE;
    int dtype = 0;
    int device = 0;
    size_t items = 0;
    bool hostTables = false; // loopback: plain heap memory

    ~GroupPlan()
    {
        if (hostTables) {
            for (auto& l : launches) {
                ::free(l.dSegs);
            }
            return;
        }
        cudaSetDevice(device);
        for (auto& l : launches) {
            if (l.dSegs != nullptr) {
                cudaFree(l.dSegs);
            }
        }
        cudaGetLastError();
    }
};

struct Communicator::ManySlot
{
    fb::GroupSeg* dSegs = nullptr;
    fb::GroupSeg* hSegs = nullptr;
    cudaEvent_t ev = nullptr;
    int device = 0;
    bool used = false;
    ~ManySlot()
    {
        cudaSetDevice(device);
        if (dSegs != nullptr) {
            cudaFree(dSegs);
        }
        if (hSegs != nullptr) {
            cudaFreeHost(hSegs);
        }
        if (ev != nullptr) {
            cudaEventDestroy(ev);
        }
        cudaGetLastError();
    }
};

Communicator::ManySlot* Communicator::nextManySlot()
{
    // table slot: pinned staging + device copy, recycled after its launch
    if (manySlots_.empty()) {
        manySlots_.resize(8);
    }
    auto& slotPtr = manySlots_[manyNext_++ % manySlots_.size()];
    if (!slotPtr) {
        slotPtr = std::make_shared<ManySlot>();
        slotPtr->device = device_;
        if (cudaMalloc((void**)&slotPtr->dSegs, FB_GROUP_MAX_SEGS * sizeof(fb::GroupSeg)) != cudaSuccess ||
            cudaHostAlloc((void**)&slotPtr->hSegs, FB_GROUP_MAX_SEGS * sizeof(fb::GroupSeg), cudaHostAllocDefault) !=
              cudaSuccess ||
            cudaEventCreateWithFlags(&slotPtr->ev, cudaEventDisableTiming) != cudaSuccess) {
            cudaGetLastError();
            slotPtr.reset();
            return nullptr;
        }
    }
    if (slotPtr->used) {
        cudaEventSynchronize(slotPtr->ev);
    }
    return slotPtr.get();
}

size_t Communicator::groupPlanLaunches(const GroupPlan& plan)
{
    return plan.launches.size();
}

namespace {
struct SegBuild
{
    std::vector<fb::GroupSeg> segs;
    uint32_t totalChunks = 0;
    uint64_t vecsPerRank = 0;
    uint64_t bytes = 0;
};
}

// This rank's share of items[0..n): the concatenation of all tensors (in
// 16-byte vectors) is cut into nranks equal ranges; a segment is the
// intersection of one tensor with this rank's range.
static int buildGroupSegs(const Communicator& c,
                          const Communicator::GroupItem* items,
                          size_t nItems,
                          size_t esize,
                          SegBuild& out)
{
    const int n = c.size();
    const int rank = c.rank();
    const uint32_t chunk = fb::fbGroupChunkVecs(n);
    uint64_t V = 0;
    for (size_t i = 0; i < nItems; i++) {
        const uint64_t bytes = (uint64_t)items[i].count * esize;
        if (bytes == 0) {
            continue;
        }
        if (!c.inHeap(items[i].send, bytes) || !c.inHeap(items[i].recv, bytes) ||
            (((uintptr_t)items[i].send | (uintptr_t)items[i].recv) & 15)) {
            return FB_E_INVALID;
        }
        V += (bytes + 15) / 16;
        out.bytes += bytes;
    }
    const uint64_t lo = V * (uint64_t)rank / n;
    const uint64_t hi = V * (uint64_t)(rank + 1) / n;
    out.vecsPerRank = (V + n - 1) / n;
    uint64_t flat = 0;
    uint64_t chunks = 0;
    for (size_t i = 0; i < nItems; i++) {
        const uint64_t bytes = (uint64_t)items[i].count * esize;
        if (bytes == 0) {
            continue;
        }
        const uint64_t vecs = (bytes + 15) / 16;
        const uint64_t full = bytes / 16;
        const uint32_t tail = (uint32_t)(bytes % 16);
        const uint64_t a = std::max(flat, lo);
        const uint64_t b = std::min(flat + vecs, hi);
        if (a < b) {
            const uint64_t v0 = a - flat;
            const uint64_t v1 = b - flat;
            fb::GroupSeg sg;
            memset(&sg, 0, sizeof(sg));
            sg.nVec = (uint32_t)(std::min(v1, full) > v0 ? std::min(v1, full) - v0 : 0);
            sg.tailBytes = (tail != 0 && v1 == vecs) ? tail : 0;
            if (sg.nVec != 0 || sg.tailBytes != 0) {
                sg.sendOff = c.offsetOf(items[i].send) + v0 * 16;
                sg.recvOff = c.offsetOf(items[i].recv) + v0 * 16;
                sg.chunk0 = (uint32_t)chunks;
                chunks += ((uint64_t)sg.nVec + (sg.tailBytes ? 1 : 0) + chunk - 1) / chunk;
                out.segs.push_back(sg);
            }
        }
        flat += vecs;
    }
    if (chunks > 0xffffffffull) {
        return FB_E_TOO_LARGE;
    }
    out.totalChunks = (uint32_t)chunks;
    return FB_OK;
}

// This rank's segments of a reduce-scatter or all-gather group: one per item,
// a whole shard each (see Communicator::GroupKind for the conditions)
static int buildShardSegs(const Communicator& c,
                          Communicator::GroupKind kind,
                          const Communicator::GroupItem* items,
                          size_t nItems,
                          size_t esize,
                          SegBuild& out)
{
    const int n = c.size();
    const int rank = c.rank();
    const uint32_t chunk = fb::fbGroupChunkVecs(n);
    const bool rs = kind == Communicator::GROUP_REDUCE_SCATTER;
    // [begin, end) of every send, by begin: peers read them (reduce-scatter)
    // or the kernel reads them (all-gather) while outputs are written
    std::vector<std::pair<uintptr_t, uintptr_t>> sends;
    for (size_t i = 0; i < nItems; i++) {
        const uint64_t shard = (uint64_t)items[i].count * esize;
        if (shard == 0) {
            continue;
        }
        const uint64_t sendBytes = rs ? shard * n : shard;
        const uint64_t recvBytes = rs ? shard : shard * n;
        if (shard % 16 != 0 || !c.inHeap(items[i].send, sendBytes) || !c.inHeap(items[i].recv, recvBytes) ||
            (((uintptr_t)items[i].send | (uintptr_t)items[i].recv) & 15)) {
            return FB_E_INVALID;
        }
        sends.push_back({ (uintptr_t)items[i].send, (uintptr_t)items[i].send + sendBytes });
    }
    std::sort(sends.begin(), sends.end());
    std::vector<uintptr_t> maxEnd(sends.size());
    for (size_t k = 0; k < sends.size(); k++) {
        maxEnd[k] = std::max(sends[k].second, k > 0 ? maxEnd[k - 1] : 0);
    }
    uint64_t chunks = 0;
    for (size_t i = 0; i < nItems; i++) {
        const uint64_t shard = (uint64_t)items[i].count * esize;
        if (shard == 0) {
            continue;
        }
        const uintptr_t lo = (uintptr_t)items[i].recv;
        const uintptr_t hi = lo + (rs ? shard : shard * n);
        // in-place all-gather: the send is block `rank` of its own output
        const uintptr_t own = (!rs && (uintptr_t)items[i].send == lo + (uint64_t)rank * shard) ? lo + rank * shard : 0;
        // sends starting below `lo` overlap iff one of them ends above it;
        // every send starting in [lo, hi) overlaps, except the own in-place one
        size_t k = std::lower_bound(sends.begin(), sends.end(), std::make_pair(lo, (uintptr_t)0)) - sends.begin();
        if (k > 0 && maxEnd[k - 1] > lo) {
            return FB_E_INVALID;
        }
        bool ownSeen = false;
        for (; k < sends.size() && sends[k].first < hi; k++) {
            if (own != 0 && !ownSeen && sends[k].first == own && sends[k].second == own + shard) {
                ownSeen = true;
                continue;
            }
            return FB_E_INVALID;
        }
        if (shard / 16 > 0xffffffffull) {
            return FB_E_TOO_LARGE;
        }
        fb::GroupSeg sg;
        memset(&sg, 0, sizeof(sg));
        sg.nVec = (uint32_t)(shard / 16);
        sg.sendOff = c.offsetOf(items[i].send) + (rs ? (uint64_t)rank * shard : 0);
        sg.recvOff = c.offsetOf(items[i].recv) + (rs ? 0 : (uint64_t)rank * shard);
        sg.chunk0 = (uint32_t)chunks;
        chunks += ((uint64_t)sg.nVec + chunk - 1) / chunk;
        if (chunks > 0xffffffffull) {
            return FB_E_TOO_LARGE;
        }
        out.segs.push_back(sg);
        out.vecsPerRank += sg.nVec;
        out.bytes += shard * n;
    }
    out.totalChunks = (uint32_t)chunks;
    return FB_OK;
}

static int buildSegs(const Communicator& c,
                     Communicator::GroupKind kind,
                     const Communicator::GroupItem* items,
                     size_t nItems,
                     size_t esize,
                     SegBuild& out)
{
    if (kind == Communicator::GROUP_ALLREDUCE) {
        return buildGroupSegs(c, items, nItems, esize, out);
    }
    return buildShardSegs(c, kind, items, nItems, esize, out);
}

// items per launch: every item yields at most one segment per rank
static const size_t GROUP_ITEMS_PER_LAUNCH = FB_GROUP_MAX_SEGS - 8;

std::shared_ptr<Communicator::GroupPlan> Communicator::prepareGroup(
  const GroupItem* items,
  size_t nItems,
  int dtype,
  int* rcOut,
  GroupKind kind)
{
    int rcLocal = FB_OK;
    int& rc = rcOut ? *rcOut : rcLocal;
    rc = FB_OK;
    if (parent_ != nullptr) {
        rc = FB_E_UNSUPPORTED; // see subset()
        return nullptr;
    }
    const size_t esize = fbDtypeSize(dtype);
    if (esize == 0 || kind < GROUP_ALLREDUCE || kind > GROUP_ALLGATHER) {
        rc = FB_E_INVALID;
        return nullptr;
    }
    bindDevice();
    auto plan = std::make_shared<GroupPlan>();
    plan->kind = kind;
    plan->dtype = dtype;
    plan->device = device_;
    plan->items = nItems;
    for (size_t begin = 0; begin < nItems; begin += GROUP_ITEMS_PER_LAUNCH) {
        const size_t cnt = std::min(GROUP_ITEMS_PER_LAUNCH, nItems - begin);
        SegBuild sb;
        rc = buildSegs(*this, kind, items + begin, cnt, esize, sb);
        if (rc != FB_OK) {
            return nullptr;
        }
        GroupLaunch l;
        l.nSegs = (uint32_t)sb.segs.size();
        l.totalChunks = sb.totalChunks;
        l.vecsPerRank = sb.vecsPerRank;
        l.bytes = sb.bytes;
        // (a rank may own nothing of a tiny group: it still takes part in the
        // barriers, with an empty table)
        const size_t tb = std::max<size_t>(sb.segs.size(), 1) * sizeof(fb::GroupSeg);
        if (loop_) {
            plan->hostTables = true;
            l.dSegs = (fb::GroupSeg*)::malloc(tb);
            if (!sb.segs.empty()) {
                memcpy(l.dSegs, sb.segs.data(), sb.segs.size() * sizeof(fb::GroupSeg));
            }
            plan->launches.push_back(l);
            continue;
        }
        if (cudaMalloc((void**)&l.dSegs, tb) != cudaSuccess) {
            cudaGetLastError();
            rc = FB_E_CUDA;
            return nullptr;
        }
        plan->launches.push_back(l);
        if (!sb.segs.empty() &&
            cudaMemcpy(l.dSegs, sb.segs.data(), sb.segs.size() * sizeof(fb::GroupSeg), cudaMemcpyHostToDevice) !=
              cudaSuccess) {
            cudaGetLastError();
            rc = FB_E_CUDA;
            return nullptr;
        }
    }
    return plan;
}

static int groupGrid(const CommConfig& cfg, int nranks, uint64_t vecsPerRank)
{
    // Derived ONLY from quantities that are identical on every rank: CTA b of
    // one rank meets CTA b of every peer at the barriers
    // a lone rank does not synchronise with anybody: two CTAs per SM for an
    // HBM-bound copy; otherwise the grid is bounded by the barrier slots
    const int slots = nranks == 1 ? 2 * FB_NUM_SMS : FB_MAX_BLOCKS / cfg.channels;
    const int cap = std::min(slots, cfg.groupBlocks > 0 ? cfg.groupBlocks : (nranks == 1 ? 2 * FB_NUM_SMS : 128));
    const uint64_t warps = (uint64_t)cfg.threads / 32;
    const uint64_t chunks = (vecsPerRank + fb::fbGroupChunkVecs(nranks) - 1) / fb::fbGroupChunkVecs(nranks);
    const uint64_t want = (chunks + warps * 2 - 1) / (warps * 2); // >= 2 chunks per warp
    return (int)std::clamp<uint64_t>(want, 1, (uint64_t)cap);
}

int Communicator::launchGroup(const GroupLaunch& l, GroupKind kind, int dtype, int op, int flags, cudaStream_t s)
{
    const int n = dev_.nranks;
    const bool ss = streamSync_ && !(flags & FB_FLAG_NOSYNC) && n > 1;
    fb::GroupArgs a;
    memset(&a, 0, sizeof(a));
    a.comm = devFor(flags);
    a.segs = l.dSegs;
    a.nSegs = l.nSegs;
    a.totalChunks = l.totalChunks;
    a.noSync = ((flags & FB_FLAG_NOSYNC) || ss || n == 1) ? 1 : 0;
    if (ss && streamBarrier(flags, s) != FB_OK) {
        return FB_E_CUDA;
    }
    const int blocks = groupGrid(cfg_, n, l.vecsPerRank);
    cudaError_t e;
    if (kind == GROUP_REDUCE_SCATTER) {
        e = k_->groupReduceScatter(a, dtype, op, blocks, cfg_.threads, s);
    } else if (kind == GROUP_ALLGATHER) {
        e = k_->groupAllGather(a, blocks, cfg_.threads, s);
    } else {
        e = k_->group(a, dtype, op, blocks, cfg_.threads, s);
    }
    if (e != cudaSuccess) {
        return FB_E_CUDA;
    }
    if (ss && streamBarrier(flags, s) != FB_OK) {
        return FB_E_CUDA;
    }
    stats_.launches++;
    stats_.bytes += l.bytes;
    if (kind == GROUP_ALLREDUCE) {
        stats_.algoCount[FB_ALGO_TWOSHOT]++;
    }
    return FB_OK;
}

int Communicator::allReduceGroup(const GroupPlan& plan, int op, int flags, cudaStream_t s)
{
    NvtxRange nvtxRange("fb::allReduceGroup");
    if (parent_ != nullptr) {
        return FB_E_UNSUPPORTED; // see subset()
    }
    if (plan.kind != GROUP_ALLREDUCE) {
        return FB_E_INVALID;
    }
    const fb::ReduceLaunchers* L = fb::findReduceLaunchers(plan.dtype, op);
    if (L == nullptr || L->group == nullptr) {
        return FB_E_UNSUPPORTED;
    }
    bindDevice();
    for (const auto& l : plan.launches) {
        int rc = launchGroup(l, GROUP_ALLREDUCE, plan.dtype, op, flags, s);
        if (rc != FB_OK) {
            return rc;
        }
    }
    lastAlgo_ = FB_ALGO_TWOSHOT;
    return FB_OK;
}

int Communicator::reduceScatterGroup(const GroupPlan& plan, int op, int flags, cudaStream_t s)
{
    NvtxRange nvtxRange("fb::reduceScatterGroup");
    if (parent_ != nullptr) {
        return FB_E_UNSUPPORTED; // see subset()
    }
    if (plan.kind != GROUP_REDUCE_SCATTER) {
        return FB_E_INVALID;
    }
    const fb::ReduceLaunchers* L = fb::findReduceLaunchers(plan.dtype, op);
    if (L == nullptr || L->groupRs == nullptr) {
        return FB_E_UNSUPPORTED;
    }
    bindDevice();
    for (const auto& l : plan.launches) {
        int rc = launchGroup(l, GROUP_REDUCE_SCATTER, plan.dtype, op, flags, s);
        if (rc != FB_OK) {
            return rc;
        }
    }
    return FB_OK;
}

int Communicator::allGatherGroup(const GroupPlan& plan, int flags, cudaStream_t s)
{
    NvtxRange nvtxRange("fb::allGatherGroup");
    if (parent_ != nullptr) {
        return FB_E_UNSUPPORTED; // see subset()
    }
    if (plan.kind != GROUP_ALLGATHER) {
        return FB_E_INVALID;
    }
    bindDevice();
    for (const auto& l : plan.launches) {
        int rc = launchGroup(l, GROUP_ALLGATHER, plan.dtype, -1, flags, s);
        if (rc != FB_OK) {
            return rc;
        }
    }
    return FB_OK;
}

int Communicator::allReduceMany(const GroupItem* items,
                                size_t nItems,
                                int dtype,
                                int op,
                                int flags,
                                cudaStream_t s)
{
    NvtxRange nvtxRange("fb::allReduceMany");
    return groupMany(GROUP_ALLREDUCE, items, nItems, dtype, op, flags, s);
}

int Communicator::reduceScatterMany(const GroupItem* items,
                                    size_t nItems,
                                    int dtype,
                                    int op,
                                    int flags,
                                    cudaStream_t s)
{
    NvtxRange nvtxRange("fb::reduceScatterMany");
    return groupMany(GROUP_REDUCE_SCATTER, items, nItems, dtype, op, flags, s);
}

int Communicator::allGatherMany(const GroupItem* items, size_t nItems, int dtype, int flags, cudaStream_t s)
{
    NvtxRange nvtxRange("fb::allGatherMany");
    return groupMany(GROUP_ALLGATHER, items, nItems, dtype, -1, flags, s);
}

int Communicator::groupMany(GroupKind kind,
                            const GroupItem* items,
                            size_t nItems,
                            int dtype,
                            int op,
                            int flags,
                            cudaStream_t s)
{
    if (parent_ != nullptr) {
        return FB_E_UNSUPPORTED; // see subset()
    }
    const size_t esize = fbDtypeSize(dtype);
    if (esize == 0) {
        return FB_E_INVALID;
    }
    // all-gather is a byte copy: any dtype has a kernel
    bool grouped = true;
    if (kind != GROUP_ALLGATHER) {
        const fb::ReduceLaunchers* L = fb::findReduceLaunchers(dtype, op);
        if (L == nullptr) {
            return FB_E_UNSUPPORTED;
        }
        grouped = (kind == GROUP_ALLREDUCE ? L->group : L->groupRs) != nullptr;
    }
    const size_t n = (size_t)dev_.nranks;
    bindDevice();
    // try the grouped path batch by batch; anything not symmetric / aligned
    // goes through the per-tensor calls (the choice depends only on arguments
    // that are symmetric across ranks)
    for (size_t begin = 0; begin < nItems; begin += GROUP_ITEMS_PER_LAUNCH) {
        const size_t cnt = std::min(GROUP_ITEMS_PER_LAUNCH, nItems - begin);
        SegBuild sb;
        int rc = grouped ? buildSegs(*this, kind, items + begin, cnt, esize, sb) : FB_E_UNSUPPORTED;
        if (rc != FB_OK) {
            for (size_t i = begin; i < begin + cnt; i++) {
                const GroupItem& it = items[i];
                const size_t bytes = it.count * esize;
                int f = flags;
                int r2 = FB_OK;
                if (kind == GROUP_ALLREDUCE) {
                    if (!inHeap(it.send, bytes)) {
                        f &= ~FB_FLAG_SYMMETRIC;
                    }
                    r2 = allReduce(it.send, it.recv, it.count, dtype, op, FB_ALGO_AUTO, f, s);
                } else if (bytes == 0) {
                    continue;
                } else if (kind == GROUP_REDUCE_SCATTER) {
                    if (!inHeap(it.send, bytes * n)) {
                        f &= ~FB_FLAG_SYMMETRIC;
                    }
                    r2 = reduceScatter(it.send, it.recv, it.count, dtype, op, f, s);
                } else {
                    if (!inHeap(it.send, bytes)) {
                        f &= ~FB_FLAG_SYMMETRIC;
                    }
                    r2 = allGather(it.send, it.recv, bytes, f, s);
                }
                if (r2 != FB_OK) {
                    return r2;
                }
            }
            continue;
        }
        GroupLaunch l;
        l.dSegs = sb.segs.data(); // the host twin reads the table in place
        l.nSegs = (uint32_t)sb.segs.size();
        l.totalChunks = sb.totalChunks;
        l.vecsPerRank = sb.vecsPerRank;
        l.bytes = sb.bytes;
        ManySlot* slot = nullptr;
        if (!loop_) {
            slot = nextManySlot();
            if (slot == nullptr) {
                return FB_E_CUDA;
            }
            if (!sb.segs.empty()) {
                memcpy(slot->hSegs, sb.segs.data(), sb.segs.size() * sizeof(fb::GroupSeg));
                if (cudaMemcpyAsync(slot->dSegs, slot->hSegs, sb.segs.size() * sizeof(fb::GroupSeg), cudaMemcpyHostToDevice, s) !=
                    cudaSuccess) {
                    return FB_E_CUDA;
                }
            }
            l.dSegs = slot->dSegs;
        }
        rc = launchGroup(l, kind, dtype, op, flags, s);
        if (rc != FB_OK) {
            return rc;
        }
        if (slot != nullptr) {
            cudaEventRecord(slot->ev, s);
            slot->used = true;
        }
    }
    if (kind == GROUP_ALLREDUCE) {
        lastAlgo_ = FB_ALGO_TWOSHOT;
    }
    return FB_OK;
}

// ---------------------------------------------------------------------------
// Data movement
// ---------------------------------------------------------------------------
int Communicator::moveLike(int mode,
                           const void* send,
                           void* recv,
                           size_t chunkBytes,
                           int root,
                           int flags,
                           cudaStream_t s)
{
    const int n = dev_.nranks;
    const int rank = dev_.rank;
    bindDevice();
    const bool symmetric = (flags & FB_FLAG_SYMMETRIC) != 0;
    const bool ss = streamSync_ && !(flags & FB_FLAG_NOSYNC) && n > 1;
    const int noSync = ((flags & FB_FLAG_NOSYNC) || ss) ? 1 : 0;
    if (chunkBytes == 0) {
        return barrier(s);
    }
    // whether this rank is a source at all
    const bool isSource =
      (mode == fb::MOVE_ALLGATHER || mode == fb::MOVE_ALLTOALL ||
       mode == fb::MOVE_GATHER) ||
      (rank == root);
    // rows x rowBytes describes the source layout per rank
    const int srcRows =
      (mode == fb::MOVE_ALLTOALL || mode == fb::MOVE_SCATTER) ? n : 1;

    lastAlgo_ = FB_ALGO_ONESHOT;
    // ---- NVLS fast paths on symmetric buffers ----
    // They move 16-byte vectors at the heap offsets of source and output.
    // Whether the all-gather output lives in the heap is part of the call's
    // contract, as for the reduce path's output: every rank passes the same
    // kind of buffer, at the same offset, so every rank takes the same path.
    if (symmetric && hasMulticast() && (chunkBytes % 16) == 0 &&
        chunkBytes >= cfg_.nvlsMinBytes &&
        ((mode == fb::MOVE_ALLGATHER && inHeap(recv, chunkBytes * n) && (offsetOf(send) % 16) == 0 &&
          (offsetOf(recv) % 16) == 0) ||
         (mode == fb::MOVE_BCAST && (offsetOf(recv) % 16) == 0))) {
        fb::NvlsArgs a;
        memset(&a, 0, sizeof(a));
        a.comm = devFor(flags);
        a.noSync = noSync;
        a.outBase = 0;
        uint64_t nVec = chunkBytes / 16;
        if (mode == fb::MOVE_ALLGATHER) {
            a.mode = fb::NVLS_ALLGATHER;
            a.sendOff = offsetOf(send);
            a.recvOff = offsetOf(recv) + (uint64_t)rank * chunkBytes;
            a.vecBegin = 0;
            a.vecEnd = nVec;
        } else {
            a.mode = fb::NVLS_BCAST;
            a.sendOff = offsetOf(recv); // bcast buffer is in-out
            a.recvOff = offsetOf(recv);
            a.vecBegin = 0;
            a.vecEnd = (rank == root) ? nVec : 0;
        }
        lastAlgo_ = FB_ALGO_NVLS;
        stats_.algoCount[FB_ALGO_NVLS]++;
        stats_.launches++;
        stats_.bytes += chunkBytes;
        if (ss && streamBarrier(flags, s) != FB_OK) {
            return FB_E_CUDA;
        }
        if (fb::launchNvls(a, -1, blocksFor(nVec, 4), cfg_.threads, s) !=
            cudaSuccess) {
            return FB_E_CUDA;
        }
        return ss ? streamBarrier(flags, s) : FB_OK;
    }

    // ---- large symmetric broadcast: scatter + allgather in one kernel ----
    // (it has a barrier between its two steps: not available in stream mode;
    // it copies 16-byte words at the buffer's heap offset)
    if (mode == fb::MOVE_BCAST && symmetric && !ss &&
        chunkBytes >= cfg_.bcast2StepMinBytes && (chunkBytes % 16) == 0 && (offsetOf(recv) % 16) == 0) {
        fb::MoveArgs a;
        memset(&a, 0, sizeof(a));
        a.comm = devFor(flags);
        a.sendOff = offsetOf(recv);
        a.recvOff = offsetOf(recv);
        a.recvLocal = (uint8_t*)recv;
        a.chunkBytes = chunkBytes;
        a.mode = fb::MOVE_BCAST_2STEP;
        a.root = root;
        a.noSync = noSync;
        lastAlgo_ = FB_ALGO_TWOSHOT;
        stats_.algoCount[FB_ALGO_TWOSHOT]++;
        stats_.launches++;
        stats_.bytes += chunkBytes;
        return k_->move(a, 16, blocksFor(chunkBytes / 16 / n, 4), cfg_.threads, s) == cudaSuccess ? FB_OK : FB_E_CUDA;
    }

    // ---- generic pull, staged in pieces when buffers are not symmetric ----
    uint64_t piece = chunkBytes;
    if (!symmetric) {
        uint64_t cap = (uint64_t)cfg_.stageBytes / srcRows;
        cap -= cap % 16;
        if (cap == 0) {
            return FB_E_TOO_LARGE;
        }
        piece = std::min<uint64_t>(chunkBytes, cap);
    }
    stats_.algoCount[FB_ALGO_ONESHOT]++;
    for (uint64_t done = 0; done < chunkBytes; done += piece) {
        const uint64_t len = std::min<uint64_t>(piece, chunkBytes - done);
        fb::MoveArgs a;
        memset(&a, 0, sizeof(a));
        a.comm = devFor(flags);
        if (!symmetric && a.comm.blockBase != 0) {
            return FB_E_INVALID;
        }
        a.mode = mode;
        a.root = root;
        a.noSync = noSync;
        a.chunkBytes = len;
        a.recvLocal = (uint8_t*)recv + done;
        a.dstStride = chunkBytes;
        if (symmetric) {
            const void* src = (mode == fb::MOVE_BCAST) ? recv : send;
            a.sendOff = offsetOf(src) + done;
            a.srcStride = chunkBytes;
        } else {
            a.sendOff = stageSendOff_;
            a.srcStride = len;
            if (isSource) {
                const uint8_t* src =
                  (const uint8_t*)((mode == fb::MOVE_BCAST) ? recv : send);
                const cudaError_t ce =
                  srcRows == 1 ? k_->copy(heapPtr(stageSendOff_), src + done, len, s)
                               : k_->copy2D(heapPtr(stageSendOff_), len, src + done, chunkBytes, len, srcRows, s);
                if (ce != cudaSuccess) {
                    return FB_E_CUDA;
                }
                stats_.stagedCopies++;
            }
        }
        // BlockBarrier pairs CTA i of every rank, so the grid, and whether the
        // TMA kernel is eligible, come from values equal on every rank: the
        // mode, the lengths, the strides and the source offset.  Only this
        // rank's destination pointer may differ between ranks (gather passes
        // none off the root); it narrows this rank's copy width, or sends a
        // rank whose destination the TMA engine cannot address to the LDG/STG
        // kernel with the same grid.  Both kernels run the same two barriers.
        const int sharedWidth =
          std::min({ alignWidth(a.sendOff), alignWidth(len), alignWidth(a.dstStride), alignWidth(a.srcStride) });
        const int width = std::min(sharedWidth, alignWidth((uint64_t)(uintptr_t)a.recvLocal));
        const bool bulk =
          k_->moveBulk != nullptr && sharedWidth == 16 && cfg_.tmaMinBytes > 0 && len >= cfg_.tmaMinBytes;
        int blocks;
        if (bulk) {
            // Large chunks: the copy engine streams 32 KiB tiles through
            // shared memory; a few CTAs (>= 4 tiles each) saturate the link
            const uint64_t pieces =
              (mode == fb::MOVE_SCATTER || mode == fb::MOVE_BCAST) ? 1 : (uint64_t)n;
            const uint64_t tiles = pieces * ((len + 32767) / 32768);
            const int maxB = std::min(cfg_.maxBlocks, FB_MAX_BLOCKS / cfg_.channels);
            blocks = (int)std::clamp<uint64_t>(tiles / 4, 1, (uint64_t)maxB);
        } else {
            blocks = blocksFor(len / sharedWidth, 2);
        }
        cudaError_t ce;
        if (ss && streamBarrier(flags, s) != FB_OK) {
            return FB_E_CUDA;
        }
        if (bulk && fb::moveBulkSupported(a)) {
            ce = k_->moveBulk(a, blocks, s);
            stats_.tmaLaunches++;
        } else {
            ce = k_->move(a, width, blocks, cfg_.threads, s);
        }
        if (ce != cudaSuccess) {
            return FB_E_CUDA;
        }
        if (ss && streamBarrier(flags, s) != FB_OK) {
            return FB_E_CUDA;
        }
        stats_.launches++;
        stats_.bytes += len;
    }
    return FB_OK;
}

int Communicator::broadcast(void* buf,
                            size_t bytes,
                            int root,
                            int flags,
                            cudaStream_t s)
{
    NvtxRange nvtxRange("fb::broadcast");
    if (root < 0 || root >= dev_.nranks) {
        return FB_E_INVALID;
    }
    if ((flags & FB_FLAG_SYMMETRIC) && !inHeap(buf, bytes)) {
        return FB_E_INVALID;
    }
    return moveLike(fb::MOVE_BCAST, buf, buf, bytes, root, flags, s);
}

int Communicator::allGather(const void* send,
                            void* recv,
                            size_t bytesPerRank,
                            int flags,
                            cudaStream_t s)
{
    NvtxRange nvtxRange("fb::allGather");
    if ((flags & FB_FLAG_SYMMETRIC) &&
        (!inHeap(send, bytesPerRank) ||
         !inHeap(recv, bytesPerRank * dev_.nranks))) {
        // pull only needs the *send* side symmetric
        if (!inHeap(send, bytesPerRank)) {
            return FB_E_INVALID;
        }
    }
    return moveLike(fb::MOVE_ALLGATHER, send, recv, bytesPerRank, 0, flags, s);
}

int Communicator::gather(const void* send,
                         void* recv,
                         size_t bytesPerRank,
                         int root,
                         int flags,
                         cudaStream_t s)
{
    NvtxRange nvtxRange("fb::gather");
    if (root < 0 || root >= dev_.nranks) {
        return FB_E_INVALID;
    }
    return moveLike(fb::MOVE_GATHER, send, recv, bytesPerRank, root, flags, s);
}

int Communicator::scatter(const void* send,
                          void* recv,
                          size_t bytesPerRank,
                          int root,
                          int flags,
                          cudaStream_t s)
{
    NvtxRange nvtxRange("fb::scatter");
    if (root < 0 || root >= dev_.nranks) {
        return FB_E_INVALID;
    }
    return moveLike(fb::MOVE_SCATTER, send, recv, bytesPerRank, root, flags, s);
}

int Communicator::allToAll(const void* send,
                           void* recv,
                           size_t bytesPerRank,
                           int flags,
                           cudaStream_t s)
{
    NvtxRange nvtxRange("fb::allToAll");
    return moveLike(fb::MOVE_ALLTOALL, send, recv, bytesPerRank, 0, flags, s);
}

int Communicator::barrier(cudaStream_t s)
{
    NvtxRange nvtxRange("fb::barrier");
    bindDevice();
    if (dev_.nranks == 1) {
        return FB_OK;
    }
    stats_.launches++;
    if (streamSync_) {
        return streamBarrier(0, s);
    }
    return k_->barrier(dev_, s) == cudaSuccess ? FB_OK : FB_E_CUDA;
}

// ---------------------------------------------------------------------------
// Set-up tail shared by both wiring modes
// ---------------------------------------------------------------------------
void Communicator::finishSetup()
{
    k_ = loop_ ? &HOST_KERNELS : &CUDA_KERNELS;
    if (dev_.heap[dev_.rank] != nullptr && heapTotal_ > 0) {
        std::unique_lock<std::shared_mutex> lk(heapRangesMx);
        heapRanges.emplace_back((const uint8_t*)dev_.heap[dev_.rank], heapTotal_);
        nHeapRanges.fetch_add(1, std::memory_order_release);
        heapRegistered_ = true;
    }
    if (loop_) {
        // the host twins synchronise inside the "kernels", like the GPU ones
        streamSync_ = false;
        streamWaitOk_ = false;
        streamWriteOk_ = false;
        return;
    }
    streamSync_ = cfg_.streamSync > 0;
    streamWaitOk_ = false;
    const DriverApi& api = getDriverApi();
    const char* off = getenv("FAABRIC_STREAM_MEMOPS");
    if (api.cuStreamWaitValue32 != nullptr && !(off != nullptr && off[0] == '0')) {
        // self-test: a wait that is already satisfied on a word of our own pad
        bindDevice();
        cudaStream_t t = nullptr;
        if (cudaStreamCreateWithFlags(&t, cudaStreamNonBlocking) == cudaSuccess) {
            CUresult r = api.cuStreamWaitValue32(
              (CUstream)t,
              (CUdeviceptr)(uintptr_t)(dev_.sig[dev_.rank] + FB_SIG_SBAR_OFF),
              0,
              CU_STREAM_WAIT_VALUE_GEQ);
            if (r == CUDA_SUCCESS && cudaStreamSynchronize(t) == cudaSuccess) {
                streamWaitOk_ = true;
            } else {
                cudaGetLastError();
            }
            // completion word: err[1], host-mapped next to the error word
            if (api.cuStreamWriteValue32 != nullptr && dev_.err != nullptr) {
                void* devPtr = nullptr;
                if (cudaHostGetDevicePointer(&devPtr, (void*)(dev_.err + 1), 0) == cudaSuccess) {
                    r = api.cuStreamWriteValue32((CUstream)t, (CUdeviceptr)(uintptr_t)devPtr, 0x5a5a0001u, 0);
                    if (r == CUDA_SUCCESS && cudaStreamSynchronize(t) == cudaSuccess &&
                        *reinterpret_cast<volatile uint32_t*>(dev_.err + 1) == 0x5a5a0001u) {
                        streamWriteOk_ = true;
                    }
                }
                cudaGetLastError();
                dev_.err[1] = 0;
            }
            cudaStreamDestroy(t);
        }
    }
}

int Communicator::streamWaitGe(cudaStream_t s,
                               const uint32_t* localWord,
                               uint32_t value)
{
    if (streamWaitOk_) {
        CUresult r = getDriverApi().cuStreamWaitValue32(
          (CUstream)s,
          (CUdeviceptr)(uintptr_t)localWord,
          value,
          CU_STREAM_WAIT_VALUE_GEQ);
        if (r == CUDA_SUCCESS) {
            return FB_OK;
        }
        // e.g. not permitted in this capture mode: use the spin kernel
    }
    return k_->waitWord(dev_, localWord, value, s) == cudaSuccess ? FB_OK : FB_E_CUDA;
}

// Stream-ordered barrier of one channel: every rank signals every peer from a
// (non-spinning) kernel and then waits for all of them at stream level.
int Communicator::streamBarrier(int flags, cudaStream_t s)
{
    const int n = dev_.nranks;
    if (n == 1) {
        return FB_OK;
    }
    int ch = FB_FLAG_GET_CHANNEL(flags) % cfg_.channels;
    const uint32_t e = ++sbarEpoch_[ch];
    const uint32_t wordOff = FB_SIG_SBAR_OFF + (uint32_t)ch * FB_MAX_RANKS;
    if (k_->signalPeers(dev_, wordOff, e, s) != cudaSuccess) {
        return FB_E_CUDA;
    }
    for (int p = 0; p < n; p++) {
        if (p == dev_.rank) {
            continue;
        }
        int rc = streamWaitGe(s, dev_.sig[dev_.rank] + wordOff + p, e);
        if (rc != FB_OK) {
            return rc;
        }
    }
    return FB_OK;
}

bool Communicator::syncStreamBounded(cudaStream_t s, uint64_t timeoutMs)
{
    if (loop_) {
        return true; // every call already ran to completion
    }
    bindDevice();
    const auto t0 = std::chrono::steady_clock::now();
    uint32_t spins = 0;
    while (true) {
        cudaError_t e = cudaStreamQuery(s);
        if (e == cudaSuccess) {
            return true;
        }
        if (e != cudaErrorNotReady) {
            cudaGetLastError();
            return false;
        }
        if (++spins > 2000) {
            std::this_thread::sleep_for(std::chrono::microseconds(50));
            auto ms = std::chrono::duration_cast<std::chrono::milliseconds>(
                        std::chrono::steady_clock::now() - t0)
                        .count();
            if ((uint64_t)ms > timeoutMs) {
                abortPendingWaits();
                cudaStreamSynchronize(s);
                return false;
            }
        }
    }
}

bool Communicator::waitStreamFast(cudaStream_t s)
{
    if (parent_ != nullptr) {
        // one completion word per rank: its sequence lives in the parent
        return parent_->waitStreamFast(s);
    }
    if (loop_) {
        return true;
    }
    bindDevice();
    if (streamWriteOk_) {
        void* devPtr = nullptr;
        cudaHostGetDevicePointer(&devPtr, (void*)(dev_.err + 1), 0);
        const uint32_t seq = ++doneSeq_ | 0x80000000u;
        if (getDriverApi().cuStreamWriteValue32((CUstream)s, (CUdeviceptr)(uintptr_t)devPtr, seq, 0) == CUDA_SUCCESS) {
            volatile uint32_t* word = reinterpret_cast<volatile uint32_t*>(dev_.err + 1);
            // typical wait is a few microseconds; give up spinning after ~1 ms
            for (int spin = 0; spin < 200000; spin++) {
                if (*word == seq) {
                    return true;
                }
                __builtin_ia32_pause();
            }
        }
    }
    if (cudaStreamSynchronize(s) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return true;
}

// A peer never arrived: flag the error and satisfy every stream-level wait
// this rank may have queued so the stream drains instead of hanging forever
// (stream memory operations have no timeout of their own).
void Communicator::abortPendingWaits()
{
    *reinterpret_cast<volatile uint32_t*>(dev_.err) = FB_ERR_HOST_ABORT;
    if (loop_) {
        return;
    }
    cudaStream_t t = nullptr;
    if (cudaStreamCreateWithFlags(&t, cudaStreamNonBlocking) != cudaSuccess) {
        cudaGetLastError();
        return;
    }
    uint32_t* pad = dev_.sig[dev_.rank];
    cudaMemcpyAsync(pad + FB_P2P_READY_OFF, recvSeq_, sizeof(recvSeq_), cudaMemcpyHostToDevice, t);
    cudaMemcpyAsync(pad + FB_P2P_ACK_OFF, sendSeq_, sizeof(sendSeq_), cudaMemcpyHostToDevice, t);
    std::vector<uint32_t> sb(FB_SIG_SBAR_WORDS);
    for (int ch = 0; ch < FB_MAX_CHANNELS; ch++) {
        for (int p = 0; p < FB_MAX_RANKS; p++) {
            sb[ch * FB_MAX_RANKS + p] = sbarEpoch_[ch];
        }
    }
    cudaMemcpyAsync(pad + FB_SIG_SBAR_OFF, sb.data(), sb.size() * 4, cudaMemcpyHostToDevice, t);
    cudaMemcpyAsync(pad + FB_SIG_USER_OFF, userSigConsumed_, sizeof(userSigConsumed_), cudaMemcpyHostToDevice, t);
    cudaStreamSynchronize(t);
    cudaStreamDestroy(t);
    cudaGetLastError();
}

// ---------------------------------------------------------------------------
// Point to point
// ---------------------------------------------------------------------------
static int p2pBlocks(size_t len)
{
    return (int)std::clamp<size_t>(len / (64 << 10), 1, 32);
}

int Communicator::sendChunk(const uint8_t* buf, size_t len, int peer, cudaStream_t s)
{
    const uint32_t seq = ++sendSeq_[peer];
    // ---- space in the byte ring of this destination (FIFO allocation) ----
    const uint64_t ringBytes = cfg_.p2pBounceBytes;
    const uint64_t need = roundUp(std::max<size_t>(len, 16), 256);
    uint64_t off = bounceHead_[peer];
    if (off + need > ringBytes) {
        off = 0; // wrap: the tail end of the ring stays unused this lap
    }
    auto& inflight = bounceInflight_[peer];
    uint32_t waitFor = 0;
    auto overlaps = [&](const BounceMsg& m) { return m.off < off + need && off < m.off + m.len; };
    while (!inflight.empty() &&
           (inflight.size() >= FB_P2P_RING - 1 || overlaps(inflight.front()))) {
        // the oldest message must have been pulled before its bytes (or its
        // descriptor slot) are reused: wait for its ack, at stream level
        waitFor = inflight.front().seq;
        inflight.pop_front();
    }
    if (waitFor != 0) {
        int rc = streamWaitGe(s, dev_.sig[dev_.rank] + FB_P2P_ACK_OFF + peer, waitFor);
        if (rc != FB_OK) {
            return rc;
        }
    }
    inflight.push_back({ seq, off, need });
    bounceHead_[peer] = off + need;

    fb::P2PArgs a;
    memset(&a, 0, sizeof(a));
    a.comm = dev_;
    a.local = const_cast<uint8_t*>(buf);
    a.bytes = len;
    a.srcOff = mboxOff_ + (uint64_t)peer * ringBytes + off;
    a.descOff = p2pDescOff_;
    a.seq = seq;
    a.peer = peer;
    a.stage = 1;
    stats_.launches++;
    stats_.bytes += len;
    int w = alignWidth((uint64_t)(uintptr_t)buf);
    return k_->p2pSend(a, w, p2pBlocks(len), s) == cudaSuccess ? FB_OK : FB_E_CUDA;
}

int Communicator::recvChunk(uint8_t* buf, size_t len, int peer, cudaStream_t s)
{
    const uint32_t seq = ++recvSeq_[peer];
    int rc = streamWaitGe(s, dev_.sig[dev_.rank] + FB_P2P_READY_OFF + peer, seq);
    if (rc != FB_OK) {
        return rc;
    }
    fb::P2PArgs a;
    memset(&a, 0, sizeof(a));
    a.comm = dev_;
    a.local = buf;
    a.bytes = len;
    a.heapBytes = heapTotal_;
    a.descOff = p2pDescOff_;
    a.seq = seq;
    a.peer = peer;
    stats_.launches++;
    int w = alignWidth((uint64_t)(uintptr_t)buf);
    return k_->p2pPull(a, w, p2pBlocks(len), s) == cudaSuccess ? FB_OK : FB_E_CUDA;
}

int Communicator::send(const void* buf, size_t bytes, int peer, cudaStream_t s)
{
    NvtxRange nvtxRange("fb::send");
    if (parent_ != nullptr) {
        return FB_E_UNSUPPORTED; // see subset()
    }
    if (peer < 0 || peer >= dev_.nranks) {
        return FB_E_INVALID;
    }
    bindDevice();
    // zero-byte messages still synchronise (one empty chunk), like the
    // reference's empty MPI messages
    size_t off = 0;
    do {
        size_t len = std::min<size_t>(bounceSlotBytes_, bytes - off);
        int rc = sendChunk((const uint8_t*)buf + off, len, peer, s);
        if (rc != FB_OK) {
            return rc;
        }
        off += len;
    } while (off < bytes);
    return FB_OK;
}

int Communicator::recv(void* buf, size_t bytes, int peer, cudaStream_t s)
{
    NvtxRange nvtxRange("fb::recv");
    if (parent_ != nullptr) {
        return FB_E_UNSUPPORTED; // see subset()
    }
    if (peer < 0 || peer >= dev_.nranks) {
        return FB_E_INVALID;
    }
    bindDevice();
    size_t off = 0;
    do {
        size_t len = std::min<size_t>(bounceSlotBytes_, bytes - off);
        int rc = recvChunk((uint8_t*)buf + off, len, peer, s);
        if (rc != FB_OK) {
            return rc;
        }
        off += len;
    } while (off < bytes);
    return FB_OK;
}

int Communicator::sendRecv(const void* sendBuf,
                           size_t sendBytes,
                           int dst,
                           void* recvBuf,
                           size_t recvBytes,
                           int src,
                           cudaStream_t s)
{
    NvtxRange nvtxRange("fb::sendRecv");
    if (parent_ != nullptr) {
        return FB_E_UNSUPPORTED; // see subset()
    }
    if (dst < 0 || dst >= dev_.nranks || src < 0 || src >= dev_.nranks) {
        return FB_E_INVALID;
    }
    bindDevice();
    size_t so = 0;
    size_t ro = 0;
    bool sendDone = false;
    bool recvDone = false;
    while (!sendDone || !recvDone) {
        if (!sendDone) {
            size_t len = std::min<size_t>(bounceSlotBytes_, sendBytes - so);
            int rc = sendChunk((const uint8_t*)sendBuf + so, len, dst, s);
            if (rc != FB_OK) {
                return rc;
            }
            so += len;
            sendDone = so >= sendBytes;
        }
        if (!recvDone) {
            size_t len = std::min<size_t>(bounceSlotBytes_, recvBytes - ro);
            int rc = recvChunk((uint8_t*)recvBuf + ro, len, src, s);
            if (rc != FB_OK) {
                return rc;
            }
            ro += len;
            recvDone = ro >= recvBytes;
        }
    }
    return FB_OK;
}

int Communicator::putSignal(const void* local,
                            uint64_t dstOffset,
                            size_t bytes,
                            int peer,
                            int signalIdx,
                            int blocks,
                            cudaStream_t s)
{
    if (parent_ != nullptr) {
        return FB_E_UNSUPPORTED; // see subset()
    }
    if (peer < 0 || peer >= dev_.nranks || signalIdx < 0 ||
        signalIdx >= FB_SIG_USER_WORDS || blocks < 1) {
        return FB_E_INVALID;
    }
    bindDevice();
    fb::PutArgs a;
    memset(&a, 0, sizeof(a));
    a.comm = dev_;
    a.local = (const uint8_t*)local;
    a.dstOff = dstOffset;
    a.bytes = bytes;
    a.peer = peer;
    a.signalIdx = signalIdx;
    int w = std::min(alignWidth((uint64_t)(uintptr_t)local),
                     alignWidth(dstOffset));
    stats_.launches++;
    stats_.bytes += bytes;
    return k_->putSignal(a, w, blocks, s) == cudaSuccess ? FB_OK : FB_E_CUDA;
}

int Communicator::waitSignal(int signalIdx, uint32_t count, cudaStream_t s)
{
    if (parent_ != nullptr) {
        return FB_E_UNSUPPORTED; // see subset()
    }
    if (signalIdx < 0 || signalIdx >= FB_SIG_USER_WORDS) {
        return FB_E_INVALID;
    }
    bindDevice();
    if (streamSync_) {
        userSigConsumed_[signalIdx] += count;
        return streamWaitGe(
          s, dev_.sig[dev_.rank] + FB_SIG_USER_OFF + signalIdx, userSigConsumed_[signalIdx]);
    }
    stats_.launches++;
    return k_->waitSignal(dev_, signalIdx, count, s) == cudaSuccess ? FB_OK : FB_E_CUDA;
}

bool Communicator::rmaTargetOk(uint64_t dstOffset, uint64_t bytes, size_t align, int peer) const
{
    return dstOffset >= userOff_ && dstOffset <= heapTotal_ && bytes <= heapTotal_ - dstOffset &&
           (uintptr_t)(dev_.heap[peer] + dstOffset) % align == 0;
}

int Communicator::accumulate(const void* origin,
                             uint64_t dstOffset,
                             size_t count,
                             int dtype,
                             int op,
                             int peer,
                             void* fetchOut,
                             cudaStream_t s)
{
    if (parent_ != nullptr) {
        return FB_E_UNSUPPORTED; // see subset()
    }
    const size_t esize = fbDtypeSize(dtype);
    if (esize == 0 || peer < 0 || peer >= dev_.nranks) {
        return FB_E_INVALID;
    }
    if (!fb::rmaSupported(dtype, op, true)) {
        return FB_E_UNSUPPORTED;
    }
    if ((op == FB_OP_NO_OP && fetchOut == nullptr) || (op != FB_OP_NO_OP && origin == nullptr && count > 0) ||
        count > heapTotal_ / esize || !rmaTargetOk(dstOffset, (uint64_t)count * esize, esize, peer)) {
        return FB_E_INVALID;
    }
    if (count == 0) {
        return FB_OK;
    }
    bindDevice();
    fb::RmaArgs a;
    memset(&a, 0, sizeof(a));
    a.target = dev_.heap[peer] + dstOffset;
    a.origin = (const uint8_t*)origin;
    a.result = (uint8_t*)fetchOut;
    a.count = count;
    stats_.launches++;
    stats_.bytes += (uint64_t)count * esize;
    return k_->rmaAccumulate(a, dtype, op, s) == cudaSuccess ? FB_OK : FB_E_CUDA;
}

int Communicator::compareAndSwap(const void* compare,
                                 const void* swap,
                                 void* result,
                                 uint64_t dstOffset,
                                 int dtype,
                                 int peer,
                                 cudaStream_t s)
{
    if (parent_ != nullptr) {
        return FB_E_UNSUPPORTED; // see subset()
    }
    const size_t esize = fbDtypeSize(dtype);
    if (esize == 0 || peer < 0 || peer >= dev_.nranks) {
        return FB_E_INVALID;
    }
    if (!fb::rmaCasSupported(dtype)) {
        return FB_E_UNSUPPORTED;
    }
    if (compare == nullptr || swap == nullptr || result == nullptr || !rmaTargetOk(dstOffset, esize, esize, peer)) {
        return FB_E_INVALID;
    }
    bindDevice();
    fb::RmaCasArgs a;
    memset(&a, 0, sizeof(a));
    a.target = dev_.heap[peer] + dstOffset;
    a.compare = (const uint8_t*)compare;
    a.swap = (const uint8_t*)swap;
    a.result = (uint8_t*)result;
    stats_.launches++;
    stats_.bytes += esize;
    return k_->rmaCompareSwap(a, dtype, s) == cudaSuccess ? FB_OK : FB_E_CUDA;
}

static_assert(sizeof(fb::RmaCopyDesc) == sizeof(fb::GroupSeg) && FB_RMA_COPY_MAX_ITEMS == FB_GROUP_MAX_SEGS,
              "copy tables share the group tables' staging slots");

int Communicator::putGetMany(const RmaCopy* items, size_t n, cudaStream_t s)
{
    if (parent_ != nullptr) {
        return FB_E_UNSUPPORTED; // see subset()
    }
    if (n > 0 && items == nullptr) {
        return FB_E_INVALID;
    }
    for (size_t i = 0; i < n; i++) {
        const RmaCopy& it = items[i];
        if (it.peer < 0 || it.peer >= dev_.nranks ||
            (it.bytes > 0 && (it.local == nullptr || !rmaTargetOk(it.offset, it.bytes, 1, it.peer)))) {
            return FB_E_INVALID;
        }
    }
    bindDevice();
    std::vector<fb::RmaCopyDesc> table;
    table.reserve(std::min<size_t>(n, FB_RMA_COPY_MAX_ITEMS));
    size_t i = 0;
    while (i < n) {
        table.clear();
        uint64_t chunks = 0;
        uint64_t bytes = 0;
        for (; i < n && table.size() < FB_RMA_COPY_MAX_ITEMS; i++) {
            const RmaCopy& it = items[i];
            if (it.bytes == 0) {
                continue;
            }
            uint8_t* remote = dev_.heap[it.peer] + it.offset;
            uint8_t* local = (uint8_t*)it.local;
            table.push_back(fb::RmaCopyDesc{ it.get ? remote : local, it.get ? local : remote, it.bytes, chunks });
            chunks += fb::fbRmaCopyChunks(it.bytes);
            bytes += it.bytes;
        }
        if (table.empty()) {
            break;
        }
        fb::RmaCopyArgs a;
        memset(&a, 0, sizeof(a));
        a.items = table.data(); // the host twin reads the table in place
        a.nItems = (uint32_t)table.size();
        a.totalChunks = chunks;
        ManySlot* slot = nullptr;
        if (!loop_) {
            slot = nextManySlot();
            if (slot == nullptr) {
                return FB_E_CUDA;
            }
            const size_t tableBytes = table.size() * sizeof(fb::RmaCopyDesc);
            memcpy(slot->hSegs, table.data(), tableBytes);
            if (cudaMemcpyAsync(slot->dSegs, slot->hSegs, tableBytes, cudaMemcpyHostToDevice, s) != cudaSuccess) {
                return FB_E_CUDA;
            }
            a.items = reinterpret_cast<const fb::RmaCopyDesc*>(slot->dSegs);
        }
        stats_.launches++;
        stats_.bytes += bytes;
        if (k_->rmaCopyMany(a, s) != cudaSuccess) {
            return FB_E_CUDA;
        }
        if (slot != nullptr) {
            cudaEventRecord(slot->ev, s);
            slot->used = true;
        }
    }
    return FB_OK;
}

} // namespace faabric::device
