#include <faabric/util/config.h>
#include <faabric/util/dirty.h>
#include <faabric/util/logging.h>
#include <faabric/util/memory.h>
#include <faabric/util/timing.h>

#include "launch_api.h"

#include <atomic>
#include <cstring>
#include <fcntl.h>
#include <linux/userfaultfd.h>
#include <mutex>
#include <unordered_map>
#include <poll.h>
#include <signal.h>
#include <stdexcept>
#include <sys/ioctl.h>
#include <sys/mman.h>
#include <sys/syscall.h>
#include <thread>
#include <unistd.h>

namespace faabric::util {

// ---------------------------------------------------------------------------
// Tracker selection
// ---------------------------------------------------------------------------
static std::shared_ptr<DirtyTracker> activeTracker;
static std::mutex trackerMx;

static std::shared_ptr<DirtyTracker> makeTracker(const std::string& mode)
{
    if (mode == "softpte") {
        return std::make_shared<SoftPTEDirtyTracker>();
    }
    if (mode == "segfault") {
        return std::make_shared<SegfaultDirtyTracker>();
    }
    if (mode == "none") {
        return std::make_shared<NoneDirtyTracker>();
    }
    if (mode == "uffd" || mode == "uffd-wp" || mode == "uffd-thread" ||
        mode == "uffd-thread-wp") {
        return std::make_shared<UffdDirtyTracker>(mode);
    }
    SPDLOG_ERROR("Unrecognised dirty tracking mode: {}", mode);
    throw std::runtime_error("Unrecognised dirty tracking mode");
}

std::shared_ptr<DirtyTracker> getDirtyTracker()
{
    std::lock_guard<std::mutex> lk(trackerMx);
    if (activeTracker == nullptr) {
        activeTracker = makeTracker(getSystemConfig().dirtyTrackingMode);
    }
    return activeTracker;
}

void resetDirtyTracker()
{
    std::lock_guard<std::mutex> lk(trackerMx);
    activeTracker = makeTracker(getSystemConfig().dirtyTrackingMode);
}

// ---------------------------------------------------------------------------
// None
// ---------------------------------------------------------------------------
void NoneDirtyTracker::clearAll()
{
    dirtyPages.clear();
}

void NoneDirtyTracker::startTracking(std::span<uint8_t> region)
{
    dirtyPages = std::vector<char>(getRequiredHostPages(region.size()), 1);
}

void NoneDirtyTracker::stopTracking(std::span<uint8_t> region) {}

std::vector<char> NoneDirtyTracker::getDirtyPages(std::span<uint8_t> region)
{
    return dirtyPages;
}

void NoneDirtyTracker::startThreadLocalTracking(std::span<uint8_t> region) {}

void NoneDirtyTracker::stopThreadLocalTracking(std::span<uint8_t> region) {}

std::vector<char> NoneDirtyTracker::getThreadLocalDirtyPages(
  std::span<uint8_t> region)
{
    return std::vector<char>(getRequiredHostPages(region.size()), 0);
}

std::vector<char> NoneDirtyTracker::getBothDirtyPages(std::span<uint8_t> region)
{
    return getDirtyPages(region);
}

// ---------------------------------------------------------------------------
// Shared record of the region currently being tracked by fault-driven
// trackers.  Process-wide records live in a table (RegionTable below),
// plus a thread-local record for per-thread attribution.
// ---------------------------------------------------------------------------
namespace {
struct TrackingRecord
{
    uint8_t* regionBase = nullptr;
    uint8_t* regionTop = nullptr;
    size_t nPages = 0;
    // atomic chars so that concurrent faulting threads can flag safely
    std::unique_ptr<std::atomic<char>[]> flags;

    void reset(std::span<uint8_t> region)
    {
        regionBase = region.data();
        regionTop = region.data() + region.size();
        nPages = getRequiredHostPages(region.size());
        flags = std::make_unique<std::atomic<char>[]>(nPages);
        for (size_t i = 0; i < nPages; i++) {
            flags[i].store(0, std::memory_order_relaxed);
        }
    }

    void clear()
    {
        regionBase = nullptr;
        regionTop = nullptr;
        nPages = 0;
        flags.reset();
    }

    bool contains(const void* addr) const
    {
        return addr >= regionBase && addr < regionTop;
    }

    void mark(const void* addr)
    {
        size_t page = ((uintptr_t)addr - (uintptr_t)regionBase) / HOST_PAGE_SIZE;
        if (page < nPages) {
            flags[page].store(1, std::memory_order_relaxed);
        }
    }

    std::vector<char> snapshot(size_t wantPages) const
    {
        std::vector<char> out(wantPages, 0);
        for (size_t i = 0; i < std::min(wantPages, nPages); i++) {
            out[i] = flags[i].load(std::memory_order_relaxed);
        }
        return out;
    }
};

// Process-wide records: one per tracked region.  A worker that serves several
// per-GPU virtual hosts runs several executors side by side, each tracking its
// own function memory (the reference tracks one region per process).  Fixed
// slots, published by storing regionBase last, so the SIGSEGV handler can walk
// the table without locks or allocation.
struct RegionTable
{
    static constexpr int SLOTS = 64;
    TrackingRecord slots[SLOTS];
    std::mutex mx; // writers only (never taken in a signal handler)

    TrackingRecord* find(const void* addr)
    {
        for (auto& r : slots) {
            uint8_t* base = __atomic_load_n(&r.regionBase, __ATOMIC_ACQUIRE);
            if (base != nullptr && addr >= base && addr < r.regionTop) {
                return &r;
            }
        }
        return nullptr;
    }

    void reset(std::span<uint8_t> region)
    {
        std::lock_guard<std::mutex> lk(mx);
        TrackingRecord* slot = nullptr;
        for (auto& r : slots) {
            if (r.regionBase == region.data()) {
                slot = &r;
                break;
            }
        }
        if (slot == nullptr) {
            for (auto& r : slots) {
                if (r.regionBase == nullptr) {
                    slot = &r;
                    break;
                }
            }
        }
        if (slot == nullptr) {
            throw std::runtime_error("Too many regions under dirty tracking");
        }
        // unpublish, rebuild, publish
        __atomic_store_n(&slot->regionBase, (uint8_t*)nullptr, __ATOMIC_RELEASE);
        TrackingRecord fresh;
        fresh.reset(region);
        slot->regionTop = fresh.regionTop;
        slot->nPages = fresh.nPages;
        slot->flags = std::move(fresh.flags);
        __atomic_store_n(&slot->regionBase, region.data(), __ATOMIC_RELEASE);
    }

    void clear()
    {
        std::lock_guard<std::mutex> lk(mx);
        for (auto& r : slots) {
            __atomic_store_n(&r.regionBase, (uint8_t*)nullptr, __ATOMIC_RELEASE);
            r.clear();
        }
    }

    void release(std::span<uint8_t> region)
    {
        std::lock_guard<std::mutex> lk(mx);
        for (auto& r : slots) {
            if (r.regionBase == region.data()) {
                // keep the flags readable until the next reset of the slot
                return;
            }
        }
    }

    std::vector<char> snapshot(std::span<uint8_t> region)
    {
        const size_t want = getRequiredHostPages(region.size());
        std::lock_guard<std::mutex> lk(mx);
        for (auto& r : slots) {
            if (r.regionBase == region.data()) {
                return r.snapshot(want);
            }
        }
        return std::vector<char>(want, 0);
    }
};

RegionTable globalRecords;
thread_local TrackingRecord threadRecord;
}

// ---------------------------------------------------------------------------
// Segfault tracker
// ---------------------------------------------------------------------------
SegfaultDirtyTracker::SegfaultDirtyTracker()
{
    setUpSignalHandler();
}

static struct sigaction previousSegvAction;

void SegfaultDirtyTracker::handler(int sig, void* infoV, void* context) noexcept
{
    auto* info = (siginfo_t*)infoV;
    void* faultAddr = info->si_addr;
    bool handled = false;
    if (threadRecord.regionBase != nullptr && threadRecord.contains(faultAddr)) {
        threadRecord.mark(faultAddr);
        handled = true;
    }
    if (TrackingRecord* rec = globalRecords.find(faultAddr)) {
        // Only attribute to the global record when no thread-local tracking
        // is active for this thread (matches the reference's split)
        if (!handled) {
            rec->mark(faultAddr);
        }
        handled = true;
    }
    if (!handled) {
        // A genuine crash: restore the previous disposition and re-raise
        ::sigaction(SIGSEGV, &previousSegvAction, nullptr);
        ::raise(SIGSEGV);
        return;
    }
    // Re-enable writes on the page
    uintptr_t page = (uintptr_t)faultAddr & ~((uintptr_t)HOST_PAGE_SIZE - 1);
    if (::mprotect((void*)page, HOST_PAGE_SIZE, PROT_READ | PROT_WRITE) != 0) {
        _exit(139);
    }
}

static void segvTrampoline(int sig, siginfo_t* info, void* context)
{
    SegfaultDirtyTracker::handler(sig, info, context);
}

void SegfaultDirtyTracker::setUpSignalHandler()
{
    struct sigaction sa;
    memset(&sa, 0, sizeof(sa));
    sa.sa_flags = SA_SIGINFO | SA_NODEFER;
    sa.sa_sigaction = segvTrampoline;
    sigemptyset(&sa.sa_mask);
    struct sigaction old;
    if (::sigaction(SIGSEGV, &sa, &old) != 0) {
        throw std::runtime_error("Failed sigaction for SIGSEGV");
    }
    if (old.sa_sigaction != segvTrampoline) {
        previousSegvAction = old;
    }
}

void SegfaultDirtyTracker::clearAll()
{
    globalRecords.clear();
    threadRecord.clear();
}

void SegfaultDirtyTracker::startTracking(std::span<uint8_t> region)
{
    if (region.empty() || region.data() == nullptr) {
        return;
    }
    PROF_START(MprotectStart)
    // (a crash handler installed after this tracker was created would have
    // taken SIGSEGV over: make sure our handler is in front, chaining to it)
    setUpSignalHandler();
    globalRecords.reset(region);
    if (::mprotect(region.data(), region.size(), PROT_READ) != 0) {
        SPDLOG_ERROR("Failed to start tracking with mprotect: {}", strerror(errno));
        throw std::runtime_error("Failed mprotect to start tracking");
    }
    PROF_END(MprotectStart)
}

void SegfaultDirtyTracker::stopTracking(std::span<uint8_t> region)
{
    if (region.empty() || region.data() == nullptr) {
        return;
    }
    if (::mprotect(region.data(), region.size(), PROT_READ | PROT_WRITE) != 0) {
        SPDLOG_ERROR("Failed to stop tracking with mprotect: {}", strerror(errno));
        throw std::runtime_error("Failed mprotect to stop tracking");
    }
}

std::vector<char> SegfaultDirtyTracker::getDirtyPages(std::span<uint8_t> region)
{
    return globalRecords.snapshot(region);
}

void SegfaultDirtyTracker::startThreadLocalTracking(std::span<uint8_t> region)
{
    if (region.empty() || region.data() == nullptr) {
        return;
    }
    threadRecord.reset(region);
}

void SegfaultDirtyTracker::stopThreadLocalTracking(std::span<uint8_t> region) {}

std::vector<char> SegfaultDirtyTracker::getThreadLocalDirtyPages(
  std::span<uint8_t> region)
{
    return threadRecord.snapshot(getRequiredHostPages(region.size()));
}

std::vector<char> SegfaultDirtyTracker::getBothDirtyPages(
  std::span<uint8_t> region)
{
    std::vector<char> g = getDirtyPages(region);
    std::vector<char> t = getThreadLocalDirtyPages(region);
    mergeDirtyPages(g, t);
    return g;
}

// ---------------------------------------------------------------------------
// Soft-dirty PTE tracker
// ---------------------------------------------------------------------------
#define PAGEMAP_ENTRY_BYTES 8
#define PAGEMAP_SOFT_DIRTY (1ull << 55)

bool SoftPTEDirtyTracker::isSupported()
{
    // Soft-dirty needs CONFIG_MEM_SOFT_DIRTY: probe by dirtying a fresh page
    int cfd = ::open("/proc/self/clear_refs", O_WRONLY);
    int pfd = ::open("/proc/self/pagemap", O_RDONLY);
    bool ok = false;
    if (cfd >= 0 && pfd >= 0) {
        void* p = ::mmap(nullptr,
                         HOST_PAGE_SIZE,
                         PROT_READ | PROT_WRITE,
                         MAP_PRIVATE | MAP_ANONYMOUS,
                         -1,
                         0);
        if (p != MAP_FAILED) {
            ((volatile char*)p)[0] = 1;
            if (::write(cfd, "4", 1) == 1) {
                uint64_t e = 0;
                off_t off = ((uintptr_t)p / HOST_PAGE_SIZE) * PAGEMAP_ENTRY_BYTES;
                bool clean = ::pread(pfd, &e, 8, off) == 8 &&
                             (e & PAGEMAP_SOFT_DIRTY) == 0;
                ((volatile char*)p)[1] = 2;
                bool dirty = ::pread(pfd, &e, 8, off) == 8 &&
                             (e & PAGEMAP_SOFT_DIRTY) != 0;
                ok = clean && dirty;
            }
            ::munmap(p, HOST_PAGE_SIZE);
        }
    }
    if (cfd >= 0) {
        ::close(cfd);
    }
    if (pfd >= 0) {
        ::close(pfd);
    }
    return ok;
}

SoftPTEDirtyTracker::SoftPTEDirtyTracker()
{
    clearRefsFd = ::open("/proc/self/clear_refs", O_WRONLY);
    pagemapFd = ::open("/proc/self/pagemap", O_RDONLY);
    if (clearRefsFd < 0 || pagemapFd < 0) {
        SPDLOG_ERROR("Could not open soft-dirty proc files: {}", strerror(errno));
        throw std::runtime_error("Could not open soft-dirty proc files");
    }
}

SoftPTEDirtyTracker::~SoftPTEDirtyTracker()
{
    if (clearRefsFd >= 0) {
        ::close(clearRefsFd);
    }
    if (pagemapFd >= 0) {
        ::close(pagemapFd);
    }
}

void SoftPTEDirtyTracker::clearAll()
{
    PROF_START(ClearSoftPTE)
    if (::write(clearRefsFd, "4", 1) != 1) {
        SPDLOG_ERROR("Failed to reset soft-dirty bits: {}", strerror(errno));
        throw std::runtime_error("Failed to reset soft-dirty bits");
    }
    PROF_END(ClearSoftPTE)
}

void SoftPTEDirtyTracker::startTracking(std::span<uint8_t> region)
{
    clearAll();
}

void SoftPTEDirtyTracker::stopTracking(std::span<uint8_t> region) {}

std::vector<char> SoftPTEDirtyTracker::getDirtyPages(std::span<uint8_t> region)
{
    PROF_START(GetDirtyRegions)
    size_t nPages = getRequiredHostPages(region.size());
    std::vector<uint64_t> entries(nPages, 0);
    off_t off = ((uintptr_t)region.data() / HOST_PAGE_SIZE) * PAGEMAP_ENTRY_BYTES;
    ssize_t want = (ssize_t)(nPages * PAGEMAP_ENTRY_BYTES);
    if (nPages > 0 && ::pread(pagemapFd, entries.data(), want, off) != want) {
        SPDLOG_ERROR("Could not read pagemap: {}", strerror(errno));
        throw std::runtime_error("Could not read pagemap");
    }
    std::vector<char> out(nPages, 0);
    for (size_t i = 0; i < nPages; i++) {
        out[i] = (entries[i] & PAGEMAP_SOFT_DIRTY) ? 1 : 0;
    }
    PROF_END(GetDirtyRegions)
    return out;
}

void SoftPTEDirtyTracker::startThreadLocalTracking(std::span<uint8_t> region) {}

void SoftPTEDirtyTracker::stopThreadLocalTracking(std::span<uint8_t> region) {}

std::vector<char> SoftPTEDirtyTracker::getThreadLocalDirtyPages(
  std::span<uint8_t> region)
{
    // Soft-dirty bits are per address space: no per-thread attribution
    return std::vector<char>(getRequiredHostPages(region.size()), 0);
}

std::vector<char> SoftPTEDirtyTracker::getBothDirtyPages(
  std::span<uint8_t> region)
{
    return getDirtyPages(region);
}

// ---------------------------------------------------------------------------
// userfaultfd write-protect tracker.  All four reference mode names are
// accepted; they all run the write-protect + event-thread mechanism here
// (missing-page mode only works on never-touched anonymous memory and
// signal-mode delivery is covered by the segfault tracker).
// ---------------------------------------------------------------------------
struct UffdDirtyTracker::Impl
{
    int uffd = -1;
    int stopPipe[2] = { -1, -1 };
    std::thread eventThread;
    std::atomic<bool> running{ false };
    std::span<uint8_t> tracked;
    // The event thread marks pages in the record the control calls reset
    std::mutex recordMx;
    // Features the kernel granted (see openUffd)
    bool wpUnpopulated = false;
    bool threadIds = false;
    // Faults carry the id of the faulting thread: a thread that asked for
    // thread-local tracking gets its own record (the counterpart of the
    // reference's per-thread SIGBUS bookkeeping, src/util/dirty.cpp:626-700)
    std::unordered_map<uint32_t, std::shared_ptr<TrackingRecord>> perThread;

    void loop()
    {
        while (running.load()) {
            pollfd fds[2] = { { uffd, POLLIN, 0 }, { stopPipe[0], POLLIN, 0 } };
            int pr = ::poll(fds, 2, 500);
            if (pr <= 0) {
                continue;
            }
            if (fds[1].revents & POLLIN) {
                break;
            }
            if (!(fds[0].revents & POLLIN)) {
                continue;
            }
            uffd_msg msg;
            ssize_t n = ::read(uffd, &msg, sizeof(msg));
            if (n != (ssize_t)sizeof(msg) || msg.event != UFFD_EVENT_PAGEFAULT) {
                continue;
            }
            void* addr = (void*)(uintptr_t)msg.arg.pagefault.address;
            {
                std::lock_guard<std::mutex> lk(recordMx);
                bool attributed = false;
                if (threadIds) {
                    auto it = perThread.find((uint32_t)msg.arg.pagefault.feat.ptid);
                    if (it != perThread.end() && it->second->contains(addr)) {
                        it->second->mark(addr);
                        attributed = true;
                    }
                }
                if (!attributed) {
                    if (TrackingRecord* rec = globalRecords.find(addr)) {
                        rec->mark(addr);
                    }
                }
            }
            // Drop write protection on the page and wake the faulting thread
            uffdio_writeprotect wp;
            wp.range.start = (uintptr_t)addr & ~((uintptr_t)HOST_PAGE_SIZE - 1);
            wp.range.len = HOST_PAGE_SIZE;
            wp.mode = 0;
            ::ioctl(uffd, UFFDIO_WRITEPROTECT, &wp);
        }
    }
};

// Opens a userfaultfd with write-protect faults, asking for the optional
// features too: protection of pages that are not populated yet (6.4+; without
// it the tracker pre-faults the region), of shared / file-backed memory
// (5.19+) and thread ids in fault messages
static int openUffd(bool* wpUnpopulated = nullptr, bool* threadIds = nullptr)
{
    const uint64_t base = UFFD_FEATURE_PAGEFAULT_FLAG_WP;
    const uint64_t wishes[] = {
        base | UFFD_FEATURE_THREAD_ID | UFFD_FEATURE_WP_UNPOPULATED | UFFD_FEATURE_WP_HUGETLBFS_SHMEM,
        base | UFFD_FEATURE_THREAD_ID | UFFD_FEATURE_WP_UNPOPULATED,
        base | UFFD_FEATURE_THREAD_ID,
        base
    };
    // FAABRIC_UFFD_FEATURES=basic behaves like an old kernel (tests)
    const char* limit = ::getenv("FAABRIC_UFFD_FEATURES");
    const bool basicOnly = limit != nullptr && std::string(limit) == "basic";
    for (uint64_t features : wishes) {
        if (basicOnly && features != base) {
            continue;
        }
        int fd = (int)::syscall(SYS_userfaultfd, O_CLOEXEC | O_NONBLOCK);
        if (fd < 0) {
            return -1;
        }
        uffdio_api api;
        memset(&api, 0, sizeof(api));
        api.api = UFFD_API;
        api.features = features;
        if (::ioctl(fd, UFFDIO_API, &api) == 0) {
            if (wpUnpopulated != nullptr) {
                *wpUnpopulated = (features & UFFD_FEATURE_WP_UNPOPULATED) != 0;
            }
            if (threadIds != nullptr) {
                *threadIds = (features & UFFD_FEATURE_THREAD_ID) != 0;
            }
            return fd;
        }
        // (a failed handshake leaves the descriptor unusable)
        ::close(fd);
    }
    return -1;
}

bool UffdDirtyTracker::isSupported()
{
    int fd = openUffd();
    if (fd < 0) {
        return false;
    }
    // Registering WP mode on an anonymous page proves kernel support
    void* p = ::mmap(nullptr,
                     HOST_PAGE_SIZE,
                     PROT_READ | PROT_WRITE,
                     MAP_PRIVATE | MAP_ANONYMOUS,
                     -1,
                     0);
    bool ok = false;
    if (p != MAP_FAILED) {
        ((volatile char*)p)[0] = 1;
        uffdio_register reg;
        memset(&reg, 0, sizeof(reg));
        reg.range.start = (uintptr_t)p;
        reg.range.len = HOST_PAGE_SIZE;
        reg.mode = UFFDIO_REGISTER_MODE_WP;
        ok = ::ioctl(fd, UFFDIO_REGISTER, &reg) == 0;
        ::munmap(p, HOST_PAGE_SIZE);
    }
    ::close(fd);
    return ok;
}

UffdDirtyTracker::UffdDirtyTracker(const std::string& modeIn)
  : mode(modeIn)
  , impl(std::make_unique<Impl>())
{
    impl->uffd = openUffd(&impl->wpUnpopulated, &impl->threadIds);
    if (impl->uffd < 0) {
        SPDLOG_ERROR("userfaultfd unavailable: {}", strerror(errno));
        throw std::runtime_error("userfaultfd unavailable");
    }
    if (::pipe(impl->stopPipe) != 0) {
        throw std::runtime_error("pipe failed");
    }
    impl->running.store(true);
    impl->eventThread = std::thread([this] { impl->loop(); });
}

UffdDirtyTracker::~UffdDirtyTracker()
{
    impl->running.store(false);
    char c = 1;
    if (::write(impl->stopPipe[1], &c, 1) != 1) {
        // nothing to do: the poll timeout ends the loop
    }
    if (impl->eventThread.joinable()) {
        impl->eventThread.join();
    }
    ::close(impl->stopPipe[0]);
    ::close(impl->stopPipe[1]);
    ::close(impl->uffd);
}

void UffdDirtyTracker::clearAll()
{
    std::lock_guard<std::mutex> lk(impl->recordMx);
    globalRecords.clear();
    threadRecord.clear();
    impl->perThread.clear();
}

void UffdDirtyTracker::startTracking(std::span<uint8_t> region)
{
    if (region.empty() || region.data() == nullptr) {
        return;
    }
    {
        std::lock_guard<std::mutex> lk(impl->recordMx);
        globalRecords.reset(region);
        impl->tracked = region;
    }
    size_t len = getRequiredHostPages(region.size()) * HOST_PAGE_SIZE;
    uffdio_register reg;
    memset(&reg, 0, sizeof(reg));
    reg.range.start = (uintptr_t)region.data();
    reg.range.len = len;
    reg.mode = UFFDIO_REGISTER_MODE_WP;
    if (::ioctl(impl->uffd, UFFDIO_REGISTER, &reg) != 0) {
        SPDLOG_ERROR("uffd register failed: {}", strerror(errno));
        throw std::runtime_error("uffd register failed");
    }
    if (!impl->wpUnpopulated) {
        // Protection only sticks to pages that have a page-table entry: map
        // the untouched ones (read-only zero pages, nothing is allocated)
        if (::madvise(region.data(), len, MADV_POPULATE_READ) != 0) {
            volatile uint8_t sink = 0;
            for (size_t off = 0; off < len; off += HOST_PAGE_SIZE) {
                sink = sink + region.data()[off];
            }
        }
    }
    uffdio_writeprotect wp;
    wp.range.start = (uintptr_t)region.data();
    wp.range.len = len;
    wp.mode = UFFDIO_WRITEPROTECT_MODE_WP;
    if (::ioctl(impl->uffd, UFFDIO_WRITEPROTECT, &wp) != 0) {
        SPDLOG_ERROR("uffd write-protect failed: {}", strerror(errno));
        throw std::runtime_error("uffd write-protect failed");
    }
}

void UffdDirtyTracker::stopTracking(std::span<uint8_t> region)
{
    if (region.empty() || region.data() == nullptr) {
        return;
    }
    size_t len = getRequiredHostPages(region.size()) * HOST_PAGE_SIZE;
    uffdio_range range;
    range.start = (uintptr_t)region.data();
    range.len = len;
    ::ioctl(impl->uffd, UFFDIO_UNREGISTER, &range);
}

std::vector<char> UffdDirtyTracker::getDirtyPages(std::span<uint8_t> region)
{
    return globalRecords.snapshot(region);
}

// (this thread's record, kept readable after tracking stops)
static thread_local std::shared_ptr<TrackingRecord> uffdThreadRecord;

void UffdDirtyTracker::startThreadLocalTracking(std::span<uint8_t> region)
{
    if (!impl->threadIds || region.empty() || region.data() == nullptr) {
        return;
    }
    auto rec = std::make_shared<TrackingRecord>();
    rec->reset(region);
    uffdThreadRecord = rec;
    std::lock_guard<std::mutex> lk(impl->recordMx);
    impl->perThread[(uint32_t)::syscall(SYS_gettid)] = std::move(rec);
}

void UffdDirtyTracker::stopThreadLocalTracking(std::span<uint8_t> region)
{
    if (!impl->threadIds) {
        return;
    }
    // (a write returns only after the event thread has recorded its fault, so
    // the record is complete here)
    std::lock_guard<std::mutex> lk(impl->recordMx);
    impl->perThread.erase((uint32_t)::syscall(SYS_gettid));
}

std::vector<char> UffdDirtyTracker::getThreadLocalDirtyPages(
  std::span<uint8_t> region)
{
    const size_t want = getRequiredHostPages(region.size());
    if (uffdThreadRecord != nullptr && uffdThreadRecord->regionBase == region.data()) {
        return uffdThreadRecord->snapshot(want);
    }
    // Without thread ids in fault messages attribution is global
    return std::vector<char>(want, 0);
}

std::vector<char> UffdDirtyTracker::getBothDirtyPages(std::span<uint8_t> region)
{
    std::vector<char> g = getDirtyPages(region);
    std::vector<char> t = getThreadLocalDirtyPages(region);
    mergeDirtyPages(g, t);
    return g;
}

// ---------------------------------------------------------------------------
// Device memory
// ---------------------------------------------------------------------------
void DeviceCompareDirtyTracker::getDirtyPagesDevice(const uint8_t* mem,
                                                    const uint8_t* base,
                                                    size_t size,
                                                    uint8_t* pageFlagsDev,
                                                    uint64_t* countDev,
                                                    void* stream)
{
    cudaError_t e = fb::launchDirtyScan(
      mem, base, size, pageFlagsDev, countDev, FB_NUM_SMS * 2, (cudaStream_t)stream);
    if (e != cudaSuccess) {
        throw std::runtime_error(std::string("dirty scan launch failed: ") +
                                 cudaGetErrorString(e));
    }
}

std::vector<char> DeviceCompareDirtyTracker::getDirtyPages(const uint8_t* mem,
                                                           const uint8_t* base,
                                                           size_t size,
                                                           int device,
                                                           void* stream)
{
    size_t nPages = (size + 4095) / 4096;
    std::vector<char> out(nPages, 0);
    if (nPages == 0) {
        return out;
    }
    int prev = -1;
    cudaGetDevice(&prev);
    cudaSetDevice(device);
    uint8_t* flags = nullptr;
    if (cudaMalloc((void**)&flags, nPages) != cudaSuccess) {
        cudaGetLastError();
        throw std::runtime_error("cudaMalloc failed in dirty scan");
    }
    try {
        getDirtyPagesDevice(mem, base, size, flags, nullptr, stream);
    } catch (...) {
        cudaFree(flags);
        throw;
    }
    cudaMemcpyAsync(
      out.data(), flags, nPages, cudaMemcpyDeviceToHost, (cudaStream_t)stream);
    cudaStreamSynchronize((cudaStream_t)stream);
    cudaFree(flags);
    if (prev >= 0) {
        cudaSetDevice(prev);
    }
    return out;
}

} // namespace faabric::util
