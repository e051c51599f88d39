#include <faabric/util/config.h>
#include <faabric/util/logging.h>
#include <faabric/util/reduce_ops.h>
#include <faabric/util/snapshot.h>
#include <faabric/util/timing.h>

#include <algorithm>
#include <cstring>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

namespace faabric::util {

std::string snapshotDataTypeStr(SnapshotDataType dt)
{
    static const char* names[] = { "Raw", "Bool", "Int", "Long", "Float", "Double" };
    int i = (int)dt;
    if (i < 0 || i > 5) {
        SPDLOG_ERROR("Cannot convert snapshot data type to string: {}", i);
        throw std::runtime_error("Cannot convert data type to string");
    }
    return names[i];
}

std::string snapshotMergeOpStr(SnapshotMergeOperation op)
{
    static const char* names[] = { "Bytewise", "Sum",  "Product", "Subtract",
                                   "Max",      "Min",  "Ignore",  "XOR" };
    int i = (int)op;
    if (i < 0 || i > 7) {
        SPDLOG_ERROR("Cannot convert snapshot merge op to string: {}", i);
        throw std::runtime_error("Cannot convert merge op to string");
    }
    return names[i];
}

// ---------------------------------------------------------------------------
// Diff
// ---------------------------------------------------------------------------
SnapshotDiff::SnapshotDiff(SnapshotDataType dataTypeIn,
                           SnapshotMergeOperation operationIn,
                           uint64_t offsetIn,
                           std::span<const uint8_t> dataIn)
  : dataType(dataTypeIn)
  , operation(operationIn)
  , offset(offsetIn)
  , data(dataIn)
{}

std::vector<uint8_t> SnapshotDiff::getDataCopy() const
{
    return std::vector<uint8_t>(data.begin(), data.end());
}

// ---------------------------------------------------------------------------
// Typed values
// ---------------------------------------------------------------------------
// The merge rules are those of faabric/util/reduce_ops.h: integers wrap,
// float Max/Min ignore a NaN operand and order -0 below +0.  "Unchanged" is a
// value comparison, so a NaN always counts as a change and ±0 never does.
template<typename T>
bool calculateDiffValue(const uint8_t* original,
                        uint8_t* updated,
                        SnapshotMergeOperation operation)
{
    T newValue = unalignedRead<T>(updated);
    T oldValue = unalignedRead<T>(original);
    if (newValue == oldValue) {
        return false;
    }
    T toSend = newValue;
    switch (operation) {
        case SnapshotMergeOperation::Sum:
            toSend = reduceSub(newValue, oldValue);
            break;
        case SnapshotMergeOperation::Subtract:
            toSend = reduceSub(oldValue, newValue);
            break;
        case SnapshotMergeOperation::Product:
            toSend = snapshotQuotient(newValue, oldValue);
            break;
        case SnapshotMergeOperation::Max:
        case SnapshotMergeOperation::Min:
            break;
        default:
            SPDLOG_ERROR("Can't calculate diff for operation: {}", (int)operation);
            throw std::runtime_error("Can't calculate diff");
    }
    unalignedWrite<T>(toSend, updated);
    return true;
}

template<typename T>
T applyDiffValue(const uint8_t* original,
                 const uint8_t* diff,
                 SnapshotMergeOperation operation)
{
    T diffValue = unalignedRead<T>(diff);
    T current = unalignedRead<T>(original);
    switch (operation) {
        case SnapshotMergeOperation::Sum:
            return reduceSum(current, diffValue);
        case SnapshotMergeOperation::Subtract:
            return reduceSub(current, diffValue);
        case SnapshotMergeOperation::Product:
            return reduceProd(current, diffValue);
        case SnapshotMergeOperation::Max:
            return reduceMax(current, diffValue);
        case SnapshotMergeOperation::Min:
            return reduceMin(current, diffValue);
        default:
            SPDLOG_ERROR("Can't apply merge operation: {}", (int)operation);
            throw std::runtime_error("Can't apply merge operation");
    }
}

template bool calculateDiffValue<int32_t>(const uint8_t*, uint8_t*, SnapshotMergeOperation);
template bool calculateDiffValue<long>(const uint8_t*, uint8_t*, SnapshotMergeOperation);
template bool calculateDiffValue<float>(const uint8_t*, uint8_t*, SnapshotMergeOperation);
template bool calculateDiffValue<double>(const uint8_t*, uint8_t*, SnapshotMergeOperation);
template int32_t applyDiffValue<int32_t>(const uint8_t*, const uint8_t*, SnapshotMergeOperation);
template long applyDiffValue<long>(const uint8_t*, const uint8_t*, SnapshotMergeOperation);
template float applyDiffValue<float>(const uint8_t*, const uint8_t*, SnapshotMergeOperation);
template double applyDiffValue<double>(const uint8_t*, const uint8_t*, SnapshotMergeOperation);

// ---------------------------------------------------------------------------
// Array comparison
// ---------------------------------------------------------------------------
void diffArrayRegions(std::vector<std::pair<uint64_t, uint64_t>>& diffs,
                      uint64_t startOffset,
                      uint64_t endOffset,
                      std::span<const uint8_t> a,
                      std::span<const uint8_t> b)
{
    const uint8_t* pa = a.data();
    const uint8_t* pb = b.data();
    bool inRun = false;
    uint64_t runStart = 0;

    auto closeRun = [&](uint64_t at) {
        if (inRun) {
            diffs.emplace_back(runStart, at - runStart);
            inRun = false;
        }
    };

    uint64_t pos = startOffset;
    while (pos < endOffset) {
        uint64_t chunkEnd = std::min<uint64_t>(pos + ARRAY_COMP_CHUNK_SIZE, endOffset);
        size_t chunkLen = (size_t)(chunkEnd - pos);
        if (memcmp(pa + pos, pb + pos, chunkLen) == 0) {
            // Whole chunk equal: any open run ends at the chunk boundary
            closeRun(pos);
            pos = chunkEnd;
            continue;
        }
        for (uint64_t i = pos; i < chunkEnd; i++) {
            bool differs = pa[i] != pb[i];
            if (differs && !inRun) {
                inRun = true;
                runStart = i;
            } else if (!differs && inRun) {
                closeRun(i);
            }
        }
        pos = chunkEnd;
    }
    closeRun(endOffset);
}

// ---------------------------------------------------------------------------
// Merge region
// ---------------------------------------------------------------------------
SnapshotMergeRegion::SnapshotMergeRegion(uint64_t offsetIn,
                                         uint64_t lengthIn,
                                         SnapshotDataType dataTypeIn,
                                         SnapshotMergeOperation operationIn)
  : offset(offsetIn)
  , length(lengthIn)
  , dataType(dataTypeIn)
  , operation(operationIn)
{}

void SnapshotMergeRegion::addDiffs(std::vector<SnapshotDiff>& diffs,
                                   std::span<const uint8_t> originalData,
                                   std::span<uint8_t> updatedData,
                                   const std::vector<char>& dirtyRegions)
{
    if (operation == SnapshotMergeOperation::Ignore) {
        return;
    }
    const uint64_t dataEnd = std::min(originalData.size(), updatedData.size());
    if (offset > dataEnd) {
        return; // region lies beyond the image or the memory
    }
    uint64_t regionEnd = length > 0 ? offset + length : dataEnd;
    regionEnd = std::min<uint64_t>(regionEnd, dataEnd);

    size_t firstPage = getRequiredHostPagesRoundDown(offset);
    size_t lastPage = getRequiredHostPages(regionEnd); // exclusive
    lastPage = std::min(lastPage, dirtyRegions.size());
    if (firstPage >= lastPage) {
        return;
    }
    bool anyDirty = std::find(dirtyRegions.begin() + firstPage,
                              dirtyRegions.begin() + lastPage,
                              1) != dirtyRegions.begin() + lastPage;
    if (!anyDirty) {
        return;
    }

    if (operation == SnapshotMergeOperation::Bytewise ||
        operation == SnapshotMergeOperation::XOR) {
        if (dataType != SnapshotDataType::Raw) {
            SPDLOG_ERROR("Merge region for {} {} not supported",
                         snapshotMergeOpStr(operation),
                         snapshotDataTypeStr(dataType));
            throw std::runtime_error("Unsupported merge op combination");
        }
        for (size_t p = firstPage; p < lastPage; p++) {
            if (dirtyRegions[p] == 0) {
                continue;
            }
            uint64_t segStart = std::max<uint64_t>(p * HOST_PAGE_SIZE, offset);
            uint64_t segEnd = std::min<uint64_t>((p + 1) * HOST_PAGE_SIZE, regionEnd);
            if (segStart >= segEnd) {
                continue;
            }
            if (operation == SnapshotMergeOperation::Bytewise) {
                std::vector<std::pair<uint64_t, uint64_t>> runs;
                diffArrayRegions(runs, segStart, segEnd, originalData, updatedData);
                for (const auto& [runOff, runLen] : runs) {
                    diffs.emplace_back(SnapshotDataType::Raw,
                                       SnapshotMergeOperation::Bytewise,
                                       runOff,
                                       updatedData.subspan(runOff, runLen));
                }
            } else {
                // In-place XOR so the diff can point straight at `updated`
                uint8_t* u = updatedData.data() + segStart;
                const uint8_t* o = originalData.data() + segStart;
                size_t n = (size_t)(segEnd - segStart);
                for (size_t i = 0; i < n; i++) {
                    u[i] ^= o[i];
                }
                diffs.emplace_back(SnapshotDataType::Raw,
                                   SnapshotMergeOperation::XOR,
                                   segStart,
                                   updatedData.subspan(segStart, n));
            }
        }
        return;
    }

    // Typed regions are arrays of floor(length / sizeof(T)) scalars, one diff
    // per changed scalar.  A scalar is diffed when its first or its last page
    // is dirty; trailing bytes and a scalar that would pass the end of the
    // data produce nothing.
    uint64_t sz = 0;
    switch (dataType) {
        case SnapshotDataType::Int:
        case SnapshotDataType::Float:
            sz = 4;
            break;
        case SnapshotDataType::Long:
        case SnapshotDataType::Double:
            sz = 8;
            break;
        default:
            SPDLOG_ERROR("Unsupported merge op combination {} {}",
                         snapshotDataTypeStr(dataType),
                         snapshotMergeOpStr(operation));
            throw std::runtime_error("Unsupported merge op combination");
    }
    auto pageDirty = [&](uint64_t byte) {
        size_t p = getRequiredHostPagesRoundDown(byte);
        return p < dirtyRegions.size() && dirtyRegions[p] != 0;
    };
    for (uint64_t off = offset; off + sz <= regionEnd; off += sz) {
        if (!pageDirty(off) && !pageDirty(off + sz - 1)) {
            continue;
        }
        uint8_t* updated = updatedData.data() + off;
        const uint8_t* original = originalData.data() + off;
        bool changed = false;
        switch (dataType) {
            case SnapshotDataType::Int:
                changed = calculateDiffValue<int32_t>(original, updated, operation);
                break;
            case SnapshotDataType::Long:
                changed = calculateDiffValue<long>(original, updated, operation);
                break;
            case SnapshotDataType::Float:
                changed = calculateDiffValue<float>(original, updated, operation);
                break;
            default:
                changed = calculateDiffValue<double>(original, updated, operation);
                break;
        }
        if (changed) {
            diffs.emplace_back(dataType, operation, off, std::span<const uint8_t>(updated, (size_t)sz));
        }
    }
}

// ---------------------------------------------------------------------------
// SnapshotData
// ---------------------------------------------------------------------------
SnapshotData::SnapshotData(size_t sizeIn)
{
    init(sizeIn, sizeIn);
}

SnapshotData::SnapshotData(size_t sizeIn, size_t maxSizeIn)
{
    init(sizeIn, maxSizeIn);
}

SnapshotData::SnapshotData(std::span<const uint8_t> dataIn)
{
    init(dataIn.size(), dataIn.size());
    writeData(dataIn);
}

SnapshotData::SnapshotData(std::span<const uint8_t> dataIn, size_t maxSizeIn)
{
    init(dataIn.size(), maxSizeIn);
    writeData(dataIn);
}

void SnapshotData::init(size_t initialSize, size_t maxSizeIn)
{
    size = initialSize;
    maxSize = maxSizeIn == 0 ? initialSize : maxSizeIn;
    if (maxSize < size) {
        maxSize = size;
    }
    if (maxSize == 0) {
        return;
    }
    // Reserve the full range, back the live part with a memfd so it can be
    // CoW-mapped into executors' address spaces
    data = allocateVirtualMemory(maxSize);
    fd = createFd(size, "snap_" + std::to_string((uintptr_t)this));
    if (size > 0) {
        mapMemoryShared({ data.get(), size }, fd);
    }
}

SnapshotData::~SnapshotData()
{
    if (fd > 0) {
        ::close(fd);
        fd = -1;
    }
}

void SnapshotData::checkWriteExtension(std::span<const uint8_t> buffer,
                                       uint64_t offset)
{
    uint64_t regionEnd = offset + buffer.size();
    if (regionEnd > maxSize) {
        SPDLOG_ERROR("Copying snapshot data over max: {} > {}", regionEnd, maxSize);
        throw std::runtime_error("Copying snapshot data over max");
    }
    if (regionEnd > size) {
        size_t newSize = (size_t)regionEnd;
        if (fd <= 0) {
            fd = createFd(0, "snap_" + std::to_string((uintptr_t)this));
        }
        resizeFd(fd, newSize);
        // Re-map the now larger live range onto the reservation
        mapMemoryShared({ data.get(), newSize }, fd);
        size = newSize;
    }
}

void SnapshotData::writeData(std::span<const uint8_t> buffer, uint64_t offset)
{
    if (buffer.empty()) {
        return;
    }
    checkWriteExtension(buffer, offset);
    uint8_t* dst = validatedOffsetPtr(offset);
    ::memcpy(dst, buffer.data(), buffer.size());
    trackedChanges.emplace_back(offset, offset + buffer.size());
}

void SnapshotData::xorData(std::span<const uint8_t> buffer, uint64_t offset)
{
    if (offset + buffer.size() > size) {
        SPDLOG_ERROR("XOR diff beyond snapshot end: {} > {}", offset + buffer.size(), size);
        throw std::runtime_error("XOR diff beyond snapshot end");
    }
    uint8_t* dst = validatedOffsetPtr(offset);
    for (size_t i = 0; i < buffer.size(); i++) {
        dst[i] ^= buffer[i];
    }
    trackedChanges.emplace_back(offset, offset + buffer.size());
}

void SnapshotData::copyInData(std::span<const uint8_t> buffer, uint64_t offset)
{
    FullLock lock(snapMx);
    writeData(buffer, offset);
}

uint8_t* SnapshotData::validatedOffsetPtr(uint64_t offset)
{
    if (offset > size) {
        SPDLOG_ERROR("Out of bounds snapshot access: {} > {}", offset, size);
        throw std::runtime_error("Out of bounds snapshot access");
    }
    return data.get() + offset;
}

const uint8_t* SnapshotData::getDataPtr(uint64_t offset)
{
    SharedLock lock(snapMx);
    return validatedOffsetPtr(offset);
}

std::vector<uint8_t> SnapshotData::getDataCopy()
{
    return getDataCopy(0, size);
}

std::vector<uint8_t> SnapshotData::getDataCopy(uint64_t offset, size_t dataSize)
{
    SharedLock lock(snapMx);
    if (offset + dataSize > size) {
        SPDLOG_ERROR("Out of bounds snapshot copy: {} + {} > {}", offset, dataSize, size);
        throw std::runtime_error("Out of bounds snapshot access");
    }
    const uint8_t* p = validatedOffsetPtr(offset);
    return std::vector<uint8_t>(p, p + dataSize);
}

void SnapshotData::mapToMemory(std::span<uint8_t> target)
{
    PROF_START(MapSnapshot)
    FullLock lock(snapMx);
    if (fd <= 0) {
        SPDLOG_ERROR("Attempting to map memory of non-restorable snapshot");
        throw std::runtime_error("Mapping non-restorable snapshot");
    }
    if (!isPageAligned(target.data())) {
        SPDLOG_ERROR("Mapping snapshot to non page-aligned address");
        throw std::runtime_error("Mapping snapshot to non page-aligned address");
    }
    if (target.size() > size) {
        SPDLOG_ERROR("Mapping target memory larger than snapshot ({} > {})", target.size(), size);
        throw std::runtime_error("Target memory larger than snapshot");
    }
    mapMemoryPrivate(target, fd);
    PROF_END(MapSnapshot)
}

void SnapshotData::addMergeRegion(uint64_t offset,
                                  size_t length,
                                  SnapshotDataType dataType,
                                  SnapshotMergeOperation operation)
{
    FullLock lock(snapMx);
    mergeRegions.emplace_back(offset, length, dataType, operation);
}

void SnapshotData::fillGapsWithBytewiseRegions()
{
    FullLock lock(snapMx);
    const std::string& mode = getSystemConfig().diffingMode;
    SnapshotMergeOperation fillOp;
    if (mode == "xor") {
        fillOp = SnapshotMergeOperation::XOR;
    } else if (mode == "bytewise") {
        fillOp = SnapshotMergeOperation::Bytewise;
    } else {
        SPDLOG_ERROR("Unsupported diffing mode: {}", mode);
        throw std::runtime_error("Unsupported diffing mode");
    }
    if (mergeRegions.empty()) {
        mergeRegions.emplace_back(0, 0, SnapshotDataType::Raw, fillOp);
        return;
    }
    std::sort(mergeRegions.begin(), mergeRegions.end());
    std::vector<SnapshotMergeRegion> filled;
    uint64_t cursor = 0;
    bool reachesEnd = false;
    for (const auto& r : mergeRegions) {
        // Each byte has one merge operation: overlapping regions, or a region
        // after one that runs to the end, are refused
        if (reachesEnd || r.offset < cursor) {
            SPDLOG_ERROR("Merge region at {} (length {}) overlaps another", r.offset, r.length);
            throw std::runtime_error("Overlapping merge regions");
        }
        if (r.offset > cursor) {
            filled.emplace_back(cursor, r.offset - cursor, SnapshotDataType::Raw, fillOp);
        }
        filled.push_back(r);
        if (r.length == 0) {
            reachesEnd = true;
            cursor = size;
        } else {
            cursor = std::max<uint64_t>(cursor, r.offset + r.length);
        }
    }
    if (!reachesEnd && cursor < size) {
        // Trailing gap: zero length means "to the end", which also covers
        // memory that has grown past the snapshot
        filled.emplace_back(cursor, 0, SnapshotDataType::Raw, fillOp);
    }
    mergeRegions = std::move(filled);
}

void SnapshotData::clearMergeRegions()
{
    FullLock lock(snapMx);
    mergeRegions.clear();
}

std::vector<SnapshotMergeRegion> SnapshotData::getMergeRegions()
{
    SharedLock lock(snapMx);
    return mergeRegions;
}

size_t SnapshotData::getQueuedDiffsCount()
{
    SharedLock lock(snapMx);
    return queuedDiffs.size();
}

void SnapshotData::queueDiffs(const std::vector<SnapshotDiff>& diffs)
{
    // The queue owns its payloads: callers (RPC handlers) may free theirs
    FullLock lock(snapMx);
    for (const auto& d : diffs) {
        queuedDiffData.emplace_back(d.getData().begin(), d.getData().end());
        queuedDiffs.emplace_back(d.getDataType(), d.getOperation(), d.getOffset(), queuedDiffData.back());
    }
}

void SnapshotData::applyDiffs(const std::vector<SnapshotDiff>& diffs)
{
    FullLock lock(snapMx);
    for (const auto& d : diffs) {
        applyDiffLocked(d);
    }
}

void SnapshotData::applyDiff(const SnapshotDiff& diff)
{
    FullLock lock(snapMx);
    applyDiffLocked(diff);
}

void SnapshotData::applyDiffLocked(const SnapshotDiff& diff)
{
    if (diff.getOperation() == SnapshotMergeOperation::Ignore) {
        return;
    }
    if (diff.getOperation() == SnapshotMergeOperation::Bytewise) {
        writeData(diff.getData(), diff.getOffset());
        return;
    }
    if (diff.getOperation() == SnapshotMergeOperation::XOR) {
        xorData(diff.getData(), diff.getOffset());
        return;
    }
    // A typed diff of L bytes holds floor(L / sizeof(T)) scalars; scalars that
    // would pass the end of the image are not applied
    const uint64_t offset = diff.getOffset();
    uint8_t* current = validatedOffsetPtr(offset);
    const uint8_t* value = diff.getData().data();
    const uint64_t len = std::min<uint64_t>(diff.getData().size(), size - offset);
    auto applyAll = [&]<typename T>() {
        const uint64_t n = len / sizeof(T);
        for (uint64_t k = 0; k < n; k++) {
            T v = applyDiffValue<T>(current + k * sizeof(T), value + k * sizeof(T), diff.getOperation());
            unalignedWrite<T>(v, current + k * sizeof(T));
        }
        if (n > 0) {
            trackedChanges.emplace_back(offset, offset + n * sizeof(T));
        }
    };
    switch (diff.getDataType()) {
        case SnapshotDataType::Int:
            applyAll.template operator()<int32_t>();
            break;
        case SnapshotDataType::Long:
            applyAll.template operator()<long>();
            break;
        case SnapshotDataType::Float:
            applyAll.template operator()<float>();
            break;
        case SnapshotDataType::Double:
            applyAll.template operator()<double>();
            break;
        default:
            SPDLOG_ERROR("Unsupported data type for merge: {} {}",
                         snapshotDataTypeStr(diff.getDataType()),
                         snapshotMergeOpStr(diff.getOperation()));
            throw std::runtime_error("Unsupported merge data type");
    }
}

int SnapshotData::writeQueuedDiffs()
{
    PROF_START(WriteQueuedDiffs)
    FullLock lock(snapMx);
    int n = (int)queuedDiffs.size();
    for (const auto& d : queuedDiffs) {
        applyDiffLocked(d);
    }
    queuedDiffs.clear();
    queuedDiffData.clear();
    PROF_END(WriteQueuedDiffs)
    return n;
}

// ---------------------------------------------------------------------------
// Checkpoint files.  Layout (little endian):
//   char[8] "FBSNAP01" | u64 size | u64 maxSize | u32 nRegions | u32 reserved
//   nRegions x { u64 offset, u64 length, u32 dataType, u32 operation }
//   size bytes of image
// ---------------------------------------------------------------------------
namespace {
constexpr char SNAP_FILE_MAGIC[8] = { 'F', 'B', 'S', 'N', 'A', 'P', '0', '1' };

struct SnapFileHeader
{
    char magic[8];
    uint64_t size;
    uint64_t maxSize;
    uint32_t nRegions;
    uint32_t reserved;
};

struct SnapFileRegion
{
    uint64_t offset;
    uint64_t length;
    uint32_t dataType;
    uint32_t operation;
};

void writeAll(int fd, const void* buf, size_t n, const std::string& path)
{
    const uint8_t* p = (const uint8_t*)buf;
    while (n > 0) {
        ssize_t w = ::write(fd, p, std::min(n, (size_t)1 << 30));
        if (w < 0) {
            if (errno == EINTR) {
                continue;
            }
            throw std::runtime_error("Writing snapshot file " + path + ": " + strerror(errno));
        }
        p += w;
        n -= (size_t)w;
    }
}

void readAll(int fd, void* buf, size_t n, const std::string& path)
{
    uint8_t* p = (uint8_t*)buf;
    while (n > 0) {
        ssize_t r = ::read(fd, p, std::min(n, (size_t)1 << 30));
        if (r < 0 && errno == EINTR) {
            continue;
        }
        if (r <= 0) {
            throw std::runtime_error("Snapshot file " + path + " is truncated or unreadable");
        }
        p += r;
        n -= (size_t)r;
    }
}
}

void SnapshotData::writeToFile(const std::string& path)
{
    // Readers may keep going; writers of the image are excluded
    SharedLock lock(snapMx);
    const std::string tmp = path + ".tmp." + std::to_string(::getpid());
    int out = ::open(tmp.c_str(), O_WRONLY | O_CREAT | O_TRUNC | O_CLOEXEC, 0644);
    if (out < 0) {
        throw std::runtime_error("Cannot create snapshot file " + tmp + ": " + strerror(errno));
    }
    try {
        SnapFileHeader h{};
        memcpy(h.magic, SNAP_FILE_MAGIC, sizeof(h.magic));
        h.size = size;
        h.maxSize = maxSize;
        h.nRegions = (uint32_t)mergeRegions.size();
        writeAll(out, &h, sizeof(h), tmp);
        for (const auto& r : mergeRegions) {
            SnapFileRegion fr{ r.offset, r.length, (uint32_t)r.dataType, (uint32_t)r.operation };
            writeAll(out, &fr, sizeof(fr), tmp);
        }
        if (size > 0) {
            writeAll(out, data.get(), size, tmp);
        }
        if (::fsync(out) != 0) {
            throw std::runtime_error("fsync of " + tmp + " failed: " + strerror(errno));
        }
    } catch (...) {
        ::close(out);
        ::unlink(tmp.c_str());
        throw;
    }
    ::close(out);
    if (::rename(tmp.c_str(), path.c_str()) != 0) {
        std::string why = strerror(errno);
        ::unlink(tmp.c_str());
        throw std::runtime_error("Cannot move snapshot file into place at " + path + ": " + why);
    }
}

std::shared_ptr<SnapshotData> SnapshotData::readFromFile(const std::string& path)
{
    int in = ::open(path.c_str(), O_RDONLY | O_CLOEXEC);
    if (in < 0) {
        throw std::runtime_error("Cannot open snapshot file " + path + ": " + strerror(errno));
    }
    std::shared_ptr<SnapshotData> snap;
    try {
        SnapFileHeader h{};
        readAll(in, &h, sizeof(h), path);
        if (memcmp(h.magic, SNAP_FILE_MAGIC, sizeof(h.magic)) != 0) {
            throw std::runtime_error(path + " is not a snapshot file");
        }
        struct stat st{};
        const uint64_t expect = sizeof(h) + (uint64_t)h.nRegions * sizeof(SnapFileRegion) + h.size;
        if (::fstat(in, &st) != 0 || (uint64_t)st.st_size != expect || h.maxSize < h.size) {
            throw std::runtime_error("Snapshot file " + path + " is truncated or corrupt");
        }
        std::vector<SnapFileRegion> regions(h.nRegions);
        if (h.nRegions > 0) {
            readAll(in, regions.data(), regions.size() * sizeof(SnapFileRegion), path);
        }
        snap = std::make_shared<SnapshotData>((size_t)h.size, (size_t)h.maxSize);
        if (h.size > 0) {
            // straight into the memfd-backed mapping
            readAll(in, snap->data.get(), h.size, path);
        }
        for (const auto& r : regions) {
            snap->addMergeRegion(r.offset, r.length, (SnapshotDataType)r.dataType, (SnapshotMergeOperation)r.operation);
        }
    } catch (...) {
        ::close(in);
        throw;
    }
    ::close(in);
    return snap;
}

void SnapshotData::clearTrackedChanges()
{
    FullLock lock(snapMx);
    trackedChanges.clear();
}

std::vector<SnapshotDiff> SnapshotData::getTrackedChanges()
{
    SharedLock lock(snapMx);
    std::vector<SnapshotDiff> out;
    if (trackedChanges.empty()) {
        return out;
    }
    std::span<const uint8_t> all(data.get(), size);
    out.reserve(trackedChanges.size());
    for (const auto& [start, end] : trackedChanges) {
        out.emplace_back(SnapshotDataType::Raw,
                         SnapshotMergeOperation::Bytewise,
                         start,
                         all.subspan(start, end - start));
    }
    return out;
}

std::vector<SnapshotDiff> SnapshotData::diffWithDirtyRegions(
  std::span<uint8_t> updated,
  const std::vector<char>& dirtyRegions)
{
    PROF_START(DiffWithSnapshot)
    SharedLock lock(snapMx);
    std::vector<SnapshotDiff> diffs;

    // Memory that grew beyond the image is always sent whole
    if (updated.size() > size) {
        diffs.emplace_back(SnapshotDataType::Raw,
                           SnapshotMergeOperation::Bytewise,
                           size,
                           updated.subspan(size));
    }
    bool anyDirty = std::find(dirtyRegions.begin(), dirtyRegions.end(), 1) !=
                    dirtyRegions.end();
    if (!anyDirty) {
        PROF_END(DiffWithSnapshot)
        return diffs;
    }
    if (mergeRegions.empty()) {
        SPDLOG_DEBUG("No merge regions set, thus no diffs");
        PROF_END(DiffWithSnapshot)
        return diffs;
    }
    std::vector<SnapshotMergeRegion> sorted = mergeRegions;
    std::sort(sorted.begin(), sorted.end());
    std::span<const uint8_t> original(data.get(), size);
    for (auto& r : sorted) {
        r.addDiffs(diffs, original, updated, dirtyRegions);
    }
    PROF_END(DiffWithSnapshot)
    return diffs;
}

} // namespace faabric::util
