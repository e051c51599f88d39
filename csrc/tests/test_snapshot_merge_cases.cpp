// Snapshot merging, host against closed forms and host against device.
//  * [snapshot][merge] (CPU): the typed merge rules of faabric/util/reduce_ops.h
//    one row per case (wrap, division by zero, MIN / -1, NaN, ±0, subnormals,
//    arrays, the image end), and fb_snapshot_prepare_regions against
//    SnapshotData::fillGapsWithBytewiseRegions on seeded random region sets.
//  * [gpu][snapshot]: a seeded differential between the host diff + apply,
//    DeviceSnapshot::diffAndPush and DeviceSnapshot::applyDiffs of the host
//    diffs, which must agree byte for byte; page stamps of syncPagesFrom /
//    pullChangedPages.
#include "fixtures.h"

#include <faabric/device/comm_abi.h>
#include <faabric/device/communicator.h>
#include <faabric/device/cuda_driver.h>
#include <faabric/snapshot/DeviceSnapshot.h>
#include <faabric/util/config.h>
#include <faabric/util/memory.h>
#include <faabric/util/snapshot.h>

#include <cuda_runtime.h>

#include <cmath>
#include <cstring>
#include <limits>
#include <random>

using namespace faabric::util;
using O = SnapshotMergeOperation;
using D = SnapshotDataType;

extern "C" int fb_snapshot_prepare_regions(const FbMergeRegionDev* in,
                                           int nIn,
                                           int fillOp,
                                           uint64_t size,
                                           FbMergeRegionDev* out,
                                           int maxOut,
                                           int32_t* typedOut,
                                           int* nTypedOut);

namespace {
struct Mode
{
    explicit Mode(const std::string& m) { getSystemConfig().diffingMode = m; }
    ~Mode() { getSystemConfig().reset(); }
};

template<typename T>
std::vector<uint8_t> bytesOf(T v)
{
    std::vector<uint8_t> b(sizeof(T));
    memcpy(b.data(), &v, sizeof(T));
    return b;
}

template<typename T>
D typeOf()
{
    if constexpr (std::is_same_v<T, int32_t>) {
        return D::Int;
    } else if constexpr (std::is_same_v<T, long>) {
        return D::Long;
    } else if constexpr (std::is_same_v<T, float>) {
        return D::Float;
    } else {
        return D::Double;
    }
}

// Host diff of one scalar that went old -> new, applied to a main image
// holding cur; the merged bits must be want's (any NaN matches a NaN want)
template<typename T>
void hostRow(O op, T old, T nw, T cur, T want, bool changed = true)
{
    Mode mode("bytewise");
    const size_t size = 2 * HOST_PAGE_SIZE;
    const uint64_t off = HOST_PAGE_SIZE - 2; // across a page, unaligned
    std::vector<uint8_t> base(size, 0), mem(size, 0), main(size, 0);
    memcpy(base.data() + off, &old, sizeof(T));
    memcpy(mem.data() + off, &nw, sizeof(T));
    memcpy(main.data() + off, &cur, sizeof(T));
    SnapshotData snap(base);
    snap.addMergeRegion(off, sizeof(T), typeOf<T>(), op);
    snap.fillGapsWithBytewiseRegions();
    auto diffs = snap.diffWithDirtyRegions(mem, std::vector<char>{ 1, 0 });
    REQUIRE_EQ(diffs.size(), changed ? 1u : 0u);
    SnapshotData target(main);
    target.applyDiffs(diffs);
    T got;
    memcpy(&got, target.getDataPtr(off), sizeof(T));
    if constexpr (std::is_floating_point_v<T>) {
        if (std::isnan(want)) {
            REQUIRE(std::isnan(got));
            return;
        }
    }
    REQUIRE(memcmp(&got, &want, sizeof(T)) == 0);
}
}

TEST_CASE("snapshot merge: integer rows wrap, and Product never divides by zero or traps", "[snapshot][merge]")
{
    const int32_t IMIN = std::numeric_limits<int32_t>::min(), IMAX = std::numeric_limits<int32_t>::max();
    const long LMIN = std::numeric_limits<long>::min(), LMAX = std::numeric_limits<long>::max();
    hostRow<int32_t>(O::Sum, IMIN, IMAX, 5, 4);           // delta MAX - MIN wraps to -1
    hostRow<int32_t>(O::Sum, 0, 1, IMAX, IMIN);
    hostRow<int32_t>(O::Subtract, 1, 0, IMIN, IMAX);
    hostRow<int32_t>(O::Subtract, IMAX, IMIN, 0, 1);      // old - new wraps to -1
    hostRow<int32_t>(O::Product, 1, 2, 1 << 30, IMIN);
    hostRow<int32_t>(O::Product, 0, 7, 9, 0);             // old == 0: factor 0
    hostRow<int32_t>(O::Product, -1, IMIN, 3, IMIN);      // MIN / -1 wraps to MIN
    hostRow<int32_t>(O::Product, 2, -7, 10, -30);         // -7 / 2 truncates to -3
    hostRow<int32_t>(O::Max, 0, -1, IMIN, -1);
    hostRow<int32_t>(O::Min, 0, IMAX, 5, 5);
    hostRow<long>(O::Sum, 0, 1, LMAX, LMIN);
    hostRow<long>(O::Subtract, 1, 0, LMIN, LMAX);
    hostRow<long>(O::Product, 1, 2, 1L << 62, LMIN);
    hostRow<long>(O::Product, 0, -7, 9, 0);
    hostRow<long>(O::Product, -1, LMIN, 1, LMIN);
    hostRow<long>(O::Max, 3, LMIN, LMAX, LMAX);
    hostRow<long>(O::Min, 3, 3, 0, 0, false);             // unchanged: no diff
}

TEST_CASE("snapshot merge: float rows follow IEEE, NaN is ignored by Max/Min, -0 < +0", "[snapshot][merge]")
{
    const float inf = std::numeric_limits<float>::infinity(), nan = std::numeric_limits<float>::quiet_NaN();
    const double dinf = std::numeric_limits<double>::infinity(), dnan = std::numeric_limits<double>::quiet_NaN();
    const float sub = std::numeric_limits<float>::denorm_min();
    hostRow<float>(O::Product, 0.0f, 3.0f, 2.0f, inf);    // new / 0
    hostRow<float>(O::Product, -0.0f, 3.0f, 2.0f, -inf);
    hostRow<float>(O::Product, 0.0f, 3.0f, 0.0f, nan);    // 0 * inf
    hostRow<double>(O::Product, 0.0, -3.0, 2.0, -dinf);
    hostRow<float>(O::Product, 0.0f, -0.0f, 2.0f, 2.0f, false); // ±0 is no change
    hostRow<float>(O::Sum, 0.0f, sub, sub, 2 * sub);      // subnormal delta kept
    hostRow<float>(O::Subtract, 3 * sub, sub, 5 * sub, 3 * sub);
    hostRow<double>(O::Sum, 0.0, 5e-324, 5e-324, 1e-323);
    hostRow<float>(O::Sum, 0.0f, 0x1p-24f, 1.0f, 1.0f);   // rounds to even
    for (auto op : { O::Max, O::Min }) {
        const bool mx = op == O::Max;
        hostRow<float>(op, 1.0f, nan, 2.0f, 2.0f);        // NaN new value: a change, ignored
        hostRow<float>(op, 1.0f, 3.0f, nan, 3.0f);        // NaN in main: replaced
        hostRow<float>(op, 1.0f, nan, nan, nan);
        hostRow<float>(op, nan, 5.0f, 4.0f, mx ? 5.0f : 4.0f);
        hostRow<float>(op, 1.0f, 0.0f, -0.0f, mx ? 0.0f : -0.0f);
        hostRow<float>(op, 1.0f, -0.0f, 0.0f, mx ? 0.0f : -0.0f);
        hostRow<float>(op, 0.0f, -0.0f, 7.0f, 7.0f, false);
        float snan;
        const uint32_t snanBits = 0x7f800001;
        memcpy(&snan, &snanBits, 4);
        hostRow<float>(op, 1.0f, snan, 2.0f, 2.0f);        // a signalling NaN is ignored too
        hostRow<float>(op, 1.0f, 3.0f, snan, 3.0f);
        hostRow<double>(op, 1.0, dnan, 2.0, 2.0);
        hostRow<double>(op, 1.0, 0.0, -0.0, mx ? 0.0 : -0.0);
        hostRow<double>(op, 1.0, -0.0, 0.0, mx ? 0.0 : -0.0);
    }
}

TEST_CASE("snapshot merge: typed arrays diff every scalar and stop at the image end", "[snapshot][merge]")
{
    Mode mode("bytewise");
    const size_t size = HOST_PAGE_SIZE - 1;
    std::vector<uint8_t> base(size, 0);
    for (int k = 0; k < 5; k++) {
        int32_t v = k + 1;
        memcpy(base.data() + 100 + 4 * k, &v, 4);
    }
    std::vector<uint8_t> mem = base;
    for (int k : { 1, 3 }) {
        int32_t v = 10 * (k + 1);
        memcpy(mem.data() + 100 + 4 * k, &v, 4);
    }
    mem[120] = 0xff; // trailing bytes of the array region: not a scalar
    long last = 7;
    memcpy(mem.data() + size - 11, &last, 8);
    mem[size - 1] = 9; // the second Long would pass the image end
    SnapshotData snap(base);
    snap.addMergeRegion(100, 22, D::Int, O::Sum);
    snap.addMergeRegion(size - 11, 16, D::Long, O::Sum);
    snap.fillGapsWithBytewiseRegions();
    std::vector<uint8_t> scratch = mem;
    auto diffs = snap.diffWithDirtyRegions(scratch, std::vector<char>{ 1 });
    REQUIRE_EQ(diffs.size(), 3u);
    REQUIRE_EQ(diffs[0].getOffset(), 104u);
    REQUIRE_EQ(diffs[1].getOffset(), 112u);
    REQUIRE_EQ(diffs[2].getOffset(), size - 11);
    for (const auto& d : diffs) {
        REQUIRE_EQ(d.getData().size(), d.getDataType() == D::Int ? 4u : 8u);
    }
    SnapshotData main(base);
    main.applyDiffs(diffs);
    auto got = main.getDataCopy();
    std::vector<int32_t> arr(5);
    memcpy(arr.data(), got.data() + 100, 20);
    REQUIRE(arr == (std::vector<int32_t>{ 1, 20, 3, 40, 5 }));
    REQUIRE_EQ((int)got[120], 0);
    REQUIRE_EQ((int)got[size - 1], 0);
    memcpy(&last, got.data() + size - 11, 8);
    REQUIRE_EQ(last, 7L);

    // a typed diff of L bytes applies floor(L / size) scalars, cut at the image end
    std::vector<uint8_t> payload(14, 0);
    int32_t three[3] = { 10, 20, 30 };
    memcpy(payload.data(), three, 12);
    payload[12] = 0x55;
    std::vector<uint8_t> tail = bytesOf<long>(5);
    auto tail2 = bytesOf<long>(6);
    tail.insert(tail.end(), tail2.begin(), tail2.end());
    SnapshotData m2(base);
    m2.applyDiffs({ SnapshotDiff(D::Int, O::Sum, 100, payload), SnapshotDiff(D::Long, O::Sum, size - 8, tail) });
    auto got2 = m2.getDataCopy();
    memcpy(arr.data(), got2.data() + 100, 20);
    REQUIRE(arr == (std::vector<int32_t>{ 11, 22, 33, 4, 5 }));
    long lv;
    memcpy(&lv, got2.data() + size - 8, 8);
    REQUIRE_EQ(lv, 5L);
    REQUIRE_EQ(m2.getSize(), size);
}

TEST_CASE("snapshot merge: device gap filling agrees with the host on random region sets", "[snapshot][merge]")
{
    std::mt19937_64 rng(20261015);
    const D types[] = { D::Raw, D::Int, D::Long, D::Float, D::Double };
    int rejected = 0;
    for (int iter = 0; iter < 400; iter++) {
        const bool xorMode = iter % 2 == 1;
        Mode mode(xorMode ? "xor" : "bytewise");
        const size_t size = 1 + rng() % (6 * HOST_PAGE_SIZE);
        const int n = (int)(rng() % 7);
        std::vector<FbMergeRegionDev> in;
        SnapshotData snap(size);
        for (int i = 0; i < n; i++) {
            uint64_t off = rng() % (size + 64);
            uint64_t len = rng() % 6 == 0 ? 0 : 1 + rng() % 600;
            D dt = types[rng() % 5];
            O op = dt == D::Raw ? (rng() % 2 ? O::Ignore : O::Bytewise) : (O)(1 + rng() % 5);
            in.push_back({ off, len, (int32_t)dt, (int32_t)op });
            snap.addMergeRegion(off, len, dt, op);
        }
        std::vector<FbMergeRegionDev> out(2 * n + 2);
        std::vector<int32_t> typed(2 * n + 2);
        int nTyped = -1;
        int got = fb_snapshot_prepare_regions(in.data(), n, xorMode ? (int)O::XOR : (int)O::Bytewise, size, out.data(), (int)out.size(), typed.data(), &nTyped);
        bool hostThrew = false;
        try {
            snap.fillGapsWithBytewiseRegions();
        } catch (std::runtime_error&) {
            hostThrew = true;
        }
        REQUIRE_EQ(hostThrew, got == FB_E_INVALID);
        if (hostThrew) {
            rejected++;
            continue;
        }
        auto want = snap.getMergeRegions();
        REQUIRE_EQ((size_t)got, want.size());
        std::vector<int32_t> wantTyped;
        for (int i = 0; i < got; i++) {
            REQUIRE_EQ(out[i].offset, want[i].offset);
            REQUIRE_EQ(out[i].length, want[i].length);
            REQUIRE_EQ(out[i].dataType, (int32_t)want[i].dataType);
            REQUIRE_EQ(out[i].op, (int32_t)want[i].operation);
            O op = want[i].operation;
            if (op != O::Bytewise && op != O::XOR && op != O::Ignore) {
                wantTyped.push_back(i);
            }
        }
        REQUIRE(std::vector<int32_t>(typed.begin(), typed.begin() + nTyped) == wantTyped);
    }
    // both outcomes were exercised
    printf("         %d of 400 region sets rejected\n", rejected);
    REQUIRE(rejected > 50);
    REQUIRE(rejected < 350);
}

// ===========================================================================
// GPU: host diff + apply == device diff-push == device apply of host diffs
// ===========================================================================
namespace {
struct TypedSpan
{
    uint64_t off;
    uint32_t sz;
    bool isFloat;
};

void putValue(std::vector<uint8_t>& buf, uint64_t off, D dt, std::mt19937_64& rng)
{
    static const uint32_t f32[] = { 0x7fc00000, 0x7f800001, 0xffc12345, 0x00000000, 0x80000000, 0x7f800000,
                                    0xff800000, 0x00000001, 0x807fffff, 0x7f7fffff, 0x3f800000, 0x33800000,
                                    0x40400000, 0xbf800000, 0x3dcccccd };
    static const uint64_t f64[] = { 0x7ff8000000000000, 0x7ff0000000000001, 0xfff8deadbeef0000, 0x0, 0x8000000000000000,
                                    0x7ff0000000000000, 0xfff0000000000000, 0x1, 0x800fffffffffffff, 0x7fefffffffffffff,
                                    0x3ff0000000000000, 0x3ca0000000000000, 0x4008000000000000, 0xbff0000000000000 };
    static const int32_t i32[] = { std::numeric_limits<int32_t>::min(), std::numeric_limits<int32_t>::max(), -1, 0, 1, 2, -2, 7 };
    static const int64_t i64[] = { std::numeric_limits<int64_t>::min(), std::numeric_limits<int64_t>::max(), -1, 0, 1, 2, -2, 1L << 40 };
    size_t sz = (dt == D::Int || dt == D::Float) ? 4 : 8;
    if (off + sz > buf.size()) {
        return;
    }
    switch (dt) {
        case D::Int:
            memcpy(buf.data() + off, &i32[rng() % 8], 4);
            break;
        case D::Long:
            memcpy(buf.data() + off, &i64[rng() % 8], 8);
            break;
        case D::Float:
            memcpy(buf.data() + off, &f32[rng() % 15], 4);
            break;
        default:
            memcpy(buf.data() + off, &f64[rng() % 14], 8);
            break;
    }
}

size_t mismatchCount(const std::vector<uint8_t>& got, const std::vector<uint8_t>& want, const std::vector<TypedSpan>& spans, const char* what)
{
    std::vector<char> nanOk(got.size(), 0);
    for (const auto& s : spans) {
        if (!s.isFloat || s.off + s.sz > got.size()) {
            continue;
        }
        bool a, b;
        if (s.sz == 4) {
            float x, y;
            memcpy(&x, got.data() + s.off, 4);
            memcpy(&y, want.data() + s.off, 4);
            a = std::isnan(x), b = std::isnan(y);
        } else {
            double x, y;
            memcpy(&x, got.data() + s.off, 8);
            memcpy(&y, want.data() + s.off, 8);
            a = std::isnan(x), b = std::isnan(y);
        }
        if (a && b) {
            memset(nanOk.data() + s.off, 1, s.sz);
        }
    }
    size_t bad = 0;
    for (size_t i = 0; i < got.size(); i++) {
        if (got[i] != want[i] && !nanOk[i]) {
            if (bad < 4) {
                printf("         %s: byte %zu is %d, want %d\n", what, i, got[i], want[i]);
            }
            bad++;
        }
    }
    return bad;
}
}

TEST_CASE("gpu: host and device snapshot merges agree byte for byte on seeded images", "[gpu][snapshot]")
{
    if (!faabric::device::cudaAvailable()) {
        SKIP_TEST("no CUDA device");
    }
    cudaSetDevice(0);
    const size_t P = HOST_PAGE_SIZE;
    const D typedTypes[] = { D::Int, D::Long, D::Float, D::Double };
    const O typedOps[] = { O::Sum, O::Subtract, O::Product, O::Max, O::Min };
    int run = 0;
    for (size_t size : { (size_t)1, (size_t)4095, P, 33 * P + 777, (size_t)(16u << 20) + 5 }) {
        const size_t nPages = (size + P - 1) / P;
        for (const char* fill : { "bytewise", "xor" }) {
            for (int dirtyMode = 0; dirtyMode < 4; dirtyMode++) { // all, none, random, odd pages only
                for (bool updateBase : { false, true }) {
                    if (size > (1u << 20) && (dirtyMode == 1 || updateBase != (dirtyMode == 2))) {
                        continue; // the 16 MiB image: two combinations are enough
                    }
                    Mode mode(fill);
                    std::mt19937_64 rng(1000 * run++ + size);
                    std::vector<uint8_t> base(size);
                    for (auto& b : base) {
                        b = (uint8_t)rng();
                    }
                    std::vector<uint8_t> mem = base;
                    const size_t nEdits = 1 + size / 500;
                    for (size_t e = 0; e < nEdits; e++) {
                        mem[rng() % size] ^= (uint8_t)(1 + rng() % 255);
                    }
                    // typed regions at every placement, walking through the image
                    std::vector<SnapshotMergeRegion> regions;
                    std::vector<TypedSpan> spans;
                    uint64_t cursor = rng() % 64;
                    const uint64_t maxGap = std::max<uint64_t>(64, size / 120);
                    int k = 0;
                    while (cursor < size) {
                        D dt = typedTypes[k % 4];
                        O op = typedOps[(k / 4) % 5];
                        const uint32_t sz = (dt == D::Int || dt == D::Float) ? 4 : 8;
                        uint64_t off = cursor;
                        uint64_t len = sz;
                        switch (rng() % 8) {
                            case 0: // naturally aligned
                                off = (cursor + sz - 1) / sz * sz;
                                break;
                            case 1: // unaligned inside a 16-byte block
                                off = (cursor + 15) / 16 * 16 + (sz == 4 ? 3 : 5);
                                break;
                            case 2: // across a 16-byte boundary
                                off = (cursor + 15) / 16 * 16 + 14;
                                break;
                            case 3: // across a page
                                off = (cursor + P - 1) / P * P + P - 2;
                                break;
                            case 4: // an array, with trailing bytes
                                len = sz * (1 + rng() % 40) + rng() % sz;
                                break;
                            case 5: // Ignore
                                dt = D::Raw;
                                op = O::Ignore;
                                len = 1 + rng() % 200;
                                break;
                            case 6: // the last whole scalar, or one that does not fit
                                off = size >= sz ? size - sz - (rng() % 2) * (rng() % sz) : cursor;
                                off = std::max(off, cursor);
                                len = rng() % 2 ? sz : 0;
                                break;
                            default: // right after the previous region
                                break;
                        }
                        if (off >= size) {
                            break;
                        }
                        regions.emplace_back(off, len, dt, op);
                        if (dt != D::Raw) {
                            const uint64_t end = len == 0 ? size : std::min<uint64_t>(size, off + len);
                            for (uint64_t s = off; s + sz <= end; s += sz) {
                                putValue(base, s, dt, rng);
                                if (rng() % 5 == 0) {
                                    memcpy(mem.data() + s, base.data() + s, sz);
                                } else {
                                    putValue(mem, s, dt, rng);
                                }
                                spans.push_back({ s, sz, dt == D::Float || dt == D::Double });
                            }
                            // a byte edit next to the scalar, in the same 16-byte vector
                            if (off > 0 && rng() % 2) {
                                mem[off - 1] ^= 0x41;
                            }
                        }
                        if (len == 0) {
                            break;
                        }
                        cursor = off + len + (rng() % 3 == 0 ? 0 : rng() % maxGap);
                        k++;
                    }
                    // main image: another writer changed it already
                    std::vector<uint8_t> mainStart = base;
                    for (size_t e = 0; e < nEdits; e++) {
                        mainStart[rng() % size] ^= 0xff;
                    }
                    for (const auto& s : spans) {
                        if (rng() % 2) {
                            putValue(mainStart, s.off, s.sz == 4 ? (s.isFloat ? D::Float : D::Int) : (s.isFloat ? D::Double : D::Long), rng);
                        }
                    }
                    std::vector<char> dirty(nPages, 1);
                    for (size_t p = 0; p < nPages; p++) {
                        dirty[p] = dirtyMode == 0 ? 1 : dirtyMode == 1 ? 0 : dirtyMode == 2 ? (char)(rng() % 2) : (char)(p % 2);
                    }

                    // 1. host: diff on a scratch copy, apply onto main
                    SnapshotData hostSnap(base);
                    for (const auto& r : regions) {
                        hostSnap.addMergeRegion(r.offset, r.length, r.dataType, r.operation);
                    }
                    hostSnap.fillGapsWithBytewiseRegions();
                    std::vector<uint8_t> scratch = mem;
                    auto diffs = hostSnap.diffWithDirtyRegions(scratch, dirty);
                    SnapshotData hostMain(mainStart);
                    hostMain.applyDiffs(diffs);
                    auto expected = hostMain.getDataCopy();
                    // the host's view of the new memory, and the counters the device reports
                    std::vector<uint8_t> newBase = base;
                    uint64_t diffBytes = 0;
                    std::vector<char> pageHasDiff(nPages, 0);
                    for (const auto& d : diffs) {
                        const uint64_t o = d.getOffset();
                        const size_t n = d.getData().size();
                        memcpy(newBase.data() + o, mem.data() + o, n);
                        if (d.getOperation() == O::XOR) {
                            for (size_t i = 0; i < n; i++) {
                                if (base[o + i] != mem[o + i]) {
                                    diffBytes++;
                                    pageHasDiff[(o + i) / P] = 1;
                                }
                            }
                        } else {
                            diffBytes += n;
                            pageHasDiff[o / P] = 1;
                        }
                    }
                    const uint64_t pagesWithDiffs = std::count(pageHasDiff.begin(), pageHasDiff.end(), 1);

                    // 2. device: fused diff + merge + push
                    faabric::snapshot::DeviceSnapshot devSnap(size, 0);
                    devSnap.copyInData(base);
                    for (const auto& r : regions) {
                        devSnap.addMergeRegion(r.offset, r.length, r.dataType, r.operation);
                    }
                    faabric::snapshot::DeviceSnapshot devMain(size, 0);
                    devMain.copyInData(mainStart);
                    auto memDev = allocateDeviceMemory(size, 0);
                    auto dirtyDev = allocateDeviceMemory(nPages, 0);
                    cudaMemcpy(memDev.ptr, mem.data(), size, cudaMemcpyHostToDevice);
                    cudaMemcpy(dirtyDev.ptr, dirty.data(), nPages, cudaMemcpyHostToDevice);
                    devSnap.diffAndPush(memDev.ptr, size, devMain.getDevicePtr(), dirtyMode == 0 ? nullptr : dirtyDev.ptr, updateBase, nullptr);
                    auto stats = devSnap.getLastStats(nullptr);
                    REQUIRE_EQ(mismatchCount(devMain.getDataCopy(), expected, spans, "diffAndPush"), 0u);
                    REQUIRE_EQ(stats.diffBytes, diffBytes);
                    REQUIRE_EQ(stats.pagesWithDiffs, pagesWithDiffs);
                    REQUIRE(devSnap.getDataCopy() == (updateBase ? newBase : base));

                    // 3. device: apply the host's diffs
                    faabric::snapshot::DeviceSnapshot devMain2(size, 0);
                    devMain2.copyInData(mainStart);
                    devMain2.applyDiffs(diffs, nullptr);
                    REQUIRE_EQ(mismatchCount(devMain2.getDataCopy(), expected, spans, "applyDiffs"), 0u);
                }
            }
        }
    }
}

TEST_CASE("gpu: page stamps mark exactly the changed pages and pulls copy exactly the later ones", "[gpu][snapshot]")
{
    if (!faabric::device::cudaAvailable()) {
        SKIP_TEST("no CUDA device");
    }
    cudaSetDevice(0);
    const size_t P = HOST_PAGE_SIZE;
    for (size_t n : { 37 * P + 123, 5 * P + 7, (size_t)100 }) {
        const size_t nPages = (n + P - 1) / P;
        std::mt19937_64 rng(n);
        std::vector<uint8_t> a(n);
        for (auto& b : a) {
            b = (uint8_t)rng();
        }
        faabric::snapshot::DeviceSnapshot img(n, 0);
        img.copyInData(a);
        auto stampsOf = [&]() {
            std::vector<uint32_t> s(nPages);
            cudaMemcpy(s.data(), img.pageStamps(), nPages * 4, cudaMemcpyDeviceToHost);
            return s;
        };
        REQUIRE(stampsOf() == std::vector<uint32_t>(nPages, 0));
        img.takePageCopyCount(0);
        auto memDev = allocateDeviceMemory(n, 0);
        // two syncs, stamped 4 and 6, each changing its own set of pages (the
        // partial last page in the second)
        std::vector<uint8_t> cur = a;
        std::vector<uint32_t> wantStamps(nPages, 0);
        for (uint32_t stamp : { 4u, 6u }) {
            std::vector<size_t> pages;
            for (size_t p = 0; p < nPages; p++) {
                if ((p + stamp) % 3 == 0 || (stamp == 6 && p == nPages - 1)) {
                    pages.push_back(p);
                }
            }
            for (size_t p : pages) {
                size_t at = std::min(n - 1, p * P + rng() % P);
                cur[at] ^= 0x80;
                wantStamps[p] = stamp;
            }
            cudaMemcpy(memDev.ptr, cur.data(), n, cudaMemcpyHostToDevice);
            img.syncPagesFrom(memDev.ptr, n, stamp, nullptr);
            REQUIRE_EQ(img.takePageCopyCount(0, nullptr), (uint64_t)pages.size());
            REQUIRE(img.getDataCopy() == cur);
            REQUIRE(stampsOf() == wantStamps);
        }
        // pulls into stale copies of `a`
        auto d1 = allocateDeviceMemory(n, 0);
        auto d2 = allocateDeviceMemory(n, 0);
        for (uint32_t since : { 0u, 4u, 5u, 6u }) {
            for (bool both : { false, true }) {
                cudaMemcpy(d1.ptr, a.data(), n, cudaMemcpyHostToDevice);
                cudaMemcpy(d2.ptr, a.data(), n, cudaMemcpyHostToDevice);
                img.pullChangedPages(d1.ptr, both ? d2.ptr : nullptr, since, n, 0, nullptr);
                std::vector<uint8_t> want = a;
                uint64_t pulled = 0;
                for (size_t p = 0; p < nPages; p++) {
                    if (wantStamps[p] > since) { // a page stamped `since` itself is not pulled
                        size_t e = std::min(n, (p + 1) * P);
                        memcpy(want.data() + p * P, cur.data() + p * P, e - p * P);
                        pulled++;
                    }
                }
                REQUIRE_EQ(img.takePageCopyCount(0, nullptr), pulled);
                std::vector<uint8_t> g1(n), g2(n);
                cudaMemcpy(g1.data(), d1.ptr, n, cudaMemcpyDeviceToHost);
                cudaMemcpy(g2.data(), d2.ptr, n, cudaMemcpyDeviceToHost);
                REQUIRE(g1 == want);
                REQUIRE(g2 == (both ? want : a));
            }
        }
    }
}
