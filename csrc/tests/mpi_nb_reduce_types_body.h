// One MPI program that checks the non-blocking and persistent reductions on
// every datatype and op, on every kind of buffer, bit for bit against a host
// fold: MPI_Ireduce, MPI_Iscan, MPI_Iexscan, blocking MPI_Exscan,
// MPI_Ireduce_scatter_block and the five persistent reduction inits.  Run by
// test_mpi_nb_reduce_types.cpp.
//
// The types, ops, inputs, folds, buffers and checks are those of
// mpi_device_reduce_body.h.  Every non-blocking call runs in a burst of
// calls on disjoint slices of one buffer pair, each slice with inputs of its
// own, waited for together; every persistent request runs several rounds,
// each with new inputs, so a start that reads stale data or re-runs a plan
// made for other requests computes a wrong result.  Besides the matrix the
// program has cases for the burst key and the plan cache (bursts whose key
// changes, MPI_Startall over requests of several keys in changing orders and
// subsets, more bursts than the plan cache holds) and runs the calls on
// sub-communicators whose order differs from the world's.
//
// Every rank runs every call and collects failures instead of returning at
// the first one, so no peer is left waiting in a collective.
#pragma once

#include "mpi_device_reduce_body.h"

#include <algorithm>
#include <functional>
#include <numeric>

namespace nb_reduce_types {

using namespace mpi_device_reduce;

// The parts of the program; each is one test case
enum class Part
{
    Bursts,
    Persistent,
    CrossKey,
    SubComms
};

struct Options
{
    Part part = Part::Bursts;
    bool cudaMalloc = false; // add the cudaMalloc placement (needs a GPU)
    bool grouped = true;     // FAABRIC_MPI_GROUP_IALLREDUCE is on
    // The GPU runs of the matrix leave out what the loopback runs already
    // check with the same code: undefined pairs (refused before any buffer is
    // looked at) and host buffers.  With `count` set the matrix runs that
    // count only and the sized counts at one root, so the GPU suite stays
    // short.
    bool deviceOnly = false;
    size_t count = 0;
};

// The communicator calls run on: its members (world ranks) in its order and
// this rank's place among them
struct Comm
{
    MPI_Comm comm;
    std::vector<int> members;
    int me;
    bool sub = false;

    int size() const { return (int)members.size(); }
    std::vector<int> first(int n) const { return { members.begin(), members.begin() + n }; }
};

// ------------------------------------------------------------------ calls ----
// The result of a call whose inputs come from a case; false when the call
// leaves this rank's recv as it was
using Want = std::function<bool(const Case&, std::vector<uint8_t>*)>;
// The non-blocking call, or the persistent init, on a send (MPI_IN_PLACE when
// in place) and a recv
using Issue = std::function<int(uint8_t*, uint8_t*, MPI_Request*)>;

struct Call
{
    Case c;           // type, op, count and placement; its seed makes the inputs
    std::string name;
    size_t sendCount; // elements of this rank's input
    size_t recvCount; // elements of this rank's recv
    bool inPlace;     // the input sits in recv and send is MPI_IN_PLACE
    int deviceDelta;  // device collectives per call on device buffers of a pair the kernels take
    int hostDelta;    // ... and of a defined pair they do not take (a host path's device legs)
    Want want;
    Issue issue;
    // the burst key, for the launch count: the call kind and the root
    int kind = 0;
    int root = 0;
};

// The case of round `round`: new inputs every round
inline Case roundCase(const Case& c, int round)
{
    Case r = c;
    r.seed = mix(c.seed ^ ((uint64_t)(round + 1) << 48));
    return r;
}

inline size_t up16(size_t n)
{
    return (n + 15) / 16 * 16;
}

// The launches a list of grouped calls makes: one per run of equal keys
inline int runsOf(const std::vector<Call>& calls, const std::vector<int>& order)
{
    int runs = 0;
    for (size_t i = 0; i < order.size(); i++) {
        const Call& a = calls[order[i]];
        const Call* b = i > 0 ? &calls[order[i - 1]] : nullptr;
        if (b == nullptr || a.kind != b->kind || a.c.t->kind != b->c.t->kind || a.c.opId() != b->c.opId() ||
            a.root != b->root) {
            runs++;
        }
    }
    return runs;
}

// Runs `calls` on disjoint slices of one send and one recv buffer at `place`
// (shifted as for elements of `shiftEs` bytes), with 16 bytes of guard
// between slices.  Without `persistent`, one round issues every call in
// order and waits for all.  With it, every call is initialised once, round r
// starts the calls `rounds[r]` in that order (MPI_Start for one,
// MPI_Startall for more) and waits, and the requests are freed at the end;
// calls not started must leave their recv alone.  Every round writes new
// inputs and guard patterns, then checks return codes, every result, send
// and every byte around the results, the world's device collective count and,
// where `launches` is set, this rank's launch count on `dev`.
inline void runCalls(Ctx& x,
                     std::vector<Call>& calls,
                     Place place,
                     size_t shiftEs,
                     bool persistent,
                     std::vector<std::vector<int>> rounds,
                     const std::vector<int>& launches,
                     faabric::device::Communicator* dev)
{
    const std::string what = calls[0].c.name() + " " + calls[0].name + (calls.size() > 1 ? " (+" + std::to_string(calls.size() - 1) + ")" : "");
    std::vector<size_t> sendOff(calls.size()), recvOff(calls.size());
    size_t sendBytes = 0, recvBytes = 0;
    for (size_t i = 0; i < calls.size(); i++) {
        const size_t es = calls[i].c.esize();
        sendOff[i] = sendBytes;
        recvOff[i] = recvBytes;
        sendBytes += up16(calls[i].sendCount * es) + 16;
        recvBytes += up16(std::max(calls[i].recvCount, calls[i].inPlace ? calls[i].sendCount : 0) * es) + 16;
    }
    Buffer send(place, sendBytes, shiftEs);
    Buffer recv(place, recvBytes, shiftEs);
    if (send.base == nullptr || recv.base == nullptr) {
        x.fail(what + ": allocation failed");
        return;
    }
    auto sendAt = [&](size_t i) { return calls[i].inPlace ? (uint8_t*)MPI_IN_PLACE : send.data + sendOff[i]; };
    std::vector<MPI_Request> reqs(calls.size(), MPI_REQUEST_NULL);
    std::vector<bool> ok(calls.size());
    for (size_t i = 0; i < calls.size(); i++) {
        ok[i] = defined(*calls[i].c.t, calls[i].c.opId());
    }
    auto checkRc = [&](size_t i, int rc) {
        if (rc != (ok[i] ? MPI_SUCCESS : MPI_ERR_OP) || (!ok[i] && reqs[i] != MPI_REQUEST_NULL)) {
            x.fail(calls[i].c.name() + " " + calls[i].name + ": returned " + std::to_string(rc));
        }
    };
    if (persistent) {
        for (size_t i = 0; i < calls.size(); i++) {
            checkRc(i, calls[i].issue(sendAt(i), recv.data + recvOff[i], &reqs[i]));
        }
        if (std::none_of(ok.begin(), ok.end(), [](bool b) { return b; })) {
            rounds.resize(1); // nothing to start: one round checks that nothing is written
        }
    } else {
        rounds.assign(1, {});
    }

    for (size_t round = 0; round < rounds.size(); round++) {
        std::vector<int> order = rounds[round];
        if (!persistent) {
            order.resize(calls.size());
            std::iota(order.begin(), order.end(), 0);
        }
        std::vector<bool> active(calls.size(), false);
        std::vector<Case> cases;
        const Case first = roundCase(calls[0].c, (int)round);
        std::vector<uint8_t> sendImg = guardImage(send.total, first.seed + 1);
        const std::vector<uint8_t> recvBefore = [&] {
            std::vector<uint8_t> img = guardImage(recv.total, first.seed + 2);
            for (size_t i = 0; i < calls.size(); i++) {
                cases.push_back(roundCase(calls[i].c, (int)round));
                const std::vector<uint8_t> in = inputOf(cases[i], x.rank, calls[i].sendCount);
                std::vector<uint8_t>& dst = calls[i].inPlace ? img : sendImg;
                const size_t at = calls[i].inPlace ? recv.dataOff() + recvOff[i] : send.dataOff() + sendOff[i];
                std::copy(in.begin(), in.end(), dst.begin() + (long)at);
            }
            return img;
        }();
        send.setImage(sendImg);
        recv.setImage(recvBefore);

        const uint64_t before = deviceCalls(x);
        const uint64_t l0 = dev != nullptr ? dev->stats().launches : 0;
        if (persistent) {
            std::vector<MPI_Request> started;
            for (int i : order) {
                if (reqs[i] != MPI_REQUEST_NULL) {
                    started.push_back(reqs[i]);
                    active[i] = true;
                }
            }
            if (!started.empty()) {
                const int rc =
                  started.size() == 1 ? MPI_Start(&started[0]) : MPI_Startall((int)started.size(), started.data());
                if (rc != MPI_SUCCESS) {
                    x.fail(what + ": start returned " + std::to_string(rc) + " in round " + std::to_string(round));
                }
                MPI_Waitall((int)started.size(), started.data(), MPI_STATUSES_IGNORE);
            }
        } else {
            for (int i : order) {
                checkRc(i, calls[i].issue(sendAt(i), recv.data + recvOff[i], &reqs[i]));
                active[i] = reqs[i] != MPI_REQUEST_NULL;
            }
            MPI_Waitall((int)reqs.size(), reqs.data(), MPI_STATUSES_IGNORE);
        }
        const uint64_t got = deviceCalls(x) - before;
        const std::string inRound = persistent ? " in round " + std::to_string(round) : "";

        uint64_t expected = 0;
        for (size_t i = 0; i < calls.size(); i++) {
            if (active[i] && place != Place::Host) {
                const bool dev = onDevice(*calls[i].c.t, calls[i].c.opId());
                expected += (uint64_t)(dev ? calls[i].deviceDelta : calls[i].hostDelta) * (uint64_t)x.size;
            }
        }
        if (got != expected) {
            x.fail(what + ": " + std::to_string(got) + " device collectives, expected " + std::to_string(expected) +
                   inRound);
        }
        if (round < launches.size() && launches[round] >= 0 && dev != nullptr) {
            const uint64_t l = dev->stats().launches - l0;
            if (l != (uint64_t)launches[round]) {
                x.fail(what + ": " + std::to_string(l) + " launches, expected " + std::to_string(launches[round]) +
                       inRound);
            }
        }

        checkImage(x, calls[0].c, calls[0].name + " (send)" + inRound, send.image(), sendImg, {}, nullptr);
        // each call's region against its own type; the other calls' regions
        // are compared by their own checks
        const std::vector<uint8_t> image = recv.image();
        std::vector<std::vector<uint8_t>> want(calls.size());
        std::vector<bool> has(calls.size(), false);
        for (size_t i = 0; i < calls.size(); i++) {
            has[i] = active[i] && ok[i] && calls[i].want(cases[i], &want[i]);
        }
        for (size_t i = 0; i < calls.size(); i++) {
            std::vector<uint8_t> others = recvBefore;
            for (size_t j = 0; j < calls.size(); j++) {
                if (j != i && has[j]) {
                    const size_t at = recv.dataOff() + recvOff[j];
                    std::copy(image.begin() + (long)at, image.begin() + (long)(at + want[j].size()),
                              others.begin() + (long)at);
                }
            }
            std::vector<Region> regions;
            if (has[i]) {
                regions.push_back({ recv.dataOff() + recvOff[i], want[i] });
            }
            checkRegions(x, cases[i], calls[i].name + (active[i] ? "" : " (not started)") + inRound, image, others,
                         regions);
        }
    }

    if (persistent) {
        for (size_t i = 0; i < calls.size(); i++) {
            if (reqs[i] != MPI_REQUEST_NULL &&
                (MPI_Request_free(&reqs[i]) != MPI_SUCCESS || reqs[i] != MPI_REQUEST_NULL)) {
                x.fail(calls[i].c.name() + " " + calls[i].name + ": MPI_Request_free failed");
            }
        }
    }
}

// A non-blocking burst of `k` copies of `call`, each slice with inputs of its
// own seed
inline void burst(Ctx& x, const Call& call, int k, Place place)
{
    std::vector<Call> calls(k, call);
    for (int j = 0; j < k; j++) {
        calls[j].c.seed = mix(call.c.seed + 0x100 * (uint64_t)(j + 1));
    }
    runCalls(x, calls, place, call.c.esize(), false, {}, {}, nullptr);
}

// One persistent request: three rounds of MPI_Start + MPI_Wait
inline void persistentRounds(Ctx& x, const Call& call, Place place)
{
    std::vector<Call> calls{ call };
    runCalls(x, calls, place, call.c.esize(), true, { { 0 }, { 0 }, { 0 } }, {}, nullptr);
}

// --------------------------------------------------------------- shapes ----
enum CallKind
{
    ALLREDUCE,
    REDUCE,
    SCAN,
    EXSCAN,
    REDUCE_SCATTER
};

// The smallest block of at least `count` elements that is whole 16-byte vectors
inline size_t wholeVectors(size_t count, size_t es)
{
    size_t b = std::max<size_t>(count, 1);
    while ((b * es) % 16 != 0) {
        b++;
    }
    return b;
}

// One call of `kind` on `cm`, non-blocking or persistent
inline Call reduceCall(const Comm& cm, const Case& c, int kind, bool persistent, int root, bool inPlace, size_t block,
                       size_t stageBytes)
{
    const size_t count = c.count;
    MPI_Datatype dt = c.t->dt;
    MPI_Op op = c.op->op;
    MPI_Comm comm = cm.comm;
    const int n = cm.size();
    const int me = cm.me;
    Call call{ c, "", count, count, inPlace, 1, 0, nullptr, nullptr, kind, root };
    switch (kind) {
        case ALLREDUCE:
            call.name = persistent ? "MPI_Allreduce_init" : "MPI_Iallreduce";
            // a sub-communicator's host all-reduce broadcasts the result
            // over the device
            call.hostDelta = cm.sub && defined(*c.t, c.opId()) ? 1 : 0;
            call.want = [cm, count](const Case& r, std::vector<uint8_t>* w) {
                *w = foldOver(r, cm.members, count);
                return true;
            };
            call.issue = [=](uint8_t* s, uint8_t* d, MPI_Request* q) {
                return persistent ? MPI_Allreduce_init(s, d, (int)count, dt, op, comm, MPI_INFO_NULL, q)
                                  : MPI_Iallreduce(s, d, (int)count, dt, op, comm, q);
            };
            break;
        case REDUCE:
            call.name = std::string(persistent ? "MPI_Reduce_init" : "MPI_Ireduce") + " root " + std::to_string(root) +
                        (inPlace ? " in place" : "");
            call.want = [cm, count, root](const Case& r, std::vector<uint8_t>* w) {
                if (cm.me != root) {
                    return false;
                }
                *w = foldOver(r, cm.members, count);
                return true;
            };
            call.issue = [=](uint8_t* s, uint8_t* d, MPI_Request* q) {
                return persistent ? MPI_Reduce_init(s, d, (int)count, dt, op, root, comm, MPI_INFO_NULL, q)
                                  : MPI_Ireduce(s, d, (int)count, dt, op, root, comm, q);
            };
            break;
        case SCAN:
        case EXSCAN: {
            const bool ex = kind == EXSCAN;
            call.name = std::string(persistent ? (ex ? "MPI_Exscan_init" : "MPI_Scan_init")
                                               : (ex ? "MPI_Iexscan" : "MPI_Iscan")) +
                        (inPlace ? " in place" : "");
            call.want = [cm, count, ex](const Case& r, std::vector<uint8_t>* w) {
                const int upto = ex ? cm.me : cm.me + 1;
                if (upto == 0) {
                    return false; // rank 0's recv of an exscan keeps every byte
                }
                *w = foldOver(r, cm.first(upto), count);
                return true;
            };
            call.issue = [=](uint8_t* s, uint8_t* d, MPI_Request* q) {
                if (persistent) {
                    return ex ? MPI_Exscan_init(s, d, (int)count, dt, op, comm, MPI_INFO_NULL, q)
                              : MPI_Scan_init(s, d, (int)count, dt, op, comm, MPI_INFO_NULL, q);
                }
                return ex ? MPI_Iexscan(s, d, (int)count, dt, op, comm, q) : MPI_Iscan(s, d, (int)count, dt, op, comm, q);
            };
            break;
        }
        default: {
            const size_t es = c.esize();
            call.name = std::string(persistent ? "MPI_Reduce_scatter_block_init" : "MPI_Ireduce_scatter_block") +
                        " block " + std::to_string(block);
            call.sendCount = block * (size_t)n;
            call.recvCount = block;
            // the device takes whole-vector blocks of symmetric, aligned
            // buffers, and otherwise messages the staging area holds
            call.deviceDelta =
              ((block * es) % 16 == 0 && (c.place == Place::Heap || block * es * (size_t)n <= stageBytes)) ? 1 : 0;
            call.want = [cm, block, me](const Case& r, std::vector<uint8_t>* w) {
                const std::vector<uint8_t> full = foldOver(r, cm.members, block * (size_t)cm.size());
                const size_t bytes = block * r.esize();
                *w = slice(full, (size_t)me * bytes, bytes);
                return true;
            };
            call.issue = [=](uint8_t* s, uint8_t* d, MPI_Request* q) {
                return persistent ? MPI_Reduce_scatter_block_init(s, d, (int)block, dt, op, comm, MPI_INFO_NULL, q)
                                  : MPI_Ireduce_scatter_block(s, d, (int)block, dt, op, comm, q);
            };
        }
    }
    return call;
}

// Every non-blocking and blocking call of one case on `cm`, with MPI_Ireduce
// at `roots`: bursts of three
inline void burstCalls(Ctx& x, const Comm& cm, const Case& c, const std::vector<int>& roots, size_t stageBytes)
{
    const int k = 3;
    for (int root : roots) {
        for (bool rootInPlace : { false, true }) {
            burst(x, reduceCall(cm, c, REDUCE, false, root, rootInPlace && cm.me == root, 0, stageBytes), k, c.place);
        }
    }
    for (int kind : { SCAN, EXSCAN }) {
        // not in place, in place on every rank, in place on odd ranks only
        for (int mode = 0; mode < 3; mode++) {
            const bool inPlace = mode == 1 || (mode == 2 && cm.me % 2 == 1);
            burst(x, reduceCall(cm, c, kind, false, 0, inPlace, 0, stageBytes), k, c.place);
        }
    }
    // blocking MPI_Exscan: rank 0's recv keeps every byte
    const std::vector<uint8_t> prefix = foldOver(c, cm.first(std::max(cm.me, 1)), c.count);
    for (bool inPlace : { false, true }) {
        runCall(x, c, inPlace ? "MPI_Exscan in place" : "MPI_Exscan", c.count, c.count, inPlace,
                cm.me == 0 ? nullptr : &prefix, 1, [&](uint8_t* s, uint8_t* r) {
                    return MPI_Exscan(s, r, (int)c.count, c.t->dt, c.op->op, cm.comm);
                });
    }
    const size_t whole = wholeVectors(c.count, c.esize());
    for (size_t block : { c.count, whole }) {
        burst(x, reduceCall(cm, c, REDUCE_SCATTER, false, 0, false, block, stageBytes), k, c.place);
        if (whole == c.count) {
            break;
        }
    }
}

// Every persistent init of one case on `cm`, with MPI_Reduce_init at `roots`
inline void persistentCalls(Ctx& x, const Comm& cm, const Case& c, const std::vector<int>& roots, size_t stageBytes)
{
    persistentRounds(x, reduceCall(cm, c, ALLREDUCE, true, 0, false, 0, stageBytes), c.place);
    for (int root : roots) {
        for (bool rootInPlace : { false, true }) {
            persistentRounds(x, reduceCall(cm, c, REDUCE, true, root, rootInPlace && cm.me == root, 0, stageBytes),
                             c.place);
        }
    }
    for (int kind : { SCAN, EXSCAN }) {
        for (bool inPlace : { false, true }) {
            persistentRounds(x, reduceCall(cm, c, kind, true, 0, inPlace, 0, stageBytes), c.place);
        }
    }
    const size_t whole = wholeVectors(c.count, c.esize());
    for (size_t block : { c.count, whole }) {
        persistentRounds(x, reduceCall(cm, c, REDUCE_SCATTER, true, 0, false, block, stageBytes), c.place);
        if (whole == c.count) {
            break;
        }
    }
}

// ------------------------------------------------------------- cross-key ----
struct Entry
{
    int kind;
    int type; // index into the type table
    int op;   // index into builtinOps()
    int root;
};

// Calls of several keys, one after another
inline std::vector<Call> entryCalls(const Comm& cm,
                                    const std::vector<Type>& types,
                                    const std::vector<Op>& ops,
                                    const std::vector<Entry>& entries,
                                    Place place,
                                    size_t count,
                                    bool persistent,
                                    uint64_t& seed,
                                    size_t stageBytes)
{
    std::vector<Call> calls;
    for (const Entry& e : entries) {
        const Case c{ &types[e.type], &ops[e.op], count, place, mix(seed++) };
        const size_t block = e.kind == REDUCE_SCATTER ? wholeVectors(count, c.esize()) : 0;
        calls.push_back(reduceCall(cm, c, e.kind, persistent, e.root, false, block, stageBytes));
    }
    return calls;
}

inline int typeIndex(const std::vector<Type>& types, MPI_Datatype dt)
{
    for (size_t i = 0; i < types.size(); i++) {
        if (types[i].dt == dt && types[i].per == 1) {
            return (int)i;
        }
    }
    return -1;
}

inline int opIndex(MPI_Op op)
{
    const std::vector<Op> ops = builtinOps();
    for (size_t i = 0; i < ops.size(); i++) {
        if (ops[i].op == op) {
            return (int)i;
        }
    }
    return -1;
}

inline void crossKey(Ctx& x,
                     const Comm& cm,
                     const std::vector<Type>& types,
                     const std::vector<Op>& ops,
                     const std::vector<Place>& places,
                     const Options& o,
                     faabric::device::Communicator* dev,
                     size_t stageBytes)
{
    auto T = [&](MPI_Datatype dt) { return typeIndex(types, dt); };
    const int SUM = opIndex(MPI_SUM), MAX = opIndex(MPI_MAX), MIN = opIndex(MPI_MIN), BXOR = opIndex(MPI_BXOR);
    const int MAXLOC = opIndex(MPI_MAXLOC), MINLOC = opIndex(MPI_MINLOC);
    const int last = cm.size() - 1;
    uint64_t seed = 0xc0ffee;
    // bursts whose key changes: one launch per run of equal keys
    const std::vector<std::vector<Entry>> bursts{
        { { ALLREDUCE, T(MPI_INT), SUM, 0 }, { ALLREDUCE, T(MPI_DOUBLE), MAX, 0 }, { ALLREDUCE, T(MPI_INT), SUM, 0 } },
        // only the datatype changes
        { { ALLREDUCE, T(MPI_INT), SUM, 0 },
          { ALLREDUCE, T(MPI_FLOAT), SUM, 0 },
          { ALLREDUCE, T(MPI_INT8_T), SUM, 0 },
          { ALLREDUCE, T(MPI_INT64_T), SUM, 0 },
          { ALLREDUCE, T(MPI_INT64_T), SUM, 0 } },
        { { ALLREDUCE, T(MPI_DOUBLE_INT), MAXLOC, 0 },
          { ALLREDUCE, T(MPI_2INT), MAXLOC, 0 },
          { ALLREDUCE, T(MPI_2INT), MINLOC, 0 },
          { ALLREDUCE, T(MPI_DOUBLE_INT), MAXLOC, 0 } },
        // the op changes halfway
        { { REDUCE, T(MPI_INT), SUM, last },
          { REDUCE, T(MPI_INT), SUM, last },
          { REDUCE, T(MPI_INT), MAX, last },
          { REDUCE, T(MPI_INT), MAX, last } },
        { { REDUCE, T(MPI_HALF), SUM, 0 }, { REDUCE, T(MPI_FLOAT), SUM, 0 }, { REDUCE, T(MPI_LONG_INT), MINLOC, 0 } },
        // the root changes, then the kind
        { { REDUCE, T(MPI_UINT16_T), BXOR, 0 },
          { REDUCE, T(MPI_UINT16_T), BXOR, last },
          { SCAN, T(MPI_UINT16_T), BXOR, 0 },
          { SCAN, T(MPI_UINT16_T), BXOR, 0 },
          { EXSCAN, T(MPI_UINT16_T), BXOR, 0 },
          { ALLREDUCE, T(MPI_UINT16_T), BXOR, 0 } },
    };
    for (Place p : places) {
        for (size_t count : { (size_t)1, (size_t)7 }) {
            for (const auto& entries : bursts) {
                std::vector<Call> calls = entryCalls(cm, types, ops, entries, p, count, false, seed, stageBytes);
                std::vector<int> order(calls.size());
                std::iota(order.begin(), order.end(), 0);
                const int launches = p == Place::Heap ? (o.grouped ? runsOf(calls, order) : (int)calls.size()) : -1;
                runCalls(x, calls, p, 8, false, {}, { launches }, dev);
            }

            // MPI_Startall over requests of several keys: in order, reversed,
            // two subsets, in order again
            const std::vector<Entry> mixed{
                { ALLREDUCE, T(MPI_INT), SUM, 0 },        { ALLREDUCE, T(MPI_INT), SUM, 0 },
                { ALLREDUCE, T(MPI_DOUBLE), MAX, 0 },     { REDUCE, T(MPI_FLOAT), SUM, last },
                { SCAN, T(MPI_INT64_T), BXOR, 0 },        { ALLREDUCE, T(MPI_DOUBLE_INT), MAXLOC, 0 },
                { EXSCAN, T(MPI_HALF), MIN, 0 },          { REDUCE_SCATTER, T(MPI_INT), SUM, 0 },
                { REDUCE, T(MPI_2INT), MINLOC, 0 },       { ALLREDUCE, T(MPI_INT), SUM, 0 },
            };
            std::vector<Call> calls = entryCalls(cm, types, ops, mixed, p, count, true, seed, stageBytes);
            std::vector<int> all(calls.size());
            std::iota(all.begin(), all.end(), 0);
            std::vector<int> reversed(all.rbegin(), all.rend());
            const std::vector<std::vector<int>> rounds{ all, reversed, { 1, 5, 8 }, { 0, 9, 2 }, { 1 }, all };
            std::vector<int> launches;
            for (const auto& r : rounds) {
                launches.push_back(p == Place::Heap ? (o.grouped ? runsOf(calls, r) : (int)r.size()) : -1);
            }
            runCalls(x, calls, p, 8, true, rounds, launches, dev);
        }
    }

    // more bursts of persistent starts than the plan cache holds, then the
    // first (evicted) bursts again and the last (cached) one
    const int bursts2 = 70;
    const std::vector<Entry> keys{ { ALLREDUCE, T(MPI_INT), SUM, 0 },
                                   { ALLREDUCE, T(MPI_DOUBLE), MAX, 0 },
                                   { ALLREDUCE, T(MPI_INT8_T), BXOR, 0 } };
    std::vector<Entry> entries;
    for (int b = 0; b < bursts2; b++) {
        entries.push_back(keys[b % keys.size()]);
        entries.push_back(keys[b % keys.size()]);
    }
    std::vector<Call> calls = entryCalls(cm, types, ops, entries, Place::Heap, 7, true, seed, stageBytes);
    std::vector<std::vector<int>> rounds;
    for (int b = 0; b < bursts2; b++) {
        rounds.push_back({ 2 * b, 2 * b + 1 });
    }
    for (int b : { 0, 1, 2, 3, 4, bursts2 - 1 }) {
        rounds.push_back({ 2 * b, 2 * b + 1 });
    }
    // (with grouping off every start is a launch of its own)
    runCalls(x, calls, Place::Heap, 8, true, rounds, std::vector<int>(rounds.size(), o.grouped ? 1 : 2), dev);
}

// --------------------------------------------------------------- program ----
inline std::vector<int> everyRoot(int n)
{
    std::vector<int> r(n);
    std::iota(r.begin(), r.end(), 0);
    return r;
}

// Returns 0, or 1 with the first failures in `why`
inline int body(int rank, int size, int worldId, const Options& o, std::string* why)
{
    Ctx x{ rank, size, &faabric::mpi::getMpiWorldRegistry().getWorld(worldId), {} };
    auto comm = x.world->getDeviceComm(rank);
    if (comm == nullptr) {
        *why = "rank " + std::to_string(rank) + ": no device communicator";
        return 1;
    }
    const auto& cfg = comm->config();
    std::vector<Place> places{ Place::Heap, Place::HeapShift, Place::Host };
    if (o.cudaMalloc) {
        places.push_back(Place::CudaOdd);
    }
    std::vector<Type> types = baseTypes();
    MPI_Datatype float3 = nullptr;
    MPI_Type_contiguous(3, MPI_FLOAT, &float3);
    MPI_Type_commit(&float3);
    types.push_back({ float3, "MPI_Type_contiguous(3, MPI_FLOAT)", Kind::F32, 3 });
    const std::vector<Op> ops = builtinOps();
    Comm world{ MPI_COMM_WORLD, everyRoot(size), rank };

    uint64_t seed = 1;
    if (o.part == Part::Bursts || o.part == Part::Persistent) {
        auto calls = [&](const Case& c, const std::vector<int>& roots) {
            if (o.part == Part::Bursts) {
                burstCalls(x, world, c, roots, cfg.stageBytes);
            } else {
                persistentCalls(x, world, c, roots, cfg.stageBytes);
            }
        };
        auto skip = [&](const Type& t, const Op& op, Place p) {
            return o.deviceOnly && (p == Place::Host || !defined(t, op.op->id));
        };
        const std::vector<size_t> small = o.count != 0 ? std::vector<size_t>{ o.count } : std::vector<size_t>{ 1, 7 };
        // every (datatype, op) pair, defined or not, on every placement
        for (const Type& t : types) {
            for (const Op& op : ops) {
                for (Place p : places) {
                    for (size_t count : small) {
                        Case c{ &t, &op, count, p, mix(seed++) };
                        if (!skip(t, op, p)) {
                            calls(c, { (int)(c.seed % (uint64_t)size) });
                        }
                    }
                }
            }
        }
        // the sizes around the LL limit, one vector and the staging pieces,
        // for a few pairs of every element width, at every root
        const std::vector<std::pair<int, int>> sized{ { 1, 9 }, { 19, 3 }, { 7, 2 }, { 12, 1 },
                                                      { 17, 0 }, { 20, 10 }, { 24, 2 } };
        for (auto [ti, oi] : sized) {
            const Type& t = types[ti];
            const Op& op = ops[oi];
            const size_t es = kindSize(t.kind) * (size_t)t.per;
            std::vector<size_t> counts{ cfg.llMaxBytes / es - 1, cfg.llMaxBytes / es + 1, cfg.stageBytes / es + 3 };
            if (16 / es > 1) {
                counts.push_back(16 / es - 1);
            }
            counts.push_back(16 / es + 1);
            for (Place p : places) {
                for (size_t count : counts) {
                    Case c{ &t, &op, count, p, mix(seed++) };
                    if (!skip(t, op, p)) {
                        calls(c, o.count != 0 ? std::vector<int>{ (int)(c.seed % (uint64_t)size) } : everyRoot(size));
                    }
                }
            }
        }
    } else if (o.part == Part::CrossKey) {
        crossKey(x, world, types, ops, places, o, comm.get(), cfg.stageBytes);
    } else {
        // a split by parity with reversed keys, and at 4 ranks and above a
        // split of it that rotates its order: the fold runs in child order
        std::vector<Comm> comms;
        MPI_Comm parity = MPI_COMM_NULL, nested = MPI_COMM_NULL;
        MPI_Comm_split(MPI_COMM_WORLD, rank % 2, size - rank, &parity);
        Comm pc{ parity, {}, -1, true };
        for (int r = size - 1; r >= 0; r--) {
            if (r % 2 == rank % 2) {
                pc.members.push_back(r);
            }
        }
        pc.me = (int)(std::find(pc.members.begin(), pc.members.end(), rank) - pc.members.begin());
        comms.push_back(pc);
        if (size >= 4) {
            const int m = pc.size();
            MPI_Comm_split(parity, 0, (pc.me + 1) % m, &nested);
            Comm nc{ nested, std::vector<int>(m), (pc.me + 1) % m, true };
            for (int i = 0; i < m; i++) {
                nc.members[(i + 1) % m] = pc.members[i];
            }
            comms.push_back(nc);
        }
        for (const Comm& cm : comms) {
            int r = -1, n = -1;
            MPI_Comm_rank(cm.comm, &r);
            MPI_Comm_size(cm.comm, &n);
            if (r != cm.me || n != cm.size()) {
                x.fail("sub-communicator: rank " + std::to_string(r) + " of " + std::to_string(n) + ", expected " +
                       std::to_string(cm.me) + " of " + std::to_string(cm.size()));
                continue;
            }
            // one pair per element width, pairs with MAXLOC / MINLOC, the
            // contiguous type, and a pair MPI does not define
            const std::vector<std::pair<MPI_Datatype, MPI_Op>> pairs{
                { MPI_INT8_T, MPI_SUM },      { MPI_BFLOAT16, MPI_MAX },  { MPI_UINT32_T, MPI_BXOR },
                { MPI_DOUBLE, MPI_SUM },      { MPI_LONG_INT, MPI_MAXLOC }, { MPI_2INT, MPI_MINLOC },
                { float3, MPI_SUM },          { MPI_FLOAT, MPI_BAND },
            };
            for (auto [dt, op] : pairs) {
                const Type* t = nullptr;
                for (const Type& ty : types) {
                    if (ty.dt == dt) {
                        t = &ty;
                    }
                }
                const Op& o2 = ops[opIndex(op)];
                for (Place p : places) {
                    for (size_t count : { (size_t)1, (size_t)7 }) {
                        Case c{ t, &o2, count, p, mix(seed++) };
                        burstCalls(x, cm, c, everyRoot(cm.size()), cfg.stageBytes);
                        persistentCalls(x, cm, c, everyRoot(cm.size()), cfg.stageBytes);
                    }
                }
            }
        }
        if (nested != MPI_COMM_NULL) {
            MPI_Comm_free(&nested);
        }
        MPI_Comm_free(&parity);
    }
    MPI_Type_free(&float3);

    if (x.failures.empty()) {
        return 0;
    }
    for (const std::string& f : x.failures) {
        *why += f + "\n";
    }
    return 1;
}

}
