#include "subcomm.h"
#include "buffers.h"

#include <faabric/util/logging.h>

#include <algorithm>
#include <atomic>
#include <map>
#include <mutex>
#include <shared_mutex>
#include <stdexcept>

namespace faabric::mpi {

SubCommunicator::SubCommunicator(int commIdIn, int worldIdIn, std::vector<int> worldRanksIn)
  : commId(commIdIn)
  , world(worldIdIn)
  , worldRanks(std::move(worldRanksIn))
{}

int SubCommunicator::commRankOf(int worldRank) const
{
    auto it = std::find(worldRanks.begin(), worldRanks.end(), worldRank);
    return it == worldRanks.end() ? -1 : (int)(it - worldRanks.begin());
}

int SubCommunicator::worldRankOf(int commRank) const
{
    if (commRank < 0 || commRank >= size()) {
        SPDLOG_ERROR("Rank {} outside communicator {} of size {}", commRank, commId, size());
        throw std::runtime_error("Rank outside the communicator");
    }
    return worldRanks[commRank];
}

void SubCommunicator::barrier(MpiWorld& w, int me)
{
    // Everyone checks in with comm rank 0, which then releases them
    faabric_datatype_t* byteType = getFaabricDatatypeFromId(FAABRIC_BYTE);
    const int leader = worldRanks[0];
    if (me == leader) {
        for (int r = 1; r < size(); r++) {
            w.recv(worldRanks[r], me, nullptr, byteType, 0, nullptr);
        }
        for (int r = 1; r < size(); r++) {
            w.send(me, worldRanks[r], nullptr, byteType, 0);
        }
    } else {
        w.send(me, leader, nullptr, byteType, 0);
        w.recv(leader, me, nullptr, byteType, 0, nullptr);
    }
}

void SubCommunicator::broadcast(MpiWorld& w, int me, int root, uint8_t* buffer, faabric_datatype_t* dt, int count)
{
    const size_t bytes = (size_t)count * dt->size;
    if (bytes > 0 && MpiWorld::isDevicePointer(buffer) && w.deviceBroadcast(deviceComm(w, me), me, root, buffer, bytes)) {
        return;
    }
    // Binomial tree over ranks relative to the root
    const int n = size();
    const int rel = (commRankOf(me) - root + n) % n;
    int mask = 1;
    while (mask < n) {
        if (rel & mask) {
            int from = (rel - mask + root) % n;
            w.recv(worldRanks[from], me, buffer, dt, count, nullptr);
            break;
        }
        mask <<= 1;
    }
    mask >>= 1;
    while (mask > 0) {
        if (rel + mask < n) {
            int to = (rel + mask + root) % n;
            w.send(me, worldRanks[to], buffer, dt, count);
        }
        mask >>= 1;
    }
}

void SubCommunicator::reduce(MpiWorld& w,
                             int me,
                             int root,
                             const uint8_t* send,
                             uint8_t* recv,
                             faabric_datatype_t* dt,
                             int count,
                             faabric_op_t* op)
{
    const size_t bytes = (size_t)count * dt->size;
    if (bytes > 0 && MpiWorld::isDevicePointer(send) && MpiWorld::deviceReducible(dt, op) &&
        w.deviceReduce(deviceComm(w, me), me, root, send, recv, dt, count, op)) {
        return;
    }
    const int n = size();
    const int myCommRank = commRankOf(me);
    if (myCommRank != root) {
        w.send(me, worldRanks[root], send, dt, count);
        return;
    }
    // Fold in rank order, right to left: r0 op (r1 op (... op r[n-1])), which
    // is what MPI asks of non-commutative operations too
    std::vector<uint8_t> all(bytes * (size_t)n);
    for (int r = 0; r < n; r++) {
        uint8_t* slot = all.data() + (size_t)r * bytes;
        if (r == root) {
            copyBytes(slot, send, bytes);
        } else {
            w.recv(worldRanks[r], me, slot, dt, count, nullptr);
        }
    }
    uint8_t* acc = all.data() + (size_t)(n - 1) * bytes;
    for (int r = n - 2; r >= 0; r--) {
        w.op_reduce(op, dt, count, all.data() + (size_t)r * bytes, acc);
    }
    copyBytes(recv, acc, bytes);
}

void SubCommunicator::allReduce(MpiWorld& w,
                                int me,
                                const uint8_t* send,
                                uint8_t* recv,
                                faabric_datatype_t* dt,
                                int count,
                                faabric_op_t* op)
{
    if (count > 0 && dt->size > 0 && MpiWorld::isDevicePointer(send) && MpiWorld::deviceReducible(dt, op) &&
        w.deviceAllReduce(deviceComm(w, me), me, send, recv, dt, count, op)) {
        return;
    }
    reduce(w, me, 0, send, recv, dt, count, op);
    broadcast(w, me, 0, recv, dt, count);
}

void SubCommunicator::scan(MpiWorld& w,
                           int me,
                           const uint8_t* send,
                           uint8_t* recv,
                           faabric_datatype_t* dt,
                           int count,
                           faabric_op_t* op)
{
    const size_t bytes = (size_t)count * dt->size;
    if (bytes > 0 && MpiWorld::isDevicePointer(send) && send != recv && MpiWorld::deviceReducible(dt, op) &&
        w.deviceScan(deviceComm(w, me), me, send, recv, dt, count, op)) {
        return;
    }
    const int myCommRank = commRankOf(me);
    std::vector<uint8_t> acc(bytes);
    copyBytes(acc.data(), send, bytes);
    if (myCommRank > 0) {
        std::vector<uint8_t> prev(bytes);
        w.recv(worldRanks[myCommRank - 1], me, prev.data(), dt, count, nullptr);
        // acc = prefix op mine
        w.op_reduce(op, dt, count, prev.data(), acc.data());
    }
    if (myCommRank < size() - 1) {
        w.send(me, worldRanks[myCommRank + 1], acc.data(), dt, count);
    }
    copyBytes(recv, acc.data(), bytes);
}

void SubCommunicator::exscan(MpiWorld& w,
                             int me,
                             const uint8_t* send,
                             uint8_t* recv,
                             faabric_datatype_t* dt,
                             int count,
                             faabric_op_t* op)
{
    const size_t bytes = (size_t)count * dt->size;
    // (in place decides nothing: see MpiWorld::exscan)
    if (bytes > 0 && MpiWorld::isDevicePointer(send) && MpiWorld::deviceReducible(dt, op) &&
        w.deviceExscan(deviceComm(w, me), me, send, recv, dt, count, op)) {
        return;
    }
    const int myCommRank = commRankOf(me);
    std::vector<uint8_t> acc(bytes);
    std::vector<uint8_t> prev(bytes);
    copyBytes(acc.data(), send, bytes);
    if (myCommRank > 0) {
        w.recv(worldRanks[myCommRank - 1], me, prev.data(), dt, count, nullptr);
        // acc = prefix op mine, before an in-place recv is overwritten
        w.op_reduce(op, dt, count, prev.data(), acc.data());
    }
    if (myCommRank < size() - 1) {
        w.send(me, worldRanks[myCommRank + 1], acc.data(), dt, count);
    }
    if (myCommRank > 0) {
        copyBytes(recv, prev.data(), bytes);
    }
}

void SubCommunicator::gather(MpiWorld& w, int me, int root, const uint8_t* send, uint8_t* recv, faabric_datatype_t* dt, int count)
{
    const size_t bytes = (size_t)count * dt->size;
    // (the root's in-place contribution sits in recv: it decides from that)
    if (bytes > 0 && MpiWorld::isDevicePointer(send != nullptr ? send : recv) &&
        w.deviceGather(deviceComm(w, me), me, root, send, recv, bytes)) {
        return;
    }
    if (commRankOf(me) != root) {
        w.send(me, worldRanks[root], send, dt, count);
        return;
    }
    for (int r = 0; r < size(); r++) {
        uint8_t* slot = recv + (size_t)r * bytes;
        if (r == root) {
            if (send != nullptr) {
                copyBytes(slot, send, bytes);
            }
        } else {
            w.recv(worldRanks[r], me, slot, dt, count, nullptr);
        }
    }
}

void SubCommunicator::scatter(MpiWorld& w, int me, int root, const uint8_t* send, uint8_t* recv, faabric_datatype_t* dt, int count)
{
    const size_t bytes = (size_t)count * dt->size;
    // (an in-place root keeps its chunk in send: it decides from that)
    if (bytes > 0 && MpiWorld::isDevicePointer(recv != nullptr ? recv : send) &&
        w.deviceScatter(deviceComm(w, me), me, root, send, recv, bytes)) {
        return;
    }
    if (commRankOf(me) != root) {
        w.recv(worldRanks[root], me, recv, dt, count, nullptr);
        return;
    }
    for (int r = 0; r < size(); r++) {
        const uint8_t* chunk = send + (size_t)r * bytes;
        if (r == root) {
            if (recv != nullptr) {
                copyBytes(recv, chunk, bytes);
            }
        } else {
            w.send(me, worldRanks[r], chunk, dt, count);
        }
    }
}

void SubCommunicator::allGather(MpiWorld& w, int me, const uint8_t* send, uint8_t* recv, faabric_datatype_t* dt, int count)
{
    const size_t bytes = (size_t)count * dt->size;
    if (bytes > 0 && MpiWorld::isDevicePointer(send) && send != recv + (size_t)commRankOf(me) * bytes &&
        w.deviceAllGather(deviceComm(w, me), me, send, recv, bytes)) {
        return;
    }
    // (an in-place chunk is skipped by the self-copy check)
    gather(w, me, 0, send, recv, dt, count);
    broadcast(w, me, 0, recv, dt, count * size());
}

void SubCommunicator::allToAll(MpiWorld& w, int me, const uint8_t* send, uint8_t* recv, faabric_datatype_t* dt, int count)
{
    const size_t bytes = (size_t)count * dt->size;
    if (bytes > 0 && MpiWorld::isDevicePointer(send) && w.deviceAllToAll(deviceComm(w, me), me, send, recv, bytes)) {
        return;
    }
    const int n = size();
    const int myCommRank = commRankOf(me);
    // Sends are eager: ship everything, then collect in rank order
    for (int r = 0; r < n; r++) {
        const uint8_t* chunk = send + (size_t)r * bytes;
        if (r == myCommRank) {
            copyBytes(recv + (size_t)r * bytes, chunk, bytes);
        } else {
            w.send(me, worldRanks[r], chunk, dt, count);
        }
    }
    for (int r = 0; r < n; r++) {
        if (r != myCommRank) {
            w.recv(worldRanks[r], me, recv + (size_t)r * bytes, dt, count, nullptr);
        }
    }
}

void SubCommunicator::reduceScatter(MpiWorld& w,
                                    int me,
                                    const uint8_t* send,
                                    uint8_t* recv,
                                    faabric_datatype_t* dt,
                                    int recvCount,
                                    faabric_op_t* op)
{
    const size_t shard = (size_t)recvCount * dt->size;
    if (shard > 0 && MpiWorld::isDevicePointer(send) && MpiWorld::deviceReducible(dt, op) &&
        w.deviceReduceScatter(deviceComm(w, me), me, send, recv, dt, recvCount, op)) {
        return;
    }
    // The rank-ordered fold of allReduce on host copies, then each member
    // keeps its own block (staged first: in place, recv is also the input)
    const int n = size();
    HostStage in;
    const uint8_t* src = in.in(send, shard * (size_t)n);
    std::vector<uint8_t> full(shard * (size_t)n);
    reduce(w, me, 0, src, full.data(), dt, recvCount * n, op);
    broadcast(w, me, 0, full.data(), dt, recvCount * n);
    copyBytes(recv, full.data() + (size_t)commRankOf(me) * shard, shard);
}

void SubCommunicator::setGraph(std::shared_ptr<Graph> g)
{
    std::lock_guard<std::mutex> lk(graphMx);
    if (topo == nullptr) {
        topo = std::move(g);
    }
}

void SubCommunicator::neighborExchange(MpiWorld& w, int me, bool allToAll, const uint8_t* send, uint8_t* recv,
                                       faabric_datatype_t* dt, int count)
{
    const size_t bytes = (size_t)count * dt->size;
    const int cr = commRankOf(me);
    const auto& dst = topo->destinations[cr];
    const auto& in = topo->in[cr];
    for (size_t i = 0; i < dst.size(); i++) {
        if (dst[i] != cr) {
            w.send(me, worldRanks[dst[i]], send + (allToAll ? i * bytes : 0), dt, count);
        }
    }
    for (size_t j = 0; j < in.size(); j++) {
        const auto [src, idx] = in[j];
        if (src == cr) {
            copyBytes(recv + j * bytes, send + (allToAll ? (size_t)idx * bytes : 0), bytes);
        } else {
            w.recv(worldRanks[src], me, recv + j * bytes, dt, count, nullptr);
        }
    }
}

void SubCommunicator::neighborExchangeV(MpiWorld& w, int me, bool allToAll, const uint8_t* send,
                                        const int* sendCounts, const int* sendDispls, faabric_datatype_t* sendType,
                                        uint8_t* recv, const int* recvCounts, const int* recvDispls,
                                        faabric_datatype_t* recvType)
{
    const int cr = commRankOf(me);
    const auto& dst = topo->destinations[cr];
    const auto& in = topo->in[cr];
    auto sendBlock = [&](size_t i) { return send + (allToAll ? (size_t)sendDispls[i] * sendType->size : 0); };
    for (size_t i = 0; i < dst.size(); i++) {
        if (dst[i] != cr) {
            w.send(me, worldRanks[dst[i]], sendBlock(i), sendType, sendCounts[allToAll ? i : 0]);
        }
    }
    for (size_t j = 0; j < in.size(); j++) {
        const auto [src, idx] = in[j];
        uint8_t* block = recv + (size_t)recvDispls[j] * recvType->size;
        if (src == cr) {
            copyBytes(block, sendBlock(idx), (size_t)recvCounts[j] * recvType->size);
        } else {
            w.recv(worldRanks[src], me, block, recvType, recvCounts[j], nullptr);
        }
    }
}

std::shared_ptr<faabric::device::Communicator> SubCommunicator::currentDevice(int me)
{
    std::lock_guard<std::mutex> lk(deviceMx);
    auto it = device.find(me);
    return it == device.end() ? nullptr : it->second.child;
}

std::shared_ptr<faabric::device::Communicator> SubCommunicator::deviceComm(MpiWorld& w, int me)
{
    {
        std::lock_guard<std::mutex> lk(deviceMx);
        const DeviceState& st = device[me];
        if (st.decided) {
            return st.child;
        }
    }
    // Slot agreement, once per rank: the lowest slot free on every member.
    // The lock is not held across it: the other ranks of this process agree
    // through the same object.  Members are world ranks, so every child (of a
    // nested split too) is cut from the world communicator.
    auto parent = w.getDeviceComm(me);
    int mask = parent != nullptr ? (int)parent->freeSubsetSlots() : 0;
    int agreed = 0;
    allReduce(w, me, (const uint8_t*)&mask, (uint8_t*)&agreed, MPI_INT, 1, MPI_BAND);
    std::shared_ptr<faabric::device::Communicator> child;
    if (agreed != 0) {
        int rc = FB_OK;
        child = parent->subset(worldRanks, __builtin_ctz((unsigned)agreed), &rc);
        if (child == nullptr) {
            // the other members run on the slot: this rank cannot fall back alone
            SPDLOG_ERROR("Communicator {}: rank {} cannot take agreed slot {} ({})", commId, me,
                         __builtin_ctz((unsigned)agreed), faabric::device::Communicator::errorString(rc));
            throw std::runtime_error("Sub-communicator slot agreement failed");
        }
        // a dist-graph communicator's child carries its topology (the
        // caller routes graphs the device cannot take to the host path)
        if (topo != nullptr && topo->maxIn <= FB_NEIGHBOR_MAX_IN_DEGREE) {
            const int cr = commRankOf(me);
            const int trc = child->setNeighbors(topo->in[cr], (int)topo->destinations[cr].size(), topo->maxOut,
                                                topo->maxIn);
            if (trc != FB_OK) {
                throw std::runtime_error(std::string("Sub-communicator topology refused: ") +
                                         faabric::device::Communicator::errorString(trc));
            }
        }
    }
    std::lock_guard<std::mutex> lk(deviceMx);
    DeviceState& st = device[me];
    st.decided = true;
    st.child = child;
    return child;
}

void SubCommunicator::releaseDevice(int me)
{
    std::shared_ptr<faabric::device::Communicator> child;
    {
        std::lock_guard<std::mutex> lk(deviceMx);
        DeviceState& st = device[me];
        st.decided = true;
        child = std::move(st.child);
    }
    // (the destructor zeroes this rank's slot pad, then frees the slot)
}

// ---------------------------------------------------------------------------
// Registries
// ---------------------------------------------------------------------------
namespace {
std::shared_mutex commsMx;
std::map<int, std::shared_ptr<SubCommunicator>> comms;

std::mutex groupsMx;
std::map<int, std::vector<int>> groups;
std::atomic<int> nextGroupId{ 1 };

uint64_t mix(uint64_t h, uint64_t v)
{
    // splitmix-style avalanche
    h ^= v + 0x9e3779b97f4a7c15ULL + (h << 6) + (h >> 2);
    h ^= h >> 30;
    h *= 0xbf58476d1ce4e5b9ULL;
    h ^= h >> 27;
    return h;
}
}

int deriveCommId(int worldId, int parentCommId, int sequence, uint64_t discriminator)
{
    uint64_t h = mix(0x243f6a8885a308d3ULL, (uint64_t)(uint32_t)worldId);
    h = mix(h, (uint64_t)(uint32_t)parentCommId);
    h = mix(h, (uint64_t)(uint32_t)sequence);
    h = mix(h, discriminator);
    // positive, and clear of the predefined communicator ids
    return (int)(h % 0x7fff0000ULL) + 1000;
}

std::shared_ptr<SubCommunicator> registerSubCommunicator(int commId, int worldId, const std::vector<int>& worldRanks)
{
    std::unique_lock<std::shared_mutex> lk(commsMx);
    auto& slot = comms[commId];
    if (slot == nullptr) {
        slot = std::make_shared<SubCommunicator>(commId, worldId, worldRanks);
    } else if (slot->ranks() != worldRanks || slot->worldId() != worldId) {
        SPDLOG_ERROR("Communicator id {} collides with a different communicator", commId);
        throw std::runtime_error("Sub-communicator id collision");
    }
    return slot;
}

std::shared_ptr<SubCommunicator> getSubCommunicator(int commId)
{
    std::shared_lock<std::shared_mutex> lk(commsMx);
    auto it = comms.find(commId);
    return it == comms.end() ? nullptr : it->second;
}

void clearSubCommunicators(int worldId)
{
    // worldId < 0: every world
    std::unique_lock<std::shared_mutex> lk(commsMx);
    for (auto it = comms.begin(); it != comms.end();) {
        it = (worldId < 0 || it->second->worldId() == worldId) ? comms.erase(it) : std::next(it);
    }
}

int registerGroup(std::vector<int> worldRanks)
{
    std::lock_guard<std::mutex> lk(groupsMx);
    int id = nextGroupId.fetch_add(1);
    groups[id] = std::move(worldRanks);
    return id;
}

bool getGroup(int groupId, std::vector<int>& worldRanks)
{
    std::lock_guard<std::mutex> lk(groupsMx);
    auto it = groups.find(groupId);
    if (it == groups.end()) {
        return false;
    }
    worldRanks = it->second;
    return true;
}

void freeGroup(int groupId)
{
    std::lock_guard<std::mutex> lk(groupsMx);
    groups.erase(groupId);
}

}
