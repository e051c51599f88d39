// The MPI_* C functions, mapped onto MpiWorld through the per-thread
// MpiContext and the ExecutorContext of the running function.  In the
// reference this shim lives in the test tree (tests/dist/mpi/mpi_native.cpp:
// 59-776) and in Faasm's WASM host interface; here it ships with the library.
// Beyond the reference's implemented set it adds Reduce_scatter (equal
// counts), Allgatherv / Gatherv / Alltoallv (equal-count fast path + generic
// point-to-point fallback), Waitall / Waitany, Initialized / Finalized,
// Init_thread / Query_thread and Get_version.
#include <faabric/executor/ExecutorContext.h>
#include <faabric/mpi/MpiContext.h>
#include <faabric/mpi/MpiWorldRegistry.h>
#include <faabric/mpi/mpi.h>
#include <faabric/util/config.h>
#include <faabric/util/logging.h>

#include "buffers.h"
#include "subcomm.h"

#include <algorithm>
#include <atomic>
#include <cstring>
#include <map>
#include <stdexcept>
#include <unistd.h>
#include <vector>

using namespace faabric::mpi;

namespace {
thread_local MpiContext executingContext;
thread_local bool mpiInitialised = false;
thread_local bool mpiFinalised = false;

// (looked up once per thread and world: every MPI call starts here, and eight
// rank threads copying the same shared_ptr bounce its reference count around)
namespace {
thread_local int cachedWorldId = -1;
thread_local MpiWorld* cachedWorld = nullptr;
}

MpiWorld& getExecutingWorld()
{
    int worldId = executingContext.getWorldId();
    if (cachedWorld == nullptr || cachedWorldId != worldId) {
        cachedWorld = &getMpiWorldRegistry().getWorld(worldId);
        cachedWorldId = worldId;
    }
    return *cachedWorld;
}

void forgetExecutingWorld()
{
    cachedWorld = nullptr;
    cachedWorldId = -1;
}

faabric::Message* getExecutingCall()
{
    return &faabric::executor::ExecutorContext::get()->getMsg();
}

int terminateMpi()
{
    struct Forget
    {
        ~Forget() { forgetExecutingWorld(); }
    } forget;
    // Destroy the MPI world
    bool mustClear = getExecutingWorld().destroy();
    if (mustClear) {
        clearSubCommunicators(executingContext.getWorldId());
        getMpiWorldRegistry().clearWorld(executingContext.getWorldId());
    }
    mpiFinalised = true;
    return MPI_SUCCESS;
}

// In-place collectives pass MPI_IN_PLACE as the send buffer
const void* resolveInPlace(const void* sendbuf, void* recvbuf)
{
    return sendbuf == MPI_IN_PLACE ? recvbuf : sendbuf;
}

// ---- sub-communicators ----
// Calls on MPI_COMM_WORLD (and cartesian views of it) take the world's fused
// paths; anything else resolves to a SubCommunicator
std::shared_ptr<SubCommunicator> subOf(MPI_Comm comm)
{
    if (comm == nullptr || comm->id == FAABRIC_COMM_WORLD) {
        return nullptr;
    }
    if (comm->id == FAABRIC_COMM_NULL) {
        throw std::runtime_error("MPI call on MPI_COMM_NULL");
    }
    auto sub = getSubCommunicator(comm->id);
    if (sub == nullptr) {
        throw std::runtime_error("Unknown communicator " + std::to_string(comm->id));
    }
    return sub;
}

// Rank of `comm` -> rank of the world
int toWorldRank(MPI_Comm comm, int rank)
{
    auto sub = subOf(comm);
    return sub == nullptr ? rank : sub->worldRankOf(rank);
}

void subCommOnly(MPI_Comm comm, const char* what)
{
    if (subOf(comm) != nullptr) {
        throw std::runtime_error(std::string(what) + " is only implemented on MPI_COMM_WORLD");
    }
}

// Creating calls issued so far on each parent communicator by this rank (they
// are collective, so every member counts the same)
thread_local std::map<int, int> commCreateSeq;

// Ranks (world numbering) of a communicator, in communicator order
std::vector<int> ranksOf(MPI_Comm comm)
{
    auto sub = subOf(comm);
    if (sub != nullptr) {
        return sub->ranks();
    }
    std::vector<int> all(getExecutingWorld().getSize());
    for (int r = 0; r < (int)all.size(); r++) {
        all[r] = r;
    }
    return all;
}

MPI_Comm makeCommHandle(int parentId, int seq, uint64_t discriminator, const std::vector<int>& worldRanks)
{
    int worldId = executingContext.getWorldId();
    int id = deriveCommId(worldId, parentId, seq, discriminator);
    registerSubCommunicator(id, worldId, worldRanks);
    return new faabric_communicator_t{ id };
}

std::map<int, faabric_request_t*>& requestTable()
{
    static thread_local std::map<int, faabric_request_t*> t;
    return t;
}

// MPI_REPLACE and MPI_NO_OP only exist for one-sided accumulates.  Collectives
// refuse them up front, before any rank sends, waits or launches.
bool accumulateOnlyOp(MPI_Op op)
{
    return op != nullptr && (op->id == FAABRIC_OP_REPLACE || op->id == FAABRIC_OP_NO_OP);
}

// A datatype as (predefined base type, base elements per element)
bool baseTypeOf(MPI_Datatype dt, MPI_Datatype* base, int* per)
{
    if (dt == nullptr) {
        return false;
    }
    int baseId = dt->id;
    *per = 1;
    if (dt->id >= FAABRIC_DERIVED_TYPE_BASE && !getContiguousType(dt->id, &baseId, per)) {
        return false;
    }
    *base = getFaabricDatatypeFromId(baseId);
    return *base != nullptr && fbDtypeFor(*base) >= 0;
}

// The element type and element count shared by the origin / result and the
// target of an accumulate.  MPI_ERR_ARG unless every buffer has the same base
// type and the same number of bytes.
int accumulateShape(const std::vector<std::pair<int, MPI_Datatype>>& sides, MPI_Datatype* base, size_t* count)
{
    int fdt = -1;
    int64_t bytes = -1;
    for (const auto& [n, dt] : sides) {
        MPI_Datatype b = nullptr;
        int per = 0;
        if (n < 0 || !baseTypeOf(dt, &b, &per)) {
            return MPI_ERR_ARG;
        }
        const int64_t sideBytes = (int64_t)n * dt->size;
        if ((fdt >= 0 && fbDtypeFor(b) != fdt) || (bytes >= 0 && sideBytes != bytes)) {
            return MPI_ERR_ARG;
        }
        fdt = fbDtypeFor(b);
        bytes = sideBytes;
        *base = b;
    }
    *count = (size_t)bytes / (size_t)(*base)->size;
    return MPI_SUCCESS;
}

// `request` non-null: the request-based form (MPI_Raccumulate,
// MPI_Rget_accumulate)
int getAccumulate(const void* origin, int originCount, MPI_Datatype originType, void* result, int resultCount,
                  MPI_Datatype resultType, int targetRank, MPI_Aint targetDisp, int targetCount, MPI_Datatype targetType,
                  MPI_Op op, MPI_Win win, MPI_Request* request = nullptr)
{
    if (win == nullptr) {
        return MPI_ERR_WIN;
    }
    if (op == nullptr || isUserOp(op)) {
        return MPI_ERR_OP;
    }
    if (op->id == FAABRIC_OP_NO_OP && result == nullptr) {
        return MPI_ERR_OP; // MPI_NO_OP only fetches
    }
    std::vector<std::pair<int, MPI_Datatype>> sides{ { targetCount, targetType } };
    if (op->id != FAABRIC_OP_NO_OP) {
        sides.emplace_back(originCount, originType); // (ignored for MPI_NO_OP)
    }
    if (result != nullptr) {
        sides.emplace_back(resultCount, resultType);
    }
    MPI_Datatype base = nullptr;
    size_t count = 0;
    int rc = accumulateShape(sides, &base, &count);
    if (rc != MPI_SUCCESS) {
        return rc;
    }
    if (request != nullptr) {
        int id = 0;
        rc = getExecutingWorld().winRaccumulate(executingContext.getRank(), win->id, (const uint8_t*)origin, count, base,
                                                op, (uint8_t*)result, targetRank, (int64_t)targetDisp, &id);
        if (rc == MPI_SUCCESS) {
            *request = new faabric_request_t{ id };
            requestTable()[id] = *request;
        }
        return rc;
    }
    return getExecutingWorld().winAccumulate(executingContext.getRank(), win->id, (const uint8_t*)origin, count, base, op,
                                             (uint8_t*)result, targetRank, (int64_t)targetDisp);
}

// MPI_Rput / MPI_Rget
int requestPutGet(void* origin, int originCount, MPI_Datatype originType, int targetRank, MPI_Aint targetDisp,
                  int targetCount, MPI_Datatype targetType, MPI_Win win, MPI_Request* request, bool get)
{
    if (win == nullptr) {
        return MPI_ERR_WIN;
    }
    if (request == nullptr || originType == nullptr || targetType == nullptr || originCount < 0 || targetCount < 0) {
        return MPI_ERR_ARG;
    }
    const size_t bytes = (size_t)originCount * originType->size;
    if (bytes != (size_t)targetCount * targetType->size) {
        return MPI_ERR_ARG;
    }
    int id = 0;
    int rc = getExecutingWorld().winRputGet(executingContext.getRank(), win->id, (uint8_t*)origin, bytes, targetRank,
                                            (int64_t)targetDisp, get, &id);
    if (rc == MPI_SUCCESS) {
        *request = new faabric_request_t{ id };
        requestTable()[id] = *request;
    }
    return rc;
}
}

extern "C"
{

int MPI_Init(int* argc, char*** argv)
{
    forgetExecutingWorld(); // a pool thread runs many functions, one world each
    faabric::Message* call = getExecutingCall();
    // A function resuming after a migration / thaw re-enters an existing
    // world: even rank 0 joins, and nobody waits for it at a start-up barrier
    auto ctx = faabric::executor::ExecutorContext::get();
    const bool resuming = ctx->getBatchRequest() != nullptr &&
                          ctx->getBatchRequest()->type() == faabric::BatchExecuteRequest::MIGRATION &&
                          call->mpiworldid() > 0;
    if (call->mpirank() <= 0 && !resuming) {
        // A world of the configured size is created by rank 0
        SPDLOG_TRACE("MPI - MPI_Init (create)");
        if (call->mpiworldsize() <= 0) {
            call->set_mpiworldsize(faabric::util::getSystemConfig().defaultMpiWorldSize);
        }
        call->set_ismpi(true);
        executingContext.createWorld(*call);
    } else {
        SPDLOG_TRACE("MPI - MPI_Init (join)");
        executingContext.joinWorld(*call);
    }
    mpiInitialised = true;
    mpiFinalised = false;
    commCreateSeq.clear();
    if (!resuming) {
        // Everyone lines up once the world is wired
        getExecutingWorld().barrier(executingContext.getRank());
    }
    return MPI_SUCCESS;
}

int MPI_Init_thread(int* argc, char*** argv, int required, int* provided)
{
    if (provided != nullptr) {
        // Ranks are threads but each rank's MPI calls come from one thread
        *provided = MPI_THREAD_SERIALIZED;
    }
    return MPI_Init(argc, argv);
}

int MPI_Query_thread(int* provided)
{
    *provided = MPI_THREAD_SERIALIZED;
    return MPI_SUCCESS;
}

int MPI_Initialized(int* flag)
{
    *flag = mpiInitialised ? 1 : 0;
    return MPI_SUCCESS;
}

int MPI_Finalized(int* flag)
{
    *flag = mpiFinalised ? 1 : 0;
    return MPI_SUCCESS;
}

int MPI_Get_version(int* version, int* subversion)
{
    *version = 3;
    *subversion = 1;
    return MPI_SUCCESS;
}

int MPI_Comm_rank(MPI_Comm comm, int* rank)
{
    SPDLOG_TRACE("MPI - MPI_Comm_rank");
    if (auto sub = subOf(comm)) {
        *rank = sub->commRankOf(executingContext.getRank());
        return MPI_SUCCESS;
    }
    *rank = executingContext.getRank();
    return MPI_SUCCESS;
}

int MPI_Comm_size(MPI_Comm comm, int* size)
{
    SPDLOG_TRACE("MPI - MPI_Comm_size");
    if (auto sub = subOf(comm)) {
        *size = sub->size();
        return MPI_SUCCESS;
    }
    *size = getExecutingWorld().getSize();
    return MPI_SUCCESS;
}

int MPI_Finalize()
{
    SPDLOG_TRACE("MPI - MPI_Finalize");
    return terminateMpi();
}

int MPI_Abort(MPI_Comm comm, int errorcode)
{
    SPDLOG_TRACE("MPI - MPI_Abort");
    return terminateMpi();
}

int MPI_Send(const void* buf, int count, MPI_Datatype datatype, int dest, int tag, MPI_Comm comm)
{
    SPDLOG_TRACE("MPI - MPI_Send {} -> {}", executingContext.getRank(), dest);
    getExecutingWorld().send(executingContext.getRank(), toWorldRank(comm, dest), (const uint8_t*)buf, datatype, count);
    return MPI_SUCCESS;
}

int MPI_Rsend(const void* buf, int count, MPI_Datatype datatype, int dest, int tag, MPI_Comm comm)
{
    // A ready-send is a send whose receive is already posted: same thing here
    return MPI_Send(buf, count, datatype, dest, tag, comm);
}

int MPI_Recv(void* buf, int count, MPI_Datatype datatype, int source, int tag, MPI_Comm comm, MPI_Status* status)
{
    SPDLOG_TRACE("MPI - MPI_Recv {} <- {}", executingContext.getRank(), source);
    getExecutingWorld().recv(toWorldRank(comm, source), executingContext.getRank(), (uint8_t*)buf, datatype, count, status);
    if (status != MPI_STATUS_IGNORE && subOf(comm) != nullptr) {
        status->MPI_SOURCE = source;
    }
    return MPI_SUCCESS;
}

int MPI_Sendrecv(const void* sendbuf, int sendcount, MPI_Datatype sendtype, int dest, int sendtag,
                 void* recvbuf, int recvcount, MPI_Datatype recvtype, int source, int recvtag,
                 MPI_Comm comm, MPI_Status* status)
{
    SPDLOG_TRACE("MPI - MPI_Sendrecv");
    getExecutingWorld().sendRecv((uint8_t*)sendbuf, sendcount, sendtype, toWorldRank(comm, dest),
                                 (uint8_t*)recvbuf, recvcount, recvtype, toWorldRank(comm, source),
                                 executingContext.getRank(), status);
    if (status != MPI_STATUS_IGNORE && subOf(comm) != nullptr) {
        status->MPI_SOURCE = source;
    }
    return MPI_SUCCESS;
}

int MPI_Isend(const void* buf, int count, MPI_Datatype datatype, int dest, int tag, MPI_Comm comm, MPI_Request* request)
{
    SPDLOG_TRACE("MPI - MPI_Isend {} -> {}", executingContext.getRank(), dest);
    int id = getExecutingWorld().isend(executingContext.getRank(), toWorldRank(comm, dest), (const uint8_t*)buf, datatype, count);
    auto* r = new faabric_request_t{ id };
    requestTable()[id] = r;
    *request = r;
    return MPI_SUCCESS;
}

int MPI_Irecv(void* buf, int count, MPI_Datatype datatype, int source, int tag, MPI_Comm comm, MPI_Request* request)
{
    SPDLOG_TRACE("MPI - MPI_Irecv {} <- {}", executingContext.getRank(), source);
    int id = getExecutingWorld().irecv(toWorldRank(comm, source), executingContext.getRank(), (uint8_t*)buf, datatype, count);
    auto* r = new faabric_request_t{ id };
    requestTable()[id] = r;
    *request = r;
    return MPI_SUCCESS;
}

int MPI_Wait(MPI_Request* request, MPI_Status* status)
{
    if (request == nullptr || *request == nullptr) {
        return MPI_SUCCESS;
    }
    int id = (*request)->id;
    SPDLOG_TRACE("MPI - MPI_Wait {}", id);
    getExecutingWorld().awaitAsyncRequest(id);
    requestTable().erase(id);
    delete *request;
    *request = nullptr;
    return MPI_SUCCESS;
}

int MPI_Waitall(int count, MPI_Request array_of_requests[], MPI_Status* array_of_statuses)
{
    for (int i = 0; i < count; i++) {
        MPI_Wait(&array_of_requests[i], MPI_STATUS_IGNORE);
    }
    return MPI_SUCCESS;
}

int MPI_Waitany(int count, MPI_Request array_of_requests[], int* index, MPI_Status* status)
{
    // Completion is in posting order per pair, so the first live request is
    // as good a choice as any
    for (int i = 0; i < count; i++) {
        if (array_of_requests[i] != nullptr) {
            MPI_Wait(&array_of_requests[i], status);
            *index = i;
            return MPI_SUCCESS;
        }
    }
    *index = MPI_UNDEFINED;
    return MPI_SUCCESS;
}

int MPI_Request_free(MPI_Request* request)
{
    if (request != nullptr && *request != nullptr) {
        getExecutingWorld().freeAsyncRequest((*request)->id);
        requestTable().erase((*request)->id);
        delete *request;
        *request = nullptr;
    }
    return MPI_SUCCESS;
}

int MPI_Get_count(const MPI_Status* status, MPI_Datatype datatype, int* count)
{
    SPDLOG_TRACE("MPI - MPI_Get_count");
    if (status->bytesSize % datatype->size != 0) {
        SPDLOG_ERROR("Incomplete message (bytes {}, datatype size {})", status->bytesSize, datatype->size);
        return 1;
    }
    *count = status->bytesSize / datatype->size;
    return MPI_SUCCESS;
}

int MPI_Probe(int source, int tag, MPI_Comm comm, MPI_Status* status)
{
    SPDLOG_TRACE("MPI - MPI_Probe");
    getExecutingWorld().probe(toWorldRank(comm, source), executingContext.getRank(), status);
    if (status != MPI_STATUS_IGNORE && subOf(comm) != nullptr) {
        status->MPI_SOURCE = source;
    }
    return MPI_SUCCESS;
}

int MPI_Barrier(MPI_Comm comm)
{
    SPDLOG_TRACE("MPI - MPI_Barrier");
    if (auto sub = subOf(comm)) {
        sub->barrier(getExecutingWorld(), executingContext.getRank());
        return MPI_SUCCESS;
    }
    getExecutingWorld().barrier(executingContext.getRank());
    return MPI_SUCCESS;
}

int MPI_Bcast(void* buffer, int count, MPI_Datatype datatype, int root, MPI_Comm comm)
{
    SPDLOG_TRACE("MPI - MPI_Bcast {} -> all", root);
    if (auto sub = subOf(comm)) {
        sub->broadcast(getExecutingWorld(), executingContext.getRank(), root, (uint8_t*)buffer, datatype, count);
        return MPI_SUCCESS;
    }
    getExecutingWorld().broadcast(root, executingContext.getRank(), (uint8_t*)buffer, datatype, count, MpiMessageType::BROADCAST);
    return MPI_SUCCESS;
}

int MPI_Scatter(const void* sendbuf, int sendcount, MPI_Datatype sendtype, void* recvbuf, int recvcount,
                MPI_Datatype recvtype, int root, MPI_Comm comm)
{
    SPDLOG_TRACE("MPI - MPI_Scatter {} -> all", root);
    if (auto sub = subOf(comm)) {
        // MPI_IN_PLACE as the root's receive buffer: its chunk stays where it is
        uint8_t* recv = recvbuf == MPI_IN_PLACE ? nullptr : (uint8_t*)recvbuf;
        const bool isRoot = sub->commRankOf(executingContext.getRank()) == root;
        sub->scatter(getExecutingWorld(), executingContext.getRank(), root, (const uint8_t*)sendbuf, recv,
                     isRoot ? sendtype : recvtype, isRoot ? sendcount : recvcount);
        return MPI_SUCCESS;
    }
    getExecutingWorld().scatter(root, executingContext.getRank(), (const uint8_t*)sendbuf, sendtype, sendcount,
                                (uint8_t*)recvbuf, recvtype, recvcount);
    return MPI_SUCCESS;
}

int MPI_Gather(const void* sendbuf, int sendcount, MPI_Datatype sendtype, void* recvbuf, int recvcount,
               MPI_Datatype recvtype, int root, MPI_Comm comm)
{
    SPDLOG_TRACE("MPI - MPI_Gather all -> {}", root);
    int rank = executingContext.getRank();
    if (auto sub = subOf(comm)) {
        const bool isRoot = sub->commRankOf(rank) == root;
        const uint8_t* chunk = sendbuf == MPI_IN_PLACE ? nullptr : (const uint8_t*)sendbuf;
        sub->gather(getExecutingWorld(), rank, root, chunk, (uint8_t*)recvbuf, isRoot ? recvtype : sendtype,
                    isRoot ? recvcount : sendcount);
        return MPI_SUCCESS;
    }
    const uint8_t* send = (const uint8_t*)sendbuf;
    if (sendbuf == MPI_IN_PLACE) {
        // The root's chunk is already in place in the receive buffer
        send = (const uint8_t*)recvbuf;
        sendcount = recvcount;
        sendtype = recvtype;
    }
    getExecutingWorld().gather(rank, root, send, sendtype, sendcount, (uint8_t*)recvbuf, recvtype, recvcount);
    return MPI_SUCCESS;
}

int MPI_Gatherv(const void* sendbuf, int sendcount, MPI_Datatype sendtype, void* recvbuf,
                const int* recvcounts, const int* displs, MPI_Datatype recvtype, int root, MPI_Comm comm)
{
    SPDLOG_TRACE("MPI - MPI_Gatherv");
    subCommOnly(comm, "MPI_Gatherv");
    MpiWorld& world = getExecutingWorld();
    int rank = executingContext.getRank();
    int size = world.getSize();
    if (rank == root) {
        for (int r = 0; r < size; r++) {
            uint8_t* dst = (uint8_t*)recvbuf + (size_t)displs[r] * recvtype->size;
            if (r == root) {
                if (sendbuf != MPI_IN_PLACE) {
                    copyBytes(dst, sendbuf, (size_t)sendcount * sendtype->size);
                }
            } else {
                world.recv(r, root, dst, recvtype, recvcounts[r], nullptr, MpiMessageType::GATHER);
            }
        }
    } else {
        world.send(rank, root, (const uint8_t*)sendbuf, sendtype, sendcount, MpiMessageType::GATHER);
    }
    return MPI_SUCCESS;
}

int MPI_Allgather(const void* sendbuf, int sendcount, MPI_Datatype sendtype, void* recvbuf, int recvcount,
                  MPI_Datatype recvtype, MPI_Comm comm)
{
    SPDLOG_TRACE("MPI - MPI_Allgather");
    int rank = executingContext.getRank();
    if (auto sub = subOf(comm)) {
        const uint8_t* chunk = sendbuf == MPI_IN_PLACE
                                 ? (const uint8_t*)recvbuf + (size_t)sub->commRankOf(rank) * recvcount * recvtype->size
                                 : (const uint8_t*)sendbuf;
        sub->allGather(getExecutingWorld(), rank, chunk, (uint8_t*)recvbuf, recvtype, recvcount);
        return MPI_SUCCESS;
    }
    const uint8_t* send = (const uint8_t*)sendbuf;
    if (sendbuf == MPI_IN_PLACE) {
        send = (const uint8_t*)recvbuf + (size_t)rank * recvcount * recvtype->size;
        sendcount = recvcount;
        sendtype = recvtype;
    }
    getExecutingWorld().allGather(rank, send, sendtype, sendcount, (uint8_t*)recvbuf, recvtype, recvcount);
    return MPI_SUCCESS;
}

int MPI_Allgatherv(const void* sendbuf, int sendcount, MPI_Datatype sendtype, void* recvbuf,
                   const int* recvcounts, const int* displs, MPI_Datatype recvtype, MPI_Comm comm)
{
    SPDLOG_TRACE("MPI - MPI_Allgatherv");
    subCommOnly(comm, "MPI_Allgatherv");
    MpiWorld& world = getExecutingWorld();
    int size = world.getSize();
    // Equal, contiguous counts are a plain all-gather (fused device kernel)
    bool regular = true;
    for (int r = 0; r < size; r++) {
        regular = regular && recvcounts[r] == recvcounts[0] && displs[r] == r * recvcounts[0];
    }
    if (regular) {
        return MPI_Allgather(sendbuf, sendcount, sendtype, recvbuf, recvcounts[0], recvtype, comm);
    }
    // Irregular: gather to rank 0 then broadcast every block
    int rank = executingContext.getRank();
    MPI_Gatherv(sendbuf, sendcount, sendtype, recvbuf, recvcounts, displs, recvtype, 0, comm);
    for (int r = 0; r < size; r++) {
        uint8_t* block = (uint8_t*)recvbuf + (size_t)displs[r] * recvtype->size;
        world.broadcast(0, rank, block, recvtype, recvcounts[r], MpiMessageType::ALLGATHER);
    }
    return MPI_SUCCESS;
}

int MPI_Reduce(const void* sendbuf, void* recvbuf, int count, MPI_Datatype datatype, MPI_Op op, int root, MPI_Comm comm)
{
    SPDLOG_TRACE("MPI - MPI_Reduce all -> {}", root);
    if (accumulateOnlyOp(op)) {
        return MPI_ERR_OP;
    }
    if (auto sub = subOf(comm)) {
        sub->reduce(getExecutingWorld(), executingContext.getRank(), root, (const uint8_t*)resolveInPlace(sendbuf, recvbuf),
                    (uint8_t*)recvbuf, datatype, count, op);
        return MPI_SUCCESS;
    }
    getExecutingWorld().reduce(executingContext.getRank(), root, (uint8_t*)resolveInPlace(sendbuf, recvbuf),
                               (uint8_t*)recvbuf, datatype, count, op);
    return MPI_SUCCESS;
}

int MPI_Reduce_scatter(const void* sendbuf, void* recvbuf, const int* recvcounts, MPI_Datatype datatype,
                       MPI_Op op, MPI_Comm comm)
{
    SPDLOG_TRACE("MPI - MPI_Reduce_scatter");
    if (accumulateOnlyOp(op)) {
        return MPI_ERR_OP;
    }
    subCommOnly(comm, "MPI_Reduce_scatter");
    MpiWorld& world = getExecutingWorld();
    int size = world.getSize();
    int rank = executingContext.getRank();
    const void* send = sendbuf;
    if (sendbuf == MPI_IN_PLACE) {
        send = recvbuf;
    }
    bool equal = true;
    for (int r = 1; r < size; r++) {
        equal = equal && recvcounts[r] == recvcounts[0];
    }
    if (!equal) {
        // Irregular blocks: reduce everything at rank 0, then hand out the
        // blocks (the fused kernel only knows equal shards)
        size_t total = 0;
        std::vector<size_t> offsets(size);
        for (int r = 0; r < size; r++) {
            offsets[r] = total;
            total += (size_t)recvcounts[r];
        }
        std::vector<uint8_t> reduced(rank == 0 ? total * datatype->size : 0);
        HostStage hostSend;
        uint8_t* src = hostSend.in((const uint8_t*)send, total * datatype->size);
        world.reduce(rank, 0, src, reduced.data(), datatype, (int)total, op);
        if (rank == 0) {
            for (int r = 1; r < size; r++) {
                world.send(0, r, reduced.data() + offsets[r] * datatype->size, datatype, recvcounts[r], MpiMessageType::SCATTER);
            }
            copyBytes(recvbuf, reduced.data(), (size_t)recvcounts[0] * datatype->size);
        } else {
            world.recv(0, rank, (uint8_t*)recvbuf, datatype, recvcounts[rank], nullptr, MpiMessageType::SCATTER);
        }
        return MPI_SUCCESS;
    }
    world.reduceScatter(rank, (uint8_t*)send, (uint8_t*)recvbuf, datatype, recvcounts[0], op);
    return MPI_SUCCESS;
}

int MPI_Allreduce(const void* sendbuf, void* recvbuf, int count, MPI_Datatype datatype, MPI_Op op, MPI_Comm comm)
{
    SPDLOG_TRACE("MPI - MPI_Allreduce");
    if (accumulateOnlyOp(op)) {
        return MPI_ERR_OP;
    }
    if (auto sub = subOf(comm)) {
        sub->allReduce(getExecutingWorld(), executingContext.getRank(), (const uint8_t*)resolveInPlace(sendbuf, recvbuf),
                       (uint8_t*)recvbuf, datatype, count, op);
        return MPI_SUCCESS;
    }
    getExecutingWorld().allReduce(executingContext.getRank(), (uint8_t*)resolveInPlace(sendbuf, recvbuf),
                                  (uint8_t*)recvbuf, datatype, count, op);
    return MPI_SUCCESS;
}

int MPI_Scan(const void* sendbuf, void* recvbuf, int count, MPI_Datatype datatype, MPI_Op op, MPI_Comm comm)
{
    SPDLOG_TRACE("MPI - MPI_Scan");
    if (accumulateOnlyOp(op)) {
        return MPI_ERR_OP;
    }
    if (auto sub = subOf(comm)) {
        sub->scan(getExecutingWorld(), executingContext.getRank(), (const uint8_t*)resolveInPlace(sendbuf, recvbuf),
                  (uint8_t*)recvbuf, datatype, count, op);
        return MPI_SUCCESS;
    }
    getExecutingWorld().scan(executingContext.getRank(), (uint8_t*)resolveInPlace(sendbuf, recvbuf),
                             (uint8_t*)recvbuf, datatype, count, op);
    return MPI_SUCCESS;
}

int MPI_Alltoall(const void* sendbuf, int sendcount, MPI_Datatype sendtype, void* recvbuf, int recvcount,
                 MPI_Datatype recvtype, MPI_Comm comm)
{
    SPDLOG_TRACE("MPI - MPI_Alltoall");
    if (auto sub = subOf(comm)) {
        sub->allToAll(getExecutingWorld(), executingContext.getRank(), (const uint8_t*)sendbuf, (uint8_t*)recvbuf, sendtype, sendcount);
        return MPI_SUCCESS;
    }
    getExecutingWorld().allToAll(executingContext.getRank(), (uint8_t*)sendbuf, sendtype, sendcount,
                                 (uint8_t*)recvbuf, recvtype, recvcount);
    return MPI_SUCCESS;
}

int MPI_Alltoallv(const void* sendbuf, const int sendcounts[], const int sdispls[], MPI_Datatype sendtype,
                  void* recvbuf, const int recvcounts[], const int rdispls[], MPI_Datatype recvtype, MPI_Comm comm)
{
    SPDLOG_TRACE("MPI - MPI_Alltoallv");
    subCommOnly(comm, "MPI_Alltoallv");
    MpiWorld& world = getExecutingWorld();
    int rank = executingContext.getRank();
    int size = world.getSize();
    // Post every receive, send, then wait: cannot deadlock whatever the sizes
    std::vector<int> reqs;
    for (int r = 0; r < size; r++) {
        uint8_t* dst = (uint8_t*)recvbuf + (size_t)rdispls[r] * recvtype->size;
        const uint8_t* src = (const uint8_t*)sendbuf + (size_t)sdispls[r] * sendtype->size;
        if (r == rank) {
            copyBytes(dst, src, (size_t)sendcounts[r] * sendtype->size);
        } else {
            reqs.push_back(world.irecv(r, rank, dst, recvtype, recvcounts[r], MpiMessageType::ALLTOALL));
        }
    }
    for (int r = 0; r < size; r++) {
        if (r != rank) {
            const uint8_t* src = (const uint8_t*)sendbuf + (size_t)sdispls[r] * sendtype->size;
            world.send(rank, r, src, sendtype, sendcounts[r], MpiMessageType::ALLTOALL);
        }
    }
    for (int id : reqs) {
        world.awaitAsyncRequest(id);
    }
    return MPI_SUCCESS;
}

int MPI_Cart_create(MPI_Comm old_comm, int ndims, const int dims[], const int periods[], int reorder, MPI_Comm* comm)
{
    SPDLOG_TRACE("MPI - MPI_Cart_create");
    subCommOnly(old_comm, "MPI_Cart_create");
    // The grid is remembered by the world; the communicator stays the world
    int rank = executingContext.getRank();
    std::vector<int> p(std::max(ndims, 2), 1);
    std::vector<int> c(std::max(ndims, 2), 0);
    std::vector<int> d(dims, dims + ndims);
    d.resize(std::max(ndims, 2), 1);
    getExecutingWorld().getCartesianRank(rank, ndims, d.data(), p.data(), c.data());
    *comm = old_comm;
    return MPI_SUCCESS;
}

int MPI_Cart_rank(MPI_Comm comm, int coords[], int* rank)
{
    SPDLOG_TRACE("MPI - MPI_Cart_rank");
    getExecutingWorld().getRankFromCoords(rank, coords);
    return MPI_SUCCESS;
}

int MPI_Cart_get(MPI_Comm comm, int maxdims, int dims[], int periods[], int coords[])
{
    SPDLOG_TRACE("MPI - MPI_Cart_get");
    if (maxdims > MPI_CART_MAX_DIMENSIONS + 1) {
        SPDLOG_ERROR("Unexpected number of max. dimensions: {}", maxdims);
        throw std::runtime_error("Bad dimensions in MPI_Cart_get");
    }
    // The grid set by MPI_Cart_create is authoritative; before that the caller's
    // dims are taken as input (what the reference does)
    auto& world = getExecutingWorld();
    std::vector<int> d(std::max(maxdims, 2), 1);
    std::vector<int> p(std::max(maxdims, 2), 1);
    std::vector<int> c(std::max(maxdims, 2), 0);
    if (!world.getCartesianDims(d.data())) {
        std::copy(dims, dims + maxdims, d.begin());
    }
    world.getCartesianRank(executingContext.getRank(), maxdims, d.data(), p.data(), c.data());
    std::copy(d.begin(), d.begin() + maxdims, dims);
    std::copy(p.begin(), p.begin() + maxdims, periods);
    std::copy(c.begin(), c.begin() + maxdims, coords);
    return MPI_SUCCESS;
}

int MPI_Cart_shift(MPI_Comm comm, int direction, int disp, int* rank_source, int* rank_dest)
{
    SPDLOG_TRACE("MPI - MPI_Cart_shift");
    getExecutingWorld().shiftCartesianCoords(executingContext.getRank(), direction, disp, rank_source, rank_dest);
    return MPI_SUCCESS;
}

int MPI_Type_size(MPI_Datatype type, int* size)
{
    SPDLOG_TRACE("MPI - MPI_Type_size");
    *size = type->size;
    return MPI_SUCCESS;
}

int MPI_Type_free(MPI_Datatype* datatype)
{
    SPDLOG_TRACE("MPI - MPI_Type_free");
    // Only derived types can be freed (the reference throws for all of them,
    // mpi_native.cpp:541-545)
    if (datatype == nullptr || *datatype == nullptr || (*datatype)->id < FAABRIC_DERIVED_TYPE_BASE) {
        return MPI_ERR_ARG;
    }
    unregisterContiguousType((*datatype)->id);
    delete *datatype;
    *datatype = MPI_DATATYPE_NULL;
    return MPI_SUCCESS;
}

int MPI_Type_contiguous(int count, MPI_Datatype oldtype, MPI_Datatype* newtype)
{
    SPDLOG_TRACE("MPI - MPI_Type_contiguous");
    // (a no-op in the reference, which leaves *newtype untouched)
    int baseId = oldtype->id, per = 1;
    if (oldtype->id >= FAABRIC_DERIVED_TYPE_BASE && !getContiguousType(oldtype->id, &baseId, &per)) {
        return MPI_ERR_ARG;
    }
    int id = registerContiguousType(baseId, count * per);
    *newtype = new faabric_datatype_t{ id, count * oldtype->size };
    return MPI_SUCCESS;
}

int MPI_Type_commit(MPI_Datatype* type)
{
    SPDLOG_TRACE("MPI - MPI_Type_commit");
    return MPI_SUCCESS;
}

int MPI_Op_create(MPI_User_function* user_fn, int commute, MPI_Op* op)
{
    SPDLOG_TRACE("MPI - MPI_Op_create");
    // (the reference throws "not implemented", mpi_native.cpp:764-772)
    *op = new faabric_op_t{ registerUserOp(user_fn, commute != 0) };
    return MPI_SUCCESS;
}

int MPI_Op_free(MPI_Op* op)
{
    SPDLOG_TRACE("MPI - MPI_Op_free");
    if (op == nullptr || *op == nullptr || !isUserOp(*op)) {
        // predefined operations cannot be freed
        return MPI_ERR_OP;
    }
    unregisterUserOp((*op)->id);
    delete *op;
    *op = MPI_OP_NULL;
    return MPI_SUCCESS;
}

int MPI_Alloc_mem(MPI_Aint size, MPI_Info info, void* baseptr)
{
    SPDLOG_TRACE("MPI - MPI_Alloc_mem");
    if (info == MPI_INFO_FAABRIC_DEVICE) {
        // "Special memory" in the MPI sense: the rank's symmetric heap in HBM,
        // mapped into every peer, so collectives on it need no staging
        void* p = getExecutingWorld().deviceAlloc(executingContext.getRank(), (size_t)size);
        if (p == nullptr) {
            return MPI_ERR_NO_MEM;
        }
        *((void**)baseptr) = p;
        return MPI_SUCCESS;
    }
    if (info != MPI_INFO_NULL) {
        throw std::runtime_error("Non-null info not supported");
    }
    *((void**)baseptr) = malloc((size_t)size);
    return MPI_SUCCESS;
}

int MPI_Free_mem(void* base)
{
    SPDLOG_TRACE("MPI - MPI_Free_mem");
    if (base == nullptr) {
        return MPI_SUCCESS;
    }
    if (MpiWorld::isDevicePointer(base)) {
        getExecutingWorld().deviceFree(executingContext.getRank(), base);
    } else {
        free(base);
    }
    return MPI_SUCCESS;
}

int MPI_Iallreduce(const void* sendbuf, void* recvbuf, int count, MPI_Datatype datatype, MPI_Op op, MPI_Comm comm, MPI_Request* request)
{
    SPDLOG_TRACE("MPI - MPI_Iallreduce");
    if (accumulateOnlyOp(op)) {
        return MPI_ERR_OP;
    }
    subCommOnly(comm, "MPI_Iallreduce");
    int id = getExecutingWorld().iAllReduce(executingContext.getRank(),
                                            (uint8_t*)resolveInPlace(sendbuf, recvbuf),
                                            (uint8_t*)recvbuf,
                                            datatype,
                                            count,
                                            op);
    auto* r = new faabric_request_t{ id };
    requestTable()[id] = r;
    *request = r;
    return MPI_SUCCESS;
}

int MPI_Reduce_scatter_block(const void* sendbuf, void* recvbuf, int recvcount, MPI_Datatype datatype,
                             MPI_Op op, MPI_Comm comm)
{
    SPDLOG_TRACE("MPI - MPI_Reduce_scatter_block");
    if (accumulateOnlyOp(op)) {
        return MPI_ERR_OP;
    }
    subCommOnly(comm, "MPI_Reduce_scatter_block");
    getExecutingWorld().reduceScatter(executingContext.getRank(), (uint8_t*)resolveInPlace(sendbuf, recvbuf),
                                      (uint8_t*)recvbuf, datatype, recvcount, op);
    return MPI_SUCCESS;
}

int MPI_Ireduce_scatter_block(const void* sendbuf, void* recvbuf, int recvcount, MPI_Datatype datatype,
                              MPI_Op op, MPI_Comm comm, MPI_Request* request)
{
    SPDLOG_TRACE("MPI - MPI_Ireduce_scatter_block");
    if (accumulateOnlyOp(op)) {
        return MPI_ERR_OP;
    }
    subCommOnly(comm, "MPI_Ireduce_scatter_block");
    int id = getExecutingWorld().iReduceScatter(executingContext.getRank(),
                                                (uint8_t*)resolveInPlace(sendbuf, recvbuf),
                                                (uint8_t*)recvbuf,
                                                datatype,
                                                recvcount,
                                                op);
    auto* r = new faabric_request_t{ id };
    requestTable()[id] = r;
    *request = r;
    return MPI_SUCCESS;
}

int MPI_Iallgather(const void* sendbuf, int sendcount, MPI_Datatype sendtype, void* recvbuf, int recvcount,
                   MPI_Datatype recvtype, MPI_Comm comm, MPI_Request* request)
{
    SPDLOG_TRACE("MPI - MPI_Iallgather");
    subCommOnly(comm, "MPI_Iallgather");
    int rank = executingContext.getRank();
    const uint8_t* send = (const uint8_t*)sendbuf;
    if (sendbuf == MPI_IN_PLACE) {
        send = (const uint8_t*)recvbuf + (size_t)rank * recvcount * recvtype->size;
        sendcount = recvcount;
        sendtype = recvtype;
    }
    int id = getExecutingWorld().iAllGather(rank, send, sendtype, sendcount, (uint8_t*)recvbuf, recvtype, recvcount);
    auto* r = new faabric_request_t{ id };
    requestTable()[id] = r;
    *request = r;
    return MPI_SUCCESS;
}

int MPI_Get_processor_name(char* name, int* resultlen)
{
    SPDLOG_TRACE("MPI - MPI_Get_processor_name");
    std::string host = faabric::util::getSystemConfig().endpointHost;
    strncpy(name, host.c_str(), MPI_MAX_PROCESSOR_NAME - 1);
    name[MPI_MAX_PROCESSOR_NAME - 1] = '\0';
    *resultlen = (int)std::min<size_t>(host.size(), MPI_MAX_PROCESSOR_NAME - 1);
    return MPI_SUCCESS;
}

double MPI_Wtime()
{
    SPDLOG_TRACE("MPI - MPI_Wtime");
    return getExecutingWorld().getWTime();
}

int MPI_Win_get_attr(MPI_Win win, int win_keyval, void* attribute_val, int* flag)
{
    SPDLOG_TRACE("MPI - MPI_Win_get_attr");
    *flag = 1;
    switch (win_keyval) {
        case MPI_WIN_BASE:
            *((void**)attribute_val) = win->basePtr;
            break;
        case MPI_WIN_SIZE: {
            // (the handle's `size` field is an int as in the reference; the
            // world keeps the real extent for windows beyond 2 GiB)
            void* base = nullptr;
            int64_t bytes = win->size;
            int unit = 0;
            if (win->id > 0) {
                getExecutingWorld().winQuery(win->id, win->rank, &base, &bytes, &unit);
            }
            *((MPI_Aint*)attribute_val) = (MPI_Aint)bytes;
            break;
        }
        case MPI_WIN_DISP_UNIT:
            *((int*)attribute_val) = win->dispUnit;
            break;
        default:
            throw std::runtime_error("Unrecognised window attribute type " + std::to_string(win_keyval));
    }
    return MPI_SUCCESS;
}

// ---- one-sided communication.  The reference declares these and throws
// (tests/dist/mpi/mpi_native.cpp:649-683); see MpiWorld::winCreate. ----
int MPI_Win_fence(int assert, MPI_Win win)
{
    SPDLOG_TRACE("MPI - MPI_Win_fence");
    if (win == nullptr) {
        return MPI_ERR_WIN;
    }
    MpiWorld& world = getExecutingWorld();
    if (world.winInPassiveEpoch(executingContext.getRank(), win->id)) {
        return MPI_ERR_RMA_SYNC;
    }
    world.winFence(executingContext.getRank(), win->id);
    return MPI_SUCCESS;
}

// ---- passive-target synchronisation; see MpiWorld::winLock ----
int MPI_Win_lock(int lock_type, int rank, int assert, MPI_Win win)
{
    SPDLOG_TRACE("MPI - MPI_Win_lock");
    if (win == nullptr) {
        return MPI_ERR_WIN;
    }
    return getExecutingWorld().winLock(executingContext.getRank(), win->id, lock_type, rank, assert);
}

int MPI_Win_unlock(int rank, MPI_Win win)
{
    SPDLOG_TRACE("MPI - MPI_Win_unlock");
    if (win == nullptr) {
        return MPI_ERR_WIN;
    }
    return getExecutingWorld().winUnlock(executingContext.getRank(), win->id, rank);
}

int MPI_Win_lock_all(int assert, MPI_Win win)
{
    SPDLOG_TRACE("MPI - MPI_Win_lock_all");
    if (win == nullptr) {
        return MPI_ERR_WIN;
    }
    return getExecutingWorld().winLockAll(executingContext.getRank(), win->id, assert);
}

int MPI_Win_unlock_all(MPI_Win win)
{
    SPDLOG_TRACE("MPI - MPI_Win_unlock_all");
    if (win == nullptr) {
        return MPI_ERR_WIN;
    }
    return getExecutingWorld().winUnlockAll(executingContext.getRank(), win->id);
}

// (target -1: every target of the epoch)
static int winFlush(int target, MPI_Win win)
{
    if (win == nullptr) {
        return MPI_ERR_WIN;
    }
    return getExecutingWorld().winFlush(executingContext.getRank(), win->id, target);
}

int MPI_Win_flush(int rank, MPI_Win win)
{
    SPDLOG_TRACE("MPI - MPI_Win_flush");
    return rank < 0 ? MPI_ERR_RANK : winFlush(rank, win);
}

int MPI_Win_flush_all(MPI_Win win)
{
    SPDLOG_TRACE("MPI - MPI_Win_flush_all");
    return winFlush(-1, win);
}

// Completing at the target too is allowed: the local variants are the same
int MPI_Win_flush_local(int rank, MPI_Win win)
{
    SPDLOG_TRACE("MPI - MPI_Win_flush_local");
    return rank < 0 ? MPI_ERR_RANK : winFlush(rank, win);
}

int MPI_Win_flush_local_all(MPI_Win win)
{
    SPDLOG_TRACE("MPI - MPI_Win_flush_local_all");
    return winFlush(-1, win);
}

// Loads and stores through MPI_Win_shared_query pointers before the call are
// ordered before those after it
int MPI_Win_sync(MPI_Win win)
{
    SPDLOG_TRACE("MPI - MPI_Win_sync");
    if (win == nullptr) {
        return MPI_ERR_WIN;
    }
    std::atomic_thread_fence(std::memory_order_seq_cst);
    return MPI_SUCCESS;
}

int MPI_Get(void* origin_addr, int origin_count, MPI_Datatype origin_datatype, int target_rank,
            MPI_Aint target_disp, int target_count, MPI_Datatype target_datatype, MPI_Win win)
{
    SPDLOG_TRACE("MPI - MPI_Get");
    if (win == nullptr) {
        return MPI_ERR_WIN;
    }
    const size_t bytes = (size_t)origin_count * origin_datatype->size;
    if (bytes != (size_t)target_count * target_datatype->size) {
        return MPI_ERR_ARG;
    }
    getExecutingWorld().winGet(executingContext.getRank(), win->id, (uint8_t*)origin_addr, bytes, target_rank, target_disp);
    return MPI_SUCCESS;
}

int MPI_Put(const void* origin_addr, int origin_count, MPI_Datatype origin_datatype, int target_rank,
            MPI_Aint target_disp, int target_count, MPI_Datatype target_datatype, MPI_Win win)
{
    SPDLOG_TRACE("MPI - MPI_Put");
    if (win == nullptr) {
        return MPI_ERR_WIN;
    }
    const size_t bytes = (size_t)origin_count * origin_datatype->size;
    if (bytes != (size_t)target_count * target_datatype->size) {
        return MPI_ERR_ARG;
    }
    getExecutingWorld().winPut(executingContext.getRank(), win->id, (const uint8_t*)origin_addr, bytes, target_rank, target_disp);
    return MPI_SUCCESS;
}

int MPI_Accumulate(const void* origin_addr, int origin_count, MPI_Datatype origin_datatype, int target_rank,
                   MPI_Aint target_disp, int target_count, MPI_Datatype target_datatype, MPI_Op op, MPI_Win win)
{
    SPDLOG_TRACE("MPI - MPI_Accumulate");
    if (op == MPI_NO_OP) {
        return MPI_ERR_OP; // only MPI_Get_accumulate / MPI_Fetch_and_op take it
    }
    return getAccumulate(origin_addr, origin_count, origin_datatype, nullptr, 0, nullptr, target_rank, target_disp,
                         target_count, target_datatype, op, win);
}

int MPI_Get_accumulate(const void* origin_addr, int origin_count, MPI_Datatype origin_datatype, void* result_addr,
                       int result_count, MPI_Datatype result_datatype, int target_rank, MPI_Aint target_disp,
                       int target_count, MPI_Datatype target_datatype, MPI_Op op, MPI_Win win)
{
    SPDLOG_TRACE("MPI - MPI_Get_accumulate");
    if (result_addr == nullptr && result_count > 0) {
        return MPI_ERR_ARG;
    }
    return getAccumulate(origin_addr, origin_count, origin_datatype, result_addr, result_count, result_datatype,
                         target_rank, target_disp, target_count, target_datatype, op, win);
}

int MPI_Fetch_and_op(const void* origin_addr, void* result_addr, MPI_Datatype datatype, int target_rank,
                     MPI_Aint target_disp, MPI_Op op, MPI_Win win)
{
    SPDLOG_TRACE("MPI - MPI_Fetch_and_op");
    if (result_addr == nullptr) {
        return MPI_ERR_ARG;
    }
    return getAccumulate(origin_addr, 1, datatype, result_addr, 1, datatype, target_rank, target_disp, 1, datatype, op, win);
}

int MPI_Compare_and_swap(const void* origin_addr, const void* compare_addr, void* result_addr, MPI_Datatype datatype,
                         int target_rank, MPI_Aint target_disp, MPI_Win win)
{
    SPDLOG_TRACE("MPI - MPI_Compare_and_swap");
    if (win == nullptr) {
        return MPI_ERR_WIN;
    }
    MPI_Datatype base = nullptr;
    int per = 0;
    if (!baseTypeOf(datatype, &base, &per) || per != 1) {
        return MPI_ERR_ARG;
    }
    return getExecutingWorld().winCompareSwap(executingContext.getRank(), win->id, (const uint8_t*)origin_addr,
                                              (const uint8_t*)compare_addr, (uint8_t*)result_addr, base, target_rank,
                                              (int64_t)target_disp);
}

// ---- request-based one-sided operations; see MpiWorld::winRputGet.  They
// need a passive epoch that covers the target (MPI_ERR_RMA_SYNC otherwise) ----
int MPI_Rput(const void* origin_addr, int origin_count, MPI_Datatype origin_datatype, int target_rank,
             MPI_Aint target_disp, int target_count, MPI_Datatype target_datatype, MPI_Win win, MPI_Request* request)
{
    SPDLOG_TRACE("MPI - MPI_Rput");
    return requestPutGet(const_cast<void*>(origin_addr), origin_count, origin_datatype, target_rank, target_disp,
                         target_count, target_datatype, win, request, false);
}

int MPI_Rget(void* origin_addr, int origin_count, MPI_Datatype origin_datatype, int target_rank,
             MPI_Aint target_disp, int target_count, MPI_Datatype target_datatype, MPI_Win win, MPI_Request* request)
{
    SPDLOG_TRACE("MPI - MPI_Rget");
    return requestPutGet(origin_addr, origin_count, origin_datatype, target_rank, target_disp, target_count,
                         target_datatype, win, request, true);
}

int MPI_Raccumulate(const void* origin_addr, int origin_count, MPI_Datatype origin_datatype, int target_rank,
                    MPI_Aint target_disp, int target_count, MPI_Datatype target_datatype, MPI_Op op, MPI_Win win,
                    MPI_Request* request)
{
    SPDLOG_TRACE("MPI - MPI_Raccumulate");
    if (win == nullptr) {
        return MPI_ERR_WIN;
    }
    if (request == nullptr) {
        return MPI_ERR_ARG;
    }
    if (op == MPI_NO_OP) {
        return MPI_ERR_OP; // as MPI_Accumulate
    }
    return getAccumulate(origin_addr, origin_count, origin_datatype, nullptr, 0, nullptr, target_rank, target_disp,
                         target_count, target_datatype, op, win, request);
}

int MPI_Rget_accumulate(const void* origin_addr, int origin_count, MPI_Datatype origin_datatype, void* result_addr,
                        int result_count, MPI_Datatype result_datatype, int target_rank, MPI_Aint target_disp,
                        int target_count, MPI_Datatype target_datatype, MPI_Op op, MPI_Win win, MPI_Request* request)
{
    SPDLOG_TRACE("MPI - MPI_Rget_accumulate");
    if (win == nullptr) {
        return MPI_ERR_WIN;
    }
    if (request == nullptr || (result_addr == nullptr && result_count > 0)) {
        return MPI_ERR_ARG;
    }
    return getAccumulate(origin_addr, origin_count, origin_datatype, result_addr, result_count, result_datatype,
                         target_rank, target_disp, target_count, target_datatype, op, win, request);
}

int MPI_Win_free(MPI_Win* win)
{
    SPDLOG_TRACE("MPI - MPI_Win_free");
    if (win == nullptr || *win == nullptr) {
        return MPI_ERR_WIN;
    }
    if (getExecutingWorld().winInPassiveEpoch(executingContext.getRank(), (*win)->id)) {
        return MPI_ERR_RMA_SYNC;
    }
    getExecutingWorld().winFree(executingContext.getRank(), (*win)->id);
    if ((*win)->ownedPtr != nullptr) {
        MPI_Free_mem((*win)->ownedPtr);
    }
    delete *win;
    *win = nullptr;
    return MPI_SUCCESS;
}

int MPI_Win_create(void* base, MPI_Aint size, int disp_unit, MPI_Info info, MPI_Comm comm, MPI_Win* win)
{
    SPDLOG_TRACE("MPI - MPI_Win_create");
    subCommOnly(comm, "MPI_Win_create");
    MpiWorld& world = getExecutingWorld();
    const int rank = executingContext.getRank();
    int winId = world.winCreate(rank, base, (int64_t)size, disp_unit);
    *win = new faabric_win_t{ world.getId(), rank, (int)std::min<MPI_Aint>(size, INT32_MAX), base, disp_unit, winId, nullptr };
    return MPI_SUCCESS;
}

int MPI_Win_allocate_shared(MPI_Aint size, int disp_unit, MPI_Info info, MPI_Comm comm, void* baseptr, MPI_Win* win)
{
    SPDLOG_TRACE("MPI - MPI_Win_allocate_shared");
    subCommOnly(comm, "MPI_Win_allocate_shared");
    MpiWorld& world = getExecutingWorld();
    if (!world.allRanksLocal()) {
        // Load/store access needs one address space: ranks of this world
        // live in several worker processes
        SPDLOG_ERROR("MPI_Win_allocate_shared on a world that spans worker processes");
        return MPI_ERR_OTHER;
    }
    // MPI_INFO_FAABRIC_DEVICE puts the segment in the rank's symmetric heap
    void* mem = nullptr;
    if (info == MPI_INFO_FAABRIC_DEVICE) {
        int rc = MPI_Alloc_mem(size, info, &mem);
        if (rc != MPI_SUCCESS) {
            return rc;
        }
    } else {
        // cache-line aligned, zeroed
        size_t rounded = ((size_t)size + 63) & ~(size_t)63;
        if (posix_memalign(&mem, 64, std::max<size_t>(rounded, 64)) != 0) {
            return MPI_ERR_NO_MEM;
        }
        memset(mem, 0, std::max<size_t>(rounded, 64));
    }
    const int rank = executingContext.getRank();
    int winId = world.winCreate(rank, mem, (int64_t)size, disp_unit);
    *((void**)baseptr) = mem;
    *win = new faabric_win_t{ world.getId(), rank, (int)std::min<MPI_Aint>(size, INT32_MAX), mem, disp_unit, winId, mem };
    return MPI_SUCCESS;
}

int MPI_Win_shared_query(MPI_Win win, int rank, MPI_Aint* size, int* disp_unit, void* baseptr)
{
    SPDLOG_TRACE("MPI - MPI_Win_shared_query");
    if (win == nullptr) {
        return MPI_ERR_WIN;
    }
    void* base = nullptr;
    int64_t bytes = 0;
    int unit = 0;
    if (!getExecutingWorld().winQuery(win->id, rank, &base, &bytes, &unit)) {
        return MPI_ERR_RANK;
    }
    *size = (MPI_Aint)bytes;
    *disp_unit = unit;
    *((void**)baseptr) = base;
    return MPI_SUCCESS;
}

int MPI_Comm_dup(MPI_Comm comm, MPI_Comm* newcomm)
{
    SPDLOG_TRACE("MPI - MPI_Comm_dup");
    // One communication context per world: the duplicate is the same handle
    // (the reference throws, mpi_native.cpp:686-690)
    if (comm != MPI_COMM_WORLD) {
        throw std::runtime_error("MPI_Comm_dup is only supported on MPI_COMM_WORLD");
    }
    *newcomm = comm;
    return MPI_SUCCESS;
}

// Fortran handles are the communicator ids
MPI_Fint MPI_Comm_c2f(MPI_Comm comm)
{
    return comm == nullptr ? FAABRIC_COMM_NULL : comm->id;
}

MPI_Comm MPI_Comm_f2c(MPI_Fint comm)
{
    if (comm == FAABRIC_COMM_WORLD) {
        return MPI_COMM_WORLD;
    }
    if (comm == FAABRIC_COMM_NULL || getSubCommunicator(comm) == nullptr) {
        return MPI_COMM_NULL;
    }
    // a fresh handle; release it with MPI_Comm_free like any other
    return new faabric_communicator_t{ comm };
}

// ---- communicator and group management.  The reference declares these
// and throws (mpi_native.cpp:686-735); see src/mpi/subcomm.h ----
int MPI_Comm_split(MPI_Comm comm, int color, int key, MPI_Comm* newcomm)
{
    SPDLOG_TRACE("MPI - MPI_Comm_split");
    MpiWorld& world = getExecutingWorld();
    const int me = executingContext.getRank();
    std::vector<int> parentRanks = ranksOf(comm);
    const int n = (int)parentRanks.size();
    const int parentId = comm->id;
    const int seq = commCreateSeq[parentId]++;
    // Everybody learns everybody's (color, key)
    int mine[2] = { color, key };
    std::vector<int> all(2 * (size_t)n);
    faabric_datatype_t* intType = getFaabricDatatypeFromId(FAABRIC_INT);
    if (auto sub = subOf(comm)) {
        sub->allGather(world, me, (const uint8_t*)mine, (uint8_t*)all.data(), intType, 2);
    } else {
        world.allGather(me, (const uint8_t*)mine, intType, 2, (uint8_t*)all.data(), intType, 2);
    }
    if (color == MPI_UNDEFINED) {
        *newcomm = MPI_COMM_NULL;
        return MPI_SUCCESS;
    }
    // Members of my color, ordered by key then by rank in the parent
    std::vector<std::pair<std::pair<int, int>, int>> members;
    for (int r = 0; r < n; r++) {
        if (all[2 * r] == color) {
            members.push_back({ { all[2 * r + 1], r }, parentRanks[r] });
        }
    }
    std::sort(members.begin(), members.end());
    std::vector<int> worldRanks;
    for (auto& m : members) {
        worldRanks.push_back(m.second);
    }
    *newcomm = makeCommHandle(parentId, seq, (uint64_t)(uint32_t)color, worldRanks);
    return MPI_SUCCESS;
}

int MPI_Comm_split_type(MPI_Comm comm, int split_type, int key, MPI_Info info, MPI_Comm* newcomm)
{
    SPDLOG_TRACE("MPI - MPI_Comm_split_type");
    if (split_type != MPI_COMM_TYPE_SHARED) {
        throw std::runtime_error("MPI_Comm_split_type: only MPI_COMM_TYPE_SHARED is supported");
    }
    // Ranks that share an address space: those served by the same worker
    // process.  Colour = lowest world rank on my host.
    MpiWorld& world = getExecutingWorld();
    const std::string myHost = world.getHostForRank(executingContext.getRank());
    int color = executingContext.getRank();
    for (int r = 0; r < world.getSize(); r++) {
        if (world.getHostForRank(r) == myHost) {
            color = r;
            break;
        }
    }
    return MPI_Comm_split(comm, color, key, newcomm);
}

int MPI_Comm_group(MPI_Comm comm, MPI_Group* group)
{
    SPDLOG_TRACE("MPI - MPI_Comm_group");
    *group = new faabric_group_t{ registerGroup(ranksOf(comm)) };
    return MPI_SUCCESS;
}

int MPI_Group_incl(MPI_Group group, int n, const int ranks[], MPI_Group* newgroup)
{
    SPDLOG_TRACE("MPI - MPI_Group_incl");
    std::vector<int> parent;
    if (group == nullptr || !getGroup(group->id, parent)) {
        return MPI_ERR_ARG;
    }
    std::vector<int> subset;
    for (int i = 0; i < n; i++) {
        if (ranks[i] < 0 || ranks[i] >= (int)parent.size()) {
            return MPI_ERR_RANK;
        }
        subset.push_back(parent[ranks[i]]);
    }
    *newgroup = new faabric_group_t{ registerGroup(std::move(subset)) };
    return MPI_SUCCESS;
}

int MPI_Group_free(MPI_Group* group)
{
    SPDLOG_TRACE("MPI - MPI_Group_free");
    if (group == nullptr || *group == nullptr) {
        return MPI_ERR_ARG;
    }
    freeGroup((*group)->id);
    delete *group;
    *group = nullptr;
    return MPI_SUCCESS;
}

static uint64_t hashRanks(const std::vector<int>& ranks)
{
    uint64_t h = 1469598103934665603ULL;
    for (int r : ranks) {
        h = (h ^ (uint64_t)(uint32_t)r) * 1099511628211ULL;
    }
    return h;
}

int MPI_Comm_create(MPI_Comm comm, MPI_Group group, MPI_Comm* newcomm)
{
    SPDLOG_TRACE("MPI - MPI_Comm_create");
    // Collective over `comm`; ranks outside the group get MPI_COMM_NULL
    const int parentId = comm->id;
    const int seq = commCreateSeq[parentId]++;
    std::vector<int> members;
    if (group == nullptr || !getGroup(group->id, members)) {
        return MPI_ERR_ARG;
    }
    const int me = executingContext.getRank();
    if (std::find(members.begin(), members.end(), me) == members.end()) {
        *newcomm = MPI_COMM_NULL;
        return MPI_SUCCESS;
    }
    *newcomm = makeCommHandle(parentId, seq, hashRanks(members), members);
    return MPI_SUCCESS;
}

int MPI_Comm_create_group(MPI_Comm comm, MPI_Group group, int tag, MPI_Comm* newcomm)
{
    SPDLOG_TRACE("MPI - MPI_Comm_create_group");
    // Collective over the GROUP only: the tag (not a per-parent counter, which
    // non-members do not advance) tells concurrent creations apart
    std::vector<int> members;
    if (group == nullptr || !getGroup(group->id, members)) {
        return MPI_ERR_ARG;
    }
    const int me = executingContext.getRank();
    if (std::find(members.begin(), members.end(), me) == members.end()) {
        *newcomm = MPI_COMM_NULL;
        return MPI_SUCCESS;
    }
    *newcomm = makeCommHandle(comm->id, -1 - tag, hashRanks(members), members);
    return MPI_SUCCESS;
}

int MPI_Comm_free(MPI_Comm* comm)
{
    SPDLOG_TRACE("MPI - MPI_Comm_free");
    if (comm == nullptr || *comm == nullptr) {
        return MPI_ERR_ARG;
    }
    // The predefined communicators (and cartesian views of the world) are not
    // owned by the caller; handles of sub-communicators are
    if ((*comm)->id != FAABRIC_COMM_WORLD && (*comm)->id != FAABRIC_COMM_NULL) {
        // frees this rank's signal slot of the fused device path
        if (auto sub = getSubCommunicator((*comm)->id)) {
            sub->releaseDevice(executingContext.getRank());
        }
        delete *comm;
    }
    *comm = MPI_COMM_NULL;
    return MPI_SUCCESS;
}

} // extern "C"
