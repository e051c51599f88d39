// Sub-communicators and groups (MPI_Comm_split / _create / _group ...).
//
// The reference declares these calls and throws "not implemented"
// (tests/dist/mpi/mpi_native.cpp:686-735).  Here a sub-communicator is an
// ordered list of world ranks.  On device buffers, MPI_Bcast, MPI_Reduce,
// MPI_Allreduce, MPI_Scan, MPI_Gather, MPI_Scatter, MPI_Allgather and
// MPI_Alltoall run the world's fused kernels over a child of the world device
// communicator (Communicator::subset), on a signal slot the members agree on
// at their first such call.  Everything else, and every call when no slot is
// free on all members, is built from the world's point-to-point layer, so it
// works for ranks in one process (queues / peer memory) and across worker
// processes (TCP) alike, on host and device buffers.
#pragma once

#include <faabric/device/communicator.h>
#include <faabric/mpi/MpiWorld.h>
#include <faabric/mpi/mpi.h>

#include <map>
#include <memory>
#include <mutex>
#include <vector>

namespace faabric::mpi {

class SubCommunicator
{
  public:
    SubCommunicator(int commIdIn, int worldIdIn, std::vector<int> worldRanksIn);

    int id() const { return commId; }

    int worldId() const { return world; }

    int size() const { return (int)worldRanks.size(); }

    const std::vector<int>& ranks() const { return worldRanks; }

    // -1 when the world rank is not a member
    int commRankOf(int worldRank) const;

    // Throws on a rank outside the communicator
    int worldRankOf(int commRank) const;

    // ---- collectives; `me` is the caller's WORLD rank, roots are COMM ranks ----
    void barrier(MpiWorld& w, int me);

    void broadcast(MpiWorld& w, int me, int root, uint8_t* buffer, faabric_datatype_t* dt, int count);

    void reduce(MpiWorld& w, int me, int root, const uint8_t* send, uint8_t* recv, faabric_datatype_t* dt, int count, faabric_op_t* op);

    void allReduce(MpiWorld& w, int me, const uint8_t* send, uint8_t* recv, faabric_datatype_t* dt, int count, faabric_op_t* op);

    void scan(MpiWorld& w, int me, const uint8_t* send, uint8_t* recv, faabric_datatype_t* dt, int count, faabric_op_t* op);

    // send == nullptr on the root means "already in place in recv"
    void gather(MpiWorld& w, int me, int root, const uint8_t* send, uint8_t* recv, faabric_datatype_t* dt, int count);

    void scatter(MpiWorld& w, int me, int root, const uint8_t* send, uint8_t* recv, faabric_datatype_t* dt, int count);

    void allGather(MpiWorld& w, int me, const uint8_t* send, uint8_t* recv, faabric_datatype_t* dt, int count);

    void allToAll(MpiWorld& w, int me, const uint8_t* send, uint8_t* recv, faabric_datatype_t* dt, int count);

    // ---- fused device path ----
    // This rank's child of its world device communicator over the members
    // (null: this communicator stays on the host path).  The first call of a
    // rank agrees on a slot with the other members: collective, so call it
    // only from a collective that every member enters with device buffers.
    std::shared_ptr<faabric::device::Communicator> deviceComm(MpiWorld& w, int me);

    // Releases the child of world rank `me` (MPI_Comm_free); later calls of
    // that rank take the host path
    void releaseDevice(int me);

  private:
    int commId;
    int world;
    std::vector<int> worldRanks;

    // Per world rank of this process: the slot agreement has run (`decided`)
    // and its result (null child: host path).  Shared by the process's ranks.
    struct DeviceState
    {
        bool decided = false;
        std::shared_ptr<faabric::device::Communicator> child;
    };
    std::mutex deviceMx;
    std::map<int, DeviceState> device;
};

// Process-wide registry.  Ids are derived from (world, parent, sequence number
// of the creating call, discriminator) so every member computes the same id
// without talking to the others.
int deriveCommId(int worldId, int parentCommId, int sequence, uint64_t discriminator);

std::shared_ptr<SubCommunicator> registerSubCommunicator(int commId, int worldId, const std::vector<int>& worldRanks);

// nullptr for MPI_COMM_WORLD / unknown ids
std::shared_ptr<SubCommunicator> getSubCommunicator(int commId);

// worldId < 0 clears the communicators of every world
void clearSubCommunicators(int worldId);

// Groups are local objects: plain lists of world ranks
int registerGroup(std::vector<int> worldRanks);

bool getGroup(int groupId, std::vector<int>& worldRanks);

void freeGroup(int groupId);

}
