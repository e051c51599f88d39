#include <faabric/mpi/MpiContext.h>
#include <faabric/mpi/MpiWorldRegistry.h>

#include "subcomm.h"
#include <faabric/util/config.h>
#include <faabric/util/gids.h>
#include <faabric/util/logging.h>

namespace faabric::mpi {

MpiWorldRegistry& getMpiWorldRegistry()
{
    static MpiWorldRegistry reg;
    return reg;
}

MpiWorld& MpiWorldRegistry::createWorld(faabric::Message& msg, int worldId, std::string hostOverride)
{
    if (worldMap.contains(worldId)) {
        SPDLOG_ERROR("World {} already exists", worldId);
        throw std::runtime_error("World already exists");
    }
    int worldSize = msg.mpiworldsize();
    if (worldSize <= 0) {
        worldSize = faabric::util::getSystemConfig().defaultMpiWorldSize;
    }
    // Only the thread that actually inserts the entry builds the world
    worldMap.tryEmplaceThenMutate(
      worldId,
      [&](bool inserted, std::shared_ptr<MpiWorld>& w) {
          if (!inserted) {
              return;
          }
          if (!hostOverride.empty()) {
              w->overrideHost(hostOverride);
          }
          w->create(msg, worldId, worldSize);
      },
      std::make_shared<MpiWorld>());
    return getWorld(worldId);
}

MpiWorld& MpiWorldRegistry::getOrInitialiseWorld(faabric::Message& msg)
{
    int worldId = msg.mpiworldid();
    // The first local rank to get here initialises the host-wide part
    worldMap.tryEmplaceThenMutate(
      worldId,
      [&](bool inserted, std::shared_ptr<MpiWorld>& w) {
          if (inserted) {
              w->initialiseFromMsg(msg);
          }
      },
      std::make_shared<MpiWorld>());
    MpiWorld& world = getWorld(worldId);
    world.initialiseRankFromMsg(msg);
    return world;
}

MpiWorld& MpiWorldRegistry::getWorld(int worldId)
{
    auto w = worldMap.get(worldId);
    if (!w.has_value()) {
        SPDLOG_ERROR("World {} not initialised", worldId);
        throw std::runtime_error("World not initialised");
    }
    return *w.value();
}

std::shared_ptr<MpiWorld> MpiWorldRegistry::findWorld(int worldId)
{
    auto w = worldMap.get(worldId);
    return w.has_value() ? w.value() : nullptr;
}

bool MpiWorldRegistry::worldExists(int worldId)
{
    return worldMap.contains(worldId);
}

void MpiWorldRegistry::clearWorld(int worldId)
{
    // sub-communicators live and die with their world
    clearSubCommunicators(worldId);
    worldMap.erase(worldId);
}

void MpiWorldRegistry::clear()
{
    clearSubCommunicators(-1);
    worldMap.clear();
}

// ---------------------------------------------------------------------------
// Context
// ---------------------------------------------------------------------------
MpiContext::MpiContext()
  : isMpi(false)
  , rank(-1)
  , worldId(-1)
{}

int MpiContext::createWorld(faabric::Message& msg)
{
    if (msg.mpirank() > 0) {
        SPDLOG_ERROR("Attempting to initialise world for non-zero rank {}", msg.mpirank());
        throw std::runtime_error("Initialising world on non-zero rank");
    }
    worldId = (int)faabric::util::generateGid();
    SPDLOG_DEBUG("Initialising world {}", worldId);
    msg.set_mpiworldid(worldId);
    MpiWorldRegistry& reg = getMpiWorldRegistry();
    MpiWorld& world = reg.createWorld(msg, worldId);
    // Rank 0 also sets up its own per-thread state
    world.initialiseRankFromMsg(msg);
    isMpi = true;
    rank = 0;
    return worldId;
}

void MpiContext::joinWorld(faabric::Message& msg)
{
    if (!msg.ismpi()) {
        // Not an MPI call
        return;
    }
    isMpi = true;
    worldId = msg.mpiworldid();
    rank = msg.mpirank();
    getMpiWorldRegistry().getOrInitialiseWorld(msg);
}

bool MpiContext::getIsMpi() const
{
    return isMpi;
}

int MpiContext::getRank() const
{
    return rank;
}

int MpiContext::getWorldId() const
{
    return worldId;
}

} // namespace faabric::mpi
