// Worker bootstrap and the single-process cluster.
//
// One header per module: the per-class headers of the reference's layout
// (faabric/runner/*.h) forward here, so either include style works.
#pragma once

#include <faabric/executor/ExecutorFactory.h>
#include <faabric/planner/PlannerServer.h>
#include <faabric/scheduler/FunctionCallServer.h>
#include <faabric/scheduler/Scheduler.h>
#include <faabric/snapshot/SnapshotServer.h>
#include <faabric/state/StateServer.h>
#include <faabric/transport/PointToPointServer.h>
#include <faabric/util/config.h>

#include <memory>
#include <string>
#include <vector>

// ==========================================================================
// runner/FaabricMain.h
// ==========================================================================
namespace faabric::runner {

// Boots a worker: crash handler, registers the host with the planner, starts
// the State / Snapshot / PointToPoint / FunctionCall servers (reference:
// src/runner/FaabricMain.cpp:11-109).  On a GPU box it also initialises CUDA
// and binds the worker to its GPU.
class FaabricMain
{
  public:
    explicit FaabricMain(std::shared_ptr<faabric::executor::ExecutorFactory> fac);

    void startBackground();

    void startRunner();

    void startFunctionCallServer();

    void startStateServer();

    void startSnapshotServer();

    void startPointToPointServer();

    void shutdown();

    // Snapshot registry <-> FAABRIC_CHECKPOINT_DIR (no-ops when unset)
    void restoreCheckpoint();

    void writeCheckpoint();

  private:
    faabric::state::StateServer stateServer;
    faabric::scheduler::FunctionCallServer functionServer;
    faabric::snapshot::SnapshotServer snapshotServer;
    faabric::transport::PointToPointServer pointToPointServer;
};

}

// ==========================================================================
// runner/LocalCluster.h
// ==========================================================================
namespace faabric::runner {

// A whole deployment inside one process: the planner, and one worker that
// registers each GPU (or any number of virtual hosts) as a separate planner
// host.  This is the single-box HGX topology - eight GPUs behind NVSwitch
// are eight "hosts" to the scheduler but share an address space, so RPCs take
// the in-process fast path and MPI ranks reach each other through peer memory.
// (The reference needs a docker-compose cluster for the same picture.)
class LocalCluster
{
  public:
    // nVirtualHosts == 0: only this host, with `slotsPerHost` slots
    LocalCluster(std::shared_ptr<faabric::executor::ExecutorFactory> factory,
                 int nVirtualHosts,
                 int slotsPerHost);

    ~LocalCluster();

    const std::vector<std::string>& hosts() const { return hostNames; }

    // Blocks until every message of the app has a result (or throws)
    std::shared_ptr<faabric::BatchExecuteRequestStatus> awaitBatch(
      std::shared_ptr<faabric::BatchExecuteRequest> req,
      int timeoutMs = 60000);

  private:
    std::vector<std::string> hostNames;
    faabric::planner::PlannerServer plannerServer;
    faabric::scheduler::FunctionCallServer functionServer;
    faabric::snapshot::SnapshotServer snapshotServer;
    faabric::transport::PointToPointServer ptpServer;
    faabric::state::StateServer stateServer;
};

}

