// Shared fixtures for the integration tests: an in-process planner + worker.
#pragma once

#include "harness.h"

#include <faabric/executor/Executor.h>
#include <faabric/executor/ExecutorContext.h>
#include <faabric/executor/ExecutorFactory.h>
#include <faabric/planner/Planner.h>
#include <faabric/planner/PlannerClient.h>
#include <faabric/planner/PlannerServer.h>
#include <faabric/scheduler/FunctionCallServer.h>
#include <faabric/scheduler/Scheduler.h>
#include <faabric/snapshot/SnapshotServer.h>
#include <faabric/state/State.h>
#include <faabric/state/StateServer.h>
#include <faabric/transport/PointToPointBroker.h>
#include <faabric/transport/PointToPointServer.h>
#include <faabric/util/batch.h>
#include <faabric/util/config.h>
#include <faabric/util/func.h>
#include <faabric/util/testing.h>

#include <atomic>
#include <cstdlib>
#include <functional>
#include <map>

namespace tests {

// The loopback device backend (heaps in host memory, no GPU needed) for the
// lifetime of the object; the configuration is reset afterwards
struct LoopbackBackend
{
    LoopbackBackend() { setenv("FAABRIC_DEVICE_BACKEND", "loopback", 1); }
    ~LoopbackBackend()
    {
        unsetenv("FAABRIC_DEVICE_BACKEND");
        faabric::util::getSystemConfig().reset();
    }
};

typedef std::function<int(faabric::executor::Executor*, int, int, std::shared_ptr<faabric::BatchExecuteRequest>)>
  TestFunction;

// Function bodies are looked up by "user/function"
std::map<std::string, TestFunction>& functionTable();

void registerTestFunction(const std::string& user, const std::string& function, TestFunction fn);

class TestExecutor : public faabric::executor::Executor
{
  public:
    explicit TestExecutor(faabric::Message& msg);

    int32_t executeTask(int threadPoolIdx, int msgIdx, std::shared_ptr<faabric::BatchExecuteRequest> req) override;

    std::span<uint8_t> getMemoryView() override;

    void setMemorySize(size_t newSize) override;

    size_t getMaxMemorySize() override;

    void restore(const std::string& snapshotKey) override;

    void reset(faabric::Message& msg) override;

    // Hook bookkeeping across all test executors
    static std::atomic<int> resetCount;
    static std::atomic<int> restoreCount;

    faabric::util::MemoryRegion memory;
    size_t memorySize = 0;
    static constexpr size_t MAX_MEMORY = (size_t)64 << 20;
};

class TestExecutorFactory : public faabric::executor::ExecutorFactory
{
  public:
    std::shared_ptr<faabric::executor::Executor> createExecutor(faabric::Message& msg) override;

    void flushHost() override { flushCount++; }

    int flushCount = 0;
};

// Planner + all worker servers in this process, this host registered with
// `slots` slots (plus optional virtual GPU hosts)
class ClusterFixture
{
  public:
    explicit ClusterFixture(int slots = 8, int nVirtualHosts = 0, int slotsPerVirtualHost = 0);

    ~ClusterFixture();

    faabric::util::SystemConfig& conf;
    faabric::planner::Planner& planner;
    faabric::planner::PlannerClient& plannerCli;
    faabric::scheduler::Scheduler& sch;
    std::shared_ptr<TestExecutorFactory> factory;
    std::vector<std::string> virtualHosts;

    faabric::Message awaitResult(const faabric::Message& msg, int timeoutMs = 10000);

    std::shared_ptr<faabric::BatchExecuteRequestStatus> awaitBatch(std::shared_ptr<faabric::BatchExecuteRequest> req,
                                                                  int timeoutMs = 20000);

  private:
    faabric::planner::PlannerServer plannerServer;
    faabric::scheduler::FunctionCallServer functionServer;
    faabric::snapshot::SnapshotServer snapshotServer;
    faabric::transport::PointToPointServer ptpServer;
    faabric::state::StateServer stateServer;
};

}
