// Environment-driven configuration.  One table describes every knob (env name,
// default, section, field); initialise() and print() both walk it, so a new
// setting is one line.  Names and defaults of the non-GPU knobs are those of
// the reference (src/util/config.cpp:19-84) so deployments carry over.
#include <faabric/util/config.h>
#include <faabric/util/environment.h>
#include <faabric/util/logging.h>
#include <faabric/util/network.h>

#include <cstdlib>
#include <string>
#include <variant>
#include <vector>

namespace faabric::util {

namespace {
using Field = std::variant<std::string SystemConfig::*, int SystemConfig::*, long SystemConfig::*>;

struct Knob
{
    const char* section;
    const char* env;
    const char* fallback;
    Field field;
};

const std::vector<Knob>& knobs()
{
    using C = SystemConfig;
    static const std::vector<Knob> table = {
        { "System", "SERIALISATION", "json", &C::serialisation },
        { "System", "LOG_LEVEL", "info", &C::logLevel },
        { "System", "LOG_FILE", "off", &C::logFile },
        { "System", "STATE_MODE", "inmemory", &C::stateMode },
        { "System", "DELTA_SNAPSHOT_ENCODING", "pages=4096;xor;zstd=1", &C::deltaSnapshotEncoding },
        { "Store", "REDIS_STATE_HOST", "localhost", &C::redisStateHost },
        { "Store", "REDIS_QUEUE_HOST", "localhost", &C::redisQueueHost },
        { "Store", "REDIS_PORT", "6379", &C::redisPort },
        { "Scheduling", "OVERRIDE_CPU_COUNT", "0", &C::overrideCpuCount },
        { "Scheduling", "OVERRIDE_FREE_CPU_START", "0", &C::overrideFreeCpuStart },
        { "Scheduling", "BATCH_SCHEDULER_MODE", "bin-pack", &C::batchSchedulerMode },
        { "Timeouts", "GLOBAL_MESSAGE_TIMEOUT", "60000", &C::globalMessageTimeout },
        { "Timeouts", "BOUND_TIMEOUT", "30000", &C::boundTimeout },
        { "Timeouts", "REAPER_INTERVAL_SECS", "30", &C::reaperIntervalSeconds },
        { "MPI", "DEFAULT_MPI_WORLD_SIZE", "5", &C::defaultMpiWorldSize },
        { "Endpoint", "ENDPOINT_INTERFACE", "", &C::endpointInterface },
        { "Endpoint", "ENDPOINT_HOST", "", &C::endpointHost },
        { "Endpoint", "ENDPOINT_PORT", "8080", &C::endpointPort },
        { "Endpoint", "ENDPOINT_NUM_THREADS", "4", &C::endpointNumThreads },
        { "Transport", "FUNCTION_SERVER_THREADS", "2", &C::functionServerThreads },
        { "Transport", "STATE_SERVER_THREADS", "2", &C::stateServerThreads },
        { "Transport", "SNAPSHOT_SERVER_THREADS", "2", &C::snapshotServerThreads },
        { "Transport", "POINT_TO_POINT_SERVER_THREADS", "8", &C::pointToPointServerThreads },
        { "Dirty tracking", "DIRTY_TRACKING_MODE", "segfault", &C::dirtyTrackingMode },
        { "Dirty tracking", "DIFFING_MODE", "xor", &C::diffingMode },
        { "Planner", "PLANNER_HOST", "planner", &C::plannerHost },
        { "Planner", "PLANNER_PORT", "8080", &C::plannerPort },
        { "GPU", "FAABRIC_GPUS", "", &C::gpus },
        { "GPU", "FAABRIC_DEVICE_BACKEND", "cuda", &C::deviceBackend },
        { "GPU", "FAABRIC_ALLREDUCE_ALGO", "auto", &C::allreduceAlgo },
        { "GPU", "FAABRIC_USE_NVLS", "1", &C::useNvls },
        { "GPU", "FAABRIC_COMM_STREAMS", "2", &C::commStreams },
        { "GPU", "FAABRIC_SYMM_HEAP_BYTES", "1073741824", &C::symmHeapBytes },
        { "GPU", "FAABRIC_SLOTS_PER_GPU", "8", &C::slotsPerGpu },
        { "GPU", "FAABRIC_PORT_OFFSET", "0", &C::portOffset },
        { "GPU", "FAABRIC_CHECKPOINT_DIR", "", &C::checkpointDir },
    };
    return table;
}
}

SystemConfig& getSystemConfig()
{
    static SystemConfig conf;
    return conf;
}

SystemConfig::SystemConfig()
{
    initialise();
}

int SystemConfig::getSystemConfIntParam(const char* name, const char* defaultValue)
{
    return (int)getSystemConfLongParam(name, defaultValue);
}

long SystemConfig::getSystemConfLongParam(const char* name, const char* defaultValue)
{
    return std::strtol(getEnvVar(name, defaultValue).c_str(), nullptr, 10);
}

void SystemConfig::initialise()
{
    for (const Knob& k : knobs()) {
        if (auto* s = std::get_if<std::string SystemConfig::*>(&k.field)) {
            this->**s = getEnvVar(k.env, k.fallback);
        } else if (auto* i = std::get_if<int SystemConfig::*>(&k.field)) {
            this->**i = getSystemConfIntParam(k.env, k.fallback);
        } else {
            this->*std::get<long SystemConfig::*>(k.field) = getSystemConfLongParam(k.env, k.fallback);
        }
    }
    if (endpointHost.empty()) {
        // Nothing configured: the primary address of the chosen interface
        endpointHost = getPrimaryIPForThisHost(endpointInterface);
    }
}

void SystemConfig::reset()
{
    initialise();
}

void SystemConfig::print()
{
    const char* section = "";
    for (const Knob& k : knobs()) {
        if (std::string(section) != k.section) {
            section = k.section;
            SPDLOG_INFO("--- {} ---", section);
        }
        std::string name(k.env);
        name.resize(std::max<size_t>(name.size() + 1, 30), ' ');
        if (auto* s = std::get_if<std::string SystemConfig::*>(&k.field)) {
            SPDLOG_INFO("{}{}", name, this->**s);
        } else if (auto* i = std::get_if<int SystemConfig::*>(&k.field)) {
            SPDLOG_INFO("{}{}", name, this->**i);
        } else {
            SPDLOG_INFO("{}{}", name, this->*std::get<long SystemConfig::*>(k.field));
        }
    }
}

} // namespace faabric::util
