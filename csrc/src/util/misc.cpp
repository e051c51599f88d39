// Small utilities: gids, random, environment, network, files, bytes, strings,
// testing flags.
#include <csignal>
#include <sys/prctl.h>
#include <faabric/util/bytes.h>
#include <faabric/util/config.h>
#include <faabric/util/environment.h>
#include <faabric/util/files.h>
#include <faabric/util/gids.h>
#include <faabric/util/network.h>
#include <faabric/util/random.h>
#include <faabric/util/string_tools.h>
#include <faabric/util/testing.h>

#include <algorithm>
#include <arpa/inet.h>
#include <atomic>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <ifaddrs.h>
#include <mutex>
#include <net/if.h>
#include <netdb.h>
#include <random>
#include <sstream>
#include <thread>
#include <unistd.h>
#include <unordered_map>

namespace faabric::device {
int cudaDeviceCountSafe();
}

namespace faabric::util {

// ------------------------------------------------------------------ gids ---
static std::atomic<unsigned int> gidCounter{ 0 };
static std::once_flag gidOnce;
static unsigned int gidBase = 0;

unsigned int generateGid()
{
    std::call_once(gidOnce, []() {
        // Mix host identity, pid and a random draw so that several workers on
        // one box (one per GPU) do not collide
        std::random_device rd;
        size_t h = std::hash<std::string>{}(getSystemConfig().endpointHost);
        h ^= (size_t)getpid() * 0x9e3779b97f4a7c15ull;
        h ^= ((size_t)rd() << 16) ^ rd();
        gidBase = (unsigned int)(h % 1000000u) * 1000u;
    });
    unsigned int v = gidBase + gidCounter.fetch_add(1) + 1;
    // Keep ids positive when stored in int32 message fields
    return v & 0x7fffffffu;
}

// ---------------------------------------------------------------- random ---
static std::mt19937& rng()
{
    static thread_local std::mt19937 gen{ std::random_device{}() };
    return gen;
}

std::string randomStringFromSet(int len, const std::string& charSet)
{
    std::uniform_int_distribution<size_t> dist(0, charSet.size() - 1);
    std::string out;
    out.reserve(len);
    for (int i = 0; i < len; i++) {
        out += charSet[dist(rng())];
    }
    return out;
}

std::string randomString(int len)
{
    static const std::string chars =
      "0123456789abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ";
    return randomStringFromSet(len, chars);
}

int randomInteger(int iStart, int iEnd)
{
    std::uniform_int_distribution<int> dist(iStart, iEnd);
    return dist(rng());
}

// ----------------------------------------------------------- environment ---
void exitWithParentIfAsked()
{
    if (getEnvVar("FAABRIC_EXIT_WITH_PARENT", "0") != "1") {
        return;
    }
    ::prctl(PR_SET_PDEATHSIG, SIGTERM);
    // the parent may already be gone: we have been re-parented to init
    if (::getppid() == 1) {
        ::raise(SIGTERM);
    }
}

std::string getEnvVar(const std::string& key, const std::string& deflt)
{
    const char* v = getenv(key.c_str());
    if (v == nullptr || *v == '\0') {
        return deflt;
    }
    return v;
}

std::string setEnvVar(const std::string& varName, const std::string& value)
{
    const char* old = getenv(varName.c_str());
    std::string original = old != nullptr ? old : "";
    setenv(varName.c_str(), value.c_str(), 1);
    return original;
}

void unsetEnvVar(const std::string& varName)
{
    unsetenv(varName.c_str());
}

unsigned int getUsableCores()
{
    int over = getSystemConfig().overrideCpuCount;
    if (over > 0) {
        return (unsigned int)over;
    }
    unsigned int n = std::thread::hardware_concurrency();
    return n == 0 ? 1 : n;
}

int getUsableGpus()
{
    return faabric::device::cudaDeviceCountSafe();
}

// --------------------------------------------------------------- network ---
// Every thread builds its own planner client and resolves PLANNER_HOST, so
// answers are kept for a while: a fan-out that starts a thousand executor
// threads then costs a lookup or two, not a thousand serialised ones, each of
// which may wait for a resolver that cannot answer.  A failure is kept only
// briefly: callers fall back to ENDPOINT_HOST while a name does not resolve,
// and a name that starts resolving is picked up within a second.
static std::mutex hostnameMx;
static std::unordered_map<std::string, std::pair<std::string, std::chrono::steady_clock::time_point>> hostnameCache;
static constexpr auto HOSTNAME_CACHE_TTL = std::chrono::seconds(5);
static constexpr auto HOSTNAME_FAILURE_TTL = std::chrono::seconds(1);

std::string getIPFromHostname(const std::string& hostname)
{
    std::lock_guard<std::mutex> lk(hostnameMx);
    auto cached = hostnameCache.find(hostname);
    if (cached != hostnameCache.end() &&
        std::chrono::steady_clock::now() - cached->second.second <
          (cached->second.first.empty() ? HOSTNAME_FAILURE_TTL : HOSTNAME_CACHE_TTL)) {
        return cached->second.first;
    }
    addrinfo hints;
    memset(&hints, 0, sizeof(hints));
    hints.ai_family = AF_INET;
    hints.ai_socktype = SOCK_STREAM;
    addrinfo* res = nullptr;
    std::string ip;
    if (getaddrinfo(hostname.c_str(), nullptr, &hints, &res) == 0 && res != nullptr) {
        char buf[INET_ADDRSTRLEN];
        auto* sa = (sockaddr_in*)res->ai_addr;
        inet_ntop(AF_INET, &sa->sin_addr, buf, sizeof(buf));
        freeaddrinfo(res);
        ip = buf;
    }
    hostnameCache[hostname] = { ip, std::chrono::steady_clock::now() };
    return ip;
}

std::string getPrimaryIPForThisHost(const std::string& interface)
{
    ifaddrs* all = nullptr;
    if (getifaddrs(&all) != 0) {
        return LOCALHOST;
    }
    std::string found;
    for (ifaddrs* a = all; a != nullptr; a = a->ifa_next) {
        if (a->ifa_addr == nullptr || a->ifa_addr->sa_family != AF_INET) {
            continue;
        }
        if ((a->ifa_flags & IFF_LOOPBACK) != 0 || (a->ifa_flags & IFF_UP) == 0) {
            continue;
        }
        std::string name = a->ifa_name;
        if (!interface.empty() && name != interface) {
            continue;
        }
        // Skip container bridges unless explicitly requested
        if (interface.empty() && (name.rfind("docker", 0) == 0 ||
                                  name.rfind("br-", 0) == 0 ||
                                  name.rfind("veth", 0) == 0)) {
            continue;
        }
        char buf[INET_ADDRSTRLEN];
        inet_ntop(AF_INET, &((sockaddr_in*)a->ifa_addr)->sin_addr, buf, sizeof(buf));
        found = buf;
        break;
    }
    freeifaddrs(all);
    return found.empty() ? LOCALHOST : found;
}

std::string gpuHostName(int gpuIdx)
{
    return "gpu" + std::to_string(gpuIdx);
}

int gpuIndexFromHostName(const std::string& host)
{
    if (host.size() > 3 && host.compare(0, 3, "gpu") == 0 &&
        stringIsInt(host.substr(3))) {
        return std::stoi(host.substr(3));
    }
    return -1;
}

// ----------------------------------------------------------------- files ---
std::string readFileToString(const std::string& path)
{
    std::ifstream f(path, std::ios::binary);
    if (!f) {
        throw std::runtime_error("Could not read file " + path);
    }
    std::ostringstream os;
    os << f.rdbuf();
    return os.str();
}

std::vector<uint8_t> readFileToBytes(const std::string& path)
{
    std::string s = readFileToString(path);
    return std::vector<uint8_t>(s.begin(), s.end());
}

void writeBytesToFile(const std::string& path, const std::vector<uint8_t>& data)
{
    std::ofstream f(path, std::ios::binary | std::ios::trunc);
    if (!f) {
        throw std::runtime_error("Could not write file " + path);
    }
    f.write((const char*)data.data(), (std::streamsize)data.size());
}

bool isWasm(const std::vector<uint8_t>& bytes)
{
    static const uint8_t magic[] = { 0x00, 0x61, 0x73, 0x6d };
    return bytes.size() >= 4 && memcmp(bytes.data(), magic, 4) == 0;
}

// ----------------------------------------------------------------- bytes ---
std::vector<uint8_t> stringToBytes(const std::string& str)
{
    return std::vector<uint8_t>(str.begin(), str.end());
}

std::string bytesToString(const std::vector<uint8_t>& bytes)
{
    return std::string(bytes.begin(), bytes.end());
}

std::string formatByteArrayToIntString(const std::vector<uint8_t>& bytes)
{
    std::ostringstream os;
    os << "[";
    for (size_t i = 0; i < bytes.size(); i++) {
        os << (int)bytes[i];
        if (i + 1 < bytes.size()) {
            os << ", ";
        }
    }
    os << "]";
    return os.str();
}

void trimTrailingZeros(std::vector<uint8_t>& vectorIn)
{
    while (!vectorIn.empty() && vectorIn.back() == 0) {
        vectorIn.pop_back();
    }
}

int safeCopyToBuffer(const std::vector<uint8_t>& dataIn,
                     uint8_t* buffer,
                     int bufferLen)
{
    // A non-positive buffer length is a size query
    if (bufferLen <= 0) {
        return (int)dataIn.size();
    }
    return safeCopyToBuffer(dataIn.data(), (int)dataIn.size(), buffer, bufferLen);
}

int safeCopyToBuffer(const uint8_t* dataIn,
                     int dataLen,
                     uint8_t* buffer,
                     int bufferLen)
{
    if (dataLen == 0) {
        return 0;
    }
    // Truncate if the destination is too small
    int n = std::min(dataLen, bufferLen);
    if (n > 0) {
        memcpy(buffer, dataIn, (size_t)n);
    }
    return std::max(n, 0);
}

std::string byteArrayToHexString(const uint8_t* data, int dataSize)
{
    static const char* hex = "0123456789abcdef";
    std::string out;
    out.reserve((size_t)dataSize * 2);
    for (int i = 0; i < dataSize; i++) {
        out += hex[data[i] >> 4];
        out += hex[data[i] & 0xf];
    }
    return out;
}

std::vector<uint8_t> hexStringToByteArray(const std::string& hexString)
{
    if (hexString.size() % 2 != 0) {
        throw std::runtime_error("Hex string must have an even length");
    }
    auto nibble = [](char c) -> int {
        if (c >= '0' && c <= '9') {
            return c - '0';
        }
        if (c >= 'a' && c <= 'f') {
            return c - 'a' + 10;
        }
        if (c >= 'A' && c <= 'F') {
            return c - 'A' + 10;
        }
        throw std::runtime_error("Invalid hex digit");
    };
    std::vector<uint8_t> out(hexString.size() / 2);
    for (size_t i = 0; i < out.size(); i++) {
        out[i] = (uint8_t)((nibble(hexString[2 * i]) << 4) |
                           nibble(hexString[2 * i + 1]));
    }
    return out;
}

// --------------------------------------------------------------- strings ---
bool isAllWhitespace(const std::string& input)
{
    return std::all_of(
      input.begin(), input.end(), [](unsigned char c) { return isspace(c); });
}

bool startsWith(const std::string& input, const std::string& subStr)
{
    if (subStr.empty()) {
        return false;
    }
    return input.rfind(subStr, 0) == 0;
}

bool endsWith(const std::string& value, const std::string& ending)
{
    if (ending.empty() || ending.size() > value.size()) {
        return false;
    }
    return std::equal(ending.rbegin(), ending.rend(), value.rbegin());
}

bool contains(const std::string& input, const std::string& subStr)
{
    return input.find(subStr) != std::string::npos;
}

std::string removeSubstr(const std::string& input, const std::string& toErase)
{
    std::string out = input;
    size_t pos = out.find(toErase);
    if (pos != std::string::npos) {
        out.erase(pos, toErase.size());
    }
    return out;
}

bool stringIsInt(const std::string& input)
{
    return !input.empty() &&
           std::all_of(input.begin(), input.end(), [](unsigned char c) {
               return isdigit(c);
           });
}

std::vector<std::string> splitString(const std::string& input, char delim)
{
    std::vector<std::string> out;
    std::string cur;
    for (char c : input) {
        if (c == delim) {
            if (!cur.empty()) {
                out.push_back(cur);
            }
            cur.clear();
        } else {
            cur += c;
        }
    }
    if (!cur.empty()) {
        out.push_back(cur);
    }
    return out;
}

std::string trim(const std::string& input)
{
    size_t b = 0;
    size_t e = input.size();
    while (b < e && isspace((unsigned char)input[b])) {
        b++;
    }
    while (e > b && isspace((unsigned char)input[e - 1])) {
        e--;
    }
    return input.substr(b, e - b);
}

std::string toLower(const std::string& input)
{
    std::string out = input;
    std::transform(out.begin(), out.end(), out.begin(), [](unsigned char c) {
        return (char)tolower(c);
    });
    return out;
}

// --------------------------------------------------------------- testing ---
static std::atomic<bool> testMode{ false };
static std::atomic<bool> mockMode{ false };

void setTestMode(bool val)
{
    testMode.store(val);
}

bool isTestMode()
{
    return testMode.load();
}

void setMockMode(bool val)
{
    mockMode.store(val);
}

bool isMockMode()
{
    return mockMode.load();
}


std::string randomStringFromSet(const std::unordered_set<std::string>& s)
{
    if (s.empty()) {
        return "";
    }
    auto it = s.begin();
    std::advance(it, randomInteger(0, (int)s.size() - 1));
    return *it;
}

// ---- util/bytes.h, util/batch.h additions ----
int bytesToInt(const std::vector<uint8_t>& bytes)
{
    if (bytes.size() != sizeof(int)) {
        throw std::runtime_error("bytesToInt needs exactly sizeof(int) bytes");
    }
    int v;
    memcpy(&v, bytes.data(), sizeof(int));
    return v;
}

int getNumFinishedMessagesInBatch(std::shared_ptr<faabric::BatchExecuteRequestStatus> berStatus)
{
    int n = 0;
    for (const auto& m : berStatus->messageresults()) {
        if (m.returnvalue() != MIGRATED_FUNCTION_RETURN_VALUE) {
            n++;
        }
    }
    return n;
}

// ---- util/state.h ----
std::string keyForUser(const std::string& user, const std::string& key)
{
    if (user.empty() || key.empty()) {
        throw std::runtime_error("Cannot have empty user or key (" + user + "/" + key + ")");
    }
    return user + "_" + key;
}

void maskDouble(unsigned int* maskArray, unsigned long idx)
{
    // (an unsigned int is half a double)
    unsigned long intIdx = 2 * idx;
    maskArray[intIdx] |= STATE_MASK_32;
    maskArray[intIdx + 1] |= STATE_MASK_32;
}

} // namespace faabric::util

// (reference: include/faabric/wasm/wasm.h declares it for the embedder)
int helloFaabricWasm()
{
    return 0;
}
