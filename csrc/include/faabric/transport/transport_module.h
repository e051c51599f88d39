// Transport: messages, endpoints, RPC servers, point-to-point groups, raw TCP.
//
// One header per module: the per-class headers of the reference's layout
// (faabric/transport/*.h) forward here, so either include style works.
#pragma once

#include <functional>

#include <faabric/batch-scheduler/SchedulingDecision.h>
#include <faabric/proto/faabric.pb.h>
#include <faabric/util/barrier.h>
#include <faabric/util/config.h>
#include <faabric/util/exception.h>
#include <faabric/util/latch.h>
#include <faabric/util/locks.h>
#include <faabric/util/queue.h>

#include <netinet/in.h>
#include <sys/socket.h>

#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <cstring>
#include <memory>
#include <mutex>
#include <queue>
#include <set>
#include <shared_mutex>
#include <span>
#include <stack>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

// ==========================================================================
// transport/Message.h
// ==========================================================================
// A received (or to-be-sent) transport message: 16-byte header + payload.
// Header layout matches the reference (transport/Message.h:11-21): code u8,
// size u64, sequence number i32, 3 bytes padding.


namespace faabric::transport {

#define NO_HEADER 0
#define HEADER_MSG_SIZE 16
#define SHUTDOWN_HEADER 220
// Sync response carrying the text of an exception thrown by the handler
#define ERROR_HEADER 221
static const std::vector<uint8_t> shutdownPayload = { 0, 0, 1, 1 };

#define NO_SEQUENCE_NUM -1

enum class MessageResponseCode
{
    SUCCESS,
    TERM,
    TIMEOUT,
    ERROR
};

class Message final
{
  public:
    Message() = default;

    // Empty message signalling an outcome (e.g. TIMEOUT)
    explicit Message(MessageResponseCode failCodeIn)
      : failCode(failCodeIn)
    {}

    Message(uint8_t codeIn, int seqIn, std::vector<uint8_t>&& payloadIn)
      : code(codeIn)
      , sequenceNum(seqIn)
      , payload(std::move(payloadIn))
    {}

    Message(uint8_t codeIn, int seqIn, const uint8_t* data, size_t size)
      : code(codeIn)
      , sequenceNum(seqIn)
      , payload(data, data + size)
    {}

    // Adopts a handler's response string as it is (the in-process sync fast
    // path hands it to the caller without another copy)
    Message(uint8_t codeIn, int seqIn, std::string&& textIn)
      : code(codeIn)
      , sequenceNum(seqIn)
      , text(std::move(textIn))
      , isText(true)
    {}

    // Non-owning view of a caller's buffer: used by the in-process sync fast
    // path, where the handler runs on the caller's stack.  Anything that
    // outlives the call must ensureOwned() first.
    static Message view(uint8_t codeIn, int seqIn, const uint8_t* data, size_t size)
    {
        Message m;
        m.code = codeIn;
        m.sequenceNum = seqIn;
        m.borrowed = std::span<const uint8_t>(data, size);
        m.isView = true;
        return m;
    }

    void ensureOwned()
    {
        if (isView) {
            payload.assign(borrowed.begin(), borrowed.end());
            borrowed = {};
            isView = false;
        }
        if (isText) {
            payload.assign(text.begin(), text.end());
            std::string().swap(text);
            isText = false;
        }
    }

    Message(Message&& other) = default;

    Message& operator=(Message&& other) = default;

    Message(const Message&) = delete;

    Message& operator=(const Message&) = delete;

    MessageResponseCode getResponseCode() const { return failCode; }

    std::vector<uint8_t> dataCopy() const
    {
        auto d = udata();
        return std::vector<uint8_t>(d.begin(), d.end());
    }

    std::span<const uint8_t> udata() const
    {
        if (isView) {
            return borrowed;
        }
        if (isText) {
            return std::span<const uint8_t>((const uint8_t*)text.data(), text.size());
        }
        return std::span<const uint8_t>(payload.data(), payload.size());
    }

    std::span<const char> data() const
    {
        auto d = udata();
        return std::span<const char>((const char*)d.data(), d.size());
    }

    std::vector<uint8_t>& buffer()
    {
        ensureOwned();
        return payload;
    }

    size_t size() const { return udata().size(); }

    uint8_t getMessageCode() const { return code; }

    int getSequenceNum() const { return sequenceNum; }

    // Serialised header
    static void writeHeader(uint8_t* out, uint8_t code, uint64_t size, int32_t seq)
    {
        memset(out, 0, HEADER_MSG_SIZE);
        out[0] = code;
        memcpy(out + 1, &size, sizeof(uint64_t));
        memcpy(out + 1 + sizeof(uint64_t), &seq, sizeof(int32_t));
    }

    static void readHeader(const uint8_t* in, uint8_t& code, uint64_t& size, int32_t& seq)
    {
        code = in[0];
        memcpy(&size, in + 1, sizeof(uint64_t));
        memcpy(&seq, in + 1 + sizeof(uint64_t), sizeof(int32_t));
    }

  private:
    uint8_t code = NO_HEADER;
    int sequenceNum = NO_SEQUENCE_NUM;
    std::vector<uint8_t> payload;
    std::span<const uint8_t> borrowed;
    bool isView = false;
    std::string text;
    bool isText = false;
    MessageResponseCode failCode = MessageResponseCode::SUCCESS;
};

}

// ==========================================================================
// transport/tcp/Socket.h
// ==========================================================================
// Raw TCP sockets: the cross-process MPI fallback data plane for host buffers
// and the carrier of the control RPC (reference: src/transport/tcp/*).


#define SocketListenBacklog 1024
#define SocketPollTimeoutMs 5000
// 16 MiB send / receive buffers
#define SocketBufferSizeBytes (16 * 1024 * 1024)

namespace faabric::transport::tcp {

void setReuseAddr(int fd);
void setNoDelay(int fd);
void setQuickAck(int fd);
void setBusyPolling(int fd);
void setNonBlocking(int fd);
void setBlocking(int fd);
bool isNonBlocking(int fd);
void setRecvTimeoutMs(int fd, int timeoutMs);
void setSendTimeoutMs(int fd, int timeoutMs);
void setRecvBufferSize(int fd, size_t bufferSize);
void setSendBufferSize(int fd, size_t bufferSize);

// IPv4 socket address (reference: include/faabric/transport/tcp/Address.h)
class Address
{
  public:
    Address(const std::string& host, int port);

    // any local interface
    explicit Address(int port);

    sockaddr* get() const { return (sockaddr*)&addr; }

    int port() const;

    std::string host() const;

  private:
    sockaddr_in addr;
};

class Socket
{
  public:
    Socket();
    explicit Socket(int connFd);
    Socket(const Socket&) = delete;
    Socket& operator=(const Socket&) = delete;
    Socket(Socket&& other) noexcept;
    Socket& operator=(Socket&& other) noexcept;
    ~Socket();

    int get() const { return fd; }
    void close();

  private:
    int fd = -1;
};

class SendSocket
{
  public:
    SendSocket(const std::string& hostIn, int portIn);

    // Retries while the peer is still coming up (30 x 200 ms by default)
    void dial(int retries = 30, int sleepMs = 200);

    void sendOne(const uint8_t* buffer, size_t bufferSize);

    int getFd() const { return sock.get(); }

  private:
    std::string host;
    int port;
    Socket sock;
};

class RecvSocket
{
  public:
    explicit RecvSocket(int portIn, const std::string& hostIn = "0.0.0.0");
    ~RecvSocket();

    void listen();

    // Returns the connection fd; throws on timeout
    int accept(int timeoutMs = SocketPollTimeoutMs);

    void recvOne(int conn, uint8_t* buffer, size_t bufferSize);

    int getPort() const { return port; }

    // the listening socket, for callers that poll it next to other fds
    int getFd() const { return sock.get(); }

  private:
    std::string host;
    int port;
    Socket sock;
    std::vector<int> openConnections;
};

}

// ==========================================================================
// transport/MessageEndpoint.h
// ==========================================================================
// Control-plane endpoints.  The reference wraps NNG sockets (push/pull,
// req/rep, inproc pairs: include/faabric/transport/MessageEndpoint.h:14-280);
// here they are plain TCP streams of framed messages plus an in-process
// registry, because on one box most peers live in the same process: a send to
// a server registered in this process skips the socket entirely.
// No payload of the data plane travels here (that is NVLink P2P).



#define DEFAULT_SEND_TIMEOUT_MS 60000
#define DEFAULT_RECV_TIMEOUT_MS 60000
#define DEFAULT_SOCKET_TIMEOUT_MS 60000

namespace faabric::transport {

class MessageTimeoutException final : public faabric::util::FaabricException
{
  public:
    explicit MessageTimeoutException(std::string message)
      : FaabricException(std::move(message))
    {}
};

class MessageEndpointServer;

// Blocking helpers over a connected stream socket
void sendFrame(int fd,
               uint8_t code,
               const uint8_t* data,
               size_t size,
               int sequenceNum);

// Returns a Message with response code TERM if the peer closed, TIMEOUT on
// timeout (timeoutMs <= 0: wait forever)
Message recvFrame(int fd, int timeoutMs);

// Base: remembers where it points and lazily connects
class SendMessageEndpoint
{
  public:
    SendMessageEndpoint(const std::string& hostIn, int portIn, int timeoutMsIn);

    virtual ~SendMessageEndpoint();

    std::string getAddress() const { return host + ":" + std::to_string(port); }

    const std::string& getHost() const { return host; }

    int getPort() const { return port; }

  protected:
    std::string host;
    int port;
    int timeoutMs;
    std::unique_ptr<tcp::SendSocket> sock;
    std::mutex sockMx;

    // nullptr when the destination is not served from this process
    MessageEndpointServer* findLocalServer(bool sync);

    int connectedFd();

    void dropConnection();
};

// Fire-and-forget (PUSH-like)
class AsyncSendMessageEndpoint final : public SendMessageEndpoint
{
  public:
    AsyncSendMessageEndpoint(const std::string& hostIn,
                             int portIn,
                             int timeoutMs = DEFAULT_SEND_TIMEOUT_MS);

    void send(uint8_t header,
              const uint8_t* data,
              size_t dataSize,
              int sequenceNum = NO_SEQUENCE_NUM);
};

// Request / response (REQ-like)
class SyncSendMessageEndpoint final : public SendMessageEndpoint
{
  public:
    SyncSendMessageEndpoint(const std::string& hostIn,
                            int portIn,
                            int timeoutMs = DEFAULT_SEND_TIMEOUT_MS);

    void sendRaw(const uint8_t* data, size_t dataSize);

    Message sendAwaitResponse(uint8_t header,
                              const uint8_t* data,
                              size_t dataSize);
};

// In-process mailboxes addressed by label: the local leg of point-to-point
// messaging (reference: inproc:// push/pull and pair endpoints)
class InprocMailbox
{
  public:
    void send(Message&& msg) { queue.enqueue(std::move(msg)); }

    // Throws MessageTimeoutException
    Message recv(int timeoutMs);

    long size() { return queue.size(); }

  private:
    faabric::util::Queue<Message> queue;
};

std::shared_ptr<InprocMailbox> getInprocMailbox(const std::string& label);

void clearInprocMailbox(const std::string& label);

void clearAllInprocMailboxes();

class AsyncInternalSendMessageEndpoint final
{
  public:
    explicit AsyncInternalSendMessageEndpoint(
      const std::string& inprocLabel,
      int timeoutMs = DEFAULT_SEND_TIMEOUT_MS);

    void send(uint8_t header,
              const uint8_t* data,
              size_t dataSize,
              int sequenceNum = NO_SEQUENCE_NUM);

  private:
    std::shared_ptr<InprocMailbox> mailbox;
};

class AsyncInternalRecvMessageEndpoint final
{
  public:
    explicit AsyncInternalRecvMessageEndpoint(
      const std::string& inprocLabel,
      int timeoutMsIn = DEFAULT_RECV_TIMEOUT_MS);

    Message recv();

  private:
    std::shared_ptr<InprocMailbox> mailbox;
    int timeoutMs;
};

// Direct pair: same thing under the names the reference uses
using AsyncDirectSendEndpoint = AsyncInternalSendMessageEndpoint;
using AsyncDirectRecvEndpoint = AsyncInternalRecvMessageEndpoint;

// ---- stand-alone receiving endpoints (reference: MessageEndpoint.h:158-253).
// The servers of this runtime are MessageEndpointServer instances; these are
// the building blocks under their reference names for code that wants a bare
// socket to pull from: a bound port (or an in-process label) whose messages
// are read by one listener thread and handed out by recv().
class PortListener;

// Identifies one attached worker of a fan endpoint and the connection of the
// message it is working on (where sendResponse() replies)
class MessageContext final
{
  public:
    MessageContext() = default;

    int getWorkerId() const { return workerId; }

    bool isValid() const { return workerId >= 0; }

  private:
    friend class FanMessageEndpoint;
    friend class RecvMessageEndpoint;
    int workerId = -1;
    mutable int replyFd = -1;
    mutable int replySeq = NO_SEQUENCE_NUM;
};

class RecvMessageEndpoint
{
  public:
    // bound TCP port
    RecvMessageEndpoint(int portIn, int timeoutMsIn);

    // in-process label
    RecvMessageEndpoint(const std::string& inprocLabel, int timeoutMsIn);

    virtual ~RecvMessageEndpoint();

    // The next message; a Message with response code TIMEOUT when none arrived
    // in time, TERM once the endpoint was stopped
    virtual Message recv();

    int getPort() const { return port; }

    void stop();

  protected:
    int port = 0;
    int timeoutMs;
    std::shared_ptr<PortListener> listener;
    std::shared_ptr<InprocMailbox> mailbox;
    MessageContext last;

    Message doRecv(MessageContext& ctx);

    void reply(const MessageContext& ctx, uint8_t header, const uint8_t* data, size_t dataSize);
};

// PULL-like: messages only
class AsyncRecvMessageEndpoint final : public RecvMessageEndpoint
{
  public:
    explicit AsyncRecvMessageEndpoint(int portIn, int timeoutMs = DEFAULT_SOCKET_TIMEOUT_MS);

    explicit AsyncRecvMessageEndpoint(const std::string& inprocLabel, int timeoutMs = DEFAULT_SOCKET_TIMEOUT_MS);
};

// REP-like: every received message is answered on its connection
class SyncRecvMessageEndpoint final : public RecvMessageEndpoint
{
  public:
    explicit SyncRecvMessageEndpoint(int portIn, int timeoutMs = DEFAULT_SOCKET_TIMEOUT_MS);

    void sendResponse(uint8_t header, const uint8_t* data, size_t dataSize);
};

// One bound port whose messages are shared out between attached workers
// (reference: the fan-in / fan-out pair in front of a server's worker threads)
class FanMessageEndpoint
{
  public:
    FanMessageEndpoint(int portIn, int timeoutMsIn, bool isAsyncIn);

    virtual ~FanMessageEndpoint();

    MessageContext attachFanOut();

    // Blocks for this worker's next message (TIMEOUT / TERM codes as above)
    Message recv(const MessageContext& ctx);

    void sendResponse(const MessageContext& ctx, uint8_t header, const uint8_t* data, size_t dataSize);

    // Every blocked and future recv() returns TERM
    void stop();

    int getPort() const { return port; }

  private:
    int port;
    int timeoutMs;
    bool isAsync;
    std::shared_ptr<PortListener> listener;
    std::atomic<int> nWorkers{ 0 };
};

class AsyncFanMessageEndpoint final : public FanMessageEndpoint
{
  public:
    explicit AsyncFanMessageEndpoint(int portIn, int timeoutMs = DEFAULT_SOCKET_TIMEOUT_MS)
      : FanMessageEndpoint(portIn, timeoutMs, true)
    {}
};

class SyncFanMessageEndpoint final : public FanMessageEndpoint
{
  public:
    explicit SyncFanMessageEndpoint(int portIn, int timeoutMs = DEFAULT_SOCKET_TIMEOUT_MS)
      : FanMessageEndpoint(portIn, timeoutMs, false)
    {}
};

}

// ==========================================================================
// transport/MessageEndpointClient.h
// ==========================================================================
namespace faabric::transport {

// A (host, asyncPort, syncPort) client.  Endpoints are not created in mock mode
// (reference: src/transport/MessageEndpointClient.cpp:7-79).
class MessageEndpointClient
{
  public:
    MessageEndpointClient(std::string hostIn,
                          int asyncPortIn,
                          int syncPortIn,
                          int timeoutMs = DEFAULT_SOCKET_TIMEOUT_MS);

    virtual ~MessageEndpointClient() = default;

    // Serialised-message variants (any class with SerializeAsString)
    template<typename M>
    void asyncSend(int header, M* msg, int sequenceNum = NO_SEQUENCE_NUM)
    {
        std::string buffer = msg->SerializeAsString();
        asyncSend(header, (const uint8_t*)buffer.data(), buffer.size(), sequenceNum);
    }

    void asyncSend(int header,
                   const uint8_t* buffer,
                   size_t bufferSize,
                   int sequenceNum = NO_SEQUENCE_NUM);

    template<typename M, typename R>
    void syncSend(int header, M* msg, R* response)
    {
        std::string buffer = msg->SerializeAsString();
        syncSend(header, (const uint8_t*)buffer.data(), buffer.size(), response);
    }

    template<typename R>
    void syncSend(int header, const uint8_t* buffer, size_t bufferSize, R* response)
    {
        Message res = syncSendRaw(header, buffer, bufferSize);
        if (!response->ParseFromArray(res.udata().data(), (int)res.udata().size())) {
            throw std::runtime_error("Error deserialising message");
        }
    }

    Message syncSendRaw(int header, const uint8_t* buffer, size_t bufferSize);

    const std::string& getHost() const { return host; }

  protected:
    const std::string host;

  private:
    const int asyncPort;
    const int syncPort;

    AsyncSendMessageEndpoint asyncEndpoint;
    SyncSendMessageEndpoint syncEndpoint;
};

}

// ==========================================================================
// transport/MessageEndpointServer.h
// ==========================================================================
// Server skeleton: one async (PULL-like) and one sync (REP-like) listener, N
// worker threads each (reference: src/transport/MessageEndpointServer.cpp:
// 18-230).  All connections of a listener are multiplexed by one epoll I/O
// thread that frames messages and hands them to the workers.  Clients that live
// in the same process bypass the sockets through the server registry.



namespace faabric::transport {

// Dedicated thread count when none is given
#define DEFAULT_MESSAGE_SERVER_THREADS 4

class MessageEndpointServer;

class MessageEndpointServerHandler
{
  public:
    MessageEndpointServerHandler(MessageEndpointServer* serverIn,
                                 bool asyncIn,
                                 const std::string& inprocLabelIn,
                                 int nThreadsIn);

    ~MessageEndpointServerHandler();

    void start(int timeoutMs);

    void join();

    // In-process delivery: enqueue for a worker (async)
    void deliverLocal(Message&& msg);

    // In-process delivery of a TYPED request: the closure runs on a worker in
    // place of doAsyncRecv (no encode / decode of the payload)
    void deliverLocalTask(std::function<void()> task);

    int getPort() const { return port; }

  private:
    struct Impl;
    std::unique_ptr<Impl> impl;
    MessageEndpointServer* server;
    bool async;
    std::string inprocLabel;
    int nThreads;
    int port = 0;
};

class MessageEndpointServer
{
  public:
    MessageEndpointServer(int asyncPortIn,
                          int syncPortIn,
                          const std::string& inprocLabelIn,
                          int nThreadsIn);

    virtual ~MessageEndpointServer();

    virtual void start(int timeoutMs = DEFAULT_SOCKET_TIMEOUT_MS);

    virtual void stop();

    virtual void onWorkerStop();

    // Test hook: the next request waits on this latch after being handled
    void setRequestLatch();

    void awaitRequestLatch();

    int getNThreads() const { return nThreads; }

    bool isStarted() const { return started.load(); }

    // ---- used by handlers and by the in-process fast path ----
    virtual void doAsyncRecv(transport::Message& message) = 0;

    // Returns the serialised response
    virtual std::string doSyncRecv(transport::Message& message) = 0;

    void handleAsync(Message& msg);

    std::string handleSync(Message& msg);

    MessageEndpointServerHandler* getAsyncHandler() { return &asyncHandler; }

    static MessageEndpointServer* findLocal(int port, bool sync);

    // Typed in-process requests (see deliverLocalTask)
    void runAsyncTask(const std::function<void()>& task);

    // The server of this process listening on `port`, if any, when `host`
    // resolves to this process (virtual hosts included) and the in-process
    // fast path is enabled
    static MessageEndpointServer* localServerFor(const std::string& host, int basePort, bool sync);

  protected:
    int asyncPort;
    int syncPort;
    std::string inprocLabel;
    int nThreads;

  private:
    friend class MessageEndpointServerHandler;

    MessageEndpointServerHandler asyncHandler;
    MessageEndpointServerHandler syncHandler;

    std::atomic<bool> started{ false };
    std::shared_ptr<faabric::util::Latch> requestLatch;
    std::mutex latchMx;

    void afterRequest();
};

// "ip" / "localhost" / this host's address all count as local
bool isLocalAddress(const std::string& host);

}

// ==========================================================================
// transport/PointToPointCall.h
// ==========================================================================
namespace faabric::transport {

enum PointToPointCall
{
    MAPPING = 0,
    MESSAGE = 1,
    LOCK_GROUP = 2,
    LOCK_GROUP_RECURSIVE = 3,
    UNLOCK_GROUP = 4,
    UNLOCK_GROUP_RECURSIVE = 5,
    // MPI passive-target one-sided requests to the process of a target rank
    // (sync; see MpiWorld::serveRmaRequest) and the grant of a queued lock
    // back to the origin's process (async)
    RMA_LOCK = 6,
    RMA_LOCK_CANCEL = 7,
    RMA_FLUSH = 8,
    RMA_UNLOCK = 9,
    RMA_LOCK_GRANT = 10,
};

}

// ==========================================================================
// transport/PointToPointClient.h
// ==========================================================================
namespace faabric::transport {

// Mock-mode capture (reference: src/transport/PointToPointClient.cpp:11-49)
std::vector<std::pair<std::string, faabric::PointToPointMappings>>
getSentMappings();

std::vector<std::pair<std::string, faabric::PointToPointMessage>>
getSentPointToPointMessages();

std::vector<std::tuple<std::string,
                       faabric::transport::PointToPointCall,
                       faabric::PointToPointMessage>>
getSentLockMessages();

void clearSentMessages();

class PointToPointClient : public faabric::transport::MessageEndpointClient
{
  public:
    explicit PointToPointClient(const std::string& hostIn);

    void sendMappings(faabric::PointToPointMappings& mappings);

    void sendMessage(const faabric::PointToPointMessage& msg,
                     int sequenceNum = NO_SEQUENCE_NUM);

    void groupLock(int appId, int groupId, int groupIdx, bool recursive = false);

    void groupUnlock(int appId,
                     int groupId,
                     int groupIdx,
                     bool recursive = false);

    // MPI passive-target request (RMA_LOCK, RMA_LOCK_CANCEL, RMA_FLUSH,
    // RMA_UNLOCK): returns the reply bytes
    std::vector<uint8_t> rmaRequest(PointToPointCall call, const std::vector<uint8_t>& request);

    void rmaLockGrant(const uint8_t* buffer, size_t bytes);

  private:
    void makeCoordinationRequest(int appId,
                                 int groupId,
                                 int groupIdx,
                                 faabric::transport::PointToPointCall call);
};

// Per-thread cached client for a host
std::shared_ptr<PointToPointClient> getPointToPointClient(
  const std::string& host);

void clearPointToPointClients();

}

// ==========================================================================
// transport/PointToPointBroker.h
// ==========================================================================
// Group messaging between the functions of an app: idx -> host mappings pushed
// by the planner, ordered send/recv, distributed locks, barriers, notify.
// Reference: include/faabric/transport/PointToPointBroker.h:26-181,
// src/transport/PointToPointBroker.cpp:79-933.  Hosts are GPUs/worker
// processes of one box; local delivery goes through in-process mailboxes, so
// per-pair FIFO order holds by construction.  Device payloads do not travel
// here (MpiWorld moves them over NVLink); this is the control plane.



#define DEFAULT_DISTRIBUTED_TIMEOUT_MS 30000

#define POINT_TO_POINT_MAIN_IDX 0

#define NO_LOCK_OWNER_IDX -1

namespace faabric::transport {

class PointToPointBroker;

}
namespace faabric::device {
class Communicator;
}
namespace faabric::transport {

class PointToPointGroup
{
  public:
    static std::shared_ptr<PointToPointGroup> getGroup(int groupId);

    static std::shared_ptr<PointToPointGroup> getOrAwaitGroup(int groupId);

    static bool groupExists(int groupId);

    static void addGroup(int appId, int groupId, int groupSize);

    static void addGroupIfNotExists(int appId, int groupId, int groupSize);

    static void clearGroup(int groupId);

    static void clear();

    PointToPointGroup(int appId, int groupIdIn, int groupSizeIn);

    void lock(int groupIdx, bool recursive);

    void unlock(int groupIdx, bool recursive);

    int getLockOwner(bool recursive);

    void localLock();

    void localUnlock();

    bool localTryLock();

    // All members on GPU hosts with a device communicator attached
    // (PointToPointBroker::createLocalDeviceGroup / joinDeviceGroup): the
    // barrier is a device barrier (flag exchange over NVLink), stream-ordered;
    // otherwise the message-based barrier of the reference
    // (src/transport/PointToPointBroker.cpp:317-379)
    void barrier(int groupIdx);

    // Stream-ordered variant: returns without synchronising `stream`
    void deviceBarrier(int groupIdx, void* stream);

    void notify(int groupIdx);

    int getNotifyCount();

  private:
    friend class PointToPointServer;

    faabric::util::SystemConfig& conf;

    int timeoutMs = DEFAULT_DISTRIBUTED_TIMEOUT_MS;

    int appId = 0;
    int groupId = 0;
    int groupSize = 0;

    std::shared_ptr<faabric::util::Barrier> localBarrier;

    std::mutex mx;

    // Local lock (all group members on this host)
    std::timed_mutex localMx;
    std::recursive_timed_mutex localRecursiveMx;

    // Distributed lock state (lives on the main host)
    std::stack<int> recursiveLockOwners;
    int lockOwnerIdx = NO_LOCK_OWNER_IDX;
    std::queue<int> lockWaiters;

    void notifyLocked(int groupIdx);

    void masterLock(int groupIdx, bool recursive);

    void masterUnlock(int groupIdx, bool recursive);

    bool isSingleHost();
};

class PointToPointBroker
{
  public:
    PointToPointBroker();

    std::string getHostForReceiver(int groupId, int recvIdx);

    int getMpiPortForReceiver(int groupId, int recvIdx);

    std::set<std::string> setUpLocalMappingsFromSchedulingDecision(
      const faabric::batch_scheduler::SchedulingDecision& decision);

    void setAndSendMappingsFromSchedulingDecision(
      const faabric::batch_scheduler::SchedulingDecision& decision);

    void sendMappingsFromSchedulingDecision(
      const faabric::batch_scheduler::SchedulingDecision& decision,
      const std::set<std::string>& hostList);

    void waitForMappingsOnThisHost(int groupId);

    std::set<int> getIdxsRegisteredForGroup(int groupId);

    std::set<std::string> getHostsRegisteredForGroup(int groupId);

    void updateHostForIdx(int groupId, int groupIdx, std::string newHost);

    void sendMessage(int groupId,
                     int sendIdx,
                     int recvIdx,
                     const uint8_t* buffer,
                     size_t bufferSize,
                     std::string hostHint,
                     bool mustOrderMsg = false);

    void sendMessage(int groupId,
                     int sendIdx,
                     int recvIdx,
                     const uint8_t* buffer,
                     size_t bufferSize,
                     bool mustOrderMsg = false,
                     int sequenceNum = NO_SEQUENCE_NUM,
                     std::string hostHint = "");

    std::vector<uint8_t> recvMessage(int groupId,
                                     int sendIdx,
                                     int recvIdx,
                                     bool mustOrderMsg = false);

    void clearGroup(int groupId);

    void clear();

    void resetThreadLocalCache();

    void postMigrationHook(int groupId, int groupIdx);

    // ---- device data plane: group idx <-> GPU ----
    // Messages whose payload lives in HBM move with the communicator's
    // point-to-point kernels (eager send into the sender's heap + pull over
    // NVLink).  Per (sender, receiver) FIFO ordering is inherent, so the
    // reference's sequence numbers / out-of-order buffer
    // (src/transport/PointToPointBroker.cpp:557-600,778-859) are not needed.
    //
    // All members in this process (one worker serving per-GPU virtual hosts):
    // devices[i] is the GPU of group idx i; empty => taken from the host names
    // of the group's mappings ("gpuN" -> N).
    void createLocalDeviceGroup(int groupId, std::vector<int> devices = {});

    // One member per process: collective call, every idx joins
    void joinDeviceGroup(int groupId, int groupIdx, int groupSize, int device);

    bool isDeviceGroup(int groupId);

    std::shared_ptr<faabric::device::Communicator> getDeviceCommunicator(int groupId, int groupIdx);

    // Stream-ordered; the buffers are device pointers
    void sendDeviceMessage(int groupId,
                           int sendIdx,
                           int recvIdx,
                           const void* deviceBuffer,
                           size_t bufferSize,
                           void* stream);

    void recvDeviceMessage(int groupId,
                           int sendIdx,
                           int recvIdx,
                           void* deviceBuffer,
                           size_t bufferSize,
                           void* stream);

    // Delivery into the local mailbox of (group, send, recv); used by the
    // server for messages that arrive from other hosts
    void deliverLocally(int groupId,
                        int sendIdx,
                        int recvIdx,
                        const uint8_t* buffer,
                        size_t bufferSize,
                        int sequenceNum);

  private:
    faabric::util::SystemConfig& conf;

    std::shared_mutex brokerMutex;

    std::unordered_map<int, std::set<int>> groupIdIdxsMap;
    std::unordered_map<std::string, std::string> mappings;
    std::unordered_map<std::string, int> mpiPortMappings;

    std::unordered_map<int, std::shared_ptr<faabric::util::FlagWaiter>>
      groupFlags;

    // groupId -> communicator of every idx served by this process
    std::unordered_map<int, std::map<int, std::shared_ptr<faabric::device::Communicator>>> deviceComms;

    // Sender side sequence counters, keyed by (group, send, recv)
    std::mutex seqMx;
    std::unordered_map<std::string, int> sentMsgCount;

    std::shared_ptr<faabric::util::FlagWaiter> getGroupFlag(int groupId);

    Message doRecvMessage(int groupId, int sendIdx, int recvIdx);

    int getAndIncrementSentMsgCount(int groupId, int sendIdx, int recvIdx);
};

PointToPointBroker& getPointToPointBroker();

}

// ==========================================================================
// transport/PointToPointServer.h
// ==========================================================================
namespace faabric::transport {

class PointToPointServer final : public MessageEndpointServer
{
  public:
    PointToPointServer();

  private:
    PointToPointBroker& broker;

    void doAsyncRecv(transport::Message& message) override;

    std::string doSyncRecv(transport::Message& message) override;

    void onWorkerStop() override;

    std::string doRecvMappings(std::span<const uint8_t> buffer);

    void recvGroupLock(std::span<const uint8_t> buffer, bool recursive);

    void recvGroupUnlock(std::span<const uint8_t> buffer, bool recursive);
};

}

// ==========================================================================
// transport/common.h
// ==========================================================================
// Well-known ports (reference: include/faabric/transport/common.h:9-29).  With
// one worker process per GPU on a box, FAABRIC_PORT_OFFSET shifts the whole
// block so workers do not collide.
#ifndef ANY_HOST
#define ANY_HOST "0.0.0.0"
#endif
#define DEFAULT_STATE_HOST ANY_HOST
#define STATE_ASYNC_PORT 8003
#define STATE_SYNC_PORT 8004
#define STATE_INPROC_LABEL "state"

#define DEFAULT_FUNCTION_CALL_HOST ANY_HOST
#define FUNCTION_CALL_ASYNC_PORT 8005
#define FUNCTION_CALL_SYNC_PORT 8006
#define FUNCTION_INPROC_LABEL "function"

#define DEFAULT_SNAPSHOT_HOST ANY_HOST
#define SNAPSHOT_ASYNC_PORT 8007
#define SNAPSHOT_SYNC_PORT 8008
#define SNAPSHOT_INPROC_LABEL "snapshot"

#define DEFAULT_POINT_TO_POINT_HOST "0.0.0.0"
#define POINT_TO_POINT_ASYNC_PORT 8009
#define POINT_TO_POINT_SYNC_PORT 8010
#define POINT_TO_POINT_INPROC_LABEL "ptp"

#define PLANNER_ASYNC_PORT 8011
#define PLANNER_SYNC_PORT 8012
#define PLANNER_INPROC_LABEL "planner"

#define MPI_BASE_PORT 8020

namespace faabric::transport {

// host may be "ip" or "ip:offset": several workers of one box (one per GPU)
// register with the planner as distinct hosts distinguished by a port offset
struct HostAddress
{
    std::string ip;
    int portOffset = 0;
};

HostAddress parseHostAddress(const std::string& host);

// Virtual host names (e.g. one per GPU of this box) served by another address
void registerHostAlias(const std::string& alias, const std::string& realAddress);

void clearHostAliases();

std::string resolveHostAlias(const std::string& host);

// True if `host` is a registered virtual host name
bool isHostAlias(const std::string& host);

// Same worker? (a virtual host and the address serving it, two virtual hosts
// of one worker, ...).  Empty names match nothing.
bool sameWorker(const std::string& hostA, const std::string& hostB);

std::string makeHostAddress(const std::string& ip, int portOffset);

// Address other workers use to reach this worker
std::string getThisHostAddress();

}

