// Communicator: one per MPI rank / GPU.  Owns the symmetric heap + signal pad,
// knows every peer's mapping of them (NVLink P2P, optional NVLS multicast) and
// launches the fused collective kernels.  All operations are stream-ordered
// and never synchronise the host; they are CUDA-graph capturable.
//
// Two wiring modes:
//   * local : all ranks live in this process (rank threads, like the
//             reference's one-thread-per-rank model), one or several GPUs;
//             several ranks may share a GPU (used by single-GPU tests).
//   * ipc   : one process per GPU (torchrun-style); handles are exchanged over
//             the Unix-socket Bootstrap (VMM fds, or legacy CUDA IPC).
#pragma once

#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <cstddef>
#include <deque>
#include <initializer_list>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "faabric/device/comm_abi.h"

namespace fb {
struct KernelTable;
struct GroupSeg;
struct GroupArgs;
}

namespace faabric::device {

class Bootstrap;

// Buffers are symmetric-heap pointers at identical offsets on every rank
#define FB_FLAG_SYMMETRIC 1
// Skip cross-rank synchronisation (profiling a single rank's data path only)
#define FB_FLAG_NOSYNC 2
// Channel id in bits 8..11: independent collectives issued on different
// channels (and different streams) may execute concurrently.  Every rank must
// use the same channel for the same logical collective.  Channels > 0 require
// symmetric buffers (the staging area is not replicated per channel).
#define FB_FLAG_CHANNEL(c) (((c) & 0xf) << 8)
#define FB_FLAG_GET_CHANNEL(f) (((f) >> 8) & 0xf)

struct CommConfig
{
    size_t heapBytes = (size_t)256 << 20; // user-visible symmetric heap
    size_t stageBytes = (size_t)32 << 20; // each of the two staging buffers
    size_t slotBytes = (size_t)128 << 10; // (legacy knob, unused)
    // p2p: bytes of bounce ring per destination peer in the sender's heap;
    // messages up to half of it are sent eagerly in one piece
    size_t p2pBounceBytes = (size_t)8 << 20;
    // CTAs of a grouped all-reduce launch (0 = as many as there are barrier
    // slots for the channel, capped at 128)
    int groupBlocks = 0;
    // Loopback backend (FAABRIC_DEVICE_BACKEND=loopback): heaps and signal
    // pads in host memory, every kernel replaced by its host twin executed on
    // the calling rank thread.  No GPU needed; one thread per rank.
    bool loopback = false;
    // Cross-rank synchronisation with stream memory operations instead of
    // in-kernel spins: needed when kernels of different ranks may not be
    // co-resident (ranks sharing one GPU, kernel-serialising profilers).
    // -1 = decide at creation (on when two ranks share a device)
    int streamSync = -1;
    uint64_t timeoutMs = 10000;           // device spin watchdog
    bool useVmm = true;
    bool useMulticast = true;
    int maxBlocks = 32;
    int threads = 512;
    int channels = 4; // concurrent collective lanes (1..FB_MAX_CHANNELS)
    // algorithm thresholds (bytes); the autotuner overwrites these
    size_t llMaxBytes = 32 << 10;
    size_t oneShotMaxBytes = 256 << 10;
    size_t nvlsMinBytes = 128 << 10;
    // integer / f64 reductions use NVLS only above this size (AUTO)
    size_t nvlsScalarMinBytes = (size_t)32 << 20;
    size_t bcast2StepMinBytes = 1 << 20;
    // pull collectives use the TMA bulk-copy engine from this chunk size
    // (per source/destination pair); 0 = never
    size_t tmaMinBytes = 256 << 10;

    // Fills defaults from FAABRIC_* environment variables
    static CommConfig fromEnv();
};

// Tuning file written by the autotuner (`python -m faabric_b200.parallel.autotune`)
// and read by every communicator when FAABRIC_TUNING_FILE names it.  One
// directive per line, '#' starts a comment:
//   allreduce <maxBytes> <oneshot|twoshot|nvls|ll>   selection table row
//   set <key> <value>                                CommConfig threshold, keys
//       llMaxBytes oneShotMaxBytes nvlsMinBytes nvlsScalarMinBytes
//       bcast2StepMinBytes tmaMinBytes maxBlocks threads channels
struct CommTuning
{
    std::vector<std::pair<uint64_t, int>> allReduceTable;
    std::vector<std::pair<std::string, uint64_t>> settings;

    // Throws std::runtime_error naming the offending line
    static CommTuning parse(const std::string& text);
    // false if the file cannot be read; parse errors throw
    static bool loadFile(const std::string& path, CommTuning& out);
    std::string serialise() const;
    void applyTo(CommConfig& cfg) const;
    bool empty() const { return allReduceTable.empty() && settings.empty(); }

    static int algoFromName(const std::string& name);
    static const char* algoName(int algo);
};

struct CommStats
{
    uint64_t launches = 0;
    uint64_t bytes = 0;
    uint64_t algoCount[FB_ALGO_COUNT] = { 0 };
    uint64_t stagedCopies = 0;
    uint64_t tmaLaunches = 0;
    // grouped segment tables built and uploaded: one per launch of a plan
    // prepareGroup makes, one per grouped batch of groupMany
    uint64_t segTables = 0;
};

class Communicator : public std::enable_shared_from_this<Communicator>
{
  public:
    ~Communicator();

    static std::vector<std::shared_ptr<Communicator>> createLocal(
      int nranks,
      const std::vector<int>& devices,
      const CommConfig& cfg);

    static std::shared_ptr<Communicator> createIpc(int rank,
                                                   int nranks,
                                                   int device,
                                                   const std::string& jobId,
                                                   const CommConfig& cfg);

    // ---- sub-communicators ----
    // Local call: no communication, no allocation.  `members` are ranks of this
    // communicator, in the order that becomes the child's rank order; this rank
    // must be one of them.  Every member must pass the same list and slot.
    // The child runs the same fused kernels over the members' heaps, with slot
    // `slot` of every member's signal region as its pads (comm_abi.h).  It
    // supports allReduce (one-shot and two-shot only), reduce, reduceScatter,
    // scan, the data-movement collectives, the grouped calls (plans and
    // *Many), barrier and the heap queries, with child ranks.  Point to
    // point, put-signal, the one-sided atomics, hostBarrier and subset return
    // FB_E_UNSUPPORTED;
    // alloc / free throw std::logic_error (heap allocation is collective over
    // the whole parent).  A child and its parent share this rank's staging
    // buffers: calls on both from one rank must be stream-ordered unless the
    // buffers are symmetric.  Returns null and sets *rc to FB_E_INVALID for an
    // empty list, a member out of range or repeated, this rank not a member,
    // or a slot out of range or in use on this rank.  Destroying the child
    // zeroes this rank's slot pad on a stream of its own, then frees the slot.
    // A child's *Many tables live in its parent's table ring (on the parent's
    // device, freed with the parent); a plan prepared on a child owns its
    // tables and frees them with cudaFree on the child's device when the
    // last reference to the plan goes.  The ring's host state is shared and
    // not synchronised: one host thread must drive a rank's parent and all
    // of its children (as MPI rank threads and LocalGroup.run do).
    // Precondition: this rank's last collective on the child has completed
    // (its stream has been waited for); the destructor does not order itself
    // after the caller's streams.
    std::shared_ptr<Communicator> subset(const std::vector<int>& members, int slot, int* rc = nullptr);
    // bit s set: slot s is free on this rank
    uint32_t freeSubsetSlots() const;
    bool isSubset() const { return parent_ != nullptr; }

    int rank() const { return dev_.rank; }
    int size() const { return dev_.nranks; }
    int device() const { return device_; }
    bool hasMulticast() const { return dev_.mcHeap != nullptr; }
    bool isLoopback() const { return loop_; }
    const std::string& backing() const { return backing_; }
    const FbCommDev& devStruct() const { return dev_; }
    CommConfig& config() { return cfg_; }
    const CommStats& stats() const { return stats_; }
    void resetStats() { stats_ = CommStats(); }

    // ---- symmetric heap allocator (call collectively, same order/sizes) ----
    // Returns an offset usable with heapPtr(); throws std::bad_alloc when full
    uint64_t alloc(size_t bytes, size_t align = 256);
    void free(uint64_t offset);
    uint8_t* heapPtr(uint64_t offset, int rank = -1) const;
    bool inHeap(const void* p, size_t bytes = 1) const;

    // In the symmetric heap of ANY communicator of this process (device or
    // loopback): a range check, no driver call
    static bool isHeapPointer(const void* p);
    uint64_t offsetOf(const void* p) const;
    size_t userHeapBytes() const { return cfg_.heapBytes; }

    // True if the reduction kernels implement (FbDtype, FbOp); the reductions
    // return FB_E_UNSUPPORTED for other pairs
    static bool reduces(int dtype, int op);

    // ---- collectives.  Return 0 or a negative FB_E_* code.  `bytes`-based
    // calls are type-agnostic; reductions take FbDtype / FbOp. ----
    int allReduce(const void* send,
                  void* recv,
                  size_t count,
                  int dtype,
                  int op,
                  int algo,
                  int flags,
                  cudaStream_t s);
    int reduce(const void* send,
               void* recv,
               size_t count,
               int dtype,
               int op,
               int root,
               int flags,
               cudaStream_t s);
    int reduceScatter(const void* send,
                      void* recv,
                      size_t recvCount,
                      int dtype,
                      int op,
                      int flags,
                      cudaStream_t s);
    int scan(const void* send,
             void* recv,
             size_t count,
             int dtype,
             int op,
             int flags,
             cudaStream_t s);
    // (Reductions with FB_FLAG_SYMMETRIC take heap buffers at any heap
    // offset: an input, or a pushed output, at an offset that is not a
    // multiple of 16 goes through the staging copy.)
    // Data movement.  Local (non-heap) destinations may sit at any alignment,
    // different on every rank.  With FB_FLAG_SYMMETRIC, every rank passes
    // the same kind of buffer at the same heap offset, outputs included: an
    // all-gather output in the heap on one rank is in the heap on all.
    int broadcast(void* buf, size_t bytes, int root, int flags, cudaStream_t s);
    int allGather(const void* send,
                  void* recv,
                  size_t bytesPerRank,
                  int flags,
                  cudaStream_t s);
    int gather(const void* send,
               void* recv,
               size_t bytesPerRank,
               int root,
               int flags,
               cudaStream_t s);
    int scatter(const void* send,
                void* recv,
                size_t bytesPerRank,
                int root,
                int flags,
                cudaStream_t s);
    int allToAll(const void* send,
                 void* recv,
                 size_t bytesPerRank,
                 int flags,
                 cudaStream_t s);
    int barrier(cudaStream_t s);

    // ---- grouped all-reduce: many independent all-reduces, ONE launch ----
    struct GroupItem
    {
        const void* send; // symmetric heap, 16-byte aligned
        void* recv;       // symmetric heap, 16-byte aligned (may equal send)
        size_t count;     // elements
    };
    struct GroupPlan;
    // What a plan's launches compute.  For the two shard kinds, GroupItem
    // .count is the per-rank element count (MPI recvcount / sendcount):
    //   GROUP_REDUCE_SCATTER: send holds size()*count elements; recv gets op
    //     over every rank p of send_p[rank*count, (rank+1)*count)
    //     (MPI_Reduce_scatter_block per item)
    //   GROUP_ALLGATHER: send holds count elements; block p of recv (size()
    //     *count elements) gets send of rank p (MPI_Allgather per item; a
    //     byte copy, any dtype)
    //   GROUP_BROADCAST: recv holds count elements (send is not read); every
    //     rank's recv gets the root's (MPI_Bcast per item; a byte copy, any
    //     dtype, any length).  Cut into equal ranges like the all-reduce.
    //   GROUP_ALLTOALL: send and recv hold size()*count elements each; block
    //     r of recv on rank p gets block p of send on rank r (MPI_Alltoall
    //     per item; a byte copy, any dtype)
    //   GROUP_GATHER: send holds count elements on every rank; block p of
    //     the root's recv (size()*count elements) gets send of rank p
    //     (MPI_Gather per item; a byte copy, any dtype).  recv is read on the
    //     root only (null elsewhere is fine).  send == recv + root*count*esize
    //     at the root is in place.
    //   GROUP_SCATTER: the mirror image: block p of the root's send
    //     (size()*count elements) goes to recv (count elements) of rank p;
    //     send is read on the root only; recv == send + root*count*esize at
    //     the root is in place.
    //   GROUP_REDUCE: send holds count elements on every rank; the root's
    //     recv (count elements) gets op over the ranks' sends in rank order,
    //     acc = send_0, acc = op(acc, send_p) for p = 1..size()-1
    //     (MPI_Reduce per item).  recv is read on the root only (null
    //     elsewhere is fine; no other rank's recv is written).  send == recv
    //     at the root is in place.
    //   GROUP_SCAN: send and recv hold count elements on every rank; rank r's
    //     recv gets op over the sends of ranks 0..r in rank order, acc =
    //     send_0, acc = op(acc, send_p) for p = 1..r (MPI_Scan per item).
    //     `root` is ignored.  send == recv is in place, on any rank.
    //   GROUP_EXSCAN: the same fold over ranks 0..r-1 (MPI_Exscan per item).
    //     Rank 0's recv is not written; on a one-member communicator nothing
    //     is written or launched.
    // Shard kinds (GROUP_REDUCE_SCATTER, GROUP_ALLGATHER, GROUP_ALLTOALL)
    // group an item only if send and recv are in the symmetric heap and
    // 16-byte aligned, count*esize is a multiple of 16, and recv overlaps no
    // send of the group on this rank.  The one exception is the in-place
    // all-gather, send == recv + rank*count*esize.  Items with count 0 are
    // skipped.
    //   GROUP_NEIGHBOR_ALLGATHER: over the topology of setNeighbors, send
    //     holds count elements and recv indeg*count; block j of recv gets
    //     the send of in-edge j's source (MPI_Neighbor_allgather per item)
    //   GROUP_NEIGHBOR_ALLTOALL: send holds outdeg*count elements and recv
    //     indeg*count; block j of recv gets block idx of the send of in-edge
    //     j = (source, idx) (MPI_Neighbor_alltoall per item)
    //   Both are byte copies of any dtype, with buffers of any device memory
    //   at any alignment (a rank's send is not read when its out-degree is
    //   0, nor its recv written when its in-degree is 0; either may then be
    //   null).  Every rank stages its send blocks, then pulls its in-edges'
    //   blocks from their sources' staging.  A launch holds at most
    //   CommConfig::stageBytes of staging per rank (the all-to-all: the
    //   largest out-degree times the launch's blocks), so a larger list is
    //   cut into several launches, at the same points on every rank.  A rank
    //   with no edge still takes part in every launch; a graph with no edge
    //   launches nothing.
    // Rooted kinds (GROUP_GATHER, GROUP_SCATTER, GROUP_REDUCE, GROUP_SCAN,
    // GROUP_EXSCAN) group every item with count > 0: buffers are any device
    // memory of this rank, at any alignment and length, and may differ
    // between ranks.  The data goes through every rank's staging buffers (the
    // reduce's and scan's results through a second one), so a plan depends
    // on neither the root nor the op, and a launch holds at most CommConfig::stageBytes per rank (rounded to
    // chunks); a larger item is cut into pieces at the same points on every
    // rank.
    enum GroupKind
    {
        GROUP_ALLREDUCE = 0,
        GROUP_REDUCE_SCATTER = 1,
        GROUP_ALLGATHER = 2,
        GROUP_BROADCAST = 3,
        GROUP_ALLTOALL = 4,
        GROUP_GATHER = 5,
        GROUP_SCATTER = 6,
        GROUP_REDUCE = 7,
        GROUP_SCAN = 8,
        GROUP_EXSCAN = 9,
        GROUP_NEIGHBOR_ALLGATHER = 10,
        GROUP_NEIGHBOR_ALLTOALL = 11,
        GROUP_NEIGHBOR_ALLGATHERV = 12,
        GROUP_NEIGHBOR_ALLTOALLV = 13
    };
    // Where the next launch of a list starts: an item, and a byte offset in
    // it (rooted kinds cut items larger than the staging buffer)
    struct GroupCursor
    {
        size_t item = 0;
        uint64_t offset = 0;
    };
    // Builds (and uploads) this rank's segment tables.  Collective: every rank
    // must pass the same list (same offsets, same counts; the rooted kinds
    // need the same counts only).  Returns null and
    // sets *rc when an item is not symmetric / aligned (FB_E_INVALID).  Works
    // on a sub-communicator's child as on any other communicator.
    std::shared_ptr<GroupPlan> prepareGroup(const GroupItem* items,
                                            size_t nItems,
                                            int dtype,
                                            int* rc = nullptr,
                                            GroupKind kind = GROUP_ALLREDUCE);
    // Launches a prepared plan of `kind`.  groupMany prepares and launches a
    // transient list (the MPI bursts), batch by batch; a batch that cannot be
    // grouped runs as per-item allReduce / reduceScatter / allGather /
    // broadcast / allToAll calls and returns their errors (reduceScatter
    // refuses shards that are not a multiple of 16 bytes with
    // FB_E_UNSUPPORTED).  `op` is read by the reducing kinds (GROUP_ALLREDUCE,
    // GROUP_REDUCE_SCATTER, GROUP_REDUCE, GROUP_SCAN, GROUP_EXSCAN) only,
    // `root` by GROUP_BROADCAST, GROUP_GATHER, GROUP_SCATTER and GROUP_REDUCE
    // only.  Both follow the same rules:
    //   - a plan of another kind, an unknown kind or a dtype of no size:
    //     FB_E_INVALID
    //   - reducing kinds: a (dtype, op) pair with no reduction at all gives
    //     FB_E_UNSUPPORTED; a pair with no grouped kernel gives
    //     FB_E_UNSUPPORTED from runGroup, and per-item calls from groupMany
    //   - GROUP_BROADCAST: a root that is not a rank of this communicator
    //     gives FB_E_INVALID; the root's buffers are only read; on a
    //     one-member communicator nothing is launched (FB_OK).  For
    //     groupMany, pass each buffer as send and recv with FB_U8 and byte
    //     counts.
    //   - GROUP_ALLTOALL on a one-member communicator runs as a local copy
    //   - GROUP_GATHER, GROUP_SCATTER, GROUP_REDUCE: a root that is not a
    //     rank of this communicator, or a channel other than 0 (the staging
    //     buffers are per rank, not per channel), gives FB_E_INVALID; so does
    //     a missing buffer this rank needs (every rank's own side -- the send
    //     of a gather or reduce -- and both on the root), checked over the
    //     whole list before its first launch.  On a one-member communicator
    //     the launch is a local copy (nothing when in place).  With
    //     FB_FLAG_NOSYNC nothing orders a peer's staging copy against the
    //     root's, so the bytes received are unspecified (the flag profiles
    //     one rank's data path only).  GROUP_REDUCE has a grouped kernel for
    //     every (dtype, op) pair that has a reduction.
    //   - GROUP_SCAN, GROUP_EXSCAN: as the rooted kinds above, with no root
    //     (any value is accepted), and every rank needs both its send and
    //     its recv.  Every (dtype, op) pair that has a reduction has a grouped
    //     kernel.
    //   - GROUP_NEIGHBOR_ALLGATHER, GROUP_NEIGHBOR_ALLTOALL: a communicator
    //     without a topology, a channel other than 0, or a missing buffer
    //     this rank needs (the send with an out-edge, the recv with an
    //     in-edge) gives FB_E_INVALID, checked over the whole list before
    //     its first launch; `op` and `root` are ignored.  On a one-member
    //     communicator the launch is a local copy.
    //   - GROUP_ALLREDUCE sets lastAlgo() to FB_ALGO_TWOSHOT
    int runGroup(GroupKind kind, const GroupPlan& plan, int op, int root, int flags, cudaStream_t s);
    int groupMany(GroupKind kind,
                  const GroupItem* items,
                  size_t nItems,
                  int dtype,
                  int op,
                  int root,
                  int flags,
                  cudaStream_t s);
    // Kernel launches of a plan (a v plan's launch window runs as several
    // rounds)
    static size_t groupPlanLaunches(const GroupPlan& plan);
    // "all-reduce", "reduce-scatter", "all-gather", "broadcast", "all-to-all",
    // "gather", "scatter", "reduce", "scan", "exscan", "neighbor-allgather",
    // "neighbor-alltoall", "neighbor-allgatherv", "neighbor-alltoallv"
    static const char* groupKindName(GroupKind kind);

    // ---- grouped neighbourhood v-collectives ----
    // One MPI_Neighbor_allgatherv / MPI_Neighbor_alltoallv call of a list over
    // the topology of setNeighbors, with counts and displacements in elements
    // of the list's dtype:
    //   GROUP_NEIGHBOR_ALLGATHERV: send holds sendCounts[0] elements (one
    //     count; sendDispls is not read); recv block j (recvCounts[j]
    //     elements at recvDispls[j]) gets the send of in-edge j's source
    //   GROUP_NEIGHBOR_ALLTOALLV: send block i (sendCounts[i] elements at
    //     sendDispls[i]) goes to out-edge i; recv block j gets the send block
    //     idx of in-edge j = (source, idx)
    // The arrays hold an entry per out-edge and per in-edge of this rank (none
    // are read for a degree of 0), and are read only by the call that takes
    // the item.  A block's count must equal the count its peer gives for the
    // same edge, as MPI requires.  Byte copies of any dtype, buffers in any
    // device memory at any alignment; a buffer may be null where all its
    // counts are 0.
    struct NeighborVItem
    {
        const void* send;
        void* recv;
        const size_t* sendCounts;
        const size_t* sendDispls;
        const size_t* recvCounts;
        const size_t* recvDispls;
    };
    // A v list runs in launch windows of whole items, cut from the largest
    // degrees alone, so every member cuts alike.  Stream k of a rank in a
    // window is the concatenation, in item order, of its edge-k blocks; a
    // launch moves at most the staging room of every stream (a round), so a
    // window takes ceil(M / W) launches, where M is its largest stream over
    // every member and W the room of one staging slot (CommConfig::stageBytes
    // over the largest out-degree for the all-to-all, rounded to
    // FB_NEIGHBOR_CHUNK, and at most M rounded up to it).  A rank knows only
    // its own streams, so M is agreed by the caller:
    //   neighborVStreams: this rank's largest stream of every window, in
    //     bytes (local; `out` gets one entry per window, none when no member
    //     has an edge);
    //   the caller takes the elementwise maximum over every member and passes
    //     it as `agreed` to prepareGroup / groupMany, which refuse a list whose
    //     agreement is shorter or longer than its windows or below one of this
    //     rank's own streams (FB_E_INVALID).  A window whose agreement is 0
    //     launches nothing.
    // Refusals, all before any launch: the rules of the equal-block neighbour
    // kinds (a communicator without a topology or a channel other than 0:
    // FB_E_INVALID), a missing count array or buffer that this rank needs
    // (FB_E_INVALID), and degrees too large for one item per window
    // (FB_E_TOO_LARGE: the largest out-degree plus in-degree above
    // FB_NEIGHBOR_V_MAX_DEGREE).  runGroup launches a v plan like any other.
    int neighborVStreams(GroupKind kind,
                         const NeighborVItem* items,
                         size_t nItems,
                         int dtype,
                         std::vector<uint64_t>& out) const;
    std::shared_ptr<GroupPlan> prepareGroup(const NeighborVItem* items,
                                            size_t nItems,
                                            int dtype,
                                            const std::vector<uint64_t>& agreed,
                                            int* rc,
                                            GroupKind kind);
    int groupMany(GroupKind kind,
                  const NeighborVItem* items,
                  size_t nItems,
                  int dtype,
                  const std::vector<uint64_t>& agreed,
                  int flags,
                  cudaStream_t s);

    // ---- neighbourhood topology of the neighbour kinds ----
    // This rank's in-edges in recv-block order, each (source rank, index of
    // the edge among the source's out-edges), and its out-degree.  The
    // largest out-degree and in-degree over every member must be passed
    // alike by every member: the staging layout and the launch cuts follow
    // from them.  Self-edges and multi-edges are allowed.  Local call, set
    // once, before the first neighbour call; the caller checks that the
    // members' edges agree (a source's out-edges are the in-edges naming
    // it).  FB_E_INVALID for a second call, a source outside the
    // communicator, an index outside [0, maxOutDegree), a degree above its
    // maximum, or more than FB_NEIGHBOR_MAX_IN_DEGREE in-edges.
    int setNeighbors(const std::vector<std::pair<int, int>>& inEdges,
                     int outDegree,
                     int maxOutDegree,
                     int maxInDegree);
    bool hasNeighbors() const { return topo_ != nullptr; }
    // This rank's (in-degree, out-degree); (0, 0) without a topology
    std::pair<int, int> neighborDegrees() const;

    // ---- point to point (per-pair FIFO; no kernel ever spins on a peer) ----
    // Operations on one ordered pair must be issued in a consistent stream
    // order on both sides.  `peer == rank()` is allowed (self message).
    int send(const void* buf, size_t bytes, int peer, cudaStream_t s);
    int recv(void* buf, size_t bytes, int peer, cudaStream_t s);
    // Exchange without the send-before-recv ordering hazard of big messages:
    // chunks of both directions are interleaved
    int sendRecv(const void* sendBuf,
                 size_t sendBytes,
                 int dst,
                 void* recvBuf,
                 size_t recvBytes,
                 int src,
                 cudaStream_t s);
    // A non-blocking stream owned by this communicator, for host-driven
    // operations that have no caller stream (group barriers).  Never the
    // legacy default stream: ranks sharing a device would serialise on it.
    cudaStream_t internalStream();
    bool streamSync() const { return streamSync_; }
    bool streamWaitSupported() const { return streamWaitOk_; }
    // Bounded wait for `s` (polls; never blocks forever on a stream-level wait
    // whose peer died).  Returns false after releasing the stuck waits.
    bool syncStreamBounded(cudaStream_t s, uint64_t timeoutMs);
    // Low-latency completion wait for host-synchronous callers (the MPI C
    // API): a stream-ordered write into host-mapped memory is polled by the
    // CPU, which saves the driver round trip of cudaStreamSynchronize.  Falls
    // back to it without stream memory operations.  False on a CUDA error.
    bool waitStreamFast(cudaStream_t s);
    // zero-copy put into a peer's symmetric buffer + signal bump
    int putSignal(const void* local,
                  uint64_t dstOffset,
                  size_t bytes,
                  int peer,
                  int signalIdx,
                  int blocks,
                  cudaStream_t s);
    int waitSignal(int signalIdx, uint32_t count, cudaStream_t s);
    // ---- one-sided atomics (MPI_Accumulate family) on a peer's symmetric heap.
    // Stream-ordered, never synchronise the host; `peer == rank()` is allowed.
    // The target is `count` elements at `dstOffset` in the user part of peer's
    // heap, each aligned to its size; origin and fetch buffers are device-
    // accessible and need no alignment.  Each target element is updated
    // atomically with respect to every other accumulate / compare-and-swap on
    // any rank.  `op` is any reduction pair of allReduce, FB_OP_REPLACE, or
    // FB_OP_NO_OP (an atomic read; needs `fetchOut`).  `fetchOut` (null: no
    // fetch) receives every element's previous value.  FB_E_UNSUPPORTED for
    // an unsupported pair, FB_E_INVALID for a range outside the heap, a
    // misaligned target or NO_OP without `fetchOut`.
    int accumulate(const void* origin,
                   uint64_t dstOffset,
                   size_t count,
                   int dtype,
                   int op,
                   int peer,
                   void* fetchOut,
                   cudaStream_t s);
    // One integer element: *result = old; if (old == *compare) target = *swap
    int compareAndSwap(const void* compare,
                       const void* swap,
                       void* result,
                       uint64_t dstOffset,
                       int dtype,
                       int peer,
                       cudaStream_t s);
    // ---- batched one-sided copies (request-based MPI_Rput / MPI_Rget) ----
    struct RmaCopy
    {
        void* local;     // memory this rank's GPU can load and store
        uint64_t offset; // user part of peer's symmetric heap
        size_t bytes;
        int peer;
        int get; // 0: local -> peer's heap at offset; 1: the other way
    };
    // Every item of the list, as one launch per FB_RMA_COPY_MAX_ITEMS items
    // (in order, on `s`).  Stream-ordered, never synchronises the host;
    // `peer == rank()` is allowed; any alignment and length.  Every item is
    // checked before anything is launched: a peer out of range, a null
    // `local`, or a range outside the peer's user heap gives FB_E_INVALID; a
    // sub-communicator gives FB_E_UNSUPPORTED.  Zero-byte items are skipped
    // (only their peer is checked).
    // Destinations that overlap within one list (or a destination that
    // overlaps a source) leave unspecified bytes there.
    int putGetMany(const RmaCopy* items, size_t n, cudaStream_t s);
    // ---- batched one-sided atomics (request-based MPI_Raccumulate /
    // MPI_Rget_accumulate) ----
    struct RmaAccumulate
    {
        const void* origin; // count elements (may be null for FB_OP_NO_OP)
        void* fetch;        // previous values, or null (no fetch)
        uint64_t offset;    // user part of peer's symmetric heap
        size_t count;
        int peer;
    };
    // Every item as accumulate() of (dtype, op) would apply it, in list order
    // where the targets of two items intersect (same peer, intersecting
    // bytes), and atomically element by element with respect to every other
    // accumulate on any rank.  Stream-ordered, never synchronises the host.
    // Every item is checked before anything is launched, by the rules and
    // codes of accumulate(); zero-count items are skipped (only their peer is
    // checked); a sub-communicator gives FB_E_UNSUPPORTED.
    //
    // Launches, in list order (each counted in stats().launches): a launch
    // takes the next item unless that item would
    //  * be its FB_RMA_ACC_MAX_ITEMS + 1-th descriptor (an item longer than
    //    FB_RMA_ACC_MAX_COUNT elements is that many descriptors),
    //  * intersect items of two different chains of the launch (a chain: the
    //    items of the launch connected by intersecting targets), or
    //  * bring the target bytes of its chain above FB_RMA_ACC_CHAIN_BYTES, or
    //  * bring the launch's chunk space (one chunk per chain, plus
    //    fbRmaAccChunks(count) per item) to 2^32 chunks, which takes more
    //    than 2^39 elements in one launch, far beyond any heap,
    // in which case it starts the next launch.  So K fetching increments of
    // one counter are one launch for K <= 1024, and their fetched values are
    // the counter's successive values in list order.
    int accumulateMany(const RmaAccumulate* items, size_t n, int dtype, int op, cudaStream_t s);

    // Device watchdog error word (FB_ERR_*); synchronises `s`
    uint32_t checkError(cudaStream_t s);
    // Same word without synchronising (caller has already waited for `s`)
    uint32_t peekError() const;
    // Host-side barrier between the ranks' host threads / processes
    // (FB_E_UNSUPPORTED on a sub-communicator)
    int hostBarrier();
    // Last algorithm picked by allReduce (for reporting / tests)
    int lastAlgo() const { return lastAlgo_; }

    // Measured selection table for allReduce: message sizes up to maxBytes[i]
    // use algos[i] (entries sorted ascending; the last entry covers the rest).
    // Written by the autotuner; empty => built-in thresholds.
    void setAllReduceTable(const std::vector<uint64_t>& maxBytes,
                           const std::vector<int>& algos);
    // Thresholds + table from a parsed tuning file
    void applyTuning(const CommTuning& tuning);
    // Reads FAABRIC_TUNING_FILE if set (malformed files are reported and ignored)
    void applyTuningFromEnv();
    int pickAllReduceAlgo(uint64_t bytes, bool nvlsOk) const;

    static const char* errorString(int code);

    // Loopback backend: is `p` inside the heap of some loopback communicator?
    // (the MPI layer treats that memory as "device" memory)
    static bool isLoopbackHeapPointer(const void* p);

  private:
    Communicator() = default;

    FbCommDev dev_{};
    CommConfig cfg_;
    CommStats stats_;
    int device_ = 0;
    std::string backing_;
    int lastAlgo_ = 0;
    std::vector<std::pair<uint64_t, int>> allReduceTable_;

    // heap layout (offsets from heap base)
    uint64_t llOff_ = 0;
    uint64_t mboxOff_ = 0; // p2p bounce rings: one byte ring per destination
    uint64_t p2pDescOff_ = 0; // descriptor rings written by the senders
    uint64_t bounceSlotBytes_ = 0; // largest single eager message (ring / 2)
    // host model of every destination's byte ring: messages issued whose
    // release (ack) has not been waited for yet, oldest first
    struct BounceMsg
    {
        uint32_t seq;
        uint64_t off;
        uint64_t len;
    };
    std::deque<BounceMsg> bounceInflight_[FB_MAX_RANKS];
    uint64_t bounceHead_[FB_MAX_RANKS] = { 0 };
    uint32_t sendSeq_[FB_MAX_RANKS] = { 0 };
    uint32_t recvSeq_[FB_MAX_RANKS] = { 0 };
    uint32_t sbarEpoch_[FB_MAX_CHANNELS] = { 0 };
    uint32_t userSigConsumed_[FB_SIG_USER_WORDS] = { 0 };
    bool loop_ = false;
    // CUDA launchers, or their host twins on the loopback backend
    const fb::KernelTable* k_ = nullptr;
    void bindDevice() const;
    bool streamSync_ = false;
    bool streamWaitOk_ = false;
    bool streamWriteOk_ = false;
    cudaStream_t internalStream_ = nullptr;
    uint32_t doneSeq_ = 0;
    // transient group tables (groupMany) and copy and accumulate tables
    // (putGetMany, accumulateMany)
    struct ManySlot;
    std::vector<std::shared_ptr<ManySlot>> manySlots_;
    size_t manyNext_ = 0;
    // The next table slot, free for the host to write (waits for the launch
    // that used it last); null on a CUDA error
    ManySlot* nextManySlot();
    // The table of one batched launch where the kernel reads it: a slot's
    // device copy (*slot set; pass it to releaseManySlot after the launch),
    // or `table` itself on the loopback backend.  Null on a CUDA error.
    const void* stageManyTable(const void* table, size_t bytes, cudaStream_t s, ManySlot** slot);
    void releaseManySlot(ManySlot* slot, cudaStream_t s);
    uint64_t stageSendOff_ = 0;
    uint64_t stageRecvOff_ = 0;
    uint64_t userOff_ = 0;
    uint64_t heapTotal_ = 0;
    bool heapRegistered_ = false;

    // allocator state
    std::mutex allocMx_;
    std::map<uint64_t, uint64_t> freeList_; // offset -> size
    std::map<uint64_t, uint64_t> allocated_;

    struct Backing;
    std::shared_ptr<Backing> backingState_;
    std::shared_ptr<Bootstrap> bootstrap_;
    // local mode: shared host barrier
    struct LocalGroup;
    std::shared_ptr<LocalGroup> localGroup_;

    struct GroupLaunch;
    struct NeighborTopo;
    std::shared_ptr<const NeighborTopo> topo_;

    // sub-communicators: the child holds its parent and the slot it uses;
    // the parent records which slots are in use on this rank
    std::shared_ptr<Communicator> parent_;
    int slot_ = -1;
    std::atomic<uint32_t> usedSlots_{ 0 };

    static std::shared_ptr<Communicator> makeRank(const CommConfig& cfg, int rank, int nranks, int device);
    void computeLayout();
    void initAllocator();
    int blocksFor(uint64_t vecs, int perThread) const;
    FbCommDev devFor(int flags) const;
    void attach(const std::vector<uint8_t*>& bases,
                uint8_t* mcBase,
                uint32_t* err,
                std::shared_ptr<Backing> backing,
                const std::string& kind);
    void finishSetup();
    template<typename Run>
    int runPhases(const GroupLaunch& l,
                  std::initializer_list<int> steps,
                  bool ss,
                  int flags,
                  cudaStream_t s,
                  Run&& run);
    int launchGroup(const GroupLaunch& l, GroupKind kind, int dtype, int op, int root, int flags, cudaStream_t s);
    bool groupMissing(GroupKind kind, int root, uint32_t missing) const;
    int groupCheck(GroupKind kind, int dtype, int op, int root, int flags, bool& grouped) const;
    template<typename Next>
    int groupWalk(GroupPlan* plan,
                  GroupKind kind,
                  int dtype,
                  int op,
                  int root,
                  int flags,
                  cudaStream_t s,
                  Next&& next);
    int neighborVCheck(GroupKind kind,
                       const NeighborVItem* items,
                       size_t nItems,
                       int dtype,
                       int flags,
                       size_t& window,
                       std::vector<uint64_t>& streams) const;
    int neighborVBatch(GroupKind kind,
                       const NeighborVItem* items,
                       size_t nItems,
                       size_t esize,
                       size_t window,
                       const std::vector<uint64_t>& agreed,
                       size_t& w,
                       std::vector<fb::GroupSeg>& segs,
                       GroupLaunch& l) const;
    int addPlanLaunch(GroupPlan& plan, const std::vector<fb::GroupSeg>& segs, GroupLaunch& l);
    int groupBatch(GroupKind kind,
                   const GroupItem* items,
                   size_t nItems,
                   size_t esize,
                   GroupCursor& at,
                   std::vector<fb::GroupSeg>& segs,
                   GroupLaunch& l) const;
    int groupPerItem(GroupKind kind,
                     const GroupItem* items,
                     size_t nItems,
                     int dtype,
                     int op,
                     int root,
                     int flags,
                     cudaStream_t s);
    int streamWaitGe(cudaStream_t s, const uint32_t* localWord, uint32_t value);
    int streamBarrier(int flags, cudaStream_t s);
    bool rmaTargetOk(uint64_t dstOffset, uint64_t bytes, size_t align, int peer) const;
    int sendChunk(const uint8_t* buf, size_t len, int peer, cudaStream_t s);
    int recvChunk(uint8_t* buf, size_t len, int peer, cudaStream_t s);
    void abortPendingWaits();

    int reduceLike(int kind,
                   const void* send,
                   void* recv,
                   size_t count,
                   int dtype,
                   int op,
                   int root,
                   int algo,
                   int flags,
                   cudaStream_t s);
    int moveLike(int mode,
                 const void* send,
                 void* recv,
                 size_t chunkBytes,
                 int root,
                 int flags,
                 cudaStream_t s);
};

// Largest in-degree of a neighbour topology.  The in-edges share the
// FB_GROUP_MAX_SEGS-entry segment table of every launch with the pieces, four
// edges per entry: up to an in-degree of 32 a launch holds 1016 pieces, at
// this limit 24, so a list of many items on a high-degree graph takes several
// launches.  (The MPI layer runs graphs above the limit on its host path.)
#define FB_NEIGHBOR_MAX_IN_DEGREE 4000
// Largest out-degree plus in-degree of the neighbour v kinds: a launch's table
// holds every stream of a rank, one entry per item and one more, so at this
// limit a launch window holds 6 items.  (The MPI layer runs graphs above it
// on its host path.)
#define FB_NEIGHBOR_V_MAX_DEGREE 256

// Error codes
#define FB_OK 0
#define FB_E_UNSUPPORTED -1 // (dtype, op) pair not supported
#define FB_E_INVALID -2     // bad argument
#define FB_E_CUDA -3        // CUDA runtime error
#define FB_E_TOO_LARGE -4   // message does not fit the staging area
#define FB_E_NO_DEVICE -5

} // namespace faabric::device
