// Host-visible launch interface of every sm_90a kernel in csrc/kernels.
// Plain C++ (no device code) so the host runtime can be built with g++ while
// the kernels are built with nvcc.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "faabric/device/comm_abi.h"

namespace fb {

// SMs of the target GPU (H100 SXM).  Default grids are sized from this
// constant rather than a device query so that every rank derives the same grid.
#define FB_NUM_SMS 132

// ---------------------------------------------------------------- reduce ----
struct ReduceArgs
{
    FbCommDev comm;
    uint64_t sendOff;   // symmetric-heap offset of every rank's input
    uint64_t recvOff;   // symmetric-heap offset of output (push modes)
    uint8_t* recvLocal; // local output pointer (pull modes), may be outside heap
    uint64_t bytes;     // total message bytes
    // The vector range [vecBegin, vecEnd) (16-byte units) this rank reduces
    uint64_t vecBegin;
    uint64_t vecEnd;
    // Where the local result vector index i lands: recvLocal + (i - outBase)*16
    uint64_t outBase;
    // How many peers are read: ranks [0, readRanks)
    int32_t readRanks;
    // Bit p set => store result to peer p at recvOff (push).  0 => local only
    uint32_t pushMask;
    // Who reduces the <16-byte tail (-1: nobody, -2: every rank)
    int32_t tailOwner;
    // skip cross-rank waits (profiling the data path under ncu only)
    int32_t noSync;
};

// Host-side launcher type shared by the per-type translation units
typedef cudaError_t (*ReduceLaunchFn)(const ReduceArgs& a,
                                      int nr,
                                      int blocks,
                                      int threads,
                                      cudaStream_t stream);

#define FB_LL_BLOCKS 8
#define FB_LL_THREADS 512
#define FB_LL_MAX_VECS (FB_LL_BLOCKS * FB_LL_THREADS)
#define FB_LL_MAX_BYTES (FB_LL_MAX_VECS * 16)
// bytes of LL area needed per rank: 2 parities x nranks x vecs x 32 B
#define FB_LL_AREA_BYTES(nranks) ((uint64_t)2 * (nranks) * FB_LL_MAX_VECS * 32)

struct LLArgs
{
    FbCommDev comm;
    const uint8_t* sendLocal;
    uint8_t* recvLocal;
    uint64_t bytes;
    uint64_t llOff; // symmetric offset of the LL slot area
    int32_t byteAccess; // local buffers are not 16-byte aligned
    int32_t pad;
};

typedef cudaError_t (*LLLaunchFn)(const LLArgs& a, cudaStream_t stream);

// ---- grouped all-reduce: MANY independent all-reduces in ONE launch ----
// The host cuts the concatenation of all tensors into N equal ownership ranges
// (one per rank) and hands every rank the list of (tensor ∩ its range)
// segments.  The kernel pays the two cross-rank barriers once for the whole
// group: barrier, every warp walks "chunks" of segments (gather from all peers,
// reduce in registers, push to all peers), barrier.
struct GroupSeg
{
    uint64_t sendOff;   // symmetric offset of this segment's input
    uint64_t recvOff;   // symmetric offset of this segment's output
    uint32_t nVec;      // full 16-byte vectors in the segment
    uint32_t chunk0;    // index of the segment's first chunk in the flat chunk space
    uint32_t tailBytes; // 1..15: a partial vector follows the nVec full ones
    uint32_t pad;
};

struct GroupArgs
{
    FbCommDev comm;
    const GroupSeg* segs; // device memory of THIS rank
    uint32_t nSegs;
    uint32_t totalChunks;
    int32_t noSync;
    int32_t root; // grouped broadcast, gather, scatter and reduce: the root rank
    // rooted kinds only: symmetric offset of every rank's staging buffer,
    // and which GROUP_PHASE_* steps this launch runs
    uint64_t stageOff;
    int32_t phase;
    int32_t exclusive; // grouped scan only: 1 for an exscan
    // grouped reduce and scan only: symmetric offset of the staging buffer
    // the results are stored in (the root's, or every rank's own)
    uint64_t stageRecvOff;
    // neighbour kinds only (see NeighborEdge): this rank's in-edges, which
    // follow the segments in the table, and the send blocks it stages
    uint32_t nEdges;
    uint32_t outDeg;
    // neighbour v kinds only (see NeighborVSeg): the round's first stream
    // byte and its width
    uint64_t vBase;
    uint64_t vWidth;
};

// vectors per warp-chunk for a world of n ranks (host and kernel must agree)
static inline int fbGroupUnroll(int nranks)
{
    // (one rank: a pure copy, as many loads in flight per thread as possible)
    return (nranks == 8) ? 2 : (nranks == 1 ? 8 : 4);
}
static inline uint32_t fbGroupChunkVecs(int nranks)
{
    return 32u * (uint32_t)fbGroupUnroll(nranks);
}
#define FB_GROUP_MAX_SEGS 1024

typedef cudaError_t (*GroupLaunchFn)(const GroupArgs& a,
                                     int blocks,
                                     int threads,
                                     cudaStream_t stream);

// ---- grouped reduce-scatter and all-gather: equal shards, ONE launch ----
// The same GroupArgs, with one segment per tensor and rank whose nVec covers
// a whole shard (shards are multiples of 16 bytes, so tailBytes is 0):
//   reduce-scatter: sendOff = off(send) + rank*shard, recvOff = off(recv);
//                   the kernel reduces over every peer's sendOff and stores
//                   to this rank's heap only.
//   all-gather:     sendOff = off(send), recvOff = off(recv) + rank*shard;
//                   the kernel loads locally and pushes to every peer.
// Both keep the grouped all-reduce's chunking (fbGroupChunkVecs) and its
// entry and exit barriers.
cudaError_t launchGroupAllGather(const GroupArgs& a,
                                 int blocks,
                                 int threads,
                                 cudaStream_t stream);

// ---- grouped broadcast: many MPI_Bcast calls from one root, ONE launch ----
// GroupArgs.root is the source rank.  The segments are the grouped
// all-reduce's (this rank's share of the list's flat vector space, with
// tailBytes 1..15 on a tensor's last segment) with sendOff == recvOff: the
// kernel loads each vector from the root's heap and stores it into every
// other rank's heap at the same offset.
cudaError_t launchGroupBroadcast(const GroupArgs& a,
                                 int blocks,
                                 int threads,
                                 cudaStream_t stream);

// ---- grouped all-to-all: many equal-block MPI_Alltoall calls, ONE launch ----
// One segment per tensor with B = nVec * 16 bytes per block: sendOff =
// off(send), recvOff = off(recv) + rank*B.  A chunk covers the same vectors
// of every block: block p of this rank's send (sendOff + p*B) is stored at
// recvOff of peer p.  Keeps fbGroupChunkVecs and the entry and exit barriers.
cudaError_t launchGroupAllToAll(const GroupArgs& a,
                                int blocks,
                                int threads,
                                cudaStream_t stream);

// ---- grouped gather, scatter, reduce and scan: many MPI_Gather /
// MPI_Scatter / MPI_Reduce calls with one root, or MPI_Scan / MPI_Exscan
// calls, ONE launch ----
// User buffers are any memory this rank's GPU can load and store, at any
// alignment; the peers exchange through their staging buffers (GroupArgs
// .stageOff).  The table is GroupSeg-sized RootedSeg entries, one per piece
// of an item (an item larger than a launch's staging room is cut into
// pieces).  Piece bytes [off, off + CB) with CB = fbGroupChunkVecs(n) * 16
// are chunk chunk0 + off / CB, and chunk ch's staging slice is [ch * CB,
// (ch + 1) * CB) of the staging buffer: so the slices follow from the counts
// alone, and every rank has the same chunk space.
//   gather:  LOCAL: every non-root copies its send into its own slices;
//            entry barrier; MOVE: the root copies peer p's slices to block p
//            of its recv, and its send to block `root` unless send is that
//            block (in place); exit barrier.
//   scatter: entry barrier; MOVE: the root copies block p of its send into
//            peer p's slices, and block `root` to its recv unless recv is
//            that block (in place); exit barrier; LOCAL: every non-root
//            copies its slices into its recv.
//   reduce:  LOCAL: every rank copies its send into its own slices
//            (stageOff); entry barrier; MOVE: the owner of chunk ch (one
//            rank, the same on every rank) folds every rank's slice of ch in
//            rank order and stores the result into the root's slice of ch at
//            stageRecvOff; exit barrier; UNSTAGE: the root copies its result
//            slices into its recv.  One rank: LOCAL copies send to recv.
//   scan:    as the reduce, but MOVE stores the running fold after rank p
//            into rank p's slice of ch at stageRecvOff (exscan, GroupArgs
//            .exclusive: rank p+1's, for p <= n-2, and rank n-1's send is
//            neither staged nor read); UNSTAGE on every rank (exscan: not
//            rank 0, whose recv is never written).  One rank: a scan's LOCAL
//            copies send to recv, an exscan does nothing.
// With noSync the launch runs the steps of `phase` with no barrier (the host
// runs the steps as separate launches around stream barriers).
struct RootedSeg
{
    uint64_t send;   // this rank's send address at the piece (0: not given)
    uint64_t recv;   // this rank's recv address at the piece (0: not given)
    uint32_t bytes;  // bytes of the piece per rank
    uint32_t chunk0; // the piece's first chunk (same field as GroupSeg's)
    uint64_t stride; // bytes per rank of the whole item: block p at p * stride
};
static_assert(sizeof(RootedSeg) == sizeof(GroupSeg), "rooted tables use GroupSeg slots");
#define GROUP_PHASE_LOCAL 1
#define GROUP_PHASE_MOVE 2
#define GROUP_PHASE_UNSTAGE 4
cudaError_t launchGroupGather(const GroupArgs& a, int blocks, int threads, cudaStream_t stream);
cudaError_t launchGroupScatter(const GroupArgs& a, int blocks, int threads, cudaStream_t stream);

// ---- grouped neighbourhood all-gather and all-to-all: many
// MPI_Neighbor_allgather / MPI_Neighbor_alltoall calls, ONE launch ----
// A staged pull over a fixed graph.  The table holds nSegs RootedSeg pieces
// (bytes of one block, the same on every rank; stride = the item's block
// bytes; chunk0 counts the launch's piece chunks, T = totalChunks in all,
// CB = FB_NEIGHBOR_CHUNK) and then this rank's nEdges in-edges, four
// NeighborEdge per GroupSeg slot.  Staging holds slots of T chunks: piece
// chunk g of slot k is chunk k * T + g.
//   LOCAL: all-to-all: send block k goes to slot k, k < outDeg; all-gather:
//          the send goes to slot 0 when outDeg > 0.
//   entry barrier
//   MOVE:  in-edge j = (src, idx) fills recv block j from src's slot idx
//          (all-gather: slot 0).  One rank: straight from its send, no
//          staging and no barrier.
//   exit barrier
// With noSync the launch runs the steps of `phase` with no barrier.
#define FB_NEIGHBOR_CHUNK 2048
struct NeighborEdge
{
    uint32_t src; // source rank
    uint32_t idx; // this edge's index among the source's out-edges
};
// GroupSeg slots of n in-edges (a macro: the kernel needs it too)
#define FB_NEIGHBOR_EDGE_SLOTS(n) (((uint32_t)(n) + 3u) / 4u)
cudaError_t launchGroupNeighbor(const GroupArgs& a, bool allToAll, int blocks, int threads, cudaStream_t stream);
cudaError_t preloadNeighborKernels();

// ---- grouped neighbourhood v-collectives: many MPI_Neighbor_allgatherv /
// MPI_Neighbor_alltoallv calls, with a size per edge, ONE launch per round ----
// A launch window of nSegs items.  A rank has S send streams (all-to-all: one
// per out-edge, S = outDeg; all-gather: S = min(outDeg, 1)) and nEdges recv
// streams, one per in-edge.  Stream k is the concatenation, in item order, of
// the window's blocks of its edge.  The table holds, per stream, nSegs + 1
// NeighborVSeg entries: {address of item m's block, offset of that block in
// the stream}, and last {0, length of the stream}.  The send streams come
// first, then the recv streams, then this rank's in-edges (NeighborEdge).  A round moves stream bytes [vBase, vBase + vWidth); staging slot
// k (all-gather: 0) holds those bytes of send stream k at k * vWidth.  The
// receiver of an edge knows its source's stream layout from its own recv
// counts, which MPI requires to match the sender's, so no displacement
// crosses ranks.  Chunk c (FB_NEIGHBOR_CHUNK bytes, totalChunks = vWidth /
// CB per slot) of slot k is staged and pulled by warp (k * totalChunks + c) %
// warps of the grid on every rank.
//   LOCAL: stage the round's bytes of every send stream
//   entry barrier
//   MOVE:  in-edge j = (src, idx) fills the round's bytes of recv stream j
//          from src's slot idx.  One rank: straight from send stream idx, no
//          staging and no barrier.
//   exit barrier
// With noSync the launch runs the steps of `phase` with no barrier.
struct NeighborVSeg
{
    uint64_t addr; // this rank's address of the item's block (0: empty block)
    uint64_t off;  // the block's first byte in the stream
};
static_assert(2 * sizeof(NeighborVSeg) == sizeof(GroupSeg), "two v entries per GroupSeg slot");
// GroupSeg slots of a v table of `streams` streams over n items, with nEdges
// in-edges right after the last entry
#define FB_NEIGHBOR_V_SLOTS(streams, n, nEdges)                                                                        \
    (((uint32_t)(streams) * ((uint32_t)(n) + 1u) * 16u + (uint32_t)(nEdges) * 8u + 31u) / 32u)
cudaError_t launchGroupNeighborV(const GroupArgs& a, bool allToAll, int blocks, int threads, cudaStream_t stream);
cudaError_t preloadNeighborVKernels();

struct ReduceLaunchers
{
    ReduceLaunchFn reduce;
    LLLaunchFn ll;
    GroupLaunchFn group;
    GroupLaunchFn groupRs; // grouped reduce-scatter
    GroupLaunchFn groupReduce; // grouped reduce (RootedSeg table)
    GroupLaunchFn groupScan;   // grouped scan and exscan (RootedSeg table)
    // Forces the CUDA module/function load of every variant (lazy loading may
    // otherwise synchronise the context while a peer rank's kernel is spinning
    // on this one => deadlock until the watchdog fires)
    cudaError_t (*preload)();
};

// Lookup implemented across coll_reduce_*.cu; returns nullptr if the
// (dtype, op) pair is not meaningful (e.g. bitwise on floats)
const ReduceLaunchers* findReduceLaunchers(int dtype, int op);
const ReduceLaunchers* findReduceLaunchersInt(int dtype, int op);
const ReduceLaunchers* findReduceLaunchersFloat(int dtype, int op);
const ReduceLaunchers* findReduceLaunchersPair(int dtype, int op);


// ------------------------------------------------------------------ move ----
enum MoveMode
{
    MOVE_ALLGATHER = 0,
    MOVE_ALLTOALL = 1,
    MOVE_GATHER = 2,
    MOVE_SCATTER = 3,
    MOVE_BCAST = 4,
    MOVE_BCAST_2STEP = 5
};

struct MoveArgs
{
    FbCommDev comm;
    uint64_t sendOff;   // symmetric offset of the source buffer(s)
    uint64_t recvOff;   // symmetric offset of the destination (2-step bcast)
    uint8_t* recvLocal; // local destination (pull modes)
    uint64_t chunkBytes; // bytes per (src,dst) pair; whole message for bcast
    uint64_t srcStride;  // allToAll/scatter: row pitch inside the source buffer
    uint64_t dstStride;  // allGather/allToAll/gather: row pitch in recvLocal
    int32_t mode;
    int32_t root;
    int32_t noSync;
};

struct P2PArgs
{
    FbCommDev comm;
    uint8_t* local;     // user buffer (send source / recv destination)
    uint64_t bytes;     // send: payload bytes; pull: capacity of `local`
    uint64_t srcOff;    // send: symmetric offset the receiver will pull from
    uint64_t heapBytes; // pull: bound for descriptor validation
    uint64_t descOff;   // symmetric offset of the descriptor rings
    uint32_t seq;       // per ordered pair, starts at 1
    int32_t peer;
    int32_t stage; // send: copy `local` to heap[rank]+srcOff first (0 = zero copy)
    int32_t pad;
};

struct PutArgs
{
    FbCommDev comm;
    const uint8_t* local;
    uint64_t dstOff;
    uint64_t bytes;
    int32_t peer;
    int32_t signalIdx;
};

cudaError_t launchMove(const MoveArgs& a,
                       int width,
                       int blocks,
                       int threads,
                       cudaStream_t s);
cudaError_t launchBarrier(const FbCommDev& c, cudaStream_t s);
cudaError_t launchP2PSend(const P2PArgs& a, int width, int blocks, cudaStream_t s);
cudaError_t launchP2PPull(const P2PArgs& a, int width, int blocks, cudaStream_t s);
// one-thread spin on a local word (fallback when stream memory ops are missing)
cudaError_t launchWaitWord(const FbCommDev& c,
                           const uint32_t* word,
                           uint32_t target,
                           cudaStream_t s);
// writes `value` to sig[p][wordOff + rank] of every peer p
cudaError_t launchSignalPeers(const FbCommDev& c,
                              uint32_t wordOff,
                              uint32_t value,
                              cudaStream_t s);
cudaError_t launchPutSignal(const PutArgs& a,
                            int width,
                            int blocks,
                            cudaStream_t s);
cudaError_t launchWaitSignal(const FbCommDev& c,
                             int signalIdx,
                             uint32_t count,
                             cudaStream_t s);


// ------------------------------------------------------------------- rma ----
// One-sided atomics on `target` (rma_kernels.cu): any memory the launching GPU
// can address, e.g. a peer's symmetric heap through its mapping, or a
// cudaMalloc window.  Every target element is updated atomically with respect
// to every other RMA kernel on any GPU.  Every target element must be aligned
// to its size (fbDtypeSize: 8 for the 8-byte pairs, 16 for the 16-byte pairs);
// origin and result buffers need no alignment.  No kernel waits on a peer or
// takes part in a barrier.
struct RmaArgs
{
    uint8_t* target;
    const uint8_t* origin; // count elements (unused for NO_OP)
    uint8_t* result;       // previous values, or null (no fetch)
    uint64_t count;
};

struct RmaCasArgs
{
    uint8_t* target;
    const uint8_t* compare; // one element each
    const uint8_t* swap;
    uint8_t* result;
};

// (dtype, op) pairs the accumulate kernels implement: every device reduction
// pair, REPLACE for every dtype, and NO_OP for every dtype when fetching
bool rmaSupported(int dtype, int op, bool fetch);
// compare-and-swap: the eight integer dtypes
bool rmaCasSupported(int dtype);
// target[i] = op(target[i], origin[i]); a.result[i] = previous target[i] when
// a.result is not null
cudaError_t launchRmaAccumulate(const RmaArgs& a, int dtype, int op, cudaStream_t s);
// result = target; if (target == compare) target = swap
cudaError_t launchRmaCompareSwap(const RmaCasArgs& a, int dtype, cudaStream_t s);
cudaError_t preloadRmaKernels();

// Batched copy (rmaCopyManyKernel): every descriptor copies `bytes` from src
// to dst, two addresses the launching GPU can load and store (its own memory,
// or a peer's heap through FbCommDev::heap[peer]).  Any alignment, any
// length.  The warps of the grid stride over the flat chunk space of the
// table: item i owns chunks [chunk0, chunk0 + fbRmaCopyChunks(bytes)).  No
// barrier, no flag words: the copy is complete when the stream passes the
// kernel.  The table is the size of a GroupSeg table, so both share one ring
// of staging slots.
struct RmaCopyDesc
{
    const uint8_t* src;
    uint8_t* dst;
    uint64_t bytes;
    uint64_t chunk0;
};
#define FB_RMA_COPY_MAX_ITEMS FB_GROUP_MAX_SEGS
#define FB_RMA_COPY_CHUNK 2048 // bytes per warp-chunk (a multiple of 16)
static inline uint64_t fbRmaCopyChunks(uint64_t bytes)
{
    return (bytes + FB_RMA_COPY_CHUNK - 1) / FB_RMA_COPY_CHUNK;
}

struct RmaCopyArgs
{
    const RmaCopyDesc* items; // device memory of the launching GPU
    uint64_t totalChunks;
    uint32_t nItems;
    uint32_t pad;
};

cudaError_t launchRmaCopyMany(const RmaCopyArgs& a, cudaStream_t s);

// Batched accumulate (rmaAccumulateManyKernel): a table of accumulates of one
// (dtype, op), each with the element rule of launchRmaAccumulate.  `target`
// is an address the launching GPU can reach (its own heap, or a peer's heap
// through FbCommDev::heap[peer]), aligned to the element size; `fetch` is
// null for an item without fetch (never for NO_OP).
//
// Items whose targets intersect must apply in list order, which warps of a
// grid do not give.  So the host lays the table out as `nChains` chains
// first, then the free items:
//  * a chain is a run of consecutive descriptors with the same chunk0 (chain
//    c has chunk0 == c, c < nChains); one warp applies its items one after the
//    other, in table order;
//  * a free item owns the chunks [chunk0, chunk0 + fbRmaAccChunks(count)),
//    FB_RMA_ACC_CHUNK elements each, spread over the warps of the grid.
// The launch is complete when the stream passes the kernel.  Unlike
// launchRmaAccumulate, f16 / bf16 SUM items without fetch take the per-element
// CAS rule, not 8-wide packed adds: the same results, at a lower rate for
// large half-precision items (a large one is better issued on its own).
struct RmaAccDesc
{
    const uint8_t* origin;
    uint8_t* fetch;
    uint8_t* target;
    uint32_t count;  // elements
    uint32_t chunk0; // first chunk (free item), or the chain's chunk
};
#define FB_RMA_ACC_MAX_ITEMS FB_GROUP_MAX_SEGS
#define FB_RMA_ACC_CHUNK 128 // elements per warp-chunk of a free item
// Largest element count of one descriptor; the host splits longer items
#define FB_RMA_ACC_MAX_COUNT ((uint32_t)1 << 30)
// Largest sum of the target bytes of one chain (see Communicator::accumulateMany)
#define FB_RMA_ACC_CHAIN_BYTES 16384
static inline uint64_t fbRmaAccChunks(uint64_t count)
{
    return (count + FB_RMA_ACC_CHUNK - 1) / FB_RMA_ACC_CHUNK;
}

struct RmaAccManyArgs
{
    const RmaAccDesc* items; // device memory of the launching GPU
    uint32_t nItems;
    uint32_t nChainItems; // items [0, nChainItems) belong to chains
    uint32_t nChains;
    uint32_t totalChunks; // nChains + the chunks of the free items
};

// rmaSupported(dtype, op, true) pairs; NO_OP needs a fetch on every item
cudaError_t launchRmaAccumulateMany(const RmaAccManyArgs& a, int dtype, int op, cudaStream_t s);


// ------------------------------------------------------------------ nvls ----
enum NvlsMode
{
    NVLS_ALLREDUCE = 0,    // ld_reduce(mc send) -> multimem.st(mc recv)
    NVLS_REDUCE_LOCAL = 1, // ld_reduce(mc send) -> local store (reduce, reduceScatter)
    NVLS_BCAST = 2,        // local load -> multimem.st
    NVLS_ALLGATHER = 3     // local load -> multimem.st at rank offset
};

struct NvlsArgs
{
    FbCommDev comm;
    uint64_t sendOff;
    uint64_t recvOff;
    uint8_t* recvLocal;
    uint64_t vecBegin;
    uint64_t vecEnd;
    uint64_t outBase;
    int32_t mode;
    int32_t noSync;
};

// -1 if the (dtype, op) pair has no in-switch reduction
int nvlsVariant(int dtype, int op);

// False for variants that reduce element-wise (integers, f64)
bool nvlsVectorised(int variant);

cudaError_t launchNvls(const NvlsArgs& a,
                       int variant,
                       int blocks,
                       int threads,
                       cudaStream_t s);


// -------------------------------------------------------------- snapshot ----
struct SnapDiffArgs
{
    const uint8_t* mem;  // executor memory (updated)
    const uint8_t* orig; // local base image the executor was restored from
    uint8_t* origW;      // writable alias of orig when updateBase != 0
    uint8_t* dst;        // main snapshot image (peer-mapped or local)
    uint64_t size;       // bytes compared (min(image size, memory size))
    const FbMergeRegionDev* regions; // sorted by offset, gaps already filled
    int32_t nRegions;
    const int32_t* typedIdx; // indices of regions with a typed merge op
    int32_t nTyped;            // > 0: clean pages before dirty ones are visited too
    const uint8_t* dirtyPages; // 1 byte per 4 KiB page, null => scan everything
    // optional: pages in which a diff starts (a changed Bytewise / XOR byte,
    // or the first byte of a typed scalar that produced a diff)
    uint8_t* pageFlagsOut;
    uint8_t* chunkFlags;       // optional: 128-byte chunks that produced a diff
    uint64_t* stats;           // [0]=diff bytes, [1]=pages flagged as above
    int32_t updateBase;        // also fold the changes into the local base
    // optional: one word per 4 KiB page of `dst`, set to `pageStamp` for every
    // page this launch changed (peers find out what to re-pull at the next fork)
    uint32_t* pageStampOut;
    uint32_t pageStamp;
};

cudaError_t launchSnapshotDiffPush(const SnapDiffArgs& a,
                                   int blocks,
                                   cudaStream_t s);
// dst page := src page wherever they differ; changed pages get `stamp`.
// stats[0] += pages copied
cudaError_t launchPageSync(const uint8_t* src,
                           uint8_t* dst,
                           uint32_t* pageStamps,
                           uint32_t stamp,
                           uint64_t size,
                           uint64_t* stats,
                           int blocks,
                           cudaStream_t s);
// Copies every page whose stamp is newer than `since` from src into dst1 (and
// dst2 when not null).  stats[0] += pages copied
cudaError_t launchPagePull(const uint8_t* src,
                           uint8_t* dst1,
                           uint8_t* dst2,
                           const uint32_t* pageStamps,
                           uint32_t since,
                           uint64_t size,
                           uint64_t* stats,
                           int blocks,
                           cudaStream_t s);
// Delta encoding of a device image: gathers the listed 4 KiB pages into a
// compact buffer, as new bytes (xorMode 0) or as new ^ old (xorMode 1)
cudaError_t launchPageGather(const uint8_t* oldImg,
                             const uint8_t* newMem,
                             const uint32_t* pages,
                             uint32_t nListed,
                             uint64_t size,
                             int xorMode,
                             uint8_t* out,
                             int blocks,
                             cudaStream_t s);
cudaError_t launchDirtyScan(const uint8_t* mem,
                            const uint8_t* base,
                            uint64_t size,
                            uint8_t* pageFlags,
                            uint64_t* nDirty,
                            int blocks,
                            cudaStream_t s);
cudaError_t launchFlagsOr(uint8_t* dst,
                          const uint8_t* src,
                          uint64_t n,
                          cudaStream_t s);
cudaError_t launchChunkRuns(const uint8_t* flags,
                            uint64_t nChunks,
                            uint32_t chunkBytes,
                            uint64_t totalBytes,
                            FbDiffDesc* out,
                            uint32_t maxOut,
                            uint32_t* count,
                            cudaStream_t s);
cudaError_t launchSnapshotApply(uint8_t* image,
                                uint64_t imageSize,
                                const FbDiffDesc* descs,
                                const uint64_t* dataOff,
                                const uint8_t* blob,
                                uint32_t nDescs,
                                cudaStream_t s);


// ----------------------------------------------------------------- state ----
// dirty mask granularity of device-resident state values
#define FB_STATE_BLOCK_BYTES 128
// Fused dirty scan + push + mask clear: every block of `src` whose mask byte is
// set is copied to `dst` (local or peer-mapped); stats[0] += dirty blocks
cudaError_t launchStatePushDirty(uint8_t* mask,
                                 const uint8_t* src,
                                 uint8_t* dst,
                                 uint64_t size,
                                 uint64_t* stats,
                                 int blocks,
                                 cudaStream_t s);
cudaError_t launchStateFlagRange(uint8_t* mask,
                                 uint64_t firstBlock,
                                 uint64_t nBlocks,
                                 cudaStream_t s);
cudaError_t preloadStateKernels();

// Preload every kernel of the library on the current device (see above)
cudaError_t preloadAllKernels();
cudaError_t preloadMoveKernels();
cudaError_t preloadRootedKernels();

// TMA bulk-copy variant of the pull collectives (coll_move_bulk.cu)
bool moveBulkSupported(const MoveArgs& a);
cudaError_t launchMoveBulk(const MoveArgs& a, int blocks, cudaStream_t s);
cudaError_t preloadMoveBulkKernel();
cudaError_t preloadNvlsKernels();
cudaError_t preloadSnapshotKernels();

} // namespace fb
