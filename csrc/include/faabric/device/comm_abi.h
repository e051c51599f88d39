// Device-communication ABI shared by host C++, CUDA kernels and the C API.
//
// Design (GPU-first, not a port): an MPI rank is bound to a GPU; every rank
// owns a *symmetric heap* (identical layout on every rank) and a *signal pad*,
// both mapped into every peer's address space over NVLink (single process:
// peer access / VMM; multi process: CUDA IPC / VMM fds).  Collectives are ONE
// kernel launch per rank that loads/stores peer memory directly and fuses the
// user reduce-op; cross-GPU synchronisation uses monotonically increasing
// flag words in the signal pads (st.release.sys / ld.acquire.sys).
//
// Reference behaviour being replaced: faabric MpiWorld collectives over
// shared-memory queues / TCP (src/mpi/MpiWorld.cpp:590-1775 in the reference).
#pragma once

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FB_MAX_RANKS 16
// Maximum CTAs per collective launch that take part in cross-rank barriers
#define FB_MAX_BLOCKS 160
// Signal pad layout (uint32 words):
//   [0, FB_MAX_BLOCKS*FB_MAX_RANKS)            barrier flags  flag[block][peer]
//   [FB_SIG_EPOCH_OFF, +FB_MAX_BLOCKS)         per-block local epoch counters
//   [FB_SIG_MBOX_OFF, ...)                     p2p words (see below)
//   [FB_SIG_USER_OFF, ...)                     user signal words
#define FB_SIG_FLAG_WORDS (FB_MAX_BLOCKS * FB_MAX_RANKS)
#define FB_SIG_EPOCH_OFF FB_SIG_FLAG_WORDS
#define FB_SIG_MBOX_OFF (FB_SIG_EPOCH_OFF + FB_MAX_BLOCKS)
// Point-to-point: per ordered pair (src -> dst)
//   ready[src]   in dst's pad : sequence number of the last message posted
//   desc[src][k] in dst's HEAP: {offLo, offHi, lenLo, lenHi} of message k % RING
//                               (FB_P2P_RING entries per source, 16 bytes each)
//   ack[dst]     in src's pad : sequence number of the last message pulled
//   done[2][peer] local       : CTA completion counters of the send / pull kernels
// The payload itself stays in the SENDER's symmetric heap (bounce ring or the
// user's own symmetric buffer); the receiver pulls it over NVLink.
#define FB_P2P_RING 64
#define FB_P2P_READY_OFF FB_SIG_MBOX_OFF
#define FB_P2P_ACK_OFF (FB_P2P_READY_OFF + FB_MAX_RANKS)
#define FB_P2P_DONE_OFF (FB_P2P_ACK_OFF + FB_MAX_RANKS)
#define FB_P2P_WORDS (4 * FB_MAX_RANKS)
// bytes of descriptor ring area in every rank's heap
#define FB_P2P_DESC_BYTES (FB_MAX_RANKS * FB_P2P_RING * 16)
#define FB_SIG_USER_OFF (FB_SIG_MBOX_OFF + 512)
// user signals (put-with-signal): value words then consumed-count words
#define FB_SIG_USER_WORDS 256
// per-CTA epoch words of the LL all-reduce (FB_LL_BLOCKS words per channel)
#define FB_SIG_LL_EPOCH_OFF (FB_SIG_USER_OFF + 2 * FB_SIG_USER_WORDS)
#define FB_MAX_CHANNELS 8
// stream-ordered barrier flags (one word per peer per channel): used when the
// cross-rank synchronisation is done with stream memory operations instead of
// in-kernel spins (several ranks time-sharing ONE GPU, profilers that
// serialise kernels)
#define FB_SIG_SBAR_OFF (FB_SIG_LL_EPOCH_OFF + 64)
#define FB_SIG_SBAR_WORDS (FB_MAX_CHANNELS * FB_MAX_RANKS)
#define FB_SIG_TOTAL_WORDS 4096
#define FB_SIG_BYTES (FB_SIG_TOTAL_WORDS * 4)
// Sub-communicator slots.  Each rank's signal region holds its own pad
// followed by FB_SUB_SLOTS more pads of FB_SIG_BYTES: slot s of rank p starts
// at sig[p] + (s + 1) * FB_SIG_TOTAL_WORDS.  A communicator over a subset of
// the ranks (Communicator::subset) uses one slot on every member as its pads,
// so its barrier epochs never mix with the parent's or another child's.
//
// Zeroing invariant: a slot pad is zeroed once when the region is created and
// then by its owner when the owner releases the slot, never when a child is
// created.  This is correct because every word a peer writes into a rank's
// pad during a collective is awaited by that rank in the same collective (the
// in-kernel flag barriers, the per-block epoch words, which only the owner
// writes, and the stream-ordered barrier: signalPeers + a wait per peer).  The
// grouped kernels (groupAllReduceKernel, groupReduceScatterKernel,
// groupAllGatherKernel, groupBroadcastKernel, groupAllToAllKernel) keep it
// too: they write a pad
// only through the entry and exit BlockBarrier syncs, each of which awaits
// the flag of every peer it signals, or run between two stream-ordered
// barriers with no in-kernel synchronisation at all.  So
// once a rank's last collective on the child has completed, no peer write to
// its pad is pending, and a free slot is all zeros.  A member that creates its
// child early may therefore signal a peer that has not created its own yet:
// zeroing at creation would wipe that signal.
#define FB_SUB_SLOTS 15

// Error word values written by device watchdogs
#define FB_ERR_NONE 0u
#define FB_ERR_BARRIER_TIMEOUT 1u
#define FB_ERR_FLAG_TIMEOUT 2u
#define FB_ERR_BAD_DESC 3u
#define FB_ERR_HOST_ABORT 4u

typedef struct FbCommDev {
    int32_t rank;
    int32_t nranks;
    // peer-mapped base pointers (index = rank); heap[rank] is local memory
    uint8_t* heap[FB_MAX_RANKS];
    uint32_t* sig[FB_MAX_RANKS];
    // NVLS multicast mappings of the same heap (null if unsupported)
    uint8_t* mcHeap;
    // device-visible error word (host-mapped or device memory), may be null
    uint32_t* err;
    // watchdog for device-side spins, nanoseconds of %globaltimer
    uint64_t timeoutNs;
    // Channel support: independent collectives may run concurrently (separate
    // streams / graph branches) when each uses its own slice of the barrier
    // flag slots.  blockBase = channel * blocksPerChannel.
    int32_t blockBase;
    // first LL epoch word of this channel (relative to FB_SIG_LL_EPOCH_OFF)
    int32_t llEpochBase;
} FbCommDev;

// ---- element types understood by the reduce kernels ----
typedef enum FbDtype {
    FB_I8 = 0,
    FB_U8 = 1,
    FB_I16 = 2,
    FB_U16 = 3,
    FB_I32 = 4,
    FB_U32 = 5,
    FB_I64 = 6,
    FB_U64 = 7,
    FB_F32 = 8,
    FB_F64 = 9,
    FB_F16 = 10,
    FB_BF16 = 11,
    // {value, int index} pairs for MAXLOC / MINLOC
    FB_F64_I32 = 12, // MPI_DOUBLE_INT (16 bytes with padding)
    FB_F32_I32 = 13,
    FB_I32_I32 = 14,
    FB_I64_I32 = 15, // MPI_LONG_INT (16 bytes with padding)
    FB_DTYPE_COUNT = 16
} FbDtype;

typedef enum FbOp {
    FB_OP_MAX = 0,
    FB_OP_MIN = 1,
    FB_OP_SUM = 2,
    FB_OP_PROD = 3,
    FB_OP_LAND = 4,
    FB_OP_LOR = 5,
    FB_OP_BAND = 6,
    FB_OP_BOR = 7,
    FB_OP_MAXLOC = 8,
    FB_OP_MINLOC = 9,
    FB_OP_LXOR = 10,
    FB_OP_BXOR = 11,
    FB_OP_COUNT = 12,
    // One-sided accumulate only (MPI_REPLACE, MPI_NO_OP), outside
    // [0, FB_OP_COUNT): no collective accepts them.  NO_OP is an atomic read
    // and needs a fetch buffer.
    FB_OP_REPLACE = 32,
    FB_OP_NO_OP = 33
} FbOp;

typedef enum FbAlgo {
    FB_ALGO_AUTO = 0,
    FB_ALGO_ONESHOT = 1, // every rank reads all peers, reduces locally
    FB_ALGO_TWOSHOT = 2, // reduce-scatter + all-gather fused in one kernel
    FB_ALGO_NVLS = 3,    // multimem.ld_reduce + multimem.st through NVSwitch
    FB_ALGO_LL = 4,      // low-latency push with flag-in-data (small msgs)
    FB_ALGO_COPY_ENGINE = 5,
    FB_ALGO_COUNT = 6
} FbAlgo;

static inline size_t fbDtypeSize(int dt)
{
    switch (dt) {
        case FB_I8:
        case FB_U8:
            return 1;
        case FB_I16:
        case FB_U16:
        case FB_F16:
        case FB_BF16:
            return 2;
        case FB_I32:
        case FB_U32:
        case FB_F32:
            return 4;
        case FB_I64:
        case FB_U64:
        case FB_F64:
        case FB_F32_I32:
        case FB_I32_I32:
            return 8;
        case FB_F64_I32:
        case FB_I64_I32:
            return 16;
        default:
            return 0;
    }
}

// ---- snapshot merge ABI (numeric values are part of the app ABI and equal
// the reference's enums: include/faabric/util/snapshot.h:37-54) ----
typedef enum FbSnapDataType {
    FB_SNAP_RAW = 0,
    FB_SNAP_BOOL = 1,
    FB_SNAP_INT = 2,
    FB_SNAP_LONG = 3,
    FB_SNAP_FLOAT = 4,
    FB_SNAP_DOUBLE = 5
} FbSnapDataType;

typedef enum FbSnapMergeOp {
    FB_MERGE_BYTEWISE = 0,
    FB_MERGE_SUM = 1,
    FB_MERGE_PRODUCT = 2,
    FB_MERGE_SUBTRACT = 3,
    FB_MERGE_MAX = 4,
    FB_MERGE_MIN = 5,
    FB_MERGE_IGNORE = 6,
    FB_MERGE_XOR = 7
} FbSnapMergeOp;

// One merge region as consumed by the fused diff kernels
typedef struct FbMergeRegionDev {
    uint64_t offset;
    uint64_t length; // 0 => to end of original
    int32_t dataType;
    int32_t op;
} FbMergeRegionDev;

// Diff descriptor emitted by the device diff kernel (chunk granularity)
typedef struct FbDiffDesc {
    uint64_t offset;
    uint64_t length;
    int32_t dataType;
    int32_t op;
} FbDiffDesc;

#ifdef __cplusplus
}
#endif
