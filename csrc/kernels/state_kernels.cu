// Device-resident StateKeyValue: the dirty-chunk scan of the reference
// (StateKeyValue::getDirtyChunks walks a per-BYTE mask on the CPU and ships one
// RPC per 64 KiB chunk: src/state/StateKeyValue.cpp:441-543,592-629) becomes
// ONE kernel that scans a device-resident mask (one byte per 128-byte block),
// copies every dirty block of the replica straight into the main copy - HBM of
// the owning GPU, written over NVLink when that is a peer - and clears the mask.
// No chunk list, no host round trip, no staging.
#include "fb_prims.cuh"
#include "launch_api.h"

namespace fb {

// Each warp takes groups of 32 consecutive mask bytes (= 4 KiB of value).
// Dirty blocks of a group are copied four at a time: 8 lanes x 16 bytes each.
__global__ void __launch_bounds__(256) statePushDirtyKernel(uint8_t* mask,
                                                           const uint8_t* src,
                                                           uint8_t* dst,
                                                           uint64_t size,
                                                           uint64_t nBlocks,
                                                           uint64_t* stats)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t nWarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    const uint64_t nGroups = (nBlocks + 31) / 32;
    uint32_t pushed = 0;
    for (uint64_t g = warp; g < nGroups; g += nWarps) {
        const uint64_t myBlock = g * 32 + lane;
        uint8_t m = 0;
        if (myBlock < nBlocks) {
            m = mask[myBlock];
        }
        uint32_t bal = __ballot_sync(0xffffffffu, m != 0);
        if (bal == 0) {
            continue;
        }
        pushed += __popc(bal);
        if (bal == 0xffffffffu && (g + 1) * 32 * FB_STATE_BLOCK_BYTES <= size) {
            // a fully dirty group is one contiguous 4 KiB run: coalesced copy
            // with eight vectors in flight per lane
            const uint64_t base = g * 32 * FB_STATE_BLOCK_BYTES;
            Vec16 v[8];
#pragma unroll
            for (int k = 0; k < 8; k++) {
                v[k] = ldVecStream(src + base + (uint64_t)(k * 32 + lane) * 16);
            }
#pragma unroll
            for (int k = 0; k < 8; k++) {
                stVec(dst + base + (uint64_t)(k * 32 + lane) * 16, v[k]);
            }
            mask[myBlock] = 0;
            continue;
        }
        const uint32_t sub = lane >> 3; // which of the 4 blocks in flight
        const uint32_t part = lane & 7; // 16-byte piece of the 128-byte block
        uint32_t rest = bal;
        while (rest != 0) {
            // sub-group k copies the k-th remaining dirty block
            const uint32_t pos = __fns(rest, 0, sub + 1);
            if (pos != 0xffffffffu) {
                const uint64_t off = (g * 32 + pos) * FB_STATE_BLOCK_BYTES + part * 16;
                if (off + 16 <= size) {
                    stVec(dst + off, ldVecStream(src + off));
                } else {
                    for (uint64_t b = off; b < size; b++) {
                        dst[b] = src[b];
                    }
                }
            }
            // drop the (up to) four lowest set bits
#pragma unroll
            for (int k = 0; k < 4; k++) {
                rest &= rest - 1;
            }
        }
        if (m != 0) {
            mask[myBlock] = 0;
        }
    }
    // one atomic per warp (the ballot made the count warp-uniform)
    if (lane == 0 && pushed != 0 && stats != nullptr) {
        atomicAdd((unsigned long long*)stats, (unsigned long long)pushed);
    }
}

// Sets mask bytes for [offset, offset+len) (block granularity) from device code
// paths that cannot use cudaMemset (capturable, stream-ordered either way)
__global__ void stateFlagRangeKernel(uint8_t* mask, uint64_t firstBlock, uint64_t nBlocks)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nBlocks) {
        mask[firstBlock + i] = 1;
    }
}

cudaError_t launchStatePushDirty(uint8_t* mask,
                                 const uint8_t* src,
                                 uint8_t* dst,
                                 uint64_t size,
                                 uint64_t* stats,
                                 int blocks,
                                 cudaStream_t s)
{
    const uint64_t nBlocks = (size + FB_STATE_BLOCK_BYTES - 1) / FB_STATE_BLOCK_BYTES;
    if (blocks <= 0) {
        const uint64_t groups = (nBlocks + 31) / 32;
        blocks = (int)((groups + 7) / 8); // 8 warps per CTA, one group per warp...
        if (blocks > FB_NUM_SMS * 4) {
            blocks = FB_NUM_SMS * 4; // ...then grid-stride
        }
        if (blocks < 1) {
            blocks = 1;
        }
    }
    statePushDirtyKernel<<<blocks, 256, 0, s>>>(mask, src, dst, size, nBlocks, stats);
    return cudaGetLastError();
}

cudaError_t launchStateFlagRange(uint8_t* mask, uint64_t firstBlock, uint64_t nBlocks, cudaStream_t s)
{
    if (nBlocks == 0) {
        return cudaSuccess;
    }
    const int threads = 256;
    const uint64_t blocks = (nBlocks + threads - 1) / threads;
    stateFlagRangeKernel<<<(unsigned)blocks, threads, 0, s>>>(mask, firstBlock, nBlocks);
    return cudaGetLastError();
}

cudaError_t preloadStateKernels()
{
    cudaFuncAttributes a;
    cudaError_t e = cudaFuncGetAttributes(&a, statePushDirtyKernel);
    if (e == cudaSuccess) {
        e = cudaFuncGetAttributes(&a, stateFlagRangeKernel);
    }
    return e;
}

} // namespace fb
