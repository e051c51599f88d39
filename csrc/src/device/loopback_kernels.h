// Launch table of the communicator, and the host twins of the collective / p2p
// kernels (loopback device backend)
#pragma once

#include "launch_api.h"

#include <vector>

namespace fb {

// Every launch the communicator makes, chosen once per communicator: the CUDA
// launchers, or their host twins (which run to completion and ignore the
// stream).  Reductions are resolved by (dtype, op).
struct KernelTable
{
    cudaError_t (*reduce)(const ReduceArgs& a, int dtype, int op, int blocks, int threads, cudaStream_t s);
    cudaError_t (*ll)(const LLArgs& a, int dtype, int op, cudaStream_t s);
    cudaError_t (*group)(const GroupArgs& a, int dtype, int op, int blocks, int threads, cudaStream_t s);
    cudaError_t (*groupReduceScatter)(const GroupArgs& a, int dtype, int op, int blocks, int threads, cudaStream_t s);
    cudaError_t (*groupAllGather)(const GroupArgs& a, int blocks, int threads, cudaStream_t s);
    cudaError_t (*move)(const MoveArgs& a, int width, int blocks, int threads, cudaStream_t s);
    // TMA bulk-copy engine (fixed block size, 16-byte aligned ranges)
    cudaError_t (*moveBulk)(const MoveArgs& a, int blocks, cudaStream_t s);
    cudaError_t (*barrier)(const FbCommDev& c, cudaStream_t s);
    cudaError_t (*p2pSend)(const P2PArgs& a, int width, int blocks, cudaStream_t s);
    cudaError_t (*p2pPull)(const P2PArgs& a, int width, int blocks, cudaStream_t s);
    cudaError_t (*putSignal)(const PutArgs& a, int width, int blocks, cudaStream_t s);
    cudaError_t (*waitSignal)(const FbCommDev& c, int signalIdx, uint32_t count, cudaStream_t s);
    cudaError_t (*waitWord)(const FbCommDev& c, const uint32_t* word, uint32_t target, cudaStream_t s);
    cudaError_t (*signalPeers)(const FbCommDev& c, uint32_t wordOff, uint32_t value, cudaStream_t s);
    cudaError_t (*rmaAccumulate)(const RmaArgs& a, int dtype, int op, cudaStream_t s);
    cudaError_t (*rmaCompareSwap)(const RmaCasArgs& a, int dtype, cudaStream_t s);
    cudaError_t (*rmaCopyMany)(const RmaCopyArgs& a, cudaStream_t s);
    // device-to-device copies: one range, and `height` rows of `width` bytes
    cudaError_t (*copy)(void* dst, const void* src, size_t bytes, cudaStream_t s);
    cudaError_t (*copy2D)(void* dst,
                          size_t dpitch,
                          const void* src,
                          size_t spitch,
                          size_t width,
                          size_t height,
                          cudaStream_t s);
};

}

namespace fb::host {

// true if (dtype, op) has an element-wise reduction
bool reducible(int dtype, int op);

cudaError_t reduceKernel(const ReduceArgs& a, int dtype, int op, int blocks, int threads, cudaStream_t s);
cudaError_t llAllReduce(const LLArgs& a, int dtype, int op, cudaStream_t s);
cudaError_t groupAllReduce(const GroupArgs& a, int dtype, int op, int blocks, int threads, cudaStream_t s); // a.segs: HOST memory
cudaError_t groupReduceScatter(const GroupArgs& a, int dtype, int op, int blocks, int threads, cudaStream_t s);
cudaError_t groupAllGather(const GroupArgs& a, int blocks, int threads, cudaStream_t s);
// The move, p2p and put twins return cudaErrorMisalignedAddress, before they
// copy or synchronise, when an address the kernel reads or writes in words of
// `width` bytes is not aligned to it (moveBulk: 16 bytes)
cudaError_t moveKernel(const MoveArgs& a, int width, int blocks, int threads, cudaStream_t s);
cudaError_t moveBulk(const MoveArgs& a, int blocks, cudaStream_t s);
cudaError_t barrierKernel(const FbCommDev& c, cudaStream_t s);
cudaError_t p2pSend(const P2PArgs& a, int width, int blocks, cudaStream_t s);
cudaError_t p2pPull(const P2PArgs& a, int width, int blocks, cudaStream_t s);
cudaError_t putSignal(const PutArgs& a, int width, int blocks, cudaStream_t s);
cudaError_t waitSignal(const FbCommDev& c, int signalIdx, uint32_t addTarget, cudaStream_t s);
cudaError_t waitWord(const FbCommDev& c, const uint32_t* word, uint32_t target, cudaStream_t s);
cudaError_t signalPeers(const FbCommDev& c, uint32_t wordOff, uint32_t value, cudaStream_t s);
// atomic with respect to the other rank threads: a CAS on the enclosing 32- or
// 64-bit word, a striped lock for 16-byte elements
cudaError_t rmaAccumulate(const RmaArgs& a, int dtype, int op, cudaStream_t s);
cudaError_t rmaCompareSwap(const RmaCasArgs& a, int dtype, cudaStream_t s);
// a.items: HOST memory; one copy per item, in list order
cudaError_t rmaCopyMany(const RmaCopyArgs& a, cudaStream_t s);
cudaError_t copy(void* dst, const void* src, size_t bytes, cudaStream_t s);
cudaError_t copy2D(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t height, cudaStream_t s);

}
