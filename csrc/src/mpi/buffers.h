// Where a buffer of the MPI layer lives, and how its bytes are copied.
//
// On the loopback device backend the symmetric heap is plain host memory:
// MpiWorld::isDevicePointer counts it as device memory when a collective picks
// its path, but it is copied with memcpy, and a machine without a GPU never
// reaches the CUDA runtime for it.  This module is the only place that knows
// that rule.
#pragma once

#include <cstddef>
#include <cstdint>
#include <vector>

namespace faabric::mpi {

// bufferDevice(): host memory (also the loopback backend's heaps, and every
// pointer when CUDA is unavailable), managed memory, or a CUDA device index
constexpr int HOST_MEMORY = -1;
constexpr int ANY_DEVICE = -2;

int bufferDevice(const void* p);

// True when memcpy may touch the buffer
bool hostAddressable(const void* p);

// memcpy between host-addressable buffers, cudaMemcpy (cudaMemcpyDefault)
// otherwise; throws std::runtime_error on a CUDA error.  Nothing to do for
// n == 0 or dst == src.
void copyBytes(void* dst, const void* src, size_t n);

// Host scratch for a buffer that MpiWorld::isDevicePointer sends down the
// device branch, so that the host algorithm it is handed to does not take
// that branch again.  Other buffers pass through untouched.
struct HostStage
{
    std::vector<uint8_t> data;
    uint8_t* target = nullptr;

    // A host copy of `p`, taken now
    uint8_t* in(const uint8_t* p, size_t bytes);

    // Host scratch for `p` (a copy of it with `preload`), written back by flush()
    uint8_t* out(uint8_t* p, size_t bytes, bool preload = false);

    void flush();
};

}
