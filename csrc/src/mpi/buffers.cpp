#include "buffers.h"

#include <faabric/device/communicator.h>
#include <faabric/device/cuda_driver.h>
#include <faabric/mpi/MpiWorld.h>

#include <cuda_runtime.h>

#include <cstring>
#include <stdexcept>
#include <string>

namespace faabric::mpi {

int bufferDevice(const void* p)
{
    if (p == nullptr || faabric::device::Communicator::isLoopbackHeapPointer(p) || !faabric::device::cudaAvailable()) {
        return HOST_MEMORY;
    }
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) {
        cudaGetLastError();
        return HOST_MEMORY;
    }
    if (attr.type == cudaMemoryTypeDevice) {
        return attr.device;
    }
    return attr.type == cudaMemoryTypeManaged ? ANY_DEVICE : HOST_MEMORY;
}

bool hostAddressable(const void* p)
{
    return !MpiWorld::isDevicePointer(p) || faabric::device::Communicator::isLoopbackHeapPointer(p);
}

void copyBytes(void* dst, const void* src, size_t n)
{
    if (n == 0 || dst == src) {
        return;
    }
    if (hostAddressable(dst) && hostAddressable(src)) {
        memcpy(dst, src, n);
        return;
    }
    cudaError_t e = cudaMemcpy(dst, src, n, cudaMemcpyDefault);
    if (e != cudaSuccess) {
        cudaGetLastError();
        throw std::runtime_error(std::string("Device copy in the MPI layer failed: ") + cudaGetErrorString(e));
    }
}

uint8_t* HostStage::in(const uint8_t* p, size_t bytes)
{
    if (bytes == 0 || !MpiWorld::isDevicePointer(p)) {
        return const_cast<uint8_t*>(p);
    }
    data.resize(bytes);
    copyBytes(data.data(), p, bytes);
    return data.data();
}

uint8_t* HostStage::out(uint8_t* p, size_t bytes, bool preload)
{
    if (bytes == 0 || !MpiWorld::isDevicePointer(p)) {
        return p;
    }
    data.resize(bytes);
    if (preload) {
        copyBytes(data.data(), p, bytes);
    }
    target = p;
    return data.data();
}

void HostStage::flush()
{
    if (target != nullptr) {
        copyBytes(target, data.data(), data.size());
    }
}

}
