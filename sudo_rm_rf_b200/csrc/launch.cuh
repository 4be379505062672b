// How the library enqueues a kernel: the dynamic shared-memory opt-in, the SM count the persistent grids are sized
// by, and the one translation of a CUDA error into SDR_ERR_CUDA.  Host code only.
#pragma once
#include <map>
#include <mutex>
#include <utility>
#include "common.cuh"

namespace sdr {

// SDR_OK, or SDR_ERR_CUDA with the runtime's last error cleared: PyTorch reads that slot after its own launches, so an
// error left in it would surface as the failure of the next, unrelated torch op.
inline int cuda_status(cudaError_t e) {
    if (e == cudaSuccess) return SDR_OK;
    cudaGetLastError();
    return SDR_ERR_CUDA;
}

// One instance for the whole library (an inline function's static), shared by every host thread.
struct LaunchState {
    std::mutex mu;
    std::map<std::pair<const void*, int>, int> smem_limit;     // (kernel, device) -> dynamic shared memory allowed
    std::map<int, int> sms;                                    // device -> SM count
};
inline LaunchState& launch_state() {
    static LaunchState s;
    return s;
}

// Lets `kern` take `smem` bytes of dynamic shared memory on the current device.  The limit is raised only when smem
// exceeds the one in force, which until then is the default of 48 KB minus the kernel's static shared memory.  It is
// never lowered, so a larger launch of the same kernel that another thread opted in a moment earlier stays allowed.
inline int allow_dynamic_smem(const void* kern, size_t smem) {
    int dev = 0;
    if (const int rc = cuda_status(cudaGetDevice(&dev))) return rc;
    LaunchState& s = launch_state();
    std::lock_guard<std::mutex> lock(s.mu);
    auto it = s.smem_limit.find({kern, dev});
    if (it == s.smem_limit.end()) {
        cudaFuncAttributes fa;
        if (const int rc = cuda_status(cudaFuncGetAttributes(&fa, kern))) return rc;
        it = s.smem_limit.emplace(std::make_pair(kern, dev), fa.maxDynamicSharedSizeBytes).first;
    }
    if (smem > (size_t)it->second) {
        const int rc = cuda_status(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        if (rc != SDR_OK) return rc;
        it->second = (int)smem;
    }
    return SDR_OK;
}

// The SM count of the current device, queried once per device; 0 when the query fails.
inline int sm_count() {
    int dev = 0;
    if (cuda_status(cudaGetDevice(&dev))) return 0;
    LaunchState& s = launch_state();
    std::lock_guard<std::mutex> lock(s.mu);
    int& n = s.sms[dev];
    if (n <= 0 && cuda_status(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev))) n = 0;
    return n;
}

// kern<<<grid, block, smem, st>>>(args...), after the opt-in smem needs.  SDR_OK or SDR_ERR_CUDA.
template <typename... P, typename... A>
int launch(void (*kern)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
    if (smem > 0)
        if (const int rc = allow_dynamic_smem(reinterpret_cast<const void*>(kern), smem)) return rc;
    kern<<<grid, block, smem, st>>>(std::forward<A>(args)...);
    return cuda_status(cudaGetLastError());
}

}  // namespace sdr
