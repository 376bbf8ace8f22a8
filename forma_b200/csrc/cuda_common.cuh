// Shared device helpers. All translation units are compiled with
//   -gencode arch=compute_90a,code=sm_90a --fmad=false -prec-div=true -prec-sqrt=true
// so that `a * b + c` is never contracted: every fused multiply-add of the
// reference (`mul_add`) is an explicit fmaf()/fma() here (SURVEY.md Appendix A).
#pragma once

#include <atomic>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <utility>

#include "device_types.h"

namespace forma {

constexpr unsigned kFullMask = 0xFFFFFFFFu;

#define FORMA_CUDA_TRY(expr)                                                            \
    do {                                                                                \
        cudaError_t _e = (expr);                                                        \
        if (_e != cudaSuccess) {                                                        \
            forma::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return FORMA_STATUS_CUDA;                                                   \
        }                                                                               \
    } while (0)

constexpr int FORMA_STATUS_OK = 0;
constexpr int FORMA_STATUS_INVALID = 1;
constexpr int FORMA_STATUS_ORDER = 2;
constexpr int FORMA_STATUS_CUDA = 3;
constexpr int FORMA_STATUS_NO_DEVICE = 4;
constexpr int FORMA_STATUS_CAPACITY = 5;

void set_error(const char* fmt, ...);

// Function attributes (dynamic shared memory opt-in, carve-out) and occupancy-derived grids
// are per device: the launchers cache them in tables indexed by the current device, so that
// one process can drive renderers on several GPUs.
constexpr int kMaxDevices = 64;
inline int current_device_index() {
    int d = 0;
    if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= kMaxDevices) d = 0;
    return d;
}
inline int device_sm_count() {
    static std::atomic<int> sms[kMaxDevices];  // zero-initialised; several host threads may ask at once
    const int d = current_device_index();
    int v = sms[d].load(std::memory_order_relaxed);
    if (!v) {
        v = 132;
        cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, d);
        if (v <= 0) v = 132;
        sms[d].store(v, std::memory_order_relaxed);
    }
    return v;
}

// Chained launches (option pdl): the kernels of a frame's chain are launched with programmatic
// stream serialization, so that a kernel's grid is launched as soon as every CTA of the kernel
// before it has exited, without waiting for that grid's completion and memory flush, and its CTAs
// start while the predecessor drains. Every kernel launched this way begins with chain_begin()
// (below), which waits until the predecessor has completed and its writes are visible. The wait
// is a no-op in a plain launch (pdl 0).
bool chained_launches();  // options().pdl != 0

template <class... KArgs, class... Args>
inline cudaError_t launch_chained(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                  Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = chained_launches() ? 1u : 0u;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// Growable device buffer (never shrinks). 80 GB of HBM3 still makes "keep the high
// water mark" the right policy for per-frame scratch.
template <class T>
struct DeviceBuffer {
    T* ptr = nullptr;
    size_t capacity = 0;
    cudaError_t reserve(size_t n, bool keep = false, cudaStream_t stream = 0) {
        if (n <= capacity) return cudaSuccess;
        size_t cap = capacity ? capacity : 1024;
        while (cap < n) cap += cap / 2 + 1024;
        T* np = nullptr;
        cudaError_t e = cudaMalloc(&np, cap * sizeof(T));
        if (e != cudaSuccess) return e;
        if (keep && ptr && capacity) {
            e = cudaMemcpyAsync(np, ptr, capacity * sizeof(T), cudaMemcpyDeviceToDevice, stream);
            if (e != cudaSuccess) return e;
            e = cudaStreamSynchronize(stream);
            if (e != cudaSuccess) return e;
        }
        if (ptr) cudaFree(ptr);
        ptr = np;
        capacity = cap;
        return cudaSuccess;
    }
    void release() {
        if (ptr) cudaFree(ptr);
        ptr = nullptr;
        capacity = 0;
    }
    ~DeviceBuffer() { release(); }
    DeviceBuffer() = default;
    DeviceBuffer(const DeviceBuffer&) = delete;
    DeviceBuffer& operator=(const DeviceBuffer&) = delete;
};

// Growable page-locked host buffer (H2D staging at full PCIe rate).
template <class T>
struct PinnedBuffer {
    T* ptr = nullptr;
    size_t capacity = 0;
    cudaError_t reserve(size_t n) {
        if (n <= capacity) return cudaSuccess;
        size_t cap = capacity ? capacity : 1024;
        while (cap < n) cap += cap / 2 + 1024;
        T* np = nullptr;
        cudaError_t e = cudaMallocHost(&np, cap * sizeof(T));
        if (e != cudaSuccess) return e;
        if (ptr) cudaFreeHost(ptr);
        ptr = np;
        capacity = cap;
        return cudaSuccess;
    }
    ~PinnedBuffer() {
        if (ptr) cudaFreeHost(ptr);
    }
    PinnedBuffer() = default;
    PinnedBuffer(const PinnedBuffer&) = delete;
    PinnedBuffer& operator=(const PinnedBuffer&) = delete;
};

#ifdef __CUDACC__
__device__ __forceinline__ unsigned lane_id() { return threadIdx.x & 31u; }

// The first statement of every kernel launched through launch_chained: this CTA waits for the grid
// before it (griddepcontrol.wait). Every such kernel reaches the wait, so that a wait on the
// predecessor implies that everything before it has completed too.
// No kernel triggers its dependents early (griddepcontrol.launch_dependents): the trigger is
// implicit when a CTA exits. Triggered at the top of every kernel, the CTAs of the next kernels
// became resident and sat in their waits beside the running grid, and the painter tables of
// paris@4K took 0.166 instead of 0.149 ms (DESIGN.md section 6).
__device__ __forceinline__ void chain_begin() { cudaGridDependencySynchronize(); }

__device__ __forceinline__ float d_rcp(float v) { return 1.0f / v; }   // IEEE division (-prec-div=true)
__device__ __forceinline__ float d_mix(float t, float a, float b) { return fmaf(t, b, fmaf(-t, a, a)); }
// Rust f32::clamp keeps NaN.
__device__ __forceinline__ float d_clamp(float v, float lo, float hi) {
    if (v < lo) v = lo;
    if (v > hi) v = hi;
    return v;
}
// Rust `as u32` from f32: saturating, NaN -> 0.
__device__ __forceinline__ uint32_t d_sat_u32(float v) {
    if (!(v > 0.0f)) return 0u;
    if (v >= 4294967296.0f) return 0xFFFFFFFFu;
    return (uint32_t)v;
}

// Warp-wide inclusive scan (shuffle based).
__device__ __forceinline__ uint32_t warp_inclusive_scan(uint32_t v) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t n = __shfl_up_sync(kFullMask, v, o);
        if (lane_id() >= (unsigned)o) v += n;
    }
    return v;
}
#endif

}  // namespace forma
