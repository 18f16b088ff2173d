// cuda_host_utils.h — small host-side helpers shared by the renderer object (crt_cuda_core.cu) and the device
// set_scene driver (scene_device_build.cuh): error checking that throws like the reference does, an owning device
// buffer, a two-pass arena for groups of temporaries, and a kernel launch that the host build of the renderer
// (tests/simt_emu) compiles unchanged.
#pragma once

#include <algorithm>
#include <stdexcept>
#include <string>

#include <cuda_runtime.h>

#define CUDA_CHECK(expr)                                                                              \
    do {                                                                                              \
        cudaError_t err__ = (expr);                                                                   \
        if (err__ != cudaSuccess) {                                                                   \
            throw std::runtime_error(std::string(#expr) + " failed: " + cudaGetErrorString(err__) +    \
                                     " (" __FILE__ ":" + std::to_string(__LINE__) + ")");             \
        }                                                                                             \
    } while (0)

namespace crt_host {

template <typename T>
struct DeviceBuffer {
    T *ptr = nullptr;
    size_t count = 0;
    ~DeviceBuffer() { release(); }
    void release()
    {
        if (ptr) {
            cudaFree(ptr);
            ptr = nullptr;
            count = 0;
        }
    }
    void alloc(size_t n)
    {
        if (n == count && ptr) {
            return;
        }
        release();
        if (n) {
            CUDA_CHECK(cudaMalloc(&ptr, n * sizeof(T)));
        }
        count = n;
    }
    void upload(const T *src, size_t n, cudaStream_t s)
    {
        alloc(n);
        if (n) {
            CUDA_CHECK(cudaMemcpyAsync(ptr, src, n * sizeof(T), cudaMemcpyHostToDevice, s));
        }
    }
};

// One cudaMalloc / cudaFree for a group of temporaries (the device set_scene needs ~25 of them, and cudaMalloc /
// cudaFree cost more than most of its kernels). Used in two passes: the ArenaBuf::alloc calls run once to add up the
// sizes, commit() allocates, and the same calls run again to hand out the pointers.
struct DeviceArena {
    char *base = nullptr;
    size_t used = 0, capacity = 0;
    ~DeviceArena()
    {
        if (base) {
            cudaFree(base);
        }
    }
    void commit()
    {
        capacity = used;
        used = 0;
        CUDA_CHECK(cudaMalloc(&base, std::max<size_t>(capacity, 256)));
    }
    void *take(size_t bytes)
    {
        used = (used + 255) & ~(size_t)255;
        void *p = base ? base + used : nullptr;
        used += bytes;
        if (base && used > capacity) {
            throw std::runtime_error("DeviceArena: the second pass asked for more than the first");
        }
        return p;
    }
};
template <typename T>
struct ArenaBuf {
    DeviceArena *arena;
    T *ptr = nullptr;
    explicit ArenaBuf(DeviceArena &a) : arena(&a) {}
    void alloc(size_t n) { ptr = static_cast<T *>(arena->take(std::max<size_t>(n, 1) * sizeof(T))); }
};

// A one-dimensional launch: chevrons under nvcc, simt::launch (simt_env.h, included first) in the host build of the
// renderer, which compiles the headers that launch through this unchanged. An empty grid launches nothing.
template <typename... P, typename... A>
inline void launch(void (*kernel)(P...), unsigned grid, unsigned block, cudaStream_t stream, A... args)
{
    if (grid == 0) {
        return;
    }
#ifdef __CUDACC__
    kernel<<<grid, block, 0, stream>>>(args...);
#else
    (void)stream;
    simt::launch(grid, block, [&] { kernel(args...); });
#endif
}

}  // namespace crt_host
