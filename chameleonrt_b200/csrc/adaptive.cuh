// adaptive.cuh — adaptive sampling (crtc_set_adaptive): blocks of pixels whose noise estimate has converged stop tracing.
//
//   k_adaptive_select   once per wavefront, before k_raygen: one warp per block of 32 local pixels (an 8x4 screen block,
//                       local_pixel_coords). The block's error E_b (the max of its in-frame pixels' e_p, a warp reduction)
//                       and its frame count c_b give n_b, the frames the block renders in this wavefront.
//   k_adaptive_readout  crtc_read_adaptive: samples (c_b * spp) and e_p per pixel into row-major buffers.
//
// k_raygen<true> enqueues only the paths of each block's first n_b frames, k_resolve<true> folds them with c_b in place of
// frame_id and folds the luminance moments (kernels.cuh). A pixel that is not enqueued costs no traversal or shading work:
// every later kernel reads its ray count from the device counters. The definitions are in include/crt_cuda.h.
//
// Kernels are launched through crt_host::launch (cuda_host_utils.h), so the host build of the renderer (tests/simt_emu) compiles
// this header unchanged.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "aov_denoise.cuh"
#include "cuda_host_utils.h"
#include "kernels.cuh"

namespace crt {

constexpr int kAdaptiveBlock = 256;  // 8 warps = 8 blocks of pixels per thread block

struct AdaptiveSelect {
    float threshold;
    uint32_t min_frames, max_frames;  // max_frames 0 = no cap
    uint32_t frames;                  // F, the frames of this wavefront
    uint32_t stat_base;               // the count at which the statistics start (AdaptiveFrame)
    uint32_t all_active;              // 1: every block with an in-frame pixel renders F frames (the mode is off, or a trial)
    uint32_t reset;                   // 1: first adaptive wavefront since a reset: every count starts at stat_base
};

// e_p = sqrt(max(0, m2 - m1^2) / (N max(m1, 1e-4))) for N = samples > 0; +inf without samples
CRT_D float adaptive_pixel_error(float2 m, uint32_t samples)
{
    if (samples == 0u) {
        return __uint_as_float(0x7f800000u);
    }
    const float var = fmaxf(0.f, m.y - m.x * m.x);
    return sqrtf(var / ((float)samples * fmaxf(m.x, 1e-4f)));
}

// One thread per local pixel (npx_local is a multiple of 4096: every warp is one whole block). Writes sel[b] = {c_b, n_b}
// and count[b] = c_b + n_b.
__global__ void __launch_bounds__(kAdaptiveBlock) k_adaptive_select(FrameLayout f, AdaptiveSelect p, uint32_t *count, uint2 *sel,
                                                                    float2 *moments)
{
    const uint32_t lp = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t b = lp >> 5;
    uint32_t x, y;
    const bool in_frame = local_pixel_coords(f, lp, x, y);
    float2 m = make_float2(0.f, 0.f);
    if (p.reset) {
        moments[lp] = m;
    } else {
        m = moments[lp];
    }
    const uint32_t c = p.reset ? p.stat_base : count[b];
    const uint32_t frames_seen = c - p.stat_base;
    float e = in_frame ? adaptive_pixel_error(m, frames_seen * f.spp) : 0.f;
    for (int off = 16; off > 0; off >>= 1) {  // e >= 0 (or +inf): the max reaches lane 0
        e = fmaxf(e, __shfl_down_sync(0xffffffffu, e, off));
    }
    const unsigned any_in = __ballot_sync(0xffffffffu, in_frame);  // (every lane has read count[b] before lane 0 writes it)
    if ((threadIdx.x & 31u) == 0u) {
        uint32_t n = 0u;
        if (any_in != 0u) {
            n = (p.all_active || frames_seen < p.min_frames || e > p.threshold) ? p.frames : 0u;
            if (p.max_frames != 0u) {
                n = min(n, p.max_frames > c ? p.max_frames - c : 0u);
            }
        }
        sel[b] = make_uint2(c, n);
        count[b] = c + n;
    }
}

// samples_full / error_full (each optional): row-major framebuffer arrays; pixels of other ranks' tiles are not written
__global__ void __launch_bounds__(256) k_adaptive_readout(FrameLayout f, const uint32_t *count, const float2 *moments,
                                                          uint32_t stat_base, uint32_t *samples_full, float *error_full)
{
    const uint32_t lp = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t x, y;
    if (lp >= f.npx_local || !local_pixel_coords(f, lp, x, y)) {
        return;
    }
    const uint32_t c = count[lp >> 5];
    const size_t p = (size_t)y * f.fb_w + x;
    if (samples_full) {
        samples_full[p] = c * f.spp;
    }
    if (error_full) {
        error_full[p] = adaptive_pixel_error(moments[lp], (c - stat_base) * f.spp);
    }
}

// Per-block state: a count (4 B) and {c_b, n_b} (8 B) per block of 32 pixels, the moments (8 B) per local pixel;
// allocated by the first adaptive wavefront after crtc_initialize. The readout buffers (8 B per framebuffer pixel) are
// allocated by the first crtc_read_adaptive.
struct AdaptiveState {
    crt_host::DeviceBuffer<uint32_t> count;
    crt_host::DeviceBuffer<uint2> sel;
    crt_host::DeviceBuffer<float2> moments;
    crt_host::DeviceBuffer<uint32_t> samples_full;
    crt_host::DeviceBuffer<float> error_full;

    void release()
    {
        count.release();
        sel.release();
        moments.release();
        samples_full.release();
        error_full.release();
    }
    void ensure(size_t npx_local)
    {
        count.alloc(npx_local / 32);
        sel.alloc(npx_local / 32);
        moments.alloc(npx_local);
    }
    AdaptiveFrame frame(uint32_t stat_base) const { return AdaptiveFrame{sel.ptr, moments.ptr, stat_base}; }
    void select(const FrameLayout &f, const AdaptiveSelect &p, cudaStream_t stream)
    {
        crt_host::launch(k_adaptive_select, f.npx_local / kAdaptiveBlock, kAdaptiveBlock, stream, f, p, count.ptr, sel.ptr, moments.ptr);
    }
    // The adaptive instantiations of the frame's first and last kernels (the mode-off ones are launched by the renderer)
    void raygen(unsigned grid, const ViewParams &view, const FrameLayout &f, const PathState &ps, const AdaptiveFrame &ad,
                cudaStream_t stream)
    {
        crt_host::launch(k_raygen<true>, grid, 256, stream, view, f, ps, ad);
    }
    void resolve(unsigned grid, const FrameLayout &f, const PathState &ps, uint32_t frame_id, float *accum_local,
                 uint32_t *img_local, float *accum_full, uint32_t *img_full, uint32_t *done_counter, uint32_t *arrive_word,
                 uint32_t seq, const AdaptiveFrame &ad, cudaStream_t stream)
    {
        crt_host::launch(k_resolve<true>, grid, 256, stream, f, ps, frame_id, accum_local, img_local, accum_full, img_full,
                   done_counter, arrive_word, seq, ad);
    }
    // host arrays in, the local pixels' values over them, host arrays out (the other ranks' pixels stay as they were)
    void readout(const FrameLayout &f, uint32_t stat_base, uint32_t *samples_out, float *error_out, cudaStream_t stream)
    {
        const size_t n = (size_t)f.fb_w * f.fb_h;
        if (samples_out) {
            samples_full.alloc(n);
            CUDA_CHECK(cudaMemcpyAsync(samples_full.ptr, samples_out, n * sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
        }
        if (error_out) {
            error_full.alloc(n);
            CUDA_CHECK(cudaMemcpyAsync(error_full.ptr, error_out, n * sizeof(float), cudaMemcpyHostToDevice, stream));
        }
        crt_host::launch(k_adaptive_readout, (f.npx_local + 255) / 256, 256, stream, f, count.ptr, moments.ptr, stat_base,
                   samples_out ? samples_full.ptr : nullptr, error_out ? error_full.ptr : nullptr);
        if (samples_out) {
            CUDA_CHECK(cudaMemcpyAsync(samples_out, samples_full.ptr, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
        }
        if (error_out) {
            CUDA_CHECK(cudaMemcpyAsync(error_out, error_full.ptr, n * sizeof(float), cudaMemcpyDeviceToHost, stream));
        }
        CUDA_CHECK(cudaStreamSynchronize(stream));
    }
};

}  // namespace crt
