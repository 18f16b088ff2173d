// wave_devcheck.cu — TEST-ONLY shared library (libcrt_wave_devcheck.so).
//
// The per-bounce kernels of kernels.cuh (k_raygen, k_traverse, k_shade, k_nee_resolve, k_resolve and the shade-queue
// sort) one launch at a time, as nvcc compiles them for sm_90a with the product's NVFLAGS, on a path state the caller
// hands over whole: every wavekat_* entry point uploads the full PathState image (and queues, counters), launches the
// product's kernel template on the grid crtc_renderer::enqueue_frame gives it (crt_cuda_core.cu) and copies the whole
// state back, so that tests/test_wavefront_device.py can feed a stage any state and look at every byte it left.
// wavefront_hostcheck.cpp exports the same entry points over its one-lane launches; tests/simt_emu/build.py compiles
// this file for the host with every launch under the SIMT emulation (32-lane warps, real atomics).
// Not linked into libcrt_cuda_core.so.
//
// State image (`st`, host pointers, capacity `cap` paths): [0..7] ray_o, ray_d, hit, thr_rng, radiance, nee_T, nee_l1,
// nee_l2 (cap float4 each), [8] sray_o and [9] sray_d (2 cap float4), [10] vis (2 cap bytes), [11] queue[0] and [12]
// queue[1] (cap uint32), [13] counters (kNumCounters uint32). Layout (`lay`): fb_w, fb_h, ntx, npx_local, spp, frames,
// number of tile ids. View (`view`): pos, dir_du, dir_dv, dir_top_left (12 floats).
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/crt_scene.h"
#include "bvh8_device.cuh"
#include "cuda_host_utils.h"
#include "host_scene.h"
#include "kernels.cuh"

namespace {

thread_local std::string g_err;

using crt_host::DeviceBuffer;
const cudaStream_t stream = nullptr;

template <typename F>
int guarded(F &&f)
{
    try {
        f();
        return 0;
    } catch (const std::exception &e) {
        g_err = e.what();
        return 1;
    }
}

void upload_bytes(DeviceBuffer<uint8_t> &d, const void *src, size_t bytes)
{
    d.upload(static_cast<const uint8_t *>(src), bytes, stream);
}

// The scene as set_scene uploads it when the BVH is built on the host (pack_scene's records).
struct WaveScene {
    DeviceBuffer<uint8_t> nodes, tris, shade, materials, lights, texels, tex;
    uint32_t num_lights = 0;
    crt::DeviceScene device_scene() const
    {
        crt::DeviceScene sc;
        sc.nodes = reinterpret_cast<const float4 *>(nodes.ptr);
        sc.tris = reinterpret_cast<const float4 *>(tris.ptr);
        sc.shade = reinterpret_cast<const float4 *>(shade.ptr);
        sc.materials = reinterpret_cast<const float4 *>(materials.ptr);
        sc.lights = reinterpret_cast<const float4 *>(lights.ptr);
        sc.texels = reinterpret_cast<const uint32_t *>(texels.ptr);
        sc.tex = reinterpret_cast<const crt::DevTex *>(tex.ptr);
        sc.tex_objects = nullptr;
        sc.num_lights = num_lights;
        sc.float_one = 0x3F800000u;
        return sc;
    }
};

constexpr int kStateArrays = 14;

size_t state_bytes(int k, size_t cap)
{
    return k < 8 ? cap * 16 : k < 10 ? 2 * cap * 16 : k == 10 ? 2 * cap : k < 13 ? cap * 4 : crt::kNumCounters * 4;
}

// One stage's path state on the device: uploaded whole, downloaded whole.
struct DevState {
    DeviceBuffer<uint8_t> a[kStateArrays];
    DeviceBuffer<unsigned long long> trav;
    crt::PathState ps{};
    size_t cap;
    DevState(void *const *st, uint32_t cap_) : cap(cap_)
    {
        for (int k = 0; k < kStateArrays; ++k) {
            upload_bytes(a[k], st[k], state_bytes(k, cap));
        }
        const unsigned long long zero[4] = {0, 0, 0, 0};
        trav.upload(zero, 4, stream);
        auto f4 = [&](int k) { return reinterpret_cast<float4 *>(a[k].ptr); };
        ps.ray_o = f4(0);
        ps.ray_d = f4(1);
        ps.hit = f4(2);
        ps.thr_rng = f4(3);
        ps.radiance = f4(4);
        ps.nee_T = f4(5);
        ps.nee_l1 = f4(6);
        ps.nee_l2 = f4(7);
        ps.sray_o = f4(8);
        ps.sray_d = f4(9);
        ps.vis = a[10].ptr;
        ps.queue[0] = reinterpret_cast<uint32_t *>(a[11].ptr);
        ps.queue[1] = reinterpret_cast<uint32_t *>(a[12].ptr);
        ps.counters = reinterpret_cast<uint32_t *>(a[13].ptr);
        ps.trav_counters = trav.ptr;
    }
    void download(void *const *st)
    {
        CUDA_CHECK(cudaGetLastError());
        for (int k = 0; k < kStateArrays; ++k) {
            if (a[k].count) {
                CUDA_CHECK(cudaMemcpyAsync(st[k], a[k].ptr, a[k].count, cudaMemcpyDeviceToHost, stream));
            }
        }
        CUDA_CHECK(cudaStreamSynchronize(stream));
    }
};

struct Layout {
    crt::FrameLayout fl{};
    DeviceBuffer<uint32_t> tile_ids;
    Layout(const uint32_t *lay, const uint32_t *tiles)
    {
        fl.fb_w = (int)lay[0];
        fl.fb_h = (int)lay[1];
        fl.ntx = lay[2];
        fl.npx_local = lay[3];
        fl.spp = lay[4];
        fl.frames = lay[5];
        tile_ids.upload(tiles, lay[6], stream);
        fl.tile_ids = tile_ids.ptr;
    }
};

crt::ViewParams view_params(const float *v, uint32_t frame_id)
{
    crt::ViewParams view;
    view.pos = make_float3(v[0], v[1], v[2]);
    view.dir_du = make_float3(v[3], v[4], v[5]);
    view.dir_dv = make_float3(v[6], v[7], v[8]);
    view.dir_top_left = make_float3(v[9], v[10], v[11]);
    view.frame_id = frame_id;
    return view;
}

// (the check runs on the process's first visible device)
int num_sms()
{
    int sms = 0;
    CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    return sms;
}

// crtc_renderer::scan_u32
void scan_u32(uint32_t *data, uint32_t n, uint32_t *scratch)
{
    const unsigned tiles = (n + crt::kBuildTile - 1) / crt::kBuildTile;
    crt::k_scan_tile<uint32_t><<<tiles, crt::kBuildBlock, 0, stream>>>(data, data, n, tiles > 1 ? scratch : nullptr);
    if (tiles <= 1) {
        return;
    }
    scan_u32(scratch, tiles, scratch + tiles);
    crt::k_scan_add<uint32_t><<<tiles, crt::kBuildBlock, 0, stream>>>(data, n, scratch);
}

}  // namespace

extern "C" {

const char *wavekat_last_error() { return g_err.c_str(); }

// The scene's records (pack_scene) on the device; null on error.
void *wavekat_scene(const crt_scene_t *scene)
{
    auto ws = std::make_unique<WaveScene>();
    const int rc = guarded([&] {
        crt::SceneRecords rec;
        crt::pack_scene(scene, 0, rec);
        upload_bytes(ws->nodes, rec.bvh.nodes.data(), rec.bvh.nodes.size() * sizeof(rec.bvh.nodes[0]));
        upload_bytes(ws->tris, rec.tris.data(), rec.tris.size() * sizeof(float));
        upload_bytes(ws->shade, rec.shade.data(), rec.shade.size() * sizeof(rec.shade[0]));
        upload_bytes(ws->materials, rec.shading.materials.data(), rec.shading.materials.size() * sizeof(crt_material_t));
        upload_bytes(ws->lights, rec.shading.lights.data(), rec.shading.lights.size() * sizeof(crt_quad_light_t));
        upload_bytes(ws->texels, rec.shading.texels.data(), rec.shading.texels.size() * sizeof(uint32_t));
        upload_bytes(ws->tex, rec.shading.tex_desc.data(), rec.shading.tex_desc.size() * sizeof(crt::TexDesc));
        ws->num_lights = (uint32_t)rec.shading.lights.size();
        CUDA_CHECK(cudaStreamSynchronize(stream));
    });
    return rc ? nullptr : ws.release();
}

void wavekat_scene_free(void *s) { delete static_cast<WaveScene *>(s); }

// k_raygen (sel != null: k_raygen<true> with that block selection, two uint32 per block of 32 local pixels) on
// enqueue_frame's grid: one thread per path of the batch, npx_local * spp * frames <= cap.
int wavekat_raygen(const float *view, uint32_t frame_id, const uint32_t *lay, const uint32_t *tile_ids, const uint32_t *sel,
                   uint32_t cap, void *const *st)
{
    return guarded([&] {
        DevState s(st, cap);
        Layout l(lay, tile_ids);
        const crt::ViewParams v = view_params(view, frame_id);
        const size_t npaths = (size_t)l.fl.npx_local * l.fl.spp * l.fl.frames;
        const unsigned g256 = (unsigned)((npaths + 255) / 256);
        DeviceBuffer<uint32_t> d_sel;
        if (g256 && sel) {
            d_sel.upload(sel, 2 * (size_t)(l.fl.npx_local / 32), stream);
            crt::AdaptiveFrame ad{};
            ad.sel = reinterpret_cast<const uint2 *>(d_sel.ptr);
            crt::k_raygen<true><<<g256, 256, 0, stream>>>(v, l.fl, s.ps, ad);
        } else if (g256) {
            crt::k_raygen<false><<<g256, 256, 0, stream>>>(v, l.fl, s.ps, crt::AdaptiveFrame{});
        }
        s.download(st);
    });
}

// One k_traverse launch as crtc_renderer::launch_traverse makes it (default options): the shadow rays counted in
// counters[any_counter] (-1: none), then the closest-hit rays through queue[queue_index] counted in
// counters[closest_counter] (-1: none), work cursor counters[work_counter].
int wavekat_traverse(void *scene, int queue_index, int closest_counter, int any_counter, int work_counter, int far_first,
                     uint32_t cap, void *const *st)
{
    return guarded([&] {
        const crt::DeviceScene sc = static_cast<WaveScene *>(scene)->device_scene();
        DevState s(st, cap);
        int per_sm = 0;
        CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, crt::k_traverse<false>, crt::kTravBlock, 0));
        const unsigned trav_grid = (unsigned)(num_sms() * std::max(1, per_sm));
        const int sched = crt::kRefillIdle | (far_first ? 0x100 : 0);
        crt::k_traverse<false><<<trav_grid, crt::kTravBlock, 0, stream>>>(
            sc, s.ps, s.ps.queue[queue_index & 1], closest_counter >= 0 ? s.ps.counters + closest_counter : nullptr,
            any_counter >= 0 ? s.ps.counters + any_counter : nullptr, s.ps.counters + work_counter, sched);
        s.download(st);
    });
}

// k_shade<false> of bounce `bounce` over queue[bounce & 1] into queue[(bounce + 1) & 1], on enqueue_frame's grid over
// the path capacity (lanes past the queue length take part in the ballots).
int wavekat_shade(void *scene, int bounce, int max_depth, uint32_t cap, void *const *st)
{
    return guarded([&] {
        const crt::DeviceScene sc = static_cast<WaveScene *>(scene)->device_scene();
        DevState s(st, cap);
        const unsigned g128 = (unsigned)((cap + 127) / 128);
        if (g128) {
            crt::k_shade<false><<<g128, 128, 0, stream>>>(sc, s.ps, s.ps.queue[bounce & 1], s.ps.queue[(bounce + 1) & 1], bounce,
                                                          max_depth);
        }
        s.download(st);
    });
}

// k_nee_resolve of bounce `bounce` over queue[bounce & 1], on enqueue_frame's capped grid-stride grid. Returns the
// grid in *grid.
int wavekat_nee_resolve(int bounce, uint32_t cap, void *const *st, uint32_t *grid)
{
    return guarded([&] {
        DevState s(st, cap);
        const unsigned g_nee = (unsigned)std::min<size_t>((cap + 255) / 256, (size_t)num_sms() * 8 * 2);
        *grid = g_nee;
        if (g_nee) {
            crt::k_nee_resolve<<<g_nee, 256, 0, stream>>>(s.ps, s.ps.queue[bounce & 1], bounce);
        }
        s.download(st);
    });
}

// k_resolve (sel != null: k_resolve<true> with that block selection, moments and stat_base) over the radiance of the
// state; accum_local (3 npx_local floats), img_local, moments (2 npx_local floats) in and out; accum_full / img_full
// (fb_w * fb_h pixels) in and out unless null.
int wavekat_resolve(const uint32_t *lay, const uint32_t *tile_ids, uint32_t frame_id, const uint32_t *sel, float *moments,
                    uint32_t stat_base, float *accum_local, uint32_t *img_local, float *accum_full, uint32_t *img_full,
                    uint32_t cap, void *const *st)
{
    return guarded([&] {
        DevState s(st, cap);
        Layout l(lay, tile_ids);
        const size_t npx = l.fl.npx_local, nfull = (size_t)l.fl.fb_w * l.fl.fb_h;
        DeviceBuffer<float> d_accum, d_accum_full, d_moments;
        DeviceBuffer<uint32_t> d_img, d_img_full, d_sel;
        d_accum.upload(accum_local, 3 * npx, stream);
        d_img.upload(img_local, npx, stream);
        if (accum_full) {
            d_accum_full.upload(accum_full, 3 * nfull, stream);
            d_img_full.upload(img_full, nfull, stream);
        }
        const unsigned gpx = (unsigned)((npx + 255) / 256);
        if (gpx && sel) {
            d_sel.upload(sel, 2 * (npx / 32), stream);
            d_moments.upload(moments, 2 * npx, stream);
            crt::AdaptiveFrame ad{};
            ad.sel = reinterpret_cast<const uint2 *>(d_sel.ptr);
            ad.moments = reinterpret_cast<float2 *>(d_moments.ptr);
            ad.stat_base = stat_base;
            crt::k_resolve<true><<<gpx, 256, 0, stream>>>(l.fl, s.ps, frame_id, d_accum.ptr, d_img.ptr, d_accum_full.ptr,
                                                           d_img_full.ptr, nullptr, nullptr, 0u, ad);
        } else if (gpx) {
            crt::k_resolve<false><<<gpx, 256, 0, stream>>>(l.fl, s.ps, frame_id, d_accum.ptr, d_img.ptr, d_accum_full.ptr,
                                                            d_img_full.ptr, nullptr, nullptr, 0u, crt::AdaptiveFrame{});
        }
        s.download(st);
        auto back = [&](void *dst, const auto &b) {
            if (b.count) {
                CUDA_CHECK(cudaMemcpyAsync(dst, b.ptr, b.count * sizeof(*b.ptr), cudaMemcpyDeviceToHost, stream));
            }
        };
        back(accum_local, d_accum);
        back(img_local, d_img);
        if (accum_full) {
            back(accum_full, d_accum_full);
            back(img_full, d_img_full);
        }
        if (sel) {
            back(moments, d_moments);
        }
        CUDA_CHECK(cudaStreamSynchronize(stream));
    });
}

// Option shade_sort: queue[bounce & 1] of bounce `bounce` bucketed by material into `sorted` (cap entries), with
// crtc_renderer::sort_shade_queue's launches (k_queue_hist, the scan, k_queue_scatter over the capacity's tiles).
int wavekat_queue_sort(void *scene, int bounce, uint32_t cap, void *const *st, uint32_t *sorted)
{
    return guarded([&] {
        const crt::DeviceScene sc = static_cast<WaveScene *>(scene)->device_scene();
        DevState s(st, cap);
        const uint32_t num_tiles = (uint32_t)((cap + crt::kSortTile - 1) / crt::kSortTile);
        const uint32_t hist_items = 256u * num_tiles;
        size_t scratch_items = 1, left = hist_items;
        while (left > (size_t)crt::kBuildTile) {
            left = (left + crt::kBuildTile - 1) / crt::kBuildTile;
            scratch_items += left;
        }
        DeviceBuffer<uint32_t> d_sorted, hist, scratch;
        d_sorted.upload(sorted, cap, stream);
        hist.alloc(hist_items);
        scratch.alloc(scratch_items);
        if (num_tiles) {
            const uint32_t *qin = s.ps.queue[bounce & 1];
            crt::k_queue_hist<256><<<num_tiles, crt::kSortBlock, 0, stream>>>(sc, s.ps, qin, bounce, hist.ptr, num_tiles);
            scan_u32(hist.ptr, hist_items, scratch.ptr);
            crt::k_queue_scatter<256><<<num_tiles, crt::kSortBlock, 0, stream>>>(sc, s.ps, qin, d_sorted.ptr, bounce, hist.ptr,
                                                                                  num_tiles);
        }
        s.download(st);
        if (cap) {
            CUDA_CHECK(cudaMemcpyAsync(sorted, d_sorted.ptr, (size_t)cap * 4, cudaMemcpyDeviceToHost, stream));
        }
        CUDA_CHECK(cudaStreamSynchronize(stream));
    });
}
}
