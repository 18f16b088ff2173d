// wavefront_hostcheck.cpp — TEST-ONLY shared library (libcrt_wavefront_hostcheck.so).
//
// Runs the product's KERNEL SOURCE on the host: kernels.cuh (k_raygen, k_shade, k_nee_resolve, k_resolve —
// the whole per-bounce logic: hit decode, material unpack, next-event estimation with MIS, continuation,
// Russian roulette, queue compaction, running-mean resolve, frames in flight) is compiled with g++ and every
// CUDA thread is executed as a plain function call, one "thread" = lane 0 of its own one-lane warp (the warp
// intrinsics degenerate to the identity, atomics to plain arithmetic). The closest-hit / any-hit stages use the
// host instantiation of bvh8_traverse.h (the warp-cooperative scheduling of k_traverse is GPU-only; its per-ray
// arithmetic is the same header). The launch sequence below mirrors crtc_renderer::enqueue_frame
// (crt_cuda_core.cu). What it buys: on a machine without a GPU, tests/test_wavefront_host.py renders frames
// through the kernels' own source and compares them with the oracle / the reference build at rounding level.
// It is not linked into libcrt_cuda_core.so and render() cannot reach it.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include <cuda_runtime.h>  // vector types only

// ---- the CUDA execution environment, for one lane ----
namespace {
struct Idx3 {
    unsigned x = 0, y = 0, z = 0;
};
}  // namespace
static thread_local Idx3 threadIdx, blockIdx, blockDim, gridDim;

template <typename T>
static inline T __ldg(const T *p)
{
    return *p;
}
static inline uint32_t __float_as_uint(float f)
{
    uint32_t u;
    std::memcpy(&u, &f, 4);
    return u;
}
static inline float __uint_as_float(uint32_t u)
{
    float f;
    std::memcpy(&f, &u, 4);
    return f;
}
static inline float __uint2float_rn(uint32_t u) { return (float)u; }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __ffs(unsigned v) { return __builtin_ffs((int)v); }
static inline unsigned __ballot_sync(unsigned, bool pred) { return pred ? 1u : 0u; }
template <typename T>
static inline T __shfl_sync(unsigned, T v, int)
{
    return v;
}
template <typename T>
static inline T __shfl_up_sync(unsigned, T v, int)
{
    return v;
}
template <typename T>
static inline T __shfl_down_sync(unsigned, T, int)
{
    return T(0);  // lanes 1..31 do not exist: they contribute nothing to a reduction
}
static inline void __syncwarp() {}
static inline unsigned __reduce_add_sync(unsigned, unsigned v) { return v; }
static inline unsigned __reduce_or_sync(unsigned, unsigned v) { return v; }
// (declarations for the block-level kernels of kernels.cuh, which are templates and never instantiated in this build)
static inline void __syncthreads() {}
static inline void __threadfence_system() {}
static inline unsigned long long crt_host_clock_ns() { return 0ull; }
template <typename T>
static inline unsigned __match_any_sync(unsigned, T)
{
    return 1u;
}
template <typename T>
static inline T atomicAdd(T *p, T v)
{
    const T old = *p;
    *p = old + v;
    return old;
}
static inline unsigned long long atomicMin(unsigned long long *p, unsigned long long v)
{
    const unsigned long long old = *p;
    *p = std::min(old, v);
    return old;
}
using std::max;
using std::min;
#ifndef __launch_bounds__
#define __launch_bounds__(...)
#endif

#include "bvh8.h"
#include "host_scene.h"
#include "kernels.cuh"

namespace {

std::string g_err;

struct HostWavefront {
    crt::SceneRecords rec;  // the scene in device layout, host memory
    uint32_t spp = 1;
    // framebuffer
    int fb_w = 0, fb_h = 0;
    uint32_t ntx = 0, npx_local = 0;
    std::vector<uint32_t> tile_ids;
    std::vector<float> accum_local, accum_full;
    std::vector<uint32_t> img_local, img_full;
    uint32_t frame_id = 0;
    int max_depth = 5;
    int rank = 0, world = 1;
    // path state
    std::vector<float4> ray_o, ray_d, hit, thr_rng, radiance, nee_T, nee_l1, nee_l2, sray_o, sray_d;
    std::vector<uint8_t> vis;
    std::vector<uint32_t> queue0, queue1, counters;
    unsigned long long trav_counters[4] = {0, 0, 0, 0};
    uint64_t last_rays = 0;

    crt::DeviceScene device_scene() const
    {
        crt::DeviceScene sc;
        sc.nodes = reinterpret_cast<const float4 *>(rec.bvh.nodes.data());
        sc.tris = reinterpret_cast<const float4 *>(rec.tris.data());
        sc.shade = reinterpret_cast<const float4 *>(rec.shade.data());
        sc.materials = reinterpret_cast<const float4 *>(rec.shading.materials.data());
        sc.lights = reinterpret_cast<const float4 *>(rec.shading.lights.data());
        sc.texels = rec.shading.texels.data();
        sc.tex = reinterpret_cast<const crt::DevTex *>(rec.shading.tex_desc.data());
        sc.num_lights = (uint32_t)rec.shading.lights.size();
        sc.float_one = 0x3F800000u;
        return sc;
    }

    void set_scene(const crt_scene_t *scene)
    {
        // crtc_renderer::set_scene: the kernels read the records where pack_scene left them
        crt::pack_scene(scene, 0, rec);
        spp = rec.shading.spp;
        frame_id = 0;
        std::fill(accum_local.begin(), accum_local.end(), 0.f);
    }

    void initialize(int w, int h)
    {
        // crtc_renderer::initialize
        fb_w = w;
        fb_h = h;
        frame_id = 0;
        ntx = crt::tiles_along(w);
        tile_ids = crt::rank_tiles(w, h, rank, world);
        npx_local = (uint32_t)tile_ids.size() * crt::kTilePixels;
        accum_local.assign((size_t)npx_local * 3, 0.f);
        img_local.assign(npx_local, 0u);
        accum_full.assign((size_t)w * h * 3, 0.f);
        img_full.assign((size_t)w * h, 0u);
    }

    template <typename F>
    static void launch(size_t nthreads, const F &kernel)
    {
        blockDim.x = 1;
        threadIdx.x = 0;
        gridDim.x = (unsigned)nthreads;  // (k_shade / k_nee_resolve stride over their queue by gridDim.x * blockDim.x)
        for (size_t i = 0; i < nthreads; ++i) {
            blockIdx.x = (unsigned)i;
            kernel();
        }
    }

    // the work of one k_traverse launch: shadow rays [0, n_any) then closest-hit rays through `queue`
    void traverse(const crt::PathState &ps, const uint32_t *queue, uint32_t n_closest, uint32_t n_any, bool far_first)
    {
        const crt::DeviceScene sc = device_scene();
        for (uint32_t j = 0; j < n_any; ++j) {
            const float4 o = ps.sray_o[j], d = ps.sray_d[j];
            const crt::Ray ray{o.x, o.y, o.z, crt::kEpsilon, d.x, d.y, d.z, o.w};
            crt::HitRecord h;
            crt::bvh8_trace<true, false>(sc.nodes, sc.tris, ray, h, nullptr, far_first);
            ps.vis[__float_as_uint(d.w)] = h.tri != crt::kMiss ? 0 : 1;
        }
        for (uint32_t j = 0; j < n_closest; ++j) {
            const uint32_t slot = queue ? queue[j] : j;
            const float4 o = ps.ray_o[slot], d = ps.ray_d[slot];
            const crt::Ray ray{o.x, o.y, o.z, o.w, d.x, d.y, d.z, d.w};
            crt::HitRecord h;
            crt::bvh8_trace<false, false>(sc.nodes, sc.tris, ray, h, nullptr);
            const bool hit = h.tri != crt::kMiss;
            ps.hit[slot] = make_float4(h.t, hit ? h.u : 0.f, hit ? h.v : 0.f, __uint_as_float(h.tri));
        }
    }

    // crtc_renderer::enqueue_frame
    void render(const float *pos, const float *dir, const float *up, float fovy, bool camera_changed, uint32_t num_frames,
                bool far_first)
    {
        if (camera_changed) {
            frame_id = 0;
        }
        const crt::ViewParams view = crt::make_view_params(pos, dir, up, fovy, fb_w, fb_h, frame_id);
        const size_t npaths = (size_t)npx_local * spp * num_frames;
        for (auto *v : {&ray_o, &ray_d, &hit, &thr_rng, &radiance, &nee_T, &nee_l1, &nee_l2}) {
            v->assign(npaths, make_float4(0.f, 0.f, 0.f, 0.f));
        }
        sray_o.assign(2 * npaths, make_float4(0.f, 0.f, 0.f, 0.f));
        sray_d.assign(2 * npaths, make_float4(0.f, 0.f, 0.f, 0.f));
        vis.assign(2 * npaths, 0);
        queue0.assign(npaths, 0u);
        queue1.assign(npaths, 0u);
        counters.assign(crt::kNumCounters, 0u);
        crt::PathState ps;
        ps.ray_o = ray_o.data();
        ps.ray_d = ray_d.data();
        ps.hit = hit.data();
        ps.thr_rng = thr_rng.data();
        ps.radiance = radiance.data();
        ps.nee_T = nee_T.data();
        ps.nee_l1 = nee_l1.data();
        ps.nee_l2 = nee_l2.data();
        ps.sray_o = sray_o.data();
        ps.sray_d = sray_d.data();
        ps.vis = vis.data();
        ps.queue[0] = queue0.data();
        ps.queue[1] = queue1.data();
        ps.counters = counters.data();
        ps.trav_counters = trav_counters;
        const crt::DeviceScene sc = device_scene();
        crt::FrameLayout fl;
        fl.fb_w = fb_w;
        fl.fb_h = fb_h;
        fl.ntx = ntx;
        fl.npx_local = npx_local;
        fl.spp = spp;
        fl.frames = num_frames;
        fl.tile_ids = tile_ids.data();

        if (npaths) {
            launch(npaths, [&] { crt::k_raygen(view, fl, ps); });
            traverse(ps, ps.queue[0], counters[crt::kCntQueue], 0, far_first);
            for (int b = 0; b < max_depth; ++b) {
                uint32_t *qin = ps.queue[b & 1], *qout = ps.queue[(b + 1) & 1];
                launch(npaths, [&] { crt::k_shade<false>(sc, ps, qin, qout, b, max_depth); });
                const bool last = b + 1 == max_depth;
                traverse(ps, qout, last ? 0u : counters[crt::kCntQueue + b + 1], counters[crt::kCntShadow + b], far_first);
                launch(npaths, [&] { crt::k_nee_resolve(ps, qin, b); });
            }
            const bool full = world == 1;
            launch(npx_local, [&] {
                crt::k_resolve(fl, ps, frame_id, accum_local.data(), img_local.data(), full ? accum_full.data() : nullptr,
                               full ? img_full.data() : nullptr, nullptr, nullptr, 0u);
            });
        }
        last_rays = 0;
        for (int b = 0; b < max_depth; ++b) {
            last_rays += counters[crt::kCntQueue + b] + counters[crt::kCntShadow + b];
        }
        frame_id += num_frames;
    }
};

// wave_devcheck.cu's state image, layout and view arguments as the kernels' structs (host pointers, used in place)
crt::PathState state_image(void *const *st)
{
    static unsigned long long trav[4];
    auto f4 = [&](int k) { return static_cast<float4 *>(st[k]); };
    crt::PathState ps;
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
    ps.vis = static_cast<uint8_t *>(st[10]);
    ps.queue[0] = static_cast<uint32_t *>(st[11]);
    ps.queue[1] = static_cast<uint32_t *>(st[12]);
    ps.counters = static_cast<uint32_t *>(st[13]);
    ps.trav_counters = trav;
    return ps;
}

crt::FrameLayout frame_layout(const uint32_t *lay, const uint32_t *tile_ids)
{
    crt::FrameLayout fl;
    fl.fb_w = (int)lay[0];
    fl.fb_h = (int)lay[1];
    fl.ntx = lay[2];
    fl.npx_local = lay[3];
    fl.spp = lay[4];
    fl.frames = lay[5];
    fl.tile_ids = tile_ids;
    return fl;
}

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

}  // namespace

extern "C" {

const char *crt_wavecheck_last_error() { return g_err.c_str(); }

void *crt_wavecheck_create(const crt_scene_t *scene, int w, int h, int max_depth, int rank, int world)
{
    try {
        auto *r = new HostWavefront();
        r->max_depth = max_depth;
        r->rank = rank;
        r->world = world;
        r->initialize(w, h);
        r->set_scene(scene);
        return r;
    } catch (const std::exception &e) {
        g_err = e.what();
        return nullptr;
    }
}

void crt_wavecheck_destroy(void *p) { delete static_cast<HostWavefront *>(p); }

// renders `num_frames` consecutive frames as one wavefront; returns the ray count (closest-hit + occlusion casts)
uint64_t crt_wavecheck_render(void *p, const float *pos, const float *dir, const float *up, float fovy, int camera_changed,
                              uint32_t num_frames, int far_first)
{
    HostWavefront *r = static_cast<HostWavefront *>(p);
    r->render(pos, dir, up, fovy, camera_changed != 0, num_frames, far_first != 0);
    return r->last_rays;
}

// crtc_renderer::assemble_rank: scatter rank `src`'s tile-local buffers into `dst`'s full frame (k_assemble)
void crt_wavecheck_assemble(void *dst_, void *src_)
{
    HostWavefront *dst = static_cast<HostWavefront *>(dst_), *src = static_cast<HostWavefront *>(src_);
    if (src->npx_local == 0) {
        return;
    }
    crt::FrameLayout f;
    f.fb_w = dst->fb_w;
    f.fb_h = dst->fb_h;
    f.ntx = dst->ntx;
    f.npx_local = src->npx_local;
    f.spp = dst->spp;
    f.frames = 1;
    f.tile_ids = src->tile_ids.data();
    HostWavefront::launch(f.npx_local, [&] {
        crt::k_assemble(f, src->accum_local.data(), src->img_local.data(), dst->accum_full.data(), dst->img_full.data());
    });
}

void crt_wavecheck_read(void *p, float *accum_full, uint32_t *img_full)
{
    HostWavefront *r = static_cast<HostWavefront *>(p);
    std::memcpy(accum_full, r->accum_full.data(), r->accum_full.size() * sizeof(float));
    std::memcpy(img_full, r->img_full.data(), r->img_full.size() * sizeof(uint32_t));
}

// ---- the per-stage entry points of wave_devcheck.cu (same names, signatures and state image), over the one-lane
// launches above: tests/test_wavefront_device.py runs each stage here on the state it gave the device ----

const char *wavekat_last_error() { return g_err.c_str(); }

void *wavekat_scene(const crt_scene_t *scene)
{
    try {
        auto *r = new HostWavefront();
        r->set_scene(scene);
        return r;
    } catch (const std::exception &e) {
        g_err = e.what();
        return nullptr;
    }
}

void wavekat_scene_free(void *s) { delete static_cast<HostWavefront *>(s); }

// (this build only) the scene's records as both builds upload them, for the restatements: field 0 shading records
// (48 B per triangle, leaf order), 1 materials (64 B each), 2 lights (80 B each), 3 texel arena (4 B per texel),
// 4 texture descriptors (16 B each). dst null: only the size. Returns the bytes, -1 for an unknown field.
long long wavekat_records(void *scene, int field, void *dst)
{
    const crt::SceneRecords &rec = static_cast<HostWavefront *>(scene)->rec;
    auto put = [&](const auto &v) {
        const size_t bytes = v.size() * sizeof(v[0]);
        if (dst && bytes) {
            std::memcpy(dst, v.data(), bytes);
        }
        return (long long)bytes;
    };
    switch (field) {
    case 0: return put(rec.shade);
    case 1: return put(rec.shading.materials);
    case 2: return put(rec.shading.lights);
    case 3: return put(rec.shading.texels);
    case 4: return put(rec.shading.tex_desc);
    default: return -1;
    }
}

int wavekat_raygen(const float *view, uint32_t frame_id, const uint32_t *lay, const uint32_t *tile_ids, const uint32_t *sel,
                   uint32_t cap, void *const *st)
{
    const crt::PathState ps = state_image(st);
    const crt::FrameLayout fl = frame_layout(lay, tile_ids);
    const crt::ViewParams v = view_params(view, frame_id);
    const size_t npaths = (size_t)fl.npx_local * fl.spp * fl.frames;
    (void)cap;
    if (sel) {
        crt::AdaptiveFrame ad{};
        ad.sel = reinterpret_cast<const uint2 *>(sel);
        HostWavefront::launch(npaths, [&] { crt::k_raygen<true>(v, fl, ps, ad); });
    } else {
        HostWavefront::launch(npaths, [&] { crt::k_raygen<false>(v, fl, ps); });
    }
    return 0;
}

int wavekat_traverse(void *scene, int queue_index, int closest_counter, int any_counter, int work_counter, int far_first,
                     uint32_t cap, void *const *st)
{
    HostWavefront *r = static_cast<HostWavefront *>(scene);
    const crt::PathState ps = state_image(st);
    (void)work_counter;
    (void)cap;
    r->traverse(ps, ps.queue[queue_index & 1], closest_counter >= 0 ? ps.counters[closest_counter] : 0u,
                any_counter >= 0 ? ps.counters[any_counter] : 0u, far_first != 0);
    return 0;
}

int wavekat_shade(void *scene, int bounce, int max_depth, uint32_t cap, void *const *st)
{
    const crt::DeviceScene sc = static_cast<HostWavefront *>(scene)->device_scene();
    const crt::PathState ps = state_image(st);
    HostWavefront::launch(cap, [&] { crt::k_shade<false>(sc, ps, ps.queue[bounce & 1], ps.queue[(bounce + 1) & 1], bounce, max_depth); });
    return 0;
}

int wavekat_nee_resolve(int bounce, uint32_t cap, void *const *st, uint32_t *grid)
{
    const crt::PathState ps = state_image(st);
    *grid = cap;
    HostWavefront::launch(cap, [&] { crt::k_nee_resolve(ps, ps.queue[bounce & 1], bounce); });
    return 0;
}

int wavekat_resolve(const uint32_t *lay, const uint32_t *tile_ids, uint32_t frame_id, const uint32_t *sel, float *moments,
                    uint32_t stat_base, float *accum_local, uint32_t *img_local, float *accum_full, uint32_t *img_full,
                    uint32_t cap, void *const *st)
{
    const crt::PathState ps = state_image(st);
    const crt::FrameLayout fl = frame_layout(lay, tile_ids);
    (void)cap;
    if (sel) {
        crt::AdaptiveFrame ad{};
        ad.sel = reinterpret_cast<const uint2 *>(sel);
        ad.moments = reinterpret_cast<float2 *>(moments);
        ad.stat_base = stat_base;
        HostWavefront::launch(fl.npx_local, [&] {
            crt::k_resolve<true>(fl, ps, frame_id, accum_local, img_local, accum_full, img_full, nullptr, nullptr, 0u, ad);
        });
    } else {
        HostWavefront::launch(fl.npx_local, [&] {
            crt::k_resolve<false>(fl, ps, frame_id, accum_local, img_local, accum_full, img_full, nullptr, nullptr, 0u);
        });
    }
    return 0;
}

// the shade-queue sort's result: a stable sort of the queue by shade_bucket (k_queue_hist / k_queue_scatter need a
// 256-thread block, which this build does not have)
int wavekat_queue_sort(void *scene, int bounce, uint32_t cap, void *const *st, uint32_t *sorted)
{
    const crt::DeviceScene sc = static_cast<HostWavefront *>(scene)->device_scene();
    const crt::PathState ps = state_image(st);
    (void)cap;
    const uint32_t *qin = ps.queue[bounce & 1];
    const uint32_t n = ps.counters[crt::kCntQueue + bounce];
    std::vector<uint32_t> q(qin, qin + n);
    std::stable_sort(q.begin(), q.end(),
                     [&](uint32_t a, uint32_t b) { return crt::shade_bucket(sc, ps, a) < crt::shade_bucket(sc, ps, b); });
    std::copy(q.begin(), q.end(), sorted);
    return 0;
}
}
