// simt_hostcheck.cpp — TEST-ONLY shared library (libcrt_simt_hostcheck.so).
//
// Executes the product's k_traverse kernel (kernels.cuh) on the host with REAL warp semantics: every CUDA thread
// of a block is an OS thread, the 32 threads of a warp rendezvous at each warp collective (__ballot_sync,
// __shfl_*_sync, __syncwarp are barrier-backed exchanges), __shared__ arrays are shared by the block's threads and
// atomics are real atomics. That is the part of the backend the other host checks cannot reach — the persistent
// warps' dynamic ray fetch and refill, the shared-memory short stack, the warp-pooled triangle tests merged by a
// 64-bit atomicMin, the merged shadow + closest launch — so that tests/test_simt_host.py can compare the
// kernel's results, ray by ray and bit by bit, with the single-ray host instantiation of bvh8_traverse.h (itself
// checked against brute force), on a machine without a GPU. One block runs at a time (the kernel is persistent:
// a single block drains the whole queue). It is not linked into libcrt_cuda_core.so and render() cannot reach it.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "simt_env.h"

#include "bvh8.h"
#include "host_scene.h"
#include "kernels.cuh"

namespace {

std::string g_err;

struct SimtCheck {
    crt::SceneRecords rec;
};

}  // namespace

extern "C" {

const char *crt_simt_last_error() { return g_err.c_str(); }

void *crt_simt_create(const crt_scene_t *scene)
{
    try {
        auto *h = new SimtCheck();
        crt::pack_scene(scene, 0, h->rec);
        return h;
    } catch (const std::exception &e) {
        g_err = e.what();
        return nullptr;
    }
}

void crt_simt_destroy(void *p) { delete static_cast<SimtCheck *>(p); }

// out4: node-phase executions, lanes active in them, triangle passes, lanes active in them (since the last reset)
void crt_simt_profile(unsigned long long *out4, int reset)
{
    out4[0] = simt::profile.node_phases.load();
    out4[1] = simt::profile.node_lanes.load();
    out4[2] = simt::profile.tri_passes.load();
    out4[3] = simt::profile.tri_lanes.load();
    if (reset) {
        simt::profile.node_phases = 0;
        simt::profile.node_lanes = 0;
        simt::profile.tri_passes = 0;
        simt::profile.tri_lanes = 0;
    }
}

// One k_traverse launch (the production instantiation, COUNT = false) of `blocks` blocks of kTravBlock threads:
// closest rays: n x 8 floats (through an identity or a permuted queue), hits out: n x 4 {t, u, v, bits(flattened
// primitive id | 0xffffffff)} — the kernel stores the leaf-order triangle index, translated here like crtc_trace_closest
// any rays: m x 8 floats {o, tnear ignored (the kernel uses kEpsilon), d, tfar}, vis out: m bytes (1 = unoccluded)
// sched: bits 0-7 refill_idle, bit 8 far-first shadow rays, bits 16-23 (here only) the DEFER instantiation: 0 / 16 / 24.
// Single-ray results for comparison come from
// libcrt_bvh8_hostcheck.so.
void crt_simt_traverse(void *p, const float *closest, uint32_t n_closest, const uint32_t *queue_perm, const float *any,
                       uint32_t n_any, int blocks, int sched, float *hits_out, uint8_t *vis_out)
{
    SimtCheck *h = static_cast<SimtCheck *>(p);
    const uint32_t slots = std::max(1u, n_closest);
    std::vector<float4> ray_o(slots), ray_d(slots), hit(slots), sray_o(std::max(1u, n_any)), sray_d(std::max(1u, n_any));
    std::vector<uint8_t> vis(std::max(1u, n_any), 7);
    std::vector<uint32_t> queue(slots), counters(crt::kNumCounters, 0u);
    for (uint32_t i = 0; i < n_closest; ++i) {
        const float *r = closest + 8 * (size_t)i;
        ray_o[i] = make_float4(r[0], r[1], r[2], r[3]);
        ray_d[i] = make_float4(r[4], r[5], r[6], r[7]);
        hit[i] = make_float4(-1.f, -1.f, -1.f, 0.f);
        queue[i] = queue_perm ? queue_perm[i] : i;
    }
    for (uint32_t j = 0; j < n_any; ++j) {
        const float *r = any + 8 * (size_t)j;
        sray_o[j] = make_float4(r[0], r[1], r[2], r[7]);
        sray_d[j] = make_float4(r[4], r[5], r[6], __uint_as_float(j));
    }
    counters[crt::kCntQueue] = n_closest;
    counters[crt::kCntShadow] = n_any;
    crt::DeviceScene sc{};
    sc.nodes = reinterpret_cast<const float4 *>(h->rec.bvh.nodes.data());
    sc.tris = reinterpret_cast<const float4 *>(h->rec.tris.data());
    sc.float_one = 0x3F800000u;
    crt::PathState ps{};
    ps.ray_o = ray_o.data();
    ps.ray_d = ray_d.data();
    ps.hit = hit.data();
    ps.sray_o = sray_o.data();
    ps.sray_d = sray_d.data();
    ps.vis = vis.data();
    ps.queue[0] = queue.data();
    ps.queue[1] = queue.data();
    ps.counters = counters.data();
    unsigned long long trav[4] = {0, 0, 0, 0};
    ps.trav_counters = trav;
    uint32_t *work_counter = counters.data() + crt::kCntWork;

    for (int b = 0; b < blocks; ++b) {
        simt::Warp warps[crt::kTravBlock / 32];
        std::vector<std::thread> threads;
        for (int t = 0; t < crt::kTravBlock; ++t) {
            threads.emplace_back([&, t, b] {
                threadIdx.x = (unsigned)t;
                blockIdx.x = (unsigned)b;
                blockDim.x = crt::kTravBlock;
                gridDim.x = (unsigned)blocks;
                simt::warp = &warps[t / 32];
                simt::lane = t % 32;
                const uint32_t *any_count = n_any ? counters.data() + crt::kCntShadow : nullptr;
                switch ((sched >> 16) & 0xff) {  // test-only selector of the instantiation (option "tri_pass_defer")
                case 16:
                    crt::k_traverse<false, 16>(sc, ps, ps.queue[0], counters.data() + crt::kCntQueue, any_count, work_counter, sched & 0xffff);
                    break;
                case 24:
                    crt::k_traverse<false, 24>(sc, ps, ps.queue[0], counters.data() + crt::kCntQueue, any_count, work_counter, sched & 0xffff);
                    break;
                default:
                    crt::k_traverse<false>(sc, ps, ps.queue[0], counters.data() + crt::kCntQueue, any_count, work_counter, sched & 0xffff);
                    break;
                }
            });
        }
        for (auto &th : threads) {
            th.join();
        }
    }
    for (uint32_t i = 0; i < n_closest; ++i) {
        hits_out[4 * i] = hit[i].x;
        hits_out[4 * i + 1] = hit[i].y;
        hits_out[4 * i + 2] = hit[i].z;
        const uint32_t leaf = __float_as_uint(hit[i].w);
        const std::vector<uint32_t> &flat_ids = h->rec.leaf_flat_ids;
        hits_out[4 * i + 3] = __uint_as_float(leaf == crt::kMiss || leaf >= flat_ids.size() ? crt::kMiss : flat_ids[leaf]);
    }
    if (n_any) {
        std::memcpy(vis_out, vis.data(), n_any);
    }
}

// Option "shade_sort" at kernel level: k_queue_hist -> exclusive scan (done here on the host; the product scans with
// the k_scan_tile / k_scan_add kernels the device BVH build uses) -> k_queue_scatter over a queue of `n` path slots
// whose capacity is `capacity` (grids cover the capacity, the length is read from the counters as on the device).
// hit_tri[slot] = leaf-order triangle of the slot's hit or kMiss; tri_material[tri] = its material id.
void crt_simt_sort_queue(const uint32_t *hit_tri, uint32_t num_slots, const uint32_t *tri_material, uint32_t num_tris,
                         const uint32_t *queue, uint32_t n, uint32_t capacity, uint32_t *sorted_out)
{
    g_err.clear();
    std::vector<float4> hit(std::max(1u, num_slots)), shade(3 * (size_t)std::max(1u, num_tris));
    for (uint32_t i = 0; i < num_slots; ++i) {
        hit[i] = make_float4(1.f, 0.f, 0.f, __uint_as_float(hit_tri[i]));
    }
    for (uint32_t t = 0; t < num_tris; ++t) {
        shade[3 * (size_t)t] = make_float4(0.f, 0.f, 1.f, __uint_as_float(tri_material[t]));
    }
    std::vector<uint32_t> counters(crt::kNumCounters, 0u);
    const int bounce = 2;
    counters[crt::kCntQueue + bounce] = n;
    crt::DeviceScene sc{};
    sc.shade = shade.data();
    crt::PathState ps{};
    ps.hit = hit.data();
    ps.counters = counters.data();
    const uint32_t num_tiles = (capacity + crt::kSortTile - 1) / crt::kSortTile;
    std::vector<uint32_t> hist(256 * (size_t)num_tiles, 0xdeadbeefu), out(std::max(1u, capacity), 0xffffffffu);
    simt::launch(num_tiles, crt::kSortBlock, [&] { crt::k_queue_hist<256>(sc, ps, queue, bounce, hist.data(), num_tiles); });
    uint32_t run = 0;
    for (uint32_t &h : hist) {
        const uint32_t c = h;
        h = run;
        run += c;
    }
    if (run != n) {
        g_err = "crt_simt_sort_queue: the histogram does not add up to the queue length";
    }
    simt::launch(num_tiles, crt::kSortBlock, [&] { crt::k_queue_scatter<256>(sc, ps, queue, out.data(), bounce, hist.data(), num_tiles); });
    std::memcpy(sorted_out, out.data(), sizeof(uint32_t) * capacity);
}
}
