// kernels.cuh — the per-frame hot path as a chain of sm_90a kernels (wavefront style).
//
// One kernel per stage over a device-resident, per-bounce compacted ray queue:
//
//   k_raygen            render_embree.ispc:212-232   rng seed, pixel jitter, primary ray
//   k_traverse_closest  render_embree.ispc:245       (rtcIntersectV)  BVH8 + Moeller-Trumbore
//   k_shade             render_embree.ispc:251-336   miss shader, hit decode, material unpack,
//                                                    NEE with MIS (emits <= 2 shadow rays),
//                                                    BSDF continuation, Russian roulette,
//                                                    warp-aggregated queue compaction
//   k_traverse_any      render_embree.ispc:144,170   (rtcOccludedV)   any-hit
//   k_nee_resolve       render_embree.ispc:148-178,301  adds the unoccluded NEE terms in the
//                                                    reference's order (light sample first)
//   k_resolve           render_embree.ispc:339-353, 358-370  sample mean, running mean, sRGB8
//
// No OptiX, no RT-core intrinsics, no tensor cores (BASELINE.json north_star).
// Compiled with -fmad=false: shading arithmetic follows the reference's operation order;
// the traversal uses explicit fma (bvh8_traverse.h).
#pragma once

#include <cmath>
#include <cstdint>
#include <vector>
#include <cuda_runtime.h>

#include "bvh8_traverse.h"
#include "shade_math.cuh"

namespace crt {

constexpr uint32_t kMiss = 0xffffffffu;
constexpr int kTile = 64;                 // render_embree.h:25
constexpr uint32_t kTilePixels = kTile * kTile;
constexpr int kMaxDepthSupported = 16;
// counters layout (uint32): [0..16] queue length entering bounce b; [17..33] shadow rays
// emitted at bounce b; [34] paths started
constexpr int kCntQueue = 0;
constexpr int kCntShadow = 17;
constexpr int kCntPaths = 34;
constexpr int kCntWork = 36;  // [36..53] work-distribution cursors of the traversal launches
constexpr int kNumCounters = 56;

struct ViewParams {
    float3 pos, dir_du, dir_dv, dir_top_left;  // embree_utils.h:137-140
    uint32_t frame_id;
};

// The camera basis on the host, render_embree.cpp:149-159 / render_optix.cpp:454-460. Its callers are compiled with
// -ffp-contract=off, so that the basis is the reference's to the bit.
inline ViewParams make_view_params(const float *pos, const float *dir_, const float *up_, float fovy, int fb_w, int fb_h,
                                   uint32_t frame_id)
{
    // glm::normalize(v) = v * inversesqrt(dot(v, v)), inversesqrt(x) = 1 / sqrt(x)
    const auto glm_normalize = [](float3 v) {
        const float inv = 1.f / std::sqrt(v.x * v.x + v.y * v.y + v.z * v.z);
        return make_float3(v.x * inv, v.y * inv, v.z * inv);
    };
    const auto cross3 = [](float3 a, float3 b) {
        return make_float3(a.y * b.z - b.y * a.z, a.z * b.x - b.z * a.x, a.x * b.y - b.x * a.y);
    };
    const float3 dir = make_float3(dir_[0], dir_[1], dir_[2]);
    const float3 up = make_float3(up_[0], up_[1], up_[2]);
    const float plane_y = 2.f * std::tan((0.5f * fovy) * 0.01745329251994329576923690768489f);
    const float plane_x = plane_y * static_cast<float>(fb_w) / static_cast<float>(fb_h);
    ViewParams v;
    v.pos = make_float3(pos[0], pos[1], pos[2]);
    const float3 du = glm_normalize(cross3(dir, up));
    v.dir_du = make_float3(du.x * plane_x, du.y * plane_x, du.z * plane_x);
    const float3 dvn = glm_normalize(cross3(v.dir_du, dir));
    v.dir_dv = make_float3(-dvn.x * plane_y, -dvn.y * plane_y, -dvn.z * plane_y);
    v.dir_top_left = make_float3(dir.x - 0.5f * v.dir_du.x - 0.5f * v.dir_dv.x,
                                 dir.y - 0.5f * v.dir_du.y - 0.5f * v.dir_dv.y,
                                 dir.z - 0.5f * v.dir_du.z - 0.5f * v.dir_dv.z);
    v.frame_id = frame_id;
    return v;
}

// Tiles along a framebuffer side of n pixels (render_embree.cpp:43-44)
inline uint32_t tiles_along(int n) { return n / kTile + (n % kTile != 0 ? 1 : 0); }

// The row-major ids of the tiles that rank `rank` of `world` renders: every world-th tile, starting at its own rank
inline std::vector<uint32_t> rank_tiles(int w, int h, int rank, int world)
{
    std::vector<uint32_t> tiles;
    for (uint32_t t = 0; t < tiles_along(w) * tiles_along(h); ++t) {
        if ((int)(t % (uint32_t)world) == rank) {
            tiles.push_back(t);
        }
    }
    return tiles;
}

struct DeviceScene {
    const float4 *nodes;      // 5 per BVH8 node
    const float4 *tris;       // 3 per triangle, leaf order: {v0|flat id}, {e1}, {e2}
    const float4 *shade;      // 3 per triangle, leaf order: TriShade
    const float4 *materials;  // 4 per material (DisneyMaterial, util/material.h:29-46)
    const float4 *lights;     // 5 per light (QuadLight, util/lights.h:6-18)
    const uint32_t *texels;
    const DevTex *tex;
    const unsigned long long *tex_objects;  // cudaTextureObject_t per texture (option "hw_textures"), else null
    uint32_t num_lights;
    uint32_t float_one;  // 0x3F800000 as a run-time value (bvh8_traverse.h: byte_unit)
};

struct FrameLayout {
    int fb_w, fb_h;
    uint32_t ntx;             // tiles per row
    uint32_t npx_local;       // num_local_tiles * 4096
    uint32_t spp;
    uint32_t frames;          // consecutive frames rendered by this launch sequence (>= 1): their
                              // frames * spp samples per pixel are in flight together
    const uint32_t *tile_ids; // global tile id of each local tile
};

struct PathState {
    float4 *ray_o;     // org.xyz, tnear
    float4 *ray_d;     // dir.xyz, tfar
    float4 *hit;       // t, u, v, bits(leaf-order triangle index | kMiss)
    float4 *thr_rng;   // path_throughput.xyz, bits(rng state)
    float4 *radiance;  // per-sample illum.xyz
    float4 *nee_T;     // throughput before this bounce's update, bits(flags: 4 = missed (environment term pending), 2 = hit (NEE valid), 1 = has shadow ray B, 8 = has nee_l1)
    float4 *nee_l1;    // light-sample contribution (without throughput); written only where it passed the pdf tests
    float4 *nee_l2;    // BSDF-sample contribution
    float4 *sray_o;    // shadow ray org.xyz, tfar   (indexed by shadow-queue position)
    float4 *sray_d;    // shadow ray dir.xyz, bits(path slot * 2 + which)
    uint8_t *vis;      // 2 per path slot: 1 = unoccluded
    uint32_t *queue[2];
    uint32_t *counters;
    unsigned long long *trav_counters;  // closest: [0] nodes visited [1] triangles tested; any-hit: [2], [3]
};

// Local pixel index -> framebuffer coordinates. Within a 64x64 tile pixels are ordered in
// 8x4 blocks so that the 32 lanes of a warp cover a compact screen rectangle.
__device__ __forceinline__ bool local_pixel_coords(const FrameLayout &f, uint32_t lp, uint32_t &x, uint32_t &y)
{
    const uint32_t lt = lp / kTilePixels, within = lp % kTilePixels;
    const uint32_t tile = __ldg(f.tile_ids + lt);
    const uint32_t blk = within >> 5, lane = within & 31u;
    x = (tile % f.ntx) * kTile + (blk & 7u) * 8u + (lane & 7u);
    y = (tile / f.ntx) * kTile + (blk >> 3) * 4u + (lane >> 3);
    return x < (uint32_t)f.fb_w && y < (uint32_t)f.fb_h;
}

// Appends one item per predicated lane with a single atomic per warp; order inside the warp is
// preserved. All 32 lanes must call.
__device__ __forceinline__ uint32_t warp_append(uint32_t *counter, bool pred)
{
    const unsigned mask = __ballot_sync(0xffffffffu, pred);
    if (mask == 0) {
        return 0;
    }
    const int lane = threadIdx.x & 31;
    const int leader = __ffs(mask) - 1;
    uint32_t base = 0;
    if (lane == leader) {
        base = atomicAdd(counter, (uint32_t)__popc(mask));
    }
    base = __shfl_sync(0xffffffffu, base, leader);
    return base + (uint32_t)__popc(mask & ((1u << lane) - 1u));
}

// Adaptive sampling (crtc_set_adaptive, adaptive.cuh): the per-block selection k_adaptive_select made for this wavefront.
// Block b = local pixels 32b .. 32b+31 (one 8x4 screen block, one warp of k_raygen and k_resolve): sel[b] = {c_b, n_b}, the
// frames the block had accumulated before this wavefront and the frames it renders in it. moments[lp] = (m1, m2), the
// running means of L and L^2, whose count starts at stat_base.
struct AdaptiveFrame {
    const uint2 *sel;
    float2 *moments;
    uint32_t stat_base;
};

// ---------------------------------------------------------------------------------------
// ADAPTIVE: only the first n_b frames of each block are enqueued, seeded as frames c_b, c_b + 1, ... of the uniform render.
template <bool ADAPTIVE = false>
__global__ void __launch_bounds__(256) k_raygen(ViewParams view, FrameLayout f, PathState ps, AdaptiveFrame ad = AdaptiveFrame{})
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t npaths = f.npx_local * f.spp * f.frames;
    bool valid = false;
    if (i < npaths) {
        // sample index over the batch: frame (view.frame_id + s / spp), sample s % spp of it
        const uint32_t lp = i % f.npx_local, s = i / f.npx_local;
        uint32_t first = view.frame_id;
        bool active = true;
        if (ADAPTIVE) {  // (warp-uniform: npx_local is a multiple of 32, so a warp's 32 paths are one block's)
            const uint2 sel = ad.sel[lp >> 5];
            first = sel.x;
            active = s < sel.y * f.spp;
        }
        uint32_t x, y;
        if (active && local_pixel_coords(f, lp, x, y)) {
            valid = true;
            // render_embree.ispc:213-232; (frame_id + k) * spp + 1 + (s - k * spp) == frame_id * spp + 1 + s
            uint32_t rng = get_rng(x + y * (uint32_t)f.fb_w, first * f.spp + 1u + s);
            const float px_x = ((float)x + lcg_randomf(rng)) / (float)(uint32_t)f.fb_w;
            const float px_y = ((float)y + lcg_randomf(rng)) / (float)(uint32_t)f.fb_h;
            const float3 dir = normalize(mk3(view.dir_du.x * px_x + view.dir_dv.x * px_y + view.dir_top_left.x,
                                             view.dir_du.y * px_x + view.dir_dv.y * px_y + view.dir_top_left.y,
                                             view.dir_du.z * px_x + view.dir_dv.z * px_y + view.dir_top_left.z));
            ps.ray_o[i] = make_float4(view.pos.x, view.pos.y, view.pos.z, 0.f);
            ps.ray_d[i] = make_float4(dir.x, dir.y, dir.z, 1e20f);
            ps.thr_rng[i] = make_float4(1.f, 1.f, 1.f, __uint_as_float(rng));
            ps.radiance[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    const uint32_t idx = warp_append(ps.counters + kCntQueue, valid);
    if (valid) {
        ps.queue[0][idx] = i;
    }
}

// ---------------------------------------------------------------------------------------
// Multi-view wavefronts (crtc_render_views): the F frames of V cameras traced together. Path i = lp + s * (V * npx_local),
// local pixel lp = v * npx_local + lp_v of view v; npx_local is a multiple of 4096, so a warp never straddles two views.
// The table is a kernel parameter (64 x 52 B, within CUDA 12.1's 32 KB limit): no upload, no synchronisation.
// view[v].frame_id = b_v, the frames view v has accumulated since its last reset.
constexpr uint32_t kMaxViews = 64;
struct ViewTable {
    ViewParams view[kMaxViews];
    uint32_t num_views;
};

// k_raygen for every view of the table: path (v, lp_v, s) is seeded as k_raygen seeds sample s of pixel lp_v for view v's
// camera and frame b_v, so that each view's paths are those of a one-view wavefront.
__global__ void __launch_bounds__(256) k_raygen_views(const __grid_constant__ ViewTable views, FrameLayout f, PathState ps)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t npx_all = f.npx_local * views.num_views;
    const uint32_t npaths = npx_all * f.spp * f.frames;
    bool valid = false;
    if (i < npaths) {
        const uint32_t lp = i % npx_all, s = i / npx_all;
        const ViewParams &view = views.view[lp / f.npx_local];
        uint32_t x, y;
        if (local_pixel_coords(f, lp % f.npx_local, x, y)) {
            valid = true;
            uint32_t rng = get_rng(x + y * (uint32_t)f.fb_w, view.frame_id * f.spp + 1u + s);
            const float px_x = ((float)x + lcg_randomf(rng)) / (float)(uint32_t)f.fb_w;
            const float px_y = ((float)y + lcg_randomf(rng)) / (float)(uint32_t)f.fb_h;
            const float3 dir = normalize(mk3(view.dir_du.x * px_x + view.dir_dv.x * px_y + view.dir_top_left.x,
                                             view.dir_du.y * px_x + view.dir_dv.y * px_y + view.dir_top_left.y,
                                             view.dir_du.z * px_x + view.dir_dv.z * px_y + view.dir_top_left.z));
            ps.ray_o[i] = make_float4(view.pos.x, view.pos.y, view.pos.z, 0.f);
            ps.ray_d[i] = make_float4(dir.x, dir.y, dir.z, 1e20f);
            ps.thr_rng[i] = make_float4(1.f, 1.f, 1.f, __uint_as_float(rng));
            ps.radiance[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    const uint32_t idx = warp_append(ps.counters + kCntQueue, valid);
    if (valid) {
        ps.queue[0][idx] = i;
    }
}

// ---------------------------------------------------------------------------------------
// Traversal kernels: persistent warps with dynamic ray fetch.
//
// Measured on the first (one-thread-per-ray) version: incoherent bounce rays ran at 7-8 active
// lanes per instruction because a warp lived as long as its longest ray. Here every warp stays
// resident, pulls rays from the queue in batches (one atomic per kFetchBatch rays), advances
// all live lanes one traversal step at a time and refills idle lanes as soon as at least
// kRefillIdle of them have finished (Aila & Laine 2009; Ylitie et al. 2017 §5). Node tests stay
// per lane; the triangles they yield are pooled across the warp and tested 32 pairs at a time
// (see the loop body). The first kSmemStack entries of each lane's traversal stack live in shared
// memory, the rest spills to local memory.
// The 9 launches of a C2 frame take 6.74 ms on an H100 80GB HBM3 at a 400 W power limit (7.02 ms with the FMNMX slab
// test before the integer one; profiles/launches_c2_h100_traverse_*.md). At (kTravBlock, 8) the kernel has 64 registers
// and no spills; (128, 9) = 56 registers measured 6.76 ms, (128, 10) = 48 registers spills 42 B and measured 7.89 ms.
// Profiling hooks of the SIMT emulation (simt_hostcheck.cpp defines them before including this file); they
// expand to nothing everywhere else, the CUDA build included.
#ifndef CRT_PROF_NODE_PHASE
#define CRT_PROF_NODE_PHASE(lane_has_node)
#define CRT_PROF_TRI_PASS(lane_has_pair)
#endif

constexpr int kTravBlock = 128;
constexpr int kSmemStack = 8;
constexpr int kRefillIdle = 4;
constexpr uint32_t kFetchBatch = 64;

// One launch serves both ray kinds so that the shadow rays of bounce b and the continuation rays
// of bounce b+1 (both known once k_shade(b) has run) share a launch: half as many traversal
// launches per frame and twice the rays per launch, which matters when a GPU only holds 1/8 of the
// image. Work items [0, n_any) are shadow rays (sray_o/sray_d -> vis[], rtcOccludedV,
// render_embree.ispc:144,170); items [n_any, n_any + n_closest) are closest-hit rays (ray_o/ray_d
// through `queue`, or identity when null -> hit[], rtcIntersectV, render_embree.ispc:245).
// DEFER > 0 (option "tri_pass_defer", off by default): a triangle pass runs only once DEFER (lane, triangle) pairs
// are pooled or no lane can descend any further; a lane whose triangle group is still untested waits. Fewer,
// fuller passes for emptier node phases (DESIGN.md §2 "Warp-level work": 0.571 -> 0.523 in the emulation's cost
// model at DEFER = 16); same results, since the closest hit does not depend on the order of the tests.
// TOP (option "bvh_top_smem", off by default): the first kTopNodes nodes of the tree (BFS order: the root, its children,
// their children = 1 + 8 + 64) are copied into shared memory at block start and read from there. BASELINE.json's
// north_star asks for BVH nodes staged in shared memory; measured on an H100 SXM it does not pay (frame +2-3 % on C2 / C4):
// those nodes are the hottest lines of the L1 anyway and the copy takes 5.8 KB per block = 47 KB of L1 per SM away.
constexpr uint32_t kTopNodes = 73;

// The hit merge of k_traverse takes the 64-bit minimum of hit_key(t) << 32 | flat id. hit_key is monotone over every
// float t (a negative t has all bits flipped, a non-negative one only its sign bit), so hits behind the origin of a ray
// with tnear < 0 (crtc_trace_closest) merge like any other. -0 takes the key of +0: test_next_triangle treats them as
// equal and breaks the tie on the flat id. hit_key_t inverts the map (giving +0 for either zero).
__device__ __forceinline__ uint32_t hit_key(float t)
{
    const uint32_t u = f2u(t + 0.f);  // -0 + 0 = +0; every other t is unchanged
    return u ^ ((uint32_t)((int32_t)u >> 31) | 0x80000000u);
}
__device__ __forceinline__ float hit_key_t(uint32_t k)
{
    return u2f(k ^ ((uint32_t)((int32_t)~k >> 31) | 0x80000000u));
}

template <bool COUNT, int DEFER = 0, bool TOP = false>
__global__ void __launch_bounds__(kTravBlock, 8)
    k_traverse(DeviceScene sc, PathState ps, const uint32_t *queue, const uint32_t *count_closest_ptr,
               const uint32_t *count_any_ptr, uint32_t *work_counter, int sched, uint32_t num_nodes = 0)
{
    __shared__ float4 sm_top[TOP ? kTopNodes * 5 : 1];
    const uint32_t top_nodes = TOP ? min(num_nodes, kTopNodes) : 0u;
    if (TOP) {
        for (uint32_t i = threadIdx.x; i < top_nodes * 5u; i += blockDim.x) {
            sm_top[i] = sc.nodes[i];
        }
        __syncthreads();
    }
    // sched: bits 0-7 = idle lanes that trigger a refill; bit 8 = shadow rays visit children far-first
    const int refill_idle = sched & 0xff;
    const bool any_far_first = (sched & 0x100) != 0;
    __shared__ uint2 sm_stack[kSmemStack * kTravBlock];
    // warp-cooperative triangle testing: per warp, every lane's ray and best hit live in
    // shared memory so that ANY lane can test a (ray, triangle) pair for its owner
    __shared__ float sm_ray[kTravBlock / 32][8][32];            // ox oy oz tnear dx dy dz tfar0
    __shared__ unsigned long long sm_key[kTravBlock / 32][32];  // hit_key(t) << 32 | flat id  (atomicMin)
    __shared__ float4 sm_hit[kTravBlock / 32][32];              // u, v, bits(leaf-order triangle | kMiss), t of the best hit: one 128-bit store
    __shared__ uint32_t sm_owner[kTravBlock / 32][32];          // owner lane of the group that starts at slot s
    __shared__ uint32_t sm_cursor[kTravBlock / 32];             // running slot cursor of the warp (never reset)
    __shared__ uint32_t sm_is_any[kTravBlock / 32][32];         // ray kind per lane (instrumented build only)
    const int warp = threadIdx.x >> 5;
    const uint32_t n_any = count_any_ptr ? *count_any_ptr : 0u;
    const uint32_t count = n_any + (count_closest_ptr ? *count_closest_ptr : 0u);
    const int lane = threadIdx.x & 31;
    const unsigned lanemask_lt = (1u << lane) - 1u;
    const uint32_t batch = count > 8u * gridDim.x * kTravBlock ? kFetchBatch : 32u;
    // traversal stack: entries [0, kSmemStack) in this thread's column of shared memory, deeper ones (rare) in local
    // memory. The depth and the column pointer are plain locals: as members of one struct with the spill array they
    // lived in local memory too (the round-2 SASS had an LDL / STL pair around every push).
    uint2 *const stack_sm = sm_stack + threadIdx.x;
    uint2 stack_spill[CRT_STACK_SIZE - kSmemStack];
    int sp = 0;
    TravState st;
    uint2 tri = make_uint2(0u, 0u);  // triangle group yielded by this lane's last node step
    TraversalCounters cnt, cnt_any;
    bool alive = false;
    bool is_any = false;  // kind of the ray this lane currently holds
    uint32_t out_index = 0;
    uint32_t batch_next = 0, batch_end = 0;  // warp-uniform
    bool drained = false;                    // warp-uniform: the queue has no more rays
    uint32_t cursor_base = 0;                // warp-uniform: value of sm_cursor[warp] before the current pass
    if (lane == 0) {
        sm_cursor[warp] = 0u;
    }
    __syncwarp();

    for (;;) {
        // ---- refill idle lanes ----
        unsigned need = __ballot_sync(0xffffffffu, !alive);
        while (need && !drained) {
            if (batch_next == batch_end) {
                uint32_t b = 0;
                if (lane == 0) {
                    b = atomicAdd(work_counter, batch);
                }
                b = __shfl_sync(0xffffffffu, b, 0);
                if (b >= count) {
                    drained = true;
                    break;
                }
                batch_next = b;
                batch_end = min(b + batch, count);
            }
            const uint32_t avail = batch_end - batch_next;
            const uint32_t r = (uint32_t)__popc(need & lanemask_lt);
            if (((need >> lane) & 1u) && r < avail) {
                const uint32_t j = batch_next + r;
                Ray ray;
                is_any = j < n_any;
                if (is_any) {
                    const float4 o = ps.sray_o[j], d = ps.sray_d[j];
                    ray = Ray{o.x, o.y, o.z, kEpsilon, d.x, d.y, d.z, o.w};
                    out_index = __float_as_uint(d.w);
                } else {
                    out_index = queue ? queue[j - n_any] : j - n_any;
                    const float4 o = ps.ray_o[out_index], d = ps.ray_d[out_index];
                    ray = Ray{o.x, o.y, o.z, o.w, d.x, d.y, d.z, d.w};
                }
                trav_init(st, ray, sc.float_one);
                if (is_any && any_far_first) {
                    trav_reverse_order(st);  // same answer, different order (bvh8_traverse.h)
                }
                sp = 0;
                tri = make_uint2(0u, 0u);
                alive = true;
                {
                    sm_ray[warp][0][lane] = ray.ox;
                    sm_ray[warp][1][lane] = ray.oy;
                    sm_ray[warp][2][lane] = ray.oz;
                    sm_ray[warp][3][lane] = ray.tnear;
                    sm_ray[warp][4][lane] = ray.dx;
                    sm_ray[warp][5][lane] = ray.dy;
                    sm_ray[warp][6][lane] = ray.dz;
                    sm_ray[warp][7][lane] = ray.tfar;
                    sm_key[warp][lane] = ((unsigned long long)hit_key(ray.tfar) << 32) | 0xffffffffull;
                    sm_hit[warp][lane] = make_float4(0.f, 0.f, __uint_as_float(kMiss), ray.tfar);
                    if (COUNT) {
                        sm_is_any[warp][lane] = is_any ? 1u : 0u;
                    }
                }
            }
            batch_next += min((uint32_t)__popc(need), avail);
            need = __ballot_sync(0xffffffffu, !alive);
        }
        if (__ballot_sync(0xffffffffu, alive) == 0u) {
            break;
        }
        // ---- advance all live lanes until enough of them have finished ----
        // Each iteration has a node phase and a triangle phase so that the lanes of a warp execute
        // the same code together; the triangles a node step yields are tested in the same iteration
        // (a per-lane postponement after Ylitie et al. 2017 §5.3 was measured and dropped, DESIGN.md §2).
        // The closest hit does not depend on the order of the tests (ties break on the primitive id).
        {
            // Warp-cooperative triangle tests. The first profiles showed the per-lane triangle loops issuing
            // half of all instructions at 3-8 active lanes. Here the node phase stays per lane, but
            // the triangles it yields are pooled across the warp: (owner lane, triangle) pairs are
            // packed into 32 slots and EVERY lane tests one pair, reading the owner's ray from shared
            // memory and merging hits with a 64-bit atomicMin on (t, flat primitive id) — the same
            // closest-hit / tie rule as the sequential test, so results are unchanged.
            __syncwarp();
            for (;;) {
                // node phase
                const bool can_step = alive && (st.cur.y & 0xff000000u) && (DEFER == 0 || tri.y == 0u);
                CRT_PROF_NODE_PHASE(can_step);
                if (can_step) {
                    const uint32_t node_index = next_child(st.cur, st.oct_inv4);
                    if (st.cur.y & 0xff000000u) {
                        if (sp < kSmemStack) {
                            stack_sm[sp * kTravBlock] = st.cur;
                        } else {
                            stack_spill[sp - kSmemStack] = st.cur;
                        }
                        ++sp;
                    }
                    if (COUNT) {
                        if (is_any) {
                            cnt_any.nodes++;
                        } else {
                            cnt.nodes++;
                        }
                    }
                    if (TOP) {  // (only the five loads differ: the test itself must not be duplicated into two divergent paths)
                        float4 n0, n1, n2, n3, n4;
                        if (node_index < top_nodes) {
                            const float4 *np = sm_top + node_index * 5u;
                            n0 = np[0], n1 = np[1], n2 = np[2], n3 = np[3], n4 = np[4];
                        } else {
                            const float4 *np = sc.nodes + (size_t)node_index * 5;
                            n0 = np[0], n1 = np[1], n2 = np[2], n3 = np[3], n4 = np[4];
                        }
                        node_intersect_loaded(n0, n1, n2, n3, n4, st, st.cur, tri);
                    } else {
                        node_intersect(sc.nodes, st, node_index, st.cur, tri);
                    }
                }
                // triangle phase: the pairs (owner lane, triangle) of this step, 32 per pass. Slots are PULLED by the
                // testing lanes: an owner only claims a range of slots (one shared-memory atomicAdd on a running
                // cursor: no scan over the lanes) and marks where it starts; slot lane p finds the last start at or
                // before p, reads the owner's group by shuffle and picks its (p - start)-th triangle. (Round 1 had the
                // owners write one slot per pair in a loop: 5 trips per pass at 3 active lanes, 12 % of the kernel's
                // issued instructions with the scan that placed them.)
                for (;;) {
                    const uint32_t k = alive ? (uint32_t)__popc(tri.y) : 0u;
                    const uint32_t total = __reduce_add_sync(0xffffffffu, k);
                    if (total == 0u) {
                        break;
                    }
                    if (DEFER > 0) {
                        // wait for a fuller pool while some lane without a pending group can still descend
                        const bool free_lane = alive && tri.y == 0u && ((st.cur.y & 0xff000000u) || sp > 0);
                        if (total < (uint32_t)DEFER && __ballot_sync(0xffffffffu, free_lane) != 0u) {
                            break;
                        }
                    }
                    uint32_t start = 32u;  // first slot of this lane's pairs (any order among the owners)
                    if (k != 0u) {
                        start = atomicAdd(&sm_cursor[warp], k) - cursor_base;
                        if (start < 32u) {
                            sm_owner[warp][start] = (uint32_t)lane;
                        }
                    }
                    cursor_base += total;
                    const uint32_t starts = __reduce_or_sync(0xffffffffu, start < 32u ? 1u << start : 0u);
                    __syncwarp();
                    const uint32_t npairs = min(total, 32u);
                    CRT_PROF_TRI_PASS((uint32_t)lane < npairs);
                    uint32_t owner = 0u, rank = 0u;
                    if ((uint32_t)lane < npairs) {
                        const uint32_t s0 = (uint32_t)msb(starts & (0xffffffffu >> (31 - lane)));  // slot 0 is always a start
                        owner = sm_owner[warp][s0];
                        rank = (uint32_t)lane - s0;
                    }
                    const uint32_t gx = __shfl_sync(0xffffffffu, tri.x, (int)owner);
                    uint32_t gy = __shfl_sync(0xffffffffu, tri.y, (int)owner);
                    // the owner's pairs that fit into this pass are consumed: its highest min(k, 32 - start) bits
                    if (k != 0u) {
                        const uint32_t fit = start < 32u ? min(k, 32u - start) : 0u;
                        if (fit == k) {
                            tri.y = 0u;
                        } else {
#pragma unroll 1
                            for (uint32_t i = 0; i < fit; ++i) {
                                tri.y ^= 1u << msb(tri.y);
                            }
                        }
                    }
                    bool won = false;
                    unsigned long long cand = 0ull;
                    uint32_t tri_index = 0u;
                    float hu = 0.f, hv = 0.f, t = 0.f;
                    if ((uint32_t)lane < npairs) {
                        // the rank-th highest set bit of the group: two predicated steps cover a leaf (<= 3 triangles)
                        uint32_t skip = rank;
#pragma unroll
                        for (int u = 0; u < 2; ++u) {
                            if (skip) {
                                gy ^= 1u << msb(gy);
                                --skip;
                            }
                        }
#pragma unroll 1
                        while (skip) {
                            gy ^= 1u << msb(gy);
                            --skip;
                        }
                        tri_index = gx + (uint32_t)msb(gy);
                        if (COUNT) {  // attribute the test to the kind of the owner's ray
                            if (sm_is_any[warp][owner]) {
                                cnt_any.tris++;
                            } else {
                                cnt.tris++;
                            }
                        }
                        Ray r;
                        r.ox = sm_ray[warp][0][owner];
                        r.oy = sm_ray[warp][1][owner];
                        r.oz = sm_ray[warp][2][owner];
                        r.tnear = sm_ray[warp][3][owner];
                        r.dx = sm_ray[warp][4][owner];
                        r.dy = sm_ray[warp][5][owner];
                        r.dz = sm_ray[warp][6][owner];
                        r.tfar = sm_ray[warp][7][owner];
                        const float4 *tp = sc.tris + (size_t)tri_index * 3;
                        const float4 t0 = tp[0], t1 = tp[1], t2 = tp[2];
                        if (tri_test(r, r.tfar, t0, t1, t2, t, hu, hv)) {
                            cand = ((unsigned long long)hit_key(t) << 32) | (unsigned long long)__float_as_uint(t0.w);
                            won = atomicMin(&sm_key[warp][owner], cand) > cand;
                        }
                    }
                    __syncwarp();
                    if (won && sm_key[warp][owner] == cand) {  // the pair that holds the minimum records u, v and its own t (-0 or +0)
                        sm_hit[warp][owner] = make_float4(hu, hv, __uint_as_float(tri_index), t);
                    }
                    __syncwarp();
                    if (total <= 32u) {
                        break;
                    }
                }
                // refresh tfar, pop, finish
                if (alive) {
                    st.tfar = hit_key_t((uint32_t)(sm_key[warp][lane] >> 32));
                    bool finished = is_any && __float_as_uint(sm_hit[warp][lane].z) != kMiss;
                    if (DEFER > 0 && finished) {
                        tri.y = 0u;  // an occluded shadow ray needs no further tests
                    }
                    if (!finished && (DEFER == 0 || tri.y == 0u) && (st.cur.y & 0xff000000u) == 0u) {
                        if (sp > 0) {
                            --sp;
                            st.cur = sp < kSmemStack ? stack_sm[sp * kTravBlock] : stack_spill[sp - kSmemStack];
                        } else {
                            finished = true;
                        }
                    }
                    if (finished) {
                        const float4 best = sm_hit[warp][lane];
                        const uint32_t htri = __float_as_uint(best.z);
                        if (is_any) {
                            ps.vis[out_index] = htri != kMiss ? 0 : 1;
                        } else {
                            ps.hit[out_index] = make_float4(best.w, htri != kMiss ? best.x : 0.f, htri != kMiss ? best.y : 0.f,
                                                            __uint_as_float(htri));
                        }
                        alive = false;
                    }
                }
                const int n_alive = __popc(__ballot_sync(0xffffffffu, alive));
                if (n_alive == 0 || (!drained && 32 - n_alive >= refill_idle)) {
                    break;
                }
            }
        }
    }
    if (COUNT) {
        unsigned long long n = cnt.nodes, t = cnt.tris, na = cnt_any.nodes, ta = cnt_any.tris;
        for (int off = 16; off > 0; off >>= 1) {
            n += __shfl_down_sync(0xffffffffu, n, off);
            t += __shfl_down_sync(0xffffffffu, t, off);
            na += __shfl_down_sync(0xffffffffu, na, off);
            ta += __shfl_down_sync(0xffffffffu, ta, off);
        }
        if (lane == 0) {
            atomicAdd(ps.trav_counters, n);
            atomicAdd(ps.trav_counters + 1, t);
            atomicAdd(ps.trav_counters + 2, na);
            atomicAdd(ps.trav_counters + 3, ta);
        }
    }
}

// ---------------------------------------------------------------------------------------
// 80 registers (6 blocks of 128 per SM) with the three BSDF evaluations inlined measured fastest:
// 3.19 ms/frame -> 2.67 ms on C2 against 4 blocks x 106 registers with out-of-line BSDF calls
// (inlining lets the compiler share sub-expressions between disney_pdf and disney_brdf; measured on an earlier GPU).
// With one texture-fetch site for the scalar parameters (unpack_material) the kernel is 7,944 SASS instructions instead
// of 12,800, and with the shadow rays and NEE terms stored as soon as they are known it spills 4 B instead of 120 B.
// k_shade's time per C2 frame, all four builds in one run on one H100 SXM (torch.profiler, scripts/profile_frame_launches.py):
// 3.21 ms before; 2.44 ms at (128, 6) = 80 registers; 2.57 ms at (128, 7) = 72 registers (52 B spilled); 2.85 ms at
// (128, 8) = 64 registers (140 B spilled). More resident warps do not pay for the spills, so the bounds stay at (128, 6).
// (A grid-stride form for the thin queues of the late bounces was measured in round 2 and dropped: those launches take
// ~49 us whatever the grid, and ncu shows why — 12 no-instruction stalls per issued instruction: a warp's first walk
// through this kernel's ~4000 executed instructions is a chain of instruction-cache misses.)
template <bool HWTEX>  // option "hw_textures": texels through cudaTextureObject_t (shade_math.cuh: TexSource)
__global__ void __launch_bounds__(128, 6) k_shade(DeviceScene sc, PathState ps, const uint32_t *queue_in,
                                               uint32_t *queue_out, int bounce, int max_depth)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t count = ps.counters[kCntQueue + bounce];
    bool emit_a = false, emit_b = false, emit_next = false;
    uint32_t slot = 0;
    float3 hit_p = mk3(0.f), dir_a = mk3(0.f), dir_b = mk3(0.f);
    float dist_a = 0.f, dist_b = 0.f;
    // what the continuation needs of a path that hit something
    bool shaded = false;
    uint32_t rng = 0u;
    float3 path_throughput = mk3(0.f), w_o = mk3(0.f), normal = mk3(0.f), v_x = mk3(0.f), v_y = mk3(0.f);
    DisneyMaterial mat{};
    if (j < count) {
        slot = queue_in[j];
        const float4 ro = ps.ray_o[slot], rd = ps.ray_d[slot], h = ps.hit[slot], tr = ps.thr_rng[slot];
        path_throughput = mk3(tr.x, tr.y, tr.z);
        rng = __float_as_uint(tr.w);
        const uint32_t tri = __float_as_uint(h.w);
        const float3 dir = mk3(rd.x, rd.y, rd.z);
        w_o = neg(dir);
        if (tri == kMiss) {
            // render_embree.ispc:258-262: illum += path_throughput * miss_shader(dir). The environment lookup (atan2f, acosf:
            // ~200 instructions that a warp here would execute for its ~6 missing lanes) is left to k_nee_resolve, which adds
            // this bounce's term to the path's radiance anyway and is memory-bound with issue slots to spare: flags = 4
            // ("missed": no NEE; k_nee_resolve must not look at hit[], which the merged traversal launch overwrites with
            // the NEXT bounce's hit before it runs — the ray direction in ray_d[slot] stays, a path that missed does not
            // continue). Same position in the path's sum as before, so the same bits.
            ps.nee_T[slot] = make_float4(path_throughput.x, path_throughput.y, path_throughput.z, __uint_as_float(4u));
        } else {
            // render_embree.ispc:264-293 (the ray-independent part was precomputed per triangle)
            shaded = true;
            hit_p = mk3(ro.x + h.x * dir.x, ro.y + h.x * dir.y, ro.z + h.x * dir.z);
            const float4 s0 = __ldg(sc.shade + 3 * (size_t)tri), s1 = __ldg(sc.shade + 3 * (size_t)tri + 1),
                         s2 = __ldg(sc.shade + 3 * (size_t)tri + 2);
            normal = mk3(s0.x, s0.y, s0.z);
            const uint32_t material_id = __float_as_uint(s0.w);
            float2 uv = make_float2(0.f, 0.f);
            if (__float_as_uint(s2.z) != 0u) {
                const float bw = 1.f - h.y - h.z;
                uv.x = s1.x * bw + s1.z * h.y + s2.x * h.z;
                uv.y = s1.y * bw + s1.w * h.y + s2.y * h.z;
            }
            const TexSource tex_source{sc.texels, sc.tex, sc.tex_objects};
            unpack_material<HWTEX>(mat, sc.materials, material_id, uv, tex_source);
            // render_embree.ispc:296-300
            if (mat.specular_transmission == 0.f && dot(w_o, normal) < 0.f) {
                normal = neg(normal);
            }
            ortho_basis(v_x, v_y, normal);

            // ---- sample_direct_light, render_embree.ispc:105-181 ----
            bool has_l1 = false;
            {
                uint32_t light_id = (uint32_t)(lcg_randomf(rng) * (float)sc.num_lights);
                light_id = min(light_id, sc.num_lights - 1u);
                {
                    const QuadLight light = load_light(sc.lights, light_id);
                    const float sx = lcg_randomf(rng);
                    const float sy = lcg_randomf(rng);
                    const float3 light_pos = sample_quad_light_position(light, sx, sy);
                    float3 light_dir = light_pos - hit_p;
                    const float light_dist = length(light_dir);
                    light_dir = normalize(light_dir);
                    const float light_pdf = quad_light_pdf(light, light_pos, light_dir);
                    const float bsdf_pdf = disney_pdf(mat, normal, w_o, light_dir, v_x, v_y);
                    // the reference traces (and counts) this shadow ray before the pdf tests
                    emit_a = true;
                    dir_a = light_dir;
                    dist_a = light_dist;
                    if (light_pdf >= kEpsilon && bsdf_pdf >= kEpsilon) {
                        const float3 bsdf = disney_brdf(mat, normal, w_o, light_dir, v_x, v_y);
                        const float w = power_heuristic(1.f, light_pdf, 1.f, bsdf_pdf);
                        const float3 l1 = bsdf * light.emission * fabsf(dot(light_dir, normal)) * w / light_pdf;
                        ps.nee_l1[slot] = make_float4(l1.x, l1.y, l1.z, 0.f);
                        has_l1 = true;
                    }
                }
                {
                    float3 w_i;
                    float bsdf_pdf;
                    const float3 bsdf = sample_disney_brdf(mat, normal, w_o, v_x, v_y, rng, w_i, bsdf_pdf);
                    // the light again (L1-resident): not live across the sampling
                    const QuadLight light = load_light(sc.lights, light_id);
                    float light_dist;
                    float3 light_pos;
                    if (!all_zero(bsdf) && bsdf_pdf >= kEpsilon &&
                        quad_intersect(light, hit_p, w_i, light_dist, light_pos)) {
                        const float light_pdf = quad_light_pdf(light, light_pos, w_i);
                        if (light_pdf >= kEpsilon) {
                            const float w = power_heuristic(1.f, bsdf_pdf, 1.f, light_pdf);
                            emit_b = true;
                            dir_b = w_i;
                            dist_b = light_dist;
                            const float3 l2 = bsdf * light.emission * fabsf(dot(w_i, normal)) * w / bsdf_pdf;
                            ps.nee_l2[slot] = make_float4(l2.x, l2.y, l2.z, 0.f);
                        }
                    }
                }
            }
            // bit 1: valid, bit 0: has ray B, bit 3: has a light-sample term. Many light samples fail the pdf tests
            // (about 42 %, DESIGN.md §2): their shadow ray is still traced and counted, but no zero term is stored or read back.
            ps.nee_T[slot] = make_float4(path_throughput.x, path_throughput.y, path_throughput.z,
                                         __uint_as_float(2u | (emit_b ? 1u : 0u) | (has_l1 ? 8u : 0u)));
        }
    }
    // ---- compaction: one atomic per warp per queue. The shadow rays are stored before the continuation is sampled,
    // so that their directions and lengths are not live across it (fewer registers; same queues, same image). ----
    const uint32_t ia = warp_append(ps.counters + kCntShadow + bounce, emit_a);
    if (emit_a) {
        ps.sray_o[ia] = make_float4(hit_p.x, hit_p.y, hit_p.z, dist_a);
        ps.sray_d[ia] = make_float4(dir_a.x, dir_a.y, dir_a.z, __uint_as_float(slot * 2u));
    }
    const uint32_t ib = warp_append(ps.counters + kCntShadow + bounce, emit_b);
    if (emit_b) {
        ps.sray_o[ib] = make_float4(hit_p.x, hit_p.y, hit_p.z, dist_b);
        ps.sray_d[ib] = make_float4(dir_b.x, dir_b.y, dir_b.z, __uint_as_float(slot * 2u + 1u));
    }
    // ---- continuation, render_embree.ispc:313-336 ----
    if (shaded) {
        float pdf;
        float3 w_i;
        const float3 bsdf = sample_disney_brdf(mat, normal, w_o, v_x, v_y, rng, w_i, pdf);
        if (!(pdf == 0.f || all_zero(bsdf))) {
            path_throughput = path_throughput * bsdf * fabsf(dot(w_i, normal)) / pdf;
            const int nb = bounce + 1;
            bool alive = true;
            if (nb > 3) {
                const float q = fmaxf(0.05f, 1.f - fmaxf(path_throughput.x, fmaxf(path_throughput.y, path_throughput.z)));
                if (lcg_randomf(rng) < q) {
                    alive = false;
                } else {
                    path_throughput = path_throughput / (1.f - q);
                }
            }
            if (alive && nb < max_depth) {
                emit_next = true;
                ps.ray_o[slot] = make_float4(hit_p.x, hit_p.y, hit_p.z, kEpsilon);
                ps.ray_d[slot] = make_float4(w_i.x, w_i.y, w_i.z, 1e20f);
                ps.thr_rng[slot] = make_float4(path_throughput.x, path_throughput.y, path_throughput.z, __uint_as_float(rng));
            }
        }
    }
    const uint32_t in = warp_append(ps.counters + kCntQueue + bounce + 1, emit_next);
    if (emit_next) {
        queue_out[in] = slot;
    }
}

// ---- option "shade_sort" (off by default): the shade queue bucketed by material id ----
// A stable one-pass counting sort of queue_in on the material of each path's hit, so that the lanes of a k_shade warp
// unpack the same material, sample the same textures and run the same BSDF lobes. 256 buckets: material ids 0..253 their
// own, every id >= 254 shares bucket 254, paths that missed are bucket 255. The image does not depend on the order of
// a queue (fixed accumulation order, DESIGN.md section 2), so frames are bit-identical with and without the sort.
// The queue length lives on the device: the grids cover the queue's capacity and tiles beyond the length count zero.
// k_queue_hist -> exclusive scan of hist (digit-major: one scan yields every (bucket, tile) offset) -> k_queue_scatter.
constexpr int kSortBlock = 256, kSortItems = 8, kSortTile = kSortBlock * kSortItems;

__device__ __forceinline__ uint32_t shade_bucket(const DeviceScene &sc, const PathState &ps, uint32_t slot)
{
    const uint32_t tri = __float_as_uint(reinterpret_cast<const float *>(ps.hit + slot)[3]);
    if (tri == kMiss) {
        return 255u;
    }
    const uint32_t material_id = __float_as_uint(reinterpret_cast<const float *>(sc.shade + 3 * (size_t)tri)[3]);
    return material_id < 254u ? material_id : 254u;
}

template <int BUCKETS>  // 256 (a template so that the one-thread host build of this header never sees its barriers)
__global__ void __launch_bounds__(kSortBlock) k_queue_hist(DeviceScene sc, PathState ps, const uint32_t *queue_in, int bounce,
                                                           uint32_t *hist, uint32_t num_tiles)
{
    static_assert(BUCKETS == kSortBlock, "one thread per bucket");
    __shared__ uint32_t h[BUCKETS];
    const uint32_t n = ps.counters[kCntQueue + bounce];
    h[threadIdx.x] = 0u;
    __syncthreads();
    const uint32_t base = blockIdx.x * (uint32_t)kSortTile;
    for (int k = 0; k < kSortItems; ++k) {
        const uint32_t i = base + (uint32_t)k * kSortBlock + threadIdx.x;
        if (i < n) {
            atomicAdd(&h[shade_bucket(sc, ps, queue_in[i])], 1u);
        }
    }
    __syncthreads();
    hist[threadIdx.x * num_tiles + blockIdx.x] = h[threadIdx.x];
}

// block = one tile of 2048 queue entries, warp w = entries [w * 256, w * 256 + 256) of it, 8 rounds of 32. An entry's
// rank among the equal buckets of its tile: earlier warps, then earlier rounds, then lower lanes (stable).
template <int BUCKETS>
__global__ void __launch_bounds__(kSortBlock) k_queue_scatter(DeviceScene sc, PathState ps, const uint32_t *queue_in,
                                                              uint32_t *queue_sorted, int bounce, const uint32_t *hist_scanned,
                                                              uint32_t num_tiles)
{
    __shared__ uint32_t cnt[kSortBlock / 32][BUCKETS];
    __shared__ uint32_t goff[BUCKETS];
    const uint32_t n = ps.counters[kCntQueue + bounce];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned lanemask_lt = (1u << lane) - 1u;
    for (int w = 0; w < kSortBlock / 32; ++w) {
        cnt[w][threadIdx.x] = 0u;
    }
    goff[threadIdx.x] = hist_scanned[threadIdx.x * num_tiles + blockIdx.x];
    __syncthreads();
    const uint32_t base = blockIdx.x * (uint32_t)kSortTile + (uint32_t)warp * 256u;
    uint32_t slot[kSortItems], where[kSortItems];  // where = bucket << 16 | rank within (warp, bucket)
    for (int r = 0; r < kSortItems; ++r) {
        const uint32_t i = base + (uint32_t)r * 32u + lane;
        const bool valid = i < n;
        slot[r] = valid ? queue_in[i] : 0u;
        const uint32_t d = valid ? shade_bucket(sc, ps, slot[r]) : (uint32_t)BUCKETS;
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const int leader = __ffs(peers) - 1;
        uint32_t before = 0u;
        if (lane == leader && valid) {
            before = cnt[warp][d];
            cnt[warp][d] = before + (uint32_t)__popc(peers);
        }
        before = __shfl_sync(0xffffffffu, before, leader);
        where[r] = (d << 16) | (before + (uint32_t)__popc(peers & lanemask_lt));
        __syncwarp();
    }
    __syncthreads();
    {   // per bucket: exclusive prefix of the warps' counts
        uint32_t run = 0u;
        for (int w = 0; w < kSortBlock / 32; ++w) {
            const uint32_t c = cnt[w][threadIdx.x];
            cnt[w][threadIdx.x] = run;
            run += c;
        }
    }
    __syncthreads();
    for (int r = 0; r < kSortItems; ++r) {
        const uint32_t i = base + (uint32_t)r * 32u + lane;
        if (i < n) {
            const uint32_t d = where[r] >> 16;
            queue_sorted[goff[d] + cnt[warp][d] + (where[r] & 0xffffu)] = slot[r];
        }
    }
}

// illum = illum + path_throughput * (L1 [if unoccluded] + L2 [if traced and unoccluded])
__global__ void __launch_bounds__(256) k_nee_resolve(PathState ps, const uint32_t *queue_in, int bounce)
{
    const uint32_t count = ps.counters[kCntQueue + bounce];
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < count; j += gridDim.x * blockDim.x) {  // grid-stride, as k_shade
    const uint32_t slot = queue_in[j];
    const float4 T = ps.nee_T[slot];
    if (__float_as_uint(T.w) & 4u) {
        // the path left the scene at this bounce (render_embree.ispc:258-262; deferred here by k_shade)
        const float4 rd = ps.ray_d[slot];
        float4 rad = ps.radiance[slot];
        const float3 c = mk3(T.x, T.y, T.z) * miss_shader(mk3(rd.x, rd.y, rd.z));
        rad.x = rad.x + c.x;
        rad.y = rad.y + c.y;
        rad.z = rad.z + c.z;
        ps.radiance[slot] = rad;
        continue;
    }
    float3 illum = mk3(0.f);
    if ((__float_as_uint(T.w) & 8u) && ps.vis[2 * slot]) {
        const float4 l1 = ps.nee_l1[slot];
        illum = mk3(l1.x, l1.y, l1.z);
    }
    if (__float_as_uint(T.w) & 1u) {
        if (ps.vis[2 * slot + 1]) {
            const float4 l2 = ps.nee_l2[slot];
            illum = illum + mk3(l2.x, l2.y, l2.z);
        }
    }
    float4 rad = ps.radiance[slot];
    rad.x = rad.x + T.x * illum.x;
    rad.y = rad.y + T.y * illum.y;
    rad.z = rad.z + T.z * illum.z;
    ps.radiance[slot] = rad;
    }
}

// ---- frame completion flags over peer memory (multi-GPU frames written by every rank's k_resolve, DESIGN.md §6) ----
// The assembling rank's full-frame image buffer ends with kSyncWords words that every rank can reach through the same
// peer mapping as the pixels: word [r] = the last frame sequence number rank r has completely stored into this frame
// (written by rank r's k_resolve: its last block to finish, after a system-scope fence, with a release store);
// word [kSyncConsumed] = the last sequence number the assembling rank is done with (it sets it when it starts its
// next frame; a peer's k_resolve of frame s + 1 waits for it, so it cannot overwrite frame s under a reader).
// No collective library and no host thread is involved in the exchange: the stores ARE the transfer, the flags the barrier.
constexpr uint32_t kSyncWords = 64;
constexpr uint32_t kSyncConsumed = 32;
constexpr unsigned long long kSyncTimeoutNs = 20ull * 1000ull * 1000ull * 1000ull;

__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t *p)
{
#if defined(__CUDA_ARCH__)
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
#else
    return __atomic_load_n(p, __ATOMIC_ACQUIRE);
#endif
}
__device__ __forceinline__ void st_release_sys(uint32_t *p, uint32_t v)
{
#if defined(__CUDA_ARCH__)
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
#else
    __atomic_store_n(p, v, __ATOMIC_RELEASE);
#endif
}
__device__ __forceinline__ unsigned long long sync_clock_ns()
{
#if defined(__CUDA_ARCH__)
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
#elif defined(__CUDACC__)
    return 0ull;  // (nvcc's host pass; never called)
#else
    return crt_host_clock_ns();  // the test-only host builds of this header
#endif
}
// lane i < n (i != skip) waits until words[i] has reached `need` (sequence numbers: wrap-safe signed distance).
// A flag that does not arrive within kSyncTimeoutNs sets *err (a mapped host word) instead of hanging the GPU.
__global__ void __launch_bounds__(32) k_wait_words(const uint32_t *words, uint32_t n, uint32_t skip, uint32_t need, uint32_t *err)
{
    const uint32_t i = threadIdx.x;
    if (i >= n || i == skip) {
        return;
    }
    const unsigned long long t0 = sync_clock_ns();
    while ((int32_t)(ld_acquire_sys(words + i) - need) < 0) {
        if (sync_clock_ns() - t0 > kSyncTimeoutNs) {
            *err = 1u + i;
            return;
        }
    }
}
__global__ void __launch_bounds__(32) k_set_word(uint32_t *word, uint32_t v)
{
    if (threadIdx.x == 0) {
        st_release_sys(word, v);
    }
}

// k_resolve's running mean: (x + n * acc) / (n + 1) for the frame with frame_id n
CRT_D float aov_running_mean(float x, float acc, uint32_t n)
{
    return (x + (float)n * acc) / (float)(n + 1u);
}

// render_embree.ispc:339-353 (sample mean + running mean) and :358-370 (sRGB8)
// ADAPTIVE: each block folds its n_b frames with its own count c_b in place of frame_id, and the luminance moments with
// them (k_aov_moments' fold); a block with n_b = 0 leaves every buffer of its pixels untouched.
template <bool ADAPTIVE = false>
__global__ void __launch_bounds__(256) k_resolve(FrameLayout f, PathState ps, uint32_t frame_id, float *accum_local,
                                                uint32_t *img_local, float *accum_full, uint32_t *img_full,
                                                uint32_t *done_counter, uint32_t *arrive_word, uint32_t seq,
                                                AdaptiveFrame ad = AdaptiveFrame{})
{
    const uint32_t lp = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t x, y;
    uint32_t first = frame_id, frames = f.frames;
    if (ADAPTIVE && lp < f.npx_local) {
        const uint2 sel = ad.sel[lp >> 5];
        first = sel.x;
        frames = sel.y;
    }
    if (lp < f.npx_local && (!ADAPTIVE || frames != 0u) && local_pixel_coords(f, lp, x, y)) {
        // the frames of the batch are folded into the running mean one after the other, exactly as if
        // they had been rendered by separate calls
        float3 illum = mk3(accum_local[3 * (size_t)lp], accum_local[3 * (size_t)lp + 1], accum_local[3 * (size_t)lp + 2]);
        float2 m = ADAPTIVE ? ad.moments[lp] : make_float2(0.f, 0.f);
        for (uint32_t k = 0; k < frames; ++k) {
            const float3 accum = illum;
            illum = mk3(0.f);
            float s1 = 0.f, s2 = 0.f;
            for (uint32_t s = 0; s < f.spp; ++s) {
                const float4 r = ps.radiance[(size_t)(k * f.spp + s) * f.npx_local + lp];
                illum = illum + mk3(r.x, r.y, r.z);
                if (ADAPTIVE) {
                    const float l = luminance(mk3(r.x, r.y, r.z));
                    s1 += l;
                    s2 += l * l;
                }
            }
            illum = illum / (float)f.spp;
            illum = (illum + (float)(first + k) * accum) / (float)(first + k + 1u);
            if (ADAPTIVE) {
                m.x = aov_running_mean(s1 / (float)f.spp, m.x, first + k - ad.stat_base);
                m.y = aov_running_mean(s2 / (float)f.spp, m.y, first + k - ad.stat_base);
            }
        }
        if (ADAPTIVE) {
            ad.moments[lp] = m;
        }
        accum_local[3 * (size_t)lp] = illum.x;
        accum_local[3 * (size_t)lp + 1] = illum.y;
        accum_local[3 * (size_t)lp + 2] = illum.z;
        const uint32_t rgba = float_to_srgb8(illum.x) | (float_to_srgb8(illum.y) << 8) | (float_to_srgb8(illum.z) << 16) |
                              0xff000000u;
        img_local[lp] = rgba;
        if (accum_full) {
            const size_t p = (size_t)y * f.fb_w + x;
            accum_full[3 * p] = illum.x;
            accum_full[3 * p + 1] = illum.y;
            accum_full[3 * p + 2] = illum.z;
            img_full[p] = rgba;
        }
    }
    // Peer-written frame: the block that finishes LAST publishes "this rank has stored frame `seq`" to the assembling
    // rank (every block fences its pixel stores at system scope before it takes a ticket).
    if (arrive_word) {
        __threadfence_system();
        __syncthreads();
        if (threadIdx.x == 0) {
            if (atomicAdd(done_counter, 1u) == gridDim.x - 1u) {
                *done_counter = 0u;
                st_release_sys(arrive_word, seq);
            }
        }
    }
}

// k_resolve for every view of the table, one thread per (view, local pixel): view v folds its frames with b_v in place of
// frame_id, into its local slots lp = v * npx_local + lp_v and its full frame at offset v * fb_w * fb_h.
__global__ void __launch_bounds__(256) k_resolve_views(const __grid_constant__ ViewTable views, FrameLayout f, PathState ps,
                                                      float *accum_local, uint32_t *img_local, float *accum_full,
                                                      uint32_t *img_full)
{
    const uint32_t lp = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t npx_all = f.npx_local * views.num_views;
    uint32_t x, y;
    if (lp >= npx_all || !local_pixel_coords(f, lp % f.npx_local, x, y)) {
        return;
    }
    const uint32_t v = lp / f.npx_local, first = views.view[v].frame_id;
    float3 illum = mk3(accum_local[3 * (size_t)lp], accum_local[3 * (size_t)lp + 1], accum_local[3 * (size_t)lp + 2]);
    for (uint32_t k = 0; k < f.frames; ++k) {
        const float3 accum = illum;
        illum = mk3(0.f);
        for (uint32_t s = 0; s < f.spp; ++s) {
            const float4 r = ps.radiance[(size_t)(k * f.spp + s) * npx_all + lp];
            illum = illum + mk3(r.x, r.y, r.z);
        }
        illum = illum / (float)f.spp;
        illum = (illum + (float)(first + k) * accum) / (float)(first + k + 1u);
    }
    accum_local[3 * (size_t)lp] = illum.x;
    accum_local[3 * (size_t)lp + 1] = illum.y;
    accum_local[3 * (size_t)lp + 2] = illum.z;
    const uint32_t rgba = float_to_srgb8(illum.x) | (float_to_srgb8(illum.y) << 8) | (float_to_srgb8(illum.z) << 16) |
                          0xff000000u;
    img_local[lp] = rgba;
    const size_t p = (size_t)v * f.fb_w * f.fb_h + (size_t)y * f.fb_w + x;
    accum_full[3 * p] = illum.x;
    accum_full[3 * p + 1] = illum.y;
    accum_full[3 * p + 2] = illum.z;
    img_full[p] = rgba;
}

// Scatter another rank's tile-local buffers into the full frame (frame-end gather, §8e)
__global__ void __launch_bounds__(256) k_assemble(FrameLayout f, const float *accum_local, const uint32_t *img_local,
                                                 float *accum_full, uint32_t *img_full)
{
    const uint32_t lp = blockIdx.x * blockDim.x + threadIdx.x;
    if (lp >= f.npx_local) {
        return;
    }
    uint32_t x, y;
    if (!local_pixel_coords(f, lp, x, y)) {
        return;
    }
    const size_t p = (size_t)y * f.fb_w + x;
    accum_full[3 * p] = accum_local[3 * (size_t)lp];
    accum_full[3 * p + 1] = accum_local[3 * (size_t)lp + 1];
    accum_full[3 * p + 2] = accum_local[3 * (size_t)lp + 2];
    img_full[p] = img_local[lp];
}

}  // namespace crt
