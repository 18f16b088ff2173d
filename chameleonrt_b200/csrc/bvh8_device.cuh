// bvh8_device.cuh — set_scene ON THE DEVICE: flattening + the BVH8 of bvh8.h (option "bvh_builder" = 1 / 2;
// SURVEY.md §8(f) rank 1). Opt-in; verified under the CPU SIMT emulation (tests/simt_emu) and on the GPU (tests/test_z_new_gpu_paths.py: frames bit-identical to the host-built tree's; tests/test_full_size_parity.py: against the oracle at full scene size).
//
// Replaces, like bvh8_build.cpp, what the reference delegates to Embree / OptiX (rtcCommitScene,
// backends/embree/embree_utils.cpp:75,128; optixAccelBuild + compaction, backends/optix/optix_utils.cpp:183-245).
// The host builder (binned SAH) stays the default: it makes the better tree; these make set_scene fast —
// streaming passes over the triangles instead of seconds of host work on C3 / C4 / C5.
//
//   0. k_flatten         instances -> one world-space triangle soup + per-triangle shading records (= the triangle half
//                        of flatten_scene, host_scene.cpp; the unique meshes are uploaded once, not once per instance)
//   1. k_lbvh_bounds     triangle boxes + bounds of the centroids (ordered-int atomics)
//   2. k_lbvh_keys       63-bit Morton code of each centroid (21 bits per axis)
//   3. radix sort        8 passes of 8 bits over (key, triangle): k_radix_hist -> scan -> k_radix_scatter (stable)
//   4. the binary tree over the sorted triangles, one of
//      PLOC (bvh_builder = 1; Meister & Bittner 2018): repeat { k_ploc_nn: every cluster finds its nearest neighbour
//        (smallest merged surface area) among the 2 x 16 clusters around it in Morton order; k_ploc_mark -> scan ->
//        k_ploc_merge: mutual nearest neighbours become a node, the cluster array is compacted } until <= 1024 are left;
//        k_ploc_tail runs the remaining rounds (two thirds of them) in one block, out of shared memory
//      LBVH (bvh_builder = 2; Karras 2012): k_lbvh_hierarchy, every internal node finds its key range and split
//        independently, then k_lbvh_refit bottom-up (the second arrival at a node proceeds)
//   5. with every node, as it is made: its box AND the 8-wide collapse's dynamic programme (collapse_dp: Ylitie et al.
//      2017 §4.1, the same recurrences as Collapser::run in bvh8_build.cpp)
//   6. per BVH8 level    k_plan_level (children of each node from the DP decisions, octant slot assignment, counts)
//                        -> scan -> k_emit_level (quantised node, next level's work list, leaf triangle order)
//   7. k_pack_leaf_order triangle + shading records in leaf order (= pack_triangles of host_scene.cpp)
//
// The closest hit of a ray does not depend on the tree (ties break on the flattened primitive id, DESIGN.md §2), so
// frames rendered over this tree are bit-identical to frames over the host-built one: that is the test
// (tests/test_simt_renderer.py on the CPU under the SIMT emulation, tests/test_z_new_gpu_paths.py on the GPU).
// No kernel here waits on another block (no look-back scans): every pass is a separate launch; the one exception is
// k_lbvh_refit's classic fence + arrival-counter hand-over between the two threads that meet at a node.
#pragma once

#include <cstdint>

#include "bvh8.h"

namespace crt {

constexpr int kBuildBlock = 256;
constexpr int kBuildItems = 8;                           // keys per thread in the sort / scan tiles
constexpr int kBuildTile = kBuildBlock * kBuildItems;    // 2048
constexpr uint32_t kB2Invalid = 0xffffffffu;
constexpr float kDevPrimCost = 0.3f, kDevNodeCost = 1.0f;  // = kPrimCost, kNodeCost of bvh8_build.cpp
typedef unsigned long long u64;

// BVH2 node ids: leaf j (the j-th triangle in Morton order) = j, internal node k = n + k, k in [0, n-1).
// LBVH: internal node 0 is the root; PLOC: nodes are numbered as they are made, the last one (n-2) is the root.
struct Lbvh {
    uint32_t n;
    const float *verts;        // 9 floats per triangle, input order
    float4 *tri_lo, *tri_hi;   // per input triangle
    uint32_t *cbounds;         // 6 ordered uints: centroid min xyz, max xyz
    uint2 *children;           // per internal node (index k)
    uint32_t *parent;          // per node id (2n-1); LBVH only
    float4 *box_lo, *box_hi;   // per node id; box_lo.w = bits(triangle count)
    uint32_t *arrivals;        // per internal node (index k); LBVH only
    float *cost;               // 7 per node id
    uint8_t *decision;         // 7 per node id: type | dist_left << 2 | dist_right << 5
};

// ---- 0. flatten: thread per flattened triangle ----
struct DevSegment {  // one (instance, geometry) pair with at least one triangle
    uint32_t flat_base, num_tris;
    uint32_t vert_off, num_verts;  // first vertex / vertex count in the vertex arena (3 floats per vertex)
    uint32_t tri_off;              // first triangle in the index arena (3 indices per triangle)
    uint32_t uv_off;               // first vertex in the uv arena (2 floats per vertex), kB2Invalid = the geometry has no uvs
    uint32_t mat_id, instance;
};

__device__ __forceinline__ void dev_normalize3(float *v)
{
    // float3.ih:63-70: c = 1/length, then multiply (as normalize3 of host_scene.cpp)
    const float l = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    const float c = 1.f / l;
    v[0] *= c;
    v[1] *= c;
    v[2] *= c;
}

// The segment of flattened triangle f: the last one with flat_base <= f.
__device__ __forceinline__ uint32_t dev_find_segment(const DevSegment *segs, uint32_t num_segs, uint32_t f)
{
    uint32_t lo = 0u, hi = num_segs - 1u;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1u) >> 1;
        if (segs[mid].flat_base <= f) {
            lo = mid;
        } else {
            hi = mid - 1u;
        }
    }
    return lo;
}

// Flattened triangle f of segment seg (k_flatten, k_reflatten of scene_update.cuh): w = its world-space vertices
// (9 floats), shade = its TriShade record. Returns false, with nothing written, if a vertex index is out of range.
// xforms: 32 floats per instance = object_to_world, world_to_object (column-major). Arithmetic and its order are
// those of flatten_scene (compiled with -fmad=false here, -ffp-contract=off there), so that the records are the same
// bits: world-space vertices, normalize(transpose(world_to_object) * normalize(cross(v1 - v0, v2 - v0)))
// (render_embree.ispc:269,288-290), material id, the three uvs, the flattened primitive id.
__device__ __forceinline__ bool dev_flatten_triangle(const DevSegment &seg, uint32_t f, const float *xforms,
                                                     const float *vert_arena, const uint32_t *index_arena,
                                                     const float *uv_arena, float *w, float4 *shade)
{
    const uint32_t p = f - seg.flat_base;
    const uint32_t *ip = index_arena + 3 * (size_t)(seg.tri_off + p);
    const uint32_t idx[3] = {ip[0], ip[1], ip[2]};
    if (idx[0] >= seg.num_verts || idx[1] >= seg.num_verts || idx[2] >= seg.num_verts) {
        return false;
    }
    const float *m = xforms + (size_t)seg.instance * 32, *w2o = m + 16;
    float vo[3][3];
    for (int k = 0; k < 3; ++k) {
        const float *v = vert_arena + 3 * (size_t)(seg.vert_off + idx[k]);
        vo[k][0] = v[0];
        vo[k][1] = v[1];
        vo[k][2] = v[2];
        w[3 * k] = m[0] * v[0] + m[4] * v[1] + m[8] * v[2] + m[12];
        w[3 * k + 1] = m[1] * v[0] + m[5] * v[1] + m[9] * v[2] + m[13];
        w[3 * k + 2] = m[2] * v[0] + m[6] * v[1] + m[10] * v[2] + m[14];
    }
    const float e1[3] = {vo[1][0] - vo[0][0], vo[1][1] - vo[0][1], vo[1][2] - vo[0][2]};
    const float e2[3] = {vo[2][0] - vo[0][0], vo[2][1] - vo[0][1], vo[2][2] - vo[0][2]};
    float n[3] = {e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]};
    dev_normalize3(n);
    float r[3];
    r[0] = w2o[0] * n[0] + w2o[1] * n[1] + w2o[2] * n[2];
    r[1] = w2o[4] * n[0] + w2o[5] * n[1] + w2o[6] * n[2];
    r[2] = w2o[8] * n[0] + w2o[9] * n[1] + w2o[10] * n[2];
    dev_normalize3(r);
    for (int k = 0; k < 3; ++k) {
        // a zero-area triangle's normal is 0 * inf: store the NaN flatten_scene gets on x86 (0xffc00000), not the
        // GPU's canonical 0x7fffffff, so that the records are the same bits on both paths
        if (r[k] != r[k]) {
            r[k] = __uint_as_float(0xffc00000u);
        }
    }
    float uv[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const bool has_uv = seg.uv_off != kB2Invalid;
    if (has_uv) {
        for (int k = 0; k < 3; ++k) {
            const float *t = uv_arena + 2 * (size_t)(seg.uv_off + idx[k]);
            uv[2 * k] = t[0];
            uv[2 * k + 1] = t[1];
        }
    }
    // TriShade (host_scene.h): {n.xyz, material}, {uv0, uv1}, {uv2, has_uv, flat id}
    shade[0] = make_float4(r[0], r[1], r[2], __uint_as_float(seg.mat_id));
    shade[1] = make_float4(uv[0], uv[1], uv[2], uv[3]);
    shade[2] = make_float4(uv[4], uv[5], __uint_as_float(has_uv ? 1u : 0u), __uint_as_float(f));
    return true;
}

__global__ void __launch_bounds__(kBuildBlock) k_flatten(const DevSegment *segs, uint32_t num_segs, const float *xforms,
                                                         const float *vert_arena, const uint32_t *index_arena,
                                                         const float *uv_arena, uint32_t total, float *verts_out,
                                                         float4 *shade_out, uint32_t *bad_index)
{
    for (uint32_t f = blockIdx.x * blockDim.x + threadIdx.x; f < total; f += gridDim.x * blockDim.x) {
        const DevSegment seg = segs[dev_find_segment(segs, num_segs, f)];
        float w[9];
        float4 shade[3];
        if (!dev_flatten_triangle(seg, f, xforms, vert_arena, index_arena, uv_arena, w, shade)) {
            *bad_index = 1u;  // reported by the host after the launch
            for (int k = 0; k < 9; ++k) {
                w[k] = 0.f;
            }
            shade[0] = shade[1] = shade[2] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        for (int k = 0; k < 9; ++k) {
            verts_out[(size_t)f * 9 + k] = w[k];
        }
        for (int k = 0; k < 3; ++k) {
            shade_out[(size_t)f * 3 + k] = shade[k];
        }
    }
}

__device__ __forceinline__ uint32_t ordered_from_float(float f)
{
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float float_from_ordered(uint32_t u)
{
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

// ---- 1. triangle boxes, centroid bounds ----
__global__ void __launch_bounds__(kBuildBlock) k_lbvh_bounds(Lbvh b)
{
    float lo[3] = {3.0e38f, 3.0e38f, 3.0e38f}, hi[3] = {-3.0e38f, -3.0e38f, -3.0e38f};
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < b.n; i += gridDim.x * blockDim.x) {
        const float *v = b.verts + (size_t)i * 9;
        float tl[3], th[3];
        for (int a = 0; a < 3; ++a) {
            tl[a] = fminf(v[a], fminf(v[3 + a], v[6 + a]));
            th[a] = fmaxf(v[a], fmaxf(v[3 + a], v[6 + a]));
            const float c = 0.5f * tl[a] + 0.5f * th[a];
            lo[a] = fminf(lo[a], c);
            hi[a] = fmaxf(hi[a], c);
        }
        b.tri_lo[i] = make_float4(tl[0], tl[1], tl[2], 0.f);
        b.tri_hi[i] = make_float4(th[0], th[1], th[2], 0.f);
    }
    for (int a = 0; a < 3; ++a) {
        for (int off = 16; off > 0; off >>= 1) {
            lo[a] = fminf(lo[a], __shfl_down_sync(0xffffffffu, lo[a], off));
            hi[a] = fmaxf(hi[a], __shfl_down_sync(0xffffffffu, hi[a], off));
        }
    }
    if ((threadIdx.x & 31) == 0) {
        for (int a = 0; a < 3; ++a) {
            atomicMin(b.cbounds + a, ordered_from_float(lo[a]));
            atomicMax(b.cbounds + 3 + a, ordered_from_float(hi[a]));
        }
    }
}

// ---- 2. Morton keys ----
__device__ __forceinline__ u64 spread21(uint32_t v)
{
    u64 x = v & 0x1fffffu;
    x = (x | (x << 32)) & 0x1f00000000ffffull;
    x = (x | (x << 16)) & 0x1f0000ff0000ffull;
    x = (x | (x << 8)) & 0x100f00f00f00f00full;
    x = (x | (x << 4)) & 0x10c30c30c30c30c3ull;
    x = (x | (x << 2)) & 0x1249249249249249ull;
    return x;
}

__global__ void __launch_bounds__(kBuildBlock) k_lbvh_keys(Lbvh b, u64 *keys, uint32_t *vals)
{
    float lo[3], scale[3];
    for (int a = 0; a < 3; ++a) {
        lo[a] = float_from_ordered(b.cbounds[a]);
        const float ext = float_from_ordered(b.cbounds[3 + a]) - lo[a];
        scale[a] = ext > 0.f ? 2097152.f / ext : 0.f;
    }
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < b.n; i += gridDim.x * blockDim.x) {
        const float4 tl = b.tri_lo[i], th = b.tri_hi[i];
        const float c[3] = {0.5f * tl.x + 0.5f * th.x, 0.5f * tl.y + 0.5f * th.y, 0.5f * tl.z + 0.5f * th.z};
        uint32_t q[3];
        for (int a = 0; a < 3; ++a) {
            const float g = fminf(fmaxf((c[a] - lo[a]) * scale[a], 0.f), 2097151.f);  // NaN -> 0
            q[a] = (uint32_t)g;
        }
        keys[i] = (spread21(q[0]) << 2) | (spread21(q[1]) << 1) | spread21(q[2]);
        vals[i] = i;
    }
}

// ---- exclusive scan (tile sums -> recursive scan of the sums -> add) ----
// One tile = kBuildTile items, thread t owns items [t*8, t*8+8) of the tile.
template <typename T>
__global__ void __launch_bounds__(kBuildBlock) k_scan_tile(const T *in, T *out, uint32_t n, T *tile_sums)
{
    __shared__ T warp_total[kBuildBlock / 32];
    const uint32_t base = blockIdx.x * (uint32_t)kBuildTile + threadIdx.x * (uint32_t)kBuildItems;
    T v[kBuildItems];
    T sum = 0;
    for (int k = 0; k < kBuildItems; ++k) {
        v[k] = base + k < n ? in[base + k] : (T)0;
        sum += v[k];
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T inc = sum;
    for (int off = 1; off < 32; off <<= 1) {
        const T o = __shfl_up_sync(0xffffffffu, inc, off);
        if (lane >= off) {
            inc += o;
        }
    }
    if (lane == 31) {
        warp_total[warp] = inc;
    }
    __syncthreads();
    T run = inc - sum;
    T total = 0;
    for (int w = 0; w < kBuildBlock / 32; ++w) {
        if (w < warp) {
            run += warp_total[w];
        }
        total += warp_total[w];
    }
    for (int k = 0; k < kBuildItems; ++k) {
        if (base + k < n) {
            out[base + k] = run;
        }
        run += v[k];
    }
    if (threadIdx.x == 0 && tile_sums) {
        tile_sums[blockIdx.x] = total;
    }
    __syncthreads();  // warp_total is reused by the next block of a grid-serial run
}

template <typename T>
__global__ void __launch_bounds__(kBuildBlock) k_scan_add(T *out, uint32_t n, const T *tile_offsets)
{
    const T add = tile_offsets[blockIdx.x];
    const uint32_t base = blockIdx.x * (uint32_t)kBuildTile;
    for (uint32_t k = threadIdx.x; k < (uint32_t)kBuildTile; k += blockDim.x) {
        if (base + k < n) {
            out[base + k] += add;
        }
    }
}

// ---- 3. radix sort pass: 8-bit digit at `shift`; block = one tile, warp w = keys [w*256, w*256+256) of it ----
__global__ void __launch_bounds__(kBuildBlock) k_radix_hist(const u64 *keys, uint32_t n, int shift, uint32_t *hist,
                                                            uint32_t num_tiles)
{
    __shared__ uint32_t h[256];
    h[threadIdx.x] = 0u;
    __syncthreads();
    const uint32_t base = blockIdx.x * (uint32_t)kBuildTile;
    for (int k = 0; k < kBuildItems; ++k) {
        const uint32_t i = base + (uint32_t)k * kBuildBlock + threadIdx.x;
        if (i < n) {
            atomicAdd(&h[(uint32_t)(keys[i] >> shift) & 0xffu], 1u);
        }
    }
    __syncthreads();
    hist[threadIdx.x * num_tiles + blockIdx.x] = h[threadIdx.x];  // digit-major: one scan gives every offset
    __syncthreads();
}

__global__ void __launch_bounds__(kBuildBlock) k_radix_scatter(const u64 *keys_in, const uint32_t *vals_in, u64 *keys_out,
                                                               uint32_t *vals_out, uint32_t n, int shift,
                                                               const uint32_t *hist_scanned, uint32_t num_tiles)
{
    __shared__ uint32_t cnt[kBuildBlock / 32][256];
    __shared__ uint32_t goff[256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned lanemask_lt = (1u << lane) - 1u;
    for (int w = 0; w < kBuildBlock / 32; ++w) {
        cnt[w][threadIdx.x] = 0u;
    }
    goff[threadIdx.x] = hist_scanned[threadIdx.x * num_tiles + blockIdx.x];
    __syncthreads();
    const uint32_t base = blockIdx.x * (uint32_t)kBuildTile + (uint32_t)warp * 256u;
    u64 key[kBuildItems];
    uint32_t val[kBuildItems], rank[kBuildItems];
    for (int r = 0; r < kBuildItems; ++r) {
        const uint32_t i = base + (uint32_t)r * 32u + lane;
        const bool valid = i < n;
        key[r] = valid ? keys_in[i] : 0ull;
        val[r] = valid ? vals_in[i] : 0u;
        const uint32_t d = valid ? ((uint32_t)(key[r] >> shift) & 0xffu) : 256u;
        // stable rank of the key among the equal digits of this warp's sub-tile: earlier rounds, then lower lanes
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const int leader = __ffs(peers) - 1;
        uint32_t before = 0u;
        if (lane == leader && valid) {
            before = cnt[warp][d];
            cnt[warp][d] = before + (uint32_t)__popc(peers);
        }
        before = __shfl_sync(0xffffffffu, before, leader);
        rank[r] = before + (uint32_t)__popc(peers & lanemask_lt);
        __syncwarp();
    }
    __syncthreads();
    {   // per digit: exclusive prefix of the warps' counts
        uint32_t run = 0u;
        for (int w = 0; w < kBuildBlock / 32; ++w) {
            const uint32_t c = cnt[w][threadIdx.x];
            cnt[w][threadIdx.x] = run;
            run += c;
        }
    }
    __syncthreads();
    for (int r = 0; r < kBuildItems; ++r) {
        const uint32_t i = base + (uint32_t)r * 32u + lane;
        if (i < n) {
            const uint32_t d = (uint32_t)(key[r] >> shift) & 0xffu;
            const uint32_t pos = goff[d] + cnt[warp][d] + rank[r];
            keys_out[pos] = key[r];
            vals_out[pos] = val[r];
        }
    }
    __syncthreads();
}

// ---- 4. Karras 2012 ----
__device__ __forceinline__ int lbvh_delta(const u64 *keys, int n, int i, int j)
{
    if (j < 0 || j >= n) {
        return -1;
    }
    const u64 a = keys[i], b = keys[j];
    if (a == b) {
        return 64 + __clz((unsigned)(i ^ j));  // equal codes: the position is the tie-breaker
    }
    return __clzll((long long)(a ^ b));
}

__global__ void __launch_bounds__(kBuildBlock) k_lbvh_hierarchy(Lbvh b, const u64 *keys)
{
    const int n = (int)b.n;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n - 1; i += gridDim.x * blockDim.x) {
        const int d = lbvh_delta(keys, n, i, i + 1) - lbvh_delta(keys, n, i, i - 1) >= 0 ? 1 : -1;
        const int dmin = lbvh_delta(keys, n, i, i - d);
        int lmax = 2;
        while (lbvh_delta(keys, n, i, i + lmax * d) > dmin) {
            lmax *= 2;
        }
        int l = 0;
        for (int t = lmax / 2; t >= 1; t /= 2) {
            if (lbvh_delta(keys, n, i, i + (l + t) * d) > dmin) {
                l += t;
            }
        }
        const int j = i + l * d;
        const int dnode = lbvh_delta(keys, n, i, j);
        int s = 0, t = l;
        do {
            t = (t + 1) / 2;
            if (lbvh_delta(keys, n, i, i + (s + t) * d) > dnode) {
                s += t;
            }
        } while (t > 1);
        const int gamma = i + s * d + min(d, 0);
        const int first = min(i, j), last = max(i, j);
        const uint32_t left = first == gamma ? (uint32_t)gamma : (uint32_t)(n + gamma);
        const uint32_t right = last == gamma + 1 ? (uint32_t)(gamma + 1) : (uint32_t)(n + gamma + 1);
        b.children[i] = make_uint2(left, right);
        b.parent[left] = (uint32_t)(n + i);
        b.parent[right] = (uint32_t)(n + i);
        b.arrivals[i] = 0u;
        if (i == 0) {
            b.parent[n] = kB2Invalid;
        }
    }
}

// ---- 5. boxes + collapse DP ----
__device__ __forceinline__ float box_half_area(const float4 lo, const float4 hi)
{
    const float dx = hi.x - lo.x, dy = hi.y - lo.y, dz = hi.z - lo.z;
    return dx * dy + dy * dz + dz * dx;
}
enum : uint8_t { kDecLeaf = 0, kDecInternal = 1, kDecDistribute = 2 };
__device__ __forceinline__ uint8_t make_decision(uint8_t type, int dl, int dr)
{
    return (uint8_t)(type | (dl << 2) | (dr << 5));
}

// leaf j = the j-th triangle in Morton order; also the initial cluster list of PLOC
__global__ void __launch_bounds__(kBuildBlock) k_bvh2_leaves(Lbvh b, const uint32_t *vals, uint32_t *clusters)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < b.n; j += gridDim.x * blockDim.x) {
        const uint32_t t = vals[j];
        float4 lo = b.tri_lo[t];
        const float4 hi = b.tri_hi[t];
        lo.w = __uint_as_float(1u);
        b.box_lo[j] = lo;
        b.box_hi[j] = hi;
        const float c = box_half_area(lo, hi) * kDevPrimCost;
        for (int i = 0; i < 7; ++i) {
            b.cost[7 * (size_t)j + i] = c;
            b.decision[7 * (size_t)j + i] = make_decision(kDecLeaf, 0, 0);
        }
        if (clusters) {
            clusters[j] = j;
        }
    }
}

// Node p over the finished subtrees l and r: box, triangle count, and cost[i] = the cheapest way to represent the
// subtree as a forest of at most i+1 BVH8 children, with the decision that achieves it.
// L2_ONLY: the children were written by OTHER blocks of the SAME launch (k_lbvh_refit): their records are read with
// ld.global.cg, so that a line this SM cached before the sibling thread wrote it cannot be served from L1.
template <bool L2_ONLY>
__device__ __forceinline__ float4 load_node4(const float4 *p)
{
    return L2_ONLY ? __ldcg(p) : *p;
}
template <bool L2_ONLY>
__device__ __forceinline__ float load_node1(const float *p)
{
    return L2_ONLY ? __ldcg(p) : *p;
}

template <bool L2_ONLY = false>
__device__ __forceinline__ void collapse_dp(const Lbvh &b, uint32_t p, uint32_t l, uint32_t r)
{
    const float4 llo = load_node4<L2_ONLY>(b.box_lo + l), lhi = load_node4<L2_ONLY>(b.box_hi + l);
    const float4 rlo = load_node4<L2_ONLY>(b.box_lo + r), rhi = load_node4<L2_ONLY>(b.box_hi + r);
    const uint32_t cnt = __float_as_uint(llo.w) + __float_as_uint(rlo.w);
    const float4 lo = make_float4(fminf(llo.x, rlo.x), fminf(llo.y, rlo.y), fminf(llo.z, rlo.z), __uint_as_float(cnt));
    const float4 hi = make_float4(fmaxf(lhi.x, rhi.x), fmaxf(lhi.y, rhi.y), fmaxf(lhi.z, rhi.z), 0.f);
    b.box_lo[p] = lo;
    b.box_hi[p] = hi;
    const float area = box_half_area(lo, hi);
    float cl[7], cr[7], cn[7];
    uint8_t dn[7];
    for (int i = 0; i < 7; ++i) {
        cl[i] = load_node1<L2_ONLY>(b.cost + 7 * (size_t)l + i);
        cr[i] = load_node1<L2_ONLY>(b.cost + 7 * (size_t)r + i);
    }
    {
        // i = 0: a single root — a leaf (<= 3 triangles) or an internal node whose 8 slots go to the two subtrees
        const float inf = __uint_as_float(0x7f800000u);
        const float cost_leaf = cnt <= 3u ? area * (float)cnt * kDevPrimCost : inf;
        float best = inf;
        int bl = 0, br = 0;
        for (int k = 0; k < 7; ++k) {
            const float c = cl[k] + cr[6 - k];
            if (c < best) {
                best = c;
                bl = k;
                br = 6 - k;
            }
        }
        const float cost_internal = best + area * kDevNodeCost;
        if (cost_leaf < cost_internal) {
            cn[0] = cost_leaf;
            dn[0] = make_decision(kDecLeaf, 0, 0);
        } else {
            cn[0] = cost_internal;
            dn[0] = make_decision(kDecInternal, bl, br);
        }
    }
    for (int i = 1; i < 7; ++i) {  // a forest of up to i+1 roots
        cn[i] = cn[i - 1];
        dn[i] = dn[i - 1];
        for (int k = 0; k < i; ++k) {
            const float c = cl[k] + cr[i - k - 1];
            if (c < cn[i]) {
                cn[i] = c;
                dn[i] = make_decision(kDecDistribute, k, i - k - 1);
            }
        }
    }
    for (int i = 0; i < 7; ++i) {
        b.cost[7 * (size_t)p + i] = cn[i];
        b.decision[7 * (size_t)p + i] = dn[i];
    }
}

// LBVH: bottom-up from every leaf; the second thread to arrive at a node finds both subtrees finished
__global__ void __launch_bounds__(kBuildBlock) k_lbvh_refit(Lbvh b)
{
    const uint32_t n = b.n;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        uint32_t p = b.parent[j];
        while (p != kB2Invalid) {
            __threadfence();  // publish this subtree before announcing it
            if (atomicAdd(&b.arrivals[p - n], 1u) == 0u) {
                break;  // the sibling subtree is not finished: its thread will continue from here
            }
            __threadfence();
            const uint2 ch = b.children[p - n];
            collapse_dp<true>(b, p, ch.x, ch.y);
            p = b.parent[p];
        }
    }
}

// ---- PLOC ----
constexpr int kPlocRadius = 16, kPlocMaxRadius = 32;

// Among candidates with EQUAL merged area (everywhere on regular geometry: a row of identical quads) the "aligned"
// partner i ^ 1 wins, then the lower position. Lowest-position-first alone turns such a row into a chain — every
// cluster points at its left neighbour and only the first pair is mutual, one merge per round; with the aligned
// partner preferred the row pairs up (0,1), (2,3), ... in a single round (rungholt_like, 179 K: 65 -> 43 rounds).
// The rank is symmetric (j == i ^ 1 <=> i == j ^ 1), so the lowest-positioned cluster of the globally best
// (area, rank) pairs and its lowest such partner always choose each other: every round merges at least one pair.
__device__ __forceinline__ uint32_t ploc_tie_rank(uint32_t i, uint32_t j)
{
    return j == (i ^ 1u) ? 0u : 1u;
}

// nn[i] = the cluster within `radius` (<= kPlocMaxRadius) positions of i whose union with i has the smallest surface area (ties:
// ploc_tie_rank). forced: pair up neighbours (i ^ 1) regardless of distance — the way out if an adversarial input
// leaves too few mutual pairs per round.
__global__ void __launch_bounds__(kBuildBlock) k_ploc_nn(Lbvh b, const uint32_t *clusters, uint32_t m, uint32_t *nn, int radius,
                                                         int forced)
{
    __shared__ float4 slo[kBuildBlock + 2 * kPlocMaxRadius], shi[kBuildBlock + 2 * kPlocMaxRadius];
    const int block_first = (int)(blockIdx.x * blockDim.x) - radius;
    for (int k = threadIdx.x; k < kBuildBlock + 2 * radius; k += blockDim.x) {
        const int pos = block_first + k;
        if (pos >= 0 && pos < (int)m) {
            const uint32_t c = clusters[pos];
            slo[k] = b.box_lo[c];
            shi[k] = b.box_hi[c];
        }
    }
    __syncthreads();
    const int i = (int)(blockIdx.x * blockDim.x + threadIdx.x);
    if (i < (int)m) {
        uint32_t best_j = (uint32_t)i;
        if (forced) {
            best_j = (uint32_t)(i ^ 1) < m ? (uint32_t)(i ^ 1) : (uint32_t)i;
        } else {
            const float4 lo = slo[threadIdx.x + radius], hi = shi[threadIdx.x + radius];
            float best = __uint_as_float(0x7f800000u);
            const int j0 = max(i - radius, 0), j1 = min(i + radius, (int)m - 1);
            for (int j = j0; j <= j1; ++j) {
                if (j == i) {
                    continue;
                }
                const float4 ol = slo[j - block_first], oh = shi[j - block_first];
                const float4 ul = make_float4(fminf(lo.x, ol.x), fminf(lo.y, ol.y), fminf(lo.z, ol.z), 0.f);
                const float4 uh = make_float4(fmaxf(hi.x, oh.x), fmaxf(hi.y, oh.y), fmaxf(hi.z, oh.z), 0.f);
                const float a = box_half_area(ul, uh);
                // (the first test also takes a NaN / inf area as the first candidate)
                if (best_j == (uint32_t)i || a < best || (a == best && ploc_tie_rank((uint32_t)i, (uint32_t)j) < ploc_tie_rank((uint32_t)i, best_j))) {
                    best = a;
                    best_j = (uint32_t)j;
                }
            }
        }
        nn[i] = best_j;
    }
    __syncthreads();
}

// counts[i] = (cluster i survives this round) << 32 | (cluster i is the lower half of a merging pair)
__global__ void __launch_bounds__(kBuildBlock) k_ploc_mark(const uint32_t *nn, uint32_t m, u64 *counts)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
        const uint32_t j = nn[i];
        const bool mutual = j != i && nn[j] == i;
        counts[i] = ((u64)(mutual && j < i ? 0u : 1u) << 32) | (mutual && i < j ? 1u : 0u);
    }
}

__global__ void __launch_bounds__(kBuildBlock) k_ploc_merge(Lbvh b, const uint32_t *clusters, const uint32_t *nn, uint32_t m,
                                                            const u64 *offsets, uint32_t nodes_made, uint32_t *clusters_out)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
        const uint32_t j = nn[i];
        const bool mutual = j != i && nn[j] == i;
        if (mutual && j < i) {
            continue;  // merged into position j
        }
        const u64 off = offsets[i];
        uint32_t c = clusters[i];
        if (mutual) {
            const uint32_t k = nodes_made + (uint32_t)off;  // internal node index
            const uint32_t other = clusters[j];
            b.children[k] = make_uint2(c, other);
            collapse_dp(b, b.n + k, c, other);
            c = b.n + k;
        }
        clusters_out[(uint32_t)(off >> 32)] = c;
    }
}

// The last rounds of PLOC in ONE block. The cluster count shrinks by about a fifth per round, so two thirds of a
// build's rounds run on fewer than kPlocTailMax clusters — from the host each of them is six tiny launches and a round
// trip for the count. Here the cluster list, the nearest-neighbour table and the boxes live in shared memory and a
// round is four block barriers. Same algorithm, same ties, same node numbering as the launches it replaces: the tree
// is identical (tested). rounds_io: rounds done so far in, total rounds out (the 256-round cut-off carries over).
constexpr int kPlocTailMax = 1024;
constexpr int kPlocTailItems = kPlocTailMax / kBuildBlock;  // consecutive clusters per thread in the scan / merge

__global__ void __launch_bounds__(kBuildBlock) k_ploc_tail(Lbvh b, const uint32_t *clusters, uint32_t m, uint32_t nodes_made,
                                                           int radius, uint32_t *rounds_io)
{
    __shared__ uint32_t cl[2][kPlocTailMax];
    __shared__ uint32_t nn[kPlocTailMax];
    __shared__ float4 slo[kPlocTailMax], shi[kPlocTailMax];
    __shared__ uint32_t warp_total[kBuildBlock / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t i = threadIdx.x; i < m; i += blockDim.x) {
        cl[0][i] = clusters[i];
    }
    uint32_t rounds = *rounds_io;
    int cur = 0;
    __syncthreads();
    while (m > 1u) {
        for (uint32_t i = threadIdx.x; i < m; i += blockDim.x) {
            const uint32_t c = cl[cur][i];
            slo[i] = b.box_lo[c];
            shi[i] = b.box_hi[c];
        }
        __syncthreads();
        const bool forced = rounds >= 256u;
        for (uint32_t i = threadIdx.x; i < m; i += blockDim.x) {  // = k_ploc_nn
            uint32_t best_j = i;
            if (forced) {
                best_j = (i ^ 1u) < m ? (i ^ 1u) : i;
            } else {
                const float4 lo = slo[i], hi = shi[i];
                float best = __uint_as_float(0x7f800000u);
                const int j0 = max((int)i - radius, 0), j1 = min((int)i + radius, (int)m - 1);
                for (int j = j0; j <= j1; ++j) {
                    if (j == (int)i) {
                        continue;
                    }
                    const float4 ol = slo[j], oh = shi[j];
                    const float4 ul = make_float4(fminf(lo.x, ol.x), fminf(lo.y, ol.y), fminf(lo.z, ol.z), 0.f);
                    const float4 uh = make_float4(fmaxf(hi.x, oh.x), fmaxf(hi.y, oh.y), fmaxf(hi.z, oh.z), 0.f);
                    const float a = box_half_area(ul, uh);
                    if (best_j == i || a < best || (a == best && ploc_tie_rank(i, (uint32_t)j) < ploc_tie_rank(i, best_j))) {
                        best = a;
                        best_j = (uint32_t)j;
                    }
                }
            }
            nn[i] = best_j;
        }
        __syncthreads();
        // = k_ploc_mark + scan: thread t owns clusters [t * 4, t * 4 + 4); keep << 16 | leader fits 32 bits (m <= 1024)
        uint32_t flags[kPlocTailItems], sum = 0u;
        for (int k = 0; k < kPlocTailItems; ++k) {
            const uint32_t i = threadIdx.x * (uint32_t)kPlocTailItems + (uint32_t)k;
            flags[k] = 0u;
            if (i < m) {
                const uint32_t j = nn[i];
                const bool mutual = j != i && nn[j] == i;
                flags[k] = ((mutual && j < i ? 0u : 1u) << 16) | (mutual && i < j ? 1u : 0u);
            }
            sum += flags[k];
        }
        uint32_t inc = sum;
        for (int off = 1; off < 32; off <<= 1) {
            const uint32_t o = __shfl_up_sync(0xffffffffu, inc, off);
            if (lane >= off) {
                inc += o;
            }
        }
        if (lane == 31) {
            warp_total[warp] = inc;
        }
        __syncthreads();
        uint32_t run = inc - sum, total = 0u;
        for (int w = 0; w < kBuildBlock / 32; ++w) {
            if (w < warp) {
                run += warp_total[w];
            }
            total += warp_total[w];
        }
        // = k_ploc_merge
        for (int k = 0; k < kPlocTailItems; ++k) {
            const uint32_t i = threadIdx.x * (uint32_t)kPlocTailItems + (uint32_t)k;
            if (i < m && (flags[k] >> 16)) {
                uint32_t c = cl[cur][i];
                if (flags[k] & 1u) {
                    const uint32_t node = nodes_made + (run & 0xffffu);
                    const uint32_t other = cl[cur][nn[i]];
                    b.children[node] = make_uint2(c, other);
                    collapse_dp(b, b.n + node, c, other);
                    c = b.n + node;
                }
                cl[cur ^ 1][run >> 16] = c;
            }
            run += flags[k];
        }
        __syncthreads();  // also makes this round's nodes (global memory) visible to the whole block
        m = total >> 16;
        nodes_made += total & 0xffffu;
        cur ^= 1;
        ++rounds;
    }
    if (threadIdx.x == 0) {
        *rounds_io = rounds;
    }
}

// ---- 6. BVH8 emission, one level at a time ----
struct LevelArgs {
    const uint32_t *work;   // BVH2 node of each BVH8 node of this level
    uint32_t count;         // nodes in this level
    uint32_t node_begin;    // index of the level's first BVH8 node
    uint32_t next_begin;    // index of the next level's first node (= node_begin + count)
    uint32_t tri_begin;     // triangles emitted by earlier levels
    uint32_t *slots;        // 8 per BVH8 node: BVH2 node in slot s, kB2Invalid = empty
    u64 *counts;            // per node of the level: inner children << 32 | leaf triangles
    const u64 *offsets;     // exclusive scan of counts
    uint32_t *next_work;
    Bvh8Node *nodes;
    uint32_t *tri_order;    // leaf order -> input triangle
};

__device__ __forceinline__ bool lbvh_is_leaf(const Lbvh &b, uint32_t node) { return node < b.n; }
__device__ __forceinline__ bool lbvh_leaf_child(const Lbvh &b, uint32_t node)
{
    return lbvh_is_leaf(b, node) || (b.decision[7 * (size_t)node] & 3u) == kDecLeaf;
}

__global__ void __launch_bounds__(kBuildBlock) k_plan_level(Lbvh b, LevelArgs lv)
{
    for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < lv.count; w += gridDim.x * blockDim.x) {
        const uint32_t root = lv.work[w];
        uint32_t children[8];
        int num = 0;
        if (lbvh_leaf_child(b, root)) {
            children[num++] = root;  // only the scene root (<= 3 triangles) can be a leaf here
        } else {
            // the forest (root, 0) of the DP, left to right (Collapser::get_children): a stack of tasks, "expand
            // the forest (node, i)" or (top bit set) "node is a child"; every task yields >= 1 of the <= 8 children
            uint32_t st_node[8];
            uint8_t st_i[8];
            int sp = 0;
            st_node[sp] = root;
            st_i[sp++] = 0;
            while (sp) {
                --sp;
                const uint32_t nd = st_node[sp];
                if (nd & 0x80000000u) {
                    children[num++] = nd & 0x7fffffffu;
                    continue;
                }
                const uint8_t d = b.decision[7 * (size_t)nd + st_i[sp]];
                const uint2 ch = b.children[nd - b.n];
                const uint8_t dl = (d >> 2) & 7u, dr = (d >> 5) & 7u;
                const bool expand_l = (b.decision[7 * (size_t)ch.x + dl] & 3u) == kDecDistribute;
                const bool expand_r = (b.decision[7 * (size_t)ch.y + dr] & 3u) == kDecDistribute;
                st_node[sp] = expand_r ? ch.y : (ch.y | 0x80000000u);  // right below left: left is handled first
                st_i[sp++] = dr;
                st_node[sp] = expand_l ? ch.x : (ch.x | 0x80000000u);
                st_i[sp++] = dl;
            }
        }
        // slot s should hold the child met first by rays of octant s (assign_slots of bvh8_build.cpp)
        const float4 plo = b.box_lo[root], phi = b.box_hi[root];
        const float cx = 0.5f * (plo.x + phi.x), cy = 0.5f * (plo.y + phi.y), cz = 0.5f * (plo.z + phi.z);
        float ox[8], oy[8], oz[8];
        for (int c = 0; c < num; ++c) {
            const float4 lo = b.box_lo[children[c]], hi = b.box_hi[children[c]];
            ox[c] = 0.5f * (lo.x + hi.x) - cx;
            oy[c] = 0.5f * (lo.y + hi.y) - cy;
            oz[c] = 0.5f * (lo.z + hi.z) - cz;
        }
        int slot_child[8];
        for (int s = 0; s < 8; ++s) {
            slot_child[s] = -1;
        }
        unsigned child_done = 0u;
        for (int it = 0; it < num; ++it) {
            float best = 3.4028235e38f;
            int bc = -1, bs = -1;
            for (int c = 0; c < num; ++c) {
                if (child_done & (1u << c)) {
                    continue;
                }
                for (int s = 0; s < 8; ++s) {
                    if (slot_child[s] >= 0) {
                        continue;
                    }
                    const float v = ox[c] * ((s & 4) ? -1.f : 1.f) + oy[c] * ((s & 2) ? -1.f : 1.f) + oz[c] * ((s & 1) ? -1.f : 1.f);
                    if (v < best || bc < 0) {
                        best = v;
                        bc = c;
                        bs = s;
                    }
                }
            }
            child_done |= 1u << bc;
            slot_child[bs] = bc;
        }
        uint32_t inner = 0u, tris = 0u;
        for (int s = 0; s < 8; ++s) {
            uint32_t cn = kB2Invalid;
            if (slot_child[s] >= 0) {
                cn = children[slot_child[s]];
                if (lbvh_leaf_child(b, cn)) {
                    tris += __float_as_uint(b.box_lo[cn].w);
                } else {
                    ++inner;
                }
            }
            lv.slots[(size_t)(lv.node_begin + w) * 8 + s] = cn;
        }
        lv.counts[w] = ((u64)inner << 32) | tris;
    }
}

__device__ __forceinline__ float pow2_biased(int e) { return __uint_as_float((uint32_t)e << 23); }

// (int)x as x86-64 converts a double (cvttsd2si): truncation toward zero, and INT_MIN for NaN and for every x outside
// [-2^31, 2^31). fill_node of bvh8_build.cpp converts that way; the device's own conversion saturates and maps NaN to
// 0, which for a child box whose lower bound is +inf gives qlo = 255 where the host builder gives 0.
__device__ __forceinline__ int double_to_int_x86(double x)
{
    return (x >= -2147483648.0 && x < 2147483648.0) ? (int)x : INT32_MIN;
}

// The quantisation frame of a BVH8 node over its box [blo, bhi] (fill_node of bvh8_build.cpp; k_emit_level, k_bvh8_refit
// of scene_update.cuh): out.p = blo and the exponents out.e; step = the grid step per axis. Flat axes get a thin but
// non-zero grid, and the far plane of the node must be representable: lo + 255 * 2^e >= hi.
// Boxes with an infinite bound (geometry at +-inf, or a sum overflowing) take the host builder's arithmetic too: the
// extent of an axis whose bounds are both +inf or both -inf is NaN and stays NaN through the two maxima (std::max's
// order, which keeps its first operand when the compare fails), and the conversions are the x86 ones.
__device__ __forceinline__ void bvh8_node_frame(const float *blo, const float *bhi, Bvh8Node &out, double *step)
{
    float max_ext = 0.f;
    for (int a = 0; a < 3; ++a) {
        out.p[a] = blo[a];
        max_ext = fmaxf(max_ext, bhi[a] - blo[a]);
    }
    for (int a = 0; a < 3; ++a) {
        const float thin = max_ext * (1.f / 65536.f);
        float ext = bhi[a] - blo[a];
        ext = ext < thin ? thin : ext;
        ext = ext < 1e-30f ? 1e-30f : ext;
        int e = double_to_int_x86(ceil(log2((double)ext / 255.0)));
        e = min(max(e, -100), 100);
        while (e < 100 && (double)blo[a] + 255.0 * ldexp(1.0, e) < (double)bhi[a]) {
            ++e;
        }
        out.e[a] = (uint8_t)(e + 127);
        step[a] = (double)pow2_biased(e + 127);
    }
}

// A child box [l3, h3] on the node's grid (bvh8_node_frame): conservative, at least one cell thick.
__device__ __forceinline__ void bvh8_quantise_child(const Bvh8Node &out, const double *step, const float *l3, const float *h3,
                                                    uint8_t *qlo, uint8_t *qhi)
{
    for (int a = 0; a < 3; ++a) {
        const double p = out.p[a], st = step[a];
        int lo = double_to_int_x86(floor(((double)l3[a] - p) / st));
        int hi = double_to_int_x86(ceil(((double)h3[a] - p) / st));
        lo = min(max(lo, 0), 255);
        hi = min(max(hi, 0), 255);
        while (lo > 0 && p + lo * st > (double)l3[a]) {  // conservative: p + q*step is exact in double
            --lo;
        }
        while (hi < 255 && p + hi * st < (double)h3[a]) {
            ++hi;
        }
        if (hi <= lo) {  // give flat boxes one grid cell of thickness
            if (hi < 255) {
                hi = lo + 1;
            } else {
                lo = hi - 1;
            }
        }
        qlo[a] = (uint8_t)lo;
        qhi[a] = (uint8_t)hi;
    }
}

__global__ void __launch_bounds__(kBuildBlock) k_emit_level(Lbvh b, LevelArgs lv, const uint32_t *vals)
{
    for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < lv.count; w += gridDim.x * blockDim.x) {
        const uint32_t root = lv.work[w];
        const u64 off = lv.offsets[w];
        const uint32_t child_first = (uint32_t)(off >> 32), tri_base = lv.tri_begin + (uint32_t)off;
        const float4 plo = b.box_lo[root], phi = b.box_hi[root];
        const float blo[3] = {plo.x, plo.y, plo.z}, bhi[3] = {phi.x, phi.y, phi.z};
        alignas(16) Bvh8Node out;
        double step[3];
        bvh8_node_frame(blo, bhi, out, step);
        out.imask = 0;
        out.child_base = lv.next_begin + child_first;
        out.tri_base = tri_base;
        uint32_t tri_off = 0u, inner_rank = 0u;
        for (int s = 0; s < 8; ++s) {
            const uint32_t cn = lv.slots[(size_t)(lv.node_begin + w) * 8 + s];
            uint8_t qlo[3] = {0, 0, 0}, qhi[3] = {0, 0, 0};
            uint8_t meta = 0;
            if (cn != kB2Invalid) {
                const float4 clo = b.box_lo[cn], chi = b.box_hi[cn];
                const float l3[3] = {clo.x, clo.y, clo.z}, h3[3] = {chi.x, chi.y, chi.z};
                bvh8_quantise_child(out, step, l3, h3, qlo, qhi);
                if (lbvh_leaf_child(b, cn)) {
                    // the <= 3 triangles under cn, left to right
                    uint32_t st[4], k = 0u;
                    int sp = 0;
                    st[sp++] = cn;
                    while (sp) {
                        const uint32_t c = st[--sp];
                        if (lbvh_is_leaf(b, c)) {
                            lv.tri_order[tri_base + tri_off + k++] = vals[c];
                        } else {
                            const uint2 ch = b.children[c - b.n];
                            st[sp++] = ch.y;
                            st[sp++] = ch.x;
                        }
                    }
                    meta = (uint8_t)(((k == 1u ? 0b001u : (k == 2u ? 0b011u : 0b111u)) << 5) | tri_off);
                    tri_off += k;
                } else {
                    meta = (uint8_t)((0b001u << 5) | (24u + (uint32_t)s));
                    out.imask |= (uint8_t)(1u << s);
                    lv.next_work[child_first + inner_rank++] = cn;
                }
            }
            out.meta[s] = meta;
            out.qlo_x[s] = qlo[0];
            out.qlo_y[s] = qlo[1];
            out.qlo_z[s] = qlo[2];
            out.qhi_x[s] = qhi[0];
            out.qhi_y[s] = qhi[1];
            out.qhi_z[s] = qhi[2];
        }
        // 5 x 128-bit stores
        const uint4 *src = reinterpret_cast<const uint4 *>(&out);
        uint4 *dst = reinterpret_cast<uint4 *>(lv.nodes + lv.node_begin + w);
        for (int q = 0; q < 5; ++q) {
            dst[q] = src[q];
        }
    }
}

// ---- 7. records in leaf order (pack_triangles, host_scene.cpp) ----
__global__ void __launch_bounds__(kBuildBlock) k_pack_leaf_order(const float *verts, const float4 *shade_in,
                                                                 const uint32_t *tri_order, uint32_t n, float4 *tris_out,
                                                                 float4 *shade_out)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t src = tri_order[i];
        const float *v = verts + (size_t)src * 9;
        const float4 s0 = shade_in[(size_t)src * 3], s1 = shade_in[(size_t)src * 3 + 1], s2 = shade_in[(size_t)src * 3 + 2];
        // TriShade: {n.xyz, material}, {uv0, uv1}, {uv2, has_uv, flat_id}
        tris_out[(size_t)i * 3] = make_float4(v[0], v[1], v[2], s2.w);
        tris_out[(size_t)i * 3 + 1] = make_float4(v[3] - v[0], v[4] - v[1], v[5] - v[2], 0.f);
        tris_out[(size_t)i * 3 + 2] = make_float4(v[6] - v[0], v[7] - v[1], v[8] - v[2], 0.f);
        shade_out[(size_t)i * 3] = s0;
        shade_out[(size_t)i * 3 + 1] = s1;
        shade_out[(size_t)i * 3 + 2] = s2;
    }
}

}  // namespace crt
