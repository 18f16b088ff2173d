// scene_device_build.cuh — the host side of set_scene ON THE DEVICE (option "bvh_builder" = 1 / 2): uploads, launches
// of the kernels of bvh8_device.cuh, the few host round trips (PLOC round counts, BVH8 level sizes). Included by
// crt_cuda_core.cu only. Fills the renderer's node / triangle / shading-record buffers exactly as the host path does
// (flatten_scene + build_bvh8 + pack_triangles); see bvh8_device.cuh for what each kernel does.
#pragma once

#include <chrono>
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../include/crt_scene.h"
#include "bvh8_device.cuh"
#include "bvh8_traverse.h"
#include "cuda_host_utils.h"
#include "host_scene.h"
#include "scene_update.cuh"

namespace crt_host {

// The device builder itself gave up on this input (as opposed to a scene error or a CUDA error): set_scene catches it
// and builds on the host instead.
struct DeviceBuildFailure : std::runtime_error {
    using std::runtime_error::runtime_error;
};

// cudaEvents that are destroyed on every exit path, exceptions included
struct EventSet {
    std::vector<cudaEvent_t> ev;
    explicit EventSet(size_t n)
    {
        ev.reserve(n);
        for (size_t i = 0; i < n; ++i) {
            cudaEvent_t e;
            CUDA_CHECK(cudaEventCreate(&e));
            ev.push_back(e);
        }
    }
    ~EventSet()
    {
        for (cudaEvent_t e : ev) {
            cudaEventDestroy(e);
        }
    }
    EventSet(const EventSet &) = delete;
    EventSet &operator=(const EventSet &) = delete;
    cudaEvent_t operator[](size_t i) const { return ev[i]; }
};

// The binary tree behind a device build, copied out before its buffers are released (bvh_devcheck.cu; the renderer
// leaves DeviceSceneBuild::dump null): the sorted Morton keys and triangle ids, the centroid bounds (ordered uints),
// and per BVH2 node id (bvh8_device.cuh: Lbvh) the children, boxes, costs and decisions.
struct Bvh2Dump {
    std::vector<crt::u64> keys;
    std::vector<uint32_t> vals;
    uint32_t cbounds[6] = {0, 0, 0, 0, 0, 0};
    std::vector<uint2> children;         // n - 1
    std::vector<float4> box_lo, box_hi;  // 2n - 1
    std::vector<float> cost;             // 7 (2n - 1)
    std::vector<uint8_t> decision;       // 7 (2n - 1)
    uint32_t root = 0;
};

struct DeviceSceneBuild {
    // in
    cudaStream_t stream = nullptr;
    int device = 0;
    int builder = 1;  // 1 = PLOC, 2 = LBVH
    int ploc_radius = crt::kPlocRadius;
    bool ploc_tail = true;
    // out: the renderer's scene buffers (leaf order) and the leaf-order -> flattened primitive id table
    DeviceBuffer<float4> *d_nodes = nullptr, *d_tris = nullptr, *d_shade = nullptr;
    std::vector<uint32_t> *leaf_flat_ids = nullptr;
    uint32_t num_nodes = 0, depth = 0;
    std::vector<uint32_t> level_begin;     // as Bvh8::level_begin
    SceneGeometry *geometry = nullptr;     // when set (option dynamic_scene): the uploaded geometry is kept there
    int rounds = 0;                        // PLOC rounds
    double build_ms = 0.0;                 // CUDA events around everything after the flattening
    double phase_ms[5] = {0, 0, 0, 0, 0};  // flatten (host wall clock), keys + sort, binary tree, BVH8 emission, packing
    Bvh2Dump *dump = nullptr;              // when set (the test-only check library): the intermediate state of the build

    void run(const crt_scene_t *scene, const crt::FlattenPlan &plan)
    {
        DeviceBuffer<float> d_verts;
        DeviceBuffer<float4> d_shade_in;
        SceneGeometry local;
        const auto t0 = std::chrono::steady_clock::now();
        flatten_on_device(scene, plan, geometry ? *geometry : local, d_verts, d_shade_in);  // (ends with a stream synchronisation)
        phase_ms[0] = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        build_on_device((uint32_t)plan.total_tris, d_verts, d_shade_in);
    }

    // exclusive scan of n items (in place allowed); `scratch` holds the tile sums of every recursion level
    template <typename T>
    void device_scan(const T *in, T *out, uint32_t n, T *scratch)
    {
        const unsigned tiles = (n + crt::kBuildTile - 1) / crt::kBuildTile;
        T *sums = tiles > 1 ? scratch : nullptr;
        crt::k_scan_tile<T><<<tiles, crt::kBuildBlock, 0, stream>>>(in, out, n, sums);
        if (tiles > 1) {
            device_scan<T>(scratch, scratch, tiles, scratch + tiles);
            crt::k_scan_add<T><<<tiles, crt::kBuildBlock, 0, stream>>>(out, n, scratch);
        }
    }
    // Stable LSD radix sort of n (key, value) pairs by the whole 64-bit key (Morton keys use 63 bits): 8 passes of
    // 8 bits, k_radix_hist -> scan of the digit-major histogram -> k_radix_scatter. The pairs end where they started
    // (an even number of passes); keys_tmp / vals_tmp hold every other pass. hist: 256 per tile of n; scratch:
    // scan_scratch_items(256 * tiles).
    void radix_sort(crt::u64 *keys, uint32_t *vals, crt::u64 *keys_tmp, uint32_t *vals_tmp, uint32_t n, uint32_t *hist,
                    uint32_t *scratch)
    {
        const uint32_t tiles = (n + crt::kBuildTile - 1) / crt::kBuildTile;
        crt::u64 *kin = keys, *kout = keys_tmp;
        uint32_t *vin = vals, *vout = vals_tmp;
        for (int shift = 0; shift < 64; shift += 8) {  // 63 key bits
            crt::k_radix_hist<<<tiles, crt::kBuildBlock, 0, stream>>>(kin, n, shift, hist, tiles);
            device_scan<uint32_t>(hist, hist, tiles * 256u, scratch);
            crt::k_radix_scatter<<<tiles, crt::kBuildBlock, 0, stream>>>(kin, vin, kout, vout, n, shift, hist, tiles);
            std::swap(kin, kout);
            std::swap(vin, vout);
        }
    }

    static size_t scan_scratch_items(size_t n)
    {
        size_t total = 0;
        while (n > (size_t)crt::kBuildTile) {
            n = (n + crt::kBuildTile - 1) / crt::kBuildTile;
            total += n;
        }
        return total + 1;
    }

    // The triangle half of flatten_scene on the device: the unique geometries are uploaded once (not once per
    // instance) and k_flatten writes the world-space soup and the shading records in flattened order.
    void flatten_on_device(const crt_scene_t *scene, const crt::FlattenPlan &plan, SceneGeometry &geom,
                           DeviceBuffer<float> &d_verts, DeviceBuffer<float4> &d_shade_in)
    {
        const uint32_t total = (uint32_t)plan.total_tris;
        geom.upload(scene, plan, stream);
        CUDA_CHECK(cudaMemsetAsync(geom.bad.ptr, 0, sizeof(uint32_t), stream));
        d_verts.alloc((size_t)total * 9);
        d_shade_in.alloc((size_t)total * 3);
        int sms = 0;
        CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
        const unsigned g = std::max(1u, std::min((total + crt::kBuildBlock - 1) / crt::kBuildBlock, (uint32_t)sms * 8u));
        crt::k_flatten<<<g, crt::kBuildBlock, 0, stream>>>(geom.segs.ptr, geom.num_segs, geom.xforms.ptr, geom.vert_arena.ptr,
                                                          geom.index_arena.ptr, geom.uv_arena.ptr, total, d_verts.ptr,
                                                          d_shade_in.ptr, geom.bad.ptr);
        uint32_t bad_host = 0u;
        CUDA_CHECK(cudaMemcpyAsync(&bad_host, geom.bad.ptr, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
        CUDA_CHECK(cudaStreamSynchronize(stream));
        if (bad_host) {
            throw std::runtime_error("triangle index out of range");
        }
    }

    void build_on_device(uint32_t n, DeviceBuffer<float> &d_verts, DeviceBuffer<float4> &d_shade_in)
    {
        if (n >= (1u << 30)) {
            throw std::runtime_error("device BVH build: at most 2^30 - 1 triangles");
        }
        int sms = 0;
        CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
        auto grid_for = [&](uint32_t items) {
            return std::max(1u, std::min((items + crt::kBuildBlock - 1) / crt::kBuildBlock, (uint32_t)sms * 8u));
        };
        const EventSet events(5);
        const cudaEvent_t ev0 = events[0], ev1 = events[1], ev_sorted = events[2], ev_tree = events[3], ev_emitted = events[4];
        const uint32_t num_b2 = 2 * n - 1, max_nodes = std::max(1u, n - 1);
        DeviceArena arena;
        ArenaBuf<float4> tri_lo(arena), tri_hi(arena), box_lo(arena), box_hi(arena), nodes_tmp(arena);
        ArenaBuf<uint32_t> cbounds(arena), vals0(arena), vals1(arena), hist(arena), d_parent(arena), arrivals(arena), slots(arena),
            work0(arena), work1(arena), tri_order(arena), clusters0(arena), clusters1(arena), nn(arena);
        ArenaBuf<crt::u64> keys0(arena), keys1(arena), counts(arena), offsets(arena), scan_scratch(arena);
        ArenaBuf<uint2> d_children(arena);
        ArenaBuf<float> cost(arena);
        ArenaBuf<uint8_t> decision(arena);
        static_assert(sizeof(crt::TriShade) == 3 * sizeof(float4), "TriShade = 3 float4");
        CUDA_CHECK(cudaEventRecord(ev0, stream));
        const uint32_t tiles = (n + crt::kBuildTile - 1) / crt::kBuildTile;
        auto carve = [&] {
            tri_lo.alloc(n);
            tri_hi.alloc(n);
            cbounds.alloc(6);
            keys0.alloc(n);
            keys1.alloc(n);
            vals0.alloc(n);
            vals1.alloc(n);
            hist.alloc((size_t)tiles * 256);
            d_children.alloc(n);
            box_lo.alloc(num_b2);
            box_hi.alloc(num_b2);
            cost.alloc((size_t)num_b2 * 7);
            decision.alloc((size_t)num_b2 * 7);
            slots.alloc((size_t)max_nodes * 8);
            work0.alloc(max_nodes);
            work1.alloc(max_nodes);
            counts.alloc(n);
            offsets.alloc(n);
            scan_scratch.alloc(std::max(scan_scratch_items(n), (scan_scratch_items((size_t)tiles * 256) + 1) / 2 + 1));
            nodes_tmp.alloc((size_t)max_nodes * 5);
            tri_order.alloc(n);
            if (builder == 2) {
                d_parent.alloc(num_b2);
                arrivals.alloc(n);
            } else {
                clusters0.alloc(n);
                clusters1.alloc(n);
                nn.alloc(n);
            }
        };
        carve();
        arena.commit();
        carve();
        const uint32_t cb_init[6] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u};
        CUDA_CHECK(cudaMemcpyAsync(cbounds.ptr, cb_init, sizeof(cb_init), cudaMemcpyHostToDevice, stream));

        crt::Lbvh b;
        b.n = n;
        b.verts = d_verts.ptr;
        b.tri_lo = tri_lo.ptr;
        b.tri_hi = tri_hi.ptr;
        b.cbounds = cbounds.ptr;
        b.children = d_children.ptr;
        b.parent = d_parent.ptr;
        b.box_lo = box_lo.ptr;
        b.box_hi = box_hi.ptr;
        b.arrivals = arrivals.ptr;
        b.cost = cost.ptr;
        b.decision = decision.ptr;
        const unsigned g = grid_for(n);
        crt::k_lbvh_bounds<<<g, crt::kBuildBlock, 0, stream>>>(b);
        crt::k_lbvh_keys<<<g, crt::kBuildBlock, 0, stream>>>(b, keys0.ptr, vals0.ptr);
        radix_sort(keys0.ptr, vals0.ptr, keys1.ptr, vals1.ptr, n, hist.ptr, reinterpret_cast<uint32_t *>(scan_scratch.ptr));
        crt::u64 *const kin = keys0.ptr;  // (eight passes: the sorted pairs are back in keys0 / vals0)
        uint32_t *const vin = vals0.ptr;
        CUDA_CHECK(cudaEventRecord(ev_sorted, stream));
        crt::u64 *h_tail = nullptr;  // pinned: last offset + last count of a scan = its total
        CUDA_CHECK(cudaMallocHost(&h_tail, 2 * sizeof(crt::u64)));
        struct FreeHost {
            void *p;
            ~FreeHost() { cudaFreeHost(p); }
        } free_tail{h_tail};
        auto scan_total = [&](uint32_t items) {  // enqueue after device_scan(counts -> offsets); valid after a sync
            CUDA_CHECK(cudaMemcpyAsync(h_tail, offsets.ptr + (items - 1), sizeof(crt::u64), cudaMemcpyDeviceToHost, stream));
            CUDA_CHECK(cudaMemcpyAsync(h_tail + 1, counts.ptr + (items - 1), sizeof(crt::u64), cudaMemcpyDeviceToHost, stream));
        };
        uint32_t root = 0u;  // a single triangle: the leaf is the root
        if (builder == 2) {
            crt::k_bvh2_leaves<<<g, crt::kBuildBlock, 0, stream>>>(b, vin, nullptr);
            if (n > 1) {
                crt::k_lbvh_hierarchy<<<grid_for(n - 1), crt::kBuildBlock, 0, stream>>>(b, kin);
                crt::k_lbvh_refit<<<g, crt::kBuildBlock, 0, stream>>>(b);
                root = n;
            }
        } else {
            uint32_t *cl = clusters0.ptr, *cl_next = clusters1.ptr;
            crt::k_bvh2_leaves<<<g, crt::kBuildBlock, 0, stream>>>(b, vin, cl);
            uint32_t m = n, nodes_made = 0;
            rounds = 0;
            while (m > 1) {
                if (ploc_tail && m <= (uint32_t)crt::kPlocTailMax) {
                    // the remaining rounds in one block (k_ploc_tail): no more round trips
                    uint32_t *rounds_dev = nn.ptr;  // free from here on
                    uint32_t rounds_host = (uint32_t)rounds;
                    CUDA_CHECK(cudaMemcpyAsync(rounds_dev, &rounds_host, sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
                    crt::k_ploc_tail<<<1, crt::kBuildBlock, 0, stream>>>(b, cl, m, nodes_made, ploc_radius, rounds_dev);
                    CUDA_CHECK(cudaMemcpyAsync(&rounds_host, rounds_dev, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
                    CUDA_CHECK(cudaStreamSynchronize(stream));
                    rounds = (int)rounds_host;
                    nodes_made += m - 1;
                    m = 1;
                    break;
                }
                // (an adversarial input can leave one mutual pair per round; after 256 rounds neighbours are paired up)
                const int forced = rounds >= 256 ? 1 : 0;
                const unsigned gm = (m + crt::kBuildBlock - 1) / crt::kBuildBlock;
                crt::k_ploc_nn<<<gm, crt::kBuildBlock, 0, stream>>>(b, cl, m, nn.ptr, ploc_radius, forced);
                crt::k_ploc_mark<<<grid_for(m), crt::kBuildBlock, 0, stream>>>(nn.ptr, m, counts.ptr);
                device_scan<crt::u64>(counts.ptr, offsets.ptr, m, scan_scratch.ptr);
                scan_total(m);
                crt::k_ploc_merge<<<grid_for(m), crt::kBuildBlock, 0, stream>>>(b, cl, nn.ptr, m, offsets.ptr, nodes_made, cl_next);
                CUDA_CHECK(cudaStreamSynchronize(stream));
                const crt::u64 total = h_tail[0] + h_tail[1];
                const uint32_t merged = (uint32_t)total, left = (uint32_t)(total >> 32);
                if (merged == 0 || left + merged != m) {
                    throw DeviceBuildFailure("device BVH build: a PLOC round made no progress");
                }
                nodes_made += merged;
                m = left;
                std::swap(cl, cl_next);
                ++rounds;
            }
            if (n > 1) {
                if (nodes_made != n - 1) {
                    throw DeviceBuildFailure("device BVH build: PLOC made " + std::to_string(nodes_made) + " of " +
                                             std::to_string(n - 1) + " nodes");
                }
                root = n + (n - 2);
            }
        }

        // BVH8 levels: the host only learns each level's size
        CUDA_CHECK(cudaEventRecord(ev_tree, stream));
        CUDA_CHECK(cudaMemcpyAsync(work0.ptr, &root, sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
        uint32_t *work = work0.ptr, *next_work = work1.ptr;
        uint32_t node_begin = 0, count = 1, tri_total = 0;
        depth = 0;
        level_begin.clear();
        while (count) {
            ++depth;
            level_begin.push_back(node_begin);
            if ((size_t)node_begin + count > max_nodes) {
                throw DeviceBuildFailure("device BVH build: node count exceeds its bound");
            }
            crt::LevelArgs lv;
            lv.work = work;
            lv.count = count;
            lv.node_begin = node_begin;
            lv.next_begin = node_begin + count;
            lv.tri_begin = tri_total;
            lv.slots = slots.ptr;
            lv.counts = counts.ptr;
            lv.offsets = offsets.ptr;
            lv.next_work = next_work;
            lv.nodes = reinterpret_cast<crt::Bvh8Node *>(nodes_tmp.ptr);
            lv.tri_order = tri_order.ptr;
            const unsigned gl = grid_for(count);
            crt::k_plan_level<<<gl, crt::kBuildBlock, 0, stream>>>(b, lv);
            device_scan<crt::u64>(counts.ptr, offsets.ptr, count, scan_scratch.ptr);
            scan_total(count);
            crt::k_emit_level<<<gl, crt::kBuildBlock, 0, stream>>>(b, lv, vin);
            CUDA_CHECK(cudaStreamSynchronize(stream));
            const crt::u64 total = h_tail[0] + h_tail[1];
            node_begin += count;
            count = (uint32_t)(total >> 32);
            tri_total += (uint32_t)total;
            std::swap(work, next_work);
        }
        if (tri_total != n) {
            throw DeviceBuildFailure("device BVH build: emitted " + std::to_string(tri_total) + " of " + std::to_string(n) +
                                     " triangles");
        }
        if (depth + 2 > CRT_STACK_SIZE) {
            throw DeviceBuildFailure("device BVH build: BVH8 depth " + std::to_string(depth) + " exceeds the traversal stack");
        }
        CUDA_CHECK(cudaEventRecord(ev_emitted, stream));
        num_nodes = node_begin;
        level_begin.push_back(num_nodes);
        d_nodes->alloc((size_t)num_nodes * 5);
        CUDA_CHECK(cudaMemcpyAsync(d_nodes->ptr, nodes_tmp.ptr, (size_t)num_nodes * 80, cudaMemcpyDeviceToDevice, stream));
        d_tris->alloc((size_t)n * 3);
        d_shade->alloc((size_t)n * 3);
        crt::k_pack_leaf_order<<<g, crt::kBuildBlock, 0, stream>>>(d_verts.ptr, d_shade_in.ptr, tri_order.ptr, n, d_tris->ptr,
                                                                  d_shade->ptr);
        CUDA_CHECK(cudaEventRecord(ev1, stream));
        CUDA_CHECK(cudaGetLastError());
        std::vector<uint32_t> order(n);
        CUDA_CHECK(cudaMemcpyAsync(order.data(), tri_order.ptr, (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
        if (dump) {
            auto fetch = [&](auto &dst, const auto *src, size_t count) {
                dst.resize(count);
                CUDA_CHECK(cudaMemcpyAsync(dst.data(), src, count * sizeof(*src), cudaMemcpyDeviceToHost, stream));
            };
            fetch(dump->keys, kin, n);
            fetch(dump->vals, vin, n);
            fetch(dump->children, d_children.ptr, n - 1);
            fetch(dump->box_lo, box_lo.ptr, num_b2);
            fetch(dump->box_hi, box_hi.ptr, num_b2);
            fetch(dump->cost, cost.ptr, (size_t)num_b2 * 7);
            fetch(dump->decision, decision.ptr, (size_t)num_b2 * 7);
            CUDA_CHECK(cudaMemcpyAsync(dump->cbounds, cbounds.ptr, sizeof(dump->cbounds), cudaMemcpyDeviceToHost, stream));
            dump->root = root;
        }
        CUDA_CHECK(cudaStreamSynchronize(stream));
        float t = 0.f;
        CUDA_CHECK(cudaEventElapsedTime(&t, ev0, ev1));
        build_ms = t;
        CUDA_CHECK(cudaEventElapsedTime(&t, ev0, ev_sorted));
        phase_ms[1] = t;
        CUDA_CHECK(cudaEventElapsedTime(&t, ev_sorted, ev_tree));
        phase_ms[2] = t;
        CUDA_CHECK(cudaEventElapsedTime(&t, ev_tree, ev_emitted));
        phase_ms[3] = t;
        CUDA_CHECK(cudaEventElapsedTime(&t, ev_emitted, ev1));
        phase_ms[4] = t;
        leaf_flat_ids->resize(n);
        for (uint32_t i = 0; i < n; ++i) {
            if (order[i] >= n) {
                throw std::runtime_error("device BVH build: triangle order out of range");
            }
            (*leaf_flat_ids)[i] = order[i];  // the flattened primitive id IS the index in flattened order
        }
    }
};

}  // namespace crt_host
