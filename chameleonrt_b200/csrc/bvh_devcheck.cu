// bvh_devcheck.cu — TEST-ONLY shared library (libcrt_bvh_devcheck.so).
//
// The device set_scene (scene_device_build.cuh driving the kernels of bvh8_device.cuh) stage by stage, through the
// product's own driver code with the product's NVFLAGS: the exclusive scan (DeviceSceneBuild::device_scan), the radix
// sort (DeviceSceneBuild::radix_sort) and the whole build (DeviceSceneBuild::run) with the renderer's output buffers
// plus the binary tree behind them (Bvh2Dump). tests/test_bvh_build_exact.py compares each with a plain restatement.
// bvhdev_update runs a set_scene with option dynamic_scene (either builder, or the host builder) and a commit of staged
// updates through the renderer's own update driver (crt_host::SceneUpdate, scene_update.cuh): tests/test_dynamic_scene.py.
// This file holds no launch and no CUDA syntax, so tests/simt_emu/build.py compiles the same file for the host
// (libcrt_bvh_devcheck_simt.so, every launch under the SIMT emulation). Not linked into libcrt_cuda_core.so.
#include <cstdint>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/crt_scene.h"
#include "cuda_host_utils.h"
#include "host_scene.h"
#include "scene_device_build.cuh"
#include "scene_update.cuh"

namespace {

thread_local std::string g_err;

using crt_host::DeviceBuffer;

// One device build: the renderer's buffers, copied back, and the binary tree behind them.
struct BuildResult {
    uint32_t n = 0, num_nodes = 0, depth = 0, rounds = 0;
    std::vector<float4> nodes, tris, shade;
    std::vector<uint32_t> leaf_flat_ids;
    crt_host::Bvh2Dump dump;
};

// A set_scene with option dynamic_scene and one commit: the renderer's buffers before and after.
struct UpdateResult {
    uint32_t n = 0, num_nodes = 0, depth = 0, launches = 0;
    std::vector<float4> nodes[2], tris[2], shade[2];  // [0] after set_scene, [1] after the commit
    std::vector<uint32_t> leaf_flat_ids, levels;
};

template <typename T>
std::vector<T> download(const DeviceBuffer<T> &b)
{
    std::vector<T> out(b.count);
    if (b.count) {
        CUDA_CHECK(cudaMemcpyAsync(out.data(), b.ptr, b.count * sizeof(T), cudaMemcpyDeviceToHost, nullptr));
    }
    return out;
}

template <typename T>
void scan(const T *in, uint32_t n, T *out)
{
    crt_host::DeviceSceneBuild job;
    DeviceBuffer<T> d, scratch;
    d.upload(in, n, nullptr);
    scratch.alloc(crt_host::DeviceSceneBuild::scan_scratch_items(n));
    job.device_scan<T>(d.ptr, d.ptr, n, scratch.ptr);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(out, d.ptr, (size_t)n * sizeof(T), cudaMemcpyDeviceToHost, nullptr));
    CUDA_CHECK(cudaStreamSynchronize(nullptr));
}

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

}  // namespace

extern "C" {

const char *bvhdev_last_error() { return g_err.c_str(); }

// exclusive scans, in -> out (n >= 1)
int bvhdev_scan_u32(const uint32_t *in, uint32_t n, uint32_t *out)
{
    return guarded([&] { scan<uint32_t>(in, n, out); });
}
int bvhdev_scan_u64(const uint64_t *in, uint32_t n, uint64_t *out)
{
    static_assert(sizeof(crt::u64) == sizeof(uint64_t), "u64");
    return guarded([&] { scan<crt::u64>(reinterpret_cast<const crt::u64 *>(in), n, reinterpret_cast<crt::u64 *>(out)); });
}

// the build's radix sort of (key, value) pairs by the 64-bit key, stable, in place (n >= 1)
int bvhdev_sort_pairs(uint64_t *keys, uint32_t *vals, uint32_t n)
{
    return guarded([&] {
        crt_host::DeviceSceneBuild job;
        const uint32_t tiles = (n + crt::kBuildTile - 1) / crt::kBuildTile;
        DeviceBuffer<crt::u64> k, k_tmp;
        DeviceBuffer<uint32_t> v, v_tmp, hist, scratch;
        k.upload(reinterpret_cast<const crt::u64 *>(keys), n, nullptr);
        v.upload(vals, n, nullptr);
        k_tmp.alloc(n);
        v_tmp.alloc(n);
        hist.alloc((size_t)tiles * 256);
        scratch.alloc(crt_host::DeviceSceneBuild::scan_scratch_items((size_t)tiles * 256));
        job.radix_sort(k.ptr, v.ptr, k_tmp.ptr, v_tmp.ptr, n, hist.ptr, scratch.ptr);
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaMemcpyAsync(keys, k.ptr, (size_t)n * 8, cudaMemcpyDeviceToHost, nullptr));
        CUDA_CHECK(cudaMemcpyAsync(vals, v.ptr, (size_t)n * 4, cudaMemcpyDeviceToHost, nullptr));
        CUDA_CHECK(cudaStreamSynchronize(nullptr));
    });
}

// set_scene on the device (builder 1 = PLOC, 2 = LBVH). info out: n, BVH8 nodes, depth, PLOC rounds, BVH2 root.
// Returns a handle for bvhdev_fetch, or null (bvhdev_last_error).
void *bvhdev_build(const crt_scene_t *scene, int builder, int ploc_tail, int ploc_radius, uint32_t *info)
{
    auto res = std::make_unique<BuildResult>();
    const int rc = guarded([&] {
        crt::FlattenPlan plan;
        crt::plan_flatten(scene, plan);
        crt::check_triangle_count(plan.total_tris);
        if (plan.total_tris == 0) {
            throw std::runtime_error("bvhdev_build: the scene has no triangles");
        }
        DeviceBuffer<float4> d_nodes, d_tris, d_shade;
        crt_host::DeviceSceneBuild job;
        job.builder = builder;
        job.ploc_tail = ploc_tail != 0;
        job.ploc_radius = ploc_radius;
        job.d_nodes = &d_nodes;
        job.d_tris = &d_tris;
        job.d_shade = &d_shade;
        job.leaf_flat_ids = &res->leaf_flat_ids;
        job.dump = &res->dump;
        job.run(scene, plan);
        res->n = (uint32_t)plan.total_tris;
        res->num_nodes = job.num_nodes;
        res->depth = job.depth;
        res->rounds = (uint32_t)job.rounds;
        res->nodes = download(d_nodes);
        res->tris = download(d_tris);
        res->shade = download(d_shade);
        CUDA_CHECK(cudaStreamSynchronize(nullptr));
    });
    if (rc) {
        return nullptr;
    }
    info[0] = res->n;
    info[1] = res->num_nodes;
    info[2] = res->depth;
    info[3] = res->rounds;
    info[4] = res->dump.root;
    return res.release();
}

// Copies one array of a build into dst, sized from bvhdev_build's info: 0 nodes (80 B per node), 1 packed triangles and
// 2 shading records (48 B per triangle, leaf order), 3 leaf_flat_ids (n), 4 sorted keys (n u64), 5 sorted triangle ids
// (n), 6 centroid bounds (6 ordered uints), 7 children (n - 1 uint2), 8 box_lo and 9 box_hi (2n - 1 float4),
// 10 cost (7 (2n - 1) floats), 11 decision (7 (2n - 1) bytes). Returns the bytes copied, -1 for an unknown field.
long long bvhdev_fetch(void *h, int field, void *dst)
{
    const BuildResult &r = *static_cast<const BuildResult *>(h);
    auto put = [&](const auto &v) {
        const size_t bytes = v.size() * sizeof(v[0]);
        if (bytes) {
            std::memcpy(dst, v.data(), bytes);
        }
        return (long long)bytes;
    };
    switch (field) {
    case 0: return put(r.nodes);
    case 1: return put(r.tris);
    case 2: return put(r.shade);
    case 3: return put(r.leaf_flat_ids);
    case 4: return put(r.dump.keys);
    case 5: return put(r.dump.vals);
    case 6: std::memcpy(dst, r.dump.cbounds, sizeof(r.dump.cbounds)); return (long long)sizeof(r.dump.cbounds);
    case 7: return put(r.dump.children);
    case 8: return put(r.dump.box_lo);
    case 9: return put(r.dump.box_hi);
    case 10: return put(r.dump.cost);
    case 11: return put(r.dump.decision);
    default: return -1;
    }
}

void bvhdev_free(void *h) { delete static_cast<BuildResult *>(h); }

// set_scene of `scene` with option dynamic_scene (builder 0 = the host builder, 1 = PLOC, 2 = LBVH), then every
// instance's transform and every geometry's vertices of `moved` (the same topology) staged and committed. info out: n,
// BVH8 nodes, depth, commit launches, levels + 1. Returns a handle for bvhdev_fetch_update, or null (bvhdev_last_error).
void *bvhdev_update(const crt_scene_t *scene, const crt_scene_t *moved, int builder, uint32_t *info)
{
    auto res = std::make_unique<UpdateResult>();
    const int rc = guarded([&] {
        crt::FlattenPlan plan;
        crt::plan_flatten(scene, plan);
        crt::check_triangle_count(plan.total_tris);
        DeviceBuffer<float4> d_nodes, d_tris, d_shade;
        crt_host::SceneUpdate upd;
        std::vector<uint32_t> flat_ids, levels;
        if (builder == 0) {
            crt::SceneRecords rec;
            crt::pack_scene(scene, 0, rec);
            d_nodes.upload(reinterpret_cast<const float4 *>(rec.bvh.nodes.data()), rec.bvh.nodes.size() * 5, nullptr);
            d_tris.upload(reinterpret_cast<const float4 *>(rec.tris.data()), rec.tris.size() / 4, nullptr);
            d_shade.upload(reinterpret_cast<const float4 *>(rec.shade.data()), rec.shade.size() * 3, nullptr);
            upd.geometry->upload(scene, plan, nullptr);
            flat_ids = rec.leaf_flat_ids;
            levels = rec.bvh.level_begin;
            res->depth = rec.bvh.max_depth;
        } else {
            crt_host::DeviceSceneBuild job;
            job.builder = builder;
            job.d_nodes = &d_nodes;
            job.d_tris = &d_tris;
            job.d_shade = &d_shade;
            job.leaf_flat_ids = &flat_ids;
            job.geometry = upd.geometry.get();
            job.run(scene, plan);
            levels = job.level_begin;
            res->depth = job.depth;
        }
        upd.keep(scene, flat_ids, levels, nullptr);
        res->n = (uint32_t)flat_ids.size();
        res->num_nodes = (uint32_t)(d_nodes.count / 5);
        res->nodes[0] = download(d_nodes);
        res->tris[0] = download(d_tris);
        res->shade[0] = download(d_shade);
        std::vector<float> xf((size_t)moved->num_instances * 16);
        for (uint32_t i = 0; i < moved->num_instances; ++i) {
            std::memcpy(&xf[(size_t)i * 16], moved->instances[i].transform, 16 * sizeof(float));
        }
        upd.stage_instances(0, moved->num_instances, xf.data());
        for (uint32_t m = 0; m < moved->num_meshes; ++m) {
            for (uint32_t g = 0; g < moved->meshes[m].num_geometries; ++g) {
                const crt_geometry_t &geom = moved->meshes[m].geometries[g];
                upd.stage_vertices(m, g, geom.vertices, geom.num_vertices);
            }
        }
        res->launches = (uint32_t)upd.commit(d_nodes.ptr, d_tris.ptr, d_shade.ptr, nullptr, 0);
        res->nodes[1] = download(d_nodes);
        res->tris[1] = download(d_tris);
        res->shade[1] = download(d_shade);
        res->leaf_flat_ids = flat_ids;
        res->levels = levels;
        CUDA_CHECK(cudaStreamSynchronize(nullptr));
        CUDA_CHECK(cudaGetLastError());
    });
    if (rc) {
        return nullptr;
    }
    info[0] = res->n;
    info[1] = res->num_nodes;
    info[2] = res->depth;
    info[3] = res->launches;
    info[4] = (uint32_t)res->levels.size();
    return res.release();
}

// One array of bvhdev_update's result: 0 / 1 / 2 nodes / packed triangles / shading records after set_scene, 3 / 4 / 5
// the same after the commit, 6 leaf_flat_ids, 7 the level boundaries (Bvh8::level_begin). Returns the bytes copied,
// -1 for an unknown field.
long long bvhdev_fetch_update(void *h, int field, void *dst)
{
    const UpdateResult &r = *static_cast<const UpdateResult *>(h);
    auto put = [&](const auto &v) {
        const size_t bytes = v.size() * sizeof(v[0]);
        if (bytes) {
            std::memcpy(dst, v.data(), bytes);
        }
        return (long long)bytes;
    };
    switch (field) {
    case 0: case 3: return put(r.nodes[field / 3]);
    case 1: case 4: return put(r.tris[field / 3]);
    case 2: case 5: return put(r.shade[field / 3]);
    case 6: return put(r.leaf_flat_ids);
    case 7: return put(r.levels);
    default: return -1;
    }
}

void bvhdev_free_update(void *h) { delete static_cast<UpdateResult *>(h); }
}
