// bvh_devcheck.cu — TEST-ONLY shared library (libcrt_bvh_devcheck.so).
//
// The device set_scene (scene_device_build.cuh driving the kernels of bvh8_device.cuh) stage by stage, through the
// product's own driver code with the product's NVFLAGS: the exclusive scan (DeviceSceneBuild::device_scan), the radix
// sort (DeviceSceneBuild::radix_sort) and the whole build (DeviceSceneBuild::run) with the renderer's output buffers
// plus the binary tree behind them (Bvh2Dump). tests/test_bvh_build_exact.py compares each with a plain restatement.
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
}
