// hostcheck.cpp — TEST-ONLY shared library (libcrt_bvh8_hostcheck.so).
//
// Runs the product's host-side scene flattening + BVH8 builder and then the *host
// instantiation* of bvh8_trace on CPU, so that the builder and the 80-byte node format can
// be validated against the CPU oracle on a machine without a GPU. It is not linked into
// libcrt_cuda_core.so and render() cannot reach it.
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "bvh8.h"
#include "bvh8_traverse.h"
#include "host_scene.h"

namespace {
struct HostCheck {
    crt::SceneRecords rec;
};
std::string g_err;
}  // namespace

extern "C" {

const char *crt_hostcheck_last_error()
{
    return g_err.c_str();
}

void *crt_hostcheck_create(const crt_scene_t *scene, int threads)
{
    try {
        auto *h = new HostCheck();
        crt::pack_scene(scene, threads, h->rec);
        return h;
    } catch (const std::exception &e) {
        g_err = e.what();
        return nullptr;
    }
}

void crt_hostcheck_destroy(void *p)
{
    delete static_cast<HostCheck *>(p);
}

// out: num_nodes, num_tris, max_depth, sah_cost*1000, build_ms
void crt_hostcheck_stats(void *p, double *out5)
{
    HostCheck *h = static_cast<HostCheck *>(p);
    out5[0] = (double)h->rec.bvh.nodes.size();
    out5[1] = (double)h->rec.bvh.tri_order.size();
    out5[2] = (double)h->rec.bvh.max_depth;
    out5[3] = h->rec.bvh.sah_cost;
    out5[4] = h->rec.bvh.build_seconds * 1e3;
}

// FNV-1a over the node array and the triangle order: lets tests assert that builder changes
// (threading, memory layout) leave the emitted BVH8 byte-identical
uint64_t crt_hostcheck_digest(void *p)
{
    HostCheck *h = static_cast<HostCheck *>(p);
    uint64_t d = 1469598103934665603ull;
    auto mix = [&](const void *data, size_t n) {
        const unsigned char *b = static_cast<const unsigned char *>(data);
        for (size_t i = 0; i < n; ++i) {
            d = (d ^ b[i]) * 1099511628211ull;
        }
    };
    mix(h->rec.bvh.nodes.data(), h->rec.bvh.nodes.size() * sizeof(crt::Bvh8Node));
    mix(h->rec.bvh.tri_order.data(), h->rec.bvh.tri_order.size() * sizeof(uint32_t));
    return d;
}

// The host-built scene as set_scene uploads it (sizes from crt_hostcheck_stats): nodes (80 B per node), tri_order (leaf
// order -> flattened triangle), packed triangles (12 floats per triangle) and shading records (48 B per triangle), both
// in leaf order. Any pointer may be null.
void crt_hostcheck_export(void *p, void *nodes, uint32_t *tri_order, float *tris, void *shade)
{
    const HostCheck *h = static_cast<const HostCheck *>(p);
    const size_t n = h->rec.bvh.tri_order.size();
    if (nodes) {
        std::memcpy(nodes, h->rec.bvh.nodes.data(), h->rec.bvh.nodes.size() * sizeof(crt::Bvh8Node));
    }
    if (tri_order && n) {
        std::memcpy(tri_order, h->rec.bvh.tri_order.data(), n * sizeof(uint32_t));
    }
    if (tris && n) {
        std::memcpy(tris, h->rec.tris.data(), n * 12 * sizeof(float));
    }
    if (shade && n) {
        std::memcpy(shade, h->rec.shade.data(), n * sizeof(crt::TriShade));
    }
}

// rays: n*8 floats; hits: n*4 floats {t,u,v,bits(flat id)}; normals (optional) n*3;
// counters (optional) n*2 uint32 {nodes visited, triangles tested}
void crt_hostcheck_trace(void *p, const float *rays, uint64_t n, int any_hit, float *hits, float *normals,
                         uint32_t *counters)
{
    HostCheck *h = static_cast<HostCheck *>(p);
    const float4 *nodes = reinterpret_cast<const float4 *>(h->rec.bvh.nodes.data());
    const float4 *tris = reinterpret_cast<const float4 *>(h->rec.tris.data());
    for (uint64_t i = 0; i < n; ++i) {
        crt::Ray r;
        std::memcpy(&r, rays + 8 * i, 32);
        crt::HitRecord hit;
        crt::TraversalCounters cnt;
        if (any_hit) {
            // any_hit == 2: children in reverse octant order (what the kernels do for shadow rays)
            crt::bvh8_trace<true, true>(nodes, tris, r, hit, &cnt, any_hit == 2);
        } else {
            crt::bvh8_trace<false, true>(nodes, tris, r, hit, &cnt);
        }
        float *o = hits + 4 * i;
        o[0] = hit.t;
        o[1] = hit.u;
        o[2] = hit.v;
        std::memcpy(&o[3], &hit.flat, 4);
        if (normals) {
            for (int k = 0; k < 3; ++k) {
                normals[3 * i + k] = hit.tri == 0xffffffffu ? 0.f : h->rec.shade[hit.tri].n[k];
            }
        }
        if (counters) {
            counters[2 * i] = cnt.nodes;
            counters[2 * i + 1] = cnt.tris;
        }
    }
}
}
