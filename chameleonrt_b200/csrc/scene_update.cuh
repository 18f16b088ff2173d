// scene_update.cuh — scene updates between frames (option "dynamic_scene"; crtc_update_instances, crtc_update_vertices,
// crtc_commit_scene): new instance transforms and new vertex positions over the SAME topology, applied on the device
// without a new set_scene. Included by scene_device_build.cuh too, whose k_flatten reads the same SceneGeometry. Every
// launch here goes through crt_host::launch, so that the host build of the renderer (tests/simt_emu) compiles this
// header unchanged.
//
//   k_reflatten     one thread per leaf-order triangle: the flattening of k_flatten (dev_flatten_triangle) for its
//                   flattened id, written straight into the renderer's triangle and shading records in leaf order, plus
//                   the triangle's world-space box (from the world vertices)
//   k_bvh8_refit    one launch per BVH8 level, deepest first, one thread per node: every slot's box is the float union of
//                   its 1-3 leaf triangles' boxes or its inner child's box (written by the previous launch), the node's
//                   box the union of its slots'; the quantisation frame and the child boxes are recomputed with
//                   k_emit_level's arithmetic (bvh8_node_frame, bvh8_quantise_child). child_base, tri_base, meta and
//                   imask stay.
//
// Both builders make every node's box the exact float union of its triangles' boxes, and the refit recomputes exactly
// that union, so a commit reproduces the node bytes the same tree would get from a build over the moved triangles, and
// the records a set_scene of the moved scene would produce. Closest hits do not depend on the tree (DESIGN.md §2), so
// frames after a commit equal frames of a fresh set_scene of the updated scene. No block waits on another: every level
// is its own launch (the rule stated at the top of bvh8_device.cuh).
#pragma once

#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/crt_scene.h"
#include "bvh8_device.cuh"
#include "cuda_host_utils.h"
#include "host_scene.h"

namespace crt {

// tri_box: 2 float4 per leaf-order triangle, {lo.xyz, 0}, {hi.xyz, 0}
__global__ void __launch_bounds__(kBuildBlock) k_reflatten(const DevSegment *segs, uint32_t num_segs, const float *xforms,
                                                           const float *vert_arena, const uint32_t *index_arena,
                                                           const float *uv_arena, const uint32_t *leaf_flat_ids, uint32_t n,
                                                           float4 *tris_out, float4 *shade_out, float4 *tri_box)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t f = leaf_flat_ids[i];
        const DevSegment seg = segs[dev_find_segment(segs, num_segs, f)];
        float w[9];
        float4 shade[3];
        dev_flatten_triangle(seg, f, xforms, vert_arena, index_arena, uv_arena, w, shade);  // (indices checked by set_scene)
        // = k_pack_leaf_order: {v0, flat id}, {v1 - v0, 0}, {v2 - v0, 0}
        tris_out[(size_t)i * 3] = make_float4(w[0], w[1], w[2], __uint_as_float(f));
        tris_out[(size_t)i * 3 + 1] = make_float4(w[3] - w[0], w[4] - w[1], w[5] - w[2], 0.f);
        tris_out[(size_t)i * 3 + 2] = make_float4(w[6] - w[0], w[7] - w[1], w[8] - w[2], 0.f);
        for (int k = 0; k < 3; ++k) {
            shade_out[(size_t)i * 3 + k] = shade[k];
        }
        // = k_lbvh_bounds
        tri_box[(size_t)i * 2] = make_float4(fminf(w[0], fminf(w[3], w[6])), fminf(w[1], fminf(w[4], w[7])),
                                             fminf(w[2], fminf(w[5], w[8])), 0.f);
        tri_box[(size_t)i * 2 + 1] = make_float4(fmaxf(w[0], fmaxf(w[3], w[6])), fmaxf(w[1], fmaxf(w[4], w[7])),
                                                 fmaxf(w[2], fmaxf(w[5], w[8])), 0.f);
    }
}

// Nodes [begin, begin + count) of one level; node_box: 2 float4 per node, as tri_box. The deeper levels are done.
__global__ void __launch_bounds__(kBuildBlock) k_bvh8_refit(uint4 *nodes, uint32_t begin, uint32_t count, const float4 *tri_box,
                                                            float4 *node_box)
{
    for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < count; w += gridDim.x * blockDim.x) {
        const uint32_t ni = begin + w;
        alignas(16) Bvh8Node node;
        uint4 *q = reinterpret_cast<uint4 *>(&node);
        for (int k = 0; k < 5; ++k) {
            q[k] = nodes[(size_t)ni * 5 + k];
        }
        const float inf = __uint_as_float(0x7f800000u);
        float blo[3] = {inf, inf, inf}, bhi[3] = {-inf, -inf, -inf};
        float slo[8][3], shi[8][3];
#pragma unroll
        for (int s = 0; s < 8; ++s) {
            const uint32_t meta = node.meta[s];
            float4 lo = make_float4(0.f, 0.f, 0.f, 0.f), hi = lo;
            if (meta != 0u) {
                if ((node.imask >> s) & 1u) {
                    const uint32_t c = node.child_base + (uint32_t)__popc(node.imask & ((1u << s) - 1u));
                    lo = node_box[(size_t)c * 2];
                    hi = node_box[(size_t)c * 2 + 1];
                } else {
                    const uint32_t t = node.tri_base + (meta & 31u), cnt = (uint32_t)__popc(meta >> 5);
                    lo = tri_box[(size_t)t * 2];
                    hi = tri_box[(size_t)t * 2 + 1];
                    for (uint32_t k = 1; k < cnt; ++k) {
                        const float4 l2 = tri_box[(size_t)(t + k) * 2], h2 = tri_box[(size_t)(t + k) * 2 + 1];
                        lo = make_float4(fminf(lo.x, l2.x), fminf(lo.y, l2.y), fminf(lo.z, l2.z), 0.f);
                        hi = make_float4(fmaxf(hi.x, h2.x), fmaxf(hi.y, h2.y), fmaxf(hi.z, h2.z), 0.f);
                    }
                }
                blo[0] = fminf(blo[0], lo.x);
                blo[1] = fminf(blo[1], lo.y);
                blo[2] = fminf(blo[2], lo.z);
                bhi[0] = fmaxf(bhi[0], hi.x);
                bhi[1] = fmaxf(bhi[1], hi.y);
                bhi[2] = fmaxf(bhi[2], hi.z);
            }
            slo[s][0] = lo.x;
            slo[s][1] = lo.y;
            slo[s][2] = lo.z;
            shi[s][0] = hi.x;
            shi[s][1] = hi.y;
            shi[s][2] = hi.z;
        }
        double step[3];
        bvh8_node_frame(blo, bhi, node, step);
#pragma unroll
        for (int s = 0; s < 8; ++s) {
            if (node.meta[s] != 0u) {
                uint8_t qlo[3], qhi[3];
                bvh8_quantise_child(node, step, slo[s], shi[s], qlo, qhi);
                node.qlo_x[s] = qlo[0];
                node.qlo_y[s] = qlo[1];
                node.qlo_z[s] = qlo[2];
                node.qhi_x[s] = qhi[0];
                node.qhi_y[s] = qhi[1];
                node.qhi_z[s] = qhi[2];
            }
        }
        for (int k = 0; k < 5; ++k) {
            nodes[(size_t)ni * 5 + k] = q[k];
        }
        node_box[(size_t)ni * 2] = make_float4(blo[0], blo[1], blo[2], 0.f);
        node_box[(size_t)ni * 2 + 1] = make_float4(bhi[0], bhi[1], bhi[2], 0.f);
    }
}

}  // namespace crt

namespace crt_host {

// The unique geometry of a scene on the device, as k_flatten and k_reflatten read it: the vertex,
// index and uv arenas (every (mesh, geometry) pair with triangles that an instance references, once), one segment per
// (instance, geometry) pair with triangles, and the instances' object_to_world | world_to_object matrices. One
// allocation (DeviceArena). The host keeps where each geometry sits and a copy of the matrices, for updates.
struct SceneGeometry {
    struct Placed {
        uint32_t vert_off, tri_off, uv_off;  // kB2Invalid: not in the arenas (no instance references it with triangles)
    };
    DeviceArena arena;
    ArenaBuf<float> vert_arena{arena}, uv_arena{arena}, xforms{arena};
    ArenaBuf<uint32_t> index_arena{arena}, bad{arena};
    ArenaBuf<crt::DevSegment> segs{arena};
    uint32_t num_segs = 0;
    size_t vert_floats = 0;                   // floats in vert_arena
    std::vector<std::vector<Placed>> placed;  // [mesh][geometry]; empty: no geometry of the mesh is in the arenas
    std::vector<float> xf;                    // 32 floats per instance, as `xforms`

    SceneGeometry() = default;
    SceneGeometry(const SceneGeometry &) = delete;
    SceneGeometry &operator=(const SceneGeometry &) = delete;

    // Uploads on `stream`; the scene's arrays must stay valid until the stream has caught up.
    void upload(const crt_scene_t *scene, const crt::FlattenPlan &plan, cudaStream_t stream)
    {
        placed.assign(scene->num_meshes, std::vector<Placed>());
        std::vector<crt::DevSegment> host_segs;
        size_t nv = 0, nt = 0, nuv = 0;
        struct Copy {
            const crt_geometry_t *geom;
            Placed at;
        };
        std::vector<Copy> copies;
        for (const crt::FlattenSegment &fs : plan.segments) {
            const crt_mesh_t &mesh = scene->meshes[fs.mesh];
            const crt_geometry_t &geom = mesh.geometries[fs.geometry];
            if (geom.num_tris == 0) {
                continue;
            }
            std::vector<Placed> &pm = placed[fs.mesh];
            if (pm.empty()) {
                pm.assign(mesh.num_geometries, Placed{crt::kB2Invalid, crt::kB2Invalid, crt::kB2Invalid});
            }
            Placed &pl = pm[fs.geometry];
            if (pl.tri_off == crt::kB2Invalid) {
                if (nv + geom.num_vertices >= 0xffffffffull || nt + geom.num_tris >= 0xffffffffull) {
                    throw std::runtime_error("device set_scene: geometry arenas exceed 2^32 - 1 elements");
                }
                pl.vert_off = (uint32_t)nv;
                pl.tri_off = (uint32_t)nt;
                nv += geom.num_vertices;
                nt += geom.num_tris;
                if (geom.uvs) {
                    pl.uv_off = (uint32_t)nuv;
                    nuv += geom.num_vertices;
                }
                copies.push_back(Copy{&geom, pl});
            }
            crt::DevSegment ds;
            ds.flat_base = (uint32_t)fs.flat_base;
            ds.num_tris = geom.num_tris;
            ds.vert_off = pl.vert_off;
            ds.num_verts = geom.num_vertices;
            ds.tri_off = pl.tri_off;
            ds.uv_off = pl.uv_off;
            ds.mat_id = fs.mat_id;
            ds.instance = fs.instance;
            host_segs.push_back(ds);
        }
        num_segs = (uint32_t)host_segs.size();
        vert_floats = nv * 3;
        auto carve = [&] {
            vert_arena.alloc(nv * 3);
            index_arena.alloc(nt * 3);
            uv_arena.alloc(nuv * 2);
            xforms.alloc((size_t)scene->num_instances * 32);
            segs.alloc(host_segs.size());
            bad.alloc(1);
        };
        carve();
        arena.commit();
        carve();
        for (const Copy &c : copies) {
            CUDA_CHECK(cudaMemcpyAsync(vert_arena.ptr + (size_t)c.at.vert_off * 3, c.geom->vertices,
                                       (size_t)c.geom->num_vertices * 3 * sizeof(float), cudaMemcpyHostToDevice, stream));
            CUDA_CHECK(cudaMemcpyAsync(index_arena.ptr + (size_t)c.at.tri_off * 3, c.geom->indices,
                                       (size_t)c.geom->num_tris * 3 * sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
            if (c.geom->uvs) {
                CUDA_CHECK(cudaMemcpyAsync(uv_arena.ptr + (size_t)c.at.uv_off * 2, c.geom->uvs,
                                           (size_t)c.geom->num_vertices * 2 * sizeof(float), cudaMemcpyHostToDevice, stream));
            }
        }
        xf.resize((size_t)scene->num_instances * 32);
        for (uint32_t i = 0; i < scene->num_instances; ++i) {
            std::memcpy(&xf[(size_t)i * 32], scene->instances[i].transform, 16 * sizeof(float));
            std::memcpy(&xf[(size_t)i * 32 + 16], &plan.w2o_all[(size_t)i * 16], 16 * sizeof(float));
        }
        CUDA_CHECK(cudaMemcpyAsync(xforms.ptr, xf.data(), xf.size() * sizeof(float), cudaMemcpyHostToDevice, stream));
        CUDA_CHECK(cudaMemcpyAsync(segs.ptr, host_segs.data(), host_segs.size() * sizeof(crt::DevSegment), cudaMemcpyHostToDevice,
                                   stream));
        CUDA_CHECK(cudaStreamSynchronize(stream));  // (host_segs is a temporary)
    }
};

// What set_scene keeps with option dynamic_scene = 1, the updates staged since, and the commit that applies them.
// Memory on the device: the unique geometry (12 B per unique vertex, + 8 B with uvs; 12 B per unique triangle; 128 B per
// instance; 32 B per (instance, geometry) segment), 4 B (leaf_flat_ids) + 32 B (tri_boxes) per flattened triangle and
// 32 B (node_boxes) per BVH8 node.
struct SceneUpdate {
    std::unique_ptr<SceneGeometry> geometry{new SceneGeometry()};
    DeviceBuffer<uint32_t> leaf_flat_ids;
    DeviceBuffer<float4> tri_boxes, node_boxes;
    std::vector<uint32_t> levels;  // Bvh8::level_begin of the tree
    uint32_t num_tris = 0;
    std::vector<std::vector<uint32_t>> num_vertices;  // [mesh][geometry] at set_scene
    // staged
    bool instances_staged = false;  // (the new matrices are in geometry->xf already)
    struct StagedVertices {
        uint32_t vert_off;
        std::vector<float> v;
    };
    std::vector<StagedVertices> vertices;

    // After the build (geometry uploaded): the leaf order, the level boundaries and the box buffers.
    void keep(const crt_scene_t *scene, const std::vector<uint32_t> &flat_ids, const std::vector<uint32_t> &level_begin,
              cudaStream_t stream)
    {
        num_tris = (uint32_t)flat_ids.size();
        levels = level_begin;
        num_vertices.assign(scene->num_meshes, std::vector<uint32_t>());
        for (uint32_t m = 0; m < scene->num_meshes; ++m) {
            for (uint32_t g = 0; g < scene->meshes[m].num_geometries; ++g) {
                num_vertices[m].push_back(scene->meshes[m].geometries[g].num_vertices);
            }
        }
        leaf_flat_ids.upload(flat_ids.data(), flat_ids.size(), stream);
        tri_boxes.alloc((size_t)num_tris * 2);
        node_boxes.alloc(levels.empty() ? 0 : (size_t)levels.back() * 2);
        CUDA_CHECK(cudaStreamSynchronize(stream));  // (flat_ids may be a temporary)
    }

    bool staged() const { return instances_staged || !vertices.empty(); }

    void stage_instances(uint32_t first, uint32_t count, const float *transforms)
    {
        const size_t num_instances = geometry->xf.size() / 32;
        if ((size_t)first + count > num_instances) {
            throw std::runtime_error("crtc_update_instances: instances " + std::to_string(first) + " + " +
                                     std::to_string(count) + " exceed the scene's " + std::to_string(num_instances));
        }
        if (count && !transforms) {
            throw std::runtime_error("crtc_update_instances: transforms is NULL");
        }
        for (uint32_t i = 0; i < count; ++i) {
            float *x = &geometry->xf[(size_t)(first + i) * 32];
            std::memcpy(x, transforms + (size_t)i * 16, 16 * sizeof(float));
            crt::mat4_inverse(x, x + 16);  // (plan_flatten's world_to_object)
        }
        instances_staged = instances_staged || count > 0;
    }

    void stage_vertices(uint32_t mesh, uint32_t geom, const float *v, uint32_t n)
    {
        if (mesh >= num_vertices.size()) {
            throw std::runtime_error("crtc_update_vertices: mesh " + std::to_string(mesh) + " out of range (the scene has " +
                                     std::to_string(num_vertices.size()) + ")");
        }
        if (geom >= num_vertices[mesh].size()) {
            throw std::runtime_error("crtc_update_vertices: geometry " + std::to_string(geom) + " out of range (mesh " +
                                     std::to_string(mesh) + " has " + std::to_string(num_vertices[mesh].size()) + ")");
        }
        if (n != num_vertices[mesh][geom]) {
            throw std::runtime_error("crtc_update_vertices: " + std::to_string(n) + " vertices; mesh " + std::to_string(mesh) +
                                     " geometry " + std::to_string(geom) + " has " + std::to_string(num_vertices[mesh][geom]) +
                                     " (the topology is fixed)");
        }
        if (n && !v) {
            throw std::runtime_error("crtc_update_vertices: vertices is NULL");
        }
        const std::vector<SceneGeometry::Placed> &pm = geometry->placed[mesh];
        if (pm.empty() || pm[geom].vert_off == crt::kB2Invalid) {
            return;  // no instance draws it: nothing to update
        }
        for (StagedVertices &sv : vertices) {
            if (sv.vert_off == pm[geom].vert_off) {
                sv.v.assign(v, v + (size_t)n * 3);
                return;
            }
        }
        vertices.push_back(StagedVertices{pm[geom].vert_off, std::vector<float>(v, v + (size_t)n * 3)});
    }

    // Enqueues the staged updates on `stream` and rewrites the triangle / shading records (leaf order) and the nodes.
    // Returns the number of kernel launches.
    int commit(float4 *nodes, float4 *tris, float4 *shade, cudaStream_t stream, int device)
    {
        SceneGeometry &g = *geometry;
        // (pageable sources: each copy has taken its bytes when the call returns)
        if (instances_staged) {
            CUDA_CHECK(cudaMemcpyAsync(g.xforms.ptr, g.xf.data(), g.xf.size() * sizeof(float), cudaMemcpyHostToDevice, stream));
        }
        for (const StagedVertices &sv : vertices) {
            CUDA_CHECK(cudaMemcpyAsync(g.vert_arena.ptr + (size_t)sv.vert_off * 3, sv.v.data(), sv.v.size() * sizeof(float),
                                       cudaMemcpyHostToDevice, stream));
        }
        instances_staged = false;
        vertices.clear();
        if (num_tris == 0) {
            return 0;
        }
        int sms = 0;
        CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
        auto grid_for = [&](uint32_t items) {
            return std::max(1u, std::min((items + crt::kBuildBlock - 1) / crt::kBuildBlock, (uint32_t)sms * 8u));
        };
        launch(crt::k_reflatten, grid_for(num_tris), crt::kBuildBlock, stream, g.segs.ptr, g.num_segs, g.xforms.ptr,
               g.vert_arena.ptr, g.index_arena.ptr, g.uv_arena.ptr, leaf_flat_ids.ptr, num_tris, tris, shade, tri_boxes.ptr);
        int launches = 1;
        for (size_t l = levels.size() - 1; l-- > 0;) {  // deepest level first
            const uint32_t count = levels[l + 1] - levels[l];
            launch(crt::k_bvh8_refit, grid_for(count), crt::kBuildBlock, stream, reinterpret_cast<uint4 *>(nodes), levels[l], count,
                   tri_boxes.ptr, node_boxes.ptr);
            ++launches;
        }
        CUDA_CHECK(cudaGetLastError());
        return launches;
    }
};

}  // namespace crt_host
