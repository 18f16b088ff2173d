// host_scene.h — what RenderCUDA::set_scene does on the host before upload.
//
// Mirrors the conversion work of RenderEmbree::set_scene (reference
// backends/embree/render_embree.cpp:58-133) and embree::Instance
// (backends/embree/embree_utils.cpp:90-104), re-designed for a single flattened,
// world-space triangle soup that a single-level BVH8 can index:
//   - every instance is flattened to world space (object_to_world applied on the host);
//   - the per-hit work of render_embree.ispc:264-293 that does not depend on the ray —
//     geometric normal -> world space, material id lookup, the three vertex uvs — is
//     precomputed per triangle;
//   - sRGB textures are linearised and re-quantised to 8 bits exactly as
//     render_embree.cpp:90-104 does, then packed (RGBA8) into one texel arena.
#pragma once

#include <cstdint>
#include <vector>

#include "../../include/crt_scene.h"
#include "bvh8.h"

namespace crt {

constexpr uint32_t kMaxTriangles = 1u << 27;  // k_traverse's pooled pairs: owner lane << 27 | leaf-order triangle index

// The layout of DevTex (shade_math.cuh)
struct TexDesc {
    uint32_t offset;  // first texel in the arena
    int32_t width, height;
    int32_t pad;
};

// Per-triangle shading record, 48 B = 3 x float4, stored in BVH leaf order on the device.
struct TriShade {
    float n[3];           // world-space geometric normal (render_embree.ispc:269,288-290)
    uint32_t material_id; // instance.material_ids[geomID] (render_embree.ispc:292-293)
    float uv[6];          // uv of v0, v1, v2 (zeros when the geometry has no uvs)
    uint32_t has_uv;
    uint32_t flat_id;     // flattened primitive id (instances -> geometries -> primitives)
};
static_assert(sizeof(TriShade) == 48, "TriShade is three float4");

// Materials, lights and the texture arena as set_scene uploads them. Every array but the lights holds at least one
// element (zeros when the scene has none), so that the device always gets valid pointers.
struct ShadingRecords {
    std::vector<crt_material_t> materials;
    std::vector<crt_quad_light_t> lights;
    std::vector<uint32_t> texels;  // RGBA8 arena
    std::vector<TexDesc> tex_desc;
    uint32_t spp = 1;  // samples per pixel, at least 1
};

// Everything set_scene uploads when the BVH is built on the host, in device layout.
struct SceneRecords {
    Bvh8 bvh;  // bvh.nodes is the device node array (5 float4 per node)
    // 12 floats per triangle in BVH leaf order: {v0.xyz, bits(flat id)}, {e1.xyz, 0}, {e2.xyz, 0} with
    // e1 = v1 - v0, e2 = v2 - v0 (the subtraction the intersector would otherwise do per test)
    std::vector<float> tris;
    std::vector<TriShade> shade;  // the shading records in the same order
    // tris and shade keep at least one (degenerate) record so empty scenes have valid pointers;
    // leaf_flat_ids (leaf-order triangle -> flattened primitive id) has the real triangles only
    std::vector<uint32_t> leaf_flat_ids;
    ShadingRecords shading;
    size_t num_tris = 0;
    double flatten_ms = 0.0, pack_ms = 0.0;  // host wall clock of the flattening and of the leaf-order packing
};

// Flattens the scene, builds the BVH8 and packs the records. threads <= 0: hardware concurrency.
// Throws std::runtime_error on malformed input (bad material / texture / mesh ids) and on scenes the kernels cannot
// hold (check_triangle_count, check_bvh_depth).
void pack_scene(const crt_scene_t *scene, int threads, SceneRecords &out);

void check_triangle_count(size_t n);
void check_bvh_depth(uint32_t depth);

// The two halves of the flattening, for the device set_scene path (bvh8_device.cuh: k_flatten does the per-triangle
// work from the plan): (1) validation of the instance / mesh / material references, one segment per (instance,
// geometry) with the index of its first flattened triangle, and every instance's world_to_object matrix
// (embree_utils.cpp:97); (2) materials, lights and the texture arena (no triangles).
struct FlattenSegment {
    uint32_t instance, mesh, geometry, mat_id;
    size_t flat_base;
};
struct FlattenPlan {
    std::vector<FlattenSegment> segments;
    std::vector<float> w2o_all;  // 16 floats per instance, column-major
    size_t total_tris = 0;
};
void plan_flatten(const crt_scene_t *scene, FlattenPlan &plan);
// world_to_object from object_to_world (16 floats each, column-major), as plan_flatten computes it
void mat4_inverse(const float *m, float *out);
void pack_shading(const crt_scene_t *scene, int threads, ShadingRecords &out);

}  // namespace crt
