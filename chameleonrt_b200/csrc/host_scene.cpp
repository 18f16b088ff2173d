// host_scene.cpp — see host_scene.h. Compiled with -ffp-contract=off: the float expressions
// below follow the reference's source order so that the precomputed per-triangle normals are
// the values render_embree.ispc:269,288-290 would compute per hit.
#include "host_scene.h"

#include "bvh8_traverse.h"
#include "host_parallel.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstring>
#include <stdexcept>
#include <string>

namespace crt {
namespace {

struct HostScene {
    std::vector<float> tri_verts;  // 9 floats per triangle: v0, v1, v2 (world space)
    std::vector<TriShade> tri_shade;
    size_t num_tris() const { return tri_shade.size(); }
};

}  // namespace

// 4x4 inverse by cofactor expansion, column-major (the role of glm::inverse in
// embree_utils.cpp:97).
void mat4_inverse(const float *m, float *out)
{
    float inv[16];
    inv[0] = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] +
             m[13] * m[6] * m[11] - m[13] * m[7] * m[10];
    inv[4] = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] -
             m[12] * m[6] * m[11] + m[12] * m[7] * m[10];
    inv[8] = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] +
             m[12] * m[5] * m[11] - m[12] * m[7] * m[9];
    inv[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] -
              m[12] * m[5] * m[10] + m[12] * m[6] * m[9];
    inv[1] = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] -
             m[13] * m[2] * m[11] + m[13] * m[3] * m[10];
    inv[5] = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] +
             m[12] * m[2] * m[11] - m[12] * m[3] * m[10];
    inv[9] = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] -
             m[12] * m[1] * m[11] + m[12] * m[3] * m[9];
    inv[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] +
              m[12] * m[1] * m[10] - m[12] * m[2] * m[9];
    inv[2] = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] +
             m[13] * m[2] * m[7] - m[13] * m[3] * m[6];
    inv[6] = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] -
             m[12] * m[2] * m[7] + m[12] * m[3] * m[6];
    inv[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] +
              m[12] * m[1] * m[7] - m[12] * m[3] * m[5];
    inv[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] -
              m[12] * m[1] * m[6] + m[12] * m[2] * m[5];
    inv[3] = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] -
             m[9] * m[2] * m[7] + m[9] * m[3] * m[6];
    inv[7] = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] +
             m[8] * m[2] * m[7] - m[8] * m[3] * m[6];
    inv[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] -
              m[8] * m[1] * m[7] + m[8] * m[3] * m[5];
    inv[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] +
              m[8] * m[1] * m[6] - m[8] * m[2] * m[5];
    float det = m[0] * inv[0] + m[1] * inv[4] + m[2] * inv[8] + m[3] * inv[12];
    det = 1.f / det;
    for (int i = 0; i < 16; ++i) {
        out[i] = inv[i] * det;
    }
}

namespace {

inline void normalize3(float *v)
{
    // float3.ih:63-70: c = 1/length, then multiply
    const float l = std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    const float c = 1.f / l;
    v[0] *= c;
    v[1] *= c;
    v[2] *= c;
}

void check_param(float x, uint32_t num_textures, const char *what, uint32_t mat)
{
    uint32_t bits;
    std::memcpy(&bits, &x, 4);
    if (bits & 0x80000000u) {
        const uint32_t id = bits & 0x1fffffffu;
        if (id >= num_textures) {
            throw std::runtime_error("material " + std::to_string(mat) + ": parameter '" + what +
                                     "' references texture " + std::to_string(id) + " but the scene has " +
                                     std::to_string(num_textures));
        }
    }
}

double ms_since(std::chrono::steady_clock::time_point t0)
{
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

}  // namespace

// k_traverse packs a pooled (owner lane, leaf-order triangle index) pair into one 32-bit slot: 5 + 27 bits
void check_triangle_count(size_t n)
{
    if (n >= (size_t)kMaxTriangles) {
        throw std::runtime_error("set_scene: " + std::to_string(n) + " triangles; this backend holds at most 2^27 - 1 (" +
                                 std::to_string(kMaxTriangles - 1) + ") per scene");
    }
}

void check_bvh_depth(uint32_t depth)
{
    if (depth + 2 > CRT_STACK_SIZE) {
        throw std::runtime_error("BVH8 depth " + std::to_string(depth) + " exceeds the traversal stack (CRT_STACK_SIZE)");
    }
}

void plan_flatten(const crt_scene_t *s, FlattenPlan &plan)
{
    plan = FlattenPlan();
    if (s->num_lights == 0) {
        throw std::runtime_error("scene has no lights (the path tracer samples exactly one quad light per bounce)");
    }
    // count
    size_t total = 0;
    for (uint32_t i = 0; i < s->num_instances; ++i) {
        const uint32_t pm = s->instances[i].parameterized_mesh_id;
        if (pm >= s->num_parameterized_meshes) {
            throw std::runtime_error("instance references a missing parameterized mesh");
        }
        const uint32_t mesh_id = s->parameterized_meshes[pm].mesh_id;
        if (mesh_id >= s->num_meshes) {
            throw std::runtime_error("parameterized mesh references a missing mesh");
        }
        const crt_mesh_t &mesh = s->meshes[mesh_id];
        if (s->parameterized_meshes[pm].num_material_ids < mesh.num_geometries) {
            throw std::runtime_error("parameterized mesh has fewer material ids than geometries");
        }
        for (uint32_t g = 0; g < mesh.num_geometries; ++g) {
            total += mesh.geometries[g].num_tris;
        }
    }
    if (total >= 0xffffffffull) {
        throw std::runtime_error("scene exceeds 2^32-1 flattened triangles");
    }
    plan.total_tris = total;
    plan.w2o_all.resize((size_t)s->num_instances * 16);
    size_t flat = 0;
    for (uint32_t i = 0; i < s->num_instances; ++i) {
        const crt_instance_t &inst = s->instances[i];
        const crt_parameterized_mesh_t &pm = s->parameterized_meshes[inst.parameterized_mesh_id];
        const crt_mesh_t &mesh = s->meshes[pm.mesh_id];
        mat4_inverse(inst.transform, &plan.w2o_all[(size_t)i * 16]);
        for (uint32_t g = 0; g < mesh.num_geometries; ++g) {
            const crt_geometry_t &geom = mesh.geometries[g];
            const uint32_t mat_id = pm.material_ids[g];
            if (mat_id >= s->num_materials) {
                throw std::runtime_error("geometry references material " + std::to_string(mat_id) +
                                         " but the scene has " + std::to_string(s->num_materials) +
                                         " (run validate_materials, util/scene.cpp:935-958)");
            }
            plan.segments.push_back(FlattenSegment{i, pm.mesh_id, g, mat_id, flat});
            flat += geom.num_tris;
        }
    }
}

namespace {

// The triangle half of the flattening; throws std::runtime_error on malformed input (bad material / mesh ids,
// vertex indices out of range)
void flatten_scene(const crt_scene_t *s, HostScene &out, int threads)
{
    FlattenPlan plan;
    plan_flatten(s, plan);
    const size_t total = plan.total_tris;
    out.tri_verts.resize(total * 9);
    out.tri_shade.resize(total);

    // one segment per (instance, geometry); its triangles are processed in fixed blocks on several threads
    struct Block {
        uint32_t segment, p_begin, p_end;
    };
    const std::vector<FlattenSegment> &segments = plan.segments;
    const std::vector<float> &w2o_all = plan.w2o_all;
    std::vector<Block> blocks;
    const uint32_t kBlockTris = 1u << 15;
    for (size_t si = 0; si < segments.size(); ++si) {
        const uint32_t nt = s->meshes[segments[si].mesh].geometries[segments[si].geometry].num_tris;
        for (uint32_t p = 0; p < nt; p += kBlockTris) {
            blocks.push_back(Block{(uint32_t)si, p, std::min(nt, p + kBlockTris)});
        }
    }
    std::atomic<bool> bad_index(false);
    parallel_blocks((uint32_t)blocks.size(), host_threads(threads), [&](uint32_t bi) {
        const Block &blk = blocks[bi];
        const FlattenSegment &seg = segments[blk.segment];
        const crt_instance_t &inst = s->instances[seg.instance];
        const crt_geometry_t &geom = s->meshes[s->parameterized_meshes[inst.parameterized_mesh_id].mesh_id].geometries[seg.geometry];
        const float *m = inst.transform;
        const float *w2o = &w2o_all[(size_t)seg.instance * 16];
        for (uint32_t p = blk.p_begin; p < blk.p_end; ++p) {
            const size_t f = seg.flat_base + p;
            const uint32_t idx[3] = {geom.indices[3 * p], geom.indices[3 * p + 1], geom.indices[3 * p + 2]};
            if (idx[0] >= geom.num_vertices || idx[1] >= geom.num_vertices || idx[2] >= geom.num_vertices) {
                bad_index = true;
                return;
            }
            float vo[3][3];
            for (int k = 0; k < 3; ++k) {
                const float *v = geom.vertices + 3 * (size_t)idx[k];
                vo[k][0] = v[0];
                vo[k][1] = v[1];
                vo[k][2] = v[2];
                float *w = &out.tri_verts[f * 9 + 3 * k];
                w[0] = m[0] * v[0] + m[4] * v[1] + m[8] * v[2] + m[12];
                w[1] = m[1] * v[0] + m[5] * v[1] + m[9] * v[2] + m[13];
                w[2] = m[2] * v[0] + m[6] * v[1] + m[10] * v[2] + m[14];
            }
            TriShade &ts = out.tri_shade[f];
            // Ng = cross(v1 - v0, v2 - v0) in object space, normalised
            const float e1[3] = {vo[1][0] - vo[0][0], vo[1][1] - vo[0][1], vo[1][2] - vo[0][2]};
            const float e2[3] = {vo[2][0] - vo[0][0], vo[2][1] - vo[0][1], vo[2][2] - vo[0][2]};
            float n[3] = {e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]};
            normalize3(n);
            // normal = normalize(transpose(world_to_object) * n), mat4.ih:11-33
            float r[3];
            r[0] = w2o[0] * n[0] + w2o[1] * n[1] + w2o[2] * n[2];
            r[1] = w2o[4] * n[0] + w2o[5] * n[1] + w2o[6] * n[2];
            r[2] = w2o[8] * n[0] + w2o[9] * n[1] + w2o[10] * n[2];
            normalize3(r);
            ts.n[0] = r[0];
            ts.n[1] = r[1];
            ts.n[2] = r[2];
            ts.material_id = seg.mat_id;
            ts.flat_id = (uint32_t)f;
            if (geom.uvs) {
                ts.has_uv = 1;
                for (int k = 0; k < 3; ++k) {
                    ts.uv[2 * k] = geom.uvs[2 * (size_t)idx[k]];
                    ts.uv[2 * k + 1] = geom.uvs[2 * (size_t)idx[k] + 1];
                }
            } else {
                ts.has_uv = 0;
                for (int k = 0; k < 6; ++k) {
                    ts.uv[k] = 0.f;
                }
            }
        }
    });
    if (bad_index) {
        throw std::runtime_error("triangle index out of range");
    }
}

}  // namespace

void pack_shading(const crt_scene_t *s, int threads, ShadingRecords &out)
{
    out.spp = std::max<uint32_t>(1u, s->samples_per_pixel);
    // materials
    out.materials.assign(s->materials, s->materials + s->num_materials);
    for (uint32_t i = 0; i < s->num_materials; ++i) {
        const crt_material_t &mt = s->materials[i];
        check_param(mt.base_color[0], s->num_textures, "base_color", i);
        check_param(mt.metallic, s->num_textures, "metallic", i);
        check_param(mt.specular, s->num_textures, "specular", i);
        check_param(mt.roughness, s->num_textures, "roughness", i);
        check_param(mt.specular_tint, s->num_textures, "specular_tint", i);
        check_param(mt.anisotropy, s->num_textures, "anisotropy", i);
        check_param(mt.sheen, s->num_textures, "sheen", i);
        check_param(mt.sheen_tint, s->num_textures, "sheen_tint", i);
        check_param(mt.clearcoat, s->num_textures, "clearcoat", i);
        check_param(mt.clearcoat_gloss, s->num_textures, "clearcoat_gloss", i);
        check_param(mt.ior, s->num_textures, "ior", i);
        check_param(mt.specular_transmission, s->num_textures, "specular_transmission", i);
    }
    out.lights.assign(s->lights, s->lights + s->num_lights);

    // textures: sRGB -> linear 8-bit (render_embree.cpp:90-104), expanded to RGBA8.
    // srgb_to_linear is util/util.cpp:102-108; its std::pow(float, 2.4) is a double pow.
    uint8_t lut[256];
    for (int v = 0; v < 256; ++v) {
        float x = v / 255.f;
        if (x <= 0.04045f) {
            x = x / 12.92f;
        } else {
            x = (float)std::pow((double)((x + 0.055f) / 1.055f), 2.4);
        }
        const float y = x * 255.f;
        lut[v] = (uint8_t)(y < 0.f ? 0.f : (y > 255.f ? 255.f : y));
    }
    size_t texels = 0;
    for (uint32_t i = 0; i < s->num_textures; ++i) {
        const crt_image_t &im = s->textures[i];
        if (im.width <= 0 || im.height <= 0 || im.channels < 1 || im.channels > 4 || !im.data) {
            throw std::runtime_error("texture " + std::to_string(i) + " has an invalid shape");
        }
        texels += (size_t)im.width * im.height;
    }
    if (texels >= 0xffffffffull) {
        throw std::runtime_error("texture arena exceeds 2^32 texels");
    }
    out.texels.resize(texels);
    out.tex_desc.resize(s->num_textures);
    // (rows of every texture in fixed blocks on several threads: C3's 11 M texels are the largest host cost of
    // set_scene once the BVH is built on the device)
    struct TexBlock {
        uint32_t tex;
        size_t px_begin, px_end;
    };
    std::vector<TexBlock> tex_blocks;
    const size_t kBlockTexels = (size_t)1 << 18;
    size_t off = 0;
    for (uint32_t i = 0; i < s->num_textures; ++i) {
        const crt_image_t &im = s->textures[i];
        out.tex_desc[i] = TexDesc{(uint32_t)off, im.width, im.height, 0};
        const size_t n = (size_t)im.width * im.height;
        for (size_t b = 0; b < n; b += kBlockTexels) {
            tex_blocks.push_back(TexBlock{i, b, std::min(n, b + kBlockTexels)});
        }
        off += n;
    }
    parallel_blocks((uint32_t)tex_blocks.size(), host_threads(threads), [&](uint32_t bi) {
        const TexBlock &tb = tex_blocks[bi];
        const crt_image_t &im = s->textures[tb.tex];
        const size_t base = out.tex_desc[tb.tex].offset;
        const bool srgb = im.color_space == CRT_COLOR_SPACE_SRGB;
        const int convert_channels = std::min(3, im.channels);
        for (size_t px = tb.px_begin; px < tb.px_end; ++px) {
            uint8_t c[4] = {0, 0, 0, 0};  // channels the image lacks read as 0 (texture2d.ih:13-27)
            for (int k = 0; k < im.channels; ++k) {
                uint8_t v = im.data[px * im.channels + k];
                if (srgb && k < convert_channels) {
                    v = lut[v];
                }
                c[k] = v;
            }
            out.texels[base + px] = (uint32_t)c[0] | ((uint32_t)c[1] << 8) | ((uint32_t)c[2] << 16) | ((uint32_t)c[3] << 24);
        }
    });
    if (out.materials.empty()) {
        out.materials.resize(1);
        std::memset(&out.materials[0], 0, sizeof(crt_material_t));
    }
    if (out.texels.empty()) {
        out.texels.assign(1, 0u);
    }
    if (out.tex_desc.empty()) {
        out.tex_desc.assign(1, TexDesc{0, 0, 0, 0});
    }
}

namespace {

// Device-format triangle records in BVH leaf order (SceneRecords::tris), and the shading records permuted into the
// same order.
void pack_triangles(const HostScene &scene, const Bvh8 &bvh, std::vector<float> &tri_records,
                    std::vector<TriShade> &shade_leaf_order, int threads)
{
    const size_t n = bvh.tri_order.size();
    tri_records.resize(n * 12);
    shade_leaf_order.resize(n);
    const size_t kBlockTris = 1u << 15;
    parallel_blocks((uint32_t)((n + kBlockTris - 1) / kBlockTris), host_threads(threads), [&](uint32_t blk) {
    const size_t end = std::min(n, (size_t)(blk + 1) * kBlockTris);
    for (size_t i = (size_t)blk * kBlockTris; i < end; ++i) {
        const uint32_t src = bvh.tri_order[i];
        const float *v = &scene.tri_verts[(size_t)src * 9];
        float *r = &tri_records[i * 12];
        const uint32_t flat = scene.tri_shade[src].flat_id;
        r[0] = v[0];
        r[1] = v[1];
        r[2] = v[2];
        std::memcpy(&r[3], &flat, 4);
        r[4] = v[3] - v[0];
        r[5] = v[4] - v[1];
        r[6] = v[5] - v[2];
        r[7] = 0.f;
        r[8] = v[6] - v[0];
        r[9] = v[7] - v[1];
        r[10] = v[8] - v[2];
        r[11] = 0.f;
        shade_leaf_order[i] = scene.tri_shade[src];
    }
    });
}

}  // namespace

void pack_scene(const crt_scene_t *s, int threads, SceneRecords &out)
{
    out = SceneRecords();
    HostScene hs;
    const auto t0 = std::chrono::steady_clock::now();
    flatten_scene(s, hs, threads);
    pack_shading(s, threads, out.shading);
    out.flatten_ms = ms_since(t0);
    out.num_tris = hs.num_tris();
    check_triangle_count(out.num_tris);
    build_bvh8(hs.tri_verts.data(), hs.num_tris(), threads, out.bvh);
    check_bvh_depth(out.bvh.max_depth);
    const auto t_pack = std::chrono::steady_clock::now();
    pack_triangles(hs, out.bvh, out.tris, out.shade, threads);
    out.pack_ms = ms_since(t_pack);
    out.leaf_flat_ids.resize(out.shade.size());
    for (size_t i = 0; i < out.shade.size(); ++i) {
        out.leaf_flat_ids[i] = out.shade[i].flat_id;
    }
    // keep at least one (degenerate) record so empty scenes have valid pointers
    if (out.tris.empty()) {
        out.tris.assign(12, 0.f);
        out.shade.resize(1);
        std::memset(&out.shade[0], 0, sizeof(TriShade));
    }
}

}  // namespace crt
