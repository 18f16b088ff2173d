// bvh8.h — compressed wide BVH (8-wide, 80-byte nodes) laid out for 128-bit loads.
//
// Replaces what the reference delegates to Embree (rtcCommitScene,
// backends/embree/embree_utils.cpp:75,128) / OptiX (optixAccelBuild,
// backends/optix/optix_utils.cpp:183-245): there is no BVH code in the reference.
// Format after Ylitie, Karras, Laine, "Efficient Incoherent Ray Traversal on GPUs Through
// Compressed Wide BVHs" (HPG 2017): one node = 5 x 16 B:
//
//   q0: p.x p.y p.z (f32 origin of the quantisation grid) | e.x e.y e.z imask (4 x u8)
//   q1: child_base (u32) | tri_base (u32) | meta[0..3] | meta[4..7]
//   q2: qlo_x[0..7] | qlo_y[0..7]
//   q3: qlo_z[0..7] | qhi_x[0..7]
//   q4: qhi_y[0..7] | qhi_z[0..7]
//
// e.* are biased exponents: the grid step on an axis is the float with bit pattern (e << 23).
// Child box plane = p + q * step. meta[i]: 0 = empty slot; inner child: 0b001 in the top 3
// bits and 24+slot in the low 5; leaf child: unary triangle count (1,2,3 -> 001,011,111) in
// the top 3 bits and the offset of its first triangle (relative to tri_base) in the low 5.
// imask bit i = slot i holds an inner child. Inner children of a node are consecutive nodes
// starting at child_base, in slot order; leaf triangles are consecutive starting at tri_base.
#pragma once

#include <cstddef>
#include <cstdint>
#include <vector>

namespace crt {

struct Bvh8Node {
    float p[3];
    uint8_t e[3];
    uint8_t imask;
    uint32_t child_base;
    uint32_t tri_base;
    uint8_t meta[8];
    uint8_t qlo_x[8];
    uint8_t qlo_y[8];
    uint8_t qlo_z[8];
    uint8_t qhi_x[8];
    uint8_t qhi_y[8];
    uint8_t qhi_z[8];
};
static_assert(sizeof(Bvh8Node) == 80, "Bvh8Node must be 80 bytes (5 x 128-bit loads)");

struct Bvh8 {
    std::vector<Bvh8Node> nodes;     // node 0 is the root
    std::vector<uint32_t> tri_order; // leaf order -> index of the input triangle
    // the nodes are numbered level by level: level k is [level_begin[k], level_begin[k + 1]), the last entry is the
    // node count (empty for a scene without triangles)
    std::vector<uint32_t> level_begin;
    float scene_lo[3], scene_hi[3];
    // build statistics
    double sah_cost = 0.0;
    uint32_t max_depth = 0;
    double build_seconds = 0.0;
};

// verts: 9 floats per triangle (v0, v1, v2), world space. threads <= 0: hardware concurrency.
void build_bvh8(const float *verts, size_t num_tris, int threads, Bvh8 &out);

}  // namespace crt
