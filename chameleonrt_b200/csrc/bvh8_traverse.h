// bvh8_traverse.h — single-ray traversal of the compressed BVH8 + Moeller-Trumbore.
//
// Replaces rtcIntersectV / rtcOccludedV (reference call sites:
// backends/embree/render_embree.ispc:245 and :144,170). Semantics kept (SURVEY.md §8c):
// closest hit with tnear < t < tfar, no backface culling, barycentrics (u,v) weight v1,v2.
//
// Written once as __host__ __device__ code: the CUDA kernels (kernels.cu) are the product;
// the host instantiation exists only so that tests can validate the builder and the node
// format on a machine without a GPU (tests/test_bvh8_host.py via libcrt_bvh8_hostcheck.so).
// render() never runs the host instantiation.
//
// Arithmetic contract for the triangle test (DESIGN.md §4; the CPU oracle states the same
// formula independently): explicit fmaf in a fixed order, NaN-failing comparisons,
// equal-t ties broken toward the lower flattened primitive id so that the result does not
// depend on traversal order.
#pragma once

#include <cstdint>

#if defined(__CUDACC__)
#define CRT_HD __host__ __device__ __forceinline__
#else
#define CRT_HD inline
#include <cmath>
#include <cstring>
#if !defined(__VECTOR_TYPES_H__)  // a host translation unit that included <cuda_runtime.h> has these already
struct float4 {
    float x, y, z, w;
};
struct float3 {
    float x, y, z;
};
struct uint2 {
    unsigned int x, y;
};
#endif
#endif

namespace crt {

CRT_HD uint32_t f2u(float f)
{
#if defined(__CUDA_ARCH__)
    return __float_as_uint(f);
#else
    uint32_t u;
    memcpy(&u, &f, 4);
    return u;
#endif
}
CRT_HD float u2f(uint32_t u)
{
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}
CRT_HD int msb(uint32_t v)  // v != 0
{
#if defined(__CUDA_ARCH__)
    return 31 - __clz((int)v);
#else
    return 31 - __builtin_clz(v);
#endif
}
CRT_HD int popc(uint32_t v)
{
#if defined(__CUDA_ARCH__)
    return __popc(v);
#else
    return __builtin_popcount(v);
#endif
}
// per byte: 0xff if the byte's top bit is set else 0x00
CRT_HD uint32_t sign_extend_s8x4(uint32_t v)
{
#if defined(__CUDA_ARCH__)
    uint32_t r;
    asm("prmt.b32 %0, %1, 0x0, 0x0000BA98;" : "=r"(r) : "r"(v));
    return r;
#else
    uint32_t r = 0;
    for (int i = 0; i < 4; ++i) {
        if (v & (0x80u << (8 * i))) {
            r |= 0xffu << (8 * i);
        }
    }
    return r;
#endif
}
CRT_HD float fma_(float a, float b, float c)
{
#if defined(__CUDA_ARCH__)
    return __fmaf_rn(a, b, c);
#else
    return fmaf(a, b, c);
#endif
}
// 1 / x for the box test only (|x| >= 1e-20, so neither the input nor the result is subnormal)
// CRT_RCP_SKEW (host builds of the host checks only): -1 moves the exact reciprocal one ulp towards zero, +1 one ulp away
// from it, so that the box test's slack for the error of the device's approximate reciprocal is tested off the GPU.
CRT_HD float rcp_box(float x)
{
#if defined(__CUDA_ARCH__)
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
#elif defined(CRT_RCP_SKEW)
    const float r = 1.f / x;
    return nextafterf(r, CRT_RCP_SKEW < 0 ? 0.f : copysignf(INFINITY, r));
#else
    return 1.f / x;
#endif
}
CRT_HD int32_t imax(int32_t a, int32_t b)
{
    return a > b ? a : b;
}
CRT_HD int32_t imin(int32_t a, int32_t b)
{
    return a < b ? a : b;
}
// three-input signed integer max / min: one VIMNMX3 each on sm_90 (DPX)
CRT_HD int32_t imax3(int32_t a, int32_t b, int32_t c)
{
#if defined(__CUDA_ARCH__)
    return __vimax3_s32(a, b, c);
#else
    return imax(a, imax(b, c));
#endif
}
CRT_HD int32_t imin3(int32_t a, int32_t b, int32_t c)
{
#if defined(__CUDA_ARCH__)
    return __vimin3_s32(a, b, c);
#else
    return imin(a, imin(b, c));
#endif
}
CRT_HD int32_t f2i(float f)
{
    return (int32_t)f2u(f);
}
CRT_HD float i2f(int32_t i)
{
    return u2f((uint32_t)i);
}

struct Ray {
    float ox, oy, oz, tnear;
    float dx, dy, dz, tfar;
};

struct HitRecord {
    float t, u, v;
    uint32_t tri;   // leaf-order triangle index, 0xffffffff = miss
    uint32_t flat;  // flattened primitive id of that triangle
};

// Moeller-Trumbore with the fixed fma order. tri = {v0.xyz|flat id, e1.xyz, e2.xyz}
CRT_HD bool tri_test(const Ray &r, float tfar, const float4 t0, const float4 t1, const float4 t2, float &t, float &u,
                     float &v)
{
    // p = cross(d, e2)
    const float px = fma_(r.dy, t2.z, -(r.dz * t2.y));
    const float py = fma_(r.dz, t2.x, -(r.dx * t2.z));
    const float pz = fma_(r.dx, t2.y, -(r.dy * t2.x));
    const float det = fma_(t1.z, pz, fma_(t1.y, py, t1.x * px));
    const float inv = 1.f / det;
    const float tx = r.ox - t0.x, ty = r.oy - t0.y, tz = r.oz - t0.z;
    u = fma_(tz, pz, fma_(ty, py, tx * px)) * inv;
    // q = cross(tv, e1)
    const float qx = fma_(ty, t1.z, -(tz * t1.y));
    const float qy = fma_(tz, t1.x, -(tx * t1.z));
    const float qz = fma_(tx, t1.y, -(ty * t1.x));
    v = fma_(r.dz, qz, fma_(r.dy, qy, r.dx * qx)) * inv;
    t = fma_(t2.z, qz, fma_(t2.y, qy, t2.x * qx)) * inv;
    return (u >= 0.f) && (v >= 0.f) && (u + v <= 1.f) && (t > r.tnear) && (t < tfar);
}

#ifndef CRT_STACK_SIZE
#define CRT_STACK_SIZE 32
#endif

struct TraversalCounters {
    uint32_t nodes = 0;
    uint32_t tris = 0;
};

// Plain per-thread array stack (host check; device fallback).
struct ArrayStack {
    uint2 e[CRT_STACK_SIZE];
    int sp = 0;
    CRT_HD void push(const uint2 v) { e[sp++] = v; }
    CRT_HD uint2 pop() { return e[--sp]; }
    CRT_HD bool empty() const { return sp == 0; }
    CRT_HD void clear() { sp = 0; }
};

// Resumable traversal state of one ray: everything derived from the ray that the node step
// needs, the current node group, and the best hit so far.
struct TravState {
    Ray ray;
    float idx, idy, idz;
    uint32_t oct_inv4;
    uint32_t one;  // 0x3F800000, deliberately opaque to the compiler (see byte_unit)
    float tfar;
    uint2 cur;
    HitRecord hit;
};

CRT_HD void trav_init(TravState &s, const Ray &ray, uint32_t one = 0x3F800000u)
{
    s.ray = ray;
    s.one = one;
    // direction reciprocal with the usual guard for zero components. On the device it is the one-instruction
    // approximation (MUFU.RCP, relative error <= 2^-23; three correctly rounded divisions were 45 of the ~120
    // instructions of a ray refill, which runs at ~5 active lanes): the reciprocal only scales the slab distances of the
    // box test, whose slack (node_intersect) covers that error; the triangle test does not use it, so hits do not change.
    const float eps = 1e-20f;
    s.idx = rcp_box(fabsf(ray.dx) > eps ? ray.dx : (ray.dx < 0.f ? -eps : eps));
    s.idy = rcp_box(fabsf(ray.dy) > eps ? ray.dy : (ray.dy < 0.f ? -eps : eps));
    s.idz = rcp_box(fabsf(ray.dz) > eps ? ray.dz : (ray.dz < 0.f ? -eps : eps));
    s.oct_inv4 =
        ((ray.dx < 0.f ? 0u : 0x04040404u) | (ray.dy < 0.f ? 0u : 0x02020202u) | (ray.dz < 0.f ? 0u : 0x01010101u));
    s.tfar = ray.tfar;
    s.hit.t = ray.tfar;
    s.hit.u = s.hit.v = 0.f;
    s.hit.tri = 0xffffffffu;
    s.hit.flat = 0xffffffffu;
    s.cur.x = 0;
    s.cur.y = 0x80000000u;  // root: "inner child in slot 7 of a virtual parent"
}

// Visit the children of every node in the REVERSE of the ray's octant order (farthest first). For an
// any-hit query the answer does not depend on the order, only the work does: on the bench scene 92 % of the
// light-sample shadow rays are occluded, mostly by geometry near the light's end of the segment, and far-first
// finds an occluder after 14 % fewer node steps and 27 % fewer triangle tests (scripts/bvh_quality.py).
CRT_HD void trav_reverse_order(TravState &s)
{
    s.oct_inv4 ^= 0x07070707u;
}

// byte j of `packed` as the float 1 + b * 2^-15, built by ONE byte-permute (no int->float
// conversion: I2F executes on the quarter-rate XU pipe, which the first profile showed at 52 %
// utilisation with 48 conversions per node). `one` must hold 0x3F800000 in a REGISTER the compiler
// cannot see through (TravState::one comes from a kernel argument): SASS PRMT takes a single
// immediate, and with the constant in a register the selector becomes the immediate instead of
// being re-materialised into a register before every PRMT.
CRT_HD float byte_unit(uint32_t packed, int j, uint32_t one)
{
#if defined(__CUDA_ARCH__)
    uint32_t r;
    switch (j) {  // j is a compile-time constant after unrolling; the selector must be an immediate
    case 0: asm("prmt.b32 %0, %1, %2, 0x7604;" : "=r"(r) : "r"(packed), "r"(one)); break;
    case 1: asm("prmt.b32 %0, %1, %2, 0x7614;" : "=r"(r) : "r"(packed), "r"(one)); break;
    case 2: asm("prmt.b32 %0, %1, %2, 0x7624;" : "=r"(r) : "r"(packed), "r"(one)); break;
    default: asm("prmt.b32 %0, %1, %2, 0x7634;" : "=r"(r) : "r"(packed), "r"(one)); break;
    }
    return __uint_as_float(r);
#else
    return u2f(one | (((packed >> (8 * j)) & 0xffu) << 8));
#endif
}

// Intersects the 8 quantised child boxes of one node. Returns the node's child group in `cur`
// (x = child_base, y = hit bits of inner children | imask) and its triangle group in `tri`
// (x = tri_base, y = hit bits of leaf triangles).
CRT_HD void node_intersect_loaded(const float4 n0, const float4 n1, const float4 n2, const float4 n3, const float4 n4,
                                  const TravState &s, uint2 &cur, uint2 &tri);
CRT_HD void node_intersect(const float4 *__restrict__ nodes, const TravState &s, uint32_t node_index, uint2 &cur,
                           uint2 &tri)
{
    const float4 *np = nodes + (size_t)node_index * 5;
    node_intersect_loaded(np[0], np[1], np[2], np[3], np[4], s, cur, tri);
}
// (the five 128-bit words of the node already in registers: k_traverse's TOP variant reads the first levels of the tree
// from a shared-memory copy)
CRT_HD void node_intersect_loaded(const float4 n0, const float4 n1, const float4 n2, const float4 n3, const float4 n4,
                                  const TravState &s, uint2 &cur, uint2 &tri)
{
    const Ray &ray = s.ray;
    const uint32_t e_imask = f2u(n0.w);
    // plane distance = q * ad0 + ob0 with ad0 = 2^e / d, ob0 = (p - o) / d. q enters as
    // qf = 1 + q * 2^-15 (byte_unit), so t = qf * ad + ob with ad = 2^15 ad0 and ob = ob0 - ad.
    const float adx = u2f((e_imask & 0xffu) << 23) * s.idx * 32768.f;
    const float ady = u2f(((e_imask >> 8) & 0xffu) << 23) * s.idy * 32768.f;
    const float adz = u2f(((e_imask >> 16) & 0xffu) << 23) * s.idz * 32768.f;
    const float ob0x = (n0.x - ray.ox) * s.idx;
    const float ob0y = (n0.y - ray.oy) * s.idy;
    const float ob0z = (n0.z - ray.oz) * s.idz;
    const float obx = ob0x - adx, oby = ob0y - ady, obz = ob0z - adz;
    // Rounding slack, per axis: |ob0| can be much larger than a plane distance (cancellation), and
    // ob0 - ad rounds at the scale of ad = 2^15 ad0 (up to 2^-9 of a grid step), so the absolute
    // error of a plane distance is bounded by ~2e-7 |ob0| + 1.2e-7 |ad| OF THAT AXIS (it grows like
    // 1/d: huge for an axis the ray is nearly parallel to, tiny for the others). Each axis'
    // interval is widened by its own bound — folded into ob, so it costs nothing per child — which
    // keeps the box test conservative with respect to the (independently rounded) triangle test,
    // including for equal-t ties, without loosening the other two axes. (A first version widened all
    // axes by the worst axis' bound: near-axis rays then visited the whole tree.)
    // (round 2: + the <= 2^-23 relative error of the approximate direction reciprocal, which scales ob0 and ad alike:
    // + 1.2e-7 |ob0| + 2.4e-7 |ad| (q ad <= 2 ad); the constants keep the factor 2 over the bound)
    const float sx = fma_(6.4e-7f, fabsf(ob0x), 7.2e-7f * fabsf(adx));
    const float sy = fma_(6.4e-7f, fabsf(ob0y), 7.2e-7f * fabsf(ady));
    const float sz = fma_(6.4e-7f, fabsf(ob0z), 7.2e-7f * fabsf(adz));
    const float obx_lo = obx - sx, obx_hi = obx + sx;
    const float oby_lo = oby - sy, oby_hi = oby + sy;
    const float obz_lo = obz - sz, obz_hi = obz + sz;
    // Slab test on the float bit patterns as signed integers (Ylitie, Karras and Laine 2017): two three-input integer
    // min/max and two two-input ones per child instead of six FMNMX, compared as floats.
    // As signed integers the non-negative floats keep their order and lie above every negative float, and the
    // negative floats are in reverse order. So over any set of non-NaN values the integer max is at most the float
    // max (it is equal when the set holds a value >= +0, otherwise it is the most negative element), and the integer
    // min is at least the float min (equal when every element is >= +0, otherwise it is the negative element closest
    // to zero). A child the float test accepts is therefore always accepted, whatever the sign of tnear: the test stays
    // conservative for caller-supplied rays with a negative tnear (crtc_trace_closest). With tnear >= +0, which every
    // ray of a frame has (k_raygen 0, k_shade and the shadow rays kEpsilon), tmin is exactly the float max, and a
    // negative tmax rejects the child under both forms (the float compare even keeps tmax = -0.0 against tmin = +0,
    // as before), so the same children are visited.
    // NaN would be a large (or, with the sign bit, a small) integer instead of being dropped like fminf / fmaxf do,
    // so the test relies on no plane distance being NaN. A finite ray (the reciprocals are clamped to |1 / d| <= 1e20)
    // against a node gives finite ad and ob0 as long as the grid step is below ~3e13 and |p - o| below ~1e18, which
    // holds for every node the builders emit when the scene and the ray origins lie within +-1e15; after that,
    // overflow can only reach +-Inf, which orders correctly. A ray with a NaN or Inf component can still make NaN
    // planes, but tri_test fails for such a ray (NaN-failing comparisons), so it hits nothing either way.
    const int32_t tnear_i = f2i(ray.tnear), tfar_i = f2i(s.tfar);
    uint32_t hitmask = 0;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const uint32_t meta4 = f2u(half == 0 ? n1.z : n1.w);
        const uint32_t is_inner4 = (meta4 & (meta4 << 1)) & 0x10101010u;
        const uint32_t inner_mask4 = sign_extend_s8x4(is_inner4 << 3);
        const uint32_t bit_index4 = (meta4 ^ (s.oct_inv4 & inner_mask4)) & 0x1f1f1f1fu;
        const uint32_t child_bits4 = (meta4 >> 5) & 0x07070707u;
        const uint32_t qlox = f2u(half == 0 ? n2.x : n2.y), qloy = f2u(half == 0 ? n2.z : n2.w);
        const uint32_t qloz = f2u(half == 0 ? n3.x : n3.y), qhix = f2u(half == 0 ? n3.z : n3.w);
        const uint32_t qhiy = f2u(half == 0 ? n4.x : n4.y), qhiz = f2u(half == 0 ? n4.z : n4.w);
        const uint32_t xmin = ray.dx < 0.f ? qhix : qlox, xmax = ray.dx < 0.f ? qlox : qhix;
        const uint32_t ymin = ray.dy < 0.f ? qhiy : qloy, ymax = ray.dy < 0.f ? qloy : qhiy;
        const uint32_t zmin = ray.dz < 0.f ? qhiz : qloz, zmax = ray.dz < 0.f ? qloz : qhiz;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float tminx = fma_(byte_unit(xmin, j, s.one), adx, obx_lo);
            const float tminy = fma_(byte_unit(ymin, j, s.one), ady, oby_lo);
            const float tminz = fma_(byte_unit(zmin, j, s.one), adz, obz_lo);
            const float tmaxx = fma_(byte_unit(xmax, j, s.one), adx, obx_hi);
            const float tmaxy = fma_(byte_unit(ymax, j, s.one), ady, oby_hi);
            const float tmaxz = fma_(byte_unit(zmax, j, s.one), adz, obz_hi);
            const float tmin = i2f(imax3(f2i(tminx), f2i(tminy), imax(f2i(tminz), tnear_i)));
            const float tmax = i2f(imin3(f2i(tmaxx), f2i(tmaxy), imin(f2i(tmaxz), tfar_i)));
            if (tmin <= tmax) {
                const uint32_t bits = (child_bits4 >> (8 * j)) & 0xffu;
                const uint32_t idx_ = (bit_index4 >> (8 * j)) & 0xffu;
                hitmask |= bits << idx_;
            }
        }
    }
    cur.x = f2u(n1.x);
    cur.y = (hitmask & 0xff000000u) | (e_imask >> 24);
    tri.x = f2u(n1.y);
    tri.y = hitmask & 0x00ffffffu;
}

// Pops the next inner child out of the node group `cur` (pushing what remains onto the stack is
// the caller's business) and returns its node index.
CRT_HD uint32_t next_child(uint2 &cur, uint32_t oct_inv4)
{
    const uint32_t hits_imask = cur.y;
    const int child_bit = msb(hits_imask);
    cur.y &= ~(1u << child_bit);
    const uint32_t slot_index = (uint32_t)(child_bit - 24) ^ (oct_inv4 & 0xffu);
    const uint32_t rel = (uint32_t)popc(hits_imask & ~(0xffffffffu << slot_index));
    return cur.x + rel;
}

// Tests the highest pending triangle of `tri` against the ray and records it if it is the new
// closest hit (ties toward the lower flattened primitive id). Returns true if a hit was recorded.
CRT_HD bool test_next_triangle(const float4 *__restrict__ tris, TravState &s, uint2 &tri)
{
    const int ti = msb(tri.y);
    tri.y &= ~(1u << ti);
    const uint32_t tri_index = tri.x + (uint32_t)ti;
    const float4 *tp = tris + (size_t)tri_index * 3;
    const float4 t0 = tp[0], t1 = tp[1], t2 = tp[2];
    float t, u, v;
    // once a hit exists, t == tfar is still let through so ties resolve by primitive id
    if (tri_test(s.ray, s.hit.tri == 0xffffffffu ? s.tfar : INFINITY, t0, t1, t2, t, u, v)) {
        const uint32_t flat = f2u(t0.w);
        if (t < s.tfar || (t == s.tfar && s.hit.tri != 0xffffffffu && flat < s.hit.flat)) {
            s.hit.t = t;
            s.hit.u = u;
            s.hit.v = v;
            s.hit.tri = tri_index;
            s.hit.flat = flat;
            s.tfar = t;
            return true;
        }
    }
    return false;
}

// One traversal step: intersect one node (or take a popped triangle group), test the
// triangles it yields, pop the next group. Returns true when the ray is finished.
// ANY_HIT: finish at the first accepted triangle. COUNT: fill counters (instrumented build used
// to derive the algorithmic byte count of SURVEY.md §8d).
template <bool ANY_HIT, bool COUNT, typename Stack>
CRT_HD bool trav_step(const float4 *__restrict__ nodes, const float4 *__restrict__ tris, TravState &s, Stack &stack,
                      TraversalCounters *counters)
{
    uint2 tri_group;
    if (s.cur.y & 0xff000000u) {
        const uint32_t node_index = next_child(s.cur, s.oct_inv4);
        if (s.cur.y & 0xff000000u) {
            stack.push(s.cur);
        }
        if (COUNT) {
            counters->nodes++;
        }
        node_intersect(nodes, s, node_index, s.cur, tri_group);
    } else {
        tri_group = s.cur;
        s.cur.x = 0;
        s.cur.y = 0;
    }
    while (tri_group.y) {
        if (COUNT) {
            counters->tris++;
        }
        if (test_next_triangle(tris, s, tri_group) && ANY_HIT) {
            return true;
        }
    }
    if ((s.cur.y & 0xff000000u) == 0) {
        if (stack.empty()) {
            return true;
        }
        s.cur = stack.pop();
    }
    return false;
}

// Whole-ray convenience wrapper (host check, simple device paths).
template <bool ANY_HIT, bool COUNT>
CRT_HD bool bvh8_trace(const float4 *__restrict__ nodes, const float4 *__restrict__ tris, const Ray &ray,
                       HitRecord &hit, TraversalCounters *counters, bool far_first = false)
{
    TravState s;
    trav_init(s, ray);
    if (far_first) {
        trav_reverse_order(s);
    }
    ArrayStack stack;
    while (!trav_step<ANY_HIT, COUNT>(nodes, tris, s, stack, counters)) {
    }
    hit = s.hit;
    return hit.tri != 0xffffffffu;
}

}  // namespace crt
