// shade_hostcheck.cpp — TEST-ONLY shared library (libcrt_shade_hostcheck.so).
//
// Compiles the product's DEVICE shading arithmetic (shade_math.cuh: rng, texture filter, quad light, Disney
// BSDF eval / pdf / sample, miss shader, sRGB8) for the HOST with g++, so that the very source the kernels
// run can be compared on a machine without a GPU, input by input, with tables computed by the reference's
// own functions (tests/golden/ref_embree_frames.npz, produced from /root/reference/backends/embree/*.ih).
// Same entry-point signatures as the oracle's oracle_kat_* (oracle/oracle.cpp). Compiled -ffp-contract=off like
// the device code's -fmad=false; transcendental functions are glibc's here and CUDA's on the device. It is not
// linked into libcrt_cuda_core.so and render() cannot reach it.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include <cuda_runtime.h>  // float3 / float4 / make_float3: host-usable vector types

// the handful of device intrinsics shade_math.cuh uses, as host functions
template <typename T>
static inline T __ldg(const T *p)
{
    return *p;
}
static inline uint32_t __float_as_uint(float f)
{
    uint32_t u;
    std::memcpy(&u, &f, 4);
    return u;
}
static inline float __uint_as_float(uint32_t u)
{
    float f;
    std::memcpy(&f, &u, 4);
    return f;
}
static inline float __uint2float_rn(uint32_t u) { return (float)u; }  // x86-64 converts round-to-nearest-even
static inline int __ffs(unsigned v) { return __builtin_ffs((int)v); }
using std::max;
using std::min;

#include "shade_math.cuh"

namespace {
crt::DisneyMaterial material_from16(const float *m)
{
    crt::DisneyMaterial d;
    d.base_color = crt::mk3(m[0], m[1], m[2]);
    d.metallic = m[3];
    d.specular = m[4];
    d.roughness = m[5];
    d.specular_tint = m[6];
    d.anisotropy = m[7];
    d.sheen = m[8];
    d.sheen_tint = m[9];
    d.clearcoat = m[10];
    d.clearcoat_gloss = m[11];
    d.ior = m[12];
    d.specular_transmission = m[13];
    return d;
}
crt::QuadLight light_from20(const float *l)
{
    crt::QuadLight q;
    q.emission = crt::mk3(l[0], l[1], l[2]);
    q.position = crt::mk3(l[4], l[5], l[6]);
    q.normal = crt::mk3(l[8], l[9], l[10]);
    q.v_x = crt::mk3(l[12], l[13], l[14]);
    q.width = l[15];
    q.v_y = crt::mk3(l[16], l[17], l[18]);
    q.height = l[19];
    return q;
}
}  // namespace

extern "C" {

void shadekat_rng(uint32_t pixel_id, uint32_t frame_id, uint32_t n, uint32_t *states, float *floats)
{
    uint32_t rng = crt::get_rng(pixel_id, frame_id);
    for (uint32_t i = 0; i < n; ++i) {
        floats[i] = crt::lcg_randomf(rng);
        states[i] = rng;
    }
}
// out: f.xyz, pdf
void shadekat_disney_eval(const float *mat16, const float *n, const float *w_o, const float *w_i, float *out4)
{
    using namespace crt;
    const DisneyMaterial mat = material_from16(mat16);
    const float3 nn = mk3(n[0], n[1], n[2]);
    float3 v_x, v_y;
    ortho_basis(v_x, v_y, nn);
    const float3 wo = mk3(w_o[0], w_o[1], w_o[2]), wi = mk3(w_i[0], w_i[1], w_i[2]);
    const float3 f = disney_brdf(mat, nn, wo, wi, v_x, v_y);
    out4[0] = f.x;
    out4[1] = f.y;
    out4[2] = f.z;
    out4[3] = disney_pdf(mat, nn, wo, wi, v_x, v_y);
}
// rng_state in/out; out: f.xyz, pdf, w_i.xyz
void shadekat_disney_sample(const float *mat16, const float *n, const float *w_o, uint32_t *rng_state, float *out7)
{
    using namespace crt;
    const DisneyMaterial mat = material_from16(mat16);
    const float3 nn = mk3(n[0], n[1], n[2]);
    float3 v_x, v_y;
    ortho_basis(v_x, v_y, nn);
    uint32_t rng = *rng_state;
    float3 w_i = mk3(0.f);
    float pdf = 0.f;
    const float3 f = sample_disney_brdf(mat, nn, mk3(w_o[0], w_o[1], w_o[2]), v_x, v_y, rng, w_i, pdf);
    *rng_state = rng;
    out7[0] = f.x;
    out7[1] = f.y;
    out7[2] = f.z;
    out7[3] = pdf;
    out7[4] = w_i.x;
    out7[5] = w_i.y;
    out7[6] = w_i.z;
}
// light20: QuadLight; out: sample_pos.xyz, pdf(p = sample_pos, dir), hit flag, t, hit_pos.xyz
void shadekat_light(const float *light20, const float *s2, const float *orig, const float *dir, float *out9)
{
    using namespace crt;
    const QuadLight l = light_from20(light20);
    const float3 p = sample_quad_light_position(l, s2[0], s2[1]);
    const float3 o = mk3(orig[0], orig[1], orig[2]), d = mk3(dir[0], dir[1], dir[2]);
    out9[0] = p.x;
    out9[1] = p.y;
    out9[2] = p.z;
    out9[3] = quad_light_pdf(l, p, d);
    float t = 0.f;
    float3 lp = mk3(0.f);
    const bool hit = quad_intersect(l, o, d, t, lp);
    out9[4] = hit ? 1.f : 0.f;
    out9[5] = hit ? t : 0.f;
    out9[6] = hit ? lp.x : 0.f;
    out9[7] = hit ? lp.y : 0.f;
    out9[8] = hit ? lp.z : 0.f;
}
// data: w*h*channels bytes, expanded to the device's RGBA8 arena layout (host_scene.cpp) before sampling
void shadekat_texture(const uint8_t *data, int w, int h, int channels, const float *uv, int n, float *out4n)
{
    using namespace crt;
    std::vector<uint32_t> texels((size_t)w * h);
    for (size_t px = 0; px < (size_t)w * h; ++px) {
        uint32_t c[4] = {0, 0, 0, 0};
        for (int k = 0; k < channels; ++k) {
            c[k] = data[px * channels + k];
        }
        texels[px] = c[0] | (c[1] << 8) | (c[2] << 16) | (c[3] << 24);
    }
    DevTex t;
    t.offset = 0;
    t.width = w;
    t.height = h;
    t.pad = 0;
    for (int i = 0; i < n; ++i) {
        const float4 c = texture_rgba(texels.data(), t, make_float2(uv[2 * i], uv[2 * i + 1]));
        out4n[4 * i] = c.x;
        out4n[4 * i + 1] = c.y;
        out4n[4 * i + 2] = c.z;
        out4n[4 * i + 3] = c.w;
    }
}
// the byte -> [0, 1] table texel channels are converted with (kByteToUnit, read through byte_to_unit)
void shadekat_byte_to_unit(float *out256)
{
    for (uint32_t q = 0; q < 256; ++q) {
        out256[q] = crt::byte_to_unit(q);
    }
}
// unpack_material<false> of material `id` at the n points uv (2n floats) over the RGBA8 arena `texels` and its
// descriptors `tex` (4 int32 each, DevTex); out: 14 floats per point (base_color.xyz, then the 11 scalar parameters)
void shadekat_unpack_material(const float *materials, uint32_t id, const uint32_t *texels, const int32_t *tex,
                              const float *uv, int n, float *out14n)
{
    using namespace crt;
    const TexSource ts{texels, reinterpret_cast<const DevTex *>(tex), nullptr};
    for (int i = 0; i < n; ++i) {
        DisneyMaterial m;
        unpack_material<false>(m, reinterpret_cast<const float4 *>(materials), id, make_float2(uv[2 * i], uv[2 * i + 1]),
                               ts);
        const float v[14] = {m.base_color.x, m.base_color.y, m.base_color.z, m.metallic, m.specular, m.roughness,
                             m.specular_tint, m.anisotropy, m.sheen, m.sheen_tint, m.clearcoat, m.clearcoat_gloss, m.ior,
                             m.specular_transmission};
        std::memcpy(out14n + 14 * i, v, sizeof v);
    }
}
void shadekat_miss(const float *dirs, int n, float *out3n)
{
    for (int i = 0; i < n; ++i) {
        const float3 c = crt::miss_shader(crt::mk3(dirs[3 * i], dirs[3 * i + 1], dirs[3 * i + 2]));
        out3n[3 * i] = c.x;
        out3n[3 * i + 1] = c.y;
        out3n[3 * i + 2] = c.z;
    }
}
void shadekat_ortho_basis(const float *n, float *out6)
{
    float3 vx, vy;
    crt::ortho_basis(vx, vy, crt::mk3(n[0], n[1], n[2]));
    out6[0] = vx.x;
    out6[1] = vx.y;
    out6[2] = vx.z;
    out6[3] = vy.x;
    out6[4] = vy.y;
    out6[5] = vy.z;
}
void shadekat_srgb8(const float *x, int n, uint8_t *out)
{
    for (int i = 0; i < n; ++i) {
        out[i] = (uint8_t)crt::float_to_srgb8(x[i]);
    }
}
}
