// shade_kat.h — TEST-ONLY: the input layouts of the shadekat_* known-answer entry points, shared by the host build
// (shade_hostcheck.cpp, g++) and the device build (shade_devcheck.cu, nvcc) of shade_math.cuh. Include after it.
#pragma once

#include <cstdint>
#include <vector>

namespace crt {

// 16 floats: base_color.xyz, metallic, specular, roughness, specular_tint, anisotropy, sheen, sheen_tint, clearcoat,
// clearcoat_gloss, ior, specular_transmission, (2 unused)
CRT_D DisneyMaterial material_from16(const float *m)
{
    DisneyMaterial d;
    d.base_color = mk3(m[0], m[1], m[2]);
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
// 20 floats: the five float4 rows of the device's light record (load_light)
CRT_D QuadLight light_from20(const float *l)
{
    QuadLight q;
    q.emission = mk3(l[0], l[1], l[2]);
    q.position = mk3(l[4], l[5], l[6]);
    q.normal = mk3(l[8], l[9], l[10]);
    q.v_x = mk3(l[12], l[13], l[14]);
    q.width = l[15];
    q.v_y = mk3(l[16], l[17], l[18]);
    q.height = l[19];
    return q;
}
// w*h*channels bytes expanded to the device's RGBA8 arena layout (host_scene.cpp): missing channels are 0
inline std::vector<uint32_t> rgba8_arena(const uint8_t *data, int w, int h, int channels)
{
    std::vector<uint32_t> texels((size_t)w * h);
    for (size_t px = 0; px < texels.size(); ++px) {
        uint32_t c[4] = {0, 0, 0, 0};
        for (int k = 0; k < channels; ++k) {
            c[k] = data[px * channels + k];
        }
        texels[px] = c[0] | (c[1] << 8) | (c[2] << 16) | (c[3] << 24);
    }
    return texels;
}

// ---- one known-answer input each: what the shadekat_* entry points compute per input ----
// get_rng(pixel_id, frame_id), then k draws: the state after each and its float
CRT_D void kat_rng(uint32_t pixel_id, uint32_t frame_id, uint32_t k, uint32_t *states, float *floats)
{
    uint32_t rng = get_rng(pixel_id, frame_id);
    for (uint32_t i = 0; i < k; ++i) {
        floats[i] = lcg_randomf(rng);
        states[i] = rng;
    }
}
// out: f.xyz, pdf
CRT_D void kat_disney_eval(const float *mat16, const float *n, const float *w_o, const float *w_i, float *out4)
{
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
CRT_D void kat_disney_sample(const float *mat16, const float *n, const float *w_o, uint32_t *rng_state, float *out7)
{
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
// out: sample_pos.xyz, pdf(p = sample_pos, dir), hit flag, t, hit_pos.xyz
CRT_D void kat_light(const float *light20, const float *s2, const float *orig, const float *dir, float *out9)
{
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
// out: texture_rgba at (u, v)
CRT_D void kat_texture(const uint32_t *texels, const DevTex t, float u, float v, float *out4)
{
    const float4 c = texture_rgba(texels, t, make_float2(u, v));
    out4[0] = c.x;
    out4[1] = c.y;
    out4[2] = c.z;
    out4[3] = c.w;
}
// out: the 14 floats of unpack_material<false> (base_color.xyz, then the 11 scalar parameters)
CRT_D void kat_unpack_material(const float *materials, uint32_t id, const TexSource &ts, float u, float v, float *out14)
{
    DisneyMaterial m;
    unpack_material<false>(m, reinterpret_cast<const float4 *>(materials), id, make_float2(u, v), ts);
    const float r[14] = {m.base_color.x, m.base_color.y, m.base_color.z, m.metallic, m.specular, m.roughness,
                         m.specular_tint, m.anisotropy, m.sheen, m.sheen_tint, m.clearcoat, m.clearcoat_gloss, m.ior,
                         m.specular_transmission};
    for (int k = 0; k < 14; ++k) {
        out14[k] = r[k];
    }
}
CRT_D void kat_miss(const float *dir, float *out3)
{
    const float3 c = miss_shader(mk3(dir[0], dir[1], dir[2]));
    out3[0] = c.x;
    out3[1] = c.y;
    out3[2] = c.z;
}
CRT_D void kat_ortho_basis(const float *n, float *out6)
{
    float3 vx, vy;
    ortho_basis(vx, vy, mk3(n[0], n[1], n[2]));
    out6[0] = vx.x;
    out6[1] = vx.y;
    out6[2] = vx.z;
    out6[3] = vy.x;
    out6[4] = vy.y;
    out6[5] = vy.z;
}

// shadekat_math_n's function codes: the transcendentals the shading code calls
enum KatMath { kSinf = 0, kCosf, kPowf, kLogf, kAtan2f, kAcosf };
CRT_D float kat_math(int fn, float x, float y)
{
    if (fn == kSinf || fn == kCosf) {  // both of one angle, as sample_disney_dir asks for them
        const float c = cosf(x), s = sinf(x);
        return fn == kSinf ? s : c;
    }
    switch (fn) {
    case kPowf: return powf(x, y);
    case kLogf: return logf(x);
    case kAtan2f: return atan2f(x, y);
    default: return acosf(x);
    }
}

}  // namespace crt
