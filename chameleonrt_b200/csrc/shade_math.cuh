// shade_math.cuh — device-side shading arithmetic of the wavefront path tracer.
//
// Every function states the reference code whose arithmetic it reproduces (operation order
// kept; the translation unit is compiled with -fmad=false, so nothing is contracted unless
// written as an explicit fma). Paths are relative to /root/reference/backends/embree/.
//   lcg_rng.ih:8-59     get_rng / lcg_random / lcg_randomf
//   util.ih:24-82       pow2, luminance, ortho_basis, mod, saturate, lerp, reflect, refract
//   float3.ih           vector operators (normalize multiplies by 1/length)
//   texture2d.ih:13-83  bilinear, wrap addressing, float->int truncation of texel coords
//   lights.ih:26-69     quad light sample / pdf / intersect
//   disney_bsdf.ih      Disney BSDF: eval, pdf, sample
//   render_embree.ispc:66-103   unpack_material; :183-196 miss_shader
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

namespace crt {

#define CRT_D __device__ __forceinline__

constexpr float kPi = 3.14159265358979323846f;
constexpr float kInvPi = 0.318309886183790671538f;
constexpr float kEpsilon = 0.0001f;

// ---- float3.ih ----
CRT_D float3 mk3(float x, float y, float z) { return make_float3(x, y, z); }
CRT_D float3 mk3(float c) { return make_float3(c, c, c); }
CRT_D float3 operator+(const float3 a, const float3 b) { return mk3(a.x + b.x, a.y + b.y, a.z + b.z); }
CRT_D float3 operator-(const float3 a, const float3 b) { return mk3(a.x - b.x, a.y - b.y, a.z - b.z); }
CRT_D float3 operator*(const float3 a, const float3 b) { return mk3(a.x * b.x, a.y * b.y, a.z * b.z); }
CRT_D float3 operator*(const float3 a, const float s) { return mk3(a.x * s, a.y * s, a.z * s); }
CRT_D float3 operator*(const float s, const float3 a) { return mk3(a.x * s, a.y * s, a.z * s); }
CRT_D float3 operator/(const float3 a, const float s) { return mk3(a.x / s, a.y / s, a.z / s); }
CRT_D float3 neg(const float3 a) { return mk3(-a.x, -a.y, -a.z); }
CRT_D float dot(const float3 a, const float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
CRT_D float length(const float3 v) { return sqrtf(v.x * v.x + v.y * v.y + v.z * v.z); }
CRT_D float3 normalize(const float3 v)
{
    const float c = 1.f / length(v);
    return mk3(v.x * c, v.y * c, v.z * c);
}
CRT_D float3 cross(const float3 a, const float3 b)
{
    return mk3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
CRT_D bool all_zero(const float3 v) { return v.x == 0.f && v.y == 0.f && v.z == 0.f; }

// ---- util.ih ----
CRT_D float pow2(float x) { return x * x; }
CRT_D float luminance(const float3 c) { return 0.2126f * c.x + 0.7152f * c.y + 0.0722f * c.z; }
CRT_D float clampf(float x, float lo, float hi) { return x < lo ? lo : (x > hi ? hi : x); }
CRT_D float saturate(float x) { return clampf(x, 0.f, 1.f); }
CRT_D float lerp(float x, float y, float s) { return x * (1.f - s) + y * s; }
CRT_D float3 lerp(float3 x, float3 y, float s) { return x * (1.f - s) + y * s; }
CRT_D float3 reflect(const float3 i, const float3 n) { return i - 2.f * n * dot(i, n); }
CRT_D float3 refract(const float3 i, const float3 n, float eta)
{
    const float n_dot_i = dot(n, i);
    const float k = 1.f - eta * eta * (1.f - n_dot_i * n_dot_i);
    if (k < 0.f) {
        return mk3(0.f);
    }
    return eta * i - (eta * n_dot_i + sqrtf(k)) * n;
}
CRT_D void ortho_basis(float3 &v_x, float3 &v_y, const float3 n)
{
    v_y = mk3(0.f);
    if (n.x < 0.6f && n.x > -0.6f) {
        v_y.x = 1.f;
    } else if (n.y < 0.6f && n.y > -0.6f) {
        v_y.y = 1.f;
    } else if (n.z < 0.6f && n.z > -0.6f) {
        v_y.z = 1.f;
    } else {
        v_y.x = 1.f;
    }
    v_x = normalize(cross(v_y, n));
    v_y = normalize(cross(n, v_x));
}
CRT_D int modi(int a, int b)
{
    if (b == 0) {
        b = 1;
    }
    const int r = a - (a / b) * b;
    return r < 0 ? r + b : r;
}

// ---- lcg_rng.ih ----
CRT_D uint32_t murmur_hash3_mix(uint32_t hash, uint32_t k)
{
    k *= 0xcc9e2d51u;
    k = (k << 15) | (k >> 17);
    k *= 0x1b873593u;
    hash ^= k;
    hash = ((hash << 13) | (hash >> 19)) * 5u + 0xe6546b64u;
    return hash;
}
CRT_D uint32_t murmur_hash3_finalize(uint32_t hash)
{
    hash ^= hash >> 16;
    hash *= 0x85ebca6bu;
    hash ^= hash >> 13;
    hash *= 0xc2b2ae35u;
    hash ^= hash >> 16;
    return hash;
}
CRT_D uint32_t get_rng(uint32_t pixel_id, uint32_t frame_id)
{
    uint32_t s = murmur_hash3_mix(0u, pixel_id);
    s = murmur_hash3_mix(s, frame_id);
    return murmur_hash3_finalize(s);
}
// ldexp((float)state, -32): round-to-nearest u32->f32 then an exact power-of-two scale
CRT_D float lcg_randomf(uint32_t &state)
{
    state = state * 1664525u + 1013904223u;
    return __uint2float_rn(state) * 2.3283064365386963e-10f;
}

// ---- texture2d.ih ----
struct DevTex {
    uint32_t offset;
    int32_t width, height;
    int32_t pad;
};
// (float)q / 255.f for every byte q, correctly rounded (the division is done once, by the compiler). A texel channel
// is converted by a lookup instead of an IEEE division (about ten instructions with its slow-path branch on the
// device). Global memory read through __ldg, not __constant__: the lanes of a warp look up different bytes, and the
// constant cache serialises different addresses. tests/test_byte_table_host.py checks every entry bit for bit.
struct ByteToUnit {
    float v[256];
};
constexpr ByteToUnit make_byte_to_unit()
{
    ByteToUnit t{};
    for (int q = 0; q < 256; ++q) {
        t.v[q] = (float)q / 255.f;
    }
    return t;
}
__device__ const ByteToUnit kByteToUnit = make_byte_to_unit();
CRT_D float byte_to_unit(uint32_t q) { return __ldg(kByteToUnit.v + q); }

// (int)x as x86-64 converts it (cvttss2si): truncation toward zero, and INT_MIN for NaN and for every x outside
// [-2^31, 2^31). The reference, the oracle and the host builds of this file convert texel coordinates that way; the
// device's own conversion saturates and maps NaN to 0, which for a finite uv*width >= 2^31 picks texel column
// INT_MAX mod width instead of INT_MIN mod width.
CRT_D int float_to_int_x86(float x)
{
    return (x >= -2147483648.f && x < 2147483648.f) ? (int)x : INT32_MIN;
}

// The four texel words under the bilinear footprint of uv and the weights of the filter (texture2d.ih:13-83).
struct TexelQuad {
    uint32_t p00, p10, p01, p11;
    float tx, ty;
};
CRT_D TexelQuad texel_quad(const uint32_t *__restrict__ texels, const DevTex t, const float2 uv)
{
    const float ux = uv.x * (float)t.width - 0.5f;
    const float uy = uv.y * (float)t.height - 0.5f;
    TexelQuad q;
    q.tx = ux - floorf(ux);
    q.ty = uy - floorf(uy);
    const int x0 = modi(float_to_int_x86(ux), t.width), y0 = modi(float_to_int_x86(uy), t.height);
    const int x1 = modi(float_to_int_x86(ux + 1.f), t.width), y1 = modi(float_to_int_x86(uy + 1.f), t.height);
    const uint32_t *const base = texels + t.offset;
    q.p00 = __ldg(base + (uint32_t)(y0 * t.width + x0));
    q.p10 = __ldg(base + (uint32_t)(y0 * t.width + x1));
    q.p01 = __ldg(base + (uint32_t)(y1 * t.width + x0));
    q.p11 = __ldg(base + (uint32_t)(y1 * t.width + x1));
    return q;
}
// One channel (0 = r .. 3 = a) of the filtered texel:
// s00*(1-tx)*(1-ty) + s10*tx*(1-ty) + s01*(1-tx)*ty + s11*tx*ty, left to right
CRT_D float bilinear_channel(const TexelQuad &q, uint32_t ch)
{
    const uint32_t s = 8u * ch;
    const float s00 = byte_to_unit((q.p00 >> s) & 0xffu), s10 = byte_to_unit((q.p10 >> s) & 0xffu);
    const float s01 = byte_to_unit((q.p01 >> s) & 0xffu), s11 = byte_to_unit((q.p11 >> s) & 0xffu);
    const float w00 = (1.f - q.tx), w10 = q.tx;
    return s00 * w00 * (1.f - q.ty) + s10 * w10 * (1.f - q.ty) + s01 * w00 * q.ty + s11 * w10 * q.ty;
}
CRT_D float4 texture_rgba(const uint32_t *__restrict__ texels, const DevTex t, const float2 uv)
{
    const TexelQuad q = texel_quad(texels, t, uv);
    return make_float4(bilinear_channel(q, 0), bilinear_channel(q, 1), bilinear_channel(q, 2), bilinear_channel(q, 3));
}
CRT_D float channel_of(const float4 c, uint32_t ch)
{
    return ch == 0 ? c.x : (ch == 1 ? c.y : (ch == 2 ? c.z : c.w));
}

// ---- lights.ih ----
struct QuadLight {
    float3 emission;
    float3 position;
    float3 normal;
    float3 v_x;
    float width;
    float3 v_y;
    float height;
};
CRT_D QuadLight load_light(const float4 *__restrict__ lights, uint32_t id)
{
    const float4 a = __ldg(lights + 5 * id), b = __ldg(lights + 5 * id + 1), c = __ldg(lights + 5 * id + 2),
                 d = __ldg(lights + 5 * id + 3), e = __ldg(lights + 5 * id + 4);
    QuadLight l;
    l.emission = mk3(a.x, a.y, a.z);
    l.position = mk3(b.x, b.y, b.z);
    l.normal = mk3(c.x, c.y, c.z);
    l.v_x = mk3(d.x, d.y, d.z);
    l.width = d.w;
    l.v_y = mk3(e.x, e.y, e.z);
    l.height = e.w;
    return l;
}
CRT_D float3 sample_quad_light_position(const QuadLight &light, float sx, float sy)
{
    return sx * light.v_x * light.width + sy * light.v_y * light.height + light.position;
}
// to_pt = p - dir (sic), lights.ih:41
CRT_D float quad_light_pdf(const QuadLight &light, const float3 p, const float3 dir)
{
    const float surface_area = light.width * light.height;
    const float3 to_pt = p - dir;
    const float dist_sqr = dot(to_pt, to_pt);
    const float n_dot_w = dot(light.normal, neg(dir));
    if (n_dot_w < kEpsilon) {
        return 0.f;
    }
    return dist_sqr / (n_dot_w * surface_area);
}
CRT_D bool quad_intersect(const QuadLight &light, const float3 orig, const float3 dir, float &t, float3 &light_pos)
{
    const float denom = dot(dir, light.normal);
    if (denom != 0.f) {
        t = dot(light.position - orig, light.normal) / denom;
        if (t < 0.f) {
            return false;
        }
        light_pos = orig + dir * t;
        const float3 hit_v = light_pos - light.position;
        if (fabsf(dot(hit_v, light.v_x)) < light.width && fabsf(dot(hit_v, light.v_y)) < light.height) {
            return true;
        }
    }
    return false;
}

// ---- disney_bsdf.ih ----
struct DisneyMaterial {
    float3 base_color;
    float metallic;
    float specular;
    float roughness;
    float specular_tint;
    float anisotropy;
    float sheen;
    float sheen_tint;
    float clearcoat;
    float clearcoat_gloss;
    float ior;
    float specular_transmission;
};

CRT_D bool same_hemisphere(const float3 w_o, const float3 w_i, const float3 n)
{
    return dot(w_o, n) * dot(w_i, n) > 0.f;
}
CRT_D float3 cos_sample_hemisphere(float ux, float uy)
{
    const float sx = 2.f * ux - 1.f, sy = 2.f * uy - 1.f;
    float radius = 0.f, theta = 0.f;
    if (!(sx == 0.f && sy == 0.f)) {
        if (fabsf(sx) > fabsf(sy)) {
            radius = sx;
            theta = kPi / 4.f * (sy / sx);
        } else {
            radius = sy;
            theta = kPi / 2.f - kPi / 4.f * (sx / sy);
        }
    }
    const float dx = radius * cosf(theta), dy = radius * sinf(theta);
    return mk3(dx, dy, sqrtf(fmaxf(0.f, 1.f - dx * dx - dy * dy)));
}
CRT_D float3 spherical_dir(float sin_theta, float cos_theta, float phi)
{
    return mk3(sin_theta * cosf(phi), sin_theta * sinf(phi), cos_theta);
}
CRT_D float power_heuristic(float n_f, float pdf_f, float n_g, float pdf_g)
{
    const float f = n_f * pdf_f;
    const float g = n_g * pdf_g;
    return (f * f) / (f * f + g * g);
}
// disney_bsdf.ih:74-76 is pow(saturate(1 - cos_theta), 5). Evaluated here as m^2 * m^2 * m: powf is
// ~100 instructions and this weight is needed ~10 times per shaded hit (it was about a third of
// k_shade's instructions); the product is within 3 ulp of the exact m^5 (2.92 ulp at most over every float
// cos_theta in [0, 1]: tests/test_shade_device.py), pow within half an ulp; the reference's own ISPC pow under
// --opt=fast-math is no closer. One of the two documented arithmetic deviations (DESIGN.md §4).
CRT_D float schlick_weight(float cos_theta)
{
    const float m = saturate(1.f - cos_theta);
#if defined(CRT_SCHLICK_POWF)  // test builds of the host checks only: the reference's own formula
    return powf(m, 5.f);
#else
    const float m2 = m * m;
    return m2 * m2 * m;
#endif
}
CRT_D float fresnel_dielectric(float cos_theta_i, float eta_i, float eta_t)
{
    const float g = pow2(eta_t) / pow2(eta_i) - 1.f + pow2(cos_theta_i);
    if (g < 0.f) {
        return 1.f;
    }
    return 0.5f * pow2(g - cos_theta_i) / pow2(g + cos_theta_i) *
           (1.f + pow2(cos_theta_i * (g + cos_theta_i) - 1.f) / pow2(cos_theta_i * (g - cos_theta_i) + 1.f));
}
CRT_D float gtr_1(float cos_theta_h, float alpha)
{
    if (alpha >= 1.f) {
        return kInvPi;
    }
    const float alpha_sqr = alpha * alpha;
    return kInvPi * (alpha_sqr - 1.f) / (logf(alpha_sqr) * (1.f + (alpha_sqr - 1.f) * cos_theta_h * cos_theta_h));
}
CRT_D float gtr_2(float cos_theta_h, float alpha)
{
    const float alpha_sqr = alpha * alpha;
    return kInvPi * alpha_sqr / pow2(1.f + (alpha_sqr - 1.f) * cos_theta_h * cos_theta_h);
}
CRT_D float gtr_2_aniso(float h_dot_n, float h_dot_x, float h_dot_y, float ax, float ay)
{
    return kInvPi / (ax * ay * pow2(pow2(h_dot_x / ax) + pow2(h_dot_y / ay) + h_dot_n * h_dot_n));
}
CRT_D float smith_shadowing_ggx(float n_dot_o, float alpha_g)
{
    const float a = alpha_g * alpha_g;
    const float b = n_dot_o * n_dot_o;
    return 1.f / (n_dot_o + sqrtf(a + b - a * b));
}
CRT_D float smith_shadowing_ggx_aniso(float n_dot_o, float o_dot_x, float o_dot_y, float ax, float ay)
{
    return 1.f / (n_dot_o + sqrtf(pow2(o_dot_x * ax) + pow2(o_dot_y * ay) + pow2(n_dot_o)));
}
CRT_D float3 to_world(const float3 h, const float3 n, const float3 v_x, const float3 v_y)
{
    return h.x * v_x + h.y * v_y + h.z * n;
}
CRT_D float3 sample_lambertian_dir(const float3 n, const float3 v_x, const float3 v_y, float sx, float sy)
{
    return to_world(normalize(cos_sample_hemisphere(sx, sy)), n, v_x, v_y);
}
CRT_D float3 sample_gtr_1_h(const float3 n, const float3 v_x, const float3 v_y, float alpha, float sx, float sy)
{
    const float phi_h = 2.f * kPi * sx;
    const float alpha_sqr = alpha * alpha;
    const float cos_theta_h_sqr = (1.f - powf(alpha_sqr, 1.f - sy)) / (1.f - alpha_sqr);
    const float cos_theta_h = sqrtf(cos_theta_h_sqr);
    const float sin_theta_h = sqrtf(1.f - cos_theta_h_sqr);
    return to_world(normalize(spherical_dir(sin_theta_h, cos_theta_h, phi_h)), n, v_x, v_y);
}
CRT_D float3 sample_gtr_2_h(const float3 n, const float3 v_x, const float3 v_y, float alpha, float sx, float sy)
{
    const float phi_h = 2.f * kPi * sx;
    const float cos_theta_h_sqr = (1.f - sy) / (1.f + (alpha * alpha - 1.f) * sy);
    const float cos_theta_h = sqrtf(cos_theta_h_sqr);
    const float sin_theta_h = sqrtf(1.f - cos_theta_h_sqr);
    return to_world(normalize(spherical_dir(sin_theta_h, cos_theta_h, phi_h)), n, v_x, v_y);
}
CRT_D float3 sample_gtr_2_aniso_h(const float3 n, const float3 v_x, const float3 v_y, float ax, float ay, float sx,
                                  float sy)
{
    const float x = 2.f * kPi * sx;
    const float3 w_h = sqrtf(sy / (1.f - sy)) * (ax * cosf(x) * v_x + ay * sinf(x) * v_y) + n;
    return normalize(w_h);
}
CRT_D float lambertian_pdf(const float3 w_i, const float3 n)
{
    const float d = dot(w_i, n);
    return d > 0.f ? d * kInvPi : 0.f;
}
CRT_D float gtr_1_pdf(const float3 w_o, const float3 w_i, const float3 n, float alpha)
{
    if (!same_hemisphere(w_o, w_i, n)) {
        return 0.f;
    }
    const float3 w_h = normalize(w_i + w_o);
    const float cos_theta_h = dot(n, w_h);
    const float d = gtr_1(cos_theta_h, alpha);
    return d * cos_theta_h / (4.f * dot(w_o, w_h));
}
CRT_D float gtr_2_pdf(const float3 w_o, const float3 w_i, const float3 n, float alpha)
{
    if (!same_hemisphere(w_o, w_i, n)) {
        return 0.f;
    }
    const float3 w_h = normalize(w_i + w_o);
    const float cos_theta_h = dot(n, w_h);
    const float d = gtr_2(cos_theta_h, alpha);
    return d * cos_theta_h / (4.f * dot(w_o, w_h));
}
CRT_D float gtr_2_transmission_pdf(const float3 w_o, const float3 w_i, const float3 n, float alpha, float ior)
{
    if (same_hemisphere(w_o, w_i, n)) {
        return 0.f;
    }
    const bool entering = dot(w_o, n) > 0.f;
    const float eta_o = entering ? 1.f : ior;
    const float eta_i = entering ? ior : 1.f;
    const float3 w_h = normalize(w_o + w_i * eta_i / eta_o);
    const float cos_theta_h = fabsf(dot(n, w_h));
    const float i_dot_h = dot(w_i, w_h);
    const float o_dot_h = dot(w_o, w_h);
    const float d = gtr_2(cos_theta_h, alpha);
    const float dwh_dwi = o_dot_h * pow2(eta_o) / pow2(eta_o * o_dot_h + eta_i * i_dot_h);
    return d * cos_theta_h * fabsf(dwh_dwi);
}
CRT_D float gtr_2_aniso_pdf(const float3 w_o, const float3 w_i, const float3 n, const float3 v_x, const float3 v_y,
                            float ax, float ay)
{
    if (!same_hemisphere(w_o, w_i, n)) {
        return 0.f;
    }
    const float3 w_h = normalize(w_i + w_o);
    const float cos_theta_h = dot(n, w_h);
    const float d = gtr_2_aniso(cos_theta_h, fabsf(dot(w_h, v_x)), fabsf(dot(w_h, v_y)), ax, ay);
    return d * cos_theta_h / (4.f * dot(w_o, w_h));
}
CRT_D float3 disney_diffuse(const DisneyMaterial &mat, const float3 n, const float3 w_o, const float3 w_i)
{
    const float3 w_h = normalize(w_i + w_o);
    const float n_dot_o = fabsf(dot(w_o, n));
    const float n_dot_i = fabsf(dot(w_i, n));
    const float i_dot_h = dot(w_i, w_h);
    const float fd90 = 0.5f + 2.f * mat.roughness * i_dot_h * i_dot_h;
    const float fi = schlick_weight(n_dot_i);
    const float fo = schlick_weight(n_dot_o);
    return mat.base_color * kInvPi * lerp(1.f, fd90, fi) * lerp(1.f, fd90, fo);
}
CRT_D float3 disney_spec_color(const DisneyMaterial &mat)
{
    const float lum = luminance(mat.base_color);
    const float3 tint = lum > 0.f ? mat.base_color / lum : mk3(1.f);
    return lerp(mat.specular * 0.08f * lerp(mk3(1.f), tint, mat.specular_tint), mat.base_color, mat.metallic);
}
CRT_D float3 disney_microfacet_isotropic(const DisneyMaterial &mat, const float3 n, const float3 w_o,
                                         const float3 w_i)
{
    const float3 w_h = normalize(w_i + w_o);
    const float3 spec = disney_spec_color(mat);
    const float alpha = fmaxf(0.001f, mat.roughness * mat.roughness);
    const float d = gtr_2(dot(n, w_h), alpha);
    const float3 f = lerp(spec, mk3(1.f), schlick_weight(dot(w_i, w_h)));
    const float g = smith_shadowing_ggx(dot(n, w_i), alpha) * smith_shadowing_ggx(dot(n, w_o), alpha);
    return d * f * g;
}
CRT_D float3 disney_microfacet_transmission_isotropic(const DisneyMaterial &mat, const float3 n, const float3 w_o,
                                                      const float3 w_i)
{
    const float o_dot_n = dot(w_o, n);
    const float i_dot_n = dot(w_i, n);
    if (o_dot_n == 0.f || i_dot_n == 0.f) {
        return mk3(0.f);
    }
    const bool entering = o_dot_n > 0.f;
    const float eta_o = entering ? 1.f : mat.ior;
    const float eta_i = entering ? mat.ior : 1.f;
    const float3 w_h = normalize(w_o + w_i * eta_i / eta_o);
    const float alpha = fmaxf(0.001f, mat.roughness * mat.roughness);
    const float d = gtr_2(fabsf(dot(n, w_h)), alpha);
    const float f = fresnel_dielectric(fabsf(dot(w_i, n)), eta_o, eta_i);
    const float g = smith_shadowing_ggx(fabsf(dot(n, w_i)), alpha) * smith_shadowing_ggx(fabsf(dot(n, w_o)), alpha);
    const float i_dot_h = dot(w_i, w_h);
    const float o_dot_h = dot(w_o, w_h);
    const float c = fabsf(o_dot_h) / fabsf(dot(w_o, n)) * fabsf(i_dot_h) / fabsf(dot(w_i, n)) * pow2(eta_o) /
                    pow2(eta_o * o_dot_h + eta_i * i_dot_h);
    return mat.base_color * c * (1.f - f) * g * d;
}
CRT_D float3 disney_microfacet_anisotropic(const DisneyMaterial &mat, const float3 n, const float3 w_o,
                                           const float3 w_i, const float3 v_x, const float3 v_y)
{
    const float3 w_h = normalize(w_i + w_o);
    const float3 spec = disney_spec_color(mat);
    const float aspect = sqrtf(1.f - mat.anisotropy * 0.9f);
    const float a = mat.roughness * mat.roughness;
    const float ax = fmaxf(0.001f, a / aspect), ay = fmaxf(0.001f, a * aspect);
    const float d = gtr_2_aniso(dot(n, w_h), fabsf(dot(w_h, v_x)), fabsf(dot(w_h, v_y)), ax, ay);
    const float3 f = lerp(spec, mk3(1.f), schlick_weight(dot(w_i, w_h)));
    const float g = smith_shadowing_ggx_aniso(dot(n, w_i), fabsf(dot(w_i, v_x)), fabsf(dot(w_i, v_y)), ax, ay) *
                    smith_shadowing_ggx_aniso(dot(n, w_o), fabsf(dot(w_o, v_x)), fabsf(dot(w_o, v_y)), ax, ay);
    return d * f * g;
}
CRT_D float disney_clear_coat(const DisneyMaterial &mat, const float3 n, const float3 w_o, const float3 w_i)
{
    const float3 w_h = normalize(w_i + w_o);
    const float alpha = lerp(0.1f, 0.001f, mat.clearcoat_gloss);
    const float d = gtr_1(dot(n, w_h), alpha);
    const float f = lerp(0.04f, 1.f, schlick_weight(dot(w_i, n)));
    const float g = smith_shadowing_ggx(dot(n, w_i), 0.25f) * smith_shadowing_ggx(dot(n, w_o), 0.25f);
    return 0.25f * mat.clearcoat * d * f * g;
}
CRT_D float3 disney_sheen(const DisneyMaterial &mat, const float3 n, const float3 w_i)
{
    const float lum = luminance(mat.base_color);
    const float3 tint = lum > 0.f ? mat.base_color / lum : mk3(1.f);
    const float3 sheen_color = lerp(mk3(1.f), tint, mat.sheen_tint);
    const float f = schlick_weight(dot(w_i, n));
    return f * mat.sheen * sheen_color;
}
// disney_bsdf.ih:311-332
CRT_D float3 disney_brdf(const DisneyMaterial &mat, const float3 n, const float3 w_o, const float3 w_i,
                         const float3 v_x, const float3 v_y)
{
    if (!same_hemisphere(w_o, w_i, n)) {
        if (mat.specular_transmission > 0.f) {
            const float3 spec_trans = disney_microfacet_transmission_isotropic(mat, n, w_o, w_i);
            return spec_trans * (1.f - mat.metallic) * mat.specular_transmission;
        }
        return mk3(0.f);
    }
    const float coat = disney_clear_coat(mat, n, w_o, w_i);
    const float3 sheen = disney_sheen(mat, n, w_i);
    const float3 diffuse = disney_diffuse(mat, n, w_o, w_i);
    float3 gloss;
    if (mat.anisotropy == 0.f) {
        gloss = disney_microfacet_isotropic(mat, n, w_o, w_i);
    } else {
        gloss = disney_microfacet_anisotropic(mat, n, w_o, w_i, v_x, v_y);
    }
    const float3 r = (diffuse + sheen) * (1.f - mat.metallic) * (1.f - mat.specular_transmission) + gloss;
    return mk3(r.x + coat, r.y + coat, r.z + coat);
}
// disney_bsdf.ih:334-359
CRT_D float disney_pdf(const DisneyMaterial &mat, const float3 n, const float3 w_o, const float3 w_i,
                       const float3 v_x, const float3 v_y)
{
    const float alpha = fmaxf(0.001f, mat.roughness * mat.roughness);
    const float aspect = sqrtf(1.f - mat.anisotropy * 0.9f);
    const float ax = fmaxf(0.001f, alpha / aspect), ay = fmaxf(0.001f, alpha * aspect);
    const float clearcoat_alpha = lerp(0.1f, 0.001f, mat.clearcoat_gloss);
    const float diffuse = lambertian_pdf(w_i, n);
    const float clear_coat = gtr_1_pdf(w_o, w_i, n, clearcoat_alpha);
    float n_comp = 3.f;
    float microfacet;
    float microfacet_transmission = 0.f;
    if (mat.anisotropy == 0.f) {
        microfacet = gtr_2_pdf(w_o, w_i, n, alpha);
    } else {
        microfacet = gtr_2_aniso_pdf(w_o, w_i, n, v_x, v_y, ax, ay);
    }
    if (mat.specular_transmission > 0.f) {
        n_comp = 4.f;
        microfacet_transmission = gtr_2_transmission_pdf(w_o, w_i, n, alpha, mat.ior);
    }
    return (diffuse + microfacet + microfacet_transmission + clear_coat) / n_comp;
}
// disney_bsdf.ih:364-413: the sampling half of sample_disney_brdf (lobe choice + direction). Consumes exactly three
// random numbers. Returns false where the reference returns early with pdf = 0 and a zero BSDF value (w_i is then the
// value the reference leaves in it).
//
// The lobe is drawn per lane, so a warp executes every lobe's code one after the other at a third of its lanes (round-2
// source profile of k_shade: 17 % of its instructions at 10.7 of 32 lanes). The three samplers share most of their work —
// one cosine and one sine of an angle, the normalisation and the change of basis of a local direction, the reflection
// about the half vector — and only what differs is left inside the per-lobe branches: the angle and the two radial
// terms. Per lane the operations and their order are exactly those of sample_lambertian_dir / sample_gtr_2_h /
// sample_gtr_1_h / sample_gtr_2_aniso_h above (bit-identical results: tests/test_shade_host.py).
CRT_D bool sample_disney_dir(const DisneyMaterial &mat, const float3 n, const float3 w_o, const float3 v_x,
                             const float3 v_y, uint32_t &rng, float3 &w_i)
{
    int component;
    if (mat.specular_transmission == 0.f) {
        component = (int)(lcg_randomf(rng) * 3.f);
        component = min(max(component, 0), 2);
    } else {
        component = (int)(lcg_randomf(rng) * 4.f);
        component = min(max(component, 0), 3);
    }
    const float sx = lcg_randomf(rng);
    const float sy = lcg_randomf(rng);
    const bool aniso = component == 1 && mat.anisotropy != 0.f;
    // ---- per lobe: the angle, and the radial terms of the local direction (a cos, a sin, z) ----
    float angle, a = 0.f, z = 0.f;
    if (component == 0) {  // cos_sample_hemisphere: concentric map
        const float ux = 2.f * sx - 1.f, uy = 2.f * sy - 1.f;
        float radius = 0.f, theta = 0.f;
        if (!(ux == 0.f && uy == 0.f)) {
            if (fabsf(ux) > fabsf(uy)) {
                radius = ux;
                theta = kPi / 4.f * (uy / ux);
            } else {
                radius = uy;
                theta = kPi / 2.f - kPi / 4.f * (ux / uy);
            }
        }
        angle = theta;
        a = radius;
    } else {
        angle = 2.f * kPi * sx;  // phi_h (sample_gtr_1_h, sample_gtr_2_h) and x (sample_gtr_2_aniso_h)
        if (!aniso) {
            float cos_theta_h_sqr;
            if (component == 2) {  // sample_gtr_1_h
                const float alpha = lerp(0.1f, 0.001f, mat.clearcoat_gloss);
                const float alpha_sqr = alpha * alpha;
                cos_theta_h_sqr = (1.f - powf(alpha_sqr, 1.f - sy)) / (1.f - alpha_sqr);
            } else {  // sample_gtr_2_h (reflection and transmission lobes)
                const float alpha = fmaxf(0.001f, mat.roughness * mat.roughness);
                cos_theta_h_sqr = (1.f - sy) / (1.f + (alpha * alpha - 1.f) * sy);
            }
            z = sqrtf(cos_theta_h_sqr);
            a = sqrtf(1.f - cos_theta_h_sqr);
        }
    }
    // ---- shared: one cosine, one sine ----
    const float c = cosf(angle), s = sinf(angle);
    float3 w;  // comp 0: the sampled direction; others: the half vector
    if (aniso) {  // sample_gtr_2_aniso_h
        const float alpha = fmaxf(0.001f, mat.roughness * mat.roughness);
        const float aspect = sqrtf(1.f - mat.anisotropy * 0.9f);
        const float ax = fmaxf(0.001f, alpha / aspect), ay = fmaxf(0.001f, alpha * aspect);
        w = normalize(sqrtf(sy / (1.f - sy)) * (ax * c * v_x + ay * s * v_y) + n);
    } else {
        // ---- shared: local direction -> normalise -> world ----
        const float hx = a * c, hy = a * s;
        const float hz = component == 0 ? sqrtf(fmaxf(0.f, 1.f - hx * hx - hy * hy)) : z;
        w = to_world(normalize(mk3(hx, hy, hz)), n, v_x, v_y);
    }
    if (component == 0) {
        w_i = w;
        return true;
    }
    if (component != 3) {  // the two reflection lobes
        w_i = reflect(neg(w_o), w);
        if (!same_hemisphere(w_o, w_i, n)) {
            w_i = mk3(0.f);
            return false;
        }
        return true;
    }
    if (dot(w_o, w) < 0.f) {
        w = neg(w);
    }
    const bool entering = dot(w_o, n) > 0.f;
    w_i = refract(neg(w_o), w, entering ? 1.f / mat.ior : mat.ior);
    return !all_zero(w_i);
}
// disney_bsdf.ih:364-429
CRT_D float3 sample_disney_brdf(const DisneyMaterial &mat, const float3 n, const float3 w_o, const float3 v_x,
                                const float3 v_y, uint32_t &rng, float3 &w_i, float &pdf)
{
    if (!sample_disney_dir(mat, n, w_o, v_x, v_y, rng, w_i)) {
        pdf = 0.f;
        return mk3(0.f);
    }
    pdf = disney_pdf(mat, n, w_o, w_i, v_x, v_y);
    return disney_brdf(mat, n, w_o, w_i, v_x, v_y);
}

// ---- render_embree.ispc:66-103 ----
// Where texels come from: the RGBA8 arena + descriptors of the software bilinear filter (texture_rgba: the reference's
// texture2d.ih, bit for bit), or — option "hw_textures", template parameter HW — one cudaTextureObject_t per texture
// (wrap addressing, linear filtering, normalised coordinates, sRGB decode in the texture unit: what the reference's
// OptiX backend does, backends/optix/optix_utils.cpp:60-85). The hardware path differs from the Embree path in the
// filter weights (8-bit fixed point) and in not re-quantising the linearised texels to 8 bits (render_embree.cpp:96-103
// does), so it has its own, looser parity tolerance (tests/test_z_new_gpu_paths.py).
struct TexSource {
    const uint32_t *texels;
    const DevTex *tex;
    const unsigned long long *objects;  // cudaTextureObject_t per texture (HW only)
};
template <bool HW>
CRT_D float4 texture_sample(const TexSource &ts, uint32_t tex_id, const float2 uv)
{
#if defined(__CUDA_ARCH__)
    if (HW) {
        return tex2D<float4>((cudaTextureObject_t)__ldg(ts.objects + tex_id), uv.x, uv.y);
    }
#endif
    return texture_rgba(ts.texels, ts.tex[tex_id], uv);
}
// A parameter word with bit 31 set is textured: bits 0-28 the texture id, bits 29-30 the channel of its texel.
template <bool HW>
CRT_D void unpack_material(DisneyMaterial &mat, const float4 *__restrict__ materials, uint32_t id, const float2 uv,
                           const TexSource &ts)
{
    const float4 m0 = __ldg(materials + 4 * id), m1 = __ldg(materials + 4 * id + 1),
                 m2 = __ldg(materials + 4 * id + 2), m3 = __ldg(materials + 4 * id + 3);
    const uint32_t mask = __float_as_uint(m0.x);
    if (mask & 0x80000000u) {
        const uint32_t tex_id = mask & 0x1fffffffu;
        if (HW) {
            const float4 c = texture_sample<HW>(ts, tex_id, uv);
            mat.base_color = mk3(c.x, c.y, c.z);
        } else {
            const TexelQuad q = texel_quad(ts.texels, ts.tex[tex_id], uv);
            mat.base_color = mk3(bilinear_channel(q, 0), bilinear_channel(q, 1), bilinear_channel(q, 2));
        }
    } else {
        mat.base_color = mk3(m0.x, m0.y, m0.z);
    }
    // The 11 scalar parameters, in the order of their words (m0.w, m1.xyzw, m2.xyzw, m3.xy). The textured ones are
    // filtered at ONE fetch site, in a loop that is not unrolled: each step filters the one channel it needs, and a
    // parameter on the same texture as the step before reuses its texel words (the metallic / roughness maps of glTF
    // share one texture). Inlining a full RGBA fetch per parameter had made this function most of k_shade's code.
    float p[11] = {m0.w, m1.x, m1.y, m1.z, m1.w, m2.x, m2.y, m2.z, m2.w, m3.x, m3.y};
    uint32_t textured = 0u;
#pragma unroll
    for (int k = 0; k < 11; ++k) {
        textured |= (__float_as_uint(p[k]) >> 31) << k;
    }
    const float *const words = reinterpret_cast<const float *>(materials + 4 * id) + 3;  // words[k] is p[k]
    uint32_t cur_tex = 0xffffffffu;  // (no texture id: ids have bits 29-31 clear)
    TexelQuad q{0u, 0u, 0u, 0u, 0.f, 0.f};
    float4 c = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
    while (textured) {
        const int k = __ffs(textured) - 1;
        textured &= textured - 1u;
        const uint32_t w = __float_as_uint(__ldg(words + k));
        const uint32_t tex_id = w & 0x1fffffffu, channel = (w >> 29) & 0x3u;
        float v;
        if (HW) {
            if (tex_id != cur_tex) {
                c = texture_sample<HW>(ts, tex_id, uv);
            }
            v = channel_of(c, channel);
        } else {
            if (tex_id != cur_tex) {
                q = texel_quad(ts.texels, ts.tex[tex_id], uv);
            }
            v = bilinear_channel(q, channel);
        }
        cur_tex = tex_id;
#pragma unroll
        for (int j = 0; j < 11; ++j) {  // p[k] = v with k known only at run time: selects keep p in registers
            if (j == k) {
                p[j] = v;
            }
        }
    }
    mat.metallic = p[0];
    mat.specular = p[1];
    mat.roughness = p[2];
    mat.specular_tint = p[3];
    mat.anisotropy = p[4];
    mat.sheen = p[5];
    mat.sheen_tint = p[6];
    mat.clearcoat = p[7];
    mat.clearcoat_gloss = p[8];
    mat.ior = p[9];
    mat.specular_transmission = p[10];
}
// (the software path under its round-1 signature: the test-only host builds call it)
CRT_D void unpack_material(DisneyMaterial &mat, const float4 *__restrict__ materials, uint32_t id, const float2 uv,
                           const uint32_t *__restrict__ texels, const DevTex *__restrict__ tex)
{
    const TexSource ts{texels, tex, nullptr};
    unpack_material<false>(mat, materials, id, uv, ts);
}

// render_embree.ispc:183-196
CRT_D float3 miss_shader(const float3 dir)
{
    const float u = (1.f + atan2f(dir.x, -dir.z) * kInvPi) * 0.5f;
    const float v = acosf(dir.y) * kInvPi;
    const int check_x = (int)(u * 10.f);
    const int check_y = (int)(v * 10.f);
    if (dir.y > -0.1f && modi(check_x + check_y, 2) == 0) {
        return mk3(0.5f);
    }
    return mk3(0.1f);
}

// float_to_srgb8 restated as round-to-nearest of the exact curve (DESIGN.md §4)
CRT_D uint32_t float_to_srgb8(float x)
{
    if (!(x > 0.f)) {
        return 0u;
    }
    if (x >= 1.f) {
        return 255u;
    }
    const float s = x <= 0.0031308f ? 12.92f * x : 1.055f * powf(x, 1.f / 2.4f) - 0.055f;
    return (uint32_t)(s * 255.f + 0.5f);
}

}  // namespace crt
