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

#include "shade_kat.h"

extern "C" {

void shadekat_rng(uint32_t pixel_id, uint32_t frame_id, uint32_t n, uint32_t *states, float *floats)
{
    crt::kat_rng(pixel_id, frame_id, n, states, floats);
}
// out: f.xyz, pdf
void shadekat_disney_eval(const float *mat16, const float *n, const float *w_o, const float *w_i, float *out4)
{
    crt::kat_disney_eval(mat16, n, w_o, w_i, out4);
}
// rng_state in/out; out: f.xyz, pdf, w_i.xyz
void shadekat_disney_sample(const float *mat16, const float *n, const float *w_o, uint32_t *rng_state, float *out7)
{
    crt::kat_disney_sample(mat16, n, w_o, rng_state, out7);
}
// light20: QuadLight; out: sample_pos.xyz, pdf(p = sample_pos, dir), hit flag, t, hit_pos.xyz
void shadekat_light(const float *light20, const float *s2, const float *orig, const float *dir, float *out9)
{
    crt::kat_light(light20, s2, orig, dir, out9);
}
// data: w*h*channels bytes, expanded to the device's RGBA8 arena layout (host_scene.cpp) before sampling
void shadekat_texture(const uint8_t *data, int w, int h, int channels, const float *uv, int n, float *out4n)
{
    const std::vector<uint32_t> texels = crt::rgba8_arena(data, w, h, channels);
    const crt::DevTex t{0u, w, h, 0};
    for (int i = 0; i < n; ++i) {
        crt::kat_texture(texels.data(), t, uv[2 * i], uv[2 * i + 1], out4n + 4 * i);
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
    const crt::TexSource ts{texels, reinterpret_cast<const crt::DevTex *>(tex), nullptr};
    for (int i = 0; i < n; ++i) {
        crt::kat_unpack_material(materials, id, ts, uv[2 * i], uv[2 * i + 1], out14n + 14 * i);
    }
}
void shadekat_miss(const float *dirs, int n, float *out3n)
{
    for (int i = 0; i < n; ++i) {
        crt::kat_miss(dirs + 3 * i, out3n + 3 * i);
    }
}
void shadekat_ortho_basis(const float *n, float *out6)
{
    crt::kat_ortho_basis(n, out6);
}
void shadekat_srgb8(const float *x, int n, uint8_t *out)
{
    for (int i = 0; i < n; ++i) {
        out[i] = (uint8_t)crt::float_to_srgb8(x[i]);
    }
}

// ---- batched: n inputs, n outputs. libcrt_shade_devcheck.so exports the same names and signatures (the same
// per-input functions, one CUDA thread each), so that one test runs against either build (tests/test_shade_device.py).
// Each returns 0 (the device build: a CUDA error code). ----
int shadekat_rng_n(const uint32_t *pixel_ids, const uint32_t *frame_ids, int n, int k, uint32_t *states, float *floats)
{
    for (int i = 0; i < n; ++i) {
        crt::kat_rng(pixel_ids[i], frame_ids[i], (uint32_t)k, states + (size_t)k * i, floats + (size_t)k * i);
    }
    return 0;
}
// one lcg_randomf per state, in place
int shadekat_lcg_n(uint32_t *states, int n, float *floats)
{
    for (int i = 0; i < n; ++i) {
        floats[i] = crt::lcg_randomf(states[i]);
    }
    return 0;
}
int shadekat_disney_eval_n(const float *mat16n, const float *n3n, const float *w_o3n, const float *w_i3n, int n, float *out4n)
{
    for (int i = 0; i < n; ++i) {
        crt::kat_disney_eval(mat16n + 16 * i, n3n + 3 * i, w_o3n + 3 * i, w_i3n + 3 * i, out4n + 4 * i);
    }
    return 0;
}
int shadekat_disney_sample_n(const float *mat16n, const float *n3n, const float *w_o3n, uint32_t *rng_n, int n,
                             float *out7n)
{
    for (int i = 0; i < n; ++i) {
        crt::kat_disney_sample(mat16n + 16 * i, n3n + 3 * i, w_o3n + 3 * i, rng_n + i, out7n + 7 * i);
    }
    return 0;
}
int shadekat_light_n(const float *light20, const float *s2n, const float *orig3n, const float *dir3n, int n, float *out9n)
{
    for (int i = 0; i < n; ++i) {
        crt::kat_light(light20, s2n + 2 * i, orig3n + 3 * i, dir3n + 3 * i, out9n + 9 * i);
    }
    return 0;
}
int shadekat_texture_n(const uint8_t *data, int w, int h, int channels, const float *uv, int n, float *out4n)
{
    shadekat_texture(data, w, h, channels, uv, n, out4n);
    return 0;
}
// n_materials, n_texels, n_tex: the lengths of the three tables (the device build copies them)
int shadekat_unpack_material_n(const float *materials, int n_materials, uint32_t id, const uint32_t *texels, int n_texels,
                               const int32_t *tex, int n_tex, const float *uv, int n, float *out14n)
{
    (void)n_materials, (void)n_texels, (void)n_tex;
    shadekat_unpack_material(materials, id, texels, tex, uv, n, out14n);
    return 0;
}
int shadekat_miss_n(const float *dirs, int n, float *out3n)
{
    shadekat_miss(dirs, n, out3n);
    return 0;
}
int shadekat_ortho_basis_n(const float *n3n, int n, float *out6n)
{
    for (int i = 0; i < n; ++i) {
        crt::kat_ortho_basis(n3n + 3 * i, out6n + 6 * i);
    }
    return 0;
}
int shadekat_srgb8_n(const float *x, int n, uint8_t *out)
{
    shadekat_srgb8(x, n, out);
    return 0;
}
int shadekat_schlick_n(const float *cos_theta, int n, float *out)
{
    for (int i = 0; i < n; ++i) {
        out[i] = crt::schlick_weight(cos_theta[i]);
    }
    return 0;
}
// fn: crt::KatMath (sinf, cosf, powf, logf, atan2f, acosf); y is read by powf and atan2f only
int shadekat_math_n(int fn, const float *x, const float *y, int n, float *out)
{
    for (int i = 0; i < n; ++i) {
        out[i] = crt::kat_math(fn, x[i], y ? y[i] : 0.f);
    }
    return 0;
}
}
