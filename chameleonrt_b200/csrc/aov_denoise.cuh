// aov_denoise.cuh — first-hit AOV buffers (option "aov") and the edge-aware à-trous denoiser behind crtc_denoise.
//
//   k_aov_primary   after the primary-ray traversal, before k_shade(0): albedo, coverage, normal and depth of the primary
//                   hits, folded into a per-pixel running mean with k_resolve's formula
//   k_aov_moments   after k_resolve: the first two moments of the per-sample luminance, same running mean
//   k_dn_prepare    demodulated radiance, variance of the pixel mean, unit normals, depth and its screen gradient
//   k_dn_atrous     one à-trous iteration of the spatial part of SVGF (Schied et al. 2017); the last one remodulates and
//                   writes float RGB and sRGB8
//
// Per-pixel AOV layout, kAovFloats floats: albedo.rgb, coverage, normal.xyz (mean of the face-forwarded unit normals, not
// renormalised), depth (mean hit distance over the samples that hit), lum_m1, lum_m2. Like accum there is a tile-local
// copy (the running mean's state) and a full row-major copy. The AOV kernels read only the path state and the scene and
// write only these buffers, so a frame renders exactly the same with and without them.
//
// Every kernel is launched through aov_launch: chevrons under nvcc, simt::launch in the host build of the renderer
// (tests/simt_emu), which compiles this header unchanged. Grids are one-dimensional for the same reason.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "cuda_host_utils.h"
#include "kernels.cuh"

namespace crt {

constexpr int kAovFloats = 10;
constexpr int kAovAlbedo = 0, kAovCoverage = 3, kAovNormal = 4, kAovDepth = 7, kAovLumM1 = 8, kAovLumM2 = 9;
constexpr int kDenoiseBlock = 256;

template <typename... P, typename... A>
inline void aov_launch(void (*kernel)(P...), unsigned grid, unsigned block, cudaStream_t stream, A... args)
{
    if (grid == 0) {
        return;
    }
#ifdef __CUDACC__
    kernel<<<grid, block, 0, stream>>>(args...);
#else
    (void)stream;
    simt::launch(grid, block, [&] { kernel(args...); });
#endif
}

// k_resolve's running mean: (x + n * acc) / (n + 1) for the frame with frame_id n
CRT_D float aov_running_mean(float x, float acc, uint32_t n)
{
    return (x + (float)n * acc) / (float)(n + 1u);
}

// One thread per local pixel; the batch's frames * spp samples in sample order, with k_resolve's slot indexing.
// Hit: base colour as k_shade unpacks it (same template branch), the TriShade normal face-forwarded as k_shade does
// (render_embree.ispc:296-300), the hit distance. Miss: albedo = the miss shader's colour (a demodulated background
// is 1), normal 0, coverage 0, no depth.
template <bool HWTEX>
__global__ void __launch_bounds__(128, 4) k_aov_primary(DeviceScene sc, FrameLayout f, PathState ps, uint32_t frame_id,
                                                      float *aov_local, float *aov_full)
{
    const uint32_t lp = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t x, y;
    if (lp >= f.npx_local || !local_pixel_coords(f, lp, x, y)) {
        return;
    }
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        acc[j] = aov_local[(size_t)kAovFloats * lp + j];
    }
    const TexSource tex_source{sc.texels, sc.tex, sc.tex_objects};
    for (uint32_t k = 0; k < f.frames; ++k) {
        float3 albedo = mk3(0.f), normal_sum = mk3(0.f);
        float coverage = 0.f, depth = 0.f;
        uint32_t hits = 0;
        for (uint32_t s = 0; s < f.spp; ++s) {
            const size_t i = (size_t)(k * f.spp + s) * f.npx_local + lp;
            const float4 rd = ps.ray_d[i], h = ps.hit[i];
            const float3 dir = mk3(rd.x, rd.y, rd.z);
            const uint32_t tri = __float_as_uint(h.w);
            if (tri == kMiss) {
                albedo = albedo + miss_shader(dir);
                continue;
            }
            const float4 s0 = __ldg(sc.shade + 3 * (size_t)tri), s1 = __ldg(sc.shade + 3 * (size_t)tri + 1),
                         s2 = __ldg(sc.shade + 3 * (size_t)tri + 2);
            float3 normal = mk3(s0.x, s0.y, s0.z);
            float2 uv = make_float2(0.f, 0.f);
            if (__float_as_uint(s2.z) != 0u) {
                const float bw = 1.f - h.y - h.z;
                uv.x = s1.x * bw + s1.z * h.y + s2.x * h.z;
                uv.y = s1.y * bw + s1.w * h.y + s2.y * h.z;
            }
            DisneyMaterial mat{};
            unpack_material<HWTEX>(mat, sc.materials, __float_as_uint(s0.w), uv, tex_source);
            if (mat.specular_transmission == 0.f && dot(neg(dir), normal) < 0.f) {
                normal = neg(normal);
            }
            albedo = albedo + mat.base_color;
            normal_sum = normal_sum + normal;
            coverage += 1.f;
            depth += h.x;
            ++hits;
        }
        albedo = albedo / (float)f.spp;
        normal_sum = normal_sum / (float)f.spp;
        const float frame[8] = {albedo.x, albedo.y, albedo.z, coverage / (float)f.spp,
                                normal_sum.x, normal_sum.y, normal_sum.z, hits ? depth / (float)hits : 0.f};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            acc[j] = aov_running_mean(frame[j], acc[j], frame_id + k);
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        aov_local[(size_t)kAovFloats * lp + j] = acc[j];
    }
    if (aov_full) {
        const size_t p = (size_t)y * f.fb_w + x;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            aov_full[(size_t)kAovFloats * p + j] = acc[j];
        }
    }
}

// Mean of L and L^2 over each frame's spp samples (L: luminance of the sample's radiance), folded like k_resolve.
__global__ void __launch_bounds__(256) k_aov_moments(FrameLayout f, PathState ps, uint32_t frame_id, float *aov_local,
                                                     float *aov_full)
{
    const uint32_t lp = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t x, y;
    if (lp >= f.npx_local || !local_pixel_coords(f, lp, x, y)) {
        return;
    }
    float m1 = aov_local[(size_t)kAovFloats * lp + kAovLumM1], m2 = aov_local[(size_t)kAovFloats * lp + kAovLumM2];
    for (uint32_t k = 0; k < f.frames; ++k) {
        float s1 = 0.f, s2 = 0.f;
        for (uint32_t s = 0; s < f.spp; ++s) {
            const float4 r = ps.radiance[(size_t)(k * f.spp + s) * f.npx_local + lp];
            const float l = luminance(mk3(r.x, r.y, r.z));
            s1 += l;
            s2 += l * l;
        }
        m1 = aov_running_mean(s1 / (float)f.spp, m1, frame_id + k);
        m2 = aov_running_mean(s2 / (float)f.spp, m2, frame_id + k);
    }
    aov_local[(size_t)kAovFloats * lp + kAovLumM1] = m1;
    aov_local[(size_t)kAovFloats * lp + kAovLumM2] = m2;
    if (aov_full) {
        const size_t p = (size_t)y * f.fb_w + x;
        aov_full[(size_t)kAovFloats * p + kAovLumM1] = m1;
        aov_full[(size_t)kAovFloats * p + kAovLumM2] = m2;
    }
}

// ---- denoiser (full frame, row-major, one thread per pixel) ----
CRT_D float3 aov_albedo_floor(const float *a)
{
    return mk3(fmaxf(a[kAovAlbedo], 1e-3f), fmaxf(a[kAovAlbedo + 1], 1e-3f), fmaxf(a[kAovAlbedo + 2], 1e-3f));
}

// iv = {accum / max(albedo, 1e-3), max(0, m2 - m1^2) / samples}; guide = {unit normal (0 where the mean normal is 0),
// depth}; grad = the depth's central difference, one-sided at the borders (0 across a one-pixel-wide image)
__global__ void __launch_bounds__(kDenoiseBlock) k_dn_prepare(int w, int h, float samples, const float *accum,
                                                              const float *aov, float4 *iv, float4 *guide, float2 *grad)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (uint32_t)w * (uint32_t)h) {
        return;
    }
    const int x = (int)(p % (uint32_t)w), y = (int)(p / (uint32_t)w);
    const float *a = aov + (size_t)kAovFloats * p;
    const float3 alb = aov_albedo_floor(a);
    const float m1 = a[kAovLumM1], m2 = a[kAovLumM2];
    iv[p] = make_float4(accum[3 * (size_t)p] / alb.x, accum[3 * (size_t)p + 1] / alb.y, accum[3 * (size_t)p + 2] / alb.z,
                        fmaxf(0.f, m2 - m1 * m1) / samples);
    const float3 n = mk3(a[kAovNormal], a[kAovNormal + 1], a[kAovNormal + 2]);
    const float len = length(n);
    const float3 nh = len > 0.f ? mk3(n.x / len, n.y / len, n.z / len) : mk3(0.f);
    const float z = a[kAovDepth];
    guide[p] = make_float4(nh.x, nh.y, nh.z, z);
    const int xl = x > 0 ? x - 1 : x, xr = x < w - 1 ? x + 1 : x, yu = y > 0 ? y - 1 : y, yd = y < h - 1 ? y + 1 : y;
    const float zx = aov[(size_t)kAovFloats * ((size_t)y * w + xr) + kAovDepth] - aov[(size_t)kAovFloats * ((size_t)y * w + xl) + kAovDepth];
    const float zy = aov[(size_t)kAovFloats * ((size_t)yd * w + x) + kAovDepth] - aov[(size_t)kAovFloats * ((size_t)yu * w + x) + kAovDepth];
    grad[p] = make_float2(xr - xl == 2 ? 0.5f * zx : zx, yd - yu == 2 ? 0.5f * zy : zy);
}

// (1, 4, 6, 4, 1) / 16 at offset d in -2..2
CRT_D float b3_weight(int d)
{
    return d == 0 ? 0.375f : (d == 1 || d == -1 ? 0.25f : 0.0625f);
}

// One iteration with step `step` = 2^i: 5x5 B3-spline taps (dy outer, dx inner; taps outside the image skipped) weighted
// by luminance (scaled by the 3x3-blurred variance), normal and depth edge-stopping functions. I' = sum w I / sum w,
// v' = sum w^2 v / (sum w)^2. LAST: remodulate by max(albedo, 1e-3) and write float RGB + sRGB8 instead of iv_out.
template <bool LAST>
__global__ void __launch_bounds__(kDenoiseBlock) k_dn_atrous(int w, int h, int step, float sigma_l, float sigma_n,
                                                             float sigma_z, const float4 *iv_in, float4 *iv_out,
                                                             const float4 *guide, const float2 *grad, const float *aov,
                                                             float *rgb_out, uint32_t *img_out)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (uint32_t)w * (uint32_t)h) {
        return;
    }
    const int x = (int)(p % (uint32_t)w), y = (int)(p / (uint32_t)w);
    // the variance at p through a 3x3 (1,2,1) x (1,2,1) / 16 blur (normalised by the weights of the taps in the image)
    float gv = 0.f, gw = 0.f;
    for (int dy = -1; dy <= 1; ++dy) {
        for (int dx = -1; dx <= 1; ++dx) {
            const int qx = x + dx, qy = y + dy;
            if (qx < 0 || qx >= w || qy < 0 || qy >= h) {
                continue;
            }
            const float k = (float)((2 - (dx < 0 ? -dx : dx)) * (2 - (dy < 0 ? -dy : dy))) * 0.0625f;
            gv += k * iv_in[(size_t)qy * w + qx].w;
            gw += k;
        }
    }
    const float4 cp = iv_in[p], gp = guide[p];
    const float2 dz = grad[p];
    const float lp = luminance(mk3(cp.x, cp.y, cp.z));
    const float l_scale = sigma_l * sqrtf(gv / gw) + 1e-10f;
    const bool p_bg = gp.x == 0.f && gp.y == 0.f && gp.z == 0.f;
    float sw = 0.f, sv = 0.f;
    float3 si = mk3(0.f);
    for (int dy = -2; dy <= 2; ++dy) {
        for (int dx = -2; dx <= 2; ++dx) {
            const int qx = x + dx * step, qy = y + dy * step;
            if (qx < 0 || qx >= w || qy < 0 || qy >= h) {
                continue;
            }
            const size_t q = (size_t)qy * w + qx;
            const float4 cq = iv_in[q], gq = guide[q];
            const float w_l = expf(-fabsf(lp - luminance(mk3(cq.x, cq.y, cq.z))) / l_scale);
            const bool q_bg = gq.x == 0.f && gq.y == 0.f && gq.z == 0.f;
            float w_n;
            if (p_bg || q_bg) {
                w_n = p_bg && q_bg ? 1.f : 0.f;
            } else {
                w_n = powf(fmaxf(0.f, gp.x * gq.x + gp.y * gq.y + gp.z * gq.z), sigma_n);
            }
            const float w_z = expf(-fabsf(gp.w - gq.w) /
                                   (sigma_z * fabsf(dz.x * (float)(step * dx) + dz.y * (float)(step * dy)) + 1e-3f));
            const float wt = b3_weight(dx) * b3_weight(dy) * w_l * w_n * w_z;
            sw += wt;
            si = si + mk3(cq.x, cq.y, cq.z) * wt;
            sv += wt * wt * cq.w;
        }
    }
    const float3 ip = si / sw;
    if (!LAST) {
        iv_out[p] = make_float4(ip.x, ip.y, ip.z, sv / (sw * sw));
        return;
    }
    const float3 rgb = ip * aov_albedo_floor(aov + (size_t)kAovFloats * p);
    rgb_out[3 * (size_t)p] = rgb.x;
    rgb_out[3 * (size_t)p + 1] = rgb.y;
    rgb_out[3 * (size_t)p + 2] = rgb.z;
    img_out[p] = float_to_srgb8(rgb.x) | (float_to_srgb8(rgb.y) << 8) | (float_to_srgb8(rgb.z) << 16) | 0xff000000u;
}

struct DenoiseParams {
    int iterations = 5;
    float sigma_l = 4.f, sigma_n = 128.f, sigma_z = 1.f;
};

// The renderer's AOV and denoiser state. AOV buffers: 40 B per local pixel (tile-padded) + 40 B per framebuffer pixel;
// denoiser buffers, allocated by the first denoise call: 72 B per framebuffer pixel.
struct AovState {
    crt_host::DeviceBuffer<float> local, full;
    crt_host::DeviceBuffer<float4> dn_iv[2], dn_guide;
    crt_host::DeviceBuffer<float2> dn_grad;
    crt_host::DeviceBuffer<float> dn_rgb;
    crt_host::DeviceBuffer<uint32_t> dn_img;

    void release()
    {
        local.release();
        full.release();
        dn_iv[0].release();
        dn_iv[1].release();
        dn_guide.release();
        dn_grad.release();
        dn_rgb.release();
        dn_img.release();
    }
    // (crtc_initialize) zeroed buffers for a new framebuffer; the denoiser's are reallocated on first use
    void allocate(size_t npx_local, size_t npx_full, cudaStream_t stream)
    {
        release();
        local.alloc(npx_local * kAovFloats);
        full.alloc(npx_full * kAovFloats);
        if (npx_local) {
            CUDA_CHECK(cudaMemsetAsync(local.ptr, 0, npx_local * kAovFloats * sizeof(float), stream));
        }
        CUDA_CHECK(cudaMemsetAsync(full.ptr, 0, npx_full * kAovFloats * sizeof(float), stream));
    }
    void launch_primary(const DeviceScene &sc, const FrameLayout &f, const PathState &ps, uint32_t frame_id,
                        cudaStream_t stream)
    {
        const unsigned g = (f.npx_local + 127) / 128;
        if (sc.tex_objects) {
            aov_launch(k_aov_primary<true>, g, 128, stream, sc, f, ps, frame_id, local.ptr, full.ptr);
        } else {
            aov_launch(k_aov_primary<false>, g, 128, stream, sc, f, ps, frame_id, local.ptr, full.ptr);
        }
    }
    void launch_moments(const FrameLayout &f, const PathState &ps, uint32_t frame_id, cudaStream_t stream)
    {
        aov_launch(k_aov_moments, (f.npx_local + 255) / 256, 256, stream, f, ps, frame_id, local.ptr, full.ptr);
    }
    // Denoises the full frame `accum` (w x h x 3, `samples` = spp * frames accumulated) into dn_rgb / dn_img.
    void denoise(int w, int h, float samples, const float *accum, const DenoiseParams &prm, cudaStream_t stream)
    {
        const size_t n = (size_t)w * h;
        if (dn_img.count != n) {
            CUDA_CHECK(cudaStreamSynchronize(stream));
            dn_iv[0].alloc(n);
            dn_iv[1].alloc(n);
            dn_guide.alloc(n);
            dn_grad.alloc(n);
            dn_rgb.alloc(3 * n);
            dn_img.alloc(n);
        }
        const unsigned g = (unsigned)((n + kDenoiseBlock - 1) / kDenoiseBlock);
        aov_launch(k_dn_prepare, g, kDenoiseBlock, stream, w, h, samples, accum, (const float *)full.ptr, dn_iv[0].ptr,
                   dn_guide.ptr, dn_grad.ptr);
        for (int i = 0; i < prm.iterations; ++i) {
            const float4 *in = dn_iv[i & 1].ptr;
            float4 *out = dn_iv[(i + 1) & 1].ptr;
            if (i + 1 == prm.iterations) {
                aov_launch(k_dn_atrous<true>, g, kDenoiseBlock, stream, w, h, 1 << i, prm.sigma_l, prm.sigma_n, prm.sigma_z, in,
                           out, (const float4 *)dn_guide.ptr, (const float2 *)dn_grad.ptr, (const float *)full.ptr, dn_rgb.ptr,
                           dn_img.ptr);
            } else {
                aov_launch(k_dn_atrous<false>, g, kDenoiseBlock, stream, w, h, 1 << i, prm.sigma_l, prm.sigma_n, prm.sigma_z, in,
                           out, (const float4 *)dn_guide.ptr, (const float2 *)dn_grad.ptr, (const float *)full.ptr, dn_rgb.ptr,
                           dn_img.ptr);
            }
        }
        CUDA_CHECK(cudaGetLastError());
    }
};

}  // namespace crt
