// aov_denoise.cuh — first-hit AOV buffers (option "aov") and the edge-aware à-trous denoiser behind crtc_denoise.
//
//   k_aov_primary   after the primary-ray traversal, before k_shade(0): albedo, coverage, normal and depth of the primary
//                   hits, folded into a per-pixel running mean with k_resolve's formula
//   k_aov_hit       (option denoise_motion, dynamic scenes) in an epoch's first wavefront, after the primary traversal:
//                   each pixel's first hit triangle and barycentrics, for k_dn_temporal<true>
//   k_aov_moments   after k_resolve: the first two moments of the per-sample luminance, same running mean
//   k_dn_prepare    demodulated radiance, variance of the pixel mean, unit normals, depth and its screen gradient
//   k_dn_temporal   (option denoise_history) the temporal half of SVGF: reprojects the history into this epoch; with
//                   <true>, through the motion of each pixel's triangle since the history was written
//   k_dn_variance   (option denoise_history) the variance from the integrated moments
//   k_dn_atrous     one à-trous iteration of the spatial part of SVGF (Schied et al. 2017); the last one remodulates and
//                   writes float RGB and sRGB8
//
// Per-pixel AOV layout, kAovFloats floats: albedo.rgb, coverage, normal.xyz (mean of the face-forwarded unit normals, not
// renormalised), depth (mean hit distance over the samples that hit), lum_m1, lum_m2. Like accum there is a tile-local
// copy (the running mean's state) and a full row-major copy. The AOV kernels read only the path state and the scene and
// write only these buffers, so a frame renders exactly the same with and without them.
//
// Every kernel is launched through crt_host::launch (cuda_host_utils.h), so that the host build of the renderer
// (tests/simt_emu) compiles this header unchanged. Grids are one-dimensional for the same reason.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "bvh8_device.cuh"
#include "cuda_host_utils.h"
#include "kernels.cuh"

namespace crt {

constexpr int kAovFloats = 10;
constexpr int kAovAlbedo = 0, kAovCoverage = 3, kAovNormal = 4, kAovDepth = 7, kAovLumM1 = 8, kAovLumM2 = 9;
constexpr int kDenoiseBlock = 256;

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

// Option "denoise_motion", on a dynamic scene, in the first wavefront of an epoch only (frame 0 is its first frame):
// one thread per local pixel writes the pixel's hit record, 3 words at the full-frame position: bits(leaf-order
// triangle), u, v of the first sample of frame 0, in sample order, that hit geometry; bits(kMiss), 0, 0 if none did.
__global__ void __launch_bounds__(256) k_aov_hit(FrameLayout f, PathState ps, float *hit_full)
{
    const uint32_t lp = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t x, y;
    if (lp >= f.npx_local || !local_pixel_coords(f, lp, x, y)) {
        return;
    }
    float rec[3] = {__uint_as_float(kMiss), 0.f, 0.f};
    for (uint32_t s = 0; s < f.spp; ++s) {
        const float4 h = ps.hit[(size_t)s * f.npx_local + lp];
        if (__float_as_uint(h.w) != kMiss) {
            rec[0] = h.w;
            rec[1] = h.y;
            rec[2] = h.z;
            break;
        }
    }
    float *o = hit_full + 3 * ((size_t)y * f.fb_w + x);
    o[0] = rec[0];
    o[1] = rec[1];
    o[2] = rec[2];
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

// ---- the denoiser's temporal history (option "denoise_history"; include/crt_cuda.h, crtc_denoise) ----
// Per framebuffer pixel, kHistFloats floats: integrated demodulated colour I.rgb, integrated luminance moments M1 and M2,
// the number of samples n they represent, the first-hit depth z and unit normal of the frame they were written for.
constexpr int kHistFloats = 10;
constexpr int kHistColor = 0, kHistM1 = 3, kHistM2 = 4, kHistCount = 5, kHistDepth = 6, kHistNormal = 7;

// The camera a history was written for: its position and the inverse of the matrix [du | dv | tl] (row-major; inverted
// in double on the host, rounded to float)
struct HistoryView {
    float3 pos;
    float minv[9];
};

// Option "denoise_motion": the live geometry of a dynamic scene (scene_update.cuh, SceneGeometry), as the denoiser
// reads it. num_xforms / num_verts count floats.
struct LiveGeometry {
    const DevSegment *segs;
    uint32_t num_segs;
    const uint32_t *leaf_flat_ids, *index_arena;
    const float *uv_arena, *xforms, *verts;
    size_t num_xforms, num_verts;
};

// What k_dn_temporal<true> needs to move a pixel's point with its triangle: the live geometry (its segments, index and
// uv arenas and leaf order also serve the snapshot: a commit does not change them) and the snapshot taken with `prev`.
struct DenoiseMotion {
    const float *hit;  // k_aov_hit's records of this epoch
    LiveGeometry live;
    const float *prev_xforms, *prev_verts;
};

// The world point at barycentrics (b1, b2) of a triangle's world vertices w (9 floats)
CRT_D float3 dn_bary_point(const float *w, float b1, float b2)
{
    return mk3(w[0] + b1 * (w[3] - w[0]) + b2 * (w[6] - w[0]), w[1] + b1 * (w[4] - w[1]) + b2 * (w[7] - w[1]),
               w[2] + b1 * (w[5] - w[2]) + b2 * (w[8] - w[2]));
}

// One thread per pixel, after k_dn_prepare. Reprojects the pixel's first hit into the previous camera, blends the
// valid bilinear taps of `prev` (null: no history) with this epoch's accum and moments, writes the result to `cur` and
// the blended colour to iv.xyz. Pixels without history keep k_dn_prepare's iv bits.
// MOTION (the geometry changed since `prev` was written): a pixel with a hit record whose triangle moved has its point
// moved by the triangle's displacement at the record's barycentrics, and its taps' normals compared with the previous
// triangle's normal on nhat_p's side; every other pixel takes the static arithmetic. <false> ignores `mo`.
template <bool MOTION>
__global__ void __launch_bounds__(kDenoiseBlock) k_dn_temporal(int w, int h, float samples, float max_history, ViewParams view,
                                                               HistoryView pv, const float *prev, const float *aov,
                                                               const float4 *guide, float4 *iv, float *cur,
                                                               DenoiseMotion mo)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (uint32_t)w * (uint32_t)h) {
        return;
    }
    const int x = (int)(p % (uint32_t)w), y = (int)(p / (uint32_t)w);
    const float *a = aov + (size_t)kAovFloats * p;
    const float4 gp = guide[p];
    const float3 np = mk3(gp.x, gp.y, gp.z);
    float n_p = 0.f;
    float hist[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
    if (prev && a[kAovCoverage] > 0.f) {
        // the world point of the pixel-centre ray (k_raygen's expression, jitter 0.5) at the AOV depth
        const float px_x = ((float)x + 0.5f) / (float)(uint32_t)w;
        const float px_y = ((float)y + 0.5f) / (float)(uint32_t)h;
        const float3 d = normalize(mk3(view.dir_du.x * px_x + view.dir_dv.x * px_y + view.dir_top_left.x,
                                       view.dir_du.y * px_x + view.dir_dv.y * px_y + view.dir_top_left.y,
                                       view.dir_du.z * px_x + view.dir_dv.z * px_y + view.dir_top_left.z));
        float3 X = mk3(view.pos.x + gp.w * d.x, view.pos.y + gp.w * d.y, view.pos.z + gp.w * d.z);
        float3 n_ref = np;  // what the taps' normals are compared with
        bool moved_ok = true;
        if (MOTION) {
            const float *rec = mo.hit + 3 * (size_t)p;
            const uint32_t tri = __float_as_uint(rec[0]);
            if (tri != kMiss) {
                const LiveGeometry &g = mo.live;
                const uint32_t f = g.leaf_flat_ids[tri];
                const DevSegment seg = g.segs[dev_find_segment(g.segs, g.num_segs, f)];
                float wc[9], wp[9];
                float4 sc[3], sp[3];
                dev_flatten_triangle(seg, f, g.xforms, g.verts, g.index_arena, g.uv_arena, wc, sc);
                dev_flatten_triangle(seg, f, mo.prev_xforms, mo.prev_verts, g.index_arena, g.uv_arena, wp, sp);
                bool same = true;
#pragma unroll
                for (int k = 0; k < 9; ++k) {
                    same = same && __float_as_uint(wc[k]) == __float_as_uint(wp[k]);
                }
                if (!same) {
                    const float3 P = dn_bary_point(wc, rec[1], rec[2]), Pp = dn_bary_point(wp, rec[1], rec[2]);
                    const float3 dp = Pp - P;
                    const float inf = __uint_as_float(0x7f800000u);
                    moved_ok = fabsf(dp.x) < inf && fabsf(dp.y) < inf && fabsf(dp.z) < inf;
                    X = X + dp;
                    const float s = dot(np, mk3(sc[0].x, sc[0].y, sc[0].z)) < 0.f ? -1.f : 1.f;
                    n_ref = mk3(s * sp[0].x, s * sp[0].y, s * sp[0].z);
                }
            }
        }
        const float3 r = X - pv.pos;
        const float al = pv.minv[0] * r.x + pv.minv[1] * r.y + pv.minv[2] * r.z;
        const float be = pv.minv[3] * r.x + pv.minv[4] * r.y + pv.minv[5] * r.z;
        const float ga = pv.minv[6] * r.x + pv.minv[7] * r.y + pv.minv[8] * r.z;
        const float sx = (al / ga) * (float)w - 0.5f, sy = (be / ga) * (float)h - 0.5f;
        // (outside this window every tap is outside the image; it also keeps NaN and huge values away from the int cast;
        // a non-finite displacement leaves the pixel without history)
        if (moved_ok && ga > 0.f && sx > -1.f && sx < (float)w && sy > -1.f && sy < (float)h) {
            const float dist = length(r);
            const float fx0 = floorf(sx), fy0 = floorf(sy);
            const float fx = sx - fx0, fy = sy - fy0;
            const int x0 = (int)fx0, y0 = (int)fy0;
            float sw = 0.f, sn = 0.f;
            float acc[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const int qx = x0 + (t & 1), qy = y0 + (t >> 1);
                if (qx < 0 || qx >= w || qy < 0 || qy >= h) {
                    continue;
                }
                const float *hq = prev + (size_t)kHistFloats * ((size_t)qy * w + qx);
                const float3 nq = mk3(hq[kHistNormal], hq[kHistNormal + 1], hq[kHistNormal + 2]);
                if (all_zero(nq)) {
                    continue;
                }
                // prev's depth gradient at q, as k_dn_prepare computes it
                const int xl = qx > 0 ? qx - 1 : qx, xr = qx < w - 1 ? qx + 1 : qx, yu = qy > 0 ? qy - 1 : qy,
                          yd = qy < h - 1 ? qy + 1 : qy;
                const float zx = prev[(size_t)kHistFloats * ((size_t)qy * w + xr) + kHistDepth] -
                                 prev[(size_t)kHistFloats * ((size_t)qy * w + xl) + kHistDepth];
                const float zy = prev[(size_t)kHistFloats * ((size_t)yd * w + qx) + kHistDepth] -
                                 prev[(size_t)kHistFloats * ((size_t)yu * w + qx) + kHistDepth];
                const float gx = xr - xl == 2 ? 0.5f * zx : zx, gy = yd - yu == 2 ? 0.5f * zy : zy;
                if (!(fabsf(hq[kHistDepth] - dist) <= 0.02f * dist + 2.f * (fabsf(gx) + fabsf(gy))) || !(dot(n_ref, nq) >= 0.9f)) {
                    continue;
                }
                const float wt = ((t & 1) ? fx : 1.f - fx) * ((t >> 1) ? fy : 1.f - fy);
                sw += wt;
                sn += wt * hq[kHistCount];
#pragma unroll
                for (int j = 0; j < 5; ++j) {
                    acc[j] += wt * hq[j];
                }
            }
            if (sw >= 0.01f) {
#pragma unroll
                for (int j = 0; j < 5; ++j) {
                    hist[j] = acc[j] / sw;
                }
                n_p = fminf(max_history, sn / sw);
            }
        }
    }
    const float4 c = iv[p];
    float now[5] = {c.x, c.y, c.z, a[kAovLumM1], a[kAovLumM2]};
    float n_t = samples;
    if (n_p > 0.f) {
        n_t = n_p + samples;
#pragma unroll
        for (int j = 0; j < 5; ++j) {
            now[j] = (n_p * hist[j] + samples * now[j]) / n_t;
        }
        iv[p] = make_float4(now[0], now[1], now[2], c.w);
    }
    float *o = cur + (size_t)kHistFloats * p;
#pragma unroll
    for (int j = 0; j < 5; ++j) {
        o[j] = now[j];
    }
    o[kHistCount] = n_t;
    o[kHistDepth] = gp.w;
    o[kHistNormal] = gp.x;
    o[kHistNormal + 1] = gp.y;
    o[kHistNormal + 2] = gp.z;
}

// One thread per pixel, after k_dn_temporal: iv.w = max(0, M2 - M1^2) / n from the integrated moments where n >= 4;
// where n < 4, from moments averaged over the 7x7 neighbourhood with the a-trous's normal and depth weights at step 1
// (taps outside the image skipped; no luminance or kernel weight).
__global__ void __launch_bounds__(kDenoiseBlock) k_dn_variance(int w, int h, float sigma_n, float sigma_z, const float *cur,
                                                               const float4 *guide, const float2 *grad, float4 *iv)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (uint32_t)w * (uint32_t)h) {
        return;
    }
    const int x = (int)(p % (uint32_t)w), y = (int)(p / (uint32_t)w);
    const float *hp = cur + (size_t)kHistFloats * p;
    const float n_t = hp[kHistCount];
    float m1 = hp[kHistM1], m2 = hp[kHistM2];
    if (n_t < 4.f) {
        const float4 gp = guide[p];
        const float2 dz = grad[p];
        const bool p_bg = gp.x == 0.f && gp.y == 0.f && gp.z == 0.f;
        float sw = 0.f, s1 = 0.f, s2 = 0.f;
        for (int dy = -3; dy <= 3; ++dy) {
            for (int dx = -3; dx <= 3; ++dx) {
                const int qx = x + dx, qy = y + dy;
                if (qx < 0 || qx >= w || qy < 0 || qy >= h) {
                    continue;
                }
                const size_t q = (size_t)qy * w + qx;
                const float4 gq = guide[q];
                const bool q_bg = gq.x == 0.f && gq.y == 0.f && gq.z == 0.f;
                float w_n;
                if (p_bg || q_bg) {
                    w_n = p_bg && q_bg ? 1.f : 0.f;
                } else {
                    w_n = powf(fmaxf(0.f, gp.x * gq.x + gp.y * gq.y + gp.z * gq.z), sigma_n);
                }
                const float w_z = expf(-fabsf(gp.w - gq.w) / (sigma_z * fabsf(dz.x * (float)dx + dz.y * (float)dy) + 1e-3f));
                const float wt = w_n * w_z;
                sw += wt;
                s1 += wt * cur[(size_t)kHistFloats * q + kHistM1];
                s2 += wt * cur[(size_t)kHistFloats * q + kHistM2];
            }
        }
        m1 = s1 / sw;
        m2 = s2 / sw;
    }
    const float4 c = iv[p];
    iv[p] = make_float4(c.x, c.y, c.z, fmaxf(0.f, m2 - m1 * m1) / n_t);
}

struct DenoiseParams {
    int iterations = 5;
    float sigma_l = 4.f, sigma_n = 128.f, sigma_z = 1.f;
};

// What a history buffer was written for: the reset epoch, the camera of that epoch's first frame and the renderer's
// geometry version (bumped by crtc_set_scene and by every commit that moves geometry)
struct HistoryTag {
    bool valid = false;
    uint64_t epoch = 0;
    ViewParams view{};
    uint64_t geometry = 0;
};

// A copy of the moving part of the geometry (instance matrices, unique vertices), taken when its history buffer was
// written under geometry version `version`
struct GeometrySnapshot {
    crt_host::DeviceBuffer<float> xforms, verts;
    bool valid = false;
    uint64_t version = 0;
    void release()
    {
        xforms.release();
        verts.release();
        valid = false;
    }
};

// The renderer's AOV and denoiser state. AOV buffers: 40 B per local pixel (tile-padded) + 40 B per framebuffer pixel;
// denoiser buffers, allocated by the first denoise call: 72 B per framebuffer pixel, + 80 B with option denoise_history
// (the two history buffers, `prev` and `cur`). Option denoise_motion, dynamic scenes only: 12 B per framebuffer pixel
// (hit records) + per history buffer a geometry snapshot of 128 B per instance and 12 B per unique vertex.
struct AovState {
    crt_host::DeviceBuffer<float> local, full;
    crt_host::DeviceBuffer<float4> dn_iv[2], dn_guide;
    crt_host::DeviceBuffer<float2> dn_grad;
    crt_host::DeviceBuffer<float> dn_rgb;
    crt_host::DeviceBuffer<uint32_t> dn_img;
    crt_host::DeviceBuffer<float> hist[2];  // hist[hist_cur] is `cur`, the other one `prev`
    HistoryTag hist_tag[2];
    int hist_cur = 0;
    crt_host::DeviceBuffer<float> hit;  // k_aov_hit's records, 3 words per framebuffer pixel
    GeometrySnapshot snap[2];           // snap[i] goes with hist[i]

    void drop_history()
    {
        hist_tag[0] = HistoryTag{};
        hist_tag[1] = HistoryTag{};
    }
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
        hist[0].release();
        hist[1].release();
        hit.release();
        snap[0].release();
        snap[1].release();
        drop_history();
    }
    // `cur` if the last denoise call was made in `epoch`, else null
    const float *history_of(uint64_t epoch) const
    {
        const HistoryTag &t = hist_tag[hist_cur];
        return t.valid && t.epoch == epoch ? hist[hist_cur].ptr : nullptr;
    }
    // The previous camera for k_dn_temporal: false if [du | dv | tl] is singular or not finite (no reprojection then)
    static bool history_view(const ViewParams &v, HistoryView &out)
    {
        const double m[3][3] = {{v.dir_du.x, v.dir_dv.x, v.dir_top_left.x},
                                {v.dir_du.y, v.dir_dv.y, v.dir_top_left.y},
                                {v.dir_du.z, v.dir_dv.z, v.dir_top_left.z}};
        const double det = m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) +
                           m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
        if (!std::isfinite(det) || det == 0.0) {
            return false;
        }
        // the adjugate over the determinant, row-major
        const double inv[9] = {(m[1][1] * m[2][2] - m[1][2] * m[2][1]) / det, (m[0][2] * m[2][1] - m[0][1] * m[2][2]) / det,
                               (m[0][1] * m[1][2] - m[0][2] * m[1][1]) / det, (m[1][2] * m[2][0] - m[1][0] * m[2][2]) / det,
                               (m[0][0] * m[2][2] - m[0][2] * m[2][0]) / det, (m[0][2] * m[1][0] - m[0][0] * m[1][2]) / det,
                               (m[1][0] * m[2][1] - m[1][1] * m[2][0]) / det, (m[0][1] * m[2][0] - m[0][0] * m[2][1]) / det,
                               (m[0][0] * m[1][1] - m[0][1] * m[1][0]) / det};
        for (int i = 0; i < 9; ++i) {
            if (!std::isfinite(inv[i])) {
                return false;
            }
            out.minv[i] = (float)inv[i];
        }
        out.pos = v.pos;
        return true;
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
            crt_host::launch(k_aov_primary<true>, g, 128, stream, sc, f, ps, frame_id, local.ptr, full.ptr);
        } else {
            crt_host::launch(k_aov_primary<false>, g, 128, stream, sc, f, ps, frame_id, local.ptr, full.ptr);
        }
    }
    // Option denoise_motion: the hit records of an epoch's first wavefront (allocated on first use)
    void launch_hit(const FrameLayout &f, const PathState &ps, cudaStream_t stream)
    {
        hit.alloc((size_t)3 * f.fb_w * f.fb_h);
        crt_host::launch(k_aov_hit, (f.npx_local + 255) / 256, 256, stream, f, ps, hit.ptr);
    }
    void launch_moments(const FrameLayout &f, const PathState &ps, uint32_t frame_id, cudaStream_t stream)
    {
        crt_host::launch(k_aov_moments, (f.npx_local + 255) / 256, 256, stream, f, ps, frame_id, local.ptr, full.ptr);
    }
    // Denoises the full frame `accum` (w x h x 3, `samples` = spp * frames accumulated) into dn_rgb / dn_img.
    // max_history > 0 (option denoise_history): the temporal pass runs between k_dn_prepare and the a-trous chain, with
    // the history of the latest earlier epoch that had a denoise call as `prev`; `epoch` and `view` are the current
    // reset epoch and the camera of its first frame. `geometry` is the renderer's geometry version; `live` (option
    // denoise_motion on a dynamic scene, else null) lets a history written under another version reproject through the
    // motion of each pixel's triangle, and has `cur` keep a snapshot of the geometry it was written under.
    void denoise(int w, int h, float samples, const float *accum, const DenoiseParams &prm, uint32_t max_history,
                 uint64_t epoch, const ViewParams &view, uint64_t geometry, const LiveGeometry *live, cudaStream_t stream)
    {
        const size_t n = (size_t)w * h;
        if (dn_img.count != n || (max_history && hist[0].count != kHistFloats * n)) {
            CUDA_CHECK(cudaStreamSynchronize(stream));
            dn_iv[0].alloc(n);
            dn_iv[1].alloc(n);
            dn_guide.alloc(n);
            dn_grad.alloc(n);
            dn_rgb.alloc(3 * n);
            dn_img.alloc(n);
            if (max_history) {
                hist[0].alloc(kHistFloats * n);
                hist[1].alloc(kHistFloats * n);
                drop_history();
            }
        }
        const unsigned g = (unsigned)((n + kDenoiseBlock - 1) / kDenoiseBlock);
        crt_host::launch(k_dn_prepare, g, kDenoiseBlock, stream, w, h, samples, accum, (const float *)full.ptr, dn_iv[0].ptr,
                   dn_guide.ptr, dn_grad.ptr);
        if (max_history) {
            if (hist_tag[hist_cur].valid && hist_tag[hist_cur].epoch < epoch) {
                hist_cur ^= 1;  // cur -> prev; the older prev is overwritten
            }
            const HistoryTag &pt = hist_tag[hist_cur ^ 1];
            const GeometrySnapshot &ps = snap[hist_cur ^ 1];
            HistoryView pv{};
            bool have_prev = pt.valid && pt.epoch < epoch && history_view(pt.view, pv);
            const bool moved = have_prev && pt.geometry != geometry;
            DenoiseMotion mo{};
            if (moved) {
                // (a history of other geometry reprojects only through its snapshot; without one it is not carried)
                have_prev = live && ps.valid && ps.version == pt.geometry && hit.count == (size_t)3 * n;
                if (have_prev) {
                    mo = DenoiseMotion{hit.ptr, *live, ps.xforms.ptr, ps.verts.ptr};
                }
            }
            const float *prev = have_prev ? (const float *)hist[hist_cur ^ 1].ptr : nullptr;
            if (moved && have_prev) {
                crt_host::launch(k_dn_temporal<true>, g, kDenoiseBlock, stream, w, h, samples, (float)max_history, view, pv,
                                 prev, (const float *)full.ptr, (const float4 *)dn_guide.ptr, dn_iv[0].ptr,
                                 hist[hist_cur].ptr, mo);
            } else {
                crt_host::launch(k_dn_temporal<false>, g, kDenoiseBlock, stream, w, h, samples, (float)max_history, view, pv,
                                 prev, (const float *)full.ptr, (const float4 *)dn_guide.ptr, dn_iv[0].ptr,
                                 hist[hist_cur].ptr, mo);
            }
            crt_host::launch(k_dn_variance, g, kDenoiseBlock, stream, w, h, prm.sigma_n, prm.sigma_z, (const float *)hist[hist_cur].ptr,
                       (const float4 *)dn_guide.ptr, (const float2 *)dn_grad.ptr, dn_iv[0].ptr);
            hist_tag[hist_cur].valid = true;
            hist_tag[hist_cur].epoch = epoch;
            hist_tag[hist_cur].view = view;
            hist_tag[hist_cur].geometry = geometry;
            GeometrySnapshot &cs = snap[hist_cur];
            if (live && !(cs.valid && cs.version == geometry)) {
                // (stream-ordered after k_dn_temporal, which read the other snapshot)
                cs.xforms.alloc(live->num_xforms);
                cs.verts.alloc(live->num_verts);
                CUDA_CHECK(cudaMemcpyAsync(cs.xforms.ptr, live->xforms, live->num_xforms * sizeof(float),
                                           cudaMemcpyDeviceToDevice, stream));
                CUDA_CHECK(cudaMemcpyAsync(cs.verts.ptr, live->verts, live->num_verts * sizeof(float),
                                           cudaMemcpyDeviceToDevice, stream));
                cs.valid = true;
                cs.version = geometry;
            }
        }
        for (int i = 0; i < prm.iterations; ++i) {
            const float4 *in = dn_iv[i & 1].ptr;
            float4 *out = dn_iv[(i + 1) & 1].ptr;
            if (i + 1 == prm.iterations) {
                crt_host::launch(k_dn_atrous<true>, g, kDenoiseBlock, stream, w, h, 1 << i, prm.sigma_l, prm.sigma_n, prm.sigma_z, in,
                           out, (const float4 *)dn_guide.ptr, (const float2 *)dn_grad.ptr, (const float *)full.ptr, dn_rgb.ptr,
                           dn_img.ptr);
            } else {
                crt_host::launch(k_dn_atrous<false>, g, kDenoiseBlock, stream, w, h, 1 << i, prm.sigma_l, prm.sigma_n, prm.sigma_z, in,
                           out, (const float4 *)dn_guide.ptr, (const float2 *)dn_grad.ptr, (const float *)full.ptr, dn_rgb.ptr,
                           dn_img.ptr);
            }
        }
        CUDA_CHECK(cudaGetLastError());
    }
};

}  // namespace crt
