// shade_devcheck.cu — TEST-ONLY shared library (libcrt_shade_devcheck.so).
//
// The product's shading arithmetic (shade_math.cuh) as nvcc compiles it for sm_90a, with the product's own flags
// (Makefile: NVFLAGS), one CUDA thread per input. It exports the batched shadekat_*_n entry points of
// libcrt_shade_hostcheck.so (the same source built by g++) under the same names and signatures, so that
// tests/test_shade_device.py runs one check against either build. It is not linked into libcrt_cuda_core.so.
#include <cstdint>
#include <vector>

#include <cuda_runtime.h>

#include "shade_math.cuh"

#include "shade_kat.h"

namespace {

constexpr int kBlock = 128;

unsigned grid_for(int n) { return (unsigned)((n + kBlock - 1) / kBlock); }

// Device copies of the host arrays of one call: inputs are uploaded, outputs downloaded by finish().
class Call {
public:
    ~Call()
    {
        for (void *p : bufs_) {
            cudaFree(p);
        }
    }
    template <typename T>
    T *in(const T *host, size_t count)
    {
        T *d = alloc<T>(count);
        if (d != nullptr && count > 0) {
            check(cudaMemcpy(d, host, count * sizeof(T), cudaMemcpyHostToDevice));
        }
        return d;
    }
    template <typename T>
    T *out(T *host, size_t count)
    {
        T *d = alloc<T>(count);
        outs_.push_back({host, d, count * sizeof(T)});
        return d;
    }
    template <typename T>
    T *inout(T *host, size_t count)
    {
        T *d = in(static_cast<const T *>(host), count);
        outs_.push_back({host, d, count * sizeof(T)});
        return d;
    }
    bool ok() const { return err_ == cudaSuccess; }
    int finish()
    {
        check(cudaGetLastError());
        check(cudaDeviceSynchronize());
        for (const Out &o : outs_) {
            if (ok() && o.bytes > 0) {
                check(cudaMemcpy(o.host, o.dev, o.bytes, cudaMemcpyDeviceToHost));
            }
        }
        return (int)err_;
    }

private:
    struct Out {
        void *host;
        void *dev;
        size_t bytes;
    };
    template <typename T>
    T *alloc(size_t count)
    {
        void *p = nullptr;
        if (ok()) {
            check(cudaMalloc(&p, count * sizeof(T) + 16));
        }
        if (p != nullptr) {
            bufs_.push_back(p);
        }
        return static_cast<T *>(p);
    }
    void check(cudaError_t e)
    {
        if (err_ == cudaSuccess && e != cudaSuccess) {
            err_ = e;
        }
    }
    std::vector<void *> bufs_;
    std::vector<Out> outs_;
    cudaError_t err_ = cudaSuccess;
};

#define KAT_THREAD                                         \
    const int i = blockIdx.x * blockDim.x + threadIdx.x; \
    if (i >= n) {                                          \
        return;                                            \
    }

__global__ void k_rng(const uint32_t *pix, const uint32_t *frame, int n, int k, uint32_t *states, float *floats)
{
    KAT_THREAD
    crt::kat_rng(pix[i], frame[i], (uint32_t)k, states + (size_t)k * i, floats + (size_t)k * i);
}
__global__ void k_lcg(uint32_t *states, int n, float *floats)
{
    KAT_THREAD
    floats[i] = crt::lcg_randomf(states[i]);
}
__global__ void k_eval(const float *mat, const float *nrm, const float *wo, const float *wi, int n, float *out)
{
    KAT_THREAD
    crt::kat_disney_eval(mat + 16 * i, nrm + 3 * i, wo + 3 * i, wi + 3 * i, out + 4 * i);
}
__global__ void k_sample(const float *mat, const float *nrm, const float *wo, uint32_t *rng, int n, float *out)
{
    KAT_THREAD
    crt::kat_disney_sample(mat + 16 * i, nrm + 3 * i, wo + 3 * i, rng + i, out + 7 * i);
}
__global__ void k_light(const float *light, const float *s2, const float *orig, const float *dir, int n, float *out)
{
    KAT_THREAD
    crt::kat_light(light, s2 + 2 * i, orig + 3 * i, dir + 3 * i, out + 9 * i);
}
__global__ void k_texture(const uint32_t *texels, crt::DevTex t, const float *uv, int n, float *out)
{
    KAT_THREAD
    crt::kat_texture(texels, t, uv[2 * i], uv[2 * i + 1], out + 4 * i);
}
__global__ void k_unpack(const float *materials, uint32_t id, const uint32_t *texels, const crt::DevTex *tex,
                         const float *uv, int n, float *out)
{
    KAT_THREAD
    const crt::TexSource ts{texels, tex, nullptr};
    crt::kat_unpack_material(materials, id, ts, uv[2 * i], uv[2 * i + 1], out + 14 * i);
}
__global__ void k_miss(const float *dirs, int n, float *out)
{
    KAT_THREAD
    crt::kat_miss(dirs + 3 * i, out + 3 * i);
}
__global__ void k_ortho(const float *nrm, int n, float *out)
{
    KAT_THREAD
    crt::kat_ortho_basis(nrm + 3 * i, out + 6 * i);
}
__global__ void k_srgb8(const float *x, int n, uint8_t *out)
{
    KAT_THREAD
    out[i] = (uint8_t)crt::float_to_srgb8(x[i]);
}
__global__ void k_schlick(const float *x, int n, float *out)
{
    KAT_THREAD
    out[i] = crt::schlick_weight(x[i]);
}
__global__ void k_math(int fn, const float *x, const float *y, int n, float *out)
{
    KAT_THREAD
    out[i] = crt::kat_math(fn, x[i], y != nullptr ? y[i] : 0.f);
}

}  // namespace

extern "C" {

int shadekat_rng_n(const uint32_t *pixel_ids, const uint32_t *frame_ids, int n, int k, uint32_t *states, float *floats)
{
    Call c;
    const uint32_t *p = c.in(pixel_ids, n), *f = c.in(frame_ids, n);
    uint32_t *s = c.out(states, (size_t)n * k);
    float *x = c.out(floats, (size_t)n * k);
    if (c.ok() && n > 0) {
        k_rng<<<grid_for(n), kBlock>>>(p, f, n, k, s, x);
    }
    return c.finish();
}
int shadekat_lcg_n(uint32_t *states, int n, float *floats)
{
    Call c;
    uint32_t *s = c.inout(states, n);
    float *x = c.out(floats, n);
    if (c.ok() && n > 0) {
        k_lcg<<<grid_for(n), kBlock>>>(s, n, x);
    }
    return c.finish();
}
int shadekat_disney_eval_n(const float *mat16n, const float *n3n, const float *w_o3n, const float *w_i3n, int n, float *out4n)
{
    Call c;
    const float *m = c.in(mat16n, 16 * (size_t)n), *nr = c.in(n3n, 3 * (size_t)n), *wo = c.in(w_o3n, 3 * (size_t)n),
                *wi = c.in(w_i3n, 3 * (size_t)n);
    float *o = c.out(out4n, 4 * (size_t)n);
    if (c.ok() && n > 0) {
        k_eval<<<grid_for(n), kBlock>>>(m, nr, wo, wi, n, o);
    }
    return c.finish();
}
int shadekat_disney_sample_n(const float *mat16n, const float *n3n, const float *w_o3n, uint32_t *rng_n, int n,
                             float *out7n)
{
    Call c;
    const float *m = c.in(mat16n, 16 * (size_t)n), *nr = c.in(n3n, 3 * (size_t)n), *wo = c.in(w_o3n, 3 * (size_t)n);
    uint32_t *r = c.inout(rng_n, n);
    float *o = c.out(out7n, 7 * (size_t)n);
    if (c.ok() && n > 0) {
        k_sample<<<grid_for(n), kBlock>>>(m, nr, wo, r, n, o);
    }
    return c.finish();
}
int shadekat_light_n(const float *light20, const float *s2n, const float *orig3n, const float *dir3n, int n, float *out9n)
{
    Call c;
    const float *l = c.in(light20, 20), *s = c.in(s2n, 2 * (size_t)n), *o = c.in(orig3n, 3 * (size_t)n),
                *d = c.in(dir3n, 3 * (size_t)n);
    float *out = c.out(out9n, 9 * (size_t)n);
    if (c.ok() && n > 0) {
        k_light<<<grid_for(n), kBlock>>>(l, s, o, d, n, out);
    }
    return c.finish();
}
int shadekat_texture_n(const uint8_t *data, int w, int h, int channels, const float *uv, int n, float *out4n)
{
    const std::vector<uint32_t> arena = crt::rgba8_arena(data, w, h, channels);
    Call c;
    const uint32_t *t = c.in(arena.data(), arena.size());
    const float *u = c.in(uv, 2 * (size_t)n);
    float *o = c.out(out4n, 4 * (size_t)n);
    if (c.ok() && n > 0) {
        k_texture<<<grid_for(n), kBlock>>>(t, crt::DevTex{0u, w, h, 0}, u, n, o);
    }
    return c.finish();
}
int shadekat_unpack_material_n(const float *materials, int n_materials, uint32_t id, const uint32_t *texels, int n_texels,
                               const int32_t *tex, int n_tex, const float *uv, int n, float *out14n)
{
    Call c;
    const float *m = c.in(materials, 16 * (size_t)n_materials);
    const uint32_t *t = c.in(texels, n_texels);
    const crt::DevTex *d = c.in(reinterpret_cast<const crt::DevTex *>(tex), n_tex);
    const float *u = c.in(uv, 2 * (size_t)n);
    float *o = c.out(out14n, 14 * (size_t)n);
    if (c.ok() && n > 0) {
        k_unpack<<<grid_for(n), kBlock>>>(m, id, t, d, u, n, o);
    }
    return c.finish();
}
int shadekat_miss_n(const float *dirs, int n, float *out3n)
{
    Call c;
    const float *d = c.in(dirs, 3 * (size_t)n);
    float *o = c.out(out3n, 3 * (size_t)n);
    if (c.ok() && n > 0) {
        k_miss<<<grid_for(n), kBlock>>>(d, n, o);
    }
    return c.finish();
}
int shadekat_ortho_basis_n(const float *n3n, int n, float *out6n)
{
    Call c;
    const float *nr = c.in(n3n, 3 * (size_t)n);
    float *o = c.out(out6n, 6 * (size_t)n);
    if (c.ok() && n > 0) {
        k_ortho<<<grid_for(n), kBlock>>>(nr, n, o);
    }
    return c.finish();
}
int shadekat_srgb8_n(const float *x, int n, uint8_t *out)
{
    Call c;
    const float *d = c.in(x, n);
    uint8_t *o = c.out(out, n);
    if (c.ok() && n > 0) {
        k_srgb8<<<grid_for(n), kBlock>>>(d, n, o);
    }
    return c.finish();
}
int shadekat_schlick_n(const float *cos_theta, int n, float *out)
{
    Call c;
    const float *d = c.in(cos_theta, n);
    float *o = c.out(out, n);
    if (c.ok() && n > 0) {
        k_schlick<<<grid_for(n), kBlock>>>(d, n, o);
    }
    return c.finish();
}
int shadekat_math_n(int fn, const float *x, const float *y, int n, float *out)
{
    Call c;
    const float *dx = c.in(x, n), *dy = y != nullptr ? c.in(y, n) : nullptr;
    float *o = c.out(out, n);
    if (c.ok() && n > 0) {
        k_math<<<grid_for(n), kBlock>>>(fn, dx, dy, n, o);
    }
    return c.finish();
}
}
