// render_cuda.h — RenderCUDA, the `crt_cuda` backend of ChameleonRT.
//
// Drop this directory into ChameleonRT as backends/cuda/ (see INTEGRATION.md): it is built as
// the MODULE library libcrt_cuda.so that `./chameleonrt cuda <scene>` dlopen()s
// (util/render_plugin.cpp:14-37). The class has the shape of the reference's other backends
// (cf. backends/embree/render_embree.h:12-44, backends/optix/render_optix.h); all rendering is
// delegated to the C ABI of include/crt_cuda.h (libcrt_cuda_core.so: host BVH8 build + the
// sm_90a wavefront kernels).
#pragma once

#include <cstdint>
#include <string>
#include <vector>
#include "render_backend.h"

#ifndef CRT_CUDA_HEADLESS
// interactive build: the display is the reference's GLDisplay, and a renderer that fills
// GLNativeRenderer::gl_display_texture is shown without a trip through host memory (util/display/gldisplay.h:35-37,
// gldisplay.cpp:107-110)
#include "display/gldisplay.h"
using RenderCUDABase = GLNativeRenderer;
struct cudaGraphicsResource;
#else
using RenderCUDABase = RenderBackend;
#endif

struct crtc_renderer;

struct RenderCUDA : RenderCUDABase {
    // One renderer per GPU (CRT_CUDA_DEVICES, default: the single device CRT_CUDA_DEVICE). Renderer i owns the image
    // tiles with tile_id % N == i (the reference's tile ids, render_embree.cpp:178-180) and resolves them straight
    // into the frame of renderers[0] over NVLink (crtc_share_frame), which is the one `img` is read from.
    std::vector<crtc_renderer *> renderers;
    crtc_renderer *renderer = nullptr;  // = renderers[0]
    glm::ivec2 fb_dims = glm::ivec2(0);
    bool native_display = false;
    int frames_since_scene = 0;  // multi-renderer mode: the first frames after set_scene are rendered blocking
    // CRT_CUDA_DENOISE=1: option "aov" on, and every frame that is read back or presented is the crtc_denoise output
    // (one renderer only)
    bool denoise = false;

    // native_display: the Display this plugin made is a GLDisplay (render_cuda_plugin.cpp), so frames go to its texture
    // through CUDA-GL interop and `img` is only read back when the application asks (readback_framebuffer: screenshots,
    // main.cpp:309-314), as backends/optix/render_optix.cpp:404-430 does. Always false in headless builds.
    explicit RenderCUDA(bool native_display = false);
    ~RenderCUDA() override;
#ifndef CRT_CUDA_HEADLESS
    cudaGraphicsResource *cu_display_texture = nullptr;  // gl_display_texture registered with CUDA
    void create_display_texture();
    void release_display_texture();
    void present_native();
#endif

    std::string name() override;
    void initialize(const int fb_width, const int fb_height) override;
    void set_scene(const Scene &scene) override;
    RenderStats render(const glm::vec3 &pos,
                       const glm::vec3 &dir,
                       const glm::vec3 &up,
                       const float fovy,
                       const bool camera_changed,
                       const bool readback_framebuffer) override;

    // Extra export for parity harnesses (SURVEY.md §8b): the accumulated float framebuffer,
    // row-major RGB, fb_width * fb_height * 3 floats.
    void read_accum(float *rgb_out);
};

// C entry points so a harness that only has the RenderBackend* can read the float framebuffer and the last frame's
// per-stage device times / counters (SURVEY.md §8b; layouts of crtc_get_stage_times / crtc_get_counters in crt_cuda.h:
// up to 7 floats and 8 counters; with several renderers the times are the first one's, the counters are summed)
extern "C" int crt_cuda_read_accum(RenderBackend *backend, float *rgb_out);
extern "C" int crt_cuda_get_stats(RenderBackend *backend, float *stage_ms, int num_stages, uint64_t *counters, int num_counters);
