// render_cuda.cpp — RenderBackend -> C ABI adapter (include/crt_cuda.h).
//
// set_scene borrows the Scene's own vectors: glm::vec3/uvec3/vec2 arrays are tightly packed
// float/uint32 triples, DisneyMaterial (util/material.h:29-46) and QuadLight
// (util/lights.h:6-18) have exactly the crt_material_t / crt_quad_light_t layout, so nothing is
// copied on this side; the core library copies what it needs (the reference destroys its Scene
// right after set_scene, main.cpp:185-214).
#include "render_cuda.h"
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <stdexcept>
#include <thread>
#include <vector>
#include "crt_cuda.h"
#include "scene.h"
#ifndef CRT_CUDA_HEADLESS
#include <cuda_gl_interop.h>
#include <cuda_runtime_api.h>
#endif

static_assert(sizeof(DisneyMaterial) == sizeof(crt_material_t), "DisneyMaterial layout");
static_assert(sizeof(QuadLight) == sizeof(crt_quad_light_t), "QuadLight layout");
static_assert(sizeof(glm::vec3) == 12 && sizeof(glm::uvec3) == 12 && sizeof(glm::vec2) == 8 &&
                  sizeof(glm::mat4) == 64,
              "GLM types must be tightly packed");

namespace {
void check(int rc)
{
    if (rc != 0) {
        // the reference's error behaviour: std::runtime_error propagating to the app
        throw std::runtime_error(std::string("crt_cuda: ") + crtc_last_error());
    }
}

long env_or(const char *name, long fallback)
{
    const char *v = std::getenv(name);
    return v && *v ? std::strtol(v, nullptr, 10) : fallback;
}

// CRT_CUDA_DEVICES: a comma-separated list of CUDA device ordinals ("0,1,2,3"; a device may be named twice, which
// shards the image over two renderers on the same GPU — only useful for testing the fan-out on a one-GPU machine).
std::vector<int> devices_from_env()
{
    std::vector<int> devices;
    if (const char *v = std::getenv("CRT_CUDA_DEVICES")) {
        const char *p = v;
        while (*p) {
            char *end = nullptr;
            const long d = std::strtol(p, &end, 10);
            if (end == p) {
                throw std::runtime_error(std::string("crt_cuda: cannot parse CRT_CUDA_DEVICES='") + v + "'");
            }
            devices.push_back(static_cast<int>(d));
            p = *end == ',' ? end + 1 : end;
        }
    }
    if (devices.empty()) {
        devices.push_back(static_cast<int>(env_or("CRT_CUDA_DEVICE", 0)));
    }
    return devices;
}
}

RenderCUDA::RenderCUDA(bool native_display_) : native_display(native_display_)
{
#ifdef CRT_CUDA_HEADLESS
    native_display = false;
#endif
    // The plugin API has no option channel (SURVEY.md §5): knobs come from the environment.
    const std::vector<int> devices = devices_from_env();
    denoise = env_or("CRT_CUDA_DENOISE", 0) != 0;
    if (denoise && devices.size() > 1) {
        throw std::runtime_error("crt_cuda: CRT_CUDA_DENOISE needs the whole frame on one GPU; it cannot be combined with "
                                 "more than one device in CRT_CUDA_DEVICES");
    }
    // CRT_CUDA_DENOISE_HISTORY=H: the denoiser carries a reprojected history of up to H samples across camera moves
    const int64_t denoise_history = env_or("CRT_CUDA_DENOISE_HISTORY", 0);
    if (denoise_history != 0 && !denoise) {
        throw std::runtime_error("crt_cuda: CRT_CUDA_DENOISE_HISTORY is the denoiser's history; it needs CRT_CUDA_DENOISE=1");
    }
    // CRT_CUDA_ADAPTIVE=<threshold>: adaptive sampling (crtc_set_adaptive), with CRT_CUDA_ADAPTIVE_MIN_FRAMES (default 4)
    // and CRT_CUDA_ADAPTIVE_MAX_FRAMES (default 0 = no cap)
    const char *adaptive_env = std::getenv("CRT_CUDA_ADAPTIVE");
    const bool adaptive = adaptive_env && *adaptive_env;
    crtc_adaptive_params_t adaptive_params = {0.f, 4, 0};
    if (adaptive) {
        char *end = nullptr;
        adaptive_params.threshold = std::strtof(adaptive_env, &end);
        if (end == adaptive_env || *end != '\0') {
            throw std::runtime_error(std::string("crt_cuda: cannot parse CRT_CUDA_ADAPTIVE='") + adaptive_env + "' as a threshold");
        }
        if (denoise) {
            throw std::runtime_error("crt_cuda: CRT_CUDA_ADAPTIVE cannot be combined with CRT_CUDA_DENOISE=1 (the denoiser "
                                     "assumes the same number of samples in every pixel)");
        }
        const long min_frames = env_or("CRT_CUDA_ADAPTIVE_MIN_FRAMES", 4), max_frames = env_or("CRT_CUDA_ADAPTIVE_MAX_FRAMES", 0);
        if (min_frames < 0 || max_frames < 0) {
            throw std::runtime_error("crt_cuda: CRT_CUDA_ADAPTIVE_MIN_FRAMES and CRT_CUDA_ADAPTIVE_MAX_FRAMES must not be negative");
        }
        adaptive_params.min_frames = static_cast<uint32_t>(min_frames);
        adaptive_params.max_frames = static_cast<uint32_t>(max_frames);
    }
    try {
        for (size_t i = 0; i < devices.size(); ++i) {
            crtc_renderer *r = nullptr;
            check(crtc_create(&r, devices[i]));
            renderers.push_back(r);
            check(crtc_set_option(r, "world_size", static_cast<int64_t>(devices.size())));
            check(crtc_set_option(r, "rank", static_cast<int64_t>(i)));
            check(crtc_set_option(r, "max_depth", env_or("CRT_CUDA_MAX_DEPTH", 5)));
            check(crtc_set_option(r, "bvh_threads", env_or("CRT_CUDA_BVH_THREADS", 0)));
            check(crtc_set_option(r, "bvh_builder", env_or("CRT_CUDA_BVH_BUILDER", 0)));  // 1 / 2 = build on the device (crt_cuda.h)
            check(crtc_set_option(r, "any_far_first", env_or("CRT_CUDA_ANY_FAR_FIRST", 2)));  // crt_cuda.h; 2 = per scene
            check(crtc_set_option(r, "shade_sort", env_or("CRT_CUDA_SHADE_SORT", 0)));  // 1 / 2 = shade queue bucketed by material
            check(crtc_set_option(r, "hw_textures", env_or("CRT_CUDA_HW_TEXTURES", 0)));  // 1 = texels through cudaTextureObject_t (crt_cuda.h)
            check(crtc_set_option(r, "stage_events", env_or("CRT_CUDA_STAGE_EVENTS", 1)));  // 0 = no per-stage timings (crt_cuda_get_stats reads 0)
            check(crtc_set_option(r, "aov", denoise ? 1 : 0));  // CRT_CUDA_DENOISE: first-hit AOVs for crtc_denoise
            if (denoise_history != 0) {
                check(crtc_set_option(r, "denoise_history", denoise_history));  // (out of range: refused here)
            }
            if (adaptive) {
                check(crtc_set_adaptive(r, &adaptive_params));  // (out of range: refused here)
            }
        }
    } catch (...) {
        for (crtc_renderer *r : renderers) {
            crtc_destroy(r);
        }
        throw;
    }
    renderer = renderers[0];
}

#ifndef CRT_CUDA_HEADLESS
namespace {
void check_cuda(cudaError_t e, const char *what)
{
    if (e != cudaSuccess) {
        throw std::runtime_error(std::string("crt_cuda: ") + what + ": " + cudaGetErrorString(e));
    }
}
}

// render_optix.cpp:104-121: an RGBA8 texture of the framebuffer's size, registered with CUDA
void RenderCUDA::create_display_texture()
{
    release_display_texture();
    glGenTextures(1, &gl_display_texture);
    glBindTexture(GL_TEXTURE_2D, gl_display_texture);
    glTexImage2D(GL_TEXTURE_2D, 0, GL_RGBA8, fb_dims.x, fb_dims.y, 0, GL_RGBA, GL_UNSIGNED_BYTE, nullptr);
    glTexParameteri(GL_TEXTURE_2D, GL_TEXTURE_MIN_FILTER, GL_NEAREST);
    glTexParameteri(GL_TEXTURE_2D, GL_TEXTURE_MAG_FILTER, GL_NEAREST);
    glTexParameteri(GL_TEXTURE_2D, GL_TEXTURE_WRAP_S, GL_CLAMP_TO_EDGE);
    glTexParameteri(GL_TEXTURE_2D, GL_TEXTURE_WRAP_T, GL_CLAMP_TO_EDGE);
    check_cuda(cudaGraphicsGLRegisterImage(&cu_display_texture, gl_display_texture, GL_TEXTURE_2D, cudaGraphicsRegisterFlagsWriteDiscard),
               "cudaGraphicsGLRegisterImage");
}

void RenderCUDA::release_display_texture()
{
    if (cu_display_texture) {
        cudaGraphicsUnregisterResource(cu_display_texture);
        cu_display_texture = nullptr;
    }
    if (gl_display_texture != GLuint(-1)) {
        glDeleteTextures(1, &gl_display_texture);
        gl_display_texture = GLuint(-1);
    }
}

// render_optix.cpp:410-426: map the texture, copy the frame into its array device to device, unmap
void RenderCUDA::present_native()
{
    check_cuda(cudaGraphicsMapResources(1, &cu_display_texture), "cudaGraphicsMapResources");
    cudaArray_t array = nullptr;
    check_cuda(cudaGraphicsSubResourceGetMappedArray(&array, cu_display_texture, 0, 0), "cudaGraphicsSubResourceGetMappedArray");
    // (every GPU's tiles are in renderers[0]'s frame by then; CRT_CUDA_DENOISE: the denoised frame instead)
    const int rc = denoise ? crtc_denoise(renderers[0], nullptr, nullptr, nullptr, array) : crtc_copy_img_to_array(renderers[0], array);
    check_cuda(cudaGraphicsUnmapResources(1, &cu_display_texture), "cudaGraphicsUnmapResources");
    check(rc);
}
#endif

RenderCUDA::~RenderCUDA()
{
#ifndef CRT_CUDA_HEADLESS
    release_display_texture();
#endif
    // the renderers that write into renderers[0]'s frame go first
    for (size_t i = renderers.size(); i-- > 0;) {
        crtc_destroy(renderers[i]);
    }
}

std::string RenderCUDA::name()
{
    return crtc_name();
}

void RenderCUDA::initialize(const int fb_width, const int fb_height)
{
    fb_dims = glm::ivec2(fb_width, fb_height);
    img.resize(static_cast<size_t>(fb_width) * fb_height);
    for (crtc_renderer *r : renderers) {
        check(crtc_initialize(r, fb_width, fb_height));
    }
    for (size_t i = 1; i < renderers.size(); ++i) {
        check(crtc_share_frame(renderers[0], renderers[i]));
    }
#ifndef CRT_CUDA_HEADLESS
    if (native_display) {
        create_display_texture();
    }
#endif
}

void RenderCUDA::set_scene(const Scene &scene)
{
    samples_per_pixel = scene.samples_per_pixel;

    std::vector<std::vector<crt_geometry_t>> geometries(scene.meshes.size());
    std::vector<crt_mesh_t> meshes(scene.meshes.size());
    for (size_t m = 0; m < scene.meshes.size(); ++m) {
        for (const auto &g : scene.meshes[m].geometries) {
            crt_geometry_t cg;
            cg.vertices = reinterpret_cast<const float *>(g.vertices.data());
            cg.uvs = g.uvs.empty() ? nullptr : reinterpret_cast<const float *>(g.uvs.data());
            cg.indices = reinterpret_cast<const uint32_t *>(g.indices.data());
            cg.num_vertices = static_cast<uint32_t>(g.vertices.size());
            cg.num_tris = static_cast<uint32_t>(g.indices.size());
            geometries[m].push_back(cg);
        }
        meshes[m].geometries = geometries[m].data();
        meshes[m].num_geometries = static_cast<uint32_t>(geometries[m].size());
    }

    std::vector<crt_parameterized_mesh_t> pms;
    for (const auto &pm : scene.parameterized_meshes) {
        crt_parameterized_mesh_t c;
        c.material_ids = pm.material_ids.data();
        c.num_material_ids = static_cast<uint32_t>(pm.material_ids.size());
        c.mesh_id = static_cast<uint32_t>(pm.mesh_id);
        pms.push_back(c);
    }

    std::vector<crt_instance_t> instances;
    for (const auto &inst : scene.instances) {
        crt_instance_t c;
        std::memcpy(c.transform, &inst.transform[0][0], sizeof(c.transform));
        c.parameterized_mesh_id = static_cast<uint32_t>(inst.parameterized_mesh_id);
        instances.push_back(c);
    }

    std::vector<crt_image_t> textures;
    for (const auto &t : scene.textures) {
        crt_image_t c;
        c.data = t.img.data();
        c.width = t.width;
        c.height = t.height;
        c.channels = t.channels;
        c.color_space = t.color_space == SRGB ? CRT_COLOR_SPACE_SRGB : CRT_COLOR_SPACE_LINEAR;
        textures.push_back(c);
    }

    crt_scene_t c;
    c.meshes = meshes.data();
    c.parameterized_meshes = pms.data();
    c.instances = instances.data();
    c.materials = reinterpret_cast<const crt_material_t *>(scene.materials.data());
    c.textures = textures.data();
    c.lights = reinterpret_cast<const crt_quad_light_t *>(scene.lights.data());
    c.num_meshes = static_cast<uint32_t>(meshes.size());
    c.num_parameterized_meshes = static_cast<uint32_t>(pms.size());
    c.num_instances = static_cast<uint32_t>(instances.size());
    c.num_materials = static_cast<uint32_t>(scene.materials.size());
    c.num_textures = static_cast<uint32_t>(textures.size());
    c.num_lights = static_cast<uint32_t>(scene.lights.size());
    c.samples_per_pixel = scene.samples_per_pixel;
    frames_since_scene = 0;
    if (renderers.size() == 1) {
        check(crtc_set_scene(renderer, &c));
        return;
    }
    // every GPU gets its own copy of the scene and builds its own BVH (the scene is replicated, SURVEY.md §8e): one
    // host thread per renderer, errors collected and rethrown here as the reference would throw them
    std::vector<std::exception_ptr> errors(renderers.size());
    std::vector<std::thread> workers;
    for (size_t i = 0; i < renderers.size(); ++i) {
        workers.emplace_back([&, i] {
            try {
                check(crtc_set_scene(renderers[i], &c));
            } catch (...) {
                errors[i] = std::current_exception();
            }
        });
    }
    for (std::thread &w : workers) {
        w.join();
    }
    for (const std::exception_ptr &e : errors) {
        if (e) {
            std::rethrow_exception(e);
        }
    }
}

RenderStats RenderCUDA::render(const glm::vec3 &pos,
                               const glm::vec3 &dir,
                               const glm::vec3 &up,
                               const float fovy,
                               const bool camera_changed,
                               const bool readback_framebuffer)
{
    // with a non-native display the app reads `img` every frame (gldisplay.cpp:111-123)
    const bool readback = readback_framebuffer || !native_display;
    if (renderers.size() > 1) {
        // fan out: every GPU is handed its share of the frame before any of them is waited for; each resolves its
        // tiles into renderers[0]'s frame, which is complete once all of them have finished
        const auto t0 = std::chrono::steady_clock::now();
        uint64_t rays = 0;
        if (frames_since_scene < 3) {
            // the per-scene choice of the shadow-ray order (any_far_first = 2, crt_cuda.h) is made from the stage times
            // of blocking frames 1 and 2: the first three frames go through crtc_render, one renderer after the other
            for (crtc_renderer *r : renderers) {
                crt_render_stats_t part;
                check(crtc_render(r, &pos.x, &dir.x, &up.x, fovy, camera_changed ? 1 : 0, 0, nullptr, &part));
                rays += part.num_rays;
            }
        } else {
            for (crtc_renderer *r : renderers) {
                check(crtc_render_async(r, &pos.x, &dir.x, &up.x, fovy, camera_changed ? 1 : 0, 1));
            }
            for (crtc_renderer *r : renderers) {
                crt_render_stats_t part;
                check(crtc_sync(r, &part, nullptr, nullptr, nullptr));
                rays += part.num_rays;
            }
        }
        ++frames_since_scene;
#ifndef CRT_CUDA_HEADLESS
        if (native_display) {
            present_native();
        }
#endif
        if (readback) {
            check(crtc_read_img(renderers[0], img.data()));
        }
        RenderStats stats;
        stats.render_time = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
        stats.rays_per_second = static_cast<float>(static_cast<double>(rays) / (stats.render_time * 1e-3));
        return stats;
    }
    crt_render_stats_t s;
    check(crtc_render(renderer,
                      &pos.x,
                      &dir.x,
                      &up.x,
                      fovy,
                      camera_changed ? 1 : 0,
                      readback && !denoise ? 1 : 0,
                      img.data(),
                      &s));
    if (readback && denoise) {
        check(crtc_denoise(renderer, nullptr, nullptr, img.data(), nullptr));
    }
#ifndef CRT_CUDA_HEADLESS
    if (native_display) {
        present_native();
    }
#endif
    RenderStats stats;
    stats.render_time = s.render_time;
    stats.rays_per_second = s.rays_per_second;
    return stats;
}

void RenderCUDA::read_accum(float *rgb_out)
{
    check(crtc_read_accum(renderer, rgb_out));
}

extern "C" int crt_cuda_read_accum(RenderBackend *backend, float *rgb_out)
{
    RenderCUDA *r = dynamic_cast<RenderCUDA *>(backend);
    if (!r) {
        return 1;
    }
    r->read_accum(rgb_out);
    return 0;
}

extern "C" int crt_cuda_get_stats(RenderBackend *backend, float *stage_ms, int num_stages, uint64_t *counters, int num_counters)
{
    RenderCUDA *r = dynamic_cast<RenderCUDA *>(backend);
    if (!r) {
        return 1;
    }
    if (stage_ms && num_stages > 0) {
        const int n = crtc_get_stage_times(r->renderers[0], stage_ms, num_stages);
        for (int i = n; i < num_stages; ++i) {
            stage_ms[i] = 0.f;
        }
    }
    if (counters && num_counters > 0) {
        for (int i = 0; i < num_counters; ++i) {
            counters[i] = 0;
        }
        for (crtc_renderer *shard : r->renderers) {
            uint64_t part[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            const int n = crtc_get_counters(shard, part, 8);
            for (int i = 0; i < n && i < num_counters; ++i) {
                counters[i] += part[i];
            }
        }
    }
    return 0;
}
