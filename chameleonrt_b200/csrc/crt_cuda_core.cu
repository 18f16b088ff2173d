// crt_cuda_core.cu — the renderer object behind the C ABI of include/crt_cuda.h.
//
// Host-side role = RenderEmbree / RenderOptiX (reference backends/embree/render_embree.cpp,
// backends/optix/render_optix.cpp): own the device scene, compute the camera basis, launch the
// frame, time it, read the framebuffer back. Everything per-frame runs on the GPU as the
// kernel chain of kernels.cuh; there is no CPU fallback anywhere in this file.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <memory>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/crt_cuda.h"
#include "adaptive.cuh"
#include "aov_denoise.cuh"
#include "bvh8.h"
#include "cuda_host_utils.h"
#include "host_scene.h"
#include "kernels.cuh"
#include "scene_device_build.cuh"
#include "scene_update.cuh"

namespace {

thread_local std::string g_last_error;

using crt_host::ArenaBuf;
using crt_host::DeviceArena;
using crt_host::DeviceBuffer;

enum Stage { kStRaygen = 0, kStPrimary, kStShade, kStTraverse, kStNee, kStResolve, kStFrame, kNumStages };

// What one enqueued frame leaves behind for later collection: its stage events and a pinned copy
// of its device counters. Several frames may be in flight (crtc_render_async), so every frame has
// its own record.
struct FrameRecord {
    std::vector<cudaEvent_t> events;
    std::vector<int> event_stage;  // stage that ENDS at event i (i >= 1)
    size_t num_events = 0;
    uint32_t *h_counters = nullptr;  // pinned
    unsigned long long *h_trav = nullptr;
    uint32_t launches = 0;
    uint32_t frames = 1;  // frames rendered by this record's launch sequence

    FrameRecord()
    {
        CUDA_CHECK(cudaMallocHost(&h_counters, crt::kNumCounters * sizeof(uint32_t)));
        CUDA_CHECK(cudaMallocHost(&h_trav, 4 * sizeof(unsigned long long)));
    }
    ~FrameRecord()
    {
        for (auto e : events) {
            cudaEventDestroy(e);
        }
        cudaFreeHost(h_counters);
        cudaFreeHost(h_trav);
    }
    bool all_stages = true;  // false: only the first and the last mark of a frame are recorded (option "stage_events" = 0)
    void mark(cudaStream_t s, int stage_ended)
    {
        if (!all_stages && stage_ended != -1 && stage_ended != kStResolve) {
            return;
        }
        if (num_events >= events.size()) {
            cudaEvent_t e;
            CUDA_CHECK(cudaEventCreate(&e));
            events.push_back(e);
            event_stage.push_back(0);
        }
        event_stage[num_events] = stage_ended;
        CUDA_CHECK(cudaEventRecord(events[num_events++], s));
    }
};

}  // namespace

struct crtc_renderer {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t own_stream = nullptr;

    // options
    int max_depth = 5;
    int rank = 0, world_size = 1;
    int bvh_threads = 0;
    int bvh_builder = 0;  // 0 = host (binned SAH, bvh8_build.cpp); on the device (bvh8_device.cuh): 1 = PLOC, 2 = LBVH
    int build_rounds = 0;
    int ploc_radius = crt::kPlocRadius;
    bool ploc_tail = true;  // the last rounds of PLOC in one block (k_ploc_tail); off only to test that the tree is the same
    bool count_traversal = false;
    int refill_idle = crt::kRefillIdle;  // idle lanes that trigger a refill of the traversal warps
    bool bvh_top_smem = false;           // option "bvh_top_smem": the first 73 BVH nodes read from a shared-memory copy (measured: no gain)
    int tri_pass_defer = 16;             // 0 / 16 (default) / 24: pooled pairs a triangle pass waits for (kernels.cuh)
    // The shade queue bucketed by material id before k_shade (k_queue_hist / k_queue_scatter): 0 = off (default),
    // 1 = from the first bounce on (primary hits keep their screen order), 2 = every shade launch. Same image.
    int shade_sort = 0;
    // Shadow rays visit the children of a node farthest-first: 0 = no, 1 = yes, 2 = auto (default) — frame 1
    // after set_scene is rendered far-first, frame 2 near-first, and far-first is kept from frame 3 on only if its
    // traversal stage was at least 3 % faster (blocking render() calls only; the image is the same either way).
    // Far-first is tried on the EARLIER, possibly colder frame on purpose: whatever warm-up effect is left works
    // against the switch, so a wrong decision can only mean staying with near-first.
    int any_far_first = 2;
    int auto_frames = 0;            // blocking frames rendered since set_scene (auto mode)
    float auto_trav_ms[2] = {0.f, 0.f};
    bool auto_decided = false, auto_choice = false;
    bool frame_far_first = false;   // the order used by the frame being enqueued

    // `blocking`: the frame comes from render(), whose stage times feed auto_tune_step(). Frames enqueued with
    // crtc_render_async never advance the trial, so while it is undecided they run near-first (the order the
    // instrumented counting pass of bench.py assumes for "undecided").
    bool pick_far_first(bool blocking) const
    {
        if (any_far_first != 2) {
            return any_far_first == 1;
        }
        return auto_decided ? auto_choice : (blocking && auto_frames == 1);
    }
    // after a blocking frame's stage times are known
    void auto_tune_step()
    {
        if (any_far_first != 2 || auto_decided) {
            return;
        }
        if (auto_frames == 1 || auto_frames == 2) {
            auto_trav_ms[auto_frames - 1] = stage_ms[kStTraverse];  // [0] far-first (frame 1), [1] near-first (frame 2)
        }
        if (auto_frames == 2) {
            auto_decided = true;
            auto_choice = auto_trav_ms[0] < 0.97f * auto_trav_ms[1];  // switch only for a clear gain
        }
        ++auto_frames;
    }

    // framebuffer layout
    int fb_w = 0, fb_h = 0;
    uint32_t ntx = 0;
    std::vector<uint32_t> local_tiles;
    uint32_t npx_local = 0;
    uint32_t frame_id = 0;
    uint32_t spp = 1;
    bool have_scene = false;

    // Option "views" (crtc_render_views): `views` is the option, `views_active` what the last crtc_initialize set up. With
    // views_active > 1 the local and full framebuffers hold that many views, view-major, and view k's frame counter is
    // view_frames[k] (frame_id is then unused).
    uint32_t views = 1, views_active = 1;
    std::vector<uint32_t> view_frames{0u};
    void require_single_view(const char *what) const
    {
        if (views_active > 1) {
            throw std::runtime_error(std::string(what) + ": this renderer was initialized with option views = " +
                                     std::to_string(views_active) + "; render with crtc_render_views and read with crtc_read_view");
        }
    }

    // device scene
    DeviceBuffer<float4> d_nodes, d_tris, d_shade, d_materials, d_lights;
    DeviceBuffer<uint32_t> d_texels;
    DeviceBuffer<crt::DevTex> d_tex;
    // option "hw_textures": one CUDA array + texture object per scene texture (wrap, linear, normalised coordinates, sRGB
    // decode in the texture unit — the reference's OptiX backend, backends/optix/optix_utils.cpp:60-85)
    bool hw_textures = false;
    std::vector<cudaArray_t> tex_arrays;
    std::vector<cudaTextureObject_t> tex_objects;
    DeviceBuffer<unsigned long long> d_tex_objects;
    void release_hw_textures()
    {
        for (cudaTextureObject_t t : tex_objects) {
            cudaDestroyTextureObject(t);
        }
        for (cudaArray_t a : tex_arrays) {
            cudaFreeArray(a);
        }
        tex_objects.clear();
        tex_arrays.clear();
    }
    void build_hw_textures(const crt_scene_t *scene)
    {
        release_hw_textures();
        if (!hw_textures || scene->num_textures == 0) {
            d_tex_objects.release();
            return;
        }
        std::vector<uchar4> rgba;
        for (uint32_t i = 0; i < scene->num_textures; ++i) {
            const crt_image_t &im = scene->textures[i];  // (shape checked by pack_shading)
            const size_t n = (size_t)im.width * im.height;
            rgba.assign(n, make_uchar4(0, 0, 0, 0));  // channels the image lacks read as 0 (texture2d.ih:13-27)
            for (size_t px = 0; px < n; ++px) {
                unsigned char c[4] = {0, 0, 0, 0};
                for (int k = 0; k < im.channels; ++k) {
                    c[k] = im.data[px * im.channels + k];
                }
                rgba[px] = make_uchar4(c[0], c[1], c[2], c[3]);
            }
            const cudaChannelFormatDesc fmt = cudaCreateChannelDesc<uchar4>();
            cudaArray_t arr = nullptr;
            CUDA_CHECK(cudaMallocArray(&arr, &fmt, (size_t)im.width, (size_t)im.height));
            tex_arrays.push_back(arr);
            CUDA_CHECK(cudaMemcpy2DToArrayAsync(arr, 0, 0, rgba.data(), (size_t)im.width * 4, (size_t)im.width * 4, (size_t)im.height,
                                                cudaMemcpyHostToDevice, stream));
            CUDA_CHECK(cudaStreamSynchronize(stream));  // `rgba` is reused
            cudaResourceDesc res = {};
            res.resType = cudaResourceTypeArray;
            res.res.array.array = arr;
            cudaTextureDesc td = {};
            td.addressMode[0] = td.addressMode[1] = cudaAddressModeWrap;
            td.filterMode = cudaFilterModeLinear;
            td.readMode = cudaReadModeNormalizedFloat;
            td.sRGB = im.color_space == CRT_COLOR_SPACE_SRGB ? 1 : 0;
            td.normalizedCoords = 1;
            cudaTextureObject_t obj = 0;
            CUDA_CHECK(cudaCreateTextureObject(&obj, &res, &td, nullptr));
            tex_objects.push_back(obj);
        }
        static_assert(sizeof(cudaTextureObject_t) == sizeof(unsigned long long), "texture handles are 64-bit");
        d_tex_objects.upload(reinterpret_cast<const unsigned long long *>(tex_objects.data()), tex_objects.size(), stream);
        CUDA_CHECK(cudaStreamSynchronize(stream));
    }
    uint32_t num_lights = 0;
    std::vector<uint32_t> leaf_flat_ids;  // host copy: leaf-order triangle -> flattened prim id
    // Option "dynamic_scene" (scene_update.cuh): `dynamic_scene` is the option, `scene_update` what the last set_scene
    // kept for updates (null with the option off). Lights need no kept state: `staged_lights` waits for the commit.
    bool dynamic_scene = false;
    std::unique_ptr<crt_host::SceneUpdate> scene_update;
    std::vector<crt_quad_light_t> staged_lights;
    bool lights_staged = false;
    double scene_info[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};  // crtc_get_scene_info
    double phase_ms[5] = {0, 0, 0, 0, 0};  // last set_scene: flatten, keys + sort, binary tree, BVH8 emission, packing

    // path state
    size_t path_capacity = 0;
    DeviceBuffer<float4> d_ray_o, d_ray_d, d_hit, d_thr_rng, d_radiance, d_nee_T, d_nee_l1, d_nee_l2, d_sray_o,
        d_sray_d;
    DeviceBuffer<uint8_t> d_vis;
    DeviceBuffer<uint32_t> d_queue0, d_queue1, d_counters;
    DeviceBuffer<uint32_t> d_queue_sorted, d_sort_hist, d_sort_scratch;  // option shade_sort
    DeviceBuffer<unsigned long long> d_trav_counters;

    // framebuffers
    DeviceBuffer<uint32_t> d_tile_ids;
    DeviceBuffer<float> d_accum_local, d_accum_full;
    DeviceBuffer<uint32_t> d_img_local, d_img_full;

    // option "aov" (aov_denoise.cuh): first-hit AOVs accumulated with the frame, and the denoiser over them. `aov` is the
    // option, `aov_active` what the last crtc_initialize set up.
    bool aov = false, aov_active = false;
    crt::AovState aov_state;
    // option "denoise_history": the most samples crtc_denoise's temporal history may carry (0 = off); `dn_history_active`
    // is what the last crtc_initialize set up. `epoch` counts accumulation resets that were followed by a frame;
    // `epoch_view` is the camera of the current epoch's first frame.
    uint32_t dn_history = 0, dn_history_active = 0;
    uint64_t epoch = 0;
    crt::ViewParams epoch_view{};
    // option "denoise_motion": a commit that moves geometry keeps the history, reprojected through each pixel's triangle;
    // `dn_motion_active` is what the last crtc_initialize set up. `geometry_version` counts crtc_set_scene calls and
    // commits with staged instances or vertices.
    bool dn_motion = false, dn_motion_active = false;
    uint64_t geometry_version = 0;
    // The frame index the current epoch's samples start from (k_raygen's seeds): 0 after every reset, except that a
    // commit keeping the history (option denoise_motion) continues from where the epoch before it ended, so that a still
    // pixel draws new samples instead of re-rendering the ones its history already holds. A camera_changed render
    // right after such a commit does not restart it.
    uint32_t sample_base = 0;
    bool motion_frames() const { return dn_motion_active && scene_update != nullptr; }
    void require_unshared_aov(const char *what) const
    {
        if (aov_active) {
            throw std::runtime_error(std::string(what) + ": the AOVs and the denoiser need the whole frame on one renderer; "
                                     "this renderer was initialized with option aov = 1");
        }
    }
    void require_aov_frame(const char *what) const
    {
        if (!aov_active) {
            throw std::runtime_error(std::string(what) + ": option aov is off (set it to 1 before crtc_initialize)");
        }
        if (frame_id == 0) {
            throw std::runtime_error(std::string(what) + ": no frame has been rendered since the last reset");
        }
    }

    // Adaptive sampling (crtc_set_adaptive, adaptive.cuh). `adaptive` = the mode is set; `adaptive_epoch` = the per-block
    // counts are in use, from the first adaptive wavefront after a reset until the next reset (switching the mode off in
    // between keeps them, with every block active); `adaptive_base` = frame_id at that first wavefront, where the
    // statistics start.
    bool adaptive = false, adaptive_epoch = false;
    crtc_adaptive_params_t adaptive_params{};
    uint32_t adaptive_base = 0;
    crt::AdaptiveState adaptive_state;
    void set_adaptive(const crtc_adaptive_params_t *params)
    {
        if (!params) {
            adaptive = false;
            return;
        }
        if (views_active > 1) {
            throw std::runtime_error("crtc_set_adaptive: adaptive sampling is not available with crtc_render_views; this renderer "
                                     "was initialized with option views = " + std::to_string(views_active));
        }
        if (aov_active) {
            throw std::runtime_error("crtc_set_adaptive: adaptive sampling cannot be combined with option aov (the AOVs and the "
                                     "denoiser assume the same number of samples in every pixel); this renderer was "
                                     "initialized with aov = 1");
        }
        if (!std::isfinite(params->threshold) || params->threshold < 0.f) {
            throw std::runtime_error("crtc_set_adaptive: threshold must be finite and >= 0");
        }
        if (params->min_frames < 1) {
            throw std::runtime_error("crtc_set_adaptive: min_frames must be >= 1");
        }
        if (params->max_frames != 0 && params->max_frames < params->min_frames) {
            throw std::runtime_error("crtc_set_adaptive: max_frames must be 0 (no cap) or >= min_frames");
        }
        adaptive = true;
        adaptive_params = *params;
    }
    void read_adaptive(uint32_t *samples_out, float *error_out)
    {
        if (!adaptive_epoch || frame_id == 0) {
            throw std::runtime_error("crtc_read_adaptive: no frame has been rendered with adaptive sampling since the last reset");
        }
        make_current();
        if ((samples_out || error_out) && npx_local) {
            adaptive_state.readout(frame_layout(), adaptive_base, samples_out, error_out, stream);
        }
        CUDA_CHECK(cudaGetLastError());
    }

    // frames: records of enqueued-but-not-collected frames, and a pool of reusable ones
    std::vector<std::unique_ptr<FrameRecord>> in_flight, record_pool;
    float stage_ms[kNumStages] = {0};   // last collected frame
    uint64_t counters_out[8] = {0};     // last collected frame

    // Peer-written frames (multi-GPU without a gather): the assembling rank exports its full-frame buffers as CUDA
    // IPC handles, the other ranks map them and their k_resolve stores each pixel there as well (st.global to a
    // peer address over NVLink). Tile ownership is disjoint, so there is nothing to reduce.
    bool frame_exported = false;
    // Completion flags of a shared frame (kernels.cuh "frame completion flags"): share_seq counts the wavefronts enqueued
    // since the frame was shared (every rank enqueues the same sequence of crtc_render / crtc_render_async calls).
    uint32_t share_seq = 0;
    DeviceBuffer<uint32_t> d_done_counter;
    uint32_t *h_sync_err = nullptr, *d_sync_err = nullptr;  // one mapped host word: a flag wait that timed out
    uint32_t *sync_words() { return d_img_full.ptr + (size_t)fb_w * fb_h; }
    uint32_t *peer_sync_words() { return peer_img_full + (size_t)fb_w * fb_h; }
    void ensure_sync_state()
    {
        if (!d_done_counter.ptr) {
            d_done_counter.alloc(1);
            CUDA_CHECK(cudaMemsetAsync(d_done_counter.ptr, 0, sizeof(uint32_t), stream));
        }
        if (!h_sync_err) {
            CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void **>(&h_sync_err), sizeof(uint32_t), cudaHostAllocMapped));
            *h_sync_err = 0u;
            CUDA_CHECK(cudaHostGetDevicePointer(reinterpret_cast<void **>(&d_sync_err), h_sync_err, 0));
        }
    }
    void reset_share_sequence()
    {
        share_seq = 0;
        if (d_img_full.ptr && fb_w) {
            CUDA_CHECK(cudaMemsetAsync(sync_words(), 0, crt::kSyncWords * sizeof(uint32_t), stream));
            CUDA_CHECK(cudaStreamSynchronize(stream));
        }
    }
    void check_sync_error()
    {
        if (h_sync_err && *h_sync_err) {
            const uint32_t who = *h_sync_err - 1u;
            *h_sync_err = 0u;
            throw std::runtime_error("shared frame: rank " + std::to_string(who) + "'s completion flag did not arrive within 20 s "
                                     "(every rank must enqueue the same sequence of frames)");
        }
    }
    // On the assembling rank, stream-ordered: everything enqueued afterwards sees the frame of the last enqueued
    // wavefront complete, every rank's tiles included.
    void frame_wait()
    {
        if (!frame_exported || world_size < 2 || share_seq == 0) {
            return;
        }
        make_current();
        ensure_sync_state();
        crt::k_wait_words<<<1, 32, 0, stream>>>(sync_words(), (uint32_t)world_size, (uint32_t)rank, share_seq, d_sync_err);
        CUDA_CHECK(cudaGetLastError());
    }
    float *peer_accum_full = nullptr;
    uint32_t *peer_img_full = nullptr;
    bool peer_is_ipc = false;  // mapped through cudaIpcOpenMemHandle (another process) or a plain peer pointer (this one)

    void close_peer_frame()
    {
        if (peer_accum_full && peer_is_ipc) {
            cudaIpcCloseMemHandle(peer_accum_full);
            cudaIpcCloseMemHandle(peer_img_full);
        }
        peer_accum_full = nullptr;
        peer_img_full = nullptr;
    }
    // The in-process form (one host thread driving several renderers, as the ChameleonRT plugin does): this renderer
    // resolves its tiles into `dst`'s full frame; different devices need peer access, which NVSwitch gives every pair.
    void share_frame_of(crtc_renderer *dst)
    {
        if (dst == this) {
            throw std::runtime_error("crtc_share_frame: source and destination are the same renderer");
        }
        if (fb_w == 0 || dst->fb_w != fb_w || dst->fb_h != fb_h) {
            throw std::runtime_error("crtc_share_frame: both renderers must be initialized with the same size");
        }
        require_unshared_aov("crtc_share_frame");
        dst->require_unshared_aov("crtc_share_frame");
        make_current();
        close_peer_frame();
        if (dst->device != device) {
            int can = 0;
            CUDA_CHECK(cudaDeviceCanAccessPeer(&can, device, dst->device));
            if (!can) {
                throw std::runtime_error("crtc_share_frame: device " + std::to_string(device) + " cannot access device " +
                                         std::to_string(dst->device));
            }
            const cudaError_t err = cudaDeviceEnablePeerAccess(dst->device, 0);
            if (err == cudaErrorPeerAccessAlreadyEnabled) {
                cudaGetLastError();  // not an error: clear it
            } else {
                CUDA_CHECK(err);
            }
        }
        peer_accum_full = dst->d_accum_full.ptr;
        peer_img_full = dst->d_img_full.ptr;
        peer_is_ipc = false;
        share_seq = 0;
        if (!dst->frame_exported) {
            dst->make_current();
            dst->reset_share_sequence();
            make_current();
        }
        dst->frame_exported = true;
    }
    void export_frame(void *handles_out)
    {
        if (fb_w == 0) {
            throw std::runtime_error("crtc_export_frame: initialize() has not been called");
        }
        require_unshared_aov("crtc_export_frame");
        make_current();
        static_assert(sizeof(cudaIpcMemHandle_t) == 64, "two 64-byte handles");
        cudaIpcMemHandle_t h[2];
        CUDA_CHECK(cudaIpcGetMemHandle(&h[0], d_accum_full.ptr));
        CUDA_CHECK(cudaIpcGetMemHandle(&h[1], d_img_full.ptr));
        std::memcpy(handles_out, h, sizeof(h));
        reset_share_sequence();
        frame_exported = true;
    }
    void import_frame(const void *handles)
    {
        make_current();
        close_peer_frame();
        if (!handles) {
            return;
        }
        require_unshared_aov("crtc_import_frame");
        cudaIpcMemHandle_t h[2];
        std::memcpy(h, handles, sizeof(h));
        void *a = nullptr, *i = nullptr;
        CUDA_CHECK(cudaIpcOpenMemHandle(&a, h[0], cudaIpcMemLazyEnablePeerAccess));
        const cudaError_t err = cudaIpcOpenMemHandle(&i, h[1], cudaIpcMemLazyEnablePeerAccess);
        if (err != cudaSuccess) {
            cudaIpcCloseMemHandle(a);
            CUDA_CHECK(err);
        }
        peer_accum_full = static_cast<float *>(a);
        peer_img_full = static_cast<uint32_t *>(i);
        peer_is_ipc = true;
        share_seq = 0;
    }

    // The caller's `img` (RenderBackend::img: a std::vector / numpy array that lives as long as the framebuffer size) is
    // page-locked on first use so that the frame-end readback is one DMA transfer instead of a staged pageable copy
    // (3.7 MB at 1280x720: ~0.35 ms -> ~0.15 ms per frame). Registration failures are not errors: the copy then stays pageable.
    void *pinned_img = nullptr;
    size_t pinned_bytes = 0;
    void unpin_img()
    {
        if (pinned_img) {
            cudaHostUnregister(pinned_img);
            cudaGetLastError();
            pinned_img = nullptr;
            pinned_bytes = 0;
        }
    }
    void pin_img(void *img, size_t bytes)
    {
        if (img == pinned_img && bytes == pinned_bytes) {
            return;
        }
        unpin_img();
        if (pin_host_buffers && cudaHostRegister(img, bytes, cudaHostRegisterDefault) == cudaSuccess) {
            pinned_img = img;
            pinned_bytes = bytes;
        } else {
            cudaGetLastError();
        }
    }
    // Option "stage_events": 1 (default) = a CUDA event after every launch, for the per-stage times of
    // crtc_get_stage_times; 0 = only at the start and the end of a frame (the stage times then read 0 except [6], the
    // whole frame; with a 1/8 shard per GPU the 27 event records are a measurable part of a 2 ms frame).
    bool stage_events = true;
    bool pin_host_buffers = true;  // option "pin_host_buffers"
    bool pin_repeated_reads = false;  // option "pin_read_img": crtc_read_img page-locks its destination too (a frame loop)

    ~crtc_renderer()
    {
        unpin_img();
        release_hw_textures();
        close_peer_frame();
        in_flight.clear();
        record_pool.clear();
        if (own_stream) {
            cudaStreamDestroy(own_stream);
        }
        if (h_sync_err) {
            cudaFreeHost(h_sync_err);
        }
    }

    void make_current() { CUDA_CHECK(cudaSetDevice(device)); }

    // persistent traversal grid: every SM filled with as many blocks as fit
    unsigned trav_grid = 0;
    int num_sms = 0;
    void launch_traverse(const crt::DeviceScene &sc, const crt::PathState &ps, const uint32_t *queue,
                         const uint32_t *count_closest, const uint32_t *count_any, uint32_t *work_counter)
    {
        if (trav_grid == 0) {
            int sms = 0, per_sm = 0;
            CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
            CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, crt::k_traverse<false>, crt::kTravBlock, 0));
            trav_grid = (unsigned)(sms * std::max(1, per_sm));
        }
        const int sched = (refill_idle & 0xff) | (frame_far_first ? 0x100 : 0);
        if (bvh_top_smem && !count_traversal && tri_pass_defer == 16) {  // experiment (kernels.cuh: TOP), default scheduling only
            crt::k_traverse<false, 16, true><<<trav_grid, crt::kTravBlock, 0, stream>>>(sc, ps, queue, count_closest, count_any, work_counter, sched,
                                                                                         (uint32_t)scene_info[1]);
            return;
        }
        // (one instantiation per variant, so that the default kernel's code does not change with the options)
        const int variant = (count_traversal ? 1 : 0) | (tri_pass_defer == 16 ? 2 : (tri_pass_defer == 24 ? 4 : 0));
        switch (variant) {
        case 0:
            crt::k_traverse<false><<<trav_grid, crt::kTravBlock, 0, stream>>>(sc, ps, queue, count_closest, count_any, work_counter, sched);
            break;
        case 1:
            crt::k_traverse<true><<<trav_grid, crt::kTravBlock, 0, stream>>>(sc, ps, queue, count_closest, count_any, work_counter, sched);
            break;
        case 2:
            crt::k_traverse<false, 16><<<trav_grid, crt::kTravBlock, 0, stream>>>(sc, ps, queue, count_closest, count_any, work_counter, sched);
            break;
        case 3:
            crt::k_traverse<true, 16><<<trav_grid, crt::kTravBlock, 0, stream>>>(sc, ps, queue, count_closest, count_any, work_counter, sched);
            break;
        case 4:
            crt::k_traverse<false, 24><<<trav_grid, crt::kTravBlock, 0, stream>>>(sc, ps, queue, count_closest, count_any, work_counter, sched);
            break;
        default:
            crt::k_traverse<true, 24><<<trav_grid, crt::kTravBlock, 0, stream>>>(sc, ps, queue, count_closest, count_any, work_counter, sched);
            break;
        }
    }

    // exclusive scan of n uint32 in place; `scratch` holds the tile sums of every recursion level. Returns its launches.
    int scan_u32(uint32_t *data, uint32_t n, uint32_t *scratch)
    {
        const unsigned tiles = (n + crt::kBuildTile - 1) / crt::kBuildTile;
        crt::k_scan_tile<uint32_t><<<tiles, crt::kBuildBlock, 0, stream>>>(data, data, n, tiles > 1 ? scratch : nullptr);
        if (tiles <= 1) {
            return 1;
        }
        const int below = scan_u32(scratch, tiles, scratch + tiles);
        crt::k_scan_add<uint32_t><<<tiles, crt::kBuildBlock, 0, stream>>>(data, n, scratch);
        return below + 2;
    }

    // Option shade_sort: queue `queue_in` of bounce `bounce` (length on the device, capacity `npaths`) bucketed by the
    // material of each path's hit into d_queue_sorted. Returns the number of launches.
    int sort_shade_queue(const crt::DeviceScene &sc, const crt::PathState &ps, const uint32_t *queue_in, int bounce, size_t npaths)
    {
        const uint32_t num_tiles = (uint32_t)((npaths + crt::kSortTile - 1) / crt::kSortTile);
        const uint32_t hist_items = 256u * num_tiles;
        size_t scratch_items = 1, left = hist_items;
        while (left > (size_t)crt::kBuildTile) {
            left = (left + crt::kBuildTile - 1) / crt::kBuildTile;
            scratch_items += left;
        }
        if (d_queue_sorted.count < npaths || d_sort_hist.count < hist_items || d_sort_scratch.count < scratch_items) {
            CUDA_CHECK(cudaStreamSynchronize(stream));  // (first frame with the option on, or a larger batch)
            d_queue_sorted.alloc(npaths);
            d_sort_hist.alloc(hist_items);
            d_sort_scratch.alloc(scratch_items);
        }
        crt::k_queue_hist<256><<<num_tiles, crt::kSortBlock, 0, stream>>>(sc, ps, queue_in, bounce, d_sort_hist.ptr, num_tiles);
        const int scans = scan_u32(d_sort_hist.ptr, hist_items, d_sort_scratch.ptr);
        crt::k_queue_scatter<256><<<num_tiles, crt::kSortBlock, 0, stream>>>(sc, ps, queue_in, d_queue_sorted.ptr, bounce, d_sort_hist.ptr, num_tiles);
        return scans + 2;
    }

    crt::DeviceScene device_scene() const
    {
        crt::DeviceScene sc;
        sc.nodes = d_nodes.ptr;
        sc.tris = d_tris.ptr;
        sc.shade = d_shade.ptr;
        sc.materials = d_materials.ptr;
        sc.lights = d_lights.ptr;
        sc.texels = d_texels.ptr;
        sc.tex = d_tex.ptr;
        sc.tex_objects = d_tex_objects.ptr;
        sc.num_lights = num_lights;
        sc.float_one = 0x3F800000u;
        return sc;
    }

    crt::FrameLayout frame_layout() const
    {
        crt::FrameLayout f;
        f.fb_w = fb_w;
        f.fb_h = fb_h;
        f.ntx = ntx;
        f.npx_local = npx_local;
        f.spp = spp;
        f.frames = 1;
        f.tile_ids = d_tile_ids.ptr;
        return f;
    }

    crt::PathState path_state()
    {
        crt::PathState ps;
        ps.ray_o = d_ray_o.ptr;
        ps.ray_d = d_ray_d.ptr;
        ps.hit = d_hit.ptr;
        ps.thr_rng = d_thr_rng.ptr;
        ps.radiance = d_radiance.ptr;
        ps.nee_T = d_nee_T.ptr;
        ps.nee_l1 = d_nee_l1.ptr;
        ps.nee_l2 = d_nee_l2.ptr;
        ps.sray_o = d_sray_o.ptr;
        ps.sray_d = d_sray_d.ptr;
        ps.vis = d_vis.ptr;
        ps.queue[0] = d_queue0.ptr;
        ps.queue[1] = d_queue1.ptr;
        ps.counters = d_counters.ptr;
        ps.trav_counters = d_trav_counters.ptr;
        return ps;
    }

    void ensure_path_buffers(size_t npaths)
    {
        if (npaths <= path_capacity && d_counters.ptr) {
            return;
        }
        d_ray_o.alloc(npaths);
        d_ray_d.alloc(npaths);
        d_hit.alloc(npaths);
        d_thr_rng.alloc(npaths);
        d_radiance.alloc(npaths);
        d_nee_T.alloc(npaths);
        d_nee_l1.alloc(npaths);
        d_nee_l2.alloc(npaths);
        d_sray_o.alloc(2 * npaths);
        d_sray_d.alloc(2 * npaths);
        d_vis.alloc(2 * npaths);
        d_queue0.alloc(npaths);
        d_queue1.alloc(npaths);
        d_counters.alloc(crt::kNumCounters);
        d_trav_counters.alloc(4);
        path_capacity = npaths;
    }

    void initialize(int w, int h)
    {
        if (w <= 0 || h <= 0) {
            throw std::runtime_error("initialize: framebuffer dimensions must be positive");
        }
        if (aov && world_size > 1) {
            throw std::runtime_error("initialize: option aov needs the whole frame on one renderer (world_size 1); "
                                     "AOVs of multi-GPU frames are not supported");
        }
        if (dn_history && !aov) {
            throw std::runtime_error("initialize: option denoise_history needs option aov = 1 (the history is built from the "
                                     "first-hit AOVs)");
        }
        if (dn_motion && !dn_history) {
            throw std::runtime_error("initialize: option denoise_motion needs option denoise_history > 0");
        }
        if (aov && adaptive) {
            throw std::runtime_error("initialize: option aov cannot be combined with adaptive sampling (the AOVs and the "
                                     "denoiser assume the same number of samples in every pixel); turn it off with "
                                     "crtc_set_adaptive(r, NULL) first");
        }
        if (views > 1) {
            const std::string v = "initialize: option views = " + std::to_string(views) + " (crtc_render_views) ";
            if (aov) {
                throw std::runtime_error(v + "cannot be combined with option aov (AOVs and the denoiser have one view)");
            }
            if (world_size > 1) {
                throw std::runtime_error(v + "needs the whole frame on one renderer (world_size 1)");
            }
            if (adaptive) {
                throw std::runtime_error(v + "cannot be combined with adaptive sampling; turn it off with crtc_set_adaptive(r, NULL) first");
            }
        }
        make_current();
        CUDA_CHECK(cudaStreamSynchronize(stream));
        unpin_img();             // (the caller's img buffer is reallocated with the new size)
        close_peer_frame();      // the frame's shape (and on the exporting rank, its buffers) change:
        frame_exported = false;  // crtc_export_frame / crtc_import_frame must be called again
        frame_id = 0;
        sample_base = 0;
        views_active = views;
        view_frames.assign(views, 0u);
        fb_w = w;
        fb_h = h;
        ntx = crt::tiles_along(w);
        local_tiles = crt::rank_tiles(w, h, rank, world_size);
        npx_local = (uint32_t)local_tiles.size() * crt::kTilePixels;
        assemble_tiles.clear();
        d_tile_ids.upload(local_tiles.data(), local_tiles.size(), stream);
        const size_t nv = views_active;
        d_accum_local.alloc((size_t)npx_local * 3 * nv);
        d_img_local.alloc(npx_local * nv);
        d_accum_full.alloc((size_t)w * h * 3 * nv);
        d_img_full.alloc((size_t)w * h * nv + crt::kSyncWords);  // + the frame completion flags (kernels.cuh)
        if (npx_local) {
            CUDA_CHECK(cudaMemsetAsync(d_accum_local.ptr, 0, (size_t)npx_local * 3 * nv * sizeof(float), stream));
            CUDA_CHECK(cudaMemsetAsync(d_img_local.ptr, 0, (size_t)npx_local * nv * 4, stream));
        }
        CUDA_CHECK(cudaMemsetAsync(d_accum_full.ptr, 0, (size_t)w * h * 3 * nv * sizeof(float), stream));
        CUDA_CHECK(cudaMemsetAsync(d_img_full.ptr, 0, ((size_t)w * h * nv + crt::kSyncWords) * 4, stream));
        aov_active = aov;
        dn_history_active = dn_history;
        dn_motion_active = dn_motion;
        if (aov_active) {  // (drops the denoiser's history too)
            aov_state.allocate(npx_local, (size_t)w * h, stream);
        } else {
            aov_state.release();
        }
        adaptive_epoch = false;
        adaptive_state.release();  // (sized by the first adaptive wavefront)
        share_seq = 0;
        CUDA_CHECK(cudaStreamSynchronize(stream));
    }

    int builder_fallbacks = 0;  // device builds that fell back to the host builder (crtc_get_option "bvh_builder_fallbacks")

    void set_scene(const crt_scene_t *scene)
    {
        make_current();
        scene_update.reset();  // (drops staged updates too)
        lights_staged = false;
        staged_lights.clear();
        frame_id = 0;
        sample_base = 0;
        adaptive_epoch = false;
        auto_frames = 0;
        auto_decided = false;
        crt::SceneRecords rec;  // the device build fills rec.shading only
        uint32_t bvh_nodes = 0, bvh_depth = 0;
        double bvh_ms = 0.0;
        size_t num_tris = 0;
        // (the plan is cheap — reference checks and counts — and gives the triangle total before anything is allocated)
        crt::FlattenPlan plan;
        crt::plan_flatten(scene, plan);
        crt::check_triangle_count(plan.total_tris);
        std::unique_ptr<crt_host::SceneUpdate> keep(dynamic_scene ? new crt_host::SceneUpdate() : nullptr);
        std::vector<uint32_t> level_begin;
        bool built_on_device = false;
        const bool try_device = bvh_builder != 0 && plan.total_tris > 0;
        if (try_device) {
            // set_scene on the device: only the references are checked and the materials / textures converted on the host
            crt::pack_shading(scene, bvh_threads, rec.shading);
            crt_host::DeviceSceneBuild job;
            job.stream = stream;
            job.device = device;
            job.builder = bvh_builder;
            job.ploc_radius = ploc_radius;
            job.ploc_tail = ploc_tail;
            job.d_nodes = &d_nodes;
            job.d_tris = &d_tris;
            job.d_shade = &d_shade;
            job.leaf_flat_ids = &leaf_flat_ids;
            job.geometry = keep ? keep->geometry.get() : nullptr;
            try {
                job.run(scene, plan);
                built_on_device = true;
            } catch (const crt_host::DeviceBuildFailure &e) {
                // the builder gave up on this input (no PLOC progress, a tree deeper than the traversal stack, ...): the
                // host builder takes over; scene errors and CUDA errors are not caught here
                std::fprintf(stderr, "crt_cuda: %s; building the BVH on the host instead\n", e.what());
                CUDA_CHECK(cudaStreamSynchronize(stream));
                builder_fallbacks++;
            }
            if (built_on_device) {
                num_tris = plan.total_tris;
                bvh_nodes = job.num_nodes;
                bvh_depth = job.depth;
                bvh_ms = job.build_ms;
                level_begin = job.level_begin;
                build_rounds = job.rounds;
                for (int i = 0; i < 5; ++i) {
                    phase_ms[i] = job.phase_ms[i];
                }
            }
        }
        if (!built_on_device) {
            crt::pack_scene(scene, bvh_threads, rec);
            phase_ms[0] = rec.flatten_ms;
            phase_ms[1] = phase_ms[2] = phase_ms[3] = 0.0;  // the host builder reports one figure: scene_info[3]
            phase_ms[4] = rec.pack_ms;
            num_tris = rec.num_tris;
            leaf_flat_ids = std::move(rec.leaf_flat_ids);
            static_assert(sizeof(crt::Bvh8Node) == 5 * sizeof(float4), "node = 5 float4");
            d_nodes.upload(reinterpret_cast<const float4 *>(rec.bvh.nodes.data()), rec.bvh.nodes.size() * 5, stream);
            d_tris.upload(reinterpret_cast<const float4 *>(rec.tris.data()), rec.tris.size() / 4, stream);
            d_shade.upload(reinterpret_cast<const float4 *>(rec.shade.data()), rec.shade.size() * 3, stream);
            bvh_nodes = (uint32_t)rec.bvh.nodes.size();
            bvh_depth = rec.bvh.max_depth;
            bvh_ms = rec.bvh.build_seconds * 1e3;
            level_begin = rec.bvh.level_begin;
            if (keep && !try_device) {
                keep->geometry->upload(scene, plan, stream);  // (a device build that fell back has uploaded it already)
            }
        }
        if (keep) {
            keep->keep(scene, leaf_flat_ids, level_begin, stream);
        }
        const crt::ShadingRecords &sh = rec.shading;
        static_assert(sizeof(crt_material_t) == 64 && sizeof(crt_quad_light_t) == 80, "layouts");
        static_assert(sizeof(crt::TexDesc) == sizeof(crt::DevTex), "layouts");
        d_materials.upload(reinterpret_cast<const float4 *>(sh.materials.data()), sh.materials.size() * 4, stream);
        d_lights.upload(reinterpret_cast<const float4 *>(sh.lights.data()), sh.lights.size() * 5, stream);
        num_lights = (uint32_t)sh.lights.size();
        d_texels.upload(sh.texels.data(), sh.texels.size(), stream);
        d_tex.upload(reinterpret_cast<const crt::DevTex *>(sh.tex_desc.data()), sh.tex_desc.size(), stream);
        CUDA_CHECK(cudaStreamSynchronize(stream));  // (rec is the staging memory of every upload above)
        build_hw_textures(scene);
        spp = sh.spp;
        have_scene = true;
        scene_info[0] = (double)num_tris;
        scene_info[1] = (double)bvh_nodes;
        scene_info[2] = (double)bvh_depth;
        scene_info[3] = bvh_ms;
        scene_info[4] = (double)bvh_nodes * 80.0;
        scene_info[5] = (double)num_tris * 48.0;
        for (int i = 0; i < 5; ++i) {
            scene_info[6 + i] = phase_ms[i];
        }
        scene_info[11] = (bvh_builder == 1 && built_on_device) ? (double)build_rounds : 0.0;
        view_frames.assign(views_active, 0u);
        if (npx_local) {
            CUDA_CHECK(cudaMemsetAsync(d_accum_local.ptr, 0, (size_t)npx_local * 3 * views_active * sizeof(float), stream));
            if (aov_active) {
                CUDA_CHECK(cudaMemsetAsync(aov_state.local.ptr, 0, (size_t)npx_local * crt::kAovFloats * sizeof(float), stream));
            }
        }
        aov_state.drop_history();  // (a history of another scene does not reproject)
        ++geometry_version;
        scene_update = std::move(keep);
    }

    // ---- scene updates (include/crt_cuda.h: crtc_update_instances ... crtc_commit_scene) ----
    crt_host::SceneUpdate &require_dynamic(const char *what)
    {
        require_scene();
        if (!scene_update) {
            throw std::runtime_error(std::string(what) + ": needs option dynamic_scene = 1 at the last crtc_set_scene");
        }
        return *scene_update;
    }
    void update_lights(const crt_quad_light_t *lights, uint32_t n)
    {
        require_scene();
        if (n == 0) {
            throw std::runtime_error("crtc_update_lights: no lights (the path tracer samples exactly one quad light per bounce)");
        }
        if (!lights) {
            throw std::runtime_error("crtc_update_lights: lights is NULL");
        }
        staged_lights.assign(lights, lights + n);
        lights_staged = true;
    }
    // Stream-ordered: frames enqueued before see the old scene, frames enqueued after the new one. Resets the
    // accumulation as camera_changed does and drops the denoiser's history (kept with option denoise_motion unless
    // lights change); nothing staged = nothing happens.
    void commit_scene()
    {
        require_scene();
        const bool geometry = scene_update && scene_update->staged(), lights = lights_staged;
        if (!geometry && !lights) {
            return;
        }
        make_current();
        if (geometry) {
            scene_update->commit(d_nodes.ptr, d_tris.ptr, d_shade.ptr, stream, device);
        }
        if (lights_staged) {
            const size_t n4 = staged_lights.size() * 5;
            if (n4 > d_lights.count) {
                CUDA_CHECK(cudaStreamSynchronize(stream));  // (frames in flight read the old buffer)
                d_lights.alloc(n4);
            }
            CUDA_CHECK(cudaMemcpyAsync(d_lights.ptr, staged_lights.data(), staged_lights.size() * sizeof(crt_quad_light_t),
                                       cudaMemcpyHostToDevice, stream));
            num_lights = (uint32_t)staged_lights.size();
            lights_staged = false;
        }
        CUDA_CHECK(cudaGetLastError());
        if (geometry) {
            ++geometry_version;
        }
        if (lights || !motion_frames()) {
            aov_state.drop_history();  // (new lights change the radiance everywhere; without motion, nothing reprojects)
            sample_base = 0;
        } else {
            sample_base += frame_id;
        }
        frame_id = 0;  // as camera_changed: accum, AOVs and the adaptive block counts restart
        view_frames.assign(views_active, 0u);
        adaptive_epoch = false;
        if (!auto_decided) {
            auto_frames = 0;  // an undecided any_far_first trial restarts
        }
    }

    // Enqueues one frame on the stream (no host synchronisation) and returns its record.
    // `num_frames` consecutive frames are rendered as ONE wavefront (their samples are in flight
    // together) and folded into the running mean in order — bit-identical to num_frames calls.
    FrameRecord &enqueue_frame(const float *pos, const float *dir, const float *up, float fovy, bool camera_changed,
                               uint32_t num_frames = 1, bool blocking = false)
    {
        if (num_frames < 1 || num_frames > 64) {
            throw std::runtime_error("render: num_frames must be in [1, 64]");
        }
        if (fb_w == 0) {
            throw std::runtime_error("render: initialize() has not been called");
        }
        if (!have_scene) {
            throw std::runtime_error("render: set_scene() has not been called");
        }
        make_current();
        if (camera_changed) {
            if (frame_id != 0) {  // (right after a commit, the commit's epoch goes on)
                sample_base = 0;
            }
            frame_id = 0;  // render_embree.cpp:145-147
            adaptive_epoch = false;
        }
        const crt::ViewParams view = crt::make_view_params(pos, dir, up, fovy, fb_w, fb_h, sample_base + frame_id);
        if (frame_id == 0) {  // the first frame since a reset starts a new epoch (crtc_denoise's history)
            ++epoch;
            epoch_view = view;
        }
        const size_t npaths = (size_t)npx_local * spp * num_frames;
        if (npaths >= 0x7fffffffull) {
            throw std::runtime_error("render: more than 2^31 paths in flight on one device");
        }
        ensure_path_buffers(npaths);
        frame_far_first = pick_far_first(blocking);
        const crt::DeviceScene sc = device_scene();
        crt::FrameLayout fl = frame_layout();
        fl.frames = num_frames;
        const crt::PathState ps = path_state();
        FrameRecord &rec = new_record();

        const bool shared_dst = frame_exported && world_size > 1, shared_src = peer_accum_full != nullptr && !frame_exported;
        if (shared_dst || shared_src) {
            ensure_sync_state();
        }
        rec.mark(stream, -1);
        if (shared_dst && share_seq > 0) {
            // starting the next wavefront: the assembling rank is done with the previous frame, peers may overwrite it
            crt::k_set_word<<<1, 32, 0, stream>>>(sync_words() + crt::kSyncConsumed, share_seq);
        }
        zero_counters();
        // adaptive sampling: which blocks render how many of this wavefront's frames, decided once per call
        const bool adaptive_frame = adaptive || adaptive_epoch;
        crt::AdaptiveSelect sel{};
        if (adaptive_frame) {
            sel.reset = adaptive_epoch ? 0u : 1u;
            if (!adaptive_epoch) {
                adaptive_epoch = true;
                adaptive_base = frame_id;
                adaptive_state.ensure(npx_local);
            }
            sel.frames = num_frames;
            sel.stat_base = adaptive_base;
            // The any_far_first trial compares the traversal times of two blocking frames, which must see the same work.
            sel.all_active = (!adaptive || (any_far_first == 2 && !auto_decided && blocking)) ? 1u : 0u;
            if (adaptive) {
                sel.threshold = adaptive_params.threshold;
                sel.min_frames = adaptive_params.min_frames;
                sel.max_frames = adaptive_params.max_frames;
            }
        }
        const crt::AdaptiveFrame ad = adaptive_state.frame(adaptive_base);
        if (npaths) {
            const unsigned g256 = (unsigned)((npaths + 255) / 256);
            if (adaptive_frame) {  // (its time counts as raygen)
                adaptive_state.select(fl, sel, stream);
                rec.launches += 1;
                adaptive_state.raygen(g256, view, fl, ps, ad, stream);
            } else {
                crt::k_raygen<<<g256, 256, 0, stream>>>(view, fl, ps);
            }
            rec.mark(stream, kStRaygen);
            launch_primary(sc, ps, rec);
            if (aov_active) {  // (its time counts as shading: the next mark closes the stage)
                aov_state.launch_primary(sc, fl, ps, frame_id, stream);
                rec.launches += 1;
                if (frame_id == 0 && motion_frames()) {  // (the same)
                    aov_state.launch_hit(fl, ps, stream);
                    rec.launches += 1;
                }
            }
            launch_bounces(sc, ps, npaths, rec);
            const unsigned gpx = (unsigned)((npx_local + 255) / 256);
            // where the resolved pixels also go as a full row-major frame: this renderer's own full frame (single
            // GPU, or the assembling rank of a peer-written frame), the assembling rank's full frame over NVLink
            // (crtc_import_frame), or nowhere (tiles are gathered afterwards: crtc_local_buffers)
            float *full_accum = nullptr;
            uint32_t *full_img = nullptr;
            if (world_size == 1 || frame_exported) {
                full_accum = d_accum_full.ptr;
                full_img = d_img_full.ptr;
            } else if (peer_accum_full) {
                full_accum = peer_accum_full;
                full_img = peer_img_full;
            }
            uint32_t *arrive = nullptr;
            if (shared_src) {
                if (share_seq > 0) {  // not before the assembling rank is done with the frame this one overwrites
                    crt::k_wait_words<<<1, 32, 0, stream>>>(peer_sync_words() + crt::kSyncConsumed, 1u, 0xffffffffu, share_seq, d_sync_err);
                }
                arrive = peer_sync_words() + rank;
            }
            if (adaptive_frame) {  // (only active pixels are stored into a shared frame: it holds the others already)
                adaptive_state.resolve(gpx, fl, ps, frame_id, d_accum_local.ptr, d_img_local.ptr, full_accum, full_img,
                                       d_done_counter.ptr, arrive, share_seq + 1u, ad, stream);
            } else {
                crt::k_resolve<<<gpx, 256, 0, stream>>>(fl, ps, frame_id, d_accum_local.ptr, d_img_local.ptr, full_accum, full_img,
                                                       d_done_counter.ptr, arrive, share_seq + 1u);
            }
            rec.launches += 1;
            if (aov_active) {  // (counted in the resolve stage)
                aov_state.launch_moments(fl, ps, frame_id, stream);
                rec.launches += 1;
            }
            rec.mark(stream, kStResolve);
        } else if (shared_src) {
            // a rank that owns no tile of this frame (more ranks than tiles) still has to say "done"
            crt::k_set_word<<<1, 32, 0, stream>>>(peer_sync_words() + rank, share_seq + 1u);
        }
        finish_record(rec, num_frames);
        frame_id += num_frames;
        if (shared_dst || shared_src) {
            ++share_seq;
        }
        return rec;
    }

    // ---- the parts of a wavefront that do not depend on its cameras (enqueue_frame, enqueue_views) ----
    FrameRecord &new_record()
    {
        if (record_pool.empty()) {
            record_pool.emplace_back(new FrameRecord());
        }
        in_flight.push_back(std::move(record_pool.back()));
        record_pool.pop_back();
        FrameRecord &rec = *in_flight.back();
        rec.num_events = 0;
        rec.launches = 0;
        rec.all_stages = stage_events || (any_far_first == 2 && !auto_decided);  // (the shadow-order trial reads the traversal stage)
        return rec;
    }
    void zero_counters()
    {
        CUDA_CHECK(cudaMemsetAsync(d_counters.ptr, 0, crt::kNumCounters * sizeof(uint32_t), stream));
        if (count_traversal) {
            CUDA_CHECK(cudaMemsetAsync(d_trav_counters.ptr, 0, 4 * sizeof(unsigned long long), stream));
        }
    }
    // closest hit of the primary rays (the raygen launch is counted here too)
    void launch_primary(const crt::DeviceScene &sc, const crt::PathState &ps, FrameRecord &rec)
    {
        launch_traverse(sc, ps, ps.queue[0], ps.counters + crt::kCntQueue, nullptr, ps.counters + crt::kCntWork);
        rec.mark(stream, kStPrimary);
        rec.launches += 2;
    }
    // per bounce: shade -> one traversal launch for this bounce's shadow rays AND the next bounce's continuation rays
    // -> NEE resolve
    void launch_bounces(const crt::DeviceScene &sc, const crt::PathState &ps, size_t npaths, FrameRecord &rec)
    {
        // k_nee_resolve strides over its queue: two waves of resident blocks cover any queue length
        if (num_sms == 0) {
            CUDA_CHECK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, device));
        }
        const unsigned g128 = (unsigned)((npaths + 127) / 128);
        const unsigned g_nee = (unsigned)std::min<size_t>((npaths + 255) / 256, (size_t)num_sms * 8 * 2);
        for (int b = 0; b < max_depth; ++b) {
            const uint32_t *qin = ps.queue[b & 1];
            uint32_t *qout = ps.queue[(b + 1) & 1];
            if (shade_sort == 2 || (shade_sort == 1 && b > 0)) {
                // (its time counts as shading: the next mark closes the stage)
                rec.launches += sort_shade_queue(sc, ps, qin, b, npaths);
                qin = d_queue_sorted.ptr;
            }
            if (sc.tex_objects) {
                crt::k_shade<true><<<g128, 128, 0, stream>>>(sc, ps, qin, qout, b, max_depth);
            } else {
                crt::k_shade<false><<<g128, 128, 0, stream>>>(sc, ps, qin, qout, b, max_depth);
            }
            rec.mark(stream, kStShade);
            const bool last = b + 1 == max_depth;
            launch_traverse(sc, ps, qout, last ? nullptr : ps.counters + crt::kCntQueue + b + 1,
                            ps.counters + crt::kCntShadow + b, ps.counters + crt::kCntWork + 1 + b);
            rec.mark(stream, kStTraverse);
            crt::k_nee_resolve<<<g_nee, 256, 0, stream>>>(ps, qin, b);
            rec.mark(stream, kStNee);
            rec.launches += 3;
        }
    }
    void finish_record(FrameRecord &rec, uint32_t num_frames)
    {
        CUDA_CHECK(cudaMemcpyAsync(rec.h_counters, d_counters.ptr, crt::kNumCounters * sizeof(uint32_t),
                                   cudaMemcpyDeviceToHost, stream));
        if (count_traversal) {
            CUDA_CHECK(cudaMemcpyAsync(rec.h_trav, d_trav_counters.ptr, 4 * sizeof(unsigned long long),
                                       cudaMemcpyDeviceToHost, stream));
        }
        CUDA_CHECK(cudaGetLastError());
        rec.frames = num_frames;
    }

    // crtc_render_views: `num_frames` frames of every view as ONE wavefront (kernels.cuh: k_raygen_views, k_resolve_views);
    // view k is seeded and folded with its own frame counter, so it ends bit-identical to a one-view renderer's frame.
    // With one view this is crtc_render_async.
    void enqueue_views(const crtc_view_t *vs, uint32_t num_views, uint32_t num_frames)
    {
        if (!vs) {
            throw std::runtime_error("crtc_render_views: views is NULL");
        }
        if (num_views != views_active) {
            throw std::runtime_error("crtc_render_views: num_views = " + std::to_string(num_views) + " differs from option views = " +
                                     std::to_string(views_active) + " of the last crtc_initialize");
        }
        if (views_active == 1) {
            enqueue_frame(vs[0].pos, vs[0].dir, vs[0].up, vs[0].fovy, vs[0].camera_changed != 0, num_frames);
            return;
        }
        if (num_frames < 1 || num_frames > 64) {
            throw std::runtime_error("crtc_render_views: num_frames must be in [1, 64]");
        }
        if (!have_scene) {
            throw std::runtime_error("crtc_render_views: set_scene() has not been called");
        }
        const size_t npaths = (size_t)npx_local * spp * num_frames * num_views;
        if (npaths >= 0x7fffffffull) {
            throw std::runtime_error("crtc_render_views: more than 2^31 paths in flight on one device (views x num_frames x spp x "
                                     "64x64-padded pixels)");
        }
        make_current();
        crt::ViewTable table{};
        table.num_views = num_views;
        for (uint32_t k = 0; k < num_views; ++k) {
            if (vs[k].camera_changed) {
                view_frames[k] = 0;
            }
            table.view[k] = crt::make_view_params(vs[k].pos, vs[k].dir, vs[k].up, vs[k].fovy, fb_w, fb_h, view_frames[k]);
        }
        ensure_path_buffers(npaths);
        frame_far_first = pick_far_first(false);
        const crt::DeviceScene sc = device_scene();
        crt::FrameLayout fl = frame_layout();
        fl.frames = num_frames;
        const crt::PathState ps = path_state();
        FrameRecord &rec = new_record();
        rec.mark(stream, -1);
        zero_counters();
        crt_host::launch(crt::k_raygen_views, (unsigned)((npaths + 255) / 256), 256, stream, table, fl, ps);
        rec.mark(stream, kStRaygen);
        launch_primary(sc, ps, rec);
        launch_bounces(sc, ps, npaths, rec);
        crt_host::launch(crt::k_resolve_views, (unsigned)(((size_t)npx_local * num_views + 255) / 256), 256, stream, table, fl, ps,
                         d_accum_local.ptr, d_img_local.ptr, d_accum_full.ptr, d_img_full.ptr);
        rec.launches += 1;
        rec.mark(stream, kStResolve);
        finish_record(rec, num_frames);
        for (uint32_t k = 0; k < num_views; ++k) {
            view_frames[k] += num_frames;
        }
    }

    void read_view(uint32_t view, float *rgb_out, uint32_t *img_out)
    {
        if (fb_w == 0) {
            throw std::runtime_error("crtc_read_view: initialize() has not been called");
        }
        if (view >= views_active) {
            throw std::runtime_error("crtc_read_view: view " + std::to_string(view) + " is out of range (option views = " +
                                     std::to_string(views_active) + " at the last crtc_initialize)");
        }
        make_current();
        frame_wait();  // (a shared one-view frame: every rank's tiles first; no-op otherwise)
        const size_t n = (size_t)fb_w * fb_h;
        if (rgb_out) {
            CUDA_CHECK(cudaMemcpyAsync(rgb_out, d_accum_full.ptr + view * n * 3, n * 3 * sizeof(float), cudaMemcpyDeviceToHost, stream));
        }
        if (img_out) {
            CUDA_CHECK(cudaMemcpyAsync(img_out, d_img_full.ptr + view * n, n * 4, cudaMemcpyDeviceToHost, stream));
        }
        CUDA_CHECK(cudaStreamSynchronize(stream));
        CUDA_CHECK(cudaGetLastError());
        check_sync_error();
    }

    // After a stream synchronisation: folds every in-flight frame's events and counters into
    // `stage_sum` / `counter_sum` (both optional) and leaves the last frame's values in
    // stage_ms / counters_out. Returns the number of frames collected.
    uint32_t collect(float *stage_sum, uint64_t *counter_sum)
    {
        uint32_t n = 0;
        for (auto &recp : in_flight) {
            FrameRecord &rec = *recp;
            for (int s = 0; s < kNumStages; ++s) {
                stage_ms[s] = 0.f;
            }
            for (size_t i = 1; rec.all_stages && i < rec.num_events; ++i) {
                float ms = 0.f;
                CUDA_CHECK(cudaEventElapsedTime(&ms, rec.events[i - 1], rec.events[i]));
                stage_ms[rec.event_stage[i]] += ms;
            }
            if (rec.num_events > 1) {
                CUDA_CHECK(cudaEventElapsedTime(&stage_ms[kStFrame], rec.events[0], rec.events[rec.num_events - 1]));
            }
            uint64_t closest = 0, shadow = 0;
            for (int b = 0; b < max_depth; ++b) {
                closest += rec.h_counters[crt::kCntQueue + b];
                shadow += rec.h_counters[crt::kCntShadow + b];
            }
            counters_out[0] = closest;
            counters_out[1] = shadow;
            counters_out[2] = rec.launches;
            counters_out[3] = count_traversal ? rec.h_trav[0] : 0;
            counters_out[4] = count_traversal ? rec.h_trav[1] : 0;
            counters_out[5] = rec.h_counters[crt::kCntQueue];
            counters_out[6] = count_traversal ? rec.h_trav[2] : 0;
            counters_out[7] = count_traversal ? rec.h_trav[3] : 0;
            for (int s = 0; stage_sum && s < kNumStages; ++s) {
                stage_sum[s] += stage_ms[s];
            }
            for (int k = 0; counter_sum && k < 8; ++k) {
                counter_sum[k] += counters_out[k];
            }
            n += rec.frames;
        }
        for (auto &recp : in_flight) {
            record_pool.push_back(std::move(recp));
        }
        in_flight.clear();
        return n;
    }

    // RenderBackend::render: enqueue, wait, collect (+ optional readback of img).
    void render(const float *pos, const float *dir, const float *up, float fovy, bool camera_changed, bool readback,
                uint32_t *img, crt_render_stats_t *stats)
    {
        enqueue_frame(pos, dir, up, fovy, camera_changed, 1, true);
        if (readback && img && world_size == 1) {
            pin_img(img, (size_t)fb_w * fb_h * 4);
            CUDA_CHECK(cudaMemcpyAsync(img, d_img_full.ptr, (size_t)fb_w * fb_h * 4, cudaMemcpyDeviceToHost, stream));
        }
        CUDA_CHECK(cudaStreamSynchronize(stream));
        CUDA_CHECK(cudaGetLastError());
        check_sync_error();
        collect(nullptr, nullptr);
        auto_tune_step();
        if (stats) {
            const uint64_t rays = counters_out[0] + counters_out[1];
            stats->render_time = stage_ms[kStFrame];
            stats->num_rays = rays;
            stats->rays_per_second =
                stage_ms[kStFrame] > 0.f ? (float)((double)rays / (stage_ms[kStFrame] * 1.0e-3)) : 0.f;
        }
    }

    // crtc_sync: waits for every frame enqueued with crtc_render_async and returns their totals.
    uint32_t sync_frames(crt_render_stats_t *total, float *stage_sum, uint64_t *counter_sum)
    {
        make_current();
        CUDA_CHECK(cudaStreamSynchronize(stream));
        CUDA_CHECK(cudaGetLastError());
        check_sync_error();
        float ssum[kNumStages] = {0};
        uint64_t csum[8] = {0};
        const uint32_t n = collect(ssum, csum);
        if (total) {
            total->render_time = ssum[kStFrame];
            total->num_rays = csum[0] + csum[1];
            total->rays_per_second = ssum[kStFrame] > 0.f ? (float)((double)total->num_rays / (ssum[kStFrame] * 1.0e-3)) : 0.f;
        }
        for (int s = 0; stage_sum && s < kNumStages; ++s) {
            stage_sum[s] = ssum[s];
        }
        for (int k = 0; counter_sum && k < 8; ++k) {
            counter_sum[k] = csum[k];
        }
        return n;
    }

    // ---- kernel-level access ----
    void upload_rays(const float *rays, uint64_t n)
    {
        ensure_path_buffers(std::max<size_t>(n, path_capacity));
        std::vector<float4> o(n), d(n);
        for (uint64_t i = 0; i < n; ++i) {
            o[i] = make_float4(rays[8 * i], rays[8 * i + 1], rays[8 * i + 2], rays[8 * i + 3]);
            d[i] = make_float4(rays[8 * i + 4], rays[8 * i + 5], rays[8 * i + 6], rays[8 * i + 7]);
        }
        CUDA_CHECK(cudaMemcpyAsync(d_ray_o.ptr, o.data(), n * sizeof(float4), cudaMemcpyHostToDevice, stream));
        CUDA_CHECK(cudaMemcpyAsync(d_ray_d.ptr, d.data(), n * sizeof(float4), cudaMemcpyHostToDevice, stream));
        const uint32_t cnt = (uint32_t)n;
        CUDA_CHECK(cudaMemcpyAsync(d_counters.ptr, &cnt, 4, cudaMemcpyHostToDevice, stream));
        CUDA_CHECK(cudaStreamSynchronize(stream));
    }

    void launch_closest(uint64_t)
    {
        CUDA_CHECK(cudaMemsetAsync(d_counters.ptr + crt::kCntWork, 0, sizeof(uint32_t), stream));
        launch_traverse(device_scene(), path_state(), nullptr, d_counters.ptr, nullptr, d_counters.ptr + crt::kCntWork);
    }

    // shadow-ray layout for the any-hit kernel: sray_o = org|tfar, sray_d = dir|bits(index)
    void stage_any(uint64_t n, const float *rays)
    {
        std::vector<float4> o(n), d(n);
        for (uint64_t i = 0; i < n; ++i) {
            o[i] = make_float4(rays[8 * i], rays[8 * i + 1], rays[8 * i + 2], rays[8 * i + 7]);
            uint32_t idx = (uint32_t)i;
            float fi;
            std::memcpy(&fi, &idx, 4);
            d[i] = make_float4(rays[8 * i + 4], rays[8 * i + 5], rays[8 * i + 6], fi);
        }
        CUDA_CHECK(cudaMemcpyAsync(d_sray_o.ptr, o.data(), n * sizeof(float4), cudaMemcpyHostToDevice, stream));
        CUDA_CHECK(cudaMemcpyAsync(d_sray_d.ptr, d.data(), n * sizeof(float4), cudaMemcpyHostToDevice, stream));
        const uint32_t cnt = (uint32_t)n;
        CUDA_CHECK(cudaMemcpyAsync(d_counters.ptr, &cnt, 4, cudaMemcpyHostToDevice, stream));
        CUDA_CHECK(cudaStreamSynchronize(stream));
    }

    void launch_any(uint64_t)
    {
        CUDA_CHECK(cudaMemsetAsync(d_counters.ptr + crt::kCntWork, 0, sizeof(uint32_t), stream));
        launch_traverse(device_scene(), path_state(), nullptr, nullptr, d_counters.ptr, d_counters.ptr + crt::kCntWork);
    }

    void require_scene() const
    {
        if (!have_scene) {
            throw std::runtime_error("set_scene() has not been called");
        }
    }

    void trace_closest(const float *rays, uint64_t n, float *hits)
    {
        require_scene();
        make_current();
        if (n == 0) {
            return;
        }
        if (n > 0x3fffffffull) {
            throw std::runtime_error("trace_closest: too many rays in one batch");
        }
        upload_rays(rays, n);
        launch_closest(n);
        std::vector<float4> h(n);
        CUDA_CHECK(cudaMemcpyAsync(h.data(), d_hit.ptr, n * sizeof(float4), cudaMemcpyDeviceToHost, stream));
        CUDA_CHECK(cudaStreamSynchronize(stream));
        CUDA_CHECK(cudaGetLastError());
        for (uint64_t i = 0; i < n; ++i) {
            uint32_t tri;
            std::memcpy(&tri, &h[i].w, 4);
            const uint32_t flat = tri == crt::kMiss ? crt::kMiss : leaf_flat_ids[tri];
            hits[4 * i] = h[i].x;
            hits[4 * i + 1] = h[i].y;
            hits[4 * i + 2] = h[i].z;
            std::memcpy(&hits[4 * i + 3], &flat, 4);
        }
    }

    void trace_any(const float *rays, uint64_t n, uint8_t *occluded)
    {
        require_scene();
        make_current();
        if (n == 0) {
            return;
        }
        if (n > 0x3fffffffull) {
            throw std::runtime_error("trace_any: too many rays in one batch");
        }
        // The any-hit kernel starts every ray at tnear = kEpsilon, like the renderer's shadow rays. A ray with any other
        // tnear goes through the closest-hit kernel instead: over the same triangle test, "occluded" is "a hit was found".
        std::vector<float> any_rays, closest_rays;
        std::vector<uint64_t> any_index, closest_index;
        for (uint64_t i = 0; i < n; ++i) {
            const bool any_kernel = rays[8 * i + 3] == crt::kEpsilon;
            std::vector<float> &dst = any_kernel ? any_rays : closest_rays;
            dst.insert(dst.end(), rays + 8 * i, rays + 8 * i + 8);
            (any_kernel ? any_index : closest_index).push_back(i);
        }
        if (!any_index.empty()) {
            const uint64_t m = any_index.size();
            ensure_path_buffers(std::max<size_t>((m + 1) / 2, path_capacity));
            stage_any(m, any_rays.data());
            launch_any(m);
            std::vector<uint8_t> vis(m);
            CUDA_CHECK(cudaMemcpyAsync(vis.data(), d_vis.ptr, m, cudaMemcpyDeviceToHost, stream));
            CUDA_CHECK(cudaStreamSynchronize(stream));
            CUDA_CHECK(cudaGetLastError());
            for (uint64_t j = 0; j < m; ++j) {
                occluded[any_index[j]] = vis[j] ? 0 : 1;
            }
        }
        if (!closest_index.empty()) {
            std::vector<float> hits(4 * closest_index.size());
            trace_closest(closest_rays.data(), closest_index.size(), hits.data());
            for (uint64_t j = 0; j < closest_index.size(); ++j) {
                uint32_t flat;
                std::memcpy(&flat, &hits[4 * j + 3], 4);
                occluded[closest_index[j]] = flat != crt::kMiss ? 1 : 0;
            }
        }
    }

    float bench_trace(const float *rays, uint64_t n, bool any_hit, int iters)
    {
        require_scene();
        make_current();
        if (n == 0 || iters <= 0) {
            return 0.f;
        }
        if (any_hit) {
            ensure_path_buffers(std::max<size_t>((n + 1) / 2, path_capacity));
            stage_any(n, rays);
        } else {
            upload_rays(rays, n);
        }
        cudaEvent_t e0, e1;
        CUDA_CHECK(cudaEventCreate(&e0));
        CUDA_CHECK(cudaEventCreate(&e1));
        for (int w = 0; w < 3; ++w) {
            any_hit ? launch_any(n) : launch_closest(n);
        }
        CUDA_CHECK(cudaStreamSynchronize(stream));
        CUDA_CHECK(cudaEventRecord(e0, stream));
        for (int i = 0; i < iters; ++i) {
            any_hit ? launch_any(n) : launch_closest(n);
        }
        CUDA_CHECK(cudaEventRecord(e1, stream));
        CUDA_CHECK(cudaStreamSynchronize(stream));
        CUDA_CHECK(cudaGetLastError());
        float ms = 0.f;
        CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
        cudaEventDestroy(e0);
        cudaEventDestroy(e1);
        return ms / iters;
    }

    void read_aov(float *out)
    {
        require_aov_frame("crtc_read_aov");
        make_current();
        CUDA_CHECK(cudaMemcpyAsync(out, aov_state.full.ptr, (size_t)fb_w * fb_h * crt::kAovFloats * sizeof(float),
                                   cudaMemcpyDeviceToHost, stream));
        CUDA_CHECK(cudaStreamSynchronize(stream));
        CUDA_CHECK(cudaGetLastError());
    }

    void read_denoise_history(float *out)
    {
        if (!dn_history_active) {
            throw std::runtime_error("crtc_read_denoise_history: option denoise_history is off (set it before crtc_initialize)");
        }
        const float *cur = aov_state.history_of(epoch);
        if (!cur || frame_id == 0) {
            throw std::runtime_error("crtc_read_denoise_history: no crtc_denoise since the last reset");
        }
        make_current();
        CUDA_CHECK(cudaMemcpyAsync(out, cur, (size_t)fb_w * fb_h * crt::kHistFloats * sizeof(float), cudaMemcpyDeviceToHost,
                                   stream));
        CUDA_CHECK(cudaStreamSynchronize(stream));
        CUDA_CHECK(cudaGetLastError());
    }

    void denoise(const crtc_denoise_params_t *params, float *rgb_out, uint32_t *img_out, void *cuda_array)
    {
        crt::DenoiseParams p;
        if (params) {
            if (params->iterations < 1 || params->iterations > 10) {
                throw std::runtime_error("crtc_denoise: iterations must be in [1, 10]");
            }
            const float s[3] = {params->sigma_luminance, params->sigma_normal, params->sigma_depth};
            for (float v : s) {
                if (!std::isfinite(v) || !(v > 0.f)) {
                    throw std::runtime_error("crtc_denoise: sigma_luminance, sigma_normal and sigma_depth must be finite and > 0");
                }
            }
            p.iterations = params->iterations;
            p.sigma_l = s[0];
            p.sigma_n = s[1];
            p.sigma_z = s[2];
        }
        require_aov_frame("crtc_denoise");
        make_current();
        crt::LiveGeometry live{};
        if (motion_frames()) {
            const crt_host::SceneGeometry &g = *scene_update->geometry;
            live = crt::LiveGeometry{g.segs.ptr, g.num_segs, scene_update->leaf_flat_ids.ptr, g.index_arena.ptr, g.uv_arena.ptr,
                                     g.xforms.ptr, g.vert_arena.ptr, g.xf.size(), g.vert_floats};
        }
        aov_state.denoise(fb_w, fb_h, (float)spp * (float)frame_id, d_accum_full.ptr, p, dn_history_active, epoch, epoch_view,
                          geometry_version, motion_frames() ? &live : nullptr, stream);
        const size_t n = (size_t)fb_w * fb_h;
        if (rgb_out) {
            CUDA_CHECK(cudaMemcpyAsync(rgb_out, aov_state.dn_rgb.ptr, n * 3 * sizeof(float), cudaMemcpyDeviceToHost, stream));
        }
        if (img_out) {
            CUDA_CHECK(cudaMemcpyAsync(img_out, aov_state.dn_img.ptr, n * 4, cudaMemcpyDeviceToHost, stream));
        }
        if (cuda_array) {
            CUDA_CHECK(cudaMemcpy2DToArrayAsync(static_cast<cudaArray_t>(cuda_array), 0, 0, aov_state.dn_img.ptr, (size_t)fb_w * 4,
                                                (size_t)fb_w * 4, (size_t)fb_h, cudaMemcpyDeviceToDevice, stream));
        }
        CUDA_CHECK(cudaStreamSynchronize(stream));
        CUDA_CHECK(cudaGetLastError());
    }

    // tile-id lists of the other ranks, cached on the device (keyed by world_size * 4096 + rank)
    std::vector<std::pair<int, std::unique_ptr<DeviceBuffer<uint32_t>>>> assemble_tiles;

    // Stream-ordered (no host synchronisation): the caller orders it after the gather.
    void assemble_rank(int src_rank, int ws, const void *accum_dev, const void *img_dev)
    {
        make_current();
        const int key = ws * 4096 + src_rank;
        DeviceBuffer<uint32_t> *d_tiles = nullptr;
        for (auto &e : assemble_tiles) {
            if (e.first == key) {
                d_tiles = e.second.get();
            }
        }
        if (!d_tiles) {
            const std::vector<uint32_t> tiles = crt::rank_tiles(fb_w, fb_h, src_rank, ws);
            assemble_tiles.emplace_back(key, std::make_unique<DeviceBuffer<uint32_t>>());
            d_tiles = assemble_tiles.back().second.get();
            d_tiles->upload(tiles.data(), tiles.size(), stream);
            CUDA_CHECK(cudaStreamSynchronize(stream));  // `tiles` is a host temporary
        }
        if (d_tiles->count == 0) {
            return;
        }
        crt::FrameLayout f = frame_layout();
        f.tile_ids = d_tiles->ptr;
        f.npx_local = (uint32_t)d_tiles->count * crt::kTilePixels;
        const unsigned g = (unsigned)((f.npx_local + 255) / 256);
        crt::k_assemble<<<g, 256, 0, stream>>>(f, static_cast<const float *>(accum_dev),
                                              static_cast<const uint32_t *>(img_dev), d_accum_full.ptr, d_img_full.ptr);
        CUDA_CHECK(cudaGetLastError());
    }
};

// ---------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------
static void require_renderer(const crtc_renderer *r)
{
    if (!r) {
        throw std::runtime_error("renderer handle is NULL");
    }
}

#define CRTC_TRY(body)                      \
    try {                                   \
        body;                               \
        return 0;                           \
    } catch (const std::exception &e) {     \
        g_last_error = e.what();            \
        return 1;                           \
    } catch (...) {                         \
        g_last_error = "unknown exception"; \
        return 1;                           \
    }

extern "C" {

const char *crtc_last_error(void)
{
    return g_last_error.c_str();
}

const char *crtc_name(void)
{
    return "CUDA wavefront (H100, BVH8)";
}

int crtc_create(crtc_renderer **out, int device)
{
    CRTC_TRY({
        if (!out) {
            throw std::runtime_error("crtc_create: out is NULL");
        }
        *out = nullptr;
        int n = 0;
        cudaError_t err = cudaGetDeviceCount(&n);
        if (err != cudaSuccess || n == 0) {
            throw std::runtime_error(std::string("crtc_create: no usable CUDA device (") +
                                     (err != cudaSuccess ? cudaGetErrorString(err) : "device count is 0") +
                                     "); this backend has no CPU fallback");
        }
        if (device < 0 || device >= n) {
            throw std::runtime_error("crtc_create: device ordinal out of range");
        }
        std::unique_ptr<crtc_renderer> r(new crtc_renderer());
        r->device = device;
        r->make_current();
        CUDA_CHECK(cudaStreamCreateWithFlags(&r->own_stream, cudaStreamNonBlocking));
        r->stream = r->own_stream;
        *out = r.release();
    })
}

void crtc_destroy(crtc_renderer *r)
{
    if (r) {
        cudaSetDevice(r->device);
        delete r;
    }
}

int crtc_set_option(crtc_renderer *r, const char *key, int64_t value)
{
    CRTC_TRY({ require_renderer(r);
        const std::string k = key ? key : "";
        if (k == "max_depth") {
            if (value < 1 || value > crt::kMaxDepthSupported) {
                throw std::runtime_error("max_depth must be in [1, 16]");
            }
            r->max_depth = (int)value;
        } else if (k == "rank") {
            r->rank = (int)value;
        } else if (k == "world_size") {
            if (value < 1) {
                throw std::runtime_error("world_size must be >= 1");
            }
            r->world_size = (int)value;
        } else if (k == "bvh_threads") {
            r->bvh_threads = (int)value;
        } else if (k == "tri_pass_defer") {
            if (value != 0 && value != 16 && value != 24) {
                throw std::runtime_error("tri_pass_defer must be 0, 16 or 24");
            }
            r->tri_pass_defer = (int)value;
        } else if (k == "shade_sort") {
            if (value < 0 || value > 2) {
                throw std::runtime_error("shade_sort must be 0, 1 or 2");
            }
            r->shade_sort = (int)value;
        } else if (k == "hw_textures") {
            r->hw_textures = value != 0;  // takes effect at the next crtc_set_scene
        } else if (k == "stage_events") {
            r->stage_events = value != 0;
        } else if (k == "bvh_top_smem") {
            r->bvh_top_smem = value != 0;
        } else if (k == "pin_host_buffers") {
            r->pin_host_buffers = value != 0;
            if (!r->pin_host_buffers) {
                r->unpin_img();
            }
        } else if (k == "pin_read_img") {
            r->pin_repeated_reads = value != 0;
        } else if (k == "bvh_ploc_tail") {
            r->ploc_tail = value != 0;
        } else if (k == "bvh_ploc_radius") {
            if (value < 1 || value > crt::kPlocMaxRadius) {
                throw std::runtime_error("bvh_ploc_radius must be in [1, 32]");
            }
            r->ploc_radius = (int)value;
        } else if (k == "bvh_builder") {
            if (value < 0 || value > 2) {
                throw std::runtime_error("bvh_builder must be 0 (host), 1 (device, PLOC) or 2 (device, LBVH)");
            }
            r->bvh_builder = (int)value;
        } else if (k == "count_traversal") {
            r->count_traversal = value != 0;
        } else if (k == "dynamic_scene") {
            if (value < 0 || value > 1) {
                throw std::runtime_error("dynamic_scene must be 0 or 1");
            }
            r->dynamic_scene = value != 0;  // takes effect at the next crtc_set_scene
        } else if (k == "aov") {
            r->aov = value != 0;  // takes effect at the next crtc_initialize
        } else if (k == "views") {
            if (value < 1 || value > crt::kMaxViews) {
                throw std::runtime_error("views must be in [1, 64]");
            }
            r->views = (uint32_t)value;  // takes effect at the next crtc_initialize
        } else if (k == "denoise_history") {
            if (value < 0 || value > 1024) {
                throw std::runtime_error("denoise_history must be in [0, 1024] (0 = off)");
            }
            r->dn_history = (uint32_t)value;  // takes effect at the next crtc_initialize
        } else if (k == "denoise_motion") {
            if (value < 0 || value > 1) {
                throw std::runtime_error("denoise_motion must be 0 or 1");
            }
            r->dn_motion = value != 0;  // takes effect at the next crtc_initialize
        } else if (k == "refill_idle") {
            r->refill_idle = (int)std::min<int64_t>(std::max<int64_t>(value, 1), 32);
        } else if (k == "any_far_first") {
            if (value < 0 || value > 2) {
                throw std::runtime_error("any_far_first must be 0 (off), 1 (on) or 2 (auto)");
            }
            r->any_far_first = (int)value;
            r->auto_frames = 0;
            r->auto_decided = false;
        } else {
            throw std::runtime_error("unknown option '" + k + "'");
        }
        // (rank may be set before world_size: the pair is validated in crtc_initialize)
    })
}

int crtc_get_option(crtc_renderer *r, const char *key, int64_t *value)
{
    CRTC_TRY({ require_renderer(r);
        const std::string k = key ? key : "";
        if (!value) {
            throw std::runtime_error("crtc_get_option: value is null");
        }
        if (k == "max_depth") {
            *value = r->max_depth;
        } else if (k == "rank") {
            *value = r->rank;
        } else if (k == "world_size") {
            *value = r->world_size;
        } else if (k == "bvh_threads") {
            *value = r->bvh_threads;
        } else if (k == "tri_pass_defer") {
            *value = r->tri_pass_defer;
        } else if (k == "hw_textures") {
            *value = r->hw_textures ? 1 : 0;
        } else if (k == "shade_sort") {
            *value = r->shade_sort;
        } else if (k == "bvh_builder") {
            *value = r->bvh_builder;
        } else if (k == "bvh_builder_fallbacks") {
            *value = r->builder_fallbacks;
        } else if (k == "bvh_build_rounds") {
            *value = r->build_rounds;  // PLOC rounds of the last device build
        } else if (k == "count_traversal") {
            *value = r->count_traversal ? 1 : 0;
        } else if (k == "dynamic_scene") {
            *value = r->dynamic_scene ? 1 : 0;
        } else if (k == "aov") {
            *value = r->aov ? 1 : 0;
        } else if (k == "views") {
            *value = r->views;
        } else if (k == "denoise_history") {
            *value = r->dn_history;
        } else if (k == "denoise_motion") {
            *value = r->dn_motion ? 1 : 0;
        } else if (k == "refill_idle") {
            *value = r->refill_idle;
        } else if (k == "any_far_first") {
            *value = r->any_far_first;
        } else if (k == "any_far_first_decision") {
            // the order frames are rendered with from now on: 0 near-first, 1 far-first, -1 auto mode still undecided
            *value = r->any_far_first != 2 ? (r->any_far_first == 1 ? 1 : 0) : (r->auto_decided ? (r->auto_choice ? 1 : 0) : -1);
        } else {
            throw std::runtime_error("unknown option '" + k + "'");
        }
    })
}

int crtc_set_stream(crtc_renderer *r, void *cuda_stream)
{
    CRTC_TRY({ require_renderer(r); r->stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : r->own_stream; })
}

int crtc_initialize(crtc_renderer *r, int fb_width, int fb_height)
{
    CRTC_TRY({ require_renderer(r);
        if (r->rank < 0 || r->rank >= r->world_size) {
            throw std::runtime_error("rank must be in [0, world_size)");
        }
        r->initialize(fb_width, fb_height);
    })
}

int crtc_set_scene(crtc_renderer *r, const crt_scene_t *scene)
{
    CRTC_TRY({ require_renderer(r);
        if (!scene) {
            throw std::runtime_error("crtc_set_scene: scene is NULL");
        }
        r->set_scene(scene);
    })
}

int crtc_update_instances(crtc_renderer *r, uint32_t first, uint32_t count, const float *transforms)
{
    CRTC_TRY({ require_renderer(r); r->require_dynamic("crtc_update_instances").stage_instances(first, count, transforms); })
}

int crtc_update_vertices(crtc_renderer *r, uint32_t mesh, uint32_t geometry, const float *vertices, uint32_t num_vertices)
{
    CRTC_TRY({ require_renderer(r); r->require_dynamic("crtc_update_vertices").stage_vertices(mesh, geometry, vertices, num_vertices); })
}

int crtc_update_lights(crtc_renderer *r, const crt_quad_light_t *lights, uint32_t num_lights)
{
    CRTC_TRY({ require_renderer(r); r->update_lights(lights, num_lights); })
}

int crtc_commit_scene(crtc_renderer *r)
{
    CRTC_TRY({ require_renderer(r); r->commit_scene(); })
}

int crtc_render(crtc_renderer *r, const float *pos, const float *dir, const float *up, float fovy, int camera_changed,
                int readback_framebuffer, uint32_t *img, crt_render_stats_t *stats)
{
    CRTC_TRY({ require_renderer(r); r->require_single_view("crtc_render"); r->render(pos, dir, up, fovy, camera_changed != 0, readback_framebuffer != 0, img, stats); })
}

int crtc_render_async(crtc_renderer *r, const float *pos, const float *dir, const float *up, float fovy,
                      int camera_changed, uint32_t num_frames)
{
    CRTC_TRY({ require_renderer(r); r->require_single_view("crtc_render_async"); r->enqueue_frame(pos, dir, up, fovy, camera_changed != 0, num_frames); })
}

int crtc_render_views(crtc_renderer *r, const crtc_view_t *views, uint32_t num_views, uint32_t num_frames)
{
    CRTC_TRY({ require_renderer(r); r->enqueue_views(views, num_views, num_frames); })
}

int crtc_read_view(crtc_renderer *r, uint32_t view, float *rgb_out, uint32_t *img_out)
{
    CRTC_TRY({ require_renderer(r); r->read_view(view, rgb_out, img_out); })
}

int crtc_sync(crtc_renderer *r, crt_render_stats_t *total, float *stage_ms_sum, uint64_t *counters_sum,
              uint32_t *num_frames)
{
    CRTC_TRY({ require_renderer(r);
        const uint32_t n = r->sync_frames(total, stage_ms_sum, counters_sum);
        if (num_frames) {
            *num_frames = n;
        }
    })
}

int crtc_read_accum(crtc_renderer *r, float *rgb_out)
{
    CRTC_TRY({ require_renderer(r);
        r->require_single_view("crtc_read_accum");
        r->make_current();
        r->frame_wait();
        CUDA_CHECK(cudaMemcpyAsync(rgb_out, r->d_accum_full.ptr, (size_t)r->fb_w * r->fb_h * 3 * sizeof(float),
                                   cudaMemcpyDeviceToHost, r->stream));
        CUDA_CHECK(cudaStreamSynchronize(r->stream));
        r->check_sync_error();
    })
}

int crtc_read_img(crtc_renderer *r, uint32_t *img)
{
    CRTC_TRY({ require_renderer(r);
        r->require_single_view("crtc_read_img");
        r->make_current();
        r->frame_wait();  // (a shared frame: every rank's tiles first; no-op otherwise)
        if (img == r->pinned_img || r->pin_repeated_reads) {  // (a caller that reads into the same buffer every frame)
            r->pin_img(img, (size_t)r->fb_w * r->fb_h * 4);
        }
        CUDA_CHECK(cudaMemcpyAsync(img, r->d_img_full.ptr, (size_t)r->fb_w * r->fb_h * 4, cudaMemcpyDeviceToHost,
                                   r->stream));
        CUDA_CHECK(cudaStreamSynchronize(r->stream));
        r->check_sync_error();
    })
}

int crtc_read_aov(crtc_renderer *r, float *out)
{
    CRTC_TRY({ require_renderer(r);
        if (!out) {
            throw std::runtime_error("crtc_read_aov: out is NULL");
        }
        r->read_aov(out);
    })
}

int crtc_denoise(crtc_renderer *r, const crtc_denoise_params_t *params, float *rgb_out, uint32_t *img_out, void *cuda_array)
{
    CRTC_TRY({ require_renderer(r); r->denoise(params, rgb_out, img_out, cuda_array); })
}

int crtc_read_denoise_history(crtc_renderer *r, float *out)
{
    CRTC_TRY({ require_renderer(r);
        if (!out) {
            throw std::runtime_error("crtc_read_denoise_history: out is NULL");
        }
        r->read_denoise_history(out);
    })
}

int crtc_set_adaptive(crtc_renderer *r, const crtc_adaptive_params_t *params)
{
    CRTC_TRY({ require_renderer(r); r->set_adaptive(params); })
}

int crtc_read_adaptive(crtc_renderer *r, uint32_t *samples_out, float *error_out)
{
    CRTC_TRY({ require_renderer(r); r->read_adaptive(samples_out, error_out); })
}

int crtc_get_stage_times(crtc_renderer *r, float *ms_out, int n)
{
    if (!r || !ms_out || n <= 0) {
        return 0;
    }
    const int m = std::min(n, (int)kNumStages);
    for (int i = 0; i < m; ++i) {
        ms_out[i] = r->stage_ms[i];
    }
    return m;
}

int crtc_get_counters(crtc_renderer *r, uint64_t *out, int n)
{
    if (!r || !out || n <= 0) {
        return 0;
    }
    const int m = std::min(n, 8);
    for (int i = 0; i < m; ++i) {
        out[i] = r->counters_out[i];
    }
    return m;
}

int crtc_get_scene_info(crtc_renderer *r, double *out, int n)
{
    if (!r || !out || n <= 0) {
        return 0;
    }
    const int m = std::min(n, 12);
    for (int i = 0; i < m; ++i) {
        out[i] = r->scene_info[i];
    }
    return m;
}

int crtc_trace_closest(crtc_renderer *r, const float *rays, uint64_t n, float *hits)
{
    CRTC_TRY({ require_renderer(r); r->trace_closest(rays, n, hits); })
}

int crtc_trace_any(crtc_renderer *r, const float *rays, uint64_t n, uint8_t *occluded)
{
    CRTC_TRY({ require_renderer(r); r->trace_any(rays, n, occluded); })
}

int crtc_bench_trace(crtc_renderer *r, const float *rays_host, uint64_t n, int any_hit, int iters, float *ms_out)
{
    CRTC_TRY({ require_renderer(r); *ms_out = r->bench_trace(rays_host, n, any_hit != 0, iters); })
}

int crtc_local_buffers(crtc_renderer *r, void **accum_dev, void **img_dev, uint32_t *num_local_tiles)
{
    CRTC_TRY({ require_renderer(r);
        r->require_single_view("crtc_local_buffers");
        *accum_dev = r->d_accum_local.ptr;
        *img_dev = r->d_img_local.ptr;
        *num_local_tiles = (uint32_t)r->local_tiles.size();
    })
}

int crtc_assemble_rank(crtc_renderer *r, int src_rank, int world_size, const void *accum_dev, const void *img_dev)
{
    CRTC_TRY({ require_renderer(r); r->require_single_view("crtc_assemble_rank"); r->assemble_rank(src_rank, world_size, accum_dev, img_dev); })
}

int crtc_export_frame(crtc_renderer *r, void *handles_out)
{
    CRTC_TRY({ require_renderer(r);
        if (!handles_out) {
            throw std::runtime_error("crtc_export_frame: null output");
        }
        r->require_single_view("crtc_export_frame");
        r->export_frame(handles_out);
    })
}

int crtc_import_frame(crtc_renderer *r, const void *handles)
{
    CRTC_TRY({ require_renderer(r); r->require_single_view("crtc_import_frame"); r->import_frame(handles); })
}

int crtc_copy_img_to_array(crtc_renderer *r, void *cuda_array)
{
    CRTC_TRY({ require_renderer(r);
        if (!cuda_array) {
            throw std::runtime_error("crtc_copy_img_to_array: array is NULL");
        }
        r->require_single_view("crtc_copy_img_to_array");
        r->make_current();
        r->frame_wait();
        CUDA_CHECK(cudaMemcpy2DToArrayAsync(static_cast<cudaArray_t>(cuda_array), 0, 0, r->d_img_full.ptr, (size_t)r->fb_w * 4,
                                            (size_t)r->fb_w * 4, (size_t)r->fb_h, cudaMemcpyDeviceToDevice, r->stream));
        CUDA_CHECK(cudaStreamSynchronize(r->stream));
        r->check_sync_error();
    })
}

int crtc_frame_wait(crtc_renderer *r)
{
    CRTC_TRY({ require_renderer(r); r->frame_wait(); })
}

int crtc_share_frame(crtc_renderer *dst, crtc_renderer *src)
{
    CRTC_TRY({
        if (!dst || !src) {
            throw std::runtime_error("crtc_share_frame: null renderer");
        }
        dst->require_single_view("crtc_share_frame");
        src->require_single_view("crtc_share_frame");
        src->share_frame_of(dst);
    })
}
}
