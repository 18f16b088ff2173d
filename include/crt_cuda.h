/* crt_cuda.h — C ABI of libcrt_cuda_core.so, the H100-native (sm_90a) wavefront path tracer that sits
 * behind ChameleonRT's RenderBackend interface.
 *
 * The reference's plugin boundary is C++ (a vtable and std::vector cross it:
 * util/render_backend.h:12-32, util/render_plugin.h:23-63). This header is the plain-C
 * surface underneath: one entry point per RenderBackend member, plain pointers and sizes, no
 * C++ or torch types. backends/cuda/render_cuda.cpp (the drop-in `crt_cuda` plugin a
 * ChameleonRT maintainer builds) and chameleonrt_b200/backend.py (ctypes) both bind exactly
 * these symbols; INTEGRATION.md shows the binding.
 *
 *   RenderBackend member (util/render_backend.h)        ->  C entry point
 *   ---------------------------------------------------------------------------------------
 *   constructor / make_renderer (render_plugin.h:41)    ->  crtc_create
 *   virtual ~RenderBackend()                 :16        ->  crtc_destroy
 *   std::string name()                       :18        ->  crtc_name
 *   void initialize(fb_width, fb_height)     :20        ->  crtc_initialize
 *   void set_scene(const Scene&)             :23        ->  crtc_set_scene
 *   RenderStats render(pos, dir, up, fovy,
 *        camera_changed, readback_framebuffer) :26-31   ->  crtc_render
 *   std::vector<uint32_t> img                :13        ->  the `img` out-parameter of crtc_render
 *   uint32_t samples_per_pixel               :14        ->  crt_scene_t::samples_per_pixel
 *
 * Error behaviour: the reference throws std::runtime_error and nothing catches it
 * (SURVEY.md §5). Here every call returns 0 on success and non-zero on failure, with the
 * message available from crtc_last_error(); the C++ plugin rethrows it as
 * std::runtime_error, the Python binding raises RuntimeError. There is NO CPU fallback: if
 * no CUDA device is usable crtc_create fails.
 *
 * Threading: like the reference, all calls on one renderer come from one thread.
 */
#ifndef CRT_CUDA_H
#define CRT_CUDA_H

#include <stdint.h>

#include "crt_scene.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct crtc_renderer crtc_renderer;

/* Message of the last failed call on this thread ("" if none). */
const char *crtc_last_error(void);

/* RenderBackend::name(). */
const char *crtc_name(void);

/* Creates a renderer on CUDA device `device` (cudaSetDevice ordinal). */
int crtc_create(crtc_renderer **out, int device);
void crtc_destroy(crtc_renderer *r);

/* Options the plugin API has no channel for (the reference hard-codes them; the plugin reads
 * CRT_CUDA_* environment variables and forwards them here). Must be set before
 * crtc_initialize / crtc_set_scene.
 *   "max_depth"   path depth, reference MAX_PATH_DEPTH = 5 (backends/embree/util.ih:10)
 *   "rank", "world_size"  image-tile sharding: this renderer owns the 64x64 tiles with
 *                 tile_id % world_size == rank (tile_id as in render_embree.cpp:178-180)
 *   "bvh_threads" host threads for the BVH8 build (0 = all)
 *   "tri_pass_defer" 0, 16 (default) or 24: scheduling variant of the traversal kernel — a warp's pooled
 *                 triangle pass waits until that many (ray, triangle) pairs are pending or no lane can descend.
 *                 Never changes a result. Measured on an H100 SXM (80 GB, 700 W; scripts/ab_options.py): 0 makes the frame
 *                 3.8 % / 3.2 % / 7.8 % longer on the C2 / C3 / C4 workloads, 24 0.7-1.4 % longer.
 *   "shade_sort"  0 (default), 1 or 2: the queue of paths to shade is bucketed by the material id of each path's hit
 *                 (one stable counting-sort pass on the device, 256 buckets) before the shading kernel runs, so that a
 *                 warp unpacks one material and runs the same BSDF lobes: 1 = from the first bounce on (primary hits
 *                 keep their screen order), 2 = every bounce. Never changes a result. Measured on an H100 SXM (80 GB, 700 W): the
 *                 frame gets 19-30 % longer on C2 / C4 and 10 % on C3 (the sort passes and the scattered path-state accesses
 *                 cost more than the coherence buys); kept as an option, off.
 *   "hw_textures" 0 (default): textures are filtered in software with the reference's own arithmetic (texture2d.ih:
 *                 float->int truncation of texel coordinates, wrap by modulo, bilinear weights in float, over the 8-bit
 *                 LINEARISED texels render_embree.cpp:96-103 produces) — bit-level parity with the Embree backend.
 *                 1: one cudaTextureObject_t per texture (wrap, linear, normalised coordinates, sRGB decode in the texture
 *                 unit), as the reference's OptiX backend does (backends/optix/optix_utils.cpp:60-85): 8-bit fixed-point
 *                 filter weights and no re-quantisation of the linearised texels, hence a looser parity with the Embree
 *                 path (dark sRGB texels are not crushed to 0). Takes effect at the next crtc_set_scene.
 *   "bvh_top_smem" 0 (default) / 1: the traversal kernel reads the first 73 BVH nodes (root + two levels) from a shared-memory
 *                 copy — BASELINE.json's north_star names this staging; measured on an H100 SXM (80 GB, 700 W) it makes the
 *                 frame 2-3 % longer on C2 / C4 (those nodes are the L1's hottest lines anyway and the copy takes 47 KB of L1
 *                 per SM), so it is off. Never changes a result.
 *   "stage_events" 1 (default): a CUDA event after every launch feeds crtc_get_stage_times; 0: events only at the start
 *                 and the end of a frame ([6], the frame time, stays; the other stage times read 0) — 28 event records cost
 *                 ~0.07 ms per frame, which matters when a GPU renders a 1/8 shard in 2 ms. May be changed between frames.
 *   "pin_host_buffers" 1 (default): the caller's img buffer is page-locked on first readback (cudaHostRegister);
 *   "pin_read_img" 1: crtc_read_img page-locks its destination too (a frame loop reading into one buffer). Default 0.
 *   "bvh_builder" where crtc_set_scene builds the BVH8: 0 = on the host (binned SAH, the default); on the device
 *                 (chameleonrt_b200/csrc/bvh8_device.cuh): 1 = PLOC (mutual nearest neighbours in Morton order),
 *                 2 = LBVH (Karras), both followed by the host builder's 8-wide collapse — a much shorter set_scene
 *                 on scenes of millions of triangles for a somewhat slower tree. Rendered frames are bit-identical
 *                 in every case (closest hits break ties on the primitive id, DESIGN.md section 2).
 *                 Developer knobs of the PLOC builder: "bvh_ploc_radius" (1..32, default 16: clusters searched on
 *                 either side) and "bvh_ploc_tail" (default 1: the last rounds run in a single block).
 *   "refill_idle" scheduling knob of the persistent traversal kernels (how many idle lanes
 *                 trigger a refill from the ray queue); the default is tuned
 *   "any_far_first" 1 = shadow (any-hit) rays visit the children of a BVH node farthest-first instead of
 *                 nearest-first. The result of an occlusion query does not depend on the order; the work does
 *                 (fewer node steps when occluders sit near the light's end of the segment, more when they sit
 *                 near the surface). 2 = decide per scene (the default): the second crtc_render frame after
 *                 crtc_set_scene runs far-first, the third near-first, and far-first is kept only if its traversal
 *                 stage was at least 3 % faster. 0 = off.
 *   "count_traversal" 1 = instrumented traversal kernels that count node visits and triangle
 *                 tests (for the algorithmic-byte figure; slower, off by default)
 *   "aov"         0 (default) / 1: first-hit AOV buffers accumulated with every frame, read with crtc_read_aov and used by
 *                 crtc_denoise. Takes effect at the next crtc_initialize. Needs the whole frame on one renderer: with
 *                 world_size > 1 crtc_initialize fails, and crtc_export_frame / crtc_import_frame / crtc_share_frame fail
 *                 on a renderer initialized with it. Two kernels per wavefront (k_aov_primary after the primary traversal,
 *                 k_aov_moments after the resolve), so counter [2] (kernel launches) grows by 2 per wavefront; their
 *                 times are counted in stage [2] (shade) and [5] (resolve) of crtc_get_stage_times. They read the path
 *                 state and write only their own buffers: accum, img and the ray counts are the same with the option on.
 *                 With option denoise_motion on a dynamic scene, an epoch's first wavefront (the first after a reset) runs
 *                 a third one, k_aov_hit (counted in stage [2]), so counter [2] grows by 3 there.
 *                 Memory: 40 B per pixel of the local tiles (64x64-padded) + 40 B per framebuffer pixel; the first
 *                 crtc_denoise adds 72 B per framebuffer pixel (1920x1080: 166 MB of AOVs + 149 MB for the denoiser).
 *   "denoise_history" H in 0..1024, 0 (default) = off: crtc_denoise carries a temporal history across accumulation
 *                 resets (camera moves), reprojected into the current camera and capped at H samples (see crtc_denoise).
 *                 Takes effect at the next crtc_initialize, which fails if it is nonzero with option aov = 0; out of
 *                 range is an error. Nothing runs in the frame path: two more kernels run inside crtc_denoise only. Memory:
 *                 the first crtc_denoise adds 80 B per framebuffer pixel (two history buffers of 10 floats; 1920x1080:
 *                 166 MB). crtc_initialize and crtc_set_scene drop the history.
 *   "denoise_motion" 0 (default) / 1: a crtc_commit_scene that moves geometry keeps the denoiser's history; the next
 *                 crtc_denoise reprojects each pixel through the motion of the triangle it sees (crtc_denoise, step b').
 *                 Takes effect at the next crtc_initialize, which fails if it is 1 with option denoise_history = 0; any
 *                 other value than 0 or 1 is an error. Acts only on scenes set with dynamic_scene = 1: with a static scene
 *                 nothing is allocated and nothing runs. On a dynamic scene: one more kernel in an epoch's first
 *                 wavefront (see "aov"); memory: 12 B per framebuffer pixel (each pixel's hit record) and, from the first
 *                 crtc_denoise, two geometry snapshots of 128 B per instance + 12 B per unique vertex, one per history
 *                 buffer (C3: 961 instances, ~2 x 0.1 MB + the vertices). Commits that change lights still drop the
 *                 history. After a commit that keeps the history, the sample sequence is not restarted: the frames
 *                 draw the samples of frame indices b, b + 1, ... (b = the frames rendered since the last other reset,
 *                 i.e. crtc_initialize, crtc_set_scene, a commit that drops the history or a camera_changed render after
 *                 a frame; a camera_changed render right after the commit does not reset b). Otherwise a still pixel
 *                 would re-render the samples its history already holds, and the history would add nothing. Frames of
 *                 camera-only epochs are unchanged. The drop-in plugin (backends/cuda) has no scene-update channel and
 *                 does not use the option.
 *   "dynamic_scene" 0 (default) / 1: crtc_set_scene keeps on the device what crtc_update_instances / crtc_update_vertices
 *                 and crtc_commit_scene need. Takes effect at the next crtc_set_scene; with 0 nothing is kept and nothing
 *                 more runs. Every builder ("bvh_builder" 0, 1, 2). Memory: the unique geometry (12 B per unique vertex,
 *                 + 8 B if it has uvs; 12 B per unique triangle; 128 B per instance; 32 B per (instance, geometry) pair),
 *                 36 B per flattened triangle and 32 B per BVH8 node.
 *   "views"       V in 1..64, 1 (default): the number of cameras crtc_render_views traces together (see there). Takes
 *                 effect at the next crtc_initialize; out of range is an error. V = 1 changes nothing.
 */
int crtc_set_option(crtc_renderer *r, const char *key, int64_t value);

/* Reads an option back. Readable keys: every key of crtc_set_option, plus "any_far_first_decision" = the shadow-ray order
 * frames are rendered with from now on (0 near-first, 1 far-first, -1 = mode 2 has not decided yet), "bvh_build_rounds" =
 * the number of PLOC rounds of the last device build, and "bvh_builder_fallbacks" = device builds that gave up on their
 * input and were redone by the host builder. */
int crtc_get_option(crtc_renderer *r, const char *key, int64_t *value);

/* Use an existing CUDA stream (cudaStream_t) for all work of this renderer; NULL = the
 * renderer's own stream. Lets a host that already owns a stream (e.g. PyTorch's current
 * stream) order and time the work with its own events. */
int crtc_set_stream(crtc_renderer *r, void *cuda_stream);

/* RenderBackend::initialize: (re)allocates the framebuffer state and resets accumulation. */
int crtc_initialize(crtc_renderer *r, int fb_width, int fb_height);

/* RenderBackend::set_scene: flattens instances, builds the BVH8 on the host, uploads
 * geometry / materials / textures / lights, resets accumulation.
 * Vertex values and instance matrices are not checked: NaN, +-inf and values up to +-FLT_MAX are accepted here and by
 * crtc_update_instances / crtc_update_vertices, by every builder (a device build that cannot progress over non-finite
 * boxes is redone by the host builder, as "bvh_builder_fallbacks" counts). A hit is what a brute-force test of every
 * world-space triangle with the kernel's float32 triangle formula finds: the closest t, ties to the lowest flattened id.
 * For every ray, traces give that hit, a miss, or a hit later in (t, id) order; never a closer or a false hit. They give
 * exactly that hit (closest hits bit for bit, occlusion answers equal) for every ray it has none for, and for every ray
 * whose hit is well conditioned, i.e. whose triangle lies within 2^16 of its longest edges of the ray origin (farther,
 * the triangle formula's own rounding can exceed the triangle), when:
 *   - all world-space vertices (NaN coordinates do not count) and ray origins lie in a box of extent at most
 *     kExactExtent = 255 * 2^46 (about 1.79e16) on each axis; or
 *   - past that extent: every coordinate is above -kExactExtent, the hit triangle lies within 2^107, and every
 *     direction component has magnitude at least 2^-12.
 * Otherwise box-test planes can overflow: 2^(e+15) / |d_a| passes FLT_MAX for a node grid step 2^e with e >= 47 and a
 * zero direction component (clamped to 1e-20), so rays straight along an axis miss a scene just wider than
 * kExactExtent; and a node whose low corner lies below the ray origin by more than FLT_MAX * |d_a| on an axis is culled
 * for that ray, so a single vertex at -inf or near -FLT_MAX hides every triangle that shares a node with it (in the
 * worst case the whole scene) from every ray. Node grids stop at 2^100, so a triangle beyond about 3.2e32 from its
 * node's low corner can be culled too. */
int crtc_set_scene(crtc_renderer *r, const crt_scene_t *scene);

/* Scene updates between frames, without a new crtc_set_scene: instances move, meshes deform, lights change. The update
 * calls only stage; crtc_commit_scene applies everything staged at once. The caller's arrays may be reused as soon as an
 * update call returns. crtc_set_scene discards staged updates.
 *   Topology is fixed: indices, uvs, materials, textures and the instance -> mesh mapping stay those of crtc_set_scene.
 *   Result: after a commit, frames, crtc_trace_closest and crtc_trace_any are bit-identical to those of a renderer that
 *   was crtc_set_scene'd with the updated scene (same options). The BVH8 keeps its topology and leaf order and its boxes
 *   are refit on the device (DESIGN.md section 2, "Scene updates"); a tree refit after large motions traces slower than
 *   a new build of the moved scene (profiles/dynamic_h100.md): crtc_set_scene is the way to get a new tree.
 * Every call fails if no scene has been set.
 *
 * crtc_update_instances: needs option dynamic_scene = 1 at the last crtc_set_scene. Instances first .. first + count - 1
 * get new object_to_world matrices, 16 floats each, column-major as crt_instance_t::transform. world_to_object is
 * computed on the host as crtc_set_scene computes it, so any matrix crtc_set_scene accepts (singular or non-finite
 * included) gives the same result as there. Fails if first + count exceeds the instance count or transforms is NULL
 * with count > 0. */
int crtc_update_instances(crtc_renderer *r, uint32_t first, uint32_t count, const float *transforms);
/* crtc_update_vertices: needs option dynamic_scene = 1 at the last crtc_set_scene. New positions of the vertices of
 * geometry `geometry` of mesh `mesh` (3 floats each, object space); every instance of the mesh moves with them. Fails if
 * the mesh or geometry id is out of range, if num_vertices differs from the geometry's vertex count at crtc_set_scene, or
 * if vertices is NULL with num_vertices > 0. A geometry that no instance references with triangles is accepted and the
 * update does nothing. Staging the same geometry twice keeps the later positions. */
int crtc_update_vertices(crtc_renderer *r, uint32_t mesh, uint32_t geometry, const float *vertices, uint32_t num_vertices);
/* crtc_update_lights: no option needed. Replaces all lights (crt_quad_light_t records, as crt_scene_t::lights); the
 * count may change. Fails if num_lights is 0 (as crtc_set_scene does) or lights is NULL. */
int crtc_update_lights(crtc_renderer *r, const crt_quad_light_t *lights, uint32_t num_lights);
/* crtc_commit_scene: applies the staged updates. Enqueued on the renderer's stream (crtc_set_stream applies) without
 * waiting for frames in flight: frames enqueued before see the old scene, frames enqueued after the new one (the
 * staged data is copied from pageable memory; a light count above every earlier one waits for the stream once). Every
 * commit with staged instances or vertices re-flattens every triangle (k_reflatten) and refits every node (one
 * k_bvh8_refit launch per BVH8 level). Then:
 *   - the accumulation resets as on camera_changed: accum, the AOVs and the adaptive block counts; the next frame equals
 *     frame 0 of a fresh renderer (with option denoise_motion keeping the history: frame b of one, see the option);
 *   - the denoiser's history is dropped (its reprojection assumes static geometry), unless option denoise_motion is on and
 *     the commit stages no lights: then it is kept and the next crtc_denoise moves it with the geometry (step b'). Either
 *     way crtc_read_denoise_history fails until the next crtc_denoise;
 *   - the any_far_first decision is kept; if mode 2 has not decided yet, its trial restarts as after crtc_set_scene;
 *   - frame counters and stage times do not include the commit's launches.
 * With nothing staged it does nothing: no reset, no launch. */
int crtc_commit_scene(crtc_renderer *r);

/* RenderBackend::render. pos/dir/up: 3 floats each; fovy in degrees. If
 * readback_framebuffer != 0 and img != NULL, img receives fb_width*fb_height RGBA8 pixels
 * (row-major, y down — RenderBackend::img). stats may be NULL. With world_size > 1 only the
 * tiles this rank owns are rendered and written; the rest of img is left untouched. */
int crtc_render(crtc_renderer *r, const float *pos, const float *dir, const float *up, float fovy,
                int camera_changed, int readback_framebuffer, uint32_t *img, crt_render_stats_t *stats);

/* Throughput variant of render for frame loops that do not need each frame's result on the host:
 * enqueues `num_frames` (>= 1) consecutive frames on the renderer's stream and returns immediately,
 * so the host can queue more work (or a gather) while they run. The frames of one call are
 * rendered as a single wavefront — num_frames * spp samples per pixel in flight together, seeded
 * and folded into the running mean exactly as num_frames separate calls would be (bit-identical
 * result) — which keeps a GPU that owns only part of the image busy. crtc_sync waits for all such frames and returns
 * their totals: `total` (render_time = sum of per-frame device times, num_rays = sum),
 * `stage_ms_sum` (7 floats, as crtc_get_stage_times), `counters_sum` (8, as crtc_get_counters),
 * `num_frames`; any of them may be NULL. The accumulation semantics are those of crtc_render. With adaptive sampling
 * (crtc_set_adaptive) a call selects its active blocks once: every pixel still holds the uniform render's result at its
 * own count, but which blocks advance may differ from num_frames separate calls. */
int crtc_render_async(crtc_renderer *r, const float *pos, const float *dir, const float *up, float fovy,
                      int camera_changed, uint32_t num_frames);
int crtc_sync(crtc_renderer *r, crt_render_stats_t *total, float *stage_ms_sum, uint64_t *counters_sum,
              uint32_t *num_frames);

/* One camera of crtc_render_views: the arguments crtc_render takes for it. */
typedef struct crtc_view_t {
    float pos[3], dir[3], up[3];
    float fovy;
    int camera_changed;
} crtc_view_t;

/* Multi-view rendering: several cameras' frames of the same scene as ONE wavefront. A renderer initialized with option
 * "views" = V > 1 keeps V accumulation buffers and V full frames, view-major, and a frame counter b_k per view.
 *   crtc_render_views enqueues num_frames (1..64) frames of each of the num_views views (num_views must equal V) as a
 *   single wavefront on the renderer's stream and returns without waiting; crtc_sync collects it like a crtc_render_async
 *   call: num_rays and the counters are summed over the views, the frame count grows by num_frames per call, the stage
 *   times are those of the one wavefront, and counter [2] (launches) equals that of a one-view crtc_render_async call with
 *   the same num_frames: no launch is added per view. Such calls never advance the "any_far_first" = 2 trial.
 *   Resets. views[k].camera_changed resets view k only (b_k = 0), as crtc_render does; crtc_initialize, crtc_set_scene
 *   and a crtc_commit_scene that applies something reset every view.
 *   Guarantee. After any sequence of crtc_render_views calls, view k's accum and img equal, bit for bit, those of a
 *   renderer with V = 1 and otherwise the same options, scene and size that received crtc_render_async calls with view k's
 *   camera, camera_changed flag and num_frames, in the same order: path (view k, pixel, sample s of the batch) is seeded as
 *   that renderer seeds it, from frame b_k; traversal, shading and next-event estimation are per path and do not depend
 *   on its queue position; the resolve folds view k's samples with b_k.
 *   Memory per view: 16 B per pixel of the 64x64-padded tiles (accum + img) + 16 B per framebuffer pixel (the full frame),
 *   and the path state of V times as many paths (about 200 B per path in flight, as for crtc_render_async).
 *   With V = 1, crtc_render_views is crtc_render_async with views[0] and crtc_read_view(r, 0, ...) reads the frame.
 *   With V > 1 the following are errors (the renderer stays usable): crtc_initialize with option "aov", with
 *   world_size > 1 or with adaptive sampling set; crtc_set_adaptive with params != NULL; crtc_render, crtc_render_async,
 *   crtc_read_accum, crtc_read_img, crtc_copy_img_to_array, crtc_export_frame, crtc_import_frame, crtc_share_frame,
 *   crtc_local_buffers and crtc_assemble_rank; and a call with V * num_frames * spp * (64x64-padded pixels) >= 2^31
 *   paths. crtc_trace_closest, crtc_trace_any, crtc_bench_trace, the scene-update calls and the options "hw_textures",
 *   "bvh_builder", "count_traversal" and "stage_events" work as with one view.
 *   Not supported: views across GPUs, AOVs and the denoiser per view, adaptive sampling per view, a different size or
 *   spp per view, non-pinhole cameras, and a channel in the drop-in plugin (which has one camera by construction). */
int crtc_render_views(crtc_renderer *r, const crtc_view_t *views, uint32_t num_views, uint32_t num_frames);
/* View `view` (< option views at the last crtc_initialize) of a multi-view renderer: its accum (fb_width*fb_height*3
 * floats, as crtc_read_accum) and img (fb_width*fb_height RGBA8, as crtc_read_img), either may be NULL. Waits for the
 * stream first, like crtc_read_accum. */
int crtc_read_view(crtc_renderer *r, uint32_t view, float *rgb_out, uint32_t *img_out);

/* The accumulated float framebuffer (what parity compares): fb_width*fb_height*3 floats,
 * row-major RGB. The reference keeps it backend-private and tile-major
 * (render_embree.h:26, render_embree.ispc:345); this is the extra export SURVEY.md §8b asks
 * for. */
int crtc_read_accum(crtc_renderer *r, float *rgb_out);

/* Per-stage device times of the last frame, in ms (CUDA events on the renderer's stream):
 * [0] raygen [1] traversal of the primary rays [2] shade [3] traversal of bounce b's shadow rays
 * together with bounce b+1's continuation rays (one launch per bounce) [4] NEE resolve
 * [5] resolve+tonemap [6] whole frame. Returns the number of entries written (<= n). */
int crtc_get_stage_times(crtc_renderer *r, float *ms_out, int n);

/* Counters of the last frame: [0] closest-hit rays [1] occlusion rays [2] kernel launches
 * [3] BVH nodes visited and [4] triangles tested by closest-hit traversal [5] paths started
 * [6] nodes visited and [7] triangles tested by any-hit traversal ([3],[4],[6],[7] only with
 * count_traversal=1). */
int crtc_get_counters(crtc_renderer *r, uint64_t *out, int n);

/* Scene/BVH facts: [0] triangles [1] BVH8 nodes [2] BVH depth [3] build ms [4] node bytes
 * [5] triangle bytes; the last crtc_set_scene in phases, ms: [6] flattening (host wall clock: host work, or uploads +
 * k_flatten), and for the device builders (CUDA events) [7] Morton keys + sort [8] binary tree (PLOC / LBVH) [9] BVH8
 * emission [10] record packing ([10] is host wall clock for the host builder, [7]-[9] are 0 there); [11] PLOC rounds. */
int crtc_get_scene_info(crtc_renderer *r, double *out, int n);

/* Kernel-level access for parity tests and micro-benchmarks: trace a batch of rays against
 * the current scene with the same traversal kernels render() uses. rays: n*8 floats
 * {ox,oy,oz,tnear,dx,dy,dz,tfar} in HOST memory; hits: n*4 floats {t,u,v,bits(flat prim id or
 * 0xffffffff)}; occluded: n bytes. A hit is a triangle at tnear < t < tfar, for any tnear, negative included (t < 0 is
 * a hit behind the origin); ties in t (-0 == +0) go to the lower primitive id, and a miss reports t = tfar. In
 * crtc_trace_any, rays whose tnear is exactly 1e-4f (the renderer's shadow rays) run the any-hit kernel; every other
 * ray runs the closest-hit kernel and is occluded when it finds a hit. Both answer for the ray's own interval. */
int crtc_trace_closest(crtc_renderer *r, const float *rays, uint64_t n, float *hits);
int crtc_trace_any(crtc_renderer *r, const float *rays, uint64_t n, uint8_t *occluded);
/* Same kernels on DEVICE-resident rays, repeated `iters` times, returning the mean kernel time
 * in ms (CUDA events). For the roofline measurement of the traversal kernel in isolation. */
int crtc_bench_trace(crtc_renderer *r, const float *rays_host, uint64_t n, int any_hit, int iters,
                     float *ms_out);

/* Multi-GPU: device pointers of this rank's tile-local buffers, for the frame-end gather over
 * NVLink (torch.distributed / NCCL moves them; this library never touches the network).
 * accum: num_local_tiles*4096*3 floats; img: num_local_tiles*4096 RGBA8. */
int crtc_local_buffers(crtc_renderer *r, void **accum_dev, void **img_dev, uint32_t *num_local_tiles);
/* On the assembling rank: scatter one rank's gathered tile-local buffers (DEVICE pointers) into
 * the full row-major frame of this renderer. */
int crtc_assemble_rank(crtc_renderer *r, int src_rank, int world_size, const void *accum_dev,
                       const void *img_dev);
/* Multi-GPU without a gather (one process per GPU): the assembling rank exports its full-frame buffers
 * (handles_out: 128 bytes = two cudaIpcMemHandle_t, accum then img) and keeps writing its own tiles there; every
 * other rank imports them (ship the 128 bytes with any transport, e.g. torch.distributed.broadcast) and from then
 * on its frame-end resolve stores each of its pixels straight into the assembling rank's frame over NVLink, next to
 * its tile-local copy. Tile ownership is disjoint: nothing is reduced, no copy kernel runs, no collective library is
 * involved: the frame ends with a few flag words that travel through the same mapping — every rank's resolve kernel
 * publishes "frame s stored" there (system-scope fence + release store by its last block), the assembling rank's
 * stream waits for all of them before anything reads the frame (crtc_frame_wait; crtc_read_img / crtc_read_accum do it
 * themselves), and a rank does not store frame s + 1 before the assembling rank has started its own frame s + 1.
 * Every rank must therefore enqueue the same sequence of crtc_render / crtc_render_async calls; a flag that does not
 * arrive within 20 s becomes an error of the next synchronising call, not a hang.
 * crtc_initialize undoes both; crtc_import_frame(r, NULL) unmaps. */
int crtc_export_frame(crtc_renderer *r, void *handles_out);
int crtc_import_frame(crtc_renderer *r, const void *handles);
/* On the assembling rank of a shared frame (exported or crtc_share_frame'd): orders the renderer's stream after every
 * rank's stores of the last enqueued frame (a 1-warp kernel that spins on the flags). A no-op on other renderers. */
int crtc_frame_wait(crtc_renderer *r);
/* The same within ONE process (one host thread driving a renderer per GPU, as backends/cuda does for
 * CRT_CUDA_DEVICES): from now on `src` resolves its tiles into `dst`'s full frame; peer access between the two
 * devices is enabled if they differ. Both must be initialized with the same size; crtc_initialize undoes it. */
int crtc_share_frame(crtc_renderer *dst, crtc_renderer *src);
/* Presentation without a host round trip (SURVEY.md §8(f) rank 3): copies the assembled RGBA8 frame, device to device, into
 * a cudaArray_t (passed as void*: this header needs no CUDA types) — the mapped array of an OpenGL texture registered with
 * cudaGraphicsGLRegisterImage, as the reference's OptiX backend presents (backends/optix/render_optix.cpp:410-426). The
 * array must live on this renderer's device and be fb_width x fb_height RGBA8. Returns when the copy has completed. */
int crtc_copy_img_to_array(crtc_renderer *r, void *cuda_array);
/* Read the assembled full frame (after crtc_assemble_rank for every rank, after every rank's peer-written
 * frame has completed, or after a world_size==1 render). */
int crtc_read_img(crtc_renderer *r, uint32_t *img);

/* Option "aov": the accumulated first-hit AOVs, fb_width*fb_height*10 floats, row-major, per pixel: albedo.rgb, coverage,
 * normal.xyz, depth, lum_m1, lum_m2. Each is a running mean over the frames since the last reset (crtc_initialize,
 * crtc_set_scene, camera_changed), with crtc_read_accum's formula, of the frame's mean over its spp samples:
 *   albedo    the base colour of the primary hit as the shading kernel unpacks it; the miss shader's colour on a miss
 *   coverage  the fraction of samples that hit geometry
 *   normal    the shading normal of the hit, face-forwarded as the shading kernel does it (0 on a miss); not renormalised
 *   depth     the hit distance along the primary ray, averaged over the samples that hit (0 if none did)
 *   lum_m1/2  mean of L and of L^2 over the samples, L = 0.2126 r + 0.7152 g + 0.0722 b of a sample's radiance
 * Fails if the option is off or no frame has been rendered since the last reset. */
int crtc_read_aov(crtc_renderer *r, float *out);

typedef struct crtc_denoise_params_t {
    int iterations;        /* K, 1..10 (default 5): a-trous steps 1, 2, 4, ... 2^(K-1) pixels */
    float sigma_luminance; /* default 4:   w_l = exp(-|l_p - l_q| / (sigma_luminance * sqrt(blurred variance) + 1e-10)) */
    float sigma_normal;    /* default 128: w_n = max(0, dot(n_p, n_q))^sigma_normal */
    float sigma_depth;     /* default 1:   w_z = exp(-|Z_p - Z_q| / (sigma_depth * |grad Z_p . step offset| + 1e-3)) */
} crtc_denoise_params_t;

/* Edge-aware a-trous denoiser over the accumulated frame (the spatial part of SVGF, Schied et al. 2017; the temporal part,
 * below, only with option "denoise_history"). Needs option "aov" and a frame, like crtc_read_aov.
 *   1. I = accum / max(albedo, 1e-3) per channel; v = max(0, lum_m2 - lum_m1^2) / (spp * frames accumulated).
 *   2. K iterations i = 0..K-1 with step h = 2^i over a 5x5 B3-spline kernel (1,4,6,4,1)/16 per axis, taps outside the
 *      image skipped, dy outer and dx inner. Per tap q of pixel p: w = k * w_l * w_n * w_z, where the luminance weight
 *      uses g_p = the 3x3 (1,2,1)x(1,2,1)/16 blur of v at p (normalised over the taps inside the image), the normal
 *      weight uses unit normals (1 if both pixels have no normal, 0 if exactly one has none) and the depth weight uses
 *      the central difference of the depth (one-sided at the borders) dotted with h*(dx, dy).
 *      I' = sum w I_q / sum w, v' = sum w^2 v_q / (sum w)^2.
 *   3. rgb = I' * max(albedo, 1e-3), img = its sRGB8 conversion (as the frame's own img), alpha 255.
 * params: NULL = the defaults; out of range (iterations outside 1..10, a sigma not finite or <= 0) is an error.
 * Outputs, each optional: rgb_out (HOST, fb_width*fb_height*3 floats), img_out (HOST, fb_width*fb_height RGBA8),
 * cuda_array (a cudaArray_t, as crtc_copy_img_to_array). All work runs on the renderer's stream (crtc_set_stream); returns
 * when the outputs are written. Scratch buffers (72 B per pixel) are allocated by the first call after crtc_initialize.
 *
 * Temporal history (option "denoise_history" = H > 0; SVGF's temporal half over a static scene). An epoch is the run of
 * frames since an accumulation reset (crtc_initialize, crtc_set_scene, a render with camera_changed); the renderer keeps
 * the camera of each epoch's first frame. Two history buffers of 10 floats per pixel, `prev` and `cur`, hold
 * (I.rgb, M1, M2, n, z, nhat.xyz): integrated demodulated colour, integrated luminance moments, the samples they
 * represent, and the depth and unit normal of step 1. A call in epoch e first turns `cur` into `prev` if `cur` was written
 * in an earlier epoch, so `prev` is the output of the last call of the latest earlier epoch that had one; every call
 * overwrites `cur`. crtc_initialize and crtc_set_scene drop both, and so does crtc_commit_scene without option
 * denoise_motion. Between steps 1 and 2 above, per pixel p = (x, y):
 *   a. N = spp * frames accumulated (as in step 1). n_p = 0 if there is no `prev` or p's coverage is 0. Otherwise:
 *   b. d = normalize(du * ((x + 0.5) / w) + dv * ((y + 0.5) / h) + tl) with the current camera's basis (the primary ray
 *      expression at jitter 0.5), X = pos + z * d, z = p's AOV depth.
 *   b'. Option denoise_motion, only when geometry moved (a commit with instances or vertices) since `prev` was written:
 *      the renderer keeps, per pixel, the leaf-order triangle and barycentrics (b1, b2) of the first sample of the
 *      epoch's first frame, in sample order, that hit geometry; with each history buffer, a copy of the instance matrices
 *      and vertices it was written under. If p has such a record and the triangle's world vertices w0, w1, w2 now differ
 *      (as bits) from w0', w1', w2' under prev's copy: X is replaced by X + (P' - P), P = w0 + b1 (w1 - w0) + b2 (w2 - w0)
 *      and P' the same over w'; in step c the normal test uses s * n' in place of nhat_p, n' = the triangle's shading
 *      normal under prev's copy, s = -1 if dot(nhat_p, n) < 0 for its current shading normal n, else 1; a non-finite
 *      P' - P gives n_p = 0. Every other pixel (no record, or a triangle that did not move) follows b and c unchanged,
 *      bit for bit. Without moved geometry, the option changes no bit of the output.
 *   c. (alpha, beta, gamma) = M'^-1 (X - pos') with M' = [du' | dv' | tl'] of prev's camera (inverted in double, rounded to
 *      float). Needs gamma > 0; then sx = (alpha / gamma) * w - 0.5, sy = (beta / gamma) * h - 0.5 and the 2x2 taps q
 *      around (sx, sy) get bilinear weights. A tap is valid when it is inside the image, prev's normal at q is nonzero,
 *      |z_q - |X - pos'|| <= 0.02 |X - pos'| + 2 (|gx_q| + |gy_q|) (g = prev's depth gradient at q, as in step 2) and
 *      dot(nhat_p, nhat_q) >= 0.9. W = the sum of the valid taps' weights; if W < 0.01, n_p = 0, else
 *      P = sum w prev_q / W for I.rgb, M1, M2 and n_p = min(H, sum w n_q / W).
 *   d. n_t = n_p + N; I_t = (n_p P_I + N I) / n_t with I of step 1, and the same for M1, M2 with lum_m1, lum_m2. Where
 *      n_p = 0 nothing is blended: I_t = I, M_t = lum_m, n_t = N. cur = (I_t, M1_t, M2_t, n_t, z, nhat); I = I_t.
 *   e. v = max(0, M2_t - M1_t^2) / n_t where n_t >= 4. Where n_t < 4, M1_t and M2_t are first replaced by their mean over
 *      the 7x7 neighbourhood (taps outside the image skipped) weighted by w_n * w_z of step 2 at h = 1 (this call's
 *      sigma_normal, sigma_depth; no luminance or kernel weight): a 1-spp frame gets a nonzero variance.
 * The history holds the integrated colour before filtering, so with a still camera its weight n_p / (n_p + N) falls as
 * frames accumulate and the output converges to the history-off result. Without history in a pixel and with N >= 4, the
 * output is bit-identical to the history-off denoiser's. */
int crtc_denoise(crtc_renderer *r, const crtc_denoise_params_t *params, float *rgb_out, uint32_t *img_out, void *cuda_array);

/* Option "denoise_history": `cur`, fb_width*fb_height*10 floats, row-major (I.rgb, M1, M2, n, z, nhat.xyz per pixel, as
 * in crtc_denoise). Fails if the option is off or no crtc_denoise has run since the last reset. */
int crtc_read_denoise_history(crtc_renderer *r, float *out);

typedef struct crtc_adaptive_params_t {
    float threshold;     /* a block stops when its error E_b is <= threshold (finite, >= 0) */
    uint32_t min_frames; /* >= 1: frames every block renders before its error is trusted */
    uint32_t max_frames; /* 0 = no cap, else >= min_frames: no block renders more frames */
} crtc_adaptive_params_t;

/* Adaptive sampling: pixel blocks whose noise estimate has converged stop tracing. Off by default; params = NULL turns it
 * off. Takes effect at the next crtc_render / crtc_render_async call. Out-of-range params are an error, and so is a
 * renderer initialized with option "aov" (the AOVs and the denoiser assume the same samples in every pixel);
 * crtc_initialize with option aov fails while the mode is set.
 *   Block. Block b is the 32 local pixels 32b .. 32b+31 in local order: an 8x4 screen rectangle aligned to the 64x64 tile
 *   grid. It keeps c_b, the frames it has accumulated since the last reset (crtc_initialize, crtc_set_scene, a render
 *   with camera_changed), and per pixel m1, m2: the running means of L and L^2 over the samples (L and the fold of
 *   crtc_read_aov's lum_m1 / lum_m2, with the block's count in place of the frame index), so that they equal lum_m1 /
 *   lum_m2 of a uniform render with option aov at the same count.
 *   Pixel error. With N = c_b * spp: e_p = sqrt(max(0, m2 - m1^2) / (N * max(m1, 1e-4))), in float (+inf where N = 0): the
 *   standard error of the mean relative to sqrt(luminance). Block error E_b = the max of e_p over its in-frame pixels.
 *   Selection, once per crtc_render / crtc_render_async call (one wavefront of F frames), from the state at that moment:
 *   a block with no in-frame pixel gets n_b = 0; otherwise n_b = F if c_b < min_frames, or E_b > threshold, or the call is
 *   a crtc_render while option any_far_first = 2 has not decided (its trial compares the traversal time of two frames,
 *   which must see the same work); else n_b = 0. With max_frames > 0, n_b is capped at max_frames - c_b.
 *   Rendering. Only the samples of a block's frames k < n_b are traced, seeded as frame c_b + k of the uniform render;
 *   the block folds them into accum with c_b in place of the frame index, then c_b += n_b. A block with n_b = 0 leaves
 *   its accum, img and moments, and its pixels of a shared full frame, untouched.
 *   Guarantee. A pixel whose block has count c holds the accum and img that a uniform render with the same camera holds
 *   after c frames, bit for bit.
 *   Epochs. The counts are used from the first adaptive call after a reset until the next reset. Switching the mode off
 *   in between keeps them and makes every in-frame block active (n_b = F), so the guarantee still holds. Switching it on
 *   after c0 uniform frames of an epoch starts every count at c0 and the moments with that call: there N = (c_b - c0) *
 *   spp, the moments fold with c_b - c0, and min_frames counts from c0.
 *   Batches. A crtc_render_async call of F frames is one selection: per pixel the result is that of c_b frames, as above,
 *   but which blocks advance may differ from F separate calls.
 *   Stats. num_rays and counter [5] (paths started) count what was traced; counter [2] (launches) grows by 1 per call
 *   for the selection kernel. Memory: 12 B per block and 8 B per local pixel, + 8 B per framebuffer pixel for the
 *   first crtc_read_adaptive. */
int crtc_set_adaptive(crtc_renderer *r, const crtc_adaptive_params_t *params);

/* Adaptive sampling: per pixel, row-major fb_width*fb_height, the samples accumulated (c_b * spp) and e_p; either output
 * may be NULL. Pixels of tiles this renderer does not own are left untouched, as crtc_read_img leaves them. Fails if no
 * frame has been rendered with adaptive sampling since the last reset. */
int crtc_read_adaptive(crtc_renderer *r, uint32_t *samples_out, float *error_out);

#ifdef __cplusplus
}
#endif

#endif
