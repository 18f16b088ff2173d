"""Host-side mirror of ChameleonRT's ``RenderBackend`` for the CUDA wavefront path tracer.

``RenderCUDA`` has the reference's backend surface (util/render_backend.h:12-32): ``name()``,
``initialize(fb_width, fb_height)``, ``set_scene(scene)``,
``render(pos, dir, up, fovy, camera_changed, readback_framebuffer) -> RenderStats`` and the
public ``img`` / ``samples_per_pixel`` members — bound with ctypes to the C ABI of
``include/crt_cuda.h`` (``libcrt_cuda_core.so``). The C++ twin that ChameleonRT itself loads is
``backends/cuda/render_cuda.cpp``; both go through exactly the same entry points.

There is no CPU fallback: if the CUDA extension is missing or no GPU is usable, construction
raises ``RuntimeError``.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

from .scene import CQuadLight, CRenderStats, CScene, RenderStats, Scene

_CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc")
_LIB_PATH = os.path.join(_CSRC, "libcrt_cuda_core.so")
_lib: Optional[C.CDLL] = None

STAGE_NAMES = ("raygen", "traverse_primary", "shade", "traverse", "nee_resolve", "resolve", "frame")
COUNTER_NAMES = ("closest_rays", "occlusion_rays", "kernel_launches", "closest_nodes_visited", "closest_tris_tested",
                 "paths", "any_nodes_visited", "any_tris_tested")
SCENE_INFO_NAMES = ("triangles", "bvh8_nodes", "bvh8_depth", "bvh_build_ms", "node_bytes", "triangle_bytes",
                    "flatten_ms", "sort_ms", "tree_ms", "emit_ms", "pack_ms", "ploc_rounds")

# Every symbol include/crt_cuda.h declares (tests check the library exports all of them).
C_ABI_SYMBOLS = (
    "crtc_last_error", "crtc_name", "crtc_create", "crtc_destroy", "crtc_set_option", "crtc_get_option", "crtc_set_stream",
    "crtc_initialize", "crtc_set_scene", "crtc_render", "crtc_render_async", "crtc_sync", "crtc_read_accum", "crtc_get_stage_times",
    "crtc_get_counters", "crtc_get_scene_info", "crtc_trace_closest", "crtc_trace_any", "crtc_bench_trace",
    "crtc_local_buffers", "crtc_assemble_rank", "crtc_export_frame", "crtc_import_frame", "crtc_share_frame", "crtc_read_img", "crtc_frame_wait", "crtc_copy_img_to_array",
    "crtc_read_aov", "crtc_denoise", "crtc_read_denoise_history", "crtc_set_adaptive", "crtc_read_adaptive",
    "crtc_update_instances", "crtc_update_vertices", "crtc_update_lights", "crtc_commit_scene",
    "crtc_render_views", "crtc_read_view",
)
# Per-pixel layout of crtc_read_aov: name -> (first float, number of floats)
AOV_LAYOUT = {"albedo": (0, 3), "coverage": (3, 1), "normal": (4, 3), "depth": (7, 1), "lum_m1": (8, 1), "lum_m2": (9, 1)}
AOV_FLOATS = 10
# Per-pixel layout of crtc_read_denoise_history
HISTORY_LAYOUT = {"color": (0, 3), "lum_m1": (3, 1), "lum_m2": (4, 1), "count": (5, 1), "depth": (6, 1), "normal": (7, 3)}
HISTORY_FLOATS = 10


class CDenoiseParams(C.Structure):
    """crtc_denoise_params_t"""
    _fields_ = [("iterations", C.c_int), ("sigma_luminance", C.c_float), ("sigma_normal", C.c_float),
                ("sigma_depth", C.c_float)]


class CAdaptiveParams(C.Structure):
    """crtc_adaptive_params_t"""
    _fields_ = [("threshold", C.c_float), ("min_frames", C.c_uint32), ("max_frames", C.c_uint32)]


class CView(C.Structure):
    """crtc_view_t"""
    _fields_ = [("pos", C.c_float * 3), ("dir", C.c_float * 3), ("up", C.c_float * 3), ("fovy", C.c_float),
                ("camera_changed", C.c_int)]


def lib_path() -> str:
    return _LIB_PATH


def load_lib() -> C.CDLL:
    """Loads libcrt_cuda_core.so (built in-tree by ``__graft_entry__.build()``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise RuntimeError(
            f"{_LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). The CUDA backend has no CPU fallback.")
    lib = C.CDLL(_LIB_PATH)
    fp = C.POINTER(C.c_float)
    vp = C.c_void_p
    lib.crtc_last_error.restype = C.c_char_p
    lib.crtc_name.restype = C.c_char_p
    lib.crtc_create.argtypes = [C.POINTER(vp), C.c_int]
    lib.crtc_destroy.argtypes = [vp]
    lib.crtc_destroy.restype = None
    lib.crtc_set_option.argtypes = [vp, C.c_char_p, C.c_int64]
    lib.crtc_get_option.argtypes = [vp, C.c_char_p, C.POINTER(C.c_int64)]
    lib.crtc_set_stream.argtypes = [vp, vp]
    lib.crtc_initialize.argtypes = [vp, C.c_int, C.c_int]
    lib.crtc_set_scene.argtypes = [vp, C.POINTER(CScene)]
    lib.crtc_render.argtypes = [vp, fp, fp, fp, C.c_float, C.c_int, C.c_int, vp, C.POINTER(CRenderStats)]
    lib.crtc_render_async.argtypes = [vp, fp, fp, fp, C.c_float, C.c_int, C.c_uint32]
    lib.crtc_sync.argtypes = [vp, C.POINTER(CRenderStats), vp, vp, C.POINTER(C.c_uint32)]
    lib.crtc_read_accum.argtypes = [vp, vp]
    lib.crtc_read_img.argtypes = [vp, vp]
    lib.crtc_frame_wait.argtypes = [vp]
    lib.crtc_get_stage_times.argtypes = [vp, vp, C.c_int]
    lib.crtc_get_counters.argtypes = [vp, vp, C.c_int]
    lib.crtc_get_scene_info.argtypes = [vp, vp, C.c_int]
    lib.crtc_trace_closest.argtypes = [vp, vp, C.c_uint64, vp]
    lib.crtc_trace_any.argtypes = [vp, vp, C.c_uint64, vp]
    lib.crtc_bench_trace.argtypes = [vp, vp, C.c_uint64, C.c_int, C.c_int, fp]
    lib.crtc_local_buffers.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(C.c_uint32)]
    lib.crtc_assemble_rank.argtypes = [vp, C.c_int, C.c_int, vp, vp]
    lib.crtc_export_frame.argtypes = [vp, C.c_char_p]
    lib.crtc_import_frame.argtypes = [vp, C.c_char_p]
    lib.crtc_share_frame.argtypes = [vp, vp]
    lib.crtc_read_aov.argtypes = [vp, vp]
    lib.crtc_denoise.argtypes = [vp, C.POINTER(CDenoiseParams), vp, vp, vp]
    lib.crtc_read_denoise_history.argtypes = [vp, vp]
    lib.crtc_set_adaptive.argtypes = [vp, C.POINTER(CAdaptiveParams)]
    lib.crtc_read_adaptive.argtypes = [vp, vp, vp]
    lib.crtc_update_instances.argtypes = [vp, C.c_uint32, C.c_uint32, vp]
    lib.crtc_update_vertices.argtypes = [vp, C.c_uint32, C.c_uint32, vp, C.c_uint32]
    lib.crtc_update_lights.argtypes = [vp, vp, C.c_uint32]
    lib.crtc_commit_scene.argtypes = [vp]
    lib.crtc_render_views.argtypes = [vp, C.POINTER(CView), C.c_uint32, C.c_uint32]
    lib.crtc_read_view.argtypes = [vp, C.c_uint32, vp, vp]
    _lib = lib
    return lib


def _vec3(v):
    a = np.ascontiguousarray(v, dtype=np.float32).reshape(3)
    return a, a.ctypes.data_as(C.POINTER(C.c_float))


class RenderCUDA:
    """``RenderBackend`` implemented by the H100 wavefront path tracer."""

    def __init__(self, device: int = 0, max_depth: int = 5, rank: int = 0, world_size: int = 1,
                 count_traversal: bool = False, bvh_threads: int = 0, stream: Optional[int] = None,
                 any_far_first: Optional[int] = None, bvh_builder: Optional[str] = None,
                 tri_pass_defer: Optional[int] = None, shade_sort: Optional[int] = None, aov: bool = False,
                 denoise_history: int = 0, dynamic_scene: bool = False, denoise_motion: bool = False, views: int = 1):
        self.lib = load_lib()
        self.h = C.c_void_p()
        self._check(self.lib.crtc_create(C.byref(self.h), device))
        self.device = device
        self.rank, self.world_size = rank, world_size
        self.max_depth = max_depth
        for key, val in (("max_depth", max_depth), ("world_size", world_size), ("rank", rank),
                         ("count_traversal", int(count_traversal)), ("bvh_threads", bvh_threads)):
            self._check(self.lib.crtc_set_option(self.h, key.encode(), val))
        # developer knobs of the traversal kernels (defaults are the tuned values)
        for env, key in (("CRT_CUDA_REFILL_IDLE", "refill_idle"), ("CRT_CUDA_ANY_FAR_FIRST", "any_far_first"),
                         ("CRT_CUDA_PLOC_RADIUS", "bvh_ploc_radius"), ("CRT_CUDA_TRI_PASS_DEFER", "tri_pass_defer"),
                         ("CRT_CUDA_SHADE_SORT", "shade_sort"), ("CRT_CUDA_HW_TEXTURES", "hw_textures")):
            if os.environ.get(env):
                self._check(self.lib.crtc_set_option(self.h, key.encode(), int(os.environ[env])))
        # CRT_CUDA_OPTIONS="key=value,key=value": any crtc_set_option key (experiments, profiling runs)
        for kv in filter(None, os.environ.get("CRT_CUDA_OPTIONS", "").split(",")):
            key, val = kv.split("=")
            self._check(self.lib.crtc_set_option(self.h, key.strip().encode(), int(val)))
        if tri_pass_defer is not None:  # 0 / 16 / 24: experimental scheduling variant of k_traverse; never changes a result
            self._check(self.lib.crtc_set_option(self.h, b"tri_pass_defer", int(tri_pass_defer)))
        if shade_sort is not None:  # 0 / 1 / 2: shade queue bucketed by material id before k_shade; never changes a result
            self._check(self.lib.crtc_set_option(self.h, b"shade_sort", int(shade_sort)))
        if any_far_first is not None:  # 0 / 1 / 2 = auto: traversal order of shadow rays; never changes a result (crt_cuda.h)
            self._check(self.lib.crtc_set_option(self.h, b"any_far_first", int(any_far_first)))
        # where set_scene builds the BVH8: "host" (binned SAH, the default), "device" (PLOC on the GPU: much faster
        # set_scene, a somewhat slower tree) or "device_lbvh" (plain Morton-order LBVH: faster still, slower tree);
        # the rendered image is the same in every case (crt_cuda.h)
        bvh_builder = bvh_builder or os.environ.get("CRT_CUDA_BVH_BUILDER")
        if bvh_builder is not None:
            names = ("host", "device", "device_lbvh")
            bvh_builder = {"0": names[0], "1": names[1], "2": names[2]}.get(str(bvh_builder), bvh_builder)  # the plugin's env var is numeric
            if bvh_builder not in names:
                raise ValueError(f"bvh_builder must be one of {names}")
            self._check(self.lib.crtc_set_option(self.h, b"bvh_builder", names.index(bvh_builder)))
        if aov:  # first-hit AOVs with every frame, for read_aov() and denoise() (crt_cuda.h: option "aov")
            self._check(self.lib.crtc_set_option(self.h, b"aov", 1))
        if denoise_history:  # denoise() carries a reprojected history of up to this many samples (option "denoise_history")
            self._check(self.lib.crtc_set_option(self.h, b"denoise_history", int(denoise_history)))
        if dynamic_scene:  # set_scene keeps what update_instances / update_vertices + commit_scene need (option "dynamic_scene")
            self._check(self.lib.crtc_set_option(self.h, b"dynamic_scene", 1))
        if denoise_motion:  # commit_scene keeps denoise()'s history, moved with the geometry (option "denoise_motion")
            self._check(self.lib.crtc_set_option(self.h, b"denoise_motion", 1))
        if views != 1:  # cameras render_views traces together (option "views")
            self._check(self.lib.crtc_set_option(self.h, b"views", int(views)))
        if stream is not None:
            self._check(self.lib.crtc_set_stream(self.h, C.c_void_p(stream)))
        self.width = self.height = 0
        self.samples_per_pixel = 1
        self.img: Optional[np.ndarray] = None

    def _check(self, rc: int) -> None:
        if rc != 0:
            raise RuntimeError(self.lib.crtc_last_error().decode())

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.lib.crtc_destroy(self.h)
                self.h = None
        except Exception:
            pass

    # ---- RenderBackend ----
    def name(self) -> str:
        return self.lib.crtc_name().decode()

    def initialize(self, fb_width: int, fb_height: int) -> None:
        self._check(self.lib.crtc_initialize(self.h, fb_width, fb_height))
        self.width, self.height = fb_width, fb_height
        self.img = np.zeros((fb_height, fb_width), dtype=np.uint32)

    def set_scene(self, scene: Scene) -> None:
        ms = scene.to_c()
        self.samples_per_pixel = scene.samples_per_pixel
        self._check(self.lib.crtc_set_scene(self.h, C.byref(ms.c)))

    def set_scene_c(self, c_scene, samples_per_pixel: int = 1) -> None:
        """crtc_set_scene on a ``crt_scene_t`` that lives in native memory — what ``scene_io.load_obj(path).c_scene`` is —
        without a trip through the Python scene model."""
        c_scene.contents.samples_per_pixel = samples_per_pixel
        self.samples_per_pixel = samples_per_pixel
        self._check(self.lib.crtc_set_scene(self.h, c_scene))

    # ---- scene updates between frames (include/crt_cuda.h: crtc_update_instances ... crtc_commit_scene) ----
    def update_instances(self, transforms, first: int = 0) -> None:
        """Stages new object_to_world matrices for instances ``first`` .. ``first + n - 1``: (n, 4, 4) or (n, 16) in
        ``Instance.transform``'s layout (row i, column j). Needs ``dynamic_scene=True`` at the last set_scene."""
        m = np.asarray(transforms, dtype=np.float32).reshape(-1, 4, 4)
        col_major = np.ascontiguousarray(m.transpose(0, 2, 1))  # crt_instance_t::transform
        self._check(self.lib.crtc_update_instances(self.h, int(first), m.shape[0], col_major.ctypes.data))

    def update_vertices(self, mesh: int, geometry: int, vertices) -> None:
        """Stages new object-space positions (n, 3) for geometry ``geometry`` of mesh ``mesh``; n must be its vertex
        count at set_scene. Needs ``dynamic_scene=True`` at the last set_scene."""
        v = np.ascontiguousarray(vertices, dtype=np.float32).reshape(-1, 3)
        self._check(self.lib.crtc_update_vertices(self.h, int(mesh), int(geometry), v.ctypes.data if len(v) else None,
                                                  v.shape[0]))

    def update_lights(self, lights) -> None:
        """Stages a new list of ``QuadLight``s (the count may change)."""
        arr = (CQuadLight * max(1, len(lights)))()
        for i, l in enumerate(lights):
            raw = np.array(l.as_floats(), dtype=np.float32)
            C.memmove(C.addressof(arr[i]), raw.ctypes.data, 80)
        self._check(self.lib.crtc_update_lights(self.h, C.addressof(arr), len(lights)))

    def commit_scene(self) -> None:
        """Applies the staged updates on the renderer's stream: later frames see the updated scene, from a reset
        accumulation. Nothing staged: nothing happens."""
        self._check(self.lib.crtc_commit_scene(self.h))

    def render(self, pos, dir, up, fovy: float, camera_changed: bool, readback_framebuffer: bool = True) -> RenderStats:
        _p, pp = _vec3(pos)
        _d, dp = _vec3(dir)
        _u, up_ = _vec3(up)
        st = CRenderStats()
        img_ptr = self.img.ctypes.data if (readback_framebuffer and self.img is not None) else None
        self._check(self.lib.crtc_render(self.h, pp, dp, up_, C.c_float(fovy), 1 if camera_changed else 0,
                                         1 if readback_framebuffer else 0, img_ptr, C.byref(st)))
        return RenderStats(st.render_time, st.rays_per_second, st.num_rays)

    # ---- throughput variant: frames in flight (see include/crt_cuda.h) ----
    def render_async(self, pos, dir, up, fovy: float, camera_changed: bool, num_frames: int = 1) -> None:
        """Enqueues ``num_frames`` consecutive frames as one wavefront (bit-identical to that many
        ``render`` calls); returns immediately."""
        _p, pp = _vec3(pos)
        _d, dp = _vec3(dir)
        _u, up_ = _vec3(up)
        self._check(self.lib.crtc_render_async(self.h, pp, dp, up_, C.c_float(fovy), 1 if camera_changed else 0,
                                               num_frames))

    # ---- multi-view rendering (include/crt_cuda.h: crtc_render_views) ----
    def render_views(self, cameras, camera_changed=True, num_frames: int = 1) -> None:
        """Enqueues ``num_frames`` frames of every camera as one wavefront (needs ``views=len(cameras)``); returns
        immediately, ``sync()`` collects it. A camera is ``(pos, dir, up, fovy)`` or a dict with ``position`` (or ``eye``),
        ``center``, ``up`` and ``fov_y``, like ``scene_io.load_scene(path).cameras``. ``camera_changed``: one bool for
        every view or one per view. View k ends bit-identical to a one-view renderer given the same render_async calls."""
        from .camera import view_args

        n = len(cameras)
        flags = [bool(camera_changed)] * n if isinstance(camera_changed, (bool, int)) else [bool(c) for c in camera_changed]
        if len(flags) != n:
            raise ValueError("camera_changed: one flag per camera")
        arr = (CView * max(1, n))()
        for k, cam in enumerate(cameras):
            pos, d, up, fovy = view_args(cam)
            arr[k] = CView((C.c_float * 3)(*pos), (C.c_float * 3)(*d), (C.c_float * 3)(*up), float(fovy), int(flags[k]))
        self._check(self.lib.crtc_render_views(self.h, arr, n, int(num_frames)))

    def read_view(self, k: int):
        """View ``k`` of a multi-view renderer (crtc_read_view): (rgb (h, w, 3) float32, img (h, w) uint32 RGBA8)."""
        rgb = np.zeros((self.height, self.width, 3), dtype=np.float32)
        img = np.zeros((self.height, self.width), dtype=np.uint32)
        self._check(self.lib.crtc_read_view(self.h, int(k), rgb.ctypes.data, img.ctypes.data))
        return rgb, img

    def set_stream(self, cuda_stream: Optional[int]) -> None:
        """crtc_set_stream: the CUDA stream (a cudaStream_t as an integer) every later launch and copy of this renderer
        goes to; None = the renderer's own non-blocking stream."""
        self._check(self.lib.crtc_set_stream(self.h, C.c_void_p(cuda_stream)))

    def set_option(self, key: str, value: int) -> None:
        """crtc_set_option (include/crt_cuda.h lists the keys); options apply to the next set_scene / frame."""
        self._check(self.lib.crtc_set_option(self.h, key.encode(), int(value)))

    def get_option(self, key: str) -> int:
        v = C.c_int64(0)
        self._check(self.lib.crtc_get_option(self.h, key.encode(), C.byref(v)))
        return int(v.value)

    def sync(self):
        """Waits for all frames queued with render_async; returns (RenderStats totals, stage ms sums,
        counter sums, number of frames)."""
        st = CRenderStats()
        stages = np.zeros(len(STAGE_NAMES), dtype=np.float32)
        counters = np.zeros(len(COUNTER_NAMES), dtype=np.uint64)
        n = C.c_uint32(0)
        self._check(self.lib.crtc_sync(self.h, C.byref(st), stages.ctypes.data, counters.ctypes.data, C.byref(n)))
        return (RenderStats(st.render_time, st.rays_per_second, st.num_rays),
                {STAGE_NAMES[i]: float(stages[i]) for i in range(len(STAGE_NAMES))},
                {COUNTER_NAMES[i]: int(counters[i]) for i in range(len(COUNTER_NAMES))}, int(n.value))

    # ---- extra exports (SURVEY.md §8b) ----
    def read_accum(self) -> np.ndarray:
        out = np.zeros((self.height, self.width, 3), dtype=np.float32)
        self._check(self.lib.crtc_read_accum(self.h, out.ctypes.data))
        return out

    def read_img(self, out: Optional[np.ndarray] = None) -> np.ndarray:
        """The sRGB8 frame (crtc_read_img). ``out``: read into this (height, width) uint32 array instead of a new one —
        a frame loop that passes ``self.img`` every time gets a page-locked destination (option "pin_read_img")."""
        if out is None:
            out = np.zeros((self.height, self.width), dtype=np.uint32)
        assert out.dtype == np.uint32 and out.shape == (self.height, self.width) and out.flags["C_CONTIGUOUS"]
        self._check(self.lib.crtc_read_img(self.h, out.ctypes.data))
        return out

    def read_aov(self) -> dict:
        """The accumulated first-hit AOVs (crtc_read_aov; needs ``aov=True``): ``albedo`` (h, w, 3), ``coverage`` (h, w),
        ``normal`` (h, w, 3, the mean normal, not renormalised), ``depth`` (h, w), ``lum_m1`` / ``lum_m2`` (h, w: the
        mean of the sample luminance and of its square), all float32."""
        a = np.zeros((self.height, self.width, AOV_FLOATS), dtype=np.float32)
        self._check(self.lib.crtc_read_aov(self.h, a.ctypes.data))
        return {k: (a[:, :, o:o + n] if n > 1 else a[:, :, o]).copy() for k, (o, n) in AOV_LAYOUT.items()}

    def denoise(self, iterations: int = 5, sigma_luminance: float = 4.0, sigma_normal: float = 128.0,
                sigma_depth: float = 1.0):
        """Edge-aware à-trous denoiser over the accumulated frame (crtc_denoise; needs ``aov=True``). Returns
        (rgb (h, w, 3) float32, img (h, w) uint32 RGBA8)."""
        prm = CDenoiseParams(int(iterations), float(sigma_luminance), float(sigma_normal), float(sigma_depth))
        rgb = np.zeros((self.height, self.width, 3), dtype=np.float32)
        img = np.zeros((self.height, self.width), dtype=np.uint32)
        self._check(self.lib.crtc_denoise(self.h, C.byref(prm), rgb.ctypes.data, img.ctypes.data, None))
        return rgb, img

    def read_denoise_history(self) -> dict:
        """The history the last denoise() wrote (crtc_read_denoise_history; needs ``denoise_history`` > 0): ``color``
        (h, w, 3, integrated demodulated colour), ``lum_m1`` / ``lum_m2`` (h, w, integrated luminance moments), ``count``
        (h, w, the samples they represent), ``depth`` (h, w) and ``normal`` (h, w, 3, unit), all float32."""
        a = np.zeros((self.height, self.width, HISTORY_FLOATS), dtype=np.float32)
        self._check(self.lib.crtc_read_denoise_history(self.h, a.ctypes.data))
        return {k: (a[:, :, o:o + n] if n > 1 else a[:, :, o]).copy() for k, (o, n) in HISTORY_LAYOUT.items()}

    def set_adaptive(self, threshold: Optional[float], min_frames: int = 4, max_frames: int = 0) -> None:
        """Adaptive sampling (crtc_set_adaptive): from the next render call on, 8x4 pixel blocks whose relative error is at
        most ``threshold`` (after ``min_frames`` frames) stop tracing; ``max_frames`` > 0 caps every block's frames.
        ``set_adaptive(None)`` turns it off."""
        if threshold is None:
            self._check(self.lib.crtc_set_adaptive(self.h, None))
            return
        prm = CAdaptiveParams(float(threshold), int(min_frames), int(max_frames))
        self._check(self.lib.crtc_set_adaptive(self.h, C.byref(prm)))

    def read_adaptive(self) -> dict:
        """Per pixel (crtc_read_adaptive): ``samples`` (h, w) uint32, the samples accumulated, and ``error`` (h, w)
        float32, the pixel error e_p the selection uses. Pixels of other ranks' tiles read 0."""
        samples = np.zeros((self.height, self.width), dtype=np.uint32)
        error = np.zeros((self.height, self.width), dtype=np.float32)
        self._check(self.lib.crtc_read_adaptive(self.h, samples.ctypes.data, error.ctypes.data))
        return {"samples": samples, "error": error}

    def stage_times(self) -> dict:
        a = np.zeros(len(STAGE_NAMES), dtype=np.float32)
        n = self.lib.crtc_get_stage_times(self.h, a.ctypes.data, len(a))
        return {STAGE_NAMES[i]: float(a[i]) for i in range(n)}

    def counters(self) -> dict:
        a = np.zeros(len(COUNTER_NAMES), dtype=np.uint64)
        n = self.lib.crtc_get_counters(self.h, a.ctypes.data, len(a))
        return {COUNTER_NAMES[i]: int(a[i]) for i in range(n)}

    def scene_info(self) -> dict:
        a = np.zeros(len(SCENE_INFO_NAMES), dtype=np.float64)
        n = self.lib.crtc_get_scene_info(self.h, a.ctypes.data, len(a))
        return {SCENE_INFO_NAMES[i]: float(a[i]) for i in range(n)}

    def trace_closest(self, rays: np.ndarray) -> np.ndarray:
        rays = np.ascontiguousarray(rays, dtype=np.float32).reshape(-1, 8)
        hits = np.zeros((rays.shape[0], 4), dtype=np.float32)
        self._check(self.lib.crtc_trace_closest(self.h, rays.ctypes.data, rays.shape[0], hits.ctypes.data))
        return hits

    def trace_any(self, rays: np.ndarray) -> np.ndarray:
        rays = np.ascontiguousarray(rays, dtype=np.float32).reshape(-1, 8)
        occ = np.zeros(rays.shape[0], dtype=np.uint8)
        self._check(self.lib.crtc_trace_any(self.h, rays.ctypes.data, rays.shape[0], occ.ctypes.data))
        return occ

    def bench_trace(self, rays: np.ndarray, any_hit: bool = False, iters: int = 10) -> float:
        rays = np.ascontiguousarray(rays, dtype=np.float32).reshape(-1, 8)
        ms = C.c_float(0)
        self._check(self.lib.crtc_bench_trace(self.h, rays.ctypes.data, rays.shape[0], 1 if any_hit else 0, iters,
                                              C.byref(ms)))
        return float(ms.value)

    # ---- multi-GPU tile gather (SURVEY.md §8e) ----
    def local_buffers(self):
        """(accum device ptr, img device ptr, number of local 64x64 tiles)."""
        a, i, n = C.c_void_p(), C.c_void_p(), C.c_uint32()
        self._check(self.lib.crtc_local_buffers(self.h, C.byref(a), C.byref(i), C.byref(n)))
        return a.value, i.value, n.value

    def export_frame(self) -> bytes:
        """On the assembling rank: 128 bytes (two CUDA IPC handles) that let the other ranks' renderers write their
        tiles straight into this renderer's full frame (crtc_export_frame)."""
        buf = C.create_string_buffer(128)
        self._check(self.lib.crtc_export_frame(self.h, buf))
        return buf.raw

    def import_frame(self, handles: Optional[bytes]) -> None:
        """On every other rank: map the assembling rank's frame (crtc_import_frame); None unmaps."""
        if handles is not None and len(handles) != 128:
            raise ValueError("import_frame expects the 128 bytes of export_frame")
        self._check(self.lib.crtc_import_frame(self.h, handles))

    def frame_wait(self) -> None:
        """crtc_frame_wait: on the assembling rank of a shared frame, orders the stream after every rank's stores."""
        self._check(self.lib.crtc_frame_wait(self.h))

    def share_frame_with(self, src: "RenderCUDA") -> None:
        """In-process multi-GPU: ``src`` (another RenderCUDA of this process, same size) resolves its tiles into this
        renderer's full frame from now on (crtc_share_frame)."""
        self._check(self.lib.crtc_share_frame(self.h, src.h))

    def assemble_rank(self, src_rank: int, world_size: int, accum_dev_ptr: int, img_dev_ptr: int) -> None:
        self._check(self.lib.crtc_assemble_rank(self.h, src_rank, world_size, C.c_void_p(accum_dev_ptr),
                                                C.c_void_p(img_dev_ptr)))
