"""Multi-view rendering (option "views"; crtc_render_views, crtc_read_view; kernels.cuh: k_raygen_views, k_resolve_views).

Every check runs on the emulated renderer (tests/simt_emu) without a GPU and on libcrt_cuda_core.so on an H100 (``-m gpu``):
  * after every call of a sequence (single frames, a batch, camera_changed on one view only), each view's accum and img
    equal, bit for bit, those of a one-view renderer given that view's render_async calls; rays and paths are the sums of
    the one-view renderers', launches those of one of them;
  * with one view, render_views is render_async;
  * scene commits between calls reset every view, on the host and the device builder;
  * (GPU) hardware textures on a textured scene, and 8 views at 1280x720;
  * every refused combination and out-of-range argument is an error that leaves the renderer usable;
  * the Python surface renders the cameras of a .crts file.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from test_denoise_history import gpu  # noqa: F401 (a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "chameleonrt_b200", "csrc")


@pytest.fixture(scope="module")
def emu(built):
    """(RenderCUDA, OracleBackend, primary_rays) with RenderCUDA bound to the emulated renderer."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "simt_emu"))
    import build as simt_build

    lib = simt_build.LIB
    stale = not os.path.exists(lib) or any(os.path.getmtime(lib) < os.path.getmtime(os.path.join(CSRC, f))
                                           for f in ("kernels.cuh", "crt_cuda_core.cu", "adaptive.cuh", "aov_denoise.cuh"))
    lib_path = simt_build.build(force=stale)
    import chameleonrt_b200.backend as backend
    from oracle import OracleBackend
    from oracle.oracle import primary_rays

    saved = (backend._LIB_PATH, backend._lib)
    backend._LIB_PATH, backend._lib = lib_path, None
    yield backend.RenderCUDA, OracleBackend, primary_rays
    backend._LIB_PATH, backend._lib = saved


def _renderer(RenderCUDA, scene, w, h, max_depth=5, hw_textures=False, **kw):
    r = RenderCUDA(0, max_depth=max_depth, **kw)
    r.set_option("hw_textures", int(hw_textures))
    r.initialize(w, h)
    r.set_scene(scene)
    return r


def cameras(cam, n):
    """`n` distinct views of the scene `cam` looks at: the eye orbits the centre, the field of view varies."""
    e, c = np.asarray(cam["eye"], np.float64), np.asarray(cam["center"], np.float64)
    out = []
    for k in range(n):
        a = np.radians(-25.0 + 50.0 * k / max(1, n - 1))
        d = e - c
        d = np.array([np.cos(a) * d[0] + np.sin(a) * d[2], d[1] + 0.1 * k, -np.sin(a) * d[0] + np.cos(a) * d[2]])
        out.append(dict(eye=tuple(c + d), center=cam["center"], up=cam["up"], fov_y=cam["fov_y"] + 4.0 * k))
    return out


def _same(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


def run_and_compare(multi, singles, cams, calls, between=None):
    """Drives `multi` with render_views and singles[k] with render_async of cams[k]; after every call each view must equal
    its one-view renderer bit for bit. `between(i)` (optional) runs before call i on every renderer."""
    from chameleonrt_b200.camera import view_args

    V = len(cams)
    for i, (flags, frames) in enumerate(calls):
        if between is not None:
            between(i)
        multi.render_views(cams, flags, frames)
        tm, _, cm, nm = multi.sync()
        rays = paths = 0
        for k, s in enumerate(singles):
            s.render_async(*view_args(cams[k]), flags[k], frames)
            ts, _, cs, ns = s.sync()
            assert ns == frames
            rays += ts.num_rays
            paths += cs["paths"]
            launches = cs["kernel_launches"]
        assert nm == frames, i
        assert tm.num_rays == rays and cm["paths"] == paths, i
        assert cm["closest_rays"] + cm["occlusion_rays"] == rays, i
        assert cm["kernel_launches"] == launches, i
        for k, s in enumerate(singles):
            rgb, img = multi.read_view(k)
            assert _same(rgb, s.read_accum()), (i, k)
            assert np.array_equal(img, s.read_img()), (i, k)
    assert multi.get_option("views") == V


def check_bit_identity(RenderCUDA, scene, cam, w, h, V=3, max_depth=5, calls=None, **kw):
    cams = cameras(cam, V)
    multi = _renderer(RenderCUDA, scene, w, h, max_depth, views=V, **kw)
    singles = [_renderer(RenderCUDA, scene, w, h, max_depth, **kw) for _ in cams]
    if calls is None:
        # F = 1 twice, F = 2, camera_changed on view 1 only, F = 1
        calls = [([True] * V, 1), ([False] * V, 1), ([False] * V, 2), ([k == 1 for k in range(V)], 2), ([False] * V, 1)]
    run_and_compare(multi, singles, cams, calls)
    # the views differ from each other (distinct cameras)
    assert not _same(multi.read_view(0)[0], multi.read_view(V - 1)[0])


def check_one_view_is_render_async(RenderCUDA, scene, cam, w, h):
    from chameleonrt_b200.camera import view_args

    a, b = _renderer(RenderCUDA, scene, w, h), _renderer(RenderCUDA, scene, w, h)
    for flag, frames in ((True, 1), (False, 2), (True, 1)):
        a.render_views([cam], flag, frames)
        b.render_async(*view_args(cam), flag, frames)
        ta, _, ca, na = a.sync()
        tb, _, cb, nb = b.sync()
        assert na == nb == frames and ta.num_rays == tb.num_rays and ca == cb
        rgb, img = a.read_view(0)
        assert _same(rgb, a.read_accum()) and np.array_equal(img, a.read_img())
        assert _same(rgb, b.read_accum()) and np.array_equal(img, b.read_img())


def check_scene_commits(RenderCUDA, scene, cam, w, h, builder):
    from chameleonrt_b200.scene import QuadLight

    V = 3
    cams = cameras(cam, V)
    kw = dict(dynamic_scene=True, bvh_builder=builder)
    multi = _renderer(RenderCUDA, scene, w, h, views=V, **kw)
    singles = [_renderer(RenderCUDA, scene, w, h, **kw) for _ in cams]
    light = scene.lights[0]

    def move(i):
        if i == 0:
            return
        xf = np.eye(4, dtype=np.float32)
        xf[:3, 3] = (0.05 * i, 0.0, -0.03 * i)
        moved = QuadLight(emission=light.emission, position=tuple(np.asarray(light.position, np.float32) + np.float32(0.02 * i)),
                          normal=light.normal, v_x=light.v_x, width=light.width, v_y=light.v_y, height=light.height)
        for r in [multi] + singles:
            r.update_instances(xf[None])
            if i == 2:
                r.update_lights([moved])
            r.commit_scene()

    # (no camera_changed after a commit: a view that the commit did not reset would differ from its one-view renderer)
    calls = [([True] * V, 1), ([False] * V, 1), ([False] * V, 2), ([False, True, False], 1)]
    run_and_compare(multi, singles, cams, calls, between=move)


def check_refusals(RenderCUDA, scene, cam, w=40, h=24):
    from chameleonrt_b200.scenes import cornell_box

    V = 2
    cams = cameras(cam, V)
    # the option
    r = RenderCUDA(0, max_depth=3)
    assert r.get_option("views") == 1
    for bad in (0, 65, -1):
        with pytest.raises(RuntimeError, match="views must be in"):
            r.set_option("views", bad)
    r.set_option("views", 64)
    assert r.get_option("views") == 64
    # initialize: aov, world_size > 1, adaptive sampling; each refusal leaves a renderer that initializes without it
    r = RenderCUDA(0, max_depth=3, views=V)
    for key, val, msg in (("aov", 1, "aov"), ("world_size", 2, "world_size 1")):
        r.set_option(key, val)
        with pytest.raises(RuntimeError, match=f"views = {V} .*{msg}"):
            r.initialize(w, h)
        r.set_option(key, 0 if key == "aov" else 1)
    r.set_adaptive(0.1)
    with pytest.raises(RuntimeError, match=f"views = {V} .*adaptive"):
        r.initialize(w, h)
    r.set_adaptive(None)
    r.initialize(w, h)
    r.set_scene(scene)
    with pytest.raises(RuntimeError, match="crtc_set_adaptive: .*crtc_render_views"):
        r.set_adaptive(0.1)
    r.set_adaptive(None)  # (switching it off is not refused)
    # the one-view calls
    other = _renderer(RenderCUDA, scene, w, h, 3)
    lib, h_ = r.lib, r.h
    calls = {
        "crtc_render": lambda: r.render(cams[0]["eye"], (0, 0, -1), (0, 1, 0), 40.0, True),
        "crtc_render_async": lambda: r.render_async(cams[0]["eye"], (0, 0, -1), (0, 1, 0), 40.0, True, 1),
        "crtc_read_accum": r.read_accum,
        "crtc_read_img": r.read_img,
        "crtc_copy_img_to_array": lambda: r._check(lib.crtc_copy_img_to_array(h_, C.c_void_p(1))),
        "crtc_export_frame": r.export_frame,
        "crtc_import_frame": lambda: r.import_frame(None),
        "crtc_local_buffers": r.local_buffers,
        "crtc_assemble_rank": lambda: r.assemble_rank(0, 1, 0, 0),
        "crtc_share_frame": lambda: r.share_frame_with(other),
    }
    for name, call in calls.items():
        with pytest.raises(RuntimeError, match=f"{name}: .*views = {V}.*crtc_render_views"):
            call()
    with pytest.raises(RuntimeError, match="crtc_share_frame: .*views"):
        other.share_frame_with(r)
    # arguments of the view calls
    with pytest.raises(RuntimeError, match=f"num_views = 3 differs from option views = {V}"):
        r.render_views(cameras(cam, 3))
    for bad in (0, 65):
        with pytest.raises(RuntimeError, match="num_frames must be in"):
            r.render_views(cams, True, bad)
    with pytest.raises(RuntimeError, match="views is NULL"):
        r._check(lib.crtc_render_views(h_, None, V, 1))
    with pytest.raises(RuntimeError, match=f"view {V} is out of range"):
        r.read_view(V)
    assert lib.crtc_read_view(h_, 0, None, None) == 0  # both outputs are optional
    for rc in (lib.crtc_render_views(None, None, 1, 1), lib.crtc_read_view(None, 0, None, None)):
        assert rc != 0 and b"NULL" in lib.crtc_last_error()
    # more than 2^31 paths: 64 views x 64 frames x 16 spp x 16 tiles of 4096 pixels
    big_scene, _ = cornell_box(spp=16)
    big = _renderer(RenderCUDA, big_scene, 256, 256, 3, views=64)
    with pytest.raises(RuntimeError, match="2\\^31 paths"):
        big.render_views(cameras(cam, 64), True, 64)
    del big
    # still usable: the same sequence as a one-view renderer per view
    singles = [_renderer(RenderCUDA, scene, w, h, 3) for _ in cams]
    run_and_compare(r, singles, cams, [([True] * V, 1), ([False] * V, 2)])


def check_crts_cameras(RenderCUDA, tmp_path, w, h):
    """render_views on a .crts file's cameras (scene_io.load_scene(...).cameras) equals one one-view render per camera."""
    pytest.importorskip("PIL")
    from chameleonrt_b200 import scene_io
    from chameleonrt_b200.camera import view_args
    from chameleonrt_b200.crts_io import write_crts
    from chameleonrt_b200.scenes import cornell_box

    scene, cam = cornell_box(spp=1)

    def look_at(eye, center, fov):
        eye, center = np.asarray(eye, np.float64), np.asarray(center, np.float64)
        f = (center - eye) / np.linalg.norm(center - eye)
        r = np.cross(f, (0.0, 1.0, 0.0))
        r /= np.linalg.norm(r)
        u = np.cross(r, f)
        m = np.eye(4)
        m[:3, 0], m[:3, 1], m[:3, 2], m[:3, 3] = r, u, -f, eye
        return dict(type="CAMERA", fov_y=fov, matrix=[float(np.float32(x)) for x in m.T.reshape(-1)])

    extra = [look_at(c["eye"], c["center"], c["fov_y"]) for c in cameras(cam, 3)]
    path = write_crts(scene, str(tmp_path / "views.crts"), extra_objects=extra)
    loaded = scene_io.load_scene(path)
    assert len(loaded.cameras) == 3
    multi = RenderCUDA(0, max_depth=5, views=3)
    multi.initialize(w, h)
    multi.set_scene_c(loaded.c_scene, 1)
    multi.render_views(loaded.cameras)
    multi.sync()
    multi.render_views(loaded.cameras, [False, True, False], 2)
    multi.sync()
    for k, c in enumerate(loaded.cameras):
        one = RenderCUDA(0, max_depth=5)
        one.initialize(w, h)
        one.set_scene_c(loaded.c_scene, 1)
        one.render_async(*view_args(c), True, 1)
        one.render_async(*view_args(c), k == 1, 2)
        one.sync()
        rgb, img = multi.read_view(k)
        assert _same(rgb, one.read_accum()) and np.array_equal(img, one.read_img()), k
    # the tuple form of a camera
    args = [view_args(c) for c in loaded.cameras]
    multi.render_views(args, True, 1)
    multi.sync()
    one = RenderCUDA(0, max_depth=5)
    one.initialize(w, h)
    one.set_scene_c(loaded.c_scene, 1)
    one.render_async(*args[2], True, 1)
    one.sync()
    assert _same(multi.read_view(2)[0], one.read_accum())
    with pytest.raises(ValueError, match="one flag per camera"):
        multi.render_views(args, [True, False])


# ---- CPU: the emulated renderer ----
def test_views_equal_one_view_renderers_on_the_emulated_renderer(emu):
    from chameleonrt_b200.scenes import cornell_box

    check_bit_identity(emu[0], *cornell_box(spp=2), 150, 90)


def test_one_view_is_render_async_on_the_emulated_renderer(emu):
    from chameleonrt_b200.scenes import cornell_box

    check_one_view_is_render_async(emu[0], *cornell_box(spp=2), 70, 42)


@pytest.mark.parametrize("builder", ["host", "device"])
def test_scene_commits_reset_every_view_on_the_emulated_renderer(emu, builder):
    from chameleonrt_b200.scenes import cornell_box

    check_scene_commits(emu[0], *cornell_box(spp=1), 70, 42, builder)


def test_refusals_on_the_emulated_renderer(emu):
    from chameleonrt_b200.scenes import cornell_box

    check_refusals(emu[0], *cornell_box(spp=1))


def test_crts_cameras_on_the_emulated_renderer(emu, tmp_path):
    check_crts_cameras(emu[0], tmp_path, 70, 42)


# ---- GPU: libcrt_cuda_core.so on the H100 ----
@pytest.mark.gpu
def test_views_equal_one_view_renderers(gpu):
    from chameleonrt_b200.scenes import cornell_box

    check_bit_identity(gpu[0], *cornell_box(spp=2), 150, 90)


@pytest.mark.gpu
def test_views_equal_one_view_renderers_hw_textures(gpu):
    from helpers import synthetic_material_scene

    scene, cam = synthetic_material_scene(spp=2)
    check_bit_identity(gpu[0], scene, cam, 150, 90, hw_textures=True)


@pytest.mark.gpu
def test_eight_views_at_1280x720(gpu):
    from chameleonrt_b200.scenes import cornell_box

    V = 8
    check_bit_identity(gpu[0], *cornell_box(spp=1), 1280, 720, V=V, max_depth=8,
                       calls=[([True] * V, 1), ([False] * V, 2), ([k == 3 for k in range(V)], 1)])


@pytest.mark.gpu
def test_one_view_is_render_async(gpu):
    from chameleonrt_b200.scenes import cornell_box

    check_one_view_is_render_async(gpu[0], *cornell_box(spp=2), 200, 130)


@pytest.mark.gpu
@pytest.mark.parametrize("builder", ["host", "device"])
def test_scene_commits_reset_every_view(gpu, builder):
    from chameleonrt_b200.scenes import cornell_box

    check_scene_commits(gpu[0], *cornell_box(spp=1), 200, 130, builder)


@pytest.mark.gpu
def test_refusals(gpu):
    from chameleonrt_b200.scenes import cornell_box

    check_refusals(gpu[0], *cornell_box(spp=1))


@pytest.mark.gpu
def test_crts_cameras(gpu, tmp_path):
    check_crts_cameras(gpu[0], tmp_path, 200, 130)
