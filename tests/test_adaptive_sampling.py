"""Adaptive sampling (crtc_set_adaptive, crtc_read_adaptive; chameleonrt_b200/csrc/adaptive.cuh, k_raygen<true>,
k_resolve<true>).

Every check runs on the emulated renderer (tests/simt_emu) without a GPU and on libcrt_cuda_core.so on an H100 (``-m gpu``):
  * with every block active (min_frames above the frames rendered) accum, img, ray and path counts and the samples equal
    the mode-off render's, every frame, for single calls and batches; only the launch count grows, by 1 per call;
  * per-pixel equality: every pixel of an adaptive render (a threshold that stops blocks early, a max_frames cap, single
    calls and batches, the mode switched off mid-epoch) holds the uniform render's accum and img at its own sample count;
  * the pixel error against a numpy float32 restatement from a uniform render's lum_m1 / lum_m2, and every call's
    selection predicted from the previous read_adaptive, on a frame with blocks partly and entirely outside it;
  * two ranks (a shared frame and a gathered one) give the one-rank frame and samples;
  * quality at an equal number of samples on a lit box over the background;
  * error paths and the drop-in plugin's CRT_CUDA_ADAPTIVE.
"""
import math
import os
import sys

import numpy as np
import pytest

from test_aov_denoise import _args
from test_denoise_history import gpu  # noqa: F401 (a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "chameleonrt_b200", "csrc")
f32 = np.float32


@pytest.fixture(scope="module")
def emu(built):
    """(RenderCUDA, OracleBackend, primary_rays) with RenderCUDA bound to the emulated renderer."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "simt_emu"))
    import build as simt_build

    # (the emulation build's freshness list predates the headers it launches kernels from)
    lib = simt_build.LIB
    stale = not os.path.exists(lib) or any(os.path.getmtime(lib) < os.path.getmtime(os.path.join(CSRC, f))
                                           for f in ("adaptive.cuh", "aov_denoise.cuh"))
    lib_path = simt_build.build(force=stale)
    import chameleonrt_b200.backend as backend
    from oracle import OracleBackend
    from oracle.oracle import primary_rays

    saved = (backend._LIB_PATH, backend._lib)
    backend._LIB_PATH, backend._lib = lib_path, None
    yield backend.RenderCUDA, OracleBackend, primary_rays
    backend._LIB_PATH, backend._lib = saved


def _renderer(RenderCUDA, scene, w, h, **kw):
    # any_far_first = 0: no shadow-order trial, which keeps every block active during its blocking frames
    kw.setdefault("any_far_first", 0)
    r = RenderCUDA(0, max_depth=5, **kw)
    r.initialize(w, h)
    r.set_scene(scene)
    return r


def lit_box_scene(spp=1):
    """A small diffuse box on a plate, lit by the OBJ loader's default light, over the miss shader's background."""
    from chameleonrt_b200.scene import DisneyMaterial, Instance, Mesh, ParameterizedMesh, Scene, default_obj_light
    from chameleonrt_b200.scenes import MeshBuilder, box, grid

    b = MeshBuilder()
    for part in box((-0.4, 0.0, -0.4), (0.4, 0.8, 0.4)):
        b.add(*part)
    box_geom = b.geometry()
    b = MeshBuilder()
    b.add(*grid((-1.0, 0.0, 1.0), (2.0, 0.0, 0.0), (0.0, 0.0, -2.0), 1, 1))
    plate = b.geometry()
    mats = [DisneyMaterial(base_color=(0.8, 0.5, 0.3), roughness=0.6), DisneyMaterial(base_color=(0.7, 0.7, 0.7), roughness=0.9)]
    scene = Scene(meshes=[Mesh([box_geom, plate])], parameterized_meshes=[ParameterizedMesh(0, [0, 1])],
                  instances=[Instance(np.eye(4, dtype=np.float32), 0)], materials=mats, textures=[],
                  lights=[default_obj_light()], samples_per_pixel=spp)
    cam = dict(eye=(0.0, 1.6, 3.2), center=(0.0, 0.3, 0.0), up=(0.0, 1.0, 0.0), fov_y=45.0)
    return scene, cam


# ---- the definition, restated (include/crt_cuda.h, crtc_set_adaptive) ----
def pixel_error(m1, m2, samples):
    m1, m2 = np.asarray(m1, f32), np.asarray(m2, f32)
    n = np.asarray(samples).astype(f32)
    var = np.maximum(f32(0.0), m2 - m1 * m1)
    with np.errstate(divide="ignore", invalid="ignore"):
        e = np.sqrt(var / (n * np.maximum(m1, f32(1e-4))))
    return np.where(np.asarray(samples) == 0, f32(np.inf), e).astype(f32)


def block_ids(w, h):
    """The block of every pixel: 8x4 screen blocks aligned to the 64x64 tile grid, so (x // 8, y // 4) names it."""
    y, x = np.mgrid[0:h, 0:w]
    return (y // 4) * ((w + 7) // 8) + x // 8


def predict_samples(state, w, h, spp, frames, threshold, min_frames, max_frames, all_active=False):
    """samples per pixel after one call of `frames` frames, from read_adaptive before it (None: the first call)."""
    ids = block_ids(w, h)
    if state is None:
        c = np.zeros((h, w), np.int64)
        err = np.full((h, w), np.inf, f32)
    else:
        c = state["samples"].astype(np.int64) // spp
        err = state["error"]
    nb = ids.max() + 1
    e_b = np.full(nb, -1.0, f32)
    np.maximum.at(e_b, ids.ravel(), err.ravel())
    c_b = np.zeros(nb, np.int64)
    c_b[ids.ravel()] = c.ravel()
    n = np.where(all_active | (c_b < min_frames) | (e_b > f32(threshold)), frames, 0)
    if max_frames:
        n = np.minimum(n, np.maximum(max_frames - c_b, 0))
    return ((c_b + n) * spp)[ids].astype(np.uint32), int(((n * spp)[ids]).sum())


def uniform_snapshots(RenderCUDA, scene, cam, w, h, frames):
    """accum and img after 1..frames uniform frames (index k = after k frames)."""
    r = _renderer(RenderCUDA, scene, w, h)
    acc, img = [None], [None]
    for f in range(frames):
        r.render(*_args(cam), f == 0, True)
        acc.append(r.read_accum())
        img.append(r.read_img().copy())
    return acc, img


def check_against_uniform(r, snaps, spp):
    acc, img = snaps
    s = r.read_adaptive()["samples"]
    assert (s % spp == 0).all()
    k = s // spp
    got_a, got_i = r.read_accum(), r.read_img()
    for c in np.unique(k):
        m = k == c
        assert 1 <= c < len(acc), c
        assert np.array_equal(got_a[m].view(np.uint32), acc[c][m].view(np.uint32)), c
        assert np.array_equal(got_i[m], img[c][m]), c
    return k


# ---- checks ----
def check_all_active_is_uniform(mods, scene, cam, w, h):
    RenderCUDA = mods[0]
    spp = scene.samples_per_pixel
    args = _args(cam)
    off, on = _renderer(RenderCUDA, scene, w, h), _renderer(RenderCUDA, scene, w, h)
    on.set_adaptive(0.0, min_frames=100)
    for f in range(3):
        s0, s1 = off.render(*args, f == 0, True), on.render(*args, f == 0, True)
        assert s0.num_rays == s1.num_rays
        c0, c1 = off.counters(), on.counters()
        assert c1.pop("kernel_launches") == c0.pop("kernel_launches") + 1 and c0 == c1
        assert np.array_equal(off.read_accum().view(np.uint32), on.read_accum().view(np.uint32))
        assert np.array_equal(off.img, on.img) and np.array_equal(off.read_img(), on.read_img())
        assert (on.read_adaptive()["samples"] == (f + 1) * spp).all()
    # batches
    off, on = _renderer(RenderCUDA, scene, w, h), _renderer(RenderCUDA, scene, w, h)
    on.set_adaptive(0.0, min_frames=100)
    for batch in ((True, 2), (False, 3)):
        off.render_async(*args, *batch)
        on.render_async(*args, *batch)
        t0, _, c0, n0 = off.sync()
        t1, _, c1, n1 = on.sync()
        assert n0 == n1 and t0.num_rays == t1.num_rays
        assert c1.pop("kernel_launches") == c0.pop("kernel_launches") + 1 and c0 == c1
        assert np.array_equal(off.read_accum().view(np.uint32), on.read_accum().view(np.uint32))
        assert np.array_equal(off.read_img(), on.read_img())
    assert (on.read_adaptive()["samples"] == 5 * spp).all()


def median_threshold(RenderCUDA, scene, cam, w, h, frames=2):
    """A threshold between the block errors of a uniform render after `frames` frames: some blocks stop, some go on."""
    r = _renderer(RenderCUDA, scene, w, h)
    r.set_adaptive(0.0, min_frames=100)
    for f in range(frames):
        r.render(*_args(cam), f == 0, True)
    e = r.read_adaptive()["error"]
    ids = block_ids(w, h)
    e_b = np.full(ids.max() + 1, -1.0, f32)
    np.maximum.at(e_b, ids.ravel(), e.ravel())
    return float(np.median(e_b[e_b >= 0]))


def check_per_pixel_equality(mods, scene, cam, w, h, frames=6):
    RenderCUDA = mods[0]
    spp = scene.samples_per_pixel
    args = _args(cam)
    snaps = uniform_snapshots(RenderCUDA, scene, cam, w, h, frames)
    thr = median_threshold(RenderCUDA, scene, cam, w, h)
    # a threshold, single calls
    r = _renderer(RenderCUDA, scene, w, h)
    r.set_adaptive(thr, min_frames=2)
    for f in range(frames):
        r.render(*args, f == 0, True)
    k = check_against_uniform(r, snaps, spp)
    assert k.min() < k.max() == frames, (k.min(), k.max())
    # a threshold, batches (2 + 3 + 1 frames)
    r = _renderer(RenderCUDA, scene, w, h)
    r.set_adaptive(thr, min_frames=2)
    for batch in ((True, 2), (False, 3), (False, 1)):
        r.render_async(*args, *batch)
    r.sync()
    k = check_against_uniform(r, snaps, spp)
    assert k.min() < k.max(), (k.min(), k.max())
    # a cap: every block renders 3 frames (min_frames) and stops there (max_frames), single calls and batches
    for calls in ([(True, 1)] + [(False, 1)] * (frames - 1), [(True, 2), (False, 4)]):
        r = _renderer(RenderCUDA, scene, w, h)
        r.set_adaptive(0.0, min_frames=3, max_frames=3)
        for batch in calls:
            r.render_async(*args, *batch)
        r.sync()
        assert (check_against_uniform(r, snaps, spp) == 3).all()
    # the mode switched off mid-epoch: every block goes on from its own count
    r = _renderer(RenderCUDA, scene, w, h)
    r.set_adaptive(thr, min_frames=2)
    for f in range(3):
        r.render(*args, f == 0, True)
    before = r.read_adaptive()["samples"]
    r.set_adaptive(None)
    r.render(*args, False, True)
    r.render_async(*args, False, 2)
    r.sync()
    k = check_against_uniform(r, snaps, spp)
    assert np.array_equal(k * spp, before + 3 * spp)
    # and a camera change ends the epoch: a mode-off render is the uniform one again, with no adaptive state to read
    r.render(*args, True, True)
    assert np.array_equal(r.read_accum().view(np.uint32), snaps[0][1].view(np.uint32))
    with pytest.raises(RuntimeError, match="no frame has been rendered with adaptive sampling"):
        r.read_adaptive()


def check_statistics_and_selection(mods, scene, cam, w, h, frames=3):
    RenderCUDA = mods[0]
    spp = scene.samples_per_pixel
    args = _args(cam)
    # e_p from a uniform render's luminance moments (option aov), at equal counts
    ref = _renderer(RenderCUDA, scene, w, h, aov=True)
    on = _renderer(RenderCUDA, scene, w, h)
    on.set_adaptive(0.0, min_frames=100)
    for f in range(frames):
        ref.render(*args, f == 0, True)
        on.render(*args, f == 0, True)
        a = ref.read_aov()
        want = pixel_error(a["lum_m1"], a["lum_m2"], (f + 1) * spp)
        got = on.read_adaptive()["error"]
        assert np.isfinite(want).all() and (want > 0).any()
        np.testing.assert_allclose(got, want, rtol=1e-5, atol=0)
    # every call's selection, predicted from the state before it
    thr = median_threshold(RenderCUDA, scene, cam, w, h)
    for min_frames, max_frames, calls in ((2, 0, [1, 1, 2, 1, 3]), (1, 5, [2, 1, 1, 3, 1])):
        r = _renderer(RenderCUDA, scene, w, h)
        r.set_adaptive(thr, min_frames=min_frames, max_frames=max_frames)
        state = None
        for i, n in enumerate(calls):
            want, paths = predict_samples(state, w, h, spp, n, thr, min_frames, max_frames)
            r.render_async(*args, i == 0, n)
            counters = r.sync()[2]
            state = r.read_adaptive()
            assert np.array_equal(state["samples"], want), i
            assert counters["paths"] == paths, i
    # option any_far_first = 2: its trial frames (blocking calls until it decides) keep every block active
    r = _renderer(RenderCUDA, scene, w, h, any_far_first=2)
    r.set_adaptive(1e30, min_frames=1)
    r.render(*args, True, True)
    assert r.get_option("any_far_first_decision") == -1
    r.render_async(*args, False, 1)  # (not a trial frame: the threshold stops everything)
    r.sync()
    assert (r.read_adaptive()["samples"] == spp).all()
    for f in range(2):
        r.render(*args, False, True)
    assert r.get_option("any_far_first_decision") != -1
    assert (r.read_adaptive()["samples"] == 3 * spp).all()
    r.render(*args, False, True)
    assert (r.read_adaptive()["samples"] == 3 * spp).all()


def check_two_ranks(mods, scene, cam, w, h):
    RenderCUDA = mods[0]
    spp = scene.samples_per_pixel
    args = _args(cam)
    thr = median_threshold(RenderCUDA, scene, cam, w, h)
    calls = [(True, 2), (False, 1), (False, 3)]

    def run(r):
        r.set_adaptive(thr, min_frames=2)

    one = _renderer(RenderCUDA, scene, w, h)
    run(one)
    for c in calls:
        one.render_async(*args, *c)
    one.sync()
    want_a, want_i, want_s = one.read_accum(), one.read_img(), one.read_adaptive()["samples"]
    assert want_s.min() < want_s.max()
    for shared in (True, False):
        ranks = [_renderer(RenderCUDA, scene, w, h, rank=k, world_size=2) for k in range(2)]
        if shared:
            ranks[0].share_frame_with(ranks[1])
        for r in ranks:
            run(r)
            for c in calls:
                r.render_async(*args, *c)
            r.sync()
        if not shared:
            for src, r in enumerate(ranks):
                acc, img, _ = r.local_buffers()
                ranks[0].assemble_rank(src, 2, acc, img)
        samples = ranks[0].read_adaptive()["samples"] + ranks[1].read_adaptive()["samples"]
        assert np.array_equal(samples, want_s), shared
        assert np.array_equal(ranks[0].read_accum().view(np.uint32), want_a.view(np.uint32)), shared
        assert np.array_equal(ranks[0].read_img(), want_i), shared
    return spp


def check_quality(mods, size=64, calls=24, threshold=0.05):
    """Lit box over the background, 1 spp: at an equal number of samples (the uniform frame gets at least as many), the
    adaptive frame's MSE against a converged uniform frame is lower than the uniform frame's."""
    RenderCUDA, OracleBackend, _ = mods
    scene, cam = lit_box_scene(spp=1)
    args = _args(cam)
    ada = _renderer(RenderCUDA, scene, size, size)
    ada.set_adaptive(threshold, min_frames=4)
    for f in range(calls):
        ada.render(*args, f == 0, True)
    total = int(ada.read_adaptive()["samples"].astype(np.int64).sum())
    frames = math.ceil(total / (size * size))
    uni = _renderer(RenderCUDA, scene, size, size)
    for f in range(frames):
        uni.render(*args, f == 0, True)
    ref_scene, _ = lit_box_scene(spp=64)
    orc = OracleBackend(fast=True)
    orc.initialize(size, size)
    orc.set_scene(ref_scene)
    for f in range(16):
        orc.render(*args, f == 0)
    ref = orc.read_accum()
    mse_uniform = float(np.mean((uni.read_accum() - ref) ** 2))
    mse_adaptive = float(np.mean((ada.read_accum() - ref) ** 2))
    print(f"quality: {total} samples adaptive, {frames * size * size} uniform ({frames} frames): "
          f"MSE uniform {mse_uniform:.5f}, adaptive {mse_adaptive:.5f}")
    assert frames < calls  # some blocks stopped
    assert mse_adaptive < mse_uniform, (mse_adaptive, mse_uniform)
    return mse_uniform, mse_adaptive


def check_errors(mods):
    from chameleonrt_b200.scenes import cornell_box

    RenderCUDA = mods[0]
    scene, cam = cornell_box(spp=1)
    r = _renderer(RenderCUDA, scene, 16, 16)
    for kw, msg in ((dict(threshold=-1.0), "threshold"), (dict(threshold=float("nan")), "threshold"),
                    (dict(threshold=float("inf")), "threshold"), (dict(threshold=0.1, min_frames=0), "min_frames"),
                    (dict(threshold=0.1, min_frames=4, max_frames=3), "max_frames")):
        with pytest.raises(RuntimeError, match=msg):
            r.set_adaptive(**kw)
    r.set_adaptive(0.1, min_frames=4, max_frames=4)
    r.set_adaptive(0.0, min_frames=1)
    with pytest.raises(RuntimeError, match="no frame has been rendered"):
        r.read_adaptive()
    r.render(*_args(cam), True, True)
    r.read_adaptive()
    assert r.lib.crtc_read_adaptive(r.h, None, None) == 0  # both outputs are optional
    r.set_scene(scene)  # a new scene resets the counts like accum
    with pytest.raises(RuntimeError, match="no frame has been rendered"):
        r.read_adaptive()
    # option aov, in either order
    r.set_option("aov", 1)
    with pytest.raises(RuntimeError, match="aov cannot be combined with adaptive"):
        r.initialize(16, 16)
    r.set_adaptive(None)
    r.initialize(16, 16)
    with pytest.raises(RuntimeError, match="cannot be combined with option aov"):
        r.set_adaptive(0.1)
    # NULL renderer handles
    for rc in (r.lib.crtc_set_adaptive(None, None), r.lib.crtc_read_adaptive(None, None, None)):
        assert rc != 0 and b"NULL" in r.lib.crtc_last_error()


# ---- CPU: the emulated renderer ----
def test_all_active_is_the_uniform_render_on_the_emulated_renderer(emu):
    from chameleonrt_b200.scenes import cornell_box

    check_all_active_is_uniform(emu, *cornell_box(spp=2), 70, 42)


def test_pixels_equal_the_uniform_render_at_their_count_on_the_emulated_renderer(emu):
    from chameleonrt_b200.scenes import cornell_box

    check_per_pixel_equality(emu, *cornell_box(spp=1), 70, 42)


def test_statistics_and_selection_on_the_emulated_renderer(emu):
    from chameleonrt_b200.scenes import cornell_box

    check_statistics_and_selection(emu, *cornell_box(spp=2), 70, 42)


def test_two_ranks_on_the_emulated_renderer(emu):
    from chameleonrt_b200.scenes import cornell_box

    check_two_ranks(emu, *cornell_box(spp=1), 70, 42)


def test_quality_on_the_emulated_renderer(emu):
    check_quality(emu)


def test_error_paths_on_the_emulated_renderer(emu):
    check_errors(emu)


def test_plugin_adaptive_variable_on_the_emulated_core(emu, tmp_path):
    """`crt_headless cuda_simt` with CRT_CUDA_ADAPTIVE: the float framebuffer it writes is Python's adaptive render of the
    same frames; refused together with CRT_CUDA_DENOISE=1."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "simt_emu"))
    import build as simt_build
    from test_reference_plugin import HEADLESS, run_headless

    if not os.path.exists(HEADLESS) or simt_build.build_plugin() is None:
        pytest.skip("needs oracle/_ref (built where the reference sources are)")
    from chameleonrt_b200.obj_io import write_obj
    from chameleonrt_b200.scenes import cornell_box

    w, h, frames, thr = 64, 48, 5, 0.3
    scene, cam = cornell_box(spp=1)
    obj = write_obj(scene, str(tmp_path / "scene.obj"))
    env = {"CRT_CUDA_ADAPTIVE": str(thr), "CRT_CUDA_ADAPTIVE_MIN_FRAMES": "2", "CRT_CUDA_ADAPTIVE_MAX_FRAMES": "4"}
    plain, v, _ = run_headless("cuda_simt", obj, cam, w, h, 1, frames, tmp_path)
    got, v2, _ = run_headless("cuda_simt", obj, cam, w, h, 1, frames, tmp_path, extra_env=env)
    assert v == v2
    r = _renderer(emu[0], scene, w, h, any_far_first=2)  # the plugin's default
    r.set_adaptive(thr, min_frames=2, max_frames=4)
    for f in range(frames):
        r.render(v[0:3], v[3:6], v[6:9], v[9], f == 0, True)
    assert np.array_equal(r.read_accum().view(np.uint32), got.view(np.uint32))
    assert not np.array_equal(plain.view(np.uint32), got.view(np.uint32))
    # two renderers sharing the frame (CRT_CUDA_DEVICES) give the same frame
    got2, _, _ = run_headless("cuda_simt", obj, cam, w, h, 1, frames, tmp_path, extra_env={**env, "CRT_CUDA_DEVICES": "0,0"})
    assert np.array_equal(got2.view(np.uint32), got.view(np.uint32))
    with pytest.raises(AssertionError, match="CRT_CUDA_DENOISE"):
        run_headless("cuda_simt", obj, cam, w, h, 1, 1, tmp_path, extra_env={**env, "CRT_CUDA_DENOISE": "1"})


# ---- GPU: libcrt_cuda_core.so on the H100 ----
@pytest.mark.gpu
def test_all_active_is_the_uniform_render(gpu):
    from chameleonrt_b200.scenes import cornell_box

    check_all_active_is_uniform(gpu, *cornell_box(spp=2), 200, 130)


@pytest.mark.gpu
def test_pixels_equal_the_uniform_render_at_their_count(gpu):
    from chameleonrt_b200.scenes import cornell_box

    check_per_pixel_equality(gpu, *cornell_box(spp=1), 200, 130, frames=8)


@pytest.mark.gpu
def test_statistics_and_selection(gpu):
    from chameleonrt_b200.scenes import cornell_box

    check_statistics_and_selection(gpu, *cornell_box(spp=2), 200, 130)


@pytest.mark.gpu
def test_two_renderers_on_one_device(gpu):
    from chameleonrt_b200.scenes import cornell_box

    check_two_ranks(gpu, *cornell_box(spp=1), 200, 130)


@pytest.mark.gpu
def test_quality(gpu):
    check_quality(gpu)


@pytest.mark.gpu
def test_error_paths(gpu):
    check_errors(gpu)
