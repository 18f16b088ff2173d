"""Scene updates between frames (option dynamic_scene; crtc_update_instances, crtc_update_vertices, crtc_update_lights,
crtc_commit_scene; chameleonrt_b200/csrc/scene_update.cuh: k_reflatten, k_bvh8_refit).

Every check runs on the emulated build (tests/simt_emu) without a GPU and on the sm_90a build with ``-m gpu``:
  * an identity commit rewrites every node, triangle record and shading record byte for byte (all three builders);
  * after moving instances (rotation, non-uniform scale, a translation larger than the scene) and deforming a shared
    mesh, every refit node passes test_bvh_build_exact.check_bvh8 (whose p / e / qlo / qhi are the float union of the
    triangles below, quantised by its numpy `quantise`), the node structure is unchanged, and the records sorted by flat
    id equal a fresh host build of the moved scene's;
  * frames (accum and img, frame after frame), trace_closest and trace_any after a commit equal those of a fresh renderer
    set_scene'd with the updated scene, for every builder and for instance, shared-vertex, light (count changes
    included) and combined updates;
  * stream order (render_async / commit / render_async), staged-but-uncommitted updates, the resets (AOVs, the
    denoiser's history, adaptive counts), two ranks, and the error paths.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from test_aov_denoise import _args
from test_bvh_build_exact import NODE, adversarial_instanced_scene, check_bvh8

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "chameleonrt_b200", "csrc")
F32, U8, U32 = np.float32, np.uint8, np.uint32
BUILDERS = ("host", "device", "device_lbvh")
# (the emulation builds' freshness lists predate the headers changed for this feature)
_NEW_SOURCES = ("scene_update.cuh", "scene_device_build.cuh", "bvh8_device.cuh", "cuda_host_utils.h", "crt_cuda_core.cu",
                "bvh_devcheck.cu", "host_scene.cpp", "bvh8_build.cpp", "bvh8.h")


def _stale(lib):
    return not os.path.exists(lib) or any(os.path.getmtime(lib) < os.path.getmtime(os.path.join(CSRC, f)) for f in _NEW_SOURCES)


# ---- the libraries under test ----
class UpdateCheck:
    """bvhdev_update of libcrt_bvh_devcheck.so (or its emulated twin): a set_scene with option dynamic_scene and one
    commit of a moved scene's transforms and vertices, through the renderer's own update driver."""

    def __init__(self, path, gpu):
        self.gpu = gpu
        self.lib = lib = C.CDLL(path)
        vp = C.c_void_p
        lib.bvhdev_last_error.restype = C.c_char_p
        lib.bvhdev_update.argtypes, lib.bvhdev_update.restype = [vp, vp, C.c_int, vp], vp
        lib.bvhdev_fetch_update.argtypes, lib.bvhdev_fetch_update.restype = [vp, C.c_int, vp], C.c_longlong
        lib.bvhdev_free_update.argtypes = [vp]

    def update(self, scene, moved, builder):
        a, b = scene.to_c(), moved.to_c()
        info = np.zeros(5, U32)
        h = self.lib.bvhdev_update(C.byref(a.c), C.byref(b.c), BUILDERS.index(builder), info.ctypes.data)
        assert h, self.lib.bvhdev_last_error().decode()
        n, nn = int(info[0]), int(info[1])
        out = dict(n=n, num_nodes=nn, depth=int(info[2]), launches=int(info[3]))
        shapes = [("nodes0", U8, (nn, 80)), ("tris0", F32, (n, 12)), ("shade0", F32, (n, 12)), ("nodes", U8, (nn, 80)),
                  ("tris", F32, (n, 12)), ("shade", F32, (n, 12)), ("leaf_flat_ids", U32, (n,)), ("levels", U32, (int(info[4]),))]
        try:
            for field, (name, dt, shape) in enumerate(shapes):
                x = np.zeros(shape, dt)
                assert self.lib.bvhdev_fetch_update(h, field, x.ctypes.data) == x.nbytes, name
                out[name] = x
        finally:
            self.lib.bvhdev_free_update(h)
        return out


@pytest.fixture(scope="module")
def emulated_check(built):
    sys.path.insert(0, os.path.join(ROOT, "tests", "simt_emu"))
    import build as simt_build

    return UpdateCheck(simt_build.build_bvh_devcheck(force=_stale(simt_build.DEVCHECK_LIB)), False)


@pytest.fixture(scope="module")
def device_check(built):
    return UpdateCheck(os.path.join(CSRC, "libcrt_bvh_devcheck.so"), True)


@pytest.fixture(params=[pytest.param("emulated_check"), pytest.param("device_check", marks=pytest.mark.gpu)], scope="module")
def upd(request):
    return request.getfixturevalue(request.param)


def _bind(lib_path):
    import chameleonrt_b200.backend as backend

    saved = (backend._LIB_PATH, backend._lib)
    backend._LIB_PATH, backend._lib = lib_path, None
    return backend, saved


@pytest.fixture(scope="module")
def emu_renderer(built):
    sys.path.insert(0, os.path.join(ROOT, "tests", "simt_emu"))
    import build as simt_build

    backend, saved = _bind(simt_build.build(force=_stale(simt_build.LIB)))
    yield backend.RenderCUDA
    backend._LIB_PATH, backend._lib = saved


@pytest.fixture(scope="module")
def gpu_renderer(built):
    backend, saved = _bind(os.path.join(CSRC, "libcrt_cuda_core.so"))
    yield backend.RenderCUDA
    backend._LIB_PATH, backend._lib = saved


@pytest.fixture(params=[pytest.param("emu_renderer"), pytest.param("gpu_renderer", marks=pytest.mark.gpu)])
def RenderCUDA(request):
    return request.getfixturevalue(request.param)


# ---- scenes ----
def _rot(ax, ang):
    c, s = np.cos(ang), np.sin(ang)
    m = np.eye(4)
    i, j = [(1, 2), (0, 2), (0, 1)][ax]
    m[i, i], m[i, j], m[j, i], m[j, j] = c, -s, s, c
    return m


def moved_transforms(scene, seed, extent):
    """Rotations about all three axes, non-uniform scale and a translation up to 1.5 x the scene's extent."""
    rng = np.random.default_rng(seed)
    out = []
    for inst in scene.instances:
        m = _rot(0, rng.uniform(-1, 1)) @ _rot(1, rng.uniform(-3, 3)) @ _rot(2, rng.uniform(-1, 1)) @ np.diag([*rng.uniform(0.5, 2, 3), 1])
        m[:3, 3] = rng.uniform(-1.5, 1.5, 3) * extent
        out.append((m @ np.asarray(inst.transform, np.float64)).astype(F32))
    return np.array(out)


def replaced(scene, transforms=None, vertices=None, lights=None):
    """A copy of `scene` with new transforms, {(mesh, geometry): vertices} and lights; topology shared."""
    import copy

    s = copy.copy(scene)
    s.meshes = [copy.copy(m) for m in scene.meshes]
    for m in s.meshes:
        m.geometries = [copy.copy(g) for g in m.geometries]
    for (mi, gi), v in (vertices or {}).items():
        s.meshes[mi].geometries[gi].vertices = np.asarray(v, F32)
    if transforms is not None:
        s.instances = [copy.copy(i) for i in scene.instances]
        for inst, t in zip(s.instances, transforms):
            inst.transform = np.asarray(t, F32)
    if lights is not None:
        s.lights = list(lights)
    return s


def deformed(scene, mesh, geom, seed):
    v = np.asarray(scene.meshes[mesh].geometries[geom].vertices, F32)
    rng = np.random.default_rng(seed)
    return (v * F32(1.3) + rng.normal(scale=0.05, size=v.shape)).astype(F32)


def small_courtyard():
    from chameleonrt_b200.scenes import san_miguel_like

    return san_miguel_like(spp=1, scale=0.002, tex_size=16)


def shared_mesh(scene):
    """(mesh, geometry) of a geometry that several instances draw."""
    count = {}
    for inst in scene.instances:
        m = scene.parameterized_meshes[inst.parameterized_mesh_id].mesh_id
        count[m] = count.get(m, 0) + 1
    m = max(count, key=count.get)
    assert count[m] > 1
    g = max(range(len(scene.meshes[m].geometries)), key=lambda k: len(scene.meshes[m].geometries[k].indices))
    return m, g


def world_tris(scene):
    """The flattened triangles (n, 3, 3) in world space in flattened order, with flatten_scene's float32 arithmetic
    (column-major matrix, the sums in source order, no fused multiply-add)."""
    out = []
    for inst in scene.instances:
        m = np.asarray(inst.transform, F32).T.reshape(-1)  # column-major
        pm = scene.parameterized_meshes[inst.parameterized_mesh_id]
        for g in scene.meshes[pm.mesh_id].geometries:
            v = np.asarray(g.vertices, F32)[np.asarray(g.indices, np.int64).reshape(-1, 3)]
            x, y, z = v[..., 0], v[..., 1], v[..., 2]
            w = [((m[a] * x + m[4 + a] * y) + m[8 + a] * z) + m[12 + a] for a in range(3)]
            out.append(np.stack(w, -1).astype(F32))
    return np.concatenate(out) if out else np.zeros((0, 3, 3), F32)


def scene_extent(scene):
    t = world_tris(scene).reshape(-1, 3)
    return float((t.max(0) - t.min(0)).max())


# ---- (1) identity commit ----
def test_identity_commit_rewrites_every_byte(upd):
    """set_scene, then a commit of the same transforms and vertices: every node, triangle and shading record is
    rewritten with the bytes it had, for the host builder, PLOC and LBVH."""
    for scene in (small_courtyard()[0], adversarial_instanced_scene()):
        for builder in BUILDERS:
            out = upd.update(scene, scene, builder)
            assert out["launches"] == 1 + len(out["levels"]) - 1, builder  # k_reflatten + one refit per level
            for k in ("nodes", "tris", "shade"):
                assert np.array_equal(out[k + "0"].view(U8), out[k].view(U8)), (builder, k)


# ---- (2) moved instances and a deformed shared mesh ----
def check_refit_bvh8(nodes, order, tris, depth):
    """check_bvh8 up to its last check: structure, every triangle once, conservative and tight slot boxes, and p / e /
    qlo / qhi equal to fill_node's quantisation of the float union of the triangles below. Its last check, that the slot
    order is what assign_slots would choose for these boxes, is a build-time choice: a refit keeps the slots (and so the
    tree and the leaf order) of the build."""
    try:
        check_bvh8(nodes, order, tris, depth)
    except AssertionError as e:
        assert "the slot order is not assign_slots' greedy order" in str(e), e


def test_refit_after_moves_is_exact(upd):
    from helpers import HostCheck

    scene = small_courtyard()[0]
    ext = scene_extent(scene)
    m, g = shared_mesh(scene)
    moved = replaced(scene, moved_transforms(scene, 5, ext), {(m, g): deformed(scene, m, g, 6)})
    tris = world_tris(moved)
    hc = HostCheck(moved)
    _, h_order, h_tris, h_shade = hc.export()
    hpos = np.empty(len(h_order), np.int64)
    hpos[h_order] = np.arange(len(h_order))
    for builder in BUILDERS:
        out = upd.update(scene, moved, builder)
        flat = out["leaf_flat_ids"]
        # every node: structure unchanged, boxes the float union of the moved triangles below, quantised as fill_node
        before, after = out["nodes0"].view(NODE), out["nodes"].view(NODE)
        for f in ("imask", "child_base", "tri_base", "meta"):
            assert np.array_equal(before[f], after[f]), (builder, f)
        assert not np.array_equal(before["p"], after["p"]), builder
        check_refit_bvh8(out["nodes"], flat, tris, out["depth"])
        # the records equal a fresh build's of the moved scene, by flat id
        assert np.array_equal(out["tris"][:, :3], tris[flat, 0]), builder
        assert np.array_equal(out["tris"].view(U32), h_tris[hpos[flat]].view(U32)), builder
        assert np.array_equal(out["shade"].view(U32), h_shade[hpos[flat]].view(U32)), builder


# ---- (3) frames ----
def small_instanced_scene(spp=1):
    """Two instances of a box mesh, one of a sphere mesh with two geometries (one without uvs) and a plate; two lights."""
    from chameleonrt_b200.scene import DisneyMaterial, Geometry, Instance, Mesh, ParameterizedMesh, QuadLight, Scene
    from chameleonrt_b200.scenes import MeshBuilder, box, grid, sphere

    b = MeshBuilder()
    for part in box((-0.3, 0.0, -0.3), (0.3, 0.6, 0.3)):
        b.add(*part)
    box_geom = b.geometry()
    sv, _, si = sphere((0.0, 0.3, 0.0), 0.3, 10, 6)
    ball = Geometry(np.asarray(sv, F32), np.asarray(si, U32))
    b = MeshBuilder()
    b.add(*grid((-1.5, 0.0, 1.5), (3.0, 0.0, 0.0), (0.0, 0.0, -3.0), 2, 2))
    plate = b.geometry()
    mats = [DisneyMaterial(base_color=(0.8, 0.5, 0.3), roughness=0.6), DisneyMaterial(base_color=(0.3, 0.6, 0.8), metallic=0.5),
            DisneyMaterial(base_color=(0.7, 0.7, 0.7), roughness=0.9)]

    def at(x, z):
        m = np.eye(4, dtype=F32)
        m[0, 3], m[2, 3] = x, z
        return m

    lights = [QuadLight((6.0, 6.0, 6.0), (-0.5, 2.0, -0.5), (0.0, -1.0, 0.0), (1.0, 0.0, 0.0), 1.0, (0.0, 0.0, 1.0), 1.0),
              QuadLight((2.0, 3.0, 4.0), (1.0, 1.5, 1.0), (-0.5, -0.7, -0.5), (0.7, 0.0, -0.7), 0.5, (0.0, 1.0, 0.0), 0.5)]
    scene = Scene(meshes=[Mesh([box_geom]), Mesh([ball, plate])], parameterized_meshes=[ParameterizedMesh(0, [0]), ParameterizedMesh(1, [1, 2])],
                  instances=[Instance(at(-0.6, 0.0), 0), Instance(at(0.6, -0.3), 0), Instance(at(0.0, 0.5), 1)],
                  materials=mats, textures=[], lights=lights, samples_per_pixel=spp)
    cam = dict(eye=(0.0, 1.8, 3.4), center=(0.0, 0.3, 0.0), up=(0.0, 1.0, 0.0), fov_y=50.0)
    return scene, cam


def updated_small_scene(scene, which):
    from chameleonrt_b200.scene import QuadLight

    t = np.array([i.transform for i in scene.instances])
    new_t = t.copy()
    new_t[1] = (_rot(1, 0.8) @ np.diag([1.3, 0.7, 1.1, 1.0]) @ t[1].astype(np.float64)).astype(F32)
    new_t[1][:3, 3] += (0.2, 0.1, 0.3)
    verts = {(0, 0): deformed(scene, 0, 0, 3)}  # the box mesh: both box instances change
    lights = [QuadLight((3.0, 5.0, 3.0), (0.5, 2.5, 0.0), (0.0, -1.0, 0.0), (0.6, 0.0, 0.0), 0.6, (0.0, 0.0, 0.6), 0.6)]
    return {"instances": (replaced(scene, transforms=new_t), dict(instances=new_t[1:2], first=1)),
            "vertices": (replaced(scene, vertices=verts), dict(vertices=verts)),
            "lights": (replaced(scene, lights=lights), dict(lights=lights)),
            "all": (replaced(scene, transforms=new_t, vertices=verts, lights=lights),
                    dict(instances=new_t[1:2], first=1, vertices=verts, lights=lights))}[which]


def stage(r, instances=None, first=0, vertices=None, lights=None):
    if instances is not None:
        r.update_instances(instances, first)
    for (m, g), v in (vertices or {}).items():
        r.update_vertices(m, g, v)
    if lights is not None:
        r.update_lights(lights)


def _renderer(RenderCUDA, scene, w, h, **kw):
    kw.setdefault("any_far_first", 0)
    r = RenderCUDA(0, max_depth=3, **kw)
    r.initialize(w, h)
    r.set_scene(scene)
    return r


def random_rays(scene, n, seed):
    t = world_tris(scene).reshape(-1, 3)
    lo, hi = t.min(0), t.max(0)
    rng = np.random.default_rng(seed)
    o = rng.uniform(lo - 1, hi + 1, (n, 3))
    d = rng.normal(size=(n, 3))
    rays = np.concatenate([o, np.full((n, 1), 1e-4), d, np.full((n, 1), 1e30)], 1).astype(F32)
    rays[::3, 3] = 0.0  # some through the closest-hit kernel in trace_any
    return rays


def frames_equal(a, b, args, frames, a_changed):
    for f in range(frames):
        a.render(*args, a_changed and f == 0, True)
        b.render(*args, f == 0, True)
        assert np.array_equal(a.read_accum().view(U32), b.read_accum().view(U32)), f
        assert np.array_equal(a.read_img(), b.read_img()), f


@pytest.mark.parametrize("which", ["instances", "vertices", "lights", "all"])
def test_frames_after_commit_equal_a_fresh_set_scene(RenderCUDA, which):
    scene, cam = small_instanced_scene()
    new, upd = updated_small_scene(scene, which)
    args = _args(cam)
    w = h = 32
    for builder in (BUILDERS if which == "all" else ("host",)):
        r = _renderer(RenderCUDA, scene, w, h, bvh_builder=builder, dynamic_scene=True)
        for f in range(2):
            r.render(*args, f == 0, True)
        stage(r, **upd)
        r.commit_scene()
        fresh = _renderer(RenderCUDA, new, w, h, bvh_builder=builder)
        frames_equal(r, fresh, args, 2, False)  # (no camera_changed: the commit reset the accumulation)
        rays = random_rays(new, 512, 9)
        assert np.array_equal(r.trace_closest(rays).view(U32), fresh.trace_closest(rays).view(U32)), builder
        assert np.array_equal(r.trace_any(rays), fresh.trace_any(rays)), builder


def test_light_count_changes_and_lights_need_no_option(RenderCUDA):
    from chameleonrt_b200.scene import QuadLight

    scene, cam = small_instanced_scene()
    args = _args(cam)
    more = scene.lights + [QuadLight((1.0, 2.0, 3.0), (0.0, 2.0, 1.0), (0.0, -1.0, 0.0), (0.4, 0.0, 0.0), 0.4, (0.0, 0.0, 0.4), 0.4)]
    r = _renderer(RenderCUDA, scene, 32, 32)  # dynamic_scene off
    for lights in (scene.lights[:1], more, scene.lights):
        r.render(*args, True, True)
        r.update_lights(lights)
        r.commit_scene()
        frames_equal(r, _renderer(RenderCUDA, replaced(scene, lights=lights), 32, 32), args, 1, False)


# ---- (4) ordering ----
def test_commit_is_stream_ordered_and_staging_alone_changes_nothing(RenderCUDA):
    scene, cam = small_instanced_scene()
    _, upd = updated_small_scene(scene, "all")
    args = _args(cam)
    a = _renderer(RenderCUDA, scene, 32, 32, dynamic_scene=True)
    a.render_async(*args, True, 2)
    stage(a, **upd)
    a.commit_scene()
    a.render_async(*args, False, 2)
    a.sync()
    b = _renderer(RenderCUDA, scene, 32, 32, dynamic_scene=True)
    for f in range(2):
        b.render(*args, f == 0, True)
    stage(b, **upd)
    b.commit_scene()
    for f in range(2):
        b.render(*args, False, True)
    assert np.array_equal(a.read_accum().view(U32), b.read_accum().view(U32))
    assert np.array_equal(a.read_img(), b.read_img())
    # staged, never committed: the frames are those of a renderer without updates
    c = _renderer(RenderCUDA, scene, 32, 32, dynamic_scene=True)
    d = _renderer(RenderCUDA, scene, 32, 32)
    c.render(*args, True, True)
    stage(c, **upd)
    d.render(*args, True, True)
    for f in range(2):
        c.render(*args, False, True)
        d.render(*args, False, True)
        assert np.array_equal(c.read_accum().view(U32), d.read_accum().view(U32)), f
    # and set_scene discards them: a commit afterwards is empty
    stage(c, **upd)
    c.set_scene(scene)
    d.set_scene(scene)
    for r in (c, d):
        r.render(*args, True, True)
    c.commit_scene()
    for r in (c, d):
        r.render(*args, False, True)
    assert np.array_equal(c.read_accum().view(U32), d.read_accum().view(U32))


# ---- (5) resets ----
def test_commit_resets_aovs_history_and_adaptive_counts(RenderCUDA):
    scene, cam = small_instanced_scene()
    new, upd = updated_small_scene(scene, "instances")
    args = _args(cam)
    r = _renderer(RenderCUDA, scene, 32, 32, dynamic_scene=True, aov=True, denoise_history=8)
    for f in range(2):
        r.render(*args, f == 0, True)
    r.denoise()
    r.read_denoise_history()
    stage(r, **upd)
    r.commit_scene()
    with pytest.raises(RuntimeError, match="no crtc_denoise since the last reset"):
        r.read_denoise_history()
    fresh = _renderer(RenderCUDA, new, 32, 32, aov=True, denoise_history=8)
    r.render(*args, False, True)
    fresh.render(*args, True, True)
    got, want = r.read_aov(), fresh.read_aov()
    for k in want:
        assert np.array_equal(got[k].view(U32), want[k].view(U32)), k
    r.denoise()
    r.read_denoise_history()
    # adaptive: every block count restarts
    a = _renderer(RenderCUDA, scene, 32, 32, dynamic_scene=True)
    a.set_adaptive(0.0, min_frames=4)
    for f in range(3):
        a.render(*args, f == 0, True)
    assert (a.read_adaptive()["samples"] == 3).all()
    stage(a, **upd)
    a.commit_scene()
    for f in range(2):
        a.render(*args, False, True)
    assert (a.read_adaptive()["samples"] == 2).all()


# ---- (6) two ranks ----
def test_two_ranks_apply_the_same_updates(RenderCUDA):
    scene, cam = small_instanced_scene()
    _, upd = updated_small_scene(scene, "all")
    args = _args(cam)
    w, h = 96, 80  # (several 64x64 tiles)

    def run(r):
        r.render(*args, True, True)
        stage(r, **upd)
        r.commit_scene()
        r.render_async(*args, False, 2)
        r.sync()

    one = _renderer(RenderCUDA, scene, w, h, dynamic_scene=True)
    run(one)
    for shared in (True, False):
        ranks = [_renderer(RenderCUDA, scene, w, h, dynamic_scene=True, rank=k, world_size=2) for k in range(2)]
        if shared:
            ranks[0].share_frame_with(ranks[1])
        for r in ranks:
            run(r)
        if not shared:
            for src, r in enumerate(ranks):
                acc, img, _ = r.local_buffers()
                ranks[0].assemble_rank(src, 2, acc, img)
        assert np.array_equal(ranks[0].read_accum().view(U32), one.read_accum().view(U32)), shared
        assert np.array_equal(ranks[0].read_img(), one.read_img()), shared


# ---- (7) errors ----
def test_error_paths(RenderCUDA):
    scene, cam = small_instanced_scene()
    args = _args(cam)
    eye = np.eye(4, dtype=F32)[None]
    r = RenderCUDA(0, max_depth=3, any_far_first=0, dynamic_scene=True)
    r.initialize(16, 16)
    for call in (lambda: r.update_instances(eye), lambda: r.update_vertices(0, 0, np.zeros((1, 3), F32)),
                 lambda: r.update_lights(scene.lights), r.commit_scene):
        with pytest.raises(RuntimeError, match="set_scene"):
            call()
    off = _renderer(RenderCUDA, scene, 16, 16)
    with pytest.raises(RuntimeError, match="needs option dynamic_scene = 1"):
        off.update_instances(eye)
    with pytest.raises(RuntimeError, match="needs option dynamic_scene = 1"):
        off.update_vertices(0, 0, scene.meshes[0].geometries[0].vertices)
    r.set_scene(scene)
    with pytest.raises(RuntimeError, match="exceed the scene's 3"):
        r.update_instances(np.repeat(eye, 2, 0), first=2)
    with pytest.raises(RuntimeError, match="mesh 2 out of range"):
        r.update_vertices(2, 0, np.zeros((1, 3), F32))
    with pytest.raises(RuntimeError, match="geometry 1 out of range"):
        r.update_vertices(0, 1, np.zeros((1, 3), F32))
    with pytest.raises(RuntimeError, match="the topology is fixed"):
        r.update_vertices(0, 0, np.zeros((5, 3), F32))
    with pytest.raises(RuntimeError, match="no lights"):
        r.update_lights([])
    lib, h = r.lib, r.h
    assert lib.crtc_update_instances(h, 0, 1, None) != 0 and "transforms is NULL" in lib.crtc_last_error().decode()
    nv = len(scene.meshes[0].geometries[0].vertices)
    assert lib.crtc_update_vertices(h, 0, 0, None, nv) != 0 and "vertices is NULL" in lib.crtc_last_error().decode()
    assert lib.crtc_update_lights(h, None, 1) != 0 and "lights is NULL" in lib.crtc_last_error().decode()
    assert lib.crtc_update_instances(h, 3, 0, None) == 0  # (an empty range stages nothing)
    # an empty commit renders on without a reset: the frames are those of a renderer that never committed
    plain = _renderer(RenderCUDA, scene, 16, 16)
    r.render(*args, True, True)
    plain.render(*args, True, True)
    r.commit_scene()
    r.render(*args, False, True)
    plain.render(*args, False, True)
    assert np.array_equal(r.read_accum().view(U32), plain.read_accum().view(U32))
    # failed updates staged nothing either
    r.commit_scene()
    r.render(*args, False, True)
    plain.render(*args, False, True)
    assert np.array_equal(r.read_accum().view(U32), plain.read_accum().view(U32))
