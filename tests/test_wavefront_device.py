"""The per-bounce kernels of kernels.cuh on the device, one launch at a time, against their host build fed the same
path state and against numpy restatements of their arithmetic.

libcrt_wave_devcheck.so (wave_devcheck.cu) launches the product's kernel templates on the grids enqueue_frame gives them,
on a full path state handed over by the test; wavefront_hostcheck.cpp exports the same entry points over one-lane
launches of the same source. The same .cu is built for the host under the SIMT emulation (tests/simt_emu: 32-lane
warps, real atomics), so every check runs without a GPU on the emulated twin and with ``-m gpu`` on an H100.

What is exact everywhere (uint32 views, NaN payloads aside): k_raygen against its restatement; k_nee_resolve against
its restatement fed the build's own miss_shader; k_resolve's accum, moments and scatter against the restatement, and
its img against the build's own float_to_srgb8; the shade-queue sort against numpy's stable sort by bucket; the
traversal's hit / vis against the host build; every byte a stage must not write; queues as multisets, each warp's
appends contiguous and in lane order; k_shade against a float32 restatement of its own glue (hit decode, uv, normal
flip, light choice, both NEE terms with MIS, shadow rays, continuation, Russian roulette) fed the build's own
unpack_material / disney_brdf / disney_pdf / sample_disney_brdf results on each path's inputs, and, on every path
where those results equal glibc's, against the host build. The same restatement fed glibc's results reproduces the
host build. CRT_SIMT_FULL=1 runs the larger emulated sizes."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from helpers import synthetic_material_scene
from test_shade_device import EDGE_DRAWS, Kat, _same, np_get_rng, np_lcg, states_before

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "chameleonrt_b200", "csrc")
FULL = os.environ.get("CRT_SIMT_FULL") == "1"
F32, U8, U32 = np.float32, np.uint8, np.uint32
MISS = 0xFFFFFFFF
TILE = 64
NUM_COUNTERS, CNT_QUEUE, CNT_SHADOW, CNT_WORK = 56, 0, 17, 36
EPS = F32(0.0001)
FLOAT4 = ("ray_o", "ray_d", "hit", "thr_rng", "radiance", "nee_T", "nee_l1", "nee_l2")
ARRAYS = FLOAT4 + ("sray_o", "sray_d", "vis", "queue0", "queue1", "counters")


# ---- the builds ----
class Wave:
    """The wavekat_* entry points of one build (wave_devcheck.cu or wavefront_hostcheck.cpp) on State objects."""

    def __init__(self, path, name, gpu):
        self.name, self.gpu = name, gpu
        self.lib = lib = C.CDLL(path)
        vp, i32, u32 = C.c_void_p, C.c_int, C.c_uint32
        lib.wavekat_last_error.restype = C.c_char_p
        lib.wavekat_scene.argtypes, lib.wavekat_scene.restype = [vp], vp
        lib.wavekat_scene_free.argtypes = [vp]
        sig = dict(raygen=[vp, u32, vp, vp, vp, u32, vp], traverse=[vp, i32, i32, i32, i32, i32, u32, vp],
                   shade=[vp, i32, i32, u32, vp], nee_resolve=[i32, u32, vp, vp],
                   resolve=[vp, vp, u32, vp, vp, u32, vp, vp, vp, vp, u32, vp], queue_sort=[vp, i32, u32, vp, vp])
        for k, a in sig.items():
            f = getattr(lib, "wavekat_" + k)
            f.argtypes, f.restype = a, C.c_int
        self.scenes = {}

    def scene(self, key, scene):
        if key not in self.scenes:
            ms = scene.to_c()
            h = self.lib.wavekat_scene(C.byref(ms.c))
            assert h, f"{self.name}: {self.lib.wavekat_last_error().decode()}"
            self.scenes[key] = h
        return self.scenes[key]

    def _call(self, fn, *args):
        rc = getattr(self.lib, "wavekat_" + fn)(*[a.ctypes.data if isinstance(a, np.ndarray) else a for a in args])
        assert rc == 0, f"{self.name}: wavekat_{fn}: {self.lib.wavekat_last_error().decode()}"

    def raygen(self, st, view, frame_id, lay, sel=None):
        out = st.copy()
        self._call("raygen", np.ascontiguousarray(view.vec, F32), frame_id, lay.arr, lay.tiles,
                   None if sel is None else np.ascontiguousarray(sel, U32), out.cap, out.ptrs())
        return out

    def traverse(self, scene, st, queue_index, closest, any_, work, far_first=False):
        out = st.copy()
        self._call("traverse", scene, queue_index, closest, any_, work, int(far_first), out.cap, out.ptrs())
        return out

    def shade(self, scene, st, bounce, max_depth):
        out = st.copy()
        self._call("shade", scene, bounce, max_depth, out.cap, out.ptrs())
        return out

    def nee_resolve(self, st, bounce):
        out = st.copy()
        grid = np.zeros(1, U32)
        self._call("nee_resolve", bounce, out.cap, out.ptrs(), grid)
        return out, int(grid[0])

    def resolve(self, st, lay, frame_id, accum, img, full=None, sel=None, moments=None, stat_base=0):
        out = st.copy()
        accum, img = accum.copy(), img.copy()
        fa, fi = (None, None) if full is None else (full[0].copy(), full[1].copy())
        mom = None if moments is None else moments.copy()
        self._call("resolve", lay.arr, lay.tiles, frame_id, None if sel is None else np.ascontiguousarray(sel, U32), mom,
                   stat_base, accum, img, fa, fi, out.cap, out.ptrs())
        return out, accum, img, fa, fi, mom

    def queue_sort(self, scene, st, bounce):
        out = st.copy()
        sorted_ = np.full(out.cap, 0xA5A5A5A5, U32)
        self._call("queue_sort", scene, bounce, out.cap, out.ptrs(), sorted_)
        return out, sorted_


class State:
    """A full PathState image of `cap` paths (wave_devcheck.cu: the order of `st`)."""

    def __init__(self, cap, seed=0, arrays=None):
        self.cap = cap
        if arrays is not None:
            self.a = arrays
            return
        rng = np.random.default_rng(seed)
        self.a = {k: rng.standard_normal((cap, 4)).astype(F32) for k in FLOAT4}
        for k in ("sray_o", "sray_d"):
            self.a[k] = rng.standard_normal((2 * cap, 4)).astype(F32)
        self.a["vis"] = rng.integers(0, 256, 2 * cap, dtype=U8)
        for k in ("queue0", "queue1"):
            self.a[k] = rng.integers(0, 2**32, cap, dtype=np.uint64).astype(U32)
        self.a["counters"] = np.zeros(NUM_COUNTERS, U32)

    def __getitem__(self, k):
        return self.a[k]

    def copy(self):
        return State(self.cap, arrays={k: v.copy() for k, v in self.a.items()})

    def ptrs(self):
        self._keep = (C.c_void_p * len(ARRAYS))(*[self.a[k].ctypes.data for k in ARRAYS])
        return self._keep

    def queue(self, b):
        return self.a["queue0" if b % 2 == 0 else "queue1"]

    def u(self, k):
        return self.a[k].view(U32)


@pytest.fixture(scope="module")
def host(built):
    return Wave(os.path.join(CSRC, "libcrt_wavefront_hostcheck.so"), "host", False)


@pytest.fixture(scope="module")
def emulated(built):
    sys.path.insert(0, os.path.join(ROOT, "tests", "simt_emu"))
    import build_wave

    return Wave(build_wave.build_wave_devcheck(), "emulated", False)


@pytest.fixture(scope="module")
def device(built):
    path = os.path.join(CSRC, "libcrt_wave_devcheck.so")
    if not os.path.exists(path):  # (a tree built before the check library existed)
        subprocess.check_call(["make", "-s", "-C", CSRC, "libcrt_wave_devcheck.so"])
    return Wave(path, "device", True)


@pytest.fixture(params=[pytest.param("emulated"), pytest.param("device", marks=pytest.mark.gpu)], scope="module")
def dev(request):
    """The device build under test: the SIMT emulation without a GPU, the sm_90a build with ``-m gpu``."""
    return request.getfixturevalue(request.param)


@pytest.fixture(scope="module")
def kats(built, dev):
    """The shading functions as the build under test computes them, and glibc's."""
    hk = Kat(os.path.join(CSRC, "libcrt_shade_hostcheck.so"), "host")
    if not dev.gpu:
        return hk, hk
    path = os.path.join(CSRC, "libcrt_shade_devcheck.so")
    if not os.path.exists(path):
        subprocess.check_call(["make", "-s", "-C", CSRC, "libcrt_shade_devcheck.so"])
    return Kat(path, "device"), hk


# ---- frame layouts and views ----
class Layout:
    def __init__(self, w, h, spp, frames, rank=0, world=1):
        self.w, self.h, self.spp, self.frames = w, h, spp, frames
        self.ntx = -(-w // TILE)
        ntiles = self.ntx * -(-h // TILE)
        self.tiles = np.array([t for t in range(ntiles) if t % world == rank], U32)
        self.npx = len(self.tiles) * TILE * TILE
        self.arr = np.array([w, h, self.ntx, self.npx, spp, frames, len(self.tiles)], U32)
        self.npaths = self.npx * spp * frames

    def coords(self, lp):
        """Local pixel -> (x, y, inside the framebuffer) (kernels.cuh: local_pixel_coords)."""
        lp = np.asarray(lp, np.int64)
        tile = self.tiles[lp // 4096].astype(np.int64)
        within = lp % 4096
        blk, lane = within >> 5, within & 31
        x = (tile % self.ntx) * TILE + (blk & 7) * 8 + (lane & 7)
        y = (tile // self.ntx) * TILE + (blk >> 3) * 4 + (lane >> 3)
        return x, y, (x < self.w) & (y < self.h)


class View:
    def __init__(self, pos, dir_, up, fovy, w, h):
        """A camera basis in the layout of make_view_params (computed here in float64: any 12 floats do)."""
        d, u = np.asarray(dir_, np.float64), np.asarray(up, np.float64)
        py = 2 * np.tan(np.radians(fovy) / 2)
        du = np.cross(d, u)
        du = du / np.linalg.norm(du) * py * w / h
        dv = np.cross(du, d)
        dv = -dv / np.linalg.norm(dv) * py
        tl = d - 0.5 * du - 0.5 * dv
        self.vec = np.concatenate([pos, du, dv, tl]).astype(F32)


def cam_view(cam, lay):
    d = np.subtract(cam["center"], cam["eye"])
    return View(cam["eye"], d / np.linalg.norm(d), cam["up"], cam["fov_y"], lay.w, lay.h)


# ---- scenes ----
def cornell(spp=1):
    from chameleonrt_b200.scenes import cornell_box

    return cornell_box(spp)


def lights_scene(spp=1):
    """Cornell with three quad lights of different sizes and emissions (the light choice)."""
    from chameleonrt_b200.scene import QuadLight

    scene, cam = cornell(spp)
    scene.lights = [QuadLight((8.0, 8.0, 8.0), (-0.3, 1.98, -0.3), (0.0, -1.0, 0.0), (1.0, 0.0, 0.0), 0.3, (0.0, 0.0, 1.0), 0.2),
                    QuadLight((2.0, 4.0, 9.0), (0.6, 1.5, -0.99), (0.0, 0.0, 1.0), (1.0, 0.0, 0.0), 0.2, (0.0, 1.0, 0.0), 0.3),
                    QuadLight((5.0, 1.0, 1.0), (-0.99, 0.4, 0.2), (1.0, 0.0, 0.0), (0.0, 0.0, 1.0), 0.4, (0.0, 1.0, 0.0), 0.1)]
    return scene, cam


def many_materials_scene(n_mat=300):
    """A soup whose triangles use n_mat materials (ids past 254 share the sort's bucket 254)."""
    from chameleonrt_b200.scene import DisneyMaterial, Geometry, Instance, Mesh, ParameterizedMesh, Scene, default_obj_light

    rng = np.random.default_rng(5)
    geoms = []
    for g in range(n_mat):
        c = rng.uniform(-1, 1, (2, 1, 3))
        v = (c + rng.normal(scale=0.05, size=(2, 3, 3))).astype(F32).reshape(-1, 3)
        geoms.append(Geometry(v, np.arange(6, dtype=U32).reshape(2, 3)))
    return Scene(meshes=[Mesh(geoms)], parameterized_meshes=[ParameterizedMesh(0, list(range(n_mat)))],
                 instances=[Instance(np.eye(4, dtype=F32), 0)], materials=[DisneyMaterial() for _ in range(n_mat)],
                 lights=[default_obj_light()])


SCENES = {"cornell": cornell, "materials": synthetic_material_scene, "lights": lights_scene}


# ---- checks shared by the stages ----
def same_bits(a, b):
    return _same(np.asarray(a, F32).ravel(), np.asarray(b, F32).ravel())


def row_same(a, b):
    """Per row: bit for bit, NaN payloads aside."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    eq = (a.view(U32) == b.view(U32)) | (np.isnan(a) & np.isnan(b))
    return eq.reshape(len(a), -1).all(1)


def warp_runs(producer, group=None, lanes=32):
    """Each warp's appends (one warp_append call: `group`) sit in consecutive queue positions, in lane order.
    `producer`: the thread that wrote each queue entry, in queue order; `lanes`: the build's warp width."""
    producer = np.asarray(producer, np.int64)
    key = producer // lanes if group is None else (producer // lanes) * 2 + np.asarray(group, np.int64)
    pos = np.lexsort((np.arange(len(key)), key))  # queue positions grouped by warp, ascending within a warp
    same = key[pos][1:] == key[pos][:-1]
    gap = np.nonzero(same & (np.diff(pos) != 1))[0]
    assert len(gap) == 0, f"warp {key[pos][gap[0]] if len(gap) else 0}: appends at non-consecutive queue positions"
    back = np.nonzero(same & (np.diff(producer[pos]) <= 0))[0]
    assert len(back) == 0, f"warp {key[pos][back[0]] if len(back) else 0}: appends out of lane order"


def untouched(before, after, keep, what):
    """The rows `keep` of every path-state array are the bytes they were."""
    for k in FLOAT4:
        assert np.array_equal(after.u(k)[keep], before.u(k)[keep]), f"{what}: {k} written outside the queue"


# ---- k_raygen ----
def np_raygen(view, frame_id, lay, sel=None):
    """kernels.cuh k_raygen, float32, -fmad=false: (valid, ray_d, rng state) per path."""
    i = np.arange(lay.npaths, dtype=np.int64)
    lp, s = i % lay.npx, i // lay.npx
    x, y, inside = lay.coords(lp)
    first = np.full(len(i), frame_id, np.uint64)
    active = np.ones(len(i), bool)
    if sel is not None:
        first = sel[lp >> 5, 0].astype(np.uint64)
        active = s < sel[lp >> 5, 1].astype(np.int64) * lay.spp
    valid = inside & active
    m32 = 0xFFFFFFFF
    frame = (first * np.uint64(lay.spp) + np.uint64(1) + s.astype(np.uint64)) & np.uint64(m32)
    rng = np_get_rng(((x + y * lay.w) & m32).astype(U32), frame.astype(U32))
    rng, r1 = np_lcg(rng)
    rng, r2 = np_lcg(rng)
    px = (x.astype(F32) + r1) / F32(lay.w)
    py = (y.astype(F32) + r2) / F32(lay.h)
    v = view.vec
    d = [v[3 + c] * px + v[6 + c] * py + v[9 + c] for c in range(3)]
    inv = F32(1) / np.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2])
    return valid, np.stack([d[0] * inv, d[1] * inv, d[2] * inv], 1), rng


def check_raygen(st, got, view, frame_id, lay, sel=None):
    valid, dirs, rng = np_raygen(view, frame_id, lay, sel)
    n = int(valid.sum())
    assert got["counters"][CNT_QUEUE] == n and np.all(got["counters"][1:] == st["counters"][1:])
    q = got["queue0"][:n].astype(np.int64)
    assert np.array_equal(np.sort(q), np.nonzero(valid)[0]), "raygen queue: wrong paths"
    assert np.array_equal(got["queue0"][n:], st["queue0"][n:]), "raygen queue: written past its length"
    warp_runs(q)
    idx = np.nonzero(valid)[0]
    assert same_bits(got["ray_d"][idx, :3], dirs[idx]), "raygen: ray directions"
    assert np.all(got["ray_d"][idx, 3] == F32(1e20))
    assert same_bits(got["ray_o"][idx], np.concatenate([np.broadcast_to(view.vec[:3], (len(idx), 3)), np.zeros((len(idx), 1), F32)], 1))
    assert np.array_equal(got.u("thr_rng")[idx, 3], rng[idx]) and np.all(got["thr_rng"][idx, :3] == F32(1))
    assert np.all(got.u("radiance")[idx] == 0)
    keep = np.ones(st.cap, bool)
    keep[idx] = False
    for k in ("ray_o", "ray_d", "thr_rng", "radiance"):
        assert np.array_equal(got.u(k)[keep], st.u(k)[keep]), f"raygen: {k} written for an invalid path"
    for k in ("hit", "nee_T", "nee_l1", "nee_l2", "sray_o", "sray_d", "vis", "queue1"):
        assert np.array_equal(got[k].view(U8), st[k].view(U8)), f"raygen: {k} written"


RAYGEN_CASES = [
    # (w, h, spp, frames, rank, world, frame_id)
    (70, 45, 2, 2, 0, 1, 0),
    (130, 70, 1, 1, 1, 2, 5),
    (70, 45, 3, 2, 0, 1, 0x55555555),  # frame_id * spp + 1 + s wraps past 2^32
    (33, 97, 1, 3, 0, 1, 2**32 - 2),
]


@pytest.mark.parametrize("case", RAYGEN_CASES, ids=lambda c: "x".join(map(str, c[:2])) + f"_spp{c[2]}_f{c[3]}_r{c[4]}of{c[5]}_id{c[6]}")
def test_raygen_matches_restatement(dev, host, case):
    w, h, spp, frames, rank, world, fid = case
    lay = Layout(w, h, spp, frames, rank, world)
    view = View((0.1, 1.0, 3.4), (0.05, -0.1, -1.0), (0, 1, 0), 40.0, w, h)
    st = State(lay.npaths + 37, seed=1)
    got = dev.raygen(st, view, fid, lay)
    check_raygen(st, got, view, fid, lay)
    ref = host.raygen(st, view, fid, lay)
    check_raygen(st, ref, view, fid, lay)


def test_raygen_adaptive_selection(dev, host):
    lay = Layout(70, 45, 2, 3)
    rng = np.random.default_rng(3)
    nblk = lay.npx // 32
    sel = np.stack([rng.integers(0, 2**32 - 8, nblk, dtype=np.uint64), rng.integers(0, 4, nblk)], 1).astype(U32)
    sel[::5, 1] = 0  # inactive blocks
    view = View((0.0, 1.0, 3.4), (0.0, 0.0, -1.0), (0, 1, 0), 40.0, lay.w, lay.h)
    st = State(lay.npaths, seed=2)
    for w in (dev, host):
        check_raygen(st, w.raygen(st, view, 7, lay, sel), view, 7, lay, sel)


# ---- k_nee_resolve ----
def np_nee_resolve(st, qin, count, miss):
    """kernels.cuh k_nee_resolve in float32 on the slots queue[:count]; `miss(dirs)` is the build's miss_shader."""
    out = st["radiance"].copy()
    slots = qin[:count].astype(np.int64)
    T = st["nee_T"][slots]
    flags = T[:, 3].view(U32)
    rad = out[slots]
    m = (flags & 4) != 0
    if m.any():
        c = T[m, :3] * miss(st["ray_d"][slots[m], :3])
        rad[m, :3] = rad[m, :3] + c
    h = ~m
    vis = st["vis"]
    illum = np.zeros((len(slots), 3), F32)
    a = h & ((flags & 8) != 0) & (vis[2 * slots] != 0)
    illum[a] = st["nee_l1"][slots[a], :3]
    b = h & ((flags & 1) != 0) & (vis[2 * slots + 1] != 0)
    illum[b] = illum[b] + st["nee_l2"][slots[b], :3]
    rad[h, :3] = rad[h, :3] + T[h, :3] * illum[h]
    out[slots] = rad
    return out


def nee_state(cap, count, seed):
    st = State(cap, seed)
    rng = np.random.default_rng(seed)
    slots = rng.permutation(cap)[:count].astype(U32)
    st.queue(0)[:count] = slots
    st["counters"][CNT_QUEUE] = count
    flags = rng.choice(np.array([4, 2, 3, 10, 11, 8, 9, 1, 0, 15], U32), cap)
    st["nee_T"][:, 3] = flags.view(F32)
    st["vis"][:] = rng.integers(0, 2, 2 * cap, dtype=U8) * rng.integers(1, 256, 2 * cap, dtype=U8)
    d = rng.standard_normal((cap, 3)).astype(F32)
    st["ray_d"][:, :3] = d / np.linalg.norm(d, axis=1, keepdims=True).astype(F32)
    edge = np.array([0, np.inf, np.nan, 1e-40, -0.0, 3e38, 1], F32)[:cap]
    st["nee_T"][:len(edge), :3] = edge[:, None]
    return st


def check_nee(dev, host, kats, cap, count, seed):
    st = nee_state(cap, count, seed)
    got, grid = dev.nee_resolve(st, 0)
    want = np_nee_resolve(st, st.queue(0), count, kats[0].miss)
    assert same_bits(got["radiance"], want), f"{dev.name}: k_nee_resolve against the restatement"
    ref, _ = host.nee_resolve(st, 0)
    assert same_bits(ref["radiance"], np_nee_resolve(st, st.queue(0), count, kats[1].miss)), "host: k_nee_resolve"
    for k in ARRAYS:
        if k != "radiance":
            assert np.array_equal(got[k].view(U8), st[k].view(U8)), f"{dev.name}: k_nee_resolve wrote {k}"
    return grid


def test_nee_resolve_matches_restatement(dev, host, kats):
    for cap, count in ((1, 0), (1, 1), (300, 257), (700, 31)):
        check_nee(dev, host, kats, cap, count, seed=cap + count)


def test_nee_resolve_grid_stride_loop(dev, host, kats):
    """A queue longer than the capped grid (num_sms * 16 blocks of 256): the stride loop runs more than once."""
    cap = 600_000 if dev.gpu else 9_000
    grid = check_nee(dev, host, kats, cap, cap - 123, seed=9)
    assert grid * 256 < cap - 123, (grid, cap)


# ---- k_resolve ----
def np_resolve(lay, st, frame_id, accum, sel=None, moments=None, stat_base=0):
    """kernels.cuh k_resolve in float32: (accum, moments, mask of the pixels written)."""
    lp = np.arange(lay.npx)
    _, _, inside = lay.coords(lp)
    first = np.full(lay.npx, frame_id, np.uint64)
    frames = np.full(lay.npx, lay.frames, np.int64)
    if sel is not None:
        first, frames = sel[lp >> 5, 0].astype(np.uint64), sel[lp >> 5, 1].astype(np.int64)
    wrote = inside & (frames != 0)
    illum = accum.reshape(-1, 3).copy()
    m = moments.copy() if moments is not None else None
    rad = st["radiance"]
    for k in range(int(frames.max(initial=0))):
        act = wrote & (frames > k)
        acc = illum.copy()
        s = np.zeros((lay.npx, 3), F32)
        s1, s2 = np.zeros(lay.npx, F32), np.zeros(lay.npx, F32)
        for j in range(lay.spp):
            r = rad[(k * lay.spp + j) * lay.npx + lp, :3]
            s = s + r
            lum = F32(0.2126) * r[:, 0] + F32(0.7152) * r[:, 1] + F32(0.0722) * r[:, 2]
            s1, s2 = s1 + lum, s2 + lum * lum
        s = s / F32(lay.spp)
        n = (first + np.uint64(k)) & np.uint64(0xFFFFFFFF)
        n1 = (n + np.uint64(1)) & np.uint64(0xFFFFFFFF)
        new = (s + n.astype(U32).astype(F32)[:, None] * acc) / n1.astype(U32).astype(F32)[:, None]
        illum[act] = new[act]
        if m is not None:
            c = ((n - np.uint64(stat_base)) & np.uint64(0xFFFFFFFF)).astype(U32)
            c1 = (c.astype(np.uint64) + 1).astype(U32)
            mx = (s1 / F32(lay.spp) + c.astype(F32) * m[:, 0]) / c1.astype(F32)
            my = (s2 / F32(lay.spp) + c.astype(F32) * m[:, 1]) / c1.astype(F32)
            m[act, 0], m[act, 1] = mx[act], my[act]
    return illum, m, wrote


def check_resolve(dev, kats, lay, frame_id, seed, sel=None, stat_base=0, nan=False, st=None):
    """k_resolve on `st` (default: random radiance) against the restatement: accum, moments, img, the full-frame
    scatter, and nothing else written."""
    rng = np.random.default_rng(seed)
    if st is None:
        st = State(lay.npaths, seed)
        st["radiance"][:] = np.abs(rng.standard_normal((lay.npaths, 4))).astype(F32) * F32(2)
    if nan:
        st["radiance"][::97, 1] = np.nan
        st["radiance"][5::101, 0] = np.inf
    accum = np.abs(rng.standard_normal(3 * lay.npx)).astype(F32)
    img = rng.integers(0, 2**32, lay.npx, dtype=np.uint64).astype(U32)
    full = (rng.standard_normal(3 * lay.w * lay.h).astype(F32), rng.integers(0, 2**32, lay.w * lay.h, dtype=np.uint64).astype(U32))
    moments = rng.standard_normal((lay.npx, 2)).astype(F32) if sel is not None else None
    got, acc, im, fa, fi, mom = dev.resolve(st, lay, frame_id, accum, img, full, sel, moments, stat_base)
    want, want_m, wrote = np_resolve(lay, st, frame_id, accum, sel, moments, stat_base)
    what = f"{dev.name}: k_resolve {lay.w}x{lay.h} spp {lay.spp} frames {lay.frames} frame_id {frame_id}"
    assert same_bits(acc.reshape(-1, 3), want), what + ": accum"
    assert np.array_equal(acc.reshape(-1, 3)[~wrote].view(U32), accum.reshape(-1, 3)[~wrote].view(U32)), what + ": stray accum"
    srgb = kats[0].srgb8(acc.reshape(-1, 3)[wrote].ravel()).reshape(-1, 3).astype(U32)
    assert np.array_equal(im[wrote], srgb[:, 0] | (srgb[:, 1] << 8) | (srgb[:, 2] << 16) | 0xFF000000), what + ": img"
    assert np.array_equal(im[~wrote], img[~wrote]), what + ": stray img"
    if sel is not None:
        assert same_bits(mom, want_m), what + ": moments"
    x, y, _ = lay.coords(np.nonzero(wrote)[0])
    p = y * lay.w + x
    want_fa, want_fi = full[0].reshape(-1, 3).copy(), full[1].copy()
    want_fa[p], want_fi[p] = acc.reshape(-1, 3)[wrote], im[wrote]
    assert same_bits(fa, want_fa) and np.array_equal(fi, want_fi), what + ": accum_full / img_full scatter"
    for k in ARRAYS:
        assert np.array_equal(got[k].view(U8), st[k].view(U8)), what + f": wrote {k}"


RESOLVE_CASES = [
    # (w, h, spp, frames, frame_id)
    (70, 45, 1, 1, 0),
    (70, 45, 3, 2, 2**24 - 1),
    (65, 64, 16, 1, 2**24 + 3),
    (40, 30, 1, 4, 2**24 - 2),
    (40, 30, 3, 3, 2**32 - 2),
]


@pytest.mark.parametrize("case", RESOLVE_CASES, ids=lambda c: f"{c[0]}x{c[1]}_spp{c[2]}_f{c[3]}_id{c[4]}")
def test_resolve_matches_restatement(dev, host, kats, case):
    w, h, spp, frames, fid = case
    lay = Layout(w, h, spp, frames)
    check_resolve(dev, kats, lay, fid, seed=fid % 1000 + spp, nan=spp == 3)
    check_resolve(host, (kats[1], kats[1]), lay, fid, seed=fid % 1000 + spp, nan=spp == 3)


def test_resolve_adaptive(dev, host, kats):
    lay = Layout(70, 45, 2, 3)
    rng = np.random.default_rng(8)
    nblk = lay.npx // 32
    sel = np.stack([rng.integers(2**24 - 4, 2**24 + 4, nblk), rng.integers(0, 4, nblk)], 1).astype(U32)
    sel[::4, 1] = 0  # blocks with n_b = 0 keep every buffer
    for w, k in ((dev, kats), (host, (kats[1], kats[1]))):
        check_resolve(w, k, lay, 0, seed=4, sel=sel, stat_base=2**24 - 9)


# ---- the shade-queue sort ----
def test_queue_sort_is_stable_by_bucket(dev, host):
    from helpers import HostCheck

    scene = many_materials_scene()
    shade = HostCheck(scene).export()[3]
    mat = shade[:, 3].view(U32)
    ntri = len(shade)
    lengths = (2048 * 3 + 517, 1, 2048) if not dev.gpu else (2048 * 40 + 517, 1, 2048, 200_000)
    for n in lengths:
        cap = n + 300
        rng = np.random.default_rng(n)
        st = State(cap, seed=n)
        tri = rng.integers(0, ntri, cap).astype(U32)
        tri[rng.random(cap) < 0.2] = MISS
        st["hit"][:, 3] = tri.view(F32)
        st.queue(1)[:n] = rng.permutation(cap)[:n].astype(U32)
        st["counters"][CNT_QUEUE + 1] = n
        q = st.queue(1)[:n]
        t = tri[q]
        bucket = np.where(t == MISS, 255, np.minimum(mat[np.where(t == MISS, 0, t)], 254))
        want = q[np.argsort(bucket, kind="stable")]
        for w in (dev, host):
            got, sorted_ = w.queue_sort(w.scene("materials300", scene), st, 1)
            assert np.array_equal(sorted_[:n], want), f"{w.name}: sorted queue of {n}"
            assert np.all(sorted_[n:] == 0xA5A5A5A5), f"{w.name}: sort wrote past the queue"
            for k in ARRAYS:
                assert np.array_equal(got[k].view(U8), st[k].view(U8)), f"{w.name}: sort wrote {k}"


# ---- k_shade ----
def shade_outputs(st, b):
    """The canonical outputs of k_shade: the continuation queue as a sorted array, the shadow rays keyed by
    sray_d.w (slot * 2 + which)."""
    n_next = int(st["counters"][CNT_QUEUE + b + 1])
    n_sh = int(st["counters"][CNT_SHADOW + b])
    qo = np.sort(st.queue(b + 1)[:n_next])
    keys = st.u("sray_d")[:n_sh, 3]
    order = np.argsort(keys)
    return qo, keys[order], st["sray_o"][:n_sh][order], st["sray_d"][:n_sh][order]


def check_shade_structure(st, got, b, max_depth, name, lanes):
    """What k_shade must do whatever its transcendentals return."""
    count = int(st["counters"][CNT_QUEUE + b])
    qin = st.queue(b)[:count].astype(np.int64)
    pos = np.full(st.cap, -1, np.int64)
    pos[qin] = np.arange(count)
    c = got["counters"]
    others = [i for i in range(NUM_COUNTERS) if i not in (CNT_QUEUE + b + 1, CNT_SHADOW + b)]
    assert np.array_equal(c[others], st["counters"][others]), f"{name}: counters"
    tri = st.u("hit")[:, 3]
    hit = np.zeros(st.cap, bool)
    hit[qin] = tri[qin] != MISS
    miss = np.zeros(st.cap, bool)
    miss[qin] = tri[qin] == MISS
    # misses: throughput and flag 4, nothing else
    assert np.array_equal(got.u("nee_T")[miss, :3], st.u("thr_rng")[miss, :3]) and np.all(got.u("nee_T")[miss, 3] == 4), f"{name}: miss terms"
    fl = got.u("nee_T")[hit, 3]
    assert np.all((fl & 2) != 0) and np.all((fl & ~np.uint32(11)) == 0), f"{name}: hit flags"
    assert np.array_equal(got.u("nee_T")[hit, :3], st.u("thr_rng")[hit, :3]), f"{name}: throughput before the bounce"
    # shadow rays: A for every hit, B exactly where flag 1 is set, at the hit point o + t d
    n_sh = int(c[CNT_SHADOW + b]) - int(st["counters"][CNT_SHADOW + b])
    base = int(st["counters"][CNT_SHADOW + b])
    keys = got.u("sray_d")[base:base + n_sh, 3].astype(np.int64)
    slots, which = keys >> 1, keys & 1
    want_a = np.nonzero(hit)[0]
    want_b = np.nonzero(hit & ((got.u("nee_T")[:, 3] & 1) != 0))[0]
    assert np.array_equal(np.sort(slots[which == 0]), want_a) and np.array_equal(np.sort(slots[which == 1]), want_b), f"{name}: shadow queue"
    ro, rd, h = st["ray_o"][slots], st["ray_d"][slots], st["hit"][slots]
    p = np.stack([ro[:, i] + h[:, 0] * rd[:, i] for i in range(3)], 1)
    assert same_bits(got["sray_o"][base:base + n_sh, :3], p), f"{name}: shadow ray origins"
    warp_runs(pos[slots], which, lanes)
    # continuation: exactly the slots whose ray was rewritten, never past max_depth, nothing on misses
    n_next = int(c[CNT_QUEUE + b + 1])
    qo = got.queue(b + 1)[:n_next].astype(np.int64)
    assert len(np.unique(qo)) == n_next and np.all(hit[qo]), f"{name}: continuation queue"
    if b + 1 >= max_depth:
        assert n_next == 0, f"{name}: continued past max_depth"
    rewritten = ~row_same(got["ray_o"], st["ray_o"]) | ~row_same(got["ray_d"], st["ray_d"])
    assert np.array_equal(np.nonzero(rewritten)[0], np.sort(qo)), f"{name}: rays rewritten outside the continuation queue"
    assert np.all(got["ray_o"][qo, 3] == EPS) and np.all(got["ray_d"][qo, 3] == F32(1e20))
    warp_runs(pos[qo], lanes=lanes)
    assert np.array_equal(got.queue(b + 1)[n_next:], st.queue(b + 1)[n_next:]), f"{name}: continuation queue written past its length"
    assert np.array_equal(got.queue(b), st.queue(b)), f"{name}: queue_in written"
    # no stray writes
    keep = np.ones(st.cap, bool)
    keep[qin] = False
    untouched(st, got, keep, name)
    for k in ("hit", "radiance"):
        assert np.array_equal(got.u(k), st.u(k)), f"{name}: {k} written"
    assert np.array_equal(got.u("sray_o")[base + n_sh:], st.u("sray_o")[base + n_sh:]), f"{name}: shadow rays past the count"
    assert np.array_equal(got["vis"], st["vis"])


def scene_records(host, handle):
    """The records both builds upload (pack_scene), from the host build: shading records, materials, lights, texel
    arena, texture descriptors."""
    lib = host.lib
    lib.wavekat_records.argtypes, lib.wavekat_records.restype = [C.c_void_p, C.c_int, C.c_void_p], C.c_longlong
    out = []
    for field, (dt, width) in enumerate(((F32, 12), (F32, 16), (F32, 20), (U32, 1), (np.int32, 4))):
        n = lib.wavekat_records(handle, field, None)
        a = np.zeros(max(n // 4, width), dt)
        assert lib.wavekat_records(handle, field, a.ctypes.data) == n
        out.append(a.reshape(-1, width) if width > 1 else a)
    return dict(zip(("shade", "materials", "lights", "texels", "tex"), out))


def _dot(a, b):
    return (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]


def _normalize(v):
    return v * (F32(1) / np.sqrt(_dot(v, v)))[:, None]


def _power_heuristic(f, g):
    return (f * f) / (f * f + g * g)


def _quad_pdf(L, p, d):
    """quad_light_pdf (lights.ih: to_pt = p - dir)."""
    area = L[:, 15] * L[:, 19]
    to_pt = p - d
    ndw = _dot(L[:, 8:11], -d)
    with np.errstate(all="ignore"):
        return np.where(ndw < EPS, F32(0), _dot(to_pt, to_pt) / (ndw * area)).astype(F32)


def _quad_intersect(L, o, d):
    """quad_intersect: (hit, t, light_pos)."""
    with np.errstate(all="ignore"):
        denom = _dot(d, L[:, 8:11])
        t = _dot(L[:, 4:7] - o, L[:, 8:11]) / denom
        lp = o + d * t[:, None]
        hv = lp - L[:, 4:7]
        hit = (denom != 0) & ~(t < 0) & (np.abs(_dot(hv, L[:, 12:15])) < L[:, 15]) & (np.abs(_dot(hv, L[:, 16:19])) < L[:, 19])
    return hit, t, lp


class ShadeCalls:
    """The shading functions k_shade calls, from one build's shadekat library; `other` (glibc's) is evaluated on the
    same inputs, and every path where a result differs is marked."""

    def __init__(self, kat, other, rec):
        self.kat, self.other, self.rec = kat, other, rec
        self.differs = None

    def _mark(self, rows, a, b):
        if self.differs is not None:
            self.differs[rows] |= ~row_same(a, b)

    def unpack(self, rows, mid, uv):
        out = np.zeros((len(mid), 16), F32)
        for m in np.unique(mid):
            k = mid == m
            args = (self.rec["materials"], int(m), self.rec["texels"], self.rec["tex"], uv[k])
            out[k, :14] = self.kat.unpack(*args)
            if self.other is not self.kat:
                self._mark(rows[k], out[k, :14], self.other.unpack(*args))
        return out

    def eval(self, rows, mat, n, wo, wi):
        if len(rows) == 0:
            return np.zeros((0, 4), F32)
        r = self.kat.eval(mat, n, wo, wi)
        if self.other is not self.kat:
            self._mark(rows, r, self.other.eval(mat, n, wo, wi))
        return r

    def sample(self, rows, mat, n, wo, rng):
        if len(rows) == 0:
            return np.zeros((0, 7), F32), np.zeros(0, U32)
        r, s = self.kat.sample(mat, n, wo, rng)
        if self.other is not self.kat:
            r2, s2 = self.other.sample(mat, n, wo, rng)
            self._mark(rows, np.concatenate([r, s.view(F32)[:, None]], 1), np.concatenate([r2, s2.view(F32)[:, None]], 1))
        return r, s


def np_shade(st, b, max_depth, calls):
    """kernels.cuh k_shade<false> in float32 (operation order as in the source, -fmad=false) on queue[b][:count],
    with the shading functions' results from `calls`. Returns the expected outputs: per-slot nee_T / nee_l1 / nee_l2
    rows, shadow rays keyed by slot * 2 + which, and the continuation's slots with their ray_o / ray_d / thr_rng."""
    rec = calls.rec
    count = int(st["counters"][CNT_QUEUE + b])
    slots = st.queue(b)[:count].astype(np.int64)
    calls.differs = np.zeros(st.cap, bool)
    ro, rd, h, tr = st["ray_o"][slots], st["ray_d"][slots], st["hit"][slots], st["thr_rng"][slots]
    tri = h[:, 3].view(U32)
    thr = tr[:, :3]
    nee_T = np.concatenate([thr, np.full((count, 1), np.uint32(4).view(F32), F32)], 1)
    hit = tri != MISS
    H = np.nonzero(hit)[0]
    sl = slots[H]
    d, o, hh, thr = rd[H, :3], ro[H, :3], h[H], thr[H].copy()
    rng = tr[H, 3].view(U32).copy()
    w_o = -d
    hit_p = o + hh[:, :1] * d
    sh = rec["shade"][tri[H]]
    normal = sh[:, 0:3].copy()
    mid = sh[:, 3].view(U32)
    uv = np.zeros((len(H), 2), F32)
    has_uv = sh[:, 10].view(U32) != 0
    bw = (F32(1) - hh[:, 1]) - hh[:, 2]
    uv[:, 0] = np.where(has_uv, (sh[:, 4] * bw + sh[:, 6] * hh[:, 1]) + sh[:, 8] * hh[:, 2], F32(0))
    uv[:, 1] = np.where(has_uv, (sh[:, 5] * bw + sh[:, 7] * hh[:, 1]) + sh[:, 9] * hh[:, 2], F32(0))
    mat = calls.unpack(sl, mid, uv)
    flip = (mat[:, 13] == 0) & (_dot(w_o, normal) < 0)
    normal[flip] = -normal[flip]
    # sample_direct_light: the light sample
    nl = len(rec["lights"])
    rng, r0 = np_lcg(rng)
    light_id = np.minimum((r0 * F32(nl)).astype(np.int64), nl - 1)
    L = rec["lights"][light_id]
    rng, sx = np_lcg(rng)
    rng, sy = np_lcg(rng)
    lpos = ((L[:, 12:15] * sx[:, None]) * L[:, 15:16] + (L[:, 16:19] * sy[:, None]) * L[:, 19:20]) + L[:, 4:7]
    ldir = lpos - hit_p
    ldist = np.sqrt(_dot(ldir, ldir))
    ldir = _normalize(ldir)
    lpdf = _quad_pdf(L, lpos, ldir)
    ev = calls.eval(sl, mat, normal, w_o, ldir)
    has_l1 = (lpdf >= EPS) & (ev[:, 3] >= EPS)
    with np.errstate(all="ignore"):
        w = _power_heuristic(lpdf, ev[:, 3])
        l1 = (((ev[:, :3] * L[:, 0:3]) * np.abs(_dot(ldir, normal))[:, None]) * w[:, None]) / lpdf[:, None]
    # the BSDF sample
    sm, rng = calls.sample(sl, mat, normal, w_o, rng)
    bsdf, bpdf, wi = sm[:, :3], sm[:, 3], sm[:, 4:7]
    qhit, qt, qpos = _quad_intersect(L, hit_p, wi)
    nonzero = ~((bsdf[:, 0] == 0) & (bsdf[:, 1] == 0) & (bsdf[:, 2] == 0))
    with np.errstate(all="ignore"):
        qpdf = _quad_pdf(L, qpos, wi)
        emit_b = nonzero & (bpdf >= EPS) & qhit & (qpdf >= EPS)
        w = _power_heuristic(bpdf, qpdf)
        l2 = (((bsdf * L[:, 0:3]) * np.abs(_dot(wi, normal))[:, None]) * w[:, None]) / bpdf[:, None]
    flags = np.uint32(2) | emit_b.astype(U32) | (has_l1.astype(U32) << 3)
    nee_T[H, 3] = flags.view(F32)
    keys = np.concatenate([sl * 2, sl[emit_b] * 2 + 1])
    sray_o = np.concatenate([np.concatenate([hit_p, ldist[:, None]], 1), np.concatenate([hit_p[emit_b], qt[emit_b, None]], 1)])
    sray_d = np.concatenate([ldir, wi[emit_b]])
    order = np.argsort(keys)
    # the continuation
    sm, rng = calls.sample(sl, mat, normal, w_o, rng)
    bsdf, pdf, wi = sm[:, :3], sm[:, 3], sm[:, 4:7]
    cont = ~((pdf == 0) | ((bsdf[:, 0] == 0) & (bsdf[:, 1] == 0) & (bsdf[:, 2] == 0)))
    with np.errstate(all="ignore"):
        thr = np.where(cont[:, None], ((thr * bsdf) * np.abs(_dot(wi, normal))[:, None]) / pdf[:, None], thr)
        alive = cont.copy()
        if b + 1 > 3:
            q = np.fmax(F32(0.05), F32(1) - np.fmax(thr[:, 0], np.fmax(thr[:, 1], thr[:, 2])))
            rr_rng, r = np_lcg(rng)
            rng = np.where(cont, rr_rng, rng)
            alive &= ~(r < q)
            thr = np.where((cont & alive)[:, None], thr / (F32(1) - q)[:, None], thr)
    emit = alive & (b + 1 < max_depth)
    E = np.nonzero(emit)[0]
    return dict(slots=slots, nee_T=nee_T, l1=(sl[has_l1], l1[has_l1]), l2=(sl[emit_b], l2[emit_b]),
                keys=keys[order], sray_o=sray_o[order], sray_d=sray_d[order], next=np.sort(sl[E]),
                next_rows=(sl[E], np.concatenate([hit_p[E], np.full((len(E), 1), EPS)], 1),
                           np.concatenate([wi[E], np.full((len(E), 1), F32(1e20))], 1),
                           np.concatenate([thr[E], rng[E].view(F32)[:, None]], 1)),
                differs=calls.differs)


def check_shade_restatement(got, want, b, name):
    """k_shade's outputs equal the restatement's, bit for bit (NaN payloads aside)."""
    sl = want["slots"]
    assert same_bits(got["nee_T"][sl], want["nee_T"]), f"{name}: nee_T"
    for k, (s, v) in (("nee_l1", want["l1"]), ("nee_l2", want["l2"])):
        assert same_bits(got[k][s, :3], v), f"{name}: {k}"
    qo, keys, so, sd = shade_outputs(got, b)
    assert np.array_equal(keys.astype(np.int64), want["keys"]), f"{name}: shadow ray keys"
    assert same_bits(so, want["sray_o"]) and same_bits(sd[:, :3], want["sray_d"]), f"{name}: shadow rays"
    assert np.array_equal(qo.astype(np.int64), want["next"]), f"{name}: continuation queue"
    s, o, d, t = want["next_rows"]
    assert same_bits(got["ray_o"][s], o) and same_bits(got["ray_d"][s], d), f"{name}: continuation rays"
    assert same_bits(got["thr_rng"][s], t), f"{name}: continuation throughput / rng"


def compare_shade(dev, host, scene_h, scene_hh, st, b, max_depth, kats, rec, record=None, what=""):
    """k_shade on the build under test and on the host build, from the same state: each equals the restatement fed
    its own shading functions, bit for bit; where the device's functions return glibc's bits on a path's inputs, the
    device's path equals the host build's."""
    got = dev.shade(scene_h, st, b, max_depth)
    ref = host.shade(scene_hh, st, b, max_depth)
    check_shade_structure(st, ref, b, max_depth, f"host {what}", 1)
    check_shade_structure(st, got, b, max_depth, f"{dev.name} {what}", 32)
    want = np_shade(st, b, max_depth, ShadeCalls(kats[0], kats[1], rec))
    check_shade_restatement(got, want, b, f"{dev.name} {what} b{b}")
    check_shade_restatement(ref, np_shade(st, b, max_depth, ShadeCalls(kats[1], kats[1], rec)), b, f"host {what} b{b}")
    count = int(st["counters"][CNT_QUEUE + b])
    qin = st.queue(b)[:count]
    agree = np.zeros(st.cap, bool)
    agree[qin] = ~want["differs"][qin]
    for k in ("ray_o", "ray_d", "thr_rng", "nee_T"):
        assert np.all(row_same(got[k], ref[k])[agree]), f"{dev.name} {what} b{b}: {k} differs from the host build where the functions agree"
    n_fn = int(want["differs"][qin].sum())
    if record is not None:
        record(f"shade_function_results_differ_{what}_b{b}", f"{n_fn}/{count}")
    if not dev.gpu:  # the emulated twin uses glibc's functions: nothing may differ
        assert n_fn == 0
        for k in ARRAYS[:8]:
            assert np.array_equal(got[k].view(U8), ref[k].view(U8)), f"{dev.name} {what}: {k}"
    return got


def lockstep(dev, host, scene, cam, lay, max_depth, record, what, kats, far_first=False):
    """One frame with enqueue_frame's launch sequence on the build under test; every stage is run on the host from
    the device's own pre-stage state, and each stage's result is checked against it."""
    sd, sh = dev.scene(what, scene), host.scene(what, scene)
    rec = scene_records(host, sh)
    view = cam_view(cam, lay)
    st = State(lay.npaths, seed=11)
    st = dev.raygen(st, view, 0, lay)
    check_raygen(State(lay.npaths, seed=11), st, view, 0, lay)
    nxt = dev.traverse(sd, st, 0, CNT_QUEUE, -1, CNT_WORK, far_first)
    ref = host.traverse(sh, st, 0, CNT_QUEUE, -1, CNT_WORK, far_first)
    assert np.array_equal(nxt.u("hit"), ref.u("hit")), f"{what}: primary hits"
    st = nxt
    for b in range(max_depth):
        st2 = compare_shade(dev, host, sd, sh, st, b, max_depth, kats, rec, record, what)
        last = b + 1 == max_depth
        closest = -1 if last else CNT_QUEUE + b + 1
        nxt = dev.traverse(sd, st2, b + 1, closest, CNT_SHADOW + b, CNT_WORK + 1 + b, far_first)
        ref = host.traverse(sh, st2, b + 1, closest, CNT_SHADOW + b, CNT_WORK + 1 + b, far_first)
        assert np.array_equal(nxt.u("hit"), ref.u("hit")) and np.array_equal(nxt["vis"], ref["vis"]), f"{what} b{b}: hit / vis"
        count = int(nxt["counters"][CNT_QUEUE + b])
        got, _ = dev.nee_resolve(nxt, b)
        assert same_bits(got["radiance"], np_nee_resolve(nxt, nxt.queue(b), count, kats[0].miss)), f"{what} b{b}: k_nee_resolve"
        st = got
    check_resolve(dev, kats, lay, 0, seed=12, st=st)


LOCKSTEP = [
    # (scene, w, h, spp, frames, rank, world, max_depth): every scene at 1 and 4 spp, a 2-frame batch and a rank tile set
    ("cornell", 70, 45, 1, 2, 0, 1, 8),
    ("cornell", 70, 45, 4, 1, 1, 2, 8),
    ("materials", 70, 45, 1, 1, 1, 2, 5),
    ("materials", 70, 45, 4, 2, 0, 1, 5),
    ("lights", 70, 45, 1, 2, 1, 2, 5),
    ("lights", 70, 45, 4, 1, 0, 1, 5),
]
if FULL:
    LOCKSTEP += [("materials", 130, 70, 4, 1, 0, 1, 8), ("cornell", 130, 70, 4, 2, 1, 2, 8)]


@pytest.mark.parametrize("case", LOCKSTEP, ids=lambda c: f"{c[0]}_{c[1]}x{c[2]}_spp{c[3]}_f{c[4]}_r{c[5]}of{c[6]}_d{c[7]}")
def test_lockstep_frame(dev, host, kats, record_property, case):
    name, w, h, spp, frames, rank, world, depth = case
    if dev.gpu:  # full-size frames on the GPU
        w, h = w * 4, h * 4
    scene, cam = SCENES[name](spp)
    lay = Layout(w, h, scene.samples_per_pixel, frames, rank, world)
    lockstep(dev, host, scene, cam, lay, depth, record_property, f"{name}_{w}x{h}_spp{spp}", kats)


# ---- crafted k_shade states ----
def crafted_shade_state(scene, cap, count, b, seed):
    """Hits on real triangles (u + v = 1, t near 0, back faces), misses, permuted slots, edge rng states, throughputs
    0 / denormal / inf / NaN."""
    from helpers import HostCheck

    hc = HostCheck(scene)
    _, _, tris, _ = hc.export()
    rng = np.random.default_rng(seed)
    st = State(cap, seed)
    slots = rng.permutation(cap)[:count].astype(U32)
    st.queue(b)[:count] = slots
    st["counters"][CNT_QUEUE + b] = count
    ntri = len(tris)
    t = rng.integers(0, ntri, cap)
    u = rng.random(cap).astype(F32)
    v = (rng.random(cap).astype(F32) * (F32(1) - u)).astype(F32)
    v[::5] = F32(1) - u[::5]  # u + v = 1
    v0, e1, e2 = tris[t, 0:3], tris[t, 4:7], tris[t, 8:11]
    p = v0 + u[:, None] * e1 + v[:, None] * e2
    d = rng.standard_normal((cap, 3)).astype(F32)
    d /= np.linalg.norm(d, axis=1, keepdims=True).astype(F32)
    dist = rng.uniform(0.05, 2.0, cap).astype(F32)
    dist[1::7] = F32(2e-4)  # t near 0
    st["ray_o"][:, :3] = p - dist[:, None] * d
    st["ray_o"][:, 3] = EPS
    st["ray_d"][:, :3] = d  # random sides: front and back faces
    st["ray_d"][:, 3] = F32(1e20)
    st["hit"][:, 0], st["hit"][:, 1], st["hit"][:, 2] = dist, u, v
    st["hit"][:, 3] = t.astype(U32).view(F32)
    st["hit"][::6, 3] = np.uint32(MISS).view(F32)
    thr = rng.uniform(0.01, 1.0, (cap, 3)).astype(F32)
    thr[2::11] = 0
    thr[3::11] = F32(1e-41)
    thr[4::13, 1] = np.inf
    thr[5::17, 2] = np.nan
    st["thr_rng"][:, :3] = thr
    states = rng.integers(0, 2**32, cap, dtype=np.uint64)
    states[::4] = EDGE_DRAWS[np.arange(len(states[::4])) % len(EDGE_DRAWS)]  # first draw at the light-id clamp
    st.u("thr_rng")[:, 3] = states_before(states)
    return st


SHADE_COUNTS = [0, 1, 31, 32, 33, 127, 128, 129]


@pytest.mark.parametrize("scene_key", ["cornell", "lights", "materials"])
def test_crafted_shade_states(dev, host, kats, record_property, scene_key):
    scene, _ = SCENES[scene_key](1)  # one light, three (lights) or one (materials)
    sd, sh = dev.scene(scene_key, scene), host.scene(scene_key, scene)
    rec = scene_records(host, sh)
    counts = SHADE_COUNTS + ([2**17 + 1] if (dev.gpu or FULL) else [257])
    for i, count in enumerate(counts):
        for b, depth in ((3, 8), (4, 8), (0, 1), (15, 16), (2, 3)):
            cap = count + 64
            st = crafted_shade_state(scene, cap, count, b, seed=100 * i + b)
            compare_shade(dev, host, sd, sh, st, b, depth, kats, rec, record_property, f"{scene_key}_n{count}")
            if not dev.gpu and count > 200:
                break


def test_light_choice_clamp_with_seven_lights(dev, host, kats, record_property):
    """Draws that round to 1.0f pick light n - 1, not n: the restatement clamps on its own, so the light (and with
    it the shadow ray, the NEE terms) the kernel chose is checked path by path."""
    scene, _ = lights_scene(1)
    scene.lights = (scene.lights * 3)[:7]
    sd, sh = dev.scene("lights7", scene), host.scene("lights7", scene)
    st = crafted_shade_state(scene, 200, 160, 0, seed=77)
    st.u("thr_rng")[:, 3] = states_before(EDGE_DRAWS[np.arange(200) % 5])
    compare_shade(dev, host, sd, sh, st, 0, 5, kats, scene_records(host, sh), record_property, "lights7")


# ---- the launch geometry of wave_devcheck.cu is enqueue_frame's ----
def _geometry(path, names):
    src = open(path).read()
    for a, b in names:
        src = re.sub(a, b, src)
    grids = {}  # every assignment of a grid variable, in source order ("tiles": scan_u32's declaration only)
    for m in re.finditer(r"\b(g256|g128|g_nee|gpx|trav_grid|num_tiles|unsigned tiles|scratch_items|left)\s*=\s*([^;{]+);", src):
        if m.group(2).strip() != "0":  # (the renderer's member initialisers)
            grids.setdefault(m.group(1), []).append(re.sub(r"\s+", "", m.group(2)))
    launches = {}
    for m in re.finditer(r"crt::(k_\w+)(?:<(?:true|false|256|uint32_t)>)?<<<([^,]+),\s*([^,]+),", src):
        launches.setdefault(m.group(1), set()).add((m.group(2).strip(), m.group(3).strip()))
    return grids, launches


def test_launch_geometry_follows_enqueue_frame():
    """wave_devcheck.cu restates the product's grids (enqueue_frame, launch_traverse, sort_shade_queue, scan_u32);
    if one of them changes in crt_cuda_core.cu, this fails until the check library follows."""
    prod = _geometry(os.path.join(CSRC, "crt_cuda_core.cu"), [(r"\bnpx_local\b", "NPX"), (r"\bnpaths\b", "NPATHS"), (r"\bsms\b", "SMS"),
                                                               (r"\bnum_sms\b", "SMS")])
    wave = _geometry(os.path.join(CSRC, "wave_devcheck.cu"), [(r"\bnpx\b", "NPX"), (r"\bcap\b", "NPATHS"), (r"\bnpaths\b", "NPATHS"),
                                                               (r"\bnum_sms\(\)", "SMS")])
    assert set(wave[0]) == {"g256", "g128", "g_nee", "gpx", "trav_grid", "num_tiles", "unsigned tiles", "scratch_items", "left"}
    for k, expr in wave[0].items():
        assert prod[0].get(k) == expr, f"{k}: {expr} here, {prod[0].get(k)} in enqueue_frame"
    for k, shapes in wave[1].items():
        assert shapes <= prod[1].get(k, set()), f"{k}: launched as {shapes} here, {prod[1].get(k)} by the renderer"
