"""The production traversal kernel (k_traverse through crtc_trace_closest / crtc_trace_any) against brute force on the
rays where a traversal goes wrong: from and towards vertices, axis-parallel with exact zeros (and -0.0) along grid lines
and box planes, direction components below the 1e-20 clamp of trav_init, negative tnear (hits behind the origin),
intervals that end or start exactly on a hit, an origin on coincident triangles (hits at t = +-0), Inf and NaN
components. Scenes are the adversarial generators of scripts/fuzz_bvh8_vs_bruteforce.py at three scene scales plus a
stack of parallel sheets with exact hit distances; every tree builder and every k_traverse instantiation runs.

The reference is OracleBackend(brute_force=True): it states the kernel's float32 triangle formula independently, so
closest hits (t, u, v, primitive id) must match bit for bit and occlusion answers must be equal.

Each test runs twice: on the emulated renderer (tests/simt_emu: the same crt_cuda_core.cu and kernels.cuh under the
SIMT emulation; one traversal variant per scene and builder, rotating) and on the GPU (every variant, larger batches).
The host check builds with a skewed box-test reciprocal run the same cases on the CPU."""
import os
import sys

import numpy as np
import pytest

from helpers import ROOT, HostCheck

sys.path.insert(0, os.path.join(ROOT, "scripts"))
import fuzz_bvh8_vs_bruteforce as fuzz  # noqa: E402
from oracle import OracleBackend  # noqa: E402

MISS = 0xFFFFFFFF
BUILDERS = ("host", "device", "device_lbvh")
# (tri_pass_defer, count_traversal, bvh_top_smem): between them every k_traverse instantiation launch_traverse picks
VARIANTS = ((16, 0, 0), (0, 0, 0), (24, 0, 0), (0, 1, 0), (16, 1, 0), (24, 1, 0), (16, 0, 1))
# fuzz.random_geometry draws its kind of scene second; these seeds give each kind
KIND_SEEDS = {"soup": 2, "slivers": 8, "sheets": 0, "huge_tiny": 1, "grid": 4}
SCALES = (1e-3, 1.0, 1e3)
SCENES = [(k, s) for k in KIND_SEEDS for s in SCALES]
BATCHES = (1, 31, 33, 4097)
TNEAR_ANY = (-1.0, 0.0, 1e-5, 1e-4, 1e-3)
INF = np.float32(np.inf)


@pytest.fixture(scope="module", params=[pytest.param("emulated"), pytest.param("gpu", marks=pytest.mark.gpu)])
def where(request, built):
    import chameleonrt_b200.backend as backend

    saved = (backend._LIB_PATH, backend._lib)
    if request.param == "emulated":
        sys.path.insert(0, os.path.join(ROOT, "tests", "simt_emu"))
        import build as simt_build

        backend._LIB_PATH, backend._lib = simt_build.build(), None
    yield request.param
    backend._LIB_PATH, backend._lib = saved


def _variants(where, i):
    """Traversal variants for the i-th (scene, builder) pair: all on the GPU, one in turn on the emulation."""
    return VARIANTS if where == "gpu" else (VARIANTS[i % len(VARIANTS)],)


def _renderer(scene, builder="host", variant=VARIANTS[0], far_first=False):
    import chameleonrt_b200.backend as backend

    defer, count, top = variant
    r = backend.RenderCUDA(0, bvh_builder=builder, tri_pass_defer=defer, count_traversal=bool(count),
                           any_far_first=1 if far_first else None)
    if top:
        r.set_option("bvh_top_smem", 1)
    r.initialize(8, 8)
    r.set_scene(scene)
    assert r.get_option("bvh_builder_fallbacks") == 0, builder
    if far_first:
        # a kernel-level trace_any visits children in the order the last frame used
        r.render((0.0, 0.0, 1.0), (0.0, 0.0, -1.0), (0.0, 1.0, 0.0), 45.0, True, True)
        assert r.get_option("any_far_first_decision") == 1
    return r


def _brute(scene):
    o = OracleBackend(brute_force=True)
    o.initialize(8, 8)
    o.set_scene(scene)
    return o


def _batched(fn, rays):
    """fn over consecutive batches of BATCHES' sizes in turn, concatenated; an empty batch first."""
    out, i, k = [fn(rays[:0])], 0, 0
    assert len(out[0]) == 0
    while i < len(rays):
        n = BATCHES[k % len(BATCHES)]
        out.append(fn(rays[i:i + n]))
        i, k = i + n, k + 1
    return np.concatenate(out)


def _assert_same(got, want, rays, what):
    """Bit for bit, except u and v of rays with a -0.0 direction component, which are compared as values: the reference
    takes every ray through its (identity) instance transform, which turns -0.0 into +0.0, while the product uses the
    direction as given, so a hit on an edge can have u or v = -0.0 on one side and +0.0 on the other."""
    g = np.asarray(got).reshape(len(want), -1)
    w = np.asarray(want).reshape(len(want), -1)
    if g.dtype == np.float32:
        differ = g.view(np.uint32) != w.view(np.uint32)
        neg0 = (rays[:, 4:7].view(np.uint32) == 0x80000000).any(1)
        differ[neg0, 1:3] = g[neg0, 1:3] != w[neg0, 1:3]
        differ = differ.any(1)
    else:
        differ = (g != w).any(1)
    bad = np.nonzero(differ)[0]
    assert len(bad) == 0, (f"{what}: {len(bad)} of {len(want)} rays differ; first rays {rays[bad[:3]].tolist()}: "
                           f"got {g[bad[:3]].tolist()}, want {w[bad[:3]].tolist()}")


def _fuzz_scene(kind, scale):
    rng = np.random.default_rng(KIND_SEEDS[kind])
    scene = fuzz.without_needles(fuzz.scene_of([fuzz.random_geometry(rng, scale)]))
    assert scene.total_tris() > 0
    return scene, rng


def _set(rays, col, values):
    out = rays.copy()
    out[:, col] = values
    return out


def _edge_rays(scene, rng, brute, n=600):
    """Closest-hit rays of every edge kind above for one scene, built from n fuzz rays (float32, about 5 n x 8)."""
    base = fuzz.random_rays(rng, scene, n)  # from / towards vertices, axis-parallel along grid lines, short segments
    axis = base[-(n // 6):]
    d = axis[:, 4:7]
    parts = [base, _set(axis, slice(4, 7), np.where(d == 0, np.float32(-0.0), d))]
    for tiny in (1e-25, -1e-25, 1e-40):  # below the 1e-20 clamp; 1e-40 is subnormal
        parts.append(_set(axis, slice(4, 7), np.where(d == 0, np.float32(tiny), d)))
    # negative tnear: the origin moved forward along the ray, tnear reaching back past part of the scene and beyond the
    # old origin (test_slab_tnear_host.py's construction)
    verts = np.concatenate([np.asarray(g.vertices, np.float32) for g in scene.meshes[0].geometries])
    ext = float((verts.max(0) - verts.min(0)).max())
    shift = (rng.uniform(0.0, 1.0, len(base)) * ext).astype(np.float32)
    moved = base.copy()
    moved[:, 0:3] += shift[:, None] * base[:, 4:7]
    moved[:, 3] = -shift * rng.uniform(0.0, 1.5, len(base)).astype(np.float32)
    parts.append(moved)
    # intervals that end or start exactly on each brute-force hit
    probe = np.concatenate([base, moved])
    h = brute.trace_closest(probe)
    hit = h[:, 3].view(np.uint32) != MISS
    r, t = probe[hit], h[hit, 0]
    parts += [_set(r, 7, t), _set(r, 7, np.nextafter(t, INF)), _set(r, 3, t), _set(r, 3, np.nextafter(t, -INF))]
    # Inf and NaN components: these hit nothing
    bad = np.repeat(base[:1], 8, 0)
    for i, (col, v) in enumerate(((0, np.inf), (1, -np.inf), (2, np.nan), (4, np.nan), (5, np.inf), (6, -np.inf),
                                  (3, np.nan), (7, np.nan))):
        bad[i, col] = v
    parts.append(bad)
    return np.ascontiguousarray(np.concatenate(parts), np.float32)


def _any_rays(closest_rays):
    """Occlusion rays: the closest-hit rays at each tnear of TNEAR_ANY, plus the originals (their own tnear)."""
    return np.ascontiguousarray(np.concatenate([closest_rays] + [_set(closest_rays, 3, tn) for tn in TNEAR_ANY]), np.float32)


# ---- a stack of parallel sheets with exact hit distances ------------------------------------------------------------
SHEETS = (-8.0, -4.0, -2.0, -1.0, -0.5, 0.0, 0.0, 0.0, 0.5, 1.0, 2.0, 4.0, 4.0)  # coincident: three at 0, two at 4


def _sheet_scene():
    """Right triangles covering x, y in [-4, 12] with x + y <= 8 in the planes z = SHEETS, in that flat-id order. The
    coincident ones list their corners in different orders (a rotation, the reverse winding), so their hit t can
    differ in the sign of zero."""
    from chameleonrt_b200.scenes import MeshBuilder

    corners = np.array([[-4.0, -4.0], [12.0, -4.0], [-4.0, 12.0]])
    orders = ([0, 1, 2], [1, 2, 0], [0, 2, 1])
    tris, seen = [], {}
    for z in SHEETS:
        k = seen[z] = seen.get(z, -1) + 1
        tris.append([[*corners[j], z] for j in orders[k]])
    v = np.array(tris, np.float32).reshape(-1, 3)
    b = MeshBuilder()
    b.add(v, np.zeros((len(v), 2), np.float32), np.arange(len(v), dtype=np.uint32).reshape(-1, 3))
    return fuzz.scene_of([b.geometry()])


def _sheet_rays():
    rays = []
    for ox, oy in ((0.25, 0.25), (-1.5, 1.0), (0.0, 0.0), (1.125, -2.0)):
        for oz in (0.0, 0.25, -3.0):
            for d in ((0.0, 0.0, 1.0), (-0.0, 0.0, -1.0), (0.0625, -0.0, 2.0), (-0.0625, 0.125, -0.5)):
                for tnear in (-16.0, -5.0, -1.0, -0.25, -0.0, 0.0, 1e-4):
                    for tfar in (1e20, 3.0, 0.5):
                        rays.append([ox, oy, oz, tnear, *d, tfar])
    return np.array(rays, np.float32)


def _sheet_expected(rays):
    """Closest hit (t, sheet id) of each ray in float64: every sheet is hit at (z - oz) / dz."""
    t = (np.array(SHEETS)[None, :] - rays[:, 2:3].astype(np.float64)) / rays[:, 6:7].astype(np.float64)
    ok = (t > rays[:, 3:4]) & (t < rays[:, 7:8])
    tm = np.where(ok, t, np.inf)
    best = tm.min(1)
    prim = np.where(ok.any(1), np.argmax(ok & (tm == best[:, None]), 1), MISS)  # first = lowest id among the ties
    return best, prim.astype(np.uint64)


def test_sheets_reference_is_exact(built):
    """The brute-force reference on the sheets gives the float64 hit distances and the lowest coincident id, including
    hits behind the origin and the +-0 hits of an origin on the three coincident sheets."""
    rays = _sheet_rays()
    h = _brute(_sheet_scene()).trace_closest(rays)
    best, prim = _sheet_expected(rays)
    got_prim = h[:, 3].view(np.uint32).astype(np.uint64)
    assert (got_prim == prim).all()
    hit = prim != MISS
    assert (h[hit, 0].astype(np.float64) == best[hit]).all()
    assert (h[~hit, 0] == rays[~hit, 7]).all()
    assert (hit & (best < 0)).sum() > 100 and (hit & (best == 0)).sum() > 50
    zero = hit & (best == 0)
    assert set(got_prim[zero].tolist()) == {SHEETS.index(0.0)}
    assert np.signbit(h[zero, 0]).any() and (~np.signbit(h[zero, 0])).any()


def test_sheets(where):
    scene, rays = _sheet_scene(), _sheet_rays()
    brute = _brute(scene)
    want, occ = brute.trace_closest(rays), brute.trace_any(_any_rays(rays))
    for builder in BUILDERS:
        for variant in VARIANTS:  # a 13-triangle scene: every variant, on the emulation too
            r = _renderer(scene, builder, variant)
            _assert_same(_batched(r.trace_closest, rays), want, rays, f"closest, {builder} {variant}")
            _assert_same(_batched(r.trace_any, _any_rays(rays)), occ, _any_rays(rays), f"any, {builder} {variant}")
    r = _renderer(scene, "host", VARIANTS[0], far_first=True)
    _assert_same(r.trace_any(_any_rays(rays)), occ, _any_rays(rays), "any, far-first")


@pytest.mark.parametrize("kind", list(KIND_SEEDS))
def test_fuzz_scenes(where, kind):
    """Each kind of fuzz scene at scales 1e-3, 1 and 1e3, over every builder: closest hits and occlusion."""
    for s, scale in enumerate(SCALES):
        scene, rng = _fuzz_scene(kind, scale)
        brute = _brute(scene)
        rays = _edge_rays(scene, rng, brute, 600 if where == "gpu" else 300)
        any_rays = _any_rays(rays)
        want, occ = brute.trace_closest(rays), brute.trace_any(any_rays)
        assert (want[-8:, 3].view(np.uint32) == MISS).all() and not occ[len(rays) - 8:len(rays)].any()
        for b, builder in enumerate(BUILDERS):
            for variant in _variants(where, 3 * (list(KIND_SEEDS).index(kind) + s) + b):
                r = _renderer(scene, builder, variant)
                what = f"{kind} at scale {scale}, {builder} {variant}"
                _assert_same(_batched(r.trace_closest, rays), want, rays, "closest, " + what)
                _assert_same(_batched(r.trace_any, any_rays), occ, any_rays, "any, " + what)
        # shadow rays (tnear = 1e-4: the any-hit kernel) visiting children far-first
        r = _renderer(scene, BUILDERS[s], VARIANTS[s], far_first=True)
        _assert_same(_batched(r.trace_any, any_rays), occ, any_rays, f"any far-first, {kind} at scale {scale}")


@pytest.mark.gpu
def test_batch_larger_than_the_persistent_grid(where):
    """2^20 + 7 rays, more than the persistent grid's warps hold at once (trav_grid x 128 threads on an H100), so warps
    refill many times; against brute force (the oracle's BVH misses some vertex hits of axis-parallel rays)."""
    if where != "gpu":
        pytest.skip("a million rays are beyond the emulation")
    scene, rng = _fuzz_scene("soup", 1.0)
    rays = fuzz.random_rays(rng, scene, (1 << 20) + 7)
    rays[::3, 3] = -rng.uniform(0.0, 4.0, len(rays[::3])).astype(np.float32)  # and a third with tnear < 0
    brute = _brute(scene)
    want, occ = brute.trace_closest(rays), brute.trace_any(rays)
    assert (want[:, 3].view(np.uint32) != MISS).mean() > 0.2
    for variant in VARIANTS:
        r = _renderer(scene, "host", variant)
        _assert_same(r.trace_closest(rays), want, rays, f"closest {variant}")
        _assert_same(r.trace_any(rays), occ, rays, f"any {variant}")


@pytest.mark.parametrize("variant", ["rcp_lo", "rcp_hi"])
def test_skewed_box_reciprocal_host_checks(built, variant):
    """The host traversal with its box-test reciprocal one ulp towards or away from zero (the device's approximate
    reciprocal may round either way; the slack in node_intersect_loaded has to cover it): the fixed fuzz seeds of
    test_bvh8_host.py and the edge cases here still agree with brute force."""
    for seed in (0, 7, 22, 53, 98, 106, 1234, 2222):
        ok, info = fuzz.one(seed, hostcheck=lambda scene, threads: HostCheck(scene, threads, variant))
        assert ok, (seed, info)
    cases = [(_sheet_scene(), None)] + [_fuzz_scene(k, s) for k, s in SCENES]
    for scene, rng in cases:
        brute = _brute(scene)
        rays = _sheet_rays() if rng is None else _edge_rays(scene, rng, brute)
        any_rays = _any_rays(rays)
        hc = HostCheck(scene, 0, variant)
        _assert_same(hc.trace(rays)[0], brute.trace_closest(rays), rays, "closest")
        occ = brute.trace_any(any_rays)
        for far_first in (False, True):
            got = (hc.trace(any_rays, any_hit=True, far_first=far_first)[0][:, 3].view(np.uint32) != MISS).astype(np.uint8)
            _assert_same(got, occ, any_rays, f"any, far_first={far_first}")
