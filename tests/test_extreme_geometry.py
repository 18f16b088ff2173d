"""Geometry at the edges of float32 through the BVH builders, the refit and the traversal: vertices at +-inf and NaN,
coordinates from 1e16 to +-FLT_MAX, a triangle of denormal extent, one spanning -3e38..3e38, and instance matrices
that are all zeros, flatten one axis, hold a NaN, translate by inf or scale by 1e38. set_scene and commits accept all
of it (include/crt_cuda.h, DESIGN.md §2).

The reference is OracleBackend(brute_force=True), as in test_traversal_edges.py; the contract is the one stated at
crtc_set_scene in include/crt_cuda.h, checked ray by ray (ray_classes):
  * every ray: brute force's answer, a miss, or a hit later in (t, primitive id) order; never a closer or false hit;
  * bit for bit equal to brute force (closest hits) and equal occlusion answers: every ray brute force misses, and every
    ray whose brute-force hit is well conditioned (the triangle within 2^16 of its longest edges of the origin), when all
    vertices and origins lie in a box of extent kExactExtent = 255 * 2^46 per axis (NaN coordinates count as absent);
  * past that extent, the same when every coordinate is above -kExactExtent, every direction component has
    magnitude at least 2^-12 and the hit triangle lies within 2^107;
  * the extent is the exact one: at it every ray above matches, one float past it rays straight down miss, for every
    builder and traversal variant.

Every check runs on the emulated build (tests/simt_emu) without a GPU and on the sm_90a build with ``-m gpu``:
  * hits of every builder (host, PLOC, LBVH) and, on the GPU, every k_traverse variant, on the grid scenes and on the
    courtyard with one instance given each extreme matrix; the host checks too;
  * the device builders' BVH8 nodes: structure, check_bvh8 inside kExactExtent, and on the GPU equal byte for
    byte to the emulated build's (the conversions to int of infinite boxes are where a GPU and a CPU differ);
  * commits of extreme transforms and vertices: the refit nodes equal a float32 restatement of k_bvh8_refit, the
    records a fresh host build's, trace_closest / trace_any / frames a fresh set_scene's, and a commit back to the
    original transforms renders the original scene again;
  * on the GPU, a refit of the C4 workload (more nodes than the refit grid's threads) node for node.
"""
import gc
import os
import sys

import numpy as np
import pytest

from helpers import ROOT, HostCheck
from test_bvh_build_exact import NODE, DevCheck, check_bvh8, quantise
from test_dynamic_scene import (UpdateCheck, _stale, frames_equal, replaced, small_courtyard, world_tris)
from test_traversal_edges import MISS, VARIANTS, _any_rays, _assert_same, _edge_rays

sys.path.insert(0, os.path.join(ROOT, "scripts"))
import fuzz_bvh8_vs_bruteforce as fuzz  # noqa: E402
from oracle import OracleBackend  # noqa: E402

CSRC = os.path.join(ROOT, "chameleonrt_b200", "csrc")
F32, F64, U8, U32 = np.float32, np.float64, np.uint8, np.uint32
BUILDERS = ("host", "device", "device_lbvh")
INF, NAN = float("inf"), float("nan")
FLT_MAX = float(np.finfo(F32).max)
EXACT_EXTENT = 255.0 * 2.0**46  # kExactExtent of include/crt_cuda.h

# ---- scenes --------------------------------------------------------------------------------------------------------
GRID = 12  # GRID x GRID squares in [-1, 1]^2 at z = 0


def _grid_tris():
    xs = np.linspace(-1.0, 1.0, GRID + 1)
    tris = []
    for i in range(GRID):
        for j in range(GRID):
            a, b, c, d = (xs[i], xs[j], 0), (xs[i + 1], xs[j], 0), (xs[i], xs[j + 1], 0), (xs[i + 1], xs[j + 1], 0)
            tris += [[a, b, c], [b, d, c]]
    return np.array(tris, F32)


def _scene(tris):
    from chameleonrt_b200.scenes import MeshBuilder

    v = np.asarray(tris, F32).reshape(-1, 3)
    b = MeshBuilder()
    b.add(v, np.zeros((len(v), 2), F32), np.arange(len(v), dtype=U32).reshape(-1, 3))
    return fuzz.scene_of([b.geometry()])


# the extra triangle sits over the grid's middle (x, y in [0.1, 0.3], z = 0.25), so it shares inner nodes with the grid
_NEAR = np.array([[0.1, 0.1, 0.25], [0.3, 0.1, 0.25], [0.1, 0.3, 0.25]], F64)


def _moved(axis, value, which):
    t = _NEAR.copy()
    t[which, axis] = value
    return t


def extreme_triangles():
    """(name, triangle (3, 3), inside kExactExtent?)."""
    out = []
    for v, tag in ((INF, "+inf"), (-INF, "-inf"), (NAN, "nan")):
        for axis in range(3):
            for which, wtag in (([0], "one"), ([0, 1, 2], "all")):
                out.append((f"{tag}_{'xyz'[axis]}_{wtag}", _moved(axis, v, which), v != v))  # NaN: a vertex that is absent
    for v in (1e16, 1e20, 1e30, 3e38, FLT_MAX, -FLT_MAX):
        # all three vertices out there on x (a triangle that keeps its shape in y and z), and one of them on z
        out.append((f"{v:g}_x_all", _NEAR + [[v, 0, 0]] * 3, abs(v) + 1 <= EXACT_EXTENT))
        out.append((f"{v:g}_z_one", _moved(2, v, [0]), abs(v) + 1 <= EXACT_EXTENT))
    out.append(("denormal_extent", np.array([[0.2, 0.2, 0.5], [0.2 + 1e-40, 0.2, 0.5], [0.2, 0.2 + 1e-40, 0.5]], F64), True))
    out.append(("span_3e38", np.array([[-3e38, 0.2, 0.5], [3e38, 0.2, 0.5], [0.0, 0.3, -3e38]], F64), False))
    # the bound itself: the grid's low corner -1 plus 255 * 2^46 (exactly representable), and the next float above it
    edge = float(F32(-1.0 + EXACT_EXTENT))
    assert edge + 1.0 == EXACT_EXTENT
    out.append(("at_the_bound", _NEAR + [[edge, 0, 0]] * 3, True))
    out.append(("past_the_bound", _NEAR + [[float(np.nextafter(F32(edge), F32(INF))), 0, 0]] * 3, False))
    return out


EXTREMES = extreme_triangles()
EXTREME_IDS = [name for name, _, _ in EXTREMES]


def extreme_scene(tri):
    return _scene(np.concatenate([_grid_tris(), np.asarray(tri, F32)[None]]))


def _brute(scene):
    o = OracleBackend(brute_force=True)
    o.initialize(8, 8)
    o.set_scene(scene)
    return o


def extreme_rays(tri, n, seed):
    """test_traversal_edges' ray families over the finite grid (from and towards vertices, axis-parallel with 0 and -0,
    below the 1e-20 clamp, negative tnear, intervals ending on hits, Inf / NaN components), rays straight down and tilted
    by 1e-3 and 0.1, rays onto the grid from 1.2e4 away, and rays from and towards the extra triangle's vertices."""
    base = _scene(_grid_tris())
    rng = np.random.default_rng(seed)
    parts = [_edge_rays(base, rng, _brute(base), n)]
    o = np.concatenate([rng.uniform(-1.1, 1.1, (n, 2)), np.full((n, 1), 1.0)], 1)
    for tilt in (0.0, 1e-3, 0.1):
        d = np.array([tilt, 0.5 * tilt, -1.0])
        parts.append(np.concatenate([o, np.zeros((n, 1)), np.tile(d / np.linalg.norm(d), (n, 1)), np.full((n, 1), 1e30)], 1))
    v = np.asarray(tri, F64)
    grid_v = _grid_tris().reshape(-1, 3).astype(F64)
    # from 1.2e4 away (COND longest grid edges are 1.54e4) onto grid vertices and points: the least conditioned rays
    # that must still be exact
    far = np.concatenate([rng.uniform(-1.0, 1.0, (n, 2)), np.full((n, 1), 1.2e4)], 1) * rng.choice([1.0, -1.0], (n, 1))
    aim = np.where(rng.random((n, 1)) < 0.5, grid_v[rng.integers(0, len(grid_v), n)],
                   np.concatenate([rng.uniform(-1.0, 1.0, (n, 2)), np.zeros((n, 1))], 1))
    parts.append(np.concatenate([far, np.zeros((n, 1)), aim - far, np.full((n, 1), 1e30)], 1))
    for k in range(3):
        g = grid_v[rng.integers(0, len(grid_v), 8)]
        with np.errstate(invalid="ignore"):
            towards = v[k] - g
        parts.append(np.concatenate([g, np.zeros((8, 1)), towards, np.full((8, 1), 1e30)], 1))
        parts.append(np.concatenate([np.repeat(v[k:k + 1], 8, 0), np.zeros((8, 1)), -towards, np.full((8, 1), 1e30)], 1))
    return np.ascontiguousarray(np.concatenate(parts), F32)


COND = 2.0**16  # a brute-force hit is well conditioned when the triangle lies within COND longest edges of the origin
MIN_DIR = 2.0**-12  # past kExactExtent: the least direction component magnitude that keeps hits
FAR = 2.0**107  # past kExactExtent: a triangle beyond it may lie outside its node's grid (exponent capped at 100)


def scene_class(tris):
    """(inside kExactExtent, every coordinate above -kExactExtent) of the world triangles (n, 3, 3); NaN is absent."""
    v = np.asarray(tris, F64).reshape(-1, 3)
    with np.errstate(invalid="ignore"):
        lo = np.array([np.nanmin(v[:, a]) if (~np.isnan(v[:, a])).any() else 0.0 for a in range(3)])
        hi = np.array([np.nanmax(v[:, a]) if (~np.isnan(v[:, a])).any() else 0.0 for a in range(3)])
        inside = bool(np.isfinite(lo).all() and np.isfinite(hi).all() and (hi - lo <= EXACT_EXTENT).all())
    return inside, bool((lo >= -EXACT_EXTENT).all())


def ray_classes(rays, want, tris):
    """Per ray: (brute force missed, brute force's hit is well conditioned, every |d_a| >= MIN_DIR and the hit
    triangle within FAR)."""
    prim = want[:, 3].view(U32)
    miss = prim == MISS
    t = np.asarray(tris, F64)[np.where(miss, 0, prim)]
    o = rays[:, :3].astype(F64)
    with np.errstate(invalid="ignore", over="ignore"):
        edge = np.sqrt(np.nanmax(((t - np.roll(t, 1, 1)) ** 2).sum(2), 1))
        dist = np.sqrt(((t.mean(1) - o) ** 2).sum(1))
        cond = ~miss & (dist <= COND * edge)
        steep = (np.abs(rays[:, 4:7]) >= MIN_DIR).all(1) & (np.abs(t) <= FAR).all((1, 2))
    return miss, cond, steep


def exact_rows(rays, want, tris):
    """The rays the contract makes bit-exact in a scene of these triangles."""
    inside, low_ok = scene_class(tris)
    miss, cond, steep = ray_classes(rays, want, tris)
    return miss | (cond & (inside | (low_ok & steep)))


def assert_hits(got, want, rays, exact, what):
    """Rays where `exact` (a bool or a mask): _assert_same. The others: each ray's answer is brute force's, a miss, or a
    hit that comes after brute force's in (t, primitive id) order, as when a culled subtree held the closest hit."""
    exact = np.broadcast_to(exact, len(want))
    g, w = np.asarray(got).reshape(len(want), -1), np.asarray(want).reshape(len(want), -1)
    if exact.any():
        _assert_same(g[exact], w[exact], rays[exact], what)
    g, w, r = g[~exact], w[~exact], rays[~exact]
    if g.dtype != np.float32:  # occlusion: never occluded where brute force is not
        bad = np.nonzero((g != 0) & (w == 0))[0]
    else:
        same = (g.view(U32) == w.view(U32)).all(1)
        gid, wid = g[:, 3].view(U32), w[:, 3].view(U32)
        later = (wid != MISS) & ((g[:, 0] > w[:, 0]) | ((g[:, 0] == w[:, 0]) & (gid > wid)))
        bad = np.nonzero(~(same | (gid == MISS) | later))[0]
    assert len(bad) == 0, (f"{what}: {len(bad)} of {len(g)} rays have a hit brute force does not; first rays "
                           f"{r[bad[:3]].tolist()}: got {g[bad[:3]].tolist()}, want {w[bad[:3]].tolist()}")


# ---- the libraries under test ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=[pytest.param("emulated"), pytest.param("gpu", marks=pytest.mark.gpu)])
def where(request, built):
    import chameleonrt_b200.backend as backend

    saved = (backend._LIB_PATH, backend._lib)
    if request.param == "emulated":
        sys.path.insert(0, os.path.join(ROOT, "tests", "simt_emu"))
        import build as simt_build

        backend._LIB_PATH, backend._lib = simt_build.build(force=_stale(simt_build.LIB)), None
    else:
        backend._LIB_PATH, backend._lib = os.path.join(CSRC, "libcrt_cuda_core.so"), None
    yield request.param
    backend._LIB_PATH, backend._lib = saved


def _emulated_devcheck_path():
    sys.path.insert(0, os.path.join(ROOT, "tests", "simt_emu"))
    import build as simt_build

    return simt_build.build_bvh_devcheck(force=_stale(simt_build.DEVCHECK_LIB))


@pytest.fixture(scope="module")
def emulated_dev(built):
    return DevCheck(_emulated_devcheck_path(), "emulated", False)


@pytest.fixture(scope="module")
def device_dev(built):
    return DevCheck(os.path.join(CSRC, "libcrt_bvh_devcheck.so"), "device", True)


@pytest.fixture(scope="module")
def emulated_upd(built):
    return UpdateCheck(_emulated_devcheck_path(), False)


@pytest.fixture(scope="module")
def device_upd(built):
    return UpdateCheck(os.path.join(CSRC, "libcrt_bvh_devcheck.so"), True)


@pytest.fixture(params=[pytest.param("emulated_upd"), pytest.param("device_upd", marks=pytest.mark.gpu)], scope="module")
def upd(request):
    return request.getfixturevalue(request.param)


def _renderer(scene, builder, variant=VARIANTS[0], **kw):
    import chameleonrt_b200.backend as backend

    defer, count, top = variant
    r = backend.RenderCUDA(0, max_depth=3, bvh_builder=builder, tri_pass_defer=defer, count_traversal=bool(count),
                           any_far_first=0, **kw)
    if top:
        r.set_option("bvh_top_smem", 1)
    r.initialize(8, 8)
    r.set_scene(scene)
    # (PLOC gives up on a round that merges nothing, which non-finite boxes can cause, and the host builder builds instead)
    assert r.get_option("bvh_builder_fallbacks") == 0 or (builder == "device" and not np.isfinite(world_tris(scene)).all()), builder
    return r


# ---- (1) hits against brute force ------------------------------------------------------------------------------------
# a ray straight down onto the grid: it hits at kExactExtent and misses one float past it, whatever the tree
SHARP_RAY = np.array([[0.05, -0.35, 1.0, 0.0, 0.0, 0.0, -1.0, 1e30]], F32)


def check_sharp(name, trace_closest, what):
    if name in ("at_the_bound", "past_the_bound"):
        hit = trace_closest(SHARP_RAY)[0, 3].view(U32) != MISS
        assert hit == (name == "at_the_bound"), f"{what}: the ray straight down {'misses' if not hit else 'hits'}"


def _expected(scene, rays):
    """Brute force's closest hits of rays, its occlusion answers of _any_rays(rays), and which rows must be exact. Brute
    force runs over the world-space triangles in flattened order, as one identity instance: the reference traces
    instanced scenes in object space, which rounds differently and cannot invert a singular matrix."""
    tris = world_tris(scene)
    brute = _brute(_scene(tris))
    any_rays = _any_rays(rays)
    want, occ = brute.trace_closest(rays), brute.trace_any(any_rays)
    ex, ex_any = exact_rows(rays, want, tris), exact_rows(any_rays, brute.trace_closest(any_rays), tris)
    return any_rays, want, occ, ex, ex_any


@pytest.mark.parametrize("case", range(len(EXTREMES)), ids=EXTREME_IDS)
def test_hits_match_brute_force(where, case):
    name, tri, _ = EXTREMES[case]
    scene = extreme_scene(tri)
    rays = extreme_rays(tri, 300 if where == "gpu" else 90, case)
    any_rays, want, occ, ex, ex_any = _expected(scene, rays)
    assert _brute(scene).trace_closest(SHARP_RAY)[0, 3].view(U32) != MISS
    for b, builder in enumerate(BUILDERS):
        variants = VARIANTS if where == "gpu" else (VARIANTS[(case + b) % len(VARIANTS)],)
        for variant in variants:
            r = _renderer(scene, builder, variant)
            what = f"{name}, {builder} {variant}"
            assert_hits(r.trace_closest(rays), want, rays, ex, "closest, " + what)
            assert_hits(r.trace_any(any_rays), occ, any_rays, ex_any, "any, " + what)
            check_sharp(name, r.trace_closest, what)


@pytest.mark.parametrize("variant", [None, "rcp_lo", "rcp_hi"])
def test_host_checks_match_brute_force(built, variant):
    """The host builder and traversal (libcrt_bvh8_hostcheck.so, the code bvh_builder = "host" runs in set_scene) and its
    builds with a skewed box-test reciprocal, on every extreme scene."""
    for case, (name, tri, _) in enumerate(EXTREMES):
        scene = extreme_scene(tri)
        rays = extreme_rays(tri, 150, case)
        any_rays, want, occ, ex, ex_any = _expected(scene, rays)
        hc = HostCheck(scene, 0, variant)
        assert_hits(hc.trace(rays)[0], want, rays, ex, f"closest, {name}")
        check_sharp(name, lambda r: hc.trace(r)[0], f"host check {variant}")
        for far_first in (False, True):
            got = (hc.trace(any_rays, any_hit=True, far_first=far_first)[0][:, 3].view(U32) != MISS).astype(U8)
            assert_hits(got, occ, any_rays, ex_any, f"any, {name}, far_first={far_first}")


# ---- (2) the device builders' nodes ----------------------------------------------------------------------------------
def check_structure(nodes_u8, order, n):
    """check_bvh8's structural half, for trees over any boxes: every triangle exactly once, imask / meta consistent,
    1..3 triangles per leaf slot, inner children consecutive at child_base and every node reached once."""
    nd = nodes_u8.view(NODE).reshape(-1)
    assert sorted(order.tolist()) == list(range(n)), "tri_order is not a permutation"
    meta = nd["meta"].astype(np.int64)
    used = meta != 0
    inner = used & ((meta & 31) >= 24)
    leaf = used & ~inner
    s8 = np.arange(8)
    assert np.array_equal(nd["imask"], (inner * (1 << s8)).sum(1)), "imask disagrees with meta"
    assert (meta[inner] == (1 << 5) | (24 + np.broadcast_to(s8, meta.shape)[inner])).all()
    unary = meta >> 5
    assert np.isin(unary[leaf], (1, 3, 7)).all(), "a leaf slot without 1 to 3 triangles"
    cnt = np.where(leaf, np.select([unary == 1, unary == 3, unary == 7], [1, 2, 3], 0), 0)
    off = np.cumsum(cnt, 1) - cnt
    assert np.array_equal(np.where(leaf, meta & 31, 0), np.where(leaf, off, 0)), "leaf triangles are not contiguous"
    rank = np.cumsum(inner, 1) - inner
    kids = np.where(inner, nd["child_base"][:, None].astype(np.int64) + rank, -1)[inner]
    assert sorted(kids.tolist()) == list(range(1, len(nd))), "inner children are not the nodes 1..N-1, once each"
    first = nd["tri_base"][:, None].astype(np.int64) + off
    idx = np.concatenate([first[leaf] + k for k in range(3)])[np.concatenate([cnt[leaf] > k for k in range(3)])]
    assert sorted(idx.tolist()) == list(range(n)), "leaf triangles are not the triangles 0..n-1, once each"


def _tris_of(scene):
    return world_tris(scene)


def _device_build_checks(dev, scene, finite):
    tris = _tris_of(scene)
    outs = {}
    for builder in ("ploc", "lbvh"):
        out = dev.build(scene, builder)
        check_structure(out["nodes"], out["leaf_flat_ids"], len(tris))
        if finite:
            check_bvh8(out["nodes"], out["leaf_flat_ids"], tris, out["depth"])
        outs[builder] = out
    return outs


def test_device_builder_nodes(emulated_dev):
    """The emulated device builders on every extreme scene: a valid tree, and check_bvh8 inside the exact bound (past
    2^100 * 255 a node's far plane is not representable, and check_bvh8's conservative test does not apply). The host
    builder's tree likewise."""
    for name, tri, exact in EXTREMES:
        scene = extreme_scene(tri)
        finite = exact and bool(np.isfinite(_tris_of(scene)).all())
        _device_build_checks(emulated_dev, scene, finite)
        hc = HostCheck(scene)
        nodes, order, _, _ = hc.export()
        check_structure(nodes, order, scene.total_tris())
        if finite:
            check_bvh8(nodes, order, _tris_of(scene), hc.stats()["depth"])


@pytest.mark.gpu
def test_gpu_nodes_equal_the_emulated_builds(emulated_dev, device_dev):
    """PLOC and LBVH on the H100 emit the same BVH8 bytes, triangle order and records as their emulated twins on every
    extreme scene: the conversions of infinite boxes to grid exponents and cells follow one rule on both."""
    for name, tri, exact in EXTREMES:
        scene = extreme_scene(tri)
        finite = exact and bool(np.isfinite(_tris_of(scene)).all())
        emu = _device_build_checks(emulated_dev, scene, finite)
        gpu = _device_build_checks(device_dev, scene, finite)
        for builder in ("ploc", "lbvh"):
            for k in ("nodes", "leaf_flat_ids"):
                a, b = emu[builder][k], gpu[builder][k]
                assert np.array_equal(a.view(U8), b.view(U8)), (name, builder, k, np.nonzero((a != b).reshape(len(a), -1).any(1))[0][:5])
            for k in ("tris", "shade"):  # (a NaN the GPU computes is its canonical one, an x86 NaN has the sign bit)
                assert _same_bits_or_nan(emu[builder][k], gpu[builder][k]), (name, builder, k)


# ---- (3) commits of extreme transforms and vertices ------------------------------------------------------------------
def refit_restated(nodes0_u8, leaf_tris):
    """k_bvh8_refit over a tree (the structure of nodes0) and the leaf-order world triangles (n, 3, 3), in float32:
    triangle boxes and every union with fmin / fmax (fminf's NaN rule), deepest level first, quantised by
    test_bvh_build_exact's quantise."""
    nd = nodes0_u8.view(NODE).reshape(-1).copy()
    N = len(nd)
    t = np.asarray(leaf_tris, F32)
    tlo = np.fmin(t[:, 0], np.fmin(t[:, 1], t[:, 2]))
    thi = np.fmax(t[:, 0], np.fmax(t[:, 1], t[:, 2]))
    meta = nd["meta"].astype(np.int64)
    used = meta != 0
    inner = used & ((nd["imask"][:, None] >> np.arange(8)) & 1).astype(bool)
    leaf = used & ~inner
    cnt = np.select([meta >> 5 == 1, meta >> 5 == 3, meta >> 5 == 7], [1, 2, 3], 0)
    rank = np.cumsum(inner, 1) - inner
    child = np.where(inner, nd["child_base"][:, None].astype(np.int64) + rank, 0)
    first = nd["tri_base"][:, None].astype(np.int64) + (meta & 31)
    # levels: BFS numbering puts every child after its parent
    lev = np.zeros(N, np.int64)
    front, depth = np.array([0]), 0
    while len(front):
        lev[front] = depth
        front, depth = child[front][inner[front]], depth + 1
    nlo, nhi = np.zeros((N, 3), F32), np.zeros((N, 3), F32)
    for lv in range(lev.max(), -1, -1):
        ids = np.nonzero(lev == lv)[0]
        m, c = leaf[ids], cnt[ids]
        f0 = np.where(m, first[ids], 0)
        slo, shi = tlo[f0], thi[f0]
        for k in (1, 2):
            mk = m & (c > k)
            fk = np.where(mk, first[ids] + k, 0)
            slo = np.where(mk[..., None], np.fmin(slo, tlo[fk]), slo)
            shi = np.where(mk[..., None], np.fmax(shi, thi[fk]), shi)
        mi = inner[ids]
        ci = child[ids]
        slo = np.where(mi[..., None], nlo[ci], slo)
        shi = np.where(mi[..., None], nhi[ci], shi)
        u = used[ids]
        # (k_bvh8_refit starts the node's union at +-inf: a node whose slots are all NaN on an axis gets +-inf there)
        blo = np.fmin(F32(INF), np.fmin.reduce(np.where(u[..., None], slo, F32(INF)), 1))
        bhi = np.fmax(F32(-INF), np.fmax.reduce(np.where(u[..., None], shi, F32(-INF)), 1))
        nlo[ids], nhi[ids] = blo, bhi
        e, qlo, qhi = quantise(blo, bhi, np.where(u[..., None], slo, 0), np.where(u[..., None], shi, 0))
        nd["p"][ids] = blo
        nd["e"][ids] = e
        nd["qlo"][ids] = np.where(u[..., None], qlo, nd["qlo"][ids].transpose(0, 2, 1)).transpose(0, 2, 1)
        nd["qhi"][ids] = np.where(u[..., None], qhi, nd["qhi"][ids].transpose(0, 2, 1)).transpose(0, 2, 1)
    return nd.view(U8).reshape(N, 80)


def _courtyard():
    return small_courtyard()[0]


def extreme_transforms(scene):
    """(name, transforms): one instance (the one with the most triangles) given each extreme matrix."""
    t = np.array([i.transform for i in scene.instances], F32)
    k = 0
    out = []
    zero = np.zeros((4, 4), F32)
    flat = np.diag([1.0, 0.0, 1.0, 1.0]).astype(F32)
    nan = np.eye(4, dtype=F32)
    nan[1, 2] = NAN
    inf_t = np.eye(4, dtype=F32)
    inf_t[0, 3] = INF
    big = np.diag([1e38, 1e38, 1e38, 1.0]).astype(F32)
    for name, m in (("zeros", zero), ("zero_scale_y", flat), ("nan", nan), ("inf_translation", inf_t), ("scale_1e38", big)):
        new = t.copy()
        new[k] = (m.astype(F64) @ t[k].astype(F64)).astype(F32) if name != "zeros" else m
        out.append((name, new))
    return out


def extreme_vertices(scene):
    """(name, {(mesh, geometry): vertices}): a geometry with one vertex moved to each extreme."""
    m, g = 0, 0
    v = np.asarray(scene.meshes[m].geometries[g].vertices, F32)
    out = []
    for name, val, axis in (("vertex_+inf", INF, 0), ("vertex_-inf", -INF, 1), ("vertex_nan", NAN, 2),
                            ("vertex_3e38", 3e38, 0), ("vertex_-flt_max", -FLT_MAX, 2)):
        w = v.copy()
        w[len(w) // 2, axis] = val
        out.append((name, {(m, g): w}))
    return out


def _commits(scene):
    return ([(n, replaced(scene, transforms=t), dict(instances=t)) for n, t in extreme_transforms(scene)]
            + [(n, replaced(scene, vertices=v), dict(vertices=v)) for n, v in extreme_vertices(scene)])


@pytest.mark.parametrize("which", range(5), ids=["zeros", "zero_scale_y", "nan", "inf_translation", "scale_1e38"])
def test_extreme_instances_match_brute_force(where, which):
    """The courtyard with one instance given each extreme matrix, set with every builder (and, on the GPU, every traversal
    variant): closest hits and occlusion against brute force, ray by ray as the contract says."""
    name, t = extreme_transforms(_courtyard())[which]
    scene = replaced(_courtyard(), transforms=t)
    rays = _scene_rays(scene, 600 if where == "gpu" else 150, which)
    any_rays, want, occ, ex, ex_any = _expected(scene, rays)
    assert ex.mean() > 0.3, name
    for b, builder in enumerate(BUILDERS):
        for variant in (VARIANTS if where == "gpu" else (VARIANTS[(which + b) % len(VARIANTS)],)):
            r = _renderer(scene, builder, variant)
            what = f"{name}, {builder} {variant}"
            assert_hits(r.trace_closest(rays), want, rays, ex, "closest, " + what)
            assert_hits(r.trace_any(any_rays), occ, any_rays, ex_any, "any, " + what)


def _same_bits_or_nan(a, b):
    """Bit for bit, except that a NaN (of a record computed from NaN vertices) may carry another sign or payload."""
    nan = np.isnan(a) & np.isnan(b)
    return bool(np.array_equal(np.where(nan, 0, a.view(U32)), np.where(nan, 0, b.view(U32))))


def test_refit_of_extreme_commits(upd):
    """set_scene of the finite courtyard with dynamic_scene, then one commit of each extreme: every refit node equals
    refit_restated, the structure is the build's, and the records equal a fresh host build's of the moved scene."""
    scene = _courtyard()
    for name, moved, _ in _commits(scene):
        tris = world_tris(moved)
        _, h_order, h_tris, h_shade = HostCheck(moved).export()
        hpos = np.empty(len(h_order), np.int64)
        hpos[h_order] = np.arange(len(h_order))
        for builder in BUILDERS:
            out = upd.update(scene, moved, builder)
            flat = out["leaf_flat_ids"]
            want = refit_restated(out["nodes0"], tris[flat])
            bad = np.nonzero((want != out["nodes"]).any(1))[0]
            assert len(bad) == 0, (name, builder, bad[:5], want[bad[:1]].view(NODE), out["nodes"][bad[:1]].view(NODE))
            before, after = out["nodes0"].view(NODE), out["nodes"].view(NODE)
            for f in ("imask", "child_base", "tri_base", "meta"):
                assert np.array_equal(before[f], after[f]), (name, builder, f)
            for k, want_r in (("tris", h_tris[hpos[flat]]), ("shade", h_shade[hpos[flat]])):
                assert _same_bits_or_nan(out[k], want_r), (name, builder, k)


def _scene_rays(scene, n, seed):
    """Random rays through the finite part of the scene: origins in its finite box, a third of them axis-parallel."""
    t = world_tris(scene).reshape(-1, 3)
    t = t[np.isfinite(t).all(1)]
    lo, hi = t.min(0), t.max(0)
    rng = np.random.default_rng(seed)
    o = rng.uniform(lo - 1, hi + 1, (n, 3))
    d = rng.normal(size=(n, 3))
    k = n // 3
    d[:k] = 0.0
    d[np.arange(k), rng.integers(0, 3, k)] = rng.choice([-1.0, 1.0], k)
    rays = np.concatenate([o, np.full((n, 1), 1e-4), d, np.full((n, 1), 1e30)], 1).astype(F32)
    rays[::4, 3] = 0.0
    return rays


def test_commits_equal_a_fresh_set_scene(where):
    """After a commit of each extreme, trace_closest, trace_any and a frame equal those of a fresh renderer set_scene'd
    with the moved scene (whose hits are brute force's up to the bound); a commit back to the original transforms and
    vertices then renders, traces and occludes exactly as the original scene."""
    from test_dynamic_scene import _args, stage

    scene = _courtyard()
    cam = dict(eye=(0.0, 2.0, 6.0), center=(0.0, 1.0, 0.0), up=(0.0, 1.0, 0.0), fov_y=60.0)
    args = _args(cam)
    rays = _scene_rays(scene, 256, 3)
    original = None
    builders = BUILDERS if where == "gpu" else ("host",)
    for c, (name, moved, change) in enumerate(_commits(scene)):
        builder = builders[c % len(builders)] if where != "gpu" else None
        for b in ((builder,) if builder else builders):
            r = _renderer(scene, b, dynamic_scene=True)
            if original is None:
                original = (r.trace_closest(rays), r.trace_any(rays))
            r.render(*args, True, True)
            stage(r, **change)
            r.commit_scene()
            fresh = _renderer(moved, b)
            frames_equal(r, fresh, args, 1, False)
            assert np.array_equal(r.trace_closest(rays).view(U32), fresh.trace_closest(rays).view(U32)), (name, b)
            assert np.array_equal(r.trace_any(rays), fresh.trace_any(rays)), (name, b)
            back = dict(instances=np.array([i.transform for i in scene.instances], F32)) if "instances" in change else \
                dict(vertices={k: scene.meshes[k[0]].geometries[k[1]].vertices for k in change["vertices"]})
            stage(r, **back)
            r.commit_scene()
            plain = _renderer(scene, b)
            frames_equal(r, plain, args, 1, False)
            assert np.array_equal(r.trace_closest(rays).view(U32), original[0].view(U32)), (name, b)
            assert np.array_equal(r.trace_any(rays), original[1]), (name, b)


# ---- (4) a refit at scale --------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refit_at_c4_scale(device_upd):
    """The C4 workload (bench.WORKLOADS["c4"]) set with the PLOC builder, then its instance rotated and moved: more
    nodes and triangles than the refit kernels' capped grids have threads, so k_reflatten and the widest k_bvh8_refit
    levels loop over the grid stride. Every node equals refit_restated."""
    import bench
    from chameleonrt_b200 import scenes

    from test_dynamic_scene import _rot

    w = bench.WORKLOADS["c4"]
    scene = getattr(scenes, w["gen"])(spp=1, **w["kw"])[0]
    t = np.array([i.transform for i in scene.instances], F64)
    m = _rot(1, 0.3) @ _rot(0, 0.1)
    m[:3, 3] = (3.0, -1.0, 2.0)
    moved = replaced(scene, transforms=np.array([(m @ x).astype(F32) for x in t]))
    out = device_upd.update(scene, moved, "device")
    assert out["n"] > 4_000_000 and out["num_nodes"] > 500_000
    want = refit_restated(out["nodes0"], world_tris(moved)[out["leaf_flat_ids"]])
    bad = np.nonzero((want != out["nodes"]).any(1))[0]
    finite = bool(np.isfinite(out["tris"]).all())
    # (several GB of host arrays: give them back before the next test, which may start a compiler)
    del out, want, scene, moved
    gc.collect()
    assert len(bad) == 0, (len(bad), bad[:5])
    assert finite
