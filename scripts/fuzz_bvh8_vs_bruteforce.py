"""Randomised check of the PRODUCT's host-side BVH8 builder + traversal (libcrt_bvh8_hostcheck.so: the same
bvh8_build.cpp and bvh8_traverse.h the CUDA backend uses) against brute-force intersection by the oracle:
triangle soups at wildly different scales, slivers, duplicated triangles, grids with coincident
vertices, huge + tiny triangles in one scene; rays from random points, from points ON triangles, axis-parallel
rays with exactly zero components travelling along grid lines, short shadow-ray segments. Closest hits must be
bit-identical (t, u, v, primitive id), occlusion answers equal. CPU only.
With --device the same scenes and rays also go through the DEVICE builders (bvh8_device.cuh: PLOC and LBVH, run under
the SIMT emulation of tests/simt_emu) and the production traversal kernel over their trees: same closest hits, bit for
bit, and the same occlusion answers as brute force.
    python scripts/fuzz_bvh8_vs_bruteforce.py [n] [first_seed] [--device]"""
import os
import sys
import warnings

import numpy as np

warnings.filterwarnings("ignore")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from chameleonrt_b200.scene import DisneyMaterial, Geometry, Instance, Mesh, ParameterizedMesh, Scene, default_obj_light  # noqa: E402
from chameleonrt_b200.scenes import MeshBuilder, grid  # noqa: E402
from helpers import HostCheck  # noqa: E402
from oracle import OracleBackend  # noqa: E402


def random_geometry(rng, scene_scale):
    b = MeshBuilder()
    # Within one scene sizes span two decades; the scene as a whole sits anywhere from 1e-3 to 1e3. (Mixing 1e-3-
    # and 1e3-sized objects in ONE scene puts millimetre triangles 1e4 units from the ray origin, where the float
    # spacing of the origin is as large as the triangle: seed 106 of the first version — no traversal can be
    # asked to agree with brute force there.)
    scale = scene_scale * 10.0 ** rng.uniform(-1, 1)
    kind = int(rng.integers(0, 5))
    n = int(rng.integers(1, 400))
    if kind == 0:      # soup
        v = rng.normal(size=(n, 3, 3)) * rng.uniform(0.01, 1.0) + rng.normal(size=(n, 1, 3)) * 2.0
    elif kind == 1:    # slivers: three nearly collinear vertices (exactly zero-area triangles are left out: with
        # det = rounding noise the triangle formula returns an arbitrary t that has nothing to do with the
        # triangle's box, so "closest hit" is not defined for them in any traversal, brute force included)
        v = rng.normal(size=(n, 1, 3)) * 2.0 + rng.normal(size=(n, 3, 1)) * rng.normal(size=(n, 1, 3)) + rng.normal(size=(n, 3, 3)) * 1e-3
    elif kind == 2:    # duplicates and coincident sheets
        base = rng.normal(size=(max(1, n // 3), 3, 3))
        v = np.concatenate([base, base, base[::-1] + 0.0])
    elif kind == 3:    # huge + tiny
        v = rng.normal(size=(n, 3, 3)) * np.where(rng.random((n, 1, 1)) < 0.1, 50.0, 0.02) + rng.normal(size=(n, 1, 3))
    else:              # axis-aligned grids on power-of-two coordinates (rays will run along their lines)
        gv, guv, gi = grid((-2.0, -2.0, float(rng.integers(-2, 3))), (4.0, 0.0, 0.0), (0.0, 4.0, 0.0), int(rng.integers(1, 17)), int(rng.integers(1, 17)))
        b.add(np.asarray(gv) * scale, guv, gi)
        return b.geometry()
    v = (v * scale).astype(np.float32)
    b.add(v.reshape(-1, 3), np.zeros((v.shape[0] * 3, 2), np.float32), np.arange(v.shape[0] * 3, dtype=np.uint32).reshape(-1, 3))
    return b.geometry()


def random_rays(rng, scene, n):
    verts = np.concatenate([np.asarray(g.vertices, np.float32) for g in scene.meshes[0].geometries])
    lo, hi = verts.min(0), verts.max(0)
    ext = np.maximum(hi - lo, 1e-6)
    o = lo + rng.random((n, 3)) * ext * rng.choice([1.0, 3.0]) - ext * rng.choice([0.0, 1.0])
    d = rng.normal(size=(n, 3))
    # a third of the rays start on a vertex / towards a vertex; a sixth are axis-parallel with exact zeros
    k = n // 3
    o[:k] = verts[rng.integers(0, len(verts), k)]
    tgt = verts[rng.integers(0, len(verts), k)]
    d[k:2 * k] = tgt - o[k:2 * k]
    ax = rng.integers(0, 3, n // 6)
    d[-(n // 6):] = 0.0
    d[np.arange(n - n // 6, n), ax] = rng.choice([-1.0, 1.0], n // 6)
    o[-(n // 6):] = verts[rng.integers(0, len(verts), n // 6)] - d[-(n // 6):] * ext.max()
    d = d / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-30)
    tnear = np.where(rng.random(n) < 0.5, 0.0, 1e-4)
    tfar = np.where(rng.random(n) < 0.5, 1e20, rng.random(n) * ext.max() * 2)
    return np.ascontiguousarray(np.concatenate([o, tnear[:, None], d, tfar[:, None]], 1), np.float32)


def scene_of(geoms):
    """A one-mesh, identity-instanced scene of the given geometries."""
    return Scene(meshes=[Mesh(geoms)], parameterized_meshes=[ParameterizedMesh(0, [0] * len(geoms))],
                 instances=[Instance(np.eye(4, dtype=np.float32), 0)], materials=[DisneyMaterial()], textures=[],
                 lights=[default_obj_light()], samples_per_pixel=1)


def without_needles(scene):
    """``scene`` with its needle triangles (2 * area / longest edge^2 < 1e-2) removed, as one geometry; the scene itself
    if it has none. Needles are ill-conditioned for the triangle formula itself: the computed t can be off by far more
    than rounding (seed 98: a 0.04-long sliver 800 units away "hit" at t = 800.911 while its box spans
    [800.939, 800.943]), so no hierarchy can agree with brute force on them."""
    tris = np.concatenate([np.asarray(g.vertices, np.float32)[np.asarray(g.indices, np.uint32).reshape(-1, 3)]
                           for g in scene.meshes[0].geometries]).astype(np.float64)
    e = [tris[:, 1] - tris[:, 0], tris[:, 2] - tris[:, 0], tris[:, 2] - tris[:, 1]]
    longest = np.maximum(np.maximum((e[0] ** 2).sum(1), (e[1] ** 2).sum(1)), (e[2] ** 2).sum(1))
    quality = np.linalg.norm(np.cross(e[0], e[1]), axis=1) / np.maximum(longest, 1e-300)
    if not (quality < 1e-2).any():
        return scene
    kept = tris[quality >= 1e-2].astype(np.float32)
    b = MeshBuilder()
    b.add(kept.reshape(-1, 3), np.zeros((len(kept) * 3, 2), np.float32), np.arange(len(kept) * 3, dtype=np.uint32).reshape(-1, 3))
    return scene_of([b.geometry()])


_backend = None


def device_builders_agree(scene, rays, hb, occ):
    """The emulated renderer over each builder's tree: closest hits == the host check's (already compared with brute
    force); occlusion == brute force's."""
    for builder in ("host", "device", "device_lbvh"):
        r = _backend.RenderCUDA(0, bvh_builder=builder)
        r.initialize(8, 8)
        r.set_scene(scene)
        if not np.array_equal(r.trace_closest(rays).view(np.uint32), hb.view(np.uint32)):
            return False
        if not np.array_equal(r.trace_any(rays).astype(bool), occ):
            return False
    return True


def one(seed, device=False, hostcheck=HostCheck):
    """Seed ``seed`` against brute force; ``hostcheck(scene, threads)`` makes the host check that is compared."""
    rng = np.random.default_rng(seed)
    scene_scale = 10.0 ** rng.uniform(-3, 3)
    geoms = [random_geometry(rng, scene_scale) for _ in range(int(rng.integers(1, 4)))]
    scene = scene_of(geoms)
    rays = random_rays(rng, scene, 600)
    threads = int(rng.integers(0, 4))
    # the comparison is about the hierarchy, not the formula: both sides run on the scene without its needles
    scene = without_needles(scene)
    if scene.total_tris() == 0:
        return True, (True, True, True, 0)
    brute = OracleBackend(brute_force=True)
    brute.initialize(8, 8)
    brute.set_scene(scene)
    hc = hostcheck(scene, threads)
    hb, _, _ = hc.trace(rays)
    ho = brute.trace_closest(rays)
    same_closest = np.array_equal(hb.view(np.uint32), ho.view(np.uint32))
    ha, _, _ = hc.trace(rays, any_hit=True)
    hf, _, _ = hc.trace(rays, any_hit=True, far_first=True)
    occ = brute.trace_any(rays).astype(bool)
    same_any = np.array_equal(ha[:, 3].view(np.uint32) != 0xFFFFFFFF, occ) and np.array_equal(hf[:, 3].view(np.uint32) != 0xFFFFFFFF, occ)
    same_device = True
    if device:
        same_device = device_builders_agree(scene, rays, hb, occ)
    return same_closest and same_any and same_device, (same_closest, same_any, same_device, scene.total_tris())


if __name__ == "__main__":
    device = "--device" in sys.argv
    args = [a for a in sys.argv[1:] if a != "--device"]
    n = int(args[0]) if len(args) > 0 else 100
    first = int(args[1]) if len(args) > 1 else 0
    if device:
        sys.path.insert(0, os.path.join(ROOT, "tests", "simt_emu"))
        import build as simt_build
        import chameleonrt_b200.backend as _backend

        _backend._LIB_PATH, _backend._lib = simt_build.build(), None
    bad = 0
    for seed in range(first, first + n):
        ok, info = one(seed, device)
        if not ok:
            bad += 1
            print("MISMATCH seed", seed, info)
    print(f"{n} random scenes x 600 rays, {bad} mismatches" + (" (host + device builders)" if device else ""))
