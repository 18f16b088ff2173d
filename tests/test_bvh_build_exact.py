"""The device BVH build (bvh8_device.cuh driven by scene_device_build.cuh, options bvh_builder = "device" /
"device_lbvh") stage by stage, against plain numpy restatements, and every BVH8 node of both builders decoded in float64.

Frames cannot see the tree (closest hits tie-break on the flattened id, DESIGN.md §5), so these checks look at the
build's own output: the exclusive scans, the radix sort, the Morton keys and centroid bounds, the binary tree (Karras
for LBVH, PLOC round by round), its boxes and the collapse DP, the emitted BVH8 node bytes and triangle order, and the
packed scene records. libcrt_bvh_devcheck.so (bvh_devcheck.cu) calls the product's own driver code; the same file is
built for the host under the SIMT emulation (tests/simt_emu), so every check runs without a GPU on the emulated device
build and with ``-m gpu`` on an H100. The BVH8 invariants of (f) also run on the host builder's tree.
Every comparison is exact (uint32 / uint64 views) unless it says float64. Set CRT_SIMT_FULL=1 for the larger
emulated sizes."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "chameleonrt_b200", "csrc")
FULL = os.environ.get("CRT_SIMT_FULL") == "1"
F32, F64, U8, U32, U64 = np.float32, np.float64, np.uint8, np.uint32, np.uint64
INVALID = 0xFFFFFFFF
TILE = 2048


# ---- the builds ----
class DevCheck:
    """bvhdev_* of libcrt_bvh_devcheck.so (``gpu``) or of its emulated twin, on numpy arrays."""

    def __init__(self, path, name, gpu):
        self.name, self.gpu = name, gpu
        self.lib = lib = C.CDLL(path)
        vp, u32 = C.c_void_p, C.c_uint32
        lib.bvhdev_last_error.restype = C.c_char_p
        for f in ("bvhdev_scan_u32", "bvhdev_scan_u64"):
            getattr(lib, f).argtypes, getattr(lib, f).restype = [vp, u32, vp], C.c_int
        lib.bvhdev_sort_pairs.argtypes, lib.bvhdev_sort_pairs.restype = [vp, vp, u32], C.c_int
        lib.bvhdev_build.argtypes, lib.bvhdev_build.restype = [vp, C.c_int, C.c_int, C.c_int, vp], vp
        lib.bvhdev_fetch.argtypes, lib.bvhdev_fetch.restype = [vp, C.c_int, vp], C.c_longlong
        lib.bvhdev_free.argtypes = [vp]

    def _check(self, rc, what):
        assert rc == 0, f"{self.name}: {what}: {self.lib.bvhdev_last_error().decode()}"

    def scan(self, a):
        a = np.ascontiguousarray(a)
        out = np.zeros_like(a)
        f = self.lib.bvhdev_scan_u64 if a.dtype == U64 else self.lib.bvhdev_scan_u32
        self._check(f(a.ctypes.data, len(a), out.ctypes.data), "scan")
        return out

    def sort(self, keys, vals):
        k, v = np.array(keys, U64), np.array(vals, U32)
        self._check(self.lib.bvhdev_sort_pairs(k.ctypes.data, v.ctypes.data, len(k)), "sort")
        return k, v

    def build(self, scene, builder, tail=True, radius=16):
        """The device set_scene of `scene`: builder "ploc" or "lbvh"."""
        ms = scene.to_c()
        info = np.zeros(5, U32)
        h = self.lib.bvhdev_build(C.byref(ms.c), 1 if builder == "ploc" else 2, int(tail), radius, info.ctypes.data)
        assert h, f"{self.name}: build: {self.lib.bvhdev_last_error().decode()}"
        n, nn = int(info[0]), int(info[1])
        nb2 = 2 * n - 1
        shapes = [("nodes", U8, (nn, 80)), ("tris", F32, (n, 12)), ("shade", F32, (n, 12)), ("leaf_flat_ids", U32, (n,)),
                  ("keys", U64, (n,)), ("vals", U32, (n,)), ("cbounds", U32, (6,)), ("children", U32, (n - 1, 2)),
                  ("box_lo", F32, (nb2, 4)), ("box_hi", F32, (nb2, 4)), ("cost", F32, (nb2, 7)), ("decision", U8, (nb2, 7))]
        out = dict(n=n, num_nodes=nn, depth=int(info[2]), rounds=int(info[3]), root=int(info[4]), builder=builder)
        try:
            for field, (name, dt, shape) in enumerate(shapes):
                a = np.zeros(shape, dt)
                got = self.lib.bvhdev_fetch(h, field, a.ctypes.data)
                assert got == a.nbytes, (name, got, a.nbytes)
                out[name] = a
        finally:
            self.lib.bvhdev_free(h)
        return out


@pytest.fixture(scope="module")
def emulated(built):
    sys.path.insert(0, os.path.join(ROOT, "tests", "simt_emu"))
    import build as simt_build

    return DevCheck(simt_build.build_bvh_devcheck(), "emulated", False)


@pytest.fixture(scope="module")
def device(built):
    path = os.path.join(CSRC, "libcrt_bvh_devcheck.so")
    if not os.path.exists(path):  # (a tree built before the check library existed)
        subprocess.check_call(["make", "-s", "-C", CSRC, "libcrt_bvh_devcheck.so"])
    return DevCheck(path, "device", True)


@pytest.fixture(params=[pytest.param("emulated"), pytest.param("device", marks=pytest.mark.gpu)], scope="module")
def dev(request):
    """The device build under test: the SIMT emulation without a GPU, the sm_90a build with ``-m gpu``."""
    return request.getfixturevalue(request.param)


# ---- scenes ----
def soup_scene(verts, idx=None):
    from chameleonrt_b200.scene import DisneyMaterial, Geometry, Instance, Mesh, ParameterizedMesh, Scene, default_obj_light

    verts = np.ascontiguousarray(np.asarray(verts, F32).reshape(-1, 3))
    idx = np.arange(len(verts), dtype=U32).reshape(-1, 3) if idx is None else np.ascontiguousarray(idx, U32)
    return Scene(meshes=[Mesh([Geometry(verts, idx)])], parameterized_meshes=[ParameterizedMesh(0, [0])],
                 instances=[Instance(np.eye(4, dtype=F32), 0)], materials=[DisneyMaterial()], lights=[default_obj_light()])


def random_soup(n, seed, spread=1.0, size=0.05):
    rng = np.random.default_rng(seed)
    c = rng.uniform(-spread, spread, (n, 1, 3))
    return (c + rng.normal(scale=size * spread, size=(n, 3, 3))).astype(F32)


def chain_soup(k=900):
    """Triangles along x whose gaps shrink by 0.5 %: every cluster's nearest neighbour is the next one, so PLOC merges
    one mutual pair per round until its 256-round cut-off pairs neighbours up."""
    x = np.cumsum(0.995 ** np.arange(k)).astype(F32)
    tri = np.array([[0, 0, 0], [1e-4, 0, 0], [0, 1e-4, 0]], F32)
    return tri[None] + np.stack([x, np.zeros(k, F32), np.zeros(k, F32)], 1)[:, None]


def key_scenes():
    """Scenes for the Morton keys: (name, triangles)."""
    rng = np.random.default_rng(11)
    flat = random_soup(300, 1)
    flat[:, :, 1] = 0.0
    one = np.array([[[0.5, -1.0, 2.0], [1.5, -0.5, 2.0], [0.7, 0.0, 3.0]]], F32)
    coincident = np.repeat(random_soup(1, 2), 40, axis=0)
    coincident[::3] = coincident[::3][:, ::-1]  # the same triangle, vertices in another order: the same centroid
    mixed = random_soup(2000, 3, spread=50.0)
    scales = np.concatenate([random_soup(400, 10 + i, spread=s) for i, s in enumerate((1e-3, 1e-1, 1.0, 1e1, 1e3))])
    huge = np.concatenate([random_soup(600, 20, spread=1.0, size=1e-4), random_soup(8, 21, spread=1.0, size=3e4)])
    rng.shuffle(huge)
    return [("flat", flat), ("one", one), ("coincident", coincident), ("mixed_sign", mixed), ("scales", scales),
            ("huge_and_tiny", huge)]


def tree_scenes(dev):
    """Scenes for the tree, the DP and the emitted BVH8: (name, scene), sized for the build under test."""
    from chameleonrt_b200.scenes import cornell_box, rungholt_like, sponza_like

    out = [("cornell", cornell_box()[0]), ("soup_2049", soup_scene(random_soup(2049, 4))),
           ("dups", soup_scene(np.repeat(random_soup(7, 5), 5, axis=0))), ("two", soup_scene(random_soup(2, 6))),
           ("sponza_small", sponza_like(spp=1, detail=0.12, tex_size=16)[0])]
    if dev.gpu or FULL:
        out.append(("rungholt_small", rungholt_like(spp=1, scale=0.25)[0]))
    if dev.gpu:
        out.append(("sponza_c2", sponza_like(spp=1, tex_size=16)[0]))
    return out


def big_scenes():
    """GPU-only sizes: a rungholt_like above 1 M triangles and a soup above 2048^2, so that every scan of the build
    (the first PLOC round's included) takes the three-level path."""
    from chameleonrt_b200.scenes import rungholt_like

    return [("rungholt_1m", rungholt_like(spp=1, scale=1.0)[0]), ("soup_4.3m", soup_scene(random_soup(2048 * 2048 + 97_000, 9)))]


def tri_verts(scene):
    """The flattened triangles (n, 3, 3) in world space, in flattened order, for single-instance identity scenes."""
    out = []
    for inst in scene.instances:
        pm = scene.parameterized_meshes[inst.parameterized_mesh_id]
        for g in scene.meshes[pm.mesh_id].geometries:
            v = np.asarray(g.vertices, F32)[np.asarray(g.indices, np.int64)]
            assert np.array_equal(inst.transform, np.eye(4, dtype=F32))
            out.append(v)
    return np.concatenate(out)


# ---- (a) scans ----
def _exclusive(a):
    c = np.cumsum(a, dtype=a.dtype)  # (wraps like the kernel's integer adds)
    return np.concatenate([np.zeros(1, a.dtype), c[:-1]])


def scan_sizes(dev):
    return [1, 255, 2047, 2048, 2049, 9 * TILE + 3] + ([TILE * TILE, TILE * TILE + 1] if dev.gpu or FULL else [])


def test_scan_against_cumsum(dev):
    """DeviceSceneBuild::device_scan (k_scan_tile, the recursive scan of the tile sums, k_scan_add), uint32 and uint64,
    against np.cumsum. The uint64 items straddle 2^32 so that carries cross the word; 2048^2 + 1 items is the smallest
    input with a third level."""
    rng = np.random.default_rng(1)
    for n in scan_sizes(dev):
        a32 = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(U32)
        assert np.array_equal(dev.scan(a32), _exclusive(a32)), ("u32", n)
        a64 = rng.integers((1 << 31) - 5, (1 << 33) + 5, n, dtype=np.uint64)
        a64[::7] = 0xFFFFFFFF
        assert np.array_equal(dev.scan(a64), _exclusive(a64)), ("u64", n)
        small = np.ones(n, U32)  # (the counts a PLOC round or a BVH8 level scans)
        assert np.array_equal(dev.scan(small), np.arange(n, dtype=U32)), ("ones", n)


# ---- (b) radix sort ----
def key_sets(n, rng):
    m63 = np.uint64((1 << 63) - 1)
    base = rng.integers(0, 1 << 63, 1, dtype=np.uint64)[0]
    return {
        "random63": rng.integers(0, 1 << 63, n, dtype=np.uint64) & m63,
        "five_values": rng.choice(rng.integers(0, 1 << 63, 5, dtype=np.uint64), n),
        "bits_56_62": (base & np.uint64((1 << 56) - 1)) | (rng.integers(0, 128, n, dtype=np.uint64) << np.uint64(56)),
        "bit_0": (base & ~np.uint64(1)) | rng.integers(0, 2, n, dtype=np.uint64),
        "all_equal": np.full(n, base, U64),
    }


def test_radix_sort_against_stable_argsort(dev):
    """DeviceSceneBuild::radix_sort (8 passes of k_radix_hist, scan, k_radix_scatter) against np.argsort(kind="stable"):
    the values are a random permutation, so they must travel with their keys and keep their order among equal keys."""
    rng = np.random.default_rng(2)
    sizes = [1, 31, 32, 33, 256, 257, 2047, 2048, 2049, 9 * TILE + 1] + ([5_000_011] if dev.gpu else [])
    for n in sizes:
        for name, keys in key_sets(n, rng).items():
            vals = rng.permutation(n).astype(U32)
            k, v = dev.sort(keys, vals)
            order = np.argsort(keys, kind="stable")
            assert np.array_equal(k, keys[order]), (name, n, "keys")
            assert np.array_equal(v, vals[order]), (name, n, "values")


# ---- (c) Morton keys, centroid bounds ----
def spread21(v):
    x = v.astype(U64) & U64(0x1FFFFF)
    for sh, mask in ((32, 0x1F00000000FFFF), (16, 0x1F0000FF0000FF), (8, 0x100F00F00F00F00F), (4, 0x10C30C30C30C30C3),
                     (2, 0x1249249249249249)):
        x = (x | (x << U64(sh))) & U64(mask)
    return x


def morton_restated(tris):
    """k_lbvh_bounds + k_lbvh_keys in float32, operation by operation: the triangle boxes, the centroids 0.5 lo + 0.5 hi,
    their bounds, scale = 2^21 / extent (0 for a flat axis), clamp to [0, 2^21 - 1], truncate, interleave x y z."""
    tl = np.fmin(tris[:, 0], np.fmin(tris[:, 1], tris[:, 2]))
    th = np.fmax(tris[:, 0], np.fmax(tris[:, 1], tris[:, 2]))
    c = F32(0.5) * tl + F32(0.5) * th
    lo = np.fmin(F32(3.0e38), c.min(0))
    hi = np.fmax(F32(-3.0e38), c.max(0))
    ext = hi - lo
    with np.errstate(divide="ignore"):
        scale = np.where(ext > 0, F32(2097152.0) / np.where(ext > 0, ext, F32(1)), F32(0)).astype(F32)
    g = np.fmin(np.fmax((c - lo) * scale, F32(0)), F32(2097151.0))
    q = g.astype(U32)
    keys = (spread21(q[:, 0]) << U64(2)) | (spread21(q[:, 1]) << U64(1)) | spread21(q[:, 2])
    return tl, th, lo, hi, keys


def _from_ordered(u):
    u = u.astype(U32)
    return np.where(u & U32(0x80000000), u & U32(0x7FFFFFFF), ~u).astype(U32).view(F32)


def test_morton_keys_and_centroid_bounds(dev):
    """The build's sorted keys and triangle ids, and its centroid bounds, against morton_restated sorted stably."""
    for name, tris in key_scenes() + [("chain", chain_soup())]:
        out = dev.build(soup_scene(tris), "lbvh")
        tl, th, lo, hi, keys = morton_restated(tris)
        cb = _from_ordered(out["cbounds"])
        assert np.array_equal(cb[:3], lo) and np.array_equal(cb[3:], hi), (name, cb, lo, hi)
        order = np.argsort(keys, kind="stable")
        assert np.array_equal(out["keys"], keys[order]), name
        assert np.array_equal(out["vals"], order.astype(U32)), name
        if name == "flat":  # (the flat axis has scale 0: its key bits are all zero)
            assert (np.bitwise_or.reduce(out["keys"]) & (spread21(np.full(1, 0x1FFFFF, U32))[0] << U64(1))) == 0


# ---- (d) the binary tree, its boxes and the collapse DP ----
def half_area(lo, hi):
    d = hi[..., :3] - lo[..., :3]
    return d[..., 0] * d[..., 1] + d[..., 1] * d[..., 2] + d[..., 2] * d[..., 0]


def check_shape(out):
    """A binary tree over exactly n leaves: every node but the root is a child exactly once; no cycles."""
    n, ch, root = out["n"], out["children"].astype(np.int64), out["root"]
    if n == 1:
        assert root == 0
        return np.zeros(1, np.int64)
    assert n <= root < 2 * n - 1
    assert ((ch >= 0) & (ch < 2 * n - 1)).all()
    seen = np.bincount(ch.ravel(), minlength=2 * n - 1)
    want = np.ones(2 * n - 1, np.int64)
    want[root] = 0
    assert np.array_equal(seen, want), "a node is a child of none or of several nodes"
    # every node reachable from the root (with in-degree 1 and 2n - 2 edges: a tree, no cycle)
    height = np.zeros(2 * n - 1, np.int64)
    level, reached = np.array([root]), 1
    depth = 0
    while len(level):
        inner = level[level >= n]
        level = ch[inner - n].ravel()
        reached += len(level)
        depth += 1
        assert depth <= 2 * n, "cycle"
    assert reached == 2 * n - 1
    # node heights (leaves 0), for the bottom-up restatements
    for _ in range(2 * n):
        h = np.maximum(height[ch[:, 0]], height[ch[:, 1]]) + 1
        if np.array_equal(height[n:], h):
            break
        height[n:] = h
    return height


def check_boxes(out, tris):
    """Leaf j's box is triangle vals[j]'s box with count 1; every internal box is the float min / max of its children's,
    value for value, and its count the sum. On the GPU this is what a stale read in k_lbvh_refit would break."""
    n, ch, lo, hi = out["n"], out["children"].astype(np.int64), out["box_lo"], out["box_hi"]
    tl = np.fmin(tris[:, 0], np.fmin(tris[:, 1], tris[:, 2]))
    th = np.fmax(tris[:, 0], np.fmax(tris[:, 1], tris[:, 2]))
    assert np.array_equal(lo[:n, :3], tl[out["vals"]]) and np.array_equal(hi[:n, :3], th[out["vals"]])
    assert (lo[:n, 3].view(U32) == 1).all()
    if n > 1:
        l, r = ch[:, 0], ch[:, 1]
        assert np.array_equal(lo[n:, :3], np.fmin(lo[l, :3], lo[r, :3])), "internal box_lo is not the children's min"
        assert np.array_equal(hi[n:, :3], np.fmax(hi[l, :3], hi[r, :3])), "internal box_hi is not the children's max"
        assert np.array_equal(lo[n:, 3].view(U32), lo[l, 3].view(U32) + lo[r, 3].view(U32))
    assert lo[out["root"], 3].view(U32) == n


def dp_restated(out, height):
    """collapse_dp / Collapser::run in float32, node by node in height order: cost[i] = the cheapest forest of at most
    i + 1 BVH8 children, and the decision (type | dist_left << 2 | dist_right << 5) that achieves it."""
    n, ch = out["n"], out["children"].astype(np.int64)
    lo, hi = out["box_lo"], out["box_hi"]
    cost = np.zeros((2 * n - 1, 7), F32)
    dec = np.zeros((2 * n - 1, 7), U8)
    cost[:n] = (half_area(lo[:n], hi[:n]) * F32(0.3))[:, None]
    cnt = lo[:, 3].view(U32).astype(np.int64)
    inf = F32(np.inf)
    for h in range(1, int(height.max()) + 1 if n > 1 else 1):
        p = np.nonzero(height[n:] == h)[0] + n
        l, r = ch[p - n, 0], ch[p - n, 1]
        cl, cr = cost[l], cost[r]
        area = half_area(lo[p], hi[p])
        c = cnt[p]
        cost_leaf = np.where(c <= 3, area * c.astype(F32) * F32(0.3), inf).astype(F32)
        sums = cl + cr[:, ::-1]  # k: cl[k] + cr[6 - k]
        bl = np.argmin(sums, axis=1)  # (strict <, first k wins: the first minimum)
        best = sums[np.arange(len(p)), bl]
        cost_int = best + area * F32(1.0)
        leaf = cost_leaf < cost_int
        cn = np.where(leaf, cost_leaf, cost_int).astype(F32)
        dn = np.where(leaf, 0, 1 | (bl << 2) | ((6 - bl) << 5)).astype(U8)
        cost[p, 0], dec[p, 0] = cn, dn
        for i in range(1, 7):
            cn, dn = cn.copy(), dn.copy()
            for k in range(i):
                s = cl[:, k] + cr[:, i - k - 1]
                better = s < cn
                cn = np.where(better, s, cn)
                dn = np.where(better, 2 | (k << 2) | ((i - k - 1) << 5), dn).astype(U8)
            cost[p, i], dec[p, i] = cn, dn
    return cost, dec


def _clz32(x):
    x = np.asarray(x, np.int64)
    return np.where(x == 0, 32, 32 - np.frexp(x.astype(F64))[1])  # (exact: x < 2^32)


def _clz64(x):
    x = np.asarray(x, U64)
    h, lo = (x >> U64(32)).astype(np.int64), (x & U64(0xFFFFFFFF)).astype(np.int64)
    return np.where(h != 0, _clz32(h), 32 + _clz32(lo))


def karras_restated(keys):
    """k_lbvh_hierarchy in integers: every internal node i finds its direction, range and split; equal keys tie-break
    on the position (64 + clz(i ^ j))."""
    n = len(keys)
    i = np.arange(n - 1, dtype=np.int64)

    def delta(a, b):
        ok = (b >= 0) & (b < n)
        bb = np.clip(b, 0, n - 1)
        ka, kb = keys[a], keys[bb]
        d = np.where(ka == kb, 64 + _clz32(a ^ bb), _clz64(ka ^ kb))
        return np.where(ok, d, -1)

    d = np.where(delta(i, i + 1) - delta(i, i - 1) >= 0, 1, -1)
    dmin = delta(i, i - d)
    lmax = np.full(n - 1, 2, np.int64)
    grow = delta(i, i + lmax * d) > dmin
    while grow.any():
        lmax = np.where(grow, lmax * 2, lmax)
        grow &= delta(i, i + lmax * d) > dmin
    l = np.zeros(n - 1, np.int64)
    t = lmax // 2
    while (t >= 1).any():
        ok = (t >= 1) & (delta(i, i + (l + t) * d) > dmin)
        l = np.where(ok, l + t, l)
        t = t // 2
    j = i + l * d
    dnode = delta(i, j)
    s = np.zeros(n - 1, np.int64)
    t = l.copy()
    live = np.ones(n - 1, bool)
    while live.any():  # do { t = (t + 1) / 2; ... } while (t > 1)
        t = np.where(live, (t + 1) // 2, t)
        ok = live & (delta(i, i + (s + t) * d) > dnode)
        s = np.where(ok, s + t, s)
        live &= t > 1
    gamma = i + s * d + np.minimum(d, 0)
    first, last = np.minimum(i, j), np.maximum(i, j)
    left = np.where(first == gamma, gamma, n + gamma)
    right = np.where(last == gamma + 1, gamma + 1, n + gamma + 1)
    return np.stack([left, right], 1).astype(U32)


def ploc_restated(out, radius=16):
    """PLOC round by round (k_ploc_nn / mark / scan / merge, and k_ploc_tail, which runs the same rounds): nearest
    neighbours by merged half area in float32, candidates in ascending position, ties to the aligned partner i ^ 1 then
    the lower position; mutual pairs merge, numbered by the exclusive scan; after 256 rounds neighbours are paired."""
    n = out["n"]
    lo = np.zeros((2 * n - 1, 3), F32)
    hi = np.zeros((2 * n - 1, 3), F32)
    lo[:n], hi[:n] = out["box_lo"][:n, :3], out["box_hi"][:n, :3]
    children = np.zeros((max(n - 1, 0), 2), U32)
    cl = np.arange(n, dtype=np.int64)
    made, rounds = 0, 0
    while len(cl) > 1:
        m = len(cl)
        pos = np.arange(m)
        if rounds >= 256:
            nn = np.where((pos ^ 1) < m, pos ^ 1, pos)
        else:
            clo, chi = lo[cl], hi[cl]
            best = np.full(m, np.inf, F32)
            best_j = pos.copy()
            for o in range(-radius, radius + 1):
                j = pos + o
                ok = (o != 0) & (j >= 0) & (j < m)
                jj = np.clip(j, 0, m - 1)
                a = half_area(np.fmin(clo, clo[jj]), np.fmax(chi, chi[jj]))
                rank_j = np.where(j == (pos ^ 1), 0, 1)
                rank_b = np.where(best_j == (pos ^ 1), 0, 1)
                take = ok & ((best_j == pos) | (a < best) | ((a == best) & (rank_j < rank_b)))
                best = np.where(take, a, best)
                best_j = np.where(take, j, best_j)
            nn = best_j
        mutual = (nn != pos) & (nn[nn] == pos)
        keep = ~(mutual & (nn < pos))
        lead = mutual & (pos < nn)
        k = made + np.cumsum(lead) - lead
        kk = k[lead]
        children[kk, 0], children[kk, 1] = cl[lead], cl[nn[lead]]
        lo[n + kk] = np.fmin(lo[cl[lead]], lo[cl[nn[lead]]])
        hi[n + kk] = np.fmax(hi[cl[lead]], hi[cl[nn[lead]]])
        assert lead.sum() > 0, "a PLOC round without a merge"
        new = np.where(lead, n + k, cl)
        cl = new[keep]
        made += int(lead.sum())
        rounds += 1
    return children, rounds


def check_tree(out, tris, dp=True, restate_topology=True):
    height = check_shape(out)
    check_boxes(out, tris)
    if restate_topology and out["n"] > 1:
        if out["builder"] == "lbvh":
            assert out["root"] == out["n"]
            assert np.array_equal(out["children"], karras_restated(out["keys"])), "LBVH children"
        else:
            assert out["root"] == 2 * out["n"] - 2
            children, rounds = ploc_restated(out)
            assert np.array_equal(out["children"], children), "PLOC children"
            assert out["rounds"] == rounds, (out["rounds"], rounds)
    if dp:
        cost, dec = dp_restated(out, height)
        assert np.array_equal(out["cost"].view(U32), cost.view(U32)), "DP costs"
        assert np.array_equal(out["decision"], dec), "DP decisions"


BUILDS = [("ploc", True), ("ploc", False), ("lbvh", True)]


def test_binary_tree_and_dp_restated(dev):
    """The dumped BVH2 of PLOC (with and without k_ploc_tail) and of LBVH: shape, boxes, the topology against the
    builder's restatement (Karras / PLOC round by round, round count included) and the collapse DP node by node."""
    cases = [(name, tri_verts(s)) for name, s in tree_scenes(dev)] + [("chain", chain_soup())] + key_scenes()
    for name, tris in cases:
        for builder, tail in BUILDS:
            out = dev.build(soup_scene(tris), builder, tail)
            check_tree(out, tris)
            if name == "chain" and builder == "ploc":
                assert out["rounds"] > 256, "the chain was meant to reach the forced pairing"


# ---- (e) the emitted BVH8, byte for byte ----
NODE = np.dtype([("p", "<f4", 3), ("e", "u1", 3), ("imask", "u1"), ("child_base", "<u4"), ("tri_base", "<u4"),
                 ("meta", "u1", 8), ("qlo", "u1", (3, 8)), ("qhi", "u1", (3, 8))])
assert NODE.itemsize == 80


def assign_slots(plo, phi, clo, chi):
    """assign_slots in float32: slot s takes the child met first by rays of octant s, greedily by the minimum of
    dot(centroid offset, d_s); ties to the lower child, then the lower slot. Returns slot -> child index (-1: empty)."""
    cx = F32(0.5) * (plo[:3] + phi[:3])
    o = F32(0.5) * (clo[:, :3] + chi[:, :3]) - cx
    sgn = np.array([[-1 if s & 4 else 1, -1 if s & 2 else 1, -1 if s & 1 else 1] for s in range(8)], F32)
    cst = o[:, 0:1] * sgn[None, :, 0] + o[:, 1:2] * sgn[None, :, 1] + o[:, 2:3] * sgn[None, :, 2]
    slot_child = np.full(8, -1)
    cst = cst.astype(F64)
    for _ in range(len(clo)):
        flat = np.argmin(cst.ravel())
        c, s = divmod(int(flat), 8)
        slot_child[s] = c
        cst[c, :] = np.inf
        cst[:, s] = np.inf
    return slot_child


def _to_int_x86(x):
    """(int)x of a float64 array as x86-64 converts it: INT_MIN for NaN and everything outside [-2^31, 2^31)."""
    with np.errstate(invalid="ignore"):
        return np.where((x >= -2.0**31) & (x < 2.0**31), x, -2.0**31)


def quantise(plo, phi, clo, chi):
    """fill_node's quantisation in float64, vectorised over nodes (plo / phi: (N, 3)) and slots (clo / chi: (N, 8, 3)).
    e is the least exponent with 255 2^e >= ext (frexp, no log2), raised until p + 255 2^e >= hi. Infinite bounds follow
    fill_node too: the extent of an axis with both bounds at the same infinity is NaN and stays NaN through its maxima
    (std::max), and the conversions to int are x86's (a NaN or infinite ext gives e = -100 before the raise)."""
    plo, phi = plo.astype(F32), phi.astype(F32)
    with np.errstate(invalid="ignore", over="ignore"):
        d = phi - plo
        max_ext = np.fmax(F32(0), np.fmax.reduce(d, 1))
        thin = max_ext[:, None] * F32(1.0 / 65536.0)
        ext = np.where(d < thin, thin, d)
        ext = np.where(ext < F32(1e-30), F32(1e-30), ext).astype(F64)
        m, ex = np.frexp(ext)
        e = np.where(np.isfinite(ext), np.where(m <= 255.0 / 256.0, ex - 8, ex - 7), -100)
        e = np.clip(e, -100, 100)
        while True:
            up = (e < 100) & (plo.astype(F64) + 255.0 * np.ldexp(1.0, e) < phi.astype(F64))
            if not up.any():
                break
            e = e + up
        st = np.ldexp(1.0, e)[:, None, :]
        p = plo.astype(F64)[:, None, :]
        lo = _to_int_x86(np.floor((clo.astype(F64) - p) / st))
        hi = _to_int_x86(np.ceil((chi.astype(F64) - p) / st))
    lo, hi = np.clip(lo, 0, 255), np.clip(hi, 0, 255)
    with np.errstate(invalid="ignore"):
        while True:
            dn = (lo > 0) & (p + lo * st > clo)
            if not dn.any():
                break
            lo -= dn
        while True:
            upm = (hi < 255) & (p + hi * st < chi)
            if not upm.any():
                break
            hi += upm
    flat = hi <= lo
    hi = np.where(flat & (hi < 255), lo + 1, hi)
    lo = np.where(flat & ~(hi < 255), hi - 1, lo)
    return (e + 127).astype(U8), lo.astype(U8), hi.astype(U8)


def emit_restated(out):
    """k_plan_level + k_emit_level over the dumped BVH2: the DP forest's children left to right, assign_slots, BFS
    numbering (child_base / tri_base from the level's exclusive scans), quantisation, meta bytes, triangle order."""
    n, ch, dec = out["n"], out["children"].astype(np.int64), out["decision"]
    lo, hi, vals = out["box_lo"], out["box_hi"], out["vals"]
    is_leaf_child = lambda c: c < n or (dec[c, 0] & 3) == 0  # noqa: E731

    def forest(root):
        res = []

        def walk(nd, i):
            d = dec[nd, i]
            l, r = ch[nd - n]
            dl, dr = (d >> 2) & 7, (d >> 5) & 7
            for c, dc in ((l, dl), (r, dr)):
                if (dec[c, dc] & 3) == 2:
                    walk(c, dc)
                else:
                    res.append(c)

        walk(root, 0)
        return res

    def leaf_tris(c):
        res, st = [], [c]
        while st:
            x = st.pop()
            if x < n:
                res.append(int(vals[x]))
            else:
                st += [ch[x - n, 1], ch[x - n, 0]]
        return res

    slots, nodes_meta = [], []
    tri_order = []
    level = [out["root"]]
    node_begin = 0
    while level:
        next_begin = node_begin + len(level)
        child_first, nxt = 0, []
        for root in level:
            kids = [root] if is_leaf_child(root) else forest(root)
            sc = assign_slots(lo[root], hi[root], lo[kids], hi[kids])
            meta = np.zeros(8, U8)
            imask, tri_off = 0, 0
            slot_nodes = np.full(8, -1, np.int64)
            tri_base = len(tri_order)
            for s in range(8):
                if sc[s] < 0:
                    continue
                c = kids[sc[s]]
                slot_nodes[s] = c
                if is_leaf_child(c):
                    t = leaf_tris(c)
                    tri_order += t
                    meta[s] = ({1: 1, 2: 3, 3: 7}[len(t)] << 5) | tri_off
                    tri_off += len(t)
                else:
                    meta[s] = (1 << 5) | (24 + s)
                    imask |= 1 << s
                    nxt.append(c)
            nodes_meta.append((root, imask, next_begin + child_first, tri_base, meta))
            child_first += bin(imask).count("1")
            slots.append(slot_nodes)
        node_begin = next_begin
        level = nxt
    N = len(nodes_meta)
    node = np.zeros(N, NODE)
    roots = np.array([m[0] for m in nodes_meta])
    slots = np.array(slots)
    valid = slots >= 0
    sn = np.where(valid, slots, 0)
    e, qlo, qhi = quantise(lo[roots, :3], hi[roots, :3], lo[sn, :3], hi[sn, :3])
    node["p"] = lo[roots, :3]
    node["e"] = e
    node["imask"] = [m[1] for m in nodes_meta]
    node["child_base"] = [m[2] for m in nodes_meta]
    node["tri_base"] = [m[3] for m in nodes_meta]
    node["meta"] = np.array([m[4] for m in nodes_meta])
    node["qlo"] = np.where(valid[:, :, None], qlo, 0).transpose(0, 2, 1)
    node["qhi"] = np.where(valid[:, :, None], qhi, 0).transpose(0, 2, 1)
    return node.view(U8).reshape(N, 80), np.array(tri_order, U32)


def test_emitted_bvh8_byte_for_byte(dev):
    """The device's BVH8 nodes and leaf triangle order equal emit_restated over its own (checked) BVH2, byte for byte."""
    cases = [(name, tri_verts(s)) for name, s in tree_scenes(dev) if name != "sponza_c2"] + [("chain", chain_soup())] + key_scenes()
    for name, tris in cases:
        for builder, tail in BUILDS[::2]:
            out = dev.build(soup_scene(tris), builder, tail)
            nodes, order = emit_restated(out)
            assert nodes.shape == out["nodes"].shape, (name, builder, nodes.shape, out["nodes"].shape)
            bad = np.nonzero((nodes != out["nodes"]).any(1))[0]
            assert len(bad) == 0, (name, builder, bad[:5], nodes[bad[:1]], out["nodes"][bad[:1]])
            assert np.array_equal(order, out["leaf_flat_ids"]), (name, builder)


# ---- (f) invariants of any BVH8 ----
def check_bvh8(nodes_u8, order, tris, depth):
    """Builder-independent checks of an emitted BVH8 (host or device), decoded in float64: structure, every triangle
    once, 1..3 per leaf slot, depth; each slot's dequantised box holds every vertex below it (conservative) and is
    within one grid step of their bound (tight; two where the flat-box rule applies); p, e, qlo / qhi equal fill_node
    recomputed from the triangle sets, and the slot order is a greedy assign_slots outcome."""
    nd = nodes_u8.view(NODE).reshape(-1)
    N, n = len(nd), len(tris)
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
    # inner children consecutive at child_base in slot order; BFS numbering; every node reached once
    rank = np.cumsum(inner, 1) - inner
    child = np.where(inner, nd["child_base"][:, None].astype(np.int64) + rank, -1)
    kids = child[inner]
    assert sorted(kids.tolist()) == list(range(1, N)), "inner children are not the nodes 1..N-1, once each"
    # triangles: each node's at [tri_base, tri_base + total), every leaf-order slot once
    first = nd["tri_base"][:, None].astype(np.int64) + off
    idx = np.concatenate([first[leaf] + k for k in range(3)])[np.concatenate([cnt[leaf] > k for k in range(3)])]
    assert sorted(idx.tolist()) == list(range(n)), "leaf triangles are not the triangles 0..n-1, once each"
    # depth
    lev = np.zeros(N, np.int64)
    parent = np.full(N, -1)
    parent[kids] = np.nonzero(inner)[0]
    for i in range(1, N):
        assert parent[i] < i
        lev[i] = lev[parent[i]] + 1
    assert lev.max() + 1 == depth
    # true bounds of the triangles under each slot (float32 min / max: what a box of them is), bottom up
    t = tris[order]  # leaf order
    tlo, thi = t.min(1), t.max(1)
    slo = np.full((N, 8, 3), np.inf, F32)
    shi = np.full((N, 8, 3), -np.inf, F32)
    for k in range(3):
        m = leaf & (cnt > k)
        ti = np.where(m, first + k, 0)
        slo = np.where(m[..., None], np.fmin(slo, tlo[ti]), slo)
        shi = np.where(m[..., None], np.fmax(shi, thi[ti]), shi)
    for lv in range(lev.max(), 0, -1):
        nodes_l = np.nonzero(lev == lv)[0]
        p = parent[nodes_l]
        ps = np.argmax(child[p] == nodes_l[:, None], 1)
        slo[p, ps] = slo[nodes_l].min(1)
        shi[p, ps] = shi[nodes_l].max(1)
    nlo, nhi = slo.min(1), shi.max(1)
    # conservative and tight, in float64
    e = nd["e"].astype(np.int64)
    st = np.ldexp(1.0, e - 127)[:, None, :]
    p = nd["p"].astype(F64)[:, None, :]
    qlo = nd["qlo"].transpose(0, 2, 1).astype(F64)
    qhi = nd["qhi"].transpose(0, 2, 1).astype(F64)
    blo, bhi = p + qlo * st, p + qhi * st
    assert (blo[used] <= slo[used]).all() and (bhi[used] >= shi[used]).all(), "a slot's box misses a vertex below it"
    thin = (qhi - qlo == 1)[used]
    slack = np.where(thin, 2.0, 1.0) * np.broadcast_to(st, blo.shape)[used]
    assert (slo[used] - blo[used] < slack).all() and (bhi[used] - shi[used] < slack).all(), "a slot's box is not tight"
    # the quantisation recomputed from the triangle sets
    assert np.array_equal(nd["p"], nlo), "p is not the node box's low corner"
    e2, qlo2, qhi2 = quantise(nlo, nhi, np.where(used[..., None], slo, 0), np.where(used[..., None], shi, 0))
    assert np.array_equal(nd["e"], e2), "e differs from fill_node's"
    assert np.array_equal(np.where(used[..., None], qlo2, 0).transpose(0, 2, 1), nd["qlo"]), "qlo differs from fill_node's"
    assert np.array_equal(np.where(used[..., None], qhi2, 0).transpose(0, 2, 1), nd["qhi"]), "qhi differs from fill_node's"
    # the slot order: a greedy assign_slots outcome (picks in ascending cost, each the minimum of what is left)
    cx = F32(0.5) * (nlo + nhi)
    with np.errstate(invalid="ignore"):  # (empty slots: inf - inf)
        o = F32(0.5) * (slo + shi) - cx[:, None, :]  # (N, child by its slot, 3)
    sgn = np.array([[-1 if s & 4 else 1, -1 if s & 2 else 1, -1 if s & 1 else 1] for s in range(8)], F32)
    cst = (o[:, :, None, 0] * sgn[None, None, :, 0] + o[:, :, None, 1] * sgn[None, None, :, 1]
           + o[:, :, None, 2] * sgn[None, None, :, 2]).astype(F64)  # (N, child, slot)
    own = np.where(used, cst[:, s8, s8], np.inf)
    pick = np.argsort(own, 1, kind="stable")
    left_c, left_s = used.copy(), np.ones((N, 8), bool)
    rows = np.arange(N)
    for k in range(8):
        s = pick[:, k]
        act = used[rows, s]
        avail = np.where(left_c[:, :, None] & left_s[:, None, :], cst, np.inf).reshape(N, 64).min(1)
        assert (~act | (own[rows, s] == avail)).all(), "the slot order is not assign_slots' greedy order"
        left_c[rows[act], s[act]] = False
        left_s[rows[act], s[act]] = False


def test_bvh8_invariants_host_builder(built):
    """check_bvh8 on the host builder's (binned SAH) tree, exported from libcrt_bvh8_hostcheck.so."""
    from helpers import HostCheck

    for name, tris in key_scenes() + [("chain", chain_soup()), ("soup_2049", random_soup(2049, 4))]:
        hc = HostCheck(soup_scene(tris))
        nodes, order, _, _ = hc.export()
        check_bvh8(nodes, order, tris, hc.stats()["depth"])
    from chameleonrt_b200.scenes import cornell_box, sponza_like

    for scene in (cornell_box()[0], sponza_like(spp=1, detail=0.3, tex_size=16)[0]):
        hc = HostCheck(scene)
        nodes, order, _, _ = hc.export()
        check_bvh8(nodes, order, tri_verts(scene), hc.stats()["depth"])


def test_bvh8_invariants_device_builders(dev):
    """check_bvh8 on the device builders' trees (PLOC and LBVH), at every size the build under test affords."""
    cases = [(name, tri_verts(s)) for name, s in tree_scenes(dev)] + [("chain", chain_soup())] + key_scenes()
    for name, tris in cases:
        for builder, tail in BUILDS[::2]:
            out = dev.build(soup_scene(tris), builder, tail)
            check_bvh8(out["nodes"], out["leaf_flat_ids"], tris, out["depth"])


@pytest.mark.gpu
def test_large_builds_on_the_gpu(device):
    """C2-and-up sizes on the H100: a rungholt_like above 1 M triangles and a soup above 2048^2 triangles, so that the
    first PLOC round's scan (and the sort's histogram scan) runs three levels deep. Keys, tree shape and boxes, the
    Karras topology, the DP and the BVH8 invariants (PLOC's topology is restated up to C2 size, above)."""
    for name, scene in big_scenes():
        tris = tri_verts(scene)
        for builder in ("ploc", "lbvh"):
            out = device.build(scene, builder)
            assert out["n"] == len(tris)
            _, _, lo, hi, keys = morton_restated(tris)
            order = np.argsort(keys, kind="stable")
            assert np.array_equal(out["keys"], keys[order]) and np.array_equal(out["vals"], order.astype(U32)), (name, builder)
            check_tree(out, tris, restate_topology=builder == "lbvh")
            check_bvh8(out["nodes"], out["leaf_flat_ids"], tris, out["depth"])


# ---- (g) scene records ----
def adversarial_instanced_scene():
    """Sheared, mirrored (negative determinant), rotated with a 1e4 translation, scaled 1e-3 and 1e3 instances; one
    geometry shared by several meshes and instances; a geometry without uvs, one with no triangles, a zero-area
    triangle; per-geometry materials; and a few thousand one-triangle instances (k_flatten's segment search)."""
    from chameleonrt_b200.scene import DisneyMaterial, Geometry, Instance, Mesh, ParameterizedMesh, Scene, default_obj_light
    from chameleonrt_b200.scenes import sphere

    rng = np.random.default_rng(7)
    sv, si = sphere((0.0, 0.0, 0.0), 1.0, 12, 8)[:2]
    sv = np.asarray(sv, F32)
    shared = Geometry(sv, np.asarray(si, U32), uvs=rng.uniform(-2, 2, (len(sv), 2)).astype(F32))
    no_uv = Geometry(rng.normal(size=(30, 3)).astype(F32), rng.integers(0, 30, (20, 3)).astype(U32))
    zverts = rng.normal(size=(6, 3)).astype(F32)
    zero_area = Geometry(zverts, np.array([[0, 1, 2], [3, 3, 4], [5, 4, 4]], U32))  # two zero-area triangles
    empty = Geometry(np.zeros((3, 3), F32), np.zeros((0, 3), U32))
    one = Geometry(np.array([[0, 0, 0], [0.01, 0, 0], [0, 0.01, 0]], F32), np.array([[0, 1, 2]], U32))
    meshes = [Mesh([shared, no_uv]), Mesh([empty, shared, zero_area]), Mesh([one])]
    pms = [ParameterizedMesh(0, [0, 1]), ParameterizedMesh(1, [2, 3, 1]), ParameterizedMesh(2, [3])]

    def rot(ax, ang):
        c, s = np.cos(ang), np.sin(ang)
        m = np.eye(4)
        i, j = [(1, 2), (0, 2), (0, 1)][ax]
        m[i, i], m[i, j], m[j, i], m[j, j] = c, -s, s, c
        return m

    xf = []
    shear = np.eye(4)
    shear[0, 1], shear[2, 0] = 0.7, -0.4
    xf.append((shear, 0))
    mirror = np.diag([-1.0, 1.0, 1.0, 1.0])
    mirror[:3, 3] = (3, 0, 0)
    xf.append((mirror, 1))
    r = rot(1, 0.7) @ rot(0, 0.3)
    r[:3, 3] = (1e4, -2e4, 5e3)
    xf.append((r, 0))
    xf.append((np.diag([1e-3, 1e-3, 1e-3, 1.0]), 1))
    xf.append((np.diag([1e3, 2e3, 1e3, 1.0]), 0))
    instances = [Instance(m.astype(F32), pm) for m, pm in xf]
    for k in range(3000):
        m = np.eye(4)
        m[:3, 3] = rng.uniform(-5, 5, 3)
        instances.append(Instance(m.astype(F32), 2))
    mats = [DisneyMaterial(base_color=(0.2 * i, 0.5, 0.5)) for i in range(4)]
    return Scene(meshes=meshes, parameterized_meshes=pms, instances=instances, materials=mats, lights=[default_obj_light()])


def test_scene_records_equal_the_hosts(dev):
    """The device's packed triangles ({v0, flat id}, e1, e2) and shading records, mapped to flattened order through
    leaf_flat_ids, equal the host's records for the same flat id bit for bit (uint32: NaN normals of zero-area
    triangles included), on adversarial_instanced_scene and on the material test scene."""
    from helpers import HostCheck, synthetic_material_scene

    for k, scene in enumerate((adversarial_instanced_scene(), synthetic_material_scene()[0])):
        hc = HostCheck(scene)
        _, h_order, h_tris, h_shade = hc.export()
        for builder in ("ploc", "lbvh"):
            out = dev.build(scene, builder)
            n = out["n"]
            assert n == len(h_order)
            d_flat = out["leaf_flat_ids"]
            assert np.array_equal(out["tris"][:, 3].view(U32), d_flat)
            assert np.array_equal(out["shade"][:, 11].view(U32), d_flat)
            hpos = np.empty(n, np.int64)
            hpos[h_order] = np.arange(n)
            want_t, want_s = h_tris[hpos[d_flat]], h_shade[hpos[d_flat]]
            assert np.array_equal(out["tris"].view(U32), want_t.view(U32)), builder
            assert np.array_equal(out["shade"].view(U32), want_s.view(U32)), builder
            assert k or np.isnan(want_s[:, :3]).any(), "the scene was meant to hold zero-area triangles"
