"""The shading arithmetic of k_shade (chameleonrt_b200/csrc/shade_math.cuh) as nvcc compiles it for sm_90a, function
by function.

libcrt_shade_devcheck.so is shade_math.cuh built with the product's NVFLAGS, one CUDA thread per input;
libcrt_shade_hostcheck.so is the same source built by g++. Both export the batched shadekat_*_n entry points, so every
check below is one function run twice: on the host build (``-m "not gpu"``, where every bit-exact claim holds exactly and
glibc's accuracy is measured) and on the device build (``-m gpu``, on an H100). The expected values come from the
reference's own tables (tests/golden/ref_embree_frames.npz), from the reference's functions where oracle/_ref was built,
from the host build, and from numpy restatements: float32 operation by operation where the claim is bit-exactness,
float64 where it is accuracy.

  * bit-exact: rng, ortho_basis, the quad light, the texture filter and the textured parameters of unpack_material
    (uv past 2^31 texels included: DESIGN.md §4, texel index conversion), schlick_weight;
  * against float64: sinf / cosf / powf / logf / atan2f / acosf over the arguments the shading code passes them,
    schlick_weight (2 ulp), float_to_srgb8 (round-half-up of the exact curve), the miss shader's checker;
  * close to the host build: BSDF value and pdf (bit-exact wherever logf agrees), sampled directions (bit-exact wherever
    sinf / cosf / powf / logf agree, within a bound derived from their accuracy elsewhere), lobe choice and rng state.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from ref_cases import kat_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "chameleonrt_b200", "csrc")
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libcrt_embree.so")
F32, U32 = np.float32, np.uint32

# Bounds on the error in ulp of each transcendental over the argument ranges of transcendental_cases (DESIGN.md §4),
# against float64. Measured maxima: on an H100 80GB HBM3 (700 W power limit, CUDA 12.9, no --use_fast_math) sinf 1.45,
# cosf 1.46, powf 0.90, logf 0.59, atan2f 1.95, acosf 1.34; in glibc (x86-64) sinf 0.56, cosf 0.56, powf 0.50,
# logf 0.50, atan2f 1.39, acosf 0.86. The BSDF, sampling, sRGB and miss-shader bounds below are derived from these.
DEVICE_ULP = {"sinf": 1.5, "cosf": 1.5, "powf": 1.0, "logf": 1.0, "atan2f": 2.0, "acosf": 1.5}
HOST_ULP = {"sinf": 1.0, "cosf": 1.0, "powf": 1.0, "logf": 1.0, "atan2f": 1.5, "acosf": 1.0}
# m^2 * m^2 * m against float64 m^5 over every float m in [0, 1] (shade_math.cuh: schlick_weight)
SCHLICK_ULP = 3.0
KAT_MATH = {"sinf": 0, "cosf": 1, "powf": 2, "logf": 3, "atan2f": 4, "acosf": 5}


# ---- the two builds ----
class Kat:
    """The shadekat_*_n entry points of one build, on numpy arrays."""

    def __init__(self, path, name):
        self.name = name
        self.lib = lib = C.CDLL(path)
        vp, i32, u32 = C.c_void_p, C.c_int, C.c_uint32
        sig = dict(rng_n=[vp, vp, i32, i32, vp, vp], lcg_n=[vp, i32, vp], disney_eval_n=[vp, vp, vp, vp, i32, vp],
                   disney_sample_n=[vp, vp, vp, vp, i32, vp], light_n=[vp, vp, vp, vp, i32, vp],
                   texture_n=[vp, i32, i32, i32, vp, i32, vp],
                   unpack_material_n=[vp, i32, u32, vp, i32, vp, i32, vp, i32, vp], miss_n=[vp, i32, vp],
                   ortho_basis_n=[vp, i32, vp], srgb8_n=[vp, i32, vp], schlick_n=[vp, i32, vp],
                   math_n=[i32, vp, vp, i32, vp])
        for k, a in sig.items():
            f = getattr(lib, "shadekat_" + k)
            f.argtypes, f.restype = a, C.c_int

    def _call(self, fn, *args):
        rc = getattr(self.lib, "shadekat_" + fn)(*[a.ctypes.data if isinstance(a, np.ndarray) else a for a in args])
        assert rc == 0, f"{self.name}: shadekat_{fn} failed with error {rc}"

    def rng(self, pix, frame, k):
        pix, frame = np.ascontiguousarray(pix, U32), np.ascontiguousarray(frame, U32)
        st, fl = np.zeros((len(pix), k), U32), np.zeros((len(pix), k), F32)
        self._call("rng_n", pix, frame, len(pix), k, st, fl)
        return st, fl

    def lcg(self, states):
        st = np.array(states, U32)
        fl = np.zeros(len(st), F32)
        self._call("lcg_n", st, len(st), fl)
        return st, fl

    def eval(self, mats, n, wo, wi):
        arrs = [np.ascontiguousarray(a, F32) for a in (mats, n, wo, wi)]
        out = np.zeros((len(arrs[1]), 4), F32)
        self._call("disney_eval_n", *arrs, len(arrs[1]), out)
        return out

    def sample(self, mats, n, wo, rng):
        arrs = [np.ascontiguousarray(a, F32) for a in (mats, n, wo)]
        st = np.array(rng, U32)
        out = np.zeros((len(st), 7), F32)
        self._call("disney_sample_n", *arrs, st, len(st), out)
        return out, st

    def light(self, light, s2, orig, d):
        arrs = [np.ascontiguousarray(a, F32) for a in (light, s2, orig, d)]
        out = np.zeros((len(arrs[1]), 9), F32)
        self._call("light_n", *arrs, len(arrs[1]), out)
        return out

    def texture(self, img, uv):
        img, uv = np.ascontiguousarray(img, np.uint8), np.ascontiguousarray(uv, F32)
        out = np.zeros((len(uv), 4), F32)
        self._call("texture_n", img, img.shape[1], img.shape[0], img.shape[2], uv, len(uv), out)
        return out

    def unpack(self, materials, mid, texels, tex, uv):
        m, t, d = np.ascontiguousarray(materials, F32), np.ascontiguousarray(texels, U32), np.ascontiguousarray(tex, np.int32)
        uv = np.ascontiguousarray(uv, F32)
        out = np.zeros((len(uv), 14), F32)
        self._call("unpack_material_n", m, len(m), mid, t, len(t), d, len(d), uv, len(uv), out)
        return out

    def _map(self, fn, x, width, dtype=F32):
        x = np.ascontiguousarray(x, F32)
        out = np.zeros((len(x), width) if width > 1 else len(x), dtype)
        self._call(fn, x, len(x), out)
        return out

    def miss(self, dirs):
        return self._map("miss_n", dirs, 3)

    def ortho(self, n):
        return self._map("ortho_basis_n", n, 6)

    def srgb8(self, x):
        return self._map("srgb8_n", x, 1, np.uint8)

    def schlick(self, x):
        return self._map("schlick_n", x, 1)

    def math(self, fn, x, y=None):
        x = np.ascontiguousarray(x, F32)
        y = None if y is None else np.ascontiguousarray(np.broadcast_to(np.asarray(y, F32), x.shape))
        out = np.zeros(len(x), F32)
        self._call("math_n", KAT_MATH[fn], x, y if y is not None else None, len(x), out)
        return out


@pytest.fixture(scope="module")
def host(built):
    return Kat(os.path.join(CSRC, "libcrt_shade_hostcheck.so"), "host")


@pytest.fixture(scope="module")
def device(built):
    path = os.path.join(CSRC, "libcrt_shade_devcheck.so")
    if not os.path.exists(path):  # (a tree built before the device check library existed)
        subprocess.check_call(["make", "-s", "-C", CSRC, "libcrt_shade_devcheck.so"])
    return Kat(path, "device")


@pytest.fixture(params=[pytest.param("host"), pytest.param("device", marks=pytest.mark.gpu)], scope="module")
def kat(request):
    """The build under test: the host build without a GPU, the device build with ``-m gpu``."""
    return request.getfixturevalue(request.param)


@pytest.fixture(scope="module")
def tables():
    return np.load(os.path.join(ROOT, "tests", "golden", "ref_embree_frames.npz"))


@pytest.fixture(scope="module")
def refispc():
    """The reference's own functions (refispc_kat_*), where oracle/_ref was built; None elsewhere."""
    if not os.path.exists(REF_LIB):
        return None
    lib = C.CDLL(REF_LIB)
    vp = C.c_void_p
    lib.refispc_kat_light.argtypes = [vp] * 5
    lib.refispc_kat_texture.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, C.c_int, vp]
    lib.refispc_kat_ortho_basis.argtypes = [vp, vp]
    return lib


# ---- helpers ----
def _bits(a):
    return np.ascontiguousarray(a, F32).view(U32)


def _same(got, want):
    """Bit for bit, NaN payloads aside: NaN in the same places."""
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    nan = np.isnan(want)
    return np.array_equal(np.isnan(got), nan) and np.array_equal(_bits(got)[~nan], _bits(want)[~nan])


def _assert_same(got, want, what):
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    if not _same(got, want):
        bad = np.nonzero(~((_bits(got) == _bits(want)) | (np.isnan(got) & np.isnan(want))).reshape(len(got), -1).all(1))[0]
        raise AssertionError(f"{what}: {len(bad)} of {len(got)} inputs differ, first at {bad[:5].tolist()}: "
                             f"{got[bad[:3]].tolist()} != {want[bad[:3]].tolist()}")


CHUNK = 1 << 24  # inputs per call: 64 MB of float32, so that sweeps of 2^30 floats keep host memory small


class FloatRange:
    """Every `stride`-th float32 in [lo, hi), for 0 <= lo < hi or lo < hi <= 0, generated CHUNK at a time."""

    def __init__(self, lo, hi, stride=1):
        self.neg = lo < 0
        lo_b, hi_b = (int(np.array([abs(v)], F32).view(U32)[0]) for v in (lo, hi))
        self.a, self.b = (hi_b + 1, lo_b + 1) if self.neg else (lo_b, hi_b)
        self.stride = stride

    def __len__(self):
        return (self.b - self.a + self.stride - 1) // self.stride

    def chunks(self):
        step = CHUNK * self.stride
        for s in range(self.a, self.b, step):
            v = np.arange(s, min(s + step, self.b), self.stride, dtype=np.uint32).view(F32)
            yield np.negative(v) if self.neg else v

    def array(self):
        return np.concatenate(list(self.chunks()))


def _chunks(x):
    for i in range(0, len(x), CHUNK):
        yield x[i:i + CHUNK]


def ulp_error(got, exact):
    """|got - exact| in units of the float32 spacing at `exact` (float64)."""
    exact = np.asarray(exact, np.float64)
    _, e = np.frexp(np.abs(exact))
    ulp = np.ldexp(1.0, np.maximum(e - 24, -149))
    return np.abs(np.asarray(got, np.float64) - exact) / ulp


def ulp_distance(a, b):
    """Number of float32 values between a and b (0 = the same float; +0 and -0 are 0 apart)."""
    def ordered(x):
        i = _bits(x).astype(np.int64)
        return np.where(i >= 0x80000000, 0x80000000 - i, i)
    return np.abs(ordered(a) - ordered(b))


def neighbours(x, k=2):
    """x and its k float32 neighbours on each side."""
    x = np.atleast_1d(np.asarray(x, F32))
    out = [x]
    lo, hi = x.copy(), x.copy()
    for _ in range(k):
        lo, hi = np.nextafter(lo, F32(-np.inf)), np.nextafter(hi, F32(np.inf))
        out += [lo, hi]
    return np.concatenate(out).astype(F32)


# ---- the rng ----
LCG_A, LCG_C = 1664525, 1013904223


def np_get_rng(pix, frame):
    m32 = 0xFFFFFFFF

    def mix(h, k):
        k = (k * 0xCC9E2D51) & m32
        k = ((k << 15) | (k >> 17)) & m32
        k = (k * 0x1B873593) & m32
        h ^= k
        return ((((h << 13) | (h >> 19)) & m32) * 5 + 0xE6546B64) & m32

    h = mix(mix(np.zeros_like(pix, np.uint64), pix.astype(np.uint64)), frame.astype(np.uint64))
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & m32
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & m32
    h ^= h >> 16
    return h.astype(U32)


def np_lcg(states):
    """(next state, its float): round-to-nearest u32 -> f32, times 2^-32."""
    s = ((states.astype(np.uint64) * LCG_A + LCG_C) & 0xFFFFFFFF).astype(U32)
    return s, s.astype(F32) * F32(2.0 ** -32)


def states_before(targets):
    """The states whose next state is `targets`."""
    inv = pow(LCG_A, -1, 1 << 32)
    return ((np.asarray(targets, np.uint64) - LCG_C) % (1 << 32) * inv % (1 << 32)).astype(U32)


# draws that round to exactly 1.0f (the clamp of the lobe choice), the largest below 1, and 0
EDGE_DRAWS = np.array([2**32 - 1, 2**32 - 100, 2**32 - 128, 2**32 - 129, 2**32 - 256, 0, 1], np.uint64)


def test_rng(kat, tables):
    k = kat_inputs()
    keys = k["rng_keys"]
    st, fl = kat.rng(keys[:, 0], keys[:, 1], 16)
    assert np.array_equal(st, tables["kat.rng_states"]) and _same(fl, tables["kat.rng_floats"])
    rs = np.random.default_rng(1)
    pix, frame = rs.integers(0, 2**32, 100_000, dtype=np.uint64).astype(U32), rs.integers(0, 2**32, 100_000, dtype=np.uint64).astype(U32)
    st, fl = kat.rng(pix, frame, 4)
    want = np_get_rng(pix, frame)
    for j in range(4):
        want, f = np_lcg(want)
        assert np.array_equal(st[:, j], want) and _same(fl[:, j], f)
    prev = states_before(EDGE_DRAWS)
    st, fl = kat.lcg(prev)
    assert np.array_equal(st, EDGE_DRAWS.astype(U32))
    assert fl.tolist() == [1.0, 1.0, 1.0, 1.0 - 2.0**-24, 1.0 - 2.0**-24, 0.0, 2.0**-32]


# ---- ortho_basis ----
def np_ortho_basis(n):
    n = n.astype(F32)
    vy = np.zeros_like(n)
    inside = lambda c: (c < F32(0.6)) & (c > F32(-0.6))  # noqa: E731
    bx, by, bz = inside(n[:, 0]), inside(n[:, 1]), inside(n[:, 2])
    vy[:, 0] = np.where(bx | (~by & ~bz), 1, 0)
    vy[:, 1] = np.where(~bx & by, 1, 0)
    vy[:, 2] = np.where(~bx & ~by & bz, 1, 0)

    def cross(a, b):
        return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                         a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)

    def normalize(v):
        c = F32(1) / np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])
        return v * c[:, None]

    vx = normalize(cross(vy, n))
    return np.concatenate([vx, normalize(cross(n, vx))], 1).astype(F32)


def edge_normals():
    """The axes, and normals with a component on or next to +-0.6f (each branch boundary of ortho_basis)."""
    out = [np.eye(3, dtype=F32), -np.eye(3, dtype=F32)]
    for c in neighbours([0.6, -0.6], 2):
        rest = np.sqrt(max(0.0, 1.0 - float(c) ** 2))
        for axis in range(3):
            for other in ([rest, 0.0], [0.0, rest], [rest * 0.6, rest * 0.8], [-rest, 0.0]):
                v = np.insert(np.array(other, np.float64), axis, float(c)).astype(F32)
                out.append(v[None])
    # the last branch: every component outside (-0.6, 0.6) is impossible for a unit vector; unnormalised normals reach it
    out.append(np.array([[0.6, 0.6, 0.6], [-0.7, 0.7, -0.7], [0.6, -0.6, 0.6]], F32))
    return np.concatenate(out).astype(F32)


def test_ortho_basis(kat, tables, refispc):
    k = kat_inputs()
    _assert_same(kat.ortho(k["dirs"]), tables["kat.ortho_basis"], "ortho_basis vs the reference's table")
    rs = np.random.default_rng(2)
    n = rs.normal(size=(100_000, 3)).astype(F32)
    n = np.concatenate([edge_normals(), (n / np.linalg.norm(n, axis=1, keepdims=True)).astype(F32)])
    got = kat.ortho(n)
    _assert_same(got, np_ortho_basis(n), "ortho_basis vs its float32 restatement")
    if refispc is not None:
        e = edge_normals()
        want = np.zeros((len(e), 6), F32)
        for i in range(len(e)):
            refispc.refispc_kat_ortho_basis(np.ascontiguousarray(e[i]).ctypes.data, want[i].ctypes.data)
        _assert_same(got[:len(e)], want, "ortho_basis vs the reference on the branch boundaries")


# ---- the quad light ----
def light_edge_cases(light):
    """(s2, orig, dir) rows: directions parallel to the light (denom == 0), hits exactly on its edges (|dot| == width /
    height: a miss), on and next to n_dot_w == kEpsilon (the pdf's cut-off)."""
    pos, w, h = light[4:7], light[15], light[19]
    s2, orig, dirs = [], [], []
    up = np.array([0, 1, 0], F32)
    for o in ([w, 0, 0], [-w, 0, 0], [0, 0, h], [0, 0, -h], [np.nextafter(w, F32(0)), 0, 0], [0, 0, np.nextafter(h, F32(0))],
              [np.nextafter(w, F32(1)), 0, 0], [0.1, 0, 0.2]):
        o = np.array([pos[0] + F32(o[0]), 0, pos[2] + F32(o[2])], F32)
        for d in (up, np.array([1, 0, 0], F32), np.array([0, 0, -1], F32), np.array([0.6, 0, 0.8], F32)):
            s2.append([0.25, 0.75]), orig.append(o), dirs.append(d)
    for y in neighbours([1e-4], 2):
        for d in ([0.3, y, 0.4], [0.0, y, 0.0], [-0.5, y, 0.1]):
            s2.append([0.5, 0.5]), orig.append([0.1, 0.3, -0.2]), dirs.append(d)
    for s in ([0, 0], [1, 1], [-1, 1], [0.5, 0.5]):
        s2.append(s), orig.append([0.1, 0.3, -0.2]), dirs.append([0, 1, 0])
    return np.array(s2, F32), np.array(orig, F32), np.array(dirs, F32)


def test_quad_light(kat, host, tables, refispc):
    k = kat_inputs()
    ns, nd = len(k["light_s"]), len(k["dirs"])
    s2 = np.repeat(k["light_s"], nd, axis=0)
    dirs = np.tile(k["dirs"], (ns, 1))
    got = kat.light(k["light"], s2, np.tile(k["light_orig"], (ns * nd, 1)), dirs)
    _assert_same(got, tables["kat.light"].reshape(-1, 9), "quad light vs the reference's table")
    es2, eorig, edir = light_edge_cases(k["light"])
    rs = np.random.default_rng(3)
    m = 100_000
    rd = rs.normal(size=(m, 3)).astype(F32)
    rd /= np.linalg.norm(rd, axis=1, keepdims=True)
    s2 = np.concatenate([es2, rs.random((m, 2)).astype(F32)])
    orig = np.concatenate([eorig, (rs.random((m, 3)) * 4 - 2).astype(F32)])
    dirs = np.concatenate([edir, rd.astype(F32)])
    got = kat.light(k["light"], s2, orig, dirs)
    _assert_same(got, host.light(k["light"], s2, orig, dirs), "quad light vs the host build")
    ne = len(es2)
    # what the edge list was made for: hits exactly on an edge miss, just inside hit, parallel rays miss; the pdf's
    # cut-off n_dot_w < kEpsilon keeps kEpsilon itself
    hit = got[:32, 4].reshape(8, 4)
    assert hit[:, 0].tolist() == [0, 0, 0, 0, 1, 1, 0, 1] and (hit[:, 1:3] == 0).all()
    eps = got[32:47, 3].reshape(5, 3)  # n_dot_w = 1e-4f, its lower and upper neighbours
    assert (eps[[0, 2, 4]] > 0).all() and (eps[[1, 3]] == 0).all()
    if refispc is not None:
        want = np.zeros((ne, 9), F32)
        for i in range(ne):
            refispc.refispc_kat_light(k["light"].ctypes.data, np.ascontiguousarray(s2[i]).ctypes.data,
                                      np.ascontiguousarray(orig[i]).ctypes.data, np.ascontiguousarray(dirs[i]).ctypes.data,
                                      want[i].ctypes.data)
        _assert_same(got[:ne], want, "quad light vs the reference on the edge cases")


# ---- the texture filter ----
BYTE_TO_UNIT = np.arange(256, dtype=F32) / F32(255)


def x86_int(x):
    """(int)x as x86-64 converts it: truncation, INT_MIN for NaN and outside [-2^31, 2^31)."""
    x = np.asarray(x, F32)
    ok = (x >= F32(-2.0**31)) & (x < F32(2.0**31))
    return np.where(ok, np.trunc(np.where(ok, x, 0)).astype(np.int64), -(2**31))


def modi(a, b):
    r = np.fmod(a, b)  # C's remainder: the sign of the dividend (a - (a / b) * b)
    return np.where(r < 0, r + b, r)


def np_texture(img, uv):
    """texture2d.ih's bilinear filter with wrap addressing, float32 operation by operation (shade_math.cuh:
    texel_quad / bilinear_channel): channels (n, 4), missing channels 0."""
    h, w, ch = img.shape
    rgba = np.zeros((h * w, 4), np.uint8)
    rgba[:, :ch] = img.reshape(h * w, ch)
    ux = uv[:, 0] * F32(w) - F32(0.5)
    uy = uv[:, 1] * F32(h) - F32(0.5)
    with np.errstate(invalid="ignore"):
        tx, ty = ux - np.floor(ux), uy - np.floor(uy)
        x0, y0 = modi(x86_int(ux), w), modi(x86_int(uy), h)
        x1, y1 = modi(x86_int(ux + F32(1)), w), modi(x86_int(uy + F32(1)), h)
        s = [BYTE_TO_UNIT[rgba[y * w + x]] for y, x in ((y0, x0), (y0, x1), (y1, x0), (y1, x1))]
        w00, w10 = (F32(1) - tx)[:, None], tx[:, None]
        one_ty, tyc = (F32(1) - ty)[:, None], ty[:, None]
        return (((s[0] * w00 * one_ty + s[1] * w10 * one_ty) + s[2] * w00 * tyc) + s[3] * w10 * tyc).astype(F32)


def texture_uvs(w, h):
    """0, -0, 1, texel centres and their neighbours, small negatives, 1e3, uv*size just below and above 2^31 (where the
    texel index conversion saturates on the device), NaN and +-inf; paired in both coordinates."""
    one = []
    for size in (w, h):
        centres = (np.arange(size, dtype=np.float64) + 0.5) / size
        big = [(2.0**31 + 0.5) / size, (2.0**31 - 64) / size, 2.0**31 / size, 2.0**32 / size, 2.0**40 / size]
        one.append(np.concatenate([
            np.array([0.0, -0.0, 1.0, -1e-3, -0.3, -1e-7, 1e3, -1e3, 0.5, np.nan, np.inf, -np.inf], F32),
            neighbours(centres, 1), neighbours(np.array(big), 3), -neighbours(np.array(big[:2]), 2)]).astype(F32))
    ux, uy = one
    k = min(len(ux), len(uy))
    pairs = [np.stack([ux, np.full_like(ux, F32(0.3))], 1), np.stack([np.full_like(uy, F32(0.7)), uy], 1),
             np.stack([ux[:k], uy[::-1][:k]], 1)]
    return np.concatenate(pairs).astype(F32)


TEXTURE_SHAPES = [(1, 1), (1, 4), (4, 1), (3, 5), (5, 3), (2, 7)]  # (height, width)


def test_texture_filter(kat, host, tables, refispc):
    k = kat_inputs()
    for ch in (1, 3, 4):
        _assert_same(kat.texture(k[f"tex{ch}"], k["uv"]), tables[f"kat.texture{ch}"], f"texture ({ch} channels) vs table")
    rs = np.random.default_rng(4)
    for h, w in TEXTURE_SHAPES:
        for ch in (1, 3, 4):
            img = rs.integers(0, 256, size=(h, w, ch), dtype=np.uint8)
            uv = texture_uvs(w, h)
            got = kat.texture(img, uv)
            _assert_same(got, np_texture(img, uv), f"texture {w}x{h}x{ch} vs its float32 restatement")
            nan = np.isnan(uv).any(1) | np.isinf(uv).any(1)
            assert np.isnan(got[nan]).all()
            if refispc is not None:
                want = np.zeros((len(uv), 4), F32)
                refispc.refispc_kat_texture(img.ctypes.data, w, h, ch, uv.ctypes.data, len(uv), want.ctypes.data)
                _assert_same(got, want, f"texture {w}x{h}x{ch} vs the reference")
    img = rs.integers(0, 256, size=(5, 3, 4), dtype=np.uint8)
    uv = (rs.random((100_000, 2)) * 8 - 4).astype(F32)
    _assert_same(kat.texture(img, uv), host.texture(img, uv), "texture vs the host build")


def test_texture_past_2_31_texels_reads_the_hosts_column(kat):
    """uv.x * width >= 2^31 on a 1x4 texture: the texel index is INT_MIN mod 4 = column 0 (the x86 conversion the
    reference and every host build use), not the device's saturated INT_MAX mod 4 = column 3."""
    img = np.zeros((1, 4, 1), np.uint8)
    img[0, :, 0] = [10, 60, 120, 250]
    uv = np.array([[2.0**31 / 4, 0.5], [2.0**33, 0.5], [1e20, 0.5]], F32)
    got = kat.texture(img, uv)[:, 0]
    assert (got == BYTE_TO_UNIT[10]).all(), f"read {got.tolist()}, the texel of column 0 is {BYTE_TO_UNIT[10]}"


def test_unpack_material_textured_parameters(kat, host):
    """unpack_material<false>: a textured base colour and textured scalar parameters (two textures, every channel, the
    parameter loop's texel reuse), bit-exact against the restated filter, at the texture uvs above."""
    rs = np.random.default_rng(5)
    imgs = [rs.integers(0, 256, size=(3, 4, 3), dtype=np.uint8), rs.integers(0, 256, size=(2, 7, 4), dtype=np.uint8)]
    words, desc, off = [], [], 0
    for img in imgs:
        h, w, ch = img.shape
        rgba = np.zeros((h * w, 4), np.uint32)
        rgba[:, :ch] = img.reshape(h * w, ch)
        words.append(rgba[:, 0] | (rgba[:, 1] << 8) | (rgba[:, 2] << 16) | (rgba[:, 3] << 24))
        desc.append([off, w, h, 0])
        off += h * w
    texels, tex = np.concatenate(words).astype(U32), np.array(desc, np.int32)

    def word(tex_id, channel=0):
        return np.array([0x80000000 | (channel << 29) | tex_id], U32).view(F32)[0]

    plain = np.array([0.7, 0.5, 0.3, 0.1, 0.5, 0.4, 0.2, 0.0, 0.3, 0.6, 0.2, 0.9, 1.45, 0.0, 0, 0], F32)
    textured = plain.copy()
    textured[0] = word(0)
    # metallic: tex 1 ch 2; roughness: tex 1 ch 1; anisotropy: tex 0 ch 0 (a switch of texture); sheen: tex 1 ch 3;
    # specular_transmission: tex 1 ch 0
    for idx, (t, c) in {3: (1, 2), 5: (1, 1), 7: (0, 0), 8: (1, 3), 13: (1, 0)}.items():
        textured[idx] = word(t, c)
    materials = np.stack([plain, textured])
    uv = np.concatenate([texture_uvs(4, 3), texture_uvs(7, 2), (rs.random((20_000, 2)) * 6 - 3).astype(F32)])
    got = kat.unpack(materials, 1, texels, tex, uv)
    f0, f1 = np_texture(imgs[0], uv), np_texture(imgs[1], uv)
    want = np.tile(plain[:14], (len(uv), 1))
    want[:, 0:3] = f0[:, 0:3]
    for idx, src in {3: f1[:, 2], 5: f1[:, 1], 7: f0[:, 0], 8: f1[:, 3], 13: f1[:, 0]}.items():
        want[:, idx] = src
    _assert_same(got, want, "textured unpack_material vs the restated filter")
    _assert_same(kat.unpack(materials, 0, texels, tex, uv[:100]), np.tile(plain[:14], (100, 1)), "untextured material")
    _assert_same(got, host.unpack(materials, 1, texels, tex, uv), "textured unpack_material vs the host build")


# ---- the transcendentals against float64 ----
def _unit_dirs(m, seed):
    d = np.random.default_rng(seed).normal(size=(m, 3))
    return (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(F32)


def transcendental_cases(exhaustive):
    """(function, range name, inputs, float64 of the exact result) per argument range the shading code uses. `inputs` is
    a FloatRange (y fixed or absent) or an (x, y) pair of arrays. Ranges of at most 2^30 floats are swept exhaustively
    on the GPU (`exhaustive`); [0, 2pi) holds 1.09e9 floats and is swept at stride 2 there. The host build is swept at a
    stride throughout."""
    s = 1 if exhaustive else 61
    big = 2 if exhaustive else 127
    two_pi = F32(2) * F32(np.pi)
    cases = []
    for fn, f64 in (("sinf", np.sin), ("cosf", np.cos)):
        # angle = 2*pi*sx in [0, 2pi) (phi of the GTR lobes) and the concentric map's theta in [-pi/4, 3pi/4]
        cases.append((fn, "[0, 2pi)", (FloatRange(0.0, two_pi, big), None), f64))
        cases.append((fn, "[-pi/4, 0)", (FloatRange(-np.pi / 4, 0.0, big), None), f64))
    rs = np.random.default_rng(6)
    m = 4_000_000 if exhaustive else 200_000
    a2 = np.exp(rs.uniform(np.log(1e-6), np.log(1e-2), m)).astype(F32)  # alpha^2 of GTR1 (clearcoat alpha 0.001 .. 0.1)
    e = (F32(1) - rs.random(m).astype(F32)).astype(F32)  # 1 - sy
    cases.append(("powf", "alpha^2 in [1e-6, 1e-2], y = 1 - s", (a2, e), np.power))
    inv24 = F32(1) / F32(2.4)
    cases.append(("powf", "(0.0031308, 1), y = 1/2.4",
                  (FloatRange(np.nextafter(F32(0.0031308), F32(1)), 1.0, s), inv24), np.power))
    cases.append(("logf", "alpha^2 in [1e-6, 1e-2]", (FloatRange(1e-6, 1e-2, s), None), np.log))
    cases.append(("acosf", "[0, 1]", (FloatRange(0.0, np.nextafter(F32(1), F32(2)), s), None), np.arccos))
    cases.append(("acosf", "[-1, 0)", (FloatRange(-1.0, 0.0, s), None), np.arccos))
    d = _unit_dirs(m, 7)
    cases.append(("atan2f", "unit directions (x, -z)", (d[:, 0], -d[:, 2]), np.arctan2))
    return cases


def _case_chunks(inputs):
    x, y = inputs
    if isinstance(x, FloatRange):
        for xc in x.chunks():
            yield xc, (None if y is None else np.full(len(xc), y, F32))
    else:
        for i in range(0, len(x), CHUNK):
            yield x[i:i + CHUNK], y[i:i + CHUNK]


def measure_transcendentals(kat, exhaustive):
    worst = {}
    for fn, rng, inputs, f64 in transcendental_cases(exhaustive):
        w, at, count = 0.0, None, 0
        for xc, yc in _case_chunks(inputs):
            got = kat.math(fn, xc, yc)
            x64 = xc.astype(np.float64)
            exact = f64(x64) if yc is None else f64(x64, yc.astype(np.float64))
            err = ulp_error(got, exact)
            j = int(np.argmax(err))
            if err[j] > w:
                w, at = float(err[j]), (float(xc[j]), None if yc is None else float(yc[j]))
            count += len(xc)
        worst[(fn, rng)] = (w, at, count)
    return worst


def test_transcendentals_against_float64(kat, record_property):
    bound = DEVICE_ULP if kat.name == "device" else HOST_ULP
    worst = measure_transcendentals(kat, exhaustive=kat.name == "device")
    lines = []
    for (fn, rng), (w, at, n) in worst.items():
        lines.append(f"{kat.name} {fn:7s} {rng:36s} n={n:>11,d} max {w:.3f} ulp at {at}")
        record_property(f"{fn} {rng}", w)
    print("\n" + "\n".join(lines))
    for (fn, rng), (w, at, _) in worst.items():
        assert w <= bound[fn], f"{kat.name} {fn} on {rng}: {w:.3f} ulp at {at} (bound {bound[fn]})"


# ---- schlick_weight ----
def test_schlick_weight(kat, host):
    """m^2 * m^2 * m with m = saturate(1 - cos): within SCHLICK_ULP of float64 m^5 for every cos in [0, 1] (the GPU: every
    float; the host: a stride), and bit-exact with the host build."""
    stride = 1 if kat.name == "device" else 31
    worst = 0.0
    for xc in FloatRange(0.0, np.nextafter(F32(1), F32(2)), stride).chunks():
        got = kat.schlick(xc)
        m = np.clip(F32(1) - xc, 0, 1).astype(np.float64)
        worst = max(worst, float(ulp_error(got, m ** 5).max()))
        if kat is not host:
            assert np.array_equal(_bits(got), _bits(host.schlick(xc)))
    edge = np.array([-0.0, -1.0, -1e-30, 2.0, np.inf, -np.inf, np.nan], F32)
    assert _same(kat.schlick(edge), host.schlick(edge))
    assert kat.schlick(edge)[:6].tolist() == [1.0, 1.0, 1.0, 0.0, 0.0, 1.0]
    print(f"\n{kat.name} schlick_weight: max {worst:.3f} ulp from float64 m^5")
    assert worst <= SCHLICK_ULP


# ---- float_to_srgb8 ----
def srgb_delta(powf_ulp):
    """How far from an integer the exact s*255 + 0.5 may be for float_to_srgb8 to still be held to round-half-up: powf
    within `powf_ulp` ulp of a result < 1 (2^-24 each), then 1.055f * p, - 0.055f, * 255.f, + 0.5f each rounded (half an
    ulp of results < 1.06, < 1, < 256, < 256)."""
    return 255.0 * (1.055 * powf_ulp * 2.0**-24 + 2.0**-24 + 2.0**-25) + 2.0**-16


def srgb_exact(x):
    """s*255 + 0.5 of the exact curve, in float64, with the function's own float32 constants."""
    x = x.astype(np.float64)
    lin = np.float64(F32(12.92)) * x
    gam = np.float64(F32(1.055)) * np.power(np.maximum(x, 0.0), np.float64(F32(1) / F32(2.4))) - np.float64(F32(0.055))
    return np.where(x <= np.float64(F32(0.0031308)), lin, gam) * 255.0 + 0.5


def test_float_to_srgb8(kat):
    delta = srgb_delta(DEVICE_ULP["powf"] if kat.name == "device" else HOST_ULP["powf"])
    code = (np.arange(1, 256) - 0.5) / 255.0
    cut = np.where(code <= 12.92 * 0.0031308, code / 12.92, ((code + 0.055) / 1.055) ** 2.4)
    extra = np.concatenate([neighbours(cut, 64), np.array([-0.0, -1e-30, -1.0, -np.inf, np.nan, 1.0, 1.5, 1e30, np.inf], F32)])
    sweep = FloatRange(0.0, np.nextafter(F32(1), F32(2)), 1 if kat.name == "device" else 127)
    flagged = decided = count = 0
    for xc in [extra.astype(F32), *sweep.chunks()]:
        count += len(xc)
        got = kat.srgb8(xc).astype(np.int64)
        with np.errstate(invalid="ignore"):
            t = srgb_exact(xc)
            want = np.where(xc > 0, np.where(xc >= 1, 255, np.floor(t)), 0).astype(np.int64)
            near = (xc > 0) & (xc < 1) & (np.abs(t - np.round(t)) < delta)
        differ = got != want
        assert not (differ & ~near).any(), f"{kat.name} float_to_srgb8 at {xc[differ & ~near][:5].tolist()}"
        flagged += int(differ.sum())
        decided += int(near.sum())
    print(f"\n{kat.name} float_to_srgb8: {count:,d} inputs, {decided} within delta = {delta:.2e} of a rounding "
          f"boundary, {flagged} codes differ from round-half-up of the exact curve")


# ---- the miss shader ----
def miss_dirs():
    """Directions on the checker's boundaries: u*10 and v*10 at integers (and their float neighbours), dir.y at -0.1
    and its neighbours, the poles, atan2(+-0, +-0), plus NaN directions."""
    out = []
    k = np.arange(11)
    for j in k:
        for i in k:
            phi, theta = np.pi * (2 * j / 10 - 1), np.pi * i / 10
            out.append([np.sin(theta) * np.sin(phi), np.cos(theta), -np.sin(theta) * np.cos(phi)])
    out = np.array(out, F32)
    rows = [out] + [np.stack([neighbours(out[:, c], 2) if c == a else np.tile(out[:, c], 5) for c in range(3)], 1)
                    for a in range(3)]
    for y in neighbours([-0.1], 3):
        rest = np.sqrt(1 - float(y) ** 2)
        rows.append(np.array([[rest, y, 0], [0, y, -rest], [-rest * 0.6, y, rest * 0.8]], F32))
    rows.append(np.array([[0, 1, 0], [0, -1, 0], [0, 1, -0.0], [-0.0, 1, 0], [-0.0, -1, -0.0], [0.0, 0.5, 0.0],
                          [-0.0, 0.5, 0.0], [0.0, -0.05, -0.0], [-0.0, -0.05, -0.0], [np.nan] * 3], F32))
    return np.concatenate(rows).astype(F32)


def miss_delta(atan_ulp, acos_ulp):
    """How far u*10 (or v*10) may be from the float64 value: atan2f within atan_ulp of |a| <= pi (2^-22 each), times
    kInvPi, + 1, * 0.5 (exact), * 10 (each rounded: half an ulp of <= 1, <= 2, <= 10); kInvPi itself is 2^-25 off."""
    du = 0.5 * ((atan_ulp * 2.0**-22 + 2.0**-24) / np.pi + 2.0**-26 + 2.0**-23) * 10 + 2.0**-21
    dv = (acos_ulp * 2.0**-22 / np.pi + 2.0**-25 + 2.0**-25) * 10 + 2.0**-21
    return max(du, dv)


def test_miss_shader(kat, tables):
    k = kat_inputs()
    b = DEVICE_ULP if kat.name == "device" else HOST_ULP
    delta = miss_delta(b["atan2f"], b["acosf"])
    dirs = np.concatenate([k["miss_dirs"], miss_dirs(), _unit_dirs(200_000, 8)]).astype(F32)
    got = kat.miss(dirs)
    assert (got[:, 0] == got[:, 1]).all() and (got[:, 1] == got[:, 2]).all()
    d = dirs.astype(np.float64)
    with np.errstate(invalid="ignore"):
        u10 = (1 + np.arctan2(d[:, 0], -d[:, 2]) / np.pi) * 0.5 * 10
        v10 = np.arccos(d[:, 1]) / np.pi * 10
        even = (np.floor(u10) + np.floor(v10)) % 2 == 0
        want = np.where((dirs[:, 1] > F32(-0.1)) & even, F32(0.5), F32(0.1))
        near = (np.abs(u10 - np.round(u10)) < delta) | (np.abs(v10 - np.round(v10)) < delta)
    want = np.where(np.isnan(dirs).any(1), F32(0.1), want)
    differ = got[:, 0] != want
    assert not (differ & ~near).any(), f"{kat.name} miss shader at {dirs[differ & ~near][:5].tolist()}"
    n_tab = len(k["miss_dirs"])
    table = tables["kat.miss"]
    assert not ((got[:n_tab, 0] != table[:, 0]) & ~near[:n_tab]).any()
    print(f"\n{kat.name} miss shader: {len(dirs):,d} directions, {int(near.sum())} within {delta:.1e} of a checker "
          f"boundary, {int(differ.sum())} on the other side of one")


# ---- the Disney BSDF: eval, pdf, sample ----
def extreme_materials():
    """The fuzz script's parameter extremes: roughness 0, anisotropy 1, ior 1, transmission 0 and 1, and mixtures."""
    mats = []
    for rough in (0.0, 0.3, 1.0):
        for aniso in (0.0, 1.0):
            for trans, ior in ((0.0, 1.5), (1.0, 1.0), (1.0, 1.5), (0.6, 1.33)):
                for metal, cc, gloss in ((0.0, 1.0, 0.0), (0.5, 0.0, 1.0), (1.0, 0.5, 0.5)):
                    mats.append([0.8, 0.5, 0.2, metal, 0.5, rough, 0.4, aniso, 0.7, 0.3, cc, gloss, ior, trans, 0, 0])
    return np.array(mats, F32)


def bsdf_inputs(m, seed):
    """m (material, n, w_o) rows: w_o grazing, equal to +-n, and random in both hemispheres."""
    rs = np.random.default_rng(seed)
    mats = extreme_materials()
    mat = mats[rs.integers(0, len(mats), m)]
    n = _unit_dirs(m, seed + 1).astype(np.float64)
    n[:6] = np.concatenate([np.eye(3), -np.eye(3)])
    wo = _unit_dirs(m, seed + 2).astype(np.float64)
    kind = rs.integers(0, 6, m)
    t = np.cross(n, _unit_dirs(m, seed + 3))
    t /= np.linalg.norm(t, axis=1, keepdims=True)
    graze = 10.0 ** rs.uniform(-7, -2, m)[:, None] * np.where(rs.random(m) < 0.5, 1, -1)[:, None]
    wo = np.where((kind == 0)[:, None], n, wo)
    wo = np.where((kind == 1)[:, None], -n, wo)
    wo = np.where((kind == 2)[:, None], t + graze * n, wo)
    wo /= np.linalg.norm(wo, axis=1, keepdims=True)
    return mat, n.astype(F32), wo.astype(F32)


def clearcoat_alpha_sqr(mat):
    g = mat[:, 11]
    a = F32(0.1) * (F32(1) - g) + F32(0.001) * g
    return (a * a).astype(F32)


def logf_agrees(kat, host, mat):
    a2 = clearcoat_alpha_sqr(mat)
    return _bits(kat.math("logf", a2)) == _bits(host.math("logf", a2))


def eval_ulp_bound():
    """Where the device's logf of GTR1's alpha^2 differs from glibc's, by at most DEVICE_ULP + HOST_ULP ulp, the clear-coat
    term differs relatively by that many 2^-23 plus one ulp per operation after it (gtr_1's multiply and divides, the
    0.25 * clearcoat * d * f * g product: 6; the pdf's d * cos / (4 dot), the sum and / n_comp: 6). Every other term is
    the same on both sides and non-negative, so a channel of f or the pdf is at most that many ulp apart."""
    return DEVICE_ULP["logf"] + HOST_ULP["logf"] + 12


def check_eval(kat, host, mat, n, wo, wi, what):
    got, want = kat.eval(mat, n, wo, wi), host.eval(mat, n, wo, wi)
    agree = logf_agrees(kat, host, mat)
    _assert_same(got[agree], want[agree], f"{what} where logf agrees")
    fin = np.isfinite(want)
    assert np.array_equal(np.isfinite(got), fin) and np.array_equal(np.isnan(got), np.isnan(want)), what
    dist = np.where(fin, ulp_distance(got, want), 0)
    assert dist.max() <= eval_ulp_bound(), f"{what}: {int(dist.max())} ulp apart (bound {eval_ulp_bound()})"
    return int((~agree).sum()), int(dist.max())


def test_disney_eval(kat, host):
    m = 100_000
    mat, n, wo = bsdf_inputs(m, 10)
    wi = _unit_dirs(m, 20)
    wi[:2000] = wo[:2000]
    wi[2000:4000] = -wo[2000:4000]
    wi[4000:6000] = n[4000:6000]
    differ, worst = check_eval(kat, host, mat, n, wo, wi, "disney eval / pdf")
    print(f"\n{kat.name} disney eval: {m:,d} inputs, logf differs on {differ}, worst {worst} ulp from the host build")


def sample_rngs(m, seed):
    """rng states: random, and ones whose first draw rounds to 1.0f (the lobe choice's clamp)."""
    st = np.random.default_rng(seed).integers(0, 2**32, m, dtype=np.uint64).astype(U32)
    st[:len(EDGE_DRAWS) * 40] = np.tile(states_before(EDGE_DRAWS), 40)
    return st


def sample_transcendentals(mat, rng):
    """The lobe sample_disney_dir draws, and the arguments of its cosf / sinf (the angle) and powf (GTR1), restated in
    float32 from the rng."""
    s1, u0 = np_lcg(rng)
    s2, sx = np_lcg(s1)
    _, sy = np_lcg(s2)
    trans = mat[:, 13] != 0
    lobe = np.where(trans, np.minimum((u0 * F32(4)).astype(np.int64), 3), np.minimum((u0 * F32(3)).astype(np.int64), 2))
    ux, uy = F32(2) * sx - F32(1), F32(2) * sy - F32(1)
    pi4, pi2 = F32(np.pi) / F32(4), F32(np.pi) / F32(2)
    with np.errstate(divide="ignore", invalid="ignore"):
        theta = np.where(np.abs(ux) > np.abs(uy), pi4 * (uy / ux), pi2 - pi4 * (ux / uy))
    theta = np.where((ux == 0) & (uy == 0), F32(0), theta).astype(F32)
    angle = np.where(lobe == 0, theta, (F32(2) * F32(np.pi)) * sx).astype(F32)
    g = mat[:, 11]
    a = F32(0.1) * (F32(1) - g) + F32(0.001) * g
    return lobe, angle, (a * a).astype(F32), (F32(1) - sy).astype(F32), sx, sy, u0


def direction_bound(mat, lobe, sx, sy, n, wo, wi_host):
    """How far a sampled w_i may move when sinf / cosf / powf are within DEVICE_ULP of each other's results and glibc's
    within HOST_ULP: d = (B_dev + B_host) * 2^-24 in each of cos, sin (and powf's result < 1); the local direction's
    radial terms move by d / (2 * radius) where a square root takes them (hz of the concentric map, z and a of GTR1:
    `margin`); normalisation, the change of basis and the reflection about the half vector (x 4), or the refraction
    through it (x (2 eta + 1 + eta^2 / sqrt(k))), scale that; plus 16 ulp of last-bit noise from the operations after the
    first difference."""
    d = max(DEVICE_ULP["sinf"] + HOST_ULP["sinf"], DEVICE_ULP["cosf"] + HOST_ULP["cosf"], DEVICE_ULP["powf"] + HOST_ULP["powf"])
    d *= 2.0**-24
    sx64, sy64 = sx.astype(np.float64), sy.astype(np.float64)
    r = np.maximum(np.abs(2 * sx64 - 1), np.abs(2 * sy64 - 1))
    g = mat[:, 11].astype(np.float64)
    a2 = (0.1 * (1 - g) + 0.001 * g) ** 2
    c2 = (1 - a2 ** (1 - sy64)) / (1 - a2)
    margin = np.where(lobe == 0, np.sqrt(np.maximum(1 - r * r, 0)),
                      np.where(lobe == 2, np.sqrt(np.clip(np.minimum(c2, 1 - c2), 0, 1)), 1.0))
    margin = np.maximum(margin, 1e-9)
    ior = mat[:, 12].astype(np.float64)
    entering = (wo.astype(np.float64) * n).sum(1) > 0
    eta = np.where(entering, 1 / ior, ior)
    # sqrt(k) of the refraction, from the host's result: w_i = eta i - (eta n.i + sqrt k) h, so h ~ eta i - w_i
    i = -wo.astype(np.float64)
    h = eta[:, None] * i - wi_host
    h /= np.maximum(np.linalg.norm(h, axis=1, keepdims=True), 1e-30)
    sqrt_k = np.abs((h * wi_host).sum(1))
    amp = np.where(lobe == 3, 2 * eta + 1 + eta * eta / np.maximum(sqrt_k, 1e-9), 4.0)
    return amp * (2 * d / margin + 16 * 2.0**-24), sqrt_k


def test_disney_sample(kat, host):
    """sample_disney_brdf: the rng state after the call is bit-exact. Where the device's sinf / cosf (and powf on the
    clear-coat lobe, logf of its alpha) return what glibc's do, so does everything else, bit for bit. Elsewhere w_i is
    within direction_bound of the host's, a discrete outcome (hemisphere test, total internal reflection) may differ only
    where its float64 margin is below that bound, and f and pdf are those of the host's eval at the device's w_i."""
    m = 100_000
    mat, n, wo = bsdf_inputs(m, 30)
    rng = sample_rngs(m, 31)
    got, st = kat.sample(mat, n, wo, rng)
    want, st_h = host.sample(mat, n, wo, rng)
    lobe, angle, a2, e, sx, sy, u0 = sample_transcendentals(mat, rng)
    assert np.array_equal(st, st_h)
    s3 = np_lcg(np_lcg(np_lcg(rng)[0])[0])[0]
    assert np.array_equal(st, s3), "the sample consumes exactly three draws"
    clamp = u0 == 1
    assert clamp.sum() >= 100 and set(np.unique(lobe[clamp])) == {2, 3}
    agree = (_bits(kat.math("cosf", angle)) == _bits(host.math("cosf", angle))) & \
            (_bits(kat.math("sinf", angle)) == _bits(host.math("sinf", angle))) & logf_agrees(kat, host, mat)
    pw = lobe == 2
    agree[pw] &= _bits(kat.math("powf", a2[pw], e[pw])) == _bits(host.math("powf", a2[pw], e[pw]))
    _assert_same(got[agree], want[agree], "sample_disney_brdf where the transcendentals agree")
    wi_d, wi_h = got[:, 4:7].astype(np.float64), want[:, 4:7].astype(np.float64)
    valid_d, valid_h = (got[:, 4:7] != 0).any(1), (want[:, 4:7] != 0).any(1)
    tol, sqrt_k = direction_bound(mat, lobe, sx, sy, n.astype(np.float64), wo, np.where(valid_h[:, None], wi_h, wi_d))
    both = valid_d & valid_h
    err = np.linalg.norm(wi_d - wi_h, axis=1)
    assert (err[both] <= tol[both]).all(), \
        f"w_i {float((err / tol)[both].max()):.2f} x the bound apart (lobes {np.unique(lobe[both & (err > tol)])})"
    flip = valid_d != valid_h
    w_valid = np.where(valid_d[:, None], wi_d, wi_h)
    hemi = np.abs((w_valid * n).sum(1))
    excused = (hemi < tol) | ((lobe == 3) & (sqrt_k < tol * 4))
    assert not (flip & ~excused).any(), f"discrete outcome differs at {np.nonzero(flip & ~excused)[0][:5].tolist()}"
    # f and pdf: the host's eval at the direction the device sampled
    ok = valid_d & ~agree
    if ok.any():
        ev = host.eval(mat[ok], n[ok], wo[ok], got[ok, 4:7])
        pdf_zero = got[ok, 3] == 0
        cmp = np.concatenate([got[ok, 0:4][~pdf_zero], ev[~pdf_zero]], 1)
        dist = np.where(np.isfinite(cmp[:, 4:]), ulp_distance(cmp[:, :4], cmp[:, 4:]), 0)
        assert dist.max(initial=0) <= eval_ulp_bound()
    print(f"\n{kat.name} disney sample: {m:,d} samples ({int(clamp.sum())} with a first draw of 1.0f), transcendentals "
          f"differ on {int((~agree).sum())}, worst w_i {float((err / tol)[both].max(initial=0)):.3f} x the bound, "
          f"{int(flip.sum())} discrete outcomes differ")
