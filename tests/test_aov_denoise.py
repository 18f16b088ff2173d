"""First-hit AOV buffers (option "aov") and the edge-aware à-trous denoiser (crtc_read_aov, crtc_denoise;
chameleonrt_b200/csrc/aov_denoise.cuh).

The same check functions run on the emulated renderer (tests/simt_emu: the product sources built for the host, every
kernel under the SIMT environment) without a GPU, and on libcrt_cuda_core.so on an H100 (``-m gpu``):
  * AOV content against an independent host computation: the oracle's primary rays and closest hits, the scene model's
    materials unpacked by the host build of the shading code (libcrt_shade_hostcheck.so), k_resolve's running mean;
  * the option changes nothing else: accum, img and ray counts are bit-identical, two more launches per wavefront;
  * batched frames give the same AOVs as single frames, and a camera change resets them;
  * the denoiser against a numpy float32 restatement of its definition (include/crt_cuda.h, crtc_denoise);
  * the denoised image is closer to a converged frame than the noisy one;
  * error paths; the drop-in plugin's CRT_CUDA_DENOISE.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from helpers import camera_for, huge_uv_scene, synthetic_material_scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "chameleonrt_b200", "csrc")
MISS = 0xFFFFFFFF


# ---- fixtures ----
@pytest.fixture(scope="module")
def emu(built):
    """(RenderCUDA, OracleBackend, primary_rays) with RenderCUDA bound to the emulated renderer."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "simt_emu"))
    import build as simt_build

    # (the emulation build's freshness list predates aov_denoise.cuh)
    lib = simt_build.LIB
    stale = not os.path.exists(lib) or os.path.getmtime(lib) < os.path.getmtime(os.path.join(CSRC, "aov_denoise.cuh"))
    lib_path = simt_build.build(force=stale)
    import chameleonrt_b200.backend as backend
    from oracle import OracleBackend
    from oracle.oracle import primary_rays

    saved = (backend._LIB_PATH, backend._lib)
    backend._LIB_PATH, backend._lib = lib_path, None
    yield backend.RenderCUDA, OracleBackend, primary_rays
    backend._LIB_PATH, backend._lib = saved


@pytest.fixture(scope="module")
def gpu(built):
    from chameleonrt_b200 import RenderCUDA
    from oracle import OracleBackend
    from oracle.oracle import primary_rays

    return RenderCUDA, OracleBackend, primary_rays


@pytest.fixture(scope="module")
def shade(built):
    lib = C.CDLL(os.path.join(CSRC, "libcrt_shade_hostcheck.so"))
    vp = C.c_void_p
    lib.shadekat_unpack_material.argtypes = [vp, C.c_uint32, vp, vp, vp, C.c_int, vp]
    lib.shadekat_miss.argtypes = [vp, C.c_int, vp]
    return lib


def _args(cam):
    c = camera_for(cam)
    return (c.eye(), c.dir(), c.up(), cam["fov_y"])


def _renderer(RenderCUDA, scene, w, h, depth=5, **kw):
    r = RenderCUDA(0, max_depth=depth, **kw)
    r.initialize(w, h)
    r.set_scene(scene)
    return r


# ---- the expected AOVs, computed on the host ----
def _srgb_lut():
    """render_embree.cpp:96-103 as host_scene.cpp computes it: 8-bit sRGB -> 8-bit linear, truncated."""
    lut = np.zeros(256, np.uint8)
    for v in range(256):
        x = np.float32(v) / np.float32(255.0)
        if x <= np.float32(0.04045):
            x = x / np.float32(12.92)
        else:
            x = np.float32(np.float64((x + np.float32(0.055)) / np.float32(1.055)) ** 2.4)
        y = x * np.float32(255.0)
        lut[v] = int(min(max(y, np.float32(0.0)), np.float32(255.0)))
    return lut


class SceneTables:
    """The scene model as the shading code sees it: per flattened triangle its material id and vertex uvs, the material
    words, and the texel arena (linearised sRGB, RGBA8 words, missing channels 0)."""

    def __init__(self, scene):
        from chameleonrt_b200.scene import SRGB, f32_bits

        mats, uvs, has_uv = [], [], []
        for inst in scene.instances:
            pm = scene.parameterized_meshes[inst.parameterized_mesh_id]
            for g, geom in enumerate(scene.meshes[pm.mesh_id].geometries):
                n = geom.num_tris()
                mats.append(np.full(n, pm.material_ids[g], np.uint32))
                if geom.uvs is not None:
                    uvs.append(np.asarray(geom.uvs, np.float32)[np.asarray(geom.indices)].reshape(n, 6))
                    has_uv.append(np.ones(n, bool))
                else:
                    uvs.append(np.zeros((n, 6), np.float32))
                    has_uv.append(np.zeros(n, bool))
        self.material_id = np.concatenate(mats)
        self.uvs = np.concatenate(uvs)
        self.has_uv = np.concatenate(has_uv)
        self.materials = np.ascontiguousarray(
            np.array([[f32_bits(v) for v in m.as_floats()] for m in scene.materials], np.uint32).view(np.float32))
        lut = _srgb_lut()
        words, desc, off = [], [], 0
        for t in scene.textures:
            img = np.asarray(t.img, np.uint8).reshape(t.height * t.width, t.channels).copy()
            if t.color_space == SRGB:
                k = min(3, t.channels)
                img[:, :k] = lut[img[:, :k]]
            rgba = np.zeros((img.shape[0], 4), np.uint32)
            rgba[:, :t.channels] = img
            words.append(rgba[:, 0] | (rgba[:, 1] << 8) | (rgba[:, 2] << 16) | (rgba[:, 3] << 24))
            desc.append([off, t.width, t.height, 0])
            off += img.shape[0]
        self.texels = np.ascontiguousarray(np.concatenate(words) if words else np.zeros(1, np.uint32))
        self.tex = np.ascontiguousarray(np.array(desc if desc else [[0, 0, 0, 0]], np.int32))

    def unpack(self, shade, prim, u, v):
        """(base colour (n, 3), specular_transmission (n,)) of the hit of flat primitive `prim` at barycentrics u, v."""
        one = np.float32(1.0)
        bw = one - u - v
        uv = self.uvs[prim]
        uvx = uv[:, 0] * bw + uv[:, 2] * u + uv[:, 4] * v
        uvy = uv[:, 1] * bw + uv[:, 3] * u + uv[:, 5] * v
        uvs = np.where(self.has_uv[prim][:, None], np.stack([uvx, uvy], 1), np.float32(0.0)).astype(np.float32)
        out = np.zeros((len(prim), 14), np.float32)
        mids = self.material_id[prim]
        for m in np.unique(mids):
            sel = np.nonzero(mids == m)[0]
            part = np.zeros((len(sel), 14), np.float32)
            q = np.ascontiguousarray(uvs[sel])
            shade.shadekat_unpack_material(self.materials.ctypes.data, int(m), self.texels.ctypes.data, self.tex.ctypes.data,
                                           q.ctypes.data, len(sel), part.ctypes.data)
            out[sel] = part
        return out[:, 0:3], out[:, 13]


def expected_aovs(mods, shade, scene, cam, w, h, frames, first_frame=0):
    """The AOV running mean after `frames` frames (frame ids first_frame..), per pixel (h, w, 8), plus the flat primitive
    ids of every sample (frames * spp, h * w)."""
    _, OracleBackend, primary_rays = mods
    spp = scene.samples_per_pixel
    tables = SceneTables(scene)
    orc = OracleBackend()
    orc.initialize(w, h)
    orc.set_scene(scene)
    acc = np.zeros((h * w, 8), np.float32)
    prims = []
    for f in range(first_frame, first_frame + frames):
        albedo = np.zeros((h * w, 3), np.float32)
        normal = np.zeros((h * w, 3), np.float32)
        coverage = np.zeros(h * w, np.float32)
        depth = np.zeros(h * w, np.float32)
        hits_n = np.zeros(h * w, np.uint32)
        for s in range(spp):
            rays = primary_rays(w, h, *_args(cam), frame_id=f, spp=spp, s=s)
            hits, normals = orc.trace_closest(rays, want_normals=True)
            prim = hits[:, 3].view(np.uint32)
            prims.append(prim.copy())
            d = rays[:, 4:7]
            hit = prim != MISS
            sample_albedo = np.zeros((h * w, 3), np.float32)
            miss_idx = np.nonzero(~hit)[0]
            if len(miss_idx):
                dirs = np.ascontiguousarray(d[miss_idx])
                ms = np.zeros((len(miss_idx), 3), np.float32)
                shade.shadekat_miss(dirs.ctypes.data, len(miss_idx), ms.ctypes.data)
                sample_albedo[miss_idx] = ms
            hi = np.nonzero(hit)[0]
            if len(hi):
                base, transmission = tables.unpack(shade, prim[hi], hits[hi, 1], hits[hi, 2])
                sample_albedo[hi] = base
                n = normals[hi]
                wo = -d[hi]
                flip = (transmission == 0) & ((wo[:, 0] * n[:, 0] + wo[:, 1] * n[:, 1]) + wo[:, 2] * n[:, 2] < 0)
                n = np.where(flip[:, None], -n, n)
                normal[hi] += n
                coverage[hi] += np.float32(1.0)
                depth[hi] += hits[hi, 0]
                hits_n[hi] += 1
            albedo += sample_albedo
        fspp = np.float32(spp)
        frame = np.concatenate([albedo / fspp, (coverage / fspp)[:, None], normal / fspp,
                                np.where(hits_n > 0, depth / np.maximum(hits_n, 1).astype(np.float32), np.float32(0.0))[:, None]],
                               axis=1).astype(np.float32)
        acc = (frame + np.float32(f) * acc) / np.float32(f + 1)
    return acc.reshape(h, w, 8), np.stack(prims)


def check_aov_content(mods, shade, scene, cam, w, h, frames=2, min_match=0.999, depth=5, exact_albedo=True):
    RenderCUDA = mods[0]
    r = RenderCUDA(0, max_depth=depth, aov=True)
    r.initialize(w, h)
    r.set_scene(scene)
    args = _args(cam)
    for f in range(frames):
        r.render(*args, f == 0, True)
    got = r.read_aov()
    want, oracle_prims = expected_aovs(mods, shade, scene, cam, w, h, frames)
    # the renderer's own closest hits of the same rays: a pixel "matches" where every sample hit the same primitive
    spp = scene.samples_per_pixel
    _, _, primary_rays = mods
    own = np.stack([r.trace_closest(primary_rays(w, h, *args, frame_id=f, spp=spp, s=s))[:, 3].view(np.uint32)
                    for f in range(frames) for s in range(spp)])
    same = (own == oracle_prims).all(axis=0).reshape(h, w)
    assert same.mean() >= min_match, f"only {same.mean():.4f} of the pixels hit the same primitives"
    coverage_ok = got["coverage"] == want[:, :, 3]
    assert coverage_ok[same].all() and coverage_ok.mean() >= min_match
    if exact_albedo:
        assert np.array_equal(got["albedo"][same].view(np.uint32), want[:, :, 0:3][same].view(np.uint32))
    else:  # barycentrics that agree to rounding only: the texture filter may land on the other side of a texel boundary
        close = (np.abs(got["albedo"] - want[:, :, 0:3]) <= 1e-4 + 1e-3 * np.abs(want[:, :, 0:3])).all(axis=-1)
        assert close[same].mean() >= min_match
    nrm_err = np.linalg.norm(got["normal"] - want[:, :, 4:7], axis=-1)
    assert (nrm_err[same] <= 1e-5 * np.linalg.norm(want[:, :, 4:7], axis=-1)[same] + 1e-7).all()
    dz = np.abs(got["depth"] - want[:, :, 7])
    assert (dz[same] <= 1e-5 * np.abs(want[:, :, 7])[same]).all()
    # the luminance moments: the running mean of what the frame's samples contributed; m2 >= m1^2 up to rounding
    assert np.isfinite(got["lum_m1"]).all() and (got["lum_m2"] >= got["lum_m1"] ** 2 * (1 - 1e-5) - 1e-12).all()
    return r, got, want, same


def check_no_effect_on_the_frame(mods, scene, cam, w, h, frames=2, depth=5):
    RenderCUDA = mods[0]
    out = []
    for aov in (False, True):
        r = _renderer(RenderCUDA, scene, w, h, depth=depth, aov=aov)
        rays = [r.render(*_args(cam), f == 0, True).num_rays for f in range(frames)]
        out.append((r.read_accum(), r.read_img().copy(), rays, r.counters()["kernel_launches"]))
    (a0, i0, n0, k0), (a1, i1, n1, k1) = out
    assert np.array_equal(a0.view(np.uint32), a1.view(np.uint32)) and np.array_equal(i0, i1) and n0 == n1
    assert k1 == k0 + 2


def check_batching_and_reset(mods, scene, cam, w, h):
    RenderCUDA = mods[0]
    args = _args(cam)
    single = _renderer(RenderCUDA, scene, w, h, aov=True)
    for f in range(3):
        single.render(*args, f == 0, True)
    want = single.read_aov()
    batched = _renderer(RenderCUDA, scene, w, h, aov=True)
    batched.render_async(*args, True, 1)
    batched.render_async(*args, False, 2)
    assert batched.sync()[3] == 3
    got = batched.read_aov()
    for k in want:
        assert np.array_equal(got[k].view(np.uint32), want[k].view(np.uint32)), k
    # a camera change resets the AOVs exactly as it resets accum
    moved = dict(cam, eye=tuple(np.asarray(cam["eye"], np.float64) + np.array([0.3, 0.1, 0.0])))
    single.render(*_args(moved), True, True)
    fresh = _renderer(RenderCUDA, scene, w, h, aov=True)
    fresh.render(*_args(moved), True, True)
    a, b = single.read_aov(), fresh.read_aov()
    for k in a:
        assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), k


# ---- the denoiser, restated from its definition (include/crt_cuda.h, crtc_denoise) ----
def _lum(c):
    return (np.float32(0.2126) * c[..., 0] + np.float32(0.7152) * c[..., 1]) + np.float32(0.0722) * c[..., 2]


def _shift(a, dx, dy, fill=0.0):
    """b[y, x] = a[y + dy, x + dx] where inside the image, `fill` elsewhere; and the mask of inside."""
    h, w = a.shape[:2]
    b = np.full_like(a, fill)
    m = np.zeros((h, w), bool)
    ys, yd = (slice(dy, h), slice(0, h - dy)) if dy >= 0 else (slice(0, h + dy), slice(-dy, h))
    xs, xd = (slice(dx, w), slice(0, w - dx)) if dx >= 0 else (slice(0, w + dx), slice(-dx, w))
    if ys.start < h and xs.start < w and ys.stop > 0 and xs.stop > 0:
        b[yd, xd] = a[ys, xs]
        m[yd, xd] = True
    return b, m


def denoise_reference(accum, aov, samples, iterations=5, sigma_l=4.0, sigma_n=128.0, sigma_z=1.0):
    f32 = np.float32
    accum = accum.astype(f32)
    alb = np.maximum(aov["albedo"], f32(1e-3))
    I = accum / alb
    v = np.maximum(f32(0.0), aov["lum_m2"] - aov["lum_m1"] * aov["lum_m1"]) / f32(samples)
    n = aov["normal"]
    ln = np.sqrt(n[..., 0] * n[..., 0] + n[..., 1] * n[..., 1] + n[..., 2] * n[..., 2])
    nh = np.where(ln[..., None] > 0, n / np.where(ln > 0, ln, f32(1.0))[..., None], f32(0.0)).astype(f32)
    bg = (nh == 0).all(axis=-1)
    Z = aov["depth"]
    h, w = Z.shape

    def grad(axis):
        size = Z.shape[axis]
        idx = np.arange(size)
        lo, hi = np.maximum(idx - 1, 0), np.minimum(idx + 1, size - 1)
        d = np.take(Z, hi, axis=axis) - np.take(Z, lo, axis=axis)
        two = (hi - lo) == 2
        shape = [1, 1]
        shape[axis] = size
        return np.where(two.reshape(shape), f32(0.5) * d, d).astype(f32)

    gx, gy = grad(1), grad(0)
    b3 = {-2: f32(0.0625), -1: f32(0.25), 0: f32(0.375), 1: f32(0.25), 2: f32(0.0625)}
    for i in range(iterations):
        step = 1 << i
        gv = np.zeros((h, w), f32)
        gw = np.zeros((h, w), f32)
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                vq, m = _shift(v, dx, dy)
                k = f32((2 - abs(dx)) * (2 - abs(dy)) * 0.0625)
                gv = np.where(m, gv + k * vq, gv)
                gw = np.where(m, gw + k, gw)
        lp = _lum(I)
        scale = f32(sigma_l) * np.sqrt(gv / gw) + f32(1e-10)
        sw = np.zeros((h, w), f32)
        sI = np.zeros((h, w, 3), f32)
        sv = np.zeros((h, w), f32)
        for dy in range(-2, 3):
            for dx in range(-2, 3):
                Iq, m = _shift(I, dx * step, dy * step)
                vq, _ = _shift(v, dx * step, dy * step)
                nq, _ = _shift(nh, dx * step, dy * step)
                Zq, _ = _shift(Z, dx * step, dy * step)
                bq, _ = _shift(bg, dx * step, dy * step, fill=True)
                w_l = np.exp(-np.abs(lp - _lum(Iq)) / scale)
                dot = (nh[..., 0] * nq[..., 0] + nh[..., 1] * nq[..., 1]) + nh[..., 2] * nq[..., 2]
                w_n = np.power(np.maximum(f32(0.0), dot), f32(sigma_n))
                w_n = np.where(bg | bq, np.where(bg & bq, f32(1.0), f32(0.0)), w_n)
                w_z = np.exp(-np.abs(Z - Zq) / (f32(sigma_z) * np.abs(gx * f32(step * dx) + gy * f32(step * dy)) + f32(1e-3)))
                wt = (b3[dx] * b3[dy] * w_l * w_n * w_z).astype(f32)
                wt = np.where(m, wt, f32(0.0))
                sw = sw + wt
                sI = sI + Iq * wt[..., None]
                sv = sv + wt * wt * vq
        I = (sI / sw[..., None]).astype(f32)
        v = (sv / (sw * sw)).astype(f32)
    return (I * alb).astype(f32)


def srgb8(x):
    x = x.astype(np.float32)
    s = np.where(x <= np.float32(0.0031308), np.float32(12.92) * x,
                 np.float32(1.055) * np.power(np.maximum(x, np.float32(0.0)), np.float32(1.0 / 2.4)) - np.float32(0.055))
    q = np.floor(s * np.float32(255.0) + np.float32(0.5))
    return np.where(x > 0, np.where(x >= 1, 255, q), 0).astype(np.uint32)


def check_filter(r, spp, frames, cases, exact_img=True):
    accum, aov = r.read_accum(), r.read_aov()
    for kw in cases:
        rgb, img = r.denoise(**kw)
        prm = dict(iterations=kw.get("iterations", 5), sigma_l=kw.get("sigma_luminance", 4.0),
                   sigma_n=kw.get("sigma_normal", 128.0), sigma_z=kw.get("sigma_depth", 1.0))
        want = denoise_reference(accum, aov, spp * frames, **prm)
        assert np.isfinite(rgb).all()
        assert (np.abs(rgb - want) <= 1e-4 * np.abs(want) + 1e-6).all(), (kw, float(np.abs(rgb - want).max()))
        c = srgb8(rgb)
        assert (img >> 24 == 0xFF).all()
        got = np.stack([(img >> (8 * k)) & 0xFF for k in range(3)], axis=-1).astype(np.int64)
        if exact_img:
            assert np.array_equal(got, c), kw
        else:  # the device powf of the sRGB curve against numpy's: a value on a rounding boundary may land one code apart
            assert np.abs(got - c.astype(np.int64)).max() <= 1, kw


def check_quality(mods, size=64):
    """Cornell, 4 spp, one frame: the denoised frame's MSE against a converged oracle frame (1024 spp) is at most half the
    noisy frame's."""
    from chameleonrt_b200.scenes import cornell_box

    RenderCUDA, OracleBackend, _ = mods
    scene, cam = cornell_box(spp=4)
    r = _renderer(RenderCUDA, scene, size, size, aov=True)
    r.render(*_args(cam), True, True)
    noisy = r.read_accum()
    rgb, _ = r.denoise()
    ref_scene, _ = cornell_box(spp=64)
    orc = OracleBackend(fast=True)
    orc.initialize(size, size)
    orc.set_scene(ref_scene)
    for f in range(16):
        orc.render(*_args(cam), f == 0)
    ref = orc.read_accum()
    mse_noisy = float(np.mean((noisy - ref) ** 2))
    mse_denoised = float(np.mean((rgb - ref) ** 2))
    assert mse_denoised <= 0.5 * mse_noisy, (mse_denoised, mse_noisy)
    return mse_noisy, mse_denoised


def check_errors(mods):
    from chameleonrt_b200.scenes import cornell_box

    RenderCUDA = mods[0]
    scene, cam = cornell_box(spp=1)
    plain = _renderer(RenderCUDA, scene, 16, 16)
    plain.render(*_args(cam), True, True)
    for call in (plain.read_aov, plain.denoise):
        with pytest.raises(RuntimeError, match="aov is off"):
            call()
    plain.set_option("aov", 1)  # takes effect at the next initialize
    assert plain.get_option("aov") == 1
    with pytest.raises(RuntimeError, match="aov is off"):
        plain.read_aov()
    r = _renderer(RenderCUDA, scene, 16, 16, aov=True)
    for call in (r.read_aov, r.denoise):
        with pytest.raises(RuntimeError, match="no frame"):
            call()
    r.render(*_args(cam), True, True)
    for kw in (dict(iterations=0), dict(iterations=11), dict(sigma_luminance=0.0), dict(sigma_normal=-1.0),
               dict(sigma_depth=float("nan")), dict(sigma_luminance=float("inf"))):
        with pytest.raises(RuntimeError, match="iterations must be|must be finite"):
            r.denoise(**kw)
    r.denoise(iterations=1)
    r.denoise(iterations=10)
    r.set_scene(scene)  # a new scene resets the AOVs like accum
    with pytest.raises(RuntimeError, match="no frame"):
        r.read_aov()
    sharded = RenderCUDA(0, rank=0, world_size=2, aov=True)
    with pytest.raises(RuntimeError, match="world_size"):
        sharded.initialize(16, 16)
    with pytest.raises(RuntimeError, match="whole frame"):
        r.export_frame()
    other = _renderer(RenderCUDA, scene, 16, 16)
    with pytest.raises(RuntimeError, match="whole frame"):
        r.share_frame_with(other)
    with pytest.raises(RuntimeError, match="whole frame"):
        other.share_frame_with(r)
    exporter = _renderer(RenderCUDA, scene, 16, 16)
    handles = exporter.export_frame()
    with pytest.raises(RuntimeError, match="whole frame"):
        r.import_frame(handles)


# ---- CPU: the emulated renderer ----
@pytest.mark.parametrize("spp", [1, 2])
def test_aov_content_on_the_emulated_renderer(emu, shade, spp):
    from chameleonrt_b200.scenes import cornell_box

    for scene, cam, (w, h) in ((*cornell_box(spp=spp), (40, 24)), (*synthetic_material_scene(spp=spp), (40, 24)),
                               (*huge_uv_scene(spp=spp), (24, 16))):
        check_aov_content(emu, shade, scene, cam, w, h, frames=2)


def test_aov_option_does_not_change_the_frame_on_the_emulated_renderer(emu):
    from chameleonrt_b200.scenes import cornell_box

    check_no_effect_on_the_frame(emu, *synthetic_material_scene(spp=2), 40, 24)
    check_no_effect_on_the_frame(emu, *cornell_box(spp=1), 70, 40)  # two tiles, ragged


def test_aov_batching_and_reset_on_the_emulated_renderer(emu):
    from chameleonrt_b200.scenes import cornell_box

    check_batching_and_reset(emu, *cornell_box(spp=2), 70, 40)


def test_denoiser_matches_its_definition_on_the_emulated_renderer(emu):
    scene, cam = synthetic_material_scene(spp=2)
    r = _renderer(emu[0], scene, 48, 32, aov=True)
    for f in range(2):
        r.render(*_args(cam), f == 0, True)
    check_filter(r, 2, 2, [dict(iterations=1), dict(iterations=5),
                           dict(iterations=3, sigma_luminance=1.5, sigma_normal=16.0, sigma_depth=0.25)])


def test_denoiser_quality_on_the_emulated_renderer(emu):
    check_quality(emu)


def test_aov_error_paths_on_the_emulated_renderer(emu):
    check_errors(emu)


def test_plugin_denoise_variable_on_the_emulated_core(emu, tmp_path):
    """`crt_headless cuda_simt` with CRT_CUDA_DENOISE=1: the image it writes is Python's denoise() of the same frames, and
    its float framebuffer does not change."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "simt_emu"))
    import build as simt_build
    from test_reference_plugin import HEADLESS, run_headless

    if not os.path.exists(HEADLESS) or simt_build.build_plugin() is None:
        pytest.skip("needs oracle/_ref (built where the reference sources are)")
    Image = pytest.importorskip("PIL.Image")
    from chameleonrt_b200.obj_io import write_obj
    from chameleonrt_b200.scenes import cornell_box

    w, h, frames = 64, 48, 2
    scene, cam = cornell_box(spp=2)
    obj = write_obj(scene, str(tmp_path / "scene.obj"))
    plain, v, _ = run_headless("cuda_simt", obj, cam, w, h, 2, frames, tmp_path)
    denoised, v2, _ = run_headless("cuda_simt", obj, cam, w, h, 2, frames, tmp_path, extra_env={"CRT_CUDA_DENOISE": "1"})
    assert v == v2 and np.array_equal(plain.view(np.uint32), denoised.view(np.uint32))
    png = np.asarray(Image.open(tmp_path / "chameleonrt.png").convert("RGBA"), np.uint32)
    png = png[..., 0] | (png[..., 1] << 8) | (png[..., 2] << 16) | (png[..., 3] << 24)
    r = _renderer(emu[0], scene, w, h, aov=True)
    for f in range(frames):
        r.render(v[0:3], v[3:6], v[6:9], v[9], f == 0, True)
    assert np.array_equal(r.read_accum().view(np.uint32), denoised.view(np.uint32))
    assert np.array_equal(r.denoise()[1], png)
    with pytest.raises(AssertionError, match="CRT_CUDA_DENOISE"):
        run_headless("cuda_simt", obj, cam, w, h, 2, 1, tmp_path, extra_env={"CRT_CUDA_DENOISE": "1", "CRT_CUDA_DEVICES": "0,1"})


# ---- GPU: libcrt_cuda_core.so on the H100 ----
@pytest.mark.gpu
def test_aov_content_cornell(gpu, shade):
    from chameleonrt_b200.scenes import cornell_box

    for spp in (1, 2):
        check_aov_content(gpu, shade, *cornell_box(spp=spp), 128, 96, frames=2)
        # uv * width past 2^31 texels: the texel index the host conversion gives (shade_math.cuh: float_to_int_x86)
        check_aov_content(gpu, shade, *huge_uv_scene(spp=spp), 64, 48, frames=2)


@pytest.mark.gpu
def test_aov_content_sponza_like(gpu, shade):
    from chameleonrt_b200.scenes import sponza_like

    check_aov_content(gpu, shade, *sponza_like(spp=2, detail=0.3, tex_size=64), 320, 180, frames=2, depth=8)


@pytest.mark.gpu
def test_aov_content_instanced_scene(gpu, shade):
    """Non-identity instances: the oracle intersects in object space, the renderer in world space, so primitives,
    barycentrics and normals agree up to the frame tests' parity tolerance (99 % of the pixels)."""
    from chameleonrt_b200.scenes import san_miguel_like

    check_aov_content(gpu, shade, *san_miguel_like(spp=2, scale=0.02, tex_size=64), 192, 108, frames=2, min_match=0.99,
                      exact_albedo=False)


@pytest.mark.gpu
def test_aov_option_does_not_change_the_c2_frame(gpu):
    from chameleonrt_b200.scenes import sponza_like

    check_no_effect_on_the_frame(gpu, *sponza_like(spp=4), 1280, 720, frames=2, depth=8)


@pytest.mark.gpu
def test_aov_batching_and_reset(gpu):
    from chameleonrt_b200.scenes import cornell_box

    check_batching_and_reset(gpu, *cornell_box(spp=2), 130, 70)


@pytest.mark.gpu
def test_denoiser_matches_its_definition(gpu):
    from chameleonrt_b200.scenes import sponza_like

    scene, cam = sponza_like(spp=2, detail=0.3, tex_size=64)
    r = _renderer(gpu[0], scene, 320, 180, depth=8, aov=True)
    for f in range(2):
        r.render(*_args(cam), f == 0, True)
    check_filter(r, 2, 2, [dict(iterations=1), dict(iterations=5),
                           dict(iterations=4, sigma_luminance=1.5, sigma_normal=16.0, sigma_depth=0.25)], exact_img=False)


@pytest.mark.gpu
def test_denoiser_quality(gpu):
    check_quality(gpu)


@pytest.mark.gpu
def test_aov_error_paths(gpu):
    check_errors(gpu)


@pytest.mark.gpu
def test_hw_textures_albedo_is_what_the_texture_unit_filters(gpu):
    """hw_textures = 1: k_aov_primary unpacks the base colour through the same unpack_material<true> branch as
    k_shade<true>, so a textured scene's albedo differs from the software path's by the texture unit's filtering only (8-bit
    weights, sRGB decoded at full precision instead of the 8-bit linearised texels), within the tolerance the frame test of
    the option uses (relative L1 <= 3 %, per-channel mean within 2 %), and the untextured parts are bit-identical."""
    from chameleonrt_b200.scenes import sponza_like

    scene, cam = sponza_like(spp=1, detail=0.3, tex_size=64)
    w, h = 160, 90
    out = {}
    for hw in (0, 1):
        r = gpu[0](0, max_depth=5, aov=True)
        r.set_option("hw_textures", hw)
        r.initialize(w, h)
        r.set_scene(scene)
        r.render(*_args(cam), True, True)
        out[hw] = r.read_aov()
    a0, a1 = out[0]["albedo"], out[1]["albedo"]
    assert np.array_equal(out[0]["coverage"], out[1]["coverage"]) and np.array_equal(out[0]["depth"], out[1]["depth"])
    differs = (a0 != a1).any(axis=-1)
    assert 0 < differs.mean() < 1  # textured surfaces differ, untextured ones and the background do not
    assert np.abs(a1 - a0).sum() <= 0.03 * np.abs(a0).sum()
    assert (np.abs(a1.mean(axis=(0, 1)) - a0.mean(axis=(0, 1))) <= 0.02 * a0.mean(axis=(0, 1))).all()
