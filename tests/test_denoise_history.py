"""The denoiser's temporal history (option "denoise_history"; crtc_denoise, crtc_read_denoise_history;
chameleonrt_b200/csrc/aov_denoise.cuh: k_dn_temporal, k_dn_variance).

Every check runs on the emulated renderer (tests/simt_emu) without a GPU and on libcrt_cuda_core.so on an H100 (``-m gpu``):
  * nothing changes with the option on where there is nothing to carry: the first epoch at spp >= 4, the epoch after
    set_scene, and every frame's accum, img, ray counts and launches;
  * the history against a numpy float32 restatement of its definition (include/crt_cuda.h, crtc_denoise), and the
    denoised output against the restated variance pass plus test_aov_denoise's restatement of the a-trous chain, fed the
    device's own history;
  * geometry, independent of the restatement: the same camera, a sideways shift over a wall, a disocclusion;
  * quality along a moving camera at 1 spp, where the history-off denoiser returns its input;
  * error paths and the drop-in plugin's CRT_CUDA_DENOISE_HISTORY.
"""
import os
import sys

import numpy as np
import pytest

from test_aov_denoise import _args, _renderer, _shift, denoise_reference, emu, srgb8  # noqa: F401 (emu: a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
H = 32


@pytest.fixture
def gpu(built):
    """(RenderCUDA, OracleBackend, primary_rays) with RenderCUDA bound to libcrt_cuda_core.so, also while the module's
    `emu` fixture (which rebinds it to the emulated renderer) is alive in the same session."""
    import chameleonrt_b200.backend as backend
    from oracle import OracleBackend
    from oracle.oracle import primary_rays

    saved = (backend._LIB_PATH, backend._lib)
    backend._LIB_PATH, backend._lib = os.path.join(ROOT, "chameleonrt_b200", "csrc", "libcrt_cuda_core.so"), None
    yield backend.RenderCUDA, OracleBackend, primary_rays
    backend._LIB_PATH, backend._lib = saved


# ---- scenes and cameras ----
def wall_scene(spp=1, box=False):
    """A fronto-parallel wall at z = 0 filling the view of `wall_camera`; with `box`, a box in front of it."""
    from chameleonrt_b200.scene import DisneyMaterial, Instance, Mesh, ParameterizedMesh, Scene, default_obj_light
    from chameleonrt_b200.scenes import MeshBuilder
    from chameleonrt_b200.scenes import box as box_parts
    from chameleonrt_b200.scenes import grid

    geoms = []
    b = MeshBuilder()
    b.add(*grid((-20, -20, 0), (40, 0, 0), (0, 40, 0), 4, 4))
    geoms.append(b.geometry())
    mats = [DisneyMaterial(base_color=(0.7, 0.6, 0.5), roughness=0.9)]
    if box:
        b = MeshBuilder()
        for part in box_parts((-0.5, -0.5, 1.0), (0.5, 0.5, 2.0)):
            b.add(*part)
        geoms.append(b.geometry())
        mats.append(DisneyMaterial(base_color=(0.2, 0.4, 0.8), roughness=0.7))
    return Scene(meshes=[Mesh(geoms)], parameterized_meshes=[ParameterizedMesh(0, list(range(len(geoms))))],
                 instances=[Instance(np.eye(4, dtype=np.float32), 0)], materials=mats, textures=[], lights=[default_obj_light()],
                 samples_per_pixel=spp)


def wall_camera(shift_x=0.0, dist=4.0):
    return dict(eye=(shift_x, 0.0, dist), center=(shift_x, 0.0, 0.0), up=(0.0, 1.0, 0.0), fov_y=40.0)


def pixel_width(cam, h, dist=4.0):
    """The width of a pixel at distance `dist` along the view direction."""
    return 2.0 * np.tan(np.radians(cam["fov_y"] * 0.5)) * dist / h


def orbit(cam, degrees):
    """`cam` with its eye rotated about the vertical axis through its centre."""
    e, c = np.asarray(cam["eye"], np.float64), np.asarray(cam["center"], np.float64)
    a = np.radians(degrees)
    d = e - c
    d = np.array([np.cos(a) * d[0] + np.sin(a) * d[2], d[1], -np.sin(a) * d[0] + np.cos(a) * d[2]])
    return dict(cam, eye=tuple(c + d))


# ---- the definition, restated (include/crt_cuda.h, crtc_denoise, steps a-e) ----
def view_params(cam, w, h):
    """make_view_params (kernels.cuh) in float32: pos, du, dv, tl."""
    args = _args(cam)
    pos, d, up = (np.asarray(v, f32) for v in args[:3])
    fovy = f32(args[3])

    def normalize(v):
        inv = f32(1.0) / np.sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2])
        return v * inv

    def cross(a, b):
        return np.array([a[1] * b[2] - b[1] * a[2], a[2] * b[0] - b[2] * a[0], a[0] * b[1] - b[0] * a[1]], f32)

    plane_y = f32(2.0) * f32(np.tan(np.float64((f32(0.5) * fovy) * f32(0.01745329251994329576923690768489))))
    plane_x = plane_y * f32(w) / f32(h)
    du = normalize(cross(d, up)) * plane_x
    dv = -normalize(cross(du, d)) * plane_y
    tl = d - f32(0.5) * du - f32(0.5) * dv
    return pos, du, dv, tl


def inverse_basis(du, dv, tl):
    """The adjugate over the determinant in double (AovState::history_view), rounded to float; row-major."""
    m = np.stack([du, dv, tl], 1).astype(np.float64)
    det = (m[0, 0] * (m[1, 1] * m[2, 2] - m[1, 2] * m[2, 1]) - m[0, 1] * (m[1, 0] * m[2, 2] - m[1, 2] * m[2, 0])
           + m[0, 2] * (m[1, 0] * m[2, 1] - m[1, 1] * m[2, 0]))
    inv = [(m[1, 1] * m[2, 2] - m[1, 2] * m[2, 1]) / det, (m[0, 2] * m[2, 1] - m[0, 1] * m[2, 2]) / det,
           (m[0, 1] * m[1, 2] - m[0, 2] * m[1, 1]) / det, (m[1, 2] * m[2, 0] - m[1, 0] * m[2, 2]) / det,
           (m[0, 0] * m[2, 2] - m[0, 2] * m[2, 0]) / det, (m[0, 2] * m[1, 0] - m[0, 0] * m[1, 2]) / det,
           (m[1, 0] * m[2, 1] - m[1, 1] * m[2, 0]) / det, (m[0, 1] * m[2, 0] - m[0, 0] * m[2, 1]) / det,
           (m[0, 0] * m[1, 1] - m[0, 1] * m[1, 0]) / det]
    return np.array(inv, f32)


def _unit_normals(n):
    ln = np.sqrt((n[..., 0] * n[..., 0] + n[..., 1] * n[..., 1]) + n[..., 2] * n[..., 2])
    return np.where(ln[..., None] > 0, n / np.where(ln > 0, ln, f32(1.0))[..., None], f32(0.0)).astype(f32)


def _depth_grad(Z):
    def grad(axis):
        size = Z.shape[axis]
        idx = np.arange(size)
        lo, hi = np.maximum(idx - 1, 0), np.minimum(idx + 1, size - 1)
        d = np.take(Z, hi, axis=axis) - np.take(Z, lo, axis=axis)
        shape = [1, 1]
        shape[axis] = size
        return np.where(((hi - lo) == 2).reshape(shape), f32(0.5) * d, d).astype(f32)

    return grad(1), grad(0)


def temporal_reference(accum, aov, samples, cam, prev, prev_cam, max_history, rel=1e-5):
    """Steps a-d. Returns (history dict as read_denoise_history gives it, n_p, near): `near` marks the pixels where a
    decision (a tap's depth or normal test, W >= 0.01) is within `rel` of its threshold."""
    h, w = aov["depth"].shape
    alb = np.maximum(aov["albedo"], f32(1e-3))
    now = np.concatenate([accum.astype(f32) / alb, aov["lum_m1"][..., None], aov["lum_m2"][..., None]], -1)
    nh = _unit_normals(aov["normal"])
    z = aov["depth"]
    N = f32(samples)
    n_p = np.zeros((h, w), f32)
    hist = np.zeros((h, w, 5), f32)
    near = np.zeros((h, w), bool)
    if prev is not None:
        pos, du, dv, tl = view_params(cam, w, h)
        ppos, pdu, pdv, ptl = view_params(prev_cam, w, h)
        mi = inverse_basis(pdu, pdv, ptl)
        ys, xs = np.mgrid[0:h, 0:w]
        px_x = (xs.astype(f32) + f32(0.5)) / f32(w)
        px_y = (ys.astype(f32) + f32(0.5)) / f32(h)
        d = np.stack([du[k] * px_x + dv[k] * px_y + tl[k] for k in range(3)], -1)
        c = f32(1.0) / np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])
        d = d * c[..., None]
        r = np.stack([(pos[k] + z * d[..., k]) - ppos[k] for k in range(3)], -1)
        al, be, ga = ((mi[3 * i] * r[..., 0] + mi[3 * i + 1] * r[..., 1]) + mi[3 * i + 2] * r[..., 2] for i in range(3))
        with np.errstate(divide="ignore", invalid="ignore"):
            sx = (al / ga) * f32(w) - f32(0.5)
            sy = (be / ga) * f32(h) - f32(0.5)
        live = (aov["coverage"] > 0) & (ga > 0) & (sx > -1) & (sx < w) & (sy > -1) & (sy < h)
        sx, sy = np.where(live, sx, f32(0.0)), np.where(live, sy, f32(0.0))
        dist = np.sqrt((r[..., 0] * r[..., 0] + r[..., 1] * r[..., 1]) + r[..., 2] * r[..., 2])
        fx0, fy0 = np.floor(sx), np.floor(sy)
        fx, fy = sx - fx0, sy - fy0
        x0, y0 = fx0.astype(np.int64), fy0.astype(np.int64)
        # (the cell of taps is not a decision: across a pixel centre the tap that leaves has weight 0)
        pz = prev["depth"]
        pn = prev["normal"]
        pgx, pgy = _depth_grad(pz)
        pvals = np.concatenate([prev["color"], prev["lum_m1"][..., None], prev["lum_m2"][..., None]], -1)
        sw = np.zeros((h, w), f32)
        sn = np.zeros((h, w), f32)
        acc = np.zeros((h, w, 5), f32)
        for t in range(4):
            qx, qy = x0 + (t & 1), y0 + (t >> 1)
            inside = live & (qx >= 0) & (qx < w) & (qy >= 0) & (qy < h)
            qxc, qyc = np.clip(qx, 0, w - 1), np.clip(qy, 0, h - 1)
            nq = pn[qyc, qxc]
            has_n = ~(nq == 0).all(-1)
            dz = np.abs(pz[qyc, qxc] - dist)
            thr = f32(0.02) * dist + f32(2.0) * (np.abs(pgx[qyc, qxc]) + np.abs(pgy[qyc, qxc]))
            dot = (nh[..., 0] * nq[..., 0] + nh[..., 1] * nq[..., 1]) + nh[..., 2] * nq[..., 2]
            ok = inside & has_n & (dz <= thr) & (dot >= f32(0.9))
            near |= inside & has_n & ((np.abs(thr - dz) <= rel * thr) | (np.abs(dot - f32(0.9)) <= rel))
            wt = ((fx if t & 1 else f32(1.0) - fx) * (fy if t >> 1 else f32(1.0) - fy)).astype(f32)
            wt = np.where(ok, wt, f32(0.0))
            sw = np.where(ok, sw + wt, sw)
            sn = np.where(ok, sn + wt * prev["count"][qyc, qxc], sn)
            acc = np.where(ok[..., None], acc + wt[..., None] * pvals[qyc, qxc], acc)
        near |= live & (np.abs(sw - f32(0.01)) <= rel * f32(0.01))
        enough = sw >= f32(0.01)
        with np.errstate(divide="ignore", invalid="ignore"):
            hist = np.where(enough[..., None], acc / sw[..., None], f32(0.0)).astype(f32)
            n_p = np.where(enough, np.minimum(f32(max_history), sn / sw), f32(0.0)).astype(f32)
    blend = n_p > 0
    n_t = np.where(blend, n_p + N, N).astype(f32)
    out = np.where(blend[..., None], (n_p[..., None] * hist + N * now) / n_t[..., None], now).astype(f32)
    cur = dict(color=out[..., 0:3], lum_m1=out[..., 3], lum_m2=out[..., 4], count=n_t, depth=z, normal=nh)
    return cur, n_p, near


def variance_moments(cur, aov, sigma_n=128.0, sigma_z=1.0):
    """Step e: the moments the variance is taken from (the 7x7 cross-bilateral mean where n < 4)."""
    nh = _unit_normals(aov["normal"])
    Z = aov["depth"]
    gx, gy = _depth_grad(Z)
    bg = (nh == 0).all(-1)
    h, w = Z.shape
    sw = np.zeros((h, w), f32)
    s1 = np.zeros((h, w), f32)
    s2 = np.zeros((h, w), f32)
    for dy in range(-3, 4):
        for dx in range(-3, 4):
            m1q, m = _shift(cur["lum_m1"], dx, dy)
            m2q, _ = _shift(cur["lum_m2"], dx, dy)
            nq, _ = _shift(nh, dx, dy)
            Zq, _ = _shift(Z, dx, dy)
            bq, _ = _shift(bg, dx, dy, fill=True)
            dot = (nh[..., 0] * nq[..., 0] + nh[..., 1] * nq[..., 1]) + nh[..., 2] * nq[..., 2]
            w_n = np.power(np.maximum(f32(0.0), dot), f32(sigma_n))
            w_n = np.where(bg | bq, np.where(bg & bq, f32(1.0), f32(0.0)), w_n)
            w_z = np.exp(-np.abs(Z - Zq) / (f32(sigma_z) * np.abs(gx * f32(dx) + gy * f32(dy)) + f32(1e-3)))
            wt = np.where(m, (w_n * w_z).astype(f32), f32(0.0))
            sw = sw + wt
            s1 = s1 + wt * m1q
            s2 = s2 + wt * m2q
    few = cur["count"] < 4
    return np.where(few, s1 / sw, cur["lum_m1"]).astype(f32), np.where(few, s2 / sw, cur["lum_m2"]).astype(f32)


def output_reference(cur, aov, **prm):
    """Steps e, 2 and 3 from the device's own history: test_aov_denoise's restatement fed I_t (remodulated), the
    moments of step e and n_t as the sample count."""
    m1, m2 = variance_moments(cur, aov, prm.get("sigma_n", 128.0), prm.get("sigma_z", 1.0))
    alb = np.maximum(aov["albedo"], f32(1e-3))
    return denoise_reference(cur["color"] * alb, dict(aov, lum_m1=m1, lum_m2=m2), cur["count"], **prm)


def _hist_close(got, want, mask, rel=1e-5):
    for k in ("color", "lum_m1", "lum_m2", "count", "depth", "normal"):
        g, e = got[k][mask], want[k][mask]
        bad = np.abs(g - e) > rel * np.abs(e) + 1e-30
        assert not bad.any(), (k, int(bad.sum()), float(np.abs(g - e).max()))


# ---- checks ----
def check_nothing_to_carry(mods, scene, cam, w, h, frames=2):
    """The first epoch (spp >= 4) and the epoch after set_scene: denoise() is bit-identical to a history-off
    renderer's; every frame's accum, img, ray counts and launches are the same with the option on."""
    RenderCUDA = mods[0]
    runs = []
    for hist in (0, H):
        r = _renderer(RenderCUDA, scene, w, h, aov=True, denoise_history=hist)
        out = []
        for f in range(frames):
            st = r.render(*_args(cam), f == 0, True)
            out.append((r.read_accum(), r.read_img().copy(), st.num_rays, r.counters()["kernel_launches"], r.denoise()))
        r.set_scene(scene)
        moved = orbit(cam, 3.0)
        for f in range(frames):
            st = r.render(*_args(moved), f == 0, True)
            out.append((r.read_accum(), r.read_img().copy(), st.num_rays, r.counters()["kernel_launches"], r.denoise()))
        runs.append(out)
    for (a0, i0, n0, k0, (rgb0, img0)), (a1, i1, n1, k1, (rgb1, img1)) in zip(*runs):
        assert np.array_equal(a0.view(np.uint32), a1.view(np.uint32)) and np.array_equal(i0, i1) and n0 == n1 and k0 == k1
        assert np.array_equal(rgb0.view(np.uint32), rgb1.view(np.uint32)) and np.array_equal(img0, img1)


def check_definition(mods, scene, cam, moved, w, h, exact_img=True):
    """Camera A for 2 frames + denoise, camera B for 1 frame + denoise: read_denoise_history() against the restated
    steps a-d, and denoise()'s output against steps e, 2, 3 fed the device's history."""
    RenderCUDA = mods[0]
    spp = scene.samples_per_pixel
    r = _renderer(RenderCUDA, scene, w, h, aov=True, denoise_history=H)
    for f in range(2):
        r.render(*_args(cam), f == 0, True)
    r.denoise()
    prev = r.read_denoise_history()
    want0, _, _ = temporal_reference(r.read_accum(), r.read_aov(), 2 * spp, cam, None, None, H)
    _hist_close(prev, want0, np.ones((h, w), bool), rel=0)  # no history yet: the frame's own values, exactly
    r.render(*_args(moved), True, True)
    accum, aov = r.read_accum(), r.read_aov()
    for prm in (dict(), dict(iterations=3, sigma_luminance=1.5, sigma_normal=16.0, sigma_depth=0.25)):
        rgb, img = r.denoise(**prm)
        got = r.read_denoise_history()
        want, n_p, near = temporal_reference(accum, aov, spp, moved, prev, cam, H)
        assert near.mean() <= 1e-3, f"{int(near.sum())} pixels within 1e-5 of a threshold"
        assert (n_p[~near] > 0).mean() >= 0.5  # the camera moved a little: most pixels carry history
        _hist_close(got, want, ~near)
        kw = dict(iterations=prm.get("iterations", 5), sigma_l=prm.get("sigma_luminance", 4.0),
                  sigma_n=prm.get("sigma_normal", 128.0), sigma_z=prm.get("sigma_depth", 1.0))
        ref = output_reference(got, aov, **kw)
        assert np.isfinite(rgb).all()
        assert (np.abs(rgb - ref) <= 1e-4 * np.abs(ref) + 1e-6).all(), (prm, float(np.abs(rgb - ref).max()))
        c = srgb8(rgb).astype(np.int64)
        g = np.stack([(img >> (8 * k)) & 0xFF for k in range(3)], axis=-1).astype(np.int64)
        assert (img >> 24 == 0xFF).all()
        assert np.array_equal(g, c) if exact_img else np.abs(g - c).max() <= 1
    return r


def check_same_camera(mods, scene, cam, w, h, frames=3):
    """camera_changed with an identical camera: n_p = min(H, n_prev) and P = prev at every covered pixel. Both epochs
    render the same frames (the seeds restart with the epoch), so their depths and normals are the same bits."""
    RenderCUDA = mods[0]
    N = f32(scene.samples_per_pixel * frames)
    r = _renderer(RenderCUDA, scene, w, h, aov=True, denoise_history=H)
    for f in range(frames):
        r.render(*_args(cam), f == 0, True)
    r.denoise()
    prev = r.read_denoise_history()
    for f in range(frames):
        r.render(*_args(cam), f == 0, True)
    r.denoise()
    got = r.read_denoise_history()
    aov = r.read_aov()
    assert np.array_equal(got["depth"], prev["depth"]) and np.array_equal(got["normal"], prev["normal"])
    cov = aov["coverage"] > 0
    assert cov.mean() > 0.5
    n_p = got["count"] - N
    assert np.allclose(n_p[cov], np.minimum(H, prev["count"][cov]), rtol=1e-5, atol=0)
    assert (n_p[~cov] == 0).all()
    for k in ("color", "lum_m1", "lum_m2"):
        now = (r.read_accum() / np.maximum(aov["albedo"], f32(1e-3))) if k == "color" else aov[k]
        col = k == "color"
        npk = n_p[..., None] if col else n_p
        # P recovered from the blend: P = (n_t I_t - N I) / n_p (the recovery itself rounds at the scale of N I / n_p)
        with np.errstate(divide="ignore", invalid="ignore"):  # (n_p = 0 off the covered pixels)
            P = ((got["count"][..., None] if col else got["count"]) * got[k] - N * now) / npk
        e = prev[k]
        # the round trip through the two cameras lands a few float ulps of the image size (well under 1e-4 pixel) off
        # the centre: a neighbour tap may get that weight, which matters where it is very different (an edge, the light)
        nb = np.zeros_like(e)
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                s, m = _shift(e, dx, dy)
                nb = np.maximum(nb, np.where(m if not col else m[..., None], np.abs(s - e), 0))
        tol = 1e-5 * np.abs(e[cov]) + 1e-4 * nb[cov] + 1e-5 * np.abs(now[cov]) * N / npk[cov] + 1e-7
        assert (np.abs(P[cov] - e[cov]) <= tol).all(), k


def check_shift(mods, w=48, h=32, k=3, box=False):
    """A fronto-parallel wall, the camera translated sideways by exactly k pixel widths at the wall's distance: interior
    pixels' history is prev shifted by k columns, the k newly exposed columns have n_p = 0; with a box in front of the
    wall, the wall pixels the box covered in the previous frame get n_p = 0."""
    RenderCUDA = mods[0]
    spp = 4
    scene = wall_scene(spp, box=box)
    cam = wall_camera()
    pw = pixel_width(cam, h)
    moved = wall_camera(shift_x=k * pw)
    r = _renderer(RenderCUDA, scene, w, h, aov=True, denoise_history=H)
    for f in range(2):
        r.render(*_args(cam), f == 0, True)
    r.denoise()
    prev = r.read_denoise_history()
    r.render(*_args(moved), True, True)
    r.denoise()
    got = r.read_denoise_history()
    aov = r.read_aov()
    N = f32(spp)
    n_p = got["count"] - N
    assert (n_p <= H).all() and (n_p >= 0).all()
    assert (n_p[:, w - k:] == 0).all()  # newly exposed on the right
    now = r.read_accum() / np.maximum(aov["albedo"], f32(1e-3))
    wall_z = 4.0
    if not box:
        inner = (slice(1, h - 1), slice(1, w - k - 1))
        assert np.allclose(n_p[inner], prev["count"][:, k:][inner], rtol=1e-4, atol=0)
        with np.errstate(divide="ignore", invalid="ignore"):  # (n_p = 0 in the newly exposed columns)
            P = (got["count"][..., None] * got["color"] - N * now) / n_p[..., None]
        e = prev["color"][:, k:][inner]
        # The AOV depth is the mean over jittered samples, not the pixel-centre ray's hit distance, so the reprojected
        # point lands a small fraction of a pixel off the column centre: allow 1/100 of a pixel times the local
        # difference to the horizontal neighbours, besides 1e-4 relative.
        pc = prev["color"][1:h - 1]
        cols = np.arange(1, w - k - 1) + k
        nb = np.maximum(np.abs(pc[:, cols + 1] - pc[:, cols]), np.abs(pc[:, cols] - pc[:, cols - 1]))
        tol = 1e-4 * np.abs(e) + 1e-2 * nb + 1e-4 * np.abs(now[inner]) * N / n_p[inner][..., None]
        assert (np.abs(P[inner] - e) <= tol).all(), float((np.abs(P[inner] - e) / np.maximum(nb, 1e-12)).max())
        return
    # the wall, now visible, where the box was in the previous frame (its 3x3 neighbourhood there all box)
    pbox = prev["depth"] < 0.9 * wall_z
    pbox_shift = np.zeros((h, w), bool)
    pbox_shift[:, :w - k] = pbox[:, k:]
    box3 = pbox_shift.copy()
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            s, m = _shift(pbox_shift, dx, dy, fill=False)
            box3 &= s | ~m
    revealed = (aov["depth"] >= 0.9 * wall_z) & box3
    assert revealed.sum() >= h // 4, int(revealed.sum())
    assert (n_p[revealed] == 0).all()
    assert (n_p[(aov["depth"] < 0.9 * wall_z)] > 0).mean() > 0.5  # the box itself keeps most of its history


def check_quality(mods, size=64, steps=8):
    """Cornell at 1 spp along 8 small orbit steps, camera_changed on every frame, denoise() after each: on the last frame
    the history-on MSE against a converged oracle frame is at most half the history-off one."""
    from chameleonrt_b200.scenes import cornell_box

    RenderCUDA, OracleBackend, _ = mods
    scene, cam = cornell_box(spp=1)
    out = {}
    for hist in (0, H):
        r = _renderer(RenderCUDA, scene, size, size, aov=True, denoise_history=hist)
        for s in range(steps):
            r.render(*_args(orbit(cam, 0.5 * s)), True, True)
            rgb, _ = r.denoise()
        out[hist] = (r.read_accum(), rgb)
        if hist:
            assert (r.read_denoise_history()["count"] <= H + 1).all()
    last = orbit(cam, 0.5 * (steps - 1))
    ref_scene, _ = cornell_box(spp=64)
    orc = OracleBackend(fast=True)
    orc.initialize(size, size)
    orc.set_scene(ref_scene)
    for f in range(16):
        orc.render(*_args(last), f == 0)
    ref = orc.read_accum()
    mse_noisy = float(np.mean((out[0][0] - ref) ** 2))
    mse_off = float(np.mean((out[0][1] - ref) ** 2))
    mse_on = float(np.mean((out[H][1] - ref) ** 2))
    assert mse_on <= 0.5 * mse_off, (mse_on, mse_off, mse_noisy)
    return mse_noisy, mse_off, mse_on


def check_errors(mods):
    from chameleonrt_b200.scenes import cornell_box

    RenderCUDA = mods[0]
    scene, cam = cornell_box(spp=1)
    r = RenderCUDA(0, denoise_history=8)
    assert r.get_option("denoise_history") == 8
    with pytest.raises(RuntimeError, match="denoise_history needs option aov"):
        r.initialize(16, 16)
    for bad in (-1, 1025):
        with pytest.raises(RuntimeError, match=r"denoise_history must be in \[0, 1024\]"):
            r.set_option("denoise_history", bad)
    r.set_option("denoise_history", 1024)
    off = _renderer(RenderCUDA, scene, 16, 16, aov=True)
    off.render(*_args(cam), True, True)
    off.denoise()
    with pytest.raises(RuntimeError, match="denoise_history is off"):
        off.read_denoise_history()
    on = _renderer(RenderCUDA, scene, 16, 16, aov=True, denoise_history=4)
    on.render(*_args(cam), True, True)
    with pytest.raises(RuntimeError, match="no crtc_denoise since the last reset"):
        on.read_denoise_history()
    on.denoise()
    assert (on.read_denoise_history()["count"] == 1).all()
    on.render(*_args(orbit(cam, 1.0)), True, True)  # a reset
    with pytest.raises(RuntimeError, match="no crtc_denoise since the last reset"):
        on.read_denoise_history()
    on.denoise()
    assert (on.read_denoise_history()["count"] <= 4 + 1).all()
    on.set_scene(scene)  # drops the history
    on.render(*_args(orbit(cam, 2.0)), True, True)
    with pytest.raises(RuntimeError, match="no crtc_denoise since the last reset"):
        on.read_denoise_history()
    on.denoise()
    assert (on.read_denoise_history()["count"] == 1).all()  # n_t = N exactly after a drop
    on.initialize(16, 16)
    on.render(*_args(cam), True, True)
    on.denoise()
    assert (on.read_denoise_history()["count"] == 1).all()


def check_moving_camera_invariants(mods, scene, cam, w, h, steps, depth=5):
    """A camera path with history on: finite outputs, 0 <= n_p <= H, n_t = n_p + N."""
    RenderCUDA = mods[0]
    spp = scene.samples_per_pixel
    r = _renderer(RenderCUDA, scene, w, h, depth=depth, aov=True, denoise_history=H)
    carried = 0.0
    for s in range(steps):
        r.render(*_args(orbit(cam, 0.25 * s)), True, True)
        rgb, img = r.denoise()
        hist = r.read_denoise_history()
        n_p = hist["count"] - f32(spp)
        assert np.isfinite(rgb).all() and all(np.isfinite(v).all() for v in hist.values())
        assert (n_p >= 0).all() and (n_p <= H).all()
        carried = float((n_p > 0).mean())
    assert carried > 0.5
    return carried


# ---- CPU: the emulated renderer ----
def test_history_changes_nothing_without_history_on_the_emulated_renderer(emu):
    from chameleonrt_b200.scenes import cornell_box

    check_nothing_to_carry(emu, *cornell_box(spp=4), 40, 24)


@pytest.mark.parametrize("spp", [1, 4])
def test_history_matches_its_definition_on_the_emulated_renderer(emu, spp):
    from helpers import synthetic_material_scene

    scene, cam = synthetic_material_scene(spp=spp)
    check_definition(emu, scene, cam, orbit(cam, 1.5), 48, 32)


def test_history_same_camera_on_the_emulated_renderer(emu):
    from chameleonrt_b200.scenes import cornell_box

    check_same_camera(emu, *cornell_box(spp=2), 40, 24)


def test_history_sideways_shift_on_the_emulated_renderer(emu):
    check_shift(emu)


def test_history_disocclusion_on_the_emulated_renderer(emu):
    check_shift(emu, box=True)


def test_history_quality_on_the_emulated_renderer(emu):
    check_quality(emu)


def test_history_error_paths_on_the_emulated_renderer(emu):
    check_errors(emu)


def test_history_invariants_on_the_emulated_renderer(emu):
    from chameleonrt_b200.scenes import cornell_box

    check_moving_camera_invariants(emu, *cornell_box(spp=1), 40, 24, 4)


def test_plugin_denoise_history_variable_on_the_emulated_core(emu, tmp_path):
    """`crt_headless cuda_simt` with CRT_CUDA_DENOISE=1 CRT_CUDA_DENOISE_HISTORY=8 writes Python's denoise() of the same
    frames with the same option; the variable without CRT_CUDA_DENOISE is refused."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "simt_emu"))
    import build as simt_build
    from test_reference_plugin import HEADLESS, run_headless

    if not os.path.exists(HEADLESS) or simt_build.build_plugin() is None:
        pytest.skip("needs oracle/_ref (built where the reference sources are)")
    Image = pytest.importorskip("PIL.Image")
    from chameleonrt_b200.obj_io import write_obj
    from chameleonrt_b200.scenes import cornell_box

    w, h, frames = 64, 48, 2
    scene, cam = cornell_box(spp=1)
    obj = write_obj(scene, str(tmp_path / "scene.obj"))
    env = {"CRT_CUDA_DENOISE": "1", "CRT_CUDA_DENOISE_HISTORY": "8"}
    accum, v, _ = run_headless("cuda_simt", obj, cam, w, h, 1, frames, tmp_path, extra_env=env)
    png = np.asarray(Image.open(tmp_path / "chameleonrt.png").convert("RGBA"), np.uint32)
    png = png[..., 0] | (png[..., 1] << 8) | (png[..., 2] << 16) | (png[..., 3] << 24)
    r = _renderer(emu[0], scene, w, h, aov=True, denoise_history=8)
    for f in range(frames):
        r.render(v[0:3], v[3:6], v[6:9], v[9], f == 0, True)
    assert np.array_equal(r.read_accum().view(np.uint32), accum.view(np.uint32))
    assert np.array_equal(r.denoise()[1], png)
    with pytest.raises(AssertionError, match="CRT_CUDA_DENOISE"):
        run_headless("cuda_simt", obj, cam, w, h, 1, 1, tmp_path, extra_env={"CRT_CUDA_DENOISE_HISTORY": "8"})


# ---- GPU: libcrt_cuda_core.so on the H100 ----
@pytest.mark.gpu
def test_history_changes_nothing_without_history(gpu):
    from chameleonrt_b200.scenes import sponza_like

    check_nothing_to_carry(gpu, *sponza_like(spp=4, detail=0.3, tex_size=64), 320, 180)


@pytest.mark.gpu
@pytest.mark.parametrize("spp", [1, 4])
def test_history_matches_its_definition(gpu, spp):
    from chameleonrt_b200.scenes import sponza_like

    scene, cam = sponza_like(spp=spp, detail=0.3, tex_size=64)
    check_definition(gpu, scene, cam, orbit(cam, 1.0), 320, 180, exact_img=False)


@pytest.mark.gpu
def test_history_same_camera(gpu):
    from chameleonrt_b200.scenes import cornell_box

    check_same_camera(gpu, *cornell_box(spp=2), 130, 70)


@pytest.mark.gpu
def test_history_sideways_shift(gpu):
    check_shift(gpu, 256, 144, k=5)


@pytest.mark.gpu
def test_history_disocclusion(gpu):
    check_shift(gpu, 256, 144, k=5, box=True)


@pytest.mark.gpu
def test_history_quality(gpu):
    check_quality(gpu)


@pytest.mark.gpu
def test_history_error_paths(gpu):
    check_errors(gpu)


@pytest.mark.gpu
def test_history_c2_camera_path(gpu):
    """C2's scene at 1280x720, 1 spp, 8 steps of a camera path with history on."""
    from chameleonrt_b200.scenes import sponza_like

    check_moving_camera_invariants(gpu, *sponza_like(spp=1), 1280, 720, 8, depth=8)
