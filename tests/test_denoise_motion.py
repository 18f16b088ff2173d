"""The denoiser's history through moving geometry (option "denoise_motion"; crtc_commit_scene, crtc_denoise;
chameleonrt_b200/csrc/aov_denoise.cuh: k_aov_hit, k_dn_temporal<true>).

Every check runs on the emulated renderer (tests/simt_emu) without a GPU and on libcrt_cuda_core.so on an H100 (``-m gpu``):
  * nothing changes with the option off or nothing moving: camera-only epochs are bit-identical to option off (accum,
    img, ray counts, history, denoised output; launches grow by one on an epoch's first wavefront only), and an identity
    commit follows the static definition; the frames after a commit that keeps the history draw new samples;
  * the history against a numpy float32 restatement of its definition (include/crt_cuda.h, crtc_denoise, step b'), with
    each pixel's first hit traced again with trace_closest, for an instance translation, an instance rotation and a
    vertex deformation;
  * geometry, independent of the restatement: a box moved sideways by k pixel widths in front of a wall;
  * light changes still drop the history; error paths;
  * quality: a Cornell box at 1 spp with one box moving and the camera still, the denoised output against a converged
    frame.
"""
import copy

import numpy as np
import pytest

from test_aov_denoise import _args, _renderer, _shift, emu  # noqa: F401 (emu: a fixture)
from test_denoise_history import (H, _depth_grad, _hist_close, _unit_normals, gpu, inverse_basis, orbit,  # noqa: F401
                                  pixel_width, view_params, wall_camera, wall_scene)

f32 = np.float32
MISS = 0xFFFFFFFF


# ---- scenes ----
def two_instance_scene(spp=1):
    """`wall_scene(box=True)` with the box as its own mesh and instance (instance 1, identity)."""
    from chameleonrt_b200.scene import Instance, Mesh, ParameterizedMesh

    s = wall_scene(spp, box=True)
    wall, box = s.meshes[0].geometries
    s.meshes = [Mesh([wall]), Mesh([box])]
    s.parameterized_meshes = [ParameterizedMesh(0, [0]), ParameterizedMesh(1, [1])]
    s.instances = [Instance(np.eye(4, dtype=f32), 0), Instance(np.eye(4, dtype=f32), 1)]
    return s


def moving_cornell(spp=1):
    """cornell_box plus a small white box as its own mesh and instance (instance 1)."""
    from chameleonrt_b200.scene import Instance, Mesh, ParameterizedMesh
    from chameleonrt_b200.scenes import MeshBuilder, box, cornell_box

    s, cam = cornell_box(spp)
    b = MeshBuilder()
    for part in box((-0.15, 0.0, 0.3), (0.15, 0.3, 0.6)):
        b.add(*part)
    s.meshes.append(Mesh([b.geometry()]))
    s.parameterized_meshes.append(ParameterizedMesh(len(s.meshes) - 1, [0]))
    s.instances.append(Instance(np.eye(4, dtype=f32), len(s.parameterized_meshes) - 1))
    return s, cam


def translation(x, y=0.0, z=0.0):
    t = np.eye(4, dtype=f32)
    t[:3, 3] = (x, y, z)
    return t


def rotation_y(degrees, centre):
    a = np.radians(degrees)
    c, s = np.cos(a), np.sin(a)
    r = np.array([[c, 0, s, 0], [0, 1, 0, 0], [-s, 0, c, 0], [0, 0, 0, 1]], np.float64)
    t, ti = np.eye(4), np.eye(4)
    t[:3, 3], ti[:3, 3] = centre, -np.asarray(centre)
    return (t @ r @ ti).astype(f32)


# ---- the scene's flattened triangles, restated (dev_flatten_triangle) ----
def flattened(scene):
    """World vertices (T, 3, 3) and shading normals (T, 3) of every flattened triangle, in flattened order, with the
    device's float32 operation order for the vertices."""
    ws, ns = [], []
    for inst in scene.instances:
        m = np.asarray(inst.transform, f32)
        w2o = np.linalg.inv(m.astype(np.float64)).astype(f32)
        pm = scene.parameterized_meshes[inst.parameterized_mesh_id]
        for g in scene.meshes[pm.mesh_id].geometries:
            v = np.asarray(g.vertices, f32)[np.asarray(g.indices, np.int64)]  # (nt, 3, 3)
            w = np.stack([((m[r, 0] * v[..., 0] + m[r, 1] * v[..., 1]) + m[r, 2] * v[..., 2]) + m[r, 3] for r in range(3)], -1)
            e1, e2 = v[:, 1] - v[:, 0], v[:, 2] - v[:, 0]
            n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                          e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], -1)
            n = n / np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])[:, None]
            n = np.stack([(w2o[0, r] * n[:, 0] + w2o[1, r] * n[:, 1]) + w2o[2, r] * n[:, 2] for r in range(3)], -1)
            n = n / np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])[:, None]
            ws.append(w.astype(f32))
            ns.append(n.astype(f32))
    return np.concatenate(ws), np.concatenate(ns)


def first_hits(r, primary_rays, cam, w, h, spp, frame_id):
    """Each pixel's hit record: the flat id, u, v of the first sample of the epoch's first frame that hit (trace_closest
    of the same primary rays; `frame_id` is the frame index its samples were drawn for), flat id MISS where none did."""
    fid = np.full(h * w, MISS, np.uint32)
    uv = np.zeros((h * w, 2), f32)
    for s in range(spp):
        hits = r.trace_closest(primary_rays(w, h, *_args(cam), frame_id=frame_id, spp=spp, s=s))
        prim = hits[:, 3].view(np.uint32)
        take = (fid == MISS) & (prim != MISS)
        fid[take] = prim[take]
        uv[take] = hits[take, 1:3]
    return fid.reshape(h, w), uv.reshape(h, w, 2)


def bary_point(wt, b1, b2):
    return np.stack([(wt[..., 0, k] + b1 * (wt[..., 1, k] - wt[..., 0, k])) + b2 * (wt[..., 2, k] - wt[..., 0, k])
                     for k in range(3)], -1)


def motion_reference(accum, aov, samples, cam, prev, prev_cam, max_history, fid, uv, cur_scene, prev_scene, rel=1e-5):
    """crtc_denoise steps a-d with step b': test_denoise_history.temporal_reference plus the displacement of each
    pixel's recorded triangle. Returns (history, n_p, near, moved)."""
    h, w = aov["depth"].shape
    alb = np.maximum(aov["albedo"], f32(1e-3))
    now = np.concatenate([accum.astype(f32) / alb, aov["lum_m1"][..., None], aov["lum_m2"][..., None]], -1)
    nh = _unit_normals(aov["normal"])
    z = aov["depth"]
    N = f32(samples)
    pos, du, dv, tl = view_params(cam, w, h)
    ppos, pdu, pdv, ptl = view_params(prev_cam, w, h)
    mi = inverse_basis(pdu, pdv, ptl)
    ys, xs = np.mgrid[0:h, 0:w]
    px_x = (xs.astype(f32) + f32(0.5)) / f32(w)
    px_y = (ys.astype(f32) + f32(0.5)) / f32(h)
    d = np.stack([du[k] * px_x + dv[k] * px_y + tl[k] for k in range(3)], -1)
    c = f32(1.0) / np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])
    d = d * c[..., None]
    X = np.stack([pos[k] + z * d[..., k] for k in range(3)], -1)
    # step b': the recorded triangle over the live and the previous geometry
    wc, nc = flattened(cur_scene)
    wp, np_ = flattened(prev_scene)
    rec = fid != MISS
    t = np.where(rec, fid, 0).astype(np.int64)
    moved = rec & ~(wc[t].view(np.uint32) == wp[t].view(np.uint32)).reshape(h, w, 9).all(-1)
    with np.errstate(invalid="ignore", over="ignore"):
        dp = bary_point(wp[t], uv[..., 0], uv[..., 1]) - bary_point(wc[t], uv[..., 0], uv[..., 1])
        finite = np.isfinite(dp).all(-1)
        X = np.where(moved[..., None], X + dp, X)
    side = np.where(((nh[..., 0] * nc[t][..., 0] + nh[..., 1] * nc[t][..., 1]) + nh[..., 2] * nc[t][..., 2]) < 0, f32(-1.0), f32(1.0))
    nref = np.where(moved[..., None], side[..., None] * np_[t], nh)
    r = np.stack([X[..., k] - ppos[k] for k in range(3)], -1)
    al, be, ga = ((mi[3 * i] * r[..., 0] + mi[3 * i + 1] * r[..., 1]) + mi[3 * i + 2] * r[..., 2] for i in range(3))
    with np.errstate(divide="ignore", invalid="ignore"):
        sx = (al / ga) * f32(w) - f32(0.5)
        sy = (be / ga) * f32(h) - f32(0.5)
    live = (aov["coverage"] > 0) & (~moved | finite) & (ga > 0) & (sx > -1) & (sx < w) & (sy > -1) & (sy < h)
    sx, sy = np.where(live, sx, f32(0.0)), np.where(live, sy, f32(0.0))
    dist = np.sqrt((r[..., 0] * r[..., 0] + r[..., 1] * r[..., 1]) + r[..., 2] * r[..., 2])
    fx0, fy0 = np.floor(sx), np.floor(sy)
    fx, fy = sx - fx0, sy - fy0
    x0, y0 = fx0.astype(np.int64), fy0.astype(np.int64)
    pz, pn = prev["depth"], prev["normal"]
    pgx, pgy = _depth_grad(pz)
    pvals = np.concatenate([prev["color"], prev["lum_m1"][..., None], prev["lum_m2"][..., None]], -1)
    sw = np.zeros((h, w), f32)
    sn = np.zeros((h, w), f32)
    acc = np.zeros((h, w, 5), f32)
    near = np.zeros((h, w), bool)
    for k in range(4):
        qx, qy = x0 + (k & 1), y0 + (k >> 1)
        inside = live & (qx >= 0) & (qx < w) & (qy >= 0) & (qy < h)
        qxc, qyc = np.clip(qx, 0, w - 1), np.clip(qy, 0, h - 1)
        nq = pn[qyc, qxc]
        has_n = ~(nq == 0).all(-1)
        dz = np.abs(pz[qyc, qxc] - dist)
        thr = f32(0.02) * dist + f32(2.0) * (np.abs(pgx[qyc, qxc]) + np.abs(pgy[qyc, qxc]))
        dot = (nref[..., 0] * nq[..., 0] + nref[..., 1] * nq[..., 1]) + nref[..., 2] * nq[..., 2]
        ok = inside & has_n & (dz <= thr) & (dot >= f32(0.9))
        near |= inside & has_n & ((np.abs(thr - dz) <= rel * thr) | (np.abs(dot - f32(0.9)) <= rel))
        wt = ((fx if k & 1 else f32(1.0) - fx) * (fy if k >> 1 else f32(1.0) - fy)).astype(f32)
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
    return cur, n_p, near, moved


# ---- checks ----
def _frame(r, cam, changed):
    st = r.render(*_args(cam), changed, True)
    return r.read_accum(), r.read_img().copy(), st.num_rays, r.counters()["kernel_launches"]


def check_nothing_moves(mods, scene, cam, w, h):
    """Camera-only epochs: option on is bit-identical to option off (history, denoised rgb / img, accum, img, rays);
    launches grow by one on each epoch's first wavefront only."""
    RenderCUDA = mods[0]
    runs = []
    for motion in (False, True):
        r = _renderer(RenderCUDA, scene, w, h, aov=True, denoise_history=H, dynamic_scene=True, denoise_motion=motion)
        out = []
        for step, frames in enumerate((2, 1, 2)):
            cam_s = orbit(cam, 1.0 * step)
            for f in range(frames):
                out.append(_frame(r, cam_s, f == 0) + (f == 0,))
            rgb, img = r.denoise()
            hist = r.read_denoise_history()
            out.append((rgb, img, np.concatenate([hist[k].reshape(h, w, -1) for k in hist], -1)))
        runs.append(out)
    for a, b in zip(*runs):
        if len(a) == 5:
            assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1]) and a[2] == b[2]
            assert b[3] == a[3] + (1 if a[4] else 0), (a[3], b[3], a[4])
        else:
            assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1])
            assert np.array_equal(a[2].view(np.uint32), b[2].view(np.uint32))


def check_identity_commit(mods, scene, cam, w, h):
    """A commit of the same matrices keeps the history, and since no triangle moved, the next denoise() follows the
    static definition (test_denoise_history.temporal_reference) at every pixel. The frame after it draws new samples
    (the sample sequence goes on), while without the option it re-renders frame 0, bit for bit as a camera_changed
    frame does."""
    from test_denoise_history import temporal_reference

    RenderCUDA = mods[0]
    spp = scene.samples_per_pixel
    same = np.stack([np.asarray(i.transform, f32) for i in scene.instances])
    accum = {}
    for motion, commit in ((True, True), (True, False), (False, True), (False, False)):
        r = _renderer(RenderCUDA, scene, w, h, aov=True, denoise_history=H, dynamic_scene=True, denoise_motion=motion)
        for f in range(2):
            r.render(*_args(cam), f == 0, True)
        r.denoise()
        prev = r.read_denoise_history()
        if commit:
            r.update_instances(same)
            r.commit_scene()
        r.render(*_args(cam), not commit, True)
        r.denoise()
        accum[motion, commit] = r.read_accum()
        if motion and commit:
            got = r.read_denoise_history()
            want, n_p, near = temporal_reference(accum[motion, commit], r.read_aov(), spp, cam, prev, cam, H)
            assert near.mean() <= 1e-3 and (n_p > 0).mean() > 0.9
            _hist_close(got, want, ~near)
    assert np.array_equal(accum[False, True].view(np.uint32), accum[False, False].view(np.uint32))
    assert np.array_equal(accum[True, False].view(np.uint32), accum[False, False].view(np.uint32))
    assert not np.array_equal(accum[True, True], accum[True, False])


def check_definition(mods, scene, cam, moved_cam, w, h, move):
    """Camera A, 2 frames + denoise; `move(r, scene)` commits a geometry change and returns the moved scene; camera B,
    1 frame + denoise: the history against motion_reference."""
    RenderCUDA, _, primary_rays = mods
    spp = scene.samples_per_pixel
    r = _renderer(RenderCUDA, scene, w, h, aov=True, denoise_history=H, dynamic_scene=True, denoise_motion=True)
    for f in range(2):
        r.render(*_args(cam), f == 0, True)
    r.denoise()
    prev = r.read_denoise_history()
    moved_scene = move(r, copy.deepcopy(scene))
    r.render(*_args(moved_cam), True, True)
    r.denoise()
    got = r.read_denoise_history()
    # (the commit kept the history, so the epoch's samples continue after the 2 frames of the one before)
    fid, uv = first_hits(r, primary_rays, moved_cam, w, h, spp, frame_id=2)
    want, n_p, near, moved = motion_reference(r.read_accum(), r.read_aov(), spp, moved_cam, prev, cam, H, fid, uv,
                                              moved_scene, scene)
    assert near.mean() <= 2e-3, f"{int(near.sum())} pixels within 1e-5 of a threshold"
    assert moved.mean() >= 0.05 and (n_p[moved & ~near] > 0).mean() >= 0.5  # the moving object carries its history
    assert (n_p[~moved & ~near] > 0).mean() >= 0.5
    _hist_close(got, want, ~near)


def _move_instance(m):
    def move(r, s):
        s.instances[1].transform = m
        r.update_instances(m[None], first=1)
        r.commit_scene()
        return s
    return move


def _deform(r, s):
    g = s.meshes[1].geometries[0]
    v = np.asarray(g.vertices, f32)
    c = v.mean(0)
    g.vertices = (c + (v - c) * np.array([1.1, 0.9, 1.0], f32) + np.array([0.05, 0.0, 0.0], f32) * (v[:, 1:2] - c[1])).astype(f32)
    r.update_vertices(1, 0, g.vertices)
    r.commit_scene()
    return s


def _n_p(r, spp):
    return r.read_denoise_history()["count"] - f32(spp)


def check_box_shift(mods, w=48, h=32, k=3):
    """A box in front of a wall, the camera still, the box moved sideways by exactly k pixel widths at its front face
    (update_vertices of its geometry): box-front pixels carry prev shifted by k columns, the wall the box uncovered has
    n_p = 0, the wall never covered keeps min(H, prev count); with the option off every pixel has n_p = 0."""
    RenderCUDA = mods[0]
    spp = 4
    scene = wall_scene(spp, box=True)
    cam = wall_camera()
    front_z, wall_z = 2.0, 4.0
    shift = f32(k * pixel_width(cam, h, dist=wall_z - front_z))
    for motion in (True, False):
        r = _renderer(RenderCUDA, scene, w, h, aov=True, denoise_history=H, dynamic_scene=True, denoise_motion=motion)
        for f in range(2):
            r.render(*_args(cam), f == 0, True)
        r.denoise()
        prev = r.read_denoise_history()
        g = scene.meshes[0].geometries[1]
        r.update_vertices(0, 1, (np.asarray(g.vertices, f32) + np.array([shift, 0, 0], f32)).astype(f32))
        r.commit_scene()
        r.render(*_args(cam), False, True)
        r.denoise()
        got = r.read_denoise_history()
        n_p = got["count"] - f32(spp)
        if not motion:
            assert (n_p == 0).all()
            continue
        aov = r.read_aov()
        assert (n_p >= 0).all() and (n_p <= H).all()

        def front(hist):  # box-front pixels (no wall sample: the front is at depth 2 to 2.3) with their 3x3 neighbourhood
            f = (hist["depth"] < 2.5) & (hist["normal"][..., 2] > 0.999)
            inner = f.copy()
            for dy in (-1, 0, 1):
                for dx in (-1, 0, 1):
                    s, m = _shift(f, dx, dy, fill=False)
                    inner &= s | ~m
            return inner

        was_box = prev["depth"] < 0.9 * wall_z
        pf = np.zeros((h, w), bool)
        pf[:, k:] = front(prev)[:, :w - k]  # prev's front, k columns to the right
        box_px = front(got) & pf
        assert box_px.sum() >= 12, int(box_px.sum())
        assert np.allclose(n_p[box_px], np.minimum(H, prev["count"][:, :w - k][box_px[:, k:]]), rtol=1e-4, atol=0)
        now = r.read_accum() / np.maximum(aov["albedo"], f32(1e-3))
        with np.errstate(divide="ignore", invalid="ignore"):
            P = (got["count"][..., None] * got["color"] - f32(spp) * now) / n_p[..., None]
        e = np.zeros_like(prev["color"])
        e[:, k:] = prev["color"][:, :w - k]
        pc = prev["color"]
        nb = np.zeros_like(e)
        nb[:, k + 1:w - 1] = np.maximum(np.abs(pc[:, 2:w - k] - pc[:, 1:w - k - 1]), np.abs(pc[:, 1:w - k - 1] - pc[:, 0:w - k - 2]))
        tol = 1e-4 * np.abs(e) + 1e-2 * nb + 1e-4 * np.abs(now) * f32(spp) / np.where(n_p > 0, n_p, 1)[..., None]
        assert (np.abs(P - e) <= tol)[box_px].all()
        wall_now = aov["depth"] >= 0.9 * wall_z
        is_box = got["depth"] < 0.9 * wall_z
        ring = np.zeros((h, w), bool)  # pixels next to the box now or before (mixed samples)
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                for b in (was_box, is_box):
                    s, _ = _shift(b, dx, dy, fill=False)
                    ring |= s
        # the wall where prev had the box's front with its whole 3x3 neighbourhood (at the box's edges prev's depth
        # gradient is large enough for the static depth test to accept a tap, with or without the option)
        uncovered = wall_now & front(prev)
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                s, m = _shift(wall_now, dx, dy, fill=False)
                uncovered &= s | ~m
        assert uncovered.sum() >= 4, int(uncovered.sum())
        assert (n_p[uncovered] == 0).all()
        never = wall_now & ~ring
        assert never.mean() > 0.5
        assert np.allclose(n_p[never], np.minimum(H, prev["count"][never]), rtol=1e-4, atol=0)


def check_non_finite(mods, w=40, h=24):
    """A history written while the box's matrix was NaN: the box's pixels get no history, the wall keeps it."""
    RenderCUDA = mods[0]
    spp = 2
    scene = two_instance_scene(spp)
    cam = wall_camera()
    r = _renderer(RenderCUDA, scene, w, h, aov=True, denoise_history=H, dynamic_scene=True, denoise_motion=True)
    r.update_instances(np.full((1, 4, 4), np.nan, f32), first=1)
    r.commit_scene()
    r.render(*_args(cam), True, True)
    r.denoise()
    r.update_instances(np.eye(4, dtype=f32)[None], first=1)
    r.commit_scene()
    r.render(*_args(cam), True, True)
    r.denoise()
    n_p, depth = _n_p(r, spp), r.read_aov()["depth"]
    box = depth < 3.6
    assert box.sum() >= 10 and (n_p[box] == 0).all()
    assert (n_p[~box] > 0).mean() > 0.9


def check_lights_and_errors(mods):
    RenderCUDA = mods[0]
    scene, cam = wall_scene(1, box=True), wall_camera()
    w, h = 24, 16
    lights = list(scene.lights)
    for what in ("lights", "both"):
        r = _renderer(RenderCUDA, scene, w, h, aov=True, denoise_history=H, dynamic_scene=True, denoise_motion=True)
        r.render(*_args(cam), True, True)
        r.denoise()
        r.update_lights(lights)
        if what == "both":
            r.update_instances(translation(0.1)[None])
        r.commit_scene()
        with pytest.raises(RuntimeError, match="no crtc_denoise since the last reset"):
            r.read_denoise_history()
        r.render(*_args(cam), True, True)
        with pytest.raises(RuntimeError, match="no crtc_denoise since the last reset"):
            r.read_denoise_history()
        r.denoise()
        assert (r.read_denoise_history()["count"] == 1).all(), what  # n_t = N exactly after a drop
    # a geometry commit keeps the history; it is readable again after the next denoise only
    r.update_instances(translation(0.0)[None])
    r.commit_scene()
    with pytest.raises(RuntimeError, match="no crtc_denoise since the last reset"):
        r.read_denoise_history()
    r.render(*_args(cam), True, True)
    with pytest.raises(RuntimeError, match="no crtc_denoise since the last reset"):
        r.read_denoise_history()
    r.denoise()
    assert (r.read_denoise_history()["count"] > 1).mean() > 0.5
    # the option's rules
    r = RenderCUDA(0, aov=True, denoise_motion=True)
    assert r.get_option("denoise_motion") == 1
    with pytest.raises(RuntimeError, match="denoise_motion needs option denoise_history"):
        r.initialize(16, 16)
    for bad in (-1, 2):
        with pytest.raises(RuntimeError, match="denoise_motion must be 0 or 1"):
            r.set_option("denoise_motion", bad)
    r.set_option("denoise_motion", 0)
    assert r.get_option("denoise_motion") == 0
    # a static scene: nothing more runs, and a light commit drops the history as without the option
    launches = []
    for motion in (False, True):
        s = _renderer(RenderCUDA, scene, w, h, aov=True, denoise_history=H, denoise_motion=motion)
        s.render(*_args(cam), True, True)
        launches.append(s.counters()["kernel_launches"])
        s.denoise()
        s.update_lights(lights)
        s.commit_scene()
        s.render(*_args(cam), True, True)
        s.denoise()
        assert (s.read_denoise_history()["count"] == 1).all()
    assert launches[0] == launches[1]


def check_quality(mods, size=64, steps=8, dx=0.015):
    """Cornell at 1 spp, camera still, a small box translated by dx per commit over `steps` commits, denoise() after
    each: on the last frame the option-on denoised MSE against a converged oracle frame of the final configuration is at
    most half the option-off one. Returns the MSEs (noisy, option off, option on)."""
    RenderCUDA, OracleBackend, _ = mods
    scene, cam = moving_cornell(spp=1)
    out = {}
    for motion in (False, True):
        r = _renderer(RenderCUDA, scene, size, size, aov=True, denoise_history=H, dynamic_scene=True, denoise_motion=motion)
        for s in range(steps):
            if s:
                r.update_instances(translation(dx * s)[None], first=len(scene.instances) - 1)
                r.commit_scene()
            r.render(*_args(cam), True, True)  # (camera_changed right after a commit: the commit's epoch goes on)
            rgb, _ = r.denoise()
        out[motion] = (r.read_accum(), rgb)
    ref_scene, _ = moving_cornell(spp=64)
    ref_scene.instances[-1].transform = translation(dx * (steps - 1))
    orc = OracleBackend(fast=True)
    orc.initialize(size, size)
    orc.set_scene(ref_scene)
    for f in range(16):
        orc.render(*_args(cam), f == 0)
    ref = orc.read_accum()
    mse_noisy = float(np.mean((out[False][0] - ref) ** 2))
    mse_off = float(np.mean((out[False][1] - ref) ** 2))
    mse_on = float(np.mean((out[True][1] - ref) ** 2))
    assert mse_on <= 0.5 * mse_off, (mse_on, mse_off, mse_noisy)
    return mse_noisy, mse_off, mse_on


MOVES = {
    "translate": _move_instance(translation(0.08, 0.03)),
    "rotate": _move_instance(rotation_y(15.0, (0.0, 0.0, 1.5))),
    "deform": _deform,
}


# ---- CPU: the emulated renderer ----
def test_motion_changes_nothing_without_motion_on_the_emulated_renderer(emu):
    check_nothing_moves(emu, two_instance_scene(2), wall_camera(), 40, 24)


def test_motion_identity_commit_on_the_emulated_renderer(emu):
    check_identity_commit(emu, two_instance_scene(2), wall_camera(), 40, 24)


@pytest.mark.parametrize("move", sorted(MOVES))
def test_motion_matches_its_definition_on_the_emulated_renderer(emu, move):
    cam = wall_camera()
    check_definition(emu, two_instance_scene(2), cam, orbit(cam, 1.0), 48, 32, MOVES[move])


def test_motion_box_shift_on_the_emulated_renderer(emu):
    check_box_shift(emu)


def test_motion_non_finite_on_the_emulated_renderer(emu):
    check_non_finite(emu)


def test_motion_lights_and_errors_on_the_emulated_renderer(emu):
    check_lights_and_errors(emu)


def test_motion_quality_on_the_emulated_renderer(emu):
    print("mse noisy / option off / option on:", check_quality(emu))


# ---- GPU: libcrt_cuda_core.so on the H100 ----
@pytest.mark.gpu
def test_motion_changes_nothing_without_motion(gpu):
    check_nothing_moves(gpu, two_instance_scene(4), wall_camera(), 320, 180)


@pytest.mark.gpu
def test_motion_identity_commit(gpu):
    check_identity_commit(gpu, two_instance_scene(4), wall_camera(), 320, 180)


@pytest.mark.gpu
@pytest.mark.parametrize("move", sorted(MOVES))
def test_motion_matches_its_definition(gpu, move):
    cam = wall_camera()
    check_definition(gpu, two_instance_scene(2), cam, orbit(cam, 1.0), 256, 144, MOVES[move])


@pytest.mark.gpu
def test_motion_box_shift(gpu):
    check_box_shift(gpu, 256, 144, k=5)


@pytest.mark.gpu
def test_motion_non_finite(gpu):
    check_non_finite(gpu, 160, 96)


@pytest.mark.gpu
def test_motion_lights_and_errors(gpu):
    check_lights_and_errors(gpu)


@pytest.mark.gpu
def test_motion_quality(gpu):
    print("mse noisy / option off / option on:", check_quality(gpu))
