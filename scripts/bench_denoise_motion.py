"""The denoiser's history through moving geometry (option denoise_motion) on the GPU (CUDA device required; there is no
CPU fallback).

  * crtc_denoise (K = 5, no outputs copied back) after a commit that moved geometry (the motion branch,
    k_dn_temporal<true>, plus the snapshot copy) against after a camera_changed frame with nothing moved (the static
    branch), alternated, medians of --calls each, at 1280x720 and 1920x1080: C2 with one geometry's vertices translated
    per commit, C3 with all its instances translated. crtc_denoise returns after a stream synchronisation, so a host
    clock around it measures the device work;
  * the snapshot copy alone: a device-to-device copy of the same bytes (128 B per instance + 12 B per unique vertex),
    CUDA events, median of 20;
  * C2's interactive loop (commit a moved geometry, render one frame, denoise) in ms per iteration with the option on
    and off, three alternated windows.

Prints a markdown report with the card's name and power limit, and writes it to --out when given.

    python scripts/bench_denoise_motion.py --out profiles/denoise_motion_h100.md
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

H = 32


def renderer(w, scene, width, height, motion):
    from chameleonrt_b200 import RenderCUDA

    r = RenderCUDA(0, max_depth=w["depth"], aov=True, denoise_history=H, dynamic_scene=True, denoise_motion=motion,
                   bvh_builder="device")
    r.initialize(width, height)
    r.set_scene(scene)
    return r


def mover(key, scene):
    """A function(r, step) that stages a small move of C2's first geometry's vertices or of every C3 instance."""
    import numpy as np

    if key == "c2":
        g = scene.meshes[0].geometries[0]
        v0 = np.asarray(g.vertices, np.float32)

        def move(r, step):
            r.update_vertices(0, 0, v0 + np.float32(0.01 * (step % 2 + 1)) * np.array([1, 0, 0], np.float32))
        return move
    t0 = np.stack([np.asarray(i.transform, np.float32) for i in scene.instances])

    def move(r, step):
        t = t0.copy()
        t[:, 0, 3] += np.float32(0.01 * (step % 2 + 1))
        r.update_instances(t)
    return move


def snapshot_bytes(scene):
    verts = set()
    for i in scene.instances:
        pm = scene.parameterized_meshes[i.parameterized_mesh_id]
        for gi, g in enumerate(scene.meshes[pm.mesh_id].geometries):
            if len(g.indices):
                verts.add((pm.mesh_id, gi, len(g.vertices)))
    return 128 * len(scene.instances) + 12 * sum(n for _, _, n in verts)


def _args(cam):
    from chameleonrt_b200 import ArcballCamera

    c = ArcballCamera(cam["eye"], cam["center"], cam["up"])
    return (c.eye(), c.dir(), c.up(), cam["fov_y"])


def branch_times(key, w, scene, cam, width, height, calls):
    """Median ms of crtc_denoise on the motion branch and on the static branch, alternated."""
    import numpy as np

    r = renderer(w, scene, width, height, True)
    move = mover(key, scene)
    args = _args(cam)
    r.render(*args, True, False)
    r.denoise()
    t = {"motion": [], "static": []}
    for i in range(calls + 2):
        for kind in ("motion", "static"):
            if kind == "motion":
                move(r, i)
                r.commit_scene()
            r.render(*args, True, False)
            t0 = time.perf_counter()
            r._check(r.lib.crtc_denoise(r.h, None, None, None, None))
            dt = (time.perf_counter() - t0) * 1e3
            if i >= 2:  # (warm-up)
                t[kind].append(dt)
    return float(np.median(t["motion"])), float(np.median(t["static"]))


def copy_time(nbytes):
    import numpy as np
    import torch

    a = torch.empty(max(nbytes // 4, 1), dtype=torch.float32, device="cuda")
    b = torch.empty_like(a)
    ts = []
    for i in range(25):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        b.copy_(a)
        e1.record()
        e1.synchronize()
        if i >= 5:
            ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def loop_times(iters, windows):
    """C2 at 1280x720: ms per (commit, render, denoise) with the option on and off, alternated windows."""
    import torch
    from bench_dynamic import workload

    w, scene, cam = workload("c2")
    move = mover("c2", scene)
    args = _args(cam)
    rs = {m: renderer(w, scene, w["w"], w["h"], m) for m in (False, True)}
    out = {False: [], True: []}
    for win in range(windows + 1):
        for m in (False, True):
            r = rs[m]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(iters):
                move(r, i)
                r.commit_scene()
                r.render(*args, True, False)
                r._check(r.lib.crtc_denoise(r.h, None, None, None, None))
            dt = (time.perf_counter() - t0) * 1e3 / iters
            if win:  # (window 0 warms up)
                out[m].append(dt)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c2,c3")
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from bench_dynamic import card, workload

    if not torch.cuda.is_available():
        raise SystemExit("bench_denoise_motion: no CUDA device")
    name, power = card()
    lines = [f"# denoise_motion on {name}, power limit {power}", "",
             f"crtc_denoise, K = 5, history H = {H}, medians of {a.calls} alternated calls (ms):", "",
             "| workload | resolution | motion branch + snapshot copy | static branch | snapshot bytes | D2D copy of those bytes (ms) |",
             "|---|---|---|---|---|---|"]
    for key in a.workloads.split(","):
        w, scene, cam = workload(key)
        nb = snapshot_bytes(scene)
        ct = copy_time(nb)
        for (wd, ht) in ((1280, 720), (1920, 1080)):
            mo, st = branch_times(key, w, scene, cam, wd, ht, a.calls)
            lines.append(f"| {key.upper()} | {wd}x{ht} | {mo:.3f} | {st:.3f} | {nb} | {ct:.3f} |")
            print(lines[-1], flush=True)
    lt = loop_times(a.iters, a.windows)
    lines += ["", f"C2 at 1280x720, one commit + one frame + crtc_denoise per iteration, ms per iteration over "
              f"{a.windows} alternated windows of {a.iters}:", "",
              "| option | windows |", "|---|---|",
              "| denoise_motion 0 | " + ", ".join(f"{x:.2f}" for x in lt[False]) + " |",
              "| denoise_motion 1 | " + ", ".join(f"{x:.2f}" for x in lt[True]) + " |"]
    report = "\n".join(lines) + "\n"
    print(report)
    if a.out:
        with open(a.out, "w") as f:
            f.write(report)


if __name__ == "__main__":
    main()
