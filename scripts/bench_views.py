"""Multi-view wavefronts (crtc_render_views) against one crtc_render_async call per view, on the GPU (CUDA device required;
there is no CPU fallback).

On C2 (sponza_like, depth 8), V distinct cameras orbiting C2's camera. Per (size, spp, V), alternated windows of the same
number of views:
  * views: a renderer with option views = V, one crtc_render_views call of 1 frame per V views;
  * one call per view: a renderer with V = 1, one crtc_render_async call of 1 frame per view (camera_changed, as switching
    cameras on one renderer requires).
Each window ends with crtc_sync. Reported per view: the device time (the sum of the wavefronts' CUDA-event frame times,
crtc_sync's render_time), the host wall time of the window (enqueue to the end of the synchronise, which includes the
gaps between wavefronts) and MRays/s over the wall time; medians over the windows. Sizes: 320x180 and 640x360 at 1 spp for
V in {1, 4, 16, 64}, and V = 4 at 1280x720 4 spp.

Prints a markdown report with the card's name, power limit and SM clocks, and writes it to --out when given.

    python scripts/bench_views.py --out profiles/views_h100.md
"""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q or "unknown"


def cameras(cam, n):
    """`n` distinct views: the eye orbits the centre over 40 degrees."""
    import numpy as np

    from chameleonrt_b200.camera import view_args

    e, c = np.asarray(cam["eye"], np.float64), np.asarray(cam["center"], np.float64)
    out = []
    for k in range(n):
        a = np.radians(-20.0 + 40.0 * k / max(1, n - 1))
        d = e - c
        d = np.array([np.cos(a) * d[0] + np.sin(a) * d[2], d[1], -np.sin(a) * d[0] + np.cos(a) * d[2]])
        out.append(view_args(dict(eye=tuple(c + d), center=cam["center"], up=cam["up"], fov_y=cam["fov_y"])))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views-per-window", type=int, default=256)
    ap.add_argument("--runs", type=int, default=5, help="alternated windows per variant")
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true", help="one small configuration (a trial run)")
    args = ap.parse_args()

    import numpy as np
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_views.py needs a CUDA device")
    from chameleonrt_b200 import RenderCUDA
    from chameleonrt_b200.scenes import sponza_like

    name, clocks = card()
    configs = [(320, 180, 1, v) for v in (1, 4, 16, 64)] + [(640, 360, 1, v) for v in (1, 4, 16, 64)] + [(1280, 720, 4, 4)]
    if args.quick:
        configs = [(320, 180, 1, 4)]
    scenes = {}
    rows = []
    for w, h, spp, V in configs:
        if spp not in scenes:
            scene, cam = sponza_like(spp=spp)
            multi, single = RenderCUDA(0, max_depth=8), RenderCUDA(0, max_depth=8)
            for r in (multi, single):
                r.initialize(64, 64)
                r.set_scene(scene)
            scenes[spp] = (cam, multi, single)
        cam, multi, single = scenes[spp]
        multi.set_option("views", V)
        multi.initialize(w, h)
        single.initialize(w, h)
        cams = cameras(cam, V)
        calls = max(1, args.views_per_window // V)
        if w * h * spp >= 1280 * 720:
            calls = max(1, calls // 16)
        nviews = calls * V

        def window_views():
            for _ in range(calls):
                multi.render_views(cams, True, 1)
            return multi.sync()

        def window_single():
            for _ in range(calls):
                for c in cams:
                    single.render_async(*c, True, 1)
            return single.sync()

        res = {"views": [], "one call per view": []}
        for fn in (window_views, window_single):  # warm-up of both shapes
            fn()
        for _ in range(args.runs):
            for key, fn in (("views", window_views), ("one call per view", window_single)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                total, _, counters, n = fn()
                wall = (time.perf_counter() - t0) * 1e3
                res[key].append((total.render_time, wall, total.num_rays, counters["kernel_launches"], n))
        for key, v in res.items():
            dev = float(np.median([x[0] for x in v])) / nviews
            wall = float(np.median([x[1] for x in v])) / nviews
            rays = v[0][2] / nviews
            rows.append((w, h, spp, V, key, dev, wall, rays / (wall * 1e-3) / 1e6, v[0][3], v[0][4]))
        print(rows[-2], rows[-1], flush=True)

    lines = [f"# Multi-view wavefronts on {name} (power limit, SM clock, max SM clock: {clocks})", "",
             "`python scripts/bench_views.py` on C2 (sponza_like, depth 8, host BVH builder), V cameras orbiting C2's camera over "
             "40 degrees, default options. Per row: the same number of views in every window "
             f"({args.views_per_window} at 1 spp, {max(1, args.views_per_window // 16)} at 1280x720 4 spp), "
             f"{args.runs} windows per variant alternated after one warm-up window each; medians. Device ms = the sum of the "
             "wavefronts' CUDA-event frame times (crtc_sync), wall ms = host clock from the first enqueue to the end of "
             "crtc_sync, both per view; MRays/s over the wall time.", "",
             "| size | spp | V | variant | device ms / view | wall ms / view | MRays/s (wall) | launches / window | frames / window |",
             "|---|---|---|---|---|---|---|---|---|"]
    for w, h, spp, V, key, dev, wall, mrays, launches, n in rows:
        lines.append(f"| {w}x{h} | {spp} | {V} | {key} | {dev:.4f} | {wall:.4f} | {mrays:.0f} | {launches} | {n} |")
    lines += ["", "Speed-up of views over one call per view (wall ms / view):", ""]
    for i in range(0, len(rows), 2):
        a, b = rows[i], rows[i + 1]
        lines.append(f"- {a[0]}x{a[1]} {a[2]} spp, V = {a[3]}: {b[6] / a[6]:.2f}x (device time {b[5] / a[5]:.2f}x)")
    text = "\n".join(lines) + "\n"
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
