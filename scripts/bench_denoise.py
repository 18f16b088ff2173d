"""Cost of option "aov" and of crtc_denoise on the GPU (CUDA device required; there is no CPU fallback).

  * C2 (sponza_like, 1280x720, 4 spp, depth 8) ms per frame with aov = 0 and aov = 1, alternated, three windows each:
    the mean device frame time (crtc_get_stage_times [6]) over --frames blocking frames after --warmup frames.
  * crtc_denoise device time (K = 5, default sigmas) at 1280x720 and 1920x1080 on C2's scene: CUDA events on the
    renderer's stream around each call (no host outputs requested, so no device-to-host copy is timed), after warm-up.

Prints a markdown table with the card's name and power limit, and writes it to --out when given.

    python scripts/bench_denoise.py --out profiles/denoise_h100.md
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q or "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--denoise-iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_denoise.py needs a CUDA device")
    from chameleonrt_b200 import ArcballCamera, RenderCUDA
    from chameleonrt_b200.backend import CDenoiseParams
    from chameleonrt_b200.scenes import sponza_like

    name, power = card()
    scene, cam = sponza_like(spp=4)
    c = ArcballCamera(cam["eye"], cam["center"], cam["up"])
    view = (c.eye(), c.dir(), c.up(), cam["fov_y"])

    renderers = {}
    for aov in (0, 1):
        r = RenderCUDA(0, max_depth=8, aov=bool(aov))
        r.initialize(1280, 720)
        r.set_scene(scene)
        for f in range(args.warmup):
            r.render(*view, f == 0, True)
        renderers[aov] = r
    frame_ms = {0: [], 1: []}
    for _ in range(args.runs):
        for aov in (0, 1):
            r = renderers[aov]
            total = 0.0
            for _f in range(args.frames):
                r.render(*view, False, True)
                total += r.stage_times()["frame"]
            frame_ms[aov].append(total / args.frames)
    stages = renderers[1].stage_times()
    del renderers

    denoise_ms = {}
    history_ms = {}
    prm = CDenoiseParams(5, 4.0, 128.0, 1.0)

    def timed(r, stream):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        r._check(r.lib.crtc_denoise(r.h, C.byref(prm), None, None, None))
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1)

    for w, h in ((1280, 720), (1920, 1080)):
        stream = torch.cuda.Stream()
        r = RenderCUDA(0, max_depth=8, aov=True, stream=stream.cuda_stream)
        r.initialize(w, h)
        r.set_scene(scene)
        r.render(*view, True, True)
        for _ in range(3):
            r._check(r.lib.crtc_denoise(r.h, C.byref(prm), None, None, None))
        times = [timed(r, stream) for _ in range(args.denoise_iters)]
        denoise_ms[(w, h)] = (float(np.median(times)), float(np.min(times)))
        # denoise_history = 32 after a camera move (a history to reproject), alternated call by call with a history-off
        # renderer on the same stream and frame
        rh = RenderCUDA(0, max_depth=8, aov=True, denoise_history=32, stream=stream.cuda_stream)
        rh.initialize(w, h)
        rh.set_scene(scene)
        rh.render(*view, True, True)
        rh._check(rh.lib.crtc_denoise(rh.h, C.byref(prm), None, None, None))
        moved = ArcballCamera(tuple(np.asarray(cam["eye"]) + np.array([0.05, 0.0, 0.0])), cam["center"], cam["up"])
        rh.render(moved.eye(), moved.dir(), moved.up(), cam["fov_y"], True, True)
        for _ in range(3):
            rh._check(rh.lib.crtc_denoise(rh.h, C.byref(prm), None, None, None))
        on, off = [], []
        for _ in range(args.denoise_iters):
            on.append(timed(rh, stream))
            off.append(timed(r, stream))
        history_ms[(w, h)] = (float(np.median(off)), float(np.median(on)), float(np.min(on)))
        del r, rh

    lines = [f"# Option aov and crtc_denoise on {name} (power limit {power})", "",
             f"`python scripts/bench_denoise.py` (frames {args.frames}, warm-up {args.warmup}, {args.runs} alternated windows).", "",
             "## C2 frame time (sponza_like, 1280x720, 4 spp, depth 8)", "",
             "| window | aov = 0 (ms/frame) | aov = 1 (ms/frame) |", "|---|---|---|"]
    for i in range(args.runs):
        lines.append(f"| {i + 1} | {frame_ms[0][i]:.3f} | {frame_ms[1][i]:.3f} |")
    m0, m1 = float(np.mean(frame_ms[0])), float(np.mean(frame_ms[1]))
    lines += [f"| mean | {m0:.3f} | {m1:.3f} ({100 * (m1 / m0 - 1):+.1f} %) |", "",
              "Stage times of the last aov = 1 frame (ms): " + ", ".join(f"{k} {v:.3f}" for k, v in stages.items()), "",
              "## crtc_denoise, K = 5, default sigmas (device time, events on the renderer's stream)", "",
              "| size | median ms | min ms |", "|---|---|---|"]
    for (w, h), (med, mn) in denoise_ms.items():
        lines.append(f"| {w}x{h} | {med:.3f} | {mn:.3f} |")
    lines += ["", "## crtc_denoise with denoise_history = 32 after a camera move, K = 5, alternated call by call with "
              "history-off calls", "", "| size | history off, median ms | history on, median ms | history on, min ms | added |",
              "|---|---|---|---|---|"]
    for (w, h), (off, on, mn) in history_ms.items():
        lines.append(f"| {w}x{h} | {off:.3f} | {on:.3f} | {mn:.3f} | {on - off:+.3f} ms |")
    text = "\n".join(lines) + "\n"
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
