"""Cost and benefit of adaptive sampling (crtc_set_adaptive) on the GPU (CUDA device required; there is no CPU fallback).

On C2 (sponza_like, 1280x720, 4 spp, depth 8), blocking crtc_render calls, device frame times from crtc_get_stage_times [6]:
  * overhead: ms/frame with the mode off and on with every block active (min_frames above the frames rendered), windows
    alternated, after warm-up;
  * MSE against a converged uniform frame vs cumulative device time, uniform and several thresholds (min_frames 4). The
    converged frame is the mean of uniform frames K+1 .. K+M (K = --calls, M = --ref-frames; 4 * M >= 1024 samples),
    recovered from the running means after K and K+M frames, so that it shares no sample with the compared frames;
  * the frame time once every block has converged (threshold 1e30 after min_frames).

Prints a markdown report with the card's name and power limit, and writes it to --out when given.

    python scripts/bench_adaptive.py --out profiles/adaptive_h100.md
"""
import argparse
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
    ap.add_argument("--frames", type=int, default=20, help="frames per overhead window")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--calls", type=int, default=64, help="render calls per MSE curve")
    ap.add_argument("--ref-frames", type=int, default=256)
    ap.add_argument("--thresholds", default="0.01,0.03,0.1,0.3")
    ap.add_argument("--width", type=int, default=1280)
    ap.add_argument("--height", type=int, default=720)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_adaptive.py needs a CUDA device")
    from chameleonrt_b200 import ArcballCamera, RenderCUDA
    from chameleonrt_b200.scenes import sponza_like

    name, power = card()
    scene, cam = sponza_like(spp=4)
    spp = scene.samples_per_pixel
    c = ArcballCamera(cam["eye"], cam["center"], cam["up"])
    view = (c.eye(), c.dir(), c.up(), cam["fov_y"])
    w, h = args.width, args.height

    def renderer():
        r = RenderCUDA(0, max_depth=8)
        r.initialize(w, h)
        r.set_scene(scene)
        return r

    # ---- overhead of the selection launch and the moment writes, every block active ----
    rs = {"off": renderer(), "on, all active": renderer()}
    rs["on, all active"].set_adaptive(0.0, min_frames=1 << 30)
    for r in rs.values():
        for f in range(args.warmup):
            r.render(*view, f == 0, True)
    frame_ms = {k: [] for k in rs}
    for _ in range(args.runs):
        for k, r in rs.items():
            total = 0.0
            for _f in range(args.frames):
                r.render(*view, False, True)
                total += r.stage_times()["frame"]
            frame_ms[k].append(total / args.frames)
    del rs

    # ---- the converged frame ----
    K, M = args.calls, args.ref_frames
    r = renderer()
    for f in range(K):
        r.render_async(*view, f == 0, 1)
    r.sync()
    a_k = r.read_accum().astype(np.float64)
    left = M
    while left:
        n = min(left, 16)
        r.render_async(*view, False, n)
        r.sync()
        left -= n
    ref = (((K + M) * r.read_accum().astype(np.float64) - K * a_k) / M).astype(np.float32)
    del r

    # ---- MSE vs cumulative device time ----
    checkpoints = sorted({x for x in (1, 2, 4, 8, 12, 16, 24, 32, 48, 64, K) if x <= K})
    curves = {}
    for thr in [None] + [float(t) for t in args.thresholds.split(",")]:
        r = renderer()
        if thr is not None:
            r.set_adaptive(thr, min_frames=4)
        t, rows = 0.0, []
        for call in range(1, K + 1):
            r.render(*view, call == 1, True)
            t += r.stage_times()["frame"]
            if call in checkpoints:
                acc = r.read_accum()
                samples = float(np.mean(r.read_adaptive()["samples"])) if thr is not None else float(call * spp)
                rows.append((call, t, samples, float(np.mean((acc - ref) ** 2))))
        curves["uniform" if thr is None else f"threshold {thr:g}"] = rows
        del r

    # ---- frame time once every block has converged ----
    r = renderer()
    r.set_adaptive(1e30, min_frames=4)
    for f in range(4 + args.warmup):
        r.render(*view, f == 0, True)
    conv = []
    for _f in range(args.frames):
        r.render(*view, False, True)
        conv.append(r.stage_times()["frame"])
    conv_counters = r.counters()
    del r

    lines = [f"# Adaptive sampling on {name} (power limit {power})", "",
             f"`python scripts/bench_adaptive.py` on C2 (sponza_like, {w}x{h}, {spp} spp, depth 8), blocking `crtc_render` "
             "calls, device frame time = crtc_get_stage_times [6].", "",
             f"## Overhead with every block active ({args.frames} frames per window, {args.runs} alternated windows, "
             f"{args.warmup} warm-up frames)", "",
             "| window | " + " | ".join(f"{k} (ms/frame)" for k in frame_ms) + " |", "|---|" + "---|" * len(frame_ms)]
    for i in range(args.runs):
        lines.append(f"| {i + 1} | " + " | ".join(f"{frame_ms[k][i]:.3f}" for k in frame_ms) + " |")
    m = {k: float(np.mean(v)) for k, v in frame_ms.items()}
    lines.append("| mean | " + " | ".join(f"{m[k]:.3f}" for k in frame_ms) + " |")
    lines += ["", f"Added by the mode: {m['on, all active'] - m['off']:+.3f} ms/frame "
              f"({100 * (m['on, all active'] / m['off'] - 1):+.1f} %).", "",
              f"## MSE against a converged uniform frame ({M * spp} spp, no sample shared) vs cumulative device time", "",
              "min_frames 4. Samples = mean samples per pixel.", "",
              "| variant | calls | device ms (cumulative) | samples | MSE |", "|---|---|---|---|---|"]
    for k, rows in curves.items():
        for call, t, s, e in rows:
            lines.append(f"| {k} | {call} | {t:.1f} | {s:.1f} | {e:.6f} |")
    # equal device time: each adaptive curve's last point against the uniform curve interpolated (in log MSE) at its time
    uni = curves["uniform"]
    ut, ue = np.array([x[1] for x in uni]), np.log(np.array([x[3] for x in uni]))
    lines += ["", "## At equal device time", "", "| variant | device ms | MSE | uniform MSE at that time | ratio |",
              "|---|---|---|---|---|"]
    for k, rows in curves.items():
        if k == "uniform":
            continue
        for call, t, s, e in rows:
            if ut[0] <= t <= ut[-1]:
                u = float(np.exp(np.interp(t, ut, ue)))
                lines.append(f"| {k} (call {call}) | {t:.1f} | {e:.6f} | {u:.6f} | {e / u:.3f} |")
    lines += ["", f"## Every block converged (threshold 1e30 after 4 frames)", "",
              f"{float(np.mean(conv)):.3f} ms/frame (min {float(np.min(conv)):.3f}), against {m['off']:.3f} ms/frame "
              f"uniform; paths started per frame: {conv_counters['paths']}, launches {conv_counters['kernel_launches']}."]
    text = "\n".join(lines) + "\n"
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
