"""Per-launch times of one frame of a bench workload, and what the compiler made of k_shade.

    python scripts/profile_frame_launches.py [--workload c2] [--frames 5] [--out FILE.md]

GPU part: W warm-up frames, then F frames under torch.profiler with CUDA activities (a run of its own: no other
timing is taken while it traces). Every kernel of a frame is listed in launch order (raygen, primary traversal,
then shade / traversal / NEE resolve per bounce, resolve: 27 launches at depth 8), with the median and the spread of
its duration over the F frames, followed by the per-kernel sums. The card's name, power limit and maximum SM clock
are read with nvidia-smi in the same run and written beside the numbers.

Build part (no GPU needed): registers, stack and spill bytes of every k_shade instantiation from the ptxas report
the Makefile keeps (chameleonrt_b200/csrc/ptxas_info.txt), and their SASS instruction counts from cuobjdump of
libcrt_cuda_core.so. `--build-only` prints just that part.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CSRC = os.path.join(ROOT, "chameleonrt_b200", "csrc")

SHADE_KERNELS = {"_ZN3crt7k_shadeILb0EEEvNS_11DeviceSceneENS_9PathStateEPKjPjii": "k_shade<false> (software bilinear, default)",
                 "_ZN3crt7k_shadeILb1EEEvNS_11DeviceSceneENS_9PathStateEPKjPjii": "k_shade<true> (hw_textures)"}


def ptxas_report(path):
    """{mangled name: {registers, stack, spill_stores, spill_loads}} from `nvcc -Xptxas -v` output."""
    out, cur = {}, None
    for line in open(path):
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1)
            out[cur] = {}
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            out[cur].update(stack=int(m.group(1)), spill_stores=int(m.group(2)), spill_loads=int(m.group(3)))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            out[cur]["registers"] = int(m.group(1))
    return out


def sass_counts(lib):
    """{mangled name: SASS instruction count} from cuobjdump -sass, or {} where cuobjdump is not found."""
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        return {}
    txt = subprocess.run([exe, "-sass", lib], capture_output=True, text=True, check=True).stdout
    out = {}
    for block in re.split(r"\n\s*Function : ", txt)[1:]:
        name = block.split("\n", 1)[0].strip()
        out[name] = len(re.findall(r"^\s+/\*[0-9a-f]{4,}\*/\s+\S", block, re.M))
    return out


def build_table():
    report = ptxas_report(os.path.join(CSRC, "ptxas_info.txt"))
    sass = sass_counts(os.path.join(CSRC, "libcrt_cuda_core.so"))
    rows = ["| kernel | SASS instructions | registers | stack B | spill stores B | spill loads B |", "|---|---:|---:|---:|---:|---:|"]
    for mangled, label in SHADE_KERNELS.items():
        p = report.get(mangled, {})
        rows.append(f"| `{label}` | {sass.get(mangled, 'n/a')} | {p.get('registers', 'n/a')} | {p.get('stack', 'n/a')} | "
                    f"{p.get('spill_stores', 'n/a')} | {p.get('spill_loads', 'n/a')} |")
    return "\n".join(rows)


def gpu_description():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm,driver_version",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q or "nvidia-smi gave no answer"


def short_name(kernel):
    m = re.search(r"crt::(k_\w+)(<[^(]*>)?", kernel)
    return (m.group(1) + (m.group(2) or "")) if m else kernel[:60]


def profile_frames(workload, warmup, frames):
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    from chameleonrt_b200 import RenderCUDA

    bench.select_workload(workload)
    scene, view = bench.make_workload()
    gpu = RenderCUDA(0, max_depth=bench.MAX_DEPTH)
    gpu.set_option("stage_events", 0)
    gpu.initialize(bench.WIDTH, bench.HEIGHT)
    gpu.set_scene(scene)
    f = 0
    for _ in range(warmup):
        gpu.render(*view, f == 0, False)
        f += 1
    torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        trace = os.path.join(tmp, "frames.pt.trace.json")
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(frames):
                gpu.render(*view, f == 0, False)
                f += 1
            torch.cuda.synchronize()
        prof.export_chrome_trace(trace)
        events = json.load(open(trace))["traceEvents"]
    kernels = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    # one frame = from one k_raygen up to the next
    starts = [i for i, e in enumerate(kernels) if "k_raygen" in e["name"]]
    per_frame = [kernels[a:b] for a, b in zip(starts, starts[1:] + [len(kernels)])]
    n = len(per_frame[0])
    if len(per_frame) != frames or any(len(p) != n for p in per_frame):
        raise RuntimeError(f"expected {frames} frames of equal launch count, got {[len(p) for p in per_frame]}")
    dur = np.array([[e["dur"] for e in p] for p in per_frame], np.float64)  # [frame, launch] in us
    names = [short_name(e["name"]) for e in per_frame[0]]
    frame_us = np.array([p[-1]["ts"] + p[-1]["dur"] - p[0]["ts"] for p in per_frame])
    return names, dur, frame_us, bench.WORKLOAD


def gpu_table(names, dur, frame_us):
    import numpy as np

    med = np.median(dur, axis=0)
    rows = ["| # | kernel | bounce | median us | min us | max us |", "|---:|---|---:|---:|---:|---:|"]
    bounce = -1
    for i, name in enumerate(names):
        if name.startswith("k_shade"):
            bounce += 1
        b = "" if name.startswith(("k_raygen", "k_resolve")) or bounce < 0 else str(bounce)
        rows.append(f"| {i + 1} | `{name}` | {b} | {med[i]:.1f} | {dur[:, i].min():.1f} | {dur[:, i].max():.1f} |")
    rows += ["", "| kernel | launches per frame | median ms per frame | share of kernel time |", "|---|---:|---:|---:|"]
    per_frame_total = np.sum(dur, axis=1)
    total_med = float(np.median(per_frame_total))
    for name in dict.fromkeys(names):
        idx = [i for i, x in enumerate(names) if x == name]
        ms = float(np.median(np.sum(dur[:, idx], axis=1))) / 1e3
        rows.append(f"| `{name}` | {len(idx)} | {ms:.3f} | {100 * ms * 1e3 / total_med:.1f} % |")
    rows.append(f"| all kernels | {len(names)} | {total_med / 1e3:.3f} | 100 % |")
    rows += ["", f"Frame span (first kernel start to last kernel end, median of {dur.shape[0]} frames): "
                 f"{float(np.median(frame_us)) / 1e3:.3f} ms."]
    return "\n".join(rows)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c2")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", type=int, default=5)
    ap.add_argument("--label", default="", help="a line written under the heading (what build this is)")
    ap.add_argument("--out", default=None, help="write the markdown here (default: stdout)")
    ap.add_argument("--build-only", action="store_true")
    args = ap.parse_args()
    parts = [f"# Per-launch times, {args.workload}", ""]
    if args.label:
        parts += [args.label, ""]
    if not args.build_only:
        names, dur, frame_us, workload = profile_frames(args.workload, args.warmup, args.frames)
        parts += [f"Workload: {workload}.", "",
                  f"GPU (nvidia-smi: name, power limit, max SM clock, driver): {gpu_description()}.", "",
                  f"torch.profiler (CUDA activities), {args.frames} frames after {args.warmup} warm-up frames, one blocking "
                  "render() per frame, stage events off.", "", gpu_table(names, dur, frame_us), ""]
    parts += ["## k_shade as compiled (ptxas -v, cuobjdump -sass)", "", build_table(), ""]
    text = "\n".join(parts)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(text)
    print(text)


if __name__ == "__main__":
    main()
