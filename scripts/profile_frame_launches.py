"""Per-launch times of one frame of a bench workload, and what the compiler made of k_shade and k_traverse.

    python scripts/profile_frame_launches.py [--workload c2] [--frames 5] [--out FILE.md]

GPU part: W warm-up frames, then F frames under torch.profiler with CUDA activities (a run of its own: no other
timing is taken while it traces). Every kernel of a frame is listed in launch order (raygen, primary traversal,
then shade / traversal / NEE resolve per bounce, resolve: 27 launches at depth 8), with the median and the spread of
its duration over the F frames, followed by the per-kernel sums. The card's name, power limit and maximum SM clock
are read with nvidia-smi in the same run and written beside the numbers.

Build part (no GPU needed): registers, stack and spill bytes of every k_shade and k_traverse instantiation from the
ptxas report the Makefile keeps (chameleonrt_b200/csrc/ptxas_info.txt), and their SASS instruction counts from
cuobjdump of libcrt_cuda_core.so; for the default k_traverse also where its five node loads sit and the static size of
its node phase and triangle pass. `--build-only` prints just that part.
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


TRAVERSE_DEFAULT = "_ZN3crt10k_traverseILb0ELi16ELb0EEEvNS_11DeviceSceneENS_9PathStateEPKjS4_S4_Pjij"


def traverse_label(mangled):
    """k_traverse<COUNT, DEFER, TOP> from its mangled name (the launch options that select each one in parentheses)."""
    m = re.match(r"_ZN3crt10k_traverseILb(\d)ELi(\d+)ELb(\d)E", mangled)
    count, defer, top = int(m.group(1)), int(m.group(2)), int(m.group(3))
    opts = [f"tri_pass_defer {defer}"] + (["count_traversal"] if count else []) + (["bvh_top_smem"] if top else [])
    default = " (default)" if mangled == TRAVERSE_DEFAULT else ""
    return f"k_traverse<{'true' if count else 'false'}, {defer}, {'true' if top else 'false'}>{default}: {', '.join(opts)}"


def sass_listing(lib):
    """{mangled name: [(offset, instruction text)]} from cuobjdump -sass, or {} where cuobjdump is not found."""
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        return {}
    txt = subprocess.run([exe, "-sass", lib], capture_output=True, text=True, check=True).stdout
    out = {}
    for block in re.split(r"\n\s*Function : ", txt)[1:]:
        name = block.split("\n", 1)[0].strip()
        out[name] = [(int(o, 16), s.strip()) for o, s in re.findall(r"^\s+/\*([0-9a-f]{4,})\*/\s+([^;]*);", block, re.M)]
    return out


def traverse_phases(ins):
    """Static shape of k_traverse's loop body: the node loads (five 128-bit loads off one base register, offsets
    0x00..0x40), the node phase from the first of them to the REDUX.SUM that sizes the triangle pass, and the pass from
    there to its hit merge (the 64-bit shared-memory atomic)."""
    redux = next((i for i, (_, s) in enumerate(ins) if s.startswith("REDUX.SUM")), None)
    if redux is None:
        return None
    # the last unpredicated 128-bit load of each offset 0x00..0x40 off one base register before the REDUX.SUM
    last = {}
    for i, (_, s) in enumerate(ins[:redux]):
        m = re.match(r"LDG\.E\.128\S* R\d+, desc\[\w+\]\[(R\d+)\.64(?:\+0x([1-4])0)?\]", s)
        if m:
            last.setdefault(m.group(1), {})[int(m.group(2) or 0)] = i
    groups = [sorted(v.values()) for v in last.values() if len(v) == 5]
    if not groups:
        return None
    node = max(groups)
    merge = next((i for i, (_, s) in enumerate(ins) if i > redux and s.startswith("ATOMS.CAS")), None)
    return {"node_loads": [ins[j][0] for j in node], "node_phase": redux - node[0],
            "tri_pass": (merge - redux + 1) if merge is not None else None,
            "vimnmx3": sum(1 for _, s in ins if s.startswith("VIMNMX3")), "fmnmx": sum(1 for _, s in ins if "FMNMX" in s)}


def build_table():
    report = ptxas_report(os.path.join(CSRC, "ptxas_info.txt"))
    sass = sass_listing(os.path.join(CSRC, "libcrt_cuda_core.so"))
    rows = ["| kernel | SASS instructions | registers | stack B | spill stores B | spill loads B |", "|---|---:|---:|---:|---:|---:|"]
    kernels = list(SHADE_KERNELS.items()) + [(m, traverse_label(m)) for m in sorted(report) if m.startswith("_ZN3crt10k_traverse")]
    for mangled, label in kernels:
        p = report.get(mangled, {})
        n = len(sass[mangled]) if mangled in sass else "n/a"
        rows.append(f"| `{label}` | {n} | {p.get('registers', 'n/a')} | {p.get('stack', 'n/a')} | "
                    f"{p.get('spill_stores', 'n/a')} | {p.get('spill_loads', 'n/a')} |")
    ph = traverse_phases(sass[TRAVERSE_DEFAULT]) if TRAVERSE_DEFAULT in sass else None
    if ph:
        loads = ", ".join(f"0x{o:04x}" for o in ph["node_loads"])
        rows += ["", f"Default k_traverse, static: node loads at {loads}; node phase {ph['node_phase']} instructions (first node "
                     f"load to the pass's REDUX.SUM); triangle pass {ph['tri_pass']} instructions (REDUX.SUM to the 64-bit "
                     f"shared-memory merge); {ph['vimnmx3']} VIMNMX3, {ph['fmnmx']} FMNMX."]
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
    parts += ["## k_shade and k_traverse as compiled (ptxas -v, cuobjdump -sass)", "", build_table(), ""]
    text = "\n".join(parts)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(text)
    print(text)


if __name__ == "__main__":
    main()
