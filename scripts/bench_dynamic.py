"""Scene updates (option dynamic_scene; crtc_commit_scene) on the GPU (CUDA device required; there is no CPU fallback).

  * commit time: CUDA events on the renderer's stream (a torch stream, crtc_set_stream) around crtc_commit_scene, median
    of --commits, on C2, C3 and C4 as bench.py generates them: every instance's transform staged (moved by a small
    translation) before each commit. Next to it, crtc_set_scene's wall time (it returns after a stream synchronisation)
    with the host builder and with the PLOC builder, option dynamic_scene off, and the set_scene time with it on;
  * tree degradation: C3's instances translated by 0.2 % to 10 % of the scene's extent (random directions, a random
    rotation about y) and committed into the tree built for the original scene, against a fresh set_scene of the same
    moved scene with the same builder: ms/frame (crtc_get_stage_times [6], blocking frames after warm-up), which tells
    when a new set_scene pays off. Frames of both are bit-identical (tests/test_dynamic_scene.py); only the time differs.

Prints a markdown report with the card's name and power limit, and writes it to --out when given.

    python scripts/bench_dynamic.py --out profiles/dynamic_h100.md
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
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q or "unknown"


def workload(key):
    import bench
    from chameleonrt_b200 import scenes

    w = bench.WORKLOADS[key]
    scene, cam = getattr(scenes, w["gen"])(spp=w["spp"], **w["kw"])
    return w, scene, cam


def num_tris(scene):
    return sum(len(g.indices) for i in scene.instances
               for g in scene.meshes[scene.parameterized_meshes[i.parameterized_mesh_id].mesh_id].geometries)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c2,c4,c3")
    ap.add_argument("--commits", type=int, default=20)
    ap.add_argument("--frames", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--moves", default="0.002,0.005,0.01,0.02,0.1")
    ap.add_argument("--builder", default="host", help="builder of the degradation runs")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_dynamic.py needs a CUDA device")
    from chameleonrt_b200 import ArcballCamera, RenderCUDA

    name, power = card()
    stream = torch.cuda.Stream()
    lines = [f"# Scene updates: commit time and tree degradation ({name}, power limit {power})", "",
             "Measured by `scripts/bench_dynamic.py` in one run. Commit: CUDA events on the renderer's stream around "
             f"crtc_commit_scene, median of {args.commits}; set_scene: host wall clock (it ends with a stream synchronisation).", "",
             "| workload | triangles | instances | BVH8 nodes | set_scene host builder (ms) | set_scene PLOC (ms) | set_scene PLOC + dynamic_scene (ms) "
             "| commit, median (ms) | commit min / max (ms) | commit launches |",
             "|---|---|---|---|---|---|---|---|---|---|"]

    def timed_set_scene(scene, w, builder, dynamic):
        r = RenderCUDA(0, max_depth=w["depth"], bvh_builder=builder, dynamic_scene=dynamic, stream=stream.cuda_stream)
        r.initialize(w["w"], w["h"])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r.set_scene(scene)
        return r, (time.perf_counter() - t0) * 1e3

    for key in filter(None, args.workloads.split(",")):
        w, scene, cam = workload(key)
        t_host = timed_set_scene(scene, w, "host", False)[1]
        timed_set_scene(scene, w, "device", False)  # (first device build: module load)
        t_ploc = timed_set_scene(scene, w, "device", False)[1]
        r, t_dyn = timed_set_scene(scene, w, "device", True)
        base = np.array([i.transform for i in scene.instances], np.float32)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ms = []
        for k in range(args.commits + 2):
            moved = base.copy()
            moved[:, :3, 3] += np.float32(1e-3 * (k % 2))
            r.update_instances(moved)
            ev[0].record(stream)
            r.commit_scene()
            ev[1].record(stream)
            stream.synchronize()
            if k >= 2:
                ms.append(ev[0].elapsed_time(ev[1]))
        info = r.scene_info()
        depth = int(info["bvh8_depth"])
        lines.append(f"| {key.upper()} | {num_tris(scene):,} | {len(scene.instances)} | {int(info['bvh8_nodes']):,} | {t_host:.0f} | "
                     f"{t_ploc:.1f} | {t_dyn:.1f} | {np.median(ms):.3f} | {min(ms):.3f} / {max(ms):.3f} | 1 + {depth} |")
        del r
        torch.cuda.empty_cache()
        print(lines[-1], flush=True)

    # ---- tree degradation on C3 ----
    w, scene, cam = workload("c3")
    c = ArcballCamera(cam["eye"], cam["center"], cam["up"])
    view = (c.eye(), c.dir(), c.up(), cam["fov_y"])
    lo, hi = np.full(3, np.inf), np.full(3, -np.inf)
    for i in scene.instances:
        pm = scene.parameterized_meshes[i.parameterized_mesh_id]
        m = np.asarray(i.transform, np.float64)
        for g in scene.meshes[pm.mesh_id].geometries:
            v = np.asarray(g.vertices, np.float64)
            if len(v):
                wv = v @ m[:3, :3].T + m[:3, 3]
                lo, hi = np.minimum(lo, wv.min(0)), np.maximum(hi, wv.max(0))
    extent = float((hi - lo).max())

    def frame_ms(r, first_changed):
        for f in range(args.warmup):
            r.render(*view, first_changed and f == 0, True)
        t = 0.0
        for _ in range(args.frames):
            r.render(*view, False, True)
            t += r.stage_times()["frame"]
        return t / args.frames

    def renderer(s, dynamic):
        r = RenderCUDA(0, max_depth=w["depth"], bvh_builder=args.builder, dynamic_scene=dynamic, any_far_first=0)
        r.initialize(w["w"], w["h"])
        r.set_scene(s)
        return r

    lines += ["", f"## Tree degradation: C3 ({num_tris(scene):,} triangles, {len(scene.instances)} instances), {w['w']}x{w['h']}, "
              f"{w['spp']} spp, depth {w['depth']}, builder {args.builder}", "",
              f"Every instance translated by the given fraction of the scene's extent ({extent:.1f}) in a random direction and "
              "rotated about y by a random angle up to that fraction of a half turn; ms/frame = crtc_get_stage_times [6], mean of "
              f"{args.frames} blocking frames after {args.warmup} warm-up frames.", "",
              "| move | refit tree (ms/frame) | fresh build of the moved scene (ms/frame) | refit / fresh |", "|---|---|---|---|"]
    r0 = renderer(scene, True)
    base_ms = frame_ms(r0, True)
    lines.append(f"| 0 (the built scene) | {base_ms:.2f} | {base_ms:.2f} | 1.00 |")
    print(lines[-1], flush=True)
    rng = np.random.default_rng(1)
    dirs = rng.normal(size=(len(scene.instances), 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    angles = rng.uniform(-1, 1, len(scene.instances))
    import copy

    for frac in [float(x) for x in args.moves.split(",")]:
        moved = []
        for i, inst in enumerate(scene.instances):
            a = angles[i] * frac * np.pi
            rot = np.eye(4)
            rot[0, 0], rot[0, 2], rot[2, 0], rot[2, 2] = np.cos(a), np.sin(a), -np.sin(a), np.cos(a)
            m = np.asarray(inst.transform, np.float64)
            t = m[:3, 3].copy()
            m = rot @ m
            m[:3, 3] = t + dirs[i] * frac * extent
            moved.append(m.astype(np.float32))
        r0.update_instances(np.array(moved))
        r0.commit_scene()
        refit = frame_ms(r0, False)
        s2 = copy.copy(scene)
        s2.instances = [copy.copy(i) for i in scene.instances]
        for inst, m in zip(s2.instances, moved):
            inst.transform = m
        fresh_r = renderer(s2, False)
        fresh = frame_ms(fresh_r, True)
        del fresh_r
        torch.cuda.empty_cache()
        lines.append(f"| {frac * 100:g} % | {refit:.2f} | {fresh:.2f} | {refit / fresh:.2f} |")
        print(lines[-1], flush=True)
    report = "\n".join(lines) + "\n"
    print(report)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(report)


if __name__ == "__main__":
    main()
