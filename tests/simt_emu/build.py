"""Builds tests/simt_emu/_build/libcrt_cuda_core_simt.so: the PRODUCT's renderer object and C ABI
(chameleonrt_b200/csrc/crt_cuda_core.cu, kernels.cuh, ...) compiled for the host, with every kernel launch executed
under the SIMT environment of chameleonrt_b200/csrc/simt_env.h and the CUDA runtime replaced by cuda_emu.cpp.
TEST INFRASTRUCTURE: the only edit made to the product source is mechanical — each
    kernel<<<grid, block, 0, stream>>>(args);
becomes
    simt::launch(grid, block, [&] { kernel(args); });
(g++ cannot parse the chevrons; crt_cuda_core.cu and its header scene_device_build.cuh are translated). Nothing in chameleonrt_b200/ loads this library; tests/test_simt_renderer.py
points a RenderCUDA at it explicitly."""
import os
import re
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "chameleonrt_b200", "csrc")
OUT = os.path.join(HERE, "_build")
LIB = os.path.join(OUT, "libcrt_cuda_core_simt.so")


def translate(src: str, expected: int) -> str:
    out, pos = [], 0
    pat = re.compile(r"(crt::k_\w+(?:<[\w, ]+>)?)<<<([^,]+),\s*([^,]+),\s*0,\s*stream>>>\(")
    n = 0
    while True:
        m = pat.search(src, pos)
        if not m:
            break
        out.append(src[pos:m.start()])
        depth, i = 1, m.end()
        while depth:
            depth += {"(": 1, ")": -1}.get(src[i], 0)
            i += 1
        assert src[i] == ";", src[m.start():i + 1]
        out.append(f"simt::launch({m.group(2).strip()}, {m.group(3).strip()}, [&] {{ {m.group(1)}({src[m.end():i - 1]}); }});")
        pos = i + 1
        n += 1
    out.append(src[pos:])
    assert n == expected, f"expected {expected} kernel launches, found {n}"
    return "".join(out)


def build(force: bool = False) -> str:
    srcs = [os.path.join(CSRC, f) for f in ("crt_cuda_core.cu", "scene_device_build.cuh", "cuda_host_utils.h", "bvh8_device.cuh", "kernels.cuh", "shade_math.cuh", "bvh8_traverse.h", "simt_env.h",
                                            "host_scene.h", "host_scene.cpp", "bvh8.h", "bvh8_build.cpp")] + [os.path.join(HERE, "cuda_emu.cpp"), __file__]
    if not force and os.path.exists(LIB) and all(os.path.getmtime(LIB) >= os.path.getmtime(s) for s in srcs):
        return LIB
    os.makedirs(OUT, exist_ok=True)
    gen = os.path.join(OUT, "crt_cuda_core_simt.cpp")
    with open(gen, "w") as f:
        f.write('#include "simt_env.h"\n' + translate(open(os.path.join(CSRC, "crt_cuda_core.cu")).read().replace(
            '"../../include/crt_cuda.h"', f'"{ROOT}/include/crt_cuda.h"'), 21))
    _write_driver()
    _link(LIB, gen)
    return LIB


def _write_driver():
    # the device set_scene driver is a header of the same translation unit: its translated copy sits next to the
    # generated source, where the quoted include finds it first
    with open(os.path.join(OUT, "scene_device_build.cuh"), "w") as f:
        f.write(translate(open(os.path.join(CSRC, "scene_device_build.cuh")).read().replace(
            '"../../include/crt_scene.h"', f'"{ROOT}/include/crt_scene.h"'), 18))


def _link(lib, gen):
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"))), "include")
    subprocess.check_call(["make", "-s", "-C", CSRC, "host_scene.o", "bvh8_build.o"])
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-pthread", "-march=x86-64-v3", "-ffp-contract=off", "-Wno-attributes",
                           "-I" + CSRC, "-I" + cuda_inc, "-shared",
                           # -Bsymbolic: the library's calls to cudaMalloc & co. must bind to ITS stubs even when a real
                           # libcudart is already in the process (torch loads one globally)
                           "-Wl,-Bsymbolic", "-o", lib, gen, os.path.join(HERE, "cuda_emu.cpp"),
                           os.path.join(CSRC, "host_scene.o"), os.path.join(CSRC, "bvh8_build.o")])


DEVCHECK_LIB = os.path.join(OUT, "libcrt_bvh_devcheck_simt.so")


def build_bvh_devcheck(force: bool = False) -> str:
    """_build/libcrt_bvh_devcheck_simt.so: chameleonrt_b200/csrc/bvh_devcheck.cu (which has no launch of its own)
    compiled for the host next to the translated scene_device_build.cuh, with every kernel launch of the device build
    under the SIMT environment (tests/test_bvh_build_exact.py)."""
    srcs = [os.path.join(CSRC, f) for f in ("bvh_devcheck.cu", "scene_device_build.cuh", "cuda_host_utils.h", "bvh8_device.cuh", "bvh8_traverse.h", "simt_env.h",
                                            "host_scene.h", "host_scene.cpp", "bvh8.h", "bvh8_build.cpp")] + [os.path.join(HERE, "cuda_emu.cpp"), __file__]
    if not force and os.path.exists(DEVCHECK_LIB) and all(os.path.getmtime(DEVCHECK_LIB) >= os.path.getmtime(s) for s in srcs):
        return DEVCHECK_LIB
    os.makedirs(OUT, exist_ok=True)
    gen = os.path.join(OUT, "bvh_devcheck_simt.cpp")
    src = open(os.path.join(CSRC, "bvh_devcheck.cu")).read()
    assert "<<<" not in src, "bvh_devcheck.cu must not launch kernels itself"
    with open(gen, "w") as f:
        f.write('#include "simt_env.h"\n' + src.replace('"../../include/crt_scene.h"', f'"{ROOT}/include/crt_scene.h"'))
    _write_driver()
    _link(DEVCHECK_LIB, gen)
    return DEVCHECK_LIB


def build_plugin(force: bool = False):
    """oracle/_ref/libcrt_cuda_simt.so: the drop-in C++ plugin (backends/cuda/*.cpp, unchanged) linked against the
    emulated core, so that `crt_headless cuda_simt <scene>` runs the whole drop-in path — the reference's loaders,
    RenderPlugin, RenderCUDA : RenderBackend, the C ABI, the kernels — without a GPU. Needs the reference headers and
    the objects oracle/ref_build compiled from the reference's util/ + imgui/ (so: only where /root/reference is);
    returns None elsewhere."""
    ref = os.environ.get("REF", "/root/reference")
    obj = os.path.join(ROOT, "oracle", "_ref", "obj")
    if not os.path.isdir(os.path.join(ref, "util")) or not os.path.isdir(obj):
        return None
    core = build(force)
    out = os.path.join(ROOT, "oracle", "_ref", "libcrt_cuda_simt.so")
    srcs = [os.path.join(ROOT, "backends", "cuda", f) for f in ("render_cuda.cpp", "render_cuda_plugin.cpp", "render_cuda.h")]
    srcs += [os.path.join(HERE, "plugin_alias.cpp"), core]
    if not force and os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(s) for s in srcs):
        return out
    objs = sorted(os.path.join(obj, f) for f in os.listdir(obj) if f.startswith(("util_", "imgui_")) and f.endswith(".o"))
    inc = [f"-I{ROOT}/third_party/miniglm", f"-I{ROOT}/third_party/sdl_stub", f"-I{ref}/util", f"-I{ref}/util/parallel_hashmap",
           f"-I{ref}/imgui", f"-I{ROOT}/include"]
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-fPIC", "-w", "-pthread", *inc, "-DCRT_CUDA_HEADLESS", "-shared", "-o", out,
                           srcs[0], srcs[1], srcs[3], *objs, "-L" + OUT, "-lcrt_cuda_core_simt", "-Wl,-rpath," + OUT])
    return out


if __name__ == "__main__":
    print(build(force=True))
    print(build_bvh_devcheck(force=True))
    print(build_plugin(force=True))
