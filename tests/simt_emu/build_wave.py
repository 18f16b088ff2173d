"""Builds tests/simt_emu/_build/libcrt_wave_devcheck_simt.so: chameleonrt_b200/csrc/wave_devcheck.cu (the per-bounce
kernels one launch at a time) compiled for the host with its launches translated as build.py translates the renderer's,
so that every stage runs on 32-lane warps with real atomics (tests/test_wavefront_device.py). A module of its own, so
that the renderer's emulated build does not go stale when this one changes."""
import os

import build as simt_build

CSRC, OUT, ROOT = simt_build.CSRC, simt_build.OUT, simt_build.ROOT
WAVE_LIB = os.path.join(OUT, "libcrt_wave_devcheck_simt.so")
LAUNCHES = 11  # the <<<...>>> launches of wave_devcheck.cu


def build_wave_devcheck(force: bool = False) -> str:
    srcs = [os.path.join(CSRC, f) for f in ("wave_devcheck.cu", "kernels.cuh", "shade_math.cuh", "bvh8_device.cuh", "cuda_host_utils.h",
                                            "bvh8_traverse.h", "simt_env.h", "host_scene.h", "host_scene.cpp", "bvh8.h", "bvh8_build.cpp")]
    srcs += [os.path.join(simt_build.HERE, "cuda_emu.cpp"), simt_build.__file__, __file__]
    if not force and os.path.exists(WAVE_LIB) and all(os.path.getmtime(WAVE_LIB) >= os.path.getmtime(s) for s in srcs):
        return WAVE_LIB
    os.makedirs(OUT, exist_ok=True)
    gen = os.path.join(OUT, "wave_devcheck_simt.cpp")
    with open(gen, "w") as f:
        f.write('#include "simt_env.h"\n' + simt_build.translate(open(os.path.join(CSRC, "wave_devcheck.cu")).read().replace(
            '"../../include/crt_scene.h"', f'"{ROOT}/include/crt_scene.h"'), LAUNCHES))
    simt_build._link(WAVE_LIB, gen)
    return WAVE_LIB


if __name__ == "__main__":
    print(build_wave_devcheck(force=True))
