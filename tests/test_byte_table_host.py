"""Texel conversion and material unpacking of the device shading source (shade_math.cuh), compiled for the host
(TEST-ONLY libcrt_shade_hostcheck.so).

- The byte -> [0, 1] table that replaces the division (float)q / 255.f holds exactly its correctly rounded quotients.
- unpack_material filters the textured scalar parameters at one fetch site, one channel per step, reusing the texel
  words of the step before when the texture is the same. Every parameter must still be, bit for bit, the channel of
  the full RGBA filter (texture_rgba, which tests/test_shade_host.py pins to the reference's texture2d.ih) that its
  word names, and every untextured parameter its own word."""
import ctypes as C
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib(built):
    lib = C.CDLL(os.path.join(ROOT, "chameleonrt_b200", "csrc", "libcrt_shade_hostcheck.so"))
    vp = C.c_void_p
    lib.shadekat_byte_to_unit.argtypes = [vp]
    lib.shadekat_texture.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, C.c_int, vp]
    lib.shadekat_unpack_material.argtypes = [vp, C.c_uint32, vp, vp, vp, C.c_int, vp]
    return lib


def test_byte_table_is_the_correctly_rounded_quotient(lib):
    table = np.zeros(256, np.float32)
    lib.shadekat_byte_to_unit(table.ctypes.data)
    want = np.arange(256, dtype=np.float32) / np.float32(255.0)  # IEEE single division, round to nearest even
    assert np.array_equal(table.view(np.uint32), want.view(np.uint32))


def _textured_word(tex_id, channel):
    return np.array([0x80000000 | (channel << 29) | tex_id], np.uint32).view(np.float32)[0]


def test_unpack_material_matches_per_parameter_filter(lib):
    rng = np.random.default_rng(7)
    sizes = [(16, 8), (5, 7), (1, 1), (32, 32)]
    texs = [rng.integers(0, 256, size=(h, w, 4), dtype=np.uint8) for w, h in sizes]
    # the device arena: RGBA8 words of every texture back to back, DevTex {offset, width, height, pad} per texture
    words = [t.reshape(-1, 4).astype(np.uint32) for t in texs]
    words = [w[:, 0] | (w[:, 1] << 8) | (w[:, 2] << 16) | (w[:, 3] << 24) for w in words]
    offsets = np.cumsum([0] + [len(w) for w in words[:-1]])
    arena = np.ascontiguousarray(np.concatenate(words).astype(np.uint32))
    desc = np.array([[o, w, h, 0] for o, (w, h) in zip(offsets, sizes)], np.int32)
    n = 257
    uv = np.concatenate([rng.uniform(-3, 3, size=(n - 1, 2)), [[0.5, 0.5]]]).astype(np.float32)
    rgba = []  # texture_rgba of every texture at every uv
    for t, (w, h) in zip(texs, sizes):
        out = np.zeros((n, 4), np.float32)
        lib.shadekat_texture(np.ascontiguousarray(t).ctypes.data, w, h, 4, uv.ctypes.data, n, out.ctypes.data)
        rgba.append(out)
    for trial in range(200):
        m = rng.uniform(0.0, 1.0, size=16).astype(np.float32)
        expect = np.zeros((n, 14), np.float32)
        if trial % 3:
            tid, ch = int(rng.integers(len(texs))), 0
            m[0] = _textured_word(tid, 0)
            expect[:, 0:3] = rgba[tid][:, 0:3]
        else:
            expect[:, 0:3] = m[0:3]
        # trial 0: no scalar parameter textured; others: a random subset, often runs on one texture
        textured = rng.random(11) < (0.0 if trial == 0 else rng.uniform(0.1, 1.0))
        tid = int(rng.integers(len(texs)))
        for k in range(11):
            if textured[k]:
                if rng.random() < 0.4:
                    tid = int(rng.integers(len(texs)))
                ch = int(rng.integers(4))
                m[3 + k] = _textured_word(tid, ch)
                expect[:, 3 + k] = rgba[tid][:, ch]
            else:
                expect[:, 3 + k] = m[3 + k]
        mats = np.ascontiguousarray(np.concatenate([rng.uniform(size=16).astype(np.float32), m]))  # material id 1
        got = np.zeros((n, 14), np.float32)
        lib.shadekat_unpack_material(mats.ctypes.data, 1, arena.ctypes.data, desc.ctypes.data, uv.ctypes.data, n,
                                     got.ctypes.data)
        assert np.array_equal(got.view(np.uint32), expect.view(np.uint32)), f"trial {trial}"
