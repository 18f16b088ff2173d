"""Camera vectors as the reference app hands them to ``RenderBackend::render``.

``main.cpp:300-301`` passes ``ArcballCamera::eye()/dir()/up()``, which are re-derived from the
inverse camera matrix (``util/arcball_camera.cpp:10-23,61-72``): ``dir`` is the normalised view
direction and ``up`` is the *re-orthogonalised* up vector, not the ``-up`` argument. This module
restates that derivation (look-at basis) in f32; it is host-side convenience, not hot path.
"""
from __future__ import annotations

import numpy as np


def _norm(v):
    v = np.asarray(v, dtype=np.float32)
    return (v / np.sqrt(np.dot(v, v), dtype=np.float32)).astype(np.float32)


class ArcballCamera:
    def __init__(self, eye, center, up):
        eye = np.asarray(eye, dtype=np.float32)
        center = np.asarray(center, dtype=np.float32)
        z_axis = _norm(center - eye)
        x_axis = _norm(np.cross(z_axis, _norm(up)).astype(np.float32))
        y_axis = _norm(np.cross(x_axis, z_axis).astype(np.float32))
        self._eye = eye
        self._dir = z_axis
        self._up = y_axis
        self._center = center

    def eye(self):
        return self._eye.copy()

    def dir(self):
        return self._dir.copy()

    def up(self):
        return self._up.copy()

    def center(self):
        return self._center.copy()


def view_args(cam):
    """``(pos, dir, up, fovy)`` for ``RenderCUDA.render``: ``cam`` is that tuple already, or a camera dict with ``position``
    (``.crts`` cameras, ``scene_io``) or ``eye`` (``scenes``), ``center``, ``up`` and ``fov_y``, seen through
    ``ArcballCamera`` as the reference app does."""
    if isinstance(cam, dict):
        c = ArcballCamera(cam["position"] if "position" in cam else cam["eye"], cam["center"], cam["up"])
        return c.eye(), c.dir(), c.up(), float(cam["fov_y"])
    pos, d, up, fovy = cam
    return pos, d, up, float(fovy)
