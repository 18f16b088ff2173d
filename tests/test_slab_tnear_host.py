"""The BVH8 box test compares the plane distances as signed integers (bvh8_traverse.h: node_intersect_loaded). That is
exact for tnear >= 0, which every ray of a frame has; caller-supplied rays (crtc_trace_closest) may start at a negative
tnear, where the integer order of negative floats is reversed and the test must stay conservative. Rays whose origin
has been moved past part of the scene, with tnear < 0 reaching back to the camera, must give the oracle's hits bit for
bit. CPU only: this runs the single-ray host instantiation of the traversal (libcrt_bvh8_hostcheck.so), which checks the
box test but not k_traverse's warp-pooled hit merge; tests/test_traversal_edges.py runs the kernel on such rays."""
import numpy as np

from chameleonrt_b200.scenes import sponza_like
from helpers import HostCheck, bounce_rays, camera_for
from oracle import OracleBackend
from oracle.oracle import primary_rays


def test_negative_tnear_matches_oracle(built):
    scene, cam = sponza_like(detail=0.35, tex_size=16)
    o = OracleBackend()
    o.initialize(8, 8)
    o.set_scene(scene)
    hc = HostCheck(scene)
    c = camera_for(cam)
    rays = primary_rays(64, 36, c.eye(), c.dir(), c.up(), cam["fov_y"])
    rays = np.concatenate([rays, bounce_rays(rays, o.trace_closest(rays))]).astype(np.float32)
    rng = np.random.default_rng(7)
    shift = rng.uniform(0.0, 8.0, len(rays)).astype(np.float32)
    moved = rays.copy()
    moved[:, 0:3] += shift[:, None] * rays[:, 4:7]
    moved[:, 3] = -shift * rng.uniform(0.0, 1.0, len(rays)).astype(np.float32)
    assert (moved[:, 3] < 0).mean() > 0.9
    ho = o.trace_closest(moved)
    hb, _, _ = hc.trace(moved)
    assert (ho.view(np.uint32) == hb.view(np.uint32)).all(), "closest hit with tnear < 0 differs from the oracle"
    behind = (ho[:, 3].view(np.uint32) != 0xFFFFFFFF) & (ho[:, 0] < 0)
    assert behind.sum() > 50, "the rays must find hits between tnear and the origin"
    ha, _, _ = hc.trace(moved, any_hit=True)
    assert ((ha[:, 3].view(np.uint32) != 0xFFFFFFFF) == o.trace_any(moved).astype(bool)).all()
