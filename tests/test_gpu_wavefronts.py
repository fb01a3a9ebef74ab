"""The two wavefronts of a context (each half of a step's camera paths, on its own stream) against one another and against the
caller's stream.

Which wavefront, slot or iteration traces a path cannot change its result (every path seeds its own RNG and writes its radiance
to R[path id], DESIGN.md section 3).  A small `max_paths_in_flight` runs many iterations, and its two halves drain at
different times: the image, the sample counts and the integer statistics must equal those of the default capacity exactly.
"""
import os

import numpy as np
import pytest

from tungsten_b200 import abi, lib, scene, synth
from oracle import pyoracle

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
STATS = ("samples", "path_rays", "shadow_rays", "hits", "path_rays_traversed", "shadow_rays_traversed")
SMALL = 1500                                  # 750 path slots per wavefront


def _stats(ctx):
    st = ctx.stats()
    return {k: int(getattr(st, k)) for k in STATS}


# cornell: analytic primitives only; cube_city: analytic primitives in BVH leaves; many_lights: > 16 samplable lights;
# materials_env: mesh lights (the closest-hit shadow queue) and an environment map; hair_sky: curves
@pytest.mark.parametrize("name", ["cornell", "cube_city", "many_lights", "materials_env", "hair_sky"])
def test_small_capacity_equals_default_capacity(name):
    fs = scene.load_scene(os.path.join(G, name, "scene.json"))
    runs = []
    for cap in (0, SMALL):
        ctx = lib.Context(fs, max_paths_in_flight=cap)
        img, cnt = ctx.render_tiles(fs.spp)
        runs.append((img, cnt, _stats(ctx)))
        ctx.close()
    (a, ca, sa), (b, cb, sb) = runs
    assert np.array_equal(a, b) and np.array_equal(ca, cb)
    assert sa == sb
    assert sa["samples"] == fs.resolution[0]*fs.resolution[1]*fs.spp


def test_small_capacity_equals_default_capacity_adaptive():
    """One adaptive step (per-block sample counts: the result-slot range is split between the wavefronts)."""
    fs = scene.load_scene(os.path.join(G, "cornell_adaptive", "scene.json"))
    n_blocks = ((fs.resolution[0] + 3)//4)*((fs.resolution[1] + 3)//4)
    runs = []
    for cap in (0, SMALL):
        ctx = lib.Context(fs, max_paths_in_flight=cap)
        ctx.render_tiles(4)
        rec = (abi.SampleRecord*n_blocks)()
        for i, r in enumerate(rec):
            r.next_sample_count = 1 + (i % 5); r.sample_index = 4
        ctx.render_adaptive(rec)
        img, cnt = ctx.read_framebuffer()
        runs.append((img, cnt, bytes(rec), _stats(ctx)))
        ctx.close()
    (a, ca, ra, sa), (b, cb, rb, sb) = runs
    assert np.array_equal(a, b) and np.array_equal(ca, cb)
    assert ra == rb
    assert sa == sb


class _DeviceFloats:
    """A device pointer as a torch tensor (__cuda_array_interface__), without a copy."""
    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": "<f4", "data": (ptr, False), "version": 2, "strides": None}


def test_render_is_complete_on_the_callers_stream():
    """A render on the caller's stream (tgb200_set_stream) is finished for whatever the caller queues on that stream after the
    call: the framebuffer copied on that stream, without a device-wide synchronisation, equals the synchronised read and the
    oracle's image.  (Wavefront 1 runs on the context's second stream; without the join before k_resolve, its paths would be
    missing from the image.)"""
    import torch
    fs = scene.load_scene(synth.cornell_box(res=(96, 96), spp=8))
    w, h = fs.resolution
    ctx = lib.Context(fs)
    ptr, n_bytes = ctx.framebuffer_device_ptr()
    assert n_bytes == w*h*12
    fb = torch.as_tensor(_DeviceFloats(ptr, (h, w, 3)), device="cuda")
    s = torch.cuda.Stream()
    ctx.set_stream(s.cuda_stream)
    ctx.clear()
    with torch.cuda.stream(s):
        ctx.render_resident(8)
        got = fb.clone()
        done = torch.cuda.Event()
        done.record(s)
    done.synchronize()
    ctx.set_stream(None)
    img, cnt = ctx.read_framebuffer()
    ctx.close()
    assert np.array_equal(got.cpu().numpy(), img)
    o = pyoracle.Oracle(fs)
    ref, rcnt = o.render(8)
    o.close()
    assert np.array_equal(cnt, rcnt)
    d = np.abs(img - ref).max(axis=2)
    assert float((d <= 1e-5*(1.0 + np.abs(ref).max(axis=2))).mean()) >= 0.9999      # as tests/test_gpu_parity.py::test_cornell_box
