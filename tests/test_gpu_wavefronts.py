"""The two wavefronts of a context (each half of a step's camera paths, on its own stream) against one another and against the
caller's stream, and the loop's grids against the default ones.

Which wavefront, slot, iteration or thread traces a path cannot change its result (every path seeds its own RNG and writes its
radiance to R[path id], DESIGN.md section 3).  A small `max_paths_in_flight` runs many iterations, and its two halves drain at
different times: the image, the sample counts and the integer statistics must equal those of the default capacity exactly.  So
must renders whose grid-stride kernels (k_regen, k_shadow_prep, k_bin_scatter) run 1 or 5 blocks (TGB_LOOP_BLOCKS: dozens of
trips per launch) or whose persistent traversal kernels run one block per SM (TGB_TRAVERSAL_BLOCKS=1), and there every integer
statistic, launch and iteration counts included, is the default's.
"""
import ctypes as C
import os

import numpy as np
import pytest

from tungsten_b200 import abi, lib, scene, synth
from oracle import pyoracle

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
STATS = ("samples", "rays", "path_rays", "shadow_rays", "hits", "path_rays_traversed", "shadow_rays_traversed")
SMALL = 1500                                  # 750 path slots per wavefront
INT_STATS = tuple(f for f, t in abi.Stats._fields_ if t is C.c_uint64)
# runs compared with the default context: (environment, max_paths_in_flight)
VARIANTS = {"small_capacity": ({}, SMALL), "loop_blocks_1": ({"TGB_LOOP_BLOCKS": "1"}, 0),
            "loop_blocks_5": ({"TGB_LOOP_BLOCKS": "5"}, 0), "traversal_blocks_1": ({"TGB_TRAVERSAL_BLOCKS": "1"}, 0)}


def all_stats(ctx):
    st = ctx.stats()
    return {k: int(getattr(st, k)) for k in INT_STATS}


def _stats(ctx, variant):
    """Every integer statistic on the grid variants; on the small capacity, which runs more iterations and launches, STATS."""
    st = all_stats(ctx)
    return st if variant != "small_capacity" else {k: st[k] for k in STATS}


def _context(fs, variant, monkeypatch):
    env, cap = VARIANTS[variant] if variant else ({}, 0)
    for k in ("TGB_LOOP_BLOCKS", "TGB_TRAVERSAL_BLOCKS"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    ctx = lib.Context(fs, max_paths_in_flight=cap)
    for k in env:
        monkeypatch.delenv(k)
    return ctx


def _first_trips(variant, paths):
    """k_regen's trips in a wavefront's first iteration of a step of `paths` camera paths, under a TGB_LOOP_BLOCKS variant (None
    for the others).  A wavefront holds 4 Mi paths by default."""
    if not variant.startswith("loop_blocks"):
        return None
    return -(-min(paths//2, 1 << 22)//(256*int(VARIANTS[variant][0]["TGB_LOOP_BLOCKS"])))


# cornell: analytic primitives only; cube_city: analytic primitives in BVH leaves; many_lights: > 16 samplable lights;
# materials_env: mesh lights (the closest-hit shadow queue) and an environment map; hair_sky: curves; cornell_mesh: a quad light
# over a mesh (any-hit shadow queries through the BVH).  The small-capacity runs keep the ids they had before the grid variants.
@pytest.mark.parametrize("name,variant", [pytest.param(n, v, id=n if v == "small_capacity" else "%s-%s" % (n, v))
                                          for v in VARIANTS
                                          for n in ["cornell", "cube_city", "many_lights", "materials_env", "hair_sky", "cornell_mesh"]])
def test_small_capacity_equals_default_capacity(name, variant, monkeypatch):
    fs = scene.load_scene(os.path.join(G, name, "scene.json"))
    runs = []
    for v in (None, variant):
        ctx = _context(fs, v, monkeypatch)
        img, cnt = ctx.render_tiles(fs.spp)
        runs.append((img, cnt, _stats(ctx, variant)))
        ctx.close()
    (a, ca, sa), (b, cb, sb) = runs
    print("%s, %s: %s k_regen trips in the first iteration; %s" % (name, variant, _first_trips(variant, fs.resolution[0]*fs.resolution[1]*fs.spp), sb))
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) and np.array_equal(ca, cb)
    assert sa == sb
    assert sa["samples"] == fs.resolution[0]*fs.resolution[1]*fs.spp


def _adaptive_runs(variant, monkeypatch):
    """One adaptive step on the default context and on `variant`.  Some blocks get no samples -- the first, the last and a run of
    20 -- so that pixels share result-slot offsets and k_regen's search over them must skip the empty ones."""
    fs = scene.load_scene(os.path.join(G, "cornell_adaptive", "scene.json"))
    n_blocks = ((fs.resolution[0] + 3)//4)*((fs.resolution[1] + 3)//4)
    empty = {0, n_blocks - 1} | set(range(n_blocks//3, n_blocks//3 + 20))
    runs = []
    for v in (None, variant):
        ctx = _context(fs, v, monkeypatch)
        ctx.render_tiles(4)
        rec = (abi.SampleRecord*n_blocks)()
        for i, r in enumerate(rec):
            r.next_sample_count = 0 if i in empty else 1 + (i % 5); r.sample_index = 4
        ctx.render_adaptive(rec)
        img, cnt = ctx.read_framebuffer()
        runs.append((img, cnt, bytes(rec), _stats(ctx, variant)))
        ctx.close()
    (a, ca, ra, sa), (b, cb, rb, sb) = runs
    paths = sum(0 if i in empty else 16*(1 + (i % 5)) for i in range(n_blocks))
    print("cornell_adaptive, %s: %d blocks (%d empty), %d paths in the step, %s k_regen trips in the first iteration; %s"
          % (variant, n_blocks, len(empty), paths, _first_trips(variant, paths), sb))
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) and np.array_equal(ca, cb)
    assert (cb.reshape(-1) == 4).sum() >= 16*len(empty)                   # the empty blocks' pixels kept the first render's 4
    assert ra == rb
    assert sa == sb


def test_small_capacity_equals_default_capacity_adaptive(monkeypatch):
    """One adaptive step (per-block sample counts: the result-slot range is split between the wavefronts)."""
    _adaptive_runs("small_capacity", monkeypatch)


@pytest.mark.parametrize("variant", ["loop_blocks_1", "loop_blocks_5", "traversal_blocks_1"])
def test_loop_grids_equal_default_grid_adaptive(variant, monkeypatch):
    _adaptive_runs(variant, monkeypatch)


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
