"""A tile list that covers a pixel twice is refused (TGB_ERR_INVALID) by every call that takes one.

k_resolve, k_unpack_tiles and k_unpack_share own one pixel per thread.  A multi-GPU context deals the tiles to its GPUs in
Morton order, where two overlapping tiles of one 16x16 cell sit next to each other: with two GPUs they go to different GPUs, both
render the shared pixels, and the gather keeps the last GPU's copy.  The check runs on the whole list before the deal.
"""
import os

import numpy as np
import pytest

from tungsten_b200 import abi, integrator, lib, scene, synth

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# two tiles each: positions 0 and 1 of the Morton deal, so one per GPU of a two-GPU context
OVERLAPPING = {
    "same_tile_twice": [(0, 0, 16, 16, 7), (0, 0, 16, 16, 7)],
    "shared_corner": [(0, 0, 16, 16, 7), (8, 8, 16, 16, 9)],
}


def _tiles(spec):
    return (abi.Tile*len(spec))(*[abi.Tile(*t) for t in spec])


def _refused(call):
    with pytest.raises(lib.TgbError) as e:
        call()
    assert e.value.code == abi.TGB_ERR_INVALID


def _check_render_calls(ctx, spec):
    """render_tiles, render_resident and render_adaptive refuse the list; the context then still renders its first tile."""
    tiles = _tiles(spec)
    _refused(lambda: ctx.render_tiles(1, tiles=tiles))
    _refused(lambda: ctx.render_resident(1, tiles=tiles))
    n_blocks = ((ctx.width + 3)//4)*((ctx.height + 3)//4)
    rec = (abi.SampleRecord*n_blocks)()
    for r in rec:
        r.next_sample_count = 1
    _refused(lambda: ctx.render_adaptive(rec, tiles=tiles))
    img, cnt = ctx.render_tiles(1, tiles=_tiles(spec[:1]))
    assert cnt[:16, :16].min() == 1 and cnt.sum() == 16*16 and np.isfinite(img).all()


@pytest.mark.parametrize("name", OVERLAPPING)
def test_two_gpu_context_refuses_overlapping_tiles(name):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    fs = scene.load_scene(os.path.join(G, "cornell", "scene.json"))
    for kw in ({"devices": [0, 1]}, {"device": 0}):
        ctx = lib.Context(fs, **kw)
        _check_render_calls(ctx, OVERLAPPING[name])
        ctx.close()


@pytest.mark.parametrize("name", OVERLAPPING)
def test_single_gpu_context_refuses_overlapping_tiles(name):
    """The same on one GPU, where tgb200_pack_tiles / tgb200_unpack_tiles took such a list and packed or wrote the shared pixels
    twice."""
    import torch
    fs = scene.load_scene(os.path.join(G, "cornell", "scene.json"))
    ctx = lib.Context(fs, device=0)
    _check_render_calls(ctx, OVERLAPPING[name])
    tiles = _tiles(OVERLAPPING[name])
    buf = torch.zeros(2*16*16*3, dtype=torch.float32, device="cuda:0")
    _refused(lambda: ctx.pack_tiles(tiles, buf.data_ptr()))
    _refused(lambda: ctx.unpack_tiles(tiles, buf.data_ptr(), 1))
    ctx.close()


def _same(got, want, what):
    for g, w in zip(got, want):
        assert np.asarray(g).tobytes() == np.asarray(w).tobytes(), what


@pytest.mark.parametrize("gpus", [1, 2])
def test_reused_context_equals_fresh_contexts(gpus):
    """One context handed tile lists that grow past its pixel capacity several times, shrink and grow again, adaptive steps over
    growing lists, and probes between renders (gpus=2: a two-GPU context dealt ever new lists, one with larger shares): every
    framebuffer, record array and probe result equals what a fresh one-GPU context gives for the same call.  The context
    re-allocates its pixel lists, result buffer, adaptive arrays and gather buffers as they grow and frees the old ones, so a
    kernel left pointing into a freed array would show here as a wrong image."""
    import torch
    from oracle import pyoracle
    from test_gpu_bounce import camera_states
    if torch.cuda.device_count() < gpus:
        pytest.skip("needs two GPUs")
    cap = 4096                                      # small: every render refills the wavefronts many times
    fs = scene.load_scene(synth.cornell_box(res=(100, 75), spp=2))
    all_tiles = list(integrator.dice_tiles(*fs.resolution, 0xBA5EBA11))

    def tiles(a, b):
        return (abi.Tile*(b - a))(*all_tiles[a:b])

    def fresh(call):
        ctx = lib.Context(fs, max_paths_in_flight=cap)
        out = call(ctx)
        ctx.close()
        return out

    def resident(ctx, t, spp_begin):
        ctx.clear()
        ctx.render_resident(2, spp_begin=spp_begin, tiles=t)
        return ctx.read_framebuffer()

    def adaptive(ctx, t, k):
        rec = (abi.SampleRecord*(((ctx.width + 3)//4)*((ctx.height + 3)//4)))()
        for i, r in enumerate(rec):
            r.next_sample_count = 1 + (i*7 + k) % 4; r.sample_index = 4 + i % 3
        ctx.clear()
        ctx.render_adaptive(rec, tiles=t)
        return ctx.read_framebuffer() + (bytes(rec),)

    n = len(all_tiles)
    if gpus == 2:
        two = lib.Context(fs, devices=[0, 1], max_paths_in_flight=cap)
        for i, t in enumerate([tiles(0, 4), tiles(0, n), tiles(2, 6)]):
            what = "two GPUs, %d tiles" % len(t)
            _same(two.render_tiles(2, spp_begin=i, tiles=t), fresh(lambda c: c.render_tiles(2, spp_begin=i, tiles=t)), what)
            _same(resident(two, t, i), fresh(lambda c: resident(c, t, i)), what + ", resident")
        two.close()
        return
    ctx = lib.Context(fs, max_paths_in_flight=cap)
    # 256, 1024, 3072 pixels, then 512, all 7500, then 1536
    for i, t in enumerate([tiles(0, 1), tiles(0, 4), tiles(0, 12), tiles(5, 7), tiles(0, n), tiles(3, 9)]):
        what = "tile list %d (%d tiles)" % (i, len(t))
        _same(ctx.render_tiles(2, spp_begin=i, tiles=t), fresh(lambda c: c.render_tiles(2, spp_begin=i, tiles=t)), what)
        _same(resident(ctx, t, i), fresh(lambda c: resident(c, t, i)), what + ", resident")
    for k, t in enumerate([tiles(0, 2), tiles(0, 10), tiles(0, n)]):
        _same(adaptive(ctx, t, k), fresh(lambda c: adaptive(c, t, k)), "adaptive step over %d tiles" % len(t))
    orc = pyoracle.Oracle(fs)
    states = camera_states(fs, orc, 3*cap + 5)
    orc.close()
    _same([ctx.bounce_probe(states)], [fresh(lambda c: c.bounce_probe(states))], "bounce_probe")
    rng = np.random.default_rng(3)
    rays = np.zeros((5000, 8), np.float32)
    rays[:, 0:3] = rng.uniform(-0.9, 0.9, (5000, 3)) + [0.0, 1.0, 0.0]
    d = rng.normal(size=(5000, 3))
    rays[:, 3:6] = d/np.linalg.norm(d, axis=1, keepdims=True); rays[:, 7] = np.inf
    _same([ctx.trace_closest(rays)], [fresh(lambda c: c.trace_closest(rays))], "trace_closest")
    for t in (tiles(0, 12), tiles(0, n)):
        _same(ctx.render_tiles(2, tiles=t), fresh(lambda c: c.render_tiles(2, tiles=t)), "after the probes, %d tiles" % len(t))
    ctx.close()
