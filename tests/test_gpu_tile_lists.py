"""A tile list that covers a pixel twice is refused (TGB_ERR_INVALID) by every call that takes one.

k_resolve, k_unpack_tiles and k_unpack_share own one pixel per thread.  A multi-GPU context deals the tiles to its GPUs in
Morton order, where two overlapping tiles of one 16x16 cell sit next to each other: with two GPUs they go to different GPUs, both
render the shared pixels, and the gather keeps the last GPU's copy.  The check runs on the whole list before the deal.
"""
import os

import numpy as np
import pytest

from tungsten_b200 import abi, lib, scene

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
