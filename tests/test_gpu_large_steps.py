"""Render calls past the host loop's limits, bit for bit against folds of the GPU's own samples (as in test_gpu_adaptive).

The library renders a call in passes.  A pass keeps every finished radiance (16 B per path) until k_resolve folds it, and
holds at most 512 Mi paths, so that buffer stays within 8 GiB.  A path id packs (sample within the pass << pix_bits) | pixel,
pix_bits = the bits of the pass's pixel count, so a pixel renders at most 2^(32 - pix_bits) samples in one pass.  Uniform
steps are split into passes by sample range, adaptive steps by runs of consecutive tiles (a 4x4 block never straddles a
16x16 tile, so every block's samples fold in one pass).  The steps here cross each of those limits; the scene is the Cornell
box with one bounce, so half a billion paths stay cheap.
"""
import hashlib
import os

import numpy as np
import pytest

from tungsten_b200 import abi, integrator, lib, scene, synth
from test_adaptive_work import RECORD, assert_records_equal
from test_gpu_adaptive import (G, SEED, SampleTable, as_records, assert_image_equal, expected_adaptive_step,
                               preloaded_framebuffer, to_ctypes)

pytestmark = pytest.mark.gpu

f32 = np.float32
PASS_PATHS = 512 << 20          # paths per pass


def short_scene(res):
    return scene.load_scene(synth.cornell_box(res=res, spp=4, max_bounces=1))


def index_bits(n):
    return max(int(n) - 1, 0).bit_length()


def read_sample(ctx, s, tiles, mean, count):
    """Every pixel of `tiles`' sample of index s, into the full-image arrays (mean, count) in place: count 1 = the sample,
    count 0 = the sample was not finite (dropped).  Pixels outside the tiles stay 0."""
    ctx.clear()
    ctx.render_resident(1, spp_begin=s, tiles=tiles)
    assert ctx.L.tgb200_read_framebuffer(ctx.h, mean.ctypes.data, count.ctypes.data) == 0


@np.errstate(all="ignore")
def fold_sample(mean, count, m, c):
    """add_sample for every pixel at once: pixels with c == 1 take m (float32, divisor float(count + 1) from uint32), the
    others keep their state."""
    ok = c == 1
    n = (count + np.uint32(1)).astype(f32)
    np.copyto(mean, mean + (m - mean)/n[..., None], where=ok[..., None])
    count += ok.astype(np.uint32)


def tiles_subset(tiles, idx):
    return (abi.Tile*len(idx))(*[tiles[i] for i in idx])


def block_mask(tiles, w, h):
    """The 4x4 blocks the tiles cover, as a flat mask over the records."""
    var_w, var_h = (w + 3)//4, (h + 3)//4
    mask = np.zeros((var_h, var_w), bool)
    for t in tiles:
        mask[t.y//4:(t.y + t.h + 3)//4, t.x//4:(t.x + t.w + 3)//4] = True
    return mask.reshape(-1)


def random_welford(n, seed):
    """Records with Welford state already in them and no samples to render."""
    rng = np.random.default_rng(seed)
    rec = np.zeros(n, RECORD)
    rec["sample_count"] = rng.integers(1, 50, n)
    rec["mean"] = rng.uniform(0.0, 2.0, n)
    rec["running_variance"] = rng.uniform(0.0, 5.0, n)
    rec["adaptive_weight"] = rng.uniform(0.0, 1.0, n)
    rec["sample_index"] = rng.integers(0, 1 << 20, n)
    return rec


# ---- 1. uniform steps of more than one sub-step -------------------------------------------------------------------------
UNIFORM = [((1024, 1024), 0, 520),                   # sub-steps of 512 + 8 samples
           ((1024, 1024), (1 << 32) - 520, 520),     # ... the second ending at sample index 0xFFFFFFFF
           ((1500, 1000), 0, 400)]                   # 357 + 43: the pixel count is not a power of two


@pytest.mark.parametrize("res,spp_begin,spp_count", UNIFORM, ids=["1024x1024-from-0", "1024x1024-to-0xFFFFFFFF", "1500x1000"])
def test_uniform_step_in_sub_steps(res, spp_begin, spp_count):
    """One render_tiles call over the whole image, more than 512 Mi paths, onto a framebuffer preloaded with counts around
    2^24: every pixel must fold samples spp_begin .. spp_begin + spp_count - 1 in order, as 1-spp calls of each index give
    them (folded as they come: a table of the rows would keep gigabytes on the host)."""
    w, h = res
    sub = PASS_PATHS//(w*h)
    assert 1 <= spp_count - sub < sub and spp_begin + spp_count - 1 <= 0xFFFFFFFF
    fs = short_scene(res)
    mean, count = preloaded_framebuffer(w, h)
    ctx = lib.Context(fs)
    try:
        got = ctx.render_tiles(spp_count, spp_begin=spp_begin, mean=mean.copy(), count=count.copy())
    finally:
        ctx.close()
    one = lib.Context(fs)
    m, c = np.zeros_like(mean), np.zeros_like(count)
    try:
        for s in range(spp_begin, spp_begin + spp_count):
            read_sample(one, s, None, m, c)
            fold_sample(mean, count, m, c)
    finally:
        one.close()
    assert_image_equal(got, (mean, count), "%dx%d, samples %d + %d" % (w, h, spp_begin, spp_count))


# ---- 2. adaptive blocks around the path-id limit --------------------------------------------------------------------------
class CoveredRow:
    """A row of samples kept for the covered pixels only, indexed [y, x] like a full image."""

    def __init__(self, values, slot):
        self.values, self.slot = values, slot

    def __getitem__(self, yx):
        return self.values[self.slot[yx]]


class CoveredSampleTable(SampleTable):
    """SampleTable that keeps only its tiles' pixels of each row: a full 4K row is 100 MB, and a hot block needs 1000."""

    def __init__(self, fs, tiles):
        super().__init__(fs, tiles)
        self.flat = np.flatnonzero(self.covered)
        self.slot = np.full(self.covered.shape, -1, np.int32)
        self.slot.flat[self.flat] = np.arange(len(self.flat))
        self.mean = np.zeros(self.covered.shape + (3,), f32)
        self.count = np.zeros(self.covered.shape, np.uint32)

    def __getitem__(self, s):
        if s not in self.rows:
            read_sample(self.ctx, s, self.tiles, self.mean, self.count)
            c = self.count.reshape(-1)[self.flat]
            m = self.mean.reshape(-1, 3)[self.flat]
            assert c.max() <= 1
            m[c == 0] = np.inf
            self.non_finite += int((c == 0).sum())
            self.rows[s] = CoveredRow(m, self.slot)
        return self.rows[s]


# image -> per-pixel sample counts of the hot blocks, about the limit 2^(32 - pix_bits) of a pass over the whole image
# (3840x2160: 8.3 M pixels, pix_bits 23, limit 512; 4099x2051 has just over 2^23 pixels: pix_bits 24, limit 256, and ragged
# right and bottom tiles)
HOT = {(3840, 2160): [511, 512, 513, 600, 1000], (4099, 2051): [255, 256, 257, 300, 500]}


@pytest.mark.parametrize("res", list(HOT), ids=["%dx%d" % r for r in HOT])
def test_adaptive_blocks_past_the_path_id_limit(res):
    """The whole tile list; every block at 0 samples except five hot ones in three tiles (the first, one in the middle, and
    the last, whose blocks are partial on the ragged image), with non-zero Welford state and a preloaded framebuffer."""
    w, h = res
    counts = HOT[res]
    assert counts[1] == 1 << (32 - index_bits(w*h))
    fs = short_scene(res)
    tiles = integrator.dice_tiles(w, h, SEED)
    var_w = (w + 3)//4
    rec = random_welford(var_w*((h + 3)//4), seed=w)
    rec["next_sample_count"] = 0
    hot_tiles = [0, len(tiles)//2 + 7, len(tiles) - 1]
    hot = []
    # (hot tile, block column, block row within it, clamped to the tile) of each count
    for k, ((j, dx, dy), n) in enumerate(zip([(0, 0, 0), (0, 3, 2), (1, 1, 1), (1, 2, 3), (2, 3, 3)], counts)):
        t = tiles[hot_tiles[j]]
        b = min(t.x//4 + dx, (t.x + t.w - 1)//4) + min(t.y//4 + dy, (t.y + t.h - 1)//4)*var_w
        assert rec[b]["next_sample_count"] == 0
        rec[b]["next_sample_count"], rec[b]["sample_index"] = n, 250 + k     # rows 250.. cross Sobol's 256 boundary
        hot.append(b)
    mean, count = preloaded_framebuffer(w, h)
    ctx = lib.Context(fs)
    try:
        ctx.write_framebuffer(mean, count)
        records = to_ctypes(rec)
        ctx.render_adaptive(records, tiles=tiles)
        got, got_rec = ctx.read_framebuffer(), as_records(records)
    finally:
        ctx.close()
    table = CoveredSampleTable(fs, tiles_subset(tiles, hot_tiles))
    try:
        want_mean, want_count, want_rec = expected_adaptive_step(mean, count, rec, table, w, h)
    finally:
        table.close()
    assert_image_equal(got, (want_mean, want_count), "%dx%d" % res)
    assert_records_equal(got_rec, want_rec, "%dx%d" % res)
    assert (got_rec["sample_count"][hot] > rec["sample_count"][hot]).all()


# ---- 3. adaptive steps past 512 Mi and past 2^32 paths ------------------------------------------------------------------
BIG = [((1024, 1024), 520), ((2048, 2048), 1025)]      # 545 M and 4.3 G paths in one step


@pytest.mark.parametrize("res,n", BIG, ids=["%dx%d-%d" % (r + (n,)) for r, n in BIG])
def test_adaptive_step_past_one_pass(res, n):
    """Every block at n samples, one render_adaptive call over the whole tile list, against the same records rendered by
    calls over disjoint parts of the list that each fit one pass; each block's record is taken from the call whose tiles
    hold it (a call leaves the other blocks' records as they were, which is checked too)."""
    w, h = res
    assert w*h*n > PASS_PATHS
    fs = short_scene(res)
    tiles = integrator.dice_tiles(w, h, SEED)
    rec = random_welford(((w + 3)//4)*((h + 3)//4), seed=n)
    rec["next_sample_count"] = n
    mean, count = preloaded_framebuffer(w, h)
    ctx = lib.Context(fs)
    try:
        ctx.write_framebuffer(mean, count)
        records = to_ctypes(rec)
        ctx.render_adaptive(records, tiles=tiles)
        got, got_rec = ctx.read_framebuffer(), as_records(records)
    finally:
        ctx.close()
    part = (128 << 20)//(256*n)                     # tiles per reference call: at most 128 Mi paths
    ref = lib.Context(fs)
    want_rec = rec.copy()
    try:
        ref.write_framebuffer(mean, count)
        for a in range(0, len(tiles), part):
            sub = tiles_subset(tiles, range(a, min(a + part, len(tiles))))
            records = to_ctypes(rec)
            ref.render_adaptive(records, tiles=sub)
            out, inside = as_records(records), block_mask(sub, w, h)
            assert_records_equal(out[~inside], rec[~inside], "outside tiles %d.." % a)
            want_rec[inside] = out[inside]
        want = ref.read_framebuffer()
    finally:
        ref.close()
    assert (want_rec["sample_count"] == rec["sample_count"] + 16*n).all()
    assert_image_equal(got, want, "%dx%d at %d" % (w, h, n))
    assert_records_equal(got_rec, want_rec, "%dx%d at %d" % (w, h, n))


def test_tile_past_one_pass_is_refused():
    """A tile whose own samples do not fit one pass (more than 512 Mi paths, or a pixel count past its path ids) is refused
    before anything renders, naming the tile; the framebuffer and records stay as they were."""
    w, h = 64, 48
    fs = short_scene((w, h))
    tiles = integrator.dice_tiles(w, h, SEED)
    var_w = (w + 3)//4
    mean, count = preloaded_framebuffer(w, h)
    ctx = lib.Context(fs)
    try:
        ctx.write_framebuffer(mean, count)
        for blocks, n in (([5 + var_w], (1 << 24) + 1), ([4 + i + j*var_w for i in range(4) for j in range(4)], (1 << 21) + 1)):
            rec = random_welford(var_w*((h + 3)//4), seed=n)
            rec["next_sample_count"] = 1
            rec["next_sample_count"][blocks] = n
            records = to_ctypes(rec)
            with pytest.raises(lib.TgbError) as e:
                ctx.render_adaptive(records, tiles=tiles)
            assert e.value.code == abi.TGB_ERR_UNSUPPORTED and "tile 1 " in str(e.value)
            assert_records_equal(as_records(records), rec, "refused")
            assert_image_equal(ctx.read_framebuffer(), (mean, count), "refused")
    finally:
        ctx.close()


# ---- 4. steps that fit one pass render as before ----------------------------------------------------------------------
# tests/golden/cornell_adaptive through the twin (three 16-spp steps) at the commit before adaptive steps were split into
# tile runs, on an H100 80GB HBM3 (700 W power limit): SHA-256 prefixes of the framebuffer (mean then count bytes) and of the final records,
# and the context's kernel launches.
CORNELL_ADAPTIVE = {"framebuffer": "6597263c88b9673a", "records": "1bf53e548ff1fd17", "kernel_launches": 621}


def test_cornell_adaptive_as_before():
    fs = scene.load_scene(os.path.join(G, "cornell_adaptive", "scene.json"))
    it = integrator.B200PathTraceIntegrator()
    it.prepareForRender(fs, SEED)
    try:
        while not it.done():
            it.startRender()
            it.waitForCompletion()
        mean, count = it.context.read_framebuffer()
        got = {"framebuffer": hashlib.sha256(mean.tobytes() + count.tobytes()).hexdigest()[:16],
               "records": hashlib.sha256(bytes(it.records)).hexdigest()[:16],
               "kernel_launches": int(it.context.stats().kernel_launches)}
    finally:
        it.teardownAfterRender()
    assert got == CORNELL_ADAPTIVE
