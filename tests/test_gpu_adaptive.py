"""Adaptive sampling's bookkeeping on the GPU, bit for bit: which samples each pixel renders, how they fold into the image
(OutputBuffer::addSample) and into the 4x4 block records (SampleRecord::addSample).

Both sides use the GPU's own samples, so a difference can only be bookkeeping.  A path depends on nothing but its pixel, its
sample index and its tile's seed (DESIGN.md section 3), so a 1-spp render_tiles call of sample index s into a fresh
framebuffer gives every pixel's sample s: count 1 means the mean IS the sample (0 + (c - 0)/1), count 0 means the sample was
not finite.  A dropped sample's luminance is taken as +Inf: the fold then leaves running_variance NaN, and the mean NaN after
any later sample, exactly as a NaN luminance would; only a block whose last sample is dropped could tell the two apart
(mean Inf or NaN), and the comparison would show it.  The expected image and records are the float32 folds of those samples in the reference's
order (PathTraceIntegrator::renderTile, PathTraceIntegrator.cpp:136-156: per block rows, then columns, then sample index).
"""
import ctypes as C
import os

import numpy as np
import pytest

from tungsten_b200 import abi, integrator, lib, scene, synth
from test_adaptive_work import RECORD, assert_records_equal, check, library_generate_work, luminance, welford

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SEED = 0xBA5EBA11
f32 = np.float32
CAPACITIES = [0, 1021, 1500]      # default, and small enough that the slot-to-pixel search runs across many refills


class SampleTable:
    """Every pixel's sample of a given sample index, rendered on a context of its own with tile list `tiles`."""

    def __init__(self, fs, tiles):
        self.ctx = lib.Context(fs)
        self.tiles = tiles
        self.rows = {}
        self.non_finite = 0             # dropped samples among the covered pixels' rows looked up so far
        w, h = fs.resolution
        self.covered = np.zeros((h, w), bool)
        for t in tiles:
            self.covered[t.y:t.y + t.h, t.x:t.x + t.w] = True

    def __getitem__(self, s):
        if s not in self.rows:
            m, c = self.ctx.render_tiles(1, spp_begin=s, tiles=self.tiles)
            assert c.max() <= 1 and (c[~self.covered] == 0).all()
            m[c == 0] = np.inf
            self.non_finite += int((self.covered & (c == 0)).sum())
            self.rows[s] = m
        return self.rows[s]

    def close(self):
        self.ctx.close()


def add_sample(mean, count, y, x, c):
    """OutputBuffer::addSample (cameras/OutputBuffer.hpp:104-132) in float32: non-finite samples are dropped, the divisor is
    float(sampleIdx + 1) from uint32."""
    if not np.isfinite(c).all():
        return
    n = f32((int(count[y, x]) + 1) & 0xFFFFFFFF)
    count[y, x] += 1
    mean[y, x] = mean[y, x] + (c - mean[y, x])/n


def expected_adaptive_step(mean, count, rec, table, w, h):
    """tgb200_render_adaptive as renderTile does it: every covered pixel of block b renders rec[b].next_sample_count samples
    from rec[b].sample_index on."""
    mean, count, rec = mean.copy(), count.copy(), rec.copy()
    var_w = (w + 3)//4
    for b in range(len(rec)):
        r = rec[b]
        bx, by = (b % var_w)*4, (b//var_w)*4
        n, base = int(r["next_sample_count"]), int(r["sample_index"])
        if n == 0:
            continue
        for y in range(by, min(by + 4, h)):
            for x in range(bx, min(bx + 4, w)):
                if not table.covered[y, x]:
                    continue
                for k in range(n):
                    c = table[base + k][y, x]
                    welford(r, luminance(c))
                    add_sample(mean, count, y, x, c)
    return mean, count, rec


def expected_uniform(mean, count, table, spp_begin, spp_count):
    mean, count = mean.copy(), count.copy()
    for y, x in zip(*np.nonzero(table.covered)):
        for k in range(spp_count):
            add_sample(mean, count, y, x, table[spp_begin + k][y, x])
    return mean, count


def as_records(records):
    return np.frombuffer(bytes(records), RECORD).copy()


def to_ctypes(rec):
    out = (abi.SampleRecord*len(rec))()
    C.memmove(out, rec.tobytes(), rec.nbytes)
    return out


def assert_image_equal(got, want, what):
    gm, gc = got
    wm, wc = want
    bad = np.argwhere(gc != wc)
    assert bad.size == 0, "%s: %d pixel counts differ, first %s: %d vs %d" % (what, len(bad), bad[0], gc[tuple(bad[0])], wc[tuple(bad[0])])
    bad = np.argwhere((gm.view(np.uint32) != wm.view(np.uint32)).any(axis=2))
    assert bad.size == 0, "%s: %d pixel means differ, first %s: %r vs %r" % (what, len(bad), bad[0], gm[tuple(bad[0])], wm[tuple(bad[0])])


def render_through_twin(fs, cap=0):
    """The Integrator twin's loop (render()), the framebuffer and records taken around each tgb200_render_adaptive call;
    every step compared with the folds of the GPU's own samples."""
    it = integrator.B200PathTraceIntegrator(max_paths_in_flight=cap)
    it.prepareForRender(fs, SEED)
    ctx = it.context
    w, h = fs.resolution
    steps = []
    render = ctx.render_adaptive

    def spy(records, seed, tiles):
        before = ctx.read_framebuffer(), as_records(records)
        render(records, seed=seed, tiles=tiles)
        steps.append((before, as_records(records), ctx.read_framebuffer()))
    ctx.render_adaptive = spy
    table = SampleTable(fs, it.tiles)
    try:
        while not it.done():
            it.startRender()
            it.waitForCompletion()
        for i, ((fb, rec), got_rec, got_fb) in enumerate(steps):
            want_mean, want_count, want_rec = expected_adaptive_step(fb[0], fb[1], rec, table, w, h)
            assert_image_equal(got_fb, (want_mean, want_count), "step %d" % i)
            assert_records_equal(got_rec, want_rec, "step %d" % i)
    finally:
        it.teardownAfterRender()
        table.close()
    return steps, table.non_finite


def test_cornell_adaptive_through_the_twin():
    """tests/golden/cornell_adaptive end to end: three 16-spp steps, the 2nd and 3rd distributed by the library's
    tgb200_generate_work."""
    fs = scene.load_scene(os.path.join(G, "cornell_adaptive", "scene.json"))
    assert fs.adaptive and fs.spp == 48 and fs.spp_step == 16
    steps, _ = render_through_twin(fs)
    assert len(steps) == 3
    assert len(np.unique(steps[1][0][1]["next_sample_count"])) > 3       # the 2nd step really was redistributed


def overflowing_light_scene(res=(32, 32)):
    """The Cornell box with a second quad light whose emission (3.4e38) is finite but overflows to +Inf in some samples."""
    hot = {"name": "hot", "transform": {"position": [0.5, 1.97, 0.5], "scale": [0.9, 1, 0.9], "rotation": [0, 0, 180]},
           "type": "quad", "bsdf": "light", "emission": [3.4e38, 3.4e38, 3.4e38]}
    sc = synth.cornell_box(res=res, spp=32, extra_prims=[hot])
    sc["renderer"].update(adaptive_sampling=True, spp_step=16)
    return scene.load_scene(sc)


def test_overflowing_samples_through_the_twin():
    """Samples that overflow to +Inf are dropped from the image but still folded into their block's record (mean = Inf,
    then NaN; running_variance NaN): the first step matches exactly, and generateWork on the records the GPU left agrees
    with the restatement.  (The hot light lights every block, so every block's mean*mean overflows too: all errors are 0 or
    NaN and the reference skips the second step, as the library does.)"""
    fs = overflowing_light_scene()
    steps, non_finite = render_through_twin(fs)
    print("overflowing light: %d non-finite samples on the GPU" % non_finite)
    assert non_finite >= 1
    rec1 = steps[0][1]
    assert not np.isfinite(rec1["mean"]).all()
    check(rec1, *fs.resolution, 16, 32)


def test_nan_weight_block_gets_the_next_step():
    """One block left as an overflowing sample leaves it (mean = Inf, running_variance = NaN) among finite blocks: its NaN
    error is clamped to the 95th percentile (Tungsten's min), the other blocks keep their counts, and the next adaptive
    step renders and matches exactly."""
    fs = scene.load_scene(os.path.join(G, "cornell_adaptive", "scene.json"))
    w, h = fs.resolution
    sampler = integrator.UniformSampler(integrator.hash32(SEED))
    tiles = integrator.dice_tiles(w, h, SEED, sampler)
    table = SampleTable(fs, tiles)
    ctx = lib.Context(fs)
    try:
        rec = np.zeros(((w + 3)//4)*((h + 3)//4), RECORD)
        mean, count = ctx.read_framebuffer()
        for cur in (0, 16):
            if cur == 16:
                rec[5]["mean"], rec[5]["running_variance"] = np.inf, np.nan
                check(rec, w, h, cur, cur + 16, state=sampler.state)
            rc, sampler.state = library_generate_work(rec, w, h, cur, cur + 16, True, sampler.state)
            assert rc == 1
            records = to_ctypes(rec)
            ctx.render_adaptive(records, tiles=tiles)
            want_mean, want_count, want_rec = expected_adaptive_step(mean, count, rec, table, w, h)
            mean, count = ctx.read_framebuffer()
            assert_image_equal((mean, count), (want_mean, want_count), "from %d spp" % cur)
            assert_records_equal(as_records(records), want_rec, "from %d spp" % cur)
            rec = as_records(records)
        assert 1 <= rec["next_sample_count"].min() and rec["next_sample_count"].max() < 1000
    finally:
        ctx.close()
        table.close()


def ragged_scene():
    return scene.load_scene(synth.cornell_box(res=(50, 37), spp=4))


@pytest.fixture(scope="module")
def ragged():
    """The 50x37 scene, a shuffled partial tile list and its sample table, shared by the tests that render with them."""
    fs = ragged_scene()
    tiles = partial_tiles(fs)
    table = SampleTable(fs, tiles)
    yield fs, tiles, table
    table.close()


def partial_tiles(fs, keep=7, seed=1):
    """A shuffled subset of the tile list (12 tiles for 50x37, with ragged right and bottom tiles)."""
    tiles = list(integrator.dice_tiles(*fs.resolution, SEED))
    rng = np.random.default_rng(seed)
    order = rng.permutation(len(tiles))[:keep]
    assert any(tiles[i].w % 4 for i in order) and any(tiles[i].h % 4 for i in order)
    return (abi.Tile*keep)(*[tiles[i] for i in order])


# (sample_index, next_sample_count): none, one, the Sobol index's 256 boundary, up to 2^32 without crossing it, many
BLOCK_RANGES = [(0, 0), (255, 1), (256, 3), (250, 12), (0xFFFFFFF0, 16), (4, 300), (1000, 0), (0xFFFFFFFE, 1), (17, 2)]
PRELOAD_COUNTS = [0, 7, (1 << 24) - 1, 1 << 24, (1 << 24) + 1]


def hand_made_records(n_blocks, seed=2):
    rng = np.random.default_rng(seed)
    rec = np.zeros(n_blocks, RECORD)
    for b in range(n_blocks):
        rec[b]["sample_index"], rec[b]["next_sample_count"] = BLOCK_RANGES[b % len(BLOCK_RANGES)]
    rec["sample_count"] = rng.integers(0, 50, n_blocks)           # Welford state already in the records
    rec["mean"] = rng.uniform(0.0, 2.0, n_blocks)
    rec["running_variance"] = rng.uniform(0.0, 5.0, n_blocks)
    rec["adaptive_weight"] = rng.uniform(0.0, 1.0, n_blocks)
    return rec


def preloaded_framebuffer(w, h, seed=3):
    rng = np.random.default_rng(seed)
    # means over seven decades: where a sample's share (c - mean)/n is not lost in the mean's rounding, the last bit of
    # float(count + 1) shows
    mean = (rng.uniform(0.0, 3.0, (h, w, 3))*10.0**rng.uniform(-7.0, 0.0, (h, w, 1))).astype(np.float32)
    count = np.array(PRELOAD_COUNTS, np.uint32)[np.arange(w*h) % len(PRELOAD_COUNTS)].reshape(h, w)
    return mean, count


@pytest.mark.parametrize("cap", CAPACITIES)
def test_hand_made_records_on_a_ragged_image(ragged, cap):
    """50x37 with a shuffled partial tile list; per-block counts 0, 1, 3, 12, 16 and 300 from sample indices around 256 and
    up to 0xFFFFFFFF; non-zero Welford state; a framebuffer preloaded with counts around 2^24, where float(count + 1)
    stops being exact.  Blocks and pixels outside the tile list keep their values."""
    fs, tiles, table = ragged
    w, h = fs.resolution
    ctx = lib.Context(fs, max_paths_in_flight=cap)
    try:
        rec = hand_made_records(((w + 3)//4)*((h + 3)//4))
        mean, count = preloaded_framebuffer(w, h)
        ctx.write_framebuffer(mean, count)
        records = to_ctypes(rec)
        ctx.render_adaptive(records, tiles=tiles)
        want_mean, want_count, want_rec = expected_adaptive_step(mean, count, rec, table, w, h)
        assert_image_equal(ctx.read_framebuffer(), (want_mean, want_count), "adaptive")
        assert_records_equal(as_records(records), want_rec, "adaptive")
        assert (want_count[table.covered] > count[table.covered]).any()
    finally:
        ctx.close()


@pytest.mark.parametrize("spp_begin,spp_count", [(0, 3), (250, 12), (0xFFFFFFF0, 16)])
@pytest.mark.parametrize("cap", [0, 1021])
def test_uniform_step_with_preloads(ragged, cap, spp_begin, spp_count):
    """render_tiles with the same preloaded framebuffer and tile list: every covered pixel folds samples
    [spp_begin, spp_begin + spp_count) in order."""
    fs, tiles, table = ragged
    w, h = fs.resolution
    ctx = lib.Context(fs, max_paths_in_flight=cap)
    try:
        mean, count = preloaded_framebuffer(w, h)
        got = ctx.render_tiles(spp_count, spp_begin=spp_begin, tiles=tiles, mean=mean.copy(), count=count.copy())
        assert_image_equal(got, expected_uniform(mean, count, table, spp_begin, spp_count), "uniform")
    finally:
        ctx.close()


def test_two_devices_adaptive_step_equals_one():
    """tgb_settings::devices = [0, 1]: the records merged from the GPU that owns each tile, and the gathered framebuffer,
    equal one GPU's, on a ragged image whose last tile column and row hold partial blocks."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    fs = ragged_scene()
    w, h = fs.resolution
    rec = hand_made_records(((w + 3)//4)*((h + 3)//4))
    mean, count = preloaded_framebuffer(w, h)
    out = []
    for kw in ({"device": 0}, {"devices": [0, 1]}):
        ctx = lib.Context(fs, **kw)
        ctx.write_framebuffer(mean, count)
        records = to_ctypes(rec)
        ctx.render_adaptive(records)
        out.append((ctx.read_framebuffer(), as_records(records)))
        ctx.close()
    (fb1, rec1), (fb2, rec2) = out
    assert_image_equal(fb2, fb1, "two GPUs")
    assert_records_equal(rec2, rec1, "two GPUs")
