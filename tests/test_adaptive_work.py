"""tgb200_generate_work against a plain restatement of the reference's adaptive sampling bookkeeping, bit for bit.

PathTraceIntegrator::generateWork, errorPercentile95, dilateAdaptiveWeights and distributeAdaptiveSamples
(PathTraceIntegrator.cpp:44-134) and SampleRecord::errorEstimate (SampleRecord.hpp:57-65) are restated below one float32
operation at a time, with the double totalWeight, Tungsten's min / max (math/MathUtil.hpp:10-26: a < b ? a : b and
a > b ? a : b, which differ from std::min / std::max when an operand is NaN) and the integrator's PCG stream drawn through
integrator.UniformSampler.  The library must agree on every record field, the sampler state and the return code.

The reference overflows `int` in (spp - 1)*w*h and in int(fractionalSamples) past 2^31; both sides are undefined there, so
no case here goes near it (the restatement asserts that it stays in range).
"""
import ctypes as C
import os

import numpy as np
import pytest

from tungsten_b200 import abi, integrator, lib

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
f32 = np.float32
ADAPTIVE_THRESHOLD = 16         # PathTraceIntegrator::AdaptiveThreshold
RECORD = np.dtype([("sample_count", "<u4"), ("next_sample_count", "<u4"), ("sample_index", "<u4"),
                   ("adaptive_weight", "<f4"), ("mean", "<f4"), ("running_variance", "<f4")])
assert RECORD.itemsize == C.sizeof(abi.SampleRecord)


def t_min(a, b):
    return a if a < b else b


def t_max(a, b):
    return a if a > b else b


def next1d(sampler):
    """UniformSampler::next1D: normalizedUint(nextI()) (math/BitManip.hpp:47-50)."""
    return np.array([(sampler.next_i() >> 9) | 0x3F800000], np.uint32).view(np.float32)[0] - f32(1.0)


@np.errstate(all="ignore")
def error_estimate(count, mean, running_variance):
    """SampleRecord::errorEstimate: variance() = runningVariance/(sampleCount - 1) in uint32, then float."""
    variance = f32(running_variance)/f32((int(count) - 1) & 0xFFFFFFFF)
    return variance/(f32(count)*t_max(f32(mean)*f32(mean), f32(1e-3)))


@np.errstate(all="ignore")
def generate_work(rec, res_x, res_y, current_spp, next_spp, adaptive, sampler):
    """PathTraceIntegrator::generateWork on a RECORD array (modified in place); returns 1 = work, 0 = skip."""
    var_w, var_h = (res_x + 3)//4, (res_y + 3)//4
    n = var_w*var_h
    assert len(rec) == n
    rec["sample_index"] += rec["next_sample_count"]             # uint32, wraps like the reference's
    spp_count = next_spp - current_spp
    if not (adaptive and current_spp >= ADAPTIVE_THRESHOLD):
        rec["next_sample_count"] = spp_count
        return 1
    # errorPercentile95
    w = [error_estimate(r["sample_count"], r["mean"], r["running_variance"]) for r in rec]
    rec["adaptive_weight"] = w
    errors = sorted(x for x in w if x > f32(0.0))
    max_error = errors[(len(errors)*95)//100] if errors else f32(0.0)
    if max_error == f32(0.0):
        return 0
    w = [t_min(x, max_error) for x in w]
    # dilateAdaptiveWeights
    for y in range(var_h):
        for x in range(var_w):
            i = x + y*var_w
            if y < var_h - 1:
                w[i] = t_max(w[i], w[i + var_w])
            if x < var_w - 1:
                w[i] = t_max(w[i], w[i + 1])
    for y in range(var_h - 1, -1, -1):
        for x in range(var_w - 1, -1, -1):
            i = x + y*var_w
            if y > 0:
                w[i] = t_max(w[i], w[i - var_w])
            if x > 0:
                w[i] = t_max(w[i], w[i - 1])
    rec["adaptive_weight"] = w
    # distributeAdaptiveSamples
    total_weight = 0.0
    for x in w:
        total_weight += float(x)
    adaptive_budget = (spp_count - 1)*res_x*res_y
    assert -2**31 <= adaptive_budget < 2**31
    budget_per_tile = int(adaptive_budget/16)                   # C's integer division truncates toward zero
    weight_to_sample = f32(np.float64(budget_per_tile)/np.float64(total_weight))
    pixel_pdf = f32(0.0)
    counts = []
    for x in w:
        fractional = x*weight_to_sample
        assert abs(fractional) < 2**31
        samples = int(fractional)
        pixel_pdf = pixel_pdf + (fractional - f32(samples))
        if next1d(sampler) < pixel_pdf:
            samples += 1
            pixel_pdf = pixel_pdf - f32(1.0)
        counts.append((samples + 1) & 0xFFFFFFFF)
    rec["next_sample_count"] = counts
    return 1


def library_generate_work(rec, res_x, res_y, current_spp, next_spp, adaptive, state):
    """tgb200_generate_work on a RECORD array (in place); returns (return code, sampler state)."""
    st = C.c_uint64(state)
    rc = lib.load().tgb200_generate_work(rec.ctypes.data, res_x, res_y, current_spp, next_spp, 1 if adaptive else 0, C.byref(st))
    return rc, st.value


def assert_records_equal(got, want, what=""):
    """Every field bit for bit, NaN equal to NaN."""
    for f in ("sample_count", "next_sample_count", "sample_index"):
        bad = np.flatnonzero(got[f] != want[f])
        assert bad.size == 0, "%s %s differs in %d records, first %d: %d vs %d" % (what, f, bad.size, bad[0], got[f][bad[0]], want[f][bad[0]])
    for f in ("adaptive_weight", "mean", "running_variance"):
        a, b = got[f], want[f]
        same = (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))
        bad = np.flatnonzero(~same)
        assert bad.size == 0, "%s %s differs in %d records, first %d: %r vs %r" % (what, f, bad.size, bad[0], a[bad[0]], b[bad[0]])


@np.errstate(all="ignore")
def welford(rec, lum):
    """SampleRecord::addSample(float) in float32 (SampleRecord.hpp:44-50) on one RECORD entry."""
    rec["sample_count"] = (int(rec["sample_count"]) + 1) & 0xFFFFFFFF
    mean = f32(rec["mean"])
    delta = f32(lum) - mean
    mean = mean + delta/f32(rec["sample_count"])
    rec["mean"] = mean
    rec["running_variance"] = f32(rec["running_variance"]) + delta*(f32(lum) - mean)


@np.errstate(all="ignore")
def luminance(c):
    """Vec3f::luminance (math/Vec.hpp:195-199): c.x*0.2126f + c.y*0.7152f + c.z*0.0722f, left to right."""
    return f32(c[0])*f32(0.2126) + f32(c[1])*f32(0.7152) + f32(c[2])*f32(0.0722)


def check(rec, res_x, res_y, current_spp, next_spp, adaptive=True, state=0x853C49E6748FEA9B):
    """Library vs restatement on copies of `rec`; returns the restatement's records and return code."""
    got, want = rec.copy(), rec.copy()
    rc, st = library_generate_work(got, res_x, res_y, current_spp, next_spp, adaptive, state)
    sampler = integrator.UniformSampler(state)
    want_rc = generate_work(want, res_x, res_y, current_spp, next_spp, adaptive, sampler)
    assert rc == want_rc
    assert st == sampler.state
    assert_records_equal(got, want, "%dx%d spp %d->%d" % (res_x, res_y, current_spp, next_spp))
    return want, want_rc


def random_records(res_x, res_y, seed):
    """Records as a 16-spp step leaves them: 16..400 samples, luminance means over decades, variances from 0 up."""
    rng = np.random.default_rng(seed)
    n = ((res_x + 3)//4)*((res_y + 3)//4)
    rec = np.zeros(n, RECORD)
    rec["sample_count"] = rng.integers(16, 400, n)
    rec["next_sample_count"] = rng.integers(1, 64, n)
    rec["sample_index"] = rng.integers(0, 1 << 20, n)
    rec["adaptive_weight"] = rng.standard_normal(n).astype(np.float32)      # stale: generateWork overwrites it
    rec["mean"] = np.exp(rng.uniform(-8.0, 4.0, n)).astype(np.float32)
    rec["running_variance"] = (rec["mean"]**2*rng.exponential(1.0, n)*rec["sample_count"]).astype(np.float32)
    rec["running_variance"][rng.random(n) < 0.05] = 0.0
    return rec


RESOLUTIONS = [(1, 1), (3, 5), (17, 9), (50, 37), (1920, 1080)]


@pytest.mark.parametrize("res", RESOLUTIONS, ids=["%dx%d" % r for r in RESOLUTIONS])
@pytest.mark.parametrize("current_spp", [15, 16])
def test_random_records(res, current_spp):
    """Random finite records on either side of the adaptive threshold; at 16 spp and above the budget is redistributed."""
    rec = random_records(*res, seed=res[0]*7919 + res[1])
    want, rc = check(rec, *res, current_spp, current_spp + 16)
    assert rc == 1
    assert np.array_equal(want["sample_index"], rec["sample_index"] + rec["next_sample_count"])
    if current_spp < ADAPTIVE_THRESHOLD:
        assert (want["next_sample_count"] == 16).all()
        assert np.array_equal(want["adaptive_weight"].view(np.uint32), rec["adaptive_weight"].view(np.uint32))
    elif len(rec) > 20:
        assert len(np.unique(want["next_sample_count"])) > 3


def test_adaptive_sampling_off():
    rec = random_records(50, 37, seed=3)
    want, rc = check(rec, 50, 37, 32, 48, adaptive=False)
    assert rc == 1 and (want["next_sample_count"] == 16).all()


def test_all_zero_error_skips_the_step():
    """Zero error everywhere: returns 0 and draws nothing, but sample_index still advances (generateWork's first loop)."""
    rec = random_records(17, 9, seed=5)
    rec["running_variance"] = 0.0
    want, rc = check(rec, 17, 9, 16, 32)
    assert rc == 0
    assert np.array_equal(want["sample_index"], rec["sample_index"] + rec["next_sample_count"])
    assert np.array_equal(want["next_sample_count"], rec["next_sample_count"])


def test_one_sample_per_block():
    """sample_count 1: variance() = x/0 (Inf weight, kept out of reach of the percentile) or 0/0 (NaN weight)."""
    rec = random_records(50, 37, seed=7)
    rec["sample_count"][::37] = 1
    rec["running_variance"][::74] = 0.0
    assert np.isnan([error_estimate(r["sample_count"], r["mean"], r["running_variance"]) for r in rec]).any()
    assert np.isinf([error_estimate(r["sample_count"], r["mean"], r["running_variance"]) for r in rec]).any()
    check(rec, 50, 37, 16, 32)


@pytest.mark.parametrize("res", [(50, 37), (17, 9), (3, 5)], ids=["50x37", "17x9", "3x5"])
def test_non_finite_means(res):
    """Mean 0; a NaN mean (max(NaN, 1e-3) = 1e-3: a finite weight); a block whose mean overflowed to Inf, which leaves
    running_variance NaN (a NaN weight, clamped to the percentile by min(NaN, maxError) = maxError)."""
    rec = random_records(*res, seed=11)
    n = len(rec)
    rec["mean"][0] = 0.0
    rec["mean"][n//2] = np.nan
    rec["mean"][n - 1] = np.inf
    rec["running_variance"][n - 1] = np.nan
    want, rc = check(rec, *res, 16, 32)
    assert rc == 1
    assert np.isfinite(want["adaptive_weight"]).all()
    assert want["next_sample_count"].max() < 10000


def test_inf_mean_block_keeps_the_step_going():
    """One overflowing sample before the threshold: its block has mean = Inf and running_variance = NaN.  The reference gives
    that block the largest weight and redistributes as usual; every block keeps a sensible sample count."""
    res = (32, 32)
    rec = random_records(*res, seed=13)
    good, _ = check(rec, *res, 16, 32)
    rec["mean"][20] = np.inf
    rec["running_variance"][20] = np.nan
    want, _ = check(rec, *res, 16, 32)
    assert want["next_sample_count"].max() <= good["next_sample_count"].max() + 64
    assert int(want["next_sample_count"].sum()) < 2*16*res[0]*res[1]


def test_slightly_negative_running_variance():
    """Welford's running variance can round below zero for constant samples: a negative weight, outside the percentile."""
    rec = random_records(50, 37, seed=17)
    rec["running_variance"][::5] = -np.float32(1e-7)*rec["mean"][::5]**2
    check(rec, 50, 37, 16, 32)


def test_weights_tied_with_the_percentile():
    """21 blocks share one weight, which is also the 95th percentile."""
    rec = random_records(160, 120, seed=19)
    w = np.array([error_estimate(r["sample_count"], r["mean"], r["running_variance"]) for r in rec])
    pos = np.flatnonzero(w > 0)
    by_rank = pos[np.argsort(w[pos], kind="stable")]
    p = (len(pos)*95)//100
    tied = by_rank[p - 10:p + 11]                 # replacing ranks p-10..p+10 with the weight of rank p leaves the others in place
    for f in ("sample_count", "mean", "running_variance"):
        rec[f][tied] = rec[f][by_rank[p]]
    w = [error_estimate(r["sample_count"], r["mean"], r["running_variance"]) for r in rec]
    errors = sorted(x for x in w if x > 0)
    assert errors[p - 10] == errors[p] == errors[p + 10]
    check(rec, 160, 120, 16, 32)


@pytest.mark.parametrize("n_positive", [1, 2, 7, 19])
def test_short_error_lists(n_positive):
    """Fewer than 20 positive errors: the percentile index (n*95)/100 lands on or near the largest."""
    rec = random_records(50, 37, seed=23 + n_positive)
    rng = np.random.default_rng(n_positive)
    keep = rng.choice(len(rec), n_positive, replace=False)
    rv = rec["running_variance"].copy()
    rec["running_variance"] = 0.0
    rec["running_variance"][keep] = np.maximum(rv[keep], 1e-3)
    want, rc = check(rec, 50, 37, 16, 32)
    assert rc == 1


def oracle_sample_table(fs, tiles, seed, indices):
    """{sample index: (h, w, 3) radiance of every pixel's sample of that index}, from the CPU oracle; non-finite samples
    (dropped by OutputBuffer::addSample, count 0) as +Inf."""
    from oracle import pyoracle
    w, h = fs.resolution
    orc = pyoracle.Oracle(fs)
    table = {}
    try:
        for s in indices:
            m, c = orc.render(1, seed=seed, spp_begin=s, tiles=tiles)
            m[c == 0] = np.inf
            table[s] = m
    finally:
        orc.close()
    return table


def fold_block_stats(rec, table, res_x, res_y):
    """renderTile's SampleRecord::addSample calls (PathTraceIntegrator.cpp:136-156) for every pixel: per block, rows, then
    columns, then sample index."""
    var_w = (res_x + 3)//4
    for b in range(len(rec)):
        r = rec[b]
        bx, by = (b % var_w)*4, (b//var_w)*4
        n, base = int(r["next_sample_count"]), int(r["sample_index"])
        for y in range(by, min(by + 4, res_y)):
            for x in range(bx, min(bx + 4, res_x)):
                for k in range(n):
                    welford(r, luminance(table[base + k][y, x]))


def test_cornell_adaptive_chain():
    """The three 16-spp steps of tests/golden/cornell_adaptive (the scene the reference binary rendered adaptively): before
    each step the library and the restatement distribute the same samples from the same records and sampler state; the
    records are then folded with the oracle's samples as renderTile folds them."""
    from tungsten_b200 import scene
    fs = scene.load_scene(os.path.join(G, "cornell_adaptive", "scene.json"))
    assert fs.adaptive and fs.spp == 48 and fs.spp_step == 16
    w, h = fs.resolution
    seed = 0xBA5EBA11
    sampler = integrator.UniformSampler(integrator.hash32(seed))
    tiles = integrator.dice_tiles(w, h, seed, sampler)
    rec = np.zeros(((w + 3)//4)*((h + 3)//4), RECORD)
    table = {}
    cur, steps = 0, 0
    while cur < fs.spp:
        nxt = min(cur + fs.spp_step, fs.spp)
        want = rec.copy()
        rc, st = library_generate_work(rec, w, h, cur, nxt, True, sampler.state)
        want_rc = generate_work(want, w, h, cur, nxt, True, sampler)
        assert rc == want_rc == 1 and st == sampler.state
        assert_records_equal(rec, want, "step %d" % steps)
        need = set(range(int(rec["sample_index"].min()), int((rec["sample_index"] + rec["next_sample_count"]).max())))
        table.update(oracle_sample_table(fs, tiles, seed, sorted(need - set(table))))
        fold_block_stats(rec, table, w, h)
        cur, steps = nxt, steps + 1
    assert steps == 3
    assert rec["sample_count"].min() >= 16*16 + 2*16 and rec["next_sample_count"].max() > 16
