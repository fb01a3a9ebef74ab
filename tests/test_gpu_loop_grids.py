"""The wavefront loop's grid-stride kernels past their first trip, and the survivor sort against an exact model.

k_regen, k_shadow_prep and k_bin_scatter launch at most the blocks that can be resident at once and loop over the count in the
control block (n_new, shadow_count, n_surv).  On an H100 one trip is ~270 k items, more than most tests' batches, so at those
sizes every thread makes one trip.  TGB_LOOP_BLOCKS caps the three grids at that many blocks in total: a trip is then exactly
T = 256 x TGB_LOOP_BLOCKS items, and a 64x64 render makes dozens of trips per launch.

  * The survivor sort (k_accum's histogram, k_iter_end's scan, k_bin_scatter) through tgb200_bin_probe, against a numpy model:
    n_sorted, the visiting order (a permutation of the traversed survivors with non-decreasing keys) and every cursor exactly, on
    both sides of trip boundaries and at the wavefront's capacity.  No image can show the order, and a duplicated entry that
    displaces another touches only the few paths involved.  A CPU test checks that the model's checker rejects wrong answers.
  * Shadow queries (k_shadow_prep) and bounce states (k_bin_scatter, k_shadow_prep) at 1 and 3 blocks give the default grid's
    bytes, and more than one default trip's worth gives what one-trip chunks give.
  * A 512x512 render, whose first k_regen per wavefront has over a million paths, equals the same render in one-trip iterations.
    (The golden scenes at 1 and 5 blocks: tests/test_gpu_wavefronts.py.)
Every test prints the trips per launch it ran (at the default grid: the least any grid of resident blocks makes, at most 2048
threads per SM).
"""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import pyoracle
from tungsten_b200 import abi, lib, scene, synth
import test_gpu_bounce as bounce
import test_gpu_shadow as shadow
from test_gpu_wavefronts import SMALL, STATS, all_stats

BINS = abi.BINS
PATTERNS = ["all untraversed", "one key 0", "one key 32767", "two alternating", "t % 33", "t // 7", "uniform, 10 % untraversed",
            "zipf", "descending"]


# ---- the exact model of the sort and its checker --------------------------------------------------------------------------
def key_pattern(name, n, rng):
    t = np.arange(n, dtype=np.int64)
    if name == "all untraversed":
        k = np.full(n, BINS)
    elif name == "one key 0":
        k = np.zeros(n, np.int64)
    elif name == "one key 32767":
        k = np.full(n, BINS - 1)
    elif name == "two alternating":                                       # lane by lane: two peer groups in every warp
        k = np.where(t % 2 == 0, 9, 30001)
    elif name == "t % 33":                                                # 32 distinct keys in every warp
        k = t % 33
    elif name == "t // 7":                                                # runs that cross warp and block edges
        k = (t//7) % BINS
    elif name == "uniform, 10 % untraversed":
        k = rng.randint(0, BINS, n); k[rng.rand(n) < 0.1] = BINS
    elif name == "zipf":                                                  # a few hot bins, scattered over the key range
        k = rng.permutation(BINS)[np.minimum(rng.zipf(1.3, n) - 1, BINS - 1)]
    elif name == "descending":
        k = (n - 1 - t)*BINS//max(n, 1)
    else:
        raise ValueError(name)
    return k.astype(np.uint32)


def model_sort(keys):
    """(order, cursors, n_sorted) of a correct sort: traversed survivors by key (stable), each bin's end."""
    keys = np.asarray(keys, np.int64)
    traversed = np.flatnonzero(keys < BINS)
    order = traversed[np.argsort(keys[traversed], kind="stable")].astype(np.uint32)
    cursors = np.cumsum(np.bincount(keys[traversed], minlength=BINS)).astype(np.uint32)
    return order, cursors, len(traversed)


def sort_errors(keys, order, cursors, n_sorted):
    """What is wrong with a sort's output against the model (empty: it is right).  The order within a bin is free."""
    keys = np.asarray(keys, np.int64); order = np.asarray(order, np.int64)
    traversed = np.flatnonzero(keys < BINS)
    errors = []
    if n_sorted != len(traversed):
        errors.append("n_sorted %d, %d keys below kBins" % (n_sorted, len(traversed)))
    if len(order) != len(traversed) or not np.array_equal(np.sort(order), traversed):
        errors.append("order is not a permutation of the traversed survivors (duplicates or holes)")
    elif (np.diff(keys[order]) < 0).any():
        errors.append("keys decrease at %d positions of order" % int((np.diff(keys[order]) < 0).sum()))
    expected = np.cumsum(np.bincount(keys[traversed], minlength=BINS))
    if len(cursors) != BINS or not np.array_equal(np.asarray(cursors, np.int64), expected):
        errors.append("cursors differ from the bins' ends at %d bins" % int((np.asarray(cursors, np.int64) != expected).sum()))
    return errors


def test_checker_rejects_wrong_sorts():
    """CPU: the checker accepts the model's answer and a reordering within a bin, and rejects each kind of wrong answer."""
    rng = np.random.RandomState(7)
    keys = key_pattern("uniform, 10 % untraversed", 5000, rng)
    keys[:64] = 0                                                         # one bin with many entries
    order, cursors, n_sorted = model_sort(keys)
    assert sort_errors(keys, order, cursors, n_sorted) == []
    same_bin = order.copy(); same_bin[:cursors[0]] = same_bin[:cursors[0]][::-1]    # bin 0 in another order: still right
    assert cursors[0] >= 64 and sort_errors(keys, same_bin, cursors, n_sorted) == []
    wrong = {}
    o = order.copy(); o[10] = o[11]; wrong["a duplicate and a missing entry"] = (o, cursors, n_sorted)
    o = order.copy(); i, j = 100, 3000
    assert keys[o[i]] != keys[o[j]]
    o[[i, j]] = o[[j, i]]; wrong["two entries of different bins swapped"] = (o, cursors, n_sorted)
    c = cursors.copy(); c[keys[order[500]]] += 1; wrong["a cursor one too high"] = (order, c, n_sorted)
    c = cursors.copy(); c[BINS - 1] -= 1; wrong["the last cursor one too low"] = (order, c, n_sorted)
    wrong["n_sorted one too high"] = (order, cursors, n_sorted + 1)
    wrong["n_sorted one too low"] = (order, cursors, n_sorted - 1)
    wrong["order one entry short"] = (order[:-1], cursors, n_sorted)
    for what, (o, c, ns) in wrong.items():
        errs = sort_errors(keys, o, c, ns)
        print("%-40s -> %s" % (what, errs))
        assert errs, what


# ---- GPU --------------------------------------------------------------------------------------------------------------------
def context(fs, monkeypatch, loop_blocks=None, cap=0):
    """A context whose grid-stride kernels run at most loop_blocks blocks (None: the default grids)."""
    if loop_blocks is None:
        monkeypatch.delenv("TGB_LOOP_BLOCKS", raising=False)
    else:
        monkeypatch.setenv("TGB_LOOP_BLOCKS", str(loop_blocks))
    ctx = lib.Context(fs, max_paths_in_flight=cap)
    monkeypatch.delenv("TGB_LOOP_BLOCKS", raising=False)
    return ctx


def trips(n, loop_blocks):
    """Trips per launch of a grid-stride kernel over n items at TGB_LOOP_BLOCKS = loop_blocks."""
    return math.ceil(n/(256*min(max(math.ceil(n/256), 1), loop_blocks))) if n else 0


def least_trips(n):
    """The fewest trips any grid of resident 256-thread blocks makes over n items on this GPU (2048 threads per SM)."""
    import torch
    return math.ceil(n/(2048*torch.cuda.get_device_properties(0).multi_processor_count))


def run_sort(ctx, keys, label):
    order, cursors, n_sorted = ctx.bin_probe(keys)
    errs = sort_errors(keys, order, cursors, n_sorted)
    big = int(np.bincount(keys[keys < BINS].astype(np.int64), minlength=1).max()) if n_sorted else 0
    print("    %-28s n %8d: n_sorted %8d, largest bin %8d%s" % (label, len(keys), n_sorted, big, ", WRONG: %s" % errs if errs else ""))
    return errs


@pytest.mark.gpu
@pytest.mark.parametrize("loop_blocks", [1, 3, None], ids=["1_block", "3_blocks", "default_grid"])
def test_survivor_sort_matches_model(loop_blocks, monkeypatch):
    fs = scene.load_scene(synth.cornell_box(res=(16, 16), spp=1))
    ctx = context(fs, monkeypatch, loop_blocks)
    cap = (ctx.scene_info()["capacity"] + 1)//2                          # wavefront 0's slots
    if loop_blocks is None:
        sizes = [1, 31, 32, 33, 255, 256, 257, 600000, cap]
    else:
        T = 256*loop_blocks
        sizes = sorted({1, 31, 32, 33, 255, 256, 257, T - 1, T, T + 1, 2*T + 1, 5*T + 37})
    rng = np.random.RandomState(loop_blocks or 0)
    failed = []
    for n in sizes:
        print("TGB_LOOP_BLOCKS=%s, n = %d: %s trips per k_bin_scatter launch" % (
            loop_blocks, n, trips(n, loop_blocks) if loop_blocks else "at least %d" % least_trips(n)))
        for p in PATTERNS:
            keys = key_pattern(p, n, rng)
            if run_sort(ctx, keys, p):
                failed.append((n, p))
    ctx.close()
    assert not failed, failed


@pytest.mark.gpu
def test_bin_probe_refusals_and_context_unchanged(scratch, monkeypatch):
    """Keys past kBins, more survivors than wavefront 0 holds and missing buffers are refused; kBins itself and n = 0 are not.
    A render after the probe equals a fresh context's, byte for byte, with the same counters."""
    fs = scene.load_scene(synth.cornell_mesh(scratch, name="bin_probe", res=(48, 48), spp=2, subdiv=2))
    small = context(fs, monkeypatch, cap=SMALL)
    cap = (small.scene_info()["capacity"] + 1)//2
    for bad in (np.full(4, BINS + 1, np.uint32), np.zeros(cap + 1, np.uint32), np.array([0, 0xFFFFFFFF], np.uint32)):
        with pytest.raises(lib.TgbError) as e:
            small.bin_probe(bad)
        assert e.value.code == abi.TGB_ERR_INVALID
    cur = np.zeros(BINS, np.uint32); ns = C.c_uint32(); k = np.zeros(4, np.uint32)
    L = small.L
    assert L.tgb200_bin_probe(small.h, 4, None, k.ctypes.data, cur.ctypes.data, C.byref(ns)) == abi.TGB_ERR_INVALID
    assert L.tgb200_bin_probe(small.h, 4, k.ctypes.data, None, cur.ctypes.data, C.byref(ns)) == abi.TGB_ERR_INVALID
    assert L.tgb200_bin_probe(small.h, 4, k.ctypes.data, k.ctypes.data, None, C.byref(ns)) == abi.TGB_ERR_INVALID
    assert L.tgb200_bin_probe(small.h, 4, k.ctypes.data, k.ctypes.data, cur.ctypes.data, None) == abi.TGB_ERR_INVALID
    order, cursors, n_sorted = small.bin_probe(np.zeros(0, np.uint32))
    assert n_sorted == 0 and len(order) == 0 and not cursors.any()
    keys = key_pattern("uniform, 10 % untraversed", cap, np.random.RandomState(3))
    keys[:7] = BINS
    assert run_sort(small, keys, "wavefront 0 full") == []
    small.close()
    fresh = lib.Context(fs); img0, cnt0 = fresh.render_tiles(2); s0 = all_stats(fresh); fresh.close()
    ctx = lib.Context(fs)
    assert run_sort(ctx, key_pattern("zipf", 300000, np.random.RandomState(4)), "before the render") == []
    img1, cnt1 = ctx.render_tiles(2); s1 = all_stats(ctx); ctx.close()
    print("after the probe: rays %d/%d, hits %d/%d" % (s0["rays"], s1["rays"], s0["hits"], s1["hits"]))
    assert np.array_equal(img0.view(np.uint32), img1.view(np.uint32)) and np.array_equal(cnt0, cnt1)
    assert s0 == s1


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cornell_mesh", "materials_env", "many_lights", "hair_sky"])
def test_shadow_queries_across_grids(name, scratch, monkeypatch):
    """The shadow probe's k_shadow_prep at 1 and 3 blocks gives the default grid's bytes, and they match the oracle under
    tests/test_gpu_shadow.py's rules."""
    fs = shadow._scene(name, scratch)
    orc = pyoracle.Oracle(fs)
    out = {}
    for lb in (None, 1, 3):
        ctx = context(fs, monkeypatch, lb)
        if lb is None:
            q, lm, strata = shadow.build_queries(fs, ctx, orc, seed=11)
        if lb == 1:                                                       # (the other grids must give the same bytes)
            out[lb], _ = shadow.compare("%s (TGB_LOOP_BLOCKS=1)" % name, fs, ctx, orc, q, lm, strata)
        else:
            out[lb] = shadow.gpu_probe(ctx, q, lm)
        ctx.close()
    queued = int((out[None][:, 6] > 0).sum())
    print("%s: %d queries, %d queued: %d / %d trips per k_shadow_prep launch at 1 / 3 blocks" % (
        name, len(q), queued, trips(queued, 1), trips(queued, 3)))
    for lb in (1, 3):
        assert np.array_equal(out[lb].view(np.uint32), out[None].view(np.uint32)), lb
    orc.close()


@pytest.mark.gpu
def test_shadow_queries_past_one_default_trip(scratch, monkeypatch):
    """A million queries at once, over 600 k of them queued (k_shadow_prep loops at the default grid), equal the same queries in
    chunks of 750, one trip each."""
    fs = shadow._scene("materials_env", scratch)
    orc = pyoracle.Oracle(fs)
    big = context(fs, monkeypatch)
    q, lm, _ = shadow.build_queries(fs, big, orc, seed=13)
    q, lm = np.tile(q, (16, 1)), np.tile(lm, (16, 1))
    a = shadow.gpu_probe(big, q, lm); big.close()
    small = context(fs, monkeypatch, cap=SMALL)
    b = shadow.gpu_probe(small, q, lm); small.close(); orc.close()
    queued = int((a[:, 6] > 0).sum())
    print("%d queries, %d queued: at least %d trips per k_shadow_prep launch at the default grid; chunks of 750 equal: %s" % (
        len(q), queued, least_trips(queued), np.array_equal(a.view(np.uint32), b.view(np.uint32))))
    assert queued > 600000
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cornell_mesh", "materials_env", "cube_city", "hair_sky"])
def test_bounce_states_across_grids(name, scratch, monkeypatch):
    """Chained bounce states (each step's inputs: the default grid's survivors of the step before) at 1 and 3 blocks give the
    default grid's bytes."""
    fs = bounce.make_scene(name, scratch)
    orc = pyoracle.Oracle(fs)
    states = bounce.realistic(fs, orc, bounce.N_PATHS)
    ctxs = {lb: context(fs, monkeypatch, lb) for lb in (None, 1, 3)}
    assert ctxs[None].scene_info()["n_nodes"] > 0                         # a BVH scene: k_bin_scatter runs
    for step in range(3):
        out = {lb: c.bounce_probe(states) for lb, c in ctxs.items()}
        print("%s, step %d: %d states: %d / %d trips per k_bin_scatter launch at 1 / 3 blocks; survivors %d" % (
            name, step, len(states), trips(len(states), 1), trips(len(states), 3), int((out[None][:, abi.BR_STATUS] == 1).sum())))
        for lb in (1, 3):
            assert np.array_equal(out[lb], out[None]), (step, lb)
        states = out[None][out[None][:, abi.BR_STATUS] == 1]
    for c in ctxs.values():
        c.close()
    orc.close()


@pytest.mark.gpu
def test_bounce_states_past_one_default_trip(scratch, monkeypatch):
    """600 k states at once (k_bin_scatter and k_shadow_prep loop at the default grid) equal the same states in chunks of 750."""
    fs = bounce.make_scene("cornell_mesh", scratch)
    orc = pyoracle.Oracle(fs)
    s = bounce.realistic(fs, orc, bounce.N_PATHS)
    s = s[np.arange(600000 + 7) % len(s)].copy()
    big = context(fs, monkeypatch); a = big.bounce_probe(s); big.close()
    small = context(fs, monkeypatch, cap=SMALL); b = small.bounce_probe(s); small.close()
    orc.close()
    print("%d states: at least %d trips per k_bin_scatter launch at the default grid; chunks of 750 equal: %s" % (
        len(s), least_trips(len(s)), np.array_equal(a, b)))
    assert np.array_equal(a, b)


@pytest.mark.gpu
def test_large_render_equals_one_trip_iterations(scratch, monkeypatch):
    """cornell_mesh at 512x512, 8 spp: each wavefront's first k_regen issues over a million camera paths.  The same render with
    750 paths per wavefront (every launch one partial trip) gives the same image, sample counts and counters."""
    fs = scene.load_scene(synth.cornell_mesh(scratch, name="loop_large", res=(512, 512), spp=8, subdiv=3))
    runs = []
    for cap in (0, SMALL):
        ctx = context(fs, monkeypatch, cap=cap)
        img, cnt = ctx.render_tiles(8)
        st = all_stats(ctx)
        runs.append((img, cnt, {k: st[k] for k in STATS}))
        ctx.close()
    first = 512*512*8//2
    print("first k_regen per wavefront: %d paths, at least %d trips at the default grid; samples %d, rays %d" % (
        first, least_trips(first), runs[0][2]["samples"], runs[0][2]["rays"]))
    (a, ca, sa), (b, cb, sb) = runs
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) and np.array_equal(ca, cb)
    assert sa == sb and sa["samples"] == 512*512*8
