"""One bounce at a time: the wavefront loop's glue (k_trace -> k_shade -> k_shadow_prep / k_shadow_bvh -> k_accum) against the
CPU oracle's traceSample loop, from the same path state on both sides.

The image tests compare whole paths, where one libm ulp early in a path changes everything after it, so their bars leave room
for a fraction of a percent of paths to differ -- room enough for a mistake in the loop's control flow that touches few paths
(roulette one bounce late, a missing PCG draw on one lobe, the NEE gate one bounce off).  Here tgb200_bounce_probe runs ONE
iteration of the renderer's own kernels -- the instantiations the context renders with -- on given path states, and
oracle_bounce_probe runs one iteration of the oracle's loop (the same function oracle_render_tiles runs) on the same states.
Both start every bounce from the same state, so the traced ray is bit-identical on both sides.

Strata: chained paths (camera states from the oracle, then each bounce's inputs = the oracle's survivors of the previous one),
settings variants, edge states (one field of a realistic state changed) and deep paths in a closed box.

Comparison (stated here, used below):
  * status, bounce, wasSpecular, sampler dimension and PCG state: exactly equal.  The exceptions are classed per path and each
    class is a row of EXCEPTIONS with its reason and the count an H100 run measured (seeded inputs: the same count every run):
      - hit tie: the two closest-hit implementations (tgb200_trace_closest and the oracle's) pick different primitives for the
        path's ray -- coplanar or touching surfaces, as test_gpu_shadow.py classes its ties -- or, on overlapping curve segments,
        different segments or the same segment at a different t;
      - flip: a discrete decision of the bounce differs although the ray is the same; the inputs of that decision differ by a
        few ulp (libm on the device against glibc: a BSDF's sin / cos / exp / pow), which moves the decision only when it sits
        on its edge;
      - NaN throughput: the one place where the NaN rule of k_shade / k_accum and traceSample's differ (see _NAN_THR);
  * origin and tmin: exact outside the classes above (the curve epsilon, 0.1 x width on `cylinder` curves and 0.01 x width
    otherwise, moves tmin);
  * direction, throughput and radiance: within per-scene ulp bars (ulp of the largest component of the vector),
    3x what an H100 run measured, except paths of the classes above and paths whose direct-light estimate differs grossly
    (> 2^16 ulp: a shadow query that grazes a silhouette decided the other way), which are counted in the "flip" rows too.
Every run prints what it measured.  Each edge stratum also asserts that its case happened: roulette killed some paths and kept
others, the sampler reached its PCG fallback, NEE was skipped at the last bounce, surface and infinite-light emission were added,
NaN paths were zeroed.

Which scene runs which k_shade instantiation (KSHADE below is checked against the context's choice, tgb200_shade_variant):
    scene              k_shade<CURVES, MATSORT, LS>    what else it covers
    cornell_box        <false, false, 1>               analytic primitives only, the Lambert-only lobe set
    cornell_mesh       <false, false, 1>               a smooth-normal mesh
    cornell_generic    <false, false, 0>               cornell_mesh forced onto the generic instantiation (TGB_LOBE_SET=0)
    materials_env      <false, true, 0>                every lobe model, a mesh light, a bitmap environment, material sort
    dirac_room         <false, true, 0>                mirror / conductor / dielectric chains: wasSpecular
    coat_room          <false, true, 0>                rough and smooth coats
    hair_scene         <true, true, 0>                 curves: the curve epsilon, the anisotropic frame
    hair_unsorted      <true, false, 0>                hair_scene with material sort off (TGB_SORT_MATERIALS=0)
    many_lights        <false, false, 1>               39 samplable lights (> 16)
    cube_city          <false, false, 1>               analytic primitives in BVH leaves
    hair_sky           <true, true, 0>                 the shipped hair scene's sphere cap (sampled) + skydome (not sampled)
    curves_cylinder    <true, false, 0>                `cylinder` curves (Lambert, curve_taper, curve_thickness): the localP
                                                       normal and the 0.1 x width curve epsilon
    curves_half_cyl    <true, true, 0>                 `half_cylinder` curves (rough plastic, subsample): the localP normal and
                                                       the 0.01 x width curve epsilon (widths 0.043-0.10: on most strands
                                                       0.01 x width is above the 5e-4 floor it is the max of)
"""
import os

import numpy as np
import pytest

from oracle import pyoracle
from tungsten_b200 import abi, lib, scene, synth

gpu = pytest.mark.gpu

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
F = np.float32
W = abi.BOUNCE_WORDS
N_PATHS = 65536 + 13                    # per scene, not a multiple of 32
SEED = 0xBA5EBA11
PCG_MUL = np.uint64(6364136223846793005)
GROSS_ULP = 2.0**16                     # a larger difference is a discrete flip (counted in EXCEPTIONS), not an ulp-level one

ORIGIN, DIR, THR, EMI = [slice(k, k + 3) for k in (abi.BR_ORIGIN, abi.BR_DIR, abi.BR_THROUGHPUT, abi.BR_EMISSION)]
EXACT = [abi.BR_BOUNCE, abi.BR_FLAGS, abi.BR_DIMENSION, abi.BR_PCG, abi.BR_PCG + 1]

KSHADE = {"cornell_box": "<false, false, 1>", "cornell_mesh": "<false, false, 1>", "cornell_generic": "<false, false, 0>",
          "materials_env": "<false, true, 0>", "dirac_room": "<false, true, 0>", "coat_room": "<false, true, 0>",
          "hair_scene": "<true, true, 0>", "hair_unsorted": "<true, false, 0>", "many_lights": "<false, false, 1>",
          "cube_city": "<false, false, 1>", "hair_sky": "<true, true, 0>", "curves_cylinder": "<true, false, 0>",
          "curves_half_cyl": "<true, true, 0>"}

# (stratum, class) -> (paths, reason), measured on an H100 80GB HBM3 at a 700 W power limit over all bounces of the stratum
_TIE_CURVES = ("the closest hits of tgb200_trace_closest and the oracle differ for the path's ray: overlapping curve segments, which "
               "the two BVHs test in different orders, so a segment is entered with another tmax and prunes other pieces (DESIGN.md "
               "section 2, tests/test_gpu_curve_hits.py's multi class)")
_TIE = "the closest hits of tgb200_trace_closest and the oracle differ for the path's ray: touching or coplanar surfaces"
_FLIP_LIGHT = ("ray, next ray and sampler state agree, only the direct light differs: a shadow query or a light choice among 39 "
               "lights decided the other way on a light-sample direction a few ulp apart")
_FLIP_HAIR = ("same status, direction and sampler state, a different throughput: the hair BCSDF's table cell, chosen from a "
              "libm result a few ulp apart")
_FLIP_CURVES = ("same status, ray and sampler state, a finished radiance far apart: a discrete part of the direct-light estimate "
                "(a shadow query grazing one of the wide, overlapping strands) decided the other way")
_NAN_THR = ("NaN throughput on a bounce that issues no shadow query: the reference adds the zero direct-light estimate times the "
            "throughput (NaN, and no NaN guard follows when the BSDF sample then fails); k_shade adds nothing.  A render never starts "
            "a bounce with a NaN throughput (k_accum ends such paths); an infinite one passes the guard (DESIGN.md)")
EXCEPTIONS = {("hair_scene", "hit tie"): (82, _TIE_CURVES), ("hair_unsorted", "hit tie"): (82, _TIE_CURVES),
              ("hair_sky", "hit tie"): (63, _TIE_CURVES), ("hair_sky misses", "hit tie"): (15, _TIE_CURVES),
              ("hair_sky misses", "flip"): (1, _FLIP_HAIR),
              ("many_lights", "hit tie"): (2, _TIE), ("many_lights", "flip"): (6, _FLIP_LIGHT),
              ("cornell_box edges", "NaN throughput"): (54, _NAN_THR),
              ("curves_cylinder", "hit tie"): (4, _TIE_CURVES), ("curves_half_cyl", "hit tie"): (102, _TIE_CURVES),
              ("curves_half_cyl", "flip"): (1, _FLIP_CURVES)}

# stratum -> (origin + tmin, direction, throughput, emission of survivors, radiance of finished paths) ulp bars: 3x what an H100 run
# measured (in the comment), at most GROSS_ULP: past it a path counts as a flip, so GROSS_ULP is the bar where 3x would exceed it.
# max_bounces 1 is bit-exact.  The wide bars are where a BSDF or light sample goes through device libm
# (rough dielectric, hair, coats), or where a direct-light estimate is the sum of several lights' terms.
ULP_BARS = {
    "cornell_box":                     (0, 6, 0, 3, 0),  # measured (0, 2, 0, 1, 0)
    "cornell_mesh":                    (0, 6, 0, 3, 0),  # measured (0, 2, 0, 1, 0)
    "cornell_generic":                 (0, 6, 0, 3, 0),  # measured (0, 2, 0, 1, 0)
    "materials_env":                   (0, 24, 249, 1401, 765),  # measured (0, 8, 83, 467, 255)
    "dirac_room":                      (0, 3, 0, 3, 1),  # measured (0, 1, 0, 1, 0.25)
    "coat_room":                       (0, 99, 465, 12, 12),  # measured (0, 33, 155, 4, 4)
    "hair_scene":                      (0, 454, 300, 2517, 564),  # measured (0, 151.2, 100, 839, 188)
    "hair_unsorted":                   (0, 454, 300, 2517, 564),  # measured (0, 151.2, 100, 839, 188)
    "many_lights":                     (0, 6, 0, GROSS_ULP, GROSS_ULP),  # measured (0, 2, 0, 36790, 18650): 3x is past the cutoff
    "cube_city":                       (0, 6, 0, 19533, 7818),  # measured (0, 2, 0, 6511, 2606)
    "hair_sky":                        (0, 504, 426, 144, 999),  # measured (0, 167.8, 142, 48, 333)
    "curves_cylinder":                 (0, 6, 0, 2517, 420),  # measured (0, 2, 0, 839, 140)
    "curves_half_cyl":                 (0, 12, 2193, 2517, 498),  # measured (0, 4, 731, 839, 166)
    "cornell_box min_bounces_2":       (0, 6, 0, 6, 0),  # measured (0, 2, 0, 2, 0)
    "cornell_box max_bounces_2":       (0, 6, 0, 0, 0),  # measured (0, 2, 0, 0, 0)
    "cornell_box no_nee":              (0, 6, 0, 0, 0),  # measured (0, 2, 0, 0, 0)
    "cornell_box one_sided":           (0, 6, 0, 0, 0),  # measured (0, 2, 0, 0, 0)
    "cornell_box consistency":         (0, 6, 0, 3, 0),  # measured (0, 2, 0, 1, 0)
    "cornell_box edges":               (0, 6, 0, 3, 0),  # measured (0, 2, 0, 1, 0)
    "cornell_box min_bounces edges":   (0, 6, 0, 6, 0),  # measured (0, 2, 0, 2, 0)
    "materials_env misses":            (0, 12, 54, 783, 6),  # measured (0, 4, 18, 261, 2)
    "hair_sky misses":                 (0, 362, 282, 189, 39),  # measured (0, 120.5, 94, 63, 13)
    "closed_box":                      (0, 3, 0, 3, 0),  # measured (0, 1, 0, 1, 0)
}
DEFAULT_BARS = (0, 0, 0, 0, 0)


# ---- the two probes and the states ----------------------------------------------------------------------------------------
def fl(states, k):
    return states[:, k].view(F)


def camera_states(fs, orc, n, spp_begin=0):
    """The camera states of n (pixel, sample) pairs: pixel i % pixels, sample spp_begin + i // pixels, the tile seeds of SEED."""
    w, h = fs.resolution
    seeds = np.zeros(w*h, np.uint32)
    for t in orc.dice_tiles(SEED):
        for y in range(t.y, t.y + t.h):
            seeds[y*w + t.x: y*w + t.x + t.w] = t.sampler_seed
    k = np.arange(n)
    rec = np.zeros((n, W), np.uint32)
    rec[:, abi.BR_PIXEL] = k % (w*h); rec[:, abi.BR_SEED] = seeds[k % (w*h)]; rec[:, abi.BR_SAMPLE] = spp_begin + k//(w*h)
    return orc.bounce(rec, camera=True)


def _vec_ulp(a, b):
    """ulp of the difference, measured in ulp of the largest magnitude of the two vectors (0 where bit-identical)."""
    with np.errstate(invalid="ignore", over="ignore"):
        m = np.maximum(np.abs(a), np.abs(b)).max(-1).astype(F)
        u = (np.abs(a.astype(np.float64) - b).max(-1)/np.spacing(m).astype(np.float64))
    same = (a.view(np.uint32) == b.view(np.uint32)).all(-1)
    return np.where(same, 0.0, np.where(np.isnan(u), np.inf, u))


def pcg_step(lo, hi, k=1):
    s = lo.astype(np.uint64) | (hi.astype(np.uint64) << np.uint64(32))
    with np.errstate(over="ignore"):
        for _ in range(k):
            s = s*PCG_MUL + np.uint64(1)
    return s


class Tally:
    """What one scene's comparisons measured: exception counts by class, worst ulp per field group."""
    def __init__(self, name):
        self.name = name; self.counts = {}; self.worst = [0.0]*5; self.paths = 0; self.flips = []

    def report(self):
        print("%s: %d path bounces; exceptions %s; worst ulp: origin %.1f, direction %.1f, throughput %.1f, emission %.1f, "
              "radiance %.1f" % (self.name, self.paths, self.counts or "none", *self.worst))
        for f in self.flips[:6]:
            print("    flip:", f)


def compare(ctx, orc, states, tally):
    """Both probes on `states`; folds the comparison into tally.  Returns (gpu, oracle) outputs."""
    g = ctx.bounce_probe(states); r = orc.bounce(states)
    tally.paths += len(states)
    ga, ra = g[:, abi.BR_STATUS], r[:, abi.BR_STATUS]
    alive = (ga == 1) & (ra == 1); done = (ga == 0) & (ra == 0)
    bad = ga != ra
    bad |= alive & (g[:, EXACT] != r[:, EXACT]).any(1)
    bad |= done & (g[:, EXACT[2:]] != r[:, EXACT[2:]]).any(1)
    u = np.zeros((len(states), 5))
    u[alive, 0] = _vec_ulp(np.concatenate([fl(g, ORIGIN), fl(g, [abi.BR_TMIN])], 1)[alive],
                           np.concatenate([fl(r, ORIGIN), fl(r, [abi.BR_TMIN])], 1)[alive])
    u[alive, 1] = _vec_ulp(fl(g, DIR)[alive], fl(r, DIR)[alive])
    u[alive, 2] = _vec_ulp(fl(g, THR)[alive], fl(r, THR)[alive])
    u[alive, 3] = _vec_ulp(fl(g, EMI)[alive], fl(r, EMI)[alive])
    u[done, 4] = _vec_ulp(fl(g, EMI)[done], fl(r, EMI)[done])
    gross = ~bad & (u > GROSS_ULP).any(1)
    # origin and tmin are exact unless the two walks found different hits for the path's ray (same segment at another t included)
    odd = bad | gross | (u[:, 0] > 0)
    if odd.any():
        idx = np.flatnonzero(odd)
        rays = np.zeros((len(idx), 8), F)
        rays[:, :3] = fl(states, ORIGIN)[idx]; rays[:, 3:6] = fl(states, DIR)[idx]; rays[:, 6] = fl(states, [abi.BR_TMIN])[idx, 0]
        rays[:, 7] = np.inf
        hg, hr = ctx.trace_closest(rays), orc.trace(rays)
        tie = (hg["primitive"] != hr["primitive"]) | ((hg["primitive"] >= 0) & ((hg["prim_id"] != hr["prim_id"]) |
                                                                               (hg["t"].view(np.uint32) != hr["t"].view(np.uint32))))
        for j, i in enumerate(idx):
            cls = "hit tie" if tie[j] else "NaN throughput" if np.isnan(fl(states, THR)[i]).any() else "flip"
            tally.counts[cls] = tally.counts.get(cls, 0) + 1
            if cls == "flip":
                tally.flips.append("bounce %d: status %d/%d, gpu %s, oracle %s" % (
                    states[i, abi.BR_BOUNCE], ga[i], ra[i], g[i].view(F)[:16].tolist(), r[i].view(F)[:16].tolist()))
    ok = ~odd
    for k in range(5):
        if ok.any():
            tally.worst[k] = max(tally.worst[k], float(u[ok, k].max()))
    return g, r


def check(tally, bars_key=None):
    tally.report()
    key = bars_key or tally.name
    expected = {cls: v[0] for (sc, cls), v in EXCEPTIONS.items() if sc == key}
    assert tally.counts == expected, (key, tally.counts, expected)
    bars = ULP_BARS.get(key, DEFAULT_BARS)
    assert all(b <= GROSS_ULP for b in bars)
    assert all(w <= b for w, b in zip(tally.worst, bars)), (key, tally.worst, bars)


def chain(ctx, orc, states, tally, max_steps=None):
    """Chained stratum: bounce k+1's inputs = the oracle's survivors of bounce k.  Returns the list of (inputs, gpu, oracle)."""
    steps = []
    while len(states) and (max_steps is None or len(steps) < max_steps):
        g, r = compare(ctx, orc, states, tally)
        steps.append((states, g, r))
        states = r[r[:, abi.BR_STATUS] == 1]
    return steps


# ---- scenes ---------------------------------------------------------------------------------------------------------------
def make_scene(name, scratch, monkeypatch=None, **kw):
    if name == "cornell_box":
        return scene.load_scene(synth.cornell_box(res=(32, 32), spp=1, **kw))
    if name in ("cornell_mesh", "cornell_generic"):
        if name == "cornell_generic":
            monkeypatch.setenv("TGB_LOBE_SET", "0")
        return scene.load_scene(synth.cornell_mesh(scratch, name="bounce_mesh", res=(32, 32), spp=1))
    if name == "dirac_room":
        return scene.load_scene(synth.dirac_room(scratch, name="bounce_dirac", res=(32, 32), spp=1))
    if name == "coat_room":
        return scene.load_scene(synth.coat_room(scratch, name="bounce_coats", res=(32, 32), spp=1))
    if name in ("hair_scene", "hair_unsorted"):
        if name == "hair_unsorted":
            monkeypatch.setenv("TGB_SORT_MATERIALS", "0")
        return scene.load_scene(synth.hair_scene(scratch, name="bounce_hair", n_curves=300, res=(32, 32), spp=1))
    if name == "many_lights":
        return scene.load_scene(synth.many_lights(scratch, name="bounce_ml", res=(32, 32), spp=1, subdiv=3))
    if name == "cube_city":
        return scene.load_scene(synth.cube_city(res=(32, 32), spp=1, n=12))
    if name == "curves_cylinder":           # test_gpu_parity.test_curves_and_hair's two non-hair modes, at probe size (the
                                            # half_cylinder strands wider, so that their epsilon is not the 5e-4 floor)
        return scene.load_scene(synth.hair_scene(scratch, name="bounce_cyl", n_curves=300, res=(32, 32), spp=1, mode="cylinder",
                                                 bsdf={"type": "lambert", "albedo": [0.6, 0.4, 0.2]}, thickness=0.015, taper=True))
    if name == "curves_half_cyl":
        return scene.load_scene(synth.hair_scene(scratch, name="bounce_half_cyl", n_curves=300, res=(32, 32), spp=1,
                                                 mode="half_cylinder", bsdf={"type": "rough_plastic", "albedo": [0.6, 0.4, 0.2],
                                                                             "roughness": 0.2}, subsample=0.3, width=0.07))
    return scene.load_scene(os.path.join(G, name, "scene.json"))          # materials_env, hair_sky


SCENES = list(KSHADE)


@gpu
@pytest.mark.parametrize("name", SCENES)
def test_chained_bounces_match_oracle(name, scratch, monkeypatch):
    fs = make_scene(name, scratch, monkeypatch)
    ctx = lib.Context(fs); orc = pyoracle.Oracle(fs)
    assert ctx.shade_variant() == KSHADE[name]
    if name.startswith("curves_"):          # the curve epsilon max(5e-4, k x width) is k x width on most strands
        p = next(p for p in fs.primitives if p.type == abi.PRIM_CURVES)
        w = np.ctypeslib.as_array(p.curve_nodes, shape=(p.n_curve_nodes*4,))[3::4]
        k = F(0.1) if p.curve_mode == abi.CURVE_CYLINDER else F(0.01)
        print("%s: %.3f of the nodes have k x width > 5e-4" % (name, float((k*w > F(5e-4)).mean())))
        assert (k*w > F(5e-4)).mean() > 0.5
    tally = Tally(name)
    steps = chain(ctx, orc, camera_states(fs, orc, N_PATHS), tally)
    alive = [int((r[:, abi.BR_STATUS] == 1).sum()) for _, _, r in steps]
    print("%s: k_shade%s, %d bounces, survivors per bounce %s" % (name, KSHADE[name], len(steps), alive[:12]))
    check(tally)
    ctx.close(); orc.close()


# ---- settings variants ----------------------------------------------------------------------------------------------------
VARIANTS = {"min_bounces_2": ("min_bounces", 2), "max_bounces_1": ("max_bounces", 1), "max_bounces_2": ("max_bounces", 2),
            "no_nee": ("enable_light_sampling", False), "one_sided": ("enable_two_sided_shading", False),
            "consistency": ("enable_consistency_checks", True)}


def variant_scene(case):
    sc = synth.cornell_box(res=(32, 32), spp=1)
    k, v = VARIANTS[case]
    sc["integrator"][k] = v
    return scene.load_scene(sc)


@gpu
@pytest.mark.parametrize("case", list(VARIANTS))
def test_settings_variants_match_oracle(case):
    fs = variant_scene(case)
    ctx = lib.Context(fs); orc = pyoracle.Oracle(fs)
    tally = Tally("cornell_box " + case)
    steps = chain(ctx, orc, camera_states(fs, orc, 16384 + 7), tally)
    max_b = fs.settings.max_bounces
    assert all((s[:, abi.BR_BOUNCE] < max_b).all() for s, _, _ in steps)
    assert all((r[r[:, abi.BR_STATUS] == 1, abi.BR_BOUNCE] < max_b).all() for _, _, r in steps)
    if case == "no_nee":
        # surface emission is the only light: the camera paths that see the light directly carry it (wasSpecular = 1)
        _, _, r0 = steps[0]
        assert (fl(r0, EMI) > 0).any()
    check(tally)
    ctx.close(); orc.close()


# ---- edge strata ----------------------------------------------------------------------------------------------------------
def realistic(fs, orc, n, bounce=1):
    """Oracle survivors at `bounce` of chained camera paths (recycled to n states)."""
    s = camera_states(fs, orc, 2*n)
    for _ in range(bounce):
        r = orc.bounce(s); s = r[r[:, abi.BR_STATUS] == 1]
    return s[np.arange(n) % len(s)].copy()


@gpu
def test_edge_states_match_oracle():
    rng = np.random.RandomState(21)
    fs = scene.load_scene(synth.cornell_box(res=(32, 32), spp=1, max_bounces=16))
    ctx = lib.Context(fs); orc = pyoracle.Oracle(fs)
    tally = Tally("cornell_box edges")
    base = realistic(fs, orc, 8192 + 5)
    n = len(base)

    # NEE skipped at the last bounce: from wasSpecular = 0 states (the light is samplable, no infinite light), nothing is added
    s = base.copy(); s[:, abi.BR_BOUNCE] = 15; s[:, abi.BR_FLAGS] = 0
    g, r = compare(ctx, orc, s, tally)
    assert (g[:, abi.BR_STATUS] == 0).all() and (g[:, EMI] == s[:, EMI]).all()
    s[:, abi.BR_BOUNCE] = 14
    g, _ = compare(ctx, orc, s, tally)
    print("last bounce: nothing added; one bounce before it: %d of %d paths gained NEE light" % (int((g[:, EMI] != s[:, EMI]).any(1).sum()), n))
    assert (g[:, EMI] != s[:, EMI]).any(1).sum() > n//10

    # roulette: throughput scaled to a max component in [0.005, 0.12) at bounces 2, 3, 4; from bounce 3 on it draws one PCG number
    s = base.copy()
    thr = fl(s, THR); scale = rng.uniform(0.005, 0.12, n).astype(F)/thr.max(1)
    s[:, THR] = (thr*scale[:, None]).astype(F).view(np.uint32)
    out = {}
    for b in (2, 3, 4):
        s[:, abi.BR_BOUNCE] = b
        out[b] = compare(ctx, orc, s, tally)
    g2, g3 = out[2][0], out[3][0]
    cont = g2[:, abi.BR_STATUS] == 1                                       # continued at bounce 2 (no roulette there)
    small = cont & (fl(g2, THR).max(1) < 0.1)                              # ... with a throughput roulette runs on from bounce 3
    killed, kept = small & (g3[:, abi.BR_STATUS] == 0), small & (g3[:, abi.BR_STATUS] == 1)
    print("roulette at bounce 3: %d eligible, %d killed, %d kept" % (int(small.sum()), int(killed.sum()), int(kept.sum())))
    assert killed.sum() > 100 and kept.sum() > 100
    # the roulette draw is the one PCG step between bounce 2's and bounce 3's sampler state; survivors are divided by its pdf
    s2 = pcg_step(g2[small, abi.BR_PCG], g2[small, abi.BR_PCG + 1])
    s3 = g3[small, abi.BR_PCG].astype(np.uint64) | (g3[small, abi.BR_PCG + 1].astype(np.uint64) << np.uint64(32))
    assert (s2 == s3).all()
    assert (fl(g3, THR)[kept].max(1) >= fl(g2, THR)[kept].max(1)).all()

    # zero throughput: the path ends at this bounce with the emission it had; NaN throughput: zeroed; NaN origin: a miss
    s = base.copy(); s[:, THR] = F(0.0).view(np.uint32)
    g, _ = compare(ctx, orc, s, tally)
    assert (g[:, abi.BR_STATUS] == 0).all() and (g[:, EMI] == s[:, EMI]).all()
    s = base.copy(); k = rng.randint(0, 3, n); s[np.arange(n), abi.BR_THROUGHPUT + k] = F(np.nan).view(np.uint32)
    g, r = compare(ctx, orc, s, tally)
    # (a path whose BSDF sample fails -- the light's null BSDF -- leaves the loop before the NaN guards, on both sides)
    zeroed = (fl(g, EMI) == 0).all(1) & (fl(s, EMI) != 0).any(1)
    print("NaN throughput: %d of %d paths finished, %d with radiance zeroed" % (int((g[:, abi.BR_STATUS] == 0).sum()), n, int(zeroed.sum())))
    assert (g[:, abi.BR_STATUS] == 0).all() and zeroed.sum() > n//4
    s = base.copy(); s[np.arange(n), abi.BR_ORIGIN + k] = F(np.nan).view(np.uint32)
    compare(ctx, orc, s, tally)

    # the sampler's switch from Sobol to PCG at dimension 1024
    s = base.copy(); s[:, abi.BR_DIMENSION] = rng.randint(1015, 1031, n)
    g, _ = compare(ctx, orc, s, tally)
    crossed = (s[:, abi.BR_DIMENSION] < 1024) & (g[:, abi.BR_DIMENSION] == 1024)
    print("dimension 1015..1030: %d crossed into the PCG fallback, outputs at dimension 1024: %d" % (int(crossed.sum()), int((g[:, abi.BR_DIMENSION] == 1024).sum())))
    assert crossed.sum() > 100 and (g[:, abi.BR_DIMENSION] >= s[:, abi.BR_DIMENSION]).all()

    # sample indices at the 256-sample boundary of the Sobol index permutation, and near 2^32
    for smp in (255, 256, 0xFFFFFFF0):
        s = base.copy(); s[:, abi.BR_SAMPLE] = smp
        compare(ctx, orc, s, tally)
    check(tally)
    ctx.close(); orc.close()


@gpu
def test_min_bounces_edges_match_oracle():
    fs = variant_scene("min_bounces_2")
    ctx = lib.Context(fs); orc = pyoracle.Oracle(fs)
    tally = Tally("cornell_box min_bounces edges")
    base = realistic(fs, orc, 8192 + 5)
    s = base.copy(); s[:, abi.BR_BOUNCE] = 0; s[:, abi.BR_FLAGS] = 1
    g, _ = compare(ctx, orc, s, tally)
    assert (g[:, EMI] == s[:, EMI]).all()                                   # bounce + 1 < min_bounces: no light at all
    s[:, abi.BR_BOUNCE] = 1                                                 # = min_bounces - 1: the NEE queries count
    g, _ = compare(ctx, orc, s, tally)
    print("bounce 1 = min_bounces - 1: %d paths gained light" % int((g[:, EMI] != s[:, EMI]).any(1).sum()))
    assert (g[:, EMI] != s[:, EMI]).any(1).sum() > 100
    check(tally)
    ctx.close(); orc.close()


@gpu
@pytest.mark.parametrize("name", ["materials_env", "hair_sky"])
def test_infinite_light_misses_match_oracle(name):
    """Rays that leave the scene: samplable (materials_env's environment, hair_sky's cap) and non-samplable (hair_sky's skydome)
    infinite lights, wasSpecular both ways, bounce below and at min_bounces."""
    rng = np.random.RandomState(31)
    fs = scene.load_scene(os.path.join(G, name, "scene.json"))
    ctx = lib.Context(fs); orc = pyoracle.Oracle(fs)
    tally = Tally(name + " misses")
    s = realistic(fs, orc, 16384 + 3)
    n = len(s)
    d = rng.normal(size=(n, 3))
    up = 2 if name == "materials_env" else 1                               # out of the room's open front / up into the sky
    d[:, up] = np.abs(d[:, up]) + 1.0; d /= np.linalg.norm(d, axis=1, keepdims=True)
    s[:, DIR] = d.astype(F).view(np.uint32)
    s[:, abi.BR_FLAGS] = rng.randint(0, 2, n)
    s[:, abi.BR_BOUNCE] = rng.randint(0, 3, n)
    g, r = compare(ctx, orc, s, tally)
    rays = np.concatenate([fl(s, ORIGIN), fl(s, DIR), fl(s, [abi.BR_TMIN]), np.full((n, 1), np.inf, F)], 1)
    miss = orc.trace(rays)["primitive"] < 0
    gained = miss & (g[:, EMI] != s[:, EMI]).any(1)
    spec = s[:, abi.BR_FLAGS] == 1
    print("%s: %d misses, infinite-light emission added to %d (wasSpecular %d / not %d)"
          % (name, int(miss.sum()), int(gained.sum()), int((gained & spec).sum()), int((gained & ~spec).sum())))
    assert miss.sum() > n//4 and (gained & spec).sum() > 100
    if name == "hair_sky":
        assert (gained & ~spec).sum() > 100                                # the skydome is not samplable: added either way
    else:
        assert not (gained & ~spec).any()                                  # a samplable environment only after specular bounces
    check(tally)
    ctx.close(); orc.close()


# ---- deep paths -----------------------------------------------------------------------------------------------------------
def closed_box():
    """A Cornell box closed by a fourth wall, camera inside, every surface Lambert with albedo 1 (the light's too): the throughput
    stays 1, roulette never runs and no path leaves the box, so every path runs to max_bounces 255."""
    sc = synth.cornell_box(res=(16, 16), spp=1, max_bounces=255, boxes=False)
    for b in sc["bsdfs"]:                                                  # (the light too: a null BSDF would end its paths)
        b["type"] = "lambert"; b["albedo"] = 1.0
    sc["bsdfs"].append({"name": "frontWall", "type": "lambert", "albedo": 1.0})
    sc["primitives"].append({"name": "frontWall", "type": "quad", "bsdf": "frontWall",
                             "transform": {"position": [0, 1, 1], "scale": [2, 4, 2], "rotation": [0, 90, -90]}})
    sc["camera"]["transform"] = {"position": [0, 1, 0.9], "look_at": [0, 1, 0], "up": [0, 1, 0]}
    sc["camera"]["fov"] = 90
    return scene.load_scene(sc)


@gpu
def test_deep_paths_match_oracle():
    fs = closed_box()
    ctx = lib.Context(fs); orc = pyoracle.Oracle(fs)
    tally = Tally("closed_box")
    steps = chain(ctx, orc, camera_states(fs, orc, 4096 + 9), tally)
    alive = [int((r[:, abi.BR_STATUS] == 1).sum()) for _, _, r in steps]
    dims = [int(s[:, abi.BR_DIMENSION].max()) for s, _, _ in steps]
    first = next((k for k, dm in enumerate(dims) if dm >= 1024), None)
    print("closed box: %d bounces, survivors at 1/100/200/254: %s, dimension 1024 first reached at bounce %s"
          % (len(steps), [alive[k] for k in (0, 99, 199, 253) if k < len(alive)], first))
    assert len(steps) == 255 and alive[253] > 0.9*alive[0]
    assert first is not None and first < 250
    check(tally)
    ctx.close(); orc.close()


# ---- the probe and the context --------------------------------------------------------------------------------------------
@gpu
def test_chunks_and_context_unchanged(scratch):
    fs = scene.load_scene(synth.many_lights(scratch, name="bounce_chunks", res=(48, 48), spp=2, subdiv=2))
    orc = pyoracle.Oracle(fs)
    small = lib.Context(fs, max_paths_in_flight=1500); big = lib.Context(fs)
    cap = small.scene_info()["capacity"]//2                                 # the first wavefront's slots
    s = realistic(fs, orc, cap + 1)
    a, b = small.bounce_probe(s), big.bounce_probe(s)
    print("wavefront capacity %d, %d states: chunked == one launch: %s" % (cap, len(s), np.array_equal(a, b)))
    assert np.array_equal(a, b)
    with pytest.raises(lib.TgbError):
        bad = s[:4].copy(); bad[:, abi.BR_BOUNCE] = fs.settings.max_bounces
        big.bounce_probe(bad)
    assert big.L.tgb200_bounce_probe(big.h, 1, None, None) == abi.TGB_ERR_INVALID
    small.close(); big.close()
    fresh = lib.Context(fs); img0, cnt0 = fresh.render_tiles(2); s0 = fresh.stats(); fresh.close()
    ctx = lib.Context(fs)
    ctx.bounce_probe(s)
    img1, cnt1 = ctx.render_tiles(2); s1 = ctx.stats(); ctx.close(); orc.close()
    print("rays %d/%d, shadow rays %d/%d, hits %d/%d" % (s0.rays, s1.rays, s0.shadow_rays, s1.shadow_rays, s0.hits, s1.hits))
    assert np.array_equal(img0.view(np.uint32), img1.view(np.uint32)) and np.array_equal(cnt0, cnt1)
    assert (s0.rays, s0.hits, s0.shadow_rays, s0.path_rays) == (s1.rays, s1.hits, s1.shadow_rays, s1.path_rays)


# ---- CPU only: the stepped oracle is the oracle ---------------------------------------------------------------------------
@pytest.mark.parametrize("name,spp_begin", [("cornell_box", 0), ("materials_env", 256), ("dirac_room", 257), ("hair_sky", 300)])
def test_oracle_steps_reproduce_the_render(name, spp_begin, scratch):
    """Camera states, then oracle steps until every path finished, give the radiance oracle_render_tiles accumulates at 1 spp,
    bit for bit (a NaN / Inf sample is the one the render drops)."""
    fs = make_scene(name, scratch)
    orc = pyoracle.Oracle(fs)
    w, h = fs.resolution
    s = camera_states(fs, orc, w*h, spp_begin)
    rad = np.zeros((w*h, 3), F)
    idx = np.arange(w*h)
    steps = 0
    while len(s):
        r = orc.bounce(s); steps += 1
        done = r[:, abi.BR_STATUS] == 0
        rad[idx[done]] = fl(r, EMI)[done]
        s, idx = r[~done], idx[~done]
    mean, cnt = orc.render(1, seed=SEED, spp_begin=spp_begin)
    mean, cnt = mean.reshape(-1, 3), cnt.reshape(-1)
    kept = cnt == 1
    print("%s at sample %d: %d pixels, %d bounces, %d samples dropped as NaN / Inf" % (name, spp_begin, w*h, steps, int((~kept).sum())))
    assert np.array_equal(rad[kept].view(np.uint32), mean[kept].view(np.uint32))
    assert (~np.isfinite(rad[~kept])).any(1).all()
    orc.close()


def test_oracle_max_bounces_0_is_black_and_steps_refuse_finished_states():
    """maxBounces 0: traceSample traces the camera ray and its loop never runs, so every sample is black.  A state at bounce
    >= maxBounces is not a path about to trace a ray: oracle_bounce_probe refuses it, as tgb200_bounce_probe does."""
    from tungsten_b200 import abi as A
    for mb in (0, 1):
        fs = scene.load_scene(synth.cornell_box(res=(16, 16), spp=1, max_bounces=mb))
        orc = pyoracle.Oracle(fs)
        mean, cnt = orc.render(4, seed=SEED)
        print("max_bounces %d: sum %.4f, %d rays" % (mb, float(mean.sum()), orc.stats.rays))
        assert (cnt == 4).all() and orc.stats.rays == 16*16*4
        assert (mean == 0).all() if mb == 0 else mean.sum() > 0
        s = camera_states(fs, orc, 64)
        s[:, A.BR_BOUNCE] = mb
        with pytest.raises(RuntimeError):
            orc.bounce(s)
        orc.close()
