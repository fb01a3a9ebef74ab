"""Curve hits one segment at a time, at the edges where a segment test goes wrong.

oracle_curve_segments_probe (Oracle.curve_segments) runs the oracle's curve frame and point_on_spline on EVERY segment of a curve
primitive with the ray's own tmin / tmax and no BVH or box culling, and reports per ray how many segments pass their root box test,
how many report a hit when tested alone, and the nearest of those hits.  A segment that misses with tmax = the ray's tmax cannot hit
with a smaller tmax (pruning only removes pieces), so every ray falls into one class:

  class    | hook answer                                  | what tgb200_trace_closest and Oracle.trace must report
  ---------+----------------------------------------------+---------------------------------------------------------------------
  none     | no segment hits alone                        | no curve hit (exact)
  inside   | exactly one hits, its hit point lies inside  | that segment, with t, u and width bit-identical to the hook's
           | the segment's curveBox shrunk by MARGIN      | (device and oracle run the same float arithmetic: -fmad=false, no
           |                                              | libm in pointOnSpline or intersectHalfCylinder)
  outside  | exactly one hits, outside that box (a half-  | any hit reported is bit-identical to the hook's; a BVH may cull the
           | cylinder piece accepts hits on the extension | segment, so the rays each walk drops are counted and pinned in
           | of its chord)                                | OUTSIDE_DROPS
  multi    | two or more segments hit alone (overlap)     | the reported segment is one that hits alone; device-versus-oracle
           |                                              | differences are counted and pinned in MULTI_MISMATCHES (the two
           |                                              | BVHs test the segments in different orders)

Scenes (curves only, lit by an environment, so every hit is a curve hit):
  edges   straight segments (three or more collinear nodes along x, y, z and an oblique axis: q0 = 0 in ray space, so tFlat is
          +-inf or NaN), a tight curl (radius 2.5 widths), widths 1e-4, 1e-3 and 0.2 (the cluster spans about 2), a node of
          width 0, linear width ramps that reach 0 at a segment's end and go negative past it, segments with n0 = n1, n1 = n2
          and all three nodes equal, the curl again translated by about 1e3, and a second primitive whose widths come from
          curve_thickness and curve_taper through the flattener;
  hair    80 curly strands (synth.curly_fibers): overlapping segments, the multi class.

Strata, each of which asserts that its case occurred: random rays; rays aimed at centreline points; silhouette rays at
w * (1 + k 2^-20), k = -4..4, from a depth-5 piece's chord, which decide `distance > width`; rays at u in {0, 2^-24, 1 - 2^-24, 1}
(strand joints and free ends); rays along the tangent (projected chord length 0 on straight segments); directions of exactly +-y
(the d == 0 branch of the curve frame); +-y with x and z components of 1e-20 and 1e-25 (x^2 + z^2 subnormal or 0); axis directions
with +-0 components; tmax and tmin one ulp before, at and after the hook's t; origins on the curve surface with tmin equal to the
curve epsilon (self-hits).

The hook itself is checked without a GPU against a float64 model of the tube (test_hook_agrees_with_float64_tube), and the oracle's
own BVH walk against the hook (test_oracle_walk_agrees_with_hook).
"""
import os

import numpy as np
import pytest

from oracle import pyoracle
from tungsten_b200 import abi, lib, scene, synth

F = np.float32
NONE, INSIDE, OUTSIDE, MULTI = 0, 1, 2, 3
CLASS_NAMES = ("none", "inside", "outside", "multi")
# a hit point counts as inside its segment's curveBox when it is at least this fraction of the box's largest extent from every face:
# the device's quantised boxes and the oracle's padded boxes both contain the float box, and the slab tests' rounding stays far below
# this (at 1e3 from the origin one ulp of a coordinate is 6e-5, of a 0.07-wide box 1e-3)
MARGIN = 2.0**-8
PIECE = 1.0/32                              # parameter length of a depth-5 piece

# (scene, walk) -> (rays of the `outside` class that walk reports no hit for, reason), measured on an H100 80GB HBM3 at a 700 W power limit (seeded: the same
# on every run).  walk: "oracle" (Oracle.trace), "device" (tgb200_trace_closest), "device, cut off" (the same with TGB_HOOK_CUT=0).
_CULLED = ("the segment's only hit lies outside its curveBox (the extension of a half-cylinder piece's chord), and the walk culled "
           "the segment by a box the ray does not reach before that hit")
_CUT = _CULLED + "; with the top-level cut the pre-test also drops hits outside every cut box"
OUTSIDE_DROPS = {("edges", "oracle"): (82, _CULLED), ("edges", "device"): (28, _CUT), ("edges", "device, cut off"): (24, _CULLED),
                 ("hair", "oracle"): (54, _CULLED), ("hair", "device"): (65, _CUT), ("hair", "device, cut off"): (65, _CULLED)}
# scene -> (rays of the `multi` class where the device and the oracle report different segments or t, reason)
_ORDER = ("two or more overlapping segments hit alone; the device's 4-ary BVH and the oracle's segment BVH2 test them in different "
          "orders, and a segment tested after a hit prunes its pieces against that hit (pointOnSpline's bound is not conservative)")
MULTI_MISMATCHES = {"edges": (1, _ORDER), "hair": (5, _ORDER)}


# ---- scenes -------------------------------------------------------------------------------------------------------------------
def _line(p0, axis, n, step, w):
    axis = np.asarray(axis, np.float64); axis /= np.linalg.norm(axis)
    p = np.asarray(p0, np.float64)[None] + step*np.arange(n)[:, None]*axis[None]
    return np.concatenate([p, np.broadcast_to(np.asarray(w, np.float64), (n,))[:, None]], 1)


def _helix(c, r, w, turns, n, drop):
    a = np.linspace(0.0, 2*np.pi*turns, n)
    p = np.stack([c[0] + r*np.cos(a), c[1] - drop*a/(2*np.pi*turns), c[2] + r*np.sin(a)], 1)
    return np.concatenate([p, np.full((n, 1), w)], 1)


def _wavy(p0, n, length, amp, w):
    s = np.linspace(0.0, 1.0, n)
    p = np.stack([p0[0] + length*s, p0[1] + amp*np.sin(2*np.pi*1.5*s), p0[2] + amp*np.cos(2*np.pi*s)], 1)
    return np.concatenate([p, np.broadcast_to(np.asarray(w, np.float64), (n,))[:, None]], 1)


FAR = np.array([600.0, 500.0, -600.0])      # the translated curl: about 1e3 from the origin


def edge_strands():
    """(strands of the half_cylinder primitive, strands of the cylinder primitive), each a float64 [k, 4] array of nodes; the second
    primitive's widths are replaced by curve_thickness and curve_taper."""
    A, B = {}, {}
    A["x"] = _line((-1.0, 1.8, 0.0), (1, 0, 0), 4, 0.15, 0.02)
    A["y"] = _line((-0.8, 1.0, 0.3), (0, 1, 0), 4, 0.15, 0.02)
    A["z"] = _line((-0.6, 1.6, -0.6), (0, 0, 1), 4, 0.15, 0.02)
    A["oblique"] = _line((-0.3, 1.3, -0.2), (1, 2, 3), 4, 0.15, 0.02)
    A["curl"] = _helix((0.5, 1.7, 0.0), 0.03, 0.012, 3.0, 31, 0.25)
    A["w1e-4"] = _wavy((-1.0, 0.9, -0.5), 8, 0.6, 0.05, 1e-4)
    A["w1e-3"] = _wavy((-1.0, 0.7, -0.5), 8, 0.6, 0.05, 1e-3)
    A["w0.2"] = _wavy((-0.4, 0.3, 0.6), 6, 1.4, 0.1, 0.2)
    A["zero node"] = _wavy((0.1, 1.1, -0.6), 5, 0.5, 0.04, [0.02, 0.0, 0.02, 0.0, 0.02])
    A["ramp to 0 at u=0"] = _line((0.2, 0.8, 0.2), (1, 0.3, 0), 3, 0.15, [-0.01, 0.01, 0.03])
    A["ramp to 0 at u=1"] = _line((0.2, 0.6, 0.2), (1, -0.2, 0.1), 3, 0.15, [0.03, 0.01, -0.01])
    a, b = np.array([0.9, 1.2, 0.4, 0.02]), np.array([1.05, 1.3, 0.45, 0.02])
    A["n0 = n1"] = np.stack([a, a, b])
    A["n1 = n2"] = np.stack([a + [0, -0.3, 0, 0], b + [0, -0.3, 0, 0], b + [0, -0.3, 0, 0]])
    A["all equal"] = np.stack([a + [0, -0.6, 0, 0]]*3)
    A["far curl"] = A["curl"] + np.concatenate([FAR, [0.0]])
    _, nodes = synth.curly_fibers(3, 10, radius=0.15, length=0.6, width=0.01, seed=4)
    for i in range(3):
        B["taper %d" % i] = nodes[10*i:10*i + 10].astype(np.float64) + [1.0, 1.7, -0.4, 0.0]
    return A, B


def _write_strands(path, strands):
    nodes = np.concatenate(list(strands.values())).astype(F)
    ends = np.cumsum([len(s) for s in strands.values()]).astype(np.uint32)
    scene.save_fiber(path, ends, nodes)
    return os.path.basename(path)


def _curve_scene(d, name, prims, cam, look_at):
    sc = {"media": [], "bsdfs": [{"name": "strand", "type": "lambert", "albedo": [0.6, 0.5, 0.4]}],
          "primitives": prims + [{"name": "env", "type": "infinite_sphere", "emission": [0.6, 0.6, 0.6], "sample": True}],
          "camera": {"tonemap": "filmic", "resolution": [32, 32], "reconstruction_filter": "tent",
                     "transform": {"position": list(cam), "look_at": list(look_at), "up": [0, 1, 0]}, "type": "pinhole", "fov": 45},
          "integrator": {"type": "path_tracer", "min_bounces": 0, "max_bounces": 8, "enable_consistency_checks": False,
                         "enable_two_sided_shading": True, "enable_light_sampling": True},
          "renderer": synth._renderer(1)}
    return scene.load_scene(sc, base_dir=d)


def build_scene(name, scratch):
    d = os.path.join(scratch, "curve_hits"); os.makedirs(d, exist_ok=True)
    if name == "edges":
        A, B = edge_strands()
        prims = [{"name": "edges", "type": "curves", "file": _write_strands(os.path.join(d, "edges_a.fiber"), A), "mode": "half_cylinder",
                  "bsdf": "strand"},
                 {"name": "tapered", "type": "curves", "file": _write_strands(os.path.join(d, "edges_b.fiber"), B), "mode": "cylinder",
                  "bsdf": "strand", "curve_thickness": 0.015, "curve_taper": True}]
        return _curve_scene(d, name, prims, (0.2, 1.3, 3.5), (0.0, 1.2, 0.0))
    if name == "hair":
        ends, nodes = synth.curly_fibers(80, 14, radius=0.3, length=0.9, width=0.012, seed=7)
        scene.save_fiber(os.path.join(d, "hair.fiber"), ends, nodes)
        prims = [{"name": "hair", "type": "curves", "file": "hair.fiber", "mode": "bcsdf_cylinder", "bsdf": "strand",
                  "transform": {"position": [0.0, 1.5, 0.0]}}]
        return _curve_scene(d, name, prims, (0.3, 1.2, 2.8), (0.0, 1.1, 0.0))
    raise KeyError(name)


def curve_prims(fs):
    return [i for i, p in enumerate(fs.primitives) if p.type == abi.PRIM_CURVES]


def segments(fs):
    """Every curve segment of the scene: primitive, segment index, nodes n0, n1, n2 (float64 of the flattened float32) [S, 3, 4]."""
    P, K, N = [], [], []
    for pi in curve_prims(fs):
        p = fs.primitives[pi]
        nodes = np.ctypeslib.as_array(p.curve_nodes, shape=(p.n_curve_nodes*4,)).reshape(-1, 4).astype(np.float64)
        segs = np.ctypeslib.as_array(p.curve_segments, shape=(p.n_curve_segments,)).astype(np.int64)
        P.append(np.full(len(segs), pi)); K.append(np.arange(len(segs)))
        N.append(np.stack([nodes[segs - 2], nodes[segs - 1], nodes[segs]], 1))
    return np.concatenate(P), np.concatenate(K), np.concatenate(N)


def coeffs(n):
    """pointOnSpline's quadratic q0 u^2 + q1 u + q2 of nodes [..., 3, 4]."""
    n0, n1, n2 = n[..., 0, :], n[..., 1, :], n[..., 2, :]
    return 0.5*n0 - n1 + 0.5*n2, n1 - n0, 0.5*(n0 + n1)


def spline(n, u):
    q0, q1, q2 = coeffs(n)
    u = np.asarray(u, np.float64)[..., None]
    return q0*u*u + q1*u + q2


def spline_d(n, u):
    q0, q1, _ = coeffs(n)
    return 2*q0*np.asarray(u, np.float64)[..., None] + q1


# ---- rays ---------------------------------------------------------------------------------------------------------------------
def _unit(v):
    v = np.asarray(v, np.float64)
    return v/np.linalg.norm(v, axis=-1, keepdims=True)


def _pack(o, d, tmin=5e-4, tmax=np.inf):
    n = len(o)
    r = np.zeros((n, 8), F)
    r[:, :3] = o; r[:, 3:6] = d; r[:, 6] = tmin; r[:, 7] = tmax
    return r


def _from_target(tgt, d, rng):
    """Rays in direction d whose line passes through tgt, starting 0.2 .. 1.5 before it."""
    d32 = np.asarray(d, F)
    dist = rng.uniform(0.2, 1.5, len(tgt))
    return _pack((tgt - d32.astype(np.float64)*dist[:, None]).astype(F), d32)


def build_strata(fs, orc, rng, n):
    """name -> rays [m, 8] float32, plus name -> what the stratum must contain (asserted once the hook has run)."""
    P, K, N = segments(fs)
    S = len(P)
    length = np.linalg.norm(N[:, 2, :3] - N[:, 0, :3], axis=1)
    live = np.linalg.norm(spline_d(N, 0.5)[:, :3], axis=1) > 0                       # not a point
    out = {}
    allp = N[:, :, :3].reshape(-1, 3)
    near = np.abs(allp).max(1) < 100.0
    lo, hi = allp[near].min(0) - 0.3, allp[near].max(0) + 0.3
    o = rng.uniform(lo, hi, (n, 3))
    out["random"] = _pack(o.astype(F), _unit(rng.normal(size=(n, 3))).astype(F))
    k = rng.randint(0, S, n); u = rng.rand(n)
    out["aimed at the centreline"] = _from_target(spline(N[k], u)[:, :3], _unit(rng.normal(size=(n, 3))), rng)
    # silhouettes: distance w * (1 + j 2^-20) from the chord of a depth-5 piece, the ray perpendicular to the chord
    m = n//9
    kk = rng.choice(np.flatnonzero(live & (length > 0)), m); piece = rng.randint(0, 32, m); s = rng.uniform(0.2, 0.8, m)
    a, b = spline(N[kk], piece*PIECE), spline(N[kk], (piece + 1)*PIECE)
    c = a + s[:, None]*(b - a)
    ch = b[:, :3] - a[:, :3]
    ok = (np.linalg.norm(ch, axis=1) > 0) & (c[:, 3] > 0)
    c, ch = c[ok], _unit(ch[ok])
    d = _unit(np.cross(ch, rng.normal(size=(len(c), 3))))
    side = _unit(np.cross(d, ch))
    rays = []
    for j in range(-4, 5):
        r = c[:, 3]*(1.0 + j*2.0**-20)
        rays.append(_from_target(c[:, :3] + side*r[:, None], d, rng))
    out["silhouette"] = np.concatenate(rays)
    # joints and free ends
    ends = np.array([0.0, 2.0**-24, 1.0 - 2.0**-24, 1.0])
    k = rng.randint(0, S, n//2); u = ends[rng.randint(0, 4, n//2)]
    out["joints and ends"] = _from_target(spline(N[k], u)[:, :3], _unit(rng.normal(size=(n//2, 3))), rng)
    # along the tangent (exactly along the straight segments: every piece projects to a point)
    k = rng.choice(np.flatnonzero(live), n//4); u = rng.choice([0.0, 0.5, 1.0, 0.3], n//4)
    t = spline_d(N[k], u)[:, :3]
    good = np.linalg.norm(t, axis=1) > 0
    out["along the tangent"] = _from_target(spline(N[k], u)[good, :3], _unit(t[good])*rng.choice([-1.0, 1.0], (int(good.sum()), 1)), rng)
    # +-y exactly, +-y with tiny x / z, axis directions with +-0 components
    k = rng.randint(0, S, n//4); u = rng.rand(n//4)
    d = np.zeros((n//4, 3)); d[:, 1] = rng.choice([-1.0, 1.0], n//4)
    out["+-y"] = _from_target(spline(N[k], u)[:, :3], d, rng)
    tiny = np.array([1e-20, -1e-20, 1e-25, -1e-25])
    k = rng.randint(0, S, n//4); u = rng.rand(n//4)
    d = np.zeros((n//4, 3), F); d[:, 1] = rng.choice([-1.0, 1.0], n//4)
    d[:, 0] = tiny[rng.randint(0, 4, n//4)]; d[:, 2] = tiny[rng.randint(0, 4, n//4)]
    out["+-y, tiny x and z"] = _from_target(spline(N[k], u)[:, :3], d, rng)
    k = rng.randint(0, S, n//4); u = rng.rand(n//4)
    d = np.where(rng.rand(n//4, 3) < 0.5, F(-0.0), F(0.0)).astype(F)
    d[np.arange(n//4), rng.randint(0, 3, n//4)] = rng.choice([-1.0, 1.0], n//4)
    out["axis, +-0 components"] = _from_target(spline(N[k], u)[:, :3], d, rng)
    # tmax / tmin one ulp before, at and after the hook's t; origins on the surface with tmin = the curve epsilon
    base = np.concatenate([out["aimed at the centreline"], out["+-y"], out["axis, +-0 components"]])
    h = hook(orc, fs, base)
    hit = np.flatnonzero(h["seg"] >= 0)
    rb, th = base[hit], h["t"][hit]
    var = []
    for col in (7, 6):
        for t in (np.nextafter(th, F(-np.inf)), th, np.nextafter(th, F(np.inf))):
            r = rb.copy(); r[:, col] = t; var.append(r)
    out["tmax and tmin at the hook's t"] = np.concatenate(var)
    p = (rb[:, :3] + rb[:, 3:6]*th[:, None]).astype(F)
    mode = np.array([fs.primitives[i].curve_mode for i in h["prim"][hit]])
    eps = np.maximum(F(5e-4), np.where(mode == abi.CURVE_CYLINDER, F(0.1), F(0.01))*h["w"][hit]).astype(F)
    out["self-hits"] = _pack(p, _unit(rng.normal(size=(len(p), 3))).astype(F), tmin=eps)
    return out


def strand_ends(fs):
    """prim -> (segment is the first of its strand, segment is the last of its strand), boolean per segment."""
    out = {}
    for pi in curve_prims(fs):
        p = fs.primitives[pi]
        segs = np.ctypeslib.as_array(p.curve_segments, shape=(p.n_curve_segments,)).astype(np.int64)
        first = np.ones(len(segs), bool); first[1:] = segs[:-1] != segs[1:] - 1
        last = np.ones(len(segs), bool); last[:-1] = segs[1:] != segs[:-1] + 1
        out[pi] = (first, last)
    return out


END = 2.0**-10                              # a hit this close (in u) to a segment's end counts as a hit at that end


def check_stratum(fs, scene_name, name, rays, h):
    """The case each stratum exists for occurred; returns what was counted, for the run's report."""
    hit = h["seg"] >= 0
    d = rays[:, 3:6]
    if name == "silhouette":
        j = np.repeat(np.arange(-4, 5), len(rays)//9)
        inner, outer = hit[j == -4].mean(), hit[j == 4].mean()
        assert hit.any() and (~hit).any() and inner > outer, (inner, outer)
        return "hit at k = -4: %.3f, at k = +4: %.3f" % (inner, outer)
    if name == "random":
        assert hit.any() and (~hit).any()
    elif name == "tmax and tmin at the hook's t":
        m = len(rays)//6
        at_tmax, above_tmax = hit[m:2*m], hit[2*m:3*m]
        assert at_tmax.mean() < above_tmax.mean()                 # the hit at exactly tmax is excluded
    elif name == "+-y":
        assert hit.any() and (d[:, 0] == 0).all() and (d[:, 2] == 0).all()
    elif name == "+-y, tiny x and z":
        xz = d[:, 0]*d[:, 0] + d[:, 2]*d[:, 2]
        sub = (xz > 0) & (xz < np.finfo(F).tiny)
        assert (hit & (xz == 0)).any() and (hit & sub).any()
        return "hits with x^2 + z^2 = 0: %d, subnormal: %d" % (int((hit & (xz == 0)).sum()), int((hit & sub).sum()))
    elif name == "axis, +-0 components":
        neg0 = ((d == 0) & np.signbit(d)).any(1)
        assert (hit & neg0).any() and (hit & ~neg0).any()
        return "hits with a -0 component: %d" % int((hit & neg0).sum())
    elif name == "joints and ends":
        ends = strand_ends(fs)
        k = np.flatnonzero(hit)
        first = np.array([ends[p][0][s] for p, s in zip(h["prim"][k], h["seg"][k])], bool)
        last = np.array([ends[p][1][s] for p, s in zip(h["prim"][k], h["seg"][k])], bool)
        at0, at1 = h["u"][k] <= END, h["u"][k] >= 1.0 - END
        n = {"free start": int((at0 & first).sum()), "joint, u = 0": int((at0 & ~first).sum()),
             "joint, u = 1": int((at1 & ~last).sum()), "free end": int((at1 & last).sum())}
        assert all(v > 0 for v in n.values()), n
        return "hits within 2^-10 of an end: %s" % n
    elif name == "along the tangent":
        # exactly along a straight axis-aligned segment every piece's projected chord has length 0 (the edges scene has such
        # segments; a curly strand only comes close)
        axial = (d == 0).sum(1) == 2
        if scene_name == "edges":
            assert (hit & axial).any()
        else:
            assert hit.any()
        return "hits along an exact axis: %d" % int((hit & axial).sum())
    else:
        assert hit.any(), name
    return ""


# ---- the hook and the comparison ----------------------------------------------------------------------------------------------
HOOK_DTYPE = np.dtype([("n_pass", "<u4"), ("n_hit", "<u4"), ("prim", "<i4"), ("seg", "<i4"), ("t", "<f4"), ("u", "<f4"), ("w", "<f4"),
                       ("slack", "<f4")])


def hook(orc, fs, rays):
    """Oracle.curve_segments over every curve primitive: counts summed, the nearest hit of all (prim -1: none)."""
    res = [(pi, orc.curve_segments(pi, rays)) for pi in curve_prims(fs)]
    out = np.zeros(len(rays), HOOK_DTYPE)
    out["prim"] = -1; out["seg"] = -1; out["t"] = np.inf
    for pi, r in res:
        out["n_pass"] += r["n_pass"]; out["n_hit"] += r["n_hit"]
        better = (r["seg"] >= 0) & ((out["seg"] < 0) | (r["t"] < out["t"]))
        for k in ("seg", "t", "u", "w", "slack"):
            out[k] = np.where(better, r[k], out[k])
        out["prim"] = np.where(better, pi, out["prim"])
    return out


def classify(h):
    c = np.full(len(h), MULTI)
    c[h["n_hit"] == 0] = NONE
    one = h["n_hit"] == 1
    c[one & (h["slack"] >= MARGIN)] = INSIDE
    c[one & ~(h["slack"] >= MARGIN)] = OUTSIDE
    return c


def _bits(a):
    return np.ascontiguousarray(a, F).view(np.uint32)


def compare(fs, orc, rays, h, cls, got):
    """got: tgb_hit records of one walk.  Returns per class: rays, exact (the hook's segment, t, u, width bit for bit), bad (a rule of
    the module's table broken), dropped (no curve hit reported)."""
    cp = curve_prims(fs)
    on = np.isin(got["primitive"], cp)
    exact = on & (got["primitive"] == h["prim"]) & (got["prim_id"] == h["seg"]) & (_bits(got["t"]) == _bits(h["t"])) \
        & (_bits(got["u"]) == _bits(h["u"])) & (_bits(got["v"]) == _bits(h["w"]))
    bad = np.zeros(len(rays), bool)
    bad |= (cls == NONE) & on
    bad |= (cls == INSIDE) & ~exact
    bad |= (cls == OUTSIDE) & on & ~exact
    m = np.flatnonzero((cls == MULTI) & on)
    if len(m):
        alone = np.zeros(len(m), bool)
        for pi in cp:
            sel = got["primitive"][m] == pi
            if sel.any():
                alone[sel] = orc.curve_segments(pi, rays[m[sel]], only=got["prim_id"][m[sel]])["n_hit"] == 1
        bad[m[~alone]] = True
    return {c: {"rays": int((cls == c).sum()), "exact": int((exact & (cls == c)).sum()), "bad": int((bad & (cls == c)).sum()),
                "dropped": int((~on & (cls == c)).sum())} for c in range(4)}, bad, exact


def report(scene_name, walk, per_stratum):
    for sname, res in per_stratum.items():
        print("%-6s %-16s %-32s " % (scene_name, walk, sname) + "  ".join(
            "%s %d/%d exact, %d bad, %d dropped" % (CLASS_NAMES[c], r["exact"], r["rays"], r["bad"], r["dropped"]) for c, r in res.items()))


def _total(per_stratum, c, key):
    return sum(r[c][key] for r in per_stratum.values())


def run_walk(fs, orc, strata, hooks, classes, walk_fn):
    per, outs = {}, {}
    for sname, rays in strata.items():
        got = walk_fn(rays)
        per[sname], _, _ = compare(fs, orc, rays, hooks[sname], classes[sname], got)
        outs[sname] = got
    return per, outs


def scene_and_strata(name, scratch, n):
    fs = build_scene(name, scratch)
    orc = pyoracle.Oracle(fs)
    strata = build_strata(fs, orc, np.random.RandomState(123 if name == "edges" else 321), n)
    hooks = {s: hook(orc, fs, r) for s, r in strata.items()}
    classes = {s: classify(h) for s, h in hooks.items()}
    for s, r in strata.items():
        c = classes[s]
        what = check_stratum(fs, name, s, r, hooks[s])
        print("%-6s %-32s %6d rays: %s%s" % (name, s, len(r), ", ".join("%s %d" % (CLASS_NAMES[k], int((c == k).sum())) for k in range(4)),
                                              "; " + what if what else ""))
    return fs, orc, strata, hooks, classes


N_RAYS = {"edges": 24000, "hair": 12000}


# ---- CPU: the oracle's own walk against the hook ----------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["edges", "hair"])
def test_oracle_walk_agrees_with_hook(name, scratch):
    """Oracle.trace (the segment BVH walk the renders use) against the hook: every rule of the module's table, and the oracle's
    drops of the outside class as pinned."""
    fs, orc, strata, hooks, classes = scene_and_strata(name, scratch, N_RAYS[name])
    per, _ = run_walk(fs, orc, strata, hooks, classes, orc.trace)
    report(name, "oracle", per)
    for c in range(4):
        assert _total(per, c, "bad") == 0, CLASS_NAMES[c]
    assert _total(per, INSIDE, "rays") > 1000 and _total(per, INSIDE, "exact") == _total(per, INSIDE, "rays")
    assert _total(per, NONE, "rays") > 1000 and _total(per, OUTSIDE, "rays") > 0
    assert _total(per, OUTSIDE, "dropped") == OUTSIDE_DROPS[(name, "oracle")][0]
    if name == "hair":
        assert _total(per, MULTI, "rays") > 100
    orc.close()


def test_comparison_rejects_wrong_answers(scratch):
    """The comparison flags an expected answer one ulp off in t, a wrong segment and a hit turned into a miss, one ray each."""
    fs, orc, strata, hooks, classes = scene_and_strata("edges", scratch, 4000)
    s = "aimed at the centreline"
    rays, h, cls = strata[s], hooks[s], classes[s]
    got = orc.trace(rays)
    _, bad, _ = compare(fs, orc, rays, h, cls, got)
    assert not bad.any()
    i = np.flatnonzero(cls == INSIDE)[:3]
    segs = segments(fs)
    for what, k in (("t one ulp off", i[0]), ("wrong segment", i[1]), ("hit turned into a miss", i[2])):
        g = got.copy()
        if what == "t one ulp off":
            g["t"][k] = np.nextafter(g["t"][k], F(np.inf))
        elif what == "wrong segment":
            n = int((segs[0] == g["primitive"][k]).sum())
            g["prim_id"][k] = (g["prim_id"][k] + 1) % n
        else:
            g["primitive"][k] = -1; g["t"][k] = np.inf
        _, bad, _ = compare(fs, orc, rays, h, cls, g)
        print("%s: %d rays flagged" % (what, int(bad.sum())))
        assert np.flatnonzero(bad).tolist() == [k], what
    orc.close()


# ---- CPU: the hook against a float64 tube -------------------------------------------------------------------------------------
def tube_model(n, o, d, grid=1025, refine=40):
    """float64, per (ray, segment) pair: f(u) = distance from the ray's line to the centreline point B(u) minus the width w(u),
    sampled on `grid` points and refined by ternary search around the best one.  Returns (min f, u at the min, the ray's entry t
    into the tube of radius w + m and the largest t of a centreline point within w + m of the line, given m) as a function of m."""
    u = np.linspace(0.0, 1.0, grid)
    B = spline(n[:, None], u[None])                                      # [pairs, grid, 4]
    v = B[..., :3] - o[:, None]
    along = (v*d[:, None]).sum(-1)
    perp = np.linalg.norm(v - along[..., None]*d[:, None], axis=-1)
    f = perp - B[..., 3]
    j = f.argmin(1)
    a, b = u[np.maximum(j - 1, 0)], u[np.minimum(j + 1, grid - 1)]

    def fu(x):
        Bx = spline(n, x)
        vx = Bx[:, :3] - o
        al = (vx*d).sum(-1)
        return np.linalg.norm(vx - al[:, None]*d, axis=-1) - Bx[:, 3]
    for _ in range(refine):
        m1, m2 = a + (b - a)/3, b - (b - a)/3
        lt = fu(m1) < fu(m2)
        b = np.where(lt, m2, b); a = np.where(lt, a, m1)
    us = 0.5*(a + b)
    fmin = np.minimum(fu(us), f.min(1))

    def t_bounds(m):
        r = B[..., 3] + m[:, None]
        inside = perp < r
        entry = np.where(inside, along - np.sqrt(np.maximum(r*r - perp*perp, 0.0)), np.inf)
        far = np.where(inside, along, -np.inf).max(1)
        return entry.min(1), far, u[entry.argmin(1)]
    return fmin, us, t_bounds, along


def tube_margin(n, o, d, us):
    """m of each pair, from the segment's depth-5 chord sagitta and its width variation:
      * the sagitta of the centreline and of the width over a piece, grown over the stretch of a chord's extension a piece's box test
        lets through (its largest node width past the piece's end, in parameter units): |q0| (ext + h/2)^2;
      * the width's change between where the ray crosses the axis and where it enters the tube (a piece is a cylinder of the width at
        the crossing, the tube a cone there): |dw/ds| w |cot| of the angle between the ray and the tangent at u*, and the cone's
        spheres reaching past the cylinder across the axis: w (sqrt(1 + (dw/ds)^2) - 1);
      * float32 rounding of the coordinates the segment test sees.
    Also returns ext."""
    q0, q1, _ = coeffs(n)
    u = np.linspace(0.0, 1.0, 65)
    speed = np.linalg.norm(2*q0[:, None, :3]*u[None, :, None] + q1[:, None, :3], axis=-1).min(1)
    wmax = np.abs(n[:, :, 3]).max(1)
    tan = spline_d(n, us)
    tl = np.linalg.norm(tan[:, :3], axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        ext = np.where(speed > 0, 2.0*wmax/speed, np.inf)
        cos = np.abs((tan[:, :3]*d).sum(1))/tl
        g = np.abs(tan[:, 3])/tl
        slope = g*wmax*cos/np.sqrt(np.maximum(1.0 - cos*cos, 0.0)) + wmax*(np.sqrt(1.0 + g*g) - 1.0)
        curv = np.linalg.norm(q0[:, :3], axis=1) + np.abs(q0[:, 3])
        scale = np.maximum(np.abs(n[:, :, :3]).max((1, 2)), np.abs(o).max(1)) + 1.0
        m = np.where(speed > 0, curv*(ext + 0.5*PIECE)**2 + slope, np.inf) + 64*np.finfo(F).eps*scale
    return np.where(np.isnan(m), np.inf, m), ext


def test_hook_agrees_with_float64_tube(scratch):
    """Where the ray passes deeper than m inside the float64 tube, away from the segment's ends, the hook reports a hit alone, at a t
    between the ray's entry into the tube of radius w + m and the farthest centreline point within w + m; where it passes farther
    than m outside, the hook reports none.  m comes from each segment's chord sagitta and width variation (tube_margin)."""
    fs = build_scene("edges", scratch)
    orc = pyoracle.Oracle(fs)
    rng = np.random.RandomState(9)
    st = build_strata(fs, orc, rng, 12000)
    rays = np.concatenate([st["random"], st["aimed at the centreline"], st["silhouette"]])
    P, K, N = segments(fs)
    # pairs: each ray with every segment it passes within 0.05 of the segment's bounding sphere
    o64, d64 = rays[:, :3].astype(np.float64), rays[:, 3:6].astype(np.float64)
    mid = spline(N, 0.5)[:, :3]
    radius = np.linalg.norm(N[:, :, :3] - mid[:, None], axis=-1).max(1) + np.abs(N[:, :, 3]).max(1) + 0.05
    v = mid[None] - o64[:, None]
    al = (v*d64[:, None]).sum(-1)
    dist = np.linalg.norm(v - al[..., None]*d64[:, None], axis=-1)
    ri, si = np.nonzero(dist < radius[None])
    o, d, n = o64[ri], d64[ri], N[si]
    cols = {k: [] for k in ("fmin", "us", "m", "ext", "entry", "far", "ue", "ahead")}
    for a in range(0, len(ri), 8192):                                            # (the model samples [pairs, grid] arrays)
        c = slice(a, a + 8192)
        fmin, us, t_bounds, along = tube_model(n[c], o[c], d[c])
        m, ext = tube_margin(n[c], o[c], d[c], us)
        entry, far, ue = t_bounds(np.where(np.isfinite(m), m, 0.0))
        ahead = along.min(1) > rays[ri[c], 6] + np.abs(n[c, :, 3]).max(1) + m + 1e-3      # the whole segment lies ahead of tmin
        for k, v in zip(cols, (fmin, us, m, ext, entry, far, ue, ahead)):
            cols[k].append(v)
    fmin, us, m, ext, entry, far, ue, ahead = [np.concatenate(cols[k]) for k in cols]
    # the ray's closest approach and its entry into the tube both away from the segment's ends (a hit whose point projects past
    # an end belongs to the next segment of the strand, or to none)
    interior = (np.minimum(us, ue) > ext + PIECE) & (np.maximum(us, ue) < 1.0 - ext - PIECE)
    res = np.concatenate([orc.curve_segments(int(pi), rays[ri[P[si] == pi]], only=K[si[P[si] == pi]]) for pi in curve_prims(fs)])
    order = np.concatenate([np.flatnonzero(P[si] == pi) for pi in curve_prims(fs)])
    h = np.empty_like(res); h[order] = res
    must_hit = ahead & interior & (fmin < -m)
    must_miss = ahead & (fmin > m)
    tol = (1.0/1024)*np.linalg.norm(spline_d(n, us)[:, :3], axis=1)                  # grid step
    t = h["t"].astype(np.float64)
    with np.errstate(invalid="ignore"):                                          # (far = -inf, m = inf where nothing is decided)
        in_range = (t >= entry - tol) & (t <= far + m + tol)
    print("%d (ray, segment) pairs: %d must hit (%d do, %d with t in range), %d must miss (%d do), %d undecided"
          % (len(ri), int(must_hit.sum()), int((must_hit & (h["n_hit"] == 1)).sum()), int((must_hit & in_range).sum()),
             int(must_miss.sum()), int((must_miss & (h["n_hit"] == 0)).sum()), int((~must_hit & ~must_miss).sum())))
    assert must_hit.sum() > 2000 and must_miss.sum() > 2000
    assert (h["n_hit"][must_hit] == 1).all() and in_range[must_hit].all()
    assert (h["n_hit"][must_miss] == 0).all()
    orc.close()


# ---- GPU: the device against the hook -----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["edges", "hair"])
def test_device_hits_agree_with_hook(name, scratch, monkeypatch):
    fs, orc, strata, hooks, classes = scene_and_strata(name, scratch, N_RAYS[name])
    monkeypatch.delenv("TGB_HOOK_CUT", raising=False)
    ctx = lib.Context(fs)
    dev, dev_out = run_walk(fs, orc, strata, hooks, classes, ctx.trace_closest)
    monkeypatch.setenv("TGB_HOOK_CUT", "0")
    nocut, _ = run_walk(fs, orc, strata, hooks, classes, ctx.trace_closest)
    monkeypatch.delenv("TGB_HOOK_CUT")
    ctx.close()
    ora, ora_out = run_walk(fs, orc, strata, hooks, classes, orc.trace)
    report(name, "device", dev); report(name, "device, cut off", nocut); report(name, "oracle", ora)
    mism = 0
    for s in strata:
        m = classes[s] == MULTI
        g, r = dev_out[s], ora_out[s]
        differ = (g["primitive"] != r["primitive"]) | (g["prim_id"] != r["prim_id"]) | (_bits(g["t"]) != _bits(r["t"]))
        mism += int((m & differ).sum())
    drops = {w: _total(p, OUTSIDE, "dropped") for w, p in (("device", dev), ("device, cut off", nocut), ("oracle", ora))}
    print("%s: outside-class drops %s (pinned %s); multi-class device/oracle mismatches %d of %d (pinned %d)"
          % (name, drops, {w: OUTSIDE_DROPS[(name, w)][0] for w in drops}, mism, _total(dev, MULTI, "rays"), MULTI_MISMATCHES[name][0]))
    for walk, per in (("device", dev), ("device, cut off", nocut), ("oracle", ora)):
        for c in range(4):
            assert _total(per, c, "bad") == 0, (walk, CLASS_NAMES[c])
    assert _total(dev, INSIDE, "exact") == _total(dev, INSIDE, "rays")
    assert drops == {w: OUTSIDE_DROPS[(name, w)][0] for w in drops}
    assert mism == MULTI_MISMATCHES[name][0]
    orc.close()
