"""Shadow queries one at a time: TraceBase::attenuatedEmission through the renderer's own shadow kernels, against the CPU oracle.

An image averages a wrong visibility decision into one path of thousands.  Here tgb200_shadow_probe sets up each query as k_shade
does (light_query: the quad / cap / environment light's own hit and the finished lightF / bsdfF, or the mesh light's closest-hit
query) and runs the real k_shadow_prep (analytic primitives, top-level cut, compaction) and k_shadow_bvh (persistent traversal,
the analytic-leaf ignore rule, the any-hit exits, shadow_resolve_closest).  oracle_shadow_probe runs the oracle's
attenuated_emission on the same float32 inputs, with NEE's f = 1, pdfL = 1, pdfB = 0 and MIS's weight = 1.

Query points: hits of seeded random rays (from the camera, then one bounce), the camera itself, points on a quad light's plane,
behind it, on a (non-light) quad's face, cube centres, and points on the line through a blocker's vertex / edge point and the
light (grazing silhouettes).  Every query uses epsilon = 5e-4, curve scenes included (a curve hit's own epsilon,
max(5e-4, k x width), is not used: the probe takes epsilon as an input and the traversal treats every value alike).
Every origin lies inside the scene's or the camera's extent, which the BVH's padding assumes.  Directions: to uniform points of the
light, to its edges and corners (l0 or l1 exactly 0 or 1), uniform on the sphere for infinite lights, axis-parallel ones with
the other components exactly +-0 or of magnitude 1e-31 (below the traversal's 1e-30 clamp).  NEE queries run with expected
distance -1 and then (second pass) at the rejection edge of `t*(1 + 1e-3) < expectedDist`: fl(t_light*(1 + 1e-3)), one ulp
either side of it, and t_light; the ulp above must be rejected on both sides, for quad and mesh lights.  MIS queries run with a
seeded BSDF pdf.

Tolerances (stated here, used below):
  * light hit (quad / cap / environment lights) and vis: exactly equal.  The only exceptions are ties: queries whose oracle
    blocker (the closest hit in [epsilon, t_light] other than the light) lies at exactly t_light in float32, or, between two
    triangles, within 4 ulp of it (a triangle test compares T with absDen*t, so coplanar triangles tie within ulps, not exactly).  Each tie category is a row of TIE_EXCEPTIONS with its reason and the count an H100 run
    measured; only the flush_lights scene has any;
  * the finished value of a query both sides see: bit-exact, NEE and MIS alike, for every light in these scenes (constant,
    bitmap environment, sphere cap, mesh), except a mesh light's MIS value (directPdf), within ULP_BARS: 3x what an H100 run
    measured.
Every run prints what it measured.
"""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import pyoracle
from tungsten_b200 import abi, lib, scene, synth

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
F = np.float32
N_QUERIES = 65536 + 13                  # not a multiple of 32

# (scene, tie, outcome) -> (mismatching queries, reason), measured on an H100 80GB HBM3 at a 400 W power limit (seeded: the same
# count on every run).  The library's blocker test accepts any primitive other than the light in [epsilon, t_light] -- a quad at
# exactly t_light blocks -- and its mesh-light query takes the first of two coplanar triangles its BVH visits.  The oracle takes
# the closest hit of the whole scene and asks whether it is the light: a later-listed quad light wins an exact tie with the
# quad it lies in, and its BVH visits coplanar triangles in another order.  Neither side is the reference's Embree order.
_QUAD_TIE = "quad light coplanar with the table quad listed before it: blocked on the GPU, the oracle's later-listed light wins"
_MESH_TIE = "mesh light coplanar with the mesh shelf: each side's closest hit is the coplanar triangle its BVH visits first"
# An any-hit query's answer does not depend on the order a walk visits the segments in, so curve blockers are exact too.  The one
# possible exception is a query whose only blocker hits outside its segment's curveBox (test_gpu_curve_hits.py's `outside` class),
# which the device's quantised boxes and the oracle's float boxes may each cull; on curve_edges an H100 run measured none.
TIE_EXCEPTIONS = {("flush_lights", "quad light, quad blocker", "gpu blocked"): (1432, _QUAD_TIE),
                  ("flush_lights", "mesh light, mesh blocker", "gpu blocked"): (174, _MESH_TIE),
                  ("flush_lights", "mesh light, mesh blocker", "gpu visible"): (2, _MESH_TIE),
                  ("settled by the analytic pass", "mesh light, mesh blocker", "gpu blocked"): (13, _MESH_TIE),
                  ("settled by the analytic pass", "mesh light, mesh blocker", "gpu visible"): (2, _MESH_TIE)}

# (light type, mis) -> ulp bar of the finished value; every other row is bit-exact.  A mesh light's MIS value holds its directPdf,
# computed from the light's hit point and normal: where the ray crosses an edge between two of the light's triangles, the two
# BVHs may report different ones, and the point moves by an ulp.  Measured 7 ulp (flush_lights, H100).
ULP_BARS = {(abi.PRIM_MESH, 1): 21}


# ---- the two probes -------------------------------------------------------------------------------------------------------
def gpu_probe(ctx, q, lm):
    q = np.ascontiguousarray(q, F); lm = np.ascontiguousarray(lm, np.int32); out = np.zeros((len(q), 8), F)
    ctx._check(ctx.L.tgb200_shadow_probe(ctx.h, len(q), q.ctypes.data, lm.ctypes.data, out.ctypes.data))
    return out


def oracle_probe(o, q, lm):
    q = np.ascontiguousarray(q, F); lm = np.ascontiguousarray(lm, np.int32); out = np.zeros((len(q), 8), F)
    assert pyoracle.lib().oracle_shadow_probe(o.h, len(q), q.ctypes.data, lm.ctypes.data, out.ctypes.data) == 0
    return out


# ---- query construction -----------------------------------------------------------------------------------------------------
def _unit(v):
    v = np.asarray(v, np.float64)
    return (v/np.linalg.norm(v, axis=-1, keepdims=True)).astype(F)


def _mesh(p):
    v = np.ctypeslib.as_array(C.cast(p.verts, C.POINTER(C.c_float)), shape=(p.n_verts*8,)).reshape(-1, 8)[:, :3].copy()
    t = np.ctypeslib.as_array(C.cast(p.tris, C.POINTER(C.c_uint32)), shape=(p.n_tris*4,)).reshape(-1, 4)[:, :3].copy()
    return v, t


def _lights(fs):
    """The samplable lights of the scene: emissive quads and meshes, infinite lights with the sample flag."""
    return [i for i, p in enumerate(fs.primitives) if p.emission_tex >= 0 and
            (p.type in (abi.PRIM_QUAD, abi.PRIM_MESH) or
             (p.type in (abi.PRIM_INFINITE_SPHERE, abi.PRIM_INFINITE_SPHERE_CAP) and p.do_sample))]


def _light_targets(p, rng, n):
    """Points on a quad / mesh light: uniform, edges and corners (None for infinite lights)."""
    if p.type == abi.PRIM_QUAD:
        b, e0, e1 = F(p.base), F(p.edge0), F(p.edge1)
        u, v = rng.rand(n).astype(F), rng.rand(n).astype(F)
        k = rng.randint(0, 4, n)
        u[k == 1] = rng.randint(0, 2, (k == 1).sum()); v[k == 2] = rng.randint(0, 2, (k == 2).sum())
        u[k == 3] = rng.randint(0, 2, (k == 3).sum()); v[k == 3] = rng.randint(0, 2, (k == 3).sum())
        return b + u[:, None]*e0 + v[:, None]*e1
    if p.type == abi.PRIM_MESH:
        vs, ts = _mesh(p)
        tri = ts[rng.randint(0, len(ts), n)]
        w = rng.dirichlet([1, 1, 1], n).astype(F)
        k = rng.randint(0, 4, n)
        w[k == 1] = np.eye(3, dtype=F)[rng.randint(0, 3, (k == 1).sum())]            # vertices
        e = rng.rand((k == 2).sum()).astype(F); w[k == 2] = np.stack([e, 1 - e, np.zeros_like(e)], 1)   # edges
        return (w[:, :, None]*vs[tri]).sum(1).astype(F)
    return None


def _blocker_points(fs, lights, rng, n):
    """Vertices and edge points of non-light meshes and cube edges and corners: rays aimed through them graze a silhouette."""
    pts = []
    for i, p in enumerate(fs.primitives):
        if i in lights:
            continue
        if p.type == abi.PRIM_MESH and p.n_tris:
            vs, ts = _mesh(p)
            tri = ts[rng.randint(0, len(ts), n)]
            e = rng.rand(n).astype(F); e[: n//2] = 0.0
            pts.append(vs[tri[:, 0]]*(1 - e)[:, None] + vs[tri[:, 1]]*e[:, None])
        elif p.type == abi.PRIM_CUBE:
            R = np.float32(p.rot).reshape(3, 3); s = F(p.scale)
            c = rng.choice([-1.0, 1.0], (n, 3)).astype(F); free = rng.randint(0, 3, n)
            c[np.arange(n)[: n//2], free[: n//2]] = rng.uniform(-1, 1, n//2)          # half on edges, half on corners
            pts.append((c*s) @ R.T + F(p.pos))
    return np.concatenate(pts).astype(F) if pts else np.zeros((0, 3), F)


def _surface_points(fs, orc, rng, n):
    """Hits of random rays from the camera, then of one random bounce from those hits (inside rooms): origins stay in the scene."""
    cam = F(fs.camera.pos)
    d = _unit(rng.normal(size=(8*n, 3)))
    rays = np.concatenate([np.tile(cam, (8*n, 1)), d, np.full((8*n, 1), 1e-4, F), np.full((8*n, 1), np.inf, F)], 1)
    h = orc.trace(rays); ok = h["primitive"] >= 0
    p1 = (rays[ok, :3] + rays[ok, 3:6]*h["t"][ok, None]).astype(F)[:n]
    d2 = _unit(rng.normal(size=(len(p1), 3)))
    rays2 = np.concatenate([p1, d2, np.full((len(p1), 1), 5e-4, F), np.full((len(p1), 1), np.inf, F)], 1)
    h2 = orc.trace(rays2); ok2 = h2["primitive"] >= 0
    p2 = (rays2[ok2, :3] + rays2[ok2, 3:6]*h2["t"][ok2, None]).astype(F)
    return np.concatenate([p1, p2, cam[None]]).astype(F)


def build_queries(fs, ctx, orc, seed, n=N_QUERIES):
    """(query float32 [n, 8], light_mis int32 [n, 2], stratum names [n])."""
    rng = np.random.RandomState(seed)
    lights = _lights(fs)
    assert lights, "scene without a samplable light"
    pts = _surface_points(fs, orc, rng, 4096)
    blk = _blocker_points(fs, lights, rng, 512)
    Q, LM, S = [], [], []

    def add(p, d, li, name, eps=5e-4):
        ok = np.isfinite(d).all(1)                                                        # (a target equal to its origin)
        p, d = p[ok], d[ok]
        m = len(p)
        q = np.zeros((m, 8), F); q[:, :3] = p; q[:, 3:6] = d; q[:, 6] = eps; q[:, 7] = -1.0
        lm = np.zeros((m, 2), np.int32); lm[:, 0] = li; lm[:, 1] = rng.randint(0, 2, m)
        mis = lm[:, 1] == 1
        q[mis, 7] = rng.uniform(0.05, 20.0, mis.sum()).astype(F)
        Q.append(q); LM.append(lm); S.extend([name]*m)

    per = max(n//(len(lights)*6), 64)
    for li in lights:
        p = fs.primitives[li]
        tgt = _light_targets(p, rng, per)
        src = pts[rng.randint(0, len(pts), per)]
        if tgt is None:                                                                   # infinite lights
            add(src, _unit(rng.normal(size=(per, 3))), li, "uniform direction")
            ax = np.zeros((per, 3), F); k = rng.randint(0, 3, per); ax[np.arange(per), k] = rng.choice([-1.0, 1.0], per)
            add(src, ax, li, "axis-parallel")
            continue
        add(src, _unit(tgt - src), li, "to the light")
        # axis-parallel towards the light's side, other components +-0 or below the 1e-30 clamp
        dd = tgt - src; k = np.argmax(np.abs(dd), 1)
        ax = np.zeros((per, 3), F); ax[np.arange(per), k] = np.sign(dd[np.arange(per), k])
        z = rng.randint(0, 3, (per, 3))
        tiny = np.where(z == 1, F(-0.0), np.where(z == 2, F(1e-31)*rng.choice([-1, 1], (per, 3)), F(0.0))).astype(F)
        ax = np.where(ax == 0, tiny, ax).astype(F)
        add(src, ax, li, "axis-parallel")
        if len(blk):
            v = blk[rng.randint(0, len(blk), per)]
            s = rng.uniform(0.05, 0.6, per).astype(F)[:, None]
            org = (v + (v - tgt)*s).astype(F)                                              # behind the blocker point, on the line to the light
            add(org, _unit(tgt - org), li, "grazing a blocker")
        if p.type == abi.PRIM_QUAD:
            nrm = _unit(np.cross(F(p.edge1), F(p.edge0)))
            add((tgt + nrm*F(0.05)).astype(F), _unit(tgt[::-1] - tgt), li, "on the light's side")
            add((tgt - nrm*F(0.05)).astype(F), _unit(rng.normal(size=(per, 3))), li, "behind the light")
            onp = (F(p.base) + rng.uniform(-0.5, 1.5, (per, 1)).astype(F)*F(p.edge0) + rng.uniform(-0.5, 1.5, (per, 1)).astype(F)*F(p.edge1)).astype(F)
            add(onp, _unit(tgt - onp), li, "on the light's plane")
        faces = [c for k, c in enumerate(fs.primitives) if c.type == abi.PRIM_QUAD and k not in lights]
        if faces:
            fq = [faces[i % len(faces)] for i in range(per)]
            fp = np.stack([F(f.base) + F(rng.rand())*F(f.edge0) + F(rng.rand())*F(f.edge1) for f in fq]).astype(F)
            add(fp, _unit(tgt - fp), li, "on a blocker's face")
        cubes = [c for c in fs.primitives if c.type == abi.PRIM_CUBE]
        if cubes:
            cp = np.stack([F(cubes[i % len(cubes)].pos) for i in range(per)]).astype(F)
            add(cp, _unit(tgt - cp), li, "inside a cube")
    q, lm = np.concatenate(Q), np.concatenate(LM)
    S = np.array(S)
    sel = rng.permutation(len(q))[:n] if len(q) >= n else np.concatenate([np.arange(len(q)), rng.randint(0, len(q), n - len(q))])
    return q[sel], lm[sel], S[sel]


FUDGE = F(1.0) + F(1e-3)                # attenuatedEmission's fudgeFactor, in float32 as both sides compute it


def nee_distance_strata(q, lm, t_light, rng):
    """NEE queries at the expected-distance rejection edge `t*(1 + 1e-3) < expectedDist`: expectedDist = fl(t_light*(1 + 1e-3))
    (kept), one ulp above it (rejected), one ulp below (kept), or t_light itself.  Returns the queries and the mask of those the
    edge rejects."""
    q = q.copy()
    nee = (lm[:, 1] == 0) & np.isfinite(t_light) & (t_light > 0)
    k = rng.randint(0, 4, len(q))
    edge = (t_light*FUDGE).astype(F)
    q[nee & (k == 0), 7] = t_light[nee & (k == 0)]
    q[nee & (k == 1), 7] = edge[nee & (k == 1)]
    q[nee & (k == 2), 7] = np.nextafter(edge, F(np.inf))[nee & (k == 2)]
    q[nee & (k == 3), 7] = np.nextafter(edge, F(-np.inf))[nee & (k == 3)]
    return q, nee & (k == 2)


def _ulp(a, b):
    with np.errstate(invalid="ignore", over="ignore"):
        m = np.maximum(np.abs(a), np.abs(b)).max(-1)
        u = (np.abs(a - b).max(-1)/np.spacing(m.astype(F))).astype(np.float64)
    return np.where((a == b).all(-1), 0.0, u)


def compare(name, fs, ctx, orc, q, lm, strata, ties_at_most=False):
    """ties_at_most: the pass moves expected distances, which can only reject tied queries: at most the recorded counts."""
    g = gpu_probe(ctx, q, lm); r = oracle_probe(orc, q, lm)
    types = np.array([fs.primitives[i].type for i in lm[:, 0]])
    analytic_light = types != abi.PRIM_MESH
    hit_bad = analytic_light & (g[:, 0] != r[:, 0])
    vis_bad = g[:, 2] != r[:, 2]
    # ties: the oracle's blocker other than the light lies at exactly the light's distance (quads), or within 4 ulp of it
    # (two triangles: each test compares T with absDen*t)
    blk = r[:, 6].astype(int)
    btype = np.array([fs.primitives[b].type if b >= 0 else -1 for b in blk])
    exact = r[:, 7] == r[:, 1]
    near = np.abs(r[:, 7] - r[:, 1]) <= 4*np.spacing(np.abs(r[:, 1]))
    tie = (blk >= 0) & (blk != lm[:, 0]) & (exact | ((btype == abi.PRIM_MESH) & (types == abi.PRIM_MESH) & near))
    bad = (hit_bad | vis_bad) & ~tie
    ties = int(((hit_bad | vis_bad) & tie).sum())
    kinds = {abi.PRIM_QUAD: "quad", abi.PRIM_MESH: "mesh", abi.PRIM_CUBE: "cube"}
    found = {}
    for i in np.flatnonzero((hit_bad | vis_bad) & tie):
        key = (name.split(" (")[0], "%s light, %s blocker" % (kinds.get(int(types[i]), "other"), kinds.get(int(btype[i]), "other")),
               "gpu %s" % ("visible" if g[i, 2] else "blocked"))
        found[key] = found.get(key, 0) + 1
    print("%s: %d queries (%d queued, %d any), light hits %d, visible %d/%d (gpu/oracle); mismatches: hit %d, vis %d, of which exact ties %d"
          % (name, len(q), int(g[:, 6].sum()), int(g[:, 7].sum()), int((g[:, 0] * analytic_light).sum()), int(g[:, 2].sum()),
             int(r[:, 2].sum()), int(hit_bad.sum()), int(vis_bad.sum()), ties))
    for s in np.unique(strata):
        m = strata == s
        print("    %-22s %6d queries, visible %6d, mismatches %d" % (s, int(m.sum()), int(r[m, 2].sum()), int(((hit_bad | vis_bad) & m).sum())))
    if bad.any():
        i = np.flatnonzero(bad)[:5]
        print("first non-tie mismatches:\n", q[i], lm[i], g[i], r[i])
    for key, cnt in sorted(found.items()):
        print("    tie: %s: %d" % (" / ".join(key), cnt))
    assert not bad.any(), "%s: %d visibility mismatches that are not ties" % (name, int(bad.sum()))
    expected = {k: v[0] for k, v in TIE_EXCEPTIONS.items() if k[0] == name.split(" (")[0]}
    if ties_at_most:
        assert all(v <= expected.get(k, 0) for k, v in found.items()), (found, expected)
    else:
        assert found == expected, (found, expected)
    both = (g[:, 2] == 1) & (r[:, 2] == 1)
    u = _ulp(g[both, 3:6], r[both, 3:6])
    for kind in np.unique(types[both]):
        for mis in (0, 1):
            m = (types[both] == kind) & (lm[both, 1] == mis)
            if not m.any():
                continue
            key = (name, int(kind), mis)
            worst = float(np.nanmax(u[m])) if m.any() else 0.0
            print("    values, light type %d %s: %d compared, max %.1f ulp, bit-exact %.5f"
                  % (kind, "MIS" if mis else "NEE", int(m.sum()), worst, float((u[m] == 0).mean())))
            assert worst <= ULP_BARS.get((int(kind), mis), 0), key
    return g, r


# ---- scenes ---------------------------------------------------------------------------------------------------------------
def _scene(name, scratch):
    if name == "cornell":
        return scene.load_scene(synth.cornell_box(res=(32, 32), spp=1))
    if name == "cube_city":
        return scene.load_scene(synth.cube_city(res=(32, 32), spp=1, n=12))
    if name == "many_lights":
        return scene.load_scene(synth.many_lights(scratch, res=(32, 32), spp=1, subdiv=3))
    if name == "flush_lights":
        return scene.load_scene(synth.flush_lights(scratch, res=(32, 32), spp=1))
    if name == "hair":
        return scene.load_scene(synth.hair_scene(scratch, n_curves=300, res=(32, 32), spp=1))
    if name == "curve_edges":
        import test_gpu_curve_hits as CH
        return CH.build_scene("edges", scratch)
    return scene.load_scene(os.path.join(G, name, "scene.json"))          # materials_env, hair_sky


SCENES = ["cornell", "cornell_analytic_bvh", "cube_city", "many_lights", "materials_env", "hair_sky", "hair", "flush_lights", "curve_edges"]


@pytest.mark.parametrize("name", SCENES)
def test_shadow_queries_match_oracle(name, scratch, monkeypatch):
    if name == "cornell_analytic_bvh":
        monkeypatch.setenv("TGB_ANALYTIC_BVH_MIN", "1")                  # the quads and cubes become BVH leaves: the ignore rule runs
    fs = _scene(name.replace("_analytic_bvh", ""), scratch)
    ctx = lib.Context(fs); orc = pyoracle.Oracle(fs)
    if name == "cornell_analytic_bvh":
        assert ctx.scene_info()["n_nodes"] > 0
    q, lm, strata = build_queries(fs, ctx, orc, seed=11)
    _, r = compare(name, fs, ctx, orc, q, lm, strata)
    # the oracle's t_light (the light's own intersect) for every light type: the GPU reports none for mesh lights
    q2, above = nee_distance_strata(q, lm, r[:, 1], np.random.RandomState(12))
    g2, r2 = compare(name + " (NEE expected distances)", fs, ctx, orc, q2, lm, strata, ties_at_most=True)
    types = np.array([fs.primitives[i].type for i in lm[:, 0]])
    for kind in (abi.PRIM_QUAD, abi.PRIM_MESH):
        m = above & (types == kind) & (r[:, 0] == 1)                  # the light is hit and the expected distance is one ulp too far
        if not m.any():
            continue
        print("    %s lights, expected distance one ulp past the edge: %d queries, rejected %d (oracle) / %d (gpu, no light hit or not visible)"
              % ("quad" if kind == abi.PRIM_QUAD else "mesh", int(m.sum()), int((r2[m, 0] == 0).sum()),
                 int(((g2[m, 0] == 0) | (g2[m, 2] == 0)).sum())))
        assert (r2[m, 0] == 0).all() and (r2[m, 2] == 0).all() and (g2[m, 2] == 0).all()
        if kind == abi.PRIM_QUAD:
            assert (g2[m, 0] == 0).all()
    if np.isin(types, (abi.PRIM_QUAD, abi.PRIM_MESH)).any():
        assert (above & (r[:, 0] == 1)).any()
    ctx.close(); orc.close()


def test_chunks_and_settled_queries(scratch):
    """n = capacity + 1 on a context of 1500 paths in flight (two chunks) gives what one chunk gives; a batch where the analytic
    pass and the cut settle almost every query and only a few reach the BVH kernel."""
    fs = scene.load_scene(synth.flush_lights(scratch, name="flush_chunks", res=(32, 32), spp=1))
    big = lib.Context(fs); orc = pyoracle.Oracle(fs)
    small = lib.Context(fs, max_paths_in_flight=1500)
    cap = small.scene_info()["capacity"]
    q, lm, _ = build_queries(fs, big, orc, seed=5, n=cap + 1)
    a, b = gpu_probe(big, q, lm), gpu_probe(small, q, lm)
    print("capacity %d, %d queries: chunked == one launch: %s" % (cap, len(q), np.array_equal(a.view(np.uint32), b.view(np.uint32))))
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    # settled: queries from the floor under the front of the room towards the ceiling light (only quads and cubes on the way: the
    # analytic pass and the cut settle them), and 1 in 64 towards the shelf's mesh light, which the BVH pass must resolve
    rng = np.random.RandomState(6)
    n = 4096
    ceil = next(i for i, p in enumerate(fs.primitives) if p.type == abi.PRIM_QUAD and p.emission_tex >= 0 and F(p.base)[1] > 1.9)
    lamp = next(i for i, p in enumerate(fs.primitives) if p.type == abi.PRIM_MESH and p.emission_tex >= 0)
    to_lamp = np.arange(n) % 64 == 0
    lp = fs.primitives[ceil]
    p = np.stack([rng.uniform(-0.9, 0.9, n), np.full(n, 0.001), rng.uniform(0.75, 0.95, n)], 1).astype(F)
    t = (F(lp.base) + rng.rand(n, 1).astype(F)*F(lp.edge0) + rng.rand(n, 1).astype(F)*F(lp.edge1)).astype(F)
    t[to_lamp] = _light_targets(fs.primitives[lamp], rng, int(to_lamp.sum()))
    p[to_lamp, 1] = 1.9                                                   # above the shelf, looking down at its light
    qs = np.zeros((n, 8), F); qs[:, :3] = p; qs[:, 3:6] = _unit(t - p); qs[:, 6] = 5e-4; qs[:, 7] = -1.0
    lms = np.stack([np.where(to_lamp, lamp, ceil), rng.randint(0, 2, n)], 1).astype(np.int32)
    qs[lms[:, 1] == 1, 7] = 1.0
    g, _ = compare("settled by the analytic pass", fs, big, orc, qs, lms, np.where(to_lamp, "to the mesh light", "to the ceiling light"))
    traversed = g[:, 6] == 2
    print("    queued %d, reached the BVH pass %d (%d of them towards the mesh light)"
          % (int((g[:, 6] > 0).sum()), int(traversed.sum()), int((traversed & to_lamp).sum())))
    assert (g[to_lamp, 6] == 2).all()                                     # a mesh light is only found by the traversal
    assert traversed.sum() <= 2*to_lamp.sum() and (g[:, 6] > 0).sum() >= 0.5*n
    big.close(); small.close(); orc.close()


def test_probe_leaves_the_context_unchanged(scratch):
    """A render after a probe equals a render on a fresh context, bit for bit, with the same ray counts."""
    fs = scene.load_scene(synth.many_lights(scratch, name="ml_probe", res=(48, 48), spp=2, subdiv=2))
    fresh = lib.Context(fs); img0, cnt0 = fresh.render_tiles(2); s0 = fresh.stats(); fresh.close()
    ctx = lib.Context(fs); orc = pyoracle.Oracle(fs)
    q, lm, _ = build_queries(fs, ctx, orc, seed=3, n=5000)
    gpu_probe(ctx, q, lm)
    img1, cnt1 = ctx.render_tiles(2); s1 = ctx.stats(); ctx.close(); orc.close()
    print("rays %d/%d, shadow rays %d/%d, hits %d/%d" % (s0.rays, s1.rays, s0.shadow_rays, s1.shadow_rays, s0.hits, s1.hits))
    assert np.array_equal(img0.view(np.uint32), img1.view(np.uint32)) and np.array_equal(cnt0, cnt1)
    assert (s0.rays, s0.hits, s0.shadow_rays, s0.path_rays) == (s1.rays, s1.hits, s1.shadow_rays, s1.path_rays)
