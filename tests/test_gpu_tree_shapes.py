"""BVH traversal on every tree shape build_scene_bvh (bvh_build.cpp) makes, down to walks that spill the stack into local memory.

The other traversal tests run realistic scenes: one large triangle tree, sometimes with a curve subtree, walked to moderate depth.
The scenes here reach the builder's other branches and the traversal's other paths.  Each row names the branch a scene reaches and
how the test knows it reached it (scene_info(): n_tris, n_nodes, bvh_depth; "off" = the same scene with its quads and cubes left in
the per-ray loop, TGB_ANALYTIC_BVH_MIN=100000):

  scene                 | contents                                       | branch reached                               | known by
  ----------------------+------------------------------------------------+----------------------------------------------+--------------------------------
  leaf1, leaf3, leaf4   | 1, 3, 4 faces of a tetrahedron (every face's   | build_from_boxes `rt.left < 0`: the root is  | n_nodes == 1, bvh_depth == 1
                        | box is the tetrahedron's box) + environment    | one leaf and three empty slots; the cut is   | (tgb200_qbvh_selftest's n_nodes
                        |                                                | that single leaf (pop_node starts in LEAF)   | on the CPU)
  leaf1_quad            | one face + a quad light (per-ray loop)         | as above, with the loop's quad               | n_nodes == 1
  curves                | 6 curves, floor + quad light (per-ray loop)    | lone curve tree copied, leaf codes flagged   | n_tris == 0, n_nodes >= 1
                        |                                                | (bit 2) and offset by n_tris = 0             |
  analytic1, 2, 5       | TGB_ANALYTIC_BVH_MIN=1: a cube; a cube + quad  | lone analytic tree copied, leaf codes moved  | n_tris == 0, n_nodes == 1 for
                        | light; 3 cubes + floor + quad light            | to analytic_base = 1 (the all-zero record    | 1 and 2 primitives (leaf cap 2)
                        |                                                | sits at 0)                                   |
  tri_analytic          | 320-triangle ball + 3 cubes, floor, 2 quad     | joint root over two subtrees; analytic codes | n_nodes >= off + 2,
                        | lights, TGB_ANALYTIC_BVH_MIN=1                 | at n_tris + 1                                | bvh_depth >= off + 1
  curves_analytic       | 8 curves + 3 cubes, floor, 2 quad lights,      | joint root over curve and analytic subtrees: | n_tris == 0, n_nodes >= off + 2,
                        | TGB_ANALYTIC_BVH_MIN=1                         | the CURVES k_shadow_bvh runs the analytic    | bvh_depth >= off + 1
                        |                                                | leaves' `ignore` rule                        |
  tri_curves_analytic   | hair_scene(head=True) + 3 cubes + a second     | joint root over three subtrees; curve codes  | n_nodes > off, bvh_depth >= off
                        | quad light, TGB_ANALYTIC_BVH_MIN=1             | at n_tris, analytic at n_tris + n_curve + 1  |
  deep                  | 200 copies of one triangle stacked at          | walks past stack entry 31 into local[]       | host count (same tree): deepest
                        | z = 1.1^k x 1e-6, TGB_TRI_LEAF=1               | while traversal_stack_need <= 80             | stack > 32 and <= need
  too_deep              | 800 copies at z = 1.13^k x 1e-27, TGB_TRI_LEAF | traversal_stack_need > 80 (83 with 4 cut     | TGB_ERR_UNSUPPORTED, host and
                        | =1                                             | boxes, 89 with 16)                           | tgb200_create alike

Every scene runs with TGB_CUT_BOXES=4 and =16.  Every ray origin and query point lies inside the scene's or the camera's extent,
which the BVH's box padding assumes (tgb200_api.cu, build_scene_bvh).

Checks on the GPU, per scene and cut size:
  * closest hits of tgb200_trace_closest against the oracle's trace: seeded rays, part of them aimed at the scene's own features
    (triangle vertices and centroids, curve nodes, quad corners, cube corners, the deep scene's stacking axis), axis-parallel
    rays whose other components are +-0 or below the 1e-30 clamp, and finite t_max one ulp either side of the oracle's hit.
    Same primitive and id except ties within 4 ulp, t and backside bit for bit; curve hits may differ as in
    test_gpu_parity.test_curve_hits_match_oracle (the oracle's segment BVH prunes in another order), counted in CURVE_MISMATCHES.
    TGB_HOOK_CUT=0 gives the same bytes;
  * shadow queries through tgb200_shadow_probe against the oracle (test_gpu_shadow.build_queries and compare): visibility exact,
    values bit for bit; TGB_SHADOW_CUT_ENTRY=0 gives the same bytes;
  * a 32x32, 4 spp image against the oracle's (test_gpu_parity._compare): >= 99.99 % of pixels within 1e-5*(1+L) and RMSE
    <= 1e-5 of the mean on the Lambert-only scenes, the curve scenes' bar (99 %, 3e-2) where there are curves.

The stack really spills: the deep scene is triangles only, so tgb200_shadow_walk_count builds the tree tgb200_create builds (same
camera, same switches) and walks the test's own queries with the kernels' arithmetic.  Its last column is the deepest stack of the
sorted walk from the root, which for a ray that hits nothing IS k_trace's closest-hit walk (same sorting network, same push order,
and a t_max that never shrinks); its second column is the any-hit walk from the cut, k_shadow_bvh's.  Both go past entry 31.
The any-hit walk does not depend on the order in which `enter` pushes the cut boxes: every entered box is walked whatever the
order, and the answer is whether any primitive blocks the segment.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from tungsten_b200 import abi, lib, scene, synth

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import shadow_walk_count as swc  # noqa: E402

F = np.float32
CUTS = ["4", "16"]
SHAPES = ["leaf1", "leaf3", "leaf4", "leaf1_quad", "curves", "analytic1", "analytic2", "analytic5", "tri_analytic",
          "curves_analytic", "tri_curves_analytic", "deep"]
CURVE_SHAPES = ("curves", "curves_analytic", "tri_curves_analytic")
BVH_SWITCHES = ("TGB_CUT_BOXES", "TGB_TRI_LEAF", "TGB_TRI_COST", "TGB_CURVE_LEAF", "TGB_CURVE_COST", "TGB_ANALYTIC_BVH_MIN",
                "TGB_HOOK_CUT", "TGB_SHADOW_CUT_ENTRY")

# closest hits on curves that differ from the oracle's other than by a tie, per scene (seeded: the same on every run), measured on
# an H100 80GB HBM3; test_curve_hits_match_oracle explains them
CURVE_MISMATCHES = {"curves": 0, "curves_analytic": 0, "tri_curves_analytic": 0}
# rays whose curve hit the top-level cut's pre-test drops (tgb200_trace_closest with the cut, against TGB_HOOK_CUT=0), per scene and
# cut size,
# measured on an H100 80GB HBM3: a half-cylinder piece accepts hits on the extension of its chord (DESIGN.md section 2), which can lie
# outside the segment's box, so a ray that misses every cut box can still hit a curve in the full traversal
CUT_DROPS = {("curves", "4"): 1, ("curves", "16"): 2, ("curves_analytic", "16"): 1}


# ---- scenes -------------------------------------------------------------------------------------------------------------------
def tetra_faces(k):
    """The first k faces of a regular tetrahedron of half-size 0.5: every face's box is the tetrahedron's box, so the SAH keeps up
    to four of them in one leaf (a split would cost 1 + n intersections against n)."""
    p = 0.5*np.array([[1, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1]], np.float64)
    faces = [(0, 1, 2), (0, 3, 1), (0, 2, 3), (1, 3, 2)]
    return np.array([np.concatenate([p[a], p[b], p[c]]) for a, b, c in faces[:k]], F)


def stacked(n, z):
    """n copies of the triangle (-1, -1), (3, -1), (-1, 3), the k-th at height z[k]."""
    tv = np.tile(F([-1, -1, 0, 3, -1, 0, -1, 3, 0]), (n, 1))
    tv[:, 2::3] = np.asarray(z, F)[:, None]
    return tv


def deep_tris():
    return stacked(200, (1e-6*1.1**np.arange(200)).astype(F))


def too_deep_tris():
    return stacked(800, (1e-27*1.13**np.arange(800)).astype(F))


def _tri_mesh(tv):
    v = np.zeros(3*len(tv), scene.VERTEX_DTYPE)
    p = tv.reshape(-1, 3, 3).astype(np.float64)
    n = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]); n /= np.linalg.norm(n, axis=1, keepdims=True)
    v["pos"] = tv.reshape(-1, 3); v["normal"] = np.repeat(n, 3, axis=0).astype(F)
    t = np.zeros(len(tv), scene.TRI_DTYPE)
    t["v0"], t["v1"], t["v2"] = np.arange(len(tv))*3, np.arange(len(tv))*3 + 1, np.arange(len(tv))*3 + 2
    return v, t


def _lambert(name, albedo):
    return {"name": name, "type": "lambert", "albedo": list(albedo)}


def _quad(name, pos, scale, rot=(0, 0, 0), bsdf="floor", **kw):
    d = {"name": name, "type": "quad", "bsdf": bsdf, "transform": {"position": list(pos), "scale": list(scale), "rotation": list(rot)}}
    d.update(kw)
    return d


def _cube(name, pos, scale, rot, bsdf="box"):
    return {"name": name, "type": "cube", "bsdf": bsdf, "transform": {"position": list(pos), "scale": list(scale), "rotation": list(rot)}}


# (lifted 0.05 off the floor: a ray lying in a cube face's plane is a case of the cube test, where the oracle and the kernels part
# ways, not of the traversal, and shadow queries start on the floor along it)
CUBES = [_cube("c0", (-0.9, 0.35, 0.6), (0.5, 0.6, 0.4), (0, 25, 0)), _cube("c1", (0.9, 0.45, -0.5), (0.4, 0.8, 0.5), (10, -30, 5)),
         _cube("c2", (0.2, 0.25, 1.1), (0.3, 0.4, 0.3), (0, 60, 0))]
LIGHTS = [_quad("l0", (0.6, 2.4, 0.8), (0.7, 1, 0.5), (0, 0, 160), bsdf="lamp", emission=[18, 15, 12]),
          _quad("l1", (-0.8, 2.2, -0.6), (0.5, 1, 0.6), (0, 40, 200), bsdf="lamp", emission=[8, 12, 16])]
FLOOR = _quad("floor", (0, 0, 0), (4, 1, 4))


def _fibers(n_curves, path):
    ends, nodes = synth.curly_fibers(n_curves, 10, width=0.02)
    scene.save_fiber(path, ends, nodes)
    return {"name": "strands", "type": "curves", "file": os.path.basename(path), "mode": "half_cylinder", "bsdf": "strand",
            "transform": {"position": [0.0, 1.55, 0.0], "scale": [1.0, 1.1, 1.0], "rotation": [0, 20, 0]}}


def _scene_dict(prims, cam, look_at, env=0.5):
    bsdfs = [_lambert("floor", [0.5, 0.5, 0.5]), _lambert("box", [0.7, 0.6, 0.4]), _lambert("mat", [0.6, 0.55, 0.7]),
             _lambert("strand", [0.6, 0.4, 0.2]), {"name": "lamp", "type": "null", "albedo": 1.0}]
    prims = list(prims) + [{"name": "env", "type": "infinite_sphere", "emission": [env, env, env], "sample": True}]
    return {"media": [], "bsdfs": bsdfs, "primitives": prims,
            "camera": {"tonemap": "filmic", "resolution": [32, 32], "reconstruction_filter": "tent",
                       "transform": {"position": list(cam), "look_at": list(look_at), "up": [0, 1, 0]}, "type": "pinhole", "fov": 35},
            "integrator": {"type": "path_tracer", "min_bounces": 0, "max_bounces": 8, "enable_consistency_checks": False,
                           "enable_two_sided_shading": True, "enable_light_sampling": True},
            "renderer": synth._renderer(4)}


def _mesh_prim(scratch, name, tv):
    scene.save_wo3(os.path.join(scratch, name + ".wo3"), *_tri_mesh(tv))
    return {"name": name, "type": "mesh", "file": name + ".wo3", "smooth": False, "bsdf": "mat"}


# below the stack, inside the extent its top triangle (z = 172.6) sets: the box padding is then what tgb200_create gives C1-like
# scenes, 1e-6 x the scene's largest coordinate
DEEP_CAM = (1.0, 1.0, -5.0)


def build_scene(shape, scratch):
    """(flat scene, environment switches) of one row of the table."""
    d = os.path.join(scratch, "shapes"); os.makedirs(d, exist_ok=True)
    env = {}
    if shape.startswith("leaf"):
        k = int(shape[4])
        prims = [_mesh_prim(d, shape, tetra_faces(k))]
        if shape == "leaf1_quad":
            prims.append(_quad("l0", (0.0, 1.2, 0.3), (0.6, 1, 0.6), (0, 0, 180), bsdf="lamp", emission=[9, 8, 7]))
        sc = _scene_dict(prims, (0.4, 0.6, 3.5), (0, 0, 0))
    elif shape == "curves":
        sc = _scene_dict([FLOOR, _fibers(6, os.path.join(d, "curves.fiber")), LIGHTS[0]], (0.3, 1.2, 3.4), (0, 0.95, 0))
    elif shape.startswith("analytic"):
        env["TGB_ANALYTIC_BVH_MIN"] = "1"
        prims = {"analytic1": [CUBES[0]], "analytic2": [CUBES[0], LIGHTS[0]], "analytic5": CUBES + [FLOOR, LIGHTS[0]]}[shape]
        sc = _scene_dict(prims, (1.5, 2.0, 4.5), (0, 0.5, 0))
    elif shape == "tri_analytic":
        env["TGB_ANALYTIC_BVH_MIN"] = "1"
        v, t = synth.icosphere(2, 0.5, displace=0.05)
        tv = v["pos"][np.stack([t["v0"], t["v1"], t["v2"]], 1)].reshape(-1, 9) + F([0, 1, 0]*3)
        sc = _scene_dict([_mesh_prim(d, "ball", tv.astype(F))] + CUBES + [FLOOR] + LIGHTS, (1.5, 2.0, 4.5), (0, 0.6, 0))
    elif shape == "curves_analytic":
        env["TGB_ANALYTIC_BVH_MIN"] = "1"
        sc = _scene_dict([_fibers(8, os.path.join(d, "curves_analytic.fiber"))] + CUBES + [FLOOR] + LIGHTS, (1.0, 1.6, 4.0), (0, 0.8, 0))
    elif shape == "tri_curves_analytic":
        env["TGB_ANALYTIC_BVH_MIN"] = "1"
        path = synth.hair_scene(d, name="tca", n_curves=40, res=(32, 32), spp=4, max_bounces=8, head=True)
        import json
        with open(path) as f:
            sc = json.load(f)
        sc["primitives"] += CUBES + [LIGHTS[1]]
        sc["bsdfs"].append(_lambert("box", [0.7, 0.6, 0.4])); sc["bsdfs"].append({"name": "lamp", "type": "null", "albedo": 1.0})
    elif shape == "deep":
        env["TGB_TRI_LEAF"] = "1"
        sc = _scene_dict([_mesh_prim(d, "deep", deep_tris())], DEEP_CAM, (1.0, 1.0, 1.0))
    elif shape == "too_deep":
        env["TGB_TRI_LEAF"] = "1"
        sc = _scene_dict([_mesh_prim(d, "too_deep", too_deep_tris())], DEEP_CAM, (1.0, 1.0, 1.0))
    else:
        raise KeyError(shape)
    return scene.load_scene(sc, base_dir=d), env


def _switches(monkeypatch, env, cut):
    for k in BVH_SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("TGB_CUT_BOXES", cut)


# ---- rays ---------------------------------------------------------------------------------------------------------------------
def _mesh(p):
    v = np.ctypeslib.as_array(C.cast(p.verts, C.POINTER(C.c_float)), shape=(p.n_verts*8,)).reshape(-1, 8)[:, :3].copy()
    t = np.ctypeslib.as_array(C.cast(p.tris, C.POINTER(C.c_uint32)), shape=(p.n_tris*4,)).reshape(-1, 4)[:, :3].copy()
    return v, t


def features(fs):
    """World-space points of the scene's own geometry: triangle vertices and centroids, curve nodes, quad corners and centres,
    cube corners and centres."""
    pts = []
    for p in fs.primitives:
        if p.type == abi.PRIM_MESH and p.n_tris:
            v, t = _mesh(p)
            pts += [v, v[t].mean(1)]
        elif p.type == abi.PRIM_CURVES and p.n_curve_nodes:
            pts.append(np.ctypeslib.as_array(p.curve_nodes, shape=(p.n_curve_nodes*4,)).reshape(-1, 4)[:, :3])
        elif p.type == abi.PRIM_QUAD:
            b, e0, e1 = F(p.base), F(p.edge0), F(p.edge1)
            pts.append(np.stack([b, b + e0, b + e1, b + e0 + e1, b + 0.5*e0 + 0.5*e1]))
        elif p.type == abi.PRIM_CUBE:
            R = np.float32(p.rot).reshape(3, 3); s = F(p.scale)
            c = np.array([[i, j, k] for i in (-1, 1) for j in (-1, 1) for k in (-1, 1)] + [[0, 0, 0]], F)
            pts.append((c*s) @ R.T + F(p.pos))
    return np.concatenate(pts).astype(F)


def _axis_dirs(rng, k):
    ax = np.zeros((k, 3), F); a = rng.randint(0, 3, k); ax[np.arange(k), a] = rng.choice([-1.0, 1.0], k)
    z = rng.randint(0, 3, (k, 3))
    tiny = np.where(z == 1, F(-0.0), np.where(z == 2, F(1e-31)*rng.choice([-1, 1], (k, 3)), F(0.0)))
    return np.where(ax == 0, tiny, ax).astype(F)


def _unit(v):
    v = np.asarray(v, np.float64)
    return (v/np.linalg.norm(v, axis=-1, keepdims=True)).astype(F)


def _pack(o, d, tnear=5e-4, tmax=np.inf):
    n = len(o)
    return np.concatenate([o, d, np.full((n, 1), tnear, F), np.full((n, 1), tmax, F)], 1).astype(F)


def stack_axis_rays(rng, n, hit):
    """Rays along +-z through the deep scene's stack: in the corner x, y in [2.3, 2.9] they are inside every box and outside every
    triangle (x + y > 2); with hit, inside the triangles (x, y > -1, x + y < 2) they stop at the lowest or highest one."""
    if hit:
        x, y = rng.uniform(-0.9, 0.9, n), rng.uniform(-0.9, 0.9, n)
    else:
        x, y = rng.uniform(2.3, 2.9, n), rng.uniform(2.3, 2.9, n)
    up = rng.rand(n) < 0.5
    o = np.stack([x, y, np.where(up, -1.0, 172.5)], 1).astype(F)
    d = np.zeros((n, 3), F); d[:, 2] = np.where(up, 1.0, -1.0)
    return _pack(o, d)


def hit_rays(fs, rng, n, trace, deep=False):
    """Seeded rays with origins inside the box of the scene's features and the camera: random directions, directions aimed at the
    features, axis-parallel ones; then finite t_max one ulp before / at / after the oracle's hit of some of them."""
    pts = features(fs)
    allp = np.concatenate([pts, F(fs.camera.pos)[None]])
    lo, hi = allp.min(0), allp.max(0)
    o = rng.uniform(lo, hi, (n, 3)).astype(F)
    d = _unit(rng.normal(size=(n, 3)))
    k = n//4
    d[:k] = _unit(pts[rng.randint(0, len(pts), k)] - o[:k])                  # aimed at vertices, centroids, nodes, corners
    d[k:k + n//8] = _axis_dirs(rng, n//8)
    ok = np.isfinite(d).all(1)
    rays = [_pack(o[ok], d[ok])]
    if deep:
        rays += [stack_axis_rays(rng, n//8, True), stack_axis_rays(rng, n//8, False)]
    rays = np.concatenate(rays)
    t = trace(rays)["t"]
    idx = np.flatnonzero(np.isfinite(t))[: n//4]
    fin = rays[idx].copy()
    sel = rng.randint(0, 3, len(idx))
    fin[:, 7] = np.where(sel == 0, np.nextafter(t[idx], F(0)), np.where(sel == 1, t[idx], np.nextafter(t[idx], F(np.inf))))
    return np.concatenate([rays, fin]).astype(F)


# ---- host-only checks (no GPU) ------------------------------------------------------------------------------------------------
def qbvh_selftest(tv, rays):
    L = lib.load()
    tv = np.ascontiguousarray(tv, F); rays = np.ascontiguousarray(rays, F)
    bad, nn, visits = C.c_uint32(), C.c_uint32(), C.c_uint64()
    rc = L.tgb200_qbvh_selftest(tv.ctypes.data, len(tv), rays.ctypes.data, len(rays), C.byref(bad), C.byref(nn), C.byref(visits))
    return rc, bad.value, nn.value, visits.value


def _host_rays(tv, rng, n, extent):
    """Rays along the stacking axis (z) and across it (x), plus random ones, from origins inside the triangles' box or just
    beyond it, all within `extent` of the origin (the scene's and the camera's extent, which the box padding assumes)."""
    p = tv.reshape(-1, 3)
    lo, hi = p.min(0), p.max(0)
    o = rng.uniform(lo, hi, (n, 3)).astype(F)
    o[: n//2, 2] = np.where(rng.rand(n//2) < 0.5, lo[2] - 0.5, hi[2] + 0.5)
    d = _unit(rng.normal(size=(n, 3)))
    d[: n//2] = 0.0; d[: n//2, 2] = np.where(o[: n//2, 2] < lo[2], 1.0, -1.0)                # along the axis, from below / above
    m = slice(n//2, 3*n//4)
    d[m] = 0.0; d[m, 0] = rng.choice([-1.0, 1.0], n//4)                                          # across it, at a triangle's height
    o[m, 0] = np.where(d[m, 0] > 0, lo[0] - 0.5, hi[0] + 0.5)
    o[m, 2] = p[rng.randint(0, len(p), n//4), 2] + rng.choice([0.0, 1e-7, -1e-7], n//4).astype(F)
    o = np.clip(o, -F(extent), F(extent))
    return _pack(o, d.astype(F), tnear=1e-4)


HOST_SHAPES = {"leaf1": (lambda: tetra_faces(1), None), "leaf3": (lambda: tetra_faces(3), None),
               "leaf4": (lambda: tetra_faces(4), None), "deep": (deep_tris, "1"), "stacked": (deep_tris, None)}


@pytest.mark.parametrize("cut", CUTS)
@pytest.mark.parametrize("shape", list(HOST_SHAPES))
def test_host_quantised_walk_equals_brute_force(shape, cut, monkeypatch):
    """The host walk over the quantised tree (tgb200_qbvh_selftest) against brute force over every triangle, bit for bit."""
    make, leaf = HOST_SHAPES[shape]
    _switches(monkeypatch, {"TGB_TRI_LEAF": leaf} if leaf else {}, cut)
    tv = make()
    rays = _host_rays(tv, np.random.RandomState(17), 4000, np.abs(tv).max())     # (the selftest's extent is its rays')
    rc, bad, nodes, visits = qbvh_selftest(tv, rays)
    print("%s, cut %s: %d triangles, %d nodes, %d rays, %d node visits, %d mismatches" % (shape, cut, len(tv), nodes, len(rays), visits, bad))
    assert rc == abi.TGB_OK and bad == 0 and visits >= len(rays)//2
    if shape.startswith("leaf"):
        assert nodes == 1


def deep_miss_queries(rng, n):
    q = stack_axis_rays(rng, n, False)
    q[:, 7] = 400.0                                                                # past the whole stack: nothing blocks them
    return q


@pytest.mark.parametrize("cut", CUTS)
def test_host_deep_walk_spills_the_stack(cut, monkeypatch):
    """The deep scene's any-hit walk from the cut, and its closest-hit walk from the root, go past stack entry 31 on rays that hit
    nothing; both stay within the bound tgb200_create checks, and the two walks agree on visibility.  Measured: with 16 cut boxes the
    walk from the cut reaches 45 entries against a need of 48, with 4 it reaches 33 of 41; the closest-hit walk reaches 33 with
    either (it starts at the root).  With the default leaf cap the same stack stays at or below 32."""
    _switches(monkeypatch, {"TGB_TRI_LEAF": "1"}, cut)
    tv = deep_tris()
    q = np.concatenate([deep_miss_queries(np.random.RandomState(5), 2000), _host_rays(tv, np.random.RandomState(6), 2000,
                                                                                        max(np.abs(tv).max(), np.abs(DEEP_CAM).max()))])
    q[:, 7] = np.where(np.isfinite(q[:, 7]), q[:, 7], 400.0)
    rc, need, out = swc.walk_counts(tv, F(DEEP_CAM), q)
    agree, text = swc.summary(out)
    print(text)
    walked = out[:, 0] != 0
    miss = walked & (out[:, 2] == 0)
    assert rc == abi.TGB_OK and agree and walked.sum() >= 2000 and miss.sum() >= 1000
    n_cut = int(max(bin(int(m)).count("1") for m in out[:, 0]))
    print("deep, cut %s: need %d, cut boxes %d, deepest stack from the cut %d, deepest stack of the closest-hit walk (root, "
          "queries that hit nothing) %d" % (cut, need, n_cut, int(out[walked, 1].max()), int(out[miss, 10].max())))
    assert 32 < out[walked, 1].max() <= need <= 80
    assert 32 < out[miss, 10].max() <= need


@pytest.mark.parametrize("cut", CUTS)
def test_host_too_deep_tree_is_refused(cut, monkeypatch):
    _switches(monkeypatch, {"TGB_TRI_LEAF": "1"}, cut)
    rc, need, _ = swc.walk_counts(too_deep_tris(), F(DEEP_CAM), deep_miss_queries(np.random.RandomState(5), 16))
    print("too_deep, cut %s: need %d" % (cut, need))
    assert rc == abi.TGB_ERR_UNSUPPORTED and need > 80


# ---- GPU ----------------------------------------------------------------------------------------------------------------------
def _info(fs, env, cut, monkeypatch, **override):
    _switches(monkeypatch, dict(env, **override), cut)
    ctx = lib.Context(fs); info = ctx.scene_info(); ctx.close()
    _switches(monkeypatch, env, cut)
    return info


def check_shape(shape, fs, env, cut, info, monkeypatch):
    """The builder branch the scene reaches, from scene_info (see the module's table)."""
    if shape.startswith("leaf"):
        assert info["n_nodes"] == 1 and info["bvh_depth"] == 1 and info["n_tris"] == int(shape[4])
    elif shape == "curves":
        assert info["n_tris"] == 0 and info["n_nodes"] >= 1
    elif shape.startswith("analytic"):
        assert info["n_tris"] == 0 and info["n_nodes"] >= 1
        if shape in ("analytic1", "analytic2"):                        # one leaf; two leaves under the root
            assert info["n_nodes"] == 1 and info["bvh_depth"] == (1 if shape == "analytic1" else 2)
    elif shape in ("tri_analytic", "curves_analytic", "tri_curves_analytic"):
        off = _info(fs, env, cut, monkeypatch, TGB_ANALYTIC_BVH_MIN="100000")
        print("    quads and cubes in the per-ray loop instead: %d nodes, depth %d" % (off["n_nodes"], off["bvh_depth"]))
        if shape == "tri_curves_analytic":                           # the tri + curve root is replaced by the three-way root
            assert info["n_nodes"] > off["n_nodes"] and info["bvh_depth"] >= off["bvh_depth"]
        else:                                                        # a new root over the old tree and the analytic one
            assert info["n_nodes"] >= off["n_nodes"] + 2 and info["bvh_depth"] >= off["bvh_depth"] + 1
        if shape == "curves_analytic":
            assert info["n_tris"] == 0
    elif shape == "deep":
        assert info["n_tris"] == 200 and info["bvh_depth"] >= 11


def _hits(shape, cut, fs, ctx, orc, rays, monkeypatch):
    ref = orc.trace(rays)
    got = ctx.trace_closest(rays)
    monkeypatch.setenv("TGB_HOOK_CUT", "0")
    nocut = ctx.trace_closest(rays)
    monkeypatch.delenv("TGB_HOOK_CUT")
    curves = [i for i, p in enumerate(fs.primitives) if p.type == abi.PRIM_CURVES]
    differ = (got.view(np.uint32).reshape(len(got), -1) != nocut.view(np.uint32).reshape(len(got), -1)).any(1)
    dropped = differ & np.isin(nocut["primitive"], curves) & (got["primitive"] < 0)
    print("    top-level cut on / off: %d rays differ, %d of them curve hits the cut pre-test drops" % (int(differ.sum()), int(dropped.sum())))
    assert not (differ & ~dropped).any(), "the top-level cut changed a hit"
    assert int(dropped.sum()) == CUT_DROPS.get((shape, cut), 0)
    same = (ref["primitive"] == got["primitive"]) & (ref["prim_id"] == got["prim_id"])
    with np.errstate(invalid="ignore"):
        tie = np.abs(ref["t"] - got["t"]) <= 4*np.spacing(np.abs(ref["t"]).astype(F))
    on_curve = np.isin(ref["primitive"], curves) | np.isin(got["primitive"], curves)
    bad = ~same & ~tie
    print("    hits: %d rays, %d hit, identical %.6f, ties %d, curve mismatches %d, other mismatches %d"
          % (len(rays), int((ref["primitive"] >= 0).sum()), same.mean(), int((~same & tie).sum()), int((bad & on_curve).sum()),
             int((bad & ~on_curve).sum())))
    assert (bad & ~on_curve).sum() == 0
    assert int((bad & on_curve).sum()) == CURVE_MISMATCHES.get(shape, 0)
    assert np.array_equal(ref["t"][same], got["t"][same]) and np.array_equal(ref["backside"][same], got["backside"][same])
    both = same & np.isin(ref["primitive"], curves)
    assert np.array_equal(ref["u"][both], got["u"][both]) and np.array_equal(ref["v"][both], got["v"][both])
    return got


def deep_shadow_queries(fs, rng, n):
    """k_shadow_bvh queries along the deep scene's stack (through the corner: they cross every box and no triangle) towards the
    environment light; they are the host count's queries too."""
    q = stack_axis_rays(rng, n, False); q[:, 7] = -1.0
    env = next(i for i, p in enumerate(fs.primitives) if p.type == abi.PRIM_INFINITE_SPHERE)
    lm = np.zeros((n, 2), np.int32); lm[:, 0] = env
    return q, lm


@pytest.mark.gpu
@pytest.mark.parametrize("cut", CUTS)
@pytest.mark.parametrize("shape", SHAPES)
def test_tree_shape_against_oracle(shape, cut, scratch, monkeypatch):
    import test_gpu_shadow as S
    from test_gpu_parity import _compare
    from oracle import pyoracle
    fs, env = build_scene(shape, scratch)
    _switches(monkeypatch, env, cut)
    ctx = lib.Context(fs); orc = pyoracle.Oracle(fs)
    info = ctx.scene_info()
    print("%s, TGB_CUT_BOXES=%s: n_tris %d, n_nodes %d, bvh_depth %d" % (shape, cut, info["n_tris"], info["n_nodes"], info["bvh_depth"]))
    check_shape(shape, fs, env, cut, info, monkeypatch)
    # closest hits
    rays = hit_rays(fs, np.random.RandomState(31), 40000, orc.trace, deep=shape == "deep")
    _hits(shape, cut, fs, ctx, orc, rays, monkeypatch)
    # shadow queries
    q, lm, strata = S.build_queries(fs, ctx, orc, seed=41, n=16384)
    if shape == "deep":
        dq, dlm = deep_shadow_queries(fs, np.random.RandomState(42), 4096)
        q, lm, strata = np.concatenate([q, dq]), np.concatenate([lm, dlm]), np.concatenate([strata, ["along the stack"]*len(dq)])
    g, _ = S.compare(shape, fs, ctx, orc, q, lm, strata)
    monkeypatch.setenv("TGB_SHADOW_CUT_ENTRY", "0")
    root = lib.Context(fs); g0 = S.gpu_probe(root, q, lm); root.close()
    monkeypatch.delenv("TGB_SHADOW_CUT_ENTRY")
    print("    shadow: %d queries, %d reached the BVH pass, identical with the cut entry off: %s"
          % (len(q), int((g[:, 6] == 2).sum()), np.array_equal(g.view(np.uint32), g0.view(np.uint32))))
    assert np.array_equal(g.view(np.uint32), g0.view(np.uint32))
    if info["n_nodes"]:
        assert (g[:, 6] == 2).any()
    if shape == "deep":
        walked = strata == "along the stack"
        assert (g[walked, 6] == 2).all() and (g[walked, 2] == 1).all()           # all of them walked the tree, none blocked
        _switches(monkeypatch, env, cut)
        hq = q[walked].copy(); hq[:, 7] = np.inf                           # the environment light's distance
        rc, need, out = swc.walk_counts(deep_tris(), F(fs.camera.pos), hq)
        print("    deep: need %d, deepest stack of these queries' walk from the cut %d (host count, same tree)"
              % (need, int(out[:, 1].max())))
        assert rc == abi.TGB_OK and 32 < out[:, 1].max() <= need
    ctx.close(); orc.close()
    # image
    if shape in CURVE_SHAPES:
        _compare(fs, 4, frac_ok=0.99, rel_rmse=3e-2, same_ray_count=False)
    else:
        _compare(fs, 4, frac_ok=0.9999, rel_rmse=1e-5, same_ray_count=False)


@pytest.mark.gpu
@pytest.mark.parametrize("cut", CUTS)
def test_too_deep_tree_is_refused(cut, scratch, monkeypatch):
    fs, env = build_scene("too_deep", scratch)
    _switches(monkeypatch, env, cut)
    with pytest.raises(lib.TgbError) as e:
        lib.Context(fs)
    print(e.value)
    assert e.value.code == abi.TGB_ERR_UNSUPPORTED and "exceeds the traversal stack" in str(e.value)


# ---- the local-memory half of the stack, on every walk ----------------------------------------------------------------------
# The deep scene's walks pass stack entry 31, but only on rays that hit nothing, whose answers a wrong local[] entry cannot change.
# The library's smem4 variant (tungsten_b200/build.py CHECKED_VARIANTS, built by build()) keeps four entries per lane in shared
# memory instead of 32, so every walk deeper than four nodes -- the hitting walks of every scene here included -- pushes and pops
# through TravStack::local.  Its hits, shadow queries and images must equal the library's byte for byte.
VARIANT_SCENES = SHAPES + ["cornell_mesh", "materials_env"]


def _variant_scene(name, scratch):
    if name == "cornell_mesh":
        return scene.load_scene(synth.cornell_mesh(scratch, res=(32, 32), spp=4, subdiv=3)), {}
    if name == "materials_env":
        return scene.load_scene(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name, "scene.json")), {}
    return build_scene(name, scratch)


def _outputs(fs, rays, q, lm):
    import test_gpu_shadow as S
    ctx = lib.Context(fs)
    hits = ctx.trace_closest(rays)
    probe = S.gpu_probe(ctx, q, lm)
    img, cnt = ctx.render_tiles(4)
    ctx.close()
    return {"hits": hits.view(np.uint8), "probe": probe.view(np.uint32), "img": img.view(np.uint32), "cnt": cnt}


def _variant_main(work, scratch):
    """Run in a process that loaded the variant library (TGB200_LIB): outputs of every scene in `work` next to its inputs."""
    print("library: %s" % lib.LIB_PATH)
    for name in VARIANT_SCENES:
        fs, env = _variant_scene(name, scratch)
        for k in BVH_SWITCHES:
            os.environ.pop(k, None)
        os.environ.update(env)
        z = np.load(os.path.join(work, name + ".in.npz"))
        np.savez(os.path.join(work, name + ".out.npz"), **_outputs(fs, z["rays"], z["q"], z["lm"]))


@pytest.mark.gpu
def test_local_memory_stack_gives_the_same_answers(scratch, tmp_path, monkeypatch):
    import subprocess
    import test_gpu_shadow as S
    from oracle import pyoracle
    from tungsten_b200 import build
    variant = build.variant_path("smem4")
    assert os.path.exists(variant), "build() makes %s" % variant
    here = os.path.dirname(os.path.abspath(__file__))
    mine = {}
    for name in VARIANT_SCENES:
        fs, env = _variant_scene(name, scratch)
        _switches(monkeypatch, env, "16")
        orc = pyoracle.Oracle(fs); ctx = lib.Context(fs)
        rays = hit_rays(fs, np.random.RandomState(51), 20000, orc.trace, deep=name == "deep")
        q, lm, _ = S.build_queries(fs, ctx, orc, seed=52, n=8192)
        ctx.close(); orc.close()
        np.savez(str(tmp_path/(name + ".in.npz")), rays=rays, q=q, lm=lm)
        mine[name] = _outputs(fs, rays, q, lm)
    monkeypatch.delenv("TGB_CUT_BOXES")
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_gpu_tree_shapes as T; T._variant_main(%r, %r)"
            % (here, os.path.dirname(here), str(tmp_path), scratch))
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, TGB200_LIB=variant), stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=600)
    print(r.stdout[-2000:])
    assert r.returncode == 0 and ("library: %s" % variant) in r.stdout
    for name in VARIANT_SCENES:
        theirs = np.load(str(tmp_path/(name + ".out.npz")))
        same = {k: np.array_equal(mine[name][k], theirs[k]) for k in mine[name]}
        print("%-20s smem4 == library: %s" % (name, same))
        assert all(same.values()), name
