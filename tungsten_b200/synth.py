"""Procedural scenes in Tungsten's own JSON + .wo3 formats.

BASELINE.json's configs name assets that are not in the reference repository (Stanford dragon,
"living-room", a 10M-triangle forest) and there is no network, so the bench and the parity tests
synthesise stand-ins of the stated size and material mix.  Everything is written as ordinary scene
files so that the reference binary (oracle/_ref), the CPU restatement and the CUDA path all load
exactly the same inputs.  Deterministic: no RNG state outside the explicit seeds.
"""
import json
import os

import numpy as np

from .scene import VERTEX_DTYPE, TRI_DTYPE, save_wo3


# ---- meshes -----------------------------------------------------------------------------------
def icosphere(subdiv, radius=1.0, displace=0.0, seed=1, lobes=0.0):
    """Unit icosahedron subdivided `subdiv` times (20*4^subdiv triangles), optional smooth
    deterministic displacement so that the surface is not a trivial sphere."""
    t = (1.0 + 5.0**0.5)/2.0
    v = np.array([[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
                  [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], dtype=np.float64)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    f = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2],
                  [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5],
                  [2, 4, 11], [6, 2, 10], [8, 6, 7], [9, 8, 1]], dtype=np.int64)
    for _ in range(subdiv):
        e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]], axis=0)
        es = np.sort(e, axis=1)
        key = es[:, 0]*(len(v) + 1) + es[:, 1]
        uniq, inv = np.unique(key, return_inverse=True)
        first = np.zeros(len(uniq), dtype=np.int64); first[inv] = np.arange(len(key))
        mid = v[es[first, 0]] + v[es[first, 1]]
        mid /= np.linalg.norm(mid, axis=1, keepdims=True)
        base = len(v)
        v = np.concatenate([v, mid], axis=0)
        n = len(f)
        m01, m12, m20 = base + inv[:n], base + inv[n:2*n], base + inv[2*n:]
        f = np.concatenate([np.stack([f[:, 0], m01, m20], 1), np.stack([f[:, 1], m12, m01], 1),
                            np.stack([f[:, 2], m20, m12], 1), np.stack([m01, m12, m20], 1)], axis=0)
    r = np.ones(len(v))
    if displace > 0.0:
        rng = np.random.RandomState(seed)
        for k in range(6):
            d = rng.normal(size=3); d /= np.linalg.norm(d)
            freq = 2.0 + 3.0*k
            r += displace/(k + 1)*np.sin(freq*(v @ d) + rng.uniform(0, 6.28))
    if lobes > 0.0:
        r += lobes*np.cos(3.0*np.arctan2(v[:, 2], v[:, 0]))*np.sin(2.0*np.arccos(np.clip(v[:, 1], -1, 1)))
    p = v*(r*radius)[:, None]
    # smooth normals from area-weighted face normals
    fn = np.cross(p[f[:, 1]] - p[f[:, 0]], p[f[:, 2]] - p[f[:, 0]])
    nrm = np.zeros_like(p)
    for k in range(3):
        np.add.at(nrm, f[:, k], fn)
    nrm /= np.maximum(np.linalg.norm(nrm, axis=1, keepdims=True), 1e-20)
    verts = np.zeros(len(p), dtype=VERTEX_DTYPE)
    verts["pos"] = p.astype(np.float32); verts["normal"] = nrm.astype(np.float32)
    verts["uv"][:, 0] = (np.arctan2(v[:, 2], v[:, 0])/(2*np.pi) + 0.5).astype(np.float32)
    verts["uv"][:, 1] = (np.arccos(np.clip(v[:, 1], -1, 1))/np.pi).astype(np.float32)
    tris = np.zeros(len(f), dtype=TRI_DTYPE)
    tris["v0"], tris["v1"], tris["v2"] = f[:, 0], f[:, 1], f[:, 2]
    return verts, tris


def grid_mesh(nx, nz, size=1.0, height=0.0, seed=3):
    """(nx x nz) quads -> 2*nx*nz triangles in the XZ plane, optional height field."""
    xs = np.linspace(-0.5, 0.5, nx + 1)*size; zs = np.linspace(-0.5, 0.5, nz + 1)*size
    X, Z = np.meshgrid(xs, zs, indexing="xy")
    Y = np.zeros_like(X)
    if height > 0.0:
        rng = np.random.RandomState(seed)
        for k in range(4):
            a, b = rng.uniform(2, 9, 2); ph = rng.uniform(0, 6.28, 2)
            Y += height/(k + 1)*np.sin(a*X/size*6.28 + ph[0])*np.cos(b*Z/size*6.28 + ph[1])
    verts = np.zeros(X.size, dtype=VERTEX_DTYPE)
    verts["pos"] = np.stack([X.ravel(), Y.ravel(), Z.ravel()], 1).astype(np.float32)
    verts["normal"][:, 1] = 1.0
    verts["uv"] = np.stack([(X.ravel()/size + 0.5), (Z.ravel()/size + 0.5)], 1).astype(np.float32)
    i = np.arange(nx)[None, :] + (nx + 1)*np.arange(nz)[:, None]
    i = i.ravel()
    tris = np.zeros(2*nx*nz, dtype=TRI_DTYPE)
    tris["v0"][0::2], tris["v1"][0::2], tris["v2"][0::2] = i, i + nx + 1, i + 1
    tris["v0"][1::2], tris["v1"][1::2], tris["v2"][1::2] = i + 1, i + nx + 1, i + nx + 2
    return verts, tris


# ---- scenes -----------------------------------------------------------------------------------
def _lambert(name, albedo):
    return {"name": name, "albedo": albedo, "type": "lambert"}


def _renderer(spp):
    return {"output_file": "out.png", "hdr_output_file": "out.pfm", "overwrite_output_files": True,
            "adaptive_sampling": False, "enable_resume_render": False, "stratified_sampler": True,
            "scene_bvh": True, "spp": spp, "spp_step": spp}


def cornell_box(res=(128, 128), spp=16, max_bounces=64, extra_bsdfs=(), extra_prims=(), boxes=True,
                light_emission=(17, 12, 4), filter_name="tent"):
    """The classic Cornell box laid out with Tungsten primitives: 5 wall quads, 2 cubes, 1 quad light
    (same construction as the reference's data/example-scenes/cornell-box, dimensions are the
    well-known Cornell measurements rescaled to a 2-unit box)."""
    white = [0.725, 0.71, 0.68]
    bsdfs = [_lambert("leftWall", [0.63, 0.065, 0.05]), _lambert("rightWall", [0.14, 0.45, 0.091]),
             _lambert("floor", white), _lambert("ceiling", white), _lambert("backWall", white),
             _lambert("shortBox", white), _lambert("tallBox", white),
             {"name": "light", "albedo": 1, "type": "null"}] + list(extra_bsdfs)
    def quad(name, pos, rot, scale=(2, 4, 2), **kw):
        d = {"name": name, "transform": {"position": list(pos), "scale": list(scale), "rotation": list(rot)},
             "type": "quad", "bsdf": name}
        d.update(kw); return d
    prims = [quad("floor", (0, 0, 0), (0, 90, 0)), quad("ceiling", (0, 2, 0), (0, 0, -180)),
             quad("backWall", (0, 1, -1), (0, 90, 90)), quad("rightWall", (1, 1, 0), (0, 180, 90)),
             quad("leftWall", (-1, 1, 0), (0, 0, 90))]
    if boxes:
        prims += [{"name": "shortBox", "type": "cube", "bsdf": "shortBox",
                   "transform": {"position": [0.328631, 0.3, 0.374592], "scale": [0.594811, 0.604394, 0.6],
                                 "rotation": [90, 90, -163.36]}},
                  {"name": "tallBox", "type": "cube", "bsdf": "tallBox",
                   "transform": {"position": [-0.335439, 0.6, -0.291415], "scale": [0.607289, 0.597739, 1.2],
                                 "rotation": [90, 180, 160.812]}}]
    prims += [quad("light", (-0.005, 1.98, -0.03), (0, 180, 180), scale=(0.47, 0.1786, 0.38),
                   emission=list(light_emission))]
    prims += list(extra_prims)
    return {"media": [], "bsdfs": bsdfs, "primitives": prims,
            "camera": {"tonemap": "filmic", "resolution": list(res), "reconstruction_filter": filter_name,
                       "transform": {"position": [0, 1, 6.8], "look_at": [0, 1, 0], "up": [0, 1, 0]},
                       "type": "pinhole", "fov": 35},
            "integrator": {"type": "path_tracer", "min_bounces": 0, "max_bounces": max_bounces,
                           "enable_consistency_checks": False, "enable_two_sided_shading": True,
                           "enable_light_sampling": True},
            "renderer": _renderer(spp)}


def write_scene(out_dir, name, scene, meshes=None):
    """Write <out_dir>/<name>.json (+ .wo3 files named by `meshes`: {filename: (verts, tris)})."""
    os.makedirs(out_dir, exist_ok=True)
    for fn, (v, t) in (meshes or {}).items():
        save_wo3(os.path.join(out_dir, fn), v, t)
    path = os.path.join(out_dir, name + ".json")
    with open(path, "w") as f:
        json.dump(scene, f, indent=1)
    return path


def cornell_mesh(out_dir, name="cornell_mesh", subdiv=3, res=(128, 128), spp=16, max_bounces=64,
                 bsdf=None, smooth=True, displace=0.15):
    """Cornell box (no cubes) + one displaced-icosphere mesh: the C1 stand-in (subdiv 7 -> 327,680 and
    subdiv 8 -> 1,310,720 triangles; the bench uses ~870k via two meshes)."""
    v, t = icosphere(subdiv, 1.0, displace=displace)
    b = bsdf or _lambert("blob", [0.6, 0.55, 0.7])
    b = dict(b); b["name"] = "blob"
    prim = {"name": "blob", "type": "mesh", "file": name + "_blob.wo3", "smooth": smooth, "bsdf": "blob",
            "transform": {"position": [0.0, 0.72, 0.0], "scale": [0.62, 0.62, 0.62], "rotation": [0, 30, 0]}}
    sc = cornell_box(res, spp, max_bounces, extra_bsdfs=[b], extra_prims=[prim], boxes=False)
    return write_scene(out_dir, name, sc, {name + "_blob.wo3": (v, t)})


def dirac_room(out_dir, name="dirac", res=(128, 128), spp=16, max_bounces=16, subdiv=3):
    """Cornell box whose boxes are a mirror (MirrorBsdf) and a smooth conductor (ConductorBsdf, gold), plus a smooth dielectric
    ball (DielectricBsdf, ior 1.5, refraction on) and a reflect-only dielectric blob: the Dirac lobes of f4."""
    v, t = icosphere(subdiv, 1.0)
    bs = [{"name": "glass", "type": "dielectric", "ior": 1.5, "albedo": 1.0},
          {"name": "lacquer", "type": "dielectric", "ior": 1.8, "enable_refraction": False, "albedo": [0.9, 0.95, 1.0]}]
    prims = [{"name": "ball", "type": "mesh", "file": name + "_ball.wo3", "smooth": True, "bsdf": "glass",
              "transform": {"position": [0.35, 0.95, 0.45], "scale": [0.3, 0.3, 0.3]}},
             {"name": "blob", "type": "mesh", "file": name + "_ball.wo3", "smooth": True, "bsdf": "lacquer",
              "transform": {"position": [-0.55, 0.3, 0.55], "scale": [0.28, 0.28, 0.28]}}]
    sc = cornell_box(res, spp, max_bounces, extra_bsdfs=bs, extra_prims=prims)
    for b in sc["bsdfs"]:
        if b["name"] == "shortBox":
            b.clear(); b.update({"name": "shortBox", "type": "mirror", "albedo": [0.95, 0.95, 0.95]})
        if b["name"] == "tallBox":
            b.clear(); b.update({"name": "tallBox", "type": "conductor", "material": "Au", "albedo": 1.0})
    return write_scene(out_dir, name, sc, {name + "_ball.wo3": (v, t)})


def cornell_dragon_standin(out_dir, name="cornell_dragon", res=(1920, 1080), spp=1024, max_bounces=64):
    """BASELINE.json config C1: Cornell box + ~870k-triangle Lambert mesh.  The Stanford dragon is not in
    the reference repository; the stand-in is a lobed, displaced icosphere at subdivision 7 (327,680
    triangles) plus a 520x520 height-field "plinth" (540,800 triangles): 868,480 triangles."""
    v, t = icosphere(7, 1.0, displace=0.22, lobes=0.25)
    gv, gt = grid_mesh(520, 520, 1.0, height=0.03)
    bs = [_lambert("dragon", [0.55, 0.62, 0.45]), _lambert("plinth", [0.7, 0.6, 0.5])]
    prims = [{"name": "dragon", "type": "mesh", "file": name + "_body.wo3", "smooth": True, "bsdf": "dragon",
              "transform": {"position": [0.0, 0.85, -0.05], "scale": [0.55, 0.55, 0.55], "rotation": [0, 25, 0]}},
             {"name": "plinth", "type": "mesh", "file": name + "_plinth.wo3", "smooth": False, "bsdf": "plinth",
              "transform": {"position": [0.0, 0.12, 0.0], "scale": [1.5, 1.0, 1.5]}}]
    sc = cornell_box(res, spp, max_bounces, extra_bsdfs=bs, extra_prims=prims, boxes=False)
    return write_scene(out_dir, name, sc, {name + "_body.wo3": (v, t), name + "_plinth.wo3": (gv, gt)})


def material_room(out_dir, name="materials", res=(128, 128), spp=16, max_bounces=16, subdiv=3, env=None):
    """Cornell-like room with one blob per in-scope lobe model (rough conductor / rough dielectric /
    plastic / rough plastic), a checker floor and a second (mesh) light: exercises chooseLight with
    several lights, mesh-light NEE, textured albedo and every BSDF on the path."""
    bsdfs = [
        {"name": "metal", "type": "rough_conductor", "albedo": 1.0, "material": "Cu", "distribution": "ggx", "roughness": 0.25},
        {"name": "glass", "type": "rough_dielectric", "albedo": 1.0, "ior": 1.5, "distribution": "ggx", "roughness": 0.15},
        {"name": "plast", "type": "plastic", "albedo": [0.2, 0.4, 0.8], "ior": 1.5, "thickness": 1.0, "sigma_a": [0.0, 0.0, 0.0]},
        {"name": "rplast", "type": "rough_plastic", "albedo": [0.8, 0.3, 0.2], "ior": 1.4, "thickness": 1.0,
         "sigma_a": [0.1, 0.2, 0.3], "distribution": "beckmann", "roughness": 0.3},
        {"name": "checker", "type": "lambert", "albedo": {"type": "checker", "on_color": [0.8, 0.8, 0.8],
                                                         "off_color": [0.15, 0.15, 0.2], "res_u": 8, "res_v": 8}},
        {"name": "lamp", "type": "null", "albedo": 1.0},
    ]
    v, t = icosphere(subdiv, 1.0, displace=0.1)
    lv, lt = grid_mesh(2, 2, 1.0)
    meshes = {name + "_blob.wo3": (v, t), name + "_lamp.wo3": (lv, lt)}
    def blob(nm, bsdf, pos, s=0.28):
        return {"name": nm, "type": "mesh", "file": name + "_blob.wo3", "smooth": True, "bsdf": bsdf,
                "transform": {"position": list(pos), "scale": [s, s, s]}}
    prims = [blob("b0", "metal", (-0.55, 0.32, 0.2)), blob("b1", "glass", (0.0, 0.95, 0.3), 0.3),
             blob("b2", "plast", (0.55, 0.32, 0.2)), blob("b3", "rplast", (0.0, 0.3, -0.45)),
             {"name": "floor2", "type": "quad", "bsdf": "checker",
              "transform": {"position": [0, 0.002, 0], "scale": [1.9, 1, 1.9]}},
             {"name": "lamp", "type": "mesh", "file": name + "_lamp.wo3", "smooth": False, "bsdf": "lamp",
              "emission": [6.0, 7.0, 9.0],
              "transform": {"position": [0.6, 1.3, -0.95], "scale": [0.5, 0.5, 0.5], "rotation": [90, 0, 0]}}]
    sc = cornell_box(res, spp, max_bounces, extra_bsdfs=bsdfs, extra_prims=prims, boxes=False)
    if env is not None:
        sc["primitives"].append({"name": "env", "type": "infinite_sphere", "emission": env, "sample": True,
                                 "transform": {"rotation": [0, 40, 0]}})
    return write_scene(out_dir, name, sc, meshes)


def coat_room(out_dir, name="coats", res=(128, 128), spp=16, max_bounces=16, subdiv=3):
    """RoughCoatBsdf three ways -- Beckmann coat with absorption over Lambert, GGX coat over a rough conductor, GGX coat over
    plastic -- on two blobs and a cube, plus a SmoothCoatBsdf blob for comparison.  The substrates are NAMED bsdfs of the scene:
    the reference prepares (prepareForRender) only the bsdfs in its scene list, an inline substrate object never is."""
    v, t = icosphere(subdiv, 1.0, displace=0.08)
    meshes = {name + "_blob.wo3": (v, t)}
    bsdfs = [
        {"name": "subLambert", "type": "lambert", "albedo": [0.6, 0.3, 0.2]},
        {"name": "subMetal", "type": "rough_conductor", "material": "Au", "distribution": "beckmann", "roughness": 0.3},
        {"name": "subPlastic", "type": "plastic", "albedo": [0.2, 0.5, 0.7], "ior": 1.5},
        {"name": "coatA", "type": "rough_coat", "distribution": "beckmann", "roughness": 0.25, "ior": 1.5, "thickness": 2.0,
         "sigma_a": [0.2, 0.1, 0.4], "substrate": "subLambert"},
        {"name": "coatB", "type": "rough_coat", "distribution": "ggx", "roughness": 0.1, "ior": 1.4, "substrate": "subMetal"},
        {"name": "coatC", "type": "rough_coat", "roughness": 0.15, "ior": 1.6, "substrate": "subPlastic"},
        {"name": "coatS", "type": "smooth_coat", "ior": 1.5, "thickness": 1.0, "sigma_a": [0.3, 0.3, 0.1], "substrate": "subMetal"},
    ]
    def blob(nm, bsdf, pos, s=0.3):
        return {"name": nm, "type": "mesh", "file": name + "_blob.wo3", "smooth": True, "bsdf": bsdf,
                "transform": {"position": list(pos), "scale": [s, s, s]}}
    prims = [blob("b0", "coatA", (-0.5, 0.32, 0.25)), blob("b1", "coatB", (0.5, 0.32, 0.25)), blob("b2", "coatS", (0.0, 1.05, -0.2), 0.28),
             {"name": "c0", "type": "cube", "bsdf": "coatC",
              "transform": {"position": [0.0, 0.25, -0.45], "scale": [0.5, 0.5, 0.5], "rotation": [0, 25, 0]}}]
    sc = cornell_box(res, spp, max_bounces, extra_bsdfs=bsdfs, extra_prims=prims, boxes=False)
    return write_scene(out_dir, name, sc, meshes)


def many_lights(out_dir, name="many_lights", n_quads=36, res=(128, 128), spp=16, max_bounces=16, subdiv=3):
    """Cornell room + blob lit by the ceiling light, a 6 x 6 grid of small coloured quad lights under the ceiling and two mesh
    lights (whose approximate radiance is "unknown" in TraceBase::chooseLight): 39 samplable lights.  The reference keeps
    one pdf per light in a vector of any length; this scene pins the device's > 16 lights path."""
    v, t = icosphere(subdiv, 1.0, displace=0.12)
    lv, lt = grid_mesh(2, 2, 1.0)
    meshes = {name + "_blob.wo3": (v, t), name + "_lamp.wo3": (lv, lt)}
    bsdfs = [_lambert("blob", [0.6, 0.55, 0.7]), {"name": "lamp", "type": "null", "albedo": 1.0}]
    prims = [{"name": "blob", "type": "mesh", "file": name + "_blob.wo3", "smooth": True, "bsdf": "blob",
              "transform": {"position": [0.0, 0.6, 0.0], "scale": [0.5, 0.5, 0.5], "rotation": [0, 30, 0]}}]
    side = int(round(n_quads**0.5))
    for k in range(n_quads):
        i, j = k % side, k//side
        x, z = -0.8 + 1.6*i/max(side - 1, 1), -0.8 + 1.6*j/max(side - 1, 1)
        em = [1.5 + 4.0*((k*7) % 5)/4.0, 1.5 + 4.0*((k*3) % 4)/3.0, 1.5 + 4.0*((k*5) % 3)/2.0]
        prims.append({"name": "q%d" % k, "type": "quad", "bsdf": "lamp", "emission": em,
                      "transform": {"position": [x, 1.9 - 0.01*(k % 3), z], "scale": [0.09, 1, 0.07], "rotation": [0, 17.0*k, 180]}})
    for k, (pos, rot) in enumerate([((0.93, 1.0, -0.3), (0, 0, 90)), ((-0.93, 0.7, 0.2), (0, 0, -90))]):
        prims.append({"name": "m%d" % k, "type": "mesh", "file": name + "_lamp.wo3", "smooth": False, "bsdf": "lamp",
                      "emission": [3.0 + 2*k, 4.0, 6.0 - 2*k],
                      "transform": {"position": list(pos), "scale": [0.3, 0.3, 0.3], "rotation": list(rot)}})
    sc = cornell_box(res, spp, max_bounces, extra_bsdfs=bsdfs, extra_prims=prims, boxes=False, light_emission=(8, 6, 2))
    return write_scene(out_dir, name, sc, meshes)


def cube_city(out_dir=None, name="cube_city", n=12, res=(128, 128), spp=16, max_bounces=8, seed=7, n_lights=6):
    """A floor, n x n rotated cubes of random height and colour and a few quad lights: hundreds of ANALYTIC primitives and no
    mesh at all.  The reference keeps such primitives in Embree's top-level user-geometry BVH (TraceableScene.hpp:112-134);
    the library moves them from its per-ray loop into BVH leaves from 24 primitives on."""
    rng = np.random.RandomState(seed)
    bsdfs = [_lambert("floor", [0.5, 0.5, 0.5]), {"name": "lamp", "type": "null", "albedo": 1.0}]
    prims = [{"name": "floor", "type": "quad", "bsdf": "floor", "transform": {"position": [0, 0, 0], "scale": [12, 1, 12]}}]
    for k in range(n*n):
        i, j = k % n, k//n
        col = [float(c) for c in 0.2 + 0.7*rng.rand(3)]
        bsdfs.append(_lambert("c%d" % k, col))
        h = float(0.2 + 1.3*rng.rand())
        x, z = -4.5 + 9.0*(i + 0.5)/n, -4.5 + 9.0*(j + 0.5)/n
        prims.append({"name": "c%d" % k, "type": "cube", "bsdf": "c%d" % k,
                      "transform": {"position": [x, 0.5*h, z], "scale": [0.55*9.0/n, h, 0.55*9.0/n], "rotation": [0, float(90*rng.rand()), 0]}})
    for k in range(n_lights):
        ang = 2*np.pi*k/n_lights
        prims.append({"name": "l%d" % k, "type": "quad", "bsdf": "lamp", "emission": [20.0 + 5*k, 18.0, 25.0 - 3*k],
                      "transform": {"position": [float(3.5*np.cos(ang)), 3.2 + 0.1*k, float(3.5*np.sin(ang))], "scale": [0.8, 1, 0.6],
                                    "rotation": [0, float(30*k), 180]}})
    sc = {"media": [], "bsdfs": bsdfs, "primitives": prims,
          "camera": {"tonemap": "filmic", "resolution": list(res), "reconstruction_filter": "tent",
                     "transform": {"position": [7.5, 5.0, 9.0], "look_at": [0, 0.6, 0], "up": [0, 1, 0]}, "type": "pinhole", "fov": 40},
          "integrator": {"type": "path_tracer", "min_bounces": 0, "max_bounces": max_bounces, "enable_consistency_checks": False,
                         "enable_two_sided_shading": True, "enable_light_sampling": True},
          "renderer": _renderer(spp)}
    if out_dir is None:
        return sc
    return write_scene(out_dir, name, sc)


def flush_lights(out_dir, name="flush_lights", res=(64, 64), spp=16, max_bounces=8):
    """Cornell box with lights flush with a blocker, so that a shadow query finds a blocker at exactly the light's distance: a
    table-top quad at y = 0.8 with two quad lights in its plane, one listed before the table and one after it, and a mesh shelf at
    y = 1.4 with a mesh light in its plane.  All of them are unrotated (normal +y), so each pair's plane is the same float32 plane
    and the hits of a ray on both are bit-identical ties."""
    sv, st = grid_mesh(4, 4, 1.0)
    lv, lt = grid_mesh(2, 2, 1.0)
    meshes = {name + "_shelf.wo3": (sv, st), name + "_lamp.wo3": (lv, lt)}
    bsdfs = [_lambert("table", [0.5, 0.45, 0.4]), {"name": "lamp", "type": "null", "albedo": 1.0}]

    def flat(nm, bsdf, pos, scale, **kw):
        d = {"name": nm, "type": "quad", "bsdf": bsdf, "transform": {"position": list(pos), "scale": list(scale)}}
        d.update(kw); return d
    prims = [flat("table", "table", (0.0, 0.8, 0.3), (1.2, 1, 1.0)),
             flat("flush_after", "lamp", (0.3, 0.8, 0.35), (0.25, 1, 0.3), emission=[6.0, 5.0, 3.0]),
             {"name": "shelf", "type": "mesh", "file": name + "_shelf.wo3", "smooth": False, "bsdf": "table",
              "transform": {"position": [0.45, 1.4, -0.5], "scale": [0.8, 1.0, 0.6]}},
             {"name": "mesh_lamp", "type": "mesh", "file": name + "_lamp.wo3", "smooth": False, "bsdf": "lamp",
              "emission": [3.0, 4.0, 6.0], "transform": {"position": [0.45, 1.4, -0.5], "scale": [0.3, 1.0, 0.3]}}]
    sc = cornell_box(res, spp, max_bounces, extra_bsdfs=bsdfs, extra_prims=prims, light_emission=(8, 6, 2))
    sc["primitives"].insert(0, flat("flush_before", "lamp", (-0.25, 0.8, 0.3), (0.3, 1, 0.25), emission=[4.0, 6.0, 5.0]))
    return write_scene(out_dir, name, sc, meshes)


# ---- HDR environment maps ----------------------------------------------------------------------
def save_rgbe(path, img):
    """Flat (non-RLE) Radiance .hdr writer; rows top-down ("-Y h +X w")."""
    img = np.asarray(img, dtype=np.float64)
    h, w, _ = img.shape
    m = img.max(axis=2)
    e = np.zeros((h, w), dtype=np.int32)
    nz = m > 1e-32
    mant, ex = np.frexp(np.where(nz, m, 1.0))
    scale = np.where(nz, mant*256.0/np.where(nz, m, 1.0), 0.0)
    rgbe = np.zeros((h, w, 4), dtype=np.uint8)
    rgbe[..., :3] = np.clip(img*scale[..., None], 0, 255).astype(np.uint8)
    rgbe[..., 3] = np.where(nz, ex + 128, 0).astype(np.uint8)
    with open(path, "wb") as f:
        f.write(b"#?RADIANCE\nFORMAT=32-bit_rle_rgbe\n\n-Y %d +X %d\n" % (h, w))
        f.write(rgbe.tobytes())


def sky_envmap(w=128, h=64, sun=(0.62, 0.35), sun_power=60.0):
    """Procedural lat-long sky: gradient + a small bright sun + a darker ground, strong enough contrast that
    the importance map (BitmapTexture::makeSamplable) matters."""
    v = (np.arange(h) + 0.5)/h
    u = (np.arange(w) + 0.5)/w
    U, V = np.meshgrid(u, v)
    up = np.cos(V*np.pi)                     # +1 at the top row
    sky = np.stack([0.25 + 0.35*np.clip(up, 0, 1), 0.35 + 0.45*np.clip(up, 0, 1), 0.6 + 0.5*np.clip(up, 0, 1)], axis=2)
    ground = np.stack([0.12 + 0*up, 0.10 + 0*up, 0.08 + 0*up], axis=2)
    img = np.where((up > 0)[..., None], sky, ground)
    d2 = ((U - sun[0])*2.0)**2 + (V - sun[1])**2
    img = img + sun_power*np.exp(-d2/0.0012)[..., None]*np.array([1.0, 0.9, 0.7])
    return img.astype(np.float32)


def materialtest_standin(out_dir, name="coat_env", res=(128, 128), spp=16, max_bounces=64, subdiv=3, env_res=(128, 64)):
    """Stand-in for BASELINE.json config C0 (data/materialtest/materialtest.json): a smooth_coat(ior 1.7, absorbing)
    over a Beckmann rough_conductor(Cu) blob, a Lambert stand, a checker-textured Lambert floor quad and an HDR
    environment map lit through importance sampling -- the same lobe / emitter / texture mix, with procedural assets."""
    v, t = icosphere(subdiv, 1.0, displace=0.12, lobes=0.2)
    sv, st = icosphere(max(subdiv - 1, 0), 1.0)
    os.makedirs(out_dir, exist_ok=True)
    save_rgbe(os.path.join(out_dir, name + "_env.hdr"), sky_envmap(*env_res))
    bsdfs = [
        {"name": "rough_metal", "albedo": 1, "type": "rough_conductor", "material": "Cu", "distribution": "beckmann", "roughness": 0.1},
        {"name": "Material", "albedo": 1, "type": "smooth_coat", "ior": 1.7, "thickness": 5, "sigma_a": [0.1, 0.2, 0.5], "substrate": "rough_metal"},
        {"name": "Stand", "albedo": 0.2, "type": "lambert"},
        {"name": "Floor", "type": "lambert", "albedo": {"type": "checker", "on_color": [0.725, 0.71, 0.68],
                                                        "off_color": [0.325, 0.31, 0.25], "res_u": 20, "res_v": 20}},
    ]
    prims = [
        {"name": "Floor", "type": "quad", "bsdf": "Floor", "transform": {"position": [-0.7, 0, -0.7], "scale": 5.4, "rotation": [0, 46.15, 180]}},
        {"name": "Envmap", "type": "infinite_sphere", "emission": name + "_env.hdr", "sample": True,
         "transform": {"rotation": [0, -67.26, 0]}},
        {"name": "Ball", "type": "mesh", "file": name + "_ball.wo3", "smooth": True, "bsdf": "Material",
         "transform": {"position": [0.15, 0.78, 0.16], "scale": 0.45}},
        {"name": "Stand", "type": "mesh", "file": name + "_stand.wo3", "smooth": True, "bsdf": "Stand",
         "transform": {"position": [0.12, 0.2, 0.13], "scale": [0.3, 0.2, 0.3]}},
    ]
    sc = {"media": [], "bsdfs": bsdfs, "primitives": prims,
          "camera": {"tonemap": "filmic", "resolution": list(res), "reconstruction_filter": "tent",
                     "transform": {"position": [3.04, 3.17, 3.2], "look_at": [0.12, 0.47, 0.16], "up": [0, 1, 0]},
                     "type": "pinhole", "fov": 35},
          "integrator": {"type": "path_tracer", "min_bounces": 0, "max_bounces": max_bounces, "enable_light_sampling": True,
                         "enable_consistency_checks": False, "enable_two_sided_shading": True},
          "renderer": _renderer(spp)}
    return write_scene(out_dir, name, sc, {name + "_ball.wo3": (v, t), name + "_stand.wo3": (sv, st)})


def instanced_forest(out_dir, name="forest", n_instances=64, tree_subdiv=2, res=(128, 128), spp=16, max_bounces=16, seed=5,
                     extent=6.0):
    """Stand-in for BASELINE.json config C3: a few tree-like masters (trunk + crown blobs) scattered as rigid instances
    (rotation about Y + translation, no scale -- `Instance` cannot scale) over a ground quad, Lambert + rough plastic,
    sky environment.  tree_subdiv 4 -> 10,240-triangle masters: 1,000 instances = 10.2 M triangles."""
    rng = np.random.RandomState(seed)
    crown_v, crown_t = icosphere(tree_subdiv, 1.0, displace=0.25, seed=7)
    trunk_v, trunk_t = icosphere(max(tree_subdiv - 1, 0), 1.0)
    os.makedirs(out_dir, exist_ok=True)
    save_rgbe(os.path.join(out_dir, name + "_env.hdr"), sky_envmap(64, 32, sun_power=25.0))
    bsdfs = [{"name": "leaf", "type": "rough_plastic", "albedo": [0.15, 0.45, 0.12], "ior": 1.5, "distribution": "ggx", "roughness": 0.25},
             {"name": "bark", "type": "lambert", "albedo": [0.35, 0.22, 0.12]},
             {"name": "ground", "type": "lambert", "albedo": {"type": "checker", "on_color": [0.45, 0.4, 0.3], "off_color": [0.3, 0.32, 0.2], "res_u": 24, "res_v": 24}}]
    masters = [{"type": "mesh", "file": name + "_crown.wo3", "smooth": True, "bsdf": "leaf",
                "transform": {"position": [0, 1.1, 0], "scale": [0.55, 0.8, 0.55]}},
               {"type": "mesh", "file": name + "_trunk.wo3", "smooth": True, "bsdf": "bark",
                "transform": {"position": [0, 0.3, 0], "scale": [0.09, 0.35, 0.09]}}]
    inst = []
    for i in range(n_instances):
        x, z = rng.uniform(-extent/2, extent/2, 2)
        ang = float(rng.uniform(0, 360))
        for mid in (0, 1):
            inst.append({"id": mid, "transform": {"position": [float(x), 0.0, float(z)], "rotation": [0, ang, 0]}})
    prims = [{"name": "ground", "type": "quad", "bsdf": "ground", "transform": {"scale": [extent*1.6, 1, extent*1.6]}},
             {"name": "forest", "type": "instances", "masters": masters, "instances": inst, "bsdf": "ground",
              "transform": {"position": [0, 0, 0], "rotation": [0, 15, 0]}},
             {"name": "sky", "type": "infinite_sphere", "emission": name + "_env.hdr", "sample": True}]
    sc = {"media": [], "bsdfs": bsdfs, "primitives": prims,
          "camera": {"tonemap": "filmic", "resolution": list(res), "reconstruction_filter": "tent",
                     "transform": {"position": [0.0, 2.6, extent*0.95], "look_at": [0, 0.6, 0], "up": [0, 1, 0]}, "type": "pinhole", "fov": 40},
          "integrator": {"type": "path_tracer", "min_bounces": 0, "max_bounces": max_bounces, "enable_light_sampling": True,
                         "enable_consistency_checks": False, "enable_two_sided_shading": True},
          "renderer": _renderer(spp)}
    return write_scene(out_dir, name, sc, {name + "_crown.wo3": (crown_v, crown_t), name + "_trunk.wo3": (trunk_v, trunk_t)})


def curly_fibers(n_curves=200, nodes_per_curve=14, radius=0.45, length=1.1, width=0.01, seed=11):
    """Curly strands hanging from a cap: returns (curve_ends uint32[n], nodes float32[n*k, 4]) for save_fiber."""
    rng = np.random.RandomState(seed)
    nodes = np.zeros((n_curves*nodes_per_curve, 4), np.float32)
    ends = (np.arange(n_curves, dtype=np.uint32) + 1)*nodes_per_curve
    s = np.linspace(0.0, 1.0, nodes_per_curve)
    for c in range(n_curves):
        a, r = rng.uniform(0, 2*np.pi), radius*np.sqrt(rng.uniform(0.02, 1.0))
        root = np.array([r*np.cos(a), 0.0, r*np.sin(a)])
        out = np.array([np.cos(a), 0.0, np.sin(a)])
        curl_r, turns, ph = rng.uniform(0.02, 0.07), rng.uniform(1.5, 4.0), rng.uniform(0, 2*np.pi)
        ang = ph + 2*np.pi*turns*s
        p = root[None, :] + np.stack([out[0]*0.25*s*s + curl_r*np.cos(ang)*s, -length*rng.uniform(0.7, 1.0)*s,
                                      out[2]*0.25*s*s + curl_r*np.sin(ang)*s], axis=1)
        nodes[c*nodes_per_curve:(c + 1)*nodes_per_curve, :3] = p
        nodes[c*nodes_per_curve:(c + 1)*nodes_per_curve, 3] = width*rng.uniform(0.6, 1.4)
    return ends, nodes


def hair_scene(out_dir, name="hair", n_curves=200, nodes_per_curve=14, mode="bcsdf_cylinder", bsdf=None, res=(128, 128),
               spp=16, max_bounces=16, thickness=None, taper=False, subsample=0.0, env=(0.35, 0.4, 0.5), width=0.01, head=False,
               shipped_lights=False, min_bounces=0):
    """C4 stand-in: curly strands (`curves` primitive + `.fiber` file) with the hair BCSDF over a Lambert floor, lit by a
    quad light and a constant environment, or -- shipped_lights -- by exactly the two emitters of the reference's
    data/example-scenes/hair/scene.json: an `infinite_sphere_cap` sun (sampled) and a `skydome` (not sampled), same parameters;
    the skydome then names "sky_image": <name>_sky.pfm, the 512x256 image Skydome::prepareForRender computes, which the caller has
    to provide (tests/golden/make_golden.py dumps it from the reference; the reference itself ignores the key)."""
    from .scene import save_fiber
    os.makedirs(out_dir, exist_ok=True)
    ends, nodes = curly_fibers(n_curves, nodes_per_curve, width=width)
    save_fiber(os.path.join(out_dir, name + ".fiber"), ends, nodes)
    hb = dict(bsdf or {"type": "hair", "albedo": 1, "scale_angle": 2.5, "melanin_ratio": 0.6,
                       "melanin_concentration": 0.8, "roughness": 0.3}); hb["name"] = "strand"
    curves = {"name": "strands", "type": "curves", "file": name + ".fiber", "mode": mode, "bsdf": "strand",
              "curve_taper": taper, "subsample": subsample,
              "transform": {"position": [0.0, 1.55, 0.0], "scale": [1.0, 1.1, 1.0], "rotation": [0, 20, 0]}}
    if thickness is not None:
        curves["curve_thickness"] = thickness
    prims = [{"name": "floor", "type": "quad", "bsdf": "floor",
              "transform": {"position": [0, 0, 0], "scale": [6, 1, 6], "rotation": [0, 0, 0]}},
             curves,
             {"name": "light", "type": "quad", "bsdf": "light", "emission": [30, 28, 24],
              "transform": {"position": [0.9, 2.6, 1.2], "scale": [0.7, 1, 0.7], "rotation": [0, 0, 150]}}]
    if shipped_lights:
        prims = prims[:2]
        rot = [34.1619, -2.60535, 23.5692]
        prims.append({"name": "sun", "transform": {"rotation": rot}, "emission": 200, "type": "infinite_sphere_cap", "sample": True, "cap_angle": 10})
        prims.append({"name": "sky", "transform": {"rotation": rot}, "type": "skydome", "temperature": 5777, "gamma_scale": 1, "turbidity": 3,
                      "intensity": 5, "sample": False, "sky_image": name + "_sky.pfm"})
    elif env is not None:
        prims.append({"name": "env", "type": "infinite_sphere", "emission": list(env), "sample": True})
    meshes = {}
    if head:        # a triangle mesh under the strands: triangles and curve segments then share one BVH (joint root)
        meshes[name + "_head.wo3"] = icosphere(2, 1.0, displace=0.05)
        prims.append({"name": "head", "type": "mesh", "file": name + "_head.wo3", "smooth": True, "bsdf": "head",
                      "transform": {"position": [0.0, 1.3, 0.0], "scale": [0.42, 0.5, 0.42], "rotation": [0, 0, 0]}})
    sc = {"media": [], "bsdfs": [_lambert("floor", [0.5, 0.5, 0.5]), hb, {"name": "light", "albedo": 1, "type": "null"},
                                 {"name": "head", "type": "rough_plastic", "albedo": [0.7, 0.5, 0.4], "roughness": 0.3}],
          "primitives": prims,
          "camera": {"tonemap": "filmic", "resolution": list(res), "reconstruction_filter": "tent",
                     "transform": {"position": [0.3, 1.2, 3.4], "look_at": [0, 0.95, 0], "up": [0, 1, 0]},
                     "type": "pinhole", "fov": 35},
          "integrator": {"type": "path_tracer", "min_bounces": min_bounces, "max_bounces": max_bounces,
                         "enable_consistency_checks": False, "enable_two_sided_shading": True,
                         "enable_light_sampling": True},
          "renderer": _renderer(spp)}
    return write_scene(out_dir, name, sc, meshes)


def lobe_zoo(out_dir, name="lobe_zoo", res=(128, 128), spp=16, max_bounces=8, subdiv=2):
    """A 5 x 5 grid of small blobs, one per BSDF parameterisation the lobe tests single out -- Phong and Beckmann rough
    dielectrics, refraction off, roughness at the 1e-3 clamp and at 1, ior near 1 and above 2.4, a conductor with k = 0,
    checker and bitmap roughness, bitmap albedo in the four filter x wrap modes, the coats -- on a checker floor, under a quad
    light and an importance-sampled HDR environment: every lobe model and lobe mask on the path at once."""
    os.makedirs(out_dir, exist_ok=True)
    v, t = icosphere(subdiv, 1.0, displace=0.1)
    save_rgbe(os.path.join(out_dir, name + "_env.hdr"), sky_envmap(64, 32, sun_power=30.0))
    rng = np.random.RandomState(5)
    save_rgbe(os.path.join(out_dir, name + "_albedo.hdr"), rng.uniform(0.05, 0.95, (3, 4, 3)))
    save_rgbe(os.path.join(out_dir, name + "_rough.hdr"), np.repeat(rng.uniform(0.01, 0.8, (2, 3, 1)), 3, axis=2))
    def bitmap(f, interpolate=True, clamp=False):
        return {"type": "bitmap", "file": name + f, "interpolate": interpolate, "clamp": clamp}
    checker = {"type": "checker", "on_color": [0.05, 0.05, 0.05], "off_color": [0.6, 0.6, 0.6], "res_u": 4, "res_v": 4}
    bsdfs = [
        {"type": "rough_dielectric", "distribution": "phong", "roughness": 0.3, "ior": 1.45},
        {"type": "rough_dielectric", "distribution": "beckmann", "roughness": 0.4, "ior": 1.6},
        {"type": "rough_dielectric", "roughness": 0.2, "enable_refraction": False},
        {"type": "rough_conductor", "roughness": 1e-4},
        {"type": "rough_dielectric", "distribution": "beckmann", "roughness": 5e-4},
        {"type": "rough_plastic", "roughness": 1.0, "albedo": [0.5, 0.6, 0.7]},
        {"type": "rough_conductor", "distribution": "beckmann", "roughness": 1.0},
        {"type": "dielectric", "ior": 1.0001},
        {"type": "rough_dielectric", "ior": 1.001, "roughness": 0.3},
        {"type": "dielectric", "ior": 2.42},
        {"type": "rough_dielectric", "ior": 2.5, "roughness": 0.2},
        {"type": "conductor", "eta": [1.5, 1.2, 0.8], "k": [0.0, 0.0, 0.0]},
        {"type": "rough_conductor", "eta": [1.5, 1.2, 0.8], "k": [0.0, 0.0, 0.0], "roughness": 0.3},
        {"type": "rough_conductor", "roughness": checker},
        {"type": "rough_dielectric", "roughness": bitmap("_rough.hdr")},
        {"type": "lambert", "albedo": bitmap("_albedo.hdr", False, True)},
        {"type": "lambert", "albedo": bitmap("_albedo.hdr", False, False)},
        {"type": "plastic", "albedo": bitmap("_albedo.hdr", True, True)},
        {"type": "rough_plastic", "albedo": bitmap("_albedo.hdr", True, False), "distribution": "phong", "roughness": 0.2},
        {"type": "rough_conductor", "distribution": "phong", "roughness": 0.2},
        {"type": "plastic", "ior": 1.5, "thickness": 2.0, "sigma_a": [0.1, 0.2, 0.3], "albedo": [0.2, 0.4, 0.8]},
        {"type": "smooth_coat", "ior": 1.7, "thickness": 5.0, "sigma_a": [0.1, 0.2, 0.5], "substrate": "zooSubstrate"},
        {"type": "rough_coat", "distribution": "beckmann", "roughness": 0.3, "ior": 1.5, "thickness": 2.0, "sigma_a": [0.2, 0.1, 0.4],
         "substrate": "zooLambert"},
        {"type": "mirror", "albedo": [0.9, 0.8, 0.7]},
        {"type": "lambert", "albedo": [0.7, 0.5, 0.3]},
    ]
    for i, b in enumerate(bsdfs):
        b["name"] = "zoo%02d" % i
    bsdfs = [{"name": "zooSubstrate", "type": "rough_conductor", "distribution": "beckmann"},          # (named before their coats)
             {"name": "zooLambert", "type": "lambert", "albedo": [0.6, 0.3, 0.2]}] + bsdfs
    bsdfs += [{"name": "zooFloor", "type": "lambert", "albedo": {"type": "checker", "on_color": [0.7, 0.7, 0.7],
                                                                 "off_color": [0.2, 0.2, 0.25], "res_u": 10, "res_v": 10}},
              {"name": "zooLight", "type": "null"}]
    prims = [{"name": "floor", "type": "quad", "bsdf": "zooFloor", "transform": {"position": [0, 0, 0], "scale": [6, 1, 6]}},
             {"name": "light", "type": "quad", "bsdf": "zooLight", "emission": [12, 10, 8],
              "transform": {"position": [0.5, 3.0, 0.8], "scale": [1.2, 1, 0.8], "rotation": [180, 20, 0]}},
             {"name": "env", "type": "infinite_sphere", "emission": name + "_env.hdr", "sample": True,
              "transform": {"rotation": [0, 30, 0]}}]
    for i in range(25):
        x, z = (i % 5 - 2)*0.5, (i//5 - 2)*0.5
        prims.append({"name": "blob%02d" % i, "type": "mesh", "file": name + "_blob.wo3", "smooth": True, "bsdf": "zoo%02d" % i,
                      "transform": {"position": [x, 0.2, z], "scale": 0.2}})
    sc = {"media": [], "bsdfs": bsdfs, "primitives": prims,
          "camera": {"tonemap": "filmic", "resolution": list(res), "reconstruction_filter": "tent",
                     "transform": {"position": [0.0, 2.6, 3.2], "look_at": [0.0, 0.15, 0.0], "up": [0, 1, 0]},
                     "type": "pinhole", "fov": 40},
          "integrator": {"type": "path_tracer", "min_bounces": 0, "max_bounces": max_bounces, "enable_light_sampling": True,
                         "enable_consistency_checks": False, "enable_two_sided_shading": True},
          "renderer": _renderer(spp)}
    return write_scene(out_dir, name, sc, {name + "_blob.wo3": (v, t)})
