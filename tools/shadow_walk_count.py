"""Count the work of C1's any-hit shadow queries on the host, for the walk k_shadow_bvh used before (children sorted near-to-far,
from the root) and the one it uses now (nearest child entered, the others pushed unsorted, from the top-level cut boxes the segment
enters).  No GPU: tgb200_shadow_walk_count builds C1's tree as tgb200_create does and walks each query with the kernels' node and
triangle arithmetic.

Queries: points on the mesh and on the room's walls, aimed at uniform points of the ceiling light, tnear = 5e-4, t_light = the
distance to the light point.  Queries that enter no cut box are counted but not walked (k_shadow_prep settles them).

    python tools/shadow_walk_count.py [--queries N] [--seed S]
"""
import argparse
import ctypes as C
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tungsten_b200 import abi, lib, scene, synth  # noqa: E402

F = np.float32


def mesh_arrays(p):
    v = np.ctypeslib.as_array(C.cast(p.verts, C.POINTER(C.c_float)), shape=(p.n_verts*8,)).reshape(-1, 8)[:, :3].copy()
    t = np.ctypeslib.as_array(C.cast(p.tris, C.POINTER(C.c_uint32)), shape=(p.n_tris*4,)).reshape(-1, 4)[:, :3].copy()
    return v, t


def quad_points(p, rng, n):
    u, v = rng.rand(n, 1).astype(F), rng.rand(n, 1).astype(F)
    return (F(p.base) + u*F(p.edge0) + v*F(p.edge1)).astype(F)


def c1_queries(fs, rng, n):
    """(triangles n x 9, queries n x 8) of the C1 scene."""
    tris, surf = [], []
    for p in fs.primitives:
        if p.type == abi.PRIM_MESH and p.n_tris:
            v, t = mesh_arrays(p)
            tris.append(v[t].reshape(-1, 9))
    tris = np.concatenate(tris).astype(F)
    light = next(p for p in fs.primitives if p.type == abi.PRIM_QUAD and p.emission_tex >= 0)
    walls = [p for p in fs.primitives if p.type == abi.PRIM_QUAD and p.emission_tex < 0]
    on_mesh = n//2
    k = rng.randint(0, len(tris), on_mesh)
    w = rng.dirichlet([1, 1, 1], on_mesh).astype(F)
    surf.append((w[:, :, None]*tris[k].reshape(-1, 3, 3)).sum(1))
    wall = rng.randint(0, len(walls), n - on_mesh)
    for i, p in enumerate(walls):
        m = int((wall == i).sum())
        if m:
            surf.append(quad_points(p, rng, m))
    p = np.concatenate(surf).astype(F)
    t = quad_points(light, rng, n)
    d64 = (t - p).astype(np.float64)
    dist = np.linalg.norm(d64, axis=1)
    q = np.zeros((n, 8), F)
    q[:, :3] = p; q[:, 3:6] = (d64/dist[:, None]).astype(F); q[:, 6] = 5e-4; q[:, 7] = dist.astype(F)
    return tris, q


def walk_counts(tris, cam, q, stack_size=0):
    L = lib.load()
    tris = np.ascontiguousarray(tris, F); q = np.ascontiguousarray(q, F); cam = np.ascontiguousarray(cam, F)
    out = np.zeros((len(q), 11), np.uint32); need = C.c_uint32(0)
    rc = L.tgb200_shadow_walk_count(tris.ctypes.data, len(tris), cam.ctypes.data, q.ctypes.data, len(q), stack_size,
                                    C.byref(need), out.ctypes.data)
    return rc, need.value, out


def summary(out):
    walked = out[:, 0] != 0
    lines = ["queries %d, entering the cut (walked) %d" % (len(out), int(walked.sum()))]
    agree = np.array_equal(out[walked, 2], out[walked, 6])
    lines.append("both walks agree on visibility for every walked query: %s" % agree)
    for label, sel in (("occluded", walked & (out[:, 6] == 1)), ("unoccluded", walked & (out[:, 6] == 0)), ("all walked", walked)):
        lines.append("%s: %d queries" % (label, int(sel.sum())))
        if not sel.any():
            continue
        for name, col in (("node visits", 3), ("leaf trips", 4), ("triangle tests", 5)):
            a, b = out[sel, col].astype(np.float64), out[sel, col + 4].astype(np.float64)
            lines.append("  %-15s root/sorted mean %7.2f p50 %4d p90 %4d | cut/unsorted mean %7.2f p50 %4d p90 %4d | ratio %.3f"
                         % (name, a.mean(), np.percentile(a, 50), np.percentile(a, 90), b.mean(), np.percentile(b, 50),
                            np.percentile(b, 90), b.mean()/max(a.mean(), 1e-30)))
    lines.append("deepest stack of the cut walk: %d" % int(out[walked, 1].max()) if walked.any() else "no walked query")
    return agree, "\n".join(lines)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=200000)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    d = tempfile.mkdtemp(prefix="tgb_walk_count_")
    fs = scene.load_scene(synth.cornell_dragon_standin(d, res=(64, 36), spp=1))
    tris, q = c1_queries(fs, np.random.RandomState(args.seed), args.queries)
    rc, need, out = walk_counts(tris, F(fs.camera.pos), q)
    if rc != abi.TGB_OK:
        sys.exit("tgb200_shadow_walk_count failed: %d (stack need %d)" % (rc, need))
    agree, text = summary(out)
    print("C1: %d triangles, traversal stack need %d entries" % (len(tris), need))
    print(text)
    sys.exit(0 if agree else 1)


if __name__ == "__main__":
    main()
