"""Host-side logic: scene flattening (fp32, reference operation order), formats, spp stepping of the Integrator
mirror, tile sharding.  No GPU, no oracle compute."""
import json
import os

import numpy as np
import pytest

from tungsten_b200 import abi, scene, synth, integrator, lib


def test_wo3_roundtrip(tmp_path):
    v, t = synth.icosphere(2)
    p = str(tmp_path/"m.wo3")
    scene.save_wo3(p, v, t)
    assert os.path.getsize(p) == 8 + 32*len(v) + 8 + 16*len(t)
    v2, t2 = scene.load_wo3(p)
    assert np.array_equal(v2, v) and np.array_equal(t2, t)
    assert len(t) == 20*4**2


def test_pfm_roundtrip(tmp_path):
    img = np.random.RandomState(0).rand(5, 7, 3).astype(np.float32)
    p = str(tmp_path/"a.pfm")
    scene.save_pfm(p, img)
    assert np.array_equal(scene.load_pfm(p), img)


def test_cornell_flattening():
    fs = scene.load_scene(synth.cornell_box(res=(100, 50), spp=4))
    assert fs.resolution == (100, 50)
    assert len(fs.primitives) == 8 and len(fs.bsdfs) == 8
    floor = fs.primitives[0]
    assert floor.type == abi.PRIM_QUAD
    # floor: scale (2,4,2), rotation (0,90,0): 2x2 square at y=0
    e0 = np.array(floor.edge0[:]); e1 = np.array(floor.edge1[:]); base = np.array(floor.base[:])
    assert abs(np.linalg.norm(e0) - 2) < 1e-6 and abs(np.linalg.norm(e1) - 2) < 1e-6
    assert abs(base[1]) < 1e-6 and np.allclose(np.abs(base[[0, 2]]), 1, atol=1e-6)
    n = np.cross(e1, e0)
    assert n[1] > 0                                    # floor normal points up
    light = fs.primitives[-1]
    assert light.emission_tex >= 0 and fs.textures[light.emission_tex].value[0] == 17
    ln = np.cross(np.array(light.edge1[:]), np.array(light.edge0[:]))
    assert ln[1] < 0                                   # light faces down
    cube = fs.primitives[5]
    assert cube.type == abi.PRIM_CUBE
    r = np.array(cube.rot[:]).reshape(3, 3)
    assert np.allclose(r @ r.T, np.eye(3), atol=1e-5)
    assert np.allclose(np.array(cube.scale[:])*2, [0.594811, 0.604394, 0.6], atol=1e-6)
    cam = fs.camera
    assert np.allclose(cam.pos[:], [0, 1, 6.8]) and cam.fov_deg == 35 and cam.filter == abi.FILTER_TENT
    m = np.array(cam.xform[:]).reshape(3, 3)
    assert np.allclose(m[:, 2], [0, 0, -1], atol=1e-6)  # looks down -z
    assert np.allclose(m[:, 0], [1, 0, 0], atol=1e-6)   # right vector after setRight(-right)
    s = fs.settings
    assert (s.max_bounces, s.min_bounces, s.enable_light_sampling, s.use_sobol) == (64, 0, 1, 1)
    assert fs.spp == 4 and fs.adaptive is False


def test_transform_parse_variants():
    ident = scene.parse_transform(None)
    assert np.array_equal(ident, np.eye(4, dtype=np.float32))
    m = scene.parse_transform({"position": [1, 2, 3], "scale": 2, "rotation": [0, 0, 0]})
    assert np.allclose(m, [[2, 0, 0, 1], [0, 2, 0, 2], [0, 0, 2, 3], [0, 0, 0, 1]])
    m = scene.parse_transform({"position": [0, 0, 0], "rotation": [0, 90, 0]})
    assert np.allclose(m[:3, :3] @ m[:3, :3].T, np.eye(3), atol=1e-6)
    assert np.allclose(m[:3, 0], [0, 0, 1], atol=1e-6) or np.allclose(m[:3, 0], [0, 0, -1], atol=1e-6)
    m16 = scene.parse_transform(list(range(16)))
    assert m16[1, 2] == 6
    with pytest.raises(scene.SceneError):
        scene.parse_transform([1, 2, 3])


def test_out_of_scope_features_are_rejected(tmp_path):
    base = synth.cornell_box(res=(8, 8), spp=1)
    for mut in [lambda s: s.__setitem__("media", [{"type": "homogeneous"}]),
                lambda s: s["integrator"].__setitem__("type", "bidirectional_path_tracer"),
                lambda s: s["camera"].__setitem__("type", "thinlens"),
                lambda s: s["bsdfs"].append({"name": "x", "type": "phong"}),
                lambda s: s["primitives"].append({"type": "sphere", "bsdf": "floor"}),
                lambda s: s["bsdfs"][0].__setitem__("bump", 0.5)]:
        s = json.loads(json.dumps(base)); mut(s)
        with pytest.raises(scene.SceneError):
            scene.load_scene(s)


def test_mesh_transform_and_material_clamp(tmp_path):
    p = synth.cornell_mesh(str(tmp_path), subdiv=1, res=(8, 8), spp=1)
    fs = scene.load_scene(p)
    mesh = [q for q in fs.primitives if q.type == abi.PRIM_MESH][0]
    assert mesh.n_tris == 80 and mesh.smooth == 1
    pos = np.ctypeslib.as_array(mesh.verts, (mesh.n_verts,))["pos"]
    assert pos[:, 1].min() > 0.0 and pos[:, 1].max() < 2.0      # inside the box
    tris = np.ctypeslib.as_array(mesh.tris, (mesh.n_tris,))
    assert tris["material"].min() == 0 and tris["material"].max() == 0


class _FakeCtx:
    def __init__(self): self.calls = []; self.aborted = False; self.adaptive_calls = []; self.L = lib.load()
    def render_resident(self, count, seed, spp_begin, tiles): self.calls.append((spp_begin, count, len(tiles)))
    def render_adaptive(self, records, seed, tiles): self.adaptive_calls.append([(r.sample_index, r.next_sample_count) for r in records])
    def clear_abort(self): self.aborted = False
    def clear(self): pass
    def close(self): pass
    def abort(self): self.aborted = True
    def read_framebuffer(self): return np.zeros((1, 1, 3), np.float32), None


def test_integrator_spp_stepping(monkeypatch):
    """Integrator::advanceSpp / done / startRender (Integrator.cpp:51, PathTraceIntegrator.cpp:220-239)."""
    sc = synth.cornell_box(res=(40, 24), spp=40); sc["renderer"]["spp_step"] = 16
    fs = scene.load_scene(sc)
    fake = _FakeCtx()
    monkeypatch.setattr(lib, "Context", lambda *a, **k: fake)
    it = integrator.B200PathTraceIntegrator()
    it.prepareForRender(fs, 0xBA5EBA11)
    assert (it.currentSpp(), it.nextSpp(), it.done()) == (0, 16, False)
    fired = []
    while not it.done():
        it.startRender(lambda: fired.append(1)); it.waitForCompletion()
    assert fake.calls == [(0, 16, 6), (16, 16, 6), (32, 8, 6)]
    assert it.currentSpp() == 40 and len(fired) == 3
    it.startRender(lambda: fired.append(1))            # no work left: callback fires synchronously
    assert len(fired) == 4
    it.teardownAfterRender()


def test_integrator_adaptive_steps_carry_block_records(monkeypatch):
    """adaptive scenes go through generateWork + the per-block records (PathTraceIntegrator.cpp:110-156): below 16 spp every
    block gets the step's sample count, sample indices accumulate."""
    sc = synth.cornell_box(res=(16, 16), spp=24); sc["renderer"]["adaptive_sampling"] = True; sc["renderer"]["spp_step"] = 8
    fs = scene.load_scene(sc)
    fake = _FakeCtx()
    monkeypatch.setattr(lib, "Context", lambda *a, **k: fake)
    it = integrator.B200PathTraceIntegrator()
    it.prepareForRender(fs, 1)
    it.startRender(); it.waitForCompletion()
    it.startRender(); it.waitForCompletion()
    assert fake.calls == [] and len(fake.adaptive_calls) == 2
    assert fake.adaptive_calls[0] == [(0, 8)]*16 and fake.adaptive_calls[1] == [(8, 8)]*16
    # third step starts at 16 spp = AdaptiveThreshold: the (all-zero) error estimate says there is nothing to do
    fired = []
    it.startRender(lambda: fired.append(1))
    assert fired == [1] and it.currentSpp() == 24 and len(fake.adaptive_calls) == 2
    it.teardownAfterRender()


def test_tile_sharding_partitions_the_image():
    tiles = integrator.dice_tiles(100, 50, 5)
    assert len(tiles) == 7*4
    seen = np.zeros((50, 100), dtype=int)
    for r in range(3):
        for t in integrator.shard_tiles(tiles, r, 3):
            seen[t.y:t.y + t.h, t.x:t.x + t.w] += 1
    assert (seen == 1).all()
    assert tiles[6].w == 4 and tiles[21].h == 2
    assert len({t.sampler_seed for t in tiles}) == len(tiles)


def test_quaternion_helpers_match_rotation_matrices():
    """QuaternionF::fromMatrix / operator* restated in fp32 (math/Quaternion.hpp:68-88,111-146)."""
    rng = np.random.RandomState(3)
    for rot in ([0, 0, 0], [10, 200, -35], [90, 0, 0], [0, 180, 0], [179, 179, 179]):
        m = scene.parse_transform({"rotation": rot})[:3, :3]
        q = scene.quat_from_matrix(m)
        assert abs(float(np.dot(q, q)) - 1.0) < 1e-5
        p = rng.normal(size=(7, 3)).astype(np.float32)
        assert np.allclose(scene.quat_rotate(q, p), p @ m.T, atol=2e-6)
    a = scene.quat_from_matrix(scene.parse_transform({"rotation": [0, 30, 0]})[:3, :3])
    b = scene.quat_from_matrix(scene.parse_transform({"rotation": [0, 45, 0]})[:3, :3])
    ab = scene.quat_from_matrix(scene.parse_transform({"rotation": [0, 75, 0]})[:3, :3])
    assert np.allclose(scene.quat_mul(a, b), ab, atol=1e-6) or np.allclose(scene.quat_mul(a, b), -ab, atol=1e-6)


def test_instances_flatten_to_world_space(tmp_path):
    p = synth.instanced_forest(str(tmp_path), n_instances=5, tree_subdiv=1, res=(8, 8), spp=1)
    fs = scene.load_scene(p)
    mesh = [q for q in fs.primitives if q.type == abi.PRIM_MESH][0]
    assert mesh.n_tris == 5*(80 + 20) and mesh.bsdf_count == 2
    pos = np.ctypeslib.as_array(mesh.verts, (mesh.n_verts,))["pos"]
    assert pos[:, 1].min() > -0.2 and pos[:, 1].max() < 2.5          # trees stand on the ground
    nrm = np.ctypeslib.as_array(mesh.verts, (mesh.n_verts,))["normal"]
    assert np.isfinite(nrm).all()


@pytest.mark.parametrize("n", [0, 1, 3, 4, 5, 64, 1280, 20480])
def test_bvh_builder_selftest(n):
    """bvh_build.cpp (host C++): every triangle in exactly one leaf, boxes nest, leaves <= 4 triangles."""
    import ctypes as C
    L = lib.load()
    L.tgb200_bvh_selftest.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    if n >= 1280:
        v, t = synth.icosphere(3 if n == 1280 else 5, displace=0.2)
        tri = np.ascontiguousarray(np.stack([v["pos"][t["v0"]], v["pos"][t["v1"]], v["pos"][t["v2"]]], axis=1), dtype=np.float32)
    else:
        rng = np.random.RandomState(n)
        c = rng.uniform(-1, 1, (n, 1, 3)); tri = (c + rng.normal(scale=0.05, size=(n, 3, 3))).astype(np.float32)
        if n >= 4:
            tri[1] = tri[0]                      # duplicates: coincident centroids must still split
            tri[2] = tri[0]
    assert len(tri) == n
    nodes, depth, leaf = C.c_uint32(), C.c_uint32(), C.c_uint32()
    rc = L.tgb200_bvh_selftest(tri.ctypes.data if n else None, n, C.byref(nodes), C.byref(depth), C.byref(leaf))
    assert rc == 0
    if n:
        assert leaf.value <= 4 and nodes.value >= 1 and depth.value <= 40


def test_fiber_roundtrip_and_curve_flattening(tmp_path):
    """.fiber reader/writer (io/CurveIO.cpp:343-403) and Curves::loadCurves/prepareForRender bookkeeping
    (Curves.cpp:268-296,572-611): thickness override, taper, subsample with the default UniformSampler seed."""
    ends, nodes = synth.curly_fibers(n_curves=40, nodes_per_curve=9)
    p = str(tmp_path/"c.fiber")
    scene.save_fiber(p, ends, nodes)
    e2, n2 = scene.load_fiber(p)
    assert np.array_equal(e2, ends) and np.array_equal(n2, nodes)
    fs = scene.FlatScene(); b = fs.add_bsdf({"type": "lambert"})
    fs.add_curves(np.eye(4, dtype=np.float32), ends, nodes, b, mode="cylinder")
    pr = fs.primitives[-1]
    assert pr.n_curve_segments == 40*(9 - 2) and pr.n_curve_nodes == len(nodes)
    segs = np.ctypeslib.as_array(pr.curve_segments, (pr.n_curve_segments,))
    assert segs[0] == 2 and segs[6] == 8 and segs[7] == 11          # a curve of k nodes has k-2 segments ending at nodes 2..k-1
    # subsample drops whole curves with the reference's PCG stream: same draw sequence -> same survivors every time
    fs2 = scene.FlatScene(); b2 = fs2.add_bsdf({"type": "lambert"})
    fs2.add_curves(np.eye(4, dtype=np.float32), ends, nodes, b2, thickness=np.float32(0.02), taper=True, subsample=0.5)
    pr2 = fs2.primitives[-1]
    assert 0 < pr2.n_curve_segments < pr.n_curve_segments and pr2.n_curve_segments % 7 == 0
    w = np.ctypeslib.as_array(pr2.curve_nodes, (pr2.n_curve_nodes*4,)).reshape(-1, 4)[:, 3]
    assert np.isclose(w[0], 0.02*(1.0 + 0.5/8.0)) and w[8] < w[0]       # taper: 1 - (t - 0.5)/(k - 1)
    with pytest.raises(scene.SceneError):
        fs.add_curves(np.eye(4, dtype=np.float32), ends, nodes, b, mode="ribbon")


def test_hair_tables_host_precompute_matches_oracle():
    """tgb200_hair_selftest (host C++ of the library) vs the oracle's restatement of HairBcsdf::precomputeAzimuthalDistributions:
    same libm, same operation order -> identical tables, sampling sums and lobe variances."""
    import ctypes as C
    from oracle import pyoracle
    L = lib.load(); O = pyoracle.lib()
    out = []
    for fn in (L.tgb200_hair_selftest, O.oracle_hair_tables):
        fn.restype = C.c_int; fn.argtypes = [C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        sa = np.array([0.25, 0.45, 1.1], np.float32)
        t = np.zeros(3*64*64*3, np.float32); s = np.zeros(3*64, np.float32); v = np.zeros(3, np.float32)
        assert fn(0.3, 2.5, sa.ctypes.data, t.ctypes.data, s.ctypes.data, v.ctypes.data) == 0
        out.append((t, s, v))
    for a, b in zip(out[0], out[1]):
        assert np.array_equal(a, b)
    t = out[0][0].reshape(3, 64, 64, 3)
    assert np.isfinite(t[:, 1:]).all() and (t[:, 1:] >= 0).all()
    assert np.allclose(out[0][2], [(np.pi/2*0.3)**2, (np.pi/4*0.3)**2, (np.pi*0.3)**2], rtol=1e-5)
    assert (t[0, 1:, :, 0] == t[0, 1:, :, 1]).all()                 # the R lobe is colourless
    assert t[1, 32, :, 2].sum() < t[1, 32, :, 0].sum()              # TT is tinted by absorption (blue absorbed most)


def test_depth_first_quantised_bvh_walk_equals_brute_force():
    """QNode4 (8-bit child boxes on a per-node power-of-two grid) + depth-first renumbering,
    walked on the HOST with the kernels' node arithmetic (one byte permute + one fma per plane): closest t of 6,000 rays ==
    brute force over all triangles bit for bit -> the quantised boxes are conservative under the kernel's rounding."""
    import ctypes as C
    from tungsten_b200 import lib, synth
    L = lib.load()
    rng = np.random.RandomState(3)
    for case in range(3):
        if case == 0:                                   # smooth closed mesh + big ground triangles (large / tiny boxes mixed)
            v, t = synth.icosphere(4, displace=0.05)
            tv = np.ascontiguousarray(v["pos"][np.stack([t["v0"], t["v1"], t["v2"]], axis=1)].reshape(-1, 9), dtype=np.float32)
            g = np.array([[-50, 0, -50, 50, 0, -50, 0, 0, 70], [-50, -1, -50, 0, -1, 70, 50, -1, -50]], dtype=np.float32)
            tv = np.concatenate([tv, g]).astype(np.float32)
        elif case == 1:                                 # random soup far from the origin (large coordinates, tiny extents)
            c = rng.uniform(900, 1000, (4000, 1, 3)); tv = (c + rng.normal(scale=0.02, size=(4000, 3, 3))).reshape(-1, 9).astype(np.float32)
        else:                                           # axis-aligned slivers (zero-extent boxes on one axis)
            a = rng.uniform(-1, 1, (3000, 3)).astype(np.float32)
            tv = np.concatenate([a, a + [0.1, 0, 0], a + [0, 0.1, 0]], axis=1).astype(np.float32)
        n = len(tv)
        lo, hi = tv.reshape(-1, 3).min(0), tv.reshape(-1, 3).max(0)
        m = 2000
        o = rng.uniform(lo - 0.3*(hi - lo), hi + 0.3*(hi - lo), (m, 3)).astype(np.float32)
        tgt = tv.reshape(-1, 3)[rng.randint(0, 3*n, m)] + rng.normal(scale=0.01, size=(m, 3))
        d = (tgt - o); d /= np.linalg.norm(d, axis=1, keepdims=True)
        d[:50, 0] = 0.0                                 # axis-parallel directions
        rays = np.concatenate([o, d.astype(np.float32), np.full((m, 1), 1e-4, np.float32), np.full((m, 1), np.inf, np.float32)], axis=1).astype(np.float32)
        bad, nn, visits = C.c_uint32(), C.c_uint32(), C.c_uint64()
        rc = L.tgb200_qbvh_selftest(tv.ctypes.data, n, rays.ctypes.data, m, C.byref(bad), C.byref(nn), C.byref(visits))
        assert rc == 0, (case, rc)
        assert bad.value == 0, (case, bad.value)
        assert visits.value > m


def _adaptive_reference_emulation(fs, seed=0xBA5EBA11):
    """The reference's adaptive loop (PathTraceIntegrator::startRender/generateWork/renderTile) with the CPU oracle as the
    per-sample renderer and the LIBRARY's host-side tgb200_generate_work as the sample distributor."""
    import ctypes as C
    from tungsten_b200 import lib, abi, integrator
    from oracle import pyoracle
    L = lib.load()
    w, h = fs.resolution
    var_w, var_h = (w + 3)//4, (h + 3)//4
    sampler = integrator.UniformSampler(integrator.hash32(seed))
    tiles = integrator.dice_tiles(w, h, seed, sampler)
    records = (abi.SampleRecord*(var_w*var_h))()
    st = C.c_uint64(sampler.state)
    orc = pyoracle.Oracle(fs)
    mean = np.zeros((h, w, 3), np.float32); count = np.zeros((h, w), np.uint32)
    cur = 0
    f32 = np.float32
    while cur < fs.spp:
        nxt = min(cur + fs.spp_step, fs.spp)
        if L.tgb200_generate_work(records, w, h, cur, nxt, 1 if fs.adaptive else 0, C.byref(st)) == 1:
            for t in tiles:
                for by in range(t.y, t.y + t.h, 4):
                    for bx in range(t.x, t.x + t.w, 4):
                        r = records[bx//4 + (by//4)*var_w]
                        blk = (abi.Tile*1)(abi.Tile(bx, by, min(4, w - bx), min(4, h - by), t.sampler_seed))
                        n = r.next_sample_count
                        if n == 0:
                            continue
                        # the block's samples one by one (for SampleRecord::addSample), then folded into the framebuffer
                        smp = np.zeros((n, h, w, 3), np.float32)
                        for i in range(n):
                            orc.render(1, seed=seed, spp_begin=r.sample_index + i, tiles=blk, threads=1, mean=smp[i], count=np.zeros((h, w), np.uint32))
                        orc.render(n, seed=seed, spp_begin=r.sample_index, tiles=blk, threads=1, mean=mean, count=count)
                        for y in range(by, min(by + 4, h)):
                            for x in range(bx, min(bx + 4, w)):
                                for i in range(n):
                                    c = smp[i, y, x]
                                    lum = f32(f32(f32(c[0]*f32(0.2126)) + f32(c[1]*f32(0.7152))) + f32(c[2]*f32(0.0722)))
                                    r.sample_count += 1
                                    delta = f32(lum - f32(r.mean))
                                    r.mean = f32(f32(r.mean) + f32(delta/f32(r.sample_count)))
                                    r.running_variance = f32(f32(r.running_variance) + f32(delta*f32(lum - f32(r.mean))))
        cur = nxt
    orc.close()
    return mean, count, records


def test_adaptive_sampling_matches_reference_binary():
    """renderer.adaptive_sampling = true (as shipped scenes have it): tgb200_generate_work (95th-percentile clamp, dilation,
    stochastic distribution, PathTraceIntegrator.cpp:44-134) driven exactly like the reference's loop, samples from the CPU
    oracle -> the framebuffer equals what the reference binary itself rendered (tests/golden/cornell_adaptive) bit for bit."""
    from tungsten_b200 import scene
    g = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cornell_adaptive")
    fs = scene.load_scene(os.path.join(g, "scene.json"))
    assert fs.adaptive and fs.spp == 48 and fs.spp_step == 16
    want = scene.load_pfm(os.path.join(g, "ref_pathseed.pfm"))
    mean, count, records = _adaptive_reference_emulation(fs)
    assert count.min() >= 16 + 2 and count.max() > 48                     # the two adaptive steps really redistributed samples (>= 1 per step)
    exact = float((np.abs(mean - want).max(axis=2) == 0).mean())
    print("adaptive: per-pixel samples %d..%d, exact %.4f" % (count.min(), count.max(), exact))
    assert exact == 1.0


def test_library_tile_deal_matches_the_python_twin():
    """tgb200_shard_tiles (the in-library multi-GPU deal) == integrator.shard_order (what bench.py's ranks use): same Morton
    order, every share covers the frame evenly."""
    import ctypes as C
    L = lib.load()
    for (w, h) in [(1920, 1080), (250, 90), (16, 16), (3840, 2160)]:
        tiles = integrator.dice_tiles(w, h, 0xBA5EBA11)
        order = (C.c_uint32*len(tiles))()
        assert L.tgb200_shard_tiles(tiles, len(tiles), order) == 0
        assert list(order) == integrator.shard_order(tiles, "morton")
        if w == 1920:
            for world in (2, 4, 8):                 # a share is a regular sub-lattice of the tile grid spanning the whole frame, not a stripe
                sizes = []
                for r in range(world):
                    mine = integrator.shard_tiles(tiles, r, world)
                    sizes.append(len(mine))
                    xs = {t.x for t in mine}; ys = {t.y for t in mine}
                    assert len(xs) >= 120//4 and len(ys) >= 68//4
                    assert max(xs) - min(xs) >= 0.9*1920 and max(ys) - min(ys) >= 0.9*1080
                assert max(sizes) - min(sizes) <= 1
