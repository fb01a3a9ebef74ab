"""The drop-in adapter's scene description against the Python flattener's, field for field and bit for bit (CPU, no GPU).

Two independent builders fill the `tgb_scene_desc` the library renders: `tungsten_b200.scene` (fp32 numpy restatement of the
reference's JSON loading and prepareForRender; every GPU test and bench.py use it) and the C++ adapter
(integration/B200PathTraceIntegrator.cpp, `Flattener`), which reads the reference's live objects and is what a user of the drop-in
runs.  Here a small C shim (tests/dropin_capture_shim.c), preloaded into the literal drop-in binary
oracle/_ref/dropin/tungsten_b200, takes the place of the library's tgb200_create: it writes the desc the adapter built, with every
array it points to, to a file and ends the process before anything touches CUDA.  That capture is compared with
scene.load_scene(...).desc() of the same JSON in canonical form:

- primitives by position (both follow Scene::primitives() order), each with the fields upload_scene (tgb200_api.cu) reads for
  its type (PRIM_FIELDS);
- BSDFs and textures resolved through bsdf_slots / substrate / albedo_tex / roughness_tex / emission_tex and compared as
  records (BSDF_FIELDS, TEX_FIELDS), so dedup and ordering may differ, and records that no primitive reaches are ignored (the
  adapter dedups by object, the Python side adds every named BSDF);
- camera, the integrator settings (the device fields excluded), and n_devices / devices[] where the scene names devices.

Every value is compared as raw 32-bit words.  There are no tolerances and no exceptions.
"""
import ctypes as C
import json
import os
import shutil
import struct
import subprocess
import zlib

import numpy as np
import pytest

from tungsten_b200 import abi, scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "oracle", "_ref", "dropin", "tungsten_b200")
SHIM_SRC = os.path.join(ROOT, "tests", "dropin_capture_shim.c")
G = os.path.join(ROOT, "tests", "golden")
FIXTURES = sorted(d for d in os.listdir(G) if os.path.isfile(os.path.join(G, d, "scene.json")))

pytestmark = pytest.mark.skipif(not os.path.exists(EXE),
                                reason="drop-in binary oracle/_ref/dropin/tungsten_b200 not built "
                                       "(build() makes it where the reference's sources are present)")

# ---- what the library reads (tgb200_api.cu, upload_scene) -------------------------------------------------------------------
# per texture type: the tgb_texture fields upload_scene and tex_eval read
TEX_FIELDS = {
    abi.TEX_CONSTANT: ("value",),
    abi.TEX_CHECKER: ("value", "value2", "res_u", "res_v"),
    abi.TEX_BITMAP: ("res_u", "res_v", "flags", "texels"),
}
# per BSDF type: the tgb_bsdf fields besides `type` and `albedo_tex` (read for every type).  "roughness" = the texture of
# roughness_tex, "substrate" = the record of bsdf `substrate`.
_ROUGH = ("distribution", "roughness")
BSDF_FIELDS = {
    abi.BSDF_NULL: (),
    abi.BSDF_LAMBERT: (),
    abi.BSDF_MIRROR: (),
    abi.BSDF_CONDUCTOR: ("eta", "k"),
    abi.BSDF_ROUGH_CONDUCTOR: ("eta", "k") + _ROUGH,
    abi.BSDF_DIELECTRIC: ("ior", "enable_refraction"),
    abi.BSDF_ROUGH_DIELECTRIC: ("ior", "enable_refraction") + _ROUGH,
    abi.BSDF_PLASTIC: ("ior", "thickness", "sigma_a"),
    abi.BSDF_ROUGH_PLASTIC: ("ior", "thickness", "sigma_a") + _ROUGH,
    abi.BSDF_SMOOTH_COAT: ("ior", "thickness", "sigma_a", "substrate"),
    abi.BSDF_ROUGH_COAT: ("ior", "thickness", "sigma_a", "substrate") + _ROUGH,
    abi.BSDF_HAIR: ("sigma_a", "hair_scale_angle_deg", "hair_roughness"),
}
# per primitive type: the tgb_primitive fields besides `type` and `emission_tex`; primitives that are not environment lights
# also have their BSDF slots compared.  A cube's and an environment sphere's `rot` count, a quad's does not; a skydome's rot is
# replaced by the identity in upload_scene.
PRIM_FIELDS = {
    abi.PRIM_MESH: ("smooth", "verts", "tris"),
    abi.PRIM_QUAD: ("base", "edge0", "edge1"),
    abi.PRIM_CUBE: ("pos", "rot", "scale"),
    abi.PRIM_INFINITE_SPHERE: ("rot", "do_sample"),
    abi.PRIM_SKYDOME: ("do_sample",),
    abi.PRIM_INFINITE_SPHERE_CAP: ("cap_dir", "cap_cos", "do_sample"),
    abi.PRIM_CURVES: ("curve_mode", "curve_nodes", "curve_segments"),
}
ENVIRONMENT = (abi.PRIM_INFINITE_SPHERE, abi.PRIM_SKYDOME, abi.PRIM_INFINITE_SPHERE_CAP)
CAMERA_FIELDS = ("pos", "xform", "fov_deg", "res_x", "res_y", "filter")
SETTINGS_FIELDS = ("min_bounces", "max_bounces", "enable_light_sampling", "enable_two_sided_shading",
                   "enable_consistency_checks", "use_sobol", "supplemental_mode")
# column names of the arrays, for the failure messages
COLUMNS = {
    "verts": ("pos[0]", "pos[1]", "pos[2]", "normal[0]", "normal[1]", "normal[2]", "uv[0]", "uv[1]"),
    "tris": ("v0", "v1", "v2", "material"),
    "curve_nodes": ("x", "y", "z", "width"),
    "curve_segments": None,
    "texels": ("r", "g", "b"),
}


# ---- one desc with all its arrays, read from a capture file or from a FlatScene --------------------------------------------
class Side:
    def __init__(self, desc, prims, bsdfs, slots, textures, arrays, texels):
        self.desc, self.prims, self.bsdfs, self.slots, self.textures = desc, prims, bsdfs, slots, textures
        self.arrays = arrays        # per primitive: {"verts", "tris", "curve_nodes", "curve_segments"} -> uint32 words
        self.texels = texels        # per texture: uint32 words (empty unless a bitmap)


def _words(b):
    return np.frombuffer(bytes(b), dtype=np.uint32)


def read_capture(blob):
    assert blob[-8:] == b"TGBCAPOK", "capture file is truncated"
    off = 0

    def block():
        nonlocal off
        n = int.from_bytes(blob[off:off + 8], "little")
        b = blob[off + 8:off + 8 + n]
        off += 8 + n
        return b

    def structs(T, b):
        assert len(b) % C.sizeof(T) == 0
        return [T.from_buffer_copy(b, i*C.sizeof(T)) for i in range(len(b)//C.sizeof(T))]
    desc = abi.SceneDesc.from_buffer_copy(block())
    prims, bsdfs = structs(abi.Primitive, block()), structs(abi.Bsdf, block())
    slots, textures = _words(block()), structs(abi.Texture, block())
    arrays = [{k: _words(block()) for k in ("verts", "tris", "curve_nodes", "curve_segments")} for _ in prims]
    texels = [_words(block()) for _ in textures]
    assert off == len(blob) - 8, "capture file has trailing bytes"
    return Side(desc, prims, bsdfs, slots, textures, arrays, texels)


def read_flat(fs):
    d = fs.desc()

    def raw(ptr, nbytes):
        return _words(C.string_at(ptr, nbytes)) if nbytes else np.zeros(0, np.uint32)
    prims = [d.primitives[i] for i in range(d.n_primitives)]
    textures = [d.textures[i] for i in range(d.n_textures)]
    arrays = [{"verts": raw(p.verts, 32*p.n_verts), "tris": raw(p.tris, 16*p.n_tris),
               "curve_nodes": raw(p.curve_nodes, 16*p.n_curve_nodes), "curve_segments": raw(p.curve_segments, 4*p.n_curve_segments)}
              for p in prims]
    texels = [raw(t.texels, 12*t.res_u*t.res_v) if t.type == abi.TEX_BITMAP else np.zeros(0, np.uint32) for t in textures]
    return Side(d, prims, [d.bsdfs[i] for i in range(d.n_bsdfs)], raw(d.bsdf_slots, 4*d.n_bsdf_slots), textures, arrays, texels)


# ---- canonical form: path -> (uint32 words as rows x columns, column names) -------------------------------------------------
def _field_words(struct_, name):
    ty = dict(struct_._fields_)[name]
    is_array = issubclass(ty, C.Array)
    values = list(getattr(struct_, name)) if is_array else [getattr(struct_, name)]
    if (ty._type_ if is_array else ty) is C.c_float:
        return np.array(values, dtype=np.float32).view(np.uint32)
    return np.array(values, dtype=np.int64).astype(np.uint32)


class Canon:
    def __init__(self, side, devices=False):
        self.s, self.out = side, {}
        self.n_bsdfs = self.n_textures = 0
        d = side.desc
        for f in CAMERA_FIELDS:
            self.put("camera." + f, _field_words(d.camera, f))
        for f in SETTINGS_FIELDS:
            self.put("settings." + f, _field_words(d.settings, f))
        if devices:
            n = d.settings.n_devices
            self.put("settings.n_devices", _field_words(d.settings, "n_devices"))
            self.put("settings.devices", _field_words(d.settings, "devices")[:n])
        for i, p in enumerate(side.prims):
            self.primitive("primitives[%d]" % i, i, p)
        self.n_primitives = len(side.prims)

    def put(self, path, words, cols=None):
        words = np.asarray(words, dtype=np.uint32)
        self.out[path] = (words.reshape(-1, len(cols)) if cols else words.reshape(1, -1), cols)

    def texture(self, path, i):
        self.n_textures += 1
        t = self.s.textures[i]
        self.put(path + ".type", [t.type])
        for f in TEX_FIELDS.get(t.type, ()):
            if f == "texels":
                self.put(path + ".texels", self.s.texels[i], COLUMNS["texels"])
            else:
                self.put(path + "." + f, _field_words(t, f))

    def bsdf(self, path, i, hops=0):
        assert hops < 4, path + ": substrate chain too deep"
        self.n_bsdfs += 1
        b = self.s.bsdfs[i]
        self.put(path + ".type", [b.type])
        self.texture(path + ".albedo", b.albedo_tex)
        for f in BSDF_FIELDS.get(b.type, ()):
            if f == "roughness":
                self.texture(path + ".roughness", b.roughness_tex)
            elif f == "substrate":
                self.bsdf(path + ".substrate", b.substrate, hops + 1)
            else:
                self.put(path + "." + f, _field_words(b, f))

    def primitive(self, path, i, p):
        self.put(path + ".type", [p.type])
        if p.emission_tex >= 0:
            self.texture(path + ".emission", p.emission_tex)
        else:
            self.put(path + ".emission", [0xFFFFFFFF])
        if p.type not in ENVIRONMENT:
            self.put(path + ".bsdf_count", [p.bsdf_count])
            for k in range(p.bsdf_count):
                self.bsdf("%s.bsdfs[%d]" % (path, k), int(self.s.slots[p.bsdf_first + k]))
        for f in PRIM_FIELDS.get(p.type, ()):
            if f in COLUMNS:
                self.put(path + "." + f, self.s.arrays[i][f], COLUMNS[f])
            else:
                self.put(path + "." + f, _field_words(p, f))

    @property
    def n_words(self):
        return sum(w.size for w, _ in self.out.values())


def _name(path, cols, r, c, shape):
    if cols:
        return "%s[%d].%s" % (path, r, cols[c])
    return path if shape[1] == 1 else "%s[%d]" % (path, c)


def compare(got, want, limit=12):
    """got = adapter, want = Python flattener; returns the list of differences, each naming the path and both values."""
    diffs = []
    for path in sorted(set(got.out) | set(want.out)):
        if path not in got.out or path not in want.out:
            diffs.append("%s: only in the %s desc" % (path, "adapter's" if path in got.out else "flattener's"))
            continue
        (a, cols), (b, _) = got.out[path], want.out[path]
        if a.shape != b.shape:
            diffs.append("%s: %d x %d words != %d x %d words" % (path, a.shape[0], a.shape[1], b.shape[0], b.shape[1]))
            continue
        for r, c in zip(*np.nonzero(a != b)):
            diffs.append("%s: 0x%08x != 0x%08x" % (_name(path, cols, r, c, a.shape), a[r, c], b[r, c]))
            if len(diffs) >= limit:
                return diffs
    return diffs


# ---- running the drop-in with the shim ----------------------------------------------------------------------------------------
@pytest.fixture(scope="session")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("shim")/"capture_shim.so")
    subprocess.run(["gcc", "-shared", "-fPIC", "-O1", "-I", os.path.join(ROOT, "include"), SHIM_SRC, "-o", so], check=True)
    return so


def run_dropin(shim, js, workdir):
    """Writes `js` (integrator type switched to b200_path_tracer) into workdir and runs the drop-in on it with the capture shim.
    Returns (exit code, output, Side or None)."""
    js = json.loads(json.dumps(js))
    js.setdefault("integrator", {})["type"] = "b200_path_tracer"
    path = os.path.join(workdir, "b200.json")
    with open(path, "w") as f:
        json.dump(js, f)
    cap = os.path.join(workdir, "capture.bin")
    if os.path.exists(cap):
        os.remove(cap)
    env = dict(os.environ, LD_PRELOAD=shim, TGB_CAPTURE=cap)
    r = subprocess.run([EXE, "-t", "1", "-d", os.path.join(workdir, "out"), path], env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=600)
    side = None
    if os.path.exists(cap):
        with open(cap, "rb") as f:
            side = read_capture(f.read())
    return r.returncode, r.stdout, side


def capture(shim, js, workdir):
    rc, log, side = run_dropin(shim, js, workdir)
    assert side is not None, "no capture file: the shim's tgb200_create did not take over (exit %d)\n%s" % (rc, log[-2000:])
    assert rc == 0, log[-2000:]
    return side


def check_equal(name, got_side, fs, devices=False):
    got, want = Canon(got_side, devices), Canon(read_flat(fs), devices)
    diffs = compare(got, want)
    print("%s: %d primitives, %d bsdf records, %d texture records, %d words compared"
          % (name, want.n_primitives, want.n_bsdfs, want.n_textures, want.n_words))
    assert not diffs, "%s: the adapter's desc differs from the flattener's (adapter != flattener):\n  " % name + "\n  ".join(diffs)
    return want


def _geometry_words(fs):
    """Every vertex, triangle, curve node and curve segment of the flattener's primitives, as 32-bit words (texels are counted
    by the texture records that reach them)."""
    n = 0
    for p in fs.primitives:
        n += 8*p.n_verts + 4*p.n_tris + 4*p.n_curve_nodes + p.n_curve_segments
    return n


# ---- (a) the fixtures ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_desc_matches_flattener(name, shim, tmp_path):
    """tests/golden/<name>/scene.json through both builders.  hair_sky: the adapter's skydome texels are the reference's own
    prepared 512x256 sky image, the flattener's are the committed scene_sky.pfm."""
    src = os.path.join(G, name)
    for f in os.listdir(src):
        if f != "scene.json":
            os.symlink(os.path.join(src, f), tmp_path/f)
    with open(os.path.join(src, "scene.json")) as f:
        js = json.load(f)
    fs = scene.load_scene(os.path.join(src, "scene.json"))
    want = check_equal(name, capture(shim, js, str(tmp_path)), fs)
    assert want.n_words >= _geometry_words(fs)


# ---- (b) the zoo: what the fixtures do not reach -----------------------------------------------------------------------------
def _write_png(path, rgb8):
    """8-bit RGB PNG (no filter, one IDAT): an LDR bitmap for the refusal table."""
    h, w, _ = rgb8.shape
    raw = b"".join(b"\0" + rgb8[y].tobytes() for y in range(h))

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)
    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0))
                + chunk(b"IDAT", zlib.compress(raw)) + chunk(b"IEND", b""))


def _zoo_files(d):
    rng = np.random.RandomState(7)
    # a mesh of 240 triangles with unit normals pointing every way, materials 0..2 plus out-of-range -1 and 7
    nv, nt = 300, 240
    v = np.zeros(nv, scene.VERTEX_DTYPE)
    v["pos"] = rng.uniform(-1.0, 1.0, (nv, 3)).astype(np.float32)
    n = rng.normal(size=(nv, 3)); v["normal"] = (n/np.linalg.norm(n, axis=1, keepdims=True)).astype(np.float32)
    v["uv"] = rng.uniform(0.0, 1.0, (nv, 2)).astype(np.float32)
    t = np.zeros(nt, scene.TRI_DTYPE)
    for k, c in enumerate(("v0", "v1", "v2")):
        t[c] = (np.arange(nt) + 37*k) % nv
    t["material"] = np.array([0, 1, 2, -1, 7], np.int32)[np.arange(nt) % 5]
    scene.save_wo3(os.path.join(d, "zoo_mesh.wo3"), v, t)
    # an emissive mesh: two triangles
    lv = np.zeros(4, scene.VERTEX_DTYPE)
    lv["pos"] = [[-0.5, 0, -0.5], [0.5, 0, -0.5], [0.5, 0, 0.5], [-0.5, 0, 0.5]]
    lv["normal"] = [0, -1, 0]; lv["uv"] = [[0, 0], [1, 0], [1, 1], [0, 1]]
    lt = np.zeros(2, scene.TRI_DTYPE); lt["v0"], lt["v1"], lt["v2"] = [0, 0], [1, 2], [2, 3]
    scene.save_wo3(os.path.join(d, "zoo_lamp.wo3"), lv, lt)
    # bitmaps of non-power-of-two sizes (PFM) and an RGBE environment
    scene.save_pfm(os.path.join(d, "tex_5x3.pfm"), rng.uniform(0.0, 2.0, (3, 5, 3)).astype(np.float32))
    scene.save_pfm(os.path.join(d, "tex_7x6.pfm"), rng.uniform(0.0, 1.0, (6, 7, 3)).astype(np.float32))
    shutil.copy(os.path.join(G, "coat_env", "scene_env.hdr"), os.path.join(d, "env.hdr"))
    # curves: 6 strands of 4..9 nodes with their own widths
    counts = np.array([4, 9, 5, 7, 6, 8]); ends = np.cumsum(counts).astype(np.uint32)
    nodes = np.zeros((int(ends[-1]), 4), np.float32)
    nodes[:, :3] = rng.uniform(-0.5, 0.5, (len(nodes), 3)); nodes[:, 3] = rng.uniform(0.005, 0.02, len(nodes))
    scene.save_fiber(os.path.join(d, "zoo.fiber"), ends, nodes)
    _write_png(os.path.join(d, "ldr.png"), rng.randint(0, 256, (3, 5, 3)).astype(np.uint8))


def _bitmap(f, interp, clamp):
    return {"type": "bitmap", "file": f, "interpolate": interp, "clamp": clamp}


def zoo_scene(filt="tent"):
    conductors = [{"name": "rc_" + m, "type": "rough_conductor", "material": m, "roughness": 0.25}
                  for m in sorted(scene.COMPLEX_IOR)]
    bsdfs = conductors + [
        {"name": "checker", "type": "lambert",
         "albedo": {"type": "checker", "on_color": [0.9, 0.6, 0.1], "off_color": [0.05, 0.2, 0.7], "res_u": 7, "res_v": 3}},
        {"name": "rc_default", "type": "rough_conductor", "distribution": "beckmann", "roughness": 0.3, "albedo": [0.9, 0.8, 0.7]},
        {"name": "rc_etak", "type": "rough_conductor", "distribution": "phong", "roughness": 0.07,
         "eta": [1.1, 0.3, 2.7], "k": [0.4, 5.5, 1.25]},
        {"name": "rc_eta_only", "type": "rough_conductor", "eta": [1.9, 1.3, 0.7]},
        {"name": "rc_k_only", "type": "rough_conductor", "k": [2.5, 3.5, 4.5]},
        {"name": "cd_default", "type": "conductor"},
        {"name": "cd_etak", "type": "conductor", "eta": [0.3, 0.6, 0.9], "k": [3.1, 2.1, 1.1]},
        {"name": "cd_eta_only", "type": "conductor", "eta": [0.35, 0.65, 0.95]},
        {"name": "cd_au", "type": "conductor", "material": "Au"},
        {"name": "mirror", "type": "mirror", "albedo": [0.95, 0.9, 0.85]},
        {"name": "glass_nort", "type": "dielectric", "ior": 1.33, "enable_refraction": False},
        {"name": "glass", "type": "dielectric", "ior": 1.7},
        {"name": "rglass_b", "type": "rough_dielectric", "ior": 1.45, "distribution": "beckmann", "roughness": 0.2,
         "enable_refraction": False},
        {"name": "rglass_p", "type": "rough_dielectric", "ior": 2.1, "distribution": "phong", "roughness": 0.05},
        {"name": "plastic", "type": "plastic", "ior": 1.4, "thickness": 0.5, "sigma_a": [0.1, 0.2, 0.3],
         "albedo": _bitmap("tex_7x6.pfm", True, False)},
        {"name": "rplastic", "type": "rough_plastic", "ior": 1.6, "thickness": 2.5, "sigma_a": 0.75, "distribution": "phong",
         "roughness": 0.15, "albedo": [0.2, 0.5, 0.3]},
        {"name": "rplastic_bm", "type": "rough_plastic", "distribution": "beckmann", "roughness": 0.4},
        {"name": "coat_inline", "type": "smooth_coat", "ior": 1.55, "thickness": 0.3, "sigma_a": [0.5, 0.1, 0.05],
         "substrate": {"type": "rough_conductor", "material": "Cr", "distribution": "ggx", "roughness": 0.12}},
        {"name": "coat_named", "type": "smooth_coat", "substrate": "checker"},
        {"name": "rcoat_inline", "type": "rough_coat", "ior": 1.45, "thickness": 0.8, "sigma_a": [0.05, 0.3, 0.6],
         "distribution": "beckmann", "roughness": 0.08, "substrate": {"type": "lambert", "albedo": [0.6, 0.2, 0.1]}},
        {"name": "rcoat_named", "type": "rough_coat", "distribution": "phong", "roughness": 0.2, "substrate": "rplastic"},
        {"name": "rcoat_default", "type": "rough_coat"},
        {"name": "hair_sigma", "type": "hair", "sigma_a": [0.3, 0.8, 1.9], "scale_angle": 3.5, "roughness": 0.25},
        {"name": "hair_melanin", "type": "hair", "melanin_ratio": 0.3, "melanin_concentration": 1.7, "roughness": 0.4},
        {"name": "null", "type": "null"},
        {"name": "scalar", "type": "lambert", "albedo": 0.35},
        {"name": "unused", "type": "lambert", "albedo": [0.1, 0.9, 0.1]},
        {"name": "rc_bitmap_rough", "type": "rough_conductor", "roughness": _bitmap("tex_7x6.pfm", False, True)},
    ]
    quad_forms = [
        [0.7, 0.0, 0.3, 1.0, 0.2, -1.1, 0.0, 2.0, -0.4, 0.0, 1.9, -3.0, 0.0, 0.0, 0.0, 1.0],      # matrix
        {"position": [0.1, 0.2, 0.3], "rotation": [12.5, -40.0, 73.0], "scale": [2.0, 0.5, 3.0]},
        {"position": [-1.0, 2.0, 0.5], "look_at": [0.3, -0.4, 2.0], "up": [0.2, 1.0, 0.1], "scale": [0.4, 1.0, 1.5]},
        {"position": [0.5, 0.0, -2.0], "x_axis": [1.0, 0.2, 0.0], "z_axis": [0.0, 0.3, 1.0]},
        {"y_axis": [0.0, 0.2, 1.0], "rotation": [90.0, 0.0, 180.0]},
        {"scale": -1.5},
    ]
    prims = [{"type": "quad", "transform": t, "bsdf": b} for t, b in zip(quad_forms, ["checker", "mirror", "scalar", "plastic",
                                                                                     "coat_named", "rc_default"])]
    for k, (interp, clamp) in enumerate([(True, False), (True, True), (False, False), (False, True)]):
        f = "tex_5x3.pfm" if k % 2 == 0 else "tex_7x6.pfm"
        prims.append({"type": "quad", "transform": {"position": [k, 0, 0], "rotation": [0, 30.0*k, 0]},
                      "bsdf": {"type": "lambert", "albedo": _bitmap(f, interp, clamp)}})
        prims.append({"type": "quad", "transform": {"position": [k, 1, 0], "scale": [1.0, 1.0, 0.5 + k]}, "bsdf": "null",
                      "emission": _bitmap(f, interp, clamp)})
    prims += [
        {"type": "cube", "transform": {"position": [1.0, -2.0, 0.5], "rotation": [33.0, -71.0, 128.0], "scale": [0.3, 1.7, 0.9]},
         "bsdf": "rglass_b"},
        {"type": "cube", "transform": [0.0, -2.0, 0.0, 1.0, 0.5, 0.0, 0.0, 0.0, 0.0, 0.0, 3.0, 0.0, 0.0, 0.0, 0.0, 1.0], "bsdf": "glass"},
        {"type": "mesh", "file": "zoo_mesh.wo3", "smooth": True, "bsdf": ["rc_Au", "coat_inline", "rcoat_named"],
         "transform": {"position": [0.0, 1.0, -1.0], "rotation": [-17.0, 25.0, 61.0], "scale": [-1.5, 0.75, 2.25]}},
        {"type": "mesh", "file": "zoo_mesh.wo3", "bsdf": "rplastic",
         "transform": [2.0, 0.1, 0.0, 0.0, 0.0, -0.5, 0.3, 1.0, 0.2, 0.0, 1.25, 0.0, 0.0, 0.0, 0.0, 1.0]},
        {"type": "mesh", "file": "zoo_lamp.wo3", "bsdf": "null", "emission": [4.0, 3.5, 2.0],
         "transform": {"position": [0.0, 3.0, 0.0], "scale": [1.3, 1.0, 0.7]}},
        {"type": "curves", "file": "zoo.fiber", "mode": "cylinder", "bsdf": "scalar", "curve_thickness": 0.013,
         "curve_taper": True, "subsample": 0.35,
         "transform": {"position": [0.2, 0.5, 0.1], "rotation": [10.0, 20.0, 30.0], "scale": [1.0, 2.5, 0.6]}},
        {"type": "curves", "file": "zoo.fiber", "mode": "bcsdf_cylinder", "bsdf": "hair_melanin", "curve_taper": True,
         "transform": {"scale": [0.8, 1.2, 1.7]}},
        {"type": "curves", "file": "zoo.fiber", "bsdf": "hair_sigma", "subsample": 0.6},
        {"name": "pivot", "type": "quad", "bsdf": "rcoat_inline",
         "transform": {"position": [5.0, 5.0, 5.0], "rotation": [-31.0, 47.0, 12.0], "scale": [1.0, 3.0, 0.5]}},
        {"type": "infinite_sphere_cap", "skydome": "pivot", "emission": [50.0, 45.0, 40.0], "cap_angle": 3.7, "sample": False},
        {"type": "infinite_sphere_cap", "transform": {"rotation": [20.0, 0.0, -65.0]}, "emission": 20.0, "cap_angle": 12.0},
        {"type": "infinite_sphere", "transform": {"rotation": [0.0, 137.0, -12.0]}, "emission": "env.hdr"},
    ]
    prims += [{"type": "quad", "transform": {"position": [0, -3, float(k)]}, "bsdf": b}
              for k, b in enumerate(["rc_etak", "rc_eta_only", "rc_k_only", "cd_default", "cd_etak", "cd_eta_only", "cd_au",
                                     "glass_nort", "rglass_p", "rplastic_bm", "rcoat_default", "rc_bitmap_rough"]
                                    + [c["name"] for c in conductors])]
    return {
        "bsdfs": bsdfs, "primitives": prims,
        "camera": {"type": "pinhole", "resolution": [37, 23], "fov": 47.5, "reconstruction_filter": filt,
                   "transform": {"position": [0.3, 1.7, 6.1], "look_at": [-0.2, 0.4, 0.0], "up": [0.1, 1.0, 0.0]}},
        "integrator": {"type": "path_tracer", "min_bounces": 2, "max_bounces": 7, "enable_light_sampling": False,
                       "enable_two_sided_shading": False, "enable_consistency_checks": True},
        "renderer": {"spp": 4, "spp_step": 4, "stratified_sampler": True, "adaptive_sampling": False,
                     "output_file": "out.png", "hdr_output_file": "out.pfm", "overwrite_output_files": True},
    }


# (filter, integrator "devices"): each filter once; the device list in both of its forms on two of them
ZOO_VARIANTS = [("dirac", None), ("box", [0, 1]), ("tent", 2), ("gaussian", None), ("mitchell_netravali", None),
                ("catmull_rom", None), ("lanczos", None)]


@pytest.mark.parametrize("filt,devices", ZOO_VARIANTS, ids=[v[0] for v in ZOO_VARIANTS])
def test_zoo_desc_matches_flattener(filt, devices, shim, tmp_path):
    _zoo_files(str(tmp_path))
    js = zoo_scene(filt)
    fs = scene.load_scene(json.loads(json.dumps(js)), base_dir=str(tmp_path))
    if devices is not None:
        js["integrator"]["devices"] = devices
        # what lib.Context(fs, devices=...) puts into the flattener's desc
        lst = devices if isinstance(devices, list) else list(range(devices))
        fs.settings.n_devices = len(lst)
        for i, dv in enumerate(lst):
            fs.settings.devices[i] = dv
    assert fs.camera.filter == scene._FILTER[filt]
    want = check_equal("zoo/" + filt, capture(shim, js, str(tmp_path)), fs, devices=devices is not None)
    assert want.n_words >= _geometry_words(fs)


# ---- refusals ------------------------------------------------------------------------------------------------------------------
def _with_bsdf(extra):
    def f(js):
        js["primitives"][0]["bsdf"] = dict({"type": "lambert"}, **extra)
    return f


def _power(js):
    del js["primitives"][0]["emission"]
    js["primitives"][0]["power"] = 10.0


def _medium(js):
    js["media"] = [{"name": "fog", "type": "homogeneous", "sigma_a": 0.1, "sigma_s": 0.2}]
    js["primitives"][0]["int_medium"] = "fog"


def _camera_type(js):
    js["camera"]["type"] = "thinlens"


def _output_buffer(js):
    js["renderer"]["output_buffers"] = [{"type": "depth", "hdr_output_file": "depth.pfm"}]


def _ribbon(js):
    js["primitives"].append({"type": "curves", "file": "zoo.fiber", "mode": "ribbon", "bsdf": "scalar"})


def _conductor(material):
    return _with_bsdf({"type": "conductor", "material": material})


# (input, mutation of a small scene, the flattener raises SceneError, the adapter refuses, why the two may differ)
REFUSALS = [
    ("bump map", _with_bsdf({"bump": {"type": "checker"}}), True, True, None),
    ("ribbon curves", _ribbon, True, True, None),
    ("medium", _medium, True, True, None),
    ("thinlens camera", _camera_type, True, True, None),
    ("power emitter", _power, True, False,
     "the adapter reads the emission the reference derives from `power` in Primitive::prepareForRender; the flattener does "
     "not restate each primitive's power-to-radiance factor"),
    ("constant bump", _with_bsdf({"bump": 0.5}), True, False,
     "a constant bump map leaves the shading frame alone (Primitive::setupTangentFrame), so the adapter lets it through; the "
     "flattener refuses every `bump`"),
    ("conductor material outside the flattener's table", _conductor("Ni"), True, False,
     "the adapter reads eta/k from the reference's full ComplexIorData table; the flattener carries the six metals the shipped "
     "scenes use"),
    ("LDR bitmap", _with_bsdf({"albedo": "ldr.png"}), True, False,
     "the adapter reads the texels the reference decoded and linearised; the flattener has no LDR decoder"),
    ("feature output buffer", _output_buffer, False, True,
     "the flattener has no notion of output buffers: it never writes the image, its caller does"),
]


def _small_scene():
    js = zoo_scene()
    js["primitives"] = [{"type": "quad", "transform": {"scale": 2.0}, "bsdf": "scalar", "emission": 1.0},
                        {"type": "quad", "transform": {"position": [0, 1, 0]}, "bsdf": "checker"}]
    return js


@pytest.mark.parametrize("case", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_refusal_matches_flattener(case, shim, tmp_path):
    """Out-of-scope inputs: where the flattener accepts, the adapter accepts with the identical desc; where the adapter refuses,
    it does so before tgb200_create: no capture file and the adapter's "b200_path_tracer: ..." failure in the log.  (The
    reference's render loop logs a scene's runtime_error as "encountered an unrecoverable error" and goes on to the next scene,
    tungsten/Shared.hpp:325-328, so the process still exits with 0.)  Each row where the two builders disagree carries its
    reason."""
    name, mutate, py_refuses, adapter_refuses, why = case
    assert (py_refuses == adapter_refuses) == (why is None)
    _zoo_files(str(tmp_path))
    js = _small_scene()
    mutate(js)
    try:
        fs = scene.load_scene(json.loads(json.dumps(js)), base_dir=str(tmp_path))
        py_err = None
    except scene.SceneError as e:
        fs, py_err = None, e
    rc, log, side = run_dropin(shim, js, str(tmp_path))
    refused = side is None
    assert rc == 0, log[-2000:]
    if refused:
        assert "encountered an unrecoverable error" in log and "b200_path_tracer:" in log, \
            "%s: no capture and no refusal by the adapter:\n%s" % (name, log[-2000:])
    print("%s: flattener %s, adapter %s" % (name, "refuses (%s)" % py_err if py_err else "accepts",
                                           "refuses" if refused else "accepts"))
    assert (py_err is not None) == py_refuses, name
    assert refused == adapter_refuses, name + ("" if refused else ": adapter accepted") + "\n" + log[-2000:]
    if fs is not None and side is not None:
        check_equal("refusals/" + name, side, fs)
