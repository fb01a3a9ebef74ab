"""Scene flattener: Tungsten scene JSON (+ .wo3 meshes, HDR/PFM bitmaps) -> POD `tgb_scene_desc`.

Host-side mirror of what the reference does between `Scene::load` and the end of the
`TraceableScene` constructor for the subset of objects on the path_tracer hot path
(reference: src/core/io/Scene.cpp:236-253,281,373; io/JsonPtr.cpp:108-186 transform parsing;
math/Mat4f.cpp:10,118; primitives/{Quad.cpp:298-305,Cube.cpp:351-355,TriangleMesh.cpp:524-552,
InfiniteSphere.cpp prepareForRender}; cameras/Camera.cpp:44-68).

All arithmetic is done in IEEE fp32 with the reference's operation order (numpy float32 scalars
and arrays, libm's cosf/sinf through ctypes), so the world-space floats handed to the C ABI are the
ones the reference computes for the same JSON.  This module contains no rendering code.
"""
import ctypes as C
import ctypes.util
import json
import os
import struct

import numpy as np

from . import abi

f32 = np.float32
_libm = C.CDLL(ctypes.util.find_library("m") or "libm.so.6")
for _n in ("cosf", "sinf", "tanf"):
    getattr(_libm, _n).restype = C.c_float
    getattr(_libm, _n).argtypes = [C.c_float]

PI = f32(3.1415926536)


def _cosf(x): return f32(_libm.cosf(float(x)))
def _sinf(x): return f32(_libm.sinf(float(x)))


class SceneError(ValueError):
    """Scene uses something outside the hot path (maps to TGB_ERR_UNSUPPORTED)."""


# ---- tiny fp32 vector helpers with the reference's operation order (math/Vec.hpp) -------------
def v3(x, y=None, z=None):
    if y is None:
        if np.ndim(x) == 0:
            return np.array([x, x, x], dtype=f32)
        return np.array(x, dtype=f32)
    return np.array([x, y, z], dtype=f32)


def dot(a, b):
    s = f32(a[0]*b[0]); s = f32(s + f32(a[1]*b[1])); s = f32(s + f32(a[2]*b[2])); return s


def cross(a, b):
    return v3(f32(a[1]*b[2]) - f32(a[2]*b[1]), f32(a[2]*b[0]) - f32(a[0]*b[2]), f32(a[0]*b[1]) - f32(a[1]*b[0]))


def length(a): return f32(np.sqrt(dot(a, a)))


def normalized(a):
    inv = f32(f32(1.0)/length(a))
    return v3(a[0]*inv, a[1]*inv, a[2]*inv)


def mat4_mul(a, b):
    r = np.zeros((4, 4), dtype=f32)
    for i in range(4):
        for t in range(4):
            s = f32(a[i, 0]*b[0, t]); s = f32(s + f32(a[i, 1]*b[1, t]))
            s = f32(s + f32(a[i, 2]*b[2, t])); s = f32(s + f32(a[i, 3]*b[3, t]))
            r[i, t] = s
    return r


def mat4_point(m, p):   # Mat4f*Vec3f (math/Mat4f.hpp:320-327)
    return v3(*[f32(f32(f32(f32(m[i, 0]*p[0]) + f32(m[i, 1]*p[1])) + f32(m[i, 2]*p[2])) + m[i, 3]) for i in range(3)])


def mat4_vector(m, p):  # Mat4f::transformVector (math/Mat4f.hpp:159-166)
    return v3(*[f32(f32(f32(m[i, 0]*p[0]) + f32(m[i, 1]*p[1])) + f32(m[i, 2]*p[2])) for i in range(3)])


def rot_yxz(rot):       # Mat4f::rotYXZ (math/Mat4f.cpp:118-131)
    r = v3(rot)*PI/f32(180.0)
    c = [_cosf(r[0]), _cosf(r[1]), _cosf(r[2])]
    s = [_sinf(r[0]), _sinf(r[1]), _sinf(r[2])]
    m = np.eye(4, dtype=f32)
    m[0, 0] = f32(c[1]*c[2]) - f32(f32(s[1]*s[0])*s[2]); m[0, 1] = f32(f32(-c[1])*s[2]) - f32(f32(s[1]*s[0])*c[2]); m[0, 2] = f32(f32(-s[1])*c[0])
    m[1, 0] = f32(c[0]*s[2]); m[1, 1] = f32(c[0]*c[2]); m[1, 2] = f32(-s[0])
    m[2, 0] = f32(s[1]*c[2]) + f32(f32(c[1]*s[0])*s[2]); m[2, 1] = f32(f32(-s[1])*s[2]) + f32(f32(c[1]*s[0])*c[2]); m[2, 2] = f32(c[1]*c[0])
    return m


def quat_from_matrix(a):      # QuaternionF::fromMatrix (math/Quaternion.hpp:111-146); a = 3x3 rotation, fp32
    a = np.asarray(a, dtype=f32)
    trace = f32(f32(a[0, 0] + a[1, 1]) + a[2, 2])
    if trace > 0.0:
        s = f32(f32(0.5)/np.sqrt(f32(trace + f32(1.0))))
        return np.array([f32(f32(0.25)/s), f32(f32(a[2, 1] - a[1, 2])*s), f32(f32(a[0, 2] - a[2, 0])*s), f32(f32(a[1, 0] - a[0, 1])*s)], dtype=f32)
    if a[0, 0] > a[1, 1] and a[0, 0] > a[2, 2]:
        s = f32(f32(2.0)*np.sqrt(f32(f32(f32(f32(1.0) + a[0, 0]) - a[1, 1]) - a[2, 2])))
        return np.array([f32(f32(a[2, 1] - a[1, 2])/s), f32(f32(0.25)*s), f32(f32(a[0, 1] + a[1, 0])/s), f32(f32(a[0, 2] + a[2, 0])/s)], dtype=f32)
    if a[1, 1] > a[2, 2]:
        s = f32(f32(2.0)*np.sqrt(f32(f32(f32(f32(1.0) + a[1, 1]) - a[0, 0]) - a[2, 2])))
        return np.array([f32(f32(a[0, 2] - a[2, 0])/s), f32(f32(a[0, 1] + a[1, 0])/s), f32(f32(0.25)*s), f32(f32(a[1, 2] + a[2, 1])/s)], dtype=f32)
    s = f32(f32(2.0)*np.sqrt(f32(f32(f32(f32(1.0) + a[2, 2]) - a[0, 0]) - a[1, 1])))
    return np.array([f32(f32(a[1, 0] - a[0, 1])/s), f32(f32(a[0, 2] + a[2, 0])/s), f32(f32(a[1, 2] + a[2, 1])/s), f32(f32(0.25)*s)], dtype=f32)


def quat_mul(a, o):            # Quaternion::operator*(Quaternion) (math/Quaternion.hpp:68-76)
    return np.array([
        f32(f32(f32(a[0]*o[0]) - f32(a[1]*o[1])) - f32(a[2]*o[2])) - f32(a[3]*o[3]),
        f32(f32(f32(a[0]*o[1]) + f32(a[1]*o[0])) + f32(a[2]*o[3])) - f32(a[3]*o[2]),
        f32(f32(f32(a[0]*o[2]) - f32(a[1]*o[3])) + f32(a[2]*o[0])) + f32(a[3]*o[1]),
        f32(f32(f32(a[0]*o[3]) + f32(a[1]*o[2])) - f32(a[2]*o[1])) + f32(a[3]*o[0])], dtype=f32)


def quat_rotate(q, o):         # Quaternion::operator*(Vec3) (math/Quaternion.hpp:78-88), vectorised over rows of o
    o = np.asarray(o, dtype=f32)
    two = f32(2.0)
    tx = two*(q[2]*o[:, 2] - q[3]*o[:, 1]); ty = two*(q[3]*o[:, 0] - q[1]*o[:, 2]); tz = two*(q[1]*o[:, 1] - q[2]*o[:, 0])
    r = np.empty_like(o)
    r[:, 0] = ((o[:, 0] + q[0]*tx) + q[2]*tz) - q[3]*ty
    r[:, 1] = ((o[:, 1] + q[0]*ty) + q[3]*tx) - q[1]*tz
    r[:, 2] = ((o[:, 2] + q[0]*tz) + q[1]*ty) - q[2]*tx
    return r


def _random_ortho(a):   # io/JsonPtr.cpp:78-89
    if abs(a[0]) > abs(a[1]):
        res = v3(0.0, 1.0, 0.0)
    else:
        res = v3(1.0, 0.0, 0.0)
    return normalized(cross(a, res))


def _gram_schmidt(a, b, c):  # io/JsonPtr.cpp:91-106 (in-place on the three arrays)
    a[:] = normalized(a)
    b[:] = b - a*dot(a, b)
    if dot(b, b) < 1e-5:
        b[:] = _random_ortho(a)
    else:
        b[:] = normalized(b)
    c[:] = c - a*dot(a, c)
    c[:] = c - b*dot(b, c)
    if dot(c, c) < 1e-5:
        c[:] = cross(a, b)
    else:
        c[:] = normalized(c)


def _vec3_field(obj, key, default=None):
    if key not in obj:
        return None if default is None else v3(default)
    v = obj[key]
    if isinstance(v, (int, float)):
        return v3(f32(v))
    if len(v) != 3:
        raise SceneError("expected a Vec3 for '%s'" % key)
    return v3([f32(x) for x in v])


def parse_transform(t):
    """JsonPtr::get(Mat4f&) (io/JsonPtr.cpp:108-186)."""
    if t is None:
        return np.eye(4, dtype=f32)
    if isinstance(t, list):
        if len(t) != 16:
            raise SceneError("matrix needs 16 elements")
        return np.array([f32(x) for x in t], dtype=f32).reshape(4, 4)
    x, y, z = v3(1.0, 0.0, 0.0), v3(0.0, 1.0, 0.0), v3(0.0, 0.0, 1.0)
    pos = _vec3_field(t, "position", 0.0)
    ex = ey = ez = False
    if "look_at" in t:
        z = _vec3_field(t, "look_at") - pos
        ez = True
    if "up" in t:
        y = _vec3_field(t, "up"); ey = True
    if "x_axis" in t:
        x = _vec3_field(t, "x_axis"); ex = True
    if "y_axis" in t:
        y = _vec3_field(t, "y_axis"); ey = True
    if "z_axis" in t:
        z = _vec3_field(t, "z_axis"); ez = True
    ident = (4 if ez else 0) + (2 if ey else 0) + (1 if ex else 0)
    order = {0: (z, y, x), 1: (x, z, y), 2: (y, z, x), 3: (y, x, z), 4: (z, y, x), 5: (z, x, y),
             6: (z, y, x), 7: (z, y, x)}[ident]
    _gram_schmidt(*order)
    if dot(cross(x, y), z) < 0.0:
        if not ex:
            x = -x
        elif not ey:
            y = -y
        else:
            z = -z
    if "scale" in t:
        sc = _vec3_field(t, "scale")
        x = x*sc[0]; y = y*sc[1]; z = z*sc[2]
    if "rotation" in t:
        tf = rot_yxz(_vec3_field(t, "rotation"))
        x = mat4_point(tf, x); y = mat4_point(tf, y); z = mat4_point(tf, z)
    m = np.eye(4, dtype=f32)
    m[:3, 0] = x; m[:3, 1] = y; m[:3, 2] = z; m[:3, 3] = pos
    return m


# ---- resources --------------------------------------------------------------------------------
VERTEX_DTYPE = np.dtype([("pos", "<f4", 3), ("normal", "<f4", 3), ("uv", "<f4", 2)])
TRI_DTYPE = np.dtype([("v0", "<u4"), ("v1", "<u4"), ("v2", "<u4"), ("material", "<i4")])


def load_wo3(path):
    """io/MeshIO.cpp:12-28: u64 nVerts, Vertex[nVerts] (32 B), u64 nTris, TriangleI[nTris] (16 B)."""
    with open(path, "rb") as f:
        nv = struct.unpack("<Q", f.read(8))[0]
        verts = np.frombuffer(f.read(32*nv), dtype=VERTEX_DTYPE).copy()
        nt = struct.unpack("<Q", f.read(8))[0]
        tris = np.frombuffer(f.read(16*nt), dtype=TRI_DTYPE).copy()
    return verts, tris


def save_wo3(path, verts, tris):
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(verts))); f.write(np.ascontiguousarray(verts, dtype=VERTEX_DTYPE).tobytes())
        f.write(struct.pack("<Q", len(tris))); f.write(np.ascontiguousarray(tris, dtype=TRI_DTYPE).tobytes())


_FIBER_MAGIC = bytes([0x80, 0xBF, 0x80, 0x46, 0x49, 0x42, 0x45, 0x52])
_FIBER_SIZES = [1, 1, 2, 2, 4, 4, 8, 8, 4, 8]


def load_fiber(path):
    """`.fiber` curve file (io/CurveIO.cpp:343-403): returns (curve_ends uint32[n_curves], nodes float32[n_nodes,4]);
    node width is 0 where the file has no `width` attribute (CurveIO leaves it to `curve_thickness`)."""
    import struct
    with open(path, "rb") as f:
        data = f.read()
    if data[:8] != _FIBER_MAGIC:
        raise SceneError("%s: not a .fiber file" % path)
    major, _minor, content = struct.unpack_from("<HHI", data, 8)
    if major != 1 or content != 0:
        raise SceneError("%s: unsupported .fiber version/content" % path)
    header_len, n_verts, n_curves = struct.unpack_from("<QQQ", data, 16)
    ends, nodes = None, np.zeros((n_verts, 4), np.float32)
    off = header_len
    while True:
        (desc_len,) = struct.unpack_from("<Q", data, off)
        if desc_len == 0:
            break
        data_len, flags, vtype, vper = struct.unpack_from("<QHBB", data, off + 8)
        name_end = data.index(b"\0", off + 20)
        name = data[off + 20:name_end].decode()
        off += desc_len
        present = data_len//(_FIBER_SIZES[vtype]*vper) if vtype < len(_FIBER_SIZES) and vper else 0
        per_curve = bool(flags & 1)

        def column(dtype, need):     # FiberAttribute::load: copy-extend a short attribute (:332-341)
            a = np.frombuffer(data, dtype=dtype, count=present*vper, offset=off).reshape(present, vper)
            if present < need:
                a = np.concatenate([a, np.repeat(a[-1:], need - present, axis=0)])
            return a[:need]
        if present > 0:
            if name == "num_vertices" and per_curve and vtype == 3 and vper == 1:
                ends = np.cumsum(column("<u2", n_curves)[:, 0].astype(np.uint64)).astype(np.uint32)
            elif name == "position" and not per_curve and vtype == 8 and vper == 3:
                nodes[:, :3] = column("<f4", n_verts)
            elif name == "width" and not per_curve and vtype == 8 and vper == 1:
                nodes[:, 3] = column("<f4", n_verts)[:, 0]
        off += data_len
    if ends is None:
        raise SceneError("%s: no num_vertices attribute" % path)
    return ends, nodes


def save_fiber(path, curve_ends, nodes):
    """Writes what load_fiber / CurveIO::loadFiber read back (per-curve node counts, positions, widths)."""
    import struct
    ends = np.asarray(curve_ends, np.uint32); nodes = np.asarray(nodes, np.float32)
    counts = np.diff(np.concatenate([[0], ends])).astype("<u2")
    blocks = [("num_vertices", 1, 3, 1, counts.tobytes()),
              ("position", 0, 8, 3, np.ascontiguousarray(nodes[:, :3], "<f4").tobytes()),
              ("width", 0, 8, 1, np.ascontiguousarray(nodes[:, 3], "<f4").tobytes())]
    out = bytearray(_FIBER_MAGIC) + struct.pack("<HHI", 1, 0, 0) + struct.pack("<QQQ", 40, len(nodes), len(ends))
    for name, flags, vtype, vper, payload in blocks:
        nm = name.encode() + b"\0"
        out += struct.pack("<QQHBB", 20 + len(nm), len(payload), flags, vtype, vper) + nm + payload
    out += struct.pack("<Q", 0)
    with open(path, "wb") as f:
        f.write(bytes(out))


def load_pfm(path):
    """Returns (h, w, 3) float32, top row first (io/ImageIO.cpp:528-544 writes rows bottom-up)."""
    with open(path, "rb") as f:
        kind = f.readline().strip()
        if kind not in (b"PF", b"Pf"):
            raise SceneError("not a PFM file: %s" % path)
        w, h = [int(x) for x in f.readline().split()]
        scale = float(f.readline())
        ch = 3 if kind == b"PF" else 1
        data = np.frombuffer(f.read(4*w*h*ch), dtype="<f4" if scale < 0 else ">f4").astype(np.float32)
    img = data.reshape(h, w, ch)[::-1]
    if ch == 1:
        img = np.repeat(img, 3, axis=2)
    return np.ascontiguousarray(img)


def save_pfm(path, img):
    img = np.asarray(img, dtype="<f4")
    with open(path, "wb") as f:
        f.write(b"PF\n%d %d\n-1.0\n" % (img.shape[1], img.shape[0]))
        f.write(np.ascontiguousarray(img[::-1]).tobytes())


def load_rgbe(path):
    """Radiance .hdr (RGBE, flat or new-style RLE).  Decode rule follows stb_image's
    stbi__hdr_convert used by the reference (thirdparty/stbi/stb_image.c): f = ldexp(1, e-(128+8)),
    rgb = mantissa*f; e == 0 -> black."""
    with open(path, "rb") as f:
        data = f.read()
    pos = 0
    def readline():
        nonlocal pos
        end = data.index(b"\n", pos); line = data[pos:end]; pos = end + 1; return line
    if not readline().startswith(b"#?"):
        raise SceneError("not a Radiance HDR file: %s" % path)
    while True:
        line = readline()
        if line == b"":
            break
    res = readline().split()
    if res[0] != b"-Y" or res[2] != b"+X":
        raise SceneError("unsupported HDR orientation")
    h, w = int(res[1]), int(res[3])
    rgbe = np.zeros((h, w, 4), dtype=np.uint8)
    buf = np.frombuffer(data, dtype=np.uint8)
    for y in range(h):
        if w < 8 or w >= 32768 or not (buf[pos] == 2 and buf[pos + 1] == 2 and not (buf[pos + 2] & 0x80)):
            rgbe[y:] = buf[pos:pos + 4*w*(h - y)].reshape(h - y, w, 4); break
        pos += 4
        for c in range(4):
            x = 0
            while x < w:
                n = int(buf[pos]); pos += 1
                if n > 128:
                    n -= 128; rgbe[y, x:x + n, c] = buf[pos]; pos += 1
                else:
                    rgbe[y, x:x + n, c] = buf[pos:pos + n]; pos += n
                x += n
    e = rgbe[..., 3].astype(np.int32)
    scale = np.where(e != 0, np.ldexp(np.float32(1.0), e - 136), np.float32(0.0)).astype(np.float32)
    return (rgbe[..., :3].astype(np.float32)*scale[..., None]).astype(np.float32)


# Named conductors used by shipped scenes (bsdfs/ComplexIorData.hpp); scenes may also give eta/k directly.
COMPLEX_IOR = {
    "Ag": ((0.1552646489, 0.1167232965, 0.1383806959), (4.8283433224, 3.1222459278, 2.1469504455)),
    "Al": ((1.6574599595, 0.8803689579, 0.5212287346), (9.2238691996, 6.2695232477, 4.8370012281)),
    "Au": ((0.1431189557, 0.3749570432, 1.4424785571), (3.9831604247, 2.3857207478, 1.6032152899)),
    "Cr": ((4.3696828663, 2.9167024892, 1.6547005413), (5.2064337956, 4.2313645277, 3.7549467933)),
    "Cu": ((0.2004376970, 0.9240334304, 1.1022119527), (3.9129485033, 2.4528477015, 2.1421879552)),
    "W":  ((4.3707029924, 3.3002972445, 2.9982666528), (3.5006778591, 2.6048652781, 2.2731930614)),
}


def _conductor_eta_k(b):
    """(eta, k) of a conductor / rough_conductor: ConductorBsdf::fromJson (ConductorBsdf.cpp:37-40), RoughConductorBsdf::fromJson
    (RoughConductorBsdf.cpp:35-39).  The constructors' own (rounded) copper constants (ConductorBsdf.cpp:20-26,
    RoughConductorBsdf.cpp:17-25); `value.getField("eta", _eta) &&
    value.getField("k", _k)` stores a given eta even when k is missing, and reads k only behind an eta; the table is consulted
    only when "material" is given, and then replaces both."""
    eta, k = (0.200438, 0.924033, 1.10221), (3.91295, 2.45285, 2.14219)
    if "eta" in b:
        eta = _vec3_field(b, "eta")
        if "k" in b:
            k = _vec3_field(b, "k")
    if "material" in b:
        if b["material"] not in COMPLEX_IOR:
            raise SceneError("conductor material '%s' not in the table" % b["material"])
        eta, k = COMPLEX_IOR[b["material"]]
    return eta, k


_CURVE_MODE = {"cylinder": abi.CURVE_CYLINDER, "half_cylinder": abi.CURVE_HALF_CYLINDER, "bcsdf_cylinder": abi.CURVE_BCSDF_CYLINDER}
_DIST = {"beckmann": abi.DIST_BECKMANN, "phong": abi.DIST_PHONG, "ggx": abi.DIST_GGX}
_FILTER = {"dirac": abi.FILTER_DIRAC, "box": abi.FILTER_BOX, "tent": abi.FILTER_TENT,
           "gaussian": abi.FILTER_GAUSSIAN, "mitchell_netravali": abi.FILTER_MITCHELL,
           "catmull_rom": abi.FILTER_CATMULL_ROM, "lanczos": abi.FILTER_LANCZOS}


class FlatScene:
    """Owns the numpy/ctypes storage behind a `tgb_scene_desc` (keeps every buffer alive)."""

    def __init__(self):
        self.textures, self.bsdfs, self.primitives, self.slots = [], [], [], []
        self._keep = []
        self.camera = abi.Camera()
        self.settings = abi.Settings(min_bounces=0, max_bounces=64, enable_light_sampling=1,
                                     enable_two_sided_shading=1, enable_consistency_checks=0,
                                     use_sobol=1, supplemental_mode=0, device=-1, max_paths_in_flight=0)
        self.spp, self.spp_step = 32, 16
        self.adaptive = True
        self.n_triangles = 0
        self.source = None

    # -- textures / bsdfs ------------------------------------------------------------------------
    def add_texture_constant(self, rgb):
        t = abi.Texture(type=abi.TEX_CONSTANT); t.value[:] = [float(f32(x)) for x in v3(rgb)]
        self.textures.append(t); return len(self.textures) - 1

    def add_texture(self, value, base_dir=".", average=False):
        """Scene::fetchTexture (io/Scene.cpp:127-151).  average: the texel conversion is TexelConversion::REQUEST_AVERAGE
        (roughness textures, e.g. RoughConductorBsdf.cpp:42) rather than REQUEST_RGB; only bitmaps honour it (Scene.cpp:130-133)."""
        if isinstance(value, (int, float)):
            return self.add_texture_constant(f32(value))
        if isinstance(value, list):
            return self.add_texture_constant([f32(x) for x in value])
        if isinstance(value, str):
            value = {"type": "bitmap", "file": value}
        ty = value.get("type")
        if ty == "constant":
            return self.add_texture(value.get("value", 0.0), base_dir)
        if ty == "checker":
            t = abi.Texture(type=abi.TEX_CHECKER)
            t.value[:] = [float(x) for x in (_vec3_field(value, "on_color") if "on_color" in value else v3(0.8))]
            t.value2[:] = [float(x) for x in (_vec3_field(value, "off_color") if "off_color" in value else v3(0.2))]
            t.res_u = int(value.get("res_u", 20)); t.res_v = int(value.get("res_v", 20))
            self.textures.append(t); return len(self.textures) - 1
        if ty == "bitmap":
            path = os.path.join(base_dir, value["file"])
            ext = os.path.splitext(path)[1].lower()
            if ext == ".pfm":
                img = load_pfm(path)
            elif ext == ".hdr":
                img = load_rgbe(path)
            else:
                raise SceneError("bitmap format outside the hot path: %s" % ext)
            if average:
                # a scalar bitmap: each texel (r + g + b)/3 in fp32 (io/ImageIO.cpp:179, applied by loadPfm/loadHdr :335,361),
                # looked up as Vec3f(scalar) (BitmapTexture.cpp:326-345)
                img = np.repeat(((img[..., 0:1] + img[..., 1:2]) + img[..., 2:3])/f32(3.0), 3, axis=2)
            if value.get("gamma_correct", True) is False:
                pass  # HDR inputs are linear either way (BitmapTexture: gamma only applies to LDR)
            return self.add_bitmap_texture(img, value.get("interpolate", True), value.get("clamp", False))
        raise SceneError("texture type outside the hot path: %r" % ty)

    def add_bitmap_texture(self, img, linear=True, clamp=False):
        """BitmapTexture over in-memory RGB fp32 texels, shape (h, w, 3), top row first (textures/BitmapTexture.cpp:52-59)."""
        img = np.ascontiguousarray(img, dtype=np.float32)
        if img.ndim != 3 or img.shape[2] != 3:
            raise SceneError("bitmap texels must have shape (h, w, 3)")
        self._keep.append(img)
        t = abi.Texture(type=abi.TEX_BITMAP, res_u=img.shape[1], res_v=img.shape[0])
        t.flags = (1 if linear else 0) | (2 if clamp else 0)
        t.texels = img.ctypes.data_as(C.POINTER(C.c_float))
        self.textures.append(t); return len(self.textures) - 1

    def add_bsdf(self, b, base_dir=".", named=None):
        ty = b.get("type", "lambert")
        o = abi.Bsdf(albedo_tex=self.add_texture(b.get("albedo", 1.0), base_dir), roughness_tex=-1,
                     substrate=-1, ior=1.5, thickness=1.0, enable_refraction=1, distribution=abi.DIST_GGX)
        if ty == "null":
            o.type = abi.BSDF_NULL
        elif ty == "lambert":
            o.type = abi.BSDF_LAMBERT
        elif ty == "rough_conductor":
            o.type = abi.BSDF_ROUGH_CONDUCTOR
            eta, k = _conductor_eta_k(b)
            o.eta[:] = [float(f32(x)) for x in eta]; o.k[:] = [float(f32(x)) for x in k]
            o.distribution = _DIST[b.get("distribution", "ggx")]
            o.roughness_tex = self.add_texture(b.get("roughness", 0.1), base_dir, average=True)
        elif ty == "mirror":
            o.type = abi.BSDF_MIRROR
        elif ty == "conductor":
            o.type = abi.BSDF_CONDUCTOR
            eta, k = _conductor_eta_k(b)
            o.eta[:] = [float(f32(x)) for x in eta]; o.k[:] = [float(f32(x)) for x in k]
        elif ty == "dielectric":
            o.type = abi.BSDF_DIELECTRIC
            o.ior = float(f32(b.get("ior", 1.5)))
            o.enable_refraction = 1 if b.get("enable_refraction", True) else 0
        elif ty == "rough_dielectric":
            o.type = abi.BSDF_ROUGH_DIELECTRIC
            o.ior = float(f32(b.get("ior", 1.5)))
            o.distribution = _DIST[b.get("distribution", "ggx")]
            o.enable_refraction = 1 if b.get("enable_refraction", True) else 0
            o.roughness_tex = self.add_texture(b.get("roughness", 0.1), base_dir, average=True)
        elif ty in ("plastic", "rough_plastic"):
            o.type = abi.BSDF_PLASTIC if ty == "plastic" else abi.BSDF_ROUGH_PLASTIC
            o.ior = float(f32(b.get("ior", 1.5)))
            o.thickness = float(f32(b.get("thickness", 1.0)))
            o.sigma_a[:] = [float(x) for x in (_vec3_field(b, "sigma_a") if "sigma_a" in b else v3(0.0))]
            if ty == "rough_plastic":
                o.distribution = _DIST[b.get("distribution", "ggx")]
                o.roughness_tex = self.add_texture(b.get("roughness", 0.02), base_dir, average=True)
        elif ty in ("smooth_coat", "rough_coat"):
            o.type = abi.BSDF_SMOOTH_COAT if ty == "smooth_coat" else abi.BSDF_ROUGH_COAT
            if ty == "rough_coat":                     # RoughCoatBsdf ctor (RoughCoatBsdf.cpp:15-23): ggx, roughness 0.02
                o.distribution = _DIST[b.get("distribution", "ggx")]
                o.roughness_tex = self.add_texture(b.get("roughness", 0.02), base_dir, average=True)
            o.ior = float(f32(b.get("ior", 1.3)))
            o.thickness = float(f32(b.get("thickness", 1.0)))
            o.sigma_a[:] = [float(x) for x in (_vec3_field(b, "sigma_a") if "sigma_a" in b else v3(0.0))]
            sub = b.get("substrate", {"type": "rough_conductor"})
            if isinstance(sub, str):
                if named is None or sub not in named:
                    raise SceneError("unknown substrate bsdf '%s'" % sub)
                o.substrate = named[sub]
            else:
                o.substrate = self.add_bsdf(sub, base_dir, named)
            if self.bsdfs[o.substrate].type in (abi.BSDF_SMOOTH_COAT, abi.BSDF_ROUGH_COAT):
                raise SceneError("nested coats are outside the hot path")
        elif ty == "hair":
            # HairBcsdf ctor defaults + fromJson + the sigma_a part of prepareForRender (bsdfs/HairBcsdf.cpp:13-21,163-171,435-443)
            o.type = abi.BSDF_HAIR
            o.hair_scale_angle_deg = float(f32(b.get("scale_angle", 2.0)))
            o.hair_roughness = float(f32(b.get("roughness", 0.1)))
            if "sigma_a" in b:
                sa = _vec3_field(b, "sigma_a")
            else:
                ratio, conc = f32(b.get("melanin_ratio", 0.5)), f32(b.get("melanin_concentration", 0.25))
                eu, pheo = v3(0.419, 0.697, 1.37), v3(0.187, 0.4, 1.05)
                sa = conc*(eu*(f32(1.0) - ratio) + pheo*ratio)
            o.sigma_a[:] = [float(f32(x)) for x in sa]
        else:
            raise SceneError("bsdf type outside the hot path: %r" % ty)
        if "bump" in b:
            raise SceneError("bump maps are outside the hot path")
        self.bsdfs.append(o)
        return len(self.bsdfs) - 1

    # -- primitives ------------------------------------------------------------------------------
    def _emission(self, p, base_dir):
        if "power" in p:
            raise SceneError("'power' emitters are outside the hot path (use 'emission')")
        return self.add_texture(p["emission"], base_dir) if "emission" in p else -1

    def add_quad(self, transform, bsdf, emission_tex=-1):
        """Quad::prepareForRender (primitives/Quad.cpp:298-305)."""
        m = transform
        base = mat4_point(m, v3(0.0))
        edge0 = mat4_vector(m, v3(1.0, 0.0, 0.0)); edge1 = mat4_vector(m, v3(0.0, 0.0, 1.0))
        base = base - edge0*f32(0.5); base = base - edge1*f32(0.5)
        p = abi.Primitive(type=abi.PRIM_QUAD, emission_tex=emission_tex, bsdf_first=len(self.slots), bsdf_count=1)
        p.base[:] = [float(x) for x in base]; p.edge0[:] = [float(x) for x in edge0]; p.edge1[:] = [float(x) for x in edge1]
        self.slots.append(bsdf); self.primitives.append(p)

    def add_cube(self, transform, bsdf, emission_tex=-1):
        """Cube::prepareForRender (primitives/Cube.cpp:351-355); Mat4f::extractRotation/extractScale."""
        m = transform
        right, up, fwd = v3(m[:3, 0]), v3(m[:3, 1]), v3(m[:3, 2])
        pos = mat4_point(m, v3(0.0))
        scale = v3(f32(length(right)*f32(0.5)), f32(length(up)*f32(0.5)), f32(length(fwd)*f32(0.5)))
        rot = np.stack([normalized(right), normalized(up), normalized(fwd)], axis=1)   # columns
        p = abi.Primitive(type=abi.PRIM_CUBE, emission_tex=emission_tex, bsdf_first=len(self.slots), bsdf_count=1)
        p.pos[:] = [float(x) for x in pos]; p.scale[:] = [float(x) for x in scale]
        p.rot[:] = [float(x) for x in rot.reshape(-1)]
        self.slots.append(bsdf); self.primitives.append(p)

    def add_mesh(self, transform, verts, tris, bsdfs, smooth=False, emission_tex=-1):
        """TriangleMesh::prepareForRender (primitives/TriangleMesh.cpp:524-552): world-space _tfVerts."""
        m = transform
        pos = verts["pos"].astype(np.float32); nrm = verts["normal"].astype(np.float32)
        out = np.zeros(len(verts), dtype=VERTEX_DTYPE)
        for i in range(3):
            out["pos"][:, i] = ((m[i, 0]*pos[:, 0] + m[i, 1]*pos[:, 1]) + m[i, 2]*pos[:, 2]) + m[i, 3]
        # Mat4f::toNormalMatrix (math/Mat4f.cpp:10-13): scale(1/|col|^2) * M  (rows scaled)
        inv = [f32(1.0)/dot(v3(m[:3, c]), v3(m[:3, c])) for c in range(3)]
        for i in range(3):
            r = [f32(inv[i]*m[i, c]) for c in range(3)]
            out["normal"][:, i] = (r[0]*nrm[:, 0] + r[1]*nrm[:, 1]) + r[2]*nrm[:, 2]
        out["uv"] = verts["uv"]
        t = np.ascontiguousarray(tris, dtype=TRI_DTYPE).copy()
        t["material"] = np.clip(t["material"], 0, max(len(bsdfs) - 1, 0))
        self._keep += [out, t]
        p = abi.Primitive(type=abi.PRIM_MESH, emission_tex=emission_tex, smooth=1 if smooth else 0,
                          bsdf_first=len(self.slots), bsdf_count=len(bsdfs), n_verts=len(out), n_tris=len(t))
        p.verts = out.ctypes.data_as(C.POINTER(abi.Vertex)); p.tris = t.ctypes.data_as(C.POINTER(abi.Triangle))
        self.slots += list(bsdfs); self.primitives.append(p)
        self.n_triangles += len(t)

    def add_instances(self, transform, masters, ids, inst_transforms):
        """Instance primitive (primitives/Instance.cpp:54-75,392-420): rigid copies (quaternion + translation, no scale) of
        master meshes.  HBM-first: with 80 GB of HBM the instances are simply FLATTENED into one world-space triangle
        mesh (no two-level BVH, no per-ray transform): world = pos_i + rot_i*(master_transform*v), exactly the point
        the reference reaches through `Instance::intersectionInfo` (Instance.cpp:325-334).
        masters: list of (verts, tris, bsdf_index, smooth, master_transform); ids: master index per instance;
        inst_transforms: (n, 4, 4) float32."""
        m = transform
        rot_p = quat_from_matrix(np.stack([normalized(v3(m[:3, 0])), normalized(v3(m[:3, 1])), normalized(v3(m[:3, 2]))], axis=1))
        prepared = []
        for (verts, tris, bsdf, smooth, mt) in masters:
            pos = verts["pos"].astype(np.float32); nrm = verts["normal"].astype(np.float32)
            wp = np.zeros_like(pos); wn = np.zeros_like(nrm)
            for i in range(3):
                wp[:, i] = ((mt[i, 0]*pos[:, 0] + mt[i, 1]*pos[:, 1]) + mt[i, 2]*pos[:, 2]) + mt[i, 3]
            inv = [f32(1.0)/dot(v3(mt[:3, c]), v3(mt[:3, c])) for c in range(3)]
            for i in range(3):
                r = [f32(inv[i]*mt[i, c]) for c in range(3)]
                wn[:, i] = (r[0]*nrm[:, 0] + r[1]*nrm[:, 1]) + r[2]*nrm[:, 2]
            prepared.append((wp, wn, verts["uv"].astype(np.float32), tris, bsdf, smooth))
        vparts, tparts, bsdfs, voff = [], [], [], 0
        smooth_any = any(p[5] for p in prepared)
        for k, mid in enumerate(ids):
            wp, wn, uv, tris, bsdf, smooth = prepared[int(mid)]
            it = np.asarray(inst_transforms[k], dtype=np.float32)
            ipos = v3(it[:3, 3])
            irot = quat_from_matrix(np.stack([normalized(v3(it[:3, 0])), normalized(v3(it[:3, 1])), normalized(v3(it[:3, 2]))], axis=1))
            p_w = mat4_point(m, ipos)                             # _instancePos[i] = _transform*_instancePos[i]
            q_w = quat_mul(rot_p, irot)                           # _instanceRot[i] = rot*_instanceRot[i]
            out = np.zeros(len(wp), dtype=VERTEX_DTYPE)
            out["pos"] = quat_rotate(q_w, wp) + p_w[None, :]
            out["normal"] = quat_rotate(q_w, wn)
            out["uv"] = uv
            t = np.array(tris, dtype=TRI_DTYPE, copy=True)
            t["v0"] += voff; t["v1"] += voff; t["v2"] += voff
            if bsdf not in bsdfs:
                bsdfs.append(bsdf)
            t["material"] = bsdfs.index(bsdf)
            vparts.append(out); tparts.append(t); voff += len(out)
        verts = np.concatenate(vparts) if vparts else np.zeros(0, dtype=VERTEX_DTYPE)
        tris = np.concatenate(tparts) if tparts else np.zeros(0, dtype=TRI_DTYPE)
        self._keep += [verts, tris]
        p = abi.Primitive(type=abi.PRIM_MESH, emission_tex=-1, smooth=1 if smooth_any else 0,
                          bsdf_first=len(self.slots), bsdf_count=max(len(bsdfs), 1), n_verts=len(verts), n_tris=len(tris))
        p.verts = verts.ctypes.data_as(C.POINTER(abi.Vertex)); p.tris = tris.ctypes.data_as(C.POINTER(abi.Triangle))
        self.slots += list(bsdfs) if bsdfs else [0]
        self.primitives.append(p)
        self.n_triangles += len(tris)

    def add_curves(self, transform, curve_ends, nodes, bsdf, mode="half_cylinder", thickness=None, taper=False,
                   subsample=0.0, emission_tex=-1):
        """Curves::loadCurves + prepareForRender (primitives/Curves.cpp:268-296,572-611): thickness override / taper,
        nodes to world space (width times the mean scale), then the list of segments that survive `subsample`."""
        from .integrator import UniformSampler
        if mode not in _CURVE_MODE:
            raise SceneError("curve mode outside the hot path: %r" % mode)
        if self.bsdfs[bsdf].type == abi.BSDF_HAIR and emission_tex >= 0:
            raise SceneError("emissive curves are outside the hot path")
        ends = np.asarray(curve_ends, np.uint32); nd = np.array(nodes, np.float32, copy=True)
        starts = np.concatenate([[0], ends[:-1]]).astype(np.int64)
        if thickness is not None or taper:
            for i in range(len(ends)):
                s, e = int(starts[i]), int(ends[i])
                w = np.full(e - s, f32(thickness), np.float32) if thickness is not None else nd[s:e, 3].copy()
                if taper:
                    t = np.arange(e - s, dtype=np.float32)          # uint32 -> float, then the fp32 expression of :288
                    w = w*(f32(1.0) - (t - f32(0.5))/f32(e - s - 1))
                nd[s:e, 3] = w
        m = transform
        sx, sy, sz = length(v3(m[:3, 0])), length(v3(m[:3, 1])), length(v3(m[:3, 2]))
        width_scale = f32(f32(f32(sx + sy) + sz)*f32(1.0/3.0))                                  # Vec::avg()
        pos = nd[:, :3].copy()
        for i in range(3):
            nd[:, i] = ((m[i, 0]*pos[:, 0] + m[i, 1]*pos[:, 1]) + m[i, 2]*pos[:, 2]) + m[i, 3]
        nd[:, 3] = nd[:, 3]*width_scale
        rng = UniformSampler(0xBA5EBA11)                                                                   # UniformSampler() default seed
        segs = []
        for i in range(len(ends)):
            if subsample > 0.0:
                xi = f32(np.uint32((rng.next_i() >> 9) | 0x3F800000).view(np.float32) - f32(1.0))
                if xi < f32(subsample):
                    continue
            segs.append(np.arange(int(starts[i]) + 2, int(ends[i]), dtype=np.uint32))
        segs = np.concatenate(segs) if segs else np.zeros(0, np.uint32)
        nd = np.ascontiguousarray(nd); segs = np.ascontiguousarray(segs)
        self._keep += [nd, segs]
        p = abi.Primitive(type=abi.PRIM_CURVES, emission_tex=emission_tex, bsdf_first=len(self.slots), bsdf_count=1,
                          n_curve_nodes=len(nd), n_curve_segments=len(segs), curve_mode=_CURVE_MODE[mode])
        p.curve_nodes = nd.ctypes.data_as(C.POINTER(abi.f32)); p.curve_segments = segs.ctypes.data_as(C.POINTER(abi.u32))
        self.slots.append(bsdf); self.primitives.append(p)
        self.n_curve_segments = getattr(self, "n_curve_segments", 0) + len(segs)

    def add_infinite_sphere(self, transform, emission_tex, sample=True):
        m = transform
        rot = np.stack([normalized(v3(m[:3, 0])), normalized(v3(m[:3, 1])), normalized(v3(m[:3, 2]))], axis=1)
        p = abi.Primitive(type=abi.PRIM_INFINITE_SPHERE, emission_tex=emission_tex, do_sample=1 if sample else 0)
        p.rot[:] = [float(x) for x in rot.reshape(-1)]
        self.primitives.append(p)

    def add_infinite_sphere_cap(self, transform, emission_tex, sample=True, cap_angle_deg=10.0):
        """InfiniteSphereCap::prepareForRender (primitives/InfiniteSphereCap.cpp:231-247): cap direction = the transform's
        image of +y, normalised; cos of the cap angle through degToRad (math/Angle.hpp:19-22) and libm's cosf."""
        cap_dir = normalized(mat4_vector(transform, v3(0.0, 1.0, 0.0)))
        rad = f32(f32(cap_angle_deg)*f32(f32(PI)/f32(180.0)))
        p = abi.Primitive(type=abi.PRIM_INFINITE_SPHERE_CAP, emission_tex=emission_tex, do_sample=1 if sample else 0)
        p.cap_dir[:] = [float(x) for x in cap_dir]; p.cap_cos = float(_cosf(rad))
        self.primitives.append(p)

    def add_skydome(self, sky_texels, sample=True):
        """Skydome (primitives/Skydome.cpp): an environment sphere looked up WITHOUT rotation whose emission is the 512x256
        image Skydome::prepareForRender computes from the Hosek-Wilkie model (thirdparty/skylight).  That model is not
        restated here: the caller passes the prepared image (the C++ adapter reads it from the live Skydome object, tests
        use an image dumped from the reference)."""
        tex = self.add_bitmap_texture(np.ascontiguousarray(sky_texels, dtype=np.float32), True, False)
        p = abi.Primitive(type=abi.PRIM_SKYDOME, emission_tex=tex, do_sample=1 if sample else 0)
        p.rot[:] = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0]
        self.primitives.append(p)

    def set_camera(self, cam, base_dir="."):
        """Camera::fromJson + PinholeCamera::fromJson (cameras/Camera.cpp:44-68, PinholeCamera.cpp:37-43)."""
        if cam.get("type", "pinhole") != "pinhole":
            raise SceneError("camera type outside the hot path: %r" % cam.get("type"))
        if cam.get("medium") is not None:
            raise SceneError("camera media are outside the hot path")
        m = parse_transform(cam.get("transform"))
        m[:3, 0] = -m[:3, 0]                                    # _transform.setRight(-_transform.right())
        c = self.camera
        c.pos[:] = [float(m[0, 3]), float(m[1, 3]), float(m[2, 3])]
        c.xform[:] = [float(x) for x in m[:3, :3].reshape(-1)]
        c.fov_deg = float(f32(cam.get("fov", 60.0)))
        res = cam.get("resolution", [1000, 563])
        if isinstance(res, (int, float)):
            res = [res, res]
        c.res_x, c.res_y = int(res[0]), int(res[1])
        flt = cam.get("reconstruction_filter", "tent")
        if flt not in _FILTER:
            raise SceneError("unknown reconstruction filter %r" % flt)
        c.filter = _FILTER[flt]

    # -- finish ----------------------------------------------------------------------------------
    def desc(self):
        d = abi.SceneDesc(abi_version=abi.ABI_VERSION, camera=self.camera, settings=self.settings)
        self._prims = (abi.Primitive*max(len(self.primitives), 1))(*self.primitives)
        self._bsdfs = (abi.Bsdf*max(len(self.bsdfs), 1))(*self.bsdfs)
        self._texs = (abi.Texture*max(len(self.textures), 1))(*self.textures)
        self._slots = (C.c_uint32*max(len(self.slots), 1))(*self.slots)
        d.primitives = self._prims; d.n_primitives = len(self.primitives)
        d.bsdfs = self._bsdfs; d.n_bsdfs = len(self.bsdfs)
        d.textures = self._texs; d.n_textures = len(self.textures)
        d.bsdf_slots = self._slots; d.n_bsdf_slots = len(self.slots)
        return d

    @property
    def resolution(self):
        return self.camera.res_x, self.camera.res_y


def load_scene(path_or_dict, base_dir=None):
    """Scene::load + loadResources + the prepare step of TraceableScene for in-scope objects."""
    if isinstance(path_or_dict, dict):
        js = path_or_dict; base_dir = base_dir or "."
    else:
        with open(path_or_dict) as f:
            js = json.load(f)
        base_dir = base_dir or os.path.dirname(os.path.abspath(path_or_dict))
    if js.get("media"):
        raise SceneError("participating media are outside the hot path")
    fs = FlatScene(); fs.source = js
    named = {}
    for b in js.get("bsdfs", []):
        idx = fs.add_bsdf(b, base_dir, named)
        if "name" in b:
            named[b["name"]] = idx

    def fetch_bsdf(v):
        if isinstance(v, str):
            if v not in named:
                raise SceneError("unknown bsdf '%s'" % v)
            return named[v]
        return fs.add_bsdf(v, base_dir, named)

    default_bsdf = None
    for p in js.get("primitives", []):
        ty = p.get("type")
        if p.get("int_medium") is not None or p.get("ext_medium") is not None:
            raise SceneError("participating media are outside the hot path")
        tf = parse_transform(p.get("transform"))
        if ty == "infinite_sphere":
            fs.add_infinite_sphere(tf, fs._emission(p, base_dir), p.get("sample", True))
            continue
        if ty == "infinite_sphere_cap":
            if p.get("skydome"):                                  # pivot object: the cap follows that primitive's transform
                piv = [q for q in js.get("primitives", []) if q.get("name") == p["skydome"]]
                if piv:
                    tf = parse_transform(piv[0].get("transform"))
            fs.add_infinite_sphere_cap(tf, fs._emission(p, base_dir), p.get("sample", True), p.get("cap_angle", 10.0))
            continue
        if ty == "skydome":
            if "sky_image" not in p:
                raise SceneError("skydome: the Hosek-Wilkie sky model is outside the hot path; pass the prepared image as 'sky_image' (PFM)")
            fs.add_skydome(load_pfm(os.path.join(base_dir, p["sky_image"])), p.get("sample", True))
            continue
        if ty == "instances":
            masters = []
            for mp in p.get("masters", []):
                if mp.get("type") != "mesh":
                    raise SceneError("instance masters other than meshes are outside the hot path")
                mb = mp.get("bsdf")
                if isinstance(mb, list):
                    raise SceneError("multi-material instance masters are outside the hot path")
                mv, mt_ = load_wo3(os.path.join(base_dir, mp["file"]))
                masters.append((mv, mt_, fetch_bsdf(mb) if mb is not None else fs.add_bsdf({"type": "lambert"}),
                                mp.get("smooth", False), parse_transform(mp.get("transform"))))
            inst = p.get("instances", [])
            if isinstance(inst, str) or "instancesA" in p or "instancesB" in p:
                raise SceneError("binary instance files are outside the hot path (list the instances inline)")
            ids = [int(i.get("id", 0)) for i in inst]
            its = np.stack([parse_transform(i.get("transform")) for i in inst]) if inst else np.zeros((0, 4, 4), np.float32)
            fs.add_instances(tf, masters, ids, its)
            continue
        if "bsdf" in p:
            bs = p["bsdf"]
            bsdfs = [fetch_bsdf(b) for b in bs] if isinstance(bs, list) else [fetch_bsdf(bs)]
        else:
            if default_bsdf is None:
                default_bsdf = fs.add_bsdf({"type": "lambert"})   # Primitive::_defaultBsdf
            bsdfs = [default_bsdf]
        em = fs._emission(p, base_dir)
        if ty == "quad":
            fs.add_quad(tf, bsdfs[0], em)
        elif ty == "cube":
            fs.add_cube(tf, bsdfs[0], em)
        elif ty == "curves":
            ends, nodes = load_fiber(os.path.join(base_dir, p["file"]))
            fs.add_curves(tf, ends, nodes, bsdfs[0], p.get("mode", "half_cylinder"),
                          f32(p["curve_thickness"]) if "curve_thickness" in p else None, p.get("curve_taper", False),
                          float(p.get("subsample", 0.0)), em)
        elif ty == "mesh":
            if p.get("recompute_normals", False) and p.get("smooth", False):
                raise SceneError("recompute_normals is outside the hot path (bake normals into the .wo3)")
            verts, tris = load_wo3(os.path.join(base_dir, p["file"]))
            fs.add_mesh(tf, verts, tris, bsdfs, p.get("smooth", False), em)
        else:
            raise SceneError("primitive type outside the hot path: %r" % ty)
    fs.set_camera(js.get("camera", {}), base_dir)
    it = js.get("integrator", {})
    if it.get("type", "path_tracer") != "path_tracer":
        raise SceneError("integrator outside the hot path: %r" % it.get("type"))
    s = fs.settings
    s.min_bounces = int(it.get("min_bounces", 0)); s.max_bounces = int(it.get("max_bounces", 64))
    s.enable_light_sampling = 1 if it.get("enable_light_sampling", True) else 0
    s.enable_two_sided_shading = 1 if it.get("enable_two_sided_shading", True) else 0
    s.enable_consistency_checks = 1 if it.get("enable_consistency_checks", False) else 0
    r = js.get("renderer", {})
    s.use_sobol = 1 if r.get("stratified_sampler", True) else 0
    fs.spp = int(r.get("spp", 32)); fs.spp_step = int(r.get("spp_step", 16))
    fs.adaptive = bool(r.get("adaptive_sampling", True))
    return fs
