"""Every refusal of tgb200_create's scene preparation, reached without a GPU.

tgb200_create checks and prepares a desc on the host before it looks for a device, so a desc outside the hot path or malformed
gets its own code (TGB_ERR_INVALID / TGB_ERR_UNSUPPORTED) and reason on any machine.  Each case takes a valid desc from the
flattener, changes one field through the ctypes structs and expects one refusal; the unmodified descs still get
TGB_ERR_NO_DEVICE without a GPU and create a context with one.
"""
import ctypes as C
import functools

import pytest

from tungsten_b200 import abi, lib, scene, synth

INV, UNS = abi.TGB_ERR_INVALID, abi.TGB_ERR_UNSUPPORTED


@pytest.fixture(scope="module")
def flat(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("refusals"))
    makers = {
        "cornell_box": lambda: synth.cornell_box(res=(16, 16), spp=1),
        "cornell_mesh": lambda: synth.cornell_mesh(d, res=(16, 16), spp=1, subdiv=1),
        "env": lambda: synth.materialtest_standin(d, res=(16, 16), spp=1, subdiv=1, env_res=(32, 16)),
        "hair": lambda: synth.hair_scene(d, n_curves=4, nodes_per_curve=6, res=(16, 16), spp=1),
    }
    return functools.lru_cache(None)(lambda name: scene.load_scene(makers[name]()))


def create(d):
    L = lib.load()
    h = C.c_void_p()
    rc = L.tgb200_create(C.byref(d), C.byref(h))
    if rc == abi.TGB_OK:
        L.tgb200_destroy(h)
    return rc, L.tgb200_last_error(None).decode()


def gpu_present():
    import torch
    return torch.cuda.is_available()


def first(d, ptype):
    return next(i for i in range(d.n_primitives) if d.primitives[i].type == ptype)


def texture(d, ttype):
    return next(i for i in range(d.n_textures) if d.textures[i].type == ttype)


def glowing(d):
    """a constant texture that glows (its value is positive)"""
    return next(i for i in range(d.n_textures) if d.textures[i].type == abi.TEX_CONSTANT and max(d.textures[i].value) > 0)


def curve_bsdf(d):
    return d.bsdfs[d.bsdf_slots[d.primitives[first(d, abi.PRIM_CURVES)].bsdf_first]]


def set_fields(obj, **kw):
    for k, v in kw.items():
        setattr(obj, k, v)


def quad_as_hair(d):
    b = d.bsdfs[d.bsdf_slots[d.primitives[first(d, abi.PRIM_QUAD)].bsdf_first]]
    set_fields(b, type=abi.BSDF_HAIR, hair_roughness=0.3, hair_scale_angle_deg=2.5)


def mesh_material_1024(d):
    """a mesh with 1025 BSDF slots whose first triangle takes the last one"""
    m = d.primitives[first(d, abi.PRIM_MESH)]
    slots = list(d.bsdf_slots[:d.n_bsdf_slots])
    new = (C.c_uint32*(len(slots) + 1025))(*(slots + [slots[m.bsdf_first]]*1025))
    tris = (abi.Triangle*m.n_tris)(*m.tris[:m.n_tris])
    tris[0].material = 1024
    d.bsdf_slots, d.n_bsdf_slots = new, len(new)
    set_fields(m, bsdf_first=len(slots), bsdf_count=1025, tris=tris)


def curve_segment_zero(d):
    c = d.primitives[first(d, abi.PRIM_CURVES)]
    segs = (C.c_uint32*c.n_curve_segments)(*c.curve_segments[:c.n_curve_segments])
    segs[0] = 0
    c.curve_segments = segs


def env_checker(d):
    t = d.textures[d.primitives[first(d, abi.PRIM_INFINITE_SPHERE)].emission_tex]
    set_fields(t, type=abi.TEX_CHECKER, value=(abi.F3)(1, 1, 1), value2=(abi.F3)(1, 1, 1))


# (id, scene, change, code, reason) -- one row per refusal of the preparation step, in the order it makes them
CASES = [
    ("bitmap_without_texels", "env", lambda d: setattr(d.textures[texture(d, abi.TEX_BITMAP)], "texels", None), INV, "has no texels"),
    ("texture_type", "cornell_box", lambda d: setattr(d.textures[0], "type", 7), UNS, "texture type 7 is outside the hot path"),
    ("bsdf_type", "cornell_box", lambda d: setattr(d.bsdfs[0], "type", 40), UNS, "bsdf type 40 is outside the hot path"),
    ("albedo_texture", "cornell_box", lambda d: setattr(d.bsdfs[0], "albedo_tex", d.n_textures), INV, "bsdf 0: bad albedo texture"),
    ("roughness_texture", "cornell_box", lambda d: set_fields(d.bsdfs[0], type=abi.BSDF_ROUGH_CONDUCTOR, roughness_tex=-1), INV,
     "bsdf 0: bad roughness texture"),
    ("coat_substrate", "cornell_box", lambda d: set_fields(d.bsdfs[0], type=abi.BSDF_SMOOTH_COAT, substrate=0), UNS,
     "bsdf 0: a coat needs a substrate"),
    ("emission_texture", "cornell_box", lambda d: setattr(d.primitives[0], "emission_tex", d.n_textures), INV,
     "primitive 0: bad emission texture"),
    ("bsdf_range", "cornell_box", lambda d: setattr(d.primitives[first(d, abi.PRIM_QUAD)], "bsdf_count", 0), INV, "bad bsdf range"),
    ("bsdf_index", "cornell_box", lambda d: d.bsdf_slots.__setitem__(d.primitives[first(d, abi.PRIM_QUAD)].bsdf_first, d.n_bsdfs),
     INV, "bad bsdf index"),
    ("hair_on_a_quad", "cornell_box", quad_as_hair, UNS, "the hair BCSDF on a primitive that is not `curves`"),
    ("mesh_null_buffers", "cornell_mesh", lambda d: setattr(d.primitives[first(d, abi.PRIM_MESH)], "verts", None), INV,
     "has null buffers"),
    ("mesh_vertex_index", "cornell_mesh", lambda d: setattr(d.primitives[first(d, abi.PRIM_MESH)], "n_verts", 1), INV,
     "vertex index out of range"),
    ("mesh_materials", "cornell_mesh", mesh_material_1024, UNS, "more than 1024 materials in one mesh"),
    ("emissive_cube", "cornell_box", lambda d: setattr(d.primitives[first(d, abi.PRIM_CUBE)], "emission_tex", glowing(d)), UNS,
     "emissive cubes are outside the hot path"),
    ("sphere_cap_angle", "env", lambda d: set_fields(d.primitives[first(d, abi.PRIM_INFINITE_SPHERE)],
                                                     type=abi.PRIM_INFINITE_SPHERE_CAP, cap_cos=1.0), INV, "cap angle must be positive"),
    ("skydome_without_image", "cornell_box", lambda d: set_fields(d.primitives[first(d, abi.PRIM_QUAD)], type=abi.PRIM_SKYDOME,
                                                                  emission_tex=-1), INV, "pass the prepared sky image"),
    ("checker_environment", "env", env_checker, UNS, "checker environment maps are outside the hot path"),
    ("curve_mode", "hair", lambda d: setattr(d.primitives[first(d, abi.PRIM_CURVES)], "curve_mode", 9), UNS, "mode outside the hot path"),
    ("emissive_curves", "hair", lambda d: setattr(d.primitives[first(d, abi.PRIM_CURVES)], "emission_tex", glowing(d)), UNS,
     "emissive curves are outside the hot path"),
    ("curves_null_buffers", "hair", lambda d: setattr(d.primitives[first(d, abi.PRIM_CURVES)], "curve_nodes", None), INV,
     "has null buffers"),
    ("textured_curves", "hair", lambda d: setattr(d.textures[curve_bsdf(d).albedo_tex], "type", abi.TEX_CHECKER), UNS,
     "textured materials on curves are outside the hot path"),
    ("curve_segment_index", "hair", curve_segment_zero, INV, "segment index out of range"),
    ("primitive_type", "cornell_box", lambda d: setattr(d.primitives[first(d, abi.PRIM_QUAD)], "type", 42), UNS,
     "primitive type 42 is outside the hot path"),
    ("bitmap_sphere_cap", "env", lambda d: set_fields(d.primitives[first(d, abi.PRIM_INFINITE_SPHERE)],
                                                      type=abi.PRIM_INFINITE_SPHERE_CAP, cap_cos=0.5, do_sample=1), UNS,
     "bitmap emission on an infinite_sphere_cap"),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_desc_is_refused_before_the_device_query(case, flat):
    _, name, change, code, reason = case
    d = flat(name).desc()
    change(d)
    rc, err = create(d)
    assert rc == code, err
    assert reason in err


def test_too_deep_tree_is_refused_before_the_device_query(scratch, monkeypatch):
    """The 800-triangle stack of test_gpu_tree_shapes.py under TGB_TRI_LEAF=1: its tree needs more traversal stack than there is."""
    import test_gpu_tree_shapes as T
    fs, env = T.build_scene("too_deep", scratch)
    T._switches(monkeypatch, env, "16")
    rc, err = create(fs.desc())
    assert rc == UNS, err
    assert "exceeds the traversal stack" in err


@pytest.mark.parametrize("name", ["cornell_box", "cornell_mesh", "env", "hair"])
def test_unmodified_desc_reaches_the_device(name, flat):
    rc, err = create(flat(name).desc())
    if gpu_present():
        assert rc == abi.TGB_OK, err
    else:
        assert rc == abi.TGB_ERR_NO_DEVICE
        assert "no CPU fallback" in err
