"""The C-ABI shared library: loads, exports every symbol include/tgb200.h declares, struct layouts agree with
the ctypes mirror, and every compute entry point fails loudly (never falls back) without a GPU."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from tungsten_b200 import abi, lib, scene, synth, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "include", "tgb200.h")


def _declared_functions():
    txt = open(HDR).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(tgb200_[a-z_0-9]+)\s*\(", txt)))


def test_library_is_built_in_tree():
    assert os.path.exists(build.build()), "libtgb200.so must be built in-tree"
    assert os.path.dirname(lib.LIB_PATH) == os.path.join(ROOT, "tungsten_b200")


def test_exports_every_declared_symbol():
    L = lib.load()
    names = _declared_functions()
    assert len(names) >= 15
    for n in names:
        assert hasattr(L, n), "libtgb200.so does not export %s" % n
    assert sorted(abi.EXPORTS) == names
    assert L.tgb200_abi_version() == abi.ABI_VERSION


def test_struct_layouts_match_header():
    structs = {"tgb_texture": abi.Texture, "tgb_bsdf": abi.Bsdf, "tgb_vertex": abi.Vertex, "tgb_triangle": abi.Triangle,
               "tgb_primitive": abi.Primitive, "tgb_camera": abi.Camera, "tgb_settings": abi.Settings,
               "tgb_scene_desc": abi.SceneDesc, "tgb_tile": abi.Tile, "tgb_ray": abi.Ray, "tgb_hit": abi.Hit,
               "tgb_stats": abi.Stats}
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "tgb200.h"\nint main(){\n'
    for n in structs:
        src += 'printf("%s %%zu\\n", sizeof(%s));\n' % (n, n)
    src += 'printf("off_prim_base %zu\\n", offsetof(tgb_primitive, base));\n'
    src += 'printf("off_desc_textures %zu\\n", offsetof(tgb_scene_desc, textures));\n return 0; }\n'
    d = tempfile.mkdtemp()
    open(os.path.join(d, "s.c"), "w").write(src)
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "s.c"), "-o", os.path.join(d, "s")])
    out = dict(l.split() for l in subprocess.check_output([os.path.join(d, "s")], text=True).strip().splitlines())
    for n, cls in structs.items():
        assert int(out[n]) == C.sizeof(cls), n
    assert int(out["off_prim_base"]) == abi.Primitive.base.offset
    assert int(out["off_desc_textures"]) == abi.SceneDesc.textures.offset
    assert C.sizeof(abi.Vertex) == 32 and C.sizeof(abi.Triangle) == 16      # == .wo3 on-disk records


def test_no_cpu_fallback_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    fs = scene.load_scene(synth.cornell_box(res=(16, 16), spp=1))
    with pytest.raises(lib.TgbError) as e:
        lib.Context(fs)
    assert e.value.code == abi.TGB_ERR_NO_DEVICE
    assert "no CPU fallback" in str(e.value)


def test_create_rejects_bad_input():
    L = lib.load()
    h = C.c_void_p()
    assert L.tgb200_create(None, C.byref(h)) == abi.TGB_ERR_INVALID
    fs = scene.load_scene(synth.cornell_box(res=(16, 16), spp=1))
    d = fs.desc(); d.abi_version = 99
    assert L.tgb200_create(C.byref(d), C.byref(h)) == abi.TGB_ERR_INVALID
    assert b"ABI version" in L.tgb200_last_error(None)
    d = fs.desc(); d.settings.use_sobol = 0
    assert L.tgb200_create(C.byref(d), C.byref(h)) == abi.TGB_ERR_UNSUPPORTED
    d = fs.desc(); d.settings.supplemental_mode = 1
    assert L.tgb200_create(C.byref(d), C.byref(h)) == abi.TGB_ERR_UNSUPPORTED
    assert L.tgb200_get_stats(None, None) == abi.TGB_ERR_INVALID
    assert L.tgb200_abort(None) == abi.TGB_ERR_INVALID
    L.tgb200_destroy(None)     # must be a no-op


def test_probe_hooks_refuse_a_missing_context():
    """The test hooks (tests/test_gpu_lobes.py) return TGB_ERR_INVALID for a NULL context before touching a device."""
    L = lib.load()
    buf = np.zeros(16, np.float32); ids = np.zeros(1, np.int32); pix = np.zeros(1, np.uint32)
    assert L.tgb200_bsdf_probe(None, 0, 0.0, 0.0, 0, 0, 1, buf.ctypes.data, buf.ctypes.data) == abi.TGB_ERR_INVALID
    assert L.tgb200_bsdf_sample_probe(None, 0, 1, ids.ctypes.data, pix.ctypes.data, 0, 0.0, 0.0, 0, 0, buf.ctypes.data,
                                      buf.ctypes.data, pix.ctypes.data) == abi.TGB_ERR_INVALID
    assert L.tgb200_light_probe(None, 0, 0, 1, 0, buf.ctypes.data, buf.ctypes.data) == abi.TGB_ERR_INVALID
    assert L.tgb200_choose_light_probe(None, 0, 1, pix.ctypes.data, 0, buf.ctypes.data, buf.ctypes.data) == abi.TGB_ERR_INVALID
    lm = np.zeros(2, np.int32)
    assert L.tgb200_shadow_probe(None, 1, buf.ctypes.data, lm.ctypes.data, buf.ctypes.data) == abi.TGB_ERR_INVALID
    assert L.tgb200_shadow_probe(None, 0, None, None, None) == abi.TGB_ERR_INVALID
    st = np.zeros(abi.BOUNCE_WORDS, np.uint32)
    assert L.tgb200_bounce_probe(None, 1, st.ctypes.data, st.ctypes.data) == abi.TGB_ERR_INVALID
    assert L.tgb200_bounce_probe(None, 0, None, None) == abi.TGB_ERR_INVALID
    cur = np.zeros(abi.BINS, np.uint32); ns = C.c_uint32()
    assert L.tgb200_bin_probe(None, 1, pix.ctypes.data, pix.ctypes.data, cur.ctypes.data, C.byref(ns)) == abi.TGB_ERR_INVALID
    assert L.tgb200_bin_probe(None, 0, None, None, None, None) == abi.TGB_ERR_INVALID
    assert L.tgb200_shade_variant(None, pix.ctypes.data) == abi.TGB_ERR_INVALID


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "tungsten_b200")
    for dp, _, fns in os.walk(pkg):
        for fn in fns:
            if fn.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                txt = open(os.path.join(dp, fn), errors="ignore").read()
                assert "pt_oracle" not in txt and "pyoracle" not in txt and "from oracle" not in txt, fn
    so = subprocess.check_output(["ldd", lib.LIB_PATH], text=True)
    assert "oracle" not in so
