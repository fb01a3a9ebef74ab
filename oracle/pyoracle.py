"""ctypes wrapper around oracle/_build/liboracle.so (CPU restatement; TEST INFRASTRUCTURE ONLY)."""
import ctypes as C
import os
import subprocess

import numpy as np

from tungsten_b200 import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

# BsdfLobes (bsdfs/BsdfLobes.hpp:13-34): the masks the probes take as `requested`
LOBE_GLOSSY_R, LOBE_GLOSSY_T, LOBE_DIFFUSE_R, LOBE_DIFFUSE_T, LOBE_SPEC_R, LOBE_SPEC_T, LOBE_ANISO, LOBE_FORWARD = \
    1, 2, 4, 8, 16, 32, 64, 128
LOBE_ALL = 2 | 8 | 32 | 1 | 4 | 16 | 64
LOBE_ALL_BUT_SPECULAR = 0xFFFFFFFF & ~(LOBE_SPEC_R | LOBE_SPEC_T | LOBE_FORWARD)


def build(force=False):
    so = os.path.join(_HERE, "_build", "liboracle.so")
    src = [os.path.join(_HERE, "pt_oracle.c"), os.path.join(_HERE, "pt_oracle.h"),
           os.path.join(_HERE, "..", "include", "tgb200.h")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in src):
        subprocess.check_call(["make", "-C", _HERE, "-s", "_build/liboracle.so"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        L.oracle_create.restype = C.c_void_p
        L.oracle_create.argtypes = [C.POINTER(abi.SceneDesc), C.c_void_p, C.c_char_p, C.c_int]
        L.oracle_destroy.argtypes = [C.c_void_p]
        L.oracle_render_tiles.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                          C.c_void_p, C.c_void_p, C.c_int, C.POINTER(abi.Stats)]
        L.oracle_trace_closest.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
        L.oracle_dice_tiles.restype = C.c_uint32
        L.oracle_dice_tiles.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
        L.oracle_hash32.restype = C.c_uint32; L.oracle_hash32.argtypes = [C.c_uint32]
        L.oracle_pcg_next.restype = C.c_uint32; L.oracle_pcg_next.argtypes = [C.POINTER(C.c_uint64)]
        L.oracle_normalized_uint.restype = C.c_float; L.oracle_normalized_uint.argtypes = [C.c_uint32]
        L.oracle_sobol_sample.restype = C.c_uint32
        L.oracle_sobol_sample.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]
        L.oracle_filter_cdf.argtypes = [C.c_uint32, C.c_void_p, C.POINTER(C.c_float)]
        L.oracle_diffuse_fresnel.restype = C.c_float; L.oracle_diffuse_fresnel.argtypes = [C.c_float, C.c_int]
        L.oracle_kat_eval.restype = C.c_int; L.oracle_kat_eval.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
        vp, u32, f32 = C.c_void_p, C.c_uint32, C.c_float
        L.oracle_bsdf_eval_lobes.restype = C.c_int
        L.oracle_bsdf_eval_lobes.argtypes = [vp, C.c_int, f32, f32, u32, vp, C.c_int, vp]
        L.oracle_bsdf_sample_lobes.restype = C.c_int
        L.oracle_bsdf_sample_lobes.argtypes = [vp, u32, u32, u32, C.c_int, vp, vp, u32, f32, f32, vp, vp, vp]
        L.oracle_light_probe_mode.restype = C.c_int
        L.oracle_light_probe_mode.argtypes = [vp, C.c_int, u32, u32, C.c_int, u32, vp, vp]
        L.oracle_choose_light.restype = C.c_int
        L.oracle_choose_light.argtypes = [vp, u32, C.c_int, vp, u32, vp, vp]
        L.oracle_shadow_probe.restype = C.c_int
        L.oracle_shadow_probe.argtypes = [vp, C.c_int, vp, vp, vp]
        L.oracle_bounce_probe.restype = C.c_int
        L.oracle_bounce_probe.argtypes = [vp, C.c_int, C.c_int, vp, vp]
        L.oracle_curve_segments_probe.restype = C.c_int
        L.oracle_curve_segments_probe.argtypes = [vp, C.c_int, vp, vp, C.c_int, vp]
        _LIB = L
    return _LIB


def sobol_table():
    p = os.path.join(_HERE, "..", "tungsten_b200", "data", "sobol_1024x32.u32")
    return np.fromfile(p, dtype="<u4").reshape(1024, 32)


class Oracle:
    def __init__(self, flat_scene):
        self.fs = flat_scene
        self._sobol = np.ascontiguousarray(sobol_table())
        self._desc = flat_scene.desc()
        err = C.create_string_buffer(512)
        self.h = lib().oracle_create(C.byref(self._desc), self._sobol.ctypes.data, err, 512)
        if not self.h:
            raise RuntimeError("oracle_create failed: %s" % err.value.decode())
        self.stats = abi.Stats()

    def close(self):
        if self.h:
            lib().oracle_destroy(self.h); self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def dice_tiles(self, seed):
        w, h = self.fs.resolution
        n = lib().oracle_dice_tiles(w, h, seed, None)
        tiles = (abi.Tile*n)()
        lib().oracle_dice_tiles(w, h, seed, tiles)
        return tiles

    def render(self, spp, seed=0xBA5EBA11, spp_begin=0, tiles=None, threads=0, mean=None, count=None):
        w, h = self.fs.resolution
        if mean is None:
            mean = np.zeros((h, w, 3), dtype=np.float32)
        if count is None:
            count = np.zeros((h, w), dtype=np.uint32)
        n = 0 if tiles is None else len(tiles)
        rc = lib().oracle_render_tiles(self.h, tiles, n, seed, spp_begin, spp, mean.ctypes.data, count.ctypes.data,
                                       threads, C.byref(self.stats))
        if rc != 0:
            raise RuntimeError("oracle_render_tiles -> %d" % rc)
        return mean, count

    def trace(self, rays):
        rays = np.ascontiguousarray(rays, dtype=np.float32).reshape(-1, 8)
        hits = (abi.Hit*len(rays))()
        lib().oracle_trace_closest(self.h, rays.ctypes.data, hits, len(rays))
        return np.ctypeslib.as_array(hits).copy() if len(rays) else np.zeros(0)

    def bounce(self, states, camera=False):
        """oracle_bounce_probe: uint32 [n, abi.BOUNCE_WORDS] path states in, the states after one loop iteration out
        (camera=True: the camera states of the records' (pixel, seed, sample))."""
        states = np.ascontiguousarray(states, dtype=np.uint32).reshape(-1, abi.BOUNCE_WORDS)
        out = np.zeros_like(states)
        rc = lib().oracle_bounce_probe(self.h, 1 if camera else 0, len(states), states.ctypes.data, out.ctypes.data)
        if rc != 0:
            raise RuntimeError("oracle_bounce_probe -> %d" % rc)
        return out

    def curve_segments(self, prim, rays, only=None):
        """oracle_curve_segments_probe: every segment of curve primitive `prim` tested alone on each ray (only: int [n], one
        segment per ray, -1 = all).  Returns a record array: n_pass (segments whose root piece passes its box test), n_hit
        (segments that report a hit), seg / t / u / w of the nearest such hit (seg -1: none), slack (where the hit point lies in
        the segment's curveBox, in units of the box's largest extent: > 0 inside)."""
        rays = np.ascontiguousarray(rays, dtype=np.float32).reshape(-1, 8)
        out = np.zeros(len(rays), CURVE_SEGMENTS_DTYPE)
        if only is not None:
            only = np.ascontiguousarray(only, dtype=np.int32)
            assert only.shape == (len(rays),)
        rc = lib().oracle_curve_segments_probe(self.h, prim, rays.ctypes.data, None if only is None else only.ctypes.data,
                                               len(rays), out.ctypes.data)
        if rc != 0:
            raise RuntimeError("oracle_curve_segments_probe: primitive %d is not a curve" % prim)
        return out


CURVE_SEGMENTS_DTYPE = np.dtype([("n_pass", "<u4"), ("n_hit", "<u4"), ("seg", "<i4"), ("t", "<f4"), ("u", "<f4"), ("w", "<f4"),
                                 ("slack", "<f4")])


def kat_eval(which, args):
    a = np.array(args, dtype=np.float32); out = np.zeros(8, dtype=np.float32)
    n = lib().oracle_kat_eval(which, a.ctypes.data, out.ctypes.data)
    return out[:n]
