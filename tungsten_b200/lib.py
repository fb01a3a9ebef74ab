"""ctypes binding of libtgb200.so.  Fails loudly if the CUDA library is missing: there is no fallback."""
import ctypes as C
import os

import numpy as np

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("TGB200_LIB", os.path.join(_HERE, "libtgb200.so"))   # TGB200_LIB: experimental variant builds
_lib = None


class TgbError(RuntimeError):
    def __init__(self, code, text):
        super().__init__("tgb200 error %d: %s" % (code, text))
        self.code = code


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError("%s is missing: build it with `python -m tungsten_b200.build` "
                          "(the CUDA library is the only implementation; there is no CPU path)" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, u32 = C.c_void_p, C.c_uint32
    L.tgb200_create.argtypes = [C.POINTER(abi.SceneDesc), C.POINTER(vp)]
    L.tgb200_render_tiles.argtypes = [vp, vp, u32, u32, u32, u32, vp, vp]
    L.tgb200_render_resident.argtypes = [vp, vp, u32, u32, u32, u32]
    L.tgb200_clear_framebuffer.argtypes = [vp]
    L.tgb200_read_framebuffer.argtypes = [vp, vp, vp]
    L.tgb200_write_framebuffer.argtypes = [vp, vp, vp]
    L.tgb200_generate_work.argtypes = [vp, u32, u32, u32, u32, C.c_int, C.POINTER(C.c_uint64)]
    L.tgb200_render_adaptive.argtypes = [vp, vp, u32, u32, vp]
    L.tgb200_framebuffer_device_ptr.argtypes = [vp, C.POINTER(vp), C.POINTER(C.c_uint64)]
    L.tgb200_trace_closest.argtypes = [vp, vp, vp, u32]
    L.tgb200_shard_tiles.argtypes = [vp, u32, vp]
    L.tgb200_pack_tiles.argtypes = [vp, vp, u32, vp]
    L.tgb200_unpack_tiles.argtypes = [vp, vp, u32, vp, u32]
    L.tgb200_get_stats.argtypes = [vp, C.POINTER(abi.Stats)]
    L.tgb200_set_profiling.argtypes = [vp, C.c_int]
    L.tgb200_set_stream.argtypes = [vp, vp]
    L.tgb200_scene_info.argtypes = [vp, C.POINTER(u32), C.POINTER(u32), C.POINTER(u32), C.POINTER(C.c_uint64), C.POINTER(u32)]
    L.tgb200_reset_stats.argtypes = [vp]
    L.tgb200_abort.argtypes = [vp]
    L.tgb200_clear_abort.argtypes = [vp]
    L.tgb200_qbvh_selftest.argtypes = [vp, u32, vp, u32, C.POINTER(u32), C.POINTER(u32), C.POINTER(C.c_uint64)]
    L.tgb200_shadow_walk_count.argtypes = [vp, u32, vp, vp, u32, u32, C.POINTER(u32), vp]
    i32, f32 = C.c_int, C.c_float
    L.tgb200_bsdf_probe.argtypes = [vp, i32, f32, f32, u32, i32, u32, vp, vp]
    L.tgb200_bsdf_sample_probe.argtypes = [vp, u32, u32, vp, vp, u32, f32, f32, u32, i32, vp, vp, vp]
    L.tgb200_light_probe.argtypes = [vp, i32, u32, u32, u32, vp, vp]
    L.tgb200_choose_light_probe.argtypes = [vp, u32, u32, vp, u32, vp, vp]
    L.tgb200_shadow_probe.argtypes = [vp, u32, vp, vp, vp]
    L.tgb200_bounce_probe.argtypes = [vp, u32, vp, vp]
    L.tgb200_bin_probe.argtypes = [vp, u32, vp, vp, vp, C.POINTER(u32)]
    L.tgb200_shade_variant.argtypes = [vp, vp]
    L.tgb200_destroy.argtypes = [vp]; L.tgb200_destroy.restype = None
    L.tgb200_last_error.argtypes = [vp]; L.tgb200_last_error.restype = C.c_char_p
    L.tgb200_abi_version.restype = u32
    _lib = L
    return L


class Context:
    """RAII wrapper of a `tgb_ctx` (one scene on one GPU)."""

    def __init__(self, flat_scene, device=-1, max_paths_in_flight=0, devices=None):
        """devices: list of CUDA ordinals -> one replica per GPU inside this process (tgb_settings::devices); tiles are dealt to
        them per render call and gathered on devices[0] over NVLink."""
        self.L = load()
        self.fs = flat_scene
        flat_scene.settings.device = device
        flat_scene.settings.max_paths_in_flight = max_paths_in_flight
        flat_scene.settings.n_devices = 0 if not devices else len(devices)
        for i, dv in enumerate(devices or []):
            flat_scene.settings.devices[i] = int(dv)
        self._desc = flat_scene.desc()
        h = C.c_void_p()
        rc = self.L.tgb200_create(C.byref(self._desc), C.byref(h))
        if rc != 0:
            raise TgbError(rc, self.L.tgb200_last_error(None).decode())
        self.h = h
        self.width, self.height = flat_scene.resolution

    def _check(self, rc):
        if rc != 0:
            raise TgbError(rc, self.L.tgb200_last_error(self.h).decode())

    def close(self):
        if getattr(self, "h", None):
            self.L.tgb200_destroy(self.h); self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def render_tiles(self, spp_count, seed=0xBA5EBA11, spp_begin=0, tiles=None, mean=None, count=None):
        """Host-buffer call (H2D of the running mean + D2H of the result inside)."""
        if mean is None:
            mean = np.zeros((self.height, self.width, 3), dtype=np.float32)
        if count is None:
            count = np.zeros((self.height, self.width), dtype=np.uint32)
        n = 0 if tiles is None else len(tiles)
        self._check(self.L.tgb200_render_tiles(self.h, tiles, n, seed, spp_begin, spp_count,
                                               mean.ctypes.data, count.ctypes.data))
        return mean, count

    def render_resident(self, spp_count, seed=0xBA5EBA11, spp_begin=0, tiles=None):
        n = 0 if tiles is None else len(tiles)
        self._check(self.L.tgb200_render_resident(self.h, tiles, n, seed, spp_begin, spp_count))

    def clear(self):
        self._check(self.L.tgb200_clear_framebuffer(self.h))

    def read_framebuffer(self):
        mean = np.zeros((self.height, self.width, 3), dtype=np.float32)
        count = np.zeros((self.height, self.width), dtype=np.uint32)
        self._check(self.L.tgb200_read_framebuffer(self.h, mean.ctypes.data, count.ctypes.data))
        return mean, count

    def write_framebuffer(self, mean, count):
        mean = np.ascontiguousarray(mean, dtype=np.float32); count = np.ascontiguousarray(count, dtype=np.uint32)
        self._check(self.L.tgb200_write_framebuffer(self.h, mean.ctypes.data, count.ctypes.data))

    def render_adaptive(self, records, seed=0xBA5EBA11, tiles=None):
        """records: ctypes array of abi.SampleRecord, one per 4x4 block (in/out)."""
        n = 0 if tiles is None else len(tiles)
        self._check(self.L.tgb200_render_adaptive(self.h, tiles, n, seed, records))

    def framebuffer_device_ptr(self):
        p = C.c_void_p(); n = C.c_uint64()
        self._check(self.L.tgb200_framebuffer_device_ptr(self.h, C.byref(p), C.byref(n)))
        return p.value, n.value

    def pack_tiles(self, tiles, dev_ptr):
        self._check(self.L.tgb200_pack_tiles(self.h, tiles, len(tiles), dev_ptr))

    def unpack_tiles(self, tiles, dev_ptr, sample_count):
        self._check(self.L.tgb200_unpack_tiles(self.h, tiles, len(tiles), dev_ptr, sample_count))

    def trace_closest(self, rays):
        rays = np.ascontiguousarray(rays, dtype=np.float32).reshape(-1, 8)
        hits = (abi.Hit*max(len(rays), 1))()
        self._check(self.L.tgb200_trace_closest(self.h, rays.ctypes.data, hits, len(rays)))
        return np.ctypeslib.as_array(hits)[:len(rays)].copy()

    def bounce_probe(self, states):
        """tgb200_bounce_probe: uint32 [n, abi.BOUNCE_WORDS] path states in, the states after one wavefront iteration out."""
        states = np.ascontiguousarray(states, dtype=np.uint32).reshape(-1, abi.BOUNCE_WORDS)
        out = np.zeros_like(states)
        self._check(self.L.tgb200_bounce_probe(self.h, len(states), states.ctypes.data, out.ctypes.data))
        return out

    def bin_probe(self, keys):
        """tgb200_bin_probe: uint32 keys of n survivors (abi.BINS: not traversed) in, (order[:n_sorted], cursors [abi.BINS],
        n_sorted) of the survivor sort out."""
        keys = np.ascontiguousarray(keys, dtype=np.uint32).reshape(-1)
        order = np.zeros(max(len(keys), 1), np.uint32)
        cursors = np.zeros(abi.BINS, np.uint32)
        n_sorted = C.c_uint32()
        self._check(self.L.tgb200_bin_probe(self.h, len(keys), keys.ctypes.data, order.ctypes.data, cursors.ctypes.data,
                                            C.byref(n_sorted)))
        return order[:min(n_sorted.value, len(keys))], cursors, n_sorted.value

    def shade_variant(self):
        """The k_shade instantiation the context renders with, as its template arguments: '<CURVES, MATSORT, LS>'."""
        v = np.zeros(4, np.uint32)
        self._check(self.L.tgb200_shade_variant(self.h, v.ctypes.data))
        return "<%s, %s, %d>" % ("true" if v[0] else "false", "true" if v[1] else "false", int(v[2]))

    def shade_emitters(self):
        """The emitter set of that instantiation (its ES argument): 1 = quad lights only, constant textures; else 0."""
        v = np.zeros(4, np.uint32)
        self._check(self.L.tgb200_shade_variant(self.h, v.ctypes.data))
        return int(v[3])

    def stats(self):
        s = abi.Stats()
        self._check(self.L.tgb200_get_stats(self.h, C.byref(s)))
        return s

    def reset_stats(self):
        self._check(self.L.tgb200_reset_stats(self.h))

    def set_stream(self, cuda_stream):
        """Run on the caller's CUDA stream (e.g. torch.cuda.current_stream().cuda_stream); None = the context's own."""
        self._check(self.L.tgb200_set_stream(self.h, cuda_stream))

    def set_profiling(self, on):
        self._check(self.L.tgb200_set_profiling(self.h, 1 if on else 0))

    def scene_info(self):
        a, b, c, d, e = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint64(), C.c_uint32()
        self._check(self.L.tgb200_scene_info(self.h, C.byref(a), C.byref(b), C.byref(c), C.byref(d), C.byref(e)))
        return {"n_tris": a.value, "n_nodes": b.value, "bvh_depth": c.value, "geom_bytes": d.value, "capacity": e.value}

    def abort(self):
        self.L.tgb200_abort(self.h)

    def clear_abort(self):
        self.L.tgb200_clear_abort(self.h)
