"""The emitter set of the all-Lambert k_shade: scenes whose surfaces are all Lambert, whose lights are all quads, with no infinite
emitter and only constant albedo and emission textures shade with k_shade<false, false, 1, 1>, which compiles none of the other
emitters' or textures' code.  Everything else that is all-Lambert keeps k_shade<false, false, 1>.

  * the choice, for named scenes and for near-misses that must stay on the general kernel (a checker albedo, a mesh light, an
    environment light), through Context.shade_variant() (unchanged: '<false, false, 1>' for all of them) and
    Context.shade_emitters();
  * the near-misses still match the CPU oracle (the bars of test_gpu_parity.py's all-Lambert scenes);
  * the new kernel renders bit for bit what the parent library rendered with the general all-Lambert kernel: images at the
    sample indices on both sides of 256 and 65536 (the Sobol index's scrambled low byte wraps there), and single bounces from
    states at sampler dimensions 1015..1030 (the switch to the PCG fallback at 1024).  The references under
    tests/golden/quad_emitters/ were recorded with `python tests/test_gpu_emitters.py --record DIR` on an H100 with the library
    of the commit before the emitter set existed.
"""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import pyoracle  # noqa: E402
from tungsten_b200 import abi, lib, scene, synth  # noqa: E402

gpu = pytest.mark.gpu

GOLDEN = os.path.join(ROOT, "tests", "golden", "quad_emitters")
SEED = 0xBA5EBA11
RES = (32, 32)
# (first sample, samples) of the recorded images: 254..257 and 65534..65537
SAMPLE_RANGES = ((254, 4), (65534, 4))
N_STATES = 2048


def _checker_albedo(out_dir):
    sc = synth.cornell_box(res=RES, spp=1)
    for b in sc["bsdfs"]:
        if b["name"] == "floor":
            b["albedo"] = {"type": "checker", "on_color": [0.8, 0.8, 0.8], "off_color": [0.15, 0.15, 0.2], "res_u": 8, "res_v": 8}
    return scene.load_scene(sc)


def _mesh_light(out_dir):
    v, t = synth.grid_mesh(2, 2, 1.0)
    sc = synth.cornell_box(res=RES, spp=1, extra_bsdfs=[{"name": "lamp", "type": "null", "albedo": 1.0}],
                           extra_prims=[{"name": "lamp", "type": "mesh", "file": "emit_lamp.wo3", "smooth": False, "bsdf": "lamp",
                                         "emission": [3.0, 4.0, 6.0],
                                         "transform": {"position": [0.93, 1.0, -0.3], "scale": [0.3, 0.3, 0.3],
                                                       "rotation": [0, 0, 90]}}])
    return scene.load_scene(synth.write_scene(out_dir, "emit_mesh_light", sc, {"emit_lamp.wo3": (v, t)}))


def _env_light(out_dir):
    sc = synth.cornell_box(res=RES, spp=1)
    sc["primitives"].append({"name": "env", "type": "infinite_sphere", "emission": [0.3, 0.4, 0.5], "sample": True,
                             "transform": {"rotation": [0, 40, 0]}})
    return scene.load_scene(sc)


# name -> (scene builder, shade_emitters())
SCENES = {
    "cornell_box": (lambda d: scene.load_scene(synth.cornell_box(res=RES, spp=1)), 1),
    "cornell_mesh": (lambda d: scene.load_scene(synth.cornell_mesh(d, name="emit_mesh", res=RES, spp=1)), 1),
    "cube_city": (lambda d: scene.load_scene(synth.cube_city(res=RES, spp=1, n=12)), 1),
    "many_lights": (lambda d: scene.load_scene(synth.many_lights(d, name="emit_ml", res=RES, spp=1)), 0),
    "checker_albedo": (_checker_albedo, 0),
    "mesh_light": (_mesh_light, 0),
    "env_light": (_env_light, 0),
}
NEAR_MISSES = ["checker_albedo", "mesh_light", "env_light"]
RECORDED = ["cornell_box", "cornell_mesh"]


def camera_states(fs, orc, n):
    """Camera states of n (pixel, sample) pairs, as test_gpu_bounce.py makes them (pixel i % pixels, sample i // pixels)."""
    w, h = fs.resolution
    seeds = np.zeros(w*h, np.uint32)
    for t in orc.dice_tiles(SEED):
        for y in range(t.y, t.y + t.h):
            seeds[y*w + t.x: y*w + t.x + t.w] = t.sampler_seed
    k = np.arange(n)
    rec = np.zeros((n, abi.BOUNCE_WORDS), np.uint32)
    rec[:, abi.BR_PIXEL] = k % (w*h); rec[:, abi.BR_SEED] = seeds[k % (w*h)]; rec[:, abi.BR_SAMPLE] = k//(w*h)
    return orc.bounce(rec, camera=True)


def probe_states(fs):
    """Camera states with their sample index set to 255 / 256 / 65535 / 65536 and, for half of them, the sampler's dimension to
    1015..1030."""
    orc = pyoracle.Oracle(fs)
    s = camera_states(fs, orc, N_STATES)
    orc.close()
    rng = np.random.RandomState(7)
    s[:, abi.BR_SAMPLE] = np.array([255, 256, 65535, 65536], np.uint32)[np.arange(N_STATES) % 4]
    deep = np.arange(N_STATES) % 8 >= 4
    s[deep, abi.BR_DIMENSION] = rng.randint(1015, 1031, int(deep.sum()))
    return s


def outputs(name, scratch, states=None):
    """What the recorded files hold: the images of SAMPLE_RANGES (mean, count) and one bounce of `states` (default probe_states)."""
    fs = SCENES[name][0](scratch)
    ctx = lib.Context(fs)
    out = {}
    for first, n in SAMPLE_RANGES:
        mean, count = ctx.render_tiles(n, seed=SEED, spp_begin=first)
        out["mean_%d" % first] = mean; out["count_%d" % first] = count
    s = probe_states(fs) if states is None else states
    out["states"] = s; out["bounce"] = ctx.bounce_probe(s)
    ctx.close()
    return out


def record(out_dir):
    import tempfile
    d = tempfile.mkdtemp(prefix="tgb_emit_")
    for name in RECORDED:
        os.makedirs(os.path.join(out_dir, name), exist_ok=True)
        for k, v in outputs(name, d).items():
            np.save(os.path.join(out_dir, name, k + ".npy"), v)


@gpu
@pytest.mark.parametrize("name", list(SCENES))
def test_emitter_set_choice(name, scratch):
    ctx = lib.Context(SCENES[name][0](scratch))
    assert ctx.shade_variant() == "<false, false, 1>"
    assert ctx.shade_emitters() == SCENES[name][1]
    ctx.close()


@gpu
@pytest.mark.parametrize("name", NEAR_MISSES)
def test_near_misses_match_oracle(name, scratch):
    fs = SCENES[name][0](scratch)
    o = pyoracle.Oracle(fs)
    ref, rcnt = o.render(8)
    ctx = lib.Context(fs)
    img, cnt = ctx.render_tiles(8)
    d = np.abs(img - ref).max(axis=2)
    frac = float((d <= 1e-5*(1.0 + np.abs(ref).max(axis=2))).mean())
    rmse = float(np.sqrt(((img - ref)**2).mean()))
    print("%s: k_shade%s emitters %d, frac within tol %.5f, rmse %.3e, mean %.4f" % (
        name, ctx.shade_variant(), ctx.shade_emitters(), frac, rmse, float(ref.mean())))
    assert np.array_equal(cnt, rcnt)
    assert frac >= 0.999 and rmse <= 1e-4*max(float(ref.mean()), 1e-3)
    ctx.close(); o.close()


@gpu
@pytest.mark.parametrize("name", RECORDED)
def test_same_output_as_the_general_kernel(name, scratch):
    fs = SCENES[name][0](scratch)
    ctx = lib.Context(fs)
    assert ctx.shade_emitters() == 1
    ctx.close()
    got = outputs(name, scratch, states=np.load(os.path.join(GOLDEN, name, "states.npy")))
    for k, v in got.items():
        want = np.load(os.path.join(GOLDEN, name, k + ".npy"))
        assert v.dtype == want.dtype and v.shape == want.shape, k
        assert np.array_equal(v.view(np.uint32), want.view(np.uint32)), "%s: %s differs from the recorded output" % (name, k)
    deep = got["states"][:, abi.BR_DIMENSION] >= 1015
    crossed = deep & (got["states"][:, abi.BR_DIMENSION] < 1024) & (got["bounce"][:, abi.BR_DIMENSION] >= 1024)
    print("%s: %d states from dimension 1015..1030, %d crossed into the PCG fallback" % (name, int(deep.sum()), int(crossed.sum())))
    assert crossed.sum() > 50


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "--record":
        record(sys.argv[2])
    else:
        sys.exit("usage: python tests/test_gpu_emitters.py --record DIR")
