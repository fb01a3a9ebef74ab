"""A render's query and hit counters, and its image, against values recorded when every warp (and every blocked shadow query)
added to the counters on its own.

The wavefront kernels add their counts to the statistics block, and allocate the entries of the shadow and survivor queues,
with one atomic per block or per traversal warp.  The images in the other tests would not notice a partial sum that was lost
or added twice, so this test pins both the counters and the framebuffer of two small renders: the Cornell box with the
displaced mesh (quad light, any-hit shadow queries) and the material room (several BSDFs).
"""
import hashlib

import numpy as np
import pytest

from tungsten_b200 import lib, scene, synth

pytestmark = pytest.mark.gpu

SPP = 16

# samples, rays, hits, path_rays, shadow_rays, sha256 of the mean (float32) then the count (uint32) framebuffer
PINNED = {
    "cornell_mesh": {"samples": 65536, "rays": 178049, "hits": 86235, "path_rays": 128867, "shadow_rays": 49182,
                     "image_sha256": "16996371d1781261861862150353e22477febe379087dc6eca07f16c2abbea8f"},
    "material_room": {"samples": 65536, "rays": 213392, "hits": 133181, "path_rays": 123711, "shadow_rays": 89681,
                      "image_sha256": "71e568ef183b220b6e851b09935a5c67decf9bd3f46ee4cc68132163f6973cd7"},
}


def make_scene(name, out_dir):
    if name == "cornell_mesh":
        return scene.load_scene(synth.cornell_mesh(out_dir, res=(64, 64), spp=SPP, subdiv=4))
    return scene.load_scene(synth.material_room(out_dir, res=(64, 64), spp=SPP, max_bounces=16, subdiv=3))


def render_counters(name, out_dir):
    ctx = lib.Context(make_scene(name, out_dir), device=0)
    try:
        mean, count = ctx.render_tiles(SPP)
        st = ctx.stats()
        h = hashlib.sha256(np.ascontiguousarray(mean, np.float32).tobytes() + np.ascontiguousarray(count, np.uint32).tobytes())
        return {"samples": int(st.samples), "rays": int(st.rays), "hits": int(st.hits), "path_rays": int(st.path_rays),
                "shadow_rays": int(st.shadow_rays), "image_sha256": h.hexdigest()}
    finally:
        ctx.close()


@pytest.mark.parametrize("name", sorted(PINNED))
def test_counters_and_image_pinned(name, tmp_path):
    got = render_counters(name, str(tmp_path))
    assert got == PINNED[name]
