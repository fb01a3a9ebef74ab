"""The any-hit shadow walk: order-free and started below the top-level cut.

k_shadow_bvh walks an occlusion query from the cut boxes its segment enters, entering the nearest hit child and pushing the others
unsorted.  The host test counts that walk against the old one (sorted, from the root) with tgb200_shadow_walk_count and checks the
traversal stack bound that tgb200_create applies; the GPU test runs the renderer's own shadow kernels with the cut entry on and off
(TGB_SHADOW_CUT_ENTRY=0 starts every query at the root) and requires identical results.
"""
import os
import sys

import numpy as np
import pytest

from tungsten_b200 import abi, lib, scene, synth

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import shadow_walk_count as swc  # noqa: E402

F = np.float32


def _room(scratch):
    fs = scene.load_scene(synth.cornell_mesh(scratch, res=(32, 32), spp=1, subdiv=4))
    return fs, swc.c1_queries(fs, np.random.RandomState(3), 20000)


def test_cut_walk_agrees_with_the_root_walk_and_visits_fewer_nodes(scratch):
    fs, (tris, q) = _room(scratch)
    rc, need, out = swc.walk_counts(tris, F(fs.camera.pos), q)
    agree, text = swc.summary(out)
    print(text)
    walked = out[:, 0] != 0
    assert rc == abi.TGB_OK and walked.sum() > 1000 and agree
    assert out[walked, 1].max() <= need                                # the bound covers the deepest stack the walk reached
    assert out[walked, 7].sum() < out[walked, 3].sum()                 # node visits: from the cut < from the root


def test_stack_bound_rejects_a_tree_deeper_than_the_stack(scratch):
    fs, (tris, q) = _room(scratch)
    rc, need, _ = swc.walk_counts(tris, F(fs.camera.pos), q[:16])
    assert rc == abi.TGB_OK and need > 8
    rc, need2, _ = swc.walk_counts(tris, F(fs.camera.pos), q[:16], stack_size=need - 1)
    assert rc == abi.TGB_ERR_UNSUPPORTED and need2 == need
    rc, _, _ = swc.walk_counts(tris, F(fs.camera.pos), q[:16], stack_size=need)
    assert rc == abi.TGB_OK


def test_walk_count_follows_the_build_switches(scratch, monkeypatch):
    # TGB_TRI_LEAF changes the tree tgb200_create builds, so it must change the tree the host count walks
    fs, (tris, q) = _room(scratch)
    monkeypatch.delenv("TGB_TRI_LEAF", raising=False)
    totals = []
    for leaf in (None, "2"):
        if leaf:
            monkeypatch.setenv("TGB_TRI_LEAF", leaf)
        rc, _, out = swc.walk_counts(tris, F(fs.camera.pos), q)
        agree, _ = swc.summary(out)
        assert rc == abi.TGB_OK and agree
        totals.append(out[:, [3, 5, 7, 9]].astype(np.int64).sum(0))   # node visits, triangle tests: root walk, cut walk
    print("node visits / triangle tests (root, cut): leaf cap 4 %s, leaf cap 2 %s" % tuple(totals))
    assert not np.array_equal(totals[0], totals[1])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cube_city", "many_lights", "hair"])
def test_cut_entry_does_not_change_shadow_queries(name, scratch, monkeypatch):
    import test_gpu_shadow as S
    from oracle import pyoracle
    fs = S._scene(name, scratch)
    outs = []
    for entry in ("1", "0"):
        monkeypatch.setenv("TGB_SHADOW_CUT_ENTRY", entry)
        ctx = lib.Context(fs)
        if not outs:
            orc = pyoracle.Oracle(fs)
            q, lm, _ = S.build_queries(fs, ctx, orc, seed=21)
            orc.close()
        outs.append(S.gpu_probe(ctx, q, lm))
        ctx.close()
    a, b = outs
    print("%s: %d queries, %d reached the BVH pass, identical with the cut entry on and off: %s"
          % (name, len(q), int((a[:, 6] == 2).sum()), np.array_equal(a.view(np.uint32), b.view(np.uint32))))
    assert (a[:, 6] == 2).any()
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
