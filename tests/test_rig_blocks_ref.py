"""The block-sparse rig's restatement (rig_blocks_ref) against the dense rig restatement (rig_ref.evaluate): the rig
pattern and the two-pass reduction from slot blocks give H_rig's blocks and g_rig on rig_case's scenes and on a rig
scene cut into voxels; every nonzero block of the dense H_rig lies on the pattern; on a rig corridor the
nested-dissection ordering puts every free extrinsic in the root separator."""
import numpy as np
import pytest

import block_hessian_ref as bh
import nd_symbolic_ref as nd
import rig_blocks_ref as rb
import rig_ref as rr
from test_gpu_rig import rig_case


def _check(sc, base, ext, base_of, lidar_of, var, include_fix=False):
    X = rr.compose(base, ext, base_of, lidar_of)
    spairs, sblocks, g, _ = bh.evaluate(sc, X, include_fix)
    Hd, gd, _, HX, gX = rr.evaluate(sc, base, ext, base_of, lidar_of, var, include_fix)
    scale = np.abs(Hd).max()
    # the slot blocks of both restatements agree to rounding (the fix scene's cancellation costs a few digits)
    assert np.abs(sblocks - bh.blocks_of(HX, spairs)).max() < 1e-11 * np.abs(HX).max()
    pairs, blocks, gr = rb.reduce(spairs, bh.blocks_of(HX, spairs), gX, base, base_of, lidar_of, var)
    assert np.abs(blocks - bh.blocks_of(Hd, pairs)).max() < 1e-12 * scale
    assert np.abs(gr - gd).max() < 1e-12 * max(np.abs(gd).max(), scale)
    on = np.zeros((len(var), len(var)), dtype=bool)
    on[pairs[:, 0], pairs[:, 1]] = on[pairs[:, 1], pairs[:, 0]] = True
    nz = np.abs(Hd.reshape(len(var), 6, len(var), 6)).max(axis=(1, 3)) > 0
    assert not (nz & ~on).any()
    return pairs


@pytest.mark.parametrize("name", ["dense", "ragged", "fix"])
@pytest.mark.parametrize("fixed_lidars", [(0,), ()])
def test_reduction_matches_dense_rig(name, fixed_lidars):
    sc, base_of, lidar_of, base, ext = rig_case(name)
    var = rr.unknowns(len(base), 2, fixed_lidars=fixed_lidars)
    for include_fix in ((False, True) if sc.get("fix10") is not None else (False,)):
        _check(sc, base, ext, base_of, lidar_of, var, include_fix)


def test_reduction_on_rig_scene_with_fixed_base():
    S = rr.rig_scene(n_base=4, pts_draw=4000)
    base, ext = rr.perturbed_start(S)
    sc = rr.cut(S, base, ext)
    var = rr.unknowns(len(base), 3, fixed_bases=(1,))
    pairs = _check(sc, base, ext, S["base_of"], S["lidar_of"], var)
    assert len(pairs) <= len(var) * (len(var) + 1) // 2


def test_corridor_pattern_and_ordering():
    B, L, w = 120, 3, 4
    sc = rb.rig_corridor(B, L, w)
    N = B * L
    spairs = bh.pairs_from_csr(N, sc["row_ptr"], sc["pose_idx"])
    for fixed_lidars in ((0,), ()):
        var = rr.unknowns(B, L, fixed_lidars=fixed_lidars)
        pairs = rb.pattern(spairs, sc["base_of"], sc["lidar_of"], B, var)
        F = len(var)
        ext = list(range(B, F))
        # bases pair with the bases within +-2w (their slots share a plane) and with every free extrinsic
        band = {(u, v) for u in range(B) for v in range(u, min(B, u + 2 * w + 1))}
        assert {(int(u), int(v)) for u, v in pairs if v < B} == band
        assert all((u, e) in {(int(a), int(b)) for a, b in pairs} for u in range(B) for e in ext)
        order = nd.nd_order(F, nd.adjacency(F, pairs))
        assert order[-len(ext):] == ext  # the root separator's highest indices: every free extrinsic
        sym = nd.symbolic(F, pairs)
        assert sym["levels"] >= len(ext)
