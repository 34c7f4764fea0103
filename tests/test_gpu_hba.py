"""Hierarchical BA on one batch (balm_b200.hba): the pyramid built with the device merge is bitwise the one built with the
numpy keyframes, its final poses are the matrix restatement of the propagation, and on a drifting trajectory the upper
layers remove drift that the bottom layer alone leaves in place."""
import os

import numpy as np
import pytest

import hba_ref
from balm_b200 import drivers, hba, io

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "realworld_points_small.npz")


def _host_merge(self, scans, windows, poses_list, voxel_size):
    return [hba_ref.keyframe_ref(scans, w, p, voxel_size) for w, p in zip(windows, poses_list)]


def _run(monkeypatch, scans, poses, host, **kw):
    """hba() with every registration recorded, keyframes from the device or from keyframe_ref."""
    from balm_b200 import Batch
    regs, cut = [], Batch.cut_scans

    def recorded_cut(self, *a, **k):
        out = cut(self, *a, **k)
        regs.append(self.download_voxels(with_keys=True))
        return out
    with monkeypatch.context() as m:
        m.setattr(Batch, "cut_scans", recorded_cut)
        if host:
            m.setattr(Batch, "merge_scans", _host_merge)
        res = hba.hba(scans, poses, **kw)
    return res, regs


def _bottom_only(layers):
    """Every window's anchor left at its input pose: the upper layers change nothing."""
    flat = [dict(lay) for lay in layers]
    for lay in flat[1:]:
        lay["poses"] = [lay["poses_in"][w] for w in lay["windows"]]
    return hba_ref.propagate_ref(flat)


@pytest.fixture(scope="module")
def drift():
    return hba_ref.drift_scene()


def test_device_pyramid_equals_host_pyramid_and_propagation(drift, monkeypatch):
    scans, gt, init = drift
    dev, regs_d = _run(monkeypatch, scans, init, host=False)
    ref, regs_h = _run(monkeypatch, scans, init, host=True)
    assert [len(lay["windows"]) for lay in dev["layers"]] == [11, 1] and len(regs_d) == len(regs_h) == 2
    assert np.array_equal(dev["poses"], ref["poses"])
    for a, b in zip(dev["layers"], ref["layers"]):
        assert a["windows"] == b["windows"] and a["status"] == b["status"] and a["n_iters"] == b["n_iters"]
        assert a["kf_sizes"] == b["kf_sizes"] and a["n_voxels"] == b["n_voxels"]
        assert all(np.array_equal(x, y) for x, y in zip(a["poses"], b["poses"]))
        assert np.array_equal(a["poses_in"], b["poses_in"])
    for rd, rh in zip(regs_d, regs_h):
        assert all(all(np.array_equal(x[k], y[k]) for k in x) for x, y in zip(rd, rh))
    assert all(st == 0 for lay in dev["layers"] for st in lay["status"])
    F = hba_ref.propagate_ref(dev["layers"])
    assert np.abs(dev["poses"] - F).max() <= 1e-12 * max(1.0, np.abs(F).max())
    assert np.abs(dev["poses"][0] - init[0]).max() <= 1e-12           # the top's slot 0 keeps the input world frame


def test_upper_layers_remove_drift(drift):
    scans, gt, init = drift
    res = hba.hba(scans, init)
    rot0, tran0 = drivers.rsme(init, gt)
    rot1, tran1 = drivers.rsme(_bottom_only(res["layers"]), gt)
    rot, tran = drivers.rsme(res["poses"], gt)
    print("drift RMSE rot [deg] / tran [m]: initial %.4f / %.4f, bottom layer only %.4f / %.4f, hba %.4f / %.4f"
          % (np.degrees(rot0), tran0, np.degrees(rot1), tran1, np.degrees(rot), tran))
    # measured on an H100: initial 0.863 deg / 0.0975 m, bottom layer only 0.759 deg / 0.0865 m, hba 0.0113 deg / 0.0012 m
    assert rot < 0.1 * rot0 and tran < 0.1 * tran0
    assert rot < 0.1 * rot1 and tran < 0.1 * tran1


def test_realworld_slice_end_to_end():
    d = np.load(GOLD)
    n = len(d["poses"])
    scans = [d["xyz"][d["frame"] == i].astype(np.float32) for i in range(n)]
    res = hba.hba(scans, np.asarray(d["poses"], dtype=np.float64), top_size=8)
    lays = res["layers"]
    assert [len(lay["windows"]) for lay in lays] == [4, 1] and lays[1]["windows"] == [[0, 1, 2, 3]]
    assert all(k > 0 for k in lays[0]["kf_sizes"]) and lays[1]["kf_sizes"] is None
    assert res["poses"].shape == (24, 12) and np.all(np.isfinite(res["poses"]))
    assert np.abs(res["poses"] - hba_ref.propagate_ref(lays)).max() <= 1e-12 * max(1.0, np.abs(res["poses"]).max())


def test_cli_gives_the_function_poses(tmp_path, capsys):
    from test_drivers import _write_dataset
    _write_dataset(tmp_path, n_poses=24, pts=4000)
    out = tmp_path / "refined.csv"
    assert hba.main(["--file_path", str(tmp_path), "--top_size", "8", "--out", str(out)]) == 0
    text = capsys.readouterr().out
    assert "The size of poses: 24" in text and "layer 1: 1 windows" in text
    R, p, _, scans = io.read_realworld_dir(str(tmp_path))
    R0, p0 = R[0].copy(), p[0].copy()
    x = drivers.pack_poses(np.einsum("ji,njk->nik", R0, R), (p - p0) @ R0)
    want = hba.hba(scans, x, top_size=8)["poses"]
    Rf, pf, _ = io.read_pose_csv(out)
    assert np.array_equal(drivers.pack_poses(Rf, pf), want)
