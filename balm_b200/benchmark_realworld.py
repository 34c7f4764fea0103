"""python -m balm_b200.benchmark_realworld --file_path DIR [--voxel_size 2]

Headless run of the reference's real-world benchmark (src/benchmark/benchmark_realworld.cpp; parameters of
launch/benchmark_realworld.launch:4-5). DIR holds alidarPose.csv and full<i>.pcd."""
import argparse
import sys

import numpy as np

from . import _lib as L
from . import drivers, io


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--file_path", required=True, help="directory with alidarPose.csv and full<i>.pcd")
    ap.add_argument("--voxel_size", type=float, default=2.0, help="root voxel edge (launch file: 2; code default 1)")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--precision", choices=["tensor", "fp64"], default="tensor")
    ap.add_argument("--max_scans", type=int, default=None, help="use only the first scans (window size)")
    ap.add_argument("--out", default=None, help="write the refined poses in alidarPose.csv format")
    ap.add_argument("--cloud_out", default=None, help="write the refined map (what the reference publishes on /map_show) as .pcd")
    ap.add_argument("--path_out", default=None, help="write the refined trajectory (/map_path) as .pcd")
    drivers.add_voxel_loss_args(ap)
    a = ap.parse_args(argv)
    res = drivers.benchmark_realworld(a.file_path, a.voxel_size, a.device,
                                      L.PREC_TENSOR if a.precision == "tensor" else L.PREC_FP64, a.max_scans,
                                      keep_scans=bool(a.cloud_out or a.path_out),
                                      voxel_loss=drivers.voxel_loss_arg(ap, a))
    if res is None:
        return 0  # the reference exits with status 0 when the plane guard fires (:208, bavoxel.hpp:1084)
    if a.out:
        R, p = drivers.unpack_poses(res["poses"])
        io.write_pose_csv(a.out, R, p)
        print("refined poses ->", a.out)
    if a.cloud_out or a.path_out:
        print("\nRefined point cloud is publishing...")  # :228-231, written to files instead
        cloud, path = drivers.data_show(res["poses"], res["scans"])
        if a.cloud_out:
            io.write_pcd(a.cloud_out, cloud)
        if a.path_out:
            io.write_pcd(a.path_out, path, intensity=None)
        print("\nRefined point cloud is published.")
    return 0


if __name__ == "__main__":
    sys.exit(main())
