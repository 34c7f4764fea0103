"""balm_b200 -- H100-native (sm_90a) implementation of the BALM 2.0 bundle-adjustment hot path
(VOX_HESS factor evaluation + BALM2::damping_iter) behind the reference's own call surface.

The arithmetic lives in libbalm_b200.so (hand-written CUDA, C ABI in include/balm_b200.h); importing the
package does not load it, using any class does, and fails loudly if the library has not been built.
"""
from . import _lib
from ._lib import PREC_BLOCKS, PREC_FP64, PREC_TENSOR, BalmError
from .context import Batch, Context, PoseGraph
from .factors import odometry_factors, pose_priors, position_priors
from .rig import calibrate_rig, rig_poses
from . import bavoxel
from . import shard
from . import io
from . import drivers
from .bavoxel import BALM2, IMUST, VOX_HESS, PointCluster

__all__ = ["Context", "Batch", "PoseGraph", "BALM2", "VOX_HESS", "IMUST", "PointCluster", "PREC_FP64", "PREC_TENSOR", "PREC_BLOCKS",
           "BalmError", "odometry_factors", "pose_priors", "position_priors", "calibrate_rig", "rig_poses",
           "bavoxel", "shard", "io", "drivers"]
